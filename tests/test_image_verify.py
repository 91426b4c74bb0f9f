"""fma_image_verify: a sleeping image is checked against the digests it carries, where it lies, without a wake.  The device tests
(-m gpu on an H100) run plain and PACKED images (bf16 pages from tests/pagegen.py: most pages code, some stay raw) in every tier,
damage one stored page in the host store, a file or a parking buffer and expect exactly that segment back, and check that nothing
else moves.  test_image_verify_against_the_host_simulated_engine runs the same tests on CPU against the host-simulated engine.
K6 itself runs against the oracle on the CPU execution model (plain and ThreadSanitizer) and on the device."""
import ctypes as C
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_resident_share import _check_restored, _load

PAGE = 2 << 20
FMA_PAGE = PAGE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cpp", "cuda_emu")
SIM = os.path.join(ROOT, "tests", "cpp", "hostsim")
CSRC = os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc")
gpu = pytest.mark.gpu
HOSTSIM = os.environ.get("FMA_HOSTSIM") == "1"


def _L():
    from fma_b200 import _lib as L

    return L


TIERS = ["host", "local", "file_buffered", "file_direct", "host_resident", "peer"]


def _sleep(engine, tier, tmp_path, monkeypatch, nbytes):
    L = _L()
    path = str(tmp_path / "v.fmaimg")
    t = {"host": L.FMA_TIER_HOST, "host_resident": L.FMA_TIER_HOST, "local": L.FMA_TIER_LOCAL, "peer": L.FMA_TIER_PEER}.get(tier, L.FMA_TIER_FILE)
    if tier.startswith("file"):
        monkeypatch.setenv("FMA_FILE_BUFFERED", "1" if tier == "file_buffered" else "0")
        engine.set_option("load_chunk_bytes", 4 << 20)     # several windows, each holding whole stored pages
        engine.set_option("load_slots", 3)
        engine.file_store(path)
    if tier == "host_resident":
        engine.set_option("resident_bytes", 24 << 20)
    if tier == "peer":
        try:
            engine.peer_reserve(1, nbytes)
        except L.FmaError as e:
            if e.code == L.FMA_EINVAL and "not visible" in e.message:
                pytest.skip("the peer tier needs a second GPU")
            raise
    engine.sleep(["weights"], tier=t, flags=L.FMA_FLAG_VERIFY)
    return path


def _with_raw_pages(engine, ref):
    """Noise in the first page of the first, a middle and the last weight segment: in a PACKED image those pages stay raw (K3)
    among coded ones (K6)."""
    widx = sorted(ref)
    rng = np.random.default_rng(11)
    for i in (widx[0], widx[len(widx) // 2], widx[-1]):
        ref[i] = ref[i].copy()
        ref[i].view(np.uint8)[:PAGE] = rng.integers(0, 256, PAGE, dtype=np.uint8)
        engine.write(i, ref[i].tobytes())


def _free_hbm():
    """Free device memory as the driver reports it (cudaMemGetInfo through torch); None on the host-simulated engine."""
    if HOSTSIM:
        return None
    import torch

    return torch.cuda.mem_get_info(0)[0]


def _snapshot(engine):
    st = engine.stats()
    keep = {k: st[k] for k in ("hbm_mapped_bytes", "host_store_bytes", "image_store_bytes", "tier", "image_packed", "parked_bytes",
                               "total_kernel_launches", "total_copy_ops", "wake_bytes_restored", "sleep_bytes_copied")}
    return keep, [dataclasses.astuple(s) for s in engine.segments()]


def _rows(engine):
    rows = engine.timeline()
    assert rows and all(r["op"] == "verify" for r in rows)
    return rows


def _verify_unchanged(engine):
    """verify_image, and everything the engine reports is as it was"""
    before = _snapshot(engine)
    bad = engine.verify_image()
    assert _snapshot(engine) == before
    return bad


@gpu
@pytest.mark.parametrize("tier", TIERS)
@pytest.mark.parametrize("pack", [0, 1])
def test_intact_image_verifies_in_every_tier(engine, oracle, tmp_path, monkeypatch, pack, tier):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    if pack:
        _with_raw_pages(engine, ref)
    engine.set_option("pack", pack)
    engine.set_option("chunk_bytes", 8 << 20)               # several launches per store
    W = sum(r.size for r in ref.values())
    _sleep(engine, tier, tmp_path, monkeypatch, W)
    if tier == "host_resident":
        assert any(s.tier == L.FMA_TIER_LOCAL for s in engine.segments() if s.has_backup)
    if pack:
        assert FMA_PAGE in engine.image_pages()[1] and 0 < engine.stats()["image_store_bytes"] < W   # coded pages and raw ones
    free0 = _free_hbm()
    assert _verify_unchanged(engine) == []
    if free0 is not None:
        assert _free_hbm() >= free0                          # no HBM taken: the kernels read every store in place
    rows = _rows(engine)
    kinds = {r["kind"] for r in rows}
    assert kinds <= {"file_io", "kernel", "total"} and "kernel" in kinds and "total" in kinds
    assert ("file_io" in kinds) == tier.startswith("file")
    if tier.startswith("file"):
        fio = [r for r in rows if r["kind"] == "file_io"][0]
        assert fio["bytes"] == engine.stats()["image_store_bytes"]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


def _page_of(engine, seg, coded):
    """(store offset, stored bytes) of a page of segment `seg` that is coded / raw in the PACKED layout (any page when plain)"""
    s = engine.segment(seg)
    off, nb = engine.image_pages()
    first = s.packed_offset // PAGE
    for p in range(first, first + s.bytes // PAGE):
        if coded is None or (nb[p] != PAGE) == coded:
            return off[p], nb[p]
    return None


def _flip_host(engine, off):
    base, n = engine.host_store_view()
    b = (C.c_uint8 * 1).from_address(base + off)
    b[0] ^= 0x04


def _flip_file(path, off):
    with open(path, "r+b") as f:
        f.seek(off)
        v = f.read(1)[0]
        f.seek(off)
        f.write(bytes([v ^ 0x04]))


@gpu
@pytest.mark.parametrize("where", ["host", "file", "local"])
@pytest.mark.parametrize("which", ["first", "last"])
@pytest.mark.parametrize("page", ["plain", "coded", "raw"])
def test_one_flipped_bit_is_found_in_its_segment(engine, oracle, tmp_path, monkeypatch, page, which, where):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=page != "plain")
    if page == "raw":
        _with_raw_pages(engine, ref)
    widx = sorted(ref)
    engine.set_option("pack", 0 if page == "plain" else 1)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)   # host tier first: its store is where the bit is flipped, then moved
    order = sorted(widx, key=lambda i: engine.segment(i).packed_offset)
    cands = order if which == "first" else order[::-1]
    hit = None
    for seg in cands:
        pg = _page_of(engine, seg, None if page == "plain" else page == "coded")
        if pg:
            hit = seg, pg
            break
    if hit is None:
        pytest.skip(f"no {page} page in the image")
    seg, (off, nb) = hit
    if where != "file":
        _flip_host(engine, off + nb // 3)
    if where == "local":
        engine.move_image(L.FMA_TIER_LOCAL)                  # the byte copy carries the damage into the parking buffer
    if where == "file":
        path = str(tmp_path / "c.fmaimg")
        engine.file_store(path)
        engine.move_image(L.FMA_TIER_FILE)
        engine.host_release()
        _flip_file(path, off + nb // 3)
    assert _verify_unchanged(engine) == [seg]
    with pytest.raises(L.FmaError) as ei:                    # the wake's own check agrees
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    assert ei.value.code == L.FMA_EINTEGRITY and f"segment {seg}" in ei.value.message


@gpu
def test_a_damaged_packed_header_counts_as_bad_not_as_an_error(engine, oracle):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=True)
    engine.set_option("pack", 1)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    seg = sorted(ref)[2]
    off, nb = _page_of(engine, seg, True)
    _flip_host(engine, off + (3 << 19) + (12 << 10))         # the page header's magic (csrc/fma_codec.h kHdrOff)
    assert _verify_unchanged(engine) == [seg]


_ADOPT_CHILD = r"""
import json, os, sys
sys.path.insert(0, {root!r})
import fma_b200
from fma_b200 import workloads as W, _lib as L
eng = fma_b200.Engine(0)
for s in W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2):
    eng.alloc(s.bytes, s.tag)
eng.image_adopt_file(sys.argv[1], ["weights"])
bad = eng.verify_image()
rows = [r["kind"] for r in eng.timeline()]
if bad:
    print(json.dumps({{"bad": bad, "rows": rows}}), flush=True)
    sys.exit(0)
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
print(json.dumps({{"bad": bad, "rows": rows, "digests": eng.digest_all(["weights"])}}), flush=True)
"""


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_adopted_file_is_verified_in_a_fresh_process(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    engine.set_option("pack", pack)
    path = str(tmp_path / "a.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    child = tmp_path / "child.py"
    child.write_text(_ADOPT_CHILD.format(root=ROOT))

    def run(p):
        r = subprocess.run([sys.executable, str(child), p], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        return json.loads(r.stdout.strip().splitlines()[-1])

    got = run(path)
    assert got["bad"] == [] and "file_io" in got["rows"]
    assert [got["digests"][i] for i in widx] == [oracle.digest(ref[i]) for i in widx]
    # a file of the same size whose image bytes were replaced: adoption reads only the descriptor and accepts it; the check names
    # every segment whose bytes changed
    img = engine.stats()["image_store_bytes"]
    other = str(tmp_path / "b.fmaimg")
    data = np.fromfile(path, dtype=np.uint8)
    order = sorted(widx, key=lambda i: engine.segment(i).packed_offset)
    off, nb = engine.image_pages()
    s1, s2 = engine.segment(order[1]), engine.segment(order[-1])
    p1, p2 = s1.packed_offset // PAGE, (s2.packed_offset + s2.bytes) // PAGE - 1
    data[off[p1]:off[p1] + nb[p1]] = np.random.default_rng(7).integers(0, 256, nb[p1], dtype=np.uint8)
    data[off[p2] + 4096:off[p2] + 8192] ^= 0x5A
    assert data.size == img + (2 << 20)
    data.tofile(other)
    got = run(other)
    assert got["bad"] == sorted([order[1], order[-1]])
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_refusals_leave_the_engine_unchanged(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)

    def refused(code, text):
        before = _snapshot(engine)
        with pytest.raises(L.FmaError) as ei:
            engine.verify_image()
        assert ei.value.code == code and text in ei.value.message, ei.value.message
        assert _snapshot(engine) == before

    refused(L.FMA_ESTATE, "nothing is asleep")              # awake
    engine.sleep(["weights"])                                # no digests recorded
    refused(L.FMA_ESTATE, "FMA_FLAG_VERIFY")
    engine.wake(None)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    engine.wake(None, flags=L.FMA_FLAG_KEEP_BACKUP)          # mapped segments keep a backup
    refused(L.FMA_ESTATE, "keeps a backup")
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    engine.wake(None)
    path = str(tmp_path / "t.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    size = os.path.getsize(path)
    os.truncate(path, size // 2)                             # cut after the sleep
    refused(L.FMA_EIO, "the image needs")
    os.unlink(path)
    refused(L.FMA_EIO, "cannot open")


@gpu
def test_verify_between_sleep_and_wake_with_incremental(engine, oracle):
    """The incremental option records digests too; a verify in between changes nothing for the clean sleep that follows."""
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=True)
    engine.set_option("pack", 1)
    engine.set_option("incremental", 1)
    engine.sleep(["weights"])
    assert _verify_unchanged(engine) == []
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    engine.sleep(["weights"])                                # clean: nothing moves
    assert engine.stats()["sleep_bytes_copied"] == 0
    assert _verify_unchanged(engine) == []
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


def _build_k6_test(out, flags, gpu_build):
    src = os.path.join(EMU, "unpack_digest_emu_test.cpp")
    if gpu_build:
        obj = out + ".o"
        subprocess.check_call(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "fma_oracle.c"), "-o", out + "_oracle.o"])
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DFMA_GPU_TEST", "-I" + CSRC,
                               "-x", "cu", "-c", src, "-o", obj])
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", obj, out + "_oracle.o", "-o", out])
    else:
        subprocess.check_call(["g++", "-std=c++17", "-g", *flags, "-DFMA_CUDA_EMU", "-include", os.path.join(EMU, "cuda_emu.h"),
                               "-I/usr/local/cuda/include", "-I" + CSRC, src, os.path.join(ROOT, "oracle", "fma_oracle.c"), "-o", out, "-lpthread"])
    return out


def test_k6_against_the_oracle_on_the_cpu_execution_model(tmp_path):
    """tests/cpp/cuda_emu/unpack_digest_emu_test.cpp: K6 == the oracle's decode + digest == K3 over K5's output, plain and under
    ThreadSanitizer (a missing barrier around the shared exception list shows up as a race)."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    def one(san, flags):
        exe = _build_k6_test(str(tmp_path / f"k6_{san}"), flags, False)
        env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
        if san != "plain":
            env["FMA_EMU_FAST"] = "1"
        r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("plain", ["-O2"]), ("tsan", ["-O1", "-fsanitize=thread"])]))
    for san, rc, out in results:
        assert rc == 0 and "unpack digest (emulated) ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out, (san, out[-3000:])


@gpu
def test_k6_against_the_oracle_on_the_device(tmp_path):
    if HOSTSIM:
        pytest.skip("a device test")
    exe = _build_k6_test(str(tmp_path / "k6_gpu"), [], True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "unpack digest (GPU) ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


# ---- the host-simulated engine ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_verify") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS,
                           os.path.join(SIM, "hostsim_verify_kernels.cpp"), "-o", out, "-lpthread"])
    return out


def test_image_verify_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider",
                        "-k", "not on_the_device"], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail


def test_image_verify_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/verify_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side: a verify whose
    file readers fail half way, and a verify racing fma_stats / fma_timeline from another thread."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"verify_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "hostsim_verify_kernels.cpp"),
                               os.path.join(SIM, "verify_sanitizer_test.cpp"), "-o", exe, "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED"):
            env.pop(key, None)
        r = subprocess.run([exe, str(tmp_path / f"{san}.fmaimg")], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "verify sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
