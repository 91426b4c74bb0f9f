"""File tier (FMA_TIER_FILE): a sleep writes the model's image to a file on local disk and holds no host store; a wake streams it
back through the staging ring.  The device tests (-m gpu on an H100) compare the file's bytes, the statistics and the restored
weights with the oracle; test_file_tier_against_the_host_simulated_engine runs the same tests on CPU against the host-simulated
engine (tests/cpp/hostsim), and the C++ scenario of tests/cpp/hostsim/file_sanitizer_test.cpp runs under ThreadSanitizer and
ASan+UBSan+LeakSan."""
import errno
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.pagegen import pages_of
from tests.test_resident_share import _check_restored, _load, _same_stored_page

PAGE = 2 << 20
TAIL = 2 << 20   # the descriptor at the end of an image file (kImageTail)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _L():
    from fma_b200 import _lib as L

    return L


def _o_direct_refused(directory) -> str | None:
    """Why O_DIRECT cannot be tested in `directory` (None: it can)."""
    p = os.path.join(str(directory), ".odirect_probe")
    try:
        os.close(os.open(p, os.O_WRONLY | os.O_CREAT | os.O_DIRECT, 0o644))
    except OSError as e:
        if e.errno == errno.EINVAL:
            return f"the filesystem of {directory} refuses O_DIRECT"
        raise
    finally:
        if os.path.exists(p):
            os.unlink(p)
    return None


def _io(monkeypatch, tmp_path, io):
    if io == "buffered":
        monkeypatch.setenv("FMA_FILE_BUFFERED", "1")
    else:
        monkeypatch.delenv("FMA_FILE_BUFFERED", raising=False)
        why = _o_direct_refused(tmp_path)
        if why:
            pytest.skip(why)


def _stored_pages(oracle, ref, widx, packed):
    return [oracle.pack_page(p) if packed else p for i in widx for p in pages_of(ref[i])]


def _check_file(engine, oracle, path, ref, widx, packed):
    """The file holds the image in the form the engine reports, then the descriptor: nothing else."""
    st = engine.stats()
    data = np.fromfile(path, dtype=np.uint8)
    assert data.size == st["image_store_bytes"] + TAIL and st["host_store_bytes"] == 0
    img = data[:st["image_store_bytes"]]
    if packed:
        want = _stored_pages(oracle, ref, widx, True)
        off, nb = engine.image_pages()
        assert nb == [p.size for p in want]
        assert all(_same_stored_page(img[o:o + n], w) for o, n, w in zip(off, nb, want))
    else:
        assert np.array_equal(img, oracle.packed_image([ref[i] for i in widx]))


@gpu
@pytest.mark.parametrize("io", ["buffered", "direct"])
@pytest.mark.parametrize("chunk", ["ragged", "one_slot"])
@pytest.mark.parametrize("pack", [0, 1])
def test_file_tier_roundtrip_matches_oracle(engine, oracle, monkeypatch, tmp_path, pack, chunk, io):
    L = _L()
    _io(monkeypatch, tmp_path, io)
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    W = sum(ref[i].size for i in widx)
    engine.set_option("pack", pack)
    if chunk == "ragged":    # ring slots of 6 MiB over segments of 2..32 MiB (PACKED: by stored bytes), several windows per slot
        engine.set_option("chunk_bytes", 6 << 20)
    engine.set_option("load_chunk_bytes", 1 << 20)
    engine.set_option("load_slots", 3)
    path = str(tmp_path / "model.fmaimg")
    engine.file_store(path)
    assert engine.stats()["io_buffer_bytes"] == 3 * ((1 << 20) + 8192)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    st = engine.stats()
    assert engine.is_sleeping() and st["tier"] == L.FMA_TIER_FILE and st["hbm_mapped_bytes"] == 0
    assert st["sleep_bytes_offloaded"] == W and st["image_packed"] == pack
    assert st["image_store_bytes"] == sum(p.size for p in _stored_pages(oracle, ref, widx, pack))
    assert st["sleep_bytes_copied"] == st["image_store_bytes"]
    assert all(s.tier == L.FMA_TIER_FILE for s in engine.segments() if s.has_backup)
    assert [r["idx"] for r in engine.timeline() if r["kind"] == "file_io"] == [1 if io == "direct" else 0]
    _check_file(engine, oracle, path, ref, widx, pack)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    st = engine.stats()
    assert st["wake_bytes_restored"] == W and st["tier"] == L.FMA_TIER_FILE and st["host_store_bytes"] == 0
    assert [r["idx"] for r in engine.timeline() if r["kind"] == "file_io"] == [1 if io == "direct" else 0]
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)          # a second cycle from the woken state (merged runs)
    engine.wake(None)
    _check_restored(engine, oracle, ptrs, ref)
    assert os.path.exists(path)                              # the caller owns the file


@gpu
def test_file_tier_tag_selective_repeated_kept_and_level2(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.file_store(str(tmp_path / "m.fmaimg"))
    for _ in range(2):
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE)      # asleep: a no-op
        engine.wake(["kv_cache"])                            # nothing read from the file
        assert engine.is_sleeping() and engine.stats()["wake_bytes_restored"] == 0
        engine.wake(["weights"])
        engine.wake(None)                                    # a retried wake finds nothing left to do
        _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    engine.wake(None, flags=L.FMA_FLAG_KEEP_BACKUP)
    assert all(s.has_backup for i, s in enumerate(engine.segments()) if i in ref)
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep([], tier=L.FMA_TIER_FILE)                   # level 2: nothing offloaded, nothing written
    assert engine.stats()["sleep_bytes_offloaded"] == 0
    engine.wake(None)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_file_tier_incremental_clean_sleep_writes_nothing(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.set_option("incremental", 1)
    engine.set_option("chunk_bytes", 8 << 20)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    full = engine.stats()["image_store_bytes"]
    assert engine.stats()["sleep_bytes_copied"] == full > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    before = open(path, "rb").read()
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)          # clean: the file outlived the wake
    st = engine.stats()
    assert st["sleep_bytes_copied"] == 0 and st["image_store_bytes"] == full and st["tier"] == L.FMA_TIER_FILE
    assert not [r for r in engine.timeline() if r["kind"] == "file_io"] and open(path, "rb").read() == before
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    i = sorted(ref)[1]                                       # one changed byte: a full sleep
    ref[i] = ref[i].copy()
    ref[i][4321] ^= 0x01
    engine.write(i, ref[i].tobytes())
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    assert engine.stats()["sleep_bytes_copied"] == engine.stats()["image_store_bytes"] > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.file_store(str(tmp_path / "other.fmaimg"))        # another file: a full sleep
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    assert engine.stats()["sleep_bytes_copied"] > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_file_tier_swap_out_to_file(built, oracle, tmp_path):
    import fma_b200

    L = _L()
    a, b = fma_b200.Engine(0), fma_b200.Engine(0)
    try:
        ta, pa, ra = _load(a, oracle, bf16=False)
        tb, pb, rb = _load(b, oracle, bf16=True)
        a.file_store(str(tmp_path / "a.fmaimg"))
        b.file_store(str(tmp_path / "b.fmaimg"))
        b.set_option("pack", 1)
        b.sleep(["weights"], tier=L.FMA_TIER_FILE)
        a.swap_out_for(b, offload_tags=("weights",), tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
        assert a.is_sleeping() and a.stats()["tier"] == L.FMA_TIER_FILE and a.stats()["host_store_bytes"] == 0
        _check_restored(b, oracle, pb, rb)
        b.swap_out_for(a, offload_tags=("weights",), tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
        _check_restored(a, oracle, pa, ra)
        assert b.stats()["image_packed"] == 1
        b.wake(None)
        _check_restored(b, oracle, pb, rb)
    finally:
        a.close()
        b.close()


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_file_tier_file_and_image_save_files_are_one_format(built, oracle, monkeypatch, tmp_path, pack):
    """A file-tier file opens with image_load (the host-store adoption), an image_save file with image_adopt_file."""
    import fma_b200

    L = _L()
    monkeypatch.setenv("FMA_HOST_STORE_SHM", "1")
    a, b = fma_b200.Engine(0), fma_b200.Engine(0)
    try:
        ta, pa, ra = _load(a, oracle, bf16=bool(pack))
        tb, pb, rb = _load(b, oracle, bf16=bool(pack))
        for e in (a, b):
            e.set_option("pack", pack)
        path = str(tmp_path / "tier.fmaimg")
        a.file_store(path)
        a.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
        for i in rb:                                         # b's contents must come back from the image, not stay
            b.fill(i, 999)
        b.image_load(path, ["weights"])
        assert b.is_sleeping() and b.stats()["tier"] == L.FMA_TIER_HOST
        b.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(b, oracle, pb, ra)
        a.wake(None)
        b.host_release()                                     # (the adopted store may be a private copy): a fresh, shareable one
        b.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)        # host tier, then image_save
        saved = str(tmp_path / "saved.fmaimg")
        b.image_save(saved)
        b.wake(None)
        for i in ra:
            a.fill(i, 999)
        a.image_adopt_file(saved, ["weights"])
        st = a.stats()
        assert a.is_sleeping() and st["tier"] == L.FMA_TIER_FILE and all(s.tier == L.FMA_TIER_FILE for s in a.segments() if s.has_backup)
        assert st["image_packed"] == pack
        a.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(a, oracle, pa, ra)
    finally:
        a.close()
        b.close()


_ADOPT_CHILD = r"""
import json, os, sys
sys.path.insert(0, {root!r})
import fma_b200
from fma_b200 import workloads as W, _lib as L
eng = fma_b200.Engine(0)
for s in W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2):
    eng.alloc(s.bytes, s.tag)
eng.image_adopt_file(sys.argv[1], ["weights"])
assert eng.is_sleeping() and eng.stats()["tier"] == L.FMA_TIER_FILE and eng.stats()["host_store_bytes"] == 0
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
print(json.dumps(eng.digest_all(["weights"])), flush=True)
"""


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_file_tier_adoption_in_a_fresh_process(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    child = tmp_path / "child.py"
    child.write_text(_ADOPT_CHILD.format(root=ROOT))
    r = subprocess.run([sys.executable, str(child), path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert [got[i] for i in sorted(ref)] == [oracle.digest(ref[i]) for i in sorted(ref)]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)               # the first process still wakes from the same file
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_file_tier_refuses_a_torn_file_and_hand_overs(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    for call in (engine.image_export, lambda: engine.image_describe(L.FMA_TIER_FILE), engine.host_store_share):
        with pytest.raises(L.FmaError) as ei:
            call()
        assert ei.value.code == L.FMA_ESTATE
    engine.wake(None)
    data = open(path, "rb").read()
    torn, foreign = str(tmp_path / "torn.fmaimg"), str(tmp_path / "foreign.fmaimg")
    with open(torn, "wb") as f:                              # every data byte, the descriptor never written
        f.write(data[:len(data) - TAIL])
    with open(foreign, "wb") as f:
        f.write(data[:len(data) - TAIL] + bytes(TAIL))
    before = engine.digest_all(["weights"])
    for p in (torn, foreign, str(tmp_path / "missing.fmaimg")):
        with pytest.raises(L.FmaError) as ei:
            engine.image_adopt_file(p, ["weights"])
        assert ei.value.code in (L.FMA_EINVAL, L.FMA_EIO)
        assert not engine.is_sleeping() and engine.digest_all(["weights"]) == before
    engine.image_adopt_file(path, ["weights"], flags=L.FMA_FLAG_VERIFY)   # sleep by adoption: the device bytes ARE the file's
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_file_tier_refusals_leave_the_engine_awake(engine, oracle, monkeypatch, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    with pytest.raises(L.FmaError) as ei:                    # no file named
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    assert ei.value.code == L.FMA_ESTATE and not engine.is_sleeping()
    engine.file_store(str(tmp_path / "no" / "such" / "dir" / "m.fmaimg"))
    with pytest.raises(L.FmaError) as ei:                    # the file cannot be created
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    assert ei.value.code == L.FMA_EIO and not engine.is_sleeping()
    engine.file_store(str(tmp_path / "m.fmaimg"))
    monkeypatch.setenv("FMA_NO_RING", "1")                   # no HBM for the staging ring
    with pytest.raises(L.FmaError) as ei:
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    assert ei.value.code == L.FMA_ENOMEM and not engine.is_sleeping()
    monkeypatch.delenv("FMA_NO_RING")
    _check_restored(engine, oracle, ptrs, ref)
    engine.file_store(None)
    with pytest.raises(L.FmaError):
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    assert not engine.is_sleeping()


_FSIZE_CHILD = r"""
import json, os, resource, signal, sys
sys.path.insert(0, {root!r})
import fma_b200
from fma_b200 import workloads as W, _lib as L
from oracle import oracle as O
eng = fma_b200.Engine(0)
table = W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2)
ref, first = {{}}, 0
for i, s in enumerate(table):
    eng.alloc(s.bytes, s.tag)
    if s.tag == "weights":
        eng.fill(i, 4242, first); ref[i] = O.digest(O.fill(s.bytes, 4242, first)); first += s.bytes // 8
W_bytes = sum(s.bytes for s in table if s.tag == "weights")
eng.set_option("chunk_bytes", 4 << 20)
eng.set_option("load_chunk_bytes", 1 << 20)
eng.file_store(sys.argv[1])
signal.signal(signal.SIGXFSZ, signal.SIG_IGN)              # a write past the limit fails with EFBIG instead of killing us
limit = W_bytes // 2
resource.setrlimit(resource.RLIMIT_FSIZE, (limit, resource.RLIM_INFINITY))
try:
    eng.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    raise SystemExit("the sleep did not fail")
except L.FmaError as e:
    assert e.code == L.FMA_EIO, e
resource.setrlimit(resource.RLIMIT_FSIZE, (resource.RLIM_INFINITY, resource.RLIM_INFINITY))
released = sum(1 for i in ref if not eng.segment(i).mapped)
assert 0 < released < len(ref), released                   # half way: some segments went, each after its bytes were written
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
eng.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)   # and with room again, a sleep and a wake
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
print("fsize ok", released, flush=True)
"""


@gpu
def test_file_tier_sleep_that_cannot_finish_its_writes_is_restored_bit_exact(built, tmp_path):
    child = tmp_path / "child.py"
    child.write_text(_FSIZE_CHILD.format(root=ROOT))
    r = subprocess.run([sys.executable, str(child), str(tmp_path / "m.fmaimg")], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0 and "fsize ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


@gpu
@pytest.mark.parametrize("io", ["buffered", "direct"])
def test_file_tier_wake_from_a_truncated_file_rolls_back_and_retries(engine, oracle, monkeypatch, tmp_path, io):
    """Cut inside a block, below the offset of the later reads: the wake refuses before it reads past the end of the file."""
    L = _L()
    _io(monkeypatch, tmp_path, io)
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.set_option("load_chunk_bytes", 1 << 20)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    keep = str(tmp_path / "keep")
    shutil.copyfile(path, keep)
    os.truncate(path, engine.stats()["image_store_bytes"] // 2 + 1000)
    with pytest.raises(L.FmaError) as ei:
        engine.wake(None)
    assert ei.value.code == L.FMA_EIO and "the image needs" in ei.value.message
    assert engine.is_sleeping() and all(not s.mapped for s in engine.segments())   # rolled back: every segment still asleep
    shutil.copyfile(keep, path)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_file_tier_ignores_the_resident_share_and_leaves_the_parking_buffer_alone(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("resident_bytes", 48 << 20)
    engine.file_store(str(tmp_path / "m.fmaimg"))
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    st = engine.stats()
    assert st["resident_bytes"] == 0 and all(s.tier == L.FMA_TIER_FILE for s in engine.segments() if s.has_backup)
    assert not any(r["kind"].startswith("res_") for r in engine.timeline())
    engine.peer_release()                                    # no parking buffer holds this image: the call is legal
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


_SHIM_CHILD = r"""
import os, sys, types
sys.path.insert(0, {root!r})
sys.modules["torch"] = types.SimpleNamespace(cuda=types.SimpleNamespace(empty_cache=lambda: None))
import fma_b200
from fma_b200 import _lib as L
from fma_b200.cumem import CuMemAllocator
eng = fma_b200.Engine(0)
for i, mib in enumerate((6, 2, 8, 4)):
    eng.alloc(mib << 20, "kv_cache" if i == 2 else "weights")
for i in (0, 1, 3):
    eng.fill(i, 77, i << 24)
before = eng.digest_all(["weights"])
a = CuMemAllocator(engine=eng)
a.sleep(("weights",))
st = eng.stats()
print("tier", st["tier"], st["host_store_bytes"], flush=True)
a.wake_up(None)
assert eng.digest_all(["weights"]) == before
print("file", os.path.exists(os.path.join(os.environ["FMA_FILE_DIR"], "Ishimi-r0.fmaimg")), flush=True)
"""


def test_shim_file_tier_names_removes_and_falls_back(hostsim_lib, tmp_path):
    """FMA_TIER=file: the rank's image goes to <FMA_FILE_DIR>/<instance id>-r<rank>.fmaimg, which is removed when the process
    exits; where the file cannot be written the shim warns and sleeps to the host tier."""
    L = _L()
    child = tmp_path / "child.py"
    child.write_text(_SHIM_CHILD.format(root=ROOT))
    base = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="1", FMA_TIER="file", FMA_INSTANCE_ID="Ishimi", RANK="0")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_NODE_AGENT_SOCK", "FMA_REMOTE_PATHS", "LOCAL_RANK"):
        base.pop(key, None)
    d = tmp_path / "images"
    d.mkdir()
    r = subprocess.run([sys.executable, str(child)], env=dict(base, FMA_FILE_DIR=str(d)), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert f"tier {L.FMA_TIER_FILE} 0" in r.stdout and "file True" in r.stdout, r.stdout
    assert os.listdir(d) == []                               # removed at exit
    r = subprocess.run([sys.executable, str(child)], env=dict(base, FMA_FILE_DIR=str(tmp_path / "missing")), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert f"tier {L.FMA_TIER_HOST} " in r.stdout and "sleeping to the host tier instead" in r.stderr, r.stdout + r.stderr[-2000:]


def test_file_routes():
    """The file case of sleep_route / wake_route in csrc/fma_layout.h (tests/cpp/file_route_test.cpp)."""
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"file_route_test_{os.getpid()}")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "file_route_test.cpp"), "-o", exe])
    try:
        assert "file routes ok" in subprocess.check_output([exe], text=True)
    finally:
        os.unlink(exe)


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_file") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS, "-o", out, "-lpthread"])
    return out


def test_file_tier_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
    # the only skips allowed are O_DIRECT ones, on a filesystem that refuses it
    skips = [l for l in r.stdout.splitlines() if l.startswith("SKIPPED")]
    assert all("refuses O_DIRECT" in l for l in skips), skips


def test_file_tier_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/file_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SIM, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"file_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "file_sanitizer_test.cpp"), "-o", exe, "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED"):
            env.pop(key, None)
        r = subprocess.run([exe, str(tmp_path / f"{san}.fmaimg")], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "file sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
