"""Demotion behind the call (fma_image_move_flags with FMA_FLAG_WRITE_BEHIND; Engine.move_image(FMA_TIER_FILE, behind=True)): a
host-tier image goes to the file tier without holding the operation lock for the disk write.  The write-behind job of a write-behind
sleep writes the host store that already holds the image, seals the file and commits; every call that takes the operation lock
pre-empts it and sees the host-tier image with its store kept.  The device tests (-m gpu on an H100) compare the file's bytes, the
statistics and the restored weights with the oracle; test_demotion_against_the_host_simulated_engine runs them on CPU against the
host-simulated engine (tests/cpp/hostsim), tests/cpp/demote_route_test.cpp checks the route, and
tests/cpp/hostsim/demote_sanitizer_test.cpp runs the job's races under ThreadSanitizer and ASan+UBSan+LeakSan."""
import os
import subprocess
import sys

import pytest

from tests.test_file_tier import _check_file, _io, _stored_pages
from tests.test_resident_share import _check_restored, _load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "cpp", "hostsim")
gpu = pytest.mark.gpu
SLOW = "200"     # FMA_WB_ITEM_DELAY_MS: the demotion is still writing when the next call comes, whatever the disk's speed


def _L():
    from fma_b200 import _lib as L

    return L


def _setup(engine, oracle, tmp_path, pack):
    """The tiny table asleep in the host tier (digests recorded), a file store named."""
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.set_option("load_chunk_bytes", 1 << 20)
    engine.set_option("load_threads", 4)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_HOST, flags=L.FMA_FLAG_VERIFY)
    return ptrs, ref, path


def _rows(engine, kind):
    return [r for r in engine.timeline() if r["kind"] == kind]


def _host_tier(engine):
    L = _L()
    st = engine.stats()
    assert engine.is_sleeping() and st["tier"] == L.FMA_TIER_HOST and st["hbm_mapped_bytes"] == 0
    assert st["host_store_bytes"] >= st["image_store_bytes"] > 0
    assert all(s.tier == L.FMA_TIER_HOST for s in engine.segments() if s.has_backup)


def _demote(engine):
    """The demotion returns with the image still in the host tier, its job writing: a "move" timeline of wb_start and total (0)."""
    L = _L()
    engine.move_image(L.FMA_TIER_FILE, behind=True)
    tl = engine.timeline()
    assert {r["op"] for r in tl} == {"move"} and [r["kind"] for r in tl] == ["wb_start", "total"], tl
    assert tl[1]["bytes"] == 0 and tl[0]["bytes"] == engine.stats()["image_store_bytes"]
    _host_tier(engine)


def _committed(engine):
    L = _L()
    st = engine.stats()
    assert engine.is_sleeping() and st["tier"] == L.FMA_TIER_FILE and st["host_store_bytes"] == 0
    assert all(s.tier == L.FMA_TIER_FILE for s in engine.segments() if s.has_backup)


def _empty(path):
    return os.path.getsize(path) == 0


@gpu
@pytest.mark.parametrize("io", ["buffered", "direct"])
@pytest.mark.parametrize("pack", [0, 1])
def test_demotion_returns_then_commits_to_the_file(engine, oracle, monkeypatch, tmp_path, pack, io):
    L = _L()
    _io(monkeypatch, tmp_path, io)
    monkeypatch.setenv("FMA_WB_ITEM_DELAY_MS", "50")
    ptrs, ref, path = _setup(engine, oracle, tmp_path, pack)
    widx = sorted(ref)
    st = engine.stats()
    assert st["image_packed"] == pack and st["image_store_bytes"] == sum(p.size for p in _stored_pages(oracle, ref, widx, pack))
    engine.prefetch_image(8 << 20)                          # a prefetched copy travels with a host -> file move
    prefetched = engine.stats()["prefetched_bytes"]
    assert prefetched > 0
    _demote(engine)
    state, pending = engine.writeback(0)
    assert state == 1 and 0 < pending <= st["image_store_bytes"]
    assert engine.writeback(None) == (0, 0)
    _committed(engine)
    assert engine.stats()["prefetched_bytes"] == prefetched
    tl = engine.timeline()
    assert {r["op"] for r in tl} == {"writeback"}
    assert [r["idx"] for r in tl if r["kind"] == "total"] == [1] and [r["idx"] for r in tl if r["kind"] == "file_io"] == [1 if io == "direct" else 0]
    _check_file(engine, oracle, path, ref, widx, pack)
    info = engine.image_file_info(path)
    assert info["packed"] == bool(pack) and info["digests"] and info["image_bytes"] == st["image_store_bytes"]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)              # from the file (and the prefetched copy), against the digests it carries
    assert engine.stats()["tier"] == L.FMA_TIER_FILE and _rows(engine, "file_io")
    _check_restored(engine, oracle, ptrs, ref)
    assert engine.writeback(0) == (0, 0)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_a_wake_mid_demotion_is_a_host_tier_wake_and_the_store_is_reused(engine, oracle, monkeypatch, tmp_path, pack):
    L = _L()
    monkeypatch.setenv("FMA_WB_ITEM_DELAY_MS", SLOW)
    ptrs, ref, path = _setup(engine, oracle, tmp_path, pack)
    pin = engine.stats()["host_store_pin_seconds"]
    _demote(engine)
    assert engine.writeback(0)[0] == 1
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)              # pre-empts the demotion
    st = engine.stats()
    assert st["tier"] == L.FMA_TIER_HOST and st["host_store_bytes"] > 0 and st["wake_bytes_restored"] > 0
    tl = engine.timeline()
    assert tl[0]["kind"] == "wb_cancel" and tl[0]["op"] == "wake" and not _rows(engine, "file_io")
    assert _empty(path) and engine.writeback(0) == (0, 0)
    _check_restored(engine, oracle, ptrs, ref)
    monkeypatch.delenv("FMA_WB_ITEM_DELAY_MS")
    engine.sleep(["weights"], tier=L.FMA_TIER_HOST, flags=L.FMA_FLAG_VERIFY)   # the kept store again: nothing pinned
    _demote(engine)
    assert engine.stats()["host_store_pin_seconds"] == pin
    assert engine.writeback(None) == (0, 0)
    _committed(engine)
    _check_file(engine, oracle, path, ref, sorted(ref), pack)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("call", ["verify", "prefetch", "move", "file_store", "host_reserve", "destroy"])
def test_every_operation_pre_empts_the_demotion_and_sees_a_host_tier_image(built, oracle, monkeypatch, tmp_path, call):
    import fma_b200

    L = _L()
    monkeypatch.setenv("FMA_WB_ITEM_DELAY_MS", SLOW)
    engine = fma_b200.Engine(0)
    try:
        ptrs, ref, path = _setup(engine, oracle, tmp_path, 0)
        store = engine.stats()["host_store_bytes"]
        _demote(engine)
        assert engine.writeback(0)[0] == 1
        if call == "destroy":
            engine.close()                                  # cancels the job: the file never carries a descriptor
            assert _empty(path)
            return
        if call == "verify":
            assert engine.verify_image() == []
            assert engine.timeline()[0]["kind"] == "wb_cancel" and engine.timeline()[0]["op"] == "verify"
        elif call == "prefetch":
            engine.prefetch_image(8 << 20)
            assert engine.stats()["prefetched_bytes"] > 0
        elif call == "move":
            engine.move_image(L.FMA_TIER_FILE)              # the synchronous move, from the host tier
            assert engine.stats()["tier"] == L.FMA_TIER_FILE
            engine.host_release()
            _check_file(engine, oracle, path, ref, sorted(ref), 0)
        elif call == "file_store":
            path = str(tmp_path / "other.fmaimg")
            engine.file_store(path)
        elif call == "host_reserve":
            engine.host_reserve(4 << 20)                    # (fits: the store holds the image and stays)
        assert engine.writeback(0) == (0, 0)
        if call != "move":
            _host_tier(engine)
            assert engine.stats()["host_store_bytes"] == store and (not os.path.exists(path) or _empty(path))
            monkeypatch.delenv("FMA_WB_ITEM_DELAY_MS")
            _demote(engine)                                 # a second demotion over the kept store, without a wake
            assert engine.writeback(None) == (0, 0)
            _committed(engine)
            _check_file(engine, oracle, path, ref, sorted(ref), 0)
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(engine, oracle, ptrs, ref)
    finally:
        engine.close()


@gpu
def test_demotion_refusals_leave_the_engine_unchanged(built, oracle, monkeypatch, tmp_path):
    import fma_b200

    L = _L()
    path = tmp_path / "m.fmaimg"

    def refused(engine, tier, code, flags=None):
        before = [(s.mapped, s.has_backup, s.tier) for s in engine.segments()], {k: engine.stats()[k] for k in ("tier", "host_store_bytes")}
        size = os.path.getsize(path) if path.exists() else None
        with pytest.raises(L.FmaError) as ei:
            if flags is None:
                engine.move_image(tier, behind=True)
            else:
                L.check(engine._lib.fma_image_move_flags(engine._h, tier, flags))
        assert ei.value.code == code, ei.value
        assert ([(s.mapped, s.has_backup, s.tier) for s in engine.segments()], {k: engine.stats()[k] for k in ("tier", "host_store_bytes")}) == before
        assert (os.path.getsize(path) if path.exists() else None) == size
        assert engine.writeback(0) == (0, 0) and not _rows(engine, "wb_start")

    engine = fma_b200.Engine(0)
    try:
        table, ptrs, ref = _load(engine, oracle, bf16=False)
        refused(engine, L.FMA_TIER_FILE, L.FMA_ESTATE)                      # nothing asleep
        engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
        refused(engine, L.FMA_TIER_FILE, L.FMA_ESTATE)                      # no fma_file_store
        refused(engine, L.FMA_TIER_LOCAL, L.FMA_EINVAL)                     # another tier pair
        refused(engine, L.FMA_TIER_PEER, L.FMA_EINVAL)
        refused(engine, L.FMA_TIER_HOST, L.FMA_EINVAL)
        refused(engine, L.FMA_TIER_FILE, L.FMA_EINVAL, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)   # a flag a move does not take
        engine.file_store(str(tmp_path / "no-such-dir" / "m.fmaimg"))
        refused(engine, L.FMA_TIER_FILE, L.FMA_EIO)                         # the file cannot be created
        engine.file_store(str(path))
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(engine, oracle, ptrs, ref)
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
        refused(engine, L.FMA_TIER_HOST, L.FMA_EINVAL)                      # file -> host is a synchronous promotion
        refused(engine, L.FMA_TIER_FILE, L.FMA_EINVAL)
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        engine.set_option("resident_bytes", 8 << 20)                        # part of the image in a resident share
        engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
        assert engine.stats()["resident_bytes"] > 0
        refused(engine, L.FMA_TIER_FILE, L.FMA_ESTATE)
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(engine, oracle, ptrs, ref)
    finally:
        engine.close()
    monkeypatch.setenv("FMA_HOST_STORE_SHM", "1")                           # a memfd store, which can be handed out
    for share in ("export", "host_store_share"):
        engine = fma_b200.Engine(0)
        try:
            table, ptrs, ref = _load(engine, oracle, bf16=False)
            engine.file_store(str(path))
            engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
            os.close(engine.image_export() if share == "export" else engine.host_store_share())
            refused(engine, L.FMA_TIER_FILE, L.FMA_ESTATE)                  # its bytes are not this engine's alone to release
            engine.move_image(L.FMA_TIER_FILE)                              # the synchronous move leaves the store to its holders
            assert engine.stats()["tier"] == L.FMA_TIER_FILE
            engine.wake(None, flags=L.FMA_FLAG_VERIFY)
            _check_restored(engine, oracle, ptrs, ref)
        finally:
            engine.close()


_FAIL_CHILD = r"""
import os, resource, signal, sys
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
eng.set_option("load_chunk_bytes", 1 << 20)
eng.file_store(sys.argv[1])
eng.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
signal.signal(signal.SIGXFSZ, signal.SIG_IGN)              # a write past the limit fails with EFBIG instead of killing us
resource.setrlimit(resource.RLIMIT_FSIZE, (W_bytes // 2, resource.RLIM_INFINITY))
eng.move_image(L.FMA_TIER_FILE, behind=True)               # returns: the disk is the job's
try:
    eng.writeback(None)
    raise SystemExit("the demotion did not fail")
except L.FmaError as e:
    assert e.code == L.FMA_EIO and "write-behind" in e.message, e
assert eng.writeback(0) == (0, 0)                          # reported once
resource.setrlimit(resource.RLIMIT_FSIZE, (resource.RLIM_INFINITY, resource.RLIM_INFINITY))
st = eng.stats()
assert st["tier"] == L.FMA_TIER_HOST and st["host_store_bytes"] >= W_bytes and os.path.getsize(sys.argv[1]) == 0
eng.move_image(L.FMA_TIER_FILE, behind=True)               # with room again, over the kept store
assert eng.writeback(None) == (0, 0) and eng.stats()["tier"] == L.FMA_TIER_FILE and eng.stats()["host_store_bytes"] == 0
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
print("demotion failure ok", flush=True)
"""


@gpu
def test_a_demotion_whose_write_fails_leaves_the_image_in_the_host_tier(built, tmp_path):
    child = tmp_path / "child.py"
    child.write_text(_FAIL_CHILD.format(root=ROOT))
    r = subprocess.run([sys.executable, str(child), str(tmp_path / "m.fmaimg")], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0 and "demotion failure ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


def test_demote_routes():
    """The write-behind case of move_route in csrc/fma_layout.h (tests/cpp/demote_route_test.cpp)."""
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"demote_route_test_{os.getpid()}")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "demote_route_test.cpp"), "-o", exe])
    try:
        assert "demote routes ok" in subprocess.check_output([exe], text=True)
    finally:
        os.unlink(exe)


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_demote") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS,
                           os.path.join(SIM, "hostsim_verify_kernels.cpp"), "-o", out, "-lpthread"])
    return out


def test_demotion_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="1")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM", "FMA_WB_ITEM_DELAY_MS", "FMA_NODE_AGENT_SOCK",
                "FMA_DEPOSIT_FILE_IMAGE", "FMA_FILE_WRITE_BEHIND", "LOCAL_RANK"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
    skips = [l for l in r.stdout.splitlines() if l.startswith("SKIPPED")]
    assert all("refuses O_DIRECT" in l for l in skips), skips


def test_demotion_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/demote_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"demote_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "hostsim_verify_kernels.cpp"),
                               os.path.join(SIM, "demote_sanitizer_test.cpp"), "-o", exe, "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_WB_ITEM_DELAY_MS"):
            env.pop(key, None)
        r = subprocess.run([exe, str(tmp_path / f"{san}.fmaimg")], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "demote sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
