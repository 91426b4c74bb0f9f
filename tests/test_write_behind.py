"""Write-behind file-tier sleep (FMA_FLAG_WRITE_BEHIND): the sleep fills the engine's pinned host store at PCIe speed and returns; a
background job writes the file and then moves the image to the file tier.  Every call that takes the operation lock pre-empts a job
still writing and sees a host-tier image.  The device tests (-m gpu on an H100) compare the file's bytes, the statistics and the
restored weights with the oracle; test_write_behind_against_the_host_simulated_engine runs them on CPU against the host-simulated
engine (tests/cpp/hostsim), tests/cpp/write_behind_route_test.cpp checks the route, and tests/cpp/hostsim/write_behind_sanitizer_test.cpp
runs the job's races under ThreadSanitizer and ASan+UBSan+LeakSan."""
import os
import subprocess
import sys

import pytest

from tests.test_file_tier import _check_file, _io, _stored_pages
from tests.test_resident_share import _check_restored, _load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "cpp", "hostsim")
gpu = pytest.mark.gpu
SLOW = "200"     # FMA_WB_ITEM_DELAY_MS: the job is still writing when the next call comes, whatever the disk's speed


def _L():
    from fma_b200 import _lib as L

    return L


def _setup(engine, oracle, tmp_path, pack, reserve=True):
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.set_option("load_chunk_bytes", 1 << 20)
    engine.set_option("load_threads", 4)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    if reserve:
        engine.host_reserve(sum(ref[i].size for i in ref))
    return ptrs, ref, path


def _rows(engine, kind):
    return [r for r in engine.timeline() if r["kind"] == kind]


def _asleep_in_host_store(engine, path):
    """What a write-behind sleep leaves while its job writes: a host-tier image, the weights unmapped, the file not yet complete."""
    L = _L()
    st = engine.stats()
    assert engine.is_sleeping() and st["tier"] == L.FMA_TIER_HOST and st["hbm_mapped_bytes"] == 0
    assert st["host_store_bytes"] >= st["image_store_bytes"] > 0
    assert all(s.tier == L.FMA_TIER_HOST for s in engine.segments() if s.has_backup)
    assert len(_rows(engine, "wb_start")) == 1 and not _rows(engine, "wb_fallback")


def _empty(path):
    return os.path.getsize(path) == 0


@gpu
@pytest.mark.parametrize("io", ["buffered", "direct"])
@pytest.mark.parametrize("pack", [0, 1])
def test_write_behind_sleep_returns_then_commits_to_the_file(engine, oracle, monkeypatch, tmp_path, pack, io):
    L = _L()
    _io(monkeypatch, tmp_path, io)
    monkeypatch.setenv("FMA_WB_ITEM_DELAY_MS", "50")
    ptrs, ref, path = _setup(engine, oracle, tmp_path, pack)
    widx = sorted(ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)
    state, pending = engine.writeback(0)
    _asleep_in_host_store(engine, path)
    st = engine.stats()
    assert state == 1 and 0 < pending <= st["image_store_bytes"]
    assert st["image_packed"] == pack and st["sleep_bytes_copied"] == st["image_store_bytes"]
    assert st["image_store_bytes"] == sum(p.size for p in _stored_pages(oracle, ref, widx, pack))
    assert engine.writeback(None) == (0, 0)
    st = engine.stats()
    assert st["tier"] == L.FMA_TIER_FILE and st["host_store_bytes"] == 0 and engine.is_sleeping()
    assert all(s.tier == L.FMA_TIER_FILE for s in engine.segments() if s.has_backup)
    tl = engine.timeline()
    assert {r["op"] for r in tl} == {"writeback"}
    assert [r["idx"] for r in tl if r["kind"] == "total"] == [1] and [r["idx"] for r in tl if r["kind"] == "file_io"] == [1 if io == "direct" else 0]
    _check_file(engine, oracle, path, ref, widx, pack)
    info = engine.image_file_info(path)
    assert info["packed"] == bool(pack) and info["digests"] and info["image_bytes"] == st["image_store_bytes"]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)               # from the file
    assert engine.stats()["tier"] == L.FMA_TIER_FILE and _rows(engine, "file_io")
    _check_restored(engine, oracle, ptrs, ref)
    assert engine.writeback(0) == (0, 0)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_a_wake_mid_write_is_a_host_tier_wake_and_the_store_is_reused(engine, oracle, monkeypatch, tmp_path, pack):
    L = _L()
    monkeypatch.setenv("FMA_WB_ITEM_DELAY_MS", SLOW)
    ptrs, ref, path = _setup(engine, oracle, tmp_path, pack)
    pin = engine.stats()["host_store_pin_seconds"]
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND)
    _asleep_in_host_store(engine, path)
    assert engine.writeback(0)[0] == 1
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)               # pre-empts the job
    st = engine.stats()
    assert st["tier"] == L.FMA_TIER_HOST and st["host_store_bytes"] > 0 and st["wake_bytes_restored"] > 0
    tl = engine.timeline()
    assert tl[0]["kind"] == "wb_cancel" and tl[0]["op"] == "wake" and not _rows(engine, "file_io")
    assert _empty(path) and engine.writeback(0) == (0, 0)
    _check_restored(engine, oracle, ptrs, ref)
    monkeypatch.delenv("FMA_WB_ITEM_DELAY_MS")
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND)   # the kept store again: nothing pinned
    _asleep_in_host_store(engine, path)
    assert engine.stats()["host_store_pin_seconds"] == pin
    assert engine.writeback(None) == (0, 0) and engine.stats()["tier"] == L.FMA_TIER_FILE
    _check_file(engine, oracle, path, ref, sorted(ref), pack)
    engine.wake(None)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("call", ["verify", "prefetch", "move", "file_store", "host_reserve", "destroy"])
def test_every_operation_pre_empts_the_job_and_sees_a_host_tier_image(built, oracle, monkeypatch, tmp_path, call):
    import fma_b200

    L = _L()
    monkeypatch.setenv("FMA_WB_ITEM_DELAY_MS", SLOW)
    engine = fma_b200.Engine(0)
    try:
        ptrs, ref, path = _setup(engine, oracle, tmp_path, 0)
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)
        assert engine.writeback(0)[0] == 1
        if call == "destroy":
            engine.close()                                   # cancels the job: the file never carries a descriptor
            assert _empty(path)
            return
        if call == "verify":
            assert engine.verify_image() == []
            assert engine.timeline()[0]["kind"] == "wb_cancel" and engine.timeline()[0]["op"] == "verify"
        elif call == "prefetch":
            engine.prefetch_image(8 << 20)
            assert engine.stats()["prefetched_bytes"] > 0
        elif call == "move":
            engine.move_image(L.FMA_TIER_FILE)               # the synchronous move, from the host tier
            assert engine.stats()["tier"] == L.FMA_TIER_FILE
            engine.host_release()
            _check_file(engine, oracle, path, ref, sorted(ref), 0)
        elif call == "file_store":
            engine.file_store(str(tmp_path / "other.fmaimg"))
        elif call == "host_reserve":
            engine.host_reserve(4 << 20)                     # (fits: the store holds the image and stays)
        assert engine.writeback(0) == (0, 0)
        if call != "move":
            st = engine.stats()
            assert _empty(path) and st["tier"] == L.FMA_TIER_HOST and st["host_store_bytes"] > 0
            assert all(s.tier == L.FMA_TIER_HOST for s in engine.segments() if s.has_backup)
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(engine, oracle, ptrs, ref)
    finally:
        engine.close()


@gpu
def test_write_behind_falls_back_to_the_synchronous_file_tier(engine, oracle, tmp_path):
    """No host store, or one too small: today's file-tier sleep, with a wb_fallback row saying why; a clean INCREMENTAL sleep
    writes nothing either way."""
    L = _L()
    ptrs, ref, path = _setup(engine, oracle, tmp_path, 0, reserve=False)
    W = sum(ref[i].size for i in ref)
    for reserve, why in ((0, 1), (W - (2 << 20), 2)):
        if reserve:
            engine.host_reserve(reserve)
        engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND)
        st = engine.stats()
        assert st["tier"] == L.FMA_TIER_FILE and [r["idx"] for r in _rows(engine, "wb_fallback")] == [why]
        assert not _rows(engine, "wb_start") and engine.writeback(0) == (0, 0)
        assert st["host_store_bytes"] == reserve
        engine.wake(None)
        _check_restored(engine, oracle, ptrs, ref)
    engine.host_release()
    engine.set_option("incremental", 1)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE)
    engine.wake(None)
    engine.host_reserve(W)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND)   # clean: nothing to write behind
    assert engine.stats()["sleep_bytes_copied"] == 0 and [r["idx"] for r in _rows(engine, "wb_fallback")] == [4]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_HOST, flags=L.FMA_FLAG_WRITE_BEHIND)     # ignored for the other tiers
    assert not _rows(engine, "wb_start") and not _rows(engine, "wb_fallback") and engine.stats()["tier"] == L.FMA_TIER_HOST
    engine.wake(None)
    _check_restored(engine, oracle, ptrs, ref)


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
eng.host_reserve(W_bytes)
signal.signal(signal.SIGXFSZ, signal.SIG_IGN)              # a write past the limit fails with EFBIG instead of killing us
resource.setrlimit(resource.RLIMIT_FSIZE, (W_bytes // 2, resource.RLIM_INFINITY))
eng.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)   # returns: the disk is the job's
try:
    eng.writeback(None)
    raise SystemExit("the write-behind did not fail")
except L.FmaError as e:
    assert e.code == L.FMA_EIO and "write-behind" in e.message, e
assert eng.writeback(0) == (0, 0)                          # reported once
resource.setrlimit(resource.RLIMIT_FSIZE, (resource.RLIM_INFINITY, resource.RLIM_INFINITY))
st = eng.stats()
assert st["tier"] == L.FMA_TIER_HOST and st["host_store_bytes"] >= W_bytes and os.path.getsize(sys.argv[1]) == 0
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
eng.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)   # with room again
assert eng.writeback(None) == (0, 0) and eng.stats()["tier"] == L.FMA_TIER_FILE
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
print("write-behind failure ok", flush=True)
"""


@gpu
def test_a_job_whose_write_fails_leaves_the_image_in_the_host_tier(built, tmp_path):
    child = tmp_path / "child.py"
    child.write_text(_FAIL_CHILD.format(root=ROOT))
    r = subprocess.run([sys.executable, str(child), str(tmp_path / "m.fmaimg")], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0 and "write-behind failure ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


@gpu
def test_swap_out_to_file_behind_both_ways(built, oracle, tmp_path):
    import fma_b200

    L = _L()
    a, b = fma_b200.Engine(0), fma_b200.Engine(0)
    try:
        ta, pa, ra = _load(a, oracle, bf16=False)
        tb, pb, rb = _load(b, oracle, bf16=True)
        b.set_option("pack", 1)
        for e, ref, name in ((a, ra, "a"), (b, rb, "b")):
            e.file_store(str(tmp_path / f"{name}.fmaimg"))
            e.host_reserve(sum(ref[i].size for i in ref))
        b.sleep(["weights"], tier=L.FMA_TIER_HOST)
        a.swap_out_for(b, offload_tags=("weights",), tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)
        _check_restored(b, oracle, pb, rb)
        assert a.is_sleeping() and a.writeback(None) == (0, 0)
        assert a.stats()["tier"] == L.FMA_TIER_FILE and a.stats()["host_store_bytes"] == 0
        assert [(r["op"], r["idx"]) for r in _rows(a, "total")] == [("writeback", 1)]   # written behind the swap, then committed
        b.swap_out_for(a, offload_tags=("weights",), tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND | L.FMA_FLAG_VERIFY)
        _check_restored(a, oracle, pa, ra)                  # woken from its file
        assert b.writeback(None) == (0, 0) and b.stats()["tier"] == L.FMA_TIER_FILE and b.stats()["image_packed"] == 1
        b.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(b, oracle, pb, rb)
    finally:
        a.close()
        b.close()


# The shim with FMA_FILE_WRITE_BEHIND=1 and a deposit: the instance sleeps (the file still being written) and exits asleep; its exit
# hook waits for the job, so the node agent keeps a complete file, which the next instance adopts.
_SHIM_INSTANCE = r"""
import os, sys, types
sys.path.insert(0, {root!r})
sys.modules.setdefault("torch", types.SimpleNamespace(cuda=types.SimpleNamespace(empty_cache=lambda: None)))
import fma_b200
from fma_b200 import _lib as L
from fma_b200.cumem import CuMemAllocator
from oracle import oracle as O
table = {models!r}[sys.argv[2]]
eng = fma_b200.Engine(0)
eng.set_option("pack", int(sys.argv[4]))
eng.set_option("load_chunk_bytes", 1 << 20)
for j, (tag, mib) in enumerate(table):
    i = eng.find(eng.alloc(mib << 20, tag))
    if tag == "weights":
        eng.write(i, O.bf16_weights((mib << 20) // 2, int(sys.argv[3]) + j).tobytes())
a = CuMemAllocator(engine=eng)
a._start_reserve()                                        # what the shim does when the weights pool closes
a.sleep(("weights",))
st = eng.stats()
assert eng.is_sleeping() and st["tier"] == L.FMA_TIER_HOST and eng.writeback(0)[0] == 1 and a._file_deposited, st
print("slept behind", flush=True)
sys.exit(0)                                               # atexit: the hook waits for the file
"""


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_shim_write_behind_deposit_waits_at_exit_and_the_agent_keeps_a_complete_file(built, tmp_path, pack):
    from tests.test_warm_start import MODELS, _last_json, _Node

    n = _Node(tmp_path)
    try:
        behind = n.script.with_name("behind.py")
        behind.write_text(_SHIM_INSTANCE.format(root=ROOT, models=MODELS))
        script = n.script
        n.script = behind
        r = n.run("Iwb", "sleep", "m1", 1, pack, env={"FMA_FILE_WRITE_BEHIND": "1", "FMA_WB_ITEM_DELAY_MS": "50", "FMA_FILE_BUFFERED": "1"})
        assert "slept behind" in r.stdout
        n.script = script
        kept = n.svc.kept()["images"]
        assert [(k["instance_id"], k["where"], k["packed"]) for k in kept] == [("Iwb", "disk", bool(pack))]
        import fma_b200

        assert fma_b200.Engine.image_file_info(n.svc._kept[("Iwb", 0)]["path"])["digests"]
        got = _last_json(n.run("Iwb", "adopt", "m1", 1, pack, env={"FMA_FILE_BUFFERED": "1"}))
        assert got["adopted"] and got["oracle"] and got["after"], got
    finally:
        n.close()


def test_write_behind_routes():
    """The write-behind case of sleep_route in csrc/fma_layout.h (tests/cpp/write_behind_route_test.cpp)."""
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"write_behind_route_test_{os.getpid()}")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "write_behind_route_test.cpp"), "-o", exe])
    try:
        assert "write-behind routes ok" in subprocess.check_output([exe], text=True)
    finally:
        os.unlink(exe)


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_wb") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS,
                           os.path.join(SIM, "hostsim_verify_kernels.cpp"), "-o", out, "-lpthread"])
    return out


def test_write_behind_against_the_host_simulated_engine(hostsim_lib, oracle):
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


def test_write_behind_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/write_behind_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"wb_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "hostsim_verify_kernels.cpp"),
                               os.path.join(SIM, "write_behind_sanitizer_test.cpp"), "-o", exe, "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_WB_ITEM_DELAY_MS"):
            env.pop(key, None)
        r = subprocess.run([exe, str(tmp_path / f"{san}.fmaimg")], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "write-behind sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
