"""fma_image_move: a sleeping model's image moves between host DRAM, a file and a parking buffer without a wake.  The device tests
(-m gpu on an H100) check the reported tier, the bytes in the destination store against the oracle and the weights restored by the
next wake; test_image_move_against_the_host_simulated_engine runs the same tests on CPU against the host-simulated engine with two
simulated GPUs (the peer cases skip on a one-GPU box), and tests/cpp/hostsim/move_sanitizer_test.cpp runs the failure scenarios
under ThreadSanitizer and ASan+UBSan+LeakSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.test_file_tier import _ADOPT_CHILD, _check_file, _stored_pages
from tests.test_resident_share import _check_restored, _load, _same_stored_page

PAGE = 2 << 20
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _L():
    from fma_b200 import _lib as L

    return L


def _tier(name):
    L = _L()
    return {"host": L.FMA_TIER_HOST, "peer": L.FMA_TIER_PEER, "local": L.FMA_TIER_LOCAL, "file": L.FMA_TIER_FILE}[name]


def _check_host(engine, oracle, ref, widx, packed):
    """The host store holds the image in the form the engine reports."""
    base, n = engine.host_store_view()
    img = np.ctypeslib.as_array((C.c_uint8 * n).from_address(base))
    assert n == engine.stats()["image_store_bytes"]
    if packed:
        want = _stored_pages(oracle, ref, widx, True)
        off, nb = engine.image_pages()
        assert nb == [p.size for p in want]
        assert all(_same_stored_page(img[o:o + k], w) for o, k, w in zip(off, nb, want))
    else:
        assert np.array_equal(img, oracle.packed_image([ref[i] for i in widx]))


def _reports(engine, tier):
    st = engine.stats()
    assert engine.is_sleeping() and st["tier"] == tier
    assert all(s.tier == tier for s in engine.segments() if s.has_backup)


def _sleep_to(engine, name, path, nbytes):
    L = _L()
    if name == "file":
        engine.file_store(path)
    if name == "peer":
        _peer(engine, nbytes)
    engine.sleep(["weights"], tier=_tier(name), flags=L.FMA_FLAG_VERIFY)
    _reports(engine, _tier(name))


def _peer(engine, nbytes):
    L = _L()
    try:
        engine.peer_reserve(1, nbytes)
    except L.FmaError as e:
        if e.code == L.FMA_EINVAL and "not visible" in e.message:
            pytest.skip("the peer tier needs a second GPU")
        raise


def _move_rows(engine):
    rows = engine.timeline()
    assert rows and all(r["op"] == "move" for r in rows)
    return {r["kind"]: r for r in rows}


DIRECTIONS = [("host", "file"), ("file", "host"), ("host", "local"), ("local", "host"), ("local", "file"), ("file", "local"),
              ("host", "peer"), ("peer", "host")]


@gpu
@pytest.mark.parametrize("src,dst", DIRECTIONS, ids=[f"{a}-{b}" for a, b in DIRECTIONS])
@pytest.mark.parametrize("pack", [0, 1])
def test_move_round_trip_matches_oracle(engine, oracle, tmp_path, pack, src, dst):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    W = sum(ref[i].size for i in widx)
    engine.set_option("pack", pack)
    engine.set_option("chunk_bytes", 6 << 20)              # several copy pieces, ragged against the segments
    engine.set_option("load_chunk_bytes", 1 << 20)
    engine.set_option("load_slots", 3)
    path = str(tmp_path / "m.fmaimg")
    _sleep_to(engine, src, path, W)
    before = engine.stats()
    S = before["image_store_bytes"]
    if dst == "file":
        engine.file_store(path)
    if dst == "peer":
        _peer(engine, S)
    engine.move_image(_tier(dst))
    _reports(engine, _tier(dst))
    st = engine.stats()
    assert st["image_store_bytes"] == S and st["image_packed"] == before["image_packed"] and st["hbm_mapped_bytes"] == 0
    rows = _move_rows(engine)
    assert rows["total"]["bytes"] == S
    assert ("file_io" in rows) == ("file" in (src, dst))
    assert ("copies_landed" in rows) == bool({"local", "peer"} & {src, dst})   # the copy engines run only for a parking buffer
    if dst == "host":
        _check_host(engine, oracle, ref, widx, st["image_packed"])
    if dst == "file":
        assert rows["file_io"]["bytes"] == S + (2 << 20)
        if src == "host":
            engine.host_release()                          # the image left the host store: its DRAM can go
        _check_file(engine, oracle, path, ref, widx, st["image_packed"])
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)             # the destination tier's route, digests from before the move
    assert engine.stats()["tier"] == _tier(dst) and engine.stats()["wake_bytes_restored"] == W
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=_tier(dst), flags=L.FMA_FLAG_VERIFY)   # and a second cycle in the new tier
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_move_chain_host_local_file_host(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    engine.set_option("pack", pack)
    engine.set_option("load_chunk_bytes", 1 << 20)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    S = engine.stats()["image_store_bytes"]
    engine.file_store(str(tmp_path / "chain.fmaimg"))
    for name in ("local", "file", "host"):
        engine.move_image(_tier(name))
        _reports(engine, _tier(name))
        assert engine.stats()["image_store_bytes"] == S
    _check_host(engine, oracle, ref, widx, engine.stats()["image_packed"])
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_move_holds_no_hbm_and_frees_the_source_store_on_release(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    aux = engine.stats()["hbm_aux_bytes"]
    with pytest.raises(L.FmaError) as ei:                  # the host store holds the sleeping image
        engine.host_release()
    assert ei.value.code == L.FMA_ESTATE
    engine.file_store(str(tmp_path / "m.fmaimg"))
    engine.move_image(L.FMA_TIER_FILE)
    st = engine.stats()
    assert st["hbm_mapped_bytes"] == 0 and st["hbm_aux_bytes"] == aux and st["host_store_bytes"] > 0   # the source stays allocated
    assert "copies_landed" not in _move_rows(engine)
    engine.host_release()
    assert engine.stats()["host_store_bytes"] == 0
    engine.move_image(L.FMA_TIER_HOST)                     # promoted back: a fresh host store, the file untouched
    st = engine.stats()
    assert st["hbm_mapped_bytes"] == 0 and st["hbm_aux_bytes"] == aux and st["host_store_bytes"] >= st["image_store_bytes"]
    engine.move_image(L.FMA_TIER_LOCAL)
    assert engine.stats()["parked_bytes"] >= engine.stats()["image_store_bytes"]
    with pytest.raises(L.FmaError) as ei:                  # the parking buffer holds the sleeping image
        engine.peer_release()
    assert ei.value.code == L.FMA_ESTATE
    engine.move_image(L.FMA_TIER_HOST)
    engine.peer_release()
    assert engine.stats()["parked_bytes"] == 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_move_refusals_leave_the_engine_unchanged(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)

    def refused(tier, code):
        before = [(s.mapped, s.has_backup, s.tier) for s in engine.segments()], engine.stats()["tier"]
        with pytest.raises(L.FmaError) as ei:
            engine.move_image(tier)
        assert ei.value.code == code, ei.value
        assert ([(s.mapped, s.has_backup, s.tier) for s in engine.segments()], engine.stats()["tier"]) == before

    refused(L.FMA_TIER_FILE, L.FMA_ESTATE)                 # nothing asleep
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    refused(7, L.FMA_EINVAL)                               # unknown tier
    refused(-1, L.FMA_EINVAL)
    refused(L.FMA_TIER_HOST, L.FMA_EINVAL)                 # the tier it is in
    refused(L.FMA_TIER_FILE, L.FMA_ESTATE)                 # no fma_file_store
    refused(L.FMA_TIER_PEER, L.FMA_ESTATE)                 # no peer parking buffer
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_LOCAL, flags=L.FMA_FLAG_VERIFY)
    refused(L.FMA_TIER_PEER, L.FMA_EINVAL)                 # one parking buffer: no PEER <-> LOCAL
    engine.wake(None, flags=L.FMA_FLAG_KEEP_BACKUP)        # mapped segments that keep their backup
    refused(L.FMA_TIER_HOST, L.FMA_ESTATE)
    _check_restored(engine, oracle, ptrs, ref)
    engine.file_store(str(tmp_path / "m.fmaimg"))
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    refused(L.FMA_TIER_FILE, L.FMA_EINVAL)                 # FILE -> FILE
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    engine.set_option("resident_bytes", 8 << 20)           # part of the image in a resident share
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    assert engine.stats()["resident_bytes"] > 0
    refused(L.FMA_TIER_FILE, L.FMA_ESTATE)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


_FSIZE_CHILD = r"""
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
try:
    eng.move_image(L.FMA_TIER_FILE)
    raise SystemExit("the move did not fail")
except L.FmaError as e:
    assert e.code == L.FMA_EIO, e
resource.setrlimit(resource.RLIMIT_FSIZE, (resource.RLIM_INFINITY, resource.RLIM_INFINITY))
st = eng.stats()
assert st["tier"] == L.FMA_TIER_HOST and all(s.tier == L.FMA_TIER_HOST for s in eng.segments() if s.has_backup), st
eng.wake(None, flags=L.FMA_FLAG_VERIFY)                    # from where it was
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
try:
    eng.image_adopt_file(sys.argv[1], ["weights"])
    raise SystemExit("the partial file was adopted")
except L.FmaError as e:
    assert e.code in (L.FMA_EINVAL, L.FMA_EIO), e
assert not eng.is_sleeping()
eng.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)            # with room again the same move works
eng.move_image(L.FMA_TIER_FILE)
eng.host_release()
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
dg = eng.digest_all(["weights"])
assert all(dg[i] == ref[i] for i in ref)
print("move fsize ok", flush=True)
"""


@gpu
def test_move_to_a_file_that_cannot_be_written_leaves_the_image_in_place(built, tmp_path):
    child = tmp_path / "child.py"
    child.write_text(_FSIZE_CHILD.format(root=ROOT))
    r = subprocess.run([sys.executable, str(child), str(tmp_path / "m.fmaimg")], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0 and "move fsize ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


@gpu
@pytest.mark.parametrize("dst", ["host", "local"])
def test_move_from_a_truncated_file_fails_and_retries(engine, oracle, tmp_path, dst):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("load_chunk_bytes", 1 << 20)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    keep = str(tmp_path / "keep")
    shutil.copyfile(path, keep)
    os.truncate(path, engine.stats()["image_store_bytes"] // 2 + 1000)
    with pytest.raises(L.FmaError) as ei:
        engine.move_image(_tier(dst))
    assert ei.value.code == L.FMA_EIO
    _reports(engine, L.FMA_TIER_FILE)
    st = engine.stats()
    assert st["host_store_bytes"] == 0 and st["parked_bytes"] == 0   # what the move created went with it
    shutil.copyfile(keep, path)
    engine.move_image(_tier(dst))
    _reports(engine, _tier(dst))
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_file_written_by_a_move_is_adopted_in_a_fresh_process(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    path = str(tmp_path / "m.fmaimg")
    engine.file_store(path)
    engine.move_image(L.FMA_TIER_FILE)
    child = tmp_path / "child.py"
    child.write_text(_ADOPT_CHILD.format(root=ROOT))
    r = subprocess.run([sys.executable, str(child), path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    import json

    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert [got[i] for i in sorted(ref)] == [oracle.digest(ref[i]) for i in sorted(ref)]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_move_with_incremental_sleeps(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.set_option("incremental", 1)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.file_store(str(tmp_path / "m.fmaimg"))
    widx = sorted(ref)
    for k, (first, moves, again) in enumerate([("host", ["file"], "file"), ("host", ["file", "host"], "host"), ("file", ["local"], "local")]):
        engine.sleep(["weights"], tier=_tier(first), flags=L.FMA_FLAG_VERIFY)
        for name in moves:
            engine.move_image(_tier(name))
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(engine, oracle, ptrs, ref)
        i = widx[1 + k]                                    # one changed segment
        ref[i] = ref[i].copy()
        ref[i][4321 + k] ^= 0x01
        engine.write(i, ref[i].tobytes())
        engine.sleep(["weights"], tier=_tier(again), flags=L.FMA_FLAG_VERIFY)
        assert engine.stats()["sleep_bytes_copied"] > 0
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_restored(engine, oracle, ptrs, ref)
        engine.sleep(["weights"], tier=_tier(again), flags=L.FMA_FLAG_VERIFY)   # unchanged since: a clean sleep is still exact
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
a.move_image("file")
st = eng.stats()
path = os.path.join(os.environ["FMA_FILE_DIR"], "Imove-r0.fmaimg")
print("demoted", st["tier"], st["host_store_bytes"], os.path.getsize(path) == st["image_store_bytes"] + (2 << 20), flush=True)
a.move_image("host")
print("promoted", eng.stats()["tier"], os.path.exists(path), flush=True)
a.wake_up(None)
assert eng.digest_all(["weights"]) == before
"""


def test_shim_move_image_names_the_file_and_removes_it_at_exit(hostsim_lib, tmp_path):
    L = _L()
    child = tmp_path / "child.py"
    child.write_text(_SHIM_CHILD.format(root=ROOT))
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="1", FMA_TIER="host", FMA_INSTANCE_ID="Imove", RANK="0")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_NODE_AGENT_SOCK", "FMA_REMOTE_PATHS", "LOCAL_RANK", "FMA_PREPIN"):
        env.pop(key, None)
    d = tmp_path / "images"
    d.mkdir()
    r = subprocess.run([sys.executable, str(child)], env=dict(env, FMA_FILE_DIR=str(d)), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert f"demoted {L.FMA_TIER_FILE} 0 True" in r.stdout and f"promoted {L.FMA_TIER_HOST} True" in r.stdout, r.stdout
    assert os.listdir(d) == []                               # removed at exit


def test_move_routes():
    """move_route in csrc/fma_layout.h against its restatement (tests/cpp/move_route_test.cpp)."""
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"move_route_test_{os.getpid()}")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "move_route_test.cpp"), "-o", exe])
    try:
        assert "move routes ok" in subprocess.check_output([exe], text=True)
    finally:
        os.unlink(exe)


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_move") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS, "-o", out, "-lpthread"])
    return out


def test_image_move_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout and "SKIPPED" not in r.stdout, tail   # two simulated GPUs: the peer cases run


def test_image_move_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/move_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SIM, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"move_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "move_sanitizer_test.cpp"), "-o", exe, "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED"):
            env.pop(key, None)
        r = subprocess.run([exe, str(tmp_path / f"{san}.fmaimg")], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "move sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
