"""Resident share (option "resident_bytes" / FMA_RESIDENT_MIB): a host-tier sleep keeps the tail of its image in the GPU's own
HBM, within a cap, so that a wake moves fewer bytes over PCIe.  The device tests (-m gpu on an H100) compare the engine's split,
host store, statistics and restored bytes with the oracle; test_resident_share_against_the_host_simulated_engine runs the same
tests on CPU against the host-simulated engine (tests/cpp/hostsim)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.pagegen import pages_of, repeat_page

PAGE = 2 << 20
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _L():
    from fma_b200 import _lib as L

    return L


def _n_gpus():
    if os.environ.get("FMA_HOSTSIM") == "1":
        return int(os.environ.get("HOSTSIM_DEVICES", "2"))
    import torch

    return torch.cuda.device_count()


def _load(engine, oracle, bf16):
    """tiny-llama-test table: nine weight segments (2..32 MiB) and two kv_cache segments.  bf16=True: dummy bf16 weights that
    the PACKED form codes (U(-1e-3, 1e-3)), every page of them distinct (tests/pagegen.py), else K0 fill."""
    from fma_b200 import workloads as W

    table = W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2)
    ptrs = [engine.alloc(s.bytes, s.tag) for s in table]
    ref, first = {}, 0
    for i, s in enumerate(table):
        if s.tag != "weights":
            continue
        if bf16:
            ref[i] = repeat_page(oracle.bf16_weights(1 << 20, 300 + i), s.bytes, seed=300, first_page=first)
            first += s.bytes // PAGE
            engine.write(i, ref[i].tobytes())
        else:
            engine.fill(i, 1234, first)
            ref[i] = oracle.fill(s.bytes, 1234, first)
            first += s.bytes // 8
    return table, ptrs, ref


def _resident_split(stored_sizes, budget):
    """The split rule, restated independently of the engine: which offloaded segments (image order, each given by its stored
    size) a host-tier sleep keeps in the GPU's own HBM under option resident_bytes = budget.  The cap is rounded down to 2 MiB;
    from the last segment back to the first, a segment stays when its stored size still fits what is left, a segment that does
    not fit is skipped."""
    left = budget // PAGE * PAGE
    keep = [False] * len(stored_sizes)
    for k in range(len(stored_sizes) - 1, -1, -1):
        if stored_sizes[k] <= left:
            keep[k] = True
            left -= stored_sizes[k]
    return keep


def _host_image(engine):
    base, n = engine.host_store_view()
    return np.ctypeslib.as_array((C.c_uint8 * n).from_address(base)).copy() if n else np.empty(0, np.uint8)


def _same_stored_page(a, b):
    from tests.test_gpu_parity import _same_stored_page as same

    return same(a, b)


def _check_restored(engine, oracle, ptrs, ref):
    assert not engine.is_sleeping()
    assert [s.va for s in engine.segments()] == ptrs
    got = engine.digest_all(["weights"])
    for i in ref:
        assert got[i] == oracle.digest(ref[i]), i
        assert engine.read(i, ref[i].size) == ref[i].tobytes(), i


MODES = ["staged", "direct", "kernel", "noring"]   # noring: STAGED without HBM for a staging ring (FMA_NO_RING=1)
BUDGETS = ["zero", "below_smallest", "one_segment", "mid", "everything"]


@gpu
@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("pack", [0, 1])
def test_resident_share_roundtrip_matches_oracle(engine, oracle, monkeypatch, pack, mode, budget):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    engine.set_option("mode", {"staged": L.FMA_MODE_STAGED, "direct": L.FMA_MODE_DIRECT, "kernel": L.FMA_MODE_KERNEL, "noring": L.FMA_MODE_STAGED}[mode])
    engine.set_option("pack", pack)
    engine.set_option("chunk_bytes", 8 << 20)   # several ring slots and several resident pieces
    if mode == "noring":
        monkeypatch.setenv("FMA_NO_RING", "1")
    coded = pack and mode in ("staged", "noring")           # the stored sizes the split counts: the PACKED form's when this sleep codes
    stored_pages = {i: [oracle.pack_page(p) if coded else p for p in pages_of(ref[i])] for i in widx}
    stored = [sum(p.size for p in stored_pages[i]) for i in widx]
    W = sum(ref[i].size for i in widx)
    cap = {"zero": 0, "below_smallest": (min(stored) - 1) // PAGE * PAGE, "one_segment": -(-stored[-1] // PAGE) * PAGE,
           "mid": sum(stored) // 2 // PAGE * PAGE, "everything": W}[budget]
    engine.set_option("resident_bytes", cap + (PAGE - 1))   # rounded down to 2 MiB
    keep = _resident_split(stored, cap)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    st = engine.stats()
    segs = engine.segments()
    assert engine.is_sleeping() and st["hbm_mapped_bytes"] == 0 and st["sleep_bytes_offloaded"] == W
    assert [segs[i].tier == L.FMA_TIER_LOCAL for i in widx] == keep                                  # the oracle's split
    res_stored = sum(s for s, k in zip(stored, keep) if k)
    host = [i for i, k in zip(widx, keep) if not k]
    host_packed = coded and mode == "staged"                  # without a ring the host part goes plain; the resident part stays coded
    assert st["resident_bytes"] == res_stored
    assert st["image_packed"] == (1 if host_packed and host else 0)
    host_stored = [p for i in host for p in (stored_pages[i] if host_packed else pages_of(ref[i]))]
    assert st["image_store_bytes"] == sum(p.size for p in host_stored)
    if budget == "zero" or (budget == "below_smallest" and not any(keep)):
        assert st["resident_bytes"] == 0 and all(s.tier == L.FMA_TIER_HOST for s in segs if s.has_backup)
    if budget == "everything":
        assert all(keep) and st["image_store_bytes"] == 0
    img = _host_image(engine) if host else np.empty(0, np.uint8)   # (an empty host part needs no store at all)
    if host_packed:
        off, nb = engine.image_pages()
        assert nb[:len(host_stored)] == [p.size for p in host_stored]
        assert all(_same_stored_page(img[o:o + n], w) for o, n, w in zip(off, nb, host_stored))
    else:
        assert np.array_equal(img, oracle.packed_image([ref[i] for i in host]))   # the host store holds the host segments only
    if any(keep):
        off, nb = engine.image_pages()
        n_host_pages = sum(ref[i].size // PAGE for i in host)
        res_sizes = [p.size for i in widx if keep[widx.index(i)] for p in stored_pages[i]]
        assert nb[n_host_pages:] == res_sizes and off[n_host_pages:] == [sum(res_sizes[:k]) for k in range(len(res_sizes))]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    st = engine.stats()
    assert st["resident_bytes"] == 0 and st["wake_bytes_restored"] == W
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"]); engine.wake(None)             # a second cycle from the woken state (merged runs)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_resident_share_off_by_default_and_timeline(engine, oracle):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.sleep(["weights"])
    assert engine.stats()["resident_bytes"] == 0 and all(s.tier == L.FMA_TIER_HOST for s in engine.segments() if s.has_backup)
    assert not any(r["kind"].startswith("res_") for r in engine.timeline())
    engine.wake(None)
    engine.set_option("resident_bytes", 64 << 20)
    engine.set_option("chunk_bytes", 8 << 20)
    engine.sleep(["weights"])
    kinds = [r["kind"] for r in engine.timeline()]
    assert "res_alloc" in kinds and "res_gather" in kinds
    engine.wake(None)
    tl = engine.timeline()
    kinds = [r["kind"] for r in tl]
    assert "res_restore" in kinds and "res_free" in kinds
    free = [r for r in tl if r["kind"] == "res_free"][0]
    restore_end = max(r["t1_ms"] for r in tl if r["kind"] == "res_restore")
    total = [r for r in tl if r["kind"] == "total"][0]
    assert restore_end <= free["t0_ms"] + 1e-3 and free["t1_ms"] <= total["t1_ms"]
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("first", ["kv_cache", "weights"])
def test_resident_share_tag_selective_retried_and_kept_wakes(engine, oracle, first):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("resident_bytes", 48 << 20)
    engine.sleep(["weights"])
    assert engine.stats()["resident_bytes"] > 0
    engine.wake([first])
    if first == "kv_cache":                                  # the weights still sleep: the buffer stays
        assert engine.stats()["resident_bytes"] > 0 and engine.is_sleeping()
    engine.wake(["weights" if first == "kv_cache" else "kv_cache"])
    engine.wake(None)                                        # a retried wake finds nothing left to do
    assert engine.stats()["resident_bytes"] == 0
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"])
    engine.wake(None, flags=L.FMA_FLAG_KEEP_BACKUP)          # the buffer is kept ...
    assert engine.stats()["resident_bytes"] > 0
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"])                                # ... until the next sleep gathers afresh
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    assert engine.stats()["resident_bytes"] == 0
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_resident_share_incremental_sleep(engine, oracle, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    engine.set_option("mode", L.FMA_MODE_STAGED)
    engine.set_option("pack", pack)
    engine.set_option("incremental", 1)
    engine.set_option("resident_bytes", 48 << 20)
    engine.sleep(["weights"])
    assert engine.stats()["sleep_bytes_copied"] == engine.stats()["image_store_bytes"] > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    engine.sleep(["weights"])                                # clean: no byte into the host store, the resident part gathered again
    st = engine.stats()
    assert st["sleep_bytes_copied"] == 0 and st["resident_bytes"] > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    segs = engine.segments()
    engine.sleep(["weights"]); segs = engine.segments(); engine.wake(None)
    res_i = next(i for i in widx if segs[i].tier == L.FMA_TIER_LOCAL)
    host_i = next(i for i in widx if segs[i].tier == L.FMA_TIER_HOST)
    for i, at in ((res_i, 4321), (host_i, 777)):             # one changed byte in a resident and in a host segment
        ref[i] = ref[i].copy(); ref[i][at] ^= 0x01
        engine.write(i, ref[i].tobytes())
    engine.sleep(["weights"])
    assert engine.stats()["sleep_bytes_copied"] > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"]); assert engine.stats()["sleep_bytes_copied"] == 0
    engine.wake(None)
    engine.set_option("resident_bytes", 16 << 20)            # a different split: a full sleep
    engine.sleep(["weights"])
    st = engine.stats()
    assert st["sleep_bytes_copied"] == st["image_store_bytes"] > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_resident_share_refuses_hand_over_until_it_is_off(engine, oracle, monkeypatch, tmp_path):
    L = _L()
    monkeypatch.setenv("FMA_HOST_STORE_SHM", "1")
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("resident_bytes", 48 << 20)
    engine.sleep(["weights"])
    before = (engine.stats()["resident_bytes"], engine.stats()["image_store_bytes"], [s.tier for s in engine.segments()])
    for call in (engine.image_export, lambda: engine.image_describe(L.FMA_TIER_HOST), engine.host_store_share,
                 lambda: engine.image_save(str(tmp_path / "img"))):
        with pytest.raises(L.FmaError) as ei:
            call()
        assert ei.value.code == L.FMA_ESTATE and "resident" in ei.value.message
    assert engine.is_sleeping() and (engine.stats()["resident_bytes"], engine.stats()["image_store_bytes"], [s.tier for s in engine.segments()]) == before
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.set_option("resident_bytes", 0)
    engine.sleep(["weights"])
    os.close(engine.image_export())
    assert len(engine.image_describe(L.FMA_TIER_HOST)) > 0
    os.close(engine.host_store_share())
    engine.wake(None)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_resident_share_swap_free_level2_and_destroy_while_asleep(built, oracle):
    import fma_b200

    L = _L()
    a, b = fma_b200.Engine(0), fma_b200.Engine(0)
    try:
        ta, pa, ra = _load(a, oracle, bf16=False)
        tb, pb, rb = _load(b, oracle, bf16=True)
        for e in (a, b):
            e.set_option("resident_bytes", 40 << 20)
        b.sleep(["weights"])
        a.swap_out_for(b, offload_tags=("weights",), flags=L.FMA_FLAG_VERIFY)
        assert a.is_sleeping() and a.stats()["resident_bytes"] > 0
        _check_restored(b, oracle, pb, rb)
        b.swap_out_for(a, offload_tags=("weights",), flags=L.FMA_FLAG_VERIFY)
        _check_restored(a, oracle, pa, ra)
        a.sleep([])                                          # level 2: nothing offloaded, nothing resident
        assert a.stats()["resident_bytes"] == 0 and a.stats()["sleep_bytes_offloaded"] == 0
        a.wake(None)
        for i in ra:                                         # (level 2 discarded the weights)
            a.write(i, ra[i].tobytes())
        a.sleep(["weights"])
        last = max(i for i in ra if a.segment(i).tier == L.FMA_TIER_LOCAL)
        a.free(pa[last])                                     # free a resident segment while asleep
        del ra[last]
        pa.pop(last)
        a.wake(None, flags=L.FMA_FLAG_VERIFY)
        ra = {(i if i < last else i - 1): v for i, v in ra.items()}
        _check_restored(a, oracle, pa, ra)
        a.sleep(["weights"])
    finally:
        a.close()                                            # destroyed while asleep with a resident buffer
        b.close()


@gpu
@pytest.mark.parametrize("tier", ["local", "peer", "paths"])
def test_resident_share_is_ignored_by_parking_tiers_and_paths(engine, oracle, tier):
    L = _L()
    if tier in ("peer", "paths") and _n_gpus() < 2:
        pytest.skip("needs a second GPU")
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    engine.set_option("resident_bytes", 48 << 20)
    t = L.FMA_TIER_HOST
    if tier == "local":
        t = L.FMA_TIER_LOCAL
    elif tier == "peer":
        engine.peer_reserve(1, sum(ref[i].size for i in ref))
        t = L.FMA_TIER_PEER
    else:
        engine.set_paths([1])
    engine.sleep(["weights"], tier=t)
    st = engine.stats()
    assert st["resident_bytes"] == 0 and all(s.tier == t for s in engine.segments() if s.has_backup)
    assert not any(r["kind"].startswith("res_") for r in engine.timeline())
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_resident_share_through_the_environment(built, oracle, monkeypatch):
    import fma_b200

    monkeypatch.setenv("FMA_RESIDENT_MIB", "48")
    with fma_b200.Engine(0) as e:
        table, ptrs, ref = _load(e, oracle, bf16=False)
        e.sleep(["weights"])
        assert 0 < e.stats()["resident_bytes"] <= 48 << 20
        e.wake(None)
        _check_restored(e, oracle, ptrs, ref)


@gpu
def test_resident_share_in_the_compiled_server(built, oracle, tmp_path):
    """fma_served with FMA_RESIDENT_MIB set: /stats shows the resident part while asleep, /digests are those of the oracle's
    fill before the sleep and after /wake_up twice."""
    import json
    import urllib.request

    exe = os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "fma_served")
    if os.environ.get("FMA_HOSTSIM") == "1":   # the same server over the host-simulated library
        lib = os.environ["FMA_B200_LIB"]
        exe = str(tmp_path / "fma_served_hostsim")
        subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc", "fma_served.cpp"),
                               lib, "-Wl,-rpath," + os.path.dirname(lib), "-o", exe, "-lpthread"])

    def call(base, method, path):
        req = urllib.request.Request(base + path, data=b"" if method == "POST" else None, method=method)
        with urllib.request.urlopen(req, timeout=60) as r:
            return r.status, r.read()

    mib = [6, 2, 4]
    p = subprocess.Popen([exe, "--port", "0", "--device", "0", "--seg", "weights:6", "--seg", "weights:2", "--seg", "kv_cache:8", "--seg", "weights:4",
                          "--seed", "1234"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=dict(os.environ, FMA_RESIDENT_MIB="6"))
    try:
        line = p.stdout.readline()
        assert line.startswith("listening on "), line + p.stderr.read()
        base = f"http://127.0.0.1:{int(line.split()[-1])}"
        want, first = [], 0
        for n in mib:
            want.append(oracle.digest(oracle.fill(n << 20, 1234, first)))
            first += (n << 20) // 8
        assert [int(x, 16) for x in json.loads(call(base, "GET", "/digests")[1])[0]] == want
        assert call(base, "POST", "/sleep") == (200, b"")
        st = json.loads(call(base, "GET", "/stats")[1])["ranks"][0]
        assert st["resident_bytes"] == 6 << 20 and st["image_store_bytes"] == 6 << 20 and st["hbm_mapped_bytes"] == 0   # 4 + 2 MiB stay
        assert call(base, "POST", "/wake_up") == (200, b"") and call(base, "POST", "/wake_up") == (200, b"")
        assert json.loads(call(base, "GET", "/stats")[1])["ranks"][0]["resident_bytes"] == 0
        assert [int(x, 16) for x in json.loads(call(base, "GET", "/digests")[1])[0]] == want
    finally:
        p.terminate()
        try:
            p.wait(timeout=30)
        except subprocess.TimeoutExpired:
            p.kill()
    assert p.returncode == 0, p.stderr.read()[-2000:]


def test_resident_split_rule():
    M = PAGE
    assert _resident_split([4 * M, 2 * M, 6 * M], 0) == [False, False, False]
    assert _resident_split([4 * M, 2 * M, 6 * M], 6 * M) == [False, False, True]
    assert _resident_split([4 * M, 2 * M, 6 * M], 7 * M) == [False, False, True]          # what is left fits nothing
    assert _resident_split([4 * M, 2 * M, 6 * M], 9 * M) == [False, True, True]           # 4 MiB does not fit the last 3: skipped
    assert _resident_split([4 * M, 2 * M, 6 * M], 12 * M + M - 1) == [True, True, True]
    assert _resident_split([3 << 20, 3 << 20], (6 << 20) + (1 << 20)) == [True, True]        # cap rounded down to 2 MiB: 6 MiB
    assert _resident_split([3 << 20, 3 << 20], 5 << 20) == [False, True]


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_res") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS, "-o", out, "-lpthread"])
    return out


def test_resident_share_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2")
    env.pop("FMA_RESIDENT_MIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout and "skipped" not in r.stdout, tail


def test_resident_share_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/resident_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SIM, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"resident_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "resident_sanitizer_test.cpp"),
                               "-o", exe, "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        env.pop("FMA_RESIDENT_MIB", None)
        r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "resident sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
