"""Every page of a PACKED image or resident share wakes in its own place (run with -m gpu on an H100).

The segments here are 5 to 9 pages long, mix coded and raw pages, and every page of them is distinct (tests/pagegen.py), so a
page restored to another page's place within its segment shows up in the bytes read back.  chunk_bytes is 6 MiB, so ring slots,
resident pieces and K4 / K5 batches end inside segments.  The cases:
  - the resident share at a mid budget, pack 1, modes staged / noring / kernel, woken tag by tag and kept (FMA_FLAG_KEEP_BACKUP);
  - an INCREMENTAL packed sleep after one page in the middle of a segment changed: its segment is re-coded in place;
  - a packed image saved to a file and loaded, and handed over to another engine.
Every byte read back is compared with the reference, and every host-image stored page with the oracle's.
test_page_placement_against_the_host_simulated_engine runs the same tests on CPU against the host-simulated engine."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.pagegen import PAGE, all_distinct, pages_of, stamp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu

SEG_PAGES = [5, 7, 6, 9, 6]        # weight segments; a kv_cache segment sits after the second
CODED = [0, 1, 2, 3, 4, 5, 7, 8]   # _pack_pages kinds the PACKED code codes
RAW = [6, 9, 10]                   # ... and the ones it stores raw
CHUNK = 6 << 20


def _L():
    from fma_b200 import _lib as L

    return L


def _kinds(i, n):
    """Page kinds of weight segment i: a raw page at every fourth position (shifted per segment), coded pages around it."""
    return [RAW[(i + j) % 3] if (i + j) % 4 == 2 else CODED[(3 * i + j) % len(CODED)] for j in range(n)]


def _load(engine, oracle):
    """Allocate the table and write distinct pages; returns (weight segment indices, reference bytes by segment index)."""
    from tests.test_gpu_parity import _pack_pages

    pool = _pack_pages(oracle)
    widx, ref, first = [], {}, 0
    for i, n in enumerate(SEG_PAGES):
        engine.alloc(n * PAGE, "weights")
        k = engine.segment_count() - 1
        widx.append(k)
        ref[k] = stamp(np.concatenate([pool[x] for x in _kinds(i, n)]), 41, first)
        first += n
        if i == 1:
            engine.alloc(4 * PAGE, "kv_cache")
    for k in widx:
        engine.write(k, ref[k].tobytes())
    assert all_distinct([p for k in widx for p in pages_of(ref[k])])
    return widx, ref


def _stored(oracle, ref, widx):
    return {k: [oracle.pack_page(p) for p in pages_of(ref[k])] for k in widx}


def _check_bytes(engine, ref):
    for k in ref:
        got = np.frombuffer(engine.read(k, ref[k].size), np.uint8)
        bad = [j for j, (a, b) in enumerate(zip(pages_of(got), pages_of(ref[k]))) if not np.array_equal(a, b)]
        assert not bad, f"segment {k}: pages {bad} differ"


def _check_host_image(engine, oracle, ref, host, stored, packed):
    """The host store holds the pages of the `host` segments, in image order: the oracle's stored pages (packed) or verbatim."""
    from tests.test_gpu_parity import _host_image, _same_stored_page

    img = _host_image(engine)
    if packed:
        want = [p for k in host for p in stored[k]]
        off, nb = engine.image_pages()
        assert nb[:len(want)] == [w.size for w in want]
        bad = [q for q, (o, n, w) in enumerate(zip(off, nb, want)) if not _same_stored_page(img[o:o + n], w)]
        assert not bad, f"host image pages {bad} are not the oracle's"
    else:
        assert np.array_equal(img[:sum(ref[k].size for k in host)], oracle.packed_image([ref[k] for k in host]))


@gpu
@pytest.mark.parametrize("mode", ["staged", "noring", "kernel"])
def test_resident_mid_budget_pages_wake_in_place(engine, oracle, monkeypatch, mode):
    from tests.test_resident_share import _resident_split

    L = _L()
    widx, ref = _load(engine, oracle)
    engine.set_option("mode", L.FMA_MODE_KERNEL if mode == "kernel" else L.FMA_MODE_STAGED)
    engine.set_option("pack", 1)
    engine.set_option("chunk_bytes", CHUNK)
    if mode == "noring":
        monkeypatch.setenv("FMA_NO_RING", "1")
    coded = mode != "kernel"                                  # the resident part is coded when the sleep codes
    stored = _stored(oracle, ref, widx)
    sizes = [sum(p.size for p in stored[k]) if coded else ref[k].size for k in widx]
    cap = sum(sizes) // 2 // PAGE * PAGE
    keep = _resident_split(sizes, cap)
    assert any(keep) and not all(keep)
    engine.set_option("resident_bytes", cap)
    for cycle in range(2):
        engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
        st = engine.stats()
        assert [engine.segment(k).tier == L.FMA_TIER_LOCAL for k in widx] == keep
        assert st["resident_bytes"] == sum(s for s, r in zip(sizes, keep) if r)
        host = [k for k, r in zip(widx, keep) if not r]
        host_packed = mode == "staged"                        # without a ring the host part goes plain
        assert st["image_packed"] == int(host_packed)
        _check_host_image(engine, oracle, ref, host, stored, host_packed)
        off, nb = engine.image_pages()
        res_sizes = [p.size if coded else PAGE for k, r in zip(widx, keep) if r for p in stored[k]]
        n_host = sum(ref[k].size for k in host) // PAGE
        assert nb[n_host:] == res_sizes and off[n_host:] == [sum(res_sizes[:q]) for q in range(len(res_sizes))]
        engine.wake(["kv_cache"])                             # the weights still sleep: the resident buffer stays
        assert engine.is_sleeping() and engine.stats()["resident_bytes"] > 0
        engine.wake(["weights"], flags=L.FMA_FLAG_VERIFY | L.FMA_FLAG_KEEP_BACKUP)
        assert not engine.is_sleeping() and engine.stats()["resident_bytes"] > 0
        _check_bytes(engine, ref)
        engine.wake(None)                                     # a retried wake finds nothing left to do
        _check_bytes(engine, ref)
        # while awake, a page in the middle of a resident segment changes: the next sleep gathers afresh, not the kept buffer
        k = next(k for k, r in zip(widx, keep) if r)
        j = len(pages_of(ref[k])) // 2
        ref[k] = ref[k].copy()
        ref[k][j * PAGE:(j + 1) * PAGE] = stamp(ref[k][j * PAGE:(j + 1) * PAGE], 43, 100 + cycle)
        engine.write(k, ref[k].tobytes())
        stored = _stored(oracle, ref, widx)
    engine.sleep(["weights"])
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    assert engine.stats()["resident_bytes"] == 0
    _check_bytes(engine, ref)


@gpu
@pytest.mark.parametrize("resident", [False, True])
def test_incremental_packed_sleep_recodes_a_changed_segment_in_place(engine, oracle, resident):
    from tests.test_resident_share import _resident_split

    L = _L()
    widx, ref = _load(engine, oracle)
    engine.set_option("mode", L.FMA_MODE_STAGED)
    engine.set_option("pack", 1)
    engine.set_option("chunk_bytes", CHUNK)
    engine.set_option("incremental", 1)
    stored = _stored(oracle, ref, widx)
    sizes = [sum(p.size for p in stored[k]) for k in widx]
    keep = [False] * len(widx)
    if resident:
        cap = -(-(sizes[-1] + sizes[-2]) // PAGE) * PAGE      # the last two segments stay on the GPU
        keep = _resident_split(sizes, cap)
        assert keep == [False, False, False, True, True]
        engine.set_option("resident_bytes", cap)
    host = [k for k, r in zip(widx, keep) if not r]
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)        # a full sleep seeds the kept image
    assert engine.stats()["image_packed"] == 1
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_bytes(engine, ref)
    for k in (host[1], host[-1]):                             # a page in the middle of a host segment gets new bytes, same stored size
        j = len(pages_of(ref[k])) // 2
        assert stored[k][j].size < PAGE                       # (a coded page)
        ref[k] = ref[k].copy()
        ref[k][j * PAGE:(j + 1) * PAGE] = stamp(ref[k][j * PAGE:(j + 1) * PAGE], 47, k)
        engine.write(k, ref[k].tobytes())
        stored = _stored(oracle, ref, widx)
        ops0 = engine.stats()["total_copy_ops"]
        engine.sleep(["weights"])
        st = engine.stats()
        assert st["image_packed"] == 1 and st["sleep_bytes_copied"] == sum(p.size for p in stored[k])   # that segment only
        assert st["total_copy_ops"] - ops0 >= 1
        _check_host_image(engine, oracle, ref, host, stored, True)                                     # the whole kept image is current
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        _check_bytes(engine, ref)
    engine.sleep(["weights"])
    assert engine.stats()["sleep_bytes_copied"] == 0
    engine.wake(None)
    _check_bytes(engine, ref)


@gpu
@pytest.mark.parametrize("how", ["save_load", "hand_over"])
def test_packed_image_moves_to_a_fresh_engine_with_every_page_in_place(engine, oracle, monkeypatch, tmp_path, how):
    import fma_b200

    L = _L()
    monkeypatch.setenv("FMA_HOST_STORE_SHM", "1")
    widx, ref = _load(engine, oracle)
    engine.set_option("mode", L.FMA_MODE_STAGED)
    engine.set_option("pack", 1)
    engine.set_option("chunk_bytes", CHUNK)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    assert engine.stats()["image_packed"] == 1
    stored = _stored(oracle, ref, widx)
    _check_host_image(engine, oracle, ref, widx, stored, True)
    want = engine.stats()["image_store_bytes"]
    fd = -1
    if how == "save_load":
        path = str(tmp_path / "model.fmaimage")
        engine.image_save(path)
    else:
        fd = engine.image_export()
    try:
        with fma_b200.Engine(0) as fresh:
            for n in SEG_PAGES[:2]:
                fresh.alloc(n * PAGE, "weights")
            fresh.alloc(4 * PAGE, "kv_cache")
            for n in SEG_PAGES[2:]:
                fresh.alloc(n * PAGE, "weights")
            fresh.set_option("chunk_bytes", CHUNK)
            if how == "save_load":
                fresh.image_load(path, ["weights"])
            else:
                fresh.image_adopt(fd, ["weights"])
            assert fresh.is_sleeping() and fresh.stats()["image_packed"] == 1 and fresh.stats()["image_store_bytes"] == want
            _check_host_image(fresh, oracle, ref, widx, stored, True)
            fresh.wake(None, flags=L.FMA_FLAG_VERIFY)
            _check_bytes(fresh, ref)
    finally:
        if fd >= 0:
            os.close(fd)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)                 # the owner still wakes from its own image
    _check_bytes(engine, ref)


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_place") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS, "-o", out, "-lpthread"])
    return out


def test_page_placement_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2")
    env.pop("FMA_RESIDENT_MIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout and "skipped" not in r.stdout, tail
