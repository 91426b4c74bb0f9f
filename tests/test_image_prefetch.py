"""fma_image_prefetch: part or all of a sleeping image is copied into its own GPU's HBM ahead of a wake, and dropped again, without
waking it.  The device tests (-m gpu on an H100) prefetch plain and PACKED images (bf16 pages from tests/pagegen.py, raw pages mixed
in) from the host store and from a file, check the split against its restatement, the wake against the oracle and the bytes the
link or the disk still moves, and cover repeats, tag-selective and KEEP_BACKUP wakes, INCREMENTAL sleeps, moves, frees, adoption,
verification, refusals and failures.  test_image_prefetch_against_the_host_simulated_engine runs the same tests on CPU against the
host-simulated engine, and tests/cpp/hostsim/prefetch_sanitizer_test.cpp runs the failure scenarios under ThreadSanitizer and
ASan+UBSan+LeakSan."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import pytest

from tests.test_file_tier import _ADOPT_CHILD
from tests.test_image_verify import _flip_file, _flip_host, _free_hbm, _page_of, _with_raw_pages
from tests.test_resident_share import _check_restored, _load, _resident_split

PAGE = 2 << 20
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "cpp", "hostsim")
gpu = pytest.mark.gpu
HOSTSIM = os.environ.get("FMA_HOSTSIM") == "1"


def _L():
    from fma_b200 import _lib as L

    return L


def _hostsim():
    """The host-simulated engine's fault injection (the library fma_b200 loaded)."""
    if not HOSTSIM:
        pytest.skip("fault injection needs the host-simulated engine")
    return C.CDLL(os.environ["FMA_B200_LIB"])


TIERS = ["host", "file_buffered", "file_direct"]


def _sleep(engine, tier, tmp_path, monkeypatch):
    L = _L()
    path = str(tmp_path / "p.fmaimg")
    if tier.startswith("file"):
        monkeypatch.setenv("FMA_FILE_BUFFERED", "1" if tier == "file_buffered" else "0")
        engine.set_option("load_chunk_bytes", 4 << 20)     # several windows
        engine.set_option("load_slots", 3)
        engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE if tier.startswith("file") else L.FMA_TIER_HOST, flags=L.FMA_FLAG_VERIFY)
    return path


def _image_order(engine, ref):
    return sorted(ref, key=lambda i: engine.segment(i).packed_offset)


def _stored(engine, order):
    """stored bytes of each segment of `order`, from the store's page table"""
    off, nb = engine.image_pages()
    out = []
    for i in order:
        s = engine.segment(i)
        out.append(sum(nb[p] for p in range(s.packed_offset // PAGE, (s.packed_offset + s.bytes) // PAGE)))
    return out


def _split_skipping_a_segment(stored):
    """the smallest 2 MiB budget whose split leaves out a segment behind one it keeps"""
    for budget in range(PAGE, sum(stored), PAGE):
        keep = _resident_split(stored, budget)
        if any(not keep[k] and any(keep[:k]) for k in range(len(keep))):
            return budget
    raise AssertionError(f"no budget skips a segment of {stored}")


def _rows(engine, op):
    rows = engine.timeline()
    assert rows and all(r["op"] == op for r in rows), rows
    return rows


def _kind_bytes(rows, kind):
    return sum(r["bytes"] for r in rows if r["kind"] == kind)


def _prefetch(engine, nbytes):
    engine.prefetch_image(nbytes)
    return engine.stats()["prefetched_bytes"]


BUDGETS = ["zero", "mid", "exact", "more"]


@gpu
@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("tier", TIERS)
@pytest.mark.parametrize("pack", [0, 1])
def test_prefetch_round_trip_matches_oracle(engine, oracle, tmp_path, monkeypatch, pack, tier, budget):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    if pack:
        _with_raw_pages(engine, ref)
    engine.set_option("pack", pack)
    engine.set_option("chunk_bytes", 8 << 20)               # several ring slots and several restore pieces
    _sleep(engine, tier, tmp_path, monkeypatch)
    order = _image_order(engine, ref)
    stored = _stored(engine, order)
    S = engine.stats()["image_store_bytes"]
    assert sum(stored) == S
    if pack:
        assert S < sum(ref[i].size for i in order) and PAGE in engine.image_pages()[1]   # coded pages and raw ones
    cap = {"zero": 0, "mid": _split_skipping_a_segment(stored), "exact": -(-S // PAGE) * PAGE, "more": S + (64 << 20)}[budget]
    keep = _resident_split(stored, cap)
    want = sum(s for s, k in zip(stored, keep) if k)
    kept_plain = sum(ref[i].size for i, k in zip(order, keep) if k)
    assert (want == S) == (budget in ("exact", "more")) and (want == 0) == (budget == "zero")
    assert _prefetch(engine, cap + (PAGE - 1)) == want           # rounded down to 2 MiB
    st = engine.stats()
    assert st["resident_bytes"] == 0 and st["image_store_bytes"] == S and engine.is_sleeping()
    assert all(s.tier == st["tier"] for s in engine.segments() if s.has_backup)   # the records still name the tier's store
    rows = _rows(engine, "prefetch")
    assert [r for r in rows if r["kind"] == "total"][0]["bytes"] == want
    assert ("file_io" in {r["kind"] for r in rows}) == (tier != "host" and want > 0)
    if tier != "host" and want:
        assert _kind_bytes(rows, "file_io") == want
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    st = engine.stats()
    assert st["prefetched_bytes"] == 0 and st["wake_bytes_restored"] == sum(ref[i].size for i in order)
    rows = _rows(engine, "wake")
    kinds = {r["kind"] for r in rows}
    assert ("pf_restore" in kinds) == (want > 0) and ("pf_free" in kinds) == (want > 0) and "res_restore" not in kinds
    if tier == "host":                                       # the link moves only what was not prefetched
        assert _kind_bytes(rows, "enqueue") == sum(ref[i].size for i in order) - kept_plain
    else:                                                    # the disk reads only the pages that were not prefetched
        assert _kind_bytes(rows, "file_io") == S - want


@gpu
@pytest.mark.parametrize("tier", ["host", "file_buffered"])
def test_prefetch_takes_hbm_and_gives_it_back_without_writing(engine, oracle, tmp_path, monkeypatch, tier):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    path = _sleep(engine, tier, tmp_path, monkeypatch)
    S = engine.stats()["image_store_bytes"]
    host_before = _host_bytes(engine)
    file_before = open(path, "rb").read() if tier != "host" else None
    free0 = _free_hbm()
    assert _prefetch(engine, S) == S
    free1 = _free_hbm()
    if free0 is not None:
        assert free0 - free1 >= S                            # the buffer, as the driver reports it
    assert _prefetch(engine, 0) == 0
    if free0 is not None:
        assert _free_hbm() >= free0 - (4 << 20)              # and back
    assert _host_bytes(engine) == host_before                # the store is untouched
    if file_before is not None:
        assert open(path, "rb").read() == file_before
    engine.prefetch_image(0)                                 # nothing prefetched: a no-op
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)               # the whole image crosses the link again
    _check_restored(engine, oracle, ptrs, ref)
    rows = _rows(engine, "wake")
    assert "pf_restore" not in {r["kind"] for r in rows}
    if tier != "host":
        assert _kind_bytes(rows, "file_io") == S


def _host_bytes(engine):
    if engine.stats()["tier"] != _L().FMA_TIER_HOST:
        return b""
    base, n = engine.host_store_view()
    return C.string_at(base, n) if n else b""


@gpu
@pytest.mark.parametrize("tier", ["host", "file_direct"])
@pytest.mark.parametrize("pack", [0, 1])
def test_repeated_prefetches_replace_each_other(engine, oracle, tmp_path, monkeypatch, pack, tier):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    _sleep(engine, tier, tmp_path, monkeypatch)
    order = _image_order(engine, ref)
    stored = _stored(engine, order)
    S = sum(stored)
    for cap in (S // 2 // PAGE * PAGE, 8 << 20, S + PAGE):   # large, smaller, then everything
        keep = _resident_split(stored, cap)
        assert _prefetch(engine, cap) == sum(s for s, k in zip(stored, keep) if k)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    assert "enqueue" not in {r["kind"] for r in _rows(engine, "wake")}   # nothing crossed the link
    # prefetch, drop, wake: the whole image moves
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE if tier != "host" else L.FMA_TIER_HOST, flags=L.FMA_FLAG_VERIFY)
    assert _prefetch(engine, S // 2 // PAGE * PAGE) > 0
    assert _prefetch(engine, 0) == 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    rows = _rows(engine, "wake")
    assert "pf_restore" not in {r["kind"] for r in rows}
    assert _kind_bytes(rows, "file_io" if tier != "host" else "enqueue") == (S if tier != "host" else sum(ref[i].size for i in order))


@gpu
@pytest.mark.parametrize("tier", ["host", "file_buffered"])
def test_tag_selective_wake_keeps_the_prefetch_until_its_segments_wake(engine, oracle, tmp_path, monkeypatch, tier):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=True)
    engine.set_option("pack", 1)
    _sleep(engine, tier, tmp_path, monkeypatch)
    n = _prefetch(engine, 24 << 20)
    assert n > 0
    engine.wake(["kv_cache"])                                # nothing prefetched wakes: the buffer stays
    assert engine.stats()["prefetched_bytes"] == n and engine.is_sleeping()
    assert engine.verify_image() == []
    engine.wake(["weights"], flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    assert engine.stats()["prefetched_bytes"] == 0
    assert "pf_restore" in {r["kind"] for r in _rows(engine, "wake")}


@gpu
def test_keep_backup_wake_releases_the_prefetch(engine, oracle, tmp_path, monkeypatch):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    _sleep(engine, "host", tmp_path, monkeypatch)
    assert _prefetch(engine, 16 << 20) > 0
    engine.wake(None, flags=L.FMA_FLAG_VERIFY | L.FMA_FLAG_KEEP_BACKUP)
    _check_restored(engine, oracle, ptrs, ref)
    assert engine.stats()["prefetched_bytes"] == 0           # the host store is the backup
    assert all(s.has_backup and s.tier == L.FMA_TIER_HOST for i, s in enumerate(engine.segments()) if i in ref)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_clean_incremental_sleep_after_a_prefetched_wake_copies_nothing(engine, oracle, tmp_path, monkeypatch, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.set_option("incremental", 1)
    path = _sleep(engine, "file_buffered", tmp_path, monkeypatch)
    before = open(path, "rb").read()
    assert _prefetch(engine, 1 << 40) == engine.stats()["image_store_bytes"]
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    assert engine.stats()["sleep_bytes_copied"] == 0
    assert open(path, "rb").read() == before
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_moves_between_host_and_file_keep_the_prefetch_and_a_move_to_local_frees_it(engine, oracle, tmp_path, pack):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    engine.set_option("pack", pack)
    engine.set_option("load_chunk_bytes", 4 << 20)
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    S = engine.stats()["image_store_bytes"]
    n = _prefetch(engine, S // 2 // PAGE * PAGE)
    assert 0 < n < S
    engine.file_store(str(tmp_path / "m.fmaimg"))
    engine.move_image(L.FMA_TIER_FILE)
    engine.host_release()
    assert engine.stats()["prefetched_bytes"] == n
    engine.move_image(L.FMA_TIER_HOST)
    assert engine.stats()["prefetched_bytes"] == n
    engine.move_image(L.FMA_TIER_FILE)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    assert _kind_bytes(_rows(engine, "wake"), "file_io") == S - n
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    assert _prefetch(engine, 8 << 20) > 0
    engine.move_image(L.FMA_TIER_LOCAL)                      # the whole image in HBM now
    assert engine.stats()["prefetched_bytes"] == 0
    with pytest.raises(L.FmaError) as ei:
        engine.prefetch_image(8 << 20)
    assert ei.value.code == L.FMA_EINVAL
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_a_prefetched_segment_freed_while_asleep(engine, oracle, tmp_path, monkeypatch):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    _sleep(engine, "file_buffered", tmp_path, monkeypatch)
    order = _image_order(engine, ref)
    stored = _stored(engine, order)
    keep = _resident_split(stored, 24 << 20)
    assert _prefetch(engine, 24 << 20) == sum(s for s, k in zip(stored, keep) if k)
    gone = [i for i, k in zip(order, keep) if k][0]
    engine.free(ptrs[gone])
    assert engine.verify_image() == []
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    assert not engine.is_sleeping() and engine.stats()["prefetched_bytes"] == 0
    got = {s.va: d for s, d in zip(engine.segments(), engine.digest_all(["weights"]))}
    for i in ref:
        if i != gone:
            assert got[ptrs[i]] == oracle.digest(ref[i]), i


@gpu
@pytest.mark.parametrize("tier", ["host", "file_buffered"])
def test_destroy_while_prefetched_leaves_nothing(built, oracle, tmp_path, monkeypatch, tier):
    import fma_b200

    free0 = _free_hbm()
    eng = fma_b200.Engine(0)
    table, ptrs, ref = _load(eng, oracle, bf16=True)
    eng.set_option("pack", 1)
    _sleep(eng, tier, tmp_path, monkeypatch)
    assert _prefetch(eng, 1 << 40) > 0
    eng.close()
    if HOSTSIM:
        lib = _hostsim()
        for f in ("hostsim_live_mapped_bytes", "hostsim_live_handles", "hostsim_live_reservations"):
            getattr(lib, f).restype = C.c_ulonglong
            assert getattr(lib, f)() == 0, f
    else:
        assert _free_hbm() >= free0 - (64 << 20)             # (the process's own CUDA context aside)


_LOAD_CHILD = r"""
import json, sys
sys.path.insert(0, {root!r})
import fma_b200
from fma_b200 import workloads as W, _lib as L
eng = fma_b200.Engine(0)
for s in W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2):
    eng.alloc(s.bytes, s.tag)
eng.image_load(sys.argv[1], ["weights"])
eng.wake(None, flags=L.FMA_FLAG_VERIFY)
print(json.dumps(eng.digest_all(["weights"])), flush=True)
"""


@gpu
@pytest.mark.parametrize("pack", [0, 1])
def test_a_prefetched_image_is_handed_over_whole(engine, oracle, tmp_path, monkeypatch, pack):
    """image_save of a prefetched host-tier image, and the file of a prefetched file-tier image, open in a fresh process"""
    L = _L()
    monkeypatch.setenv("FMA_HOST_STORE_SHM", "1")
    table, ptrs, ref = _load(engine, oracle, bf16=bool(pack))
    widx = sorted(ref)
    engine.set_option("pack", pack)

    def child(src, path):
        f = tmp_path / "child.py"
        f.write_text(src.format(root=ROOT))
        r = subprocess.run([sys.executable, str(f), path], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        got = json.loads(r.stdout.strip().splitlines()[-1])
        assert [got[i] for i in widx] == [oracle.digest(ref[i]) for i in widx]

    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    assert _prefetch(engine, 16 << 20) > 0
    saved = str(tmp_path / "saved.fmaimg")
    engine.image_save(saved)
    child(_LOAD_CHILD, saved)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    path = str(tmp_path / "f.fmaimg")
    engine.file_store(path)
    engine.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
    assert _prefetch(engine, 16 << 20) > 0
    child(_ADOPT_CHILD, path)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("where", ["host", "file"])
@pytest.mark.parametrize("page", ["plain", "coded", "raw"])
def test_verify_checks_the_store_and_the_prefetched_copy(engine, oracle, tmp_path, monkeypatch, page, where):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=page != "plain")
    if page == "raw":
        _with_raw_pages(engine, ref)
    engine.set_option("pack", 0 if page == "plain" else 1)
    path = _sleep(engine, "host" if where == "host" else "file_buffered", tmp_path, monkeypatch)
    order = _image_order(engine, ref)
    hit = None
    for seg in order[::-1]:                                  # a prefetched (tail) segment with such a page
        pg = _page_of(engine, seg, None if page == "plain" else page == "coded")
        if pg:
            hit = seg, pg
            break
    if hit is None:
        pytest.skip(f"no {page} page in the image")
    seg, (off, nb) = hit
    at = off + nb // 3
    flip = (lambda: _flip_host(engine, at)) if where == "host" else (lambda: _flip_file(path, at))
    S = engine.stats()["image_store_bytes"]
    # damaged before the prefetch: the copy carries it; reported once while prefetched, and after the drop
    flip()
    assert _prefetch(engine, S + PAGE) == S
    assert engine.verify_image() == [seg]
    engine.prefetch_image(0)
    assert engine.verify_image() == [seg]
    # the store repaired after the prefetch: only the copy in HBM is bad, and the wake restores from it
    assert _prefetch(engine, S + PAGE) == S
    flip()
    assert engine.verify_image() == [seg]
    with pytest.raises(L.FmaError) as ei:
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    assert ei.value.code == L.FMA_EINTEGRITY and f"segment {seg}" in ei.value.message


@gpu
def test_refusals_leave_the_engine_unchanged(engine, oracle, tmp_path):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)

    def snapshot():
        st = engine.stats()
        keep = {k: st[k] for k in ("tier", "prefetched_bytes", "resident_bytes", "image_store_bytes", "parked_bytes", "hbm_mapped_bytes")}
        rows = engine.timeline()
        return keep, [(s.mapped, s.has_backup, s.tier, s.packed_offset) for s in engine.segments()], rows[0]["op"] if rows else None

    def refused(code, text):
        before = snapshot()
        with pytest.raises(L.FmaError) as ei:
            engine.prefetch_image(8 << 20)
        assert ei.value.code == code and text in ei.value.message, ei.value.message
        assert snapshot() == before
        engine.prefetch_image(0)                             # the hand-back always succeeds
        assert snapshot() == before

    refused(L.FMA_ESTATE, "no image is asleep")              # awake
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    engine.wake(None, flags=L.FMA_FLAG_KEEP_BACKUP)          # mapped segments keep a backup
    refused(L.FMA_ESTATE, "KEEP_BACKUP")
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    engine.wake(None)
    engine.set_option("resident_bytes", 8 << 20)             # a resident share from the sleep
    engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    assert engine.stats()["resident_bytes"] > 0
    refused(L.FMA_ESTATE, "set it to 0 and sleep again")
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    engine.set_option("resident_bytes", 0)
    engine.sleep(["weights"], tier=L.FMA_TIER_LOCAL, flags=L.FMA_FLAG_VERIFY)
    refused(L.FMA_EINVAL, "in HBM already")                  # parked in this GPU's HBM
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_a_truncated_file_fails_the_prefetch_and_leaves_no_buffer(engine, oracle, tmp_path, monkeypatch):
    L = _L()
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    path = _sleep(engine, "file_buffered", tmp_path, monkeypatch)
    keep = str(tmp_path / "keep")
    shutil.copyfile(path, keep)
    S = engine.stats()["image_store_bytes"]
    os.truncate(path, S - (3 << 20))                         # the tail, which a prefetch reads, is gone
    free0 = _free_hbm()
    with pytest.raises(L.FmaError) as ei:
        engine.prefetch_image(S)
    assert ei.value.code == L.FMA_EIO
    st = engine.stats()
    assert st["prefetched_bytes"] == 0 and st["tier"] == L.FMA_TIER_FILE and engine.is_sleeping()
    if free0 is not None:
        assert _free_hbm() >= free0 - (4 << 20)
    shutil.copyfile(keep, path)
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
def test_no_hbm_for_the_buffer_is_enomem_with_nothing_left(engine, oracle, tmp_path, monkeypatch):
    L = _L()
    sim = _hostsim()
    sim.hostsim_live_handles.restype = C.c_ulonglong
    table, ptrs, ref = _load(engine, oracle, bf16=False)
    _sleep(engine, "host", tmp_path, monkeypatch)
    handles = sim.hostsim_live_handles()
    sim.hostsim_fail_create_after(C.c_long(0))
    try:
        with pytest.raises(L.FmaError) as ei:
            engine.prefetch_image(16 << 20)
    finally:
        sim.hostsim_fail_create_after(C.c_long(-1))
    assert ei.value.code == L.FMA_ENOMEM
    assert engine.stats()["prefetched_bytes"] == 0 and sim.hostsim_live_handles() == handles
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)


@gpu
@pytest.mark.parametrize("tier", ["host", "file_buffered"])
def test_a_failed_wake_keeps_the_prefetch_for_its_retry(engine, oracle, tmp_path, monkeypatch, tier):
    L = _L()
    sim = _hostsim()
    table, ptrs, ref = _load(engine, oracle, bf16=True)
    engine.set_option("pack", 1)
    _sleep(engine, tier, tmp_path, monkeypatch)
    n = _prefetch(engine, 24 << 20)
    assert n > 0
    sim.hostsim_fail_call_after(b"cuMemMap", C.c_long(1))    # the second mapping of the wake fails
    try:
        with pytest.raises(L.FmaError):
            engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    finally:
        sim.hostsim_fail_call_after(b"cuMemMap", C.c_long(-1))
    assert engine.is_sleeping() and engine.stats()["prefetched_bytes"] == n
    assert all(not s.mapped for i, s in enumerate(engine.segments()) if i in ref)   # rolled back
    engine.wake(None, flags=L.FMA_FLAG_VERIFY)
    _check_restored(engine, oracle, ptrs, ref)
    assert "pf_restore" in {r["kind"] for r in _rows(engine, "wake")}


def test_prefetch_routes():
    """prefetch_route in csrc/fma_layout.h against its restatement (tests/cpp/prefetch_route_test.cpp)."""
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"prefetch_route_test_{os.getpid()}")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "prefetch_route_test.cpp"), "-o", exe])
    try:
        assert "prefetch routes ok" in subprocess.check_output([exe], text=True)
    finally:
        os.unlink(exe)


_SHIM_CHILD = r"""
import os, sys, types
sys.path.insert(0, {root!r})
sys.modules["torch"] = types.SimpleNamespace(cuda=types.SimpleNamespace(empty_cache=lambda: None))
import fma_b200
from fma_b200.cumem import CuMemAllocator
eng = fma_b200.Engine(0)
for i, mib in enumerate((6, 2, 8, 4)):
    eng.alloc(mib << 20, "kv_cache" if i == 2 else "weights")
for i in (0, 1, 3):
    eng.fill(i, 77, i << 24)
before = eng.digest_all(["weights"])
a = CuMemAllocator(engine=eng)
assert a.prefetch_image(64) == 0                    # awake: nothing to do
a.sleep(("weights",))
n = a.prefetch_image(5)                              # 4 MiB: the last weight segment fits, the 2 MiB one before it does not
assert n == eng.stats()["prefetched_bytes"] == 4 << 20, n
assert a.prefetch_image(64) == 12 << 20
a.wake_up(None)
assert eng.digest_all(["weights"]) == before and eng.stats()["prefetched_bytes"] == 0
print("shim prefetch ok", eng.stats()["tier"], flush=True)
"""


@pytest.mark.parametrize("tier", ["host", "file"])
def test_shim_prefetch_image(hostsim_lib, tmp_path, tier):
    L = _L()
    child = tmp_path / "child.py"
    child.write_text(_SHIM_CHILD.format(root=ROOT))
    d = tmp_path / "images"
    d.mkdir()
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="1", FMA_TIER=tier, FMA_INSTANCE_ID="Ipf", RANK="0",
               FMA_FILE_DIR=str(d))
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_NODE_AGENT_SOCK", "FMA_REMOTE_PATHS", "LOCAL_RANK", "FMA_PREPIN"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, str(child)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert f"shim prefetch ok {L.FMA_TIER_FILE if tier == 'file' else L.FMA_TIER_HOST}" in r.stdout, r.stdout


# ---- the host-simulated engine ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_prefetch") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS,
                           os.path.join(SIM, "hostsim_verify_kernels.cpp"), "-o", out, "-lpthread"])
    return out


def test_image_prefetch_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout and "SKIPPED" not in r.stdout, tail


def test_image_prefetch_scenario_under_sanitizers(tmp_path):
    """tests/cpp/hostsim/prefetch_sanitizer_test.cpp under ThreadSanitizer and under ASan+UBSan+LeakSan, side by side."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_engine_hostsim import INC, SRCS

    def one(san, flags):
        exe = str(tmp_path / f"prefetch_{san}")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", *flags, *INC, *SRCS, os.path.join(SIM, "prefetch_sanitizer_test.cpp"), "-o", exe,
                               "-lpthread"])
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", TSAN_OPTIONS="halt_on_error=1", HOSTSIM_DEVICES="1")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED"):
            env.pop(key, None)
        r = subprocess.run([exe, str(tmp_path / f"{san}.fmaimg")], env=env, capture_output=True, text=True, timeout=900)
        return san, r.returncode, r.stdout + r.stderr

    with ThreadPoolExecutor(2) as pool:
        results = list(pool.map(lambda a: one(*a), [("tsan", ["-fsanitize=thread"]), ("asan", ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"])]))
    for san, rc, out in results:
        assert rc == 0 and "prefetch sanitizer scenario ok" in out, (san, out[-3000:])
        assert "WARNING: ThreadSanitizer" not in out and "ERROR: AddressSanitizer" not in out and "runtime error:" not in out, (san, out[-3000:])
