"""K1/K2 pipeline shapes, grid-stride loops and memory kinds on the device (run with -m gpu on an H100).

The kernel-level binaries (tests/cpp/cuda_emu/, built by build()) compare K0-K5 with the oracle at every legal TMA shape,
across the grid caps and in mapped pinned host memory.  The engine-level tests below check the same through the C-ABI:
the shape options, the zero-copy packed wake, the incremental sleep's trust in K3, and the refusal of a shape that cannot
run BEFORE a sleep or wake touches anything.  Those do not depend on real kernels, so tests/test_engine_hostsim.py also runs
them against the host-simulated engine; the binary and raw-op tests skip there."""
import os
import re
import subprocess

import numpy as np
import pytest

from tests.pagegen import stamp

pytestmark = pytest.mark.gpu

PAGE = 2 << 20
HOSTSIM = os.environ.get("FMA_HOSTSIM") == "1"
EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "cuda_emu")


def _L():
    from fma_b200 import _lib as L

    return L


def _run_binary(name, env=None):
    if HOSTSIM:
        pytest.skip("a device binary: nothing to run on the host simulation")
    exe = os.path.join(EMU, name)
    if not os.path.exists(exe):
        pytest.skip(f"not built (make -C tests/cpp/cuda_emu {name})")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})))
    print(r.stdout)
    return r


def test_kernels_binary_runs_every_legal_tma_shape_on_the_device():
    """K0-K3 at every legal TMA shape x 2 CTA counts, gather and scatter, 1 / 5 / 67 pages, LDG, clamped and refused shapes,
    mapped pinned host memory, and K0/K3 on both sides of the grid cap (kernels_emu_test.cpp)."""
    r = _run_binary("kernels_gpu_test")
    assert r.returncode == 0 and "kernels (GPU) ok" in r.stdout, (r.stdout + r.stderr)[-3000:]
    assert "140 of 140 legal shapes x 2 CTA counts = 280 shape runs" in r.stdout and "20 of them at 67 pages" in r.stdout, r.stdout
    assert "page counts { 1 16 17 200 }" in r.stdout, r.stdout


def test_pack_kernels_binary_strides_every_cta_over_raw_and_coded_items():
    """pack_kernels_emu_test.cpp with the grid capped at one CTA per SM: the alternating RAW / coded launch has at least two
    work items per CTA, so K4p / K4 / K5 reuse their shared state across items of both kinds on the device."""
    r = _run_binary("pack_kernels_gpu_test", {"FMA_PACK_CTAS_PER_SM": "1"})
    assert r.returncode == 0 and "pack kernels (GPU) ok" in r.stdout, (r.stdout + r.stderr)[-3000:]
    m = re.search(r"items/grid = ([0-9.]+)", r.stdout)
    assert m and float(m.group(1)) >= 2.0, r.stdout


def _legal_shapes():
    return [(t, s, p) for t in (1, 2, 4, 8, 16, 32, 64) for p in range(1, 5) for s in range(2, 9) if p * s * (t << 10) + 128 <= 227 << 10]


def _set_shape(engine, tile_bytes, stages, pipes, ctas_per_sm=1):
    engine.set_option("tma_tile_bytes", tile_bytes)
    engine.set_option("tma_stages", stages)
    engine.set_option("tma_pipes", pipes)
    engine.set_option("tma_ctas_per_sm", ctas_per_sm)


def test_tma_shape_sweep_through_the_c_abi(engine, oracle):
    """A seeded part of the shape sweep through set_option + op_page_copy on VMM segments: the engine's own option path."""
    if HOSTSIM:
        pytest.skip("raw kernel operation: the host simulation has no kernels")
    L = _L()
    shapes = _legal_shapes()
    assert len(shapes) == 140
    rng = np.random.default_rng(17)
    pick = [shapes[i] for i in sorted(rng.choice(len(shapes), 16, replace=False))] + [(1, 4096, 5), (4, 0, 0)]   # last two: clamped
    n = 7
    src = oracle.fill(n * PAGE, 5, 0)
    engine.alloc(n * PAGE, "default")
    engine.alloc(n * PAGE, "default")
    engine.write(0, src.tobytes())
    base, out = engine.segment(0).va, engine.segment(1).va
    dst = engine.scratch_alloc(n * PAGE)
    for k, (tile, stages, pipes) in enumerate(pick):
        _set_shape(engine, tile << 10, stages, pipes, 1 + 3 * (k % 2))
        perm = rng.permutation(n).tolist()
        engine.op_page_copy(n, src_pages=[base + p * PAGE for p in perm], dst_base=dst, variant=L.FMA_KERNEL_TMA)
        engine.op_page_copy(n, src_base=dst, dst_base=out, variant=L.FMA_KERNEL_TMA)
        assert engine.read(1, n * PAGE) == oracle.gather([src[p * PAGE:(p + 1) * PAGE] for p in perm]).tobytes(), (tile, stages, pipes)
        engine.op_page_copy(n, src_base=dst, dst_pages=[out + p * PAGE for p in perm], variant=L.FMA_KERNEL_TMA)
        assert engine.read(1, n * PAGE) == src.tobytes(), (tile, stages, pipes)
    _set_shape(engine, 64 << 10, 8, 4)                                  # 2 MiB of shared memory: refused, nothing written
    engine.write(1, b"\x5a" * PAGE)
    with pytest.raises(L.FmaError):
        engine.op_page_copy(1, src_base=base, dst_base=out, variant=L.FMA_KERNEL_TMA)
    assert engine.read(1, PAGE) == b"\x5a" * PAGE
    engine.scratch_free(dst)
    print(f"C-ABI sweep: {len(pick)} TMA shapes")


def _pages_for_packing(oracle):
    """bf16 weights (coded), noise (raw) and a page with exactly 2048 exceptions (coded, at the capacity edge)."""
    rng = np.random.default_rng(23)
    n = 1 << 20
    uni = oracle.bf16_weights(n, 3)
    noise = rng.integers(0, 1 << 16, n, dtype=np.uint16)
    cap = np.full(n, 0x3F80, np.uint16)
    cap[rng.choice(n, 2048, replace=False)] = 0x00D5
    return [p.view(np.uint8) for p in (uni, noise, cap)]


def test_zero_copy_packed_wake_reads_the_pinned_store(engine, oracle, monkeypatch):
    """FMA_NO_RING=1 after a packed STAGED sleep: no staging ring, so K5 decodes the stored pages straight from the pinned host
    store through its device alias (mode DIRECT); tag by tag, then everything; bytes and device addresses unchanged."""
    L = _L()
    uni, noise, cap = _pages_for_packing(oracle)
    blobs = {"weights": stamp(np.concatenate([uni, noise, cap, uni]), 23, 0),      # every page its own (tests/pagegen.py)
             "lora": stamp(np.concatenate([cap, noise, uni]), 23, 4)}
    ptrs, idx = [], {}
    for tag in ("weights", "kv_cache", "lora"):
        ptrs.append(engine.alloc(blobs[tag].size if tag in blobs else 2 * PAGE, tag))
        idx[tag] = len(ptrs) - 1
    for tag, b in blobs.items():
        engine.write(idx[tag], b.tobytes())
    engine.set_option("mode", L.FMA_MODE_STAGED)
    engine.set_option("pack", 1)
    engine.set_option("chunk_bytes", 4 << 20)
    engine.sleep(["weights", "lora"], flags=L.FMA_FLAG_VERIFY)
    st = engine.stats()
    assert st["image_packed"] == 1 and st["mode"] == L.FMA_MODE_STAGED
    off, nb = engine.image_pages()
    assert nb.count(PAGE) == 2 and nb.count(L.FMA_PACKED_PAGE_BYTES) == 5
    monkeypatch.setenv("FMA_NO_RING", "1")
    for tags in (["lora"], None):
        engine.wake(tags, flags=L.FMA_FLAG_VERIFY)
        st = engine.stats()
        assert st["mode"] == L.FMA_MODE_DIRECT and st["wake_bytes_restored"] > 0, st
    assert not engine.is_sleeping() and [s.va for s in engine.segments()] == ptrs
    for tag, b in blobs.items():
        assert engine.read(idx[tag], b.size) == b.tobytes(), tag
    print("zero-copy packed wake: no ring, mode DIRECT, K5 read 7 stored pages from the pinned host store")


def _flip_positions(words):
    """Word positions in a 4-page segment: its ends, both sides of the first page boundary, one word per lane and per vector
    of a K3 thread (thread t of a 32 KiB tile reads words (u * 256 + t) * 2 and +1 for u < 8), and 32 seeded positions."""
    wpp = PAGE // 8
    pos = [0, words - 1, wpp - 1, wpp]
    pos += [wpp + 4096 * 3 + (u * 256 + lane) * 2 + (lane & 1) for lane in range(32) for u in (lane % 8,)]
    pos += np.random.default_rng(29).integers(0, words, 32).tolist()
    return pos


def test_incremental_sleep_sees_one_flipped_bit(engine, oracle):
    """After an incremental clean cycle, one bit flipped anywhere in a weight segment must make the next sleep copy, and the
    wake must return the flipped bytes: K3 is the only thing that decides."""
    L = _L()
    seg_bytes = 4 * PAGE
    engine.alloc(seg_bytes, "weights")
    engine.alloc(seg_bytes, "weights")
    engine.alloc(2 * PAGE, "kv_cache")
    ref = [oracle.fill(seg_bytes, 41, 0).copy(), oracle.fill(seg_bytes, 41, seg_bytes // 8).copy()]
    for i, r in enumerate(ref):
        engine.write(i, r.tobytes())
    engine.set_option("mode", L.FMA_MODE_STAGED)
    engine.set_option("incremental", 1)
    engine.sleep(["weights"]); engine.wake(None)
    engine.sleep(["weights"])
    assert engine.stats()["sleep_bytes_copied"] == 0                   # clean: nothing moved
    engine.wake(None)
    words = ref[0].view(np.uint64)
    for k, w in enumerate(_flip_positions(seg_bytes // 8)):
        words[w] ^= np.uint64(1) << np.uint64(k % 64)
        engine.write(0, words[w:w + 1].tobytes(), offset=w * 8)
        engine.sleep(["weights"])
        assert engine.stats()["sleep_bytes_copied"] > 0, (k, w)
        engine.wake(None)
        assert engine.read(0, seg_bytes) == ref[0].tobytes(), (k, w)
        assert engine.read(1, seg_bytes) == ref[1].tobytes(), (k, w)


FITS = (16 << 10, 3, 2)


@pytest.mark.parametrize("how", ["option", "env", "env_tile"])
@pytest.mark.parametrize("mode", ["staged", "kernel"])
def test_an_unfit_tma_shape_is_refused_before_anything_moves(built, oracle, monkeypatch, how, mode):
    """A shape whose pipeline does not fit shared memory (or whose tile does not divide the page): sleep and wake return
    FMA_EINVAL before anything is unmapped or copied; the engine stays as it was, kv_cache included; with a fitting shape
    the same sleep and wake are bit-exact.  Set through set_option or FMA_TMA_* (which seed the same fields)."""
    import fma_b200

    L = _L()
    if how == "env":
        monkeypatch.setenv("FMA_TMA_TILE_KIB", "64"); monkeypatch.setenv("FMA_TMA_STAGES", "8"); monkeypatch.setenv("FMA_TMA_PIPES", "4")
    elif how == "env_tile":
        monkeypatch.setenv("FMA_TMA_TILE_KIB", "3")
    engine = fma_b200.Engine(0)
    try:
        table = [(3 * PAGE, "weights"), (2 * PAGE, "kv_cache"), (PAGE, "weights")]
        ptrs = [engine.alloc(b, t) for b, t in table]
        data = [oracle.fill(b, 61, 1000 * i).tobytes() for i, (b, _) in enumerate(table)]
        for i, d in enumerate(data):
            engine.write(i, d)
        engine.set_option("mode", L.FMA_MODE_STAGED if mode == "staged" else L.FMA_MODE_KERNEL)

        def unfit():
            if how == "option":
                _set_shape(engine, 64 << 10, 8, 4)

        def fit():
            _set_shape(engine, *FITS)

        def intact(sleeping):
            assert engine.is_sleeping() == sleeping
            segs = engine.segments()
            assert [s.va for s in segs] == ptrs
            if not sleeping:
                assert all(s.mapped for s in segs)
                for i, d in enumerate(data):
                    assert engine.read(i, len(d)) == d, i
            else:
                assert not any(s.mapped for s in segs)

        unfit()
        with pytest.raises(L.FmaError) as ei:
            engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
        assert ei.value.code == L.FMA_EINVAL, ei.value
        intact(False)
        fit()
        engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
        intact(True)
        if how == "option":
            unfit()
        else:
            engine.set_option("tma_tile_bytes", 32 << 10); engine.set_option("tma_stages", 8)      # 512 KiB of shared memory
        with pytest.raises(L.FmaError) as ei:
            engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        assert ei.value.code == L.FMA_EINVAL, ei.value
        intact(True)
        fit()
        engine.wake(["weights"], flags=L.FMA_FLAG_VERIFY)
        engine.wake(None)
        for i, (_, tag) in enumerate(table):
            if tag == "weights":
                assert engine.read(i, len(data[i])) == data[i], i
        # out-of-range stages and pipes are clamped, not refused: 1 KiB x 8 stages x 4 pipes runs
        _set_shape(engine, 1 << 10, 4096, 5)
        engine.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
        engine.wake(None, flags=L.FMA_FLAG_VERIFY)
        for i, (_, tag) in enumerate(table):
            if tag == "weights":
                assert engine.read(i, len(data[i])) == data[i], i
    finally:
        engine.close()


def test_a_swap_with_an_unfit_shape_on_either_side_starts_neither_half(built, oracle):
    """fma_swap sleeps one engine while it wakes another: an unfit shape on the waking side must not leave the other engine
    asleep with nothing woken in its place."""
    import fma_b200

    L = _L()
    out_e, in_e = fma_b200.Engine(0), fma_b200.Engine(0)
    try:
        data = {}
        for k, e in enumerate((out_e, in_e)):
            e.alloc(2 * PAGE, "weights")
            data[k] = oracle.fill(2 * PAGE, 71 + k, 0).tobytes()
            e.write(0, data[k])
            e.set_option("mode", L.FMA_MODE_STAGED)
        in_e.sleep(["weights"])
        _set_shape(in_e, 64 << 10, 8, 4)
        with pytest.raises(L.FmaError) as ei:
            out_e.swap_out_for(in_e, ["weights"])
        assert ei.value.code == L.FMA_EINVAL, ei.value
        assert not out_e.is_sleeping() and in_e.is_sleeping() and out_e.read(0, 2 * PAGE) == data[0]
        _set_shape(in_e, *FITS)
        out_e.swap_out_for(in_e, ["weights"])
        assert out_e.is_sleeping() and not in_e.is_sleeping() and in_e.read(0, 2 * PAGE) == data[1]
    finally:
        out_e.close()
        in_e.close()
