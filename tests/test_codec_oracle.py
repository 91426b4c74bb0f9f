"""The "FMP4" page code of packed host images: the oracle's value-by-value restatement (oracle/fma_oracle.c) against
the format's algebra.  The engine's kernels are compared with this oracle in tests/test_gpu_parity.py (on the CUDA host
simulation here, on an H100 with -m gpu)."""
import numpy as np
import pytest

PAGE = 2 << 20
N = 1 << 20
PACKED = (3 << 19) + (16 << 10)
EMAX_OFF, EXC_OFF, HDR_OFF = 3 << 19, (3 << 19) + 4096, (3 << 19) + 4096 + 8192


def _page(values: np.ndarray) -> np.ndarray:
    return values.astype(np.uint16).view(np.uint8)


def test_constants_match_the_kernel_header():
    import re, os
    src = open(os.path.join(os.path.dirname(__file__), "..", "llm-d-fast-model-actuation_b200", "csrc", "fma_codec.h")).read()
    assert "kExcCap = 2048" in src and "kTileValues = 256" in src and "kMaxDelta = 13" in src
    assert re.search(r"kMagic = 0x34504D46u", src)
    kern = open(os.path.join(os.path.dirname(__file__), "..", "llm-d-fast-model-actuation_b200", "csrc", "fma_kernels.h")).read()
    assert "((3u << 19) + (16u << 10))" in kern


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_round_trip_is_exact_for_weights_and_for_noise(oracle, seed):
    rng = np.random.default_rng(seed)
    for page in (oracle.bf16_weights(N, seed).view(np.uint8),
                 _page(rng.normal(0, 0.05, N).astype(np.float32).view(np.uint32) >> 16),
                 rng.integers(0, 256, PAGE, dtype=np.uint8)):
        stored = oracle.pack_page(page)
        assert stored.size in (PACKED, PAGE)
        assert np.array_equal(oracle.unpack_page(stored), page)


def test_known_answer_small_cases(oracle):
    # all 1.0 (0x3F80): emax 127 everywhere, all codes 0, sm bytes 0x00
    st = oracle.pack_page(_page(np.full(N, 0x3F80)))
    assert st.size == PACKED and not st[:EMAX_OFF].any() and (st[EMAX_OFF:EXC_OFF] == 127).all()
    assert st[HDR_OFF:HDR_OFF + 8].view(np.uint32).tolist() == [0x34504D46, 0]
    # one tile: value 0 = -2.0 (0xC000, e=128), value 1 = 0.5 (0x3F00, e=126), value 2 = +0, value 3 = 2^-20 (e=107) -> exception
    v = np.full(N, 0x3F80)
    v[:4] = [0xC000, 0x3F00, 0x0000, (107 << 7) | 0x15]
    st = oracle.pack_page(_page(v))
    assert st[EMAX_OFF] == 128 and st[0] == 0x80 and st[1] == 0x00 and st[3] == 0x15
    nib = st[1 << 20:(1 << 20) + 2]
    assert (nib[0] & 0xF, nib[0] >> 4, nib[1] & 0xF, nib[1] >> 4) == (0, 2, 14, 15)
    assert st[(1 << 20) + 2] == 0x11                                  # 1.0 under emax 128 -> code 1, twice
    assert st[HDR_OFF + 4:HDR_OFF + 8].view(np.uint32)[0] == 1
    assert st[EXC_OFF:EXC_OFF + 4].view(np.uint32)[0] == 3 | (107 << 20)
    assert np.array_equal(oracle.unpack_page(st), _page(v))


def test_exception_capacity_edge_and_raw_fallback(oracle):
    rng = np.random.default_rng(0)
    v = np.full(N, 0x3F80)
    idx = rng.choice(N, 2049, replace=False)
    v[idx[:2048]] = 0x0080                                            # e = 1, 126 binades below: exception
    st = oracle.pack_page(_page(v))
    assert st.size == PACKED and st[HDR_OFF + 4:HDR_OFF + 8].view(np.uint32)[0] == 2048
    assert np.array_equal(oracle.unpack_page(st), _page(v))
    v[idx[2048]] = 0x0080
    st = oracle.pack_page(_page(v))
    assert st.size == PAGE and np.array_equal(st, _page(v))           # one too many: verbatim


def test_malformed_stored_pages_are_rejected(oracle):
    st = oracle.pack_page(oracle.bf16_weights(N, 9).view(np.uint8))
    bad = st.copy(); bad[HDR_OFF] ^= 1
    with pytest.raises(ValueError):
        oracle.unpack_page(bad)
    bad = st.copy(); bad[HDR_OFF + 4:HDR_OFF + 8] = np.array([4096], np.uint32).view(np.uint8)
    with pytest.raises(ValueError):
        oracle.unpack_page(bad)
    with pytest.raises(ValueError):
        oracle.unpack_page(st[:-16])


def test_compression_ratio_on_dummy_and_gaussian_weights(oracle):
    """What the packed image buys: 0.758 of the bytes for bf16 weights (vLLM dummy weights and N(0, sigma))."""
    for page in (oracle.bf16_weights(N, 4).view(np.uint8),
                 _page(np.random.default_rng(4).normal(0, 0.02, N).astype(np.float32).view(np.uint32) >> 16)):
        assert oracle.pack_page(page).size == PACKED
    assert abs(PACKED / PAGE - 0.7578125) < 1e-12


def test_format_is_pinned_by_the_golden_fixture(oracle):
    """tests/golden/fmp4_pages.json (tests/golden/make_fmp4_golden.py): SHA-256 of the stored form of seeded pages.  The oracle
    zero-fills what the format leaves unspecified and emits exceptions in index order, so its stored pages are canonical."""
    import hashlib
    import importlib.util
    import json
    import os

    here = os.path.dirname(__file__)
    spec = importlib.util.spec_from_file_location("make_fmp4_golden", os.path.join(here, "golden", "make_fmp4_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    want = {p["name"]: p for p in json.load(open(os.path.join(here, "golden", "fmp4_pages.json")))["pages"]}
    seen = 0
    for name, page in gen.pages():
        w = want[name]
        assert hashlib.sha256(page.tobytes()).hexdigest() == w["input_sha256"], f"{name}: the generator's input changed"
        stored = oracle.pack_page(page)
        assert stored.size == w["stored_bytes"] and hashlib.sha256(stored.tobytes()).hexdigest() == w["stored_sha256"], name
        seen += 1
    assert seen == len(want) == 7


def _numpy_pack(page: np.ndarray) -> np.ndarray:
    """A third, vectorised restatement of the format (numpy), written from the spec in csrc/fma_codec.h — not from the C oracle."""
    v = page.view(np.uint16).astype(np.uint32)
    e = (v >> 7) & 0xFF
    emax = e.reshape(-1, 256).max(axis=1)
    d = np.repeat(emax, 256) - e
    code = np.where(d <= 13, d, np.where(e == 0, 14, 15)).astype(np.uint8)
    exc = np.flatnonzero(code == 15)
    if exc.size > 2048:
        return page.copy()
    out = np.zeros(PACKED, np.uint8)
    out[:N] = (((v >> 15) << 7) | (v & 0x7F)).astype(np.uint8)
    out[N:N + N // 2] = code[0::2] | (code[1::2] << 4)
    out[EMAX_OFF:EMAX_OFF + 4096] = emax.astype(np.uint8)
    out[EXC_OFF:EXC_OFF + 4 * exc.size] = (exc.astype(np.uint32) | (e[exc] << 20)).astype("<u4").view(np.uint8)
    out[HDR_OFF:HDR_OFF + 8] = np.array([0x34504D46, exc.size], "<u4").view(np.uint8)
    return out


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_oracle_agrees_with_an_independent_numpy_restatement(oracle, seed):
    rng = np.random.default_rng(seed)
    gau = _page(rng.normal(0, 0.03, N).astype(np.float32).view(np.uint32) >> 16)
    sparse = gau.copy().view(np.uint16); sparse[rng.random(N) < 0.2] = 0
    heavy = _page((rng.standard_t(3, N) * 0.01).astype(np.float32).view(np.uint32) >> 16)
    for page in (gau, sparse.view(np.uint8), heavy, oracle.bf16_weights(N, seed).view(np.uint8), rng.integers(0, 256, PAGE, dtype=np.uint8)):
        assert np.array_equal(oracle.pack_page(page), _numpy_pack(page))
