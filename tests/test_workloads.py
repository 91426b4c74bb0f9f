"""Allocation tables reproduce the per-rank shapes of SURVEY.md §8a / BASELINE.md §2 (known answers)."""
import fma_b200  # noqa: F401
from fma_b200 import workloads as W

MiB, GiB = 1 << 20, 1 << 30


def _large(table):
    return [s for s in table if s.note not in ("small-pool", "20MiB-pool")]


def test_llama3_8b_table():
    t = W.allocation_table("llama-3-8b")
    assert len(t) == 132 and len(_large(t)) == 130                     # 130 large tensors + the small-pool segment + the rotary cache's 20 MiB segment: what a LIVE vLLM allocates
    sizes = sorted({s.bytes // MiB for s in _large(t)})
    assert sizes == [32, 48, 112, 224, 1002]                            # o, qkv, down, gate_up, embed/lm_head
    assert W.weight_bytes(t) == 15338 * MiB == 16083058688              # 14.958 GiB of tensors + the small-pool segment + 20 MiB for the rotary cache: vLLM's own "14.98 GiB is backed up"
    assert t[0].bytes == 1002 * MiB and t[-1].bytes == 1002 * MiB       # embed first, lm_head last
    assert [s.bytes // MiB for s in t[1:7]] == [48, 32, 2, 20, 224, 112]   # qkv, o, rotary (inv_freq -> small pool, cos_sin_cache -> 20 MiB pool), gate_up, down: the live order


def test_llama3_70b_tp8_rank_table():
    t = W.allocation_table("llama-3-70b-tp8")
    assert len(_large(t)) == 321 and len(t) == 324                     # one 16 MiB o_proj best-fits into the tail of the rotary cache's 20 MiB segment
    assert sorted({s.bytes // MiB for s in _large(t)}) == [16, 20, 56, 112, 252]   # 250.5 MiB embed -> 252 MiB segment
    assert abs(W.weight_bytes(t) / GiB - 16.44) < 0.01
    assert all(s.bytes % (2 * MiB) == 0 for s in t)


def test_mistral_and_opt():
    assert abs(W.weight_bytes(W.allocation_table("mistral-7b")) / GiB - 13.52) < 0.01
    opt = W.allocation_table("opt-125m")
    assert abs(sum(n for _, n in W.model_tensors("opt-125m")) / MiB - 238.9) < 0.5   # BASELINE.md: 238.9 MiB fp16
    assert W.weight_bytes(opt) >= 238 * MiB


def test_kv_cache_is_tagged_and_never_counted_as_weights():
    t = W.allocation_table("llama-3-8b", kv_cache_bytes=32 * GiB)
    kv = [s for s in t if s.tag == "kv_cache"]
    assert len(kv) == 32 and sum(s.bytes for s in kv) == 32 * GiB
    assert W.weight_bytes(t) == 15338 * MiB
    assert [s.tag for s in t].index("kv_cache") == 132                  # allocated after the weights


def test_segment_size_classes():
    segs = W.simulate_segments([("a", 8 << 10)] * 65 + [("m", 3 * MiB)] * 7 + [("big", 10 * MiB + 1)], "weights")
    assert [s.bytes // MiB for s in segs] == [2, 20, 20]           # "big" best-fits into the 17 MiB tail of the 2nd 20 MiB segment
    segs = W.simulate_segments([("m", 3 * MiB)] * 6 + [("big", 18 * MiB + 1)], "weights")
    assert [s.bytes // MiB for s in segs] == [20, 20]              # >= 10 MiB with no fitting tail: own segment rounded to 2 MiB
