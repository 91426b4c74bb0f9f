"""Synthetic per-rank allocation tables for the BASELINE.json configs (SURVEY.md §8a/§8d).

A table is what the allocator sees at load time: a list of (segment_bytes, tag) in allocation
order.  PyTorch hands the pluggable allocator *segments*, not tensors, so tensors are first run
through the caching allocator's sizing rules (torch:include/c10/core/AllocatorConfig.h:17-25,
as restated in SURVEY.md §8c): <= 1 MiB -> packed into 2 MiB small-pool segments; 1..10 MiB ->
packed into 20 MiB segments; >= 10 MiB -> own segment rounded up to 2 MiB.  Tensor order follows
vLLM's module construction order (embed, per layer qkv/o/gate_up/down/norms, final norm, lm_head),
which is what makes device VAs scattered the way the reference's are.

Only shapes are modelled: there is no floating-point work anywhere on this path.
"""
from __future__ import annotations

import dataclasses

MiB = 1 << 20
GiB = 1 << 30
PAGE = 2 * MiB
K_SMALL_SIZE = 1 * MiB        # kSmallSize
K_SMALL_BUFFER = 2 * MiB      # kSmallBuffer
K_MIN_LARGE_ALLOC = 10 * MiB  # kMinLargeAlloc
K_LARGE_BUFFER = 20 * MiB     # kLargeBuffer
K_ROUND_LARGE = 2 * MiB       # kRoundLarge
K_MIN_BLOCK = 512             # kMinBlockSize


@dataclasses.dataclass(frozen=True)
class SegmentSpec:
    bytes: int
    tag: str
    note: str = ""


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def simulate_segments(tensors: list[tuple[str, int]], tag: str) -> list[SegmentSpec]:
    """Run tensors (no frees during load) through the caching allocator's placement rules and return the
    segments it requests from the pluggable allocator, in request order.  Modelled (and pinned against a live
    vLLM + torch run by tests/golden/vllm_cumem_roundtrip.json): 512 B size rounding; two pools (<= 1 MiB small,
    else large); best-fit reuse of the free remainder of earlier segments of the same pool — a 12 MiB tensor does
    land in the tail of a 20 MiB segment; a remainder is only split off when it is worth keeping
    (> 1 MiB in the large pool, >= 512 B in the small pool)."""
    segs: list[SegmentSpec] = []
    free = {"small": [], "large": []}  # free block sizes per pool

    def place(pool: str, size: int, seg_bytes: int, note: str) -> None:
        blocks = free[pool]
        fit = min((b for b in blocks if b >= size), default=None)   # lower_bound: smallest block that fits
        if fit is None:
            segs.append(SegmentSpec(seg_bytes, tag, note))
            fit = seg_bytes
        else:
            blocks.remove(fit)
        rem = fit - size
        if (pool == "small" and rem >= K_MIN_BLOCK) or (pool == "large" and rem > K_SMALL_SIZE):
            blocks.append(rem)

    for name, nbytes in tensors:
        size = _round_up(max(nbytes, 1), K_MIN_BLOCK)
        if size <= K_SMALL_SIZE:
            place("small", size, K_SMALL_BUFFER, "small-pool")
        elif size < K_MIN_LARGE_ALLOC:
            place("large", size, K_LARGE_BUFFER, "20MiB-pool")
        else:
            place("large", size, _round_up(size, K_ROUND_LARGE), name)
    return segs


def _llama_tensors(*, hidden: int, inter: int, heads: int, kv_heads: int, head_dim: int, vocab: int, layers: int,
                   tp: int, dtype_bytes: int = 2, tie_embeddings: bool = False, max_pos: int | None = None) -> list[tuple[str, int]]:
    """Fused vLLM layouts per TP rank: qkv_proj, o_proj, gate_up_proj, down_proj, two RMSNorm weights — plus, with ``max_pos``, the
    non-parameter buffers a live vLLM allocates under the ``weights`` tag (SURVEY.md §8d): the rotary embedding built right after
    layer 0's o_proj (``inv_freq``: the first small-pool allocation; ``cos_sin_cache`` = max_pos x head_dim x dtype: 1-10 MiB, so a
    20 MiB large-pool segment), shared by all layers.  What a live vLLM 0.22 + torch 2.11 weights pool holds for Llama-3-8B
    shapes (``scripts/e2e_launcher_vllm.py`` compares the two): 132 segments, 16 083 058 688 bytes, order
    [1002, 48, 32, 2, 20, 224, 112, ...] MiB."""
    b = dtype_bytes
    q_rows = heads * head_dim // tp
    kv_rows = max(kv_heads // tp, 1) * head_dim
    vocab_rows = _round_up(vocab, 64 * tp) // tp if vocab % tp else vocab // tp
    t: list[tuple[str, int]] = [("embed_tokens", vocab_rows * hidden * b)]
    for i in range(layers):
        t.append((f"L{i}.qkv_proj", (q_rows + 2 * kv_rows) * hidden * b))
        t.append((f"L{i}.o_proj", hidden * q_rows * b))
        if i == 0 and max_pos:
            t.append(("rotary_emb.inv_freq", head_dim // 2 * 4))
            t.append(("rotary_emb.cos_sin_cache", max_pos * head_dim * b))
        t.append((f"L{i}.gate_up_proj", 2 * (inter // tp) * hidden * b))
        t.append((f"L{i}.down_proj", hidden * (inter // tp) * b))
        t.append((f"L{i}.input_layernorm", hidden * b))
        t.append((f"L{i}.post_attention_layernorm", hidden * b))
    t.append(("norm", hidden * b))
    if not tie_embeddings:
        t.append(("lm_head", vocab_rows * hidden * b))
    return t


def _opt_tensors(*, hidden: int, ffn: int, vocab: int, max_pos: int, layers: int, dtype_bytes: int = 2):
    b = dtype_bytes
    t: list[tuple[str, int]] = [("embed_tokens", vocab * hidden * b), ("embed_positions", (max_pos + 2) * hidden * b)]
    for i in range(layers):
        t += [(f"L{i}.qkv_proj.weight", 3 * hidden * hidden * b), (f"L{i}.qkv_proj.bias", 3 * hidden * b),
              (f"L{i}.out_proj.weight", hidden * hidden * b), (f"L{i}.out_proj.bias", hidden * b),
              (f"L{i}.self_attn_layer_norm.w", hidden * b), (f"L{i}.self_attn_layer_norm.b", hidden * b),
              (f"L{i}.fc1.weight", ffn * hidden * b), (f"L{i}.fc1.bias", ffn * b),
              (f"L{i}.fc2.weight", hidden * ffn * b), (f"L{i}.fc2.bias", hidden * b),
              (f"L{i}.final_layer_norm.w", hidden * b), (f"L{i}.final_layer_norm.b", hidden * b)]
    t += [("final_layer_norm.w", hidden * b), ("final_layer_norm.b", hidden * b)]  # lm_head tied to embed_tokens
    return t


MODELS = {
    # name: (tensor generator kwargs, layers for the kv split)
    "llama-3-8b": dict(kind="llama", hidden=4096, inter=14336, heads=32, kv_heads=8, head_dim=128, vocab=128256,
                       layers=32, tp=1, max_pos=8192),
    "llama-3-70b-tp8": dict(kind="llama", hidden=8192, inter=28672, heads=64, kv_heads=8, head_dim=128, vocab=128256,
                            layers=80, tp=8, max_pos=8192),
    "mistral-7b": dict(kind="llama", hidden=4096, inter=14336, heads=32, kv_heads=8, head_dim=128, vocab=32768,
                       layers=32, tp=1, max_pos=32768),
    "opt-125m": dict(kind="opt", hidden=768, ffn=3072, vocab=50272, max_pos=2048, layers=12),
    # small shapes for tests / smoke (same structure, seconds on the oracle)
    "tiny-llama-test": dict(kind="llama", hidden=1024, inter=6144, heads=16, kv_heads=4, head_dim=64, vocab=16384,
                            layers=3, tp=1),
}


def model_tensors(name: str) -> list[tuple[str, int]]:
    cfg = dict(MODELS[name])
    kind = cfg.pop("kind")
    return _llama_tensors(**cfg) if kind == "llama" else _opt_tensors(**cfg)


def allocation_table(name: str, kv_cache_bytes: int = 0, kv_tensors: int | None = None) -> list[SegmentSpec]:
    """Per-rank table: `weights` segments in load order, then `kv_cache` segments (remapped on wake,
    never copied: Worker.sleep level 1 offloads only ("weights",), gpu_worker.py:169-170)."""
    table = simulate_segments(model_tensors(name), "weights")
    if kv_cache_bytes > 0:
        n = kv_tensors or MODELS[name]["layers"]
        per = _round_up(kv_cache_bytes // n, PAGE)
        table += simulate_segments([(f"kv.{i}", per) for i in range(n)], "kv_cache")
    return table


def weight_bytes(table: list[SegmentSpec]) -> int:
    return sum(s.bytes for s in table if s.tag == "weights")


def total_bytes(table: list[SegmentSpec]) -> int:
    return sum(s.bytes for s in table)
