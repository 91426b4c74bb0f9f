"""Demotion behind the call (fma_image_move_flags with FMA_FLAG_WRITE_BEHIND) on one GPU: Llama-3-8B's table (4 GiB kv), plain (K0
fill, incompressible) and PACKED (bf16 dummy weights) alternating, its file in DIR.  Engine A is demoted; engine B, with the same
table, sleeps in the host tier beside it.  Per step and form:
  - the return time of move_image(file, behind=True) against the synchronous move_image(file), both from a host-tier sleep;
  - the demotion's commit time (fma_image_writeback) and the disk's write rate it implies (stored bytes over commit time);
  - a host-tier wake of B while A's demotion writes (checked to still be writing when B's wake returns) against the same wake
    undisturbed, taken in the same step;
  - a wake of A that pre-empts its own demotion: its time and its wb_cancel row.
Every wake is checked with K3 digests.  The card's name and power limit and DIR's filesystem are read in the same run.

    python scripts/demote_bench.py DIR [--steps 2] [--warmup 0] [--out profiles/demote_h100.json]

Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=0)
    ap.add_argument("--kv-gib", type=float, default=4.0)
    ap.add_argument("--workload", default="llama-3-8b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import fma_b200
    from bench import fill_weights, gpu_identity
    from fma_b200 import _lib as L
    from fma_b200 import workloads as W
    from prefetch_bench import filesystem_of

    os.makedirs(args.dir, exist_ok=True)
    gpu = gpu_identity(0)
    bit_exact = True

    def woke(e, want):
        nonlocal bit_exact
        ok = e.digest_all(["weights"]) == want
        bit_exact = bit_exact and ok
        return ok

    def timed(f):
        t0 = time.perf_counter()
        f()
        return time.perf_counter() - t0

    results = {}
    for form in ("plain", "packed"):
        a, b = fma_b200.Engine(0), fma_b200.Engine(0)
        t = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
        for e, seed in ((a, 1234), (b, 4321)):
            for s in t:
                e.alloc(s.bytes, s.tag)
            fill_weights(e, t, seed, "prng" if form == "plain" else "bf16", torch)
            e.set_option("pack", 1 if form == "packed" else 0)
        path = os.path.join(args.dir, f"demote_bench_{form}.fmaimg")
        a.file_store(path)
        want_a, want_b = a.digest_all(["weights"]), b.digest_all(["weights"])
        b.sleep(["weights"], tier=L.FMA_TIER_HOST)
        samples = []
        for step in range(args.warmup + args.steps):
            s = {}
            # the synchronous move, then a wake from the file
            a.sleep(["weights"], tier=L.FMA_TIER_HOST)
            stored = a.stats()["image_store_bytes"]
            s["sync_move_s"] = timed(lambda: a.move_image(L.FMA_TIER_FILE))
            s["file_wake_s"] = timed(lambda: a.wake(None))
            s["exact_sync"] = woke(a, want_a)
            # the demotion: return, commit, then a wake from the file
            a.sleep(["weights"], tier=L.FMA_TIER_HOST)
            t0 = time.perf_counter()
            a.move_image(L.FMA_TIER_FILE, behind=True)
            s["demote_return_s"] = time.perf_counter() - t0
            a.writeback(None)
            s["demote_commit_s"] = time.perf_counter() - t0
            s["commit_tier"] = a.stats()["tier"]
            s["commit_gbs"] = stored / s["demote_commit_s"] / 1e9
            s["file_wake_after_commit_s"] = timed(lambda: a.wake(None))
            s["exact_commit"] = woke(a, want_a)
            # B's host-tier wake undisturbed, then while A's demotion writes
            s["b_wake_alone_s"] = timed(lambda: b.wake(None))
            s["exact_b_alone"] = woke(b, want_b)
            b.sleep(["weights"], tier=L.FMA_TIER_HOST)
            a.sleep(["weights"], tier=L.FMA_TIER_HOST)
            a.move_image(L.FMA_TIER_FILE, behind=True)
            s["b_wake_beside_demotion_s"] = timed(lambda: b.wake(None))
            s["demotion_wrote_throughout"] = a.writeback(0)[0] == 1
            s["exact_b_beside"] = woke(b, want_b)
            b.sleep(["weights"], tier=L.FMA_TIER_HOST)
            # A's wake pre-empts its own demotion
            s["a_wake_mid_demotion_s"] = timed(lambda: a.wake(None))
            c = [r for r in a.timeline() if r["kind"] == "wb_cancel"]
            s["wb_cancel_s"] = (c[0]["t1_ms"] - c[0]["t0_ms"]) * 1e-3 if c else None
            s["exact_mid_demotion"] = woke(a, want_a)
            print(f"{form} step {step}: {json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in s.items()})}",
                  file=sys.stderr, flush=True)
            if step >= args.warmup:
                samples.append(s)
        med = {k: statistics.median(x[k] for x in samples) for k in samples[0] if isinstance(samples[0][k], (int, float))
               and not isinstance(samples[0][k], bool) and all(x[k] is not None for x in samples)}
        results[form] = dict(weight_bytes=W.weight_bytes(t), stored_bytes=stored, median=med, steps=samples)
        a.file_store(None)
        if os.path.exists(path):
            os.unlink(path)
        a.close()
        b.close()

    out = {"metric": "demote", "unit": "s / GB/s of stored bytes", "workload": args.workload, "kv_gib": args.kv_gib, "steps": args.steps,
           "warmup": args.warmup, "file_dir": filesystem_of(args.dir), "gpu": gpu, "bit_exact": bit_exact, "results": results,
           "not_measured": ["the node's peak host bytes with three child processes under a budget of two images"]}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
