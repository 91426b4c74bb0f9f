"""Write-behind file-tier sleep (FMA_FLAG_WRITE_BEHIND) on one GPU: Llama-3-8B's table (32 GiB kv by default), plain (K0 fill,
incompressible) and PACKED (bf16 dummy weights) alternating, its file in DIR.  Per step and form:
  - a synchronous file-tier sleep vs a write-behind sleep: time to return, and the HBM cudaMemGetInfo reports freed at that moment;
  - the write-behind's time to commit (fma_image_writeback), as a rate of stored bytes against DIR's raw O_DIRECT write rate
    (12 threads x 16 MiB over 4 GiB) from the same run, and the pinned host DRAM the engine holds before and after the commit;
  - a wake right after a write-behind sleep returns (it pre-empts the job: the wb_cancel row) vs a host-tier wake, and a wake after
    the commit vs a wake after a synchronous file-tier sleep;
  - fma_swap of A (this model, asleep to the file tier) with B (the same weights, 4 GiB kv, waking from the host tier): synchronous,
    write-behind and host tier.
Every wake is checked with K3 digests.  The card's name and power limit are read in the same run.

    python scripts/write_behind_bench.py DIR [--steps 3] [--warmup 1] [--kv-gib 32] [--out profiles/write_behind_h100.json]

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
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--kv-gib", type=float, default=32.0)
    ap.add_argument("--workload", default="llama-3-8b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import fma_b200
    from bench import fill_weights, gpu_identity
    from file_tier_bench import raw_rate
    from fma_b200 import _lib as L
    from fma_b200 import workloads as W
    from prefetch_bench import filesystem_of

    os.makedirs(args.dir, exist_ok=True)
    gpu = gpu_identity(0)
    roof = {}
    try:
        rp = os.path.join(args.dir, "write_behind_bench_raw.bin")
        roof["file_raw_o_direct_write_gbs"] = raw_rate(rp, 4 << 30, 12, 16 << 20, True)
        os.unlink(rp)
    except OSError as e:
        roof["file_raw_o_direct_write_gbs"] = None
        print(f"no O_DIRECT roofline: {e}", file=sys.stderr)
    print(f"rooflines: {roof}", file=sys.stderr, flush=True)

    def free_hbm():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]

    def pinned(e):
        st = e.stats()
        return st["host_store_bytes"] + st["io_buffer_bytes"]

    def row(e, kind):
        return [r for r in e.timeline() if r["kind"] == kind]

    results = {}
    bit_exact = True
    for form in ("plain", "packed"):
        a, b = fma_b200.Engine(0), fma_b200.Engine(0)
        ta = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
        tb = W.allocation_table(args.workload, kv_cache_bytes=4 << 30)
        for e, t in ((a, ta), (b, tb)):
            for s in t:
                e.alloc(s.bytes, s.tag)
            fill_weights(e, t, 1234, "prng" if form == "plain" else "bf16", torch)
            e.set_option("pack", 1 if form == "packed" else 0)
        Wb = W.weight_bytes(ta)
        path = os.path.join(args.dir, f"write_behind_bench_{form}.fmaimg")
        a.file_store(path)
        a.host_reserve(Wb)
        b.host_reserve(Wb)
        want_a, want_b = a.digest_all(["weights"]), b.digest_all(["weights"])
        b.sleep(["weights"], tier=L.FMA_TIER_HOST)

        def woke(e, want):
            nonlocal bit_exact
            ok = e.digest_all(["weights"]) == want
            bit_exact = bit_exact and ok
            return ok

        samples = []
        for step in range(args.warmup + args.steps):
            s = {}
            # synchronous file-tier sleep, then a file-tier wake (the host store stays pinned: the write-behind sleeps reuse it)
            f0 = free_hbm()
            t0 = time.perf_counter()
            a.sleep(["weights"], tier=L.FMA_TIER_FILE)
            s["sync_sleep_return_s"] = time.perf_counter() - t0
            s["sync_freed_at_return"] = free_hbm() - f0
            stored = a.stats()["image_store_bytes"]
            t0 = time.perf_counter()
            a.wake(None)
            s["file_wake_after_sync_s"] = time.perf_counter() - t0
            s["exact_sync"] = woke(a, want_a)
            # write-behind sleep: return, freed HBM, commit, pinned DRAM around the commit, then a wake from the file
            f0 = free_hbm()
            t0 = time.perf_counter()
            a.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND)
            s["wb_sleep_return_s"] = time.perf_counter() - t0
            s["wb_freed_at_return"] = free_hbm() - f0
            s["wb_taken"] = bool(row(a, "wb_start"))
            s["pinned_before_commit"] = pinned(a)
            a.writeback(None)
            s["wb_commit_s"] = time.perf_counter() - t0
            s["wb_commit_tier"] = a.stats()["tier"]
            s["pinned_after_commit"] = pinned(a)
            s["commit_gbs"] = stored / max(s["wb_commit_s"] - s["wb_sleep_return_s"], 1e-9) / 1e9
            t0 = time.perf_counter()
            a.wake(None)
            s["file_wake_after_commit_s"] = time.perf_counter() - t0
            s["exact_commit"] = woke(a, want_a)
            a.host_reserve(Wb)    # (the commit released the store: pinned again outside the measured calls)
            # a wake mid-write, against a host-tier wake
            a.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_WRITE_BEHIND)
            s["pending_at_wake"] = a.writeback(0)[1]
            t0 = time.perf_counter()
            a.wake(None)
            s["wake_mid_write_s"] = time.perf_counter() - t0
            c = row(a, "wb_cancel")
            s["wb_cancel_s"] = (c[0]["t1_ms"] - c[0]["t0_ms"]) * 1e-3 if c else None
            s["exact_mid_write"] = woke(a, want_a)
            a.sleep(["weights"], tier=L.FMA_TIER_HOST)
            t0 = time.perf_counter()
            a.wake(None)
            s["host_wake_s"] = time.perf_counter() - t0
            s["exact_host"] = woke(a, want_a)
            # hot swap A -> B and back: A to the file tier (synchronous / write-behind) or the host tier, B from the host tier
            for name, tier, flags in (("sync", L.FMA_TIER_FILE, 0), ("write_behind", L.FMA_TIER_FILE, L.FMA_FLAG_WRITE_BEHIND),
                                      ("host", L.FMA_TIER_HOST, 0)):
                t0 = time.perf_counter()
                a.swap_out_for(b, offload_tags=("weights",), tier=tier, flags=flags)
                s[f"swap_{name}_s"] = time.perf_counter() - t0
                s[f"exact_swap_{name}"] = woke(b, want_b)
                a.writeback(None)
                if a.stats()["host_store_bytes"] == 0:
                    a.host_reserve(Wb)
                b.sleep(["weights"], tier=L.FMA_TIER_HOST)
                a.wake(None)
                woke(a, want_a)
            print(f"{form} step {step}: {json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in s.items()})}",
                  file=sys.stderr, flush=True)
            if step >= args.warmup:
                samples.append(s)
        med = {k: statistics.median(x[k] for x in samples) for k in samples[0] if isinstance(samples[0][k], (int, float))
               and not isinstance(samples[0][k], bool) and all(x[k] is not None for x in samples)}
        results[form] = dict(weight_bytes=Wb, stored_bytes=stored, median=med, steps=samples,
                             commit_fraction_of_raw_write=(med["commit_gbs"] / roof["file_raw_o_direct_write_gbs"]
                                                           if roof.get("file_raw_o_direct_write_gbs") else None))
        a.file_store(None)
        if os.path.exists(path):
            os.unlink(path)
        a.close()
        b.close()

    out = {"metric": "write_behind", "unit": "s / GB/s of stored bytes", "workload": args.workload, "kv_gib": args.kv_gib,
           "steps": args.steps, "warmup": args.warmup, "file_dir": filesystem_of(args.dir), "gpu": gpu, "bit_exact": bit_exact,
           "rooflines": roof, "results": results}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
