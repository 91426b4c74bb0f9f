"""fma_image_prefetch on one GPU: Llama-3-8B's table (32 GiB kv by default), plain (K0 fill, incompressible) and PACKED (bf16 dummy
weights) alternating, asleep in the host store and in a file in DIR.  Each step prefetches a budget of 0, 4 GiB (the controller's
per-sleeper unit) or the whole image, times the prefetch and the wake that follows, reads from the wake's timeline how many bytes
still crossed the link (host tier: the enqueue row, in weight bytes) or came off the disk (file tier: the file_io row, stored bytes),
and checks the weights with K3 digests.  The option "incremental" is on, so each sleep after the first is clean and moves nothing:
every step starts from the same image.  Once per form and tier, cudaMemGetInfo is read before a whole-image prefetch, after it and
after prefetch_image(0).  Rooflines from the same run: a plain pinned 8 GiB H2D copy, and DIR's raw O_DIRECT read rate with
12 threads x 16 MiB over a 4 GiB file.

    python scripts/prefetch_bench.py DIR [--steps 3] [--warmup 1] [--kv-gib 32] [--out profiles/image_prefetch_h100.json]

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


def filesystem_of(path: str) -> dict:
    """mount point and filesystem type of `path` (the longest matching entry of /proc/mounts)"""
    path = os.path.realpath(path)
    best = {"mount": None, "fstype": None}
    try:
        with open("/proc/mounts") as f:
            for line in f:
                dev, mnt, fstype = line.split()[:3]
                if (path == mnt or path.startswith(mnt.rstrip("/") + "/")) and len(mnt) >= len(best["mount"] or ""):
                    best = {"mount": mnt, "fstype": fstype, "device": dev}
    except OSError:
        pass
    return best


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
    from verify_bench import h2d_rate

    os.makedirs(args.dir, exist_ok=True)
    roof = {"host_h2d_gbs": h2d_rate(torch, 8 << 30)}
    try:
        rp = os.path.join(args.dir, "prefetch_bench_raw.bin")
        threads, chunk, n = 12, 16 << 20, 4 << 30
        raw_rate(rp, n, threads, chunk, True)
        roof["file_raw_o_direct_read_gbs"] = raw_rate(rp, n, threads, chunk, False)
        os.unlink(rp)
    except OSError as e:
        roof["file_raw_o_direct_read_gbs"] = None
        print(f"no O_DIRECT roofline: {e}", file=sys.stderr)
    print(f"rooflines: {roof}", file=sys.stderr, flush=True)

    tiers = {"host": L.FMA_TIER_HOST, "file": L.FMA_TIER_FILE}
    budgets = {"zero": 0, "4gib": 4 << 30, "whole": 1 << 50}
    rows, hbm = {}, {}
    bit_exact = True
    for form in ("plain", "packed"):
        eng = fma_b200.Engine(0)
        table = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
        for s in table:
            eng.alloc(s.bytes, s.tag)
        fill_weights(eng, table, 1234, "prng" if form == "plain" else "bf16", torch)
        eng.set_option("pack", 1 if form == "packed" else 0)
        eng.set_option("incremental", 1)
        path = os.path.join(args.dir, f"prefetch_bench_{form}.fmaimg")
        eng.file_store(path)
        want = eng.digest_all(["weights"])
        Wb = W.weight_bytes(table)
        for tname, tier in tiers.items():
            eng.sleep(["weights"], tier=tier, flags=L.FMA_FLAG_VERIFY)
            S = eng.stats()["image_store_bytes"]
            # HBM as the driver reports it: before a whole-image prefetch, after it, after the hand-back
            torch.cuda.synchronize()
            f0 = torch.cuda.mem_get_info(0)[0]
            eng.prefetch_image(budgets["whole"])
            f1 = torch.cuda.mem_get_info(0)[0]
            pf = eng.stats()["prefetched_bytes"]
            eng.prefetch_image(0)
            f2 = torch.cuda.mem_get_info(0)[0]
            hbm[f"{form}_{tname}"] = dict(free_before=f0, free_prefetched=f1, free_after_drop=f2, prefetched_bytes=pf,
                                          taken=f0 - f1, given_back=f2 - f1)
            for bname, budget in budgets.items():
                samples = []
                for step in range(args.warmup + args.steps):
                    if not eng.is_sleeping():
                        eng.sleep(["weights"], tier=tier, flags=L.FMA_FLAG_VERIFY)
                    clean = eng.stats()["sleep_bytes_copied"]
                    t0 = time.perf_counter()
                    eng.prefetch_image(budget)
                    pf_s = time.perf_counter() - t0
                    pf_bytes = eng.stats()["prefetched_bytes"]
                    pf_rows = eng.timeline()
                    t0 = time.perf_counter()
                    eng.wake(None, flags=L.FMA_FLAG_VERIFY)
                    wake_s = time.perf_counter() - t0
                    tl = eng.timeline()
                    link = sum(r["bytes"] for r in tl if r["kind"] == ("enqueue" if tname == "host" else "file_io"))
                    restore = [r for r in tl if r["kind"] == "pf_restore"]
                    exact = eng.digest_all(["weights"]) == want
                    bit_exact = bit_exact and exact
                    if step >= args.warmup:
                        samples.append(dict(prefetch_s=pf_s if pf_bytes else 0.0, prefetch_gbs=pf_bytes / pf_s / 1e9 if pf_bytes else None,
                                            prefetched_bytes=pf_bytes, wake_s=wake_s, wake_engine_s=eng.stats()["wake_seconds"],
                                            link_bytes=link, restore_pieces=len(restore),
                                            restore_kernel_s=sum(r["t1_ms"] - r["t0_ms"] for r in restore) * 1e-3,
                                            prefetch_rows=sorted({r["kind"] for r in pf_rows}),
                                            previous_sleep_bytes_copied=clean, bit_exact=exact))
                    print(f"{form} {tname} {bname} step {step}: prefetch {pf_bytes / 2**30:.2f} GiB in {pf_s:.3f} s, wake {wake_s:.3f} s, "
                          f"link {link / 2**30:.2f} GiB, exact {exact}", file=sys.stderr, flush=True)
                prs = [r["prefetch_gbs"] for r in samples if r["prefetch_gbs"]]
                rows[f"{form}_{tname}_{bname}"] = dict(
                    stored_bytes=S, weight_bytes=Wb, prefetched_bytes=samples[0]["prefetched_bytes"],
                    median_prefetch_s=statistics.median(r["prefetch_s"] for r in samples),
                    median_prefetch_gbs=statistics.median(prs) if prs else None,
                    median_wake_s=statistics.median(r["wake_s"] for r in samples),
                    link_bytes_per_wake=samples[0]["link_bytes"], steps=samples)
        eng.file_store(None)
        if os.path.exists(path):
            os.unlink(path)
        eng.close()

    def against(key):
        r = rows[key]
        if r["median_prefetch_gbs"] is None:
            return None
        ref = roof["host_h2d_gbs"] if "_host_" in key else roof.get("file_raw_o_direct_read_gbs")
        return r["median_prefetch_gbs"] / ref if ref else None

    out = {"metric": "image_prefetch", "unit": "s / GB/s of stored bytes", "workload": args.workload, "kv_gib": args.kv_gib,
           "steps": args.steps, "warmup": args.warmup, "file_dir": filesystem_of(args.dir), "gpu": gpu_identity(0), "bit_exact": bit_exact,
           "rooflines": roof, "hbm": hbm, "results": rows,
           "prefetch_fraction_of_roofline": {k: against(k) for k in rows}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
