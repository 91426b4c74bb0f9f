"""fma_image_verify on one GPU: Llama-3-8B's table, plain (K0 fill, incompressible) and PACKED (bf16 dummy weights), checked where
the sleeping image lies: the host store (K3 / K6 read it through its device alias, zero-copy over PCIe), this GPU's parking buffer
(HBM) and a file in DIR (reader threads pread into the pinned I/O windows, the kernels read each window over PCIe).  Each step
verifies each form in each tier once.  Rooflines from the same run: a plain pinned 8 GiB H2D copy (host), DIR's raw O_DIRECT read
rate with 12 threads x 16 MiB (file, as scripts/file_tier_bench.py measures it) and the H100's 3.35 TB/s HBM peak (local), beside
the kernels' own device-timed rate (the timeline's kernel rows).

    python scripts/verify_bench.py DIR [--steps 3] [--warmup 1] [--kv-gib 8] [--out profiles/image_verify_h100.json]

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

HBM_PEAK_GBS = 3350.0   # H100 SXM data sheet


def h2d_rate(torch, nbytes: int) -> float:
    """GB/s of one plain cudaMemcpyAsync from pinned host memory to HBM (median of 5)."""
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    rates = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        d.copy_(h, non_blocking=True)
        b.record()
        b.synchronize()
        rates.append(nbytes / (a.elapsed_time(b) * 1e-3) / 1e9)
    del h, d
    torch.cuda.empty_cache()
    return statistics.median(rates)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--kv-gib", type=float, default=8.0)
    ap.add_argument("--workload", default="llama-3-8b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import fma_b200
    from bench import fill_weights, gpu_identity
    from file_tier_bench import raw_rate
    from fma_b200 import _lib as L
    from fma_b200 import workloads as W

    tiers = {"host": L.FMA_TIER_HOST, "local": L.FMA_TIER_LOCAL, "file": L.FMA_TIER_FILE}
    os.makedirs(args.dir, exist_ok=True)
    probe = os.path.join(args.dir, ".fma_odirect_probe")
    try:
        os.close(os.open(probe, os.O_WRONLY | os.O_CREAT | os.O_DIRECT, 0o644))
        direct_ok = True
    except OSError:
        direct_ok = False
    finally:
        if os.path.exists(probe):
            os.unlink(probe)

    roof = {"host_h2d_gbs": h2d_rate(torch, 8 << 30), "local_hbm_peak_gbs": HBM_PEAK_GBS}
    table0 = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
    Wb = W.weight_bytes(table0)
    if direct_ok:
        rp = os.path.join(args.dir, "verify_bench_raw.bin")
        threads, chunk = 12, 16 << 20
        n = Wb // chunk * chunk
        raw_rate(rp, n, threads, chunk, True)
        roof["file_raw_o_direct_read_gbs"] = raw_rate(rp, n, threads, chunk, False)
        os.unlink(rp)
    print(f"rooflines: {roof}", file=sys.stderr, flush=True)

    rows = {}
    bit_exact = True
    for form in ("plain", "packed"):
        eng = fma_b200.Engine(0)
        table = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
        for s in table:
            eng.alloc(s.bytes, s.tag)
        fill_weights(eng, table, 1234, "prng" if form == "plain" else "bf16", torch)
        eng.set_option("pack", 1 if form == "packed" else 0)
        path = os.path.join(args.dir, f"verify_bench_{form}.fmaimg")
        eng.file_store(path)
        want = eng.digest_all(["weights"])
        eng.sleep(["weights"], tier=L.FMA_TIER_HOST, flags=L.FMA_FLAG_VERIFY)
        S = eng.stats()["image_store_bytes"]
        for name in ("host", "local", "file"):
            if name != "host":
                eng.move_image(tiers[name])
            samples = []
            for step in range(args.warmup + args.steps):
                t0 = time.perf_counter()
                bad = eng.verify_image()
                wall = time.perf_counter() - t0
                assert bad == [], bad
                tl = eng.timeline()
                kern = [r for r in tl if r["kind"] == "kernel"]
                io = [r for r in tl if r["kind"] == "file_io"]
                k_s = sum(r["t1_ms"] - r["t0_ms"] for r in kern) * 1e-3
                if step >= args.warmup:
                    samples.append(dict(wall_s=wall, gbs=S / wall / 1e9, kernel_s=k_s, kernel_gbs=S / k_s / 1e9 if k_s else None,
                                        launches=len(kern), io=("o_direct" if io[0]["idx"] == 1 else "page_cache") if io else None))
                print(f"{form} {name} step {step}: {wall:.3f} s ({S / wall / 1e9:.2f} GB/s stored bytes), kernels {k_s:.3f} s",
                      file=sys.stderr, flush=True)
            rows[f"{form}_{name}"] = dict(stored_bytes=S, weight_bytes=Wb, median_s=statistics.median(r["wall_s"] for r in samples),
                                          median_gbs=statistics.median(r["gbs"] for r in samples),
                                          median_kernel_gbs=statistics.median(r["kernel_gbs"] for r in samples if r["kernel_gbs"]),
                                          steps=samples)
        eng.wake(None, flags=L.FMA_FLAG_VERIFY)
        bit_exact = bit_exact and eng.digest_all(["weights"]) == want
        eng.file_store(None)
        if os.path.exists(path):
            os.unlink(path)
        eng.close()

    def against(key):
        tier = key.split("_", 1)[1]
        r = {"host": roof["host_h2d_gbs"], "local": HBM_PEAK_GBS, "file": roof.get("file_raw_o_direct_read_gbs")}[tier]
        return rows[key]["median_gbs"] / r if r else None

    out = {"metric": "image_verify_gbs", "unit": "GB/s of stored bytes", "workload": args.workload, "steps": args.steps,
           "warmup": args.warmup, "io_mode": "o_direct" if direct_ok else "page_cache", "gpu": gpu_identity(0), "bit_exact": bit_exact,
           "rooflines": roof, "results": rows, "fraction_of_roofline": {k: against(k) for k in rows}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
