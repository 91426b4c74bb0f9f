#!/usr/bin/env python
"""Resident share sweep on one GPU: the Llama-3-8B table (32 GiB kv_cache) with bf16 dummy weights (U(-1e-3, 1e-3), as
bench.py's packed child fills them), slept and woken at resident budgets of 0, 1, 2 and 3 GiB x pack 0 / 1.  The cells are
alternated within one process, step by step, after a warm-up of every cell.

Per cell: median and min-max of the wake and sleep latency, the bytes that cross PCIe per wake (image_store_bytes), the
resident bytes, bit-exactness by K3 digests on every wake, the HBM nvidia-smi reports for this process while it sleeps
(--query-compute-apps, read-only; None when nvidia-smi lists no process with this pid, as inside some containers), the HBM in
use on the whole device (cudaMemGetInfo: includes every other process on the GPU) and, from the last wake's timeline, when the resident restore and the buffer's release ended
against the last scatter of the host part.  Then a clean incremental sleep with and without a resident share.

    python scripts/resident_sweep.py --steps 10 --warmup 2 --out /tmp/resident_sweep
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GiB = 1 << 30


def process_hbm_mib() -> int | None:
    """HBM nvidia-smi attributes to this process (the number a per-GPU sleeper budget is compared against)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout
        for line in out.strip().splitlines():
            pid, mib = [x.strip() for x in line.split(",")]
            if int(pid) == os.getpid():
                return int(mib)
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return None


def timeline_marks(tl) -> dict:
    """When the resident restore and the release ended vs. the last launch of the host part (ms since the wake's entry)."""
    k = [r for r in tl if r["kind"] == "kernel"]
    res = [r for r in tl if r["kind"] == "res_restore"]
    free = [r for r in tl if r["kind"] == "res_free"]
    total = [r for r in tl if r["kind"] == "total"]
    return {"last_host_scatter_end_ms": round(max(r["t1_ms"] for r in k), 2) if k else None,
            "res_restore_end_ms": round(max(r["t1_ms"] for r in res), 2) if res else None,
            "res_restore_launches": len(res),
            "res_free_ms": [round(free[0]["t0_ms"], 2), round(free[0]["t1_ms"], 2)] if free else None,
            "wake_total_ms": round(total[0]["t1_ms"], 2) if total else None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--kv-gib", type=float, default=32)
    ap.add_argument("--budgets-gib", default="0,1,2,3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bench
    import fma_b200
    from fma_b200 import workloads as W

    torch.cuda.set_device(0)
    workload = bench.workload_for(1, None)
    eng = fma_b200.Engine(0)
    table = W.allocation_table(workload, kv_cache_bytes=int(args.kv_gib * GiB))
    for s in table:
        eng.alloc(s.bytes, s.tag)
    Wb = W.weight_bytes(table)
    bench.fill_weights(eng, table, 1234, "bf16", torch)
    before = eng.digest_all(["weights"])
    eng.host_reserve(Wb)
    budgets = [int(float(b) * GiB) for b in args.budgets_gib.split(",")]
    cells = [(pack, b) for pack in (0, 1) for b in budgets]
    rows = {c: [] for c in cells}
    hbm_asleep = {}
    marks = {}
    for step in range(args.warmup + args.steps):
        for c in cells:
            pack, b = c
            eng.set_option("pack", pack)
            eng.set_option("resident_bytes", b)
            eng.sleep(["weights"])
            s1 = eng.stats()
            if step == args.warmup:
                free, total = torch.cuda.mem_get_info()
                hbm_asleep[c] = (process_hbm_mib(), (total - free) >> 20)
            eng.wake(None)
            s2 = eng.stats()
            ok = eng.digest_all(["weights"]) == before
            if step >= args.warmup:
                rows[c].append((s1, s2, ok))
            if step == args.warmup + args.steps - 1:
                marks[c] = timeline_marks(eng.timeline())
    free, total = torch.cuda.mem_get_info()
    hbm_awake = (process_hbm_mib(), (total - free) >> 20)
    result = {"gpu": bench.gpu_identity(0), "workload": workload, "weights_gib": round(Wb / GiB, 3), "kv_gib": args.kv_gib,
              "contents": "bf16 U(-1e-3, 1e-3)", "steps": args.steps, "warmup": args.warmup, "hbm_process_awake_mib": hbm_awake[0], "hbm_device_used_awake_mib": hbm_awake[1], "cells": []}
    for c in cells:
        r = rows[c]
        wake = [x[1]["wake_seconds"] for x in r]
        sleep = [x[0]["sleep_seconds"] for x in r]
        result["cells"].append({
            "pack": c[0], "budget_gib": c[1] / GiB,
            "wake_s_median": round(statistics.median(wake), 5), "wake_s_min_max": [round(min(wake), 5), round(max(wake), 5)],
            "sleep_s_median": round(statistics.median(sleep), 5), "sleep_s_min_max": [round(min(sleep), 5), round(max(sleep), 5)],
            "link_bytes_per_wake": r[-1][0]["image_store_bytes"], "resident_bytes": r[-1][0]["resident_bytes"],
            "image_packed": r[-1][0]["image_packed"], "bit_exact_every_wake": all(x[2] for x in r),
            "hbm_process_asleep_mib": hbm_asleep[c][0], "hbm_device_used_asleep_mib": hbm_asleep[c][1],
            "last_wake_timeline": marks.get(c)})
    # a clean INCREMENTAL sleep with and without a resident share (plain image): the first sleep seeds the digests
    inc = []
    eng.set_option("pack", 0)
    eng.set_option("incremental", 1)
    for b in (0, budgets[-1]):
        eng.set_option("resident_bytes", b)
        cyc = []
        for _ in range(4):
            eng.sleep(["weights"]); s1 = eng.stats()
            eng.wake(None); s2 = eng.stats()
            cyc.append({"sleep_s": round(s1["sleep_seconds"], 5), "sleep_bytes_copied": s1["sleep_bytes_copied"],
                        "resident_bytes": s1["resident_bytes"], "wake_s": round(s2["wake_seconds"], 5)})
        inc.append({"budget_gib": b / GiB, "cycles": cyc, "bit_exact": eng.digest_all(["weights"]) == before})
    eng.set_option("incremental", 0)
    result["incremental"] = inc
    eng.close()
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "resident_sweep.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
