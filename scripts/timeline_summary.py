#!/usr/bin/env python
"""Summarise the per-rank phase timelines bench.py --timeline wrote (fma_timeline) as markdown: for every rank the VMM calls of
the wake's mapper thread (start, duration, bytes), when the enqueue finished, the cadence of the K2 launches (= arrival of the H2D
ring slots: a gap longer than one slot's DMA time is a stall), for a resident share when its restore and the buffer's release
ended against the last K2 (both should end before it: off the critical path), and the total.

    python scripts/timeline_summary.py gpurun_out/tl/A [label] >> profiles/wake_timeline_r2.md
"""
import csv
import glob
import os
import statistics
import sys


def load(path):
    rows = list(csv.DictReader(open(path)))
    for r in rows:
        r["t0_ms"] = float(r["t0_ms"]); r["t1_ms"] = float(r["t1_ms"]); r["bytes"] = int(r["bytes"]); r["idx"] = int(r["idx"])
    return rows


def main():
    d = sys.argv[1]
    label = sys.argv[2] if len(sys.argv) > 2 else os.path.basename(d.rstrip("/"))
    files = sorted(glob.glob(os.path.join(d, "n*_rank*.csv")))
    if not files:
        sys.exit(f"no timelines under {d}")
    print(f"\n### {label}\n")
    print("| rank | wake total ms | plan ms | ring map (start→dur) | backed maps: n, first start→last end, Σdur, max dur | remap maps (start→dur, GiB) | gate waits Σ ms | enqueue end ms | K2: n, first begin, last end, median gap ms, max gap ms (at) | resident: restore end, release end ms | drain ms |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for f in files:
        rows = [r for r in load(f) if r["op"] == "wake"]
        rank = os.path.basename(f).split("rank")[1].split(".")[0]
        by = lambda k: [r for r in rows if r["kind"] == k]
        tot = by("total")[0]["t1_ms"] if by("total") else float("nan")
        plan = by("plan")[0]["t1_ms"] if by("plan") else float("nan")
        ring = by("map_ring")
        ring_s = f"{ring[0]['t0_ms']:.2f}→{ring[0]['t1_ms'] - ring[0]['t0_ms']:.2f}" if ring else "–"
        mb = by("map_backed")
        mb_s = (f"{len(mb)}, {mb[0]['t0_ms']:.1f}→{mb[-1]['t1_ms']:.1f}, {sum(r['t1_ms'] - r['t0_ms'] for r in mb):.1f}, "
                f"{max(r['t1_ms'] - r['t0_ms'] for r in mb):.1f}") if mb else "–"
        mr = by("map_remap")
        mr_s = "; ".join(f"{r['t0_ms']:.1f}→{r['t1_ms'] - r['t0_ms']:.1f} ({r['bytes'] / 2**30:.0f})" for r in mr) or "–"
        gw = sum(r["t1_ms"] - r["t0_ms"] for r in by("gate_wait"))
        enq = by("enqueue")[0]["t1_ms"] if by("enqueue") else float("nan")
        k = sorted(by("kernel"), key=lambda r: r["t0_ms"])
        if len(k) > 1:
            gaps = [k[i + 1]["t0_ms"] - k[i]["t0_ms"] for i in range(len(k) - 1)]
            gi = max(range(len(gaps)), key=lambda i: gaps[i])
            k_s = f"{len(k)}, {k[0]['t0_ms']:.1f}, {k[-1]['t1_ms']:.1f}, {statistics.median(gaps):.2f}, {gaps[gi]:.1f} (@{k[gi]['t0_ms']:.0f})"
        else:
            k_s = f"{len(k)}"
        rr, rf = by("res_restore"), by("res_free")
        res_s = (f"{max(r['t1_ms'] for r in rr):.1f}, " + (f"{rf[0]['t1_ms']:.1f}" if rf else "–")) if rr else "–"
        dr = by("drain")
        dr_s = f"{dr[0]['t1_ms'] - dr[0]['t0_ms']:.1f}" if dr else "–"
        print(f"| {rank} | {tot:.1f} | {plan:.2f} | {ring_s} | {mb_s} | {mr_s} | {gw:.1f} | {enq:.1f} | {k_s} | {res_s} | {dr_s} |")


if __name__ == "__main__":
    main()
