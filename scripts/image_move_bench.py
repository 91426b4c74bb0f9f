"""Moves of a sleeping image between tiers on one GPU (fma_image_move): Llama-3-8B's table, plain (K0 fill, incompressible) and
PACKED (bf16 dummy weights), alternating over the timed steps.  Every step moves each form's image through the six directions of one
GPU, host -> file -> host -> local -> file -> local -> host, and times each move and the wake that follows it (the image is slept
back to the move's destination before the next move).  A plain host-tier wake is timed in the same alternation, to set the wake
after a file -> host promotion against it.  Rooflines from the same run: DIR's sequential O_DIRECT write and read rate with the
engine's thread count and chunk size (as scripts/file_tier_bench.py measures it) and a plain pinned D2H / H2D copy rate.

    python scripts/image_move_bench.py DIR [--steps 2] [--warmup 0] [--kv-gib 8] [--out profiles/image_move_h100.json]

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

MOVES = [("host", "file"), ("file", "host"), ("host", "local"), ("local", "file"), ("file", "local"), ("local", "host")]


def pinned_copy_rate(torch, nbytes: int) -> dict:
    """GB/s of one plain cudaMemcpyAsync each way between pinned host memory and HBM (median of 5)."""
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    out = {}
    for name, dst, src in (("h2d_gbs", d, h), ("d2h_gbs", h, d)):
        rates = []
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dst.copy_(src, non_blocking=True)
            b.record()
            b.synchronize()
            rates.append(nbytes / (a.elapsed_time(b) * 1e-3) / 1e9)
        out[name] = statistics.median(rates)
    del h, d
    torch.cuda.empty_cache()
    out["bytes"] = nbytes
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=0)
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

    tier = {"host": L.FMA_TIER_HOST, "local": L.FMA_TIER_LOCAL, "file": L.FMA_TIER_FILE}
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

    engines, tables, digests, paths = {}, {}, {}, {}
    for form in ("plain", "packed"):
        eng = fma_b200.Engine(0)
        table = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
        for s in table:
            eng.alloc(s.bytes, s.tag)
        fill_weights(eng, table, 1234, "prng" if form == "plain" else "bf16", torch)
        eng.set_option("pack", 1 if form == "packed" else 0)
        paths[form] = os.path.join(args.dir, f"image_move_bench_{form}.fmaimg")
        eng.file_store(paths[form])
        engines[form], tables[form] = eng, table
        digests[form] = eng.digest_all(["weights"])
        eng.sleep(["weights"], tier=L.FMA_TIER_HOST)   # one model on the GPU at a time; this sleep is not timed
    Wb = W.weight_bytes(tables["plain"])
    threads, chunk = 12, 16 << 20                     # the engine's load_threads / load_chunk_bytes defaults

    roof = {"pinned": pinned_copy_rate(torch, 4 << 30)}
    print(f"pinned copy: {roof['pinned']}", file=sys.stderr, flush=True)
    if direct_ok:
        rp = os.path.join(args.dir, "image_move_bench_raw.bin")
        n = Wb // chunk * chunk
        roof["raw_o_direct"] = {"write_gbs": raw_rate(rp, n, threads, chunk, True), "read_gbs": raw_rate(rp, n, threads, chunk, False),
                                "bytes": n, "threads": threads, "chunk_bytes": chunk}
        os.unlink(rp)
        print(f"raw O_DIRECT: {roof['raw_o_direct']}", file=sys.stderr, flush=True)

    rows = {f: [] for f in engines}
    bit_exact = True

    def rate(nbytes, s):
        return nbytes / s / 1e9

    for step in range(args.warmup + args.steps):
        for form, eng in engines.items():        # asleep in the host tier
            row = {}
            for src, dst in MOVES:
                t0 = time.perf_counter()
                eng.move_image(tier[dst])
                move_s = time.perf_counter() - t0
                st = eng.stats()
                tl = eng.timeline()
                S = st["image_store_bytes"]
                io = [r for r in tl if r["kind"] == "file_io"]
                cp = [r for r in tl if r["kind"] == "copies_landed"]
                key = f"{src}_to_{dst}"
                row[key] = dict(move_s=move_s, bytes=S, gbs=rate(S, move_s),
                                file_io_s=(io[0]["t1_ms"] - io[0]["t0_ms"]) * 1e-3 if io else None,
                                io=("o_direct" if io and io[0]["idx"] == 1 else "page_cache") if io else None,
                                copies_s=(cp[0]["t1_ms"] - cp[0]["t0_ms"]) * 1e-3 if cp else None)
                if dst == "host":
                    row[key]["pin_s"] = st["host_store_pin_seconds"]   # the promotion pinned a fresh host store
                if src == "host":
                    eng.host_release()            # a demotion frees the host store (what a caller under DRAM pressure does)
                if src == "local":
                    eng.peer_release()            # ... and an eviction the parking HBM
                eng.wake(None)
                st = eng.stats()
                row[key].update(wake_s=st["wake_seconds"], wake_gbs=rate(st["wake_bytes_restored"], st["wake_seconds"]))
                print(f"step {step} {form} {key}: move {move_s:.3f} s ({row[key]['gbs']:.2f} GB/s), wake {st['wake_seconds']:.3f} s",
                      file=sys.stderr, flush=True)
                bit_exact = bit_exact and eng.digest_all(["weights"]) == digests[form]
                eng.sleep(["weights"], tier=tier[dst])   # back to sleep where the image was moved to (not timed)
            # a plain host-tier wake of the same image (slept there by the last line), in the same alternation
            eng.wake(None)
            st = eng.stats()
            row["host_wake"] = dict(wake_s=st["wake_seconds"], wake_gbs=rate(st["wake_bytes_restored"], st["wake_seconds"]))
            bit_exact = bit_exact and eng.digest_all(["weights"]) == digests[form]
            eng.sleep(["weights"], tier=L.FMA_TIER_HOST)
            if step >= args.warmup:
                rows[form].append(row)
    for form, eng in engines.items():
        eng.wake(None)
        bit_exact = bit_exact and eng.digest_all(["weights"]) == digests[form]
        eng.file_store(None)
        if os.path.exists(paths[form]):
            os.unlink(paths[form])
        eng.close()

    def med(form, key, field):
        return statistics.median(r[key][field] for r in rows[form])

    keys = [f"{a}_to_{b}" for a, b in MOVES]
    summary = {f: {k: {fld: med(f, k, fld) for fld in ("move_s", "gbs", "wake_s", "wake_gbs")} for k in keys} for f in rows}
    for f in rows:
        summary[f]["host_wake"] = {fld: med(f, "host_wake", fld) for fld in ("wake_s", "wake_gbs")}
    raw = roof.get("raw_o_direct")
    pin = roof["pinned"]
    roofline = {"host_to_file": raw["write_gbs"] if raw else None, "local_to_file": raw["write_gbs"] if raw else None,
                "file_to_host": raw["read_gbs"] if raw else None, "file_to_local": raw["read_gbs"] if raw else None,
                "host_to_local": pin["h2d_gbs"], "local_to_host": pin["d2h_gbs"]}
    out = {
        "metric": "image_move_gbs_fraction_of_roofline", "workload": args.workload, "kv_gib": args.kv_gib,
        "steps": args.steps, "warmup": args.warmup, "dir": os.path.abspath(args.dir),
        "io_mode": "o_direct" if direct_ok else "page_cache", "gpu": gpu_identity(0), "bit_exact": bit_exact, "weight_bytes": Wb,
        "rooflines": roof, "median": summary, "steps_detail": rows,
        "fraction_of_roofline": {f: {k: summary[f][k]["gbs"] / roofline[k] if roofline[k] else None for k in keys} for f in rows},
        "wake_after_promotion_over_host_wake": {f: summary[f]["file_to_host"]["wake_s"] / summary[f]["host_wake"]["wake_s"] for f in rows},
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
