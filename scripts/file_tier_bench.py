"""File tier on one GPU: Llama-3-8B's table (32 GiB of kv_cache by default) slept to a file in DIR and woken from it, plain (K0
fill, incompressible) and PACKED (bf16 dummy weights), alternating over the timed steps; beside it, DIR's own sequential O_DIRECT
write and read rate with the engine's thread count, chunk size and file size, measured in the same run: the tier's roofline.

    python scripts/file_tier_bench.py DIR [--steps 5] [--warmup 1] [--kv-gib 32] [--out profiles/file_tier_h100.json]

Prints one JSON line (and writes it to --out).  Caches are never dropped (that needs root): if DIR refuses O_DIRECT every number
is a page-cache number and the line says so ("io_mode": "page_cache")."""
from __future__ import annotations

import argparse
import json
import mmap
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def raw_rate(path: str, nbytes: int, threads: int, chunk: int, write: bool) -> float:
    """GB/s of `threads` threads moving `nbytes` of `path` in `chunk`-sized O_DIRECT pwrite / pread calls, in file order."""
    fd = os.open(path, (os.O_WRONLY | os.O_CREAT if write else os.O_RDONLY) | os.O_DIRECT, 0o644)
    n_chunks = nbytes // chunk
    nxt = [0]
    lock = threading.Lock()

    def worker():
        buf = mmap.mmap(-1, chunk)          # page aligned, as O_DIRECT wants
        if write:
            buf.write(os.urandom(1 << 20) * (chunk >> 20))
        mv = memoryview(buf)
        while True:
            with lock:
                k = nxt[0]
                nxt[0] += 1
            if k >= n_chunks:
                break
            if write:
                os.pwrite(fd, mv, k * chunk)
            else:
                os.preadv(fd, [mv], k * chunk)
        mv.release()
        buf.close()

    t0 = time.perf_counter()
    th = [threading.Thread(target=worker) for _ in range(threads)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if write:
        os.fdatasync(fd)
    dt = time.perf_counter() - t0
    os.close(fd)
    return n_chunks * chunk / dt / 1e9


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--kv-gib", type=float, default=32.0)
    ap.add_argument("--workload", default="llama-3-8b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import fma_b200
    from bench import fill_weights, gpu_identity
    from fma_b200 import _lib as L
    from fma_b200 import workloads as W

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

    engines, tables, digests = {}, {}, {}
    for form in ("plain", "packed"):
        eng = fma_b200.Engine(0)
        table = W.allocation_table(args.workload, kv_cache_bytes=int(args.kv_gib * (1 << 30)))
        for s in table:
            eng.alloc(s.bytes, s.tag)
        fill_weights(eng, table, 1234, "prng" if form == "plain" else "bf16", torch)
        eng.set_option("pack", 1 if form == "packed" else 0)
        eng.file_store(os.path.join(args.dir, f"file_tier_bench_{form}.fmaimg"))
        engines[form], tables[form] = eng, table
        digests[form] = eng.digest_all(["weights"])
        eng.sleep(["weights"], tier=L.FMA_TIER_FILE)   # one model on the GPU at a time; this sleep is not timed
    Wb = W.weight_bytes(tables["plain"])
    threads, chunk = 12, 16 << 20               # the engine's load_threads / load_chunk_bytes defaults

    roof = {}
    if direct_ok:
        rp = os.path.join(args.dir, "file_tier_bench_raw.bin")
        n = Wb // chunk * chunk
        roof = {"write_gbs": raw_rate(rp, n, threads, chunk, True), "read_gbs": raw_rate(rp, n, threads, chunk, False),
                "bytes": n, "threads": threads, "chunk_bytes": chunk}
        os.unlink(rp)

    rows = {"plain": [], "packed": []}
    bit_exact = True
    for step in range(args.warmup + args.steps):
        for form in ("plain", "packed"):
            eng = engines[form]
            eng.wake(None)                          # from the file: the set-up sleep's image, or the previous step's
            if step > 0:
                st = eng.stats()
                tl = eng.timeline()
                io = [r["idx"] for r in tl if r["kind"] == "file_io"]
                if step > args.warmup:
                    rows[form][-1].update(wake_s=st["wake_seconds"], wake_file_gbs=st["image_store_bytes"] / st["wake_seconds"] / 1e9,
                                          wake_weight_gbs=st["wake_bytes_restored"] / st["wake_seconds"] / 1e9,
                                          wake_io=("o_direct" if io and io[0] == 1 else "page_cache"))
            bit_exact = bit_exact and eng.digest_all(["weights"]) == digests[form]
            eng.sleep(["weights"], tier=L.FMA_TIER_FILE)
            st = eng.stats()
            io = [r["idx"] for r in eng.timeline() if r["kind"] == "file_io"]
            if step >= args.warmup:
                rows[form].append(dict(sleep_s=st["sleep_seconds"], file_bytes=st["image_store_bytes"], weight_bytes=st["sleep_bytes_offloaded"],
                                       sleep_file_gbs=st["image_store_bytes"] / st["sleep_seconds"] / 1e9,
                                       sleep_weight_gbs=st["sleep_bytes_offloaded"] / st["sleep_seconds"] / 1e9,
                                       sleep_io=("o_direct" if io and io[0] == 1 else "page_cache"),
                                       host_store_bytes=st["host_store_bytes"], io_buffer_bytes=st["io_buffer_bytes"]))
    for form in ("plain", "packed"):                # the last sleep's wake, and the last check
        eng = engines[form]
        eng.wake(None)
        st = eng.stats()
        rows[form][-1].update(wake_s=st["wake_seconds"], wake_file_gbs=st["image_store_bytes"] / st["wake_seconds"] / 1e9,
                              wake_weight_gbs=st["wake_bytes_restored"] / st["wake_seconds"] / 1e9,
                              wake_io=("o_direct" if any(r["kind"] == "file_io" and r["idx"] == 1 for r in eng.timeline()) else "page_cache"))
        bit_exact = bit_exact and eng.digest_all(["weights"]) == digests[form]
        eng.file_store(None)
        os.unlink(os.path.join(args.dir, f"file_tier_bench_{form}.fmaimg"))
        eng.close()

    def med(form, key):
        return statistics.median(r[key] for r in rows[form])

    summary = {f: {k: med(f, k) for k in ("sleep_s", "wake_s", "sleep_file_gbs", "wake_file_gbs", "sleep_weight_gbs", "wake_weight_gbs")}
               for f in rows}
    out = {
        "metric": "file_tier_wake_file_gbs_fraction_of_raw_read", "workload": args.workload, "kv_gib": args.kv_gib,
        "steps": args.steps, "warmup": args.warmup, "dir": os.path.abspath(args.dir),
        "io_mode": "o_direct" if direct_ok and all(r["wake_io"] == "o_direct" for f in rows for r in rows[f]) else "page_cache",
        "gpu": gpu_identity(0), "bit_exact": bit_exact, "weight_bytes": Wb, "raw_o_direct": roof, "median": summary, "steps_detail": rows,
        "wake_fraction_of_raw_read": {f: summary[f]["wake_file_gbs"] / roof["read_gbs"] for f in rows} if roof else None,
        "sleep_fraction_of_raw_write": {f: summary[f]["sleep_file_gbs"] / roof["write_gbs"] for f in rows} if roof else None,
        "packed_wake_time_over_plain": summary["packed"]["wake_s"] / summary["plain"]["wake_s"],
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
