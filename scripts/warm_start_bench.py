"""Warm start from a kept image file on one GPU, beside the two other ways the same weights come back.  Llama-3-8B's weights
(workloads.py), plain (K0 fill, incompressible) and PACKED (bf16 dummy weights), from a file in DIR, O_DIRECT and buffered:

  warm_start  the span from the close of the weights pool to the weights restored and verified: fma_image_adopt_file of the kept
              file, then a wake of the weights with FMA_FLAG_VERIFY (what the allocator shim does with FMA_ADOPT_FILE=1)
  cold_load   the same weight bytes, as a checkpoint would hold them, streamed into the segments by fma_load_file
  host_memfd  adoption of a deposited host memfd (fma_image_adopt of the exported store, then the same wake)

Each is timed --steps times after --warmup runs and the median is kept; every warm start's weights are checked against the K3
digests of the instance that slept.  Before each buffered run the file's pages are dropped from the page cache with
posix_fadvise(DONTNEED) on that file.  The card's name and power limit are read in the same run.

    python scripts/warm_start_bench.py [DIR] [--steps 3] [--warmup 1] [--out profiles/warm_start_h100.json]

Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def drop_cache(path: str) -> None:
    fd = os.open(path, os.O_RDONLY)
    try:
        os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
    finally:
        os.close(fd)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("dir", nargs="?", default=None, help="directory for the image files (default: a temporary one)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workload", default="llama-3-8b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import fma_b200
    from bench import fill_weights, gpu_identity
    from fma_b200 import _lib as L
    from fma_b200 import workloads as W
    from prefetch_bench import filesystem_of

    if not torch.cuda.is_available():
        raise SystemExit("warm_start_bench needs a GPU")
    work = args.dir or tempfile.mkdtemp(prefix="fma-warm-")
    os.makedirs(work, exist_ok=True)
    table = [s for s in W.allocation_table(args.workload, kv_cache_bytes=2 << 30) if s.tag == "weights"]
    Wb = W.weight_bytes(table)

    def loaded(form: str, host_shm: bool = False):
        os.environ.pop("FMA_HOST_STORE_SHM", None)
        if host_shm:
            os.environ["FMA_HOST_STORE_SHM"] = "1"
        eng = fma_b200.Engine(0)
        for s in table:
            eng.alloc(s.bytes, s.tag)
        eng.set_option("pack", 1 if form == "packed" else 0)
        return eng

    def timed(run, reps):
        out = []
        for k in range(args.warmup + reps):
            t = run()
            if k >= args.warmup:
                out.append(t)
        return out

    rows = {}
    bit_exact = True
    plain_file = None
    for form in ("plain", "packed"):
        # the instance that slept: its file-tier image with digests, and its host memfd (what deposit_host hands over)
        a = loaded(form, host_shm=True)
        fill_weights(a, table, 1234, "prng" if form == "plain" else "bf16", torch)
        want = a.digest_all(["weights"])
        path = os.path.join(work, f"warm_{form}.fmaimg")
        a.file_store(path)
        a.sleep(["weights"], tier=L.FMA_TIER_FILE, flags=L.FMA_FLAG_VERIFY)
        stored = a.stats()["image_store_bytes"]
        a.wake(None)
        a.sleep(["weights"], tier=L.FMA_TIER_HOST, flags=L.FMA_FLAG_VERIFY)
        memfd = a.image_export()
        a.close()
        if form == "plain":
            plain_file = path

        b = loaded(form)

        def warm(io):
            nonlocal bit_exact
            if io == "buffered":
                drop_cache(path)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b.image_adopt_file(path, ["weights"])
            b.wake(["weights"], flags=L.FMA_FLAG_VERIFY)
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            bit_exact &= b.digest_all(["weights"]) == want
            return t

        for io in ("direct", "buffered"):
            if io == "buffered":
                os.environ["FMA_FILE_BUFFERED"] = "1"
            else:
                os.environ.pop("FMA_FILE_BUFFERED", None)
            ts = timed(lambda: warm(io), args.steps)
            direct = [r["idx"] for r in b.timeline() if r["kind"] == "file_io"]
            rows[f"warm_start_{form}_{io}"] = {"seconds": statistics.median(ts), "all_seconds": ts, "stored_bytes": stored, "weight_bytes": Wb,
                                               "weight_gbs": Wb / statistics.median(ts) / 1e9, "file_io_o_direct": direct == [1]}
            print(f"{form} {io}: {rows[f'warm_start_{form}_{io}']}", file=sys.stderr, flush=True)
        os.environ.pop("FMA_FILE_BUFFERED", None)

        def host():
            nonlocal bit_exact
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b.image_adopt(memfd, ["weights"])
            b.wake(["weights"], flags=L.FMA_FLAG_VERIFY)
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            bit_exact &= b.digest_all(["weights"]) == want
            return t

        ts = timed(host, args.steps)
        rows[f"host_memfd_{form}"] = {"seconds": statistics.median(ts), "all_seconds": ts, "weight_bytes": Wb, "weight_gbs": Wb / statistics.median(ts) / 1e9}
        print(f"{form} host memfd: {rows[f'host_memfd_{form}']}", file=sys.stderr, flush=True)
        os.close(memfd)
        b.close()

    # the cold load of the same bytes: the plain image file holds every weight segment back to back, as a checkpoint would
    c = loaded("plain")
    spans, off = [], 0
    for i, s in enumerate(c.segments()):
        spans.append((off, s.bytes, s.va))
        off += s.bytes
    for io in ("direct", "buffered"):
        def cold():
            if io == "buffered":
                drop_cache(plain_file)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            c.load_file(plain_file, spans, o_direct=io == "direct")
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        ts = timed(cold, args.steps)
        rows[f"cold_load_{io}"] = {"seconds": statistics.median(ts), "all_seconds": ts, "weight_bytes": Wb, "weight_gbs": Wb / statistics.median(ts) / 1e9}
        print(f"cold {io}: {rows[f'cold_load_{io}']}", file=sys.stderr, flush=True)
    c.close()
    if not args.dir:
        shutil.rmtree(work, ignore_errors=True)

    res = {"bench": "warm_start", "workload": args.workload, "gpu": gpu_identity(0), "filesystem": filesystem_of(work),
           "steps": args.steps, "warmup": args.warmup, "bit_exact": bit_exact, "rows": rows}
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
