"""BASELINE config 4: model swap under one process, Llama-3-8B <-> Mistral-7B on one GPU.
Serial (sleep A, then wake B: what two independent reconciles of the reference do, SURVEY.md §3.4) vs
fma_swap (D2H of A overlapped with H2D of B on opposite PCIe directions)."""
import os, sys, json, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fma_b200
from fma_b200 import workloads as W, _lib as L
A = fma_b200.Engine(0); B = fma_b200.Engine(0)
def load(eng, model, seed):
    t = W.allocation_table(model, kv_cache_bytes=16 << 30)
    for s in t: eng.alloc(s.bytes, s.tag)
    fw = 0
    for i, s in enumerate(t):
        if s.tag == "weights": eng.fill(i, seed, fw); fw += s.bytes // 8
    eng.host_reserve(W.weight_bytes(t))
    return W.weight_bytes(t), eng.digest_all(["weights"])
wa, da = load(A, "llama-3-8b", 1); wb, db = load(B, "mistral-7b", 2)
B.sleep(["weights"])
rows = []
for rep in range(4):
    t0 = time.perf_counter(); A.sleep(["weights"]); t1 = time.perf_counter(); B.wake(None); t2 = time.perf_counter()
    serial_ab = t2 - t0
    t0 = time.perf_counter(); B.sleep(["weights"]); A.wake(None); serial_ba = time.perf_counter() - t0
    t0 = time.perf_counter(); A.swap_out_for(B, ["weights"]); swap_ab = time.perf_counter() - t0
    sa, sb = A.stats(), B.stats()
    t0 = time.perf_counter(); B.swap_out_for(A, ["weights"]); swap_ba = time.perf_counter() - t0
    rows.append(dict(serial_ab=serial_ab, serial_ba=serial_ba, swap_ab=swap_ab, swap_ba=swap_ba,
                     swap_ab_sleepA=sa["sleep_seconds"], swap_ab_wakeB=sb["wake_seconds"],
                     d2h_gbs=wa / sa["sleep_copy_seconds"] / 1e9, h2d_gbs=wb / sb["wake_copy_seconds"] / 1e9))
    print({k: round(v, 4) for k, v in rows[-1].items()}, flush=True)
ok = A.digest_all(["weights"]) == da
B.sleep(["weights"]) if not B.is_sleeping() else None
A.sleep(["weights"]); B.wake(None); ok = ok and B.digest_all(["weights"]) == db
print("bit_exact", ok)
os.makedirs("gpurun_out/swap", exist_ok=True)
json.dump(dict(rows=rows, bit_exact=ok, wa=wa, wb=wb), open("gpurun_out/swap/swap_bench.json", "w"), indent=1)
