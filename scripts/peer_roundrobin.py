"""BASELINE config 5: four sleeping Llama-3-8B models parked in idle GPUs' HBM over NVSwitch, round-robin wake.
One process drives 4 engines (GPUs 0-3); each parks its image on GPU 4-7 (FMA_TIER_PEER: cuMemCreate on the peer +
cuMemMap/SetAccess into the owner, K1/K2 move pages over NVLink).  Reports wake latency and GB/s vs 450 GB/s (H100 NVLink 4, per direction)."""
import os, sys, json, time, threading
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fma_b200
from fma_b200 import workloads as W, _lib as L
import torch
n = torch.cuda.device_count()
half = n // 2
assert half >= 1, "needs >= 2 GPUs"
table = W.allocation_table("llama-3-8b", kv_cache_bytes=16 << 30)
Wb = W.weight_bytes(table)
engs, digs = [], []
for g in range(half):
    e = fma_b200.Engine(g)
    for s in table: e.alloc(s.bytes, s.tag)
    fw = 0
    for i, s in enumerate(table):
        if s.tag == "weights": e.fill(i, 1234 + g, fw); fw += s.bytes // 8
    digs.append(e.digest_all(["weights"]))
    e.peer_reserve(half + g, Wb)
    engs.append(e)
res = {"n_gpus": n, "models": half, "W": Wb, "roundrobin": [], "concurrent": []}
for e in engs: e.sleep(["weights"], tier=L.FMA_TIER_PEER)
for rnd in range(3):
    for g, e in enumerate(engs):
        e.wake(None); st = e.stats()
        res["roundrobin"].append(dict(gpu=g, wake_s=st["wake_seconds"], copy_s=st["wake_copy_seconds"], map_s=st["wake_map_seconds"],
                                      gbs_e2e=Wb / st["wake_seconds"] / 1e9, gbs_dev=Wb / st["wake_copy_seconds"] / 1e9))
        e.sleep(["weights"], tier=L.FMA_TIER_PEER); st = e.stats()
        res["roundrobin"][-1].update(sleep_s=st["sleep_seconds"], sleep_gbs_dev=Wb / st["sleep_copy_seconds"] / 1e9)
for rnd in range(3):
    out = [None] * half
    def w(g):
        engs[g].wake(None); out[g] = engs[g].stats()["wake_seconds"]
    ths = [threading.Thread(target=w, args=(g,)) for g in range(half)]
    t0 = time.perf_counter(); [t.start() for t in ths]; [t.join() for t in ths]; wall = time.perf_counter() - t0
    res["concurrent"].append(dict(wall_s=wall, per_engine=out, aggregate_gbs=half * Wb / wall / 1e9))
    for e in engs: e.sleep(["weights"], tier=L.FMA_TIER_PEER)
for e in engs: e.wake(None)
res["bit_exact"] = all(e.digest_all(["weights"]) == d for e, d in zip(engs, digs))
rr = res["roundrobin"][half:]
print("round-robin wake: mean %.4f s, %.0f GB/s e2e (%.2f of 900), device-timed %.0f GB/s; sleep gather %.0f GB/s" % (
    sum(r["wake_s"] for r in rr) / len(rr), sum(r["gbs_e2e"] for r in rr) / len(rr), sum(r["gbs_e2e"] for r in rr) / len(rr) / 900,
    sum(r["gbs_dev"] for r in rr) / len(rr), sum(r["sleep_gbs_dev"] for r in rr) / len(rr)))
print("concurrent wake of %d models:" % half, [(round(c["wall_s"], 4), round(c["aggregate_gbs"])) for c in res["concurrent"]], "bit_exact", res["bit_exact"])
os.makedirs("gpurun_out/peer", exist_ok=True); json.dump(res, open("gpurun_out/peer/peer_roundrobin.json", "w"), indent=1)
