"""Generates tests/golden/vllm_cumem_roundtrip.json on a GPU machine with vLLM by running the reference data path itself:
vLLM's unmodified CuMemAllocator (vllm:device_allocator/cumem.py:177-249, the code POST /sleep and /wake_up
reach through inference_server/launcher/launcher.py) over the tensors of the `tiny-llama-test` model (torch's caching allocator turns them into segments).

    python tests/golden/make_vllm_cumem_golden.py [OUT_DIR]    # writes OUT_DIR/vllm_cumem_roundtrip.json (default: tests/golden)

Every weight tensor is loaded with the oracle's splitmix64 stream (seed 1234, word index continuing across
tensors), sent through sleep(offload_tags=("weights",)) -> wake_up(), read back, and hashed with SHA-256
(independent of the oracle's own digest).  kv_cache tensors are filled with 0x5A and recorded as
"not restored".  The fixture therefore pins: (1) the reference round trip is the identity on weight bytes at
the same device address, (2) the reference's segment sizes (alignedSize) for this table, (3) what happens to
non-offloaded tags."""
import hashlib, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import fma_b200  # table shapes only
from fma_b200 import workloads as W
from oracle import oracle as O
from vllm.device_allocator.cumem import CuMemAllocator
import vllm

SEED = 1234
MODEL = "tiny-llama-test"
tensors = W.model_tensors(MODEL)                     # (name, nbytes) in vLLM construction order
kv_specs = [("kv.0", 16 << 20), ("kv.1", 16 << 20)]
alloc = CuMemAllocator.get_instance()
weights, kvs = [], []
with alloc.use_memory_pool(tag="weights"):
    for name, nbytes in tensors:
        weights.append(torch.empty(nbytes, dtype=torch.uint8, device="cuda"))
with alloc.use_memory_pool(tag="kv_cache"):
    for name, nbytes in kv_specs:
        kvs.append(torch.full((nbytes,), 0x5A, dtype=torch.uint8, device="cuda"))
first = 0
firsts = []
for t in weights:
    host = torch.from_numpy(O.fill(t.numel(), SEED, first).copy())
    t.copy_(host); firsts.append(first); first += t.numel() // 8
torch.cuda.synchronize()
ptrs_before = [t.data_ptr() for t in weights + kvs]
seg_sizes = sorted((d.handle[2], d.handle[1], d.tag) for d in alloc.pointer_to_data.values())
t0 = time.perf_counter(); alloc.sleep(offload_tags=("weights",)); torch.cuda.synchronize(); t1 = time.perf_counter()
alloc.wake_up(); torch.cuda.synchronize(); t2 = time.perf_counter()
out = {"generator": "tests/golden/make_vllm_cumem_golden.py", "vllm_version": vllm.__version__, "torch": torch.__version__,
       "gpu": torch.cuda.get_device_name(0), "model": MODEL, "kv_specs": kv_specs, "seed": SEED,
       "same_device_addresses": [t.data_ptr() for t in weights + kvs] == ptrs_before,
       "reference_segments": [{"bytes": b, "tag": tag} for _, b, tag in seg_sizes],
       "sleep_s": t1 - t0, "wake_s": t2 - t1, "weights": [], "kv_cache": []}
for (name, nbytes), t, fw in zip(tensors, weights, firsts):
    b = t.cpu().numpy()
    out["weights"].append({"name": name, "bytes": int(b.size), "first_word": fw,
                           "sha256": hashlib.sha256(b.tobytes()).hexdigest(), "oracle_digest": O.digest(b, fw)})
for t in kvs:
    b = t.cpu().numpy()
    out["kv_cache"].append({"bytes": int(b.size), "restored": bool((b == 0x5A).all())})
out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
os.makedirs(out_dir, exist_ok=True)
p = os.path.join(out_dir, "vllm_cumem_roundtrip.json")
json.dump(out, open(p, "w"), indent=1)
print("wrote", p, "same_va", out["same_device_addresses"], "n_weights", len(weights), "segments", len(seg_sizes),
      "kv restored", [k["restored"] for k in out["kv_cache"]])
