"""Probe (a few seconds on one GPU): does VA alignment / handle size change what a run costs to map?
Prints cuMemGetAllocationGranularity (minimum vs recommended) and times cuMemCreate / Map / SetAccess / Unmap of one
16 GiB run for VA reservations aligned to 2 MiB, 32 MiB, 512 MiB and 1 GiB (the engine's arenas are aligned to the
minimum granularity today, csrc/fma_engine.cu arena_take).  Output: gpurun_out/vmm/gran_probe.json."""
import json
import os
import time

from cuda.bindings import driver as cu


def ck(r):
    err, rest = (r[0], r[1:]) if isinstance(r, tuple) else (r, ())
    if err != cu.CUresult.CUDA_SUCCESS:
        raise RuntimeError(str(err))
    return rest[0] if len(rest) == 1 else rest


ck(cu.cuInit(0)); dev = ck(cu.cuDeviceGet(0)); ctx = ck(cu.cuDevicePrimaryCtxRetain(dev)); ck(cu.cuCtxSetCurrent(ctx))
prop = cu.CUmemAllocationProp(); prop.type = cu.CUmemAllocationType.CU_MEM_ALLOCATION_TYPE_PINNED
prop.location.type = cu.CUmemLocationType.CU_MEM_LOCATION_TYPE_DEVICE; prop.location.id = 0
acc = cu.CUmemAccessDesc(); acc.location.type = cu.CUmemLocationType.CU_MEM_LOCATION_TYPE_DEVICE; acc.location.id = 0
acc.flags = cu.CUmemAccess_flags.CU_MEM_ACCESS_FLAGS_PROT_READWRITE
MiB = 1 << 20
gmin = ck(cu.cuMemGetAllocationGranularity(prop, cu.CUmemAllocationGranularity_flags.CU_MEM_ALLOC_GRANULARITY_MINIMUM))
grec = ck(cu.cuMemGetAllocationGranularity(prop, cu.CUmemAllocationGranularity_flags.CU_MEM_ALLOC_GRANULARITY_RECOMMENDED))
res = {"granularity_min": int(gmin), "granularity_recommended": int(grec), "runs": []}
size = 16 * 1024 * MiB
for align in (2 * MiB, 32 * MiB, 512 * MiB, 1024 * MiB):
    va = ck(cu.cuMemAddressReserve(size, align, 0, 0))
    rows = []
    for rep in range(4):
        t0 = time.perf_counter(); h = ck(cu.cuMemCreate(size, prop, 0)); t1 = time.perf_counter()
        ck(cu.cuMemMap(va, size, 0, h, 0)); t2 = time.perf_counter()
        ck(cu.cuMemSetAccess(va, size, [acc], 1)); t3 = time.perf_counter()
        ck(cu.cuMemsetD8(va, 0x5A, size)); ck(cu.cuCtxSynchronize()); t4 = time.perf_counter()
        ck(cu.cuMemUnmap(va, size)); t5 = time.perf_counter()
        ck(cu.cuMemRelease(h)); t6 = time.perf_counter()
        rows.append({"create_ms": round((t1 - t0) * 1e3, 3), "map_ms": round((t2 - t1) * 1e3, 3), "access_ms": round((t3 - t2) * 1e3, 3),
                     "memset_16gib_ms": round((t4 - t3) * 1e3, 3), "unmap_ms": round((t5 - t4) * 1e3, 3), "release_ms": round((t6 - t5) * 1e3, 3)})
    ck(cu.cuMemAddressFree(va, size))
    res["runs"].append({"va_align_mib": align // MiB, "va": hex(int(va)), "reps": rows})
    print(align // MiB, "MiB aligned:", rows[-1], flush=True)
os.makedirs("gpurun_out/vmm", exist_ok=True)
json.dump(res, open("gpurun_out/vmm/gran_probe.json", "w"), indent=1)
print(json.dumps({k: res[k] for k in ("granularity_min", "granularity_recommended")}))
