// fma_engine.cu — host side of the H100 sleep/wake weight-movement engine (C-ABI in
// include/fma_engine.h).  No kernels live here; see fma_kernels.cu.
//
// What it replaces in the reference's hot path (SURVEY.md §8a):
//   a1 CuMemAllocator.sleep      vllm:device_allocator/cumem.py:177-225   -> fma_sleep
//   a2 CuMemAllocator.wake_up    vllm:device_allocator/cumem.py:227-249   -> fma_wake
//   a3 pointer_to_data registry  cumem.py:47-55,131,140-175               -> Engine::segs
//   a5 my_malloc/my_free/create_and_map/unmap_and_release (cumem_allocator.abi3.so, T3)
//   a6 blocking cudaMemcpy       cuda_wrapper.py:168-173                  -> multi-stream async copy engines / K1,K2
//
// Design (H100-first, not a port):
//   * one Engine per GPU / process (rank); segments are CUDA-VMM ranges whose VA reservation
//     outlives unmap so every tensor keeps its device address across sleep -> wake;
//   * a sleeping model is a PACKED IMAGE: its offloaded segments concatenated page by page
//     (2 MiB VMM pages) in allocation order, held in one pre-pinned NUMA-local host store,
//     or a parking buffer in a peer GPU's HBM (NVLink tier);
//   * wake overlaps three things the reference serialises: cuMemCreate/Map/SetAccess of the
//     next segments (mapper thread), H2D DMA on several copy-engine streams, and (staged /
//     kernel modes) the K2 page scatter;
//   * the driver API is resolved at run time (cudaGetDriverEntryPoint) so the library loads
//     on a box without libcuda — and then refuses to do anything (FMA_ENODRIVER).
#include "fma_internal.h"

namespace fma_impl {

// ------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------
thread_local char tl_err[512] = "";

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(tl_err, sizeof(tl_err), fmt, ap);
    va_end(ap);
    return code;
}

double now_s() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}



// ------------------------------------------------------------------------------------
// driver API, resolved lazily through the (static) runtime: no link-time libcuda dependency
// ------------------------------------------------------------------------------------

Driver g_drv;
static std::once_flag g_drv_once;
char g_drv_err[256] = "";

template <typename F>
static bool resolve(const char* name, F& fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
        snprintf(g_drv_err, sizeof(g_drv_err), "cannot resolve driver symbol %s: %s", name,
                 e != cudaSuccess ? cudaGetErrorString(e) : "not found");
        cudaGetLastError();
        return false;
    }
    fn = reinterpret_cast<F>(p);
    return true;
}

static void load_driver() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        snprintf(g_drv_err, sizeof(g_drv_err), "no usable CUDA driver/device: %s",
                 e != cudaSuccess ? cudaGetErrorString(e) : "0 devices");
        cudaGetLastError();
        return;
    }
    bool ok = resolve("cuGetErrorString", g_drv.GetErrorString) && resolve("cuMemAddressReserve", g_drv.MemAddressReserve) &&
              resolve("cuMemAddressFree", g_drv.MemAddressFree) && resolve("cuMemCreate", g_drv.MemCreate) &&
              resolve("cuMemRelease", g_drv.MemRelease) && resolve("cuMemMap", g_drv.MemMap) &&
              resolve("cuMemUnmap", g_drv.MemUnmap) && resolve("cuMemSetAccess", g_drv.MemSetAccess) &&
              resolve("cuMemGetAllocationGranularity", g_drv.MemGetAllocationGranularity) &&
              resolve("cuMemExportToShareableHandle", g_drv.MemExportToShareableHandle) &&
              resolve("cuMemImportFromShareableHandle", g_drv.MemImportFromShareableHandle);
    g_drv.ok = ok;
}

bool driver_ready() {
    std::call_once(g_drv_once, load_driver);
    return g_drv.ok;
}

const char* cu_err(CUresult r) {
    const char* s = nullptr;
    if (g_drv.GetErrorString && g_drv.GetErrorString(r, &s) == CUDA_SUCCESS && s) return s;
    return "unknown CUresult";
}





size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

static fma_engine_t* g_current = nullptr;
static std::mutex g_current_mu;


// ------------------------------------------------------------------------------------
// VMM primitives (replace cumem_allocator's create_and_map / unmap_and_release)
// ------------------------------------------------------------------------------------
CUmemAllocationProp device_prop(int device) {
    CUmemAllocationProp prop;
    memset(&prop, 0, sizeof(prop));
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device;
    return prop;
}

// Maps `h` at `va` and grants each of `devices` read/write access (once per device).  On failure nothing stays mapped, *call
// names the call that failed, and the caller still owns `h`.
static CUresult map_with_access(CUdeviceptr va, size_t bytes, CUmemGenericAllocationHandle h, std::initializer_list<int> devices, const char** call) {
    CUmemAccessDesc acc[2];
    size_t n = 0;
    for (int d : devices) {
        if (n == 2 || (n == 1 && acc[0].location.id == d)) continue;
        memset(&acc[n], 0, sizeof(acc[n]));
        acc[n].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        acc[n].location.id = d;
        acc[n++].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    }
    *call = "cuMemMap";
    CUresult r = g_drv.MemMap(va, bytes, 0, h, 0);
    if (r != CUDA_SUCCESS) return r;
    *call = "cuMemSetAccess";
    r = g_drv.MemSetAccess(va, bytes, acc, n);
    if (r != CUDA_SUCCESS) g_drv.MemUnmap(va, bytes);
    return r;
}

// create + map + set access, then drop the handle: the physical memory stays alive until cuMemUnmap
// (scripts/vmm_span_probe.py checks this), which makes teardown a single driver call per range.
int vmm_create_and_map(int device, CUdeviceptr va, size_t bytes) {
    CUmemAllocationProp prop = device_prop(device);
    CUmemGenericAllocationHandle h = 0;
    DRV(g_drv.MemCreate(&h, bytes, &prop, 0));
    const char* call = nullptr;
    const CUresult r = map_with_access(va, bytes, h, {device}, &call);
    if (r != CUDA_SUCCESS) {
        g_drv.MemRelease(h);
        return fail(FMA_ECUDA, "%s failed: %s", call, cu_err(r));
    }
    DRV(g_drv.MemRelease(h));
    return FMA_OK;
}

int vmm_create(int device, size_t bytes, bool exportable, CUmemGenericAllocationHandle* out) {
    CUmemAllocationProp prop = device_prop(device);
    if (exportable) prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    const CUresult r = g_drv.MemCreate(out, bytes, &prop, 0);
    if (r != CUDA_SUCCESS)
        return fail(r == CUDA_ERROR_OUT_OF_MEMORY ? FMA_ENOMEM : FMA_ECUDA, "cuMemCreate(%zu bytes on device %d) failed: %s", bytes, device, cu_err(r));
    return FMA_OK;
}

int vmm_import(int fd, CUmemGenericAllocationHandle* out) {
    const CUresult r = g_drv.MemImportFromShareableHandle(out, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
    if (r != CUDA_SUCCESS)
        return fail(r == CUDA_ERROR_OUT_OF_MEMORY ? FMA_ENOMEM : FMA_ECUDA, "cuMemImportFromShareableHandle(fd %d) failed: %s", fd, cu_err(r));
    return FMA_OK;
}

int vmm_buffer_map(CUmemGenericAllocationHandle h, size_t bytes, std::initializer_list<int> access_devices, const char* what, VmmBuffer* out) {
    VmmBuffer b;
    b.bytes = bytes;
    b.handle = h;
    const char* call = "cuMemAddressReserve";
    CUresult r = g_drv.MemAddressReserve(&b.va, bytes, FMA_PAGE_BYTES, 0, 0);
    if (r == CUDA_SUCCESS) {
        r = map_with_access(b.va, bytes, h, access_devices, &call);
        if (r != CUDA_SUCCESS) g_drv.MemAddressFree(b.va, bytes);
    }
    if (r != CUDA_SUCCESS) {
        g_drv.MemRelease(h);
        return fail(FMA_ECUDA, "%s(%s) failed: %s", call, what, cu_err(r));
    }
    *out = b;
    return FMA_OK;
}

void vmm_buffer_free(VmmBuffer& b) {
    if (!b.va) return;
    g_drv.MemUnmap(b.va, b.bytes);
    g_drv.MemAddressFree(b.va, b.bytes);
    g_drv.MemRelease(b.handle);
    b = VmmBuffer{};
}

// ---- arenas ----------------------------------------------------------------------------------------
int arena_take(fma_engine_t* e, int tag, size_t bytes, int* out_arena, CUdeviceptr* out_va) {
    for (size_t i = 0; i < e->arenas.size(); ++i) {
        Arena& a = e->arenas[i];
        size_t off = 0;
        if (a.tag != tag || !fma_layout::arena_take(a, bytes, &off)) continue;  // first fit among holes, else bump
        *out_arena = (int)i;
        *out_va = a.base + off;
        return FMA_OK;
    }
    Arena a;
    a.tag = tag;
    size_t want = std::max<size_t>((size_t)std::max(env_int("FMA_ARENA_GIB", 256), 1) << 30, round_up(bytes, e->gran));
    CUresult r = CUDA_ERROR_OUT_OF_MEMORY;
    while (true) {  // VA is plentiful, but shrink gracefully if a huge reservation is refused
        CUdeviceptr base = 0;
        r = g_drv.MemAddressReserve(&base, want, e->gran, 0, 0);
        a.base = (uint64_t)base;
        if (r == CUDA_SUCCESS || want <= round_up(bytes, e->gran)) break;
        want = std::max(want / 2, round_up(bytes, e->gran));
    }
    if (r != CUDA_SUCCESS) return fail(FMA_ENOMEM, "cuMemAddressReserve(%zu) failed: %s", want, cu_err(r));
    a.cap = want;
    a.top = bytes;
    e->arenas.push_back(a);
    *out_arena = (int)e->arenas.size() - 1;
    *out_va = a.base;
    return FMA_OK;
}

// Unmap one unit (or, for `span_bytes` > unit.bytes, a VA-contiguous group of units in one driver call) and forget it.
// Caller has made sure nothing on the device still touches the range.
int unmap_units(fma_engine_t* e, CUdeviceptr va, size_t span_bytes) {
    DRV(g_drv.MemUnmap(va, span_bytes));
    forget_units(e, va, span_bytes);
    return FMA_OK;
}

// The ring's fields once its memory is gone (freed, or unmapped with the unit that carried it).
static void detach_ring(fma_engine_t* e) {
    e->ring_attached = false;
    e->ring_unit_va = 0;
    for (int i = 0; i < kMaxRing; ++i) e->ring[i] = nullptr;
    e->n_ring = 0;
    e->ring_slot_bytes = 0;
}

void forget_units(fma_engine_t* e, CUdeviceptr va, size_t bytes) {
    auto it = e->units.lower_bound(va);
    while (it != e->units.end() && it->first < va + bytes) {
        Arena& a = e->arenas[it->second.arena];
        for (auto& z : it->second.zombies) arena_give_back(a, z.first - a.base, z.second);
        it = e->units.erase(it);
    }
    if (e->ring_attached && e->ring_unit_va >= va && e->ring_unit_va < va + bytes) detach_ring(e);  // the ring went with its unit
}

// ------------------------------------------------------------------------------------
// engine resources
// ------------------------------------------------------------------------------------
int ensure_streams(fma_engine_t* e) {
    if (e->ks) return FMA_OK;
    int n = e->cfg.copy_streams > 0 ? e->cfg.copy_streams : 4;
    n = std::min(n, kMaxStreams);
    for (int i = 0; i < kMaxStreams; ++i) {  // all created up front; n_cs selects how many are used
        RT(cudaStreamCreateWithFlags(&e->cs[i], cudaStreamNonBlocking));
        RT(cudaEventCreateWithFlags(&e->ev_cs[i], cudaEventDisableTiming));
    }
    e->n_cs = n;
    RT(cudaStreamCreateWithFlags(&e->ks, cudaStreamNonBlocking));
    RT(cudaEventCreate(&e->ev_start));
    RT(cudaEventCreate(&e->ev_end));
    return FMA_OK;
}

int ensure_tables(fma_engine_t* e, size_t n_pages) {
    if (n_pages <= e->d_tab_cap) return FMA_OK;
    size_t cap = std::max<size_t>(round_up(n_pages, 4096), 16384);
    if (e->d_tab) cudaFree(e->d_tab);
    if (e->h_tab) cudaFreeHost(e->h_tab);
    e->d_tab = nullptr;
    e->h_tab = nullptr;
    e->d_tab_cap = 0;
    RT(cudaMalloc(&e->d_tab, 2 * cap * sizeof(uint64_t)));       // [src table | dst table]
    RT(cudaHostAlloc(&e->h_tab, 2 * cap * sizeof(uint64_t), cudaHostAllocDefault));
    e->d_tab_cap = cap;
    return FMA_OK;
}

int ensure_desc(fma_engine_t* e, size_t n_pages) {
    if (n_pages <= e->desc_cap) return FMA_OK;
    size_t cap = std::max<size_t>(round_up(n_pages, 4096), 16384);
    if (e->d_desc) cudaFree(e->d_desc);
    if (e->h_desc) cudaFreeHost(e->h_desc);
    if (e->d_dig) cudaFree(e->d_dig);
    if (e->h_dig) cudaFreeHost(e->h_dig);
    e->d_desc = nullptr; e->h_desc = nullptr; e->d_dig = nullptr; e->h_dig = nullptr;
    e->desc_cap = 0;
    RT(cudaMalloc(&e->d_desc, cap * sizeof(fma_k_page_desc)));
    RT(cudaHostAlloc(&e->h_desc, cap * sizeof(fma_k_page_desc), cudaHostAllocDefault));
    RT(cudaMalloc(&e->d_dig, cap * sizeof(uint64_t)));
    RT(cudaHostAlloc(&e->h_dig, cap * sizeof(uint64_t), cudaHostAllocDefault));
    e->desc_cap = cap;
    return FMA_OK;
}

int ensure_pack_bufs(fma_engine_t* e, size_t n_pages) {
    if (n_pages <= e->pdesc_cap) return FMA_OK;
    size_t cap = std::max<size_t>(round_up(n_pages, 4096), 16384);
    if (e->d_pdesc) cudaFree(e->d_pdesc);
    if (e->h_pdesc) cudaFreeHost(e->h_pdesc);
    if (e->d_psize) cudaFree(e->d_psize);
    if (e->h_psize) cudaFreeHost(e->h_psize);
    e->d_pdesc = nullptr; e->h_pdesc = nullptr; e->d_psize = nullptr; e->h_psize = nullptr;
    e->pdesc_cap = 0;
    RT(cudaMalloc(&e->d_pdesc, cap * sizeof(fma_k_pack_desc)));
    RT(cudaHostAlloc(&e->h_pdesc, cap * sizeof(fma_k_pack_desc), cudaHostAllocDefault));
    RT(cudaMalloc(&e->d_psize, (cap + 1) * sizeof(uint32_t)));
    RT(cudaHostAlloc(&e->h_psize, (cap + 1) * sizeof(uint32_t), cudaHostAllocDefault));
    e->pdesc_cap = cap;
    return FMA_OK;
}

// DMA chunk for DIRECT (round-robin over copy streams) and ring-slot size for STAGED.  H2D over PCIe Gen5 saturates
// well below 32 MiB per copy; a K1/K2 launch issued while a copy engine is busy pays a fixed launch latency of tens of
// microseconds, which large (512 MiB) ring slots keep a small fraction of each launch (scripts/staged_sweep.py,
// scripts/k_contention.py measure both).
size_t direct_chunk(const fma_engine_t* e) {
    return e->cfg.chunk_bytes ? round_up((size_t)e->cfg.chunk_bytes, FMA_PAGE_BYTES) : ((size_t)32 << 20);
}
size_t staged_slot(const fma_engine_t* e) {
    return e->cfg.chunk_bytes ? round_up((size_t)e->cfg.chunk_bytes, FMA_PAGE_BYTES) : ((size_t)512 << 20);
}

void release_ring(fma_engine_t* e) {
    if (e->n_ring && e->ring[0] && !e->ring_attached) cudaFree(e->ring[0]);  // one allocation backs every slot
    detach_ring(e);                     // an attached ring goes away with its unit's cuMemUnmap
    cudaGetLastError();
}

// The HBM staging ring lives from the start of a wake to the end of the next sleep: a serving model keeps it
// (1 GiB of 80 GB) so that /sleep needs no allocation, a SLEEPING model does not hold it (FMA_RING_PERSIST=1 keeps
// it, trading 1 GiB of a sleeper's HBM for one driver call less at wake).  It is freed at the END of sleep,
// synchronously: on these shared hosts a cudaFree of 1 GiB takes anywhere from 0.8 ms to 300 ms (driver stalls), which
// must never sit inside the wake latency — and freeing it from a background thread was measured to block the next
// wake's first driver call instead.  ONE cudaMalloc backs all slots: every driver call at the start of a wake is
// on the critical path and is serialised with the other ranks' calls.  `image_bytes` caps the slot size.
size_t ring_slot_for(const fma_engine_t* e, size_t image_bytes) {
    return std::min(staged_slot(e), round_up(std::max<size_t>(image_bytes, 1), FMA_PAGE_BYTES));
}
int ring_slots_for(const fma_engine_t* e) { return e->cfg.ring_slots > 0 ? std::min(e->cfg.ring_slots, kMaxRing) : 2; }

int ensure_ring_events(fma_engine_t* e, int n) {
    for (int i = 0; i < n; ++i) {
        if (!e->ev_ring_full[i]) RT(cudaEventCreateWithFlags(&e->ev_ring_full[i], cudaEventDisableTiming));
        if (!e->ev_ring_free[i]) RT(cudaEventCreateWithFlags(&e->ev_ring_free[i], cudaEventDisableTiming));
    }
    return FMA_OK;
}

// FMA_NO_RING=1 (read at every sleep and wake): behave as if HBM were too full for a staging ring.  Test and A/B knob: it
// reaches the ring-less paths, e.g. K5 decoding a packed image straight from pinned host memory, without filling the GPU.
bool no_ring() { return env_int("FMA_NO_RING", 0) != 0; }

int ensure_ring(fma_engine_t* e, size_t image_bytes) {
    size_t slot = ring_slot_for(e, image_bytes);
    int n = ring_slots_for(e);
    if (e->n_ring == n && e->ring_slot_bytes == slot) return FMA_OK;
    if (e->ring_attached && e->n_ring >= 2 && e->ring_slot_bytes >= FMA_PAGE_BYTES) return FMA_OK;  // keep what the unit carries
    release_ring(e);
    void* base = nullptr;
    cudaError_t r = cudaMalloc(&base, slot * n);
    if (r != cudaSuccess) {
        cudaGetLastError();
        return fail(FMA_ENOMEM, "cannot allocate %d x %zu byte HBM staging ring: %s", n, slot, cudaGetErrorString(r));
    }
    for (int i = 0; i < n; ++i) e->ring[i] = static_cast<char*>(base) + (size_t)i * slot;
    RC(ensure_ring_events(e, n));
    e->n_ring = n;
    e->ring_slot_bytes = slot;
    return FMA_OK;
}

int ensure_event_pool(fma_engine_t* e, size_t n) {
    while (e->ev_pool.size() < n) {
        cudaEvent_t ev;
        RT(cudaEventCreate(&ev));
        e->ev_pool.push_back(ev);
    }
    return FMA_OK;
}

// ------------------------------------------------------------------------------------
// host store: one NUMA-local, pre-pinned arena (replaces per-segment torch.empty(pin_memory=True),
// cumem.py:204-209).  mmap + mbind + parallel first-touch + cudaHostRegister, fallback cudaHostAlloc.
// ------------------------------------------------------------------------------------
int gpu_numa_node(int device) {
    if (const char* fake = getenv("FMA_NUMA_MAP")) {   // "0,1,1" = visible device index -> NUMA node: overrides sysfs (wrong / missing numa_node files; tests)
        int d = 0;
        for (const char* q = fake; *q; ++q) {
            if (*q == ',') { ++d; continue; }
            if (d == device) return atoi(q);
        }
        return -1;
    }
    char bus[64] = "";
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    for (char* p = bus; *p; ++p) *p = (char)tolower(*p);
    char path[160];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

void host_store_free(HostStore& h) {
    if (!h.base) return;
    if (h.registered) {
        cudaHostUnregister(h.base);
        munmap(h.base, h.map_bytes ? h.map_bytes : h.cap);
    } else {
        cudaFreeHost(h.base);
    }
    if (h.fd >= 0) close(h.fd);
    cudaGetLastError();
    h = HostStore{};
}

void invalidate_shadows(fma_engine_t* e) {
    std::lock_guard<std::mutex> lk(e->mu);
    for (Segment& s : e->segs) s.shadow_off = kNoOffset;
    e->shadow_image_bytes = 0;
    e->shadow_store_bytes = 0;
    e->shadow_packed = false;
}

// per-node path counts of the MULTI-PATH configuration ("" = off or all on one node): what a store's striping depends on
static std::string paths_signature(const fma_engine_t* e) {
    std::map<int, int> per_node;
    for (const WakePath& wp : e->paths)
        if (wp.numa_node >= 0 && wp.numa_node < 64) ++per_node[wp.numa_node];
    if (per_node.size() < 2 || e->cfg.numa_bind == 0) return "";
    std::string s;
    for (auto& kv : per_node) s += std::to_string(kv.first) + ":" + std::to_string(kv.second) + ",";
    return s;
}

int host_store_reserve(fma_engine_t* e, size_t bytes) {
    bytes = round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), FMA_PAGE_BYTES);
    if (e->host.base && e->host.cap >= bytes) return FMA_OK;
    if (e->shadow_tier == FMA_TIER_HOST) invalidate_shadows(e);  // a new store starts empty
    host_store_free(e->host);
    const double t0 = now_s();
    HostStore h;
    h.cap = bytes;
    const int want_bind = e->cfg.numa_bind != 0;  // -1 (default) and 1 both bind
    const int node = want_bind ? gpu_numa_node(e->device) : -1;
    const bool use_register = env_int("FMA_HOST_REGISTER", 1) != 0;
    const bool use_shm = env_int("FMA_HOST_STORE_SHM", 0) != 0;
    if (use_register || use_shm) {
        void* p = MAP_FAILED;
        h.map_bytes = bytes;
        if (use_shm) {  // memfd: the image can be handed to another process (fma_image_export)
            h.fd = (int)syscall(SYS_memfd_create, "fma-host-store", 1u /* MFD_CLOEXEC */);
            if (h.fd >= 0 && ftruncate(h.fd, (off_t)(bytes + kImageTail)) == 0) {
                h.map_bytes = bytes + kImageTail;
                p = mmap(nullptr, h.map_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, h.fd, 0);
            }
            if (p == MAP_FAILED && h.fd >= 0) {
                close(h.fd);
                h.fd = -1;
                h.map_bytes = bytes;
            }
        }
        if (p == MAP_FAILED) p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (p != MAP_FAILED) {
            madvise(p, bytes, MADV_HUGEPAGE);
            // MULTI-PATH wake configured (fma_paths_set): stripe the store over the NUMA nodes of the paths' GPUs in proportion
            // to the number of paths on each node, so that every path can pull chunks that are LOCAL to its GPU's socket.
            // Helpers on the other socket than a store they read from pull it across the socket interconnect and lose about
            // half of their link rate.
            std::map<int, int> per_node;
            if (want_bind)
                for (const WakePath& wp : e->paths)
                    if (wp.numa_node >= 0 && wp.numa_node < 64) ++per_node[wp.numa_node];
            h.placed_for = paths_signature(e);
            if (per_node.size() > 1 && per_node.size() * FMA_PAGE_BYTES <= bytes) {
                size_t total_paths = 0, done_paths = 0, begin = 0;
                for (auto& kv : per_node) total_paths += (size_t)kv.second;
                if (node >= 0 && per_node.count(node)) {  // the engine's own node first: a single-path wake then starts local
                    std::vector<std::pair<int, int>> order{{node, per_node[node]}};
                    for (auto& kv : per_node)
                        if (kv.first != node) order.push_back(kv);
                    for (size_t i = 0; i < order.size(); ++i) {
                        done_paths += (size_t)order[i].second;
                        size_t end = i + 1 == order.size() ? bytes : round_up(bytes / total_paths * done_paths, FMA_PAGE_BYTES);
                        end = std::min(end, bytes);
                        if (end <= begin) continue;
                        unsigned long mask = 1ul << order[i].first;
                        syscall(SYS_mbind, (char*)p + begin, end - begin, 1, &mask, sizeof(mask) * 8, 0);   // best effort (MPOL_PREFERRED)
                        h.ranges.push_back(HostStore::NumaRange{begin, end, order[i].first});
                        begin = end;
                    }
                    h.numa_node = node;
                }
            }
            if (h.ranges.empty() && node >= 0 && node < 64) {
                unsigned long mask = 1ul << node;
                // MPOL_PREFERRED = 1: fall back to the other node rather than fail under pressure
                if (syscall(SYS_mbind, p, bytes, 1, &mask, sizeof(mask) * 8, 0) == 0) h.numa_node = node;
            }
            if (h.ranges.empty()) h.ranges.push_back(HostStore::NumaRange{0, bytes, h.numa_node});
            // parallel first touch so the pages exist before the (serial) pin
            int nt = std::max(1, std::min(env_int("FMA_TOUCH_THREADS", 8), 32));
            std::vector<std::thread> th;
            const size_t per = round_up((bytes + nt - 1) / nt, FMA_PAGE_BYTES);
            for (int t = 0; t < nt; ++t) {
                size_t lo = (size_t)t * per, hi = std::min(bytes, lo + per);
                if (lo >= hi) break;
                th.emplace_back([p, lo, hi] { memset((char*)p + lo, 0, hi - lo); });
            }
            for (auto& t : th) t.join();
            cudaError_t r = cudaHostRegister(p, h.map_bytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
            if (r == cudaSuccess) {
                h.base = p;
                h.registered = true;
            } else {
                cudaGetLastError();
                munmap(p, h.map_bytes);
                if (h.fd >= 0) close(h.fd);
                h.fd = -1;
                h.map_bytes = 0;
            }
        }
    }
    if (!h.base) {
        void* p = nullptr;
        cudaError_t r = cudaHostAlloc(&p, bytes, cudaHostAllocPortable | cudaHostAllocMapped);
        if (r != cudaSuccess) {
            cudaGetLastError();
            return fail(FMA_ENOMEM, "cannot pin %zu bytes of host store: %s", bytes, cudaGetErrorString(r));
        }
        h.base = p;
        h.registered = false;
        h.numa_node = -1;
    }
    void* alias = nullptr;
    if (cudaHostGetDevicePointer(&alias, h.base, 0) == cudaSuccess) h.dev_alias = alias;
    else cudaGetLastError();
    h.pin_seconds = now_s() - t0;
    e->host = h;
    e->st.host_store_bytes = h.cap;
    e->st.host_store_pin_seconds = h.pin_seconds;
    e->st.host_store_numa_node = h.numa_node;
    return FMA_OK;
}

int open_path(WakePath& p, int slots) {
    if (!p.remote) {
        DeviceGuard g(p.device);
        RT(cudaStreamCreateWithFlags(&p.copy, cudaStreamNonBlocking));
        for (int i = 0; i < slots; ++i) RT(cudaEventCreateWithFlags(&p.ev_full[i], cudaEventDisableTiming));
    }
    RT(cudaStreamCreateWithFlags(&p.kern, cudaStreamNonBlocking));
    for (int i = 0; i < slots; ++i) RT(cudaEventCreateWithFlags(&p.ev_free[i], cudaEventDisableTiming));
    RT(cudaEventCreateWithFlags(&p.ev_done, cudaEventDisableTiming));
    return FMA_OK;
}

void close_path(fma_engine_t* e, WakePath& p) {
    if (!p.remote) {
        DeviceGuard g(p.device);
        if (p.copy) cudaStreamSynchronize(p.copy);
        if (p.copy) cudaStreamDestroy(p.copy);
        for (cudaEvent_t ev : p.ev_full)
            if (ev) cudaEventDestroy(ev);
    }
    DeviceGuard g(e->device);
    if (p.kern) cudaStreamSynchronize(p.kern);
    if (p.kern) cudaStreamDestroy(p.kern);
    for (cudaEvent_t ev : p.ev_free)
        if (ev) cudaEventDestroy(ev);
    if (p.ev_done) cudaEventDestroy(p.ev_done);
    vmm_buffer_free(p.staging);
}

void paths_release(fma_engine_t* e) {
    if (e->mbox) {   // tell a helper that may still be pulling to stop, then let go of the mailbox
        e->mbox->abort.store(1);
        munmap(e->mbox, sizeof(PullMailbox));
        e->mbox = nullptr;
    }
    if (e->mbox_fd >= 0) close(e->mbox_fd);
    e->mbox_fd = -1;
    for (WakePath& p : e->paths) close_path(e, p);
    e->paths.clear();
    e->path_slot_bytes = 0;
    e->path_slots = 0;
    cudaGetLastError();
}

int paths_fail(fma_engine_t* e, int rc) {
    char keep[512];
    snprintf(keep, sizeof(keep), "%s", tl_err);
    paths_release(e);
    return fail(rc, "%s", keep);
}

int park_release(fma_engine_t* e) {
    if (!e->park.va) return FMA_OK;
    if (e->shadow_tier == FMA_TIER_PEER || e->shadow_tier == FMA_TIER_LOCAL) invalidate_shadows(e);  // the parking buffer held the kept image
    cudaDeviceSynchronize();
    vmm_buffer_free(e->park);
    return FMA_OK;
}

// One VMM allocation of `bytes` in `device`'s HBM, mapped at a VA of its own with access for the engine's GPU (and for `device`):
// the peer / local parking buffer, and the resident part of a host-tier image.
int park_store_create(fma_engine_t* e, int device, size_t bytes, ParkStore* out) {
    bytes = round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), e->gran);
    int ndev = 0;
    RT(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(FMA_EINVAL, "parking device %d not visible (have %d)", device, ndev);
    if (device != e->device) {
        int can = 0;
        RT(cudaDeviceCanAccessPeer(&can, e->device, device));
        if (!can) return fail(FMA_ECUDA, "device %d cannot access peer %d (no NVLink/P2P path)", e->device, device);
        // make sure the peer's primary context exists (cuMemCreate needs the device initialised)
        DeviceGuard g(device);
        RT(cudaFree(nullptr));
    }
    CUmemGenericAllocationHandle h = 0;
    RC(vmm_create(device, bytes, false, &h));
    RC(vmm_buffer_map(h, bytes, {e->device, device}, "park", out));
    out->device = device;
    return FMA_OK;
}

int park_reserve(fma_engine_t* e, int park_device, size_t bytes) {
    bytes = round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), e->gran);
    if (e->park.va && e->park.device == park_device && e->park.bytes >= bytes) return FMA_OK;
    park_release(e);
    return park_store_create(e, park_device, bytes, &e->park);
}

void resident_release(fma_engine_t* e) {
    vmm_buffer_free(e->res);
    e->res_packed = false;
    e->res_off.clear();
    e->res_bytes.clear();
    e->res_store_bytes = 0;
}

void prefetch_release(fma_engine_t* e) {
    vmm_buffer_free(e->pf);
    e->pf_off.clear();
    e->pf_bytes.clear();
    e->pf_store_bytes = 0;
    std::lock_guard<std::mutex> lk(e->mu);
    for (Segment& s : e->segs) s.prefetch_off = kNoOffset;
}

bool image_in(fma_engine_t* e, ImageIn where) {
    std::lock_guard<std::mutex> lk(e->mu);
    for (const Segment& s : e->segs) {
        if (!s.has_backup) continue;
        switch (where) {
            case ImageIn::Host: if (s.backup_tier == FMA_TIER_HOST) return true; break;
            case ImageIn::NotHost: if (s.backup_tier != FMA_TIER_HOST && s.backup_tier != FMA_TIER_FILE) return true; break;
            case ImageIn::Local: if (!s.mapped && s.backup_tier == FMA_TIER_LOCAL) return true; break;
            case ImageIn::AnyAsleep: if (!s.mapped) return true; break;
        }
    }
    return false;
}

// ------------------------------------------------------------------------------------
// allocation
// ------------------------------------------------------------------------------------
int engine_alloc(fma_engine_t* e, size_t bytes, int tag, void** out) {
    if (bytes == 0) bytes = 1;
    const size_t sz = round_up(bytes, e->gran);
    std::lock_guard<std::mutex> lk(e->mu);
    int arena = -1;
    CUdeviceptr va = 0;
    RC(arena_take(e, tag, sz, &arena, &va));
    const int rc = vmm_create_and_map(e->device, va, sz);
    if (rc != FMA_OK) {
        arena_give_back(e->arenas[arena], va - e->arenas[arena].base, sz);
        return rc;
    }
    Unit u;
    u.va = va;
    u.bytes = sz;
    u.live_bytes = sz;
    u.arena = arena;
    e->units[va] = u;
    Segment s;
    s.va = va;
    s.bytes = sz;
    s.requested = bytes;
    s.tag = tag;
    s.arena = arena;
    s.unit_va = va;
    s.mapped = true;
    s.seq = e->next_seq++;
    e->by_va[va] = e->segs.size();
    e->segs.push_back(s);
    *out = reinterpret_cast<void*>(va);
    return FMA_OK;
}

int engine_free(fma_engine_t* e, void* ptr) {
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->by_va.find(reinterpret_cast<CUdeviceptr>(ptr));
    if (it == e->by_va.end()) return fail(FMA_ENOTFOUND, "pointer %p is not an engine segment", ptr);
    const size_t idx = it->second;
    const Segment s = e->segs[idx];
    e->segs.erase(e->segs.begin() + idx);
    e->by_va.clear();
    for (size_t i = 0; i < e->segs.size(); ++i) e->by_va[e->segs[i].va] = i;
    Arena& a = e->arenas[s.arena];
    if (!s.mapped) {  // asleep: nothing is mapped there, the VA is free again at once
        arena_give_back(a, s.va - a.base, s.bytes);
        return FMA_OK;
    }
    auto uit = e->units.find(s.unit_va);
    if (uit == e->units.end()) return fail(FMA_ESTATE, "segment %p has no mapping unit", ptr);
    Unit& u = uit->second;
    u.live_bytes -= s.bytes;
    u.zombies.emplace_back(s.va, s.bytes);
    if (u.live_bytes == 0) {
        // Drain work that may still touch the range before it is unmapped — the reference does
        // torch.cuda.synchronize() in its free callback for the same reason (cumem.py:156-169).
        cudaDeviceSynchronize();
        return unmap_units(e, u.va, u.bytes);
    }
    // The segment sits inside a run that was mapped as one unit (cuMemUnmap cannot split a mapping): it is gone
    // from the table now; its physical pages go with the unit at the next sleep / when the run empties.
    return FMA_OK;
}

// ------------------------------------------------------------------------------------
// packed image planning helpers shared by the pipelines
// ------------------------------------------------------------------------------------
// Fill h_tab[0..n) with the device address of every page of the packed image, in order.
size_t build_page_table(const std::vector<Extent>& ex, uint64_t* tab) {
    size_t n = 0;
    for (const Extent& x : ex)
        for (size_t o = 0; o < x.bytes; o += FMA_PAGE_BYTES) tab[n++] = (uint64_t)x.va + o;
    return n;
}

int check_pack_errors(fma_engine_t* e, const char* fmt) {
    RT(cudaMemcpyAsync(e->h_psize + e->pdesc_cap, e->d_psize + e->pdesc_cap, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    if (e->h_psize[e->pdesc_cap]) return fail(FMA_EINTEGRITY, fmt, e->h_psize[e->pdesc_cap]);
    return FMA_OK;
}

int flush_kernel_times(fma_engine_t* e) {
    if (!e->pending_events) return FMA_OK;
    double s = 0;
    for (size_t i = 0; i + 1 < e->pending_events; i += 2) {
        float ms = 0, ms0 = 0;
        RT(cudaEventElapsedTime(&ms, e->ev_pool[i], e->ev_pool[i + 1]));
        s += ms * 1e-3;
        // device-side timeline: launch i/2 ran [ms0, ms0 + ms) after ev_start (recorded tl_dev_base after the entry)
        if (cudaEventElapsedTime(&ms0, e->ev_start, e->ev_pool[i]) == cudaSuccess) {
            const double t0 = e->tl_entry + e->tl_dev_base + ms0 * 1e-3;
            e->tl_add(i / 2 < e->tl_kkind.size() ? e->tl_kkind[i / 2] : "kernel", (int)(i / 2), t0, t0 + ms * 1e-3, i / 2 < e->tl_kbytes.size() ? e->tl_kbytes[i / 2] : 0);
        } else {
            cudaGetLastError();
        }
    }
    e->st.kernel_seconds = s;
    e->st.kernel_bytes = e->pending_kernel_bytes;
    e->pending_events = 0;
    e->pending_kernel_bytes = 0;
    return FMA_OK;
}

// A sleep or wake that may launch K1 / K2 checks the engine's TMA shape before it unmaps, maps or copies anything: the
// launch wrapper refuses a shape that cannot run, and by the time of the first launch a sleep has already discarded
// segments while others are still mapped.  set_option checks one key at a time (a shape is set key by key, through
// combinations that do not fit), and FMA_TMA_* only seeds the same fields, so both are checked here.
int check_tma_shape(const fma_engine_t* e, int tier) {
    if (e->cfg.kernel != FMA_KERNEL_TMA || fma_layout::resolve_mode(e->cfg.mode, tier) == FMA_MODE_DIRECT) return FMA_OK;
    fma_k_tma_cfg c = e->tma;
    if (fma_k_tma_shape_fits(&c)) return FMA_OK;
    return fail(FMA_EINVAL, "TMA shape does not fit (tile %u B, %u stages, %u pipes): the tile must be >= 1 KiB, a multiple of 16 dividing "
                "2 MiB, and pipes x stages x tile + 128 B <= 227 KiB of shared memory", e->tma.tile_bytes, c.stages, c.pipes);
}

uint64_t store_dev_base(const fma_engine_t* e, int tier) {
    return tier == FMA_TIER_HOST ? (uint64_t)(uintptr_t)e->host.dev_alias : (uint64_t)e->park.va;
}
void* store_copy_base(const fma_engine_t* e, int tier) {   // (the FILE tier has no store in memory)
    return tier == FMA_TIER_HOST ? e->host.base : tier == FMA_TIER_FILE ? nullptr : reinterpret_cast<void*>(e->park.va);
}

// ------------------------------------------------------------------------------------
// digest of a set of segments in ONE launch (K3)
// ------------------------------------------------------------------------------------
int digest_segments(fma_engine_t* e, const std::vector<size_t>& idx, std::vector<uint64_t>* out) {
    size_t n_pages = 0;
    for (size_t i : idx) n_pages += e->segs[i].bytes / FMA_PAGE_BYTES;
    out->assign(idx.size(), 0);
    if (!n_pages) return FMA_OK;
    RC(ensure_streams(e));
    RC(ensure_desc(e, n_pages));
    size_t p = 0;
    for (size_t i : idx) {
        const Segment& s = e->segs[i];
        for (size_t o = 0; o < s.bytes; o += FMA_PAGE_BYTES, ++p) {
            e->h_desc[p].addr = (uint64_t)s.va + o;
            e->h_desc[p].first_word = o / 8;
        }
    }
    RT(cudaMemcpyAsync(e->d_desc, e->h_desc, n_pages * sizeof(fma_k_page_desc), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemsetAsync(e->d_dig, 0, n_pages * sizeof(uint64_t), e->ks));
    RT(fma_k_launch_page_digest(e->d_desc, (uint32_t)n_pages, e->d_dig, e->ks));
    RT(cudaMemcpyAsync(e->h_dig, e->d_dig, n_pages * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    e->st.total_kernel_launches += 1;
    p = 0;
    for (size_t k = 0; k < idx.size(); ++k) {
        uint64_t acc = 0;
        const size_t np = e->segs[idx[k]].bytes / FMA_PAGE_BYTES;
        for (size_t j = 0; j < np; ++j) acc += e->h_dig[p++];
        (*out)[k] = acc;
    }
    return FMA_OK;
}

int check_engine(fma_engine_t* e) {
    if (!e) return fail(FMA_EINVAL, "engine handle is NULL");
    return FMA_OK;
}

}  // namespace fma_impl

using namespace fma_impl;

// ======================================================================================
// C ABI
// ======================================================================================
extern "C" {

int fma_abi_version(void) { return FMA_ABI_VERSION; }
const char* fma_last_error(void) { return tl_err; }

int fma_driver_available(void) {
    if (driver_ready()) return FMA_OK;
    return fail(FMA_ENODRIVER, "%s", g_drv_err[0] ? g_drv_err : "CUDA driver not available");
}

int fma_engine_create(int device, const fma_config_t* cfg, fma_engine_t** out) {
    if (!out) return fail(FMA_EINVAL, "out is NULL");
    *out = nullptr;
    if (cfg && cfg->abi_version != FMA_ABI_VERSION)
        return fail(FMA_EINVAL, "config abi_version %u != library %d", cfg->abi_version, FMA_ABI_VERSION);
    if (!driver_ready()) return fail(FMA_ENODRIVER, "%s", g_drv_err[0] ? g_drv_err : "CUDA driver not available");
    int ndev = 0;
    RT(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(FMA_EINVAL, "device %d out of range (have %d)", device, ndev);
    DeviceGuard guard(device);
    RT(cudaFree(nullptr));  // make the primary context current on this thread
    fma_engine_t* e = new fma_engine();
    e->device = device;
    if (cfg) e->cfg = *cfg;
    e->cfg.abi_version = FMA_ABI_VERSION;
    if (e->cfg.numa_bind == 0 && !cfg) e->cfg.numa_bind = -1;
    // experiment knobs (documented in DESIGN.md); the config struct wins when set
    if (!e->cfg.mode) e->cfg.mode = env_int("FMA_MODE", 0);
    if (!e->cfg.kernel) e->cfg.kernel = env_int("FMA_KERNEL", 0);
    if (!e->cfg.copy_streams) e->cfg.copy_streams = env_int("FMA_COPY_STREAMS", 0);
    if (!e->cfg.chunk_bytes) e->cfg.chunk_bytes = (uint64_t)env_int("FMA_CHUNK_MIB", 0) << 20;
    if (!e->cfg.ring_slots) e->cfg.ring_slots = env_int("FMA_RING_SLOTS", 0);
    if (!e->cfg.map_threads) e->cfg.map_threads = env_int("FMA_MAP_THREADS", 0);
    if (!e->cfg.pack) e->cfg.pack = env_int("FMA_PACK", 0);
    e->incremental = env_int("FMA_INCREMENTAL", 0);
    e->resident_cap = (uint64_t)std::max(env_int("FMA_RESIDENT_MIB", 0), 0) << 20 & ~(uint64_t)(FMA_PAGE_BYTES - 1);
    e->tma.tile_bytes = (uint32_t)env_int("FMA_TMA_TILE_KIB", (int)(e->tma.tile_bytes >> 10)) << 10;
    e->tma.stages = (uint32_t)env_int("FMA_TMA_STAGES", (int)e->tma.stages);
    e->tma.pipes = (uint32_t)env_int("FMA_TMA_PIPES", (int)e->tma.pipes);
    e->tma.ctas_per_sm = (uint32_t)env_int("FMA_TMA_CTAS_PER_SM", (int)e->tma.ctas_per_sm);
    CUmemAllocationProp prop = device_prop(device);
    size_t gran = 0;
    CUresult r = g_drv.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
    if (r != CUDA_SUCCESS || gran == 0) {
        delete e;
        return fail(FMA_ECUDA, "cuMemGetAllocationGranularity failed: %s", cu_err(r));
    }
    if (gran % FMA_PAGE_BYTES != 0 && FMA_PAGE_BYTES % gran != 0) {
        delete e;
        return fail(FMA_ECUDA, "VMM granularity %zu incompatible with the 2 MiB engine page", gran);
    }
    e->gran = std::max(gran, FMA_PAGE_BYTES);
    e->tags.push_back("default");  // tag 0 == CuMemAllocator.default_tag (cumem.py:116)
    int rc = ensure_streams(e);
    if (rc != FMA_OK) {
        delete e;
        return rc;
    }
    *out = e;
    return FMA_OK;
}

int fma_engine_destroy(fma_engine_t* e) {
    if (!e) return FMA_OK;
    {
        std::lock_guard<std::mutex> lk(g_current_mu);
        if (g_current == e) g_current = nullptr;
    }
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    for (auto& kv : e->units) g_drv.MemUnmap(kv.second.va, kv.second.bytes);
    e->units.clear();
    for (Arena& a : e->arenas) g_drv.MemAddressFree(a.base, a.cap);
    e->arenas.clear();
    e->segs.clear();
    host_store_free(e->host);
    park_release(e);
    resident_release(e);
    prefetch_release(e);
    paths_release(e);
    release_ring(e);
    for (int i = 0; i < kMaxRing; ++i) {
        if (e->ev_ring_full[i]) cudaEventDestroy(e->ev_ring_full[i]);
        if (e->ev_ring_free[i]) cudaEventDestroy(e->ev_ring_free[i]);
    }
    if (e->d_tab) cudaFree(e->d_tab);
    if (e->h_tab) cudaFreeHost(e->h_tab);
    if (e->d_desc) cudaFree(e->d_desc);
    if (e->h_desc) cudaFreeHost(e->h_desc);
    if (e->d_dig) cudaFree(e->d_dig);
    if (e->h_dig) cudaFreeHost(e->h_dig);
    if (e->d_pdesc) cudaFree(e->d_pdesc);
    if (e->h_pdesc) cudaFreeHost(e->h_pdesc);
    if (e->d_psize) cudaFree(e->d_psize);
    if (e->h_psize) cudaFreeHost(e->h_psize);
    for (cudaEvent_t ev : e->ev_pool) cudaEventDestroy(ev);
    for (cudaEvent_t ev : e->ev_stage) cudaEventDestroy(ev);
    for (cudaEvent_t ev : e->ev_load) cudaEventDestroy(ev);
    if (e->load_ring) cudaFreeHost(e->load_ring);
    for (int i = 0; i < kMaxStreams; ++i) {
        if (e->cs[i]) cudaStreamDestroy(e->cs[i]);
        if (e->ev_cs[i]) cudaEventDestroy(e->ev_cs[i]);
    }
    if (e->ks) cudaStreamDestroy(e->ks);
    if (e->ev_start) cudaEventDestroy(e->ev_start);
    if (e->ev_end) cudaEventDestroy(e->ev_end);
    if (e->ev_res_done) cudaEventDestroy(e->ev_res_done);
    cudaGetLastError();
    delete e;
    return FMA_OK;
}

int fma_set_current(fma_engine_t* e) {
    std::lock_guard<std::mutex> lk(g_current_mu);
    g_current = e;
    return FMA_OK;
}
fma_engine_t* fma_get_current(void) {
    std::lock_guard<std::mutex> lk(g_current_mu);
    return g_current;
}

int fma_tag_intern(fma_engine_t* e, const char* name) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!name) return fail(FMA_EINVAL, "tag name is NULL");
    std::lock_guard<std::mutex> lk(e->mu);
    for (size_t i = 0; i < e->tags.size(); ++i)
        if (e->tags[i] == name) return (int)i;
    if (e->tags.size() >= FMA_MAX_TAGS) return fail(FMA_ENOMEM, "more than %d tags", FMA_MAX_TAGS);
    e->tags.push_back(name);
    return (int)e->tags.size() - 1;
}

int fma_tag_name(fma_engine_t* e, int tag, char* buf, size_t buflen) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> lk(e->mu);
    if (tag < 0 || (size_t)tag >= e->tags.size() || !buf || !buflen) return fail(FMA_ENOTFOUND, "unknown tag %d", tag);
    snprintf(buf, buflen, "%s", e->tags[tag].c_str());
    return FMA_OK;
}

int fma_set_current_tag(fma_engine_t* e, int tag) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> lk(e->mu);
    if (tag < 0 || (size_t)tag >= e->tags.size()) return fail(FMA_ENOTFOUND, "unknown tag %d", tag);
    e->current_tag = tag;
    return FMA_OK;
}

void* my_malloc(ssize_t size, int device, void* /*stream*/) {
    fma_engine_t* e = fma_get_current();
    if (!e) {
        // same convenience as the reference module, whose globals exist as soon as it is loaded
        if (fma_engine_create(device, nullptr, &e) != FMA_OK) return nullptr;
        fma_set_current(e);
    }
    if (e->device != device) {
        fail(FMA_EINVAL, "my_malloc for device %d but the current engine owns device %d", device, e->device);
        return nullptr;
    }
    if (size < 0) return nullptr;
    DeviceGuard guard(e->device);
    int tag;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        tag = e->current_tag;
    }
    void* p = nullptr;
    if (engine_alloc(e, (size_t)size, tag, &p) != FMA_OK) return nullptr;
    return p;
}

void my_free(void* ptr, ssize_t /*size*/, int /*device*/, void* /*stream*/) {
    fma_engine_t* e = fma_get_current();
    if (!e || !ptr) return;
    DeviceGuard guard(e->device);
    engine_free(e, ptr);
}

int fma_alloc(fma_engine_t* e, size_t bytes, int tag, void** out_ptr) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out_ptr) return fail(FMA_EINVAL, "out_ptr is NULL");
    {
        std::lock_guard<std::mutex> lk(e->mu);
        if (tag < 0 || (size_t)tag >= e->tags.size()) return fail(FMA_ENOTFOUND, "unknown tag %d", tag);
    }
    DeviceGuard guard(e->device);
    return engine_alloc(e, bytes, tag, out_ptr);
}

int fma_free(fma_engine_t* e, void* ptr) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    DeviceGuard guard(e->device);
    return engine_free(e, ptr);
}

int fma_segment_count(fma_engine_t* e) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> lk(e->mu);
    return (int)e->segs.size();
}

int fma_segment_info(fma_engine_t* e, int index, fma_segment_info_t* out) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out) return fail(FMA_EINVAL, "out is NULL");
    std::lock_guard<std::mutex> lk(e->mu);
    if (index < 0 || (size_t)index >= e->segs.size()) return fail(FMA_ENOTFOUND, "segment index %d out of range", index);
    const Segment& s = e->segs[index];
    out->va = (uint64_t)s.va;
    out->bytes = s.bytes;
    out->requested_bytes = s.requested;
    out->packed_offset = s.packed_off;
    out->seq = s.seq;
    out->tag = s.tag;
    out->mapped = s.mapped ? 1 : 0;
    out->has_backup = s.has_backup ? 1 : 0;
    out->tier = s.backup_tier;
    return FMA_OK;
}

int fma_segment_find(fma_engine_t* e, const void* ptr) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->by_va.find(reinterpret_cast<CUdeviceptr>(ptr));
    if (it == e->by_va.end()) return fail(FMA_ENOTFOUND, "pointer %p is not an engine segment", ptr);
    return (int)it->second;
}

uint64_t fma_current_usage(fma_engine_t* e) {
    if (!e) return 0;
    std::lock_guard<std::mutex> lk(e->mu);
    uint64_t sum = 0;
    for (const Segment& s : e->segs) sum += s.bytes;
    return sum;
}

// One operation per engine at a time: the controller retries POST /wake_up after its 5 s timeout
// (inference-server.go:1699-1716), so a second call can arrive while the first is still mapping; it waits and then finds
// nothing left to do (idempotence, abstract.py:336-338).
int fma_sleep(fma_engine_t* e, uint64_t offload_tag_mask, int tier, uint32_t flags) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    return do_sleep(e, offload_tag_mask, tier, flags);
}

int fma_wake(fma_engine_t* e, uint64_t tag_mask, uint32_t flags) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    return do_wake(e, tag_mask, flags);
}

// Text timeline of the last sleep / wake: one line per event, "op,kind,idx,t0_ms,t1_ms,bytes" (times since the call's entry;
// `kernel` rows are device-timed).  Returns the number of bytes the full text needs (excluding the NUL); writes at most cap-1.
int fma_timeline(fma_engine_t* e, char* buf, size_t cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    {
        DeviceGuard guard(e->device);
        RC(flush_kernel_times(e));
    }
    std::lock_guard<std::mutex> lk(e->tl_mu);
    std::string out;
    char line[160];
    for (const TimelineEv& ev : e->tl) {
        snprintf(line, sizeof(line), "%s,%s,%d,%.3f,%.3f,%llu\n", e->tl_op, ev.kind, ev.idx, ev.t0 * 1e3, ev.t1 * 1e3, (unsigned long long)ev.bytes);
        out += line;
    }
    if (buf && cap) {
        const size_t n = std::min(out.size(), cap - 1);
        memcpy(buf, out.data(), n);
        buf[n] = 0;
    }
    return (int)out.size();
}

int fma_is_sleeping(fma_engine_t* e) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> lk(e->mu);
    for (const Segment& s : e->segs)
        if (!s.mapped) return 1;
    return 0;
}

int fma_swap(fma_engine_t* out_e, uint64_t offload_tag_mask, int tier, fma_engine_t* in_e, uint64_t wake_tag_mask,
             uint32_t flags) {
    if (check_engine(out_e) != FMA_OK || check_engine(in_e) != FMA_OK) return FMA_EINVAL;
    if (out_e == in_e) return fail(FMA_EINVAL, "swap needs two different engines");
    {  // neither half starts when the other would refuse its shape
        int rc = check_tma_shape(out_e, tier);
        if (rc == FMA_OK) rc = check_tma_shape(in_e, in_e->image_tier);
        if (rc != FMA_OK) return rc;
    }
    int rc_sleep = FMA_OK;
    char sleep_msg[512] = "";
    std::thread t([&] {
        std::lock_guard<std::mutex> op(out_e->op_mu);
        rc_sleep = do_sleep(out_e, offload_tag_mask, tier, flags);
        if (rc_sleep != FMA_OK) snprintf(sleep_msg, sizeof(sleep_msg), "%s", tl_err);
    });
    int rc_wake;
    {
        std::lock_guard<std::mutex> op(in_e->op_mu);
        rc_wake = do_wake(in_e, wake_tag_mask, flags);
    }
    t.join();
    if (rc_wake != FMA_OK) return rc_wake;
    if (rc_sleep != FMA_OK) return fail(rc_sleep, "%s", sleep_msg);
    return FMA_OK;
}

// Store management takes the engine's operation lock: the Python shim pre-pins from a background thread right after the weights
// pool closes (cumem.py), and a /sleep arriving meanwhile must wait for that pin instead of racing it.  The segment table is
// only ever walked under e->mu (torch may be allocating the kv_cache pool on another thread at that moment).
int fma_host_reserve(fma_engine_t* e, size_t bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (e->host.cap < bytes && image_in(e, ImageIn::Host)) return fail(FMA_ESTATE, "cannot regrow the host store while it holds a sleeping image");
    DeviceGuard guard(e->device);
    return host_store_reserve(e, bytes);
}

int fma_host_release(fma_engine_t* e) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (image_in(e, ImageIn::Host)) return fail(FMA_ESTATE, "host store holds a sleeping image");
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    invalidate_shadows(e);
    host_store_free(e->host);
    e->st.host_store_bytes = 0;
    return FMA_OK;
}

int fma_host_store_view(fma_engine_t* e, const void** base, uint64_t* bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!base || !bytes) return fail(FMA_EINVAL, "NULL out pointer");
    if (!e->host.base || e->image_tier != FMA_TIER_HOST) return fail(FMA_ESTATE, "no host image");
    *base = e->host.base;
    *bytes = e->image_packed ? e->image_store_bytes : e->image_bytes;  // what the image occupies in the store
    return FMA_OK;
}

int fma_peer_reserve(fma_engine_t* e, int peer_device, size_t bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (image_in(e, ImageIn::NotHost)) return fail(FMA_ESTATE, "parking buffer holds a sleeping image");
    DeviceGuard guard(e->device);
    return park_reserve(e, peer_device, bytes);
}

int fma_peer_release(fma_engine_t* e) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (image_in(e, ImageIn::NotHost)) return fail(FMA_ESTATE, "parking buffer holds a sleeping image");
    DeviceGuard guard(e->device);
    return park_release(e);
}

// ---- node-level parking buffers (SURVEY section 8f-1): exportable VMM allocations ------------------------------------------
// The reference launcher pins every instance to its own GPUs (inference_server/launcher/launcher.py:171-187 overwrites
// CUDA_VISIBLE_DEVICES), so an instance cannot cuMemCreate on an idle peer itself, and whatever it allocates dies with it —
// exactly when the controller would otherwise cold-start (pkg/controller/dual-pods/inference-server.go:416-448).  A node-level
// owner (the node agent, which sees every GPU) therefore creates the parking buffer with a POSIX-fd shareable handle, keeps
// it alive, and hands the fd to instances (SCM_RIGHTS / inheritance); an instance imports it, maps it and grants access to
// ITS GPU only — reads and writes then go over NVLink / NVSwitch although the buffer's GPU is not visible to the instance.
namespace {
struct Parking {
    CUmemGenericAllocationHandle handle;
    size_t bytes;
    int device;
};
std::mutex g_parking_mu;
std::map<uint64_t, Parking> g_parkings;
uint64_t g_next_parking = 1;
}  // namespace

int fma_parking_create(int device, size_t bytes, uint64_t* out_handle, int* out_fd) {
    if (!out_handle || !out_fd) return fail(FMA_EINVAL, "out pointers are NULL");
    if (!driver_ready()) return fail(FMA_ENODRIVER, "%s", g_drv_err);
    int ndev = 0;
    RT(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(FMA_EINVAL, "device %d not visible (have %d)", device, ndev);
    DeviceGuard guard(device);
    RT(cudaFree(nullptr));  // the device's primary context must exist
    CUmemAllocationProp prop = device_prop(device);
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gran = FMA_PAGE_BYTES;
    DRV(g_drv.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
    bytes = round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), std::max<size_t>(gran, FMA_PAGE_BYTES));
    Parking p;
    p.bytes = bytes;
    p.device = device;
    RC(vmm_create(device, bytes, true, &p.handle));
    int fd = -1;
    CUresult r = g_drv.MemExportToShareableHandle(&fd, p.handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    if (r != CUDA_SUCCESS) {
        g_drv.MemRelease(p.handle);
        return fail(FMA_ECUDA, "cuMemExportToShareableHandle failed: %s", cu_err(r));
    }
    std::lock_guard<std::mutex> lk(g_parking_mu);
    *out_handle = g_next_parking++;
    g_parkings[*out_handle] = p;
    *out_fd = fd;
    return FMA_OK;
}

int fma_parking_export(uint64_t handle, int* out_fd, uint64_t* out_bytes) {
    if (!out_fd) return fail(FMA_EINVAL, "out_fd is NULL");
    std::lock_guard<std::mutex> lk(g_parking_mu);
    auto it = g_parkings.find(handle);
    if (it == g_parkings.end()) return fail(FMA_ENOTFOUND, "unknown parking handle %llu", (unsigned long long)handle);
    int fd = -1;
    DRV(g_drv.MemExportToShareableHandle(&fd, it->second.handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    *out_fd = fd;
    if (out_bytes) *out_bytes = it->second.bytes;
    return FMA_OK;
}

int fma_parking_destroy(uint64_t handle) {
    std::lock_guard<std::mutex> lk(g_parking_mu);
    auto it = g_parkings.find(handle);
    if (it == g_parkings.end()) return fail(FMA_ENOTFOUND, "unknown parking handle %llu", (unsigned long long)handle);
    g_drv.MemRelease(it->second.handle);  // the memory goes once the last importer has unmapped it
    g_parkings.erase(it);
    return FMA_OK;
}

int fma_peer_attach(fma_engine_t* e, int fd, size_t bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (fd < 0 || bytes == 0 || bytes % FMA_PAGE_BYTES) return fail(FMA_EINVAL, "attach needs the owner's fd and the buffer's size (a multiple of 2 MiB)");
    std::lock_guard<std::mutex> op(e->op_mu);
    if (image_in(e, ImageIn::NotHost)) return fail(FMA_ESTATE, "parking buffer holds a sleeping image");
    DeviceGuard guard(e->device);
    RC(park_release(e));
    CUmemGenericAllocationHandle h = 0;
    RC(vmm_import(fd, &h));
    char what[160];
    snprintf(what, sizeof(what), "attach, %zu bytes: the size the owner created? a P2P path from device %d to the buffer's GPU?", bytes, e->device);
    RC(vmm_buffer_map(h, bytes, {e->device}, what, &e->park));
    e->park.device = kForeignDevice;
    return FMA_OK;
}

// A private, empty host store whose NUMA placement no longer fits the MULTI-PATH configuration (paths set, changed or cleared
// after it was pinned) is placed again: now, not inside the next sleep.  A store that holds an image, is shared or was adopted
// stays as it is.
static int replace_store_for_paths(fma_engine_t* e) {
    if (e->host.base && !image_in(e, ImageIn::Host) && !e->host.shared && e->host.fd < 0 && e->host.registered && e->host.placed_for != paths_signature(e)) {
        const size_t cap = e->host.cap;
        if (e->shadow_tier == FMA_TIER_HOST) invalidate_shadows(e);
        host_store_free(e->host);
        RC(host_store_reserve(e, cap));
    }
    return FMA_OK;
}

// MULTI-PATH wake: declare the idle peer GPUs whose PCIe links a host-tier wake of this engine may borrow (n = 0: none).
// slot_bytes / slots: size and depth of the staging buffer each path (own link included) gets; 0 = defaults (128 MiB x 3).
int fma_paths_set(fma_engine_t* e, const int* helper_devices, int n, size_t slot_bytes, int slots) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (n < 0 || n > kMaxPaths - 1 || (n && !helper_devices)) return fail(FMA_EINVAL, "0..%d helper devices", kMaxPaths - 1);
    std::lock_guard<std::mutex> op(e->op_mu);
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    paths_release(e);
    if (n == 0) return replace_store_for_paths(e);   // a striped store goes back to the engine's own NUMA node
    slot_bytes = round_up(slot_bytes ? slot_bytes : ((size_t)128 << 20), FMA_PAGE_BYTES);
    slots = slots > 0 ? std::min(slots, kMaxRing) : 3;
    int ndev = 0;
    RT(cudaGetDeviceCount(&ndev));
    std::vector<int> devs{e->device};
    for (int i = 0; i < n; ++i) {
        const int d = helper_devices[i];
        if (d < 0 || d >= ndev || std::find(devs.begin(), devs.end(), d) != devs.end())
            return fail(FMA_EINVAL, "helper device %d is not visible, is the engine's own GPU, or is listed twice", d);
        int can = 0;
        RT(cudaDeviceCanAccessPeer(&can, e->device, d));
        if (!can) return fail(FMA_ECUDA, "device %d cannot access helper %d (no NVLink/P2P path)", e->device, d);
        devs.push_back(d);
    }
    e->path_slot_bytes = slot_bytes;
    e->path_slots = slots;
    const size_t bytes = slot_bytes * (size_t)slots;
    for (int d : devs) {
        e->paths.emplace_back();
        WakePath& p = e->paths.back();
        p.device = d;
        p.numa_node = gpu_numa_node(d);
        char what[64];
        snprintf(what, sizeof(what), "path staging on device %d", d);
        CUmemGenericAllocationHandle h = 0;
        int rc = FMA_OK;
        {
            DeviceGuard g(d);
            if (cudaFree(nullptr) != cudaSuccess) rc = fail(FMA_ECUDA, "cannot initialise helper device %d", d);
            if (rc == FMA_OK) rc = vmm_create(d, bytes, false, &h);
            if (rc == FMA_OK) rc = vmm_buffer_map(h, bytes, {d, e->device}, what, &p.staging);
        }
        if (rc == FMA_OK) rc = open_path(p, slots);
        if (rc != FMA_OK) return paths_fail(e, rc);
    }
    return replace_store_for_paths(e);
}

int fma_digest_segment(fma_engine_t* e, int index, uint64_t* out) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out) return fail(FMA_EINVAL, "out is NULL");
    if (index < 0 || (size_t)index >= e->segs.size()) return fail(FMA_ENOTFOUND, "segment index %d out of range", index);
    if (!e->segs[index].mapped) return fail(FMA_ESTATE, "segment %d is not mapped", index);
    DeviceGuard guard(e->device);
    std::vector<uint64_t> dg;
    int rc = digest_segments(e, {(size_t)index}, &dg);
    if (rc == FMA_OK) *out = dg[0];
    return rc;
}

int fma_digest_all(fma_engine_t* e, uint64_t tag_mask, uint64_t* out, int n) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out || n < (int)e->segs.size()) return fail(FMA_EINVAL, "out too small: %d < %zu", n, e->segs.size());
    DeviceGuard guard(e->device);
    std::vector<size_t> idx;
    for (size_t i = 0; i < e->segs.size(); ++i) {
        out[i] = 0;
        const Segment& s = e->segs[i];
        if (s.mapped && (!tag_mask || tag_bit_set(tag_mask, s.tag))) idx.push_back(i);
    }
    std::vector<uint64_t> dg;
    RC(digest_segments(e, idx, &dg));
    for (size_t k = 0; k < idx.size(); ++k) out[idx[k]] = dg[k];
    return FMA_OK;
}

int fma_fill_segment(fma_engine_t* e, int index, uint64_t seed, uint64_t first_word) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (index < 0 || (size_t)index >= e->segs.size()) return fail(FMA_ENOTFOUND, "segment index %d out of range", index);
    const Segment& s = e->segs[index];
    if (!s.mapped) return fail(FMA_ESTATE, "segment %d is not mapped", index);
    DeviceGuard guard(e->device);
    const size_t n_pages = s.bytes / FMA_PAGE_BYTES;
    RC(ensure_desc(e, n_pages));
    for (size_t p = 0; p < n_pages; ++p) {
        e->h_desc[p].addr = (uint64_t)s.va + p * FMA_PAGE_BYTES;
        e->h_desc[p].first_word = first_word + p * (FMA_PAGE_BYTES / 8);
    }
    RT(cudaMemcpyAsync(e->d_desc, e->h_desc, n_pages * sizeof(fma_k_page_desc), cudaMemcpyHostToDevice, e->ks));
    RT(fma_k_launch_fill(e->d_desc, (uint32_t)n_pages, seed, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    e->st.total_kernel_launches += 1;
    return FMA_OK;
}

int fma_segment_write(fma_engine_t* e, int index, uint64_t offset, const void* host_src, uint64_t bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (index < 0 || (size_t)index >= e->segs.size()) return fail(FMA_ENOTFOUND, "segment index %d out of range", index);
    const Segment& s = e->segs[index];
    if (!s.mapped) return fail(FMA_ESTATE, "segment %d is not mapped", index);
    if (offset + bytes > s.bytes) return fail(FMA_EINVAL, "write past the end of segment %d", index);
    DeviceGuard guard(e->device);
    RT(cudaMemcpyAsync(reinterpret_cast<void*>(s.va + offset), host_src, bytes, cudaMemcpyHostToDevice, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    return FMA_OK;
}

int fma_segment_read(fma_engine_t* e, int index, uint64_t offset, void* host_dst, uint64_t bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (index < 0 || (size_t)index >= e->segs.size()) return fail(FMA_ENOTFOUND, "segment index %d out of range", index);
    const Segment& s = e->segs[index];
    if (!s.mapped) return fail(FMA_ESTATE, "segment %d is not mapped", index);
    if (offset + bytes > s.bytes) return fail(FMA_EINVAL, "read past the end of segment %d", index);
    DeviceGuard guard(e->device);
    RT(cudaMemcpyAsync(host_dst, reinterpret_cast<const void*>(s.va + offset), bytes, cudaMemcpyDeviceToHost, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    return FMA_OK;
}

int fma_op_page_copy(fma_engine_t* e, const uint64_t* src_pages, uint64_t src_base, const uint64_t* dst_pages,
                     uint64_t dst_base, uint32_t n_pages, int kernel_variant, float* out_ms) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!n_pages) return FMA_OK;
    DeviceGuard guard(e->device);
    RC(ensure_tables(e, n_pages));
    const uint64_t* d_src = nullptr;
    const uint64_t* d_dst = nullptr;
    if (src_pages) {
        memcpy(e->h_tab, src_pages, n_pages * sizeof(uint64_t));
        RT(cudaMemcpyAsync(e->d_tab, e->h_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
        d_src = e->d_tab;
    }
    if (dst_pages) {
        memcpy(e->h_tab + e->d_tab_cap, dst_pages, n_pages * sizeof(uint64_t));
        RT(cudaMemcpyAsync(e->d_tab + e->d_tab_cap, e->h_tab + e->d_tab_cap, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
        d_dst = e->d_tab + e->d_tab_cap;
    }
    RT(cudaEventRecord(e->ev_start, e->ks));
    RT(fma_k_launch_page_copy(d_src, src_base, d_dst, dst_base, n_pages, kernel_variant, &e->tma, e->ks));
    RT(cudaEventRecord(e->ev_end, e->ks));
    RT(cudaEventSynchronize(e->ev_end));
    e->st.total_kernel_launches += 1;
    if (out_ms) RT(cudaEventElapsedTime(out_ms, e->ev_start, e->ev_end));
    return FMA_OK;
}

int fma_op_page_digest(fma_engine_t* e, const uint64_t* pages, uint64_t base, const uint64_t* first_word, uint32_t n_pages,
                       uint64_t* out_page_digests, float* out_ms) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!n_pages) return FMA_OK;
    if (!out_page_digests) return fail(FMA_EINVAL, "out is NULL");
    DeviceGuard guard(e->device);
    RC(ensure_desc(e, n_pages));
    for (uint32_t p = 0; p < n_pages; ++p) {
        e->h_desc[p].addr = pages ? pages[p] : base + (uint64_t)p * FMA_PAGE_BYTES;
        e->h_desc[p].first_word = first_word ? first_word[p] : (uint64_t)p * (FMA_PAGE_BYTES / 8);
    }
    RT(cudaMemcpyAsync(e->d_desc, e->h_desc, n_pages * sizeof(fma_k_page_desc), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemsetAsync(e->d_dig, 0, n_pages * sizeof(uint64_t), e->ks));
    RT(cudaEventRecord(e->ev_start, e->ks));
    RT(fma_k_launch_page_digest(e->d_desc, n_pages, e->d_dig, e->ks));
    RT(cudaEventRecord(e->ev_end, e->ks));
    RT(cudaMemcpyAsync(e->h_dig, e->d_dig, n_pages * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    e->st.total_kernel_launches += 1;
    memcpy(out_page_digests, e->h_dig, n_pages * sizeof(uint64_t));
    if (out_ms) RT(cudaEventElapsedTime(out_ms, e->ev_start, e->ev_end));
    return FMA_OK;
}

// ---- PACKED image: page layout query + raw K4p / K4 / K5 ----------------------------------------------------
int fma_image_pages(fma_engine_t* e, uint64_t* out_offsets, uint32_t* out_bytes, uint32_t cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!image_in(e, ImageIn::AnyAsleep)) return 0;
    const size_t n = e->image_bytes / FMA_PAGE_BYTES;
    for (size_t p = 0; p < n && p < cap; ++p) {
        if (out_offsets) out_offsets[p] = e->image_packed ? e->img_off[p] : (uint64_t)p * FMA_PAGE_BYTES;
        if (out_bytes) out_bytes[p] = e->image_packed ? e->img_bytes[p] : (uint32_t)FMA_PAGE_BYTES;
    }
    // RESIDENT share: the resident part's pages follow the host part's, with offsets in the resident buffer
    const size_t nr = e->res.va ? (e->res_packed ? e->res_bytes.size() : e->res_store_bytes / FMA_PAGE_BYTES) : 0;
    for (size_t q = 0; q < nr && n + q < cap; ++q) {
        if (out_offsets) out_offsets[n + q] = e->res_packed ? e->res_off[q] : (uint64_t)q * FMA_PAGE_BYTES;
        if (out_bytes) out_bytes[n + q] = e->res_packed ? e->res_bytes[q] : (uint32_t)FMA_PAGE_BYTES;
    }
    return (int)(n + nr);
}

int fma_op_pack_probe(fma_engine_t* e, const uint64_t* pages, uint64_t base, uint32_t n_pages, uint32_t* out_stored_bytes, float* out_ms) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!n_pages) return FMA_OK;
    if (!out_stored_bytes) return fail(FMA_EINVAL, "out is NULL");
    DeviceGuard guard(e->device);
    RC(ensure_tables(e, n_pages));
    RC(ensure_pack_bufs(e, n_pages));
    for (uint32_t p = 0; p < n_pages; ++p) e->h_tab[p] = pages ? pages[p] : base + (uint64_t)p * FMA_PAGE_BYTES;
    RT(cudaMemcpyAsync(e->d_tab, e->h_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    RT(cudaEventRecord(e->ev_start, e->ks));
    RT(fma_k_launch_pack_probe(e->d_tab, n_pages, e->d_psize, e->ks));
    RT(cudaEventRecord(e->ev_end, e->ks));
    RT(cudaMemcpyAsync(e->h_psize, e->d_psize, n_pages * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    e->st.total_kernel_launches += 1;
    memcpy(out_stored_bytes, e->h_psize, n_pages * sizeof(uint32_t));
    if (out_ms) RT(cudaEventElapsedTime(out_ms, e->ev_start, e->ev_end));
    return FMA_OK;
}

// shared by fma_op_pack / fma_op_unpack: stored pages back to back from store_base, device pages from a table or a base
static int run_pack_op(fma_engine_t* e, bool unpack, const uint64_t* dev_pages, uint64_t dev_base, uint64_t store_base,
                const uint32_t* stored_bytes, uint32_t n_pages, float* out_ms) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!n_pages) return FMA_OK;
    if (!stored_bytes) return fail(FMA_EINVAL, "stored_bytes is NULL");
    DeviceGuard guard(e->device);
    RC(ensure_pack_bufs(e, n_pages));
    uint64_t off = 0;
    for (uint32_t p = 0; p < n_pages; ++p) {
        if (stored_bytes[p] != FMA_K_PACKED_PAGE_BYTES && stored_bytes[p] != FMA_PAGE_BYTES)
            return fail(FMA_EINVAL, "stored size %u of page %u is neither packed nor raw", stored_bytes[p], p);
        const uint64_t dev = dev_pages ? dev_pages[p] : dev_base + (uint64_t)p * FMA_PAGE_BYTES;
        set_pack_desc(e->h_pdesc[p], unpack ? store_base + off : dev, unpack ? dev : store_base + off, stored_bytes[p]);
        off += stored_bytes[p];
    }
    uint32_t* d_err = e->d_psize + e->pdesc_cap;
    RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, n_pages * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemsetAsync(d_err, 0, sizeof(uint32_t), e->ks));
    RT(cudaEventRecord(e->ev_start, e->ks));
    if (unpack) RT(fma_k_launch_unpack(e->d_pdesc, n_pages, d_err, e->ks));
    else RT(fma_k_launch_pack(e->d_pdesc, n_pages, d_err, e->ks));
    RT(cudaEventRecord(e->ev_end, e->ks));
    const int rc = check_pack_errors(e, unpack ? "%u page(s) could not be decoded (malformed stored page)"
                                           : "%u page(s) could not be coded (more exceptions than the probe saw)");
    e->st.total_kernel_launches += 1;
    if (out_ms) RT(cudaEventElapsedTime(out_ms, e->ev_start, e->ev_end));
    return rc;
}

int fma_op_pack(fma_engine_t* e, const uint64_t* src_pages, uint64_t src_base, uint64_t dst_base, const uint32_t* stored_bytes,
                uint32_t n_pages, float* out_ms) {
    return run_pack_op(e, false, src_pages, src_base, dst_base, stored_bytes, n_pages, out_ms);
}

int fma_op_unpack(fma_engine_t* e, uint64_t src_base, const uint32_t* stored_bytes, const uint64_t* dst_pages, uint64_t dst_base,
                  uint32_t n_pages, float* out_ms) {
    return run_pack_op(e, true, dst_pages, dst_base, src_base, stored_bytes, n_pages, out_ms);
}

int fma_scratch_alloc(fma_engine_t* e, size_t bytes, uint64_t* out_dev_ptr) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out_dev_ptr) return fail(FMA_EINVAL, "out is NULL");
    DeviceGuard guard(e->device);
    void* p = nullptr;
    cudaError_t r = cudaMalloc(&p, bytes);
    if (r != cudaSuccess) {
        cudaGetLastError();
        return fail(FMA_ENOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(r));
    }
    *out_dev_ptr = (uint64_t)(uintptr_t)p;
    return FMA_OK;
}

int fma_scratch_free(fma_engine_t* e, uint64_t dev_ptr) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    DeviceGuard guard(e->device);
    RT(cudaFree(reinterpret_cast<void*>((uintptr_t)dev_ptr)));
    return FMA_OK;
}

int fma_set_option(fma_engine_t* e, const char* key, int64_t value) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!key) return fail(FMA_EINVAL, "key is NULL");
    const std::string k(key);
    if (k == "mode") {
        if (value < FMA_MODE_AUTO || value > FMA_MODE_KERNEL) return fail(FMA_EINVAL, "bad mode %lld", (long long)value);
        e->cfg.mode = (int32_t)value;
    } else if (k == "kernel") {
        if (value != FMA_KERNEL_TMA && value != FMA_KERNEL_LDG) return fail(FMA_EINVAL, "bad kernel %lld", (long long)value);
        e->cfg.kernel = (int32_t)value;
    } else if (k == "copy_streams") {
        if (value < 1 || value > kMaxStreams) return fail(FMA_EINVAL, "copy_streams must be 1..%d", kMaxStreams);
        e->cfg.copy_streams = (int32_t)value;
        e->n_cs = (int)value;
    } else if (k == "chunk_bytes") {
        if (value < (int64_t)FMA_PAGE_BYTES) return fail(FMA_EINVAL, "chunk_bytes must be >= 2 MiB");
        e->cfg.chunk_bytes = (uint64_t)value;
    } else if (k == "ring_slots") {
        if (value < 2 || value > kMaxRing) return fail(FMA_EINVAL, "ring_slots must be 2..%d", kMaxRing);
        e->cfg.ring_slots = (int32_t)value;
    } else if (k == "map_threads") {
        if (value < 1 || value > 8) return fail(FMA_EINVAL, "map_threads must be 1..8");
        e->cfg.map_threads = (int32_t)value;
    } else if (k == "pack") {
        if (value != 0 && value != 1) return fail(FMA_EINVAL, "pack must be 0 or 1");
        e->cfg.pack = (int32_t)value;
    } else if (k == "incremental") {
        if (value != 0 && value != 1) return fail(FMA_EINVAL, "incremental must be 0 or 1");
        e->incremental = (int)value;
    } else if (k == "resident_bytes") {
        if (value < 0) return fail(FMA_EINVAL, "resident_bytes must be >= 0");
        e->resident_cap = (uint64_t)value & ~(uint64_t)(FMA_PAGE_BYTES - 1);
    } else if (k == "tma_tile_bytes") {
        if (value < 1024 || (FMA_PAGE_BYTES % (size_t)value) != 0 || value % 16) return fail(FMA_EINVAL, "bad tma tile %lld", (long long)value);
        e->tma.tile_bytes = (uint32_t)value;
    } else if (k == "tma_stages") {
        e->tma.stages = (uint32_t)value;
    } else if (k == "tma_pipes") {
        e->tma.pipes = (uint32_t)value;
    } else if (k == "tma_ctas_per_sm") {
        e->tma.ctas_per_sm = (uint32_t)value;
    } else if (k == "load_threads") {
        if (value < 1 || value > 64) return fail(FMA_EINVAL, "load_threads must be 1..64");
        e->load_threads = (int)value;
    } else if (k == "load_chunk_bytes") {
        if (value < (1 << 20) || value % 4096) return fail(FMA_EINVAL, "load_chunk_bytes must be >= 1 MiB and 4 KiB aligned");
        e->load_chunk = (size_t)value;
    } else if (k == "load_slots") {
        if (value < 2 || value > 256) return fail(FMA_EINVAL, "load_slots must be 2..256");
        e->load_slots = (int)value;
    } else {
        return fail(FMA_ENOTFOUND, "unknown option %s", key);
    }
    return FMA_OK;
}

int fma_stats(fma_engine_t* e, fma_stats_t* out) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out) return fail(FMA_EINVAL, "out is NULL");
    {
        DeviceGuard guard(e->device);
        RC(flush_kernel_times(e));
    }
    *out = e->st;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        uint64_t mapped = 0;
        for (const auto& kv : e->units) mapped += kv.second.bytes;
        out->hbm_mapped_bytes = mapped;
    }
    uint64_t own_staging = 0;   // multi-path staging slots that live in THIS GPU's HBM (helpers' slots are their GPUs' business)
    for (const WakePath& wp : e->paths)
        if (!wp.remote && wp.device == e->device) own_staging += wp.staging.bytes;
    out->hbm_aux_bytes = own_staging + (e->ring_attached ? 0 : (uint64_t)e->n_ring * e->ring_slot_bytes) + 2 * e->d_tab_cap * sizeof(uint64_t) +
                         e->desc_cap * (sizeof(fma_k_page_desc) + sizeof(uint64_t)) +
                         e->pdesc_cap * (sizeof(fma_k_pack_desc) + sizeof(uint32_t));
    out->parked_bytes = e->park.bytes;
    out->image_packed = e->image_packed ? 1 : 0;
    out->image_store_bytes = e->image_store_bytes;
    out->resident_bytes = e->res.va ? e->res_store_bytes : 0;
    out->io_buffer_bytes = e->load_ring_bytes;
    out->prefetched_bytes = e->pf_store_bytes.load();
    return FMA_OK;
}

}  // extern "C"
