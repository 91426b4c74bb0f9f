// hostsim_cuda.cpp — HOST SIMULATION of the CUDA runtime + VMM driver calls the engine uses.  TEST INFRASTRUCTURE ONLY.
//
// Purpose: run the host engine's logic (csrc/fma_engine.cu, fma_sleep.cu, fma_wake.cu, fma_load.cu, fma_image.cu:
// segment table, arenas, runs, ring, mapper/unmapper threads, stage events,
// error paths) on a machine without a GPU, under ASan/TSan if wanted.  It is linked ONLY into
// tests/cpp/hostsim/libfma_b200_hostsim.so by tests/test_engine_hostsim.py; the product library
// (llm-d-fast-model-actuation_b200/libfma_b200.so) contains none of this and refuses to run without a GPU.
//
// "Device memory" is host memory.  VMM is modelled with mmap so that the semantics the engine relies on are REAL:
//   cuMemAddressReserve -> PROT_NONE reservation; cuMemMap -> fresh zero pages at that VA (MAP_FIXED);
//   cuMemUnmap -> the pages are gone (PROT_NONE again; touching them faults) and only WHOLE mappings may be unmapped,
//   a range spanning several whole mappings is accepted, a sub-range is CUDA_ERROR_INVALID_VALUE (as the driver does,
//   scripts/vmm_span_probe.py); memory lives until unmap even if the handle was released right after cuMemMap.
// Streams execute eagerly (a copy has happened when cudaMemcpyAsync returns); events record wall-clock time.
// Fault injection: the Nth cuMemCreate (hostsim_fail_create_after), large cudaMemcpyAsync (hostsim_fail_memcpy_after) or call
// of a named VMM / stream / event / memset function (hostsim_fail_call_after) from now fails as if the device were out of memory.
#include <cuda.h>
#include <cuda_runtime.h>

#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <string>

namespace {
std::mutex g_mu;
struct Mapping { size_t bytes; unsigned long long handle; };
std::map<unsigned long long, size_t> g_reservations;          // va -> size
std::map<unsigned long long, Mapping> g_mappings;             // va -> mapping
std::map<unsigned long long, size_t> g_handles;               // handle -> size (alive until released AND unmapped)
std::map<unsigned long long, int> g_handle_fd;                // exportable handles (CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR): memfd behind them
std::set<unsigned long long> g_released;
std::atomic<unsigned long long> g_next_handle{1};
thread_local int tl_device = 0;
thread_local cudaError_t tl_last = cudaSuccess;
std::atomic<long> g_fail_create_after{-1};                    // fault injection: fail the Nth cuMemCreate from now
std::atomic<long> g_fail_memcpy_after{-1};                    // fault injection: fail the Nth large cudaMemcpyAsync from now
std::map<std::string, long> g_fail_call_after;                // fault injection by call name: fail its Nth call from now (g_mu)

// true when this call of `name` is the one hostsim_fail_call_after picked
bool injected(const char* name) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_fail_call_after.find(name);
    if (it == g_fail_call_after.end() || it->second < 0) return false;
    return it->second-- == 0;
}

int device_count() {
    const char* v = getenv("HOSTSIM_DEVICES");
    return v ? atoi(v) : 2;
}
double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
struct Event { double t_ms = 0; };
struct Stream { int dummy; };

CUresult simGetErrorString(CUresult r, const char** s) {
    *s = r == CUDA_SUCCESS ? "no error" : r == CUDA_ERROR_INVALID_VALUE ? "invalid argument" : r == CUDA_ERROR_OUT_OF_MEMORY ? "out of memory" : "hostsim error";
    return CUDA_SUCCESS;
}
CUresult simMemGetAllocationGranularity(size_t* g, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) {
    *g = 2u << 20;
    return CUDA_SUCCESS;
}
CUresult simMemAddressReserve(CUdeviceptr* ptr, size_t size, size_t, CUdeviceptr, unsigned long long) {
    if (injected("cuMemAddressReserve")) return CUDA_ERROR_OUT_OF_MEMORY;
    void* p = mmap(nullptr, size, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) return CUDA_ERROR_OUT_OF_MEMORY;
    // 2 MiB alignment like the driver: over-reserve is unnecessary for tests (mmap of GiB-sized ranges is 2 MiB aligned
    // only by luck), so align by re-mapping inside a padded reservation
    munmap(p, size);
    const size_t pad = size + (2u << 20);
    char* q = (char*)mmap(nullptr, pad, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (q == (char*)MAP_FAILED) return CUDA_ERROR_OUT_OF_MEMORY;
    char* a = (char*)(((uintptr_t)q + (2u << 20) - 1) & ~(uintptr_t)((2u << 20) - 1));
    if (a > q) munmap(q, a - q);
    if (a + size < q + pad) munmap(a + size, (q + pad) - (a + size));
    std::lock_guard<std::mutex> lk(g_mu);
    g_reservations[(unsigned long long)a] = size;
    *ptr = (CUdeviceptr)a;
    return CUDA_SUCCESS;
}
CUresult simMemAddressFree(CUdeviceptr ptr, size_t size) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_reservations.find(ptr);
    if (it == g_reservations.end() || it->second != size) return CUDA_ERROR_INVALID_VALUE;
    for (auto& m : g_mappings)
        if (m.first >= ptr && m.first < ptr + size) return CUDA_ERROR_INVALID_VALUE;  // still mapped inside
    munmap((void*)ptr, size);
    g_reservations.erase(it);
    return CUDA_SUCCESS;
}
CUresult simMemCreate(CUmemGenericAllocationHandle* h, size_t size, const CUmemAllocationProp* prop, unsigned long long) {
    if (!prop || prop->location.id < 0 || prop->location.id >= device_count() || size % (2u << 20)) return CUDA_ERROR_INVALID_VALUE;
    long f = g_fail_create_after.load();
    if (f >= 0 && g_fail_create_after.fetch_sub(1) == 0) return CUDA_ERROR_OUT_OF_MEMORY;
    std::lock_guard<std::mutex> lk(g_mu);
    *h = g_next_handle++;
    g_handles[*h] = size;
    if (prop->requestedHandleTypes == CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) {   // shareable: the "physical memory" is a memfd
        int fd = (int)syscall(SYS_memfd_create, "hostsim-vmm", 1u);
        if (fd < 0 || ftruncate(fd, (off_t)size) != 0) return CUDA_ERROR_OUT_OF_MEMORY;
        g_handle_fd[*h] = fd;
    }
    return CUDA_SUCCESS;
}
CUresult simMemExportToShareableHandle(void* out, CUmemGenericAllocationHandle h, CUmemAllocationHandleType t, unsigned long long) {
    if (injected("cuMemExportToShareableHandle")) return CUDA_ERROR_OUT_OF_MEMORY;
    std::lock_guard<std::mutex> lk(g_mu);
    if (t != CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR || !g_handle_fd.count(h)) return CUDA_ERROR_INVALID_VALUE;
    const int fd = dup(g_handle_fd[h]);
    if (fd < 0) return CUDA_ERROR_OUT_OF_MEMORY;
    *static_cast<int*>(out) = fd;
    return CUDA_SUCCESS;
}
CUresult simMemImportFromShareableHandle(CUmemGenericAllocationHandle* h, void* os_handle, CUmemAllocationHandleType t) {
    if (injected("cuMemImportFromShareableHandle")) return CUDA_ERROR_OUT_OF_MEMORY;
    if (t != CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) return CUDA_ERROR_INVALID_VALUE;
    const int fd = dup((int)(uintptr_t)os_handle);
    struct stat sb;
    if (fd < 0 || fstat(fd, &sb) != 0 || sb.st_size <= 0) return CUDA_ERROR_INVALID_VALUE;
    std::lock_guard<std::mutex> lk(g_mu);
    *h = g_next_handle++;
    g_handles[*h] = (size_t)sb.st_size;
    g_handle_fd[*h] = fd;
    return CUDA_SUCCESS;
}
static void drop_handle_locked(unsigned long long h) {
    g_handles.erase(h);
    g_released.erase(h);
    auto it = g_handle_fd.find(h);
    if (it != g_handle_fd.end()) { close(it->second); g_handle_fd.erase(it); }
}
CUresult simMemRelease(CUmemGenericAllocationHandle h) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_handles.count(h) || g_released.count(h)) return CUDA_ERROR_INVALID_VALUE;
    g_released.insert(h);
    bool mapped = false;
    for (auto& m : g_mappings) mapped |= m.second.handle == h;
    if (!mapped) drop_handle_locked(h);
    return CUDA_SUCCESS;
}
CUresult simMemMap(CUdeviceptr ptr, size_t size, size_t offset, CUmemGenericAllocationHandle h, unsigned long long) {
    if (injected("cuMemMap")) return CUDA_ERROR_OUT_OF_MEMORY;
    std::lock_guard<std::mutex> lk(g_mu);
    if (offset != 0 || !g_handles.count(h) || g_handles[h] != size) return CUDA_ERROR_INVALID_VALUE;
    bool inside = false;
    for (auto& r : g_reservations) inside |= ptr >= r.first && ptr + size <= r.first + r.second;
    if (!inside) return CUDA_ERROR_INVALID_VALUE;
    for (auto& m : g_mappings)
        if (ptr < m.first + m.second.bytes && m.first < ptr + size) return CUDA_ERROR_INVALID_VALUE;  // overlaps a live mapping
    void* p = g_handle_fd.count(h) ? mmap((void*)ptr, size, PROT_NONE, MAP_FIXED | MAP_SHARED, g_handle_fd[h], 0)   // shared with importers
                                   : mmap((void*)ptr, size, PROT_NONE, MAP_FIXED | MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) return CUDA_ERROR_OUT_OF_MEMORY;
    g_mappings[ptr] = Mapping{size, h};
    return CUDA_SUCCESS;
}
CUresult simMemSetAccess(CUdeviceptr ptr, size_t size, const CUmemAccessDesc* desc, size_t n) {
    if (injected("cuMemSetAccess")) return CUDA_ERROR_OUT_OF_MEMORY;
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_mappings.find(ptr);
    if (it == g_mappings.end() || it->second.bytes != size || !desc || !n) return CUDA_ERROR_INVALID_VALUE;
    if (mprotect((void*)ptr, size, PROT_READ | PROT_WRITE) != 0) return CUDA_ERROR_OUT_OF_MEMORY;   // accessible only after SetAccess
    return CUDA_SUCCESS;
}
CUresult simMemUnmap(CUdeviceptr ptr, size_t size) {
    std::lock_guard<std::mutex> lk(g_mu);
    // the range must be exactly a sequence of whole, adjacent mappings
    unsigned long long pos = ptr;
    auto it = g_mappings.find(ptr);
    while (pos < ptr + size) {
        if (it == g_mappings.end() || it->first != pos) return CUDA_ERROR_INVALID_VALUE;
        pos += it->second.bytes;
        ++it;
    }
    if (pos != ptr + size) return CUDA_ERROR_INVALID_VALUE;
    it = g_mappings.find(ptr);
    while (it != g_mappings.end() && it->first < ptr + size) {
        const unsigned long long h = it->second.handle;
        it = g_mappings.erase(it);
        if (g_released.count(h)) drop_handle_locked(h);   // released handle + last mapping gone: memory freed
    }
    mmap((void*)ptr, size, PROT_NONE, MAP_FIXED | MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);  // contents are gone
    return CUDA_SUCCESS;
}
}  // namespace

// test hooks (resolved with dlsym by the tests)
extern "C" __attribute__((visibility("default"))) unsigned long long hostsim_live_mapped_bytes() {
    std::lock_guard<std::mutex> lk(g_mu);
    unsigned long long s = 0;
    for (auto& m : g_mappings) s += m.second.bytes;
    return s;
}
extern "C" __attribute__((visibility("default"))) unsigned long long hostsim_live_handles() {
    std::lock_guard<std::mutex> lk(g_mu);
    return g_handles.size();
}
extern "C" __attribute__((visibility("default"))) unsigned long long hostsim_live_reservations() {
    std::lock_guard<std::mutex> lk(g_mu);
    return g_reservations.size();
}
extern "C" __attribute__((visibility("default"))) void hostsim_fail_create_after(long n) { g_fail_create_after.store(n); }
// fail the Nth call of `name` ("cuMemMap", "cudaEventCreateWithFlags", ...) from now; n < 0 disarms it
extern "C" __attribute__((visibility("default"))) void hostsim_fail_call_after(const char* name, long n) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_fail_call_after[name] = n;
}
extern "C" __attribute__((visibility("default"))) void hostsim_fail_memcpy_after(long n) { g_fail_memcpy_after.store(n); }
static std::atomic<long long> g_malloc_limit{0};  // > 0: cudaMalloc of more bytes fails ("HBM full": no staging ring)
extern "C" __attribute__((visibility("default"))) void hostsim_malloc_limit(long long bytes) { g_malloc_limit.store(bytes); }

extern "C" {
cudaError_t cudaGetDeviceCount(int* n) { *n = device_count(); return cudaSuccess; }
cudaError_t cudaSetDevice(int d) { if (d < 0 || d >= device_count()) return cudaErrorInvalidDevice; tl_device = d; return cudaSuccess; }
cudaError_t cudaGetDevice(int* d) { *d = tl_device; return cudaSuccess; }
cudaError_t cudaGetLastError(void) { cudaError_t e = tl_last; tl_last = cudaSuccess; return e; }
const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "hostsim runtime error"; }
cudaError_t cudaDeviceSynchronize(void) { return cudaSuccess; }
cudaError_t cudaDeviceGetPCIBusId(char* buf, int len, int dev) { snprintf(buf, len, "0000:%02x:00.0", 0x10 + dev); return cudaSuccess; }
cudaError_t cudaDeviceCanAccessPeer(int* can, int a, int b) { *can = (a != b && a < device_count() && b < device_count()); return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 148; return cudaSuccess; }
cudaError_t cudaMalloc(void** p, size_t n) { if (g_malloc_limit.load() > 0 && (long long)n > g_malloc_limit.load()) { *p = nullptr; tl_last = cudaErrorMemoryAllocation; return cudaErrorMemoryAllocation; } *p = aligned_alloc(2u << 20, ((n + (2u << 20) - 1) / (2u << 20)) * (2u << 20)); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { *p = aligned_alloc(4096, ((n + 4095) / 4096) * 4096); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaHostRegister(void*, size_t, unsigned) {
    if (getenv("HOSTSIM_FAIL_HOST_REGISTER")) { tl_last = cudaErrorInvalidValue; return cudaErrorInvalidValue; }   // "this mapping cannot be pinned"
    return cudaSuccess;
}
cudaError_t cudaHostUnregister(void*) { return cudaSuccess; }
cudaError_t cudaHostGetDevicePointer(void** d, void* h, unsigned) { *d = h; return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { if (injected("cudaStreamCreateWithFlags")) return tl_last = cudaErrorMemoryAllocation; *s = (cudaStream_t) new Stream(); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { delete (Stream*)s; return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t) new Event(); return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { if (injected("cudaEventCreateWithFlags")) return tl_last = cudaErrorMemoryAllocation; *e = (cudaEvent_t) new Event(); return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete (Event*)e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { ((Event*)e)->t_ms = now_ms(); return cudaSuccess; }
cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }   // eager streams: whatever was recorded has completed
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(((Event*)b)->t_ms - ((Event*)a)->t_ms); if (*ms <= 0) *ms = 1e-3f; return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) {
    if (n >= (1u << 20)) {  // only bulk copies (page tables and descriptors are small)
        long f = g_fail_memcpy_after.load();
        if (f >= 0 && g_fail_memcpy_after.fetch_sub(1) == 0) return cudaErrorLaunchFailure;
    }
    memcpy(d, s, n);
    return cudaSuccess;
}
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) {
    if (injected("cudaMemsetAsync")) return tl_last = cudaErrorLaunchFailure;   // (fma_image_verify clears its digest accumulators first)
    memset(d, v, n);
    return cudaSuccess;
}
cudaError_t cudaGetDriverEntryPoint(const char* name, void** fn, unsigned long long, cudaDriverEntryPointQueryResult* st) {
    struct { const char* n; void* f; } tab[] = {
        {"cuGetErrorString", (void*)simGetErrorString}, {"cuMemAddressReserve", (void*)simMemAddressReserve},
        {"cuMemAddressFree", (void*)simMemAddressFree}, {"cuMemCreate", (void*)simMemCreate}, {"cuMemRelease", (void*)simMemRelease},
        {"cuMemMap", (void*)simMemMap}, {"cuMemUnmap", (void*)simMemUnmap}, {"cuMemSetAccess", (void*)simMemSetAccess},
        {"cuMemGetAllocationGranularity", (void*)simMemGetAllocationGranularity},
        {"cuMemExportToShareableHandle", (void*)simMemExportToShareableHandle}, {"cuMemImportFromShareableHandle", (void*)simMemImportFromShareableHandle}};
    for (auto& t : tab)
        if (!strcmp(t.n, name)) { *fn = t.f; if (st) *st = cudaDriverEntryPointSuccess; return cudaSuccess; }
    if (st) *st = cudaDriverEntryPointSymbolNotFound;
    return cudaErrorInvalidValue;
}
}  // extern "C"
