// fma_kernels.cu — sm_90a kernels of the sleep/wake weight-movement path.
//
//   K0  fma_k_fill         counter-based splitmix64 fill of pages (synthetic weight blobs)
//   K1/K2 fma_k_page_copy_* page-table driven gather / scatter of 2 MiB VMM pages:
//        *_tma : one elected thread per warp drives a multi-stage ring of
//                cp.async.bulk global->shared (mbarrier complete_tx) and
//                cp.async.bulk shared->global (bulk_group) copies  (SASS: UBLKCP)
//        *_ldg : 128-bit LDG.NC / STG.CS grid-stride copy (comparison variant)
//   K3  fma_k_page_digest  position-sensitive 64-bit digest, exact integer arithmetic
//
// There is no incumbent kernel in the reference: vLLM's sleep/wake moves bytes with one
// blocking cudaMemcpy per segment (vllm:device_allocator/cumem.py:198-213,237-249 via
// vllm:distributed/device_communicators/cuda_wrapper.py:168-173).  These kernels exist so
// that (a) many scattered segments become ONE contiguous stream for the copy engines,
// (b) the peer-HBM tier moves pages over NVLink from SMs, (c) bit-identity is provable on
// the device.  All work is HBM/NVLink/PCIe-bound byte movement; no tensor cores.
//
// Definitions that must stay bit-exact with oracle/fma_oracle.c: splitmix64, digest.
#include <cuda_runtime.h>
#include <stdint.h>
#include "fma_kernels.h"

#define FMA_GOLDEN 0x9E3779B97F4A7C15ull
// FMA_CUDA_EMU (tests/cpp/cuda_emu/, test infrastructure) runs this file's kernels on a CPU model of the execution hierarchy;
// it brings its own FMA_LAUNCH and replaces the PTX wrappers below.  The nvcc build is unaffected (same SASS).
#if !defined(FMA_CUDA_EMU) && !defined(FMA_LAUNCH)
#define FMA_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

namespace {

__device__ __forceinline__ uint64_t fmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

#if !defined(FMA_CUDA_EMU)
// ------------------------------------------------------------------------------------
// PTX wrappers (sm_90 bulk async copy + mbarrier)
// ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// global -> shared, completion signalled on an mbarrier (TMA bulk load; SASS UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar,
                                         uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
// shared -> global, tracked by the thread's bulk async-group (TMA bulk store)
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes, uint64_t pol) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst),
                 "r"(src_smem), "r"(bytes), "l"(pol) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
#else  // FMA_CUDA_EMU: the same names on the CPU execution model (tests/cpp/cuda_emu/cuda_emu.h, test infrastructure)
inline uint32_t smem_u32(const void* p) { return fma_emu::handle_of(p); }
inline void mbar_init(uint32_t bar, uint32_t count) { fma_emu::mbar_init(static_cast<uint64_t*>(fma_emu::ptr_of(bar)), count); }
inline void mbar_expect_tx(uint32_t bar, uint32_t bytes) { fma_emu::mbar_expect_tx(static_cast<uint64_t*>(fma_emu::ptr_of(bar)), bytes); }
inline void mbar_wait(uint32_t bar, uint32_t parity) { fma_emu::mbar_wait(static_cast<uint64_t*>(fma_emu::ptr_of(bar)), parity); }
inline uint64_t policy_evict_first() { return 0; }
inline void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t) {
    fma_emu::bulk_g2s(fma_emu::ptr_of(dst_smem), src, bytes, static_cast<uint64_t*>(fma_emu::ptr_of(bar)));
}
inline void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes, uint64_t) { fma_emu::bulk_s2g(dst, fma_emu::ptr_of(src_smem), bytes); }
inline void bulk_commit() { fma_emu::bulk_commit(); }
template <int N> inline void bulk_wait_read() { fma_emu::bulk_wait_keep(N); }
inline void bulk_wait_all() { fma_emu::bulk_wait_keep(0); }
inline void fence_proxy_async() {}
inline void fence_mbar_init() {}
#endif

__device__ __forceinline__ uint64_t page_addr(const uint64_t* __restrict__ tab, uint64_t base, uint32_t p) {
    return tab ? __ldg(tab + p) : base + (uint64_t)p * FMA_K_PAGE_BYTES;
}

// ------------------------------------------------------------------------------------
// K1/K2 (TMA variant).  Work unit = tile of `tile_bytes` (divides the 2 MiB page), so a
// tile never straddles two pages and its source/destination are one table lookup each.
// Each warp's lane 0 is an independent "pipe" owning `stages` smem buffers: tiles
// q, q+Q, q+2Q ... (Q = total pipes), so concurrently running pipes stream adjacent tiles.
//   iteration i:  wait full[s]  ->  bulk store tile i  ->  commit
//                 wait until store i-1 has finished READING smem  ->  refill its buffer with
//                 tile i-1+stages.   stages-1 loads stay in flight per pipe.
// ------------------------------------------------------------------------------------
constexpr int kMaxStages = 8;
constexpr int kMaxPipes = 4;  // warps per CTA

__global__ void __launch_bounds__(32 * kMaxPipes, 1)
fma_k_page_copy_tma(const uint64_t* __restrict__ src_tab, uint64_t src_base, const uint64_t* __restrict__ dst_tab,
                    uint64_t dst_base, uint32_t n_pages, uint32_t tile_bytes, uint32_t stages) {
#if !defined(FMA_CUDA_EMU)
    extern __shared__ __align__(128) unsigned char smem_raw[];
#else
    alignas(128) static unsigned char smem_raw[227u * 1024u];  // CTAs run one after the other on the CPU model
#endif
    __shared__ __align__(8) uint64_t full_bar[kMaxPipes][kMaxStages];

    if ((threadIdx.x & 31) != 0) return;  // one elected thread per warp; no block-wide sync is used below
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t pipes_per_cta = blockDim.x >> 5;
    const uint64_t q = (uint64_t)blockIdx.x * pipes_per_cta + warp;
    const uint64_t Q = (uint64_t)gridDim.x * pipes_per_cta;
    const uint32_t tiles_per_page = FMA_K_PAGE_BYTES / tile_bytes;
    const uint64_t n_tiles = (uint64_t)n_pages * tiles_per_page;
    if (q >= n_tiles) return;
    const uint64_t n_my = (n_tiles - q + Q - 1) / Q;

    // dynamic smem base is only guaranteed 16 B aligned by the ABI; align to 128 B ourselves
    uint32_t smem_base = (smem_u32(smem_raw) + 127u) & ~127u;
    const uint32_t my_smem = smem_base + warp * stages * tile_bytes;
    for (uint32_t s = 0; s < stages; ++s) mbar_init(smem_u32(&full_bar[warp][s]), 1);
    fence_mbar_init();
    fence_proxy_async();
    const uint64_t pol = policy_evict_first();

    auto tile_src = [&](uint64_t i) -> const void* {
        const uint64_t t = q + i * Q;
        const uint32_t p = (uint32_t)(t / tiles_per_page);
        const uint32_t o = (uint32_t)(t % tiles_per_page) * tile_bytes;
        return reinterpret_cast<const void*>(page_addr(src_tab, src_base, p) + o);
    };
    auto tile_dst = [&](uint64_t i) -> void* {
        const uint64_t t = q + i * Q;
        const uint32_t p = (uint32_t)(t / tiles_per_page);
        const uint32_t o = (uint32_t)(t % tiles_per_page) * tile_bytes;
        return reinterpret_cast<void*>(page_addr(dst_tab, dst_base, p) + o);
    };
    auto issue_load = [&](uint64_t i) {
        const uint32_t s = (uint32_t)(i % stages);
        const uint32_t bar = smem_u32(&full_bar[warp][s]);
        mbar_expect_tx(bar, tile_bytes);
        bulk_g2s(my_smem + s * tile_bytes, tile_src(i), tile_bytes, bar, pol);
    };

    const uint64_t pro = n_my < stages ? n_my : stages;
    for (uint64_t i = 0; i < pro; ++i) issue_load(i);

    for (uint64_t i = 0; i < n_my; ++i) {
        const uint32_t s = (uint32_t)(i % stages);
        mbar_wait(smem_u32(&full_bar[warp][s]), (uint32_t)((i / stages) & 1));
        bulk_s2g(tile_dst(i), my_smem + s * tile_bytes, tile_bytes, pol);
        bulk_commit();
        if (i >= 1 && (i - 1) + stages < n_my) {
            bulk_wait_read<1>();  // every group but the newest has finished reading its smem buffer
            issue_load(i - 1 + stages);
        }
    }
    bulk_wait_all();  // stores fully performed before the CTA (and its smem) retires
}

// ------------------------------------------------------------------------------------
// K1/K2 (LDG variant): 256 threads, each moves 2 x UNROLL x 16 B per tile with streaming hints.
// ------------------------------------------------------------------------------------
// 128-bit streaming load/store (LDG.E.128 / STG.E.128, the widest global access sm_90 has): vector v of a tile
// is at byte 16 * v, thread t takes v = t, t + 256, ... so every warp instruction covers 512 contiguous bytes.
// Nothing is allocated in L1, and the L2 policy marks the lines evict-first: the data is touched once.
struct __align__(16) u64x2 { uint64_t a, b; };
#if !defined(FMA_CUDA_EMU)
__device__ __forceinline__ u64x2 ld_stream(const u64x2* p, uint64_t pol) {
    u64x2 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;"
                 : "=l"(v.a), "=l"(v.b) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_stream(u64x2* p, const u64x2& v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.u64 [%0], {%1,%2}, %3;" ::"l"(p), "l"(v.a), "l"(v.b),
                 "l"(pol) : "memory");
}
#else
inline u64x2 ld_stream(const u64x2* p, uint64_t) { return *p; }
inline void st_stream(u64x2* p, const u64x2& v, uint64_t) { *p = v; }
#endif

template <int UNROLL>
__global__ void __launch_bounds__(256)
fma_k_page_copy_ldg(const uint64_t* __restrict__ src_tab, uint64_t src_base, const uint64_t* __restrict__ dst_tab,
                    uint64_t dst_base, uint32_t n_pages) {
    constexpr int kVecs = 2 * UNROLL;  // 16-byte vectors per thread and tile
    constexpr uint32_t kTile = 256u * 16u * kVecs;
    constexpr uint32_t kTilesPerPage = FMA_K_PAGE_BYTES / kTile;
    const uint64_t pol = policy_evict_first();
    const uint64_t n_tiles = (uint64_t)n_pages * kTilesPerPage;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const uint32_t p = (uint32_t)(t / kTilesPerPage);
        const uint32_t o = (uint32_t)(t % kTilesPerPage) * kTile;
        const u64x2* __restrict__ s = reinterpret_cast<const u64x2*>(page_addr(src_tab, src_base, p) + o) + threadIdx.x;
        u64x2* __restrict__ d = reinterpret_cast<u64x2*>(page_addr(dst_tab, dst_base, p) + o) + threadIdx.x;
        u64x2 v[kVecs];
#pragma unroll
        for (int u = 0; u < kVecs; ++u) v[u] = ld_stream(s + u * 256, pol);
#pragma unroll
        for (int u = 0; u < kVecs; ++u) st_stream(d + u * 256, v[u], pol);
    }
}

// ------------------------------------------------------------------------------------
// K3: per-page digest.  digest(page p) = sum_j fmix64(w_j + (first_word[p] + j + 1) * GOLDEN)
// over the page's 2^18 little-endian 64-bit words; sums are mod 2^64 so any reduction order
// is exact.  out[p] must be zero on entry (atomicAdd accumulation, one per CTA-tile).
// ------------------------------------------------------------------------------------
constexpr int kDigVecs = 8;  // 16-byte vectors per thread and tile
__global__ void __launch_bounds__(256)
fma_k_page_digest(const fma_k_page_desc* __restrict__ pages, uint32_t n_pages, unsigned long long* __restrict__ out) {
    constexpr uint32_t kTile = 256u * 16u * kDigVecs;  // 32 KiB
    constexpr uint32_t kTilesPerPage = FMA_K_PAGE_BYTES / kTile;
    __shared__ unsigned long long warp_sums[8];
    const uint64_t pol = policy_evict_first();
    const uint64_t n_tiles = (uint64_t)n_pages * kTilesPerPage;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const uint32_t p = (uint32_t)(t / kTilesPerPage);
        const uint32_t o = (uint32_t)(t % kTilesPerPage) * kTile;
        const fma_k_page_desc pd = pages[p];
        const u64x2* __restrict__ s = reinterpret_cast<const u64x2*>(pd.addr + o) + threadIdx.x;
        u64x2 v[kDigVecs];
#pragma unroll
        for (int u = 0; u < kDigVecs; ++u) v[u] = ld_stream(s + u * 256, pol);
        uint64_t acc = 0;
#pragma unroll
        for (int u = 0; u < kDigVecs; ++u) {
            const uint64_t j = pd.first_word + (uint64_t)(o / 8) + (uint64_t)(u * 256 + threadIdx.x) * 2;
            acc += fmix64(v[u].a + (j + 1) * FMA_GOLDEN);
            acc += fmix64(v[u].b + (j + 2) * FMA_GOLDEN);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
        if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long tot = 0;
#pragma unroll
            for (int w = 0; w < 8; ++w) tot += warp_sums[w];
            atomicAdd(out + p, tot);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------
// K0: fill.  word j of page p = splitmix64(seed, first_word[p] + j) = fmix64(seed + (k+1)*GOLDEN)
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fma_k_fill(const fma_k_page_desc* __restrict__ pages, uint32_t n_pages, uint64_t seed) {
    constexpr int kVecs = 8;  // 16-byte vectors per thread and tile
    constexpr uint32_t kTile = 256u * 16u * kVecs;
    constexpr uint32_t kTilesPerPage = FMA_K_PAGE_BYTES / kTile;
    const uint64_t pol = policy_evict_first();
    const uint64_t n_tiles = (uint64_t)n_pages * kTilesPerPage;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const uint32_t p = (uint32_t)(t / kTilesPerPage);
        const uint32_t o = (uint32_t)(t % kTilesPerPage) * kTile;
        const fma_k_page_desc pd = pages[p];
        u64x2* __restrict__ d = reinterpret_cast<u64x2*>(pd.addr + o) + threadIdx.x;
#pragma unroll
        for (int u = 0; u < kVecs; ++u) {
            const uint64_t k = pd.first_word + (uint64_t)(o / 8) + (uint64_t)(u * 256 + threadIdx.x) * 2;
            u64x2 v;
            v.a = fmix64(seed + (k + 1) * FMA_GOLDEN);
            v.b = fmix64(seed + (k + 2) * FMA_GOLDEN);
            st_stream(d + u * 256, v, pol);
        }
    }
}

int g_sm_count = 0;

int sm_count() {
    if (!g_sm_count) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
        if (g_sm_count <= 0) g_sm_count = 132;  // H100 SXM
    }
    return g_sm_count;
}

}  // namespace

// ------------------------------------------------------------------------------------
// launch wrappers (internal C++ interface used by fma_engine.cu)
// ------------------------------------------------------------------------------------
fma_k_tma_cfg fma_k_default_tma_cfg() {
    // 2 pipes x 3 stages x 16 KiB = 96 KiB of smem per SM, 64 KiB of loads in flight: on H100 (132 SMs,
    // 3.35 TB/s HBM3) that is about 8.4 MiB in flight against the ~2.5 MiB that bandwidth x ~0.7 us of DRAM
    // latency needs, with the smem well inside the 227 KiB a block may use.
    fma_k_tma_cfg c;
    c.tile_bytes = 16u << 10;
    c.stages = 3;
    c.pipes = 2;
    c.ctas_per_sm = 1;
    return c;
}

cudaError_t fma_k_launch_page_copy(const uint64_t* src_tab, uint64_t src_base, const uint64_t* dst_tab,
                                   uint64_t dst_base, uint32_t n_pages, int variant, const fma_k_tma_cfg* cfg_in,
                                   cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    if (variant == FMA_K_VARIANT_TMA) {
        fma_k_tma_cfg c = cfg_in ? *cfg_in : fma_k_default_tma_cfg();
        if (!fma_k_tma_shape_fits(&c)) return cudaErrorInvalidValue;
        static_assert(kMaxStages == 8 && kMaxPipes == 4, "fma_k_tma_shape_fits clamps to these");
        const size_t smem = (size_t)c.pipes * c.stages * c.tile_bytes + 128;
#if !defined(FMA_CUDA_EMU)
        cudaError_t err = cudaFuncSetAttribute(fma_k_page_copy_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return err;
#endif
        const uint64_t n_tiles = (uint64_t)n_pages * (FMA_K_PAGE_BYTES / c.tile_bytes);
        uint64_t grid = (uint64_t)sm_count() * c.ctas_per_sm;
        const uint64_t need = (n_tiles + c.pipes - 1) / c.pipes;
        if (grid > need) grid = need;
        FMA_LAUNCH(fma_k_page_copy_tma, (unsigned)grid, 32 * c.pipes, smem, stream, src_tab, src_base, dst_tab, dst_base, n_pages,
                   c.tile_bytes, c.stages);
        return cudaGetLastError();
    } else if (variant == FMA_K_VARIANT_LDG) {
        constexpr int U = 4;
        const uint64_t n_tiles = (uint64_t)n_pages * (FMA_K_PAGE_BYTES / (256u * 32u * U));
        uint64_t grid = (uint64_t)sm_count() * 4;
        if (grid > n_tiles) grid = n_tiles;
        FMA_LAUNCH(fma_k_page_copy_ldg<U>, (unsigned)grid, 256, 0, stream, src_tab, src_base, dst_tab, dst_base, n_pages);
        return cudaGetLastError();
    }
    return cudaErrorInvalidValue;
}

cudaError_t fma_k_launch_page_digest(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t* out_zeroed,
                                     cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    const uint64_t n_tiles = (uint64_t)n_pages * (FMA_K_PAGE_BYTES / (256u * 16u * kDigVecs));
    uint64_t grid = (uint64_t)sm_count() * 8;
    if (grid > n_tiles) grid = n_tiles;
    FMA_LAUNCH(fma_k_page_digest, (unsigned)grid, 256, 0, stream, pages, n_pages, reinterpret_cast<unsigned long long*>(out_zeroed));
    return cudaGetLastError();
}

cudaError_t fma_k_launch_fill(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t seed, cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    const uint64_t n_tiles = (uint64_t)n_pages * (FMA_K_PAGE_BYTES / (256u * 32u * 4));
    uint64_t grid = (uint64_t)sm_count() * 8;
    if (grid > n_tiles) grid = n_tiles;
    FMA_LAUNCH(fma_k_fill, (unsigned)grid, 256, 0, stream, pages, n_pages, seed);
    return cudaGetLastError();
}
