// fma_pack_kernels.cu — sm_90a kernels of the PACKED host image (format: fma_codec.h).
//
//   K4p fma_k_pack_probe   per page: would it pack?  -> stored size (kPackedBytes or 2 MiB raw)
//   K4  fma_k_pack         gather + encode: scattered 2 MiB device pages -> packed pages in a contiguous ring slot
//   K5  fma_k_unpack       decode + scatter: packed pages in a ring slot -> the segments' device pages
//   K6  fma_k_unpack_digest decode + K3 digest of stored pages where they lie, writing no page (fma_image_verify)
//
// They take the place of K1/K2 (fma_kernels.cu) when the engine's `pack` option is on and the tier is host DRAM: the
// copy engines then move 0.758 x the bytes over PCIe Gen5, which is what bounds a wake (DESIGN.md §4).  The reference
// has no such stage (vllm:device_allocator/cumem.py:198-213 copies verbatim).
//
// Work decomposition: a page is cut into kParts = 8 parts of 512 tiles; one CTA (8 warps) per (page, part), grid-stride over
// the work items; a warp owns a 256-value tile (one 16-byte load per lane, 512 B per warp and instruction), four tiles in
// flight per warp.  Tile maximum by redux.sync.  K4: exception slots of a page come from ONE counter in global memory (the
// low 24 bits of the page descriptor's `state` word; the high 8 bits count finished parts and the part that finishes last
// writes the page header); each part stages its 512 B slice of the emax plane in shared memory.  K5: each part decodes its
// tiles and then patches the exceptions that fall into its value range.
// Why parts: with one CTA per page a ring slot's worth of pages (256-337) is only about two waves of H100's 132 SMs, each
// SM holding a fraction of the warps it could; 8 x as many, 8 x smaller work items fill the machine at every slot size.
// HBM-bound: reads 2 MiB, writes 1.52 MiB per page, all accesses whole 32-byte sectors except the (rare) exception patches.  All arithmetic is in fma_codec.h, shared with the CPU stand-in that the host-simulated engine
// tests run, and restated in oracle/fma_oracle.c.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "fma_codec.h"
#include "fma_kernels.h"

namespace {

using namespace fma_codec;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kU = 4;  // tiles in flight per warp

// Streaming loads / stores: the image is touched once, so nothing is allocated in L1.  FMA_CUDA_EMU (tests/cpp/cuda_emu/,
// test infrastructure) runs this file on a CPU and replaces the PTX by plain accesses; the launch macro likewise.
#if !defined(FMA_CUDA_EMU)
#define FMA_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint2 ld_stream8(const void* p) {
    uint2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ld_stream4(const void* p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream16(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream8(void* p, uint32_t a, uint32_t b) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void st_stream4(void* p, uint32_t a) {
    asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(a) : "memory");
}
#else
inline uint4 ld_stream16(const void* p) { uint4 v; memcpy(&v, p, 16); return v; }
inline uint2 ld_stream8(const void* p) { uint2 v; memcpy(&v, p, 8); return v; }
inline uint32_t ld_stream4(const void* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline void st_stream16(void* p, const uint4& v) { memcpy(p, &v, 16); }
inline void st_stream8(void* p, uint32_t a, uint32_t b) { uint32_t t[2] = {a, b}; memcpy(p, t, 8); }
inline void st_stream4(void* p, uint32_t a) { memcpy(p, &a, 4); }
#endif

// tile handled by (iteration, warp, u): consecutive warps take consecutive groups of kU tiles
__device__ __forceinline__ uint32_t tile_of(uint32_t it, uint32_t warp, uint32_t u) { return (it * kWarps + warp) * kU + u; }
constexpr uint32_t kIters = kTiles / (kWarps * kU);  // 128 iterations cover a page
constexpr uint32_t kParts = 8;                       // work items per page
constexpr uint32_t kItersPart = kIters / kParts;     // 16
constexpr uint32_t kTilesPart = kTiles / kParts;     // 512
constexpr uint32_t kValuesPart = kValues / kParts;   // 131072
constexpr uint32_t kCountMask = 0x00FFFFFFu;         // fma_k_pack_desc::state: exceptions so far | finished parts << 24

__device__ __forceinline__ void copy_part_raw(const unsigned char* src, unsigned char* dst, uint32_t part) {
    const uint32_t lo = part * (kPageBytes / kParts), hi = lo + kPageBytes / kParts;
    for (uint32_t o = lo + threadIdx.x * 16u; o < hi; o += kThreads * 16u * 4u) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = ld_stream16(src + o + u * kThreads * 16u);
#pragma unroll
        for (int u = 0; u < 4; ++u) st_stream16(dst + o + u * kThreads * 16u, v[u]);
    }
}

// ------------------------------------------------------------------------------------
// K4p: count the exceptions a page would need
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
fma_k_pack_probe(const uint64_t* __restrict__ src_tab, uint32_t n_pages, uint32_t* __restrict__ out_bytes) {
    __shared__ uint32_t s_nexc;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t p = blockIdx.x; p < n_pages; p += gridDim.x) {
        if (threadIdx.x == 0) s_nexc = 0;
        __syncthreads();
        const unsigned char* src = reinterpret_cast<const unsigned char*>(__ldg(src_tab + p));
        uint32_t mine = 0;
        for (uint32_t it = 0; it < kIters; ++it) {
            uint4 v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) v[u] = ld_stream16(src + tile_of(it, warp, u) * 512u + lane * 16u);
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
                const uint32_t emax = __reduce_max_sync(0xffffffffu, lane_max_exp(w));
                uint32_t lo, hi, nib, xm;
                lane_encode(w, emax, lo, hi, nib, xm);
                mine += __popc(xm);
            }
        }
        mine = __reduce_add_sync(0xffffffffu, mine);
        if (lane == 0 && mine) atomicAdd(&s_nexc, mine);
        __syncthreads();
        if (threadIdx.x == 0) out_bytes[p] = s_nexc <= kExcCap ? kPackedBytes : kPageBytes;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------
// K4: gather + encode
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
fma_k_pack(fma_k_pack_desc* __restrict__ descs, uint32_t n_pages, uint32_t* __restrict__ err) {
    __shared__ __align__(16) unsigned char s_emax[kTilesPart];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n_items = n_pages * kParts;
    for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const uint32_t p = item / kParts, part = item % kParts;
        const unsigned char* src = reinterpret_cast<const unsigned char*>(descs[p].src);
        unsigned char* dst = reinterpret_cast<unsigned char*>(descs[p].dst);
        if (descs[p].mode == FMA_K_PACK_RAW) {
            copy_part_raw(src, dst, part);
            continue;
        }
        uint32_t* state = &descs[p].state;   // zeroed by the host with the descriptor upload
        uint32_t* exc = reinterpret_cast<uint32_t*>(dst + kExcOff);
        for (uint32_t it = part * kItersPart; it < (part + 1) * kItersPart; ++it) {
            uint4 v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) v[u] = ld_stream16(src + tile_of(it, warp, u) * 512u + lane * 16u);
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const uint32_t tile = tile_of(it, warp, u);
                const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
                const uint32_t emax = __reduce_max_sync(0xffffffffu, lane_max_exp(w));
                uint32_t lo, hi, nib, xm;
                lane_encode(w, emax, lo, hi, nib, xm);
                st_stream8(dst + kSmOff + tile * kTileValues + lane * 8u, lo, hi);
                st_stream4(dst + kNibOff + tile * (kTileValues / 2) + lane * 4u, nib);
                if (lane == 0) s_emax[tile - part * kTilesPart] = (unsigned char)emax;
                while (xm) {  // rare: a value more than 13 binades below its tile's maximum
                    const uint32_t k = __ffs(xm) - 1;
                    xm &= xm - 1;
                    const uint32_t slot = atomicAdd(state, 1u) & kCountMask;
                    const uint32_t word = k < 2 ? v[u].x : k < 4 ? v[u].y : k < 6 ? v[u].z : v[u].w;  // no dynamic index
                    const uint32_t val = (word >> (16 * (k & 1))) & 0xFFFFu;
                    if (slot < kExcCap) exc[slot] = exc_entry(tile * kTileValues + lane * kLaneValues + k, exp_of(val));
                }
            }
        }
        __syncthreads();   // the part's emax slice is complete; every exception slot this CTA takes has been taken
        if (threadIdx.x < kTilesPart / 16)
            st_stream16(dst + kEmaxOff + part * kTilesPart + threadIdx.x * 16u, *reinterpret_cast<const uint4*>(s_emax + threadIdx.x * 16u));
        if (threadIdx.x == 0) {
            __threadfence();
            const uint32_t old = atomicAdd(state, 1u << 24);
            if ((old >> 24) == kParts - 1) {   // the last part of the page to finish writes the header
                const uint32_t n_exc = old & kCountMask;
                uint32_t* hdr = reinterpret_cast<uint32_t*>(dst + kHdrOff);
                hdr[0] = kMagic;
                hdr[1] = n_exc;
                if (n_exc > kExcCap) atomicAdd(err, 1u);  // the page changed after the probe: the caller fails the sleep
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------
// K5: decode + scatter
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 8)   // 32 registers: 8 CTAs (64 warps) per SM — K5 is latency-bound, occupancy is what it needs
fma_k_unpack(const fma_k_pack_desc* __restrict__ descs, uint32_t n_pages, uint32_t* __restrict__ err) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n_items = n_pages * kParts;
    for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const uint32_t p = item / kParts, part = item % kParts;
        const unsigned char* src = reinterpret_cast<const unsigned char*>(descs[p].src);
        unsigned char* dst = reinterpret_cast<unsigned char*>(descs[p].dst);
        if (descs[p].mode == FMA_K_PACK_RAW) {
            copy_part_raw(src, dst, part);
            continue;
        }
        const uint32_t magic = ld_stream4(src + kHdrOff), n_exc = ld_stream4(src + kHdrOff + 4);
        if (magic != kMagic || n_exc > kExcCap) {  // uniform per CTA; counted once per page
            if (threadIdx.x == 0 && part == 0) atomicAdd(err, 1u);
            continue;
        }
        for (uint32_t it = part * kItersPart; it < (part + 1) * kItersPart; ++it) {
            uint2 sm[kU];
            uint32_t nib[kU], emax[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const uint32_t tile = tile_of(it, warp, u);
                sm[u] = ld_stream8(src + kSmOff + tile * kTileValues + lane * 8u);
                nib[u] = ld_stream4(src + kNibOff + tile * (kTileValues / 2) + lane * 4u);
                emax[u] = __ldg(src + kEmaxOff + tile);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t w[4];
                lane_decode(sm[u].x, sm[u].y, nib[u], emax[u], w);
                st_stream16(dst + tile_of(it, warp, u) * 512u + lane * 16u, make_uint4(w[0], w[1], w[2], w[3]));
            }
        }
        __syncthreads();  // the part's values are written (block-visible) before the exceptions patch them
        const uint32_t* exc = reinterpret_cast<const uint32_t*>(src + kExcOff);
        for (uint32_t i = threadIdx.x; i < n_exc; i += kThreads) {   // every part scans the page's list (<= 8 KiB) for its own range
            const uint32_t entry = ld_stream4(exc + i);
            const uint32_t index = exc_index(entry);
            if (index / kValuesPart != part) continue;
            unsigned short* pv = reinterpret_cast<unsigned short*>(dst) + index;
            *pv = (unsigned short)apply_exception(__ldcg(pv), entry);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------
// K6: decode + digest.  The K3 digest (fma_kernels.cu) of the page K5 would write, without writing it: a sleeping image is
// checked where it lies, with nothing mapped.  K5's work items; each decoded 64-bit word goes straight into
// sum_j fmix64(w_j + (first_word + j + 1) * GOLDEN).  The exceptions of a part then correct the words they patch: a word's
// term as decoded (exponent 0) is replaced by its term with every patch of that word applied, as K5's patch loop leaves it.
// ------------------------------------------------------------------------------------
#define FMA_DIGEST_GOLDEN 0x9E3779B97F4A7C15ull
__device__ __forceinline__ uint64_t digest_mix(uint64_t z) {   // fmix64, as K3 and oracle/fma_oracle.c define it
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t digest_term(uint64_t w, uint64_t pos) { return digest_mix(w + (pos + 1) * FMA_DIGEST_GOLDEN); }

// word `wd` (4 values) of a coded page as lane_decode leaves it, before any exception patch
__device__ __forceinline__ uint64_t decoded_word(const unsigned char* src, uint32_t wd) {
    const uint32_t v0 = (wd * 4u) & ~7u;   // the lane's first value
    const uint2 sm = ld_stream8(src + kSmOff + v0);
    uint32_t w[4];
    lane_decode(sm.x, sm.y, ld_stream4(src + kNibOff + v0 / 2), __ldg(src + kEmaxOff + v0 / kTileValues), w);
    return (wd & 1) ? ((uint64_t)w[3] << 32 | w[2]) : ((uint64_t)w[1] << 32 | w[0]);
}

__global__ void __launch_bounds__(kThreads, 8)   // K5's shape: 32 registers, 8 CTAs per SM
fma_k_unpack_digest(const fma_k_page_desc* __restrict__ pages, uint32_t n_pages, unsigned long long* __restrict__ out,
                    uint32_t* __restrict__ err) {
    __shared__ uint32_t s_exc[kExcCap];          // the part's exception entries
    __shared__ uint32_t s_n;
    __shared__ unsigned long long s_sum[kWarps];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n_items = n_pages * kParts;
    for (uint32_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const uint32_t p = item / kParts, part = item % kParts;
        const unsigned char* src = reinterpret_cast<const unsigned char*>(pages[p].addr);
        const uint64_t first_word = pages[p].first_word;
        const uint32_t magic = ld_stream4(src + kHdrOff), n_exc = ld_stream4(src + kHdrOff + 4);
        if (magic != kMagic || n_exc > kExcCap) {  // uniform per CTA; counted once per page, and the page adds nothing
            if (threadIdx.x == 0 && part == 0) atomicAdd(err, 1u);
            continue;
        }
        if (threadIdx.x == 0) s_n = 0;
        uint64_t acc = 0;
        for (uint32_t it = part * kItersPart; it < (part + 1) * kItersPart; ++it) {
            uint2 sm[kU];
            uint32_t nib[kU], emax[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const uint32_t tile = tile_of(it, warp, u);
                sm[u] = ld_stream8(src + kSmOff + tile * kTileValues + lane * 8u);
                nib[u] = ld_stream4(src + kNibOff + tile * (kTileValues / 2) + lane * 4u);
                emax[u] = __ldg(src + kEmaxOff + tile);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                uint32_t w[4];
                lane_decode(sm[u].x, sm[u].y, nib[u], emax[u], w);
                const uint64_t j = first_word + tile_of(it, warp, u) * (kTileValues / 4) + lane * 2u;   // the lane's first word
                acc += digest_term((uint64_t)w[1] << 32 | w[0], j);
                acc += digest_term((uint64_t)w[3] << 32 | w[2], j + 1);
            }
        }
        __syncthreads();   // s_n is zero
        const uint32_t* exc = reinterpret_cast<const uint32_t*>(src + kExcOff);
        for (uint32_t i = threadIdx.x; i < n_exc; i += kThreads) {   // every part scans the page's list for its own range, as K5
            const uint32_t entry = ld_stream4(exc + i);
            if (exc_index(entry) / kValuesPart == part) s_exc[atomicAdd(&s_n, 1u)] = entry;
        }
        __syncthreads();
        const uint32_t m = s_n;
        for (uint32_t i = threadIdx.x; i < m; i += kThreads) {   // rare: one thread per patched word, the word's first entry here
            const uint32_t wd = exc_index(s_exc[i]) / 4u;
            bool first = true;
            for (uint32_t k = 0; k < i && first; ++k) first = exc_index(s_exc[k]) / 4u != wd;
            if (!first) continue;
            const uint64_t before = decoded_word(src, wd);
            uint64_t after = before;
            for (uint32_t k = i; k < m; ++k) {
                const uint32_t entry = s_exc[k], v = exc_index(entry);
                if (v / 4u != wd) continue;
                const uint32_t sh = 16u * (v & 3u);
                after = (after & ~(0xFFFFull << sh)) | (uint64_t)apply_exception((uint32_t)(after >> sh) & 0xFFFFu, entry) << sh;
            }
            acc += digest_term(after, first_word + wd) - digest_term(before, first_word + wd);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
        if (lane == 0) s_sum[warp] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long tot = 0;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) tot += s_sum[w];
            atomicAdd(out + p, tot);
        }
        __syncthreads();   // s_exc, s_n and s_sum are free for the next item
    }
}

int g_pack_sm_count = 0;
int pack_sm_count() {
    if (!g_pack_sm_count) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_pack_sm_count, cudaDevAttrMultiProcessorCount, dev);
        if (g_pack_sm_count <= 0) g_pack_sm_count = 132;  // H100 SXM
    }
    return g_pack_sm_count;
}
unsigned pack_grid(uint32_t n_items) {
    // Grid cap = SMs x CTAs per SM (grid-stride loop over pages beyond it).  8 CTAs of 256 threads fit an SM at 32 registers
    // (K4p, K5), 5 at K4's 48.  FMA_PACK_CTAS_PER_SM overrides it for sweeps (read once).
    static int per_sm = 0;
    if (!per_sm) {
        const char* v = getenv("FMA_PACK_CTAS_PER_SM");
        per_sm = v && atoi(v) > 0 ? atoi(v) : 8;
    }
    const uint64_t cap = (uint64_t)pack_sm_count() * (uint64_t)per_sm;
    return (unsigned)(n_items < cap ? n_items : cap);
}

}  // namespace

cudaError_t fma_k_launch_pack_probe(const uint64_t* src_tab, uint32_t n_pages, uint32_t* out_bytes, cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    FMA_LAUNCH(fma_k_pack_probe, pack_grid(n_pages), kThreads, 0, stream, src_tab, n_pages, out_bytes);
    return cudaGetLastError();
}

cudaError_t fma_k_launch_pack(fma_k_pack_desc* descs, uint32_t n_pages, uint32_t* err_count, cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    FMA_LAUNCH(fma_k_pack, pack_grid(n_pages * kParts), kThreads, 0, stream, descs, n_pages, err_count);
    return cudaGetLastError();
}

cudaError_t fma_k_launch_unpack(const fma_k_pack_desc* descs, uint32_t n_pages, uint32_t* err_count, cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    FMA_LAUNCH(fma_k_unpack, pack_grid(n_pages * kParts), kThreads, 0, stream, descs, n_pages, err_count);
    return cudaGetLastError();
}

cudaError_t fma_k_launch_unpack_digest(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t* out_zeroed, uint32_t* err_count,
                                       cudaStream_t stream) {
    if (n_pages == 0) return cudaSuccess;
    FMA_LAUNCH(fma_k_unpack_digest, pack_grid(n_pages * kParts), kThreads, 0, stream, pages, n_pages,
               reinterpret_cast<unsigned long long*>(out_zeroed), err_count);
    return cudaGetLastError();
}
