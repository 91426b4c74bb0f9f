// fma_kernels.h — internal C++ interface between the host engine and the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define FMA_K_PAGE_BYTES (2u << 20)
#define FMA_K_VARIANT_TMA 0
#define FMA_K_VARIANT_LDG 1

struct fma_k_page_desc {
    uint64_t addr;        // device address of a 2 MiB page
    uint64_t first_word;  // index of the page's first 64-bit word inside its segment / stream
};

struct fma_k_tma_cfg {
    uint32_t tile_bytes;   // bulk-copy size; divides 2 MiB, multiple of 16
    uint32_t stages;       // smem buffers per pipe (2..8)
    uint32_t pipes;        // warps (independent pipelines) per CTA (1..4)
    uint32_t ctas_per_sm;  // grid = SMs * ctas_per_sm (persistent, tile-strided)
};

fma_k_tma_cfg fma_k_default_tma_cfg();

// The shape rules of the TMA page copy, shared by its launch wrapper and by the engine, which checks a shape before a
// sleep or wake starts: stages are clamped to 2..8, pipes to 1..4 and ctas_per_sm to >= 1; the tile must be at least 1 KiB,
// a multiple of 16 and divide the 2 MiB page, and pipes x stages x tile (+ 128 B of alignment slack) must fit the 227 KiB
// of shared memory a block may use.  Clamps *c in place; false = the shape cannot run.
inline bool fma_k_tma_shape_fits(fma_k_tma_cfg* c) {
    if (c->stages < 2) c->stages = 2;
    if (c->stages > 8) c->stages = 8;
    if (c->pipes < 1) c->pipes = 1;
    if (c->pipes > 4) c->pipes = 4;
    if (c->ctas_per_sm < 1) c->ctas_per_sm = 1;
    if (c->tile_bytes < 1024 || (FMA_K_PAGE_BYTES % c->tile_bytes) != 0 || (c->tile_bytes % 16) != 0) return false;
    return (uint64_t)c->pipes * c->stages * c->tile_bytes + 128 <= 227u * 1024u;
}

// K1/K2: tables are DEVICE arrays of device addresses (nullptr => contiguous from *_base).
cudaError_t fma_k_launch_page_copy(const uint64_t* src_tab, uint64_t src_base, const uint64_t* dst_tab,
                                   uint64_t dst_base, uint32_t n_pages, int variant, const fma_k_tma_cfg* cfg,
                                   cudaStream_t stream);
// K3: out must be zeroed (n_pages x u64).
cudaError_t fma_k_launch_page_digest(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t* out_zeroed,
                                     cudaStream_t stream);
// K0
cudaError_t fma_k_launch_fill(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t seed, cudaStream_t stream);

// ---- PACKED host image (fma_pack_kernels.cu; format in fma_codec.h) -------------------------------------------
#define FMA_K_PACK_RAW 0     // page stored verbatim (2 MiB)
#define FMA_K_PACK_BF16 1    // page stored in the "FMP4" code (fma_codec::kPackedBytes)
#define FMA_K_PACKED_PAGE_BYTES ((3u << 19) + (16u << 10))

struct fma_k_pack_desc {
    uint64_t src;   // K4: device address of the 2 MiB page          K5: address of the stored page (ring slot / store alias)
    uint64_t dst;   // K4: where the stored page goes (ring slot)    K5: device address of the 2 MiB page
    uint32_t mode;  // FMA_K_PACK_*
    uint32_t state; // K4 scratch, MUST be 0 at launch: exceptions taken so far (low 24 bits) | finished parts of the page << 24
};

// K4p: out_bytes[p] = stored size of page p (FMA_K_PACKED_PAGE_BYTES, or FMA_K_PAGE_BYTES when it has to stay raw)
cudaError_t fma_k_launch_pack_probe(const uint64_t* src_tab, uint32_t n_pages, uint32_t* out_bytes, cudaStream_t stream);
// K4 / K5: *err_count (device, zeroed by the caller) counts pages that could not be coded / decoded
cudaError_t fma_k_launch_pack(fma_k_pack_desc* descs, uint32_t n_pages, uint32_t* err_count, cudaStream_t stream);   // writes descs[].state
cudaError_t fma_k_launch_unpack(const fma_k_pack_desc* descs, uint32_t n_pages, uint32_t* err_count, cudaStream_t stream);
// K6: out_zeroed[p] += the K3 digest of the page K5 would decode from the coded page pages[p].addr (first_word as for K3); nothing
// else is written.  *err_count counts malformed pages as K5 does, and such a page adds nothing to its accumulator.
// Declared weak: the engine's host translation units are also built without the kernels, against stand-ins for the launch
// wrappers (a host simulation), and fma_image_verify refuses a PACKED image when this wrapper is absent.
__attribute__((weak)) cudaError_t fma_k_launch_unpack_digest(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t* out_zeroed,
                                                             uint32_t* err_count, cudaStream_t stream);
