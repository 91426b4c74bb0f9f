// hostsim_kernels.cpp — host stand-ins for the kernel LAUNCH WRAPPERS (fma_kernels.h) so the engine's host logic can run
// without a GPU.  TEST INFRASTRUCTURE ONLY (see hostsim_cuda.cpp); the real kernels live in csrc/fma_kernels.cu.
// The arithmetic is the definition shared with oracle/fma_oracle.c (splitmix64 fill, fmix64 digest).
#include <cstring>

#include "fma_kernels.h"

static const uint64_t GOLDEN = 0x9E3779B97F4A7C15ull;
static inline uint64_t fmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

fma_k_tma_cfg fma_k_default_tma_cfg() { return fma_k_tma_cfg{16u << 10, 3, 2, 1}; }

cudaError_t fma_k_launch_page_copy(const uint64_t* src_tab, uint64_t src_base, const uint64_t* dst_tab, uint64_t dst_base, uint32_t n_pages,
                                   int variant, const fma_k_tma_cfg* cfg, cudaStream_t) {
    if (variant != FMA_K_VARIANT_TMA && variant != FMA_K_VARIANT_LDG) return cudaErrorInvalidValue;
    if (variant == FMA_K_VARIANT_TMA) {  // the real wrapper's clamps and rules, so both refuse the same shapes
        fma_k_tma_cfg c = cfg ? *cfg : fma_k_default_tma_cfg();
        if (!fma_k_tma_shape_fits(&c)) return cudaErrorInvalidValue;
    }
    for (uint32_t p = 0; p < n_pages; ++p) {
        const uint64_t s = src_tab ? src_tab[p] : src_base + (uint64_t)p * FMA_K_PAGE_BYTES;
        const uint64_t d = dst_tab ? dst_tab[p] : dst_base + (uint64_t)p * FMA_K_PAGE_BYTES;
        memcpy(reinterpret_cast<void*>(d), reinterpret_cast<const void*>(s), FMA_K_PAGE_BYTES);
    }
    return cudaSuccess;
}

cudaError_t fma_k_launch_page_digest(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t* out_zeroed, cudaStream_t) {
    for (uint32_t p = 0; p < n_pages; ++p) {
        const uint64_t* w = reinterpret_cast<const uint64_t*>(pages[p].addr);
        uint64_t acc = 0;
        for (uint64_t j = 0; j < FMA_K_PAGE_BYTES / 8; ++j) acc += fmix64(w[j] + (pages[p].first_word + j + 1) * GOLDEN);
        out_zeroed[p] += acc;
    }
    return cudaSuccess;
}

cudaError_t fma_k_launch_fill(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t seed, cudaStream_t) {
    for (uint32_t p = 0; p < n_pages; ++p) {
        uint64_t* w = reinterpret_cast<uint64_t*>(pages[p].addr);
        for (uint64_t j = 0; j < FMA_K_PAGE_BYTES / 8; ++j) w[j] = fmix64(seed + (pages[p].first_word + j + 1) * GOLDEN);
    }
    return cudaSuccess;
}

// ---- PACKED host image: K4p / K4 / K5 stand-ins.  Same per-lane arithmetic as the kernels (fma_codec.h), the warp
// and CTA structure replaced by loops: tile = 32 "lanes" of 8 values. ------------------------------------------
#include "fma_codec.h"
namespace fc = fma_codec;

static void load_lane(const unsigned char* src, uint32_t tile, uint32_t lane, uint32_t w[4]) { memcpy(w, src + tile * 512u + lane * 16u, 16); }

static uint32_t tile_emax(const unsigned char* src, uint32_t tile) {
    uint32_t emax = 0;
    for (uint32_t lane = 0; lane < 32; ++lane) {
        uint32_t w[4];
        load_lane(src, tile, lane, w);
        const uint32_t m = fc::lane_max_exp(w);
        emax = m > emax ? m : emax;
    }
    return emax;
}

cudaError_t fma_k_launch_pack_probe(const uint64_t* src_tab, uint32_t n_pages, uint32_t* out_bytes, cudaStream_t) {
    for (uint32_t p = 0; p < n_pages; ++p) {
        const unsigned char* src = reinterpret_cast<const unsigned char*>(src_tab[p]);
        uint32_t n_exc = 0;
        for (uint32_t tile = 0; tile < fc::kTiles; ++tile) {
            const uint32_t emax = tile_emax(src, tile);
            for (uint32_t lane = 0; lane < 32; ++lane) {
                uint32_t w[4], lo, hi, nib, xm;
                load_lane(src, tile, lane, w);
                fc::lane_encode(w, emax, lo, hi, nib, xm);
                n_exc += (uint32_t)__builtin_popcount(xm);
            }
        }
        out_bytes[p] = n_exc <= fc::kExcCap ? fc::kPackedBytes : fc::kPageBytes;
    }
    return cudaSuccess;
}

cudaError_t fma_k_launch_pack(fma_k_pack_desc* descs, uint32_t n_pages, uint32_t* err_count, cudaStream_t) {
    for (uint32_t p = 0; p < n_pages; ++p) {
        const unsigned char* src = reinterpret_cast<const unsigned char*>(descs[p].src);
        unsigned char* dst = reinterpret_cast<unsigned char*>(descs[p].dst);
        if (descs[p].mode == FMA_K_PACK_RAW) {
            memcpy(dst, src, FMA_K_PAGE_BYTES);
            continue;
        }
        uint32_t n_exc = 0;
        for (uint32_t tile = 0; tile < fc::kTiles; ++tile) {
            const uint32_t emax = tile_emax(src, tile);
            dst[fc::kEmaxOff + tile] = (unsigned char)emax;
            for (uint32_t lane = 0; lane < 32; ++lane) {
                uint32_t w[4], lo, hi, nib, xm;
                load_lane(src, tile, lane, w);
                fc::lane_encode(w, emax, lo, hi, nib, xm);
                memcpy(dst + fc::kSmOff + tile * fc::kTileValues + lane * 8u, &lo, 4);
                memcpy(dst + fc::kSmOff + tile * fc::kTileValues + lane * 8u + 4, &hi, 4);
                memcpy(dst + fc::kNibOff + tile * (fc::kTileValues / 2) + lane * 4u, &nib, 4);
                for (uint32_t k = 0; k < 8; ++k)
                    if (xm & (1u << k)) {
                        const uint32_t val = (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
                        const uint32_t entry = fc::exc_entry(tile * fc::kTileValues + lane * fc::kLaneValues + k, fc::exp_of(val));
                        if (n_exc < fc::kExcCap) memcpy(dst + fc::kExcOff + 4 * n_exc, &entry, 4);
                        ++n_exc;
                    }
            }
        }
        memcpy(dst + fc::kHdrOff, &fc::kMagic, 4);
        memcpy(dst + fc::kHdrOff + 4, &n_exc, 4);
        if (n_exc > fc::kExcCap) ++*err_count;
    }
    return cudaSuccess;
}

cudaError_t fma_k_launch_unpack(const fma_k_pack_desc* descs, uint32_t n_pages, uint32_t* err_count, cudaStream_t) {
    for (uint32_t p = 0; p < n_pages; ++p) {
        const unsigned char* src = reinterpret_cast<const unsigned char*>(descs[p].src);
        unsigned char* dst = reinterpret_cast<unsigned char*>(descs[p].dst);
        if (descs[p].mode == FMA_K_PACK_RAW) {
            memcpy(dst, src, FMA_K_PAGE_BYTES);
            continue;
        }
        uint32_t magic, n_exc;
        memcpy(&magic, src + fc::kHdrOff, 4);
        memcpy(&n_exc, src + fc::kHdrOff + 4, 4);
        if (magic != fc::kMagic || n_exc > fc::kExcCap) {
            ++*err_count;
            continue;
        }
        for (uint32_t tile = 0; tile < fc::kTiles; ++tile)
            for (uint32_t lane = 0; lane < 32; ++lane) {
                uint32_t lo, hi, nib, w[4];
                memcpy(&lo, src + fc::kSmOff + tile * fc::kTileValues + lane * 8u, 4);
                memcpy(&hi, src + fc::kSmOff + tile * fc::kTileValues + lane * 8u + 4, 4);
                memcpy(&nib, src + fc::kNibOff + tile * (fc::kTileValues / 2) + lane * 4u, 4);
                fc::lane_decode(lo, hi, nib, src[fc::kEmaxOff + tile], w);
                memcpy(dst + tile * 512u + lane * 16u, w, 16);
            }
        for (uint32_t i = 0; i < n_exc; ++i) {
            uint32_t entry;
            memcpy(&entry, src + fc::kExcOff + 4 * i, 4);
            uint16_t v;
            memcpy(&v, dst + 2 * fc::exc_index(entry), 2);
            v = (uint16_t)fc::apply_exception(v, entry);
            memcpy(dst + 2 * fc::exc_index(entry), &v, 2);
        }
    }
    return cudaSuccess;
}
