// hostsim_verify_kernels.cpp — host stand-in for the K6 launch wrapper (fma_k_launch_unpack_digest), linked next to
// hostsim_kernels.cpp when the host-simulated engine runs fma_image_verify.  TEST INFRASTRUCTURE ONLY; the kernel lives in
// csrc/fma_pack_kernels.cu.  It decodes a stored page as the K5 stand-in does and digests the result as the K3 stand-in does.
#include <cstring>
#include <vector>

#include "fma_codec.h"
#include "fma_kernels.h"

namespace fc = fma_codec;

static inline uint64_t fmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

cudaError_t fma_k_launch_unpack_digest(const fma_k_page_desc* pages, uint32_t n_pages, uint64_t* out_zeroed, uint32_t* err_count, cudaStream_t) {
    std::vector<uint16_t> v(fc::kValues);
    for (uint32_t p = 0; p < n_pages; ++p) {
        const unsigned char* src = reinterpret_cast<const unsigned char*>(pages[p].addr);
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
                memcpy(v.data() + tile * fc::kTileValues + lane * 8u, w, 16);
            }
        for (uint32_t i = 0; i < n_exc; ++i) {
            uint32_t entry;
            memcpy(&entry, src + fc::kExcOff + 4 * i, 4);
            v[fc::exc_index(entry)] = (uint16_t)fc::apply_exception(v[fc::exc_index(entry)], entry);
        }
        uint64_t acc = 0;
        for (uint64_t j = 0; j < fc::kValues / 4; ++j) {
            uint64_t w;
            memcpy(&w, v.data() + 4 * j, 8);
            acc += fmix64(w + (pages[p].first_word + j + 1) * 0x9E3779B97F4A7C15ull);
        }
        out_zeroed[p] += acc;
    }
    return cudaSuccess;
}
