// Runs the ACTUAL kernel source csrc/fma_kernels.cu — K0 fill, K1/K2 page copy (the TMA pipeline and the LDG variant), K3
// digest — on the CPU execution model of cuda_emu.h (lazy async proxy included) and checks it against the oracle
// (oracle/fma_oracle.c).  These kernels are tested on the H100 (tests -m gpu); this adds
// what the GPU cannot show cheaply: ThreadSanitizer over their shared-memory traffic, and a standing CPU regression test
// of the exact source that ships.  Built by tests/test_kernels_emulated.py with g++ -DFMA_CUDA_EMU -include cuda_emu.h.
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

extern "C" cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
extern "C" cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 3; return cudaSuccess; }  // 3 "SMs"
extern "C" cudaError_t cudaGetLastError(void) { return cudaSuccess; }

#include "../../../llm-d-fast-model-actuation_b200/csrc/fma_kernels.cu"

extern "C" {
void fma_oracle_fill(uint64_t* dst, uint64_t n_words, uint64_t seed, uint64_t first_word);
uint64_t fma_oracle_digest(const void* src, uint64_t n_bytes, uint64_t first_word);
}

static const size_t PAGE = FMA_K_PAGE_BYTES;

int main() {
    const uint32_t n = 5;
    std::vector<unsigned char> a(n * PAGE), b(n * PAGE, 0xCD), c(n * PAGE, 0xEF), want(n * PAGE);
    std::vector<fma_k_page_desc> desc(n);
    const uint64_t seed = 0xDEADBEEF;
    // K0: pages filled in a scattered order with arbitrary stream positions == oracle fill
    const uint64_t first[n] = {0, 1, (1ull << 40) + 12345, 7 * (PAGE / 8), 99};
    for (uint32_t p = 0; p < n; ++p) {
        desc[p] = fma_k_page_desc{(uint64_t)(uintptr_t)(a.data() + ((p * 2) % n) * PAGE), first[p]};
        fma_oracle_fill(reinterpret_cast<uint64_t*>(want.data() + ((p * 2) % n) * PAGE), PAGE / 8, seed, first[p]);
    }
    assert(fma_k_launch_fill(desc.data(), n, seed, nullptr) == cudaSuccess);
    if (a != want) { fprintf(stderr, "K0 fill differs from the oracle\n"); return 1; }

    // K3: per-page digests (accumulated with atomicAdd into zeroed slots) == oracle digest with the page's word offset
    std::vector<uint64_t> dig(n, 0);
    assert(fma_k_launch_page_digest(desc.data(), n, dig.data(), nullptr) == cudaSuccess);
    for (uint32_t p = 0; p < n; ++p)
        if (dig[p] != fma_oracle_digest(reinterpret_cast<const void*>(desc[p].addr), PAGE, first[p])) { fprintf(stderr, "K3 digest of page %u differs\n", p); return 1; }

    // K1/K2: gather permuted pages into a contiguous image, scatter it back; LDG variant and several TMA pipeline shapes
    std::vector<uint64_t> src_tab(n), dst_tab(n);
    const uint32_t perm[n] = {3, 0, 4, 1, 2};
    for (uint32_t p = 0; p < n; ++p) src_tab[p] = (uint64_t)(uintptr_t)(a.data() + perm[p] * PAGE);
    struct Cfg { int variant; fma_k_tma_cfg c; };
    const Cfg cfgs[] = {{FMA_K_VARIANT_LDG, {0, 0, 0, 0}}, {FMA_K_VARIANT_TMA, {16u << 10, 3, 2, 1}}, {FMA_K_VARIANT_TMA, {32u << 10, 3, 2, 1}},
                        {FMA_K_VARIANT_TMA, {8u << 10, 2, 1, 1}}, {FMA_K_VARIANT_TMA, {64u << 10, 3, 1, 1}}, {FMA_K_VARIANT_TMA, {8u << 10, 3, 4, 2}}};
    for (const Cfg& k : cfgs) {
        std::fill(b.begin(), b.end(), 0xCD);
        assert(fma_k_launch_page_copy(src_tab.data(), 0, nullptr, (uint64_t)(uintptr_t)b.data(), n, k.variant, k.variant == FMA_K_VARIANT_TMA ? &k.c : nullptr, nullptr) == cudaSuccess);
        for (uint32_t p = 0; p < n; ++p)
            if (memcmp(b.data() + p * PAGE, a.data() + perm[p] * PAGE, PAGE) != 0) { fprintf(stderr, "K1 gather: page %u wrong (variant %d, tile %u)\n", p, k.variant, k.c.tile_bytes); return 1; }
        std::fill(c.begin(), c.end(), 0xEF);
        for (uint32_t p = 0; p < n; ++p) dst_tab[p] = (uint64_t)(uintptr_t)(c.data() + perm[p] * PAGE);
        assert(fma_k_launch_page_copy(nullptr, (uint64_t)(uintptr_t)b.data(), dst_tab.data(), 0, n, k.variant, k.variant == FMA_K_VARIANT_TMA ? &k.c : nullptr, nullptr) == cudaSuccess);
        if (c != a) { fprintf(stderr, "K2 scatter does not restore the pages (variant %d, tile %u)\n", k.variant, k.c.tile_bytes); return 1; }
    }
    // a TMA shape that does not fit is refused, as on the device
    fma_k_tma_cfg bad{512, 3, 2, 1};
    assert(fma_k_launch_page_copy(src_tab.data(), 0, nullptr, (uint64_t)(uintptr_t)b.data(), n, FMA_K_VARIANT_TMA, &bad, nullptr) == cudaErrorInvalidValue);
    puts("kernels (emulated) ok");
    return 0;
}
