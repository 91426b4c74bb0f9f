// K6 (fma_k_unpack_digest, csrc/fma_pack_kernels.cu) against the oracle and against K3 over K5's output.  The ACTUAL kernel
// sources run on the CPU execution model of cuda_emu.h (g++ -DFMA_CUDA_EMU -include cuda_emu.h, plain and under ThreadSanitizer,
// built and run by tests/test_image_verify.py), and the same file compiled by nvcc -x cu -DFMA_GPU_TEST runs them on the GPU with
// every buffer in managed memory.
//
// Pages are coded by the oracle (oracle/fma_oracle.c), so the kernel decodes a stored form it did not write.  The reference digest of
// a stored page is the oracle's decode followed by the oracle's digest at the page's word offset; offsets are large and random, so a
// kernel that mixes up word positions fails.
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#if defined(FMA_GPU_TEST)
#include <cuda_runtime.h>
#include <new>
template <class T>
struct DevAlloc {
    typedef T value_type;
    DevAlloc() = default;
    template <class U> DevAlloc(const DevAlloc<U>&) {}
    T* allocate(size_t n) { void* p = nullptr; if (cudaMallocManaged(&p, n * sizeof(T)) != cudaSuccess) throw std::bad_alloc(); return static_cast<T*>(p); }
    void deallocate(T* p, size_t) { cudaFree(p); }
    template <class U> bool operator==(const DevAlloc<U>&) const { return true; }
    template <class U> bool operator!=(const DevAlloc<U>&) const { return false; }
};
#define DEVICE_SYNC() do { cudaError_t _e = cudaDeviceSynchronize(); if (_e != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(_e)); return 2; } } while (0)
#else
extern "C" cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
extern "C" cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 3; return cudaSuccess; }  // 3 "SMs": grid-stride loops run
extern "C" cudaError_t cudaGetLastError(void) { return cudaSuccess; }
template <class T> using DevAlloc = std::allocator<T>;
#define DEVICE_SYNC() do { } while (0)
#endif

#include "../../../llm-d-fast-model-actuation_b200/csrc/fma_pack_kernels.cu"
#include "../../../llm-d-fast-model-actuation_b200/csrc/fma_kernels.cu"

extern "C" {
uint32_t fma_oracle_pack_page(const void* page, void* stored);
int fma_oracle_unpack_page(const void* stored, uint32_t stored_bytes, void* page);
uint64_t fma_oracle_digest(const void* src, uint64_t n_bytes, uint64_t first_word);
}

static const size_t PAGE = 2u << 20, N = 1u << 20, PACKED = FMA_K_PACKED_PAGE_BYTES;
static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 16); }
static uint64_t rnd64() { return (uint64_t)rnd() << 32 | rnd(); }

typedef std::vector<uint16_t> Page;
template <class T> using DVec = std::vector<T, DevAlloc<T>>;
static Page weights(uint32_t e_lo, uint32_t span) {
    Page p(N);
    for (auto& v : p) { uint32_t x = rnd(); v = (uint16_t)(((x >> 31) << 15) | ((e_lo + (x >> 8) % span) << 7) | ((x >> 16) & 0x7F)); }
    return p;
}

// the reference: the oracle decodes the stored page, the oracle digests the result at `first_word`
static uint64_t oracle_stored_digest(const unsigned char* stored, uint64_t first_word) {
    Page page(N);
    if (fma_oracle_unpack_page(stored, (uint32_t)PACKED, page.data()) != 0) { fprintf(stderr, "the oracle cannot decode a stored page\n"); exit(1); }
    return fma_oracle_digest(page.data(), PAGE, first_word);
}

static int run_all() {
    using namespace fma_codec;
    std::vector<Page> pages;
    pages.push_back(weights(110, 12));                                   // no exception
    { Page p = weights(110, 12); for (int k = 0; k < 400; ++k) p[rnd() % N] = (uint16_t)((rnd() & 0x8000) | 0x0080 | (rnd() & 0x7F)); pages.push_back(p); }  // ~400 exceptions, scattered
    {   // exceptions sharing 64-bit words: 1, 2, 3 and 4 patched values in one word, in every part
        Page p(N, 0x3F80);
        for (size_t q = 0; q < kParts; ++q) {
            const size_t w = q * kValuesPart + 4 * (size_t)(rnd() % (kValuesPart / 4 - 8));
            p[w] = 0x00D5;
            p[w + 4] = 0x8081; p[w + 7] = 0x0102;
            p[w + 9] = 0x0083; p[w + 10] = 0x80D5; p[w + 11] = 0x0101;
            p[w + 12] = 0x0081; p[w + 13] = 0x0082; p[w + 14] = 0x8083; p[w + 15] = 0x0084;
        }
        pages.push_back(p);
    }
    { Page p(N, 0x3F80); for (int k = 0; k < 2048; ++k) p[3 * kValuesPart + (size_t)k * 64 + 17] = 0x00D5; pages.push_back(p); }   // 2048 in part 3
    { Page p(N, 0x3F80); for (int k = 0; k < 2048; ++k) p[(size_t)k * 4 + (k & 3)] = 0x0100 + (uint16_t)(k & 0x3F); pages.push_back(p); }  // 2048 in words 0..2047
    { Page p = weights(120, 6); p[0] = 0x0001; p[5] = 0x7F80; p[300000] = 0xFFC1; p[N - 1] = 0x00D5; pages.push_back(p); }       // edges, inf / nan
    pages.push_back(Page(N, 0));
    if (getenv("FMA_EMU_FAST")) pages.resize(4);                         // sanitizer runs: shared words and the full part are kept
    const uint32_t n = (uint32_t)pages.size();

    DVec<unsigned char> store((size_t)n * PACKED);
    std::vector<uint64_t> want(n);
    DVec<fma_k_page_desc> d(n);
    for (uint32_t p = 0; p < n; ++p) {
        std::vector<unsigned char> st(PAGE);
        if (fma_oracle_pack_page(pages[p].data(), st.data()) != PACKED) { fprintf(stderr, "test page %u does not code\n", p); return 1; }
        memcpy(store.data() + (size_t)p * PACKED, st.data(), PACKED);
        const uint64_t first_word = (rnd64() >> 8) * 8 + (p & 1);   // large, and odd for every other page
        d[p] = fma_k_page_desc{(uint64_t)(uintptr_t)(store.data() + (size_t)p * PACKED), first_word};
        want[p] = oracle_stored_digest(st.data(), first_word);
    }

    // K6 == oracle
    DVec<uint64_t> out(n, 0);
    DVec<uint32_t> errv(1, 0);
    assert(fma_k_launch_unpack_digest(d.data(), n, out.data(), errv.data(), nullptr) == cudaSuccess);
    DEVICE_SYNC();
    if (errv[0] != 0) { fprintf(stderr, "K6 reports %u malformed pages\n", errv[0]); return 1; }
    for (uint32_t p = 0; p < n; ++p)
        if (out[p] != want[p]) { fprintf(stderr, "page %u: K6 %016llx, oracle %016llx\n", p, (unsigned long long)out[p], (unsigned long long)want[p]); return 1; }

    // K6 == K3 over K5's output
    DVec<uint16_t> decoded((size_t)n * N, 0xABCD);
    DVec<fma_k_pack_desc> pd(n);
    DVec<fma_k_page_desc> dd(n);
    for (uint32_t p = 0; p < n; ++p) {
        pd[p] = fma_k_pack_desc{d[p].addr, (uint64_t)(uintptr_t)(decoded.data() + (size_t)p * N), FMA_K_PACK_BF16, 0};
        dd[p] = fma_k_page_desc{(uint64_t)(uintptr_t)(decoded.data() + (size_t)p * N), d[p].first_word};
    }
    assert(fma_k_launch_unpack(pd.data(), n, errv.data(), nullptr) == cudaSuccess);
    DVec<uint64_t> k3(n, 0);
    assert(fma_k_launch_page_digest(dd.data(), n, k3.data(), nullptr) == cudaSuccess);
    DEVICE_SYNC();
    for (uint32_t p = 0; p < n; ++p) {
        if (memcmp(decoded.data() + (size_t)p * N, pages[p].data(), PAGE) != 0) { fprintf(stderr, "page %u: K5 does not restore it\n", p); return 1; }
        if (k3[p] != out[p]) { fprintf(stderr, "page %u: K3 over K5 %016llx, K6 %016llx\n", p, (unsigned long long)k3[p], (unsigned long long)out[p]); return 1; }
    }

    // one flipped bit in each plane of a stored page changes its digest; the same page twice in a launch adds up twice
    {
        const uint32_t at[4] = {kSmOff + 4097, kNibOff + 777, kEmaxOff + 100, kExcOff + 0};
        DVec<unsigned char> flip(4 * PACKED);
        DVec<fma_k_page_desc> fd(5);
        for (int k = 0; k < 4; ++k) {
            memcpy(flip.data() + (size_t)k * PACKED, store.data() + PACKED, PACKED);   // page 1 has exceptions
            flip[(size_t)k * PACKED + at[k]] ^= 0x10;
            fd[k] = fma_k_page_desc{(uint64_t)(uintptr_t)(flip.data() + (size_t)k * PACKED), d[1].first_word};
        }
        fd[4] = d[1];
        DVec<uint64_t> fo(5, 0);
        errv[0] = 0;
        assert(fma_k_launch_unpack_digest(fd.data(), 5, fo.data(), errv.data(), nullptr) == cudaSuccess);
        DEVICE_SYNC();
        for (int k = 0; k < 4; ++k) {
            const uint64_t ref = oracle_stored_digest(flip.data() + (size_t)k * PACKED, d[1].first_word);
            if (fo[k] != ref || fo[k] == want[1]) { fprintf(stderr, "flip in plane %d: K6 %016llx, oracle %016llx\n", k, (unsigned long long)fo[k], (unsigned long long)ref); return 1; }
        }
        if (fo[4] != want[1] || errv[0] != 0) { fprintf(stderr, "the intact copy of page 1 differs\n"); return 1; }
    }

    // malformed pages: counted once each, nothing added
    {
        DVec<unsigned char> dmg(2 * PACKED);
        memcpy(dmg.data(), store.data(), PACKED);
        memcpy(dmg.data() + PACKED, store.data(), PACKED);
        dmg[kHdrOff] ^= 0xFF;                                             // bad magic
        const uint32_t too_many = kExcCap + 1;
        memcpy(dmg.data() + PACKED + kHdrOff + 4, &too_many, 4);          // too many exceptions
        DVec<fma_k_page_desc> bd(2);
        bd[0] = fma_k_page_desc{(uint64_t)(uintptr_t)dmg.data(), 0};
        bd[1] = fma_k_page_desc{(uint64_t)(uintptr_t)(dmg.data() + PACKED), 0};
        DVec<uint64_t> bo(2, 0);
        errv[0] = 0;
        assert(fma_k_launch_unpack_digest(bd.data(), 2, bo.data(), errv.data(), nullptr) == cudaSuccess);
        DEVICE_SYNC();
        if (errv[0] != 2 || bo[0] != 0 || bo[1] != 0) { fprintf(stderr, "malformed pages: err %u, sums %llx %llx\n", errv[0], (unsigned long long)bo[0], (unsigned long long)bo[1]); return 1; }
    }
    return 0;
}

int main() {
    const int rc = run_all();
    if (rc) return rc;
#if defined(FMA_GPU_TEST)
    puts("unpack digest (GPU) ok");
#else
    puts("unpack digest (emulated) ok");
#endif
    return 0;
}
