// Runs the ACTUAL kernel source csrc/fma_pack_kernels.cu (K4p / K4 / K5) on the CPU execution model of cuda_emu.h and
// checks it against the oracle (oracle/fma_oracle.c) page by page: probe decisions, stored bytes (exceptions compared
// as sets), decode, gather/scatter through descriptor tables, the error counter.  Built by tests/test_kernels_emulated.py
// with g++ -DFMA_CUDA_EMU -include cuda_emu.h, plain and under ThreadSanitizer (missing barriers = data races).
//
// The SAME file is the GPU-side kernel test: `nvcc -x cu -DFMA_GPU_TEST ...` (tests/cpp/cuda_emu/Makefile ->
// tests/cpp/cuda_emu/pack_kernels_gpu_test, run on an H100 by tests/test_gpu_parity.py::test_pack_kernels_binary_on_the_device) compiles the real kernels and
// keeps every buffer in managed memory, so a mismatch on the device is reported with the page it happened in,
// without the engine in the way.
#include <algorithm>
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#if defined(FMA_GPU_TEST)
#include <cuda_runtime.h>
#include <new>
template <class T>
struct DevAlloc {  // managed memory: the host-side checks read what the kernels wrote
    typedef T value_type;
    DevAlloc() = default;
    template <class U> DevAlloc(const DevAlloc<U>&) {}
    T* allocate(size_t n) { void* p = nullptr; if (cudaMallocManaged(&p, n * sizeof(T)) != cudaSuccess) throw std::bad_alloc(); return static_cast<T*>(p); }
    void deallocate(T* p, size_t) { cudaFree(p); }
    template <class U> bool operator==(const DevAlloc<U>&) const { return true; }
    template <class U> bool operator!=(const DevAlloc<U>&) const { return false; }
};
#define DEVICE_SYNC() do { cudaError_t _e = cudaDeviceSynchronize(); if (_e != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(_e)); return 2; } } while (0)
static unsigned char* host_mapped(size_t n, unsigned char** dev) {  // pinned host memory the device reads over the link
    void *h = nullptr, *d = nullptr;
    if (cudaHostAlloc(&h, n, cudaHostAllocMapped) != cudaSuccess || cudaHostGetDevicePointer(&d, h, 0) != cudaSuccess) throw std::bad_alloc();
    *dev = static_cast<unsigned char*>(d);
    return static_cast<unsigned char*>(h);
}
static const bool kOnDevice = true;
#else
// the runtime calls the launch wrappers make
extern "C" cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
extern "C" cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 3; return cudaSuccess; }  // 3 "SMs": grid-stride loops get exercised
extern "C" cudaError_t cudaGetLastError(void) { return cudaSuccess; }
template <class T> using DevAlloc = std::allocator<T>;
#define DEVICE_SYNC() do { } while (0)
static unsigned char* host_mapped(size_t n, unsigned char** dev) { *dev = static_cast<unsigned char*>(malloc(n)); return *dev; }
static const bool kOnDevice = false;
#endif

#include "../../../llm-d-fast-model-actuation_b200/csrc/fma_pack_kernels.cu"

extern "C" {
uint32_t fma_oracle_pack_page(const void* page, void* stored);
int fma_oracle_unpack_page(const void* stored, uint32_t stored_bytes, void* page);
}

static const size_t PAGE = 2u << 20, N = 1u << 20, PACKED = FMA_K_PACKED_PAGE_BYTES;
static uint32_t rng_state = 2463534242u;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 17; rng_state ^= rng_state << 5; return rng_state; }

typedef std::vector<uint16_t, DevAlloc<uint16_t>> Page;   // device-visible
typedef std::vector<unsigned char, DevAlloc<unsigned char>> Bytes;
template <class T> using DVec = std::vector<T, DevAlloc<T>>;
static Page weights(uint32_t e_lo, uint32_t span) {  // bf16 values with exponents e_lo .. e_lo+span-1
    Page p(N);
    for (auto& v : p) { uint32_t x = rnd(); v = (uint16_t)(((x >> 31) << 15) | ((e_lo + (x >> 8) % span) << 7) | ((x >> 16) & 0x7F)); }
    return p;
}

static bool same_stored(const unsigned char* a, const unsigned char* b, uint32_t bytes) {
    if (bytes == PAGE) return memcmp(a, b, PAGE) == 0;
    using namespace fma_codec;
    uint32_t na, nb;
    memcpy(&na, a + kHdrOff + 4, 4); memcpy(&nb, b + kHdrOff + 4, 4);
    if (memcmp(a, b, kExcOff) != 0 || na != nb || memcmp(a + kHdrOff, b + kHdrOff, 4) != 0) return false;
    std::vector<uint32_t> ea(na), eb(nb);
    memcpy(ea.data(), a + kExcOff, 4 * na); memcpy(eb.data(), b + kExcOff, 4 * nb);
    std::sort(ea.begin(), ea.end()); std::sort(eb.begin(), eb.end());
    return ea == eb;
}

static int run_all() {
    std::vector<Page> pages;
    pages.push_back(weights(110, 12));                                  // well inside 13 binades
    pages.push_back(weights(100, 27));                                  // wide: many exceptions -> probably raw
    { Page p = weights(118, 9); for (size_t i = 0; i < N; i += 3) p[i] = (i & 1) ? 0x8000 : 0; pages.push_back(p); }          // +-0 sprinkled
    { Page p(N, 0x3F80); for (int k = 0; k < 2048; ++k) p[(size_t)k * 509 + 7] = 0x00D5; pages.push_back(p); }                 // exactly 2048 exceptions
    { Page p(N, 0x3F80); for (int k = 0; k < 2049; ++k) p[(size_t)k * 509 + 7] = 0x00D5; pages.push_back(p); }                 // 2049 -> raw
    { Page p(N); for (auto& v : p) v = (uint16_t)rnd(); pages.push_back(p); }                                                   // noise -> raw
    pages.push_back(Page(N, 0));                                        // zeros
    { Page p = weights(120, 6); p[5] = 0x7F80; p[300000] = 0xFFC1; p[N - 1] = 0x0001; pages.push_back(p); }                    // inf / nan / denormal at the edges
    // K4 shares one exception counter among the 8 parts of a page and the last part to finish writes the header; K5 gives an
    // exception to the part whose value range (kValuesPart = 131072 values) holds its index.  0x3F80 has exponent 127,
    // 0x00D5 exponent 1: one exception each.
    { Page p(N, 0x3F80); for (int k = 0; k < 2048; ++k) p[3 * kValuesPart + (size_t)k * 64 + 17] = 0x00D5; pages.push_back(p); }   // all 2048 in part 3
    { Page p(N, 0x3F80); for (size_t q = 0; q < kParts; ++q) for (int k = 0; k < 256; ++k) p[q * kValuesPart + (size_t)k * 512 + 5] = 0x00D5; pages.push_back(p); }  // 256 per part
    { Page p = weights(118, 9); for (size_t q = 0; q < kParts; ++q) { p[q * kValuesPart] = 0x00D5; p[q * kValuesPart + kValuesPart - 1] = 0x80D5; } pages.push_back(p); }  // first + last value of every part
    {   // tile maxima 0, 1, 13, 14, 15, 255 and 127, with values exactly 13 (code 13) and 14 (code 14 for zeros, else an exception)
        // binades below them; tiles of emax 0 hold only zeros and denormals
        Page p(N);
        const uint32_t emax_of[8] = {0, 1, 13, 14, 15, 255, 127, 0};
        for (uint32_t t = 0; t < fma_codec::kTiles; ++t) {
            const uint32_t em = emax_of[t % 8];
            for (uint32_t i = 0; i < fma_codec::kTileValues; ++i) {
                const uint32_t x = rnd();
                uint32_t e = em;
                switch (i % 4) {
                    case 0: e = em; break;
                    case 1: e = em >= 13 ? em - 13 : 0; break;                // code 13 (em = 13: a zero / denormal coded 13)
                    case 2: e = 0; break;                                      // zero / denormal: code <= 13, or 14
                    case 3: e = i == 3 && em >= 14 ? em - 14 : em >= 13 ? em - 13 : em; break;  // one value per tile 14 binades down
                }
                p[t * fma_codec::kTileValues + i] = (uint16_t)(((x >> 31) << 15) | (e << 7) | ((x >> 16) & 0x7F));
            }
        }
        pages.push_back(p);
    }
    if (getenv("FMA_EMU_FAST")) pages.resize(5);                        // sanitizer runs: the first five pages cover every branch but noise / inf
    const uint32_t n = (uint32_t)pages.size();

    // K4p vs oracle
    DVec<uint64_t> tab(n);
    for (uint32_t p = 0; p < n; ++p) tab[p] = (uint64_t)(uintptr_t)pages[p].data();
    DVec<uint32_t> sizes(n, 0);
    assert(fma_k_launch_pack_probe(tab.data(), n, sizes.data(), nullptr) == cudaSuccess);
    DEVICE_SYNC();
    std::vector<Bytes> want(n, Bytes(PAGE));
    uint32_t n_raw = 0;
    for (uint32_t p = 0; p < n; ++p) {
        const uint32_t w = fma_oracle_pack_page(pages[p].data(), want[p].data());
        if (w != sizes[p]) { fprintf(stderr, "page %u: probe says %u, oracle %u\n", p, sizes[p], w); return 1; }
        n_raw += w == PAGE;
    }
    assert(n_raw >= 1 && n_raw <= 3);

    // K4: gather in a permuted order into one contiguous store
    std::vector<uint32_t> perm(n);
    for (uint32_t k = 0; k < n; ++k) perm[k] = (7 * k + 3) % n;          // a permutation for n = 5 and n = 12
    uint64_t total = 0;
    for (uint32_t p : perm) total += sizes[p];
    Bytes store(total, 0xEE);
    DVec<fma_k_pack_desc> d(n);
    std::vector<uint64_t> off(n);
    uint64_t o = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const uint32_t p = perm[k];
        off[k] = o;
        d[k] = fma_k_pack_desc{tab[p], (uint64_t)(uintptr_t)(store.data() + o), sizes[p] == PAGE ? (uint32_t)FMA_K_PACK_RAW : (uint32_t)FMA_K_PACK_BF16, 0};
        o += sizes[p];
    }
    DVec<uint32_t> errv(1, 0);
    uint32_t& err = errv[0];
    assert(fma_k_launch_pack(d.data(), n, &err, nullptr) == cudaSuccess);
    DEVICE_SYNC();
    assert(err == 0);
    for (uint32_t k = 0; k < n; ++k)
        if (!same_stored(store.data() + off[k], want[perm[k]].data(), sizes[perm[k]])) { fprintf(stderr, "stored page %u differs from the oracle's\n", perm[k]); return 1; }

    // K5: scatter back to fresh pages; also decode the ORACLE's stored pages with the kernel
    std::vector<Page> back(n, Page(N, 0xABCD));
    for (uint32_t k = 0; k < n; ++k) { d[k].src = (uint64_t)(uintptr_t)(store.data() + off[k]); d[k].dst = (uint64_t)(uintptr_t)back[perm[k]].data(); }
    assert(fma_k_launch_unpack(d.data(), n, &err, nullptr) == cudaSuccess);
    DEVICE_SYNC();
    assert(err == 0);
    for (uint32_t p = 0; p < n; ++p)
        if (back[p] != pages[p]) { fprintf(stderr, "page %u does not survive the round trip\n", p); return 1; }
    for (uint32_t k = 0; k < n; ++k) { d[k].src = (uint64_t)(uintptr_t)want[perm[k]].data(); std::fill(back[perm[k]].begin(), back[perm[k]].end(), 0x1234); }
    assert(fma_k_launch_unpack(d.data(), n, &err, nullptr) == cudaSuccess);
    DEVICE_SYNC();
    assert(err == 0);
    for (uint32_t p = 0; p < n; ++p) assert(back[p] == pages[p]);
    // and the oracle decodes the kernel's stored pages
    for (uint32_t k = 0; k < n; ++k) {
        Page out(N);
        assert(fma_oracle_unpack_page(store.data() + off[k], sizes[perm[k]], out.data()) == 0 && out == pages[perm[k]]);
    }

    // K5 reads the stored pages straight from mapped pinned host memory (the zero-copy packed wake)
    {
        unsigned char* h_dev = nullptr;
        unsigned char* h = host_mapped(total, &h_dev);
        memcpy(h, store.data(), total);
        for (uint32_t k = 0; k < n; ++k) { d[k].src = (uint64_t)(uintptr_t)(h_dev + off[k]); std::fill(back[perm[k]].begin(), back[perm[k]].end(), 0x5A5A); }
        err = 0;
        assert(fma_k_launch_unpack(d.data(), n, &err, nullptr) == cudaSuccess);
        DEVICE_SYNC();
        assert(err == 0);
        for (uint32_t p = 0; p < n; ++p)
            if (back[p] != pages[p]) { fprintf(stderr, "page %u: K5 from mapped host memory differs\n", p); return 1; }
#if defined(FMA_GPU_TEST)
        cudaFreeHost(h);
#else
        free(h);
#endif
    }

    // RAW and coded descriptors alternate in one launch with more work items than CTAs: every CTA strides over items of both
    // kinds (K4p / K5 reuse their shared state across items, K4 its emax slice).  The CPU model's grid is 3 SMs x 8 CTAs;
    // on the device FMA_PACK_CTAS_PER_SM=1 makes it 132 CTAs, and then the launch must reach 2 items per CTA.
    {
        std::vector<uint32_t> raw, coded;
        for (uint32_t p = 0; p < n; ++p) (sizes[p] == PAGE ? raw : coded).push_back(p);
        const uint32_t cap = pack_grid(0xFFFFFFFFu);
        const uint32_t n_alt = std::min<uint32_t>((2 * cap + kParts - 1) / kParts + 1, 40);
        std::vector<uint32_t> src(n_alt);
        for (uint32_t k = 0; k < n_alt; ++k) src[k] = k % 2 ? coded[(k / 2) % coded.size()] : raw[(k / 2) % raw.size()];
        DVec<uint64_t> atab(n_alt);
        for (uint32_t k = 0; k < n_alt; ++k) atab[k] = tab[src[k]];
        DVec<uint32_t> asz(n_alt, 0);
        assert(fma_k_launch_pack_probe(atab.data(), n_alt, asz.data(), nullptr) == cudaSuccess);
        DEVICE_SYNC();
        std::vector<uint64_t> aoff(n_alt);
        uint64_t atotal = 0;
        for (uint32_t k = 0; k < n_alt; ++k) {
            if (asz[k] != sizes[src[k]]) { fprintf(stderr, "strided probe: page %u says %u\n", k, asz[k]); return 1; }
            aoff[k] = atotal;
            atotal += asz[k];
        }
        Bytes astore(atotal, 0xEE);
        DVec<fma_k_pack_desc> ad(n_alt);
        for (uint32_t k = 0; k < n_alt; ++k)
            ad[k] = fma_k_pack_desc{atab[k], (uint64_t)(uintptr_t)(astore.data() + aoff[k]), asz[k] == PAGE ? (uint32_t)FMA_K_PACK_RAW : (uint32_t)FMA_K_PACK_BF16, 0};
        err = 0;
        assert(fma_k_launch_pack(ad.data(), n_alt, &err, nullptr) == cudaSuccess);
        DEVICE_SYNC();
        assert(err == 0);
        for (uint32_t k = 0; k < n_alt; ++k) {
            if (!same_stored(astore.data() + aoff[k], want[src[k]].data(), asz[k])) { fprintf(stderr, "strided K4: stored page %u differs from the oracle's\n", k); return 1; }
            Page out(N);
            if (fma_oracle_unpack_page(astore.data() + aoff[k], asz[k], out.data()) != 0 || out != pages[src[k]]) { fprintf(stderr, "strided K4: the oracle cannot decode page %u\n", k); return 1; }
        }
        std::vector<Page> aback(n_alt, Page(N, 0xABCD));
        for (uint32_t k = 0; k < n_alt; ++k) { ad[k].src = (uint64_t)(uintptr_t)(astore.data() + aoff[k]); ad[k].dst = (uint64_t)(uintptr_t)aback[k].data(); }
        assert(fma_k_launch_unpack(ad.data(), n_alt, &err, nullptr) == cudaSuccess);
        DEVICE_SYNC();
        assert(err == 0);
        for (uint32_t k = 0; k < n_alt; ++k)
            if (aback[k] != pages[src[k]]) { fprintf(stderr, "strided K5: page %u differs\n", k); return 1; }
        const uint32_t items = n_alt * kParts, grid = pack_grid(items);
        printf("K4/K5 strided launch: %u pages (RAW and coded alternate), %u items, grid %u, items/grid = %.2f\n", n_alt, items, grid, (double)items / grid);
        if ((!kOnDevice || getenv("FMA_PACK_CTAS_PER_SM")) && items < 2 * grid) { fprintf(stderr, "the strided launch has fewer than 2 items per CTA\n"); return 1; }
    }

    // error counters: a page forced into the coded form although it overflows; a damaged header
    DVec<fma_k_pack_desc> bad(1, fma_k_pack_desc{tab[4], (uint64_t)(uintptr_t)store.data(), FMA_K_PACK_BF16, 0});
    err = 0;
    assert(fma_k_launch_pack(bad.data(), 1, &err, nullptr) == cudaSuccess);
    DEVICE_SYNC();
    assert(err == 1);
    Bytes dmg(want[0].begin(), want[0].begin() + PACKED);
    dmg[fma_codec::kHdrOff] ^= 0xFF;
    Page sink(N);
    bad[0] = fma_k_pack_desc{(uint64_t)(uintptr_t)dmg.data(), (uint64_t)(uintptr_t)sink.data(), FMA_K_PACK_BF16, 0};
    err = 0;
    assert(fma_k_launch_unpack(bad.data(), 1, &err, nullptr) == cudaSuccess);
    DEVICE_SYNC();
    assert(err == 1);
    return 0;
}

int main() {
    const int rc = run_all();
    if (rc) return rc;
#if defined(FMA_GPU_TEST)
    puts("pack kernels (GPU) ok");
#else
    puts("pack kernels (emulated) ok");
#endif
    return 0;
}
