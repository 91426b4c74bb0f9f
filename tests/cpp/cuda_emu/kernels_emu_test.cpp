// Runs the ACTUAL kernel source csrc/fma_kernels.cu — K0 fill, K1/K2 page copy (the TMA pipeline and the LDG variant), K3
// digest — and checks it against the oracle (oracle/fma_oracle.c).
//
// Two builds of this one file:
//   * g++ -DFMA_CUDA_EMU -include cuda_emu.h (tests/test_kernels_emulated.py): the CPU execution model, lazy async proxy
//     included, plain and under ThreadSanitizer.  It starts an OS thread per GPU thread, so it runs a subset: every 4th
//     shape, 8 source pages and no 200-page K0/K3 run (FMA_EMU_FAST=1, the sanitizer build: every 10th shape, fewer still).
//   * nvcc -x cu -DFMA_GPU_TEST (tests/cpp/cuda_emu/Makefile -> kernels_gpu_test, run on an H100 by
//     tests/test_gpu_kernel_shapes.py): the real PTX (mbarrier parity, expect_tx, cp.async.bulk wait_group) and real
//     concurrency.  Buffers are device memory read back with cudaMemcpy; the zero-copy cases use mapped pinned host memory.
//
// What runs:
//   K1/K2  every legal TMA shape (tile 1..64 KiB, stages 2..8, pipes 1..4, smem <= 227 KiB: 140 shapes), each at
//          ctas_per_sm 1 and one of {2, 4}, gather and scatter, at 1 and 5 pages, and at 67 pages for a seeded subset;
//          the LDG variant at the same page counts; a gather that lists one source page twice; source or destination in
//          mapped pinned host memory; out-of-range stages / pipes (clamped) and shapes that cannot run (refused by the
//          launch wrapper before any launch, the destination untouched).
//   K0/K3  scattered descriptors, a page listed twice, first_word near 2^64 (the word counter wraps), and page counts on
//          both sides of the grid cap (SMs x 8 CTAs x 32 KiB tiles): 1, 16, 17 and 200 pages.
// 1-page copies are read back byte for byte; larger ones are checked page by page through K3 digests (on the device; the
// CPU model compares bytes, which costs nothing there) against the oracle's digest of the expected page.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <random>
#include <vector>

#if defined(FMA_GPU_TEST)
#include <cuda_runtime.h>
static void sync_or_die() {
    const cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(e)); exit(2); }
}
static unsigned char* dev_bytes(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n) != cudaSuccess) { fprintf(stderr, "cudaMalloc(%zu) failed\n", n); exit(2); }
    return static_cast<unsigned char*>(p);
}
static void dev_free(void* p) { cudaFree(p); }
static void to_host(void* dst, const void* src, size_t n) { if (cudaMemcpy(dst, src, n, cudaMemcpyDefault) != cudaSuccess) { fprintf(stderr, "cudaMemcpy failed\n"); exit(2); } }
static void to_dev(void* dst, const void* src, size_t n) { to_host(dst, src, n); }
struct Mapped { unsigned char* host; unsigned char* dev; };
static Mapped host_mapped(size_t n) {
    void *h = nullptr, *d = nullptr;
    if (cudaHostAlloc(&h, n, cudaHostAllocMapped) != cudaSuccess || cudaHostGetDevicePointer(&d, h, 0) != cudaSuccess) {
        fprintf(stderr, "cudaHostAlloc(%zu, mapped) failed\n", n);
        exit(2);
    }
    return Mapped{static_cast<unsigned char*>(h), static_cast<unsigned char*>(d)};
}
static void fill_bytes(void* p, int v, size_t n) { if (cudaMemset(p, v, n) != cudaSuccess) { fprintf(stderr, "cudaMemset failed\n"); exit(2); } sync_or_die(); }
static const bool kOnDevice = true;
#else
extern "C" cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
extern "C" cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 3; return cudaSuccess; }  // 3 "SMs": grid-stride loops run
extern "C" cudaError_t cudaGetLastError(void) { return cudaSuccess; }
static void sync_or_die() {}
static unsigned char* dev_bytes(size_t n) { return static_cast<unsigned char*>(aligned_alloc(4096, (n + 4095) & ~(size_t)4095)); }
static void dev_free(void* p) { free(p); }
static void to_host(void* dst, const void* src, size_t n) { memcpy(dst, src, n); }
static void to_dev(void* dst, const void* src, size_t n) { memcpy(dst, src, n); }
struct Mapped { unsigned char* host; unsigned char* dev; };
static Mapped host_mapped(size_t n) { unsigned char* p = dev_bytes(n); return Mapped{p, p}; }
static void fill_bytes(void* p, int v, size_t n) { memset(p, v, n); }
static const bool kOnDevice = false;
#endif

#include "../../../llm-d-fast-model-actuation_b200/csrc/fma_kernels.cu"

extern "C" {
void fma_oracle_fill(uint64_t* dst, uint64_t n_words, uint64_t seed, uint64_t first_word);
uint64_t fma_oracle_digest(const void* src, uint64_t n_bytes, uint64_t first_word);
}

static const size_t PAGE = FMA_K_PAGE_BYTES, WORDS = PAGE / 8;
static const uint64_t SEED = 0xDEADBEEF;

static void die(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
    exit(1);
}
template <class T> static T* dev_array(size_t n) { return reinterpret_cast<T*>(dev_bytes(n * sizeof(T))); }
static uint64_t addr(const void* p) { return (uint64_t)(uintptr_t)p; }

// ---- K0 / K3 -----------------------------------------------------------------------------------------------------
// `n` descriptors over the first pages of `buf` in a scattered order, the last one repeating an earlier page (same stream
// position); page q of the stream starts at word first + q * WORDS, which wraps past 2^64 when first is near it
static void fill_and_digest(unsigned char* buf, uint32_t n, uint64_t first, std::mt19937_64& rng) {
    const uint32_t n_distinct = n > 1 ? n - 1 : 1;
    std::vector<uint32_t> page(n_distinct);
    std::iota(page.begin(), page.end(), 0u);
    std::shuffle(page.begin(), page.end(), rng);
    if (n > 1) page.push_back(page[n / 2]);
    std::vector<fma_k_page_desc> desc(n);
    for (uint32_t k = 0; k < n; ++k) desc[k] = fma_k_page_desc{addr(buf + (size_t)page[k] * PAGE), first + page[k] * WORDS};
    fma_k_page_desc* d_desc = dev_array<fma_k_page_desc>(n);
    to_dev(d_desc, desc.data(), n * sizeof(fma_k_page_desc));
    fill_bytes(buf, 0xA5, n_distinct * PAGE);
    if (fma_k_launch_fill(d_desc, n, SEED, nullptr) != cudaSuccess) die("K0 launch refused (%u pages)", n);
    sync_or_die();
    std::vector<uint64_t> want(WORDS), got(WORDS), want_dig(n_distinct);
    for (uint32_t q = 0; q < n_distinct; ++q) {
        fma_oracle_fill(want.data(), WORDS, SEED, first + q * WORDS);
        to_host(got.data(), buf + (size_t)q * PAGE, PAGE);
        if (got != want) die("K0: page %u of %u (first_word %llu) differs from the oracle", q, n, (unsigned long long)first);
        want_dig[q] = fma_oracle_digest(want.data(), PAGE, first + q * WORDS);
    }
    uint64_t* d_dig = dev_array<uint64_t>(n);
    fill_bytes(d_dig, 0, n * sizeof(uint64_t));
    if (fma_k_launch_page_digest(d_desc, n, d_dig, nullptr) != cudaSuccess) die("K3 launch refused (%u pages)", n);
    sync_or_die();
    std::vector<uint64_t> dig(n);
    to_host(dig.data(), d_dig, n * sizeof(uint64_t));
    for (uint32_t k = 0; k < n; ++k)
        if (dig[k] != want_dig[page[k]]) die("K3: descriptor %u (page %u of %u, first_word %llu) differs from the oracle", k, page[k], n, (unsigned long long)first);
    dev_free(d_desc);
    dev_free(d_dig);
}

// ---- K1 / K2 -----------------------------------------------------------------------------------------------------
struct Pool {
    std::vector<unsigned char> a_host;  // the oracle's stream, n_a pages (page q = words q*WORDS ...)
    unsigned char* a;                   // the same on the device, written by K0
    unsigned char* b;                   // contiguous image
    unsigned char* c;                   // scatter destination, n_a pages
    uint32_t n_a;
    std::vector<uint64_t> dig_a;        // oracle digest of page q of a (first_word q*WORDS)
    uint64_t* d_tab;                    // device page table
    fma_k_page_desc* d_desc;
    uint64_t* d_dig;
};

static const uint64_t* upload_tab(Pool& P, const std::vector<uint64_t>& tab) {
    to_dev(P.d_tab, tab.data(), tab.size() * sizeof(uint64_t));
    return P.d_tab;
}

// page p of the destination (address dst[p]) must hold page want[p] of `a`
static void expect_pages(Pool& P, const std::vector<uint64_t>& dst, const std::vector<uint32_t>& want, const char* what) {
    const uint32_t n = (uint32_t)want.size();
    if (n == 1 || !kOnDevice) {
        std::vector<unsigned char> got(PAGE);
        for (uint32_t p = 0; p < n; ++p) {
            to_host(got.data(), reinterpret_cast<const void*>((uintptr_t)dst[p]), PAGE);
            if (memcmp(got.data(), P.a_host.data() + (size_t)want[p] * PAGE, PAGE) != 0) die("%s: page %u of %u differs", what, p, n);
        }
        return;
    }
    std::vector<fma_k_page_desc> desc(n);
    for (uint32_t p = 0; p < n; ++p) desc[p] = fma_k_page_desc{dst[p], want[p] * WORDS};
    to_dev(P.d_desc, desc.data(), n * sizeof(fma_k_page_desc));
    fill_bytes(P.d_dig, 0, n * sizeof(uint64_t));
    if (fma_k_launch_page_digest(P.d_desc, n, P.d_dig, nullptr) != cudaSuccess) die("%s: K3 refused", what);
    sync_or_die();
    std::vector<uint64_t> dig(n);
    to_host(dig.data(), P.d_dig, n * sizeof(uint64_t));
    for (uint32_t p = 0; p < n; ++p)
        if (dig[p] != P.dig_a[want[p]]) die("%s: page %u of %u differs (K3 digest)", what, p, n);
}

static std::vector<uint64_t> pages_of(const unsigned char* base, const std::vector<uint32_t>& idx) {
    std::vector<uint64_t> v;
    for (uint32_t q : idx) v.push_back(addr(base + (size_t)q * PAGE));
    return v;
}
static std::vector<uint32_t> first_n(uint32_t n) {
    std::vector<uint32_t> v(n);
    std::iota(v.begin(), v.end(), 0u);
    return v;
}

static char g_what[160];
static const char* describe(int variant, const fma_k_tma_cfg* c, uint32_t n, const char* dir) {
    if (variant == FMA_K_VARIANT_LDG || !c) snprintf(g_what, sizeof(g_what), "%s %s of %u pages", variant == FMA_K_VARIANT_LDG ? "LDG" : "TMA (default shape)", dir, n);
    else snprintf(g_what, sizeof(g_what), "TMA %s of %u pages, tile %u B, %u stages, %u pipes, %u CTAs/SM", dir, n, c->tile_bytes, c->stages, c->pipes, c->ctas_per_sm);
    return g_what;
}

// K1: gather `want` (pages of a, `src` = where they sit) into the contiguous image b; K2: scatter b to `dst` pages
static void gather(Pool& P, int variant, const fma_k_tma_cfg* cfg, const std::vector<uint64_t>& src, const std::vector<uint32_t>& want) {
    const uint32_t n = (uint32_t)want.size();
    fill_bytes(P.b, 0xCD, n * PAGE);
    const char* what = describe(variant, cfg, n, "gather");
    if (fma_k_launch_page_copy(upload_tab(P, src), 0, nullptr, addr(P.b), n, variant, cfg, nullptr) != cudaSuccess) die("%s: refused", what);
    sync_or_die();
    expect_pages(P, pages_of(P.b, first_n(n)), want, what);
}
static void scatter(Pool& P, int variant, const fma_k_tma_cfg* cfg, const std::vector<uint64_t>& dst, const std::vector<uint32_t>& want) {
    const uint32_t n = (uint32_t)want.size();
    for (uint64_t d : dst) fill_bytes(reinterpret_cast<void*>((uintptr_t)d), 0xEF, PAGE);
    const char* what = describe(variant, cfg, n, "scatter");
    if (fma_k_launch_page_copy(nullptr, addr(P.b), upload_tab(P, dst), 0, n, variant, cfg, nullptr) != cudaSuccess) die("%s: refused", what);
    sync_or_die();
    expect_pages(P, dst, want, what);
}

// gather n randomly chosen pages of a into b, then scatter b to the same pages of c
static void gather_scatter(Pool& P, int variant, const fma_k_tma_cfg* cfg, uint32_t n, std::mt19937_64& rng) {
    std::vector<uint32_t> pick = first_n(P.n_a);
    std::shuffle(pick.begin(), pick.end(), rng);
    pick.resize(n);
    gather(P, variant, cfg, pages_of(P.a, pick), pick);
    scatter(P, variant, cfg, pages_of(P.c, pick), pick);
}

int main() {
    const bool fast = getenv("FMA_EMU_FAST") != nullptr;  // the CPU model under ThreadSanitizer: a subset
    std::mt19937_64 rng(20261015);

    // K0 / K3 on both sides of the grid cap, with the word counter wrapping past 2^64 inside the stream
    {
        const std::vector<uint32_t> counts = kOnDevice ? std::vector<uint32_t>{1, 16, 17, 200} : fast ? std::vector<uint32_t>{1, 17} : std::vector<uint32_t>{1, 16, 17};
        const uint64_t firsts[] = {0, (1ull << 40) + 12345, ~0ull - 3 * WORDS - 5, ~0ull};
        unsigned char* buf = dev_bytes((size_t)counts.back() * PAGE);
        for (uint32_t n : counts)
            for (uint64_t f : firsts) fill_and_digest(buf, n, f, rng);
        dev_free(buf);
        printf("K0/K3: page counts {");
        for (uint32_t n : counts) printf(" %u", n);
        printf(" } x 4 stream positions (one wrapping past 2^64) match the oracle\n");
    }

    Pool P;
    P.n_a = kOnDevice ? 67 : 8;
    P.a = dev_bytes((size_t)P.n_a * PAGE);
    P.b = dev_bytes((size_t)P.n_a * PAGE);
    P.c = dev_bytes((size_t)P.n_a * PAGE);
    P.d_tab = dev_array<uint64_t>(P.n_a);
    P.d_desc = dev_array<fma_k_page_desc>(P.n_a);
    P.d_dig = dev_array<uint64_t>(P.n_a);
    {   // the source pool: K0 over scattered descriptors == the oracle's stream, byte for byte
        P.a_host.resize((size_t)P.n_a * PAGE);
        fma_oracle_fill(reinterpret_cast<uint64_t*>(P.a_host.data()), P.n_a * WORDS, SEED, 0);
        std::vector<uint32_t> order = first_n(P.n_a);
        std::shuffle(order.begin(), order.end(), rng);
        std::vector<fma_k_page_desc> desc;
        for (uint32_t q : order) desc.push_back(fma_k_page_desc{addr(P.a + (size_t)q * PAGE), q * WORDS});
        to_dev(P.d_desc, desc.data(), desc.size() * sizeof(fma_k_page_desc));
        if (fma_k_launch_fill(P.d_desc, P.n_a, SEED, nullptr) != cudaSuccess) die("K0 refused");
        sync_or_die();
        std::vector<unsigned char> got((size_t)P.n_a * PAGE);
        to_host(got.data(), P.a, got.size());
        if (got != P.a_host) die("K0: the source pool differs from the oracle");
        for (uint32_t q = 0; q < P.n_a; ++q) P.dig_a.push_back(fma_oracle_digest(P.a_host.data() + (size_t)q * PAGE, PAGE, q * WORDS));
    }

    // every legal TMA shape, enumerated from the rules restated here (not from the wrapper)
    std::vector<fma_k_tma_cfg> shapes;
    for (uint32_t tile = 1024; tile <= (64u << 10); tile *= 2)
        for (uint32_t pipes = 1; pipes <= 4; ++pipes)
            for (uint32_t stages = 2; stages <= 8; ++stages)
                if ((uint64_t)pipes * stages * tile + 128 <= 227u * 1024u) shapes.push_back(fma_k_tma_cfg{tile, stages, pipes, 1});
    if (shapes.size() != 140) die("expected 140 legal TMA shapes, enumerated %zu", shapes.size());
    std::vector<fma_k_tma_cfg> runs;
    const size_t every = kOnDevice ? 1 : fast ? 10 : 4;  // the CPU model starts an OS thread per GPU thread: a subset there
    for (size_t i = 0; i < shapes.size(); ++i) {
        if (i % every) continue;
        runs.push_back(shapes[i]);
        fma_k_tma_cfg more = shapes[i];
        more.ctas_per_sm = (i % 2) ? 4 : 2;
        runs.push_back(more);
    }
    std::vector<size_t> big(runs.size());  // the seeded subset that also runs at n_a pages
    std::iota(big.begin(), big.end(), (size_t)0);
    std::shuffle(big.begin(), big.end(), rng);
    big.resize(std::min<size_t>(big.size(), kOnDevice ? 20 : fast ? 0 : 2));
    for (size_t r = 0; r < runs.size(); ++r) {
        gather_scatter(P, FMA_K_VARIANT_TMA, &runs[r], 1, rng);
        gather_scatter(P, FMA_K_VARIANT_TMA, &runs[r], 5, rng);
    }
    for (size_t r : big) gather_scatter(P, FMA_K_VARIANT_TMA, &runs[r], P.n_a, rng);
    printf("K1/K2 TMA: %zu of %zu legal shapes x 2 CTA counts = %zu shape runs, gather + scatter at 1 and 5 pages, %zu of them at %u pages\n",
           runs.size() / 2, shapes.size(), runs.size(), big.size(), P.n_a);

    for (uint32_t n : {1u, 5u, P.n_a}) gather_scatter(P, FMA_K_VARIANT_LDG, nullptr, n, rng);
    gather_scatter(P, FMA_K_VARIANT_TMA, nullptr, 5, rng);  // the default shape

    // a gather that lists one source page several times
    for (int variant : {FMA_K_VARIANT_TMA, FMA_K_VARIANT_LDG}) {
        const std::vector<uint32_t> want = {3, 1, 3, 2, 3};
        gather(P, variant, nullptr, pages_of(P.a, want), want);
    }

    // stages and pipes out of range are clamped (2..8, 1..4): the bytes are those of the clamped shape
    {
        const fma_k_tma_cfg clamped[] = {{4096, 0, 2, 1}, {4096, 1, 2, 1}, {4096, 9, 2, 1}, {4096, 4096, 2, 1}, {4096, 3, 0, 1},
                                         {4096, 3, 5, 1}, {1024, 4096, 5, 0}};
        for (const fma_k_tma_cfg& c : clamped) {
            gather_scatter(P, FMA_K_VARIANT_TMA, &c, 1, rng);
            gather_scatter(P, FMA_K_VARIANT_TMA, &c, 5, rng);
        }
        printf("K1/K2 TMA: %zu out-of-range shapes run as their clamped shapes\n", sizeof(clamped) / sizeof(clamped[0]));
    }

    // shapes that cannot run are refused by the launch wrapper before anything is launched: the destination keeps its bytes
    {
        const fma_k_tma_cfg bad[] = {{512, 3, 2, 1}, {3000, 3, 2, 1}, {4u << 20, 3, 2, 1}, {64u << 10, 8, 4, 1}, {64u << 10, 4, 1, 1},
                                     {32u << 10, 8, 1, 1}, {8u << 10, 8, 4, 1}, {16u << 10, 9, 2, 1}, {16u << 10, 4096, 2, 1}, {32u << 10, 3, 5, 1}};
        const uint64_t* tab = upload_tab(P, pages_of(P.a, first_n(2)));
        std::vector<unsigned char> got(2 * PAGE);
        for (const fma_k_tma_cfg& c : bad) {
            fill_bytes(P.b, 0xCD, 2 * PAGE);
            if (fma_k_launch_page_copy(tab, 0, nullptr, addr(P.b), 2, FMA_K_VARIANT_TMA, &c, nullptr) != cudaErrorInvalidValue)
                die("TMA shape tile %u, %u stages, %u pipes was not refused", c.tile_bytes, c.stages, c.pipes);
            sync_or_die();
            if (cudaGetLastError() != cudaSuccess) die("a refused shape left a launch error behind");
            to_host(got.data(), P.b, got.size());
            for (size_t i = 0; i < got.size(); ++i)
                if (got[i] != 0xCD) die("refused TMA shape (tile %u, %u stages, %u pipes) wrote byte %zu", c.tile_bytes, c.stages, c.pipes, i);
        }
        printf("K1/K2 TMA: %zu unfit shapes refused before any launch\n", sizeof(bad) / sizeof(bad[0]));
    }

    // zero-copy tiers: source or destination in mapped pinned host memory (the device reads / writes it over the link)
    {
        const uint32_t n = 5;
        Mapped h = host_mapped(n * PAGE);
        const fma_k_tma_cfg small{1024, 8, 4, 2};
        struct V { int variant; const fma_k_tma_cfg* cfg; };
        const std::vector<uint32_t> want = {4, 0, 3, 1, 2};
        for (V v : {V{FMA_K_VARIANT_TMA, nullptr}, V{FMA_K_VARIANT_TMA, &small}, V{FMA_K_VARIANT_LDG, nullptr}}) {
            memcpy(h.host, P.a_host.data(), n * PAGE);  // host page q = source page q
            gather(P, v.variant, v.cfg, pages_of(h.dev, want), want);
            memset(h.host, 0xEF, n * PAGE);
            if (fma_k_launch_page_copy(nullptr, addr(P.b), upload_tab(P, pages_of(h.dev, want)), 0, n, v.variant, v.cfg, nullptr) != cudaSuccess)
                die("scatter to mapped host memory refused");
            sync_or_die();
            if (memcmp(h.host, P.a_host.data(), n * PAGE) != 0) die("%s: scatter to mapped host memory differs", describe(v.variant, v.cfg, n, "scatter"));
        }
        printf("K1/K2: gather from and scatter to mapped pinned host memory match (TMA default, TMA 1 KiB x 8 x 4, LDG)\n");
    }

#if defined(FMA_GPU_TEST)
    puts("kernels (GPU) ok");
#else
    puts("kernels (emulated) ok");
#endif
    return 0;
}
