// File tier (FMA_TIER_FILE) on the host simulation under ThreadSanitizer / AddressSanitizer (built and run by tests/test_file_tier.py):
// reader / writer threads over the I/O windows beside the unmapper and mapper threads.  A sleep whose writes stop half way (the
// process's file-size limit, SIGXFSZ ignored) fails with FMA_EIO and a wake restores every segment; a wake from a truncated file
// fails, is rolled back and succeeds once the file is whole again; the retried sleep and an adoption by a second engine work; the
// engines are destroyed, one of them asleep, with nothing left mapped.  Before all that, a filesystem without room for the image
// (fstatvfs answered by the interposer below) makes the sleep fail with FMA_EIO, fully awake and with the file untouched.
#include <atomic>
#include <cassert>
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include <dlfcn.h>
#include <sys/resource.h>
#include <sys/statvfs.h>
#include <sys/stat.h>
#include <unistd.h>

#include "fma_engine.h"

extern "C" unsigned long long hostsim_live_mapped_bytes();

#define OK(x)                                                                          \
    do {                                                                               \
        int _rc = (x);                                                                 \
        if (_rc != 0) { fprintf(stderr, "%s -> %d: %s\n", #x, _rc, fma_last_error()); abort(); } \
    } while (0)

static const size_t P = FMA_PAGE_BYTES;

// The engine is linked into this binary, so its fstatvfs calls land here: >= 0 = the free blocks the filesystem reports.
static std::atomic<long> g_free_blocks{-1};
extern "C" int fstatvfs(int fd, struct statvfs* buf) noexcept {
    using Real = int (*)(int, struct statvfs*);
    static const Real real = reinterpret_cast<Real>(dlsym(RTLD_NEXT, "fstatvfs"));
    const int r = real(fd, buf);
    if (r == 0 && g_free_blocks.load() >= 0) buf->f_bavail = (fsblkcnt_t)g_free_blocks.load();
    return r;
}

static std::vector<uint64_t> digests(fma_engine_t* e) {
    int n = fma_segment_count(e);
    std::vector<uint64_t> d(n > 0 ? n : 1);
    OK(fma_digest_all(e, 0, d.data(), n));
    d.resize(n);
    return d;
}

static int n_mapped(fma_engine_t* e) {
    int k = 0;
    for (int i = 0; i < fma_segment_count(e); ++i) {
        fma_segment_info_t si;
        OK(fma_segment_info(e, i, &si));
        k += si.mapped;
    }
    return k;
}

static void set_fsize(rlim_t lim) {
    struct rlimit rl = {lim, RLIM_INFINITY};
    if (setrlimit(RLIMIT_FSIZE, &rl) != 0) abort();
}

static fma_engine_t* make(int* w, std::vector<uint64_t>* d0) {
    fma_engine_t* e = nullptr;
    OK(fma_engine_create(0, nullptr, &e));
    *w = fma_tag_intern(e, "weights");
    const int kv = fma_tag_intern(e, "kv_cache");
    const size_t sizes[] = {8 * P, 3 * P, P, 12 * P, 6 * P, P, 5 * P};
    for (size_t s : sizes) { void* p; OK(fma_alloc(e, s, *w, &p)); }
    void* pk; OK(fma_alloc(e, 20 * P, kv, &pk));
    OK(fma_set_option(e, "chunk_bytes", 5 * P));
    OK(fma_set_option(e, "load_chunk_bytes", 1 << 20));
    OK(fma_set_option(e, "load_slots", 3));
    OK(fma_set_option(e, "load_threads", 4));
    if (d0) {
        for (int i = 0; i < 7; ++i) OK(fma_fill_segment(e, i, 1234, (uint64_t)i << 24));
        *d0 = digests(e);
    }
    return e;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const char* path = argv[1];
    signal(SIGXFSZ, SIG_IGN);
    int w = 0;
    std::vector<uint64_t> d0;
    fma_engine_t* a = make(&w, &d0);
    auto same = [&](fma_engine_t* e) { const auto d = digests(e); for (int i = 0; i < 7; ++i) assert(d[i] == d0[i]); };
    OK(fma_file_store(a, path));
    const uint64_t W = 36 * P;

    // 0. no room on the filesystem: FMA_EIO before anything is released or truncated
    {
        const std::string full = std::string(path) + ".full";
        FILE* f0 = fopen(full.c_str(), "wb");
        const std::vector<char> old(4096, 'x');
        assert(f0 && fwrite(old.data(), 1, old.size(), f0) == old.size());
        fclose(f0);
        OK(fma_file_store(a, full.c_str()));
        g_free_blocks.store(0);
        const int rc0 = fma_sleep(a, 1ull << w, FMA_TIER_FILE, FMA_FLAG_VERIFY);
        g_free_blocks.store(-1);
        assert(rc0 == FMA_EIO && n_mapped(a) == 8 && fma_is_sleeping(a) == 0);
        struct stat sb0;
        assert(stat(full.c_str(), &sb0) == 0 && sb0.st_size == 4096);
        same(a);
        unlink(full.c_str());
        OK(fma_file_store(a, path));
    }

    // 1. the writes stop half way: FMA_EIO, the released segments are in the file, a wake restores everything
    set_fsize(W / 2);
    int rc = fma_sleep(a, 1ull << w, FMA_TIER_FILE, FMA_FLAG_VERIFY);
    set_fsize(RLIM_INFINITY);
    assert(rc == FMA_EIO);
    const int left = n_mapped(a);
    assert(left > 0 && left < 8);
    OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
    same(a);

    // 2. a whole sleep, then a wake from a truncated file: rolled back, and retried once the file is whole again
    OK(fma_sleep(a, 1ull << w, FMA_TIER_FILE, FMA_FLAG_VERIFY));
    fma_stats_t st;
    OK(fma_stats(a, &st));
    assert(st.tier == FMA_TIER_FILE && st.host_store_bytes == 0 && st.image_store_bytes == W && st.io_buffer_bytes == 3 * ((1 << 20) + 8192));
    struct stat sb;
    assert(stat(path, &sb) == 0 && (uint64_t)sb.st_size == W + (2u << 20));
    std::vector<char> keep((size_t)sb.st_size);
    FILE* f = fopen(path, "rb");
    assert(f && fread(keep.data(), 1, keep.size(), f) == keep.size());
    fclose(f);
    assert(truncate(path, (off_t)(W / 3)) == 0);
    rc = fma_wake(a, 0, 0);
    assert(rc == FMA_EIO && n_mapped(a) == 0);
    f = fopen(path, "wb");
    assert(f && fwrite(keep.data(), 1, keep.size(), f) == keep.size());
    fclose(f);
    OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
    same(a);

    // 3. a second engine adopts the file while the first is asleep on it too; both wake bit-exact
    OK(fma_sleep(a, 1ull << w, FMA_TIER_FILE, FMA_FLAG_VERIFY));
    int wb = 0;
    fma_engine_t* b = make(&wb, nullptr);
    OK(fma_image_adopt_file(b, path, 1ull << wb, 0));
    assert(fma_is_sleeping(b) == 1);
    OK(fma_wake(b, 0, FMA_FLAG_VERIFY));
    same(b);
    OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
    same(a);

    // 4. destroyed, one of them asleep in the file tier
    OK(fma_sleep(b, 1ull << wb, FMA_TIER_HOST, 0));
    OK(fma_sleep(a, 1ull << w, FMA_TIER_FILE, 0));
    OK(fma_engine_destroy(a));
    OK(fma_engine_destroy(b));
    assert(hostsim_live_mapped_bytes() == 0);
    unlink(path);
    puts("file sanitizer scenario ok");
    return 0;
}
