// fma_image_prefetch on the host simulation under ThreadSanitizer / AddressSanitizer (built and run by tests/test_image_prefetch.py):
// the file tier's reader threads filling the pinned I/O windows and the copy streams taking them into the prefetch buffer.
//   readers that fail half way through a prefetch: FMA_EIO, no buffer left, and the same prefetch then succeeds;
//   prefetches from the file and from the host store racing fma_stats / fma_timeline on another thread;
//   a wake that fails after a prefetch (a cuMemMap refused): rolled back with the buffer kept, and its retry restores from it;
//   the engine destroyed while a prefetch exists.
// At the end no mapping, handle, VA reservation or file descriptor is left.
#include <atomic>
#include <cassert>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <initializer_list>
#include <string>
#include <thread>
#include <vector>

#include <dirent.h>
#include <dlfcn.h>
#include <unistd.h>

#include "fma_engine.h"

extern "C" unsigned long long hostsim_live_mapped_bytes();
extern "C" unsigned long long hostsim_live_handles();
extern "C" unsigned long long hostsim_live_reservations();
extern "C" void hostsim_fail_call_after(const char* name, long n);

#define OK(x)                                                                          \
    do {                                                                               \
        int _rc = (x);                                                                 \
        if (_rc != 0) { fprintf(stderr, "%s -> %d: %s\n", #x, _rc, fma_last_error()); abort(); } \
    } while (0)

static const size_t P = FMA_PAGE_BYTES;

// The engine is linked into this binary, so its pread calls land here: after g_reads_left more reads, every read fails with EIO.
static std::atomic<long> g_reads_left{-1};
template <class F>
static ssize_t counted(F real, int fd, void* buf, size_t n, off_t off) {
    if (g_reads_left.load() >= 0 && g_reads_left.fetch_sub(1) <= 0) {
        errno = EIO;
        return -1;
    }
    return real(fd, buf, n, off);
}
extern "C" ssize_t pread(int fd, void* buf, size_t n, off_t off) {
    using Real = ssize_t (*)(int, void*, size_t, off_t);
    static const Real real = reinterpret_cast<Real>(dlsym(RTLD_NEXT, "pread"));
    return counted(real, fd, buf, n, off);
}
extern "C" ssize_t pread64(int fd, void* buf, size_t n, off_t off) {
    using Real = ssize_t (*)(int, void*, size_t, off_t);
    static const Real real = reinterpret_cast<Real>(dlsym(RTLD_NEXT, "pread64"));
    return counted(real, fd, buf, n, off);
}

static int open_fds() {
    int n = 0;
    DIR* d = opendir("/proc/self/fd");
    if (!d) return -1;
    while (readdir(d)) ++n;
    closedir(d);
    return n;
}

static std::vector<uint64_t> digests(fma_engine_t* e) {
    const int n = fma_segment_count(e);
    std::vector<uint64_t> d(n > 0 ? n : 1);
    OK(fma_digest_all(e, 0, d.data(), n));
    d.resize(n);
    return d;
}

static uint64_t prefetched(fma_engine_t* e) {
    fma_stats_t st;
    OK(fma_stats(e, &st));
    return st.prefetched_bytes;
}

int main(int argc, char** argv) {
    const std::string path = argc > 1 ? argv[1] : "/tmp/fma_prefetch_sanitizer.fmaimg";
    const int fds0 = open_fds();
    fma_engine_t* e = nullptr;
    OK(fma_engine_create(0, nullptr, &e));
    const int w = fma_tag_intern(e, "weights"), kv = fma_tag_intern(e, "kv_cache");
    const size_t sizes[] = {8 * P, 3 * P, P, 12 * P, 6 * P, P, 5 * P};
    for (size_t s : sizes) { void* p; OK(fma_alloc(e, s, w, &p)); }
    void* pk; OK(fma_alloc(e, 20 * P, kv, &pk));
    OK(fma_set_option(e, "chunk_bytes", 5 * P));
    OK(fma_set_option(e, "load_chunk_bytes", 2 << 20));   // one page per window (what a verify of a file needs): many reads
    OK(fma_set_option(e, "load_slots", 3));
    OK(fma_set_option(e, "load_threads", 4));
    for (int i = 0; i < 7; ++i) OK(fma_fill_segment(e, i, 4321, (uint64_t)i << 24));
    const std::vector<uint64_t> d0 = digests(e);
    auto wake_exact = [&] {
        OK(fma_wake(e, 0, FMA_FLAG_VERIFY));
        const auto d = digests(e);
        for (int i = 0; i < 7; ++i) assert(d[i] == d0[i]);
        assert(prefetched(e) == 0);
    };
    const uint64_t W = 36 * P;
    OK(fma_file_store(e, path.c_str()));

    // 1. readers that fail half way: FMA_EIO and no buffer; then the same prefetch succeeds and the wake is exact
    OK(fma_sleep(e, 1ull << w, FMA_TIER_FILE, FMA_FLAG_VERIFY));
    g_reads_left = 7;
    int rc = fma_image_prefetch(e, 20 * P);
    g_reads_left = -1;
    if (rc != FMA_EIO) { fprintf(stderr, "a failed read gave %d: %s\n", rc, fma_last_error()); return 1; }
    assert(prefetched(e) == 0 && fma_is_sleeping(e) == 1);
    OK(fma_image_prefetch(e, 20 * P));
    assert(prefetched(e) == 16 * P);   // from the tail: 5, 1, 6; 12 does not fit what is left, 1 and 3 do, 8 does not
    int bad[8];
    rc = fma_image_verify(e, bad, 8);
    if (rc != 0) { fprintf(stderr, "verify of the prefetched image gave %d: %s\n", rc, fma_last_error()); return 1; }
    wake_exact();

    // 2. prefetches racing fma_stats / fma_timeline, from the file and from the host store
    for (int tier : {FMA_TIER_FILE, FMA_TIER_HOST}) {
        OK(fma_sleep(e, 1ull << w, tier, FMA_FLAG_VERIFY));
        prefetched(e);   // the sleep's kernel times are read here, before the race (fma_stats and an operation both read them)
        std::atomic<bool> stop{false};
        std::thread reader([&] {
            std::vector<char> buf(1 << 16);
            fma_stats_t st;
            while (!stop.load()) {
                fma_stats(e, &st);
                fma_timeline(e, buf.data(), buf.size());
            }
        });
        for (uint64_t cap : std::initializer_list<uint64_t>{W, 4 * P, 0, 16 * P}) OK(fma_image_prefetch(e, cap));
        stop = true;
        reader.join();
        assert(prefetched(e) > 0);
        wake_exact();
    }

    // 3. a wake that fails after a prefetch is rolled back with the buffer kept; its retry restores from it
    OK(fma_sleep(e, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
    OK(fma_image_prefetch(e, 16 * P));
    const uint64_t n = prefetched(e);
    assert(n > 0);
    hostsim_fail_call_after("cuMemMap", 1);
    rc = fma_wake(e, 0, FMA_FLAG_VERIFY);
    hostsim_fail_call_after("cuMemMap", -1);
    assert(rc != FMA_OK && fma_is_sleeping(e) == 1 && prefetched(e) == n);
    wake_exact();

    // 4. destroyed while a prefetch exists
    OK(fma_sleep(e, 1ull << w, FMA_TIER_FILE, 0));
    OK(fma_image_prefetch(e, W));
    assert(prefetched(e) == W);
    OK(fma_engine_destroy(e));
    unlink(path.c_str());
    if (hostsim_live_mapped_bytes() || hostsim_live_handles() || hostsim_live_reservations()) { fprintf(stderr, "VMM state left behind\n"); return 1; }
    if (open_fds() != fds0) { fprintf(stderr, "file descriptors left open: %d -> %d\n", fds0, open_fds()); return 1; }
    puts("prefetch sanitizer scenario ok");
    return 0;
}
