// fma_image_move on the host simulation under ThreadSanitizer / AddressSanitizer (built and run by tests/test_image_move.py): the file
// tier's reader / writer threads reading into and writing out of the host store, and the copy streams of the parking buffer.  Every
// failing move leaves the image where it was and a wake restores it bit-exact:
//   a filesystem without room for the image (fstatvfs answered by the interposer below): FMA_EIO, the file untouched;
//   writes that stop half way (the process's file-size limit, SIGXFSZ ignored): FMA_EIO, the file emptied;
//   a read from a truncated file: FMA_EIO, the host store the move made released; the same move succeeds on the whole file;
//   a local parking buffer whose cuMemCreate fails: FMA_ENOMEM, nothing parked.
// At the end no mapping, handle, VA reservation or file descriptor is left.
#include <atomic>
#include <cassert>
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include <dirent.h>
#include <dlfcn.h>
#include <sys/resource.h>
#include <sys/statvfs.h>
#include <sys/stat.h>
#include <unistd.h>

#include "fma_engine.h"

extern "C" unsigned long long hostsim_live_mapped_bytes();
extern "C" unsigned long long hostsim_live_handles();
extern "C" unsigned long long hostsim_live_reservations();
extern "C" void hostsim_fail_create_after(long n);

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

static int open_fds() {
    int n = 0;
    DIR* d = opendir("/proc/self/fd");
    if (!d) return -1;
    while (readdir(d)) ++n;
    closedir(d);
    return n;
}

static std::vector<uint64_t> digests(fma_engine_t* e) {
    int n = fma_segment_count(e);
    std::vector<uint64_t> d(n > 0 ? n : 1);
    OK(fma_digest_all(e, 0, d.data(), n));
    d.resize(n);
    return d;
}

static int tier_of(fma_engine_t* e) {
    fma_stats_t st;
    OK(fma_stats(e, &st));
    for (int i = 0; i < fma_segment_count(e); ++i) {
        fma_segment_info_t si;
        OK(fma_segment_info(e, i, &si));
        if (si.has_backup) assert(si.tier == st.tier && !si.mapped);
    }
    return st.tier;
}

static uint64_t stat_of(fma_engine_t* e, uint64_t fma_stats_t::*field) {
    fma_stats_t st;
    OK(fma_stats(e, &st));
    return st.*field;
}

static void set_fsize(rlim_t lim) {
    struct rlimit rl = {lim, RLIM_INFINITY};
    if (setrlimit(RLIMIT_FSIZE, &rl) != 0) abort();
}

static off_t file_size(const char* path) {
    struct stat sb;
    return stat(path, &sb) == 0 ? sb.st_size : -1;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const char* path = argv[1];
    signal(SIGXFSZ, SIG_IGN);
    const int fds0 = open_fds();
    fma_engine_t* e = nullptr;
    OK(fma_engine_create(0, nullptr, &e));
    const int w = fma_tag_intern(e, "weights"), kv = fma_tag_intern(e, "kv_cache");
    const size_t sizes[] = {8 * P, 3 * P, P, 12 * P, 6 * P, P, 5 * P};
    for (size_t s : sizes) { void* p; OK(fma_alloc(e, s, w, &p)); }
    void* pk; OK(fma_alloc(e, 20 * P, kv, &pk));
    OK(fma_set_option(e, "chunk_bytes", 5 * P));
    OK(fma_set_option(e, "load_chunk_bytes", 1 << 20));
    OK(fma_set_option(e, "load_slots", 3));
    OK(fma_set_option(e, "load_threads", 4));
    for (int i = 0; i < 7; ++i) OK(fma_fill_segment(e, i, 1234, (uint64_t)i << 24));
    const std::vector<uint64_t> d0 = digests(e);
    auto wake_exact = [&] {
        OK(fma_wake(e, 0, FMA_FLAG_VERIFY));
        const auto d = digests(e);
        for (int i = 0; i < 7; ++i) assert(d[i] == d0[i]);
    };
    const uint64_t W = 36 * P;
    OK(fma_file_store(e, path));

    // 0. no room on the filesystem: FMA_EIO before a byte is written, the file as it was
    {
        FILE* f0 = fopen(path, "wb");
        const std::vector<char> old(4096, 'x');
        assert(f0 && fwrite(old.data(), 1, old.size(), f0) == old.size());
        fclose(f0);
        OK(fma_sleep(e, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
        g_free_blocks.store(0);
        const int rc = fma_image_move(e, FMA_TIER_FILE);
        g_free_blocks.store(-1);
        assert(rc == FMA_EIO && tier_of(e) == FMA_TIER_HOST && file_size(path) == 4096);
        wake_exact();
    }

    // 1. the writes stop half way: FMA_EIO, the image still in the host store, the file emptied (no descriptor)
    OK(fma_sleep(e, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
    set_fsize(W / 2);
    int rc = fma_image_move(e, FMA_TIER_FILE);
    set_fsize(RLIM_INFINITY);
    assert(rc == FMA_EIO && tier_of(e) == FMA_TIER_HOST && file_size(path) == 0);
    OK(fma_image_move(e, FMA_TIER_FILE));          // with the limit lifted
    assert(tier_of(e) == FMA_TIER_FILE && file_size(path) == (off_t)(W + (2u << 20)));
    OK(fma_host_release(e));
    assert(stat_of(e, &fma_stats_t::host_store_bytes) == 0);

    // 2. a read from a truncated file: FMA_EIO, the host store the move made released; the whole file moves
    std::vector<char> keep((size_t)file_size(path));
    FILE* f = fopen(path, "rb");
    assert(f && fread(keep.data(), 1, keep.size(), f) == keep.size());
    fclose(f);
    assert(truncate(path, (off_t)(W / 3)) == 0);
    rc = fma_image_move(e, FMA_TIER_HOST);
    assert(rc == FMA_EIO && tier_of(e) == FMA_TIER_FILE && stat_of(e, &fma_stats_t::host_store_bytes) == 0);
    f = fopen(path, "wb");
    assert(f && fwrite(keep.data(), 1, keep.size(), f) == keep.size());
    fclose(f);
    OK(fma_image_move(e, FMA_TIER_HOST));
    assert(tier_of(e) == FMA_TIER_HOST);
    wake_exact();

    // 3. the local parking buffer cannot be created: FMA_ENOMEM, nothing parked; then it can
    OK(fma_sleep(e, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
    hostsim_fail_create_after(0);
    rc = fma_image_move(e, FMA_TIER_LOCAL);
    hostsim_fail_create_after(-1);
    assert(rc == FMA_ENOMEM && tier_of(e) == FMA_TIER_HOST && stat_of(e, &fma_stats_t::parked_bytes) == 0);
    OK(fma_image_move(e, FMA_TIER_LOCAL));
    OK(fma_image_move(e, FMA_TIER_FILE));
    OK(fma_peer_release(e));
    assert(stat_of(e, &fma_stats_t::parked_bytes) == 0 && tier_of(e) == FMA_TIER_FILE);
    wake_exact();

    // destroyed asleep in the file it was moved to
    OK(fma_sleep(e, 1ull << w, FMA_TIER_HOST, 0));
    OK(fma_image_move(e, FMA_TIER_FILE));
    OK(fma_engine_destroy(e));
    assert(hostsim_live_mapped_bytes() == 0 && hostsim_live_handles() == 0 && hostsim_live_reservations() == 0);
    assert(open_fds() == fds0);
    unlink(path);
    puts("move sanitizer scenario ok");
    return 0;
}
