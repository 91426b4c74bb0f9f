// fma_image_verify on the host simulation under ThreadSanitizer / AddressSanitizer (built and run by tests/test_image_verify.py):
//   a file-tier image checked through the I/O windows, intact and with one flipped byte;
//   a check whose file readers fail half way (pread answered with EIO by the interposer below): FMA_EIO, nothing changed, and the
//   next check succeeds;
//   checks racing fma_stats / fma_timeline from another thread;
//   a wake afterwards restores every segment bit-exact.
// At the end no mapping, handle, VA reservation or file descriptor is left.
#include <atomic>
#include <cassert>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include <dirent.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <unistd.h>

#include "fma_engine.h"

extern "C" unsigned long long hostsim_live_mapped_bytes();
extern "C" unsigned long long hostsim_live_handles();
extern "C" unsigned long long hostsim_live_reservations();

#define OK(x)                                                                          \
    do {                                                                               \
        int _rc = (x);                                                                 \
        if (_rc != 0) { fprintf(stderr, "%s -> %d: %s\n", #x, _rc, fma_last_error()); abort(); } \
    } while (0)

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
    std::vector<uint64_t> d(n);
    for (int i = 0; i < n; ++i) OK(fma_digest_segment(e, i, &d[i]));
    return d;
}

int main(int argc, char** argv) {
    const std::string path = argc > 1 ? argv[1] : "/tmp/fma_verify_sanitizer.fmaimg";
    const int fds0 = open_fds();
    fma_engine_t* e = nullptr;
    OK(fma_engine_create(0, nullptr, &e));
    const int w = fma_tag_intern(e, "weights");
    const size_t sizes[] = {6u << 20, 2u << 20, 10u << 20, 4u << 20};
    for (size_t i = 0; i < 4; ++i) {
        void* p = nullptr;
        OK(fma_alloc(e, sizes[i], w, &p));
        OK(fma_fill_segment(e, (int)i, 99 + i, i << 24));
    }
    const std::vector<uint64_t> before = digests(e);
    OK(fma_set_option(e, "load_chunk_bytes", 2 << 20));   // one stored page per window: many reads
    OK(fma_set_option(e, "load_slots", 3));
    OK(fma_file_store(e, path.c_str()));
    OK(fma_sleep(e, 1ull << w, FMA_TIER_FILE, FMA_FLAG_VERIFY));
    int bad[8];
    assert(fma_image_verify(e, bad, 8) == 0);

    // readers that fail half way
    g_reads_left = 5;
    const int rc = fma_image_verify(e, bad, 8);
    g_reads_left = -1;
    if (rc != FMA_EIO) { fprintf(stderr, "a failed read gave %d: %s\n", rc, fma_last_error()); return 1; }
    assert(fma_is_sleeping(e) == 1 && fma_image_verify(e, bad, 8) == 0);

    // one flipped byte in the third segment's stored bytes
    {
        fma_segment_info_t si;
        OK(fma_segment_info(e, 2, &si));
        const int fd = open(path.c_str(), O_RDWR);
        unsigned char b = 0;
        assert(pread(fd, &b, 1, (off_t)si.packed_offset + 12345) == 1);
        b ^= 0x20;
        assert(pwrite(fd, &b, 1, (off_t)si.packed_offset + 12345) == 1);
        assert(fma_image_verify(e, bad, 8) == 1 && bad[0] == 2);
        b ^= 0x20;
        assert(pwrite(fd, &b, 1, (off_t)si.packed_offset + 12345) == 1);
        close(fd);
    }

    // checks racing fma_stats / fma_timeline
    std::atomic<bool> stop{false};
    std::thread reader([&] {
        std::vector<char> buf(1 << 16);
        fma_stats_t st;
        while (!stop.load()) {
            fma_stats(e, &st);
            fma_timeline(e, buf.data(), buf.size());
        }
    });
    for (int k = 0; k < 4; ++k) assert(fma_image_verify(e, bad, 8) == 0);
    stop = true;
    reader.join();

    OK(fma_wake(e, 0, FMA_FLAG_VERIFY));
    if (digests(e) != before) { fprintf(stderr, "the wake after the checks is not bit-exact\n"); return 1; }
    OK(fma_engine_destroy(e));
    unlink(path.c_str());
    if (hostsim_live_mapped_bytes() || hostsim_live_handles() || hostsim_live_reservations()) { fprintf(stderr, "VMM state left behind\n"); return 1; }
    if (open_fds() != fds0) { fprintf(stderr, "file descriptors left open: %d -> %d\n", fds0, open_fds()); return 1; }
    puts("verify sanitizer scenario ok");
    return 0;
}
