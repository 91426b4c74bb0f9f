// Write-behind file-tier sleeps (FMA_FLAG_WRITE_BEHIND) on the host simulation under ThreadSanitizer / AddressSanitizer (built and
// run by tests/test_write_behind.py): the job's writer threads and its commit beside the calls that pre-empt it.  A commit races a
// wake (and a thread polling fma_image_writeback) over many rounds; every call that takes the operation lock pre-empts a job still
// writing and then works on a host-tier image; an engine is destroyed while its job writes; a job whose writes stop half way (the
// process's file-size limit, SIGXFSZ ignored) reports FMA_EIO once and leaves the image in the host tier.  Every wake is bit-exact,
// and at the end no mapping, handle, reservation or thread is left.
#include <atomic>
#include <cassert>
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include <sys/resource.h>
#include <sys/stat.h>
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

static const size_t P = FMA_PAGE_BYTES;
static const uint64_t W = 36 * P;

static std::vector<uint64_t> digests(fma_engine_t* e) {
    int n = fma_segment_count(e);
    std::vector<uint64_t> d(n > 0 ? n : 1);
    OK(fma_digest_all(e, 0, d.data(), n));
    d.resize(n);
    return d;
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
    OK(fma_set_option(e, "load_threads", 4));
    for (int i = 0; i < 7; ++i) OK(fma_fill_segment(e, i, 1234, (uint64_t)i << 24));
    *d0 = digests(e);
    OK(fma_host_reserve(e, W));
    return e;
}

static int tier_of(fma_engine_t* e) {
    fma_stats_t st;
    OK(fma_stats(e, &st));
    return st.tier;
}

static off_t size_of(const char* path) {
    struct stat sb;
    return stat(path, &sb) == 0 ? sb.st_size : -1;
}

static int threads() {   // of this process
    FILE* f = fopen("/proc/self/status", "r");
    char line[256];
    int n = -1;
    while (f && fgets(line, sizeof(line), f))
        if (sscanf(line, "Threads: %d", &n) == 1) break;
    if (f) fclose(f);
    return n;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const char* path = argv[1];
    signal(SIGXFSZ, SIG_IGN);
    int w = 0;
    std::vector<uint64_t> d0;
    fma_engine_t* a = make(&w, &d0);
    const int threads0 = threads();   // (after the first threads of the process: a sanitizer's own helper thread has started)
    auto same = [&](fma_engine_t* e) { const auto d = digests(e); for (int i = 0; i < 7; ++i) assert(d[i] == d0[i]); };
    const uint64_t mask = 1ull << w;
    OK(fma_file_store(a, path));

    // 1. a commit races a wake: whichever takes the lock first, the wake is bit-exact and the file is whole or empty
    std::atomic<bool> stop{false};
    std::thread poller([&] {
        while (!stop.load()) {
            uint64_t pending = 0;
            const int r = fma_image_writeback(a, 0.0005, &pending);
            assert(r == 0 || r == 1);
            assert(pending <= W);
        }
    });
    int committed = 0;
    for (int round = 0; round < 12; ++round) {
        OK(fma_sleep(a, mask, FMA_TIER_FILE, FMA_FLAG_WRITE_BEHIND | FMA_FLAG_VERIFY));
        if (round % 3 == 1) usleep(2000);
        if (round % 3 == 2) assert(fma_image_writeback(a, -1.0, nullptr) == 0);
        committed += tier_of(a) == FMA_TIER_FILE;
        OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
        same(a);
        const off_t sz = size_of(path);
        assert(sz == 0 || sz == (off_t)(W + (2u << 20)));
        OK(fma_host_reserve(a, W));   // (a committed image released the store: the next round needs it again)
    }
    stop.store(true);
    poller.join();
    assert(committed >= 4);

    // 2. every call that takes the operation lock pre-empts a job still writing, then sees a host-tier image
    setenv("FMA_WB_ITEM_DELAY_MS", "20", 1);
    const std::string other = std::string(path) + ".other";
    for (int call = 0; call < 8; ++call) {
        OK(fma_sleep(a, mask, FMA_TIER_FILE, FMA_FLAG_WRITE_BEHIND | FMA_FLAG_VERIFY));
        uint64_t pending = 0;
        assert(fma_image_writeback(a, 0, &pending) == 1 && pending > 0);
        int bad = -1, fd = -1;
        switch (call) {
            case 0: assert(fma_image_verify(a, &bad, 1) == 0); break;
            case 1: OK(fma_image_prefetch(a, 4 * P)); break;
            case 2: OK(fma_image_move(a, FMA_TIER_FILE)); break;
            case 3: OK(fma_file_store(a, other.c_str())); break;
            case 4: OK(fma_host_reserve(a, W)); break;
            case 5: assert(fma_host_release(a) == FMA_ESTATE); break;       // the store holds the sleeping image
            case 6: assert(fma_image_export(a, &fd) == FMA_ESTATE); break;  // not shareable (no memfd store)
            case 7: assert(fma_sleep(a, mask, FMA_TIER_FILE, FMA_FLAG_WRITE_BEHIND) == 0); break;   // asleep: a no-op
        }
        assert(fma_image_writeback(a, 0, nullptr) == 0);
        assert(tier_of(a) == (call == 2 ? FMA_TIER_FILE : FMA_TIER_HOST));
        if (call != 2) assert(size_of(path) == 0);
        OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
        same(a);
        if (call == 2) OK(fma_host_reserve(a, W));
        if (call == 3) OK(fma_file_store(a, path));
    }
    unlink(other.c_str());

    // 3. a job whose writes stop half way: FMA_EIO once, the image stays in the host tier, the file is emptied
    unsetenv("FMA_WB_ITEM_DELAY_MS");
    struct rlimit rl = {(rlim_t)(W / 2), RLIM_INFINITY};
    assert(setrlimit(RLIMIT_FSIZE, &rl) == 0);
    OK(fma_sleep(a, mask, FMA_TIER_FILE, FMA_FLAG_WRITE_BEHIND | FMA_FLAG_VERIFY));
    assert(fma_image_writeback(a, -1.0, nullptr) == FMA_EIO);
    assert(fma_image_writeback(a, 0, nullptr) == 0);
    rl.rlim_cur = RLIM_INFINITY;
    assert(setrlimit(RLIMIT_FSIZE, &rl) == 0);
    assert(tier_of(a) == FMA_TIER_HOST && size_of(path) == 0);
    OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
    same(a);

    // 4. destroyed while its job writes (and a second engine destroyed with a committed image)
    int wb2 = 0;
    std::vector<uint64_t> d1;
    fma_engine_t* b = make(&wb2, &d1);
    const std::string bpath = std::string(path) + ".b";
    OK(fma_file_store(b, bpath.c_str()));
    OK(fma_sleep(b, 1ull << wb2, FMA_TIER_FILE, FMA_FLAG_WRITE_BEHIND));
    assert(fma_image_writeback(b, -1.0, nullptr) == 0 && tier_of(b) == FMA_TIER_FILE);
    setenv("FMA_WB_ITEM_DELAY_MS", "20", 1);
    OK(fma_sleep(a, mask, FMA_TIER_FILE, FMA_FLAG_WRITE_BEHIND));
    assert(fma_image_writeback(a, 0, nullptr) == 1);
    OK(fma_engine_destroy(a));
    assert(size_of(path) == 0);
    OK(fma_engine_destroy(b));
    unsetenv("FMA_WB_ITEM_DELAY_MS");
    assert(hostsim_live_mapped_bytes() == 0 && hostsim_live_handles() == 0 && hostsim_live_reservations() == 0);
    assert(threads() == threads0);
    unlink(path);
    unlink(bpath.c_str());
    puts("write-behind sanitizer scenario ok");
    return 0;
}
