// Every HBM buffer the engine maps at a VA of its own — the peer / local parking buffer, the resident share, an attached parking
// buffer, the multi-path staging of fma_paths_set and fma_paths_attach, the owner's helper staging and a node-level parking buffer —
// with each driver and runtime call of its setup failed in turn through the simulation's fault injection (built and run by
// tests/test_engine_hostsim.py under ThreadSanitizer and under ASan+UBSan+LeakSan).  After every failure:
//   * the code follows one rule: cuMemCreate / import out of memory -> FMA_ENOMEM, any other failed call -> FMA_ECUDA;
//   * no mapping, handle, VA reservation or open fd is left behind;
//   * the engine still sleeps and wakes bit-exact.
// A failed resident-share allocation is not an error: the sleep keeps everything in the host store.  Last, the parking-buffer
// calls refuse while a resident share sleeps (they ask "is any image outside the host store?").
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <dirent.h>
#include <unistd.h>

#include "fma_engine.h"

extern "C" unsigned long long hostsim_live_mapped_bytes();
extern "C" unsigned long long hostsim_live_handles();
extern "C" unsigned long long hostsim_live_reservations();
extern "C" void hostsim_fail_create_after(long n);
extern "C" void hostsim_fail_call_after(const char* name, long n);

#define OK(x)                                                                          \
    do {                                                                               \
        int _rc = (x);                                                                 \
        if (_rc != 0) { fprintf(stderr, "%s -> %d: %s\n", #x, _rc, fma_last_error()); abort(); } \
    } while (0)

static int g_failures = 0;   // every failed check is reported, then the scenario fails at the end
#define CHECK(cond, ...)                                                                                  \
    do {                                                                                                  \
        if (!(cond)) { ++g_failures; fprintf(stderr, "FAILED (%s): ", #cond); fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } \
    } while (0)

static const size_t P = FMA_PAGE_BYTES;

struct Live {
    unsigned long long mapped, handles, reservations, fds;
    bool operator==(const Live& o) const { return mapped == o.mapped && handles == o.handles && reservations == o.reservations && fds == o.fds; }
};

static Live live() {
    Live l{hostsim_live_mapped_bytes(), hostsim_live_handles(), hostsim_live_reservations(), 0};
    if (DIR* d = opendir("/proc/self/fd")) {
        while (dirent* de = readdir(d)) l.fds += de->d_name[0] != '.';
        closedir(d);
    }
    return l;
}

static void arm(const char* call, long n) {
    if (!strcmp(call, "cuMemCreate")) hostsim_fail_create_after(n);
    else hostsim_fail_call_after(call, n);
}

static fma_engine_t* g_e = nullptr;
static int g_w = 0;
static std::vector<uint64_t> g_d0;

static std::vector<uint64_t> digests() {
    std::vector<uint64_t> d(fma_segment_count(g_e));
    OK(fma_digest_all(g_e, 0, d.data(), (int)d.size()));
    return d;
}

static void sleeps_and_wakes_bit_exact(const char* what) {
    int rc = fma_sleep(g_e, 1ull << g_w, FMA_TIER_HOST, FMA_FLAG_VERIFY);
    if (rc == FMA_OK) rc = fma_wake(g_e, 0, FMA_FLAG_VERIFY);
    CHECK(rc == FMA_OK && fma_is_sleeping(g_e) == 0 && digests() == g_d0, "%s: the engine no longer sleeps and wakes bit-exact (%d: %s)", what, rc,
          fma_last_error());
}

// The want-code of a failed call under the rule.
static int want_code(const char* call) {
    return !strcmp(call, "cuMemCreate") || !strcmp(call, "cuMemImportFromShareableHandle") ? FMA_ENOMEM : FMA_ECUDA;
}

// Fails the 1st, 2nd, ... call of `call` that `attempt` makes, until an attempt makes fewer calls and succeeds; `undo` gives back
// what that attempt made.
template <class A, class U>
static void each_failure(const char* what, const char* call, A attempt, U undo) {
    int failed = 0;
    for (long n = 0; n < 32; ++n) {
        const Live before = live();
        arm(call, n);
        const int rc = attempt();
        arm(call, -1);
        if (rc == FMA_OK) {
            undo();
            CHECK(failed > 0, "%s never calls %s", what, call);
            return;
        }
        ++failed;
        CHECK(rc == want_code(call), "%s, %s #%ld failed: returned %d, want %d (%s)", what, call, n, rc, want_code(call), fma_last_error());
        const Live after = live();
        CHECK(after == before, "%s, %s #%ld failed: mapped %llu -> %llu, handles %llu -> %llu, reservations %llu -> %llu, fds %llu -> %llu", what, call, n,
              before.mapped, after.mapped, before.handles, after.handles, before.reservations, after.reservations, before.fds, after.fds);
        sleeps_and_wakes_bit_exact(what);
    }
    CHECK(false, "%s: %s never succeeds", what, call);
}

static const char* const kCreate[] = {"cuMemCreate", "cuMemAddressReserve", "cuMemMap", "cuMemSetAccess"};
static const char* const kImport[] = {"cuMemImportFromShareableHandle", "cuMemAddressReserve", "cuMemMap", "cuMemSetAccess"};
static const char* const kPath[] = {"cuMemCreate", "cuMemAddressReserve", "cuMemMap", "cuMemSetAccess", "cudaStreamCreateWithFlags", "cudaEventCreateWithFlags"};
static const char* const kAttach[] = {"cuMemCreate", "cuMemImportFromShareableHandle", "cuMemAddressReserve", "cuMemMap", "cuMemSetAccess",
                                      "cudaStreamCreateWithFlags", "cudaEventCreateWithFlags"};
static const char* const kHelper[] = {"cuMemCreate", "cuMemExportToShareableHandle", "cuMemAddressReserve", "cuMemMap", "cuMemSetAccess",
                                      "cudaStreamCreateWithFlags", "cudaEventCreateWithFlags"};
static const char* const kParking[] = {"cuMemCreate", "cuMemExportToShareableHandle"};

static uint64_t resident_bytes() {
    fma_stats_t st;
    OK(fma_stats(g_e, &st));
    return st.resident_bytes;
}

int main() {
    OK(fma_engine_create(0, nullptr, &g_e));
    g_w = fma_tag_intern(g_e, "weights");
    for (size_t pages : {6, 3, 1, 4}) {
        void* p;
        OK(fma_alloc(g_e, pages * P, g_w, &p));
        OK(fma_fill_segment(g_e, fma_segment_count(g_e) - 1, 4321, (uint64_t)pages << 30));
    }
    g_d0 = digests();
    OK(fma_host_reserve(g_e, 14 * P));
    sleeps_and_wakes_bit_exact("first cycle");
    const int helper_dev = 1;
    // made once, up front: what the attach calls import
    uint64_t parking = 0, staging = 0;
    int parking_fd = -1, staging_fd = -1;
    OK(fma_parking_create(1, 14 * P, &parking, &parking_fd));
    OK(fma_helper_open(1, 2 * P, 2, &staging, &staging_fd));

    for (const char* call : kCreate)
        each_failure("fma_peer_reserve", call, [] { return fma_peer_reserve(g_e, 1, 14 * P); }, [] { OK(fma_peer_release(g_e)); });
    for (const char* call : kCreate)
        each_failure("local-tier sleep", call, [] { return fma_sleep(g_e, 1ull << g_w, FMA_TIER_LOCAL, FMA_FLAG_VERIFY); },
                     [] { OK(fma_wake(g_e, 0, FMA_FLAG_VERIFY)); OK(fma_peer_release(g_e)); CHECK(digests() == g_d0, "local-tier cycle"); });
    for (const char* call : kImport)
        each_failure("fma_peer_attach", call, [&] { return fma_peer_attach(g_e, parking_fd, 14 * P); }, [] { OK(fma_peer_release(g_e)); });
    for (const char* call : kPath)
        each_failure("fma_paths_set", call, [&] { return fma_paths_set(g_e, &helper_dev, 1, 2 * P, 2); }, [] { OK(fma_paths_set(g_e, nullptr, 0, 0, 0)); });
    for (const char* call : kAttach) {
        int mbox = -1;
        each_failure("fma_paths_attach", call, [&] { return fma_paths_attach(g_e, &staging_fd, 1, 2 * P, 2, &mbox); },
                     [] { OK(fma_paths_set(g_e, nullptr, 0, 0, 0)); });
    }
    for (const char* call : kHelper) {
        uint64_t h = 0;
        int fd = -1;
        each_failure("fma_helper_open", call, [&] { return fma_helper_open(1, 2 * P, 2, &h, &fd); }, [&] { OK(fma_helper_close(h)); close(fd); });
    }
    for (const char* call : kParking) {
        uint64_t h = 0;
        int fd = -1;
        each_failure("fma_parking_create", call, [&] { return fma_parking_create(1, 4 * P, &h, &fd); }, [&] { OK(fma_parking_destroy(h)); close(fd); });
    }

    // The resident share's allocation fails inside a host-tier sleep: the sleep keeps the whole image in the host store.
    OK(fma_set_option(g_e, "resident_bytes", 4 * P));
    for (const char* call : kCreate) {
        int fell_back = 0;
        for (long n = 0; n < 32; ++n) {
            // what a plain host-tier sleep leaves: the fallback must leave exactly that
            OK(fma_set_option(g_e, "resident_bytes", 0));
            OK(fma_sleep(g_e, 1ull << g_w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
            const Live plain = live();
            OK(fma_wake(g_e, 0, FMA_FLAG_VERIFY));
            OK(fma_set_option(g_e, "resident_bytes", 4 * P));
            arm(call, n);
            const int rc = fma_sleep(g_e, 1ull << g_w, FMA_TIER_HOST, FMA_FLAG_VERIFY);
            arm(call, -1);
            CHECK(rc == FMA_OK, "resident share, %s #%ld failed: the sleep returned %d (%s)", call, n, rc, fma_last_error());
            const bool resident = resident_bytes() > 0;
            const Live after = live();
            if (!resident)
                CHECK(after == plain, "resident share, %s #%ld failed: mapped %llu -> %llu, handles %llu -> %llu, reservations %llu -> %llu, fds %llu -> %llu",
                      call, n, plain.mapped, after.mapped, plain.handles, after.handles, plain.reservations, after.reservations, plain.fds, after.fds);
            OK(fma_wake(g_e, 0, FMA_FLAG_VERIFY));
            CHECK(digests() == g_d0, "resident share, %s #%ld failed: the wake is not bit-exact", call, n);
            if (resident) break;
            ++fell_back;
        }
        CHECK(fell_back > 0, "a resident share's allocation never calls %s", call);
    }

    // While a resident share sleeps, the parking-buffer calls refuse as if the parking buffer held the image.
    OK(fma_sleep(g_e, 1ull << g_w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
    CHECK(resident_bytes() > 0, "no resident share");
    CHECK(fma_peer_reserve(g_e, 1, 14 * P) == FMA_ESTATE, "fma_peer_reserve while a resident share sleeps");
    CHECK(fma_peer_release(g_e) == FMA_ESTATE, "fma_peer_release while a resident share sleeps");
    CHECK(fma_peer_attach(g_e, parking_fd, 14 * P) == FMA_ESTATE, "fma_peer_attach while a resident share sleeps");
    OK(fma_wake(g_e, 0, FMA_FLAG_VERIFY));
    OK(fma_peer_reserve(g_e, 1, 14 * P));
    OK(fma_peer_release(g_e));
    OK(fma_set_option(g_e, "resident_bytes", 0));

    OK(fma_helper_close(staging));
    OK(fma_parking_destroy(parking));
    close(staging_fd);
    close(parking_fd);
    OK(fma_engine_destroy(g_e));
    CHECK(hostsim_live_mapped_bytes() == 0 && hostsim_live_handles() == 0 && hostsim_live_reservations() == 0, "left behind at the end");
    if (g_failures) {
        fprintf(stderr, "%d checks failed\n", g_failures);
        return 1;
    }
    puts("vmm failure scenario ok");
    return 0;
}
