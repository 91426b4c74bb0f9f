// Resident share (option "resident_bytes") on the host simulation under ThreadSanitizer / AddressSanitizer (built and run by
// tests/test_resident_share.py), with failures injected through the simulation's counters: the resident allocation fails (the
// sleep falls back to a plain host-tier sleep), a D2H fails half way through a sleep, cuMemCreate fails on a later run of a wake
// (rollback, then the retry restores everything from the buffer that survived), and the engine is destroyed while asleep.
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "fma_engine.h"

extern "C" unsigned long long hostsim_live_mapped_bytes();
extern "C" unsigned long long hostsim_live_handles();
extern "C" void hostsim_fail_create_after(long n);
extern "C" void hostsim_fail_memcpy_after(long n);

#define OK(x)                                                                          \
    do {                                                                               \
        int _rc = (x);                                                                 \
        if (_rc != 0) { fprintf(stderr, "%s -> %d: %s\n", #x, _rc, fma_last_error()); abort(); } \
    } while (0)

static const size_t P = FMA_PAGE_BYTES;

static std::vector<uint64_t> digests(fma_engine_t* e) {
    int n = fma_segment_count(e);
    std::vector<uint64_t> d(n > 0 ? n : 1);
    OK(fma_digest_all(e, 0, d.data(), n));
    d.resize(n);
    return d;
}

static fma_stats_t stats(fma_engine_t* e) {
    fma_stats_t st;
    OK(fma_stats(e, &st));
    return st;
}

static int n_resident(fma_engine_t* e) {
    int k = 0;
    for (int i = 0; i < fma_segment_count(e); ++i) {
        fma_segment_info_t si;
        OK(fma_segment_info(e, i, &si));
        k += si.has_backup && si.tier == FMA_TIER_LOCAL;
    }
    return k;
}

int main() {
    fma_engine_t* a = nullptr;
    OK(fma_engine_create(0, nullptr, &a));
    int w = fma_tag_intern(a, "weights"), kv = fma_tag_intern(a, "kv_cache");
    const size_t sizes[] = {8 * P, 3 * P, P, 12 * P, 6 * P, P, 5 * P};
    for (size_t s : sizes) { void* p; OK(fma_alloc(a, s, w, &p)); }
    void* pk; OK(fma_alloc(a, 20 * P, kv, &pk));
    for (int i = 0; i < 7; ++i) OK(fma_fill_segment(a, i, 1234, (uint64_t)i << 24));
    const auto d0 = digests(a);
    auto same = [&](const std::vector<uint64_t>& d) { for (int i = 0; i < 7; ++i) assert(d[i] == d0[i]); };
    OK(fma_set_option(a, "chunk_bytes", 5 * P));
    OK(fma_set_option(a, "resident_bytes", 12 * P));           // the last three segments: 5 + 1 + 6 pages

    for (int mode : {FMA_MODE_STAGED, FMA_MODE_DIRECT, FMA_MODE_KERNEL}) {
        OK(fma_set_option(a, "mode", mode));
        OK(fma_sleep(a, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
        assert(n_resident(a) == 3 && stats(a).resident_bytes == 12 * P && stats(a).image_store_bytes == 24 * P);
        OK(fma_wake(a, 1ull << kv, 0));                         // tag-selective: the buffer stays while weights sleep
        assert(stats(a).resident_bytes == 12 * P);
        OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
        assert(stats(a).resident_bytes == 0);
        same(digests(a));
    }
    OK(fma_set_option(a, "mode", FMA_MODE_STAGED));

    // the resident allocation fails (HBM too full): a plain host-tier sleep of everything
    hostsim_fail_create_after(0);
    OK(fma_sleep(a, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
    hostsim_fail_create_after(-1);
    assert(n_resident(a) == 0 && stats(a).resident_bytes == 0 && stats(a).image_store_bytes == 36 * P);
    OK(fma_wake(a, 0, FMA_FLAG_VERIFY));
    same(digests(a));

    // a D2H fails half way through a sleep: the wake restores everything bit-exact
    for (int mode : {FMA_MODE_STAGED, FMA_MODE_DIRECT}) {
        OK(fma_set_option(a, "mode", mode));
        hostsim_fail_memcpy_after(3);
        int rc = fma_sleep(a, 1ull << w, FMA_TIER_HOST, 0);
        hostsim_fail_memcpy_after(-1);
        assert(rc != 0);
        OK(fma_wake(a, 0, 0));
        assert(fma_is_sleeping(a) == 0);
        same(digests(a));
    }
    OK(fma_set_option(a, "mode", FMA_MODE_STAGED));

    // cuMemCreate fails on a later run of a wake: rollback, the buffer survives, the retry restores everything
    int injected = 0;
    for (int fail_at = 1; fail_at <= 6; ++fail_at) {
        OK(fma_sleep(a, 1ull << w, FMA_TIER_HOST, 0));
        hostsim_fail_create_after(fail_at);
        int rc = fma_wake(a, 0, 0);
        hostsim_fail_create_after(-1);
        if (rc != 0) {
            ++injected;
            for (int i = 0; i < fma_segment_count(a); ++i) {
                fma_segment_info_t si;
                OK(fma_segment_info(a, i, &si));
                assert(si.mapped == 0);
                if (si.tag == w) assert(si.has_backup == 1);
            }
            assert(stats(a).resident_bytes == 12 * P);
            OK(fma_wake(a, 0, 0));
        }
        assert(fma_is_sleeping(a) == 0 && stats(a).resident_bytes == 0);
        same(digests(a));
    }
    assert(injected >= 2);

    // destroyed while asleep with a resident buffer: no mapping, no handle left behind
    OK(fma_sleep(a, 1ull << w, FMA_TIER_HOST, FMA_FLAG_VERIFY));
    assert(stats(a).resident_bytes == 12 * P);
    OK(fma_engine_destroy(a));
    assert(hostsim_live_mapped_bytes() == 0 && hostsim_live_handles() == 0);
    printf("resident sanitizer scenario ok\n");
    return 0;
}
