// The file case of the sleep / wake routes in csrc/fma_layout.h (built and run by tests/test_file_tier.py): every input a
// file-tier sleep or wake can present, against the rule restated here.
#include <cassert>
#include <cstdio>

#include "fma_layout.h"

using namespace fma_layout;

// A file-tier sleep: nothing moves (adopted image, clean INCREMENTAL sleep, nothing offloaded), or the ring-staged pipeline with a
// disk stage, PACKED when asked and the probe found it worth it; without a ring it is refused.  Always STAGED, always asks for a
// ring, asks for the probe when PACKED is on; partial sleeps, multi-path and the configured mode play no part.
static SleepRoute sleep_restated(const SleepFacts& f) {
    if (f.adopt || f.clean) return SleepRoute{SleepPipeKind::Adopt, FMA_MODE_STAGED, false, false};
    if (!f.ring) return SleepRoute{SleepPipeKind::NoRing, FMA_MODE_STAGED, true, f.pack};
    return SleepRoute{f.pack && f.worth_packing ? SleepPipeKind::FilePacked : SleepPipeKind::File, FMA_MODE_STAGED, true, f.pack};
}

// A file-tier wake: plain and PACKED images alike through the ring; no ring (or FMA_NO_RING) while bytes move: refused.
static WakeRoute wake_restated(const WakeFacts& f) {
    if (f.moves && (f.no_ring || !f.ring)) return WakeRoute{WakePipeKind::NoRing, FMA_MODE_STAGED, !f.no_ring};
    return WakeRoute{WakePipeKind::File, FMA_MODE_STAGED, f.moves && !f.no_ring};
}

static bool same(const SleepRoute& a, const SleepRoute& b) {
    return a.pipe == b.pipe && a.mode == b.mode && a.wants_ring == b.wants_ring && a.wants_probe == b.wants_probe;
}
static bool same(const WakeRoute& a, const WakeRoute& b) { return a.pipe == b.pipe && a.mode == b.mode && a.wants_ring == b.wants_ring; }

int main() {
    for (int cfg : {FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL}) assert(resolve_mode(cfg, FMA_TIER_FILE) == FMA_MODE_STAGED);
    size_t n_sleep = 0, n_wake = 0;
    for (int cfg : {FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL})
        for (int bits = 0; bits < 1 << 8; ++bits) {
            SleepFacts f{FMA_TIER_FILE, resolve_mode(cfg, FMA_TIER_FILE), (bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0, (bits & 8) != 0,
                         (bits & 16) != 0, false, false, (bits & 32) != 0, (bits & 64) != 0, (bits & 128) != 0};
            if ((f.mbox && !f.paths) || (f.adopt && f.clean)) continue;
            const SleepRoute r = sleep_route(f);
            assert(same(r, sleep_restated(f)));
            SleepFacts g = f;                 // an answer the route does not want does not change it
            g.ring = !f.ring;
            if (!r.wants_ring) assert(same(sleep_route(g), r));
            g = f;
            g.worth_packing = !f.worth_packing;
            if (!r.wants_probe) assert(same(sleep_route(g), r));
            ++n_sleep;
        }
    for (int cfg : {FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL})
        for (int bits = 0; bits < 1 << 5; ++bits) {
            const WakeFacts f{FMA_TIER_FILE, resolve_mode(cfg, FMA_TIER_FILE), (bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0, (bits & 8) != 0, (bits & 16) != 0};
            const WakeRoute r = wake_route(f);
            assert(same(r, wake_restated(f)));
            WakeFacts g = f;
            g.ring = !f.ring;
            if (!r.wants_ring) assert(same(wake_route(g), r));
            ++n_wake;
        }
    assert(n_sleep == 4 * 144 && n_wake == 128);
    // the other tiers do not take the file's pipelines
    for (int tier : {FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL}) {
        const SleepFacts f{tier, resolve_mode(FMA_MODE_AUTO, tier), true, false, false, false, false, false, false, true};
        const SleepPipeKind k = sleep_route(f).pipe;
        assert(k != SleepPipeKind::File && k != SleepPipeKind::FilePacked && k != SleepPipeKind::NoRing);
        const WakePipeKind wk = wake_route(WakeFacts{tier, resolve_mode(FMA_MODE_AUTO, tier), true, false, true, false, false}).pipe;
        assert(wk != WakePipeKind::File && wk != WakePipeKind::NoRing);
    }
    std::puts("file routes ok");
    return 0;
}
