// The write-behind case of the sleep route in csrc/fma_layout.h (built and run by tests/test_write_behind.py): every input a
// file-tier sleep with FMA_FLAG_WRITE_BEHIND can present, against the rule restated here, and the flag ignored for the other tiers.
#include <cassert>
#include <cstdio>

#include "fma_layout.h"

using namespace fma_layout;

// Why write-behind is not taken: nothing to write (adopted, clean, partial), then no host store, a shared one, one too small.
static int fallback_restated(const SleepFacts& f) {
    if (f.adopt || f.clean || f.partial || f.partial_packed) return kWbNothingToWrite;
    if (!f.host_store) return kWbNoStore;
    if (f.store_shared) return kWbSharedStore;
    return f.store_cap < f.stored ? kWbSmallStore : kWbTaken;
}

// A file-tier sleep with the flag: the file tier's route, except that a full sleep with a private store that fits runs the host
// tier's ring-staged pipeline (PACKED under the same rule) and is marked write-behind.  Without a ring it is refused as before.
static SleepRoute restated(const SleepFacts& f) {
    const int why = fallback_restated(f);
    if (f.adopt || f.clean) return SleepRoute{SleepPipeKind::Adopt, FMA_MODE_STAGED, false, false, false, why};
    if (!f.ring) return SleepRoute{SleepPipeKind::NoRing, FMA_MODE_STAGED, true, f.pack, false, why};
    const bool packed = f.pack && f.worth_packing;
    if (why == kWbTaken) return SleepRoute{packed ? SleepPipeKind::StagedPacked : SleepPipeKind::Staged, FMA_MODE_STAGED, true, f.pack, true, why};
    return SleepRoute{packed ? SleepPipeKind::FilePacked : SleepPipeKind::File, FMA_MODE_STAGED, true, f.pack, false, why};
}

static bool same(const SleepRoute& a, const SleepRoute& b) {
    return a.pipe == b.pipe && a.mode == b.mode && a.wants_ring == b.wants_ring && a.wants_probe == b.wants_probe &&
           a.write_behind == b.write_behind && a.wb_fallback == b.wb_fallback;
}

int main() {
    const uint64_t P = kPageBytes, W = 40 * P;
    size_t n = 0, taken = 0;
    int seen[5] = {};
    for (int cfg : {FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL})
        for (int bits = 0; bits < 1 << 9; ++bits)
            for (uint64_t cap : {(uint64_t)0, W / 2, W - P, W, W + 8 * P})
                for (uint64_t stored : {W, W * 3 / 4}) {   // plain, or what K4p found for PACKED
                    SleepFacts f{FMA_TIER_FILE, resolve_mode(cfg, FMA_TIER_FILE), (bits & 1) != 0, (bits & 2) != 0, false, (bits & 4) != 0,
                                 (bits & 8) != 0, false, false, true, (bits & 16) != 0, (bits & 32) != 0};
                    f.write_behind = true;
                    f.host_store = (bits & 64) != 0;
                    f.store_shared = f.host_store && (bits & 128) != 0;
                    f.store_cap = f.host_store ? cap : 0;
                    f.stored = stored;
                    if (f.adopt && f.clean) continue;
                    if (!f.host_store && cap) continue;
                    const SleepRoute r = sleep_route(f);
                    assert(same(r, restated(f)));
                    if (r.write_behind) {
                        assert(f.host_store && !f.store_shared && f.store_cap >= f.stored && f.ring && !f.adopt && !f.clean);
                        ++taken;
                    }
                    ++seen[r.wb_fallback];
                    SleepFacts g = f;       // without the flag: the file tier's route, no fallback recorded
                    g.write_behind = false;
                    const SleepRoute s = sleep_route(g);
                    assert(!s.write_behind && s.wb_fallback == kWbTaken);
                    assert(s.pipe != SleepPipeKind::Staged && s.pipe != SleepPipeKind::StagedPacked);
                    assert(s.wants_ring == r.wants_ring && s.wants_probe == r.wants_probe);   // the flag asks for nothing else
                    ++n;
                }
    assert(taken > 0);
    for (int k = 0; k < 5; ++k) assert(seen[k] > 0);
    // the named cases, once each: a fitting private store is taken; no store, a small one, a shared one and a clean INCREMENTAL
    // sleep fall back to the synchronous file-tier sleep
    SleepFacts base{FMA_TIER_FILE, FMA_MODE_STAGED, false, false, false, false, false, false, false, true};
    base.write_behind = true;
    base.host_store = true;
    base.store_cap = W;
    base.stored = W;
    assert(sleep_route(base).write_behind && sleep_route(base).pipe == SleepPipeKind::Staged);
    SleepFacts f = base;
    f.pack = true;
    assert(sleep_route(f).pipe == SleepPipeKind::StagedPacked && sleep_route(f).wants_probe);
    f = base; f.host_store = false; f.store_cap = 0;
    assert(sleep_route(f).pipe == SleepPipeKind::File && sleep_route(f).wb_fallback == kWbNoStore);
    f = base; f.store_cap = W - P;
    assert(sleep_route(f).pipe == SleepPipeKind::File && sleep_route(f).wb_fallback == kWbSmallStore);
    f = base; f.store_shared = true;
    assert(sleep_route(f).pipe == SleepPipeKind::File && sleep_route(f).wb_fallback == kWbSharedStore);
    f = base; f.clean = true;
    assert(sleep_route(f).pipe == SleepPipeKind::Adopt && sleep_route(f).wb_fallback == kWbNothingToWrite);
    // the flag is ignored for the other tiers: the same route as without it, nothing recorded
    for (int tier : {FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL})
        for (int bits = 0; bits < 1 << 5; ++bits) {
            SleepFacts g{tier, resolve_mode(FMA_MODE_AUTO, tier), (bits & 1) != 0, false, false, false, (bits & 2) != 0, false, false, true,
                         (bits & 4) != 0, (bits & 8) != 0};
            g.host_store = (bits & 16) != 0;
            g.store_cap = g.host_store ? W : 0;
            g.stored = W;
            const SleepRoute without = sleep_route(g);
            g.write_behind = true;
            const SleepRoute with = sleep_route(g);
            assert(same(with, without) && !with.write_behind && with.wb_fallback == kWbTaken);
        }
    std::printf("write-behind routes ok (%zu cases, %zu taken)\n", n, taken);
    return 0;
}
