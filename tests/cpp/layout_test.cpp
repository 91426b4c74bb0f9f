// CPU test of the engine's address-space layout logic (csrc/fma_layout.h): compiled with g++ by tests/test_layout_cpu.py.
#include <cassert>
#include <cstdio>
#include <random>
#include <thread>

#include "fma_layout.h"

using namespace fma_layout;
static const size_t P = 2u << 20;

static void test_bump_and_first_fit() {
    Arena a; a.base = 0x7000000000ull; a.cap = 64 * P;
    size_t o1, o2, o3, o4;
    assert(arena_take(a, 4 * P, &o1) && o1 == 0);
    assert(arena_take(a, 2 * P, &o2) && o2 == 4 * P);
    assert(arena_take(a, 6 * P, &o3) && o3 == 6 * P && a.top == 12 * P);
    arena_give_back(a, o2, 2 * P);                       // hole in the middle
    assert(a.holes.size() == 1 && a.top == 12 * P);
    assert(arena_take(a, 3 * P, &o4) && o4 == 12 * P);   // does not fit the 2-page hole: bump
    size_t o5; assert(arena_take(a, P, &o5) && o5 == 4 * P);          // first fit splits the hole
    size_t o6; assert(arena_take(a, P, &o6) && o6 == 5 * P && a.holes.empty());
    size_t big; assert(!arena_take(a, 64 * P, &big));    // beyond the reservation
}

static void test_coalescing_and_top_lowering() {
    Arena a; a.cap = 32 * P;
    size_t o[5];
    for (int i = 0; i < 5; ++i) assert(arena_take(a, 2 * P, &o[i]));
    arena_give_back(a, o[1], 2 * P);
    arena_give_back(a, o[3], 2 * P);
    assert(a.holes.size() == 2);
    arena_give_back(a, o[2], 2 * P);                     // bridges both neighbours
    assert(a.holes.size() == 1 && a.holes.begin()->first == o[1] && a.holes.begin()->second == 6 * P);
    arena_give_back(a, o[4], 2 * P);                     // touches the bump pointer: everything above o[0] is free again
    assert(a.holes.empty() && a.top == 2 * P);
    arena_give_back(a, o[0], 2 * P);
    assert(a.top == 0);
}

static void test_random_alloc_free_never_overlaps() {
    std::mt19937 rng(7);
    Arena a; a.cap = 4096 * P;
    std::map<size_t, size_t> live;  // off -> len
    for (int step = 0; step < 20000; ++step) {
        if (live.empty() || rng() % 3) {
            const size_t len = (1 + rng() % 8) * P;
            size_t off;
            if (!arena_take(a, len, &off)) continue;
            auto nx = live.lower_bound(off);
            assert(nx == live.end() || off + len <= nx->first);
            if (nx != live.begin()) { auto pv = std::prev(nx); assert(pv->first + pv->second <= off); }
            assert(off + len <= a.top);
            live[off] = len;
        } else {
            auto it = live.begin(); std::advance(it, rng() % live.size());
            arena_give_back(a, it->first, it->second);
            live.erase(it);
        }
        size_t used = 0, holes = 0;
        for (auto& kv : live) used += kv.second;
        for (auto& kv : a.holes) holes += kv.second;
        assert(used + holes == a.top);                    // every byte below the bump pointer is live or a hole
    }
}

static void test_plan_runs() {
    // arena 0 = weights (backed up): a | b | hole | c ; arena 1 = kv_cache (remap only): k0 | k1
    std::vector<SegView> v = {
        {10, 0, 100 * P, 4 * P, true, 0},       {11, 0, 104 * P, 2 * P, true, 4 * P},
        {12, 0, 108 * P, 6 * P, true, 6 * P},   {20, 1, 900 * P, 8 * P, false, 0},
        {21, 1, 908 * P, 8 * P, false, 0},
    };
    auto runs = plan_runs(v, true);
    assert(runs.size() == 3);
    assert(runs[0].has_backup && runs[0].va == 100 * P && runs[0].bytes == 6 * P && runs[0].segs == std::vector<size_t>({10, 11}));
    assert(runs[1].has_backup && runs[1].va == 108 * P && runs[1].bytes == 6 * P && runs[1].first_off == 6 * P);
    assert(!runs[2].has_backup && runs[2].bytes == 16 * P && runs[2].segs == std::vector<size_t>({20, 21}));
    auto pieces = plan_runs(v, false);                    // FMA_MERGE_RUNS=0: one run per segment, same order rules
    assert(pieces.size() == 5 && pieces[0].segs[0] == 10 && pieces[3].segs[0] == 20);
    // image order wins over VA order among backed-up runs (a reused hole can sit below older data)
    std::vector<SegView> w = {{1, 0, 10 * P, 2 * P, true, 8 * P}, {2, 0, 20 * P, 2 * P, true, 0}};
    auto r2 = plan_runs(w, true);
    assert(r2.size() == 2 && r2[0].segs[0] == 2 && r2[1].segs[0] == 1);
    // a mapped/remap-only segment between two backed-up ones never merges across
    std::vector<SegView> x = {{1, 0, 0, P, true, 0}, {2, 0, P, P, false, 0}, {3, 0, 2 * P, P, true, P}};
    auto r3 = plan_runs(x, true);
    assert(r3.size() == 3 && r3[0].segs[0] == 1 && r3[1].segs[0] == 3 && r3[2].segs[0] == 2);
    assert(plan_runs({}, true).empty());
    // pieces: a contiguous backed-up run of 4+2+6+3 pages cut at >= 5 pages -> (4+2), (6), (3); the remap-only run stays whole
    std::vector<SegView> y = {{1, 0, 0, 4 * P, true, 0}, {2, 0, 4 * P, 2 * P, true, 4 * P}, {3, 0, 6 * P, 6 * P, true, 6 * P},
                              {4, 0, 12 * P, 3 * P, true, 12 * P}, {5, 1, 500 * P, 9 * P, false, 0}, {6, 1, 509 * P, 9 * P, false, 0}};
    auto r4 = plan_runs(y, true, 5 * P);
    assert(r4.size() == 4 && r4[0].bytes == 6 * P && r4[1].bytes == 6 * P && r4[2].bytes == 3 * P && !r4[3].has_backup && r4[3].bytes == 18 * P);
    assert(r4[0].va + r4[0].bytes == r4[1].va && r4[1].va + r4[1].bytes == r4[2].va && r4[1].segs == std::vector<size_t>({3}));
    assert(plan_runs(y, true, 0).size() == 2);
}

static const uint32_t C = 1589248;  // a coded page's stored size

static std::vector<PagePlan> pages_with(const std::vector<uint64_t>& off, const std::vector<uint32_t>& bytes, size_t need = 0) {
    std::vector<PagePlan> v;
    for (size_t p = 0; p < off.size(); ++p) v.push_back(PagePlan{0x100000000ull + p * P, off[p], bytes[p], need});
    return v;
}

static bool same(const std::vector<Batch>& b, const std::vector<Batch>& want) {
    if (b.size() != want.size()) return false;
    for (size_t i = 0; i < b.size(); ++i)
        if (b[i].p0 != want[i].p0 || b[i].np != want[i].np || b[i].stored != want[i].stored || b[i].need != want[i].need) return false;
    return true;
}

static void test_plan_pages() {
    // given out of image order: a (2 pages at image page 3), b (3 pages at image page 0), c (1 page at image page 5)
    std::vector<SegPages> segs = {{900 * P, 2 * P, 3 * P, 7}, {100 * P, 3 * P, 0, 2}, {500 * P, P, 5 * P, 4}};
    std::vector<PagePlan> pg;
    uint64_t bad = 0;
    assert(plan_pages(segs, nullptr, nullptr, &pg, &bad) && pg.size() == 6);   // plain image: stored verbatim at its image offset
    const uint64_t va[] = {100 * P, 101 * P, 102 * P, 900 * P, 901 * P, 500 * P};
    const size_t need[] = {2, 2, 2, 7, 7, 4};
    for (size_t p = 0; p < 6; ++p) assert(pg[p].va == va[p] && pg[p].off == p * P && pg[p].bytes == P && pg[p].need == need[p]);
    // PACKED layout, indexed by image page
    const std::vector<uint64_t> off = {0, C, 2 * C, 3 * C, 3 * C + P, 4 * C + P};
    const std::vector<uint32_t> bytes = {C, C, C, (uint32_t)P, C, C};
    assert(plan_pages(segs, &off, &bytes, &pg, &bad) && pg.size() == 6);
    for (size_t p = 0; p < 6; ++p) assert(pg[p].va == va[p] && pg[p].off == off[p] && pg[p].bytes == bytes[p] && pg[p].need == need[p]);
    // a tag-selective wake: only some segments, same image pages and layout entries
    assert(plan_pages({segs[0]}, &off, &bytes, &pg, &bad) && pg.size() == 2 && pg[0].off == 3 * C && pg[1].off == 3 * C + P && pg[1].bytes == C);
    // a page outside the layout
    const std::vector<uint64_t> short_off(off.begin(), off.begin() + 4);
    assert(!plan_pages(segs, &short_off, &bytes, &pg, &bad) && bad == 4 * P);
    assert(plan_pages({}, nullptr, nullptr, &pg, &bad) && pg.empty());
}

static void test_batches_by_stored_bytes() {
    // STAGED + PACKED: stored bytes <= one ring slot, adjacent in the store.  Pages 0-3 coded, 4 raw, 5-6 coded; a gap before page 5.
    const std::vector<uint64_t> off = {0, C, 2 * C, 3 * C, 4 * C, 5 * C + P, 6 * C + P};
    const std::vector<uint32_t> bytes = {C, C, C, C, (uint32_t)P, C, C};
    std::vector<Batch> b;
    assert(plan_batches(pages_with(off, bytes), SIZE_MAX, 3 * P, true, &b));   // 3 coded pages fit 6 MiB, the 4th does not
    assert(same(b, {{0, 3, 3 * C, 0}, {3, 2, C + P, 0}, {5, 2, 2 * C, 0}}));
    assert(!plan_batches(pages_with(off, bytes), SIZE_MAX, P - 1, true, &b));  // a raw page larger than the slot
    assert(!plan_batches(pages_with(off, bytes), SIZE_MAX, C - 1, true, &b));
    // INCREMENTAL: the changed pages only (holes between them), each in its old place
    std::vector<PagePlan> all = pages_with(off, bytes), sub;
    for (size_t p : {1, 2, 4, 6}) sub.push_back(all[p]);
    assert(plan_batches(sub, SIZE_MAX, 3 * P, true, &b) && same(b, {{0, 2, 2 * C, 0}, {2, 1, P, 0}, {3, 1, C, 0}}));
    // a byte cap that ends a batch inside a segment: the cap, not the segment, decides
    assert(plan_batches(pages_with({0, C, 2 * C, 3 * C}, {C, C, C, C}), SIZE_MAX, 2 * C, true, &b) && same(b, {{0, 2, 2 * C, 0}, {2, 2, 2 * C, 0}}));
}

static void test_batches_by_pages() {
    // STAGED / MULTI-PATH of a plain image: a page count per slot, adjacent in the store; `need` = the largest in the batch
    std::vector<PagePlan> pg = pages_with({0, P, 2 * P, 3 * P, 9 * P, 10 * P, 11 * P}, std::vector<uint32_t>(7, (uint32_t)P));
    const size_t need[] = {1, 1, 3, 2, 5, 4, 4};
    for (size_t p = 0; p < pg.size(); ++p) pg[p].need = need[p];
    std::vector<Batch> b;
    assert(plan_batches(pg, 3, UINT64_MAX, true, &b));   // the gap after page 3 (a segment that is not woken) ends a batch
    assert(same(b, {{0, 3, 3 * P, 3}, {3, 1, P, 2}, {4, 3, 3 * P, 5}}));
    assert(!plan_batches(pg, 0, UINT64_MAX, true, &b));  // a slot smaller than a page
    // K1 / K2 / K4 / K5 in place: by count, not adjacent, even when the pages are packed
    assert(plan_batches(pg, 3, UINT64_MAX, false, &b) && same(b, {{0, 3, 3 * P, 3}, {3, 3, 3 * P, 5}, {6, 1, P, 4}}));
    std::vector<PagePlan> packed = pages_with({0, C, 5 * P, 5 * P + C, 9 * P}, {C, C, C, (uint32_t)P, C}, 6);
    assert(plan_batches(packed, 2, UINT64_MAX, false, &b) && same(b, {{0, 2, 2 * C, 6}, {2, 2, C + P, 6}, {4, 1, C, 6}}));
    // next_batch alone: the first cut of a launch the wake may then extend over pages already mapped
    const Batch first = next_batch(pg, 4, 2, UINT64_MAX, false);
    assert(first.p0 == 4 && first.np == 2 && first.need == 5 && first.stored == 2 * P);
    assert(plan_batches({}, 3, UINT64_MAX, true, &b) && b.empty());
}

static void test_chunk_queues() {
    const std::vector<NumaRange> ranges = {{0, 10 * P, 0}, {10 * P, 20 * P, 1}};
    const std::vector<uint64_t> off = {0, 4 * P, 8 * P, 12 * P, 16 * P, 19 * P};   // chunks 0-2 on node 0, 3-5 on node 1
    {
        ChunkQueues q(off, ranges);
        size_t c, got[6];
        for (size_t i = 0; i < 6; ++i) assert(q.take(1, &got[i]));   // own node's queue first, in image order, then the other
        const size_t want[] = {3, 4, 5, 0, 1, 2};
        for (size_t i = 0; i < 6; ++i) assert(got[i] == want[i]);
        assert(!q.take(1, &c) && !q.take(0, &c));
    }
    {
        ChunkQueues q(off, ranges);
        size_t c;
        assert(q.take(7, &c) && c == 0);   // a path on no node of the store: the queues in order
        assert(q.take(0, &c) && c == 1);
        assert(q.take(1, &c) && c == 3);
    }
    {
        ChunkQueues q(off, {});   // no NUMA placement: one queue, image order
        size_t c;
        for (size_t i = 0; i < 6; ++i) assert(q.take(1, &c) && c == i);
        assert(!q.take(0, &c));
    }
    // several threads: every chunk is taken exactly once
    std::vector<uint64_t> many;
    for (size_t i = 0; i < 5000; ++i) many.push_back((i * 7919 % 20) * P);
    ChunkQueues q(many, ranges);
    std::vector<std::atomic<int>> taken(many.size());
    for (auto& t : taken) t.store(0);
    std::vector<std::thread> th;
    for (int t = 0; t < 6; ++t)
        th.emplace_back([&, t] {
            size_t c;
            while (q.take(t % 3, &c)) taken[c].fetch_add(1);
        });
    for (auto& t : th) t.join();
    for (auto& t : taken) assert(t.load() == 1);
}

static void test_resident_split() {
    const uint64_t M = P;
    auto split = [](std::vector<uint64_t> s, uint64_t cap) { return resident_split(s, cap); };
    using K = std::vector<char>;
    assert(split({4 * M, 2 * M, 6 * M}, 0) == K({0, 0, 0}));
    assert(split({4 * M, 2 * M, 6 * M}, 6 * M) == K({0, 0, 1}));
    assert(split({4 * M, 2 * M, 6 * M}, 7 * M) == K({0, 0, 1}));        // what is left fits nothing
    assert(split({4 * M, 2 * M, 6 * M}, 9 * M) == K({0, 1, 1}));        // 4 pages do not fit the last 3: skipped
    assert(split({4 * M, 2 * M, 6 * M}, 12 * M + M - 1) == K({1, 1, 1}));
    assert(split({3 << 20, 3 << 20}, 6 << 20) == K({1, 1}));            // (the engine rounds the cap down to 2 MiB first)
    assert(split({3 << 20, 3 << 20}, 5 << 20) == K({0, 1}));
    assert(split({}, 8 * M).empty());
    // against a brute-force restatement: from the last extent back, keep one when the kept ones after it leave room for it
    std::mt19937 rng(11);
    for (int it = 0; it < 2000; ++it) {
        std::vector<uint64_t> s(rng() % 9);
        for (auto& x : s) x = (rng() % 3 == 0) ? (1 + rng() % 6) * P : (1 + rng() % 6) * (uint64_t)C;
        const uint64_t cap = rng() % 40 * P;
        const K keep = resident_split(s, cap);
        assert(keep.size() == s.size());
        for (size_t k = 0; k < s.size(); ++k) {
            uint64_t after = 0;
            for (size_t j = k + 1; j < s.size(); ++j) after += keep[j] ? s[j] : 0;
            assert(keep[k] == (after + s[k] <= cap));
        }
    }
}

// ---- routes: the sleep and wake restated the way do_sleep / do_wake spelled them out before the routes were made functions.
// One deliberate difference: a partial-packed sleep wants no ring here.  do_sleep used to call ensure_ring(e, W) for it a second
// time, after the partial check had got the ring; that call returned at once (ring count and slot size already matched).
static const int H = FMA_TIER_HOST, DIR = FMA_MODE_DIRECT, STG = FMA_MODE_STAGED, KRN = FMA_MODE_KERNEL;

static SleepRoute sleep_restated(const SleepFacts& f) {
    const bool adopt = f.adopt || f.clean;
    int mode = f.partial ? DIR : f.mode;
    const bool multipath = f.paths && !f.mbox && f.tier == H && mode == STG && !f.partial && !f.partial_packed && !adopt && !f.pack && f.multipath_env;
    const bool wants_ring = !adopt && mode == STG && !multipath && !f.partial_packed;  // (a partial-packed sleep has its ring already)
    if (wants_ring && !f.ring) mode = DIR;
    const bool pack_path = (f.tier == H && mode == STG) || (f.tier != H && mode == KRN);
    const bool wants_probe = !adopt && !f.partial_packed && f.pack && pack_path;
    const bool packed = wants_probe && f.worth_packing;
    using K = SleepPipeKind;
    const K pipe = adopt ? K::Adopt : f.partial_packed ? K::PartialPacked : f.partial ? K::PartialDirect : mode == DIR ? K::Direct
                 : mode == KRN ? (packed ? K::KernelPacked : K::Kernel) : multipath && !packed ? K::Multipath : packed ? K::StagedPacked : K::Staged;
    return SleepRoute{pipe, mode, wants_ring, wants_probe};
}

static WakeRoute wake_restated(const WakeFacts& f) {
    int mode = f.mode;
    if (f.image_packed && f.tier == H) mode = STG;
    const bool multipath = f.paths && f.tier == H && mode == STG && !f.image_packed;
    bool wants_ring = false;
    if (f.moves && mode == STG && multipath) {
    } else if (f.moves && mode == STG && f.no_ring) {
        mode = DIR;
    } else if (f.moves && mode == STG) {
        wants_ring = true;
        if (!f.ring) mode = DIR;
    }
    using K = WakePipeKind;
    const K pipe = f.image_packed ? (mode == STG ? K::PackedRing : K::PackedZeroCopy) : multipath ? K::Multipath : mode == DIR ? K::Direct
                 : mode == KRN ? K::Kernel : K::Staged;
    return WakeRoute{pipe, mode, wants_ring};
}

static bool same(const SleepRoute& a, const SleepRoute& b) {
    return a.pipe == b.pipe && a.mode == b.mode && a.wants_ring == b.wants_ring && a.wants_probe == b.wants_probe;
}
static bool same(const WakeRoute& a, const WakeRoute& b) { return a.pipe == b.pipe && a.mode == b.mode && a.wants_ring == b.wants_ring; }

static void test_resolve_mode() {
    assert(resolve_mode(FMA_MODE_AUTO, H) == STG && resolve_mode(FMA_MODE_AUTO, FMA_TIER_PEER) == KRN);
    assert(resolve_mode(STG, FMA_TIER_LOCAL) == KRN && resolve_mode(DIR, FMA_TIER_PEER) == DIR && resolve_mode(KRN, H) == KRN);
}

static SleepFacts sleep_facts(int tier, int mode, bool pack) { return SleepFacts{tier, mode, pack, false, false, false, false, false, false, true}; }

static void test_sleep_route_quirks() {
    using K = SleepPipeKind;
    // a partial sleep reports DIRECT, whatever the configured mode
    SleepFacts f = sleep_facts(H, STG, false);
    f.partial = true;
    assert(same(sleep_route(f), SleepRoute{K::PartialDirect, DIR, false, false}));
    // a clean (adopt) sleep reports the resolved mode and asks for no ring and no probe
    f = sleep_facts(H, KRN, true);
    f.clean = true;
    assert(same(sleep_route(f), SleepRoute{K::Adopt, KRN, false, false}));
    // the resident split probes on the route asked before the ring is known, and a ring that then fails drops the probe's verdict
    f = sleep_facts(H, STG, true);
    assert(sleep_route(f).wants_probe && sleep_route(f).pipe == K::StagedPacked);
    f.ring = false;
    assert(same(sleep_route(f), SleepRoute{K::Direct, DIR, true, false}));
    // a partial-packed sleep has its ring already and keeps the image's form
    f = sleep_facts(H, STG, true);
    f.partial_packed = true;
    assert(same(sleep_route(f), SleepRoute{K::PartialPacked, STG, false, false}));
    // the parking tiers pack through K4 straight into the store
    assert(sleep_route(sleep_facts(FMA_TIER_PEER, KRN, true)).pipe == K::KernelPacked);
    f = sleep_facts(FMA_TIER_LOCAL, KRN, true);
    f.worth_packing = false;
    assert(sleep_route(f).pipe == K::Kernel);
    // multi-path: plain images only, local paths only, and FMA_MULTIPATH_SLEEP=0 turns it off; it needs no ring
    f = sleep_facts(H, STG, false);
    f.paths = true;
    assert(same(sleep_route(f), SleepRoute{K::Multipath, STG, false, false}));
    f.multipath_env = false;
    assert(sleep_route(f).pipe == K::Staged && sleep_route(f).wants_ring);
    f.multipath_env = true;
    f.mbox = true;
    assert(sleep_route(f).pipe == K::Staged);
}

static void test_wake_route_quirks() {
    using K = WakePipeKind;
    // a packed host-tier image without a ring: K5 reads the store itself, and the wake reports DIRECT
    WakeFacts f{H, DIR, true, false, true, false};
    assert(same(wake_route(f), WakeRoute{K::PackedRing, STG, true}));   // a packed host-tier image wants a ring whatever the mode
    f.ring = false;
    assert(same(wake_route(f), WakeRoute{K::PackedZeroCopy, DIR, true}));
    f = WakeFacts{H, STG, true, false, true, true};                     // FMA_NO_RING: not even asked
    assert(same(wake_route(f), WakeRoute{K::PackedZeroCopy, DIR, false}));
    // parking tiers: K5 / K2 read the store itself
    assert(same(wake_route(WakeFacts{FMA_TIER_PEER, KRN, true, false, true, false}), WakeRoute{K::PackedZeroCopy, KRN, false}));
    assert(same(wake_route(WakeFacts{FMA_TIER_LOCAL, KRN, false, true, true, false}), WakeRoute{K::Kernel, KRN, false}));
    // multi-path: a plain host-tier image, no ring; nothing that crosses the link asks for no ring either
    assert(same(wake_route(WakeFacts{H, STG, false, true, true, false}), WakeRoute{K::Multipath, STG, false}));
    assert(same(wake_route(WakeFacts{H, STG, false, false, false, false}), WakeRoute{K::Staged, STG, false}));
    assert(same(wake_route(WakeFacts{H, STG, false, false, true, true}), WakeRoute{K::Direct, DIR, false}));
}

// every input the engine can present, against the restatement; an answer the route does not want does not change it
static void test_routes_exhaustive() {
    size_t n_sleep = 0, n_wake = 0;
    for (int tier : {FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL})
        for (int cfg : {FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL})
            for (int bits = 0; bits < 1 << 7; ++bits)
                for (int outcome = 0; outcome < 4; ++outcome) {   // none, clean, partial, partial-packed
                    const int mode = resolve_mode(cfg, tier);
                    SleepFacts f{tier, mode, (bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0, (bits & 8) != 0,
                                 outcome == 1, outcome == 2, outcome == 3, (bits & 16) != 0, (bits & 32) != 0, (bits & 64) != 0};
                    if ((f.mbox && !f.paths) || (f.adopt && outcome)) continue;   // (adopt: no INCREMENTAL check)
                    if ((f.partial || f.partial_packed) && tier != H) continue;                   // partial sleeps are host-tier only
                    if (f.partial_packed && !(f.pack && mode == STG)) continue;
                    const SleepRoute r = sleep_route(f);
                    assert(same(r, sleep_restated(f)));
                    SleepFacts g = f;
                    g.ring = !f.ring;
                    if (!r.wants_ring) assert(same(sleep_route(g), r));
                    g = f;
                    g.worth_packing = !f.worth_packing;
                    if (!r.wants_probe) assert(same(sleep_route(g), r));
                    ++n_sleep;
                }
    for (int tier : {FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL})
        for (int cfg : {FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL})
            for (int bits = 0; bits < 1 << 5; ++bits) {
                const WakeFacts f{tier, resolve_mode(cfg, tier), (bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0, (bits & 8) != 0, (bits & 16) != 0};
                const WakeRoute r = wake_route(f);
                assert(same(r, wake_restated(f)));
                WakeFacts g = f;
                g.ring = !f.ring;
                if (!r.wants_ring) assert(same(wake_route(g), r));
                ++n_wake;
            }
    assert(n_sleep == 1968 && n_wake == 384);   // the feasible inputs
}

int main() {
    test_bump_and_first_fit();
    test_coalescing_and_top_lowering();
    test_random_alloc_free_never_overlaps();
    test_plan_runs();
    test_plan_pages();
    test_batches_by_stored_bytes();
    test_batches_by_pages();
    test_chunk_queues();
    test_resident_split();
    test_resolve_mode();
    test_sleep_route_quirks();
    test_wake_route_quirks();
    test_routes_exhaustive();
    std::puts("layout ok");
    return 0;
}
