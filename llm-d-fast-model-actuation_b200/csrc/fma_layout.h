// fma_layout.h — pure host logic of the engine's layout (no CUDA): VA arenas with first-fit hole reuse, grouping of
// sleeping segments into runs, and the pages, batches, chunk queues and resident split of the sleep / wake copy pipelines.
// Header-only so that tests/test_layout_cpu.py can compile and exercise it with g++ on a machine without a GPU; the engine
// (fma_engine.cu, fma_sleep.cu, fma_wake.cu) uses exactly these functions.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <iterator>
#include <map>
#include <vector>

#include "../../include/fma_engine.h"

namespace fma_layout {

// One VA arena per tag: segments of a tag are bump-allocated next to each other, so that after a sleep the whole tag
// can be re-created with ONE cuMemCreate + cuMemMap + cuMemSetAccess (a "run") instead of three driver calls per
// segment.  Driver VMM calls serialise across processes, so the number of calls, not the bytes, sets the cost of a remap
// when other processes make VMM calls too (scripts/vmm_span_probe.py compares pieces with one run).
struct Arena {
    uint64_t base = 0;                  // device VA of the reservation
    size_t cap = 0;
    size_t top = 0;                     // bump pointer
    int tag = 0;
    std::map<size_t, size_t> holes;     // freed ranges below top: offset -> length
};

// Return [off, off+len) to the arena: merge with neighbouring holes; a hole that touches the bump pointer lowers it.
inline void arena_give_back(Arena& a, size_t off, size_t len) {
    auto it = a.holes.emplace(off, len).first;
    if (it != a.holes.begin()) {
        auto prev = std::prev(it);
        if (prev->first + prev->second == it->first) {
            prev->second += it->second;
            a.holes.erase(it);
            it = prev;
        }
    }
    auto next = std::next(it);
    if (next != a.holes.end() && it->first + it->second == next->first) {
        it->second += next->second;
        a.holes.erase(next);
    }
    if (it->first + it->second == a.top) {
        a.top = it->first;
        a.holes.erase(it);
    }
}

// First fit among the holes, else bump.  Returns false if the arena cannot hold `bytes`.
inline bool arena_take(Arena& a, size_t bytes, size_t* out_off) {
    for (auto it = a.holes.begin(); it != a.holes.end(); ++it) {
        if (it->second < bytes) continue;
        const size_t off = it->first, len = it->second;
        a.holes.erase(it);
        if (len > bytes) a.holes.emplace(off + bytes, len - bytes);
        *out_off = off;
        return true;
    }
    if (a.top + bytes <= a.cap) {
        *out_off = a.top;
        a.top += bytes;
        return true;
    }
    return false;
}

// A sleeping segment as the run planner sees it.
struct SegView {
    size_t index;        // caller's index
    int arena;
    uint64_t va;
    size_t bytes;
    bool has_backup;
    uint64_t packed_off; // only meaningful with has_backup
};

struct Run {
    uint64_t va = 0;
    size_t bytes = 0;
    int arena = -1;
    bool has_backup = false;
    uint64_t first_off = 0;       // packed offset of its first segment (ordering key)
    std::vector<size_t> segs;     // caller indices, ascending VA
};

// Group sleeping segments (already sorted by (arena, va)) into maximal VA-contiguous runs of one arena and one backup
// state; order: runs with a backup first, by image offset (they gate the copy pipeline), remap-only runs after them.
// piece_bytes > 0 cuts backed-up runs into pieces of at least that size (at segment boundaries): more, smaller mappings, so
// that a slow or stalled driver call delays only what lies behind it while the copy pipeline works on the pieces before it.
inline std::vector<Run> plan_runs(const std::vector<SegView>& sorted, bool merge, size_t piece_bytes = 0) {
    std::vector<Run> runs;
    for (const SegView& s : sorted) {
        if (merge && !runs.empty() && runs.back().arena == s.arena && runs.back().va + runs.back().bytes == s.va &&
            runs.back().has_backup == s.has_backup && !(piece_bytes && s.has_backup && runs.back().bytes >= piece_bytes)) {
            runs.back().bytes += s.bytes;
            runs.back().segs.push_back(s.index);
        } else {
            Run r;
            r.va = s.va; r.bytes = s.bytes; r.arena = s.arena; r.has_backup = s.has_backup;
            r.first_off = s.has_backup ? s.packed_off : UINT64_MAX;
            r.segs.push_back(s.index);
            runs.push_back(std::move(r));
        }
    }
    // stable: keeps VA order among runs of equal key
    std::vector<Run> ordered;
    for (int pass = 0; pass < 2; ++pass)
        for (Run& r : runs)
            if (r.has_backup == (pass == 0)) ordered.push_back(std::move(r));
    // runs with a backup by image offset
    size_t nb = 0;
    while (nb < ordered.size() && ordered[nb].has_backup) ++nb;
    for (size_t i = 1; i < nb; ++i)  // insertion sort: a handful of runs
        for (size_t j = i; j > 0 && ordered[j].first_off < ordered[j - 1].first_off; --j) std::swap(ordered[j], ordered[j - 1]);
    return ordered;
}

// ---- pages and batches of the sleep / wake copy pipelines ----
constexpr uint64_t kPageBytes = (uint64_t)2 << 20;  // == FMA_PAGE_BYTES

// A segment as the page planner sees it: `need` = the mapper work items a wake must have mapped before its pages are written.
struct SegPages {
    uint64_t va;
    uint64_t bytes;
    uint64_t packed_off;
    size_t need;
};

// One image page of an operation: its device address, where and how large it is in the store, and its segment's `need`.
struct PagePlan {
    uint64_t va;
    uint64_t off;
    uint32_t bytes;
    size_t need;
};

// The pages of `segs` in image order (by packed_off).  With a PACKED layout, image page p (= packed offset / 2 MiB) is stored
// at off[p] and takes bytes[p]; without one (off == nullptr) every page is stored verbatim at its image offset.  Returns false
// when a page lies outside the layout (*bad_off = its image offset).
inline bool plan_pages(std::vector<SegPages> segs, const std::vector<uint64_t>* off, const std::vector<uint32_t>* bytes,
                       std::vector<PagePlan>* out, uint64_t* bad_off) {
    std::stable_sort(segs.begin(), segs.end(), [](const SegPages& a, const SegPages& b) { return a.packed_off < b.packed_off; });
    out->clear();
    for (const SegPages& s : segs)
        for (uint64_t o = 0; o < s.bytes; o += kPageBytes) {
            const uint64_t img = s.packed_off + o;
            if (off && img / kPageBytes >= off->size()) {
                *bad_off = img;
                return false;
            }
            out->push_back(PagePlan{s.va + o, off ? (*off)[img / kPageBytes] : img, off ? (*bytes)[img / kPageBytes] : (uint32_t)kPageBytes, s.need});
        }
    return true;
}

// Pages [p0, p0 + np) that go in one launch or one copy: `stored` bytes in the store, `need` the largest need among them.
struct Batch {
    size_t p0, np;
    uint64_t stored;
    size_t need;
};

// The batch that starts at page p0: as many consecutive pages as fit max_pages and max_bytes (stored bytes), and with
// store_adjacent only pages that follow each other in the store (one memcpy moves them).  np == 0: page p0 fits no batch.
inline Batch next_batch(const std::vector<PagePlan>& pages, size_t p0, size_t max_pages, uint64_t max_bytes, bool store_adjacent) {
    Batch b{p0, 0, 0, 0};
    for (size_t q = p0; q < pages.size() && b.np < max_pages && b.stored + pages[q].bytes <= max_bytes; ++q) {
        if (b.np && store_adjacent && pages[q].off != pages[q - 1].off + pages[q - 1].bytes) break;
        b.stored += pages[q].bytes;
        b.need = std::max(b.need, pages[q].need);
        ++b.np;
    }
    return b;
}

// All pages cut into batches (next_batch, one after the other).  Returns false when a page fits no batch.
inline bool plan_batches(const std::vector<PagePlan>& pages, size_t max_pages, uint64_t max_bytes, bool store_adjacent,
                         std::vector<Batch>* out) {
    out->clear();
    for (size_t p = 0; p < pages.size(); p += out->back().np) {
        out->push_back(next_batch(pages, p, max_pages, max_bytes, store_adjacent));
        if (!out->back().np) return false;
    }
    return true;
}

// NUMA placement of a host store by byte range.
struct NumaRange {
    size_t begin, end;
    int node;
};

// Chunk queues by NUMA node of the store range a chunk starts in: a path takes from its own node's queue first and then helps
// with the others, so bytes cross the socket interconnect only to balance the tail.  take() is safe from several threads.
class ChunkQueues {
  public:
    ChunkQueues(const std::vector<uint64_t>& chunk_off, const std::vector<NumaRange>& ranges) {
        for (size_t c = 0; c < chunk_off.size(); ++c) {
            int node = -1;
            for (const NumaRange& r : ranges)
                if (chunk_off[c] >= r.begin && chunk_off[c] < r.end) node = r.node;
            size_t qi = 0;
            while (qi < node_.size() && node_[qi] != node) ++qi;
            if (qi == node_.size()) {
                node_.push_back(node);
                chunks_.emplace_back();
            }
            chunks_[qi].push_back(c);
        }
        next_ = std::vector<std::atomic<size_t>>(node_.size());
        for (auto& a : next_) a.store(0);
    }
    // the next chunk (index into chunk_off) for a path on `my_node`; false when every chunk has been taken
    bool take(int my_node, size_t* out) {
        for (int pass = 0; pass < 2; ++pass)
            for (size_t qi = 0; qi < node_.size(); ++qi) {
                if ((pass == 0) != (node_[qi] == my_node)) continue;
                const size_t k = next_[qi].fetch_add(1);
                if (k < chunks_[qi].size()) {
                    *out = chunks_[qi][k];
                    return true;
                }
            }
        return false;
    }

  private:
    std::vector<int> node_;                    // queue -> node
    std::vector<std::vector<size_t>> chunks_;  // queue -> chunk indices, image order
    std::vector<std::atomic<size_t>> next_;
};

// RESIDENT share: walking the extents (stored size each, image order) from the last to the first, an extent stays resident if
// its stored size still fits what is left of `cap`.  Returns keep[k] for every extent.
inline std::vector<char> resident_split(const std::vector<uint64_t>& stored, uint64_t cap) {
    std::vector<char> keep(stored.size(), 0);
    for (size_t k = stored.size(); k-- > 0;)
        if (stored[k] <= cap) {
            keep[k] = 1;
            cap -= stored[k];
        }
    return keep;
}

// ---- which pipeline a sleep / wake runs ----
// The configured mode as a tier runs it: AUTO is STAGED on the host tier, KERNEL on the parking tiers (staging helps over PCIe).
inline int resolve_mode(int cfg_mode, int tier) {
    if (tier == FMA_TIER_FILE) return FMA_MODE_STAGED;   // the file tier has one pipeline: the staging ring with a disk stage
    int m = cfg_mode;
    if (m == FMA_MODE_AUTO) m = (tier == FMA_TIER_HOST) ? FMA_MODE_STAGED : FMA_MODE_KERNEL;
    if (tier != FMA_TIER_HOST && m == FMA_MODE_STAGED) m = FMA_MODE_KERNEL;
    return m;
}

enum class SleepPipeKind { Adopt, PartialDirect, PartialPacked, Direct, Kernel, KernelPacked, Staged, StagedPacked, Multipath, File, FilePacked, NoRing };

// What a sleep knows when it picks its pipeline.  `ring` and `worth_packing` are answers of calls with side effects (a ring
// allocation, the K4p probe): ask with both true, make the calls the route wants, then ask again with the answers.
struct SleepFacts {
    int tier, mode;            // mode: resolve_mode of the configured mode
    bool pack, paths, mbox;    // option "pack"; MULTI-PATH configured; ... with remote paths
    bool adopt;                // nothing moves: an adopted image, or no bytes to offload
    // INCREMENTAL: the store holds exactly this image; only the changed segments move (plain image); only the changed pages
    // are re-coded in place (PACKED image: their stored sizes held, and a staging ring was had for them)
    bool clean, partial, partial_packed;
    bool multipath_env, ring = true, worth_packing = true;  // FMA_MULTIPATH_SLEEP; a staging ring is available; K4p found it worth packing
    // WRITE-BEHIND (FMA_FLAG_WRITE_BEHIND, file tier only): the sleep fills the engine's host store and a job writes the file later
    bool write_behind = false;        // the flag was passed
    bool host_store = false, store_shared = false;   // the engine holds a host store; somebody else may hold it too (read-only)
    uint64_t store_cap = 0, stored = 0;              // its capacity; the image's stored bytes (plain size until K4p has run)
};

// Why a write-behind sleep was not taken (the timeline's "wb_fallback" row carries it as idx); 0: taken, or not asked for
enum WbFallback { kWbTaken = 0, kWbNoStore = 1, kWbSmallStore = 2, kWbSharedStore = 3, kWbNothingToWrite = 4 };

struct SleepRoute {
    SleepPipeKind pipe;
    int mode;                  // what fma_stats_t.mode reports
    bool wants_ring, wants_probe;  // `ring` / `worth_packing` decide the pipe
    bool write_behind = false;     // a file-tier sleep that runs as a host-tier sleep into the host store (pipe Staged / StagedPacked)
    int wb_fallback = kWbTaken;    // asked for write-behind and not taken: why
};

// The host store a write-behind sleep fills is one the engine already holds: private, and big enough for the stored image.  The
// engine never pins a store inside a sleep.  A sleep that writes nothing (adopted, clean INCREMENTAL) keeps its path.
inline int write_behind_fallback(const SleepFacts& f) {
    if (f.adopt || f.clean || f.partial || f.partial_packed) return kWbNothingToWrite;
    if (!f.host_store) return kWbNoStore;
    if (f.store_shared) return kWbSharedStore;
    if (f.store_cap < f.stored) return kWbSmallStore;
    return kWbTaken;
}

inline SleepRoute sleep_route(const SleepFacts& f) {
    const bool wb_asked = f.write_behind && f.tier == FMA_TIER_FILE;   // (ignored for the other tiers)
    const int wb_why = wb_asked ? write_behind_fallback(f) : kWbTaken;
    if (f.adopt || f.clean) return SleepRoute{SleepPipeKind::Adopt, f.mode, false, false, false, wb_why};
    if (f.partial_packed) return SleepRoute{SleepPipeKind::PartialPacked, f.mode, false, false};
    if (f.partial) return SleepRoute{SleepPipeKind::PartialDirect, FMA_MODE_DIRECT, false, false};
    // FILE: the ring-staged pipeline with a disk stage behind it, PACKED when asked and worth it; without a ring nothing moves.
    // WRITE-BEHIND: the host tier's ring-staged pipeline into the host store, under the same ring and PACKED rules
    if (f.tier == FMA_TIER_FILE) {
        const bool packed = f.pack && f.worth_packing, wb = wb_asked && wb_why == kWbTaken;
        const SleepPipeKind k = !f.ring ? SleepPipeKind::NoRing
                              : wb      ? (packed ? SleepPipeKind::StagedPacked : SleepPipeKind::Staged)
                                        : (packed ? SleepPipeKind::FilePacked : SleepPipeKind::File);
        return SleepRoute{k, FMA_MODE_STAGED, true, f.pack, wb && f.ring, wb_why};
    }
    SleepRoute r{SleepPipeKind::Staged, f.mode, false, false};
    // MULTI-PATH: a full, plain host-tier sleep is striped over the paths' links, each with its own staging slots
    const bool multipath = f.paths && !f.mbox && f.tier == FMA_TIER_HOST && f.mode == FMA_MODE_STAGED && !f.pack && f.multipath_env;
    r.wants_ring = f.mode == FMA_MODE_STAGED && !multipath;
    if (r.wants_ring && !f.ring) r.mode = FMA_MODE_DIRECT;  // HBM too full for a ring
    // PACKED: through the staging ring on the host tier; K4 writes the store itself on the parking tiers
    r.wants_probe = f.pack && ((f.tier == FMA_TIER_HOST && r.mode == FMA_MODE_STAGED) || (f.tier != FMA_TIER_HOST && r.mode == FMA_MODE_KERNEL));
    const bool packed = r.wants_probe && f.worth_packing;
    if (r.mode == FMA_MODE_DIRECT) r.pipe = SleepPipeKind::Direct;
    else if (r.mode == FMA_MODE_KERNEL) r.pipe = packed ? SleepPipeKind::KernelPacked : SleepPipeKind::Kernel;
    else if (multipath) r.pipe = SleepPipeKind::Multipath;
    else r.pipe = packed ? SleepPipeKind::StagedPacked : SleepPipeKind::Staged;
    return r;
}

enum class WakePipeKind { PackedRing, PackedZeroCopy, Direct, Kernel, Staged, Multipath, File, NoRing };

// What a wake knows when it picks its pipeline; `ring` as in SleepFacts (a ring attached to the first run, or allocated).
struct WakeFacts {
    int tier, mode;            // mode: resolve_mode of the configured mode
    bool image_packed, paths;  // the sleeping image is PACKED; MULTI-PATH configured
    bool moves;                // bytes cross the link (a resident share's do not)
    bool no_ring, ring = true; // FMA_NO_RING; a staging ring is available
};
struct WakeRoute {
    WakePipeKind pipe;
    int mode;                  // what fma_stats_t.mode reports
    bool wants_ring;           // `ring` decides the pipe
};

inline WakeRoute wake_route(const WakeFacts& f) {
    // FILE: plain or PACKED pages come through the ring (FMA_NO_RING: as if HBM had no room for one)
    if (f.tier == FMA_TIER_FILE) return WakeRoute{f.moves && (f.no_ring || !f.ring) ? WakePipeKind::NoRing : WakePipeKind::File, FMA_MODE_STAGED, f.moves && !f.no_ring};
    // a PACKED image can only be read by K5: through the staging ring, or straight from the store
    WakeRoute r{WakePipeKind::Staged, f.image_packed && f.tier == FMA_TIER_HOST ? FMA_MODE_STAGED : f.mode, false};
    const bool multipath = f.paths && f.tier == FMA_TIER_HOST && r.mode == FMA_MODE_STAGED && !f.image_packed;
    r.wants_ring = f.moves && r.mode == FMA_MODE_STAGED && !multipath && !f.no_ring;
    if (f.moves && r.mode == FMA_MODE_STAGED && !multipath && (f.no_ring || !f.ring)) r.mode = FMA_MODE_DIRECT;
    if (f.image_packed) r.pipe = r.mode == FMA_MODE_STAGED ? WakePipeKind::PackedRing : WakePipeKind::PackedZeroCopy;
    else if (multipath) r.pipe = WakePipeKind::Multipath;
    else if (r.mode == FMA_MODE_DIRECT) r.pipe = WakePipeKind::Direct;
    else if (r.mode == FMA_MODE_KERNEL) r.pipe = WakePipeKind::Kernel;
    return r;
}

// ---- which copy a move of a sleeping image between tiers runs (fma_image_move) ----
// Park: the parking buffer, of the peer tier or the local one.  Every tier stores the image in one layout, so a move is a byte copy.
enum class MovePipeKind { HostPark, ParkHost, HostFile, FileHost, ParkFile, FilePark, Refused };

struct MoveFacts {
    bool asleep;          // a segment with a backup is unmapped
    bool backup_mapped;   // a segment with a backup is mapped (a KEEP_BACKUP wake, a partly woken image)
    bool resident;        // part of the image sleeps in a resident share
    bool prepared;        // the destination is ready: PEER, a peer parking buffer that holds the image; FILE, a path (HOST and LOCAL: always)
};
struct MoveRoute {
    MovePipeKind pipe;
    int error;            // FMA_OK, or the code of the refusal
    const char* why;      // the refusal's reason
};

inline bool is_park_tier(int tier) { return tier == FMA_TIER_PEER || tier == FMA_TIER_LOCAL; }

inline MoveRoute move_route(int from, int to, const MoveFacts& f) {
    auto refuse = [](int code, const char* why) { return MoveRoute{MovePipeKind::Refused, code, why}; };
    if (to < FMA_TIER_HOST || to > FMA_TIER_FILE) return refuse(FMA_EINVAL, "unknown tier");
    if (!f.asleep) return refuse(FMA_ESTATE, "no image is asleep");
    if (f.backup_mapped) return refuse(FMA_ESTATE, "a segment with a backup is mapped (a KEEP_BACKUP or partial wake): wake or sleep it fully first");
    if (f.resident) return refuse(FMA_ESTATE, "part of the image sleeps in the resident share, which does not move");
    if (from < FMA_TIER_HOST || from > FMA_TIER_FILE) return refuse(FMA_EINVAL, "the image's tier is unknown");
    if (to == from) return refuse(FMA_EINVAL, "the image already sleeps in that tier");
    if (is_park_tier(from) && is_park_tier(to)) return refuse(FMA_EINVAL, "there is one parking buffer: no move between the peer and local tiers");
    if (!f.prepared)
        return refuse(FMA_ESTATE, to == FMA_TIER_FILE ? "a move to the file tier needs fma_file_store(path) first"
                                                      : "a move to the peer tier needs a peer parking buffer that holds the image (fma_peer_reserve / fma_peer_attach)");
    if (from == FMA_TIER_HOST) return MoveRoute{to == FMA_TIER_FILE ? MovePipeKind::HostFile : MovePipeKind::HostPark, FMA_OK, ""};
    if (from == FMA_TIER_FILE) return MoveRoute{to == FMA_TIER_HOST ? MovePipeKind::FileHost : MovePipeKind::FilePark, FMA_OK, ""};
    return MoveRoute{to == FMA_TIER_HOST ? MovePipeKind::ParkHost : MovePipeKind::ParkFile, FMA_OK, ""};
}

// ---- whether part of a sleeping image may be prefetched into its GPU's HBM (fma_image_prefetch with a budget) ----
// The segments it copies are the resident share's choice over stored sizes (resident_split); what is decided here is the refusal.
struct PrefetchFacts {
    int tier;             // the image's tier
    bool asleep;          // a segment with a backup is unmapped
    bool backup_mapped;   // a segment with a backup is mapped (a KEEP_BACKUP wake, a partly woken image)
    bool resident;        // the image keeps a resident share from its sleep
};
struct PrefetchRoute {
    int error;            // FMA_OK, or the code of the refusal
    const char* why;
};

inline PrefetchRoute prefetch_route(const PrefetchFacts& f) {
    if (f.backup_mapped) return PrefetchRoute{FMA_ESTATE, "a segment with a backup is mapped (a KEEP_BACKUP or partial wake): wake or sleep it fully first"};
    if (!f.asleep) return PrefetchRoute{FMA_ESTATE, "no image is asleep"};
    if (f.resident)
        return PrefetchRoute{FMA_ESTATE, "part of the image sleeps in a resident share (option resident_bytes): set it to 0 and sleep again to prefetch instead"};
    if (f.tier != FMA_TIER_HOST && f.tier != FMA_TIER_FILE) return PrefetchRoute{FMA_EINVAL, "the image sleeps in a parking buffer: it is in HBM already"};
    return PrefetchRoute{FMA_OK, ""};
}

}  // namespace fma_layout
