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

}  // namespace fma_layout
