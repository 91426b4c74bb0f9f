// fma_layout.h — pure host logic of the engine's address-space layout (no CUDA): VA arenas with first-fit hole reuse,
// and grouping of sleeping segments into runs.  Header-only so that tests/test_layout_cpu.py can compile and exercise
// it with g++ on a machine without a GPU; the engine (fma_engine.cu, fma_wake.cu) uses exactly these functions.
#pragma once
#include <stddef.h>
#include <stdint.h>

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

}  // namespace fma_layout
