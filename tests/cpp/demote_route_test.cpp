// The write-behind case of move_route in csrc/fma_layout.h (built and run by tests/test_image_demote.py): every (from, to, facts)
// input a move with FMA_FLAG_WRITE_BEHIND can present, against the rule restated here, and the route without the flag unchanged.
#include <cassert>
#include <cstdio>

#include "fma_layout.h"

using namespace fma_layout;

// The synchronous move's refusals first, with their codes, except that a pair other than host -> file is a bad argument named
// before a missing set-up; then a shared host store; then the write-behind pipe.
static MoveRoute restated(int from, int to, const MoveFacts& f) {
    MoveFacts sync = f;
    sync.write_behind = false;
    const MoveRoute s = move_route(from, to, sync);
    if (s.error == FMA_EINVAL) return s;
    if (s.error != FMA_OK && (!f.asleep || f.backup_mapped || f.resident)) return s;
    if (!(from == FMA_TIER_HOST && to == FMA_TIER_FILE)) return MoveRoute{MovePipeKind::Refused, FMA_EINVAL, ""};
    if (s.error != FMA_OK) return s;
    if (f.store_shared) return MoveRoute{MovePipeKind::Refused, FMA_ESTATE, ""};
    return MoveRoute{MovePipeKind::HostFileBehind, FMA_OK, ""};
}

int main() {
    size_t n = 0, behind = 0;
    for (int from = -1; from <= 4; ++from)
        for (int to = -1; to <= 4; ++to)
            for (int bits = 0; bits < 1 << 5; ++bits) {
                MoveFacts f{(bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0, (bits & 8) != 0};
                f.store_shared = (bits & 16) != 0;
                const MoveRoute without = move_route(from, to, f);   // the flag not passed: the shared store changes nothing
                MoveFacts g = f;
                g.store_shared = false;
                const MoveRoute plain = move_route(from, to, g);
                assert(without.pipe == plain.pipe && without.error == plain.error && without.pipe != MovePipeKind::HostFileBehind);
                f.write_behind = true;
                const MoveRoute r = move_route(from, to, f), w = restated(from, to, f);
                assert(r.pipe == w.pipe && r.error == w.error);
                assert((r.error == FMA_OK) == (r.pipe == MovePipeKind::HostFileBehind));
                assert(r.why && (r.error == FMA_OK || *r.why));
                if (r.error == FMA_OK) {
                    assert(from == FMA_TIER_HOST && to == FMA_TIER_FILE && f.asleep && !f.backup_mapped && !f.resident && f.prepared && !f.store_shared);
                    ++behind;
                }
                ++n;
            }
    assert(n == 6 * 6 * 32 && behind == 1);
    // the named cases: taken; a shared store; the other tier pairs; the synchronous move's refusals keep their codes
    const MoveFacts ok{true, false, false, true, true, false};
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, ok).pipe == MovePipeKind::HostFileBehind);
    MoveFacts f = ok;
    f.store_shared = true;
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, f).error == FMA_ESTATE);
    for (int from : {FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL, FMA_TIER_FILE})
        for (int to : {FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL, FMA_TIER_FILE})
            if (!(from == FMA_TIER_HOST && to == FMA_TIER_FILE)) assert(move_route(from, to, ok).error == FMA_EINVAL);
    f = ok; f.prepared = false;
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, f).error == FMA_ESTATE);   // no fma_file_store
    f = ok; f.asleep = false;
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, f).error == FMA_ESTATE);
    f = ok; f.backup_mapped = true;
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, f).error == FMA_ESTATE);
    f = ok; f.resident = true;
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, f).error == FMA_ESTATE);
    std::printf("demote routes ok (%zu cases)\n", n);
    return 0;
}
