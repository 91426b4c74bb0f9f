// move_route in csrc/fma_layout.h (built and run by tests/test_image_move.py): every (from, to, facts) input a move can present,
// against the rule restated here.
#include <cassert>
#include <cstdio>

#include "fma_layout.h"

using namespace fma_layout;

static bool parks(int t) { return t == FMA_TIER_PEER || t == FMA_TIER_LOCAL; }

// A move needs a sleeping image, no mapped backup and no resident share, a known destination other than the image's own tier and
// not the other parking tier, and a prepared destination (checked last, so a bad argument is named before a missing set-up).  What
// is copied depends only on which two stores are involved: the host store, the parking buffer or a file.
static MoveRoute restated(int from, int to, const MoveFacts& f) {
    const MoveRoute no_estate{MovePipeKind::Refused, FMA_ESTATE, ""}, no_einval{MovePipeKind::Refused, FMA_EINVAL, ""};
    if (to < 0 || to > 3) return no_einval;
    if (!f.asleep || f.backup_mapped || f.resident) return no_estate;
    if (from < 0 || from > 3 || from == to || (parks(from) && parks(to))) return no_einval;
    if (!f.prepared) return no_estate;
    const bool h0 = from == FMA_TIER_HOST, h1 = to == FMA_TIER_HOST, f0 = from == FMA_TIER_FILE, f1 = to == FMA_TIER_FILE;
    MovePipeKind k = MovePipeKind::Refused;
    if (h0 && parks(to)) k = MovePipeKind::HostPark;
    if (parks(from) && h1) k = MovePipeKind::ParkHost;
    if (h0 && f1) k = MovePipeKind::HostFile;
    if (f0 && h1) k = MovePipeKind::FileHost;
    if (parks(from) && f1) k = MovePipeKind::ParkFile;
    if (f0 && parks(to)) k = MovePipeKind::FilePark;
    return MoveRoute{k, FMA_OK, ""};
}

int main() {
    size_t n = 0, moves = 0;
    for (int from = -1; from <= 4; ++from)
        for (int to = -1; to <= 4; ++to)
            for (int bits = 0; bits < 1 << 4; ++bits) {
                const MoveFacts f{(bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0, (bits & 8) != 0};
                const MoveRoute r = move_route(from, to, f), w = restated(from, to, f);
                assert(r.pipe == w.pipe && r.error == w.error);
                assert((r.error == FMA_OK) == (r.pipe != MovePipeKind::Refused));
                assert(r.why && (r.error == FMA_OK || *r.why));   // every refusal says why
                moves += r.error == FMA_OK;
                ++n;
            }
    assert(n == 6 * 6 * 16);
    assert(moves == 10);   // the 10 pairs of distinct known tiers that are not PEER <-> LOCAL, each with one set of facts
    // the six directions of one GPU, and host <-> peer
    const MoveFacts ok{true, false, false, true};
    assert(move_route(FMA_TIER_HOST, FMA_TIER_FILE, ok).pipe == MovePipeKind::HostFile);
    assert(move_route(FMA_TIER_FILE, FMA_TIER_HOST, ok).pipe == MovePipeKind::FileHost);
    assert(move_route(FMA_TIER_HOST, FMA_TIER_LOCAL, ok).pipe == MovePipeKind::HostPark);
    assert(move_route(FMA_TIER_LOCAL, FMA_TIER_HOST, ok).pipe == MovePipeKind::ParkHost);
    assert(move_route(FMA_TIER_LOCAL, FMA_TIER_FILE, ok).pipe == MovePipeKind::ParkFile);
    assert(move_route(FMA_TIER_FILE, FMA_TIER_LOCAL, ok).pipe == MovePipeKind::FilePark);
    assert(move_route(FMA_TIER_HOST, FMA_TIER_PEER, ok).pipe == MovePipeKind::HostPark);
    assert(move_route(FMA_TIER_PEER, FMA_TIER_HOST, ok).pipe == MovePipeKind::ParkHost);
    assert(move_route(FMA_TIER_FILE, FMA_TIER_FILE, ok).error == FMA_EINVAL);
    assert(move_route(FMA_TIER_PEER, FMA_TIER_LOCAL, ok).error == FMA_EINVAL);
    std::puts("move routes ok");
    return 0;
}
