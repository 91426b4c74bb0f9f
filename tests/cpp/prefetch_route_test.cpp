// prefetch_route in csrc/fma_layout.h (built and run by tests/test_image_prefetch.py): every input a prefetch can present, against
// the rule restated here; and the segments a prefetch keeps (resident_split over stored sizes) as its budget grows.
#include <cassert>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "fma_layout.h"

using namespace fma_layout;

// A prefetch needs no mapped backup, a sleeping image and no resident share from its sleep (FMA_ESTATE, in that order), and an
// image in the host tier or the file tier: one in a parking buffer is in HBM already (FMA_EINVAL, named after the state).
static int restated(const PrefetchFacts& f) {
    if (!f.asleep || f.backup_mapped || f.resident) return FMA_ESTATE;
    if (f.tier != FMA_TIER_HOST && f.tier != FMA_TIER_FILE) return FMA_EINVAL;
    return FMA_OK;
}

// From the last segment to the first, a segment is kept when its stored size fits what is left of the budget.
static std::vector<char> kept(const std::vector<uint64_t>& stored, uint64_t budget) {
    std::vector<char> k(stored.size(), 0);
    uint64_t left = budget;
    for (size_t i = stored.size(); i-- > 0;)
        if (stored[i] <= left) {
            k[i] = 1;
            left -= stored[i];
        }
    return k;
}

int main() {
    size_t n = 0, allowed = 0;
    for (int tier = -1; tier <= 4; ++tier)
        for (int bits = 0; bits < 1 << 3; ++bits) {
            const PrefetchFacts f{tier, (bits & 1) != 0, (bits & 2) != 0, (bits & 4) != 0};
            const PrefetchRoute r = prefetch_route(f);
            assert(r.error == restated(f));
            assert(r.why && (r.error == FMA_OK || *r.why));   // every refusal says why
            allowed += r.error == FMA_OK;
            ++n;
        }
    assert(n == 6 * 8 && allowed == 2);   // asleep, nothing mapped with a backup, no resident share; host or file
    assert(prefetch_route(PrefetchFacts{FMA_TIER_LOCAL, false, false, false}).error == FMA_ESTATE);   // nothing asleep comes first

    // stored sizes of a PACKED image (coded and raw pages mixed): every budget from 0 past the whole image, in 2 MiB steps
    const uint64_t P = kPageBytes, C = 1589248;   // a coded page's stored size is not a 2 MiB multiple
    const std::vector<uint64_t> stored = {8 * C, 3 * P, C, 12 * C + P, 6 * C, P, 5 * C};
    uint64_t total = 0;
    for (uint64_t s : stored) total += s;
    for (uint64_t budget = 0; budget <= total + 2 * P; budget += P) {
        const std::vector<char> k = resident_split(stored, budget);
        assert(k == kept(stored, budget));
        uint64_t sum = 0;
        for (size_t i = 0; i < k.size(); ++i) sum += k[i] ? stored[i] : 0;
        assert(sum <= budget);
        if (budget >= total) assert(sum == total);   // a budget of the whole image keeps all of it
    }
    std::puts("prefetch routes ok");
    return 0;
}
