"""tests/pagegen.py on CPU: a stamped page keeps every exponent, so the PACKED code makes the same decision about it as about
the page it came from (same stored size, same exception count), and stamped pages are pairwise distinct."""
import numpy as np

from tests.pagegen import PAGE, TILE_VALUES, all_distinct, pages_of, repeat_page, stamp
from tests.test_gpu_parity import _pack_pages


def _n_exc(stored):
    hdr = (3 << 19) + 4096 + 8192
    return int(stored[hdr + 4:hdr + 8].view(np.uint32)[0])


def test_stamp_keeps_the_packed_code_decision_of_every_page_kind(oracle):
    pool = _pack_pages(oracle)
    stamped = []
    for k, page in enumerate(pool):
        want = oracle.pack_page(page)
        for page_id in (0, 1, 1000 + k):
            s = stamp(page, 5, page_id)
            got = oracle.pack_page(s)
            assert got.size == want.size, (k, page_id)
            if want.size < PAGE:
                assert _n_exc(got) == _n_exc(want), (k, page_id)
            assert np.array_equal(oracle.unpack_page(got), s), (k, page_id)
            a, b = page.view(np.uint16), s.view(np.uint16)
            changed = np.flatnonzero(a != b)
            assert np.all(changed % TILE_VALUES == 0), k                     # only the first value of a tile
            assert not np.any((a ^ b) & 0x7F80), k                           # never an exponent bit
            assert changed.size > 0.9 * (PAGE // 2 // TILE_VALUES), (k, changed.size)
            stamped.append(s)
    sizes = [oracle.pack_page(p).size for p in pool]
    assert sizes.count(PAGE) == 3                                              # cap_over, noise and fp16 stay raw
    assert _n_exc(oracle.pack_page(stamp(pool[5], 5, 9))) == 2048             # cap_ok keeps exactly 2048 exceptions
    assert all_distinct(stamped + pool)


def test_a_stamped_segment_is_its_pages_stamped_one_by_one(oracle):
    page = oracle.bf16_weights(1 << 20, 300).view(np.uint8)
    seg = repeat_page(page, 7 * PAGE, seed=3, first_page=40)
    assert seg.dtype == np.uint8 and seg.size == 7 * PAGE
    for k, p in enumerate(pages_of(seg)):
        assert np.array_equal(p, stamp(page, 3, 40 + k)), k
    other = repeat_page(page, 7 * PAGE, seed=4, first_page=40)
    assert all_distinct(pages_of(seg) + pages_of(other) + [page])
    assert np.array_equal(stamp(page, 3, 40), stamp(page, 3, 40))             # deterministic
    assert not all_distinct([page, page.copy()])
