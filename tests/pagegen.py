"""Distinct 2 MiB test pages for the PACKED image and the resident share.

A segment filled by repeating one page cannot show a page restored to the wrong place within it: every page holds the same
bytes, so reads, digests and FMA_FLAG_VERIFY all match.  stamp() gives every page its own bytes and keeps everything the
PACKED code (csrc/fma_codec.h) decides about it.  It rewrites the sign bit and the low 7 mantissa bits of the first value of
every 256-value tile (bf16 = s(1) e(8) m(7)) with a hash of (seed, page id, tile), and leaves every exponent as it was.  A
value's code, its tile's emax, the page's exception count and so the raw / coded decision depend on exponents only, so
oracle.pack_page(stamp(p)).size == oracle.pack_page(p).size for every page p."""
import hashlib

import numpy as np

PAGE = 2 << 20
TILE_VALUES = 256
TILES = PAGE // 2 // TILE_VALUES                 # 4096 tiles of a page
EXPONENT = np.uint16(0x7F80)


def _mix(x: np.ndarray) -> np.ndarray:
    """splitmix64's finaliser on a uint64 array (wraps modulo 2^64)."""
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def stamp(buf: np.ndarray, seed: int, first_page: int = 0) -> np.ndarray:
    """A uint8 copy of `buf` (whole 2 MiB pages) in which page k carries the stamp of (seed, first_page + k)."""
    out = np.ascontiguousarray(buf).view(np.uint8).copy()
    assert out.size % PAGE == 0, out.size
    n = out.size // PAGE
    lead = out.view(np.uint16).reshape(n, TILES, TILE_VALUES)[:, :, 0]        # first value of every tile: a strided view
    page = np.arange(first_page, first_page + n, dtype=np.uint64)[:, None]
    tile = np.arange(TILES, dtype=np.uint64)[None, :]
    h = _mix(((page << np.uint64(12)) | tile) ^ _mix(np.full(1, seed, np.uint64)))
    bits = ((((h >> np.uint64(7)) & np.uint64(1)) << np.uint64(15)) | (h & np.uint64(0x7F))).astype(np.uint16)
    lead[...] = (lead & EXPONENT) | bits
    return out


def repeat_page(page: np.ndarray, nbytes: int, seed: int, first_page: int = 0) -> np.ndarray:
    """nbytes (whole pages) of `page` repeated, each copy stamped with its own id: first_page, first_page + 1, ..."""
    return stamp(np.resize(np.ascontiguousarray(page).view(np.uint8), nbytes), seed, first_page)


def pages_of(buf: np.ndarray) -> list[np.ndarray]:
    return [buf[o:o + PAGE] for o in range(0, buf.size, PAGE)]


def all_distinct(pages) -> bool:
    """No two of the given 2 MiB pages are byte-identical (compared by a 256-bit hash of each)."""
    keys = [hashlib.blake2b(np.ascontiguousarray(p).view(np.uint8), digest_size=32).digest() for p in pages]
    return len(set(keys)) == len(keys)
