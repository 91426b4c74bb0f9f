// fma_codec.h — the page code of PACKED host images: a lossless re-packing of bf16 weight pages that moves 24 %
// fewer bytes over PCIe (the link, not HBM, bounds a host-tier wake: DESIGN.md §4).
//
// No counterpart in the reference: vLLM's sleep copies every segment verbatim (vllm:device_allocator/cumem.py:198-213).
// The code is exact — unpack(pack(page)) == page for ANY 2 MiB of bytes — and a page that does not look like bf16
// weights simply stays raw, so the round trip stays bit-identical to the reference's (SURVEY.md §8c invariant).
//
// This header is the single definition of the format's per-lane arithmetic.  It is compiled three ways: into the
// sm_90a kernels K4/K5 (csrc/fma_pack_kernels.cu: one warp per tile, one lane per 8 values), into the host
// simulation's stand-ins (tests/cpp/hostsim/hostsim_kernels.cpp: the same lane functions in a loop), and it is
// restated independently, value by value, in oracle/fma_oracle.c (the checker).
//
// Format v1 ("FMP4").  A page is 2^20 little-endian 16-bit values v = s(1) e(8) m(7) (bf16).  Tiles of 256 values.
//   emax[t]   = max e over tile t
//   code(v)   = emax - e          if emax - e <= 13
//             = 14                if e == 0            (zeros / denormals far below the tile's range)
//             = 15                otherwise            -> exception entry (index << 0 | e << 20), at most kExcCap a page
//   packed page (kPackedBytes = 1.5 MiB + 16 KiB = 0.758 of a page), all offsets 16-byte aligned:
//     [kSmOff   , +1 MiB  )  byte i      = s << 7 | m          of value i
//     [kNibOff  , +512 KiB)  byte j      = code(2j) | code(2j+1) << 4
//     [kEmaxOff , +4 KiB  )  byte t      = emax[t]
//     [kExcOff  , +8 KiB  )  u32 entries, order unspecified, the first n_exc are valid
//     [kHdrOff  , +4 KiB  )  u32 magic "FMP4", u32 n_exc, rest unspecified
//   A page with more than kExcCap exceptions (fp8 / fp16 / int data, noise) is stored raw: 2 MiB, verbatim.
//   The stored size tells the two apart.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FMA_HD __host__ __device__ __forceinline__
#else
#define FMA_HD inline
#endif

namespace fma_codec {

constexpr uint32_t kPageBytes = 2u << 20;
constexpr uint32_t kValues = 1u << 20;
constexpr uint32_t kTileValues = 256;
constexpr uint32_t kTiles = kValues / kTileValues;  // 4096
constexpr uint32_t kLaneValues = 8;                 // one 16-byte load
constexpr uint32_t kExcCap = 2048;
constexpr uint32_t kSmOff = 0;
constexpr uint32_t kNibOff = kValues;                    // 1 MiB
constexpr uint32_t kEmaxOff = kNibOff + kValues / 2;     // 1.5 MiB
constexpr uint32_t kExcOff = kEmaxOff + kTiles;          // + 4 KiB
constexpr uint32_t kHdrOff = kExcOff + 4 * kExcCap;      // + 8 KiB
constexpr uint32_t kPackedBytes = kHdrOff + 4096;        // 1.5 MiB + 16 KiB
constexpr uint32_t kMagic = 0x34504D46u;                 // "FMP4"
constexpr uint32_t kCodeZero = 14, kCodeExc = 15, kMaxDelta = 13;

FMA_HD uint32_t exp_of(uint32_t v16) { return (v16 >> 7) & 0xFFu; }
FMA_HD uint32_t sm_of(uint32_t v16) { return ((v16 >> 8) & 0x80u) | (v16 & 0x7Fu); }
FMA_HD uint32_t exc_entry(uint32_t index, uint32_t e) { return index | (e << 20); }
FMA_HD uint32_t exc_index(uint32_t entry) { return entry & 0xFFFFFu; }
FMA_HD uint32_t exc_exp(uint32_t entry) { return (entry >> 20) & 0xFFu; }

// w[0..3] = 8 consecutive values (value k in bits 16*(k&1) of w[k>>1]) -> the largest exponent among them
FMA_HD uint32_t lane_max_exp(const uint32_t w[4]) {
    uint32_t mx = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 8; ++k) {
        const uint32_t e = exp_of(w[k >> 1] >> (16 * (k & 1)));
        mx = e > mx ? e : mx;
    }
    return mx;
}

// 8 values + their tile's emax -> 8 sign/mantissa bytes (sm_lo = values 0..3, little-endian), 8 nibbles (value k in
// bits 4k), and a mask of the values that need an exception entry (bit k)
FMA_HD void lane_encode(const uint32_t w[4], uint32_t emax, uint32_t& sm_lo, uint32_t& sm_hi, uint32_t& nib, uint32_t& exc_mask) {
    uint32_t lo = 0, hi = 0, nb = 0, xm = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 8; ++k) {
        const uint32_t v = (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
        const uint32_t e = exp_of(v);
        const uint32_t d = emax - e;
        uint32_t c;
        if (d <= kMaxDelta) c = d;
        else if (e == 0) c = kCodeZero;
        else { c = kCodeExc; xm |= 1u << k; }
        nb |= c << (4 * k);
        if (k < 4) lo |= sm_of(v) << (8 * k);
        else hi |= sm_of(v) << (8 * (k - 4));
    }
    sm_lo = lo; sm_hi = hi; nib = nb; exc_mask = xm;
}

// inverse; values coded 15 come back with exponent 0 and are patched from the exception list afterwards
FMA_HD void lane_decode(uint32_t sm_lo, uint32_t sm_hi, uint32_t nib, uint32_t emax, uint32_t w[4]) {
    w[0] = w[1] = w[2] = w[3] = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 8; ++k) {
        const uint32_t sm = ((k < 4 ? sm_lo >> (8 * k) : sm_hi >> (8 * (k - 4)))) & 0xFFu;
        const uint32_t c = (nib >> (4 * k)) & 0xFu;
        const uint32_t e = c <= kMaxDelta ? (emax - c) & 0xFFu : 0u;
        const uint32_t v = ((sm & 0x80u) << 8) | (e << 7) | (sm & 0x7Fu);
        w[k >> 1] |= v << (16 * (k & 1));
    }
}

// patch one exception into a decoded value
FMA_HD uint32_t apply_exception(uint32_t v16, uint32_t entry) { return (v16 & 0x807Fu) | (exc_exp(entry) << 7); }

}  // namespace fma_codec
