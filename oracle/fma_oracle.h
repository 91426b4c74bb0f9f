/*
 * fma_oracle.h — CPU ORACLE for the sleep/wake weight-movement path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * link, load or call anything in oracle/.  The product (llm-d-fast-model-actuation_b200/) never
 * does, and fails loudly when its CUDA library is missing.
 *
 * What it restates (the algorithm lives in third-party vLLM, which the reference pins at v0.15.1
 * — dockerfiles/Dockerfile.launcher.benchmark:1 — and only triggers over HTTP,
 * pkg/controller/dual-pods/inference-server.go:1118-1137,1329-1339):
 *   - CuMemAllocator.sleep   vllm:device_allocator/cumem.py:177-225  -> fma_oracle_sleep
 *   - CuMemAllocator.wake_up vllm:device_allocator/cumem.py:227-249  -> fma_oracle_wake
 * plus the definitions this repo adds and must keep bit-exact between CPU and GPU:
 *   - packed-image page gather / scatter (K1/K2)                      -> fma_oracle_gather/scatter
 *   - splitmix64 counter-based fill (K0)                              -> fma_oracle_fill
 *   - position-sensitive 64-bit digest (K3)                           -> fma_oracle_digest
 *   - the "FMP4" page code of packed host images (K4/K5; format spec in
 *     llm-d-fast-model-actuation_b200/csrc/fma_codec.h, restated here value by value,
 *     independently of that header)                                   -> fma_oracle_pack_page/unpack_page
 *
 * PARITY PINNING: the reference's own tests hold no golden vector for this path (SURVEY.md
 * §8c: vLLM is MagicMock'ed, test_launcher.py:32-38).  Pins used instead:
 *   (1) splitmix64 published known-answer vector (seed 1234567) — tests/test_oracle.py;
 *   (2) golden fixtures produced by running vLLM's OWN CuMemAllocator on an H100
 *       (tests/golden/make_vllm_cumem_golden.py -> tests/golden/vllm_cumem_roundtrip.json):
 *       segment sizes/tags and before/after digests of the real reference data path.
 */
#ifndef FMA_ORACLE_H
#define FMA_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define FMA_ORACLE_PAGE_BYTES ((size_t)2u << 20)

/* k-th output (0-based) of Vigna's splitmix64 stream started at `seed`. */
uint64_t fma_oracle_splitmix64(uint64_t seed, uint64_t k);
/* dst[j] = splitmix64(seed, first_word + j), j < n_words. */
void     fma_oracle_fill(uint64_t* dst, uint64_t n_words, uint64_t seed, uint64_t first_word);
/* sum_j fmix64(w_j + (first_word + j + 1) * GOLDEN) mod 2^64 over the n_bytes/8 LE words. */
uint64_t fma_oracle_digest(const void* src, uint64_t n_bytes, uint64_t first_word);

/* K1: dst + p*PAGE <- src_pages[p]  ;  K2: dst_pages[p] <- src + p*PAGE. */
void fma_oracle_gather(const void* const* src_pages, uint32_t n_pages, void* dst);
void fma_oracle_scatter(const void* src, void* const* dst_pages, uint32_t n_pages);

/* "FMP4" page code.  pack: 2 MiB page -> stored page; returns the stored size: FMA_ORACLE_PACKED_BYTES, or
 * FMA_ORACLE_PAGE_BYTES when the page needs more than 2048 exceptions and is stored verbatim.  Exceptions are
 * emitted in increasing index order; bytes of the stored page the format leaves unspecified are zero.
 * unpack: inverse; returns 0, or -1 if the stored page is malformed (bad size / magic / count). */
#define FMA_ORACLE_PACKED_BYTES ((size_t)((3u << 19) + (16u << 10)))
uint32_t fma_oracle_pack_page(const void* page, void* stored);
int      fma_oracle_unpack_page(const void* stored, uint32_t stored_bytes, void* page);

/* ---- restatement of the reference hot loops over a CPU stand-in for device memory ---- */
typedef struct fma_oracle_seg {
    void*    dev;        /* stand-in for the mapped device range; NULL while "unmapped"      */
    uint64_t bytes;      /* alignedSize (cumem.py HandleType[1])                             */
    int32_t  tag;
    int32_t  pad;
    void*    backup;     /* cpu_backup_tensor (cumem.py:55); NULL if none                    */
} fma_oracle_seg_t;

/* cumem.py:198-213: in table order, if tag in offload mask: allocate a fresh buffer and copy;
 * then unmap+release every segment.  Returns bytes backed up. */
uint64_t fma_oracle_sleep(fma_oracle_seg_t* segs, uint32_t n, uint64_t offload_tag_mask);
/* cumem.py:237-249: in table order, for tags in mask (0 = all): create+map; if a backup exists
 * copy it back and drop it.  Re-created memory without backup is left filled with `poison`
 * (the reference leaves it uninitialised).  Returns bytes restored. */
uint64_t fma_oracle_wake(fma_oracle_seg_t* segs, uint32_t n, uint64_t tag_mask, uint8_t poison);

#ifdef __cplusplus
}
#endif
#endif
