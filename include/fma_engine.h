/*
 * fma_engine.h — C-ABI of the H100-native sleep / wake / hot-swap weight-movement engine.
 *
 * This is the drop-in boundary (SURVEY.md §8b, surface B3) for the ONE hot path of
 * llm-d-fast-model-actuation: moving an inference server's weight segments HBM -> host (or
 * peer HBM) on `POST /sleep` and back on `POST /wake_up`.  In the reference those bytes are
 * moved by third-party vLLM code which the reference only triggers over HTTP
 * (pkg/controller/dual-pods/inference-server.go:1329-1339 sleep, :1118-1137 wake_up,
 * :1595-1607 is_sleeping).  Each entry point below names the reference-side interface
 * it replaces (vllm: = the vLLM tree the reference pins and launches through
 * inference_server/launcher/launcher.py:38,829-837).
 *
 * Conventions: plain C, no torch / CUDA types in signatures (device pointers are
 * `void*` / uint64_t, streams are `void*`).  Every function returns 0 on success or a
 * negative FMA_E* code and never throws; `fma_last_error()` gives the message of the
 * calling thread's last failure.  An engine handle is thread-compatible (callers serialise
 * calls on one handle) while sleep/wake are internally multi-threaded and multi-stream and
 * never need the Python GIL.  All buffers are caller-owned except the engine handle.
 *
 * The library has NO CPU fallback: on a box without a CUDA driver `fma_engine_create`
 * fails with FMA_ENODRIVER and nothing else moves bytes.
 */
#ifndef FMA_ENGINE_H
#define FMA_ENGINE_H

#include <stddef.h>
#include <stdint.h>
#include <sys/types.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FMA_ABI_VERSION 2   /* 2: fma_stats_t grew (sleep_bytes_copied), fma_config_t.pack, packed-image and image-file entry points */

#if defined(__GNUC__)
#define FMA_API __attribute__((visibility("default")))
#else
#define FMA_API
#endif

/* ---- error codes ------------------------------------------------------------------ */
#define FMA_OK          0
#define FMA_EINVAL     -1   /* bad argument                                            */
#define FMA_ENODRIVER  -2   /* libcuda.so.1 / no CUDA device: the engine refuses to run */
#define FMA_ECUDA      -3   /* a CUDA driver/runtime call failed (see fma_last_error)   */
#define FMA_ENOMEM     -4   /* host or device memory exhausted                          */
#define FMA_ESTATE     -5   /* call not legal in the current sleep state                */
#define FMA_ENOTFOUND  -6   /* unknown pointer / segment / tag                          */
#define FMA_EINTEGRITY -7   /* digest mismatch after wake (only with FMA_FLAG_VERIFY)   */
#define FMA_EIO        -8   /* a read or write of a file failed (a full disk included)  */

/* ---- units ------------------------------------------------------------------------ */
/* The engine's unit of placement is the 2 MiB VMM page (cuMemGetAllocationGranularity
 * minimum on H100).  Every segment handed out by my_malloc / fma_alloc is a whole number
 * of pages, so the packed image of a sleeping model is a concatenation of pages and
 * gather / scatter are page-table driven (K1/K2, csrc/fma_kernels.cu).                  */
#define FMA_PAGE_BYTES  ((size_t)2u << 20)
#define FMA_MAX_TAGS    64
/* An image file or exported host store ends in its descriptor: the last FMA_IMAGE_TAIL_BYTES bytes (fma_image_export,
 * fma_image_adopt_file, fma_image_file_info). */
#define FMA_IMAGE_TAIL_BYTES ((size_t)2u << 20)

/* ---- tiers ------------------------------------------------------------------------ */
#define FMA_TIER_HOST   0   /* pinned host-DRAM store over PCIe Gen5 (copy engines)      */
#define FMA_TIER_PEER   1   /* peer-GPU HBM parking buffer over NVLink / NVSwitch        */
#define FMA_TIER_LOCAL  2   /* parking buffer in the SAME GPU's HBM (kernel roofline/test)*/
#define FMA_TIER_FILE   3   /* a file on local disk (fma_file_store): no host store while asleep */

/* ---- data-path modes (how bytes cross the link) ----------------------------------- */
#define FMA_MODE_AUTO     0
#define FMA_MODE_DIRECT   1  /* copy engines move each segment chunk <-> store directly   */
#define FMA_MODE_STAGED   2  /* K1 TMA-gather -> contiguous HBM ring -> copy engines;
                                wake: copy engines -> ring -> K2 TMA-scatter              */
#define FMA_MODE_KERNEL   3  /* K1/K2 read/write the store themselves: mapped pinned host
                                memory (zero-copy PCIe), or peer / local HBM (NVLink tier) */

/* ---- kernel variants (K1/K2 page copy) -------------------------------------------- */
#define FMA_KERNEL_TMA   0   /* cp.async.bulk (UBLKCP) + mbarrier multi-stage ring        */
#define FMA_KERNEL_LDG   1   /* 128-bit LDG/STG grid-stride copy, streaming cache hints   */

/* ---- flags for fma_sleep / fma_wake ----------------------------------------------- */
#define FMA_FLAG_VERIFY   (1u << 0)  /* K3 digest before sleep, re-check after wake       */
#define FMA_FLAG_KEEP_BACKUP (1u << 1) /* wake does not drop the backup (tests, re-wake)  */
#define FMA_FLAG_WRITE_BEHIND (1u << 2) /* fma_sleep / fma_swap to FMA_TIER_FILE: sleep into the host store at PCIe speed and
                                          write the file after the call returns (see fma_image_writeback); other tiers: ignored */

typedef struct fma_engine fma_engine_t;

typedef struct fma_config {
    uint32_t abi_version;       /* FMA_ABI_VERSION                                        */
    int32_t  mode;              /* FMA_MODE_*            (0 = auto)                        */
    int32_t  kernel;            /* FMA_KERNEL_*                                            */
    int32_t  copy_streams;      /* copy-engine streams per direction (0 = default 4)       */
    uint64_t chunk_bytes;       /* DMA chunk (DIRECT, 0 = 32 MiB) / ring-slot size (STAGED, 0 = 512 MiB) */
    int32_t  ring_slots;        /* HBM staging ring slots for STAGED (0 = default 2); the ring is
                                   transient: allocated per sleep/wake call, freed before return */
    int32_t  map_threads;       /* host threads doing cuMemCreate/Map on wake (0 = 1)      */
    int32_t  numa_bind;         /* 1 = bind the host store to the GPU's NUMA node (default),
                                   0 = leave placement to the OS, -1 = default             */
    int32_t  pack;              /* 1 = PACKED host image: bf16 pages are stored in the lossless "FMP4" code
                                   (csrc/fma_codec.h, 0.758 of their size) by K4 on sleep and decoded by K5 on
                                   wake; pages that do not code well stay raw.  Host tier: through the staging ring
                                   (STAGED); peer / local tiers: K4 / K5 write / read the parking store themselves;
                                   0 = off */
    uint64_t reserved[6];
} fma_config_t;

typedef struct fma_segment_info {
    uint64_t va;                /* device virtual address (stable across sleep/wake)       */
    uint64_t bytes;             /* page-aligned size                                       */
    uint64_t requested_bytes;   /* size the caller asked for                               */
    uint64_t packed_offset;     /* offset inside the packed store image, UINT64_MAX if none */
    uint64_t seq;               /* allocation order                                         */
    int32_t  tag;               /* interned tag id                                          */
    int32_t  mapped;            /* 1 = physical memory mapped                               */
    int32_t  has_backup;        /* 1 = bytes live in a store (host / peer / local)          */
    int32_t  tier;              /* tier holding the backup                                  */
} fma_segment_info_t;

typedef struct fma_stats {
    /* last sleep */
    double   sleep_seconds;         /* wall, entry -> exit of fma_sleep                     */
    double   sleep_copy_seconds;    /* device time first copy/kernel -> last (CUDA events)  */
    double   sleep_unmap_seconds;   /* host time in cuMemUnmap/Release                      */
    uint64_t sleep_bytes_offloaded; /* W: bytes that crossed the link                       */
    uint64_t sleep_bytes_discarded;
    /* last wake */
    double   wake_seconds;          /* wall, entry -> exit of fma_wake                      */
    double   wake_copy_seconds;     /* device time first copy/kernel -> last (CUDA events)  */
    double   wake_map_seconds;      /* host time in cuMemCreate/Map/SetAccess (all threads) */
    double   wake_first_copy_delay; /* wall from entry until the first H2D was enqueued     */
    uint64_t wake_bytes_restored;   /* W                                                    */
    uint64_t wake_bytes_remapped_only;
    /* kernels (K1/K2) of the last sleep / wake, summed over launches, CUDA events          */
    double   kernel_seconds;
    uint64_t kernel_bytes;          /* algorithmic bytes: read + write                      */
    uint32_t kernel_launches;
    uint32_t copy_ops;              /* cudaMemcpyAsync calls issued                         */
    /* host store */
    uint64_t host_store_bytes;
    double   host_store_pin_seconds;
    int32_t  host_store_numa_node;
    int32_t  tier;
    int32_t  mode;
    int32_t  image_packed;          /* 1 = the sleeping image is in the PACKED form (config.pack) */
    /* lifetime counters */
    uint64_t total_kernel_launches;
    uint64_t total_copy_ops;
    /* memory accounting NOW (for sleeper budgets: the controller today assumes 4096 MiB per sleeper,
     * cmd/dual-pods-controller/main.go:72-74, and scrapes nvidia-smi, inference-server.go:1609-1636) */
    uint64_t hbm_mapped_bytes;      /* physical HBM behind live mapping units of this engine            */
    uint64_t hbm_aux_bytes;         /* staging ring + page tables + digest scratch on this GPU           */
    uint64_t parked_bytes;          /* parking buffer held in a peer's (or this GPU's) HBM               */
    uint64_t image_store_bytes;     /* bytes the last sleep's image takes in its store: == sleep_bytes_offloaded,
                                       or less for a PACKED image (these are the bytes that cross PCIe); with a
                                       resident share only the host-store part                              */
    uint64_t sleep_bytes_copied;    /* bytes the last sleep actually moved into the store: image_store_bytes for a full
                                       sleep, 0 for a clean INCREMENTAL sleep, the changed segments for a partial one */
    uint64_t resident_bytes;        /* HBM the resident part of a sleeping host-tier image holds on this GPU now
                                       (option "resident_bytes"; its stored bytes, in one allocation rounded up to
                                       2 MiB); 0 when there is none                                          */
    uint64_t io_buffer_bytes;       /* pinned host DRAM of the engine's file I/O windows (fma_load_file and the file tier;
                                       pinned once per engine): all the host DRAM a file-tier sleeper holds        */
    uint64_t prefetched_bytes;      /* HBM the prefetched copy of a sleeping image holds on this GPU now (fma_image_prefetch;
                                       its stored bytes, in one allocation rounded up to 2 MiB); not in resident_bytes */
} fma_stats_t;

/* ---- library ---------------------------------------------------------------------- */
FMA_API int          fma_abi_version(void);
FMA_API const char*  fma_last_error(void);
/* 0 if a CUDA driver and at least one device are usable from this process. */
FMA_API int          fma_driver_available(void);

/* ---- engine lifecycle ------------------------------------------------------------- */
/* Replaces: the per-process CuMemAllocator singleton (vllm:device_allocator/cumem.py:118-138)
 * and the C module init `init_module` of cumem_allocator (SURVEY.md §2 T3). */
FMA_API int  fma_engine_create(int device, const fma_config_t* cfg, fma_engine_t** out);
FMA_API int  fma_engine_destroy(fma_engine_t* e);
/* The engine that `my_malloc` / `my_free` route to (torch's pluggable-allocator signature
 * carries no user pointer; same process-global convention as the reference C module). */
FMA_API int  fma_set_current(fma_engine_t* e);
FMA_API fma_engine_t* fma_get_current(void);

/* ---- tags (vLLM uses "weights", "kv_cache", "default": gpu_worker.py:337,557; cumem.py:116) */
FMA_API int  fma_tag_intern(fma_engine_t* e, const char* name);      /* -> tag id >= 0              */
FMA_API int  fma_tag_name(fma_engine_t* e, int tag, char* buf, size_t buflen);
/* Tag applied to subsequent allocations — replaces `CuMemAllocator.current_tag`
 * (cumem.py:133,276-277) set by `use_memory_pool(tag)`. */
FMA_API int  fma_set_current_tag(fma_engine_t* e, int tag);

/* ---- allocation ------------------------------------------------------------------- */
/* Exact torch CUDAPluggableAllocator signatures
 * (torch:include/torch/csrc/cuda/CUDAPluggableAllocator.h:20-22), same symbol names the
 * reference passes to torch (cumem.py:71-73 "my_malloc","my_free").  They replace
 * cumem_allocator's my_malloc/my_free: cuMemAddressReserve + cuMemCreate + cuMemMap +
 * cuMemSetAccess, and the inverse.  On failure my_malloc returns NULL. */
FMA_API void* my_malloc(ssize_t size, int device, void* stream);
FMA_API void  my_free(void* ptr, ssize_t size, int device, void* stream);
/* Same thing for non-torch callers (Go via cgo, tests). */
FMA_API int  fma_alloc(fma_engine_t* e, size_t bytes, int tag, void** out_ptr);
FMA_API int  fma_free(fma_engine_t* e, void* ptr);

/* ---- segment table — replaces `pointer_to_data` (cumem.py:47-55,131) -------------- */
FMA_API int       fma_segment_count(fma_engine_t* e);
FMA_API int       fma_segment_info(fma_engine_t* e, int index, fma_segment_info_t* out);
FMA_API int       fma_segment_find(fma_engine_t* e, const void* ptr);     /* -> index or FMA_ENOTFOUND */
/* Σ bytes of live segments — replaces CuMemAllocator.get_current_usage (cumem.py:310-318) */
FMA_API uint64_t  fma_current_usage(fma_engine_t* e);

/* ---- the hot path ----------------------------------------------------------------- */
/* fma_sleep replaces CuMemAllocator.sleep(offload_tags) (cumem.py:177-225): every live
 * segment whose tag bit is set in `offload_tag_mask` is backed up into the tier's store,
 * then EVERY segment is unmapped and its physical memory released; VAs stay reserved.
 * Calling it while already asleep is a harmless no-op (Executor.sleep, abstract.py:323-325). */
FMA_API int  fma_sleep(fma_engine_t* e, uint64_t offload_tag_mask, int tier, uint32_t flags);
/* fma_wake replaces CuMemAllocator.wake_up(tags) (cumem.py:227-249): every segment whose
 * tag bit is in `tag_mask` (0 = all tags) gets fresh physical memory at the SAME VA; if it
 * has a backup the bytes are copied back and the backup dropped.  Idempotent and retry-safe
 * (the controller retries /wake_up: inference-server.go:477-480,1699-1716). */
FMA_API int  fma_wake(fma_engine_t* e, uint64_t tag_mask, uint32_t flags);
/* 1 while any segment is unmapped — the worker-level truth behind GET /is_sleeping
 * (pkg/api/interface.go:129-133; cmd/test-server/main.go:69-81). */
FMA_API int  fma_is_sleeping(fma_engine_t* e);
/* Hot swap (BASELINE config 4): sleep `out_e` and wake `in_e` concurrently so that the
 * D2H of the old model and the H2D of the new one use both PCIe directions at once. */
FMA_API int  fma_swap(fma_engine_t* out_e, uint64_t offload_tag_mask, int tier,
              fma_engine_t* in_e, uint64_t wake_tag_mask, uint32_t flags);

/* ---- stores ----------------------------------------------------------------------- */
/* Pre-pin `bytes` of host store (NUMA-local to the GPU) off the critical path; fma_sleep
 * grows it on demand otherwise.  Replaces the per-segment `torch.empty(pin_memory=True)`
 * inside the reference's sleep loop (cumem.py:204-209). */
FMA_API int  fma_host_reserve(fma_engine_t* e, size_t bytes);
FMA_API int  fma_host_release(fma_engine_t* e);
/* Read-only view of the packed host image (valid while asleep in FMA_TIER_HOST). */
FMA_API int  fma_host_store_view(fma_engine_t* e, const void** base, uint64_t* bytes);
/* Reserve a parking buffer of `bytes` in `peer_device`'s HBM, mapped P2P into this
 * engine's device (cuMemCreate on the peer + cuMemMap + cuMemSetAccess for both). */
FMA_API int  fma_peer_reserve(fma_engine_t* e, int peer_device, size_t bytes);
FMA_API int  fma_peer_release(fma_engine_t* e);

/* ---- image hand-over between processes (SURVEY.md §5 checkpoint/resume, §8f-1) ---------------------------------
 * In the reference the level-1 backup is owned by the sleeping process and dies with it, after which the controller
 * cold-starts a new instance (pkg/controller/dual-pods/inference-server.go:416-448).  With FMA_HOST_STORE_SHM=1 the host
 * store is a memfd: a sleeping engine can hand its packed image (data + a descriptor of segment sizes, tags and K3
 * digests) to another process as a file descriptor, and an engine that has allocated the SAME segment sequence (same
 * model, freshly created, contents irrelevant) adopts it and is then "asleep with that image": a following fma_wake
 * restores the weights at PCIe speed instead of re-reading a checkpoint.  The fd may also be a regular FILE holding
 * the same bytes (Engine.image_save / image_load in the Python binding): if its mapping cannot be pinned in place the
 * image is copied once into an anonymous pinned store.  A PACKED image travels with its page table (descriptor v2).
 * Tests: in-process and cross-process, plain and PACKED (tests/test_gpu_parity.py). */
FMA_API int  fma_image_export(fma_engine_t* e, int* out_fd);          /* caller owns (closes) the returned fd          */
/* flags: FMA_FLAG_VERIFY = "sleep by adoption": the engine holds the weights itself (another replica of the model the image
 * came from) and its device bytes must match the image's digests — then its device side is released and it shares that
 * image (one host copy per node instead of one per replica); on a mismatch nothing is touched and FMA_EINTEGRITY comes back. */
FMA_API int  fma_image_adopt(fma_engine_t* e, int fd, uint64_t tag_mask, uint32_t flags);  /* fd stays owned by the caller */

/* ---- FILE tier: a sleeping model's image on local disk, no host store while asleep ------------------------------------
 * A host-tier sleeper holds its whole image in pinned host DRAM, and host DRAM is what limits the sleepers of a node.  In the
 * reference a model that did not fit is deleted and cold-started (pkg/controller/dual-pods/inference-server.go:416-448).
 * fma_sleep(..., FMA_TIER_FILE, ...) writes the image to the file named by fma_file_store: the STAGED pipeline (K1 gather, or
 * K4 gather + encode with config.pack, into the HBM staging ring -> D2H into the engine's pinned I/O windows) with writer threads
 * that pwrite each window at its place in the file.  fma_wake reads it back: reader threads pread ahead into the windows -> H2D into
 * the ring -> K2 / K5.  The file has the layout image_save writes: the image bytes (the PACKED form's stored pages back to back),
 * then the descriptor in the last 2 MiB, written after one fdatasync, so a torn file is never adopted.  I/O goes through O_DIRECT
 * when the file's filesystem accepts it, else through the page cache with posix_fadvise(DONTNEED) behind it (timeline row
 * "file_io": idx 1 = O_DIRECT, 0 = buffered; FMA_FILE_BUFFERED=1 forces the buffered path).  What stays in host DRAM is the I/O
 * windows (fma_stats_t.io_buffer_bytes), pinned once per engine by fma_file_store / fma_image_adopt_file.
 * Failures: the free space is checked (fstatvfs) before anything is released; if it is short, or the file cannot be opened,
 * FMA_EIO comes back with the engine fully awake.  A unit is unmapped only after its bytes' pwrite has returned, so a sleep whose
 * write fails half way (FMA_EIO) leaves every released segment in the file and a wake restores them.  A wake whose read fails
 * (FMA_EIO, e.g. the file was truncated) is rolled back like any failed wake and can be retried.  The tier needs a staging ring:
 * without HBM for one a sleep returns FMA_ENOMEM fully awake and a wake FMA_ENOMEM rolled back.  Combinations: PACKED both
 * ways; INCREMENTAL clean sleeps only (the file outlives the wake: a clean sleep to the same path writes 0 bytes, anything else
 * is a full sleep); the resident share and multi-path are ignored; fma_image_export, fma_image_describe and
 * fma_host_store_share return FMA_ESTATE for a file-tier image (the file itself is the hand-over). */
/* The file the next file-tier sleep writes (created or overwritten; the caller owns the path, the engine never unlinks it);
 * NULL forgets the path.  Pins the engine's I/O windows if they are not yet pinned. */
FMA_API int  fma_file_store(fma_engine_t* e, const char* path);
/* Like fma_image_adopt, from a file written by a file-tier sleep or by image_save: the engine must be fully awake with the same
 * segment sequence for tag_mask, and FMA_FLAG_VERIFY means sleep by adoption.  Reads only the descriptor tail, pins nothing
 * else; the engine is then asleep in FMA_TIER_FILE and a wake streams the data from `path`.  A file whose descriptor does not
 * parse (torn, foreign) is refused with FMA_EINVAL and nothing touched. */
FMA_API int  fma_image_adopt_file(fma_engine_t* e, const char* path, uint64_t tag_mask, uint32_t flags);
/* WRITE-BEHIND: a file-tier sleep whose time is not bound by the disk.  A file-tier sleep holds the GPU's HBM until its last pwrite
 * has returned, so a hot swap's wake waits for the sleeper's disk.  With FMA_FLAG_WRITE_BEHIND a full file-tier sleep runs as a
 * host-tier sleep (the STAGED pipeline, plain or PACKED) into the engine's pinned host store and returns at PCIe speed; a background
 * job (one thread per engine) then pwrites the store to the fma_file_store file and seals it (fdatasync, descriptor, fdatasync) as
 * fma_image_move(FMA_TIER_FILE) does.  Once the file is complete the job takes the operation lock and commits: every backed-up
 * segment and fma_stats_t.tier report FMA_TIER_FILE, and the host store is released (after the lock, so a wake does not wait for
 * its cudaHostUnregister + munmap) — the state fma_image_move(FMA_TIER_FILE) followed by fma_host_release leaves.
 * Taken only when the engine already holds a private (not shared) host store of at least the image's stored bytes: one from
 * fma_host_reserve, or kept from an earlier host-tier sleep or wake.  The sleep never pins one.  Otherwise, and for a sleep that
 * writes nothing (a clean INCREMENTAL sleep), the sleep is the ordinary file-tier sleep and its timeline has a "wb_fallback" row
 * whose idx says why: 1 no host store, 2 too small, 3 shared, 4 nothing to write.  The cost is a pinned image-sized store while
 * awake and until the commit.  The free-space check and the file's creation come before anything is released (FMA_EIO, fully
 * awake, as in the file tier); a sleep that fails otherwise fails as a host-tier sleep, and nothing is written behind it.
 * Until the commit the image is a host-tier image in every respect (fma_stats_t.tier, fma_segment_info tier, host_store_bytes).
 * Pre-emption: every call that takes the operation lock (sleep, wake, swap, move, verify, prefetch, export / describe / share,
 * adoptions, host / peer reserve and release, paths, fma_file_store, fma_engine_destroy) first cancels a job still writing and
 * joins it — waiting at most for the pwrite each writer has in flight (one load_chunk_bytes item) or an fdatasync — then sees the
 * host-tier image: a wake during the write is a host-tier wake.  The file is emptied (it never carries a descriptor) and the store
 * kept, so the next write-behind sleep reuses it.  A commit that loses the race for the lock is cancelled the same way, even with
 * every byte written.  A job whose write fails leaves the image in the host tier and the store kept, empties the file and reports
 * the error once, through fma_image_writeback.  fma_stats and fma_image_writeback do not pre-empt.
 * Timeline: the sleep's host-tier rows and "wb_start"; at commit or cancel op "writeback" with rows file_io and total (idx 1
 * committed, 0 cancelled; bytes written); a call that cancelled a job starts its own timeline with a "wb_cancel" row (how long the
 * cancel took; its times are before the call's own entry). */
/* Waits up to timeout_s (0: polls; a negative value waits as long as it takes) for the last write-behind job.  Returns 1 while it
 * still writes (*out_pending_bytes, if given: the image bytes not yet written), 0 when none is pending (it committed, was
 * cancelled, or none was started), or the negative code of a job that failed — once per failure, with fma_last_error set on
 * the caller's thread. */
FMA_API int  fma_image_writeback(fma_engine_t* e, double timeout_s, uint64_t* out_pending_bytes);
/* What an image file holds, read from its descriptor tail alone: no engine, no driver and no CUDA call, so a node-level owner can
 * judge a dead instance's image file (keep it for a warm start, or delete it) on any host.  The tail is read by the same parser
 * every adoption uses.  Tags are reported by name, in image order of first appearance: tag ids belong to one engine
 * (fma_tag_intern), so a caller that adopts the file interns these names in its own engine.
 * Errors: FMA_EIO when the file cannot be opened or read, or is shorter than an image and its descriptor (including a file of at
 * most FMA_IMAGE_TAIL_BYTES); FMA_EINVAL for a torn, foreign or malformed tail (what fma_image_adopt_file refuses before it looks
 * at an engine). */
typedef struct {
    uint64_t image_bytes;         /* stored bytes in front of the descriptor (the PACKED form's pages back to back)       */
    uint64_t weight_bytes;        /* bytes of the segments the image restores                                             */
    uint32_t n_segments;
    uint32_t version;             /* descriptor version: 1 plain, 2 PACKED                                                */
    int32_t  packed;
    int32_t  digests;             /* 1: every segment carries a K3 digest (a wake with FMA_FLAG_VERIFY checks them all)    */
    uint32_t n_tags;
    uint32_t reserved0;
    char     tags[FMA_MAX_TAGS][32];   /* NUL-terminated names, n_tags of them                                            */
    uint64_t reserved[4];
} fma_image_file_info_t;
FMA_API int  fma_image_file_info(const char* path, fma_image_file_info_t* out);

/* ---- moving a sleeping image between tiers, without waking it ----------------------------------------------------------
 * A sleeper's tier is otherwise fixed at sleep time, and waking it to sleep again takes HBM that belongs to whoever serves on the
 * GPU.  fma_image_move copies the image of a sleeping engine to `tier` and makes it sleep there: a host-tier sleeper is demoted to
 * disk when host DRAM runs short, a parked image leaves the parking GPU's HBM, a file-tier image is promoted to host DRAM ahead of
 * an expected wake.  Every tier stores the image in one layout, so a move is a byte copy (nothing is decoded or re-encoded, no
 * weight memory is mapped): host <-> parking buffer by the copy engines (direct_chunk pieces over the engine's copy streams);
 * host <-> file by the file tier's reader / writer threads, pread / pwrite straight into / out of the pinned store (O_DIRECT under
 * the file tier's rule); parking buffer <-> file through the pinned I/O windows.
 * The destination is prepared as a sleep to its tier prepares it: FMA_TIER_HOST reserves the host store (a shared one is first
 * swapped for a private one), FMA_TIER_LOCAL reserves the parking buffer on the engine's own GPU (the only move that allocates HBM),
 * FMA_TIER_PEER needs a parking buffer (fma_peer_reserve / fma_peer_attach) of at least image_store_bytes, FMA_TIER_FILE needs
 * fma_file_store(path): free space is checked (fstatvfs) before a byte is written, and the file is completed like a file-tier
 * sleep's (fdatasync, descriptor, fdatasync), so fma_image_adopt_file and image_load open it.
 * After success every backed-up segment and fma_stats_t.tier report `tier`, K3 digests still hold (FMA_FLAG_VERIFY on the next wake
 * checks them), and the next fma_wake takes that tier's route.  The source is left as it was: the host store and the parking buffer
 * stay allocated (fma_host_release / fma_peer_release now succeed) and a source file is never touched.
 * Refusals leave the engine unchanged: FMA_ESTATE when nothing sleeps, a backed-up segment is mapped (a KEEP_BACKUP or partial
 * wake), part of the image is in a resident share, or the destination is not prepared; FMA_EINVAL for an unknown tier, the tier
 * the image is in (FILE -> FILE included) and PEER <-> LOCAL (there is one parking buffer).  A move that fails (FMA_EIO, FMA_ENOMEM,
 * FMA_ECUDA) leaves the image where it was: records and statistics unchanged, a host store or local buffer it created released, and
 * the host store or parking buffer (a peer's or an attached one included) that it would have replaced kept, a destination file
 * emptied (never with a descriptor).  A replaced store or buffer is released only once the move has succeeded.  Only the engine's own streams and events are synchronised, so another
 * engine of the process may serve meanwhile; host <-> file moves make no CUDA call beyond pinning a host store they create.  fma_timeline: op "move", rows file_io,
 * copies_landed (the copy engines ran) and total (bytes = image_store_bytes). */
FMA_API int  fma_image_move(fma_engine_t* e, int tier);

/* Check the sleeping image against the K3 digests it carries, where it lies (host store, parking buffer, resident share, file),
 * without mapping a segment.  Returns the number of segments whose stored bytes do not match (0 = intact) and writes up to `cap`
 * of their indices (fma_segment_info order) to `out_bad`; or a negative error.
 * Every segment that has a backup and is unmapped is checked: plain pages by K3 and PACKED pages by K6, which decodes a stored page
 * as K5 would and digests it without writing it.  A stored PACKED page that cannot be decoded (bad magic, too many exceptions, a
 * size that disagrees with the page table) counts its segment as bad.  The kernels read the parking buffer and the resident share
 * in HBM, the host store through its device alias and a file through the engine's pinned I/O windows (reader threads pread whole
 * stored pages into them, O_DIRECT when the filesystem accepts it), so no HBM is taken; a host store without a device alias is
 * copied through 2 x 64 MiB of HBM scratch, freed before the call returns.  An adopted image (fma_image_adopt, _adopt_file,
 * _adopt_parked) is checked against the digests that came with it: fma_image_adopt_file reads only the descriptor, and this call
 * reads the rest.  FMA_ESTATE, with the engine unchanged: nothing is asleep, a segment to check carries no digest (sleep with
 * FMA_FLAG_VERIFY or the "incremental" option), or a mapped segment keeps a backup (a KEEP_BACKUP or partial wake).  FMA_EIO: the
 * image file cannot be opened or is shorter than the image.  No segment, tier, store, statistic or INCREMENTAL shadow changes;
 * the timeline records op "verify" with file_io, kernel and total rows (total's idx = the number of bad segments). */
FMA_API int  fma_image_verify(fma_engine_t* e, int* out_bad, int cap);

/* Prefetch part or all of the sleeping image into this engine's own GPU ahead of a wake, or drop that copy, without waking it.
 * A wake is bounded by the link its image crosses (PCIe for the host tier, the disk for the file tier); the resident share keeps
 * bytes off it too, but is fixed at sleep time and only given back by a wake.  Once a caller knows which sleeper wakes next, and
 * how much HBM the GPU can spare, it copies that much of the image into HBM here, and gives it back with bytes = 0.
 * `bytes` is rounded down to 2 MiB.  The segments copied follow the resident share's rule over stored sizes: from the last segment
 * in image order to the first, a segment is taken if its stored size still fits what is left (a budget of image_store_bytes or
 * more takes all of it).  They go, back to back, into ONE VMM allocation on the engine's GPU; a PACKED image's stored pages stay
 * coded (0.758 of the bf16 weights).  From the host store the copy engines move them (direct_chunk pieces over the engine's copy
 * streams); from a file, the file tier's reader threads pread them into the pinned I/O windows and the copy engines take them from
 * there (O_DIRECT under the file tier's rule).  The tier's store keeps every byte: the prefetch is a copy, so dropping it copies
 * nothing, and hand-overs (fma_image_export, _describe, fma_host_store_share, a file adopted elsewhere), the K3 digests and the
 * INCREMENTAL shadows are unaffected.  Nothing is mapped and no segment record but the prefetch's own table changes.
 * The next fma_wake restores the prefetched segments from HBM through the resident share's restore (K2 / K5 pieces between the link
 * part's launches, as soon as their runs are mapped) and moves only the others over the link (a file-tier wake reads only their
 * pages); the buffer is freed once that restore has completed and every run is mapped, while a prefetched segment still sleeps
 * after a tag-selective wake it stays, after an FMA_FLAG_KEEP_BACKUP wake it goes (the store is the backup), and a wake that fails
 * is rolled back with the buffer kept for the retry.  fma_image_move between the host and file tiers keeps it; a move to the peer
 * or local tier frees it after success.  fma_image_verify checks the prefetched copy as well as the store (K3 plain, K6 PACKED).
 * A segment freed while asleep leaves the table; fma_engine_destroy frees the buffer.
 * A call while a prefetch exists replaces it: the old buffer is freed first, so only the new part's HBM is needed.  bytes = 0
 * frees it and succeeds when there is none, whatever the engine's state.  Refusals leave the engine unchanged: FMA_ESTATE when
 * nothing is asleep, a backed-up segment is mapped (a KEEP_BACKUP or partial wake), or the image keeps a resident share from its
 * sleep (set resident_bytes to 0 and sleep again); FMA_EINVAL when the image sleeps in the peer or local tier (it is in HBM already).
 * Failures leave no buffer and the image, its tier and every statistic as they were: FMA_ENOMEM (no HBM for the buffer), FMA_EIO
 * (the image file cannot be opened, is shorter than the image or a read fails), FMA_ECUDA.  Like every image call it runs alone on
 * the engine (it waits for a sleep, wake, move or verify in flight), synchronises only the engine's own streams and events, and
 * records timeline op "prefetch" with rows file_io, copies_landed and total (idx = segments, bytes = stored bytes prefetched).
 * fma_stats_t.prefetched_bytes reports the buffer's stored bytes. */
FMA_API int  fma_image_prefetch(fma_engine_t* e, uint64_t bytes);

/* ---- MULTI-PATH wake: borrow idle peers' PCIe links ---------------------------------------------------------------------
 * A host-tier wake is bounded by ONE x16 Gen5 link (55.6 GB/s measured of 64): 0.29 s for Llama-3-8B however good the engine
 * is.  When other GPUs of the box are idle (BASELINE config 5: the GPUs that only park sleepers; any N=1 deployment on an
 * 8-GPU node) their links are idle too.  fma_paths_set names such helper GPUs; a following fma_wake of a plain host image
 * then cuts the image into chunks, lets every path — own link included — pull chunks through ITS copy engine into a small
 * staging buffer in ITS HBM, and K2 on the waking GPU gathers each chunk over NVLink / NVSwitch into the destination pages.
 * n = 0 turns it off.  slot_bytes / slots: staging per path (0 = 128 MiB x 3).  The reference has one blocking cudaMemcpy
 * per segment on one link (cumem.py:237-249). */
FMA_API int  fma_paths_set(fma_engine_t* e, const int* helper_devices, int n, size_t slot_bytes, int slots);

/* ---- MULTI-PATH wake across processes --------------------------------------------------------------------------------------
 * Under the launcher an instance cannot see (or drive) the idle GPUs whose links it would like to borrow.  The node-level owner
 * can.  OWNER: fma_helper_open(device) creates one staging buffer per helper GPU (exportable; *out_fd goes to the instance),
 * fma_store_attach(fd) maps + pins the instance's memfd host store (fma_host_store_share; FMA_HOST_STORE_SHM=1), and
 * fma_helper_pull(helper, store, mailbox_fd, path_index >= 1, generation, timeout_s) serves one wake on one path: that GPU's copy
 * engine pulls chunks over that GPU's link and publishes "chunk landed" per slot in the mailbox.  INSTANCE: fma_paths_attach(engine,
 * staging fds...) maps the staging buffers for ITS GPU (NVLink), creates the mailbox (*out_mailbox_fd: send it, dup'ed, to the
 * owner) and from then on fma_wake runs K2 on every remote slot the owner reports as landed, while its own link pulls from the
 * same work counter.  fma_pull_next_generation(engine) is what the owner's helpers must be told to wait for BEFORE fma_wake is
 * called.  A pull request that never arrives costs nothing but speed: the paths that do work finish the wake.  Exactly one
 * fma_helper_pull serves a path in a wake: a repeated request, one for a wake that is over, or one whose wake never uses the
 * paths returns FMA_ESTATE without having written to the mailbox.  fma_helper_close / fma_store_detach make the pulls that still
 * use the object leave (FMA_ESTATE) and return after they have. */
FMA_API int       fma_helper_open(int device, size_t slot_bytes, int slots, uint64_t* out_handle, int* out_fd);
FMA_API int       fma_helper_close(uint64_t handle);
FMA_API int       fma_store_attach(int fd, uint64_t* out_handle);
FMA_API int       fma_store_detach(uint64_t handle);
FMA_API int       fma_helper_pull(uint64_t helper, uint64_t store, int mailbox_fd, int path_index, uint64_t generation, double timeout_s);
FMA_API int       fma_paths_attach(fma_engine_t* e, const int* staging_fds, int n, size_t slot_bytes, int slots, int* out_mailbox_fd);
FMA_API uint64_t  fma_pull_next_generation(fma_engine_t* e);
FMA_API int       fma_host_store_share(fma_engine_t* e, int* out_fd);

/* ---- node-level parking buffers (exportable; SURVEY section 8f-1) ------------------- */
/* The reference launcher restricts every instance to its own GPUs (inference_server/launcher/launcher.py:171-187), and
 * whatever an instance allocates dies with it — which is when the controller cold-starts
 * (pkg/controller/dual-pods/inference-server.go:416-448).  A node-level owner (the node agent) therefore creates the
 * parking buffer: a VMM allocation in `device`'s HBM with a POSIX-fd shareable handle.  *out_fd can be sent to any process
 * on the node (SCM_RIGHTS, inheritance); the buffer lives until fma_parking_destroy AND the last importer has let go. */
FMA_API int  fma_parking_create(int device, size_t bytes, uint64_t* out_handle, int* out_fd);
FMA_API int  fma_parking_export(uint64_t handle, int* out_fd, uint64_t* out_bytes);   /* another fd for another instance   */
FMA_API int  fma_parking_destroy(uint64_t handle);
/* Instance side: use the owner's buffer (`bytes` = the size it was created with, a multiple of 2 MiB) as this engine's
 * peer-tier store.  Imports the handle, maps it and grants access to the ENGINE's GPU only; the buffer's GPU need not be
 * visible to this process.  Replaces fma_peer_reserve for instances that cannot see their parking GPU. */
FMA_API int  fma_peer_attach(fma_engine_t* e, int fd, size_t bytes);
/* Hand-over of an image parked in such a buffer.  fma_image_describe(tier) returns the descriptor of the image sleeping in
 * `tier` (segment sizes, tags, K3 digests, page table of a PACKED image; at most 2 MiB; call with buf=NULL to size it) —
 * the owner keeps it next to the fd.  A fresh engine with the same segment sequence (another process, after the first one
 * died) calls fma_peer_attach and then fma_image_adopt_parked: it releases its device side and wakes from the parked image.
 * With FMA_FLAG_VERIFY the engine's current device bytes must equal the image's (sleep by adoption). */
FMA_API int  fma_image_describe(fma_engine_t* e, int tier, void* buf, size_t cap);
FMA_API int  fma_image_adopt_parked(fma_engine_t* e, const void* desc, size_t desc_bytes, uint64_t tag_mask, uint32_t flags);

/* ---- integrity (K3) and synthetic data (K0) --------------------------------------- */
/* 64-bit position-sensitive digest of a mapped segment, computed on the device.
 * Definition: oracle/fma_oracle.h `fma_oracle_digest`. */
FMA_API int  fma_digest_segment(fma_engine_t* e, int index, uint64_t* out);
/* Digests of all mapped segments whose tag is in tag_mask (0 = all); out[i] for table
 * index i, untouched entries set to 0.  One kernel launch for the whole table. */
FMA_API int  fma_digest_all(fma_engine_t* e, uint64_t tag_mask, uint64_t* out, int n);
/* Counter-based PRNG fill of a mapped segment (splitmix64, oracle `fma_oracle_fill`):
 * word j of the segment = splitmix64(seed, first_word + j). */
FMA_API int  fma_fill_segment(fma_engine_t* e, int index, uint64_t seed, uint64_t first_word);
/* Host <-> segment byte access through the engine (tests, Go callers without torch). */
FMA_API int  fma_segment_write(fma_engine_t* e, int index, uint64_t offset, const void* host_src, uint64_t bytes);
FMA_API int  fma_segment_read(fma_engine_t* e, int index, uint64_t offset, void* host_dst, uint64_t bytes);

/* ---- PACKED host image (config.pack / option "pack"; format: csrc/fma_codec.h) ------------------------------
 * No counterpart in the reference: vLLM's sleep copies every segment verbatim (vllm:device_allocator/cumem.py:198-213).
 * These entry points only expose the image's layout and the three kernels for tests and measurement; the feature itself
 * rides inside fma_sleep / fma_wake. */
/* Where each 2 MiB page of the sleeping image lives in the store: page p (= packed_offset / FMA_PAGE_BYTES of the
 * segment that owns it) occupies out_bytes[p] bytes at out_offsets[p].  Returns the number of image pages (also when
 * cap is smaller; then only cap entries are written), 0 if nothing sleeps.  For an image that is not packed the
 * answer is the identity layout (offset p * 2 MiB, 2 MiB each). */
FMA_API int  fma_image_pages(fma_engine_t* e, uint64_t* out_offsets, uint32_t* out_bytes, uint32_t cap);
/* K4p / K4 / K5 on caller-provided pages (parity tests, roofline measurement).  K4p: out_stored_bytes[p] = size page p
 * would take (host array).  K4: device pages -> stored pages laid out back to back from dst_base with the sizes K4p
 * reports (out_stored_bytes as returned by K4p).  K5: inverse.  *out_ms (optional) = CUDA-event duration. */
FMA_API int  fma_op_pack_probe(fma_engine_t* e, const uint64_t* pages, uint64_t base, uint32_t n_pages,
                               uint32_t* out_stored_bytes, float* out_ms);
FMA_API int  fma_op_pack(fma_engine_t* e, const uint64_t* src_pages, uint64_t src_base, uint64_t dst_base,
                         const uint32_t* stored_bytes, uint32_t n_pages, float* out_ms);
FMA_API int  fma_op_unpack(fma_engine_t* e, uint64_t src_base, const uint32_t* stored_bytes, const uint64_t* dst_pages,
                           uint64_t dst_base, uint32_t n_pages, float* out_ms);

/* ---- raw kernel entry points (parity tests and roofline measurement) -------------- */
/* K1/K2: copy n_pages pages of FMA_PAGE_BYTES.  src_pages / dst_pages are HOST arrays of
 * device addresses (NULL = contiguous from src_base / dst_base).  Runs on an engine
 * stream; *out_ms (optional) = CUDA-event duration of the launch. */
FMA_API int  fma_op_page_copy(fma_engine_t* e, const uint64_t* src_pages, uint64_t src_base,
                      const uint64_t* dst_pages, uint64_t dst_base, uint32_t n_pages,
                      int kernel_variant, float* out_ms);
/* K3 over raw pages: out_page_digests[p] = digest of page p with word index base
 * first_word[p] (NULL = p * FMA_PAGE_BYTES/8). */
FMA_API int  fma_op_page_digest(fma_engine_t* e, const uint64_t* pages, uint64_t base,
                        const uint64_t* first_word, uint32_t n_pages,
                        uint64_t* out_page_digests, float* out_ms);
/* Plain device scratch for the raw ops above (not tracked as segments). */
FMA_API int  fma_scratch_alloc(fma_engine_t* e, size_t bytes, uint64_t* out_dev_ptr);
FMA_API int  fma_scratch_free(fma_engine_t* e, uint64_t dev_ptr);

/* ---- cold load: file -> HBM through the same pinned-ring + copy-engine mover (SURVEY.md §8f-3) ------------- */
/* "load_model" in the reference is create-instance -> vLLM's own checkpoint loader
 * (inference_server/launcher/launcher.py:656-669,799-837; vllm:v1/worker/gpu_worker.py:335-342), which copies tensor
 * by tensor from pageable (mmap'ed safetensors) memory.  fma_load_file streams byte ranges of one file into device
 * addresses inside engine segments: reader threads pread() into a small pinned bounce ring, copy engines move each
 * chunk as soon as it is read.  Spans are (file offset, bytes, destination device address); a safetensors header
 * maps to spans directly (llm-d-fast-model-actuation_b200/loader.py). */
typedef struct fma_load_span {
    uint64_t file_offset;
    uint64_t bytes;
    uint64_t dst;               /* device address; must lie inside a mapped segment of this engine */
} fma_load_span_t;

typedef struct fma_load_stats {
    double   seconds;           /* wall, entry -> all bytes resident in HBM                          */
    double   read_seconds;      /* summed over reader threads: time inside pread()                   */
    uint64_t bytes;
    uint32_t chunks;
    uint32_t threads;
    uint64_t reserved[4];
} fma_load_stats_t;

#define FMA_LOAD_O_DIRECT (1u << 0)  /* bypass the page cache (4 KiB-aligned reads into the bounce ring)  */
/* The bounce ring is the engine's pinned I/O windows, which the file tier shares; a failed read returns FMA_EINVAL. */

FMA_API int  fma_load_file(fma_engine_t* e, const char* path, const fma_load_span_t* spans, uint32_t n_spans,
                           uint32_t flags, fma_load_stats_t* out_stats);

/* ---- tuning ----------------------------------------------------------------------- */
/* Change one knob of a live engine (between operations).  Keys: "mode", "kernel",
 * "copy_streams", "chunk_bytes", "ring_slots", "map_threads", "pack", "incremental" (1 = a host-tier sleep whose offloaded segments still have the K3 digests and image
 * offsets of the copy the host store kept from the last wake releases the device side without moving a byte; anything else
 * is a full sleep), "resident_bytes" (cap, rounded down to 2 MiB,
 * on the HBM a sleeping host-tier image may keep on this GPU: walking the offloaded segments from the last in image order to the
 * first, every segment whose stored size still fits the remaining cap stays here and is restored by an HBM-to-HBM copy at wake
 * instead of crossing PCIe; 0 = off, also FMA_RESIDENT_MIB at engine creation.  Ignored by peer / local-tier sleeps and while
 * helper paths are configured.  Resident segments report tier FMA_TIER_LOCAL and an offset in the resident part; their pages
 * follow the host part's in fma_image_pages.  While an image keeps a resident part, fma_image_export, fma_image_describe and
 * fma_host_store_share return FMA_ESTATE.  If the allocation fails the sleep is a plain host-tier sleep), "tma_tile_bytes",
 * "tma_stages", "tma_pipes", "tma_ctas_per_sm", "load_threads", "load_chunk_bytes", "load_slots". */
FMA_API int  fma_set_option(fma_engine_t* e, const char* key, int64_t value);

/* ---- stats ------------------------------------------------------------------------ */
FMA_API int  fma_stats(fma_engine_t* e, fma_stats_t* out);

/* Per-phase timeline of the last fma_sleep / fma_wake / fma_image_move / fma_image_verify / fma_image_prefetch as text, one event per line:
 *   "<op>,<kind>,<idx>,<t0_ms>,<t1_ms>,<bytes>\n"   (times since the call's entry)
 * kinds: plan, map_ring / map_backed / map_remap (one cuMemCreate+Map+SetAccess each, mapper thread), gate_wait,
 * enqueue, copies_landed, wait_all_mapped, drain, unmap (sleep), kernel (K1/K2/K4/K5 launches, K3/K6 pairs of a verify, device-timed), total;
 * multi-path operations add path_chunks / path_local (idx = the path's GPU, bytes = what that path moved / moved NUMA-locally);
 * a resident share adds res_alloc (sleep) / res_free (wake) for the resident buffer's VMM calls, res_fallback (its allocation
 * failed: plain sleep), and res_gather / res_restore rows for its K1 / K4 and K2 / K5 launches (device-timed, like kernel); the
 * file tier adds file_io (idx 1 = O_DIRECT, 0 = page cache; from the file's open to its last write / read returned, bytes = file bytes).
 * The reference has no tracing on this path (SURVEY.md section 5); this is what shows WHICH phase bounds a wake.
 * Returns the length of the full text (call with buf=NULL to size it), or a negative error. */
FMA_API int  fma_timeline(fma_engine_t* e, char* buf, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* FMA_ENGINE_H */
