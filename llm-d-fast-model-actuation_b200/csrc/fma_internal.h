// fma_internal.h — what the translation units of the host engine share (NOT part of the C-ABI; include/fma_engine.h is).
//
//   fma_engine.cu   errors, driver resolution, VMM primitives, arenas, engine resources, stores, allocator, the C-ABI
//   fma_sleep.cu    SLEEP pipeline (do_sleep) and the PACKED image plan
//   fma_wake.cu     WAKE pipeline (do_wake)
//   fma_load.cu     file I/O: reader / writer threads over the pinned I/O windows (cold load fma_load_file, FILE tier)
//   fma_image.cu    image hand-over between engines / processes (fma_image_export / fma_image_adopt), moves between tiers (fma_image_move),
//                  checks in place (fma_image_verify), prefetch into HBM (fma_image_prefetch), the write-behind job of a file-tier sleep
//                  (fma_image_writeback)
//
// Everything below lives in namespace fma_impl; the library is built with -fvisibility=hidden, so none of it is exported.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cerrno>
#include <cstring>
#include <initializer_list>
#include <iterator>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <thread>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "../../include/fma_engine.h"
#include "fma_kernels.h"
#include "fma_layout.h"
#include "fma_pull.h"

namespace fma_impl {

// ------------------------------------------------------------------------------------
// errors, time, small utilities (defined in fma_engine.cu)
// ------------------------------------------------------------------------------------
extern thread_local char tl_err[512];
int fail(int code, const char* fmt, ...);
double now_s();
size_t round_up(size_t x, size_t a);
int env_int(const char* name, int dflt);

#define RT(call)                                                                                          \
    do {                                                                                                  \
        cudaError_t _e = (call);                                                                          \
        if (_e != cudaSuccess)                                                                            \
            return fail(FMA_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

#define RC(expr) do { int _rc = (expr); if (_rc != FMA_OK) return _rc; } while (0)   // an FMA_* error code goes back to the caller

// ------------------------------------------------------------------------------------
// driver API, resolved lazily through the (static) runtime: no link-time libcuda dependency
// ------------------------------------------------------------------------------------
struct Driver {
    bool ok = false;
    CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
    CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
    CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
    CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
    CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
};
extern Driver g_drv;
extern char g_drv_err[256];
bool driver_ready();
const char* cu_err(CUresult r);

#define DRV(call)                                                                                         \
    do {                                                                                                  \
        CUresult _r = (call);                                                                             \
        if (_r != CUDA_SUCCESS)                                                                           \
            return fail(_r == CUDA_ERROR_OUT_OF_MEMORY ? FMA_ENOMEM : FMA_ECUDA, "%s failed: %s (%s:%d)", #call, \
                        cu_err(_r), __FILE__, __LINE__);                                                  \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    bool changed = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) {
            cudaSetDevice(dev);
            changed = true;
        }
    }
    ~DeviceGuard() {
        if (changed && prev >= 0) cudaSetDevice(prev);
    }
};

// ------------------------------------------------------------------------------------
// data structures
// ------------------------------------------------------------------------------------
constexpr uint64_t kNoOffset = UINT64_MAX;

struct Segment {
    CUdeviceptr va = 0;
    size_t bytes = 0;       // page-aligned
    size_t requested = 0;
    int tag = 0;
    uint64_t seq = 0;
    int arena = -1;         // VA arena the segment lives in
    CUdeviceptr unit_va = 0;  // key of the mapping unit that backs it (0 while unmapped)
    bool mapped = false;
    bool has_backup = false;
    int backup_tier = FMA_TIER_HOST;
    uint64_t packed_off = kNoOffset;
    uint64_t digest = 0;
    bool digest_valid = false;
    // INCREMENTAL sleep: after a host-tier wake the store still holds this segment's bytes at shadow_off, and `digest` is
    // their K3 digest; kNoOffset = no such copy (never slept, image overwritten or released, layout changed)
    uint64_t shadow_off = kNoOffset;
    // PREFETCH (fma_image_prefetch): a copy of its stored bytes is in the prefetch buffer, at this offset of the prefetch part's
    // image space; backup_tier and packed_off still name the tier's store, which keeps every byte
    uint64_t prefetch_off = kNoOffset;
};

using fma_layout::Arena;
using fma_layout::arena_give_back;

// A live physical mapping: [va, va+bytes).  At load time a unit is one segment; after a wake it is a whole run.
// The physical handle is released right after cuMemMap (the memory lives until cuMemUnmap), so a unit is just a range.
struct Unit {
    CUdeviceptr va = 0;
    size_t bytes = 0;
    size_t live_bytes = 0;              // bytes of segments still allocated inside it
    int arena = -1;
    std::vector<std::pair<CUdeviceptr, size_t>> zombies;  // freed segments whose VA returns when the unit is unmapped
};

struct HostStore {
    void* base = nullptr;       // host pointer
    void* dev_alias = nullptr;  // device-visible alias of base (mapped pinned)
    size_t cap = 0;
    bool registered = false;    // mmap + cudaHostRegister (else cudaHostAlloc)
    int numa_node = -1;
    double pin_seconds = 0;
    int fd = -1;                // memfd backing (FMA_HOST_STORE_SHM=1 or an adopted image); -1 = anonymous memory
    bool shared = false;        // somebody else may hold this image too (exported, or adopted in place): it is READ-ONLY from
                                // now on — a sleep that has to write gets a fresh private store first (copy-on-write per store)
    bool fd_handed_out = false; // fma_host_store_share gave its memfd to a node-level owner, who may read it: a demotion
                                // (fma_image_move_flags, FMA_FLAG_WRITE_BEHIND) may not release it
    size_t map_bytes = 0;       // bytes mapped at base (cap + descriptor tail for memfd stores)
    // NUMA placement by byte range (MULTI-PATH wake: each path pulls the part of the image that lives on ITS GPU's node, so no
    // path drags its share across the socket interconnect); one range covering everything otherwise
    using NumaRange = fma_layout::NumaRange;
    std::vector<NumaRange> ranges;
    std::string placed_for;     // "node:paths,node:paths" the striping was computed for ("" = one node)
};

// Descriptor of a packed image, stored in the last 2 MiB of a memfd-backed store (fma_image_export / fma_image_adopt).
constexpr uint64_t kImageMagic = 0x31304d49414d46ull;  // "FMAIM01"
constexpr size_t kImageTail = FMA_IMAGE_TAIL_BYTES;
struct ImageSegDesc {
    uint64_t bytes;
    uint64_t packed_off;
    uint64_t digest;
    uint32_t digest_valid;
    uint32_t tag_len;
    char tag[32];
};
struct ImageHeader {
    uint64_t magic;
    uint32_t version;
    uint32_t n_segments;
    uint64_t image_bytes;
};
constexpr uint32_t kFlagAdopt = 1u << 31;  // internal: "sleep" onto an adopted image without copying

struct VmmBuffer {  // one VMM allocation, mapped at a VA of its own; it keeps its handle until vmm_buffer_free
    CUdeviceptr va = 0;
    size_t bytes = 0;
    CUmemGenericAllocationHandle handle = 0;
};

constexpr int kForeignDevice = -2;  // ParkStore::device of an attached buffer: it lives on a GPU this process may not even see

struct ParkStore : VmmBuffer {  // peer-HBM or local-HBM parking buffer (P2P mapped), or the resident share
    int device = -1;            // kForeignDevice: imported from a node-level owner's fd (fma_peer_attach)
};

constexpr int kMaxStreams = 8;
constexpr int kMaxRing = 8;
constexpr int kMaxPaths = 8;

// MULTI-PATH wake (fma_paths_set): one PCIe path into the waking GPU per entry.  Path 0 is the engine's own link; every other
// path is an idle peer GPU whose copy engine pulls chunks of the host image over ITS x16 link into a small staging buffer in
// ITS HBM, from where K2 on the waking GPU gathers them over NVLink / NVSwitch (450 GB/s per direction on H100 >> k x ~55 GB/s) straight into the
// destination pages.  A lone wake is then bounded by k links instead of one (DESIGN.md section 3).
struct WakePath {
    int device = -1;                         // -1 for a REMOTE path: a helper GPU this process cannot see (fma_paths_attach)
    bool remote = false;                     // the node-level owner drives the H2D into this path's slots (fma_pull.h)
    int numa_node = -1;                      // of `device` (sysfs); -1 unknown
    VmmBuffer staging;                       // n_slots x slot_bytes in `device`'s HBM (remote: imported); access for `device` and the engine's GPU
    cudaStream_t copy = nullptr;             // on `device`: H2D host store -> slot
    cudaStream_t kern = nullptr;             // on the engine's GPU: K2 slot -> destination pages
    cudaEvent_t ev_full[kMaxRing] = {};      // on `device`
    cudaEvent_t ev_free[kMaxRing] = {};      // on the engine's GPU
    cudaEvent_t ev_done = nullptr;           // on the engine's GPU
};

// Per-phase timeline of the last sleep / wake (fma_timeline): host-side phases (VMM calls of the mapper / unmapper threads,
// enqueue, drain) and device-side kernel launches (K1 / K2 / K4 / K5), all in seconds since the operation's entry.
struct TimelineEv {
    char kind[16];
    int32_t idx;
    double t0, t1;
    uint64_t bytes;
};

class FileIO;

// WRITE-BEHIND (FMA_FLAG_WRITE_BEHIND): the background job that writes a file-tier sleep's image from the host store to its file
// after the sleep returned (fma_image.cu).  One per engine.  It holds no op_mu while it writes: every call that takes op_mu first
// cancels a job still writing and joins it (OpLock), and the job takes op_mu only to commit, giving up when a call cancels it.
struct WriteBehind {
    enum State { Idle, Writing, Committed, Cancelled, Failed };
    std::mutex mu;                    // guards everything below but `th`
    std::condition_variable cv;       // `cancel` was set
    std::thread th;                   // joined by a pre-emption while Writing, else by the next job or fma_engine_destroy (a
                                      // committed job may still be freeing the store it detached)
    State state = Idle;
    bool cancel = false;
    bool reported = true;             // a failure has been returned by fma_image_writeback
    int error = 0;                    // FMA_OK, or the failed job's code and message
    char msg[512] = "";
    FileIO* io = nullptr;             // the writers, while they run
    uint64_t bytes = 0, piece = 0;    // the image's stored bytes; the bytes of one write item (the last may be shorter)
    uint64_t written = 0;             // image bytes written, once the writers have finished
    double t_entry = 0;               // the job's start: the origin of its "writeback" timeline
    double file_t0 = 0, file_t1 = 0;  // its "file_io" row (idx: `direct`), for the call that cancels it
    bool direct = false;
};

}  // namespace fma_impl

using namespace fma_impl;  // internal header: only the engine's own translation units include it

struct fma_engine {
    int device = 0;
    size_t gran = FMA_PAGE_BYTES;
    fma_config_t cfg{};
    std::mutex mu;  // guards segs / tags (my_malloc can arrive from any torch thread)
    std::mutex op_mu;  // one sleep / wake / swap / image operation per engine at a time (a controller retry may overlap a call in flight)
    std::vector<Segment> segs;  // allocation order == reference dict order (cumem.py:198,237)
    std::map<CUdeviceptr, size_t> by_va;
    std::vector<Arena> arenas;
    std::map<CUdeviceptr, Unit> units;  // live mappings, keyed (and therefore ordered) by VA
    uint64_t next_seq = 0;
    std::vector<std::string> tags;
    int current_tag = 0;

    HostStore host;
    ParkStore park;
    // RESIDENT share (option "resident_bytes", FMA_RESIDENT_MIB): a host-tier sleep keeps the tail of its image in ONE VMM
    // allocation on this GPU (`res`, device == the engine's).  Segments whose bytes live there have backup_tier == FMA_TIER_LOCAL
    // and packed_off = their offset in the resident part (its own image space, laid out like the host part).
    uint64_t resident_cap = 0;        // option: HBM the sleeping image may keep here (2 MiB multiple; 0 = off)
    ParkStore res;
    bool res_packed = false;          // the resident part holds stored pages of the PACKED form (res_off / res_bytes)
    std::vector<uint64_t> res_off;
    std::vector<uint32_t> res_bytes;
    uint64_t res_store_bytes = 0;     // bytes the resident part occupies in `res`
    cudaEvent_t ev_res_done = nullptr;  // wake: the resident part's last restore launch has completed
    std::vector<uint64_t> res_seqs;   // Segment::seq of the segments the last sleep kept resident (INCREMENTAL: same split or full sleep)
    // PREFETCH (fma_image_prefetch): a copy of part of a sleeping host- or file-tier image in ONE VMM allocation on this GPU (`pf`),
    // the prefetched segments back to back in image order and laid out like the resident part (pf_off / pf_bytes: each page's
    // stored offset and size when the image is PACKED).  The tier's store stays complete, so dropping it copies nothing.
    ParkStore pf;
    std::vector<uint64_t> pf_off;
    std::vector<uint32_t> pf_bytes;
    std::atomic<uint64_t> pf_store_bytes{0};   // bytes the prefetched part occupies in `pf` (fma_stats reads it without op_mu)
    uint64_t image_bytes = 0;  // W of the current packed image
    int image_tier = FMA_TIER_HOST;
    // PACKED host image (option "pack", fma_codec.h): image page p (= packed_off / 2 MiB) is stored at
    // img_off[p] in the store and takes img_bytes[p] bytes (FMA_K_PACKED_PAGE_BYTES coded, 2 MiB raw)
    bool image_packed = false;
    std::vector<uint64_t> img_off;
    std::vector<uint32_t> img_bytes;
    uint64_t image_store_bytes = 0;  // bytes the image occupies in its store (== image_bytes unless packed)
    // INCREMENTAL sleep (option "incremental"): weights do not change while a model serves, so after a wake the host store
    // still holds the image.  The next sleep digests the segments on the device (K3, one HBM read) and, if every offloaded
    // segment still has the digest and the image offset of that copy, releases the device side WITHOUT moving a byte.
    int incremental = 0;
    int shadow_tier = FMA_TIER_HOST;  // the store the shadows live in (host store, or the peer / local parking buffer)
    bool shadow_packed = false;       // form / size of the image the shadows belong to (img_off / img_bytes are kept for it)
    uint64_t shadow_store_bytes = 0;
    uint64_t shadow_image_bytes = 0;
    fma_k_pack_desc* d_pdesc = nullptr;  // per-page descriptors of K4 / K5
    fma_k_pack_desc* h_pdesc = nullptr;
    uint32_t* d_psize = nullptr;         // K4p output; d_psize[pdesc_cap] is the K4/K5 error counter
    uint32_t* h_psize = nullptr;
    size_t pdesc_cap = 0;

    cudaStream_t cs[kMaxStreams] = {};  // copy-engine streams
    int n_cs = 0;
    cudaStream_t ks = nullptr;          // kernel stream
    cudaEvent_t ev_start = nullptr, ev_end = nullptr;
    cudaEvent_t ev_cs[kMaxStreams] = {};
    std::vector<cudaEvent_t> ev_pool;   // timing pairs for kernels
    std::vector<cudaEvent_t> ev_stage;  // "these segments are dead" markers for the sleep-side unmapper
    // HBM staging ring (STAGED mode)
    void* ring[kMaxRing] = {};
    cudaEvent_t ev_ring_full[kMaxRing] = {};
    cudaEvent_t ev_ring_free[kMaxRing] = {};
    int n_ring = 0;
    size_t ring_slot_bytes = 0;
    bool ring_attached = false;         // ring lives in the tail of a mapping unit (no cudaMalloc / cudaFree of its own)
    CUdeviceptr ring_unit_va = 0;       // that unit's key
    // device page tables (uploaded per operation)
    uint64_t* d_tab = nullptr;
    size_t d_tab_cap = 0;  // entries
    uint64_t* h_tab = nullptr;  // pinned mirror
    fma_k_page_desc* d_desc = nullptr;
    fma_k_page_desc* h_desc = nullptr;
    uint64_t* d_dig = nullptr;
    uint64_t* h_dig = nullptr;
    size_t desc_cap = 0;

    // I/O windows (pinned host), persistent and small: the cold load's bounce ring and the FILE tier's disk stage.  Pinned with
    // the load_* options in force when ensure_io_windows last ran; an operation uses them as they are
    void* load_ring = nullptr;
    size_t load_ring_bytes = 0;
    size_t io_window_bytes = 0;          // each window: a load chunk + 8 KiB of O_DIRECT alignment slack
    int io_windows = 0;
    std::vector<cudaEvent_t> ev_load;    // per window: the copy into / out of it has finished
    int load_threads = 12;               // pread from the page cache is the limiter: enough readers to keep
    size_t load_chunk = (size_t)16 << 20;  // one PCIe Gen5 link busy (tests/tools/load_bench.py measures it)
    int load_slots = 24;

    // MULTI-PATH wake
    std::vector<WakePath> paths;
    size_t path_slot_bytes = 0;
    int path_slots = 0;
    PullMailbox* mbox = nullptr;             // remote paths (fma_paths_attach): shared with the node-level owner
    int mbox_fd = -1;
    uint64_t pull_generation = 0;

    // FILE tier
    std::string file_path;               // fma_file_store: where the next file-tier sleep writes ("" = nowhere)
    std::string image_file;              // the file the last file-tier image was written to / adopted from (read by the wake)
    WriteBehind wb;                      // WRITE-BEHIND: the job that writes a host-tier image to file_path after its sleep

    fma_k_tma_cfg tma = fma_k_default_tma_cfg();
    fma_stats_t st{};
    // K1/K2 event pairs of the last operation whose elapsed times have not been read yet
    size_t pending_events = 0;
    uint64_t pending_kernel_bytes = 0;
    // timeline of the last operation (fma_timeline)
    std::mutex tl_mu;
    std::vector<TimelineEv> tl;
    std::vector<uint64_t> tl_kbytes;   // algorithmic bytes of each pending kernel launch (pairs in ev_pool)
    std::vector<const char*> tl_kkind; // timeline kind of each pending kernel launch ("kernel", "res_gather", "res_restore")
    char tl_op[16] = "";
    double tl_entry = 0;               // now_s() at the operation's entry
    double tl_dev_base = 0;            // host time (since entry) at which ev_start was recorded: origin of the device-side events
    // the "wb_cancel" row of the pre-emption that opened the current call (OpLock): its timeline starts with it
    bool tl_carry = false;
    double tl_carry_t0 = 0, tl_carry_t1 = 0;
    uint64_t tl_carry_bytes = 0;
    void tl_begin(const char* op, double t_entry) {
        std::lock_guard<std::mutex> lk(tl_mu);
        tl.clear();
        tl_kbytes.clear();
        tl_kkind.clear();
        snprintf(tl_op, sizeof(tl_op), "%s", op);
        tl_entry = t_entry;
        tl_dev_base = 0;
        if (tl_carry) tl.push_back(TimelineEv{"wb_cancel", 0, tl_carry_t0 - t_entry, tl_carry_t1 - t_entry, tl_carry_bytes});
    }
    void tl_add(const char* kind, int idx, double t0_abs, double t1_abs, uint64_t bytes) {
        std::lock_guard<std::mutex> lk(tl_mu);
        TimelineEv ev;
        snprintf(ev.kind, sizeof(ev.kind), "%s", kind);
        ev.idx = idx;
        ev.t0 = t0_abs - tl_entry;
        ev.t1 = t1_abs - tl_entry;
        ev.bytes = bytes;
        tl.push_back(ev);
    }
};

namespace fma_impl {

inline int tag_bit_set(uint64_t mask, int tag) { return (int)((mask >> tag) & 1ull); }
int check_engine(fma_engine_t* e);

// ---- VMM primitives, arenas (fma_engine.cu) ----
int vmm_create_and_map(int device, CUdeviceptr va, size_t bytes);
// A VMM buffer is made in two steps: a handle (created on `device`, exportable as a POSIX fd or not; or imported from an fd),
// then vmm_buffer_map.  Out of memory in the first step is FMA_ENOMEM; every other failure is FMA_ECUDA.
int vmm_create(int device, size_t bytes, bool exportable, CUmemGenericAllocationHandle* out);
int vmm_import(int fd, CUmemGenericAllocationHandle* out);
// Reserves a VA of its own for `h`, maps it and grants `access_devices` read/write access (a device listed twice once).  Takes `h`:
// on failure nothing is left, `h` included, and the message names `what`.
int vmm_buffer_map(CUmemGenericAllocationHandle h, size_t bytes, std::initializer_list<int> access_devices, const char* what, VmmBuffer* out);
void vmm_buffer_free(VmmBuffer& b);   // unmap, release, free the VA; an empty buffer is left as it is
int unmap_units(fma_engine_t* e, CUdeviceptr va, size_t span_bytes);
// drop the (unmapped) units in [va, va + bytes) from the table: zombies' VA back to their arenas, an attached ring detached
void forget_units(fma_engine_t* e, CUdeviceptr va, size_t bytes);
// ---- engine resources (fma_engine.cu) ----
int ensure_streams(fma_engine_t* e);
int ensure_tables(fma_engine_t* e, size_t n_pages);
int ensure_desc(fma_engine_t* e, size_t n_pages);
int ensure_pack_bufs(fma_engine_t* e, size_t n_pages);
size_t direct_chunk(const fma_engine_t* e);
size_t staged_slot(const fma_engine_t* e);
void release_ring(fma_engine_t* e);
size_t ring_slot_for(const fma_engine_t* e, size_t image_bytes);
int ring_slots_for(const fma_engine_t* e);
int ensure_ring_events(fma_engine_t* e, int n);
int ensure_ring(fma_engine_t* e, size_t image_bytes);
bool no_ring();
int ensure_event_pool(fma_engine_t* e, size_t n);
// ---- stores (fma_engine.cu) ----
void host_store_free(HostStore& h);
int gpu_numa_node(int device);
int host_store_reserve(fma_engine_t* e, size_t bytes);
// A wake path's streams and events for `slots` slots: a local path's copy stream and ev_full on its GPU, then the kernel stream,
// ev_free and ev_done on the current GPU (the engine's).  On failure the caller closes the path.
int open_path(WakePath& p, int slots);
void close_path(fma_engine_t* e, WakePath& p);   // undoes open_path, whatever of it was done, and frees the path's staging
void paths_release(fma_engine_t* e);
int paths_fail(fma_engine_t* e, int rc);         // fma_paths_set / fma_paths_attach failed: release every path, keep the message
int park_release(fma_engine_t* e);
int park_reserve(fma_engine_t* e, int park_device, size_t bytes);
int park_store_create(fma_engine_t* e, int device, size_t bytes, ParkStore* out);   // one VMM allocation, mapped for e's GPU (+ device's)
void resident_release(fma_engine_t* e);              // drop the resident buffer (caller: nothing on the device still reads it)
void prefetch_release(fma_engine_t* e);              // drop the prefetch buffer and its table (same condition; takes e->mu)
// Does a segment's image live in the store `where` names (takes e->mu)?
enum class ImageIn {
    Host,           // the host store
    NotHost,        // the parking buffer: any tier but the host's and the file's, so a resident share (FMA_TIER_LOCAL) counts too
    Local,          // FMA_TIER_LOCAL, with the segment unmapped
    AnyAsleep,      // any store, with the segment unmapped
};
bool image_in(fma_engine_t* e, ImageIn where);
// a sleeping image keeps part of itself in the resident buffer
inline bool resident_asleep(fma_engine_t* e) { return e->res.va && image_in(e, ImageIn::Local); }
// A hand-over of the sleeping image (fma_image_export / _describe, fma_host_store_share) cannot take that part along
inline int refuse_resident_handover(fma_engine_t* e) {
    if (!resident_asleep(e)) return FMA_OK;
    return fail(FMA_ESTATE, "part of the sleeping image is resident in this process's own HBM (option resident_bytes) and cannot be handed over: set it to 0 and sleep again");
}
// A wake restores a segment from HBM instead of its tier's store when its bytes are in the resident share or in the prefetch
// buffer (an image has one or the other, never both).  Its offset in that part's image space, or kNoOffset.
inline uint64_t hbm_offset(const fma_engine_t* e, const Segment& s) {
    if (!s.has_backup) return kNoOffset;
    if (s.backup_tier == FMA_TIER_LOCAL && e->image_tier == FMA_TIER_HOST) return s.packed_off;   // the resident share
    return s.prefetch_off;
}
struct HbmPart {   // that part: its buffer, its form and (PACKED) its page table
    uint64_t base;
    bool packed;
    const std::vector<uint64_t>* off;
    const std::vector<uint32_t>* bytes;
};
inline HbmPart hbm_part(const fma_engine_t* e) {
    if (e->pf.va) return HbmPart{(uint64_t)e->pf.va, e->image_packed, &e->pf_off, &e->pf_bytes};
    return HbmPart{(uint64_t)e->res.va, e->res_packed, &e->res_off, &e->res_bytes};
}
CUmemAllocationProp device_prop(int device);
// ---- image descriptor (fma_image.cu): what a sleeping image is made of, so another engine / process can adopt it ----
int image_descriptor_build(fma_engine_t* e, int tier, std::vector<char>* out);
// A descriptor as its format defines it, before any engine is matched against it: header, one entry per segment and, for
// version 2 (PACKED), the page table.
struct ImageDescriptor {
    ImageHeader hd;
    std::vector<ImageSegDesc> ds;
    std::vector<uint64_t> page_off;     // version 2: the PACKED image's page table
    std::vector<uint32_t> page_bytes;
};
// Reads the descriptor in `tail` for a store of `store_cap` bytes.  It comes from a file or another process, so everything it
// claims is bounded before it is used as a length.  Torn, foreign or malformed: FMA_EINVAL.  Every adoption parses through it.
int image_descriptor_read(const char* tail, size_t tail_bytes, size_t store_cap, ImageDescriptor* out);
void invalidate_shadows(fma_engine_t* e);   // the host store no longer holds a usable copy of any segment
// ---- file I/O (fma_load.cu) ----
int ensure_io_windows(fma_engine_t* e);   // pin the I/O windows for the current load_* options (and their events)
struct FileFd {   // closes on every exit path
    int fd = -1;
    ~FileFd() { if (fd >= 0) close(fd); }
};
// Reader or writer threads over the engine's pinned I/O windows.  Item k of `items` goes through window k % io_windows, and the
// caller's thread calls copy(k, dev, stream) for every item, in item order.  copy enqueues the item's copy between its window and
// the device memory `dev` on `stream`, and records the window's event behind it:
//   read:  readers pread item k into its window -> copy(k) waits for that, enqueues the H2D out of the window -> the reader of
//          item k + n reuses the window once that H2D has finished
//   write: copy(k) waits until the pwrite of item k - n has returned, enqueues the D2H into the window -> a writer pwrites item k
//          once that D2H has finished
// With O_DIRECT a read may start below its item and a write must be 4 KiB aligned (the FILE tier's always are).  In the page
// cache's mode every range read or written is dropped from it behind the I/O (posix_fadvise DONTNEED).
// With `mem` (a pinned host store: fma_image_move between the host and file tiers) there are no windows and no copies: item k is
// read into / written from mem + its file offset, and the threads run on their own until finish().  With O_DIRECT, `mem` and every
// item must then be 4 KiB aligned.
class FileIO {
  public:
    struct Item {
        uint64_t file_off, bytes;
    };
    // the most one item through a window moves: the window less its O_DIRECT slack (ensure_io_windows)
    static uint64_t max_item(const fma_engine_t* e) { return e->io_window_bytes - 8192; }
    // `ranges` cut into items of at most one window each, in order; (*ends)[r]: one past the last item of range r
    static std::vector<Item> cut(const fma_engine_t* e, const std::vector<Item>& ranges, std::vector<size_t>* ends = nullptr);
    // item_delay_ms: each thread waits that long before each item (FMA_WB_ITEM_DELAY_MS, a test knob of the write-behind job);
    // cancel() ends the wait
    FileIO(fma_engine_t* e, int fd, bool write, bool direct, std::vector<Item> items, uint64_t file_bytes, const char* path, char* mem = nullptr,
           int item_delay_ms = 0);
    ~FileIO();
    static constexpr int kCancelled = 1;   // the error of a cancelled I/O (never returned by the C-ABI)
    // The threads leave after the item each is doing (with `mem`; the write-behind job); finish() then returns kCancelled
    void cancel() { set_error(kCancelled, "file I/O of %s was cancelled", path_); }
    int copy(size_t k, void* dev, cudaStream_t stream);   // FMA_OK, a CUDA error, or (the I/O failed) finish()'s error
    // read: copy() without the copy.  enqueue(window) puts work on `stream` that reads item k in place in its pinned window (a
    // kernel reading it over the link, fma_image_verify), and the window is handed back behind that work.
    template <class Enqueue>
    int read_in_place(size_t k, cudaStream_t stream, Enqueue enqueue) {
        return post(k, stream, [&](char* win) { return enqueue(static_cast<const char*>(win)); });
    }
    size_t written();                  // items whose pwrite has returned, as a prefix of `items`
    int finish();                      // joins the threads and waits for every posted copy; FMA_OK or the first error (FMA_EIO / FMA_ECUDA)
    double io_seconds() const { return io_ns_.load() * 1e-9; }
    int threads() const { return (int)th_.size(); }

  private:
    // waits for item k's window, enqueue(window) on `stream`, records the window's event behind it and marks the item posted
    template <class Enqueue>
    int post(size_t k, cudaStream_t stream, Enqueue enqueue) {
        bool failed;
        {   // read: item k is in its window; write: the window's last pwrite (item k - n) has returned
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&] { return error_ != FMA_OK || (write_ ? k < (size_t)n_ || done_[k - n_] : ready_[k]); });
            failed = error_ != FMA_OK;
        }
        if (failed) return finish();
        char* win = window(k);
        if (direct_ && !write_) win += items_[k].file_off & 4095;   // the O_DIRECT read started at the block below the item
        RC(enqueue(win));
        RT(cudaEventRecord(e_->ev_load[k % n_], stream));
        std::lock_guard<std::mutex> lk(mu_);
        posted_[k] = 1;
        n_posted_ = std::max(n_posted_, k + 1);
        ++n_posted_items_;
        cv_.notify_all();
        return FMA_OK;
    }
    void worker();
    char* window(size_t k) const;      // where item k's I/O starts in its window (4 KiB aligned for O_DIRECT)
    void set_error(int code, const char* fmt, ...);
    int stop();                        // finish() without setting the thread's error message
    fma_engine_t* e_;
    int fd_;
    bool write_, direct_;
    std::vector<Item> items_;
    uint64_t file_bytes_;
    const char* path_;
    char* mem_;
    int n_;
    int item_delay_ms_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::vector<char> ready_, posted_, done_;   // read: item read; both: copy enqueued; write: pwrite returned
    size_t written_ = 0, n_posted_ = 0, n_posted_items_ = 0;   // n_posted_: 1 + the highest item posted
    std::atomic<size_t> next_{0};
    std::atomic<uint64_t> io_ns_{0};
    int error_ = FMA_OK;
    char msg_[512] = "";
    std::vector<std::thread> th_;
    bool stopped_ = false;
};

// The FILE tier's image file as one operation reads or writes it: a wake, a verify, a prefetch or a move out of the tier reads it;
// a file-tier sleep or a move into the tier writes it.  It owns the fd, whether that is O_DIRECT (when the filesystem accepts it
// and FMA_FILE_BUFFERED is not 1), the time it was opened and the operation's "file_io" timeline row: from the open to the end,
// idx 1 with O_DIRECT, over every byte read, or over the image and its descriptor written.  Failures to open: FMA_EIO.
class ImageFile {
  public:
    explicit ImageFile(fma_engine_t* e) : e_(e) {}
    // Reads `items` of `path`.  A file that ends before the furthest item does (truncated or replaced) is refused before a read
    // is issued; then *io's readers start (`mem`: see FileIO).
    int read(const std::string& path, std::vector<FileIO::Item> items, std::optional<FileIO>* io, char* mem = nullptr);
    // Opens `path` (created if need be) to write an image of `bytes`, and empties it only once its filesystem has room for the
    // image and its descriptor (fstatvfs).  Short of room, the file is left untouched.
    int create(const std::string& path, uint64_t bytes);
    void write(std::vector<FileIO::Item> items, std::optional<FileIO>* io, char* mem = nullptr, int item_delay_ms = 0);   // *io's writers of `items`
    // Read: every read has returned and every copy out of a window has finished (io.finish()), then the row.
    int finish(FileIO& io);
    // Write, after the last item: fdatasync, then the descriptor of the image sleeping in `tier`'s store (image_descriptor_build)
    // in the kImageTail bytes behind the image, then fdatasync again, so a torn file fails descriptor parsing; then the row.
    int seal(int tier);
    // The same with a descriptor built before, and no row: the write-behind job writes the file outside the operation lock and
    // records its row at the end (restart_clock: the row starts when its write does, after the sleep that created the file)
    int seal_with(const std::vector<char>& desc);
    void restart_clock() { t0_ = now_s(); }
    double started() const { return t0_; }
    bool direct() const { return direct_; }
    int fd() const { return file_.fd; }
    const std::string& path() const { return path_; }
    // The kImageTail bytes at the end of the image file `path` (opened into *f): *store_cap is what lies before them.  No engine.
    // Cannot open or read it: FMA_EIO; too short to hold a descriptor: `short_code`.
    static int read_tail(const char* path, int short_code, FileFd* f, size_t* store_cap, std::vector<char>* tail);
    // The "file_io" timeline row (idx 1 with O_DIRECT) of an I/O over [t0, t1): the write-behind job records its own at its end
    static void file_io_row(fma_engine_t* e, bool direct, double t0, double t1, uint64_t bytes);

  private:
    int row(uint64_t bytes);
    fma_engine_t* e_;
    std::string path_;
    FileFd file_;
    bool direct_ = false;
    double t0_ = 0;
    uint64_t bytes_ = 0;   // read: every item's; write: the image's
};

// ---- WRITE-BEHIND (fma_image.cu) ----
// Starts the job that writes the host-tier image a write-behind sleep just made to `file` (created and emptied by that sleep) and,
// once every byte and the descriptor are on disk, moves the image to the file tier (caller: that sleep, under op_mu).
void writeback_start(fma_engine_t* e, std::unique_ptr<ImageFile> file);
// A job still writing is cancelled and joined (caller holds op_mu): its file is emptied, its store stays the engine's host store,
// and the caller sees an ordinary host-tier image.  The time it took becomes a "wb_cancel" row.
void writeback_preempt(fma_engine_t* e);
void writeback_join(fma_engine_t* e);   // whatever the job's state, its thread has ended (the next job, fma_engine_destroy)

// One sleep / wake / swap / image or store operation per engine at a time, and a write-behind job still writing pre-empted first
struct OpLock {
    fma_engine_t* e;
    std::lock_guard<std::mutex> lk;
    explicit OpLock(fma_engine_t* eng) : e(eng), lk(eng->op_mu) { writeback_preempt(e); }
    ~OpLock() { e->tl_carry = false; }
};

// ---- pipelines ----
int do_sleep(fma_engine_t* e, uint64_t offload_mask, int tier, uint32_t flags);   // fma_sleep.cu
int do_wake(fma_engine_t* e, uint64_t tag_mask, uint32_t flags);                  // fma_wake.cu

// ------------------------------------------------------------------------------------
// packed image planning
// ------------------------------------------------------------------------------------
struct Extent {          // one segment's slice of the packed image
    size_t seg_index;
    CUdeviceptr va;
    size_t bytes;
    uint64_t packed_off;
};

size_t build_page_table(const std::vector<Extent>& ex, uint64_t* tab);

struct CopyTimer {  // device-time bracket over all engine streams
    fma_engine_t* e;
    int begin() {
        RT(cudaEventRecord(e->ev_start, e->ks));
        e->tl_dev_base = now_s() - e->tl_entry;
        for (int i = 0; i < e->n_cs; ++i) RT(cudaStreamWaitEvent(e->cs[i], e->ev_start, 0));
        return FMA_OK;
    }
    int end(double* seconds) {
        for (int i = 0; i < e->n_cs; ++i) {
            RT(cudaEventRecord(e->ev_cs[i], e->cs[i]));
            RT(cudaStreamWaitEvent(e->ks, e->ev_cs[i], 0));
        }
        RT(cudaEventRecord(e->ev_end, e->ks));
        RT(cudaEventSynchronize(e->ev_end));
        float ms = 0;
        RT(cudaEventElapsedTime(&ms, e->ev_start, e->ev_end));
        *seconds = ms * 1e-3;
        return FMA_OK;
    }
};

struct KernelTimes {  // event pairs around each K1/K2 launch on the kernel stream
    fma_engine_t* e;
    size_t used = 0;
    uint64_t bytes = 0;
    const char* kind = "kernel";   // timeline kind of the launches that follow
    int launch(const uint64_t* src_tab, uint64_t src_base, const uint64_t* dst_tab, uint64_t dst_base, uint32_t n_pages) {
        return launch_on(e->ks, src_tab, src_base, dst_tab, dst_base, n_pages);
    }
    // same on another stream of the engine's GPU (multi-path wake: one kernel stream per path; the caller serialises the calls)
    int launch_on(cudaStream_t stream, const uint64_t* src_tab, uint64_t src_base, const uint64_t* dst_tab, uint64_t dst_base, uint32_t n_pages) {
        int rc = ensure_event_pool(e, used + 2);
        if (rc != FMA_OK) return rc;
        RT(cudaEventRecord(e->ev_pool[used], stream));
        RT(fma_k_launch_page_copy(src_tab, src_base, dst_tab, dst_base, n_pages, e->cfg.kernel, &e->tma, stream));
        RT(cudaEventRecord(e->ev_pool[used + 1], stream));
        used += 2;
        bytes += 2ull * n_pages * FMA_PAGE_BYTES;
        e->tl_kbytes.push_back(2ull * n_pages * FMA_PAGE_BYTES);
        e->tl_kkind.push_back(kind);
        return FMA_OK;
    }
    // K4 / K5 (packed image): bracket a launch the caller makes itself; `b` = algorithmic bytes (read + write)
    int begin() {
        int rc = ensure_event_pool(e, used + 2);
        if (rc != FMA_OK) return rc;
        RT(cudaEventRecord(e->ev_pool[used], e->ks));
        return FMA_OK;
    }
    int end(uint64_t b) {
        RT(cudaEventRecord(e->ev_pool[used + 1], e->ks));
        used += 2;
        bytes += b;
        e->tl_kbytes.push_back(b);
        e->tl_kkind.push_back(kind);
        return FMA_OK;
    }
    // Called after the streams are synchronised.  Reading ~100s of event pairs costs ~1 ms, so it is
    // deferred to fma_stats() / the next operation instead of sitting inside the wake latency.
    int collect() {
        e->pending_events = used;
        e->pending_kernel_bytes = bytes;
        e->st.kernel_launches = (uint32_t)(used / 2);
        e->st.total_kernel_launches += used / 2;
        return FMA_OK;
    }
};

int flush_kernel_times(fma_engine_t* e);
int check_tma_shape(const fma_engine_t* e, int tier);
uint64_t store_dev_base(const fma_engine_t* e, int tier);
void* store_copy_base(const fma_engine_t* e, int tier);
int digest_segments(fma_engine_t* e, const std::vector<size_t>& idx, std::vector<uint64_t>* out);

static_assert(fma_layout::kPageBytes == FMA_PAGE_BYTES, "the layout planner's page is the engine's page");
using fma_layout::Batch;
using fma_layout::PagePlan;
// pages per launch of K1 / K2 / K4 / K5 when they read or write the store in place, counted even when the pages are packed
inline size_t slot_pages(const fma_engine_t* e) { return std::max<size_t>(staged_slot(e) / FMA_PAGE_BYTES, 1); }

// K4 / K5 descriptor of one page: a stored size of a whole page means the page is stored verbatim
inline void set_pack_desc(fma_k_pack_desc& d, uint64_t src, uint64_t dst, uint32_t stored_bytes) {
    d.src = src;
    d.dst = dst;
    d.mode = stored_bytes == FMA_PAGE_BYTES ? FMA_K_PACK_RAW : FMA_K_PACK_BF16;
    d.state = 0;
}
// Reads the K4 / K5 error counter d_psize[pdesc_cap] (synchronises the kernel stream); a non-zero count fails with
// FMA_EINTEGRITY and `fmt`, which takes the count as its one %u.
int check_pack_errors(fma_engine_t* e, const char* fmt);

// "Move these pages with a kernel", the same call for both page forms, so that a copy pipeline is written once: plain 2 MiB
// pages go through K1 / K2 and page tables, PACKED pages through K4 / K5 and descriptors.  One side of every page is its device
// address (PagePlan::va).  The other, the store side, is wherever the pipeline says: in the store itself, or in a ring slot.
struct PageKernels {
    fma_engine_t* e;
    KernelTimes& kt;
    bool to_store;   // a sleep: gather / code into the store side; else a wake: scatter / decode out of it
    bool packed;
    size_t at = 0;   // first entry of the engine's table and descriptor buffers to use (a RESIDENT share's sit behind the host part's)
    // Enqueues, on the kernel stream, the upload of what the launches over `pages` read: descriptors (PACKED), or the two page
    // tables of a wake.  store_addr(q) is the store side of page q.  clear_errors: zero the K4 / K5 error counter too (an
    // operation does that once, before its first PACKED launch).  A plain sleep has nothing to add: its table of device addresses
    // is the image's page table, which SleepPipe::plan uploads for every sleep pipeline, and its store side is always a base.
    template <class StoreAddr>
    int prepare(const std::vector<PagePlan>& pages, bool clear_errors, StoreAddr store_addr) {
        const size_t n = pages.size();
        if (packed) {
            RC(ensure_pack_bufs(e, at + n));
            for (size_t q = 0; q < n; ++q) {
                const uint64_t st = store_addr(q);
                set_pack_desc(e->h_pdesc[at + q], to_store ? pages[q].va : st, to_store ? st : pages[q].va, pages[q].bytes);
            }
            RT(cudaMemcpyAsync(e->d_pdesc + at, e->h_pdesc + at, n * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
            if (clear_errors) RT(cudaMemsetAsync(e->d_psize + e->pdesc_cap, 0, sizeof(uint32_t), e->ks));
        } else if (!to_store) {
            RC(ensure_tables(e, at + n));
            uint64_t* dev = e->h_tab + at;                  // destination page addresses
            uint64_t* st = e->h_tab + e->d_tab_cap + at;    // source page addresses (may be sparse in the store)
            for (size_t q = 0; q < n; ++q) {
                dev[q] = pages[q].va;
                st[q] = store_addr(q);
            }
            RT(cudaMemcpyAsync(e->d_tab + at, dev, n * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
            RT(cudaMemcpyAsync(e->d_tab + e->d_tab_cap + at, st, n * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
        }
        return FMA_OK;
    }
    // One launch over the pages of `b`, timed by `kt`.  Plain pages whose store side is contiguous take its address as
    // store_base; 0: their store side is the table `prepare` uploaded (a wake in place: a batch may span pages apart in the store).
    int launch(const Batch& b, uint64_t store_base = 0) {
        const size_t p = at + b.p0;
        if (!packed) {
            const uint64_t* dev = e->d_tab + p;
            const uint64_t* st = store_base ? nullptr : e->d_tab + e->d_tab_cap + p;
            return to_store ? kt.launch(dev, 0, st, store_base, (uint32_t)b.np) : kt.launch(st, store_base, dev, 0, (uint32_t)b.np);
        }
        uint32_t* d_err = e->d_psize + e->pdesc_cap;
        RC(kt.begin());
        if (to_store) RT(fma_k_launch_pack(e->d_pdesc + p, (uint32_t)b.np, d_err, e->ks));
        else RT(fma_k_launch_unpack(e->d_pdesc + p, (uint32_t)b.np, d_err, e->ks));
        return kt.end((uint64_t)b.np * FMA_PAGE_BYTES + b.stored);
    }
};

// The ring slots of a staged sleep or wake: runs of `pages` adjacent in the store that fit one slot, by their stored bytes (PACKED)
// or by their number.  Batch c of *slots goes through slot c % n_ring, and (*in_ring)[q] is where page q lies in it.
inline int plan_ring_slots(const fma_engine_t* e, bool packed, const std::vector<PagePlan>& pages, std::vector<Batch>* slots,
                           std::vector<uint64_t>* in_ring) {
    if (!fma_layout::plan_batches(pages, packed ? SIZE_MAX : e->ring_slot_bytes / FMA_PAGE_BYTES, packed ? e->ring_slot_bytes : UINT64_MAX, true, slots))
        return fail(FMA_EINVAL, "ring slot of %zu bytes cannot hold one page", e->ring_slot_bytes);
    in_ring->assign(pages.size(), 0);
    for (size_t c = 0; c < slots->size(); ++c) {
        const Batch& sl = (*slots)[c];
        for (size_t q = sl.p0; q < sl.p0 + sl.np; ++q)
            (*in_ring)[q] = (uint64_t)(uintptr_t)e->ring[c % e->n_ring] + (pages[q].off - pages[sl.p0].off);
    }
    return FMA_OK;
}

// What the workers of a MULTI-PATH sleep or wake share: one thread per path, and the first error wins.
struct PathWorkers {
    std::atomic<int> error{FMA_OK};
    char err_msg[512] = "";
    std::mutex kt_mu;                 // an operation has one KernelTimes: the paths' launches take turns
    std::vector<uint32_t> per_path;   // chunks each path moved
    void fail_once(int code, size_t pi, int device, const char* what, const char* why) {
        int expect = FMA_OK;
        if (error.compare_exchange_strong(expect, code)) snprintf(err_msg, sizeof(err_msg), "%s failed on path %zu (device %d): %s", what, pi, device, why);
    }
    // worker(pi) on a thread per path, on the engine's GPU and with the path's kernel stream behind ev_tab (the page table must be
    // on the device before any path's kernel reads it); returns when every worker has returned
    template <class Worker>
    void run(fma_engine_t* e, cudaEvent_t ev_tab, Worker worker) {
        per_path.assign(e->paths.size(), 0);
        std::vector<std::thread> th;
        for (size_t pi = 0; pi < e->paths.size(); ++pi)
            th.emplace_back([&, pi] {
                cudaSetDevice(e->device);
                const cudaError_t ce = cudaStreamWaitEvent(e->paths[pi].kern, ev_tab, 0);
                if (ce != cudaSuccess) return fail_once(FMA_ECUDA, pi, e->paths[pi].device, "cudaStreamWaitEvent(table)", cudaGetErrorString(ce));
                worker(pi);
            });
        for (auto& t : th) t.join();
    }
};

// No kernel ran in this operation: its kernel statistics read zero.
inline void zero_kernel_stats(fma_engine_t* e) {
    e->pending_events = 0;
    e->st.kernel_seconds = 0;
    e->st.kernel_bytes = 0;
    e->st.kernel_launches = 0;
}


}  // namespace fma_impl
