// fma_pull.cu — MULTI-PATH wake across processes (see fma_pull.h): the node-level owner's helper side and the instance's attach.
// Part of the host engine (C-ABI in include/fma_engine.h); no kernels here.
#include "fma_internal.h"

#include <deque>
#include <memory>

namespace {

struct HelperStaging {   // owner side: n_slots x slot_bytes in one helper GPU's HBM, exportable, mapped for that GPU
    int device = -1;
    size_t slot_bytes = 0;
    int slots = 0;
    VmmBuffer buf;
    cudaStream_t copy = nullptr;
    cudaEvent_t ev[kMaxRing] = {};
    std::atomic<int> users{0};          // pulls running on this staging buffer right now
    std::atomic<bool> closing{false};   // fma_helper_close is waiting for them: leave
};

struct AttachedStore {   // owner side: another process's memfd host store, mapped and pinned here too
    void* base = nullptr;
    size_t bytes = 0;
    std::atomic<int> users{0};
    std::atomic<bool> closing{false};
};

// A close / detach takes the object out of the table (no new pull finds it), raises `closing` and waits until the pulls that
// still use it have left; only then are the stream, the mapping and the pinned range torn down.
std::mutex g_mu;
std::map<uint64_t, std::shared_ptr<HelperStaging>> g_helpers;
std::map<uint64_t, std::shared_ptr<AttachedStore>> g_stores;
uint64_t g_next = 1;

PullMailbox* map_mailbox(int fd) {
    void* p = mmap(nullptr, sizeof(PullMailbox), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    return p == MAP_FAILED ? nullptr : static_cast<PullMailbox*>(p);
}

void nap() { std::this_thread::sleep_for(std::chrono::microseconds(20)); }

// what fma_helper_open made, whatever of it exists
void helper_free(HelperStaging& h) {
    DeviceGuard guard(h.device);
    if (h.copy) cudaStreamSynchronize(h.copy);
    if (h.copy) cudaStreamDestroy(h.copy);
    for (cudaEvent_t ev : h.ev)
        if (ev) cudaEventDestroy(ev);
    vmm_buffer_free(h.buf);
    cudaGetLastError();
}

}  // namespace

extern "C" {

// ---- owner side ---------------------------------------------------------------------------------------------------------
int fma_helper_open(int device, size_t slot_bytes, int slots, uint64_t* out_handle, int* out_fd) {
    if (!out_handle || !out_fd) return fail(FMA_EINVAL, "out pointers are NULL");
    if (!driver_ready()) return fail(FMA_ENODRIVER, "%s", g_drv_err);
    int ndev = 0;
    RT(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(FMA_EINVAL, "device %d not visible (have %d)", device, ndev);
    slot_bytes = round_up(slot_bytes ? slot_bytes : ((size_t)128 << 20), FMA_PAGE_BYTES);
    slots = slots > 0 ? std::min(slots, (int)kPullMaxSlots) : 3;
    DeviceGuard guard(device);
    RT(cudaFree(nullptr));
    auto hp = std::make_shared<HelperStaging>();
    HelperStaging& h = *hp;
    h.device = device;
    h.slot_bytes = slot_bytes;
    h.slots = slots;
    const size_t bytes = slot_bytes * (size_t)slots;
    char what[64];
    snprintf(what, sizeof(what), "helper staging on device %d", device);
    CUmemGenericAllocationHandle handle = 0;
    RC(vmm_create(device, bytes, true, &handle));
    RC(vmm_buffer_map(handle, bytes, {device}, what, &h.buf));
    int fd = -1;
    int rc = FMA_OK;
    const CUresult r = g_drv.MemExportToShareableHandle(&fd, h.buf.handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    if (r != CUDA_SUCCESS) rc = fail(FMA_ECUDA, "cuMemExportToShareableHandle(%s) failed: %s", what, cu_err(r));
    if (rc == FMA_OK && cudaStreamCreateWithFlags(&h.copy, cudaStreamNonBlocking) != cudaSuccess) rc = fail(FMA_ECUDA, "copy stream on helper device %d", device);
    for (int i = 0; i < slots && rc == FMA_OK; ++i)
        if (cudaEventCreateWithFlags(&h.ev[i], cudaEventDisableTiming) != cudaSuccess) rc = fail(FMA_ECUDA, "event on helper device %d", device);
    if (rc != FMA_OK) {
        helper_free(h);
        if (fd >= 0) close(fd);
        return rc;
    }
    std::lock_guard<std::mutex> lk(g_mu);
    *out_handle = g_next++;
    g_helpers[*out_handle] = hp;
    *out_fd = fd;
    return FMA_OK;
}

int fma_helper_close(uint64_t handle) {
    std::shared_ptr<HelperStaging> hp;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_helpers.find(handle);
        if (it == g_helpers.end()) return fail(FMA_ENOTFOUND, "unknown helper handle");
        hp = it->second;
        g_helpers.erase(it);
    }
    HelperStaging& h = *hp;
    h.closing.store(true);
    while (h.users.load() > 0) nap();   // a pull notices `closing` within one poll interval (or one chunk copy)
    helper_free(h);
    return FMA_OK;
}

int fma_store_attach(int fd, uint64_t* out_handle) {
    if (!out_handle) return fail(FMA_EINVAL, "out_handle is NULL");
    if (!driver_ready()) return fail(FMA_ENODRIVER, "%s", g_drv_err);
    struct stat sb;
    if (fstat(fd, &sb) != 0 || sb.st_size <= 0) return fail(FMA_EINVAL, "not a store fd");
    void* p = mmap(nullptr, (size_t)sb.st_size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (p == MAP_FAILED) return fail(FMA_ENOMEM, "cannot map the store: %s", strerror(errno));
    cudaError_t r = cudaHostRegister(p, (size_t)sb.st_size, cudaHostRegisterPortable);
    if (r != cudaSuccess) {
        cudaGetLastError();
        munmap(p, (size_t)sb.st_size);
        return fail(FMA_ENOMEM, "cannot pin the attached store: %s", cudaGetErrorString(r));
    }
    auto sp = std::make_shared<AttachedStore>();
    sp->base = p;
    sp->bytes = (size_t)sb.st_size;
    std::lock_guard<std::mutex> lk(g_mu);
    *out_handle = g_next++;
    g_stores[*out_handle] = sp;
    return FMA_OK;
}

int fma_store_detach(uint64_t handle) {
    std::shared_ptr<AttachedStore> sp;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_stores.find(handle);
        if (it == g_stores.end()) return fail(FMA_ENOTFOUND, "unknown store handle");
        sp = it->second;
        g_stores.erase(it);
    }
    sp->closing.store(true);
    while (sp->users.load() > 0) nap();
    cudaHostUnregister(sp->base);
    munmap(sp->base, sp->bytes);
    cudaGetLastError();
    return FMA_OK;
}

// Serve ONE wake on one path: wait until the instance has published the chunk table of `generation`, then pull chunks from the
// shared counter into this helper's staging slots — H2D by THIS GPU's copy engine over THIS GPU's link — and tell the instance, slot
// by slot, when a chunk has landed.  Blocking; returns when the path is done, the wake is aborted, or nothing moves for timeout_s.
int fma_helper_pull(uint64_t helper, uint64_t store, int mailbox_fd, int path_index, uint64_t generation, double timeout_s) {
    if (path_index < 1 || path_index >= (int)kPullMaxPaths) return fail(FMA_EINVAL, "path index %d", path_index);
    std::shared_ptr<HelperStaging> hp;
    std::shared_ptr<AttachedStore> sp;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto hi = g_helpers.find(helper);
        auto si = g_stores.find(store);
        if (hi == g_helpers.end() || si == g_stores.end()) return fail(FMA_ENOTFOUND, "unknown helper / store handle");
        hp = hi->second;
        sp = si->second;
        hp->users.fetch_add(1);   // under g_mu: a close that has already taken the object out of the table is never seen here
        sp->users.fetch_add(1);
    }
    struct Leave {
        HelperStaging& h; AttachedStore& s;
        ~Leave() { h.users.fetch_sub(1); s.users.fetch_sub(1); }
    } leave{*hp, *sp};
    HelperStaging& h = *hp;
    AttachedStore& st = *sp;
    auto closing = [&] { return h.closing.load() || st.closing.load(); };
    PullMailbox* mb = map_mailbox(mailbox_fd);
    if (!mb) return fail(FMA_ENOMEM, "cannot map the mailbox");
    int rc = FMA_OK;
    // The mailbox belongs to the instance's wake of `generation`.  Until this helper has CLAIMED its path in that wake, and again
    // as soon as the instance has moved on, it leaves quietly: it never writes a word of a wake it does not serve.
    bool serving = false;
    auto done = [&](int code) {
        if (code != FMA_OK && serving && mb->generation.load(std::memory_order_acquire) == generation) {
            mb->helper_error[path_index].store((uint32_t)(-code));
            mb->abort.store(1);
        }
        munmap(mb, sizeof(PullMailbox));
        return code;
    };
    if (mb->magic.load() != kPullMagic || mb->version != kPullVersion) return done(fail(FMA_EINVAL, "not a pull mailbox"));
    if ((int)mb->n_slots != h.slots || mb->slot_bytes != h.slot_bytes) return done(fail(FMA_EINVAL, "mailbox and staging disagree on the slot shape"));
    DeviceGuard guard(h.device);
    double t_last = now_s();
    for (;;) {   // the instance is still planning its wake
        const uint64_t g = mb->generation.load(std::memory_order_acquire);
        if (g == generation) break;
        if (g > generation) return done(fail(FMA_ESTATE, "generation %llu is over (the mailbox is at %llu)", (unsigned long long)generation, (unsigned long long)g));
        if (closing()) return done(fail(FMA_ESTATE, "the helper / the store is being closed"));
        if (now_s() - t_last > timeout_s) return done(fail(FMA_ESTATE, "the wake of generation %llu never started", (unsigned long long)generation));
        nap();
    }
    const uint32_t n = mb->n_chunks.load();
    std::atomic<uint32_t>* state = mb->slot_state[path_index];
    {   // "this path is being served": the instance waits for its done word.  One helper per path and wake: a repeated request loses here.
        uint64_t nobody = 0;
        if (!mb->helper_seen[path_index].compare_exchange_strong(nobody, generation, std::memory_order_acq_rel))
            return done(fail(FMA_ESTATE, "path %d of generation %llu is already served", path_index, (unsigned long long)generation));
    }
    serving = true;
    bool superseded = false;   // the instance has moved on to another wake
    // A word goes 0 -> value only.  The slot was free when its copy was issued; if a word of ANOTHER generation sits there now (a helper
    // left over from an aborted wake got in between), the instance clears it when it looks at the slot: wait for that.  1 = published,
    // 0 = the instance has moved on, < 0 = error.
    auto publish = [&](int slot, uint32_t value) -> int {
        const double t0 = now_s();
        for (;;) {
            uint32_t seen = 0;
            if (state[slot].compare_exchange_strong(seen, pull_word(generation, value), std::memory_order_acq_rel)) return 1;
            if (mb->generation.load(std::memory_order_acquire) != generation) return 0;
            if (pull_word_is_of(seen, generation)) return fail(FMA_ESTATE, "slot %d of path %d holds a word this helper did not write", slot, path_index);
            if (mb->abort.load() || closing() || now_s() - t0 > timeout_s) return fail(FMA_ESTATE, "slot %d of path %d never became free", slot, path_index);
            nap();
        }
    };
    struct Fly { int slot; uint32_t chunk; };
    std::deque<Fly> fly;
    uint32_t seq = 0;
    bool more = true;
    t_last = now_s();
    while (rc == FMA_OK) {
        if (mb->generation.load(std::memory_order_acquire) != generation) { superseded = true; rc = fail(FMA_ESTATE, "generation %llu is over", (unsigned long long)generation); break; }
        if (mb->abort.load()) { rc = fail(FMA_ESTATE, "the wake was aborted"); break; }
        if (closing()) { rc = fail(FMA_ESTATE, "the helper / the store is being closed"); break; }   // chunks this path took are lost: the wake fails and rolls back
        // publish copies that have landed (block on the oldest when nothing else can be done)
        bool progressed = false;
        while (!fly.empty()) {
            const bool must = (int)fly.size() == h.slots || !more;
            cudaError_t q = must ? cudaEventSynchronize(h.ev[fly.front().slot]) : cudaEventQuery(h.ev[fly.front().slot]);
            if (q == cudaErrorNotReady) { cudaGetLastError(); break; }
            if (q != cudaSuccess) { rc = fail(FMA_ECUDA, "H2D on helper device %d failed: %s", h.device, cudaGetErrorString(q)); break; }
            const int pub = mb->generation.load(std::memory_order_acquire) != generation ? 0 : publish(fly.front().slot, fly.front().chunk + 1);
            if (pub == 0) { superseded = true; rc = fail(FMA_ESTATE, "generation %llu is over", (unsigned long long)generation); }
            if (pub < 0) rc = pub;
            if (rc != FMA_OK) break;
            fly.pop_front();
            progressed = true;
        }
        if (rc != FMA_OK) break;
        if (!more && fly.empty()) break;
        if (more && (int)fly.size() < h.slots) {
            const int slot = (int)(seq % (uint32_t)h.slots);
            if (state[slot].load(std::memory_order_acquire) == 0) {   // the instance's K2 has drained what this slot held before
                const uint32_t c = mb->next_chunk.fetch_add(1);
                if (c >= n) {
                    more = false;
                } else {
                    const PullChunk ch = mb->chunks[c];
                    if (ch.store_off + ch.bytes > st.bytes || ch.bytes > h.slot_bytes) { rc = fail(FMA_EINVAL, "chunk %u is outside the store / larger than a slot", c); break; }
                    cudaError_t ce = cudaMemcpyAsync(reinterpret_cast<void*>(h.buf.va + (size_t)slot * h.slot_bytes), static_cast<char*>(st.base) + ch.store_off, ch.bytes,
                                                     cudaMemcpyDefault, h.copy);
                    if (ce == cudaSuccess) ce = cudaEventRecord(h.ev[slot], h.copy);
                    if (ce != cudaSuccess) { rc = fail(FMA_ECUDA, "H2D on helper device %d failed: %s", h.device, cudaGetErrorString(ce)); break; }
                    fly.push_back(Fly{slot, c});
                    ++seq;
                }
                progressed = true;
            }
        }
        if (progressed) {
            t_last = now_s();
        } else {
            if (now_s() - t_last > timeout_s) { rc = fail(FMA_ESTATE, "no progress for %.1f s on path %d", timeout_s, path_index); break; }
            nap();
        }
    }
    if (rc == FMA_OK) {   // tell the instance this path is finished: in the slot it will look at next, once that slot is free
        const int slot = (int)(seq % (uint32_t)h.slots);
        t_last = now_s();
        while (state[slot].load(std::memory_order_acquire) != 0) {
            if (mb->generation.load(std::memory_order_acquire) != generation) { superseded = true; rc = fail(FMA_ESTATE, "generation %llu is over", (unsigned long long)generation); break; }
            if (mb->abort.load() || closing() || now_s() - t_last > timeout_s) { rc = fail(FMA_ESTATE, "the instance never drained the last slot of path %d", path_index); break; }
            nap();
        }
        if (rc == FMA_OK && mb->generation.load(std::memory_order_acquire) == generation) {
            const int pub = publish(slot, kPullDoneValue);
            if (pub < 0) rc = pub;
        }
    }
    cudaStreamSynchronize(h.copy);
    if (superseded) serving = false;
    return done(rc);
}

// ---- instance side ------------------------------------------------------------------------------------------------------
// The owner's staging buffers (fds from fma_helper_open, one per helper GPU this process cannot see) become remote paths of a
// multi-path wake; *out_mailbox_fd is the mailbox to hand to the owner (it stays owned by the engine; dup it to keep it).
int fma_paths_attach(fma_engine_t* e, const int* staging_fds, int n, size_t slot_bytes, int slots, int* out_mailbox_fd) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (n < 1 || n > (int)kPullMaxPaths - 1 || !staging_fds || !out_mailbox_fd) return fail(FMA_EINVAL, "1..%d staging fds and an out pointer", (int)kPullMaxPaths - 1);
    if (slot_bytes == 0 || slot_bytes % FMA_PAGE_BYTES || slots < 1 || slots > (int)kPullMaxSlots) return fail(FMA_EINVAL, "attach needs the slot shape the owner created");
    OpLock op(e);
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    paths_release(e);
    e->path_slot_bytes = slot_bytes;
    e->path_slots = slots;
    const size_t bytes = slot_bytes * (size_t)slots;
    for (int i = -1; i < n; ++i) {   // i == -1: the engine's own link (a local path, as in fma_paths_set)
        e->paths.emplace_back();
        WakePath& p = e->paths.back();
        p.remote = i >= 0;
        if (!p.remote) {
            p.device = e->device;
            p.numa_node = gpu_numa_node(e->device);
        }
        char what[64];
        snprintf(what, sizeof(what), "staging buffer of path %d", i + 1);
        CUmemGenericAllocationHandle h = 0;
        int rc = p.remote ? vmm_import(staging_fds[i], &h) : vmm_create(e->device, bytes, false, &h);
        if (rc == FMA_OK) rc = vmm_buffer_map(h, bytes, {e->device}, what, &p.staging);
        if (rc == FMA_OK) rc = open_path(p, slots);
        if (rc != FMA_OK) return paths_fail(e, rc);
    }
    e->mbox_fd = (int)syscall(SYS_memfd_create, "fma-pull-mailbox", 1u);
    if (e->mbox_fd < 0 || ftruncate(e->mbox_fd, (off_t)sizeof(PullMailbox)) != 0)
        return paths_fail(e, fail(FMA_ENOMEM, "cannot create the mailbox: %s", strerror(errno)));
    if (!(e->mbox = map_mailbox(e->mbox_fd))) return paths_fail(e, fail(FMA_ENOMEM, "cannot map the mailbox"));
    PullMailbox* mb = e->mbox;   // a fresh memfd is zero-filled: atomics start at 0
    mb->version = kPullVersion;
    mb->n_slots = (uint32_t)slots;
    mb->slot_bytes = slot_bytes;
    mb->magic.store(kPullMagic, std::memory_order_release);
    e->pull_generation = 0;
    *out_mailbox_fd = e->mbox_fd;
    return FMA_OK;
}

// The generation the NEXT multi-path wake will publish (the owner's helpers wait for exactly that value).
uint64_t fma_pull_next_generation(fma_engine_t* e) { return e ? e->pull_generation + 1 : 0; }

// The memfd behind the host store (FMA_HOST_STORE_SHM=1) for the owner to fma_store_attach — unlike fma_image_export this does not
// make the store read-only: the owner only reads it while a wake pulls.  The caller closes the returned fd.
int fma_host_store_share(fma_engine_t* e, int* out_fd) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!out_fd) return fail(FMA_EINVAL, "out_fd is NULL");
    OpLock op(e);
    RC(refuse_resident_handover(e));
    if (e->image_tier == FMA_TIER_FILE && image_in(e, ImageIn::AnyAsleep)) return fail(FMA_ESTATE, "the sleeping image is in a file: the file itself is the hand-over");
    if (e->host.fd < 0 || !e->host.base) return fail(FMA_ESTATE, "the host store is not shareable (set FMA_HOST_STORE_SHM=1 before the first sleep / host_reserve)");
    const int fd = dup(e->host.fd);
    if (fd < 0) return fail(FMA_ENOMEM, "dup failed: %s", strerror(errno));
    e->host.fd_handed_out = true;
    *out_fd = fd;
    return FMA_OK;
}

}  // extern "C"
