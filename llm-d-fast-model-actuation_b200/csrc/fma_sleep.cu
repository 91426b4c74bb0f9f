// fma_sleep.cu — SLEEP: vllm:device_allocator/cumem.py:177-225 -> do_sleep (and the PACKED image plan)
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"
#include "fma_gate.h"

namespace fma_impl {

namespace {

// K4p over the pages of `ex`: the stored size of each lands in e->h_psize[0, n_pages).  pack_pages: descriptors to provide for.
int pack_probe(fma_engine_t* e, const std::vector<Extent>& ex, size_t n_pages, size_t pack_pages) {
    int rc = ensure_tables(e, n_pages);
    if (rc != FMA_OK) return rc;
    rc = ensure_pack_bufs(e, pack_pages);
    if (rc != FMA_OK) return rc;
    build_page_table(ex, e->h_tab);
    RT(cudaMemcpyAsync(e->d_tab, e->h_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    RT(fma_k_launch_pack_probe(e->d_tab, (uint32_t)n_pages, e->d_psize, e->ks));
    RT(cudaMemcpyAsync(e->h_psize, e->d_psize, n_pages * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->ks));
    RT(cudaStreamSynchronize(e->ks));
    e->st.total_kernel_launches += 1;
    return FMA_OK;
}

// K3 digests of the segments of `ex` become their recorded digests; *out (if given) receives them too, in `ex` order.
int digest_and_mark(fma_engine_t* e, const std::vector<Extent>& ex, std::vector<uint64_t>* out = nullptr) {
    std::vector<size_t> idx;
    for (const Extent& x : ex) idx.push_back(x.seg_index);
    std::vector<uint64_t> dg;
    int rc = digest_segments(e, idx, &dg);
    if (rc != FMA_OK) return rc;
    for (size_t k = 0; k < idx.size(); ++k) {
        e->segs[idx[k]].digest = dg[k];
        e->segs[idx[k]].digest_valid = true;
    }
    if (out) *out = std::move(dg);
    return FMA_OK;
}

const char* const kPackChanged = "%u page(s) changed between the pack probe and the pack: weights were written during sleep";

}  // namespace

// ------------------------------------------------------------------------------------
// PACKED host image: K4p over every page of the image, then the store layout on the host.
// Stored pages are laid back to back (sizes are multiples of 16 KiB), so every ring slot's D2H / H2D is one
// contiguous copy.  *packed = false when coding would save < 5 % (fp8 / int / already dense data): the caller then
// takes the plain path and the probe (one HBM read of the image, ~3 ms per 16 GiB) is all it cost.
// ------------------------------------------------------------------------------------
int plan_packed_image(fma_engine_t* e, const std::vector<Extent>& ex, uint64_t W, std::vector<uint64_t>* off,
                      std::vector<uint32_t>* bytes, uint64_t* stored_total, bool* packed) {
    *packed = false;
    *stored_total = W;
    const size_t n_pages = W / FMA_PAGE_BYTES;
    RT(cudaDeviceSynchronize());  // the caller's streams may still be writing weights (same reason as in do_sleep)
    int rc = pack_probe(e, ex, n_pages, n_pages);
    if (rc != FMA_OK) return rc;
    off->resize(n_pages);
    bytes->resize(n_pages);
    uint64_t total = 0;
    for (size_t p = 0; p < n_pages; ++p) {
        const uint32_t b = e->h_psize[p];
        if (b != FMA_K_PACKED_PAGE_BYTES && b != FMA_PAGE_BYTES) return fail(FMA_ECUDA, "pack probe returned size %u for page %zu", b, p);
        (*off)[p] = total;
        (*bytes)[p] = b;
        total += b;
    }
    if (total * 100 > W * 95) return FMA_OK;
    *stored_total = total;
    *packed = true;
    return FMA_OK;
}

namespace {

// ---- unmapper thread: cuMemUnmap runs UNDER the copy pipeline instead of after it -----------------------
// (cumem.py:213 unmaps each segment right after its blocking copy.)  The thread only issues driver calls on
// ranges planned here; the table is updated by this thread after it has been joined.  Adjacent units are
// unmapped with ONE spanning cuMemUnmap (allowed across whole mappings, scripts/vmm_span_probe.py).
struct Range {
    CUdeviceptr va;
    size_t bytes;
};
struct Stage {
    cudaEvent_t ev;
    std::vector<Range> ranges;
};
struct Unmapper {
    fma_engine_t* e;
    std::mutex mu;
    std::condition_variable cv;
    std::vector<Stage> stages;
    bool closed = false;
    int error = FMA_OK;
    char msg[512] = "";
    double seconds = 0;
    std::vector<Range> first;  // ranges with nothing to wait for (discarded tags)
    std::vector<Range> done;   // ranges actually unmapped
    std::thread th;
    void unmap_range(const Range& r, bool dbg) {
        double a;
        CUresult r1;
        {
            GateHold hold(kGateUnmap, 0.1);   // nothing waits for an unmap: yield (bounded) to calls that gate a wake's copies
            a = now_s();
            r1 = g_drv.MemUnmap(r.va, r.bytes);
        }
        const double b = now_s();
        seconds += b - a;
        e->tl_add("unmap", (int)done.size(), a, b, r.bytes);
        if (r1 != CUDA_SUCCESS) {
            std::lock_guard<std::mutex> lk(mu);
            if (error == FMA_OK) {
                error = FMA_ECUDA;
                snprintf(msg, sizeof(msg), "cuMemUnmap(%zu bytes) failed: %s", r.bytes, cu_err(r1));
            }
            return;
        }
        if (dbg && (b - a) > 5e-3)
            fprintf(stderr, "[fma] slow unmap va=0x%llx bytes=%zu unmap=%.1f ms\n", (unsigned long long)r.va, r.bytes, (b - a) * 1e3);
        done.push_back(r);
    }
    void run() {
        cudaSetDevice(e->device);
        const bool dbg = env_int("FMA_DEBUG_VMM", 0) != 0;
        for (const Range& r : first) unmap_range(r, dbg);
        size_t k = 0;
        for (;;) {
            Stage st;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return stages.size() > k || closed; });
                if (k >= stages.size()) break;
                st = stages[k];
            }
            cudaError_t r = cudaEventSynchronize(st.ev);
            if (r != cudaSuccess) {
                std::lock_guard<std::mutex> lk(mu);
                if (error == FMA_OK) {
                    error = FMA_ECUDA;
                    snprintf(msg, sizeof(msg), "cudaEventSynchronize(stage) failed: %s", cudaGetErrorString(r));
                }
                break;  // never unmap memory whose copy may not have finished
            }
            for (const Range& rg : st.ranges) unmap_range(rg, dbg);
            ++k;
        }
    }
    void publish(Stage&& st) {
        {
            std::lock_guard<std::mutex> lk(mu);
            stages.push_back(std::move(st));
        }
        cv.notify_all();
    }
    void finish() {
        {
            std::lock_guard<std::mutex> lk(mu);
            closed = true;
        }
        cv.notify_all();
        if (th.joinable()) th.join();
    }
    ~Unmapper() { finish(); }
};

// Whatever the unmapper really unmapped is applied to the table on EVERY exit path (also the error returns
// below), so that a failed sleep never leaves units the table believes mapped but the driver has released.
struct ApplyUnmapped {
    Unmapper* un;
    fma_engine_t* e;
    const std::vector<Extent>* ex;   // offloaded extents: a unit is only ever unmapped after its bytes reached the store,
    int tier;                        // so an unmapped offloaded segment HAS a backup even if the sleep fails later
    size_t applied = 0;
    void run() {
        std::lock_guard<std::mutex> lk(e->mu);
        for (; applied < un->done.size(); ++applied) {
            const Range& r = un->done[applied];
            auto it = e->units.lower_bound(r.va);
            while (it != e->units.end() && it->first < r.va + r.bytes) {
                Arena& a = e->arenas[it->second.arena];
                for (auto& z : it->second.zombies) arena_give_back(a, z.first - a.base, z.second);
                it = e->units.erase(it);
            }
            if (e->ring_attached && e->ring_unit_va >= r.va && e->ring_unit_va < r.va + r.bytes) {
                for (int i = 0; i < kMaxRing; ++i) e->ring[i] = nullptr;
                e->n_ring = 0; e->ring_slot_bytes = 0; e->ring_attached = false; e->ring_unit_va = 0;
            }
            for (Segment& sg : e->segs)
                if (sg.va >= r.va && sg.va < r.va + r.bytes) {
                    sg.mapped = false;
                    sg.unit_va = 0;
                }
            for (const Extent& x : *ex)
                if (x.va >= r.va && x.va < r.va + r.bytes) {
                    Segment& sg = e->segs[x.seg_index];
                    sg.has_backup = true;
                    sg.backup_tier = tier;
                    sg.packed_off = x.packed_off;
                }
        }
        if (!un->done.empty()) {  // even a failed sleep leaves an image a later wake can restore from
            e->image_tier = tier;
        }
    }
    ~ApplyUnmapped() {
        un->finish();
        run();
    }
};

// Units in VA order, split into "discarded" (release now) and "offloaded" (release once the image has their
// bytes).  image_end = packed offset just past the unit's last live segment.
struct PlannedUnit {
    CUdeviceptr va;
    size_t bytes;
    uint64_t image_end;
};

// What the copy pipelines of one sleep share.  Each pipeline enqueues the work that moves image[0, W) into the store
// and tells the unmapper, through publish_consumed(image_done, stream), which units are dead once `stream` gets there.
struct SleepPipe {
    fma_engine_t* e;
    const std::vector<Extent>& ex;
    uint64_t W;
    int tier;
    char* store;           // host pointer of the store (copy-engine target), or the parking buffer
    KernelTimes& kt;
    uint32_t& copy_ops;
    std::function<int(uint64_t, cudaStream_t)> publish_consumed;
    const std::vector<size_t>* subset = nullptr;  // INCREMENTAL + PACKED: only these image pages (ascending) are re-coded, in place
    bool resident = false;  // the extents go to the resident buffer (e->res, its own page layout res_off / res_bytes), not the tier's store
    int publish_gathered(size_t pages_done) { return publish_consumed((uint64_t)pages_done * FMA_PAGE_BYTES, e->ks); }
    // the image's pages, stored in the PACKED layout or verbatim; their device addresses in order -> e->h_tab / e->d_tab
    int plan(bool packed, std::vector<PagePlan>* pages) {
        std::vector<fma_layout::SegPages> segs;
        for (const Extent& x : ex) segs.push_back(fma_layout::SegPages{(uint64_t)x.va, x.bytes, x.packed_off, 0});
        const std::vector<uint64_t>& off = resident ? e->res_off : e->img_off;
        const std::vector<uint32_t>& bytes = resident ? e->res_bytes : e->img_bytes;
        uint64_t bad = 0;
        if (!fma_layout::plan_pages(segs, packed ? &off : nullptr, &bytes, pages, &bad))
            return fail(FMA_ESTATE, "image offset %llu is outside the packed image's page table", (unsigned long long)bad);
        int rc = ensure_tables(e, pages->size());
        if (rc != FMA_OK) return rc;
        build_page_table(ex, e->h_tab);
        RT(cudaMemcpyAsync(e->d_tab, e->h_tab, pages->size() * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
        return FMA_OK;
    }
    int direct();
    int kernel_packed();
    int kernel();
    int staged_packed();
    int staged();
    int multipath();
};

// DIRECT: copy engines move each segment chunk straight into the packed image
int SleepPipe::direct() {
    int rc = FMA_OK;
    const size_t chunk = direct_chunk(e);
    // copy engines straight from the segments into the packed image, chunks round-robin over the streams;
    // every `slot` bytes of image the streams are joined so that one event marks the units behind it dead
    const size_t slot = staged_slot(e);
    uint64_t next_join = slot;
    int k = 0;
    for (const Extent& x : ex) {
        for (size_t o = 0; o < x.bytes; o += chunk, ++k) {
            const size_t n = std::min(chunk, x.bytes - o);
            RT(cudaMemcpyAsync(store + x.packed_off + o, reinterpret_cast<void*>(x.va + o), n, cudaMemcpyDefault,
                               e->cs[k % e->n_cs]));
            ++copy_ops;
        }
        const uint64_t image_done = x.packed_off + x.bytes;
        if (image_done >= next_join || &x == &ex.back()) {
            for (int i = 1; i < e->n_cs; ++i) {  // stream 0 waits for the others
                RT(cudaEventRecord(e->ev_cs[i], e->cs[i]));
                RT(cudaStreamWaitEvent(e->cs[0], e->ev_cs[i], 0));
            }
            rc = publish_consumed(image_done, e->cs[0]);
            if (rc != FMA_OK) return rc;
            next_join = image_done + slot;
        }
    }
    return rc;
}

// KERNEL + PACKED (parking tiers): K4 encodes straight into the peer / local HBM store
int SleepPipe::kernel_packed() {
    std::vector<PagePlan> pages;
    int rc = plan(true, &pages);
    if (rc != FMA_OK) return rc;
    // PACKED image in a parking tier: K4 encodes straight into the peer / local HBM store (0.758 of the bytes
    // over NVLink and of the parking GPU's HBM), batches as below
    rc = ensure_pack_bufs(e, pages.size());
    if (rc != FMA_OK) return rc;
    const uint64_t dbase = resident ? (uint64_t)e->res.va : store_dev_base(e, tier);
    for (size_t p = 0; p < pages.size(); ++p) set_pack_desc(e->h_pdesc[p], pages[p].va, dbase + pages[p].off, pages[p].bytes);
    uint32_t* d_err = e->d_psize + e->pdesc_cap;
    RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, pages.size() * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemsetAsync(d_err, 0, sizeof(uint32_t), e->ks));
    std::vector<Batch> batches;
    fma_layout::plan_batches(pages, slot_pages(e), UINT64_MAX, false, &batches);
    for (const Batch& b : batches) {
        rc = kt.begin();
        if (rc != FMA_OK) return rc;
        RT(fma_k_launch_pack(e->d_pdesc + b.p0, (uint32_t)b.np, d_err, e->ks));
        rc = kt.end((uint64_t)b.np * FMA_PAGE_BYTES + b.stored);
        if (rc != FMA_OK) return rc;
        ++copy_ops;
        rc = publish_gathered(b.p0 + b.np);
        if (rc != FMA_OK) return rc;
    }
    return rc;
}

// KERNEL: K1 writes the store itself (mapped pinned host memory, peer or local HBM)
int SleepPipe::kernel() {
    std::vector<PagePlan> pages;
    int rc = plan(false, &pages);
    if (rc != FMA_OK) return rc;
    // K1 writes the store itself: mapped pinned host memory (PCIe posted writes) or peer/local HBM;
    // launched in slot-sized batches so finished segments can be released while later ones still move
    const uint64_t dbase = resident ? (uint64_t)e->res.va : store_dev_base(e, tier);
    std::vector<Batch> batches;
    fma_layout::plan_batches(pages, slot_pages(e), UINT64_MAX, false, &batches);
    for (const Batch& b : batches) {
        rc = kt.launch(e->d_tab + b.p0, 0, nullptr, dbase + pages[b.p0].off, (uint32_t)b.np);
        if (rc != FMA_OK) return rc;
        ++copy_ops;
        rc = publish_gathered(b.p0 + b.np);
        if (rc != FMA_OK) return rc;
    }
    return rc;
}

// STAGED + PACKED: K4 gather + encode -> ring slot (stored pages back to back) -> one D2H per slot
int SleepPipe::staged_packed() {
    std::vector<PagePlan> pages;
    int rc = plan(true, &pages);
    if (rc != FMA_OK) return rc;
    rc = ensure_ring(e, W);
    if (rc != FMA_OK) return rc;
    // the image pages this sleep codes: all of them, or (incremental) the pages of the changed segments, whose stored size
    // is known not to change, so each goes back to its old place in the kept image
    std::vector<size_t> img_page(pages.size());
    for (size_t p = 0; p < pages.size(); ++p) img_page[p] = p;
    if (subset) {
        img_page = *subset;
        std::vector<PagePlan> sel;
        for (size_t p : img_page) sel.push_back(pages[p]);
        pages = std::move(sel);
    }
    std::vector<Batch> slots;  // pages adjacent in the store that together fit a ring slot
    if (!fma_layout::plan_batches(pages, SIZE_MAX, e->ring_slot_bytes, true, &slots))
        return fail(FMA_EINVAL, "ring slot of %zu bytes cannot hold one page", e->ring_slot_bytes);
    for (size_t c = 0; c < slots.size(); ++c)
        for (size_t k = slots[c].p0; k < slots[c].p0 + slots[c].np; ++k)
            set_pack_desc(e->h_pdesc[k], pages[k].va, (uint64_t)(uintptr_t)e->ring[c % e->n_ring] + (pages[k].off - pages[slots[c].p0].off), pages[k].bytes);
    uint32_t* d_err = e->d_psize + e->pdesc_cap;
    RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, pages.size() * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemsetAsync(d_err, 0, sizeof(uint32_t), e->ks));
    cudaStream_t last_stream = e->cs[0];
    for (size_t c = 0; c < slots.size(); ++c) {
        const Batch& sl = slots[c];
        const int slot = (int)(c % e->n_ring);
        cudaStream_t cstream = e->cs[c % e->n_cs];
        if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(e->ks, e->ev_ring_free[slot], 0));
        rc = kt.begin();
        if (rc != FMA_OK) return rc;
        RT(fma_k_launch_pack(e->d_pdesc + sl.p0, (uint32_t)sl.np, d_err, e->ks));
        rc = kt.end((uint64_t)sl.np * FMA_PAGE_BYTES + sl.stored);
        if (rc != FMA_OK) return rc;
        RT(cudaEventRecord(e->ev_ring_full[slot], e->ks));
        RT(cudaStreamWaitEvent(cstream, e->ev_ring_full[slot], 0));
        RT(cudaMemcpyAsync(store + pages[sl.p0].off, e->ring[slot], sl.stored, cudaMemcpyDefault, cstream));
        if (c > 0) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[(c - 1) % e->n_ring], 0));  // same chaining as below
        RT(cudaEventRecord(e->ev_ring_free[slot], cstream));
        ++copy_ops;
        // every image byte below the last page of this slot is in the store: coded just now, or kept from the last wake
        rc = publish_consumed((uint64_t)(img_page[sl.p0 + sl.np - 1] + 1) * FMA_PAGE_BYTES, cstream);
        if (rc != FMA_OK) return rc;
        last_stream = cstream;
    }
    if (subset) rc = publish_consumed(W, last_stream);  // the clean tail of the image needs no copy
    return rc;
}

// STAGED: K1 gather -> HBM ring slot -> one large D2H per slot
int SleepPipe::staged() {
    std::vector<PagePlan> pages;
    int rc = plan(false, &pages);
    if (rc != FMA_OK) return rc;
    rc = ensure_ring(e, W);
    if (rc != FMA_OK) return rc;
    std::vector<Batch> slots;
    if (!fma_layout::plan_batches(pages, e->ring_slot_bytes / FMA_PAGE_BYTES, UINT64_MAX, true, &slots))
        return fail(FMA_EINVAL, "ring slot of %zu bytes cannot hold one page", e->ring_slot_bytes);
    for (size_t c = 0; c < slots.size(); ++c) {
        const Batch& sl = slots[c];
        const int slot = (int)(c % e->n_ring);
        cudaStream_t cstream = e->cs[c % e->n_cs];
        if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(e->ks, e->ev_ring_free[slot], 0));
        rc = kt.launch(e->d_tab + sl.p0, 0, nullptr, (uint64_t)(uintptr_t)e->ring[slot], (uint32_t)sl.np);
        if (rc != FMA_OK) return rc;
        RT(cudaEventRecord(e->ev_ring_full[slot], e->ks));
        RT(cudaStreamWaitEvent(cstream, e->ev_ring_full[slot], 0));
        RT(cudaMemcpyAsync(store + pages[sl.p0].off, e->ring[slot], sl.stored, cudaMemcpyDefault, cstream));
        // "slot free" also means "every earlier slot has reached the store" (chained through the previous
        // slot's event), so the unmapper below never releases device memory whose bytes are not yet on the host
        if (c > 0) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[(c - 1) % e->n_ring], 0));
        RT(cudaEventRecord(e->ev_ring_free[slot], cstream));
        ++copy_ops;
        rc = publish_consumed((uint64_t)(sl.p0 + sl.np) * FMA_PAGE_BYTES, cstream);  // units fully in the store are dead
        if (rc != FMA_OK) return rc;
    }
    return rc;
}

// MULTI-PATH sleep (fma_paths_set): the mirror image of the multi-path wake.  K1 on the sleeping GPU gathers a chunk of the image
// into a staging slot of a PATH — its own HBM, or a helper GPU's HBM over NVLink — and THAT GPU's copy engine moves the slot into
// the host store over THAT GPU's x16 link; chunk queues per NUMA node of the (striped) store, self-balancing.  Nothing is unmapped
// before every byte has reached the store (one publish at the end), so a failure half way leaves the engine awake and intact.
int SleepPipe::multipath() {
    std::vector<PagePlan> pages;
    int rc = plan(false, &pages);
    if (rc != FMA_OK) return rc;
    rc = ensure_ring_events(e, 1);
    if (rc != FMA_OK) return rc;
    cudaEvent_t ev_tab = e->ev_ring_full[0];
    RT(cudaEventRecord(ev_tab, e->ks));
    std::vector<Batch> chunks;
    fma_layout::plan_batches(pages, std::max<size_t>(e->path_slot_bytes / FMA_PAGE_BYTES, 1), UINT64_MAX, true, &chunks);
    std::vector<uint64_t> chunk_off;
    for (const Batch& ch : chunks) chunk_off.push_back(pages[ch.p0].off);
    fma_layout::ChunkQueues queues(chunk_off, e->host.ranges);
    std::atomic<int> error{FMA_OK};
    std::mutex kt_mu;
    char err_msg[512] = "";
    std::vector<uint32_t> per_path(e->paths.size(), 0);
    auto worker = [&](size_t pi) {
        WakePath& path = e->paths[pi];
        cudaSetDevice(e->device);
        auto failw = [&](int code, const char* what, cudaError_t ce) {
            int expect = FMA_OK;
            if (error.compare_exchange_strong(expect, code)) snprintf(err_msg, sizeof(err_msg), "%s failed on path %zu (device %d): %s", what, pi, path.device, cudaGetErrorString(ce));
        };
        cudaError_t ce = cudaStreamWaitEvent(path.kern, ev_tab, 0);
        if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaStreamWaitEvent(table)", ce);
        uint32_t mine = 0;
        for (;;) {
            if (error.load() != FMA_OK) return;
            size_t c = 0;
            if (!queues.take(path.numa_node, &c)) break;
            const Batch& ch = chunks[c];
            const int slot = (int)(mine % (uint32_t)e->path_slots);
            if (mine >= (uint32_t)e->path_slots) {   // the D2H that used this slot before has drained it (event on the path's GPU)
                ce = cudaEventSynchronize(path.ev_full[slot]);
                if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventSynchronize(slot drained)", ce);
            }
            char* slot_ptr = reinterpret_cast<char*>(path.va) + (size_t)slot * e->path_slot_bytes;
            {
                std::lock_guard<std::mutex> lk(kt_mu);
                const int krc = kt.launch_on(path.kern, e->d_tab + ch.p0, 0, nullptr, (uint64_t)(uintptr_t)slot_ptr, (uint32_t)ch.np);   // K1: gather -> slot
                if (krc != FMA_OK) return failw(krc, "K1 launch", cudaGetLastError());
            }
            ce = cudaEventRecord(path.ev_free[slot], path.kern);           // (event on the engine's GPU) the slot is full
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot full)", ce);
            ce = cudaStreamWaitEvent(path.copy, path.ev_free[slot], 0);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaStreamWaitEvent(slot full)", ce);
            ce = cudaMemcpyAsync(store + chunk_off[c], slot_ptr, ch.stored, cudaMemcpyDefault, path.copy);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaMemcpyAsync(D2H)", ce);
            ce = cudaEventRecord(path.ev_full[slot], path.copy);           // (event on the path's GPU) the slot is drained
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot drained)", ce);
            ++mine;
        }
        per_path[pi] = mine;
    };
    std::vector<std::thread> th;
    for (size_t pi = 0; pi < e->paths.size(); ++pi) th.emplace_back(worker, pi);
    for (auto& t : th) t.join();
    for (WakePath& path : e->paths) {   // every D2H has landed before anything is released (and before an error is reported)
        cudaError_t ce = cudaStreamSynchronize(path.copy);
        if (ce != cudaSuccess && error.load() == FMA_OK) {
            error.store(FMA_ECUDA);
            snprintf(err_msg, sizeof(err_msg), "D2H on path device %d failed: %s", path.device, cudaGetErrorString(ce));
        }
    }
    if (error.load() != FMA_OK) return fail(error.load(), "%s", err_msg);
    for (size_t pi = 0; pi < e->paths.size(); ++pi) {
        copy_ops += per_path[pi];
        e->tl_add("path_chunks", e->paths[pi].device, e->tl_entry, now_s(), (uint64_t)per_path[pi] * e->path_slot_bytes);
    }
    return publish_consumed(W, e->ks);   // all bytes are in the store: every offloaded unit may go
}

}  // namespace

// ------------------------------------------------------------------------------------
// SLEEP
// ------------------------------------------------------------------------------------
int do_sleep(fma_engine_t* e, uint64_t offload_mask, int tier, uint32_t flags) {
    DeviceGuard guard(e->device);
    int rc = flush_kernel_times(e);
    if (rc != FMA_OK) return rc;
    const double t_entry = now_s();
    rc = ensure_streams(e);
    if (rc != FMA_OK) return rc;

    // Executor.sleep is a no-op while sleeping (abstract.py:323-325)
    bool any_unmapped = false, any_mapped = false;
    for (const Segment& s : e->segs) (s.mapped ? any_mapped : any_unmapped) = true;
    if (any_unmapped || !any_mapped) return FMA_OK;
    rc = check_tma_shape(e, tier);
    if (rc != FMA_OK) return rc;
    e->tl_begin("sleep", t_entry);
    if (e->res.va) {  // a resident buffer kept by an FMA_FLAG_KEEP_BACKUP wake: this sleep gathers its resident part afresh
        RT(cudaDeviceSynchronize());
        GateHold hold(kGateUnmap, 0.1);
        resident_release(e);
    }

    // plan: offloaded segments -> packed image, in (arena, VA) order.  Arenas are bump-allocated per tag, so this is
    // allocation order (the reference's dict order, cumem.py:198) unless a freed hole was reused.
    std::vector<size_t> by_addr(e->segs.size());
    for (size_t i = 0; i < by_addr.size(); ++i) by_addr[i] = i;
    std::sort(by_addr.begin(), by_addr.end(), [&](size_t a, size_t b) {
        const Segment &x = e->segs[a], &y = e->segs[b];
        return x.arena != y.arena ? x.arena < y.arena : x.va < y.va;
    });
    std::vector<Extent> ex;
    uint64_t W = 0, discarded = 0;
    // the store that would hold the kept image: the host store, or the parking buffer of the same (peer / local) tier
    const bool kept_store = tier == FMA_TIER_HOST ? e->host.base != nullptr
                                                  : (e->park.va != 0 && (tier == FMA_TIER_LOCAL ? e->park.device == e->device : e->park.device != e->device));
    bool shadows_match = e->incremental && tier == e->shadow_tier && !(flags & kFlagAdopt) && kept_store;
    std::vector<uint64_t> shadow_digest;  // digest of the copy the store holds, per extent
    std::vector<uint64_t> shadow_at;      // where the store holds it (kNoOffset: no usable copy)
    for (size_t i : by_addr) {
        Segment& s = e->segs[i];
        if (tag_bit_set(offload_mask, s.tag)) {
            shadows_match = shadows_match && s.digest_valid && s.shadow_off == W;  // same bytes expected at the same image offset
            shadow_digest.push_back(s.digest);
            shadow_at.push_back(s.digest_valid ? s.shadow_off : kNoOffset);
            ex.push_back(Extent{i, s.va, s.bytes, W});
            W += s.bytes;
        } else {
            discarded += s.bytes;
        }
        s.has_backup = false;
        s.packed_off = kNoOffset;
        s.digest_valid = false;
    }
    // RESIDENT share (option "resident_bytes"): the tail of the image stays in one VMM allocation on this GPU.  Walking the
    // offloaded segments from the last to the first, a segment stays if its stored size (2 MiB pages, or its pages' PACKED sizes)
    // still fits what is left of the cap; the host store then holds only the other segments, back to back in image order.
    std::vector<Extent> ex_res;       // resident extents, packed_off = offset in the resident part
    uint64_t W_all = W;
    std::vector<uint64_t> res_seqs;
    bool pre_planned = false, pre_packed = false;  // the PACKED plan of the host part, made here already (K4p over the whole image)
    std::vector<uint64_t> pre_off;
    std::vector<uint32_t> pre_bytes;
    uint64_t pre_total = 0;
    if (e->resident_cap && tier == FMA_TIER_HOST && e->paths.empty() && !(flags & kFlagAdopt) && W) {
        if (e->cfg.pack && resolve_mode(e, tier) == FMA_MODE_STAGED) {
            rc = plan_packed_image(e, ex, W, &pre_off, &pre_bytes, &pre_total, &pre_packed);
            if (rc != FMA_OK) return rc;
            pre_planned = true;
        }
        std::vector<uint64_t> stored(ex.size());
        for (size_t k = 0; k < ex.size(); ++k) {
            stored[k] = pre_packed ? 0 : ex[k].bytes;
            if (pre_packed)
                for (uint64_t o = 0; o < ex[k].bytes; o += FMA_PAGE_BYTES) stored[k] += pre_bytes[(ex[k].packed_off + o) / FMA_PAGE_BYTES];
        }
        const std::vector<char> res = fma_layout::resident_split(stored, e->resident_cap);
        uint64_t res_stored = 0;
        for (size_t k = 0; k < ex.size(); ++k) res_stored += res[k] ? stored[k] : 0;
        if (res_stored) {
            ParkStore buf;
            const double a = now_s();
            int arc;
            {
                GateHold hold(kGateUnmap, 0.1);   // an allocation of a sleep: as patient as the sleep's unmaps
                arc = park_store_create(e, e->device, res_stored, &buf);
            }
            const double b = now_s();
            if (arc != FMA_OK) {  // HBM too full: a plain host-tier sleep of everything
                e->tl_add("res_fallback", 0, a, b, res_stored);
                cudaGetLastError();
            } else {
                e->tl_add("res_alloc", 0, a, b, buf.cap);
                std::vector<Extent> ex_host;
                std::vector<uint64_t> h_off, r_off, h_digest;
                std::vector<uint32_t> h_bytes, r_bytes;
                uint64_t Wh = 0, Wr = 0, hs = 0, rs = 0;
                bool host_shadows = true;
                for (size_t k = 0; k < ex.size(); ++k) {
                    Extent x = ex[k];
                    const uint64_t p0 = x.packed_off / FMA_PAGE_BYTES;
                    if (res[k]) {
                        x.packed_off = Wr;
                        Wr += x.bytes;
                        ex_res.push_back(x);
                        res_seqs.push_back(e->segs[x.seg_index].seq);
                    } else {
                        x.packed_off = Wh;
                        Wh += x.bytes;
                        ex_host.push_back(x);
                        host_shadows = host_shadows && shadow_at[k] == x.packed_off;
                        h_digest.push_back(shadow_digest[k]);
                    }
                    if (pre_packed)
                        for (uint64_t p = p0; p < p0 + x.bytes / FMA_PAGE_BYTES; ++p) {
                            (res[k] ? r_off : h_off).push_back(res[k] ? rs : hs);
                            (res[k] ? r_bytes : h_bytes).push_back(pre_bytes[p]);
                            (res[k] ? rs : hs) += pre_bytes[p];
                        }
                }
                e->res = buf;
                e->res_packed = pre_packed;
                e->res_off = std::move(r_off);
                e->res_bytes = std::move(r_bytes);
                e->res_store_bytes = res_stored;
                ex = std::move(ex_host);
                W = Wh;
                shadows_match = e->incremental && tier == e->shadow_tier && kept_store && host_shadows;
                shadow_digest = std::move(h_digest);
                if (pre_packed) {
                    pre_off = std::move(h_off);
                    pre_bytes = std::move(h_bytes);
                    pre_total = hs;
                } else {
                    pre_total = Wh;
                }
            }
        }
    }
    shadows_match = shadows_match && res_seqs == e->res_seqs;  // INCREMENTAL: a different split is a full sleep
    e->res_seqs = res_seqs;
    // INCREMENTAL sleep: does the host store still hold exactly this image?  One K3 pass over the device copy decides.
    bool clean = false, partial = false, partial_packed = false, digests_known = false;
    std::vector<Extent> dirty;        // segments whose device bytes differ from the copy in the store
    std::vector<size_t> dirty_pages;  // their image pages (PACKED image)
    if (shadows_match && W && W == e->shadow_image_bytes && (tier == FMA_TIER_HOST ? e->host.cap : e->park.cap) >= e->shadow_store_bytes) {
        RT(cudaDeviceSynchronize());  // the caller's streams may still be writing weights
        std::vector<uint64_t> now;
        rc = digest_and_mark(e, ex, &now);  // either way these are the digests of what sleeps now
        if (rc != FMA_OK) return rc;
        uint64_t dirty_bytes = 0;
        for (size_t k = 0; k < ex.size(); ++k)
            if (now[k] != shadow_digest[k]) {
                dirty.push_back(ex[k]);
                dirty_bytes += ex[k].bytes;
            }
        digests_known = true;
        clean = dirty.empty();
        // a few changed segments (an adapter, fp8 KV scales reset after wake, one synced layer): only they cross the link, into
        // their old place in the kept image (partial sleeps are a host-tier refinement; in a parking tier a changed image is
        // simply parked again)
        partial = tier == FMA_TIER_HOST && !clean && !e->shadow_packed && 2 * dirty_bytes <= W && !e->host.shared;  // a shared image is read-only
        // PACKED image: a changed page can go back to its old place only if its stored size stays what it was (K4p on those pages)
        if (tier == FMA_TIER_HOST && !clean && e->shadow_packed && e->cfg.pack && 2 * dirty_bytes <= W && !e->host.shared && resolve_mode(e, tier) == FMA_MODE_STAGED) {
            for (const Extent& x : dirty)
                for (size_t o = 0; o < x.bytes; o += FMA_PAGE_BYTES) dirty_pages.push_back((size_t)((x.packed_off + o) / FMA_PAGE_BYTES));
            rc = pack_probe(e, dirty, dirty_pages.size(), std::max<size_t>(dirty_pages.size(), W / FMA_PAGE_BYTES));
            if (rc != FMA_OK) return rc;
            partial_packed = dirty_pages.size() <= e->img_bytes.size();
            for (size_t q = 0; q < dirty_pages.size() && partial_packed; ++q)
                partial_packed = dirty_pages[q] < e->img_bytes.size() && e->h_psize[q] == e->img_bytes[dirty_pages[q]];
            if (partial_packed && (no_ring() || ensure_ring(e, W) != FMA_OK)) partial_packed = false;  // no HBM for a ring: full sleep through the plain path
        }
    }
    if (clean) flags |= kFlagAdopt;                  // release the device side only: not a byte moves
    else if (!partial && !partial_packed) invalidate_shadows(e);  // this sleep rewrites the store (or leaves the host tier alone: be conservative)
    int mode = partial ? FMA_MODE_DIRECT : resolve_mode(e, tier);
    // MULTI-PATH (fma_paths_set): a full, plain host-tier sleep is striped over the paths' links; every path has its own staging slots
    const bool multipath = !e->paths.empty() && !e->mbox && tier == FMA_TIER_HOST && mode == FMA_MODE_STAGED && !partial && !partial_packed && !clean &&
                           !(flags & kFlagAdopt) && !e->cfg.pack && env_int("FMA_MULTIPATH_SLEEP", 1) != 0;
    if (W && !(flags & kFlagAdopt) && mode == FMA_MODE_STAGED && !multipath && (no_ring() || ensure_ring(e, W) != FMA_OK)) mode = FMA_MODE_DIRECT;  // HBM too full for a ring
    // PACKED image (config.pack): decide per page what its stored form is BEFORE the store is sized
    bool packed = false;
    uint64_t Wp = W;
    if (clean || partial_packed) {  // the image in the store, its form and its page table stay as they are
        packed = e->shadow_packed;
        Wp = e->shadow_store_bytes;
        e->image_packed = packed;
        e->image_store_bytes = Wp;
        e->image_bytes = W;
    } else {
        std::vector<uint64_t> pk_off;
        std::vector<uint32_t> pk_bytes;
        // host tier: through the staging ring (STAGED); parking tiers (peer / local HBM): K4 writes the store itself (KERNEL)
        const bool pack_path = (tier == FMA_TIER_HOST && mode == FMA_MODE_STAGED) || (tier != FMA_TIER_HOST && mode == FMA_MODE_KERNEL);
        if (W && e->cfg.pack && !(flags & kFlagAdopt) && pack_path) {
            if (pre_planned) {
                pk_off = std::move(pre_off);
                pk_bytes = std::move(pre_bytes);
                Wp = pre_total;
                packed = pre_packed;
            } else {
                rc = plan_packed_image(e, ex, W, &pk_off, &pk_bytes, &Wp, &packed);
                if (rc != FMA_OK) return rc;
            }
        }
        e->image_packed = packed;
        e->image_store_bytes = Wp;
        e->img_off = packed ? std::move(pk_off) : std::vector<uint64_t>();
        e->img_bytes = packed ? std::move(pk_bytes) : std::vector<uint32_t>();
        if (packed) e->image_bytes = W;  // the layout above is indexed by image page: valid from here on, also if the sleep fails
    }
    if (W) {
        if (tier == FMA_TIER_HOST && (flags & kFlagAdopt)) {
            if (!e->host.base) return fail(FMA_ESTATE, "adopt without a store");  // the adopted store IS the image: never re-sized
        } else if (tier == FMA_TIER_HOST) {
            if (e->host.shared) {  // this sleep writes: leave the shared image to its other holders and take a private store
                invalidate_shadows(e);
                host_store_free(e->host);
            }
            rc = host_store_reserve(e, Wp);
            if (rc != FMA_OK) return rc;
            if (mode == FMA_MODE_KERNEL && !e->host.dev_alias) return fail(FMA_ECUDA, "host store has no device alias for zero-copy mode");
        } else if (tier == FMA_TIER_PEER) {
            if (!e->park.va || e->park.cap < Wp || e->park.device == e->device)
                return fail(FMA_ESTATE, "peer tier needs fma_peer_reserve(peer_device, >= %llu bytes) first", (unsigned long long)Wp);
        } else if (tier == FMA_TIER_LOCAL) {
            rc = park_reserve(e, e->device, Wp);
            if (rc != FMA_OK) return rc;
        } else {
            return fail(FMA_EINVAL, "unknown tier %d", tier);
        }
    }

    // The caller's own streams may still be writing weights: drain the device once, as the
    // reference's blocking cudaMemcpy on the legacy stream implicitly does (before anything reads the segments).
    RT(cudaDeviceSynchronize());

    const bool adopt = (flags & kFlagAdopt) != 0;  // the store already holds the image: release the device side only
    if (((flags & FMA_FLAG_VERIFY) || e->incremental) && W && !adopt && !digests_known) {  // incremental: digests seed the next sleep's check
        rc = digest_and_mark(e, ex);
        if (rc != FMA_OK) return rc;
    }

    // ---- RESIDENT share: K1 / K4 gather the resident segments into e->res (HBM only, a few ms), ahead of the host part's
    // pipeline on the kernel stream.  Synchronised before the host part starts: it rewrites the page tables, and the units
    // that hold only resident segments are unmapped right away below.
    CopyTimer timer{e};
    KernelTimes kt{e};
    uint32_t copy_ops = 0;
    double copy_s = 0;
    if (!ex_res.empty()) {
        if ((flags & FMA_FLAG_VERIFY) || e->incremental) {
            rc = digest_and_mark(e, ex_res);
            if (rc != FMA_OK) return rc;
        }
        rc = timer.begin();
        if (rc != FMA_OK) return rc;
        uint32_t res_launches = 0;
        SleepPipe rp{e, ex_res, W_all - W, FMA_TIER_LOCAL, nullptr, kt, res_launches, [](uint64_t, cudaStream_t) { return FMA_OK; }};
        rp.resident = true;
        kt.kind = "res_gather";
        rc = e->res_packed ? rp.kernel_packed() : rp.kernel();
        kt.kind = "kernel";
        if (rc != FMA_OK) return rc;
        if (e->res_packed) rc = check_pack_errors(e, kPackChanged);
        else RT(cudaStreamSynchronize(e->ks));
        if (rc != FMA_OK) return rc;
        std::lock_guard<std::mutex> lk(e->mu);
        for (const Extent& x : ex_res) {
            Segment& sg = e->segs[x.seg_index];
            sg.has_backup = true;
            sg.backup_tier = FMA_TIER_LOCAL;
            sg.packed_off = x.packed_off;
        }
    }

    // ---- unmapper thread (types above): cuMemUnmap runs UNDER the copy pipeline instead of after it ----
    Unmapper un;
    un.e = e;
    ApplyUnmapped apply_unmapped{&un, e, &ex, tier};

    std::vector<PlannedUnit> off_units;  // same order as the image
    auto add_range = [](std::vector<Range>& v, CUdeviceptr va, size_t bytes) {
        if (!v.empty() && v.back().va + v.back().bytes == va) v.back().bytes += bytes;  // VA-adjacent: one driver call
        else v.push_back(Range{va, bytes});
    };
    {
        std::map<CUdeviceptr, uint64_t> unit_end;  // unit -> image_end (offloaded units only)
        for (const Extent& x : ex) {
            const CUdeviceptr key = e->segs[x.seg_index].unit_va;
            uint64_t& end = unit_end[key];
            end = std::max<uint64_t>(end, x.packed_off + x.bytes);
        }
        // arenas in index order, units by VA inside: identical to the image order
        std::vector<const Unit*> ordered;
        for (auto& kv : e->units) ordered.push_back(&kv.second);
        std::sort(ordered.begin(), ordered.end(), [](const Unit* a, const Unit* b) { return a->arena != b->arena ? a->arena < b->arena : a->va < b->va; });
        for (const Unit* u : ordered) {
            auto it = unit_end.find(u->va);
            if (e->ring_attached && u->va == e->ring_unit_va && mode == FMA_MODE_STAGED) continue;  // holds the ring: unmapped after the last D2H
            if (it == unit_end.end()) add_range(un.first, u->va, u->bytes);
            else off_units.push_back(PlannedUnit{u->va, u->bytes, it->second});
        }
    }
    size_t next_unit = 0;  // first offloaded unit not yet handed to the unmapper
    size_t stage_events_used = 0;
    auto stage_event = [&](cudaStream_t stream, cudaEvent_t* out) -> int {
        if (stage_events_used == e->ev_stage.size()) {
            cudaEvent_t ev;
            RT(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            e->ev_stage.push_back(ev);
        }
        *out = e->ev_stage[stage_events_used++];
        RT(cudaEventRecord(*out, stream));
        return FMA_OK;
    };
    // everything whose bytes are inside image[0, image_done) and has been read by work enqueued on `stream` so far
    auto publish_consumed = [&](uint64_t image_done, cudaStream_t stream) -> int {
        Stage st;
        while (next_unit < off_units.size() && off_units[next_unit].image_end <= image_done) {
            add_range(st.ranges, off_units[next_unit].va, off_units[next_unit].bytes);
            ++next_unit;
        }
        if (st.ranges.empty()) return FMA_OK;
        int r = stage_event(stream, &st.ev);
        if (r != FMA_OK) return r;
        un.publish(std::move(st));
        return FMA_OK;
    };
    const bool overlap_unmap = env_int("FMA_OVERLAP_UNMAP", 1) != 0;
    if (overlap_unmap) un.th = std::thread([&un] { un.run(); });

    if (W && adopt) {
        publish_consumed(W, e->ks);  // nothing to copy: every offloaded unit can go at once
        zero_kernel_stats(e);
        if (!e->ring_attached && env_int("FMA_RING_PERSIST", 0) == 0) release_ring(e);  // a sleeping model holds no staging ring
    } else if (W) {
        char* store = static_cast<char*>(store_copy_base(e, tier));
        if (ex_res.empty()) {  // (else the resident gather opened the device-time bracket)
            rc = timer.begin();
            if (rc != FMA_OK) return rc;
        }
        SleepPipe pipe{e, partial ? dirty : ex, W, tier, store, kt, copy_ops, publish_consumed};
        if (partial_packed) {  // only the changed segments' pages are re-coded, each into its old place
            pipe.subset = &dirty_pages;
            rc = pipe.staged_packed();
        } else if (partial) {  // only the changed segments move; everything below each of them is in the store already
            rc = pipe.direct();
            if (rc == FMA_OK) rc = publish_consumed(W, e->cs[0]);  // cs[0] has joined the other streams after the last extent
        } else if (mode == FMA_MODE_DIRECT) rc = pipe.direct();
        else if (mode == FMA_MODE_KERNEL) rc = packed ? pipe.kernel_packed() : pipe.kernel();
        else if (multipath && !packed) rc = pipe.multipath();
        else rc = packed ? pipe.staged_packed() : pipe.staged();
        if (rc != FMA_OK) return rc;
        {
            std::lock_guard<std::mutex> lk(un.mu);
            un.closed = true;
        }
        un.cv.notify_all();
        rc = timer.end(&copy_s);
        if (rc != FMA_OK) return rc;
        rc = kt.collect();
        if (rc != FMA_OK) return rc;
        if (packed) {  // K4 counts pages that no longer fit the form the probe chose (weights written during the sleep)
            rc = check_pack_errors(e, kPackChanged);
            if (rc != FMA_OK) return rc;
        }
        if (env_int("FMA_RING_PERSIST", 0) == 0 || e->ring_attached) release_ring(e);  // while the unmapper finishes its last ranges
    }
    if (!ex_res.empty() && (!W || adopt)) {  // only the resident gather ran: close its bracket
        rc = timer.end(&copy_s);
        if (rc != FMA_OK) return rc;
        rc = kt.collect();
        if (rc != FMA_OK) return rc;
    }
    un.finish();
    if (un.error != FMA_OK) return fail(un.error, "%s", un.msg);

    // apply what the unmapper did to the table, then unmap whatever is left (FMA_OVERLAP_UNMAP=0, nothing
    // offloaded, ...) — every unit goes (cumem.py:213), VAs stay reserved
    for (const Extent& x : ex) {
        Segment& s = e->segs[x.seg_index];
        s.has_backup = true;
        s.backup_tier = tier;
        s.packed_off = x.packed_off;
    }
    apply_unmapped.run();
    {
        std::lock_guard<std::mutex> lk(e->mu);
        std::vector<Range> rest;
        for (auto& kv : e->units) add_range(rest, kv.second.va, kv.second.bytes);
        const double a0 = now_s();
        for (const Range& r : rest) {
            rc = unmap_units(e, r.va, r.bytes);
            if (rc != FMA_OK) return rc;
        }
        un.seconds += now_s() - a0;
        for (Segment& s : e->segs) {
            s.mapped = false;
            s.unit_va = 0;
        }
    }
    e->image_bytes = W;
    e->image_tier = tier;

    e->tl_add("total", 0, t_entry, now_s(), W_all);
    e->st.sleep_seconds = now_s() - t_entry;
    e->st.sleep_copy_seconds = copy_s;
    e->st.sleep_unmap_seconds = un.seconds;
    e->st.sleep_bytes_offloaded = W_all;
    {
        uint64_t copied = 0;  // what this sleep moved into the store
        if (partial) for (const Extent& x : dirty) copied += x.bytes;
        else if (partial_packed) for (size_t p : dirty_pages) copied += e->img_bytes[p];
        else if (!adopt) copied = Wp;
        e->st.sleep_bytes_copied = copied;
    }
    e->st.sleep_bytes_discarded = discarded;
    e->st.copy_ops = copy_ops;
    e->st.total_copy_ops += copy_ops;
    e->st.tier = tier;
    e->st.mode = mode;
    if (!W && ex_res.empty()) zero_kernel_stats(e);
    return FMA_OK;
}

}  // namespace fma_impl
