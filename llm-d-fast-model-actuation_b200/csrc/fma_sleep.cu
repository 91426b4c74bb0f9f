// fma_sleep.cu — SLEEP: vllm:device_allocator/cumem.py:177-225 -> do_sleep (and the PACKED image plan)
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"
#include "fma_gate.h"

namespace fma_impl {

namespace {

// K4p over the pages of `ex`: the stored size of each lands in e->h_psize[0, n_pages).  pack_pages: descriptors to provide for.
int pack_probe(fma_engine_t* e, const std::vector<Extent>& ex, size_t n_pages, size_t pack_pages) {
    RC(ensure_tables(e, n_pages));
    RC(ensure_pack_bufs(e, pack_pages));
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
    RC(digest_segments(e, idx, &dg));
    for (size_t k = 0; k < idx.size(); ++k) {
        e->segs[idx[k]].digest = dg[k];
        e->segs[idx[k]].digest_valid = true;
    }
    if (out) *out = std::move(dg);
    return FMA_OK;
}

// x's bytes are in the store of `tier`, at x.packed_off
void mark_backed_up(fma_engine_t* e, const Extent& x, int tier) {
    Segment& s = e->segs[x.seg_index];
    s.has_backup = true;
    s.backup_tier = tier;
    s.packed_off = x.packed_off;
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
    RC(pack_probe(e, ex, n_pages, n_pages));
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
// Units in VA order, split into "discarded" (release now) and "offloaded" (release once the image has their
// bytes).  image_end = packed offset just past the unit's last live segment.
struct PlannedUnit {
    CUdeviceptr va;
    size_t bytes;
    uint64_t image_end;
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
    std::vector<PlannedUnit> off_units;  // offloaded units, same order as the image
    size_t next_unit = 0;                // first offloaded unit not yet handed to the thread
    size_t stage_events_used = 0;
    std::thread th;
    explicit Unmapper(fma_engine_t* eng) : e(eng) {}
    static void add_range(std::vector<Range>& v, CUdeviceptr va, size_t bytes) {
        if (!v.empty() && v.back().va + v.back().bytes == va) v.back().bytes += bytes;  // VA-adjacent: one driver call
        else v.push_back(Range{va, bytes});
    }
    // every unit: discarded (unmapped first) or offloaded (once the image has its bytes); keep_ring: the unit that holds the
    // ring is unmapped after the last D2H
    void plan(const std::vector<Extent>& ex, bool keep_ring) {
        std::map<CUdeviceptr, uint64_t> unit_end;  // unit -> image_end (offloaded units only)
        for (const Extent& x : ex) {
            uint64_t& end = unit_end[e->segs[x.seg_index].unit_va];
            end = std::max<uint64_t>(end, x.packed_off + x.bytes);
        }
        // arenas in index order, units by VA inside: identical to the image order
        std::vector<const Unit*> ordered;
        for (auto& kv : e->units) ordered.push_back(&kv.second);
        std::sort(ordered.begin(), ordered.end(), [](const Unit* a, const Unit* b) { return a->arena != b->arena ? a->arena < b->arena : a->va < b->va; });
        for (const Unit* u : ordered) {
            auto it = unit_end.find(u->va);
            if (e->ring_attached && u->va == e->ring_unit_va && keep_ring) continue;
            if (it == unit_end.end()) add_range(first, u->va, u->bytes);
            else off_units.push_back(PlannedUnit{u->va, u->bytes, it->second});
        }
    }
    int stage_event(cudaStream_t stream, cudaEvent_t* out) {
        if (stage_events_used == e->ev_stage.size()) {
            cudaEvent_t ev;
            RT(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            e->ev_stage.push_back(ev);
        }
        *out = e->ev_stage[stage_events_used++];
        RT(cudaEventRecord(*out, stream));
        return FMA_OK;
    }
    // everything whose bytes are inside image[0, image_done) and has been read by work enqueued on `stream` so far (no stream:
    // those bytes are in the store already, the FILE tier's written frontier)
    int publish_consumed(uint64_t image_done, cudaStream_t stream) {
        Stage st;
        while (next_unit < off_units.size() && off_units[next_unit].image_end <= image_done) {
            add_range(st.ranges, off_units[next_unit].va, off_units[next_unit].bytes);
            ++next_unit;
        }
        if (st.ranges.empty()) return FMA_OK;
        st.ev = nullptr;
        if (stream) RC(stage_event(stream, &st.ev));
        {
            std::lock_guard<std::mutex> lk(mu);
            stages.push_back(std::move(st));
        }
        cv.notify_all();
        return FMA_OK;
    }
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
            cudaError_t r = st.ev ? cudaEventSynchronize(st.ev) : cudaSuccess;
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
    void close() {  // nothing more to come: the thread ends after the last published stage
        {
            std::lock_guard<std::mutex> lk(mu);
            closed = true;
        }
        cv.notify_all();
    }
    void finish() {
        close();
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
            forget_units(e, r.va, r.bytes);
            for (Segment& sg : e->segs)
                if (sg.va >= r.va && sg.va < r.va + r.bytes) {
                    sg.mapped = false;
                    sg.unit_va = 0;
                }
            for (const Extent& x : *ex)
                if (x.va >= r.va && x.va < r.va + r.bytes) mark_backed_up(e, x, tier);
        }
        if (!un->done.empty()) e->image_tier = tier;  // even a failed sleep leaves an image a later wake can restore from
    }
    ~ApplyUnmapped() {
        un->finish();
        run();
    }
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
    Unmapper* un;          // releases units behind the pipeline; null: nothing is released (the resident gather)
    const std::vector<size_t>* subset = nullptr;  // INCREMENTAL + PACKED: only these image pages (ascending) are re-coded, in place
    bool resident = false;  // the extents go to the resident buffer (e->res, its own page layout res_off / res_bytes), not the tier's store
    ImageFile* file = nullptr;   // FILE tier: the staged pipeline writes the image to this file, not to `store`
    int publish_consumed(uint64_t image_done, cudaStream_t stream) { return un ? un->publish_consumed(image_done, stream) : FMA_OK; }
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
        RC(ensure_tables(e, pages->size()));
        build_page_table(ex, e->h_tab);
        RT(cudaMemcpyAsync(e->d_tab, e->h_tab, pages->size() * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
        return FMA_OK;
    }
    int direct();
    int in_place(bool packed);
    int staged(bool packed);
    int multipath();
};

// DIRECT: copy engines move each segment chunk straight into the packed image
int SleepPipe::direct() {
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
            RC(publish_consumed(image_done, e->cs[0]));
            next_join = image_done + slot;
        }
    }
    return FMA_OK;
}

// IN PLACE: K1 / K4 write the store themselves: mapped pinned host memory (PCIe posted writes) or peer / local HBM (a PACKED
// image: 0.758 of the bytes over NVLink and of the parking GPU's HBM)
int SleepPipe::in_place(bool packed) {
    std::vector<PagePlan> pages;
    RC(plan(packed, &pages));
    const uint64_t dbase = resident ? (uint64_t)e->res.va : store_dev_base(e, tier);
    PageKernels pk{e, kt, true, packed};
    RC(pk.prepare(pages, true, [&](size_t q) { return dbase + pages[q].off; }));
    // launched in slot-sized batches so finished segments can be released while later ones still move
    std::vector<Batch> batches;
    fma_layout::plan_batches(pages, slot_pages(e), UINT64_MAX, false, &batches);
    for (const Batch& b : batches) {
        RC(pk.launch(b, dbase + pages[b.p0].off));
        ++copy_ops;
        RC(publish_gathered(b.p0 + b.np));
    }
    return FMA_OK;
}

// STAGED: K1 gather / K4 gather + encode -> HBM ring slot (a PACKED image: stored pages back to back) -> one large D2H per slot.
// The FILE tier (file_fd) puts a disk stage behind the ring: each slot drains into the engine's pinned I/O windows, one D2H per
// window, and writer threads pwrite each window at its place in the file.  A unit is then released once every byte of it has been
// WRITTEN (the writes' frontier, not the D2H's), so a sleep whose write fails half way leaves every released segment in the file.
int SleepPipe::staged(bool packed) {
    std::vector<PagePlan> pages;
    RC(plan(packed, &pages));   // (the route has the ring)
    // the image pages this sleep moves: all of them, or (incremental) the pages of the changed segments, whose stored size
    // is known not to change, so each goes back to its old place in the kept image
    std::vector<size_t> img_page(pages.size());
    for (size_t p = 0; p < pages.size(); ++p) img_page[p] = p;
    if (subset) {
        img_page = *subset;
        std::vector<PagePlan> sel;
        for (size_t p : img_page) sel.push_back(pages[p]);
        pages = std::move(sel);
    }
    std::vector<Batch> slots;
    std::vector<uint64_t> in_ring;
    RC(plan_ring_slots(e, packed, pages, &slots, &in_ring));
    PageKernels pk{e, kt, true, packed};
    RC(pk.prepare(pages, true, [&](size_t q) { return in_ring[q]; }));
    // every image byte below the last page of slot c is in the store once slot c is (moved, or kept from the last wake)
    auto image_end = [&](size_t c) { return (uint64_t)(img_page[slots[c].p0 + slots[c].np - 1] + 1) * FMA_PAGE_BYTES; };
    // FILE: every slot cut into window-sized writes; slot c's are items [slot_end[c - 1], slot_end[c])
    std::vector<FileIO::Item> items;
    std::vector<size_t> slot_end;
    std::optional<FileIO> io;
    if (file) {
        for (const Batch& sl : slots) items.push_back(FileIO::Item{pages[sl.p0].off, sl.stored});
        items = FileIO::cut(e, items, &slot_end);
        file->write(items, &io);
    }
    size_t k = 0, slots_written = 0;
    auto publish_written = [&]() -> int {   // units whose every page is in a slot that has been written are dead
        const size_t n = io->written();
        while (slots_written < slots.size() && slot_end[slots_written] <= n) ++slots_written;
        return slots_written ? publish_consumed(image_end(slots_written - 1), nullptr) : FMA_OK;
    };
    cudaStream_t last_stream = e->cs[0];
    for (size_t c = 0; c < slots.size(); ++c) {
        const Batch& sl = slots[c];
        const int slot = (int)(c % e->n_ring);
        char* ring = static_cast<char*>(e->ring[slot]);
        cudaStream_t cstream = e->cs[c % e->n_cs];
        if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(e->ks, e->ev_ring_free[slot], 0));
        RC(pk.launch(sl, (uint64_t)(uintptr_t)ring));
        RT(cudaEventRecord(e->ev_ring_full[slot], e->ks));
        RT(cudaStreamWaitEvent(cstream, e->ev_ring_full[slot], 0));
        if (io) {
            for (; k < slot_end[c]; ++k, ++copy_ops) {
                RC(io->copy(k, ring + (items[k].file_off - pages[sl.p0].off), cstream));
                RC(publish_written());
            }
        } else {
            RT(cudaMemcpyAsync(store + pages[sl.p0].off, ring, sl.stored, cudaMemcpyDefault, cstream));
            ++copy_ops;
            // "slot free" also means "every earlier slot has reached the store" (chained through the previous
            // slot's event), so the unmapper below never releases device memory whose bytes are not yet on the host
            if (c > 0) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[(c - 1) % e->n_ring], 0));
        }
        RT(cudaEventRecord(e->ev_ring_free[slot], cstream));
        if (!io) RC(publish_consumed(image_end(c), cstream));   // units fully in the store are dead
        last_stream = cstream;
    }
    if (io) {
        RC(io->finish());   // every pwrite has returned
        return publish_consumed(W, nullptr);
    }
    return subset ? publish_consumed(W, last_stream) : FMA_OK;  // the clean tail of the image needs no copy
}

// MULTI-PATH sleep (fma_paths_set): the mirror image of the multi-path wake.  K1 on the sleeping GPU gathers a chunk of the image
// into a staging slot of a PATH — its own HBM, or a helper GPU's HBM over NVLink — and THAT GPU's copy engine moves the slot into
// the host store over THAT GPU's x16 link; chunk queues per NUMA node of the (striped) store, self-balancing.  Nothing is unmapped
// before every byte has reached the store (one publish at the end), so a failure half way leaves the engine awake and intact.
int SleepPipe::multipath() {
    std::vector<PagePlan> pages;
    RC(plan(false, &pages));
    RC(ensure_ring_events(e, 1));
    cudaEvent_t ev_tab = e->ev_ring_full[0];
    RT(cudaEventRecord(ev_tab, e->ks));
    std::vector<Batch> chunks;
    fma_layout::plan_batches(pages, std::max<size_t>(e->path_slot_bytes / FMA_PAGE_BYTES, 1), UINT64_MAX, true, &chunks);
    std::vector<uint64_t> chunk_off;
    for (const Batch& ch : chunks) chunk_off.push_back(pages[ch.p0].off);
    fma_layout::ChunkQueues queues(chunk_off, e->host.ranges);
    PathWorkers pw;
    pw.run(e, ev_tab, [&](size_t pi) {
        WakePath& path = e->paths[pi];
        auto failw = [&](int code, const char* what, cudaError_t ce) { pw.fail_once(code, pi, path.device, what, cudaGetErrorString(ce)); };
        cudaError_t ce;
        uint32_t mine = 0;
        for (;;) {
            if (pw.error.load() != FMA_OK) return;
            size_t c = 0;
            if (!queues.take(path.numa_node, &c)) break;
            const Batch& ch = chunks[c];
            const int slot = (int)(mine % (uint32_t)e->path_slots);
            if (mine >= (uint32_t)e->path_slots) {   // the D2H that used this slot before has drained it (event on the path's GPU)
                ce = cudaEventSynchronize(path.ev_full[slot]);
                if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventSynchronize(slot drained)", ce);
            }
            char* slot_ptr = reinterpret_cast<char*>(path.staging.va) + (size_t)slot * e->path_slot_bytes;
            {
                std::lock_guard<std::mutex> lk(pw.kt_mu);
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
        pw.per_path[pi] = mine;
    });
    for (WakePath& path : e->paths) {   // every D2H has landed before anything is released (and before an error is reported)
        cudaError_t ce = cudaStreamSynchronize(path.copy);
        if (ce != cudaSuccess && pw.error.load() == FMA_OK) {
            pw.error.store(FMA_ECUDA);
            snprintf(pw.err_msg, sizeof(pw.err_msg), "D2H on path device %d failed: %s", path.device, cudaGetErrorString(ce));
        }
    }
    if (pw.error.load() != FMA_OK) return fail(pw.error.load(), "%s", pw.err_msg);
    for (size_t pi = 0; pi < e->paths.size(); ++pi) {
        copy_ops += pw.per_path[pi];
        e->tl_add("path_chunks", e->paths[pi].device, e->tl_entry, now_s(), (uint64_t)pw.per_path[pi] * e->path_slot_bytes);
    }
    return publish_consumed(W, e->ks);   // all bytes are in the store: every offloaded unit may go
}

// What one sleep moves and how, filled in phase by phase by do_sleep.
struct SleepPlan {
    int tier;
    uint32_t flags;
    std::vector<Extent> ex;       // offloaded extents the tier's store receives, image order
    std::vector<Extent> ex_res;   // RESIDENT share: extents kept in e->res, packed_off = offset in the resident part
    uint64_t W = 0, W_all = 0, discarded = 0;   // bytes of ex, of everything offloaded, of the discarded tags
    // the store that would hold the kept image exists; INCREMENTAL: it may still hold exactly this image
    bool kept_store = false, shadows_match = false;
    // per extent: digest of the copy the store holds, and where it holds it (kNoOffset: no usable copy)
    std::vector<uint64_t> shadow_digest, shadow_at, res_seqs;
    // the image in the store: PACKED or not, its page table and its bytes; planned by the resident split (pre_planned: K4p over
    // the whole image before the ring is known) or by route_sleep
    bool pre_planned = false, packed = false;
    std::vector<uint64_t> pk_off;
    std::vector<uint32_t> pk_bytes;
    uint64_t Wp = 0;
    bool clean = false, partial = false, partial_packed = false, digests_known = false;   // INCREMENTAL outcome
    std::vector<Extent> dirty;        // segments whose device bytes differ from the copy in the store
    std::vector<size_t> dirty_pages;  // their image pages (PACKED image)
    fma_layout::SleepRoute route{};
    CopyTimer timer;                  // device-time bookkeeping of the copies
    KernelTimes kt;
    uint32_t copy_ops = 0;
    double copy_s = 0;
    ImageFile file;                   // FILE tier: the file this sleep writes, opened by size_store
    SleepPlan(fma_engine_t* e, int t, uint32_t f) : tier(t), flags(f), timer{e}, kt{e}, file(e) {}
    bool adopt() const { return (flags & kFlagAdopt) || clean || !W; }  // not a byte moves (the route is then Adopt)
};

fma_layout::SleepFacts sleep_facts(const fma_engine_t* e, const SleepPlan& p) {
    return fma_layout::SleepFacts{p.tier, fma_layout::resolve_mode(e->cfg.mode, p.tier), e->cfg.pack != 0, !e->paths.empty(), e->mbox != nullptr,
                                  (p.flags & kFlagAdopt) || !p.W, p.clean, p.partial, p.partial_packed, env_int("FMA_MULTIPATH_SLEEP", 1) != 0};
}

// `path` is a file of an image of store_bytes (plus the descriptor tail)
bool file_holds(const std::string& path, uint64_t store_bytes) {
    struct stat sb;
    return store_bytes && stat(path.c_str(), &sb) == 0 && (uint64_t)sb.st_size == store_bytes + kImageTail;
}

// 1. offloaded segments -> packed image, in (arena, VA) order.  Arenas are bump-allocated per tag, so this is allocation order
// (the reference's dict order, cumem.py:198) unless a freed hole was reused.
void plan_image(fma_engine_t* e, uint64_t offload_mask, SleepPlan& p) {
    std::vector<size_t> by_addr(e->segs.size());
    for (size_t i = 0; i < by_addr.size(); ++i) by_addr[i] = i;
    std::sort(by_addr.begin(), by_addr.end(), [&](size_t a, size_t b) {
        const Segment &x = e->segs[a], &y = e->segs[b];
        return x.arena != y.arena ? x.arena < y.arena : x.va < y.va;
    });
    // the store that would hold the kept image: the host store, or the parking buffer of the same (peer / local) tier
    // or (FILE) the file the last file-tier image went to, when this sleep writes the same path and the file has that image's size
    p.kept_store = p.tier == FMA_TIER_HOST ? e->host.base != nullptr
                 : p.tier == FMA_TIER_FILE ? !e->file_path.empty() && e->file_path == e->image_file && file_holds(e->image_file, e->shadow_store_bytes)
                                           : (e->park.va != 0 && (p.tier == FMA_TIER_LOCAL ? e->park.device == e->device : e->park.device != e->device));
    p.shadows_match = e->incremental && p.tier == e->shadow_tier && !(p.flags & kFlagAdopt) && p.kept_store;
    for (size_t i : by_addr) {
        Segment& s = e->segs[i];
        if (tag_bit_set(offload_mask, s.tag)) {
            p.shadows_match = p.shadows_match && s.digest_valid && s.shadow_off == p.W;  // same bytes expected at the same image offset
            p.shadow_digest.push_back(s.digest);
            p.shadow_at.push_back(s.digest_valid ? s.shadow_off : kNoOffset);
            p.ex.push_back(Extent{i, s.va, s.bytes, p.W});
            p.W += s.bytes;
        } else {
            p.discarded += s.bytes;
        }
        s.has_backup = false;
        s.packed_off = kNoOffset;
        s.digest_valid = false;
    }
    p.W_all = p.W;
}

// 2. RESIDENT share (option "resident_bytes"): the tail of the image stays in one VMM allocation on this GPU.  Walking the
// offloaded segments from the last to the first, a segment stays if its stored size (2 MiB pages, or its pages' PACKED sizes)
// still fits what is left of the cap; the host store then holds only the other segments, back to back in image order.
int split_resident(fma_engine_t* e, SleepPlan& p) {
    if (!e->resident_cap || p.tier != FMA_TIER_HOST || !e->paths.empty() || (p.flags & kFlagAdopt) || !p.W) return FMA_OK;
    if (fma_layout::sleep_route(sleep_facts(e, p)).wants_probe) {  // asked before the ring is known
        RC(plan_packed_image(e, p.ex, p.W, &p.pk_off, &p.pk_bytes, &p.Wp, &p.packed));
        p.pre_planned = true;
    }
    std::vector<uint64_t> stored(p.ex.size());
    for (size_t k = 0; k < p.ex.size(); ++k) {
        stored[k] = p.packed ? 0 : p.ex[k].bytes;
        if (p.packed)
            for (uint64_t o = 0; o < p.ex[k].bytes; o += FMA_PAGE_BYTES) stored[k] += p.pk_bytes[(p.ex[k].packed_off + o) / FMA_PAGE_BYTES];
    }
    const std::vector<char> res = fma_layout::resident_split(stored, e->resident_cap);
    uint64_t res_stored = 0;
    for (size_t k = 0; k < p.ex.size(); ++k) res_stored += res[k] ? stored[k] : 0;
    if (!res_stored) return FMA_OK;
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
        return FMA_OK;
    }
    e->tl_add("res_alloc", 0, a, b, buf.bytes);
    // the two parts, each laid out back to back in image order: [0] the host store, [1] the resident buffer
    struct Part {
        std::vector<Extent> ex;
        std::vector<uint64_t> off;     // PACKED: stored offset and size of each image page
        std::vector<uint32_t> bytes;
        uint64_t W = 0, stored = 0;
    } part[2];
    std::vector<uint64_t> h_digest;
    bool host_shadows = true;
    for (size_t k = 0; k < p.ex.size(); ++k) {
        Part& d = part[(int)res[k]];
        Extent x = p.ex[k];
        const uint64_t p0 = x.packed_off / FMA_PAGE_BYTES;
        x.packed_off = d.W;
        d.W += x.bytes;
        d.ex.push_back(x);
        if (res[k]) {
            p.res_seqs.push_back(e->segs[x.seg_index].seq);
        } else {
            host_shadows = host_shadows && p.shadow_at[k] == x.packed_off;
            h_digest.push_back(p.shadow_digest[k]);
        }
        if (p.packed)
            for (uint64_t q = p0; q < p0 + x.bytes / FMA_PAGE_BYTES; ++q) {
                d.off.push_back(d.stored);
                d.bytes.push_back(p.pk_bytes[q]);
                d.stored += p.pk_bytes[q];
            }
    }
    e->res = buf;
    e->res_packed = p.packed;
    e->res_off = std::move(part[1].off);
    e->res_bytes = std::move(part[1].bytes);
    e->res_store_bytes = res_stored;
    p.ex = std::move(part[0].ex);
    p.ex_res = std::move(part[1].ex);
    p.W = part[0].W;
    p.shadows_match = e->incremental && p.tier == e->shadow_tier && p.kept_store && host_shadows;
    p.shadow_digest = std::move(h_digest);
    p.Wp = p.packed ? part[0].stored : part[0].W;
    if (p.packed) {
        p.pk_off = std::move(part[0].off);
        p.pk_bytes = std::move(part[0].bytes);
    }
    return FMA_OK;
}

// 3. INCREMENTAL sleep: does the store still hold exactly this image?  One K3 pass over the device copy decides.
int check_incremental(fma_engine_t* e, SleepPlan& p) {
    p.shadows_match = p.shadows_match && p.res_seqs == e->res_seqs;  // a different split is a full sleep
    e->res_seqs = p.res_seqs;
    const uint64_t W = p.W;
    if (!p.shadows_match || !W || W != e->shadow_image_bytes || (p.tier == FMA_TIER_HOST ? e->host.cap : p.tier == FMA_TIER_FILE ? e->shadow_store_bytes : e->park.bytes) < e->shadow_store_bytes) return FMA_OK;
    RT(cudaDeviceSynchronize());  // the caller's streams may still be writing weights
    std::vector<uint64_t> now;
    RC(digest_and_mark(e, p.ex, &now));  // either way these are the digests of what sleeps now
    uint64_t dirty_bytes = 0;
    for (size_t k = 0; k < p.ex.size(); ++k)
        if (now[k] != p.shadow_digest[k]) {
            p.dirty.push_back(p.ex[k]);
            dirty_bytes += p.ex[k].bytes;
        }
    p.digests_known = true;
    p.clean = p.dirty.empty();
    // a few changed segments (an adapter, fp8 KV scales reset after wake, one synced layer): only they cross the link, into
    // their old place in the kept image (partial sleeps are a host-tier refinement; in a parking tier a changed image is
    // simply parked again)
    const bool few = p.tier == FMA_TIER_HOST && !p.clean && 2 * dirty_bytes <= W && !e->host.shared;  // a shared image is read-only
    p.partial = few && !e->shadow_packed;
    // PACKED image: a changed page can go back to its old place only if its stored size stays what it was (K4p on those pages)
    if (few && e->shadow_packed && fma_layout::sleep_route(sleep_facts(e, p)).wants_probe) {
        for (const Extent& x : p.dirty)
            for (size_t o = 0; o < x.bytes; o += FMA_PAGE_BYTES) p.dirty_pages.push_back((size_t)((x.packed_off + o) / FMA_PAGE_BYTES));
        RC(pack_probe(e, p.dirty, p.dirty_pages.size(), std::max<size_t>(p.dirty_pages.size(), W / FMA_PAGE_BYTES)));
        bool fits = p.dirty_pages.size() <= e->img_bytes.size();
        for (size_t q = 0; q < p.dirty_pages.size() && fits; ++q)
            fits = p.dirty_pages[q] < e->img_bytes.size() && e->h_psize[q] == e->img_bytes[p.dirty_pages[q]];
        p.partial_packed = fits && !no_ring() && ensure_ring(e, W) == FMA_OK;  // no HBM for a ring: full sleep through the plain path
    }
    return FMA_OK;
}

// 4. the pipeline (fma_layout::sleep_route), with the staging ring and the PACKED plan it needs, BEFORE the store is sized
int route_sleep(fma_engine_t* e, SleepPlan& p) {
    if (!p.clean && !p.partial && !p.partial_packed) invalidate_shadows(e);  // this sleep rewrites the store (or leaves the host tier alone: be conservative)
    fma_layout::SleepFacts f = sleep_facts(e, p);
    if (fma_layout::sleep_route(f).wants_ring) f.ring = !no_ring() && ensure_ring(e, p.W) == FMA_OK;
    p.route = fma_layout::sleep_route(f);
    if (p.route.pipe == fma_layout::SleepPipeKind::NoRing) return fail(FMA_ENOMEM, "the file tier needs an HBM staging ring and there is no room for one");
    const bool kept = p.clean || p.partial_packed;  // the image in the store, its form and its page table stay as they are
    if (kept) {
        p.packed = e->shadow_packed;
        p.Wp = e->shadow_store_bytes;
    } else if (p.route.wants_probe) {
        if (!p.pre_planned) RC(plan_packed_image(e, p.ex, p.W, &p.pk_off, &p.pk_bytes, &p.Wp, &p.packed));
        f.worth_packing = p.packed;
        p.route = fma_layout::sleep_route(f);
    } else {  // (a plan of the resident split is dropped)
        p.packed = false;
        p.Wp = p.W;
    }
    e->image_packed = p.packed;
    e->image_store_bytes = p.Wp;
    if (!kept) {
        e->img_off = p.packed ? std::move(p.pk_off) : std::vector<uint64_t>();
        e->img_bytes = p.packed ? std::move(p.pk_bytes) : std::vector<uint32_t>();
    }
    if (kept || p.packed) e->image_bytes = p.W;  // the layout is indexed by image page: valid from here on, also if the sleep fails
    return FMA_OK;
}

// FILE: open the file, check that the filesystem has room for the image and its descriptor, and only then empty the file
int open_sleep_file(fma_engine_t* e, SleepPlan& p) {
    if (e->file_path.empty()) return fail(FMA_ESTATE, "the file tier needs fma_file_store(path) first");
    if (!e->load_ring) return fail(FMA_ESTATE, "the engine's I/O windows are not pinned");
    RC(p.file.create(e->file_path, p.Wp));
    e->image_file = e->file_path;
    return FMA_OK;
}

// 5. a store of the tier that holds Wp bytes
int size_store(fma_engine_t* e, SleepPlan& p) {
    if (!p.W) return FMA_OK;
    if (p.tier == FMA_TIER_HOST && p.adopt()) {
        if (!e->host.base) return fail(FMA_ESTATE, "adopt without a store");  // the adopted store IS the image: never re-sized
    } else if (p.tier == FMA_TIER_HOST) {
        if (e->host.shared) {  // this sleep writes: leave the shared image to its other holders and take a private store
            invalidate_shadows(e);
            host_store_free(e->host);
        }
        RC(host_store_reserve(e, p.Wp));
        if (p.route.mode == FMA_MODE_KERNEL && !e->host.dev_alias) return fail(FMA_ECUDA, "host store has no device alias for zero-copy mode");
    } else if (p.tier == FMA_TIER_PEER) {
        if (!e->park.va || e->park.bytes < p.Wp || e->park.device == e->device)
            return fail(FMA_ESTATE, "peer tier needs fma_peer_reserve(peer_device, >= %llu bytes) first", (unsigned long long)p.Wp);
    } else if (p.tier == FMA_TIER_LOCAL) {
        return park_reserve(e, e->device, p.Wp);
    } else if (p.tier == FMA_TIER_FILE) {
        if (!p.adopt()) return open_sleep_file(e, p);   // (an adopted or clean image is in its file already)
    } else {
        return fail(FMA_EINVAL, "unknown tier %d", p.tier);
    }
    return FMA_OK;
}

// 6. RESIDENT share: K1 / K4 gather the resident segments into e->res (HBM only, a few ms), ahead of the host part's pipeline on
// the kernel stream.  Synchronised before the host part starts: it rewrites the page tables, and the units that hold only
// resident segments are unmapped right away after it.
int gather_resident(fma_engine_t* e, SleepPlan& p) {
    if (p.ex_res.empty()) return FMA_OK;
    if ((p.flags & FMA_FLAG_VERIFY) || e->incremental) RC(digest_and_mark(e, p.ex_res));
    RC(p.timer.begin());
    uint32_t res_launches = 0;
    SleepPipe rp{e, p.ex_res, p.W_all - p.W, FMA_TIER_LOCAL, nullptr, p.kt, res_launches, nullptr};  // units go with the host part
    rp.resident = true;
    p.kt.kind = "res_gather";
    const int rc = rp.in_place(e->res_packed);
    p.kt.kind = "kernel";
    if (rc != FMA_OK) return rc;
    if (e->res_packed) RC(check_pack_errors(e, kPackChanged));
    else RT(cudaStreamSynchronize(e->ks));
    std::lock_guard<std::mutex> lk(e->mu);
    for (const Extent& x : p.ex_res) mark_backed_up(e, x, FMA_TIER_LOCAL);
    return FMA_OK;
}

// 7. the copy pipeline of the route, with the unmapper releasing units behind it
int run_pipeline(fma_engine_t* e, SleepPlan& p, Unmapper& un) {
    using fma_layout::SleepPipeKind;
    if (p.W && p.adopt()) {
        un.publish_consumed(p.W, e->ks);  // nothing to copy: every offloaded unit can go at once
        zero_kernel_stats(e);
        if (!e->ring_attached && env_int("FMA_RING_PERSIST", 0) == 0) release_ring(e);  // a sleeping model holds no staging ring
    } else if (p.W) {
        char* store = static_cast<char*>(store_copy_base(e, p.tier));
        if (p.ex_res.empty()) RC(p.timer.begin());  // (else the resident gather opened the device-time bracket)
        SleepPipe pipe{e, p.partial ? p.dirty : p.ex, p.W, p.tier, store, p.kt, p.copy_ops, &un};
        switch (p.route.pipe) {
        case SleepPipeKind::PartialPacked:  // only the changed segments' pages are re-coded, each into its old place
            pipe.subset = &p.dirty_pages;
            RC(pipe.staged(true));
            break;
        case SleepPipeKind::PartialDirect:  // only the changed segments move; everything below each of them is in the store already
            RC(pipe.direct());
            RC(un.publish_consumed(p.W, e->cs[0]));  // cs[0] has joined the other streams after the last extent
            break;
        case SleepPipeKind::Direct: RC(pipe.direct()); break;
        case SleepPipeKind::Kernel: RC(pipe.in_place(false)); break;
        case SleepPipeKind::KernelPacked: RC(pipe.in_place(true)); break;
        case SleepPipeKind::Multipath: RC(pipe.multipath()); break;
        case SleepPipeKind::StagedPacked: RC(pipe.staged(true)); break;
        case SleepPipeKind::Staged: RC(pipe.staged(false)); break;
        case SleepPipeKind::File:
        case SleepPipeKind::FilePacked:
            pipe.file = &p.file;
            RC(pipe.staged(p.route.pipe == SleepPipeKind::FilePacked));
            break;
        case SleepPipeKind::NoRing:   // (refused by route_sleep)
        case SleepPipeKind::Adopt: return fail(FMA_ESTATE, "an adopted image has no copy pipeline");  // (handled above)
        }
        un.close();
        RC(p.timer.end(&p.copy_s));
        RC(p.kt.collect());
        if (p.packed) RC(check_pack_errors(e, kPackChanged));  // K4 counts pages that no longer fit the form the probe chose (weights written during the sleep)
        if (env_int("FMA_RING_PERSIST", 0) == 0 || e->ring_attached) release_ring(e);  // while the unmapper finishes its last ranges
    }
    if (!p.ex_res.empty() && (!p.W || p.adopt())) {  // only the resident gather ran: close its bracket
        RC(p.timer.end(&p.copy_s));
        RC(p.kt.collect());
    }
    return FMA_OK;
}

// 8. apply what the unmapper did to the table, then unmap whatever is left (FMA_OVERLAP_UNMAP=0, nothing offloaded, ...) —
// every unit goes (cumem.py:213), VAs stay reserved; then the stats
int finish_sleep(fma_engine_t* e, SleepPlan& p, Unmapper& un, ApplyUnmapped& apply_unmapped, double t_entry) {
    un.finish();
    if (un.error != FMA_OK) return fail(un.error, "%s", un.msg);
    for (const Extent& x : p.ex) mark_backed_up(e, x, p.tier);
    apply_unmapped.run();
    {
        std::lock_guard<std::mutex> lk(e->mu);
        std::vector<Range> rest;
        for (auto& kv : e->units) Unmapper::add_range(rest, kv.second.va, kv.second.bytes);
        const double a0 = now_s();
        for (const Range& r : rest) RC(unmap_units(e, r.va, r.bytes));
        un.seconds += now_s() - a0;
        for (Segment& s : e->segs) {
            s.mapped = false;
            s.unit_va = 0;
        }
    }
    e->image_bytes = p.W;
    e->image_tier = p.tier;
    if (p.file.fd() >= 0) RC(p.file.seal(FMA_TIER_FILE));   // (the image is asleep in the file either way: a wake reads what was written)

    e->tl_add("total", 0, t_entry, now_s(), p.W_all);
    e->st.sleep_seconds = now_s() - t_entry;
    e->st.sleep_copy_seconds = p.copy_s;
    e->st.sleep_unmap_seconds = un.seconds;
    e->st.sleep_bytes_offloaded = p.W_all;
    uint64_t copied = 0;  // what this sleep moved into the store
    if (p.partial) for (const Extent& x : p.dirty) copied += x.bytes;
    else if (p.partial_packed) for (size_t q : p.dirty_pages) copied += e->img_bytes[q];
    else if (!p.adopt()) copied = p.Wp;
    e->st.sleep_bytes_copied = copied;
    e->st.sleep_bytes_discarded = p.discarded;
    e->st.copy_ops = p.copy_ops;
    e->st.total_copy_ops += p.copy_ops;
    e->st.tier = p.tier;
    e->st.mode = p.route.mode;
    if (!p.W && p.ex_res.empty()) zero_kernel_stats(e);
    return FMA_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------
// SLEEP
// ------------------------------------------------------------------------------------
int do_sleep(fma_engine_t* e, uint64_t offload_mask, int tier, uint32_t flags) {
    DeviceGuard guard(e->device);
    RC(flush_kernel_times(e));
    const double t_entry = now_s();
    RC(ensure_streams(e));

    // Executor.sleep is a no-op while sleeping (abstract.py:323-325)
    bool any_unmapped = false, any_mapped = false;
    for (const Segment& s : e->segs) (s.mapped ? any_mapped : any_unmapped) = true;
    if (any_unmapped || !any_mapped) return FMA_OK;
    RC(check_tma_shape(e, tier));
    e->tl_begin("sleep", t_entry);
    if (e->res.va) {  // a resident buffer kept by an FMA_FLAG_KEEP_BACKUP wake: this sleep gathers its resident part afresh
        RT(cudaDeviceSynchronize());
        GateHold hold(kGateUnmap, 0.1);
        resident_release(e);
    }
    if (e->pf.va) {  // a prefetch left behind by segments freed while asleep: this sleep writes a new image
        RT(cudaDeviceSynchronize());
        prefetch_release(e);
    }

    SleepPlan p(e, tier, flags);
    plan_image(e, offload_mask, p);
    RC(split_resident(e, p));
    RC(check_incremental(e, p));
    RC(route_sleep(e, p));
    RC(size_store(e, p));

    // The caller's own streams may still be writing weights: drain the device once, as the
    // reference's blocking cudaMemcpy on the legacy stream implicitly does (before anything reads the segments).
    RT(cudaDeviceSynchronize());
    if (((flags & FMA_FLAG_VERIFY) || e->incremental) && p.W && !p.adopt() && !p.digests_known) {  // incremental: digests seed the next sleep's check
        RC(digest_and_mark(e, p.ex));
    }
    RC(gather_resident(e, p));

    // ---- unmapper thread (types above): cuMemUnmap runs UNDER the copy pipeline instead of after it ----
    Unmapper un(e);
    ApplyUnmapped apply_unmapped{&un, e, &p.ex, tier};
    un.plan(p.ex, p.route.mode == FMA_MODE_STAGED);
    if (env_int("FMA_OVERLAP_UNMAP", 1) != 0) un.th = std::thread([&un] { un.run(); });
    RC(run_pipeline(e, p, un));
    return finish_sleep(e, p, un, apply_unmapped, t_entry);
}

}  // namespace fma_impl
