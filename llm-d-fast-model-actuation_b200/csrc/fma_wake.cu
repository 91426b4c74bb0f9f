// fma_wake.cu — WAKE: vllm:device_allocator/cumem.py:227-249 -> do_wake
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"
#include "fma_gate.h"

namespace fma_impl {

namespace {

using fma_layout::Run;

// ---- mapper thread(s): one create + map + set-access per run, in `runs` order ----------------------
// A wake that fails is rolled back (the destructor, unless committed): every run THIS call mapped is unmapped again (its segments still have their
// backup), so the table is what it was at entry and the controller's retry (inference-server.go:477-480) redoes the whole wake.
// Leaving the mapped prefix in place would make the retry skip it (`mapped` == already awake) and report success over
// weights that were never copied back — vLLM's allocator raises in that situation (cumem.py:237-249).
struct Mapper {
    fma_engine_t* e;
    const std::vector<Run>& runs;
    bool ring_run;                 // the staging ring is work item 0
    double t_entry;
    size_t n_backup_runs = 0;
    double expected_copy_s = 0, remap_delay_s = 0;   // of the host part; remap-only runs start no earlier than this after entry
    bool remap_after_copy = false; // ... nor before copies_landed
    int gate_first = 0;            // cross-process VMM gate: announced for the call that gates the first copy
    std::mutex mu{};
    std::condition_variable cv{};
    std::atomic<size_t> done{0};   // number of work items fully mapped (prefix; written under mu)
    int error = FMA_OK;
    char msg[512] = "";
    std::vector<char> item_done{};
    std::atomic<size_t> next_item{0};
    std::atomic<uint64_t> map_ns{0};
    std::atomic<bool> copies_landed{false};
    std::vector<std::thread> threads{};
    bool committed = false;        // the wake has succeeded: nothing to roll back

    void start(int tier, double copy_s) {
        for (const Run& r : runs) n_backup_runs += r.has_backup;
        expected_copy_s = copy_s;
        // Remap-only runs wait a fifth of the expected copy time (host tier) or half of it (NVLink): far below the slack.
        const int forced_delay_ms = env_int("FMA_REMAP_DELAY_MS", -1);
        remap_delay_s = forced_delay_ms >= 0 ? forced_delay_ms * 1e-3 : expected_copy_s * (tier == FMA_TIER_HOST ? 0.2 : 0.5);
        // FMA_REMAP_AFTER_COPY=1: remap-only runs (kv_cache) are mapped only after this rank's last copy has LANDED — a 32 GiB
        // cuMemCreate/Map/SetAccess then never runs beside this rank's DMA (its cost, a few ms, is added to the wake instead of
        // hidden under it).  A/B knob for the question "does a large VMM call slow a running H2D stream down?".
        remap_after_copy = env_int("FMA_REMAP_AFTER_COPY", 0) != 0 && n_backup_runs > 0;
        // Cross-process VMM gate (fma_gate.h): tell the other engines on this host that a call which gates a first copy is coming
        gate_first = n_backup_runs ? gate_announce(kGateFirst) : 0;
        item_done.assign(runs.size(), 0);
        const int n_threads = std::max(1, std::min(e->cfg.map_threads > 0 ? e->cfg.map_threads : 1, 8));
        for (int t = 0; t < n_threads; ++t) threads.emplace_back([this] { run(); });
    }
    void run() {
        cudaSetDevice(e->device);
        for (;;) {
            const size_t k = next_item.fetch_add(1);
            if (k >= runs.size()) break;
            {
                std::lock_guard<std::mutex> lk(mu);
                if (error != FMA_OK) break;
            }
            const Run& run = runs[k];
            if (!run.has_backup && n_backup_runs && remap_delay_s > 0) {
                // Remap-only runs (kv_cache) have the whole copy time as slack, the weights run only the ring's worth
                // (~19 ms).  Driver VMM calls of ALL processes on the host serialise, so a rank that maps its kv early
                // delays another rank's weights mapping: give every rank's weights a head start.
                const double wait = t_entry + remap_delay_s - now_s();
                if (wait > 0) std::this_thread::sleep_for(std::chrono::duration<double>(wait));
            }
            if (!run.has_backup && remap_after_copy) {
                while (!copies_landed.load(std::memory_order_acquire)) {
                    {
                        std::lock_guard<std::mutex> lk(mu);
                        if (error != FMA_OK) break;
                    }
                    std::this_thread::sleep_for(std::chrono::microseconds(200));
                }
            }
            const bool is_ring = ring_run && k == 0;
            // gate class: whatever gates the first copy (ring, or the first backed-up item when there is no ring run) goes
            // first on the whole host; the other backed-up items have one ring's worth of slack; remap-only runs have what is
            // left of the copy time.
            const bool first_item = run.has_backup && k == 0;
            const int cls = first_item ? kGateFirst : run.has_backup ? std::min(kGateWeights + (int)k - (ring_run ? 1 : 0), kGateWeightsLast) : kGateRemap;
            const double left = std::max(0.0, t_entry + expected_copy_s * 0.8 - now_s());
            const double t_ask = now_s();
            int r;
            double t0;
            {
                GateHold hold(cls, cls >= kGateRemap ? left : std::min(left, 0.05));
                if (first_item) retract_gate();
                t0 = now_s();
                r = vmm_create_and_map(e->device, run.va, run.bytes);
            }
            const double t1 = now_s();
            map_ns.fetch_add((uint64_t)((t1 - t0) * 1e9));
            if (t0 - t_ask > 1e-4) e->tl_add("gate_wait", (int)k, t_ask, t0, 0);
            e->tl_add(is_ring ? "map_ring" : run.has_backup ? "map_backed" : "map_remap", (int)k, t0, t1, run.bytes);
            std::lock_guard<std::mutex> lk(mu);
            if (r != FMA_OK) {
                error = r;
                snprintf(msg, sizeof(msg), "%s", tl_err);
                if (is_ring) {  // the ring never came to exist
                    arena_give_back(e->arenas[run.arena], run.va - e->arenas[run.arena].base, run.bytes);
                    release_ring(e);
                }
            } else {
                Unit u;
                u.va = run.va; u.bytes = run.bytes; u.arena = run.arena;
                if (is_ring) u.zombies.emplace_back(run.va, run.bytes);  // ring VA returns to the arena when the unit is unmapped
                for (size_t i : run.segs) {
                    u.live_bytes += e->segs[i].bytes;
                    e->segs[i].mapped = true;
                    e->segs[i].unit_va = run.va;
                }
                // holes inside a run cannot exist (runs are VA-contiguous live segments), so bytes == live_bytes
                e->units[run.va] = u;
                item_done[k] = 1;
                while (done < runs.size() && item_done[done]) ++done;
            }
            cv.notify_all();
        }
    }
    int wait_mapped(size_t upto) {  // wait until items [0, upto) are mapped; the error code of a failed mapping (text in msg)
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return done >= upto || error != FMA_OK; });
        return error;
    }
    int wait(size_t upto) {  // the same, failing with the mapping's message
        const int mrc = wait_mapped(upto);
        return mrc == FMA_OK ? FMA_OK : fail(mrc, "%s", msg);
    }
    void retract_gate() {
        if (gate_first) gate_retract(gate_first);
        gate_first = 0;
    }
    void join() {
        for (auto& t : threads)
            if (t.joinable()) t.join();
    }
    ~Mapper() {  // the rollback of a failed wake
        if (committed) return;
        char keep[512];
        snprintf(keep, sizeof(keep), "%s", tl_err);
        {
            std::lock_guard<std::mutex> lk(mu);
            if (error == FMA_OK) error = FMA_ESTATE;   // the mapper threads stop
        }
        copies_landed.store(true, std::memory_order_release);
        join();
        retract_gate();
        cudaDeviceSynchronize();
        cudaGetLastError();
        for (size_t k = 0; k < runs.size(); ++k) {
            if (!item_done[k]) continue;
            for (size_t i : runs[k].segs) {
                e->segs[i].mapped = false;
                e->segs[i].unit_va = 0;
            }
            unmap_units(e, runs[k].va, runs[k].bytes);  // the ring run gives its VA back to the arena through its zombie entry
        }
        e->pending_events = 0;
        snprintf(tl_err, sizeof(tl_err), "%s", keep);
    }
};

// RESIDENT share: K2 / K5 copy the resident segments from e->res into their pages, on the kernel stream in pieces of at most one
// ring slot, each launched between two of the host part's launches once its destination is mapped (in the second half of the
// host part's launches the pipeline waits for that mapping); the tables sit behind the host part's in the same buffers.
struct ResidentRestore {
    fma_engine_t* e;
    Mapper& mapper;
    KernelTimes& kt;
    const std::vector<size_t>& with_res;
    const std::vector<size_t>& seg_run;
    uint64_t W_res;
    size_t n_host_pages;
    bool image_packed;             // WakePipe::packed clears the K5 error counter
    std::vector<Batch> pieces{};
    size_t next = 0;
    int setup();
    int launch_next();
    // after (host part's pages launched so far, host part's pages): launch the next piece if due
    int pump(size_t launched, size_t total) {
        if (next >= pieces.size()) return FMA_OK;
        if (2 * launched < total && mapper.done.load() < pieces[next].need) return FMA_OK;
        return launch_next();
    }
};

// What the copy pipelines of one wake share.  A pipeline enqueues the work that brings the backed-up segments'
// bytes from the store into their (re-)mapped runs; wait(n) blocks until the mapper has mapped work items [0, n).
struct WakePipe {
    fma_engine_t* e;
    const std::vector<size_t>& with_backup;   // segment indices that have a backup, image order
    const std::vector<size_t>& seg_run;       // segment -> index of its run in the mapper's work list
    uint64_t W;
    int tier;
    int mode;
    bool ring_run;                             // the staging ring is work item 0
    const char* store;
    KernelTimes& kt;
    uint32_t& copy_ops;
    double& first_copy_delay;
    double t_entry;
    Mapper& mapper;
    // pumped after each K2 / K5 launch: a RESIDENT share's restore launches a piece there (a slot's hand-back waits for one at most)
    ResidentRestore* between = nullptr;
    void copied() {
        if (!copy_ops) first_copy_delay = now_s() - t_entry;
        ++copy_ops;
    }
    int packed();
    int direct();
    int paged();
    int multipath();
};

// The segments `idx` as the page planner sees them: each waits for the mapper work item of its run.
std::vector<fma_layout::SegPages> wake_segs(const fma_engine_t* e, const std::vector<size_t>& idx, const std::vector<size_t>& seg_run) {
    std::vector<fma_layout::SegPages> v;
    for (size_t i : idx) v.push_back(fma_layout::SegPages{(uint64_t)e->segs[i].va, e->segs[i].bytes, e->segs[i].packed_off, seg_run[i] + 1});
    return v;
}

int ResidentRestore::setup() {
    if (!e->res.va) return fail(FMA_ESTATE, "the resident part of the image is gone");
    const size_t n_res = W_res / FMA_PAGE_BYTES, n_all = n_host_pages + n_res;
    RC(ensure_tables(e, n_all));
    if (e->res_packed) RC(ensure_pack_bufs(e, n_all));
    if (!e->ev_res_done && cudaEventCreateWithFlags(&e->ev_res_done, cudaEventDisableTiming) != cudaSuccess)
        return fail(FMA_ECUDA, "cudaEventCreate(resident) failed");
    std::vector<PagePlan> pages;
    uint64_t bad = 0;
    if (!fma_layout::plan_pages(wake_segs(e, with_res, seg_run), e->res_packed ? &e->res_off : nullptr, &e->res_bytes, &pages, &bad))
        return fail(FMA_ESTATE, "segment outside the resident part's page table");
    uint64_t* dst_tab = e->h_tab + n_host_pages;
    uint64_t* src_tab = e->h_tab + e->d_tab_cap + n_host_pages;
    for (size_t q = 0; q < pages.size(); ++q) {
        if (e->res_packed) {
            set_pack_desc(e->h_pdesc[n_host_pages + q], (uint64_t)e->res.va + pages[q].off, pages[q].va, pages[q].bytes);
        } else {
            dst_tab[q] = pages[q].va;
            src_tab[q] = (uint64_t)e->res.va + pages[q].off;
        }
    }
    fma_layout::plan_batches(pages, slot_pages(e), UINT64_MAX, false, &pieces);
    if (e->res_packed) {
        RT(cudaMemcpyAsync(e->d_pdesc + n_host_pages, e->h_pdesc + n_host_pages, n_res * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
        if (!image_packed) RT(cudaMemsetAsync(e->d_psize + e->pdesc_cap, 0, sizeof(uint32_t), e->ks));   // (WakePipe::packed clears it otherwise)
    } else {
        RT(cudaMemcpyAsync(e->d_tab + n_host_pages, dst_tab, n_res * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
        RT(cudaMemcpyAsync(e->d_tab + e->d_tab_cap + n_host_pages, src_tab, n_res * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    }
    return FMA_OK;
}

int ResidentRestore::launch_next() {
    const Batch& pc = pieces[next];
    RC(mapper.wait(pc.need));
    int r;
    kt.kind = "res_restore";
    if (e->res_packed) {
        r = kt.begin();
        if (r == FMA_OK) {
            cudaError_t ce = fma_k_launch_unpack(e->d_pdesc + n_host_pages + pc.p0, (uint32_t)pc.np, e->d_psize + e->pdesc_cap, e->ks);
            r = ce == cudaSuccess ? kt.end((uint64_t)pc.np * FMA_PAGE_BYTES + pc.stored) : fail(FMA_ECUDA, "K5 (resident) launch failed: %s", cudaGetErrorString(ce));
        }
    } else {
        r = kt.launch(e->d_tab + e->d_tab_cap + n_host_pages + pc.p0, 0, e->d_tab + n_host_pages + pc.p0, 0, (uint32_t)pc.np);
    }
    kt.kind = "kernel";
    if (r != FMA_OK) return r;
    if (++next == pieces.size()) RT(cudaEventRecord(e->ev_res_done, e->ks));
    return FMA_OK;
}

// PACKED image: H2D of the stored pages (0.758 of the bytes) -> ring slot -> K5 decode + scatter; or K5 reads the store itself
int WakePipe::packed() {
    // K5 reads the store itself when it is peer / local HBM, or when no ring could be had (then over PCIe)
    const bool zero_copy = mode != FMA_MODE_STAGED;
    if (zero_copy && tier == FMA_TIER_HOST && !e->host.dev_alias)
        return fail(FMA_ENOMEM, "no HBM for a staging ring and the host store has no device alias: a packed image cannot be woken");
    std::vector<PagePlan> pages;
    uint64_t bad = 0;
    if (!fma_layout::plan_pages(wake_segs(e, with_backup, seg_run), &e->img_off, &e->img_bytes, &pages, &bad))
        return fail(FMA_ESTATE, "segment at image offset %llu is outside the packed image's page table", (unsigned long long)bad);
    const size_t n_pages = pages.size();
    RC(ensure_pack_bufs(e, n_pages));
    uint32_t* d_err = e->d_psize + e->pdesc_cap;
    RT(cudaMemsetAsync(d_err, 0, sizeof(uint32_t), e->ks));
    if (!zero_copy) {
        if (ring_run) RC(mapper.wait(1));   // (else the route has the ring)
        std::vector<Batch> slots;  // pages that are adjacent in the store and fit one ring slot
        if (!fma_layout::plan_batches(pages, SIZE_MAX, e->ring_slot_bytes, true, &slots))
            return fail(FMA_EINVAL, "ring slot of %zu bytes cannot hold one page", e->ring_slot_bytes);
        for (size_t c = 0; c < slots.size(); ++c)
            for (size_t q = slots[c].p0; q < slots[c].p0 + slots[c].np; ++q)
                set_pack_desc(e->h_pdesc[q], (uint64_t)(uintptr_t)e->ring[c % e->n_ring] + (pages[q].off - pages[slots[c].p0].off), pages[q].va, pages[q].bytes);
        RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, n_pages * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
        for (size_t c = 0; c < slots.size(); ++c) {
            const Batch& sl = slots[c];
            const int slot = (int)(c % e->n_ring);
            cudaStream_t cstream = e->cs[c % e->n_cs];
            if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[slot], 0));
            RT(cudaMemcpyAsync(e->ring[slot], store + pages[sl.p0].off, sl.stored, cudaMemcpyDefault, cstream));
            copied();
            RT(cudaEventRecord(e->ev_ring_full[slot], cstream));
            RC(mapper.wait(sl.need));
            RT(cudaStreamWaitEvent(e->ks, e->ev_ring_full[slot], 0));
            RC(kt.begin());
            RT(fma_k_launch_unpack(e->d_pdesc + sl.p0, (uint32_t)sl.np, d_err, e->ks));
            RC(kt.end((uint64_t)sl.np * FMA_PAGE_BYTES + sl.stored));
            RT(cudaEventRecord(e->ev_ring_free[slot], e->ks));
            if (between) RC(between->pump(sl.p0 + sl.np, n_pages));
        }
    } else {
        const uint64_t sbase = store_dev_base(e, tier);
        for (size_t q = 0; q < n_pages; ++q) set_pack_desc(e->h_pdesc[q], sbase + pages[q].off, pages[q].va, pages[q].bytes);
        RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, n_pages * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
        std::vector<Batch> batches;
        fma_layout::plan_batches(pages, slot_pages(e), UINT64_MAX, false, &batches);
        for (const Batch& b : batches) {
            RC(mapper.wait(b.need));
            RC(kt.begin());
            RT(fma_k_launch_unpack(e->d_pdesc + b.p0, (uint32_t)b.np, d_err, e->ks));
            RC(kt.end((uint64_t)b.np * FMA_PAGE_BYTES + b.stored));
            copied();
            if (between) RC(between->pump(b.p0 + b.np, n_pages));
        }
    }
    return FMA_OK;
}

// DIRECT: copy engines move each chunk of the image straight into its segment as soon as the segment is mapped
int WakePipe::direct() {
    const size_t chunk = direct_chunk(e);
    int k = 0;
    for (size_t i : with_backup) {
        RC(mapper.wait(seg_run[i] + 1));
        const Segment& s = e->segs[i];
        for (size_t o = 0; o < s.bytes; o += chunk, ++k) {
            const size_t n = std::min(chunk, s.bytes - o);
            RT(cudaMemcpyAsync(reinterpret_cast<void*>(s.va + o), store + s.packed_off + o, n, cudaMemcpyDefault,
                                    e->cs[k % e->n_cs]));
            copied();
        }
    }
    return FMA_OK;
}

// KERNEL / STAGED: page-table driven — K2 reads the store itself, or H2D -> ring slot -> K2 scatter
int WakePipe::paged() {
    // page table of the DESTINATIONS in image order (== with_backup order only if every backed-up segment is woken), with the
    // latest work item each page needs
    std::vector<PagePlan> pages;
    uint64_t bad = 0;
    fma_layout::plan_pages(wake_segs(e, with_backup, seg_run), nullptr, nullptr, &pages, &bad);
    const size_t n_pages = pages.size();
    RC(ensure_tables(e, n_pages));
    uint64_t* dst_tab = e->h_tab;                 // destination page addresses
    uint64_t* src_tab = e->h_tab + e->d_tab_cap;  // source page addresses inside the store (may be sparse)
    const uint64_t sbase = store_dev_base(e, tier);
    for (size_t p = 0; p < n_pages; ++p) {
        dst_tab[p] = pages[p].va;
        src_tab[p] = sbase + pages[p].off;
    }
    RT(cudaMemcpyAsync(e->d_tab, dst_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemcpyAsync(e->d_tab + e->d_tab_cap, src_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    const uint64_t* d_dst = e->d_tab;
    const uint64_t* d_src = e->d_tab + e->d_tab_cap;
    if (mode == FMA_MODE_KERNEL) {
        // K2 reads the store itself (zero-copy PCIe reads, or NVLink/HBM loads); launch batches as the
        // mapper makes progress so the scatter overlaps cuMemCreate/Map of later segments
        for (size_t p0 = 0; p0 < n_pages;) {
            Batch b = fma_layout::next_batch(pages, p0, slot_pages(e), UINT64_MAX, false);
            RC(mapper.wait(b.need));
            // opportunistically extend the batch over everything already mapped
            const size_t have = mapper.done.load();
            while (p0 + b.np < n_pages && pages[p0 + b.np].need <= have) ++b.np;
            RC(kt.launch(d_src + p0, 0, d_dst + p0, 0, (uint32_t)b.np));
            copied();
            p0 += b.np;
            if (between) RC(between->pump(p0, n_pages));
        }
    } else {  // STAGED: copy engine H2D store -> ring slot (starts at t=0), K2 scatter once the targets are mapped
        if (ring_run) RC(mapper.wait(1));  // the ring is run 0 (1 GiB, ~0.2 ms to map): wait for it before the first H2D
        // the store image may be only partially woken; H2D works on runs that are contiguous in the store
        std::vector<Batch> slots;
        if (!fma_layout::plan_batches(pages, e->ring_slot_bytes / FMA_PAGE_BYTES, UINT64_MAX, true, &slots))
            return fail(FMA_EINVAL, "ring slot of %zu bytes cannot hold one page", e->ring_slot_bytes);
        for (size_t c = 0; c < slots.size(); ++c) {
            const Batch& sl = slots[c];
            const int slot = (int)(c % e->n_ring);
            cudaStream_t cstream = e->cs[c % e->n_cs];
            if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[slot], 0));
            RT(cudaMemcpyAsync(e->ring[slot], store + pages[sl.p0].off, sl.stored, cudaMemcpyDefault, cstream));
            copied();
            RT(cudaEventRecord(e->ev_ring_full[slot], cstream));
            RC(mapper.wait(sl.need));
            RT(cudaStreamWaitEvent(e->ks, e->ev_ring_full[slot], 0));
            RC(kt.launch(nullptr, (uint64_t)(uintptr_t)e->ring[slot], d_dst + sl.p0, 0, (uint32_t)sl.np));
            RT(cudaEventRecord(e->ev_ring_free[slot], e->ks));
            if (between) RC(between->pump(sl.p0 + sl.np, n_pages));
        }
    }
    return FMA_OK;
}

// MULTI-PATH (fma_paths_set): the host image is cut into chunks; every path — the engine's own PCIe link and one per idle peer
// GPU — pulls the next chunk whenever one of its staging slots is free (H2D by THAT GPU's copy engine over THAT GPU's x16
// link), and K2 on the waking GPU gathers the chunk from the path's staging slot (own HBM, or the peer's HBM over NVLink) into
// the destination pages.  Self-balancing: a slower path (other NUMA node, busy link) simply takes fewer chunks.
int WakePipe::multipath() {
    std::vector<PagePlan> pages;
    uint64_t bad = 0;
    fma_layout::plan_pages(wake_segs(e, with_backup, seg_run), nullptr, nullptr, &pages, &bad);
    const size_t n_pages = pages.size();
    RC(ensure_tables(e, n_pages));
    for (size_t p = 0; p < n_pages; ++p) e->h_tab[p] = pages[p].va;
    RT(cudaMemcpyAsync(e->d_tab, e->h_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    RC(ensure_ring_events(e, 1));
    cudaEvent_t ev_tab = e->ev_ring_full[0];   // the page table must be on the device before any path's K2 reads it
    RT(cudaEventRecord(ev_tab, e->ks));
    std::vector<Batch> chunks;
    fma_layout::plan_batches(pages, std::max<size_t>(e->path_slot_bytes / FMA_PAGE_BYTES, 1), UINT64_MAX, true, &chunks);
    std::vector<uint64_t> chunk_off;
    for (const Batch& ch : chunks) chunk_off.push_back(pages[ch.p0].off);
    // a path drains the chunk queue of ITS GPU's NUMA node first and then helps with the others (HostStore::ranges)
    fma_layout::ChunkQueues queues(chunk_off, e->host.ranges);
    // REMOTE paths (fma_paths_attach): helpers in the node-level owner's process pull from the SAME work counter, which therefore
    // lives in the shared mailbox together with the chunk table of this wake (fma_pull.h); published with the generation bump.
    PullMailbox* mb = e->mbox;
    if (mb) {
        if (chunks.size() > kPullMaxChunks) RC(fail(FMA_EINVAL, "%zu chunks exceed the mailbox's table (use larger path slots)", chunks.size()));
        for (size_t c = 0; c < chunks.size(); ++c) mb->chunks[c] = PullChunk{chunk_off[c], (uint32_t)chunks[c].stored, 0};
        for (uint32_t pi = 0; pi < kPullMaxPaths; ++pi) {
            mb->helper_error[pi].store(0);
            mb->helper_seen[pi].store(0);
            for (uint32_t sl = 0; sl < kPullMaxSlots; ++sl) mb->slot_state[pi][sl].store(0);
        }
        mb->abort.store(0);
        mb->next_chunk.store(0);
        mb->n_chunks.store((uint32_t)chunks.size());
        mb->generation.store(++e->pull_generation, std::memory_order_release);   // the helpers start pulling here
    }
    auto take_chunk = [&](int my_node, size_t* out) -> bool {
        if (mb) {
            const uint32_t k = mb->next_chunk.fetch_add(1);
            if (k >= chunks.size()) return false;
            *out = k;
            return true;
        }
        return queues.take(my_node, out);
    };
    std::atomic<int> error{FMA_OK};
    std::atomic<bool> first_copy_seen{false};
    std::mutex kt_mu;
    char err_msg[512] = "";
    std::vector<uint32_t> per_path(e->paths.size(), 0), per_path_local(e->paths.size(), 0);
    auto worker = [&](size_t pi) {
        WakePath& path = e->paths[pi];
        cudaSetDevice(e->device);
        auto failw = [&](int code, const char* what, cudaError_t ce) {
            int expect = FMA_OK;
            if (error.compare_exchange_strong(expect, code)) snprintf(err_msg, sizeof(err_msg), "%s failed on path %zu (device %d): %s", what, pi, path.device, ce == cudaSuccess ? (code == FMA_ESTATE || code == FMA_EINTEGRITY ? what : mapper.msg) : cudaGetErrorString(ce));
        };
        cudaError_t ce = cudaStreamWaitEvent(path.kern, ev_tab, 0);
        if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaStreamWaitEvent(table)", ce);
        uint32_t mine = 0;
        if (path.remote) {
            // The owner's helper fills this path's slots in sequence and publishes "chunk c has landed" per slot; K2 gathers the slot
            // over NVLink and the slot is handed back as soon as that K2 has completed (checked without blocking).
            std::atomic<uint32_t>* state = mb->slot_state[pi];
            bool busy[kMaxRing] = {};
            const double patience = std::max(2.0, (double)env_int("FMA_PULL_TIMEOUT_S", 5));
            double t_last = now_s();
            for (;;) {
                if (error.load() != FMA_OK || mb->abort.load()) {
                    if (error.load() == FMA_OK) failw(FMA_ESTATE, "the owner's helper aborted the pull", cudaSuccess);
                    return;
                }
                bool progressed = false;
                for (int sl = 0; sl < e->path_slots; ++sl)      // hand drained slots back
                    if (busy[sl]) {
                        cudaError_t q = cudaEventQuery(path.ev_free[sl]);
                        if (q == cudaSuccess) {
                            busy[sl] = false;
                            state[sl].store(0, std::memory_order_release);
                            progressed = true;
                        } else if (q != cudaErrorNotReady) {
                            return failw(FMA_ECUDA, "K2 on a remote slot", q);
                        } else {
                            cudaGetLastError();
                        }
                    }
                const int slot = (int)(mine % (uint32_t)e->path_slots);
                uint32_t st = busy[slot] ? 0 : state[slot].load(std::memory_order_acquire);
                if (st != 0 && !pull_word_is_of(st, e->pull_generation)) {   // left behind by a helper of an earlier, aborted wake: not ours
                    state[slot].compare_exchange_strong(st, 0, std::memory_order_acq_rel);
                    st = 0;
                }
                st = pull_word_value(st);
                if (st == kPullDoneValue) break;
                // nobody serves this path (no pull request reached the owner, or it came too late) and the other paths have taken
                // every chunk: nothing will ever arrive here — the wake completes over the paths that did work
                if (st == 0 && mb->next_chunk.load() >= chunks.size() && mb->helper_seen[pi].load(std::memory_order_acquire) != e->pull_generation) {
                    bool any_busy = false;
                    for (int sl = 0; sl < e->path_slots; ++sl) any_busy = any_busy || busy[sl];
                    if (!any_busy) break;
                }
                if (st != 0) {
                    const size_t c = st - 1;
                    if (c >= chunks.size()) return failw(FMA_EINTEGRITY, "the mailbox names a chunk that does not exist", cudaSuccess);
                    const Batch& ch = chunks[c];
                    const int mrc = mapper.wait_mapped(ch.need);
                    if (mrc != FMA_OK) return failw(mrc, "mapping", cudaSuccess);
                    char* slot_ptr = reinterpret_cast<char*>(path.staging.va) + (size_t)slot * e->path_slot_bytes;
                    {
                        std::lock_guard<std::mutex> lk(kt_mu);
                        const int krc = kt.launch_on(path.kern, nullptr, (uint64_t)(uintptr_t)slot_ptr, e->d_tab + ch.p0, 0, (uint32_t)ch.np);
                        if (krc != FMA_OK) return failw(krc, "K2 launch", cudaGetLastError());
                    }
                    ce = cudaEventRecord(path.ev_free[slot], path.kern);
                    if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot drained)", ce);
                    busy[slot] = true;
                    if (!first_copy_seen.exchange(true)) first_copy_delay = now_s() - t_entry;
                    ++mine;
                    progressed = true;
                }
                if (progressed) {
                    t_last = now_s();
                } else {
                    if (now_s() - t_last > patience) return failw(FMA_ESTATE, "no chunk from the owner's helper within the timeout (is the pull request running?)", cudaSuccess);
                    std::this_thread::sleep_for(std::chrono::microseconds(20));
                }
            }
            per_path[pi] = mine;
            ce = cudaEventRecord(path.ev_done, path.kern);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(done)", ce);
            return;
        }
        for (;;) {
            if (error.load() != FMA_OK) return;
            size_t c = 0;
            if (!take_chunk(path.numa_node, &c)) break;
            const Batch& ch = chunks[c];
            {
                const uint64_t off = chunk_off[c];
                for (const HostStore::NumaRange& r : e->host.ranges)
                    if (off >= r.begin && off < r.end && r.node == path.numa_node) ++per_path_local[pi];
            }
            const int slot = (int)(mine % (uint32_t)e->path_slots);
            if (mine >= (uint32_t)e->path_slots) {   // K2 has read the chunk that used this slot before
                ce = cudaEventSynchronize(path.ev_free[slot]);
                if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventSynchronize(slot free)", ce);
            }
            char* slot_ptr = reinterpret_cast<char*>(path.staging.va) + (size_t)slot * e->path_slot_bytes;
            ce = cudaMemcpyAsync(slot_ptr, store + chunk_off[c], ch.stored, cudaMemcpyDefault, path.copy);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaMemcpyAsync(H2D)", ce);
            if (!first_copy_seen.exchange(true)) first_copy_delay = now_s() - t_entry;
            ce = cudaEventRecord(path.ev_full[slot], path.copy);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot full)", ce);
            const int mrc = mapper.wait_mapped(ch.need);
            if (mrc != FMA_OK) return failw(mrc, "mapping", cudaSuccess);
            ce = cudaStreamWaitEvent(path.kern, path.ev_full[slot], 0);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaStreamWaitEvent(slot full)", ce);
            {
                std::lock_guard<std::mutex> lk(kt_mu);
                const int krc = kt.launch_on(path.kern, nullptr, (uint64_t)(uintptr_t)slot_ptr, e->d_tab + ch.p0, 0, (uint32_t)ch.np);
                if (krc != FMA_OK) return failw(krc, "K2 launch", cudaGetLastError());
            }
            ce = cudaEventRecord(path.ev_free[slot], path.kern);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot free)", ce);
            ++mine;
        }
        per_path[pi] = mine;
        ce = cudaEventRecord(path.ev_done, path.kern);
        if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(done)", ce);
    };
    std::vector<std::thread> th;
    for (size_t pi = 0; pi < e->paths.size(); ++pi) th.emplace_back(worker, pi);
    for (auto& t : th) t.join();
    if (error.load() != FMA_OK) {
        if (mb) mb->abort.store(1);                                          // the owner's helpers stop pulling
        for (WakePath& path : e->paths)
            if (path.copy) cudaStreamSynchronize(path.copy);                 // nothing may still be writing the staging slots
        return fail(error.load(), "%s", err_msg);
    }
    for (size_t pi = 0; pi < e->paths.size(); ++pi) {
        RT(cudaStreamWaitEvent(e->ks, e->paths[pi].ev_done, 0));   // the wake's device-time bracket and the final sync cover every path
        copy_ops += per_path[pi];
        const int idx = e->paths[pi].remote ? -(int)pi : e->paths[pi].device;   // remote paths: -(path index), their GPU is not visible here
        e->tl_add("path_chunks", idx, t_entry, now_s(), (uint64_t)per_path[pi] * e->path_slot_bytes);
        e->tl_add("path_local", idx, t_entry, now_s(), (uint64_t)per_path_local[pi] * e->path_slot_bytes);
    }
    return FMA_OK;
}

// A RESIDENT share's segments: their bytes are in e->res, their offsets in the resident part.
bool is_resident(const fma_engine_t* e, const Segment& s) { return s.has_backup && s.backup_tier == FMA_TIER_LOCAL && e->image_tier == FMA_TIER_HOST; }

// Work list: RUNS — maximal VA-contiguous groups of sleeping segments of one arena — so a whole tag is re-created with one
// cuMemCreate + cuMemMap + cuMemSetAccess.  Runs that have a backup come first, in image order (they gate the copy pipeline);
// remap-only runs (e.g. kv_cache) are mapped after them.  No runs: nothing to wake.
int plan_wake_runs(fma_engine_t* e, uint64_t tag_mask, double t_entry, std::vector<Run>* runs) {
    std::vector<size_t> cand;
    for (size_t i = 0; i < e->segs.size(); ++i) {
        const Segment& s = e->segs[i];
        if (s.mapped) continue;                                  // idempotent: already awake
        if (tag_mask && !tag_bit_set(tag_mask, s.tag)) continue;  // tags is None or data.tag in tags (cumem.py:238)
        cand.push_back(i);
    }
    if (cand.empty()) return FMA_OK;
    RC(check_tma_shape(e, e->image_tier));
    e->tl_begin("wake", t_entry);
    std::sort(cand.begin(), cand.end(), [&](size_t a, size_t b) {
        const Segment &x = e->segs[a], &y = e->segs[b];
        return x.arena != y.arena ? x.arena < y.arena : x.va < y.va;
    });
    std::vector<fma_layout::SegView> view;
    for (size_t i : cand) {
        const Segment& s = e->segs[i];
        // a RESIDENT share's segments (their offsets are in the resident part) are mapped after the host part's
        const uint64_t key = is_resident(e, s) ? (1ull << 62) + s.packed_off : s.packed_off;
        view.push_back(fma_layout::SegView{i, s.arena, (uint64_t)s.va, s.bytes, s.has_backup, key});
    }
    // FMA_MAP_PIECE_MIB (default 2048; 0 = whole runs): backed-up runs are mapped in pieces of about that size, cut at segment
    // boundaries.  One 15 GiB mapping has only the ring's slack of a few milliseconds, and a shared host's driver calls
    // sometimes stall for tens of milliseconds; with pieces K2 starts on the first piece and every later call has the copy
    // time of the pieces before it as slack.
    *runs = fma_layout::plan_runs(view, env_int("FMA_MERGE_RUNS", 1) != 0, (size_t)std::max(env_int("FMA_MAP_PIECE_MIB", 2048), 0) << 20);
    return FMA_OK;
}

// Staging ring.  Steady state: the ring is its OWN small run (2 x 512 MiB) placed right after the first backed-up
// run at the arena's bump pointer and mapped FIRST — a 1 GiB cuMemCreate/Map/SetAccess costs ~0.2 ms, the H2D
// stream starts as soon as it exists, and the big weights run (whose mapping takes 1.4 ms alone but tens of ms
// when 8 ranks wake at once) keeps the ring's ~19 ms of slack.  At the next sleep the ring goes with a cuMemUnmap
// like every other unit: no cudaMalloc / cudaFree anywhere (a cudaFree of 1 GiB stalls 0.8-300 ms on these hosts).
// Needs the run to end at its arena's bump pointer; otherwise (or FMA_RING_ATTACH=0) one cudaMalloc provides it.
// Either way the ring must exist BEFORE the other runs start taking HBM.  false: HBM too full for a ring.
bool ring_for_wake(fma_engine_t* e, std::vector<Run>& runs, uint64_t w_bytes, bool* ring_run) {
    if (!e->n_ring) {
        const Run& r0 = runs[0];
        Arena& a = e->arenas[r0.arena];
        const size_t slot = ring_slot_for(e, w_bytes);
        const size_t total = slot * ring_slots_for(e);
        // end of the VA-contiguous chain of backed-up runs that starts with the first one (one run, or its pieces)
        uint64_t chain_end = r0.va + r0.bytes;
        for (size_t k = 1; k < runs.size() && runs[k].has_backup && runs[k].arena == r0.arena && runs[k].va == chain_end; ++k) chain_end += runs[k].bytes;
        const bool at_top = r0.has_backup && (chain_end == a.base + a.top) && a.top + total <= a.cap;
        if (at_top && env_int("FMA_RING_ATTACH", 1) != 0 && ensure_ring_events(e, ring_slots_for(e)) == FMA_OK) {
            Run rr;
            rr.va = chain_end; rr.bytes = total; rr.arena = r0.arena; rr.has_backup = true; rr.first_off = 0;  // no segments
            a.top += total;  // later allocations of this tag land after the ring; the range returns at unmap
            e->n_ring = ring_slots_for(e);
            e->ring_slot_bytes = slot;
            e->ring_attached = true;
            e->ring_unit_va = rr.va;
            for (int i = 0; i < e->n_ring; ++i) e->ring[i] = reinterpret_cast<void*>(rr.va + (size_t)i * slot);
            runs.insert(runs.begin(), std::move(rr));
            *ring_run = true;
            return true;
        }
    }
    return ensure_ring(e, w_bytes) == FMA_OK;  // (else copy engines go straight into the runs)
}

// FMA_FLAG_VERIFY: every restored segment against its digest from before the sleep
int verify_wake(fma_engine_t* e, const std::vector<size_t>& with_backup, int* verify_rc) {
    std::vector<size_t> idx;
    for (size_t i : with_backup)
        if (e->segs[i].digest_valid) idx.push_back(i);
    std::vector<uint64_t> dg;
    RC(digest_segments(e, idx, &dg));
    for (size_t k = 0; k < idx.size(); ++k)
        if (dg[k] != e->segs[idx[k]].digest)
            *verify_rc = fail(FMA_EINTEGRITY, "segment %zu (va 0x%llx): digest %016llx after wake != %016llx before sleep", idx[k],
                              (unsigned long long)e->segs[idx[k]].va, (unsigned long long)dg[k], (unsigned long long)e->segs[idx[k]].digest);
    return FMA_OK;
}

// data.cpu_backup_tensor = None (cumem.py:249), unless FMA_FLAG_KEEP_BACKUP
void drop_backups(fma_engine_t* e, const std::vector<size_t>& with_backup, uint64_t W, int tier, bool verified) {
    for (size_t i : with_backup) {
        Segment& s = e->segs[i];
        // INCREMENTAL sleep: the host store keeps these bytes; remember where, together with their digest
        const bool kept = s.digest_valid && verified && !is_resident(e, s);   // (the resident buffer does not outlive the wake)
        s.shadow_off = kept ? s.packed_off : kNoOffset;   // host store or parking buffer: both outlive the wake
        s.has_backup = false;
        s.packed_off = kNoOffset;
    }
    if (W) {
        e->shadow_tier = tier;
        e->shadow_packed = e->image_packed;
        e->shadow_store_bytes = e->image_store_bytes;
        e->shadow_image_bytes = e->image_bytes;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------
// WAKE
// ------------------------------------------------------------------------------------
int do_wake(fma_engine_t* e, uint64_t tag_mask, uint32_t flags) {
    DeviceGuard guard(e->device);
    RC(flush_kernel_times(e));
    const double t_entry = now_s();
    RC(ensure_streams(e));
    std::vector<Run> runs;
    RC(plan_wake_runs(e, tag_mask, t_entry, &runs));
    if (runs.empty()) return FMA_OK;
    const int tier = e->image_tier;

    std::vector<size_t> with_backup, with_host, with_res;  // segment indices, image order; with_backup by store: host part, RESIDENT share
    std::vector<size_t> seg_run(e->segs.size(), 0);       // segment -> index of its run in `runs`
    uint64_t W = 0, W_res = 0, remapped_only = 0;         // W: what crosses the link (a resident share's segments do not)
    for (size_t r = 0; r < runs.size(); ++r) {
        for (size_t i : runs[r].segs) {
            seg_run[i] = r;
            if (!runs[r].has_backup) {
                remapped_only += e->segs[i].bytes;
                continue;
            }
            with_backup.push_back(i);
            const bool res = is_resident(e, e->segs[i]);
            (res ? with_res : with_host).push_back(i);
            (res ? W_res : W) += e->segs[i].bytes;
        }
    }
    fma_layout::WakeFacts facts{tier, fma_layout::resolve_mode(e->cfg.mode, tier), e->image_packed, !e->paths.empty(), W != 0, no_ring()};
    bool ring_run = false;
    if (fma_layout::wake_route(facts).wants_ring) facts.ring = ring_for_wake(e, runs, W, &ring_run);
    if (ring_run)  // the ring became run 0
        for (size_t& r : seg_run) ++r;
    const fma_layout::WakeRoute route = fma_layout::wake_route(facts);
    const bool dbg_t = env_int("FMA_DEBUG_TIMING", 0) != 0;
    const double t_ring = now_s();
    e->tl_add("plan", (int)runs.size(), t_entry, t_ring, 0);
    Mapper mapper{e, runs, ring_run, t_entry};
    // expected copy time of the host part: 55 GB/s per host-tier link (a multi-path wake has as many links as paths), 600 GB/s over NVLink
    mapper.start(tier, (double)W / (tier == FMA_TIER_HOST ? 55e9 * (route.pipe == fma_layout::WakePipeKind::Multipath ? (double)e->paths.size() : 1.0) : 600e9));

    // ---- copy pipeline --------------------------------------------------------------------------
    CopyTimer timer{e};
    KernelTimes kt{e};
    uint32_t copy_ops = 0;
    double copy_s = 0, first_copy_delay = 0;
    ResidentRestore res{e, mapper, kt, with_res, seg_run, W_res, W / FMA_PAGE_BYTES, facts.image_packed};
    const bool res_packed = W_res && e->res_packed;   // (the buffer may be released before the K5 error count is read)
    if (W || W_res) {
        const char* store = static_cast<const char*>(store_copy_base(e, tier));
        if (W && !store) return fail(FMA_ESTATE, "backup store of tier %d is gone", tier);
        if (W && tier == FMA_TIER_HOST && route.mode == FMA_MODE_KERNEL && !e->host.dev_alias)
            return fail(FMA_ECUDA, "host store has no device alias for zero-copy mode");
        RC(timer.begin());
        if (W_res) RC(res.setup());
        if (W) {
            WakePipe pipe{e, with_host, seg_run, W, tier, route.mode, ring_run, store, kt, copy_ops, first_copy_delay, t_entry, mapper, W_res ? &res : nullptr};
            const double t_enq0 = now_s();
            switch (route.pipe) {
            case fma_layout::WakePipeKind::PackedRing: case fma_layout::WakePipeKind::PackedZeroCopy: RC(pipe.packed()); break;
            case fma_layout::WakePipeKind::Multipath: RC(pipe.multipath()); break;
            case fma_layout::WakePipeKind::Direct: RC(pipe.direct()); break;
            case fma_layout::WakePipeKind::Kernel: case fma_layout::WakePipeKind::Staged: RC(pipe.paged()); break;
            }
            e->tl_add("enqueue", (int)copy_ops, t_enq0, now_s(), W);
        }
        while (res.next < res.pieces.size()) RC(res.launch_next());   // what the host part's launches left (or had no room for)
    }
    if (mapper.remap_after_copy && W) {  // let the DMA finish before the remap-only runs are touched
        const double t_w0 = now_s();
        for (int i = 0; i < e->n_cs; ++i) RT(cudaStreamSynchronize(e->cs[i]));
        RT(cudaStreamSynchronize(e->ks));
        e->tl_add("copies_landed", 0, t_w0, now_s(), W);
    }
    mapper.copies_landed.store(true, std::memory_order_release);
    // every requested segment must be mapped before wake returns (cumem.py:237-240)
    {
        const double t_w0 = now_s();
        RC(mapper.wait(runs.size()));
        e->tl_add("wait_all_mapped", (int)runs.size(), t_w0, now_s(), 0);
    }
    mapper.join();
    mapper.retract_gate();
    // RESIDENT share: the buffer goes once its restore has completed and every run is mapped (a wake that fails before that is
    // rolled back and its retry needs the buffer), under the host part's copy; it stays while a resident segment still sleeps
    // (tag-selective wake) and with FMA_FLAG_KEEP_BACKUP.
    if (e->res.va && !(flags & FMA_FLAG_KEEP_BACKUP)) {
        bool still_asleep = false;
        for (const Segment& s : e->segs) still_asleep = still_asleep || (is_resident(e, s) && !s.mapped);
        if (!still_asleep) {
            if (res.next) RT(cudaEventSynchronize(e->ev_res_done));
            const double a = now_s();
            const uint64_t cap = e->res.bytes;
            {
                GateHold hold(kGateUnmap, 0.1);
                resident_release(e);
            }
            e->tl_add("res_free", 0, a, now_s(), cap);
        }
    }
    const double t_joined = now_s();
    double t_copy_end = t_joined;
    if (W || W_res) {
        RC(timer.end(&copy_s));
        e->tl_add("drain", 0, t_joined, now_s(), W);
        RC(kt.collect());
        if (facts.image_packed || res_packed)  // K5 counts stored pages it could not read (bad magic / count): the image is damaged
            RC(check_pack_errors(e, "%u stored page(s) of the packed image are malformed"));
        t_copy_end = now_s();
    }
    if (dbg_t)
        fprintf(stderr, "[fma] wake phases: plan+ring %.1f ms | enqueue+map-wait %.1f ms | drain %.1f ms | ring free %.1f ms | runs %zu\n",
                (t_ring - t_entry) * 1e3, (t_joined - t_ring) * 1e3, (t_copy_end - t_joined) * 1e3, (now_s() - t_copy_end) * 1e3, runs.size());
    mapper.committed = true;

    int verify_rc = FMA_OK;
    if ((flags & FMA_FLAG_VERIFY) && (W || W_res)) RC(verify_wake(e, with_backup, &verify_rc));
    if (!(flags & FMA_FLAG_KEEP_BACKUP)) drop_backups(e, with_backup, W, tier, verify_rc == FMA_OK);

    e->tl_add("total", 0, t_entry, now_s(), W + W_res);
    e->st.wake_seconds = now_s() - t_entry;
    e->st.wake_copy_seconds = copy_s;
    e->st.wake_map_seconds = mapper.map_ns.load() * 1e-9;
    e->st.wake_first_copy_delay = first_copy_delay;
    e->st.wake_bytes_restored = W + W_res;
    e->st.wake_bytes_remapped_only = remapped_only;
    e->st.copy_ops = copy_ops;
    e->st.total_copy_ops += copy_ops;
    e->st.tier = tier;
    e->st.mode = route.mode;
    if (!W && !W_res) zero_kernel_stats(e);
    return verify_rc;
}

}  // namespace fma_impl
