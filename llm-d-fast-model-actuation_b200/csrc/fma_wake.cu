// fma_wake.cu — WAKE: vllm:device_allocator/cumem.py:227-249 -> do_wake
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"
#include "fma_gate.h"

namespace fma_impl {

namespace {

// What the copy pipelines of one wake share.  A pipeline enqueues the work that brings the backed-up segments'
// bytes from the store into their (re-)mapped runs; wait_mapped(n) blocks until the mapper thread has mapped work
// items [0, n) (or failed: the error code comes back, its text is in map_msg).
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
    std::function<int(size_t)> wait_mapped;
    std::function<size_t()> mapped_now;
    const char* map_msg;
};

#define PIPE_CHECK(x)                 \
    do {                              \
        int _rc = (x);                \
        if (_rc != FMA_OK) return _rc; \
    } while (0)

// PACKED image: H2D of the stored pages (0.758 of the bytes) -> ring slot -> K5 decode + scatter; or K5 reads the store itself
int wake_packed(WakePipe& pipe) {
    fma_engine_t* e = pipe.e;
    const std::vector<size_t>& with_backup = pipe.with_backup;
    const std::vector<size_t>& seg_run = pipe.seg_run;
    KernelTimes& kt = pipe.kt;
    uint32_t& copy_ops = pipe.copy_ops;
    double& first_copy_delay = pipe.first_copy_delay;
    const double t_entry = pipe.t_entry;
    const int tier = pipe.tier;
    const int mode = pipe.mode;
    const bool ring_run = pipe.ring_run;
    const char* store = pipe.store;
    const uint64_t W = pipe.W;
    auto wait_mapped = [&](size_t upto) { return pipe.wait_mapped(upto); };
    // ---- PACKED image: H2D of the stored pages (0.758 of the bytes) -> ring slot -> K5 decode + scatter ----
    // K5 reads the store itself when it is peer / local HBM, or when no ring could be had (then over PCIe)
    const bool zero_copy = mode != FMA_MODE_STAGED;
    if (zero_copy && tier == FMA_TIER_HOST && !e->host.dev_alias)
        PIPE_CHECK(fail(FMA_ENOMEM, "no HBM for a staging ring and the host store has no device alias: a packed image cannot be woken"));
    struct Dst { uint64_t packed_off; size_t w; };
    std::vector<Dst> d;
    for (size_t w = 0; w < with_backup.size(); ++w) d.push_back(Dst{e->segs[with_backup[w]].packed_off, w});
    std::sort(d.begin(), d.end(), [](const Dst& a, const Dst& b) { return a.packed_off < b.packed_off; });
    const size_t n_pages = W / FMA_PAGE_BYTES;
    PIPE_CHECK(ensure_pack_bufs(e, n_pages));
    std::vector<size_t> need_item(n_pages);
    std::vector<uint64_t> soff(n_pages), dsts(n_pages);
    std::vector<uint32_t> sbytes(n_pages);
    size_t p = 0;
    for (const Dst& x : d) {
        const Segment& s = e->segs[with_backup[x.w]];
        for (size_t o = 0; o < s.bytes; o += FMA_PAGE_BYTES, ++p) {
            const size_t lp = (size_t)((s.packed_off + o) / FMA_PAGE_BYTES);
            if (lp >= e->img_off.size()) PIPE_CHECK(fail(FMA_ESTATE, "segment at image offset %llu is outside the packed image's page table", (unsigned long long)(s.packed_off + o)));
            soff[p] = e->img_off[lp];
            sbytes[p] = e->img_bytes[lp];
            dsts[p] = (uint64_t)s.va + o;
            need_item[p] = seg_run[with_backup[x.w]] + 1;
        }
    }
    uint32_t* d_err = e->d_psize + e->pdesc_cap;
    RT(cudaMemsetAsync(d_err, 0, sizeof(uint32_t), e->ks));
    if (!zero_copy) {
        if (ring_run) {
            int mrc0 = wait_mapped(1);
            if (mrc0 != FMA_OK) PIPE_CHECK(fail(mrc0, "%s", pipe.map_msg));
        } else {
            PIPE_CHECK(ensure_ring(e, W));
        }
        struct Slot { size_t p0, np; uint64_t bytes; };
        std::vector<Slot> slots;  // pages that are adjacent in the store and fit one ring slot
        for (size_t q = 0; q < n_pages;) {
            Slot sl{q, 0, 0};
            while (q < n_pages && sl.bytes + sbytes[q] <= e->ring_slot_bytes && (sl.np == 0 || soff[q] == soff[q - 1] + sbytes[q - 1])) {
                sl.bytes += sbytes[q];
                ++sl.np;
                ++q;
            }
            if (!sl.np) PIPE_CHECK(fail(FMA_EINVAL, "ring slot of %zu bytes cannot hold one page", e->ring_slot_bytes));
            slots.push_back(sl);
        }
        for (size_t c = 0; c < slots.size(); ++c)
            for (size_t q = slots[c].p0; q < slots[c].p0 + slots[c].np; ++q) {
                fma_k_pack_desc& pd = e->h_pdesc[q];
                pd.src = (uint64_t)(uintptr_t)e->ring[c % e->n_ring] + (soff[q] - soff[slots[c].p0]);
                pd.dst = dsts[q];
                pd.mode = sbytes[q] == FMA_PAGE_BYTES ? FMA_K_PACK_RAW : FMA_K_PACK_BF16;
                pd.state = 0;
            }
        RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, n_pages * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
        for (size_t c = 0; c < slots.size(); ++c) {
            const Slot& sl = slots[c];
            const int slot = (int)(c % e->n_ring);
            cudaStream_t cstream = e->cs[c % e->n_cs];
            if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[slot], 0));
            RT(cudaMemcpyAsync(e->ring[slot], store + soff[sl.p0], sl.bytes, cudaMemcpyDefault, cstream));
            if (!copy_ops) first_copy_delay = now_s() - t_entry;
            ++copy_ops;
            RT(cudaEventRecord(e->ev_ring_full[slot], cstream));
            size_t need = 0;
            for (size_t q = sl.p0; q < sl.p0 + sl.np; ++q) need = std::max(need, need_item[q]);
            int mrc = wait_mapped(need);
            if (mrc != FMA_OK) PIPE_CHECK(fail(mrc, "%s", pipe.map_msg));
            RT(cudaStreamWaitEvent(e->ks, e->ev_ring_full[slot], 0));
            PIPE_CHECK(kt.begin());
            RT(fma_k_launch_unpack(e->d_pdesc + sl.p0, (uint32_t)sl.np, d_err, e->ks));
            PIPE_CHECK(kt.end((uint64_t)sl.np * FMA_PAGE_BYTES + sl.bytes));
            RT(cudaEventRecord(e->ev_ring_free[slot], e->ks));
        }
    } else {
        const uint64_t sbase = store_dev_base(e, tier);
        for (size_t q = 0; q < n_pages; ++q) {
            fma_k_pack_desc& pd = e->h_pdesc[q];
            pd.src = sbase + soff[q];
            pd.dst = dsts[q];
            pd.mode = sbytes[q] == FMA_PAGE_BYTES ? FMA_K_PACK_RAW : FMA_K_PACK_BF16;
            pd.state = 0;
        }
        RT(cudaMemcpyAsync(e->d_pdesc, e->h_pdesc, n_pages * sizeof(fma_k_pack_desc), cudaMemcpyHostToDevice, e->ks));
        const size_t batch_pages = std::max<size_t>(staged_slot(e) / FMA_PAGE_BYTES, 1);
        for (size_t p0 = 0; p0 < n_pages;) {
            const size_t np = std::min(batch_pages, n_pages - p0);
            size_t need = 0;
            uint64_t stored = 0;
            for (size_t q = p0; q < p0 + np; ++q) {
                need = std::max(need, need_item[q]);
                stored += sbytes[q];
            }
            int mrc = wait_mapped(need);
            if (mrc != FMA_OK) PIPE_CHECK(fail(mrc, "%s", pipe.map_msg));
            PIPE_CHECK(kt.begin());
            RT(fma_k_launch_unpack(e->d_pdesc + p0, (uint32_t)np, d_err, e->ks));
            PIPE_CHECK(kt.end((uint64_t)np * FMA_PAGE_BYTES + stored));
            if (!copy_ops) first_copy_delay = now_s() - t_entry;
            ++copy_ops;
            p0 += np;
        }
    }
    return FMA_OK;
}

// DIRECT: copy engines move each chunk of the image straight into its segment as soon as the segment is mapped
int wake_direct(WakePipe& pipe) {
    fma_engine_t* e = pipe.e;
    const std::vector<size_t>& with_backup = pipe.with_backup;
    const std::vector<size_t>& seg_run = pipe.seg_run;
    uint32_t& copy_ops = pipe.copy_ops;
    double& first_copy_delay = pipe.first_copy_delay;
    const double t_entry = pipe.t_entry;
    const char* store = pipe.store;
    auto wait_mapped = [&](size_t upto) { return pipe.wait_mapped(upto); };
    const size_t chunk = direct_chunk(e);
    int k = 0;
    for (size_t w = 0; w < with_backup.size(); ++w) {
        int mrc = wait_mapped(seg_run[with_backup[w]] + 1);
        if (mrc != FMA_OK) PIPE_CHECK(fail(mrc, "%s", pipe.map_msg));
        const Segment& s = e->segs[with_backup[w]];
        for (size_t o = 0; o < s.bytes; o += chunk, ++k) {
            const size_t n = std::min(chunk, s.bytes - o);
            RT(cudaMemcpyAsync(reinterpret_cast<void*>(s.va + o), store + s.packed_off + o, n, cudaMemcpyDefault,
                                    e->cs[k % e->n_cs]));
            if (!copy_ops) first_copy_delay = now_s() - t_entry;
            ++copy_ops;
        }
    }
    return FMA_OK;
}

// KERNEL / STAGED: page-table driven — K2 reads the store itself, or H2D -> ring slot -> K2 scatter
int wake_paged(WakePipe& pipe) {
    fma_engine_t* e = pipe.e;
    const std::vector<size_t>& with_backup = pipe.with_backup;
    const std::vector<size_t>& seg_run = pipe.seg_run;
    KernelTimes& kt = pipe.kt;
    uint32_t& copy_ops = pipe.copy_ops;
    double& first_copy_delay = pipe.first_copy_delay;
    const double t_entry = pipe.t_entry;
    const int tier = pipe.tier;
    const int mode = pipe.mode;
    const bool ring_run = pipe.ring_run;
    const char* store = pipe.store;
    const uint64_t W = pipe.W;
    auto wait_mapped = [&](size_t upto) { return pipe.wait_mapped(upto); };
    auto mapped_now = [&]() { return pipe.mapped_now(); };
    // page table of the DESTINATIONS, ordered by packed offset (== with_backup order by construction
    // only if every backed-up segment is woken; build explicitly from packed offsets to stay general)
    struct Dst { uint64_t packed_off; size_t w; };
    std::vector<Dst> d;
    for (size_t w = 0; w < with_backup.size(); ++w) d.push_back(Dst{e->segs[with_backup[w]].packed_off, w});
    std::sort(d.begin(), d.end(), [](const Dst& a, const Dst& b) { return a.packed_off < b.packed_off; });
    // runs of pages: (image page index, destination address), plus the latest work item each page needs
    size_t n_pages = W / FMA_PAGE_BYTES;
    PIPE_CHECK(ensure_tables(e, n_pages));
    uint64_t* dst_tab = e->h_tab;                 // destination page addresses
    uint64_t* src_tab = e->h_tab + e->d_tab_cap;  // source page addresses inside the store (may be sparse)
    std::vector<size_t> need_item(n_pages);
    const uint64_t sbase = store_dev_base(e, tier);
    size_t p = 0;
    for (const Dst& x : d) {
        const Segment& s = e->segs[with_backup[x.w]];
        for (size_t o = 0; o < s.bytes; o += FMA_PAGE_BYTES, ++p) {
            dst_tab[p] = (uint64_t)s.va + o;
            src_tab[p] = sbase + s.packed_off + o;
            need_item[p] = seg_run[with_backup[x.w]] + 1;
        }
    }
    RT(cudaMemcpyAsync(e->d_tab, dst_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    RT(cudaMemcpyAsync(e->d_tab + e->d_tab_cap, src_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    const uint64_t* d_dst = e->d_tab;
    const uint64_t* d_src = e->d_tab + e->d_tab_cap;
    if (mode == FMA_MODE_KERNEL) {
        // K2 reads the store itself (zero-copy PCIe reads, or NVLink/HBM loads); launch batches as the
        // mapper makes progress so the scatter overlaps cuMemCreate/Map of later segments
        const size_t batch_pages = std::max<size_t>(staged_slot(e) / FMA_PAGE_BYTES, 1);
        size_t p0 = 0;
        while (p0 < n_pages) {
            size_t np = std::min(batch_pages, n_pages - p0);
            size_t need = 0;
            for (size_t q = p0; q < p0 + np; ++q) need = std::max(need, need_item[q]);
            int mrc = wait_mapped(need);
            if (mrc != FMA_OK) PIPE_CHECK(fail(mrc, "%s", pipe.map_msg));
            // opportunistically extend the batch over everything already mapped
            const size_t have = mapped_now();
            while (p0 + np < n_pages && need_item[p0 + np] <= have) ++np;
            PIPE_CHECK(kt.launch(d_src + p0, 0, d_dst + p0, 0, (uint32_t)np));
            if (!copy_ops) first_copy_delay = now_s() - t_entry;
            ++copy_ops;
            p0 += np;
        }
    } else {  // STAGED: copy engine H2D store -> ring slot (starts at t=0), K2 scatter once the targets are mapped
        if (ring_run) {  // the ring is run 0 (1 GiB, ~0.2 ms to map): wait for it before the first H2D
            int mrc0 = wait_mapped(1);
            if (mrc0 != FMA_OK) PIPE_CHECK(fail(mrc0, "%s", pipe.map_msg));
        } else {
            PIPE_CHECK(ensure_ring(e, W));
        }
        const size_t slot_pages = e->ring_slot_bytes / FMA_PAGE_BYTES;
        // the store image may be only partially woken; H2D works on runs that are contiguous in the store
        size_t c = 0;
        size_t p0 = 0;
        while (p0 < n_pages) {
            size_t np = 1;
            while (np < slot_pages && p0 + np < n_pages && src_tab[p0 + np] == src_tab[p0 + np - 1] + FMA_PAGE_BYTES) ++np;
            const int slot = (int)(c % e->n_ring);
            cudaStream_t cstream = e->cs[c % e->n_cs];
            if (c >= (size_t)e->n_ring) RT(cudaStreamWaitEvent(cstream, e->ev_ring_free[slot], 0));
            RT(cudaMemcpyAsync(e->ring[slot], store + (src_tab[p0] - sbase), np * FMA_PAGE_BYTES, cudaMemcpyDefault, cstream));
            if (!copy_ops) first_copy_delay = now_s() - t_entry;
            ++copy_ops;
            RT(cudaEventRecord(e->ev_ring_full[slot], cstream));
            size_t need = 0;
            for (size_t q = p0; q < p0 + np; ++q) need = std::max(need, need_item[q]);
            int mrc = wait_mapped(need);
            if (mrc != FMA_OK) PIPE_CHECK(fail(mrc, "%s", pipe.map_msg));
            RT(cudaStreamWaitEvent(e->ks, e->ev_ring_full[slot], 0));
            PIPE_CHECK(kt.launch(nullptr, (uint64_t)(uintptr_t)e->ring[slot], d_dst + p0, 0, (uint32_t)np));
            RT(cudaEventRecord(e->ev_ring_free[slot], e->ks));
            p0 += np;
            ++c;
        }
    }
    return FMA_OK;
}

// MULTI-PATH (fma_paths_set): the host image is cut into chunks; every path — the engine's own PCIe link and one per idle peer
// GPU — pulls the next chunk whenever one of its staging slots is free (H2D by THAT GPU's copy engine over THAT GPU's x16
// link), and K2 on the waking GPU gathers the chunk from the path's staging slot (own HBM, or the peer's HBM over NVLink) into
// the destination pages.  Self-balancing: a slower path (other NUMA node, busy link) simply takes fewer chunks.
int wake_multipath(WakePipe& pipe) {
    fma_engine_t* e = pipe.e;
    const std::vector<size_t>& with_backup = pipe.with_backup;
    const std::vector<size_t>& seg_run = pipe.seg_run;
    KernelTimes& kt = pipe.kt;
    const char* store = pipe.store;
    const uint64_t W = pipe.W;
    struct Dst { uint64_t packed_off; size_t w; };
    std::vector<Dst> d;
    for (size_t w = 0; w < with_backup.size(); ++w) d.push_back(Dst{e->segs[with_backup[w]].packed_off, w});
    std::sort(d.begin(), d.end(), [](const Dst& a, const Dst& b) { return a.packed_off < b.packed_off; });
    const size_t n_pages = W / FMA_PAGE_BYTES;
    PIPE_CHECK(ensure_tables(e, n_pages));
    uint64_t* dst_tab = e->h_tab;
    std::vector<uint64_t> src_off(n_pages);
    std::vector<size_t> need_item(n_pages);
    size_t p = 0;
    for (const Dst& x : d) {
        const Segment& s = e->segs[with_backup[x.w]];
        for (size_t o = 0; o < s.bytes; o += FMA_PAGE_BYTES, ++p) {
            dst_tab[p] = (uint64_t)s.va + o;
            src_off[p] = s.packed_off + o;
            need_item[p] = seg_run[with_backup[x.w]] + 1;
        }
    }
    RT(cudaMemcpyAsync(e->d_tab, dst_tab, n_pages * sizeof(uint64_t), cudaMemcpyHostToDevice, e->ks));
    cudaEvent_t ev_tab = nullptr;   // the page table must be on the device before any path's K2 reads it
    PIPE_CHECK(ensure_ring_events(e, 1));
    ev_tab = e->ev_ring_full[0];
    RT(cudaEventRecord(ev_tab, e->ks));
    struct Chunk { size_t p0, np, need; };
    std::vector<Chunk> chunks;
    const size_t chunk_pages = std::max<size_t>(e->path_slot_bytes / FMA_PAGE_BYTES, 1);
    for (size_t q = 0; q < n_pages;) {
        Chunk c{q, 1, need_item[q]};
        while (c.np < chunk_pages && q + c.np < n_pages && src_off[q + c.np] == src_off[q + c.np - 1] + FMA_PAGE_BYTES) {
            c.need = std::max(c.need, need_item[q + c.np]);
            ++c.np;
        }
        chunks.push_back(c);
        q += c.np;
    }
    // chunk queues by NUMA node of the store range the chunk lives in (HostStore::ranges): a path drains the queue of ITS GPU's
    // node first and then helps with the others, so bytes cross the socket interconnect only to balance the tail
    std::vector<int> q_node;                       // queue -> node
    std::vector<std::vector<size_t>> q_chunks;     // queue -> chunk indices, image order
    for (size_t c = 0; c < chunks.size(); ++c) {
        const uint64_t off = src_off[chunks[c].p0];
        int node = -1;
        for (const HostStore::NumaRange& r : e->host.ranges)
            if (off >= r.begin && off < r.end) node = r.node;
        size_t qi = 0;
        while (qi < q_node.size() && q_node[qi] != node) ++qi;
        if (qi == q_node.size()) {
            q_node.push_back(node);
            q_chunks.emplace_back();
        }
        q_chunks[qi].push_back(c);
    }
    std::vector<std::atomic<size_t>> q_next(q_node.size());
    for (auto& a : q_next) a.store(0);
    // REMOTE paths (fma_paths_attach): helpers in the node-level owner's process pull from the SAME work counter, which therefore
    // lives in the shared mailbox together with the chunk table of this wake (fma_pull.h); published with the generation bump.
    PullMailbox* mb = e->mbox;
    if (mb) {
        if (chunks.size() > kPullMaxChunks) PIPE_CHECK(fail(FMA_EINVAL, "%zu chunks exceed the mailbox's table (use larger path slots)", chunks.size()));
        for (size_t c = 0; c < chunks.size(); ++c) mb->chunks[c] = PullChunk{src_off[chunks[c].p0], (uint32_t)(chunks[c].np * FMA_PAGE_BYTES), 0};
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
        for (int pass = 0; pass < 2; ++pass)
            for (size_t qi = 0; qi < q_node.size(); ++qi) {
                if ((pass == 0) != (q_node[qi] == my_node)) continue;   // own node's queue first
                const size_t k = q_next[qi].fetch_add(1);
                if (k < q_chunks[qi].size()) {
                    *out = q_chunks[qi][k];
                    return true;
                }
            }
        return false;
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
            if (error.compare_exchange_strong(expect, code)) snprintf(err_msg, sizeof(err_msg), "%s failed on path %zu (device %d): %s", what, pi, path.device, ce == cudaSuccess ? (code == FMA_ESTATE || code == FMA_EINTEGRITY ? what : pipe.map_msg) : cudaGetErrorString(ce));
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
                    const Chunk& ch = chunks[c];
                    const int mrc = pipe.wait_mapped(ch.need);
                    if (mrc != FMA_OK) return failw(mrc, "mapping", cudaSuccess);
                    char* slot_ptr = reinterpret_cast<char*>(path.va) + (size_t)slot * e->path_slot_bytes;
                    {
                        std::lock_guard<std::mutex> lk(kt_mu);
                        const int krc = kt.launch_on(path.kern, nullptr, (uint64_t)(uintptr_t)slot_ptr, e->d_tab + ch.p0, 0, (uint32_t)ch.np);
                        if (krc != FMA_OK) return failw(krc, "K2 launch", cudaGetLastError());
                    }
                    ce = cudaEventRecord(path.ev_free[slot], path.kern);
                    if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot drained)", ce);
                    busy[slot] = true;
                    if (!first_copy_seen.exchange(true)) pipe.first_copy_delay = now_s() - pipe.t_entry;
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
            const Chunk& ch = chunks[c];
            {
                const uint64_t off = src_off[ch.p0];
                for (const HostStore::NumaRange& r : e->host.ranges)
                    if (off >= r.begin && off < r.end && r.node == path.numa_node) ++per_path_local[pi];
            }
            const int slot = (int)(mine % (uint32_t)e->path_slots);
            if (mine >= (uint32_t)e->path_slots) {   // K2 has read the chunk that used this slot before
                ce = cudaEventSynchronize(path.ev_free[slot]);
                if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventSynchronize(slot free)", ce);
            }
            char* slot_ptr = reinterpret_cast<char*>(path.va) + (size_t)slot * e->path_slot_bytes;
            ce = cudaMemcpyAsync(slot_ptr, store + src_off[ch.p0], ch.np * FMA_PAGE_BYTES, cudaMemcpyDefault, path.copy);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaMemcpyAsync(H2D)", ce);
            if (!first_copy_seen.exchange(true)) pipe.first_copy_delay = now_s() - pipe.t_entry;
            ce = cudaEventRecord(path.ev_full[slot], path.copy);
            if (ce != cudaSuccess) return failw(FMA_ECUDA, "cudaEventRecord(slot full)", ce);
            const int mrc = pipe.wait_mapped(ch.need);
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
        pipe.copy_ops += per_path[pi];
        const int idx = e->paths[pi].remote ? -(int)pi : e->paths[pi].device;   // remote paths: -(path index), their GPU is not visible here
        e->tl_add("path_chunks", idx, pipe.t_entry, now_s(), (uint64_t)per_path[pi] * e->path_slot_bytes);
        e->tl_add("path_local", idx, pipe.t_entry, now_s(), (uint64_t)per_path_local[pi] * e->path_slot_bytes);
    }
    return FMA_OK;
}

#undef PIPE_CHECK

}  // namespace

// ------------------------------------------------------------------------------------
// WAKE
// ------------------------------------------------------------------------------------
struct MapProgress {
    std::mutex mu;
    std::condition_variable cv;
    size_t done = 0;      // number of work items fully mapped (prefix)
    int error = FMA_OK;
    char msg[512] = "";
};

int do_wake(fma_engine_t* e, uint64_t tag_mask, uint32_t flags) {
    DeviceGuard guard(e->device);
    int rc = flush_kernel_times(e);
    if (rc != FMA_OK) return rc;
    const double t_entry = now_s();
    rc = ensure_streams(e);
    if (rc != FMA_OK) return rc;

    // Work list: RUNS — maximal VA-contiguous groups of sleeping segments of one arena — so a whole tag is
    // re-created with one cuMemCreate + cuMemMap + cuMemSetAccess.  Runs that have a backup come first, in image
    // order (they gate the copy pipeline); remap-only runs (e.g. kv_cache) are mapped after them.
    using Run = fma_layout::Run;
    std::vector<Run> runs;
    {
        std::vector<size_t> cand;
        for (size_t i = 0; i < e->segs.size(); ++i) {
            const Segment& s = e->segs[i];
            if (s.mapped) continue;                                  // idempotent: already awake
            if (tag_mask && !tag_bit_set(tag_mask, s.tag)) continue;  // tags is None or data.tag in tags (cumem.py:238)
            cand.push_back(i);
        }
        if (cand.empty()) return FMA_OK;
        rc = check_tma_shape(e, e->image_tier);
        if (rc != FMA_OK) return rc;
        e->tl_begin("wake", t_entry);
        std::sort(cand.begin(), cand.end(), [&](size_t a, size_t b) {
            const Segment &x = e->segs[a], &y = e->segs[b];
            return x.arena != y.arena ? x.arena < y.arena : x.va < y.va;
        });
        std::vector<fma_layout::SegView> view;
        for (size_t i : cand) {
            const Segment& s = e->segs[i];
            view.push_back(fma_layout::SegView{i, s.arena, (uint64_t)s.va, s.bytes, s.has_backup, s.packed_off});
        }
        // FMA_MAP_PIECE_MIB (default 2048; 0 = whole runs): backed-up runs are mapped in pieces of about that size, cut at segment
        // boundaries.  One 15 GiB mapping has only the ring's slack of a few milliseconds, and a shared host's driver calls
        // sometimes stall for tens of milliseconds; with pieces K2 starts on the first piece and every later call has the copy
        // time of the pieces before it as slack.
        runs = fma_layout::plan_runs(view, env_int("FMA_MERGE_RUNS", 1) != 0, (size_t)std::max(env_int("FMA_MAP_PIECE_MIB", 2048), 0) << 20);
    }
    const int tier = e->image_tier;
    int mode = resolve_mode(e, tier);
    // A PACKED image can only be read by K5: through the staging ring, or (no HBM for a ring) straight from the
    // mapped pinned store.
    const bool packed = e->image_packed;
    if (packed && tier == FMA_TIER_HOST) mode = FMA_MODE_STAGED;

    // Staging ring.  Steady state: the ring is its OWN small run (2 x 512 MiB) placed right after the first backed-up
    // run at the arena's bump pointer and mapped FIRST — a 1 GiB cuMemCreate/Map/SetAccess costs ~0.2 ms, the H2D
    // stream starts as soon as it exists, and the big weights run (whose mapping takes 1.4 ms alone but tens of ms
    // when 8 ranks wake at once) keeps the ring's ~19 ms of slack.  At the next sleep the ring goes with a cuMemUnmap
    // like every other unit: no cudaMalloc / cudaFree anywhere (a cudaFree of 1 GiB stalls 0.8-300 ms on these hosts).
    // Needs the run to end at its arena's bump pointer; otherwise (or FMA_RING_ATTACH=0) one cudaMalloc provides it.
    // Either way the ring must exist BEFORE the other runs start taking HBM.
    bool ring_run = false;
    // MULTI-PATH: idle peers' PCIe links are borrowed for a host-tier wake of a plain image (fma_paths_set)
    const bool multipath = !e->paths.empty() && tier == FMA_TIER_HOST && mode == FMA_MODE_STAGED && !packed;
    {
        uint64_t w_bytes = 0;
        for (const Run& r : runs)
            if (r.has_backup) w_bytes += r.bytes;
        if (w_bytes && mode == FMA_MODE_STAGED && multipath) {
            // every path brings its own staging slots: no ring
        } else if (w_bytes && mode == FMA_MODE_STAGED && no_ring()) {
            mode = FMA_MODE_DIRECT;  // as when HBM is too full for a ring
        } else if (w_bytes && mode == FMA_MODE_STAGED && !e->n_ring) {
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
                ring_run = true;
            } else if (ensure_ring(e, w_bytes) != FMA_OK) {
                mode = FMA_MODE_DIRECT;  // HBM too full for a ring: copy engines go straight into the runs
            }
        } else if (w_bytes && mode == FMA_MODE_STAGED && ensure_ring(e, w_bytes) != FMA_OK) {
            mode = FMA_MODE_DIRECT;
        }
    }

    std::vector<size_t> with_backup, remap_only;  // segment indices, image order
    std::vector<size_t> seg_run(e->segs.size(), 0);  // segment -> index of its run in `runs`
    size_t n_backup_runs = 0;
    for (size_t r = 0; r < runs.size(); ++r) {
        if (runs[r].has_backup) ++n_backup_runs;
        for (size_t i : runs[r].segs) {
            seg_run[i] = r;
            (runs[r].has_backup ? with_backup : remap_only).push_back(i);
        }
    }
    const bool dbg_t = env_int("FMA_DEBUG_TIMING", 0) != 0;
    const double t_ring = now_s();
    double remap_delay_s;
    {
        uint64_t w_bytes = 0;
        for (size_t i : with_backup) w_bytes += e->segs[i].bytes;
        // a fifth of the expected host-tier copy time (55 GB/s), half of the NVLink one (600 GB/s): far below the slack
        // (a multi-path wake has as many links as paths: its copy time, and with it the head start, shrinks accordingly)
        const double expected = (double)w_bytes / (tier == FMA_TIER_HOST ? 55e9 * (multipath ? (double)e->paths.size() : 1.0) : 600e9);
        const int forced = env_int("FMA_REMAP_DELAY_MS", -1);
        remap_delay_s = forced >= 0 ? forced * 1e-3 : expected * (tier == FMA_TIER_HOST ? 0.2 : 0.5);
    }

    // FMA_REMAP_AFTER_COPY=1: remap-only runs (kv_cache) are mapped only after this rank's last copy has LANDED — a 32 GiB
    // cuMemCreate/Map/SetAccess then never runs beside this rank's DMA (its cost, a few ms, is added to the wake instead of
    // hidden under it).  A/B knob for the question "does a large VMM call slow a running H2D stream down?".
    const bool remap_after_copy = env_int("FMA_REMAP_AFTER_COPY", 0) != 0 && n_backup_runs > 0;
    std::atomic<bool> copies_landed{false};
    e->tl_add("plan", (int)runs.size(), t_entry, t_ring, 0);
    // Cross-process VMM gate (fma_gate.h): tell the other engines on this host that a call which gates a first copy is coming
    int gate_first = n_backup_runs ? gate_announce(kGateFirst) : 0;
    const double expected_copy_s = [&] {
        uint64_t w = 0;
        for (size_t i : with_backup) w += e->segs[i].bytes;
        return (double)w / (tier == FMA_TIER_HOST ? 55e9 * (multipath ? (double)e->paths.size() : 1.0) : 600e9);
    }();

    // ---- mapper thread(s): one create + map + set-access per run, in `runs` order ----------------------
    MapProgress prog;
    std::vector<char> item_done(runs.size(), 0);
    std::atomic<size_t> next_item{0};
    std::atomic<uint64_t> map_ns{0};
    const int n_map = std::max(1, std::min(e->cfg.map_threads > 0 ? e->cfg.map_threads : 1, 8));
    auto mapper = [&]() {
        cudaSetDevice(e->device);
        for (;;) {
            const size_t k = next_item.fetch_add(1);
            if (k >= runs.size()) break;
            {
                std::lock_guard<std::mutex> lk(prog.mu);
                if (prog.error != FMA_OK) break;
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
                        std::lock_guard<std::mutex> lk(prog.mu);
                        if (prog.error != FMA_OK) break;
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
                if (first_item && gate_first) {
                    gate_retract(gate_first);
                    gate_first = 0;
                }
                t0 = now_s();
                r = vmm_create_and_map(e->device, run.va, run.bytes);
            }
            const double t1 = now_s();
            map_ns.fetch_add((uint64_t)((t1 - t0) * 1e9));
            if (t0 - t_ask > 1e-4) e->tl_add("gate_wait", (int)k, t_ask, t0, 0);
            e->tl_add(is_ring ? "map_ring" : run.has_backup ? "map_backed" : "map_remap", (int)k, t0, t1, run.bytes);
            std::lock_guard<std::mutex> lk(prog.mu);
            if (r != FMA_OK) {
                prog.error = r;
                snprintf(prog.msg, sizeof(prog.msg), "%s", tl_err);
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
                while (prog.done < runs.size() && item_done[prog.done]) ++prog.done;
            }
            prog.cv.notify_all();
        }
    };
    std::vector<std::thread> mappers;
    for (int t = 0; t < n_map; ++t) mappers.emplace_back(mapper);
    auto join_mappers = [&]() {
        for (auto& t : mappers)
            if (t.joinable()) t.join();
    };
    auto wait_mapped = [&](size_t upto) -> int {  // wait until items [0, upto) are mapped
        std::unique_lock<std::mutex> lk(prog.mu);
        prog.cv.wait(lk, [&] { return prog.done >= upto || prog.error != FMA_OK; });
        return prog.error;
    };
    auto mapped_now = [&]() -> size_t {
        std::lock_guard<std::mutex> lk(prog.mu);
        return prog.done;
    };
    // A wake that fails is rolled back: every run THIS call mapped is unmapped again (its segments still have their backup),
    // so the table is what it was at entry and the controller's retry (inference-server.go:477-480) redoes the whole wake.
    // Leaving the mapped prefix in place would make the retry skip it (`mapped` == already awake) and report success over
    // weights that were never copied back — vLLM's allocator raises in that situation (cumem.py:237-249).
    auto abort_wake = [&](int code) -> int {
        char keep[512];
        snprintf(keep, sizeof(keep), "%s", tl_err);
        {
            std::lock_guard<std::mutex> lk(prog.mu);
            if (prog.error == FMA_OK) prog.error = code;
        }
        copies_landed.store(true, std::memory_order_release);
        join_mappers();
        if (gate_first) {
            gate_retract(gate_first);
            gate_first = 0;
        }
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
        return code;
    };
#define WAKE_CHECK(x)                     \
    do {                                  \
        int _rc = (x);                    \
        if (_rc != FMA_OK) return abort_wake(_rc); \
    } while (0)
#define WAKE_RT(call)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) WAKE_CHECK(fail(FMA_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__)); \
    } while (0)

    // ---- copy pipeline --------------------------------------------------------------------------
    uint64_t W = 0;
    for (size_t i : with_backup) W += e->segs[i].bytes;
    CopyTimer timer{e};
    KernelTimes kt{e};
    uint32_t copy_ops = 0;
    double copy_s = 0, first_copy_delay = 0;
    if (W) {
        const char* store = static_cast<const char*>(store_copy_base(e, tier));
        if (!store) WAKE_CHECK(fail(FMA_ESTATE, "backup store of tier %d is gone", tier));
        if (tier == FMA_TIER_HOST && mode == FMA_MODE_KERNEL && !e->host.dev_alias)
            WAKE_CHECK(fail(FMA_ECUDA, "host store has no device alias for zero-copy mode"));
        WAKE_CHECK(timer.begin());
        WakePipe pipe{e, with_backup, seg_run, W, tier, mode, ring_run, store, kt, copy_ops, first_copy_delay, t_entry, wait_mapped, mapped_now, prog.msg};
        const double t_enq0 = now_s();
        if (packed) WAKE_CHECK(wake_packed(pipe));
        else if (multipath) WAKE_CHECK(wake_multipath(pipe));
        else if (mode == FMA_MODE_DIRECT) WAKE_CHECK(wake_direct(pipe));
        else WAKE_CHECK(wake_paged(pipe));
        e->tl_add("enqueue", (int)copy_ops, t_enq0, now_s(), W);
    }
    if (remap_after_copy && W) {  // let the DMA finish before the remap-only runs are touched
        const double t_w0 = now_s();
        for (int i = 0; i < e->n_cs; ++i) WAKE_RT(cudaStreamSynchronize(e->cs[i]));
        WAKE_RT(cudaStreamSynchronize(e->ks));
        e->tl_add("copies_landed", 0, t_w0, now_s(), W);
    }
    copies_landed.store(true, std::memory_order_release);
    // every requested segment must be mapped before wake returns (cumem.py:237-240)
    {
        const double t_w0 = now_s();
        int mrc = wait_mapped(runs.size());
        if (mrc != FMA_OK) WAKE_CHECK(fail(mrc, "%s", prog.msg));
        e->tl_add("wait_all_mapped", (int)runs.size(), t_w0, now_s(), 0);
    }
    join_mappers();
    if (gate_first) {
        gate_retract(gate_first);
        gate_first = 0;
    }
    const double t_joined = now_s();
    double t_copy_end = t_joined;
    if (W) {
        WAKE_CHECK(timer.end(&copy_s));
        e->tl_add("drain", 0, t_joined, now_s(), W);
        WAKE_CHECK(kt.collect());
        if (packed) {  // K5 counts stored pages it could not read (bad magic / count): the image is damaged
            WAKE_RT(cudaMemcpyAsync(e->h_psize + e->pdesc_cap, e->d_psize + e->pdesc_cap, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->ks));
            WAKE_RT(cudaStreamSynchronize(e->ks));
            if (e->h_psize[e->pdesc_cap]) WAKE_CHECK(fail(FMA_EINTEGRITY, "%u stored page(s) of the packed image are malformed", e->h_psize[e->pdesc_cap]));
        }
        t_copy_end = now_s();
    }
    if (dbg_t)
        fprintf(stderr, "[fma] wake phases: plan+ring %.1f ms | enqueue+map-wait %.1f ms | drain %.1f ms | ring free %.1f ms | runs %zu\n",
                (t_ring - t_entry) * 1e3, (t_joined - t_ring) * 1e3, (t_copy_end - t_joined) * 1e3, (now_s() - t_copy_end) * 1e3, runs.size());
#undef WAKE_CHECK
#undef WAKE_RT

    uint64_t remapped_only = 0;
    for (size_t i : remap_only) remapped_only += e->segs[i].bytes;

    int verify_rc = FMA_OK;
    if ((flags & FMA_FLAG_VERIFY) && W) {
        std::vector<size_t> idx;
        for (size_t i : with_backup)
            if (e->segs[i].digest_valid) idx.push_back(i);
        std::vector<uint64_t> dg;
        rc = digest_segments(e, idx, &dg);
        if (rc != FMA_OK) return rc;
        for (size_t k = 0; k < idx.size(); ++k)
            if (dg[k] != e->segs[idx[k]].digest)
                verify_rc = fail(FMA_EINTEGRITY, "segment %zu (va 0x%llx): digest %016llx after wake != %016llx before sleep", idx[k],
                                 (unsigned long long)e->segs[idx[k]].va, (unsigned long long)dg[k],
                                 (unsigned long long)e->segs[idx[k]].digest);
    }
    if (!(flags & FMA_FLAG_KEEP_BACKUP)) {
        for (size_t i : with_backup) {  // data.cpu_backup_tensor = None (cumem.py:249)
            Segment& s = e->segs[i];
            // INCREMENTAL sleep: the host store keeps these bytes; remember where, together with their digest
            s.shadow_off = (s.digest_valid && verify_rc == FMA_OK) ? s.packed_off : kNoOffset;   // host store or parking buffer: both outlive the wake
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

    e->tl_add("total", 0, t_entry, now_s(), W);
    e->st.wake_seconds = now_s() - t_entry;
    e->st.wake_copy_seconds = copy_s;
    e->st.wake_map_seconds = map_ns.load() * 1e-9;
    e->st.wake_first_copy_delay = first_copy_delay;
    e->st.wake_bytes_restored = W;
    e->st.wake_bytes_remapped_only = remapped_only;
    e->st.copy_ops = copy_ops;
    e->st.total_copy_ops += copy_ops;
    e->st.tier = tier;
    e->st.mode = mode;
    if (!W) {
        e->pending_events = 0;
        e->st.kernel_seconds = 0;
        e->st.kernel_bytes = 0;
        e->st.kernel_launches = 0;
    }
    return verify_rc;
}

}  // namespace fma_impl
