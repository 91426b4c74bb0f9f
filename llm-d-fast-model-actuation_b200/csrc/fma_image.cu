// fma_image.cu — image hand-over: a sleeping model's host image outlives its engine / process (memfd store + descriptor)
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"

using namespace fma_impl;

namespace fma_impl {

// Descriptor of the image sleeping in `tier`'s store: header, one ImageSegDesc per offloaded segment in image order and, for a
// PACKED image (version 2), the per-page stored sizes (offsets are their prefix sums).  At most kImageTail bytes.
int image_descriptor_build(fma_engine_t* e, int tier, std::vector<char>* out) {
    std::vector<const Segment*> segs;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (const Segment& s : e->segs)
            if (s.has_backup && (tier == FMA_TIER_HOST ? s.backup_tier == FMA_TIER_HOST : s.backup_tier != FMA_TIER_HOST) && !s.mapped) segs.push_back(&s);
    }
    if (segs.empty()) return fail(FMA_ESTATE, "nothing is asleep in that store");
    std::sort(segs.begin(), segs.end(), [](const Segment* a, const Segment* b) { return a->packed_off < b->packed_off; });
    const size_t n_img_pages = e->image_packed ? e->img_bytes.size() : 0;
    const size_t total = sizeof(ImageHeader) + segs.size() * sizeof(ImageSegDesc) + sizeof(uint32_t) * (1 + n_img_pages);
    if (total > kImageTail) return fail(FMA_ENOMEM, "too many segments / pages for the descriptor");
    out->assign(total, 0);
    char* tail = out->data();
    ImageHeader hd{kImageMagic, e->image_packed ? 2u : 1u, (uint32_t)segs.size(), e->image_bytes};
    memcpy(tail, &hd, sizeof(hd));
    for (size_t i = 0; i < segs.size(); ++i) {
        ImageSegDesc d;
        memset(&d, 0, sizeof(d));
        d.bytes = segs[i]->bytes;
        d.packed_off = segs[i]->packed_off;
        d.digest = segs[i]->digest;
        d.digest_valid = segs[i]->digest_valid ? 1 : 0;
        const std::string& t = e->tags[segs[i]->tag];
        d.tag_len = (uint32_t)std::min<size_t>(t.size(), sizeof(d.tag) - 1);
        memcpy(d.tag, t.data(), d.tag_len);
        memcpy(tail + sizeof(hd) + i * sizeof(d), &d, sizeof(d));
    }
    char* pt = tail + sizeof(hd) + segs.size() * sizeof(ImageSegDesc);
    const uint32_t np = (uint32_t)n_img_pages;
    memcpy(pt, &np, sizeof(np));
    if (np) memcpy(pt + sizeof(np), e->img_bytes.data(), n_img_pages * sizeof(uint32_t));
    return FMA_OK;
}

namespace {

// Parsed + validated descriptor, matched against the engine's segments for `tag_mask` (same order rule as fma_sleep).
struct ParsedImage {
    ImageHeader hd;
    std::vector<ImageSegDesc> ds;
    std::vector<size_t> order;          // engine segment index of descriptor entry i
    std::vector<uint64_t> page_off;     // version 2: the PACKED image's page table
    std::vector<uint32_t> page_bytes;
};

int image_descriptor_parse(fma_engine_t* e, const char* tail, size_t tail_bytes, size_t store_cap, uint64_t tag_mask, ParsedImage* out) {
    ParsedImage& pi = *out;
    if (tail_bytes < sizeof(ImageHeader)) return fail(FMA_EINVAL, "image descriptor missing or corrupt");
    memcpy(&pi.hd, tail, sizeof(pi.hd));
    const ImageHeader& hd = pi.hd;
    if (hd.magic != kImageMagic || (hd.version != 1 && hd.version != 2) || (hd.version == 1 && hd.image_bytes > store_cap) ||
        sizeof(ImageHeader) + (size_t)hd.n_segments * sizeof(ImageSegDesc) + sizeof(uint32_t) > tail_bytes)
        return fail(FMA_EINVAL, "image descriptor missing or corrupt");
    if (hd.version == 2) {
        const char* pt = tail + sizeof(hd) + (size_t)hd.n_segments * sizeof(ImageSegDesc);
        uint32_t np = 0;
        memcpy(&np, pt, sizeof(np));
        if ((uint64_t)np * FMA_PAGE_BYTES != hd.image_bytes || sizeof(ImageHeader) + (size_t)hd.n_segments * sizeof(ImageSegDesc) + sizeof(uint32_t) * (1 + (size_t)np) > tail_bytes)
            return fail(FMA_EINVAL, "packed image: page table does not match the image size");
        pi.page_bytes.resize(np);
        pi.page_off.resize(np);
        memcpy(pi.page_bytes.data(), pt + sizeof(np), (size_t)np * sizeof(uint32_t));
        uint64_t total = 0;
        for (uint32_t q = 0; q < np; ++q) {
            if (pi.page_bytes[q] != FMA_K_PACKED_PAGE_BYTES && pi.page_bytes[q] != FMA_PAGE_BYTES) return fail(FMA_EINVAL, "packed image: bad stored page size");
            pi.page_off[q] = total;
            total += pi.page_bytes[q];
        }
        if (total > store_cap) return fail(FMA_EINVAL, "packed image: stored pages exceed the store");
    }
    std::lock_guard<std::mutex> lk(e->mu);
    for (size_t i = 0; i < e->segs.size(); ++i)
        if (tag_bit_set(tag_mask, e->segs[i].tag)) pi.order.push_back(i);
    std::sort(pi.order.begin(), pi.order.end(), [&](size_t a, size_t b) {
        const Segment &x = e->segs[a], &y = e->segs[b];
        return x.arena != y.arena ? x.arena < y.arena : x.va < y.va;
    });
    if (pi.order.size() != hd.n_segments) return fail(FMA_EINVAL, "image and engine disagree on the number of segments");
    pi.ds.resize(hd.n_segments);
    uint64_t off = 0;
    for (size_t i = 0; i < pi.ds.size(); ++i) {
        memcpy(&pi.ds[i], tail + sizeof(hd) + i * sizeof(ImageSegDesc), sizeof(ImageSegDesc));
        const Segment& s = e->segs[pi.order[i]];
        // the descriptor comes from a file or another process: bound what it claims before using it as a length
        if (pi.ds[i].tag_len >= sizeof(pi.ds[i].tag) || pi.ds[i].digest_valid > 1) return fail(FMA_EINVAL, "image descriptor is malformed (tag length / digest flag)");
        if (pi.ds[i].bytes != s.bytes || pi.ds[i].packed_off != off || std::string(pi.ds[i].tag, pi.ds[i].tag_len) != e->tags[s.tag])
            return fail(FMA_EINVAL, "image and engine disagree on a segment's size, offset or tag");
        off += s.bytes;
    }
    if (off != hd.image_bytes) return fail(FMA_EINVAL, "image size mismatch");
    return FMA_OK;
}

// after do_sleep(kFlagAdopt): take over the exporter's page table and integrity data
void image_apply(fma_engine_t* e, ParsedImage& pi) {
    if (pi.hd.version == 2) {  // wake through K5 with the exporter's page table
        e->image_packed = true;
        e->image_store_bytes = pi.page_off.empty() ? 0 : pi.page_off.back() + pi.page_bytes.back();
        e->img_off = std::move(pi.page_off);
        e->img_bytes = std::move(pi.page_bytes);
    }
    for (size_t i = 0; i < pi.ds.size(); ++i) {  // integrity data travels with the image: FMA_FLAG_VERIFY on wake checks it
        Segment& s = e->segs[pi.order[i]];
        s.digest = pi.ds[i].digest;
        s.digest_valid = pi.ds[i].digest_valid != 0;
    }
}

// ---- moves of a sleeping image between tiers (fma_image_move) ----
// Every tier holds the image in one layout (plain pages back to back, or the PACKED form's stored pages at img_off[p]), so a move
// copies image_store_bytes bytes from offset 0 of one store to offset 0 of the other and changes nothing but the engine's records.

// Copy engines between the pinned host store and the parking buffer: direct_chunk pieces round-robin over the copy streams.
int move_host_park(fma_engine_t* e, bool to_park, uint64_t bytes, uint32_t* ops) {
    char* host = static_cast<char*>(e->host.base);
    char* park = reinterpret_cast<char*>(e->park.va);
    const size_t chunk = direct_chunk(e);
    size_t k = 0;
    for (uint64_t o = 0; o < bytes; o += chunk, ++k) {
        const size_t n = (size_t)std::min<uint64_t>(chunk, bytes - o);
        RT(cudaMemcpyAsync(to_park ? park + o : host + o, to_park ? host + o : park + o, n, cudaMemcpyDefault, e->cs[k % e->n_cs]));
        ++*ops;
    }
    return FMA_OK;
}

// The pinned host store <-> a file: FileIO's threads pread / pwrite straight into / out of the store, no copy engine involved.
int move_host_file(fma_engine_t* e, bool to_file, int fd, bool direct, uint64_t bytes, uint64_t file_bytes, const char* path) {
    const uint64_t piece = round_up(std::max<size_t>(e->load_chunk, 4096), 4096);
    std::vector<FileIO::Item> items;
    for (uint64_t o = 0; o < bytes; o += piece) items.push_back(FileIO::Item{o, std::min(piece, bytes - o)});
    FileIO io(e, fd, to_file, direct, std::move(items), file_bytes, path, static_cast<char*>(e->host.base));
    return io.finish();
}

// The parking buffer <-> a file through the engine's pinned I/O windows: the file tier's disk stage without the HBM ring.
int move_park_file(fma_engine_t* e, bool to_file, int fd, bool direct, uint64_t bytes, uint64_t file_bytes, const char* path, uint32_t* ops) {
    const std::vector<FileIO::Item> items = FileIO::cut(e, {FileIO::Item{0, bytes}});
    FileIO io(e, fd, to_file, direct, items, file_bytes, path);
    for (size_t k = 0; k < items.size(); ++k, ++*ops)
        RC(io.copy(k, reinterpret_cast<char*>(e->park.va) + items[k].file_off, e->cs[k % e->n_cs]));
    return io.finish();   // every pread / pwrite has returned and every copy into or out of a window has finished
}

// What a move has set up so far, so that a failure can undo it
struct MoveState {
    FileFd file;
    bool direct = false;
    bool file_emptied = false;   // the destination file has been emptied: a failure leaves no descriptor in it
    bool made_host = false;      // the host store, or the local parking buffer, was created by this move
    bool made_park = false;
    bool copies = false;         // the copy streams ran
};

int run_move(fma_engine_t* e, fma_layout::MovePipeKind pipe, int from, int to, MoveState& ms) {
    using fma_layout::MovePipeKind;
    const uint64_t bytes = e->image_store_bytes;
    const bool park_side = pipe != MovePipeKind::HostFile && pipe != MovePipeKind::FileHost;
    ms.copies = park_side;
    if (park_side) RC(ensure_streams(e));
    // the destination, prepared as a sleep to its tier prepares it
    if (to == FMA_TIER_HOST) {
        if (e->host.shared) {   // the shared image is read-only: leave it to its other holders and take a private store
            invalidate_shadows(e);
            host_store_free(e->host);
            e->st.host_store_bytes = 0;
        }
        ms.made_host = !e->host.base || e->host.cap < round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), FMA_PAGE_BYTES);
        RC(host_store_reserve(e, bytes));
    } else if (to == FMA_TIER_LOCAL) {
        const size_t need = round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), e->gran);
        ms.made_park = !(e->park.va && e->park.device == e->device && e->park.bytes >= need);
        if (ms.made_park && e->park.va) {   // a buffer that does not fit, or a peer's (it holds nothing of this image), goes
            if (e->shadow_tier == FMA_TIER_PEER || e->shadow_tier == FMA_TIER_LOCAL) invalidate_shadows(e);
            vmm_buffer_free(e->park);
        }
        if (ms.made_park) RC(park_store_create(e, e->device, need, &e->park));
    }
    // the file side: the destination emptied once the filesystem has room; the source checked to hold the whole image
    const double t_io = now_s();
    const std::string path = to == FMA_TIER_FILE ? e->file_path : e->image_file;
    uint64_t file_bytes = 0;
    if (to == FMA_TIER_FILE) {
        RC(open_image_file(path.c_str(), true, &ms.file.fd, &ms.direct));
        RC(open_file_store(ms.file.fd, bytes, path.c_str()));
        ms.file_emptied = true;
    } else if (from == FMA_TIER_FILE) {
        RC(open_image_source(path.c_str(), bytes, &ms.file.fd, &ms.direct, &file_bytes));
    }
    // the bytes
    uint32_t ops = 0;
    CopyTimer timer{e};
    const double t_copy = now_s();
    if (park_side) RC(timer.begin());
    switch (pipe) {
    case MovePipeKind::HostPark: RC(move_host_park(e, true, bytes, &ops)); break;
    case MovePipeKind::ParkHost: RC(move_host_park(e, false, bytes, &ops)); break;
    case MovePipeKind::HostFile: RC(move_host_file(e, true, ms.file.fd, ms.direct, bytes, 0, path.c_str())); break;
    case MovePipeKind::FileHost: RC(move_host_file(e, false, ms.file.fd, ms.direct, bytes, file_bytes, path.c_str())); break;
    case MovePipeKind::ParkFile: RC(move_park_file(e, true, ms.file.fd, ms.direct, bytes, 0, path.c_str(), &ops)); break;
    case MovePipeKind::FilePark: RC(move_park_file(e, false, ms.file.fd, ms.direct, bytes, file_bytes, path.c_str(), &ops)); break;
    case MovePipeKind::Refused: return fail(FMA_EINVAL, "a refused move has no copy");   // (refused before)
    }
    if (park_side) {
        double copy_s = 0;
        RC(timer.end(&copy_s));   // joins the copy streams only
        e->tl_add("copies_landed", (int)ops, t_copy, now_s(), bytes);
    }
    // a file written by a move is completed as a file-tier sleep completes it: it opens with fma_image_adopt_file and image_load
    if (to == FMA_TIER_FILE) {
        std::vector<char> desc;
        RC(image_descriptor_build(e, from, &desc));
        RC(close_file_store(ms.file.fd, bytes, path.c_str(), ms.direct, desc));
    }
    if (ms.file.fd >= 0) e->tl_add("file_io", ms.direct ? 1 : 0, t_io, now_s(), to == FMA_TIER_FILE ? bytes + kImageTail : bytes);
    e->st.copy_ops = ops;
    e->st.total_copy_ops += ops;
    return FMA_OK;
}

// A failed move: nothing may still copy into what goes, what the move created goes, and a destination file keeps no descriptor
void undo_move(fma_engine_t* e, MoveState& ms) {
    if (ms.copies)
        for (int i = 0; i < e->n_cs; ++i) cudaStreamSynchronize(e->cs[i]);
    if (ms.made_host) {
        host_store_free(e->host);
        e->st.host_store_bytes = 0;
    }
    if (ms.made_park) vmm_buffer_free(e->park);
    if (ms.file_emptied) {   // what was written goes too (best effort: without its descriptor the file is refused anyway)
        const int r = ftruncate(ms.file.fd, 0);
        (void)r;
    }
    cudaGetLastError();
}

// ---- checking a sleeping image where it lies (fma_image_verify) ----
// K3 digests plain pages and K6 decodes and digests PACKED ones, both straight out of the store: the parking buffer or the
// resident share in HBM, the pinned host store through its device alias, a file through the pinned I/O windows.  Each kernel adds
// a page's digest into that page's accumulator (d_dig, one per page of the check), and the host sums a segment's pages.
struct Verifier {
    explicit Verifier(fma_engine_t* engine) : e(engine) {}
    fma_engine_t* e;
    struct Seg { size_t index; uint64_t va, digest; };
    std::vector<Seg> segs;            // the segments checked, by engine index
    std::vector<uint64_t> sum;        // their digests as computed
    std::vector<size_t> seg_of;       // accumulator i -> position in `segs`
    std::vector<uint64_t> kbytes;     // stored bytes read by each timed launch pair
    size_t n_ev = 0;
    static constexpr size_t kScratch = (size_t)64 << 20;   // host store without a device alias: two HBM buffers of this size
    void* scratch[2] = {};

    // The pages of the segments `pos` (positions in `segs`) in a store with the page table (off, bytes), off == nullptr: pages stored
    // verbatim at their image offsets.  PagePlan::need carries the page's segment position (nothing waits for a mapper here).
    int plan(const std::vector<size_t>& pos, const std::vector<uint64_t>* off, const std::vector<uint32_t>* bytes, std::vector<PagePlan>* pages) {
        std::vector<fma_layout::SegPages> v;
        for (size_t k : pos) {
            const Segment& s = e->segs[segs[k].index];
            v.push_back(fma_layout::SegPages{s.va, s.bytes, s.packed_off, k});
        }
        uint64_t bad = 0;
        if (!fma_layout::plan_pages(v, off, bytes, pages, &bad))
            return fail(FMA_ESTATE, "segment at image offset %llu is outside the packed image's page table", (unsigned long long)bad);
        return FMA_OK;
    }

    // One launch pair over pages [b.p0, b.p0 + b.np) of `pages`, whose accumulators start at `at`: K6 over the coded pages, K3 over
    // the raw ones.  src(q) is where page q can be read on the device now.
    template <class Src>
    int launch(const std::vector<PagePlan>& pages, size_t at, const Batch& b, Src src) {
        size_t lo = at + b.p0, hi = at + b.p0 + b.np;   // coded pages fill the accumulators from the front, raw ones from the back
        for (size_t q = b.p0; q < b.p0 + b.np; ++q) {
            const size_t i = pages[q].bytes == FMA_PAGE_BYTES ? --hi : lo++;
            e->h_desc[i].addr = src(q);
            e->h_desc[i].first_word = (pages[q].va - segs[pages[q].need].va) / 8;
            seg_of[i] = pages[q].need;
        }
        const size_t p0 = at + b.p0, n_coded = lo - p0, n_raw = b.np - n_coded;
        RT(cudaMemcpyAsync(e->d_desc + p0, e->h_desc + p0, b.np * sizeof(fma_k_page_desc), cudaMemcpyHostToDevice, e->ks));
        RC(ensure_event_pool(e, n_ev + 2));
        RT(cudaEventRecord(e->ev_pool[n_ev], e->ks));
        if (n_coded) {
            if (!fma_k_launch_unpack_digest) return fail(FMA_ECUDA, "this library was built without K6: a PACKED image cannot be checked");
            RT(fma_k_launch_unpack_digest(e->d_desc + p0, (uint32_t)n_coded, e->d_dig + p0, e->d_psize + e->pdesc_cap, e->ks));
        }
        RT(fma_k_launch_page_digest(e->d_desc + lo, (uint32_t)n_raw, e->d_dig + lo, e->ks));
        RT(cudaEventRecord(e->ev_pool[n_ev + 1], e->ks));
        n_ev += 2;
        kbytes.push_back(b.stored);
        return FMA_OK;
    }

    // a store the device reads in place (HBM, or pinned host memory through its alias) at `base`
    int in_place(const std::vector<PagePlan>& pages, size_t at, uint64_t base) {
        std::vector<Batch> batches;
        fma_layout::plan_batches(pages, slot_pages(e), UINT64_MAX, false, &batches);
        for (const Batch& b : batches) RC(launch(pages, at, b, [&](size_t q) { return base + pages[q].off; }));
        return FMA_OK;
    }

    // a host store without a device alias: runs of pages copied into two HBM scratch buffers in turn, checked there
    int staged_host(const std::vector<PagePlan>& pages, size_t at) {
        std::vector<Batch> batches;
        if (!fma_layout::plan_batches(pages, SIZE_MAX, kScratch, true, &batches)) return fail(FMA_EINVAL, "a stored page does not fit %zu bytes of scratch", kScratch);
        RC(ensure_ring_events(e, 2));
        for (int i = 0; i < 2 && i < (int)batches.size(); ++i)
            if (cudaMalloc(&scratch[i], kScratch) != cudaSuccess) {
                cudaGetLastError();
                return fail(FMA_ENOMEM, "cannot allocate 2 x %zu bytes of HBM scratch to check a host store without a device alias", kScratch);
            }
        for (size_t c = 0; c < batches.size(); ++c) {
            const Batch& b = batches[c];
            const int s = (int)(c % 2);
            char* buf = static_cast<char*>(scratch[s]);
            if (c >= 2) RT(cudaStreamWaitEvent(e->cs[0], e->ev_ring_free[s], 0));
            RT(cudaMemcpyAsync(buf, static_cast<const char*>(e->host.base) + pages[b.p0].off, b.stored, cudaMemcpyHostToDevice, e->cs[0]));
            RT(cudaEventRecord(e->ev_ring_full[s], e->cs[0]));
            RT(cudaStreamWaitEvent(e->ks, e->ev_ring_full[s], 0));
            RC(launch(pages, at, b, [&](size_t q) { return (uint64_t)(uintptr_t)buf + (pages[q].off - pages[b.p0].off); }));
            RT(cudaEventRecord(e->ev_ring_free[s], e->ks));
        }
        return FMA_OK;
    }

    // the image file: reader threads pread runs of whole stored pages into the pinned I/O windows, the kernels read each window
    // over the link, and the window goes back to its reader behind them
    int file(const std::vector<PagePlan>& pages, size_t at) {
        if (!e->load_ring) RC(ensure_io_windows(e));
        const uint64_t window = e->io_window_bytes - 8192;   // (the windows' O_DIRECT slack, ensure_io_windows)
        std::vector<Batch> batches;
        if (!fma_layout::plan_batches(pages, SIZE_MAX, window, true, &batches))
            return fail(FMA_EINVAL, "a stored page does not fit an I/O window of %llu bytes", (unsigned long long)window);
        std::vector<FileIO::Item> items;
        uint64_t need = 0, read_bytes = 0;
        for (const Batch& b : batches) {
            items.push_back(FileIO::Item{pages[b.p0].off, b.stored});
            need = std::max(need, pages[b.p0].off + b.stored);
            read_bytes += b.stored;
        }
        const double t_io = now_s();
        FileFd f;
        bool direct = false;
        uint64_t file_bytes = 0;
        RC(open_image_source(e->image_file.c_str(), need, &f.fd, &direct, &file_bytes));
        FileIO io(e, f.fd, false, direct, items, file_bytes, e->image_file.c_str());
        for (size_t c = 0; c < batches.size(); ++c) {
            const Batch& b = batches[c];
            RC(io.read_in_place(c, e->ks, [&](const char* win) {
                return launch(pages, at, b, [&](size_t q) { return (uint64_t)(uintptr_t)win + (pages[q].off - pages[b.p0].off); });
            }));
        }
        RC(io.finish());   // every read has returned and every kernel over a window has finished
        e->tl_add("file_io", direct ? 1 : 0, t_io, now_s(), read_bytes);
        return FMA_OK;
    }

    int run(const std::vector<size_t>& main, const std::vector<size_t>& res) {
        std::vector<PagePlan> mp, rp;
        RC(plan(main, e->image_packed ? &e->img_off : nullptr, &e->img_bytes, &mp));
        RC(plan(res, e->res_packed ? &e->res_off : nullptr, &e->res_bytes, &rp));
        const size_t n = mp.size() + rp.size();
        RC(ensure_streams(e));
        RC(ensure_desc(e, n));
        seg_of.assign(n, 0);
        RT(cudaEventRecord(e->ev_start, e->ks));
        e->tl_dev_base = now_s() - e->tl_entry;
        RT(cudaMemsetAsync(e->d_dig, 0, n * sizeof(uint64_t), e->ks));
        const auto coded = [](const PagePlan& q) { return q.bytes != FMA_PAGE_BYTES; };
        if (std::any_of(mp.begin(), mp.end(), coded) || std::any_of(rp.begin(), rp.end(), coded)) {
            RC(ensure_pack_bufs(e, 1));   // (K6 counts malformed pages in K5's error counter)
            RT(cudaMemsetAsync(e->d_psize + e->pdesc_cap, 0, sizeof(uint32_t), e->ks));
        }
        if (!mp.empty()) {
            switch (e->image_tier) {
            case FMA_TIER_HOST:
                RC(e->host.dev_alias ? in_place(mp, 0, (uint64_t)(uintptr_t)e->host.dev_alias) : staged_host(mp, 0));
                break;
            case FMA_TIER_FILE: RC(file(mp, 0)); break;
            default:
                if (!e->park.va) return fail(FMA_ESTATE, "the parking buffer that holds the image is gone");
                RC(in_place(mp, 0, (uint64_t)e->park.va));
            }
        }
        if (!rp.empty()) {
            if (!e->res.va) return fail(FMA_ESTATE, "the resident part of the image is gone");
            RC(in_place(rp, mp.size(), (uint64_t)e->res.va));
        }
        RT(cudaMemcpyAsync(e->h_dig, e->d_dig, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->ks));
        RT(cudaStreamSynchronize(e->ks));
        sum.assign(segs.size(), 0);
        for (size_t i = 0; i < n; ++i) sum[seg_of[i]] += e->h_dig[i];
        for (size_t i = 0; i + 1 < n_ev; i += 2) {   // device-timed launch rows
            float ms0 = 0, ms = 0;
            RT(cudaEventElapsedTime(&ms0, e->ev_start, e->ev_pool[i]));
            RT(cudaEventElapsedTime(&ms, e->ev_pool[i], e->ev_pool[i + 1]));
            const double t0 = e->tl_entry + e->tl_dev_base + ms0 * 1e-3;
            e->tl_add("kernel", (int)(i / 2), t0, t0 + ms * 1e-3, kbytes[i / 2]);
        }
        return FMA_OK;
    }

    ~Verifier() {   // nothing may still read the scratch when it goes
        if (scratch[0] || scratch[1]) {
            cudaStreamSynchronize(e->cs[0]);
            cudaStreamSynchronize(e->ks);
        }
        for (void* p : scratch)
            if (p) cudaFree(p);
        cudaGetLastError();
    }
};

}  // namespace
}  // namespace fma_impl

extern "C" {

int fma_image_export(fma_engine_t* e, int* out_fd) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (!out_fd) return fail(FMA_EINVAL, "out_fd is NULL");
    if (resident_asleep(e)) return fail(FMA_ESTATE, "part of the sleeping image is resident in this process's own HBM (option resident_bytes) and cannot be handed over: set it to 0 and sleep again");
    if (e->image_tier == FMA_TIER_FILE && image_in(e, ImageIn::AnyAsleep)) return fail(FMA_ESTATE, "the sleeping image is in a file: the file itself is the hand-over");
    if (e->host.fd < 0 || !e->host.base) return fail(FMA_ESTATE, "the host store is not shareable (set FMA_HOST_STORE_SHM=1 before the first sleep)");
    if (e->image_tier != FMA_TIER_HOST) return fail(FMA_ESTATE, "no host-tier image");
    std::vector<char> desc;
    int drc = image_descriptor_build(e, FMA_TIER_HOST, &desc);
    if (drc != FMA_OK) return drc;
    memcpy(static_cast<char*>(e->host.base) + e->host.cap, desc.data(), desc.size());
    int fd = dup(e->host.fd);
    if (fd < 0) return fail(FMA_ENOMEM, "dup failed: %s", strerror(errno));
    e->host.shared = true;  // whoever receives the fd reads this image: never write it again (see HostStore::shared)
    *out_fd = fd;
    return FMA_OK;
}

int fma_image_adopt(fma_engine_t* e, int fd, uint64_t tag_mask, uint32_t flags) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (!tag_mask) return fail(FMA_EINVAL, "adopt needs the tag mask the image was slept with");
    for (const Segment& s : e->segs)
        if (!s.mapped) return fail(FMA_ESTATE, "adopt needs a fully awake engine");
    struct stat sb;
    if (fstat(fd, &sb) != 0 || (size_t)sb.st_size <= kImageTail) return fail(FMA_EINVAL, "not an image fd");
    const size_t map_bytes = (size_t)sb.st_size, cap = map_bytes - kImageTail;
    int myfd = dup(fd);
    if (myfd < 0) return fail(FMA_ENOMEM, "dup failed: %s", strerror(errno));
    void* p = mmap(nullptr, map_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, myfd, 0);
    if (p == MAP_FAILED) {
        close(myfd);
        return fail(FMA_ENOMEM, "cannot map the image: %s", strerror(errno));
    }
    auto bail = [&](int code, const char* why) {
        munmap(p, map_bytes);
        close(myfd);
        return fail(code, "%s", why);
    };
    const char* tail = static_cast<const char*>(p) + cap;
    ParsedImage pi;
    {
        int prc = image_descriptor_parse(e, tail, kImageTail, cap, tag_mask, &pi);
        if (prc != FMA_OK) {
            char why[512];
            snprintf(why, sizeof(why), "%s", tl_err);
            return bail(prc, why);
        }
    }
    const ImageHeader& hd = pi.hd;
    std::vector<ImageSegDesc>& ds = pi.ds;
    const std::vector<size_t>& order = pi.order;
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    if (flags & FMA_FLAG_VERIFY) {
        // "Sleep by adoption": this engine HAS the weights and wants to share somebody else's image of the same model (a second
        // replica on the node: one host copy for all).  Only legal if its device bytes are what the image holds — K3 digests
        // against the descriptor's; a mismatch leaves the engine awake and untouched.
        std::vector<uint64_t> now;
        int vrc = digest_segments(e, order, &now);
        if (vrc != FMA_OK) {
            munmap(p, map_bytes);
            close(myfd);
            return vrc;
        }
        for (size_t i = 0; i < ds.size(); ++i)
            if (!ds[i].digest_valid || ds[i].digest != now[i])
                return bail(FMA_EINTEGRITY, ds[i].digest_valid ? "the image holds different bytes than this engine's segments" : "the image carries no digests to compare with");
    }
    invalidate_shadows(e);
    host_store_free(e->host);
    const double t0 = now_s();
    cudaError_t r = cudaHostRegister(p, map_bytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
    HostStore h;
    if (r != cudaSuccess) {
        // The mapping cannot be pinned in place (e.g. an image FILE on a filesystem whose pages the driver will not lock):
        // copy it once into an anonymous pinned store — a load from the page cache, several threads — and let go of the fd.
        cudaGetLastError();
        void* q = nullptr;
        r = cudaHostAlloc(&q, map_bytes, cudaHostAllocPortable | cudaHostAllocMapped);
        if (r != cudaSuccess) {
            cudaGetLastError();
            return bail(FMA_ENOMEM, "cannot pin the adopted image, in place or as a copy");
        }
        const int nt = std::max(1, std::min(env_int("FMA_TOUCH_THREADS", 8), 32));
        const size_t per = round_up((map_bytes + nt - 1) / nt, FMA_PAGE_BYTES);
        std::vector<std::thread> th;
        for (int t = 0; t < nt; ++t) {
            const size_t lo = (size_t)t * per, hi = std::min(map_bytes, lo + per);
            if (lo >= hi) break;
            th.emplace_back([p, q, lo, hi] { memcpy(static_cast<char*>(q) + lo, static_cast<const char*>(p) + lo, hi - lo); });
        }
        for (auto& t : th) t.join();
        munmap(p, map_bytes);
        close(myfd);
        h.base = q; h.cap = cap; h.map_bytes = 0; h.fd = -1; h.registered = false;
        p = q;
    } else {
        h.base = p; h.cap = cap; h.map_bytes = map_bytes; h.fd = myfd; h.registered = true;
        h.shared = true;  // the exporter (and other adopters) map the same pages
    }
    void* alias = nullptr;
    if (cudaHostGetDevicePointer(&alias, p, 0) == cudaSuccess) h.dev_alias = alias;
    else cudaGetLastError();
    h.pin_seconds = now_s() - t0;
    e->host = h;
    e->st.host_store_bytes = cap;
    e->st.host_store_pin_seconds = h.pin_seconds;
    // release the device side exactly as a sleep would, without copying anything out
    RC(do_sleep(e, tag_mask, FMA_TIER_HOST, (flags & ~FMA_FLAG_VERIFY) | kFlagAdopt));
    (void)hd;
    image_apply(e, pi);
    return FMA_OK;
}

// ---- FILE tier (see include/fma_engine.h) -----------------------------------------------------------------------------

int fma_file_store(fma_engine_t* e, const char* path) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (!path) {
        e->file_path.clear();
        return FMA_OK;
    }
    if (!*path) return fail(FMA_EINVAL, "empty path");
    DeviceGuard guard(e->device);
    if (!e->load_ring) RC(ensure_io_windows(e));   // pinned once per engine, never inside a sleep or wake
    e->file_path = path;
    return FMA_OK;
}

int fma_image_adopt_file(fma_engine_t* e, const char* path, uint64_t tag_mask, uint32_t flags) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (!path || !tag_mask) return fail(FMA_EINVAL, "adopt needs the file and the tag mask the image was slept with");
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (const Segment& s : e->segs)
            if (!s.mapped) return fail(FMA_ESTATE, "adopt needs a fully awake engine");
    }
    FileFd f;
    f.fd = open(path, O_RDONLY | O_CLOEXEC);
    if (f.fd < 0) return fail(FMA_EIO, "cannot open %s: %s", path, strerror(errno));
    struct stat sb;
    if (fstat(f.fd, &sb) != 0 || (size_t)sb.st_size <= kImageTail) return fail(FMA_EINVAL, "%s is not an image file", path);
    const size_t cap = (size_t)sb.st_size - kImageTail;
    std::vector<char> tail(kImageTail);
    for (size_t got = 0; got < kImageTail;) {
        const ssize_t n = pread(f.fd, tail.data() + got, kImageTail - got, (off_t)(cap + got));
        if (n < 0 && errno == EINTR) continue;
        if (n <= 0) return fail(FMA_EIO, "cannot read the descriptor of %s: %s", path, n < 0 ? strerror(errno) : "the file ends early");
        got += (size_t)n;
    }
    ParsedImage pi;
    RC(image_descriptor_parse(e, tail.data(), kImageTail, cap, tag_mask, &pi));
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    if (flags & FMA_FLAG_VERIFY) {  // "sleep by adoption" (see fma_image_adopt): only if this engine's bytes ARE the image's
        std::vector<uint64_t> now;
        RC(digest_segments(e, pi.order, &now));
        for (size_t i = 0; i < pi.ds.size(); ++i)
            if (!pi.ds[i].digest_valid || pi.ds[i].digest != now[i])
                return fail(FMA_EINTEGRITY, pi.ds[i].digest_valid ? "the image holds different bytes than this engine's segments" : "the image carries no digests to compare with");
    }
    if (!e->load_ring) RC(ensure_io_windows(e));
    invalidate_shadows(e);
    RC(do_sleep(e, tag_mask, FMA_TIER_FILE, (flags & ~FMA_FLAG_VERIFY) | kFlagAdopt));
    image_apply(e, pi);
    e->image_file = path;
    return FMA_OK;
}

// ---- the same hand-over for an image PARKED in peer HBM (fma_peer_attach'ed buffer of a node-level owner) ----------------
// The buffer itself is the owner's; what has to travel is the descriptor: the owner keeps it next to the fd.

int fma_image_describe(fma_engine_t* e, int tier, void* buf, size_t cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (resident_asleep(e)) return fail(FMA_ESTATE, "part of the sleeping image is resident in this process's own HBM (option resident_bytes) and cannot be handed over: set it to 0 and sleep again");
    if (tier != e->image_tier) return fail(FMA_ESTATE, "no image sleeps in tier %d", tier);
    if (tier == FMA_TIER_FILE) return fail(FMA_ESTATE, "the sleeping image is in a file: the file itself is the hand-over (its descriptor is its tail)");
    std::vector<char> desc;
    RC(image_descriptor_build(e, tier, &desc));
    if (buf && cap >= desc.size()) memcpy(buf, desc.data(), desc.size());
    return (int)desc.size();
}

int fma_image_adopt_parked(fma_engine_t* e, const void* desc, size_t desc_bytes, uint64_t tag_mask, uint32_t flags) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (!desc || !tag_mask) return fail(FMA_EINVAL, "adopt needs the descriptor and the tag mask the image was slept with");
    if (!e->park.va || e->park.device == e->device) return fail(FMA_ESTATE, "adopt_parked needs an attached / reserved peer parking buffer first");
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (const Segment& s : e->segs)
            if (!s.mapped) return fail(FMA_ESTATE, "adopt needs a fully awake engine");
    }
    ParsedImage pi;
    RC(image_descriptor_parse(e, static_cast<const char*>(desc), desc_bytes, e->park.bytes, tag_mask, &pi));
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    if (flags & FMA_FLAG_VERIFY) {  // "sleep by adoption" (see fma_image_adopt): only if this engine's bytes ARE the image's
        std::vector<uint64_t> now;
        RC(digest_segments(e, pi.order, &now));
        for (size_t i = 0; i < pi.ds.size(); ++i)
            if (!pi.ds[i].digest_valid || pi.ds[i].digest != now[i])
                return fail(FMA_EINTEGRITY, pi.ds[i].digest_valid ? "the image holds different bytes than this engine's segments" : "the image carries no digests to compare with");
    }
    if (e->shadow_tier != FMA_TIER_HOST) invalidate_shadows(e);
    RC(do_sleep(e, tag_mask, FMA_TIER_PEER, (flags & ~FMA_FLAG_VERIFY) | kFlagAdopt));
    image_apply(e, pi);
    return FMA_OK;
}

// ---- moving a sleeping image to another tier (see include/fma_engine.h) -------------------------------------------------
int fma_image_move(fma_engine_t* e, int tier) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    const int from = e->image_tier;
    fma_layout::MoveFacts facts{};
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (const Segment& s : e->segs)
            if (s.has_backup) (s.mapped ? facts.backup_mapped : facts.asleep) = true;
    }
    facts.resident = resident_asleep(e);
    facts.prepared = tier == FMA_TIER_PEER ? e->park.va && e->park.device != e->device && e->park.bytes >= e->image_store_bytes
                   : tier == FMA_TIER_FILE ? !e->file_path.empty()
                                           : true;
    const fma_layout::MoveRoute route = fma_layout::move_route(from, tier, facts);
    if (route.error != FMA_OK) return fail(route.error, "image move from tier %d to tier %d: %s", from, tier, route.why);

    DeviceGuard guard(e->device);
    RC(flush_kernel_times(e));
    const double t_entry = now_s();
    e->tl_begin("move", t_entry);
    MoveState ms;
    const int rc = run_move(e, route.pipe, from, tier, ms);
    if (rc != FMA_OK) {
        undo_move(e, ms);   // the image stays where it was, its records untouched
        return rc;
    }
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (Segment& s : e->segs)
            if (s.has_backup && !s.mapped) s.backup_tier = tier;
    }
    e->image_tier = tier;
    if (tier == FMA_TIER_FILE) e->image_file = e->file_path;
    // INCREMENTAL: the copy a clean sleep may keep lay in the store the image left; the next wake records the new one
    invalidate_shadows(e);
    e->st.tier = tier;
    e->tl_add("total", 0, t_entry, now_s(), e->image_store_bytes);
    return FMA_OK;
}

// ---- checking a sleeping image against its digests where it lies (see include/fma_engine.h) ------------------------------
int fma_image_verify(fma_engine_t* e, int* out_bad, int cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (cap < 0 || (cap > 0 && !out_bad)) return fail(FMA_EINVAL, "out_bad is NULL or cap is negative");
    Verifier v(e);
    std::vector<size_t> main, res;   // positions in v.segs: the image's own store, the resident share
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (size_t i = 0; i < e->segs.size(); ++i) {
            const Segment& s = e->segs[i];
            if (!s.has_backup) continue;
            if (s.mapped) return fail(FMA_ESTATE, "segment %zu is mapped and keeps a backup (a KEEP_BACKUP or partial wake): wake the rest or sleep again first", i);
            if (!s.digest_valid)
                return fail(FMA_ESTATE, "segment %zu of the sleeping image carries no digest: sleep with FMA_FLAG_VERIFY or the incremental option to record them", i);
            const bool resident = s.backup_tier == FMA_TIER_LOCAL && e->image_tier == FMA_TIER_HOST;
            (resident ? res : main).push_back(v.segs.size());
            v.segs.push_back(Verifier::Seg{i, (uint64_t)s.va, s.digest});
        }
    }
    if (v.segs.empty()) return fail(FMA_ESTATE, "nothing is asleep");
    DeviceGuard guard(e->device);
    RC(flush_kernel_times(e));   // (the last operation's kernel rows and times, before the timeline turns to this call)
    const double t_entry = now_s();
    e->tl_begin("verify", t_entry);
    const int rc = v.run(main, res);
    if (e->ks) cudaStreamSynchronize(e->ks);   // nothing still reads a store or the descriptors, also after a failure
    if (rc != FMA_OK) return rc;
    int n_bad = 0;
    for (size_t k = 0; k < v.segs.size(); ++k)
        if (v.sum[k] != v.segs[k].digest) {
            if (n_bad < cap) out_bad[n_bad] = (int)v.segs[k].index;
            ++n_bad;
        }
    e->tl_add("total", n_bad, t_entry, now_s(), e->image_store_bytes + e->res_store_bytes);
    return n_bad;
}


}  // extern "C"
