// fma_image.cu — image hand-over: a sleeping model's host image outlives its engine / process (memfd store + descriptor)
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"

using namespace fma_impl;

namespace fma_impl {

namespace {

// The sleeping segments (they keep a backup and are unmapped) that `pick` takes, by engine index in image order (takes e->mu)
template <class Pick>
std::vector<size_t> sleeping_segments(fma_engine_t* e, Pick pick) {
    std::vector<size_t> v;
    std::lock_guard<std::mutex> lk(e->mu);
    for (size_t i = 0; i < e->segs.size(); ++i)
        if (e->segs[i].has_backup && !e->segs[i].mapped && pick(e->segs[i])) v.push_back(i);
    std::sort(v.begin(), v.end(), [&](size_t a, size_t b) { return e->segs[a].packed_off < e->segs[b].packed_off; });
    return v;
}

// Is a segment's image asleep (kept and unmapped), and is one mapped again while it keeps its backup (takes e->mu)?
void sleep_state(fma_engine_t* e, bool* asleep, bool* backup_mapped) {
    std::lock_guard<std::mutex> lk(e->mu);
    for (const Segment& s : e->segs)
        if (s.has_backup) *(s.mapped ? backup_mapped : asleep) = true;
}

}  // namespace

// Descriptor of the image sleeping in `tier`'s store: header, one ImageSegDesc per offloaded segment in image order and, for a
// PACKED image (version 2), the per-page stored sizes (offsets are their prefix sums).  At most kImageTail bytes.
int image_descriptor_build(fma_engine_t* e, int tier, std::vector<char>* out) {
    const std::vector<size_t> segs = sleeping_segments(e, [&](const Segment& s) {
        return tier == FMA_TIER_HOST ? s.backup_tier == FMA_TIER_HOST : s.backup_tier != FMA_TIER_HOST;
    });
    if (segs.empty()) return fail(FMA_ESTATE, "nothing is asleep in that store");
    const size_t n_img_pages = e->image_packed ? e->img_bytes.size() : 0;
    const size_t total = sizeof(ImageHeader) + segs.size() * sizeof(ImageSegDesc) + sizeof(uint32_t) * (1 + n_img_pages);
    if (total > kImageTail) return fail(FMA_ENOMEM, "too many segments / pages for the descriptor");
    out->assign(total, 0);
    char* tail = out->data();
    ImageHeader hd{kImageMagic, e->image_packed ? 2u : 1u, (uint32_t)segs.size(), e->image_bytes};
    memcpy(tail, &hd, sizeof(hd));
    for (size_t i = 0; i < segs.size(); ++i) {
        const Segment& s = e->segs[segs[i]];
        ImageSegDesc d;
        memset(&d, 0, sizeof(d));
        d.bytes = s.bytes;
        d.packed_off = s.packed_off;
        d.digest = s.digest;
        d.digest_valid = s.digest_valid ? 1 : 0;
        const std::string& t = e->tags[s.tag];
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

int image_descriptor_read(const char* tail, size_t tail_bytes, size_t store_cap, ImageDescriptor* out) {
    ImageDescriptor& pi = *out;
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
    pi.ds.resize(hd.n_segments);
    uint64_t off = 0;
    for (size_t i = 0; i < pi.ds.size(); ++i) {
        memcpy(&pi.ds[i], tail + sizeof(hd) + i * sizeof(ImageSegDesc), sizeof(ImageSegDesc));
        if (pi.ds[i].tag_len >= sizeof(pi.ds[i].tag) || pi.ds[i].digest_valid > 1) return fail(FMA_EINVAL, "image descriptor is malformed (tag length / digest flag)");
        if (pi.ds[i].packed_off != off || pi.ds[i].bytes > hd.image_bytes - off) return fail(FMA_EINVAL, "image descriptor is malformed (segment offsets)");
        off += pi.ds[i].bytes;
    }
    if (off != hd.image_bytes) return fail(FMA_EINVAL, "image size mismatch");
    return FMA_OK;
}

namespace {

// A descriptor matched against the engine's segments for `tag_mask` (same order rule as fma_sleep).
struct ParsedImage : ImageDescriptor {
    std::vector<size_t> order;          // engine segment index of descriptor entry i
};

int image_descriptor_parse(fma_engine_t* e, const char* tail, size_t tail_bytes, size_t store_cap, uint64_t tag_mask, ParsedImage* out) {
    ParsedImage& pi = *out;
    RC(image_descriptor_read(tail, tail_bytes, store_cap, &pi));
    const ImageHeader& hd = pi.hd;
    std::lock_guard<std::mutex> lk(e->mu);
    for (size_t i = 0; i < e->segs.size(); ++i)
        if (tag_bit_set(tag_mask, e->segs[i].tag)) pi.order.push_back(i);
    std::sort(pi.order.begin(), pi.order.end(), [&](size_t a, size_t b) {
        const Segment &x = e->segs[a], &y = e->segs[b];
        return x.arena != y.arena ? x.arena < y.arena : x.va < y.va;
    });
    if (pi.order.size() != hd.n_segments) return fail(FMA_EINVAL, "image and engine disagree on the number of segments");
    uint64_t off = 0;
    for (size_t i = 0; i < pi.ds.size(); ++i) {
        const Segment& s = e->segs[pi.order[i]];
        if (pi.ds[i].bytes != s.bytes || pi.ds[i].packed_off != off || std::string(pi.ds[i].tag, pi.ds[i].tag_len) != e->tags[s.tag])
            return fail(FMA_EINVAL, "image and engine disagree on a segment's size, offset or tag");
        off += s.bytes;
    }
    if (off != hd.image_bytes) return fail(FMA_EINVAL, "image size mismatch");
    return FMA_OK;
}

// after do_sleep(kFlagAdopt): take over the exporter's page table and integrity data (caller holds e->mu)
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

// An adoption releases the device side as a sleep would: every segment must be mapped (takes e->mu)
int adopt_needs_awake(fma_engine_t* e) {
    std::lock_guard<std::mutex> lk(e->mu);
    for (const Segment& s : e->segs)
        if (!s.mapped) return fail(FMA_ESTATE, "adopt needs a fully awake engine");
    return FMA_OK;
}

// What every adoption does once its entry point holds the descriptor (`desc`, the image's store: store_cap bytes): parse it against
// the segments of `tag_mask`; with FMA_FLAG_VERIFY, check that the device holds what the image holds; take_store() sets the store
// up; then the device side goes exactly as a sleep to `tier` would release it, without copying anything out, and the engine takes
// over the exporter's page table and digests.
template <class TakeStore>
int adopt(fma_engine_t* e, const char* desc, size_t desc_bytes, size_t store_cap, uint64_t tag_mask, uint32_t flags, int tier, TakeStore take_store) {
    ParsedImage pi;
    RC(image_descriptor_parse(e, desc, desc_bytes, store_cap, tag_mask, &pi));
    DeviceGuard guard(e->device);
    cudaDeviceSynchronize();
    if (flags & FMA_FLAG_VERIFY) {
        // "Sleep by adoption": this engine HAS the weights and wants to share somebody else's image of the same model (a second
        // replica on the node: one host copy for all).  Only legal if its device bytes are what the image holds — K3 digests
        // against the descriptor's; a mismatch leaves the engine awake and untouched.
        std::vector<uint64_t> now;
        RC(digest_segments(e, pi.order, &now));
        for (size_t i = 0; i < pi.ds.size(); ++i)
            if (!pi.ds[i].digest_valid || pi.ds[i].digest != now[i])
                return fail(FMA_EINTEGRITY, pi.ds[i].digest_valid ? "the image holds different bytes than this engine's segments" : "the image carries no digests to compare with");
    }
    RC(take_store());
    RC(do_sleep(e, tag_mask, tier, (flags & ~FMA_FLAG_VERIFY) | kFlagAdopt));
    std::lock_guard<std::mutex> lk(e->mu);
    image_apply(e, pi);
    return FMA_OK;
}

// An exported image's memfd (a dup of it) and its shared mapping: unmapped and closed on every exit path, unless the host store
// takes them over
struct ImageMapping {
    int fd = -1;
    void* base = nullptr;
    size_t bytes = 0;
    ~ImageMapping() {
        if (base) munmap(base, bytes);
        if (fd >= 0) close(fd);
    }
};

// The adopted memfd image becomes the host store: pinned in place, or copied once into anonymous pinned memory
int adopt_host_store(fma_engine_t* e, ImageMapping& m) {
    const size_t cap = m.bytes - kImageTail;
    invalidate_shadows(e);
    host_store_free(e->host);
    const double t0 = now_s();
    void* p = m.base;
    cudaError_t r = cudaHostRegister(p, m.bytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
    HostStore h;
    if (r != cudaSuccess) {
        // The mapping cannot be pinned in place (e.g. an image FILE on a filesystem whose pages the driver will not lock):
        // copy it once into an anonymous pinned store — a load from the page cache, several threads — and let go of the fd.
        cudaGetLastError();
        void* q = nullptr;
        r = cudaHostAlloc(&q, m.bytes, cudaHostAllocPortable | cudaHostAllocMapped);
        if (r != cudaSuccess) {
            cudaGetLastError();
            return fail(FMA_ENOMEM, "cannot pin the adopted image, in place or as a copy");
        }
        const int nt = std::max(1, std::min(env_int("FMA_TOUCH_THREADS", 8), 32));
        const size_t per = round_up((m.bytes + nt - 1) / nt, FMA_PAGE_BYTES);
        std::vector<std::thread> th;
        for (int t = 0; t < nt; ++t) {
            const size_t lo = (size_t)t * per, hi = std::min(m.bytes, lo + per);
            if (lo >= hi) break;
            th.emplace_back([p, q, lo, hi] { memcpy(static_cast<char*>(q) + lo, static_cast<const char*>(p) + lo, hi - lo); });
        }
        for (auto& t : th) t.join();
        h.base = q; h.cap = cap; h.map_bytes = 0; h.fd = -1; h.registered = false;
        p = q;
    } else {
        h.base = p; h.cap = cap; h.map_bytes = m.bytes; h.fd = m.fd; h.registered = true;
        h.shared = true;  // the exporter (and other adopters) map the same pages
        m.base = nullptr;   // the store's now
        m.fd = -1;
    }
    void* alias = nullptr;
    if (cudaHostGetDevicePointer(&alias, p, 0) == cudaSuccess) h.dev_alias = alias;
    else cudaGetLastError();
    h.pin_seconds = now_s() - t0;
    e->host = h;
    e->st.host_store_bytes = cap;
    e->st.host_store_pin_seconds = h.pin_seconds;
    return FMA_OK;
}

// ---- copies between a store and an HBM buffer, for moves and prefetches ----

// Nothing the engine's streams were given still runs (a failure's clean-up, before what they copy into or out of goes)
inline void drain(fma_engine_t* e) {
    for (int i = 0; i < e->n_cs; ++i) cudaStreamSynchronize(e->cs[i]);
    if (e->ks) cudaStreamSynchronize(e->ks);
    cudaGetLastError();
}

// Copies store ranges into (to_hbm) or out of the HBM buffer `hbm`: range r (its offset in the store, its bytes) is at hbm + at[r].
// The host store: direct_chunk pieces round-robin over the copy streams.  A file (io: the readers or writers of
// FileIO::cut(ranges)): one copy per window item, item k on copy stream k % n_cs.  *ops counts the copies.
int copy_ranges(fma_engine_t* e, const std::vector<FileIO::Item>& ranges, const std::vector<uint64_t>& at, char* hbm, bool to_hbm, FileIO* io,
                uint32_t* ops) {
    if (io) {
        std::vector<size_t> ends;
        const std::vector<FileIO::Item> items = FileIO::cut(e, ranges, &ends);
        for (size_t k = 0, r = 0; k < items.size(); ++k, ++*ops) {
            while (k >= ends[r]) ++r;
            RC(io->copy(k, hbm + at[r] + (items[k].file_off - ranges[r].file_off), e->cs[k % e->n_cs]));
        }
        return io->finish();   // every pread / pwrite has returned and every copy into or out of a window has finished
    }
    char* host = static_cast<char*>(e->host.base);
    if (!host) return fail(FMA_ESTATE, "the host store that holds the image is gone");
    const size_t chunk = direct_chunk(e);
    for (size_t r = 0; r < ranges.size(); ++r)
        for (uint64_t o = 0; o < ranges[r].bytes; o += chunk, ++*ops) {
            const size_t n = (size_t)std::min<uint64_t>(chunk, ranges[r].bytes - o);
            char* h = host + ranges[r].file_off + o;
            char* d = hbm + at[r] + o;
            RT(cudaMemcpyAsync(to_hbm ? d : h, to_hbm ? h : d, n, cudaMemcpyDefault, e->cs[*ops % e->n_cs]));
        }
    return FMA_OK;
}

// The copy engines' part of an operation, timed on the engine's streams only: the CopyTimer bracket around copy(), which counts
// the copies it enqueues in *ops, and the "copies_landed" row over `bytes`
template <class Copy>
int timed_copies(fma_engine_t* e, uint64_t bytes, uint32_t* ops, Copy copy) {
    RC(ensure_streams(e));
    CopyTimer timer{e};
    const double t0 = now_s();
    RC(timer.begin());
    RC(copy());
    double copy_s = 0;
    RC(timer.end(&copy_s));   // joins the copy streams only
    e->tl_add("copies_landed", (int)*ops, t0, now_s(), bytes);
    return FMA_OK;
}

// ---- moves of a sleeping image between tiers (fma_image_move) ----
// Every tier holds the image in one layout (plain pages back to back, or the PACKED form's stored pages at img_off[p]), so a move
// copies image_store_bytes bytes from offset 0 of one store to offset 0 of the other and changes nothing but the engine's records.

// The items of a move between the pinned host store and a file: FileIO's threads pread / pwrite them straight into / out of the
// store, no copy engine involved.
std::vector<FileIO::Item> move_host_file(const fma_engine_t* e, uint64_t bytes) {
    const uint64_t piece = round_up(std::max<size_t>(e->load_chunk, 4096), 4096);
    std::vector<FileIO::Item> items;
    for (uint64_t o = 0; o < bytes; o += piece) items.push_back(FileIO::Item{o, std::min(piece, bytes - o)});
    return items;
}

// What a move has set up so far, so that a failure can undo it
struct MoveState {
    explicit MoveState(fma_engine_t* e) : file(e) {}
    ImageFile file;
    bool file_emptied = false;   // the destination file has been emptied: a failure leaves no descriptor in it
    bool made_host = false;      // the host store, or the local parking buffer, was created by this move
    bool made_park = false;
    bool copies = false;         // the copy streams ran
    HostStore old_host;          // what the created store or buffer replaces: released once the move has succeeded, kept if it fails
    uint64_t old_host_bytes = 0;
    ParkStore old_park;
};

int run_move(fma_engine_t* e, fma_layout::MovePipeKind pipe, int from, int to, MoveState& ms) {
    using fma_layout::MovePipeKind;
    const uint64_t bytes = e->image_store_bytes;
    const bool park_side = pipe != MovePipeKind::HostFile && pipe != MovePipeKind::FileHost;
    ms.copies = park_side;
    // the destination, prepared as a sleep to its tier prepares it
    // (a shared host store is read-only: its other holders keep it, and this engine takes a private one)
    if (to == FMA_TIER_HOST) {
        ms.made_host = e->host.shared || !e->host.base || e->host.cap < round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), FMA_PAGE_BYTES);
        if (ms.made_host) {   // a store that does not fit holds nothing of this image, but it goes only once the move has succeeded
            invalidate_shadows(e);
            ms.old_host = e->host;
            ms.old_host_bytes = e->st.host_store_bytes;
            e->host = HostStore{};
            e->st.host_store_bytes = 0;
        }
        RC(host_store_reserve(e, bytes));
    } else if (to == FMA_TIER_LOCAL) {
        const size_t need = round_up(std::max<size_t>(bytes, FMA_PAGE_BYTES), e->gran);
        ms.made_park = !(e->park.va && e->park.device == e->device && e->park.bytes >= need);
        if (ms.made_park) {   // likewise a buffer that does not fit, or a peer's (an attached one included)
            ms.old_park = e->park;
            e->park = ParkStore{};
            RC(park_store_create(e, e->device, need, &e->park));
        }
    }
    // the file side: the destination emptied once the filesystem has room; the source checked to hold the whole image.  A
    // parking buffer's bytes go through the engine's pinned I/O windows (the file tier's disk stage without the HBM ring).
    std::optional<FileIO> io;
    if (to == FMA_TIER_FILE || from == FMA_TIER_FILE) {
        std::vector<FileIO::Item> items = park_side ? FileIO::cut(e, {FileIO::Item{0, bytes}}) : move_host_file(e, bytes);
        char* mem = park_side ? nullptr : static_cast<char*>(e->host.base);
        if (to == FMA_TIER_FILE) {
            RC(ms.file.create(e->file_path, bytes));
            ms.file_emptied = true;
            ms.file.write(std::move(items), &io, mem);
        } else {
            RC(ms.file.read(e->image_file, std::move(items), &io, mem));
        }
    }
    // the bytes
    uint32_t ops = 0;
    if (park_side) {
        const bool to_park = fma_layout::is_park_tier(to);
        RC(timed_copies(e, bytes, &ops, [&] {
            return copy_ranges(e, {FileIO::Item{0, bytes}}, {0}, reinterpret_cast<char*>(e->park.va), to_park, io ? &*io : nullptr, &ops);
        }));
    } else {
        RC(io->finish());
    }
    // a file written by a move is completed as a file-tier sleep completes it: it opens with fma_image_adopt_file and image_load
    if (to == FMA_TIER_FILE) {
        RC(ms.file.seal(from));
    } else if (from == FMA_TIER_FILE) {
        RC(ms.file.finish(*io));
    }
    e->st.copy_ops = ops;
    e->st.total_copy_ops += ops;
    return FMA_OK;
}

// A failed move: nothing may still copy into what goes, what the move created goes (the store or buffer it replaced comes back),
// and a destination file keeps no descriptor
void undo_move(fma_engine_t* e, MoveState& ms) {
    if (ms.copies) drain(e);
    if (ms.made_host) {   // the store the engine had before, as it was
        host_store_free(e->host);
        e->host = ms.old_host;
        e->st.host_store_bytes = ms.old_host_bytes;
    }
    if (ms.made_park) {
        vmm_buffer_free(e->park);
        e->park = ms.old_park;
    }
    if (ms.file_emptied) {   // what was written goes too (best effort: without its descriptor the file is refused anyway)
        const int r = ftruncate(ms.file.fd(), 0);
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
    // prefetched: the segments' copies in the prefetch buffer (offsets prefetch_off), not the store's.
    int plan(const std::vector<size_t>& pos, const std::vector<uint64_t>* off, const std::vector<uint32_t>* bytes, std::vector<PagePlan>* pages,
             bool prefetched = false) {
        std::vector<fma_layout::SegPages> v;
        for (size_t k : pos) {
            const Segment& s = e->segs[segs[k].index];
            v.push_back(fma_layout::SegPages{s.va, s.bytes, prefetched ? s.prefetch_off : s.packed_off, k});
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
        const uint64_t window = FileIO::max_item(e);
        std::vector<Batch> batches;
        if (!fma_layout::plan_batches(pages, SIZE_MAX, window, true, &batches))
            return fail(FMA_EINVAL, "a stored page does not fit an I/O window of %llu bytes", (unsigned long long)window);
        std::vector<FileIO::Item> items;
        for (const Batch& b : batches) items.push_back(FileIO::Item{pages[b.p0].off, b.stored});
        ImageFile file(e);
        std::optional<FileIO> io;
        RC(file.read(e->image_file, std::move(items), &io));
        for (size_t c = 0; c < batches.size(); ++c) {
            const Batch& b = batches[c];
            RC(io->read_in_place(c, e->ks, [&](const char* win) {
                return launch(pages, at, b, [&](size_t q) { return (uint64_t)(uintptr_t)win + (pages[q].off - pages[b.p0].off); });
            }));
        }
        return file.finish(*io);   // every read has returned and every kernel over a window has finished
    }

    int run(const std::vector<size_t>& main, const std::vector<size_t>& res, const std::vector<size_t>& pf) {
        std::vector<PagePlan> mp, rp, fp;
        RC(plan(main, e->image_packed ? &e->img_off : nullptr, &e->img_bytes, &mp));
        RC(plan(res, e->res_packed ? &e->res_off : nullptr, &e->res_bytes, &rp));
        RC(plan(pf, e->image_packed ? &e->pf_off : nullptr, &e->pf_bytes, &fp, true));
        const size_t n = mp.size() + rp.size() + fp.size();
        RC(ensure_streams(e));
        RC(ensure_desc(e, n));
        seg_of.assign(n, 0);
        RT(cudaEventRecord(e->ev_start, e->ks));
        e->tl_dev_base = now_s() - e->tl_entry;
        RT(cudaMemsetAsync(e->d_dig, 0, n * sizeof(uint64_t), e->ks));
        const auto coded = [](const PagePlan& q) { return q.bytes != FMA_PAGE_BYTES; };
        if (std::any_of(mp.begin(), mp.end(), coded) || std::any_of(rp.begin(), rp.end(), coded) || std::any_of(fp.begin(), fp.end(), coded)) {
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
        if (!fp.empty()) {   // the prefetched copy, checked in HBM beside the store it came from
            if (!e->pf.va) return fail(FMA_ESTATE, "the prefetched part of the image is gone");
            RC(in_place(fp, mp.size() + rp.size(), (uint64_t)e->pf.va));
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

// ---- prefetching part of a sleeping image into its GPU's HBM (fma_image_prefetch) ----
// The segments a budget takes, in image order, and the copies that bring them: store range r (file_off = its offset in the store)
// lands at at[r] in the buffer.  The buffer holds the segments back to back, so store-adjacent segments make one range.
struct PrefetchPlan {
    std::vector<size_t> segs;           // engine indices
    std::vector<uint64_t> seg_off;      // their prefetch_off
    std::vector<uint64_t> off;          // PACKED: stored offset and size of each page of the prefetched part
    std::vector<uint32_t> bytes;
    std::vector<FileIO::Item> ranges;
    std::vector<uint64_t> at;
    uint64_t stored = 0;
};

int plan_prefetch(fma_engine_t* e, uint64_t budget, PrefetchPlan* p) {
    const std::vector<size_t> order = sleeping_segments(e, [](const Segment&) { return true; });
    std::vector<uint64_t> stored(order.size(), 0);
    for (size_t k = 0; k < order.size(); ++k) {
        const Segment& s = e->segs[order[k]];
        if (!e->image_packed) {
            stored[k] = s.bytes;
            continue;
        }
        const uint64_t p0 = s.packed_off / FMA_PAGE_BYTES, np = s.bytes / FMA_PAGE_BYTES;
        if (p0 + np > e->img_bytes.size()) return fail(FMA_ESTATE, "segment %zu lies outside the packed image's page table", order[k]);
        for (uint64_t q = p0; q < p0 + np; ++q) stored[k] += e->img_bytes[q];
    }
    const std::vector<char> keep = fma_layout::resident_split(stored, budget);
    uint64_t image_off = 0;
    for (size_t k = 0; k < order.size(); ++k) {
        if (!keep[k]) continue;
        const Segment& s = e->segs[order[k]];
        const uint64_t p0 = s.packed_off / FMA_PAGE_BYTES;
        const uint64_t from = e->image_packed ? e->img_off[p0] : s.packed_off;
        p->segs.push_back(order[k]);
        p->seg_off.push_back(image_off);
        image_off += s.bytes;
        if (e->image_packed)
            for (uint64_t q = p0; q < p0 + s.bytes / FMA_PAGE_BYTES; ++q) {
                p->off.push_back(p->stored + (e->img_off[q] - from));
                p->bytes.push_back(e->img_bytes[q]);
            }
        if (!p->ranges.empty() && p->ranges.back().file_off + p->ranges.back().bytes == from) {
            p->ranges.back().bytes += stored[k];
        } else {
            p->ranges.push_back(FileIO::Item{from, stored[k]});
            p->at.push_back(p->stored);
        }
        p->stored += stored[k];
    }
    return FMA_OK;
}

// The copies into `dst` (the new buffer), timed on the engine's streams only.  From a file, reader threads pread the ranges into
// the pinned I/O windows, one H2D per window.
int prefetch_copy(fma_engine_t* e, const PrefetchPlan& p, char* dst) {
    ImageFile file(e);
    std::optional<FileIO> io;
    uint32_t ops = 0;
    return timed_copies(e, p.stored, &ops, [&] {
        if (e->image_tier != FMA_TIER_FILE) return copy_ranges(e, p.ranges, p.at, dst, true, nullptr, &ops);
        if (!e->load_ring) RC(ensure_io_windows(e));
        RC(file.read(e->image_file, FileIO::cut(e, p.ranges), &io));
        RC(copy_ranges(e, p.ranges, p.at, dst, true, &*io, &ops));
        return file.finish(*io);
    });
}

// ---- WRITE-BEHIND: the file of a file-tier sleep written after the sleep returned (see include/fma_engine.h) ----------------

// Under op_mu, once the file is complete: the image moves to the file tier as fma_image_move(FMA_TIER_FILE) moves it, and the host
// store is detached for the job to free after the lock.  A descriptor that no longer describes the sleeping image (a segment freed
// while the job wrote) is not committed.
bool writeback_commit(fma_engine_t* e, const std::string& path, const std::vector<char>& desc, HostStore* detached) {
    std::vector<char> now;
    if (image_descriptor_build(e, FMA_TIER_HOST, &now) != FMA_OK || now != desc) return false;
    {
        std::lock_guard<std::mutex> lk(e->mu);   // (fma_segment_info and fma_stats read these without op_mu)
        for (Segment& s : e->segs)
            if (s.has_backup && !s.mapped) s.backup_tier = FMA_TIER_FILE;
        e->st.tier = FMA_TIER_FILE;
        e->st.host_store_bytes = 0;
    }
    e->image_tier = FMA_TIER_FILE;
    e->image_file = path;
    invalidate_shadows(e);   // (the copy a clean sleep may keep lay in the store the image left)
    *detached = e->host;
    e->host = HostStore{};
    return true;
}

// The job's thread: the FileIO writers pwrite the store straight into the file, the descriptor seals it, and the commit takes op_mu
// unless a call that holds it has cancelled the job meanwhile.  The file keeps no descriptor unless the image moved to it.
void writeback_run(fma_engine_t* e, std::unique_ptr<ImageFile> file, std::vector<char> desc, std::vector<FileIO::Item> items, char* store,
                   int item_delay_ms) {
    WriteBehind& wb = e->wb;
    cudaSetDevice(e->device);
    auto cancelled = [&] {
        std::lock_guard<std::mutex> lk(wb.mu);
        return wb.cancel;
    };
    file->restart_clock();
    std::optional<FileIO> io;
    file->write(std::move(items), &io, store, item_delay_ms);
    {
        std::lock_guard<std::mutex> lk(wb.mu);
        wb.io = &*io;
        if (wb.cancel) io->cancel();
    }
    int rc = io->finish();   // every writer has left
    {
        std::lock_guard<std::mutex> lk(wb.mu);
        wb.written = std::min<uint64_t>(io->written() * wb.piece, wb.bytes);
        wb.io = nullptr;
    }
    io.reset();
    if (rc == FMA_OK && !cancelled()) rc = file->seal_with(desc);
    const double t_file = now_s();
    char msg[512];
    snprintf(msg, sizeof(msg), "write-behind of %.200s: %.280s", file->path().c_str(), tl_err);
    bool locked = false;   // the commit's op_mu, or the cancel of the call that holds it
    while (rc == FMA_OK && !locked) {
        locked = e->op_mu.try_lock();
        if (locked) break;
        std::unique_lock<std::mutex> lk(wb.mu);
        if (wb.cv.wait_for(lk, std::chrono::milliseconds(1), [&] { return wb.cancel; })) break;
    }
    HostStore detached;
    bool committed = false;
    if (locked) {
        committed = writeback_commit(e, file->path(), desc, &detached);
        DeviceGuard guard(e->device);
        flush_kernel_times(e);   // (the sleep's kernel rows belong to the sleep's timeline)
        e->tl_begin("writeback", wb.t_entry);
        ImageFile::file_io_row(e, file->direct(), file->started(), t_file, wb.written + (committed ? kImageTail : 0));
        e->tl_add("total", committed ? 1 : 0, wb.t_entry, now_s(), wb.written);
    }
    if (!committed) {   // cancelled or failed: what was written goes (without its descriptor the file is refused anyway)
        const int r = ftruncate(file->fd(), 0);
        (void)r;
    }
    {
        std::lock_guard<std::mutex> lk(wb.mu);
        wb.direct = file->direct();
        wb.file_t0 = file->started();
        wb.file_t1 = t_file;
        if (committed) {
            wb.state = WriteBehind::Committed;
        } else if (rc != FMA_OK && rc != FileIO::kCancelled) {
            wb.state = WriteBehind::Failed;
            wb.error = rc;
            wb.reported = false;
            snprintf(wb.msg, sizeof(wb.msg), "%s", msg);
        } else {
            wb.state = WriteBehind::Cancelled;
        }
    }
    wb.cv.notify_all();
    if (locked) e->op_mu.unlock();
    file.reset();
    host_store_free(detached);   // after the lock: a wake does not wait for cudaHostUnregister + munmap
    cudaGetLastError();
}

}  // namespace

void writeback_join(fma_engine_t* e) {
    if (e->wb.th.joinable()) e->wb.th.join();
}

void writeback_start(fma_engine_t* e, std::unique_ptr<ImageFile> file) {
    WriteBehind& wb = e->wb;
    writeback_join(e);   // a committed job may still be freeing its store
    const uint64_t bytes = e->image_store_bytes;
    std::vector<FileIO::Item> items = move_host_file(e, bytes);
    std::vector<char> desc;   // built now, under op_mu: the job reads nothing of the engine's records
    const int rc = image_descriptor_build(e, FMA_TIER_HOST, &desc);
    std::lock_guard<std::mutex> lk(wb.mu);
    wb.cancel = false;
    wb.io = nullptr;
    wb.bytes = bytes;
    wb.piece = items.empty() ? 0 : items[0].bytes;
    wb.written = 0;
    wb.t_entry = now_s();
    if (rc != FMA_OK) {   // the image stays in the host tier; the file, emptied by the sleep, stays empty
        wb.state = WriteBehind::Failed;
        wb.error = rc;
        wb.reported = false;
        snprintf(wb.msg, sizeof(wb.msg), "write-behind of %.200s: %.280s", file->path().c_str(), tl_err);
        return;
    }
    wb.state = WriteBehind::Writing;
    wb.error = FMA_OK;
    wb.reported = true;
    wb.th = std::thread(writeback_run, e, std::move(file), std::move(desc), std::move(items), static_cast<char*>(e->host.base),
                        env_int("FMA_WB_ITEM_DELAY_MS", 0));
}

void writeback_preempt(fma_engine_t* e) {
    WriteBehind& wb = e->wb;
    {
        std::lock_guard<std::mutex> lk(wb.mu);
        if (wb.state != WriteBehind::Writing) return;
        wb.cancel = true;
        if (wb.io) wb.io->cancel();
    }
    wb.cv.notify_all();
    const double t0 = now_s();
    wb.th.join();   // at most the pwrite each writer has in flight, or an fdatasync
    const double t1 = now_s();
    if (wb.state != WriteBehind::Cancelled) return;   // (failed first: fma_image_writeback reports it)
    DeviceGuard guard(e->device);
    flush_kernel_times(e);
    e->tl_begin("writeback", wb.t_entry);
    ImageFile::file_io_row(e, wb.direct, wb.file_t0, wb.file_t1, wb.written);
    e->tl_add("total", 0, wb.t_entry, t1, wb.written);
    e->tl_add("wb_cancel", 0, t0, t1, wb.written);
    e->tl_carry = true;   // the caller's own timeline, if it starts one, opens with this row
    e->tl_carry_t0 = t0;
    e->tl_carry_t1 = t1;
    e->tl_carry_bytes = wb.written;
}

}  // namespace fma_impl

extern "C" {

int fma_image_writeback(fma_engine_t* e, double timeout_s, uint64_t* out_pending_bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    WriteBehind& wb = e->wb;
    std::unique_lock<std::mutex> lk(wb.mu);
    const auto settled = [&] { return wb.state != WriteBehind::Writing; };
    if (timeout_s < 0 || std::isinf(timeout_s)) wb.cv.wait(lk, settled);
    else if (timeout_s > 0) wb.cv.wait_for(lk, std::chrono::duration<double>(timeout_s), settled);
    if (out_pending_bytes) *out_pending_bytes = 0;
    if (wb.state == WriteBehind::Writing) {
        if (out_pending_bytes) *out_pending_bytes = wb.bytes - (wb.io ? std::min<uint64_t>(wb.io->written() * wb.piece, wb.bytes) : wb.written);
        return 1;
    }
    if (wb.state == WriteBehind::Failed && !wb.reported) {   // once per failure, on the caller's thread
        wb.reported = true;
        return fail(wb.error, "%s", wb.msg);
    }
    return FMA_OK;
}

int fma_image_export(fma_engine_t* e, int* out_fd) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
    if (!out_fd) return fail(FMA_EINVAL, "out_fd is NULL");
    RC(refuse_resident_handover(e));
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
    OpLock op(e);
    if (!tag_mask) return fail(FMA_EINVAL, "adopt needs the tag mask the image was slept with");
    RC(adopt_needs_awake(e));
    struct stat sb;
    if (fstat(fd, &sb) != 0 || (size_t)sb.st_size <= kImageTail) return fail(FMA_EINVAL, "not an image fd");
    ImageMapping m;
    m.bytes = (size_t)sb.st_size;
    const size_t cap = m.bytes - kImageTail;
    m.fd = dup(fd);
    if (m.fd < 0) return fail(FMA_ENOMEM, "dup failed: %s", strerror(errno));
    void* p = mmap(nullptr, m.bytes, PROT_READ | PROT_WRITE, MAP_SHARED, m.fd, 0);
    if (p == MAP_FAILED) return fail(FMA_ENOMEM, "cannot map the image: %s", strerror(errno));
    m.base = p;
    return adopt(e, static_cast<const char*>(p) + cap, kImageTail, cap, tag_mask, flags, FMA_TIER_HOST, [&] { return adopt_host_store(e, m); });
}

// ---- FILE tier (see include/fma_engine.h) -----------------------------------------------------------------------------

int fma_file_store(fma_engine_t* e, const char* path) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
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
    OpLock op(e);
    if (!path || !tag_mask) return fail(FMA_EINVAL, "adopt needs the file and the tag mask the image was slept with");
    RC(adopt_needs_awake(e));
    FileFd f;
    size_t cap = 0;
    std::vector<char> tail;
    RC(ImageFile::read_tail(path, FMA_EINVAL, &f, &cap, &tail));
    RC(adopt(e, tail.data(), kImageTail, cap, tag_mask, flags, FMA_TIER_FILE, [&] {
        if (!e->load_ring) RC(ensure_io_windows(e));
        invalidate_shadows(e);
        return FMA_OK;
    }));
    e->image_file = path;
    return FMA_OK;
}

// ---- the same hand-over for an image PARKED in peer HBM (fma_peer_attach'ed buffer of a node-level owner) ----------------
// The buffer itself is the owner's; what has to travel is the descriptor: the owner keeps it next to the fd.

int fma_image_describe(fma_engine_t* e, int tier, void* buf, size_t cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
    RC(refuse_resident_handover(e));
    if (tier != e->image_tier) return fail(FMA_ESTATE, "no image sleeps in tier %d", tier);
    if (tier == FMA_TIER_FILE) return fail(FMA_ESTATE, "the sleeping image is in a file: the file itself is the hand-over (its descriptor is its tail)");
    std::vector<char> desc;
    RC(image_descriptor_build(e, tier, &desc));
    if (buf && cap >= desc.size()) memcpy(buf, desc.data(), desc.size());
    return (int)desc.size();
}

int fma_image_adopt_parked(fma_engine_t* e, const void* desc, size_t desc_bytes, uint64_t tag_mask, uint32_t flags) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
    if (!desc || !tag_mask) return fail(FMA_EINVAL, "adopt needs the descriptor and the tag mask the image was slept with");
    if (!e->park.va || e->park.device == e->device) return fail(FMA_ESTATE, "adopt_parked needs an attached / reserved peer parking buffer first");
    RC(adopt_needs_awake(e));
    return adopt(e, static_cast<const char*>(desc), desc_bytes, e->park.bytes, tag_mask, flags, FMA_TIER_PEER, [&] {
        if (e->shadow_tier != FMA_TIER_HOST) invalidate_shadows(e);
        return FMA_OK;
    });
}

// ---- moving a sleeping image to another tier (see include/fma_engine.h) -------------------------------------------------
int fma_image_move(fma_engine_t* e, int tier) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
    const int from = e->image_tier;
    fma_layout::MoveFacts facts{};
    sleep_state(e, &facts.asleep, &facts.backup_mapped);
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
    MoveState ms(e);
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
    host_store_free(ms.old_host);   // (what the new store or buffer replaced: nothing of the image was in it)
    vmm_buffer_free(ms.old_park);
    e->image_tier = tier;
    if (tier == FMA_TIER_FILE) e->image_file = e->file_path;
    if (fma_layout::is_park_tier(tier)) prefetch_release(e);   // the whole image is in HBM now; host <-> file keeps the copy
    // INCREMENTAL: the copy a clean sleep may keep lay in the store the image left; the next wake records the new one
    invalidate_shadows(e);
    e->st.tier = tier;
    e->tl_add("total", 0, t_entry, now_s(), e->image_store_bytes);
    return FMA_OK;
}

// ---- checking a sleeping image against its digests where it lies (see include/fma_engine.h) ------------------------------
int fma_image_verify(fma_engine_t* e, int* out_bad, int cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
    if (cap < 0 || (cap > 0 && !out_bad)) return fail(FMA_EINVAL, "out_bad is NULL or cap is negative");
    Verifier v(e);
    std::vector<size_t> main, res, pf;   // positions in v.segs: the image's own store, the resident share, the prefetched copy
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
            if (s.prefetch_off != kNoOffset) {   // checked a second time, where the wake will read it
                pf.push_back(v.segs.size());
                v.segs.push_back(Verifier::Seg{i, (uint64_t)s.va, s.digest});
            }
        }
    }
    if (v.segs.empty()) return fail(FMA_ESTATE, "nothing is asleep");
    DeviceGuard guard(e->device);
    RC(flush_kernel_times(e));   // (the last operation's kernel rows and times, before the timeline turns to this call)
    const double t_entry = now_s();
    e->tl_begin("verify", t_entry);
    const int rc = v.run(main, res, pf);
    if (e->ks) cudaStreamSynchronize(e->ks);   // nothing still reads a store or the descriptors, also after a failure
    if (rc != FMA_OK) return rc;
    int n_bad = 0;
    for (size_t k = 0; k < v.segs.size(); ++k)   // a segment checked in two places and bad in both counts once
        if (v.sum[k] != v.segs[k].digest && (k == 0 || v.segs[k - 1].index != v.segs[k].index || v.sum[k - 1] == v.segs[k - 1].digest)) {
            if (n_bad < cap) out_bad[n_bad] = (int)v.segs[k].index;
            ++n_bad;
        }
    e->tl_add("total", n_bad, t_entry, now_s(), e->image_store_bytes + e->res_store_bytes + e->pf_store_bytes.load());
    return n_bad;
}

// ---- prefetching part of a sleeping image into HBM ahead of a wake (see include/fma_engine.h) ------------------------------
int fma_image_prefetch(fma_engine_t* e, uint64_t bytes) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    OpLock op(e);
    DeviceGuard guard(e->device);
    if (!bytes) {   // the hand-back: nothing on the device reads the buffer between operations
        prefetch_release(e);
        return FMA_OK;
    }
    fma_layout::PrefetchFacts facts{e->image_tier, false, false, e->res.va != 0};
    sleep_state(e, &facts.asleep, &facts.backup_mapped);
    const fma_layout::PrefetchRoute route = fma_layout::prefetch_route(facts);
    if (route.error != FMA_OK) return fail(route.error, "image prefetch: %s", route.why);
    RC(flush_kernel_times(e));   // (the last operation's kernel rows and times, before the timeline turns to this call)
    const double t_entry = now_s();
    e->tl_begin("prefetch", t_entry);
    prefetch_release(e);   // a new prefetch replaces the old one, whose HBM goes first
    PrefetchPlan p;
    RC(plan_prefetch(e, bytes & ~(uint64_t)(FMA_PAGE_BYTES - 1), &p));
    if (p.stored) {
        ParkStore buf;
        RC(park_store_create(e, e->device, p.stored, &buf));
        const int rc = prefetch_copy(e, p, reinterpret_cast<char*>(buf.va));
        if (rc != FMA_OK) {   // nothing may still copy into the buffer when it goes
            drain(e);
            vmm_buffer_free(buf);
            return rc;
        }
        {
            std::lock_guard<std::mutex> lk(e->mu);
            for (size_t k = 0; k < p.segs.size(); ++k) e->segs[p.segs[k]].prefetch_off = p.seg_off[k];
        }
        e->pf = buf;
        e->pf_off = std::move(p.off);
        e->pf_bytes = std::move(p.bytes);
        e->pf_store_bytes = p.stored;
    }
    e->tl_add("total", (int)p.segs.size(), t_entry, now_s(), p.stored);
    return FMA_OK;
}

}  // extern "C"
