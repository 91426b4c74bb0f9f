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

}  // namespace
}  // namespace fma_impl

extern "C" {

int fma_image_export(fma_engine_t* e, int* out_fd) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (!out_fd) return fail(FMA_EINVAL, "out_fd is NULL");
    if (resident_asleep(e)) return fail(FMA_ESTATE, "part of the sleeping image is resident in this process's own HBM (option resident_bytes) and cannot be handed over: set it to 0 and sleep again");
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

// ---- the same hand-over for an image PARKED in peer HBM (fma_peer_attach'ed buffer of a node-level owner) ----------------
// The buffer itself is the owner's; what has to travel is the descriptor: the owner keeps it next to the fd.

int fma_image_describe(fma_engine_t* e, int tier, void* buf, size_t cap) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    std::lock_guard<std::mutex> op(e->op_mu);
    if (resident_asleep(e)) return fail(FMA_ESTATE, "part of the sleeping image is resident in this process's own HBM (option resident_bytes) and cannot be handed over: set it to 0 and sleep again");
    if (tier != e->image_tier) return fail(FMA_ESTATE, "no image sleeps in tier %d", tier);
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


}  // extern "C"
