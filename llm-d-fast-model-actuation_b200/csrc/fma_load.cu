// fma_load.cu — file I/O: reader / writer threads over a small ring of pinned host windows, for the cold load (checkpoint file ->
// HBM, SURVEY.md §8f-3) and for the FILE tier's sleep and wake (fma_sleep.cu / fma_wake.cu)
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"

#include <sys/statvfs.h>

namespace fma_impl {

int ensure_io_windows(fma_engine_t* e) {
    const int n_slots = e->load_slots;
    const size_t slot_bytes = e->load_chunk + 8192;  // slack for O_DIRECT alignment on both ends
    if (e->io_windows != n_slots || e->io_window_bytes != slot_bytes) {
        if (e->load_ring) cudaFreeHost(e->load_ring);
        e->load_ring = nullptr;
        e->load_ring_bytes = 0;
        e->io_windows = 0;
        e->io_window_bytes = 0;
        cudaError_t r = cudaHostAlloc(&e->load_ring, slot_bytes * n_slots, cudaHostAllocPortable);
        if (r != cudaSuccess) {
            cudaGetLastError();
            e->load_ring = nullptr;
            return fail(FMA_ENOMEM, "cannot pin the %zu byte I/O windows: %s", slot_bytes * n_slots, cudaGetErrorString(r));
        }
        e->load_ring_bytes = slot_bytes * n_slots;
        e->io_windows = n_slots;
        e->io_window_bytes = slot_bytes;
    }
    while ((int)e->ev_load.size() < n_slots) {
        cudaEvent_t ev;
        RT(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        e->ev_load.push_back(ev);
    }
    return FMA_OK;
}

namespace {

// Opens `path` for the FILE tier (write: created, not truncated), with O_DIRECT when the filesystem accepts it and
// FMA_FILE_BUFFERED is not 1; *direct tells which.  Failure: FMA_EIO.
int open_image_file(const char* path, bool write, int* fd, bool* direct) {
    const int flags = (write ? O_WRONLY | O_CREAT : O_RDONLY) | O_CLOEXEC;
    *direct = env_int("FMA_FILE_BUFFERED", 0) == 0;
    *fd = *direct ? open(path, flags | O_DIRECT, 0644) : -1;
    if (*fd < 0 && *direct && errno != EINVAL) return fail(FMA_EIO, "cannot open %s: %s", path, strerror(errno));
    if (*fd < 0) {   // the filesystem refuses O_DIRECT (EINVAL), or the page cache was asked for
        *direct = false;
        *fd = open(path, flags, 0644);
        if (*fd < 0) return fail(FMA_EIO, "cannot open %s: %s", path, strerror(errno));
    }
    return FMA_OK;
}

// open_image_file for reading an image of `need` bytes: a file that holds fewer is refused with FMA_EIO; *file_bytes: its size
int open_image_source(const char* path, uint64_t need, int* fd, bool* direct, uint64_t* file_bytes) {
    RC(open_image_file(path, false, fd, direct));
    struct stat sb;
    if (fstat(*fd, &sb) != 0) return fail(FMA_EIO, "fstat(%s) failed: %s", path, strerror(errno));
    if ((uint64_t)sb.st_size < need)
        return fail(FMA_EIO, "%s holds %llu bytes, the image needs %llu", path, (unsigned long long)sb.st_size, (unsigned long long)need);
    *file_bytes = (uint64_t)sb.st_size;
    return FMA_OK;
}

// The filesystem of the open file `fd` has room for an image of `bytes` and its descriptor (fstatvfs), and only then the file is
// emptied.  Short of room: FMA_EIO with the file untouched.
int open_file_store(int fd, uint64_t bytes, const char* path) {
    struct statvfs vs;
    struct stat sb;
    if (fstatvfs(fd, &vs) != 0 || fstat(fd, &sb) != 0) return fail(FMA_EIO, "fstatvfs(%s) failed: %s", path, strerror(errno));
    const uint64_t need = bytes + kImageTail, room = (uint64_t)vs.f_bavail * vs.f_frsize + (uint64_t)sb.st_blocks * 512;  // (its own blocks come back)
    if (room < need) return fail(FMA_EIO, "%s: %llu bytes free, the image needs %llu", path, (unsigned long long)room, (unsigned long long)need);
    if (ftruncate(fd, 0) != 0) return fail(FMA_EIO, "ftruncate(%s) failed: %s", path, strerror(errno));
    return FMA_OK;
}

// After the image's last write: fdatasync, then `desc` in the kImageTail bytes behind the image, then fdatasync again
int close_file_store(int fd, uint64_t bytes, const char* path, bool direct, const std::vector<char>& desc) {
    if (fdatasync(fd) != 0) return fail(FMA_EIO, "fdatasync(%s) failed: %s", path, strerror(errno));
    void* buf = nullptr;
    if (desc.size() > kImageTail || posix_memalign(&buf, 4096, kImageTail) != 0) return fail(FMA_ENOMEM, "no memory for the descriptor");
    memset(buf, 0, kImageTail);
    memcpy(buf, desc.data(), desc.size());
    uint64_t done = 0;
    while (done < kImageTail) {
        const ssize_t n = pwrite(fd, static_cast<char*>(buf) + done, kImageTail - done, (off_t)(bytes + done));
        if (n < 0 && errno == EINTR) continue;
        if (n <= 0) break;
        done += (uint64_t)n;
    }
    const int err = errno;
    free(buf);
    if (done < kImageTail) return fail(FMA_EIO, "writing the descriptor of %s failed: %s", path, strerror(err));
    if (fdatasync(fd) != 0) return fail(FMA_EIO, "fdatasync(%s) failed: %s", path, strerror(errno));
    if (!direct) posix_fadvise(fd, 0, 0, POSIX_FADV_DONTNEED);   // clean now: the page cache lets go of the image
    return FMA_OK;
}

}  // namespace

int ImageFile::read(const std::string& path, std::vector<FileIO::Item> items, std::optional<FileIO>* io, char* mem) {
    path_ = path;
    t0_ = now_s();
    uint64_t need = 0, file_bytes = 0;
    for (const FileIO::Item& it : items) {
        need = std::max(need, it.file_off + it.bytes);
        bytes_ += it.bytes;
    }
    RC(open_image_source(path_.c_str(), need, &file_.fd, &direct_, &file_bytes));
    io->emplace(e_, file_.fd, false, direct_, std::move(items), file_bytes, path_.c_str(), mem);
    return FMA_OK;
}

int ImageFile::create(const std::string& path, uint64_t bytes) {
    path_ = path;
    t0_ = now_s();
    bytes_ = bytes;
    RC(open_image_file(path_.c_str(), true, &file_.fd, &direct_));
    return open_file_store(file_.fd, bytes, path_.c_str());
}

void ImageFile::write(std::vector<FileIO::Item> items, std::optional<FileIO>* io, char* mem) {
    io->emplace(e_, file_.fd, true, direct_, std::move(items), 0, path_.c_str(), mem);
}

int ImageFile::finish(FileIO& io) {
    RC(io.finish());
    return row(bytes_);
}

int ImageFile::seal(int tier) {
    std::vector<char> desc;
    RC(image_descriptor_build(e_, tier, &desc));
    RC(close_file_store(file_.fd, bytes_, path_.c_str(), direct_, desc));
    return row(bytes_ + kImageTail);
}

int ImageFile::row(uint64_t bytes) {
    e_->tl_add("file_io", direct_ ? 1 : 0, t0_, now_s(), bytes);
    return FMA_OK;
}

std::vector<FileIO::Item> FileIO::cut(const fma_engine_t* e, const std::vector<Item>& ranges, std::vector<size_t>* ends) {
    const uint64_t piece = max_item(e);
    std::vector<Item> items;
    for (const Item& r : ranges) {
        for (uint64_t o = 0; o < r.bytes; o += piece) items.push_back(Item{r.file_off + o, std::min(piece, r.bytes - o)});
        if (ends) ends->push_back(items.size());
    }
    return items;
}

FileIO::FileIO(fma_engine_t* e, int fd, bool write, bool direct, std::vector<Item> items, uint64_t file_bytes, const char* path, char* mem)
    : e_(e), fd_(fd), write_(write), direct_(direct), items_(std::move(items)), file_bytes_(file_bytes), path_(path), mem_(mem), n_(e->io_windows),
      ready_(items_.size(), 0), posted_(items_.size(), mem ? 1 : 0), done_(items_.size(), 0) {
    if (mem_) {   // nothing is copied into or out of a window: every item is "posted" from the start
        n_posted_items_ = items_.size();
        for (const Item& it : items_)
            if (direct_ && ((it.file_off | it.bytes | (uint64_t)(uintptr_t)mem_) & 4095)) {
                set_error(FMA_EINVAL, "I/O item of %llu bytes at %llu is not aligned for O_DIRECT", (unsigned long long)it.bytes, (unsigned long long)it.file_off);
                return;
            }
    } else {
        if (!n_ || !e->load_ring) {
            set_error(FMA_ESTATE, "the engine's I/O windows are not pinned");
            return;
        }
        for (const Item& it : items_)
            if (it.bytes > max_item(e) || (direct_ && write_ && ((it.file_off | it.bytes) & 4095))) {
                set_error(FMA_EINVAL, "I/O item of %llu bytes at %llu does not fit a window", (unsigned long long)it.bytes, (unsigned long long)it.file_off);
                return;
            }
    }
    const int n_threads = std::max(1, std::min<int>(e->load_threads, (int)std::max<size_t>(items_.size(), 1)));
    for (int t = 0; t < n_threads && !items_.empty(); ++t) th_.emplace_back([this] { worker(); });
}

FileIO::~FileIO() { stop(); }   // (keeps the message of whatever made the caller leave)

void FileIO::set_error(int code, const char* fmt, ...) {
    std::lock_guard<std::mutex> lk(mu_);
    if (error_ == FMA_OK) {
        error_ = code;
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(msg_, sizeof(msg_), fmt, ap);
        va_end(ap);
    }
    cv_.notify_all();
}

void FileIO::worker() {
    if (!mem_) cudaSetDevice(e_->device);
    for (;;) {
        const size_t k = next_.fetch_add(1);
        if (k >= items_.size()) break;
        const Item& it = items_[k];
        char* abuf = mem_ ? mem_ + it.file_off : nullptr;
        if (!mem_) {
            const size_t w = k % n_;
            {   // read: the window's last copy has been enqueued (k - n posted); write: this item's D2H has been enqueued
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return error_ != FMA_OK || (write_ ? posted_[k] : (k < (size_t)n_ || posted_[k - n_])); });
                if (error_ != FMA_OK) break;
            }
            if (write_ || k >= (size_t)n_) {   // ... and has finished
                const cudaError_t r = cudaEventSynchronize(e_->ev_load[w]);
                if (r != cudaSuccess) return set_error(FMA_ECUDA, "cudaEventSynchronize(I/O window) failed: %s", cudaGetErrorString(r));
            }
            abuf = window(k);
        } else {
            std::lock_guard<std::mutex> lk(mu_);
            if (error_ != FMA_OK) break;   // another item failed: the I/O stops
        }
        const double t0 = now_s();
        uint64_t done = 0;
        int err = 0;
        if (write_) {
            while (done < it.bytes) {
                const ssize_t n = pwrite(fd_, abuf + done, it.bytes - done, (off_t)(it.file_off + done));
                if (n < 0 && errno == EINTR) continue;
                if (n <= 0) { err = n < 0 ? errno : ENOSPC; break; }
                done += (uint64_t)n;
            }
        } else {
            const uint64_t a_off = direct_ ? (it.file_off & ~4095ull) : it.file_off;
            const uint64_t delta = it.file_off - a_off, need = delta + it.bytes;
            uint64_t want = direct_ ? round_up(need, 4096) : it.bytes;   // at most the window (a chunk + 8 KiB of slack)
            const uint64_t end = round_up(file_bytes_, 4096);              // O_DIRECT reads stop at the file's last block
            if (direct_) want = a_off >= end ? 0 : std::min(want, end - a_off);
            while (done < need) {
                const ssize_t n = pread(fd_, abuf + done, want - done, (off_t)(a_off + done));
                if (n < 0 && errno == EINTR) continue;
                if (n <= 0) { err = n < 0 ? errno : 0; break; }
                done += (uint64_t)n;
            }
            if (done < need) done = UINT64_MAX;
        }
        io_ns_.fetch_add((uint64_t)((now_s() - t0) * 1e9));
        if (write_ ? done < it.bytes : done == UINT64_MAX)
            return set_error(FMA_EIO, "%s of %llu bytes at offset %llu of %s failed: %s", write_ ? "write" : "read", (unsigned long long)it.bytes,
                             (unsigned long long)it.file_off, path_, err ? strerror(err) : "the file ends early");
        if (!direct_) posix_fadvise(fd_, (off_t)it.file_off, (off_t)it.bytes, POSIX_FADV_DONTNEED);   // (written pages go after fdatasync)
        std::lock_guard<std::mutex> lk(mu_);
        if (write_) {
            done_[k] = 1;
            while (written_ < items_.size() && done_[written_]) ++written_;
        } else {
            ready_[k] = 1;
        }
        cv_.notify_all();
    }
}

char* FileIO::window(size_t k) const {
    char* buf = static_cast<char*>(e_->load_ring) + (k % n_) * e_->io_window_bytes;
    return direct_ ? reinterpret_cast<char*>(round_up(reinterpret_cast<uintptr_t>(buf), 4096)) : buf;
}

int FileIO::copy(size_t k, void* dev, cudaStream_t stream) {
    return post(k, stream, [&](char* win) -> int {
        RT(cudaMemcpyAsync(write_ ? win : dev, write_ ? dev : win, items_[k].bytes, cudaMemcpyDefault, stream));
        return FMA_OK;
    });
}

size_t FileIO::written() {
    std::lock_guard<std::mutex> lk(mu_);
    return written_;
}

int FileIO::stop() {
    if (!stopped_) {
        {   // the caller stopped before its last item (its own error): threads that wait for a copy it will never post leave
            std::lock_guard<std::mutex> lk(mu_);
            if (error_ == FMA_OK && n_posted_items_ < items_.size()) {
                error_ = FMA_ESTATE;
                snprintf(msg_, sizeof(msg_), "file I/O of %s stopped before its last item", path_);
            }
            cv_.notify_all();
        }
        for (auto& t : th_) t.join();
        for (size_t w = 0; w < std::min<size_t>(n_posted_, (size_t)n_); ++w) {   // nothing may still copy into or out of a window
            const cudaError_t r = cudaEventSynchronize(e_->ev_load[w]);
            if (r != cudaSuccess && error_ == FMA_OK) {
                error_ = FMA_ECUDA;
                snprintf(msg_, sizeof(msg_), "cudaEventSynchronize(I/O window) failed: %s", cudaGetErrorString(r));
            }
        }
        stopped_ = true;
    }
    return error_;
}

int FileIO::finish() { return stop() == FMA_OK ? FMA_OK : fail(error_, "%s", msg_); }

}  // namespace fma_impl

using namespace fma_impl;

extern "C" {

int fma_load_file(fma_engine_t* e, const char* path, const fma_load_span_t* spans, uint32_t n_spans, uint32_t flags,
                  fma_load_stats_t* out_stats) {
    if (check_engine(e) != FMA_OK) return FMA_EINVAL;
    if (!path || (!spans && n_spans)) return fail(FMA_EINVAL, "NULL path or spans");
    const double t_entry = now_s();
    DeviceGuard guard(e->device);
    RC(ensure_streams(e));
    const bool direct = (flags & FMA_LOAD_O_DIRECT) != 0;
    FileFd f;
    f.fd = open(path, O_RDONLY | (direct ? O_DIRECT : 0));
    if (f.fd < 0) return fail(FMA_EINVAL, "cannot open %s: %s", path, strerror(errno));
    struct stat sb;
    if (fstat(f.fd, &sb) != 0) return fail(FMA_EINVAL, "fstat(%s) failed: %s", path, strerror(errno));
    // every destination must be device memory this engine has mapped; every source range must be inside the file
    std::vector<FileIO::Item> items;
    std::vector<uint64_t> dst;
    uint64_t total = 0;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (uint32_t i = 0; i < n_spans; ++i) {
            const fma_load_span_t& sp = spans[i];
            if (!sp.bytes) continue;
            if (sp.file_offset + sp.bytes > (uint64_t)sb.st_size) return fail(FMA_EINVAL, "span %u reads past the end of %s", i, path);
            // the range may span several VA-adjacent mapping units (segments of one arena sit back to back)
            bool ok = true;
            for (uint64_t pos = sp.dst, end = sp.dst + sp.bytes; pos < end;) {
                auto it = e->units.upper_bound((CUdeviceptr)pos);
                if (it == e->units.begin()) { ok = false; break; }
                --it;
                const uint64_t u_end = (uint64_t)it->second.va + it->second.bytes;
                if (pos < it->second.va || pos >= u_end) { ok = false; break; }
                pos = u_end;
            }
            if (!ok)
                return fail(FMA_EINVAL, "span %u: destination 0x%llx+%llu is not inside a mapped segment", i, (unsigned long long)sp.dst,
                            (unsigned long long)sp.bytes);
            for (uint64_t o = 0; o < sp.bytes; o += e->load_chunk) {
                items.push_back(FileIO::Item{sp.file_offset + o, std::min<uint64_t>(e->load_chunk, sp.bytes - o)});
                dst.push_back(sp.dst + o);
            }
            total += sp.bytes;
        }
    }
    RC(ensure_io_windows(e));
    // readers pread ahead into the windows; this thread moves each chunk to its destination as soon as it has been read
    FileIO io(e, f.fd, false, direct, items, (uint64_t)sb.st_size, path);
    int rc = FMA_OK;
    for (size_t k = 0; k < items.size(); ++k)
        if ((rc = io.copy(k, reinterpret_cast<void*>((uintptr_t)dst[k]), e->cs[k % e->n_cs])) != FMA_OK) break;
    if (rc == FMA_OK) rc = io.finish();
    for (int i = 0; i < e->n_cs; ++i) RT(cudaStreamSynchronize(e->cs[i]));
    if (rc == FMA_EIO) {   // a failed read of a cold load has always been FMA_EINVAL
        char why[512];
        snprintf(why, sizeof(why), "%s", tl_err);
        rc = fail(FMA_EINVAL, "%s", why);
    }
    if (rc != FMA_OK) return rc;
    e->st.total_copy_ops += items.size();
    if (out_stats) {
        memset(out_stats, 0, sizeof(*out_stats));
        out_stats->seconds = now_s() - t_entry;
        out_stats->read_seconds = io.io_seconds();
        out_stats->bytes = total;
        out_stats->chunks = (uint32_t)items.size();
        out_stats->threads = (uint32_t)io.threads();
    }
    return FMA_OK;
}

}  // extern "C"
