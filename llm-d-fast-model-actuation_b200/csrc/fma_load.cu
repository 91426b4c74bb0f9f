// fma_load.cu — cold load: checkpoint file -> HBM through a pinned bounce ring and the copy engines (SURVEY.md §8f-3)
// Part of the host engine (see fma_internal.h for the map of translation units; C-ABI in include/fma_engine.h).
#include "fma_internal.h"

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
    int fd = open(path, O_RDONLY | (direct ? O_DIRECT : 0));
    if (fd < 0) return fail(FMA_EINVAL, "cannot open %s: %s", path, strerror(errno));
    struct stat sb;
    if (fstat(fd, &sb) != 0) {
        close(fd);
        return fail(FMA_EINVAL, "fstat(%s) failed: %s", path, strerror(errno));
    }
    // every destination must be device memory this engine has mapped; every source range must be inside the file
    struct Item { uint64_t file_off, bytes, dst; };
    std::vector<Item> items;
    uint64_t total = 0;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (uint32_t i = 0; i < n_spans; ++i) {
            const fma_load_span_t& sp = spans[i];
            if (!sp.bytes) continue;
            if (sp.file_offset + sp.bytes > (uint64_t)sb.st_size) {
                close(fd);
                return fail(FMA_EINVAL, "span %u reads past the end of %s", i, path);
            }
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
            if (!ok) {
                close(fd);
                return fail(FMA_EINVAL, "span %u: destination 0x%llx+%llu is not inside a mapped segment", i,
                            (unsigned long long)sp.dst, (unsigned long long)sp.bytes);
            }
            for (uint64_t o = 0; o < sp.bytes; o += e->load_chunk)
                items.push_back(Item{sp.file_offset + o, std::min<uint64_t>(e->load_chunk, sp.bytes - o), sp.dst + o});
            total += sp.bytes;
        }
    }
    const int n_slots = e->load_slots;
    const size_t slot_bytes = e->load_chunk + 8192;  // slack for O_DIRECT alignment on both ends
    if (e->load_ring_bytes < slot_bytes * n_slots) {
        if (e->load_ring) cudaFreeHost(e->load_ring);
        e->load_ring = nullptr;
        e->load_ring_bytes = 0;
        cudaError_t r = cudaHostAlloc(&e->load_ring, slot_bytes * n_slots, cudaHostAllocPortable);
        if (r != cudaSuccess) {
            cudaGetLastError();
            close(fd);
            return fail(FMA_ENOMEM, "cannot pin the %zu byte load ring: %s", slot_bytes * n_slots, cudaGetErrorString(r));
        }
        e->load_ring_bytes = slot_bytes * n_slots;
    }
    while ((int)e->ev_load.size() < n_slots) {
        cudaEvent_t ev;
        cudaError_t r = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        if (r != cudaSuccess) {
            close(fd);
            return fail(FMA_ECUDA, "cudaEventCreate failed: %s", cudaGetErrorString(r));
        }
        e->ev_load.push_back(ev);
    }
    // Slot s is used by items s, s+n, s+2n, ... strictly in that order (threads run ahead of each other):
    // slot_gen[s] counts the uses whose H2D has been ENQUEUED; the event tells when that H2D has finished.
    std::mutex mu;
    std::condition_variable cv;
    std::vector<uint64_t> slot_gen(n_slots, 0);
    std::atomic<size_t> next{0};
    std::atomic<uint64_t> read_ns{0};
    int error = FMA_OK;
    char msg[512] = "";
    const int n_threads = std::max(1, std::min<int>(e->load_threads, (int)std::max<size_t>(items.size(), 1)));
    auto worker = [&]() {
        cudaSetDevice(e->device);
        for (;;) {
            const size_t k = next.fetch_add(1);
            if (k >= items.size()) break;
            const int s = (int)(k % n_slots);
            const uint64_t my_gen = k / n_slots;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return slot_gen[s] == my_gen || error != FMA_OK; });
                if (error != FMA_OK) break;
            }
            char* buf = static_cast<char*>(e->load_ring) + (size_t)s * slot_bytes;
            if (my_gen > 0) {
                cudaError_t r = cudaEventSynchronize(e->ev_load[s]);  // the previous chunk in this slot has left
                if (r != cudaSuccess) {
                    std::lock_guard<std::mutex> lk(mu);
                    if (error == FMA_OK) { error = FMA_ECUDA; snprintf(msg, sizeof(msg), "cudaEventSynchronize: %s", cudaGetErrorString(r)); }
                    cv.notify_all();
                    break;
                }
            }
            const Item& it = items[k];
            const uint64_t a_off = direct ? (it.file_off & ~4095ull) : it.file_off;
            const uint64_t delta = it.file_off - a_off;
            uint64_t want = direct ? round_up(delta + it.bytes, 4096) : it.bytes;
            if (direct && a_off + want > (uint64_t)round_up((size_t)sb.st_size, 4096)) want = round_up((size_t)sb.st_size, 4096) - a_off;
            char* rbuf = direct ? reinterpret_cast<char*>(round_up(reinterpret_cast<uintptr_t>(buf), 4096)) : buf;
            const double t0 = now_s();
            uint64_t got = 0;
            bool io_err = false;
            while (got < (direct ? delta + it.bytes : it.bytes)) {
                ssize_t n = pread(fd, rbuf + got, want - got, (off_t)(a_off + got));
                if (n < 0 && errno == EINTR) continue;
                if (n <= 0) { io_err = (got < delta + it.bytes); break; }
                got += (uint64_t)n;
            }
            read_ns.fetch_add((uint64_t)((now_s() - t0) * 1e9));
            cudaError_t r = cudaSuccess;
            if (!io_err) {
                cudaStream_t st = e->cs[k % e->n_cs];
                r = cudaMemcpyAsync(reinterpret_cast<void*>((uintptr_t)it.dst), rbuf + delta, it.bytes, cudaMemcpyHostToDevice, st);
                if (r == cudaSuccess) r = cudaEventRecord(e->ev_load[s], st);
            }
            std::lock_guard<std::mutex> lk(mu);
            if (io_err || r != cudaSuccess) {
                if (error == FMA_OK) {
                    error = io_err ? FMA_EINVAL : FMA_ECUDA;
                    snprintf(msg, sizeof(msg), io_err ? "short read at offset %llu of %s: %s" : "H2D of chunk at %llu failed (%s): %s",
                             (unsigned long long)it.file_off, path, io_err ? strerror(errno) : cudaGetErrorString(r));
                }
            } else {
                slot_gen[s] = my_gen + 1;
            }
            cv.notify_all();
            if (error != FMA_OK) break;
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; ++t) th.emplace_back(worker);
    for (auto& t : th) t.join();
    close(fd);
    for (int i = 0; i < e->n_cs; ++i) {
        cudaError_t r = cudaStreamSynchronize(e->cs[i]);
        if (r != cudaSuccess && error == FMA_OK) {
            error = FMA_ECUDA;
            snprintf(msg, sizeof(msg), "cudaStreamSynchronize failed: %s", cudaGetErrorString(r));
        }
    }
    if (error != FMA_OK) return fail(error, "%s", msg);
    e->st.total_copy_ops += items.size();
    if (out_stats) {
        memset(out_stats, 0, sizeof(*out_stats));
        out_stats->seconds = now_s() - t_entry;
        out_stats->read_seconds = read_ns.load() * 1e-9;
        out_stats->bytes = total;
        out_stats->chunks = (uint32_t)items.size();
        out_stats->threads = (uint32_t)n_threads;
    }
    return FMA_OK;
}


}  // extern "C"
