// fma_gate.cu — cross-process VMM gate (see fma_gate.h).  Host code only; no CUDA calls.
#include "fma_gate.h"

#include <atomic>
#include <cerrno>
#include <chrono>
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>

#include <fcntl.h>
#include <pthread.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

namespace fma_impl {

namespace {

constexpr uint32_t kMagic = 0x464d4147u;  // "FMAG"
constexpr uint32_t kVersion = 3;
constexpr int kSlots = 128;

struct Slot {
    std::atomic<int32_t> pid;                    // 0 = free
    std::atomic<int32_t> want[kGateClasses];     // calls of each class this process is waiting to make / has announced
};

struct Shm {
    std::atomic<uint32_t> magic;                 // written last by the creator
    uint32_t version;
    pthread_mutex_t mu;                          // robust, process-shared: held around one VMM call
    Slot slots[kSlots];
};

struct Local {
    std::mutex open_mu;
    std::atomic<int> opened_pid{0};   // the gate was opened by this pid (a forked child must claim a slot of its own); written last, release
    bool atexit_set = false;
    Shm* shm = nullptr;
    int slot = -1;
    std::atomic<bool> enabled{false};
    std::mutex st_mu;
    GateStats st;
};
Local g;

double mono_s() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

bool pid_alive(int32_t pid) {
    if (pid <= 0) return false;
    return kill(pid, 0) == 0 || errno != ESRCH;
}

void open_gate() {
    const char* on = getenv("FMA_VMM_GATE");
    // On unless FMA_VMM_GATE=0 (the A/B switch: bench.py at N > 1 with and without it).
    if (on && *on && atoi(on) == 0) return;
    char name[128];
    const char* forced = getenv("FMA_VMM_GATE_NAME");
    if (forced && *forced) snprintf(name, sizeof(name), "%s%s", forced[0] == '/' ? "" : "/", forced);
    else snprintf(name, sizeof(name), "/fma_b200_gate.%u", (unsigned)getuid());
    bool creator = false;
    int fd = shm_open(name, O_RDWR | O_CREAT | O_EXCL, 0600);
    if (fd >= 0) {
        creator = true;
        if (ftruncate(fd, (off_t)sizeof(Shm)) != 0) {
            close(fd);
            shm_unlink(name);
            return;
        }
    } else {
        fd = shm_open(name, O_RDWR, 0600);
        if (fd < 0) return;
        // the creator may still be sizing it
        for (int i = 0; i < 2000; ++i) {
            struct stat sb;
            if (fstat(fd, &sb) == 0 && (size_t)sb.st_size >= sizeof(Shm)) break;
            std::this_thread::sleep_for(std::chrono::microseconds(100));
        }
    }
    void* p = mmap(nullptr, sizeof(Shm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) return;
    Shm* s = static_cast<Shm*>(p);
    if (creator) {
        pthread_mutexattr_t a;
        pthread_mutexattr_init(&a);
        pthread_mutexattr_setpshared(&a, PTHREAD_PROCESS_SHARED);
        pthread_mutexattr_setrobust(&a, PTHREAD_MUTEX_ROBUST);
        pthread_mutex_init(&s->mu, &a);
        pthread_mutexattr_destroy(&a);
        s->version = kVersion;
        s->magic.store(kMagic, std::memory_order_release);
    } else {
        bool ok = false;
        for (int i = 0; i < 20000 && !ok; ++i) {  // <= 2 s for the creator to finish
            ok = s->magic.load(std::memory_order_acquire) == kMagic;
            if (!ok) std::this_thread::sleep_for(std::chrono::microseconds(100));
        }
        if (!ok || s->version != kVersion) {  // stale segment of another build: do without a gate rather than guess its layout
            munmap(p, sizeof(Shm));
            return;
        }
    }
    const int32_t me = (int32_t)getpid();
    int slot = -1;
    for (int round = 0; round < 2 && slot < 0; ++round) {
        for (int i = 0; i < kSlots && slot < 0; ++i) {
            int32_t cur = s->slots[i].pid.load();
            if (cur == me) {  // our own pid from an earlier life (pid reuse): take it over
                slot = i;
            } else if (cur == 0 || (round == 1 && !pid_alive(cur))) {
                if (s->slots[i].pid.compare_exchange_strong(cur, me)) slot = i;
            }
        }
    }
    if (slot < 0) {
        munmap(p, sizeof(Shm));
        return;
    }
    for (int c = 0; c < kGateClasses; ++c) s->slots[slot].want[c].store(0);
    g.shm = s;
    g.slot = slot;
    g.enabled = true;
    if (!g.atexit_set) {
        g.atexit_set = true;
        atexit([] {
            if (g.shm && g.slot >= 0 && g.opened_pid.load() == (int)getpid()) {
                for (int c = 0; c < kGateClasses; ++c) g.shm->slots[g.slot].want[c].store(0);
                g.shm->slots[g.slot].pid.store(0);
            }
        });
    }
}

// does anybody — another live process, or another thread of this one (two engines in one process: a hot swap) — want a class
// above (numerically below) `cls`?  The caller itself only ever counts in want[cls], so its own slot can be scanned as well.
bool higher_waiting(int cls, bool check_alive) {
    Shm* s = g.shm;
    for (int i = 0; i < kSlots; ++i) {
        const int32_t pid = s->slots[i].pid.load(std::memory_order_relaxed);
        if (!pid) continue;
        for (int c = 0; c < cls; ++c) {
            if (s->slots[i].want[c].load(std::memory_order_relaxed) > 0) {
                if (check_alive && i != g.slot && !pid_alive(pid)) {  // reclaim a dead process's slot
                    for (int k = 0; k < kGateClasses; ++k) s->slots[i].want[k].store(0);
                    int32_t expect = pid;
                    s->slots[i].pid.compare_exchange_strong(expect, 0);
                    break;
                }
                return true;
            }
        }
    }
    return false;
}

bool lock_bounded(double seconds) {
    struct timespec ts;
    clock_gettime(CLOCK_REALTIME, &ts);
    const double t = ts.tv_sec + ts.tv_nsec * 1e-9 + seconds;
    ts.tv_sec = (time_t)t;
    ts.tv_nsec = (long)((t - (double)ts.tv_sec) * 1e9);
    int r = pthread_mutex_timedlock(&g.shm->mu, &ts);
    if (r == EOWNERDEAD) {  // the holder died inside a VMM call: the state it guarded is the driver's, nothing to repair
        pthread_mutex_consistent(&g.shm->mu);
        r = 0;
    }
    return r == 0;
}

}  // namespace

bool gate_enabled() {
    const int me = (int)getpid();
    if (g.opened_pid.load(std::memory_order_acquire) == me) return g.enabled.load(std::memory_order_relaxed);   // fast path
    std::lock_guard<std::mutex> lk(g.open_mu);
    if (g.opened_pid.load(std::memory_order_relaxed) != me) {   // first use in this process — also in a child forked after the parent's first use
        g.enabled.store(false);
        g.shm = nullptr;
        g.slot = -1;
        open_gate();
        g.opened_pid.store(me, std::memory_order_release);
    }
    return g.enabled.load();
}

int gate_announce(int cls) {
    if (!gate_enabled() || cls < 0 || cls >= kGateClasses) return 0;
    g.shm->slots[g.slot].want[cls].fetch_add(1);
    return cls + 1;
}

void gate_retract(int handle) {
    if (handle <= 0 || !g.enabled) return;
    g.shm->slots[g.slot].want[handle - 1].fetch_sub(1);
}

int gate_acquire(int cls, double max_wait_s) {
    if (!gate_enabled() || cls < 0 || cls >= kGateClasses) return 0;
    const double t0 = mono_s();
    Slot& me = g.shm->slots[g.slot];
    me.want[cls].fetch_add(1);
    bool yielded = false, timed_out = false, locked = false;
    int spins = 0;
    for (;;) {
        const double waited = mono_s() - t0;
        if (cls > 0 && waited < max_wait_s && higher_waiting(cls, (++spins % 64) == 0)) {
            yielded = true;
            std::this_thread::sleep_for(std::chrono::microseconds(100));
            continue;
        }
        if (cls > 0 && waited >= max_wait_s && higher_waiting(cls, false)) timed_out = true;
        if (!lock_bounded(2.0)) {
            timed_out = true;
            break;
        }
        // a higher class may have arrived while we waited for the lock: let it pass (bounded)
        if (cls > 0 && (mono_s() - t0) < max_wait_s && higher_waiting(cls, false)) {
            pthread_mutex_unlock(&g.shm->mu);
            yielded = true;
            std::this_thread::sleep_for(std::chrono::microseconds(100));
            continue;
        }
        locked = true;
        break;
    }
    me.want[cls].fetch_sub(1);
    {
        std::lock_guard<std::mutex> lk(g.st_mu);
        ++g.st.acquires;
        if (yielded) ++g.st.yielded;
        if (timed_out) ++g.st.timeouts;
        g.st.wait_s += mono_s() - t0;
    }
    return locked ? 1 : 0;
}

void gate_release(int token) {
    if (token == 1 && g.enabled) pthread_mutex_unlock(&g.shm->mu);
}

GateStats gate_stats() {
    std::lock_guard<std::mutex> lk(g.st_mu);
    return g.st;
}

}  // namespace fma_impl
