// fma_gate.h — cross-process VMM gate (internal; host only).
//
// cuMemCreate / cuMemMap / cuMemSetAccess / cuMemUnmap of ALL processes on one host serialise inside the driver
// (scripts/vmm_span_probe.py), in arrival order.  When N ranks wake at once that order is wrong: the call that gates
// a rank's first H2D (its 1 GiB staging ring, then the first piece of its weights run) can queue behind another rank's
// 32 GiB kv_cache remap, which nothing waits for.  The reference has the same property, only worse (three calls per
// segment, cumem.py:240 -> create_and_map).  The gate is a priority lock in POSIX shared memory that every engine on the
// host takes around its VMM calls: the driver serialises them anyway, so holding our own lock costs nothing and decides
// the ORDER — class 0 (gates a first copy) before the weights pieces in round robin across ranks (class = piece index) before
// remap-only runs (the whole copy time of slack) before sleep-side unmaps — and un-contended calls are faster than calls of
// several ranks that collide in the driver (bench.py --timeline shows the per-call times).
//
// Failure model: everything is bounded.  A waiter gives up waiting for higher classes after `max_wait_s` and a lock that
// cannot be had within 2 s is skipped (the driver's own lock still serialises), so a dead or wedged peer can delay a
// call, never hang it.  The mutex is robust (a holder that died is recovered by the next locker).  Per-process slots
// carry the pid; slots of dead pids are reclaimed.  On by default; FMA_VMM_GATE=0 disables it; FMA_VMM_GATE_NAME picks the segment
// (default "/fma_b200_gate.<uid>": the engines of one pod / one launcher share /dev/shm and therefore one gate).
#pragma once
#include <cstddef>
#include <cstdint>

namespace fma_impl {

constexpr int kGateFirst = 0;      // gates a first copy: the staging ring (or the first piece when there is no ring)
constexpr int kGateWeights = 1;    // 1 .. kGateWeightsLast: the k-th piece of the backed-up runs — every rank's piece k goes before anybody's
constexpr int kGateWeightsLast = 13;   // piece k+1 (round robin across ranks: a rank needs piece k only after (k-1) x 39 ms of H2D)
constexpr int kGateRemap = 14;     // remap-only runs (kv_cache): the whole copy time of slack
constexpr int kGateUnmap = 15;     // unmaps of a sleep: nothing waits for them
constexpr int kGateClasses = 16;

struct GateStats {
    uint64_t acquires = 0;
    uint64_t yielded = 0;      // acquires that waited for a higher class at least once
    double wait_s = 0;         // total time between asking and holding
    uint64_t timeouts = 0;     // gave up waiting (bounded) or could not take the lock
};

// Take the gate for one VMM call of class `cls`; waits at most max_wait_s for higher classes of other processes to finish.
// Returns a token for gate_release (0 = gate disabled / unavailable: nothing to release).
int gate_acquire(int cls, double max_wait_s);
void gate_release(int token);
// A process announces "I am about to issue class-`cls` calls" (e.g. at wake entry, before planning), so that lower classes of
// other processes already yield while it is still on its way to the first call.  Returns a handle for gate_retract.
int gate_announce(int cls);
void gate_retract(int handle);
GateStats gate_stats();
bool gate_enabled();

struct GateHold {  // RAII
    int token;
    GateHold(int cls, double max_wait_s) : token(gate_acquire(cls, max_wait_s)) {}
    ~GateHold() { gate_release(token); }
    GateHold(const GateHold&) = delete;
    GateHold& operator=(const GateHold&) = delete;
};

}  // namespace fma_impl
