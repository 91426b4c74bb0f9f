"""The node agent's host-memory budget for live sleepers (FMA_NODE_SLEEPER_DRAM_GIB; parking.py SleeperDramBudget): least recently
slept host-tier sleepers are demoted to disk behind the call (Engine.move_image(file, behind=True)) while the ranks' pinned host bytes
exceed the budget, and file-tier sleepers are promoted back, most recently slept first, when a whole image fits again.

The policy tests drive the books with sleeper_state reports and record the commands: fully deterministic.  The cross-process test
runs child processes through the allocator shim over the agent's real socket, on the host-simulated engine (CPU) and on the H100
(-m gpu): three sleepers under a budget of two images; the least recently slept is demoted, a wake mid-write is a host-tier wake,
a wake after the commit reads the file, and both are bit-exact against the oracle."""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GiB = 1 << 30
W = 10 * GiB


def _budget(budget=2 * W + GiB):
    from fma_b200.parking import SleeperDramBudget

    sent = []
    return SleeperDramBudget(budget, lambda key, op: sent.append((key[0], op))), sent


def _state(inst, slept_at, tier="host", asleep=True, host=W, demoting=False, file_dir="/d", **kw):
    return dict({"op": "sleeper_state", "instance": inst, "rank": 0, "asleep": asleep, "tier": tier, "host_bytes": host, "image_bytes": W,
                 "slept_at": slept_at, "demoting": demoting, "file_dir": file_dir, "shared": False}, **kw)


def test_least_recently_slept_is_demoted_and_its_bytes_count_until_the_commit():
    b, sent = _budget()
    b.report(_state("A", 1))
    b.report(_state("B", 2))
    assert sent == [] and b.used() == 2 * W
    b.report(_state("C", 3))
    assert sent == [("A", "demote")]                             # over budget: the least recently slept
    b.report(_state("C", 3))
    assert sent == [("A", "demote")]                             # asked once: the command is in flight
    b.report(_state("A", 1, demoting=True, answer="demote"))
    assert b.used() == 3 * W and b.sleepers()["A"]["demoting"]   # not freed before the commit
    b.report(_state("A", 1, tier="file", host=0))
    assert b.used() == 2 * W and sent == [("A", "demote")]


def test_awake_shared_refused_and_demoting_sleepers_are_never_demoted():
    b, sent = _budget(budget=W // 2)
    b.report(_state("awake", 1, asleep=False))                   # a write-behind reserve, held while it serves
    b.report(_state("shared", 2, shared=True))                   # a deposited store
    b.report(_state("file", 3, tier="file", host=0))
    b.report(_state("peer", 4, tier="peer", host=0))
    assert sent == []
    b.report(_state("X", 5))
    assert sent == [("X", "demote")]
    b.report(_state("X", 5, answer="demote", error="refused", code=-3))   # refused: not asked again until it sleeps again
    b.report(_state("X", 5))
    assert sent == [("X", "demote")]
    b.report(_state("X", 6))
    assert sent == [("X", "demote"), ("X", "demote")]


def test_one_demotion_per_directory_at_a_time():
    b, sent = _budget(budget=0)
    b.report(_state("A", 1, file_dir="/d1"))
    b.report(_state("B", 2, file_dir="/d1"))
    b.report(_state("C", 3, file_dir="/d2"))
    assert sent == [("A", "demote"), ("C", "demote")]            # B waits for A's directory
    b.report(_state("A", 1, demoting=True, answer="demote", file_dir="/d1"))
    b.report(_state("C", 3, demoting=True, answer="demote", file_dir="/d2"))
    assert len(sent) == 2
    b.report(_state("A", 1, tier="file", host=0, file_dir="/d1"))                # A committed: /d1 is free
    assert sent[2:] == [("B", "demote")]


def test_a_cancelled_demotion_counts_again_and_the_policy_reruns():
    b, sent = _budget()
    for i, n in enumerate("ABC"):
        b.report(_state(n, i + 1))
    b.report(_state("A", 1, demoting=True, answer="demote"))
    b.report(_state("A", 1, asleep=False, demoting=False))       # a wake cut the demotion short: A is host and awake
    assert b.used() == 3 * W and sent == [("A", "demote"), ("B", "demote")]   # the next least recently slept
    b.report(_state("B", 2, demoting=True, answer="demote"))
    b.report(_state("B", 2, tier="file", host=0))
    b.report(_state("A", 7))                                     # A sleeps again: within budget, nothing moves
    assert sent == [("A", "demote"), ("B", "demote")] and b.used() == 2 * W


def test_promotion_most_recently_slept_first_while_a_whole_image_fits():
    b, sent = _budget(budget=3 * W)
    b.report(_state("X", 0, host=3 * W))
    b.report(_state("A", 1, tier="file", host=0))
    b.report(_state("B", 2, tier="file", host=0))
    assert sent == []                                            # no room
    b.drop(("X", 0))
    assert sent == [("B", "promote")]                            # one at a time, the most recent first
    b.report(_state("B", 2, host=W, answer="promote"))
    assert sent == [("B", "promote"), ("A", "promote")]
    b.report(_state("A", 1, host=W, answer="promote"))
    b.report(_state("D", 4, host=W))
    b.report(_state("C", 3, tier="file", host=0))
    assert sent[2:] == []                                        # 3 W used: C's image does not fit


def test_explicit_promotion_answers_409_when_the_image_does_not_fit_and_exit_frees_room():
    b, sent = _budget(budget=2 * W)
    b.report(_state("A", 1))
    b.report(_state("B", 2))
    b.report(_state("C", 3, tier="file", host=0))
    assert b.promote("C") is False and sent == []
    assert b.promote("nobody") is None
    b.drop(("A", 0))                                             # A's process exited: its bytes leave the books ...
    assert b.used() == W and sent == [("C", "promote")]          # ... and the room promotes C
    assert "A" not in b.sleepers()
    b.report(_state("C", 3, host=W, answer="promote"))
    b.drop(("B", 0))
    b.report(_state("D", 4, tier="file", host=0))
    assert sent[-1] == ("D", "promote") and b.promote("D") == [0]   # promoted by the policy already: not asked twice
    assert sent.count(("D", "promote")) == 1


def test_a_failed_promotion_is_not_retried_until_the_rank_sleeps_again():
    b, sent = _budget(budget=3 * W)
    b.report(_state("A", 1, tier="file", host=0))
    assert sent == [("A", "promote")]
    for _ in range(5):                                           # it keeps failing (no memory to pin, the file unreadable)
        b.report(_state("A", 1, tier="file", host=0, answer="promote", error="cannot pin", code=-4))
        b.report(_state("A", 1, tier="file", host=0))
    assert sent == [("A", "promote")]
    b.report(_state("B", 2, host=W))                             # other reports re-run the policy: still not asked
    assert sent == [("A", "promote")]
    b.report(_state("A", 3, tier="file", host=0))                # slept again: it may be promoted again
    assert sent == [("A", "promote"), ("A", "promote")]


def test_a_demotion_whose_write_failed_is_not_retried_until_the_rank_sleeps_again():
    b, sent = _budget()
    for i, n in enumerate("ABC"):
        b.report(_state(n, i + 1))
    assert sent == [("A", "demote")]
    b.report(_state("A", 1, demoting=True, answer="demote"))
    b.report(_state("A", 1, failed="demote"))                    # the write failed (EIO, EFBIG, a quota): the image stays host
    assert sent == [("A", "demote"), ("B", "demote")]            # the next one goes instead; A is not rewritten to the same failure
    b.report(_state("B", 2, demoting=True, answer="demote"))
    b.report(_state("B", 2, failed="demote"))
    assert sent[2:] == [("C", "demote")]
    b.report(_state("C", 3, demoting=True, answer="demote"))
    b.report(_state("C", 3, failed="demote"))
    for n, t in (("A", 1), ("B", 2), ("C", 3)):
        b.report(_state(n, t))
    assert len(sent) == 3                                        # every one failed since its sleep: nothing is retried
    b.report(_state("A", 4))                                     # A slept again
    assert sent[3:] == [("A", "demote")]


def test_a_write_behind_sleep_counts_as_writing_until_its_commit_is_reported():
    b, sent = _budget(budget=3 * W)
    b.report(_state("X", 1, tier="file", host=0))
    assert sent == [("X", "promote")]
    b.report(_state("X", 1, tier="file", host=0, answer="promote", error="e", code=-4))
    b.report(_state("A", 2, host=W, demoting=True))              # a write-behind file-tier sleep, still writing
    b.report(_state("Y", 3, tier="file", host=0))
    assert sent == [("X", "promote")]                            # no promotion while it writes
    b.report(_state("A", 2, tier="file", host=0))                # its commit, reported by the rank's waiter
    assert sent == [("X", "promote"), ("Y", "promote")] and b.used() == 0


def test_the_sleeper_routes(built, tmp_path):
    """GET /v2/node/sleepers carries the budget only when it is set; POST .../promote answers 404, 409, nothing to do, or the ranks
    it asked."""
    import socket

    from fastapi.testclient import TestClient

    from fma_b200.node_agent import NodeAgent, create_app, sleeper_budget_settings
    from fma_b200.parking import ParkingService

    assert sleeper_budget_settings({}) == {"sleeper_dram_bytes": None}
    assert sleeper_budget_settings({"FMA_NODE_SLEEPER_DRAM_GIB": "1.5"}) == {"sleeper_dram_bytes": 3 << 29}
    sock_dir = tempfile.mkdtemp(prefix="fma-", dir="/tmp")
    plain = ParkingService(os.path.join(sock_dir, "p.sock"), 1, make_buffer=object)
    svc = ParkingService(os.path.join(sock_dir, "b.sock"), 1, make_buffer=object, sleeper_dram_bytes=2 * W)
    ours, theirs = socket.socketpair()
    try:
        assert plain.sleeper_budget is None
        got = TestClient(create_app(NodeAgent(mock_gpus=True, log_dir=str(tmp_path), start_method="spawn", preload=(), parking=plain)))
        assert "sleeper_dram_bytes" not in got.get("/v2/node/sleepers").json()
        assert got.post("/v2/node/sleepers/A/promote").status_code == 404
        c = TestClient(create_app(NodeAgent(mock_gpus=True, log_dir=str(tmp_path), start_method="spawn", preload=(), parking=svc)))
        svc._sleeper_conns[("D", 0)] = (ours, __import__("threading").Lock())   # D's end of its connection
        budget = svc.sleeper_budget
        budget.report(_state("A", 1))
        budget.report(_state("B", 2))
        budget.report(_state("D", 3, tier="file", host=0))
        res = c.get("/v2/node/sleepers").json()
        assert res["sleeper_dram_bytes"] == 2 * W and res["sleeper_dram_budget_bytes"] == 2 * W
        assert c.post("/v2/node/sleepers/nobody/promote").status_code == 404
        assert c.post("/v2/node/sleepers/D/promote").status_code == 409          # A and B fill the budget
        r = c.post("/v2/node/sleepers/A/promote")
        assert r.status_code == 200 and r.json()["promoting"] is False           # in host DRAM already: nothing to do
        budget.drop(("B", 0))                                                      # B exited: the policy promotes D itself
        assert json.loads(theirs.recv(1 << 10).decode()) == {"op": "promote"}
        budget.report(_state("D", 3, tier="file", host=0, answer="promote", error="e", code=-4))
        r = c.post("/v2/node/sleepers/D/promote")                                  # asked explicitly, after a failure: sent once more
        assert r.status_code == 200 and r.json() == {"instance_id": "D", "promoting": True, "ranks": [0]}
        assert json.loads(theirs.recv(1 << 10).decode()) == {"op": "promote"}
    finally:
        ours.close()
        theirs.close()
        shutil.rmtree(sock_dir, ignore_errors=True)


# ---- across processes: the shim's channel over the agent's socket ---------------------------------------------------------
_CHILD = r"""
import json, os, sys, types
sys.path.insert(0, {root!r})
sys.modules.setdefault("torch", types.SimpleNamespace(cuda=types.SimpleNamespace(empty_cache=lambda: None)))
import fma_b200
from fma_b200 import workloads as W, _lib as L
from fma_b200.cumem import CuMemAllocator
from oracle import oracle as O
eng = fma_b200.Engine(0)
eng.set_option("load_chunk_bytes", 1 << 20)
eng.set_option("load_threads", 4)
table = W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2)
ref, first, seed = {{}}, 0, int(sys.argv[1])
for i, s in enumerate(table):
    eng.alloc(s.bytes, s.tag)
    if s.tag == "weights":
        eng.fill(i, seed, first); ref[i] = O.digest(O.fill(s.bytes, seed, first)); first += s.bytes // 8
a = CuMemAllocator(engine=eng)
print(json.dumps({{"ready": True}}), flush=True)
for line in sys.stdin:
    cmd = line.strip()
    if cmd == "sleep":
        a.sleep(("weights",))
    elif cmd == "wake":
        a.wake_up(None)
    elif cmd == "reserve":                                # what the shim does when the weights pool closes
        a._start_reserve()
        a._join_reserve()
    elif cmd == "fsize":                                  # writes past half an image fail with EFBIG (SIGXFSZ ignored)
        import resource, signal
        signal.signal(signal.SIGXFSZ, signal.SIG_IGN)
        resource.setrlimit(resource.RLIMIT_FSIZE, (sum(s.bytes for s in table if s.tag == "weights") // 2, resource.RLIM_INFINITY))
    elif cmd == "exit":
        break
    st = eng.stats()
    dg = eng.digest_all(["weights"]) if not eng.is_sleeping() else {{}}
    tl = eng.timeline()
    print(json.dumps({{"cmd": cmd, "tier": st["tier"], "host_bytes": st["host_store_bytes"], "exact": all(dg[i] == ref[i] for i in ref) if dg else None,
                      "wb_cancel": any(r["kind"] == "wb_cancel" for r in tl), "ops": sorted({{r["op"] for r in tl}}),
                      "copied": st["sleep_bytes_copied"]}}), flush=True)
"""


class _Child:
    def __init__(self, script, name, seed, env):
        self.name = name
        self.p = subprocess.Popen([sys.executable, str(script), str(seed)], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                  text=True, cwd=ROOT, env=dict(env, FMA_INSTANCE_ID=name))
        assert json.loads(self.p.stdout.readline() or "{}").get("ready"), self.p.stderr.read()[-3000:]

    def do(self, cmd):
        self.p.stdin.write(cmd + "\n")
        self.p.stdin.flush()
        line = self.p.stdout.readline()
        assert line, self.p.stderr.read()[-3000:]
        return json.loads(line)

    def close(self):
        if self.p.poll() is None:
            try:
                self.p.stdin.write("exit\n")
                self.p.stdin.flush()
            except OSError:
                pass
            try:
                self.p.wait(timeout=60)
            except subprocess.TimeoutExpired:
                self.p.kill()
                self.p.wait()


def _until(what, cond, timeout=300):
    t0 = time.time()
    while not cond():
        assert time.time() - t0 < timeout, f"the agent's books never showed {what}"
        time.sleep(0.05)


class _Node:
    """A parking service with a sleeper budget of ``images`` tiny-llama images, and child processes driven through the shim."""

    def __init__(self, tmp_path, images, extra_env):
        from fma_b200 import workloads as Wl
        from fma_b200.parking import ParkingService

        self.image = sum(s.bytes for s in Wl.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2) if s.tag == "weights")
        self.sock_dir = tempfile.mkdtemp(prefix="fma-", dir="/tmp")   # (a unix socket path is at most 107 bytes)
        self.svc = ParkingService(os.path.join(self.sock_dir, "agent.sock"), 1, make_buffer=object, sleeper_dram_bytes=int(self.image * images))
        self.svc.start()
        self.budget = self.svc.sleeper_budget
        self.script = tmp_path / "child.py"
        self.script.write_text(_CHILD.format(root=ROOT))
        file_dir = tmp_path / "files"
        file_dir.mkdir()
        self.env = dict(os.environ, FMA_NODE_AGENT_SOCK=self.svc.sock_path, FMA_NODE_SLEEPER_DRAM_GIB=str(self.budget.budget / GiB),
                        FMA_FILE_DIR=str(file_dir), FMA_FILE_BUFFERED="1", FMA_WB_ITEM_DELAY_MS="100")
        for key in ("FMA_TIER", "FMA_DEPOSIT_HOST_IMAGE", "FMA_DEPOSIT_FILE_IMAGE", "FMA_FILE_WRITE_BEHIND", "FMA_RESIDENT_MIB", "FMA_HOST_STORE_SHM",
                    "FMA_REMOTE_PATHS", "LOCAL_RANK", "RANK"):
            self.env.pop(key, None)
        self.env.update(extra_env)
        self.kids = {}

    def start(self, name, seed):
        self.kids[name] = _Child(self.script, name, seed, self.env)
        return self.kids[name]

    def book(self, name):
        """The rank's own last report (the command in flight not merged in)."""
        return self.budget._books.get((name, 0), {})

    def finish(self):
        for n, k in self.kids.items():
            k.close()
            assert k.p.returncode == 0, k.p.stderr.read()[-3000:]
        _until("every sleeper dropped at exit", lambda: not self.budget.sleepers())
        assert self.budget.used() == 0

    def close(self):
        for k in self.kids.values():
            k.close()
        self.svc.close()
        shutil.rmtree(self.sock_dir, ignore_errors=True)
        assert all(k.p.poll() is not None for k in self.kids.values())   # no process left behind


def _committed(n, name):
    b = n.book(name)
    return b.get("tier") == "file" and b.get("host_bytes") == 0 and not b.get("demoting")


def _three_sleepers_under_a_two_image_budget(tmp_path, extra_env):
    n = _Node(tmp_path, 2.5, extra_env)
    try:
        A, B, C = n.start("A", 11), n.start("B", 22), n.start("C", 33)
        for k in (A, B, C):
            r = k.do("sleep")
            # a full host-tier sleep that met no demotion: no write-behind job was cancelled, nothing written behind it
            assert r["tier"] == 0 and r["copied"] >= n.image and not r["wb_cancel"] and r["ops"] == ["sleep"], r
        # three images over a budget of two and a half: A, the least recently slept, is demoted; B and C stay in DRAM
        _until("A demoting", lambda: n.book("A").get("demoting"))
        assert not n.budget.sleepers()["B"]["demoting"] and not n.budget.sleepers()["C"]["demoting"]
        r = A.do("wake")                                         # mid-write: a host-tier wake that pre-empts the demotion
        assert r["exact"] and r["tier"] == 0 and r["wb_cancel"] and r["host_bytes"] >= n.image, r
        # A is awake and still holds its store: the next least recently slept sleeper, B, goes; its commit frees its bytes
        _until("B committed", lambda: _committed(n, "B"))
        assert n.book("C")["tier"] == "host" and n.budget.used() <= n.budget.budget
        assert n.budget.promote("B") is False                    # A's store and C's image leave no room for B's
        # A sleeps before C, then B wakes from its file and sleeps again: three images, and A is the least recently slept
        assert C.do("wake")["exact"]
        assert A.do("sleep")["tier"] == 0 and C.do("sleep")["tier"] == 0
        r = B.do("wake")                                         # after the commit: from the file
        assert r["exact"] and r["tier"] == 3 and r["host_bytes"] == 0, r
        assert B.do("sleep")["tier"] == 0
        _until("A committed", lambda: _committed(n, "A"))
        assert n.book("B")["tier"] == "host" and n.book("C")["tier"] == "host"
        r = A.do("wake")                                         # A from the file after its commit
        assert r["exact"] and r["tier"] == 3 and not r["wb_cancel"], r
        n.finish()
    finally:
        n.close()


def test_write_behind_sleeps_report_their_commit_their_failure_and_the_reserve(hostsim_lib, oracle, tmp_path):
    """FMA_FILE_WRITE_BEHIND=1 under the budget: the commit of a write-behind file-tier sleep reaches the agent (the rank is no longer
    demoting, its bytes are freed), the reserve pinned in the background after a wake is counted, and a write that fails is
    reported once and not retried by the policy."""
    n = _Node(tmp_path, 0.5, {"FMA_B200_LIB": hostsim_lib, "FMA_HOSTSIM": "1", "HOSTSIM_DEVICES": "1", "FMA_TIER": "file",
                              "FMA_FILE_WRITE_BEHIND": "1"})
    try:
        A = n.start("A", 11)
        A.do("reserve")
        r = A.do("sleep")                                        # returns with the file being written behind it
        assert r["tier"] == 0 and r["host_bytes"] >= n.image, r
        _until("the write-behind commit", lambda: _committed(n, "A"))
        assert n.budget.used() == 0
        r = A.do("wake")                                         # from the file; the shim pins the next store in the background
        assert r["exact"] and r["tier"] == 3, r
        _until("the reserve", lambda: not n.book("A").get("asleep") and n.book("A").get("host_bytes", 0) >= n.image)
        assert not n.budget._pending                             # over budget while awake: never demoted
        A.do("fsize")
        r = A.do("sleep")
        _until("the failed write", lambda: "demote" in n.book("A").get("failed_ops", ()) and not n.book("A").get("demoting"))
        b = n.book("A")
        assert b["asleep"] and b["tier"] == "host" and b["host_bytes"] >= n.image
        time.sleep(0.5)
        assert not n.budget._pending and "demote" in n.book("A")["failed_ops"]   # over budget, but not rewritten to the same failure
        n.finish()
    finally:
        n.close()


@pytest.mark.gpu
def test_three_sleepers_under_a_two_image_budget_on_the_gpu(built, tmp_path):
    _three_sleepers_under_a_two_image_budget(tmp_path, {})


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_budget") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS,
                           os.path.join(ROOT, "tests", "cpp", "hostsim", "hostsim_verify_kernels.cpp"), "-o", out, "-lpthread"])
    return out


def test_three_sleepers_under_a_two_image_budget_on_the_host_simulated_engine(hostsim_lib, oracle, tmp_path):
    _three_sleepers_under_a_two_image_budget(tmp_path, {"FMA_B200_LIB": hostsim_lib, "FMA_HOSTSIM": "1", "HOSTSIM_DEVICES": "1"})
