"""Warm start from a kept image file: an instance that sleeps to the file tier deposits its image file with the node agent's
parking service (FMA_DEPOSIT_FILE_IMAGE=1) and exits asleep; the service keeps the file; the next instance with the same ID adopts
it when its weights pool closes (FMA_ADOPT_FILE=1) and wakes with its digests verified.

The -m gpu tests run that sequence with real processes on the engine: plain and PACKED, O_DIRECT and buffered, and once through a
host memfd that the service spilled to disk.  test_warm_start_against_the_host_simulated_engine reruns them on CPU against the
host-simulated engine (tests/cpp/hostsim).  The other tests need no GPU: fma_image_file_info against the engine's own statistics,
and the service's books (exit hook, leases, disk budget, DRAM spill, re-listing, GET /v2/node/images)."""
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import pytest

from tests.test_file_tier import _o_direct_refused

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAIL = 2 << 20
GiB = 1 << 30
gpu = pytest.mark.gpu

MODELS = {"m1": [("weights", 6), ("weights", 2), ("kv_cache", 8), ("weights", 4), ("weights", 10)],
          "m2": [("weights", 4), ("weights", 4), ("kv_cache", 8), ("weights", 4)]}

# One instance.  argv: phase, model, seed, pack.  Phases:
#   sleep  - load the model, sleep to the file tier through the allocator shim (which deposits the file) and exit asleep
#   host   - load the model, sleep to the host tier through the allocator shim (FMA_DEPOSIT_HOST_IMAGE=1 deposits the memfd),
#            exit asleep
#   cycle  - load the model, sleep to the file tier through the shim (deposited), wake (withdrawn), exit
#   adopt  - load junk (as --load-format dummy would), then what the shim does when the weights pool closes; print the outcome,
#            then sleep to the file tier once more (its own path) and wake
#   info   - load the model, sleep to the host tier with digests and image_save it to argv[5]; print stats and the descriptor
_INSTANCE = r"""
import json, os, sys, types
sys.path.insert(0, {root!r})
sys.modules.setdefault("torch", types.SimpleNamespace(cuda=types.SimpleNamespace(empty_cache=lambda: None)))
import fma_b200
from fma_b200 import _lib as L
from fma_b200.cumem import CuMemAllocator
from fma_b200.parking import ParkingClient
from oracle import oracle as O
phase, model, seed, pack = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
table = {models!r}[model]
eng = fma_b200.Engine(0)
eng.set_option("pack", pack)
eng.set_option("chunk_bytes", 4 << 20)
eng.set_option("load_chunk_bytes", 1 << 20)
ref = {{}}
for j, (tag, mib) in enumerate(table):
    if tag == "weights" or phase != "adopt":             # (an instance allocates its kv cache after the weights pool closed)
        i = eng.find(eng.alloc(mib << 20, tag))
        if tag == "weights":
            ref[i] = O.bf16_weights((mib << 20) // 2, seed + j)
            eng.write(i, (ref[i] if phase != "adopt" else O.bf16_weights((mib << 20) // 2, 999 + j)).tobytes())
a = CuMemAllocator(engine=eng)
if phase == "sleep":
    a.sleep(("weights",))
    assert eng.is_sleeping() and eng.stats()["tier"] == L.FMA_TIER_FILE
    print("slept", json.dumps(eng.stats()["image_packed"]), flush=True)
    sys.exit(0)                                           # normal exit: atexit hooks run
if phase == "host":
    a.sleep(("weights",))
    assert eng.is_sleeping() and eng.stats()["tier"] == L.FMA_TIER_HOST
    print("slept", flush=True)
    sys.exit(0)
if phase == "cycle":
    a.sleep(("weights",))
    a.wake_up(None)
    assert all(eng.read(i, ref[i].nbytes) == ref[i].tobytes() for i in ref)
    print("cycled", flush=True)
    sys.exit(0)
if phase == "info":
    eng.sleep(["weights"], flags=L.FMA_FLAG_VERIFY)
    eng.image_save(sys.argv[5])
    st = eng.stats()
    print(json.dumps({{"image_store_bytes": st["image_store_bytes"], "sleep_bytes_offloaded": st["sleep_bytes_offloaded"],
                      "image_packed": st["image_packed"], "segments": sum(1 for t, _ in table if t == "weights")}}), flush=True)
    sys.exit(0)
try:
    adopted = a._adopt_kept_file()
except L.FmaError as e:
    print(json.dumps({{"error": e.code}}), flush=True)
    sys.exit(0)
same = all(eng.read(i, ref[i].nbytes) == ref[i].tobytes() for i in ref)
out = {{"adopted": adopted, "oracle": same, "tier": eng.stats()["tier"], "sleeping": eng.is_sleeping()}}
for tag, mib in table:
    if tag != "weights":
        eng.alloc(mib << 20, tag)
a.sleep(("weights",))                                     # a later file-tier sleep writes this rank's own file
out["own_file"] = a._file_path
a.wake_up(None)
junk = {{i: O.bf16_weights(ref[i].size, 999 + j) for i, j in zip(sorted(ref), [j for j, (t, _) in enumerate(table) if t == "weights"])}}
out["after"] = all(eng.read(i, ref[i].nbytes) == (ref[i] if adopted else junk[i]).tobytes() for i in ref)
print(json.dumps(out), flush=True)
"""


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


class _Node:
    """A parking service with kept files, and instances of it as real processes."""

    def __init__(self, tmp_path, **budgets):
        from fma_b200.parking import ParkingService

        self.sock_dir = tempfile.mkdtemp(prefix="fma-", dir="/tmp")
        self.file_dir = tmp_path / "images"
        self.file_dir.mkdir(exist_ok=True)
        self.keep_dir = str(self.file_dir / "kept")
        self.svc = ParkingService(os.path.join(self.sock_dir, "a.sock"), n_devices=1, keep_dir=self.keep_dir, **budgets)
        self.svc.start()
        self.script = tmp_path / "instance.py"
        self.script.write_text(_INSTANCE.format(root=ROOT, models=MODELS))
        self.env = dict(os.environ, FMA_NODE_AGENT_SOCK=self.svc.sock_path, FMA_TIER="file", FMA_FILE_DIR=str(self.file_dir),
                        FMA_DEPOSIT_FILE_IMAGE="1", FMA_ADOPT_FILE="1", RANK="0")
        for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_HOST_STORE_SHM", "FMA_REMOTE_PATHS", "LOCAL_RANK", "FMA_ADOPT_PARKED"):
            self.env.pop(key, None)

    def run(self, iid, phase, model="m1", seed=1, pack=0, *extra, env=None):
        r = subprocess.run([sys.executable, str(self.script), phase, model, str(seed), str(pack), *extra], cwd=ROOT,
                           env=dict(self.env, FMA_INSTANCE_ID=iid, **(env or {})), capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        self.svc.instance_exited(iid)                     # what the node agent's child-exit path does
        return r

    def close(self):
        self.svc.close()
        shutil.rmtree(self.sock_dir, ignore_errors=True)


def _last_json(r):
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.fixture()
def node(built, tmp_path):
    n = _Node(tmp_path)
    yield n
    n.close()


@gpu
@pytest.mark.parametrize("io", ["buffered", "direct"])
@pytest.mark.parametrize("pack", [0, 1])
def test_a_deleted_sleepers_next_instance_warm_starts_from_its_kept_file(node, tmp_path, pack, io):
    env = {"FMA_FILE_BUFFERED": "1"} if io == "buffered" else {}
    if io == "direct":
        node.env.pop("FMA_FILE_BUFFERED", None)
        if _o_direct_refused(node.file_dir):
            pytest.skip(_o_direct_refused(node.file_dir))
    node.run("Ia", "sleep", "m1", 1, pack, env=env)
    assert os.listdir(node.file_dir) == ["kept"]          # the instance's own file went into the keep directory
    kept = node.svc.kept()["images"]
    assert [(k["instance_id"], k["where"], k["packed"], k["leased"]) for k in kept] == [("Ia", "disk", bool(pack), False)]
    path = node.svc._kept[("Ia", 0)]["path"]
    before = _sha(path)
    got = _last_json(node.run("Ia", "adopt", "m1", 1, pack, env=env))
    assert got["adopted"] and got["oracle"] and not got["sleeping"] and got["after"], got
    assert got["own_file"] != path and _sha(path) == before   # the adopter never writes the kept file
    assert node.svc.kept()["images"][0]["leased"] is False
    # another model under the same ID: refused before the wake, the loaded weights stay
    got = _last_json(node.run("Ia", "adopt", "m2", 1, pack, env=env))
    assert got["adopted"] is False and got["after"], got
    # one damaged byte: the wake fails its digests, the instance raises and the entry is gone
    with open(path, "r+b") as f:
        f.seek(3 << 20)
        b = f.read(1)
        f.seek(3 << 20)
        f.write(bytes([b[0] ^ 0x40]))
    r = node.run("Ia", "adopt", "m1", 1, pack, env=env)
    assert _last_json(r) == {"error": -7}, r.stdout
    assert node.svc.kept()["images"] == [] and not os.path.exists(path)


@gpu
def test_a_spilled_host_deposit_warm_starts_from_disk(built, tmp_path):
    """The shim's own host deposit (FMA_DEPOSIT_HOST_IMAGE=1) carries digests, so the spill keeps it on disk."""
    n = _Node(tmp_path, keep_dram_bytes=0)                 # every host deposit goes to disk
    try:
        n.run("Ih", "host", "m1", 5, 1, env={"FMA_HOST_STORE_SHM": "1", "FMA_TIER": "host", "FMA_DEPOSIT_HOST_IMAGE": "1", "FMA_PREPIN": "0"})
        n.svc.wait_spills()
        assert n.svc.lookup_host("Ih", 0) is None
        assert [(k["where"], k["packed"]) for k in n.svc.kept()["images"]] == [("disk", True)]
        got = _last_json(n.run("Ih", "adopt", "m1", 5, 1))
        assert got["adopted"] and got["oracle"] and got["after"], got
    finally:
        n.close()


@gpu
def test_a_file_whose_deposit_was_withdrawn_or_refused_is_removed_at_exit(built, tmp_path):
    n = _Node(tmp_path)
    try:
        n.run("Ic", "cycle")                                # deposited, then withdrawn by the wake: the shim and the agent remove it
        assert os.listdir(n.file_dir) == ["kept"] and n.svc.kept()["images"] == []
    finally:
        n.close()
    n = _Node(tmp_path)
    n.svc.keep_dir = None                                  # an agent that keeps no files refuses the deposit
    try:
        n.run("Ir", "sleep")
        assert os.listdir(n.file_dir) == ["kept"]          # nobody took the file: the shim removed it at exit
    finally:
        n.close()


def test_warm_start_against_the_host_simulated_engine(hostsim_lib, oracle):
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="1")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, tail
    skips = [l for l in r.stdout.splitlines() if l.startswith("SKIPPED")]
    assert all("refuses O_DIRECT" in l for l in skips), skips


@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_warm") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS, "-o", out, "-lpthread"])
    return out


@pytest.fixture(scope="module")
def images(hostsim_lib, tmp_path_factory):
    """Image files written by the host-simulated engine: plain and PACKED with digests (image_save), and a file-tier image
    without digests; with what the engine reported about each."""
    d = tmp_path_factory.mktemp("images")
    script = d / "instance.py"
    script.write_text(_INSTANCE.format(root=ROOT, models=MODELS))
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="1", FMA_HOST_STORE_SHM="1", FMA_FILE_BUFFERED="1",
               FMA_TIER="file", FMA_FILE_DIR=str(d), FMA_INSTANCE_ID="Inodigests", RANK="0")
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_NODE_AGENT_SOCK", "FMA_DEPOSIT_FILE_IMAGE", "LOCAL_RANK"):
        env.pop(key, None)
    out = {}
    for pack in (0, 1):
        p = str(d / f"saved{pack}.fmaimg")
        r = subprocess.run([sys.executable, str(script), "info", "m1", "3", str(pack), p], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        out[pack] = (p, _last_json(r))
    nod = str(d / "nodigests.fmaimg")   # a file-tier sleep without FMA_FLAG_VERIFY (the shim's default) records no digests
    child = ("import sys, types; sys.path.insert(0, %r); sys.modules['torch'] = types.SimpleNamespace(cuda=types.SimpleNamespace(empty_cache=lambda: None))\n"
             "import fma_b200; from fma_b200 import _lib as L\n"
             "e = fma_b200.Engine(0); [e.alloc(m << 20, 'weights') for m in (2, 4)]; e.file_store(%r); e.sleep(['weights'], tier=L.FMA_TIER_FILE)\n"
             "import os; os._exit(0)\n") % (ROOT, nod)
    subprocess.check_call([sys.executable, "-c", child], env=env, cwd=ROOT)
    out["nodigests"] = nod
    return out


def test_image_file_info_reads_a_file_without_an_engine_or_a_driver(built, images, tmp_path):
    """The product library on this host has no driver, yet fma_image_file_info describes files the engine wrote, with the fields
    the engine reported for them; broken files are refused."""
    import fma_b200
    from fma_b200 import _lib as L

    for pack in (0, 1):
        path, st = images[pack]
        info = fma_b200.Engine.image_file_info(path)
        assert info == {"image_bytes": st["image_store_bytes"], "weight_bytes": st["sleep_bytes_offloaded"], "n_segments": st["segments"],
                        "version": 2 if pack else 1, "packed": bool(pack), "digests": True, "tags": ["weights"]}, (info, st)
    assert fma_b200.Engine.image_file_info(images["nodigests"])["digests"] is False
    data = open(images[0][0], "rb").read()
    cases = {"truncated": data[:-1], "zeroed_tail": data[:-TAIL] + bytes(TAIL), "foreign": data[:-TAIL] + os.urandom(TAIL),
             "short_image": data[:4096] + data[-TAIL:], "too_short": data[:TAIL]}
    for name, blob in cases.items():
        p = tmp_path / name
        p.write_bytes(blob)
        with pytest.raises(L.FmaError) as ei:
            fma_b200.Engine.image_file_info(str(p))
        assert ei.value.code == (L.FMA_EIO if name in ("short_image", "too_short") else L.FMA_EINVAL), (name, ei.value)
    with pytest.raises(L.FmaError) as ei:
        fma_b200.Engine.image_file_info(str(tmp_path / "missing"))
    assert ei.value.code == L.FMA_EIO


# ---- the parking service's books, without an engine ----------------------------------------------------------------------
_DEPOSITOR = r"""
import sys
sys.path.insert(0, {root!r})
import fma_b200
from fma_b200.parking import ParkingClient
cli = ParkingClient(sys.argv[1])
for op in sys.argv[4:]:
    getattr(cli, op)(sys.argv[2], 0, *([sys.argv[3]] if op == "deposit_file" else []))
"""


def _books(tmp_path, images, **kw):
    from fma_b200.parking import ParkingService

    sock_dir = tempfile.mkdtemp(prefix="fma-", dir="/tmp")
    keep = kw.pop("keep_dir", str(tmp_path / "kept"))
    svc = ParkingService(os.path.join(sock_dir, "a.sock"), n_devices=1, keep_dir=keep, **kw)
    svc.start()
    script = tmp_path / "depositor.py"
    script.write_text(_DEPOSITOR.format(root=ROOT))

    def deposit(iid, src, *ops):
        dst = str(tmp_path / f"{iid}-r0.fmaimg")
        shutil.copyfile(src, dst)
        subprocess.check_call([sys.executable, str(script), svc.sock_path, iid, dst, *ops], cwd=ROOT)
        svc.instance_exited(iid)
        return dst

    return svc, deposit, sock_dir


def test_exit_hook_keeps_only_a_standing_deposit_with_digests(built, images, tmp_path):
    svc, deposit, sock_dir = _books(tmp_path, images)
    try:
        a = deposit("Ia", images[0][0], "deposit_file")
        assert not os.path.exists(a) and [k["instance_id"] for k in svc.kept()["images"]] == ["Ia"]
        b = deposit("Ib", images[0][0], "deposit_file", "withdraw_file")      # woken after the deposit: not kept
        assert not os.path.exists(b)
        c = deposit("Ic", images["nodigests"], "deposit_file")                # no digests: not kept
        assert not os.path.exists(c)
        d = deposit("Id", images[0][0])                                       # never deposited: not the owner's to touch
        assert os.path.exists(d)
        assert [k["instance_id"] for k in svc.kept()["images"]] == ["Ia"]
        e = tmp_path / "link.fmaimg"
        os.symlink(a, e)
        with pytest.raises(ValueError):
            svc.deposit_file("Ie", 0, str(e))
    finally:
        svc.close()
        shutil.rmtree(sock_dir, ignore_errors=True)


def test_disk_budget_evicts_least_recently_deposited_but_never_a_leased_file(built, images, tmp_path):
    size = os.path.getsize(images[0][0])
    svc, deposit, sock_dir = _books(tmp_path, images, keep_disk_bytes=2 * size)
    try:
        from fma_b200.parking import ParkingClient

        cli = ParkingClient(svc.sock_path)
        deposit("I1", images[0][0], "deposit_file")
        deposit("I2", images[0][0], "deposit_file")
        leased = cli.lookup_file("I1", 0)
        assert leased and os.path.exists(leased)
        deposit("I3", images[0][0], "deposit_file")                           # I1 is older but leased: I2 goes
        assert sorted(k["instance_id"] for k in svc.kept()["images"]) == ["I1", "I3"] and os.path.exists(leased)
        assert [k["leased"] for k in svc.kept()["images"] if k["instance_id"] == "I1"] == [True]
        cli.lookup_done("I1", 0)
        deposit("I4", images[0][0], "deposit_file")                           # now I1 is the oldest unleased one
        assert sorted(k["instance_id"] for k in svc.kept()["images"]) == ["I3", "I4"] and not os.path.exists(leased)
        assert cli.lookup_file("I3", 0) and (svc.instance_exited("I3") or True)   # a lease also ends when its instance exits
        assert all(not k["leased"] for k in svc.kept()["images"])
        assert cli.lookup_file("nobody", 0) is None
        st = svc.kept()
        assert st["disk_bytes"] == 2 * size and st["disk_budget_bytes"] == 2 * size
    finally:
        svc.close()
        shutil.rmtree(sock_dir, ignore_errors=True)
    svc, deposit, sock_dir = _books(tmp_path, images, keep_dir=str(tmp_path / "small"), keep_disk_bytes=size - 1)
    try:
        a = deposit("Ibig", images[0][0], "deposit_file")                     # bigger than the whole budget: not kept
        assert not os.path.exists(a) and svc.kept()["images"] == []
    finally:
        svc.close()
        shutil.rmtree(sock_dir, ignore_errors=True)


def test_dram_spill_writes_the_memfd_byte_for_byte_and_relisting_recovers(built, images, tmp_path):
    data = open(images[1][0], "rb").read()
    svc, deposit, sock_dir = _books(tmp_path, images, keep_dram_bytes=len(data) + 1)
    try:
        fds = []
        for iid in ("Ih1", "Ih2"):
            fd = os.memfd_create(iid)
            os.write(fd, data)
            fds.append(fd)
            svc.deposit_host(iid, 0, fd)
            svc.wait_spills()
        assert svc.lookup_host("Ih1", 0) is None and svc.lookup_host("Ih2", 0) is not None    # the older one went to disk
        path = svc.lookup_file("Ih1", 0)
        assert open(path, "rb").read() == data
        svc.lookup_done("Ih1", 0)
        listing = svc.kept()
        assert [(k["instance_id"], k["where"], k["packed"]) for k in listing["images"]] == [("Ih2", "dram", True), ("Ih1", "disk", True)]
        assert listing["dram_bytes"] == len(data) and listing["dram_budget_bytes"] == len(data) + 1
        svc.keep_dram_bytes = 0
        bad = os.memfd_create("Inod")                      # an image without digests cannot be kept on disk: it stays in DRAM
        os.write(bad, open(images["nodigests"], "rb").read())
        fds.append(bad)
        svc.deposit_host("Inod", 0, bad)
        svc.wait_spills()
        assert svc.lookup_host("Inod", 0) is not None and svc.lookup_file("Inod", 0) is None and svc.lookup_host("Ih2", 0) is None
        assert not any(n.startswith("Inod") for n in os.listdir(tmp_path / "kept"))
        for fd in fds:
            os.close(fd)
    finally:
        svc.close()
        shutil.rmtree(sock_dir, ignore_errors=True)
    keep = str(tmp_path / "kept")
    with open(os.path.join(keep, "Ihalf-r0.fmaimg.tmp"), "wb") as f:           # a spill cut short by a kill
        f.write(data[: len(data) // 2])
    shutil.copyfile(images["nodigests"], os.path.join(keep, "Ibad-r0.fmaimg"))
    older = os.path.join(keep, "Iold-r0.fmaimg")
    shutil.copyfile(images[0][0], older)
    os.utime(older, (time.time() - 100, time.time() - 100))
    svc, deposit, sock_dir = _books(tmp_path, images)
    try:
        assert sorted(os.listdir(keep)) == ["Ih1-r0.fmaimg", "Ih2-r0.fmaimg", "Iold-r0.fmaimg"]
        assert [k["instance_id"] for k in svc.kept()["images"]] == ["Iold", "Ih1", "Ih2"]   # mtime order
    finally:
        svc.close()
        shutil.rmtree(sock_dir, ignore_errors=True)


def test_node_agent_lists_kept_images_and_passes_the_budgets_on(built, images, tmp_path):
    from fastapi.testclient import TestClient

    from fma_b200.node_agent import NodeAgent, create_app, keep_settings

    assert keep_settings({"FMA_FILE_DIR": "/d"}) == {"keep_dir": "/d/kept", "keep_disk_bytes": None, "keep_dram_bytes": None}
    assert keep_settings({"FMA_KEEP_DIR": "/k", "FMA_KEEP_DISK_GIB": "1.5"})["keep_disk_bytes"] == int(1.5 * GiB)
    assert keep_settings({}) == {"keep_dir": None, "keep_disk_bytes": None, "keep_dram_bytes": None}
    svc, deposit, sock_dir = _books(tmp_path, images, keep_disk_bytes=GiB)
    try:
        deposit("Ia", images[1][0], "deposit_file")
        agent = NodeAgent(mock_gpus=True, log_dir=str(tmp_path), start_method="spawn", preload=(), parking=svc)
        c = TestClient(create_app(agent))
        got = c.get("/v2/node/images").json()
        assert [(i["instance_id"], i["rank"], i["where"], i["packed"], i["leased"]) for i in got["images"]] == [("Ia", 0, "disk", True, False)]
        assert got["disk_bytes"] == got["images"][0]["bytes"] == os.path.getsize(images[1][0]) and got["disk_budget_bytes"] == GiB
        assert got["images"][0]["kept_at"] > 0
        assert c.get("/").json()["endpoints"]["images"] == "GET /v2/node/images"
        assert NodeAgent(mock_gpus=True, start_method="spawn", preload=()).images()["images"] == []
    finally:
        svc.close()
        shutil.rmtree(sock_dir, ignore_errors=True)
