"""Node-level ownership of sleeping images in peer HBM (SURVEY.md §8f-1; VERDICT r1 "missing" 1).

The reference launcher pins every instance to its own GPUs (``inference_server/launcher/launcher.py:171-187`` overwrites
``CUDA_VISIBLE_DEVICES``), so an instance can neither allocate on an idle peer nor keep anything alive past its own death —
and the controller cold-starts a new instance exactly then (``pkg/controller/dual-pods/inference-server.go:416-448``).  The
node agent sees every GPU, so IT owns the parking buffers (``ParkingBuffer``: exportable VMM allocations) and hands file
descriptors to instances over a unix socket (``SCM_RIGHTS``); an instance attaches (``Engine.peer_attach``), sleeps to the peer
tier and deposits the image descriptor with the owner.  A later instance with the same ID — after a crash, a restart, a
reschedule onto the same node — looks the image up, attaches, adopts and wakes over NVLink instead of loading a checkpoint.

Wire format (one request per connection, JSON line + optional fd in the ancillary data):

    {"op": "park",    "instance": id, "rank": r, "bytes": n[, "device": d]} -> {"ok": true, "bytes": N, "device": d} + fd
    {"op": "deposit", "instance": id, "rank": r, "descriptor": hex}          -> {"ok": true}
    {"op": "lookup",  "instance": id, "rank": r}                             -> {"ok": true, "bytes": N, "device": d, "descriptor": hex} + fd
                                                                                | {"ok": false, "error": "..."}
    {"op": "deposit_host", "instance": id, "rank": r} + fd (memfd host store) -> {"ok": true}     the HOST-tier image (store + descriptor in its tail,
    {"op": "lookup_host",  "instance": id, "rank": r}                        -> {"ok": true} + fd | {"ok": false}   fma_image_export) outlives the instance too
    {"op": "helpers_open", "instance": id, "rank": r, "n": k, "avoid": [...], "slot_bytes": b, "slots": s}
                                                                             -> {"ok": true, "devices": [...]} + k fds   MULTI-PATH wake across processes:
    {"op": "pull", "instance": id, "rank": r, "generation": g} + [mailbox fd, store fd] -> {"ok": true}       the owner's helper GPUs pull for the instance
    {"op": "release", "instance": id[, "rank": r]}                           -> {"ok": true, "released": k}
    {"op": "stats"}                                                          -> {"ok": true, "parked_mib_per_device": {d: MiB}, "images": [...]}

Kept image files (opt-in: ``keep_dir``), so a deleted sleeper's next instance warm-starts from local disk:

    {"op": "deposit_file",  "instance": id, "rank": r, "path": p}            -> {"ok": true}   the file-tier image at p is the owner's from now on
    {"op": "withdraw_file", "instance": id, "rank": r}                       -> {"ok": true}   woken: p is no longer an image to keep
    {"op": "lookup_file",   "instance": id, "rank": r}                       -> {"ok": true, "path": kept path} (takes a lease) | {"ok": false}
    {"op": "lookup_done",   "instance": id, "rank": r[, "drop": true]}       -> {"ok": true}   ends the lease; drop: the file failed its digests
    {"op": "kept"}                                                           -> {"ok": true, "images": [...], "dram_bytes": ..., ...}

Live sleepers' host memory (opt-in: ``sleeper_dram_bytes``, FMA_NODE_SLEEPER_DRAM_GIB; SleeperDramBudget), one persistent
connection per rank, JSON lines both ways:

    {"op": "sleeper", "instance": id, "rank": r}                             -> {"ok": true}, then the connection stays open:
    up:   {"op": "sleeper_state", "asleep", "tier", "host_bytes", "image_bytes", "slept_at", "demoting", "file_dir", "shared"[, "answer", "error", "code"][, "failed"]}
    down: {"op": "demote"} | {"op": "promote"}

When an instance exits (``instance_exited``, from the node agent's child-exit path) with a file deposit standing, the file is kept
if ``fma_image_file_info`` accepts it and every segment carries a digest: it is renamed into ``keep_dir``.  Any other file the
instance deposited is unlinked.  Host memfds beyond ``keep_dram_bytes`` are spilled to kept files, oldest first; kept files beyond
``keep_disk_bytes`` are evicted least recently deposited first, never while leased.  On start the owner re-lists ``keep_dir``.

Placement: the caller may name the device; otherwise the owner picks the visible GPU with the fewest parked bytes that is not in
``avoid`` (the instance's own GPUs).  Through NVSwitch every peer is equally far, so this is a capacity decision (SURVEY §8e).
"""
from __future__ import annotations

import errno
import json
import logging
import os
import socket
import stat
import struct
import threading
import time
import urllib.parse
from typing import Callable, Dict, Optional, Tuple

MiB = 1 << 20
GiB = 1 << 30
logger = logging.getLogger("fma_b200.parking")


def _image_info(path: str) -> Optional[dict]:
    """fma_image_file_info of ``path`` (the one reader of the image format), None when it refuses the file."""
    from .engine import Engine, FmaError

    try:
        return Engine.image_file_info(path)
    except FmaError as e:
        logger.warning("fma_b200: %s is not a readable image: %s", path, e)
        return None


def _parked_packed(descriptor: bytes, store_bytes: int) -> Optional[bool]:
    """Whether a parked image is PACKED, from its descriptor alone: fma_image_file_info reads it behind a sparse memfd that stands
    for the parking buffer's bytes (none of them is written)."""
    from ._lib import FMA_IMAGE_TAIL_BYTES

    fd = os.memfd_create("fma-parked-descriptor", os.MFD_CLOEXEC)
    try:
        os.ftruncate(fd, store_bytes + FMA_IMAGE_TAIL_BYTES)
        os.pwrite(fd, descriptor, store_bytes)
        info = _image_info(f"/proc/self/fd/{fd}")
    finally:
        os.close(fd)
    return None if info is None else info["packed"]


def _kept_name(instance: str, rank: int) -> str:
    return f"{urllib.parse.quote(instance, safe='')}-r{int(rank)}.fmaimg"


def _parse_kept_name(name: str) -> Optional[Tuple[str, int]]:
    stem, sep, rank = name[:-len(".fmaimg")].rpartition("-r")
    if not name.endswith(".fmaimg") or not sep or not rank.isdigit():
        return None
    return urllib.parse.unquote(stem), int(rank)


class SleeperDramBudget:
    """FMA_NODE_SLEEPER_DRAM_GIB: the pinned host memory of a node's LIVE sleepers, the sum of the ``host_bytes`` each rank reports,
    kept within a budget.  Each rank is its own sleeper, keyed (instance, rank).  Pure bookkeeping over the ranks' ``sleeper_state``
    reports: ``send(key, op)`` delivers "demote" (the rank runs ``move_image(file, behind=True)``) or "promote" (``move_image(host)``)
    and the rank answers with a report that carries ``answer``.

    Demotion: while the sum is over budget, host-tier sleepers are demoted, least recently slept first; never an awake rank, one
    already demoting or with a command in flight, one whose store is shared or deposited (``shared``), or one whose demotion was
    refused or whose write failed since it last slept.  One demotion per file-tier directory (``file_dir``) at a time, so they do not split a disk.  A
    rank's bytes stop counting only when it reports the commit (tier "file", host_bytes 0); while a demotion writes, its bytes are
    set against the excess only so that no further rank is demoted for the same bytes.  A cancelled demotion (a wake cut it short)
    reports host_bytes again, and the policy re-runs on every report.
    Promotion: with no demotion writing and none needed, the most recently slept file-tier sleeper is promoted if its whole image
    fits under the budget; one at a time (a promotion is synchronous in the rank); never one whose promotion failed since it last
    slept.
    A failure is remembered per operation until the rank sleeps again (a new ``slept_at``): a command answered with ``error``, or a
    report with ``failed`` (a write-behind write that failed).  So neither a refusal nor a failing disk or pin is retried in a loop."""

    def __init__(self, budget_bytes: int, send: Callable[[Tuple[str, int], str], None]):
        self.budget = int(budget_bytes)
        self._send = send
        self._lock = threading.Lock()
        self._books: Dict[Tuple[str, int], dict] = {}     # (instance, rank) -> its last report
        self._pending: Dict[Tuple[str, int], str] = {}    # a command sent and not yet answered

    def used(self) -> int:
        with self._lock:
            return sum(int(s["host_bytes"]) for s in self._books.values())

    def report(self, state: dict) -> None:
        key = (str(state["instance"]), int(state.get("rank", 0)))
        with self._lock:
            old = self._books.get(key, {})
            s = dict(state)
            # operations that failed since this sleep: not asked again until the rank sleeps again
            s["failed_ops"] = set(old.get("failed_ops", ())) if old.get("slept_at") == s.get("slept_at") else set()
            if state.get("answer") and state.get("error"):
                s["failed_ops"].add(state["answer"])
            if state.get("failed"):
                s["failed_ops"].add(state["failed"])
            self._books[key] = s
            if state.get("answer"):
                self._pending.pop(key, None)
            cmds = self._plan()
        self._deliver(cmds)

    def drop(self, key: Tuple[str, int]) -> None:
        """The rank's connection closed (its process exited): its bytes leave the books, which may leave room for a promotion."""
        with self._lock:
            self._books.pop(key, None)
            self._pending.pop(key, None)
            cmds = self._plan()
        self._deliver(cmds)

    def promote(self, instance: str):
        """Promote every file-tier rank of ``instance`` ahead of an expected wake (an explicit request: also one whose promotion
        failed before).  None: no such sleeper; False: its images do not fit under the budget (nothing is sent); else the ranks being
        promoted (asked now or already), empty when none sleeps in the file tier (awake, or already in host DRAM)."""
        with self._lock:
            keys = [k for k in self._books if k[0] == instance]
            if not keys:
                return None
            asleep_in_file = [k for k in keys if self._books[k].get("asleep") and self._books[k].get("tier") == "file"]
            todo = [k for k in asleep_in_file if k not in self._pending]   # (a promotion in flight is not asked twice)
            need = sum(int(self._books[k].get("image_bytes", 0)) for k in todo)
            if sum(int(s["host_bytes"]) for s in self._books.values()) + need > self.budget:
                return False
            for k in todo:
                self._pending[k] = "promote"
        self._deliver([(k, "promote") for k in todo])
        return [k[1] for k in asleep_in_file]

    def sleepers(self) -> Dict[str, dict]:
        """Per instance: the tier of its rank 0, its ranks' host bytes, and whether one of them is demoting."""
        out: Dict[str, dict] = {}
        with self._lock:
            for (inst, rank), s in sorted(self._books.items()):
                o = out.setdefault(inst, {"tier": s.get("tier"), "host_bytes": 0, "demoting": False})
                o["host_bytes"] += int(s["host_bytes"])
                o["demoting"] = o["demoting"] or bool(s.get("demoting")) or self._pending.get((inst, rank)) == "demote"
        return out

    def _in_flight(self, key) -> bool:
        return bool(self._books[key].get("demoting")) or self._pending.get(key) == "demote"

    def _plan(self) -> list:
        cmds = []
        used = sum(int(s["host_bytes"]) for s in self._books.values())
        writing = [k for k in self._books if self._in_flight(k)]
        excess = used - sum(int(self._books[k]["host_bytes"]) for k in writing) - self.budget
        if excess > 0:
            busy = {self._books[k].get("file_dir") for k in writing}
            for k, s in sorted(self._books.items(), key=lambda kv: (kv[1].get("slept_at", 0), kv[0])):
                if excess <= 0:
                    break
                if (not s.get("asleep") or s.get("tier") != "host" or k in self._pending or self._in_flight(k) or s.get("shared")
                        or "demote" in s["failed_ops"] or s.get("file_dir") in busy or not int(s["host_bytes"])):
                    continue
                cmds.append((k, "demote"))
                self._pending[k] = "demote"
                busy.add(s.get("file_dir"))
                excess -= int(s["host_bytes"])
            return cmds
        if writing or self._pending:
            return cmds
        for k, s in sorted(self._books.items(), key=lambda kv: (kv[1].get("slept_at", 0), kv[0]), reverse=True):
            if (s.get("asleep") and s.get("tier") == "file" and "promote" not in s["failed_ops"]
                    and used + int(s.get("image_bytes", 0)) <= self.budget):
                cmds.append((k, "promote"))
                self._pending[k] = "promote"
                break
        return cmds

    def _deliver(self, cmds) -> None:
        for key, op in cmds:
            try:
                self._send(key, op)
            except OSError as e:            # the rank is gone: its connection's close drops it
                logger.warning("fma_b200: cannot send %s to %s rank %d: %s", op, key[0], key[1], e)
                with self._lock:
                    self._pending.pop(key, None)


class ParkingService:
    """Owner side.  ``make_buffer(device, nbytes)`` must return an object with ``.nbytes``, ``.device``, ``.export_fd()`` and
    ``.close()`` — ``fma_b200.ParkingBuffer`` in production."""

    def __init__(self, sock_path: str, n_devices: int, make_buffer: Optional[Callable] = None, keep_dir: Optional[str] = None,
                 keep_disk_bytes: Optional[int] = None, keep_dram_bytes: Optional[int] = None, sleeper_dram_bytes: Optional[int] = None):
        """``keep_dir`` turns on kept image files (None: the file ops are refused and host deposits are unbounded, as before);
        ``keep_disk_bytes`` / ``keep_dram_bytes`` bound the kept files and the deposited host memfds (None: no bound).
        ``sleeper_dram_bytes`` bounds the host bytes of live sleepers (SleeperDramBudget; None: no bound, as before)."""
        self.sock_path = sock_path
        self.n_devices = n_devices
        if make_buffer is None:
            from .engine import ParkingBuffer

            make_buffer = ParkingBuffer
        self._make = make_buffer
        self._lock = threading.Lock()
        self._images: Dict[Tuple[str, int], dict] = {}   # (instance, rank) -> {"buf", "descriptor"}
        self._host_images: Dict[Tuple[str, int], int] = {}   # (instance, rank) -> fd of the memfd host store (image + descriptor)
        self._helpers: Dict[Tuple[str, int], list] = {}      # (instance, rank) -> [HelperStaging] (remote wake paths, one per helper GPU)
        self._stores: Dict[Tuple[int, int], int] = {}        # (st_dev, st_ino) of an instance's memfd store -> attached-store handle
        self._host_at: Dict[Tuple[str, int], float] = {}     # (instance, rank) -> when its host memfd was deposited
        self._spilling: set = set()                          # host images being written to kept files
        self._unspillable: set = set()                       # (key, fd) of host images that could not be kept on disk: they stay
        self._spill_pending = False                          # a deposit arrived since the spill thread last looked
        self._spill_thread: Optional[threading.Thread] = None
        self._admitting = 0                                  # bytes of kept files being renamed into place (counted in the budget)
        # kept image files: the standing file deposits of live instances, and the files this owner keeps (dict order: least
        # recently deposited first)
        self._file_deps: Dict[Tuple[str, int], dict] = {}    # (instance, rank) -> {"path", "ino": (st_dev, st_ino), "standing"}
        self._kept: Dict[Tuple[str, int], dict] = {}         # (instance, rank) -> {"path", "bytes", "packed", "kept_at", "leases"}
        self.keep_dir = keep_dir
        self.keep_disk_bytes = keep_disk_bytes
        self.keep_dram_bytes = keep_dram_bytes
        if keep_dir:
            os.makedirs(keep_dir, exist_ok=True)
            self._relist()
        self._srv: Optional[socket.socket] = None
        self._thread: Optional[threading.Thread] = None
        self._stop = False
        # live sleepers' host memory (opt-in): one persistent connection per rank ("sleeper" op), commands sent down it
        self._sleeper_conns: Dict[Tuple[str, int], Tuple[socket.socket, threading.Lock]] = {}
        self.sleeper_budget = SleeperDramBudget(sleeper_dram_bytes, self._send_sleeper) if sleeper_dram_bytes is not None else None

    def _send_sleeper(self, key: Tuple[str, int], op: str) -> None:
        if key not in self._sleeper_conns:
            raise OSError(f"no connection from {key[0]} rank {key[1]}")
        conn, lock = self._sleeper_conns[key]
        with lock:
            conn.sendall((json.dumps({"op": op}) + "\n").encode())

    def _serve_sleeper(self, conn: socket.socket, instance: str, rank: int) -> None:
        """A rank's persistent connection: its sleeper_state reports come up, demote / promote go down; its close (the process
        exited) drops the rank from the budget's books."""
        key = (instance, int(rank))
        self._sleeper_conns[key] = (conn, threading.Lock())
        conn.sendall((json.dumps({"ok": True}) + "\n").encode())
        buf = b""
        try:
            while True:
                more = conn.recv(1 << 16)
                if not more:
                    break
                buf += more
                while b"\n" in buf:
                    line, buf = buf.split(b"\n", 1)
                    msg = json.loads(line.decode())
                    if msg.get("op") == "sleeper_state":
                        self.sleeper_budget.report(dict(msg, instance=instance, rank=int(rank)))
        except OSError:
            pass
        finally:
            if self._sleeper_conns.get(key, (None,))[0] is conn:
                del self._sleeper_conns[key]
            self.sleeper_budget.drop(key)

    # ---- bookkeeping ------------------------------------------------------------------------------------------
    def parked_bytes_per_device(self) -> Dict[int, int]:
        out = {d: 0 for d in range(self.n_devices)}
        with self._lock:
            for img in self._images.values():
                out[img["buf"].device] += img["buf"].nbytes
        return out

    def stats(self) -> dict:
        per = self.parked_bytes_per_device()
        with self._lock:
            images = [{"instance": k[0], "rank": k[1], "device": v["buf"].device, "mib": v["buf"].nbytes // MiB,
                       "has_image": v["descriptor"] is not None} for k, v in sorted(self._images.items())]
            host = [{"instance": k[0], "rank": k[1], "mib": os.fstat(fd).st_size // MiB} for k, fd in sorted(self._host_images.items())]
        return {"parked_mib_per_device": {str(d): b // MiB for d, b in per.items()}, "images": images, "host_images": host}

    def _candidates(self, avoid) -> list:
        """GPUs outside `avoid`, least parked bytes first (lowest index on a tie)."""
        per = self.parked_bytes_per_device()
        cands = [d for d in range(self.n_devices) if d not in set(avoid or [])]
        if not cands:
            raise ValueError("no GPU left to park on")
        return sorted(cands, key=lambda d: (per[d], d))

    # ---- operations -------------------------------------------------------------------------------------------
    def park(self, instance: str, rank: int, nbytes: int, device: Optional[int] = None, avoid=None):
        key = (instance, int(rank))
        with self._lock:
            old = self._images.get(key)
        if old is not None and old["buf"].nbytes >= nbytes and (device is None or old["buf"].device == device):
            old["descriptor"] = None                      # about to be overwritten by a new sleep
            return old["buf"]
        if old is not None:
            self.release(instance, rank)
        # What this service has parked is all it knows about a GPU's HBM: an awake instance may fill the rest.  So the least-loaded
        # candidate is only tried first; a GPU that cannot take the buffer (cuMemCreate fails) passes it on to the next one, and
        # only when none can is the park refused — the caller then sleeps to the host tier (cumem.py).
        last = None
        for dev in (self._candidates(avoid) if device is None else [int(device)]):
            try:
                buf = self._make(dev, int(nbytes))
            except Exception as e:      # noqa: BLE001
                last = e
                continue
            with self._lock:
                self._images[key] = {"buf": buf, "descriptor": None}
            return buf
        raise RuntimeError(f"no GPU can take {int(nbytes) // MiB} MiB right now: {last}")

    def deposit(self, instance: str, rank: int, descriptor: bytes) -> None:
        with self._lock:
            img = self._images[(instance, int(rank))]
            img["descriptor"], img["kept_at"] = bytes(descriptor), time.time()

    def lookup(self, instance: str, rank: int):
        with self._lock:
            img = self._images.get((instance, int(rank)))
            if img is None or img["descriptor"] is None:
                return None
            return img["buf"], img["descriptor"]

    def deposit_host(self, instance: str, rank: int, fd: int) -> None:
        """Keep (a dup of) the memfd behind a sleeping instance's host store: image + descriptor, as fma_image_export hands it out."""
        key = (instance, int(rank))
        with self._lock:
            old = self._host_images.pop(key, None)
            self._host_images[key] = os.dup(fd)
            self._host_at[key] = time.time()
            self._unspillable = {u for u in self._unspillable if u[0] != key}
        if old is not None:
            os.close(old)
        self._kick_spill()

    def lookup_host(self, instance: str, rank: int) -> Optional[int]:
        with self._lock:
            return self._host_images.get((instance, int(rank)))

    # ---- kept image files ---------------------------------------------------------------------------------------
    def _need_keep_dir(self) -> None:
        if not self.keep_dir:
            raise RuntimeError("this node agent keeps no image files (no FMA_KEEP_DIR)")

    def deposit_file(self, instance: str, rank: int, path: str, uid: Optional[int] = None) -> None:
        """A live instance's file-tier image at ``path`` becomes this owner's: kept if the instance exits with the deposit standing,
        unlinked otherwise.  Only a regular file (not a link) of the depositing user (``uid``, from the socket's credentials) is
        taken, and only that very file (device and inode) is renamed or unlinked later."""
        self._need_keep_dir()
        st = os.lstat(path)
        if not stat.S_ISREG(st.st_mode) or (uid is not None and st.st_uid != uid):
            raise ValueError(f"{path} is not a regular file of the depositing user")
        with self._lock:
            self._file_deps[(instance, int(rank))] = {"path": os.path.abspath(path), "ino": (st.st_dev, st.st_ino), "standing": True}

    def withdraw_file(self, instance: str, rank: int) -> None:
        with self._lock:
            dep = self._file_deps.get((instance, int(rank)))
            if dep is not None:
                dep["standing"] = False

    def lookup_file(self, instance: str, rank: int) -> Optional[str]:
        """Path of the kept file of (instance, rank), under a lease that lasts until ``lookup_done`` or the instance's exit."""
        with self._lock:
            k = self._kept.get((instance, int(rank)))
            if k is None:
                return None
            k["leases"] += 1
            return k["path"]

    def lookup_done(self, instance: str, rank: int, drop: bool = False) -> None:
        """Ends a lease.  ``drop``: the adopter found the image damaged (FMA_EINTEGRITY), so it is deleted."""
        key = (instance, int(rank))
        with self._lock:
            k = self._kept.get(key)
            if k is None:
                return
            k["leases"] = max(0, k["leases"] - 1)
            if drop:
                del self._kept[key]
        if drop:
            _unlink(k["path"])

    def instance_exited(self, instance: str) -> None:
        """The node agent's child-exit hook: the instance's leases end, and each file it deposited is kept (deposit standing, the
        file parses and carries digests) or unlinked.  Idempotent."""
        with self._lock:
            for key, k in self._kept.items():
                if key[0] == instance:
                    k["leases"] = 0
            deps = [(key, self._file_deps.pop(key)) for key in [key for key in self._file_deps if key[0] == instance]]
        for key, dep in deps:
            try:
                st = os.lstat(dep["path"])
            except FileNotFoundError:
                continue
            if (st.st_dev, st.st_ino) != dep["ino"]:
                continue                                   # not the file that was deposited: not ours to touch
            if dep["standing"]:
                self._admit(key, dep["path"])
            else:
                _unlink(dep["path"])

    def _file_info(self, path: str) -> Optional[dict]:
        """fma_image_file_info of a file that may be kept: None unless it parses and every segment carries a digest (an adopter
        wakes with FMA_FLAG_VERIFY, which checks only the segments that carry one)."""
        info = _image_info(path)
        if info is None:
            return None
        if not info["digests"]:
            logger.warning("fma_b200: %s carries no digests (sleep with FMA_FLAG_VERIFY): not kept", path)
            return None
        return info

    def _admit(self, key: Tuple[str, int], path: str, kept_at: Optional[float] = None) -> bool:
        """Move the image file ``path`` into keep_dir as the kept image of ``key`` (replacing an older one), within the disk budget;
        a file that cannot be kept is unlinked.  True when it was kept."""
        info = self._file_info(path)
        nbytes = os.path.getsize(path) if info else 0
        if info is None or (self.keep_disk_bytes is not None and nbytes > self.keep_disk_bytes):
            if info is not None:
                logger.warning("fma_b200: %s (%.2f GiB) is bigger than the kept-image budget: not kept", path, nbytes / GiB)
            _unlink(path)
            return False
        dest = os.path.join(self.keep_dir, _kept_name(*key))
        with self._lock:
            old = self._kept.pop(key, None)
            evict = self._evictions(nbytes)
            if evict is None:
                if old is not None:
                    self._kept[key] = old
                leased = True
            else:
                leased = False
                for v in evict:
                    del self._kept[v]
                self._admitting += nbytes                 # until the entry is in place, a concurrent admission counts these bytes
        if leased:
            logger.warning("fma_b200: no room for %s among leased kept images: not kept", path)
            _unlink(path)
            return False
        try:
            os.rename(path, dest)
        except OSError as e:                              # another filesystem than keep_dir's, for one
            logger.warning("fma_b200: cannot move %s to %s (%s): not kept", path, dest, e)
            _unlink(path)
            dest = None
        for p in [v["path"] for v in evict.values()] + ([old["path"]] if old is not None and old["path"] != dest else []):
            _unlink(p)
        with self._lock:
            self._admitting -= nbytes
            if dest is not None:
                self._kept[key] = {"path": dest, "bytes": nbytes, "packed": info["packed"], "kept_at": kept_at or time.time(), "leases": 0}
        return dest is not None

    def _evictions(self, nbytes: int) -> Optional[Dict[Tuple[str, int], dict]]:
        """Kept images to evict, least recently deposited first and never a leased one, so that ``nbytes`` more fit the disk
        budget; None when they cannot (caller holds the lock)."""
        if self.keep_disk_bytes is None:
            return {}
        over = sum(k["bytes"] for k in self._kept.values()) + self._admitting + nbytes - self.keep_disk_bytes
        out: Dict[Tuple[str, int], dict] = {}
        for key, k in self._kept.items():
            if over <= 0:
                break
            if k["leases"] == 0:
                out[key] = k
                over -= k["bytes"]
        return out if over <= 0 else None

    def _kick_spill(self) -> None:
        """Spills run on one background thread, so a deposit's reply never waits for another image's disk write."""
        if not self.keep_dir or self.keep_dram_bytes is None:
            return
        with self._lock:
            self._spill_pending = True
            if self._spill_thread is None:
                self._spill_thread = threading.Thread(target=self._spill_worker, name="fma-spill", daemon=True)
                self._spill_thread.start()

    def _spill_worker(self) -> None:
        while True:
            with self._lock:
                if not self._spill_pending or self._stop:
                    self._spill_thread = None
                    return
                self._spill_pending = False
            self._spill_over_budget()

    def wait_spills(self) -> None:
        """Returns once no spill is running or pending."""
        while True:
            with self._lock:
                t = self._spill_thread
            if t is None:
                return
            t.join()

    def _spill_over_budget(self) -> None:
        """Write the oldest deposited host memfds to kept files until the rest fit ``keep_dram_bytes``.  One that cannot be kept
        stays in DRAM (and is not tried again): a spill never loses an image."""
        while True:
            with self._lock:
                total = sum(os.fstat(fd).st_size for fd in self._host_images.values())
                live = {k: fd for k, fd in self._host_images.items() if k not in self._spilling and (k, fd) not in self._unspillable}
                if total <= self.keep_dram_bytes or not live:
                    return
                key = min(live, key=lambda k: self._host_at.get(k, 0.0))
                self._spilling.add(key)
                fd, at = live[key], self._host_at.get(key)
            try:
                self._spill(key, fd, at)
            finally:
                with self._lock:
                    self._spilling.discard(key)

    def _spill(self, key: Tuple[str, int], fd: int, kept_at: Optional[float]) -> None:
        """One host memfd to a kept file: a byte copy (the memfd has image_save's layout) to ``<name>.tmp``, fdatasync, rename; only
        then is the memfd closed, so lookup_host misses and lookup_file hits.  If the file cannot be kept (no digests, no room, a
        failed write), the memfd stays where it is."""
        tmp = os.path.join(self.keep_dir, _kept_name(*key) + ".tmp")
        n = os.fstat(fd).st_size
        try:
            out = os.open(tmp, os.O_WRONLY | os.O_CREAT | os.O_TRUNC | os.O_CLOEXEC, 0o600)
            try:
                off = 0
                while off < n:
                    chunk = os.pread(fd, min(64 * MiB, n - off), off)
                    if not chunk:
                        raise OSError(errno.EIO, "the host image ends early")
                    off += os.pwrite(out, chunk, off)
                os.fdatasync(out)
            finally:
                os.close(out)
        except OSError as e:
            logger.warning("fma_b200: cannot spill the host image of %s rank %d to %s (%s)", key[0], key[1], tmp, e)
            _unlink(tmp)
            kept = False
        else:
            kept = self._admit(key, tmp, kept_at)
        with self._lock:
            if self._host_images.get(key) != fd:
                return                                     # replaced or released meanwhile: that path closes it
            if not kept:
                logger.warning("fma_b200: the host image of %s rank %d stays in DRAM, over the budget", key[0], key[1])
                self._unspillable.add((key, fd))
                return
            del self._host_images[key]
            self._host_at.pop(key, None)
        os.close(fd)
        logger.info("fma_b200: host image of %s rank %d (%.2f GiB) spilled to disk", key[0], key[1], n / GiB)

    def _relist(self) -> None:
        """Start-up: ``*.tmp`` leftovers of an interrupted spill go; every image file that fma_image_file_info accepts is kept, in
        mtime order, within the disk budget."""
        found = []
        for name in os.listdir(self.keep_dir):
            p = os.path.join(self.keep_dir, name)
            if name.endswith(".tmp"):
                _unlink(p)
            elif _parse_kept_name(name) is not None and os.path.isfile(p):
                found.append((os.path.getmtime(p), name, p))
        for mtime, name, p in sorted(found):
            info = self._file_info(p)
            if info is None:
                _unlink(p)
                continue
            with self._lock:
                self._kept[_parse_kept_name(name)] = {"path": p, "bytes": os.path.getsize(p), "packed": info["packed"], "kept_at": mtime, "leases": 0}
        with self._lock:
            evict = self._evictions(0) or {}
            for key in evict:
                del self._kept[key]
        for k in evict.values():
            _unlink(k["path"])

    def kept(self) -> dict:
        """Every image kept for a dead or future instance: parked in peer HBM, host memfds in DRAM, files on disk."""
        out = []
        with self._lock:
            for (inst, rank), v in sorted(self._images.items()):
                if v["descriptor"] is not None:
                    out.append({"instance_id": inst, "rank": rank, "where": "peer", "bytes": v["buf"].nbytes,
                                "packed": _parked_packed(v["descriptor"], v["buf"].nbytes), "kept_at": v.get("kept_at"), "leased": False})
            dram = 0
            for (inst, rank), fd in sorted(self._host_images.items()):
                n = os.fstat(fd).st_size
                dram += n
                info = _image_info(f"/proc/self/fd/{fd}")
                out.append({"instance_id": inst, "rank": rank, "where": "dram", "bytes": n, "packed": None if info is None else info["packed"],
                            "kept_at": self._host_at.get((inst, rank)), "leased": False})
            disk = 0
            for (inst, rank), k in self._kept.items():
                disk += k["bytes"]
                out.append({"instance_id": inst, "rank": rank, "where": "disk", "bytes": k["bytes"], "packed": k["packed"], "kept_at": k["kept_at"],
                            "leased": k["leases"] > 0})
        return {"images": out, "dram_bytes": dram, "dram_budget_bytes": self.keep_dram_bytes, "disk_bytes": disk,
                "disk_budget_bytes": self.keep_disk_bytes, "keep_dir": self.keep_dir}

    # ---- MULTI-PATH wake across processes (fma_pull.h): helpers owned here pull chunks for an instance that cannot see their GPUs ----
    def helpers_open(self, instance: str, rank: int, n: int, avoid=None, slot_bytes: int = 128 << 20, slots: int = 3) -> list:
        from .engine import HelperStaging

        key = (instance, int(rank))
        with self._lock:
            have = self._helpers.get(key)
        if have and len(have) == n and have[0].slot_bytes == slot_bytes and have[0].slots == slots:
            return have
        for h in have or []:
            h.close()
        cands = [d for d in range(self.n_devices) if d not in set(avoid or [])][: int(n)]
        made = [HelperStaging(d, slot_bytes, slots) for d in cands]
        with self._lock:
            self._helpers[key] = made
        return made

    def pull(self, instance: str, rank: int, generation: int, mailbox_fd: int, store_fd: int, timeout_s: float = 5.0) -> int:
        """Start one pull thread per helper of (instance, rank) for the wake `generation`; returns the number of helpers."""
        from .engine import store_attach

        st = os.fstat(store_fd)
        skey = (st.st_dev, st.st_ino)
        with self._lock:
            helpers = list(self._helpers.get((instance, int(rank)), []))
            if skey not in self._stores:
                self._stores[skey] = store_attach(store_fd)
            store = self._stores[skey]
        mb = os.dup(mailbox_fd)
        left = [len(helpers)]

        def run(h, path_index):
            try:
                h.pull(store, mb, path_index, generation, timeout_s)
            except Exception:      # a failed / superseded pull only costs speed: the instance's other paths finish the wake
                pass
            finally:
                with self._lock:
                    left[0] -= 1
                    last = left[0] == 0
                if last:
                    os.close(mb)

        for k, h in enumerate(helpers):
            threading.Thread(target=run, args=(h, k + 1), name=f"fma-pull-{h.device}", daemon=True).start()
        if not helpers:
            os.close(mb)
        return len(helpers)

    def release(self, instance: str, rank: Optional[int] = None) -> int:
        with self._lock:
            for k in [k for k in self._helpers if k[0] == instance and (rank is None or k[1] == int(rank))]:
                for h in self._helpers.pop(k):
                    h.close()
        with self._lock:
            keys = [k for k in self._images if k[0] == instance and (rank is None or k[1] == int(rank))]
            bufs = [self._images.pop(k)["buf"] for k in keys]
            hkeys = [k for k in self._host_images if k[0] == instance and (rank is None or k[1] == int(rank))]
            hfds = [self._host_images.pop(k) for k in hkeys]
            for k in hkeys:
                self._host_at.pop(k, None)
            self._unspillable = {u for u in self._unspillable if u[0] not in hkeys}
        for b in bufs:
            b.close()
        for fd in hfds:
            os.close(fd)
        return len(bufs) + len(hfds)

    # ---- socket server ----------------------------------------------------------------------------------------
    def start(self) -> None:
        try:
            os.unlink(self.sock_path)
        except FileNotFoundError:
            pass
        self._srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self._srv.bind(self.sock_path)
        os.chmod(self.sock_path, 0o600)
        self._srv.listen(64)
        self._thread = threading.Thread(target=self._serve, name="fma-parking", daemon=True)
        self._thread.start()

    def _serve(self) -> None:
        while not self._stop:
            try:
                conn, _ = self._srv.accept()
            except OSError:
                return
            threading.Thread(target=self._handle, args=(conn,), daemon=True).start()

    def _handle(self, conn: socket.socket) -> None:
        fd_to_close = None
        got_fds: list = []
        try:
            data, got_fds, _, _ = socket.recv_fds(conn, 1 << 20, 4)
            while not data.endswith(b"\n"):
                more = conn.recv(1 << 20)
                if not more:
                    break
                data += more
            req = json.loads(data.decode())
            op, fds = req.get("op"), []
            if op == "park":
                buf = self.park(req["instance"], req.get("rank", 0), int(req["bytes"]), req.get("device"), req.get("avoid"))
                fd_to_close = buf.export_fd()
                fds = [fd_to_close]
                rep = {"ok": True, "bytes": buf.nbytes, "device": buf.device}
            elif op == "deposit":
                self.deposit(req["instance"], req.get("rank", 0), bytes.fromhex(req["descriptor"]))
                rep = {"ok": True}
            elif op == "lookup":
                hit = self.lookup(req["instance"], req.get("rank", 0))
                if hit is None:
                    rep = {"ok": False, "error": "no parked image for that instance / rank"}
                else:
                    fd_to_close = hit[0].export_fd()
                    fds = [fd_to_close]
                    rep = {"ok": True, "bytes": hit[0].nbytes, "device": hit[0].device, "descriptor": hit[1].hex()}
            elif op == "deposit_host":
                if not got_fds:
                    rep = {"ok": False, "error": "deposit_host needs the store's fd in the ancillary data"}
                else:
                    self.deposit_host(req["instance"], req.get("rank", 0), got_fds[0])
                    rep = {"ok": True}
            elif op == "lookup_host":
                hfd = self.lookup_host(req["instance"], req.get("rank", 0))
                if hfd is None:
                    rep = {"ok": False, "error": "no host image for that instance / rank"}
                else:
                    fds = [hfd]
                    rep = {"ok": True, "bytes": os.fstat(hfd).st_size}
            elif op == "helpers_open":
                hs = self.helpers_open(req["instance"], req.get("rank", 0), int(req["n"]), req.get("avoid"), int(req.get("slot_bytes") or (128 << 20)), int(req.get("slots") or 3))
                fds = [h.fd for h in hs]
                rep = {"ok": True, "devices": [h.device for h in hs], "slot_bytes": hs[0].slot_bytes if hs else 0, "slots": hs[0].slots if hs else 0}
            elif op == "pull":
                if len(got_fds) < 2:
                    rep = {"ok": False, "error": "pull needs the mailbox fd and the store fd"}
                else:
                    rep = {"ok": True, "helpers": self.pull(req["instance"], req.get("rank", 0), int(req["generation"]), got_fds[0], got_fds[1], float(req.get("timeout_s", 5.0)))}
            elif op == "release":
                rep = {"ok": True, "released": self.release(req["instance"], req.get("rank"))}
            elif op == "stats":
                rep = {"ok": True, **self.stats()}
            elif op == "deposit_file":
                uid = struct.unpack("3i", conn.getsockopt(socket.SOL_SOCKET, socket.SO_PEERCRED, struct.calcsize("3i")))[1]
                self.deposit_file(req["instance"], req.get("rank", 0), req["path"], uid=uid)
                rep = {"ok": True}
            elif op == "withdraw_file":
                self.withdraw_file(req["instance"], req.get("rank", 0))
                rep = {"ok": True}
            elif op == "lookup_file":
                path = self.lookup_file(req["instance"], req.get("rank", 0))
                rep = {"ok": True, "path": path} if path else {"ok": False, "error": "no kept image file for that instance / rank"}
            elif op == "lookup_done":
                self.lookup_done(req["instance"], req.get("rank", 0), bool(req.get("drop")))
                rep = {"ok": True}
            elif op == "kept":
                rep = {"ok": True, **self.kept()}
            elif op == "sleeper" and self.sleeper_budget is not None:
                self._serve_sleeper(conn, req["instance"], req.get("rank", 0))
                return
            else:
                rep = {"ok": False, "error": f"unknown op {op!r}"}
            socket.send_fds(conn, [(json.dumps(rep) + "\n").encode()], fds)
        except Exception as e:  # a bad request must not take the owner down
            try:
                conn.sendall((json.dumps({"ok": False, "error": str(e)[:200]}) + "\n").encode())
            except OSError:
                pass
        finally:
            if fd_to_close is not None:
                os.close(fd_to_close)
            for fd in got_fds:
                os.close(fd)
            conn.close()

    def close(self) -> None:
        self.wait_spills()
        self._stop = True
        if self._srv is not None:
            self._srv.close()
        try:
            os.unlink(self.sock_path)
        except FileNotFoundError:
            pass
        with self._lock:
            bufs = [v["buf"] for v in self._images.values()]
            self._images.clear()
            hfds = list(self._host_images.values())
            self._host_images.clear()
        for b in bufs:
            b.close()
        for fd in hfds:
            os.close(fd)


def _unlink(path: str) -> None:
    try:
        os.unlink(path)
    except FileNotFoundError:
        pass


class ParkingClient:
    """Instance side (the allocator shim, one per rank).  ``sock_path`` comes from ``FMA_NODE_AGENT_SOCK``."""

    def __init__(self, sock_path: Optional[str] = None):
        self.sock_path = sock_path or os.environ.get("FMA_NODE_AGENT_SOCK", "")
        if not self.sock_path:
            raise RuntimeError("no node agent socket (FMA_NODE_AGENT_SOCK)")
        self._mailbox = -1
        self._last_fds: list = []

    def _rpc(self, req: dict, send_fds=()):
        with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as s:
            s.connect(self.sock_path)
            if send_fds:
                socket.send_fds(s, [(json.dumps(req) + "\n").encode()], list(send_fds))
            else:
                s.sendall((json.dumps(req) + "\n").encode())
            data, fds, _, _ = socket.recv_fds(s, 1 << 22, 8)
            while not data.endswith(b"\n"):
                more = s.recv(1 << 22)
                if not more:
                    break
                data += more
        rep = json.loads(data.decode())
        self._last_fds = list(fds)
        return rep, (fds[0] if fds else None)

    def park(self, engine, instance: str, rank: int, nbytes: int, device: Optional[int] = None, avoid=None) -> dict:
        rep, fd = self._rpc({"op": "park", "instance": instance, "rank": rank, "bytes": nbytes, "device": device, "avoid": avoid})
        if not rep.get("ok") or fd is None:
            raise RuntimeError(rep.get("error", "park refused"))
        try:
            engine.peer_attach(fd, rep["bytes"])
        finally:
            os.close(fd)
        return rep

    def deposit(self, engine, instance: str, rank: int, tier: int = 1) -> None:
        rep, _ = self._rpc({"op": "deposit", "instance": instance, "rank": rank, "descriptor": engine.image_describe(tier).hex()})
        if not rep.get("ok"):
            raise RuntimeError(rep.get("error", "deposit refused"))

    def adopt(self, engine, instance: str, rank: int, tags=("weights",)) -> bool:
        """If the owner holds a parked image for (instance, rank): attach + adopt it (the engine is then asleep with that image and
        a wake restores the weights over NVLink).  False = nothing parked: load the checkpoint as usual."""
        rep, fd = self._rpc({"op": "lookup", "instance": instance, "rank": rank})
        if not rep.get("ok") or fd is None:
            return False
        try:
            engine.peer_attach(fd, rep["bytes"])
            engine.image_adopt_parked(bytes.fromhex(rep["descriptor"]), list(tags))
        finally:
            os.close(fd)
        return True

    def deposit_host(self, engine, instance: str, rank: int) -> None:
        """HOST tier: hand the sleeping image's memfd (store + descriptor; needs FMA_HOST_STORE_SHM=1) to the owner."""
        fd = engine.image_export()
        try:
            rep, _ = self._rpc({"op": "deposit_host", "instance": instance, "rank": rank}, send_fds=[fd])
        finally:
            os.close(fd)
        if not rep.get("ok"):
            raise RuntimeError(rep.get("error", "deposit_host refused"))

    def adopt_host(self, engine, instance: str, rank: int, tags=("weights",)) -> bool:
        """If the owner keeps a host image for (instance, rank): adopt it (the engine is then asleep with that image)."""
        rep, fd = self._rpc({"op": "lookup_host", "instance": instance, "rank": rank})
        if not rep.get("ok") or fd is None:
            return False
        try:
            engine.image_adopt(fd, list(tags))
        finally:
            os.close(fd)
        return True

    def deposit_file(self, instance: str, rank: int, path: str) -> None:
        """FILE tier: the image this rank just wrote to ``path`` becomes the owner's, kept if the process exits with it standing."""
        rep, _ = self._rpc({"op": "deposit_file", "instance": instance, "rank": rank, "path": os.path.abspath(path)})
        if not rep.get("ok"):
            raise RuntimeError(rep.get("error", "deposit_file refused"))

    def withdraw_file(self, instance: str, rank: int) -> None:
        rep, _ = self._rpc({"op": "withdraw_file", "instance": instance, "rank": rank})
        if not rep.get("ok"):
            raise RuntimeError(rep.get("error", "withdraw_file refused"))

    def lookup_file(self, instance: str, rank: int) -> Optional[str]:
        """Path of a kept image file for (instance, rank), leased until ``lookup_done``; None when there is none."""
        rep, _ = self._rpc({"op": "lookup_file", "instance": instance, "rank": rank})
        return rep["path"] if rep.get("ok") else None

    def lookup_done(self, instance: str, rank: int, drop: bool = False) -> None:
        self._rpc({"op": "lookup_done", "instance": instance, "rank": rank, "drop": drop})

    def kept(self) -> dict:
        return self._rpc({"op": "kept"})[0]

    def attach_remote_paths(self, engine, instance: str, rank: int, n_helpers: int, avoid=None, slot_bytes: int = 128 << 20, slots: int = 3) -> int:
        """MULTI-PATH wake for an instance that cannot see the helper GPUs: the owner opens one staging buffer per helper, the engine maps
        them for its GPU (``Engine.paths_attach``) and keeps the mailbox; ``request_pull`` then goes before every host-tier wake."""
        rep, _ = self._rpc({"op": "helpers_open", "instance": instance, "rank": rank, "n": n_helpers, "avoid": avoid, "slot_bytes": slot_bytes, "slots": slots})
        fds = list(self._last_fds)
        try:
            if not rep.get("ok") or not fds:
                raise RuntimeError(rep.get("error", "no helper GPU available"))
            self._mailbox = engine.paths_attach(fds, rep["slot_bytes"], rep["slots"])
        finally:
            for fd in fds:
                os.close(fd)
        return len(fds)

    def request_pull(self, engine, instance: str, rank: int, timeout_s: float = 5.0) -> int:
        """Tell the owner's helpers to serve the NEXT wake of this engine (call right before ``Engine.wake``)."""
        store = engine.host_store_share()
        try:
            rep, _ = self._rpc({"op": "pull", "instance": instance, "rank": rank, "generation": engine.pull_next_generation(), "timeout_s": timeout_s},
                               send_fds=[self._mailbox, store])
        finally:
            os.close(store)
        return int(rep.get("helpers", 0)) if rep.get("ok") else 0

    def release(self, instance: str, rank: Optional[int] = None) -> int:
        rep, _ = self._rpc({"op": "release", "instance": instance, "rank": rank})
        return int(rep.get("released", 0))

    def stats(self) -> dict:
        return self._rpc({"op": "stats"})[0]
