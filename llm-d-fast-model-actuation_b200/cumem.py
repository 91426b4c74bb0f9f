"""Drop-in for ``vllm.device_allocator.cumem.CuMemAllocator`` (SURVEY.md §8b, surface B2).

Same class name, singleton accessor, method names, argument meaning and error behaviour as the
reference's allocator shim, so vLLM's ``Worker.sleep`` / ``Worker.wake_up`` / ``load_model``
(vllm:v1/worker/gpu_worker.py:157-209,335-342) run unchanged on top of the H100 engine:

    reference (vllm:device_allocator/cumem.py)            this module
    ------------------------------------------            -----------------------------------
    CuMemAllocator.get_instance()          :118-128       CuMemAllocator.get_instance()
    .use_memory_pool(tag)                  :251-308       .use_memory_pool(tag)
    .sleep(offload_tags)                   :177-225       .sleep(offload_tags)   -> fma_sleep
    .wake_up(tags)                         :227-249       .wake_up(tags)         -> fma_wake
    .get_current_usage()                   :310-318       .get_current_usage()   -> fma_current_usage
    .pointer_to_data                       :131           .pointer_to_data (read-only view of the C table)
    my_malloc / my_free in cumem_allocator.abi3.so        my_malloc / my_free in libfma_b200.so

Differences that are the point of the rewrite: the registry lives in C (no Python callbacks from
inside the allocator), the host backup is ONE pre-pinned NUMA-local arena instead of a
``torch.empty(pin_memory=True)`` per segment inside the sleep loop, and copies are asynchronous
over several copy-engine streams overlapped with cuMemCreate/cuMemMap.

``install_into_vllm()`` swaps the class into an imported vLLM so the unmodified reference launcher
(inference_server/launcher/launcher.py:799-837) serves /sleep and /wake_up through this engine.
"""
from __future__ import annotations

import atexit
import dataclasses
import gc
import json
import logging
import os
import socket
import threading
import time
from contextlib import contextmanager
from typing import Any

from . import _lib as L
from .engine import Engine, EngineConfig

logger = logging.getLogger("vllm.fma_b200.cumem")  # child of vLLM's configured logger, so INFO lines reach the instance log

# py_device, py_alignedSize, py_d_mem, py_p_memHandle  (cumem.py:47-48); the 4th slot carries the
# engine's segment sequence number instead of a heap pointer to a CUmemGenericAllocationHandle.
HandleType = tuple[int, int, int, int]


@dataclasses.dataclass
class AllocationData:
    handle: HandleType
    tag: str
    cpu_backup_tensor: Any = None  # always None: the backup lives in the engine's packed host store
    mapped: bool = True
    has_backup: bool = False


def _tier_from_env() -> int:
    return {"host": L.FMA_TIER_HOST, "peer": L.FMA_TIER_PEER, "local": L.FMA_TIER_LOCAL, "file": L.FMA_TIER_FILE}[
        os.environ.get("FMA_TIER", "host").lower()]


def _file_tier_path() -> str:
    """FMA_TIER=file: this rank's image file, ``<FMA_FILE_DIR>/<instance id>-r<rank>.fmaimg`` (removed when the process exits)."""
    d = os.environ.get("FMA_FILE_DIR")
    if not d:
        raise L.FmaError(L.FMA_EINVAL, "FMA_TIER=file needs FMA_FILE_DIR=<directory on a local disk>")
    return os.path.join(d, f"{_instance_id()}-r{_rank()}.fmaimg")


def _remove_file(path: str) -> None:
    try:
        os.unlink(path)
    except OSError:
        pass


class CuMemAllocator:
    """Singleton per process, exactly like the reference (the C side keeps the current engine in a
    process global because torch's pluggable-allocator signature has no user pointer)."""

    instance: "CuMemAllocator | None" = None
    default_tag: str = "default"

    @staticmethod
    def get_instance() -> "CuMemAllocator":
        if CuMemAllocator.instance is None:
            CuMemAllocator.instance = CuMemAllocator()
        return CuMemAllocator.instance

    def __init__(self, device: int | None = None, config: EngineConfig | None = None, engine: Any = None):
        """``engine`` may be injected (tests of the host logic); normally the allocator creates its own."""
        if engine is not None:
            self.device = 0 if device is None else device
            self.engine = engine
        else:
            import torch

            if not torch.cuda.is_available():
                raise L.FmaError(L.FMA_ENODRIVER, "CuMemAllocator needs a CUDA device; there is no CPU fallback")
            self.device = torch.cuda.current_device() if device is None else device
            self.engine = Engine(self.device, config)
        self.engine.make_current()
        self.current_tag: str = CuMemAllocator.default_tag
        self.allocator_and_pools: dict[str, Any] = {}
        self._reserve_thread: threading.Thread | None = None
        self._file_path: str | None = None     # FMA_TIER=file: this rank's image file, once named
        self._file_deposited = False           # FMA_DEPOSIT_FILE_IMAGE=1: the node agent holds a standing deposit of that file
        # MULTI-PATH wake across processes (FMA_REMOTE_PATHS=k): the node agent's helper GPUs pull for this instance; that needs the
        # host store as a memfd the agent can map, so the switch is thrown before the store is first reserved
        self._remote = None
        # FMA_NODE_SLEEPER_DRAM_GIB (with a node agent): the agent's host-memory budget may demote / promote this rank's image
        self._ctl_lock = threading.Lock()          # this rank's sleep and wake against the agent's commands
        self._channel: "_SleeperChannel | None" = None
        self._slept_at = 0.0
        self._report_lock = threading.Lock()       # one report at a time, each read and sent together: the agent sees them in order
        self._waiting = False                      # a waiter thread reports the end of the write-behind job (under _report_lock)
        if int(os.environ.get("FMA_REMOTE_PATHS", "0") or 0) > 0 and os.environ.get("FMA_NODE_AGENT_SOCK"):
            os.environ["FMA_HOST_STORE_SHM"] = "1"

    # ---- registry view -----------------------------------------------------------------
    @property
    def pointer_to_data(self) -> dict[int, AllocationData]:
        out: dict[int, AllocationData] = {}
        for s in self.engine.segments():
            out[s.va] = AllocationData((self.device, s.bytes, s.va, s.seq), s.tag, None, s.mapped, s.has_backup)
        return out

    def get_current_usage(self) -> int:
        return self.engine.current_usage()

    # ---- hot path ----------------------------------------------------------------------
    def sleep(self, offload_tags: tuple[str, ...] | str | None = None) -> None:
        if self._channel is None and os.environ.get("FMA_NODE_AGENT_SOCK") and os.environ.get("FMA_NODE_SLEEPER_DRAM_GIB"):
            try:
                self._channel = _SleeperChannel(self)
            except OSError as e:
                logger.warning("fma_b200: cannot reach the node agent's sleeper budget (%s): this rank is not demoted", e)
        with self._ctl_lock:
            self._sleep(offload_tags)
            self._slept_at = time.time()
        self._report()

    def _sleep(self, offload_tags: tuple[str, ...] | str | None) -> None:
        if offload_tags is None:
            offload_tags = (CuMemAllocator.default_tag,)
        elif isinstance(offload_tags, str):
            offload_tags = (offload_tags,)
        assert isinstance(offload_tags, tuple)
        self._join_reserve()
        self._check_writeback()
        import torch

        tier = _tier_from_env()
        owner = None
        if tier == L.FMA_TIER_PEER:
            nbytes = sum(s.bytes for s in self.engine.segments() if s.tag in offload_tags)
            if os.environ.get("FMA_NODE_AGENT_SOCK"):
                # Under the launcher an instance sees only its own GPUs (launcher.py:171-187): the node agent owns the parking
                # buffer (parking.py), this rank attaches to it and deposits the image descriptor afterwards, so the parked
                # weights outlive this process.
                from .parking import ParkingClient

                owner = ParkingClient()
                try:
                    owner.park(self.engine, _instance_id(), _rank(), nbytes, avoid=_own_gpu_indices())
                except (RuntimeError, OSError, L.FmaError) as e:
                    # no peer has room (or the agent is gone): the sleep itself must not fail for that — the host tier always works
                    logger.warning("fma_b200: cannot park %.2f GiB on a peer GPU (%s): sleeping to the host tier instead", nbytes / 1024**3, e)
                    owner, tier = None, L.FMA_TIER_HOST
            else:
                # parking GPU for the NVLink tier: FMA_PEER_DEVICE (index among the devices this process sees)
                peer = int(os.environ.get("FMA_PEER_DEVICE", "-1"))
                if peer < 0:
                    raise L.FmaError(L.FMA_EINVAL, "FMA_TIER=peer needs FMA_NODE_AGENT_SOCK (node-level owner) or FMA_PEER_DEVICE=<visible device index of the parking GPU>")
                try:
                    self.engine.peer_reserve(peer, nbytes)
                except L.FmaError as e:
                    if e.code != L.FMA_ENOMEM:
                        raise
                    logger.warning("fma_b200: GPU %d cannot take %.2f GiB right now (%s): sleeping to the host tier instead", peer, nbytes / 1024**3, e.message)
                    tier = L.FMA_TIER_HOST
        elif tier == L.FMA_TIER_FILE and self._file_path is None:
            # (also after adopting a kept file: that file is the node agent's and is only read, never written)
            self._file_path = _file_tier_path()
            self.engine.file_store(self._file_path)
            atexit.register(self._remove_own_file)
            atexit.register(self._finish_writeback)   # (runs first)
        deposit_host = (tier == L.FMA_TIER_HOST and os.environ.get("FMA_DEPOSIT_HOST_IMAGE") == "1" and os.environ.get("FMA_NODE_AGENT_SOCK")
                        and os.environ.get("FMA_HOST_STORE_SHM") == "1")
        if deposit_host:
            # a resident share lives in this process's HBM and cannot be handed over: the deposit wins
            if int(os.environ.get("FMA_RESIDENT_MIB", "0") or 0) > 0:
                logger.warning("fma_b200: FMA_DEPOSIT_HOST_IMAGE=1 takes precedence over FMA_RESIDENT_MIB: the whole image goes to the host store")
            self.engine.set_option("resident_bytes", 0)
        try:
            # a deposited image (file, or host memfd the node agent may spill to a kept file) is adopted by another process, whose
            # wake checks it against these digests
            deposits = deposit_host or (tier == L.FMA_TIER_FILE and _deposits_file())
            # FMA_FILE_WRITE_BEHIND=1: into the host store pinned after load (or kept), the file written behind the sleep
            behind = tier == L.FMA_TIER_FILE and _write_behind()
            self.engine.sleep(offload_tags, tier=tier, flags=(L.FMA_FLAG_VERIFY if deposits else 0) | (L.FMA_FLAG_WRITE_BEHIND if behind else 0))
        except L.FmaError as e:
            # the file tier refused before releasing anything (no room on the disk, no HBM for its staging ring): the host tier works
            if tier != L.FMA_TIER_FILE or e.code not in (L.FMA_EIO, L.FMA_ENOMEM) or self.engine.is_sleeping():
                raise
            logger.warning("fma_b200: cannot sleep to %s (%s): sleeping to the host tier instead", self._file_path, e.message)
            self.engine.sleep(offload_tags, tier=L.FMA_TIER_HOST)
        if owner is not None and self.engine.stats()["sleep_bytes_offloaded"]:
            owner.deposit(self.engine, _instance_id(), _rank(), tier)
        elif deposit_host and self.engine.stats()["sleep_bytes_offloaded"]:
            # HOST tier, opt-in: hand the memfd behind the store to the node agent so the image outlives this process.  The exported
            # store is read-only from then on: this engine's NEXT sleep takes (and pins) a fresh private store — right for an instance
            # that is about to be deleted, wrong for one that sleeps and wakes all day, hence not the default.
            from .parking import ParkingClient

            ParkingClient().deposit_host(self.engine, _instance_id(), _rank())
        elif _deposits_file() and ((self.engine.stats()["tier"] == L.FMA_TIER_FILE and self.engine.stats()["sleep_bytes_copied"])
                                   or self._writing_behind()):
            self._deposit_file()
        st = self.engine.stats()
        total = st["sleep_bytes_offloaded"] + st["sleep_bytes_discarded"]
        # same INFO line the reference emits (cumem.py:215-222; parsed by llm-d-benchmark), plus GB/s
        logger.info(
            "CuMemAllocator: sleep freed %.2f GiB memory in total, of which %.2f GiB is backed up in CPU and the "
            "rest %.2f GiB is discarded directly.", total / 1024**3, st["sleep_bytes_offloaded"] / 1024**3,
            st["sleep_bytes_discarded"] / 1024**3)
        if st["sleep_copy_seconds"] > 0:
            logger.info("fma_b200: sleep %.3f s, D2H %.1f GB/s", st["sleep_seconds"],
                        st["sleep_bytes_offloaded"] / st["sleep_copy_seconds"] / 1e9)
        if st.get("image_packed"):
            logger.info("fma_b200: packed image: %.2f GiB stored for %.2f GiB of weights (%.3f)", st["image_store_bytes"] / 1024**3,
                        st["sleep_bytes_offloaded"] / 1024**3, st["image_store_bytes"] / max(st["sleep_bytes_offloaded"], 1))
        gc.collect()
        torch.cuda.empty_cache()

    def wake_up(self, tags: list[str] | None = None) -> None:
        with self._ctl_lock:
            self._wake_up(tags)
        self._report()

    def _wake_up(self, tags: list[str] | None) -> None:
        moves_an_image = tags is None or any(t != "kv_cache" for t in tags)   # the kv cache is discarded on sleep: waking it copies nothing
        if self._remote is not None and moves_an_image and self.engine.is_sleeping() and _tier_from_env() == L.FMA_TIER_HOST:
            try:    # the owner's helpers serve the wake that follows; if the request fails, the instance's own link does it all
                self._remote.request_pull(self.engine, _instance_id(), _rank())
            except Exception as e:      # noqa: BLE001
                logger.warning("fma_b200: pull request to the node agent failed (%s): waking over the own link only", e)
        if self._file_deposited and (tags is None or "weights" in tags):
            # the weights are about to serve, and may change: the file is no image to keep once this process exits
            self._file_deposited = False
            try:
                from .parking import ParkingClient

                ParkingClient().withdraw_file(_instance_id(), _rank())
            except Exception as e:      # noqa: BLE001
                logger.warning("fma_b200: cannot withdraw the image file from the node agent (%s)", e)
        self._check_writeback()
        self.engine.wake(tags)
        st = self.engine.stats()
        if st["wake_copy_seconds"] > 0:
            logger.info("fma_b200: wake %.3f s, H2D %.1f GB/s", st["wake_seconds"],
                        st["wake_bytes_restored"] / st["wake_copy_seconds"] / 1e9)
        if _write_behind() and not st["host_store_bytes"] and not self.engine.is_sleeping():
            # the write-behind committed and released the store: the next sleep needs one again, pinned off its critical path
            self._join_reserve()
            self._start_reserve()

    def move_image(self, tier: str) -> None:
        """Move this rank's sleeping image without waking it.  ``"file"`` demotes it to ``<FMA_FILE_DIR>/<instance id>-r<rank>.fmaimg``
        (the file tier's name, removed when the process exits) and then releases the host store; ``"host"`` promotes it back to
        host DRAM ahead of a wake and leaves the file to the exit hook."""
        self._join_reserve()
        if tier == "file":
            self._name_own_file()
            self.engine.move_image(L.FMA_TIER_FILE)
            self.engine.host_release()
        elif tier == "host":
            self.engine.move_image(L.FMA_TIER_HOST)
        else:
            raise L.FmaError(L.FMA_EINVAL, f"move_image: tier {tier!r} is not 'host' or 'file'")
        logger.info("fma_b200: sleeping image moved to the %s tier (%.2f GiB)", tier, self.engine.stats()["image_store_bytes"] / 1024**3)
        self._report()

    def _name_own_file(self) -> None:
        if self._file_path is None:
            self._file_path = _file_tier_path()
            self.engine.file_store(self._file_path)
            atexit.register(self._remove_own_file)

    # ---- the node agent's host-memory budget (FMA_NODE_SLEEPER_DRAM_GIB) --------------------------------------------------
    def _agent_command(self, op: str) -> None:
        """``demote``: the image goes to this rank's file behind the call (``move_image(file, behind=True)``), and the state is
        reported again when the write commits, is cancelled or fails.  ``promote``: back to host DRAM (synchronous).  A command
        that finds the rank awake is a no-op.  The lock only orders the command against a sleep or wake in progress; the engine
        call runs outside it, so a wake that comes meanwhile pre-empts a demotion (or waits for a promotion) in the engine."""
        with self._ctl_lock:
            asleep = self.engine.is_sleeping()
        if not asleep or op not in ("demote", "promote"):
            self._report(answer=op)
            return
        try:
            if op == "demote":
                self._name_own_file()
                self.engine.move_image(L.FMA_TIER_FILE, behind=True)
            else:
                self.engine.move_image(L.FMA_TIER_HOST)
        except L.FmaError as e:
            logger.info("fma_b200: the node agent's %s of this rank's image was refused: %s", op, e)
            self._report(answer=op, error=e)
            return
        self._report(answer=op)

    def _await_writeback(self) -> None:
        """A write-behind job is writing (a write-behind sleep's, or a demotion's): report again once it has committed, been
        cancelled or failed, so the agent's books never keep a rank demoting."""
        while True:
            failed = None
            try:
                self.engine.writeback(None)     # (waits without pre-empting)
            except L.FmaError as e:
                self._warn_writeback(e)
                failed = "demote"
            if not self._report(failed=failed, waiter=True):   # (a job started meanwhile: wait for that one too)
                return

    def _report(self, answer: str | None = None, error: L.FmaError | None = None, failed: str | None = None, waiter: bool = False) -> bool:
        """This rank's sleeper_state for the agent's budget: host_bytes is the pinned host store, a write-behind reserve held
        while awake included.  ``failed``: a write-behind write failed (the agent does not demote this rank again until it sleeps
        again).  While a job writes, a waiter reports its end."""
        ch = self._channel
        if ch is None:
            if waiter:
                self._waiting = False
            return False
        with self._report_lock:
            return self._send_report(ch, answer, error, failed, waiter)

    def _send_report(self, ch: "_SleeperChannel", answer, error, failed, waiter: bool) -> bool:
        try:
            demoting = self.engine.writeback(0.0)[0] == 1
        except L.FmaError as e:
            self._warn_writeback(e)
            demoting, failed = False, "demote"
        if waiter:
            self._waiting = demoting
        elif demoting and not self._waiting:
            self._waiting = True
            threading.Thread(target=self._await_writeback, name="fma-writeback-waiter", daemon=True).start()
        st = self.engine.stats()
        msg = {"op": "sleeper_state", "instance": _instance_id(), "rank": _rank(), "asleep": self.engine.is_sleeping(),
               "tier": _TIER_NAMES.get(st["tier"], str(st["tier"])), "host_bytes": st["host_store_bytes"], "image_bytes": st["image_store_bytes"],
               "slept_at": self._slept_at, "demoting": demoting, "file_dir": os.environ.get("FMA_FILE_DIR", ""),
               "shared": os.environ.get("FMA_DEPOSIT_HOST_IMAGE") == "1"}
        if answer:
            msg["answer"] = answer
        if error is not None:
            msg["error"], msg["code"] = error.message[:200], error.code
        if failed:
            msg["failed"] = failed
        try:
            ch.send(msg)
        except OSError as e:
            logger.warning("fma_b200: the node agent's sleeper budget is gone (%s)", e)
            self._channel = None
        return demoting

    def verify_image(self) -> bool:
        """Check this rank's sleeping image where it lies (host DRAM, disk or parking HBM) against the digests recorded when it
        slept with FMA_FLAG_VERIFY, without waking it: False when a segment's stored bytes do not match, so the caller can cold-start
        instead of waking wrong weights.  Raises FmaError if the image carries no digests or nothing is asleep."""
        bad = self.engine.verify_image()
        if bad:
            logger.warning("fma_b200: sleeping image fails verification in %d segment(s): %s", len(bad), bad[:8])
        return not bad

    def prefetch_image(self, mib: int) -> int:
        """Copy up to ``mib`` MiB of this rank's sleeping image (its tail, in stored bytes) from host DRAM or disk into its own GPU's
        HBM ahead of a wake, so that the wake moves that much less over the link; 0 gives the HBM back.  A no-op while awake.
        Returns the bytes prefetched."""
        if not self.engine.is_sleeping():
            return 0
        self._join_reserve()
        self.engine.prefetch_image(int(mib) << 20)
        n = self.engine.stats()["prefetched_bytes"]
        logger.info("fma_b200: %.2f GiB of the sleeping image prefetched into HBM", n / 1024**3)
        return n

    # ---- pool --------------------------------------------------------------------------
    @contextmanager
    def use_memory_pool(self, tag: str | None = None):
        import torch

        if tag is None:
            tag = CuMemAllocator.default_tag
        assert isinstance(tag, str)
        conf = os.environ.get("PYTORCH_CUDA_ALLOC_CONF", "")
        expandable_was_enabled = "expandable_segments:True" in conf  # incompatible with the pool (cumem.py:266-274)
        if expandable_was_enabled:
            torch.cuda.memory._set_allocator_settings("expandable_segments:False")
        old_tag = self.current_tag
        self.current_tag = tag
        self.engine.make_current()
        self.engine.set_current_tag(tag)
        try:
            new_alloc = torch.cuda.memory.CUDAPluggableAllocator(L.lib_path(), "my_malloc", "my_free")
            mem_pool = torch.cuda.memory.MemPool(new_alloc._allocator)
            data = (mem_pool, new_alloc)
            with torch.cuda.memory.use_mem_pool(mem_pool):
                self.allocator_and_pools[tag] = data  # keep alive (pytorch#146431, cumem.py:285-289)
                yield
                # release segments that ended up empty (e.g. load-time temporaries), cumem.py:299-303
                for allocation in mem_pool.snapshot():
                    if allocation["allocated_size"] == 0:
                        try:
                            self.engine.free(allocation["address"])
                        except L.FmaError:
                            pass
        finally:
            self.current_tag = old_tag
            self.engine.set_current_tag(old_tag)
            if expandable_was_enabled:
                torch.cuda.memory._set_allocator_settings("expandable_segments:True")
        if tag == "weights":
            # one line for tooling (scripts/e2e_launcher_vllm.py validates the synthetic tables of workloads.py against it, SURVEY §8d)
            segs = [s for s in self.engine.segments() if s.tag == "weights"]
            hist: dict[int, int] = {}
            for sg in segs:
                hist[sg.bytes >> 20] = hist.get(sg.bytes >> 20, 0) + 1
            logger.info("fma_b200: weights pool closed: %s", json.dumps({"segments": len(segs), "bytes": sum(sg.bytes for sg in segs),
                                                                          "first_mib": [sg.bytes >> 20 for sg in segs[:6]],
                                                                          "mib_histogram": {str(k): v for k, v in sorted(hist.items())}}))
        adopted = False
        if tag == "weights" and os.environ.get("FMA_ADOPT_PARKED") == "1" and os.environ.get("FMA_NODE_AGENT_SOCK"):
            adopted = self._adopt_parked_image()
        if tag == "weights" and not adopted and os.environ.get("FMA_ADOPT_FILE") == "1" and os.environ.get("FMA_NODE_AGENT_SOCK"):
            self._adopt_kept_file()
        if tag == "weights" and self._remote is None and int(os.environ.get("FMA_REMOTE_PATHS", "0") or 0) > 0 \
                and os.environ.get("FMA_NODE_AGENT_SOCK") and _tier_from_env() == L.FMA_TIER_HOST:
            try:
                from .parking import ParkingClient

                cli = ParkingClient()
                n = cli.attach_remote_paths(self.engine, _instance_id(), _rank(), int(os.environ["FMA_REMOTE_PATHS"]), avoid=_own_gpu_indices())
                self._remote = cli
                logger.info("fma_b200: %d remote wake path(s) through the node agent's helper GPUs", n)
            except Exception as e:      # noqa: BLE001
                logger.warning("fma_b200: no remote wake paths (%s): host-tier wakes use the own link only", e)
        if tag == "weights" and ((os.environ.get("FMA_PREPIN", "1") != "0" and _tier_from_env() == L.FMA_TIER_HOST) or _write_behind()):
            self._start_reserve()

    def _adopt_parked_image(self) -> bool:
        """Warm start (SURVEY §8f-1): an earlier instance with this instance ID parked its weights with the node agent and died
        (or was deleted) asleep — the controller would cold-start here (inference-server.go:416-448).  The weights pool has just
        been filled by the loader (``--load-format dummy`` is enough: contents are about to be replaced); if the owner holds an image
        for (instance, rank) whose segment sequence matches, adopt it and wake: the weights come back over NVLink, digests
        verified.  Anything else (no image, another model) leaves the loaded weights as they are."""
        import time

        from .parking import ParkingClient

        t0 = time.perf_counter()
        try:
            cli = ParkingClient()
            if not cli.adopt(self.engine, _instance_id(), _rank(), tags=("weights",)) and \
                    not cli.adopt_host(self.engine, _instance_id(), _rank(), tags=("weights",)):
                logger.info("fma_b200: no parked image for instance %s rank %d: keeping the loaded weights", _instance_id(), _rank())
                return False
            self.engine.wake(["weights"], flags=L.FMA_FLAG_VERIFY)
            st = self.engine.stats()
            logger.info("fma_b200: adopted the parked image of instance %s rank %d: %.2f GiB restored from %s in %.3f s (digests verified)",
                        _instance_id(), _rank(), st["wake_bytes_restored"] / 1024**3, {L.FMA_TIER_HOST: "the host store", L.FMA_TIER_PEER: "peer HBM"}.get(st["tier"], f"tier {st['tier']}"),
                        time.perf_counter() - t0)
            return True
        except L.FmaError as e:
            if self.engine.is_sleeping():
                raise                                   # half way: do not serve from unmapped weights
            logger.warning("fma_b200: parked image not adopted (%s): keeping the loaded weights", e)
            return False

    def _adopt_kept_file(self) -> bool:
        """Warm start from disk (FMA_ADOPT_FILE=1): an earlier instance with this instance ID slept to the file tier, deposited its
        image file with the node agent and was deleted; the agent kept the file.  The weights pool has just been filled by the
        loader (``--load-format dummy`` is enough): adopt the kept file and wake with its digests verified.  A miss or a refusal
        before the wake (another segment sequence, an unreadable file) keeps the loaded weights; weights that fail their digests
        raise, and the agent drops the file.  The kept file is only read: this rank's own file-tier sleeps write its own path."""
        import time

        from .parking import ParkingClient

        t0 = time.perf_counter()
        iid, rank = _instance_id(), _rank()
        try:
            cli = ParkingClient()
            path = cli.lookup_file(iid, rank)
        except (RuntimeError, OSError) as e:
            logger.warning("fma_b200: cannot ask the node agent for a kept image file (%s): keeping the loaded weights", e)
            return False
        if path is None:
            logger.info("fma_b200: no kept image file for instance %s rank %d: keeping the loaded weights", iid, rank)
            return False
        drop = False
        try:
            try:
                self.engine.image_adopt_file(path, ("weights",))
            except L.FmaError as e:
                if self.engine.is_sleeping():
                    raise
                logger.warning("fma_b200: kept image file %s not adopted (%s): keeping the loaded weights", path, e)
                return False
            try:
                self.engine.wake(["weights"], flags=L.FMA_FLAG_VERIFY)
            except L.FmaError as e:
                drop = e.code == L.FMA_EINTEGRITY       # never serve weights that failed their digests; the file goes
                raise
            st = self.engine.stats()
            logger.info("fma_b200: adopted the kept image file of instance %s rank %d: %.2f GiB restored from %s in %.3f s (digests verified)",
                        iid, rank, st["wake_bytes_restored"] / 1024**3, path, time.perf_counter() - t0)
            return True
        finally:
            try:
                cli.lookup_done(iid, rank, drop=drop)
            except (RuntimeError, OSError) as e:
                logger.warning("fma_b200: cannot end the lease on %s with the node agent (%s)", path, e)

    def _deposit_file(self) -> None:
        """FMA_DEPOSIT_FILE_IMAGE=1: the file this sleep wrote goes to the node agent, which keeps it if the process exits asleep.
        If the agent cannot take it, the file is removed at exit as usual; the sleep itself never fails for that."""
        from .parking import ParkingClient

        try:
            ParkingClient().deposit_file(_instance_id(), _rank(), self._file_path)
            self._file_deposited = True
        except (RuntimeError, OSError) as e:
            logger.warning("fma_b200: cannot deposit %s with the node agent (%s): it is removed when this process exits", self._file_path, e)

    def _writing_behind(self) -> bool:
        """A write-behind job of the last sleep is writing this rank's file, or has moved the image there already."""
        if not _write_behind():
            return False
        try:
            return self.engine.writeback(0.0)[0] == 1 or self.engine.stats()["tier"] == L.FMA_TIER_FILE
        except L.FmaError as e:
            self._warn_writeback(e)
            return False

    def _check_writeback(self) -> None:
        """A failed write-behind is reported once: the image then sleeps on in host DRAM."""
        if not _write_behind():
            return
        try:
            self.engine.writeback(0.0)
        except L.FmaError as e:
            self._warn_writeback(e)

    def _warn_writeback(self, e: L.FmaError) -> None:
        logger.warning("fma_b200: the sleeping image could not be written to %s (%s): it stays in host DRAM (%.2f GiB pinned)",
                       self._file_path, e.message, self.engine.stats()["host_store_bytes"] / 1024**3)

    def _finish_writeback(self) -> None:
        """At exit, before the engine goes: a deposited file a write-behind job still writes is completed (destroying the engine
        would cancel the job, and the node agent would find an empty file)."""
        if self._file_deposited:
            try:
                self.engine.writeback(None)
            except L.FmaError as e:
                self._warn_writeback(e)

    def _remove_own_file(self) -> None:
        """At exit: this rank's image file goes, unless a deposit with the node agent stands (the agent owns the file then)."""
        if self._file_path is not None and not self._file_deposited:
            _remove_file(self._file_path)

    # ---- pre-pinning off the critical path -----------------------------------------------
    def _start_reserve(self) -> None:
        """Pin the host store for the weights as soon as they are loaded, in the background, so the
        first /sleep does not pay for it (the reference pins inside its sleep loop, cumem.py:204-209)."""
        nbytes = sum(s.bytes for s in self.engine.segments() if s.tag == "weights")
        if not nbytes:
            return

        def run():
            try:
                self.engine.host_reserve(nbytes)
            except L.FmaError as e:  # sleep will retry and report
                logger.warning("background host_reserve failed: %s", e)
            self._report()   # (the node agent's budget counts the pinned store)

        self._reserve_thread = threading.Thread(target=run, name="fma-prepin", daemon=True)
        self._reserve_thread.start()

    def _join_reserve(self) -> None:
        if self._reserve_thread is not None:
            self._reserve_thread.join()
            self._reserve_thread = None


def _instance_id() -> str:
    """The controller's instance ID (``"I" + base64url(sha256(...)) + "i"``, inference-server.go:801-829): the node agent passes it to
    its children as FMA_INSTANCE_ID; a bare process falls back to its pid."""
    return os.environ.get("FMA_INSTANCE_ID") or f"pid{os.getpid()}"


_TIER_NAMES = {L.FMA_TIER_HOST: "host", L.FMA_TIER_PEER: "peer", L.FMA_TIER_LOCAL: "local", L.FMA_TIER_FILE: "file"}


class _SleeperChannel:
    """This rank's persistent connection to the node agent's host-memory budget (parking.py ``sleeper`` op): sleeper_state reports
    go up, demote / promote commands come down and are run by a daemon thread, which owns the connection's reading end."""

    def __init__(self, alloc: CuMemAllocator):
        self._alloc = alloc
        self._send_lock = threading.Lock()
        self._sock = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self._sock.connect(os.environ["FMA_NODE_AGENT_SOCK"])
        self._sock.sendall((json.dumps({"op": "sleeper", "instance": _instance_id(), "rank": _rank()}) + "\n").encode())
        self._rfile = self._sock.makefile("rb")
        rep = json.loads(self._rfile.readline() or b"{}")
        if not rep.get("ok"):
            self._sock.close()
            raise OSError(rep.get("error", "the node agent keeps no sleeper budget"))
        threading.Thread(target=self._run, name="fma-sleeper-channel", daemon=True).start()

    def send(self, msg: dict) -> None:
        with self._send_lock:
            self._sock.sendall((json.dumps(msg) + "\n").encode())

    def _run(self) -> None:
        try:
            for line in self._rfile:
                self._alloc._agent_command(json.loads(line).get("op", ""))
        except (OSError, ValueError) as e:
            logger.warning("fma_b200: the node agent's sleeper channel closed (%s)", e)


def _deposits_file() -> bool:
    """FMA_DEPOSIT_FILE_IMAGE=1 (with FMA_TIER=file and a node agent): file-tier images are deposited with the agent."""
    return os.environ.get("FMA_DEPOSIT_FILE_IMAGE") == "1" and bool(os.environ.get("FMA_NODE_AGENT_SOCK")) and _tier_from_env() == L.FMA_TIER_FILE


def _write_behind() -> bool:
    """FMA_FILE_WRITE_BEHIND=1 (with FMA_TIER=file): sleeps return once the image is in the host store, pinned in the background after
    load and after a wake whose store was released; the file is written behind them (FMA_FLAG_WRITE_BEHIND)."""
    return os.environ.get("FMA_FILE_WRITE_BEHIND") == "1" and _tier_from_env() == L.FMA_TIER_FILE


def _rank() -> int:
    return int(os.environ.get("RANK", os.environ.get("LOCAL_RANK", "0")) or 0)


def _own_gpu_indices() -> list[int]:
    """Node-level GPU indices this instance runs on (never park a model on its own GPU): FMA_NODE_GPU_INDICES, set by the node
    agent next to CUDA_VISIBLE_DEVICES."""
    v = os.environ.get("FMA_NODE_GPU_INDICES", "")
    return [int(x) for x in v.split(",") if x.strip().isdigit()]


def install_into_vllm() -> None:
    """Replace vLLM's allocator class with this one (call before the engine core starts workers)."""
    import vllm.device_allocator.cumem as ref

    ref.CuMemAllocator = CuMemAllocator  # type: ignore[misc]
    ref.cumem_available = True


__all__ = ["CuMemAllocator", "AllocationData", "HandleType", "install_into_vllm"]
