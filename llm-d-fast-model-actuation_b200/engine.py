"""Object wrapper over the C-ABI engine handle (thin; all work happens in libfma_b200.so)."""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Iterable, Sequence

from . import _lib as L
from ._lib import FmaError, check


@dataclasses.dataclass
class EngineConfig:
    mode: int = L.FMA_MODE_AUTO
    kernel: int = L.FMA_KERNEL_TMA
    copy_streams: int = 0
    chunk_bytes: int = 0
    ring_slots: int = 0
    map_threads: int = 0
    numa_bind: int = -1
    pack: int = 0            # 1 = PACKED host image (lossless bf16 page code, csrc/fma_codec.h)

    def to_c(self) -> L.fma_config_t:
        c = L.fma_config_t()
        c.abi_version = L.FMA_ABI_VERSION
        c.mode, c.kernel, c.copy_streams = self.mode, self.kernel, self.copy_streams
        c.chunk_bytes, c.ring_slots, c.map_threads, c.numa_bind = (
            self.chunk_bytes, self.ring_slots, self.map_threads, self.numa_bind)
        c.pack = self.pack
        return c


@dataclasses.dataclass
class SegmentInfo:
    index: int
    va: int
    bytes: int
    requested_bytes: int
    packed_offset: int | None
    seq: int
    tag: str
    mapped: bool
    has_backup: bool
    tier: int


class Engine:
    """One engine per GPU (rank).  Mirrors the role of the per-process ``CuMemAllocator`` singleton
    (vllm:device_allocator/cumem.py:92-138) but holds no Python-side registry: the segment table
    lives in C so sleep/wake never need the GIL."""

    def __init__(self, device: int = 0, config: EngineConfig | None = None):
        self._lib = L.load_library()
        self._h = C.c_void_p()
        cfg = (config or EngineConfig()).to_c()
        check(self._lib.fma_engine_create(device, C.byref(cfg), C.byref(self._h)))
        self.device = device
        self._tag_ids: dict[str, int] = {"default": 0}

    # -- lifecycle ------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.fma_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def make_current(self) -> None:
        check(self._lib.fma_set_current(self._h))

    # -- tags -----------------------------------------------------------------------------
    def tag_id(self, name: str) -> int:
        if name not in self._tag_ids:
            self._tag_ids[name] = check(self._lib.fma_tag_intern(self._h, name.encode()))
        return self._tag_ids[name]

    def tag_mask(self, names: Iterable[str] | None) -> int:
        if names is None:
            return 0
        m = 0
        for n in names:
            m |= 1 << self.tag_id(n)
        return m

    def set_current_tag(self, name: str) -> None:
        check(self._lib.fma_set_current_tag(self._h, self.tag_id(name)))

    def _tag_name(self, tag: int) -> str:
        for k, v in self._tag_ids.items():
            if v == tag:
                return k
        buf = C.create_string_buffer(128)
        check(self._lib.fma_tag_name(self._h, tag, buf, len(buf)))
        name = buf.value.decode()
        self._tag_ids[name] = tag
        return name

    # -- allocation -----------------------------------------------------------------------
    def alloc(self, nbytes: int, tag: str = "default") -> int:
        p = C.c_void_p()
        check(self._lib.fma_alloc(self._h, nbytes, self.tag_id(tag), C.byref(p)))
        return int(p.value)

    def free(self, ptr: int) -> None:
        check(self._lib.fma_free(self._h, C.c_void_p(ptr)))

    def segment_count(self) -> int:
        return check(self._lib.fma_segment_count(self._h))

    def segment(self, index: int) -> SegmentInfo:
        s = L.fma_segment_info_t()
        check(self._lib.fma_segment_info(self._h, index, C.byref(s)))
        return SegmentInfo(index, s.va, s.bytes, s.requested_bytes,
                           None if s.packed_offset == L.NO_OFFSET else s.packed_offset, s.seq, self._tag_name(s.tag),
                           bool(s.mapped), bool(s.has_backup), s.tier)

    def segments(self) -> list[SegmentInfo]:
        return [self.segment(i) for i in range(self.segment_count())]

    def find(self, ptr: int) -> int:
        return check(self._lib.fma_segment_find(self._h, C.c_void_p(ptr)))

    def current_usage(self) -> int:
        return int(self._lib.fma_current_usage(self._h))

    # -- hot path -------------------------------------------------------------------------
    def sleep(self, offload_tags: Sequence[str] = ("default",), tier: int = L.FMA_TIER_HOST, flags: int = 0) -> None:
        check(self._lib.fma_sleep(self._h, self.tag_mask(offload_tags), tier, flags))

    def wake(self, tags: Sequence[str] | None = None, flags: int = 0) -> None:
        check(self._lib.fma_wake(self._h, self.tag_mask(tags), flags))

    def is_sleeping(self) -> bool:
        return bool(check(self._lib.fma_is_sleeping(self._h)))

    def swap_out_for(self, incoming: "Engine", offload_tags: Sequence[str] = ("default",),
                     tier: int = L.FMA_TIER_HOST, wake_tags: Sequence[str] | None = None, flags: int = 0) -> None:
        """Sleep *this* engine's model while waking ``incoming``'s, both PCIe directions at once."""
        check(self._lib.fma_swap(self._h, self.tag_mask(offload_tags), tier, incoming._h,
                                 incoming.tag_mask(wake_tags), flags))

    # -- stores ---------------------------------------------------------------------------
    def host_reserve(self, nbytes: int) -> None:
        check(self._lib.fma_host_reserve(self._h, nbytes))

    def host_release(self) -> None:
        check(self._lib.fma_host_release(self._h))

    def host_store_view(self) -> tuple[int, int]:
        base, n = C.c_void_p(), C.c_uint64()
        check(self._lib.fma_host_store_view(self._h, C.byref(base), C.byref(n)))
        return int(base.value), int(n.value)

    def peer_reserve(self, peer_device: int, nbytes: int) -> None:
        check(self._lib.fma_peer_reserve(self._h, peer_device, nbytes))

    def peer_release(self) -> None:
        check(self._lib.fma_peer_release(self._h))

    def set_paths(self, helper_devices: Sequence[int], slot_bytes: int = 0, slots: int = 0) -> None:
        """MULTI-PATH wake: idle peer GPUs whose PCIe links a host-tier wake may borrow ([] = off).  See fma_paths_set."""
        arr = (C.c_int * max(len(helper_devices), 1))(*helper_devices)
        check(self._lib.fma_paths_set(self._h, arr, len(helper_devices), slot_bytes, slots))

    def paths_attach(self, staging_fds: Sequence[int], slot_bytes: int, slots: int) -> int:
        """MULTI-PATH wake across processes: the node-level owner's staging buffers (``HelperStaging.fd``) become remote paths.  Returns
        the mailbox fd (owned by the engine: ``os.dup`` it before sending it away)."""
        arr = (C.c_int * len(staging_fds))(*staging_fds)
        mb = C.c_int(-1)
        check(self._lib.fma_paths_attach(self._h, arr, len(staging_fds), slot_bytes, slots, C.byref(mb)))
        return int(mb.value)

    def pull_next_generation(self) -> int:
        return int(self._lib.fma_pull_next_generation(self._h))

    def host_store_share(self) -> int:
        """fd of the memfd behind the host store (FMA_HOST_STORE_SHM=1), for the owner's ``fma_store_attach``; the caller closes it."""
        fd = C.c_int(-1)
        check(self._lib.fma_host_store_share(self._h, C.byref(fd)))
        return int(fd.value)

    def peer_attach(self, fd: int, nbytes: int) -> None:
        """Use a node-level owner's parking buffer (``ParkingBuffer``; fd received over SCM_RIGHTS / inherited) as this engine's
        peer-tier store.  The buffer's GPU need not be visible to this process (launcher.py:171-187 hides it)."""
        check(self._lib.fma_peer_attach(self._h, fd, nbytes))

    def image_describe(self, tier: int = L.FMA_TIER_PEER) -> bytes:
        """Descriptor of the image sleeping in ``tier`` (the node-level owner keeps it next to the buffer's fd)."""
        n = check(self._lib.fma_image_describe(self._h, tier, None, 0))
        buf = C.create_string_buffer(n)
        check(self._lib.fma_image_describe(self._h, tier, buf, n))
        return buf.raw

    def image_adopt_parked(self, descriptor: bytes, tags: Sequence[str], flags: int = 0) -> None:
        """After ``peer_attach``: become 'asleep with the image parked in that buffer' (same segment sequence for ``tags``)."""
        check(self._lib.fma_image_adopt_parked(self._h, descriptor, len(descriptor), self.tag_mask(tags), flags))

    # -- integrity / synthetic data -------------------------------------------------------
    def digest(self, index: int) -> int:
        out = C.c_uint64()
        check(self._lib.fma_digest_segment(self._h, index, C.byref(out)))
        return int(out.value)

    def digest_all(self, tags: Sequence[str] | None = None) -> list[int]:
        n = self.segment_count()
        out = (C.c_uint64 * max(n, 1))()
        check(self._lib.fma_digest_all(self._h, self.tag_mask(tags), out, n))
        return [int(out[i]) for i in range(n)]

    def fill(self, index: int, seed: int, first_word: int = 0) -> None:
        check(self._lib.fma_fill_segment(self._h, index, seed, first_word))

    def write(self, index: int, data: bytes | bytearray | memoryview, offset: int = 0) -> None:
        buf = (C.c_char * len(data)).from_buffer_copy(bytes(data))
        check(self._lib.fma_segment_write(self._h, index, offset, buf, len(data)))

    def read(self, index: int, nbytes: int, offset: int = 0) -> bytes:
        buf = C.create_string_buffer(nbytes)
        check(self._lib.fma_segment_read(self._h, index, offset, buf, nbytes))
        return buf.raw

    def write_ptr(self, index: int, host_ptr: int, nbytes: int, offset: int = 0) -> None:
        check(self._lib.fma_segment_write(self._h, index, offset, C.c_void_p(host_ptr), nbytes))

    def read_ptr(self, index: int, host_ptr: int, nbytes: int, offset: int = 0) -> None:
        check(self._lib.fma_segment_read(self._h, index, offset, C.c_void_p(host_ptr), nbytes))

    # -- raw kernels ----------------------------------------------------------------------
    def op_page_copy(self, n_pages: int, src_pages: Sequence[int] | None = None, src_base: int = 0,
                     dst_pages: Sequence[int] | None = None, dst_base: int = 0, variant: int = L.FMA_KERNEL_TMA) -> float:
        sp = (C.c_uint64 * n_pages)(*src_pages) if src_pages is not None else None
        dp = (C.c_uint64 * n_pages)(*dst_pages) if dst_pages is not None else None
        ms = C.c_float()
        check(self._lib.fma_op_page_copy(self._h, sp, src_base, dp, dst_base, n_pages, variant, C.byref(ms)))
        return float(ms.value)

    def op_page_digest(self, n_pages: int, pages: Sequence[int] | None = None, base: int = 0,
                       first_word: Sequence[int] | None = None) -> tuple[list[int], float]:
        pp = (C.c_uint64 * n_pages)(*pages) if pages is not None else None
        fw = (C.c_uint64 * n_pages)(*first_word) if first_word is not None else None
        out = (C.c_uint64 * n_pages)()
        ms = C.c_float()
        check(self._lib.fma_op_page_digest(self._h, pp, base, fw, n_pages, out, C.byref(ms)))
        return [int(x) for x in out], float(ms.value)

    # -- PACKED image ---------------------------------------------------------------------
    def image_pages(self) -> tuple[list[int], list[int]]:
        """(store offset, stored bytes) of every 2 MiB page of the sleeping image, in image order."""
        n = check(self._lib.fma_image_pages(self._h, None, None, 0))
        off, nb = (C.c_uint64 * max(n, 1))(), (C.c_uint32 * max(n, 1))()
        check(self._lib.fma_image_pages(self._h, off, nb, n))
        return [int(off[i]) for i in range(n)], [int(nb[i]) for i in range(n)]

    def op_pack_probe(self, n_pages: int, pages: Sequence[int] | None = None, base: int = 0) -> tuple[list[int], float]:
        pp = (C.c_uint64 * n_pages)(*pages) if pages is not None else None
        out = (C.c_uint32 * n_pages)()
        ms = C.c_float()
        check(self._lib.fma_op_pack_probe(self._h, pp, base, n_pages, out, C.byref(ms)))
        return [int(x) for x in out], float(ms.value)

    def op_pack(self, stored_bytes: Sequence[int], dst_base: int, src_pages: Sequence[int] | None = None, src_base: int = 0) -> float:
        n = len(stored_bytes)
        sp = (C.c_uint64 * n)(*src_pages) if src_pages is not None else None
        ms = C.c_float()
        check(self._lib.fma_op_pack(self._h, sp, src_base, dst_base, (C.c_uint32 * n)(*stored_bytes), n, C.byref(ms)))
        return float(ms.value)

    def op_unpack(self, stored_bytes: Sequence[int], src_base: int, dst_pages: Sequence[int] | None = None, dst_base: int = 0) -> float:
        n = len(stored_bytes)
        dp = (C.c_uint64 * n)(*dst_pages) if dst_pages is not None else None
        ms = C.c_float()
        check(self._lib.fma_op_unpack(self._h, src_base, (C.c_uint32 * n)(*stored_bytes), dp, dst_base, n, C.byref(ms)))
        return float(ms.value)

    def scratch_alloc(self, nbytes: int) -> int:
        out = C.c_uint64()
        check(self._lib.fma_scratch_alloc(self._h, nbytes, C.byref(out)))
        return int(out.value)

    def scratch_free(self, ptr: int) -> None:
        check(self._lib.fma_scratch_free(self._h, ptr))

    # -- image hand-over ------------------------------------------------------------------
    def image_export(self) -> int:
        """File descriptor of the sleeping image (needs FMA_HOST_STORE_SHM=1); the caller closes it."""
        fd = C.c_int(-1)
        check(self._lib.fma_image_export(self._h, C.byref(fd)))
        return int(fd.value)

    def image_adopt(self, fd: int, tags: Sequence[str], flags: int = 0) -> None:
        """Become 'asleep with that image': this engine must hold the same segment sequence for ``tags``."""
        check(self._lib.fma_image_adopt(self._h, fd, self.tag_mask(tags), flags))

    def image_save(self, path: str) -> int:
        """Persist the sleeping image (store + descriptor) as a file; a later process with the same segment table can
        ``image_load`` it instead of loading weights.  Needs FMA_HOST_STORE_SHM=1.  Returns the bytes written."""
        import os
        import shutil

        fd = self.image_export()
        try:
            with os.fdopen(os.dup(fd), "rb") as src, open(path + ".tmp", "wb") as dst:
                shutil.copyfileobj(src, dst, length=64 << 20)
                n = dst.tell()
            os.replace(path + ".tmp", path)
            return n
        finally:
            os.close(fd)

    def image_load(self, path: str, tags: Sequence[str], flags: int = 0) -> None:
        """``image_adopt`` from a file written by ``image_save``: afterwards this engine is asleep with that image."""
        import os

        fd = os.open(path, os.O_RDWR)
        try:
            self.image_adopt(fd, tags, flags)
        finally:
            os.close(fd)

    # -- FILE tier ------------------------------------------------------------------------
    def file_store(self, path: str | None) -> None:
        """The file the next ``sleep(tier=FMA_TIER_FILE)`` writes (None forgets it).  The caller owns the file; the engine never
        removes it.  Pins the engine's I/O windows (``stats()["io_buffer_bytes"]``) the first time."""
        check(self._lib.fma_file_store(self._h, None if path is None else path.encode()))

    def image_adopt_file(self, path: str, tags: Sequence[str], flags: int = 0) -> None:
        """Become 'asleep in the file tier' with the image in ``path`` (written by a file-tier sleep or by ``image_save``): this
        engine must hold the same segment sequence for ``tags``.  Reads only the descriptor; ``wake`` streams the data."""
        check(self._lib.fma_image_adopt_file(self._h, path.encode(), self.tag_mask(tags), flags))

    def writeback(self, timeout_s: float | None = 0.0) -> tuple[int, int]:
        """The last write-behind job (``sleep(tier=FMA_TIER_FILE, flags=FMA_FLAG_WRITE_BEHIND)``), after waiting up to ``timeout_s``
        seconds for it (0 polls, None waits until it ends): (1, bytes not yet written) while it writes, (0, 0) once it committed
        (the image sleeps in the file tier), was pre-empted by another call, or when none was started.  Raises FmaError, once, for
        a job whose write failed: the image then still sleeps in the host tier."""
        pending = C.c_uint64()
        state = check(self._lib.fma_image_writeback(self._h, -1.0 if timeout_s is None else float(timeout_s), C.byref(pending)))
        return state, int(pending.value)

    @staticmethod
    def image_file_info(path: str) -> dict:
        """What the image file at ``path`` holds, from its descriptor tail alone (fma_image_file_info): no engine, no GPU.  Keys:
        image_bytes (stored), weight_bytes, n_segments, version, packed, digests (every segment carries one) and tags (names).
        Raises FmaError: FMA_EIO for a file that cannot be read or is shorter than its image, FMA_EINVAL for a torn or foreign
        tail."""
        lib = L.load_library()
        out = L.fma_image_file_info_t()
        check(lib.fma_image_file_info(path.encode(), C.byref(out)))
        return {"image_bytes": out.image_bytes, "weight_bytes": out.weight_bytes, "n_segments": out.n_segments, "version": out.version,
                "packed": bool(out.packed), "digests": bool(out.digests), "tags": [out.tags[i].value.decode() for i in range(out.n_tags)]}

    def move_image(self, tier: int, behind: bool = False) -> None:
        """Move the sleeping image to ``tier`` without waking it (fma_image_move): host DRAM, a file (``file_store`` first), a peer's
        parking buffer (``peer_reserve`` first) or this GPU's.  The source store stays allocated until ``host_release`` /
        ``peer_release``; a source file is never touched.

        ``behind=True`` (host tier to FMA_TIER_FILE only, fma_image_move_flags with FMA_FLAG_WRITE_BEHIND): returns once the file is
        checked and emptied; the write-behind job writes it from the host store, then moves the image to the file tier and frees
        the store.  ``writeback`` waits for it; any later call that takes the operation lock (a wake included) pre-empts it and
        sees the host-tier image.  A shared host store is refused (FMA_ESTATE)."""
        if behind:
            check(self._lib.fma_image_move_flags(self._h, tier, L.FMA_FLAG_WRITE_BEHIND))
        else:
            check(self._lib.fma_image_move(self._h, tier))

    def verify_image(self) -> list[int]:
        """Check the sleeping image against the digests it carries, where it lies, without waking it (fma_image_verify): the
        indices of the segments whose stored bytes do not match, [] when it is intact.  Raises FmaError when nothing is asleep, a
        segment carries no digest (sleep with FMA_FLAG_VERIFY or ``incremental``), a mapped segment keeps a backup, or the image
        file cannot be read whole (FMA_EIO)."""
        n = self.segment_count()
        bad = (C.c_int * max(n, 1))()
        k = check(self._lib.fma_image_verify(self._h, bad, n))
        return sorted(bad[i] for i in range(min(k, n)))

    def prefetch_image(self, nbytes: int) -> None:
        """Copy the tail of the sleeping image, up to ``nbytes`` of stored bytes (rounded down to 2 MiB), into this GPU's HBM ahead
        of a wake, without waking it (fma_image_prefetch); 0 gives that HBM back.  The next ``wake`` restores those segments from
        HBM and moves only the others over PCIe or from disk.  ``stats()["prefetched_bytes"]`` is what the copy holds.  Raises
        FmaError when nothing is asleep, a mapped segment keeps a backup, the image has a resident share (FMA_ESTATE) or sleeps in
        a parking buffer (FMA_EINVAL), or when HBM (FMA_ENOMEM) or the image file (FMA_EIO) fails it."""
        check(self._lib.fma_image_prefetch(self._h, nbytes))

    # -- cold load -------------------------------------------------------------------------
    def load_file(self, path: str, spans: Sequence[tuple[int, int, int]], o_direct: bool = False) -> dict:
        """Stream (file_offset, nbytes, device_address) spans of one file into mapped segments."""
        arr = (L.fma_load_span_t * max(len(spans), 1))()
        for i, (off, n, dst) in enumerate(spans):
            arr[i].file_offset, arr[i].bytes, arr[i].dst = off, n, dst
        st = L.fma_load_stats_t()
        check(self._lib.fma_load_file(self._h, path.encode(), arr, len(spans), L.FMA_LOAD_O_DIRECT if o_direct else 0, C.byref(st)))
        return {"seconds": st.seconds, "read_seconds": st.read_seconds, "bytes": st.bytes, "chunks": st.chunks, "threads": st.threads}

    def set_option(self, key: str, value: int) -> None:
        check(self._lib.fma_set_option(self._h, key.encode(), int(value)))

    # -- stats ----------------------------------------------------------------------------
    def stats(self) -> dict:
        st = L.fma_stats_t()
        check(self._lib.fma_stats(self._h, C.byref(st)))
        return st.as_dict()

    def timeline(self) -> list[dict]:
        """Per-phase timeline of the last sleep / wake (fma_timeline): rows of op, kind, idx, t0_ms, t1_ms, bytes."""
        n = self._lib.fma_timeline(self._h, None, 0)
        if n < 0:
            check(n)
        buf = C.create_string_buffer(n + 1)
        check(min(self._lib.fma_timeline(self._h, buf, n + 1), 0))
        rows = []
        for line in buf.value.decode().splitlines():
            op, kind, idx, t0, t1, b = line.split(",")
            rows.append({"op": op, "kind": kind, "idx": int(idx), "t0_ms": float(t0), "t1_ms": float(t1), "bytes": int(b)})
        return rows


class HelperStaging:
    """Owner side of a remote wake path: a staging buffer in ``device``'s HBM plus that GPU's copy stream (fma_helper_open).  ``pull``
    serves one wake of an instance that attached ``fd`` (blocking: run it in a thread per helper)."""

    def __init__(self, device: int, slot_bytes: int = 128 << 20, slots: int = 3):
        self._lib = L.load_library()
        h, fd = C.c_uint64(), C.c_int(-1)
        check(self._lib.fma_helper_open(device, slot_bytes, slots, C.byref(h), C.byref(fd)))
        self.handle, self.fd, self.device, self.slot_bytes, self.slots = int(h.value), int(fd.value), device, slot_bytes, slots

    def pull(self, store_handle: int, mailbox_fd: int, path_index: int, generation: int, timeout_s: float = 5.0) -> None:
        check(self._lib.fma_helper_pull(self.handle, store_handle, mailbox_fd, path_index, generation, timeout_s))

    def close(self) -> None:
        if self.handle:
            import os

            self._lib.fma_helper_close(self.handle)
            self.handle = 0
            try:
                os.close(self.fd)
            except OSError:
                pass


def store_attach(fd: int) -> int:
    """Owner side: map + pin an instance's memfd host store (``Engine.host_store_share``); returns the handle for ``HelperStaging.pull``."""
    lib = L.load_library()
    h = C.c_uint64()
    check(lib.fma_store_attach(fd, C.byref(h)))
    return int(h.value)


def store_detach(handle: int) -> None:
    check(L.load_library().fma_store_detach(handle))


class ParkingBuffer:
    """Node-level owner's side of the peer tier: an exportable VMM allocation in ``device``'s HBM (fma_parking_create).  The
    owner process must see ``device``; instances need not.  ``fd`` / ``export_fd()`` go to instances (``Engine.peer_attach``)."""

    def __init__(self, device: int, nbytes: int):
        self._lib = L.load_library()
        h, fd, nb = C.c_uint64(), C.c_int(-1), C.c_uint64()
        check(self._lib.fma_parking_create(device, nbytes, C.byref(h), C.byref(fd)))
        self.handle, self.fd, self.device = int(h.value), int(fd.value), device
        fd2 = C.c_int(-1)
        check(self._lib.fma_parking_export(self.handle, C.byref(fd2), C.byref(nb)))
        import os

        os.close(fd2.value)
        self.nbytes = int(nb.value)

    def export_fd(self) -> int:
        fd = C.c_int(-1)
        check(self._lib.fma_parking_export(self.handle, C.byref(fd), None))
        return int(fd.value)

    def close(self) -> None:
        if self.handle:
            import os

            self._lib.fma_parking_destroy(self.handle)
            self.handle = 0
            try:
                os.close(self.fd)
            except OSError:
                pass


__all__ = ["Engine", "EngineConfig", "SegmentInfo", "FmaError", "ParkingBuffer", "HelperStaging", "store_attach", "store_detach"]
