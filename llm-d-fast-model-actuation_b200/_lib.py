"""ctypes binding of include/fma_engine.h (one-to-one; no logic)."""
from __future__ import annotations

import ctypes as C
import os

FMA_ABI_VERSION = 2
FMA_PAGE_BYTES = 2 << 20
FMA_PACKED_PAGE_BYTES = (3 << 19) + (16 << 10)   # stored size of a page in the "FMP4" code (csrc/fma_codec.h)
FMA_MAX_TAGS = 64
FMA_IMAGE_TAIL_BYTES = 2 << 20   # the descriptor at the end of an image file or exported host store

FMA_OK, FMA_EINVAL, FMA_ENODRIVER, FMA_ECUDA, FMA_ENOMEM, FMA_ESTATE, FMA_ENOTFOUND, FMA_EINTEGRITY, FMA_EIO = (
    0, -1, -2, -3, -4, -5, -6, -7, -8)
ERROR_NAMES = {
    FMA_EINVAL: "FMA_EINVAL", FMA_ENODRIVER: "FMA_ENODRIVER", FMA_ECUDA: "FMA_ECUDA", FMA_ENOMEM: "FMA_ENOMEM",
    FMA_ESTATE: "FMA_ESTATE", FMA_ENOTFOUND: "FMA_ENOTFOUND", FMA_EINTEGRITY: "FMA_EINTEGRITY", FMA_EIO: "FMA_EIO",
}
FMA_TIER_HOST, FMA_TIER_PEER, FMA_TIER_LOCAL, FMA_TIER_FILE = 0, 1, 2, 3
FMA_MODE_AUTO, FMA_MODE_DIRECT, FMA_MODE_STAGED, FMA_MODE_KERNEL = 0, 1, 2, 3
FMA_KERNEL_TMA, FMA_KERNEL_LDG = 0, 1
FMA_FLAG_VERIFY, FMA_FLAG_KEEP_BACKUP, FMA_FLAG_WRITE_BEHIND = 1, 2, 4
NO_OFFSET = (1 << 64) - 1


class FmaError(RuntimeError):
    """Raised for every negative return code of the C-ABI (mirrors the reference C module's
    ``RuntimeError("CUDA Error: ...")``, SURVEY.md §8b B2)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"{ERROR_NAMES.get(code, code)}: {message}")
        self.code = code
        self.message = message


class fma_config_t(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("mode", C.c_int32), ("kernel", C.c_int32), ("copy_streams", C.c_int32),
        ("chunk_bytes", C.c_uint64), ("ring_slots", C.c_int32), ("map_threads", C.c_int32),
        ("numa_bind", C.c_int32), ("pack", C.c_int32), ("reserved", C.c_uint64 * 6),
    ]


class fma_segment_info_t(C.Structure):
    _fields_ = [
        ("va", C.c_uint64), ("bytes", C.c_uint64), ("requested_bytes", C.c_uint64), ("packed_offset", C.c_uint64),
        ("seq", C.c_uint64), ("tag", C.c_int32), ("mapped", C.c_int32), ("has_backup", C.c_int32), ("tier", C.c_int32),
    ]


class fma_stats_t(C.Structure):
    _fields_ = [
        ("sleep_seconds", C.c_double), ("sleep_copy_seconds", C.c_double), ("sleep_unmap_seconds", C.c_double),
        ("sleep_bytes_offloaded", C.c_uint64), ("sleep_bytes_discarded", C.c_uint64),
        ("wake_seconds", C.c_double), ("wake_copy_seconds", C.c_double), ("wake_map_seconds", C.c_double),
        ("wake_first_copy_delay", C.c_double), ("wake_bytes_restored", C.c_uint64),
        ("wake_bytes_remapped_only", C.c_uint64),
        ("kernel_seconds", C.c_double), ("kernel_bytes", C.c_uint64), ("kernel_launches", C.c_uint32),
        ("copy_ops", C.c_uint32),
        ("host_store_bytes", C.c_uint64), ("host_store_pin_seconds", C.c_double),
        ("host_store_numa_node", C.c_int32), ("tier", C.c_int32), ("mode", C.c_int32), ("image_packed", C.c_int32),
        ("total_kernel_launches", C.c_uint64), ("total_copy_ops", C.c_uint64),
        ("hbm_mapped_bytes", C.c_uint64), ("hbm_aux_bytes", C.c_uint64), ("parked_bytes", C.c_uint64),
        ("image_store_bytes", C.c_uint64), ("sleep_bytes_copied", C.c_uint64), ("resident_bytes", C.c_uint64),
        ("io_buffer_bytes", C.c_uint64), ("prefetched_bytes", C.c_uint64),
    ]

    def as_dict(self) -> dict:
        return {n: getattr(self, n) for n, _ in self._fields_ if not n.startswith("reserved")}


class fma_load_span_t(C.Structure):
    _fields_ = [("file_offset", C.c_uint64), ("bytes", C.c_uint64), ("dst", C.c_uint64)]


class fma_load_stats_t(C.Structure):
    _fields_ = [("seconds", C.c_double), ("read_seconds", C.c_double), ("bytes", C.c_uint64), ("chunks", C.c_uint32),
                ("threads", C.c_uint32), ("reserved", C.c_uint64 * 4)]


FMA_LOAD_O_DIRECT = 1


class fma_image_file_info_t(C.Structure):
    _fields_ = [("image_bytes", C.c_uint64), ("weight_bytes", C.c_uint64), ("n_segments", C.c_uint32), ("version", C.c_uint32),
                ("packed", C.c_int32), ("digests", C.c_int32), ("n_tags", C.c_uint32), ("reserved0", C.c_uint32),
                ("tags", (C.c_char * 32) * FMA_MAX_TAGS), ("reserved", C.c_uint64 * 4)]


def lib_path() -> str:
    """Path of the in-tree shared library (built by ``__graft_entry__.build()`` / csrc/Makefile)."""
    return os.environ.get("FMA_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libfma_b200.so")


_PROTOTYPES = {
    # name: (restype, argtypes)
    "fma_abi_version": (C.c_int, []),
    "fma_last_error": (C.c_char_p, []),
    "fma_driver_available": (C.c_int, []),
    "fma_engine_create": (C.c_int, [C.c_int, C.POINTER(fma_config_t), C.POINTER(C.c_void_p)]),
    "fma_engine_destroy": (C.c_int, [C.c_void_p]),
    "fma_set_current": (C.c_int, [C.c_void_p]),
    "fma_get_current": (C.c_void_p, []),
    "fma_tag_intern": (C.c_int, [C.c_void_p, C.c_char_p]),
    "fma_tag_name": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]),
    "fma_set_current_tag": (C.c_int, [C.c_void_p, C.c_int]),
    "my_malloc": (C.c_void_p, [C.c_ssize_t, C.c_int, C.c_void_p]),
    "my_free": (None, [C.c_void_p, C.c_ssize_t, C.c_int, C.c_void_p]),
    "fma_alloc": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "fma_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fma_segment_count": (C.c_int, [C.c_void_p]),
    "fma_segment_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(fma_segment_info_t)]),
    "fma_segment_find": (C.c_int, [C.c_void_p, C.c_void_p]),
    "fma_current_usage": (C.c_uint64, [C.c_void_p]),
    "fma_sleep": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.c_uint32]),
    "fma_wake": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32]),
    "fma_is_sleeping": (C.c_int, [C.c_void_p]),
    "fma_swap": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.c_uint32]),
    "fma_host_reserve": (C.c_int, [C.c_void_p, C.c_size_t]),
    "fma_host_release": (C.c_int, [C.c_void_p]),
    "fma_host_store_view": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]),
    "fma_peer_reserve": (C.c_int, [C.c_void_p, C.c_int, C.c_size_t]),
    "fma_peer_release": (C.c_int, [C.c_void_p]),
    "fma_digest_segment": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]),
    "fma_digest_all": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_int]),
    "fma_fill_segment": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint64]),
    "fma_segment_write": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64]),
    "fma_segment_read": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64]),
    "fma_op_page_copy": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64), C.c_uint64,
                                   C.c_uint32, C.c_int, C.POINTER(C.c_float)]),
    "fma_op_page_digest": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64), C.c_uint32,
                                     C.POINTER(C.c_uint64), C.POINTER(C.c_float)]),
    "fma_image_pages": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_uint32]),
    "fma_op_pack_probe": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint32),
                                    C.POINTER(C.c_float)]),
    "fma_op_pack": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32), C.c_uint32,
                              C.POINTER(C.c_float)]),
    "fma_op_unpack": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_uint64, C.c_uint32,
                                C.POINTER(C.c_float)]),
    "fma_scratch_alloc": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]),
    "fma_scratch_free": (C.c_int, [C.c_void_p, C.c_uint64]),
    "fma_load_file": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(fma_load_span_t), C.c_uint32, C.c_uint32,
                                C.POINTER(fma_load_stats_t)]),
    "fma_image_export": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "fma_image_adopt": (C.c_int, [C.c_void_p, C.c_int, C.c_uint64, C.c_uint32]),
    "fma_file_store": (C.c_int, [C.c_void_p, C.c_char_p]),
    "fma_image_adopt_file": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint32]),
    "fma_image_writeback": (C.c_int, [C.c_void_p, C.c_double, C.POINTER(C.c_uint64)]),
    "fma_image_file_info": (C.c_int, [C.c_char_p, C.POINTER(fma_image_file_info_t)]),
    "fma_image_move": (C.c_int, [C.c_void_p, C.c_int]),
    "fma_image_move_flags": (C.c_int, [C.c_void_p, C.c_int, C.c_uint32]),
    "fma_image_verify": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int]),
    "fma_image_prefetch": (C.c_int, [C.c_void_p, C.c_uint64]),
    "fma_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    "fma_stats": (C.c_int, [C.c_void_p, C.POINTER(fma_stats_t)]),
    "fma_timeline": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "fma_paths_set": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_size_t, C.c_int]),
    "fma_helper_open": (C.c_int, [C.c_int, C.c_size_t, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "fma_helper_close": (C.c_int, [C.c_uint64]),
    "fma_store_attach": (C.c_int, [C.c_int, C.POINTER(C.c_uint64)]),
    "fma_store_detach": (C.c_int, [C.c_uint64]),
    "fma_helper_pull": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_uint64, C.c_double]),
    "fma_paths_attach": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_size_t, C.c_int, C.POINTER(C.c_int)]),
    "fma_pull_next_generation": (C.c_uint64, [C.c_void_p]),
    "fma_host_store_share": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "fma_parking_create": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "fma_parking_export": (C.c_int, [C.c_uint64, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]),
    "fma_parking_destroy": (C.c_int, [C.c_uint64]),
    "fma_peer_attach": (C.c_int, [C.c_void_p, C.c_int, C.c_size_t]),
    "fma_image_describe": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "fma_image_adopt_parked": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint32]),
}

_lib = None


def load_library() -> C.CDLL:
    """dlopen libfma_b200.so and type every entry point.  Fails loudly if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise FmaError(FMA_ENODRIVER, f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU fallback for the weight-movement path)")
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    for name, (restype, argtypes) in _PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.fma_abi_version() != FMA_ABI_VERSION:
        raise FmaError(FMA_EINVAL, f"ABI mismatch: library {lib.fma_abi_version()} != binding {FMA_ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int) -> int:
    if rc < 0:
        raise FmaError(rc, (load_library().fma_last_error() or b"").decode(errors="replace"))
    return rc
