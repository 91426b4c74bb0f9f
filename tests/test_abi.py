"""The C-ABI library builds for sm_90a, loads on a CPU-only box, exports every symbol include/*.h
declares, matches the ctypes mirror byte for byte, and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fma_engine.h")


def _declared():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"^FMA_API\s+[\w\s\*]+?\b(fma_\w+|my_malloc|my_free)\s*\(", src, re.M)))


def test_header_declares_the_hot_path_entry_points():
    names = _declared()
    for must in ("my_malloc", "my_free", "fma_engine_create", "fma_sleep", "fma_wake", "fma_is_sleeping", "fma_swap",
                 "fma_host_reserve", "fma_peer_reserve", "fma_digest_all", "fma_stats", "fma_last_error"):
        assert must in names
    assert len(names) >= 38


def test_library_exports_every_declared_symbol(built):
    import fma_b200

    out = subprocess.check_output(["nm", "-D", "--defined-only", fma_b200.lib_path()], text=True)
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    missing = [n for n in _declared() if n not in exported]
    assert not missing, missing
    # nothing else leaks (static cudart stays private so it cannot clash with torch's libcudart)
    assert all(n.startswith("fma_") or n in ("my_malloc", "my_free") for n in exported), exported
    binding = set(__import__("fma_b200")._lib._PROTOTYPES)
    assert binding == set(_declared())


def test_library_has_no_link_time_cuda_dependency(built):
    import fma_b200

    out = subprocess.check_output(["ldd", fma_b200.lib_path()], text=True)
    assert "libcuda" not in out and "libcudart" not in out


def test_struct_layouts_match_the_header(built, tmp_path):
    from fma_b200 import _lib as L

    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fma_engine.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n",'
                   "sizeof(fma_config_t),sizeof(fma_segment_info_t),sizeof(fma_stats_t),offsetof(fma_stats_t,kernel_seconds),"
                   "offsetof(fma_stats_t,host_store_bytes),offsetof(fma_segment_info_t,tag));}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [C.sizeof(L.fma_config_t), C.sizeof(L.fma_segment_info_t), C.sizeof(L.fma_stats_t),
                   L.fma_stats_t.kernel_seconds.offset, L.fma_stats_t.host_store_bytes.offset,
                   L.fma_segment_info_t.tag.offset]


def test_sass_contains_tma_bulk_copies(built):
    """K1/K2 are Hopper-native: the SASS must show UBLKCP (cp.async.bulk), mbarrier waits (SYNCS) and 128-bit
    streaming LDG/STG, the widest global access sm_90 has."""
    import fma_b200

    sass = subprocess.check_output(["cuobjdump", "-sass", fma_b200.lib_path()], text=True)
    assert "sm_90a" in sass
    assert "UBLKCP" in sass and "SYNCS" in sass
    assert "LDG.E.NA.128" in sass and "STG.E.NA.128" in sass


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="CPU-only behaviour")
def test_no_cpu_fallback_without_a_driver(built):
    import fma_b200
    from fma_b200 import _lib as L

    lib = fma_b200.load_library()
    assert lib.fma_abi_version() == 2
    assert lib.fma_driver_available() == L.FMA_ENODRIVER
    with pytest.raises(fma_b200.FmaError) as ei:
        fma_b200.Engine(0)
    assert ei.value.code == L.FMA_ENODRIVER
    assert lib.my_malloc(1 << 21, 0, None) is None          # the torch entry point cannot hand out memory either
    # NULL-handle calls fail cleanly instead of crashing
    assert lib.fma_sleep(None, 1, 0, 0) == L.FMA_EINVAL
    assert lib.fma_wake(None, 0, 0) == L.FMA_EINVAL
    assert lib.fma_is_sleeping(None) == L.FMA_EINVAL


@pytest.mark.skipif(_has_gpu(), reason="CPU-only behaviour")
def test_missing_library_is_a_loud_error(built, monkeypatch):
    from fma_b200 import _lib as L

    monkeypatch.setenv("FMA_B200_LIB", "/nonexistent/libfma_b200.so")
    monkeypatch.setattr(L, "_lib", None)
    with pytest.raises(L.FmaError):
        L.load_library()


@pytest.mark.skipif(_has_gpu(), reason="CPU-only behaviour")
def test_cumem_shim_refuses_without_gpu(built):
    from fma_b200 import cumem
    from fma_b200._lib import FmaError

    cumem.CuMemAllocator.instance = None
    with pytest.raises(FmaError):
        cumem.CuMemAllocator.get_instance()
