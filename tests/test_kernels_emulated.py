"""The ACTUAL kernel sources of the packed-image path (csrc/fma_pack_kernels.cu: K4p, K4, K5) and of the hot path (csrc/fma_kernels.cu,
whose mbarrier / cp.async.bulk traffic runs on a LAZY model of the async proxy — a copy happens when somebody legitimately waits
for it, so a missing wait yields wrong bytes) executed on a CPU model of
the CUDA execution hierarchy (tests/cpp/cuda_emu/cuda_emu.h: a CTA = blockDim OS threads, __syncthreads = barrier, warp
collectives = warp barrier + scratch line, __shared__ = static) and compared with the oracle page by page.  Under
ThreadSanitizer a missing __syncthreads() shows up as a data race (checked by mutation when this was written).

Test infrastructure only; nothing here ships.  What it cannot show — the PTX load/store wrappers, coalescing, speed —
is what the -m gpu tests and the ncu profiles are for."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cpp", "cuda_emu")
CSRC = os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc")


def _build_and_run(tmp_path, src, name, san, flags, marker):
    exe = str(tmp_path / f"{name}_{san}")
    subprocess.check_call(["g++", "-std=c++17", "-g", *flags, "-DFMA_CUDA_EMU", "-include", os.path.join(EMU, "cuda_emu.h"),
                           "-I/usr/local/cuda/include", "-I" + CSRC, os.path.join(EMU, src), os.path.join(ROOT, "oracle", "fma_oracle.c"),
                           "-o", exe, "-lpthread"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    if san != "plain":
        env["FMA_EMU_FAST"] = "1"          # fewer pages under the sanitizer (every code branch is still taken)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and marker in out, (name, san, out[-3000:])
    assert "WARNING: ThreadSanitizer" not in out, (name, san, out[-3000:])
    return True


def test_kernel_sources_on_the_cpu_execution_model(tmp_path):
    """Four builds side by side: {packed-image kernels (K4p, K4, K5: sub-page work items, a global exception counter per page, last-part header), hot-path kernels (K0, K1/K2 TMA over a
    subset of the legal shapes, clamped and refused shapes + LDG, K3 — the source the GPU tests run on the H100; the emulation guards leave its nvcc SASS byte-identical)}
    x {plain, ThreadSanitizer}, each against the oracle."""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from concurrent.futures import ThreadPoolExecutor

    jobs = [("pack_kernels_emu_test.cpp", "pack_emu", "pack kernels (emulated) ok"), ("kernels_emu_test.cpp", "kernels_emu", "kernels (emulated) ok")]
    variants = [("plain", ["-O2"]), ("tsan", ["-O1", "-fsanitize=thread"])]
    with ThreadPoolExecutor(4) as pool:
        futs = [pool.submit(_build_and_run, tmp_path, src, name, san, flags, marker) for src, name, marker in jobs for san, flags in variants]
        assert all(f.result() for f in futs)
