"""The engine's layout logic (VA arenas with first-fit reuse, run planning, and the pages, batches, chunk queues and resident
split of the sleep / wake copy pipelines) is plain C++ in csrc/fma_layout.h and is what the engine (csrc/fma_engine.cu,
fma_sleep.cu, fma_wake.cu) compiles in; exercised here on CPU with g++ (incl. a 20k-step randomised alloc/free invariant check)."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_layout_logic(tmp_path):
    exe = str(tmp_path / "layout_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-Wall", "-Wextra", "-Werror", "-I",
                           os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "layout_test.cpp"), "-o", exe])
    out = subprocess.check_output([exe], text=True)
    assert "layout ok" in out


def test_image_operations_write_each_shared_step_once():
    """The operations on a sleeping image (adoption from a memfd, a file or a parking buffer; move, verify, prefetch) and the
    file tier's sleep and wake share one adoption path, one reader and writer of the image file and one store <-> HBM copy."""
    csrc = os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc")
    read = {f: open(os.path.join(csrc, f)).read() for f in sorted(os.listdir(csrc)) if f.endswith((".cu", ".h", ".cpp"))}
    src, image = "".join(read.values()), read["fma_image.cu"]
    for msg in ("the image holds different bytes than this engine's segments", "the image carries no digests to compare with",
                "adopt needs a fully awake engine"):
        assert image.count(msg) == 1, msg
    assert src.count("cannot be handed over") == 1   # the resident share's hand-over refusal
    for fn in ("open_image_source", "open_file_store", "close_file_store"):   # call sites, not the definition
        assert len(re.findall(r"(?<!int )\b%s\(" % fn, src)) == 1, fn
    assert src.count('tl_add("file_io"') == 1
    assert image.count("direct_chunk(e)") == 1


def test_engine_uses_the_tested_header():
    csrc = os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "csrc")
    read = {f: open(os.path.join(csrc, f)).read() for f in ("fma_internal.h", "fma_engine.cu", "fma_sleep.cu", "fma_wake.cu")}
    src = "".join(read.values())
    assert '#include "fma_layout.h"' in src and "fma_layout::plan_runs(" in src and "fma_layout::arena_take(" in src
    for f in ("fma_sleep.cu", "fma_wake.cu"):   # every copy pipeline takes its pages, batches and chunk queues from the header
        for fn in ("fma_layout::plan_pages(", "fma_layout::plan_batches(", "fma_layout::ChunkQueues "):
            assert fn in read[f], (f, fn)
    assert "fma_layout::next_batch(" in read["fma_wake.cu"] and "fma_layout::resident_split(" in read["fma_sleep.cu"]
    for f in ("fma_sleep.cu", "fma_wake.cu"):   # no pipeline plans by hand any more
        for local in ("struct Dst", "struct Slot", "struct Chunk", "struct ResPiece", "need_item"):
            assert local not in read[f], (f, local)
    # the pipeline each sleep / wake runs is chosen by the header's routes, and the two functions are short orchestrators
    assert "fma_layout::sleep_route(" in read["fma_sleep.cu"] and "fma_layout::wake_route(" in read["fma_wake.cu"]
    assert "int resolve_mode(" not in read["fma_engine.cu"] + read["fma_internal.h"]
    wake_pipe = read["fma_wake.cu"].split("struct WakePipe {", 1)[1].split("\n};", 1)[0]
    assert "std::function" not in wake_pipe
    for f, fn in (("fma_sleep.cu", "int do_sleep("), ("fma_wake.cu", "int do_wake(")):
        body = read[f].split(fn, 1)[1].split("\n}\n", 1)[0]
        for local in ("MapProgress", "partial_packed", "pre_planned"):
            assert local not in body, (fn, local)
