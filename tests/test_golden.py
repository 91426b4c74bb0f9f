"""The oracle vs the golden fixture produced by the reference data path itself (vLLM's CuMemAllocator run
on an H100 by tests/golden/make_vllm_cumem_golden.py): weight bytes after the reference's sleep -> wake are
exactly the bytes that went in, at the same device addresses; segment sizes follow the 2 MiB rounding the
allocation tables assume; non-offloaded tags do not come back."""
import hashlib
import json
import os

import fma_b200  # noqa: F401
from fma_b200 import workloads as W

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "vllm_cumem_roundtrip.json")


def test_reference_roundtrip_is_identity_on_oracle_bytes(oracle):
    g = json.load(open(GOLDEN))
    assert g["same_device_addresses"] is True
    tensors = W.model_tensors(g["model"])
    assert [(w["name"], w["bytes"]) for w in g["weights"]] == [(n, b) for n, b in tensors]
    first = 0
    for w in g["weights"]:
        assert w["first_word"] == first
        buf = oracle.fill(w["bytes"], g["seed"], first)
        assert hashlib.sha256(buf.tobytes()).hexdigest() == w["sha256"]
        assert oracle.digest(buf, first) == w["oracle_digest"]
        first += w["bytes"] // 8


def test_reference_segment_sizes_match_the_table_model():
    """What torch + vLLM's allocator really produced for these tensors == workloads.simulate_segments."""
    g = json.load(open(GOLDEN))
    mine = W.simulate_segments(W.model_tensors(g["model"]), "weights") + \
        W.simulate_segments([(n, b) for n, b in g["kv_specs"]], "kv_cache")
    assert sorted((s["bytes"], s["tag"]) for s in g["reference_segments"]) == sorted((s.bytes, s.tag) for s in mine)


def test_reference_does_not_restore_discarded_tags():
    g = json.load(open(GOLDEN))
    assert g["kv_cache"] and not any(k["restored"] for k in g["kv_cache"])
