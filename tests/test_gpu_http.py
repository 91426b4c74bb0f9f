"""The controller's three HTTP calls against an engine on a real H100 (SURVEY.md section 8 a9 / B1).

The dual-pods controller drives an inference server with exactly POST /sleep (inference-server.go:1329-1339, default client, must
be 200), GET /is_sleeping (:1595-1607) and POST /wake_up (:1118-1137, 5 s timeout, retried => must be idempotent); the executable
spec of the server side is cmd/test-server/main.go:69-91.  Here those calls go over a real socket into (a) ``fma_b200.server`` —
the FastAPI mirror of vLLM's dev-mode routes — on top of an Engine that holds K0-filled weights on cuda:0, and (b) the compiled
``fma_served`` (csrc/fma_served.cpp), and what the engine moved is compared with the ORACLE: the host image bytes after /sleep,
the weight bytes and K3 digests after /wake_up, device addresses unchanged."""
import ctypes as C
import json
import os
import socket
import subprocess
import threading
import time
import urllib.error
import urllib.request

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _call(base, method, path, timeout=60):
    req = urllib.request.Request(base + path, data=b"" if method == "POST" else None, method=method)
    try:
        with urllib.request.urlopen(req, timeout=timeout) as r:
            return r.status, r.read()
    except urllib.error.HTTPError as e:
        return e.code, e.read()


def test_controller_sequence_over_http_moves_the_bytes_the_oracle_says(engine, oracle):
    import uvicorn

    from fma_b200 import workloads as W
    from fma_b200.server import EngineBackend, create_app

    table = W.allocation_table("tiny-llama-test", kv_cache_bytes=32 << 20, kv_tensors=2)
    ptrs = [engine.alloc(s.bytes, s.tag) for s in table]
    ref, first = {}, 0
    for i, s in enumerate(table):
        if s.tag == "weights":
            engine.fill(i, 1234, first)
            ref[i] = oracle.fill(s.bytes, 1234, first)
            first += s.bytes // 8
    want_digests = {i: oracle.digest(ref[i]) for i in ref}
    image = oracle.packed_image([ref[i] for i in sorted(ref)])

    port = _free_port()
    server = uvicorn.Server(uvicorn.Config(create_app(EngineBackend([engine])), host="127.0.0.1", port=port, log_level="warning"))
    th = threading.Thread(target=server.run, daemon=True)
    th.start()
    base = f"http://127.0.0.1:{port}"
    try:
        for _ in range(200):
            try:
                if _call(base, "GET", "/health", timeout=2)[0] == 200:
                    break
            except Exception:
                time.sleep(0.05)
        assert json.loads(_call(base, "GET", "/is_sleeping")[1]) == {"is_sleeping": False}
        for cycle in range(2):
            # ensureUnbound: POST /sleep must answer exactly 200, only when every byte is in the store
            assert _call(base, "POST", "/sleep") == (200, b"")
            assert json.loads(_call(base, "GET", "/is_sleeping")[1]) == {"is_sleeping": True}
            st = engine.stats()
            assert engine.is_sleeping() and st["hbm_mapped_bytes"] == 0 and st["sleep_bytes_offloaded"] == image.size
            hb, n = engine.host_store_view()
            got = np.ctypeslib.as_array((C.c_uint8 * n).from_address(hb))
            assert n == image.size and np.array_equal(got, image), "host image after POST /sleep != the oracle's gather"
            assert _call(base, "POST", "/sleep") == (200, b"")                       # sleeping twice is harmless (abstract.py:323-325)
            # wakeSleeper: 5 s timeout, retried by the controller -> twice
            t0 = time.perf_counter()
            assert _call(base, "POST", "/wake_up", timeout=5) == (200, b"")
            assert time.perf_counter() - t0 < 5.0
            assert _call(base, "POST", "/wake_up", timeout=5) == (200, b"")
            assert json.loads(_call(base, "GET", "/is_sleeping")[1]) == {"is_sleeping": False}
            assert [s.va for s in engine.segments()] == ptrs
            dg = engine.digest_all(["weights"])
            assert all(dg[i] == want_digests[i] for i in ref)
            for i in ref:
                assert engine.read(i, table[i].bytes) == ref[i].tobytes()
        # vLLM API compatibility the controller never uses: level 2, tag-selective wake
        assert _call(base, "POST", "/sleep?level=2&mode=abort")[0] == 200
        assert engine.stats()["sleep_bytes_offloaded"] == 0
        assert _call(base, "POST", "/wake_up?tags=weights")[0] == 200
        assert json.loads(_call(base, "GET", "/is_sleeping")[1])["is_sleeping"] is True
        assert _call(base, "POST", "/wake_up?tags=kv_cache")[0] == 200
        assert json.loads(_call(base, "GET", "/is_sleeping")[1])["is_sleeping"] is False
    finally:
        server.should_exit = True
        th.join(timeout=20)


def test_compiled_server_over_http_matches_oracle_digests(built, oracle):
    """csrc/fma_served.cpp (the compiled host side over the C-ABI, the reference's cmd/test-server with engines instead of an
    atomic bool) on the real device: K3 digests served over HTTP == oracle digests of the oracle's K0 fill, before and after
    the controller's sleep -> wake sequence."""
    exe = os.path.join(ROOT, "llm-d-fast-model-actuation_b200", "fma_served")
    if os.environ.get("FMA_HOSTSIM") == "1":
        pytest.skip("the product binary links the CUDA library (the host-simulated build is tests/test_engine_hostsim.py)")
    if not os.path.exists(exe):
        pytest.skip("fma_served not built")
    mib = [6, 2, 4]            # --seg <tag>:<MiB>
    p = subprocess.Popen([exe, "--port", "0", "--device", "0", "--seg", "weights:6", "--seg", "weights:2", "--seg", "kv_cache:8", "--seg", "weights:4",
                          "--seed", "1234"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        line = p.stdout.readline()
        assert line.startswith("listening on "), line + p.stderr.read()
        base = f"http://127.0.0.1:{int(line.split()[-1])}"
        want, first = [], 0
        for n in mib:
            want.append(oracle.digest(oracle.fill(n << 20, 1234, first)))
            first += (n << 20) // 8
        st, body = _call(base, "GET", "/digests")
        assert st == 200 and [int(x, 16) for x in json.loads(body)[0]] == want, body
        assert _call(base, "POST", "/sleep") == (200, b"")
        assert json.loads(_call(base, "GET", "/is_sleeping")[1]) == {"is_sleeping": True}
        stats = json.loads(_call(base, "GET", "/stats")[1])
        assert stats["ranks"][0]["sleep_bytes_offloaded"] == sum(mib) << 20 and stats["ranks"][0]["hbm_mapped_bytes"] == 0
        assert _call(base, "POST", "/wake_up", timeout=5) == (200, b"") and _call(base, "POST", "/wake_up", timeout=5) == (200, b"")
        assert json.loads(_call(base, "GET", "/is_sleeping")[1]) == {"is_sleeping": False}
        st, body = _call(base, "GET", "/digests")
        assert st == 200 and [int(x, 16) for x in json.loads(body)[0]] == want
    finally:
        p.terminate()
        try:
            p.wait(timeout=30)
        except subprocess.TimeoutExpired:
            p.kill()
    assert p.returncode == 0, p.stderr.read()[-2000:]
