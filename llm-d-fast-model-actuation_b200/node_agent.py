"""Node agent: a launcher-compatible REST service that OWNS the node's inference-server instances (SURVEY.md §8f-1).

Wire-compatible with the reference launcher (inference_server/launcher/launcher.py:558-790; Go mirror
pkg/controller/dual-pods/launcherclient.go:72-98) — same paths, status codes and JSON shapes, pinned by differential
tests against the live, unmodified launcher (tests/test_node_agent_differential.py):

    GET    /health                              200 {"status": "OK"}
    PUT    /v2/vllm/instances/{id}              201 state | 409 duplicate      body: VllmConfig{options,gpu_uuids?,env_vars?,annotations?}
    POST   /v2/vllm/instances                   201 state (generated id)
    GET    /v2/vllm/instances[?detail=false]    200 {revision,total_instances,running_instances,instances:[state]}
    GET    /v2/vllm/instances/{id}              200 state | 404
    DELETE /v2/vllm/instances/{id}              200 state("terminated"/"not_running") | 404
    DELETE /v2/vllm/instances                   200 {"status":"all_stopped",...}
    GET    /v2/vllm/instances/{id}/log          200 | 206 (Range: bytes=a-[b]) | 416 (Content-Range: bytes */N) | 400 | 404
    GET    /v2/vllm/instances/watch[?since=N]   NDJSON {"type":"CREATED|STOPPED|DELETED","object":state}, 410 if N fell out of the buffer

What it adds — the reason a node-level owner exists (BASELINE configs 4 and 5) — are node-scoped actuation routes that
fan the three dev-mode calls out to instance ports and can run them CONCURRENTLY across instances, which two
independent controller reconciles never do (SURVEY.md §3.4):

    POST /v2/vllm/instances/{id}/sleep | /wake_up     proxy to the instance's inference port, returns seconds
    GET  /v2/vllm/instances/{id}/is_sleeping
    POST /v2/node/swap {"sleep": idA, "wake": idB}     sleep(A) || wake(B): D2H of A and H2D of B on opposite PCIe directions
    GET  /v2/node/sleepers                             who sleeps where (for sleeper budgets)
    GET  /v2/node/images                               images kept for dead instances: peer HBM, host DRAM, disk (parking.py)

Design differences from the reference (this is not a port): instances are forked by a single-threaded *fork server*
that has pre-imported the serving stack (the reference forks from its asyncio server process), exits are observed by
one waiter thread per child (no event-loop fd readers), state lives behind one lock + condition variable, and the watch
stream is a plain generator.  Children run exactly what the reference's child runs: env applied, ``options.split()``
parsed by vLLM's own parser, ``run_server(args)``.
"""
from __future__ import annotations

import argparse
import asyncio
import collections
import json
import logging
import multiprocessing
import os
import re
import signal
import sys
import threading
import time
import urllib.error
import urllib.request
import uuid
from typing import Dict, List, Optional

from fastapi import FastAPI, Header, HTTPException, Query
from fastapi.responses import JSONResponse, Response, StreamingResponse
from pydantic import BaseModel

logger = logging.getLogger("fma_b200.node_agent")

MAX_LOG_RESPONSE_BYTES = 1024 * 1024     # launcher.py: default window of a log read
MAX_EVENTS = 1000                         # watch buffer depth
ISC_PORT_ANNOTATION = "inference-port"    # launcherclient.go:49


class VllmConfig(BaseModel):              # launcher.py:60-64 / launcherclient.go:72-78
    options: str
    gpu_uuids: Optional[List[str]] = None
    env_vars: Optional[Dict[str, str]] = None
    annotations: Optional[Dict[str, str]] = None


class SwapRequest(BaseModel):
    sleep: str
    wake: str


# ------------------------------------------------------------------------------------------------------------------
# child process
# ------------------------------------------------------------------------------------------------------------------
def _child_main(config: dict, log_path: str, extra_env: Optional[Dict[str, str]] = None) -> None:
    """What runs in the forked child — same steps as the reference's ``vllm_kickoff`` (launcher.py:799-837)."""
    os.setpgrp()                                          # own process group: SIGKILL can take EngineCore along
    fd = os.open(log_path, os.O_WRONLY | os.O_CREAT | os.O_APPEND, 0o644)
    os.dup2(fd, 1); os.dup2(fd, 2); os.close(fd)
    sys.stdout = os.fdopen(1, "w", buffering=1); sys.stderr = os.fdopen(2, "w", buffering=1)
    for k, v in (extra_env or {}).items():
        os.environ.setdefault(k, v)
    for k, v in (config.get("env_vars") or {}).items():
        os.environ[k] = v
    from vllm.entrypoints.openai.api_server import run_server
    from vllm.entrypoints.openai.cli_args import make_arg_parser, validate_parsed_serve_args
    from vllm.entrypoints.utils import cli_env_setup
    from vllm.utils.argparse_utils import FlexibleArgumentParser

    cli_env_setup()
    parser = make_arg_parser(FlexibleArgumentParser(description="vLLM OpenAI-Compatible RESTful API server."))
    args = parser.parse_args(config["options"].split())
    validate_parsed_serve_args(args)
    try:
        import uvloop

        uvloop.run(run_server(args))
    except ImportError:
        import asyncio

        asyncio.run(run_server(args))


def _translate_gpu_uuids(uuids: List[str], mock: bool) -> List[str]:
    """UUID -> CUDA index (gputranslator.py:135-195): NVML in real mode, ``GPU-<i>`` in mock mode."""
    if mock:
        out = []
        for u in uuids:
            m = re.fullmatch(r"GPU-(\d+)", u)
            if not m:
                raise ValueError(f"unknown mock GPU UUID {u}")
            out.append(m.group(1))
        return out
    import pynvml

    pynvml.nvmlInit()
    table = {}
    for i in range(pynvml.nvmlDeviceGetCount()):
        u = pynvml.nvmlDeviceGetUUID(pynvml.nvmlDeviceGetHandleByIndex(i))
        table[u.decode() if isinstance(u, bytes) else u] = str(i)
    missing = [u for u in uuids if u not in table]
    if missing:
        raise ValueError(f"GPU UUID(s) not on this node: {missing}")
    return [table[u] for u in uuids]


# ------------------------------------------------------------------------------------------------------------------
# agent
# ------------------------------------------------------------------------------------------------------------------
class _Instance:
    def __init__(self, instance_id: str, config: VllmConfig, log_dir: str):
        self.id = instance_id
        self.config = config
        self.proc: multiprocessing.process.BaseProcess | None = None
        self.revision: int | None = None
        self.log_path = os.path.join(log_dir, f"node-agent-{os.getpid()}-vllm-{instance_id}.log")
        self.deleting = False

    def state(self, status: str | None = None) -> dict:
        if status is None:
            status = "running" if self.proc is not None and self.proc.is_alive() else "stopped"
        return {"status": status, "instance_id": self.id, "revision": self.revision, **self.config.model_dump(exclude_none=True)}

    def inference_port(self) -> int:
        ann = self.config.annotations or {}
        if ISC_PORT_ANNOTATION in ann:
            return int(ann[ISC_PORT_ANNOTATION])
        m = re.search(r"--port[ =](\d+)", self.config.options)
        if not m:
            raise KeyError(f"instance {self.id}: no inference port (annotation {ISC_PORT_ANNOTATION!r} or --port)")
        return int(m.group(1))


class NodeAgent:
    def __init__(self, mock_gpus: bool = False, log_dir: str = "/tmp", start_method: str = "forkserver",
                 preload: tuple[str, ...] = ("vllm.entrypoints.openai.api_server",), parking=None):
        self.mock_gpus = mock_gpus
        self.log_dir = log_dir
        self.parking = parking                     # parking.ParkingService (node-level owner of peer-HBM images), or None
        self._lock = threading.Condition()
        self._instances: Dict[str, _Instance] = {}
        self._revision = 0
        self._events: collections.deque = collections.deque(maxlen=MAX_EVENTS)   # (revision, type, object)
        self._ctx = multiprocessing.get_context(start_method)
        if start_method == "forkserver":
            # the serving stack is imported ONCE, in the fork server; every instance starts as a fork of it
            self._ctx.set_forkserver_preload(list(preload))

    # ---- events ---------------------------------------------------------------------------------------------
    @property
    def revision(self) -> int:
        return self._revision

    def _publish(self, inst: _Instance, kind: str, obj: dict) -> None:   # caller holds the lock
        self._events.append((obj["revision"], kind, obj))
        self._lock.notify_all()

    def oldest_revision(self) -> int:
        """Exclusive lower bound of what the buffer still holds."""
        return self._revision - len(self._events)

    def watch_start(self, since: Optional[int]) -> tuple[int, List[str]]:
        """Cursor + the lines a fresh watcher gets first: a CREATED event per existing instance (launcher.py:617-627)."""
        with self._lock:
            if since is not None:
                return since, []
            return self._revision, [json.dumps({"type": "CREATED", "object": i.state()}) + "\n" for i in self._instances.values()]

    def events_after(self, pos: int) -> Optional[tuple[int, List[str]]]:
        """Events with revision > pos as NDJSON lines and the new cursor; None if pos fell out of the buffer."""
        with self._lock:
            if pos < self.oldest_revision():
                return None
            lines = [json.dumps({"type": k, "object": o}) + "\n" for (r, k, o) in self._events if r > pos]
            return self._revision, lines

    # ---- lifecycle ------------------------------------------------------------------------------------------
    def create(self, config: VllmConfig, instance_id: Optional[str] = None) -> dict:
        instance_id = instance_id or str(uuid.uuid4())
        with self._lock:
            if instance_id in self._instances:
                raise ValueError(f"Instance with ID {instance_id} already exists")
            cfg = config.model_copy(deep=True)
            extra_env: Dict[str, str] = {}    # for the child only: never part of the reported state (the wire contract is the launcher's)
            if cfg.gpu_uuids:
                idx = _translate_gpu_uuids(cfg.gpu_uuids, self.mock_gpus)
                cfg.env_vars = dict(cfg.env_vars or {})
                cfg.env_vars["CUDA_VISIBLE_DEVICES"] = ",".join(idx)
                extra_env["FMA_NODE_GPU_INDICES"] = ",".join(idx)      # node-level indices: where NOT to park this model
            if self.parking is not None:   # the instance's allocator shim parks on buffers THIS process owns (parking.py)
                extra_env["FMA_NODE_AGENT_SOCK"] = self.parking.sock_path
                extra_env["FMA_INSTANCE_ID"] = instance_id
                if self.parking.keep_dir:
                    extra_env["FMA_KEEP_DIR"] = self.parking.keep_dir
                    for var, n in (("FMA_KEEP_DISK_GIB", self.parking.keep_disk_bytes), ("FMA_KEEP_DRAM_GIB", self.parking.keep_dram_bytes)):
                        if n is not None:
                            extra_env[var] = str(n / (1 << 30))
            inst = _Instance(instance_id, cfg, self.log_dir)
            open(inst.log_path, "wb").close()
            inst.proc = self._ctx.Process(target=_child_main, args=(cfg.model_dump(exclude_none=True), inst.log_path, extra_env), daemon=False)
            inst.proc.start()
            self._instances[instance_id] = inst
            self._revision += 1
            inst.revision = self._revision
            result = inst.state()
            self._publish(inst, "CREATED", result)
        threading.Thread(target=self._wait_exit, args=(inst,), name=f"exit-{instance_id}", daemon=True).start()
        return result

    def _exited(self, inst: _Instance) -> None:
        """The instance's process is gone: the parking service settles the image files it deposited and the leases it held."""
        if self.parking is not None:
            try:
                self.parking.instance_exited(inst.id)
            except Exception as e:      # noqa: BLE001 — bookkeeping must not break the instance's lifecycle
                logger.warning("exit hook of instance %s failed: %s", inst.id, e)

    def _wait_exit(self, inst: _Instance) -> None:
        inst.proc.join()
        if not inst.deleting:
            self._exited(inst)
        with self._lock:
            if inst.deleting or self._instances.get(inst.id) is not inst:
                return                                                # a DELETE is reporting this exit
            self._revision += 1
            inst.revision = self._revision
            obj = inst.state("stopped")
            obj["exit_code"] = inst.proc.exitcode
            self._publish(inst, "STOPPED", obj)

    def stop(self, instance_id: str, timeout: float = 10.0) -> dict:
        with self._lock:
            inst = self._instances.get(instance_id)
            if inst is None:
                raise KeyError(instance_id)
            inst.deleting = True
        was_alive = inst.proc.is_alive()
        if was_alive:
            inst.proc.terminate()                                     # SIGTERM first (vLLM shuts its engine core down)
            inst.proc.join(timeout)
            if inst.proc.is_alive():
                try:
                    os.killpg(inst.proc.pid, signal.SIGKILL)          # then the whole process group
                except ProcessLookupError:
                    pass
                inst.proc.join()
        self._exited(inst)
        try:
            os.unlink(inst.log_path)
        except FileNotFoundError:
            pass
        with self._lock:
            self._revision += 1
            inst.revision = self._revision
            result = inst.state("stopped")
            self._instances.pop(instance_id, None)
            self._publish(inst, "DELETED", result)
        return result

    def stop_all(self, timeout: float = 10.0) -> dict:
        results = []
        for iid in list(self._instances):
            try:
                results.append(self.stop(iid, timeout))
            except KeyError:
                continue
        return {"status": "all_stopped", "stopped_instances": results, "total_stopped": len(results)}

    # ---- queries --------------------------------------------------------------------------------------------
    def get(self, instance_id: str) -> _Instance:
        with self._lock:
            if instance_id not in self._instances:
                raise KeyError(instance_id)
            return self._instances[instance_id]

    def all_status(self) -> dict:
        with self._lock:
            states = [i.state() for i in self._instances.values()]
            return {"revision": self._revision, "total_instances": len(states),
                    "running_instances": sum(1 for s in states if s["status"] == "running"), "instances": states}

    def ids(self) -> dict:
        with self._lock:
            ids = list(self._instances)
            return {"revision": self._revision, "instance_ids": ids, "count": len(ids)}

    def log_bytes(self, instance_id: str, start: int, end: Optional[int]) -> tuple[bytes, int]:
        inst = self.get(instance_id)
        try:
            total = os.path.getsize(inst.log_path)
        except FileNotFoundError:
            total = 0
        if start >= total:
            raise LogRangeNotAvailable(total)
        last = min(start + MAX_LOG_RESPONSE_BYTES - 1 if end is None else end, total - 1)
        with open(inst.log_path, "rb") as f:
            f.seek(start)
            return f.read(last - start + 1), total

    # ---- node-scoped actuation (what a per-instance controller cannot do) -----------------------------------------
    def _call(self, inst: _Instance, method: str, path: str, timeout: float = 600.0) -> tuple[int, str, float]:
        url = f"http://127.0.0.1:{inst.inference_port()}{path}"
        req = urllib.request.Request(url, data=b"" if method == "POST" else None, method=method)
        t0 = time.perf_counter()
        try:
            with urllib.request.urlopen(req, timeout=timeout) as r:
                return r.status, r.read().decode(), time.perf_counter() - t0
        except urllib.error.HTTPError as e:
            return e.code, e.read().decode(), time.perf_counter() - t0

    def actuate(self, instance_id: str, what: str) -> dict:
        inst = self.get(instance_id)
        status, body, secs = self._call(inst, "GET" if what == "is_sleeping" else "POST", "/" + what)
        out = {"instance_id": instance_id, "action": what, "status_code": status, "seconds": round(secs, 6)}
        if what == "is_sleeping" and status == 200:
            out.update(json.loads(body))
        return out

    def swap(self, sleep_id: str, wake_id: str) -> dict:
        """sleep(A) and wake_up(B) at the same time: the two instances are separate processes with separate engines, so
        A's D2H and B's H2D run on opposite PCIe directions (in-process equivalent: fma_swap)."""
        a, b = self.get(sleep_id), self.get(wake_id)
        res: dict = {}

        def run(key, inst, path):
            res[key] = self._call(inst, "POST", path)

        t0 = time.perf_counter()
        ts = [threading.Thread(target=run, args=("sleep", a, "/sleep")), threading.Thread(target=run, args=("wake", b, "/wake_up"))]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        return {"sleep": {"instance_id": sleep_id, "status_code": res["sleep"][0], "seconds": round(res["sleep"][2], 6)},
                "wake": {"instance_id": wake_id, "status_code": res["wake"][0], "seconds": round(res["wake"][2], 6)},
                "seconds": round(time.perf_counter() - t0, 6)}

    def sleepers(self) -> dict:
        out = []
        for iid in list(self._instances):
            try:
                inst = self.get(iid)
                st = self.actuate(iid, "is_sleeping")
                out.append({"instance_id": iid, "is_sleeping": st.get("is_sleeping"),
                            "cuda_visible_devices": (inst.config.env_vars or {}).get("CUDA_VISIBLE_DEVICES")})
            except Exception as e:  # an instance that is still starting has no port yet
                out.append({"instance_id": iid, "is_sleeping": None, "error": str(e)[:120]})
        res = {"sleepers": out, "sleeping_count": sum(1 for s in out if s.get("is_sleeping"))}
        if self.parking is not None:
            # what a sleeper costs in HBM, per GPU index, in MiB — the unit accelMemoryIsLowEnough compares against
            # (inference-server.go:1609-1636; budget = count x 4096 MiB, cmd/dual-pods-controller/main.go:72-74)
            res.update(self.parking.stats())
        return res

    def images(self) -> dict:
        """Images kept for dead or future instances and the DRAM / disk budgets they count against (parking.py ``kept``)."""
        if self.parking is None:
            return {"images": [], "dram_bytes": 0, "dram_budget_bytes": None, "disk_bytes": 0, "disk_budget_bytes": None, "keep_dir": None}
        return self.parking.kept()


class LogRangeNotAvailable(Exception):
    def __init__(self, available: int):
        super().__init__()
        self.available = available


_RANGE = re.compile(r"^bytes=(\d+)-(\d*)$")


def parse_range(header: str) -> tuple[int, Optional[int]]:
    m = _RANGE.match(header.strip())
    if not m:
        raise ValueError(f"Unsupported or malformed Range header: {header}")
    start = int(m.group(1))
    end = int(m.group(2)) if m.group(2) else None
    if end is not None and end < start:
        raise ValueError(f"Range end ({end}) must be >= start ({start})")
    return start, end


# ------------------------------------------------------------------------------------------------------------------
# REST
# ------------------------------------------------------------------------------------------------------------------
def create_app(agent: NodeAgent) -> FastAPI:
    app = FastAPI()
    app.state.agent = agent

    @app.on_event("shutdown")
    def _shutdown():
        agent.stop_all()

    @app.get("/health")
    def health():
        return JSONResponse({"status": "OK"})

    @app.get("/")
    def index():
        return JSONResponse({"name": "H100 node agent (launcher-compatible instance management + node-scoped actuation)", "version": "2.0",
                             "endpoints": {"index": "GET /", "health": "GET /health",
                                           "create_instance": "POST /v2/vllm/instances",
                                           "create_named_instance": "PUT /v2/vllm/instances/{instance_id}",
                                           "delete_instance": "DELETE /v2/vllm/instances/{instance_id}",
                                           "delete_all_instances": "DELETE /v2/vllm/instances",
                                           "get_instance_status": "GET /v2/vllm/instances/{instance_id}",
                                           "get_all_instances": "GET /v2/vllm/instances",
                                           "get_instance_logs": "GET /v2/vllm/instances/{instance_id}/log",
                                           "watch_instances": "GET /v2/vllm/instances/watch",
                                           "sleep_instance": "POST /v2/vllm/instances/{instance_id}/sleep",
                                           "wake_instance": "POST /v2/vllm/instances/{instance_id}/wake_up",
                                           "swap": "POST /v2/node/swap", "sleepers": "GET /v2/node/sleepers",
                                           "images": "GET /v2/node/images"}})

    @app.get("/v2/vllm/instances/watch")
    async def watch(since: Optional[int] = Query(None)):
        if since is not None and since < agent.oldest_revision():
            raise HTTPException(status_code=410, detail=f"Requested revision {since} is no longer available. "
                                f"Oldest available: {agent.oldest_revision()}.")

        async def stream():
            pos, first = agent.watch_start(since)
            for line in first:
                yield line
            while True:                                   # cancelled by the server when the client goes away
                got = agent.events_after(pos)
                if got is None:
                    return
                pos, lines = got
                for line in lines:
                    yield line
                await asyncio.sleep(0.05)

        return StreamingResponse(stream(), media_type="application/x-ndjson", headers={"X-Content-Type-Options": "nosniff"})

    @app.post("/v2/vllm/instances")
    def create(cfg: VllmConfig):
        try:
            return JSONResponse(agent.create(cfg), status_code=201)
        except Exception as e:
            raise HTTPException(status_code=500, detail=str(e))

    @app.put("/v2/vllm/instances/{instance_id}")
    def create_named(instance_id: str, cfg: VllmConfig):
        try:
            return JSONResponse(agent.create(cfg, instance_id), status_code=201)
        except ValueError as e:
            raise HTTPException(status_code=409, detail=str(e))
        except Exception as e:
            raise HTTPException(status_code=500, detail=str(e))

    @app.delete("/v2/vllm/instances/{instance_id}")
    def delete(instance_id: str):
        try:
            return JSONResponse(agent.stop(instance_id))
        except KeyError:
            raise HTTPException(status_code=404, detail=f"Instance {instance_id} not found")

    @app.delete("/v2/vllm/instances")
    def delete_all():
        return JSONResponse(agent.stop_all())

    @app.get("/v2/vllm/instances")
    def list_all(detail: bool = True):
        return JSONResponse(agent.all_status() if detail else agent.ids())

    @app.get("/v2/vllm/instances/{instance_id}")
    def get_one(instance_id: str):
        try:
            return JSONResponse(agent.get(instance_id).state())
        except KeyError:
            raise HTTPException(status_code=404, detail=f"Instance {instance_id} not found")

    @app.get("/v2/vllm/instances/{instance_id}/log")
    def get_log(instance_id: str, range: Optional[str] = Header(None, alias="Range")):
        try:
            if range is None:
                start, end, partial = 0, None, False
            else:
                try:
                    start, end = parse_range(range)
                except ValueError as exc:
                    raise HTTPException(status_code=400, detail=str(exc))
                partial = True
            data, total = agent.log_bytes(instance_id, start, end)
            return Response(content=data, status_code=206 if partial else 200, media_type="application/octet-stream",
                            headers={"Accept-Ranges": "bytes", "Content-Range": f"bytes {start}-{start + len(data) - 1}/{total}"})
        except KeyError:
            raise HTTPException(status_code=404, detail=f"Instance {instance_id} not found")
        except LogRangeNotAvailable as e:
            return Response(content=b"", status_code=416, media_type="application/octet-stream",
                            headers={"Content-Range": f"bytes */{e.available}"})

    # ---- node-scoped actuation ------------------------------------------------------------------------------------
    def _act(instance_id: str, what: str):
        try:
            return JSONResponse(agent.actuate(instance_id, what))
        except KeyError as e:
            raise HTTPException(status_code=404, detail=str(e))
        except Exception as e:
            raise HTTPException(status_code=502, detail=f"instance {instance_id} did not answer: {e}")

    @app.post("/v2/vllm/instances/{instance_id}/sleep")
    def sleep_one(instance_id: str):
        return _act(instance_id, "sleep")

    @app.post("/v2/vllm/instances/{instance_id}/wake_up")
    def wake_one(instance_id: str):
        return _act(instance_id, "wake_up")

    @app.get("/v2/vllm/instances/{instance_id}/is_sleeping")
    def is_sleeping_one(instance_id: str):
        return _act(instance_id, "is_sleeping")

    @app.post("/v2/node/swap")
    def swap(req: SwapRequest):
        try:
            return JSONResponse(agent.swap(req.sleep, req.wake))
        except KeyError as e:
            raise HTTPException(status_code=404, detail=str(e))
        except Exception as e:
            raise HTTPException(status_code=502, detail=str(e))

    @app.get("/v2/node/sleepers")
    def sleepers():
        return JSONResponse(agent.sleepers())

    @app.get("/v2/node/images")
    def images():
        return JSONResponse(agent.images())

    return app


def keep_settings(env) -> dict:
    """Kept image files (parking.py), opt-in: FMA_KEEP_DIR (default: ``kept`` under FMA_FILE_DIR, the children's file-tier directory,
    so a kept file is a rename away), FMA_KEEP_DISK_GIB and FMA_KEEP_DRAM_GIB (unset: no bound)."""
    keep_dir = env.get("FMA_KEEP_DIR") or (os.path.join(env["FMA_FILE_DIR"], "kept") if env.get("FMA_FILE_DIR") else None)
    gib = lambda v: int(float(env[v]) * (1 << 30)) if env.get(v) else None    # noqa: E731
    return {"keep_dir": keep_dir, "keep_disk_bytes": gib("FMA_KEEP_DISK_GIB"), "keep_dram_bytes": gib("FMA_KEEP_DRAM_GIB")}


def main() -> None:
    import uvicorn

    ap = argparse.ArgumentParser(description="H100 node agent (launcher-compatible)")
    ap.add_argument("--mock-gpus", action="store_true")
    ap.add_argument("--mock-gpu-count", type=int, default=8)   # accepted for CLI compatibility with launcher.py:857-899
    ap.add_argument("--host", default="0.0.0.0")
    ap.add_argument("--port", type=int, default=8001)          # pkg/controller/common/interface.go:38
    ap.add_argument("--log-level", default="info", choices=["critical", "error", "warning", "info", "debug"])
    ap.add_argument("--log-dir", default="/tmp")
    ap.add_argument("--parking", action="store_true", help="own the node's peer-HBM parking buffers (parking.py): instances started by this agent "
                                                           "park sleeping weights on idle GPUs through it and the images outlive them")
    a = ap.parse_args()
    logging.basicConfig(level=getattr(logging, a.log_level.upper()), format="%(asctime)s - %(name)s - %(levelname)s - %(message)s")
    parking = None
    if a.parking:
        from .parking import ParkingService

        if a.mock_gpus:
            n_dev = a.mock_gpu_count
        else:
            import pynvml

            pynvml.nvmlInit()
            n_dev = pynvml.nvmlDeviceGetCount()
        parking = ParkingService(os.path.join(a.log_dir, f"fma_node_agent.{os.getpid()}.sock"), n_devices=n_dev, **keep_settings(os.environ))
        parking.start()
    agent = NodeAgent(mock_gpus=a.mock_gpus, log_dir=a.log_dir, parking=parking)
    uvicorn.run(create_app(agent), host=a.host, port=a.port, log_level=a.log_level)


if __name__ == "__main__":
    main()
