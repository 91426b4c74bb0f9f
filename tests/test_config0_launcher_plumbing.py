"""BASELINE config 0 (plumbing, no GPU): the launcher-compatible node agent (scripts/run_node_agent.py; its REST contract is
pinned to the reference launcher's answers by tests/test_node_agent_differential.py) creates an instance from the same JSON
the Go controller sends (pkg/controller/dual-pods/launcherclient.go:72-78), forks the child, and the controller's
sleep -> is_sleeping -> wake_up sequence works against the child's port.
The child is the route-compatible stand-in of SURVEY.md §8c-iv (CPU-worker semantics: nothing moves)."""
import json
import os
import socket
import subprocess
import sys
import time
import urllib.error
import urllib.request


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAUNCHER = os.path.join(ROOT, "scripts", "run_node_agent.py")


def _port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _http(method, url, body=None, timeout=10):
    data = json.dumps(body).encode() if body is not None else (b"" if method in ("POST", "PUT") else None)
    req = urllib.request.Request(url, data=data, method=method, headers={"Content-Type": "application/json"})
    try:
        with urllib.request.urlopen(req, timeout=timeout) as r:
            return r.status, r.read().decode()
    except urllib.error.HTTPError as e:
        return e.code, e.read().decode()


def _wait(url, seconds):
    t0 = time.time()
    while time.time() - t0 < seconds:
        try:
            if _http("GET", url, timeout=2)[0] == 200:
                return True
        except Exception:
            pass
        time.sleep(0.3)
    return False


def test_launcher_compatible_agent_drives_sleep_wake(built, tmp_path):
    lport, vport = _port(), _port()
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "scripts", "vllm_cpu_standin"), os.path.join(ROOT, "scripts", "k8s_stub"),
                                         ROOT, env.get("PYTHONPATH", "")])
    log = open(tmp_path / "launcher.log", "w")
    proc = subprocess.Popen([sys.executable, LAUNCHER, "--mock-gpus", "--mock-gpu-count", "1", "--host", "127.0.0.1", "--port", str(lport)],
                            env=env, cwd=os.path.dirname(LAUNCHER), stdout=log, stderr=subprocess.STDOUT)
    try:
        assert _wait(f"http://127.0.0.1:{lport}/health", 60), open(tmp_path / "launcher.log").read()[-2000:]
        body = {"options": f"--model facebook/opt-125m --enable-sleep-mode --port {vport} --host 127.0.0.1",
                "env_vars": {"VLLM_SERVER_DEV_MODE": "1"}, "annotations": {"isc-name": "cfg0", "inference-port": str(vport)}}
        st, txt = _http("PUT", f"http://127.0.0.1:{lport}/v2/vllm/instances/cfg0", body)
        assert st == 201, txt
        assert json.loads(txt)["instance_id"] == "cfg0"
        assert _http("PUT", f"http://127.0.0.1:{lport}/v2/vllm/instances/cfg0", body)[0] == 409          # duplicate id
        assert _wait(f"http://127.0.0.1:{vport}/health", 60)
        st, txt = _http("GET", f"http://127.0.0.1:{lport}/v2/vllm/instances")
        listing = json.loads(txt)
        assert listing["running_instances"] == 1 and listing["instances"][0]["status"] == "running"
        base = f"http://127.0.0.1:{vport}"
        assert json.loads(_http("GET", base + "/is_sleeping")[1]) == {"is_sleeping": False}
        assert _http("POST", base + "/sleep")[0] == 200                                                   # ensureUnbound
        assert json.loads(_http("GET", base + "/is_sleeping")[1]) == {"is_sleeping": True}                # querySleeping
        assert 200 <= _http("POST", base + "/wake_up")[0] < 300                                           # wakeSleeper
        assert 200 <= _http("POST", base + "/wake_up")[0] < 300                                           # retried: harmless
        assert json.loads(_http("GET", base + "/is_sleeping")[1]) == {"is_sleeping": False}
        assert _http("DELETE", f"http://127.0.0.1:{lport}/v2/vllm/instances/cfg0")[0] == 200
        assert _http("DELETE", f"http://127.0.0.1:{lport}/v2/vllm/instances/cfg0")[0] == 404
    finally:
        proc.terminate()
        try:
            proc.wait(timeout=20)
        except Exception:
            proc.kill()
