"""End-to-end drop-in check on a GPU machine (SURVEY.md §7 step 7, BASELINE.md §3): the UNMODIFIED reference launcher
(inference_server/launcher/ of a reference checkout, named by REFERENCE_LAUNCHER_DIR) forks a real vLLM server with a dummy-weight
Llama model; the same HTTP calls the dual-pods controller makes (`POST /sleep`, `GET /is_sleeping`, `POST /wake_up`,
pkg/controller/dual-pods/inference-server.go:1329-1339,1595-1607,1118-1137) are timed by wall clock, once with vLLM's
own allocator and once with FMA_B200=1 in the instance's env_vars (-> plugin/ -> fma_b200.cumem).  A generation
request before sleep and after wake must return identical tokens (greedy), i.e. the weights came back bit-identical."""
import json, os, subprocess, sys, time, urllib.request, urllib.error

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = sys.argv[1] if len(sys.argv) > 1 else "llama-3-8b"
TP = int(sys.argv[2]) if len(sys.argv) > 2 else 1
CFGS = {
    "llama-3-8b": dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8, vocab_size=128256),
    "llama-1b": dict(hidden_size=2048, intermediate_size=8192, num_hidden_layers=16, num_attention_heads=32, num_key_value_heads=8, vocab_size=128256),
}
mdir = f"/tmp/fma_models/{MODEL}"; os.makedirs(mdir, exist_ok=True)
cfg = dict(architectures=["LlamaForCausalLM"], model_type="llama", hidden_act="silu", max_position_embeddings=8192, rms_norm_eps=1e-5,
           rope_theta=500000.0, tie_word_embeddings=False, torch_dtype="bfloat16", bos_token_id=128000, eos_token_id=128001, **CFGS[MODEL])
json.dump(cfg, open(f"{mdir}/config.json", "w"))
OUT = os.path.join(ROOT, "gpurun_out", "e2e"); os.makedirs(OUT, exist_ok=True)
LAUNCHER_DIR = os.environ.get("REFERENCE_LAUNCHER_DIR", "")
LPORT, VPORT = 8001, 8005
# Arms (E2E_ARMS=comma list).  Default: vLLM's allocator vs the engine, dummy weights.  Extra arms:
#   fma_b200_packed  the engine with the PACKED host image (FMA_PACK=1; dummy weights are bf16 U(-1e-3, 1e-3): they code)
#   ckpt_default / ckpt_fma   a synthetic safetensors checkpoint of the same shape, loaded by vLLM's own loader vs
#                             --load-format fma (the engine's file -> HBM stream); both must generate the same tokens
ARMS = os.environ.get("E2E_ARMS", "reference,fma_b200").split(",")
#   fma_b200_peer_parked   (E2E_LAUNCHER=node_agent, >= 2 GPUs) the instance sees only GPU 0 (gpu_uuids -> CUDA_VISIBLE_DEVICES), sleeps to the
#                          peer tier through the node agent's parking service, is DELETED asleep, and a new instance with the same ID adopts the
#                          parked image at start-up (FMA_ADOPT_PARKED=1) and must generate the same tokens
ARM_ENV = {"reference": {}, "fma_b200": {"FMA_B200": "1"}, "fma_b200_packed": {"FMA_B200": "1", "FMA_PACK": "1"},
           "ckpt_default": {"FMA_B200": "1"}, "ckpt_fma": {"FMA_B200": "1"},
           "fma_b200_peer_parked": {"FMA_B200": "1", "FMA_TIER": "peer"}}
USE_AGENT = os.environ.get("E2E_LAUNCHER", "reference") == "node_agent"
ARM_LOAD = {"ckpt_default": "auto", "ckpt_fma": "fma"}


def write_checkpoint(path):
    """Random bf16 LlamaForCausalLM checkpoint (HF tensor names) in one safetensors file, written by the repo's own writer."""
    import numpy as np
    sys.path.insert(0, ROOT)
    import fma_b200  # noqa: F401
    from fma_b200 import loader
    c = CFGS[MODEL]; h, inter, L, nh, nkv, v = c["hidden_size"], c["intermediate_size"], c["num_hidden_layers"], c["num_attention_heads"], c["num_key_value_heads"], c["vocab_size"]
    hd = h // nh
    rng = np.random.default_rng(1234)
    def t(name, *shape, ones=False):
        n = int(np.prod(shape))
        if ones:
            a = np.full(n, 0x3F80, np.uint16)
        else:
            a = (rng.normal(0, 0.02, n).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        return (name, "BF16", tuple(shape), a.tobytes())
    def tensors():
        yield t("model.embed_tokens.weight", v, h)
        for i in range(L):
            p = f"model.layers.{i}."
            yield t(p + "self_attn.q_proj.weight", nh * hd, h); yield t(p + "self_attn.k_proj.weight", nkv * hd, h)
            yield t(p + "self_attn.v_proj.weight", nkv * hd, h); yield t(p + "self_attn.o_proj.weight", h, nh * hd)
            yield t(p + "mlp.gate_proj.weight", inter, h); yield t(p + "mlp.up_proj.weight", inter, h); yield t(p + "mlp.down_proj.weight", h, inter)
            yield t(p + "input_layernorm.weight", h, ones=True); yield t(p + "post_attention_layernorm.weight", h, ones=True)
        yield t("model.norm.weight", h, ones=True)
        yield t("lm_head.weight", v, h)
    loader.write_safetensors(path, tensors())


if any(a in ARM_LOAD for a in ARMS) and not os.path.exists(f"{mdir}/model.safetensors"):
    t0 = time.time(); write_checkpoint(f"{mdir}/model.safetensors"); print(f"checkpoint written in {time.time() - t0:.1f} s", flush=True)

def http(method, url, body=None, timeout=600):
    data = json.dumps(body).encode() if body is not None else (b"" if method in ("POST", "PUT") else None)
    req = urllib.request.Request(url, data=data, method=method, headers={"Content-Type": "application/json"})
    t0 = time.perf_counter()
    try:
        with urllib.request.urlopen(req, timeout=timeout) as r:
            return r.status, r.read().decode(), time.perf_counter() - t0
    except urllib.error.HTTPError as e:
        return e.code, e.read().decode(), time.perf_counter() - t0

env = dict(os.environ)
env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "plugin"), ROOT, os.path.join(ROOT, "scripts", "k8s_stub"), env.get("PYTHONPATH", "")])
if USE_AGENT:   # this repo's launcher-compatible node agent, owning the parking buffers
    launcher = subprocess.Popen([sys.executable, os.path.join(ROOT, "scripts", "run_node_agent.py"), "--port", str(LPORT), "--host", "127.0.0.1", "--parking",
                                 "--log-dir", OUT], env=env, cwd=ROOT, stdout=open(f"{OUT}/launcher.log", "w"), stderr=subprocess.STDOUT)
else:
    launcher = subprocess.Popen([sys.executable, os.path.join(LAUNCHER_DIR, "launcher.py"), "--port", str(LPORT), "--host", "127.0.0.1"],
                                env=env, cwd=LAUNCHER_DIR, stdout=open(f"{OUT}/launcher.log", "w"), stderr=subprocess.STDOUT)
results = {}
try:
    for _ in range(240):
        try:
            if http("GET", f"http://127.0.0.1:{LPORT}/health", timeout=2)[0] == 200: break
        except Exception:
            time.sleep(1)
    else:
        raise SystemExit("launcher did not come up")
    options = (f"--model {mdir} --load-format dummy --skip-tokenizer-init --enable-sleep-mode --port {VPORT} --host 127.0.0.1 "
               f"--enforce-eager --max-model-len 2048 --gpu-memory-utilization 0.30 --no-enable-prefix-caching"
               + (f" --tensor-parallel-size {TP}" if TP > 1 else ""))
    for arm in ARMS:
        extra_env = ARM_ENV[arm]
        iid = f"e2e-{arm}"
        arm_options = options.replace("--load-format dummy", f"--load-format {ARM_LOAD[arm]}") if arm in ARM_LOAD else options
        body = {"options": arm_options, "env_vars": {"VLLM_SERVER_DEV_MODE": "1", **extra_env}, "annotations": {"isc-name": "e2e", "inference-port": str(VPORT)}}
        if arm == "fma_b200_peer_parked":
            import pynvml
            pynvml.nvmlInit()
            u = pynvml.nvmlDeviceGetUUID(pynvml.nvmlDeviceGetHandleByIndex(0))
            body["gpu_uuids"] = [u.decode() if isinstance(u, bytes) else u]       # -> CUDA_VISIBLE_DEVICES=0: the parking GPU is invisible to the instance
        st, txt, _ = http("PUT", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}", body)
        assert st == 201, (st, txt)
        t0 = time.time(); up = False
        while time.time() - t0 < 600:
            try:
                if http("GET", f"http://127.0.0.1:{VPORT}/health", timeout=2)[0] == 200: up = True; break
            except Exception:
                pass
            time.sleep(2)
        log = http("GET", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}/log")[1]
        if not up:
            open(f"{OUT}/{arm}_vllm.log", "w").write(log); results[arm] = {"error": "vLLM did not become healthy", "log_tail": log[-1500:]}
            http("DELETE", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}"); continue
        load_s = time.time() - t0
        def gen():
            st, txt, _ = http("POST", f"http://127.0.0.1:{VPORT}/v1/completions", {"model": mdir, "prompt": [1, 2, 3, 4, 5, 6, 7, 8], "max_tokens": 16, "temperature": 0.0, "return_token_ids": True})
            try:
                c = json.loads(txt)["choices"][0]; return c.get("token_ids") or c.get("text")
            except Exception:
                return f"ERR {st} {txt[:200]}"
        before = gen()
        rows = []
        for rep in range(4):
            s_st, _, s_t = http("POST", f"http://127.0.0.1:{VPORT}/sleep")
            sl = json.loads(http("GET", f"http://127.0.0.1:{VPORT}/is_sleeping")[1])
            w_st, _, w_t = http("POST", f"http://127.0.0.1:{VPORT}/wake_up")
            aw = json.loads(http("GET", f"http://127.0.0.1:{VPORT}/is_sleeping")[1])
            rows.append(dict(sleep_status=s_st, sleep_s=s_t, is_sleeping_after_sleep=sl["is_sleeping"], wake_status=w_st, wake_s=w_t, is_sleeping_after_wake=aw["is_sleeping"]))
        after = gen()
        log = http("GET", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}/log")[1]
        open(f"{OUT}/{arm}_vllm.log", "w").write(log)
        lines = [l for l in log.splitlines() if "It took" in l or "sleep freed" in l or "fma_b200" in l or "Loading weights took" in l]
        results[arm] = dict(load_s=load_s, rows=rows, tokens_before=before, tokens_after=after, same_tokens=before == after,
                            uses_fma=any("fma_b200" in l for l in lines), vllm_log_lines=lines[-12:])
        pool = [l for l in log.splitlines() if "weights pool closed:" in l]
        if pool and TP == 1:
            # SURVEY §8d: the synthetic allocation tables (workloads.py, derived from model shapes + torch's segment rules) against what a
            # LIVE vLLM + torch really allocated under the "weights" tag: segment count, total bytes, size histogram, leading order
            try:
                sys.path.insert(0, ROOT)
                import fma_b200  # noqa: F401
                from fma_b200 import workloads as Wl
                live = json.loads(pool[-1].split("weights pool closed:", 1)[1].strip())
                syn = [x for x in Wl.allocation_table(MODEL) if x.tag == "weights"]
                hist = {}
                for x in syn:
                    hist[str(x.bytes >> 20)] = hist.get(str(x.bytes >> 20), 0) + 1
                synth = {"segments": len(syn), "bytes": sum(x.bytes for x in syn), "first_mib": [x.bytes >> 20 for x in syn[:6]],
                         "mib_histogram": dict(sorted(hist.items(), key=lambda kv: int(kv[0])))}
                results[arm]["table_validation"] = {"live": live, "synthetic": synth, "same_segment_count": live["segments"] == synth["segments"],
                                                    "same_bytes": live["bytes"] == synth["bytes"], "same_histogram": live["mib_histogram"] == synth["mib_histogram"],
                                                    "same_leading_order": live["first_mib"] == synth["first_mib"]}
            except Exception as e:
                results[arm]["table_validation"] = {"error": str(e)[:200]}
        print(arm, json.dumps(results[arm])[:1800], flush=True)
        if arm == "fma_b200_peer_parked":
            # park, delete the instance ASLEEP, start a new one with the same ID: it adopts the image the node agent kept
            s_st, _, s_t = http("POST", f"http://127.0.0.1:{VPORT}/sleep")
            sleepers = json.loads(http("GET", f"http://127.0.0.1:{LPORT}/v2/node/sleepers")[1])
            http("DELETE", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}")
            time.sleep(8)
            body["env_vars"]["FMA_ADOPT_PARKED"] = "1"
            st, txt, _ = http("PUT", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}", body)
            t0 = time.time(); up = False
            while st == 201 and time.time() - t0 < 600:
                try:
                    if http("GET", f"http://127.0.0.1:{VPORT}/health", timeout=2)[0] == 200: up = True; break
                except Exception:
                    pass
                time.sleep(2)
            log2 = http("GET", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}/log")[1]
            open(f"{OUT}/{arm}_second_instance_vllm.log", "w").write(log2)
            tokens2 = gen() if up else None
            results[arm + "_restart"] = dict(put_status=st, up=up, start_s=time.time() - t0, sleepers_while_parked=sleepers, tokens=tokens2,
                                             same_tokens_as_first_instance=tokens2 == before,
                                             adopt_log_lines=[l for l in log2.splitlines() if "adopted the parked image" in l or "parked image" in l][-4:])
            print(arm + "_restart", json.dumps(results[arm + "_restart"])[:1500], flush=True)
        st, _, _ = http("DELETE", f"http://127.0.0.1:{LPORT}/v2/vllm/instances/{iid}")
        time.sleep(8)
finally:
    if "ckpt_default" in results and "ckpt_fma" in results and "tokens_before" in results["ckpt_default"] and "tokens_before" in results["ckpt_fma"]:
        results["ckpt_loaders_agree"] = results["ckpt_default"]["tokens_before"] == results["ckpt_fma"]["tokens_before"]
    json.dump(results, open(f"{OUT}/e2e_launcher_vllm_{MODEL}_tp{TP}.json", "w"), indent=1)
    launcher.terminate()
    try: launcher.wait(timeout=20)
    except Exception: launcher.kill()
