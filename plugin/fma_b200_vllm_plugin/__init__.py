"""vLLM general plugin: routes vLLM's sleep/wake allocator to the H100 engine when FMA_B200=1.

vLLM calls every entry point of group ``vllm.general_plugins`` in the API-server, engine-core and worker
processes (vllm:plugins/__init__.py:69-82, v1/engine/core.py:108, v1/worker/worker_base.py:247) before a worker
first touches ``vllm.device_allocator.cumem.CuMemAllocator`` (late imports in v1/worker/gpu_worker.py:158,182,202).
The switch travels per instance through ``InferenceServerConfig.spec.modelServerConfig.env_vars``
(api/fma/v1alpha1/inferenceserverconfig_types.go:46-48) -> launcher ``VllmConfig.env_vars`` -> ``set_env_vars``
(inference_server/launcher/launcher.py:824-826,840-849); nothing in the reference changes.
"""
import os


def register() -> None:
    if os.environ.get("FMA_B200", "0") != "1":
        return
    import fma_b200  # noqa: F401  (repo root on PYTHONPATH)
    from fma_b200 import cumem

    cumem.install_into_vllm()
    try:                                   # --load-format fma: checkpoint files -> HBM through the engine's mover
        from fma_b200 import vllm_loader

        vllm_loader.register()
    except Exception as e:                 # a vLLM without the loader registry: sleep/wake still works
        import logging

        logging.getLogger("fma_b200").warning("--load-format fma not registered: %s", e)
