"""swiftllm_b200 - H100-native (sm_90a) data plane for swiftLLM's `LlamaModel`.

Mirrors the reference package surface that belongs to the hot path:
    swiftllm_b200.EngineConfig, swiftllm_b200.LlamaModel           (swiftllm/__init__.py:2,9)
    swiftllm_b200.worker.kernels.*                                 (swiftllm/worker/kernels/*)
    swiftllm_b200.swiftllm_c.swap_blocks                           (csrc/ -> module swiftllm_c)
The control plane (Engine, Scheduler, API server, tokenizer) is out of scope; the unmodified reference Engine can
drive this LlamaModel (INTEGRATION.md).
"""
from swiftllm_b200.engine_config import EngineConfig
from swiftllm_b200.model_config import LlamaModelConfig
from swiftllm_b200.worker.model import LlamaModel

__all__ = ["EngineConfig", "LlamaModelConfig", "LlamaModel"]
