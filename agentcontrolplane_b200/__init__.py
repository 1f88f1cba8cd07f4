"""agentcontrolplane_b200 — H100-native `provider: local` for ACP's Task -> LLM step.

Only what the hot path needs lives here: `csrc/` (sm_90a CUDA kernels, the continuous-batching
engine and the C ABI of include/acp_infer.h), `engine.py` (ctypes binding) and `llmclient.py`
(mirror of the reference's acp/internal/llmclient interface for tests and bench).
"""
