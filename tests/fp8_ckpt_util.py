"""Writes compressed-tensors FP8_DYNAMIC Llama checkpoints (config.json with quantization_config + safetensors with
F8_E4M3 weights and weight_scale tensors) from the FP8 oracle's quantised synthetic weights (oracle/fp8.py)."""
import json
import os

import numpy as np
import torch
from safetensors.torch import save_file

from ckpt_util import hf_config, tensors_from_oracle
from oracle.fp8 import E4M3_MAX, Fp8LlamaConfig, e4m3_decode, e4m3_encode, shared_quant_weights
from oracle.llama_oracle import PRESETS


def quantization_config(strategy: str = "channel") -> dict:
    from compressed_tensors.quantization import QuantizationConfig, preset_name_to_scheme
    scheme = preset_name_to_scheme("FP8_DYNAMIC", ["Linear"])
    scheme.weights.strategy = strategy
    q = QuantizationConfig(config_groups={"group_0": scheme}, quant_method="compressed-tensors",
                           format="float-quantized", ignore=["lm_head"], quantization_status="compressed")
    return json.loads(q.model_dump_json())


def _parts(cfg):
    q, kv, f = cfg.q_dim, cfg.kv_dim, cfg.ffn
    return [("self_attn.q_proj", "wqkv", 0, q), ("self_attn.k_proj", "wqkv", q, q + kv),
            ("self_attn.v_proj", "wqkv", q + kv, q + 2 * kv), ("self_attn.o_proj", "wo", 0, cfg.hidden),
            ("mlp.gate_proj", "wgu", 0, f), ("mlp.up_proj", "wgu", f, 2 * f), ("mlp.down_proj", "wdown", 0, cfg.hidden)]


def quantised_tensors(cfg: Fp8LlamaConfig, seed: int, strategy: str = "channel", scale_dtype=torch.float32) -> dict:
    """{hf name: (codes uint8 [rows][cols], scales fp32 [rows] as the loader reads them)} of every projection.
    channel: the oracle's codes and per-row scales (scales rounded to scale_dtype).  tensor: one scale per tensor,
    fp32(max amax / 448), and the bf16 weights re-quantised with it by the same clamp + e4m3 rounding."""
    qw = shared_quant_weights(cfg, seed)
    out = {}
    for l in range(cfg.layers):
        for name, which, r0, r1 in _parts(cfg):
            codes, s = (a[r0:r1] for a in getattr(qw, which)(l))
            if strategy == "tensor":
                w = getattr(qw.bf16, which)(l)[r0:r1]
                st = np.float32(np.max(np.abs(w)) / E4M3_MAX)
                codes = e4m3_encode(np.clip((w / st).astype(np.float32), -E4M3_MAX, E4M3_MAX))
                s = np.full(r1 - r0, st, np.float32)
            s = torch.from_numpy(np.ascontiguousarray(s)).to(scale_dtype).float().numpy()
            out[f"model.layers.{l}.{name}"] = (codes, s)
    return out


def write_fp8_checkpoint(path: str, cfg: Fp8LlamaConfig, seed: int, strategy: str = "channel",
                         scale_dtype=torch.float32) -> dict:
    os.makedirs(path, exist_ok=True)
    t = tensors_from_oracle(PRESETS[cfg.base], seed)
    q = quantised_tensors(cfg, seed, strategy, scale_dtype)
    for name, (codes, s) in q.items():
        t[name + ".weight"] = torch.from_numpy(np.ascontiguousarray(codes)).view(torch.float8_e4m3fn)
        st = torch.from_numpy(np.ascontiguousarray(s)).to(scale_dtype)
        t[name + ".weight_scale"] = st.reshape(-1, 1) if strategy == "channel" else st[:1].reshape(())
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(hf_config(PRESETS[cfg.base], quantization_config=quantization_config(strategy)), f)
    save_file({k: v.contiguous() for k, v in t.items()}, os.path.join(path, "model.safetensors"))
    return q


class CheckpointQuantWeights:
    """The projections of a written FP8 checkpoint in the oracle's QuantWeights interface (logical row order)."""

    def __init__(self, cfg: Fp8LlamaConfig, q: dict):
        self.cfg, self.q, self._dec = cfg, q, {}

    def _cat(self, l, which):
        key = (l, which)
        if key not in self._dec:
            parts = [self.q[f"model.layers.{l}.{n}"] for n, w, _, _ in _parts(self.cfg) if w == which]
            self._dec[key] = (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
        return self._dec[key]

    def decoded(self, qw):
        key = id(qw[0])
        if key not in self._dec:
            self._dec[key] = e4m3_decode(qw[0]).astype(np.float64)
        return self._dec[key]

    def wqkv(self, l):
        return self._cat(l, "wqkv")

    def wo(self, l):
        return self._cat(l, "wo")

    def wgu(self, l):
        return self._cat(l, "wgu")

    def wdown(self, l):
        return self._cat(l, "wdown")
