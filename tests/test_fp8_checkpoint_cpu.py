"""FP8 checkpoints without a GPU: the external pin of the FP8 numerics contract (a compressed-tensors FP8_DYNAMIC
checkpoint written from the oracle's quantised weights, run by transformers + compressed-tensors in fp32, against
the FP8 oracle's fp32 forward), the loader's parsing of F8_E4M3 tensors and quantization_config (every variant it
does not serve is refused with the field named), and the FP8 split-K rule."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from agentcontrolplane_b200 import host
from ckpt_util import hf_config
from oracle.fp8 import FP8_PRESETS, Fp8LlamaOracle
from oracle.llama_oracle import PRESETS

SEED = 0xACB200


def test_external_pin_transformers_compressed_tensors(tmp_path):
    """transformers + compressed-tensors decompress the checkpoint (codes x s_w) and fake-quantise every Linear input
    per token with s = amax / 448: the same contract.  fp32 on both sides; the difference is fp32 summation order."""
    pytest.importorskip("compressed_tensors")
    transformers = pytest.importorskip("transformers")
    from fp8_ckpt_util import write_fp8_checkpoint
    cfg = FP8_PRESETS["tiny-fp8"]
    write_fp8_checkpoint(str(tmp_path), cfg, SEED)
    transformers.utils.logging.set_verbosity_error()
    m = transformers.AutoModelForCausalLM.from_pretrained(str(tmp_path), dtype=torch.float32).eval()
    # fp32 summation order differs between torch and numpy; where it moves an activation across an e4m3 rounding
    # boundary, one code differs and every later position of that prompt moves with it (by < 0.05 here).  So: every
    # prompt agrees to 1e-5 at its first position, most positions agree to 1e-5, and none drifts further than 0.1.
    from oracle.llama_oracle import LlamaOracle
    close, total = 0, 0
    for seed in range(4):
        rng = np.random.default_rng(seed)
        prompt = [128000] + [int(t) for t in rng.integers(0, 256, size=24)]
        with torch.no_grad():
            hf = m(torch.tensor([prompt])).logits[0].float().numpy()
        orc = Fp8LlamaOracle(cfg, SEED, mode="fp32").forward(prompt, all_logits=True)
        d = np.max(np.abs(hf - orc), axis=1)
        assert d[0] < 1e-5 and d.max() < 0.1, (seed, d.tolist())
        close += int(np.sum(d < 1e-5))
        total += len(d)
        # the pin discriminates: the bf16 weights without FP8 are far from it
        bf = LlamaOracle(PRESETS["tiny"], SEED, mode="fp32").forward(prompt[:1], all_logits=True)
        assert np.max(np.abs(hf[0] - bf[0])) > 1e3 * d[0]
    assert close >= total // 2, (close, total)   # measured 67 of 100


def _qcfg(strategy="channel"):
    from fp8_ckpt_util import quantization_config
    return quantization_config(strategy)


def _small_checkpoint(path, qc, model_type="llama"):
    """config.json of a tiny Llama with `qc` as quantization_config, and one FP8 projection + its scale"""
    os.makedirs(path, exist_ok=True)
    cfg = PRESETS["tiny-moe" if model_type == "mixtral" else "tiny"]
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(hf_config(cfg, **({"quantization_config": qc} if qc is not None else {})), f)
    codes = torch.arange(512 * 512, dtype=torch.int64).remainder(0x7E).to(torch.uint8).reshape(512, 512)
    save_file({"model.layers.0.self_attn.o_proj.weight": codes.view(torch.float8_e4m3fn),
               "model.layers.0.self_attn.o_proj.weight_scale": torch.ones(512, 1, dtype=torch.bfloat16)},
              os.path.join(path, "model.safetensors"))
    return str(path)


@pytest.mark.parametrize("strategy", ["channel", "tensor"])
def test_fp8_checkpoint_is_indexed(tmp_path, strategy):
    idx = host.checkpoint_index(_small_checkpoint(tmp_path, _qcfg(strategy)))
    t = idx["tensors"]["model.layers.0.self_attn.o_proj.weight"]
    assert t["dtype"] == "F8_E4M3" and t["shape"] == [512, 512] and t["nbytes"] == 512 * 512
    assert idx["tensors"]["model.layers.0.self_attn.o_proj.weight_scale"]["nbytes"] == 512 * 2
    assert idx["model"]["weight_dtype"] == "fp8_e4m3"
    assert host.checkpoint_index(_small_checkpoint(tmp_path / "plain", None))["model"]["weight_dtype"] == "bf16"


def _variant(edit):
    q = copy.deepcopy(_qcfg())
    edit(q)
    return q


def _g(q):
    return q["config_groups"]["group_0"]


REFUSED = {
    "quant_method": lambda q: q.update(quant_method="gptq"),
    "format": lambda q: q.update(format="pack-quantized"),
    "kv_cache_scheme": lambda q: q.update(kv_cache_scheme={"num_bits": 8, "type": "float", "strategy": "tensor", "dynamic": False}),
    "config_groups": lambda q: q["config_groups"].update(group_1=copy.deepcopy(_g(q))),
    "config_groups.group_0.targets": lambda q: _g(q).update(targets=["Linear", "Embedding"]),
    "config_groups.group_0.weights.type": lambda q: _g(q)["weights"].update(type="int"),
    "config_groups.group_0.weights.num_bits": lambda q: _g(q)["weights"].update(num_bits=4),
    "config_groups.group_0.weights.strategy": lambda q: _g(q)["weights"].update(strategy="group", group_size=128),
    "config_groups.group_0.weights.dynamic": lambda q: _g(q)["weights"].update(dynamic=True),
    "config_groups.group_0.weights.block_structure": lambda q: _g(q)["weights"].update(block_structure=[128, 128]),
    "config_groups.group_0.input_activations.dynamic": lambda q: _g(q)["input_activations"].update(dynamic=False),
    "config_groups.group_0.input_activations.strategy": lambda q: _g(q)["input_activations"].update(strategy="tensor"),
    "config_groups.group_0.input_activations": lambda q: _g(q).update(input_activations=None),
    "config_groups.group_0.output_activations": lambda q: _g(q).update(output_activations=copy.deepcopy(_g(q)["input_activations"])),
    "ignore": lambda q: q.update(ignore=[]),
}


@pytest.mark.parametrize("field", sorted(REFUSED))
def test_unsupported_quantization_config_is_refused_by_name(tmp_path, field):
    with pytest.raises(ValueError) as e:
        host.checkpoint_index(_small_checkpoint(tmp_path, _variant(REFUSED[field])))
    assert f"quantization_config.{field} " in str(e.value), str(e.value)


def test_block_strategy_is_refused(tmp_path):
    q = _variant(lambda q: _g(q)["weights"].update(strategy="block", block_structure=[128, 128]))
    with pytest.raises(ValueError, match="quantization_config.config_groups.group_0.weights.strategy"):
        host.checkpoint_index(_small_checkpoint(tmp_path, q))


def test_fp8_mixture_of_experts_is_refused(tmp_path):
    with pytest.raises(ValueError, match="quantization_config: FP8 is not supported for mixture-of-experts"):
        host.checkpoint_index(_small_checkpoint(tmp_path, _qcfg(), model_type="mixtral"))


def test_fp8_splitk_rule_and_workspace():
    """FP8 k-blocks hold 128 codes: the factors of the 8B shapes depend only on (M, K) for steps of <= 256 rows
    (batch invariance), and the FP8 workspace holds the planes of every step height."""
    from agentcontrolplane_b200 import _lib
    lib = _lib.load_host()
    f = lib.acp_host_splitk_factor_fp8
    f.restype, f.argtypes = ctypes.c_int, [ctypes.c_int] * 5
    w = lib.acp_host_splitk_workspace_bytes_fp8
    w.restype, w.argtypes = ctypes.c_size_t, [ctypes.c_int] * 5
    shapes = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}
    for name, (M, K) in shapes.items():
        small = {f(M, K, n, 222, 0) for n in (1, 7, 64, 200, 256)}
        assert len(small) == 1, (name, small)
        s = small.pop()
        assert 1 <= s <= (K // 128) // 4 or s == 1, (name, s)     # at least 4 FP8 k-blocks per split
        for max_batch in (64, 256, 512, 1024):
            ws = w(M, K, max_batch, 222, 0)
            for n in range(1, max_batch + 1, 37):
                assert f(M, K, n, 222, 0) * n * M * 4 <= ws, (name, max_batch, n)
    assert tuple(f(M, K, 64, 222, 0) for M, K in shapes.values()) == (5, 7, 1, 7)
    assert f(512, 512, 16, 222, 0) == 1                            # tiny O: 4 k-blocks, one split
