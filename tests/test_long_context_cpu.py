"""Long contexts without a GPU: a Llama-3.1 checkpoint keeps its 131072-token window, the oracle's RoPE tables
past the original 8192 positions follow transformers' "llama3" scaling, and the engine's Llama-3.1 presets
(csrc/model_config.cc) are the models the tests' oracle configurations (llama31_presets.py) describe."""
import dataclasses

import numpy as np
import pytest
import torch

from agentcontrolplane_b200 import host
from oracle.llama_oracle import PRESETS, LlamaConfig, rope_inv_freq, rope_tables
from ckpt_util import write_checkpoint
from llama31_presets import BASE as NEW_PRESETS, LLAMA31

CFG = LlamaConfig("ckpt-test", hidden=256, layers=2, heads=2, kv_heads=1, ffn=512, vocab=1024)
SCALING = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
           "original_max_position_embeddings": 8192}


def test_checkpoint_keeps_its_131072_token_window(tmp_path):
    d = str(tmp_path / "m31")
    write_checkpoint(d, CFG, 5, rope_scaling=SCALING, max_position_embeddings=131072)
    m = host.checkpoint_index(d)["model"]
    assert m["max_pos"] == 131072
    assert m["rope_scaling"] == [8.0, 1.0, 4.0, 8192.0]
    d2 = str(tmp_path / "m3")
    write_checkpoint(d2, CFG, 5, max_position_embeddings=8192)
    m2 = host.checkpoint_index(d2)["model"]
    assert m2["max_pos"] == 8192 and m2["rope_scaling"] is None


def test_oracle_rope_tables_past_8192_match_transformers_llama3():
    from transformers import LlamaConfig as HFConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    cfg = LLAMA31["tiny-3.1"]
    cos, sin = rope_tables(cfg, cfg.max_pos)
    assert cos.shape == (131072, 64)
    hf = HFConfig(hidden_size=cfg.hidden, num_attention_heads=cfg.heads, num_key_value_heads=cfg.kv_heads,
                  head_dim=128, rope_theta=cfg.rope_theta, max_position_embeddings=131072, rope_scaling=SCALING)
    rot = LlamaRotaryEmbedding(hf, device="cpu")
    pos = torch.arange(8192, 131072, dtype=torch.int64)[None]
    hc, hs = rot(torch.zeros(1, dtype=torch.float32), pos)
    hc, hs = hc[0, :, :64].numpy(), hs[0, :, :64].numpy()
    assert hc.dtype == np.float32
    # both take angle = fp32(pos * inv_freq); the inverse frequencies may differ in their last bit (transformers
    # derives them in fp32, the engine and the oracle in double), which moves an angle by up to pos * ulp(inv)
    inv_hf = rot.inv_freq.double().numpy()
    inv = rope_inv_freq(cfg).astype(np.float64)
    np.testing.assert_allclose(inv, inv_hf, rtol=3e-7)
    p = np.arange(8192, 131072, dtype=np.float64)[:, None]
    ang = p * inv[None, :]
    tol = p * np.abs(inv - inv_hf)[None, :] + 2.0 * np.spacing(ang.astype(np.float32)) + 2e-6
    assert (np.abs(cos[8192:] - hc) <= tol).all()
    assert (np.abs(sin[8192:] - hs) <= tol).all()
    # the scaled (low-frequency) bands are what changes past the original window
    plain = rope_tables(dataclasses.replace(cfg, rope_scaling=None), 131072)[0]
    assert not np.array_equal(plain[8192:, -1], cos[8192:, -1])


@pytest.mark.parametrize("name", sorted(NEW_PRESETS))
def test_llama31_presets_are_the_same_model_in_engine_and_oracle(name):
    eng, orc = host.model_preset(name), LLAMA31[name]
    assert (eng["hidden"], eng["layers"], eng["heads"], eng["kv_heads"], eng["ffn"], eng["vocab"], eng["experts"]) == \
        (orc.hidden, orc.layers, orc.heads, orc.kv_heads, orc.ffn, orc.vocab, orc.experts)
    assert eng["rope_theta"] == orc.rope_theta and abs(eng["eps"] - orc.eps) < 1e-12
    assert eng["max_pos"] == orc.max_pos == 131072
    assert tuple(eng["rope_scaling"]) == tuple(float(v) for v in orc.rope_scaling) == (8.0, 1.0, 4.0, 8192.0)
    assert np.array_equal(np.array(eng["rope_inv_freq"], np.float32), rope_inv_freq(orc))
    assert eng["weight_dtype"] == "bf16"
    # the Llama-3 preset it extends: identical but for the window and the scaling
    base_e, base_o = host.model_preset(NEW_PRESETS[name]), PRESETS[NEW_PRESETS[name]]
    same = ("hidden", "layers", "heads", "kv_heads", "ffn", "vocab", "rope_theta", "eps", "experts")
    assert {k: eng[k] for k in same} == {k: base_e[k] for k in same}
    assert dataclasses.replace(orc, name=base_o.name, max_pos=base_o.max_pos, rope_scaling=None) == base_o
    assert base_e["max_pos"] == 8192 and base_e["rope_scaling"] is None


def test_fp8_suffix_covers_the_llama31_presets():
    for name in ("llama-3.1-8b-fp8", "llama-3.1-8b-l2-fp8"):
        m = host.model_preset(name)
        assert m["weight_dtype"] == "fp8_e4m3" and m["max_pos"] == 131072
    with pytest.raises(KeyError):
        host.model_preset("llama-3.1-70b")
