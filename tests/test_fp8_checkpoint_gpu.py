"""FP8 checkpoints on the GPU: compressed-tensors FP8_DYNAMIC checkpoints written from the oracle's quantised
weights.  With the oracle's own per-channel F32 scales the engine is bit-identical to the synthetic `-fp8` preset
(same codes, same scales, same index map); with BF16 scales and with per-tensor scales it matches the FP8 oracle
run on exactly the checkpoint's codes and scales."""
import numpy as np
import pytest
import torch

from agentcontrolplane_b200.engine import Engine
from fp8_ckpt_util import CheckpointQuantWeights, write_fp8_checkpoint
from oracle.fp8 import FP8_PRESETS, Fp8LlamaOracle
from test_engine_gpu import SEED, _prompt, assert_tokens_match
from test_fp8_gpu import FP8_LOGIT_RTOL

pytestmark = pytest.mark.gpu

CFG = FP8_PRESETS["tiny-fp8"]


def _run(eng, name, prompt, n, logits):
    t = eng.submit({"model": name, "max_tokens": n, "acp": {"prompt_token_ids": prompt, "return_logits": logits}})
    assert eng.wait(t, 120000)
    lg = eng.logits(t, logits, 128256)
    st, body = eng.result(t)
    assert st == 200, body
    return body["acp"]["token_ids"], lg


def _engine(weights=None):
    cfg = {"model": "tiny-fp8", "max_batch": 16, "kv_pages": 256, "max_tokens_per_step": 1024}
    if weights:
        cfg["weights"] = weights
        cfg["model"] = "ck"
    return Engine(cfg)


@pytest.fixture(scope="module")
def synthetic_run():
    prompts = [_prompt(np.random.default_rng(s), n) for s, n in ((1, 45), (2, 300))]
    with _engine() as e:
        return prompts, [_run(e, "tiny-fp8", p, 6, 3) for p in prompts]


def test_channel_f32_checkpoint_equals_synthetic(tmp_path, synthetic_run):
    prompts, want = synthetic_run
    write_fp8_checkpoint(str(tmp_path), CFG, SEED, "channel", torch.float32)
    with _engine(str(tmp_path)) as e:
        assert e.stats()["weight_dtype"] == "fp8_e4m3"
        for p, (toks, lg) in zip(prompts, want):
            t2, lg2 = _run(e, "ck", p, 6, 3)
            assert t2 == toks
            assert np.array_equal(lg2, lg)


@pytest.mark.parametrize("strategy,scale_dtype", [("channel", torch.bfloat16), ("tensor", torch.float32),
                                                  ("tensor", torch.bfloat16)])
def test_checkpoint_scale_variants_match_oracle(tmp_path, strategy, scale_dtype):
    q = write_fp8_checkpoint(str(tmp_path), CFG, SEED, strategy, scale_dtype)
    prompt = _prompt(np.random.default_rng(1), 45)
    with _engine(str(tmp_path)) as e:
        toks, lg = _run(e, "ck", prompt, 8, 1)
    orc = Fp8LlamaOracle(CFG, SEED)
    orc.qw = CheckpointQuantWeights(CFG, q)
    ref = orc.forward(prompt)[-1]
    tol = FP8_LOGIT_RTOL * float(np.std(ref))
    assert np.max(np.abs(lg[0] - ref)) < tol, float(np.max(np.abs(lg[0] - ref)))
    orc2 = Fp8LlamaOracle(CFG, SEED)
    orc2.qw = CheckpointQuantWeights(CFG, q)
    want, margins = orc2.greedy(prompt, 8, eos=(128001, 128008, 128009))
    assert_tokens_match(toks, want, margins, tol=tol)
