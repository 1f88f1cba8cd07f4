"""acp_infer_init {"weights": <dir>}: a HuggingFace-format checkpoint (written with the real
`safetensors` library from the oracle's seeded weights) must produce EXACTLY the tokens and logits
of the engine's synthetic-weight path — the loader's tiling / gate-up interleaving / q-k-v fusion /
dtype conversion is then proven against the layout every other parity test already pins."""
import numpy as np
import pytest
import torch

from agentcontrolplane_b200 import _lib
from agentcontrolplane_b200.engine import Engine
from ckpt_util import write_checkpoint
from oracle.llama_oracle import PRESETS

pytestmark = pytest.mark.gpu
SEED = 0xACB200
BASE = {"max_batch": 8, "kv_pages": 128, "max_tokens_per_step": 1024, "max_pages_per_seq": 16}


def _gen(e, model, prompts, n_new):
    ts = [e.submit({"model": model, "max_tokens": n_new, "acp": {"prompt_token_ids": p, "return_logits": 2}}) for p in prompts]
    out = []
    for t in ts:
        assert e.wait(t, 120000)
        lg = e.logits(t, 2, 128256)
        st, body = e.result(t)
        assert st == 200, body
        out.append((body["acp"]["token_ids"], lg))
    return out


@pytest.fixture(scope="module")
def prompts():
    rng = np.random.default_rng(21)
    return [[128000] + [int(t) for t in rng.integers(0, 256, size=n - 1)] for n in (7, 64, 300)]


@pytest.fixture(scope="module")
def synthetic(prompts):
    with Engine(dict(BASE, model="tiny-g2")) as e:
        return _gen(e, "tiny-g2", prompts, 6)


@pytest.mark.parametrize("variant", ["bf16", "sharded", "f32"])
def test_checkpoint_equals_synthetic_weights(tmp_path, prompts, synthetic, variant):
    d = str(tmp_path / "tiny-g2-ckpt")
    write_checkpoint(d, PRESETS["tiny-g2"], SEED, shards=3 if variant == "sharded" else 1,
                     dtype=torch.float32 if variant == "f32" else torch.bfloat16)
    with Engine(dict(BASE, weights=d)) as e:
        assert e.stats()["model"] == "tiny-g2-ckpt"          # default served name = directory name
        got = _gen(e, "tiny-g2-ckpt", prompts, 6)
        st, body = e.complete({"model": "something-else", "max_tokens": 2, "acp": {"prompt_token_ids": prompts[0]}})
        assert st == 404
    for (a, la), (b, lb) in zip(got, synthetic):
        assert a == b and np.array_equal(la, lb)


def test_checkpoint_tensor_parallel(tmp_path, prompts, synthetic):
    if _lib.load().acp_kernel_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    d = str(tmp_path / "ckpt-tp")
    write_checkpoint(d, PRESETS["tiny-g2"], SEED)
    with Engine(dict(BASE, weights=d, model="m", tp=2)) as e:
        got = [e.complete({"model": "m", "max_tokens": 6, "acp": {"prompt_token_ids": p}})[1]["acp"]["token_ids"] for p in prompts]
    with Engine(dict(BASE, model="tiny-g2", tp=2)) as e:
        want = [e.complete({"model": "tiny-g2", "max_tokens": 6, "acp": {"prompt_token_ids": p}})[1]["acp"]["token_ids"] for p in prompts]
    assert got == want


def test_missing_tensor_fails_init(tmp_path):
    """A checkpoint missing one tensor is refused at init: a bf16 weight, or an FP8 projection's weight_scale."""
    import os
    from safetensors.torch import load_file, save_file
    from fp8_ckpt_util import write_fp8_checkpoint
    from oracle.fp8 import FP8_PRESETS
    for name, write, missing in (
            ("broken", lambda d: write_checkpoint(d, PRESETS["tiny"], SEED), "model.layers.1.mlp.down_proj.weight"),
            ("broken-fp8", lambda d: write_fp8_checkpoint(d, FP8_PRESETS["tiny-fp8"], SEED),
             "model.layers.1.mlp.down_proj.weight_scale")):
        d = str(tmp_path / name)
        write(d)
        f = os.path.join(d, "model.safetensors")
        t = load_file(f)
        del t[missing]
        save_file(t, f)
        with pytest.raises(RuntimeError):
            Engine(dict(BASE, weights=d))


def test_checkpoint_with_its_own_tokenizer_json(tmp_path):
    """A checkpoint directory that ships tokenizer.json is served with THAT vocabulary: the chat
    template is tokenised by the byte-level BPE (tests/test_tokenizer_cpu.py pins it to HuggingFace
    `tokenizers`), stop tokens are the tokenizer's own ids, and the text is detokenised with it."""
    import json
    import os
    import shutil

    from agentcontrolplane_b200 import host
    from oracle.llama_oracle import LlamaOracle
    here = os.path.dirname(os.path.abspath(__file__))
    tok_file = os.path.join(here, "golden", "llama3_style_tokenizer.json")
    gold = json.load(open(os.path.join(here, "golden", "tokenizer_golden.json")))
    d = str(tmp_path / "served-model")
    write_checkpoint(d, PRESETS["tiny"], SEED)
    shutil.copy(tok_file, os.path.join(d, "tokenizer.json"))
    req = {"model": "served-model", "max_tokens": 12, "messages": [
        {"role": "system", "content": "You are a helpful assistant."},
        {"role": "user", "content": "What is the capital of France?"}]}
    want_prompt = host.render_prompt_with(req, tok_file)["token_ids"]
    stops = tuple(gold["special"][k] for k in ("<|eot_id|>", "<|eom_id|>", "<|end_of_text|>"))
    with Engine(dict(BASE, weights=d)) as e:
        assert e.stats()["tokenizer"] == "byte-level-bpe"
        st, body = e.complete(req)
        assert st in (200, 422), body          # 422 = the random-weight model stopped immediately
        if st == 200:
            ids = body["acp"]["token_ids"]
            assert body["usage"]["prompt_tokens"] == len(want_prompt)
            want, margins = LlamaOracle(PRESETS["tiny"], SEED, mode="bf16").greedy(want_prompt, 12, eos=stops)
            for i, (g, w) in enumerate(zip(ids, want)):
                if g != w:
                    assert margins[i] < 0.06, (ids, want, margins)
                    break
            text_ids = ids[:-1] if ids and ids[-1] in stops else ids
            import re
            squash = lambda t: re.sub("\ufffd+", "\ufffd", t)      # replacement granularity for invalid UTF-8 may differ
            assert squash(body["choices"][0]["message"]["content"]) == squash(host.tokenizer_decode(text_ids, tok_file).decode(errors="replace"))
    # a tokenizer whose ids exceed the model's vocabulary is refused at init
    small = str(tmp_path / "small-vocab")
    from oracle.llama_oracle import LlamaConfig
    write_checkpoint(small, LlamaConfig("small", hidden=256, layers=1, heads=2, kv_heads=1, ffn=512, vocab=1024), SEED)
    shutil.copy(tok_file, os.path.join(small, "tokenizer.json"))
    with pytest.raises(RuntimeError):
        Engine(dict(BASE, weights=small))


def test_llama31_rope_scaling_checkpoint_matches_oracle(tmp_path):
    """config.json rope_scaling {"rope_type": "llama3"}: the engine's scaled RoPE table is bit-identical
    to the oracle's (tests/test_checkpoint_cpu.py), so greedy tokens must match the bf16 oracle."""
    import dataclasses
    from oracle.llama_oracle import LlamaOracle
    scaling = (8.0, 1.0, 4.0, 64)
    cfg = dataclasses.replace(PRESETS["tiny"], name="tiny-rope31", rope_scaling=scaling)
    d = str(tmp_path / "rope31")
    write_checkpoint(d, cfg, SEED, rope_scaling={"rope_type": "llama3", "factor": scaling[0], "low_freq_factor": scaling[1],
                                                 "high_freq_factor": scaling[2], "original_max_position_embeddings": scaling[3]})
    rng = np.random.default_rng(31)
    prompt = [128000] + [int(t) for t in rng.integers(0, 256, size=199)]
    with Engine(dict(BASE, weights=d, model="m")) as e:
        st, body = e.complete({"model": "m", "max_tokens": 8, "acp": {"prompt_token_ids": prompt}})
        assert st == 200, body
        got = body["acp"]["token_ids"]
    want, margins = LlamaOracle(cfg, SEED, mode="bf16").greedy(prompt, 8, eos=(128001, 128008, 128009))
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            assert margins[i] < 0.06, (got, want, margins)
            break


def test_mixtral_checkpoint_equals_synthetic_weights(tmp_path, prompts):
    """A Mixtral-format checkpoint (model_type mixtral; block_sparse_moe.gate + experts.<e>.{w1, w3, w2}, the hub
    layout of Mixtral-8x7B) loads into the router / grouped expert tensors and gives exactly the synthetic path's
    tokens and logits."""
    with Engine(dict(BASE, model="tiny-moe")) as e:
        want = _gen(e, "tiny-moe", prompts, 6)
    d = str(tmp_path / "tiny-moe-ckpt")
    write_checkpoint(d, PRESETS["tiny-moe"], SEED, shards=2)
    idx = __import__("agentcontrolplane_b200.host", fromlist=["host"]).checkpoint_index(d)
    assert idx["config"]["model_type"] == "mixtral" and idx["model"]["layers"] == 2
    with Engine(dict(BASE, weights=d)) as e:
        got = _gen(e, "tiny-moe-ckpt", prompts, 6)
    for (a, la), (b, lb) in zip(got, want):
        assert a == b and np.array_equal(la, lb)
