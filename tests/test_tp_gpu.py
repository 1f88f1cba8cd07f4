"""Tensor parallelism (DESIGN.md §6): a TP=2 engine (one process, two GPUs, NCCL all-reduce over
NVLink) must emit the same greedy tokens as the TP=1 engine and the oracle on the same synthetic
weights.  Needs >= 2 GPUs; skipped on a 1-GPU machine."""
import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from agentcontrolplane_b200.engine import Engine
from oracle.llama_oracle import PRESETS, LlamaOracle

pytestmark = pytest.mark.gpu
SEED = 0xACB200


def _ngpu():
    return _lib.load().acp_kernel_device_count()


def _gen(eng, model, prompts, n_new):
    ts = [eng.submit({"model": model, "max_tokens": n_new, "acp": {"prompt_token_ids": p}}) for p in prompts]
    out = []
    for t in ts:
        assert eng.wait(t, 120000)
        st, body = eng.result(t)
        assert st == 200, body
        out.append(body["acp"]["token_ids"])
    return out


@pytest.mark.parametrize("tp,comm", [(2, "p2p"), (2, "nccl"), (4, "p2p"), (8, "p2p")])
def test_tp_matches_tp1_and_oracle(tp, comm):
    """comm = "p2p": fused peer-memory all-reduce + residual + RMSNorm (tp_comm.cu, the default);
    comm = "nccl": ncclAllReduce + add_rmsnorm (the baseline path)."""
    if _ngpu() < tp:
        pytest.skip(f"needs {tp} GPUs")
    model = "tiny-g2" if tp == 2 else "llama-3-8b-l2"
    cfg = PRESETS[model]
    rng = np.random.default_rng(tp)
    prompts = [[128000] + [int(t) for t in rng.integers(0, 256, size=n - 1)] for n in (5, 40, 97, 300)]
    n_new = 6
    base = {"model": model, "max_batch": 16, "kv_pages": 256, "max_tokens_per_step": 1024}
    with Engine(dict(base, tp=tp, tp_comm=comm)) as e:
        got_tp = _gen(e, model, prompts, n_new)
        s = e.stats()
        assert s["tp"] == tp
        # sampling / return_logits under the vocab-parallel LM head: logits are all-gathered, the sampler
        # then sees exactly the TP=1 logits layout (checked against the sampling oracle on those logits)
        t = e.submit({"model": model, "max_tokens": 3, "temperature": 0.7, "top_k": 20, "seed": 77,
                      "acp": {"prompt_token_ids": prompts[1], "return_logits": 3}})
        assert e.wait(t, 120000)
        lg_tp = e.logits(t, 3, 128256)
        st, body = e.result(t)
        assert st == 200, body
        from oracle import sampling_oracle as S
        for step, tok in enumerate(body["acp"]["token_ids"]):
            assert tok in S.candidates(lg_tp[step], 0.7, 20, 1.0, 77, step), (step, tok)
    with Engine(base) as e:
        got_1 = _gen(e, model, prompts, n_new)
        t = e.submit({"model": model, "max_tokens": 1, "acp": {"prompt_token_ids": prompts[1], "return_logits": 1}})
        assert e.wait(t, 120000)
        lg_1 = e.logits(t, 1, 128256)
        e.result(t)
    # first-position logits: TP shards sum partial products in a different order (one rounding after the exchange).
    # Bound: the engine tests' relative policy (8 % of the logit std, DESIGN.md §5)
    tol = max(3e-2, 0.08 * float(np.std(lg_1[0])))
    assert np.max(np.abs(lg_tp[0] - lg_1[0])) < tol, (float(np.max(np.abs(lg_tp[0] - lg_1[0]))), tol)
    for p, a, b in zip(prompts, got_tp, got_1):
        want, margins = LlamaOracle(cfg, SEED, mode="bf16").greedy(p, n_new, eos=(128001, 128008, 128009))
        for i, (x, y, w) in enumerate(zip(a, b, want)):
            if x != w or y != w:
                assert margins[i] < 0.06, (tp, len(p), a, b, want, margins)   # near-tie policy
                break


@pytest.mark.parametrize("tp,comm", [(2, "p2p"), (2, "nccl"), (4, "p2p"), (8, "p2p")])
def test_expert_parallel_matches_single_gpu_and_oracle(tp, comm):
    """Mixtral-style MoE with the experts spread over the tensor-parallel ranks (tp = 2: four experts per GPU;
    tp = 8: one expert per GPU, BASELINE config 4's layout): the weighted combine runs as the row-parallel
    exchange, one rounding after it, so tokens equal the single-GPU engine's and the oracle's."""
    if _ngpu() < tp:
        pytest.skip(f"needs {tp} GPUs")
    model = "tiny-moe" if tp == 2 else "mixtral-8x7b-l2"   # 2 KV heads / 8 KV heads: the head split must divide
    cfg = PRESETS[model]
    rng = np.random.default_rng(100 + tp)
    prompts = [[128000] + [int(t) for t in rng.integers(0, 256, size=n - 1)] for n in (4, 33, 120, 290)]
    n_new = 5
    base = {"model": model, "max_batch": 16, "kv_pages": 256, "max_tokens_per_step": 1024}
    with Engine(dict(base, tp=tp, tp_comm=comm)) as e:
        got_tp = _gen(e, model, prompts, n_new)
        assert e.stats()["tp"] == tp
    with Engine(base) as e:
        got_1 = _gen(e, model, prompts, n_new)
    for p, a, b in zip(prompts, got_tp, got_1):
        orc = LlamaOracle(cfg, SEED, mode="bf16")
        want, margins = orc.greedy(p, n_new, eos=(128001, 128008, 128009))
        for i, (x, y, w) in enumerate(zip(a, b, want)):
            if x != w or y != w:
                # near tie of the logits, or of the discrete routing (tests/test_engine_gpu.py ROUTER_GAP_TOL)
                assert margins[i] < 0.08 or orc.min_router_gap < 1e-2, (tp, len(p), a, b, want, margins, orc.min_router_gap)
                break
