"""Parity of the CUDA engine at the FULL BASELINE model — Llama-3-8B shapes, all 32 layers — on ONE GPU,
against two independent checkers that run as fp32 torch on the same GPU (test side only):

  (a) tests/torch_oracle.py `TorchLlamaOracle` (bf16 mode): the numpy oracle's restatement with the
      engine's bf16 rounding points, pinned to the numpy oracle and to HuggingFace on CPU
      (tests/test_torch_oracle_cpu.py).
  (b) HuggingFace `transformers.LlamaForCausalLM` holding the same weights, fp32 compute — "the
      reference's llmclient path pointed at the same weights" (SURVEY.md §8c(iii);
      acp/internal/llmclient/langchaingo_client.go:102 is the call a provider serving this checkpoint
      answers).  HF has no bf16 rounding points, so this comparison is statistical (relative RMS logit
      error, correlation, arg-max agreement where HF's own margin clears the noise).

Two weight regimes, because rounding noise behaves very differently in them (scripts/fulldepth_probe.py
measures both):

  * DAMPED, w_std = 0.005 — every layer's update is of the order of the residual stream, as in a
    trained network.  bf16 rounding noise stays at ~1 % of the logit scale through all 32 layers
    (max |engine - bf16 oracle| = 0.054 logit std; vs HF fp32: 1.2 % relative RMS).  This is the
    asserting regime: any indexing / layout / masking / layer-wiring bug at depth moves logits by
    O(1) logit std and fails it.
  * BENCH weights, w_std = 0.02 (what bench.py runs) — each layer's update is ~85x the embedding
    scale and the random network is chaotic: a single flipped bf16 rounding grows by ~10 % per layer
    (0.046 logit std at 2 layers, 0.106 at 8, 0.28 at 32, the same growth against the bf16-mirroring
    oracle and against HF fp32).  No fixed-precision implementation can agree tightly here; the test
    asserts the bounds measured for that growth, token equality wherever the oracle's margin clears
    them, and a correlation floor.

Workload = BASELINE config 1's batch: 64 concurrent requests x 512-token windows through the engine
together; the checkers run a sample (one forward pass of the 8B model each).
"""
import dataclasses

import numpy as np
import pytest

from agentcontrolplane_b200.engine import Engine
from oracle.llama_oracle import PRESETS

pytestmark = pytest.mark.gpu

MODEL = "llama-3-8b"
SEED = 0xACB200
N_NEW = 6
SAMPLE = [0, 9, 22, 37, 50, 63]
# regime -> (max |engine - bf16 oracle| in units of the logit std, relative RMS vs HF fp32); the bounds leave
# about 2x head-room over what scripts/fulldepth_probe.py reports, for other prompts
REGIMES = {"damped": (0.005, 0.11, 0.03), "bench": (0.02, 0.6, 0.15)}


@pytest.fixture(scope="module", params=list(REGIMES))
def run(request):
    import torch
    from torch_oracle import TorchWeights
    w_std, tol_rel, hf_rel = REGIMES[request.param]
    rng = np.random.default_rng(20260921)
    prompts = [[128000] + [int(t) for t in rng.integers(0, 256, size=511)] for _ in range(64)]
    with Engine({"model": MODEL, "max_batch": 64, "kv_pages": 64 * 18 + 8, "max_tokens_per_step": 4096,
                 "max_pages_per_seq": 32, "prefix_cache": False, "w_std": w_std}) as eng:
        ts = [eng.submit({"model": MODEL, "max_tokens": N_NEW,
                          "acp": {"prompt_token_ids": p, "return_logits": N_NEW if i in SAMPLE else 0}})
              for i, p in enumerate(prompts)]
        outs = {}
        for i, t in enumerate(ts):
            assert eng.wait(t, 600000)
            lg = eng.logits(t, N_NEW, 128256) if i in SAMPLE else None
            st, body = eng.result(t)
            assert st == 200, body
            outs[i] = (body["acp"]["token_ids"], lg)
        stats = eng.stats()
    assert stats["layers"] == 32 and stats["prefill_tokens"] == 64 * 512
    weights = TorchWeights(dataclasses.replace(PRESETS[MODEL], w_std=w_std), SEED, device="cuda:0")
    yield request.param, prompts, outs, weights, tol_rel, hf_rel
    del weights
    torch.cuda.empty_cache()


def test_full_depth_tokens_and_logits_match_the_bf16_oracle(run):
    from torch_oracle import TorchLlamaOracle
    regime, prompts, outs, weights, tol_rel, _ = run
    worst, n_tok, n_eq = 0.0, 0, 0
    for i in SAMPLE:
        got, lg = outs[i]
        want, margins, ref_lg = TorchLlamaOracle(weights).greedy(prompts[i], N_NEW, eos=(128001, 128008, 128009))
        for j, (g, w) in enumerate(zip(got, want)):
            std = float(np.std(ref_lg[j]))
            d = float(np.max(np.abs(lg[j] - ref_lg[j]))) / std
            worst = max(worst, d)
            assert d < tol_rel, (regime, i, j, d)
            assert np.corrcoef(lg[j], ref_lg[j])[0, 1] > 0.995
            n_tok += 1
            if g != w:
                # near-tie policy (DESIGN.md §5): either candidate is legitimate when the oracle's own
                # top-1/top-2 margin is inside twice the logit tolerance; continuations differ from here on
                assert margins[j] < 2 * tol_rel * std, (regime, i, j, got, want, margins)
                break
            n_eq += 1
    print(f"full-depth 8B [{regime}]: max |logit diff| vs bf16 torch oracle = {worst:.4f} logit std; "
          f"{n_eq}/{n_tok} compared tokens identical")
    assert n_eq >= 0.7 * n_tok


def test_full_depth_logits_match_huggingface_fp32(run):
    import torch
    from torch_oracle import hf_model_from_weights
    regime, prompts, outs, weights, tol_rel, hf_rel = run
    model = hf_model_from_weights(weights, "cuda:0")
    rels, agree, decided = [], 0, 0
    with torch.no_grad():
        for i in SAMPLE:
            got, lg = outs[i]
            ref = model(torch.tensor([prompts[i]], device="cuda:0")).logits[0, -1].float().cpu().numpy()
            diff = lg[0] - ref
            rms = float(np.sqrt(np.mean(diff ** 2)))
            rels.append(rms / float(np.std(ref)))
            top2 = np.partition(ref, -2)[-2:]
            if top2[1] - top2[0] > 8 * rms:          # HF's own choice is clear of the rounding noise
                decided += 1
                agree += int(got[0] == int(np.argmax(ref)))
            assert np.corrcoef(lg[0], ref)[0, 1] > 0.98
    del model
    torch.cuda.empty_cache()
    print(f"full-depth 8B [{regime}] vs HF fp32: relative RMS logit error {max(rels):.4f} (max over {len(rels)}); "
          f"arg-max agreement {agree}/{decided} where HF's margin > 8 sigma")
    assert max(rels) < hf_rel, rels
    assert agree == decided
