"""The persistent prefill GEMM hands every finished tile to its epilogue warps through one whole-tile staging
buffer per CTA, which they store (bf16) or turn into SwiGLU outputs while the consumers run the next tile.
At prefill sizes each CTA reuses that buffer for many tiles, so these cases check the hand-over at the
Llama-3-8B layer shapes (N = 4096 tokens) and at an odd m-tile count with several pairs per cluster, ragged M
and a ragged last n-tile.  The tiled kernel is the reference, bit for bit; the test hooks also fail if any
store lands past the end of the output."""
import numpy as np
import pytest

from test_fp8_gpu import _operands, gemm_fp8
from test_gemm_gpu import _gemm, _rand_bits

pytestmark = pytest.mark.gpu

CASES = [
    (28672, 4096, 256, 3),    # gate/up + SwiGLU: 112 m-tiles x 16 n-tiles, ~27 tiles per CTA
    (6144, 4096, 256, 0),     # QKV, bf16 out
    (5720, 4196, 192, 0),     # 45 m-tiles (odd, the last ragged), last n-tile of 100 tokens (68 for FP8)
    (5720, 4196, 192, 3),     # the same with SwiGLU; 2860 output columns: rows not 16-byte aligned
]


@pytest.mark.parametrize("M,N,K,epi", CASES)
def test_persistent_staged_epilogue_matches_tiled(M, N, K, epi):
    rng = np.random.default_rng(M + N + K + epi)
    w = _rand_bits(rng, (M, K), 0.05)
    x = _rand_bits(rng, (N, K), 1.0)
    tiled, _, _, _ = _gemm(w, x, epi=epi, bn=256)
    pers, _, _, _ = _gemm(w, x, epi=epi, bn=-1)
    assert np.array_equal(tiled, pers), int(np.count_nonzero(tiled != pers))


@pytest.mark.parametrize("M,N,K,epi", CASES)
def test_fp8_persistent_staged_epilogue_matches_tiled(M, N, K, epi):
    rng = np.random.default_rng(M + N + K + epi + 1)
    w, s_w, x, s_x = _operands(rng, M, N, K)
    a, _ = gemm_fp8(w, s_w, x, s_x, epi=epi, bn=-1)
    b, _ = gemm_fp8(w, s_w, x, s_x, epi=epi, bn=128)
    assert np.array_equal(a, b), int(np.count_nonzero(a != b))
