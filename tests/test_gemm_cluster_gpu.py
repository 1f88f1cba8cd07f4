"""The persistent prefill GEMM runs as 2-CTA clusters: the CTAs of a cluster take m-tiles 2p and 2p+1 of one
n-tile and multicast halves of the activation tile to each other.  These cases cover the edges of that split
(one m-tile, an odd m-tile count, fewer tile pairs than clusters, ragged M and N) in every flavour; the tiled
kernel is the reference, bit for bit (same k order per output element)."""
import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from test_fp8_gpu import _operands, gemm_fp8
from test_gemm_gpu import _gemm, _rand_bits

pytestmark = pytest.mark.gpu


def test_persistent_cluster_count():
    lib = _lib.load()
    for fp8 in (0, 1):
        for epi in (0, 1, 3):
            c = lib.acp_kernel_gemm_persistent_clusters(fp8, epi)
            assert c > 0, (fp8, epi, c)


@pytest.mark.parametrize("M,N,K,epi", [
    (128, 300, 256, 0),       # one m-tile: the second CTA of every cluster has no W tile and stores nothing
    (256, 600, 256, 0),       # 3 tile pairs, far fewer than co-resident clusters
    (200, 520, 128, 0),       # ragged M inside the pair, ragged last n-tile
    (2688, 2600, 192, 0),     # 21 m-tiles (odd) x 11 n-tiles: several pairs per cluster
    (384, 700, 320, 3),       # SwiGLU, odd m-tiles, ragged last n-tile (188 rows)
    (2048, 1100, 256, 3),     # SwiGLU, ragged last n-tile (76 rows)
    (384, 700, 256, 1),       # one fp32 plane, odd m-tiles
])
def test_persistent_cluster_edges_match_tiled(M, N, K, epi):
    rng = np.random.default_rng(M * 7 + N + K + epi)
    w = _rand_bits(rng, (M, K), 0.05)
    x = _rand_bits(rng, (N, K), 1.0)
    tiled, _, _, _ = _gemm(w, x, epi=epi, bn=256)
    pers, _, _, _ = _gemm(w, x, epi=epi, bn=-1)
    assert np.array_equal(tiled, pers), int(np.count_nonzero(tiled != pers))


@pytest.mark.parametrize("epi", [0, 3])
@pytest.mark.parametrize("M,K,N", [(384, 512, 700), (128, 256, 300), (2688, 1024, 1500)])
def test_fp8_persistent_cluster_edges_match_tiled(M, K, N, epi):
    rng = np.random.default_rng(M + N + K + epi)
    w, s_w, x, s_x = _operands(rng, M, N, K)
    a, _ = gemm_fp8(w, s_w, x, s_x, epi=epi, bn=-1)
    b, _ = gemm_fp8(w, s_w, x, s_x, epi=epi, bn=128)
    assert np.array_equal(a, b)
