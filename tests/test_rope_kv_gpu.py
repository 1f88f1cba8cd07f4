"""rope_kv_kernel (agentcontrolplane_b200/csrc/kernels.cu) -- the RoPE + paged K/V scatter that writes everything the
prefill attention kernels read -- bit-exact against oracle/attention_oracle.py through the hook acp_kernel_rope_kv
(include/acp_infer_kernels.h): rows of several sequences at page and table edges up to position 131071 (Llama-3.1
scaled tables), bf16 or split-K fp32 input, no store outside the rows' cache slots and q rows."""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from oracle import attention_oracle as ao
from oracle.bf16 import bf16_round, bf16_round_to_bits, bits_to_f32
from llama31_presets import LLAMA31
from oracle.llama_oracle import rope_tables

pytestmark = pytest.mark.gpu

POSITIONS = [0, 1, 31, 32, 4095, 4096, 131071]
HEADS, KV_HEADS = 8, 2


def _rope_kv(qkv, splits, seq, pos, B, cos, sin, stale=0):
    lib = _lib.load()
    T = len(pos)
    u16p, f32p, i32p = (ctypes.POINTER(t) for t in (ctypes.c_uint16, ctypes.c_float, ctypes.c_int))
    lib.acp_kernel_rope_kv.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, i32p, i32p,
                                       ctypes.c_int, f32p, f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_uint16, u16p, u16p, u16p]
    data = bf16_round_to_bits(qkv) if splits == 0 else np.ascontiguousarray(qkv, np.float32)
    seq_a, pos_a = np.asarray(seq, np.int32), np.asarray(pos, np.int32)
    q = np.zeros((T, HEADS, 128), np.uint16)
    k = np.zeros((T, KV_HEADS, 128), np.uint16)
    v = np.zeros_like(k)
    rc = lib.acp_kernel_rope_kv(data.ctypes.data, splits, T + 5, T, seq_a.ctypes.data_as(i32p),
                                pos_a.ctypes.data_as(i32p), B, cos.ctypes.data_as(f32p), sin.ctypes.data_as(f32p),
                                cos.shape[0], HEADS, KV_HEADS, stale, q.ctypes.data_as(u16p), k.ctypes.data_as(u16p),
                                v.ctypes.data_as(u16p))
    assert rc == 0, f"acp_kernel_rope_kv rc={rc}"
    return q, k, v


@pytest.fixture(scope="module")
def tables():
    return tuple(np.ascontiguousarray(t) for t in rope_tables(LLAMA31["tiny-3.1"], 131072))


def _rows():
    """three sequences; every position of POSITIONS in sequence 1, a few in the others (rows interleaved)"""
    seq, pos = [], []
    for p in POSITIONS:
        seq.append(1); pos.append(p)
    for p in (0, 33, 4096):
        seq.append(0); pos.append(p)
    for p in (31, 131071):
        seq.append(2); pos.append(p)
    order = np.random.default_rng(0).permutation(len(seq))
    return [seq[i] for i in order], [pos[i] for i in order]


def _expect(x, pos, cos, sin):
    """reduced QKV rows [T][ld] -> q, k, v bf16 values"""
    qd, kvd = HEADS * 128, KV_HEADS * 128
    c, s = cos[pos][:, None, :], sin[pos][:, None, :]
    q = ao.rope(x[:, :qd].reshape(-1, HEADS, 128), c, s)
    k = ao.rope(x[:, qd:qd + kvd].reshape(-1, KV_HEADS, 128), c, s)
    return q, k, x[:, qd + kvd:].reshape(-1, KV_HEADS, 128)


@pytest.mark.parametrize("splits", [0, 1, 9])
def test_rope_kv_is_bit_exact(tables, splits):
    """random fp32 split-K planes (not exact sums) are reduced in index order like the oracle's reduce_planes"""
    cos, sin = tables
    seq, pos = _rows()
    rng = np.random.default_rng(splits)
    ld = (HEADS + 2 * KV_HEADS) * 128
    if splits == 0:
        data = bf16_round(rng.standard_normal((len(pos), ld)).astype(np.float32))
        x = data
    else:
        data = (rng.standard_normal((splits, len(pos), ld)) / np.sqrt(splits)).astype(np.float32)
        x = ao.reduce_planes(data)
    got = _rope_kv(data, splits, seq, pos, 3, cos, sin, stale=0xFFFF)
    for g, want, name in zip(got, _expect(x, np.asarray(pos), cos, sin), "qkv"):
        assert np.array_equal(bits_to_f32(g), want), name


def test_split_k_planes_that_sum_to_the_bf16_rows_give_its_bits(tables):
    cos, sin = tables
    seq, pos = _rows()
    rng = np.random.default_rng(7)
    x = bf16_round(rng.standard_normal((len(pos), (HEADS + 2 * KV_HEADS) * 128)).astype(np.float32))
    base = _rope_kv(x, 0, seq, pos, 3, cos, sin)
    for splits in (1, 9):
        got = _rope_kv(ao.split_exact(x, splits, rng), splits, seq, pos, 3, cos, sin)
        for a, b in zip(base, got):
            assert np.array_equal(a, b), splits
