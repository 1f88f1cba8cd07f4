"""FP8 (e4m3) numerics without a GPU: the oracle's e4m3 codec and row quantiser (oracle/fp8.py) against
torch and ml_dtypes, the FP8 presets, and the FP8 forward pass against the bf16 one."""
import numpy as np
import pytest

from oracle.bf16 import bits_to_f32
from oracle.fp8 import (E4M3_MAX, FP8_PRESETS, Fp8LlamaOracle, e4m3_decode, e4m3_encode, fp8_matmul,
                        quantize_rows)
from oracle.llama_oracle import PRESETS, LlamaOracle

SEED = 0xACB200


def _bf16_values_within_range():
    v = bits_to_f32(np.arange(1 << 16, dtype=np.uint32).astype(np.uint16))
    return v[np.isfinite(v) & (np.abs(v) <= E4M3_MAX)]


def test_encode_equals_torch_on_every_bf16_value():
    """Every finite bf16 value within +-448: ties (e4m3 midpoints have 5 significant bits), subnormals,
    +-0 and the +-448 boundary are all among them."""
    torch = pytest.importorskip("torch")
    v = _bf16_values_within_range()
    want = torch.from_numpy(v).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert np.array_equal(e4m3_encode(v), want)
    for probe in (0.0, -0.0, 448.0, -448.0, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -6, 17.0, 19.0, 432.0, 440.0):
        t = torch.tensor([probe], dtype=torch.float32).to(torch.float8_e4m3fn).view(torch.uint8).item()
        assert e4m3_encode(np.array([probe], np.float32))[0] == t, probe


def test_encode_equals_ml_dtypes_on_every_bf16_value():
    ml_dtypes = pytest.importorskip("ml_dtypes")
    v = _bf16_values_within_range()
    assert np.array_equal(e4m3_encode(v), v.astype(ml_dtypes.float8_e4m3fn).view(np.uint8))


def test_decode_roundtrips_every_finite_code():
    codes = np.array([c for c in range(256) if (c & 0x7F) != 0x7F], np.uint8)
    vals = e4m3_decode(codes)
    back = e4m3_encode(vals)
    assert np.array_equal(back[codes != 0x80], codes[codes != 0x80])   # -0 encodes back to 0x80
    assert e4m3_decode(np.array([0x7E]))[0] == 448.0 and e4m3_decode(np.array([0x01]))[0] == 2.0 ** -9


def test_encode_refuses_out_of_range():
    with pytest.raises(ValueError):
        e4m3_encode(np.array([465.0], np.float32))


def test_row_quantizer():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((4, 256)) * np.array([[1e-3], [1.0], [30.0], [1.0]])).astype(np.float32)
    x[3] = 0.0
    x[3, 1::2] = -0.0
    codes, s = quantize_rows(x)
    assert s[3] == 1.0 and np.array_equal(codes[3], np.tile([0x00, 0x80], 128))   # zero row: s = 1, signed zeros
    amax = np.max(np.abs(x[:3]), axis=1)
    assert np.array_equal(s[:3], (amax / np.float32(448)).astype(np.float32))
    for r in range(3):                                                 # the amax element maps to +-448
        assert np.abs(e4m3_decode(codes[r])).max() == 448.0
    deq = e4m3_decode(codes[:3]) * s[:3, None]
    assert np.all(np.abs(deq - x[:3]) <= np.abs(x[:3]) * 2.0 ** -4 + s[:3, None] * 2.0 ** -9)


def test_fp8_matmul_is_exact_then_scaled():
    rng = np.random.default_rng(1)
    w, s_w = quantize_rows(rng.standard_normal((64, 512)).astype(np.float32))
    x, s_x = quantize_rows(rng.standard_normal((8, 512)).astype(np.float32))
    y = fp8_matmul(x, s_x, w, s_w)
    acc = np.array([[float(sum(float(a) * float(b) for a, b in zip(e4m3_decode(x[n]), e4m3_decode(w[m]))))
                     for m in range(4)] for n in range(2)], np.float32)
    assert np.array_equal(y[:2, :4], ((acc * s_w[None, :4]).astype(np.float32) * s_x[:2, None]).astype(np.float32))


def test_presets_mirror_their_bf16_base():
    assert sorted(FP8_PRESETS) == sorted(f"{b}-fp8" for b in ("tiny", "tiny-g2", "tiny-g8", "llama-3-8b-l2", "llama-3-8b"))
    for name, cfg in FP8_PRESETS.items():
        base = PRESETS[cfg.base]
        assert name == base.name + "-fp8"
        for f in ("hidden", "layers", "heads", "kv_heads", "ffn", "vocab", "rope_theta", "w_std", "experts"):
            assert getattr(cfg, f) == getattr(base, f), (name, f)


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_fp8_forward_stays_close_to_bf16(mode):
    """FP8 projections move the logits, but by a small fraction of their spread."""
    rng = np.random.default_rng(2)
    prompt = [128000] + [int(t) for t in rng.integers(0, 256, size=20)]
    a = Fp8LlamaOracle(FP8_PRESETS["tiny-fp8"], SEED, mode=mode).forward(prompt)[-1]
    b = LlamaOracle(PRESETS["tiny"], SEED, mode=mode).forward(prompt)[-1]
    assert 0 < np.max(np.abs(a - b)) < 0.5 * np.std(b)
