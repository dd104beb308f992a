"""The fused 32-channel residual unit's paired kernel (two output rows per MMA row, DESIGN §4.0) on the GPU.

Uniform rows of a fused RU(32) run the paired kernel; stacked rows (many streams with short chunks) and varlen rows run the unpaired
kernel with the same one-tap accumulation groups, so the two must agree bit for bit.  `adec_test_residual_unit` builds the op the way
the models do; ADEC_STACK_ROWS=0 makes a handle keep every stream in its own tiles, which selects the paired kernel."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

C, K = 32, 7


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def lib():
    from audiodec_b200 import _lib
    return _lib.load()


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    w1 = torch.randn(C, C, K, generator=g) * 1.2 / (K * C) ** 0.5
    w2 = torch.randn(C, C, 1, generator=g) * 0.6 / C ** 0.5
    return w1.numpy().copy(), w2.numpy().copy()


def _run(lib, x, w1, w2, d, state):
    from audiodec_b200 import _lib
    B, _, T = x.shape
    y = np.zeros((B, C, T), np.float32)
    rc = lib.adec_test_residual_unit(0, _p(x), B, C, T, _p(w1), _p(w2), K, d, _p(state), _p(y))
    assert rc == 0, _lib.last_error(None)
    return y


def test_wgmma_n64_columns_equal_n32(lib):
    """The premise of the paired kernel: column n of the fp16-split group as m64n64 equals, bit for bit, column n of the same group as
    m64n32 on that column's half of the weights.  Operands are random fp16 hi / lo pieces of the engine's magnitudes (weights scaled
    to [2^12, 2^13), W_his = 2^-11 W_hi), so partial sums carry and cancel in the low bits."""
    from audiodec_b200 import _lib
    rng = np.random.default_rng(5)
    x = rng.standard_normal((64, 32)).astype(np.float32)
    hi = x.astype(np.float16)
    lo = ((x - hi.astype(np.float32)) * 2048.0).astype(np.float16)
    w = (rng.standard_normal((32, 64)) * 2000.0).astype(np.float32)
    whi = w.astype(np.float16)
    wlo = (w - whi.astype(np.float32)).astype(np.float16)
    whis = (whi.astype(np.float32) / 2048.0).astype(np.float16)
    # [plane][kb][row][8]: K block kb holds channels 8 kb .. 8 kb + 7
    a = np.ascontiguousarray(np.stack([hi, lo]).reshape(2, 64, 4, 8).transpose(0, 2, 1, 3))
    b = np.ascontiguousarray(np.stack([whi, wlo, whis]).transpose(0, 2, 1).reshape(3, 64, 4, 8).transpose(0, 2, 1, 3))
    d64 = np.zeros((64, 64), np.float32)
    d32 = np.zeros((64, 64), np.float32)
    rc = lib.adec_test_wgmma_columns(0, _p(a), _p(b), _p(d64), _p(d32))
    assert rc == 0, _lib.last_error(None)
    exact = lo.astype(np.float64) @ whis.astype(np.float64) + hi.astype(np.float64) @ (wlo.astype(np.float64) + whi.astype(np.float64))
    assert np.abs(d64 - exact).max() <= 1e-5 * np.abs(exact).max()        # the operands went where the layout says
    np.testing.assert_array_equal(d64.view(np.uint32), d32.view(np.uint32))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("d", [1, 3, 9])
def test_paired_ru32_matches_fp64(lib, monkeypatch, d, B):
    """Two chained chunks whose lengths are not multiples of the paired tile (256 rows at dil 1, 252 at dil 3 and 9), against an
    fp64 model of residual_unit.py:78-81 on the same fp32 inputs, at the fp32-grade engine's 1e-5."""
    monkeypatch.setenv("ADEC_CONV_PATH", "f16")
    monkeypatch.setenv("ADEC_STACK_ROWS", "0")
    w1, w2 = _weights(100 + d)
    g = torch.Generator().manual_seed(7 * d + B)
    st = np.zeros((B, C, 6 * d), np.float32)
    st64 = torch.zeros(B, C, 6 * d, dtype=torch.float64)
    for T in (1000, 611):
        x = torch.randn(B, C, T, generator=g).numpy().copy()
        y = _run(lib, x, w1, w2, d, st)
        xx = torch.cat([st64, torch.nn.functional.elu(torch.from_numpy(x).double())], -1)
        st64 = xx[:, :, -6 * d:]
        mid = torch.nn.functional.conv1d(xx, torch.from_numpy(w1).double(), None, dilation=d)
        ref = torch.from_numpy(x).double() + torch.nn.functional.conv1d(torch.nn.functional.elu(mid), torch.from_numpy(w2).double())
        np.testing.assert_allclose(y, ref.numpy(), atol=1e-5, rtol=0)
        np.testing.assert_allclose(st, st64.numpy(), atol=1e-6)


@pytest.mark.parametrize("B,T", [(3, 20), (8, 40)])
@pytest.mark.parametrize("d", [1, 3, 9])
def test_paired_equals_stacked_bitwise(lib, monkeypatch, d, B, T):
    """Short chunks of several streams: stacked rows (unpaired kernel) and one tile per stream (paired kernel) give the same outputs
    and the same causal state, bit for bit, over three chained chunks."""
    monkeypatch.setenv("ADEC_CONV_PATH", "f16")
    w1, w2 = _weights(200 + d)
    g = torch.Generator().manual_seed(11 * d + B)
    st_s = (0.5 * torch.randn(B, C, 6 * d, generator=g)).numpy().copy()
    st_p = st_s.copy()
    for _ in range(3):
        x = torch.randn(B, C, T, generator=g).numpy().copy()
        monkeypatch.setenv("ADEC_STACK_ROWS", "1")
        y_s = _run(lib, x, w1, w2, d, st_s)
        monkeypatch.setenv("ADEC_STACK_ROWS", "0")
        y_p = _run(lib, x, w1, w2, d, st_p)
        np.testing.assert_array_equal(y_p, y_s)
        np.testing.assert_array_equal(st_p, st_s)
