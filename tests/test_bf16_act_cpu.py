"""CPU-only checks of the vocoder's bf16-activation mode (compute_dtype 2): the Python-side mode selection and its rejections, the
bf16 decode entry points in the binding table, and the server's widening of a bf16 decoder output to float32 frames."""
import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S


def test_bindings_declare_the_bf16_decode_entry_points():
    from audiodec_b200 import _lib
    for name in ("adec_decode_bf16", "adec_decode_offline_bf16"):
        res, args = _lib.SYMBOLS[name]
        assert res is _lib.c_int and len(args) == 6


def test_set_activation_dtype_selects_compute_dtype():
    from audiodec_b200.codec import HiFiGANStreamGenerator
    d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    assert d.set_activation_dtype(torch.bfloat16) is d                  # chainable: d.set_activation_dtype(...).to(dev)
    assert d._cfg.compute_dtype == 2
    d.set_activation_dtype(torch.float32)
    assert d._cfg.compute_dtype == 0
    # float32 activations return to whatever .to(dtype) chose, in either call order
    d.to(torch.bfloat16).set_activation_dtype(torch.bfloat16)
    assert d._cfg.compute_dtype == 2
    d.to(torch.float32)
    assert d._cfg.compute_dtype == 2                                   # operand dtype alone does not leave the bf16-activation mode
    d.to(torch.bfloat16)
    d.set_activation_dtype(torch.float32)
    assert d._cfg.compute_dtype == 1
    d.to(torch.float32)
    assert d._cfg.compute_dtype == 0


def test_set_activation_dtype_rejections():
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).set_activation_dtype(torch.bfloat16)   # the encoder side stays fp32-grade
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).set_activation_dtype(torch.float32)
    with pytest.raises(NotImplementedError):
        HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS).set_activation_dtype(torch.float16)


def test_server_widens_bf16_decoder_output_to_float32_frames():
    from audiodec_b200.server import MultiStreamCodecServer

    class Bf16Vocoder:                       # stand-in with the surface of a bf16-activation HiFiGANStreamGenerator
        def encode(self, x):
            return x

        quantize = lookup = encode

        def decode(self, zq):
            return (0.5 * zq).to(torch.bfloat16)

    c = Bf16Vocoder()
    srv = MultiStreamCodecServer(c, c, c, n_streams=3, frame_size=8, sample_rate=8000, max_latency=1.0)
    frames = np.arange(24, dtype=np.float32).reshape(3, 8) / 32.0     # exact in bf16
    for s in range(3):
        srv.submit(s, frames[s])
    assert srv.step() == 3
    for s in range(3):
        out = srv.poll(s)
        assert out.dtype == np.float32 and out.shape == (8,)
        np.testing.assert_array_equal(out, 0.5 * frames[s])
