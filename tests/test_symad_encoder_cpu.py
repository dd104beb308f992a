"""CPU-only checks of the symAD encoder-only generator: its config, its dtype rules, and what it does not have."""
import inspect

import pytest
import torch

from audiodec_b200 import synthetic as S


def test_encoder_only_config_mirrors_the_full_generator():
    from audiodec_b200 import _lib
    from audiodec_b200.codec import SymADEncoderStreamGenerator, SymADStreamGenerator
    for params in (S.SYMAD_PARAMS, S.SYMAAD_PARAMS, S.SYMAD_C16_PARAMS):
        e, f = SymADEncoderStreamGenerator(**params), SymADStreamGenerator(**params)
        assert e._cfg.model_type == _lib.MODEL_SYMAD_ENCODER == 3 and f._cfg.model_type == _lib.MODEL_SYMAD
        for name, _ in _lib.AdecConfig._fields_:
            if name != "model_type":
                a, b = getattr(e._cfg, name), getattr(f._cfg, name)
                assert (list(a) if hasattr(a, "__len__") else a) == (list(b) if hasattr(b, "__len__") else b), name
        assert e.code_dim == f.code_dim and e.enc_strides == f.enc_strides
        for name in ("decode", "lookup", "lookup_packed", "unpack", "decode_offline", "quantize_forward", "zq_moments"):
            assert not hasattr(e, name), name
        for name in ("initial_encoder", "encode", "quantize", "quantize_fused", "quantize_offline", "pack", "encode_offline", "encode_offline_varlen",
                     "encode_streams", "state_dict", "stream_state", "load_stream_state", "set_streams", "copy_stream_state"):
            assert callable(getattr(e, name)), name
    with pytest.raises(NotImplementedError):
        SymADEncoderStreamGenerator(codec="unknown")
    params = inspect.signature(SymADEncoderStreamGenerator.__init__).parameters
    assert list(params)[0] == "self" and set(S.SYMAD_PARAMS) <= set(params) and params["enc_strides"].default == (3, 4, 5, 5)


def test_encoder_only_dtype_modes():
    """The decoder-only generators' rules: .to(bfloat16) = mode 1, set_activation_dtype(bfloat16) = mode 2 in either call order,
    float32 activations return to the operand mode; fp16 is not built."""
    from audiodec_b200.codec import SymADEncoderStreamGenerator
    e = SymADEncoderStreamGenerator(**S.SYMAD_PARAMS)
    assert e._cfg.compute_dtype == 0
    assert e.to(torch.bfloat16) is e and e._cfg.compute_dtype == 1 and e.state_dtype == torch.float32
    assert e.set_activation_dtype(torch.bfloat16) is e and e._cfg.compute_dtype == 2
    assert e.state_dtype == torch.bfloat16 and e._act_dtype == torch.bfloat16
    e.to(torch.float32)
    assert e._cfg.compute_dtype == 2
    e.set_activation_dtype(torch.float32)
    assert e._cfg.compute_dtype == 0
    e.bfloat16()
    assert e._cfg.compute_dtype == 1
    with pytest.raises(NotImplementedError):
        e.to(torch.float16)
    with pytest.raises(NotImplementedError):
        e.set_activation_dtype(torch.float16)


def test_new_symbols_are_bound():
    from audiodec_b200 import _lib
    for name in ("adec_encode_bf16", "adec_encode_offline_bf16", "adec_encode_offline_varlen_bf16", "adec_encode_streams_bf16",
                 "adec_quantize_bf16", "adec_quantize_ex_bf16"):
        assert name in _lib.SYMBOLS, name


def test_transmitter_graph_and_codec_check_take_the_encoder_only_class():
    from audiodec_b200.codec import SymADEncoderStreamGenerator, TransmitterGraph, is_library_codec
    e = SymADEncoderStreamGenerator(**S.SYMAD_PARAMS)
    assert not is_library_codec(e, e, e)                 # no handle yet, and it has no codebooks to serve as rx_encoder
    with pytest.raises(RuntimeError, match="call .to"):
        TransmitterGraph(e, 1, 1500)
