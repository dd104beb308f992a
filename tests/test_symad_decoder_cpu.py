"""CPU-only checks of the symAD decoder-only generator: its config, the bf16 mode selection it shares with the vocoder, and the
refusals of the full symAD generator, which stay."""
import pytest
import torch

from audiodec_b200 import synthetic as S


def test_decoder_only_config_mirrors_the_full_generator():
    from audiodec_b200 import _lib
    from audiodec_b200.codec import SymADDecoderStreamGenerator, SymADStreamGenerator
    for params in (S.SYMAD_PARAMS, S.SYMAAD_PARAMS, S.SYMAD_C16_PARAMS):
        d, f = SymADDecoderStreamGenerator(**params), SymADStreamGenerator(**params)
        assert d._cfg.model_type == _lib.MODEL_SYMAD_DECODER == 2 and f._cfg.model_type == _lib.MODEL_SYMAD
        for name, _ in _lib.AdecConfig._fields_:
            if name != "model_type":
                a, b = getattr(d._cfg, name), getattr(f._cfg, name)
                assert (list(a) if hasattr(a, "__len__") else a) == (list(b) if hasattr(b, "__len__") else b), name
        assert d.code_dim == f.code_dim and not hasattr(d, "encode") and not hasattr(d, "quantize") and not hasattr(d, "lookup")
    with pytest.raises(NotImplementedError):
        SymADDecoderStreamGenerator(codec="unknown")
    import inspect
    for cls in (SymADDecoderStreamGenerator, SymADStreamGenerator):       # the reference's generator_params keywords
        params = inspect.signature(cls.__init__).parameters
        assert list(params)[0] == "self" and set(S.SYMAD_PARAMS) <= set(params) and params["enc_strides"].default == (3, 4, 5, 5)


def test_decoder_only_dtype_modes():
    """The vocoder's rules: .to(bfloat16) = mode 1, set_activation_dtype(bfloat16) = mode 2 in either call order, float32
    activations return to the operand mode."""
    from audiodec_b200.codec import SymADDecoderStreamGenerator
    d = SymADDecoderStreamGenerator(**S.SYMAD_PARAMS)
    assert d._cfg.compute_dtype == 0
    assert d.to(torch.bfloat16) is d and d._cfg.compute_dtype == 1
    assert d.set_activation_dtype(torch.bfloat16) is d and d._cfg.compute_dtype == 2
    d.to(torch.float32)
    assert d._cfg.compute_dtype == 2
    d.set_activation_dtype(torch.float32)
    assert d._cfg.compute_dtype == 0
    d.bfloat16()
    assert d._cfg.compute_dtype == 1
    with pytest.raises(NotImplementedError):
        d.set_activation_dtype(torch.float16)
    with pytest.raises(NotImplementedError):
        d.to(torch.float16)


def test_full_generator_keeps_its_refusals():
    from audiodec_b200.codec import SymADStreamGenerator
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).to(torch.bfloat16)
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).set_activation_dtype(torch.bfloat16)
