"""Whole fp32 decoders and vocoders against fp64: the checker tests/test_models_fp64_gpu.py holds the released models to, and its
controls, on the oracle alone (no GPU).

A model's waveform `got` passes when

    max |got - y64| <= factor * max(e32, 2^-23 * max |y64|),   e32 = max |y32 - y64|,

where y64 is the oracle run in fp64 and y32 the oracle run in fp32 (the reference's own arithmetic), both on the same fp32 latents from
the same warm state.  Every live pad_buffer is held to the same rule with its own e32; a buffer whose op applies ELU to its input may
also differ by act_elu's documented 2.4e-7 absolute error.  The op tests (test_conv_fp32_layers_gpu.py) build each op from their own
weights; this rule is what sees a plan that wires a real checkpoint's ops wrongly or packs a layer's weights at the wrong precision.

Negative controls: the fp64 oracle with one causal conv of the symAD decoder or of HiFi-GAN v1 degraded to what a broken fp32-grade
path leaves (its weights rounded to 1xTF32, or its operands and state rounded to fp16) must fail check_model, though most of these pass
the parity tests' 1e-4 max-abs tolerance.  A state window one row off in one layer must fail check_states, which names that layer.
Positive controls: the fp32 oracle itself, and the oracle with a model of the kernels' ELU, pass."""
import functools
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from audiodec_b200 import synthetic as S
from oracle import audiodec_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FLOOR = 2.0 ** -23
ELU_ABS = 2.4e-7        # act_elu (csrc/kernels.cuh): within 2.4e-7 ABSOLUTE of expm1
WAVE_TOL = 1e-4         # the parity tests' max-abs tolerance
RECEPTIVE = 8192        # load_receiver's warm-up length (bin/stream.py:70)

MODELS = {   # name -> (encoder params, vocoder params or None, the parity tests' golden clip)
    "symAD": ("SYMAD_PARAMS", None, "symad_oneshot.npz"),
    "symAAD": ("SYMAAD_PARAMS", None, "aad_oneshot.npz"),
    "c16": ("SYMAD_C16_PARAMS", None, "c16_oneshot.npz"),
    "v0": ("SYMAD_PARAMS", "HIFIGAN_V0_PARAMS", "v0_oneshot.npz"),
    "v1": ("SYMAD_PARAMS", "HIFIGAN_V1_PARAMS", "v1_oneshot.npz"),
    "v2": ("SYMAD_PARAMS", "HIFIGAN_V2_PARAMS", "v2_oneshot.npz"),
}


@functools.lru_cache(None)
def weights(model):
    """(encoder params, encoder state dict, vocoder params or None, vocoder state dict or None): the parity tests' seeds"""
    ep, vp, _ = MODELS[model]
    ep, vp = getattr(S, ep), getattr(S, vp) if vp else None
    return ep, S.symad_state_dict(ep, seed=0), vp, S.hifigan_state_dict(vp, seed=1) if vp else None


def golden_x(model):
    return torch.from_numpy(np.load(os.path.join(GOLDEN, MODELS[model][2]))["x"])


def decoder_oracle(model, dtype):
    ep, esd, vp, vsd = weights(model)
    return O.SymADOracle(ep, esd, dtype=dtype) if vp is None else O.HiFiGANOracle(vp, vsd, dtype=dtype)


def elu_keys(model):
    """the pad_buffers whose op applies ELU to its input: every residual unit's dilated conv; symAAD also the transposed convs, the
    head and the projector"""
    ep, _, vp, _ = weights(model)
    if vp is not None:
        return set()
    act = ep.get("codec") == "activate_audiodec"
    keys = {f"encoder.conv_blocks.{i}.res_units.{j}.conv1.pad_buffer" for i in range(len(ep["enc_strides"])) for j in range(3)}
    for i in range(len(ep["dec_strides"])):
        pre = f"decoder.conv_blocks.{i}.1" if act else f"decoder.conv_blocks.{i}"
        keys |= {f"{pre}.res_units.{j}.conv1.pad_buffer" for j in range(3)}
        if act:
            keys.add(f"{pre}.conv.pad_buffer")
    if act:
        keys |= {"decoder.conv2.pad_buffer", "projector.project.pad_buffer"}
    return keys


def pad_buffers(o):
    """the oracle's causal state, keyed as the reference names its pad_buffers, in fp64"""
    return OrderedDict((k + ".pad_buffer", v.double()) for k, v in o.state.items())


def oracle_warm_zq(model):
    """load_receiver's warm-up latents from the fp32 oracle: rx_encoder.initial_encoder(8192)"""
    ep, esd, _, _ = weights(model)
    return O.SymADOracle(ep, esd).initial_encoder(RECEPTIVE)


def run_oracle(model, dtype, zq, zq_warm, mode):
    """The oracle decoder in `dtype` on fp32 latents zq (1, F, D), widened exactly.  mode "stream": one streaming call; an int n:
    streaming calls of n frames; both after initial_decoder(zq_warm).  "offline": Decoder.forward / Generator.forward from zero state
    (transposed convs replicate the first frame).  -> (y (1, 1, F * hop) fp64, pad_buffers after the last call or None)"""
    o = decoder_oracle(model, dtype)
    if mode == "offline":
        f = o.forward_decode if isinstance(o, O.SymADOracle) else o.forward
        return f(zq.transpose(1, 2)).double(), None
    o.initial_decoder(zq_warm)
    n = zq.shape[1] if mode == "stream" else mode
    y = torch.cat([o.decode(zq[:, i:i + n]) for i in range(0, zq.shape[1], n)], -1)
    return y.double(), pad_buffers(o)


# ------------------------------------------------------------------------------------------------------------------------------
# the checker
# ------------------------------------------------------------------------------------------------------------------------------
def check_model(got, y32, y64, factor, slack=0.0):
    """(passed, e, e32, bar): got passes when e = max |got - y64| <= bar = factor * max(e32, 2^-23 * max |y64|) + slack, with
    e32 = max |y32 - y64|.  A NaN in got fails."""
    got, y32, y64 = (torch.as_tensor(t).double().cpu() for t in (got, y32, y64))
    assert got.shape == y32.shape == y64.shape, (tuple(got.shape), tuple(y32.shape), tuple(y64.shape))
    if got.numel() == 0:
        return True, 0.0, 0.0, 0.0
    e = (got - y64).abs().max().item()
    e32 = (y32 - y64).abs().max().item()
    bar = factor * max(e32, FLOOR * y64.abs().max().item()) + slack
    return bool(e <= bar), e, e32, bar


def check_states(got, st32, st64, factor, elu_keys=()):
    """Every pad_buffer of st64, in st64's order (layer order), by check_model's rule with its own e32; keys in elu_keys also get
    ELU_ABS.  -> (the first key that fails or None, [(key, e, e32, bar)])"""
    bad, rows = None, []
    for k, s64 in st64.items():
        ok, e, e32, bar = check_model(got[k], st32[k], s64, factor, ELU_ABS if k in elu_keys else 0.0)
        rows.append((k, e, e32, bar))
        if not ok and bad is None:
            bad = k
    return bad, rows


# ------------------------------------------------------------------------------------------------------------------------------
# controls, on the golden clip's codes from the warm fp32 oracle encoder, decoded from load_receiver's warm state
# ------------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def clip_zq(model):
    """the golden clip through the warm fp32 oracle transmitter (bin/stream.py:61): zq (1, F, D); its indices are the golden file's"""
    ep, esd, _, _ = weights(model)
    tx = O.SymADOracle(ep, esd)
    tx.initial_encoder(RECEPTIVE)
    idx = tx.quantize(tx.encode(golden_x(model)))
    np.testing.assert_array_equal(idx.numpy(), np.load(os.path.join(GOLDEN, MODELS[model][2]))["idx"])
    return tx.lookup(idx)


@functools.lru_cache(None)
def reference_run(model):
    """(y32, st32, y64, st64): one streaming call over the clip, fp32 and fp64"""
    zq, zw = clip_zq(model), oracle_warm_zq(model)
    y32, st32 = run_oracle(model, torch.float32, zq, zw, "stream")
    y64, st64 = run_oracle(model, torch.float64, zq, zw, "stream")
    return y32, st32, y64, st64


def _tf32(t):
    """round to 1xTF32 (10-bit mantissa, ties away from zero), as a tensor-core path without the split would take the operand"""
    u = t.float().view(torch.int32)
    return ((u + 0x1000) & ~0x1FFF).view(torch.float32).to(t.dtype)


def _fp16(t):
    return t.half().to(t.dtype)


def _degrade(monkeypatch, n_layers, target, defect):
    """the oracle's causal_conv1d_infer with layer `target` (of n_layers per decode call, in call order) degraded: "w_tf32" rounds
    its weights to 1xTF32, "a_fp16" its operands and state to fp16"""
    real = O.causal_conv1d_infer
    calls = [0]

    def conv(x, w, b, state, stride=1, dilation=1, groups=1):
        hit = calls[0] % n_layers == target
        calls[0] += 1
        if hit and defect == "w_tf32":
            w = _tf32(w)
        elif hit:
            x, state = _fp16(x), _fp16(state)
        return real(x, w, b, state, stride, dilation, groups)
    monkeypatch.setattr(O, "causal_conv1d_infer", conv)


def _n_layers(model, monkeypatch):
    """causal_conv1d_infer calls per decode call of the model's decoder"""
    real = O.causal_conv1d_infer
    calls = [0]
    zq = clip_zq(model)[:, :1]

    def conv(*a, **k):
        calls[0] += 1
        return real(*a, **k)
    with monkeypatch.context() as m:
        m.setattr(O, "causal_conv1d_infer", conv)
        decoder_oracle(model, torch.float64).decode(zq)
    return calls[0]


@pytest.mark.parametrize("model,n_expected", [("symAD", 14), ("v1", 26)])
def test_checker_rejects_one_degraded_layer(model, n_expected, monkeypatch):
    """Every causal conv of the decoder, one at a time, with its weights rounded to 1xTF32 and, separately, its operands and state
    rounded to fp16: check_model (factor 4) rejects every case.  In at least half of the layers, one of the two defects passes the
    parity tests' 1e-4."""
    n = _n_layers(model, monkeypatch)
    assert n == n_expected
    y32, _, y64, _ = reference_run(model)
    zq, zw = clip_zq(model), oracle_warm_zq(model)
    passed, hidden, lines = [], set(), []
    for defect in ("w_tf32", "a_fp16"):
        for target in range(n):
            with monkeypatch.context() as m:
                _degrade(m, n, target, defect)
                y, _ = run_oracle(model, torch.float64, zq, zw, "stream")
            ok, e, e32, bar = check_model(y, y32, y64, 4.0)
            if e <= WAVE_TOL:
                hidden.add(target)
            lines.append(f"{model} layer {target:2d} {defect}: e = {e:.3g} ({e / e32:.0f} e32), within 1e-4: {e <= WAVE_TOL}")
            if ok:
                passed.append(lines[-1])
    print("\n".join(lines))
    print(f"{model}: {len(hidden)} of {n} layers have a defect within 1e-4; {len(passed)} degraded decoders pass check_model")
    assert not passed, passed
    assert 2 * len(hidden) >= n, f"{model}: only {len(hidden)} of {n} layers have a defect within 1e-4"


@pytest.mark.parametrize("model,key", [("symAD", "decoder.conv_blocks.1.res_units.2.conv1.pad_buffer"),
                                       ("symAD", "decoder.conv2.pad_buffer"),
                                       ("v1", "input_conv.pad_buffer"),
                                       ("v1", "blocks.2.convs1.1.pad_buffer")])
def test_checker_names_a_state_window_one_row_off(model, key, monkeypatch):
    """The fp64 state with one causal conv's window ending one row early (its last P rows of state || input, shifted back by one):
    check_states rejects it and names that layer's key; every other key passes."""
    _, st32, _, st64 = reference_run(model)
    real = O.causal_conv1d_infer
    shifted = []

    def conv(x, w, b, state, stride=1, dilation=1, groups=1):
        y, new = real(x, w, b, state, stride, dilation, groups)
        shifted.append((new, torch.cat((state, x), -1)[:, :, -new.shape[-1] - 1:-1]))
        return y, new
    monkeypatch.setattr(O, "causal_conv1d_infer", conv)
    run_oracle(model, torch.float64, clip_zq(model), oracle_warm_zq(model), "stream")
    got = OrderedDict(st64)
    got[key] = next(s for new, s in shifted[::-1] if torch.equal(new.double(), st64[key]))
    assert not torch.equal(got[key], st64[key])
    bad, rows = check_states(got, st32, st64, 4.0, elu_keys(model))
    assert bad == key, (bad, [r for r in rows if r[0] == key])
    assert check_states(st64, st32, st64, 4.0, elu_keys(model))[0] is None


@pytest.mark.parametrize("model", sorted(MODELS))
def test_checker_accepts_the_fp32_oracle(model):
    y32, st32, y64, st64 = reference_run(model)
    ok, e, e32, bar = check_model(y32, y32, y64, 4.0)
    print(f"{model}: max |y| = {y64.abs().max().item():.3g}  e32 = {e32:.3g}")
    assert ok and e32 > 0
    assert set(st32) == set(st64)
    assert check_states(st32, st32, st64, 4.0, elu_keys(model))[0] is None


def _elu_kernel_model(seed):
    """act_elu's documented error as a model: fp64 exp of the fp32 input, times (1 + d) with |d| <= 2^-22, rounded to fp32, minus 1
    in fp32; fp32 and other dtypes keep F.elu"""
    real = F.elu
    gen = torch.Generator().manual_seed(seed)

    def elu(t, alpha=1.0, inplace=False):
        if t.dtype != torch.float64:
            return real(t, alpha, inplace)
        d = (torch.rand(t.shape, generator=gen, dtype=torch.float64) * 2 - 1) * 2.0 ** -22
        e = (torch.exp(t.float().double()) * (1 + d)).float()
        return torch.where(t > 0, t, (e - 1).double())
    return elu


@pytest.mark.parametrize("model", ["symAD", "symAAD", "c16"])
def test_checker_accepts_the_kernel_elu_model(model, monkeypatch):
    """The fp64 oracle with the kernels' ELU model passes check_model and check_states at factor 4, and uses at most half of the
    output bar: the documented ELU gap leaves room for the convs' own error."""
    y32, st32, y64, st64 = reference_run(model)
    monkeypatch.setattr(O.F, "elu", _elu_kernel_model(1))
    y, st = run_oracle(model, torch.float64, clip_zq(model), oracle_warm_zq(model), "stream")
    ok, e, e32, bar = check_model(y, y32, y64, 4.0)
    print(f"{model}: ELU model e = {e:.3g}  e32 = {e32:.3g}  ({e / e32:.2f} e32)")
    assert ok and e <= 2 * e32, (e, e32)
    bad, rows = check_states(st, st32, st64, 4.0, elu_keys(model))
    assert bad is None, [r for r in rows if r[0] == bad]
