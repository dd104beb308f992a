"""The vocoder's bf16 kernels layer by layer (compute_dtype 1: bf16 operands, fp32 storage; 2: bf16 operands and bf16 storage) against
an exact rounding model, through `adec_test_vocoder_layer`.

The contract the code implements, which `_model` restates:
  * conv / transposed-conv weights are rounded to bf16 (nearest-even) by the host packer; biases, the norm's mean / scale and the head's
    weights and bias stay fp32;
  * an operand is bf16_rne(fp32 pre_act(x)), x being fp32 (mode 1) or bf16 (mode 2); LeakyReLU is `x > 0 ? x : x * slope` and the
    norm `(x - mean) / scale`, both IEEE fp32; causal-state rows hold post-activation values, fp32 in mode 1 and bf16 in mode 2;
  * a conv output is sum(a * w) with fp32 accumulation, + bias, + residual, in fp32, stored once (fp32, or bf16_rne in mode 2);
  * the head's operand is lrelu(x), rounded to bf16 only in mode 2 (the value the bf16 state keeps); its output is
    tanhf(sum + bias), an fp32 FMA chain, stored as fp32 or bf16;
  * the new state is rows [T, T + P) of state || stored(act(x)), compared bit for bit.
Products of bf16 (or fp32) values are exact in fp64, so `exact` below is the fp64 sum of the exact products and only the fp32
accumulation order is unknown.  With S = sum |a w| + |bias| + |res| per output element, its error is below delta:
  * tensor-core convs, delta = 2^-16 S.  A group (one 32-channel piece x at most 2 taps: 64 products) accumulates in the tensor core
    in at most 64 steps; if each errs by at most a truncating fp32 add (< 2^-23 of the running sum), a group errs by < 2^-17 of its
    own sum |a w|, and those sums add up to at most S.  The groups (at most 48: 8 pieces x 6 groups at C = 256, K = 11), the bias and the
    residual then take at most 50 round-to-nearest fp32 adds, < 50 * 2^-24 S < 2^-18.3 S.  Together < 2^-16 S.  The per-step premise
    is the tensor core's behaviour, which NVIDIA does not document; the measured error (1.4e-7 S, about 2^-22.7) is far inside it.
  * head, delta = 2^-18 S + 2 fp32 ulps: per lane a 28-term fp32 FMA chain, then 3 shuffle adds and the bias add, < 32 * 2^-24 S =
    2^-19 S; tanhf adds at most 2 ulps (CUDA's stated bound) and tanh is 1-Lipschitz.
Mode 1 must land within delta (+ the fp32 rounding of the stored value); mode 2 between bf16_rne(exact - delta) and
bf16_rne(exact + delta), and at least 99 % of elements on bf16_rne(exact) itself.  That interval cannot tell how a store rounds a value
that lies exactly on a bf16 tie, so the tie cases below build data whose stored values are exact ties whatever the accumulation order,
and require nearest-even on every one.

The inputs include values and weights that sit exactly halfway between two bf16 values (round-half-even vs half-away), exact zeros and
negative values through LeakyReLU.  The negative controls (no GPU) feed the checker outputs of deliberately wrong models - round toward
zero, half away from zero, the residual added after rounding, a bf16 bias, bf16 head weights, a state window one row off - and
require each to be rejected on the same data the GPU cases use."""
import ctypes

import numpy as np
import pytest

ACT_NONE, ACT_LRELU, ACT_NORM = 0, 2, 3
SLOPE = 0.1          # HIFIGAN_V*_PARAMS negative_slope
HEAD_SLOPE = 0.01    # HiFiGAN.py output LeakyReLU

# name -> layer spec, with the shapes build_hifigan gives the ops of the v1 / v2 / v0 plans (synthetic.HIFIGAN_V*_PARAMS)
CASES = {
    "input_conv": dict(kind=0, Cin=64, Cout=512, K=7, dil=1, G=1, pre=ACT_NORM),
    "upsamples.0": dict(kind=1, Cin=512, Cout=256, up=5, pre=ACT_LRELU),
    "upsamples.3": dict(kind=1, Cin=64, Cout=32, up=3, pre=ACT_LRELU),                          # 96 outputs: one padded 128 tile
    "v1.blocks.0.convs1.0": dict(kind=0, Cin=768, Cout=768, K=11, dil=1, G=3, shared=True, pre=ACT_LRELU),   # NT 128
    "v1.blocks.1.convs1.1": dict(kind=0, Cin=384, Cout=384, K=11, dil=3, G=3, pre=ACT_LRELU),
    "v2.blocks.2.convs1.2": dict(kind=0, Cin=192, Cout=192, K=3, dil=5, G=3, pre=ACT_LRELU),                 # NT 64
    "v1.blocks.3.convs1.2": dict(kind=0, Cin=96, Cout=96, K=11, dil=5, G=3, pre=ACT_LRELU),                  # NT 32, P 50
    "v1.blocks.0.convs2.1": dict(kind=0, Cin=768, Cout=768, K=11, dil=1, G=3, pre=ACT_LRELU, res=True),
    "v2.blocks.3.convs2.0": dict(kind=0, Cin=96, Cout=96, K=3, dil=1, G=3, pre=ACT_LRELU, res=True),
    "blocks.0.conv_out": dict(kind=0, Cin=768, Cout=256, K=1, dil=1, G=1, pre=ACT_NONE),                     # 24 input pieces
    "blocks.3.conv_out": dict(kind=0, Cin=96, Cout=32, K=1, dil=1, G=1, pre=ACT_NONE),                       # 3 input pieces
    "output_conv": dict(kind=2, Cin=32, Cout=1, K=7, pre=ACT_LRELU),
}
# (B, consecutive chunk lengths): the state carries over; every sequence has a chunk shorter than P where P > 1 (P = 6 .. 50), and
# the small chunks at B > 1 take the stacked-row path
RUNS = [(1, (300, 1, 129)), (3, (128, 5, 127)), (16, (5, 1, 129))]


# ------------------------------------------------------------------------------------------------ rounding
def bf16_round(x, mode="rne"):
    """fp32 values -> the fp32 values of their bf16 rounding: 'rne' nearest-even (the kernels, the host packer, torch), 'rna' nearest
    with ties away from zero, 'rz' toward zero."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).copy()
    if mode == "rne":
        u += np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))
    elif mode == "rna":
        u += np.uint32(0x8000)
    return (u & np.uint32(0xFFFF0000)).view(np.float32)


def bf16_round64(x):
    """fp64 values -> bf16_rne of each, as fp64 (one rounding: no detour through fp32)."""
    u = np.ascontiguousarray(x, np.float64).view(np.uint64).copy()
    u += np.uint64((1 << 44) - 1) + ((u >> np.uint64(45)) & np.uint64(1))
    return (u & ~np.uint64((1 << 45) - 1)).view(np.float64)


def to_words(x):
    """bf16-representable fp32 values -> bf16 words."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    assert not (u & np.uint32(0xFFFF)).any()
    return (u >> np.uint32(16)).astype(np.uint16)


def from_words(w):
    return (w.astype(np.uint32) << np.uint32(16)).view(np.float32)


def ties(shape, rng):
    """fp32 values exactly halfway between two bf16 values, O(1), both signs, the lower neighbour even or odd at random."""
    u = bf16_round(rng.standard_normal(shape).astype(np.float32), "rz").view(np.uint32)
    return (u | np.uint32(0x8000)).view(np.float32)


# ------------------------------------------------------------------------------------------------ the model
def _act(x, pre, slope, mean=None, scale=None):
    """fp32 pre-activation as the kernels compute it."""
    if pre == ACT_LRELU:
        return np.where(x > 0, x, x * np.float32(slope)).astype(np.float32)
    if pre == ACT_NORM:
        return ((x - mean[None, :, None]) / scale[None, :, None]).astype(np.float32)
    return x


def _model(spec, mode, x, state, w, bias, res=None, mean=None, scale=None, offline=False, defect=None):
    """One layer.  x, state, res: the stored values (fp32 arrays, bf16-representable in mode 2).  Returns (exact, S, y, new_state):
    exact and S per output element (fp64), y what a kernel with `defect` (None = the contract) stores, new_state the state it leaves.
    defect: 'out_rz' / 'state_rz' outputs / new state rounded toward zero; 'out_rna' / 'state_rna' / 'act_rna' / 'w_rna' outputs /
    new state / activation operands / weights rounded half away from zero; 'res_after_round' the residual added to the rounded conv output; 'bias_bf16'; 'head_w_bf16'; 'state_shift'
    the state window one row early."""
    kind, pre = spec["kind"], spec["pre"]
    slope = HEAD_SLOPE if kind == 2 else SLOPE
    store = bf16_round if mode == 2 else (lambda v: v)
    store_st = (lambda v: bf16_round(v, defect[6:])) if defect in ("state_rz", "state_rna") else store
    B, _, T = x.shape
    ax = _act(x, pre, slope, mean, scale)
    if offline:
        state = ax[:, :, :1] if kind == 1 else np.zeros_like(state)        # ReplicationPad1d of the transposed convs / zero history
    xx = np.concatenate([state, store(ax)], -1)                            # x~ = history || chunk, post-activation, as stored
    P = state.shape[-1]
    sh = 1 if defect == "state_shift" else 0
    new_state = np.concatenate([state, store_st(ax)], -1)[:, :, T - sh:T - sh + P]
    if kind == 2:
        a = (bf16_round(xx) if mode == 2 else xx).astype(np.float64)      # head: stored4<BST>, fp32 otherwise
        wq = (bf16_round(w) if defect == "head_w_bf16" else w).astype(np.float64)
    else:
        a = bf16_round(xx, "rna" if defect == "act_rna" else "rne").astype(np.float64)
        wq = bf16_round(w, "rna" if defect == "w_rna" else "rne").astype(np.float64)
    bq = np.zeros(1, np.float64) if bias is None else (bf16_round(bias) if defect == "bias_bf16" else bias).astype(np.float64)
    if kind == 1:
        up = spec["up"]
        cols = np.concatenate([a[:, :, 1:], a[:, :, :-1]], 1).transpose(0, 2, 1).reshape(B * T, -1)    # (x[j], x[j-1])
        wr = np.concatenate([wq[:, :, :up], wq[:, :, up:]], 0)                                        # (2 Cin, Cout, up)
        wr = wr.transpose(0, 2, 1).reshape(wr.shape[0], -1)                                             # (2 Cin, up * Cout)
        s, sa = cols @ wr, np.abs(cols) @ np.abs(wr)
        Cout = spec["Cout"]
        fix = lambda v: v.reshape(B, T, up, Cout).transpose(0, 3, 1, 2).reshape(B, Cout, T * up)
        s, sa = fix(s), fix(sa)
        s, sa = s + bq[None, :, None], sa + np.abs(bq)[None, :, None]
    else:
        K, dil = w.shape[-1], spec.get("dil", 1)
        G = spec.get("G", 1)
        cin_g, cout_g = w.shape[1], w.shape[0] // G
        s, sa = [], []
        for g in range(G):
            ag = a if spec.get("shared") or G == 1 else a[:, g * cin_g:(g + 1) * cin_g]
            cols = np.stack([ag[:, :, k * dil:k * dil + T] for k in range(K)], -1).transpose(0, 2, 1, 3).reshape(B * T, -1)
            wg = wq[g * cout_g:(g + 1) * cout_g].reshape(cout_g, -1).T
            s.append((cols @ wg).reshape(B, T, cout_g))
            sa.append((np.abs(cols) @ np.abs(wg)).reshape(B, T, cout_g))
        s, sa = np.concatenate(s, -1).transpose(0, 2, 1), np.concatenate(sa, -1).transpose(0, 2, 1)
        s, sa = s + bq[None, :, None], sa + np.abs(bq)[None, :, None]
    r = 0.0 if res is None else res.astype(np.float64)
    exact, S = s + r, sa + np.abs(r)
    if kind == 2:
        exact = np.tanh(exact)
    if mode == 1:
        y = exact.astype(np.float32)
    elif defect in ("out_rz", "out_rna"):
        y = bf16_round(exact.astype(np.float32), defect[4:])
    elif defect == "res_after_round":
        y = bf16_round(bf16_round(s.astype(np.float32)) + res)
    else:
        y = bf16_round64(exact).astype(np.float32)
    if defect is not None and defect not in ("out_rz", "res_after_round"):
        # the defect moved the sums: the contract's exact / S stay those of the correct model
        exact, S = _model(spec, mode, x, state, w, bias, res, mean, scale, offline)[:2]
    return exact, S, y, new_state


def check(spec, mode, y, exact, S):
    """(ok, statistic): mode 1 the largest |y - exact| / S, mode 2 the fraction of elements equal to bf16_rne(exact)."""
    y = y.astype(np.float64)
    delta = (2.0 ** -18 * S + 2.0 ** -22 * np.abs(exact)) if spec["kind"] == 2 else 2.0 ** -16 * S
    if mode == 1:
        err = np.abs(y - exact)
        ok = bool(np.all(err <= delta + 2.0 ** -24 * np.abs(y)))
        return ok, float(np.max(err / np.maximum(S, 1e-30)))
    inside = (bf16_round64(exact - delta) <= y) & (y <= bf16_round64(exact + delta))
    frac = float(np.mean(y == bf16_round64(exact)))
    return bool(inside.all()) and frac >= 0.99, frac


# ------------------------------------------------------------------------------------------------ data
def make_layer(name, seed=0):
    """Weights (with bf16 ties), bias, norm statistics of one case."""
    spec = CASES[name]
    rng = np.random.default_rng(seed)
    kind, Cin, Cout = spec["kind"], spec["Cin"], spec["Cout"]
    if kind == 1:
        shape, fan = (Cin, Cout, 2 * spec["up"]), 2 * Cin
    else:
        G = spec.get("G", 1)
        shape, fan = (Cout, Cin // G, spec["K"]), Cin // G * spec["K"]
    w = rng.standard_normal(shape).astype(np.float32)
    t = rng.random(shape) < 0.25
    w[t] = ties(int(t.sum()), rng)
    w *= np.float32(2.0 ** -np.round(np.log2(np.sqrt(fan))))      # ~ 1 / sqrt(fan-in); a power of two keeps the ties
    bias = (0.5 * rng.standard_normal(Cout)).astype(np.float32)
    mean = (0.2 * rng.standard_normal(Cin)).astype(np.float32)
    scale = (1.0 + 0.5 * rng.random(Cin)).astype(np.float32)
    return spec, w, bias, mean, scale


def lrelu_ties(slope):
    """The bf16 values x whose fp32 x * slope lies exactly halfway between two bf16 values.  For the vocoder's slopes (0.1: 26 values,
    0.01: 5, both lower-neighbour parities) every such product is subnormal: no normal-range LeakyReLU output of a bf16 value is a tie."""
    x = from_words(np.arange(0x8000, 0xFF80, dtype=np.uint16))      # every finite negative bf16 value
    return x[((x * np.float32(slope)).view(np.uint32) & np.uint32(0xFFFF)) == 0x8000]


def make_input(spec, mode, B, T, rng, channels, slope=None):
    """O(1) values, negative ones, exact zeros and bf16 ties: halfway values themselves in fp32 storage, and with bf16 storage (which
    cannot hold them) the bf16 values whose LeakyReLU(slope) is one, so that the bf16 state and head operands round ties."""
    x = rng.standard_normal((B, channels, T)).astype(np.float32)
    t = rng.random(x.shape) < (0.25 if mode == 1 else 0.0625 if slope is not None else 0.0)
    x[t] = ties(int(t.sum()), rng) if mode == 1 else rng.choice(lrelu_ties(slope), int(t.sum()))
    x[rng.random(x.shape) < 0.0625] = 0.0
    return bf16_round(x) if mode == 2 else x


def in_channels(spec):
    return spec["Cin"] // spec["G"] if spec.get("shared") else spec["Cin"]


def history(spec):
    if spec["kind"] == 1:
        return 1
    return (spec["K"] - 1) * spec.get("dil", 1)


def out_shape(spec, B, T):
    if spec["kind"] == 1:
        return (B, spec["Cout"], T * spec["up"])
    return (B, spec["Cout"], T)


def sequence(name, mode, B, chunks, seed, offline=False):
    """Inputs of a run: [(x, res)] per chunk plus the initial state (post-activation values, as stored)."""
    spec = CASES[name]
    rng = np.random.default_rng(1000 * seed + 17 * B + mode)
    slope = (HEAD_SLOPE if spec["kind"] == 2 else SLOPE) if spec["pre"] == ACT_LRELU else None
    st = make_input(spec, mode, B, history(spec), rng, in_channels(spec), slope)
    if slope is not None:
        st = _act(st, ACT_LRELU, slope)
    st = bf16_round(st) if mode == 2 else st
    items = []
    for T in chunks:
        x = make_input(spec, mode, B, T, rng, in_channels(spec), slope)
        res = make_input(spec, mode, B, T, rng, spec["Cout"]) if spec.get("res") else None
        items.append((x, res))
    return st, items


# ------------------------------------------------------------------------------------------------ the library
def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def run_layer(lib, layer, mode, x, state, res, offline=False):
    """adec_test_vocoder_layer on cuda:0 for layer = (spec, w, bias, mean, scale); returns (y values, new state values) as fp32
    arrays."""
    from audiodec_b200 import _lib
    spec, w, bias, mean, scale = layer
    B, _, T = x.shape
    # copies: the library updates the state in place, and the caller's arrays stay the model's inputs
    enc = (lambda v: np.ascontiguousarray(to_words(v))) if mode == 2 else (lambda v: np.array(v, np.float32, order="C"))
    dec = from_words if mode == 2 else (lambda v: v)
    xs, rs, ss = enc(x), None if res is None else enc(res), enc(state)
    y = np.zeros(out_shape(spec, B, T), np.uint16 if mode == 2 else np.float32)
    rc = lib.adec_test_vocoder_layer(0, mode, spec["kind"], _p(xs), B, spec["Cin"], T, _p(w), _p(bias), spec["Cout"], spec.get("K", 0),
                                     spec.get("dil", 1), spec.get("up", 1), spec.get("G", 1), int(spec.get("shared", False)), spec["pre"],
                                     HEAD_SLOPE if spec["kind"] == 2 else SLOPE, _p(mean), _p(scale), _p(rs), int(offline), _p(ss), _p(y))
    assert rc == 0, _lib.last_error(None)
    return dec(y), dec(ss)


@pytest.fixture(scope="module")
def lib():
    from audiodec_b200 import _lib
    return _lib.load()


def _check_run(lib, name, mode, B, chunks, offline=False):
    layer = spec, w, bias, mean, scale = make_layer(name)
    st, items = sequence(name, mode, B, chunks, 0, offline)
    for T, (x, res) in zip(chunks, items):
        y, st_k = run_layer(lib, layer, mode, x, st, res, offline)
        exact, S, _, st_m = _model(spec, mode, x, st, w, bias, res, mean, scale, offline)
        ok, stat = check(spec, mode, y, exact, S)
        state_ok = offline or np.array_equal(st_k.view(np.uint32), st_m.view(np.uint32))
        what = "max |y - exact| / S" if mode == 1 else "fraction == bf16_rne(exact)"
        print(f"[bf16 layers] {name} mode {mode} B={B} T={T}{' offline' if offline else ''}: {what} "
              f"{stat:.3e}, state {'bit-equal' if state_ok and not offline else 'n/a' if offline else 'DIFFERS'}")
        assert ok, (name, mode, B, T, stat)
        assert state_ok, (name, mode, B, T, "state")
        if not offline:
            st = st_k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", sorted(CASES))
def test_layer_matches_rounding_model(lib, name, mode):
    """Each op of the v1 / v2 / v0 plans, B in {1, 3, 16}, three consecutive chunks of T in {1, 5, 127, 128, 129, 300}."""
    for B, chunks in RUNS:
        _check_run(lib, name, mode, B, chunks)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["upsamples.0", "upsamples.3"])
def test_transposed_conv_offline(lib, name, mode):
    """Generator.forward: the transposed convs replicate their first input row (hist_rep) instead of reading state."""
    for B, T in ((1, 300), (3, 5), (16, 129)):
        _check_run(lib, name, mode, B, (T,), offline=True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_stacked_rows_off(lib, monkeypatch, mode):
    """The stacked case again with one row space per stream (ADEC_STACK_ROWS=0, read when the handle is created)."""
    monkeypatch.setenv("ADEC_STACK_ROWS", "0")
    _check_run(lib, "v1.blocks.3.convs1.2", mode, 16, (5, 1, 129))


@pytest.mark.gpu
def test_rejects_fp32_grade_modes(lib):
    from audiodec_b200 import _lib
    x = np.zeros((1, 32, 4), np.float32)
    w = np.zeros((1, 32, 7), np.float32)
    st = np.zeros((1, 32, 6), np.float32)
    y = np.zeros((1, 1, 4), np.float32)
    for cd in (0, 3):
        assert lib.adec_test_vocoder_layer(0, cd, 2, _p(x), 1, 32, 4, _p(w), None, 1, 7, 1, 1, 1, 0, ACT_LRELU, 0.01, None, None, None, 0,
                                           _p(st), _p(y)) != 0
        assert "compute_dtype must be 1 or 2" in _lib.last_error(None)


# ------------------------------------------------------------------------------------------------ stored values on exact ties
TIE_CASES = ["blocks.3.conv_out", "input_conv", "output_conv"]


def tie_case(name, B=3, T=129, seed=11):
    """Mode-2 data whose stored values are exact bf16 ties whatever the accumulation order, with both lower-neighbour parities:
      blocks.3.conv_out  one-hot weights and bias 2^(e-8) per channel: every output is x + 2^(e-8) for a bf16 x of binade e, exact in
                         fp32 (the epilogue's st2);
      input_conv         mean = -2^(e-8), scale = 1: every normalised value x + 2^(e-8) (the state write-back's st4, the operands);
      output_conv        one weight 2^-14 (channel 0, current row) and bias 2^-22: s = x 2^-14 + 2^-22 with |s| < 2^-13, where
                         tanhf(s) = s (s^3 / 3 is below 1/16 of an fp32 ulp of s) (the head's st1).
    Returns (layer, state, x)."""
    spec = CASES[name]
    rng = np.random.default_rng(seed)
    _, w, bias, mean, scale = make_layer(name)
    cin, cout = spec["Cin"], spec["Cout"]

    def binade(shape, e, signed=True):      # bf16 values (1 + m / 128) 2^e, m >= 1: x +- 2^(e-8) stays inside the binade
        v = (1 + rng.integers(1, 128, shape) / 128.0) * 2.0 ** e
        return (v * rng.choice([-1.0, 1.0], shape) if signed else v).astype(np.float32)

    x = bf16_round(rng.standard_normal((B, cin, T)).astype(np.float32))
    st = bf16_round(rng.standard_normal((B, cin, history(spec))).astype(np.float32))
    if name == "blocks.3.conv_out":
        e = rng.integers(-3, 4, cout)
        w = np.zeros_like(w)
        w[np.arange(cout), np.arange(cout), 0] = 1.0
        bias = (2.0 ** (e - 8)).astype(np.float32)
        x[:, :cout] = binade((B, cout, T), e[None, :, None])
    elif name == "input_conv":
        e = rng.integers(-3, 4, cin)
        mean, scale = (-(2.0 ** (e - 8))).astype(np.float32), np.ones(cin, np.float32)
        x = binade((B, cin, T), e[None, :, None])
    else:
        w = np.zeros_like(w)
        w[0, 0, -1] = 2.0 ** -14
        bias = np.array([2.0 ** -22], np.float32)
        x[:, 0] = binade((B, T), 0, signed=False)
        st = bf16_round(_act(st, ACT_LRELU, HEAD_SLOPE))
    return (spec, w, bias, mean, scale), st, x


def tie_values(layer, x, exact):
    """The fp32 values the kernel rounds to bf16 in a tie case: the normalised chunk (input_conv: its state rows), else the outputs."""
    spec, _, _, mean, scale = layer
    return _act(x, ACT_NORM, 0.0, mean, scale) if spec["pre"] == ACT_NORM else exact.astype(np.float32)


def tie_stats(v):
    u = np.ascontiguousarray(v, np.float32).view(np.uint32)
    tie = (u & np.uint32(0xFFFF)) == 0x8000
    return float(tie.mean()), float(((u[tie] >> np.uint32(16)) & np.uint32(1)).mean())


def check_ties(layer, mode, x, st, y, new_state, defect=None):
    """(outputs ok, state ok) of a tie case against the contract: outputs stored as bf16_rne of their (exact) fp32 value, the
    state bit for bit."""
    spec, w, bias, mean, scale = layer
    exact, S, _, st_m = _model(spec, mode, x, st, w, bias, None, mean, scale)
    out_ok = check(spec, mode, y, exact, S)[0] if spec["pre"] == ACT_NORM else \
        bool(np.array_equal(y.view(np.uint32), bf16_round(exact.astype(np.float32)).view(np.uint32)))
    return out_ok, bool(np.array_equal(new_state.view(np.uint32), st_m.view(np.uint32)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", TIE_CASES)
def test_bf16_storage_rounds_ties_to_even(lib, name):
    """bf16 storage (st2 / st4 / st1) on values exactly halfway between two bf16 values: nearest-even, not half away from zero."""
    layer, st, x = tie_case(name)
    y, st_k = run_layer(lib, layer, 2, x, st, None)
    exact = _model(layer[0], 2, x, st, *layer[1:3], None, *layer[3:])[0]
    frac, odd = tie_stats(tie_values(layer, x, exact))
    out_ok, state_ok = check_ties(layer, 2, x, st, y, st_k)
    print(f"[bf16 ties] {name}: {frac:.3f} of the rounded values are ties ({odd:.2f} with an odd lower neighbour), outputs "
          f"{'ok' if out_ok else 'WRONG'}, state {'bit-equal' if state_ok else 'DIFFERS'}")
    assert frac > 0.99 and 0.3 < odd < 0.7
    assert out_ok and state_ok


# ------------------------------------------------------------------------------------------------ negative controls (no GPU)
def test_model_rounding_equals_torch_on_ties():
    import torch
    rng = np.random.default_rng(5)
    t = ties(4096, rng)
    lower_odd = (bf16_round(t, "rz").view(np.uint32) >> np.uint32(16)) & np.uint32(1)
    assert 0 < lower_odd.mean() < 1          # both even and odd lower neighbours
    ref = torch.from_numpy(t).to(torch.bfloat16).float().numpy()
    np.testing.assert_array_equal(bf16_round(t).view(np.uint32), ref.view(np.uint32))
    np.testing.assert_array_equal(bf16_round64(t.astype(np.float64)).astype(np.float32).view(np.uint32), ref.view(np.uint32))
    assert not np.array_equal(bf16_round(t, "rna"), ref) and not np.array_equal(bf16_round(t, "rz"), ref)
    x = rng.standard_normal(4096).astype(np.float32)
    np.testing.assert_array_equal(bf16_round(x).view(np.uint32), torch.from_numpy(x).to(torch.bfloat16).float().numpy().view(np.uint32))


def _control(name, mode, defect, B=3, chunks=(128, 5), offline=False):
    """Outputs / state of the model with `defect` on the GPU cases' data: does the checker reject them?  Also checks that the defect-free
    model's own outputs pass (the bounds are not vacuous the other way either)."""
    spec, w, bias, mean, scale = make_layer(name)
    st, items = sequence(name, mode, B, chunks, 0, offline)
    out_rejected = state_rejected = False
    for x, res in items:
        exact, S, y, st_m = _model(spec, mode, x, st, w, bias, res, mean, scale, offline)
        assert check(spec, mode, y, exact, S)[0]
        _, _, y_bad, st_bad = _model(spec, mode, x, st, w, bias, res, mean, scale, offline, defect=defect)
        out_rejected |= not check(spec, mode, y_bad, exact, S)[0]
        state_rejected |= not np.array_equal(st_bad.view(np.uint32), st_m.view(np.uint32))
        st = st_m
    return out_rejected, state_rejected


@pytest.mark.parametrize("name,mode,defect", [
    ("v1.blocks.3.convs1.2", 2, "out_rz"),
    ("v2.blocks.3.convs2.0", 2, "out_rz"),
    ("output_conv", 2, "out_rz"),
    ("blocks.3.conv_out", 1, "act_rna"),
    ("v2.blocks.2.convs1.2", 1, "act_rna"),
    ("upsamples.3", 1, "act_rna"),
    ("blocks.3.conv_out", 1, "w_rna"),
    ("blocks.3.conv_out", 2, "w_rna"),
    ("upsamples.3", 2, "w_rna"),
    ("v2.blocks.3.convs2.0", 2, "res_after_round"),
    ("v1.blocks.0.convs2.1", 2, "res_after_round"),
    ("input_conv", 1, "bias_bf16"),
    ("blocks.3.conv_out", 2, "bias_bf16"),
    ("upsamples.3", 2, "bias_bf16"),
    ("output_conv", 1, "head_w_bf16"),
    ("output_conv", 2, "head_w_bf16"),
])
def test_checker_rejects_wrong_outputs(name, mode, defect):
    out_rejected, _ = _control(name, mode, defect)
    assert out_rejected, f"{defect} on {name} mode {mode} passes the output check"


@pytest.mark.parametrize("name,mode,defect", [
    ("v1.blocks.3.convs1.2", 1, "state_shift"),
    ("input_conv", 2, "state_shift"),
    ("output_conv", 2, "state_shift"),
    ("v1.blocks.3.convs1.2", 2, "state_rz"),
    ("upsamples.3", 2, "state_rz"),
    ("output_conv", 2, "state_rz"),
    ("v1.blocks.3.convs1.2", 2, "state_rna"),      # the subnormal LeakyReLU ties
    ("upsamples.3", 2, "state_rna"),
    ("output_conv", 2, "state_rna"),
])
def test_checker_rejects_wrong_state(name, mode, defect):
    _, state_rejected = _control(name, mode, defect)
    assert state_rejected, f"{defect} on {name} mode {mode} passes the state comparison"


@pytest.mark.parametrize("name,defect", [
    ("blocks.3.conv_out", "out_rna"), ("output_conv", "out_rna"), ("blocks.3.conv_out", "out_rz"), ("input_conv", "state_rna"),
])
def test_tie_checks_reject_half_away(name, defect):
    """The tie cases see a store that rounds half away from zero (or toward zero), and the contract's own outputs pass them."""
    layer, st, x = tie_case(name)
    spec, w, bias, mean, scale = layer
    exact, _, y, new_state = _model(spec, 2, x, st, w, bias, None, mean, scale)
    if spec["kind"] == 2:
        y = bf16_round(exact.astype(np.float32))        # tanhf(s) = s, rounded once: the fp64 tanh(s) lies just below the tie
    assert check_ties(layer, 2, x, st, y, new_state) == (True, True)
    _, _, y_bad, st_bad = _model(spec, 2, x, st, w, bias, None, mean, scale, defect=defect)
    assert check_ties(layer, 2, x, st, y_bad, st_bad) != (True, True)
