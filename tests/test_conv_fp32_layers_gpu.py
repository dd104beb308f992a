"""The fp32-grade conv engines (fp16-split wgmma, 3xTF32 wgmma, FFMA) op by op against fp64, in every row space.

Each case is one op shape of the released fp32 plans (symAD / symAAD / c16 encoder and decoder, HiFi-GAN v0 / v1 / v2 in fp32 mode),
built by the model builders and run through the codec call path by `adec_test_conv_op`.  Per op the error is

    e = max |y - exact| / S,   S = sum |a w| + |bias| + |res|   (the fused residual unit: recursed through its intermediate)

with `exact` computed in fp64 from the same fp32 inputs.  The yardstick is the reference's own fp32 path (torch conv1d / F.elu in fp32
on the CPU), scored the same way (e_ref): e <= BAR_FACTOR * max(e_ref, 2^-23).  The data are chosen where kernels go wrong: exact
zeros, negatives through ELU and LeakyReLU, channels scaled from 2^-20 to 2^10, small ELU inputs in [-1e-2, -1e-5], values near
2^-14 and 2^-24 and up to just under 6e4, weights spread over 2^24, and one all-zero-weight op.  Every op also runs on a second
weight set, the channel ladder (apply_ladder): output columns from 2^0 down to 2^-100 and one zero column, which one fp16 weight
scale per op cannot hold.  The ELU's known gap (accurate to 2.4e-7 absolute, not relative) is pinned by a strict xfail of its own;
the other ELU ops and states are held to that contract.  So is the fp16-split engine's activation envelope: receptive fields below
fp16's normal range (test_activation_envelope).

Every utterance must give the same output and state bits in every row space: uniform B = 1 (unstacked: the paired kernel for RU(32)),
stacked streams, varlen, and stream slots (two calls, so the slots' ping-pong bits flip; streams a call does not advance keep their
state bits).  The CPU tests at the end run the same checker on wrong arithmetic and wrong row maps, which it must reject."""
import ctypes
import os
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

BAR_FACTOR = 4.0
BAR_FLOOR = 2.0 ** -23
ELU_ABS = 2.4e-7      # act_elu (csrc/kernels.cuh): ex2.approx(x log2 e) - 1, within 2.4e-7 ABSOLUTE of expm1
ACT_NONE, ACT_ELU, ACT_LRELU, ACT_NORM = 0, 1, 2, 3
PREC_TF32, PREC_F16 = 2, 3
CONV, RU, CONVTR, STEM, HEAD = 0, 1, 2, 3, 4


def _case(name, kind, cin=32, cout=32, k=1, s=1, d=1, g=1, shared=0, pre=ACT_NONE, slope=0.0, nct=0, tanh=0, bias=True,
          res=False, zero_w=False):
    if kind == RU:      # residual_unit.py: ELU before the dilated conv and on the intermediate
        pre = ACT_ELU
    return dict(name=name, kind=kind, Cin=cin, Cout=cout, K=k, stride=s, dil=d, groups=g, shared_in=shared, pre_act=pre, slope=slope,
                out_nct=nct, post_tanh=tanh, bias=bias, res=res, zero_w=zero_w)


# Every distinct op shape of the fp32 plans (adec.cu build_symad / build_hifigan; the params of audiodec_b200/synthetic.py)
CASES = [
    # symAD / symAAD / c16 encoder
    _case("enc.stem", STEM, 1, 32, 7),
    _case("enc.ru32.d1", RU, 32, 32, 7, d=1, bias=False),
    _case("enc.ru32.d9", RU, 32, 32, 7, d=9, bias=False),
    _case("enc.ru64.d3", RU, 64, 64, 7, d=3, bias=False),
    _case("enc.ru128.d9", RU, 128, 128, 7, d=9, bias=False),
    _case("enc.ru256.d1(split)", RU, 256, 256, 7, d=1, bias=False),
    _case("enc.down.s2", CONV, 32, 64, 4, s=2),
    _case("enc.down.s3", CONV, 32, 64, 6, s=3),
    _case("enc.down.s4", CONV, 64, 128, 8, s=4),
    _case("enc.down.s5", CONV, 128, 256, 10, s=5),
    _case("enc.down.s8", CONV, 256, 512, 16, s=8),
    _case("projector", CONV, 512, 64, 3, nct=1, bias=False),
    _case("projector.symAAD", CONV, 512, 64, 3, nct=1, pre=ACT_ELU, bias=False),
    # decoder
    _case("decoder.conv1", CONV, 64, 512, 7),
    _case("dec.up.s5", CONVTR, 512, 256, s=5),
    _case("dec.up.s3.symAAD", CONVTR, 64, 32, s=3, pre=ACT_ELU),
    _case("dec.up.s8.c16", CONVTR, 512, 256, s=8),
    _case("dec.ru32.d3", RU, 32, 32, 7, d=3, bias=False),
    _case("decoder.conv2", HEAD, 32, 1, 7),
    _case("decoder.conv2.symAAD", HEAD, 32, 1, 7, pre=ACT_ELU, tanh=1),
    # HiFi-GAN v0 / v1 / v2, fp32 mode
    _case("input_conv.norm", CONV, 64, 512, 7, pre=ACT_NORM),
    _case("upsamples.0", CONVTR, 512, 256, s=5, pre=ACT_LRELU, slope=0.1),
    _case("upsamples.3(96 cols)", CONVTR, 64, 32, s=3, pre=ACT_LRELU, slope=0.1),
    _case("convs1.0.v1.nt128", CONV, 128 * 3, 128 * 3, 11, d=1, g=3, shared=1, pre=ACT_LRELU, slope=0.1),
    _case("convs1.1.v1.nt64", CONV, 64 * 3, 64 * 3, 11, d=3, g=3, pre=ACT_LRELU, slope=0.1),
    _case("convs2.v1.nt32", CONV, 32 * 3, 32 * 3, 11, g=3, pre=ACT_LRELU, slope=0.1, res=True),
    _case("convs2.v2.nt64", CONV, 64 * 3, 64 * 3, 3, g=3, pre=ACT_LRELU, slope=0.1, res=True),
    _case("convs1.2.v2.nt32", CONV, 32 * 3, 32 * 3, 3, d=5, g=3, pre=ACT_LRELU, slope=0.1),
    _case("conv_out", CONV, 64 * 3, 64, 1),
    _case("conv_out.zero_w", CONV, 32 * 3, 32, 1, zero_w=True),
    _case("output_conv", HEAD, 32, 1, 7, pre=ACT_LRELU, slope=0.01, tanh=1),
]


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _hist(c):
    """history rows P of the op"""
    if c["kind"] in (STEM, HEAD):
        return 6
    if c["kind"] == CONVTR:
        return 1
    return (c["K"] - 1) * c["dil"]


def _cin_x(c):
    return 1 if c["kind"] == STEM else c["Cin"] // c["groups"] if c["shared_in"] else c["Cin"]


def _cout(c):
    return 1 if c["kind"] == HEAD else c["Cout"]


def _outlen(c, L):
    if c["kind"] == CONVTR:
        return L * c["stride"]
    return (L - 1) // c["stride"] + 1 if c["kind"] == CONV else L


# ------------------------------------------------------------------------------------------------------------------------------
# data
# ------------------------------------------------------------------------------------------------------------------------------
def gen_x(rng, C, L, regime, big=5.9e4):
    """regime 0: O(1) with exact zeros; 1: channels scaled 2^-20..2^10; 2: small ELU inputs in [-1e-2, -1e-5] (a fifth positive);
    3: O(1) rows with values near 2^-14 and 2^-24 mixed in; 4: up to just under `big`"""
    if regime == 0:
        x = rng.standard_normal((C, L))
        x[rng.random((C, L)) < 0.15] = 0.0
    elif regime == 1:
        x = rng.standard_normal((C, L)) * 2.0 ** rng.integers(-20, 11, size=(C, 1))
    elif regime == 2:
        x = -(10.0 ** rng.uniform(-5, -2, (C, L)))
        x[rng.random((C, L)) < 0.2] *= -1
    elif regime == 3:
        x = rng.standard_normal((C, L))
        m = rng.random((C, L))
        x[m < 0.3] = 2.0 ** -14 * (1 + rng.random(int((m < 0.3).sum())))
        x[(m >= 0.3) & (m < 0.5)] = -(2.0 ** -24) * rng.integers(1, 8, int(((m >= 0.3) & (m < 0.5)).sum()))
    else:
        x = rng.uniform(-1, 1, (C, L)) * big
    return x.astype(np.float32)


LADDER_K = [0, 100, 60] + list(range(1, 31))    # 2^-k per output column, cycled; column LADDER_ZERO is all zero
LADDER_ZERO = 5
GROUP_LOW = 2.0 ** -20                          # grouped ops: all of group 1 at this scale


def ladder(n, shift=0):
    """per-column factors 2^-k, k cycling through LADDER_K from position `shift`, and one zero column"""
    f = np.array([2.0 ** -LADDER_K[(i + shift) % len(LADDER_K)] for i in range(n)])
    if n > LADDER_ZERO:
        f[LADDER_ZERO] = 0.0
    return f


def apply_ladder(c, W):
    """The channel ladder: every output column of the op scaled by its own 2^-k (kept within each column: the per-element 2^24
    spread), as a weight-normed layer with small gains g_co has.  Bias, residual and (residual unit) skip channels follow their
    column's factor, so that neither |bias| nor |res| dominates S.  Transposed convs: the ladder runs over the s * Cout effective
    columns (channel co at phase r: column r * Cout + co); the bias of co takes its smallest phase factor.  Grouped ops: group 1 at
    2^-20.  The fused unit: w and w2 take ladders of their own.  Returns W with "xs" / "rs", the per-channel factors of the input
    (the skip) and of the residual, or None."""
    k = c["kind"]
    W = dict(W)
    w, b = W["w"].astype(np.float64), None if W["b"] is None else W["b"].astype(np.float64)
    W["xs"] = W["rs"] = None
    if k == CONVTR:
        cin, cout, K = w.shape
        s = K // 2
        f = ladder(s * cout).reshape(s, cout)                    # [r, co]
        w = w * np.concatenate([f.T, f.T], 1)[None]               # taps r and s + r of (co, r)
        if b is not None:
            b = b * f.min(0)
    else:
        f = ladder(w.shape[0])
        if c["groups"] > 1:
            cg = w.shape[0] // c["groups"]
            f[cg:2 * cg] = GROUP_LOW
        w = w * f[:, None, None]
        if b is not None:
            b = b * f
        if c["res"]:
            W["rs"] = f
    if k == RU:
        f2 = ladder(c["Cout"], shift=11)
        W["w2"] = (W["w2"].astype(np.float64) * f2[:, None, None]).astype(np.float32)
        W["xs"] = f2
    W["w"] = w.astype(np.float32)
    W["b"] = None if b is None else b.astype(np.float32)
    return W


def gen_weights(rng, c):
    """weights spread over 2^24 in magnitude within every op; None for the w2 of non-RU ops"""
    k = c["kind"]
    if k == STEM:
        shape, fan = (32, 1, 7), 7
    elif k == HEAD:
        shape, fan = (1, 32, 7), 224
    elif k == CONVTR:
        shape, fan = (c["Cin"], c["Cout"], 2 * c["stride"]), 2 * c["Cin"]
    else:
        shape, fan = (c["Cout"], c["Cin"] // c["groups"], c["K"]), c["Cin"] // c["groups"] * c["K"]
    w = rng.standard_normal(shape) / np.sqrt(fan) * 2.0 ** rng.uniform(-12, 12, shape) / 2.0 ** 6
    if c["zero_w"]:
        w[:] = 0
    w2 = None
    if k == RU:
        w2 = (rng.standard_normal((c["Cout"], c["Cout"], 1)) / np.sqrt(c["Cout"]) * 2.0 ** rng.uniform(-12, 12, (c["Cout"], c["Cout"], 1))
              / 2.0 ** 6).astype(np.float32)
    nb = 32 if k == STEM else 1 if k == HEAD else c["Cout"]
    b = (rng.standard_normal(nb) * 0.5).astype(np.float32) if c["bias"] else None
    mean = scale = None
    if c["pre_act"] == ACT_NORM:
        mean = (rng.standard_normal(c["Cin"]) * 0.2).astype(np.float32)
        scale = (1.0 + 0.5 * rng.random(c["Cin"])).astype(np.float32)
    return dict(w=w.astype(np.float32), w2=w2, b=b, mean=mean, scale=scale)


# ------------------------------------------------------------------------------------------------------------------------------
# references: fp64 exact with its S, and the same ops in torch fp32 (the yardstick)
# ------------------------------------------------------------------------------------------------------------------------------
def act(c, x, W, dt):
    """pre-activation of x (fp32 data) in dtype dt (torch)"""
    t = torch.from_numpy(x).to(dt)
    p = c["pre_act"]
    if p == ACT_ELU:
        return torch.where(t > 0, t, torch.expm1(t)) if dt == torch.float64 else F.elu(t)
    if p == ACT_LRELU:
        return F.leaky_relu(t, float(np.float32(c["slope"])))
    if p == ACT_NORM:
        return (t - torch.from_numpy(W["mean"]).to(dt)[:, None]) / torch.from_numpy(W["scale"]).to(dt)[:, None]
    return t


def reference(c, W, x, hist, dt, res=None, elu_fn=None, offline=False):
    """one utterance: x (Cin_x, L) fp32, hist (Cin_x, P) fp32 already activated (the state), or None for offline (zero history,
    first-row replication in a transposed conv).  Returns (y, S); S is None in fp32 runs.  elu_fn overrides the ELU (negative
    controls)."""
    tt = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dt)
    k, P = c["kind"], _hist(c)
    ex = dt == torch.float64
    a = act(c, x, W, dt) if elu_fn is None or c["pre_act"] != ACT_ELU else elu_fn(tt(x))
    w, b = tt(W["w"]), tt(W["b"])
    if hist is None:
        h = a[:, :1].expand(-1, P) if k == CONVTR else torch.zeros(a.shape[0], P, dtype=dt)
    else:
        h = tt(hist)
    xx = torch.cat([h, a], 1)
    ab = (lambda v: v.abs()) if ex else (lambda v: v)
    if k == CONVTR:
        s = c["stride"]
        prev = xx[:, :-1]
        cur = xx[:, 1:]
        def tr(u, v, wt):
            y = torch.einsum("ct,cor->otr", u, wt[:, :, :s]) + torch.einsum("ct,cor->otr", v, wt[:, :, s:])
            return y.reshape(wt.shape[1], -1)
        y = tr(cur, prev, w) + (b[:, None] if b is not None else 0)
        S = tr(cur.abs(), prev.abs(), w.abs()) + (b.abs()[:, None] if b is not None else 0) if ex else None
        return y, S
    if c["shared_in"]:
        xx = xx.repeat(c["groups"], 1)
    conv = lambda u, wt, bb: F.conv1d(u[None], wt, bb, stride=c["stride"] if k == CONV else 1, dilation=c["dil"],
                                      groups=c["groups"] if k == CONV else 1)[0]
    if k == RU:
        mid = conv(xx, w, None)
        am = torch.where(mid > 0, mid, torch.expm1(mid)) if ex else (F.elu(mid) if elu_fn is None else elu_fn(mid))
        y = tt(x) + conv(am, tt(W["w2"]), None)
        if not ex:
            return y, None
        smid = conv(xx.abs(), w.abs(), None)
        S = tt(x).abs() + conv(am.abs(), tt(W["w2"]).abs(), None) + conv(smid, tt(W["w2"]).abs(), None)
        return y, S
    y = conv(xx, w, b)
    if res is not None:
        y = y + tt(res)
    S = None
    if ex:
        S = conv(xx.abs(), w.abs(), None if b is None else b.abs())
        if res is not None:
            S = S + tt(res).abs()
    if k == HEAD and c["post_tanh"]:
        y = torch.tanh(y)
    return y, S


def err(y, exact, S, slack=0.0):
    """max (|y - exact| - slack) / S over the elements with S > 0; elements with S == 0 must be within slack (inf otherwise)"""
    y = np.asarray(y, np.float64)
    exact = np.asarray(exact, np.float64)
    S = np.asarray(S, np.float64)
    d = np.maximum(np.abs(y - exact) - slack, 0.0)
    if not np.all(np.isfinite(y)):
        return np.inf
    if np.any(d[S == 0] > 0):
        return np.inf
    m = S > 0
    return float((d[m] / S[m]).max()) if m.any() else 0.0


def bar(e_ref, engine="f16", n_terms=1):
    """the tensor-core engines: BAR_FACTOR * max(e_ref, 2^-23).  The FFMA engine (ADEC_CONV_PATH=ffma) sums each output as one serial
    fp32 FMA chain over its n_terms products, which torch's blocked sums beat by up to 8.5x on the long-K ops (DESIGN section 3); it is
    held to that chain's worst-case bound n_terms * 2^-24 where that is looser."""
    b = BAR_FACTOR * max(e_ref, BAR_FLOOR)
    return max(b, n_terms * 2.0 ** -24) if engine == "ffma" else b


def elu_slack(c, W, x, hist):
    """What act_elu's documented 2.4e-7 ABSOLUTE error (ELU_ABS) can add to each output: ELU_ABS on every activated chunk value
    (state rows are read as stored), propagated through |w| (the fused unit: through its intermediate, whose own ELU adds ELU_ABS)."""
    if c["pre_act"] != ACT_ELU:
        return 0.0
    k, P, d = c["kind"], _hist(c), torch.float64
    e = torch.full(x.shape, ELU_ABS, dtype=d)
    if hist is None and k == CONVTR:
        h = e[:, :1].expand(-1, P)
    else:
        h = torch.zeros(x.shape[0], P, dtype=d)
    ee = torch.cat([h, e], 1)
    w = torch.from_numpy(W["w"]).to(d).abs()
    if k == CONVTR:
        s = c["stride"]
        t = torch.einsum("ct,cor->otr", ee[:, 1:], w[:, :, :s]) + torch.einsum("ct,cor->otr", ee[:, :-1], w[:, :, s:])
        return t.reshape(w.shape[1], -1).numpy()
    conv = lambda u, wt: F.conv1d(u[None], wt, None, stride=c["stride"] if k == CONV else 1, dilation=c["dil"],
                                  groups=c["groups"] if k == CONV else 1)[0]
    if k == RU:
        return conv(conv(ee, w) + ELU_ABS, torch.from_numpy(W["w2"]).to(d).abs()).numpy()
    return conv(ee, w).numpy()


def _terms(c):
    """products per output of the op's longest sum"""
    k = c["kind"]
    return {STEM: 7, HEAD: 224, CONVTR: 2 * c["Cin"], RU: c["Cin"] * c["K"]}.get(k, c["Cin"] // c["groups"] * c["K"])


def expected_state(c, W, hist, x):
    """rows [L, L + P) of state || act(x), in fp32 (bit for bit for every activation but ELU)"""
    a = act(c, x, W, torch.float32).numpy()
    xx = np.concatenate([hist, a], 1)
    return xx[:, xx.shape[1] - _hist(c):]


# ------------------------------------------------------------------------------------------------------------------------------
# the GPU entry point
# ------------------------------------------------------------------------------------------------------------------------------
def run_op(c, W, mode, lengths, xs, B, n_streams=None, streams=None, states=None, res=None, max_launch=64, flag_out=None):
    """lengths (n_calls, B); xs: list over calls of lists over utterances of (Cin_x, L); states (n_streams, Cin_x, P) or None.
    Returns (ys per call per utterance, states, launch records).  Checks the range flag of every run against its documented
    contract: on f16, a tensor-core launch whose output reaches |y| >= 6e4 (inf included) sets it, reported once; the stem and head
    kernels, tf32 and FFMA never set it.  flag_out: a list that receives the two flag reads."""
    from audiodec_b200 import _lib
    lib = _lib.load()
    lengths = np.ascontiguousarray(lengths, np.int32)
    n_calls = lengths.shape[0]
    d = _lib.AdecTestOp(kind=c["kind"], Cin=c["Cin"], Cout=c["Cout"], K=c["K"], stride=c["stride"], dil=c["dil"], groups=c["groups"],
                        shared_in=c["shared_in"], pre_act=c["pre_act"], slope=c["slope"], out_nct=c["out_nct"], post_tanh=c["post_tanh"],
                        w=_p(W["w"]), w2=_p(W["w2"]), bias=_p(W["b"]), mean=_p(W["mean"]), scale=_p(W["scale"]))
    x = np.ascontiguousarray(np.concatenate([u.ravel() for call in xs for u in call]).astype(np.float32))
    cout = _cout(c)
    outl = [[_outlen(c, int(L)) for L in row] for row in lengths]
    y = np.zeros(sum(cout * o for row in outl for o in row), np.float32)
    r = None if res is None else np.ascontiguousarray(np.concatenate([u.ravel() for call in res for u in call]).astype(np.float32))
    st = None if states is None else np.ascontiguousarray(states, np.float32)
    launched = np.zeros(max_launch * _lib.TEST_REC, np.int32)
    ptr = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    sl = None if streams is None else np.ascontiguousarray(streams, np.int32)
    flag = np.full(2, -1, np.int32)
    rc = lib.adec_test_conv_op(0, ctypes.byref(d), mode, n_calls, B, n_streams or B, ptr(lengths), None if sl is None else ptr(sl),
                               _p(x), _p(r), _p(st), _p(y), ptr(launched), max_launch, ptr(flag))
    assert rc == 0, _lib.last_error(None)
    f16_tc = os.environ.get("ADEC_CONV_PATH", "f16") == "f16" and c["kind"] in (CONV, RU, CONVTR)
    want = f16_tc and not np.abs(y).max() < 6e4
    split = c["kind"] == RU and c["Cout"] > 128       # its first launch's output (the intermediate) is checked as well
    assert flag[1] == 0 and (flag[0] == want or (split and f16_tc and flag[0] == 1)), \
        f"{c['name']}: range flag {tuple(flag)} with max |y| = {np.abs(y).max():.6g}"
    if flag_out is not None:
        flag_out.extend(int(v) for v in flag)
    ys, at = [], 0
    for row in outl:
        ys.append([])
        for o in row:
            ys[-1].append(y[at:at + cout * o].reshape(cout, o))
            at += cout * o
    recs = [tuple(v) for v in launched.reshape(-1, _lib.TEST_REC) if v[0] >= 0]
    return ys, st, recs


# ------------------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------------------
LAUNCHED = set()
REPORT = []


def _lengths(c):
    s = c["stride"] if c["kind"] == CONV else 1
    P = _hist(c)
    ls = [1, 2, s - 1, s, s + 1, max(1, P // 2), 127, 128, 129, 252, 256, 3 * 128 + 5]
    macs = c["Cin"] * c["Cout"] * 2 * c["stride"] if c["kind"] == CONVTR else c["Cin"] // c["groups"] * c["K"] * c["Cout"] // c["stride"]
    wide = macs > 1 << 20
    if wide:        # keeps the fp64 reference of the widest ops to about a second
        ls = [1, 2, s - 1, s, s + 1, max(1, P // 2), 128, 129, 256]
    out = []
    for L in ls:
        if L >= 1 and L not in out:
            out.append(L)
    return out


def _check(tag, c, W, y, xs, hist, res=None, slack=True):
    """(e of the kernel's y, e_ref); slack: allow ELU ops act_elu's documented absolute error (elu_slack)"""
    ex, S = reference(c, W, xs, hist, torch.float64, res=res, offline=hist is None)
    y32, _ = reference(c, W, xs, hist, torch.float32, res=res, offline=hist is None)
    sl = elu_slack(c, W, xs, hist) if slack else 0.0
    return err(y, ex.numpy(), S.numpy(), sl), err(y32.numpy(), ex.numpy(), S.numpy())


# (case, weight set): "spread" (gen_weights) under the case's name, "ladder" (apply_ladder) under name-ladder
CASE_WEIGHTS = ([pytest.param(c, "spread", id=c["name"]) for c in CASES] +
                [pytest.param(c, "ladder", id=c["name"] + "-ladder") for c in CASES])


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["f16", "tf32", "ffma"])
@pytest.mark.parametrize("case,weights", CASE_WEIGHTS)
def test_op_all_row_spaces(case, engine, weights, monkeypatch):
    """weights: "spread" (gen_weights) or "ladder" (apply_ladder: output columns from 2^0 down to 2^-100 and 0)"""
    c = case
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    rng = np.random.default_rng(zlib.crc32(c["name"].encode()))
    W = gen_weights(rng, c)
    if weights == "ladder":
        W = apply_ladder(c, W)
    cin, P, cout = _cin_x(c), _hist(c), _cout(c)
    big = 1e3 if c["kind"] == RU else 5.9e4

    def scaled(f):
        return lambda C, L, r: gen_x(rng, C, L, r % 5, big) if f is None else (gen_x(rng, C, L, r % 5, big) * f[:, None]).astype(np.float32)
    gx, gr = scaled(W.get("xs")), scaled(W.get("rs"))     # input channels (the skip), residual channels
    lens = _lengths(c)
    n = len(lens)
    xs = [gx(cin, L, i % 5) for i, L in enumerate(lens)]
    sts = np.stack([gx(cin, P, i + 2) for i in range(n)] + [gx(cin, P, 0) for _ in range(2)])
    if c["pre_act"] == ACT_ELU:       # a state holds activated values
        sts = np.maximum(sts, -1.0).astype(np.float32)
    res = [gr(cout, _outlen(c, L), 0) for L in lens] if c["res"] else None
    e_max = eref_max = 0.0

    def score(tag, y, x, hist, r=None):
        nonlocal e_max, eref_max
        e, eref = _check(tag, c, W, y, x, hist, r)
        e_max, eref_max = max(e_max, e), max(eref_max, eref)
        b = bar(eref, engine, _terms(c))
        assert e <= b, f"{c['name']} {engine} {weights} {tag}: e = {e:.3g} > bar(e_ref = {eref:.3g}) = {b:.3g}"

    def check_state(tag, got, hist, x):
        want = expected_state(c, W, hist, x)
        if c["pre_act"] == ACT_ELU:
            a64 = act(c, x, W, torch.float64).numpy()
            ex = np.concatenate([hist, a64], 1)[:, -P:]
            eref = err(want, ex, np.abs(ex))
            d = np.abs(got.astype(np.float64) - ex)
            assert np.all(d <= ELU_ABS + bar(eref) * np.abs(ex)), \
                f"{c['name']} {engine} {weights} {tag}: ELU state off by {d.max():.3g} (e_ref = {eref:.3g})"
        else:
            np.testing.assert_array_equal(got, want, err_msg=f"{c['name']} {engine} {weights} {tag}: state")

    # ---- uniform B = 1 per utterance, unstacked (RU(32): the paired kernel), two consecutive chunks; history from its state
    monkeypatch.setenv("ADEC_STACK_ROWS", "0")
    xs2 = [gx(cin, L, i + 3) for i, L in enumerate(lens)]
    res2 = [gr(cout, _outlen(c, L), 0) for L in lens] if c["res"] else None
    uni_y, uni_st1, uni_st2 = [], [], []
    for i, L in enumerate(lens):
        r1 = None if res is None else [[res[i]]]
        ys, st1, recs = run_op(c, W, 0, [[L]], [[xs[i]]], 1, states=sts[i:i + 1].copy(), res=r1)
        LAUNCHED.update((engine,) + r for r in recs)
        score(f"uniform L={L}", ys[0][0], xs[i], sts[i], None if res is None else res[i])
        if P:
            check_state(f"uniform L={L}", st1[0], sts[i], xs[i])
        ys2, st2, _ = run_op(c, W, 0, [[L], [L]], [[xs[i]], [xs2[i]]], 1, states=sts[i:i + 1].copy(),
                             res=None if res is None else [[res[i]], [res2[i]]])
        np.testing.assert_array_equal(ys2[0][0], ys[0][0], err_msg=f"{c['name']} {engine}: uniform call 1, L={L}")
        score(f"uniform call 2 L={L}", ys2[1][0], xs2[i], st1[0], None if res is None else res2[i])
        uni_y.append((ys[0][0], ys2[1][0]))
        uni_st1.append(st1[0])
        uni_st2.append(st2[0])
    monkeypatch.delenv("ADEC_STACK_ROWS")
    # ---- stacked: 16 streams of short chunks (the tensor-core engines stack them into shared tiles)
    Ls = 5
    xs16 = [gx(cin, Ls, j % 5) for j in range(16)]
    xs16b = [gx(cin, Ls, j + 2) for j in range(16)]
    st16 = np.stack([gx(cin, P, j + 1) for j in range(16)])
    if c["pre_act"] == ACT_ELU:
        st16 = np.maximum(st16, -1.0).astype(np.float32)
    res16 = [gr(cout, _outlen(c, Ls), 0) for _ in range(16)] if c["res"] else None
    ys16, st16_out, recs = run_op(c, W, 0, [[Ls] * 16], [xs16], 16, states=st16.copy(), res=None if res16 is None else [res16])
    LAUNCHED.update((engine,) + r for r in recs)
    tc = [r for r in recs if r[0] == 0]
    assert all(r[7] == 1 for r in tc), f"{c['name']} {engine}: the 16 short streams did not run stacked: {tc}"
    for j in range(16):
        score(f"stacked #{j}", ys16[0][j], xs16[j], st16[j], None if res16 is None else res16[j])
        if P:
            check_state(f"stacked #{j}", st16_out[j], st16[j], xs16[j])
    if engine == "ffma":
        REPORT.append(f"{c['name']:24s} {engine:5s} {weights:6s} uniform+stacked   e = {e_max:.3g}  e_ref = {eref_max:.3g}")
        return
    # the same 16 chunks as one slot call: every output and state bit as stacked
    ys16s, st16s, _ = run_op(c, W, 3, [[Ls] * 16], [xs16], 16, n_streams=16, streams=[list(range(16))], states=st16.copy(),
                             res=None if res16 is None else [res16])
    for j in range(16):
        np.testing.assert_array_equal(ys16s[0][j], ys16[0][j], err_msg=f"{c['name']} {engine}: slot vs stacked #{j}")
    if P:
        np.testing.assert_array_equal(st16s, st16_out, err_msg=f"{c['name']} {engine}: slot vs stacked states")
    # ---- stream slots, two calls on one handle.  Call 1: every utterance and the 16 short streams; two streams idle.  Call 2:
    # every utterance again, 14 of the short streams and the two idle ones; the last two short streams sit out.
    ns = n + 16 + 2
    perm = rng.permutation(ns)
    slot_u, slot_s, idle = perm[:n], perm[n:n + 16], perm[n + 16:]
    init = np.zeros((ns, cin, P), np.float32)
    init[slot_u], init[slot_s] = sts[:n], st16
    init[idle] = sts[n:]
    x_idle = [gx(cin, Ls, j) for j in range(2)]
    r_idle = [gr(cout, _outlen(c, Ls), 0) for _ in range(2)] if c["res"] else None
    L1 = lens + [Ls] * 16
    calls_x = [xs + xs16, xs2 + xs16b[:14] + x_idle]
    calls_r = None if res is None else [res + res16, res2 + res16[:14] + r_idle]
    streams = [list(slot_u) + list(slot_s), list(slot_u) + list(slot_s[:14]) + list(idle)]
    ys_s, st_s, recs = run_op(c, W, 3, [L1, L1], calls_x, n + 16, n_streams=ns, streams=streams, states=init.copy(), res=calls_r)
    LAUNCHED.update((engine,) + r for r in recs)
    for i in range(n):
        for k in range(2):
            np.testing.assert_array_equal(ys_s[k][i], uni_y[i][k], err_msg=f"{c['name']} {engine}: slots vs uniform, call {k + 1}, L={lens[i]}")
        if P:
            np.testing.assert_array_equal(st_s[slot_u[i]], uni_st2[i], err_msg=f"{c['name']} {engine}: slot state, L={lens[i]}")
    for j in range(16):
        np.testing.assert_array_equal(ys_s[0][n + j], ys16[0][j], err_msg=f"{c['name']} {engine}: slots vs stacked #{j}")
    for j in range(14):
        score(f"slots call 2 short #{j}", ys_s[1][n + j], xs16b[j], st16_out[j], None if res16 is None else res16[j])
        if P:
            check_state(f"slots call 2 short #{j}", st_s[slot_s[j]], st16_out[j], xs16b[j])
    for j in range(2):
        score(f"slots call 2 idle #{j}", ys_s[1][n + 14 + j], x_idle[j], init[idle[j]], None if r_idle is None else r_idle[j])
        if P:
            check_state(f"slots call 2 idle #{j}", st_s[idle[j]], init[idle[j]], x_idle[j])
            # the streams call 2 did not advance keep the state call 1 left, bit for bit
            np.testing.assert_array_equal(st_s[slot_s[14 + j]], st16_out[14 + j], err_msg=f"{c['name']} {engine}: sat-out stream")
    # ---- offline: varlen over every utterance plus 200 one-row utterances sharing a tile, against uniform offline calls
    ones = [gx(cin, 1, j % 5) for j in range(200)] if not c["res"] else []
    Lv = lens + [1] * len(ones)
    resv = None if res is None else [res]
    ys_v, _, recs = run_op(c, W, 2, [Lv], [xs + ones], len(Lv), res=resv)
    LAUNCHED.update((engine,) + r for r in recs)
    for i, L in enumerate(lens):
        yo, _, recs = run_op(c, W, 1, [[L]], [[xs[i]]], 1, res=None if res is None else [[res[i]]])
        LAUNCHED.update((engine,) + r for r in recs)
        np.testing.assert_array_equal(ys_v[0][i], yo[0][0], err_msg=f"{c['name']} {engine}: varlen vs offline, L={L}")
        score(f"offline L={L}", yo[0][0], xs[i], None, None if res is None else res[i])
    if ones:
        yo, _, _ = run_op(c, W, 1, [[1] * len(ones)], [ones], len(ones))
        for j in range(len(ones)):
            np.testing.assert_array_equal(ys_v[0][n + j], yo[0][j], err_msg=f"{c['name']} {engine}: one-row utterance #{j}")
    REPORT.append(f"{c['name']:24s} {engine:5s} {weights:6s} all row spaces    e = {e_max:.3g}  e_ref = {eref_max:.3g}")


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="act_elu is accurate to 2.4e-7 ABSOLUTE, not relative to the value: small ELU inputs lose "
                                       "precision on every engine (DESIGN section 3)")
@pytest.mark.parametrize("engine", ["f16", "tf32"])
def test_elu_small_activations_relative(engine, monkeypatch):
    """ELU inputs in [-1e-2, -1e-5] through a residual unit and its state: held to the same relative bar as every other op, which
    the current ELU misses (H100: output e 1.4e-5 against e_ref 2.9e-7, state e 5.6e-3 against 5.8e-8).  Strict: a relative-accurate ELU makes this pass, and
    then the marker goes."""
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    c = CASES[1]
    rng = np.random.default_rng(7)
    W = gen_weights(rng, c)
    x = gen_x(rng, 32, 200, 2)
    st = np.maximum(gen_x(rng, 32, 6, 2), -1.0).astype(np.float32)
    ys, st_out, _ = run_op(c, W, 0, [[200]], [[x]], 1, states=st[None].copy())
    e, eref = _check("small ELU", c, W, ys[0][0], x, st, slack=False)
    ex = np.concatenate([st, act(c, x, W, torch.float64).numpy()], 1)[:, -6:]
    es = err(st_out[0], ex, np.abs(ex))
    esref = err(expected_state(c, W, st, x), ex, np.abs(ex))
    REPORT.append(f"small ELU inputs {engine:5s} output e = {e:.3g} e_ref = {eref:.3g}; state e = {es:.3g} e_ref = {esref:.3g}")
    assert e <= bar(eref) and es <= bar(esref), (e, eref, es, esref)


# ops without ELU (whose absolute error would mask this one): the 1x1, LeakyReLU, a plain k7 conv and a LeakyReLU transposed conv
ENVELOPE_OPS = ["conv_out", "convs2.v1.nt32", "decoder.conv1", "upsamples.0"]
F16_RANGE_XFAIL = pytest.mark.xfail(strict=True, reason="the fp16-split activation pieces are unscaled: a receptive field below "
                                                        "fp16's normal range (2^-14) leaves both subnormal (DESIGN section 3)")


@pytest.mark.gpu
@pytest.mark.parametrize("engine,m", [pytest.param(e, m, marks=F16_RANGE_XFAIL if e == "f16" and m >= 20 else ())
                                      for e in ("f16", "tf32", "ffma") for m in (0, 8, 14, 20, 24, 30)])
def test_activation_envelope(engine, m, monkeypatch):
    """O(1) weights, no bias, chunk and state rows whose whole receptive field is 2^-m * O(1): held to the op bar.  The fp16-split
    engine splits activations without a scale, so it holds only down to about 2^-14; below that (m >= 20) it is a strict xfail."""
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    rng = np.random.default_rng(100 + m)
    bad = []
    for name in ENVELOPE_OPS:
        c = dict(next(c for c in CASES if c["name"] == name), bias=False, res=False)
        W = gen_weights(rng, c)
        W["w"] = (rng.standard_normal(W["w"].shape) / np.sqrt(_terms(c))).astype(np.float32)
        cin, P, L = _cin_x(c), _hist(c), 200
        x = (gen_x(rng, cin, L, 0) * 2.0 ** -m).astype(np.float32)
        st = (gen_x(rng, cin, P, 0) * 2.0 ** -m).astype(np.float32)
        ys, _, _ = run_op(c, W, 0, [[L]], [[x]], 1, states=st[None].copy())
        e, eref = _check("envelope", c, W, ys[0][0], x, st)
        b = bar(eref, engine, _terms(c))
        REPORT.append(f"envelope 2^-{m:<2d} {name:16s} {engine:5s} e = {e:.3g}  e_ref = {eref:.3g}  bar = {b:.3g}")
        print(REPORT[-1])
        if not e <= b:
            bad.append(REPORT[-1])
    assert not bad, bad


# entries of kTcKernels (adec.cu) of the fp32-grade precisions: (NT, fuse, pre-activation, prec, varlen, paired)
def _tc_entries():
    out = []
    for prec in (PREC_F16, PREC_TF32):
        for nt in (128, 64, 32):
            for fuse, pre in ((1, ACT_ELU), (0, ACT_NONE), (0, ACT_ELU), (0, ACT_LRELU), (0, ACT_NORM)):
                for vl in (0, 1):
                    out.append((nt, fuse, pre, prec, vl, 0))
                if nt == 32 and fuse and prec == PREC_F16:
                    out.append((nt, fuse, pre, prec, 0, 1))
    return out


def _plan_launches(engine):
    """(NT, fuse, pre, prec, varlen, paired) of every tensor-core launch the released fp32 plans make, recorded on real handles:
    uniform B = 1 (unstacked: long chunks), 16 stacked streams and a varlen batch, encoder and decoder"""
    from audiodec_b200 import _lib
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    lib = _lib.load()
    dev = torch.device("cuda:0")
    seen = set()

    def collect(g, run):
        lib.adec_record_launches(g._h, 1)
        run(g)
        torch.cuda.synchronize()
        n = lib.adec_launch_records(g._h, None, 0)
        buf = np.zeros(n * _lib.TEST_REC, np.int32)
        lib.adec_launch_records(g._h, buf.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), n)
        lib.adec_record_launches(g._h, 0)
        seen.update(tuple(int(v) for v in r[1:7]) for r in buf.reshape(-1, _lib.TEST_REC) if r[0] == 0)

    torch.manual_seed(0)
    for params in (S.SYMAD_PARAMS, S.SYMAAD_PARAMS, S.SYMAD_C16_PARAMS):
        g = SymADStreamGenerator(**params)
        g.load_state_dict(S.symad_state_dict(params, seed=0))
        g = g.eval().to(dev)

        def run_symad(g):
            z = g.encode(0.1 * torch.randn(1, 1, 40 * 320, device=dev))
            g.decode(torch.randn(1, z.shape[-1], 64, device=dev))
            g.encode(0.1 * torch.randn(16, 1, 40, device=dev))       # short chunks: stacked tiles down to RU(32)
            g.decode(torch.randn(16, 1, 64, device=dev))
            z, frames = g.encode_offline_varlen([0.1 * torch.randn(1, n, device=dev) for n in (3000, 700)])
            g.decode_offline_varlen(z, frames)
        collect(g, run_symad)
    for params in (S.HIFIGAN_V0_PARAMS, S.HIFIGAN_V1_PARAMS, S.HIFIGAN_V2_PARAMS):
        g = HiFiGANStreamGenerator(**params)
        g.load_state_dict(S.hifigan_state_dict(params, seed=1))
        g = g.eval().to(dev)

        def run_hifigan(g):
            g.decode(torch.randn(1, 40, 64, device=dev))
            g.decode(torch.randn(16, 1, 64, device=dev))
            g.forward_varlen(torch.randn(1, 64, 13, device=dev), [10, 3])
        collect(g, run_hifigan)
    return seen


def _case_launches(engine):
    """the same for the op cases, each run uniform unstacked, as 16 stacked streams and varlen"""
    rng = np.random.default_rng(11)
    seen = set()
    for c in CASES:
        W = gen_weights(rng, c)
        cin = _cin_x(c)
        res = lambda Ls: None if not c["res"] else [[gen_x(rng, _cout(c), _outlen(c, L), 0) for L in Ls]]
        runs = [(0, [130], 1), (0, [5] * 16, 16), (2, [130, 5], 2)]
        for mode, Ls, B in runs:
            os.environ["ADEC_STACK_ROWS"] = "0" if B == 1 else "1"
            try:
                _, _, recs = run_op(c, W, mode, [Ls], [[gen_x(rng, cin, L, 0) for L in Ls]], B, res=res(Ls))
            finally:
                del os.environ["ADEC_STACK_ROWS"]
            seen.update(tuple(int(v) for v in r[1:7]) for r in recs if r[0] == 0)
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["f16", "tf32"])
def test_instantiation_coverage(engine, monkeypatch):
    """Every tensor-core instantiation a released fp32 plan selects (recorded on real symAD / symAAD / c16 and HiFi-GAN v0 / v1 / v2
    handles, uniform, stacked and varlen) is launched by the op cases, so a plan op shape missing from CASES fails here.  Prints the
    fp32-grade kTcKernels entries no plan selects."""
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    plan, cases = _plan_launches(engine), _case_launches(engine)
    prec = PREC_F16 if engine == "f16" else PREC_TF32
    assert plan, "no tensor-core launch recorded"
    assert plan <= cases, f"{engine}: plan instantiations no case launches: {sorted(plan - cases)}"
    unused = [e for e in _tc_entries() if e[3] == prec and e not in plan]
    for line in REPORT:
        print(line)
    print(f"{engine}: instantiations the plans select (NT, fuse, pre, prec, varlen, paired): {sorted(plan)}")
    print(f"{engine}: fp32-grade kTcKernels entries no released plan selects: {unused}")
    if engine == "f16":
        assert any(r[5] for r in plan), "the paired RU(32) kernel never ran"


# ------------------------------------------------------------------------------------------------------------------------------
# range flag of the fp16-split engine at the op: the documented threshold, inf, and tf32
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["f16", "tf32"])
def test_range_flag_op_threshold(engine, monkeypatch):
    """A 1x1 identity conv whose output is exactly 6e4 (every fp16 piece exact) sets the f16 flag, reported once then 0; an output of
    5.9e4 does not; an inf output (weights 1e35) sets it.  tf32 never sets it."""
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    c = _case("flag", CONV, 32, 32, 1, bias=False)
    for value, wscale, want in ((6e4, 1.0, 1), (5.9e4, 1.0, 0), (1e4, 1e35, 1)):
        W = dict(w=(np.eye(32, dtype=np.float32) * np.float32(wscale))[:, :, None].copy(), w2=None, b=None, mean=None, scale=None)
        x = np.zeros((32, 8), np.float32)
        x[5, 3] = value
        flag = []
        ys, _, _ = run_op(c, W, 0, [[8]], [[x]], 1, states=np.zeros((1, 32, 0), np.float32), flag_out=flag)
        y = ys[0][0][5, 3]
        assert (y == np.float32(value * wscale)) if np.isfinite(np.float32(value * wscale)) else np.isinf(y)
        assert flag == [want if engine == "f16" else 0, 0], (value, wscale, flag)


# ------------------------------------------------------------------------------------------------------------------------------
# range flag of the fp16-split engine, through the public API
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["f16", "tf32"])
def test_range_flag_public_api(engine, monkeypatch, symad_sd):
    """A symAD encoder whose projector weight is scaled until z crosses 6e4 raises the flag on f16 (reported once, then cleared),
    and adec_codec_host fails with its message; tf32 has no range limit and never sets it.  The unscaled model does not set it."""
    from audiodec_b200 import synthetic as S
    from audiodec_b200 import _lib
    from audiodec_b200.codec import SymADStreamGenerator
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    x = 0.1 * torch.randn(1, 1, 3000)
    for scale, want in ((1.0, False), (1e7, engine == "f16")):
        sd = {k: v.clone() for k, v in symad_sd.items()}
        sd["projector.project.conv.weight"] = sd["projector.project.conv.weight"] * scale
        g = SymADStreamGenerator(**S.SYMAD_PARAMS)
        g.load_state_dict(sd)
        g = g.eval().to(dev)
        g.initial_encoder(8192, dev)
        z = g.encode(x.to(dev))
        torch.cuda.synchronize()
        assert g.range_error() is want, f"{engine} scale {scale}: max |z| = {z.abs().max().item():.3g}"
        assert g.range_error() is False
        if want:
            lib = _lib.load()
            xh = x.numpy().copy()
            F_ = lib.adec_frames_for(g._h, xh.shape[-1])
            idx = np.zeros((S.SYMAD_PARAMS["codebook_num"], 1, F_), np.int64)
            y = np.zeros(F_ * 300, np.float32)
            rc = lib.adec_codec_host(g._h, g._h, _p(xh), 1, xh.shape[-1], _p(idx), _p(y), None)
            assert rc != 0 and "6e4" in _lib.last_error(g._h)


# ------------------------------------------------------------------------------------------------------------------------------
# negative controls (CPU): wrong arithmetic and wrong row maps, scored by the same checker, must fail it
# ------------------------------------------------------------------------------------------------------------------------------
def _f16(v):
    return v.astype(np.float16).astype(np.float64)


def _tf32(v):
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32).astype(np.float64)


def _bf16(v):
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32).astype(np.float64)


def _model_products(a, w, model, scale="column"):
    """a (T, K) fp32 activations, w (K, N) fp32 weights -> the sums one engine model forms (fp64 accumulation of its products).
    scale: the fp16 planes' power of two 2^p, max |w| 2^p in [4096, 8192), per output "column" (the engine) or per "op"; p = 0 where
    the max is 0, and 2^-p stays a normal float (adec.cu finalize_op_wg)"""
    a = a.astype(np.float64)
    w = w.astype(np.float64)
    wmax = np.abs(w).max(0, keepdims=True) if scale == "column" else np.abs(w).max(keepdims=True)
    p = np.where(wmax > 0, np.clip(13 - np.frexp(wmax)[1], -127, 126), 0)
    ws = w * 2.0 ** p
    w_hi = _f16(ws)
    w_lo = _f16(ws - w_hi)
    w_his = _f16(w_hi / 2048)
    a_hi = _f16(a)
    lo_scale = 1.0 if model == "no_lo_scale" else 2048.0
    a_lo = _f16((a - a_hi) * lo_scale)
    if model in ("f16_split", "no_lo_scale"):
        return (a_lo @ w_his + a_hi @ w_lo + a_hi @ w_hi) * 2.0 ** -p
    if model == "hi_only":
        return (a_hi @ w_hi) * 2.0 ** -p
    if model == "two_products":
        return (a_hi @ w_lo + a_hi @ w_hi) * 2.0 ** -p
    if model == "tf32x1":
        return _tf32(a) @ _tf32(w)
    if model == "bf16":
        return _bf16(a) @ _bf16(w)
    raise ValueError(model)


def _cpu_case(rng, C=64, K=7, T=300):
    a = np.concatenate([gen_x(rng, C, T, r) for r in (0, 1, 3)], 1).T.copy()     # rows: O(1), channel-scaled, near 2^-14 / 2^-24
    w = (rng.standard_normal((C, K)) * 2.0 ** rng.uniform(-12, 12, (C, K))).astype(np.float32)
    exact = a.astype(np.float64) @ w.astype(np.float64)
    S = np.abs(a.astype(np.float64)) @ np.abs(w.astype(np.float64))
    ref32 = (torch.from_numpy(a) @ torch.from_numpy(w)).numpy()
    return a, w, exact, S, err(ref32, exact, S)


def test_checker_accepts_the_fp16_split_model():
    a, w, exact, S, e_ref = _cpu_case(np.random.default_rng(1))
    e = err(_model_products(a, w, "f16_split"), exact, S)
    assert e <= bar(e_ref), (e, e_ref)


N_TERMS_MAX = max(_terms(c) for c in CASES)


@pytest.mark.parametrize("engine", ["f16", "ffma"])
@pytest.mark.parametrize("model", ["hi_only", "two_products", "tf32x1", "bf16", "no_lo_scale"])
def test_checker_rejects_wrong_arithmetic(model, engine):
    """against the tensor-core bar, and against the FFMA bar at the longest sum any case has (its loosest)"""
    a, w, exact, S, e_ref = _cpu_case(np.random.default_rng(1))
    e = err(_model_products(a, w, model), exact, S)
    b = bar(e_ref, engine, N_TERMS_MAX)
    assert e > b, f"{model}: e = {e:.3g} passes the {engine} bar {b:.3g}"


def test_checker_ladder_needs_per_column_scales():
    """The channel ladder (apply_ladder's columns, 224 O(1) products per output with the 2^24 per-element spread) through the same
    checker: the fp16-split model with one scale per op fails it (columns 2^-17 and below lose W_lo to fp16 subnormals), the model
    with one scale per column passes it."""
    rng = np.random.default_rng(3)
    K, N = 224, 2 * len(LADDER_K)
    a = gen_x(rng, K, 400, 0).T.copy()
    w = (rng.standard_normal((K, N)) / np.sqrt(K) * 2.0 ** rng.uniform(-12, 12, (K, N)) / 2.0 ** 6 * ladder(N)).astype(np.float32)
    exact = a.astype(np.float64) @ w.astype(np.float64)
    S = np.abs(a.astype(np.float64)) @ np.abs(w.astype(np.float64))
    e_ref = err((torch.from_numpy(a) @ torch.from_numpy(w)).numpy(), exact, S)
    e_op = err(_model_products(a, w, "f16_split", scale="op"), exact, S)
    e_col = err(_model_products(a, w, "f16_split", scale="column"), exact, S)
    assert e_op > bar(e_ref), f"per-op scale: e = {e_op:.3g} passes the bar {bar(e_ref):.3g}"
    assert e_col <= bar(e_ref), f"per-column scale: e = {e_col:.3g} > bar {bar(e_ref):.3g}"


def _elu_abs_model(t):
    """the ELU of the old kernel comment: expm1 within 2.4e-7 ABSOLUTE (exp(x) carried to 2^-22 relative, then - 1)"""
    e = torch.exp(t.double())
    e = e * (1 + 2.0 ** -22 * torch.sign(torch.sin(1e4 * t.double())))
    return torch.where(t > 0, t.double(), (e - 1)).to(t.dtype)


def test_checker_rejects_absolute_elu_on_small_activations():
    rng = np.random.default_rng(2)
    c = _case("ru", RU, 32, 32, 7, d=3, bias=False)
    W = gen_weights(rng, c)
    x = gen_x(rng, 32, 200, 2)
    hist = np.zeros((32, 18), np.float32)
    ex, S = reference(c, W, x, hist, torch.float64)
    y32, _ = reference(c, W, x, hist, torch.float32)
    bad, _ = reference(c, W, x, hist, torch.float32, elu_fn=_elu_abs_model)
    e_ref = err(y32.numpy(), ex.numpy(), S.numpy())
    assert e_ref <= bar(e_ref)
    e = err(bad.numpy(), ex.numpy(), S.numpy())
    assert e > bar(e_ref), f"e = {e:.3g}, e_ref = {e_ref:.3g}"


def _row_map_case(kind):
    rng = np.random.default_rng(4)
    if kind == "convtr":
        c = _case("tr", CONVTR, 32, 32, s=4)
    else:
        c = _case("conv", CONV, 32, 32, 7, d=3)
    W = gen_weights(rng, c)
    x = gen_x(rng, 32, 40, 0)
    hist = gen_x(rng, 32, _hist(c), 0)
    return c, W, x, hist


@pytest.mark.parametrize("wrong", ["history_one_row_off", "varlen_reads_predecessor", "convtr_no_first_row_replication",
                                   "slot_reads_stale_buffer"])
def test_checker_rejects_wrong_row_maps(wrong):
    c, W, x, hist = _row_map_case("convtr" if wrong == "convtr_no_first_row_replication" else "conv")
    rng = np.random.default_rng(5)
    if wrong == "history_one_row_off":          # stream call: the window starts one row late
        good = hist
        bad_hist = np.concatenate([hist[:, 1:], x[:, :1]], 1)
        ex, S = reference(c, W, x, good, torch.float64)
        y, _ = reference(c, W, x, bad_hist, torch.float32)
    elif wrong == "varlen_reads_predecessor":   # offline utterance: its halo holds the previous utterance's rows, not zeros
        pred = gen_x(rng, 32, _hist(c), 0)
        ex, S = reference(c, W, x, None, torch.float64, offline=True)
        y, _ = reference(c, W, x, pred, torch.float32)
    elif wrong == "convtr_no_first_row_replication":   # offline transposed conv with a zero history row
        ex, S = reference(c, W, x, None, torch.float64, offline=True)
        y, _ = reference(c, W, x, np.zeros((32, 1), np.float32), torch.float32)
    else:                                       # a slot whose bit says "other buffer" reads the one from two calls ago
        stale = gen_x(rng, 32, _hist(c), 0)
        ex, S = reference(c, W, x, hist, torch.float64)
        y, _ = reference(c, W, x, stale, torch.float32)
    e_ref = err(reference(c, W, x, None if "varlen" in wrong or "convtr" in wrong else hist, torch.float32,
                          offline="varlen" in wrong or "convtr" in wrong)[0].numpy(), ex.numpy(), S.numpy())
    e = err(y.numpy(), ex.numpy(), S.numpy())
    assert e > bar(e_ref), f"{wrong}: e = {e:.3g}"


def test_test_op_struct_matches_header():
    import re
    from audiodec_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "audiodec_b200.h")).read()
    body = hdr[hdr.index("typedef struct adec_test_op {"):hdr.index("} adec_test_op;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for group in re.findall(r"\b(?:int|float|const float)\s+([^;]+);", body):
        fields += [f.strip().lstrip("*") for f in group.split(",")]
    assert fields == [f[0] for f in _lib.AdecTestOp._fields_]


# ------------------------------------------------------------------------------------------------------------------------------
# whole encoder: the golden symAD input at four amplitudes, against the oracle in fp64
# ------------------------------------------------------------------------------------------------------------------------------
def decidable_frames(z64, embeds64, delta):
    """frames whose fp64 residual-VQ decisions no perturbation of z with L2 norm <= delta can change: at every stage the top-2
    distance gap exceeds 2 * delta * |e1 - e2| (a perturbation d moves |r - e_j|^2 - |r - e_i|^2 by at most 2 |d| |e_j - e_i|)"""
    r = z64.T.copy()                                     # (F, D)
    ok = np.ones(r.shape[0], bool)
    idx = []
    for e in embeds64:                                   # (D, N)
        dist = (r ** 2).sum(1, keepdims=True) - 2 * r @ e + (e ** 2).sum(0, keepdims=True)
        o = np.argsort(dist, 1)[:, :2]
        rows = np.arange(r.shape[0])
        gap = dist[rows, o[:, 1]] - dist[rows, o[:, 0]]
        ok &= gap > 2 * delta * np.linalg.norm(e[:, o[:, 0]] - e[:, o[:, 1]], axis=0)
        idx.append(o[:, 0])
        r = r - e[:, o[:, 0]].T
    return ok, np.stack(idx)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["f16", "tf32"])
@pytest.mark.parametrize("model", ["symAD", "symAAD", "c16"])
def test_encoder_amplitude_sweep(model, engine, monkeypatch, golden_dir):
    """The golden symAD clip scaled by 2^-k, k in {0, 4, 8, 12, 16, 20, 24} (quiet audio: the ELU's small-activation gap is where
    it would show), exact digital silence and isolated clicks in silence, through the symAD, symAAD (ELU before the projector) and
    c16 (strides 2 / 4 / 5 / 8, 16 codebooks) encoders: offline z within 4x the fp32 oracle's own error against the fp64 oracle, and
    the code indices equal to the fp32 oracle's on every frame whose fp64 decisions are wider than the measured z error.  The biases
    keep the activations O(1) past the first layer, so even silence stays inside the fp16-split activation envelope
    (test_activation_envelope)."""
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import SymADStreamGenerator
    from oracle import audiodec_oracle as O
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    dev = torch.device("cuda:0")
    params = {"symAD": S.SYMAD_PARAMS, "symAAD": S.SYMAAD_PARAMS, "c16": S.SYMAD_C16_PARAMS}[model]
    sd = S.symad_state_dict(params, seed=0)
    g = SymADStreamGenerator(**params)
    g.load_state_dict(sd)
    g = g.eval().to(dev)
    o32 = O.SymADOracle(params, sd)
    o64 = O.SymADOracle(params, sd, dtype=torch.float64)
    embeds64 = [e.numpy() for e in o64.embeds]
    n = params["codebook_size"]
    x0 = torch.from_numpy(np.load(os.path.join(golden_dir, "symad_oneshot.npz"))["x"])
    clicks = torch.zeros_like(x0)
    clicks[..., [100, 2345, 2346, 7001, x0.shape[-1] - 1]] = torch.tensor([0.5, -0.25, 0.125, -1.0, 0.75])
    inputs = [(f"amplitude 2^-{k:<2d}", x0 * 2.0 ** -k) for k in (0, 4, 8, 12, 16, 20, 24)]
    inputs += [("digital silence", torch.zeros_like(x0)), ("clicks in silence", clicks)]
    for tag, x in inputs:
        zk = g.encode_offline(x.to(dev))
        idx_k = g.quantize(zk).cpu().numpy()
        zk = zk.cpu().double()[0].numpy()
        z32 = o32.forward_encode(x)
        idx32 = o32.quantize(z32).numpy()
        z32 = z32.double()[0].numpy()
        z64 = o64.forward_encode(x)[0].numpy()
        ek, e32 = np.abs(zk - z64).max(), np.abs(z32 - z64).max()
        delta = max(np.linalg.norm(zk - z64, axis=0).max(), np.linalg.norm(z32 - z64, axis=0).max())
        ok, idx64 = decidable_frames(z64, embeds64, delta)
        idx64 = idx64 + n * np.arange(len(embeds64))[:, None]
        REPORT.append(f"{model:6s} {tag:18s} {engine:5s} max|z| = {np.abs(z64).max():.3g}  z err = {ek:.3g}  fp32 oracle z err = {e32:.3g}  "
                      f"decidable frames {ok.sum()}/{ok.size}  index mismatches vs fp32 oracle: {(idx_k != idx32).any(0).sum()}")
        print(REPORT[-1])
        assert ek <= 4 * max(e32, 2.0 ** -23 * np.abs(z64).max()), REPORT[-1]
        np.testing.assert_array_equal(idx32[:, ok], idx64[:, ok])
        np.testing.assert_array_equal(idx_k[:, ok], idx32[:, ok], err_msg=REPORT[-1])
        assert ok.sum() >= ok.size // 2, REPORT[-1]
