"""The symAD decoder's bf16 kernels op by op (compute_dtype 1: bf16 operands, fp32 storage; 2: bf16 operands and bf16 storage)
against an exact rounding model, through `adec_test_conv_op` with compute_dtype 1 / 2 (the ops as a decoder-only handle builds them),
in every row space: chunked streams, stacked streams, varlen and stream slots.

The contract `_model` restates (DESIGN §3):
  * weights of the conv ops are rounded to bf16 (nearest-even) by the host packer; biases and the head's weights stay fp32;
  * an operand is bf16_rne(ELU(x)) (x fp32 in mode 1, bf16 in mode 2), causal-state rows hold the post-activation rows as stored;
  * fused residual unit: intermediate operand = bf16_rne(ELU(fp32 sum of the dilated conv)), rounded once; output = fp32 1x1 sum
    + x as stored, stored once (fp32, or bf16_rne in mode 2);
  * split residual unit (C = 256): the dilated conv's fp32 sum is stored (fp32 / bf16), then the 1x1 launch's operand is
    bf16_rne(ELU(stored value)) and its output the 1x1 sum + x as stored;
  * transposed conv (symAAD): operands bf16_rne(ELU(x)), output sum + bias; heads: fp32 weights, operand ELU(x) or x (bf16-rounded only
    in mode 2), output the fp32 sum, tanh for symAAD.
The kernel's ELU is ex2.approx(x log2 e) - 1, within 2.4e-7 absolute of expm1, and the tensor core's accumulation order is not
documented, so the model carries every value as an interval: operands [bf16(ELU(x) - 2.4e-7), bf16(ELU(x) + 2.4e-7)], sums as
interval dot products widened by 2^-16 S (S = sum |a w|, the vocoder tests' bound: a group of at most 64 products truncating at
each step plus at most 50 round-to-nearest adds), heads by 2^-18 S + 2 ulps (an fp32 FMA chain; tanhf).  Every output must lie in
its interval (stored: rounded like the kernel stores), and at least 99 % must equal the contract applied to the exact value.

That interval cannot see an accumulation order, so one case builds data whose group partial sums are exact in fp32 and whose
cross-group round-to-nearest adds are not: the kernel must equal the emulated two-taps-per-group order (WgCfg::tpg) bit for bit,
through an intermediate that is an exact bf16 tie.  Negative controls (no GPU) feed the checker the outputs of wrong models - the
intermediate rounded twice (torch's bf16 conv then bf16 ELU), the intermediate left unrounded, an fp32 skip in mode 2, and one tap
per group - and require each to be rejected."""
import ctypes

import numpy as np
import pytest

from test_vocoder_bf16_layers_gpu import bf16_round, from_words, ties, to_words

ELU_ABS = 2.4e-7
CONV, RU, CONVTR, HEAD = 0, 1, 2, 4
ACT_NONE, ACT_ELU = 0, 1

# name -> op, the shapes build_symad_decoder gives the symAD / symAAD decoders (synthetic.SYMAD*_PARAMS)
CASES = {
    "ru32.d1": dict(kind=RU, C=32, dil=1), "ru32.d3": dict(kind=RU, C=32, dil=3), "ru32.d9": dict(kind=RU, C=32, dil=9),
    "ru64.d1": dict(kind=RU, C=64, dil=1), "ru64.d9": dict(kind=RU, C=64, dil=9),
    "ru128.d3": dict(kind=RU, C=128, dil=3), "ru128.d9": dict(kind=RU, C=128, dil=9),
    "ru256.split.d1": dict(kind=RU, C=256, dil=1), "ru256.split.d9": dict(kind=RU, C=256, dil=9),
    "convtr.symAAD.s3": dict(kind=CONVTR, Cin=64, Cout=32, up=3, pre=ACT_ELU),
    "convtr.symAAD.s5": dict(kind=CONVTR, Cin=256, Cout=128, up=5, pre=ACT_ELU),
    "head.symAD": dict(kind=HEAD, pre=ACT_NONE, tanh=0), "head.symAAD": dict(kind=HEAD, pre=ACT_ELU, tanh=1),
}
# row spaces: (test_conv_op mode, n_streams, calls); a call is [(stream, rows)], its streams' chunks in order.  Mode 0: uniform
# streams (one chunk shorter than the history; B = 8 short chunks take the stacked rows), 2: varlen, 3: stream slots
RUNS = [(0, 1, [[(0, 130)], [(0, 5)], [(0, 71)]]), (0, 8, [[(s, 5) for s in range(8)]]), (2, 3, [[(0, 130), (1, 7), (2, 1)]]),
        (3, 4, [[(2, 6), (0, 40)], [(0, 1), (2, 9)]])]


# ------------------------------------------------------------------------------------------------ the model
def elu64(x):
    x = x.astype(np.float64)
    return np.where(x > 0, x, np.expm1(np.minimum(x, 0)))


def act_iv(x, pre):
    """fp32 pre-activation interval of the kernel's ELU (exact for x > 0 and for no activation)"""
    if pre == ACT_NONE:
        return x.astype(np.float64), x.astype(np.float64)
    e = elu64(x)
    slack = np.where(x > 0, 0.0, ELU_ABS)
    return e - slack, e + slack


def b16(v):
    """bf16_rne of fp32(v), as fp64: what a kernel stores for an fp32 value v (monotone in v)"""
    return bf16_round(np.asarray(v, np.float64).astype(np.float32)).astype(np.float64)


def store_iv(lo, hi, mode):
    return (b16(lo), b16(hi)) if mode == 2 else (lo, hi)


def dot_iv(clo, chi, w):
    """interval of cols @ w.T for cols in [clo, chi]; S = sum |a| |w|"""
    wp, wn = np.maximum(w, 0), np.minimum(w, 0)
    lo = clo @ wp.T + chi @ wn.T
    hi = chi @ wp.T + clo @ wn.T
    S = np.maximum(np.abs(clo), np.abs(chi)) @ np.abs(w).T
    return lo, hi, S


def taps(a, K, dil, T):
    """(C, P + T) window -> (T, C * K) columns of a causal dilated conv"""
    return np.stack([a[:, k * dil:k * dil + T] for k in range(K)], -1).transpose(1, 0, 2).reshape(T, -1)


def model(case, mode, x, w, w2=None, bias=None, replicate=False, defect=None):
    """One utterance or stream sequence x (Cin, T), fp32 as stored, from zero history (replicate: the transposed conv's first-row
    pad of the offline calls).  Returns (lo, hi, centre) per output: fp64 bounds of what the kernel may store and the contract
    applied to exact arithmetic, as stored.  defect: the stored output of a wrong model instead of the centre."""
    c = CASES[case]
    kind = c["kind"]
    T = x.shape[1]
    if kind == RU:
        K, dil = w.shape[-1], c["dil"]
        P = (K - 1) * dil
        lo, hi = act_iv(x, ACT_ELU)
        alo, ahi = b16(lo), b16(hi)
        ac = b16(elu64(x))
        z = np.zeros((x.shape[0], P))
        alo, ahi, ac = (np.concatenate([z, v], 1) for v in (alo, ahi, ac))
        wq = bf16_round(w).astype(np.float64).reshape(w.shape[0], -1)
        l1, h1, S1 = dot_iv(taps(alo, K, dil, T), taps(ahi, K, dil, T), wq)
        s1 = taps(ac, K, dil, T) @ wq.T                          # (T, C) exact
        d1 = 2.0 ** -16 * S1
        split = c["C"] > 128
        st = (lambda v: b16(v)) if (split and mode == 2) else (lambda v: v)
        ml = b16(elu64(st(l1 - d1)) - ELU_ABS)
        mh = b16(elu64(st(h1 + d1)) + ELU_ABS)
        mid = b16(elu64(st(s1)))
        if defect == "mid_twice":
            mid = b16(elu64(b16(s1)).astype(np.float32))
        elif defect == "mid_unrounded":
            mid = elu64(s1).astype(np.float32).astype(np.float64)
        w2q = bf16_round(w2[:, :, 0]).astype(np.float64)
        l2, h2, S2 = dot_iv(ml, mh, w2q)
        s2 = mid @ w2q.T
        xr = x.T.astype(np.float64)
        if defect == "skip_fp32":
            xr = c["x_fp32"].T.astype(np.float64)
        d2 = 2.0 ** -16 * S2
        lo, hi, cen = l2 - d2 + xr, h2 + d2 + xr, s2 + xr
        tanh = False
    elif kind == CONVTR:
        up = c["up"]
        lo, hi = act_iv(x, c["pre"])
        alo, ahi, ac = b16(lo), b16(hi), b16(elu64(x))
        first = [v[:, :1] if replicate else np.zeros((x.shape[0], 1)) for v in (alo, ahi, ac)]
        alo, ahi, ac = (np.concatenate([f, v], 1) for f, v in zip(first, (alo, ahi, ac)))
        wq = bf16_round(w).astype(np.float64)
        wr = np.concatenate([wq[:, :, :up], wq[:, :, up:]], 0).transpose(0, 2, 1).reshape(2 * w.shape[0], -1)   # (x[j], x[j-1])
        cols = lambda a: np.concatenate([a[:, 1:], a[:, :-1]], 0).T
        l, h, S = dot_iv(cols(alo), cols(ahi), wr.T)
        cen = cols(ac) @ wr
        fix = lambda v: v.reshape(T, up, -1).reshape(T * up, -1)
        bq = np.tile(bias.astype(np.float64), up)
        d = 2.0 ** -16 * (S + np.abs(bq))
        lo, hi, cen = fix(l + bq - d), fix(h + bq + d), fix(cen + bq)
        tanh = False
    else:                                                        # head: fp32 weights, operand rounded to bf16 only in mode 2
        lo, hi = act_iv(x, c["pre"])
        ac = elu64(x) if c["pre"] == ACT_ELU else x.astype(np.float64)
        if mode == 2:
            lo, hi, ac = b16(lo), b16(hi), b16(ac)
        z = np.zeros((32, 6))
        lo, hi, ac = (np.concatenate([z, v], 1) for v in (lo, hi, ac))
        wf = w.astype(np.float64).reshape(1, -1)
        l, h, S = dot_iv(taps(lo, 7, 1, T), taps(hi, 7, 1, T), wf)
        cen = taps(ac, 7, 1, T) @ wf.T
        d = 2.0 ** -18 * S
        lo, hi = l - d, h + d
        tanh = bool(c["tanh"])
        if tanh:
            lo, hi, cen = np.tanh(lo) - 2.0 ** -22, np.tanh(hi) + 2.0 ** -22, np.tanh(cen)
    lo, hi = lo - 2.0 ** -24 * np.abs(lo), hi + 2.0 ** -24 * np.abs(hi)   # the fp32 rounding of the last add
    lo, hi = store_iv(lo, hi, mode)
    cen = b16(cen) if mode == 2 else cen.astype(np.float32).astype(np.float64)
    return lo.T, hi.T, cen.T


def check(y, lo, hi, cen, mode):
    """(ok, statistic): every output inside its interval; mode 2 also at least 99 % of them equal to the contract applied to the
    exact value (the statistic: that fraction; mode 1: the largest distance from it relative to the interval's half width)"""
    y = y.astype(np.float64)
    inside = bool(np.all((lo <= y) & (y <= hi)))
    if mode == 1:
        return inside, float(np.max(np.abs(y - cen) / np.maximum(0.5 * (hi - lo), 1e-30)))
    frac = float(np.mean(y == cen))
    return inside and frac >= 0.99, frac


# ------------------------------------------------------------------------------------------------ data
def make_op(case, rng):
    c = CASES[case]
    if c["kind"] == RU:
        C = c["C"]
        w = rng.standard_normal((C, C, 7)).astype(np.float32)
        t = rng.random(w.shape) < 0.25
        w[t] = ties(int(t.sum()), rng)
        w *= np.float32(2.0 ** -np.round(np.log2(np.sqrt(7 * C))))
        w2 = (rng.standard_normal((C, C, 1)) * 0.6 / np.sqrt(C)).astype(np.float32)
        return dict(w=w, w2=w2, b=None)
    if c["kind"] == CONVTR:
        w = (rng.standard_normal((c["Cin"], c["Cout"], 2 * c["up"])) * 0.8 / np.sqrt(2 * c["Cin"])).astype(np.float32)
        return dict(w=w, w2=None, b=(0.1 * rng.standard_normal(c["Cout"])).astype(np.float32))
    return dict(w=(rng.standard_normal((1, 32, 7)) * 0.25 / np.sqrt(224)).astype(np.float32), w2=None, b=None)


def cin(case):
    c = CASES[case]
    return c.get("C") or c.get("Cin") or 32


def make_x(case, L, mode, rng):
    """O(1) activations with exact zeros, negatives through ELU and, in mode 1, bf16 ties; (fp32 as the kernel reads it, unrounded)"""
    x = rng.standard_normal((cin(case), L)).astype(np.float32)
    x[rng.random(x.shape) < 0.05] = 0.0
    t = rng.random(x.shape) < 0.2
    x[t] = ties(int(t.sum()), rng)
    return (bf16_round(x) if mode == 2 else x), x


def cout_of(case):
    c = CASES[case]
    return c.get("C") or c.get("Cout") or 1


def outlen(case, L):
    return L * CASES[case].get("up", 1)


# ------------------------------------------------------------------------------------------------ the GPU entry point
def run(case, W, compute_dtype, mode, n_streams, calls, xs):
    """xs[k][j]: call k's utterance j (Cin, L), fp32 values (bf16-representable in mode 2).  Returns (ys like xs, launch records)."""
    from audiodec_b200 import _lib
    lib = _lib.load()
    c = CASES[case]
    p = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)
    kind = c["kind"]
    d = _lib.AdecTestOp(kind=kind, Cin=cin(case), Cout=cout_of(case), K=7, stride=c.get("up", 1), dil=c.get("dil", 1), groups=1,
                        shared_in=0, pre_act=c.get("pre", ACT_ELU), slope=0.0, out_nct=0, post_tanh=c.get("tanh", 0),
                        w=p(W["w"]), w2=p(W["w2"]), bias=p(W["b"]), mean=None, scale=None, compute_dtype=compute_dtype)
    B = len(calls[0])
    lengths = np.array([[L for _, L in call] for call in calls], np.int32)
    streams = np.array([[s for s, _ in call] for call in calls], np.int32)
    flat = np.concatenate([u.ravel() for call in xs for u in call]).astype(np.float32)
    x = to_words(flat) if compute_dtype == 2 else flat
    ny = sum(cout_of(case) * outlen(case, L) for call in calls for _, L in call)
    y = np.zeros(ny, np.uint16 if compute_dtype == 2 else np.float32)
    P = {RU: 6 * c.get("dil", 1), CONVTR: 1, HEAD: 6}[kind]
    st = np.zeros(n_streams * cin(case) * P, y.dtype)
    rec = np.zeros(16 * _lib.TEST_REC, np.int32)
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    rc = lib.adec_test_conv_op(0, ctypes.byref(d), mode, len(calls), B, n_streams, ip(lengths), ip(streams) if mode == 3 else None,
                               p(x), None, p(st), p(y), ip(rec), 16, None)
    assert rc == 0, _lib.last_error(None)
    yv = from_words(y) if compute_dtype == 2 else y
    ys, at = [], 0
    for call in calls:
        ys.append([])
        for _, L in call:
            n = cout_of(case) * outlen(case, L)
            ys[-1].append(yv[at:at + n].reshape(cout_of(case), -1))
            at += n
    return ys, [tuple(r) for r in rec.reshape(-1, _lib.TEST_REC) if r[0] >= 0]


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("compute_dtype", [1, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_op_against_rounding_model(case, compute_dtype):
    """Every row space of RUNS: each stream's (or utterance's) outputs, its chunks in call order, inside the model's interval for its
    whole sequence from zero history; in mode 2, 99 % of all the case's outputs on the exact value.  The launches run PREC_BF16, fused where the unit is fused, with bf16 storage in mode 2."""
    rng = np.random.default_rng(sorted(CASES).index(case) + 100 * compute_dtype)
    W = make_op(case, rng)
    pooled = []
    for mode, n_streams, calls in RUNS:
        xs = [[make_x(case, L, compute_dtype, rng)[0] for _, L in call] for call in calls]
        ys, recs = run(case, W, compute_dtype, mode, n_streams, calls, xs)
        seqs = {}
        for k, call in enumerate(calls):
            for j, (s, _) in enumerate(call):
                key = (k, j) if mode == 2 else s
                seqs.setdefault(key, ([], []))
                seqs[key][0].append(xs[k][j])
                seqs[key][1].append(ys[k][j])
        for key, (xl, yl) in seqs.items():
            lo, hi, cen = model(case, compute_dtype, np.concatenate(xl, 1), W["w"], W["w2"], W["b"], replicate=mode == 2)
            y = np.concatenate(yl, 1)
            assert np.all((lo <= y) & (y <= hi)), (case, compute_dtype, mode, key)
            pooled.append((y.ravel(), lo.ravel(), hi.ravel(), cen.ravel()))
        tc = [r for r in recs if r[0] == 0]
        if CASES[case]["kind"] != HEAD:
            fused = CASES[case]["kind"] == RU and CASES[case]["C"] <= 128
            assert tc and all(r[4] == 1 and r[8] == (compute_dtype == 2) and not r[6] and r[2] == fused for r in tc), recs
    # the 99 % share over every output of the case (a few-row run can hold one cancelling sum near a bf16 rounding boundary)
    ok, stat = check(*(np.concatenate(v) for v in zip(*pooled)), compute_dtype)
    print(f"[symAD bf16 layers] {case} mode {compute_dtype}: " +
          (f"largest |y - exact| / half interval {stat:.3g}" if compute_dtype == 1 else f"fraction on the exact value {stat:.4f}"))
    assert ok, (case, compute_dtype, stat)


def grouping_case(C, dil, B0=40, T=80):
    """Data whose dilated-conv group partials are exact in fp32 and whose cross-group adds round: channel 0 holds 2^24 and channel 1
    2^16 at row B0 (their tap sum M = 2^24 + 2^16 is a bf16 tie), channel 2 holds 1 at rows B0 + 2 dil and B0 + 3 dil; output
    channel 0 sums channels 0..2 over all taps, the 1x1 is the identity.  Two taps per group give M + 2 at outputs B0 - j dil
    (j = 0, 2), one tap per group gives M (the tie), whose bf16 rounding differs by 2^17."""
    x = np.zeros((C, T), np.float32)
    x[0, B0], x[1, B0] = 2.0 ** 24, 2.0 ** 16
    x[2, B0 + 2 * dil] = x[2, B0 + 3 * dil] = 1.0
    w = np.zeros((C, C, 7), np.float32)
    w[0, :3, :] = 1.0
    w2 = np.eye(C, dtype=np.float32)[:, :, None]
    return x, w, w2


def emulate_grouped(x, w, w2, dil, tpg, mode):
    """The fused unit on exact-group data: group partials (asserted exact in fp32) added in tap order with fp32 round-to-nearest adds,
    then the contract's roundings.  Returns the stored output (C, T)."""
    C, T = x.shape
    a = np.concatenate([np.zeros((C, 6 * dil)), bf16_round(x).astype(np.float64)], 1)      # ELU is exact for x >= 0
    acc = np.zeros((T, C), np.float32)
    for t0 in range(0, 7, tpg):
        g = sum(a[:, (t0 + k) * dil:(t0 + k) * dil + T].T @ w[:, :, t0 + k].astype(np.float64).T for k in range(min(tpg, 7 - t0)))
        assert np.all(g.astype(np.float32) == g)
        acc = (acc + g.astype(np.float32)).astype(np.float32)
    mid = bf16_round(acc)
    s2 = mid.astype(np.float64) @ w2[:, :, 0].T.astype(np.float64)
    assert np.all(s2.astype(np.float32) == s2)
    y = (s2.astype(np.float32) + x.T).astype(np.float32)
    return (bf16_round(y) if mode == 2 else y).T


@pytest.mark.gpu
@pytest.mark.parametrize("compute_dtype", [1, 2])
@pytest.mark.parametrize("C,dil", [(32, 1), (64, 3), (128, 9)])
def test_fused_unit_tap_grouping_bitwise(C, dil, compute_dtype):
    """Two taps per group in every row space: the uniform chunked stream, 8 stacked streams and varlen all equal the emulated
    grouping bit for bit, through an intermediate that is an exact bf16 tie (nearest-even)."""
    x, w, w2 = grouping_case(C, dil)
    want = emulate_grouped(x, w, w2, dil, 2, compute_dtype)
    assert not np.array_equal(want, emulate_grouped(x, w, w2, dil, 1, compute_dtype))
    case = {32: "ru32.d1", 64: "ru64.d9", 128: "ru128.d9"}[C]
    saved = CASES[case]["dil"]
    CASES[case]["dil"] = dil
    try:
        W = dict(w=w, w2=w2, b=None)
        T = x.shape[1]
        ys, _ = run(case, W, compute_dtype, 0, 1, [[(0, 50)], [(0, T - 50)]], [[x[:, :50]], [x[:, 50:]]])
        np.testing.assert_array_equal(np.concatenate([ys[0][0], ys[1][0]], 1), want)
        ys, _ = run(case, W, compute_dtype, 0, 8, [[(s, T) for s in range(8)]], [[x] * 8])
        for s in range(8):
            np.testing.assert_array_equal(ys[0][s], want)
        ys, _ = run(case, W, compute_dtype, 2, 2, [[(0, 9), (1, T)]], [[x[:, :9], x]])
        np.testing.assert_array_equal(ys[0][1], want)
    finally:
        CASES[case]["dil"] = saved


# ------------------------------------------------------------------------------------------------ negative controls (no GPU)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("case", ["ru32.d3", "ru128.d9", "ru256.split.d1"])
def test_checker_rejects_wrong_intermediates(case, mode):
    """The checker accepts the contract's own output and rejects the intermediate rounded twice (torch's bf16 conv output, then a
    bf16 ELU) and the intermediate left unrounded, on the data the GPU cases use."""
    rng = np.random.default_rng(7)
    W = make_op(case, rng)
    x = make_x(case, 150, mode, rng)[0]
    lo, hi, cen = model(case, mode, x, W["w"], W["w2"])
    assert check(cen, lo, hi, cen, mode)[0]
    for defect in ("mid_twice", "mid_unrounded"):
        if CASES[case]["C"] > 128 and mode == 2 and defect == "mid_twice":
            continue            # the split unit's mode-2 contract is exactly that double rounding (its conv output is stored as bf16)
        y = model(case, mode, x, W["w"], W["w2"], defect=defect)[2]
        assert not check(y, lo, hi, cen, mode)[0], (case, mode, defect, check(y, lo, hi, cen, mode)[1])


@pytest.mark.parametrize("case", ["ru32.d1", "ru64.d9", "ru256.split.d9"])
def test_checker_rejects_fp32_skip_in_mode2(case):
    """Mode 2 adds x as stored (bf16); adding the fp32 value it was rounded from is rejected."""
    rng = np.random.default_rng(9)
    W = make_op(case, rng)
    x16, x32 = make_x(case, 150, 2, rng)
    lo, hi, cen = model(case, 2, x16, W["w"], W["w2"])
    CASES[case]["x_fp32"] = x32
    try:
        y = model(case, 2, x16, W["w"], W["w2"], defect="skip_fp32")[2]
    finally:
        del CASES[case]["x_fp32"]
    assert not check(y, lo, hi, cen, 2)[0], check(y, lo, hi, cen, 2)[1]


@pytest.mark.parametrize("mode", [1, 2])
def test_checker_rejects_wrong_tap_grouping(mode):
    """One tap per group is told apart from the kernels' two on the grouping data, at every dilation of the units."""
    for C, dil in ((32, 1), (64, 3), (128, 9)):
        x, w, w2 = grouping_case(C, dil)
        assert not np.array_equal(emulate_grouped(x, w, w2, dil, 1, mode), emulate_grouped(x, w, w2, dil, 2, mode))
