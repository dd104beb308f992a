"""The symAD encoder's bf16 ops (compute_dtype 1: bf16 operands, fp32 storage; 2: bf16 operands and bf16 storage) op by op against
an exact rounding model, through `adec_test_conv_op` with a compute_dtype, in every row space: chunked streams, stacked streams,
varlen and stream slots.
The encoder's residual units are the decoder's fused / split units, covered by test_symad_bf16_layers_gpu.py.

The contract `model` restates (DESIGN §3):
  * strided conv (kernel 2s, a 2-tap conv over the s*Cin row view): operand bf16_rne(x), weights bf16_rne(w), fp32 accumulation,
    output sum + bias, stored once (fp32, or bf16_rne in mode 2); the causal state holds the last 2s - 1 input rows as stored;
  * projector (kernel 3, no bias, channels-first z): operand bf16_rne(x) or bf16_rne(ELU(x)) (symAAD), output the sum, stored once;
  * stem: fp32 weights and the fp32 FMA chain in both modes: mode 1 equals compute_dtype 0 bit for bit, and mode 2 (bf16 x, state and
    output) is bf16_rne of compute_dtype 0's output for the same bf16 x, bit for bit, on data that puts outputs on exact bf16 ties.
Sums are intervals as in the decoder's layer tests: exact dot products of the bf16 operands widened by 2^-16 S (S = sum |a w|), the
ELU by its 2.4e-7 bound, and the fp32 rounding of the last add.  The data holds exact bf16 ties, so a kernel that rounds operands
another way lands outside.  Negative controls (no GPU) feed the checker the outputs of wrong models - operands rounded toward zero,
and a causal window one row off - and require each to be rejected."""
import ctypes

import numpy as np
import pytest

from test_symad_bf16_layers_gpu import ACT_ELU, ACT_NONE, act_iv, b16, dot_iv, elu64
from test_vocoder_bf16_layers_gpu import bf16_round, from_words, ties, to_words

CONV, STEM = 0, 3
PREC_BF16 = 1
# the encoder's strided convs (synthetic.SYMAD_PARAMS: strides 3 4 5 5; SYMAD_C16_PARAMS: 2 4 5 8) and the projector
CASES = {
    "strided.s2": dict(Cin=32, Cout=64, s=2), "strided.s3": dict(Cin=32, Cout=64, s=3), "strided.s4": dict(Cin=64, Cout=128, s=4),
    "strided.s5": dict(Cin=128, Cout=256, s=5), "strided.s8": dict(Cin=256, Cout=512, s=8),
    "projector": dict(Cin=512, Cout=64, s=1, K=3, pre=ACT_NONE), "projector.elu": dict(Cin=512, Cout=64, s=1, K=3, pre=ACT_ELU),
}


def runs(s):
    """row spaces (test_conv_op mode, n_streams, calls), chunk lengths whole multiples of the stride in the streaming modes"""
    return [(0, 1, [[(0, 40 * s)], [(0, 5 * s)], [(0, 17 * s)]]), (0, 8, [[(b, 5 * s) for b in range(8)]]),
            (2, 3, [[(0, 130 * s + 1), (1, 7), (2, 1)]]), (3, 4, [[(2, 6 * s), (0, 2 * s)], [(0, s), (2, 3 * s)]])]


def kernel_of(case):
    c = CASES[case]
    return c.get("K", 2 * c["s"])


def model(case, x, w, bias, rounding="rne", off=False, mode=1):
    """x (Cin, T) fp32 from zero history -> (lo, hi, centre) (Cout, Tout) of the fp32 output.  rounding / off (every tap one row
    older): wrong models."""
    c = CASES[case]
    s, K, pre = c["s"], kernel_of(case), c.get("pre", ACT_NONE)
    rnd = (lambda v: bf16_round(np.asarray(v, np.float64).astype(np.float32), "rz").astype(np.float64)) if rounding == "rz" else b16
    lo, hi = act_iv(x, pre)
    alo, ahi, ac = rnd(lo), rnd(hi), rnd(elu64(x) if pre == ACT_ELU else x)
    P = K - 1 + (1 if off else 0)
    z = np.zeros((x.shape[0], P))
    alo, ahi, ac = (np.concatenate([z, v], 1) for v in (alo, ahi, ac))
    T = x.shape[1]
    Tout = (T - 1) // s + 1
    cols = lambda a: np.stack([a[:, t * s:t * s + K] for t in range(Tout)], 0).reshape(Tout, -1)   # (Tout, Cin * K)
    wq = bf16_round(w).astype(np.float64).reshape(w.shape[0], -1)
    l, h, S = dot_iv(cols(alo), cols(ahi), wq)
    cen = cols(ac) @ wq.T
    bq = np.zeros(w.shape[0]) if bias is None else bias.astype(np.float64)
    d = 2.0 ** -16 * S
    lo, hi, cen = l - d + bq, h + d + bq, cen + bq
    lo, hi = lo - 2.0 ** -24 * np.abs(lo), hi + 2.0 ** -24 * np.abs(hi)
    if mode == 2:
        return b16(lo).T, b16(hi).T, b16(cen).T
    return lo.T, hi.T, cen.astype(np.float32).astype(np.float64).T


def make_op(case, rng):
    c = CASES[case]
    K = kernel_of(case)
    w = rng.standard_normal((c["Cout"], c["Cin"], K)).astype(np.float32)
    t = rng.random(w.shape) < 0.25
    w[t] = ties(int(t.sum()), rng)
    w *= np.float32(2.0 ** -np.round(np.log2(np.sqrt(K * c["Cin"]))))
    b = None if case.startswith("projector") else (0.1 * rng.standard_normal(c["Cout"])).astype(np.float32)
    return w, b


def make_x(case, L, rng, mode=1):
    """mode 1: fp32 with exact bf16 ties; mode 2: bf16-representable values (what the kernel reads)"""
    x = rng.standard_normal((CASES[case]["Cin"], L)).astype(np.float32)
    x[rng.random(x.shape) < 0.05] = 0.0
    t = rng.random(x.shape) < 0.3
    x[t] = ties(int(t.sum()), rng)
    return bf16_round(x) if mode == 2 else x


def run(kind, Cin, Cout, K, stride, pre, out_nct, w, b, compute_dtype, mode, n_streams, calls, xs, P):
    """xs[k][j]: call k's utterance j (Cin, L) fp32.  Returns (ys like xs, launch records)."""
    from audiodec_b200 import _lib
    lib = _lib.load()
    p = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)
    d = _lib.AdecTestOp(kind=kind, Cin=Cin, Cout=Cout, K=K, stride=stride, dil=1, groups=1, shared_in=0, pre_act=pre, slope=0.0,
                        out_nct=out_nct, post_tanh=0, w=p(w), w2=None, bias=p(b), mean=None, scale=None, compute_dtype=compute_dtype)
    B = len(calls[0])
    lengths = np.array([[L for _, L in call] for call in calls], np.int32)
    streams = np.array([[s for s, _ in call] for call in calls], np.int32)
    x = np.concatenate([u.ravel() for call in xs for u in call]).astype(np.float32)
    if compute_dtype == 2:
        x = to_words(x)
    tout = lambda L: (L - 1) // stride + 1
    y = np.zeros(sum(Cout * tout(L) for call in calls for _, L in call), np.uint16 if compute_dtype == 2 else np.float32)
    st = np.zeros(n_streams * Cin * P, y.dtype)
    rec = np.zeros(16 * _lib.TEST_REC, np.int32)
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    rc = lib.adec_test_conv_op(0, ctypes.byref(d), mode, len(calls), B, n_streams, ip(lengths), ip(streams) if mode == 3 else None,
                               p(x), None, p(st), p(y), ip(rec), 16, None)
    assert rc == 0, _lib.last_error(None)
    if compute_dtype == 2:
        y = from_words(y)
    ys, at = [], 0
    for call in calls:
        ys.append([])
        for _, L in call:
            n = Cout * tout(L)
            ys[-1].append(y[at:at + n].reshape(Cout, -1))
            at += n
    return ys, [tuple(r) for r in rec.reshape(-1, _lib.TEST_REC) if r[0] >= 0]


def _sequences(mode, calls, xs, ys):
    seqs = {}
    for k, call in enumerate(calls):
        for j, (s, _) in enumerate(call):
            key = (k, j) if mode == 2 else s
            seqs.setdefault(key, ([], []))
            seqs[key][0].append(xs[k][j])
            seqs[key][1].append(ys[k][j])
    return {k: (np.concatenate(a, 1), np.concatenate(b, 1)) for k, (a, b) in seqs.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("compute_dtype", [1, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_op_against_rounding_model(case, compute_dtype):
    """Every row space: each stream's (or utterance's) outputs, its chunks in call order, inside the model's interval for its whole
    sequence from zero history (mode 2: stored bf16, and at least 99 % of all outputs on the contract applied to the exact value, which
    puts the strided-conv and channels-first z stores on their ties); the launches are PREC_BF16, with bf16 storage exactly in mode 2."""
    c = CASES[case]
    rng = np.random.default_rng(sorted(CASES).index(case) + 700 + 100 * compute_dtype)
    w, b = make_op(case, rng)
    worst, on, n = 0.0, 0, 0
    for mode, n_streams, calls in runs(c["s"]):
        xs = [[make_x(case, L, rng, compute_dtype) for _, L in call] for call in calls]
        ys, recs = run(CONV, c["Cin"], c["Cout"], kernel_of(case), c["s"], c.get("pre", ACT_NONE), int(case.startswith("projector")),
                       w, b, compute_dtype, mode, n_streams, calls, xs, kernel_of(case) - 1)
        for key, (x, y) in _sequences(mode, calls, xs, ys).items():
            lo, hi, cen = model(case, x, w, b, mode=compute_dtype)
            assert np.all((lo <= y) & (y <= hi)), (case, compute_dtype, mode, key, np.max(np.maximum(lo - y, y - hi)))
            worst = max(worst, float(np.max(np.abs(y - cen) / np.maximum(0.5 * (hi - lo), 1e-30))))
            on, n = on + int(np.sum(y == cen)), n + y.size
        assert recs and all(r[0] == 0 and r[4] == PREC_BF16 and r[8] == (compute_dtype == 2) for r in recs), recs
    print(f"[symAD tx bf16 layers] {case} mode {compute_dtype}: largest |y - exact| / half interval {worst:.3g}, on the exact value "
          f"{on / n:.4f}")
    if compute_dtype == 2:
        assert on >= 0.99 * n, (case, on / n)


def stem_weights(rng):
    """(name, w, bias): weights that are bf16 ties (bf16 weights would move every output); and one tap of 2^-m_c with a bias of
    2^-(8 + m_c), which puts the output 2^-m_c (x + 2^-8) of every input x = 1 + k 2^-7 on an exact bf16 tie, half of them with an
    odd lower neighbour (round-to-nearest-even goes up, truncation down)"""
    m = np.arange(32) % 4
    tie = np.zeros((32, 1, 7), np.float32)
    tie[:, 0, 6] = 2.0 ** -m
    return [("tie_weights", ties((32, 1, 7), rng) * np.float32(0.3), (0.1 * rng.standard_normal(32)).astype(np.float32)),
            ("tie_outputs", tie, (2.0 ** -(8 + m)).astype(np.float32))]


def stem_x(name, L, rng):
    if name == "tie_outputs":
        return (1.0 + rng.integers(0, 128, (1, L)) * 2.0 ** -7).astype(np.float32)
    return bf16_round(rng.standard_normal((1, L)).astype(np.float32) * np.float32(0.1))


def stem64(x, w, b):
    """the stem's exact output (32, T) from zero history, fp64"""
    xp = np.concatenate([np.zeros((1, 6)), x.astype(np.float64)], 1)
    y = np.stack([xp[0, t:t + 7] for t in range(x.shape[1])], 0) @ w[:, 0, :].astype(np.float64).T
    return (y + (0.0 if b is None else b.astype(np.float64))).T


@pytest.mark.gpu
@pytest.mark.parametrize("compute_dtype", [1, 2])
def test_stem_keeps_fp32_weights(compute_dtype):
    """compute_dtype 1 and 2 build the stem with fp32 weights, as compute_dtype 0 does: in every row space mode 1 equals compute_dtype
    0 bit for bit, and mode 2 (bf16 x, state and output) equals bf16_rne of compute_dtype 0's output on the same bf16 x - including
    outputs that are exact bf16 ties."""
    rng = np.random.default_rng(7 + compute_dtype)
    for name, w, b in stem_weights(rng):
        for mode, n_streams, calls in runs(1):
            xs = [[stem_x(name, L, rng) for _, L in call] for call in calls]
            yk, rk = run(STEM, 1, 32, 7, 1, ACT_NONE, 0, w, b, compute_dtype, mode, n_streams, calls, xs, 6)
            y0, r0 = run(STEM, 1, 32, 7, 1, ACT_NONE, 0, w, b, 0, mode, n_streams, calls, xs, 6)
            for a0, ak in zip((v for call in y0 for v in call), (v for call in yk for v in call)):
                np.testing.assert_array_equal(ak, bf16_round(a0) if compute_dtype == 2 else a0, err_msg=f"{name} mode {mode}")
            assert all(r[0] == 2 and r[8] == (compute_dtype == 2) for r in rk) and len(rk) == len(r0), (rk, r0)


# ------------------------------------------------------------------------------------------------ negative controls (no GPU)
@pytest.mark.parametrize("defect", ["rz", "off"])
@pytest.mark.parametrize("case", ["strided.s3", "strided.s8", "projector.elu"])
def test_checker_rejects_wrong_models(case, defect):
    """The centre of a wrong model (operands rounded toward zero, or a causal window one row off) lies outside the right model's
    interval somewhere: the checker would catch a kernel that computed it."""
    rng = np.random.default_rng(11)
    w, b = make_op(case, rng)
    x = make_x(case, 12 * CASES[case]["s"], rng)
    lo, hi, cen = model(case, x, w, b)
    assert np.all((lo <= cen) & (cen <= hi))
    _, _, bad = model(case, x, w, b, rounding=defect if defect == "rz" else "rne", off=defect == "off")
    assert not np.all((lo <= bad) & (bad <= hi)), (case, defect)


@pytest.mark.parametrize("defect", ["bf16_weights", "rz_store"])
def test_stem_checks_reject_wrong_models(defect):
    """On the stem test's data, a stem with bf16 weights, or one that stores bf16 by rounding toward zero, gives other bits than the
    contract somewhere, so the bit-for-bit comparison would catch it."""
    rng = np.random.default_rng(7)
    for name, w, b in stem_weights(rng):
        if name != {"bf16_weights": "tie_weights", "rz_store": "tie_outputs"}[defect]:
            continue
        x = stem_x(name, 200, rng)
        good = bf16_round(stem64(x, w, b).astype(np.float32))
        if defect == "bf16_weights":
            bad = bf16_round(stem64(x, bf16_round(w), b).astype(np.float32))
        else:
            bad = bf16_round(stem64(x, w, b).astype(np.float32), "rz")
        assert np.any(bad != good), (name, defect)
