"""The vocoder's bf16 ops (compute_dtype 1: bf16 operands, fp32 storage; 2: bf16 operands and bf16 storage) op by op in every row
space through `adec_test_conv_op`, against the rounding model of test_vocoder_bf16_layers_gpu (`_model`, `check`), and the coverage of
every bf16 launch the released plans make.

Each case of the vocoder suite's CASES runs in four row spaces:
  * uniform: one stream (B = 1, ADEC_STACK_ROWS=0), three consecutive chunks of 300, 1 and 129 rows (1 < P for every P > 1);
  * stacked: 16 streams, consecutive chunks of 5, 1 and 3 rows, stacked into shared 128-row tiles;
  * varlen (offline): utterances of 300, 127, 128 and 129 rows, of fewer rows than P, and runs of 1-row utterances that share tiles,
    each from zero history (a transposed conv replicates its own first row);
  * slots: two calls on 8 stream slots that replay the uniform stream and six stacked ones; each call advances six slots, so the
    ping-pong bits flip per stream while one slot sits out the second call, one the first and one both.
Every output passes `check` against `_model` of its own stream or utterance (the statistic per row space: mode 1 the largest
|y - exact| / S, mode 2 the share of outputs on bf16_rne(exact)), and the state each stream is left with is the model's bit for bit,
an idle stream's included.  Per utterance, outputs are equal bit for bit across row spaces: the slots against the uniform and stacked
runs, varlen against uniform offline calls (mode 1 of the test entry point).  The mode-2 data hold the inputs the vocoder suite uses to
hit exact bf16 ties (`ties` in mode 1, the subnormal `lrelu_ties` in mode 2) and weights that are ties.

`adec_test_conv_op` builds the op as a symAD decoder-only handle does; `adec_test_vocoder_layer` as a HiFi-GAN handle does.  The two
must build the same op: same output and state bits for every case.  The bench's configs[3] shape (256 streams of 5-row chunks, mode 2)
runs against the model and against B = 1 calls of chosen streams.  `test_bf16_instantiation_coverage` records every launch of real
bf16 handles (HiFi-GAN v0 / v1 / v2, symAD / symAAD / c16 decoder and encoder) and requires each record to be produced by an op case
in a row space a test checks.  The CPU negative controls feed the checker and the row-space comparison wrong row maps."""
import contextlib
import ctypes
import os
import zlib

import numpy as np
import pytest

import test_symad_bf16_layers_gpu as dec_suite
import test_symad_encoder_bf16_layers_gpu as enc_suite
from test_vocoder_bf16_layers_gpu import (ACT_LRELU, ACT_NONE, ACT_NORM, CASES, HEAD_SLOPE, SLOPE, _act, _model, bf16_round, bf16_round64,
                                          check, from_words, history, in_channels, lrelu_ties, make_input, make_layer, out_shape,
                                          run_layer, sequence, to_words)

PREC_BF16 = 1
LAUNCH_TC, LAUNCH_HEAD = 0, 3
TEST_CONV, TEST_CONVTR, TEST_HEAD = 0, 2, 4
STREAM, OFFLINE, VARLEN, SLOTS = 0, 1, 2, 3

UNIFORM = (300, 1, 129)           # the uniform stream's chunks
STACKED = (5, 1, 3)               # every stacked stream's chunks
N_STACKED = 16
# slot -> the stream it replays: "u" the uniform one, j stacked stream j.  Slot calls advance six slots each, in this row order:
# slot 3 sits out the second call, slot 6 the first, slot 7 both
SLOT_SOURCE = ["u", 0, 1, 2, 3, 4, 5, 6]
SLOT_CALLS = [[3, 0, 1, 2, 4, 5], [5, 0, 6, 2, 1, 4]]
ROW_SPACES = ("uniform", "stacked", "varlen", "slots")


def varlen_lengths(P):
    """300 / 127 / 128 / 129 rows, fewer rows than P (where P > 1), and 1-row utterances, 24 of them in a row"""
    short = max(1, P // 2)
    return [300, 1, 1, 1, short, 127, 1, 128, 129] + [1] * 24 + [short, 1]


# ------------------------------------------------------------------------------------------------ data and model
def make_data(name, mode):
    """The inputs of every row space of one case: the uniform stream (state, [(x, res)]), the stacked streams, the varlen utterances"""
    spec = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 100 * mode)
    slope = (HEAD_SLOPE if spec["kind"] == 2 else SLOPE) if spec["pre"] == ACT_LRELU else None
    cx, P = in_channels(spec), history(spec)

    def chunk(T):
        x = make_input(spec, mode, 1, T, rng, cx, slope)[0]
        if spec["kind"] == 2:
            # LeakyReLU(0.01) shrinks the negative inputs a hundredfold; half of those not on a tie 2^7 times larger (still bf16 values)
            # give operands of the positive ones' size, whose rounding to bf16 (mode 2) then shows in the outputs
            m = (x < 0) & (rng.random(x.shape) < 0.5) & ~np.isin(x, lrelu_ties(HEAD_SLOPE))
            x[m] *= np.float32(128.0)
        return x, make_input(spec, mode, 1, T, rng, spec["Cout"])[0] if spec.get("res") else None

    def state():        # post-activation values, as stored
        st = make_input(spec, mode, 1, P, rng, cx, slope)
        st = _act(st, ACT_LRELU, slope) if slope is not None else st
        return (bf16_round(st) if mode == 2 else st)[0]
    return dict(u=(state(), [chunk(T) for T in UNIFORM]), s=[(state(), [chunk(T) for T in STACKED]) for _ in range(N_STACKED)],
                v=[chunk(T) for T in varlen_lengths(P)])


def model_stream(layer, mode, st, chunks):
    """Streams (B, C, P) through consecutive chunks [(x (B, C, T), res or None)] -> ([(exact, S, y)] per chunk, [state before chunk 0,
    after chunk 0, ...])"""
    spec, w, bias, mean, scale = layer
    outs, states = [], [st]
    for x, r in chunks:
        exact, S, y, st = _model(spec, mode, x, st, w, bias, r, mean, scale)
        outs.append((exact, S, y))
        states.append(st)
    return outs, states


def model_offline(layer, mode, x, r, history_rows=None):
    """One utterance (C, T) from zero history (a transposed conv: its first row replicated) -> (exact, S, y) (Cout, T').
    history_rows: read these rows (C, P) as history instead (the negative controls' wrong row maps)."""
    spec, w, bias, mean, scale = layer
    rr = None if r is None else r[None]
    if history_rows is None:
        z = np.zeros((1, in_channels(spec), history(spec)), np.float32)
        exact, S, y, _ = _model(spec, mode, x[None], z, w, bias, rr, mean, scale, offline=True)
    else:
        exact, S, y, _ = _model(spec, mode, x[None], history_rows[None], w, bias, rr, mean, scale)
    return exact[0], S[0], y[0]


def stacked_chunks(D, streams):
    """the stacked streams' chunks as batched arrays"""
    out = []
    for k in range(len(STACKED)):
        x = np.stack([D["s"][j][1][k][0] for j in streams])
        r = None if D["s"][0][1][k][1] is None else np.stack([D["s"][j][1][k][1] for j in streams])
        out.append((x, r))
    return out


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------------------ the test entry point
@contextlib.contextmanager
def stack_rows(on):
    """ADEC_STACK_ROWS for the handles created inside (read when a handle is created)"""
    old = os.environ.get("ADEC_STACK_ROWS")
    os.environ["ADEC_STACK_ROWS"] = "1" if on else "0"
    try:
        yield
    finally:
        if old is None:
            del os.environ["ADEC_STACK_ROWS"]
        else:
            os.environ["ADEC_STACK_ROWS"] = old


def op_desc(layer, mode):
    """adec_test_op of a vocoder case, as build_hifigan builds the op"""
    from audiodec_b200 import _lib
    spec, w, bias, mean, scale = layer
    p = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)
    norm = spec["pre"] == ACT_NORM
    common = dict(w=p(w), w2=None, bias=p(bias), mean=p(mean) if norm else None, scale=p(scale) if norm else None, compute_dtype=mode,
                  out_nct=0, dil=spec.get("dil", 1))
    if spec["kind"] == 0:
        return _lib.AdecTestOp(kind=TEST_CONV, Cin=spec["Cin"], Cout=spec["Cout"], K=spec["K"], stride=1, groups=spec["G"],
                               shared_in=int(spec.get("shared", False)), pre_act=spec["pre"], slope=SLOPE, post_tanh=0, **common)
    if spec["kind"] == 1:
        return _lib.AdecTestOp(kind=TEST_CONVTR, Cin=spec["Cin"], Cout=spec["Cout"], K=2 * spec["up"], stride=spec["up"], groups=1,
                               shared_in=0, pre_act=ACT_LRELU, slope=SLOPE, post_tanh=0, **common)
    return _lib.AdecTestOp(kind=TEST_HEAD, Cin=32, Cout=1, K=7, stride=1, groups=1, shared_in=0, pre_act=ACT_LRELU, slope=HEAD_SLOPE,
                           post_tanh=1, **common)


def run_op(layer, mode, call_mode, xs, res=None, states=None, streams=None, n_streams=None):
    """adec_test_conv_op with compute_dtype `mode`.  xs[k][j]: call k's utterance j (Cin_x, L), fp32 values (bf16-representable in
    mode 2); res like the outputs, or None; states (n_streams, Cin_x, P) or None; streams (n_calls, B) in call mode 3.  Returns
    (ys[k][j] (Cout, L'), the states after the calls (modes 0 and 3), the launch records)."""
    from audiodec_b200 import _lib
    lib = _lib.load()
    spec = layer[0]
    enc = to_words if mode == 2 else (lambda v: np.asarray(v, np.float32))
    dec = from_words if mode == 2 else (lambda v: v)
    flat = lambda parts: np.ascontiguousarray(enc(np.concatenate([u.ravel() for call in parts for u in call]).astype(np.float32)))
    lengths = np.ascontiguousarray([[u.shape[1] for u in call] for call in xs], np.int32)
    B = lengths.shape[1]
    x = flat(xs)
    r = None if res is None else flat(res)
    oshape = lambda L: out_shape(spec, 1, int(L))[1:]
    y = np.zeros(sum(int(np.prod(oshape(L))) for L in lengths.ravel()), np.uint16 if mode == 2 else np.float32)
    P = history(spec)
    # a copy: the library writes the new states in place, and the caller's states stay the model's inputs
    st = None if states is None or P == 0 else np.ascontiguousarray(enc(np.array(states, np.float32)))
    sl = None if streams is None else np.ascontiguousarray(streams, np.int32)
    rec = np.zeros(64 * _lib.TEST_REC, np.int32)
    d = op_desc(layer, mode)
    p = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)
    ip = lambda a: None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    rc = lib.adec_test_conv_op(0, ctypes.byref(d), call_mode, len(xs), B, n_streams or B, ip(lengths), ip(sl), p(x), p(r), p(st), p(y),
                               ip(rec), 64, None)
    assert rc == 0, _lib.last_error(None)
    yv = dec(y)
    ys, at = [], 0
    for row in lengths:
        ys.append([])
        for L in row:
            n = int(np.prod(oshape(L)))
            ys[-1].append(yv[at:at + n].reshape(oshape(L)))
            at += n
    st_out = None if st is None else dec(st).reshape(np.shape(states))
    return ys, st_out, [tuple(int(v) for v in q) for q in rec.reshape(-1, _lib.TEST_REC) if q[0] >= 0]


def slot_plan():
    """per slot call: [(slot, source, chunk index)] in row order"""
    done = [0] * len(SLOT_SOURCE)
    plan = []
    for call in SLOT_CALLS:
        plan.append([])
        for s in call:
            plan[-1].append((s, SLOT_SOURCE[s], done[s]))
            done[s] += 1
    return plan, done


def row_space_runs(layer, mode, D):
    """The four row spaces of one case, plus the uniform offline calls varlen is compared with.  Returns {row space: (ys, states,
    launch records)}."""
    src = lambda s: D["u"] if s == "u" else D["s"][s]
    rs = lambda parts: None if parts[0][0] is None else parts
    R = {}
    st_u, ch_u = D["u"]
    with stack_rows(False):
        R["uniform"] = run_op(layer, mode, STREAM, [[x] for x, _ in ch_u], rs([[r] for _, r in ch_u]), st_u[None])
    R["stacked"] = run_op(layer, mode, STREAM, [[D["s"][j][1][k][0] for j in range(N_STACKED)] for k in range(len(STACKED))],
                          rs([[D["s"][j][1][k][1] for j in range(N_STACKED)] for k in range(len(STACKED))]),
                          np.stack([D["s"][j][0] for j in range(N_STACKED)]))
    plan, _ = slot_plan()
    R["slots"] = run_op(layer, mode, SLOTS, [[src(q)[1][k][0] for _, q, k in call] for call in plan],
                        rs([[src(q)[1][k][1] for _, q, k in call] for call in plan]), np.stack([src(q)[0] for q in SLOT_SOURCE]),
                        streams=SLOT_CALLS, n_streams=len(SLOT_SOURCE))
    R["varlen"] = run_op(layer, mode, VARLEN, [[x for x, _ in D["v"]]], rs([[r for _, r in D["v"]]]))
    R["offline"] = run_op(layer, mode, OFFLINE, [[x] for x, _ in D["v"]], rs([[r] for _, r in D["v"]]))
    return R


# ------------------------------------------------------------------------------------------------ GPU tests
def _pool(parts):
    return [np.concatenate([np.ravel(p[i]) for p in parts]) for i in range(3)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", sorted(CASES))
def test_op_in_every_row_space(name, mode):
    layer = make_layer(name)
    spec = layer[0]
    P = history(spec)
    D = make_data(name, mode)
    R = row_space_runs(layer, mode, D)
    pooled = {k: [] for k in ROW_SPACES}            # (y, exact, S) per output block
    wrong = []                                      # states and cross-row-space comparisons that differ
    # uniform: the stream's three chunks and its state
    ys, st, _ = R["uniform"]
    m_u, sts_u = model_stream(layer, mode, D["u"][0][None], [(x[None], None if r is None else r[None]) for x, r in D["u"][1]])
    for k, (exact, S, _) in enumerate(m_u):
        pooled["uniform"].append((ys[k][0], exact[0], S[0]))
    if P and not same_bits(st[0], sts_u[-1][0]):
        wrong.append("uniform state")
    # stacked: 16 streams, three chunks each, their states
    ys, st, _ = R["stacked"]
    m_s, sts_s = model_stream(layer, mode, np.stack([D["s"][j][0] for j in range(N_STACKED)]), stacked_chunks(D, range(N_STACKED)))
    for k, (exact, S, _) in enumerate(m_s):
        for j in range(N_STACKED):
            pooled["stacked"].append((ys[k][j], exact[j], S[j]))
    if P and not same_bits(st, sts_s[-1]):
        wrong.append("stacked states")
    # slots: each output equals the uniform / stacked run's output of the same chunk, and each slot's state is its source stream's
    # after the chunks the slot took (an idle slot's: its initial state)
    ys, st, _ = R["slots"]
    plan, done = slot_plan()
    for c, call in enumerate(plan):
        for j, (s, q, k) in enumerate(call):
            ref_y = R["uniform"][0][k][0] if q == "u" else R["stacked"][0][k][q]
            exact, S, _ = m_u[k] if q == "u" else m_s[k]
            b = 0 if q == "u" else q
            if not same_bits(ys[c][j], ref_y):
                wrong.append(f"slot {s} call {c + 1} differs from its stream's chunk {k} in columns "
                             f"{np.flatnonzero((bits(ys[c][j]) != bits(ref_y)).any(0))[:12]}")
            pooled["slots"].append((ys[c][j], exact[b], S[b]))
    if P:
        for s, q in enumerate(SLOT_SOURCE):
            want = sts_u[done[s]][0] if q == "u" else sts_s[done[s]][q]
            if not same_bits(st[s], want):
                wrong.append(f"slot {s} state after {done[s]} chunks")
    # varlen: every utterance from zero history, equal to the uniform offline call of it alone
    ys, _, _ = R["varlen"]
    yo = R["offline"][0]
    for i, (x, r) in enumerate(D["v"]):
        exact, S, _ = model_offline(layer, mode, x, r)
        pooled["varlen"].append((ys[0][i], exact, S))
        if not same_bits(ys[0][i], yo[i][0]):
            wrong.append(f"varlen utterance {i} ({x.shape[1]} rows) differs from its offline call")
    # the launches: PREC_BF16, bf16 storage exactly in mode 2, varlen kernels in modes 2 / 3, stacked tiles for the 16 streams
    for key in ROW_SPACES:
        recs = R[key][2]
        kinds = {LAUNCH_HEAD} if spec["kind"] == 2 else {LAUNCH_TC}
        if not (recs and {q[0] for q in recs} == kinds and all(q[8] == (mode == 2) and q[5] == (key in ("varlen", "slots")) for q in recs)
                and (spec["kind"] == 2 or all(q[4] == PREC_BF16 and q[7] == (key == "stacked") for q in recs))):
            wrong.append(f"{key} launches {recs}")
    line, bad = [], []
    for key in ROW_SPACES + ("offline",):
        parts = pooled[key] if key != "offline" else [(yo[i][0], e, S) for i, (_, e, S) in enumerate(pooled["varlen"])]
        ok, stat = check(spec, mode, *_pool(parts))
        line.append(f"{key} {stat:.4g}")
        if not ok:
            bad.append(key)
    print(f"[bf16 row spaces] {name} mode {mode} ({'max |y - exact| / S' if mode == 1 else 'share on bf16_rne(exact)'}): " +
          ", ".join(line))
    assert not bad, (name, mode, "outside the model", bad, line, wrong)
    assert not wrong, (name, mode, wrong)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", sorted(CASES))
def test_entry_points_build_the_same_op(name, mode):
    """adec_test_conv_op (the op as a symAD decoder-only handle builds it) and adec_test_vocoder_layer (as a HiFi-GAN handle builds
    it) give the same output and state bits: 3 streams through chunks of 128 and 5 rows (the second stacked), and offline."""
    from audiodec_b200 import _lib
    lib = _lib.load()
    layer = make_layer(name)
    st0, chunks = sequence(name, mode, 3, (128, 5), 3)
    ys, st, _ = run_op(layer, mode, STREAM, [list(x) for x, _ in chunks], None if chunks[0][1] is None else [list(r) for _, r in chunks],
                       st0)
    st_l = st0
    for k, (x, r) in enumerate(chunks):
        y_l, st_l = run_layer(lib, layer, mode, x, st_l, r)
        for j in range(3):
            assert same_bits(ys[k][j], y_l[j]), (name, mode, f"chunk {k} stream {j}: the two entry points differ")
    if history(layer[0]):
        assert same_bits(st, st_l), (name, mode, "state: the two entry points differ")
    x, r = chunks[0]
    yo, _, _ = run_op(layer, mode, OFFLINE, [list(x)], None if r is None else [list(r)])
    y_l, _ = run_layer(lib, layer, mode, x, st0, r, offline=True)
    for j in range(3):
        assert same_bits(yo[0][j], y_l[j]), (name, mode, f"offline stream {j}: the two entry points differ")


# the ops of the bench's configs[3] shape checked there: convs1.0 at NT 128 (shared_in), a residual convs2, upsamples.3, the head
CONFIGS3_CASES = ["v1.blocks.0.convs1.0", "v1.blocks.0.convs2.1", "upsamples.3", "output_conv"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CONFIGS3_CASES)
def test_configs3_shape(name):
    """256 stacked streams, two consecutive 5-row chunks, mode 2 (the convs run more than one wave of persistent tiles, many streams per
    tile): every output against the model, every state bit for bit, and streams 0, 1, 127 and 255 bit for bit against B = 1 calls."""
    mode, n, T = 2, 256, 5
    layer = make_layer(name)
    spec = layer[0]
    P = history(spec)
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 3)
    slope = (HEAD_SLOPE if spec["kind"] == 2 else SLOPE) if spec["pre"] == ACT_LRELU else None
    st0 = bf16_round(_act(make_input(spec, mode, n, P, rng, in_channels(spec), slope), ACT_LRELU, slope))
    chunks = [(make_input(spec, mode, n, T, rng, in_channels(spec), slope),
               make_input(spec, mode, n, T, rng, spec["Cout"]) if spec.get("res") else None) for _ in range(2)]
    ys, st, recs = run_op(layer, mode, STREAM, [list(x) for x, _ in chunks], None if chunks[0][1] is None else [list(r) for _, r in chunks],
                          st0)
    m, sts = model_stream(layer, mode, st0, chunks)
    parts = [(ys[k][j], m[k][0][j], m[k][1][j]) for k in range(2) for j in range(n)]
    ok, stat = check(spec, mode, *_pool(parts))
    assert ok, (name, stat)
    if P:
        assert same_bits(st, sts[-1]), (name, "states")
    assert all(q[7] == 1 for q in recs if q[0] == LAUNCH_TC), recs
    for j in (0, 1, 127, 255):
        y1, st1, _ = run_op(layer, mode, STREAM, [[x[j]] for x, _ in chunks], None if chunks[0][1] is None else [[r[j]] for _, r in chunks],
                            st0[j:j + 1])
        for k in range(2):
            assert same_bits(ys[k][j], y1[k][0]), (name, f"stream {j} chunk {k}: 256 stacked streams differ from B = 1")
        if P:
            assert same_bits(st[j], st1[0]), (name, f"stream {j} state")
    print(f"[bf16 configs[3]] {name}: share on bf16_rne(exact) {stat:.4f}, launches {sorted(set(recs))}")


# ------------------------------------------------------------------------------------------------ bf16 instantiation coverage
def _tc_entries():
    """bf16 entries of kTcKernels (adec.cu): (NT, fuse, pre, prec, varlen, bst)"""
    out = []
    for nt in (128, 64, 32):
        for bst in (0, 1):
            for fuse, pre in ((0, ACT_NONE), (0, ACT_LRELU), (0, ACT_NORM), (1, 1), (0, 1)):
                for vl in (0, 1):
                    out.append((nt, fuse, pre, PREC_BF16, vl, bst))
    return out


def _plan_records(mode):
    """{launch record: where it was first seen} of real bf16 handles in compute_dtype `mode`: HiFi-GAN v0 / v1 / v2 and the symAD /
    symAAD / c16 decoder-only and encoder-only handles, each in a long uniform chunk, 16 stacked short streams, 256 streams of 5 frames,
    an offline varlen batch and a slot call"""
    import torch
    from audiodec_b200 import _lib
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADDecoderStreamGenerator, SymADEncoderStreamGenerator
    lib = _lib.load()
    dev = torch.device("cuda:0")
    seen = {}

    def collect(label, g, run):
        lib.adec_record_launches(g._h, 1)
        run(g)
        torch.cuda.synchronize()
        n = lib.adec_launch_records(g._h, None, 0)
        buf = np.zeros(max(n, 1) * _lib.TEST_REC, np.int32)
        lib.adec_launch_records(g._h, buf.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), n)
        lib.adec_record_launches(g._h, 0)
        for q in buf[:n * _lib.TEST_REC].reshape(-1, _lib.TEST_REC):
            seen.setdefault(tuple(int(v) for v in q), label)

    def bf16(g):
        return g.set_activation_dtype(torch.bfloat16) if mode == 2 else g.to(torch.bfloat16)

    def decoder_calls(varlen):
        def run(g):
            D = 64
            g.decode(torch.randn(1, 120, D, device=dev))
            g.decode(torch.randn(16, 2, D, device=dev))
            g.decode(torch.randn(256, 5, D, device=dev))
            varlen(g)(torch.randn(1, D, 61, device=dev), [40, 3, 1, 17])
            g.decode_streams(torch.randn(15, D, device=dev), [5, 2, 1, 7], [3, 100, 7, 255])
        return run

    torch.manual_seed(0)
    for tag, params in (("v0", S.HIFIGAN_V0_PARAMS), ("v1", S.HIFIGAN_V1_PARAMS), ("v2", S.HIFIGAN_V2_PARAMS)):
        g = HiFiGANStreamGenerator(**params)
        g.load_state_dict(S.hifigan_state_dict(params, seed=1))
        g = bf16(g).eval().to(dev)
        collect(f"HiFi-GAN {tag}", g, decoder_calls(lambda g: g.forward_varlen))
    for tag, params in (("symAD", S.SYMAD_PARAMS), ("symAAD", S.SYMAAD_PARAMS), ("c16", S.SYMAD_C16_PARAMS)):
        sd = S.symad_state_dict(params, seed=0)
        g = SymADDecoderStreamGenerator(**params)
        g.load_state_dict(sd)
        g = bf16(g).eval().to(dev)
        collect(f"{tag} decoder", g, decoder_calls(lambda g: g.decode_offline_varlen))
        hop = int(np.prod(params["enc_strides"]))
        g = SymADEncoderStreamGenerator(**params)
        g.load_state_dict(sd)
        g = bf16(g).eval().to(dev)

        def run_encoder(g):
            x = lambda *s: 0.1 * torch.randn(*s, device=dev)
            g.encode(x(1, 1, 120 * hop))
            g.encode(x(16, 1, 2 * hop))
            g.encode(x(256, 1, 5 * hop))
            g.encode_offline_varlen([x(n * hop) for n in (40, 3, 1, 17)])
            g.encode_streams([x(n * hop) for n in (5, 2, 1, 7)], [3, 100, 7, 255])
        collect(f"{tag} encoder", g, run_encoder)
    return seen


def _case_records(mode):
    """{launch record: case} of the op cases in the row spaces their tests check: this file's, the symAD decoder suite's (RUNS) and the
    symAD encoder suite's (runs(s); the stem with its tie weights, checked bit for bit against compute_dtype 0)"""
    seen = {}

    def add(label, recs):
        for q in recs:
            seen.setdefault(tuple(int(v) for v in q), label)
    for name in sorted(CASES):
        R = row_space_runs(make_layer(name), mode, make_data(name, mode))
        for key in ROW_SPACES + ("offline",):
            add(f"{name} {key}", R[key][2])
    rng = np.random.default_rng(0)
    for case in sorted(dec_suite.CASES):
        W = dec_suite.make_op(case, rng)
        for call_mode, n_streams, calls in dec_suite.RUNS:
            xs = [[dec_suite.make_x(case, L, mode, rng)[0] for _, L in call] for call in calls]
            add(f"symAD decoder {case} mode {call_mode}", dec_suite.run(case, W, mode, call_mode, n_streams, calls, xs)[1])
    for case, c in sorted(enc_suite.CASES.items()):
        w, b = enc_suite.make_op(case, rng)
        K = enc_suite.kernel_of(case)
        for call_mode, n_streams, calls in enc_suite.runs(c["s"]):
            xs = [[enc_suite.make_x(case, L, rng, mode) for _, L in call] for call in calls]
            add(f"symAD encoder {case} mode {call_mode}",
                enc_suite.run(enc_suite.CONV, c["Cin"], c["Cout"], K, c["s"], c.get("pre", ACT_NONE), int(case.startswith("projector")),
                              w, b, mode, call_mode, n_streams, calls, xs, K - 1)[1])
    name, w, b = enc_suite.stem_weights(rng)[0]
    for call_mode, n_streams, calls in enc_suite.runs(1):
        xs = [[enc_suite.stem_x(name, L, rng) for _, L in call] for call in calls]
        add(f"symAD encoder stem mode {call_mode}",
            enc_suite.run(enc_suite.STEM, 1, 32, 7, 1, ACT_NONE, 0, w, b, mode, call_mode, n_streams, calls, xs, 6)[1])
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_bf16_instantiation_coverage(mode):
    """Every launch record (kind, NT, fuse, pre, prec, varlen, paired, stacked, bst) of the released bf16 plans is produced by an op
    case in a row space its test checks, so a plan launch missing from the cases fails here.  Prints the plan's records and the bf16
    kTcKernels entries no plan selects."""
    plan, cases = _plan_records(mode), _case_records(mode)
    assert plan, "no launch recorded"
    assert all(q[4] == PREC_BF16 for q in plan if q[0] == LAUNCH_TC) and all(q[8] == (mode == 2) for q in plan), sorted(plan)
    missing = sorted(set(plan) - set(cases))
    print(f"mode {mode}: launch records of the plans (kind, NT, fuse, pre, prec, varlen, paired, stacked, bst):")
    for q in sorted(plan):
        print(f"  {q}  first in {plan[q]}; case: {cases.get(q, 'NONE')}")
    used = {(q[1], q[2], q[3], q[4], q[5], q[8]) for q in plan if q[0] == LAUNCH_TC}
    print(f"mode {mode}: bf16 kTcKernels entries (NT, fuse, pre, prec, varlen, bst) no plan selects: "
          f"{[e for e in _tc_entries() if e[5] == (mode == 2) and e not in used]}")
    assert not missing, f"mode {mode}: plan launches no checked case produces: " + "; ".join(f"{q} ({plan[q]})" for q in missing)


# ------------------------------------------------------------------------------------------------ negative controls (no GPU)
def _rejects(spec, mode, bad, good):
    """(the checker rejects the wrong outputs, the bit comparison with the right ones rejects them): bad / good [(y, exact, S)] with
    the contract's exact and S"""
    ok, _ = check(spec, mode, *_pool(bad))
    return not ok, any(not same_bits(b[0], g[0]) for b, g in zip(bad, good))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["v1.blocks.3.convs1.2", "input_conv", "v1.blocks.0.convs2.1", "output_conv"])
def test_controls_varlen_predecessor_history(name, mode):
    """A varlen utterance that reads the rows before it (its predecessors' last rows, as stored) as history instead of zeros"""
    layer = make_layer(name)
    spec = layer[0]
    P = history(spec)
    D = make_data(name, mode)
    store = bf16_round if mode == 2 else (lambda v: v)
    slope = (HEAD_SLOPE if spec["kind"] == 2 else SLOPE) if spec["pre"] == ACT_LRELU else None
    act = lambda x: _act(x[None], spec["pre"], slope, layer[3], layer[4])[0]
    prev = np.zeros((in_channels(spec), P), np.float32)
    bad, good = [], []
    for x, r in D["v"]:
        exact, S, y = model_offline(layer, mode, x, r)
        good.append((y, exact, S))
        bad.append((model_offline(layer, mode, x, r, history_rows=prev)[2], exact, S))
        prev = np.concatenate([prev, store(act(x))], 1)[:, -P:]
    assert _rejects(spec, mode, bad, good) == (True, True)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["upsamples.0", "upsamples.3"])
def test_controls_varlen_convtr_replicates_previous_row(name, mode):
    """A varlen transposed conv that replicates the previous utterance's last row instead of its own first row"""
    layer = make_layer(name)
    spec = layer[0]
    D = make_data(name, mode)
    store = bf16_round if mode == 2 else (lambda v: v)
    prev = np.zeros((spec["Cin"], 1), np.float32)
    bad, good = [], []
    for x, r in D["v"]:
        exact, S, y = model_offline(layer, mode, x, r)
        good.append((y, exact, S))
        bad.append((model_offline(layer, mode, x, r, history_rows=prev)[2], exact, S))
        prev = store(_act(x[None], ACT_LRELU, SLOPE))[0][:, -1:]
    assert _rejects(spec, mode, bad, good) == (True, True)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["v1.blocks.3.convs1.2", "upsamples.3", "v2.blocks.3.convs2.0", "output_conv"])
def test_controls_slot_reads_stale_buffer(name, mode):
    """A slot call that reads the ping-pong buffer the stream's previous call read (its state before that call): the second call's
    outputs of every slot advanced twice, and the state it leaves where the chunk is shorter than P"""
    layer = make_layer(name)
    spec = layer[0]
    D = make_data(name, mode)
    plan, _ = slot_plan()
    bad, good, state_bad = [], [], False
    for s, q, k in plan[1]:
        if k != 1:
            continue
        st0, ch = D["u"] if q == "u" else D["s"][q]
        m, sts = model_stream(layer, mode, st0[None], [(x[None], None if r is None else r[None]) for x, r in ch[:2]])
        x, r = ch[1]
        exact, S, y, st_bad = _model(spec, mode, x[None], sts[0], *layer[1:3], None if r is None else r[None], *layer[3:])
        good.append((m[1][2][0], m[1][0][0], m[1][1][0]))
        bad.append((y[0], m[1][0][0], m[1][1][0]))
        state_bad |= not same_bits(st_bad, sts[2])
    assert _rejects(spec, mode, bad, good) == (True, True)
    assert state_bad or history(spec) <= min(STACKED[1], UNIFORM[1])      # a chunk of at least P rows overwrites the whole state


def _grouped_model(layer, mode, x, hists, res):
    """A grouped conv whose group g reads history hists[g] (B, Cin_g, P): the non-shared grouped model on x repeated per group
    (shared_in) -> (exact, S, y)"""
    spec, w, bias, mean, scale = layer
    G = spec["G"]
    xx = np.concatenate([x] * G, 1) if spec.get("shared") else x
    exact, S, y, _ = _model(dict(spec, shared=False), mode, xx, np.concatenate(hists, 1), w, bias, res, mean, scale)
    return exact, S, y


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["v1.blocks.0.convs1.0", "v1.blocks.1.convs1.1"])
def test_controls_grouped_state_from_another_group(name, mode):
    """A grouped conv whose group g takes its history from another group's channels: shared_in (convs1.0, one copy of the shared
    input) read at group g's channel offset g * Cin_g as a non-shared state is laid out, which in the one-copy rows of the 16 stacked
    streams is the copy g rows later (running into the next stream's rows); a non-shared conv reading group g + 1's channels"""
    layer = make_layer(name)
    spec = layer[0]
    G, P = spec["G"], history(spec)
    D = make_data(name, mode)
    st = np.stack([D["s"][j][0] for j in range(N_STACKED)])
    x, r = stacked_chunks(D, range(N_STACKED))[0]
    exact, S, y, _ = _model(spec, mode, x, st, *layer[1:3], r, *layer[3:])
    cg = in_channels(spec) if spec.get("shared") else spec["Cin"] // G
    if spec.get("shared"):
        # the rows (stream, P, Cin_g) of every stream one after the other; group g's row p read g rows later
        rows = np.concatenate([st.transpose(0, 2, 1).reshape(-1, cg), np.zeros((G, cg), np.float32)])
        hists = [np.stack([rows[b * P + g:b * P + g + P].T for b in range(N_STACKED)]) for g in range(G)]
        assert _grouped_model(layer, mode, x, [st] * G, r)[2].shape == y.shape
        assert same_bits(_grouped_model(layer, mode, x, [st] * G, r)[2], y)      # the rewrite is the model itself
    else:
        hists = [st[:, ((g + 1) % G) * cg:((g + 1) % G + 1) * cg] for g in range(G)]
    y_bad = _grouped_model(layer, mode, x, hists, r)[2]
    assert _rejects(spec, mode, [(y_bad, exact, S)], [(y, exact, S)]) == (True, True)


@pytest.mark.parametrize("chunks", ["uniform", "varlen"])
def test_controls_head_operand_not_rounded(chunks):
    """A mode-2 head whose chunk operands are the fp32 LeakyReLU(0.01) values, not rounded to bf16 (the state rows are bf16 either way)"""
    layer = make_layer("output_conv")
    spec = layer[0]
    D = make_data("output_conv", 2)
    bad, good = [], []
    if chunks == "uniform":
        st = D["u"][0][None]
        for x, _ in D["u"][1]:
            exact, S, y, st_next = _model(spec, 2, x[None], st, *layer[1:3], None, *layer[3:])
            e1 = _model(spec, 1, x[None], st, *layer[1:3], None, *layer[3:])[0]
            good.append((y, exact, S))
            bad.append((bf16_round64(e1).astype(np.float32), exact, S))
            st = st_next
    else:
        for x, _ in D["v"]:
            exact, S, y = model_offline(layer, 2, x, None)
            good.append((y, exact, S))
            bad.append((bf16_round64(model_offline(layer, 1, x, None)[0]).astype(np.float32), exact, S))
    assert _rejects(spec, 2, bad, good) == (True, True)


def test_row_space_data_hit_ties():
    """The mode-2 data of the LeakyReLU cases hold the subnormal LeakyReLU ties and the mode-1 data exact bf16 ties (what the vocoder
    suite's inputs hold), in every row space"""
    for name in ("v1.blocks.3.convs1.2", "output_conv"):
        spec = CASES[name]
        slope = HEAD_SLOPE if spec["kind"] == 2 else SLOPE
        for mode in (1, 2):
            D = make_data(name, mode)
            for key, xs in (("uniform", [x for x, _ in D["u"][1]]), ("stacked", [x for s in D["s"] for x, _ in s[1]]),
                            ("varlen", [x for x, _ in D["v"]])):
                x = np.concatenate([v.ravel() for v in xs])
                v = (x * np.float32(slope)).astype(np.float32) if mode == 2 else x
                tie = (v.view(np.uint32) & np.uint32(0xFFFF)) == 0x8000
                assert tie.mean() > 0.02, (name, mode, key, tie.mean())
