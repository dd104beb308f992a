"""Stream state out of and into a handle (adec_get_stream_state / adec_set_stream_state, state_dict(), SessionCodecServer.detach /
attach): against the reference's own pad_buffers and resume, bit for bit across handles, row spaces and dtypes, and the rejections."""
import io
import os

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CHUNK = 1500


def _bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _eq(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(_bits(a), _bits(b)), (what, (a.float() - b.float()).abs().max().item())


# ------------------------------------------------------------------ generators
SYMAD_KINDS = {"symad": S.SYMAD_PARAMS, "symaad": S.SYMAAD_PARAMS, "c16": S.SYMAD_C16_PARAMS}
VOC_KINDS = {"v0": S.HIFIGAN_V0_PARAMS, "v1": S.HIFIGAN_V1_PARAMS, "v2": S.HIFIGAN_V2_PARAMS}
_SD = {}


def _sd(kind):
    if kind not in _SD:
        if kind in SYMAD_KINDS or kind == "symad_dec":
            _SD[kind] = S.symad_state_dict(SYMAD_KINDS.get(kind, S.SYMAD_PARAMS), seed=0)
        else:
            _SD[kind] = S.hifigan_state_dict(VOC_KINDS[kind], seed=1)
    return _SD[kind]


def make(kind, mode=0, sd=None):
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADDecoderStreamGenerator, SymADStreamGenerator
    if kind in SYMAD_KINDS:
        g = SymADStreamGenerator(**SYMAD_KINDS[kind])
    elif kind == "symad_dec":
        g = SymADDecoderStreamGenerator(**S.SYMAD_PARAMS)
    else:
        g = HiFiGANStreamGenerator(**VOC_KINDS[kind])
    g.load_state_dict(_sd(kind) if sd is None else sd)
    if mode >= 1:
        g = g.to(torch.bfloat16)
    if mode == 2:
        g = g.set_activation_dtype(torch.bfloat16)
    return g.eval().to(DEV)


def full(kind):
    return kind in SYMAD_KINDS


def zq_dim(g):
    return getattr(g, "code_dim", None) or g.in_channels


def inputs(g, kind, n, gen, frames=5):
    """one chunk per stream: samples for a full symAD handle, zq (channels-last) for a decoder"""
    if full(kind):
        hop = int(np.prod(g.enc_strides))
        return [0.1 * torch.randn(frames * hop, generator=gen).to(DEV) for _ in range(n)]
    return [torch.randn(frames, zq_dim(g), generator=gen).to(DEV) for _ in range(n)]


def uniform(g, kind, xs):
    """the uniform streaming call over every stream of the handle -> [(z, idx, y)] per stream (z, idx None for decoders)"""
    x = torch.stack(xs)
    if full(kind):
        z = g.encode(x.unsqueeze(1))
        idx = g.quantize(z)
        idx = idx.unsqueeze(1) if idx.dim() == 2 else idx
        y = g.decode(g.lookup(idx))
        return [(z[i], idx[:, i], y[i]) for i in range(len(xs))]
    y = g.decode(x)
    return [(None, None, y[i]) for i in range(len(xs))]


def slots(g, kind, xs, streams):
    if full(kind):
        z, frames = g.encode_streams(xs, streams)
        idx = g.quantize(z)
        ys = g.decode_streams(g.lookup(idx), frames, streams)
        out, o = [], 0
        for f, y in zip(frames, ys):
            out.append((z[0, :, o:o + f], idx[:, o:o + f], y))
            o += f
        return out
    frames = [x.shape[0] for x in xs]
    return [(None, None, y) for y in g.decode_streams(torch.cat(xs), frames, streams)]


def same_out(a, b, what):
    for (za, ia, ya), (zb, ib, yb) in zip(a, b):
        if za is not None:
            _eq(za, zb, what + " z")
            assert torch.equal(ia.cpu(), ib.cpu()), what + " idx"
        _eq(ya.reshape(-1), yb.reshape(-1), what + " y")


# ------------------------------------------------------------------ 1. against the reference
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_state.npz")
REF_MODELS = {"vctk_v1": ("symad", "v1"), "vctk_v0": ("symad", "v0"), "vctk_activate_sym": ("symaad", "symaad")}


def _golden():
    return np.load(GOLDEN)


def _ref_pb(g, model, who):
    """key -> (every s-th channel of the reference's pad_buffer, s, its max |v|, its fp64 sum) (make_golden_state.py)"""
    shapes = dict(zip((str(k) for k in g[f"{model}/{who}/keys"]), (str(v) for v in g[f"{model}/{who}/shapes"])))
    vals, out, o = g[f"{model}/{who}/pb_vals"], {}, 0
    for k, (st, rmax, rsum) in zip(g[f"{model}/{who}/pb_keys"], g[f"{model}/{who}/pb_stats"]):
        k = str(k)
        _, c, p = (int(v) for v in shapes[k].split(","))
        shape = (1, -(-c // int(st)), p)
        n = shape[1] * p
        out[k] = (vals[o:o + n].reshape(shape), int(st), float(rmax), float(rsum))
        o += n
    assert o == vals.size
    return out


def state_within(ours, ref_pb, tol=1e-4):
    """the step-1 checker: every pad_buffer within tol * max(1, max |ref|) of the reference's on the stored channels, and the whole
    buffer's max |v| and mean within the same bar -> worst ratio (<= 1 passes)"""
    worst = 0.0
    for k, (r, st, rmax, rsum) in ref_pb.items():
        o = ours[k].float().cpu().numpy()
        sub = o[:, ::int(st), :]
        if sub.shape != r.shape:
            return float("inf")
        bar = tol * max(1.0, float(rmax))
        worst = max(worst, float(np.abs(sub - r).max()) / bar, abs(float(np.abs(o).max()) - float(rmax)) / bar,
                    abs(float(o.astype(np.float64).sum()) - float(rsum)) / (bar * o.size))
    return worst


def _warm(tx, rx, dec):
    tx.initial_encoder(8192, DEV)
    dec.initial_decoder(rx.initial_encoder(8192, DEV))


def _run(tx, rx, dec, x):
    z = tx.encode(x)
    idx = tx.quantize(z)
    return idx, dec.decode(rx.lookup(idx))


@pytest.mark.parametrize("model", list(REF_MODELS))
def test_state_dict_against_reference(model):
    g = _golden()
    assert str(g["enc_digest"]) == S.state_dict_digest(S.symad_state_dict(seed=0))
    assert str(g["v1_digest"]) == S.state_dict_digest(S.hifigan_state_dict(seed=1))
    enc_kind, dec_kind = REF_MODELS[model]
    tx, rx, dec = make(enc_kind), make(enc_kind), make(dec_kind)
    _warm(tx, rx, dec)
    x = torch.from_numpy(g["x"]).to(DEV)
    split, n = int(g["split"]), x.shape[-1] // CHUNK
    for c in range(split):
        _run(tx, rx, dec, x[:, :, c * CHUNK:(c + 1) * CHUNK])
    torch.cuda.synchronize()
    worst = {}
    sds = {"tx": tx.state_dict(), "dec": dec.state_dict()}
    for who, sd in sds.items():
        keys = [str(k) for k in g[f"{model}/{who}/keys"]]
        shapes = [tuple(int(v) for v in str(s).split(",")) for s in g[f"{model}/{who}/shapes"]]
        assert sorted(sd.keys()) == sorted(keys), (who, set(sd) ^ set(keys))
        for k, shp in zip(keys, shapes):
            assert tuple(sd[k].shape) == shp, (who, k, tuple(sd[k].shape), shp)
        worst[who] = state_within(sd, _ref_pb(g, model, who))
        assert worst[who] <= 1.0, (model, who, worst[who])
    print(f"{model}: worst pad_buffer error / bar: tx {worst['tx']:.3g}, dec {worst['dec']:.3g}")
    # the dicts just checked against the reference's, through torch.save / torch.load, into fresh objects: chunks split.. n continue
    # the reference's stream (its own resume of its dicts is exact, make_golden_state.py)
    fresh = []
    for kind, who in ((enc_kind, "tx"), (dec_kind, "dec")):
        buf = io.BytesIO()
        torch.save({k: v.cpu() for k, v in sds[who].items()}, buf)
        buf.seek(0)
        fresh.append(make(kind, sd=torch.load(buf)))
    ftx, fdec = fresh
    idx, ys = [], []
    for c in range(split, n):
        i, y = _run(ftx, rx, fdec, x[:, :, c * CHUNK:(c + 1) * CHUNK])
        idx.append(i.cpu())
        ys.append(y.cpu())
    np.testing.assert_array_equal(torch.cat(idx, -1).numpy(), g[f"{model}/idx"])
    err = float(np.abs(torch.cat(ys, -1).numpy() - g[f"{model}/y"]).max())
    assert err <= 1e-4, (model, err)


def test_checker_rejects_wrong_exports():
    """negative controls of the step-1 checker: a state one call stale, channels-last without the transpose, and (AD v0) the head of
    the synthesized rows instead of the tail"""
    g = _golden()
    model = "vctk_v0"
    tx, rx, dec = make("symad"), make("symad"), make("v0")
    _warm(tx, rx, dec)
    x = torch.from_numpy(g["x"]).to(DEV)
    split = int(g["split"])
    stale = None
    for c in range(split):
        if c == split - 1:
            stale = dec.state_dict()
            stale = {k: v.clone() for k, v in stale.items()}
        _run(tx, rx, dec, x[:, :, c * CHUNK:(c + 1) * CHUNK])
    ref = _ref_pb(g, model, "dec")
    good = dec.state_dict()
    assert state_within(good, ref) <= 1.0
    assert state_within(stale, ref) > 1.0
    cl = {k: (v.reshape(v.shape[0], v.shape[2], v.shape[1]).transpose(1, 2) if k in ref and v.shape[1] > 1 and v.shape[2] > 1 else v)
          for k, v in good.items()}
    assert state_within(cl, ref) > 1.0
    head = dict(good)
    kbig = max(range(3), key=lambda b: S.HIFIGAN_V0_PARAMS["resblock_kernel_sizes"][b])
    for b in range(3):
        if b == kbig:
            continue
        k = f"blocks.0.blocks.{b}.convs1.0.pad_buffer"
        p = good[k].shape[2]
        head[k] = good[f"blocks.0.blocks.{kbig}.convs1.0.pad_buffer"][:, :, :p]
    assert state_within(head, ref) > 1.0


# ------------------------------------------------------------------ 2. bit-exact resume in another handle
RESUME = [("symad", 0), ("symad_dec", 0), ("symad_dec", 1), ("symad_dec", 2), ("v0", 0), ("v0", 1), ("v0", 2),
          ("v1", 0), ("v1", 1), ("v1", 2), ("v2", 0), ("v2", 1), ("v2", 2), ("symaad", 0), ("c16", 0)]


def _warm_one(g, kind, gen):
    uniform(g, kind, inputs(g, kind, 1, gen, frames=7))


@pytest.mark.parametrize("stack", ["1", "0"])
@pytest.mark.parametrize("kind,mode", RESUME)
def test_resume_uniform(kind, mode, stack, monkeypatch):
    monkeypatch.setenv("ADEC_STACK_ROWS", stack)
    gen = torch.Generator().manual_seed(11)
    a, b = make(kind, mode), make(kind, mode)
    _warm_one(a, kind, gen)
    a.set_streams(3)
    b.set_streams(5)
    for _ in range(3):
        uniform(a, kind, inputs(a, kind, 3, gen))
    uniform(b, kind, inputs(b, kind, 5, gen))                        # b's own streams hold something else
    st = a.stream_state([0, 1, 2])
    dst = [4, 0, 2]
    b.load_stream_state(dst, st, a.state_layout)
    for _ in range(2):
        xa = inputs(a, kind, 3, gen)
        xb = inputs(b, kind, 5, gen)
        for i, d in enumerate(dst):
            xb[d] = xa[i]
        oa, ob = uniform(a, kind, xa), uniform(b, kind, xb)
        same_out(oa, [ob[d] for d in dst], f"{kind} mode {mode}")
    _eq(a.stream_state([0, 1, 2]), b.stream_state(dst), f"{kind} mode {mode} next export")


@pytest.mark.parametrize("kind,mode", RESUME)
def test_resume_slots(kind, mode):
    """export while slot bits are set, and after set_streams resizes; import into other slots of a handle of another size"""
    gen = torch.Generator().manual_seed(12)
    a, b = make(kind, mode), make(kind, mode)
    _warm_one(a, kind, gen)
    _warm_one(b, kind, gen)
    a.set_streams(4)
    b.set_streams(6)
    slots(a, kind, inputs(a, kind, 4, gen), [0, 1, 2, 3])
    slots(a, kind, inputs(a, kind, 2, gen, frames=3), [1, 3])          # streams 1 and 3 now sit in the other buffer
    st = a.stream_state([3, 0, 1])
    b.load_stream_state([5, 2, 0], st)
    xa = inputs(a, kind, 3, gen, frames=4)
    same_out(slots(a, kind, xa, [3, 0, 1]), slots(b, kind, xa, [5, 2, 0]), f"{kind} mode {mode} slots")
    _eq(a.stream_state([3, 0, 1]), b.stream_state([5, 2, 0]), f"{kind} mode {mode} slots next export")
    a.set_streams(7)                                                   # resize after slot calls
    st = a.stream_state([1, 6])
    b.load_stream_state([1, 3], st)
    xa = inputs(a, kind, 2, gen, frames=2)
    same_out(slots(a, kind, xa, [1, 6]), slots(b, kind, xa, [1, 3]), f"{kind} mode {mode} after resize")


@pytest.mark.parametrize("kind,mode", [("symad", 0), ("v0", 0), ("v1", 2), ("symad_dec", 2)])
@pytest.mark.parametrize("batch", [1, 3])
def test_load_state_dict_of_state_dict(kind, mode, batch):
    gen = torch.Generator().manual_seed(13)
    a = make(kind, mode)
    _warm_one(a, kind, gen)
    a.set_streams(batch)
    for _ in range(2):
        uniform(a, kind, inputs(a, kind, batch, gen))
    sd = a.state_dict()
    for key, c, p in a.state_layout:
        assert tuple(sd[key].shape) == (batch, c, p) and sd[key].dtype == a.state_dtype, key
    b = make(kind, mode, sd={k: v.cpu() for k, v in sd.items()})
    assert b.n_streams == batch
    _eq(a.stream_state(range(batch)), b.stream_state(range(batch)), f"{kind} B={batch} loaded state")
    xa = inputs(a, kind, batch, gen)
    same_out(uniform(a, kind, xa), uniform(b, kind, xa), f"{kind} B={batch} resumed")


# ------------------------------------------------------------------ 3. export changes nothing; import leaves other streams alone
@pytest.mark.parametrize("kind,mode", [("symad", 0), ("v1", 2), ("v0", 1)])
def test_export_changes_nothing(kind, mode):
    gen = torch.Generator().manual_seed(14)
    a, b = make(kind, mode), make(kind, mode)
    for g in (a, b):
        g.set_streams(4)
    plan = [("u", None), ("s", [2, 0]), ("u", None), ("s", [1]), ("s", [3, 1, 0])]
    for what, streams in plan:
        xs = inputs(a, kind, 4 if streams is None else len(streams), gen)
        oa = uniform(a, kind, xs) if what == "u" else slots(a, kind, xs, streams)
        b.stream_state(range(4))
        b.stream_state([3])
        ob = uniform(b, kind, xs) if what == "u" else slots(b, kind, xs, streams)
        same_out(oa, ob, f"{kind} export between calls")
    _eq(a.stream_state(range(4)), b.stream_state(range(4)), "final state")
    before = b.stream_state(range(4))
    b.load_stream_state([1, 2], torch.zeros_like(before[:2]))
    after = b.stream_state(range(4))
    _eq(before[[0, 3]], after[[0, 3]], "streams an import does not name")
    assert not torch.any(after[[1, 2]].float() != 0)


# ------------------------------------------------------------------ 4. rejections and the range flag
def test_rejections():
    a = make("v1")
    a.set_streams(3)
    st = a.stream_state([0, 1])
    with pytest.raises(RuntimeError, match="listed twice"):
        a.load_stream_state([0, 0], st)
    with pytest.raises(RuntimeError, match="out of range"):
        a.load_stream_state([0, 3], st)
    with pytest.raises(RuntimeError, match="out of range"):
        a.stream_state([-1])
    with pytest.raises(ValueError):
        a.load_stream_state([0], st)                                   # wrong shape: two rows for one stream
    with pytest.raises(RuntimeError, match="move it"):
        a.load_stream_state([0, 1], st.cpu())
    with pytest.raises(ValueError):
        a.load_stream_state([0, 1], st.to(torch.bfloat16))             # dtype
    b = make("v1", 2)
    with pytest.raises(ValueError):
        b.load_stream_state([0], a.stream_state([0]).to(torch.bfloat16)[:, :-1])
    b.load_stream_state([0], a.stream_state([0]).to(torch.bfloat16), a.state_layout)   # same layout, bf16 words: accepted
    c = make("v0")
    with pytest.raises(ValueError, match="layout"):
        c.load_stream_state([0], a.stream_state([0]), a.state_layout)
    d = make("symad_dec")
    assert all(not k.startswith(("encoder.", "projector.")) for k, _, _ in d.state_layout)
    sd = make("symad").state_dict()
    assert all(k in sd for k, _, _ in d.state_layout)


@pytest.mark.parametrize("engine,flag", [("f16", True), ("tf32", False)])
def test_import_sets_range_flag(engine, flag, monkeypatch):
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    g = make("v1")
    g.set_streams(2)
    assert not g.range_error()
    st = g.stream_state([1])
    g.load_stream_state([1], st)
    assert not g.range_error()
    st[0, st.shape[1] // 2] = 6e4
    g.load_stream_state([1], st)
    assert g.range_error() == flag


def test_state_elems_match_design():
    """bytes per stream: 41,510 encoder + 1,024 projector values for symAD's encoder half, 174,336 for the v1 decoder"""
    sym, voc = make("symad"), make("v1")
    enc = sum(c * p for k, c, p in sym.state_layout if k.startswith("encoder."))
    proj = sum(c * p for k, c, p in sym.state_layout if k.startswith("projector."))
    assert (enc, proj) == (41510, 1024)
    assert sum(c * p for _, c, p in voc.state_layout) == 174336
    assert voc.stream_state([0]).shape == (1, 174336)


# ------------------------------------------------------------------ 5. the session server
def _codec(dev, mode=2):
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    sd_e, sd_d = _sd("symad"), _sd("v1")
    tx, rx = (SymADStreamGenerator(**S.SYMAD_PARAMS) for _ in range(2))
    for g in (tx, rx):
        g.load_state_dict(sd_e)
        g.eval().to(dev)
    dec = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    dec.load_state_dict(sd_d)
    dec = dec.to(torch.bfloat16).set_activation_dtype(torch.bfloat16).eval().to(dev)
    tx.initial_encoder(8192, dev)
    dec.initial_decoder(rx.initial_encoder(8192, dev))
    return tx, rx, dec


def _server(dev, wire):
    from audiodec_b200.server import SessionCodecServer
    return SessionCodecServer(*_codec(dev), capacity=8, frame_size=1500, sample_rate=24000, max_latency=10.0, device=dev, wire=wire)


def _migrate(dev_b, wire):
    src, ref, dst = _server(DEV, wire), _server(DEV, wire), _server(dev_b, wire)
    rng = np.random.default_rng(5)
    sess = [src.open() for _ in range(3)]
    assert [ref.open() for _ in range(3)] == sess
    dst.open()                                            # the destination already serves someone
    frames = {s: [(0.1 * rng.standard_normal(1500)).astype(np.float32) for _ in range(8)] for s in sess}
    got = {s: [] for s in sess}
    want = {s: [] for s in sess}
    mover, moved_to = sess[1], None
    for k in range(8):
        for s in sess:
            if k == 4:
                break                                     # submitted before the detach
            if s == mover and moved_to is not None:
                dst.submit(moved_to, frames[s][k], t_capture=float(k))
            else:
                src.submit(s, frames[s][k], t_capture=float(k))
            ref.submit(s, frames[s][k], t_capture=float(k))
        if k == 3:                                        # one frame decoded and not yet polled, one queued: both must travel
            src.step()
            ref.step()
            for s in sess:
                src.submit(s, frames[s][4], t_capture=4.0)
                ref.submit(s, frames[s][4], t_capture=4.0)
            state = src.detach(mover)
            assert len(state.outputs) == 1 and len(state.inputs) == 1
            moved_to = dst.attach(state.to(dev_b))
            assert dst.statistics()["per_stream"][moved_to]["n_frames"] == 0
            assert dst.pending(moved_to) == 1
            continue
        src.step()
        ref.step()
        dst.step()
        for s in sess:
            y = dst.poll(moved_to) if s == mover and moved_to is not None else src.poll(s)
            if y is not None:
                got[s].append(y)
            y = ref.poll(s)
            if y is not None:
                want[s].append(y)
    for s in sess:                                        # drain what the servers still hold
        while (y := (dst.poll(moved_to) if s == mover else src.poll(s))) is not None:
            got[s].append(y)
        while (y := ref.poll(s)) is not None:
            want[s].append(y)
    for s in sess:
        assert len(got[s]) == len(want[s]) == 8, (s, len(got[s]), len(want[s]))
        for a, b in zip(got[s], want[s]):
            assert np.array_equal(a.view(np.int32), b.view(np.int32)), s
    with pytest.raises(KeyError):
        src.detach(mover)
    state = dst.detach(moved_to)
    while len(src.open_streams) < 8:
        src.open()
    with pytest.raises(RuntimeError, match="full"):
        src.attach(state.to(DEV))


@pytest.mark.parametrize("wire", [False, True])
def test_session_migrates_between_servers(wire):
    _migrate(DEV, wire)


def test_session_migrates_across_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    _migrate(torch.device("cuda:1"), True)
