"""Graphed streaming steps (TransmitterGraph / ReceiverGraph, adec_graph_*): a graph launch is the eager call sequence it replaces, bit
for bit - indices or packed bytes, waveforms, the causal state left behind, the range and index flags and launch_count - whatever
happens on the same handles between launches.  Every case runs two codec sets built from the same synthetic weights, one eager and
one graphed."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ENC = {"symad": S.SYMAD_PARAMS, "symaad": S.SYMAAD_PARAMS, "c16": S.SYMAD_C16_PARAMS}
VOC = {"v0": S.HIFIGAN_V0_PARAMS, "v1": S.HIFIGAN_V1_PARAMS, "v2": S.HIFIGAN_V2_PARAMS}
# name -> (encoder kind, decoder kind, decoder mode)
MODELS = {
    "vctk_sym": ("symad", "symad", 0),
    "libritts_v1": ("symad", "v1", 0),
    "vctk_v0": ("symad", "v0", 0),
    "vctk_v2": ("symad", "v2", 0),
    "vctk_activate_sym": ("symaad", "symaad", 0),
    "vctk_c16h320_sym": ("c16", "c16", 0),
    "symad_dec_mode0": ("symad", "symad_dec", 0),
    "symad_dec_mode1": ("symad", "symad_dec", 1),
    "symad_dec_mode2": ("symad", "symad_dec", 2),
    "v1_mode1": ("symad", "v1", 1),
    "v1_mode2": ("symad", "v1", 2),
}
_SD = {}


def _sd(kind):
    if kind not in _SD:
        _SD[kind] = S.hifigan_state_dict(VOC[kind], seed=1) if kind in VOC else S.symad_state_dict(ENC.get(kind, S.SYMAD_PARAMS), seed=0)
    return _SD[kind]


def make(kind, mode=0):
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADDecoderStreamGenerator, SymADStreamGenerator
    if kind in ENC:
        g = SymADStreamGenerator(**ENC[kind])
    elif kind == "symad_dec":
        g = SymADDecoderStreamGenerator(**S.SYMAD_PARAMS)
    else:
        g = HiFiGANStreamGenerator(**VOC[kind])
    g.load_state_dict(_sd(kind))
    if mode >= 1:
        g = g.to(torch.bfloat16)
    if mode == 2:
        g = g.set_activation_dtype(torch.bfloat16)
    return g.eval().to(DEV)


def codec_set(model):
    enc, dec, mode = MODELS[model]
    return make(enc), make(enc), make(dec, mode)


def chunk_of(model):
    return 5 * int(np.prod(ENC[MODELS[model][0]]["enc_strides"]))


def _bits(t):
    t = t.detach().contiguous()
    if t.dtype in (torch.int64, torch.uint8):
        return t.cpu()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _eq(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(_bits(a), _bits(b)), what


def eager_step(tx, rx, dec, x, wire):
    z = tx.encode(x)
    if wire:
        _, out, _ = tx.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)
        zq = rx.lookup_packed(out)
    else:
        out = tx.quantize(z)
        zq = rx.lookup(out)
    return out, dec.decode(zq)


class Graphed:
    """A codec set driven through its graphs (rebuilt when B or the chunk changes)."""

    def __init__(self, tx, rx, dec):
        self.tx, self.rx, self.dec = tx, rx, dec
        self.key = None

    def step(self, x, wire):
        from audiodec_b200.codec import ReceiverGraph, TransmitterGraph
        key = (x.shape[0], x.shape[-1], wire)
        if key != self.key:
            f = self.tx._lib.adec_frames_for(self.tx._h, x.shape[-1])
            self.txg = TransmitterGraph(self.tx, x.shape[0], x.shape[-1], wire=wire)
            self.rxg = ReceiverGraph(self.rx, self.dec, x.shape[0], f, wire=wire)
            self.key = key
        out = self.txg(x).clone()
        return out, self.rxg(out).clone()


def check_state(a, b, what):
    for ga, gb, name in ((a[0], b[0], "tx"), (a[2], b[2], "decoder")):
        n = ga.n_streams
        assert gb.n_streams == n, what
        _eq(ga.stream_state(range(n)), gb.stream_state(range(n)), f"{what}: {name} state")
        assert ga.launch_count == gb.launch_count, (what, name, ga.launch_count, gb.launch_count)
    assert a[1].launch_count == b[1].launch_count, (what, "rx")


def run_pair(eager, graphed, x, wire, what):
    oe, ye = eager_step(*eager, x, wire)
    og, yg = graphed.step(x, wire)
    _eq(oe, og, f"{what}: indices / packed")
    _eq(ye, yg, f"{what}: waveform")


# ------------------------------------------------------------------ 1. equality matrix
@pytest.mark.parametrize("model", list(MODELS))
def test_graph_equals_eager(model):
    eager, gset = codec_set(model), codec_set(model)
    graphed = Graphed(*gset)
    gen = torch.Generator().manual_seed(11)
    T = chunk_of(model)
    combos = [(1, False), (1, True), (3, False), (3, True)] + ([(48, False), (48, True)] if model == "vctk_sym" else [])
    for B, wire in combos:
        for c in range(8):
            x = (0.1 * torch.randn(B, 1, T, generator=gen)).to(DEV)
            run_pair(eager, graphed, x, wire, f"{model} B={B} wire={wire} chunk {c}")
        check_state(eager, gset, f"{model} B={B} wire={wire}")
    if model == "vctk_sym":
        from audiodec_b200.codec import _lib
        lib = _lib.load()
        rec = ctypes_records(lib, gset[0], lambda: gset[0].encode((0.1 * torch.randn(48, 1, T, generator=gen)).to(DEV)))
        assert any(r[7] for r in rec), "B = 48 must stack rows in the uniform calls"


def ctypes_records(lib, g, fn):
    import ctypes
    lib.adec_record_launches(g._h, 1)
    fn()
    torch.cuda.synchronize()
    n = lib.adec_launch_records(g._h, None, 0)
    buf = (ctypes.c_int * (9 * max(n, 1)))()
    lib.adec_launch_records(g._h, buf, n)
    lib.adec_record_launches(g._h, 0)
    return [list(buf[9 * i:9 * i + 9]) for i in range(n)]


# ------------------------------------------------------------------ 2. interleaving graph and eager steps
def test_interleaved_with_eager():
    eager, gset = codec_set("libritts_v1"), codec_set("libritts_v1")
    graphed = Graphed(*gset)
    gen = torch.Generator().manual_seed(12)
    pattern = "GEGGEGGGEG"
    inst = []
    for c, p in enumerate(pattern):
        x = (0.1 * torch.randn(2, 1, 1500, generator=gen)).to(DEV)
        oe, ye = eager_step(*eager, x, False)
        og, yg = graphed.step(x, False) if p == "G" else eager_step(*gset, x, False)
        _eq(oe, og, f"chunk {c}")
        _eq(ye, yg, f"chunk {c}")
        inst.append((graphed.txg.info()["instantiations"], graphed.rxg.info()["instantiations"]))
    check_state(eager, gset, "interleaved")
    # G at parity 0 (creation), E, G at parity 0 again, G at parity 1 (second executable, built once), then only reuse
    assert inst[0] == (1, 1) and inst[3] == (2, 2) and inst[-1] == (2, 2), inst


# ------------------------------------------------------------------ 3. invalidation
def _both(eager, gset, fn):
    fn(eager)
    fn(gset)


def test_invalidation():
    eager, gset = codec_set("symad_dec_mode2"), codec_set("symad_dec_mode2")
    graphed = Graphed(*gset)
    gen = torch.Generator().manual_seed(13)
    B = 3

    def step(what):
        """two graphed steps (one at each state parity) against the eager twin -> instantiations of (tx graph, rx graph)"""
        for k in range(2):
            x = (0.1 * torch.randn(B, 1, 1500, generator=gen)).to(DEV)
            run_pair(eager, graphed, x, False, f"{what} ({k})")
        check_state(eager, gset, what)
        return graphed.txg.info()["instantiations"], graphed.rxg.info()["instantiations"]

    base = step("first")
    assert base == (2, 2)

    def resize(s):
        for g in (s[0], s[2]):
            g.set_streams(8)
            g.set_streams(B)
    _both(eager, gset, resize)
    after = step("set_streams(8) and back")
    assert after == (4, 4), "growing the state buffers re-captures both graphs at both parities"

    def longer(s):
        eager_step(*s, (0.1 * torch.randn(B, 1, 4 * 1500, generator=torch.Generator().manual_seed(5))).to(DEV), False)
    _both(eager, gset, longer)
    base, after = after, step("workspace growth")
    assert after == (6, 6), "a grown workspace re-captures"

    def load_state(s):
        for g in (s[0], s[2]):
            g.load_stream_state([1], g.stream_state([0]))
    _both(eager, gset, load_state)
    base, after = after, step("load_stream_state")
    assert after == base, "an import moves no pointer: no re-capture"

    _both(eager, gset, lambda s: [g.copy_stream_state(2, [0]) for g in (s[0], s[2])])
    step("copy_stream_state")

    def slots(s):
        tx, rx, dec = s
        z, frames = tx.encode_streams([(0.1 * torch.randn(1500, generator=torch.Generator().manual_seed(6))).to(DEV)], [1])
        zq = rx.lookup(tx.quantize(z))
        dec.decode_streams(zq, frames, [1])
    _both(eager, gset, slots)
    step("encode_streams / decode_streams (dirty slot bits)")

    _both(eager, gset, lambda s: [g.reset_buffer() for g in s])
    step("reset_buffer")


# ------------------------------------------------------------------ 4. creation changes nothing
def test_creation_is_free():
    from audiodec_b200.codec import ReceiverGraph, TransmitterGraph
    eager, gset = codec_set("vctk_sym"), codec_set("vctk_sym")
    gen = torch.Generator().manual_seed(14)
    x0 = (0.1 * torch.randn(3, 1, 1500, generator=gen)).to(DEV)
    eager_step(*eager, x0, False), eager_step(*gset, x0, False)
    txg = TransmitterGraph(gset[0], 3, 1500)
    rxg = ReceiverGraph(gset[1], gset[2], 3, 5, wire=True)
    check_state(eager, gset, "after creation")
    for c in range(3):
        x = (0.1 * torch.randn(3, 1, 1500, generator=gen)).to(DEV)
        oe, ye = eager_step(*eager, x, False)
        og, yg = eager_step(*gset, x, False)
        _eq(oe, og, "idx"), _eq(ye, yg, "y")
    check_state(eager, gset, "eager calls after creation")
    del txg, rxg


# ------------------------------------------------------------------ 5. flags and counters
def test_flags_and_counters():
    eager, gset = codec_set("vctk_sym"), codec_set("vctk_sym")
    graphed = Graphed(*gset)
    gen = torch.Generator().manual_seed(15)
    x = (0.1 * torch.randn(2, 1, 1500, generator=gen)).to(DEV)
    l0 = [g.launch_count for g in eager]
    run_pair(eager, graphed, x, False, "first")
    per = [g.launch_count - l for g, l in zip(eager, l0)]
    assert graphed.txg.info()["kernels"] == per[0]
    assert graphed.rxg.info()["kernels"] == per[1] + per[2]
    assert graphed.txg.info()["programmatic_edges"] > 0 and graphed.rxg.info()["programmatic_edges"] > 0
    for k in range(3):
        run_pair(eager, graphed, (0.1 * torch.randn(2, 1, 1500, generator=gen)).to(DEV), False, f"chunk {k}")
    check_state(eager, gset, "launch counts")
    assert not eager[0].range_error() and not gset[0].range_error()
    # past the fp16-split range: the projector weight scaled by 1e7 drives z beyond 6e4 (the recipe test_range_flag_public_api uses)
    from audiodec_b200.codec import SymADStreamGenerator
    loud = {k: v.clone() for k, v in _sd("symad").items()}
    loud["projector.project.conv.weight"] = loud["projector.project.conv.weight"] * 1e7
    sets = []
    for _ in range(2):
        tx = SymADStreamGenerator(**S.SYMAD_PARAMS)
        tx.load_state_dict(loud)
        sets.append((tx.eval().to(DEV), make("symad"), make("symad")))
    g2 = Graphed(*sets[1])
    x = (0.1 * torch.randn(1, 1, 1500, generator=gen)).to(DEV)
    run_pair(sets[0], g2, x, False, "loud step")
    flags = (sets[0][0].range_error(), sets[1][0].range_error())
    assert flags == (True, True), ("a replay past the fp16-split range sets the flag as eager does", flags)
    assert (sets[0][0].range_error(), sets[1][0].range_error()) == (False, False), "reported once"
    bad = graphed.txg.output.clone()
    bad[0, 0, 0] = 10 ** 6
    eager[1].lookup(bad)
    graphed.rxg(bad)
    assert eager[1].index_error() and gset[1].index_error()
    assert not gset[1].index_error()


def test_programmatic_edges_off_without_pdl():
    code = ("from audiodec_b200 import synthetic as S; from audiodec_b200.codec import SymADStreamGenerator, TransmitterGraph; "
            "g = SymADStreamGenerator(**S.SYMAD_PARAMS); g.load_state_dict(S.symad_state_dict(seed=0)); g = g.eval().to('cuda:0'); "
            "print('EDGES', TransmitterGraph(g, 1, 1500).info()['programmatic_edges'])")
    env = dict(os.environ, ADEC_PDL="0")
    out = subprocess.run([sys.executable, "-c", code], cwd=REPO, env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "EDGES 0" in out.stdout, out.stdout


# ------------------------------------------------------------------ 6. eager fallback while profiling
def test_profile_runs_eager():
    """Profiling and launch records on while the graphs are created and launched: the capture leaves no event or record behind, and
    every launch runs eagerly, so the reports list exactly the launches that ran."""
    from audiodec_b200 import _lib
    eager, gset = codec_set("libritts_v1"), codec_set("libritts_v1")
    graphed = Graphed(*gset)
    gen = torch.Generator().manual_seed(16)
    lib = _lib.load()
    gset[2].profile(True)
    lib.adec_record_launches(gset[2]._h, 1)
    l0 = gset[2].launch_count
    for k in range(2):
        run_pair(eager, graphed, (0.1 * torch.randn(2, 1, 1500, generator=gen)).to(DEV), False, f"profiled {k}")
    n = gset[2].launch_count - l0
    rows = gset[2].profile_report()
    recs = lib.adec_launch_records(gset[2]._h, None, 0)
    lib.adec_record_launches(gset[2]._h, 0)
    gset[2].profile(False)
    assert len(rows) == n > 0, "every launch of the profiled steps is in the report, and nothing else"
    assert recs == n, "launch records list exactly the launches that ran"
    check_state(eager, gset, "profiled")
    run_pair(eager, graphed, (0.1 * torch.randn(2, 1, 1500, generator=gen)).to(DEV), False, "after profiling")
    check_state(eager, gset, "after profiling")


# ------------------------------------------------------------------ 7. bf16 lookup
def _bf16_cases():
    from oracle import rvq_cases as C
    return [build() for build in C.all_cases().values()]


@pytest.mark.parametrize("B", [1, 3])
def test_lookup_bf16(B):
    from audiodec_b200.codec import SymADStreamGenerator
    gen = torch.Generator().manual_seed(17)
    for case in _bf16_cases():
        g = SymADStreamGenerator(**case.params)
        g.load_state_dict(case.state_dict())
        g = g.eval().to(DEV)
        F = case.frames.shape[0] // B
        idx = g.quantize(torch.from_numpy(case.z(B, F)).to(DEV))
        nq, n = case.params["codebook_num"], case.params["codebook_size"]
        rnd = torch.randint(0, n, (nq, B, F), generator=gen) + n * torch.arange(nq).view(nq, 1, 1)
        rnd = rnd.squeeze(1) if B == 1 else rnd
        for what, i in (("rvq", idx), ("random", rnd.to(DEV))):
            ref = g.lookup(i).to(torch.bfloat16)
            _eq(g.lookup(i, dtype=torch.bfloat16), ref, f"{case.name} {what} indices")
            _eq(g.lookup_packed(g.pack(i), dtype=torch.bfloat16), ref, f"{case.name} {what} packed")


# ------------------------------------------------------------------ 8. callers
@pytest.mark.parametrize("wire", [False, True])
def test_server_lock_step(wire):
    from audiodec_b200.server import MultiStreamCodecServer
    rng = np.random.default_rng(3)
    frames = (0.1 * rng.standard_normal((6, 8, 1500))).astype(np.float32)
    kw = dict(n_streams=8, frame_size=1500, sample_rate=24000, max_latency=1.0, device=DEV, wire=wire)
    ref_srv = MultiStreamCodecServer(*codec_set("libritts_v1"), **kw)       # the eager call sequence of the same server
    ref = []
    for k in range(6):
        with torch.no_grad():
            y = ref_srv._eager_pass(torch.from_numpy(frames[k]).view(8, 1, 1500), DEV, None)
        ref.append(y.float().cpu().numpy().reshape(8, -1)[:, :1500])
    srv = MultiStreamCodecServer(*codec_set("libritts_v1"), **kw)
    got = []
    for k in range(6):
        for s in range(8):
            srv.submit(s, frames[k, s])
        assert srv.step() == 8
        got.append(np.stack([srv.poll(s) for s in range(8)]))
    assert srv._graphs is not None, "the lock-step server runs graphs on library generators"
    assert np.array_equal(np.stack(ref), np.stack(got))
    assert srv.wire_bytes == ref_srv.wire_bytes


def test_streamer_process_frames():
    import time
    from audiodec_b200.utils.audiodec import AudioDecStreamer
    rng = np.random.default_rng(4)
    frames = [(0.1 * rng.standard_normal((1500, 1))).astype(np.float32) for _ in range(12)]
    tx, rx, dec = codec_set("vctk_sym")
    st = AudioDecStreamer(0, 0, frame_size=1500, max_latency=1e9, tx_encoder=tx, tx_device=DEV, rx_encoder=rx, decoder=dec, rx_device=DEV)
    outs = st.process_frames(frames)
    got = [o for o in outs if np.any(o)]       # frames _process took from output_queue (silence until the pipeline has filled)
    t0 = time.time()
    while len(got) < len(frames) and time.time() - t0 < 120:
        try:
            y = st.output_queue.get(timeout=1)
        except Exception:
            continue
        got.append(y.squeeze(0).detach().cpu().transpose(1, 0).contiguous().numpy())
    assert st._tx_graph is not None and st._rx_graph is not None
    assert st._tx_graph.info()["instantiations"] == 2 and st._rx_graph.info()["instantiations"] == 2, "both parities launched"
    etx, erx, edec = codec_set("vctk_sym")             # the eager twin
    ref = []
    with torch.no_grad():
        for f in frames:
            x = torch.from_numpy(f).transpose(1, 0).contiguous().unsqueeze(0).to(DEV)
            ref.append(edec.decode(erx.lookup(etx.quantize(etx.encode(x)))).squeeze(0).cpu().transpose(1, 0).contiguous().numpy())
    assert len(got) == len(ref)
    for i, (o, r) in enumerate(zip(got, ref)):
        assert np.array_equal(o, r), i


# ------------------------------------------------------------------ 9. refusals
def test_refusals():
    from audiodec_b200.codec import ReceiverGraph, TransmitterGraph
    tx, rx, dec = codec_set("symad_dec_mode0")
    with pytest.raises(TypeError, match="SymADStreamGenerator"):
        TransmitterGraph(dec, 1, 1500)
    from audiodec_b200 import _lib
    import ctypes
    lib = _lib.load()
    g = ctypes.c_void_p()
    buf = torch.zeros(1 << 16, device=DEV)
    assert lib.adec_graph_create(_lib.GRAPH_TX, dec._h, None, 1, 1500, 0, ctypes.c_void_p(buf.data_ptr()),
                                 ctypes.c_void_p(buf.data_ptr()), ctypes.byref(g)) != 0
    assert "decoder-only" in _lib.last_error(dec._h)
    txg = TransmitterGraph(tx, 2, 1500)
    with pytest.raises(RuntimeError, match="expected input of shape"):
        txg(torch.zeros(2, 1, 1200, device=DEV))
    rxg = ReceiverGraph(rx, dec, 2, 5)
    tx._h = None
    tx.to(DEV)
    with pytest.raises(RuntimeError, match="replaced"):
        txg(txg.input)
    rxg(rxg.input)


def test_handles_on_two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs: the refusal of handles on different devices is unverified on one")
    from audiodec_b200.codec import ReceiverGraph, SymADStreamGenerator
    rx = make("symad")
    d = SymADStreamGenerator(**S.SYMAD_PARAMS)
    d.load_state_dict(_sd("symad"))
    d = d.eval().to(torch.device("cuda:1"))
    with pytest.raises(RuntimeError, match="device"):
        ReceiverGraph(rx, d, 1, 5)
