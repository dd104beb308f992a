"""Stream slots (adec_encode_streams / adec_decode_streams[_bf16] / adec_copy_stream_state) and SessionCodecServer: any subset of a
handle's streams advances by chunks of its own lengths in one launch sequence, and every stream must come out exactly as a B = 1
streaming handle fed that stream's chunks alone."""
import ctypes
import os

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WAVE_TOL = 1e-4
HOP = 300


def _bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _symad(sd):
    from audiodec_b200.codec import SymADStreamGenerator
    g = SymADStreamGenerator(**S.SYMAD_PARAMS)
    g.load_state_dict(sd)
    return g.eval().to(DEV)


def _voc(sd, mode):
    from audiodec_b200.codec import HiFiGANStreamGenerator
    d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    d.load_state_dict(sd)
    if mode >= 1:
        d = d.to(torch.bfloat16)
    if mode == 2:
        d = d.set_activation_dtype(torch.bfloat16)
    return d.eval().to(DEV)


class Codec:
    """tx / rx / decoder warmed like AudioDec.load_transmitter / load_receiver (bin/stream.py:56-77); warm() again after a reset gives
    the same state."""

    def __init__(self, symad_sd, voc_sd=None, mode=0):
        self.tx, self.rx = _symad(symad_sd), _symad(symad_sd)
        self.dec = _symad(symad_sd) if voc_sd is None else _voc(voc_sd, mode)
        self.warm()

    def warm(self):
        for g in (self.tx, self.rx, self.dec):
            g.reset_buffer()
        self.tx.initial_encoder(8192, DEV)
        self.dec.initial_decoder(self.rx.initial_encoder(8192, DEV))

    def set_streams(self, n):
        for g in (self.tx, self.dec):
            g.set_streams(n)

    def uniform(self, x):
        """(B, T) chunks, one per stream of the handle -> z, idx, y per the uniform calls"""
        z = self.tx.encode(x.view(x.shape[0], 1, -1))
        idx = self.tx.quantize(z)
        if idx.dim() == 2:
            idx = idx.unsqueeze(1)
        y = self.dec.decode(self.rx.lookup(idx))
        return z, idx, y

    def slots(self, chunks, streams):
        z, frames = self.tx.encode_streams(chunks, streams)
        idx = self.tx.quantize(z)                                   # (Nq, sum F): B = 1 layout
        ys = self.dec.decode_streams(self.rx.lookup(idx), frames, streams)
        out, o = [], 0
        for f, y in zip(frames, ys):
            out.append((z[:, :, o:o + f], idx[:, o:o + f], y))
            o += f
        return out


def _replay(ref, chunks):
    """a B = 1 handle, warmed, fed `chunks` in order -> [(z, idx, y)] per chunk"""
    ref.set_streams(1)
    ref.warm()
    out = []
    for x in chunks:
        z, idx, y = ref.uniform(x.view(1, -1))
        out.append((z, idx[:, 0], y))
    return out


def _same(got, want, what):
    for (z, i, y), (z1, i1, y1) in zip(got, want):
        assert torch.equal(_bits(z), _bits(z1)), what
        assert torch.equal(i.cpu(), i1.cpu()), what
        assert y.dtype == y1.dtype and y.numel() == y1.numel(), what
        assert torch.equal(_bits(y.reshape(-1)), _bits(y1.reshape(-1))), (what, (y.float() - y1.float()).abs().max().item())


def _codec_pair(symad_sd, hifigan_sd, dec_kind):
    voc, mode = (None, 0) if dec_kind == "symad" else (hifigan_sd, int(dec_kind[-1]))
    return Codec(symad_sd, voc, mode), Codec(symad_sd, voc, mode)


# ------------------------------------------------------------------ 1. random schedule, bit for bit against B = 1 handles
CASES = [("f16", "symad"), ("tf32", "symad"), ("f16", "v1_mode0"), ("f16", "v1_mode1"), ("f16", "v1_mode2")]


@pytest.mark.parametrize("engine,dec_kind", CASES)
def test_random_schedule_bit_exact(symad_sd, hifigan_sd, engine, dec_kind, monkeypatch):
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    cap, steps = 8, 12
    c, ref = _codec_pair(symad_sd, hifigan_sd, dec_kind)
    c.set_streams(cap)
    rng = np.random.default_rng(7)
    fed = {s: [] for s in range(cap)}
    got = {s: [] for s in range(cap)}
    for k in range(steps):
        n = 1 if k == 2 else cap if k in (0, 5) else int(rng.integers(1, cap + 1))
        streams = [int(s) for s in rng.permutation(cap)[:n]]
        lens = [int(rng.integers(1, 6)) * HOP for _ in streams]
        if k in (3, 8):
            lens[0] += int(rng.integers(1, HOP))                  # lengths that are not multiples of the hop
        chunks = [0.1 * torch.randn(t, device=DEV) for t in lens]
        for s, x, o in zip(streams, chunks, c.slots(chunks, streams)):
            fed[s].append(x)
            got[s].append(o)
    torch.cuda.synchronize()
    for s in range(cap):
        _same(got[s], _replay(ref, fed[s]), (engine, dec_kind, s))


# ------------------------------------------------------------------ 2. the reference's golden stream through slot calls
@pytest.mark.parametrize("engine", ["f16", "tf32"])
def test_golden_stream_through_slots(golden_dir, symad_sd, engine, monkeypatch):
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    g = np.load(os.path.join(golden_dir, "symad_stream.npz"))
    c = Codec(symad_sd)
    c.set_streams(4)
    x = torch.from_numpy(g["x"]).to(DEV).view(-1)
    n = int(g["chunk"])
    idx, ys = [], []
    for k, i in enumerate(range(0, x.numel(), n)):
        others = [s for s in (0, 1, 3) if (k + s) % 2 == 0]        # other streams of other lengths, in and out
        streams = others[:1] + [2] + others[1:]
        chunks = [0.1 * torch.randn(HOP * (1 + s) + 7 * s, device=DEV) if s != 2 else x[i:i + n] for s in streams]
        out = c.slots(chunks, streams)[streams.index(2)]
        idx.append(out[1].cpu())
        ys.append(out[2].reshape(-1).cpu())
    np.testing.assert_array_equal(torch.cat(idx, -1).numpy(), g["idx"].reshape(g["idx"].shape[0], -1))
    np.testing.assert_allclose(torch.cat(ys).numpy(), g["y"].reshape(-1), atol=WAVE_TOL)


# ------------------------------------------------------------------ 3. idle means untouched; 4. join without bleed
def test_idle_stream_is_untouched(symad_sd):
    a, b = Codec(symad_sd), Codec(symad_sd)
    a.set_streams(4)
    b.set_streams(4)
    torch.manual_seed(3)
    xs = [0.1 * torch.randn(1500, device=DEV) for _ in range(6)]
    got_a, got_b = [], []
    for k in range(9):
        others = [1, 2, 3]
        if k in (3, 4, 5):                                          # stream 0 absent for three steps in `a`
            a.slots([torch.randn(900, device=DEV) * 0.1 for _ in others], others)
        else:
            j = k if k < 3 else k - 3
            got_a.append(a.slots([xs[j]] + [torch.randn(600, device=DEV) * 0.1 for _ in others], [0] + others)[0])
    for j in range(6):
        got_b.append(b.slots([xs[j]], [0])[0])
    _same(got_a, got_b, "gap")


def test_join_without_bleed(symad_sd, hifigan_sd):
    for dec_kind in ("symad", "v1_mode2"):
        c, ref = _codec_pair(symad_sd, hifigan_sd, dec_kind)
        cap = 4
        c.set_streams(cap + 1)                                      # slot cap = the warm template
        torch.manual_seed(4)
        for _ in range(3):
            c.slots([0.1 * torch.randn(1500, device=DEV) for _ in range(cap)], list(range(cap)))
        for g in (c.tx, c.dec):
            g.copy_stream_state(cap, [1])                           # stream 1 closes, a new caller joins in its slot
        xs = [0.1 * torch.randn(1200, device=DEV) for _ in range(3)]
        got = [c.slots([xs[j], 0.1 * torch.randn(300, device=DEV)], [1, 3])[0] for j in range(3)]
        _same(got, _replay(ref, xs), dec_kind)


# ------------------------------------------------------------------ 5. mixing with the uniform calls
def test_uniform_calls_resize_and_reset_after_slots(symad_sd):
    c, ref = Codec(symad_sd), Codec(symad_sd)
    c.set_streams(4)
    torch.manual_seed(5)
    fed = {s: [] for s in range(6)}
    got = {s: [] for s in range(6)}

    def slot_step(streams, t=900):
        chunks = [0.1 * torch.randn(t, device=DEV) for _ in streams]
        for s, x, o in zip(streams, chunks, c.slots(chunks, streams)):
            fed[s].append(x)
            got[s].append(o)

    def uniform_step(n, t=600):
        x = 0.1 * torch.randn(n, t, device=DEV)
        z, idx, y = c.uniform(x)
        for s in range(n):
            fed[s].append(x[s])
            got[s].append((z[s:s + 1], idx[:, s], y[s]))

    slot_step([0, 2])
    slot_step([2, 3, 0])
    uniform_step(4)                        # streams 0 / 2 flipped once or twice, 1 never: each continues from its latest state
    slot_step([1])
    c.set_streams(6)                       # grow: 0..3 keep their state, 4 and 5 start from zero history
    slot_step([0, 1, 3])
    uniform_step(6)
    c.set_streams(3)                       # shrink
    slot_step([2, 0])
    uniform_step(3)
    torch.cuda.synchronize()
    for s in range(4):
        _same(got[s], _replay(ref, fed[s]), s)
    c.tx.reset_buffer()
    c.dec.reset_buffer()
    x = [0.1 * torch.randn(1500, device=DEV) for _ in range(3)]
    out = c.slots(x, [0, 1, 2])
    ref.set_streams(1)
    ref.tx.reset_buffer()
    ref.dec.reset_buffer()
    for s in range(3):
        ref.tx.reset_buffer()
        ref.dec.reset_buffer()
        z, idx, y = ref.uniform(x[s].view(1, -1))
        _same([out[s]], [(z, idx[:, 0], y)], ("reset", s))


def test_set_streams_after_slot_calls_on_a_side_stream(symad_sd, hifigan_sd):
    """Slot calls on a torch side stream (non-blocking with respect to stream 0), then set_streams from the default stream at once:
    the resize waits for the slot calls before it moves any state, so every stream continues from its latest state."""
    c, ref = _codec_pair(symad_sd, hifigan_sd, "v1_mode0")
    c.set_streams(8)
    torch.manual_seed(12)
    fed = {s: [] for s in range(8)}
    got = {s: [] for s in range(8)}
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        for streams in ([0, 3, 5], [3, 1, 7, 6], [5]):
            chunks = [0.1 * torch.randn(12000, device=DEV) for _ in streams]     # long chunks: the slot calls are still running
            for s, x, o in zip(streams, chunks, c.slots(chunks, streams)):
                fed[s].append(x)
                got[s].append(o)
    c.set_streams(10)                                             # from the default stream, with no synchronise in between
    torch.cuda.current_stream(DEV).wait_stream(side)
    streams = list(range(8))
    chunks = [0.1 * torch.randn(1500, device=DEV) for _ in streams]
    for s, x, o in zip(streams, chunks, c.slots(chunks, streams)):
        fed[s].append(x)
        got[s].append(o)
    torch.cuda.synchronize()
    for s in range(8):
        _same(got[s], _replay(ref, fed[s]), ("side stream", s))


# ------------------------------------------------------------------ 6. launches and profiled bytes
def test_launches_and_profiled_bytes(symad_sd, hifigan_sd):
    for dec_kind in ("symad", "v1_mode2"):
        c, u = _codec_pair(symad_sd, hifigan_sd, dec_kind)
        c.set_streams(8)
        u.set_streams(3)
        x = 0.1 * torch.randn(3, 1500, device=DEV)
        n0 = [g.launch_count for g in (u.tx, u.dec)]
        u.uniform(x)
        per_uniform = [g.launch_count - n for g, n in zip((u.tx, u.dec), n0)]
        for g in (c.tx, c.dec, u.tx, u.dec):
            g.profile(True)
        n0 = [g.launch_count for g in (c.tx, c.dec)]
        c.slots(list(x), [5, 1, 6])
        assert [g.launch_count - n for g, n in zip((c.tx, c.dec), n0)] == per_uniform
        u.uniform(x)
        for gs, gu in ((c.tx, u.tx), (c.dec, u.dec)):
            rs, ru = gs.profile_report(), gu.profile_report()
            assert [r[0] for r in rs] == [r[0] for r in ru]
            assert [r[2] for r in rs] == [r[2] for r in ru], dec_kind
            gs.profile(False)
            gu.profile(False)


# ------------------------------------------------------------------ 7. offline varlen after slot calls
def test_offline_varlen_unchanged_after_slots(symad_sd):
    c = Codec(symad_sd)
    c.set_streams(4)
    torch.manual_seed(6)
    c.slots([0.1 * torch.randn(900, device=DEV) for _ in range(2)], [3, 1])
    xs = [0.1 * torch.randn(n, device=DEV) for n in (300, 4801, 1500)]
    z, frames = c.tx.encode_offline_varlen(xs)
    o = 0
    for x, f in zip(xs, frames):
        assert torch.equal(_bits(z[:, :, o:o + f]), _bits(c.tx.encode_offline(x.view(1, 1, -1))))
        o += f


# ------------------------------------------------------------------ 8. rejections
def test_rejections(symad_sd, hifigan_sd, monkeypatch):
    from audiodec_b200 import _lib
    lib = _lib.load()
    enc, voc, voc2 = _symad(symad_sd), _voc(hifigan_sd, 0), _voc(hifigan_sd, 2)
    for g in (enc, voc, voc2):
        g.set_streams(4)
    s = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    buf = torch.zeros(1 << 16, device=DEV)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)
    ints = lambda *v: (ctypes.c_int * max(1, len(v)))(*v)

    def fails(h, rc, *words):
        assert rc != 0
        msg = _lib.last_error(h)
        assert all(w in msg for w in words), msg
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(300), ints(0), 0, p(buf), s), "encode_streams", "B must be >= 1")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), None, ints(0), 1, p(buf), s), "encode_streams", "lengths is NULL")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(300), None, 1, p(buf), s), "encode_streams", "streams is NULL")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(300, 0), ints(0, 1), 2, p(buf), s), "utterance 1", ">= 1")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(300), ints(4), 1, p(buf), s), "stream 4", "out of range")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(300), ints(-1), 1, p(buf), s), "stream -1", "out of range")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(300, 300), ints(2, 2), 2, p(buf), s), "stream 2", "twice")
    fails(enc._h, lib.adec_encode_streams(enc._h, p(buf), ints(1 << 30, 1 << 30), ints(0, 1), 2, p(buf), s), "32-bit row indexing")
    fails(voc._h, lib.adec_encode_streams(voc._h, p(buf), ints(300), ints(0), 1, p(buf), s), "not a symAD handle")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), ints(5), ints(0), 0, p(buf), s), "decode_streams", "B must be >= 1")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), None, ints(0), 1, p(buf), s), "decode_streams", "NULL")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), ints(5), None, 1, p(buf), s), "decode_streams", "streams is NULL")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), ints(5, 0), ints(0, 1), 2, p(buf), s), "utterance 1")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), ints(5, 5), ints(1, 1), 2, p(buf), s), "stream 1", "twice")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), ints(5), ints(9), 1, p(buf), s), "stream 9", "out of range")
    fails(voc._h, lib.adec_decode_streams(voc._h, p(buf), ints(1 << 24), ints(0), 1, p(buf), s), "32-bit row indexing")
    fails(voc2._h, lib.adec_decode_streams(voc2._h, p(buf), ints(5), ints(0), 1, p(buf), s), "adec_decode_streams_bf16")
    fails(voc._h, lib.adec_decode_streams_bf16(voc._h, p(buf), ints(5), ints(0), 1, p(buf), s), "adec_decode_streams", "fp32")
    fails(voc2._h, lib.adec_decode_streams_bf16(voc2._h, p(buf, 2), ints(5), ints(0), 1, p(buf), s), "16-byte aligned")
    fails(voc2._h, lib.adec_decode_streams_bf16(voc2._h, p(buf), ints(5), ints(0), 1, p(buf, 4), s), "16-byte aligned")
    fails(enc._h, lib.adec_copy_stream_state(enc._h, 4, ints(0), 1, s), "copy_stream_state", "src 4")
    fails(enc._h, lib.adec_copy_stream_state(enc._h, 0, ints(1, 7), 2, s), "copy_stream_state", "dst 7")
    monkeypatch.setenv("ADEC_CONV_PATH", "ffma")
    e0 = _symad(symad_sd)
    fails(e0._h, lib.adec_encode_streams(e0._h, p(buf), ints(300), ints(0), 1, p(buf), s), "FFMA", "tf32")
    with pytest.raises(RuntimeError, match="FFMA"):
        e0.encode_streams([buf[:300]], [0])


# ------------------------------------------------------------------ 9. SessionCodecServer
def _session(symad_sd, voc_sd, mode, cap, fs, sr):
    from audiodec_b200.server import SessionCodecServer
    c = Codec(symad_sd, voc_sd, mode)
    return SessionCodecServer(c.tx, c.rx, c.dec, capacity=cap, frame_size=fs, sample_rate=sr, max_latency=1.0, device="cuda:0",
                              wire=True)


def _churn(srv, steps, rng, fs):
    """sessions open, idle and close over `steps` steps; returns {session: frames in}, {session: frames out}"""
    live, ins, outs = {}, {}, {}
    for k in range(steps):
        if k in (0, 4, 9, 14):
            for _ in range(3 if k == 0 else 2):
                if len(live) < srv.capacity:
                    q = len(ins)
                    live[q] = srv.open()
                    ins[q], outs[q] = [], []
        for q, s in live.items():
            if rng.random() < 0.25:
                continue                                           # idle this step
            f = (0.1 * rng.standard_normal(fs)).astype(np.float32)
            srv.submit(s, f)
            ins[q].append(f)
        srv.step()
        for q, s in live.items():
            while (y := srv.poll(s)) is not None:
                outs[q].append(y)
        for q in [q for q in live if k > 2 and rng.random() < 0.12]:
            srv.close(live.pop(q))
    return ins, outs


@pytest.mark.parametrize("dec_kind", ["symad", "v1"])
def test_session_server_churn_matches_oracle(symad_sd, hifigan_sd, dec_kind):
    """issue item 9 at the configs[3] (libritts v1) layout: symAD encoder, and the symAD or the HiFi-GAN v1 (fp32) decoder"""
    from oracle import audiodec_oracle as O
    fs, sr, steps = 1500, 24000, 20
    v1 = dec_kind == "v1"
    srv = _session(symad_sd, hifigan_sd if v1 else None, 0, 6, fs, sr)
    ins, outs = _churn(srv, steps, np.random.default_rng(9), fs)
    st = srv.statistics()
    assert st["underruns"] > 0 and st["frame_drops"] == 0 and len(ins) >= 6
    checked = 0
    for q in ins:
        assert len(outs[q]) == len(ins[q]), q
        orc = O.CodecOracle(S.SYMAD_PARAMS, symad_sd, *((S.HIFIGAN_V1_PARAMS, hifigan_sd) if v1 else ()))
        for x, y in zip(ins[q], outs[q]):
            with torch.no_grad():
                _, _, _, ry = orc.run(torch.from_numpy(x).view(1, 1, fs))
            np.testing.assert_allclose(y, ry.numpy().reshape(-1)[:fs], atol=WAVE_TOL)
            checked += 1
    assert checked > 30


def test_session_server_indices_match_oracle(symad_sd):
    from oracle import audiodec_oracle as O
    c = Codec(symad_sd)
    c.set_streams(5)
    torch.manual_seed(10)
    xs = {s: [0.1 * torch.randn(1500) for _ in range(4)] for s in (0, 3)}
    got = {0: [], 3: []}
    for k in range(4):
        streams = [3, 0] if k != 2 else [0]
        for s, (_, idx, _) in zip(streams, c.slots([xs[s][k if s == 0 else (k if k < 2 else k - 1)].to(DEV) for s in streams], streams)):
            got[s].append(idx.cpu())
    for s, n in ((0, 4), (3, 3)):
        orc = O.CodecOracle(S.SYMAD_PARAMS, symad_sd)
        for k in range(n):
            with torch.no_grad():
                _, ridx, _, _ = orc.run(xs[s][k].view(1, 1, -1))
            assert torch.equal(got[s][k], ridx), (s, k)


def test_session_server_bf16_decoder_within_configs3_bar(golden_dir, symad_sd, hifigan_sd):
    g = np.load(os.path.join(golden_dir, "bf16_act.npz"))
    fs, sr, steps, cap = 1500, 24000, 3, 64
    srv16, srv32 = (_session(symad_sd, hifigan_sd, m, cap, fs, sr) for m in (2, 0))
    rng = np.random.default_rng(3)
    frames = (0.1 * rng.standard_normal((steps, cap, fs))).astype(np.float32)
    for srv in (srv16, srv32):
        ids = [srv.open() for _ in range(cap)]
        for k in range(steps):
            for s in ids:
                if (k + s) % 5 != 0:
                    srv.submit(s, frames[k, s])
            srv.step()
    v1_32, v1_16 = torch.from_numpy(g["v1_y_fp32"]), torch.from_numpy(g["v1_y_bf16"])
    ref_err = (v1_16 - v1_32).abs().max().item()
    ref_snr = (10 * torch.log10(v1_32.pow(2).mean() / (v1_16 - v1_32).pow(2).mean())).item()
    def drain(srv, s):
        out = []
        while (y := srv.poll(s)) is not None:
            out.append(y)
        return out
    for s in (0, 21, 42, 63):
        o16, o32 = drain(srv16, s), drain(srv32, s)
        assert len(o16) == len(o32) > 0 and all(o.dtype == np.float32 for o in o16)
        y, y32 = torch.from_numpy(np.concatenate(o16)), torch.from_numpy(np.concatenate(o32))
        err = (y - y32).abs().max().item()
        snr = (10 * torch.log10(y32.pow(2).mean() / (y - y32).pow(2).mean())).item()
        assert err <= 1.2 * ref_err and snr >= ref_snr - 2.0, (s, err, snr)
