"""The receiver's playout clock on the GPU.  lookup_packed_playout against a numpy float32 model of its three row kinds, bit for bit, in
fp32 and bf16, with its real and interpolated rows equal to lookup_packed_conceal's; the C ABI's refusals; the codec's silence frame;
and ReceiverSessionServer(playout_delay=D) end to end for vctk_sym and libritts v1 in receiver modes 0, 1 and 2: jitter within D
against a receiver without a playout clock fed in order, and a loss with a held follower, a late arrival and an end-of-spurt loss
(fade, pause, resume) against a B = 1 decoder fed the model's zq, with a session moved in the middle of a fade."""
import ctypes
import re

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S
from audiodec_b200 import wire

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FS = 1500                              # 5 frames of hop 300 per packet
FPP = FS // 300
RATE = {"vctk_sym": 48000, "libritts_v1": 24000}


def interp(a, t, j, den):
    """fl(fl(fl(j / den) * fl(t - a)) + a) in float32"""
    a, t = np.asarray(a, dtype=np.float32), np.asarray(t, dtype=np.float32)
    return (np.float32(j) / np.float32(den)) * (t - a) + a


def row_model(row, sums, anchors, targets):
    """one output row of adec_lookup_packed_playout in float32 (anchors as they were before the call)"""
    src, nxt, tgt, slot, j, den = row
    if src >= 0:
        return sums[src]
    if nxt >= 0:
        return sums[nxt].copy() if slot < 0 else interp(anchors[slot], sums[nxt], j, den)
    return targets[tgt].copy() if slot < 0 or j >= den else interp(anchors[slot], targets[tgt], j, den)


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


def _bf16_bits(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).view(torch.int16).numpy()


def _gen(sd):
    from audiodec_b200.codec import SymADStreamGenerator
    g = SymADStreamGenerator(**S.SYMAD_PARAMS)
    g.load_state_dict(sd)
    return g.eval().to(DEV)


def _tx(sd):
    g = _gen(sd)
    g.initial_encoder(8192, DEV)
    return g


def _rx(model, symad_sd, hifigan_sd, mode):
    """rx_encoder (codebooks) and a decoder in dtype mode 0 / 1 / 2, warmed as load_receiver leaves them"""
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADDecoderStreamGenerator
    rx = _gen(symad_sd)
    if model == "vctk_sym":
        d = SymADDecoderStreamGenerator(**S.SYMAD_PARAMS)
        d.load_state_dict(symad_sd)
    else:
        d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
        d.load_state_dict(hifigan_sd)
    if mode >= 1:
        d = d.to(torch.bfloat16)
    if mode == 2:
        d = d.set_activation_dtype(torch.bfloat16)
    d = d.eval().to(DEV)
    d.initial_decoder(rx.initial_encoder(8192, DEV))
    return rx, d


def _receiver(model, symad_sd, hifigan_sd, mode, cap, **kw):
    from audiodec_b200.server import ReceiverSessionServer
    return ReceiverSessionServer(*_rx(model, symad_sd, hifigan_sd, mode), capacity=cap, frames_per_packet=FPP,
                                 sample_rate=RATE[model], device=DEV, **kw)


def _packets(symad_sd, model, sids, n, seed):
    """n packets per session id from one transmitter server, as {sid: [bytes by sequence number]}"""
    from audiodec_b200.server import TransmitterSessionServer
    txs = TransmitterSessionServer(_tx(symad_sd), capacity=len(sids), frame_size=FS, sample_rate=RATE[model], max_latency=10.0,
                                   device=DEV)
    for sid in sids:
        txs.open(sid)
    rng = np.random.default_rng(seed)
    out = {sid: [] for sid in sids}
    for _ in range(n):
        for sid in sids:
            txs.submit(sid, (0.1 * rng.standard_normal(FS)).astype(np.float32))
        txs.step()
        for sid, buf in txs.poll_packets():
            out[sid].append(buf)
    return out


def _packed(buf):
    p = wire.decode_packet(buf)
    return torch.frombuffer(bytearray(p.payload), dtype=torch.uint8).view(p.frames, -1).to(DEV)


def _drain(srv, sid):
    out = []
    while (y := srv.poll(sid)) is not None:
        out.append(y)
    return out


# ------------------------------------------------------------------ the kernel against the model
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernel_equals_the_model(symad_sd, dtype):
    g = _gen(symad_sd)
    nq, n, d = g.codebook_num, S.SYMAD_PARAMS["codebook_size"], g.code_dim
    rng = np.random.default_rng(8)
    f = 29
    idx = torch.from_numpy(rng.integers(0, n, (nq, f)) + np.arange(nq)[:, None] * n).to(DEV)
    packed = g.pack(idx)
    sums = g.lookup_packed(packed)[0].cpu().numpy()
    a0 = (rng.standard_normal((6, d)) * np.float32(0.3)).astype(np.float32)
    t0 = (rng.standard_normal((2, d)) * np.float32(0.2)).astype(np.float32)
    anchors, targets = torch.from_numpy(a0).to(DEV), torch.from_numpy(t0).to(DEV)
    # real rows (some storing an anchor), interpolated rows, fade rows below, at and beyond den, and without an anchor
    rows = [(4, -1, -1, -1, 0, 0), (7, -1, -1, 3, 0, 0), (-1, 11, -1, 0, 1, 4), (-1, 11, -1, 0, 3, 4), (-1, 2, -1, -1, 1, 2),
            (-1, -1, 0, 1, 1, 10), (-1, -1, 0, 1, 9, 10), (-1, -1, 0, 1, 10, 10), (-1, -1, 1, 1, 37, 10), (-1, -1, 1, -1, 2, 10),
            (-1, -1, 1, 2, 1, 1), (28, -1, -1, 5, 0, 0), (-1, -1, 0, 0, 3, 7), (13, -1, -1, 4, 0, 0)]
    rows += [(-1, int(rng.integers(0, f)), -1, 2, int(j), 101) for j in rng.integers(1, 101, 150)]
    rows += [(-1, -1, int(rng.integers(0, 2)), int(rng.integers(0, 3)), int(j), 60) for j in rng.integers(1, 90, 150)]
    rows += [(int(s), -1, -1, -1, 0, 0) for s in rng.integers(0, f, 100)]
    launches = g.launch_count
    zq = g.lookup_packed_playout(packed, np.asarray(rows, np.int32), anchors, targets, dtype=dtype)
    assert g.launch_count == launches + 1
    assert zq.shape == (1, len(rows), d) and zq.dtype == dtype
    want = np.stack([row_model(r, sums, a0, t0) for r in rows])
    got = zq[0].cpu()
    if dtype == torch.float32:
        assert np.array_equal(_bits(got.numpy()), _bits(want))
    else:
        assert np.array_equal(got.view(torch.int16).numpy(), _bf16_bits(want))
    assert np.array_equal(_bits(want[7]), _bits(t0[0])) and not np.array_equal(_bits(want[6]), _bits(t0[0]))
    av = anchors.cpu().numpy()
    for slot, src in ((3, 7), (5, 28), (4, 13)):
        assert np.array_equal(_bits(av[slot]), _bits(sums[src]))
    assert np.array_equal(_bits(av[:3]), _bits(a0[:3]))
    # real and interpolated rows are lookup_packed_conceal's, on the same inputs
    keep = [i for i, r in enumerate(rows) if r[0] >= 0 or r[1] >= 0]
    conceal_rows = np.asarray([(r[0], r[1], r[3], r[4], r[5]) for r in (rows[i] for i in keep)], np.int32)
    ref = g.lookup_packed_conceal(packed, conceal_rows, torch.from_numpy(a0).to(DEV), dtype=dtype)[0].cpu()
    assert np.array_equal(ref.view(torch.int16 if dtype == torch.bfloat16 else torch.int32).numpy(),
                          got[keep].view(torch.int16 if dtype == torch.bfloat16 else torch.int32).numpy())
    assert not g.index_error()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_a_step_where_every_session_fades_stages_no_frames(symad_sd, dtype):
    g = _gen(symad_sd)
    d = g.code_dim
    a0 = np.linspace(-1, 1, 2 * d, dtype=np.float32).reshape(2, d)
    t0 = np.full((1, d), 0.125, np.float32)
    rows = [(-1, -1, 0, 0, 1, 3), (-1, -1, 0, 0, 2, 3), (-1, -1, 0, 1, 5, 3), (-1, -1, 0, -1, 1, 3)]
    empty = torch.zeros(0, g.packed_frame_bytes(), dtype=torch.uint8, device=DEV)
    zq = g.lookup_packed_playout(empty, rows, torch.from_numpy(a0).to(DEV), torch.from_numpy(t0).to(DEV), dtype=dtype)[0].cpu()
    want = np.stack([row_model(r, None, a0, t0) for r in rows])
    if dtype == torch.float32:
        assert np.array_equal(_bits(zq.numpy()), _bits(want))
    else:
        assert np.array_equal(zq.view(torch.int16).numpy(), _bf16_bits(want))


# ------------------------------------------------------------------ refusals
def _call(g, packed, f, rows, anchors, targets, zq, bf16=False):
    from audiodec_b200 import _lib
    lib = _lib.load()
    arr = (_lib.AdecPlayoutRow * len(rows))(*[_lib.AdecPlayoutRow(*r) for r in rows])
    fn = lib.adec_lookup_packed_playout_bf16 if bf16 else lib.adec_lookup_packed_playout
    rc = fn(g._h, ctypes.c_void_p(packed.data_ptr()), f, ctypes.cast(arr, ctypes.c_void_p), len(rows),
            ctypes.c_void_p(anchors.data_ptr()), anchors.shape[0], ctypes.c_void_p(targets.data_ptr()), targets.shape[0],
            ctypes.c_void_p(zq.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    return rc, _lib.last_error(g._h)


@pytest.mark.parametrize("rows,field", [
    ([(3, -1, -1, -1, 0, 0)], r"rows\[0\]\.src = 3 is out of range"),
    ([(-2, 0, -1, -1, 1, 2)], r"rows\[0\]\.src = -2"),
    ([(0, 1, -1, -1, 0, 0)], r"rows\[0\]\.next = 1"),
    ([(-1, 3, -1, -1, 1, 2)], r"rows\[0\]\.next = 3 is out of range"),
    ([(-1, -2, 0, -1, 1, 2)], r"rows\[0\]\.next = -2 is out of range"),
    ([(0, -1, 0, -1, 0, 0)], r"rows\[0\]\.target = 0: only a fade row"),
    ([(-1, 0, 0, -1, 1, 2)], r"rows\[0\]\.target = 0: only a fade row"),
    ([(-1, -1, 1, -1, 1, 2)], r"rows\[0\]\.target = 1 is out of range"),
    ([(-1, -1, -1, -1, 1, 2)], r"rows\[0\]\.target = -1 is out of range"),
    ([(0, -1, -1, 2, 0, 0)], r"rows\[0\]\.slot = 2 is out of range"),
    ([(-1, -1, 0, -2, 1, 2)], r"rows\[0\]\.slot = -2 is out of range"),
    ([(-1, 0, -1, 0, 1, 1)], r"rows\[0\]\.den = 1: an interpolated row"),
    ([(-1, 0, -1, 0, 3, 3)], r"rows\[0\]\.j = 3 is outside"),
    ([(-1, -1, 0, 0, 1, 0)], r"rows\[0\]\.den = 0: a fade row"),
    ([(-1, -1, 0, 0, 0, 2)], r"rows\[0\]\.j = 0: a fade row"),
    ([(0, -1, -1, 1, 0, 0), (-1, -1, 0, 1, 1, 2)], r"rows\[1\]\.slot = 1: anchor 1 is read by row 1 and written by row 0"),
    ([(-1, -1, 0, 1, 1, 2), (0, -1, -1, 1, 0, 0)], r"rows\[1\]\.slot = 1: anchor 1 is read by row 0 and written by row 1"),
    ([(0, -1, -1, 0, 0, 0), (1, -1, -1, 0, 0, 0)], r"rows\[1\]\.slot = 0: anchor 0 is written by rows 0 and 1"),
])
def test_bad_descriptors_are_refused_by_name(symad_sd, rows, field):
    g = _gen(symad_sd)
    packed = g.pack(torch.zeros(g.codebook_num, 3, dtype=torch.int64, device=DEV))
    anchors = torch.full((2, g.code_dim), 5.0, device=DEV)
    targets = torch.full((1, g.code_dim), 6.0, device=DEV)
    zq = torch.full((len(rows), g.code_dim), 7.0, device=DEV)
    launches = g.launch_count
    for bf16 in (False, True):
        rc, msg = _call(g, packed, 3, rows, anchors, targets, zq, bf16)
        assert rc != 0 and ("lookup_packed_playout_bf16" if bf16 else "lookup_packed_playout") in msg
        assert re.search(field, msg), msg
    assert g.launch_count == launches
    torch.cuda.synchronize()
    assert (anchors == 5.0).all() and (zq == 7.0).all()
    with pytest.raises(RuntimeError, match="rows"):
        g.lookup_packed_playout(packed, rows, anchors, targets)


def test_encoder_and_decoder_only_handles_refuse(symad_sd):
    from audiodec_b200.codec import SymADDecoderStreamGenerator, SymADEncoderStreamGenerator
    handles = []
    for cls in (SymADEncoderStreamGenerator, SymADDecoderStreamGenerator):
        h = cls(**S.SYMAD_PARAMS)
        h.load_state_dict(symad_sd)
        handles.append(h.eval().to(DEV))
    packed = torch.zeros(2, 10, dtype=torch.uint8, device=DEV)
    anchors, targets, zq = (torch.zeros(1, 64, device=DEV) for _ in range(3))
    for g, word in zip(handles, ("encoder-only", "decoder-only")):
        for bf16 in (False, True):
            rc, msg = _call(g, packed, 2, [(0, -1, -1, 0, 0, 0)], anchors, targets, zq, bf16)
            assert rc != 0 and word in msg and "lookup_packed_playout" in msg, msg
        assert not hasattr(g, "lookup_packed_playout")


# ------------------------------------------------------------------ the silence frame
def test_silence_frame_is_stateless_steady_and_the_offline_codes_sum(symad_sd):
    g = _tx(symad_sd)
    g.set_streams(3)
    g.encode(0.1 * torch.randn(3, 1, 900, device=DEV))                # live, different state in every stream
    before = g.stream_state(range(3)).clone()
    sf = g.silence_frame()
    assert sf.shape == (g.code_dim,) and sf.dtype == torch.float32 and sf.device == DEV
    assert g.n_streams == 3 and torch.equal(g.stream_state(range(3)), before)
    ref = _gen(symad_sd)
    zeros = torch.zeros(1, 1, 8400, device=DEV)                       # 8192 rounded up to a multiple of the hop, 300
    zq, idx = ref.quantize_offline(ref.encode_offline(zeros))
    assert np.array_equal(_bits(sf.cpu().numpy()), _bits(zq[0, :, -1].cpu().numpy()))
    assert torch.equal(idx[:, 0, -1], idx[:, 0, -2])                  # a steady state
    assert torch.equal(g.silence_frame(), sf)


# ------------------------------------------------------------------ end to end
N = 16


def _expected(packets, schedule, ref_rx, ref_dec, mode, silence):
    """The PCM of a B = 1 decoder fed, packet by packet, the zq of `schedule`: ("real", q), ("interp", m, first j, den) toward packet
    m's first frame, ("fade", frames, first j, den) toward the silence frame, from the anchor of the last real packet."""
    dt = torch.bfloat16 if mode == 2 else torch.float32
    want, anchor = [], None
    for e in schedule:
        if e[0] == "real":
            packed = _packed(packets[e[1]])
            anchor = ref_rx.lookup_packed(packed)[0, -1].cpu().numpy()
            zq, f = ref_rx.lookup_packed(packed, dtype=dt), packed.shape[0]
        else:
            if e[0] == "interp":
                b = _packed(packets[e[1]])
                t, f = ref_rx.lookup_packed(b)[0, 0].cpu().numpy(), b.shape[0]
            else:
                t, f = silence, e[1]
            rows = [t if anchor is None or (e[0] == "fade" and e[2] + i >= e[3]) else interp(anchor, t, e[2] + i, e[3]) for i in range(f)]
            zq = torch.from_numpy(np.stack(rows).astype(np.float32)).to(DEV).view(1, f, -1).to(dt)
        want.append(ref_dec.decode_streams(zq, [f], [0])[0].float().reshape(-1).cpu().numpy())
    return want


def _traffic():
    """per session: {step: [sequence numbers arriving before it]} over 24 steps, and the schedule a playout_delay=1 receiver plays.
    Session 1: packet 3 lost with 4 held behind it, and arriving late at step 9.  Session 2: its talk spurt ends with a lost packet 5;
    four fades (fade_frames 10), a pause rewound to 5, and a resume at step 15 that conceals 5 toward 6.  Session 3: jitter only.
    Every session ends with four fades and a pause."""
    arr1 = {q: [q] for q in range(N) if q != 3}
    arr1.setdefault(9, []).append(3)
    arr2 = {q: [q] for q in range(5)}
    arr2.update({15: [6], 16: [7], 17: [8]})
    arr3 = {0: [0], 1: [2, 1], 2: [3], 3: [], 4: [5, 4]}
    arr3.update({q: [q] for q in range(6, N)})
    fades = [("fade", FPP, 1 + k * FPP, 2 * FPP) for k in range(4)]
    sch1 = [("real", q) for q in range(3)] + [("interp", 4, 1, FPP + 1)] + [("real", q) for q in range(4, N)] + fades
    sch2 = [("real", q) for q in range(5)] + fades + [("interp", 6, 4 * FPP + 1, 5 * FPP + 1)] + [("real", q) for q in (6, 7, 8)] + fades
    sch3 = [("real", q) for q in range(N)] + fades
    return {1: (arr1, sch1), 2: (arr2, sch2), 3: (arr3, sch3)}


def _play(srv, packets, traffic, steps, move=None):
    """run the traffic through srv; move = (sid, when(server, slot), destination): detach the session there once `when` holds"""
    got = {sid: [] for sid in traffic}
    cur = {sid: srv for sid in traffic}
    for t in range(steps):
        for sid, (arr, _) in traffic.items():
            for q in arr.get(t, []):
                cur[sid].submit_packet(packets[sid][q])
        if move is not None and cur[move[0]] is srv and move[1](srv, srv._ids[move[0]]):
            assert move[2].attach(srv.detach(move[0]).to(DEV)) == move[0]
            cur[move[0]] = move[2]
        for s in {id(x): x for x in cur.values()}.values():
            s.step()
        for sid in traffic:
            got[sid].extend(_drain(cur[sid], sid))
    return got, cur


@pytest.mark.parametrize("model", ["vctk_sym", "libritts_v1"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_playout_pcm_equals_the_reference_decoder(symad_sd, hifigan_sd, model, mode):
    traffic = _traffic()
    packets = _packets(symad_sd, model, sorted(traffic), N, seed=31)
    rxs = _receiver(model, symad_sd, hifigan_sd, mode, cap=4, playout_delay=1)
    for sid in traffic:
        rxs.open(sid)
    got, _ = _play(rxs, packets, traffic, 24)
    st = rxs.statistics()["per_session"]
    assert (st[1]["losses"], st[1]["concealed"], st[1]["late"], st[1]["packets"], st[1]["pauses"]) == (1, 1, 1, N - 1, 1)
    assert (st[2]["underruns"], st[2]["faded_frames"], st[2]["pauses"], st[2]["losses"], st[2]["packets"]) == (8, 8 * FPP, 2, 1, 8)
    assert (st[3]["losses"], st[3]["underruns"], st[3]["packets"], st[3]["late"]) == (0, 4, N, 0)
    silence = rxs.rx_encoder.silence_frame().cpu().numpy()
    for sid, (_, sch) in traffic.items():
        ref_rx, ref_dec = _rx(model, symad_sd, hifigan_sd, mode)
        want = _expected(packets[sid], sch, ref_rx, ref_dec, mode, silence)
        assert len(got[sid]) == len(want), sid
        for k, (a, b) in enumerate(zip(got[sid], want)):
            assert a.dtype == np.float32 and a.shape == b.shape == (FS,)
            assert np.array_equal(_bits(a), _bits(b)), (model, mode, sid, k)


@pytest.mark.parametrize("model,mode", [("vctk_sym", 0), ("vctk_sym", 2), ("libritts_v1", 1), ("libritts_v1", 2)])
def test_jitter_within_the_delay_equals_a_receiver_without_a_clock_fed_in_order(symad_sd, hifigan_sd, model, mode):
    sids = [4, 7, 9]
    n = 12
    packets = _packets(symad_sd, model, sids, n, seed=5)
    on = _receiver(model, symad_sd, hifigan_sd, mode, cap=3, playout_delay=2)
    off = _receiver(model, symad_sd, hifigan_sd, mode, cap=3)
    rng = np.random.default_rng(11)
    arrive = {}
    for sid in sids:
        on.open(sid), off.open(sid)
        for q in range(n):
            arrive.setdefault(q + (int(rng.integers(0, 3)) if q else 0), []).append((sid, q))
    got = {(w, sid): [] for w in ("on", "off") for sid in sids}
    for t in range(n + 2):
        batch = arrive.get(t, [])
        rng.shuffle(batch)
        for sid, q in batch:
            assert on.submit_packet(packets[sid][q])
        if t < n:
            for sid in sids:
                off.submit_packet(packets[sid][t])
            off.step()
        on.step()
        for sid in sids:
            got["on", sid].extend(_drain(on, sid))
            got["off", sid].extend(_drain(off, sid))
    for sid in sids:
        assert len(got["on", sid]) == len(got["off", sid]) == n
        for a, b in zip(got["on", sid], got["off", sid]):
            assert np.array_equal(_bits(a), _bits(b))
        st = on.statistics()["per_session"][sid]
        assert (st["losses"], st["concealed"], st["underruns"], st["packets"]) == (0, 0, 0, n)
    assert all(t.is_pinned() for t in on._rows_host) and on._rows_host[0].data_ptr() != on._rows_host[1].data_ptr()


def test_a_session_moved_in_the_middle_of_a_fade_continues_bit_for_bit(symad_sd, hifigan_sd):
    model, mode = "libritts_v1", 2
    traffic = {2: _traffic()[2], 3: _traffic()[3]}
    packets = _packets(symad_sd, model, [2, 3], N, seed=9)
    ref = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, playout_delay=1)
    a = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, playout_delay=1)
    b = _receiver(model, symad_sd, hifigan_sd, mode, cap=3, playout_delay=1)
    for srv in (ref, a):
        srv.open(2), srv.open(3)
    b.open(11)                                                        # the destination serves someone: another slot
    for _ in range(3):
        b.step()                                                      # and its step count differs
    want, _ = _play(ref, packets, traffic, 24)
    got, cur = _play(a, packets, traffic, 24, move=(2, lambda s, slot: s.stats[slot].underruns == 2, b))
    assert cur[2] is b and cur[3] is a and b._ids[2] == 1 and ref._ids[2] == 0
    for sid in (2, 3):
        assert len(got[sid]) == len(want[sid])
        for x, y in zip(got[sid], want[sid]):
            assert np.array_equal(_bits(x), _bits(y))
    st = b.statistics()["per_session"][2]
    assert (st["underruns"], st["pauses"], st["concealed"], st["packets"]) == (6, 2, 1, 3)
