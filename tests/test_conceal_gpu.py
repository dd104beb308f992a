"""Receiver loss concealment on the GPU.  lookup_packed_conceal against a numpy float32 model of its formula, bit for bit, in fp32 and
bf16, and on all-ones packed fields; ReceiverSessionServer(conceal_packets=2) against a B = 1 reference decoder fed the real packets'
lookup_packed zq and the model's concealed zq, packet by packet, for vctk_sym and libritts v1 in receiver modes 0, 1 and 2; no loss
against conceal_packets=0 and SessionCodecServer(wire=True); a session moved in the middle of a gap; and the C ABI's refusals."""
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
RATE = {"vctk_sym": 48000, "libritts_v1": 24000}
K = 2


def conceal_model(a, s_b, j, den):
    """the concealed zq in float32: fl(fl(fl(j / den) * fl(s_b - a)) + a); a None: s_b"""
    s_b = np.asarray(s_b, dtype=np.float32)
    if a is None:
        return s_b.copy()
    a = np.asarray(a, dtype=np.float32)
    w = np.float32(j) / np.float32(den)
    return (w * (s_b - a)) + a


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


def _bf16_bits(x):
    """float32 values -> the bits of their round-to-nearest-even bf16"""
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


def _receiver(model, symad_sd, hifigan_sd, mode, cap, k=K):
    from audiodec_b200.server import ReceiverSessionServer
    return ReceiverSessionServer(*_rx(model, symad_sd, hifigan_sd, mode), capacity=cap, frames_per_packet=FS // 300,
                                 sample_rate=RATE[model], device=DEV, conceal_packets=k)


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
    rng = np.random.default_rng(5)
    f = 37
    idx = torch.from_numpy(rng.integers(0, n, (nq, f)) + np.arange(nq)[:, None] * n).to(DEV)
    packed = g.pack(idx)                                                          # (F, bytes)
    sums = g.lookup_packed(packed)[0].cpu().numpy()                               # (F, D) fp32, the real rows' values
    n_anchors = 6
    a0 = (rng.standard_normal((n_anchors, d)) * np.float32(0.3)).astype(np.float32)
    anchors = torch.from_numpy(a0).to(DEV)
    # real rows, some storing an anchor; concealed rows on anchors 0..2, one without an anchor, j up to den - 1
    rows = [(5, -1, -1, 0, 0), (9, -1, 3, 0, 0), (-1, 11, 0, 1, 4), (-1, 11, 0, 2, 4), (-1, 11, 0, 3, 4), (-1, 2, -1, 1, 2),
            (0, -1, -1, 0, 0), (-1, 36, 1, 1, 7), (-1, 36, 1, 6, 7), (-1, 20, 2, 1, 2), (36, -1, 5, 0, 0), (17, -1, 4, 0, 0)]
    rows += [(-1, int(rng.integers(0, f)), 2, int(j), 101) for j in rng.integers(1, 101, 300)]
    rows += [(int(s), -1, -1, 0, 0) for s in rng.integers(0, f, 200)]
    launches = g.launch_count
    zq = g.lookup_packed_conceal(packed, np.asarray(rows, np.int32), anchors, dtype=dtype)
    assert g.launch_count == launches + 1
    assert zq.shape == (1, len(rows), d) and zq.dtype == dtype
    want = np.stack([sums[src] if src >= 0 else conceal_model(a0[slot] if slot >= 0 else None, sums[nxt], j, den)
                     for src, nxt, slot, j, den in rows])
    got = zq[0].cpu()
    if dtype == torch.float32:
        assert np.array_equal(_bits(got.numpy()), _bits(want))
    else:
        assert np.array_equal(got.view(torch.int16).numpy(), _bf16_bits(want))
        ref = g.lookup_packed(packed, dtype=torch.bfloat16)[0].cpu().view(torch.int16).numpy()
        real = [i for i, r in enumerate(rows) if r[0] >= 0]
        assert np.array_equal(got.view(torch.int16).numpy()[real], ref[[rows[i][0] for i in real]])
    # the model really interpolates: the concealed rows differ from s_b and from a
    assert not np.array_equal(want[2], sums[11]) and not np.array_equal(want[2], a0[0])
    # anchors: the written ones hold their real row's fp32 sum, the others are untouched
    av = anchors.cpu().numpy()
    for slot, src in ((3, 9), (5, 36), (4, 17)):
        assert np.array_equal(_bits(av[slot]), _bits(sums[src]))
    assert np.array_equal(_bits(av[:3]), _bits(a0[:3]))
    assert not g.index_error()


def test_all_ones_fields_are_in_range_and_leave_the_flag_clear(symad_sd):
    """The library builds 1024-word codebooks only, so a packed 10-bit field cannot hold an out-of-range index: the largest, 1023 in
    every stage (all-ones bytes), is looked up like any other, in real and in concealed rows, and the index flag stays clear."""
    g = _gen(symad_sd)
    nb = g.packed_frame_bytes()
    packed = torch.cat([torch.full((1, nb), 0xFF, dtype=torch.uint8, device=DEV), torch.zeros(1, nb, dtype=torch.uint8, device=DEV)])
    want = g.lookup_packed(packed)[0].cpu().numpy()
    top = g.lookup(torch.arange(g.codebook_num, device=DEV).view(-1, 1) * 1024 + 1023)[0, 0].cpu().numpy()
    assert np.array_equal(_bits(want[0]), _bits(top))
    anchors = torch.zeros(1, g.code_dim, device=DEV)
    zq = g.lookup_packed_conceal(packed, [(0, -1, -1, 0, 0), (-1, 0, 0, 1, 2), (1, -1, -1, 0, 0)], anchors)[0].cpu().numpy()
    assert np.array_equal(_bits(zq[0]), _bits(want[0])) and np.array_equal(_bits(zq[2]), _bits(want[1]))
    assert np.array_equal(_bits(zq[1]), _bits(conceal_model(np.zeros(g.code_dim, np.float32), want[0], 1, 2)))
    assert not g.index_error()


# ------------------------------------------------------------------ end to end against a B = 1 reference decoder
DROPS = {1: {0}, 2: {5}, 3: {3, 4, 5, 6, 11}}       # the first packet; one in the middle; a run of 4 (> K) and a later single loss
N_PACKETS = 18


def _expected(packets, drops, ref_rx, ref_dec, mode):
    """the PCM of a B = 1 decoder fed, packet by packet, lookup_packed of the real packets and the model's zq for the concealed ones"""
    dt = torch.bfloat16 if mode == 2 else torch.float32
    want, anchor, q, n = [], None, 0, len(packets)
    while q < n:
        if q in drops:
            end = q
            while end in drops:
                end += 1
            b = _packed(packets[end])
            s_b = ref_rx.lookup_packed(b)[0, 0].cpu().numpy()
            c = min(end - q, K)
            m = c * b.shape[0]
            for p in range(c):
                zq = np.stack([conceal_model(anchor, s_b, p * b.shape[0] + i + 1, m + 1) for i in range(b.shape[0])])
                zq = torch.from_numpy(zq).to(DEV).view(1, -1, zq.shape[-1]).to(dt)
                want.append(ref_dec.decode_streams(zq, [b.shape[0]], [0])[0].float().reshape(-1).cpu().numpy())
            q = end
            continue
        packed = _packed(packets[q])
        zq32 = ref_rx.lookup_packed(packed)
        anchor = zq32[0, -1].cpu().numpy()
        y = ref_dec.decode_streams(ref_rx.lookup_packed(packed, dtype=dt), [packed.shape[0]], [0])[0]
        want.append(y.float().reshape(-1).cpu().numpy())
        q += 1
    return want


@pytest.mark.parametrize("model", ["vctk_sym", "libritts_v1"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_concealed_pcm_equals_the_reference_decoder(symad_sd, hifigan_sd, model, mode):
    sids = sorted(DROPS)
    packets = _packets(symad_sd, model, sids, N_PACKETS, seed=21)
    rxs = _receiver(model, symad_sd, hifigan_sd, mode, cap=len(sids) + 1)
    for sid in sids:
        rxs.open(sid)
    got = {sid: [] for sid in sids}
    for q in range(N_PACKETS):                                        # one packet per session per step, as they are sent
        for sid in sids:
            if q not in DROPS[sid]:
                assert rxs.submit_packet(packets[sid][q])
        rxs.step()
        for sid in sids:
            got[sid].extend(_drain(rxs, sid))
    while rxs.step():
        for sid in sids:
            got[sid].extend(_drain(rxs, sid))
    st = rxs.statistics()["per_session"]
    for sid in sids:
        runs = _runs(DROPS[sid])
        concealed = sum(min(r, K) for r in runs)
        assert (st[sid]["losses"], st[sid]["concealed"]) == (len(DROPS[sid]), concealed), sid
        assert st[sid]["packets"] == N_PACKETS - len(DROPS[sid]) and st[sid]["concealed_frames"] == concealed * (FS // 300)
        ref_rx, ref_dec = _rx(model, symad_sd, hifigan_sd, mode)
        want = _expected(packets[sid], DROPS[sid], ref_rx, ref_dec, mode)
        assert len(got[sid]) == len(want) == N_PACKETS - len(DROPS[sid]) + concealed, sid
        for k, (a, b) in enumerate(zip(got[sid], want)):
            assert a.dtype == np.float32 and a.shape == b.shape == (FS,)
            assert np.array_equal(_bits(a), _bits(b)), (model, mode, sid, k)


def _runs(drops):
    runs, prev = [], None
    for q in sorted(drops):
        if prev is not None and q == prev + 1:
            runs[-1] += 1
        else:
            runs.append(1)
        prev = q
    return runs


@pytest.mark.parametrize("model,mode", [("vctk_sym", 0), ("libritts_v1", 2)])
def test_no_loss_equals_conceal_off_and_the_loopback(symad_sd, hifigan_sd, model, mode):
    from audiodec_b200.server import SessionCodecServer, TransmitterSessionServer
    rx_enc, dec = _rx(model, symad_sd, hifigan_sd, mode)
    loop = SessionCodecServer(_tx(symad_sd), rx_enc, dec, capacity=2, frame_size=FS, sample_rate=RATE[model], max_latency=10.0,
                              device=DEV, wire=True)
    txs = TransmitterSessionServer(_tx(symad_sd), capacity=2, frame_size=FS, sample_rate=RATE[model], max_latency=10.0, device=DEV)
    on = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, k=K)
    off = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, k=0)
    slots = {sid: loop.open() for sid in (4, 7)}
    for srv in (txs, on, off):
        for sid in slots:
            srv.open(sid)
    rng = np.random.default_rng(2)
    got = {(w, sid): [] for w in ("loop", "on", "off") for sid in slots}
    for _ in range(8):
        for sid, s in slots.items():
            x = (0.1 * rng.standard_normal(FS)).astype(np.float32)
            loop.submit(s, x)
            txs.submit(sid, x)
        loop.step()
        txs.step()
        for _, buf in txs.poll_packets():
            on.submit_packet(buf)
            off.submit_packet(buf)
        on.step()
        off.step()
        for sid, s in slots.items():
            got["loop", sid].extend(_drain(loop, s))
            got["on", sid].extend(_drain(on, sid))
            got["off", sid].extend(_drain(off, sid))
    for sid in slots:
        assert len(got["on", sid]) == len(got["off", sid]) == len(got["loop", sid]) == 8
        for a, b, c in zip(got["on", sid], got["off", sid], got["loop", sid]):
            assert np.array_equal(_bits(a), _bits(b)) and np.array_equal(_bits(a), _bits(c))
        st = on.statistics()["per_session"][sid]
        assert (st["losses"], st["concealed"], st["packets"]) == (0, 0, 8)


def test_session_moved_in_the_middle_of_a_gap_continues_bit_for_bit(symad_sd, hifigan_sd):
    model, mode = "libritts_v1", 2
    drops = {3, 4, 5}                                                 # K = 3: three concealed packets
    packets = _packets(symad_sd, model, [1], 14, seed=6)[1]
    ref = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, k=3)
    a = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, k=3)
    b = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, k=3)
    ref.open(1), a.open(1), b.open(9)                                 # the destination serves someone: another slot
    want, got, cur, moved = [], [], a, False
    for q in range(14):
        if q not in drops:
            ref.submit_packet(packets[q])
            cur.submit_packet(packets[q])
        ref.step()
        cur.step()
        want.extend(_drain(ref, 1))
        if not moved and cur.statistics()["per_session"][1]["concealed"] == 1:
            st = a.detach(1)                                          # one concealed packet decoded and unpolled, two to come
            assert st.conceal is not None and st.conceal[0] == 2 and st.anchor is not None and len(st.outputs) == 1
            assert b.attach(st.to(DEV)) == 1 and b._ids[1] == 1
            cur, moved = b, True
        else:
            got.extend(_drain(cur, 1))
    while ref.step() + cur.step():
        want.extend(_drain(ref, 1))
        got.extend(_drain(cur, 1))
    want.extend(_drain(ref, 1))
    got.extend(_drain(cur, 1))
    assert moved and len(got) == len(want) == 14
    for x, y in zip(got, want):
        assert np.array_equal(_bits(x), _bits(y))
    assert b.statistics()["per_session"][1]["concealed"] == 2


# ------------------------------------------------------------------ refusals
def _call(g, packed, rows, anchors, zq, bf16=False):
    from audiodec_b200 import _lib
    lib = _lib.load()
    arr = (_lib.AdecConcealRow * len(rows))(*[_lib.AdecConcealRow(*r) for r in rows])
    fn = lib.adec_lookup_packed_conceal_bf16 if bf16 else lib.adec_lookup_packed_conceal
    rc = fn(g._h, ctypes.c_void_p(packed.data_ptr()), packed.shape[0], arr, len(rows), ctypes.c_void_p(anchors.data_ptr()),
            anchors.shape[0], ctypes.c_void_p(zq.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    return rc, _lib.last_error(g._h)


@pytest.mark.parametrize("rows,field", [
    ([(3, -1, -1, 0, 0)], r"rows\[0\]\.src = 3 is out of range"),
    ([(-2, 0, -1, 1, 2)], r"rows\[0\]\.src = -2"),
    ([(0, 1, -1, 0, 0)], r"rows\[0\]\.next = 1"),
    ([(-1, 3, -1, 1, 2)], r"rows\[0\]\.next = 3 is out of range"),
    ([(-1, -1, -1, 1, 2)], r"rows\[0\]\.next = -1 is out of range"),
    ([(0, -1, 2, 0, 0)], r"rows\[0\]\.slot = 2 is out of range"),
    ([(0, -1, 0, 0, 0), (-1, 0, -2, 1, 2)], r"rows\[1\]\.slot = -2 is out of range"),
    ([(-1, 0, 0, 1, 1)], r"rows\[0\]\.den = 1"),
    ([(-1, 0, 0, 0, 3)], r"rows\[0\]\.j = 0 is outside"),
    ([(-1, 0, 0, 3, 3)], r"rows\[0\]\.j = 3 is outside"),
    ([(0, -1, 1, 0, 0), (-1, 2, 1, 1, 2)], r"rows\[1\]\.slot = 1: anchor 1 is read by row 1 and written by row 0"),
    ([(-1, 2, 1, 1, 2), (0, -1, 1, 0, 0)], r"rows\[1\]\.slot = 1: anchor 1 is read by row 0 and written by row 1"),
    ([(0, -1, 0, 0, 0), (1, -1, 0, 0, 0)], r"rows\[1\]\.slot = 0: anchor 0 is written by rows 0 and 1"),
])
def test_bad_descriptors_are_refused_by_name(symad_sd, rows, field):
    g = _gen(symad_sd)
    packed = g.pack(torch.zeros(g.codebook_num, 3, dtype=torch.int64, device=DEV))
    anchors = torch.full((2, g.code_dim), 5.0, device=DEV)
    zq = torch.full((len(rows), g.code_dim), 7.0, device=DEV)
    launches = g.launch_count
    for bf16 in (False, True):
        rc, msg = _call(g, packed, rows, anchors, zq, bf16)
        assert rc != 0 and ("lookup_packed_conceal_bf16" if bf16 else "lookup_packed_conceal") in msg
        assert re.search(field, msg), msg
    assert g.launch_count == launches
    torch.cuda.synchronize()
    assert (anchors == 5.0).all() and (zq == 7.0).all()                           # nothing ran
    with pytest.raises(RuntimeError, match="rows"):
        g.lookup_packed_conceal(packed, rows, anchors)


def test_encoder_and_decoder_only_handles_refuse(symad_sd):
    from audiodec_b200.codec import SymADDecoderStreamGenerator, SymADEncoderStreamGenerator
    enc = SymADEncoderStreamGenerator(**S.SYMAD_PARAMS)
    enc.load_state_dict(symad_sd)
    enc = enc.eval().to(DEV)
    dec = SymADDecoderStreamGenerator(**S.SYMAD_PARAMS)
    dec.load_state_dict(symad_sd)
    dec = dec.eval().to(DEV)
    packed = torch.zeros(2, 10, dtype=torch.uint8, device=DEV)
    anchors = torch.zeros(1, 64, device=DEV)
    zq = torch.zeros(1, 64, device=DEV)
    for g, word in ((enc, "encoder-only"), (dec, "decoder-only")):
        for bf16 in (False, True):
            rc, msg = _call(g, packed, [(0, -1, 0, 0, 0)], anchors, zq, bf16)
            assert rc != 0 and word in msg and "lookup_packed_conceal" in msg, msg
        assert not hasattr(g, "lookup_packed_conceal")
