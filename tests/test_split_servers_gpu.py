"""TransmitterSessionServer -> wire packets -> ReceiverSessionServer against SessionCodecServer(wire=True) on the same frames: the PCM
bit for bit and the packets' payloads byte for byte, in every receiver dtype mode and transmitter modes 0 and 2, with sessions
opening and closing, idle steps, and packets shuffled across sessions and reordered within the window.  Sessions moved between
transmitter servers and between receiver servers mid-call change nothing.  A dropped packet is reported and the rest decode as a
decoder fed only the frames received."""
import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S
from audiodec_b200 import wire

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FS = 1500                              # 5 frames of hop 300 per packet
RATE = {"vctk_sym": 48000, "libritts_v1": 24000}


def _tx(sd, kind):
    """kind: 'full' (SymADStreamGenerator), 'enc0' / 'enc2' (encoder-only, fp32 / bf16 activations)"""
    from audiodec_b200.codec import SymADEncoderStreamGenerator, SymADStreamGenerator
    g = (SymADStreamGenerator if kind == "full" else SymADEncoderStreamGenerator)(**S.SYMAD_PARAMS)
    g.load_state_dict(sd)
    if kind == "enc2":
        g = g.set_activation_dtype(torch.bfloat16)
    g = g.eval().to(DEV)
    g.initial_encoder(8192, DEV)
    return g


def _rx(model, symad_sd, hifigan_sd, mode):
    """rx_encoder (codebooks) and a decoder in dtype mode 0 / 1 / 2, warmed as load_receiver leaves them"""
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADDecoderStreamGenerator, SymADStreamGenerator
    rx = SymADStreamGenerator(**S.SYMAD_PARAMS)
    rx.load_state_dict(symad_sd)
    rx = rx.eval().to(DEV)
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


def _split(model, symad_sd, hifigan_sd, tx_kind, mode, cap):
    from audiodec_b200.server import ReceiverSessionServer, TransmitterSessionServer
    txs = TransmitterSessionServer(_tx(symad_sd, tx_kind), capacity=cap, frame_size=FS, sample_rate=RATE[model], max_latency=10.0,
                                   device=DEV)
    rxs = ReceiverSessionServer(*_rx(model, symad_sd, hifigan_sd, mode), capacity=cap, frames_per_packet=FS // 300,
                                sample_rate=RATE[model], device=DEV)
    return txs, rxs


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


def _drain(srv, sid):
    out = []
    while (y := srv.poll(sid)) is not None:
        out.append(y)
    return out


CASES = [("vctk_sym", "full", 0), ("vctk_sym", "enc0", 1), ("vctk_sym", "enc2", 2),
         ("libritts_v1", "full", 0), ("libritts_v1", "enc2", 1), ("libritts_v1", "enc0", 2)]


@pytest.mark.parametrize("model,tx_kind,mode", CASES)
def test_loopback_equality(symad_sd, hifigan_sd, model, tx_kind, mode):
    from audiodec_b200.server import SessionCodecServer
    cap, steps = 5, 12
    rx_enc, dec = _rx(model, symad_sd, hifigan_sd, mode)
    loop = SessionCodecServer(_tx(symad_sd, tx_kind), rx_enc, dec, capacity=cap, frame_size=FS, sample_rate=RATE[model],
                              max_latency=10.0, device=DEV, wire=True)
    fused = []                                              # the loopback's fused-RVQ bytes, step by step
    orig = loop.tx_encoder.quantize_fused

    def record(z, **kw):
        out = orig(z, **kw)
        fused.append(out[1].cpu().numpy())
        return out
    loop.tx_encoder.quantize_fused = record
    txs, rxs = _split(model, symad_sd, hifigan_sd, tx_kind, mode, cap + 3)

    rng = np.random.default_rng(11)
    slot, sent, want, got = {}, {}, {}, {}                  # per wire session id
    closing, delayed, highest = set(), [], {}
    next_sid, inversions = 100, 0
    for k in range(steps):
        if k in (0, 3, 7):                                  # sessions open at different steps
            for _ in range(3 if k == 0 else 2):
                if len(slot) < cap:
                    sid, next_sid = next_sid, next_sid + 7
                    slot[sid] = loop.open()
                    txs.open(sid)
                    rxs.open(sid)
                    sent[sid], want[sid], got[sid] = 0, [], []
        fed = []
        for sid, s in slot.items():
            if rng.random() < 0.3:
                continue                                    # no audio for this session this step
            x = (0.1 * rng.standard_normal(FS)).astype(np.float32)
            loop.submit(s, x)
            txs.submit(sid, x)
            fed.append((s, sid))
        n_fused = len(fused)
        loop.step()
        txs.step()
        for sid, s in slot.items():
            want[sid].extend(_drain(loop, s))
        packets = txs.poll_packets()
        assert sorted(sid for sid, _ in packets) == sorted(sid for _, sid in fed)
        if fed:                                             # payloads = the loopback's fused-RVQ bytes, session by session
            rows = fused[n_fused].reshape(len(fed), FS // 300, -1)
            order = {sid: i for i, (_, sid) in enumerate(sorted(fed))}
            for sid, buf in packets:
                p = wire.decode_packet(buf)
                assert p.seq == sent[sid] and p.frames == FS // 300
                assert p.payload == rows[order[sid]].tobytes(), (k, sid)
                sent[sid] += 1
        # the network: this step's packets shuffled across sessions, some held back a step (reordered within the window)
        now, later = [], []
        for i in rng.permutation(len(packets)):
            (later if rng.random() < 0.3 else now).append(packets[i][1])
        for buf in delayed + now if rng.random() < 0.5 else now + delayed:
            p = wire.decode_packet(buf)
            inversions += p.seq < highest.get(p.session_id, -1)
            highest[p.session_id] = max(p.seq, highest.get(p.session_id, -1))
            assert rxs.submit_packet(buf)
        delayed = later
        rxs.step()
        for sid in rxs.open_sessions:
            got[sid].extend(_drain(rxs, sid))
        if k in (4, 9) and slot:                            # a session ends: the loopback and the transmitter close it now
            sid = sorted(slot)[k % len(slot)]
            loop.close(slot.pop(sid))
            txs.close(sid)
            closing.add(sid)
        for sid in list(closing):                           # the receiver once it has decoded everything sent
            if rxs.statistics()["per_session"][sid]["packets"] == sent[sid]:
                got[sid].extend(_drain(rxs, sid))
                rxs.close(sid)
                closing.discard(sid)
    for buf in delayed:
        rxs.submit_packet(buf)
    while rxs.step():
        pass
    st = rxs.statistics()
    for sid in got:
        if sid in rxs.open_sessions:
            got[sid].extend(_drain(rxs, sid))
            ps = st["per_session"][sid]
            assert ps["losses"] == 0 and ps["duplicates"] == 0 and ps["packets"] == sent[sid]
    assert st["unknown_session_packets"] == 0
    assert inversions > 0
    assert len(got) >= 6 and sum(len(v) for v in want.values()) > 20
    for sid in got:
        assert len(got[sid]) == len(want[sid]) == sent[sid], sid
        for a, b in zip(got[sid], want[sid]):
            assert a.dtype == b.dtype == np.float32 and a.shape == b.shape == (FS,)
            assert np.array_equal(_bits(a), _bits(b)), (model, tx_kind, mode, sid)


def test_sessions_migrate_between_transmitters_and_between_receivers(symad_sd, hifigan_sd):
    """session 1 moves from transmitter a to b with a frame queued, session 2 from receiver a to b with a packet held out of order
    and two frames not yet polled: both come out bit for bit as through one transmitter and one receiver"""
    model, mode = "libritts_v1", 2
    tx0, rx0 = _split(model, symad_sd, hifigan_sd, "full", mode, 4)        # nothing moves
    txa, rxa = _split(model, symad_sd, hifigan_sd, "full", mode, 4)
    txb, rxb = _split(model, symad_sd, hifigan_sd, "full", mode, 4)
    for srv in (tx0, rx0, txa, rxa):
        for sid in (1, 2):
            srv.open(sid)
    txb.open(9), rxb.open(9)                                # the destinations already serve someone
    rng = np.random.default_rng(4)
    tx_of, rx_of = {1: txa, 2: txa}, {1: rxa, 2: rxa}
    ref, got = {1: [], 2: []}, {1: [], 2: []}
    late = None
    for k in range(9):
        for sid in (1, 2):
            x = (0.1 * rng.standard_normal(FS)).astype(np.float32)
            tx0.submit(sid, x)
            tx_of[sid].submit(sid, x)
        if k == 3:
            for sid in (1, 2):                              # a backlog of one frame, so the moved session carries a queued frame
                tx0.submit(sid, np.zeros(FS, np.float32))
                tx_of[sid].submit(sid, np.zeros(FS, np.float32))
            st = txa.detach(1)
            assert st.session_id == 1 and st.seq == 3 and len(st.inputs) == 2
            assert txb.attach(st.to(DEV)) == 1
            tx_of[1] = txb
        for t in (tx0, txa, txb):
            t.step()
        for _, buf in tx0.poll_packets():
            rx0.submit_packet(buf)
        for sid, buf in txa.poll_packets() + txb.poll_packets():
            if sid == 2 and k == 5:
                late = buf                                  # session 2's packet 5 is late: it reaches receiver b after packet 6
                continue
            assert rx_of[sid].submit_packet(buf)
        if k == 6:
            st = rxa.detach(2)
            assert st.session_id == 2 and st.seq == 5 and [p.seq for p in st.inputs] == [6] and len(st.outputs) == 2
            assert rxb.attach(st.to(DEV)) == 2
            rx_of[2] = rxb
            assert rxb.submit_packet(late)
        for r in (rx0, rxa, rxb):
            r.step()
        for sid in (1, 2):
            ref[sid].extend(_drain(rx0, sid))
            if sid == 1 or k not in (3, 4, 5):              # session 2's frames 3 and 4 wait unpolled and travel with it
                got[sid].extend(_drain(rx_of[sid], sid))
    for t in (tx0, txa, txb):                               # the backlog frame
        t.step()
        for sid, buf in t.poll_packets():
            (rx0 if t is tx0 else rx_of[sid]).submit_packet(buf)
    for r in (rx0, rxa, rxb):
        while r.step():
            pass
    for sid in (1, 2):
        ref[sid].extend(_drain(rx0, sid))
        got[sid].extend(_drain(rx_of[sid], sid))
        assert len(got[sid]) == len(ref[sid]) == 10, (sid, len(got[sid]), len(ref[sid]))
        for a, b in zip(got[sid], ref[sid]):
            assert np.array_equal(_bits(a), _bits(b)), sid
    st = rxb.statistics()["per_session"][2]
    assert st["losses"] == 0 and st["reorders"] == 1 and st["packets"] == 5


@pytest.mark.parametrize("mode", [0, 2])
def test_loss_is_reported_and_the_rest_decodes(symad_sd, hifigan_sd, mode):
    model = "libritts_v1"
    txs, rxs = _split(model, symad_sd, hifigan_sd, "enc0", mode, 3)
    ref_rx, ref_dec = _rx(model, symad_sd, hifigan_sd, mode)
    txs.open(5), rxs.open(5)
    rng = np.random.default_rng(8)
    n, lost = 6 + rxs.reorder_window, 2
    for _ in range(n):
        txs.submit(5, (0.1 * rng.standard_normal(FS)).astype(np.float32))
        txs.step()
    packets = [buf for _, buf in txs.poll_packets()]
    for q, buf in enumerate(packets):
        if q != lost:
            rxs.submit_packet(buf)
    got = []
    while rxs.step():
        got.extend(_drain(rxs, 5))
    st = rxs.statistics()["per_session"][5]
    assert st["losses"] == 1 and st["packets"] == n - 1 and st["frames"] == (n - 1) * (FS // 300)
    # a decoder fed only the frames received, packet by packet
    dt = torch.bfloat16 if mode == 2 else torch.float32
    want = []
    for q, buf in enumerate(packets):
        if q == lost:
            continue
        p = wire.decode_packet(buf)
        packed = torch.frombuffer(bytearray(p.payload), dtype=torch.uint8).view(1, p.frames, -1).to(DEV)
        y = ref_dec.decode_streams(ref_rx.lookup_packed(packed, dtype=dt), [p.frames], [0])[0]
        want.append(y.float().reshape(-1).cpu().numpy())
    assert len(got) == len(want) == n - 1
    for a, b in zip(got, want):
        assert np.array_equal(_bits(a), _bits(b))
