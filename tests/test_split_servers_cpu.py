"""The wire packet (audiodec_b200.wire) and the split session servers without a GPU: packet round trip and every malformed header, and
TransmitterSessionServer / ReceiverSessionServer on duck-typed stand-ins: packets per step, in-order delivery, duplicates, reordering
within the window, losses past it, packets for unknown or closed sessions, and detach / attach on both sides."""
import struct

import numpy as np
import pytest
import torch

from audiodec_b200 import wire
from audiodec_b200.server import ReceiverSessionServer, SessionState, TransmitterSessionServer

NQ, NB = 8, 2          # the stand-ins' codebook count and packed bytes per frame


# ------------------------------------------------------------------ packets
def test_packet_round_trip_and_layout():
    payload = bytes(range(3 * 10))
    buf = wire.encode_packet(0xDEADBEEF, 7, 8, 10, payload)
    assert len(buf) == wire.HEADER_BYTES + 30 == 46
    assert buf[:2] == b"AD" and buf[2] == 1 and buf[3] == 8
    assert struct.unpack_from("<IIHH", buf, 4) == (0xDEADBEEF, 7, 3, 10)
    assert buf[16:] == payload
    p = wire.decode_packet(buf, codebook_num=8, frame_bytes=10)
    assert p == wire.Packet(0xDEADBEEF, 7, 3, 8, 10, payload)
    assert wire.decode_packet(bytearray(buf)) == p                      # any bytes-like buffer
    assert wire.decode_packet(np.frombuffer(buf, np.uint8)) == p


def test_encode_rejects_what_the_header_cannot_hold():
    for args, field in (((1 << 32, 0, 8, 10, bytes(10)), "session_id"), ((0, -1, 8, 10, bytes(10)), "seq"),
                        ((0, 0, 256, 10, bytes(10)), "codebook_num"), ((0, 0, 8, 0, b""), "frame_bytes"),
                        ((0, 0, 8, 10, bytes(15)), "payload"), ((0, 0, 8, 10, b""), "payload")):
        with pytest.raises(ValueError, match=field):
            wire.encode_packet(*args)


def _hdr(magic=b"AD", version=1, nq=8, sid=1, seq=0, frames=2, nb=10):
    return struct.pack("<2sBBIIHH", magic, version, nq, sid, seq, frames, nb)


@pytest.mark.parametrize("buf,field", [
    (b"", "header"),
    (_hdr()[:15], "header"),
    (_hdr(magic=b"XD") + bytes(20), "magic"),
    (_hdr(version=2) + bytes(20), "version"),
    (_hdr(version=0) + bytes(20), "version"),
    (_hdr() + bytes(19), "payload"),
    (_hdr() + bytes(21), "payload"),
    (_hdr(), "payload"),
    (_hdr(frames=0), "frames"),
    (_hdr(nq=16) + bytes(20), "codebook_num"),
    (_hdr(nb=20) + bytes(40), "frame_bytes"),
])
def test_malformed_packets_raise_value_error(buf, field):
    with pytest.raises(ValueError, match=field):
        wire.decode_packet(buf, codebook_num=8, frame_bytes=10)


def test_unchecked_codec_fields_still_check_the_buffer():
    assert wire.decode_packet(_hdr(nq=16) + bytes(20)).codebook_num == 16
    with pytest.raises(ValueError, match="frames"):
        wire.decode_packet(_hdr(frames=1, nb=0))


# ------------------------------------------------------------------ stand-ins
class SlotState:
    """Per-slot float state with the generators' slot and state calls."""
    state_layout = [("pad_buffer", 1, 1)]

    def __init__(self, warm):
        self.carry = torch.tensor([float(warm)])

    @property
    def n_streams(self):
        return self.carry.numel()

    def set_streams(self, n):
        self.carry = self.carry.repeat(n)

    def copy_stream_state(self, src, dst):
        for d in dst:
            self.carry[d] = self.carry[src]

    def stream_state(self, streams):
        return self.carry[list(streams)].view(-1, 1).clone()

    def load_stream_state(self, streams, state, layout=None):
        self.carry[list(streams)] = state.view(-1)


class FakeTx(SlotState):
    """One code frame per sample; code = sample + carry[slot] (mod 256), carry[slot] = last sample.  A frame packs to (code, NQ)."""
    codebook_num = NQ

    def __init__(self):
        super().__init__(3.0)
        self.calls = []

    def encode_streams(self, chunks, streams):
        self.calls.append(list(streams))
        out = []
        for x, s in zip(chunks, streams):
            out.append(x + self.carry[s])
            self.carry[s] = x[-1]
        return torch.cat(out).view(1, 1, -1), [c.numel() for c in chunks]

    def quantize_fused(self, z, want_idx, want_packed, want_zq):
        assert (want_idx, want_packed, want_zq) == (False, True, False)
        code = z.reshape(-1).round().to(torch.int64) % 256
        return None, torch.stack([code, torch.full_like(code, NQ)], 1).to(torch.uint8), None


class FakeRx:
    codebook_num = NQ

    def packed_frame_bytes(self):
        return NB

    def lookup_packed(self, packed):
        assert packed.dtype == torch.uint8 and packed.shape[0] == 1 and packed.shape[2] == NB
        return packed[..., :1].to(torch.float32)                         # (1, F, 1)


class FakeDec(SlotState):
    """Two samples per frame: y = 1000 * (frames decoded by the slot so far) + code, so the output shows the order of decoding."""

    def __init__(self):
        super().__init__(0.0)
        self.calls = []

    def decode_streams(self, zq, frames, streams):
        self.calls.append((list(frames), list(streams)))
        out, o = [], 0
        for f, s in zip(frames, streams):
            pos = self.carry[s] + torch.arange(f, dtype=torch.float32)
            y = 1000.0 * pos + zq.reshape(-1)[o:o + f]
            out.append(y.repeat_interleave(2).view(1, 1, -1))
            self.carry[s] += f
            o += f
        return out


def _rx(cap=3, fpp=4):
    dec = FakeDec()
    return ReceiverSessionServer(FakeRx(), dec, capacity=cap, frames_per_packet=fpp, sample_rate=8000), dec


def _pkt(sid, seq, codes):
    return wire.encode_packet(sid, seq, NQ, NB, bytes(b for c in codes for b in (c, NQ)))


def _drain(srv, sid):
    out = []
    while (y := srv.poll(sid)) is not None:
        out.append(y)
    return out


def _frames(ys):
    """decoded stand-in output -> [(slot position, code)] per frame"""
    v = np.concatenate(ys)[::2] if ys else np.zeros(0)
    return [(int(x) // 1000, int(x) % 1000) for x in v]


# ------------------------------------------------------------------ receiver ordering
def test_in_order_delivery_one_packet_per_session_per_step():
    srv, dec = _rx()
    a, b = srv.open(70), srv.open(5)
    assert (a, b) == (70, 5) and srv.open_sessions == [5, 70]
    for k in range(3):
        assert srv.submit_packet(_pkt(70, k, [10 + k, 20 + k]))
    assert srv.submit_packet(_pkt(5, 0, [1, 2, 3]))
    assert srv.step() == 2
    assert dec.calls[-1] == ([3, 2], [srv._ids[5], srv._ids[70]])     # sessions in id order, each with its own frame count
    assert srv.step() == 1 and srv.step() == 1 and srv.step() == 0
    ys = _drain(srv, 70)
    assert len(ys) == 3 and all(y.dtype == np.float32 and y.size == 4 for y in ys)
    assert _frames(ys) == [(0, 10), (1, 20), (2, 11), (3, 21), (4, 12), (5, 22)]
    assert _frames(_drain(srv, 5)) == [(0, 1), (1, 2), (2, 3)]
    st = srv.statistics()["per_session"][70]
    assert (st["packets"], st["frames"], st["duplicates"], st["reorders"], st["losses"]) == (3, 6, 0, 0, 0)
    # 3 packets of 16 + 4 bytes over 6 frames x 2 samples at 8 kHz
    assert st["wire_kbps"] == pytest.approx(8e-3 * 60 / (12 / 8000))


def test_duplicates_are_dropped():
    srv, _ = _rx()
    srv.open(1)
    assert srv.submit_packet(_pkt(1, 0, [1]))
    assert not srv.submit_packet(_pkt(1, 0, [9]))                     # held already
    srv.step()
    assert not srv.submit_packet(_pkt(1, 0, [9]))                     # decoded already
    assert srv.submit_packet(_pkt(1, 2, [3]))
    assert not srv.submit_packet(_pkt(1, 2, [9]))
    assert srv.submit_packet(_pkt(1, 1, [2]))
    srv.step(), srv.step()
    assert _frames(_drain(srv, 1)) == [(0, 1), (1, 2), (2, 3)]
    st = srv.statistics()["per_session"][1]
    assert st["duplicates"] == 3 and st["packets"] == 3 and st["losses"] == 0


def test_reordering_within_the_window():
    srv, _ = _rx()
    srv.open(4)
    order = [1, 3, 0, 2, 4]                                           # never more than reorder_window held behind a gap
    for q in order:
        assert srv.submit_packet(_pkt(4, q, [q]))
    assert srv.step() == 1
    while srv.step():
        pass
    assert _frames(_drain(srv, 4)) == [(k, k) for k in range(5)]
    st = srv.statistics()["per_session"][4]
    assert st["reorders"] == 2 and st["losses"] == 0 and st["packets"] == 5


def test_held_packets_wait_for_a_missing_one():
    srv, _ = _rx()
    srv.open(4)
    for q in range(1, 1 + srv.reorder_window):
        srv.submit_packet(_pkt(4, q, [q]))
    assert srv.step() == 0 and srv.poll(4) is None                    # waiting for packet 0
    srv.submit_packet(_pkt(4, 0, [0]))
    while srv.step():
        pass
    assert _frames(_drain(srv, 4)) == [(k, k) for k in range(1 + srv.reorder_window)]


def test_loss_past_the_window():
    srv, dec = _rx()
    srv.open(9)
    srv.submit_packet(_pkt(9, 0, [0, 0]))
    srv.step()
    w = srv.reorder_window
    for q in range(3, 3 + w + 1):                                     # 1 and 2 never come: w + 1 packets held behind them
        srv.submit_packet(_pkt(9, q, [q, q]))
    assert srv.statistics()["per_session"][9]["losses"] == 2
    assert not srv.submit_packet(_pkt(9, 1, [1, 1]))                  # too late: given up
    while srv.step():
        pass
    # no concealment: the decoder advanced only by the frames received, 2 per packet
    got = _frames(_drain(srv, 9))
    assert got == [(k, c) for k, c in enumerate(c for q in [0] + list(range(3, 4 + w)) for c in (q, q))]
    st = srv.statistics()["per_session"][9]
    assert (st["packets"], st["losses"], st["duplicates"]) == (w + 2, 2, 1)
    # a gap that opens behind a packet still to be decoded is given up by the step that finds it
    n = 4 + w
    srv.submit_packet(_pkt(9, n, [1]))
    for q in range(n + 2, n + 3 + w):
        srv.submit_packet(_pkt(9, q, [2]))
    assert srv.step() == 1 and srv.statistics()["per_session"][9]["losses"] == 2
    assert srv.step() == 1 and srv.statistics()["per_session"][9]["losses"] == 3


def test_packets_for_unknown_or_closed_sessions():
    srv, _ = _rx()
    assert not srv.submit_packet(_pkt(3, 0, [1]))
    srv.open(3)
    srv.submit_packet(_pkt(3, 0, [1]))
    srv.submit_packet(_pkt(3, 1, [2]))
    srv.step()
    srv.close(3)
    assert not srv.submit_packet(_pkt(3, 2, [3]))
    assert srv.statistics()["unknown_session_packets"] == 2
    assert srv.step() == 0
    with pytest.raises(KeyError):
        srv.poll(3)
    srv.open(3)                                                       # the id opens again as a new session, from the template
    assert srv.submit_packet(_pkt(3, 0, [7]))
    srv.step()
    assert _frames(_drain(srv, 3)) == [(0, 7)]


def test_receiver_rejections():
    srv, _ = _rx(cap=1, fpp=2)
    srv.open(1)
    with pytest.raises(ValueError, match="already open"):
        srv.open(1)
    with pytest.raises(RuntimeError, match="full"):
        srv.open(2)
    with pytest.raises(ValueError, match="frames"):
        srv.submit_packet(_pkt(1, 0, [1, 2, 3]))                      # more than frames_per_packet
    with pytest.raises(ValueError, match="frame_bytes"):
        srv.submit_packet(wire.encode_packet(1, 0, NQ, 3, bytes(3)))
    with pytest.raises(ValueError, match="codebook_num"):
        srv.submit_packet(wire.encode_packet(1, 0, 16, NB, bytes(2)))
    with pytest.raises(ValueError, match="magic"):
        srv.submit_packet(b"XX" + _pkt(1, 0, [1])[2:])
    assert srv.statistics()["per_session"][1]["packets"] == 0


def test_receiver_detach_attach_moves_state_held_packets_and_frames():
    a, da = _rx()
    b, db = _rx()
    a.open(8), b.open(1)
    for q in (0, 1, 3):
        a.submit_packet(_pkt(8, q, [q, q]))
    a.step()                                                          # packet 0 decoded, not polled; 1 and 3 held
    st = a.detach(8)
    assert st.session_id == 8 and st.seq == 1 and [p.seq for p in st.inputs] == [1, 3] and len(st.outputs) == 1
    assert a.open_sessions == []
    with pytest.raises(ValueError, match="wire session id"):
        b.attach(SessionState(st.layouts, st.states, [], []))
    assert b.attach(st) == 8 and b.open_sessions == [1, 8]
    b.submit_packet(_pkt(8, 2, [2, 2]))
    while b.step():
        pass
    assert _frames(_drain(b, 8)) == [(k, q) for k, q in enumerate(q for q in range(4) for _ in range(2))]
    assert b.statistics()["per_session"][8]["packets"] == 3


# ------------------------------------------------------------------ transmitter
def _tx(cap=3):
    tx = FakeTx()
    return TransmitterSessionServer(tx, capacity=cap, frame_size=4, sample_rate=8000, max_latency=1.0), tx


def test_transmitter_packets_per_step():
    srv, tx = _tx()
    srv.open(20), srv.open(10), srv.open(30)
    with pytest.raises(ValueError, match="already open"):
        srv.open(10)
    srv.submit(20, np.full(4, 1.0, np.float32))
    srv.submit(10, np.full(4, 2.0, np.float32))
    assert srv.step() == 2
    assert tx.calls[-1] == [srv._ids[10], srv._ids[20]]               # no silence for the idle session 30
    srv.submit(20, np.full(4, 5.0, np.float32))
    assert srv.step() == 1 and srv.step() == 0
    pk = srv.poll_packets()
    assert [sid for sid, _ in pk] == [10, 20, 20] and srv.poll_packets() == []
    ps = [wire.decode_packet(b, NQ, NB) for _, b in pk]
    assert [(p.session_id, p.seq, p.frames) for p in ps] == [(10, 0, 4), (20, 0, 4), (20, 1, 4)]
    assert ps[1].payload == bytes([4, NQ] * 4)                        # 1 + the template's warm carry 3
    assert ps[2].payload == bytes([6, NQ] * 4)                        # 5 + carry 1
    st = srv.statistics()
    assert st["per_session"][20]["n_frames"] == 2 and st["per_session"][30]["underruns"] == 3
    assert st["wire_bytes"] == 3 * (16 + 8)


def test_transmitter_detach_attach_keeps_sequence_and_state():
    a, _ = _tx()
    b, _ = _tx()
    a.open(5)
    b.open(6)
    a.submit(5, np.full(4, 1.0, np.float32))
    a.step()
    a.submit(5, np.full(4, 2.0, np.float32))
    st = a.detach(5)
    assert st.session_id == 5 and st.seq == 1 and len(st.inputs) == 1 and st.outputs == []
    with pytest.raises(KeyError):
        a.submit(5, np.zeros(4, np.float32))
    assert b.attach(st) == 5 and b.pending(5) == 1
    b.step()
    (sid, buf), = [p for p in b.poll_packets() if p[0] == 5]
    p = wire.decode_packet(buf)
    assert p.seq == 1 and p.payload == bytes([3, NQ] * 4)            # 2 + the moved carry 1
    with pytest.raises(ValueError, match="already open"):
        b.attach(st)


def test_transmitter_to_receiver_on_stand_ins():
    """packets shuffled across sessions reach the receiver, which gives each session its frames in order"""
    tx_srv, _ = _tx()
    rx_srv, _ = _rx(fpp=4)
    for sid in (1, 2):
        tx_srv.open(sid), rx_srv.open(sid)
    rng = np.random.default_rng(0)
    sent = {1: [], 2: []}
    for k in range(6):
        for sid in (1, 2):
            if (k + sid) % 3:
                f = np.full(4, float(10 * sid + k), np.float32)
                tx_srv.submit(sid, f)
                sent[sid].append(f)
        tx_srv.step()
    pk = tx_srv.poll_packets()
    for i in rng.permutation(len(pk)):
        rx_srv.submit_packet(pk[i][1])
    while rx_srv.step():
        pass
    for sid in (1, 2):
        got = _frames(_drain(rx_srv, sid))
        assert len(got) == 4 * len(sent[sid])
        assert [pos for pos, _ in got] == list(range(len(got)))
        assert rx_srv.statistics()["per_session"][sid]["losses"] == 0
