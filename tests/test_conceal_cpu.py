"""Receiver loss concealment without a GPU: ReceiverSessionServer(conceal_packets=K) on duck-typed stand-ins whose
lookup_packed_conceal is a numpy float32 model of the kernel.  Which sequence numbers are concealed and with how many frames, one
concealed packet per session per step before the packet after the gap, the samples delivered, the counters, late packets, a lost first
packet, detach / attach in the middle of a gap, and conceal_packets=0 unchanged.  Also the descriptor struct against the header."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from audiodec_b200 import wire
from audiodec_b200.server import ReceiverSessionServer

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NQ, NB = 8, 2          # the stand-ins' codebook count and packed bytes per frame
K = 2


def conceal_model(a, s_b, j, den):
    """the concealed zq in float32: fl(fl(fl(j / den) * fl(s_b - a)) + a); a None: s_b"""
    s_b = np.asarray(s_b, dtype=np.float32)
    if a is None:
        return s_b.copy()
    a = np.asarray(a, dtype=np.float32)
    w = np.float32(j) / np.float32(den)
    return (w * (s_b - a)) + a


# ------------------------------------------------------------------ stand-ins
class SlotState:
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


class FakeRx:
    """A frame's lookup sum is its first packed byte (code_dim 1).  lookup_packed_conceal checks the descriptors as the C ABI does and
    computes the rows with conceal_model."""
    codebook_num = NQ
    code_dim = 1

    def __init__(self):
        self.plain_calls = 0
        self.rows = []                                                # descriptors of every concealing lookup

    def packed_frame_bytes(self):
        return NB

    def lookup_packed(self, packed):
        self.plain_calls += 1
        return packed[..., :1].to(torch.float32)

    def lookup_packed_conceal(self, packed, rows, anchors):
        assert packed.dtype == torch.uint8 and packed.dim() == 2 and packed.shape[1] == NB
        assert rows.dtype == np.int32 and rows.shape[1] == 5 and anchors.dtype == torch.float32
        self.rows.append(rows.copy())
        f = packed.shape[0]
        sums = packed[:, 0].to(torch.float32).numpy()
        av = anchors.numpy()                                          # the same memory: stores go to the server's anchors
        written = {int(r[2]) for r in rows if r[0] >= 0 and r[2] >= 0}
        read = {int(r[2]) for r in rows if r[0] < 0 and r[2] >= 0}
        assert not written & read and len(written) == sum(1 for r in rows if r[0] >= 0 and r[2] >= 0)
        before = av.copy()
        out = np.empty((len(rows), 1), np.float32)
        for i, (src, nxt, slot, j, den) in enumerate(rows):
            if src >= 0:
                assert src < f and nxt == -1
                out[i] = sums[src]
                if slot >= 0:
                    av[slot] = sums[src]
            else:
                assert src == -1 and 0 <= nxt < f and den >= 2 and 1 <= j < den
                out[i] = conceal_model(before[slot] if slot >= 0 else None, sums[nxt:nxt + 1], j, den)
        return torch.from_numpy(out).view(1, -1, 1)


class FakeDec(SlotState):
    """Two samples per frame: (frames the slot decoded before it, its zq value)."""

    def __init__(self):
        super().__init__(0.0)
        self.calls = []

    def decode_streams(self, zq, frames, streams):
        self.calls.append((list(frames), list(streams)))
        out, o = [], 0
        for f, s in zip(frames, streams):
            pos = self.carry[s] + torch.arange(f, dtype=torch.float32)
            out.append(torch.stack([pos, zq.reshape(-1)[o:o + f]], 1).reshape(1, 1, -1))
            self.carry[s] += f
            o += f
        return out


def _rx(k=K, cap=3, fpp=4):
    rx, dec = FakeRx(), FakeDec()
    return ReceiverSessionServer(rx, dec, capacity=cap, frames_per_packet=fpp, sample_rate=8000, conceal_packets=k), rx, dec


def _pkt(sid, seq, codes):
    return wire.encode_packet(sid, seq, NQ, NB, bytes(b for c in codes for b in (c, NQ)))


def _drain(srv, sid):
    out = []
    while (y := srv.poll(sid)) is not None:
        out.append(y)
    return out


def _frames(ys):
    """decoded stand-in output -> [(slot position, zq)] per frame"""
    v = np.concatenate(ys).reshape(-1, 2) if ys else np.zeros((0, 2), np.float32)
    return [(int(p), np.float32(z)) for p, z in v]


def _codes(seq, frames):
    return [(7 * seq + 3 * i + 1) % 251 for i in range(frames)]


# ------------------------------------------------------------------ which sequence numbers, how many frames, in what order
@pytest.mark.parametrize("gap", [1, K, K + 3])
def test_the_last_k_lost_packets_are_concealed_with_the_next_packets_frame_count(gap):
    srv, rx, dec = _rx()
    srv.open(9)
    srv.submit_packet(_pkt(9, 0, _codes(0, 2)))
    assert srv.step() == 1 and len(_drain(srv, 9)) == 1
    w, b, fb = srv.reorder_window, 1 + gap, 3                        # b carries 3 frames, the others 2
    for q in range(b, b + w + 1):
        assert srv.submit_packet(_pkt(9, q, _codes(q, fb if q == b else 2)))
    c = min(gap, K)
    st = srv.statistics()["per_session"][9]
    assert st["losses"] == gap and st["concealed"] == 0                # given up, nothing decoded yet
    per_step = []
    while srv.step():
        per_step.append(_frames(_drain(srv, 9)))
    # one packet per step: c concealed packets of b's 3 frames, then b, then the rest in order
    assert [len(x) for x in per_step] == [fb] * c + [fb] + [2] * w
    m, a, s_b = c * fb, np.float32(_codes(0, 2)[-1]), np.float32(_codes(b, 1)[0])
    want = [conceal_model(a, s_b, j, m + 1) for j in range(1, m + 1)]
    got = [z for x in per_step[:c] for _, z in x]
    assert np.array_equal(np.asarray(got, np.float32).view(np.int32), np.asarray(want, np.float32).view(np.int32))
    assert [z for _, z in per_step[c]] == [np.float32(v) for v in _codes(b, fb)]
    pos = [p for x in per_step for p, _ in x]
    assert pos == list(range(2, 2 + len(pos)))                       # the decoder's state runs through the gap
    for rows in rx.rows[1:1 + c]:                                     # concealed rows read the slot's anchor, one staged frame
        assert (rows[:, 0] == -1).all() and (rows[:, 1] == 0).all() and (rows[:, 2] == srv._ids[9]).all()
        assert (rows[:, 4] == m + 1).all()
    assert np.concatenate([r[:, 3] for r in rx.rows[1:1 + c]]).tolist() == list(range(1, m + 1))
    st = srv.statistics()["per_session"][9]
    assert (st["losses"], st["concealed"], st["concealed_frames"]) == (gap, c, m)
    assert (st["packets"], st["frames"]) == (w + 2, 2 + fb + 2 * w)
    assert st["wire_kbps"] == pytest.approx(8e-3 * ((w + 2) * 16 + (2 + fb + 2 * w) * NB) / ((2 + fb + 2 * w) * 2 / 8000))


def test_concealed_packets_one_per_session_per_step_beside_other_sessions():
    srv, rx, dec = _rx()
    srv.open(1), srv.open(2)
    for sid in (1, 2):
        srv.submit_packet(_pkt(sid, 0, [sid]))
    srv.step()
    for q in range(3, 3 + srv.reorder_window + 1):                    # session 1 loses 1 and 2; session 2 loses nothing
        srv.submit_packet(_pkt(1, q, [q]))
    for q in range(1, 8):
        srv.submit_packet(_pkt(2, q, [10 + q]))
    assert srv.step() == 2
    assert dec.calls[-1] == ([1, 1], [srv._ids[1], srv._ids[2]])
    rows = rx.rows[-1]                                                # session 1: a concealed row on the one staged frame of b
    assert rows.tolist() == [[-1, 0, srv._ids[1], 1, 3], [1, -1, srv._ids[2], 0, 0]]
    assert srv.step() == 2 and rx.rows[-1].tolist() == [[-1, 0, srv._ids[1], 2, 3], [1, -1, srv._ids[2], 0, 0]]
    assert srv.step() == 2 and rx.rows[-1][0].tolist() == [0, -1, srv._ids[1], 0, 0]     # b, real again


# ------------------------------------------------------------------ samples and counters over random losses
def test_delivered_samples_are_sent_minus_lost_unconcealed():
    rng = np.random.default_rng(3)
    srv, _, _ = _rx(k=K)
    srv.open(4)
    n, fpp, w = 80, 2, srv.reorder_window
    lost = set()
    q = 2
    while q < n - w - 2:                                              # runs of 1 .. 4 losses, each followed by enough packets
        if rng.random() < 0.2:
            run = int(rng.integers(1, 5))
            lost.update(range(q, q + run))
            q += run + w + 1
        else:
            q += 1
    unconcealed, concealed, runs = 0, 0, []
    for q in sorted(lost):
        if q - 1 not in lost:
            runs.append(1)
        else:
            runs[-1] += 1
    for r in runs:
        concealed += min(r, K)
        unconcealed += r - min(r, K)
    delivered = 0
    for q in (q for q in range(n) if q not in lost):
        srv.submit_packet(_pkt(4, q, _codes(q, fpp)))
        srv.step()
        delivered += sum(y.size for y in _drain(srv, 4))
    while srv.step():
        delivered += sum(y.size for y in _drain(srv, 4))
    hop = 2
    assert delivered == (n - unconcealed) * fpp * hop
    st = srv.statistics()["per_session"][4]
    assert (st["losses"], st["concealed"], st["concealed_frames"]) == (len(lost), concealed, concealed * fpp)
    assert (st["packets"], st["frames"]) == (n - len(lost), (n - len(lost)) * fpp)
    assert len(runs) >= 3 and unconcealed > 0


def test_late_packet_for_a_concealed_sequence_number_is_a_duplicate():
    srv, _, _ = _rx()
    srv.open(1)
    srv.submit_packet(_pkt(1, 0, [5]))
    srv.step()
    for q in range(2, 3 + srv.reorder_window):
        srv.submit_packet(_pkt(1, q, [q]))
    assert not srv.submit_packet(_pkt(1, 1, [1]))                     # given up, concealment pending
    srv.step()
    assert not srv.submit_packet(_pkt(1, 1, [1]))                     # concealed already
    while srv.step():
        pass
    st = srv.statistics()["per_session"][1]
    assert (st["duplicates"], st["concealed"], st["losses"], st["packets"]) == (2, 1, 1, 1 + srv.reorder_window + 1)


def test_a_lost_first_packet_is_concealed_without_an_anchor():
    srv, rx, _ = _rx()
    srv.open(6)
    for q in range(1, 2 + srv.reorder_window):
        srv.submit_packet(_pkt(6, q, [40 + q, 50 + q]))
    srv.step()
    assert rx.rows[-1].tolist() == [[-1, 0, -1, 1, 3], [-1, 0, -1, 2, 3]]
    assert _frames(_drain(srv, 6)) == [(0, np.float32(41)), (1, np.float32(41))]
    srv.step()
    assert rx.rows[-1].tolist() == [[0, -1, -1, 0, 0], [1, -1, srv._ids[6], 0, 0]]


# ------------------------------------------------------------------ migration
def test_detach_attach_in_the_middle_of_a_gap_changes_nothing():
    ref, _, _ = _rx(k=3)
    a, _, _ = _rx(k=3)
    b, _, _ = _rx(k=3)
    for srv in (ref, a):
        srv.open(8)
    b.open(1)                                                         # the destination serves someone: session 8 gets another slot
    traffic = [q for q in range(14) if q not in (2, 3, 4, 5)]         # a gap of 4: the last 3 concealed
    got, want = [], []
    cur = a
    for k, q in enumerate(traffic):
        for srv in (ref, cur):
            srv.submit_packet(_pkt(8, q, _codes(q, 2)))
            srv.step()
        want.extend(_drain(ref, 8))
        if cur is a and a._plan[a._ids[8]] is not None and a._plan[a._ids[8]][2] > 0:
            slot = a._ids[8]
            st = a.detach(8)                                          # one concealed packet decoded, two to come, one unpolled
            assert st.anchor is not None and st.anchor.tolist() == [np.float32(_codes(1, 2)[-1])]
            assert st.conceal == (2, 2, 2, 6) and len(st.outputs) == 1
            assert b.attach(st) == 8 and b._ids[8] != slot
            cur = b
        else:
            got.extend(_drain(cur, 8))
    for srv in (ref, cur):
        while srv.step():
            pass
    want.extend(_drain(ref, 8))
    got.extend(_drain(cur, 8))
    assert cur is b
    assert _frames(got) == _frames(want) and len(_frames(got)) == 2 * (len(traffic) + 3)
    assert b.statistics()["per_session"][8]["concealed"] == 2


def test_a_session_from_a_receiver_without_concealment_attaches_without_anchor():
    a, _, _ = _rx(k=0)
    b, rx, _ = _rx(k=2)
    a.open(3)
    a.submit_packet(_pkt(3, 0, [9]))
    a.step()
    st = a.detach(3)
    assert st.anchor is None and st.conceal is None
    b.attach(st)
    for q in range(2, 3 + b.reorder_window):
        b.submit_packet(_pkt(3, q, [q]))
    b.step()
    assert rx.rows[-1][0].tolist() == [-1, 0, -1, 1, 2]               # no anchor: the concealed frame is s_b


# ------------------------------------------------------------------ concealment off is today's receiver
def test_conceal_off_is_unchanged_on_the_loss_traffic():
    srv, rx, dec = _rx(k=0)
    srv.open(9)
    srv.submit_packet(_pkt(9, 0, [0, 0]))
    srv.step()
    w = srv.reorder_window
    for q in range(3, 3 + w + 1):
        srv.submit_packet(_pkt(9, q, [q, q]))
    assert srv.statistics()["per_session"][9]["losses"] == 2
    assert not srv.submit_packet(_pkt(9, 1, [1, 1]))
    while srv.step():
        pass
    got = _frames(_drain(srv, 9))
    assert got == [(k, np.float32(c)) for k, c in enumerate(c for q in [0] + list(range(3, 4 + w)) for c in (q, q))]
    st = srv.statistics()["per_session"][9]
    assert (st["packets"], st["losses"], st["duplicates"], st["concealed"], st["concealed_frames"]) == (w + 2, 2, 1, 0, 0)
    n = 4 + w
    srv.submit_packet(_pkt(9, n, [1]))
    for q in range(n + 2, n + 3 + w):
        srv.submit_packet(_pkt(9, q, [2]))
    assert srv.step() == 1 and srv.statistics()["per_session"][9]["losses"] == 2
    assert srv.step() == 1 and srv.statistics()["per_session"][9]["losses"] == 3
    assert rx.rows == [] and rx.plain_calls == len(dec.calls) and srv._anchors is None
    assert srv.detach(9).anchor is None


def test_conceal_packets_must_not_be_negative():
    with pytest.raises(ValueError, match="conceal_packets"):
        _rx(k=-1)


# ------------------------------------------------------------------ the C ABI's descriptor
def test_conceal_row_struct_matches_header():
    from audiodec_b200 import _lib
    hdr = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    body = hdr[hdr.index("typedef struct adec_conceal_row {"):hdr.index("} adec_conceal_row;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"int32_t\s+(\w+);", body) == [f[0] for f in _lib.AdecConcealRow._fields_]
    assert ctypes.sizeof(_lib.AdecConcealRow) == 20
    for name in ("adec_lookup_packed_conceal", "adec_lookup_packed_conceal_bf16"):
        m = re.search(name + r"\s*\(([^)]*)\)", hdr)
        assert m and len(_lib.SYMBOLS[name][1]) == len(m.group(1).split(",")), name
