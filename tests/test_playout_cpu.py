"""The receiver's playout clock without a GPU: ReceiverSessionServer(playout_delay=D) on duck-typed stand-ins whose
lookup_packed_playout is a numpy float32 model of the kernel's three row kinds.  When a session starts playing, jitter within D, the
three per-step rules and their j / den, late against duplicate packets, pause and rewind, a lost first packet, detach / attach while
buffering, in the middle of a gap and in the middle of a fade, the ValueErrors, and the descriptor struct and tables."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from audiodec_b200 import server as server_mod
from audiodec_b200 import wire
from audiodec_b200.server import ReceiverSessionServer

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NQ, NB = 8, 2          # the stand-ins' codebook count and packed bytes per frame
SILENCE = np.float32(-3.0)


def interp(a, t, j, den):
    """fl(fl(fl(j / den) * fl(t - a)) + a) in float32"""
    a, t = np.float32(a), np.float32(t)
    return (np.float32(j) / np.float32(den)) * (t - a) + a


def playout_model(rows, sums, anchors, targets):
    """the kernel's rows in float32: real, interpolated (toward frame next) and fade (toward targets[target]) -> (R, D), and the anchor
    stores of the real rows"""
    before = anchors.copy()
    out = np.empty((len(rows), anchors.shape[1]), np.float32)
    for i, (src, nxt, tgt, slot, j, den) in enumerate(rows):
        if src >= 0:
            out[i] = sums[src]
            if slot >= 0:
                anchors[slot] = sums[src]
        elif nxt >= 0:
            out[i] = sums[nxt] if slot < 0 else interp(before[slot], sums[nxt], j, den)
        else:
            out[i] = targets[tgt] if slot < 0 or j >= den else interp(before[slot], targets[tgt], j, den)
    return out


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
    """A frame's lookup sum is its first packed byte (code_dim 1).  lookup_packed_playout checks the descriptors as the C ABI does and
    computes the rows with playout_model."""
    codebook_num = NQ
    code_dim = 1

    def __init__(self):
        self.rows = []                                                # descriptors of every lookup
        self.row_ptrs = []                                            # the host memory they were passed in

    def packed_frame_bytes(self):
        return NB

    def silence_frame(self):
        return torch.tensor([SILENCE])

    def lookup_packed_playout(self, packed, rows, anchors, targets):
        assert packed.dtype == torch.uint8 and packed.dim() == 2 and packed.shape[1] == NB
        assert rows.dtype == np.int32 and rows.ndim == 2 and rows.shape[1] == 6 and rows.flags.c_contiguous
        self.rows.append(rows.copy())
        self.row_ptrs.append(rows.ctypes.data)
        f = packed.shape[0]
        written = [int(r[3]) for r in rows if r[0] >= 0 and r[3] >= 0]
        read = {int(r[3]) for r in rows if r[0] < 0 and r[3] >= 0}
        assert not set(written) & read and len(set(written)) == len(written)
        for src, nxt, tgt, slot, j, den in rows:
            if src >= 0:
                assert src < f and nxt == -1 and tgt == -1
            elif nxt >= 0:
                assert src == -1 and nxt < f and tgt == -1 and den >= 2 and 1 <= j < den
            else:
                assert src == -1 and 0 <= tgt < targets.shape[0] and j >= 1 and den >= 1
        sums = packed[:, :1].to(torch.float32).numpy()
        out = playout_model(rows, sums, anchors.numpy(), targets.numpy())     # anchors: the server's memory, stored in place
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


def _rx(d=2, cap=3, fpp=2, **kw):
    rx, dec = FakeRx(), FakeDec()
    return ReceiverSessionServer(rx, dec, capacity=cap, frames_per_packet=fpp, sample_rate=8000, playout_delay=d, **kw), rx, dec


def _pkt(sid, seq, codes):
    return wire.encode_packet(sid, seq, NQ, NB, bytes(b for c in codes for b in (c, NQ)))


def _codes(seq, frames=2):
    return [(7 * seq + 3 * i + 1) % 251 for i in range(frames)]


def _drain(srv, sid):
    out = []
    while (y := srv.poll(sid)) is not None:
        out.append(y)
    return out


def _frames(ys):
    """decoded stand-in output -> [(slot position, zq)] per frame"""
    v = np.concatenate(ys).reshape(-1, 2) if ys else np.zeros((0, 2), np.float32)
    return [(int(p), np.float32(z)) for p, z in v]


def _run(srv, sid, arrivals, steps):
    """arrivals: {step: [seq, ...]} submitted before that step -> per step the [(pos, zq)] the session got"""
    out = []
    for t in range(steps):
        for q in arrivals.get(t, []):
            srv.submit_packet(_pkt(sid, q, _codes(q)))
        srv.step()
        out.append(_frames(_drain(srv, sid)))
    return out


def _bits(x):
    return np.asarray(x, np.float32).view(np.int32).tolist()


# ------------------------------------------------------------------ buffering and jitter
@pytest.mark.parametrize("d", [0, 2])
def test_a_session_starts_playing_d_steps_after_its_first_packet(d):
    srv, rx, _ = _rx(d=d)
    srv.open(5)
    got = _run(srv, 5, {1: [0], 2: [1], 3: [2]}, 6)
    start = 1 + d
    assert [len(x) for x in got[:start]] == [0] * start
    assert [[z for _, z in x] for x in got[start:start + 3]] == [[np.float32(c) for c in _codes(q)] for q in range(3)]
    st = srv.statistics()["per_session"][5]
    assert st["packets"] == 3 and st["underruns"] == 6 - start - 3 and st["buffered"] == 0


def test_jitter_within_the_delay_conceals_nothing():
    rng = np.random.default_rng(4)
    srv, rx, _ = _rx(d=2)
    srv.open(1)
    n = 30
    arrivals = {}
    for q in range(n):                                                # sent at step q, arriving 0 .. 2 steps later (the first on time)
        arrivals.setdefault(q + (int(rng.integers(0, 3)) if q else 0), []).append(q)
    for t in arrivals:
        rng.shuffle(arrivals[t])
    got = _run(srv, 1, arrivals, n + 2)
    played = [z for x in got for _, z in x]
    assert played == [np.float32(c) for q in range(n) for c in _codes(q)]
    assert [len(x) for x in got] == [0, 0] + [2] * n                  # one packet per step from step D on
    st = srv.statistics()["per_session"][1]
    assert (st["losses"], st["concealed"], st["underruns"], st["late"], st["packets"]) == (0, 0, 0, 0, n)
    assert st["reorders"] > 0


# ------------------------------------------------------------------ rules 1 to 3
def test_a_loss_with_a_held_follower_is_interpolated_toward_it():
    srv, rx, _ = _rx(d=1)
    srv.open(2)
    slot = srv._ids[2]
    # 0, 1 on time; 2 and 3 lost; 4 arrives in time for its step
    got = _run(srv, 2, {0: [0], 1: [1], 3: [4], 4: [5]}, 7)
    a, s4 = np.float32(_codes(1)[-1]), np.float32(_codes(4)[0])
    # step 3 conceals 2 (c = 0, den = 0 + (4 - 2) * 2 + 1 = 5), step 4 conceals 3 (c = 2, den = 2 + 1 * 2 + 1 = 5)
    assert rx.rows[2].tolist() == [[-1, 0, -1, slot, 1, 5], [-1, 0, -1, slot, 2, 5]]
    assert rx.rows[3].tolist() == [[-1, 0, -1, slot, 3, 5], [-1, 0, -1, slot, 4, 5]]
    assert _bits([z for _, z in got[3] + got[4]]) == _bits([interp(a, s4, j, 5) for j in range(1, 5)])
    assert [z for _, z in got[5]] == [np.float32(c) for c in _codes(4)]
    assert [p for x in got for p, _ in x] == list(range(12))          # the decoder runs through the gap
    st = srv.statistics()["per_session"][2]
    assert (st["losses"], st["concealed"], st["concealed_frames"], st["packets"], st["frames"]) == (2, 2, 4, 4, 8)
    assert st["wire_kbps"] == pytest.approx(8e-3 * 4 * (16 + 2 * NB) / (8 * 2 / 8000))


def test_an_underrun_fades_toward_the_silence_frame_then_pauses_and_resumes_at_the_senders_next_packet():
    srv, rx, dec = _rx(d=0, fade_frames=3, max_fade_packets=2)
    srv.open(3)
    slot = srv._ids[3]
    got = _run(srv, 3, {0: [0], 1: [1]}, 5)                          # the sender goes quiet after 1
    a = np.float32(_codes(1)[-1])
    assert rx.rows[2].tolist() == [[-1, -1, 0, slot, 1, 3], [-1, -1, 0, slot, 2, 3]]
    assert rx.rows[3].tolist() == [[-1, -1, 0, slot, 3, 3], [-1, -1, 0, slot, 4, 3]]
    assert _bits([z for _, z in got[2] + got[3]]) == _bits([interp(a, SILENCE, 1, 3), interp(a, SILENCE, 2, 3), SILENCE, SILENCE])
    assert got[4] == [] and len(rx.rows) == 4                         # paused: buffering again
    st = srv.statistics()["per_session"][3]
    assert (st["underruns"], st["faded_frames"], st["pauses"], st["losses"]) == (2, 4, 1, 0)
    assert srv._next[slot] == 2
    # the sender's next packet is 2: it is neither late nor a duplicate, and it plays
    got = _run(srv, 3, {0: [2], 1: [3]}, 2)
    assert [z for _, z in got[0] + got[1]] == [np.float32(c) for q in (2, 3) for c in _codes(q)]
    st = srv.statistics()["per_session"][3]
    assert (st["late"], st["duplicates"], st["packets"]) == (0, 0, 4)
    assert dec.carry[slot] == 12                                      # 4 real packets and 2 fade packets of 2 frames


def test_a_fade_packet_has_the_last_real_packets_frame_count_and_j_runs_on_from_c():
    srv, rx, _ = _rx(d=0, fpp=4, max_fade_packets=3)
    srv.open(1)
    srv.submit_packet(_pkt(1, 0, _codes(0, 3)))
    srv.step()
    srv.step()
    assert rx.rows[-1][:, 4].tolist() == [1, 2, 3] and (rx.rows[-1][:, 5] == 8).all()    # den = fade_frames = 2 * 4
    srv.step()
    assert rx.rows[-1][:, 4].tolist() == [4, 5, 6]
    # a fade before any real frame: no anchor (the silence frame itself)
    srv2, rx2, _ = _rx(d=0, fpp=4)
    srv2.open(1)
    srv2.submit_packet(_pkt(1, 1, _codes(1)))                         # packet 0 lost, 1 held: an interpolation toward 1 without anchor
    srv2.step()
    assert rx2.rows[-1].tolist() == [[-1, 0, -1, -1, 1, 3], [-1, 0, -1, -1, 2, 3]]
    srv2.step()
    srv2.step()
    assert rx2.rows[-1][:, 3].tolist() == [srv2._ids[1]] * 2 and rx2.rows[-1][:, 4].tolist() == [1, 2]


def test_a_lost_first_packet_is_interpolated_without_an_anchor():
    srv, rx, _ = _rx(d=1)
    srv.open(6)
    got = _run(srv, 6, {0: [1], 1: [2]}, 4)
    assert rx.rows[0].tolist() == [[-1, 0, -1, -1, 1, 3], [-1, 0, -1, -1, 2, 3]]
    s1 = np.float32(_codes(1)[0])
    assert [z for _, z in got[1]] == [s1, s1]
    assert [z for _, z in got[2]] == [np.float32(c) for c in _codes(1)]
    assert srv.statistics()["per_session"][6]["losses"] == 1


def test_late_and_duplicate_packets_are_told_apart():
    srv, _, _ = _rx(d=0)
    srv.open(1)
    _run(srv, 1, {0: [0], 1: [2]}, 3)                                 # 1 concealed at step 1
    assert not srv.submit_packet(_pkt(1, 1, _codes(1)))               # given up: late
    assert not srv.submit_packet(_pkt(1, 0, _codes(0)))               # decoded: duplicate
    assert srv.submit_packet(_pkt(1, 4, _codes(4)))
    assert not srv.submit_packet(_pkt(1, 4, _codes(4)))               # held: duplicate
    st = srv.statistics()["per_session"][1]
    assert (st["late"], st["duplicates"], st["losses"], st["buffered"]) == (1, 2, 1, 1)


def test_a_gap_does_not_wait_for_the_reorder_window():
    srv, rx, _ = _rx(d=0)
    srv.open(1)
    _run(srv, 1, {0: [0], 1: [2]}, 2)
    assert len(rx.rows) == 2 and rx.rows[1][0, 0] == -1 and rx.rows[1][0, 1] == 0
    assert srv.statistics()["per_session"][1]["losses"] == 1


def test_several_sessions_share_one_lookup_and_one_decode_per_step():
    srv, rx, dec = _rx(d=0, cap=3)
    for sid in (1, 2, 3):
        srv.open(sid)
    srv.submit_packet(_pkt(1, 0, _codes(0)))
    srv.submit_packet(_pkt(2, 0, _codes(0)))
    srv.submit_packet(_pkt(3, 0, _codes(0)))
    srv.step()
    srv.submit_packet(_pkt(1, 1, _codes(1)))                          # 1 real, 2 faded, 3 interpolated toward 2
    srv.submit_packet(_pkt(3, 2, _codes(2)))
    assert srv.step() == 3
    s1, s2, s3 = (srv._ids[k] for k in (1, 2, 3))
    assert rx.rows[-1].tolist() == [[0, -1, -1, -1, 0, 0], [1, -1, -1, s1, 0, 0], [-1, -1, 0, s2, 1, 4], [-1, -1, 0, s2, 2, 4],
                                    [-1, 2, -1, s3, 1, 3], [-1, 2, -1, s3, 2, 3]]
    assert dec.calls[-1] == ([2, 2, 2], [s1, s2, s3])
    assert len(rx.rows) == 2


# ------------------------------------------------------------------ migration
def _migrate(when, traffic, steps, d=1, **kw):
    """run traffic on a reference receiver and on a receiver whose session moves to a third after `when(srv, slot)` is first true"""
    ref, _, _ = _rx(d=d, **kw)
    a, _, _ = _rx(d=d, **kw)
    b, _, _ = _rx(d=d, **kw)
    ref.open(8), a.open(8)
    b.open(1)                                                         # the destination serves someone: session 8 gets another slot
    for _ in range(3):
        b.step()                                                      # and has counted other steps
    got, want, cur, moved = [], [], a, None
    for t in range(steps):
        for q in traffic.get(t, []):
            ref.submit_packet(_pkt(8, q, _codes(q)))
            cur.submit_packet(_pkt(8, q, _codes(q)))
        if cur is a and when(a, a._ids[8]):
            st = a.detach(8)
            moved = st
            assert b.attach(st) == 8
            cur = b
        ref.step()
        cur.step()
        want.extend(_drain(ref, 8))
        got.extend(_drain(cur, 8))
    assert moved is not None
    assert _frames(got) == _frames(want)
    return moved, ref, b


def test_detach_attach_while_buffering():
    st, ref, b = _migrate(lambda s, slot: len(s._held[slot]) == 2, {0: [0], 1: [1], 3: [2]}, 8, d=3)
    assert st.playout["playing"] is False and st.playout["waited"] == [1, 0]
    assert ref.statistics()["per_session"][8]["packets"] == b.statistics()["per_session"][8]["packets"] == 3


def test_detach_attach_in_the_middle_of_a_gap():
    st, ref, b = _migrate(lambda s, slot: s.stats[slot].concealed == 1, {0: [0], 1: [1], 2: [5], 5: [6]}, 10)
    assert st.playout["playing"] and st.playout["c"] == 2 and st.playout["given_up"] == [2] and st.anchor is not None
    assert b.statistics()["per_session"][8]["concealed"] == 2
    assert not b.submit_packet(_pkt(8, 2, _codes(2))) and b.statistics()["per_session"][8]["late"] == 1


def test_detach_attach_in_the_middle_of_a_fade():
    st, ref, b = _migrate(lambda s, slot: s.stats[slot].underruns == 2, {0: [0], 1: [1], 9: [2], 10: [3]}, 14)
    assert st.playout["fades"] == 2 and st.playout["c"] == 4 and st.playout["last_frames"] == 2
    for srv in (ref, b):
        s = srv.statistics()["per_session"][8]
        assert (s["pauses"], s["packets"]) == (1, 2 if srv is b else 4)


def test_a_session_cannot_move_between_playout_and_other_receivers():
    a, _, _ = _rx(d=1)
    b = ReceiverSessionServer(FakeRx(), FakeDec(), capacity=2, frames_per_packet=2, sample_rate=8000)
    a.open(1), b.open(2)
    with pytest.raises(ValueError, match="playout"):
        b.attach(a.detach(1))
    with pytest.raises(ValueError, match="playout"):
        a.attach(b.detach(2))


# ------------------------------------------------------------------ refusals and defaults
@pytest.mark.parametrize("kw,field", [({"conceal_packets": 2}, "conceal_packets"), ({"playout_delay": -1}, "playout_delay"),
                                      ({"fade_frames": 0}, "fade_frames"), ({"max_fade_packets": 0}, "max_fade_packets"),
                                      ({"silence_frame": [1.0, 2.0]}, "silence_frame")])
def test_bad_arguments_are_refused(kw, field):
    args = dict(playout_delay=1)
    args.update(kw)
    with pytest.raises(ValueError, match=field):
        ReceiverSessionServer(FakeRx(), FakeDec(), capacity=2, frames_per_packet=2, **args)


def test_defaults_and_the_silence_frame_override():
    srv, _, _ = _rx(d=1, fpp=3)
    assert (srv.fade_frames, srv.max_fade_packets) == (6, 4)
    assert srv._targets.tolist() == [[float(SILENCE)]]
    srv2, _, _ = _rx(d=1, silence_frame=[0.25])
    assert srv2._targets.tolist() == [[0.25]]
    off = ReceiverSessionServer(FakeRx(), FakeDec(), capacity=2, frames_per_packet=2)
    off.open(0)
    assert off.playout_delay is None and "late" not in off.statistics()["per_session"][0] and off.detach(0).playout is None


# ------------------------------------------------------------------ the descriptor tables and the C ABI's struct
def test_descriptors_go_through_two_page_locked_tables_in_turn(monkeypatch):
    asked = []
    real = server_mod._pinned

    def spy(n, dtype, device):
        t = real(n, dtype, device)
        asked.append((n, dtype, device, t))
        return t

    monkeypatch.setattr(server_mod, "_pinned", spy)
    srv, rx, _ = _rx(d=0, cap=3, fpp=2)
    tables = [t for n, dt, _, t in asked if dt == torch.int32]
    assert len(tables) == 2 and all(t.numel() == 3 * 2 * 6 for t in tables)
    assert [t.data_ptr() for t in srv._rows_host] == [t.data_ptr() for t in tables]
    srv.open(1)
    for q in range(4):
        srv.submit_packet(_pkt(1, q, _codes(q)))
        srv.step()
    ptrs = [t.data_ptr() for t in tables]
    assert rx.row_ptrs == [ptrs[0], ptrs[1], ptrs[0], ptrs[1]]


def test_playout_row_struct_matches_header():
    from audiodec_b200 import _lib
    hdr = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    body = hdr[hdr.index("typedef struct adec_playout_row {"):hdr.index("} adec_playout_row;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"int32_t\s+(\w+);", body) == [f[0] for f in _lib.AdecPlayoutRow._fields_]
    assert ctypes.sizeof(_lib.AdecPlayoutRow) == 24
    for name in ("adec_lookup_packed_playout", "adec_lookup_packed_playout_bf16"):
        m = re.search(name + r"\s*\(([^)]*)\)", hdr)
        assert m and len(_lib.SYMBOLS[name][1]) == len(m.group(1).split(",")), name
