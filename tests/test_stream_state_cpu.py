"""Stream state without a GPU: the bindings declare the state entry points, the Python argument checks, and SessionCodecServer's detach /
attach bookkeeping (queues, session ids, errors, fresh counters) on a stand-in codec with per-slot state."""
import os
import re

import numpy as np
import pytest
import torch

from audiodec_b200 import _lib
from audiodec_b200.codec import _check_state, _stream_ids
from audiodec_b200.server import SessionCodecServer, SessionState

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("adec_state_entries", "adec_state_entry", "adec_stream_state_elems", "adec_get_stream_state", "adec_set_stream_state")


def test_bindings_declare_the_state_entry_points():
    header = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    for name in NEW:
        assert name in _lib.SYMBOLS
        m = re.search(r"(?:int|int64_t)\s+" + name + r"\(([^)]*)\)", header)
        assert m, name
        assert len(_lib.SYMBOLS[name][1]) == len(m.group(1).split(",")), name


def test_argument_checks():
    assert _stream_ids(3) == [3]
    assert _stream_ids(range(2)) == [0, 1]
    with pytest.raises(TypeError):
        _stream_ids([0, 1.0])
    with pytest.raises(TypeError):
        _stream_ids([True])
    dev = torch.device("cpu")
    ok = torch.zeros(2, 10)
    assert _check_state(ok, 2, 10, torch.float32, dev) is ok
    with pytest.raises(TypeError):
        _check_state(np.zeros((2, 10), np.float32), 2, 10, torch.float32, dev)
    with pytest.raises(ValueError, match="bfloat16"):
        _check_state(ok, 2, 10, torch.bfloat16, dev)
    with pytest.raises(ValueError, match=r"\(3, 10\)"):
        _check_state(ok, 3, 10, torch.float32, dev)
    with pytest.raises(RuntimeError, match="move it"):
        _check_state(ok, 2, 10, torch.float32, torch.device("cuda", 0))
    odd = torch.zeros(41)[1:].view(2, 20)[:, :10]             # not contiguous and not 16-byte aligned: handed over as an aligned copy
    got = _check_state(odd, 2, 10, torch.float32, dev)
    assert got.is_contiguous() and got.data_ptr() % 16 == 0


class SlotCodec:
    """Stand-in with per-slot state (z_b = x_b + carry[slot], carry[slot] = x_b[-1], hop 1) and the state export / import surface."""

    def __init__(self, layout=(("enc.pad_buffer", 1, 1),)):
        self.carry = torch.zeros(1)
        self.state_layout = [tuple(e) for e in layout]

    @property
    def n_streams(self):
        return self.carry.numel()

    def set_streams(self, n):
        self.carry = self.carry.repeat(n)

    def copy_stream_state(self, src, dst):
        for d in dst:
            self.carry[d] = self.carry[src]

    def stream_state(self, streams):
        return self.carry[list(streams)].clone().view(-1, 1)

    def load_stream_state(self, streams, state, layout=None):
        assert layout is None or [tuple(e) for e in layout] == self.state_layout
        self.carry[list(streams)] = state.view(-1)

    def encode_streams(self, chunks, streams):
        out = []
        for x, s in zip(chunks, streams):
            out.append(x + self.carry[s])
            self.carry[s] = x[-1]
        return torch.cat(out).view(1, 1, -1), [c.numel() for c in chunks]

    def quantize(self, z):
        return z

    def lookup(self, idx):
        return idx.reshape(1, -1, 1)

    def decode_streams(self, zq, frames, streams):
        return list(torch.split(2.0 * zq.reshape(-1), frames))


def _srv(cap=3, codec=None):
    c = codec or SlotCodec()
    t = [10.0]

    def clock():
        t[0] += 0.001
        return t[0]
    return SessionCodecServer(c, c, c, capacity=cap, frame_size=4, sample_rate=8000, max_latency=1.0, clock=clock), c


def _frame(v):
    return np.full(4, v, np.float32)


def test_detach_attach_moves_state_and_frames():
    a, ca = _srv()
    b, cb = _srv()
    s0, s1 = a.open(), a.open()
    b.open()
    for v in (1.0, 2.0):
        a.submit(s1, _frame(v), t_capture=5.0)
    a.submit(s0, _frame(7.0))
    a.step()                                                  # s1: frame 1 decoded (not polled), frame 2 queued
    st = a.detach(s1)
    assert isinstance(st, SessionState)
    assert [float(f[0]) for f, _ in st.inputs] == [2.0] and st.inputs[0][1] == 5.0
    assert len(st.outputs) == 1 and float(st.outputs[0][0]) == 2.0
    assert a.open_streams == [s0]
    with pytest.raises(KeyError):
        a.submit(s1, _frame(0.0))
    with pytest.raises(KeyError):
        a.detach(s1)
    dst = b.attach(st)
    assert dst == 1 and b.open_streams == [0, 1]
    assert b.pending(dst) == 1
    assert b.statistics()["per_stream"][dst]["n_frames"] == 0
    assert float(b.poll(dst)[0]) == 2.0                       # the undelivered frame
    b.step()
    # frame 2 continues the moved state: 2 * (2 + carry 1) = 6 (a fresh slot would give 4)
    assert float(b.poll(dst)[0]) == 6.0
    assert b.stats[dst].n_frames == 1
    # the freed slot is reused by the next open, from the template
    assert a.open() == s1
    a.submit(s1, _frame(3.0))
    a.step()
    assert float(a.poll(s1)[0]) == 6.0                        # 2 * (3 + 0): nothing of the detached session
    assert float(a.poll(s0)[0]) == 14.0


def test_attach_errors():
    a, _ = _srv(cap=1)
    s = a.open()
    st = a.detach(s)
    a.open()
    with pytest.raises(RuntimeError, match="full"):
        a.attach(st)
    other, _ = _srv(codec=SlotCodec(layout=(("dec.pad_buffer", 2, 1),)))
    with pytest.raises(ValueError, match="layout"):
        other.attach(st)
    with pytest.raises(ValueError):
        other.attach(SessionState([], [], [], []))
    assert other.open_streams == [] and len(other._free) == 3   # a refused attach takes no slot


def test_detach_waits_for_the_step_in_progress():
    """a detach issued while a step runs returns after the step has handed off the session's frame"""
    import threading
    a, c = _srv()
    s = a.open()
    a.submit(s, _frame(1.0))
    started, release = threading.Event(), threading.Event()
    orig = c.decode_streams

    def slow(zq, frames, streams):
        started.set()
        release.wait(5)
        return orig(zq, frames, streams)
    c.decode_streams = slow
    t = threading.Thread(target=a.step)
    t.start()
    started.wait(5)
    out = {}
    d = threading.Thread(target=lambda: out.setdefault("st", a.detach(s)))
    d.start()
    d.join(0.2)
    assert d.is_alive()                                        # blocked behind the step
    release.set()
    t.join(5)
    d.join(5)
    assert len(out["st"].outputs) == 1 and float(out["st"].outputs[0][0]) == 2.0
