"""Stream slots without a GPU: the bindings declare the new entry points, and SessionCodecServer's session logic (open, close, reuse,
capacity, no silence fed, queues dropped on close, statistics) on a stand-in codec with per-slot state."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from audiodec_b200 import _lib
from audiodec_b200.server import SessionCodecServer

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("adec_encode_streams", "adec_decode_streams", "adec_decode_streams_bf16", "adec_copy_stream_state")


def test_bindings_declare_the_slot_entry_points():
    header = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    for name in NEW:
        assert name in _lib.SYMBOLS
        m = re.search(r"int " + name + r"\(([^)]*)\)", header)
        assert m, name
        assert len(_lib.SYMBOLS[name][1]) == len(m.group(1).split(",")), name
    assert _lib.SYMBOLS["adec_encode_streams"][1][2] == ctypes.POINTER(ctypes.c_int)


class SlotCodec:
    """Stand-in with per-slot state: encode_streams(chunks, streams) gives z_b = x_b + carry[slot], carry[slot] = x_b[-1].  One frame
    per sample (hop 1).  Records which streams every call advanced."""

    def __init__(self):
        self.carry = torch.zeros(1)
        self.calls = []
        self.during_encode = None

    @property
    def n_streams(self):
        return self.carry.numel()

    def set_streams(self, n):
        assert self.carry.numel() == 1
        self.carry = self.carry.repeat(n)

    def copy_stream_state(self, src, dst):
        for d in dst:
            self.carry[d] = self.carry[src]

    def encode_streams(self, chunks, streams):
        self.calls.append(list(streams))
        if self.during_encode:
            self.during_encode()
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
        y = 2.0 * zq.reshape(-1)
        return list(torch.split(y, frames))


class Clock:
    def __init__(self):
        self.t = 10.0

    def __call__(self):
        self.t += 0.001
        return self.t


def _srv(cap=3, **kw):
    c = SlotCodec()
    c.carry[0] = 0.5                                       # the warm state the template keeps
    kw.setdefault("max_latency", 1.0)
    return SessionCodecServer(c, c, c, capacity=cap, frame_size=4, sample_rate=8000, clock=Clock(), **kw), c


def _frame(v):
    return np.full(4, v, dtype=np.float32)


def test_open_close_reuse_and_capacity():
    srv, c = _srv(cap=2)
    assert c.carry.numel() == 3 and srv.template == 2
    a, b = srv.open(), srv.open()
    assert {a, b} == {0, 1} and srv.open_streams == [0, 1]
    with pytest.raises(RuntimeError, match="full"):
        srv.open()
    srv.submit(a, _frame(1.0))
    assert srv.step() == 1
    assert np.allclose(srv.poll(a), 2.0 * (np.array([1.0, 1.0, 1.0, 1.0]) + 0.5))   # started from the template's warm state
    srv.close(a)
    with pytest.raises(KeyError):
        srv.submit(a, _frame(1.0))
    with pytest.raises(KeyError):
        srv.close(a)
    a2 = srv.open()
    assert a2 == a and float(c.carry[a2]) == 0.5               # the reused slot starts warm, without the previous caller's history
    assert float(c.carry[srv.template]) == 0.5                 # the template is never advanced


def test_idle_streams_are_not_fed_and_keep_their_state():
    srv, c = _srv(cap=3)
    ids = [srv.open() for _ in range(3)]
    srv.submit(ids[0], _frame(1.0))
    srv.submit(ids[2], _frame(3.0))
    assert srv.step() == 2
    assert c.calls[-1] == [ids[0], ids[2]]                     # no silence for the idle stream
    assert float(c.carry[ids[1]]) == 0.5
    srv.submit(ids[1], _frame(2.0))
    assert srv.step() == 1 and c.calls[-1] == [ids[1]]
    assert np.allclose(srv.poll(ids[1]), 2.0 * (2.0 + 0.5))
    assert srv.step() == 0 and len(c.calls) == 2               # nothing queued: no codec call at all
    st = srv.statistics()
    assert st["frames"] == 3 and st["underruns"] == 1 + 2 + 3 and st["capacity"] == 3 and st["open_streams"] == 3


def test_close_drops_queues_and_drop_policy_still_applies():
    srv, c = _srv(cap=2, max_latency=2 * 4 / 8000)
    a, b = srv.open(), srv.open()
    for v in range(5):
        srv.submit(a, _frame(float(v)))
    assert srv.pending(a) == 2 and srv.stats[a].frame_drops == 3
    srv.submit(b, _frame(7.0))
    srv.step()
    assert srv.poll(b) is not None and srv.poll(a) is not None
    srv.close(a)
    assert srv.pending(a) == 0 and srv.poll(a) is None
    assert srv.step() == 0


def test_start_stop_thread():
    srv, c = _srv(cap=2)
    s = srv.open()
    srv._clock = __import__("time").time
    srv.start(period=0.002)
    srv.submit(s, _frame(1.0))
    import time
    t0 = time.time()
    while srv.poll(s) is None and time.time() - t0 < 5:
        time.sleep(0.002)
    srv.stop()
    assert srv.statistics()["frames"] == 1


def test_generators_must_hold_one_warmed_stream():
    c = SlotCodec()
    c.set_streams(4)                                           # e.g. reused from a lock-step server
    with pytest.raises(ValueError, match="one"):
        SessionCodecServer(c, c, c, capacity=2, frame_size=4, sample_rate=8000)


def test_statistics_count_open_streams_and_advanced_audio():
    srv, c = _srv(cap=4, wire=True)
    a, b = srv.open(), srv.open()
    c.pack = lambda idx: idx.contiguous().view(torch.uint8)   # 4 bytes per frame sample of the stand-in's float "indices"
    c.unpack = lambda packed: packed.view(torch.float32)
    for k in range(3):
        srv.submit(a, _frame(1.0))
        if k == 0:
            srv.submit(b, _frame(2.0))
        srv.step()
    st = srv.statistics()
    assert st["n_streams"] == st["open_streams"] == 2 and st["capacity"] == 4 and st["frames"] == 4
    # 4 frames of 4 samples, 16 bytes each on the wire, over 4 * 4 / 8000 s of audio
    assert st["wire_kbps_per_stream"] == pytest.approx(8e-3 * 4 * 16 / (4 * 4 / 8000))


def test_reopened_slot_never_gets_the_previous_callers_frame():
    """close(s) while a step holds s's frame, and a new caller open()s the same slot before the step hands its outputs out: the old
    caller's frame must be dropped, not delivered to the new session."""
    import threading
    srv, c = _srv(cap=2)
    a = srv.open()
    srv.submit(a, _frame(1.0))
    opener = []

    def close_and_reopen():                                    # inside the codec call, like a caller hanging up mid-step
        srv.close(a)
        t = threading.Thread(target=lambda: opener.append(srv.open()))
        t.start()                                              # blocks on the codec lock until the step leaves the codec
        opener.append(t)
    c.during_encode = close_and_reopen
    clock = srv._clock

    def clock_after_reopen():                                  # the step reads the clock between the codec and the hand-out:
        if len(opener) == 1:                                   # let the new caller finish open() there (the losing interleaving)
            opener[0].join()
        return clock()
    srv._clock = clock_after_reopen
    assert srv.step() == 1
    c.during_encode = None
    assert opener[1] == a and a in srv.open_streams            # the new caller got the same slot ...
    assert srv.poll(a) is None                                 # ... and not the old caller's frame
    assert srv.stats[a].n_frames == 0
    srv.submit(a, _frame(3.0))
    assert srv.step() == 1
    assert np.allclose(srv.poll(a), 2.0 * (3.0 + 0.5))         # it starts from the template's warm state
