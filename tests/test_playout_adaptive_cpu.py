"""The adaptive playout clock without a GPU: ReceiverSessionServer(playout_delay=D, max_playout_delay=D_max) on duck-typed stand-ins
whose lookup_packed_timescale is a numpy float32 model of the kernel's five row kinds, against a model of the content queue, the delay
policy and the rows written here.  A jitter-free run against the fixed clock, the model step by step on clean, jittered, spiked and
drifting traces, what adaptation buys on a spike and under clock drift, rows that start from a frame staged in the same launch, a pause
in the middle of an offset queue, detach / attach, and the refusals."""
import collections

import numpy as np
import pytest
import torch

from audiodec_b200 import wire
from audiodec_b200.server import ReceiverSessionServer

NQ, NB = 8, 2          # the stand-ins' codebook count and packed bytes per frame
SILENCE = np.float32(-3.0)


def interp(a, t, j, den):
    """fl(fl(fl(j / den) * fl(t - a)) + a) in float32"""
    a, t = np.float32(a), np.float32(t)
    return (np.float32(j) / np.float32(den)) * (t - a) + a


def timescale_model(rows, sums, anchors, targets):
    """the kernel's rows in float32: real, interpolated, fade, between and frame-started fade -> (R, D); stores the real rows' anchors"""
    before = anchors.copy()
    out = np.empty((len(rows), anchors.shape[1]), np.float32)
    for i, (src, nxt, tgt, slot, j, den) in enumerate(rows):
        if src >= 0 and nxt >= 0:
            out[i] = interp(sums[src], sums[nxt], j, den)
        elif src >= 0 and tgt >= 0:
            out[i] = targets[tgt] if j >= den else interp(sums[src], targets[tgt], j, den)
        elif src >= 0:
            out[i] = sums[src]
            if slot >= 0:
                anchors[slot] = sums[src]
        elif nxt >= 0:
            out[i] = sums[nxt] if slot < 0 else interp(before[slot], sums[nxt], j, den)
        else:
            out[i] = targets[tgt] if slot < 0 or j >= den else interp(before[slot], targets[tgt], j, den)
    return out


# ------------------------------------------------------------------ stand-ins
class FakeRx:
    """A frame's lookup sum is its first packed byte (code_dim 1); its second byte tells frames apart.  Both lookups check their
    descriptors as the C ABI does and compute the rows with timescale_model."""
    codebook_num = NQ
    code_dim = 1

    def __init__(self):
        self.calls = []                                               # (entry point, rows, packed bytes) of every lookup

    def packed_frame_bytes(self):
        return NB

    def silence_frame(self):
        return torch.tensor([SILENCE])

    def _lookup(self, name, packed, rows, anchors, targets):
        assert packed.dtype == torch.uint8 and packed.dim() == 2 and packed.shape[1] == NB
        assert rows.dtype == np.int32 and rows.ndim == 2 and rows.shape[1] == 6 and rows.flags.c_contiguous
        f = packed.shape[0]
        written = [int(r[3]) for r in rows if r[0] >= 0 and r[3] >= 0]
        read = {int(r[3]) for r in rows if r[0] < 0 and r[3] >= 0}
        assert not set(written) & read and len(set(written)) == len(written)
        for src, nxt, tgt, slot, j, den in rows:
            if src >= 0 and (nxt >= 0 or tgt >= 0):
                assert name == "timescale" and src < f and slot == -1
                assert (nxt < f and tgt == -1 and 1 <= j < den) if nxt >= 0 else (tgt < targets.shape[0] and j >= 1 and den >= 1)
            elif src >= 0:
                assert src < f and nxt == -1 and tgt == -1
            elif nxt >= 0:
                assert src == -1 and nxt < f and tgt == -1 and den >= 2 and 1 <= j < den
            else:
                assert src == -1 and 0 <= tgt < targets.shape[0] and j >= 1 and den >= 1
        self.calls.append((name, rows.copy(), packed.numpy().copy()))
        sums = packed[:, :1].to(torch.float32).numpy()
        out = timescale_model(rows, sums, anchors.numpy(), targets.numpy())     # anchors: the server's memory, stored in place
        return torch.from_numpy(out).view(1, -1, 1)

    def lookup_packed_playout(self, packed, rows, anchors, targets):
        return self._lookup("playout", packed, rows, anchors, targets)

    def lookup_packed_timescale(self, packed, rows, anchors, targets):
        return self._lookup("timescale", packed, rows, anchors, targets)


class FakeDec:
    """Two samples per frame: (frames the slot decoded before it, its zq value)."""
    state_layout = [("pad_buffer", 1, 1)]

    def __init__(self):
        self.carry = torch.tensor([0.0])
        self.calls = []

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

    def decode_streams(self, zq, frames, streams):
        self.calls.append((list(frames), list(streams)))
        out, o = [], 0
        for f, s in zip(frames, streams):
            pos = self.carry[s] + torch.arange(f, dtype=torch.float32)
            out.append(torch.stack([pos, zq.reshape(-1)[o:o + f]], 1).reshape(1, 1, -1))
            self.carry[s] += f
            o += f
        return out


P = 5


def _rx(d=1, dmax=6, cap=2, fpp=P, **kw):
    rx, dec = FakeRx(), FakeDec()
    kw = dict(kw, playout_delay=d)
    if dmax is not None:
        kw["max_playout_delay"] = dmax
    return ReceiverSessionServer(rx, dec, capacity=cap, frames_per_packet=fpp, sample_rate=8000, **kw), rx, dec


def _fid(seq, i):
    return seq * P + i


def _pkt(sid, seq, frames=P):
    """frame i of packet seq: first byte its lookup sum, second its id's high part (the pair tells every frame of a trace apart)"""
    return wire.encode_packet(sid, seq, NQ, NB, bytes(b for i in range(frames) for b in (_fid(seq, i) % 251 + 1, _fid(seq, i) // 251)))


def _frame_id(b):
    return (int(b[1]) * 251 + int(b[0]) - 1)


def _rows_by_id(rows, packed):
    """descriptors with src / next mapped from staged indices to frame ids"""
    return [(_frame_id(packed[r[0]]) if r[0] >= 0 else -1, _frame_id(packed[r[1]]) if r[1] >= 0 else -1, *map(int, r[2:])) for r in rows]


def _drain(srv, sid):
    out = []
    while (y := srv.poll(sid)) is not None:
        out.append(y)
    return out


def _bits(x):
    return np.asarray(x, np.float32).view(np.int32).tolist()


# ------------------------------------------------------------------ traces: {step: [sequence numbers arriving before it]}
def trace(kind, n, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "clean":
        at = list(range(n))
    elif kind == "jitter":
        at = [q + (int(rng.integers(0, 3)) if q else 0) for q in range(n)]
    elif kind == "spike":                                             # 0 jitter, 0 - 4 steps for 200 packets, 0 again
        at = [q + (int(rng.integers(0, 5)) if 100 <= q < 300 else 0) for q in range(n)]
    elif kind == "drift+":                                            # the sender's clock runs 1 % fast
        at = [int(q / 1.01) for q in range(n)]
    elif kind == "drift-":
        at = [int(q / 0.99) for q in range(n)]
    else:
        raise ValueError(kind)
    out = {}
    for q, t in enumerate(at):
        out.setdefault(t, []).append(q)
    for t in out:
        rng.shuffle(out[t])
    return out


TRACES = ("clean", "jitter", "spike", "drift+", "drift-")


# ------------------------------------------------------------------ the model
class Model:
    """One session of the adaptive clock in slot `slot`, by the rules as stated: rules 1 - 3 fill a queue of content frames, the delay
    decides C, and C content frames become P rows.  Rows carry frame ids in place of staged indices."""

    def __init__(self, d, dmax, window=64, fade_frames=2 * P, max_fade=4, slot=0):
        self.d, self.dmax, self.fade_frames, self.max_fade, self.slot = d, dmax, fade_frames, max_fade, slot
        self.k = self.next = self.c = self.fades = 0
        self.held, self.given_up, self.queue = {}, set(), []
        self.lat = collections.deque(maxlen=window)
        self.playing, self.anchor = False, None
        self.n = collections.Counter()
        self.deltas = []

    def submit(self, seq):
        if seq in self.given_up:
            self.n["late"] += 1
            self.lat.append(self.k - seq)
        elif seq >= self.next and seq not in self.held:
            self.held[seq] = self.k
            self.lat.append(self.k - seq)

    def target(self):
        j = max(self.lat) - min(self.lat) if len(self.lat) >= 2 else 0
        return min(max(j, self.d), self.dmax)

    def _packet(self):
        nxt = self.next
        self.next += 1
        if self.held.pop(nxt, None) is not None:
            self.c = self.fades = 0
            return [("r", _fid(nxt, i)) for i in range(P)]
        self.given_up.add(nxt)
        c = self.c
        self.c += P
        if self.held:
            m = min(self.held)
            self.fades = 0
            return [("i", _fid(m, 0), c + 1 + i, c + (m - nxt) * P + 1) for i in range(P)]
        self.n["underruns"] += 1
        self.n["faded_frames"] += P
        self.fades += 1
        if self.fades == self.max_fade:
            self.n["pauses"] += 1
            self.playing = False
            self.next -= self.max_fade
            self.given_up -= set(range(self.next, self.next + self.max_fade))
            self.fades = 0
        return [("f", c + 1 + i, self.fade_frames) for i in range(P)]

    def step(self):
        """-> the session's rows this step, or None"""
        rows = None
        if not self.playing and any(self.k - t >= self.target() for t in self.held.values()):
            self.playing = True
        if self.playing:
            lam = (self.target() + 1) * P
            pos = (self.next - 1) * P + P - len(self.queue) if self.queue else self.next * P
            delta = (self.k - min(self.lat) + 1) * P - pos
            self.deltas.append((self.k, delta))
            run = 0
            if not self.queue or self.queue[0][0] == "r":
                run = len(self.queue) + P * next(i for i in range(10**6) if self.next + i not in self.held)
            c = P + 1 if delta > lam and run >= P + 1 else P - 1 if delta < lam and run >= P - 1 else P
            self.n["compressed" if c > P else "expanded" if c < P else "plain"] += 1
            while len(self.queue) < c:
                self.queue += self._packet()
            win, self.queue = self.queue[:c], self.queue[c:]
            if not self.playing:
                self.queue = []
                self.lat.clear()
            rows = self._rows(win)
        self.k += 1
        return rows

    def _rows(self, win):
        s, rows = self.slot, []
        if len(win) != P:
            for i in range(P):
                m, r = divmod(i * (len(win) - 1), P - 1)
                rows.append((win[m][1], -1, -1, s if m == len(win) - 1 else -1, 0, 0) if r == 0 else
                            (win[m][1], win[m + 1][1], -1, -1, r, P - 1))
        else:
            reals = [i for i, e in enumerate(win) if e[0] == "r"]
            last = reals[-1] if reals else -1
            for i, e in enumerate(win):
                if e[0] == "r":
                    rows.append((e[1], -1, -1, s if i == last else -1, 0, 0))
                    continue
                src = win[last][1] if 0 <= last < i else (self.anchor if last >= 0 else None)
                slot = s if last < 0 and self.anchor is not None else -1
                if e[0] == "i":
                    rows.append((src, e[1], -1, -1, e[2], e[3]) if src is not None else (-1, e[1], -1, slot, e[2], e[3]))
                else:
                    rows.append((src, -1, 0, -1, e[1], e[2]) if src is not None else (-1, -1, 0, slot, e[1], e[2]))
        reals = [e[1] for e in win if e[0] == "r"]
        if reals:
            self.anchor = reals[-1]
        return rows


# ------------------------------------------------------------------ running a receiver over a trace
def _play(srv, rx, sid, arrivals, steps):
    """-> per step: the session's rows (frame ids) or None, its decoded [(position, zq)], its Delta (adaptive) and the lookup's name"""
    slot = srv._ids[sid]
    out = []
    for t in range(steps):
        for q in arrivals.get(t, []):
            srv.submit_packet(_pkt(sid, q))
        n_calls = len(rx.calls)
        srv.step()
        rows = None
        if len(rx.calls) > n_calls:
            name, r, packed = rx.calls[-1]
            rows = _rows_by_id(r, packed)
        ys = _drain(srv, sid)
        v = np.concatenate(ys).reshape(-1, 2) if ys else np.zeros((0, 2), np.float32)
        out.append((rows, [(int(p), np.float32(z)) for p, z in v], srv.stats[slot].delay_frames))
    return out


def _fixed_deltas(srv, sid, arrivals, steps, window=64):
    """Delta = (k - min lateness + 1) * P - next * P of a fixed-delay receiver at each step it plays (its queue is always aligned)"""
    slot = srv._ids[sid]
    lat = collections.deque(maxlen=window)
    pauses, out = 0, []
    for t in range(steps):
        for q in arrivals.get(t, []):
            ok = srv.submit_packet(_pkt(sid, q))
            if ok or q in srv._given_up[slot]:
                lat.append(t - q)
        playing_before, nxt = srv._playing[slot], srv._next[slot]
        n = srv.stats[slot].underruns + srv.stats[slot].packets + srv.stats[slot].concealed
        srv.step()
        if srv.stats[slot].underruns + srv.stats[slot].packets + srv.stats[slot].concealed > n:
            out.append((t, (t - min(lat) + 1) * P - nxt * P))
        if srv.stats[slot].pauses > pauses:
            pauses = srv.stats[slot].pauses
            lat.clear()
        _drain(srv, sid)
    return out


# ------------------------------------------------------------------ 1. a clean run is the fixed clock
@pytest.mark.parametrize("d", [0, 2])
def test_a_clean_run_plays_the_fixed_clocks_rows_and_pcm(d):
    n, steps = 60, 70                                                 # the sender stops: fades and a pause at the end
    ad, rxa, _ = _rx(d=d, dmax=5)
    fx, rxf, _ = _rx(d=d, dmax=None)
    ad.open(3), fx.open(3)
    got = _play(ad, rxa, 3, trace("clean", n), steps)
    want = _play(fx, rxf, 3, trace("clean", n), steps)
    assert [g[:2] for g in got] == [w[:2] for w in want]
    assert [_bits([z for _, z in g[1]]) for g in got] == [_bits([z for _, z in w[1]]) for w in want]
    assert {c[0] for c in rxa.calls} == {"timescale"} and {c[0] for c in rxf.calls} == {"playout"}
    st = ad.statistics()["per_session"][3]
    assert (st["compressed"], st["expanded"], st["target_delay"]) == (0, 0, d)
    assert {g[2] for g in got[d:n]} == {(d + 1) * P}
    sf = fx.statistics()["per_session"][3]
    for key in ("packets", "frames", "underruns", "faded_frames", "pauses", "late", "losses"):
        assert st[key] == sf[key], key


# ------------------------------------------------------------------ 2. the receiver is the model, step by step
@pytest.mark.parametrize("kind", TRACES)
def test_rows_equal_the_model_on_every_trace(kind):
    n = 500
    arrivals = trace(kind, n, seed=3)
    srv, rx, _ = _rx(d=1, dmax=6)
    srv.open(9)
    model = Model(1, 6, slot=srv._ids[9])
    got = _play(srv, rx, 9, arrivals, n + 30)
    for t in range(n + 30):
        for q in arrivals.get(t, []):
            model.submit(q)
        want = model.step()
        assert got[t][0] == want, (kind, t)
    st = srv.statistics()["per_session"][9]
    assert (st["compressed"], st["expanded"]) == (model.n["compressed"], model.n["expanded"])
    assert (st["underruns"], st["faded_frames"], st["pauses"], st["late"]) == \
        (model.n["underruns"], model.n["faded_frames"], model.n["pauses"], model.n["late"])
    if kind != "clean":
        assert st["compressed"] + st["expanded"] > 0


# ------------------------------------------------------------------ 3. a jitter spike
def _outcome(dmax, d, kind, n=600, extra=20, seed=5):
    arrivals = trace(kind, n, seed=seed)
    srv, rx, _ = _rx(d=d, dmax=dmax)
    srv.open(1)
    if dmax is None:
        deltas = _fixed_deltas(srv, 1, arrivals, n + extra)
    else:
        deltas = [(t, g[2]) for t, g in enumerate(_play(srv, rx, 1, arrivals, n + extra)) if g[0] is not None]
    return srv.statistics()["per_session"][1], deltas


def test_jitter_spikes_cost_less_than_a_small_fixed_delay_and_add_less_delay_than_a_large_one():
    """Over twelve seeded spikes: the adaptive clock [1, 6] loses fewer packets and fade frames in all than a fixed D = 1 (on one
    spike it can lose more: it learns the jitter as it comes, while the fixed clock's pause-and-rewind buys it a large delay for
    good), never pauses more, and keeps a lower mean delay than a fixed D = 6 on every spike."""
    mean = lambda ds: np.mean([x for t, x in ds if t < 600])        # noqa: E731
    cost = {"adaptive": 0, "small": 0}
    for seed in range(12):
        ad, ad_d = _outcome(6, 1, "spike", seed=seed)
        small, _ = _outcome(None, 1, "spike", seed=seed)
        large, large_d = _outcome(None, 6, "spike", seed=seed)
        cost["adaptive"] += ad["late"] + ad["faded_frames"]
        cost["small"] += small["late"] + small["faded_frames"]
        assert ad["pauses"] <= small["pauses"]
        assert mean(ad_d) < mean(large_d)
        assert ad["compressed"] > 0
        # the spike's last packet (299) arrives by step 303 and has left the window 64 packets later; by step 500 the compressions
        # have brought the delay back to (D + 1) * P
        settled = [x for t, x in ad_d if 500 <= t < 600]
        assert settled and set(settled) == {2 * P}, seed
    assert cost["adaptive"] < cost["small"], cost


# ------------------------------------------------------------------ 4. clock drift
def test_a_fast_sender_grows_the_fixed_buffer_and_not_the_adaptive_delay():
    fixed, _ = _outcome(None, 2, "drift+", extra=-10)                 # 590 steps, while the sender still sends
    assert 2 + 4 <= fixed["buffered"] <= 2 + 7                        # D, and about one packet more per 100 steps
    ad, ad_d = _outcome(6, 2, "drift+", extra=-10)
    lam = (ad["target_delay"] + 1) * P
    assert all(abs(x - lam) <= P for t, x in ad_d) and ad["compressed"] > 0
    assert ad["buffered"] <= 2


def test_a_slow_sender_underruns_the_fixed_clock_and_not_the_adaptive_one():
    fixed, _ = _outcome(None, 2, "drift-")
    assert fixed["underruns"] >= 3
    srv, rx, _ = _rx(d=2, dmax=6, jitter_window=64)
    srv.open(1)
    arrivals = trace("drift-", 600, seed=5)
    slot = srv._ids[1]
    converged, after = None, 0
    for t in range(600):
        for q in arrivals.get(t, []):
            srv.submit_packet(_pkt(1, q))
        before = srv.stats[slot].underruns
        srv.step()
        _drain(srv, 1)
        st = srv.stats[slot]
        if converged is None and st.delay_frames is not None and st.delay_frames >= (srv._target(slot) + 1) * P:
            converged = t
        elif converged is not None:
            after += st.underruns - before
    assert converged is not None and converged < 100 and after == 0
    assert srv.stats[slot].expanded > 0


# ------------------------------------------------------------------ 5. rows that start from a frame of the same launch
def _after_a_scaled_step(lost_next):
    """D = 0, D_max = 3.  Packet 0 plays at once; 1 is missing at step 1 (a fade) and arrives late at step 2 with 2: the lateness
    spread raises the target to 1 packet and step 2 expands, leaving one frame of 2 queued.  Then 3 is lost with 4 held (a
    concealment) or the sender stops (an underrun), right after that scaled step."""
    srv, rx, _ = _rx(d=0, dmax=3)
    srv.open(1)
    slot = srv._ids[1]
    arrivals = {0: [0], 2: [1, 2], 3: [4] if lost_next else []}
    rows = []
    for t in range(6):
        for q in arrivals.get(t, []):
            srv.submit_packet(_pkt(1, q))
        srv.step()
        rows.append(_rows_by_id(rx.calls[-1][1], rx.calls[-1][2]))
    return srv, rx, slot, rows


def _anchor_split(rx, call):
    """the call's rows computed in two launches: every real row first (storing the anchor), then every other row reading the anchor
    stored from its src frame -> zq of the rows in their original order"""
    _, rows, packed = rx.calls[call]
    sums = packed[:, :1].astype(np.float32)
    anchors = np.zeros((rows.shape[0] + 1, 1), np.float32)
    targets = np.array([[SILENCE]], np.float32)
    first = np.array([(r[0], -1, -1, i, 0, 0) for i, r in enumerate(rows) if r[0] >= 0], np.int32)
    timescale_model(first, sums, anchors, targets)
    second = []
    for i, (src, nxt, tgt, slot, j, den) in enumerate(rows):
        if src >= 0 and (nxt >= 0 or tgt >= 0):
            second.append((-1, nxt, tgt, i, j, den))
        elif src >= 0:
            second.append((src, -1, -1, -1, 0, 0))
        else:
            second.append((src, nxt, tgt, slot, j, den))
    return timescale_model(np.asarray(second, np.int32), sums, anchors, targets)


@pytest.mark.parametrize("lost_next", [True, False])
def test_a_loss_or_an_underrun_right_after_a_scaled_step_starts_from_the_staged_frame(lost_next):
    srv, rx, slot, rows = _after_a_scaled_step(lost_next)
    st = srv.stats[slot]
    assert st.compressed + st.expanded >= 1
    kinds = [(r[0] >= 0, r[1] >= 0, r[2] >= 0) for step in rows for r in step]
    mixed = [i for i, step in enumerate(rows) if any(r[0] >= 0 and r[3] >= 0 for r in step)
             and any(r[0] >= 0 and (r[1] >= 0 or r[2] >= 0) and r[4] > 0 and r[5] != P - 1 for r in step)]
    assert mixed, rows
    step = rows[mixed[0]]
    last_real = max(i for i, r in enumerate(step) if r[1] == -1 and r[2] == -1)
    anchor_frame = step[last_real][0]
    after = step[last_real + 1:]
    assert after and all(r[0] == anchor_frame and r[3] == -1 for r in after)
    if lost_next:
        assert all(r[1] == _fid(4, 0) and r[2] == -1 for r in after) and st.concealed == 1
    else:
        assert all(r[1] == -1 and r[2] == 0 for r in after) and st.underruns >= 1
    assert any(k for k in kinds)
    call = len(rx.calls) - len(rows) + mixed[0]
    _, rows_raw, packed = rx.calls[call]
    sums = packed[:, :1].astype(np.float32)
    one = timescale_model(rows_raw, sums, np.zeros((2, 1), np.float32), np.array([[SILENCE]], np.float32))
    assert _bits(one) == _bits(_anchor_split(rx, call))


# ------------------------------------------------------------------ 6. a pause in the middle of an offset queue
def test_a_pause_drops_an_offset_queue_and_the_next_spurt_starts_aligned_with_a_fresh_window():
    srv, rx, _ = _rx(d=0, dmax=3, max_fade_packets=2)
    srv.open(1)
    slot = srv._ids[1]
    for t, qs in enumerate([[0], [], [1, 2], []]):                  # as _after_a_scaled_step: step 2 expands, then the sender stops
        for q in qs:
            srv.submit_packet(_pkt(1, q))
        srv.step()
    st = srv.stats[slot]
    assert st.expanded == 1 and len(srv._queue[slot]) == 1 and srv._playing[slot]     # an offset queue of one fade frame
    srv.step()                                                        # the second fade packet in a row: a pause
    _, rows, _ = rx.calls[-1]
    assert rows[:, 2].tolist() == [0] * P and rows[:, 4].tolist() == [P, P + 1, P + 2, P + 3, P + 4]
    assert st.pauses == 1 and not srv._playing[slot]
    assert srv._queue[slot] == [] and len(srv._lat[slot]) == 0 and srv._next[slot] == 3
    # the next spurt: packet 3 arrives 30 steps after its send time; the window holds its lateness alone
    for _ in range(30):
        srv.step()
    srv.submit_packet(_pkt(1, 3))
    srv.step()
    assert list(srv._lat[slot]) == [srv._steps - 1 - 3]
    _, rows, packed = rx.calls[-1]
    assert _rows_by_id(rows, packed) == [(_fid(3, i), -1, -1, slot if i == P - 1 else -1, 0, 0) for i in range(P)]
    assert st.delay_frames == P and srv._queue[slot] == []          # a fresh spurt at D = 0: Delta = Lambda = P, aligned


# ------------------------------------------------------------------ 7. moving sessions
def _migrate(when, arrivals, steps):
    ref, _, _ = _rx(d=1, dmax=4)
    a, _, _ = _rx(d=1, dmax=4)
    b, _, _ = _rx(d=1, dmax=4, cap=3)
    ref.open(8), a.open(8)
    b.open(1)                                                         # the destination serves someone: session 8 gets another slot
    for _ in range(3):
        b.step()                                                      # and has counted other steps
    got, want, cur, moved = [], [], a, None
    for t in range(steps):
        for q in arrivals.get(t, []):
            ref.submit_packet(_pkt(8, q))
            cur.submit_packet(_pkt(8, q))
        if cur is a and when(a, a._ids[8]):
            moved = a.detach(8)
            assert b.attach(moved) == 8
            cur = b
        ref.step()
        cur.step()
        want.extend(_drain(ref, 8))
        got.extend(_drain(cur, 8))
    assert moved is not None
    assert _bits(np.concatenate(got)) == _bits(np.concatenate(want))
    return moved, ref, b


SPIKE_THEN_STOP = {0: [0], 1: [1], 2: [], 3: [2], 6: [3, 4, 5, 6, 7], 7: [8], 8: [9], 9: [10], 10: [11], 11: [12]}


def test_detach_attach_while_buffering():
    st, ref, b = _migrate(lambda s, slot: len(s._held[slot]) == 1 and not s._playing[slot], {1: [0], 2: [1], 3: [2]}, 10)
    assert st.playout["queue"] == [] and st.playout["lateness"] == [1 - 1 - 0]


def test_detach_attach_in_the_middle_of_a_scaled_run():
    st, ref, b = _migrate(lambda s, slot: s.stats[slot].compressed + s.stats[slot].expanded == 1 and s._queue[slot], SPIKE_THEN_STOP,
                          30)
    assert st.playout["queue"] and all(e[0] == 0 for e in st.playout["queue"])
    sa, sb = ref.statistics()["per_session"][8], b.statistics()["per_session"][8]
    assert sa["delay_frames"] == sb["delay_frames"] and sa["target_delay"] == sb["target_delay"]


def test_detach_attach_in_the_middle_of_a_fade():
    st, ref, b = _migrate(lambda s, slot: s.stats[slot].underruns == 2, SPIKE_THEN_STOP, 40)
    assert st.playout["fades"] == 2 and st.anchor is not None and st.playout["anchor_frame"] is not None


def test_a_session_cannot_move_between_adaptive_and_fixed_receivers():
    a, _, _ = _rx(d=1, dmax=3)
    b, _, _ = _rx(d=1, dmax=None)
    a.open(1), b.open(2)
    with pytest.raises(ValueError, match="adaptive"):
        b.attach(a.detach(1))
    with pytest.raises(ValueError, match="adaptive"):
        a.attach(b.detach(2))


# ------------------------------------------------------------------ 8. refusals
@pytest.mark.parametrize("kw,field", [({"playout_delay": None}, "playout_delay"), ({"max_playout_delay": 1}, "max_playout_delay"),
                                      ({"frames_per_packet": 1}, "frames_per_packet"), ({"jitter_window": 1}, "jitter_window")])
def test_bad_arguments_are_refused(kw, field):
    args = dict(playout_delay=2, max_playout_delay=4, frames_per_packet=P)
    args.update(kw)
    with pytest.raises(ValueError, match=field):
        ReceiverSessionServer(FakeRx(), FakeDec(), capacity=2, **args)


def test_a_packet_of_another_frame_count_is_refused():
    srv, _, _ = _rx(d=1, dmax=3)
    srv.open(1)
    with pytest.raises(ValueError, match="frames"):
        srv.submit_packet(_pkt(1, 0, frames=P - 1))
    fixed, _, _ = _rx(d=1, dmax=None)
    fixed.open(1)
    assert fixed.submit_packet(_pkt(1, 0, frames=P - 1))              # the fixed clock takes short packets as before
