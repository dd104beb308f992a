"""Multi-stream duplex codec server (SURVEY.md 8(f) rank 3).

The reference's ``AudioCodecStreamer`` (bin/stream.py:80-366) serves ONE stream: a sound-card callback puts a frame on
``encoder_queue``, an encoder thread and a decoder thread each run a batch-1 model call per frame
(bin/stream.py:212-239), and ``_process`` (bin/stream.py:242-278) does the latency accounting and the frame-drop policy.
On an H100 one batch-1 call uses a sliver of the GPU, so this server generalises the same loop to N concurrent streams
that share every launch:

    submit(stream, frame)      <- what the sound-card callback does with ``indata``          (bin/stream.py:248-251)
    step()                     <- ONE encode -> quantize -> [pack -> unpack] -> lookup -> decode over all N streams
                                  (the bodies of _run_encoder / _run_decoder, bin/stream.py:212-239)
    poll(stream)               <- what the callback does to fill ``outdata``                   (bin/stream.py:253-272)

Streams advance in lock step: the causal state of all N streams lives in the codec handles as one (N, P, C) tensor per
layer and every launch moves every stream forward by exactly one frame.  A stream that has no frame queued when the step
runs is fed silence (counted as an ``underrun``); a stream whose backlog exceeds ``max_latency`` has its oldest frames
dropped (counted in ``frame_drops``), which is the reference's flush-when-late policy (bin/stream.py:262-270) applied
per stream.  The codec objects are duck-typed exactly like the reference's (``encode / quantize / lookup / decode``), so
the class also runs on stand-ins in the CPU tests.

SessionCodecServer advances only the open sessions that have audio, through stream slots.  TransmitterSessionServer and
ReceiverSessionServer split it at the wire: the first turns sessions' PCM into packets of packed code frames (audiodec_b200.wire), the
second turns packets back into PCM, so the two halves can run in different processes on different machines.
"""
from __future__ import annotations

import collections
import contextlib
import threading
import time
from typing import Deque, Dict, List, Optional, Tuple

import numpy as np
import torch

from .codec import ReceiverGraph, TransmitterGraph, is_library_codec
from .wire import HEADER_BYTES, Packet, decode_packet, encode_packet


class StreamStats:
    """Per-stream counters, same quantities as AudioCodecStreamer._exit prints (bin/stream.py:296-312)."""

    def __init__(self):
        self.n_frames = 0          # frames that went through the codec
        self.frame_drops = 0       # input frames discarded because the stream was running late
        self.underruns = 0         # steps in which the stream had nothing queued (silence was encoded instead)
        self.latencies: List[float] = []

    def as_dict(self):
        lat = np.asarray(self.latencies, dtype=np.float64)
        return {"n_frames": self.n_frames, "frame_drops": self.frame_drops, "underruns": self.underruns,
                "latency_ms": (float(lat.mean() * 1e3), float(lat.std() * 1e3)) if lat.size else (float("nan"), float("nan"))}


def _frame_in(frame, frame_size: int) -> np.ndarray:
    f = np.asarray(frame, dtype=np.float32).reshape(-1)
    if f.shape[0] != frame_size:
        raise ValueError(f"frame has {f.shape[0]} samples, server frame_size is {frame_size}")
    return f


def _queue_frame(q: Deque, item, max_backlog: int, stats: StreamStats) -> None:
    """Append (frame, capture stamp) to a stream's input queue; a stream running late loses its OLDEST frames (bin/stream.py:262-270)."""
    q.append(item)
    while len(q) > max_backlog:
        q.popleft()
        stats.frame_drops += 1


class MultiStreamCodecServer:
    """N lock-stepped duplex streams through one batched launch sequence per frame period.

    tx_encoder / rx_encoder / decoder: the three objects ``AudioDec.load_transmitter`` / ``load_receiver`` produce
    (bin/stream.py:56-77), already warmed for ONE stream; the first step replicates that warm state to ``n_streams``.
    frame_size: samples per frame per stream, a multiple of the codec hop (demoStream.py:28 default 1500 = 5 hops of 300).
    max_latency: seconds of backlog a stream may accumulate before its oldest frames are dropped (bin/stream.py:262).
    wire: if True the indices travel as the packed bitstream (``pack`` on the tx side, ``unpack`` on the rx side).
    """

    def __init__(self, tx_encoder, rx_encoder, decoder, n_streams: int, frame_size: int = 1500, sample_rate: int = 48000,
                 max_latency: float = 0.1, device=None, wire: bool = False, clock=time.time):
        if n_streams < 1:
            raise ValueError("n_streams must be >= 1")
        if frame_size < 1:
            raise ValueError("frame_size must be >= 1")
        self.tx_encoder, self.rx_encoder, self.decoder = tx_encoder, rx_encoder, decoder
        self.n_streams, self.frame_size, self.sample_rate = n_streams, frame_size, sample_rate
        self.max_latency, self.wire, self._clock = max_latency, wire, clock
        self.device = torch.device(device) if device is not None else None
        self.max_backlog = max(1, int(max_latency * sample_rate / frame_size))     # frames a stream may have queued
        self._in: List[Deque[Tuple[np.ndarray, float]]] = [collections.deque() for _ in range(n_streams)]
        self._out: List[Deque[np.ndarray]] = [collections.deque() for _ in range(n_streams)]
        self.stats = [StreamStats() for _ in range(n_streams)]
        self.step_times: List[float] = []
        self.wire_bytes = 0
        self._lock = threading.Lock()          # submit/poll may come from audio callbacks while step() runs in a worker
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self._x_host = None                    # pinned staging buffers, allocated on the first step
        self._x_np = None
        self._y_host = None
        self._graphs = None                    # (key, TransmitterGraph, ReceiverGraph) of the lock-step pass on library generators

    # ------------------------------------------------------------------ producer / consumer side (audio callbacks)
    def submit(self, stream: int, frame, t_capture: Optional[float] = None) -> None:
        """Queue one (frame_size,) float32 frame of stream `stream`.  Late streams lose their OLDEST queued frames."""
        f = _frame_in(frame, self.frame_size)
        with self._lock:
            _queue_frame(self._in[stream], (f, self._clock() if t_capture is None else t_capture), self.max_backlog, self.stats[stream])

    def poll(self, stream: int) -> Optional[np.ndarray]:
        """Next decoded (frame_size,) frame of `stream`, or None if the pipeline has nothing for it yet (the reference
        plays zeros in that case, bin/stream.py:273-274)."""
        with self._lock:
            q = self._out[stream]
            return q.popleft() if q else None

    def pending(self, stream: int) -> int:
        with self._lock:
            return len(self._in[stream])

    # ------------------------------------------------------------------ one batched step
    def _staging(self, like: torch.device):
        if self._x_host is None:
            pin = like.type == "cuda"
            self._x_host = torch.zeros(self.n_streams, 1, self.frame_size, dtype=torch.float32, pin_memory=pin)
            self._x_np = self._x_host.numpy()          # same memory: frames are copied in with numpy (≈1 us each, no tensor wrappers)
        return self._x_host

    def step(self) -> int:
        """Run the codec once over all streams.  Returns the number of streams that had a real frame this step."""
        t0 = self._clock()
        dev = self.device if self.device is not None else torch.device("cpu")
        x_host = self._staging(dev)
        x_np = self._x_np
        stamps: List[Optional[float]] = [None] * self.n_streams
        with self._lock:
            for s in range(self.n_streams):
                q = self._in[s]
                if q:
                    f, t = q.popleft()
                    x_np[s, 0] = f
                    stamps[s] = t
                else:
                    x_np[s, 0] = 0.0
                    self.stats[s].underruns += 1
        live = sum(t is not None for t in stamps)
        y_all, now = self._codec_pass(x_host, dev)
        with self._lock:
            for s in range(self.n_streams):
                t = stamps[s]
                if t is None:
                    continue                        # silence went in to keep the stream's state in step; nothing to play
                st = self.stats[s]
                self._out[s].append(y_all[s])
                st.n_frames += 1
                st.latencies.append(now - t)
        self.step_times.append(now - t0)
        return live

    def _codec_pass(self, x_host, dev, streams=None, codec_lock=None):
        """encode -> [wire] hand-off -> decode of the staged frames x_host (n, 1, frame_size), then the decoded frames back to the host.
        streams: the slots the frames advance (encode_streams / decode_streams), or None for all streams in lock step.  codec_lock is
        held while the codec runs.  Returns (decoded frames (n, frame_size) float32, the clock when they reached the host)."""
        n = x_host.shape[0]
        with torch.no_grad(), codec_lock or contextlib.nullcontext():
            if streams is None and dev.type == "cuda" and is_library_codec(self.tx_encoder, self.rx_encoder, self.decoder):
                y = self._graph_pass(x_host, dev)
            else:
                y = self._eager_pass(x_host, dev, streams)
            if y.device.type == "cuda":
                # device -> PINNED host buffer (a pageable destination is staged through a driver bounce buffer), then one synchronise
                if self._y_host is None or self._y_host.shape != y.shape or self._y_host.dtype != y.dtype:
                    self._y_host = torch.empty(y.shape, dtype=y.dtype, pin_memory=True)
                self._y_host.copy_(y, non_blocking=True)
                torch.cuda.current_stream(y.device).synchronize()
                y_host = self._y_host
            else:
                y_host = y
        now = self._clock()
        if y_host.dtype == torch.bfloat16:
            y_host = y_host.float()             # a bf16-activation decoder: half the D2H bytes, widened here; frames out stay float32
        return y_host.numpy().reshape(n, -1)[:, :self.frame_size].copy(), now    # one copy; the queues hold row views of it

    def _eager_pass(self, x_host, dev, streams):
        """The codec calls one by one (duck-typed codec objects, and the slot calls of SessionCodecServer) -> decoded frames."""
        n = x_host.shape[0]
        x = x_host.to(dev, non_blocking=True)
        if streams is None:
            z = self.tx_encoder.encode(x)                                   # utils/audiodec.py:100-102
        else:
            z, frames = self.tx_encoder.encode_streams(list(x.view(n, -1)), streams)
        if self.wire and hasattr(self.tx_encoder, "quantize_fused") and hasattr(self.rx_encoder, "lookup_packed"):
            # the RVQ kernel writes the bitstream itself; the receiver looks the codewords up straight from the packed bytes
            _, packed, _ = self.tx_encoder.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)
            self.wire_bytes += packed.numel()
            zq = self.rx_encoder.lookup_packed(packed)
        elif self.wire:
            packed = self.tx_encoder.pack(self.tx_encoder.quantize(z))
            self.wire_bytes += packed.numel()
            zq = self.rx_encoder.lookup(self.rx_encoder.unpack(packed))
        else:
            zq = self.rx_encoder.lookup(self.tx_encoder.quantize(z))
        if streams is None:
            return self.decoder.decode(zq).detach()                         # utils/audiodec.py:104-106
        # every chunk is frame_size samples: equal frame counts
        return torch.cat([v.reshape(1, -1) for v in self.decoder.decode_streams(zq, frames, streams)]).detach()

    def _graph_pass(self, x_host, dev):
        """The lock-step pass on the library's generators as two graph launches (TransmitterGraph, ReceiverGraph), bit for bit the eager
        calls.  The graphs are built on the first step and again when the shape or a generator's handle changes.  Returns the decoded
        frames on the device (the ReceiverGraph's static output, read before the next step)."""
        n, t = x_host.shape[0], x_host.shape[-1]
        wire = bool(self.wire)
        key = (n, t, wire, dev, tuple(g._h.value for g in (self.tx_encoder, self.rx_encoder, self.decoder)))
        if self._graphs is None or self._graphs[0] != key:
            self._graphs = None
            frames = self.tx_encoder._lib.adec_frames_for(self.tx_encoder._h, t)
            self._graphs = (key, TransmitterGraph(self.tx_encoder, n, t, wire=wire),
                            ReceiverGraph(self.rx_encoder, self.decoder, n, frames, wire=wire))
        _, txg, rxg = self._graphs
        txg.input.copy_(x_host, non_blocking=True)
        out = txg(txg.input)
        if wire:
            self.wire_bytes += out.numel()
        return rxg(out)

    # ------------------------------------------------------------------ real-time loop (the two worker threads of the reference, merged)
    def start(self, period: Optional[float] = None) -> None:
        """Tick `step()` every `period` seconds (default: the frame period) on a daemon thread until `stop()`."""
        if self._thread is not None:
            return
        period = self.frame_size / self.sample_rate if period is None else period
        self._stop.clear()

        def loop():
            nxt = time.time()
            while not self._stop.is_set():
                self.step()
                nxt += period
                delay = nxt - time.time()
                if delay > 0:
                    self._stop.wait(delay)
                else:
                    nxt = time.time()               # running behind: do not try to catch up, the drop policy handles backlog

        self._thread = threading.Thread(target=loop, daemon=True)
        self._thread.start()

    def stop(self) -> None:
        self._stop.set()
        if self._thread is not None:
            self._thread.join()
            self._thread = None

    # ------------------------------------------------------------------ reporting
    def statistics(self) -> Dict:
        st = np.asarray(self.step_times, dtype=np.float64)
        per_stream = [s.as_dict() for s in self.stats]
        lat = np.concatenate([np.asarray(s.latencies, dtype=np.float64) for s in self.stats]) if self.stats else np.zeros(0)
        frames = sum(p["n_frames"] for p in per_stream)
        return {
            "n_streams": self.n_streams, "steps": int(st.size),
            "step_ms": (float(st.mean() * 1e3), float(st.std() * 1e3)) if st.size else (float("nan"), float("nan")),
            "latency_ms": (float(lat.mean() * 1e3), float(lat.std() * 1e3)) if lat.size else (float("nan"), float("nan")),
            "frames": frames, "frame_drops": sum(p["frame_drops"] for p in per_stream),
            "underruns": sum(p["underruns"] for p in per_stream),
            "realtime_factor": (frames * self.frame_size / self.sample_rate) / float(st.sum()) if st.size and st.sum() > 0 else float("nan"),
            "wire_kbps_per_stream": (8e-3 * self.wire_bytes / self.n_streams) / (st.size * self.frame_size / self.sample_rate)
                                    if self.wire and st.size else None,
            "per_stream": per_stream,
        }


class SessionState:
    """What a detached session needs to continue on another server of the same kind (same config and dtypes, on any device): per
    stateful generator of the server its state_layout and its (1, S) device state, the queued input (frames with their capture stamps
    on SessionCodecServer and TransmitterSessionServer, held packets on ReceiverSessionServer), and the decoded frames it has not polled
    yet.  On the split servers also the session's wire id and the next sequence number it sends or expects.  On a ReceiverSessionServer
    that conceals losses also the fp32 anchor row (the lookup sum of the session's last real frame, a (code_dim,) device tensor, None
    before its first real frame) and the concealment still pending, (packets left, frames per packet, frames concealed so far, frames in
    the gap), or None.  On a ReceiverSessionServer with a playout clock also `playout`, a dict of the playout position: whether the
    session is playing, the steps each held packet has waited (in the order of `inputs`), the frames concealed or faded since the last
    real frame, the consecutive fade packets, the last real packet's frame count and the sequence numbers given up by the clock, and with
    an adaptive delay also the content queue (frames not yet played; o is frames_per_packet minus their count), the frame the anchor
    was taken from, and the talk spurt's lateness window (relative to the step count); None elsewhere."""

    def __init__(self, layouts, states, inputs, outputs, session_id=None, seq=0, anchor=None, conceal=None, playout=None):
        self.layouts: List[list] = layouts
        self.states: List[torch.Tensor] = states
        self.inputs: list = inputs
        self.outputs: List[np.ndarray] = outputs
        self.session_id: Optional[int] = session_id
        self.seq: int = seq
        self.anchor: Optional[torch.Tensor] = anchor
        self.conceal: Optional[Tuple[int, int, int, int]] = conceal
        self.playout: Optional[dict] = playout

    def to(self, device) -> "SessionState":
        """A copy with the states and the anchor on `device` (the frames are host arrays and are shared)."""
        return SessionState(self.layouts, [t.to(device) for t in self.states], list(self.inputs), list(self.outputs), self.session_id,
                            self.seq, None if self.anchor is None else self.anchor.to(device), self.conceal, self.playout)


class _SessionSlots:
    """The slot bookkeeping of the session servers.  Every stateful generator holds `capacity` stream slots plus one template slot (the
    last) with the warm state that ``load_transmitter`` / ``load_receiver`` left in it; the template is never advanced.  A session is
    opened in a free slot from the template or attached from a detached SessionState, and is known to the caller by an id: the slot
    itself (``_open_slot()``) or an id the caller chose (``_open_slot(sid)``).  Subclasses keep their per-slot queues and counters and
    say how to clear, export and import them (``_reset_slot`` / ``_take_slot`` / ``_restore_slot``, called with ``_lock`` held).

    Locks: ``_lock`` guards the queues and the slot lists (submit / poll may come from audio callbacks while step() runs in a worker),
    ``_codec_lock`` the generators (driven by step(), open() and attach() from different threads), ``_step_lock`` a whole step, output
    hand-off included, so that detach() waits for it."""

    _noun = "stream"

    def __init__(self, capacity: int, stateful):
        if capacity < 1:
            raise ValueError("capacity must be >= 1")
        self.capacity = capacity
        self.template = capacity                      # slot index of the warm template
        stateful = tuple(stateful)
        self._stateful = [g for i, g in enumerate(stateful) if g not in stateful[:i]]
        for g in self._stateful:
            if g.n_streams != 1:                      # growing from more than one stream adds zero-history slots: a cold template
                raise ValueError(f"{type(g).__name__} holds {g.n_streams} streams; {type(self).__name__} needs generators with the one "
                                 "warmed stream that load_transmitter / load_receiver leave")
        for g in self._stateful:
            g.set_streams(capacity + 1)               # replicates the one warmed stream into every slot
        self._free = list(range(capacity))
        self._open: set = set()
        self._ids: Dict[int, int] = {}                # session id -> slot
        self._session = [0] * capacity                # per slot: bumped by every open, so a step hands out only its own session's frames
        self._lock = threading.Lock()
        self._codec_lock = threading.Lock()
        self._step_lock = threading.Lock()

    def _reset_slot(self, s: int) -> None:
        raise NotImplementedError

    def _take_slot(self, s: int):
        """-> (inputs, outputs, seq) of slot s, leaving its queues empty"""
        raise NotImplementedError

    def _restore_slot(self, s: int, state: SessionState) -> None:
        raise NotImplementedError

    def _export_slot(self, s: int) -> dict:
        """-> the SessionState keywords of what slot s carries besides its queues and causal state (called before _take_slot)"""
        return {}

    def _slot(self, sid) -> int:
        s = self._ids.get(sid)
        if s is None or s not in self._open:
            raise KeyError(f"{self._noun} {sid} is not open")
        return s

    def _claim(self, sid):
        """A free slot for session `sid` (None: the slot is the id) -> (sid, slot); the slot is reserved, not yet open.  _lock held."""
        if sid is not None and sid in self._ids:
            raise ValueError(f"{self._noun} {sid} is already open")
        if not self._free:
            raise RuntimeError(f"server is full: all {self.capacity} streams are open")
        s = min(self._free)
        self._free.remove(s)
        self._session[s] += 1
        sid = s if sid is None else sid
        self._ids[sid] = s
        return sid, s

    def _open_slot(self, sid=None):
        """Start a session in a free slot, warm as the template; returns its id."""
        with self._lock:
            sid, s = self._claim(sid)
            self._reset_slot(s)
        with self._codec_lock:
            for g in self._stateful:
                g.copy_stream_state(self.template, [s])
        with self._lock:
            self._open.add(s)
        return sid

    def _close_slot(self, sid) -> None:
        with self._lock:
            s = self._slot(sid)
            self._open.remove(s)
            del self._ids[sid]
            self._reset_slot(s)
            self._free.append(s)

    def _detach_slot(self, sid) -> SessionState:
        with self._step_lock:
            with self._lock:
                s = self._slot(sid)
                self._open.remove(s)
                del self._ids[sid]
                extra = self._export_slot(s)
                inputs, outputs, seq = self._take_slot(s)
            with self._codec_lock:       # the slot stays taken until its state is out
                states = [g.stream_state([s]) for g in self._stateful]
            layouts = [list(g.state_layout) for g in self._stateful]
            with self._lock:
                self._free.append(s)
        return SessionState(layouts, states, inputs, outputs, seq=seq, **extra)

    def _attach_slot(self, state: SessionState, sid=None):
        if len(state.states) != len(self._stateful) or len(state.layouts) != len(self._stateful):
            raise ValueError(f"the session holds the state of {len(state.states)} generators; this server has {len(self._stateful)}")
        for g, layout in zip(self._stateful, state.layouts):
            if [tuple(e) for e in layout] != [tuple(e) for e in g.state_layout]:
                raise ValueError(f"the session's state layout does not match this server's {type(g).__name__}")
        with self._lock:
            sid, s = self._claim(sid)
        try:
            with self._codec_lock:
                for g, layout, t in zip(self._stateful, state.layouts, state.states):
                    g.load_stream_state([s], t, layout)
        except Exception:
            with self._lock:
                del self._ids[sid]
                self._free.append(s)
            raise
        with self._lock:
            self._restore_slot(s, state)
            self._open.add(s)
        return sid


class SessionCodecServer(_SessionSlots, MultiStreamCodecServer):
    """Duplex streams that open and close while others run, each advanced only when it has audio.

    The codec handles hold ``capacity`` stream slots plus one template slot (the last) with the warm state that
    ``load_transmitter`` / ``load_receiver`` left in the objects; the template is never advanced.  ``open()`` copies the template
    into a free slot, so a new caller starts exactly where a freshly warmed codec starts and inherits nothing of the slot's previous
    caller.  ``step()`` runs ONE slot call per codec stage (``encode_streams`` -> quantize -> ``decode_streams``) over the open
    streams that have a frame queued: idle streams are not fed silence, their causal state stays as it is, and a step costs what
    its streams cost, not what the capacity costs.  ``submit`` / ``poll`` / the drop policy / ``start`` / ``stop`` are the lock-step
    server's; the per-stream counters in ``statistics()`` are per slot.  ``detach()`` closes a stream and returns its causal state and its
    queued and undelivered frames; ``attach()`` continues it in a free slot of this or another server, on any device.  The generators must hold ONE warmed stream when the server is
    built (what load_transmitter / load_receiver leave), since only that stream is replicated into the slots.
    """

    def __init__(self, tx_encoder, rx_encoder, decoder, capacity: int, frame_size: int = 1500, sample_rate: int = 48000,
                 max_latency: float = 0.1, device=None, wire: bool = False, clock=time.time):
        MultiStreamCodecServer.__init__(self, tx_encoder, rx_encoder, decoder, capacity, frame_size=frame_size, sample_rate=sample_rate,
                                        max_latency=max_latency, device=device, wire=wire, clock=clock)
        _SessionSlots.__init__(self, capacity, (tx_encoder, decoder))

    def _reset_slot(self, s):
        self._in[s].clear()
        self._out[s].clear()

    def _take_slot(self, s):
        inputs, outputs = list(self._in[s]), list(self._out[s])
        self._reset_slot(s)
        return inputs, outputs, 0

    def _restore_slot(self, s, state):
        self._reset_slot(s)
        self._in[s].extend(state.inputs)
        self._out[s].extend(state.outputs)
        self.stats[s] = StreamStats()

    # ------------------------------------------------------------------ sessions
    def open(self) -> int:
        """Start a stream in a free slot, warm as the template; returns its id.  Raises RuntimeError when every slot is taken."""
        return self._open_slot()

    def close(self, stream: int) -> None:
        """End stream `stream`: its slot becomes free and its queued input and output are dropped."""
        self._close_slot(stream)

    def detach(self, stream: int) -> SessionState:
        """Close stream `stream` and return what it needs to continue elsewhere (attach(), on this or another server): its causal state
        in every stateful generator, its queued input frames and its undelivered output frames.  Waits for a step in progress to finish
        and hand off its frames, so no frame in flight is lost.  Raises KeyError if the stream is not open."""
        return self._detach_slot(stream)

    def attach(self, state: SessionState) -> int:
        """Open a stream in a free slot from a detached session instead of the template: it continues exactly where it left off, with
        its queued and undelivered frames, and fresh per-stream counters.  The state must be on this server's device (SessionState.to).
        Raises ValueError if the session comes from codecs of another layout, RuntimeError when every slot is taken."""
        return self._attach_slot(state)

    @property
    def open_streams(self) -> List[int]:
        with self._lock:
            return sorted(self._open)

    def submit(self, stream: int, frame, t_capture: Optional[float] = None) -> None:
        if stream not in self._open:
            raise KeyError(f"stream {stream} is not open")
        super().submit(stream, frame, t_capture)

    # ------------------------------------------------------------------ one step over the streams that have audio
    def step(self) -> int:
        """Advance every open stream that has a frame queued by that frame.  Returns the number of streams advanced."""
        with self._step_lock:
            return self._step()

    def _step(self) -> int:
        t0 = self._clock()
        dev = self.device if self.device is not None else torch.device("cpu")
        x_host = self._staging(dev)
        x_np = self._x_np
        streams: List[int] = []
        stamps: List[float] = []
        sessions: List[int] = []
        with self._lock:
            for s in sorted(self._open):
                q = self._in[s]
                if q:
                    f, t = q.popleft()
                    x_np[len(streams), 0] = f
                    streams.append(s)
                    stamps.append(t)
                    sessions.append(self._session[s])
                else:
                    self.stats[s].underruns += 1
        n = len(streams)
        if n == 0:
            self.step_times.append(self._clock() - t0)
            return 0
        y_all, now = self._codec_pass(x_host[:n], dev, streams, self._codec_lock)
        with self._lock:
            for k, s in enumerate(streams):
                if s not in self._open or self._session[s] != sessions[k]:
                    continue                        # closed (and maybe reopened by a new caller) while the step ran: the frame is dropped
                st = self.stats[s]
                self._out[s].append(y_all[k])
                st.n_frames += 1
                st.latencies.append(now - stamps[k])
        self.step_times.append(now - t0)
        return n

    def statistics(self) -> Dict:
        """The lock-step server's report, with `n_streams` = the streams open now, `capacity`, and the wire bitrate per second of
        audio actually advanced (streams come and go, so neither the capacity nor the steps divide it)."""
        out = super().statistics()
        n_open = len(self.open_streams)
        out["capacity"] = self.capacity
        out["n_streams"] = out["open_streams"] = n_open
        frames = out["frames"]
        out["wire_kbps_per_stream"] = (8e-3 * self.wire_bytes) / (frames * self.frame_size / self.sample_rate) if self.wire and frames else None
        return out


def _pinned(n: int, dtype, device) -> torch.Tensor:
    """A 1-D host buffer of n elements, page-locked when the codec runs on a GPU (a pageable copy is staged by the driver)."""
    return torch.empty(n, dtype=dtype, pin_memory=device.type == "cuda")


def _ms(times: List[float]):
    st = np.asarray(times, dtype=np.float64)
    return (float(st.mean() * 1e3), float(st.std() * 1e3)) if st.size else (float("nan"), float("nan"))


class TransmitterSessionServer(_SessionSlots):
    """The sending half of SessionCodecServer: sessions of PCM frames in, one wire packet (audiodec_b200.wire) per session per step out.

    tx_encoder: a SymADStreamGenerator or SymADEncoderStreamGenerator in any dtype mode, holding the one warmed stream
    ``load_transmitter`` leaves.  Sessions are known by a u32 id the caller chooses and shares with the receiver: ``open(session_id)``
    starts one warm from the template slot, ``close`` ends it, ``detach`` / ``attach`` move its causal state, its queued frames and its
    next sequence number to another transmitter server.  ``submit`` queues a (frame_size,) frame with the lock-step server's drop
    policy.  ``step()`` runs ONE ``encode_streams`` over the open sessions that have a frame queued, ONE fused quantize that writes the
    packed bytes, and ONE device-to-host copy of only those bytes; ``poll_packets()`` returns the packets made so far as
    (session_id, bytes), in step order and, within a step, in session id order.  Packets already made stay with the server that made
    them when their session is detached.  Moving the bytes to the receiver is the caller's business."""

    _noun = "session"

    def __init__(self, tx_encoder, capacity: int, frame_size: int = 1500, sample_rate: int = 48000, max_latency: float = 0.1,
                 device=None):
        if frame_size < 1:
            raise ValueError("frame_size must be >= 1")
        self.tx_encoder = tx_encoder
        self.frame_size, self.sample_rate, self.max_latency = frame_size, sample_rate, max_latency
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.max_backlog = max(1, int(max_latency * sample_rate / frame_size))     # frames a session may have queued
        super().__init__(capacity, (tx_encoder,))
        self._in: List[Deque[Tuple[np.ndarray, float]]] = [collections.deque() for _ in range(capacity)]
        self._seq = [0] * capacity
        self.stats = [StreamStats() for _ in range(capacity)]
        self._packets: Deque[Tuple[int, bytes]] = collections.deque()
        self.step_times: List[float] = []
        self.wire_bytes = 0
        self._x_host = _pinned(capacity * frame_size, torch.float32, self.device).view(capacity, frame_size)
        self._x_np = self._x_host.numpy()
        self._p_host = None                            # the packed bytes of a step, sized on the first step

    def _reset_slot(self, s):
        self._in[s].clear()
        self._seq[s] = 0
        self.stats[s] = StreamStats()

    def _take_slot(self, s):
        inputs, seq = list(self._in[s]), self._seq[s]
        self._reset_slot(s)
        return inputs, [], seq

    def _restore_slot(self, s, state):
        self._reset_slot(s)
        self._in[s].extend(state.inputs)
        self._seq[s] = state.seq

    # ------------------------------------------------------------------ sessions
    def open(self, session_id: int) -> int:
        """Start session `session_id` (a u32) warm as the template.  ValueError if it is open already, RuntimeError when every slot
        is taken."""
        if not 0 <= session_id < 1 << 32:
            raise ValueError(f"session id {session_id} does not fit in a u32")
        return self._open_slot(session_id)

    def close(self, session_id: int) -> None:
        """End the session: its slot becomes free and its queued frames are dropped."""
        self._close_slot(session_id)

    def detach(self, session_id: int) -> SessionState:
        """Close the session and return its causal state, queued frames and next sequence number (waits for a step in progress)."""
        state = self._detach_slot(session_id)
        state.session_id = session_id
        return state

    def attach(self, state: SessionState) -> int:
        """Continue a session detached from a transmitter server of the same config and dtype, under its own id, from its next
        sequence number.  The state must be on this server's device (SessionState.to)."""
        if state.session_id is None:
            raise ValueError("the session has no wire session id: it was not detached from a transmitter server")
        return self._attach_slot(state, state.session_id)

    @property
    def open_sessions(self) -> List[int]:
        with self._lock:
            return sorted(self._ids)

    def submit(self, session_id: int, frame, t_capture: Optional[float] = None) -> None:
        """Queue one (frame_size,) float32 frame of the session.  A late session loses its OLDEST queued frames."""
        f = _frame_in(frame, self.frame_size)
        with self._lock:
            s = self._slot(session_id)
            _queue_frame(self._in[s], (f, time.time() if t_capture is None else t_capture), self.max_backlog, self.stats[s])

    def pending(self, session_id: int) -> int:
        with self._lock:
            return len(self._in[self._slot(session_id)])

    def poll_packets(self) -> List[Tuple[int, bytes]]:
        """Every packet made since the last call, as (session_id, bytes), in the order the steps made them."""
        with self._lock:
            out = list(self._packets)
            self._packets.clear()
        return out

    # ------------------------------------------------------------------ one step
    def step(self) -> int:
        """Encode one queued frame of every open session that has one, into one packet each.  Returns the number of packets made."""
        with self._step_lock:
            return self._step()

    def _step(self) -> int:
        t0 = time.time()
        slots, sids, stamps, sessions = [], [], [], []
        with self._lock:
            for sid, s in sorted(self._ids.items()):
                if s not in self._open:
                    continue
                q = self._in[s]
                if q:
                    f, t = q.popleft()
                    self._x_np[len(slots)] = f
                    slots.append(s)
                    sids.append(sid)
                    stamps.append(t)
                    sessions.append(self._session[s])
                else:
                    self.stats[s].underruns += 1
        n = len(slots)
        if n == 0:
            self.step_times.append(time.time() - t0)
            return 0
        tx = self.tx_encoder
        with torch.no_grad(), self._codec_lock:
            x = self._x_host[:n].to(self.device, non_blocking=True)
            z, frames = tx.encode_streams(list(x), slots)
            _, packed, _ = tx.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)    # (sum F, frame_bytes)
            nb = packed.shape[-1]
            if self._p_host is None or self._p_host.numel() < packed.numel():
                self._p_host = _pinned(max(packed.numel(), self.capacity * frames[0] * nb), torch.uint8, self.device)
            p_host = self._p_host[:packed.numel()]
            p_host.copy_(packed.reshape(-1), non_blocking=True)
            if packed.device.type == "cuda":
                torch.cuda.current_stream(packed.device).synchronize()
        now = time.time()
        buf = p_host.numpy()
        made = 0
        with self._lock:
            o = 0
            for k, s in enumerate(slots):
                payload = buf[o * nb:(o + frames[k]) * nb]
                o += frames[k]
                if s not in self._open or self._session[s] != sessions[k]:
                    continue                        # closed while the step ran: no packet, and no sequence number spent
                pkt = encode_packet(sids[k], self._seq[s], tx.codebook_num, nb, payload)
                self._seq[s] += 1
                self._packets.append((sids[k], pkt))
                self.wire_bytes += len(pkt)
                st = self.stats[s]
                st.n_frames += 1
                st.latencies.append(now - stamps[k])
                made += 1
        self.step_times.append(now - t0)
        return made

    def statistics(self) -> Dict:
        """steps, ms per step (mean, std), the open sessions and, per open session, the input counters of StreamStats (n_frames: frames
        encoded here) and the next sequence number."""
        with self._lock:
            per = {sid: dict(self.stats[s].as_dict(), next_seq=self._seq[s]) for sid, s in sorted(self._ids.items())}
        return {"capacity": self.capacity, "open_sessions": len(per), "steps": len(self.step_times), "step_ms": _ms(self.step_times),
                "wire_bytes": self.wire_bytes, "per_session": per}


class ReceiveStats:
    """Per-session counters of a ReceiverSessionServer."""

    def __init__(self):
        self.packets = 0           # packets decoded
        self.frames = 0            # code frames decoded
        self.bytes = 0             # wire bytes of the decoded packets, headers included
        self.samples = 0           # PCM samples decoded
        self.duplicates = 0        # packets dropped because the session had already decoded, held or given up their sequence number
        self.reorders = 0          # packets that arrived after a packet with a higher sequence number and were put back in order
        self.losses = 0            # sequence numbers given up as lost
        self.concealed = 0         # lost sequence numbers decoded as concealed packets (conceal_packets > 0)
        self.concealed_frames = 0  # code frames of those packets
        self.late = 0              # packets dropped because the playout clock had given their sequence number up (playout_delay)
        self.underruns = 0         # playout steps with nothing held: a fade packet was played
        self.faded_frames = 0      # code frames of those fade packets
        self.pauses = 0            # times the session stopped playing after max_fade_packets fade packets in a row
        self.compressed = 0        # adaptive playout steps that played frames_per_packet + 1 content frames
        self.expanded = 0          # adaptive playout steps that played frames_per_packet - 1 content frames
        self.delay_frames = None   # the delay in code frames at the session's last adaptive playout step

    def as_dict(self, sample_rate, buffered=None, target=None):
        """packets, frames and wire_kbps count the real packets only; buffered (the packets held ahead of the playout point) adds the
        playout counters, target (the adaptive clock's target delay in packets) the adaptive ones"""
        out = {"packets": self.packets, "frames": self.frames, "duplicates": self.duplicates, "reorders": self.reorders,
               "losses": self.losses, "concealed": self.concealed, "concealed_frames": self.concealed_frames,
               "wire_kbps": 8e-3 * self.bytes / (self.samples / sample_rate) if self.samples else None}
        if buffered is not None:
            out.update(late=self.late, underruns=self.underruns, faded_frames=self.faded_frames, pauses=self.pauses, buffered=buffered)
        if target is not None:
            out.update(target_delay=target, delay_frames=self.delay_frames, compressed=self.compressed, expanded=self.expanded)
        return out


class ReceiverSessionServer(_SessionSlots):
    """The receiving half of SessionCodecServer: wire packets (audiodec_b200.wire) in, decoded PCM frames per session out.

    rx_encoder: a SymADStreamGenerator, for its codebooks (as in ``load_receiver``).  decoder: any of the library's decoders in any dtype
    mode, holding the one warmed stream ``load_receiver`` leaves; bf16 output (bf16 activations) is widened to float32 frames.
    frames_per_packet: the most code frames a packet may carry (the transmitter's frame_size over the codec hop), which sizes the
    staging buffers.  ``open(session_id)`` binds a remote session to a warm slot; ``close``, ``detach`` and ``attach`` move the
    decoder state, the held packets and the undelivered PCM frames.

    ``submit_packet(bytes)`` parses and checks a packet (ValueError when it is malformed or made for another codec).  The defined
    receive behaviour, per session: sequence numbers start at 0 and do not wrap.  A packet whose session is not open is counted
    (``unknown_session_packets``) and dropped.  A packet whose sequence number the session has already decoded, holds or given up as
    lost is counted in ``duplicates`` and dropped.  Packets are decoded in sequence order; one that arrives early is held.  When
    ``reorder_window`` packets are held behind a missing one and another arrives (or a step finds more than that many), the missing
    sequence numbers are counted as ``losses`` and decoding continues with the next packet held.  With ``conceal_packets = 0`` (the
    default) nothing is concealed: the decoder advances only by the frames it received, so a loss shortens the session's output by the
    lost packets' frames.

    ``conceal_packets = K > 0`` conceals losses.  When a session gives up a gap of G sequence numbers in front of held packet b, the
    last min(G, K) of them are decoded as concealed packets of b.frames frames each (any earlier ones stay lost), one per step and in
    sequence order, before b; their PCM is queued for ``poll`` like a real packet's, so the output stays in step with the sender and
    the decoder's causal state runs through the gap.  Concealed frame j of the M = min(G, K) * b.frames frames in the gap is the fp32
    interpolation a + fl(j / (M + 1)) * (s_b - a), each operation rounded on its own, between a, the lookup sum of the session's last
    real frame, and s_b, the sum of b's first frame (s_b alone if the session has decoded no real frame yet); a decoder with bf16
    activations gets it rounded once to bf16.  ``losses`` still counts all G; ``concealed`` and ``concealed_frames`` count what was
    concealed, and the other counters count real packets only.  A loss needs a following packet to be concealed, so one at the end of
    a talk spurt waits as before.  A late packet for a concealed sequence number is a duplicate.

    ``step()`` takes the next in-order packet of every open session that has one, copies their payloads to the device in ONE copy,
    runs ONE ``lookup_packed`` over the concatenated frames and ONE ``decode_streams`` with each session's frame count, and copies the
    PCM back in ONE copy.  With concealment the lookup is ONE ``lookup_packed_conceal`` instead, which also keeps every session's
    anchor row (a (capacity, code_dim) fp32 device tensor); a session that conceals this step stages b's first frame in place of a
    payload.  ``poll(session_id)`` returns the session's next decoded frame (frames x hop float32 samples) or None.  ``detach`` /
    ``attach`` also carry the anchor row and any concealment still pending; a receiver without concealment drops them.

    ``playout_delay = D`` (None, the default, is the receiver above) runs a playout clock instead: a fixed-delay jitter buffer in which
    ``step()`` is one packet period, ticked by the caller at the packet rate, and every playing session gets exactly one packet of PCM
    per step.  ``submit_packet`` stamps a packet with the steps completed so far; one whose sequence number the session has decoded or
    holds is a duplicate, one the clock has already given up is ``late``; both are dropped, and nothing is given up for the reorder
    window.  A session starts playing at the first step where it holds a packet stamped at least D steps earlier.  Then, each step:
    (1) the next packet is held: it is decoded.  (2) It is missing but a later packet m is held: one loss, and the next packet is
    concealed as m.frames frames interpolated from the anchor (the session's last real frame) toward m's first frame, j = c + 1 ...
    c + m.frames and den = c + (m - next) * m.frames + 1, where c counts the frames concealed or faded since the last real frame (m's
    first frame itself with no anchor).  (3) Nothing is held: an underrun, played as a fade packet of the last real packet's frame
    count (frames_per_packet before any) whose frames go from the anchor toward the codec's silence frame, j = c + 1 ... and
    den = ``fade_frames``, the silence frame itself from j >= den on.  Rules 2 and 3 give the sequence number up.  After
    ``max_fade_packets`` fade packets in a row the session pauses: it goes back to buffering and rewinds to the first sequence number
    the fades gave up, so a sender that went quiet resumes at its own next packet; the decoder state runs on through the fade.  Each
    step is ONE ``lookup_packed_playout`` over real, interpolated and fade rows (descriptors in two page-locked tables used in turn)
    and ONE ``decode_streams``.  The silence frame is ``rx_encoder.silence_frame()`` unless ``silence_frame`` gives one.  This is a
    continuity and timing rule: it keeps every session's output running at the packet rate; how the concealed and faded audio sounds
    is not claimed.  ``detach`` / ``attach`` carry the playout position (SessionState.playout) between playout receivers; a session
    cannot move between a playout receiver and one without.

    ``max_playout_delay = D_max`` (with ``playout_delay = D``, D <= D_max) adapts the delay to the jitter it measures, by playing
    buffered content faster or slower in the latent domain.  Every packet must then carry P = frames_per_packet >= 2 frames.  Rules 1 - 3
    above, unchanged, fill a per-session queue of content frames one packet at a time; every step plays exactly P output frames of every
    playing session, made from C = P - 1, P or P + 1 content frames.  Each packet that is not a duplicate (late ones included) has
    lateness stamp - seq; the session keeps the last ``jitter_window`` of the current talk spurt (a pause clears them).  The target is
    T = min(max(J, D), D_max) packets with J = max - min of that window (0 with fewer than two values); a buffering session starts
    playing under the rule above with T for D.  The delay at step k (steps completed) is Delta = (k - min lateness + 1) * P - p frames,
    p = q * P + o, where q is the sequence number of the next content frame and o the frames of it already played; without jitter it
    stays at Lambda = (T + 1) * P.  With L the real frames available in a row from the playout point (queued, then held in sequence),
    a step compresses (C = P + 1) when Delta > Lambda and L >= P + 1, else expands (C = P - 1) when Delta < Lambda and L >= P - 1, else
    plays C = P; so only runs of real frames are scaled.  Output frame i of a scaled window q_0 ... q_{C-1} is, with
    m, r = divmod(i * (C - 1), P - 1), the real frame q_m when r = 0 and otherwise q_m interpolated toward q_{m+1} with j = r,
    den = P - 1; the first and last output frames are real.  A concealed or fade frame that shares a step with the real frame it
    starts from is computed from that frame staged in the same launch.  The pause of rule 3 plays the rest of that step's P frames from
    the fade packet, then drops the queue.  Each step is ONE ``lookup_packed_timescale`` and ONE ``decode_streams``.  statistics() adds
    target_delay, delay_frames, compressed and expanded; a session moves only between two adaptive receivers.  When every step plays
    C = P from o = 0 (a jitter-free session, for one), the rows and the PCM are the fixed clock's."""

    _noun = "session"
    reorder_window = 4                 # packets held behind a missing one before it is given up

    def __init__(self, rx_encoder, decoder, capacity: int, frames_per_packet: int, sample_rate: int = 48000, device=None,
                 conceal_packets: int = 0, playout_delay: Optional[int] = None, fade_frames: Optional[int] = None,
                 max_fade_packets: int = 4, silence_frame=None, max_playout_delay: Optional[int] = None, jitter_window: int = 64):
        if frames_per_packet < 1:
            raise ValueError("frames_per_packet must be >= 1")
        if max_playout_delay is not None:
            if playout_delay is None:
                raise ValueError("max_playout_delay needs playout_delay: the delay adapts between the two")
            if max_playout_delay < playout_delay:
                raise ValueError(f"max_playout_delay = {max_playout_delay} is below playout_delay = {playout_delay}")
            if frames_per_packet < 2:
                raise ValueError("frames_per_packet must be >= 2 with max_playout_delay: a scaled step interpolates between frames")
            if jitter_window < 2:
                raise ValueError("jitter_window must be >= 2")
        if conceal_packets < 0:
            raise ValueError("conceal_packets must be >= 0")
        if playout_delay is not None:
            if conceal_packets:
                raise ValueError("playout_delay and conceal_packets > 0 exclude each other: the playout clock conceals by itself")
            if playout_delay < 0:
                raise ValueError("playout_delay must be >= 0")
            fade_frames = 2 * frames_per_packet if fade_frames is None else fade_frames
            if fade_frames < 1:
                raise ValueError("fade_frames must be >= 1")
            if max_fade_packets < 1:
                raise ValueError("max_fade_packets must be >= 1")
        self.playout_delay, self.fade_frames, self.max_fade_packets = playout_delay, fade_frames, max_fade_packets
        self.max_playout_delay, self.jitter_window = max_playout_delay, jitter_window
        self.rx_encoder, self.decoder = rx_encoder, decoder
        self.frames_per_packet, self.sample_rate = frames_per_packet, sample_rate
        self.conceal_packets = conceal_packets
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.codebook_num, self.frame_bytes = rx_encoder.codebook_num, rx_encoder.packed_frame_bytes()
        super().__init__(capacity, (decoder,))
        self._held: List[Dict[int, Packet]] = [{} for _ in range(capacity)]
        self._next = [0] * capacity
        self._out: List[Deque[np.ndarray]] = [collections.deque() for _ in range(capacity)]
        self.stats = [ReceiveStats() for _ in range(capacity)]
        self.unknown_session_packets = 0
        self.step_times: List[float] = []
        # a decoder with bf16 activations takes bf16 zq: the lookup rounds its fp32 sum once, as the decoder's own cast would
        self._zq_kw = {"dtype": torch.bfloat16} if getattr(decoder, "_act_bf16", False) else {}
        # an adaptive step stages up to P + 2 frames of a session: its window, the packet a concealment leads to, the anchor's frame
        staged = frames_per_packet + (2 if max_playout_delay is not None else 0)
        self._p_host = _pinned(capacity * staged * self.frame_bytes, torch.uint8, self.device)
        self._p_np = self._p_host.numpy()
        self._y_host = None                            # the PCM of a step, sized on the first step
        # concealment: per slot the fp32 lookup sum of the last real frame decoded, whether there is one, and the pending plan
        # [packets left, frames per packet, frames concealed so far, frames in the gap]
        self._anchors = torch.zeros(capacity, rx_encoder.code_dim, dtype=torch.float32, device=self.device) \
            if conceal_packets or playout_delay is not None else None
        self._has_anchor = [False] * capacity
        self._plan: List[Optional[list]] = [None] * capacity
        # playout: steps completed; per slot the arrival stamp of each held packet, whether it plays, the frames concealed or faded
        # since its last real frame, its consecutive fade packets, its last real packet's frame count and the sequence numbers the
        # clock gave up (a later arrival of one is late)
        self._steps = 0
        self._stamp: List[Dict[int, int]] = [{} for _ in range(capacity)]
        self._playing = [False] * capacity
        self._c = [0] * capacity
        self._fades = [0] * capacity
        self._last_frames: List[Optional[int]] = [None] * capacity
        self._given_up: List[set] = [set() for _ in range(capacity)]
        # adaptive playout: per slot the content frames not yet played ((0, packet, frame index, 0) real, (1, packet m, j, den)
        # interpolated toward m's first frame, (2, None, j, den) fade), the (packet, frame index) the anchor was taken from, and the
        # lateness of the talk spurt's last jitter_window packets
        self._queue: List[list] = [[] for _ in range(capacity)]
        self._anchor_frame: List[Optional[tuple]] = [None] * capacity
        self._lat: List[Deque[int]] = [collections.deque(maxlen=jitter_window) for _ in range(capacity)]
        if playout_delay is not None:
            sf = rx_encoder.silence_frame() if silence_frame is None else silence_frame
            sf = torch.as_tensor(sf, dtype=torch.float32).to(self.device)
            if sf.numel() != rx_encoder.code_dim:
                raise ValueError(f"silence_frame has {sf.numel()} values, the codec's frames have {rx_encoder.code_dim}")
            self._targets = sf.reshape(1, -1).contiguous()
            # the descriptors of a step go through two page-locked (R_max, 6) tables used in turn
            r_max = capacity * frames_per_packet
            self._rows_host = [_pinned(r_max * 6, torch.int32, self.device).view(r_max, 6) for _ in range(2)]
            self._rows_np = [t.numpy() for t in self._rows_host]
            self._rows_turn = 0

    def _reset_slot(self, s):
        self._held[s].clear()
        self._next[s] = 0
        self._out[s].clear()
        self.stats[s] = ReceiveStats()
        self._has_anchor[s] = False
        self._plan[s] = None
        self._stamp[s].clear()
        self._playing[s] = False
        self._c[s] = self._fades[s] = 0
        self._last_frames[s] = None
        self._given_up[s] = set()
        self._queue[s] = []
        self._anchor_frame[s] = None
        self._lat[s].clear()

    def _export_slot(self, s):
        if self.playout_delay is not None:
            po = {"playing": self._playing[s], "waited": [self._steps - self._stamp[s][q] for q in sorted(self._held[s])],
                  "c": self._c[s], "fades": self._fades[s], "last_frames": self._last_frames[s], "given_up": sorted(self._given_up[s])}
            if self.max_playout_delay is not None:
                po.update(queue=list(self._queue[s]), anchor_frame=self._anchor_frame[s],
                          lateness=[v - self._steps for v in self._lat[s]])
            return {"anchor": self._anchors[s].clone() if self._has_anchor[s] else None, "playout": po}
        if not self.conceal_packets:
            return {}
        plan = self._plan[s]
        return {"anchor": self._anchors[s].clone() if self._has_anchor[s] else None, "conceal": None if plan is None else tuple(plan)}

    def _take_slot(self, s):
        inputs, outputs, seq = [self._held[s][q] for q in sorted(self._held[s])], list(self._out[s]), self._next[s]
        self._reset_slot(s)
        return inputs, outputs, seq

    def _restore_slot(self, s, state):
        self._reset_slot(s)
        self._held[s].update((p.seq, p) for p in state.inputs)
        self._next[s] = state.seq
        self._out[s].extend(state.outputs)
        if self.playout_delay is not None:
            po = state.playout
            self._stamp[s].update((p.seq, self._steps - w) for p, w in zip(state.inputs, po["waited"]))
            self._playing[s], self._c[s], self._fades[s] = po["playing"], po["c"], po["fades"]
            self._last_frames[s], self._given_up[s] = po["last_frames"], set(po["given_up"])
            if self.max_playout_delay is not None:
                self._queue[s], self._anchor_frame[s] = list(po["queue"]), po["anchor_frame"]
                self._lat[s].extend(v + self._steps for v in po["lateness"])
        if self.conceal_packets or self.playout_delay is not None:
            if state.anchor is not None:
                self._anchors[s].copy_(state.anchor)
                self._has_anchor[s] = True
            if state.conceal is not None:
                self._plan[s] = list(state.conceal)

    # ------------------------------------------------------------------ sessions
    def open(self, session_id: int) -> int:
        """Bind remote session `session_id` to a warm slot; its first packet is sequence number 0.  ValueError if it is open
        already, RuntimeError when every slot is taken."""
        return self._open_slot(session_id)

    def close(self, session_id: int) -> None:
        """End the session: its slot becomes free, its held packets and undelivered frames are dropped."""
        self._close_slot(session_id)

    def detach(self, session_id: int) -> SessionState:
        """Close the session and return its decoder state, held packets, undelivered frames and the next sequence number it expects
        (waits for a step in progress)."""
        state = self._detach_slot(session_id)
        state.session_id = session_id
        return state

    def attach(self, state: SessionState) -> int:
        """Continue a session detached from a receiver server of the same config and dtype, under its own id, with fresh counters.
        The state must be on this server's device (SessionState.to)."""
        if state.session_id is None:
            raise ValueError("the session has no wire session id: it was not detached from a receiver server")
        if (state.playout is None) != (self.playout_delay is None):
            raise ValueError("a session moves between two receivers with a playout clock or two without: this one "
                             + ("has one" if self.playout_delay is not None else "has none") + ", the session's had "
                             + ("none" if state.playout is None else "one"))
        if state.playout is not None and ("queue" in state.playout) != (self.max_playout_delay is not None):
            raise ValueError("a session moves between two receivers with an adaptive playout delay or two with a fixed one: this one's is "
                             + ("adaptive" if self.max_playout_delay is not None else "fixed") + ", the session's was "
                             + ("adaptive" if "queue" in state.playout else "fixed"))
        return self._attach_slot(state, state.session_id)

    @property
    def open_sessions(self) -> List[int]:
        with self._lock:
            return sorted(self._ids)

    def _give_up_gap(self, s) -> None:
        """More than reorder_window packets held behind a missing one: count the missing ones lost and move on to the first held.  With
        concealment, plan the last conceal_packets of them as concealed packets of the first held packet's frame count."""
        held = self._held[s]
        if len(held) > self.reorder_window and self._next[s] not in held:
            first = min(held)
            gap = first - self._next[s]
            self.stats[s].losses += gap
            self._next[s] = first
            if self.conceal_packets:
                n, f = min(gap, self.conceal_packets), held[first].frames
                self._plan[s] = [n, f, 0, n * f]

    def submit_packet(self, buf) -> bool:
        """Take one packet.  Returns True if it was queued for decoding, False if it was counted and dropped (session not open,
        duplicate).  Raises ValueError for a malformed packet, one made for another codec, or one of more than frames_per_packet
        frames."""
        p = decode_packet(buf, self.codebook_num, self.frame_bytes)
        if p.frames > self.frames_per_packet:
            raise ValueError(f"frames: packet has {p.frames}, this receiver takes at most {self.frames_per_packet}")
        if self.max_playout_delay is not None and p.frames != self.frames_per_packet:
            raise ValueError(f"frames: packet has {p.frames}, an adaptive playout delay needs exactly {self.frames_per_packet}")
        with self._lock:
            s = self._ids.get(p.session_id)
            if s is None or s not in self._open:
                self.unknown_session_packets += 1
                return False
            held, st = self._held[s], self.stats[s]
            if self.playout_delay is not None and p.seq in self._given_up[s]:
                st.late += 1
                if self.max_playout_delay is not None:
                    self._lat[s].append(self._steps - p.seq)
                return False
            if p.seq < self._next[s] or p.seq in held:
                st.duplicates += 1
                return False
            if any(q > p.seq for q in held):
                st.reorders += 1
            held[p.seq] = p
            if self.playout_delay is not None:
                self._stamp[s][p.seq] = self._steps
                if self.max_playout_delay is not None:
                    self._lat[s].append(self._steps - p.seq)
            else:
                self._give_up_gap(s)
            return True

    def poll(self, session_id: int) -> Optional[np.ndarray]:
        """The session's next decoded frame (float32, frames x hop samples), or None."""
        with self._lock:
            q = self._out[self._slot(session_id)]
            return q.popleft() if q else None

    # ------------------------------------------------------------------ one step
    def step(self) -> int:
        """Decode the next in-order packet of every open session that has one, or its next concealed packet.  Returns the number of
        packets decoded, concealed ones included."""
        with self._step_lock:
            if self.max_playout_delay is not None:
                return self._adaptive_step()
            if self.playout_delay is not None:
                return self._playout_step()
            return self._step()

    def _step(self) -> int:
        t0 = time.time()
        # (slot, open counter, packet, concealment): a real packet with None, or a concealed one with (first j, M + 1, anchor slot or
        # -1) and the packet after the gap, still held, as its packet
        taken: List[Tuple[int, int, Packet, Optional[Tuple[int, int, int]]]] = []
        with self._lock:
            for sid, s in sorted(self._ids.items()):
                if s not in self._open:
                    continue
                self._give_up_gap(s)
                plan = self._plan[s]
                if plan is not None:
                    taken.append((s, self._session[s], self._held[s][self._next[s]],
                                  (plan[2] + 1, plan[3] + 1, s if self._has_anchor[s] else -1)))
                    plan[0] -= 1
                    plan[2] += plan[1]
                    if plan[0] == 0:
                        self._plan[s] = None
                    continue
                p = self._held[s].pop(self._next[s], None)
                if p is not None:
                    self._next[s] += 1
                    taken.append((s, self._session[s], p, None))
                    self._has_anchor[s] = True
        if not taken:
            self.step_times.append(time.time() - t0)
            return 0
        nb = self.frame_bytes
        frames = [p.frames for _, _, p, _ in taken]
        total = sum(frames)
        o = 0
        staged = []                                    # per taken packet: its first frame in the staged bytes
        for _, _, p, c in taken:
            n = nb if c is not None else len(p.payload)   # a concealed packet stages only the first frame after the gap
            self._p_np[o:o + n] = np.frombuffer(p.payload, dtype=np.uint8, count=n)
            staged.append(o // nb)
            o += n
        with torch.no_grad(), self._codec_lock:
            if self.conceal_packets:
                packed = self._p_host[:o].to(self.device, non_blocking=True).view(o // nb, nb)
                zq = self.rx_encoder.lookup_packed_conceal(packed, self._conceal_rows(taken, frames, staged), self._anchors,
                                                           **self._zq_kw)
            else:
                packed = self._p_host[:total * nb].to(self.device, non_blocking=True).view(1, total, nb)
                zq = self.rx_encoder.lookup_packed(packed, **self._zq_kw)
            ys = self.decoder.decode_streams(zq, frames, [s for s, _, _, _ in taken])
            y = torch.cat([v.reshape(-1) for v in ys])
            hop = y.numel() // total
            if self._y_host is None or self._y_host.dtype != y.dtype or self._y_host.numel() < y.numel():
                self._y_host = _pinned(max(y.numel(), self.capacity * self.frames_per_packet * hop), y.dtype, self.device)
            y_host = self._y_host[:y.numel()]
            y_host.copy_(y, non_blocking=True)
            if y.device.type == "cuda":
                torch.cuda.current_stream(y.device).synchronize()
        # one copy out of the staging buffer (widened from bf16 with bf16 activations); the queues hold views of it
        y_np = (y_host.float() if y_host.dtype == torch.bfloat16 else y_host.clone()).numpy()
        with self._lock:
            o = 0
            for (s, session, p, c), f in zip(taken, frames):
                chunk = y_np[o * hop:(o + f) * hop]
                o += f
                if s not in self._open or self._session[s] != session:
                    continue                        # closed while the step ran: the frame is dropped
                self._out[s].append(chunk)
                st = self.stats[s]
                if c is not None:
                    st.concealed += 1
                    st.concealed_frames += f
                    continue
                st.packets += 1
                st.frames += f
                st.bytes += HEADER_BYTES + len(p.payload)
                st.samples += chunk.size
        self.step_times.append(time.time() - t0)
        return len(taken)

    @staticmethod
    def _conceal_rows(taken, frames, staged) -> np.ndarray:
        """The (R, 5) adec_conceal_row descriptors (src, next, slot, j, den) of a step, one per zq row.  A real packet's rows read its
        staged frames, and its last row stores the session's anchor.  A concealed packet's rows read the one staged frame after the gap
        and the session's anchor (or none), with j counted on from where the gap's previous packets stopped."""
        f = np.asarray(frames, dtype=np.int64)
        if not any(t[3] for t in taken):                 # no concealment this step: row r reads staged frame r
            rows = np.zeros((int(f.sum()), 5), dtype=np.int32)
            rows[:, 0] = np.arange(rows.shape[0])
            rows[:, 1:3] = -1
            rows[np.cumsum(f) - 1, 2] = [t[0] for t in taken]
            return rows
        real = np.array([c is None for *_, c in taken])
        first_j = np.array([0 if c is None else c[0] for *_, c in taken], dtype=np.int64)
        den = np.array([0 if c is None else c[1] for *_, c in taken], dtype=np.int64)
        slot = np.array([s if c is None else c[2] for s, *_, c in taken], dtype=np.int64)
        k = np.arange(int(f.sum())) - np.repeat(np.cumsum(f) - f, f)          # row within its packet
        real_r, base = np.repeat(real, f), np.repeat(np.asarray(staged, dtype=np.int64), f)
        rows = np.empty((k.size, 5), dtype=np.int32)
        rows[:, 0] = np.where(real_r, base + k, -1)
        rows[:, 1] = np.where(real_r, -1, base)
        rows[:, 2] = np.where(real_r & (k != np.repeat(f - 1, f)), -1, np.repeat(slot, f))
        rows[:, 3] = np.where(real_r, 0, np.repeat(first_j, f) + k)
        rows[:, 4] = np.repeat(den, f)
        return rows

    def _playout_plan(self, s) -> Optional[tuple]:
        """What playing slot s plays this step, with _lock held: (kind, packet or None, frames, j of the first row, den); kind 0 is a
        real packet, 1 an interpolated packet toward held packet m (the packet), 2 a fade packet.  Updates the slot's position and
        counters, pauses it after max_fade_packets fades."""
        held, st, nxt, c = self._held[s], self.stats[s], self._next[s], self._c[s]
        p = held.pop(nxt, None)
        self._next[s] = nxt + 1
        if p is not None:                                              # rule 1
            del self._stamp[s][nxt]
            self._c[s] = self._fades[s] = 0
            self._last_frames[s] = p.frames
            return 0, p, p.frames, 0, 0
        self._given_up[s].add(nxt)
        if held:                                                       # rule 2
            m = min(held)
            f = held[m].frames
            st.losses += 1
            st.concealed += 1
            st.concealed_frames += f
            self._c[s] = c + f
            self._fades[s] = 0
            return 1, held[m], f, c + 1, c + (m - nxt) * f + 1
        f = self._last_frames[s] or self.frames_per_packet             # rule 3
        st.underruns += 1
        st.faded_frames += f
        self._c[s] = c + f
        self._fades[s] += 1
        if self._fades[s] == self.max_fade_packets:                    # pause: back to buffering, rewound past the fades
            st.pauses += 1
            self._playing[s] = False
            self._next[s] -= self.max_fade_packets
            self._given_up[s].difference_update(range(self._next[s], self._next[s] + self.max_fade_packets))
            self._fades[s] = 0
        return 2, None, f, c + 1, self.fade_frames

    def _playout_step(self) -> int:
        """One packet period of the playout clock: one packet of PCM for every playing session."""
        t0 = time.time()
        now, delay = self._steps, self.playout_delay
        taken = []                                     # (slot, open counter, kind, packet, frames, first j, den, anchor slot or -1)
        with self._lock:
            for sid, s in sorted(self._ids.items()):
                if s not in self._open:
                    continue
                if not self._playing[s]:
                    if not any(now - t >= delay for t in self._stamp[s].values()):
                        continue
                    self._playing[s] = True
                kind, p, f, j, den = self._playout_plan(s)
                taken.append((s, self._session[s], kind, p, f, j, den, s if self._has_anchor[s] or kind == 0 else -1))
                if kind == 0:
                    self._has_anchor[s] = True
            self._steps += 1
        if not taken:
            self.step_times.append(time.time() - t0)
            return 0
        nb = self.frame_bytes
        o = 0
        staged = []                                    # per taken packet: its first frame in the staged bytes
        for _, _, kind, p, *_ in taken:
            staged.append(o // nb)
            if kind == 2:
                continue
            n = len(p.payload) if kind == 0 else nb    # an interpolated packet stages only m's first frame
            self._p_np[o:o + n] = np.frombuffer(p.payload, dtype=np.uint8, count=n)
            o += n
        frames = [t[4] for t in taken]
        rows = self._playout_rows(taken, staged)
        with torch.no_grad(), self._codec_lock:
            packed = self._p_host[:o].to(self.device, non_blocking=True).view(o // nb, nb)
            zq = self.rx_encoder.lookup_packed_playout(packed, rows, self._anchors, self._targets, **self._zq_kw)
            y_np, hop = self._decode_to_host(zq, frames, [t[0] for t in taken])
        with self._lock:
            o = 0
            for (s, session, kind, p, f, *_) in taken:
                chunk = y_np[o * hop:(o + f) * hop]
                o += f
                if s not in self._open or self._session[s] != session:
                    continue                        # closed while the step ran: the frame is dropped
                self._out[s].append(chunk)
                if kind == 0:
                    st = self.stats[s]
                    st.packets += 1
                    st.frames += f
                    st.bytes += HEADER_BYTES + len(p.payload)
                    st.samples += chunk.size
        self.step_times.append(time.time() - t0)
        return len(taken)

    def _decode_to_host(self, zq, frames, slots):
        """ONE decode_streams of the step's zq, and its PCM back in ONE copy -> (float32 samples, hop)"""
        ys = self.decoder.decode_streams(zq, frames, slots)
        y = torch.cat([v.reshape(-1) for v in ys])
        hop = y.numel() // sum(frames)
        if self._y_host is None or self._y_host.dtype != y.dtype or self._y_host.numel() < y.numel():
            self._y_host = _pinned(max(y.numel(), self.capacity * self.frames_per_packet * hop), y.dtype, self.device)
        y_host = self._y_host[:y.numel()]
        y_host.copy_(y, non_blocking=True)
        if y.device.type == "cuda":
            torch.cuda.current_stream(y.device).synchronize()
        return (y_host.float() if y_host.dtype == torch.bfloat16 else y_host.clone()).numpy(), hop

    def _target(self, s) -> int:
        """the adaptive clock's target delay of slot s in packets: the window's lateness spread, within [D, D_max]"""
        lat = self._lat[s]
        j = max(lat) - min(lat) if len(lat) >= 2 else 0
        return min(max(j, self.playout_delay), self.max_playout_delay)

    def _adaptive_window(self, s, k) -> list:
        """The content frames playing slot s plays at step k (steps completed), with _lock held: decides C from the delay, fills the
        queue by rules 1 - 3 (_playout_plan) one packet at a time, and takes C frames off it."""
        P, q, st = self.frames_per_packet, self._queue[s], self.stats[s]
        lam = (self._target(s) + 1) * P
        nxt = self._next[s]
        seq, o = (nxt - 1, P - len(q)) if q else (nxt, 0)
        delta = (k - min(self._lat[s]) + 1) * P - (seq * P + o)
        st.delay_frames = delta
        avail = 0                                                      # L: real frames in a row from the playout point
        if not q or q[0][0] == 0:
            avail, held = len(q), self._held[s]
            while avail < P + 1 and nxt in held:
                avail += P
                nxt += 1
        c = P
        if delta > lam and avail >= P + 1:
            c = P + 1
            st.compressed += 1
        elif delta < lam and avail >= P - 1:
            c = P - 1
            st.expanded += 1
        while len(q) < c:
            kind, p, f, j, den = self._playout_plan(s)
            if kind == 0:
                q.extend((0, p, i, 0) for i in range(f))
                st.packets += 1
                st.frames += f
                st.bytes += HEADER_BYTES + len(p.payload)
            else:
                q.extend((kind, p, j + i, den) for i in range(f))
        win = q[:c]
        del q[:c]
        if not self._playing[s]:                                       # paused by a fade packet: what it did not play is dropped
            q.clear()
            self._lat[s].clear()
        return win

    def _window_rows(self, s, win, stage, rows) -> None:
        """Append slot s's P adec_playout_row descriptors for the content frames `win` to `rows`; stage(packet, i) stages frame i of a
        packet (once per step) and returns its index.  The last real frame of the window stores the anchor; a concealed or fade frame
        in a window with a real frame starts from a staged frame (the last real one before it, or the frame the old anchor came from),
        since a launch may not both write and read one anchor."""
        P, C = self.frames_per_packet, len(win)
        if C != P:                                                     # a scaled run of real frames
            for i in range(P):
                m, r = divmod(i * (C - 1), P - 1)
                a = win[m]
                if r == 0:
                    rows.append((stage(a[1], a[2]), -1, -1, s if m == C - 1 else -1, 0, 0))
                else:
                    b = win[m + 1]
                    rows.append((stage(a[1], a[2]), stage(b[1], b[2]), -1, -1, r, P - 1))
            return
        last = -1
        for i, e in enumerate(win):
            if e[0] == 0:
                last = i
        for i, (kind, p, j, den) in enumerate(win):
            if kind == 0:
                rows.append((stage(p, j), -1, -1, s if i == last else -1, 0, 0))
                continue
            src = (win[last][1], win[last][2]) if i > last >= 0 else self._anchor_frame[s] if last >= 0 else None
            src = -1 if src is None else stage(*src)
            slot = s if last < 0 and self._has_anchor[s] else -1
            if kind == 1:
                rows.append((src, stage(p, 0), -1, -1 if src >= 0 else slot, j, den))
            else:
                rows.append((src, -1, 0, -1 if src >= 0 else slot, j, den))

    def _adaptive_step(self) -> int:
        """One packet period of the adaptive playout clock: P output frames for every playing session."""
        t0 = time.time()
        now, P = self._steps, self.frames_per_packet
        taken, rows, chunks = [], [], []               # taken: (slot, open counter, real content frames played)
        nst = [0]                                      # frames staged so far
        nb = self.frame_bytes
        with self._lock:
            for sid, s in sorted(self._ids.items()):
                if s not in self._open:
                    continue
                if not self._playing[s]:
                    target = self._target(s)
                    if not any(now - t >= target for t in self._stamp[s].values()):
                        continue
                    self._playing[s] = True
                win = self._adaptive_window(s, now)
                p = win[0][1]
                if len(win) == P and win[0][0] == 0 and win[0][2] == 0 and win[-1][1] is p:
                    # one whole real packet, the common step: its payload staged in one piece, the fixed clock's rows
                    base = nst[0]
                    chunks.append(p.payload)
                    nst[0] += P
                    rows.extend([(base + i, -1, -1, -1, 0, 0) for i in range(P - 1)])
                    rows.append((base + P - 1, -1, -1, s, 0, 0))
                    self._anchor_frame[s] = (p, P - 1)
                    self._has_anchor[s] = True
                    taken.append((s, self._session[s], P))
                    continue
                staged = {}

                def stage(p, i):
                    key = (id(p), i)
                    if key not in staged:
                        staged[key] = nst[0]
                        chunks.append(p.payload[i * nb:(i + 1) * nb])
                        nst[0] += 1
                    return staged[key]

                self._window_rows(s, win, stage, rows)
                real = [e for e in win if e[0] == 0]
                if real:
                    self._anchor_frame[s] = (real[-1][1], real[-1][2])
                    self._has_anchor[s] = True
                taken.append((s, self._session[s], len(real)))
            self._steps += 1
        if not taken:
            self.step_times.append(time.time() - t0)
            return 0
        o = nst[0] * nb
        self._p_np[:o] = np.frombuffer(b"".join(chunks), dtype=np.uint8)
        table = self._rows_np[self._rows_turn]
        self._rows_turn ^= 1
        table[:len(rows)] = rows
        with torch.no_grad(), self._codec_lock:
            packed = self._p_host[:o].to(self.device, non_blocking=True).view(o // nb, nb)
            zq = self.rx_encoder.lookup_packed_timescale(packed, table[:len(rows)], self._anchors, self._targets, **self._zq_kw)
            y_np, hop = self._decode_to_host(zq, [P] * len(taken), [t[0] for t in taken])
        with self._lock:
            for i, (s, session, real) in enumerate(taken):
                if s not in self._open or self._session[s] != session:
                    continue                        # closed while the step ran: the frame is dropped
                chunk = y_np[i * P * hop:(i + 1) * P * hop]
                self._out[s].append(chunk)
                self.stats[s].samples += real * hop
        self.step_times.append(time.time() - t0)
        return len(taken)

    def _playout_rows(self, taken, staged) -> np.ndarray:
        """The (R, 6) adec_playout_row descriptors (src, next, target, slot, j, den) of a playout step, written into the next of the
        two page-locked tables.  A real packet's rows read its staged frames and its last row stores the session's anchor; an
        interpolated packet's rows read the one staged frame of m; a fade packet's rows read the silence frame (target 0).  The
        step synchronises on its output before the table comes round again."""
        table = self._rows_np[self._rows_turn]
        self._rows_turn ^= 1
        f = np.fromiter((t[4] for t in taken), dtype=np.int64, count=len(taken))
        ends = np.cumsum(f)
        rows = table[:int(ends[-1])]
        if not any(t[2] for t in taken):               # every packet real: row r reads staged frame r
            rows[:, 0] = np.arange(rows.shape[0])
            rows[:, 1:4] = -1
            rows[ends - 1, 3] = [t[0] for t in taken]
            rows[:, 4:] = 0
            return rows
        kind = np.repeat(np.fromiter((t[2] for t in taken), dtype=np.int64, count=len(taken)), f)
        k = np.arange(rows.shape[0]) - np.repeat(ends - f, f)                 # row within its packet
        base = np.repeat(np.asarray(staged, dtype=np.int64), f)
        real = kind == 0
        rows[:, 0] = np.where(real, base + k, -1)
        rows[:, 1] = np.where(kind == 1, base, -1)
        rows[:, 2] = np.where(kind == 2, 0, -1)
        rows[:, 3] = np.where(real & (k != np.repeat(f - 1, f)), -1, np.repeat([t[7] for t in taken], f))
        rows[:, 4] = np.where(real, 0, np.repeat([t[5] for t in taken], f) + k)
        rows[:, 5] = np.where(real, 0, np.repeat([t[6] for t in taken], f))
        return rows

    def statistics(self) -> Dict:
        """steps, ms per step (mean, std), the open sessions, packets for sessions that were not open, and per open session: packets,
        frames, duplicates, reorders, losses, concealed packets and frames, and the wire kbps received (real packet bytes, headers
        included, over the seconds of real audio decoded).  With a playout clock also late, underruns, faded_frames, pauses and
        buffered (the packets held ahead of the playout point).  With an adaptive delay also target_delay (packets), delay_frames (the
        delay at the session's last played step, in code frames) and the compressed and expanded step counts."""
        with self._lock:
            po, ad = self.playout_delay is not None, self.max_playout_delay is not None
            per = {sid: self.stats[s].as_dict(self.sample_rate, len(self._held[s]) if po else None, self._target(s) if ad else None)
                   for sid, s in sorted(self._ids.items())}
        return {"capacity": self.capacity, "open_sessions": len(per), "steps": len(self.step_times), "step_ms": _ms(self.step_times),
                "unknown_session_packets": self.unknown_session_packets, "per_session": per}
