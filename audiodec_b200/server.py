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
        f = np.asarray(frame, dtype=np.float32).reshape(-1)
        if f.shape[0] != self.frame_size:
            raise ValueError(f"frame has {f.shape[0]} samples, server frame_size is {self.frame_size}")
        with self._lock:
            q = self._in[stream]
            q.append((f, self._clock() if t_capture is None else t_capture))
            while len(q) > self.max_backlog:
                q.popleft()
                self.stats[stream].frame_drops += 1

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
    """What a detached session needs to continue on another SessionCodecServer (of the same config and dtypes, on any device):
    per stateful generator of the server its state_layout and its (1, S) device state, the queued input frames with their capture
    stamps, and the decoded frames it has not polled yet."""

    def __init__(self, layouts, states, inputs, outputs):
        self.layouts: List[list] = layouts
        self.states: List[torch.Tensor] = states
        self.inputs: List[Tuple[np.ndarray, float]] = inputs
        self.outputs: List[np.ndarray] = outputs

    def to(self, device) -> "SessionState":
        """A copy with the states on `device` (the frames are host arrays and are shared)."""
        return SessionState(self.layouts, [t.to(device) for t in self.states], list(self.inputs), list(self.outputs))


class SessionCodecServer(MultiStreamCodecServer):
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
        super().__init__(tx_encoder, rx_encoder, decoder, capacity, frame_size=frame_size, sample_rate=sample_rate,
                         max_latency=max_latency, device=device, wire=wire, clock=clock)
        self.capacity = capacity
        self.template = capacity                      # slot index of the warm template
        self._stateful = [g for i, g in enumerate((tx_encoder, decoder)) if g not in (tx_encoder, decoder)[:i]]
        for g in self._stateful:
            if g.n_streams != 1:                      # growing from more than one stream adds zero-history slots: a cold template
                raise ValueError(f"{type(g).__name__} holds {g.n_streams} streams; SessionCodecServer needs generators with the one "
                                 "warmed stream that load_transmitter / load_receiver leave")
        for g in self._stateful:
            g.set_streams(capacity + 1)               # replicates the one warmed stream into every slot
        self._free = list(range(capacity))
        self._open: set = set()
        self._session = [0] * capacity                # per slot: bumped by every open(), so a step hands out only its own session's frames
        self._codec_lock = threading.Lock()           # the codec handles are driven by step() and open() from different threads
        self._step_lock = threading.Lock()            # held for a whole step, output hand-off included: detach() waits for it

    # ------------------------------------------------------------------ sessions
    def open(self) -> int:
        """Start a stream in a free slot, warm as the template; returns its id.  Raises RuntimeError when every slot is taken."""
        with self._lock:
            if not self._free:
                raise RuntimeError(f"server is full: all {self.capacity} streams are open")
            s = min(self._free)
            self._free.remove(s)
            self._session[s] += 1
            self._in[s].clear()
            self._out[s].clear()
        with self._codec_lock:
            for g in self._stateful:
                g.copy_stream_state(self.template, [s])
        with self._lock:
            self._open.add(s)
        return s

    def close(self, stream: int) -> None:
        """End stream `stream`: its slot becomes free and its queued input and output are dropped."""
        with self._lock:
            if stream not in self._open:
                raise KeyError(f"stream {stream} is not open")
            self._open.remove(stream)
            self._in[stream].clear()
            self._out[stream].clear()
            self._free.append(stream)

    def detach(self, stream: int) -> SessionState:
        """Close stream `stream` and return what it needs to continue elsewhere (attach(), on this or another server): its causal state
        in every stateful generator, its queued input frames and its undelivered output frames.  Waits for a step in progress to finish
        and hand off its frames, so no frame in flight is lost.  Raises KeyError if the stream is not open."""
        with self._step_lock:
            with self._lock:
                if stream not in self._open:
                    raise KeyError(f"stream {stream} is not open")
                self._open.remove(stream)
                inputs, outputs = list(self._in[stream]), list(self._out[stream])
                self._in[stream].clear()
                self._out[stream].clear()
            with self._codec_lock:       # the slot stays taken until its state is out
                states = [g.stream_state([stream]) for g in self._stateful]
            layouts = [list(g.state_layout) for g in self._stateful]
            with self._lock:
                self._free.append(stream)
        return SessionState(layouts, states, inputs, outputs)

    def attach(self, state: SessionState) -> int:
        """Open a stream in a free slot from a detached session instead of the template: it continues exactly where it left off, with
        its queued and undelivered frames, and fresh per-stream counters.  The state must be on this server's device (SessionState.to).
        Raises ValueError if the session comes from codecs of another layout, RuntimeError when every slot is taken."""
        if len(state.states) != len(self._stateful) or len(state.layouts) != len(self._stateful):
            raise ValueError(f"the session holds the state of {len(state.states)} generators; this server has {len(self._stateful)}")
        for g, layout in zip(self._stateful, state.layouts):
            if [tuple(e) for e in layout] != [tuple(e) for e in g.state_layout]:
                raise ValueError(f"the session's state layout does not match this server's {type(g).__name__}")
        with self._lock:
            if not self._free:
                raise RuntimeError(f"server is full: all {self.capacity} streams are open")
            s = min(self._free)
            self._free.remove(s)
            self._session[s] += 1
        try:
            with self._codec_lock:
                for g, layout, t in zip(self._stateful, state.layouts, state.states):
                    g.load_stream_state([s], t, layout)
        except Exception:
            with self._lock:
                self._free.append(s)
            raise
        with self._lock:
            self._in[s].clear()
            self._in[s].extend(state.inputs)
            self._out[s].clear()
            self._out[s].extend(state.outputs)
            self.stats[s] = StreamStats()
            self._open.add(s)
        return s

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
