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
import threading
import time
from typing import Deque, Dict, List, Optional, Tuple

import numpy as np
import torch


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
        with torch.no_grad():
            x = x_host.to(dev, non_blocking=True)
            z = self.tx_encoder.encode(x)                                       # utils/audiodec.py:100-102
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
            y = self.decoder.decode(zq).detach()                                # utils/audiodec.py:104-106
            if y.device.type == "cuda":
                # device -> PINNED host buffer (a pageable destination is staged through a driver bounce buffer), then one synchronise
                if self._y_host is None or self._y_host.shape != y.shape:
                    self._y_host = torch.empty(y.shape, dtype=y.dtype, pin_memory=True)
                self._y_host.copy_(y, non_blocking=True)
                torch.cuda.current_stream(y.device).synchronize()
                y_host = self._y_host
            else:
                y_host = y
        now = self._clock()
        if y_host.dtype == torch.bfloat16:
            y_host = y_host.float()             # a bf16-activation decoder: half the D2H bytes, widened here; frames out stay float32
        y_all = y_host.numpy().reshape(self.n_streams, -1)[:, :self.frame_size].copy()    # one copy; the queues hold row views of it
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
