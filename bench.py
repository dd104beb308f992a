#!/usr/bin/env python3
"""bench.py - 48 kHz samples/s through encode -> quantize -> lookup -> decode (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--workload symad|v1|v1_bf16|stream_v1]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W

One "step" = one pass of the hot path over one batch of synthetic utterances (BASELINE configs[1]:
symAD_vctk_48000_hop300, 64 x 48000 samples, fp32, per GPU).  Utterances are independent, so N GPUs
each run their own 64-utterance shard with no data-path collective (weak scaling, SURVEY.md 8(e));
NCCL is used only for the timing barrier and the max-over-ranks of the device time.

`value`      : whole-job samples/s, inputs resident in HBM, CUDA events on the launching stream.
`e2e`        : same metric through the reference-facing call with HOST buffers (adec_codec_host: H2D of the
               waveforms + the four calls + D2H of indices and waveforms inside the timed region).
`roofline`   : `frac` is the WHOLE STEP against the HBM roofline under SURVEY.md 8(d)'s per-conv-layer algorithmic
               byte model (9,323.2 B/sample for symAD fp32) and MEASURED_PEAKS.json's copy bandwidth; `kernel_frac`
               is the same for the dominant launch alone; `compute` is the step against the tensor-core ceiling
               this process measured with the library's own wgmma probe (adec_probe_mma).
`parity`     : after the timed region, utterances of the timed batch against the oracle (the oracle is the checker).
`extra_workloads` (N=1): BASELINE configs[2] (AD v1, fp32 and bf16 vocoder), configs[3] (256 streams x 1500-sample
               chunks @ 24 kHz) and the B=1 per-chunk latency the reference publishes (figs/latency.jpg Table 4).
`cpu_baseline` / `gpu_eager_baseline`: the reference's path (oracle port: the same torch ops in the reference's order) on
               the host cores - one process and all cores - and, informational, as eager PyTorch on this GPU.
`--impl reference`: the reference's own CPU implementation of the path.  The reference is pure Python on
               torch CPU ops and cannot travel to the GPU box, so this leg times the oracle port on all host cores.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SAMPLE_RATE = 48000
T_SAMPLES = 48000
BATCH_PER_GPU = 64
# SURVEY.md 8(d): algorithmic bytes / FLOPs per input sample, fp32 activations, per-conv-layer model
ENC_B, RVQ_B, SYMDEC_B, HIFI_B = 1398192.0, 576.0, 1398192.0, 4183472.0     # per 300-sample frame
ALG_BYTES_PER_SAMPLE = {"symad": (ENC_B + RVQ_B + SYMDEC_B) / 300.0, "v1": (ENC_B + RVQ_B + HIFI_B) / 300.0,
                        "v1_bf16": (ENC_B + RVQ_B + HIFI_B) / 300.0}
ALG_FLOP_PER_SAMPLE = {"symad": 549432.0, "v1": 2265247.0, "v1_bf16": 2265247.0}
ALG_BYTES_PER_SAMPLE["stream_v1"] = ALG_BYTES_PER_SAMPLE["v1"]
ALG_FLOP_PER_SAMPLE["stream_v1"] = ALG_FLOP_PER_SAMPLE["v1"]
FFMA_PEAK_TFLOPS = 132 * 128 * 2 * 1.98e9 / 1e12      # H100 SXM: 132 SMs x 128 FP32 lanes x 2 at 1.98 GHz; not measured, informational
WORKLOAD_NAME = {"symad": "symAD_vctk_48000_hop300", "v1": "AudioDec_v1 (symAD encoder + HiFi-GAN v1 vocoder), fp32",
                 "v1_bf16": "AudioDec_v1 (symAD encoder fp32-grade + HiFi-GAN v1 vocoder with bf16 conv operands)",
                 "stream_v1": "libritts_v1 streaming: 256 streams x 1500-sample chunks @ 24 kHz (one chunk per step)"}
WORKLOAD_CFG = {"symad": 1, "v1": 2, "v1_bf16": 2, "stream_v1": 3}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)", d
    return 3350.0, "fallback (NVIDIA H100 SXM data sheet: 3.35 TB/s HBM3, not measured)", {}


class ClockSampler:
    """SM clock, power and throttle reasons DURING the timed region (measured in-process).  Default source is NVML in a
    thread of this process (the library nvidia-smi itself reads; no subprocess, 20 ms period); ADEC_BENCH_SAMPLER=smi runs the
    recipe's `nvidia-smi -lms 100` loop instead, =off disables sampling."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    # nvmlClocksEventReasons bits (nvml.h)
    REASONS = (("hw_slowdown", 0x8), ("sw_thermal_slowdown", 0x20), ("hw_thermal_slowdown", 0x40), ("sw_power_cap", 0x4))

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None
        self.mode = os.environ.get("ADEC_BENCH_SAMPLER", "nvml")
        self._stop = threading.Event()
        self._thread = None

    def start(self):
        if self.mode == "off":
            return
        if self.mode == "nvml":
            try:
                import pynvml
                import torch
                pynvml.nvmlInit()
                pr = torch.cuda.get_device_properties(self.index)      # CUDA_VISIBLE_DEVICES may renumber: address by PCI bus id
                try:
                    h = pynvml.nvmlDeviceGetHandleByPciBusId(f"{pr.pci_domain_id:08x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0")
                except Exception:
                    vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
                    phys = int(vis.split(",")[self.index]) if vis and all(v.strip().isdigit() for v in vis.split(",")) else self.index
                    h = pynvml.nvmlDeviceGetHandleByIndex(phys)
                self._max = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))

                def loop():
                    while not self._stop.is_set():
                        try:
                            sm = float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
                            pw = pynvml.nvmlDeviceGetPowerUsage(h) / 1e3
                            try:
                                rs = int(pynvml.nvmlDeviceGetCurrentClocksEventReasons(h))
                            except Exception:
                                rs = int(pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h))
                            self.rows.append((time.time(), (sm, pw, rs)))
                        except Exception:
                            pass
                        self._stop.wait(0.02)
                self._thread = threading.Thread(target=loop, daemon=True)
                self._thread.start()
                return
            except Exception:
                self.mode = "smi"          # NVML binding unavailable: fall back to the nvidia-smi loop
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.index), "-lms", "100"], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), [c.strip() for c in line.split(",")]))

    def stop(self, t0, t1):
        if self.mode == "off":
            return {"sampler": "off"}
        if self._thread is not None:
            self._stop.set()
            self._thread.join(timeout=1.0)
            rows = [r for (t, r) in self.rows if t0 <= t <= t1] or [r for (_, r) in self.rows]
            if not rows:
                return None
            reasons = sorted({name for (_, _, rs) in rows for name, bit in self.REASONS if rs & bit})
            return {"sm_mhz": statistics.median(r[0] for r in rows), "sm_max_mhz": self._max, "reasons": reasons,
                    "samples": len(rows), "power_w_max": max(r[1] for r in rows), "sampler": "nvml, 20 ms period, in-process thread"}
        if self.proc is None:
            return None
        time.sleep(0.15)
        self.proc.terminate()
        rows = [r for (t, r) in self.rows if t0 <= t <= t1 + 0.2 and len(r) >= 9] or [r for (_, r) in self.rows if len(r) >= 9]
        if not rows:
            return None
        try:
            sm = [float(r[1]) for r in rows]
            reasons = set()
            for r in rows:
                for name, col in (("hw_slowdown", 5), ("hw_thermal_slowdown", 6), ("sw_thermal_slowdown", 7), ("sw_power_cap", 8)):
                    if r[col].lower().startswith("active"):
                        reasons.add(name)
            return {"sm_mhz": statistics.median(sm), "sm_max_mhz": float(rows[0][2]), "reasons": sorted(reasons),
                    "samples": len(rows), "power_w_max": max(float(r[3]) for r in rows), "sampler": "nvidia-smi -lms 100"}
        except Exception:
            return None


def build_codec(workload, device):
    """tx_encoder / rx_encoder / decoder warmed like AudioDec.load_transmitter / load_receiver (bin/stream.py:56-77)."""
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    sd = S.symad_state_dict(seed=0)
    objs = []
    for _ in range(2):
        g = SymADStreamGenerator(**S.SYMAD_PARAMS)
        g.load_state_dict(sd)
        objs.append(g.eval().to(device))
    if workload in ("v1", "v1_bf16", "stream_v1"):
        d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
        d.load_state_dict(S.hifigan_state_dict(seed=1))
        if workload == "v1_bf16":
            d = d.to(torch.bfloat16)           # what `decoder.to(torch.bfloat16)` asks of the reference
    else:
        d = SymADStreamGenerator(**S.SYMAD_PARAMS)
        d.load_state_dict(sd)
    d = d.eval().to(device)
    tx, rx = objs
    tx.initial_encoder(8192, device)                       # bin/stream.py:61
    d.initial_decoder(rx.initial_encoder(8192, device))    # bin/stream.py:70,76
    torch.cuda.synchronize(device)
    return tx, rx, d


def build_oracle(workload):
    from audiodec_b200 import synthetic as S
    from oracle import audiodec_oracle as O
    sd = S.symad_state_dict(seed=0)
    if workload in ("v1", "v1_bf16", "stream_v1"):
        return O.CodecOracle(S.SYMAD_PARAMS, sd, S.HIFIGAN_V1_PARAMS, S.hifigan_state_dict(seed=1))
    return O.CodecOracle(S.SYMAD_PARAMS, sd)


def workload_shape(workload):
    if workload == "stream_v1":
        return 256, 1500, 24000          # demoStream.py:28 default frame size, 256 concurrent streams, libritts 24 kHz
    if workload == "v1_bf16":
        return 128, T_SAMPLES, SAMPLE_RATE
    return BATCH_PER_GPU, T_SAMPLES, SAMPLE_RATE


def codec_step(tx, rx, dec, x):
    """One pass of the path; returns what its caller receives: waveform, code indices, latent z, quantized latent zq."""
    z = tx.encode(x)
    idx = tx.quantize(z)
    zq = rx.lookup(idx)
    return dec.decode(zq), idx, z, zq


def parity_vs_oracle(workload, dev, x_batch, sel, chunks=1):
    """Fresh, warmed codec vs the oracle on rows `sel` of one timed batch (demoFile.py:58-61 per utterance; `chunks` > 1 cuts the
    input into consecutive chunks like the streamer does).  A differing frame counts as equal only if the reference's own top-2
    margin at the first differing stage is a numerical tie (< 1e-6)."""
    import torch
    from oracle import audiodec_oracle as O
    tx, rx, dec = build_codec(workload, dev)
    orc = build_oracle(workload)
    xs = x_batch.cpu()
    T = xs.shape[-1] // chunks
    ys, idxs, rys, ridxs, rzs = [], [], [], [], []
    for c in range(chunks):
        xc = xs[:, :, c * T:(c + 1) * T].contiguous()
        y, idx = codec_step(tx, rx, dec, xc.to(dev))[:2]
        ys.append(y.cpu()), idxs.append(idx.cpu() if idx.dim() == 3 else idx.cpu().unsqueeze(1))
        with torch.no_grad():
            rz, ridx, _, ry = orc.run(xc[sel])
        rys.append(ry), ridxs.append(ridx if ridx.dim() == 3 else ridx.unsqueeze(1)), rzs.append(rz)
    y, idx, ry, ridx, rz = torch.cat(ys, -1), torch.cat(idxs, -1), torch.cat(rys, -1), torch.cat(ridxs, -1), torch.cat(rzs, -1)
    idx = idx[:, sel]
    bad = idx != ridx
    _, _, margins = O.rvq_forward_index(rz.transpose(1, 2), orc.tx_encoder.embeds, return_margins=True)
    ties = []
    for b, f in zip(*torch.nonzero(bad.any(0), as_tuple=True)):
        ties.append(float(margins[int(torch.nonzero(bad[:, b, f])[0]), b, f]))
    ok = ~bad.any(0)
    hop = y.shape[-1] // idx.shape[-1]
    err = (y[sel] - ry).abs()[:, 0].reshape(len(sel), -1, hop)[ok]
    return {"utterances": len(sel), "rows": [int(s) for s in sel], "frames": int(ok.numel()), "frames_differing": int((~ok).sum()),
            "idx_equal": bool(all(m < 1e-6 for m in ties)), "tie_margins": sorted(ties)[:8],
            "wave_max_abs": float(err.max()) if err.numel() else None,
            "tolerance": {"idx": "equal (ties < 1e-6 of the reference's own margin)", "wave_max_abs": 1e-4},
            "checker": "oracle/audiodec_oracle.py CodecOracle.run on the same rows, fresh warmed state on both sides"}


def probe_compute(dev_index):
    """Measured tensor-core ceilings of the conv engine, by tile shape (adec_probe_mma: MMAs only, engine's smem operand layout)."""
    import ctypes
    from audiodec_b200 import _lib
    lib = _lib.load()
    out = {}
    for name, kind in (("f16", 1), ("tf32", 0)):
        for nt in (256, 128, 64, 32):
            tf, ms = ctypes.c_double(), ctypes.c_double()
            rc = lib.adec_probe_mma(dev_index, kind, nt, 6000 if nt >= 128 else 12000, ctypes.byref(tf), ctypes.byref(ms))
            if rc == 0:
                out[f"{name}_n{nt}_tflops"] = tf.value
    return out


def time_device_loop(step, steps, warmup, dev, barrier):
    import torch
    for i in range(warmup):
        step(i)
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        out = step(i)
    e1.record()
    barrier()
    return e0.elapsed_time(e1), out


def measure_extra(workload, dev, steps, peak):
    """One extra workload in the same process (N=1): device-resident timing, step roofline fraction, per-launch top-3."""
    import torch
    B, T, sr = workload_shape(workload)
    tx, rx, dec = build_codec(workload, dev)
    gen = torch.Generator().manual_seed(4242)
    xs = [(0.1 * torch.randn(B, 1, T, generator=gen)).to(dev) for _ in range(4)]
    sync = lambda: torch.cuda.synchronize(dev)
    l0 = tx.launch_count + rx.launch_count + dec.launch_count
    # median of three back-to-back regions of `steps` steps, like the headline (a single ~100 ms region is a coin flip on a power-capped box)
    runs = []
    for r in range(3):
        ms_r, y = time_device_loop(lambda i: codec_step(tx, rx, dec, xs[i % 4])[0], steps, 3 if r == 0 else 0, dev, sync)
        runs.append(ms_r)
    ms = sorted(runs)[1]
    launches = (tx.launch_count + rx.launch_count + dec.launch_count - l0) // (3 * steps + 3)
    assert torch.isfinite(y).all()
    sps = B * T * steps / (ms / 1e3)
    out = {"workload": WORKLOAD_NAME[workload] + f", batch={B}x{T}", "baseline_config": f"configs[{WORKLOAD_CFG[workload]}]",
           "ms_per_step": ms / steps, "regions_ms_per_step": [round(v / steps, 3) for v in runs], "samples_per_s": sps,
           "realtime_factor": sps / sr, "steps": steps, "launches_per_step": int(launches),
           "roofline_step_frac": ALG_BYTES_PER_SAMPLE[workload] * sps / 1e9 / peak,
           "useful_tflops": ALG_FLOP_PER_SAMPLE[workload] * sps / 1e12}
    dec.profile(True)
    codec_step(tx, rx, dec, xs[0])
    sync()
    rows = dec.profile_report()
    dec.profile(False)
    top = sorted(rows, key=lambda r: -r[1])[:3]
    out["decoder_top3_launches"] = [{"op": n, "ms": m, "GBps_alg": b / m / 1e6} for n, m, b in top]
    del tx, rx, dec
    return out


def measure_stream_server(dev, steps):
    """configs[3] through the multi-stream server: host frames in, host frames out, one batched launch sequence per chunk."""
    import numpy as np
    from audiodec_b200.server import MultiStreamCodecServer
    B, T, sr = workload_shape("stream_v1")
    tx, rx, dec = build_codec("stream_v1", dev)
    srv = MultiStreamCodecServer(tx, rx, dec, n_streams=B, frame_size=T, sample_rate=sr, max_latency=1.0, device=dev)
    rng = np.random.default_rng(7)
    frames = (0.1 * rng.standard_normal((4, B, T))).astype(np.float32)
    for k in range(steps + 3):
        for s in range(B):
            srv.submit(s, frames[k % 4, s])
        if k == 3:
            srv.step_times.clear()
        srv.step()
    st = srv.statistics()
    return {"api": "MultiStreamCodecServer.submit/step/poll (host frames in and out, H2D + D2H inside step())", "n_streams": B,
            "step_ms_mean_std": st["step_ms"], "chunk_period_ms": 1e3 * T / sr,
            "samples_per_s": B * T / (st["step_ms"][0] * 1e-3), "realtime_factor": B * T / (st["step_ms"][0] * 1e-3) / sr}


def measure_latency_b1(dev, chunks=60):
    """The only numbers the reference publishes (figs/latency.jpg Table 4, RTX 3090: encoder 5.1 ms + symAD decoder 3.2 ms per chunk
    at batch 1), timed the way bin/stream.py:218-223,233-238 does: wall clock around encode+quantize resp. lookup+decode with a
    device synchronise."""
    import torch
    out = {"chunk_samples": 1500, "batch": 1, "timing": "wall clock + device synchronise per call pair, like bin/stream.py:218-238",
           "reference_published_ms": {"encoder": 5.1, "decoder_symAD": 3.2, "hardware": "RTX 3090 (figs/latency.jpg Table 4)"}}
    for wl, key in (("symad", "decoder_symAD"), ("v1", "decoder_hifigan_v1")):
        tx, rx, dec = build_codec(wl, dev)
        x = 0.1 * torch.randn(1, 1, 1500, device=dev)
        te, td = [], []
        for k in range(chunks + 5):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            idx = tx.quantize(tx.encode(x))
            torch.cuda.synchronize(dev)
            t1 = time.perf_counter()
            dec.decode(rx.lookup(idx))
            torch.cuda.synchronize(dev)
            t2 = time.perf_counter()
            if k >= 5:
                te.append((t1 - t0) * 1e3), td.append((t2 - t1) * 1e3)
        if wl == "symad":
            out["encoder_ms_mean_std"] = (statistics.mean(te), statistics.pstdev(te))
            out["encoder_launches"] = int(tx.launch_count // (chunks + 5 + 1))
        out[key + "_ms_mean_std"] = (statistics.mean(td), statistics.pstdev(td))
        out[key + "_launches"] = int((rx.launch_count + dec.launch_count) // (chunks + 5 + 1))
        del tx, rx, dec
    return out


def dump_outputs(out_dir, arrays):
    """What the last timed step returned to its caller, as <name>.npy: float tensors as float32, integer ones as float64 (exact)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        a = t.detach().cpu().numpy()
        np.save(os.path.join(out_dir, name + ".npy"), a.astype(np.float32 if a.dtype.kind == "f" else np.float64))


def run_ours(args):
    import torch
    import torch.distributed as dist
    from audiodec_b200.codec import codec_host

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run --nproc-per-node N for --gpus N > 1")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    B, T, sr = workload_shape(args.workload)
    tx, rx, dec = build_codec(args.workload, dev)

    # synthetic inputs (SURVEY 8(d)): 0.1*randn, seed 1337 (+rank); several distinct resident batches
    gen = torch.Generator().manual_seed(1337 + rank)
    n_in = 4
    x_host = [(0.1 * torch.randn(B, 1, T, generator=gen)).pin_memory() for _ in range(n_in)]
    x_dev = [x.to(dev) for x in x_host]

    def step(i):
        return codec_step(tx, rx, dec, x_dev[i % n_in])

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def max_over_ranks(ms):
        if world == 1:
            return ms
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # pre-warm: clocks / power state settle over the first ~second of load; these steps are not counted in W.  The clock sampler
    # starts BEFORE the warm-up steps and nothing idles between warm-up and the timed region: a 250 ms pause there (round 1 slept to let
    # the sampler spin up) lets some boxes drop their power state, and the first timed steps then run at ramping clocks (measured with
    # per-launch kernel traces: the same kernels ran ~20 % slower in a timed region entered after the pause).
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    t_pre = time.time()
    while time.time() - t_pre < 1.5:
        step(0)
        torch.cuda.synchronize(dev)
    for i in range(args.warmup):
        step(i)
    # The timed region - EXACTLY K steps between barrier + synchronize on both sides, device time by CUDA events, max over ranks - is
    # measured `--regions` R times back to back and the MEDIAN region is reported (all R values are on the line as
    # `timed_regions_ms_per_step`).  Reason: on a shared, power-limited GPU an occasional region runs slow while the rest stay put;
    # a single region is a coin flip, the median is not.
    regions = []
    for r in range(max(1, args.regions)):
        l0 = tx.launch_count + rx.launch_count + dec.launch_count
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        w0 = time.time()
        e0.record()
        for i in range(args.steps):
            y, idx, z, zq = step(i)
        e1.record()
        barrier()
        w1 = time.time()
        regions.append((max_over_ranks(e0.elapsed_time(e1)), w0, w1))
    order = sorted(range(len(regions)), key=lambda k: regions[k][0])
    ms_total, w0, w1 = regions[order[(len(regions) - 1) // 2]]
    clocks = sampler.stop(w0, w1) if rank == 0 else None
    if os.environ.get("ADEC_BENCH_DEBUG") and rank == 0:
        # diagnostic: the same K steps with a device synchronise after each (does sustained back-to-back load run slower on this box?)
        print("sampler rows in the timed region:", [(round(t - w0, 3), r) for (t, r) in sampler.rows if w0 <= t <= w1], file=sys.stderr)
        per = []
        for i in range(args.steps):
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record(); step(i); a1.record()
            torch.cuda.synchronize(dev)
            per.append(a0.elapsed_time(a1))
        print(f"synced per-step ms: {[round(v, 3) for v in per]}; back-to-back mean {ms_total / args.steps:.3f}", file=sys.stderr)
    launches = (tx.launch_count + rx.launch_count + dec.launch_count - l0)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"waveform": y, "code_indices": idx, "z": z, "zq": zq})
    assert torch.isfinite(y).all()
    if tx.range_error() or dec.range_error():
        raise SystemExit("an activation left the fp16-split range of the conv engine: results invalid")

    # ---- e2e: host buffers through adec_codec_host (H2D + 4 calls + D2H inside the timed region)
    for i in range(min(args.warmup, 2)):
        codec_host(tx, dec, x_host[i % n_in], reuse_buffers=True)
    barrier()
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e2.record()
    for i in range(args.steps):
        idx_h, y_h = codec_host(tx, dec, x_host[i % n_in], reuse_buffers=True)
    e3.record()
    barrier()
    ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    F = idx_h.shape[-1]
    hop = y_h.shape[-1] // F

    # ---- per-launch CUDA-event timing of two extra steps (same inputs, same stream): which kernel dominates, and its
    #      achieved algorithmic GB/s.  Outside the timed region so the events do not perturb `value`.
    prof = None
    if rank == 0:
        tx.profile(True), dec.profile(True)
        for i in range(2):
            step(i)
        torch.cuda.synchronize(dev)
        rows = tx.profile_report() + dec.profile_report()
        tx.profile(False), dec.profile(False)
        agg = {}
        for name, ms, nbytes in rows:
            a = agg.setdefault(name, [0, 0.0, nbytes])
            a[0] += 1
            a[1] += ms
        tot = sum(v[1] for v in agg.values())
        top = sorted(agg.items(), key=lambda kv: -kv[1][1])
        if args.breakdown:
            for k, v in agg.items():
                print(f"  {k:44s} {v[1] / v[0]:8.3f} ms  {v[2] / (v[1] / v[0]) / 1e6:8.1f} GB/s(alg)", file=sys.stderr)
            print(f"  sum of launches per step: {tot / 2:.3f} ms", file=sys.stderr)
        dname, (dn, dms, dbytes) = top[0]
        step_ms = ms_total / args.steps                 # shares are of the TIMED step (which also holds the RVQ / lookup launches)
        prof = {"kernel": dname, "launch_ms": dms / dn, "alg_bytes_per_launch": dbytes, "share_of_step": (dms / dn) / step_ms,
                "conv_launches_ms_per_step": tot / 2,
                "top5": [{"op": k, "ms": v[1] / v[0], "GBps": v[2] / (v[1] / v[0]) / 1e6} for k, v in top[:5]]}

    if world > 1:
        dist.destroy_process_group()
    if rank != 0:
        return
    samples_per_step = world * B * T
    value = samples_per_step * args.steps / (ms_total / 1e3)
    e2e_value = samples_per_step * args.steps / (ms_e2e / 1e3)
    peak, peak_src, peaks = measured_peaks()
    per_gpu = value / world
    alg_b = ALG_BYTES_PER_SAMPLE[args.workload]
    achieved = alg_b * per_gpu / 1e9
    k_achieved = prof["alg_bytes_per_launch"] / (prof["launch_ms"] * 1e-3) / 1e9 if prof else achieved
    conv_path = os.environ.get("ADEC_CONV_PATH", "f16")
    engine = {"f16": "wg_conv_kernel (wgmma, fp16-split operands x3 products)", "tc": "wg_conv_kernel (wgmma, fp16-split operands x3 products)",
              "tf32": "wg_conv_kernel (wgmma 3xTF32)", "ffma": "conv_gemm_kernel (fp32 FFMA)"}.get(conv_path, conv_path)
    # compute ceiling: measured here with the library's own MMA-only probe; the tensor-core engines issue 3 MMAs per fp32-grade MAC
    probe = probe_compute(local)
    useful_tflops = ALG_FLOP_PER_SAMPLE[args.workload] * per_gpu / 1e12
    mma_per_mac = {"f16": 3.0, "tc": 3.0, "tf32": 3.0, "ffma": None}.get(conv_path)
    pk = probe.get("tf32_n256_tflops" if conv_path == "tf32" else "f16_n256_tflops")
    compute = {"probe": "adec_probe_mma: every SM streams wgmma (2 warpgroups x M=64, N in 64-column slices) from shared-memory operands, nothing else",
               "measured_tflops": probe, "useful_tflops": useful_tflops, "tensor_products_per_useful_mac": mma_per_mac,
               "issued_tflops": useful_tflops * mma_per_mac if mma_per_mac else None,
               "peak_tflops": pk, "frac": (useful_tflops * mma_per_mac / pk) if (mma_per_mac and pk) else None,
               "samples_per_s_at_peak": (pk * 1e12 / (ALG_FLOP_PER_SAMPLE[args.workload] * mma_per_mac)) if (mma_per_mac and pk) else None,
               "cublas_bf16_tflops_sustained": peaks.get("bf16_tflops_sustained")}
    line = {
        "metric": "48 kHz audio samples/s, encode+quantize+lookup+decode (% HBM roofline in `roofline`)",
        "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_total / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "timed_regions_ms_per_step": [round(r[0] / args.steps, 4) for r in regions],
        "timed_region_choice": f"median of {len(regions)} back-to-back regions of exactly {args.steps} steps each (barrier + synchronize on both sides of every region)",
        "dtype": "bf16" if args.workload == "v1_bf16" else "f32",
        "data": "synthetic (0.1*randn waveforms, seeded synthetic checkpoint; the reference ships no weights)",
        "config": {"workload": WORKLOAD_NAME[args.workload] + f" batch={B}x{T} per GPU (BASELINE configs[{WORKLOAD_CFG[args.workload]}])",
                   "utterances_per_gpu": B, "samples_per_utterance": T, "parallelism": f"independent utterance shards x{world}, no collective",
                   "l2": "per-step activation working set ~3 GB per GPU >> 50 MB L2; inputs rotate over 4 distinct resident batches",
                   "realtime_factor_per_gpu": per_gpu / sr},
        "gpu_launches": int(launches),
        "e2e": {"value": e2e_value, "unit": "samples/s", "h2d_bytes_per_step": B * T * 4,
                "d2h_bytes_per_step": B * F * hop * 4 + 8 * B * F * 8, "ms_per_step": ms_e2e / args.steps,
                "api": "audiodec_b200.codec.codec_host -> adec_codec_host (pinned host buffers, per GPU)"},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "peak_source": peak_src,
                     "model": f"whole step: {alg_b:.1f} algorithmic B/sample (SURVEY.md 8(d) per-conv-layer model) x samples/s per GPU",
                     "kernel": engine + " launch of " + (prof["kernel"] if prof else "?"),
                     "kernel_frac": k_achieved / peak, "kernel_achieved": k_achieved,
                     "kernel_launch_ms": prof["launch_ms"] if prof else None,
                     "kernel_alg_bytes_per_launch": prof["alg_bytes_per_launch"] if prof else None,
                     "kernel_share_of_step": prof["share_of_step"] if prof else None,
                     "conv_launches_ms_per_step": prof["conv_launches_ms_per_step"] if prof else None,
                     "top5_launches": prof["top5"] if prof else None,
                     "compute": compute,
                     "fp32_ffma_peak_tflops_nominal": FFMA_PEAK_TFLOPS},
        "conv_path": conv_path,
        "clocks": clocks,
    }
    if args.parity:
        sel = sorted({0, B // 3, (2 * B) // 3, B - 1})
        if args.workload == "stream_v1":
            xs = torch.cat([x_host[k] for k in range(3)], -1)      # 3 consecutive chunks of the 256 streams
            line["parity"] = parity_vs_oracle(args.workload, dev, xs, sel, chunks=3)
        elif args.workload != "v1_bf16":
            line["parity"] = parity_vs_oracle(args.workload, dev, x_host[0], sel)
    if world == 1 and args.extra and args.workload == "symad":
        extra = {}
        del tx, rx, dec
        torch.cuda.empty_cache()
        for wl, st in (("v1", 3), ("v1_bf16", 3), ("stream_v1", 20)):
            try:
                extra[wl] = measure_extra(wl, dev, st, peak)
            except Exception as e:       # an extra must never take the headline line down
                extra[wl] = {"error": f"{type(e).__name__}: {e}"}
        try:
            extra["stream_v1"]["server"] = measure_stream_server(dev, 10)
            if args.parity:
                g2 = torch.Generator().manual_seed(99)
                xs = 0.1 * torch.randn(256, 1, 4500, generator=g2)
                extra["stream_v1"]["parity"] = parity_vs_oracle("stream_v1", dev, xs, [0, 85, 170, 255], chunks=3)
        except Exception as e:
            extra["stream_v1"]["server_error"] = f"{type(e).__name__}: {e}"
        try:
            extra["latency_b1_1500"] = measure_latency_b1(dev)
        except Exception as e:
            extra["latency_b1_1500"] = {"error": f"{type(e).__name__}: {e}"}
        line["extra_workloads"] = extra
    if args.cpu_baseline and world == 1:          # reported at N=1 only (rank 0); the reference arm covers every N
        wl = "v1" if args.workload in ("v1", "v1_bf16", "stream_v1") else "symad"
        line["cpu_baseline"] = cpu_baseline(wl, n_utt=args.cpu_utts, threads=best_cpu_threads(wl))
        line["cpu_baseline"]["all_cores"] = cpu_all_cores(wl, line["cpu_baseline"]["cores"])
        if args.extra:
            line["gpu_eager_baseline"] = gpu_eager_baseline(wl, dev)
    print(json.dumps(line), flush=True)


def cpu_baseline(workload, n_utt=4, seconds=1.0, threads=None, budget_s=15.0):
    """The reference's CPU path (oracle port: same torch CPU ops) on a bounded sample: up to `n_utt` utterances of
    `seconds` s, one after another (the reference's streaming path is batch-1 only, conv_layer.py:144-146), cut short
    after `budget_s` seconds of host work (never below 2 utterances) so a slow host cannot stretch the run."""
    import torch
    if threads:
        torch.set_num_threads(threads)
    cores = torch.get_num_threads()
    codec = build_oracle(workload)
    torch.manual_seed(1337)
    T = int(seconds * SAMPLE_RATE)
    xs = [0.1 * torch.randn(1, 1, T) for _ in range(min(n_utt, 8))]     # distinct inputs, cycled
    with torch.no_grad():
        codec.run(xs[0][:, :, :6000])          # warm the thread pool / oneDNN primitive cache
        t0 = time.perf_counter()
        done = 0
        while done < n_utt:
            codec.run(xs[done % len(xs)])
            done += 1
            if done >= 2 and time.perf_counter() - t0 > budget_s:
                break
        dt = time.perf_counter() - t0
    n_utt = done
    return {"value": n_utt * T / dt, "unit": "samples/s", "cores": cores, "kind": "port", "utterances": n_utt,
            "sample": f"{n_utt} utterances x {seconds:g} s @ 48 kHz, per-utterance loop (reference streaming path is batch-1), "
                      f"torch {torch.__version__} CPU fp32, {cores} threads; {dt:.2f} s wall",
            "realtime_factor": n_utt * T / dt / SAMPLE_RATE}


def _cpu_worker(args):
    workload, threads, n_utt, budget = args
    r = cpu_baseline(workload, n_utt=n_utt, threads=threads, budget_s=budget)
    return r["utterances"], r["utterances"] * T_SAMPLES / r["value"]


def cpu_all_cores(workload, threads, budget_s=12.0):
    """BASELINE.md section 3 asks for the CPU path on ALL host cores: N = cores // threads independent processes (the reference runs
    one utterance per process, demoFile.py), each with the best single-process thread count; aggregate = total samples / slowest."""
    import multiprocessing as mp
    ncpu = os.cpu_count() or 1
    nproc = max(1, ncpu // max(1, threads))
    if nproc == 1:
        return {"processes": 1, "threads_per_process": threads, "note": "one process already uses every core"}
    try:
        ctx = mp.get_context("spawn")
        t0 = time.perf_counter()
        with ctx.Pool(nproc) as pool:
            res = pool.map(_cpu_worker, [(workload, threads, 64, budget_s)] * nproc)
        wall = time.perf_counter() - t0
        total = sum(u for u, _ in res) * T_SAMPLES
        slowest = max(t for _, t in res)
        return {"value": total / slowest, "unit": "samples/s", "processes": nproc, "threads_per_process": threads, "cores": nproc * threads,
                "host_cpus": ncpu, "utterances": sum(u for u, _ in res), "wall_s": wall,
                "sample": f"{nproc} processes x {threads} threads, each a per-utterance loop time-bounded at {budget_s:g} s"}
    except Exception as e:
        return {"error": f"{type(e).__name__}: {e}"}


def gpu_eager_baseline(workload, dev, n_utt=6):
    """Informational (SURVEY.md 2 / 8(d)): the reference's path as eager PyTorch ops on THIS GPU (oracle port moved to cuda: cuDNN /
    cuBLAS kernels, ~400 launches per utterance), per-utterance loop like the reference must run (its streaming state is batch-1),
    with TF32 off (fp32-grade, the comparable arm) and on (torch's default for cuDNN convs)."""
    import torch
    out = {"kind": "oracle port on cuda (torch eager, cuDNN/cuBLAS); informational, not the graded reference arm"}
    try:
        for name, flag in (("tf32_off", False), ("tf32_on", True)):
            torch.backends.cudnn.allow_tf32 = flag
            torch.backends.cuda.matmul.allow_tf32 = flag
            codec = build_oracle(workload)
            for part in (codec.tx_encoder, codec.rx_encoder, codec.decoder):
                part.to(dev)
            torch.manual_seed(1337)
            xs = [0.1 * torch.randn(1, 1, T_SAMPLES, device=dev) for _ in range(n_utt)]
            with torch.no_grad():
                codec.run(xs[0])
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                for x in xs:
                    codec.run(x)
                torch.cuda.synchronize(dev)
                dt = time.perf_counter() - t0
            out[name] = {"samples_per_s": n_utt * T_SAMPLES / dt, "ms_per_utterance_second": 1e3 * dt / n_utt}
    except Exception as e:
        out["error"] = f"{type(e).__name__}: {e}"
    finally:
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cuda.matmul.allow_tf32 = False
    return out


def best_cpu_threads(workload):
    """The reference's demo default is 4 threads (demoFile.py:28); more threads help up to a point and then hurt (small
    convs, oversubscription).  Pick the fastest of a few counts on a 0.25 s clip so the CPU arm is not handicapped."""
    import torch
    ncpu = os.cpu_count() or 1
    cands = sorted({c for c in (4, 8, 16, 32, 64, ncpu) if c <= ncpu})
    best, best_v = cands[0], 0.0
    for c in cands:
        v = cpu_baseline(workload, n_utt=1, seconds=0.25, threads=c)["value"]
        if v > best_v:
            best, best_v = c, v
    torch.set_num_threads(best)
    return best


def run_reference(args):
    rank = int(os.environ.get("RANK", 0))
    if rank != 0:
        return
    world = int(os.environ.get("WORLD_SIZE", 1))
    wl = "v1" if args.workload in ("v1", "v1_bf16", "stream_v1") else "symad"
    threads = best_cpu_threads(wl)
    per = []
    n_utt = args.ref_utts                       # 16: ~1 s of host work per step on the box's cores, K=10 steps stay well under a minute
    for _ in range(args.warmup):
        cpu_baseline(wl, n_utt=min(2, n_utt))
    t_all0 = time.perf_counter()
    last = None
    for _ in range(args.steps):
        last = cpu_baseline(wl, n_utt=n_utt)
        per.append(last["value"])
    dt = time.perf_counter() - t_all0
    one_proc = statistics.median(per)
    allc = cpu_all_cores(wl, threads)
    value = max(one_proc, allc.get("value", 0.0))      # "all the host threads it can use": the better of one process and N processes
    B, T, _ = workload_shape(args.workload)
    line = {
        "impl": "reference",
        "metric": "48 kHz audio samples/s, encode+quantize+lookup+decode (% HBM roofline in `roofline`)",
        "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * last["utterances"] * T_SAMPLES / one_proc, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic (same seeded checkpoint and waveform distribution as the CUDA arm)",
        "config": {"workload": WORKLOAD_NAME[args.workload] + f" batch={B}x{T} per GPU (BASELINE configs[{WORKLOAD_CFG[args.workload]}]); "
                               "each step a bounded sample of it",
                   "note": "reference = pure-Python torch-CPU path; timed via the oracle port (identical torch ops/order) because "
                           "the reference is not installed where the benchmark runs; rank 0 only; value = best of one process (median over steps) and "
                           "all-cores multi-process"},
        "cpu_baseline": dict(last, value=value, one_process=one_proc, all_cores=allc, cores=allc.get("cores", last["cores"])),
        "e2e": {"value": value, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0, "wall_s": dt,
    }
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="symad", choices=["symad", "v1", "v1_bf16", "stream_v1"],
                    help="symad = BASELINE configs[1] (default, the headline); v1 / v1_bf16 = configs[2] (fp32 resp. bf16 vocoder, batch 128); "
                         "stream_v1 = configs[3]: 256 streams x 1500-sample chunks @ 24 kHz")
    ap.add_argument("--no-cpu-baseline", dest="cpu_baseline", action="store_false")
    ap.add_argument("--no-extra", dest="extra", action="store_false", help="skip extra_workloads and the eager-GPU baseline")
    ap.add_argument("--no-parity", dest="parity", action="store_false", help="skip the oracle check of the timed batch")
    ap.add_argument("--cpu-utts", type=int, default=192,
                    help="utterances of the bounded CPU sample (192 x 1 s = three steps' worth of audio, 10-15 s of host work)")
    ap.add_argument("--ref-utts", type=int, default=16, help="--impl reference: utterances per step (each step time-bounded at 15 s)")
    ap.add_argument("--regions", type=int, default=5, help="timed K-step regions measured back to back; the median is reported, all are listed")
    ap.add_argument("--breakdown", action="store_true", help="print per-launch CUDA-event times to stderr")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="--impl ours: write the last timed step's outputs to DIR/<name>.npy - waveform (B,1,T), z (B,D,F) and zq (B,F,D) "
                         "as float32, code_indices (Nq,B,F) as float64")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs applies to --impl ours only")
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
