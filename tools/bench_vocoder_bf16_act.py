#!/usr/bin/env python3
"""The HiFi-GAN vocoder's two bf16 modes side by side on BASELINE configs[2] and configs[3]:

    python tools/bench_vocoder_bf16_act.py [--steps 5] [--regions 3] [--server-steps 20]

  mode 1  `decoder.to(torch.bfloat16)`: bf16 conv operands, fp32 activations / state / decode I/O (what bench.py --workload v1_bf16 times)
  mode 2  `decoder.set_activation_dtype(torch.bfloat16)`: bf16 operands and bf16 activations / state / decode I/O

configs[2] is AD v1 (symAD encoder fp32-grade + HiFi-GAN v1) at 128 x 48000 per step.  The two modes run in ONE process, their timed
regions alternated (mode 1, mode 2, mode 1, ...), and each mode reports the median region.  Per mode it prints ms/step and samples/s,
the whole-step fraction of the HBM bound under SURVEY.md section 8(d)'s C3 byte model (11,633 B/sample with bf16 activations), the
decoder's top-5 launches with their algorithmic GB/s (adec_profile_report), the configs[3] step through MultiStreamCodecServer
(libritts v1, 256 streams x 1500 samples at 24 kHz; the two servers' steps alternated) with the decoder's kernel time in it, and a
parity block: 4 rows of the timed batch from a fresh codec against the fp32 oracle under the reference-derived bar of
tests/test_vocoder_bf16_act_gpu.py.  The GPU's name, power limit and SM clocks are read in the same run.  Prints one JSON object;
writes nothing.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (build_codec-style warm-up, codec_step, the timing loop, peaks and the clock sampler)

C3_BYTES_PER_SAMPLE = 11633.0          # SURVEY.md 8(d) C3: AD v1 with bf16 activations
B, T, SR = 128, 48000, 48000
SEL = [0, 42, 85, 127]


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, plim, smax, sm = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": smax, "sm_clock_now": sm}
    except Exception as e:                          # the timing stands without it; say why it is missing
        return {"error": f"nvidia-smi query failed: {e}"}


def build(mode, dev):
    """Warmed tx / rx encoders and a v1 decoder in bf16 mode `mode` (bin/stream.py:56-77)."""
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    sd = S.symad_state_dict(seed=0)
    enc = []
    for _ in range(2):
        e = SymADStreamGenerator(**S.SYMAD_PARAMS)
        e.load_state_dict(sd)
        enc.append(e.eval().to(dev))
    d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    d.load_state_dict(S.hifigan_state_dict(seed=1))
    d = d.to(torch.bfloat16)
    if mode == 2:
        d = d.set_activation_dtype(torch.bfloat16)
    d = d.eval().to(dev)
    tx, rx = enc
    tx.initial_encoder(8192, dev)
    d.initial_decoder(rx.initial_encoder(8192, dev))
    torch.cuda.synchronize(dev)
    return tx, rx, d


def top_launches(tx, rx, dec, x, dev, n=5):
    import torch
    dec.profile(True)
    bench.codec_step(tx, rx, dec, x)
    torch.cuda.synchronize(dev)
    rows = dec.profile_report()
    dec.profile(False)
    return [{"op": name, "ms": round(ms, 4), "alg_bytes": b, "GBps_alg": round(b / ms / 1e6, 1)}
            for name, ms, b in sorted(rows, key=lambda r: -r[1])[:n]]


def server_steps(dev, steps):
    """configs[3] through MultiStreamCodecServer with a mode-1 and a mode-2 decoder, their steps alternated; per mode the host-clock
    step (H2D, all launches, D2H, frame hand-off) and the decoder's kernel time in one profiled step."""
    import numpy as np
    import torch
    from audiodec_b200.server import MultiStreamCodecServer
    n, fs, sr = 256, 1500, 24000
    rng = np.random.default_rng(7)
    frames = (0.1 * rng.standard_normal((4, n, fs))).astype(np.float32)
    srv = {}
    for m in (1, 2):
        tx, rx, dec = build(m, dev)
        srv[m] = MultiStreamCodecServer(tx, rx, dec, n_streams=n, frame_size=fs, sample_rate=sr, max_latency=1.0, device=dev)
    for k in range(steps + 3):
        for m in (1, 2):
            for s in range(n):
                srv[m].submit(s, frames[k % 4, s])
            if k == 3:
                srv[m].step_times.clear()
            srv[m].step()
            for s in range(n):
                srv[m].poll(s)
    out = {}
    for m in (1, 2):
        st = srv[m].statistics()
        dec = srv[m].decoder
        for s in range(n):
            srv[m].submit(s, frames[0, s])
        dec.profile(True)
        srv[m].step()
        torch.cuda.synchronize(dev)
        rows = dec.profile_report()
        dec.profile(False)
        out[m] = {"n_streams": n, "chunk_samples": fs, "sample_rate": sr, "steps": steps, "step_ms_mean_std": st["step_ms"],
                  "decoder_kernel_ms_per_step": sum(r[1] for r in rows), "decoder_alg_bytes_per_step": sum(r[2] for r in rows),
                  "chunk_period_ms": 1e3 * fs / sr}
    return out


def parity(mode, dev, x, oracle_out, bar):
    """Fresh warmed codec on the timed batch; rows SEL against the fp32 oracle.  Frames whose code indices differ from the oracle
    are counted and left out of the waveform comparison (the encoder is fp32-grade; a difference there is a tie, not the vocoder)."""
    import torch
    tx, rx, dec = build(mode, dev)
    y, idx = bench.codec_step(tx, rx, dec, x)[:2]
    y, idx = y.float().cpu()[SEL], idx.cpu()[:, SEL]
    _, ridx, _, ry = oracle_out
    ok = ~(idx != ridx).any(0)
    ok_s = ok.repeat_interleave(300, dim=-1).unsqueeze(1)
    d, r = (y - ry)[ok_s], ry[ok_s]
    err = d.abs().max().item()
    snr = (10 * torch.log10(r.pow(2).mean() / d.pow(2).mean())).item()
    return {"rows": SEL, "frames": int(ok.numel()), "frames_idx_differ": int((~ok).sum()), "max_abs_vs_fp32": err, "snr_db_vs_fp32": snr,
            "bar": bar, "pass": bool(err <= bar["max_abs"] and snr >= bar["snr_db"])}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=5, help="steps per timed region")
    ap.add_argument("--regions", type=int, default=3, help="timed regions per mode (median reported)")
    ap.add_argument("--server-steps", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_vocoder_bf16_act: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda:0")
    peak, peak_src, _ = bench.measured_peaks()
    out = {"gpu": gpu_info(0), "config": f"BASELINE configs[2]: AD v1, batch {B}x{T} per step", "c3_bytes_per_sample": C3_BYTES_PER_SAMPLE,
           "hbm_GBps_denominator": peak, "hbm_denominator_source": peak_src, "modes": {}}
    codecs = {m: build(m, dev) for m in (1, 2)}
    gen = torch.Generator().manual_seed(4242)
    xs = [(0.1 * torch.randn(B, 1, T, generator=gen)).to(dev) for _ in range(4)]
    sync = lambda: torch.cuda.synchronize(dev)
    for m in (1, 2):                                           # warm every shape of the timed window
        for i in range(3):
            bench.codec_step(*codecs[m], xs[i % 4])
    sync()
    clocks = bench.ClockSampler(0)
    clocks.start()
    import time
    t0 = time.time()
    runs = {1: [], 2: []}
    for r in range(args.regions):
        for m in (1, 2):
            ms, y = bench.time_device_loop(lambda i: bench.codec_step(*codecs[m], xs[i % 4])[0], args.steps, 0, dev, sync)
            runs[m].append(ms / args.steps)
            assert torch.isfinite(y.float()).all()
    out["sm_clocks_during_timing"] = clocks.stop(t0, time.time())
    for m in (1, 2):
        ms = statistics.median(runs[m])
        sps = B * T / (ms / 1e3)
        out["modes"][str(m)] = {"regions_ms_per_step": [round(v, 3) for v in runs[m]], "ms_per_step": ms, "samples_per_s": sps,
                                "c3_step_frac_of_hbm_bound": C3_BYTES_PER_SAMPLE * sps / 1e9 / peak,
                                "decoder_top5_launches": top_launches(*codecs[m], xs[0], dev)}
    del codecs
    torch.cuda.empty_cache()
    for m, r in server_steps(dev, args.server_steps).items():
        out["modes"][str(m)]["configs3_server"] = r
    torch.cuda.empty_cache()
    g = np.load(os.path.join(ROOT, "tests", "golden", "bf16_act.npz"))
    y32, y16 = torch.from_numpy(g["v1_y_fp32"]), torch.from_numpy(g["v1_y_bf16"])
    ref_err = (y16 - y32).abs().max().item()
    ref_snr = (10 * torch.log10(y32.pow(2).mean() / (y16 - y32).pow(2).mean())).item()
    bar = {"max_abs": 1.2 * ref_err, "snr_db": ref_snr - 2.0, "derived_from": "the reference's own bf16 v1 output (tests/golden/bf16_act.npz)"}
    orc = bench.build_oracle("v1")
    with torch.no_grad():
        oracle_out = orc.run(xs[0].cpu()[SEL])
    for m in (1, 2):
        out["modes"][str(m)]["parity"] = parity(m, dev, xs[0], oracle_out, bar)
        torch.cuda.empty_cache()
    out["speedup_mode2_over_mode1"] = out["modes"]["1"]["ms_per_step"] / out["modes"]["2"]["ms_per_step"]
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
