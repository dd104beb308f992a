#!/usr/bin/env python3
"""The non-streaming codec (codecTest.py's workload: a corpus of utterances of different lengths) three ways, in one process:

    python tools/bench_offline_varlen.py [--regions 3] [--bucket 16]

  (a) one utterance per call: encode_offline -> quantize_offline -> forward / decode_offline at B = 1 (what codecTest.py does)
  (b) sorted by length, `--bucket` utterances per batch padded to the batch's longest, uniform offline calls, outputs cropped
  (c) the same buckets as varlen calls (encode_offline_varlen -> quantize_offline -> forward_varlen / decode_offline_varlen): no padding

The corpus is SYNTHETIC: 256 mono 48 kHz utterances of seeded noise, lengths log-normal around 3 s clipped to [0.5, 12] s.  Two
models: AD v1 (symAD encoder + RVQ + HiFi-GAN v1, fp32) and vctk_sym (symAD encoder + RVQ + symAD decoder), synthetic weights.  The
arms' timed regions are alternated (a, b, c, a, b, c, ...); each arm reports the median region as input samples per second, end to
end from device-resident audio to device-resident waveforms.  Also reported: (b)'s padded-row fraction computed from the shapes,
whether (c)'s waveforms equal (a)'s bit for bit, and the GPU's name and power limit read in the same run.  Prints one JSON object;
writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SR, N_UTT = 48000, 256


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, plim, smax = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": smax}
    except Exception as e:                          # the timing stands without it; say why it is missing
        return {"error": f"nvidia-smi query failed: {e}"}


def corpus_lengths(seed=0):
    import numpy as np
    r = np.random.default_rng(seed)
    secs = np.clip(np.exp(r.normal(np.log(3.0), 0.5, N_UTT)), 0.5, 12.0)
    return [int(s * SR) for s in secs]


def models(dev):
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    enc = SymADStreamGenerator(**S.SYMAD_PARAMS)
    enc.load_state_dict(S.symad_state_dict(seed=0))
    enc = enc.eval().to(dev)
    v1 = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    v1.load_state_dict(S.hifigan_state_dict(seed=1))
    sym = SymADStreamGenerator(**S.SYMAD_PARAMS)
    sym.load_state_dict(S.symad_state_dict(seed=0))
    torch.cuda.synchronize(dev)
    return enc, {"ad_v1": (v1.eval().to(dev), lambda c: v1.forward(c), v1.forward_varlen),
                 "vctk_sym": (sym.eval().to(dev), lambda c: sym.decode_offline(c), sym.decode_offline_varlen)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--regions", type=int, default=3)
    ap.add_argument("--bucket", type=int, default=16)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_offline_varlen needs a CUDA device")
    dev = torch.device("cuda", args.device)
    lengths = corpus_lengths()
    torch.manual_seed(0)
    xs = [0.1 * torch.randn(n, device=dev) for n in lengths]
    order = sorted(range(N_UTT), key=lambda i: lengths[i])
    buckets = [order[i:i + args.bucket] for i in range(0, N_UTT, args.bucket)]
    padded = sum(len(b) * max(lengths[i] for i in b) for b in buckets)
    enc, decs = models(dev)
    hop = enc._lib.adec_hop_length(enc._h)

    def arm_a(dec):
        out = [None] * N_UTT
        for i, x in enumerate(xs):
            zq, _ = enc.quantize_offline(enc.encode_offline(x.view(1, 1, -1)))
            out[i] = dec(zq)[0, 0]
        return out

    def arm_b(dec):
        out = [None] * N_UTT
        for b in buckets:
            tmax = max(lengths[i] for i in b)
            x = torch.zeros(len(b), 1, tmax, device=dev)
            for k, i in enumerate(b):
                x[k, 0, :lengths[i]] = xs[i]
            zq, _ = enc.quantize_offline(enc.encode_offline(x))
            y = dec(zq)
            for k, i in enumerate(b):
                out[i] = y[k, 0, :-(-lengths[i] // hop) * hop]
        return out

    def arm_c(dec_vl):
        out = [None] * N_UTT
        for b in buckets:
            z, frames = enc.encode_offline_varlen([xs[i] for i in b])
            zq, _ = enc.quantize_offline(z)
            for i, y in zip(b, dec_vl(zq, frames)):
                out[i] = y[0, 0]
        return out

    result = {"corpus": f"synthetic: {N_UTT} mono {SR} Hz utterances of seeded noise, lengths log-normal around 3 s clipped to [0.5, 12] s",
              "total_seconds": round(sum(lengths) / SR, 1), "bucket": args.bucket,
              "padded_fraction_b": round(1.0 - sum(lengths) / padded, 4), "gpu": gpu_info(args.device), "models": {}}
    for name, (_, dec, dec_vl) in decs.items():
        arms = {"a_per_utterance": lambda: arm_a(dec), "b_padded_buckets": lambda: arm_b(dec), "c_varlen_buckets": lambda: arm_c(dec_vl)}
        for fn in arms.values():                    # warm-up: every shape of the timed regions
            fn()
        torch.cuda.synchronize(dev)
        times = {k: [] for k in arms}
        outs = {}
        for _ in range(args.regions):
            for k, fn in arms.items():
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                outs[k] = fn()
                torch.cuda.synchronize(dev)
                times[k].append(time.perf_counter() - t0)
        med = {k: statistics.median(v) for k, v in times.items()}
        same = all(torch.equal(ya, yc) for ya, yc in zip(outs["a_per_utterance"], outs["c_varlen_buckets"]))
        result["models"][name] = {
            "samples_per_s": {k: round(sum(lengths) / t) for k, t in med.items()},
            "region_s": {k: [round(t, 4) for t in v] for k, v in times.items()},
            "speedup_c_over_b": round(med["b_padded_buckets"] / med["c_varlen_buckets"], 3),
            "speedup_c_over_a": round(med["a_per_utterance"] / med["c_varlen_buckets"], 3),
            "c_equals_a_bitwise": same}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
