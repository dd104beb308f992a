#!/usr/bin/env python3
"""The batched codecStatistic.py end to end on a synthetic corpus, and the repo's CPU oracle port as a baseline:

    python tools/bench_codec_statistic.py [--regions 3] [--baseline_utts 16] [--batch_seconds 600]

The corpus is SYNTHETIC: 256 mono 48 kHz PCM16 wav files (synthetic.make_wav_corpus), lengths log-normal around 3 s clipped to
[0.5, 12] s, written with the symAD analyzer of make_model_zoo(..., "vctk_sym", seed=0) and a statistic config to a temporary
directory that is removed at the end.  After one warm-up run, each of --regions runs of the CLI (audiodec_b200.codec_statistic.main)
reports, and the median is taken of: end-to-end input samples per second (wall clock from the config to the saved file, model load
included), the host's wav read time (in the background thread), and the GPU time (CUDA events around each batch's encode ->
quantize_forward -> zq_moments).  Also the moment kernels alone on the whole corpus's frames as one batch (events, mean of 20).
Baseline, labelled as such: oracle/audiodec_oracle.py's torch-CPU forward_encode + forward_quantize one file at a time plus the
numpy merge, on the first --baseline_utts files, with the core count and torch's thread count.  The GPU's name and power limit are
read in the same run.  Prints one JSON object."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--regions", type=int, default=3)
    ap.add_argument("--baseline_utts", type=int, default=16)
    ap.add_argument("--batch_seconds", type=float, default=600.0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import yaml
    if not torch.cuda.is_available():
        raise SystemExit("bench_codec_statistic needs a CUDA device")
    from audiodec_b200 import codec_statistic as CS
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec_test import find_wavs
    from audiodec_b200.wavio import read_wav

    lengths = corpus_lengths()
    work = tempfile.mkdtemp(prefix="adec_stats_bench_")
    cwd = os.getcwd()
    try:
        os.chdir(work)
        _, analyzer, _ = S.make_model_zoo(work, "vctk_sym", seed=0)
        S.make_wav_corpus(os.path.join(work, "corpus", "train"), 0, lengths, SR)
        cfg = {"data": {"path": "corpus", "subset": {"train": "train"}}, "analyzer": os.path.relpath(analyzer, work),
               "stats": "stats/bench.npy"}
        with open("statistic.yaml", "w") as f:
            yaml.safe_dump(cfg, f)
        argv = ["-c", "statistic.yaml", "--cuda", str(args.device), "--batch_seconds", str(args.batch_seconds)]
        CS.main(argv)                                                  # warm-up: module load, every batch shape
        runs = []
        for _ in range(args.regions):
            timing = {}
            torch.cuda.synchronize(args.device)
            t0 = time.perf_counter()
            CS.main(argv, timing=timing)
            timing["wall_s"] = time.perf_counter() - t0
            runs.append(timing)
        stats_gpu = np.load(cfg["stats"])

        # the moment kernels alone, the whole corpus as one batch
        from audiodec_b200.codec import SymADStreamGenerator, varlen_layout
        dev = torch.device("cuda", args.device)
        enc = SymADStreamGenerator(**S.SYMAD_PARAMS)
        enc.load_state_dict(S.symad_state_dict(seed=0))
        enc = enc.eval().to(dev)
        frames, _ = varlen_layout(lengths, S.SYMAD_PARAMS["enc_strides"])
        zq = torch.randn(sum(frames), 64, device=dev)
        enc.zq_moments(zq, frames)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(20):
            enc.zq_moments(zq, frames)
        ev[1].record()
        torch.cuda.synchronize(dev)
        moments_ms = ev[0].elapsed_time(ev[1]) / 20

        # baseline: the oracle port on the CPU, one file at a time (what codecStatistic.py does on a CPU)
        from oracle.audiodec_oracle import SymADOracle
        orc = SymADOracle(S.SYMAD_PARAMS, S.symad_state_dict(seed=0))
        utts = find_wavs(cfg["data"]["path"] + "/train")[:args.baseline_utts]
        merge = CS.StandardScalerMerge(64)
        t0, n_base = time.perf_counter(), 0
        with torch.no_grad():
            for _, p in utts:
                a, _ = read_wav(p)
                x = torch.from_numpy(a).transpose(1, 0).unsqueeze(0)
                zqo = orc.forward_quantize(orc.forward_encode(x))[0].transpose(0, 1).double().numpy()
                s = zqo.sum(0)
                d = zqo - s / len(zqo)
                merge.update(len(zqo), s, (d * d).sum(0) - d.sum(0) ** 2 / len(zqo))
                n_base += a.shape[0]
        base_s = time.perf_counter() - t0
    finally:
        os.chdir(cwd)
        shutil.rmtree(work, ignore_errors=True)

    med = {k: statistics.median(r[k] for r in runs) for k in ("wall_s", "read_s", "gpu_s")}
    total = runs[0]["samples"]
    print(json.dumps({
        "corpus": f"synthetic: {N_UTT} mono {SR} Hz PCM16 wav files, lengths log-normal around 3 s clipped to [0.5, 12] s",
        "total_seconds": round(total / SR, 1), "frames": sum(frames), "batch_seconds": args.batch_seconds, "gpu": gpu_info(args.device),
        "cli": {"samples_per_s": round(total / med["wall_s"]), "wall_s": round(med["wall_s"], 3), "host_read_s": round(med["read_s"], 3),
                "gpu_s": round(med["gpu_s"], 3), "gpu_samples_per_s": round(total / med["gpu_s"]),
                "regions": [{k: round(v, 4) for k, v in r.items() if k != "samples"} for r in runs]},
        "zq_moments_ms_whole_corpus": round(moments_ms, 4),
        "baseline_oracle_cpu": {"what": "oracle port: torch-CPU forward_encode + forward_quantize per file + numpy merge",
                                "files": len(utts), "samples_per_s": round(n_base / base_s), "cpu_cores": os.cpu_count(),
                                "torch_threads": torch.get_num_threads()},
        "stats_finite": bool(np.isfinite(stats_gpu).all())}))


if __name__ == "__main__":
    main()
