"""Batched codecStatistic.py: the per-channel mean and scale of the quantized codes over a wav corpus, the stats/*.npy file every
HiFi-GAN vocoder normalises its input with (HiFiGAN.py:206-219).

    python -m audiodec_b200.codec_statistic -c config/statistic/<tag>.yaml [--subset train] [--subset_num -1] [--cuda 0] \\
        [--batch_seconds 600]

Same flags, config keys (``stats``, ``analyzer``, ``data.path``, ``data.subset[subset]``; paths relative to the current directory),
wav discovery and output file as the reference's codecStatistic.py (:63-112).  The reference runs encoder -> projector ->
Quantizer.forward once per file and calls StandardScaler.partial_fit on each file's (F, 64) codes.  Here the files, read in sorted
order, are packed into varlen batches of at most --batch_seconds of audio: one varlen encode, one RVQ launch that writes
Quantizer.forward's zq (the sum of r + (e - r) over stages), and two launches of per-utterance fp64 moments.  The (n, sum, m2) rows
come back to the host and are merged once per utterance in file order with sklearn 1.9's update, restated below in numpy fp64 (the
package does not import sklearn).  A background thread reads the next batch while the GPU works on the current one.  Every
utterance's moments depend on its own frames only, so the file does not depend on --batch_seconds."""
from __future__ import annotations

import argparse
import logging
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
import yaml

from audiodec_b200.codec import SymADStreamGenerator
from audiodec_b200.codec_test import batches, find_wavs, load_config
from audiodec_b200.wavio import read_wav

_ANALYZER_TYPES = ("symAudioDec", "symAudioDecUniv")      # codecStatistic.py:82-85


class StandardScalerMerge:
    """StandardScaler.partial_fit (scikit-learn 1.9: preprocessing/_data.py, utils/extmath.py _incremental_mean_and_var) restated in
    numpy fp64 for inputs given as per-call moments.  One update(n, sum, m2) is one partial_fit of an (n, D) array X with
    sum = sum_f X and m2 = sum_f (X - T)^2 - (sum_f (X - T))^2 / n, T = sum / n (the corrected two-pass term sklearn computes); no
    NaNs, no sample weights."""

    def __init__(self, dim):
        self.n = 0.0                                   # n_samples_seen_ (as float64, how the update uses it)
        self.mean = np.zeros(dim, np.float64)
        self.var = np.zeros(dim, np.float64)

    def update(self, n, s, m2):
        n = float(n)
        s, m2 = np.asarray(s, np.float64), np.asarray(m2, np.float64)
        last_n = self.n
        last_sum = self.mean * last_n
        upd_n = last_n + n
        upd_mean = (last_sum + s) / upd_n
        if last_n == 0:                                # `zeros = last_sample_count == 0` case: the new term alone
            upd_unnorm = m2
        else:
            last_over_new = last_n / n
            upd_unnorm = self.var * last_n + m2 + last_over_new / upd_n * (last_sum / last_over_new - s) ** 2   # Chan et al.
        self.n, self.mean, self.var = upd_n, upd_mean, upd_unnorm / upd_n

    def scale(self):
        """scale_ = sqrt(var_), with _is_constant_feature's channels set to 1 (_handle_zeros_in_scale with constant_mask)."""
        eps = np.finfo(np.float64).eps
        constant = self.var <= self.n * eps * self.var + (self.n * self.mean * eps) ** 2
        scale = np.sqrt(self.var)
        scale[constant] = 1.0
        return scale

    def stats(self):
        """[mean_, scale_] as float32 (2, D): what codecStatistic.py:106-111 saves."""
        return np.stack([self.mean, self.scale()], axis=0).astype(np.float32)


def _need(cfg, *keys):
    v = cfg
    for k in keys:
        if not isinstance(v, dict) or k not in v:
            raise SystemExit(f"the config names no {'.'.join(str(x) for x in keys)} (codecStatistic.py:47-50, :65-68)")
        v = v[k]
    return v


def _read(utt_path):
    utt, path = utt_path
    audio, _ = read_wav(path)
    if audio.shape[1] != 1:
        # the reference feeds (1, C, T) to a 1-input conv and raises; say which file it is
        raise SystemExit(f"{path} has {audio.shape[1]} channels; the analyzer takes mono audio")
    return utt, audio


def accumulate(encoder, utts, sample_rate, batch_seconds, on_batch=None, timing=None):
    """Fit the merge over utts [(utt_id, path)] in order, at most batch_seconds of audio per GPU batch.  on_batch(utt_ids, frames,
    idx (Nq, sum F) device int64) sees each batch's indices.  timing (dict) receives the host read seconds, the GPU seconds (events
    around each batch's launches) and the number of samples."""
    dev = encoder._device
    merge = StandardScalerMerge(encoder.code_dim)
    read_s, gpu_ms, samples = 0.0, 0.0, 0

    def read_next(it):
        t0 = time.perf_counter()
        run = next(it, None)
        return run, time.perf_counter() - t0

    runs = batches(map(_read, utts), sample_rate, batch_seconds)
    with ThreadPoolExecutor(1) as pool, torch.no_grad():
        fut = pool.submit(read_next, runs)
        while True:
            run, dt = fut.result()
            read_s += dt
            if run is None:
                break
            fut = pool.submit(read_next, runs)            # the next batch is read while this one runs
            lengths = [a.shape[0] for _, a in run]
            x = torch.from_numpy(np.concatenate([a[:, 0] for _, a in run])).pin_memory().to(dev, non_blocking=True)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            z, frames = encoder.encode_offline_varlen(list(torch.split(x, lengths)))
            zq, idx = encoder.quantize_forward(z)
            s, m2 = encoder.zq_moments(zq, frames)
            ev[1].record()
            rows = torch.stack([s, m2]).cpu().numpy()   # (2, B, D); synchronises
            gpu_ms += ev[0].elapsed_time(ev[1])
            samples += sum(lengths)
            if on_batch is not None:
                on_batch([u for u, _ in run], frames, idx.reshape(idx.size(0), -1))
            for b, n in enumerate(frames):
                merge.update(n, rows[0, b], rows[1, b])
    if timing is not None:
        timing.update(read_s=read_s, gpu_s=gpu_ms / 1e3, samples=samples)
    return merge


def _arguments(argv):
    ap = argparse.ArgumentParser(description="Mean and scale of the quantized codes over a wav corpus, on an H100, many files per batch")
    ap.add_argument("-c", "--config", type=str, required=True)
    ap.add_argument("--subset", type=str, default="train")
    ap.add_argument("--subset_num", type=int, default=-1)
    ap.add_argument("--cuda", type=int, default=0, help="CUDA ordinal; negative (a CPU run) is refused")
    ap.add_argument("--batch_seconds", type=float, default=600.0,
                    help="most audio (seconds at the analyzer's sampling_rate) packed into one batch")
    return ap.parse_args(argv)


def main(argv=None, on_batch=None, timing=None):
    args = _arguments(argv)
    logging.basicConfig(level=logging.INFO, stream=sys.stdout, format="%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s")
    if args.cuda < 0:
        raise SystemExit("audiodec_b200 has no CPU path: pass --cuda <ordinal>")
    if args.batch_seconds <= 0:
        raise SystemExit("--batch_seconds must be > 0")
    with open(args.config) as f:
        config = yaml.load(f, Loader=yaml.FullLoader)
    stats_path, analyzer = _need(config, "stats"), _need(config, "analyzer")
    data_path = os.path.join(_need(config, "data", "path"), _need(config, "data", "subset", args.subset))
    if not os.path.exists(analyzer):
        raise SystemExit(f"{analyzer} does not exist!")
    analyzer_cfg = load_config(analyzer)
    kind = analyzer_cfg.get("model_type", "symAudioDec")
    if kind not in _ANALYZER_TYPES:
        raise NotImplementedError(f"Analyzer {kind} is not supported!")
    if analyzer_cfg["generator_params"].get("input_channels", 1) > 1:
        raise NotImplementedError("only mono analyzers are built (input_channels = 1)")
    if not os.path.exists(data_path):
        raise SystemExit(f"{data_path} does not exist!")
    try:
        utts = find_wavs(data_path, args.subset_num)
    except ValueError as e:
        raise SystemExit(str(e)) from None
    logging.info(f"The number of {args.subset} audio files = {len(utts)}.")

    dev = torch.device("cuda", args.cuda)
    encoder = SymADStreamGenerator(**analyzer_cfg["generator_params"])
    encoder.load_state_dict(torch.load(analyzer, map_location="cpu")["model"]["generator"])
    encoder = encoder.eval().to(dev)
    logging.info(f"Loaded Analyzer from {analyzer}.")
    with torch.cuda.device(dev):
        merge = accumulate(encoder, utts, analyzer_cfg.get("sampling_rate", 48000), args.batch_seconds, on_batch, timing)
    if os.path.dirname(stats_path):
        os.makedirs(os.path.dirname(stats_path), exist_ok=True)
    np.save(stats_path, merge.stats(), allow_pickle=False)
    logging.info(f"Finished statistical calculation of {len(utts)} utterances.")
    return stats_path


if __name__ == "__main__":
    main()
