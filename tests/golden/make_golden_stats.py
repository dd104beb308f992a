#!/usr/bin/env python3
"""Golden statistics of codecStatistic.py from the UNMODIFIED reference.

Run in the build container only (needs /root/reference, CPU, scikit-learn):   python tests/golden/make_golden_stats.py

Writes a synthetic wav corpus (audiodec_b200.synthetic.make_wav_corpus: 40 mono 48 kHz files in nested folders, from 1 sample up to
8 s, plus files that are not *.wav and must be ignored), a statistic config and the synthetic symAD analyzer of
make_model_zoo(..., "vctk_sym", seed=0), then runs the reference's codecStatistic.StatisticMain itself (load_dataset,
load_analyzer, run) for the whole corpus and for --subset_num 7.  soundfile is not in this image; a stand-in built on
scipy.io.wavfile gives what sf.read does for PCM16: float64 samples / 32768, (T, C) with always_2d.  The analyzer's quantizer is
wrapped to record its indices (ResidualVQ.forward_index on the same z) next to the forward it runs.

Stores tests/golden/stats_vctk.npz: the corpus recipe, the sha256 of every wav, both stats arrays, and the reference's local
indices of every frame (uint16, (Nq, sum F) in file order, with the per-file frame counts).  Nothing under tests/ reads
/root/reference at test time."""
import hashlib
import os
import sys
import tempfile
import types
import warnings
from argparse import Namespace

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.dont_write_bytecode = True
sys.path.insert(0, "/root/reference")
sys.path.insert(0, REPO)
warnings.filterwarnings("ignore")

from audiodec_b200 import synthetic as S  # noqa: E402

torch.set_num_threads(4)

SEED, SR = 7, 48000
# 1 sample, under one hop, one hop and around it, two hops, 0.1 s, 1 s, 8 s, and 28 log-uniform lengths in between
FIXED = [1, 2, 150, 299, 300, 301, 599, 600, 601, 4800, 48000, 384000]
EXTRA = ["notes.txt", "spk1/utt_0001.wav.txt", "spk2/sess0/list.scp"]      # not *.wav: find_files skips them
STATS_REL = "stats/symAD_vctk_48000_hop300_synthetic.npy"


def lengths():
    rng = np.random.default_rng(SEED)
    rand = np.exp(rng.uniform(np.log(1000), np.log(200000), 28)).astype(np.int64)
    return FIXED + [int(x) for x in rand]


def write_corpus(root):
    paths = S.make_wav_corpus(root, SEED, lengths(), SR)
    for rel in EXTRA:
        os.makedirs(os.path.dirname(os.path.join(root, rel)) or root, exist_ok=True)
        with open(os.path.join(root, rel), "w") as f:
            f.write("not audio\n")
    return paths


def _soundfile_standin():
    from scipy.io import wavfile

    def read(path, always_2d=False, dtype="float64"):
        fs, raw = wavfile.read(path)
        assert raw.dtype == np.int16
        data = raw.astype(np.float64) / 32768.0
        if always_2d and data.ndim == 1:
            data = data[:, None]
        return data.astype(dtype), fs

    return types.SimpleNamespace(read=read, __name__="soundfile")


def main():
    sys.modules["soundfile"] = _soundfile_standin()
    import codecStatistic
    scratch = tempfile.mkdtemp(prefix="adec_golden_stats_")
    os.chdir(scratch)
    _, analyzer, _ = S.make_model_zoo(scratch, "vctk_sym", seed=0)
    corpus = os.path.join("corpus", "train")
    paths = write_corpus(corpus)
    cfg = {"sampling_rate": SR, "data": {"path": "corpus", "subset": {"train": "train"}},
           "analyzer": os.path.relpath(analyzer, scratch), "stats": STATS_REL}
    with open("statistic.yaml", "w") as f:
        yaml.safe_dump(cfg, f)

    out = {}
    for tag, subset_num in (("full", -1), ("sub7", 7)):
        sm = codecStatistic.StatisticMain(Namespace(config="statistic.yaml", subset="train", subset_num=subset_num))
        sm.load_dataset("train", subset_num)
        sm.load_analyzer()
        q = sm.analyzer.quantizer
        recorded = []
        forward = q.forward

        def recording_forward(z, q=q, forward=forward, recorded=recorded):
            recorded.append(q.codebook.forward_index(z.transpose(2, 1))[1].reshape(len(q.codebook.layers), -1).numpy())
            return forward(z)

        q.forward = recording_forward
        sm.run()
        out[f"stats_{tag}"] = np.load(STATS_REL)
        if tag == "full":
            files = [os.path.relpath(f, corpus) for f in sm.dataset.filenames]
            out["files"] = np.array(files)
            out["frames"] = np.array([r.shape[1] for r in recorded], np.int64)
            out["idx"] = np.concatenate(recorded, axis=1).astype(np.uint16)
    rel = [os.path.relpath(p, corpus) for p in paths]
    sha = [hashlib.sha256(open(p, "rb").read()).hexdigest() for p in paths]
    np.savez_compressed(os.path.join(HERE, "stats_vctk.npz"), seed=SEED, sr=SR, lengths=np.array(lengths(), np.int64),
                        wavs=np.array(rel), sha256=np.array(sha), extra=np.array(EXTRA), config=yaml.safe_dump(cfg),
                        torch=torch.__version__, **out)
    print("files", len(out["files"]), "frames", int(out["frames"].sum()), "stats", out["stats_full"].shape,
          "scale range", float(out["stats_full"][1].min()), float(out["stats_full"][1].max()))


if __name__ == "__main__":
    main()
