"""CPU checks of the batched codecStatistic.py: the host merge against scikit-learn's StandardScaler, negative controls that the
same check must reject, the CLI's refusals, and the golden corpus recipe."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import yaml

from audiodec_b200 import synthetic as S
from audiodec_b200.codec_statistic import StandardScalerMerge

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "stats_vctk.npz")
D = 64


def _utterances(seed=0):
    """Per-utterance float32 (F, 64) arrays: random lengths with single-frame ones among them; channel 0 is constant (0.3 in fp32,
    whose widened sum is not n * 0.3 exactly), channel 1 has mean 1e3 and std 1e-3, the rest are Gaussian with per-channel means."""
    rng = np.random.default_rng(seed)
    lengths = [1, 57, 1, 1, 400, 3, 1000, 2, 1, 250, 1, 31, 4096, 1]
    means = rng.normal(0, 0.5, D)
    out = []
    for n in lengths:
        x = (means + rng.standard_normal((n, D))).astype(np.float32)
        x[:, 0] = np.float32(0.3)
        x[:, 1] = (1e3 + 1e-3 * rng.standard_normal(n)).astype(np.float32)
        out.append(x)
    return out


def _moments(x, acc=np.float64, centred=True):
    """(n, sum, m2) of one utterance as the device computes them: the corrected two-pass term, accumulated in `acc`."""
    n = x.shape[0]
    xs = x.astype(acc)
    s = xs.sum(0, dtype=acc)
    if not centred:                                     # the textbook one-pass form sum x^2 - n mean^2
        return n, s, (xs * xs).sum(0, dtype=acc) - n * (s / n) ** 2
    d = xs - s / n
    return n, s, (d * d).sum(0, dtype=acc) - d.sum(0, dtype=acc) ** 2 / n


def _sklearn(utts):
    sk = pytest.importorskip("sklearn.preprocessing")
    scaler = sk.StandardScaler()
    for x in utts:
        scaler.partial_fit(x)
    return scaler.mean_, scaler.scale_


def _rel(a, b):
    return float(np.max(np.abs(np.asarray(a, np.float64) - b) / np.maximum(np.abs(b), 1e-300)))


def _merged(utts, **kw):
    m = StandardScalerMerge(D)
    for x in utts:
        m.update(*_moments(x, **kw))
    return m


def test_merge_equals_standard_scaler_partial_fit():
    utts = _utterances()
    mean, scale = _sklearn(utts)
    m = _merged(utts)
    assert _rel(m.mean, mean) <= 1e-12 and _rel(m.scale(), scale) <= 1e-12
    assert scale[0] == 1.0 and m.scale()[0] == 1.0                  # the constant channel
    assert 5e-4 < scale[1] < 2e-3                                    # the offset channel keeps its spread
    st = m.stats()
    assert st.dtype == np.float32 and st.shape == (2, D)
    # one utterance, and single-frame utterances only (each adds no spread of its own)
    for sub in (utts[:1], [u for u in utts if len(u) == 1]):
        mean, scale = _sklearn(sub)
        m = _merged(sub)
        assert _rel(m.mean, mean) <= 1e-12 and _rel(m.scale(), scale) <= 1e-12


class _Ddof1(StandardScalerMerge):
    def scale(self):
        var = self.var
        self.var = var * self.n / (self.n - 1)
        try:
            return super().scale()
        finally:
            self.var = var


class _NoConstant(StandardScalerMerge):
    def scale(self):
        return np.sqrt(self.var)


@pytest.mark.parametrize("control", ["ddof1", "fp32_accumulation", "uncentred", "no_constant_handling"])
def test_negative_controls_fail_the_same_check(control):
    """Each wrong statistic a port could plausibly compute misses sklearn by more than the 1e-12 bar the merge meets."""
    utts = _utterances()
    mean, scale = _sklearn(utts)
    if control in ("ddof1", "no_constant_handling"):
        m = (_Ddof1 if control == "ddof1" else _NoConstant)(D)
        for x in utts:
            m.update(*_moments(x))
    elif control == "fp32_accumulation":
        m = _merged(utts, acc=np.float32)
    else:
        m = _merged(utts, centred=False)
    err = max(_rel(m.mean, mean), _rel(m.scale(), scale))
    assert err > 1e-12, f"{control} passes the check (error {err:.3g})"


def _cli(*args, cwd):
    return subprocess.run([sys.executable, "-m", "audiodec_b200.codec_statistic", *args], cwd=cwd, capture_output=True, text=True,
                          env=dict(os.environ, PYTHONPATH=REPO))


def test_cli_refusals(tmp_path):
    _, enc, _ = S.make_model_zoo(str(tmp_path), "vctk_sym")
    os.makedirs(tmp_path / "corpus" / "train" / "empty")
    cfg = {"data": {"path": "corpus", "subset": {"train": "train"}}, "analyzer": os.path.relpath(enc, tmp_path), "stats": "stats/x.npy"}

    def write(c):
        with open(tmp_path / "s.yaml", "w") as f:
            yaml.safe_dump(c, f)

    write(cfg)
    r = _cli("-c", "s.yaml", "--cuda", "-1", cwd=tmp_path)
    assert r.returncode != 0 and "no CPU path" in r.stderr
    r = _cli("-c", "s.yaml", "--batch_seconds", "0", cwd=tmp_path)
    assert r.returncode != 0 and "batch_seconds" in r.stderr
    for key in ("stats", "analyzer"):
        write({k: v for k, v in cfg.items() if k != key})
        r = _cli("-c", "s.yaml", cwd=tmp_path)
        assert r.returncode != 0 and f"names no {key}" in r.stderr
    write(cfg)
    r = _cli("-c", "s.yaml", "--subset", "valid", cwd=tmp_path)
    assert r.returncode != 0 and "data.subset.valid" in r.stderr
    r = _cli("-c", "s.yaml", cwd=tmp_path)                          # a folder with no *.wav under it
    assert r.returncode != 0 and "no *.wav files" in r.stderr
    acfg = yaml.safe_load(open(os.path.join(os.path.dirname(enc), "config.yml")))
    acfg["model_type"] = "HiFiGAN"
    with open(os.path.join(os.path.dirname(enc), "config.yml"), "w") as f:
        yaml.safe_dump(acfg, f)
    r = _cli("-c", "s.yaml", cwd=tmp_path)
    assert r.returncode != 0 and "Analyzer HiFiGAN is not supported!" in r.stderr
    assert not os.path.exists(tmp_path / "stats" / "x.npy")


def test_stereo_wav_is_refused_by_name(tmp_path):
    from scipy.io import wavfile
    from audiodec_b200.codec_statistic import _read
    p = str(tmp_path / "two.wav")
    wavfile.write(p, 48000, np.zeros((100, 2), np.int16))
    with pytest.raises(SystemExit, match="two.wav has 2 channels"):
        _read(("two", p))


def write_golden_corpus(root, g):
    """The golden's corpus: its wavs from the recorded recipe, plus the files that are not *.wav."""
    paths = S.make_wav_corpus(str(root), int(g["seed"]), [int(n) for n in g["lengths"]], int(g["sr"]))
    for rel in g["extra"]:
        os.makedirs(os.path.dirname(os.path.join(root, str(rel))) or str(root), exist_ok=True)
        with open(os.path.join(root, str(rel)), "w") as f:
            f.write("not audio\n")
    return paths


def test_recipe_regenerates_the_golden_corpus(tmp_path):
    from audiodec_b200.codec_test import find_wavs
    g = np.load(GOLDEN)
    paths = write_golden_corpus(tmp_path, g)
    assert [os.path.relpath(p, tmp_path) for p in paths] == list(g["wavs"])
    assert [hashlib.sha256(open(p, "rb").read()).hexdigest() for p in paths] == list(g["sha256"])
    # the reference's discovery order (sorted recursive *.wav, the extras skipped) is find_wavs'
    assert [os.path.relpath(p, tmp_path) for _, p in find_wavs(str(tmp_path))] == list(g["files"])
    assert int(g["frames"].sum()) == g["idx"].shape[1] and g["idx"].dtype == np.uint16
