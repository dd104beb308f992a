"""The corpus-statistics path on the GPU: quantize_forward bit for bit against the C spec's ResidualVQ.forward sum, the moment kernel
against a numpy fp64 two-pass and against itself at other places in a batch, and the batched codecStatistic.py CLI against the
statistics and indices the unmodified reference computed (tests/golden/make_golden_stats.py)."""
import os

import numpy as np
import pytest
import torch
import yaml

from audiodec_b200 import synthetic as S
from oracle import rvq_cases as C
from oracle import rvq_spec as R

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "stats_vctk.npz")
SHAPES = [(1, 1), (3, 37), (96, 33), (64, 160)]
FULL = 8192
SEG = 256                       # MOM_SEG in csrc/kernels.cuh: rows per segment of the moment kernel
DEV = torch.device("cuda:0")


def _generator(params, sd):
    from audiodec_b200.codec import SymADStreamGenerator
    g = SymADStreamGenerator(**params)
    g.load_state_dict(sd)
    return g.eval().to(DEV)


def _compared(nfr):
    if nfr <= FULL:
        return np.arange(nfr)
    return np.unique(np.concatenate([np.arange(512), np.arange(512, nfr - 512, 37), np.arange(nfr - 512, nfr)]))


def _bits_equal(got, want, what):
    bad = np.argwhere(got.view(np.int32) != want.view(np.int32))
    assert len(bad) == 0, f"{what}: {len(bad)} differ, first at {bad[:4].tolist()}: got {got[tuple(bad[:4].T)]}, want {want[tuple(bad[:4].T)]}"


@pytest.mark.parametrize("name", sorted(C.all_cases()))
def test_quantize_forward_equals_the_spec(name):
    """zq = the spec's qsum and idx = the spec's indices, bit for bit, on the tie-making inputs (g: the r + (e - r) rounding, e:
    subnormals) and shapes whose blocks straddle utterances."""
    c = C.all_cases()[name]()
    g = _generator(c.params, c.state_dict())
    nq, D, _ = c.embeds.shape
    need = np.unique(np.concatenate([_compared(b * f) for b, f in SHAPES]))     # frame k of every shape is frames[k]
    spec_idx, spec_q, _ = R.rvq_frames(c.frames[need], c.embeds)
    for B, F in SHAPES:
        nfr = B * F
        sel = _compared(nfr)
        at = np.searchsorted(need, sel)
        zq, idx = g.quantize_forward(torch.from_numpy(c.z(B, F)).to(DEV))
        assert zq.shape == (B, D, F) and idx.shape == (nq, B, F)
        got_q = zq.transpose(1, 2).reshape(nfr, D).cpu().numpy()[sel]
        _bits_equal(got_q, spec_q[at], f"{name} {B}x{F} zq")
        assert np.array_equal(idx.reshape(nq, nfr).cpu().numpy()[:, sel], spec_idx[:, at]), f"{name} {B}x{F} indices"
        assert torch.equal(idx, g.quantize(torch.from_numpy(c.z(B, F)).to(DEV)).reshape(nq, B, F))


def test_forward_sum_turns_negative_zero_positive():
    """Channel 0 of every codeword and of z is -0: lookup's codeword sum stays -0, the forward sum starts from 0. and is +0 (as
    the spec's 0.f + qq and ResidualVQ.forward's Python 0. make it)."""
    params = S.SYMAD_PARAMS
    sd = S.symad_state_dict(params, seed=0)
    nq = params["codebook_num"]
    for i in range(nq):
        e = sd[f"quantizer.codebook.layers.{i}.embed"]
        e[0] = -0.0
        sd[f"quantizer.codebook.layers.{i}.embed_avg"] = e.clone()
    embeds = np.stack([sd[f"quantizer.codebook.layers.{i}.embed"].numpy() for i in range(nq)])
    z = np.random.default_rng(3).standard_normal((2, 64, 45)).astype(np.float32) * 0.5
    z[:, 0] = -0.0
    g = _generator(params, sd)
    zq, idx = g.quantize_forward(torch.from_numpy(z).to(DEV))
    want_idx, want_q, _ = R.rvq_frames(z.transpose(0, 2, 1).reshape(-1, 64), embeds)
    got = zq.transpose(1, 2).reshape(-1, 64).cpu().numpy()
    _bits_equal(got, want_q, "forward sum")
    assert np.array_equal(idx.reshape(nq, -1).cpu().numpy(), want_idx)
    assert np.all(got[:, 0].view(np.int32) == 0)                                  # +0
    _, _, lz = g.quantize_fused(torch.from_numpy(z).to(DEV), True, False, True)
    assert np.all(lz.reshape(-1, 64).cpu().numpy()[:, 0].view(np.uint32) == 0x80000000)   # lookup's sum: -0


def _ref_moments(x):
    x = x.astype(np.float64)
    n = x.shape[0]
    s = x.sum(0)
    d = x - s / n
    return s, (d * d).sum(0) - d.sum(0) ** 2 / n, np.abs(x).sum(0), (d * d).sum(0)


def _zq_rows(frames, seed):
    """float32 (sum F, 64): channel 0 constant, channel 1 mean 1e3 / std 1e-3, the rest Gaussian around per-channel means."""
    rng = np.random.default_rng(seed)
    x = (rng.normal(0, 0.5, 64) + rng.standard_normal((sum(frames), 64))).astype(np.float32)
    x[:, 0] = np.float32(0.3)
    x[:, 1] = (1e3 + 1e-3 * rng.standard_normal(len(x))).astype(np.float32)
    return x


@pytest.fixture(scope="module")
def symad():
    return _generator(S.SYMAD_PARAMS, S.symad_state_dict(seed=0))


def test_moments_equal_numpy_two_pass(symad):
    frames = [1, 2, SEG - 1, SEG, SEG + 1, 70001] + [1] * 300
    x = _zq_rows(frames, 0)
    s, m2 = symad.zq_moments(torch.from_numpy(x).to(DEV), frames)
    s, m2 = s.cpu().numpy(), m2.cpu().numpy()
    eps = np.finfo(np.float64).eps
    at = 0
    for b, n in enumerate(frames):
        rs, rm2, abs_sum, sq = _ref_moments(x[at:at + n])
        at += n
        assert np.all(np.abs(s[b] - rs) <= 1e-13 * abs_sum), f"utterance {b} ({n} frames): sum"
        # m2 relative to sum (x - T)^2, with sklearn's constant-feature floor (n |mean| eps)^2 for the constant channel
        floor = (n * np.abs(rs / n) * eps) ** 2
        assert np.all(np.abs(m2[b] - rm2) <= 1e-13 * sq + floor), f"utterance {b} ({n} frames): m2 {np.abs(m2[b] - rm2).max()}"
    assert np.all(m2[frames.index(1)] == 0.0)


def test_moments_do_not_depend_on_the_batch(symad):
    """Each utterance's (sum, m2) bit for bit: alone, and at two other offsets inside a batch."""
    utt_frames = [1, 2, SEG - 1, SEG, SEG + 1, 3000]
    utts = [_zq_rows([n], 10 + i) for i, n in enumerate(utt_frames)]
    fill_a, fill_b = [37, 1, 5], [1] * 300 + [SEG + 3]
    xa, xb = _zq_rows(fill_a, 1), _zq_rows(fill_b, 2)

    def run(parts, frames):
        s, m2 = symad.zq_moments(torch.from_numpy(np.concatenate(parts)).to(DEV), frames)
        return s.cpu().numpy(), m2.cpu().numpy()

    for u, n in zip(utts, utt_frames):
        s0, m0 = run([u], [n])
        s1, m1 = run([xa, u, xb], fill_a + [n] + fill_b)
        s2, m2 = run([xb, xa, u], fill_b + fill_a + [n])
        k1, k2 = len(fill_a), len(fill_b) + len(fill_a)
        for s, m, k in ((s1, m1, k1), (s2, m2, k2)):
            assert np.array_equal(s[k].view(np.int64), s0[0].view(np.int64)), f"{n} frames: sum moved"
            assert np.array_equal(m[k].view(np.int64), m0[0].view(np.int64)), f"{n} frames: m2 moved"


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """The golden's corpus, analyzer and config regenerated in a scratch directory (the CLI's paths are relative to it)."""
    from test_codec_statistic_cpu import write_golden_corpus
    g = np.load(GOLDEN)
    root = tmp_path_factory.mktemp("stats")
    S.make_model_zoo(str(root), "vctk_sym", seed=0)
    cfg = yaml.safe_load(str(g["config"]))
    write_golden_corpus(root / cfg["data"]["path"] / cfg["data"]["subset"]["train"], g)
    with open(root / "statistic.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    return root, cfg, g


def _run_cli(root, cfg, *args, on_batch=None, stats=None):
    from audiodec_b200 import codec_statistic
    cwd = os.getcwd()
    os.chdir(root)
    try:
        if stats:
            c = dict(cfg, stats=stats)
            with open("statistic_alt.yaml", "w") as f:
                yaml.safe_dump(c, f)
        codec_statistic.main(["-c", "statistic_alt.yaml" if stats else "statistic.yaml", *args], on_batch=on_batch)
    finally:
        os.chdir(cwd)
    return np.load(os.path.join(root, stats or cfg["stats"]))


def _close(got, want):
    assert got.dtype == np.float32 and got.shape == (2, 64)
    assert np.abs(got[0] - want[0]).max() <= 2e-6, f"mean max-abs {np.abs(got[0] - want[0]).max():.3g}"
    assert (np.abs(got[1] - want[1]) / want[1]).max() <= 2e-6, f"scale rel {(np.abs(got[1] - want[1]) / want[1]).max():.3g}"


def test_cli_matches_the_reference(corpus):
    root, cfg, g = corpus
    seen = []

    def on_batch(utt_ids, frames, idx):
        seen.append(idx.cpu().numpy())

    stats = _run_cli(root, cfg, on_batch=on_batch)
    _close(stats, g["stats_full"])
    idx = np.concatenate(seen, axis=1)
    nq = idx.shape[0]
    local = idx - 1024 * np.arange(nq)[:, None]
    assert local.shape == g["idx"].shape and np.array_equal(local, g["idx"].astype(np.int64))
    _close(_run_cli(root, cfg, "--subset_num", "7", stats="stats/sub7.npy"), g["stats_sub7"])

    # the file is what register_stats reads, and its rows, as a vocoder's mean / scale, decode
    from audiodec_b200.codec import HiFiGANStreamGenerator
    sd = S.hifigan_state_dict(seed=1)
    sd["mean"], sd["scale"] = torch.from_numpy(stats[0].copy()), torch.from_numpy(stats[1].copy())
    voc = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    voc.load_state_dict(sd)
    voc = voc.eval().to(DEV)
    enc = _generator(S.SYMAD_PARAMS, S.symad_state_dict(seed=0))
    torch.manual_seed(5)
    zq, _ = enc.quantize_forward(enc.encode_offline(0.1 * torch.randn(1, 1, 9600, device=DEV)))
    y = voc.forward(zq)
    assert y.shape == (1, 1, 9600) and torch.isfinite(y).all() and y.abs().max() < 1


def test_cli_output_does_not_depend_on_batch_seconds(corpus):
    root, cfg, _ = corpus
    _run_cli(root, cfg, "--batch_seconds", "1", stats="stats/b1.npy")
    _run_cli(root, cfg, "--batch_seconds", "600", stats="stats/b600.npy")
    a, b = (open(os.path.join(root, "stats", f), "rb").read() for f in ("b1.npy", "b600.npy"))
    assert a == b
