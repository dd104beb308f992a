"""The non-streaming codec over utterances of different lengths in one launch sequence (adec_encode_offline_varlen,
adec_decode_offline_varlen[_bf16]): each utterance must come out exactly as a uniform offline call of its own length gives it."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WAVE_TOL, Z_TOL = 1e-4, 2e-5


def _enc(params=S.SYMAD_PARAMS):
    from audiodec_b200.codec import SymADStreamGenerator
    g = SymADStreamGenerator(**params)
    g.load_state_dict(S.symad_state_dict(params, seed=0))
    return g.eval().to(DEV)


def _voc(params=S.HIFIGAN_V1_PARAMS, mode=0):
    from audiodec_b200.codec import HiFiGANStreamGenerator
    d = HiFiGANStreamGenerator(**params)
    d.load_state_dict(S.hifigan_state_dict(params, seed=1))
    if mode >= 1:
        d = d.to(torch.bfloat16)
    if mode == 2:
        d = d.set_activation_dtype(torch.bfloat16)
    return d.eval().to(DEV)


def _dec_varlen(dec, zq, frames):
    from audiodec_b200.codec import HiFiGANStreamGenerator
    return dec.forward_varlen(zq, frames) if isinstance(dec, HiFiGANStreamGenerator) else dec.decode_offline_varlen(zq, frames)


def _dec_uniform(dec, zq):
    from audiodec_b200.codec import HiFiGANStreamGenerator
    return dec.forward(zq) if isinstance(dec, HiFiGANStreamGenerator) else dec.decode_offline(zq)


def _bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


# ------------------------------------------------------------------ 1. pinned to the reference's golden vectors
OFFLINE = {"offline_symad.npz": ("SYMAD_PARAMS", None), "offline_aad.npz": ("SYMAAD_PARAMS", None),
           "offline_c16.npz": ("SYMAD_C16_PARAMS", None), "offline_v1.npz": ("SYMAD_PARAMS", "HIFIGAN_V1_PARAMS"),
           "offline_v0.npz": ("SYMAD_PARAMS", "HIFIGAN_V0_PARAMS")}


@pytest.mark.parametrize("engine", ["f16", "tf32"])
@pytest.mark.parametrize("fname", sorted(OFFLINE))
def test_prefixes_match_the_reference(golden_dir, fname, engine, monkeypatch):
    """Prefixes of the golden utterances, mixed across rows, in one varlen batch: the reference forward is causal, so every output
    is a prefix of the golden output (indices bit-identical to a uniform call, z / y within the suite's tolerances)."""
    monkeypatch.setenv("ADEC_CONV_PATH", engine)
    g = np.load(os.path.join(golden_dir, fname))
    ep, vp = (getattr(S, n) if n else None for n in OFFLINE[fname])
    enc = _enc(ep)
    dec = _voc(vp) if vp else _enc(ep)
    hop = dec._lib.adec_hop_length(dec._h)
    B, T = g["x"].shape[0], g["x"].shape[2]
    cuts = [n for n in (1, 299, 300, 301, 1799, T) if n <= T]
    utts = [(i % B, n) for i, n in enumerate(cuts + cuts[::-1])]          # rows interleaved, short and long mixed
    x = torch.from_numpy(g["x"]).to(DEV)
    z, frames = enc.encode_offline_varlen([x[b, 0, :n] for b, n in utts])
    zq, idx = enc.quantize_offline(z)
    ys = _dec_varlen(dec, zq, frames)
    _, ref_idx = enc.quantize_offline(enc.encode_offline(x))
    torch.cuda.synchronize()
    o = 0
    for (b, n), f, y in zip(utts, frames, ys):
        assert f == enc._lib.adec_frames_for(enc._h, n)
        np.testing.assert_allclose(z[0, :, o:o + f].cpu().numpy(), g["z"][b, :, :f], atol=Z_TOL)
        np.testing.assert_allclose(zq[0, :, o:o + f].cpu().numpy(), g["zq"][b, :, :f], atol=5e-6)
        assert torch.equal(idx[:, 0, o:o + f].cpu(), ref_idx[:, b, :f].cpu()), (fname, b, n)
        assert tuple(y.shape) == (1, 1, f * hop)
        np.testing.assert_allclose(y[0, 0].cpu().numpy(), g["y"][b, 0, :f * hop], atol=WAVE_TOL)
        o += f


# ------------------------------------------------------------------ 2. bit-exact against per-utterance uniform calls at real sizes
def _lengths(n=64, seed=5):
    """300 .. 12 x 48000 samples, log-spaced with jitter: most are shorter than one 128-row tile of the deep layers."""
    r = np.random.default_rng(seed)
    base = np.exp(np.linspace(np.log(300), np.log(12 * 48000), n))
    lens = np.clip((base * r.uniform(0.8, 1.2, n)).astype(int), 300, 12 * 48000)
    lens[0], lens[-1] = 300, 12 * 48000
    return [int(v) for v in r.permutation(lens)]


@pytest.fixture(scope="module")
def corpus():
    torch.manual_seed(11)
    return [0.1 * torch.randn(n, device=DEV) for n in _lengths()]


@pytest.fixture(scope="module")
def symad_varlen(corpus):
    enc = _enc()
    z, frames = enc.encode_offline_varlen(corpus)
    zq, idx = enc.quantize_offline(z)
    return enc, z, frames, zq, idx


def test_encoder_and_rvq_bit_exact_vs_uniform(corpus, symad_varlen):
    enc, z, frames, zq, idx = symad_varlen
    o = 0
    for x, f in zip(corpus, frames):
        z1 = enc.encode_offline(x.view(1, 1, -1))
        zq1, idx1 = enc.quantize_offline(z1)
        assert z1.shape[2] == f
        assert torch.equal(_bits(z[:, :, o:o + f]), _bits(z1))
        assert torch.equal(idx[:, 0, o:o + f].cpu(), idx1[:, 0].cpu())
        assert torch.equal(_bits(zq[:, :, o:o + f]), _bits(zq1))
        o += f


@pytest.mark.parametrize("dec_kind", ["symad", "v1_mode0", "v1_mode1", "v1_mode2"])
def test_decoder_bit_exact_vs_uniform(symad_varlen, dec_kind):
    _, _, frames, zq, _ = symad_varlen
    dec = _enc() if dec_kind == "symad" else _voc(mode=int(dec_kind[-1]))
    ys = _dec_varlen(dec, zq, frames)
    assert all(y.untyped_storage().data_ptr() == ys[0].untyped_storage().data_ptr() for y in ys)   # views of one buffer
    o = 0
    for f, y in zip(frames, ys):
        y1 = _dec_uniform(dec, zq[:, :, o:o + f])
        assert y.dtype == y1.dtype and y.shape == y1.shape
        assert torch.equal(_bits(y), _bits(y1)), (dec_kind, f)
        o += f


# ------------------------------------------------------------------ 3. invariances
def test_permutation_and_batch_of_one(corpus, symad_varlen):
    enc, z, frames, _, _ = symad_varlen
    perm = np.random.default_rng(3).permutation(len(corpus))
    zp, fp = enc.encode_offline_varlen([corpus[i] for i in perm])
    offs = np.concatenate([[0], np.cumsum(frames)])
    assert fp == [frames[i] for i in perm]
    o = 0
    for i, f in zip(perm, fp):
        assert torch.equal(_bits(zp[:, :, o:o + f]), _bits(z[:, :, offs[i]:offs[i] + f]))
        o += f
    dec = _voc()
    zq, _ = enc.quantize_offline(z)
    ys = dec.forward_varlen(zq, frames)
    zqp = torch.cat([zq[:, :, offs[i]:offs[i] + frames[i]] for i in perm], dim=2)
    for i, y in zip(perm, dec.forward_varlen(zqp, fp)):
        assert torch.equal(_bits(y), _bits(ys[i]))
    x = corpus[7]
    z1, f1 = enc.encode_offline_varlen([x])
    assert torch.equal(_bits(z1), _bits(enc.encode_offline(x.view(1, 1, -1)))) and f1 == [z1.shape[2]]
    zq1, _ = enc.quantize_offline(z1)
    assert torch.equal(_bits(dec.forward_varlen(zq1, f1)[0]), _bits(dec.forward(zq1)))


# ------------------------------------------------------------------ 4. accounting
def test_launches_and_profiled_bytes():
    enc, dec = _enc(), _voc()
    torch.manual_seed(2)
    xs = [0.1 * torch.randn(n, device=DEV) for n in (300, 1799, 9000, 48000, 301)]
    n0 = enc.launch_count
    enc.encode_offline(xs[0].view(1, 1, -1))
    per_call = enc.launch_count - n0
    for k in (1, 2, 5):
        n0 = enc.launch_count
        enc.encode_offline_varlen(xs[:k])
        assert enc.launch_count - n0 == per_call, k
    z, frames = enc.encode_offline_varlen(xs)
    zq, _ = enc.quantize_offline(z)
    n0 = dec.launch_count
    dec.forward(zq[:, :, :frames[0]])
    per_call = dec.launch_count - n0
    n0 = dec.launch_count
    dec.forward_varlen(zq, frames)
    assert dec.launch_count - n0 == per_call

    def report(g, fn):
        g.profile(True)
        fn()
        rows = g.profile_report()
        g.profile(False)
        return rows
    for g, run_vl, run_one, parts in (
            (enc, lambda: enc.encode_offline_varlen(xs), lambda x: enc.encode_offline(x.view(1, 1, -1)), xs),
            (dec, lambda: dec.forward_varlen(zq, frames), lambda c: dec.forward(c),
             list(torch.split(zq, frames, dim=2)))):
        vl = report(g, run_vl)
        ones = [report(g, lambda p=p: run_one(p)) for p in parts]
        assert [r[0] for r in vl] == [r[0] for r in ones[0]]
        for i, (name, _, nbytes) in enumerate(vl):
            assert nbytes == sum(o[i][2] for o in ones), name


# ------------------------------------------------------------------ 5. rejections
def test_rejections(monkeypatch):
    from audiodec_b200 import _lib
    lib = _lib.load()
    enc, voc, voc2 = _enc(), _voc(), _voc(mode=2)
    s = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    buf = torch.zeros(1 << 16, device=DEV)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)
    ints = lambda *v: (ctypes.c_int * max(1, len(v)))(*v)

    def fails(h, rc, *words):
        assert rc != 0
        msg = _lib.last_error(h)
        assert all(w in msg for w in words), msg
    fails(enc._h, lib.adec_encode_offline_varlen(enc._h, p(buf), ints(300), 0, p(buf), s), "encode_offline_varlen", "B must be >= 1")
    fails(enc._h, lib.adec_encode_offline_varlen(enc._h, p(buf), ints(300, 0), 2, p(buf), s), "utterance 1", ">= 1")
    fails(enc._h, lib.adec_encode_offline_varlen(enc._h, p(buf), ints(-5), 1, p(buf), s), "utterance 0", ">= 1")
    fails(enc._h, lib.adec_encode_offline_varlen(enc._h, p(buf), ints(1 << 30, 1 << 30), 2, p(buf), s), "32-bit row indexing")
    fails(voc._h, lib.adec_encode_offline_varlen(voc._h, p(buf), ints(300), 1, p(buf), s), "not a symAD handle")
    fails(voc._h, lib.adec_decode_offline_varlen(voc._h, p(buf), ints(5), 0, p(buf), s), "decode_offline_varlen", "B must be >= 1")
    fails(voc._h, lib.adec_decode_offline_varlen(voc._h, p(buf), ints(5, 0), 2, p(buf), s), "utterance 1")
    fails(voc._h, lib.adec_decode_offline_varlen(voc._h, p(buf), ints(1 << 24), 1, p(buf), s), "32-bit row indexing")
    # compute_dtype 2: the bf16 entry point, named in the message of the other one, and 16-byte aligned buffers
    fails(voc2._h, lib.adec_decode_offline_varlen(voc2._h, p(buf), ints(5), 1, p(buf), s), "adec_decode_offline_varlen_bf16")
    fails(voc._h, lib.adec_decode_offline_varlen_bf16(voc._h, p(buf), ints(5), 1, p(buf), s), "adec_decode_offline_varlen", "fp32")
    fails(voc2._h, lib.adec_decode_offline_varlen_bf16(voc2._h, p(buf, 2), ints(5), 1, p(buf), s), "16-byte aligned")
    fails(voc2._h, lib.adec_decode_offline_varlen_bf16(voc2._h, p(buf), ints(5), 1, p(buf, 4), s), "16-byte aligned")
    # the FFMA engine has no varlen kernels
    monkeypatch.setenv("ADEC_CONV_PATH", "ffma")
    e0 = _enc()
    fails(e0._h, lib.adec_encode_offline_varlen(e0._h, p(buf), ints(300), 1, p(buf), s), "FFMA", "tf32")
    with pytest.raises(RuntimeError, match="FFMA"):
        e0.encode_offline_varlen([buf[:300]])


# ------------------------------------------------------------------ 6. Python API and the batched codecTest.py
def _audio(seed, n, c):
    return (0.1 * np.random.default_rng(seed).standard_normal((n, c))).astype(np.float32)


def test_offline_codec_many_equals_per_file():
    from audiodec_b200.codec import OfflineCodec
    for dec in (_voc(), _enc()):
        oc = OfflineCodec(_enc(), dec)
        audios = [_audio(1, 4801, 2), _audio(2, 300, 1), _audio(3, 20000, 3), _audio(4, 1, 1)]
        zqs = oc.encode_many(audios)
        ys = oc.decode_many(zqs)
        for a, zq, y in zip(audios, zqs, ys):
            zq1 = oc.encode(a)
            y1 = oc.decode(zq1)
            assert zq.shape == zq1.shape and torch.equal(_bits(zq), _bits(zq1))
            assert y.shape == y1.shape and torch.equal(_bits(y), _bits(y1))


def test_codec_test_cli_matches_per_file_calls(tmp_path):
    from audiodec_b200.codec import HiFiGANStreamGenerator, OfflineCodec, SymADStreamGenerator
    from audiodec_b200.wavio import read_wav, write_wav_pcm16
    sr, enc_ckpt, dec_ckpt = S.make_model_zoo(str(tmp_path / "zoo"), "vctk_v1")
    wav_dir = tmp_path / "corpus" / "test"
    wav_dir.mkdir(parents=True)
    for i, n in enumerate((48000 + 17, 3001, 150000)):
        write_wav_pcm16(str(wav_dir / f"utt{i}.wav"), _audio(10 + i, n, 1), sr)
    cfg_path = os.path.join(os.path.dirname(enc_ckpt), "config.yml")
    cfg = yaml.safe_load(open(cfg_path))
    cfg["data"] = {"path": str(tmp_path / "corpus"), "subset": {"clean_test": "test"}}
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    out = tmp_path / "out"
    r = subprocess.run([sys.executable, "-m", "audiodec_b200.codec_test", "--encoder", enc_ckpt, "--decoder", dec_ckpt,
                        "--output_dir", str(out), "--batch_seconds", "2"], cwd=REPO, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "RTF" in r.stdout
    enc = SymADStreamGenerator(**S.SYMAD_PARAMS)
    enc.load_state_dict(torch.load(enc_ckpt)["model"]["generator"])
    dec = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    dec.load_state_dict(torch.load(dec_ckpt)["model"]["generator"])
    oc = OfflineCodec(enc.eval().to(DEV), dec.eval().to(DEV))
    outdir = out / "symAD_vctk_48000_hop300-AudioDec_v1_symAD_vctk_48000_hop300_clean_200000-500000" / "test"
    for i in range(3):
        audio, _ = read_wav(str(wav_dir / f"utt{i}.wav"))
        y = oc.decode(oc.encode(audio)).squeeze(1).transpose(1, 0).cpu().numpy()
        ref = tmp_path / f"ref{i}.wav"
        write_wav_pcm16(str(ref), y, sr)
        assert (outdir / f"utt{i}_output.wav").read_bytes() == ref.read_bytes(), i
