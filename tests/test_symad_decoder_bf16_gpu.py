"""The symAD decoder-only handle (ADEC_MODEL_SYMAD_DECODER, `SymADDecoderStreamGenerator`) and its bf16 modes: compute_dtype 1
(`.to(torch.bfloat16)`: bf16 conv operands, fp32 activations and I/O) and 2 (`set_activation_dtype(torch.bfloat16)`: bf16
activations, causal state and decode I/O as well).

In fp32 (compute_dtype 0) the handle runs the full symAD handle's decoder op list, so its output equals SymADStreamGenerator.decode
bit for bit in every call mode.  The bf16 bars are derived from the reference itself, as for the vocoder
(tests/golden/make_golden_symad_bf16.py dumps its fp32 and its own bf16 output for the same zq):
    max-abs vs the fp32 reference          <= 1.2 x the reference's own bf16 error
    SNR vs the fp32 reference              >= the reference's own bf16 SNR - 2 dB
    max-abs vs the reference's bf16 output <= 2.4 x the reference's own bf16 error"""
import ctypes
import functools
import os

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PARAMS = {"sym": S.SYMAD_PARAMS, "aad": S.SYMAAD_PARAMS, "c16": S.SYMAD_C16_PARAMS}
PREC_BF16 = 1
LAUNCH_TC, LAUNCH_HEAD = 0, 3


@pytest.fixture(scope="module")
def g(golden_dir):
    g = np.load(os.path.join(golden_dir, "symad_bf16.npz"))
    for model in PARAMS:                # the synthetic weights the goldens were made with
        assert str(g["digest_" + model]) == S.state_dict_digest(_sd(model)), model
    return g


@functools.lru_cache(maxsize=None)
def _sd(model):
    return S.symad_state_dict(PARAMS[model], seed=0)


def _full(model):
    from audiodec_b200.codec import SymADStreamGenerator
    d = SymADStreamGenerator(**PARAMS[model])
    d.load_state_dict(_sd(model))
    return d.eval().to(DEV)


def _dec(model, mode):
    """A decoder-only handle in compute_dtype `mode` on cuda:0 (not yet warmed)."""
    from audiodec_b200.codec import SymADDecoderStreamGenerator
    d = SymADDecoderStreamGenerator(**PARAMS[model])
    d.load_state_dict(_sd(model))
    if mode == 1:
        d = d.to(torch.bfloat16)
    elif mode == 2:
        d = d.set_activation_dtype(torch.bfloat16)
    return d.eval().to(DEV)


def _zq(g, model):
    return torch.from_numpy(g[model + "_zq"]).to(DEV)


def _warm(d, g, model):
    d.initial_decoder(torch.from_numpy(g[model + "_warm_zq"]).to(DEV))        # load_receiver's warm-up (bin/stream.py:70,76)
    return d


def _eq(a, b, what):
    torch.cuda.synchronize()
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item())


def _varlen_split(zq, frames):
    """channels-first (1, D, sum F_b) of the first sum(frames) rows of zq (1, F, D), and the per-utterance channels-first pieces"""
    c = zq[0, :sum(frames)].transpose(0, 1).unsqueeze(0).contiguous()
    return c, list(torch.split(c, frames, dim=2))


# ------------------------------------------------------------------------------------------------ fp32: one decoder path
@pytest.mark.parametrize("model", sorted(PARAMS))
def test_fp32_decoder_only_equals_full_handle(g, model):
    """compute_dtype 0: one-shot, 5-frame chunks, B = 8, offline, varlen and stream slots of the decoder-only handle equal the full
    symAD handle's decode bit for bit - the same op list, so no second fp32 decoder path exists."""
    zq = _zq(g, model)
    full, dec = _warm(_full(model), g, model), _warm(_dec(model, 0), g, model)
    assert dec._lib.adec_hop_length(dec._h) == full._lib.adec_hop_length(full._h)
    assert dec._lib.adec_frames_for(dec._h, 12345) == full._lib.adec_frames_for(full._h, 12345)
    _eq(dec.decode(zq), full.decode(zq), "one-shot")
    _eq(torch.cat([dec.decode(zq[:, i:i + 5]) for i in range(0, 20, 5)], -1),
        torch.cat([full.decode(zq[:, i:i + 5]) for i in range(0, 20, 5)], -1), "chunked")
    torch.manual_seed(8)
    zq8 = (zq + 0.3 * torch.randn(8, *zq.shape[1:], device=DEV)).contiguous()
    _eq(dec.decode(zq8), full.decode(zq8), "B = 8")
    _eq(dec.decode_offline(zq8.transpose(1, 2)), full.decode_offline(zq8.transpose(1, 2)), "offline")
    frames = [7, 17, 11]
    c, _ = _varlen_split(zq, frames)
    for a, b in zip(dec.decode_offline_varlen(c, frames), full.decode_offline_varlen(c, frames)):
        _eq(a, b, "varlen")
    for h in (dec, full):
        h.set_streams(4)
    for k, streams in enumerate(([2, 0], [1, 3, 0], [3])):
        fr = [5 + 2 * j for j in range(len(streams))]
        zs = zq8[k, :sum(fr)]
        for a, b in zip(dec.decode_streams(zs, fr, streams), full.decode_streams(zs, fr, streams)):
            _eq(a, b, f"slots call {k}")


# ------------------------------------------------------------------------------------------------ bf16 parity vs the reference
def _bar(y, y32, y16, what):
    ref_err = (y16 - y32).abs().max().item()
    ref_snr = (10 * torch.log10(y32.pow(2).mean() / (y16 - y32).pow(2).mean())).item()
    err = (y - y32).abs().max().item()
    snr = (10 * torch.log10(y32.pow(2).mean() / (y - y32).pow(2).mean())).item()
    err16 = (y - y16).abs().max().item()
    print(f"[symAD bf16] {what}: max-abs vs fp32 reference {err:.3e} (reference's own bf16 {ref_err:.3e}), SNR {snr:.1f} dB "
          f"(reference {ref_snr:.1f} dB), vs reference bf16 {err16:.3e}")
    assert err <= 1.2 * ref_err, (what, err, ref_err)
    assert snr >= ref_snr - 2.0, (what, snr, ref_snr)
    assert err16 <= 2.4 * ref_err, (what, err16, ref_err)


CASES = {"sym": ("sym", None), "sym_stream": ("sym", 5), "aad": ("aad", None), "c16": ("c16", None), "sym_forward": ("sym", "forward")}


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_bf16_parity_vs_reference(g, case, mode):
    """decode one-shot (symAD, symAAD, c16), in 5-frame chunks (symAD) and Decoder.forward (symAD, decode_offline), in both bf16
    modes, under the reference-derived bar.  Mode 1 returns fp32, mode 2 bf16."""
    model, how = CASES[case]
    d = _warm(_dec(model, mode), g, model)
    zq = _zq(g, model)
    if how is None:
        y = d.decode(zq.to(torch.bfloat16) if mode == 2 else zq)
    elif how == "forward":
        y = d.decode_offline(zq.transpose(1, 2))
    else:
        y = torch.cat([d.decode(zq[:, i:i + how]) for i in range(0, zq.shape[1], how)], -1)
    torch.cuda.synchronize()
    y32, y16 = torch.from_numpy(g[case + "_y_fp32"]), torch.from_numpy(g[case + "_y_bf16"])
    assert y.dtype == (torch.bfloat16 if mode == 2 else torch.float32) and tuple(y.shape) == tuple(y32.shape)
    _bar(y.float().cpu(), y32, y16, f"{case} mode {mode}")


# ------------------------------------------------------------------------------------------------ mode 2: row spaces agree bit for bit
def test_mode2_chunked_equals_oneshot(g):
    zq = _zq(g, "sym").to(torch.bfloat16)
    d1, d2 = _warm(_dec("sym", 2), g, "sym"), _warm(_dec("sym", 2), g, "sym")
    _eq(torch.cat([d2.decode(zq[:, i:i + 5]) for i in range(0, zq.shape[1], 5)], -1), d1.decode(zq), "chunked vs one-shot")


def test_mode2_batch_rows_are_independent_streams(g):
    torch.manual_seed(8)
    zq = (_zq(g, "sym") + 0.3 * torch.randn(8, 40, 64, device=DEV)).to(torch.bfloat16)
    y8 = _warm(_dec("sym", 2), g, "sym").decode(zq)
    d1 = _dec("sym", 2)
    for b in range(8):
        d1.reset_buffer()
        _warm(d1, g, "sym")
        _eq(y8[b:b + 1], d1.decode(zq[b:b + 1]), f"row {b}")


@pytest.mark.parametrize("model", sorted(PARAMS))
def test_mode2_varlen_equals_per_utterance_offline(g, model):
    frames = [9, 23, 1, 5]                               # 38 frames: every model's clip has that many (c16: hop 320)
    c, parts = _varlen_split(_zq(g, model), frames)
    d = _dec(model, 2)
    ys = d.decode_offline_varlen(c, frames)
    for b, p in enumerate(parts):
        _eq(ys[b], d.decode_offline(p), f"utterance {b}")


@pytest.mark.parametrize("model", sorted(PARAMS))
def test_mode2_slots_equal_b1_streams(g, model):
    """Three slot calls over subsets of 4 streams with their own chunk lengths equal B = 1 streaming decodes of each stream."""
    torch.manual_seed(5)
    zq = (_zq(g, model)[0] + 0.3 * torch.randn(4, *_zq(g, model).shape[1:], device=DEV)).to(torch.bfloat16)
    d = _warm(_dec(model, 2), g, model)
    d.set_streams(4)
    ref = [_warm(_dec(model, 2), g, model) for _ in range(4)]
    pos = [0] * 4
    for streams, fr in (([2, 0], [5, 3]), ([1, 3, 0], [4, 6, 1]), ([3, 2], [2, 7])):
        zs = torch.cat([zq[s, pos[s]:pos[s] + f] for s, f in zip(streams, fr)])
        ys = d.decode_streams(zs, fr, streams)
        for y, s, f in zip(ys, streams, fr):
            _eq(y, ref[s].decode(zq[s:s + 1, pos[s]:pos[s] + f]), f"stream {s}")
            pos[s] += f


# ------------------------------------------------------------------------------------------------ the launches
def _records(d, zq):
    from audiodec_b200 import _lib
    lib = d._lib
    lib.adec_record_launches(d._h, 1)
    d.decode(zq)
    torch.cuda.synchronize()
    n = lib.adec_launch_records(d._h, None, 0)
    rec = _lib.TEST_REC
    buf = (ctypes.c_int * (rec * n))()
    lib.adec_launch_records(d._h, buf, n)
    lib.adec_record_launches(d._h, 0)
    return [tuple(buf[rec * i:rec * i + rec]) for i in range(n)]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("model", sorted(PARAMS))
def test_every_conv_launch_runs_bf16(g, model, mode):
    """Every tensor-core launch of the bf16 decoder runs PREC_BF16: the fused residual units (C = 32, 64, 128), both launches of the
    split RU(256), the transposed convs and decoder.conv1, on bf16 storage (BST) in mode 2 and fp32 storage in mode 1; the head
    runs its bf16-storage kernel in mode 2."""
    d = _warm(_dec(model, mode), g, model)
    zq = _zq(g, model)
    recs = _records(d, zq.to(torch.bfloat16) if mode == 2 else zq)
    tc = [r for r in recs if r[0] == LAUNCH_TC]
    assert tc and all(r[4] == PREC_BF16 and r[8] == (mode == 2) for r in tc), recs
    assert [r[8] for r in recs if r[0] == LAUNCH_HEAD] == [int(mode == 2)], recs
    fused = [r for r in tc if r[2]]
    assert sorted({r[1] for r in fused}) == [32, 64, 128] and len(fused) == 9, fused
    assert all(r[3] == 1 for r in fused)                     # ELU
    assert not any(r[6] for r in tc)                         # no paired launch in bf16


def test_profile_bytes_mode2_are_half_of_mode1(g):
    rows = []
    for mode in (1, 2):
        d = _dec("sym", mode)
        zq = _zq(g, "sym")[:, :10]
        zq = zq.to(torch.bfloat16) if mode == 2 else zq
        d.decode(zq)
        d.profile(True)
        d.decode(zq)
        rows.append(d.profile_report())
        d.profile(False)
    r1, r2 = rows
    assert len(r1) == len(r2) > 0
    for (n1, _, b1), (n2, _, b2) in zip(r1, r2):
        assert n1 == n2 and b1 > 0 and b2 * 2 == b1, (n1, b1, b2)


# ------------------------------------------------------------------------------------------------ the receiver
def _encoders(model):
    from audiodec_b200.codec import SymADStreamGenerator
    out = []
    for _ in range(2):
        e = SymADStreamGenerator(**PARAMS[model])
        e.load_state_dict(_sd(model))
        out.append(e.eval().to(DEV))
    return out


def _receiver(model):
    """tx_encoder, rx_encoder and a mode-2 decoder-only decoder, warmed as load_transmitter / load_receiver warm them."""
    tx, rx = _encoders(model)
    d = _dec(model, 2)
    tx.initial_encoder(8192, DEV)
    d.initial_decoder(rx.initial_encoder(8192, DEV))
    return tx, rx, d


def test_session_server_takes_mode2_decoder():
    """SessionCodecServer with a mode-2 decoder-only decoder: float32 frames, equal bit for bit to the device path of each stream
    (B = 1 encode -> quantize -> lookup -> decode on its own warmed generators, widened to float32)."""
    from audiodec_b200.server import SessionCodecServer
    fs, steps = 1500, 3
    srv = SessionCodecServer(*_receiver("sym"), capacity=3, frame_size=fs, sample_rate=48000, max_latency=1.0, device="cuda:0")
    ids = [srv.open(), srv.open()]
    rng = np.random.default_rng(3)
    frames = (0.1 * rng.standard_normal((steps, 2, fs))).astype(np.float32)
    for k in range(steps):
        for j, s in enumerate(ids):
            srv.submit(s, frames[k, j])
        assert srv.step() == 2
    for j, s in enumerate(ids):
        tx, rx, d = _receiver("sym")
        for k in range(steps):
            out = srv.poll(s)
            assert out.dtype == np.float32 and out.shape == (fs,)
            x = torch.from_numpy(frames[k, j]).view(1, 1, fs).to(DEV)
            y = d.decode(rx.lookup(tx.quantize(tx.encode(x))))
            np.testing.assert_array_equal(out, y.float().cpu().numpy().reshape(-1))


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections(g, monkeypatch):
    from audiodec_b200 import _lib
    from audiodec_b200.codec import SymADDecoderStreamGenerator, codec_host
    lib = _lib.load()
    d0, d2 = _dec("sym", 0), _dec("sym", 2)
    s = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    buf = torch.zeros(1 << 16, device=DEV)
    p = ctypes.c_void_p(buf.data_ptr())
    ints = lambda *v: (ctypes.c_int * len(v))(*v)
    no_rvq = "decoder-only"
    for name, rc in (("encode", lib.adec_encode(d0._h, p, 1, 300, p, s)),
                     ("encode_offline", lib.adec_encode_offline(d0._h, p, 1, 300, p, s)),
                     ("encode_streams", lib.adec_encode_streams(d0._h, p, ints(300), ints(0), 1, p, s)),
                     ("quantize", lib.adec_quantize(d0._h, p, 1, 1, p, s)),
                     ("quantize_ex", lib.adec_quantize_ex(d0._h, p, 1, 1, p, None, None, s)),
                     ("quantize_forward", lib.adec_quantize_forward(d0._h, p, 1, 1, p, p, s)),
                     ("lookup", lib.adec_lookup(d0._h, p, 1, 1, p, s)),
                     ("lookup_packed", lib.adec_lookup_packed(d0._h, p, 1, 1, p, s)),
                     ("pack_indices", lib.adec_pack_indices(d0._h, p, 1, 1, p, s)),
                     ("unpack_indices", lib.adec_unpack_indices(d0._h, p, 1, 1, p, s)),
                     ("zq_moments", lib.adec_zq_moments(d0._h, p, ints(1), 1, p, p, s))):
        assert rc != 0 and no_rvq in _lib.last_error(d0._h), (name, _lib.last_error(d0._h))
    assert lib.adec_packed_frame_bytes(d0._h) == -1
    # the host path: fp32 activations only on the decoder side, a full symAD handle on the encoder side
    tx, _ = _encoders("sym")
    x = torch.zeros(1, 1, 1500).pin_memory()
    with pytest.raises(RuntimeError, match="bf16 activations"):
        codec_host(tx, d2, x)
    d1 = _dec("sym", 1)
    _, y1 = codec_host(tx, d1, x)
    _, y0 = codec_host(tx, d0, x)
    assert y1.dtype == y0.dtype == torch.float32 and y1.shape == y0.shape == (1, 1, 1500)
    assert lib.adec_codec_host(d0._h, d0._h, ctypes.c_void_p(x.data_ptr()), 1, 1500, None, p, s) != 0
    assert no_rvq in _lib.last_error(d0._h)
    # the activation dtype is fixed when the handle is created
    with pytest.raises(RuntimeError):
        d2.set_activation_dtype(torch.float32)
    # bf16 is built for the f16 engine only; fp32 runs on every engine
    for path in ("tf32", "ffma"):
        monkeypatch.setenv("ADEC_CONV_PATH", path)
        for mode in (1, 2):
            with pytest.raises(RuntimeError, match="f16 tensor-core engine"):
                _dec("sym", mode)
        _dec("sym", 0)
    monkeypatch.delenv("ADEC_CONV_PATH")
    # the full symAD handle keeps its refusal; the message names both decoder handles
    from audiodec_b200.codec import SymADStreamGenerator
    cfg = SymADStreamGenerator(**S.SYMAD_PARAMS)._cfg
    cfg.compute_dtype = 1
    h = ctypes.c_void_p()
    assert lib.adec_create(ctypes.byref(cfg), 0, ctypes.byref(h)) != 0
    assert "HiFi-GAN" in _lib.last_error(None) and "ADEC_MODEL_SYMAD_DECODER" in _lib.last_error(None)
    # decoder.* keys stay strict
    d = SymADDecoderStreamGenerator(**S.SYMAD_PARAMS)
    d.load_state_dict(dict(_sd("sym"), **{"decoder.bogus": torch.zeros(1)}))
    with pytest.raises(RuntimeError, match="unexpected key in state dict: decoder.bogus"):
        d.to(DEV)
