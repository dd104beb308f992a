"""End-to-end parity on the GPU, through the reference-facing API (audiodec_b200.codec /
audiodec_b200.utils.audiodec -> C ABI -> sm_90a kernels), against
  (1) the golden vectors dumped from the unmodified reference (tests/golden/*.npz), and
  (2) the oracle (oracle/audiodec_oracle.py) on fresh seeded inputs.
Bar (BASELINE.json north_star): code indices bit-identical, fp32 waveforms within 1e-4 max-abs."""
import os

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
WAVE_TOL = 1e-4       # north_star tolerance
Z_TOL = 2e-5


def _codec(symad_sd, dec=None):
    """tx_encoder / rx_encoder / decoder warmed like AudioDec.load_transmitter/load_receiver (bin/stream.py:56-77)."""
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    dev = torch.device("cuda:0")
    out = []
    for _ in range(2):
        g = SymADStreamGenerator(**S.SYMAD_PARAMS)
        g.load_state_dict(symad_sd)
        out.append(g.eval().to(dev))
    if dec is None:
        d = SymADStreamGenerator(**S.SYMAD_PARAMS)
        d.load_state_dict(symad_sd)
    else:
        d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
        d.load_state_dict(dec)
    d = d.eval().to(dev)
    tx, rx = out
    tx.initial_encoder(8192, dev)
    zq = rx.initial_encoder(8192, dev)
    d.initial_decoder(zq)
    return tx, rx, d, zq


def _run(tx, rx, dec, x):
    z = tx.encode(x.cuda())
    idx = tx.quantize(z)
    zq = rx.lookup(idx)
    y = dec.decode(zq)
    torch.cuda.synchronize()
    return z.cpu(), idx.cpu(), zq.cpu(), y.cpu()


def test_symad_oneshot_golden(golden_dir, symad_sd, conv_path):
    g = np.load(os.path.join(golden_dir, "symad_oneshot.npz"))
    tx, rx, dec, zq0 = _codec(symad_sd)
    assert tuple(zq0.shape) == (1, 28, 64)
    np.testing.assert_allclose(zq0.cpu().numpy(), g["warm_zq"], atol=Z_TOL)
    z, idx, zq, y = _run(tx, rx, dec, torch.from_numpy(g["x"]))
    assert idx.dtype == torch.int64 and tuple(idx.shape) == (8, 40) and tuple(y.shape) == (1, 1, 12000)
    np.testing.assert_allclose(z.numpy(), g["z"], atol=Z_TOL)
    np.testing.assert_array_equal(idx.numpy(), g["idx"])              # bit-identical code indices
    np.testing.assert_allclose(zq.numpy(), g["zq"], atol=Z_TOL)
    np.testing.assert_allclose(y.numpy(), g["y"], atol=WAVE_TOL)


def test_symad_stream_chunks_golden(golden_dir, symad_sd, conv_path):
    g = np.load(os.path.join(golden_dir, "symad_stream.npz"))
    tx, rx, dec, _ = _codec(symad_sd)
    x = torch.from_numpy(g["x"])
    n = int(g["chunk"])
    outs = [_run(tx, rx, dec, x[:, :, i:i + n]) for i in range(0, x.shape[-1], n)]
    np.testing.assert_array_equal(torch.cat([o[1] for o in outs], -1).numpy(), g["idx"])
    np.testing.assert_allclose(torch.cat([o[3] for o in outs], -1).numpy(), g["y"], atol=WAVE_TOL)


def test_symad_ragged_golden(golden_dir, symad_sd):
    g = np.load(os.path.join(golden_dir, "symad_ragged.npz"))
    tx, rx, dec, _ = _codec(symad_sd)
    z, idx, zq, y = _run(tx, rx, dec, torch.from_numpy(g["x"]))
    assert z.shape[-1] == 14 and y.shape[-1] == 4200
    np.testing.assert_array_equal(idx.numpy(), g["idx"])
    np.testing.assert_allclose(y.numpy(), g["y"], atol=WAVE_TOL)


def test_symad_batch3_golden(golden_dir, symad_sd):
    g = np.load(os.path.join(golden_dir, "symad_batch3.npz"))
    tx, rx, dec, _ = _codec(symad_sd)
    z, idx, zq, y = _run(tx, rx, dec, torch.from_numpy(g["x"]))
    assert tuple(idx.shape) == (8, 3, 20) and tuple(zq.shape) == (3, 20, 64)
    np.testing.assert_array_equal(idx.numpy(), g["idx"])
    np.testing.assert_allclose(zq.numpy(), g["zq"], atol=Z_TOL)
    np.testing.assert_allclose(y.numpy(), g["y"], atol=WAVE_TOL)


def test_v1_vocoder_golden(golden_dir, symad_sd, hifigan_sd, conv_path):
    g = np.load(os.path.join(golden_dir, "v1_oneshot.npz"))
    tx, rx, dec, _ = _codec(symad_sd, hifigan_sd)
    z, idx, zq, y = _run(tx, rx, dec, torch.from_numpy(g["x"]))
    np.testing.assert_array_equal(idx.numpy(), g["idx"])
    np.testing.assert_allclose(y.numpy(), g["y"], atol=WAVE_TOL)
    gs = np.load(os.path.join(golden_dir, "v1_stream.npz"))
    tx, rx, dec, _ = _codec(symad_sd, hifigan_sd)
    x = torch.from_numpy(gs["x"])
    ys = [_run(tx, rx, dec, x[:, :, i:i + 1500])[3] for i in range(0, x.shape[-1], 1500)]
    np.testing.assert_allclose(torch.cat(ys, -1).numpy(), gs["y"], atol=WAVE_TOL)


def test_v1_vocoder_bf16_mode(golden_dir, symad_sd, hifigan_sd):
    """BASELINE configs[2]: HiFi-GAN v1 vocoder with bf16 conv operands (`decoder.to(torch.bfloat16)`), encoder / RVQ fp32-grade.
    The reference defines no reduced-precision tolerance, so it is derived from the reference itself (tests/golden/make_golden_bf16.py):
    its own bf16 vocoder is 1.70e-2 max-abs / 36.9 dB SNR away from its fp32 output on this clip.  Bar: indices bit-identical (the
    encoder side is untouched), waveform within 2e-2 max-abs and >= 35 dB SNR of the fp32 reference - i.e. no worse than the
    reference's own bf16 path - and within 4e-2 of the reference's bf16 output."""
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    g = np.load(os.path.join(golden_dir, "v1_bf16.npz"))
    dev = torch.device("cuda:0")
    enc = []
    for _ in range(2):
        e = SymADStreamGenerator(**S.SYMAD_PARAMS)
        e.load_state_dict(symad_sd)
        enc.append(e.eval().to(dev))
    d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    d.load_state_dict(hifigan_sd)
    d = d.to(torch.bfloat16).eval().to(dev)
    tx, rx = enc
    tx.initial_encoder(8192, dev)
    d.initial_decoder(rx.initial_encoder(8192, dev))
    z, idx, zq, y = _run(tx, rx, d, torch.from_numpy(g["x"]))
    np.testing.assert_array_equal(idx.numpy(), g["idx"])
    y32, y16 = torch.from_numpy(g["y_fp32"]), torch.from_numpy(g["y_bf16"])
    err = (y - y32).abs().max().item()
    snr = (10 * torch.log10(y32.pow(2).mean() / (y - y32).pow(2).mean())).item()
    ref_err = (y16 - y32).abs().max().item()
    print(f"[parity] bf16 vocoder: max-abs vs fp32 reference {err:.3e} (reference's own bf16: {ref_err:.3e}), SNR {snr:.1f} dB, "
          f"vs reference bf16 {(y - y16).abs().max().item():.3e}")
    assert err <= 2e-2 and snr >= 35.0
    assert (y - y16).abs().max().item() <= 4e-2
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).to(torch.bfloat16)          # the encoder side has no reduced-precision mode


def test_quantize_bit_exact_vs_oracle_same_z(symad_sd):
    """Given the SAME z, the CUDA RVQ reproduces torch-CPU's decisions: compare 64x160 frames x 8 stages.  It also equals the
    C spec (oracle/rvq_oracle.c) on every one of the 81 920 decisions with no tolerance: that comparison does not rest on the
    CPU's MKL summation order, which the torch comparison below does."""
    from oracle import audiodec_oracle as O
    from oracle import rvq_spec
    tx, rx, dec, _ = _codec(symad_sd)
    torch.manual_seed(3)
    z = 0.6 * torch.randn(64, 64, 160)
    orc = O.SymADOracle(S.SYMAD_PARAMS, symad_sd)
    ridx, margins = orc.quantize(z, return_margins=True)
    idx = tx.quantize(z.cuda()).cpu()
    sidx, _ = rvq_spec.quantize(z.numpy(), torch.stack(orc.embeds).numpy())
    np.testing.assert_array_equal(idx.numpy(), sidx)
    bad = (idx != ridx)
    # a differing decision is only tolerated on a numerical tie of the reference itself
    assert bad.sum().item() == 0 or margins[bad].max().item() < 1e-6, f"{bad.sum().item()} mismatches"
    zq = rx.lookup(idx.cuda()).cpu()
    np.testing.assert_array_equal(zq.numpy(), orc.lookup(ridx).numpy() if bad.sum() == 0 else zq.numpy())


def _first_mismatch_margins(idx, ridx, margins):
    """(Nq,B,F) indices: per frame with a differing code, the reference's own relative top-2 margin at the FIRST differing stage
    (later stages of that frame quantise a different residual, so their margins say nothing)."""
    bad = (idx != ridx)
    out = []
    for b, f in zip(*torch.nonzero(bad.any(0), as_tuple=True)):
        i = int(torch.nonzero(bad[:, b, f])[0])
        out.append(float(margins[i, b, f]))
    return out


MARGIN_TOL = 1e-6     # a differing decision is only accepted on a numerical tie of the reference itself


def test_batch_vs_oracle_seeded(symad_sd, conv_path):
    """BASELINE config 2 shape at reduced size: 8 x 0.5 s through the whole path vs the oracle.  Indices must be equal; a
    differing frame is accepted only where the reference's own top-2 margin at the first differing stage is a tie (< 1e-6)."""
    from oracle import audiodec_oracle as O
    tx, rx, dec, _ = _codec(symad_sd)
    torch.manual_seed(1337)
    x = 0.1 * torch.randn(8, 1, 24000)
    z, idx, zq, y = _run(tx, rx, dec, x)
    ref = O.CodecOracle(S.SYMAD_PARAMS, symad_sd)
    rz, ridx, rzq, ry = ref.run(x)
    np.testing.assert_allclose(z.numpy(), rz.numpy(), atol=Z_TOL)
    _, _, margins = O.rvq_forward_index(rz.transpose(1, 2), ref.tx_encoder.embeds, return_margins=True)
    ties = _first_mismatch_margins(idx, ridx, margins)
    print(f"[parity] {conv_path}: {len(ties)} of {idx.shape[1] * idx.shape[2]} frames differ; reference margins there: {sorted(ties)[:8]}; "
          f"smallest margin overall {margins.min().item():.3e}; z max-abs err {(z - rz).abs().max().item():.3e}")
    assert all(m < MARGIN_TOL for m in ties), f"{len(ties)} frames differ beyond a tie: margins {sorted(ties, reverse=True)[:8]}"
    ok = ~(idx != ridx).any(0)
    err = (y - ry).abs()[:, 0].reshape(8, -1, 300)[ok].max().item()
    assert err <= WAVE_TOL, err


def test_full_size_batch_vs_oracle(symad_sd):
    """BASELINE configs[1] at FULL size (64 x 48000, the benchmarked batch, seed 1337): utterances 0, 21, 42 and 63 of the batch
    against the oracle run on those rows (demoFile.py:58-61 per utterance): indices equal, waveform within 1e-4."""
    from oracle import audiodec_oracle as O
    tx, rx, dec, _ = _codec(symad_sd)
    torch.manual_seed(1337)
    x = 0.1 * torch.randn(64, 1, 48000)
    z, idx, zq, y = _run(tx, rx, dec, x)
    sel = [0, 21, 42, 63]
    ref = O.CodecOracle(S.SYMAD_PARAMS, symad_sd)
    rz, ridx, rzq, ry = ref.run(x[sel])
    _, _, margins = O.rvq_forward_index(rz.transpose(1, 2), ref.tx_encoder.embeds, return_margins=True)
    ties = _first_mismatch_margins(idx[:, sel], ridx, margins)
    print(f"[parity] full size: {len(ties)} of {len(sel) * idx.shape[2]} frames differ; margins {sorted(ties)[:8]}; "
          f"z max-abs err {(z[sel] - rz).abs().max().item():.3e}")
    assert all(m < MARGIN_TOL for m in ties), f"frames differ beyond a tie: margins {sorted(ties, reverse=True)[:8]}"
    ok = ~(idx[:, sel] != ridx).any(0)
    err = (y[sel] - ry).abs()[:, 0].reshape(len(sel), -1, 300)[ok].max().item()
    print(f"[parity] full size: waveform max-abs err {err:.3e}")
    assert err <= WAVE_TOL, err


def test_batch_rows_are_independent_streams(symad_sd):
    """batch-vs-single invariance (SURVEY section 4 (iii)): row b of a batched call == that utterance alone."""
    torch.manual_seed(5)
    x = 0.1 * torch.randn(4, 1, 6000)
    tx, rx, dec, _ = _codec(symad_sd)
    z, idx, zq, y = _run(tx, rx, dec, x)
    for b in (0, 3):
        t1, r1, d1, _ = _codec(symad_sd)
        z1, idx1, zq1, y1 = _run(t1, r1, d1, x[b:b + 1])
        assert torch.equal(idx[:, b], idx1)
        assert torch.equal(y[b], y1[0])


def test_size_independent_properties_full_size(symad_sd):
    """BASELINE config 2 full size (64 x 48000): properties that need no oracle run -
    chunked == one-shot (indices and waveform bit for bit), lookup(quantize(.)) consistent, output finite."""
    tx, rx, dec, _ = _codec(symad_sd)
    torch.manual_seed(1337)
    x = 0.1 * torch.randn(64, 1, 48000)
    z, idx, zq, y = _run(tx, rx, dec, x)
    assert tuple(idx.shape) == (8, 64, 160) and tuple(y.shape) == (64, 1, 48000)
    assert torch.isfinite(y).all() and idx.min() >= 0 and idx.max() < 8192
    for i in range(8):
        assert idx[i].min() >= 1024 * i and idx[i].max() < 1024 * (i + 1)
    tx2, rx2, dec2, _ = _codec(symad_sd)
    parts = [_run(tx2, rx2, dec2, x[:, :, i:i + 12000]) for i in range(0, 48000, 12000)]
    assert torch.equal(torch.cat([p[1] for p in parts], -1), idx)
    assert torch.equal(torch.cat([p[3] for p in parts], -1), y)


def test_no_cpu_fallback(symad_sd):
    from audiodec_b200.codec import SymADStreamGenerator
    g = SymADStreamGenerator(**S.SYMAD_PARAMS)
    g.load_state_dict(symad_sd)
    with pytest.raises(RuntimeError):
        g.to("cpu")
    with pytest.raises(RuntimeError):
        g.encode(torch.zeros(1, 1, 300))


def test_codec_host_path_matches_device_path(golden_dir, symad_sd):
    """adec_codec_host (host buffers: H2D + four calls + D2H) == the four calls on device tensors == golden."""
    from audiodec_b200.codec import codec_host
    g = np.load(os.path.join(golden_dir, "symad_batch3.npz"))
    tx, rx, dec, _ = _codec(symad_sd)
    idx_h, y_h = codec_host(tx, dec, torch.from_numpy(g["x"]).pin_memory())
    assert tuple(idx_h.shape) == (8, 3, 20) and not idx_h.is_cuda and not y_h.is_cuda
    np.testing.assert_array_equal(idx_h.numpy(), g["idx"])
    np.testing.assert_allclose(y_h.numpy(), g["y"], atol=WAVE_TOL)


VARIANTS = {   # golden file -> (encoder params, vocoder params or None)
    "v2_oneshot.npz": ("SYMAD_PARAMS", "HIFIGAN_V2_PARAMS"),
    "v0_oneshot.npz": ("SYMAD_PARAMS", "HIFIGAN_V0_PARAMS"),
    "aad_oneshot.npz": ("SYMAAD_PARAMS", None),
    "c16_oneshot.npz": ("SYMAD_C16_PARAMS", None),
}


def _variant_codec(ep, esd, vp, vsd):
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    dev = torch.device("cuda:0")
    objs = []
    for _ in range(3):
        g = SymADStreamGenerator(**ep)
        g.load_state_dict(esd)
        objs.append(g)
    tx, rx, dec = objs
    if vp is not None:
        dec = HiFiGANStreamGenerator(**vp)
        dec.load_state_dict(vsd)
    tx, rx, dec = tx.eval().to(dev), rx.eval().to(dev), dec.eval().to(dev)
    tx.initial_encoder(8192, dev)
    dec.initial_decoder(rx.initial_encoder(8192, dev))
    return tx, rx, dec


@pytest.mark.parametrize("fname", sorted(VARIANTS))
def test_released_variants_golden(golden_dir, fname):
    """The rest of the assign_model table (utils/audiodec.py:109-179): HiFi-GAN v2 / v0, symAAD, 16-codebook hop-320."""
    g = np.load(os.path.join(golden_dir, fname))
    ep, vp = (getattr(S, n) if n else None for n in VARIANTS[fname])
    esd = S.symad_state_dict(ep, seed=0)
    vsd = S.hifigan_state_dict(vp, seed=1) if vp else None
    x = torch.from_numpy(g["x"])
    tx, rx, dec = _variant_codec(ep, esd, vp, vsd)
    z, idx, zq, y = _run(tx, rx, dec, x)
    assert tuple(idx.shape) == tuple(g["idx"].shape) and tuple(y.shape) == tuple(g["y"].shape)
    np.testing.assert_array_equal(idx.numpy(), g["idx"])
    np.testing.assert_allclose(y.numpy(), g["y"], atol=WAVE_TOL)
    tx, rx, dec = _variant_codec(ep, esd, vp, vsd)
    outs = [_run(tx, rx, dec, x[:, :, i:i + 3200]) for i in (0, 3200)]
    np.testing.assert_array_equal(torch.cat([o[1] for o in outs], -1).numpy(), g["idx_chunks"])
    np.testing.assert_allclose(torch.cat([o[3] for o in outs], -1).numpy(), g["y_chunks"], atol=WAVE_TOL)


def test_index_bitstream_matches_oracle_and_round_trips(symad_sd):
    """SURVEY 8(f) rank 2: Nq x 10-bit packed frames.  The pack kernel reproduces the numpy oracle's bytes, unpack inverts it
    bit-exactly on indices the quantiser really emits (ragged B x F), and the decoded audio is unchanged by the round trip."""
    from oracle import bitstream_oracle as BO
    tx, rx, dec, _ = _codec(symad_sd)
    torch.manual_seed(11)
    z = 0.6 * torch.randn(3, 64, 37)
    idx = tx.quantize(z.cuda())                                    # (8,3,37)
    assert tx.packed_frame_bytes() == BO.frame_bytes(8, 1024) == 10
    packed = tx.pack(idx)
    assert packed.dtype == torch.uint8 and tuple(packed.shape) == (3, 37, 10)
    np.testing.assert_array_equal(packed.cpu().numpy(), BO.pack_indices(idx.cpu().numpy(), 1024))
    back = rx.unpack(packed)
    assert back.dtype == torch.int64
    np.testing.assert_array_equal(back.cpu().numpy(), idx.cpu().numpy())
    np.testing.assert_array_equal(rx.lookup(back).cpu().numpy(), rx.lookup(idx).cpu().numpy())
    assert not tx.index_error() and not rx.index_error()
    # B == 1 keeps the reference's 2-D (Nq,F) shape on both sides
    idx1 = tx.quantize(z[:1].cuda())
    p1 = tx.pack(idx1)
    assert tuple(idx1.shape) == (8, 37) and tuple(p1.shape) == (37, 10)
    np.testing.assert_array_equal(rx.unpack(p1).cpu().numpy(), idx1.cpu().numpy())
    # extremes: all-zero and all-max local indices
    for v in (0, 1023):
        e = (torch.full((8, 2, 5), v, dtype=torch.int64) + 1024 * torch.arange(8).view(8, 1, 1)).cuda()
        pe = tx.pack(e)
        np.testing.assert_array_equal(pe.cpu().numpy(), BO.pack_indices(e.cpu().numpy(), 1024))
        np.testing.assert_array_equal(rx.unpack(pe).cpu().numpy(), e.cpu().numpy())
    # an index outside its stage's range is flagged (the reference's F.embedding would raise), then the flag clears
    bad = idx.clone()
    bad[3, 1, 2] = 5 * 1024 + 7                                     # stage-3 row holding a stage-5 index
    tx.pack(bad)
    assert tx.index_error() and not tx.index_error()
    bad[3, 1, 2] = 8 * 1024 + 1
    rx.lookup(bad)
    assert rx.index_error() and not rx.index_error()


@pytest.mark.parametrize("B,F", [(3, 37), (1, 5), (64, 160), (256, 5)])
def test_fused_quantize_pack_lookup_is_bit_identical(symad_sd, B, F):
    """SURVEY 8(f) rank 2: the RVQ kernel's fused outputs (indices, packed frames, zq) equal quantize -> pack -> lookup, and
    lookup_packed equals lookup(unpack(.)), bit for bit - over ragged, single-stream, benchmark-size and 256-stream shapes (each
    picks a different frames-per-pass / passes-per-block launch)."""
    tx, rx, dec, _ = _codec(symad_sd)
    torch.manual_seed(100 + B)
    z = (0.6 * torch.randn(B, 64, F)).cuda()
    idx = tx.quantize(z)
    packed = tx.pack(idx)
    zq = rx.lookup(idx)
    fi, fp, fz = tx.quantize_fused(z, want_idx=True, want_packed=True, want_zq=True)
    assert torch.equal(fi, idx) and torch.equal(fp, packed) and torch.equal(fz, zq)
    assert torch.equal(rx.lookup_packed(packed), zq)
    only = tx.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)
    assert only[0] is None and only[2] is None and torch.equal(only[1], packed)
    assert not tx.index_error() and not rx.index_error()
    bad = packed.clone().reshape(-1, packed.shape[-1])
    bad[0, 0] = 0xFF; bad[0, 1] = 0xFF                              # 10-bit code 1023 is valid; force stage 1 out of range is impossible
    rx.lookup_packed(bad.reshape(packed.shape))                     # (every 10-bit value < 1024): the flag must stay clear
    assert not rx.index_error()


def test_index_bitstream_16_codebooks():
    """symAD_c16 (16 codebooks, hop 320): 16 x 10 bit = 20 bytes / frame = 24 kbit/s at 48 kHz."""
    from audiodec_b200.codec import SymADStreamGenerator
    from oracle import bitstream_oracle as BO
    g = SymADStreamGenerator(**S.SYMAD_C16_PARAMS)
    g.load_state_dict(S.symad_state_dict(S.SYMAD_C16_PARAMS, seed=0))
    g = g.eval().to(torch.device("cuda:0"))
    rng = np.random.default_rng(5)
    idx = rng.integers(0, 1024, (16, 2, 9)) + 1024 * np.arange(16)[:, None, None]
    p = g.pack(torch.from_numpy(idx).cuda())
    assert tuple(p.shape) == (2, 9, 20)
    np.testing.assert_array_equal(p.cpu().numpy(), BO.pack_indices(idx, 1024))
    np.testing.assert_array_equal(g.unpack(p).cpu().numpy(), idx)


OFFLINE = {   # golden file -> (encoder params, vocoder params or None)
    "offline_symad.npz": ("SYMAD_PARAMS", None), "offline_aad.npz": ("SYMAAD_PARAMS", None),
    "offline_c16.npz": ("SYMAD_C16_PARAMS", None), "offline_v1.npz": ("SYMAD_PARAMS", "HIFIGAN_V1_PARAMS"),
    "offline_v0.npz": ("SYMAD_PARAMS", "HIFIGAN_V0_PARAMS"),
}


@pytest.mark.parametrize("fname", sorted(OFFLINE))
def test_offline_forward_golden(golden_dir, fname, conv_path):
    """SURVEY 8(f) rank 4: the non-streaming batch forward (codecTest.py:78-95) against vectors dumped from the reference's base
    Generator classes: zero left-pad on every causal conv, first-frame replication on every transposed conv."""
    from audiodec_b200.codec import HiFiGANStreamGenerator, OfflineCodec, SymADStreamGenerator
    g = np.load(os.path.join(golden_dir, fname))
    ep, vp = (getattr(S, n) if n else None for n in OFFLINE[fname])
    dev = torch.device("cuda:0")
    enc = SymADStreamGenerator(**ep)
    enc.load_state_dict(S.symad_state_dict(ep, seed=0))
    enc = enc.eval().to(dev)
    if vp is None:
        dec = SymADStreamGenerator(**ep)
        dec.load_state_dict(S.symad_state_dict(ep, seed=0))
    else:
        dec = HiFiGANStreamGenerator(**vp)
        dec.load_state_dict(S.hifigan_state_dict(vp, seed=1))
    dec = dec.eval().to(dev)
    x = torch.from_numpy(g["x"]).cuda()
    # a streaming call first: the offline forward must not depend on whatever state the handle holds
    enc.initial_encoder(8192, dev)
    z = enc.encode_offline(x)
    zq, idx = enc.quantize_offline(z)
    y = dec.forward(zq) if vp is not None else dec.decode_offline(zq)
    torch.cuda.synchronize()
    assert tuple(z.shape) == tuple(g["z"].shape) and tuple(zq.shape) == tuple(g["zq"].shape) and tuple(y.shape) == tuple(g["y"].shape)
    np.testing.assert_allclose(z.cpu().numpy(), g["z"], atol=Z_TOL)
    np.testing.assert_allclose(zq.cpu().numpy(), g["zq"], atol=5e-6)        # sum of codewords vs sum of x+(e-x) roundings
    np.testing.assert_allclose(y.cpu().numpy(), g["y"], atol=WAVE_TOL)
    # same through the codecTest.py-shaped wrapper ((T,C) audio in), and a different batch size on the same handles
    oc = OfflineCodec(enc, dec)
    audio = g["x"][:, 0, :].T                                              # (T, C=B)
    y2 = oc.decode(oc.encode(audio))
    np.testing.assert_array_equal(y2.cpu().numpy(), y.cpu().numpy())
    y1 = oc.decode(oc.encode(audio[:, :1]))
    np.testing.assert_allclose(y1.cpu().numpy(), g["y"][:1], atol=WAVE_TOL)
    y3 = oc.decode(oc.encode(np.concatenate([audio, audio[:, :1]], axis=1)))
    np.testing.assert_allclose(y3.cpu().numpy()[-1], g["y"][0], atol=WAVE_TOL)


def test_multi_stream_server_matches_per_stream_oracle(symad_sd):
    """SURVEY 8(f) rank 3: three lock-stepped streams through the batched server (indices over the packed wire format) equal
    three independent reference-style streams, including a stream that under-runs one step (it is fed silence)."""
    from audiodec_b200.server import MultiStreamCodecServer
    from oracle import audiodec_oracle as O
    tx, rx, dec, _ = _codec(symad_sd)
    n, fs, steps = 3, 1500, 3
    srv = MultiStreamCodecServer(tx, rx, dec, n_streams=n, frame_size=fs, sample_rate=48000, max_latency=1.0,
                                 device="cuda:0", wire=True)
    torch.manual_seed(5)
    frames = 0.1 * torch.randn(steps, n, fs)
    skip = (1, 2)                                                  # stream 2 has nothing queued at step 1
    for k in range(steps):
        for s in range(n):
            if (k, s) != skip:
                srv.submit(s, frames[k, s].numpy())
        assert srv.step() == (n - 1 if k == skip[0] else n)
    for s in range(n):
        orc = O.CodecOracle(S.SYMAD_PARAMS, symad_sd)
        for k in range(steps):
            x = torch.zeros(1, 1, fs) if (k, s) == skip else frames[k, s].view(1, 1, fs)
            y = orc.run(x)[-1]
            if (k, s) == skip:
                continue
            out = srv.poll(s)
            assert out is not None and out.shape == (fs,)
            np.testing.assert_allclose(out, y.numpy().reshape(-1)[:fs], atol=WAVE_TOL)
        assert srv.poll(s) is None
    st = srv.statistics()
    assert st["frames"] == steps * n - 1 and st["underruns"] == 1 and st["frame_drops"] == 0
    assert st["wire_kbps_per_stream"] == pytest.approx(12.8)       # 8 x 10 bit per 300-sample frame at 48 kHz
    assert not tx.index_error() and not rx.index_error()
