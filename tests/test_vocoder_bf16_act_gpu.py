"""The HiFi-GAN vocoder with bf16 activations (compute_dtype 2, `set_activation_dtype(torch.bfloat16)`): bf16 operands with fp32
accumulation as in the bf16-operand mode, and every activation, the causal state and decode's zq / y stored as bf16 - the data
layout and dtype contract of the reference's `decoder.to(torch.bfloat16)`.

The reference defines no reduced-precision tolerance, so each case's bar is derived from the reference itself
(tests/golden/make_golden_bf16_act.py dumps its fp32 and its own bf16 output for the same zq):
    max-abs vs the fp32 reference        <= 1.2 x the reference's own bf16 error
    SNR vs the fp32 reference            >= the reference's own bf16 SNR - 2 dB
    max-abs vs the reference's bf16 output <= 2.4 x the reference's own bf16 error
For v1 one-shot (1.70e-2, 36.9 dB) that is the 2e-2 / 35 dB / 4e-2 bar of the bf16-operand mode."""
import ctypes
import os

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(os.path.join(golden_dir, "bf16_act.npz"))


def _decoder(params, act_bf16=True, operand_bf16=False):
    """A HiFi-GAN decoder on cuda:0 (not yet warmed)."""
    from audiodec_b200.codec import HiFiGANStreamGenerator
    d = HiFiGANStreamGenerator(**params)
    d.load_state_dict(S.hifigan_state_dict(params, seed=1))
    if operand_bf16:
        d = d.to(torch.bfloat16)
    if act_bf16:
        d = d.set_activation_dtype(torch.bfloat16)
    return d.eval().to(DEV)


def _warm(d, g):
    d.initial_decoder(torch.from_numpy(g["warm_zq"]).to(DEV))       # fp32 zq: cast to bf16 on the device (load_receiver's warm-up)
    return d


def _bar(y, y32, y16, what):
    """Assert the reference-derived bar (module docstring); y, y32, y16 float32 CPU tensors of one shape."""
    ref_err = (y16 - y32).abs().max().item()
    ref_snr = (10 * torch.log10(y32.pow(2).mean() / (y16 - y32).pow(2).mean())).item()
    err = (y - y32).abs().max().item()
    snr = (10 * torch.log10(y32.pow(2).mean() / (y - y32).pow(2).mean())).item()
    err16 = (y - y16).abs().max().item()
    print(f"[bf16 act] {what}: max-abs vs fp32 reference {err:.3e} (reference's own bf16 {ref_err:.3e}), SNR {snr:.1f} dB "
          f"(reference {ref_snr:.1f} dB), vs reference bf16 {err16:.3e}")
    assert err <= 1.2 * ref_err, (what, err, ref_err)
    assert snr >= ref_snr - 2.0, (what, snr, ref_snr)
    assert err16 <= 2.4 * ref_err, (what, err16, ref_err)


CASES = {"v1": ("HIFIGAN_V1_PARAMS", None), "v1_stream": ("HIFIGAN_V1_PARAMS", 5), "v0": ("HIFIGAN_V0_PARAMS", None),
         "v2": ("HIFIGAN_V2_PARAMS", None)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_stream_decode_parity_vs_reference(g, case):
    """StreamGenerator.decode one-shot (v1, v0, v2) and in 5-frame chunks (v1): bf16 zq in (one-shot) or fp32 zq cast on the device
    (chunks), bf16 y out, under the reference-derived bar."""
    params, chunk = CASES[case]
    d = _warm(_decoder(getattr(S, params)), g)
    zq = torch.from_numpy(g["zq"]).to(DEV)
    if chunk is None:
        y = d.decode(zq.to(torch.bfloat16))
    else:
        y = torch.cat([d.decode(zq[:, i:i + chunk]) for i in range(0, zq.shape[1], chunk)], -1)
    torch.cuda.synchronize()
    y32, y16 = torch.from_numpy(g[case + "_y_fp32"]), torch.from_numpy(g[case + "_y_bf16"])
    assert y.dtype == torch.bfloat16 and tuple(y.shape) == tuple(y32.shape)
    _bar(y.float().cpu(), y32, y16, case)


def test_forward_parity_vs_reference(g):
    """Generator.forward (the non-streaming path: zero left-pad, first-frame replication in the transposed convs), channels-first
    zq in bf16 or fp32, bf16 y out; the call does not depend on the streaming state the handle held."""
    d = _warm(_decoder(S.HIFIGAN_V1_PARAMS), g)
    c = torch.from_numpy(g["zq"]).to(DEV).transpose(1, 2)
    y = d.forward(c.to(torch.bfloat16))
    y_f = d(c)
    torch.cuda.synchronize()
    y32, y16 = torch.from_numpy(g["v1_forward_y_fp32"]), torch.from_numpy(g["v1_forward_y_bf16"])
    assert y.dtype == torch.bfloat16 and tuple(y.shape) == tuple(y32.shape)
    assert torch.equal(y, y_f)
    _bar(y.float().cpu(), y32, y16, "v1_forward")


def test_chunked_equals_oneshot_bitwise(g):
    """The causal state holds the same bf16 post-activation rows that a one-shot window reads, and every kernel rounds the same
    fp32 value for a given output row wherever the row falls in a tile, so 8 chunks of 5 frames equal one 40-frame call bit for bit."""
    zq = torch.from_numpy(g["zq"]).to(DEV).to(torch.bfloat16)
    d1 = _warm(_decoder(S.HIFIGAN_V1_PARAMS), g)
    d2 = _warm(_decoder(S.HIFIGAN_V1_PARAMS), g)
    y1 = d1.decode(zq)
    y2 = torch.cat([d2.decode(zq[:, i:i + 5]) for i in range(0, zq.shape[1], 5)], -1)
    torch.cuda.synchronize()
    assert torch.equal(y1, y2), (y1.float() - y2.float()).abs().max().item()


def test_batch_rows_are_independent_streams(g):
    """B = 8 in one call (the first layers stack the 8 streams' rows into shared tiles) equals 8 calls of B = 1, bit for bit."""
    torch.manual_seed(8)
    zq = (torch.from_numpy(g["zq"]) + 0.3 * torch.randn(8, 40, 64)).to(DEV).to(torch.bfloat16)
    d8 = _warm(_decoder(S.HIFIGAN_V1_PARAMS), g)
    y8 = d8.decode(zq)
    d1 = _decoder(S.HIFIGAN_V1_PARAMS)
    for b in range(8):
        d1.reset_buffer()
        _warm(d1, g)
        y1 = d1.decode(zq[b:b + 1])
        assert torch.equal(y8[b:b + 1], y1), (b, (y8[b:b + 1].float() - y1.float()).abs().max().item())


def _server(act_bf16, n, fs, sr):
    from audiodec_b200.codec import SymADStreamGenerator
    from audiodec_b200.server import MultiStreamCodecServer
    sd = S.symad_state_dict(seed=0)
    enc = []
    for _ in range(2):
        e = SymADStreamGenerator(**S.SYMAD_PARAMS)
        e.load_state_dict(sd)
        enc.append(e.eval().to(DEV))
    tx, rx = enc
    d = _decoder(S.HIFIGAN_V1_PARAMS, act_bf16=act_bf16)
    tx.initial_encoder(8192, DEV)                                  # bin/stream.py:61,70,76
    d.initial_decoder(rx.initial_encoder(8192, DEV))
    return MultiStreamCodecServer(tx, rx, d, n_streams=n, frame_size=fs, sample_rate=sr, max_latency=1.0, device="cuda:0")


def test_configs3_server_shape(g):
    """BASELINE configs[3]: libritts v1 (24 kHz), 256 streams x 3 chunks of 1500 samples through MultiStreamCodecServer with a
    bf16-activation decoder.  Frames come out float32; rows 0 / 85 / 170 / 255 against the same server with an fp32 decoder, under
    the v1 bar relative to fp32."""
    n, fs, sr, steps = 256, 1500, 24000, 3
    srv16, srv32 = _server(True, n, fs, sr), _server(False, n, fs, sr)
    rng = np.random.default_rng(3)
    frames = (0.1 * rng.standard_normal((steps, n, fs))).astype(np.float32)
    for k in range(steps):
        for srv in (srv16, srv32):
            for s in range(n):
                srv.submit(s, frames[k, s])
            assert srv.step() == n
    v1_32, v1_16 = torch.from_numpy(g["v1_y_fp32"]), torch.from_numpy(g["v1_y_bf16"])
    ref_err = (v1_16 - v1_32).abs().max().item()
    ref_snr = (10 * torch.log10(v1_32.pow(2).mean() / (v1_16 - v1_32).pow(2).mean())).item()
    for s in (0, 85, 170, 255):
        out16 = [srv16.poll(s) for _ in range(steps)]
        out32 = [srv32.poll(s) for _ in range(steps)]
        assert all(o.dtype == np.float32 and o.shape == (fs,) for o in out16)
        y, y32 = torch.from_numpy(np.concatenate(out16)), torch.from_numpy(np.concatenate(out32))
        err = (y - y32).abs().max().item()
        snr = (10 * torch.log10(y32.pow(2).mean() / (y - y32).pow(2).mean())).item()
        print(f"[bf16 act] server row {s}: max-abs vs fp32 server {err:.3e}, SNR {snr:.1f} dB")
        assert err <= 1.2 * ref_err and snr >= ref_snr - 2.0, (s, err, snr)


def test_profile_bytes_are_half_of_the_operand_mode():
    """Algorithmic bytes of every vocoder launch (profile_report) with bf16 activations are half those of the bf16-operand mode on
    the same shape: 2 bytes per stored activation element instead of 4."""
    rows = []
    for act in (False, True):
        d = _decoder(S.HIFIGAN_V1_PARAMS, act_bf16=act, operand_bf16=True)
        zq = torch.randn(2, 10, 64, device=DEV)
        d.decode(zq)
        d.profile(True)
        d.decode(zq)
        rows.append(d.profile_report())
        d.profile(False)
    r1, r2 = rows
    assert len(r1) == len(r2) > 0
    for (n1, _, b1), (n2, _, b2) in zip(r1, r2):
        assert n1 == n2 and b1 > 0 and b2 * 2 == b1, (n1, b1, b2)


def test_rejections(g, symad_sd, monkeypatch):
    from audiodec_b200 import _lib
    from audiodec_b200.codec import SymADStreamGenerator, codec_host
    lib = _lib.load()
    d2 = _decoder(S.HIFIGAN_V1_PARAMS)
    d1 = _decoder(S.HIFIGAN_V1_PARAMS, act_bf16=False, operand_bf16=True)
    s = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    zq32 = torch.zeros(1, 5, 64, device=DEV)
    y32 = torch.empty(1, 1, 1500, device=DEV)
    zq16 = torch.zeros(1, 5, 64, device=DEV, dtype=torch.bfloat16)
    y16 = torch.empty(1, 1, 1500, device=DEV, dtype=torch.bfloat16)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)
    # fp32 entry points on a bf16-activation handle name the bf16 ones, and the reverse
    for fn, want in (("adec_decode", "adec_decode_bf16"), ("adec_decode_offline", "adec_decode_offline_bf16")):
        assert getattr(lib, fn)(d2._h, p(zq32), 1, 5, p(y32), s) != 0
        assert want in _lib.last_error(d2._h)
    for fn, want in (("adec_decode_bf16", "adec_decode"), ("adec_decode_offline_bf16", "adec_decode_offline")):
        assert getattr(lib, fn)(d1._h, p(zq16), 1, 5, p(y16), s) != 0
        assert want in _lib.last_error(d1._h) and "fp32" in _lib.last_error(d1._h)
    # external bf16 pointers must be 16-byte aligned
    zq_big = torch.zeros(1, 6, 64, device=DEV, dtype=torch.bfloat16)
    assert lib.adec_decode_bf16(d2._h, p(zq_big, 2), 1, 5, p(y16), s) != 0 and "16-byte aligned" in _lib.last_error(d2._h)
    y_big = torch.empty(1, 1, 1508, device=DEV, dtype=torch.bfloat16)
    assert lib.adec_decode_bf16(d2._h, p(zq16), 1, 5, p(y_big, 4), s) != 0 and "16-byte aligned" in _lib.last_error(d2._h)
    # through Python an offset view of zq is realigned, not rejected
    flat = torch.zeros(5 * 64 + 1, device=DEV, dtype=torch.bfloat16)
    assert flat[1:].data_ptr() % 16 == 2
    y_view = d2.decode(flat[1:].view(1, 5, 64))
    torch.cuda.synchronize()
    assert y_view.dtype == torch.bfloat16 and tuple(y_view.shape) == (1, 1, 1500)
    # the host path carries fp32 only
    tx = SymADStreamGenerator(**S.SYMAD_PARAMS)
    tx.load_state_dict(symad_sd)
    tx = tx.eval().to(DEV)
    with pytest.raises(RuntimeError, match="bf16 activations"):
        codec_host(tx, d2, torch.zeros(1, 1, 1500).pin_memory())
    # the activation dtype is fixed when the handle is created
    with pytest.raises(RuntimeError):
        d2.set_activation_dtype(torch.float32)
    with pytest.raises(RuntimeError):
        d1.set_activation_dtype(torch.bfloat16)
    # compute_dtype 2 is built for HiFi-GAN handles on the f16 engine only
    cfg = SymADStreamGenerator(**S.SYMAD_PARAMS)._cfg
    cfg.compute_dtype = 2
    h = ctypes.c_void_p()
    assert lib.adec_create(ctypes.byref(cfg), 0, ctypes.byref(h)) != 0 and "HiFi-GAN" in _lib.last_error(None)
    cfg.compute_dtype = 3
    assert lib.adec_create(ctypes.byref(cfg), 0, ctypes.byref(h)) != 0 and "compute_dtype" in _lib.last_error(None)
    for path in ("tf32", "ffma"):
        monkeypatch.setenv("ADEC_CONV_PATH", path)
        with pytest.raises(RuntimeError, match="f16 tensor-core engine"):
            _decoder(S.HIFIGAN_V1_PARAMS)
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).set_activation_dtype(torch.bfloat16)
