"""The symAD encoder-only handle (ADEC_MODEL_SYMAD_ENCODER, `SymADEncoderStreamGenerator`) and its bf16 modes: compute_dtype 1
(`.to(torch.bfloat16)`: the encoder's and the projector's convs on bf16 operands, fp32 x, activations, state and z) and 2
(`set_activation_dtype(torch.bfloat16)`: x, every activation, the causal state and z in bf16 as well).  The stem keeps fp32 weights
in both; the RVQ runs unchanged on z (widened exactly from bf16 in mode 2).

In fp32 (compute_dtype 0) the handle runs the full symAD handle's encoder op list and RVQ, so z, indices, packed bytes and state equal
SymADStreamGenerator's bit for bit in every call mode.  The bf16 bars are derived from the reference itself
(tests/golden/make_golden_tx_bf16.py dumps its fp32 and its own bf16 transmitter output for the same clip), e_ref = the reference's
own bf16 z error:
    z max-abs vs the fp32 reference          <= 1.2 e_ref
    z SNR vs the fp32 reference              >= the reference's own bf16 SNR - 2 dB
    z max-abs vs the reference's bf16 z      <= 2.4 e_ref
and the indices (a) are the C spec applied to the returned z, bit for bit (packed bytes: the bitstream oracle's), (b) equal the fp32
reference's on every frame whose decisions no perturbation as large as the frame's z error can change, and (c) give at least the
reference's bf16 share of frames whose indices all equal fp32's."""
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
CASES = {"sym": "sym", "sym_stream": "sym", "aad": "aad", "c16": "c16", "sym_forward": "sym"}
PREC_BF16, PREC_F16 = 1, 3
LAUNCH_TC, LAUNCH_STEM = 0, 2


@pytest.fixture(scope="module")
def g(golden_dir):
    g = np.load(os.path.join(golden_dir, "tx_bf16.npz"))
    for model in PARAMS:                # the synthetic weights the goldens were made with
        assert str(g["digest_" + model]) == S.state_dict_digest(_sd(model)), model
    return g


@functools.lru_cache(maxsize=None)
def _sd(model):
    return S.symad_state_dict(PARAMS[model], seed=0)


def _full(model):
    from audiodec_b200.codec import SymADStreamGenerator
    t = SymADStreamGenerator(**PARAMS[model])
    t.load_state_dict(_sd(model))
    return t.eval().to(DEV)


def _enc(model, mode, warm=8192):
    """An encoder-only handle in compute_dtype `mode` on cuda:0, warmed as load_transmitter warms it (warm = None: not warmed)."""
    from audiodec_b200.codec import SymADEncoderStreamGenerator
    t = SymADEncoderStreamGenerator(**PARAMS[model])
    t.load_state_dict(_sd(model))
    if mode == 1:
        t = t.to(torch.bfloat16)
    elif mode == 2:
        t = t.set_activation_dtype(torch.bfloat16)
    t = t.eval().to(DEV)
    if warm:
        t.initial_encoder(warm, DEV)
    return t


def _embeds(model):
    sd = _sd(model)
    return [sd[f"quantizer.codebook.layers.{i}.embed"].numpy() for i in range(PARAMS[model]["codebook_num"])]


def _eq(a, b, what):
    torch.cuda.synchronize()
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item() if a.is_floating_point() else "indices")


def _chunked(t, x, chunk):
    zs, ids = [], []
    for i in range(0, x.shape[-1], chunk):
        z = t.encode(x[..., i:i + chunk])
        zs.append(z)
        ids.append(t.quantize(z))
    return torch.cat(zs, -1), torch.cat(ids, -1)


# ------------------------------------------------------------------------------------------------ fp32: one transmitter path
@pytest.mark.parametrize("model", sorted(PARAMS))
def test_fp32_encoder_only_equals_full_handle(g, model):
    """compute_dtype 0: one-shot, chunked, B = 8 stacked rows, offline, varlen and stream slots of the encoder-only handle give the
    full symAD handle's z, indices and packed bytes bit for bit, and the same causal state (the encoder's part of the full layout)."""
    x = torch.from_numpy(g["x"]).to(DEV)
    full, enc = _full(model), _enc(model, 0, warm=None)
    for t in (full, enc):
        t.initial_encoder(8192, DEV)
    hop = enc._lib.adec_hop_length(enc._h)
    assert hop == full._lib.adec_hop_length(full._h) and enc.packed_frame_bytes() == full.packed_frame_bytes()
    assert enc._lib.adec_frames_for(enc._h, 12345) == full._lib.adec_frames_for(full._h, 12345)
    n_enc = len(enc.state_layout)
    assert enc.state_layout == full.state_layout[:n_enc] and all(k.startswith(("encoder.", "projector.")) for k, _, _ in enc.state_layout)
    z = enc.encode(x)
    _eq(z, full.encode(x), "one-shot z")
    _eq(enc.quantize(z), full.quantize(z), "indices")
    _eq(enc.quantize_fused(z, want_idx=True, want_packed=True, want_zq=False)[1], full.quantize_fused(z, True, True, False)[1], "packed")
    _eq(enc.pack(enc.quantize(z)), full.pack(full.quantize(z)), "pack")
    for a, b in zip(_chunked(enc, x, 5 * hop), _chunked(full, x, 5 * hop)):
        _eq(a, b, "chunked")
    _eq(enc.stream_state(0), full.stream_state(0)[:, :enc.stream_state(0).shape[1]], "state")
    torch.manual_seed(8)
    x8 = 0.1 * torch.randn(8, 1, 5 * hop, device=DEV)
    _eq(enc.encode(x8), full.encode(x8), "B = 8")
    _eq(enc.encode_offline(x8), full.encode_offline(x8), "offline")
    xs = [x[0, 0, :7001], x[0, 0, 100:3100], x[0, 0, :1]]
    _eq(enc.encode_offline_varlen(xs)[0], full.encode_offline_varlen(xs)[0], "varlen")
    for t in (enc, full):
        t.set_streams(4)
    for k, streams in enumerate(([2, 0], [1, 3, 0], [3])):
        chunks = [x8[k + j, 0, :hop * (2 + j)] for j in range(len(streams))]
        _eq(enc.encode_streams(chunks, streams)[0], full.encode_streams(chunks, streams)[0], f"slots call {k}")


# ------------------------------------------------------------------------------------------------ bf16 parity vs the reference
def _decidable(z64, embeds, delta):
    """frames whose fp64 RVQ decisions no perturbation of L2 norm <= delta[f] can change (test_encoder_amplitude_sweep's rule, per
    frame)"""
    r = z64.T.copy()
    ok = np.ones(r.shape[0], bool)
    for e in embeds:
        e = e.astype(np.float64)
        dist = (r ** 2).sum(1, keepdims=True) - 2 * r @ e + (e ** 2).sum(0, keepdims=True)
        o = np.argsort(dist, 1)[:, :2]
        rows = np.arange(r.shape[0])
        ok &= dist[rows, o[:, 1]] - dist[rows, o[:, 0]] > 2 * delta * np.linalg.norm(e[:, o[:, 0]] - e[:, o[:, 1]], axis=0)
        r = r - e[:, o[:, 0]].T
    return ok


def _tx_case(t, g, case):
    x = torch.from_numpy(g["x"]).to(DEV)
    if case == "sym_forward":
        z = t.encode_offline(x)
        return z, t.quantize(z)
    if case == "sym_stream":
        return _chunked(t, x, int(g["chunk_frames"]) * t._lib.adec_hop_length(t._h))
    z = t.encode(x)
    return z, t.quantize(z)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_bf16_against_reference(g, case, mode):
    """compute_dtype 1 and 2 against the reference's fp32 and bf16 transmitters on the same clip: the z bars, and indices (a) - (c)."""
    from oracle import bitstream_oracle, rvq_spec
    model = CASES[case]
    t = _enc(model, mode, warm=int(g["warm_len"]))
    z, idx = _tx_case(t, g, case)
    z32, z16 = (torch.from_numpy(g[f"{case}_z_{d}"]).double() for d in ("fp32", "bf16"))
    i32, i16 = g[f"{case}_idx_fp32"], g[f"{case}_idx_bf16"]
    zk = z.double().cpu()
    ref_err = (z16 - z32).abs().max().item()
    ref_snr = (10 * torch.log10(z32.pow(2).mean() / (z16 - z32).pow(2).mean())).item()
    err = (zk - z32).abs().max().item()
    snr = (10 * torch.log10(z32.pow(2).mean() / (zk - z32).pow(2).mean())).item()
    err16 = (zk - z16).abs().max().item()
    ik = idx.cpu().numpy()
    frames_eq = (ik == i32).all(0).mean()
    ref_frames_eq = (i16 == i32).all(0).mean()
    delta = np.linalg.norm((zk - z32)[0].numpy(), axis=0)
    ok = _decidable(z32[0].numpy(), _embeds(model), delta)
    assert z.dtype == (torch.bfloat16 if mode == 2 else torch.float32)
    print(f"[symAD tx bf16] {case} mode {mode}: z max-abs vs fp32 reference {err:.3e} (reference's own bf16 {ref_err:.3e}), SNR {snr:.1f} dB "
          f"(reference {ref_snr:.1f} dB), vs reference bf16 {err16:.3e}; frames with all indices equal to fp32 {frames_eq:.3f} "
          f"(reference bf16 {ref_frames_eq:.3f}); decidable frames {ok.sum()}/{ok.size}")
    assert err <= 1.2 * ref_err, (case, err, ref_err)
    assert snr >= ref_snr - 2.0, (case, snr, ref_snr)
    assert err16 <= 2.4 * ref_err, (case, err16, ref_err)
    # (a) the spec on the returned z, and the bitstream
    spec, _ = rvq_spec.quantize(z.float().cpu().numpy(), np.stack(_embeds(model)))
    np.testing.assert_array_equal(ik, spec[:, 0])
    _, packed, _ = t.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)
    np.testing.assert_array_equal(packed.cpu().numpy(), bitstream_oracle.pack_indices(spec, PARAMS[model]["codebook_size"])[0])
    # (b) decidable frames, (c) the share of whole frames
    np.testing.assert_array_equal(ik[:, ok], i32[:, ok])
    assert frames_eq >= ref_frames_eq, (case, frames_eq, ref_frames_eq)


@pytest.mark.parametrize("mode", [1, 2])
def test_bf16_launches_and_row_spaces(g, mode):
    """compute_dtype 1 / 2: every conv launch is PREC_BF16, unpaired, with bf16 storage exactly in mode 2, and so is the stem; chunked
    equals one call, B stacked rows equal B single-stream handles, varlen equals per-utterance offline, slot calls equal B = 1
    streams, and an exported state continues bit for bit in another handle."""
    from audiodec_b200 import _lib
    x = torch.from_numpy(g["x"]).to(DEV)
    t = _enc("sym", mode)
    hop = t._lib.adec_hop_length(t._h)
    rec = np.zeros(256 * _lib.TEST_REC, np.int32)
    assert t._lib.adec_record_launches(t._h, 1) == 0
    z1 = t.encode(x[..., :40 * hop])
    n = t._lib.adec_launch_records(t._h, rec.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), 256)
    assert t._lib.adec_record_launches(t._h, 0) == 0
    recs = [tuple(r) for r in rec.reshape(-1, _lib.TEST_REC)[:n]]
    bst = mode == 2
    assert recs[0][0] == LAUNCH_STEM and recs[0][8] == bst, recs
    assert all(r[0] == LAUNCH_TC and r[4] == PREC_BF16 and not r[6] and r[8] == bst for r in recs[1:]), recs
    assert z1.dtype == (torch.bfloat16 if bst else torch.float32)
    t2 = _enc("sym", mode)
    _eq(_chunked(t2, x[..., :40 * hop], 5 * hop)[0], z1, "chunked vs one call")
    torch.manual_seed(3)
    x4 = 0.1 * torch.randn(4, 1, 6 * hop, device=DEV)
    t4 = _enc("sym", mode)
    z4 = t4.encode(x4)
    for b in range(4):
        _eq(_enc("sym", mode).encode(x4[b:b + 1]), z4[b:b + 1], f"stacked row {b}")
    xs = [x[0, 0, :7001], x4[1, 0], x[0, 0, :1]]
    zv, frames = t.encode_offline_varlen(xs)
    for xu, zu in zip(xs, torch.split(zv, frames, dim=2)):
        _eq(t.encode_offline(xu.view(1, 1, -1)), zu.contiguous(), "varlen vs offline")
    s = _enc("sym", mode)
    s.set_streams(4)
    singles = [_enc("sym", mode) for _ in range(4)]
    for k, streams in enumerate(([2, 0], [1, 3, 0], [3])):
        chunks = [x4[(k + j) % 4, 0, :hop * (2 + j)] for j in range(len(streams))]
        zs, fr = s.encode_streams(chunks, streams)
        for zu, c, st in zip(torch.split(zs, fr, dim=2), chunks, streams):
            _eq(singles[st].encode(c.view(1, 1, -1)), zu.contiguous(), f"slot {st} call {k}")
    a, b = _enc("sym", mode), _enc("sym", mode, warm=None)
    a.encode(x[..., :7 * hop])
    b.load_stream_state(0, a.stream_state(0), a.state_layout)
    _eq(b.encode(x[..., 7 * hop:19 * hop]), a.encode(x[..., 7 * hop:19 * hop]), "export / import")


@pytest.mark.parametrize("wire", [False, True])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_transmitter_graph_equals_eager(g, mode, wire):
    """TransmitterGraph on an encoder-only handle: every launch equals the eager encode + quantize (packed bytes with wire), and the
    causal state advances as the eager calls advance it."""
    from audiodec_b200.codec import TransmitterGraph, is_library_codec
    torch.manual_seed(5)
    hop = 300
    xs = 0.1 * torch.randn(4, 3, 1, 5 * hop, device=DEV)
    ge, ee = _enc("sym", mode), _enc("sym", mode)
    for t in (ge, ee):
        t.set_streams(3)
    graph = TransmitterGraph(ge, 3, 5 * hop, wire=wire)
    for k in range(4):
        out = graph(xs[k]).clone()
        z = ee.encode(xs[k])
        ref = ee.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)[1] if wire else ee.quantize(z)
        _eq(out, ref, f"step {k}")
    _eq(ge.stream_state(range(3)), ee.stream_state(range(3)), "state")
    assert is_library_codec(ge, _full("sym"), _full("sym"))


def test_refusals():
    """What the encoder-only handle does not run fails with a message naming it; fp32 compute with a bf16 activation mode, and the
    full handle's bf16, stay refused."""
    from audiodec_b200 import _lib
    from audiodec_b200.codec import SymADEncoderStreamGenerator, SymADStreamGenerator
    t = _enc("sym", 1)
    lib, h, s = t._lib, t._h, t._stream()
    z = t.encode(torch.zeros(1, 1, 3000, device=DEV))
    idx = t.quantize(z)
    zq = torch.empty(1, 10, 64, device=DEV)
    y = torch.empty(1, 1, 3000, device=DEV)
    p = lambda a: ctypes.c_void_p(a.data_ptr())
    ip = (ctypes.c_int * 1)(10)
    calls = {
        "decode": lambda: lib.adec_decode(h, p(zq), 1, 10, p(y), s),
        "decode_offline": lambda: lib.adec_decode_offline(h, p(zq), 1, 10, p(y), s),
        "lookup": lambda: lib.adec_lookup(h, p(idx), 1, 10, p(zq), s),
        "unpack_indices": lambda: lib.adec_unpack_indices(h, p(torch.zeros(1, 10, 10, dtype=torch.uint8, device=DEV)), 1, 10, p(idx), s),
        "quantize_ex (zq)": lambda: lib.adec_quantize_ex(h, p(z), 1, 10, p(idx), None, p(zq), s),
        "quantize_forward": lambda: lib.adec_quantize_forward(h, p(z), 1, 10, p(idx), p(zq), s),
        "zq_moments": lambda: lib.adec_zq_moments(h, p(zq), ip, 1, p(torch.empty(64, dtype=torch.float64, device=DEV)),
                                                  p(torch.empty(64, dtype=torch.float64, device=DEV)), s),
    }
    for what, call in calls.items():
        assert call() != 0, what
        assert "ADEC_MODEL_SYMAD_ENCODER" in _lib.last_error(h), (what, _lib.last_error(h))
    full = _full("sym")
    xh = torch.zeros(1, 1, 3000)
    yh = torch.empty(1, 1, 3000)
    assert lib.adec_codec_host(h, full._h, p(xh), 1, 3000, None, p(yh), s) != 0
    assert "ADEC_MODEL_SYMAD_ENCODER" in _lib.last_error(h)
    with pytest.raises(RuntimeError, match="no lookup"):
        t.quantize_fused(z)
    # the dtype of the call must be the handle's, both ways
    xb = torch.zeros(1, 1, 3000, device=DEV, dtype=torch.bfloat16)
    zb = torch.empty(1, 64, 10, device=DEV, dtype=torch.bfloat16)
    assert lib.adec_encode_bf16(h, p(xb), 1, 3000, p(zb), s) != 0 and "fp32 activations" in _lib.last_error(h)
    assert lib.adec_quantize_bf16(h, p(zb), 1, 10, p(idx), s) != 0 and "fp32 activations" in _lib.last_error(h)
    t2 = _enc("sym", 2)
    assert lib.adec_encode(t2._h, p(torch.zeros(1, 1, 3000, device=DEV)), 1, 3000, p(z), s) != 0
    assert "adec_encode_bf16" in _lib.last_error(t2._h)
    assert lib.adec_quantize(t2._h, p(z), 1, 10, p(idx), s) != 0 and "adec_quantize_bf16" in _lib.last_error(t2._h)
    assert lib.adec_quantize_ex_bf16(t2._h, p(zb), 1, 10, p(idx), None, p(zq), s) != 0
    assert "ADEC_MODEL_SYMAD_ENCODER" in _lib.last_error(t2._h)
    assert lib.adec_quantize_bf16(full._h, p(zb), 1, 10, p(idx), s) != 0 and "fp32 activations" in _lib.last_error(full._h)
    cfg = _lib.AdecConfig()
    ctypes.memmove(ctypes.byref(cfg), ctypes.byref(t._cfg), ctypes.sizeof(cfg))
    hh = ctypes.c_void_p()
    cfg.model_type, cfg.compute_dtype = _lib.MODEL_SYMAD, 1
    assert lib.adec_create(ctypes.byref(cfg), 0, ctypes.byref(hh)) != 0
    assert "HiFi-GAN" in _lib.last_error(None) and "ADEC_MODEL_SYMAD_DECODER" in _lib.last_error(None)
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).to(torch.bfloat16)
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(**S.SYMAD_PARAMS).set_activation_dtype(torch.bfloat16)
    with pytest.raises(NotImplementedError):
        SymADEncoderStreamGenerator(**S.SYMAD_PARAMS).set_activation_dtype(torch.float16)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("path", ["tf32", "ffma"])
def test_bf16_needs_the_f16_engine(monkeypatch, path, mode):
    """compute_dtype 1 and 2 on the tf32 or FFMA engine are refused at creation, with the engine named."""
    from audiodec_b200.codec import SymADEncoderStreamGenerator
    monkeypatch.setenv("ADEC_CONV_PATH", path)
    t = SymADEncoderStreamGenerator(**S.SYMAD_PARAMS)
    t.load_state_dict(_sd("sym"))
    t = t.to(torch.bfloat16) if mode == 1 else t.set_activation_dtype(torch.bfloat16)
    with pytest.raises(RuntimeError, match="f16 tensor-core engine"):
        t.to(DEV)


@pytest.mark.parametrize("name", sorted(__import__("oracle.rvq_cases", fromlist=["all_cases"]).all_cases()))
def test_rvq_on_bf16_z_equals_the_spec(name):
    """The tie-heavy rvq_cases families rounded to bf16, quantized by a compute_dtype 2 handle (rvq_kernel's bf16-z input): indices
    and packed bytes equal the C spec applied to the widened z and the bitstream oracle, with no tolerance, at shapes that take the
    three frames-per-pass variants."""
    from audiodec_b200.codec import SymADEncoderStreamGenerator
    from oracle import bitstream_oracle, rvq_cases, rvq_spec
    c = rvq_cases.all_cases()[name]()
    t = SymADEncoderStreamGenerator(**c.params)
    t.load_state_dict(c.state_dict())
    t = t.set_activation_dtype(torch.bfloat16).eval().to(DEV)
    for B, F in ((1, 7), (3, 37), (96, 33), (64, 160)):
        if B * F > len(c.frames):
            continue
        z = torch.from_numpy(c.z(B, F)).to(DEV).to(torch.bfloat16)
        idx, packed, _ = t.quantize_fused(z, want_idx=True, want_packed=True, want_zq=False)
        zw = z.float().cpu().numpy()
        spec = rvq_spec.rvq_frames(zw.transpose(0, 2, 1).reshape(B * F, -1), c.embeds)[0].reshape(-1, B, F)
        got = idx.cpu().numpy().reshape(spec.shape)
        np.testing.assert_array_equal(got, spec, err_msg=f"{name} {B}x{F}")
        np.testing.assert_array_equal(packed.cpu().numpy().reshape(B, F, -1), bitstream_oracle.pack_indices(spec, c.params["codebook_size"]))
        np.testing.assert_array_equal(t.quantize(z).cpu().numpy().reshape(spec.shape), spec)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_servers_with_encoder_only_transmitter(mode):
    """MultiStreamCodecServer (its graphed lock-step pass) and SessionCodecServer (slot calls, and a session detached from one server
    and attached to another whose transmitter has the same config and dtype) with an encoder-only tx_encoder: every decoded frame
    equals the eager encode -> quantize -> lookup -> decode of the same frames, bit for bit."""
    from audiodec_b200.server import MultiStreamCodecServer, SessionCodecServer
    torch.manual_seed(11)
    n, frame = 3, 1500
    frames = (0.1 * torch.randn(4, n, frame)).numpy()

    def eager(k_steps):
        tx, rx, dec = _enc("sym", mode), _full("sym"), _full("sym")
        dec.initial_decoder(rx.initial_encoder(8192, DEV))
        out = []
        for k in range(k_steps):
            x = torch.from_numpy(frames[k]).to(DEV).view(n, 1, frame)
            out.append(dec.decode(rx.lookup(tx.quantize(tx.encode(x)))).cpu().numpy().reshape(n, -1))
        return out

    def codec():
        tx, rx, dec = _enc("sym", mode), _full("sym"), _full("sym")
        dec.initial_decoder(rx.initial_encoder(8192, DEV))
        return tx, rx, dec

    ref = eager(4)
    srv = MultiStreamCodecServer(*codec(), n, frame_size=frame, device=DEV)
    for k in range(4):
        for s in range(n):
            srv.submit(s, frames[k, s])
        assert srv.step() == n
        for s in range(n):
            np.testing.assert_array_equal(srv.poll(s), ref[k][s], err_msg=f"lock-step {k} {s}")
    assert srv._graphs is not None                           # the lock step ran as graphs on the library's generators
    a, b = SessionCodecServer(*codec(), n, frame_size=frame, device=DEV), SessionCodecServer(*codec(), n, frame_size=frame, device=DEV)
    ids = [a.open() for _ in range(n)]
    for k in range(4):
        srv_k = a if k < 2 else b
        if k == 2:
            ids = [b.attach(a.detach(i)) for i in ids]
        for s, i in enumerate(ids):
            srv_k.submit(i, frames[k, s])
        srv_k.step()
        for s, i in enumerate(ids):
            np.testing.assert_array_equal(srv_k.poll(i), ref[k][s], err_msg=f"session {k} {s}")
