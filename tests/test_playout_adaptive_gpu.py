"""The adaptive playout clock on the GPU.  lookup_packed_timescale against a numpy float32 model of its five row kinds, bit for bit, in
fp32 and bf16, with its real, interpolated and fade rows equal to lookup_packed_playout's and its rows that start from a staged frame
equal to anchor-read rows of a second launch; the C ABI's refusals; and ReceiverSessionServer(playout_delay=D, max_playout_delay=D_max)
end to end for vctk_sym and libritts v1 in receiver modes 0, 1 and 2 under a jitter spike and a slow sender, against a B = 1 decoder
fed the model's zq, and on a clean run against the fixed clock."""
import ctypes
import re

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S
from test_playout_adaptive_cpu import timescale_model, trace
from test_playout_gpu import DEV, FPP, _bf16_bits, _bits, _drain, _gen, _packets, _receiver, _rx

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ the kernel against the model
def _inputs(g, f=29, seed=8):
    nq, n, d = g.codebook_num, S.SYMAD_PARAMS["codebook_size"], g.code_dim
    rng = np.random.default_rng(seed)
    idx = torch.from_numpy(rng.integers(0, n, (nq, f)) + np.arange(nq)[:, None] * n).to(DEV)
    packed = g.pack(idx)
    sums = g.lookup_packed(packed)[0].cpu().numpy()
    a0 = (rng.standard_normal((6, d)) * np.float32(0.3)).astype(np.float32)
    t0 = (rng.standard_normal((2, d)) * np.float32(0.2)).astype(np.float32)
    return rng, packed, sums, a0, t0


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernel_equals_the_model_on_all_five_row_kinds(symad_sd, dtype):
    g = _gen(symad_sd)
    rng, packed, sums, a0, t0 = _inputs(g)
    f = packed.shape[0]
    anchors, targets = torch.from_numpy(a0).to(DEV), torch.from_numpy(t0).to(DEV)
    rows = [(4, -1, -1, -1, 0, 0), (7, -1, -1, 3, 0, 0), (-1, 11, -1, 0, 1, 4), (-1, -1, 0, 1, 9, 10), (-1, -1, 1, -1, 2, 10),
            (5, 6, -1, -1, 1, 4), (5, 6, -1, -1, 3, 4), (6, 5, -1, -1, 1, 2), (9, -1, 0, -1, 1, 10), (9, -1, 1, -1, 10, 10),
            (9, -1, 0, -1, 37, 10), (28, -1, 1, -1, 1, 1), (28, -1, -1, 5, 0, 0), (13, -1, -1, 4, 0, 0)]
    rows += [(int(rng.integers(0, f)), int(rng.integers(0, f)), -1, -1, int(j), FPP - 1) for j in rng.integers(1, FPP - 1, 200)]
    rows += [(int(rng.integers(0, f)), -1, int(rng.integers(0, 2)), -1, int(j), 60) for j in rng.integers(1, 90, 150)]
    rows += [(-1, int(rng.integers(0, f)), -1, 2, int(j), 101) for j in rng.integers(1, 101, 100)]
    rows += [(-1, -1, int(rng.integers(0, 2)), int(rng.integers(0, 3)), int(j), 60) for j in rng.integers(1, 90, 100)]
    rows += [(int(s), -1, -1, -1, 0, 0) for s in rng.integers(0, f, 100)]
    rows = np.asarray(rows, np.int32)
    launches = g.launch_count
    zq = g.lookup_packed_timescale(packed, rows, anchors, targets, dtype=dtype)
    assert g.launch_count == launches + 1 and zq.shape == (1, len(rows), g.code_dim) and zq.dtype == dtype
    want_anchors = a0.copy()
    want = timescale_model(rows, sums, want_anchors, t0)
    got = zq[0].cpu()
    if dtype == torch.float32:
        assert np.array_equal(_bits(got.numpy()), _bits(want))
    else:
        assert np.array_equal(got.view(torch.int16).numpy(), _bf16_bits(want))
    assert np.array_equal(_bits(anchors.cpu().numpy()), _bits(want_anchors))
    # the rows lookup_packed_playout also takes are its rows, bit for bit
    keep = [i for i, r in enumerate(rows) if r[0] < 0 or (r[1] < 0 and r[2] < 0)]
    ref = g.lookup_packed_playout(packed, rows[keep], torch.from_numpy(a0).to(DEV), targets, dtype=dtype)[0].cpu()
    view = torch.int16 if dtype == torch.bfloat16 else torch.int32
    assert np.array_equal(ref.view(view).numpy(), got[keep].view(view).numpy())
    assert not g.index_error()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_rows_from_a_staged_frame_equal_anchor_read_rows_of_a_second_launch(symad_sd, dtype):
    g = _gen(symad_sd)
    rng, packed, sums, a0, t0 = _inputs(g, seed=3)
    targets = torch.from_numpy(t0).to(DEV)
    staged = [(3, 8, -1, -1, 1, 4), (3, 8, -1, -1, 3, 4), (17, 2, -1, -1, 5, 11), (17, -1, 0, -1, 2, 10), (21, -1, 1, -1, 9, 10),
              (21, -1, 1, -1, 10, 10)]
    one = g.lookup_packed_timescale(packed, staged, torch.zeros(1, g.code_dim, device=DEV), targets, dtype=dtype)[0].cpu()
    anchors = torch.zeros(3, g.code_dim, device=DEV)
    g.lookup_packed_playout(packed, [(3, -1, -1, 0, 0, 0), (17, -1, -1, 1, 0, 0), (21, -1, -1, 2, 0, 0)], anchors, targets)
    slot = {3: 0, 17: 1, 21: 2}
    split = [(-1, n, t, slot[s], j, den) for s, n, t, _, j, den in staged]
    two = g.lookup_packed_playout(packed, split, anchors, targets, dtype=dtype)[0].cpu()
    view = torch.int16 if dtype == torch.bfloat16 else torch.int32
    assert np.array_equal(one.view(view).numpy(), two.view(view).numpy())


# ------------------------------------------------------------------ refusals
def _call(g, packed, f, rows, anchors, targets, zq, bf16=False):
    from audiodec_b200 import _lib
    lib = _lib.load()
    arr = (_lib.AdecPlayoutRow * len(rows))(*[_lib.AdecPlayoutRow(*r) for r in rows])
    fn = lib.adec_lookup_packed_timescale_bf16 if bf16 else lib.adec_lookup_packed_timescale
    rc = fn(g._h, ctypes.c_void_p(packed.data_ptr()), f, ctypes.cast(arr, ctypes.c_void_p), len(rows),
            ctypes.c_void_p(anchors.data_ptr()), anchors.shape[0], ctypes.c_void_p(targets.data_ptr()), targets.shape[0],
            ctypes.c_void_p(zq.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    return rc, _lib.last_error(g._h)


@pytest.mark.parametrize("rows,field", [
    ([(0, 1, -1, 0, 1, 2)], r"rows\[0\]\.slot = 0: a between row starts from frame src and has slot = -1"),
    ([(0, 1, -1, -1, 0, 2)], r"rows\[0\]\.j = 0 is outside \[1, den = 2\)"),
    ([(0, 1, -1, -1, 2, 2)], r"rows\[0\]\.j = 2 is outside \[1, den = 2\)"),
    ([(0, 1, -1, -1, 1, 1)], r"rows\[0\]\.den = 1: a between row needs den >= 2"),
    ([(0, -1, 0, 1, 1, 2)], r"rows\[0\]\.slot = 1: a frame-started fade starts from frame src and has slot = -1"),
    ([(0, -1, 0, -1, 0, 2)], r"rows\[0\]\.j = 0: a fade row needs j >= 1"),
    ([(0, -1, 0, -1, 1, 0)], r"rows\[0\]\.den = 0: a fade row needs den >= 1"),
    ([(3, 1, -1, -1, 1, 2)], r"rows\[0\]\.src = 3 is out of range"),
    ([(3, -1, 0, -1, 1, 2)], r"rows\[0\]\.src = 3 is out of range"),
    ([(0, 3, -1, -1, 1, 2)], r"rows\[0\]\.next = 3 is out of range"),
    ([(0, -2, -1, -1, 1, 2)], r"rows\[0\]\.next = -2 is out of range"),
    ([(0, -1, 1, -1, 1, 2)], r"rows\[0\]\.target = 1 is out of range"),
    ([(0, 1, 0, -1, 1, 2)], r"rows\[0\]\.target = 0: only a fade row"),
    ([(-1, 0, 0, -1, 1, 2)], r"rows\[0\]\.target = 0: only a fade row"),
    ([(0, -1, -1, 1, 0, 0), (-1, -1, 0, 1, 1, 2)], r"rows\[1\]\.slot = 1: anchor 1 is read by row 1 and written by row 0"),
])
def test_bad_descriptors_are_refused_by_name(symad_sd, rows, field):
    g = _gen(symad_sd)
    packed = g.pack(torch.zeros(g.codebook_num, 3, dtype=torch.int64, device=DEV))
    anchors = torch.full((2, g.code_dim), 5.0, device=DEV)
    targets = torch.full((1, g.code_dim), 6.0, device=DEV)
    zq = torch.full((len(rows), g.code_dim), 7.0, device=DEV)
    launches = g.launch_count
    for bf16 in (False, True):
        rc, msg = _call(g, packed, 3, rows, anchors, targets, zq, bf16)
        assert rc != 0 and ("lookup_packed_timescale_bf16" if bf16 else "lookup_packed_timescale") in msg
        assert re.search(field, msg), msg
    assert g.launch_count == launches
    torch.cuda.synchronize()
    assert (anchors == 5.0).all() and (zq == 7.0).all()
    with pytest.raises(RuntimeError, match="rows"):
        g.lookup_packed_timescale(packed, rows, anchors, targets)


def test_encoder_and_decoder_only_handles_refuse(symad_sd):
    from audiodec_b200.codec import SymADDecoderStreamGenerator, SymADEncoderStreamGenerator
    packed = torch.zeros(2, 10, dtype=torch.uint8, device=DEV)
    anchors, targets, zq = (torch.zeros(1, 64, device=DEV) for _ in range(3))
    for cls, word in ((SymADEncoderStreamGenerator, "encoder-only"), (SymADDecoderStreamGenerator, "decoder-only")):
        h = cls(**S.SYMAD_PARAMS)
        h.load_state_dict(symad_sd)
        g = h.eval().to(DEV)
        for bf16 in (False, True):
            rc, msg = _call(g, packed, 2, [(0, 1, -1, -1, 1, 2)], anchors, targets, zq, bf16)
            assert rc != 0 and word in msg and "lookup_packed_timescale" in msg, msg
        assert not hasattr(g, "lookup_packed_timescale")


# ------------------------------------------------------------------ end to end
def _spike(n):
    """0 jitter, then 0 - 4 steps for packets 20 .. 59, then 0 again"""
    rng = np.random.default_rng(17)
    out = {}
    for q in range(n):
        out.setdefault(q + (int(rng.integers(0, 5)) if 20 <= q < 60 else 0), []).append(q)
    return out


def _record(rx):
    """wrap rx.lookup_packed_timescale to keep every call's packed frames (host), rows and the anchors before the call"""
    calls, real = [], rx.lookup_packed_timescale

    def spy(packed, rows, anchors, targets, **kw):
        calls.append((packed.clone(), np.array(rows), anchors.cpu().numpy().copy(), targets.cpu().numpy().copy()))
        return real(packed, rows, anchors, targets, **kw)

    rx.lookup_packed_timescale = spy
    return calls


@pytest.mark.parametrize("model", ["vctk_sym", "libritts_v1"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_adaptive_pcm_equals_a_decoder_fed_the_models_zq(symad_sd, hifigan_sd, model, mode):
    n, steps = 260, 270
    traffic = {1: _spike(n), 2: trace("drift-", n, seed=4)}
    packets = _packets(symad_sd, model, sorted(traffic), n, seed=23)
    srv = _receiver(model, symad_sd, hifigan_sd, mode, cap=3, playout_delay=1, max_playout_delay=6)
    calls = _record(srv.rx_encoder)
    for sid in traffic:
        srv.open(sid)
    got = {sid: [] for sid in traffic}
    played = []                                                       # per lookup: the sessions it played, in row order
    for t in range(steps):
        for sid, arr in traffic.items():
            for q in arr.get(t, []):
                srv.submit_packet(packets[sid][q])
        k = len(calls)
        srv.step()
        grew = []
        for sid in sorted(traffic):
            ys = _drain(srv, sid)
            assert len(ys) <= 1
            if ys:
                grew.append(sid)
            got[sid].extend(ys)
        if len(calls) > k:
            played.append(grew)
        else:
            assert not grew
    st = srv.statistics()["per_session"]
    assert st[1]["compressed"] + st[1]["expanded"] > 0 and st[2]["expanded"] > 0
    # the model's zq of every step, from the staged frames' fp32 sums, fed block by block to a B = 1 decoder per session
    dt = torch.bfloat16 if mode == 2 else torch.float32
    ref = {sid: _rx(model, symad_sd, hifigan_sd, mode)[1] for sid in traffic}
    want = {sid: [] for sid in traffic}
    for (packed, rows, anchors, targets), sids in zip(calls, played):
        assert len(rows) == FPP * len(sids)
        sums = srv.rx_encoder.lookup_packed(packed)[0].cpu().numpy() if packed.shape[0] else None      # None: every row fades
        zq = timescale_model(rows, sums, anchors, targets)
        for b, sid in enumerate(sids):
            x = torch.from_numpy(zq[b * FPP:(b + 1) * FPP].copy()).to(DEV).view(1, FPP, -1).to(dt)
            want[sid].append(ref[sid].decode_streams(x, [FPP], [0])[0].float().reshape(-1).cpu().numpy())
    for sid in traffic:
        assert len(got[sid]) == len(want[sid]) > 0, sid
        for k, (a, b) in enumerate(zip(got[sid], want[sid])):
            assert np.array_equal(_bits(a), _bits(b)), (model, mode, sid, k)


@pytest.mark.parametrize("model,mode", [("vctk_sym", 0), ("libritts_v1", 2)])
def test_a_clean_run_equals_the_fixed_clock(symad_sd, hifigan_sd, model, mode):
    sids, n = [4, 7], 24
    packets = _packets(symad_sd, model, sids, n, seed=5)
    ad = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, playout_delay=2, max_playout_delay=5)
    fx = _receiver(model, symad_sd, hifigan_sd, mode, cap=2, playout_delay=2)
    got = {(w, sid): [] for w in ("ad", "fx") for sid in sids}
    for sid in sids:
        ad.open(sid), fx.open(sid)
    for t in range(n + 8):                                            # the senders stop: fades and pauses at the end
        for sid in sids:
            if t < n:
                ad.submit_packet(packets[sid][t])
                fx.submit_packet(packets[sid][t])
        ad.step(), fx.step()
        for sid in sids:
            got["ad", sid].extend(_drain(ad, sid))
            got["fx", sid].extend(_drain(fx, sid))
    for sid in sids:
        assert len(got["ad", sid]) == len(got["fx", sid]) >= n
        for a, b in zip(got["ad", sid], got["fx", sid]):
            assert np.array_equal(_bits(a), _bits(b))
        st = ad.statistics()["per_session"][sid]
        assert (st["compressed"], st["expanded"], st["delay_frames"]) == (0, 0, 3 * FPP)
