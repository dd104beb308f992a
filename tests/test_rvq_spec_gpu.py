"""rvq_kernel, lookup_kernel and the bitstream kernels against the plain-C spec (oracle/rvq_oracle.c via oracle/rvq_spec.py) and
the bitstream oracle, with no tolerance, on inputs built so that the nearest-codeword search has ties to decide
(oracle/rvq_cases.py; tests/test_rvq_spec_cpu.py checks that each case holds them).

Shapes: B x F where blocks straddle utterances and the last block is partial, plus a size for every launch adec_quantize_ex
picks.  (FP, n_pass, blocks) = frames per pass, passes per block and grid size, as the cost rule in launch_rvq chooses them on an
H100 SXM (132 SMs; the occupancy query gives 2 blocks per SM for FP 8 and FP 12 and 1 for FP 16, whose 168 registers per thread
leave room for one 256-thread block):
    (1, 1), (1, 7)   -> (8, 1, 1)          (3, 37)   -> (8, 1, 14)       (333, 1)  -> (8, 1, 42)
    (256, 5)         -> (8, 1, 160)        (32, 66)  -> (8, 1, 264)      (96, 33)  -> (12, 1, 264)
    (128, 33)        -> (8, 2, 264)        (64, 160) -> (8, 5, 256)      (160, 165) -> (12, 8, 275), more than one wave
With one block per SM, FP 16 costs more than FP 8 at every size, so the rule never picks it.

Every frame is compared up to 8192 frames; above that the first and last 512 and every 37th frame in between (frames are
independent in the kernel and in the spec)."""
import itertools

import numpy as np
import pytest
import torch

from audiodec_b200 import synthetic as S
from oracle import bitstream_oracle as BO
from oracle import rvq_cases as C
from oracle import rvq_spec as R

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (1, 7), (3, 37), (333, 1), (256, 5), (32, 66), (96, 33), (128, 33), (64, 160), (160, 165)]
FULL = 8192
_CASES = C.all_cases()


def _compared(nfr):
    if nfr <= FULL:
        return np.arange(nfr)
    return np.unique(np.concatenate([np.arange(512), np.arange(512, nfr - 512, 37), np.arange(nfr - 512, nfr)]))


class _Spec:
    """The spec's indices per frame of one case, computed once for every shape that contains the frame."""

    def __init__(self, case):
        self.case = case
        self.idx = np.full((case.embeds.shape[0], len(case.frames)), -1, np.int64)

    def __call__(self, frames):
        todo = frames[self.idx[0, frames] < 0]
        if len(todo):
            self.idx[:, todo] = R.rvq_frames(self.case.frames[todo], self.case.embeds)[0]
        return self.idx[:, frames]


@pytest.fixture(scope="module", params=sorted(_CASES))
def case(request):
    from audiodec_b200.codec import SymADStreamGenerator
    c = _CASES[request.param]()
    g = SymADStreamGenerator(**c.params)
    g.load_state_dict(c.state_dict())
    g = g.eval().to(torch.device("cuda:0"))
    return c, g, _Spec(c)


def _mismatch(got, want, what):
    bad = np.argwhere(got != want)
    return f"{what}: {len(bad)} differ, first at {bad[:4].tolist()}: got {got[tuple(bad[:4].T)]}, want {want[tuple(bad[:4].T)]}"


@pytest.mark.parametrize("B,F", SHAPES)
def test_rvq_and_lookup_equal_the_spec(case, B, F):
    c, g, spec = case
    nq, D, N = c.embeds.shape
    nfr = B * F
    sel = _compared(nfr)
    ref_idx = spec(sel)                                                  # (nq, len(sel))
    ref_zq = R.lookup(ref_idx, c.embeds)                                 # (len(sel), D)
    ref_packed = BO.pack_indices(ref_idx[:, None], N)[0]                 # (len(sel), bytes)
    z = torch.from_numpy(c.z(B, F)).cuda()

    def check(idx=None, packed=None, zq=None):
        if idx is not None:
            got = idx.reshape(nq, nfr).cpu().numpy()[:, sel]
            assert np.array_equal(got, ref_idx), _mismatch(got, ref_idx, f"{c.name} {B}x{F} indices")
        if packed is not None:
            got = packed.reshape(nfr, -1).cpu().numpy()[sel]
            assert np.array_equal(got, ref_packed), _mismatch(got, ref_packed, f"{c.name} {B}x{F} packed bytes")
        if zq is not None:
            got = zq.reshape(nfr, D).cpu().numpy()[sel]
            assert np.array_equal(got.view(np.int32), ref_zq.view(np.int32)), _mismatch(got, ref_zq, f"{c.name} {B}x{F} zq")

    idx = g.quantize(z)
    check(idx=idx)
    for want in itertools.product((True, False), repeat=3):
        if any(want):
            out = g.quantize_fused(z, *want)
            assert [o is not None for o in out] == list(want)
            check(*out)
    # the lookup side on the kernel's own indices, every frame: lookup, lookup straight from the bitstream, unpack(pack(.))
    all_idx = idx.reshape(nq, nfr).cpu().numpy()
    want_zq = R.lookup(all_idx, c.embeds)
    zq = g.lookup(idx).reshape(nfr, D).cpu().numpy()
    assert np.array_equal(zq.view(np.int32), want_zq.view(np.int32)), _mismatch(zq, want_zq, f"{c.name} {B}x{F} lookup")
    packed = g.pack(idx)
    check(packed=packed)
    zqp = g.lookup_packed(packed).reshape(nfr, D).cpu().numpy()
    assert np.array_equal(zqp.view(np.int32), want_zq.view(np.int32)), _mismatch(zqp, want_zq, f"{c.name} {B}x{F} lookup_packed")
    back = g.unpack(packed).reshape(nq, nfr).cpu().numpy()
    assert np.array_equal(back, all_idx)
    assert not g.index_error()
