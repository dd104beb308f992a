"""CPU checks of the tie cases that tests/test_rvq_spec_gpu.py runs through the RVQ kernel (oracle/rvq_cases.py): each case holds
the decisions it was built for, the C spec (oracle/rvq_oracle.c) agrees with torch where that agreement does not depend on a
summation order, and each wrong model of the kernel changes at least one decision of the cases meant to catch it."""
import numpy as np
import pytest
import torch

from oracle import audiodec_oracle as O
from oracle import rvq_cases as C
from oracle import rvq_spec as R

FRAMES = 512
_CASES = C.all_cases()


@pytest.fixture(scope="module")
def spec():
    """name -> (case, idx, qsum, dist) of the spec on the first FRAMES frames."""
    out = {}

    def get(name):
        if name not in out:
            c = _CASES[name]()
            out[name] = (c,) + R.rvq_frames(c.frames[:FRAMES], c.embeds, dist=True)
        return out[name]
    return get


def _torch_idx(c):
    x = torch.from_numpy(c.frames[:FRAMES]).unsqueeze(0)
    _, idx = O.rvq_forward_index(x, [torch.from_numpy(e) for e in c.embeds], True)
    return idx.squeeze(1).numpy()


def _staged(c, pick="first", update="spec"):
    """The spec run one stage at a time (nq = 1 per call) with the decision and the residual update done here, so that a wrong
    tie-break or residual rounding can be modelled.  numpy float32 rounds every operation and has no FMA, like the spec."""
    r = c.frames[:FRAMES].copy()
    nq, _, N = c.embeds.shape
    out = []
    for i in range(nq):
        _, _, dist = R.rvq_frames(r, c.embeds[i:i + 1], dist=True)
        d = dist[0]
        w = d.argmin(-1) if pick == "first" else N - 1 - d[:, ::-1].argmin(-1)
        q = c.embeds[i][:, w].T
        r = r - (r + (q - r)) if update == "spec" else r - q
        out.append(w + N * i)
    return np.stack(out)


@pytest.mark.parametrize("name", sorted(_CASES))
def test_case_has_the_decisions_it_is_built_for(spec, name):
    c, idx, qsum, dist = spec(name)
    prof = C.tie_profile(dist, idx)
    print(f"[rvq cases] {name}: {prof}")
    nq = c.embeds.shape[0]
    ties_per_stage = (dist == dist.min(-1, keepdims=True)).sum(-1) > 1
    if name.startswith(("a_", "b_", "f_c16_dup")):
        # ties at every reduction level of the kernel, and in every stage
        assert prof["thread"] > 0 and prof["lane"] > 0 and prof["warp"] > 0, prof
        assert ties_per_stage.any(1).all()
    if name == "a_dyadic":
        # every distance is exact: the float64 distance of the spec's own residual chain, rounded to fp32, equals it
        r = c.frames[:FRAMES].astype(np.float64)
        for i in range(nq):
            E = c.embeds[i].astype(np.float64)
            exact = (r * r).sum(1)[:, None] - 2 * r @ E + (E * E).sum(0)[None]
            assert np.array_equal(dist[i], exact.astype(np.float32)) and np.array_equal(exact.astype(np.float32), exact)
            r = r - E[:, idx[i] - c.embeds.shape[2] * i].T
    if name.startswith(("b_", "f_c16_dup")):
        # every stage of every frame chooses between identical columns, and every group wins somewhere in every stage
        assert prof["ties"] == prof["decisions"]
        w = idx - c.embeds.shape[2] * np.arange(nq)[:, None]
        for g in C.GROUPS:
            assert (w == g[0]).any(1).all(), g
    if name.startswith(("c_", "f_c16_round")):
        assert prof["ties"] > 0 and prof["thread"] + prof["lane"] + prof["warp"] > 0
    if name == "d_zero_residual":
        # stage 1 sees a residual of exactly 0 (distance == ||e||^2) and takes the pair member the cascade order prefers
        e2 = np.stack([R.codeword_norms(e) for e in c.embeds])
        assert np.array_equal(dist[1], np.broadcast_to(e2[1], dist[1].shape))
        for i, cu, cw in c.pairs:
            assert np.array_equal(e2[i], C.cascade_norms(c.embeds[i]))
            seq = C.sequential_norms(c.embeds[i])
            assert e2[i].argmin() == cu and seq.argmin() == cw, (i, cu, cw)
        assert (idx[1] == c.pairs[0][1] + c.embeds.shape[2]).all()
    if name == "g_residual_rounding":
        # stage 1 sees 1 - 2^-24 in component j, where the zero vector (column 1000) is strictly nearer than 2 u_j (column j)
        j = np.abs(c.frames[:FRAMES]).argmax(1)
        assert (idx[0] == j).all() and (idx[1] == 1000 + c.embeds.shape[2]).all()
        assert (dist[1][:, 1000] < dist[1][np.arange(FRAMES), j]).all()
    if name == "e_subnormal":
        # the distances are subnormal fp32 and decide: a flush-to-zero build would see all-zero distances and take index 0
        tiny = np.finfo(np.float32).tiny
        assert ((dist != 0) & (np.abs(dist) < tiny)).mean() > 0.5
        assert (idx - c.embeds.shape[2] * np.arange(nq)[:, None] != 0).mean() > 0.9


@pytest.mark.parametrize("name", ["a_dyadic", "b_duplicates", "f_c16_duplicates"])
def test_spec_equals_torch_where_the_ties_are_order_free(spec, name):
    """Exact arithmetic (a) or identical columns (b): the tie does not depend on a summation order, so the spec and the torch
    oracle must make every decision alike on any CPU."""
    c, idx, _, _ = spec(name)
    np.testing.assert_array_equal(idx, _torch_idx(c))


@pytest.mark.parametrize("name", ["c_rounding", "d_zero_residual", "e_subnormal", "f_c16_rounding"])
def test_spec_vs_torch_on_order_dependent_cases_is_reported(spec, name):
    """Rounding ties, cascade norms and subnormals: agreement rests on torch-CPU summing in the spec's order (MKL's path, which
    test_c_rvq_oracle_matches_torch_bitwise pins on random data).  Another CPU may differ without the kernel being wrong, so
    this only reports."""
    c, idx, _, _ = spec(name)
    same = int((idx == _torch_idx(c)).sum())
    print(f"[rvq cases] {name}: spec and torch agree on {same} of {idx.size} decisions")


def test_staged_model_is_the_spec(spec):
    """The stage-at-a-time model below, with the right tie-break and residual update, reproduces the spec."""
    for name in ("a_dyadic", "c_rounding", "g_residual_rounding"):
        c, idx, _, _ = spec(name)
        np.testing.assert_array_equal(_staged(c), idx)


@pytest.mark.parametrize("name", ["a_dyadic", "b_duplicates", "c_rounding"])
def test_last_index_tie_break_is_caught(spec, name):
    c, idx, _, _ = spec(name)
    changed = int((_staged(c, pick="last") != idx).sum())
    print(f"[rvq cases] {name}: a last-index tie-break changes {changed} decisions")
    assert changed > 0


def test_sequential_norms_are_caught(spec):
    c, idx, _, _ = spec("d_zero_residual")
    e2 = np.stack([C.sequential_norms(e) for e in c.embeds])
    midx, _, _ = R.rvq_frames(c.frames[:FRAMES], c.embeds, e2=e2)
    changed = int((midx != idx).sum())
    print(f"[rvq cases] d_zero_residual: sequential ||e||^2 changes {changed} decisions")
    assert changed > 0


def test_plain_residual_update_is_caught(spec):
    """With |e| << |r| (case c) the update r - e equals r - (r + (e - r)) bit for bit, so only case g can tell them apart."""
    for name in ("c_rounding", "g_residual_rounding"):
        c, idx, _, _ = spec(name)
        changed = int((_staged(c, update="plain") != idx).sum())
        print(f"[rvq cases] {name}: residual r - e instead of r - (r + (e - r)) changes {changed} decisions")
    assert changed > 0
