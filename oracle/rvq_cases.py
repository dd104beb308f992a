"""TEST INFRASTRUCTURE ONLY - residual-VQ inputs on which the nearest-codeword search has to decide ties.

With seeded Gaussian codebooks and z, two codewords essentially never share the minimum distance, so a kernel could break ties
the wrong way, sum ||e||^2 in another order or round the residual differently and still return the indices of every seeded test.
Each builder here starts from the synthetic symAD state dict, replaces the codebooks (`embed`; `embed_avg` and `cluster_size`
follow it) and streams frames chosen so that those decisions happen:

  a  dyadic      codewords in {-1/2, 0, 1/2}, z in multiples of 1/4: every fp32 product and sum is exact, so many codewords are
                 exactly equidistant whatever the order, and only the tie-break decides
  b  duplicates  identical codeword columns at each reduction level of rvq_kernel (GROUPS), in every stage; each frame is a sum of
                 one group's lowest member per stage, so every stage decides between identical columns
  c  rounding    the seed codebooks with Gaussian z scaled by 2^10 .. 2^20: distances of distinct codewords round to one value
  d  zero_residual  frames equal to stage-0 codewords, so stage 1 sees a residual of exactly 0 and picks the codeword with the
                 smallest ||e||^2; stages >= 1 hold two permutations of one short vector whose cascade sums (the host's order) and
                 sequential sums order them oppositely
  e  subnormal   codebooks scaled by 2^-68 and z by 2^-68 .. 2^-126: squares, norms and distances are subnormal fp32
  g  residual_rounding  the one pattern where the residual update r - (r + (e - r)) differs from r - e, followed by a stage
                 whose decision flips with it (see residual_rounding)

Frame k of a (B, F) call is frames[k] with (b, f) = divmod(k, F), so every shape reads a prefix of one stream and a spec result
computed for frame k serves every shape that contains it.
"""
import numpy as np
import torch

from audiodec_b200 import synthetic as S

N_FRAMES = 26400          # the largest shape of tests/test_rvq_spec_gpu.py (160 x 165)
THREADS, WARP = 256, 32   # rvq_kernel: thread t holds codewords t, t + 256, t + 512, t + 768

# Codeword groups made identical in every stage of case b; the lowest index must win.  In rvq_kernel:
#   (300, 556)       one thread (44), slots m = 1 and m = 2: the per-thread loop
#   (1, 256)         one warp, the lower index in the higher lane (lane 1 vs lane 0): the xor shuffle
#   (254, 257)       the lower index in the higher warp (warp 7 vs warp 0): the cross-warp loop
#   (0, 1023)        the two ends of the codebook
#   (40, 264, 296)   a triple: 296 shares thread 40, 264 sits in warp 0 below 40's warp 1
GROUPS = ((300, 556), (1, 256), (254, 257), (0, 1023), (40, 264, 296))


class Case:
    def __init__(self, name, params, embeds, frames):
        self.name, self.params = name, params
        self.embeds = np.ascontiguousarray(embeds, dtype=np.float32)      # (nq, D, N)
        self.frames = np.ascontiguousarray(frames, dtype=np.float32)      # (N_FRAMES, D)
        assert self.embeds.shape == (params["codebook_num"], params["code_dim"], params["codebook_size"])
        assert self.frames.shape[1] == params["code_dim"]

    def state_dict(self, seed=0):
        sd = S.symad_state_dict(self.params, seed=seed)
        for i, e in enumerate(self.embeds):
            t = torch.from_numpy(e.copy())
            pre = f"quantizer.codebook.layers.{i}"
            assert sd[f"{pre}.embed"].shape == t.shape
            sd[f"{pre}.embed"] = t
            sd[f"{pre}.embed_avg"] = t.clone()
            sd[f"{pre}.cluster_size"] = torch.zeros(t.shape[1])
        return sd

    def z(self, B, F):
        """(B, D, F) float32 as encode() returns it: frame k = frames[k], k = b * F + f."""
        d = self.frames.shape[1]
        return np.ascontiguousarray(self.frames[:B * F].reshape(B, F, d).transpose(0, 2, 1))


def _seed_embeds(params, seed=0):
    sd = S.symad_state_dict(params, seed=seed)
    return np.stack([sd[f"quantizer.codebook.layers.{i}.embed"].numpy() for i in range(params["codebook_num"])])


def dyadic(params=S.SYMAD_PARAMS, seed=0, n=N_FRAMES):
    rng = np.random.default_rng(1000 + seed)
    nq, d, N = params["codebook_num"], params["code_dim"], params["codebook_size"]
    E = rng.integers(-1, 2, (nq, d, N)) * (rng.random((nq, d, N)) < 0.2) * 0.5
    x = rng.integers(-4, 5, (n, d)) * 0.25
    return Case("a_dyadic", params, E, x)


def duplicates(params=S.SYMAD_PARAMS, seed=0, n=N_FRAMES):
    rng = np.random.default_rng(2000 + seed)
    nq = params["codebook_num"]
    # stage i scaled by 0.45^i (instead of the seed's 0.88^i) so that a sum of one codeword per stage is quantised back into
    # those codewords: the later stages then decide between duplicated columns as well
    E = _seed_embeds(params, seed) * (0.45 / 0.88) ** np.arange(nq)[:, None, None]
    for g in GROUPS:
        E[:, :, list(g[1:])] = E[:, :, g[:1]]
    pick = rng.integers(0, len(GROUPS), (n, nq))
    lows = np.array([g[0] for g in GROUPS])[pick]                          # (n, nq)
    x = np.zeros((n, E.shape[1]), np.float64)
    for i in range(nq):
        x += E[i][:, lows[:, i]].T
    x += 0.05 * np.abs(E[-1]).mean() * rng.standard_normal(x.shape)
    return Case("b_duplicates", params, E.astype(np.float32), x)


def rounding(params=S.SYMAD_PARAMS, seed=0, n=N_FRAMES):
    rng = np.random.default_rng(3000 + seed)
    scale = 2.0 ** (10 + np.arange(n) % 11)                                 # 2^10 .. 2^20, cycling over the frames
    x = 0.6 * rng.standard_normal((n, params["code_dim"])) * scale[:, None]
    return Case("c_rounding", params, _seed_embeds(params, seed), x)


def cascade_norms(E):
    """numpy float32 restatement of ||e||^2 in the host's order (rvq_oracle.c adec_oracle_codeword_norms), E (D, N)."""
    E = np.asarray(E, np.float32)
    total = None
    for b in range(0, E.shape[0], 16):
        part = np.zeros(E.shape[1], np.float32)
        for k in range(b, min(b + 16, E.shape[0])):
            part = part + E[k] * E[k]
        total = part if total is None else total + part
    return total


def sequential_norms(E):
    """||e||^2 summed over the rows one after another: the order the host must NOT use."""
    E = np.asarray(E, np.float32)
    total = np.zeros(E.shape[1], np.float32)
    for k in range(E.shape[0]):
        total = total + E[k] * E[k]
    return total


def permuted_pair(rng, d, scale):
    """Two permutations (u, w) of one vector with cascade(u) < cascade(w) but sequential(u) > sequential(w)."""
    v = (scale * rng.standard_normal(d)).astype(np.float32)
    for _ in range(100000):
        P = np.stack([v[rng.permutation(d)] for _ in range(2)], 1)        # (D, 2)
        c, s = cascade_norms(P), sequential_norms(P)
        if c[0] < c[1] and s[0] > s[1]:
            return P[:, 0], P[:, 1]
    raise RuntimeError("no permuted pair found")


def zero_residual(params=S.SYMAD_PARAMS, seed=0, n=N_FRAMES):
    rng = np.random.default_rng(4000 + seed)
    nq, d, N = params["codebook_num"], params["code_dim"], params["codebook_size"]
    E = _seed_embeds(params, seed)
    pairs = []
    for i in range(1, nq):
        # the pair is far shorter than every other codeword of the stage, so it holds the two smallest norms; the winner u
        # sits at the higher column in odd stages, so that the index order does not decide for it
        u, w = permuted_pair(rng, d, 0.02 * 0.88 ** i)
        cu, cw = (97 * i) % N, (97 * i + 500) % N
        if i % 2:
            cu, cw = cw, cu
        E[i][:, cu], E[i][:, cw] = u, w
        pairs.append((i, cu, cw))
    x = E[0][:, rng.integers(0, N, n)].T
    c = Case("d_zero_residual", params, E, x)
    c.pairs = pairs                                                         # (stage, cascade winner, sequential winner)
    return c


def subnormal(params=S.SYMAD_PARAMS, seed=0, n=N_FRAMES):
    rng = np.random.default_rng(5000 + seed)
    E = _seed_embeds(params, seed) * 2.0 ** -68
    scale = 2.0 ** -np.array([68, 72, 80, 100, 110, 126])[np.arange(n) % 6]   # z from ~2e-21 down to ~7e-39
    x = 0.6 * rng.standard_normal((n, params["code_dim"])) * scale[:, None]
    return Case("e_subnormal", params, E, x)


def residual_rounding(params=S.SYMAD_PARAMS, seed=0, n=N_FRAMES):
    """The update r - (r + (e - r)) equals r - e in fp32 round-to-nearest unless |e| > 2|r| and r - e lands on a rounding tie at
    the bottom of a binade (with |e| << |r|, as in case c, the two are identical).  Here stage 0 maps z = -a u_j onto the codeword
    -(a + 1 + 2^-24) u_j: the exact residual 1 + 2^-24 is such a tie, r - e rounds it to 1 and the reference's form gives
    1 - 2^-24.  Stage 1 holds 2 u_j at column j and the zero vector at column 1000: from 1 - 2^-24 the zero vector is strictly
    nearer, from 1 the two are tied and column j would win."""
    rng = np.random.default_rng(6000 + seed)
    nq, d, N = params["codebook_num"], params["code_dim"], params["codebook_size"]
    E = 10.0 * _seed_embeds(params, seed)                                  # every other codeword is far away
    a = (2 ** 23 + 1 + 2 * rng.choice(2 ** 22, 8 * d, replace=False)) * 2.0 ** -24   # odd multiples of 2^-24 in [0.5, 1)
    r, e = (-a).astype(np.float32), (-(a + 1 + 2.0 ** -24)).astype(np.float32)
    a = a[(r - (r + (e - r))) != (r - e)][:d]                              # half of them: r + (e - r) rounds away from e
    assert len(a) == d
    for j in range(d):
        E[0][:, j] = 0.0
        E[0][j, j] = -(a[j] + 1 + 2.0 ** -24)                              # exact in fp32: a multiple of 2^-23 in [1, 2)
        E[1][:, j] = 0.0
        E[1][j, j] = 2.0
    E[1][:, 1000] = 0.0
    j = rng.integers(0, d, n)
    x = np.zeros((n, d))
    x[np.arange(n), j] = -a[j]
    assert np.array_equal(E[0].astype(np.float32).astype(np.float64), E[0])
    return Case("g_residual_rounding", params, E, x)


def all_cases():
    """name -> builder; f = the 16-codebook variant with cases b and c."""
    c16 = S.SYMAD_C16_PARAMS
    return {"a_dyadic": dyadic, "b_duplicates": duplicates, "c_rounding": rounding, "d_zero_residual": zero_residual,
            "e_subnormal": subnormal, "g_residual_rounding": residual_rounding,
            "f_c16_duplicates": lambda: _renamed(duplicates(c16), "f_c16_duplicates"),
            "f_c16_rounding": lambda: _renamed(rounding(c16), "f_c16_rounding")}


def _renamed(case, name):
    case.name = name
    return case


def tie_profile(dist, idx):
    """Ties in the spec's distances dist (nq, frames, N) at its decisions idx (nq, frames) flat.  Counts the decisions where
      ties     more than one codeword has the minimum distance
      thread   another minimum sits in the winner's rvq_kernel thread (a `>=` in the per-thread loop would take it)
      lane     another minimum sits in the winner's warp at a lower lane (a shuffle without the index tie-break would take it)
      warp     another minimum sits in a lower warp (a cross-warp loop without the index tie-break would take it)
    and checks that the winner is the lowest index with the minimum distance."""
    nq, frames, N = dist.shape
    w = idx - N * np.arange(nq)[:, None]
    mn = dist.min(-1, keepdims=True)
    at_min = dist == mn
    cols = np.arange(N)
    first = at_min.argmax(-1)
    assert np.array_equal(first, w), "the spec's index is not the first minimum"
    other = at_min & (cols != w[..., None])
    t, tw = cols % THREADS, (w % THREADS)[..., None]
    return {"decisions": nq * frames,
            "ties": int(other.any(-1).sum()),
            "thread": int((other & (t == tw)).any(-1).sum()),
            "lane": int((other & (t // WARP == tw // WARP) & (t % WARP < tw % WARP)).any(-1).sum()),
            "warp": int((other & (t // WARP < tw // WARP)).any(-1).sum())}
