#!/usr/bin/env python3
"""Design check (numpy, CPU) for DESIGN.md section 8 item 1: two output time steps per MMA row.

A dilated causal conv  y[t] = sum_k W[k] x~[t + k d]  (x~ = history ++ chunk, K taps, dilation d) is evaluated for the row pairs
(t, t + d), t in the EVEN d-blocks of the time axis, as ONE GEMM with N = 2 C_out columns [y(t) | y(t + d)]:

    [y(t) | y(t+d)] = sum_{j=0..K} x~[t + j d] . [W_j | W_{j-1}],     W_{-1} = W_K = 0

i.e. K + 1 taps against paired weights instead of 2 K taps.  With the window stored DE-INTERLEAVED by (t // d) % 2 (rows of even
blocks in one array, rows of odd blocks in another, each contiguous), x~[t + j d] for the even-block rows t is a row-shifted slice of
the even array when j is even and of the odd array when j is odd - still "a tap is a shifted start address".  This script checks the
identity and the index arithmetic against the direct formula.  The kernel that uses it is the paired variant of the fused RU(32),
`wg_conv_kernel<32, true, ACT_ELU, PREC_F16, false, false, true>` (audiodec_b200/csrc/wg_conv.cuh); `kernel_tiles` restates its tile,
window and row arithmetic (`pair_tt`, `pair_rows`, the producers' de-interleaved store and the epilogue's output rows)."""
import numpy as np


def direct(xt, W, d):
    K, Cin, Cout = W.shape
    T = xt.shape[0] - (K - 1) * d
    return sum(xt[k * d:k * d + T] @ W[k] for k in range(K))


def paired(xt, W, d):
    """Returns (T, Cout) computed through the paired GEMM on de-interleaved arrays."""
    K, Cin, Cout = W.shape
    P = (K - 1) * d
    T = xt.shape[0] - P
    assert T % (2 * d) == 0, "tile of 2 d-blocks granularity"
    n = xt.shape[0] + d                                     # one extra block of zeros so the last pair's reads stay in range
    xz = np.concatenate([xt, np.zeros((2 * d + d, Cin), xt.dtype)])
    blk = (np.arange(xz.shape[0]) // d) % 2
    even, odd = xz[blk == 0], xz[blk == 1]                  # de-interleaved storage: row r of `even` is time (r // d) * 2 d + r % d
    Wp = np.zeros((K + 1, Cin, 2 * Cout), W.dtype)          # [W_j | W_{j-1}]
    Wp[:K, :, :Cout] = W
    Wp[1:, :, Cout:] = W
    M = T // 2                                              # even-block output rows
    acc = np.zeros((M, 2 * Cout), np.float64)
    for j in range(K + 1):
        src = even if j % 2 == 0 else odd                   # x~[t + j d] for t in the even blocks
        shift = (j // 2) * d                                # row shift inside that array
        acc += src[shift:shift + M].astype(np.float64) @ Wp[j].astype(np.float64)
    y = np.zeros((T, Cout), np.float64)
    te = np.arange(T)[(np.arange(T) // d) % 2 == 0]         # times of the even-block rows, in storage order
    y[te] = acc[:, :Cout]
    y[te + d] = acc[:, Cout:]
    return y


def pair_tt(d, TT=128):
    """Output rows per tile: 2 d-blocks per pair, as many pairs as fit in 128 MMA rows (256, 252, 252 at d = 1, 3, 9)."""
    return 2 * d * (TT // d)


def pair_rows(K, d, TT=128):
    """Rows of each de-interleaved array: 128 MMA rows plus the largest shift, (K - 1) / 2 d."""
    return TT + (K - 1) // 2 * d


def kernel_tiles(xt, W, d, TT=128):
    """(T, Cout) the way the paired kernel computes it: tiles of pair_tt(d) output rows; the tile's window rows m (time j0 + m,
    m < pair_tt + (K - 1) d) stored at row srow(m) of one buffer holding the even array and, from row pair_rows(K, d), the odd one;
    MMA row r reads tap j at srow base (j % 2) pair_rows + (j // 2) d + r, and holds outputs t and t + d of the tile,
    t = (r // d) 2 d + r % d; rows r >= pair_tt / 2 are computed and dropped."""
    K, Cin, Cout = W.shape
    T = xt.shape[0] - (K - 1) * d
    tt, pr = pair_tt(d, TT), pair_rows(K, d, TT)
    wrows = tt + (K - 1) * d
    Wp = np.zeros((K + 1, Cin, 2 * Cout), np.float64)
    Wp[:K, :, :Cout] = W
    Wp[1:, :, Cout:] = W
    y = np.full((T, Cout), np.nan)
    for j0 in range(0, T, tt):
        buf = np.full((2 * pr, Cin), np.nan)          # rows no producer writes stay NaN: a valid row that read one would show
        for m in range(wrows):
            blk = m // d
            buf[(blk & 1) * pr + (blk >> 1) * d + m - blk * d] = xt[j0 + m] if j0 + m < xt.shape[0] else 0.0
        acc = np.zeros((TT, 2 * Cout))
        for j in range(K + 1):
            base = (j & 1) * pr + (j >> 1) * d
            acc += buf[base:base + TT] @ Wp[j]
        for r in range(tt // 2):
            t = j0 + (r // d) * 2 * d + r % d
            assert np.isfinite(acc[r]).all(), "a valid MMA row read a window row the producers did not write"
            for hp in range(2):
                if t + hp * d < T:
                    y[t + hp * d] = acc[r, hp * Cout:(hp + 1) * Cout]
    assert np.isfinite(y).all(), "an output row no tile wrote"
    return y


if __name__ == "__main__":
    rng = np.random.default_rng(0)
    for (K, d, C, T) in ((7, 1, 32, 256), (7, 3, 32, 252), (7, 9, 32, 288), (11, 5, 32, 260), (11, 1, 64, 128)):
        W = rng.standard_normal((K, C, C)).astype(np.float32) / 8
        xt = rng.standard_normal((T + (K - 1) * d, C)).astype(np.float32)
        err = np.abs(paired(xt, W, d) - direct(xt.astype(np.float64), W.astype(np.float64), d)).max()
        print(f"K={K} d={d} C={C} T={T}: max |paired - direct| = {err:.2e}; MMAs per 2 output rows {2 * K} -> {K + 1} (N {C} -> {2 * C})")
    for (d, T) in ((1, 1000), (3, 611), (9, 1000), (9, 20)):
        W = rng.standard_normal((7, 8, 8)) / 8
        xt = rng.standard_normal((T + 6 * d, 8))
        err = np.abs(kernel_tiles(xt, W, d) - direct(xt, W, d)).max()
        print(f"kernel tiles d={d} (tile {pair_tt(d)} rows, arrays of {pair_rows(7, d)}) T={T}: max |tiles - direct| = {err:.2e}")
