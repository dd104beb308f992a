"""TEST INFRASTRUCTURE ONLY - ctypes binding of oracle/rvq_oracle.c, the plain-C spec of the residual VQ.

`rvq_kernel` copies that file's rounding order instruction for instruction (DESIGN.md section 3).  The spec is compiled with
-ffp-contract=off and calls glibc's correctly rounded `fmaf`, so what it computes does not depend on the CPU: the kernels can be
held to it with no tolerance on any machine.  Nothing under audiodec_b200/ imports this file.

Layouts: `embeds` (nq, D, N) = the state dict's `quantizer.codebook.layers.{i}.embed` stacked; `z` (B, D, F) as `encode()` returns
it; indices (nq, B, F) int64 flat (local index + N*i, vq_module.py:145-146); frame k of a (B, F) call is (b, f) = divmod(k, F).
"""
import ctypes
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "rvq_oracle.c")
LIB = os.path.join(_HERE, "_build", "librvq_oracle.so")


def build(force=False):
    """Compile the spec into oracle/_build/ when it is missing or older than its source (what __graft_entry__.build() runs)."""
    if force or not os.path.exists(LIB) or os.path.getmtime(SRC) > os.path.getmtime(LIB):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", LIB, SRC, "-lm"])
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        so = ctypes.CDLL(LIB)
        vp, i = ctypes.c_void_p, ctypes.c_int
        so.adec_oracle_codeword_norms.argtypes = [vp, i, i, vp]
        so.adec_oracle_rvq.argtypes = [vp, i, i, vp, i, i, vp, vp, vp]
        so.adec_oracle_rvq_e2.argtypes = [vp, i, i, vp, vp, i, i, vp, vp, vp]
        so.adec_oracle_lookup.argtypes = [vp, i, i, vp, i, vp]
        for f in (so.adec_oracle_codeword_norms, so.adec_oracle_rvq, so.adec_oracle_rvq_e2, so.adec_oracle_lookup):
            f.restype = None
        _lib = so
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _f32(a):
    return np.ascontiguousarray(np.asarray(a), dtype=np.float32)


def codeword_norms(embed):
    """embed (D, N) -> ||e||^2 (N,) in torch's order (cascade sum over blocks of 16 rows): what the host uploads as e2."""
    embed = _f32(embed)
    d, n = embed.shape
    e2 = np.empty(n, np.float32)
    lib().adec_oracle_codeword_norms(_p(embed), d, n, _p(e2))
    return e2


def rvq_frames(x, embeds, dist=False, e2=None, threads=None):
    """x (frames, D) -> (idx (nq, frames) int64 flat, qsum (frames, D), dist (nq, frames, N) float32 or None).

    qsum is ResidualVQ.forward's quantized_out, the sum over stages of r + (e - r).  dist[i, k, c] is the spec's fp32 distance
    of frame k's stage-i residual to codeword c.  `e2` (nq, N) replaces the spec's codeword norms (a model of a host that sums
    them in another order).  Frames are independent, so they are split over threads (ctypes releases the GIL for the call)."""
    x, embeds = _f32(x), _f32(embeds)
    frames, d = x.shape
    nq, d2, n = embeds.shape
    assert d == d2
    if e2 is not None:
        e2 = _f32(e2)
        assert e2.shape == (nq, n)
    idx = np.empty((nq, frames), np.int64)
    qsum = np.empty((frames, d), np.float32)
    dd = np.empty((nq, frames, n), np.float32) if dist else None
    threads = threads or os.cpu_count() or 1
    step = max(1, -(-frames // threads))

    def run(k0):
        k1 = min(frames, k0 + step)
        ci = np.empty((nq, k1 - k0), np.int64)
        cd = np.empty((nq, k1 - k0, n), np.float32) if dist else None
        xs = np.ascontiguousarray(x[k0:k1])
        if e2 is None:
            lib().adec_oracle_rvq(_p(xs), k1 - k0, d, _p(embeds), nq, n, _p(ci), _p(qsum[k0:k1]), _p(cd))
        else:
            lib().adec_oracle_rvq_e2(_p(xs), k1 - k0, d, _p(embeds), _p(e2), nq, n, _p(ci), _p(qsum[k0:k1]), _p(cd))
        idx[:, k0:k1] = ci
        if dist:
            dd[:, k0:k1] = cd

    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(run, range(0, frames, step)))
    return idx, qsum, dd


def quantize(z, embeds, dist=False):
    """z (B, D, F) -> (idx (nq, B, F) int64 flat, dist (nq, B, F, N) or None): what quantize() must return."""
    z = _f32(z)
    b, d, f = z.shape
    idx, _, dd = rvq_frames(z.transpose(0, 2, 1).reshape(b * f, d), embeds, dist)
    return idx.reshape(-1, b, f), (dd.reshape(dd.shape[0], b, f, -1) if dist else None)


def lookup(idx, embeds):
    """idx (nq, ..., F) int64 flat -> zq (..., F, D) = sum over stages of codebook[idx[i]], in stage order (vq_module.py:159-161).

    This is the zq the product's lookup and fused quantize return (the codewords summed), not the sum of x + (e - x) that
    ResidualVQ.forward accumulates."""
    embeds = _f32(embeds)
    nq, d, n = embeds.shape
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    assert idx.shape[0] == nq
    assert idx.min() >= 0 and idx.max() < nq * n
    frames = int(np.prod(idx.shape[1:]))
    codebook = np.ascontiguousarray(embeds.transpose(0, 2, 1).reshape(nq * n, d))
    zq = np.empty((frames, d), np.float32)
    lib().adec_oracle_lookup(_p(idx), nq, frames, _p(codebook), d, _p(zq))
    return zq.reshape(*idx.shape[1:], d)
