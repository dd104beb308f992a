#!/usr/bin/env python3
"""Generate tests/golden/stream_state.npz by running the UNMODIFIED reference (CPU, needs /root/reference):

    python tests/golden/make_golden_state.py

For vctk_v1, vctk_v0 and vctk_activate_sym (synthetic weights, load_codec of make_golden.py): a seeded 12000-sample clip is streamed
in 1500-sample chunks through encode -> quantize -> lookup -> decode.  After chunk 4 the full state_dict() of tx_encoder and decoder is
recorded: every key with its shape and dtype, and for every pad_buffer (C, P) the whole-buffer max |v| and fp64 sum, and the values
of every s-th channel (s = ceil(C * P / SAMPLE), all P rows; SAMPLE values or fewer per buffer).  The full values of all six dicts are
1.8 MB of incompressible floats; the channel sample keeps the fixture small while a transposed, stale or misplaced buffer still differs
at sampled positions.  Those dicts are then loaded into freshly loaded objects, and chunks 5-8 are run by both the fresh and the original
objects; the reference's own resume is exact, which is checked here.  The fixture holds chunks 5-8's indices and waveform, and the
weight digests.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (puts the reference and the repository on sys.path)
from audiodec_b200 import synthetic as S  # noqa: E402

MODELS = ("vctk_v1", "vctk_v0", "vctk_activate_sym")
CHUNK, N_CHUNKS, SPLIT = 1500, 8, 4
SAMPLE = 256


def channel_stride(c, p):
    """the channel stride of a pad_buffer's stored sample (tests/test_stream_state_gpu.py reads it back from the fixture)"""
    return max(1, -(-c * p // SAMPLE))


def main():
    scratch = tempfile.mkdtemp(prefix="adec_golden_state_")
    out = dict(torch=torch.__version__, chunk=CHUNK, split=SPLIT)
    torch.manual_seed(2024)
    x = 0.1 * torch.randn(1, 1, CHUNK * N_CHUNKS)
    out["x"] = x.numpy()
    for model in MODELS:
        a = MG.load_codec(scratch, model)
        for c in range(SPLIT):
            MG.run_path(a, x[:, :, c * CHUNK:(c + 1) * CHUNK])
        sds = {"tx": a.tx_encoder.state_dict(), "dec": a.decoder.state_dict()}
        for who, sd in sds.items():
            out[f"{model}/{who}/keys"] = np.array(list(sd.keys()))
            out[f"{model}/{who}/shapes"] = np.array([",".join(map(str, v.shape)) for v in sd.values()])
            out[f"{model}/{who}/dtypes"] = np.array([str(v.dtype) for v in sd.values()])
            keys, stats, vals = [], [], []
            for k, v in sd.items():
                if k.endswith("pad_buffer"):
                    v = v.numpy().astype(np.float32)
                    st = channel_stride(v.shape[1], v.shape[2])
                    keys.append(k)
                    stats.append([st, np.abs(v).max(), v.astype(np.float64).sum()])
                    vals.append(v[:, ::st, :].reshape(-1))
            # one array each: pad_buffer keys, (stride, max |v|, sum) per key, and the samples (1, ceil(C / s), P) one after the other
            out[f"{model}/{who}/pb_keys"] = np.array(keys)
            out[f"{model}/{who}/pb_stats"] = np.array(stats, dtype=np.float64)
            out[f"{model}/{who}/pb_vals"] = np.concatenate(vals)
        b = MG.load_codec(scratch, model)
        b.tx_encoder.load_state_dict({k: v.clone() for k, v in sds["tx"].items()})
        b.decoder.load_state_dict({k: v.clone() for k, v in sds["dec"].items()})
        idx, ys = [], []
        for c in range(SPLIT, N_CHUNKS):
            xc = x[:, :, c * CHUNK:(c + 1) * CHUNK]
            _, ia, _, ya = MG.run_path(a, xc)
            _, ib, _, yb = MG.run_path(b, xc)
            assert torch.equal(ia, ib) and torch.equal(ya, yb), f"{model}: the reference's own resume is not exact"
            idx.append(ia), ys.append(ya)
        out[f"{model}/idx"] = torch.cat(idx, -1).numpy()
        out[f"{model}/y"] = torch.cat(ys, -1).numpy()
        print(model, "tx keys", len(sds["tx"]), "dec keys", len(sds["dec"]), "y absmax", torch.cat(ys, -1).abs().max().item())
    out["enc_digest"] = S.state_dict_digest(S.symad_state_dict(seed=0))
    out["aad_digest"] = S.state_dict_digest(S.symad_state_dict(S.SYMAAD_PARAMS, seed=0))
    out["v1_digest"] = S.state_dict_digest(S.hifigan_state_dict(seed=1))
    out["v0_digest"] = S.state_dict_digest(S.hifigan_state_dict(S.HIFIGAN_V0_PARAMS, seed=1))
    path = os.path.join(HERE, "stream_state.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
