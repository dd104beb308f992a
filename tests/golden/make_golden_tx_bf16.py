#!/usr/bin/env python3
"""Golden vectors for the symAD transmitter in bf16 (the encoder-only handle), from the UNMODIFIED reference on CPU:

    python tests/golden/make_golden_tx_bf16.py          (build container only: needs /root/reference)

For each case one 0.25 s clip of 0.1 randn goes through the reference's `tx_encoder` twice, each freshly made and warmed by
load_transmitter (initial_encoder over `warm_len` zeros, bin/stream.py:61):
  <case>_z_fp32, <case>_idx_fp32 : the transmitter in fp32, and
  <case>_z_bf16, <case>_idx_bf16 : the same transmitter after `.to(torch.bfloat16)` fed x.bfloat16() - weights, pad_buffers, every
                                   activation and z in bf16 (torch CPU bf16 convolutions), its own bf16 RVQ on that z.
Cases: vctk_sym ("sym"), vctk_activate_sym ("aad") and vctk_c16h320_sym ("c16") one-shot encode + quantize, vctk_sym in 5-frame
chunks ("sym_stream"), and vctk_sym non-streaming Encoder.forward + Projector.forward ("sym_forward", zero left-pad).  The reference
defines no reduced-precision tolerance; the tests derive their bars from each case's pair.
"""
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.dont_write_bytecode = True
sys.path.insert(0, "/root/reference")
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)
warnings.filterwarnings("ignore")

from audiodec_b200 import synthetic as S  # noqa: E402
from make_golden import load_codec  # noqa: E402

torch.set_num_threads(4)
CHUNK_FRAMES = 5
WARM_LEN = 8192
MODELS = {"sym": "vctk_sym", "aad": "vctk_activate_sym", "c16": "vctk_c16h320_sym"}


def stream_tx(tx, x, chunk=None):
    """encode + quantize of x in one call, or in chunks of `chunk` samples -> (z (1, D, F) float, idx (Nq, F))"""
    with torch.no_grad():
        parts = [x] if chunk is None else [x[..., i:i + chunk] for i in range(0, x.shape[-1], chunk)]
        zs, ids = [], []
        for p in parts:
            z = tx.encode(p)
            ids.append(tx.quantize(z))
            zs.append(z.float())
        return torch.cat(zs, -1), torch.cat(ids, -1)


def report(name, z32, z16, i32, i16):
    err = (z16 - z32).abs()
    snr = 10 * torch.log10(z32.pow(2).mean() / (z16 - z32).pow(2).mean())
    print(f"{name}: reference bf16 z vs fp32 max abs {err.max().item():.4e}, SNR {snr.item():.1f} dB, z rms "
          f"{z32.pow(2).mean().sqrt().item():.3f}, indices equal {(i16 == i32).float().mean().item():.3f}, frames equal "
          f"{(i16 == i32).all(0).float().mean().item():.3f}, shape {tuple(z32.shape)}")


def main():
    scratch = tempfile.mkdtemp(prefix="adec_golden_tx_bf16_")
    torch.manual_seed(1337)
    x = 0.1 * torch.randn(1, 1, 12000)
    out = dict(x=x.numpy(), chunk_frames=CHUNK_FRAMES, warm_len=WARM_LEN)
    for name, model in MODELS.items():
        hop = int(np.prod(S.ENCODER_PARAMS.get(S.MODEL_TABLE[model][1], S.SYMAD_PARAMS)["enc_strides"]))
        for case, chunk in ((name, None), (name + "_stream", CHUNK_FRAMES * hop)) if name == "sym" else ((name, None),):
            z32, i32 = stream_tx(load_codec(scratch, model).tx_encoder, x, chunk)
            tx = load_codec(scratch, model).tx_encoder          # fresh warm state, then cast the whole transmitter (pad_buffers included)
            tx.to(torch.bfloat16)
            z16, i16 = stream_tx(tx, x.to(torch.bfloat16), chunk)
            report(case, z32, z16, i32, i16)
            out[case + "_z_fp32"], out[case + "_idx_fp32"] = z32.numpy(), i32.numpy()
            out[case + "_z_bf16"], out[case + "_idx_bf16"] = z16.numpy(), i16.numpy()
    # vctk_sym non-streaming Encoder.forward + Projector.forward (codecTest.py:78-90), zero left-pad
    g = load_codec(scratch, "vctk_sym").tx_encoder
    with torch.no_grad():
        z32 = g.projector(g.encoder(x))
        i32 = g.quantize(z32)
        g.to(torch.bfloat16)
        z16 = g.projector(g.encoder(x.to(torch.bfloat16)))
        i16 = g.quantize(z16)
        z16 = z16.float()
    report("sym_forward", z32, z16, i32, i16)
    out["sym_forward_z_fp32"], out["sym_forward_idx_fp32"] = z32.numpy(), i32.numpy()
    out["sym_forward_z_bf16"], out["sym_forward_idx_bf16"] = z16.numpy(), i16.numpy()
    digests = {"digest_" + name: S.state_dict_digest(S.symad_state_dict(S.ENCODER_PARAMS.get(S.MODEL_TABLE[model][1], S.SYMAD_PARAMS), seed=0))
               for name, model in MODELS.items()}
    np.savez_compressed(os.path.join(HERE, "tx_bf16.npz"), **out, **digests, torch=torch.__version__, threads=4)


if __name__ == "__main__":
    main()
