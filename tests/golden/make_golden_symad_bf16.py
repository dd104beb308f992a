#!/usr/bin/env python3
"""Golden vectors for the symAD decoder's bf16 modes (the decoder-only handle, compute_dtype 1 and 2), from the UNMODIFIED reference
on CPU:

    python tests/golden/make_golden_symad_bf16.py          (build container only: needs /root/reference)

For each model one 0.25 s clip goes through the reference's own fp32 load_transmitter / load_receiver / encode / quantize / lookup;
its zq then drives the receiver's `decoder` object twice:
  <case>_y_fp32 : the decoder in fp32, and
  <case>_y_bf16 : the same decoder after `.to(torch.bfloat16)` fed zq.bfloat16() - weights, pad_buffers and every activation in
                  bf16 (torch CPU bf16 convolutions): what the reference returns when asked for bf16.
Cases: vctk_sym ("sym"), vctk_activate_sym ("aad") and vctk_c16h320_sym ("c16") one-shot StreamGenerator.decode, vctk_sym decode in
5-frame chunks ("sym_stream"), and vctk_sym non-streaming Decoder.forward ("sym_forward": channels-first zq, zero left-pad).  The
reference defines no reduced-precision tolerance; the tests derive their bar from each case's pair.  `<model>_zq` is the model's
clip, `<model>_warm_zq` what load_receiver's warm-up feeds to decoder.initial_decoder (bin/stream.py:70,76).
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
MODELS = {"sym": "vctk_sym", "aad": "vctk_activate_sym", "c16": "vctk_c16h320_sym"}


def stream_decode(dec, zq, chunk=None):
    with torch.no_grad():
        if chunk is None:
            return dec.decode(zq).float()
        return torch.cat([dec.decode(zq[:, i:i + chunk]).float() for i in range(0, zq.shape[1], chunk)], -1)


def report(name, y32, y16):
    err = (y16 - y32).abs()
    snr = 10 * torch.log10(y32.pow(2).mean() / (y16 - y32).pow(2).mean())
    print(f"{name}: reference bf16 vs fp32 max abs {err.max().item():.4e}, SNR {snr.item():.1f} dB, shape {tuple(y32.shape)}")


def main():
    scratch = tempfile.mkdtemp(prefix="adec_golden_symad_bf16_")
    torch.manual_seed(1337)
    x = 0.1 * torch.randn(1, 1, 12000)
    out = dict(x=x.numpy(), chunk_frames=CHUNK_FRAMES)
    for name, model in MODELS.items():
        a = load_codec(scratch, model)
        etag = S.MODEL_TABLE[model][1]
        with torch.no_grad():
            zq = a.rx_encoder.lookup(a.tx_encoder.quantize(a.tx_encoder.encode(x)))
            fresh = a._load_encoder(os.path.join(scratch, f"exp/autoencoder/{etag}/checkpoint-{S.MODEL_TABLE[model][2]}steps.pkl")).eval()
            warm_zq = fresh.initial_encoder(8192, "cpu")
        out[name + "_zq"], out[name + "_warm_zq"] = zq.numpy(), warm_zq.numpy()
        for case, chunk in ((name, None), (name + "_stream", CHUNK_FRAMES)) if name == "sym" else ((name, None),):
            y32 = stream_decode(load_codec(scratch, model).decoder, zq, chunk)
            b = load_codec(scratch, model)                  # fresh warm state, then cast the whole decoder (pad_buffers included)
            b.decoder.to(torch.bfloat16)
            y16 = stream_decode(b.decoder, zq.to(torch.bfloat16), chunk)
            report(case, y32, y16)
            out[case + "_y_fp32"], out[case + "_y_bf16"] = y32.numpy(), y16.numpy()
    # vctk_sym non-streaming Decoder.forward (decoder.py:135-140), as codecTest.py:91-94 calls it: zq channels-first
    dec = load_codec(scratch, "vctk_sym").decoder.decoder
    c = torch.from_numpy(out["sym_zq"]).transpose(1, 2).contiguous()
    with torch.no_grad():
        y32 = dec(c)
        dec.to(torch.bfloat16)
        y16 = dec(c.to(torch.bfloat16)).float()
    report("sym_forward", y32, y16)
    out["sym_forward_y_fp32"], out["sym_forward_y_bf16"] = y32.numpy(), y16.numpy()
    digests = {"digest_" + name: S.state_dict_digest(S.symad_state_dict(S.ENCODER_PARAMS.get(S.MODEL_TABLE[model][1], S.SYMAD_PARAMS), seed=0))
               for name, model in MODELS.items()}
    np.savez_compressed(os.path.join(HERE, "symad_bf16.npz"), **out, **digests, torch=torch.__version__, threads=4)


if __name__ == "__main__":
    main()
