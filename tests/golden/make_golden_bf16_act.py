#!/usr/bin/env python3
"""Golden vectors for the vocoder's bf16-activation mode (compute_dtype 2), from the UNMODIFIED reference on CPU:

    python tests/golden/make_golden_bf16_act.py          (build container only: needs /root/reference)

One 0.25 s clip (the clip of make_golden_bf16.py) goes through the reference's own fp32 load_transmitter / load_receiver / encode /
quantize / lookup; its zq then drives each vocoder case twice:
  <case>_y_fp32 : the vocoder in fp32 (the oracle every other test uses), and
  <case>_y_bf16 : the same vocoder after `.to(torch.bfloat16)` fed zq.bfloat16() - weights, stats, pad_buffers and every activation
                  in bf16 (torch CPU bf16 convolutions): what the reference returns when asked for bf16.
Cases: v1 / v0 (MultiReceptiveField) / v2 one-shot StreamGenerator.decode, v1 decode in 5-frame (1500-sample) chunks, and v1
non-streaming Generator.forward (channels-first input, zero left-pad).  The reference defines no reduced-precision tolerance; the test
derives its bar from each case's pair.  `warm_zq` is what load_receiver feeds to decoder.initial_decoder (bin/stream.py:70,76).
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
CHUNK_FRAMES = 5                       # 1500 samples at hop 300 (demoStream.py:28 default frame size)


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
    from models.vocoder.HiFiGAN import Generator
    scratch = tempfile.mkdtemp(prefix="adec_golden_bf16_act_")
    torch.manual_seed(1337)
    x = 0.1 * torch.randn(1, 1, 12000)
    a = load_codec(scratch, "vctk_v1")
    with torch.no_grad():
        zq = a.rx_encoder.lookup(a.tx_encoder.quantize(a.tx_encoder.encode(x)))          # (1, 40, 64)
        fresh = a._load_encoder(os.path.join(scratch, "exp/autoencoder/symAD_vctk_48000_hop300/checkpoint-200000steps.pkl")).eval()
        warm_zq = fresh.initial_encoder(8192, "cpu")
    out = dict(x=x.numpy(), zq=zq.numpy(), warm_zq=warm_zq.numpy(), chunk_frames=CHUNK_FRAMES)
    for case, model, chunk in (("v1", "vctk_v1", None), ("v1_stream", "vctk_v1", CHUNK_FRAMES), ("v0", "vctk_v0", None),
                               ("v2", "vctk_v2", None)):
        y32 = stream_decode(load_codec(scratch, model).decoder, zq, chunk)
        b = load_codec(scratch, model)                  # fresh warm state, then cast the whole vocoder (pad_buffers included)
        b.decoder.to(torch.bfloat16)
        y16 = stream_decode(b.decoder, zq.to(torch.bfloat16), chunk)
        report(case, y32, y16)
        out[case + "_y_fp32"], out[case + "_y_bf16"] = y32.numpy(), y16.numpy()
    # v1 non-streaming Generator.forward (HiFiGAN.py:141-161), as codecTest.py:91-94 calls it: zq channels-first
    g = Generator(**S.HIFIGAN_V1_PARAMS)                # cwd is the scratch tree: the cwd-relative stats path resolves
    g.load_state_dict(S.hifigan_state_dict(seed=1))
    g.eval()
    c = zq.transpose(1, 2).contiguous()
    with torch.no_grad():
        y32 = g(c)
        g.to(torch.bfloat16)
        y16 = g(c.to(torch.bfloat16)).float()
    report("v1_forward", y32, y16)
    out["v1_forward_y_fp32"], out["v1_forward_y_bf16"] = y32.numpy(), y16.numpy()
    np.savez_compressed(os.path.join(HERE, "bf16_act.npz"), **out,
                        enc_digest=S.state_dict_digest(S.symad_state_dict(seed=0)), dec_digest=S.state_dict_digest(S.hifigan_state_dict(seed=1)),
                        torch=torch.__version__, threads=4)


if __name__ == "__main__":
    main()
