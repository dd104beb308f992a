"""File demo with the reference's command line (demoFile.py:20-70):

    python -m audiodec_b200.demo_file --model vctk_v1 -i input.wav -o output.wav [--cuda 0]

wav -> AudioDec.load_transmitter / load_receiver -> encode -> quantize -> lookup -> decode -> PCM_16 wav, on the GPU.
``--cuda -1`` (the reference's CPU mode) is refused: this implementation has no CPU path."""
from __future__ import annotations

import argparse
import os

import numpy as np
import torch

from audiodec_b200.utils.audiodec import AudioDec, assign_model
from audiodec_b200.wavio import read_wav, write_wav_pcm16


def run_file(audiodec, data: np.ndarray) -> np.ndarray:
    """(T, C) float -> (T, C) float through the four calls of demoFile.py:55-62 (channels ride the batch dimension)."""
    x = torch.tensor(np.expand_dims(data.transpose(1, 0), axis=1), dtype=torch.float).to(audiodec.tx_device)   # (T,C) -> (C,1,T)
    with torch.no_grad():
        z = audiodec.tx_encoder.encode(x)
        idx = audiodec.tx_encoder.quantize(z)
        zq = audiodec.rx_encoder.lookup(idx)
        y = audiodec.decoder.decode(zq)[:, :, :x.size(-1)]
    return y.squeeze(1).transpose(1, 0).cpu().numpy()


def _arguments(argv):
    """Same flags as the reference demo (demoFile.py:21-27)."""
    ap = argparse.ArgumentParser(description="wav -> AudioDec codec on an H100 -> wav")
    ap.add_argument("--model", default="libritts_v1", help="name from assign_model's table")
    ap.add_argument("-i", "--input", required=True, help="input wav (sample rate must match the model)")
    ap.add_argument("-o", "--output", required=True, help="output wav, written as PCM_16")
    ap.add_argument("--cuda", type=int, default=0, help="CUDA ordinal; negative (the reference's CPU mode) is refused")
    ap.add_argument("--num_threads", type=int, default=4, help="host threads for torch (only plumbing runs there)")
    return ap.parse_args(argv)


def main(argv=None):
    opt = _arguments(argv)
    if opt.cuda < 0:
        raise SystemExit("audiodec_b200 has no CPU path: pass --cuda <ordinal>")
    torch.set_num_threads(opt.num_threads)
    rate, enc_ckpt, dec_ckpt = assign_model(opt.model)          # NotImplementedError for an unknown name, like the reference
    if not os.path.exists(opt.input):
        raise ValueError(f"Input file {opt.input} does not exist!")
    dev = f"cuda:{opt.cuda}"
    codec = AudioDec(tx_device=dev, rx_device=dev)
    codec.load_transmitter(enc_ckpt)
    codec.load_receiver(enc_ckpt, dec_ckpt)
    audio, fs = read_wav(opt.input)
    assert fs == rate, f"data ({fs}Hz) is not matched to model ({rate}Hz)!"
    write_wav_pcm16(opt.output, run_file(codec, audio), fs)
    print(f"wrote {opt.output}: {audio.shape[0] / fs:.2f} s, {audio.shape[1]} channel(s)")


if __name__ == "__main__":
    main()
