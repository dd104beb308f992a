"""Batched codecTest.py: transcode a folder of wav files through the non-streaming codec, many utterances per launch sequence.

    python -m audiodec_b200.codec_test --encoder exp/autoencoder/<tag>/checkpoint-<n>steps.pkl \\
        --decoder exp/vocoder/<tag>/checkpoint-<n>steps.pkl --output_dir output [--subset clean_test] [--subset_num -1] \\
        [--specific_folder False] [--cuda 0] [--batch_seconds 600]

Same flags, wav discovery, output directory naming and `<utt_id>_output.wav` PCM_16 files as the reference's codecTest.py
(codecTest.py:35-48, :99-127; bin/test.py:89-106).  The reference runs encode -> decode once per file; here the files, read in sorted
order, are packed into varlen batches of at most --batch_seconds of audio (OfflineCodec.encode_many / decode_many), and every
utterance comes out as a per-file call would give it, so the output does not depend on the batching.  ``--cuda -1`` (the reference's
CPU mode) is refused: this implementation has no CPU path."""
from __future__ import annotations

import argparse
import fnmatch
import logging
import os
import sys
import time

import torch
import yaml

from audiodec_b200.codec import HiFiGANStreamGenerator, OfflineCodec, SymADStreamGenerator
from audiodec_b200.wavio import read_wav, write_wav_pcm16

_AUTOENCODER_TYPES = ("symAudioDec", "symAudioDecUniv")      # codecTest.py:54-57
_VOCODER_TYPES = ("HiFiGAN", "UnivNet")                      # codecTest.py:66-71


def load_config(checkpoint, config_name="config.yml"):
    """bin/utils.py:17-22: the config.yml beside the checkpoint."""
    with open(os.path.join(os.path.dirname(checkpoint), config_name)) as f:
        return yaml.load(f, Loader=yaml.Loader)


def find_wavs(data_path, subset_num=-1):
    """dataloader/dataset.py:63-84: *.wav under data_path (recursive), sorted, the first subset_num if > 0 -> [(utt_id, path)]."""
    files = []
    for root, _, names in os.walk(data_path, followlinks=True):
        files += [os.path.join(root, n) for n in fnmatch.filter(names, "*.wav")]
    files = sorted(files)
    if subset_num > 0:
        files = files[:subset_num]
    if not files:
        raise ValueError(f"no *.wav files under {data_path}")
    return [(os.path.splitext(os.path.basename(f))[0], f) for f in files]


def output_dir(encoder, decoder, encoder_config, subset, output_name, specific_folder="False"):
    """codecTest.py:99-115."""
    if specific_folder == "True":
        return output_name
    enc_name = os.path.dirname(encoder).split("/")[-1]
    dec_name = os.path.dirname(decoder).split("/")[-1]
    enc_ckpt = os.path.basename(encoder).split("steps")[0].split("-")[-1]
    dec_ckpt = os.path.basename(decoder).split("steps")[0].split("-")[-1]
    return os.path.join(output_name, f"{enc_name}-{dec_name}_{enc_ckpt}-{dec_ckpt}", encoder_config["data"]["subset"][subset])


def _load_generator(checkpoint, config, allowed):
    kind = config.get("model_type", "symAudioDec")
    if kind in _AUTOENCODER_TYPES:
        cls = SymADStreamGenerator
    elif kind in _VOCODER_TYPES and allowed == "decoder":
        cls = HiFiGANStreamGenerator
    else:
        raise NotImplementedError(f"{allowed.capitalize()} {kind} is not supported!")
    gen = cls(**config["generator_params"])
    gen.load_state_dict(torch.load(checkpoint, map_location="cpu")["model"]["generator"])
    return gen


def batches(items, sample_rate, batch_seconds):
    """Consecutive runs of (utt_id, audio) holding at most batch_seconds of audio (at least one file each)."""
    cap = batch_seconds * sample_rate
    run, total = [], 0
    for item in items:
        n = item[1].shape[0] * item[1].shape[1]
        if run and total + n > cap:
            yield run
            run, total = [], 0
        run.append(item)
        total += n
    if run:
        yield run


def _arguments(argv):
    ap = argparse.ArgumentParser(description="Transcode a wav folder through the AudioDec codec on an H100, many files per batch")
    ap.add_argument("--subset", type=str, default="clean_test")
    ap.add_argument("--subset_num", type=int, default=-1)
    ap.add_argument("--encoder", type=str, required=True)
    ap.add_argument("--decoder", type=str, required=True)
    ap.add_argument("--output_dir", type=str, required=True)
    ap.add_argument("--specific_folder", choices=("True", "False"), default="False")
    ap.add_argument("--cuda", type=int, default=0, help="CUDA ordinal; negative (the reference's CPU mode) is refused")
    ap.add_argument("--batch_seconds", type=float, default=600.0, help="most audio (seconds, all channels) packed into one batch")
    return ap.parse_args(argv)


def main(argv=None):
    args = _arguments(argv)
    logging.basicConfig(level=logging.INFO, stream=sys.stdout, format="%(asctime)s (%(module)s:%(lineno)d) %(levelname)s: %(message)s")
    if args.cuda < 0:
        raise SystemExit("audiodec_b200 has no CPU path: pass --cuda <ordinal>")
    if args.batch_seconds <= 0:
        raise SystemExit("--batch_seconds must be > 0")
    for ckpt in (args.encoder, args.decoder):
        if not os.path.exists(ckpt):
            raise SystemExit(f"{ckpt} does not exist!")
    enc_cfg, dec_cfg = load_config(args.encoder), load_config(args.decoder)
    if args.subset not in (enc_cfg.get("data") or {}).get("subset", {}):
        raise SystemExit(f"the encoder's config.yml names no data.path / data.subset['{args.subset}'] (codecTest.py:35-48)")
    data_path = os.path.join(enc_cfg["data"]["path"], enc_cfg["data"]["subset"][args.subset])
    if not os.path.exists(data_path):
        raise SystemExit(f"{data_path} does not exist!")
    utts = find_wavs(data_path, args.subset_num)
    logging.info(f"The number of utterances = {len(utts)}.")

    dev = torch.device("cuda", args.cuda)
    encoder = _load_generator(args.encoder, enc_cfg, "encoder").eval().to(dev)
    decoder = _load_generator(args.decoder, dec_cfg, "decoder").eval().to(dev)
    logging.info(f"Loaded Encoder from {args.encoder} and Decoder from {args.decoder}.")
    if enc_cfg["generator_params"].get("input_channels", 1) > 1:
        raise NotImplementedError("only mono generators are built (codecTest.py's multi-channel mode needs input_channels > 1)")
    codec = OfflineCodec(encoder, decoder)
    outdir = output_dir(args.encoder, args.decoder, enc_cfg, args.subset, args.output_dir, args.specific_folder)
    os.makedirs(outdir, exist_ok=True)

    sr = dec_cfg["sampling_rate"]
    total_rtf, n = 0.0, 0
    with torch.no_grad():
        for run in batches(((u, read_wav(p)[0]) for u, p in utts), sr, args.batch_seconds):
            start = time.time()
            ys = codec.decode_many(codec.encode_many([a for _, a in run]))
            ys = [y.squeeze(1).transpose(1, 0).float().cpu().numpy() for y in ys]       # (T, C), like bin/test.py:94
            rtf = (time.time() - start) / (sum(len(y) for y in ys) / sr)
            for (utt_id, _), y in zip(run, ys):
                write_wav_pcm16(os.path.join(outdir, f"{utt_id}_output.wav"), y, sr)
            total_rtf += rtf * len(run)
            n += len(run)
    logging.info("Finished generation of %d utterances (RTF = %.03f)." % (n, total_rtf / n))
    return outdir


if __name__ == "__main__":
    main()
