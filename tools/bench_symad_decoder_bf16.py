#!/usr/bin/env python3
"""The symAD decoder in fp32 against its two bf16 modes on the decoder-only handle:

    python tools/bench_symad_decoder_bf16.py [--steps 5] [--regions 5]

  fp32    the full SymADStreamGenerator's decode (fp16-split three-product MMAs, fp32 activations): what bench.py's headline runs
  mode 1  SymADDecoderStreamGenerator.to(torch.bfloat16): bf16 conv operands, fp32 activations / state / decode I/O
  mode 2  SymADDecoderStreamGenerator.set_activation_dtype(torch.bfloat16): bf16 operands and bf16 activations / state / decode I/O

Shapes: the headline batch (vctk_sym, 64 x 48000 samples = 160 frames per stream, 48 kHz, uniform rows) and the streaming shape
of the 24 kHz model (libritts_sym, 256 streams x 1500 samples = 5 frames each, which takes the stacked-row path).  Per shape it times
the decode alone (zq already on the device, in the decoder's input dtype) and the whole encode -> quantize_fused -> decode step, the
three decoders in ONE process with their timed regions alternated, CUDA events around each region, median region reported.  Per
shape and decoder it also lists every decoder launch's CUDA-event time from one profiled decode (adec_profile_report), summed by
layer kind, with the 32-channel residual units (the fp32 handle's paired kernel, the bf16 modes' unpaired one) broken out.  The
GPU's name, power limit and SM clocks are read in the same run.  Prints one JSON object; writes nothing."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the timing loop and the clock sampler)
from bench_vocoder_bf16_act import gpu_info  # noqa: E402

SHAPES = {"headline_vctk_sym": (64, 48000, 48000), "stream_libritts_sym": (256, 1500, 24000)}
KINDS = ("fp32", "mode1", "mode2")


def build(dev):
    """Warmed tx / rx encoders and the three decoders (bin/stream.py:56-77).  vctk_sym and libritts_sym share the generator
    params; only the sample rate differs."""
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import SymADDecoderStreamGenerator, SymADStreamGenerator
    sd = S.symad_state_dict(seed=0)

    def gen(cls, mode=0):
        g = cls(**S.SYMAD_PARAMS)
        g.load_state_dict(sd)
        if mode == 1:
            g = g.to(torch.bfloat16)
        elif mode == 2:
            g = g.set_activation_dtype(torch.bfloat16)
        return g.eval().to(dev)

    tx, rx = gen(SymADStreamGenerator), gen(SymADStreamGenerator)
    decs = {"fp32": gen(SymADStreamGenerator), "mode1": gen(SymADDecoderStreamGenerator, 1), "mode2": gen(SymADDecoderStreamGenerator, 2)}
    tx.initial_encoder(8192, dev)
    warm = rx.initial_encoder(8192, dev)
    for d in decs.values():
        d.initial_decoder(warm)
    torch.cuda.synchronize(dev)
    return tx, decs


def layer_kind(name):
    if name.endswith(".conv2") and "res_units" in name:
        return "ru_split_1x1"
    if "res_units" in name:
        return "ru"
    if name == "decoder.conv1":
        return "conv1"
    if name == "decoder.conv2":
        return "head"
    return "convtr"


def launches(dec, zq, dev):
    """One profiled decode: [(op, ms)] and the ms per layer kind, the 32-channel units (decoder.conv_blocks.3) apart."""
    import torch
    dec.profile(True)
    dec.decode(zq)
    torch.cuda.synchronize(dev)
    rows = dec.profile_report()
    dec.profile(False)
    kinds = {}
    for name, ms, _ in rows:
        k = layer_kind(name)
        if k == "ru" and ".conv_blocks.3." in name:
            k = "ru32"
        kinds[k] = round(kinds.get(k, 0.0) + ms, 4)
    return {"total_ms": round(sum(r[1] for r in rows), 4), "by_kind_ms": kinds,
            "per_launch_ms": [(name, round(ms, 4)) for name, ms, _ in rows]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=5, help="steps per timed region")
    ap.add_argument("--regions", type=int, default=5, help="timed regions per decoder (median reported)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_symad_decoder_bf16: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda:0")
    sync = lambda: torch.cuda.synchronize(dev)
    out = {"gpu": gpu_info(0), "shapes": {}}
    tx, decs = build(dev)
    clocks = bench.ClockSampler(0)
    clocks.start()
    t0 = time.time()
    for shape, (B, T, sr) in SHAPES.items():
        gen = torch.Generator().manual_seed(4242)
        xs = [(0.1 * torch.randn(B, 1, T, generator=gen)).to(dev) for _ in range(4)]
        zqs = [tx.quantize_fused(tx.encode(x), want_idx=False)[2] for x in xs]
        zin = {k: [z.to(torch.bfloat16) if k == "mode2" else z for z in zqs] for k in KINDS}

        def step(k, i):
            return decs[k].decode(tx.quantize_fused(tx.encode(xs[i % 4]), want_idx=False)[2])

        res = {k: {"decode": [], "step": []} for k in KINDS}
        for k in KINDS:                                   # warm every shape of the timed windows
            for i in range(3):
                decs[k].decode(zin[k][i % 4])
                step(k, i)
        sync()
        for r in range(args.regions):
            for k in KINDS:
                ms, y = bench.time_device_loop(lambda i: decs[k].decode(zin[k][i % 4]), args.steps, 0, dev, sync)
                res[k]["decode"].append(ms / args.steps)
                assert torch.isfinite(y.float()).all()
            for k in KINDS:
                ms, _ = bench.time_device_loop(lambda i: step(k, i), args.steps, 0, dev, sync)
                res[k]["step"].append(ms / args.steps)
        o = {"batch": B, "samples": T, "sample_rate": sr, "frames_per_stream": zqs[0].shape[1], "decoders": {}}
        for k in KINDS:
            dm, sm = statistics.median(res[k]["decode"]), statistics.median(res[k]["step"])
            o["decoders"][k] = {"decode_ms": dm, "decode_regions_ms": [round(v, 3) for v in res[k]["decode"]],
                                "step_ms": sm, "step_regions_ms": [round(v, 3) for v in res[k]["step"]],
                                "decode_samples_per_s": B * T / (dm / 1e3), "launches": launches(decs[k], zin[k][0], dev)}
        for k in ("mode1", "mode2"):
            o[f"decode_speedup_{k}_over_fp32"] = o["decoders"]["fp32"]["decode_ms"] / o["decoders"][k]["decode_ms"]
            o[f"step_speedup_{k}_over_fp32"] = o["decoders"]["fp32"]["step_ms"] / o["decoders"][k]["step_ms"]
        out["shapes"][shape] = o
        del xs, zqs, zin
        torch.cuda.empty_cache()
    out["sm_clocks_during_timing"] = clocks.stop(t0, time.time())
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
