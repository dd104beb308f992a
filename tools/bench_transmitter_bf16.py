#!/usr/bin/env python3
"""The symAD transmitter (encode + quantize) in fp32 against the encoder-only handle's two bf16 modes:

    python tools/bench_transmitter_bf16.py [--steps 5] [--regions 5] [--parent-tree DIR [--bench-steps 50]]

  fp32    the full SymADStreamGenerator's encode + quantize (fp16-split three-product MMAs): what bench.py's headline runs
  mode 1  SymADEncoderStreamGenerator.to(torch.bfloat16): bf16 conv operands, fp32 x / activations / state / z, the same RVQ
  mode 2  SymADEncoderStreamGenerator.set_activation_dtype(torch.bfloat16): bf16 x / activations / state / z as well, the RVQ on
          the widened bf16 z

Shapes: the headline batch (vctk_sym, 64 x 48000 samples, uniform rows) and the streaming shape of the 24 kHz model (libritts_sym,
256 streams x 1500 samples, stacked rows, packed bytes as a wire transmitter sends them).  The transmitters run in ONE process with
their timed regions alternated, CUDA events around each region, median region reported.  Per shape and transmitter it also sums
one profiled encode's launch times by layer kind.  It also times the AD v1 step of BASELINE configs[2] (128 x 48000, the v1 vocoder
with bf16 activations) with the fp32 transmitter against the mode-2 one, alternated the same way.  With --parent-tree (a checkout
of the parent commit, built), bench.py runs twice from that tree and twice from this one, alternated, in child processes that run
before this process takes the GPU, and its ms per step are reported (each tree loads its own library and Python package).  The
GPU's name, power limit and SM clocks are read in the same run.  Prints one JSON object; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the timing loop and the clock sampler)
from bench_vocoder_bf16_act import gpu_info  # noqa: E402

SHAPES = {"headline_vctk_sym": (64, 48000, 48000, False), "stream_libritts_sym": (256, 1500, 24000, True)}
KINDS = ("fp32", "mode1", "mode2")


def build(dev):
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import SymADEncoderStreamGenerator, SymADStreamGenerator
    sd = S.symad_state_dict(seed=0)
    txs = {}
    for k, cls in (("fp32", SymADStreamGenerator), ("mode1", SymADEncoderStreamGenerator), ("mode2", SymADEncoderStreamGenerator)):
        g = cls(**S.SYMAD_PARAMS)
        g.load_state_dict(sd)
        if k == "mode1":
            g = g.to(torch.bfloat16)
        elif k == "mode2":
            g = g.set_activation_dtype(torch.bfloat16)
        txs[k] = g.eval().to(dev)
        txs[k].initial_encoder(8192, dev)
    torch.cuda.synchronize(dev)
    return txs


def layer_kind(name):
    if name == "encoder.conv":
        return "stem"
    if name.endswith(".conv2") and "res_units" in name:
        return "ru_split_1x1"
    if "res_units" in name:
        return "ru32" if ".conv_blocks.0." in name else "ru"
    if name.startswith("projector"):
        return "projector"
    return "strided"


def launches(tx, x, dev):
    import torch
    tx.profile(True)
    tx.encode(x)
    torch.cuda.synchronize(dev)
    rows = tx.profile_report()
    tx.profile(False)
    kinds = {}
    for name, ms, _ in rows:
        k = layer_kind(name)
        kinds[k] = round(kinds.get(k, 0.0) + ms, 4)
    return {"encode_total_ms": round(sum(r[1] for r in rows), 4), "by_kind_ms": kinds}


def configs2_step(txs, args, dev, sync):
    """BASELINE configs[2]: 128 x 48000 through encode -> quantize -> lookup -> the AD v1 vocoder with bf16 activations, with the fp32
    transmitter and with the mode-2 one (the receiver is the same: rx lookup in bf16, then the vocoder)"""
    import torch
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from bench_vocoder_bf16_act import build as build_v1
    _, rx, dec = build_v1(2, dev)
    gen = torch.Generator().manual_seed(4243)
    xs = [(0.1 * torch.randn(128, 1, 48000, generator=gen)).to(dev) for _ in range(2)]

    def step(k, i):
        tx = txs[k]
        return dec.decode(rx.lookup(tx.quantize(tx.encode(xs[i % 2])), dtype=torch.bfloat16))

    res = {k: [] for k in ("fp32", "mode2")}
    for k in res:
        step(k, 0)
    sync()
    for r in range(args.regions):
        for k in res:
            ms, _ = bench.time_device_loop(lambda i: step(k, i), args.steps, 0, dev, sync)
            res[k].append(ms / args.steps)
    o = {k: {"step_ms": statistics.median(v), "regions_ms": [round(x, 3) for x in v]} for k, v in res.items()}
    o["speedup_mode2_tx_over_fp32_tx"] = o["fp32"]["step_ms"] / o["mode2"]["step_ms"]
    del xs
    torch.cuda.empty_cache()
    return o


def bench_py_ab(parent_tree, steps):
    """bench.py's headline ms per step from the parent tree and from this one, alternated twice, each in its own process"""
    out = {"parent": [], "this": []}
    env = dict(os.environ)
    env.pop("ADEC_LIB_PATH", None)
    for _ in range(2):
        for which in ("parent", "this"):
            tree = os.path.abspath(parent_tree) if which == "parent" else ROOT
            r = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", "10"],
                               env=env, capture_output=True, text=True, cwd=tree)
            lines = [ln for ln in r.stdout.splitlines() if ln.strip().startswith("{")]
            if r.returncode or not lines:
                raise RuntimeError(f"bench.py on {which} failed (exit {r.returncode}): {r.stderr[-2000:]}")
            out[which].append(round(json.loads(lines[-1])["ms_per_step"], 3))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=5, help="steps per timed region")
    ap.add_argument("--regions", type=int, default=5, help="timed regions per transmitter (median reported)")
    ap.add_argument("--parent-tree", default=None, help="a built checkout of the parent commit: also time bench.py there and here")
    ap.add_argument("--bench-steps", type=int, default=50, help="bench.py --steps for --parent-tree")
    args = ap.parse_args()
    ab = bench_py_ab(args.parent_tree, args.bench_steps) if args.parent_tree else None   # before this process takes the GPU
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_transmitter_bf16: needs a CUDA device (there is no CPU measurement)")
    dev = torch.device("cuda:0")
    sync = lambda: torch.cuda.synchronize(dev)
    out = {"gpu": gpu_info(0), "shapes": {}}
    txs = build(dev)
    clocks = bench.ClockSampler(0)
    clocks.start()
    t0 = time.time()
    for shape, (B, T, sr, wire) in SHAPES.items():
        gen = torch.Generator().manual_seed(4242)
        xs = [(0.1 * torch.randn(B, 1, T, generator=gen)).to(dev) for _ in range(4)]

        def step(k, i):
            z = txs[k].encode(xs[i % 4])
            if wire:
                return txs[k].quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)[1]
            return txs[k].quantize(z)

        res = {k: [] for k in KINDS}
        for k in KINDS:
            for i in range(3):
                step(k, i)
        sync()
        for r in range(args.regions):
            for k in KINDS:
                ms, _ = bench.time_device_loop(lambda i: step(k, i), args.steps, 0, dev, sync)
                res[k].append(ms / args.steps)
        ref = step("fp32", 0)
        o = {"batch": B, "samples": T, "sample_rate": sr, "wire": wire, "tx": {}}
        for k in ("mode1", "mode2"):
            o[f"frames_with_equal_codes_{k}_vs_fp32"] = (step(k, 0) == ref).all(-1 if wire else 0).float().mean().item()
        for k in KINDS:
            m = statistics.median(res[k])
            o["tx"][k] = {"encode_quantize_ms": m, "regions_ms": [round(v, 3) for v in res[k]], "launches": launches(txs[k], xs[0], dev)}
        for k in ("mode1", "mode2"):
            o[f"speedup_{k}_over_fp32"] = o["tx"]["fp32"]["encode_quantize_ms"] / o["tx"][k]["encode_quantize_ms"]
        out["shapes"][shape] = o
        del xs
        torch.cuda.empty_cache()
    out["configs2_ad_v1_step"] = configs2_step(txs, args, dev, sync)
    out["sm_clocks_during_timing"] = clocks.stop(t0, time.time())
    if ab:
        out["bench_py_parent_vs_this"] = ab
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
