#!/usr/bin/env python3
"""One step of each vocoder workload, written to files so that two builds of the library can be compared bit for bit:

    ADEC_LIB_PATH=<library A> python tools/step_outputs.py DIR_A
    ADEC_LIB_PATH=<library B> python tools/step_outputs.py DIR_B
    python tools/step_outputs.py --compare DIR_A DIR_B

Workloads (seeded inputs, synthetic checkpoints): v1 (symAD encoder + HiFi-GAN v1, 8 x 48000), v1_bf16 mode 1 (`decoder.to(torch.bfloat16)`)
and mode 2 (`set_activation_dtype(torch.bfloat16)`, bf16 decode I/O), and stream_v1 (256 streams, two consecutive 1500-sample chunks, so
the second reads the causal state the first wrote).  Each writes waveform, code indices, z and zq as .npy (bf16 tensors as their 16-bit
patterns).  --compare reports every file whose bytes differ and exits 1 if any does.  The headline workload has bench.py --dump-outputs.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def save(out_dir, prefix, tensors):
    import numpy as np
    import torch
    for name, t in tensors.items():
        t = t.detach()
        if t.dtype == torch.bfloat16:
            t = t.view(torch.int16)
        np.save(os.path.join(out_dir, f"{prefix}_{name}.npy"), t.cpu().numpy())


def run(out_dir):
    import torch
    import bench
    import bench_vocoder_bf16_act      # its build(mode, dev): the two bf16 modes, warmed
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(2024)
    x = (0.1 * torch.randn(8, 1, 48000, generator=gen)).to(dev)
    xs = (0.1 * torch.randn(256, 1, 3000, generator=gen)).to(dev)
    for name in ("v1", "v1_bf16_mode1", "v1_bf16_mode2"):
        tx, rx, dec = bench.build_codec("v1", dev) if name == "v1" else bench_vocoder_bf16_act.build(int(name[-1]), dev)
        y, idx, z, zq = bench.codec_step(tx, rx, dec, x)
        save(out_dir, name, {"waveform": y, "code_indices": idx, "z": z, "zq": zq})
        del tx, rx, dec
    tx, rx, dec = bench.build_codec("stream_v1", dev)
    for c in range(2):
        y, idx, z, zq = bench.codec_step(tx, rx, dec, xs[:, :, c * 1500:(c + 1) * 1500].contiguous())
        save(out_dir, f"stream_v1_chunk{c}", {"waveform": y, "code_indices": idx, "z": z, "zq": zq})
    torch.cuda.synchronize(dev)
    print(f"wrote {len(os.listdir(out_dir))} files to {out_dir}")


def compare(a, b):
    names = sorted(set(os.listdir(a)) | set(os.listdir(b)))
    bad = []
    for n in names:
        pa, pb = os.path.join(a, n), os.path.join(b, n)
        if not (os.path.exists(pa) and os.path.exists(pb)):
            bad.append(f"{n}: missing on one side")
            continue
        with open(pa, "rb") as fa, open(pb, "rb") as fb:
            if fa.read() != fb.read():
                bad.append(f"{n}: bytes differ")
    for line in bad:
        print(line)
    print(f"{len(names) - len(bad)} of {len(names)} files byte-identical")
    return 1 if bad or not names else 0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("dirs", nargs="+", help="output directory, or the two directories to compare")
    ap.add_argument("--compare", action="store_true")
    args = ap.parse_args()
    if args.compare:
        if len(args.dirs) != 2:
            ap.error("--compare takes two directories")
        sys.exit(compare(*args.dirs))
    run(args.dirs[0])


if __name__ == "__main__":
    main()
