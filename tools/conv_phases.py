#!/usr/bin/env python3
"""Where the conv engine's cycles go, per launch of one warmed headline step (symAD, 64 x 48000, fp32):

    python tools/conv_phases.py [--lib PATH] [--build-dir DIR] [--batch 64] [--samples 48000] [--json OUT]

Builds the library with -DADEC_PHASES into its own directory (a temporary one unless --build-dir is given; --lib uses an already
instrumented library instead), loads it through ADEC_LIB_PATH in a child process with ADEC_KTRACE=1, runs two warm-up steps and one
traced step, and prints each wg_conv_kernel launch of the traced step with the shares of its role's cycles per phase:

  consumers   win (waiting for a window piece), wgt (waiting for a weight stage), mma (MMA groups and their partial sums),
              mid (the fused unit's intermediate), epi (the epilogue: scale, bias, residual, stores)
  producers   free (waiting for a free window buffer), load (global loads until their data is there), conv (activation, operand split,
              shared-memory stores)
  weights     wfree: the weight producer's share of time spent waiting for a free stage

The counters are summed over the CTAs of a launch (csrc/kernels.cuh, ADEC_PHASES).  The instrumented kernels are slower than the
default build, so the shares, not the times, are the result.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KT_REC = 16            # values per record of an ADEC_PHASES library (csrc/kernels.cuh)
PHASES = ["win", "wgt", "mma", "mid", "epi", "free", "load", "conv", "wfree", "wissue"]
CONSUMER, PRODUCER = PHASES[:5], PHASES[5:8]
PREC = {1: "bf16", 2: "tf32", 3: "f16"}


def build(build_dir):
    import __graft_entry__ as g
    lib = os.path.join(build_dir, "libaudiodec_b200.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + g.NVCC_FLAGS + ["-DADEC_PHASES", "-o", lib, os.path.join(ROOT, "audiodec_b200", "csrc", "adec.cu")])
    return lib


def describe(d, tout):
    nt, cin, cout = d & 0xFF, (d >> 32) & 0xFFFF, (d >> 48) & 0xFFFF
    ktaps, dil = (d >> 16) & 0xFF, (d >> 24) & 0xFF
    kind = "fused RU" if d >> 8 & 1 else ("conv+res" if d >> 9 & 1 else "conv")
    flags = "".join(f" {n}" for b, n in ((10, "paired"), (11, "varlen"), (12, "bf16-io")) if d >> b & 1)
    return f"{kind} {cin}->{cout} k{ktaps} d{dil} NT{nt} {PREC.get(d >> 13 & 3, '?')}{flags} Tout {tout}"


def child(batch, samples):
    import ctypes
    import torch
    import bench
    from audiodec_b200 import _lib
    dev = torch.device("cuda:0")
    tx, rx, dec = bench.build_codec("symad", dev)
    x = (0.1 * torch.randn(batch, 1, samples, generator=torch.Generator().manual_seed(1337))).to(dev)
    lib = _lib.load()
    buf = (ctypes.c_ulonglong * (4096 * KT_REC))()

    def records(codec):
        n = lib.adec_ktrace(codec._h, buf, 4096)
        if n < 0:
            raise SystemExit("adec_ktrace failed: set ADEC_KTRACE=1 and load an ADEC_PHASES library")
        return [list(buf[i * KT_REC:(i + 1) * KT_REC]) for i in range(n)]

    for _ in range(2):
        bench.codec_step(tx, rx, dec, x)
    for c in (tx, rx, dec):
        records(c)
    bench.codec_step(tx, rx, dec, x)
    torch.cuda.synchronize(dev)
    out = []
    for part, c in (("encoder", tx), ("decoder", dec)):
        for r in records(c):
            if r[5] != len(PHASES):
                raise SystemExit(f"record has {r[5]} phase counters, expected {len(PHASES)}: not an ADEC_PHASES library of this version")
            cyc = dict(zip(PHASES, r[6:6 + len(PHASES)]))
            out.append({"part": part, "launch": describe(r[3], r[4]), "us": (r[1] - r[0]) / 1e3, "cycles": cyc})
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "batch": batch, "samples": samples, "launches": out}))


def shares(cyc, keys):
    tot = sum(cyc[k] for k in keys)
    return {k: (cyc[k] / tot if tot else 0.0) for k in keys}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", help="an ADEC_PHASES library to load instead of building one")
    ap.add_argument("--build-dir", help="where to build the instrumented library (default: a temporary directory)")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--samples", type=int, default=48000)
    ap.add_argument("--json", help="also write the per-launch counters and shares to this file")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.batch, args.samples)
    with tempfile.TemporaryDirectory() as tmp:
        lib = args.lib or build(args.build_dir or tmp)
        env = dict(os.environ, ADEC_LIB_PATH=os.path.abspath(lib), ADEC_KTRACE="1")
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--batch", str(args.batch), "--samples", str(args.samples)],
                             env=env, capture_output=True, text=True)
    if res.returncode:
        sys.stderr.write(res.stderr)
        raise SystemExit(res.returncode)
    data = json.loads(res.stdout.strip().splitlines()[-1])
    print(f"{data['gpu']}: one warmed step of {data['batch']} x {data['samples']} samples; shares of each role's cycles")
    print(f"{'part':8s} {'launch':58s} {'us':>8s} | " + " ".join(f"{k:>5s}" for k in CONSUMER) + " | " +
          " ".join(f"{k:>5s}" for k in PRODUCER) + " | wfree")
    for L in data["launches"]:
        c, p = shares(L["cycles"], CONSUMER), shares(L["cycles"], PRODUCER)
        w = shares(L["cycles"], ["wfree", "wissue"])["wfree"]
        L["consumer_shares"], L["producer_shares"], L["weight_wait_share"] = c, p, w
        print(f"{L['part']:8s} {L['launch']:58s} {L['us']:8.1f} | " + " ".join(f"{c[k]:5.2f}" for k in CONSUMER) + " | " +
              " ".join(f"{p[k]:5.2f}" for k in PRODUCER) + f" | {w:5.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(data, f, indent=1)


if __name__ == "__main__":
    main()
