"""Graphed streaming steps against the eager call sequence (TransmitterGraph / ReceiverGraph).

1. Batch-1 latency, the reference's Table 4 shape: vctk_sym at 600 / 1200 / 2400 / 4800-sample chunks.  The transmitter half
   (encode + quantize) and the receiver half (lookup + decode) are each timed by the host clock around the call plus a device
   synchronise, as bin/stream.py times them, and by CUDA events.  Eager and graphed alternate region by region.
2. Lock step, device-resident: libritts v1 at 1500 samples (24 kHz) for B in {1, 16, 64, 256}, ms per step.
3. Through MultiStreamCodecServer.step(): 16 and 256 streams, wire mode, graphed (the server's default on library generators) against
   the server's eager pass.
Prints one JSON document; needs an H100 (no CPU fallback).  Synthetic weights (audiodec_b200.synthetic)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiodec_b200 import synthetic as S  # noqa: E402
from audiodec_b200.codec import HiFiGANStreamGenerator, ReceiverGraph, SymADStreamGenerator, TransmitterGraph # noqa: E402
from audiodec_b200.server import MultiStreamCodecServer # noqa: E402

DEV = torch.device("cuda:0")


def codec(voc):
    sd = S.symad_state_dict(seed=0)
    gens = []
    for _ in range(2):
        g = SymADStreamGenerator(**S.SYMAD_PARAMS)
        g.load_state_dict(sd)
        gens.append(g.eval().to(DEV))
    if voc:
        d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
        d.load_state_dict(S.hifigan_state_dict(seed=1))
    else:
        d = SymADStreamGenerator(**S.SYMAD_PARAMS)
        d.load_state_dict(sd)
    tx, rx = gens
    return tx, rx, d.eval().to(DEV)


def halves(tx, rx, dec, B, T, graphed):
    """(transmitter half, receiver half, launches per step) as callables on device input x / indices"""
    if graphed:
        f = tx._lib.adec_frames_for(tx._h, T)
        txg, rxg = TransmitterGraph(tx, B, T), ReceiverGraph(rx, dec, B, f)
        return (lambda x: txg(x)), (lambda idx: rxg(idx)), txg.info()["kernels"] + rxg.info()["kernels"]
    return (lambda x: tx.quantize(tx.encode(x))), (lambda idx: dec.decode(rx.lookup(idx))), None


def summary(v):
    v = sorted(v)
    return {"median": round(statistics.median(v), 4), "min": round(v[0], 4), "max": round(v[-1], 4)}


def latency_b1(regions, chunks_per_region):
    out = {}
    for T in (600, 1200, 2400, 4800):
        tx, rx, dec = codec(False)
        x = 0.1 * torch.randn(1, 1, T, device=DEV)
        fns = {m: halves(tx, rx, dec, 1, T, m == "graphed") for m in ("eager", "graphed")}
        res = {m: {"tx_host_ms": [], "rx_host_ms": [], "tx_event_ms": [], "rx_event_ms": []} for m in fns}
        for m, (ftx, frx, _) in fns.items():      # warm up both
            for _ in range(10):
                frx(ftx(x))
        torch.cuda.synchronize()
        for r in range(regions):
            for m in ("eager", "graphed") if r % 2 == 0 else ("graphed", "eager"):
                ftx, frx, _ = fns[m]
                th, rh = [], []
                for _ in range(chunks_per_region):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    idx = ftx(x)
                    torch.cuda.synchronize()
                    t1 = time.perf_counter()
                    frx(idx)
                    torch.cuda.synchronize()
                    th.append((t1 - t0) * 1e3), rh.append((time.perf_counter() - t1) * 1e3)
                res[m]["tx_host_ms"].append(statistics.median(th))
                res[m]["rx_host_ms"].append(statistics.median(rh))
                e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                torch.cuda.synchronize()
                e[0].record()
                for _ in range(chunks_per_region):
                    idx = ftx(x)
                e[1].record()
                for _ in range(chunks_per_region):
                    frx(idx)
                e[2].record()
                torch.cuda.synchronize()
                res[m]["tx_event_ms"].append(e[0].elapsed_time(e[1]) / chunks_per_region)
                res[m]["rx_event_ms"].append(e[1].elapsed_time(e[2]) / chunks_per_region)
        out[f"chunk_{T}"] = {m: {k: summary(v) for k, v in d.items()} for m, d in res.items()}
        out[f"chunk_{T}"]["kernels_per_step"] = fns["graphed"][2]
        del fns
    return out


def lock_step(regions, steps):
    out = {}
    for B in (1, 16, 64, 256):
        tx, rx, dec = codec(True)
        xs = [0.1 * torch.randn(B, 1, 1500, device=DEV) for _ in range(4)]
        fns = {m: halves(tx, rx, dec, B, 1500, m == "graphed") for m in ("eager", "graphed")}
        for m, (ftx, frx, _) in fns.items():
            for i in range(5):
                frx(ftx(xs[i % 4]))
        torch.cuda.synchronize()
        l0 = tx.launch_count + rx.launch_count + dec.launch_count
        fns["eager"][1](fns["eager"][0](xs[0]))
        launches = tx.launch_count + rx.launch_count + dec.launch_count - l0
        res = {"eager": [], "graphed": []}
        for r in range(regions):
            for m in ("eager", "graphed") if r % 2 == 0 else ("graphed", "eager"):
                ftx, frx, _ = fns[m]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(steps):
                    frx(ftx(xs[i % 4]))
                e1.record()
                torch.cuda.synchronize()
                res[m].append(e0.elapsed_time(e1) / steps)
        out[f"B{B}"] = {"ms_per_step": {m: summary(v) for m, v in res.items()}, "launches_per_step_eager": launches,
                        "kernels_per_step_graphed": fns["graphed"][2]}
    return out


def server(regions, steps):
    out = {}
    rng = np.random.default_rng(7)
    for B in (16, 256):
        frames = (0.1 * rng.standard_normal((4, B, 1500))).astype(np.float32)
        srv = MultiStreamCodecServer(*codec(True), n_streams=B, frame_size=1500, sample_rate=24000, max_latency=10.0, device=DEV,
                                     wire=True)
        x_host = torch.from_numpy(frames).pin_memory()
        res = {"eager": [], "graphed": []}

        def run(m, n):
            # both arms run the whole lock-step pass (H2D, codec, D2H, frames to numpy); the eager arm swaps the graph launches for
            # the server's eager call sequence
            if m == "eager":
                srv._graph_pass = lambda x, dev: srv._eager_pass(x, dev, None)
            else:
                srv.__dict__.pop("_graph_pass", None)
            for k in range(n):
                srv._codec_pass(x_host[k % 4].view(B, 1, 1500), DEV)
        run("graphed", 5), run("eager", 5)
        for r in range(regions):
            for m in ("eager", "graphed") if r % 2 == 0 else ("graphed", "eager"):
                t0 = time.perf_counter()
                run(m, steps)
                res[m].append((time.perf_counter() - t0) * 1e3 / steps)
        out[f"B{B}_wire"] = {"ms_per_step_host_to_host": {m: summary(v) for m, v in res.items()}}
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # read-only query; the numbers stand without it
        q = f"unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(DEV), "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--chunks", type=int, default=100)
    ap.add_argument("--steps", type=int, default=100)
    a = ap.parse_args()
    res = {"card_before": card()}
    tx, rx, dec = codec(False)
    g = TransmitterGraph(tx, 1, 1500)
    r = ReceiverGraph(rx, dec, 1, 5)
    res["vctk_sym_b1_1500"] = {"tx": g.info(), "rx": r.info()}
    del g, r, tx, rx, dec
    res["latency_b1"] = latency_b1(a.regions, a.chunks)
    res["lock_step_libritts_v1_1500"] = lock_step(a.regions, a.steps)
    res["server_wire"] = server(a.regions, max(10, a.steps // 5))
    res["card_after"] = card()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
