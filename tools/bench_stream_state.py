"""Stream state export / import (adec_get_stream_state / adec_set_stream_state) and session migration between SessionCodecServers.

  * device time of one export and one import of 1, 16 and 256 streams (CUDA events around `--iters` calls, median of `--regions`) on the
    libritts v1 transmitter encoder (symAD, full handle) and HiFi-GAN v1 decoder, and on vctk_sym (the symAD handle that decodes too),
    with the values per stream that adec_stream_state_elems reports;
  * the configs[3] session server (libritts v1, 1500-sample chunks at 24 kHz, capacity 256, wire mode, 128 open sessions that each
    submit a frame per step): host time of step(), and of step() plus one session detached from it and attached to a second server of
    the same shape on the same GPU (steps alternate; after a plain step one session goes back, untimed, so both servers keep their load).

The GPU's name and power limit are read in the same run.  Prints one JSON object.

    python tools/bench_stream_state.py [--iters 50] [--regions 5] [--steps 40]
"""
import argparse
import json
import os
import statistics
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from bench_stream_sessions import CAP, FS, SR, build, gpu_info  # noqa: E402

STREAMS = (1, 16, 256)


def time_io(g, n, iters, regions):
    import torch
    ids = list(range(n))
    st = g.stream_state(ids)
    out = {}
    for what, fn in (("get", lambda: g.stream_state(ids)), ("set", lambda: g.load_stream_state(ids, st))):
        for _ in range(3):
            fn()
        ms = []
        for _ in range(regions):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1) / iters)
        out[what + "_us"] = round(statistics.median(ms) * 1e3, 2)
    out["bytes"] = st.numel() * st.element_size()
    out["GB_per_s_get"] = round(out["bytes"] / (out["get_us"] * 1e-6) / 1e9, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    import numpy as np
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import SymADStreamGenerator
    from audiodec_b200.server import SessionCodecServer
    dev = torch.device("cuda:0")
    info = gpu_info(0)
    res = {"gpu": info, "io": {}, "elems_per_stream": {}}
    tx, rx, dec = build(dev, max(STREAMS))
    sym = SymADStreamGenerator(**S.SYMAD_PARAMS)
    sym.load_state_dict(S.symad_state_dict(seed=0))
    sym = sym.eval().to(dev)
    sym.set_streams(max(STREAMS))
    for name, g in (("libritts_v1_tx_encoder", tx), ("libritts_v1_decoder", dec), ("vctk_sym", sym)):
        lay = g.state_layout
        res["elems_per_stream"][name] = {
            "total": sum(c * p for _, c, p in lay),
            "encoder": sum(c * p for k, c, p in lay if k.startswith("encoder.")),
            "projector": sum(c * p for k, c, p in lay if k.startswith("projector.")),
            "decoder": sum(c * p for k, c, p in lay if not k.startswith(("encoder.", "projector."))),
        }
        res["io"][name] = {str(n): time_io(g, n, args.iters, args.regions) for n in STREAMS}
    del tx, rx, dec, sym

    # the session server, with and without one migration per step
    n_open = 128
    rng = np.random.default_rng(0)
    frames = [(0.1 * rng.standard_normal(FS)).astype(np.float32) for _ in range(8)]
    a = SessionCodecServer(*build(dev, 1), capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=1.0, device="cuda:0", wire=True)
    b = SessionCodecServer(*build(dev, 1), capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=1.0, device="cuda:0", wire=True)
    sa = [a.open() for _ in range(n_open)]
    sb = [b.open() for _ in range(n_open)]
    ms = {"step": [], "step_and_migrate": []}
    for k in range(args.steps * 2 + 4):
        for i, s in enumerate(sa):
            a.submit(s, frames[(k + i) % 8])
        for i, s in enumerate(sb):
            b.submit(s, frames[(k + i) % 8])
        migrate = k % 2 == 1
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        a.step()
        if migrate:
            sb.append(b.attach(a.detach(sa.pop(0))))
        t1 = time.perf_counter()
        if not migrate and len(sa) < n_open:
            sa.append(a.attach(b.detach(sb.pop(0))))      # the way back, outside the timed region
        b.step()
        for s in sa:
            a.poll(s)
        for s in sb:
            b.poll(s)
        if k >= 4:
            ms["step_and_migrate" if migrate else "step"].append((t1 - t0) * 1e3)
    res["server"] = {"open_sessions": n_open, "capacity": CAP, "wire": True,
                     "host_ms_median": {k: round(statistics.median(v), 3) for k, v in ms.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
