"""Receiver loss concealment at the BASELINE configs[3] shape: libritts v1 (symAD codebooks + HiFi-GAN v1 decoder, fp32, synthetic
weights), 1500-sample packets (5 code frames) at 24 kHz, capacity 256.

Four ReceiverSessionServers, each with 256 open sessions, are fed the same packet streams (one TransmitterSessionServer made them
beforehand, one packet per session per step):
    off      conceal_packets=0, no loss (today's receiver)
    on       conceal_packets=2, no loss
    on_1pct  conceal_packets=2, each packet dropped with probability 0.01 (seeded)
    on_5pct  conceal_packets=2, each packet dropped with probability 0.05 (seeded)
At an occupancy of k sessions, k of the 256 get a packet each step.  Each arm runs `--steps` steps per region with the host clock around
every step() (H2D, launches, D2H and hand-off included).  Regions alternate the arms, region 0 warms up, and every figure is the
median of the regions' per-step medians.  Every step the `on` arm's PCM is compared bit for bit with the `off` arm's.

Then the lookup launch alone at the 256-session shape (1280 rows): lookup_packed against lookup_packed_conceal, on all-real rows as a
loss-free step builds them and on all-concealed rows.  Two figures per call: the kernel's device time from torch.profiler (run on
its own), and CUDA-event time over `--calls` back-to-back calls (the concealing call includes its host-side descriptor check and the
descriptor upload).  The GPU's name, power limit and SM clocks are read before and after the timing.  Prints one JSON object.

    python tools/bench_receiver_conceal.py [--steps 20] [--regions 5] [--calls 200]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_stream_sessions import build, gpu_info  # noqa: E402

CAP, FS, SR, FPP = 256, 1500, 24000, 5
OCCUPANCY = (16, 64, 256)
ARMS = (("off", 0, 0.0), ("on", 2, 0.0), ("on_1pct", 2, 0.01), ("on_5pct", 2, 0.05))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--calls", type=int, default=200)
    args = ap.parse_args()
    import numpy as np
    import torch
    from audiodec_b200 import wire
    from audiodec_b200.server import ReceiverSessionServer, TransmitterSessionServer
    if not torch.cuda.is_available():
        raise SystemExit("bench_receiver_conceal needs a CUDA device")
    dev = torch.device("cuda:0")
    info_before = gpu_info(0)

    # the packet streams: every session active in every occupancy needs one packet per step of every region
    need = (args.regions + 1) * args.steps * len(OCCUPANCY)
    tx = build(dev, 1)[0]
    tx_srv = TransmitterSessionServer(tx, capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=10.0, device=dev)
    for sid in range(CAP):
        tx_srv.open(sid)
    rng = np.random.default_rng(0)
    stream = {sid: [] for sid in range(CAP)}
    for _ in range(need):
        x = (0.1 * rng.standard_normal((CAP, FS))).astype(np.float32)
        for sid in range(CAP):
            tx_srv.submit(sid, x[sid])
        tx_srv.step()
        for sid, buf in tx_srv.poll_packets():
            stream[sid].append(buf)
    del tx_srv, tx

    arms = {}
    for name, k_conceal, p in ARMS:
        _, rx, dec = build(dev, 1)
        srv = ReceiverSessionServer(rx, dec, capacity=CAP, frames_per_packet=FPP, sample_rate=SR, device=dev, conceal_packets=k_conceal)
        for sid in range(CAP):
            srv.open(sid)
        arms[name] = {"srv": srv, "p": p, "cursor": [0] * CAP, "rng": np.random.default_rng(1 + len(arms)), "dropped": 0}
    active = {k: list(range(0, CAP, CAP // k))[:k] for k in OCCUPANCY}
    parity = True
    last_off = {}

    def run(name, k):
        nonlocal parity
        a = arms[name]
        srv, t = a["srv"], []
        for i in range(args.steps):
            for sid in active[k]:
                buf = stream[sid][a["cursor"][sid]]
                a["cursor"][sid] += 1
                if a["p"] and a["rng"].random() < a["p"]:
                    a["dropped"] += 1
                    continue
                srv.submit_packet(buf)
            t0 = time.perf_counter()
            srv.step()
            t.append(time.perf_counter() - t0)
            out = {}
            for sid in active[k]:
                while (y := srv.poll(sid)) is not None:
                    out.setdefault(sid, []).append(y)
            if name == "off":
                last_off[i] = out
            elif name == "on":
                parity &= out.keys() == last_off[i].keys() and all(
                    len(v) == len(last_off[i][sid]) and all(np.array_equal(y.view(np.int32), w.view(np.int32))
                                                            for y, w in zip(v, last_off[i][sid])) for sid, v in out.items())
        return statistics.median(t)

    res = {k: {name: [] for name, _, _ in ARMS} for k in OCCUPANCY}
    for r in range(args.regions + 1):
        for k in OCCUPANCY:
            for name, _, _ in ARMS:
                t = run(name, k)
                if r:                                    # region 0 warms every shape up
                    res[k][name].append(t)
    torch.cuda.synchronize(dev)

    # the lookup launch alone, at the 256-session shape
    rx_srv = arms["on"]["srv"]
    rx = rx_srv.rx_encoder
    nb = rx.packed_frame_bytes()
    payload = b"".join(wire.decode_packet(stream[sid][0]).payload for sid in range(CAP))
    packed = torch.frombuffer(bytearray(payload), dtype=torch.uint8).view(CAP * FPP, nb).to(dev)
    anchors = torch.zeros(CAP, rx.code_dim, dtype=torch.float32, device=dev)
    f = np.full(CAP, FPP)
    real_rows = ReceiverSessionServer._conceal_rows([(s, 0, None, None) for s in range(CAP)], f, list(range(0, CAP * FPP, FPP)))
    conc_rows = np.stack([np.full(CAP * FPP, -1), np.arange(CAP * FPP), np.repeat(np.arange(CAP), FPP),
                          np.tile(np.arange(1, FPP + 1), CAP), np.full(CAP * FPP, 2 * FPP + 1)], 1).astype(np.int32)
    calls = {"plain": lambda: rx.lookup_packed(packed.view(1, CAP * FPP, nb)),
             "conceal_real_rows": lambda: rx.lookup_packed_conceal(packed, real_rows, anchors),
             "conceal_concealed_rows": lambda: rx.lookup_packed_conceal(packed, conc_rows, anchors)}
    for fn in calls.values():
        fn()
    torch.cuda.synchronize(dev)
    ev = {name: [] for name in calls}
    for _ in range(5):
        for name, fn in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.calls):
                fn()
            e1.record()
            torch.cuda.synchronize(dev)
            ev[name].append(e0.elapsed_time(e1) * 1e3 / args.calls)
    kern = {}
    from torch.profiler import ProfilerActivity, profile
    for name, fn in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                fn()
            torch.cuda.synchronize(dev)
        rows = [e for e in prof.key_averages() if "lookup" in e.key and "kernel" in e.key]
        kern[name] = {e.key: round(e.device_time_total / max(1, e.count), 3) for e in rows}
    info_after = gpu_info(0)

    def ms(x):
        return round(1e3 * x, 3)

    table = {}
    for k in OCCUPANCY:
        row = {f"{name}_step_ms": ms(statistics.median(res[k][name])) for name, _, _ in ARMS}
        row["regions_ms"] = {name: [ms(x) for x in res[k][name]] for name, _, _ in ARMS}
        table[k] = row
    counts = {}
    for name, _, _ in ARMS:
        per = arms[name]["srv"].statistics()["per_session"].values()
        counts[name] = {"dropped": arms[name]["dropped"], "losses": sum(p["losses"] for p in per),
                        "concealed": sum(p["concealed"] for p in per), "packets": sum(p["packets"] for p in per)}
    print(json.dumps({
        "gpu_before": info_before, "gpu_after": info_after,
        "shape": {"capacity": CAP, "frame_size": FS, "sample_rate": SR, "frames_per_packet": FPP, "conceal_packets": 2,
                  "model": "symAD codebooks + HiFi-GAN v1 (libritts v1), fp32"},
        "steps_per_region": args.steps, "regions": args.regions,
        "pcm_bit_exact_on_vs_off": parity, "sessions": table, "arm_counts": counts,
        "lookup_1280_rows": {"event_us_per_call": {n: round(statistics.median(v), 2) for n, v in ev.items()},
                             "event_us_regions": {n: [round(x, 2) for x in v] for n, v in ev.items()},
                             "profiler_kernel_us": kern},
    }, indent=1))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
