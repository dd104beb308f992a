"""The split session servers against the loopback session server at the BASELINE configs[3] shape: libritts v1 (symAD encoder +
HiFi-GAN v1 decoder, fp32, synthetic weights), 1500-sample frames at 24 kHz, capacity 256.

Three servers, each with 256 open sessions: SessionCodecServer(wire=True) (encode_streams -> fused RVQ to packed bytes ->
lookup_packed -> decode_streams in one step()), TransmitterSessionServer (encode_streams -> fused RVQ -> packets) and
ReceiverSessionServer (packets -> lookup_packed -> decode_streams).  At an occupancy of k sessions, k of the 256 have a frame each step
(the others are idle and cost nothing).  Each arm runs `--steps` steps per region with the host clock around every step() (H2D,
launches, D2H and hand-off included); the split arm also times the receiver's submit_packet() calls of a step.  Regions alternate
loopback and split arm by arm, region 0 warms up, and every figure is the median of the regions' per-step medians.  Every step the
receiver's PCM is compared bit for bit with the loopback server's for the same sessions and frames.  The GPU's name, power limit and
SM clocks are read before and after the timing.  Prints one JSON object.

    python tools/bench_split_servers.py [--steps 20] [--regions 5]
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

CAP, FS, SR = 256, 1500, 24000
OCCUPANCY = (16, 64, 256)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    from audiodec_b200.server import ReceiverSessionServer, SessionCodecServer, TransmitterSessionServer
    if not torch.cuda.is_available():
        raise SystemExit("bench_split_servers needs a CUDA device")
    dev = torch.device("cuda:0")
    info_before = gpu_info(0)
    tx, rx, dec = build(dev, 1)
    loop = SessionCodecServer(tx, rx, dec, capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=10.0, device=dev, wire=True)
    tx2 = build(dev, 1)[0]
    tx_srv = TransmitterSessionServer(tx2, capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=10.0, device=dev)
    _, rx3, dec3 = build(dev, 1)
    rx_srv = ReceiverSessionServer(rx3, dec3, capacity=CAP, frames_per_packet=FS // 300, sample_rate=SR, device=dev)
    slot = {sid: loop.open() for sid in range(CAP)}
    for sid in range(CAP):
        tx_srv.open(sid)
        rx_srv.open(sid)
    rng = np.random.default_rng(0)
    frames = (0.1 * rng.standard_normal((args.steps, CAP, FS))).astype(np.float32)
    active = {k: list(range(0, CAP, CAP // k))[:k] for k in OCCUPANCY}

    parity = True
    packet_bytes = set()
    loop_out = {}

    def run_loop(k):
        t = []
        for i in range(args.steps):
            for sid in active[k]:
                loop.submit(slot[sid], frames[i, sid])
            t0 = time.perf_counter()
            loop.step()
            t.append(time.perf_counter() - t0)
            loop_out[i] = {sid: loop.poll(slot[sid]) for sid in active[k]}
        return {"step": statistics.median(t)}

    def run_split(k, want):
        nonlocal parity
        t_tx, t_parse, t_rx = [], [], []
        for i in range(args.steps):
            for sid in active[k]:
                tx_srv.submit(sid, frames[i, sid])
            t0 = time.perf_counter()
            tx_srv.step()
            t1 = time.perf_counter()
            packets = tx_srv.poll_packets()
            t2 = time.perf_counter()
            for _, buf in packets:
                rx_srv.submit_packet(buf)
            t3 = time.perf_counter()
            rx_srv.step()
            t4 = time.perf_counter()
            t_tx.append(t1 - t0)
            t_parse.append(t3 - t2)
            t_rx.append(t4 - t3)
            packet_bytes.update(len(b) for _, b in packets)
            for sid in active[k]:
                y = rx_srv.poll(sid)
                parity &= y is not None and np.array_equal(y.view(np.int32), want[i][sid].view(np.int32))
        return {"tx_step": statistics.median(t_tx), "rx_submit_packets": statistics.median(t_parse), "rx_step": statistics.median(t_rx)}

    res = {k: {"loopback": [], "split": []} for k in OCCUPANCY}
    for r in range(args.regions + 1):
        for k in OCCUPANCY:
            a = run_loop(k)
            want = dict(loop_out)
            b = run_split(k, want)
            if r:                                    # region 0 warms every shape up
                res[k]["loopback"].append(a)
                res[k]["split"].append(b)
    torch.cuda.synchronize(dev)
    info_after = gpu_info(0)

    def med(rows, key):
        return round(1e3 * statistics.median(x[key] for x in rows), 3)

    table = {}
    for k in OCCUPANCY:
        lo, sp = res[k]["loopback"], res[k]["split"]
        row = {"loopback_step_ms": med(lo, "step"), "tx_step_ms": med(sp, "tx_step"), "rx_step_ms": med(sp, "rx_step"),
               "rx_submit_packets_ms": med(sp, "rx_submit_packets"),
               "regions_ms": {"loopback": [round(1e3 * x["step"], 3) for x in lo],
                              "tx": [round(1e3 * x["tx_step"], 3) for x in sp], "rx": [round(1e3 * x["rx_step"], 3) for x in sp]}}
        row["tx_plus_rx_over_loopback"] = round((row["tx_step_ms"] + row["rx_step_ms"]) / row["loopback_step_ms"], 3)
        table[k] = row
    print(json.dumps({
        "gpu_before": info_before, "gpu_after": info_after,
        "shape": {"capacity": CAP, "frame_size": FS, "sample_rate": SR, "model": "symAD + HiFi-GAN v1 (libritts v1), fp32"},
        "steps_per_region": args.steps, "regions": args.regions,
        "pcm_bit_exact_vs_loopback": parity, "bytes_per_packet": sorted(packet_bytes),
        "sessions": table,
    }, indent=1))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
