"""The receiver's playout clock at the configs[3] shape: libritts v1 (symAD codebooks + HiFi-GAN v1 decoder, fp32, synthetic
weights), 1500-sample packets (5 code frames) at 24 kHz, capacity 256.

Eight ReceiverSessionServers are fed the same packet streams (one TransmitterSessionServer made them beforehand, one packet per session
per step), four with conceal_packets=2 and four with playout_delay=2:
    *_clean     no loss, no jitter
    *_jit       no loss, every packet delayed by 0 - 2 steps (seeded)
    *_1pct      the jitter, and each packet dropped with probability 0.01 (seeded)
    *_5pct      the jitter, and each packet dropped with probability 0.05 (seeded)
At an occupancy of k sessions, a region opens k sessions on every receiver, runs `--steps` + 2 steps and closes them again; the host
clock is taken around each of the last `--steps` step() calls (H2D, launches, D2H and hand-off included), so the playout arms are
timed only once every session plays.  Regions alternate the arms, region 0 warms up, and every figure is the median of the regions'
per-step medians.  The clean arms' PCM is compared bit for bit, session by session.

Then the lookup launch alone at the 256-session shape (1280 rows): lookup_packed_conceal on real and on concealed rows against
lookup_packed_playout on real, on half interpolated / half fade, and on fade rows (no packed frame staged), as kernel device time from
torch.profiler; and the host time of one lookup_packed_playout call with its descriptors in pageable memory against a page-locked
table (the call returns before the kernel runs, so this is the check, the upload's enqueue and the launch).  The GPU's name, power
limit and SM clocks are read before and after the timing.  Prints one JSON object.

    python tools/bench_receiver_playout.py [--steps 20] [--regions 5] [--calls 200]
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

CAP, FS, SR, FPP, D = 256, 1500, 24000, 5, 2
OCCUPANCY = (16, 64, 256)
ARMS = tuple((f"{kind}_{tag}", kind, p, jit) for kind in ("conceal", "playout")
             for tag, p, jit in (("clean", 0.0, False), ("jit", 0.0, True), ("1pct", 0.01, True), ("5pct", 0.05, True)))


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
        raise SystemExit("bench_receiver_playout needs a CUDA device")
    dev = torch.device("cuda:0")
    info_before = gpu_info(0)

    n_pkt = args.steps + D
    tx = build(dev, 1)[0]
    tx_srv = TransmitterSessionServer(tx, capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=10.0, device=dev)
    for sid in range(CAP):
        tx_srv.open(sid)
    rng = np.random.default_rng(0)
    stream = {sid: [] for sid in range(CAP)}
    for _ in range(n_pkt):
        x = (0.1 * rng.standard_normal((CAP, FS))).astype(np.float32)
        for sid in range(CAP):
            tx_srv.submit(sid, x[sid])
        tx_srv.step()
        for sid, buf in tx_srv.poll_packets():
            stream[sid].append(buf)
    del tx_srv, tx

    arms = {}
    for name, kind, p, jit in ARMS:
        _, rx, dec = build(dev, 1)
        kw = {"conceal_packets": 2} if kind == "conceal" else {"playout_delay": D}
        srv = ReceiverSessionServer(rx, dec, capacity=CAP, frames_per_packet=FPP, sample_rate=SR, device=dev, **kw)
        arms[name] = {"srv": srv, "p": p, "jit": jit, "rng": np.random.default_rng(1 + len(arms)), "dropped": 0, "counts": {}}
    active = {k: list(range(0, CAP, CAP // k))[:k] for k in OCCUPANCY}
    clean_pcm = {}
    parity = True

    def run(name, k):
        nonlocal parity
        a = arms[name]
        srv, t, due = a["srv"], [], {}
        for sid in active[k]:
            srv.open(sid)
        pcm = {sid: [] for sid in active[k]}
        for i in range(n_pkt):
            for sid in active[k]:
                if a["p"] and a["rng"].random() < a["p"]:
                    a["dropped"] += 1
                    continue
                due.setdefault(i + (int(a["rng"].integers(0, 3)) if a["jit"] else 0), []).append(stream[sid][i])
            for buf in due.pop(i, []):
                srv.submit_packet(buf)
            t0 = time.perf_counter()
            srv.step()
            if i >= D:
                t.append(time.perf_counter() - t0)
            for sid in active[k]:
                while (y := srv.poll(sid)) is not None:
                    pcm[sid].append(y)
        for sid, st in srv.statistics()["per_session"].items():
            for key, v in st.items():
                if isinstance(v, int):
                    a["counts"][key] = a["counts"].get(key, 0) + v
        for sid in active[k]:
            srv.close(sid)
        if name.endswith("_clean"):
            other = clean_pcm.pop(k, None)
            if other is None:
                clean_pcm[k] = pcm
            else:
                for sid in active[k]:
                    n = min(len(pcm[sid]), len(other[sid]))
                    parity &= n >= args.steps and all(np.array_equal(x.view(np.int32), y.view(np.int32))
                                                      for x, y in zip(pcm[sid][:n], other[sid][:n]))
        return statistics.median(t)

    res = {k: {name: [] for name, *_ in ARMS} for k in OCCUPANCY}
    for r in range(args.regions + 1):
        for k in OCCUPANCY:
            for name, *_ in ARMS:
                t = run(name, k)
                if r:                                    # region 0 warms every shape up
                    res[k][name].append(t)
    torch.cuda.synchronize(dev)

    # the lookup launch alone, at the 256-session shape
    rx = arms["playout_clean"]["srv"].rx_encoder
    nb = rx.packed_frame_bytes()
    r = CAP * FPP
    payload = b"".join(wire.decode_packet(stream[sid][0]).payload for sid in range(CAP))
    packed = torch.frombuffer(bytearray(payload), dtype=torch.uint8).view(r, nb).to(dev)
    anchors = torch.zeros(CAP, rx.code_dim, dtype=torch.float32, device=dev)
    targets = rx.silence_frame().view(1, -1).contiguous()
    session = np.repeat(np.arange(CAP), FPP)
    last = np.tile(np.arange(FPP) == FPP - 1, CAP)
    j = np.tile(np.arange(1, FPP + 1), CAP)
    c_real = np.stack([np.arange(r), np.full(r, -1), np.where(last, session, -1), np.zeros(r), np.zeros(r)], 1).astype(np.int32)
    c_conc = np.stack([np.full(r, -1), np.arange(r), session, j, np.full(r, 2 * FPP + 1)], 1).astype(np.int32)
    p_real = np.stack([c_real[:, 0], c_real[:, 1], np.full(r, -1), c_real[:, 2], c_real[:, 3], c_real[:, 4]], 1).astype(np.int32)
    p_fade = np.stack([np.full(r, -1), np.full(r, -1), np.zeros(r), session, j, np.full(r, 2 * FPP)], 1).astype(np.int32)
    half = (session % 2 == 0)[:, None]
    p_mixed = np.where(half, np.stack([np.full(r, -1), np.arange(r), np.full(r, -1), session, j, np.full(r, 2 * FPP + 1)], 1),
                       p_fade).astype(np.int32)
    empty = packed[:0]
    calls = {"conceal_real_rows": lambda: rx.lookup_packed_conceal(packed, c_real, anchors),
             "conceal_concealed_rows": lambda: rx.lookup_packed_conceal(packed, c_conc, anchors),
             "playout_real_rows": lambda: rx.lookup_packed_playout(packed, p_real, anchors, targets),
             "playout_interp_and_fade_rows": lambda: rx.lookup_packed_playout(packed, p_mixed, anchors, targets),
             "playout_fade_rows_F0": lambda: rx.lookup_packed_playout(empty, p_fade, anchors, targets)}
    for fn in calls.values():
        fn()
    torch.cuda.synchronize(dev)
    kern = {}
    from torch.profiler import ProfilerActivity, profile
    for name, fn in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                fn()
            torch.cuda.synchronize(dev)
        rows = [e for e in prof.key_averages() if "lookup" in e.key and "kernel" in e.key]
        kern[name] = {e.key: round(e.device_time_total / max(1, e.count), 3) for e in rows}

    # host time per call: pageable descriptors against a page-locked table (the server's two tables, used in turn)
    pinned = [torch.empty(r, 6, dtype=torch.int32, pin_memory=True) for _ in range(2)]
    for t_ in pinned:
        t_.numpy()[:] = p_real
    pinned_np = [t_.numpy() for t_ in pinned]
    pageable = [p_real.copy(), p_real.copy()]
    host = {"pageable": [], "page_locked": []}
    for _ in range(5):
        for name, tables in (("pageable", pageable), ("page_locked", pinned_np)):
            t = []
            for i in range(args.calls):
                t0 = time.perf_counter()
                rx.lookup_packed_playout(packed, tables[i & 1], anchors, targets)
                t.append(time.perf_counter() - t0)
                if i % 16 == 15:
                    torch.cuda.synchronize(dev)          # keep the queue short: the figure is the host side of one call
            torch.cuda.synchronize(dev)
            host[name].append(statistics.median(t) * 1e6)
    info_after = gpu_info(0)

    def ms(x):
        return round(1e3 * x, 3)

    table = {}
    for k in OCCUPANCY:
        row = {f"{name}_step_ms": ms(statistics.median(res[k][name])) for name, *_ in ARMS}
        row["regions_ms"] = {name: [ms(x) for x in res[k][name]] for name, *_ in ARMS}
        table[k] = row
    counts = {name: dict(arms[name]["counts"], dropped=arms[name]["dropped"]) for name, *_ in ARMS}
    print(json.dumps({
        "gpu_before": info_before, "gpu_after": info_after,
        "shape": {"capacity": CAP, "frame_size": FS, "sample_rate": SR, "frames_per_packet": FPP, "conceal_packets": 2,
                  "playout_delay": D, "model": "symAD codebooks + HiFi-GAN v1 (libritts v1), fp32"},
        "steps_per_region": args.steps, "regions": args.regions,
        "pcm_bit_exact_clean_playout_vs_conceal": parity, "sessions": table, "arm_counts": counts,
        "lookup_1280_rows_profiler_kernel_us": kern,
        "playout_call_host_us": {n: round(statistics.median(v), 2) for n, v in host.items()},
        "playout_call_host_us_regions": {n: [round(x, 2) for x in v] for n, v in host.items()},
    }, indent=1))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
