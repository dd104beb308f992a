"""The adaptive playout clock at the configs[3] shape: libritts v1 (symAD codebooks + HiFi-GAN v1 decoder, fp32, synthetic weights),
1500-sample packets (5 code frames) at 24 kHz, capacity 256.

Three receiver arms: fixed playout_delay=2, fixed playout_delay=6 and adaptive playout_delay=1, max_playout_delay=6.

1. The lookup launch alone at 1280 rows, as kernel device time from torch.profiler: lookup_packed_timescale on real rows and on rows
   80 % of which are between rows, against lookup_packed_playout on real rows.
2. Step host time at 16 / 64 / 256 sessions under one 0 - 2-step jitter trace (seeded), every arm fed the same packets: a region
   opens k sessions, runs `--steps` + 8 steps and closes them; the host clock is taken around each of the last `--steps` step()
   calls (H2D, launches, D2H and hand-off included).  Regions alternate the arms, region 0 warms up, and every figure is the median of
   the regions' per-step medians.
3. What each arm buys, per trace, over 16 sessions of 600 steps (seeds 0 - 15): the mean delay Delta in ms, underruns, faded frames,
   late packets and pauses.  Delta = (k - min lateness + 1) * P - p frames at each step a session plays (min over the talk spurt's
   last 64 packets; p its playout position); a fixed arm keeps no Delta, so it is computed here by the same formula.  Traces: clean,
   0 - 2-step jitter, a spike (0 jitter, 0 - 4 steps for packets 100 - 299, 0 again), and a sender clock 1 % fast and 1 % slow.
   These counters come from host rules and are the same on any machine.

The GPU's name, power limit and SM clocks are read before and after.  Prints one JSON object.

    python tools/bench_receiver_adaptive.py [--steps 20] [--regions 5] [--calls 200]
"""
import argparse
import collections
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
ARMS = (("fixed_d2", {"playout_delay": 2}), ("fixed_d6", {"playout_delay": 6}),
        ("adaptive_1_6", {"playout_delay": 1, "max_playout_delay": 6}))
TRACES = ("clean", "jitter", "spike", "drift_fast", "drift_slow")
OUTCOME_STEPS, OUTCOME_SESSIONS, WINDOW = 600, 16, 64


def arrival_steps(kind, n, rng):
    """the step before which each of n packets (sent one per step) arrives"""
    if kind == "clean":
        return list(range(n))
    if kind == "jitter":
        return [q + (int(rng.integers(0, 3)) if q else 0) for q in range(n)]
    if kind == "spike":
        return [q + (int(rng.integers(0, 5)) if 100 <= q < 300 else 0) for q in range(n)]
    if kind == "drift_fast":
        return [int(q / 1.01) for q in range(n)]
    if kind == "drift_slow":
        return [int(q / 0.99) for q in range(n)]
    raise ValueError(kind)


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
        raise SystemExit("bench_receiver_adaptive needs a CUDA device")
    dev = torch.device("cuda:0")
    info_before = gpu_info(0)

    n_pkt = max(args.steps + 8, OUTCOME_STEPS + 16)   # a sender 1 % fast sends 606 packets in 600 steps: none runs dry
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
    for name, kw in ARMS:
        _, rx, dec = build(dev, 1)
        arms[name] = ReceiverSessionServer(rx, dec, capacity=CAP, frames_per_packet=FPP, sample_rate=SR, device=dev, **kw)

    # ---- 1. the lookup launch alone, 1280 rows
    rx = arms["adaptive_1_6"].rx_encoder
    nb = rx.packed_frame_bytes()
    r = CAP * FPP
    payload = b"".join(wire.decode_packet(stream[sid][0]).payload for sid in range(CAP))
    packed = torch.frombuffer(bytearray(payload), dtype=torch.uint8).view(r, nb).to(dev)
    anchors = torch.zeros(CAP, rx.code_dim, dtype=torch.float32, device=dev)
    targets = rx.silence_frame().view(1, -1).contiguous()
    session = np.repeat(np.arange(CAP), FPP)
    last = np.tile(np.arange(FPP) == FPP - 1, CAP)
    real = np.stack([np.arange(r), np.full(r, -1), np.full(r, -1), np.where(last, session, -1), np.zeros(r), np.zeros(r)], 1)
    real = real.astype(np.int32)
    between = real.copy()
    pick = np.random.default_rng(2).random(r) < 0.8      # a between row from frame r to frame r + 1
    nxt = np.minimum(np.arange(r) + 1, r - 1)
    between[pick] = np.stack([np.arange(r), nxt, np.full(r, -1), np.full(r, -1), np.full(r, 2), np.full(r, FPP - 1)], 1)[pick]
    calls = {"timescale_real_rows": lambda: rx.lookup_packed_timescale(packed, real, anchors, targets),
             "timescale_80pct_between_rows": lambda: rx.lookup_packed_timescale(packed, between, anchors, targets),
             "playout_real_rows": lambda: rx.lookup_packed_playout(packed, real, anchors, targets)}
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
        ev = [e for e in prof.key_averages() if "lookup" in e.key and "kernel" in e.key]
        kern[name] = {e.key: round(e.device_time_total / max(1, e.count), 3) for e in ev}
    kern["between_rows"] = int(pick.sum())

    # ---- 2. step host time under one jitter trace
    jit_rng = np.random.default_rng(7)
    due_at = {sid: arrival_steps("jitter", args.steps + 8, jit_rng) for sid in range(CAP)}
    active = {k: list(range(0, CAP, CAP // k))[:k] for k in OCCUPANCY}

    def timed(name, k):
        srv, t, due = arms[name], [], {}
        for sid in active[k]:
            srv.open(sid)
            for q, a in enumerate(due_at[sid]):
                due.setdefault(a, []).append(stream[sid][q])
        for i in range(args.steps + 8):
            for buf in due.pop(i, []):
                srv.submit_packet(buf)
            t0 = time.perf_counter()
            srv.step()
            if i >= 8:
                t.append(time.perf_counter() - t0)
            for sid in active[k]:
                while srv.poll(sid) is not None:
                    pass
        for sid in active[k]:
            srv.close(sid)
        return statistics.median(t)

    res = {k: {name: [] for name, _ in ARMS} for k in OCCUPANCY}
    for reg in range(args.regions + 1):
        for k in OCCUPANCY:
            for name, _ in ARMS:
                t = timed(name, k)
                if reg:                                  # region 0 warms every shape up
                    res[k][name].append(t)
    torch.cuda.synchronize(dev)
    info_mid = gpu_info(0)

    # ---- 3. what each arm buys, per trace
    sids = list(range(OUTCOME_SESSIONS))
    frame_ms = 1e3 * FS / FPP / SR

    def outcome(name, kind):
        srv = arms[name]
        adaptive = srv.max_playout_delay is not None
        due = {}
        for sid in sids:
            for q, a in enumerate(arrival_steps(kind, n_pkt, np.random.default_rng(100 + sid))):
                due.setdefault(a, []).append((sid, q))
            srv.open(sid)
        lat = {sid: collections.deque(maxlen=WINDOW) for sid in sids}
        pauses = {sid: 0 for sid in sids}
        deltas = []
        for k in range(OUTCOME_STEPS):
            for sid, q in due.pop(k, []):
                s = srv._ids[sid]
                if srv.submit_packet(stream[sid][q]) or q in srv._given_up[s]:
                    lat[sid].append(k - q)
            before = {sid: (srv._next[srv._ids[sid]], srv._playing[srv._ids[sid]]) for sid in sids}
            srv.step()
            for sid in sids:
                s = srv._ids[sid]
                played = srv.poll(sid) is not None
                while srv.poll(sid) is not None:
                    pass
                if played:
                    deltas.append(srv.stats[s].delay_frames if adaptive else (k - min(lat[sid]) + 1) * FPP - before[sid][0] * FPP)
                if srv.stats[s].pauses > pauses[sid]:
                    pauses[sid] = srv.stats[s].pauses
                    lat[sid].clear()
        per = srv.statistics()["per_session"]
        out = {key: sum(per[sid][key] for sid in sids) for key in ("underruns", "faded_frames", "late", "pauses", "losses", "concealed")}
        if adaptive:
            out.update(compressed=sum(per[sid]["compressed"] for sid in sids), expanded=sum(per[sid]["expanded"] for sid in sids))
        out["mean_delay_ms"] = round(float(np.mean(deltas)) * frame_ms, 2)
        for sid in sids:
            srv.close(sid)
        return out

    outcomes = {kind: {name: outcome(name, kind) for name, _ in ARMS} for kind in TRACES}
    info_after = gpu_info(0)

    def ms(x):
        return round(1e3 * x, 3)

    table = {}
    for k in OCCUPANCY:
        row = {f"{name}_step_ms": ms(statistics.median(res[k][name])) for name, _ in ARMS}
        row["regions_ms"] = {name: [ms(x) for x in res[k][name]] for name, _ in ARMS}
        table[k] = row
    print(json.dumps({
        "gpu_before": info_before, "gpu_mid": info_mid, "gpu_after": info_after,
        "shape": {"capacity": CAP, "frame_size": FS, "sample_rate": SR, "frames_per_packet": FPP,
                  "model": "symAD codebooks + HiFi-GAN v1 (libritts v1), fp32"},
        "steps_per_region": args.steps, "regions": args.regions,
        "lookup_1280_rows_profiler_kernel_us": kern, "sessions": table,
        "outcomes": {"sessions": OUTCOME_SESSIONS, "steps": OUTCOME_STEPS, "frame_ms": frame_ms, "traces": outcomes},
    }, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
