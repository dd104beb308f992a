"""Stream slots against the lock-step streaming step at the BASELINE configs[3] shape: libritts v1 (symAD encoder + HiFi-GAN v1
decoder, synthetic weights), 1500-sample chunks at 24 kHz, capacity 256, wire mode (fused RVQ + bitstream, lookup from the packed
bytes).

Arms: the lock-step uniform step over all 256 streams (encode -> quantize_fused -> lookup_packed -> decode), and slot steps
(encode_streams -> quantize_fused -> lookup_packed -> decode_streams) advancing 256, 128, 64 and 16 of the 256 streams.  Each arm is
timed device-resident (CUDA events around `--steps` steps, input already on the GPU) and through its server (MultiStreamCodecServer
with 256 streams, SessionCodecServer with that many open streams; host clock per step, H2D and D2H included).  Regions are alternated
arm by arm and every arm reports the median of `--regions` regions.  At full occupancy the slot step's waveforms are checked bit for
bit against the lock-step step's in the same run, and the per-launch times of both are listed.  The GPU's name and power limit are
read in the same run.  Prints one JSON object.

    python tools/bench_stream_sessions.py [--steps 20] [--regions 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CAP, FS, SR = 256, 1500, 24000
OCCUPANCY = (256, 128, 64, 16)


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, plim, smax, sm = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock_max": smax, "sm_clock_now": sm}
    except Exception as e:                          # the timing stands without it; say why it is missing
        return {"error": f"nvidia-smi query failed: {e}"}


def build(dev, n):
    """Warmed tx / rx encoders and a v1 decoder (bin/stream.py:56-77), with n stream slots on the stateful handles."""
    import torch
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    sd = S.symad_state_dict(seed=0)
    enc = []
    for _ in range(2):
        e = SymADStreamGenerator(**S.SYMAD_PARAMS)
        e.load_state_dict(sd)
        enc.append(e.eval().to(dev))
    d = HiFiGANStreamGenerator(**S.HIFIGAN_V1_PARAMS)
    d.load_state_dict(S.hifigan_state_dict(seed=1))
    d = d.eval().to(dev)
    tx, rx = enc
    tx.initial_encoder(8192, dev)
    d.initial_decoder(rx.initial_encoder(8192, dev))
    tx.set_streams(n)
    d.set_streams(n)
    torch.cuda.synchronize(dev)
    return tx, rx, d


def lockstep_step(c, x):
    tx, rx, d = c
    _, packed, _ = tx.quantize_fused(tx.encode(x), want_idx=False, want_packed=True, want_zq=False)
    return d.decode(rx.lookup_packed(packed))


def slot_step(c, chunks, streams):
    tx, rx, d = c
    z, frames = tx.encode_streams(chunks, streams)
    _, packed, _ = tx.quantize_fused(z, want_idx=False, want_packed=True, want_zq=False)
    return d.decode_streams(rx.lookup_packed(packed), frames, streams)


def per_launch(c, fn):
    """{op name: ms} summed over the encoder's and decoder's launches of one profiled step"""
    import torch
    tx, _, d = c
    for g in (tx, d):
        g.profile(True)
    fn()
    torch.cuda.synchronize()
    out = {}
    for tag, g in (("enc", tx), ("dec", d)):
        for name, ms, _ in g.profile_report():
            out[f"{tag}:{name}"] = out.get(f"{tag}:{name}", 0.0) + ms
        g.profile(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=3)
    ap.add_argument("--server_steps", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    from audiodec_b200.server import MultiStreamCodecServer, SessionCodecServer
    dev = torch.device("cuda:0")
    info = gpu_info(0)
    lock, slot = build(dev, CAP), build(dev, CAP)
    torch.manual_seed(0)
    x = 0.1 * torch.randn(CAP, 1, FS, device=dev)
    chunks = list(x.view(CAP, FS))

    # parity at full occupancy: both handles warmed the same way, the same chunks, two steps
    parity = True
    for _ in range(2):
        y_lock = lockstep_step(lock, x).view(CAP, -1)
        y_slot = torch.stack([y.view(-1) for y in slot_step(slot, chunks, list(range(CAP)))])
        parity &= bool(torch.equal(y_lock.view(torch.int32), y_slot.view(torch.int32)))

    arms = {"lockstep_256": lambda: lockstep_step(lock, x)}
    for k in OCCUPANCY:
        streams = list(range(0, CAP, CAP // k))[:k]
        arms[f"slots_{k}"] = lambda ks=[chunks[s] for s in streams], ss=streams: slot_step(slot, ks, ss)
    for fn in arms.values():
        fn()
    torch.cuda.synchronize(dev)
    times = {a: [] for a in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.regions):
        for a, fn in arms.items():
            e0.record()
            for _ in range(args.steps):
                fn()
            e1.record()
            e1.synchronize()
            times[a].append(e0.elapsed_time(e1) / args.steps)
    device = {a: {"ms_per_step": round(statistics.median(t), 4), "regions_ms": [round(v, 4) for v in t]} for a, t in times.items()}
    base = device["lockstep_256"]["ms_per_step"]
    for a, v in device.items():
        v["speedup_vs_lockstep"] = round(base / v["ms_per_step"], 2)

    # per-launch times at full occupancy: where a slot step differs from the lock-step step
    pl_lock, pl_slot = per_launch(lock, arms["lockstep_256"]), per_launch(slot, arms["slots_256"])
    deltas = sorted(((n, pl_slot.get(n, 0.0) - pl_lock.get(n, 0.0)) for n in set(pl_lock) | set(pl_slot)), key=lambda r: -abs(r[1]))

    # through the servers: 256 lock-step streams against the session server with k open streams, steps alternated by region
    rng = np.random.default_rng(1)
    frame = (0.1 * rng.standard_normal(FS)).astype(np.float32)
    srv_lock = MultiStreamCodecServer(*build(dev, 1), n_streams=CAP, frame_size=FS, sample_rate=SR, max_latency=1.0, device="cuda:0",
                                      wire=True)
    srv_sess = {}
    for k in OCCUPANCY:
        s = SessionCodecServer(*build(dev, 1), capacity=CAP, frame_size=FS, sample_rate=SR, max_latency=1.0, device="cuda:0", wire=True)
        ids = [s.open() for _ in range(k)]
        srv_sess[k] = (s, ids)
    servers = {"lockstep_256": (srv_lock, list(range(CAP)))}
    servers.update({f"slots_{k}": v for k, v in srv_sess.items()})
    host = {a: [] for a in servers}
    for r in range(args.regions + 1):
        for a, (srv, ids) in servers.items():
            srv.step_times.clear()
            for _ in range(args.server_steps):
                for s in ids:
                    srv.submit(s, frame)
                srv.step()
                for s in ids:
                    srv.poll(s)
            if r:                                    # region 0 warms the staging buffers
                host[a].append(1e3 * statistics.median(srv.step_times))
    server = {a: {"ms_per_step": round(statistics.median(t), 3), "regions_ms": [round(v, 3) for v in t]} for a, t in host.items()}
    base = server["lockstep_256"]["ms_per_step"]
    for a, v in server.items():
        v["speedup_vs_lockstep"] = round(base / v["ms_per_step"], 2)

    print(json.dumps({
        "gpu": info, "shape": {"capacity": CAP, "frame_size": FS, "sample_rate": SR, "model": "symAD + HiFi-GAN v1 (libritts v1), fp32",
                               "wire": True},
        "steps_per_region": args.steps, "regions": args.regions,
        "parity_full_occupancy_bit_exact": parity,
        "device_resident": device,
        "server_host_clock": server,
        "full_occupancy_launch_deltas_ms": [{"op": n, "slot_minus_lockstep_ms": round(d, 4), "lockstep_ms": round(pl_lock.get(n, 0.0), 4)}
                                            for n, d in deltas[:8]],
    }, indent=1))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
