"""The released fp32 decoders and vocoders, whole, against the oracle in fp64: symAD, symAAD and c16 on SymADStreamGenerator, HiFi-GAN
v0 / v1 / v2 on HiFiGANStreamGenerator, built from the parity tests' synthetic checkpoints by the real plan, on every fp32-grade
engine (f16 split, 3xTF32, FFMA).

The decoder is warmed as load_receiver warms it (bin/stream.py:70-76): the kernel's rx_encoder.initial_encoder(8192) gives the warm
zq, which must equal the fp32 oracle's, and that one fp32 tensor warms the kernel, the fp32 oracle and the fp64 oracle alike.  Three
fp32 latent sequences go to all three identically:
  golden   the model's golden clip through its own warm encoder (indices equal to the golden file's), then lookup;
  codes    160 frames of codes drawn uniformly per stage, then lookup;
  playout  what a playout receiver decodes: real frames, three frames concealed toward the next real frame, a fade toward the
           codec's silence frame that runs past j >= den, eight silence frames, real frames again (rows as test_playout_cpu.interp
           computes them in fp32).
Each runs in every call mode against the fp64 oracle run the same way: one streaming call, streaming chunks of 1 and 7 frames (and 5,
configs[3]'s chunk, for HiFi-GAN), and offline.  The bar is test_models_fp64_cpu.check_model: max |y - y64| <= factor * max(e32,
2^-23 max |y64|) with e32 the fp32 oracle's own error, factor 4 on the tensor-core engines (the op tests' factor) and 8 on FFMA,
whose serial FMA chains err more on the long-K ops.  After the last call of each streaming mode every live pad_buffer is held to the
same rule against the oracle's state (check_states), so a failure names the first layer that went wrong.  The chunked waveforms must
equal the one-call waveform bit for bit."""
import time
from collections import OrderedDict

import numpy as np
import pytest
import torch

from test_models_fp64_cpu import (GOLDEN, MODELS, RECEPTIVE, check_model, check_states, elu_keys, golden_x, oracle_warm_zq,
                                  run_oracle, weights)
from test_playout_cpu import interp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FACTOR = {"f16": 4.0, "tf32": 4.0, "ffma": 8.0}
CODES_FRAMES = 160
REPORT = []


def _gen(model, which):
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    ep, esd, vp, vsd = weights(model)
    g = HiFiGANStreamGenerator(**vp) if which == "decoder" and vp is not None else SymADStreamGenerator(**ep)
    g.load_state_dict(vsd if which == "decoder" and vp is not None else esd)
    return g.eval().to(DEV)


def _decoder(model, zq_warm):
    d = _gen(model, "decoder")
    d.initial_decoder(zq_warm.to(DEV))
    return d


def playout_latents(real, silence):
    """(R, D) float32: real frames 0-9; three frames concealed toward frame 10 (j = 1..3, den = 4); frames 10-15; a fade from frame 15
    toward the silence frame, j = 1..6 over den = 4 (j >= den plays the silence frame itself); eight silence frames; frames 16 on"""
    rows = list(real[:10])
    rows += [interp(real[9], real[10], j, 4) for j in (1, 2, 3)]
    rows += list(real[10:16])
    rows += [silence if j >= 4 else interp(real[15], silence, j, 4) for j in range(1, 7)]
    rows += [silence] * 8 + list(real[16:])
    return np.stack(rows).astype(np.float32)


def latents(model, rx):
    """{"golden", "codes", "playout"} -> fp32 zq (1, F, D) on the CPU, from the kernel's encoder and lookup"""
    ep, _, _, _ = weights(model)
    tx = _gen(model, "encoder")
    tx.initial_encoder(RECEPTIVE, DEV)
    idx = tx.quantize(tx.encode(golden_x(model).to(DEV)))
    np.testing.assert_array_equal(idx.cpu().numpy(), np.load(f"{GOLDEN}/{MODELS[model][2]}")["idx"])
    golden = rx.lookup(idx).cpu()
    nq, n = ep["codebook_num"], ep["codebook_size"]
    codes = np.random.default_rng(160).integers(0, n, (nq, CODES_FRAMES)) + n * np.arange(nq)[:, None]
    codes = rx.lookup(torch.from_numpy(codes).to(DEV)).cpu()
    playout = playout_latents(golden[0].numpy(), rx.silence_frame().cpu().numpy())
    return {"golden": golden, "codes": codes, "playout": torch.from_numpy(playout)[None]}


@pytest.fixture(scope="module")
def cache():
    """the latents of the first engine, and the fp32 / fp64 oracle results, shared by the engines"""
    return {}


def _references(cache, model, latent, zq, zq_warm, mode):
    key = (model, latent, mode)
    if key not in cache:
        cache[key] = run_oracle(model, torch.float32, zq, zq_warm, mode) + run_oracle(model, torch.float64, zq, zq_warm, mode)
    return cache[key]


@pytest.mark.parametrize("latent", ["golden", "codes", "playout"])
@pytest.mark.parametrize("model", list(MODELS))
def test_model_against_fp64(model, latent, conv_path, cache):
    t0 = time.time()
    factor = FACTOR[conv_path]
    hifigan = weights(model)[2] is not None
    rx = _gen(model, "encoder")
    zq_warm = rx.initial_encoder(RECEPTIVE, DEV).cpu()
    if ("warm", model) not in cache:
        cache[("warm", model)] = oracle_warm_zq(model)
    assert torch.equal(zq_warm, cache[("warm", model)]), "the kernel's warm zq differs from the fp32 oracle's"
    lat = latents(model, rx)
    for k, v in cache.setdefault(("latents", model), lat).items():
        assert torch.equal(lat[k], v), f"{conv_path}: the {k} latents differ from the first engine's"
    zq = lat[latent]
    F_ = zq.shape[1]
    failures = []
    y_one = None
    for mode in ["stream", 1, 7] + ([5] if hifigan else []) + ["offline"]:
        y32, st32, y64, st64 = _references(cache, model, latent, zq, zq_warm, mode)
        if mode == "offline":
            dec = _gen(model, "decoder")
            zc = zq.transpose(1, 2).to(DEV)
            y = (dec.forward(zc) if hifigan else dec.decode_offline(zc)).cpu()
        else:
            dec = _decoder(model, zq_warm)
            n = F_ if mode == "stream" else mode
            y = torch.cat([dec.decode(zq[:, i:i + n].to(DEV)) for i in range(0, F_, n)], -1).cpu()
        ok, e, e32, bar = check_model(y, y32, y64, factor)
        name = mode if isinstance(mode, str) else f"chunks {mode}"
        line = f"{model:6s} {conv_path:5s} {latent:7s} {name:9s} e = {e:.3g}  e32 = {e32:.3g}  e/e32 = {e / e32:.2f}"
        if not ok:
            failures.append(f"{line}: over the bar {bar:.3g}")
        if mode != "offline":
            keys = [k for k, _, _ in dec.state_layout]
            assert sorted(keys) == sorted(st64), "the handle's state map and the oracle's pad_buffers differ"
            sd = dec.state_dict()
            bad, rows = check_states({k: sd[k].cpu() for k in keys}, st32, OrderedDict((k, st64[k]) for k in keys), factor,
                                     elu_keys(model))
            share = lambda r: r[1] / r[3] if r[3] else 0.0
            worst = max(rows, key=share)
            line += f"  states: worst {worst[0]} e = {worst[1]:.3g} e32 = {worst[2]:.3g} ({share(worst):.2f} of its bar)"
            if bad is not None:
                k, es, es32, sbar = next(r for r in rows if r[0] == bad)
                failures.append(f"{line}: first failing state {bad}: e = {es:.3g} over its bar {sbar:.3g} (e32 = {es32:.3g})")
        if mode == "stream":
            y_one = y
        elif mode != "offline" and not torch.equal(y, y_one):
            failures.append(f"{line}: chunks of {mode} differ from one call by up to {(y - y_one).abs().max().item():.3g}")
        REPORT.append(line)
        print(line)
    print(f"{model} {conv_path} {latent}: {time.time() - t0:.1f} s")
    assert not failures, "\n".join(failures)
