"""Synthetic checkpoints for the AudioDec streaming path.

The reference ships no weights (only ``exp/**/config.yml`` and ``stats/*.npy``), so
parity tests, ``bench.py`` and ``smoke()`` all run on *synthetic* checkpoints.  This
module builds state-dicts with exactly the key set / shapes that the reference's
``StreamGenerator.load_state_dict(strict=True)`` expects
(``utils/audiodec.py:40-41,54-55``; key list probed from
``models/autoencoder/AudioDec.py:166`` and ``models/vocoder/HiFiGAN.py:222``) from
nothing but a seed, so that the same weights can be re-created on the GPU box where
``/root/reference`` does not exist.  Nothing here imports the reference.

Hyper-parameters below are the ``generator_params`` of the released experiment
configs (``exp/autoencoder/symAD_vctk_48000_hop300/config.yml:102-134``,
``exp/vocoder/AudioDec_v1_symAD_vctk_48000_hop300_clean/config.yml:102-130``).
"""
from __future__ import annotations

import hashlib
import os
from collections import OrderedDict

import torch
import yaml

SYMAD_PARAMS = dict(
    input_channels=1, output_channels=1, encode_channels=32, decode_channels=32,
    code_dim=64, codebook_num=8, codebook_size=1024, bias=True,
    enc_ratios=[2, 4, 8, 16], dec_ratios=[16, 8, 4, 2],
    enc_strides=[3, 4, 5, 5], dec_strides=[5, 5, 4, 3],
    mode="causal", codec="audiodec", projector="conv1d", quantier="residual_vq",
)

HIFIGAN_V1_PARAMS = dict(
    in_channels=64, out_channels=1, channels=512, kernel_size=7,
    upsample_scales=[5, 5, 4, 3], upsample_kernel_sizes=[10, 10, 8, 6],
    resblock_kernel_sizes=[11], resblock_dilations=[[1, 3, 5]], groups=3, bias=True,
    use_additional_convs=True, nonlinear_activation="LeakyReLU",
    nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True,
    stats="stats/synthetic.npy",
)

SYMAD_C16_PARAMS = dict(SYMAD_PARAMS, codebook_num=16, enc_strides=[2, 4, 5, 8], dec_strides=[8, 5, 4, 2])
SYMAAD_PARAMS = dict(SYMAD_PARAMS, codec="activate_audiodec", use_weight_norm=True)
HIFIGAN_V2_PARAMS = dict(HIFIGAN_V1_PARAMS, resblock_kernel_sizes=[3])
HIFIGAN_V0_PARAMS = dict(HIFIGAN_V1_PARAMS, groups=1, resblock_kernel_sizes=[3, 7, 11],
                         resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]])

# model name -> (sample_rate, encoder tag, encoder steps, decoder kind, decoder tag, decoder steps)
# mirrors the table in utils/audiodec.py:109-179 (only the entries this repo implements).
MODEL_TABLE = {
    "vctk_sym": (48000, "symAD_vctk_48000_hop300", 200000, "autoencoder", "symAD_vctk_48000_hop300", 700000),
    "vctk_v1": (48000, "symAD_vctk_48000_hop300", 200000, "vocoder", "AudioDec_v1_symAD_vctk_48000_hop300_clean", 500000),
    "libritts_sym": (24000, "symAD_libritts_24000_hop300", 500000, "autoencoder", "symAD_libritts_24000_hop300", 1000000),
    "libritts_v1": (24000, "symAD_libritts_24000_hop300", 500000, "vocoder", "AudioDec_v1_symAD_libritts_24000_hop300_clean", 500000),
    "vctk_v0": (48000, "symAD_vctk_48000_hop300", 200000, "vocoder", "AudioDec_v0_symAD_vctk_48000_hop300_clean", 500000),
    "vctk_v2": (48000, "symAD_vctk_48000_hop300", 200000, "vocoder", "AudioDec_v2_symAD_vctk_48000_hop300_clean", 500000),
    "vctk_activate_sym": (48000, "symAAD_vctk_48000_hop300", 200000, "autoencoder", "symAAD_vctk_48000_hop300", 700000),
    "vctk_c16h320_sym": (48000, "symAD_c16_vctk_48000_hop320", 500000, "autoencoder", "symAD_c16_vctk_48000_hop320", 1000000),
}
# which generator_params each checkpoint directory uses
ENCODER_PARAMS = {"symAAD_vctk_48000_hop300": SYMAAD_PARAMS, "symAD_c16_vctk_48000_hop320": SYMAD_C16_PARAMS}
VOCODER_PARAMS = {"AudioDec_v0_symAD_vctk_48000_hop300_clean": HIFIGAN_V0_PARAMS,
                  "AudioDec_v2_symAD_vctk_48000_hop300_clean": HIFIGAN_V2_PARAMS}


def _randn(gen, *shape, std=1.0):
    return torch.randn(*shape, generator=gen, dtype=torch.float32) * std


def symad_state_dict(params=None, seed=0, codebook_scale=None):
    """State dict of ``models.autoencoder.AudioDec.StreamGenerator`` (symAD).

    Weight scales are chosen so that activations stay O(1) through the 60 conv layers
    and the residual-VQ sees residual norms comparable to its codeword norms (the
    default torch init gives |z| ~ 0.05 against randn codebooks, which makes every
    nearest-neighbour decision degenerate - SURVEY.md section 8(c))."""
    p = dict(SYMAD_PARAMS if params is None else params)
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    ec, dc = p["encode_channels"], p["decode_channels"]
    k = 7

    wn = bool(p.get("use_weight_norm", False))          # symAAD: every conv is weight-normed (AudioDec.py:152-162)
    act = p.get("codec", "audiodec") == "activate_audiodec"

    def put_weight(key, w):
        """plain `weight`, or an equivalent (weight_g, weight_v) pair: w = g * v/||v|| over dims != 0"""
        if not wn:
            sd[key + ".weight"] = w
        else:
            sd[key + ".weight_g"] = w.flatten(1).norm(dim=1).reshape(-1, 1, 1)
            sd[key + ".weight_v"] = w * (0.5 + torch.rand(w.shape[0], 1, 1, generator=g))   # any per-row rescale of v

    def conv(prefix, cout, cin, ks, bias, gain=1.0, dil=1, sub="conv"):
        sd[f"{prefix}.pad_buffer"] = torch.zeros(1, cin, (ks - 1) * dil)
        put_weight(f"{prefix}.{sub}", _randn(g, cout, cin, ks, std=gain / (cin * ks) ** 0.5))
        if bias:
            sd[f"{prefix}.{sub}.bias"] = _randn(g, cout, std=0.1)

    def res_unit(prefix, c, dil):
        conv(f"{prefix}.conv1", c, c, k, False, gain=1.2, dil=dil)
        put_weight(f"{prefix}.conv2", _randn(g, c, c, 1, std=0.6 / c ** 0.5))

    # encoder (models/autoencoder/modules/encoder.py:84-142)
    conv("encoder.conv", ec, p["input_channels"], k, False, gain=3.0)
    cin = ec
    for i, s in enumerate(p["enc_strides"]):
        cout = ec * p["enc_ratios"][i]
        for j, d in enumerate((1, 3, 9)):
            res_unit(f"encoder.conv_blocks.{i}.res_units.{j}", cin, d)
        conv(f"encoder.conv_blocks.{i}.conv", cout, cin, 2 * s, p["bias"], gain=0.8)
        cin = cout
    enc_out = cin
    # decoder (models/autoencoder/modules/decoder.py:84-148)
    conv("decoder.conv1", dc * p["dec_ratios"][0], p["code_dim"], k, False, gain=1.0)
    for i, s in enumerate(p["dec_strides"]):
        cin = dc * p["dec_ratios"][i]
        cout = dc * p["dec_ratios"][i + 1] if i < len(p["dec_strides"]) - 1 else dc
        pre = f"decoder.conv_blocks.{i}.1" if act else f"decoder.conv_blocks.{i}"     # decoder.py:183-195: Sequential(act, block)
        sd[f"{pre}.conv.pad_buffer"] = torch.zeros(1, cin, 1)
        put_weight(f"{pre}.conv.deconv", _randn(g, cin, cout, 2 * s, std=0.8 / (2 * cin) ** 0.5))
        if p["bias"]:
            sd[f"{pre}.conv.deconv.bias"] = _randn(g, cout, std=0.1)
        for j, d in enumerate((1, 3, 9)):
            res_unit(f"{pre}.res_units.{j}", cout, d)
    conv("decoder.conv2", p["output_channels"], dc, k, False, gain=0.25)
    # projector (models/autoencoder/modules/projector.py:40)
    conv("projector.project", p["code_dim"], enc_out, 3, False, gain=1.0)
    # residual VQ codebooks (layers/vq_module.py:40-43)
    cs = 0.55 if codebook_scale is None else codebook_scale
    for i in range(p["codebook_num"]):
        e = _randn(g, p["code_dim"], p["codebook_size"], std=cs * 0.88 ** i)
        sd[f"quantizer.codebook.layers.{i}.embed"] = e
        sd[f"quantizer.codebook.layers.{i}.cluster_size"] = torch.zeros(p["codebook_size"])
        sd[f"quantizer.codebook.layers.{i}.embed_avg"] = e.clone()
    # preserve the reference's key order where load_state_dict does not care; it does not.
    return sd


def hifigan_state_dict(params=None, seed=1):
    """State dict of ``models.vocoder.HiFiGAN.StreamGenerator`` (AD v1: MultiGroupConv1d,
    weight-normed: ``weight_g``/``weight_v`` pairs, HiFiGAN.py:193-203)."""
    p = dict(HIFIGAN_V1_PARAMS if params is None else params)
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    ch, grp = p["channels"], p["groups"]
    ks = p["kernel_size"]
    rk = p["resblock_kernel_sizes"][0]
    dils = p["resblock_dilations"][0]
    sd["mean"] = _randn(g, p["in_channels"], std=0.2)
    sd["scale"] = 1.0 + 0.5 * torch.rand(p["in_channels"], generator=g)

    def wn_conv(prefix, cout, cin_g, k, bias, gain, dil=1, sub="conv", cin_total=None, pad=True):
        if pad:
            sd[f"{prefix}.pad_buffer"] = torch.zeros(1, cin_total or cin_g, (k - 1) * dil)
        if bias:
            sd[f"{prefix}.{sub}.bias"] = _randn(g, cout, std=0.05)
        v = _randn(g, cout, cin_g, k, std=1.0)
        # effective weight = g * v/||v||; ||v|| ~ sqrt(cin_g*k) so g ~ gain gives std ~ gain/sqrt(fan_in)
        sd[f"{prefix}.{sub}.weight_g"] = (gain * (0.75 + 0.5 * torch.rand(cout, 1, 1, generator=g)))
        sd[f"{prefix}.{sub}.weight_v"] = v

    wn_conv("input_conv", ch, p["in_channels"], ks, True, gain=1.0)
    for i, s in enumerate(p["upsample_scales"]):
        cin, cout = ch // 2 ** i, ch // 2 ** (i + 1)
        pre = f"upsamples.{i}"
        sd[f"{pre}.pad_buffer"] = torch.zeros(1, cin, 1)
        sd[f"{pre}.deconv.bias"] = _randn(g, cout, std=0.05)
        # weight norm over dims (1,2) of (Cin,Cout,K): one g per INPUT channel
        sd[f"{pre}.deconv.weight_g"] = 1.4 * (cout * 2 * s) ** 0.5 / (2 * cin) ** 0.5 * (0.75 + 0.5 * torch.rand(cin, 1, 1, generator=g))
        sd[f"{pre}.deconv.weight_v"] = _randn(g, cin, cout, 2 * s, std=1.0)
        if grp == 1 and len(p["resblock_kernel_sizes"]) > 1:
            # AD v0: MultiReceptiveField = mean of one HiFiGANResidualBlock per kernel size (multi_fusion.py:23-79)
            for b, (rkb, dilb) in enumerate(zip(p["resblock_kernel_sizes"], p["resblock_dilations"])):
                for j, d in enumerate(dilb):
                    wn_conv(f"blocks.{i}.blocks.{b}.convs1.{j}", cout, cout, rkb, p["bias"], gain=0.9, dil=d)
                for j, d in enumerate(dilb):
                    wn_conv(f"blocks.{i}.blocks.{b}.convs2.{j}", cout, cout, rkb, p["bias"], gain=0.5, dil=1)
            continue
        c3 = cout * grp
        for j, d in enumerate(dils):
            wn_conv(f"blocks.{i}.convs1.{j}", c3, cout, rk, p["bias"], gain=0.9, dil=d, cin_total=c3)
        for j, d in enumerate(dils):
            wn_conv(f"blocks.{i}.convs2.{j}", c3, cout, rk, p["bias"], gain=0.5, dil=1, cin_total=c3)
        wn_conv(f"blocks.{i}.conv_out", cout, c3, 1, False, gain=1.0, pad=False, sub="__none__")
        # Conv1d1x1 is the module itself (no ".conv" sub-module): rename keys
        for nm in ("weight_g", "weight_v"):
            sd[f"blocks.{i}.conv_out.{nm}"] = sd.pop(f"blocks.{i}.conv_out.__none__.{nm}")
    wn_conv("output_conv", p["out_channels"], ch // 2 ** len(p["upsample_scales"]), ks, True, gain=0.7)
    return sd


def state_dict_digest(sd) -> str:
    """sha256 over keys+raw bytes: pins that regenerated weights equal the ones the golden
    vectors were produced with."""
    h = hashlib.sha256()
    for k_, v in sd.items():
        h.update(k_.encode())
        h.update(v.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def write_checkpoint(root, kind, tag, steps, model_type, params, sd, sampling_rate):
    """Write ``<root>/exp/<kind>/<tag>/{config.yml,checkpoint-<steps>steps.pkl}`` in the layout
    the reference loader reads (bin/stream.py:48-53, utils/audiodec.py:40-41)."""
    d = os.path.join(root, "exp", kind, tag)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "config.yml"), "w") as f:
        yaml.safe_dump({"model_type": model_type, "sampling_rate": sampling_rate,
                        "generator_params": params}, f)
    path = os.path.join(d, f"checkpoint-{steps}steps.pkl")
    torch.save({"model": {"generator": sd}}, path)
    return path


def make_wav_corpus(root, seed, lengths, sr=48000):
    """Write len(lengths) mono PCM16 wav files of lengths[i] samples under ``root``, spread over nested folders
    (``spk<i % 3>/[sess<i % 2>/]utt_<i>.wav``), from nothing but the seed: band-limited noise with a per-file level and a
    per-file DC offset, so that every code channel has a mean and a spread.  Returns the paths in the order of ``lengths``."""
    import numpy as np
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    paths = []
    for i, n in enumerate(lengths):
        d = os.path.join(root, f"spk{i % 3}", f"sess{i % 2}") if i % 4 else os.path.join(root, f"spk{i % 3}")
        os.makedirs(d, exist_ok=True)
        level, dc = 0.05 + 0.25 * rng.random(), 0.02 * rng.standard_normal()
        # brown noise minus its trailing 64-sample mean; cumulative sums and element-wise arithmetic only (no BLAS, whose
        # summation order depends on the CPU), so the bytes are the same on every machine
        x = np.cumsum(rng.standard_normal(int(n))) * 0.05
        c = np.concatenate([np.zeros(64), np.cumsum(x)])
        x = x - (c[64:] - c[:-64]) / 64.0
        x = level * x / max(1e-9, np.abs(x).max()) + dc
        pcm = np.clip(np.rint(x * 32767.0), -32768, 32767).astype(np.int16)
        p = os.path.join(d, f"utt_{i:04d}.wav")
        wavfile.write(p, int(sr), pcm)
        paths.append(p)
    return paths


def make_model_zoo(root, model="vctk_sym", seed=0):
    """Create the synthetic checkpoint tree for one ``assign_model`` name under ``root``.
    Returns (sample_rate, encoder_checkpoint, decoder_checkpoint) as absolute paths."""
    import numpy as np
    sr, etag, esteps, dkind, dtag, dsteps = MODEL_TABLE[model]
    eparams = dict(ENCODER_PARAMS.get(etag, SYMAD_PARAMS))
    enc_sd = symad_state_dict(eparams, seed=seed)
    enc = write_checkpoint(root, "autoencoder", etag, esteps, "symAudioDec", eparams, enc_sd, sr)
    if dkind == "autoencoder":
        dec = write_checkpoint(root, "autoencoder", dtag, dsteps, "symAudioDec", eparams, enc_sd, sr)
    else:
        vparams = dict(VOCODER_PARAMS.get(dtag, HIFIGAN_V1_PARAMS))
        dec_sd = hifigan_state_dict(vparams, seed=seed + 1)
        os.makedirs(os.path.join(root, "stats"), exist_ok=True)
        np.save(os.path.join(root, "stats", "synthetic.npy"),
                np.stack([dec_sd["mean"].numpy(), dec_sd["scale"].numpy()]).astype("float32"))
        dec = write_checkpoint(root, "vocoder", dtag, dsteps, "HiFiGAN", vparams, dec_sd, sr)
    return sr, enc, dec
