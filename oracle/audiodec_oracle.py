"""ORACLE - test infrastructure only.  NOT part of the product path.

CPU restatement (torch fp32 on CPU, the same arithmetic backend the reference itself
calls: ``torch.nn.functional.conv1d / conv_transpose1d / matmul / embedding``) of the
reference's *streaming forward path*:

    encode -> quantize -> lookup -> decode      (demoFile.py:58-61)

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may
import this file; the product (``audiodec_b200/``) never does.

Parity status: **pinned** against outputs of the unmodified reference run in the build
container (``tests/golden/make_golden.py`` imports ``/root/reference`` and dumps the
vectors; ``tests/test_oracle_golden.py`` checks this file against them).  The reference
has no tests / golden vectors of its own (SURVEY.md section 4), so those dumps are the
only pin that exists.

Every function cites the reference file:line whose behaviour it restates.  Unlike the
reference (whose ``pad_buffer`` is shaped (1,C,P) and therefore batch-1 only,
layers/conv_layer.py:144-146), the state here is (B,C,P): ``set_batch`` repeats the
warmed batch-1 state, which the survey probed to be bit-identical per row.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- layers
def causal_conv1d_infer(x, weight, bias, state, stride=1, dilation=1, groups=1):
    """layers/conv_layer.py:153-156 (CausalConv1d.inference).
    x (B,Cin,T), state (B,Cin,P) with P=(k-1)*dilation -> (y, new_state)."""
    xx = torch.cat((state, x), -1)                      # :154
    p = state.shape[-1]
    new_state = xx[:, :, xx.shape[-1] - p:] if p > 0 else state  # :155
    y = F.conv1d(xx, weight, bias, stride=stride, padding=0, dilation=dilation, groups=groups)  # :156 / :55-64
    return y, new_state


def causal_convtr1d_infer(x, weight, bias, state, stride):
    """layers/conv_layer.py:194-197 (CausalConvTranspose1d.inference); weight (Cin,Cout,2*stride),
    state (B,Cin,1) = previous input frame."""
    xx = torch.cat((state, x), -1)                      # :195
    new_state = xx[:, :, -state.shape[-1]:]             # :196
    y = F.conv_transpose1d(xx, weight, bias, stride=stride, padding=0, output_padding=0)
    return y[:, :, stride:-stride], new_state           # :197


def fold_weight_norm(weight_g, weight_v):
    """torch.nn.utils.weight_norm with default dim=0 (HiFiGAN.py:193-203): w = g * v/||v||,
    norm over all dims but 0.  Recomputed on every forward in the reference; folded once here."""
    return torch._weight_norm(weight_v, weight_g, 0)


# --------------------------------------------------------------------------- RVQ
def vq_forward_index(x, embed):
    """layers/vq_module.py:90-104 (VectorQuantize.forward_index). x (...,D), embed (D,N)."""
    flatten = x.reshape(-1, embed.shape[0])
    dist = (flatten.pow(2).sum(1, keepdim=True)
            - 2 * flatten @ embed
            + embed.pow(2).sum(0, keepdim=True))        # :93-97 (python precedence: (2*flatten)@embed)
    _, ind = (-dist).max(1)                             # :98  first index on ties
    ind = ind.view(*x.shape[:-1])
    quantize = F.embedding(ind, embed.transpose(0, 1))  # :101
    quantize = x + (quantize - x)                       # :102 straight-through form kept: it changes rounding
    return quantize, ind, dist


def rvq_forward_index(x, embeds, flatten_idx=True, return_margins=False):
    """layers/vq_module.py:136-149 (ResidualVQ.forward_index). x (B,F,D) -> indices (Nq,B,F)
    (the reference then does ``.squeeze(1)`` which only removes B when B==1)."""
    residual = x
    quantized_out = 0.0
    all_idx, margins = [], []
    n = embeds[0].shape[1]
    for i, e in enumerate(embeds):
        q, ind, dist = vq_forward_index(residual, e)
        if return_margins:
            top2 = torch.topk(-dist, 2, dim=1).values
            margins.append(((top2[:, 0] - top2[:, 1]) / dist.min(1).values.abs().clamp_min(1e-30)).view(*ind.shape))
        residual = residual - q                          # :143
        quantized_out = quantized_out + q                # :144
        if flatten_idx:
            ind = ind + n * i                            # :145-146
        all_idx.append(ind)
    idx = torch.stack(all_idx)                           # :148
    if return_margins:
        return quantized_out, idx, torch.stack(margins)
    return quantized_out, idx


def rvq_lookup(idx, codebook):
    """layers/vq_module.py:159-161 with the flat codebook of :151-157."""
    return torch.sum(F.embedding(idx, codebook), dim=0, keepdim=(idx.dim() == 2))


# --------------------------------------------------------------------------- symAD autoencoder
class SymADOracle:
    """models/autoencoder/AudioDec.py:166-256 (StreamGenerator, codec='audiodec')."""

    def __init__(self, params, state_dict, dtype=torch.float32):
        """dtype: the precision every weight, state and activation is computed in (float64: the exact reference of the tests'
        precision checks; the default float32 is the reference's own arithmetic)."""
        self.p = dict(params)
        self.dtype = dtype
        self.sd = {k: v.detach().clone().to(dtype) for k, v in state_dict.items()}
        # use_weight_norm (symAAD, AudioDec.py:152-162): weight = g * v/||v||, recomputed per call in the reference
        for k in list(self.sd):
            if k.endswith("weight_g"):
                base = k[:-len("weight_g")]
                self.sd[base + "weight"] = fold_weight_norm(self.sd[k], self.sd[base + "weight_v"])
        # codec='activate_audiodec' (ActivateEncoder/ActivateDecoder, encoder.py:145-175, decoder.py:151-214)
        self.activate = self.p.get("codec", "audiodec") == "activate_audiodec"
        self.offline = False          # forward_*: CausalConvTranspose1d.forward pads with the first frame (conv_layer.py:189-192)
        self.state = OrderedDict()
        self.reset_buffer()
        self.embeds = [self.sd[f"quantizer.codebook.layers.{i}.embed"] for i in range(self.p["codebook_num"])]
        self.codebook = None

    # -- state ------------------------------------------------------------------
    def reset_buffer(self):                              # AudioDec.py:250-256
        self.state = OrderedDict((k[:-len(".pad_buffer")], torch.zeros_like(v))
                                 for k, v in self.sd.items() if k.endswith(".pad_buffer"))

    def set_batch(self, b):
        for k, v in self.state.items():
            if v.shape[0] != b:
                assert v.shape[0] == 1, "can only expand batch-1 state"
                self.state[k] = v.repeat(b, 1, 1)

    def to(self, device):
        """Move weights and causal state (bench.py's informational eager-GPU baseline: the same torch ops on a CUDA device)."""
        mv = lambda t: t.to(device) if torch.is_tensor(t) else t
        for name in ("sd", "w", "state"):
            d = getattr(self, name, None)
            if d is not None:
                for k in list(d):
                    d[k] = mv(d[k])
        for name in ("mean", "scale", "codebook"):
            if getattr(self, name, None) is not None:
                setattr(self, name, mv(getattr(self, name)))
        if getattr(self, "embeds", None) is not None:
            self.embeds = [mv(e) for e in self.embeds]
        return self

    def _ensure_batch(self, b):
        any_state = next(iter(self.state.values()))
        if any_state.shape[0] != b:
            self.set_batch(b)

    # -- building blocks ----------------------------------------------------------
    def _conv(self, name, x, stride=1, dilation=1, sub="conv"):
        w = self.sd[f"{name}.{sub}.weight"]
        b = self.sd.get(f"{name}.{sub}.bias")
        y, self.state[name] = causal_conv1d_infer(x, w, b, self.state[name], stride, dilation)
        return y

    def _res_unit(self, name, x, dilation):
        """models/autoencoder/modules/residual_unit.py:78-81; ELU alpha=1 (config: default)."""
        y = self._conv(f"{name}.conv1", F.elu(x), 1, dilation)
        y = F.conv1d(F.elu(y), self.sd[f"{name}.conv2.weight"], None)
        return x + y

    # -- API ------------------------------------------------------------------------
    def initial(self):                                   # vq_module.py:151-157
        cb = torch.stack([e.transpose(0, 1) for e in self.embeds])
        self.codebook = cb.reshape(-1, cb.size(-1))

    def initial_encoder(self, receptive_length):         # AudioDec.py:216-221
        self.initial()
        z = self.encode(torch.zeros(1, self.p["input_channels"], receptive_length))
        return self.lookup(self.quantize(z))

    def initial_decoder(self, zq):                       # AudioDec.py:224-225
        self.decode(zq)

    def encode(self, x):                                 # AudioDec.py:228-234 -> encoder.py:137-142, :76-81
        self._ensure_batch(x.shape[0])
        h = self._conv("encoder.conv", x.to(self.dtype))
        for i, s in enumerate(self.p["enc_strides"]):
            for j, d in enumerate((1, 3, 9)):
                h = self._res_unit(f"encoder.conv_blocks.{i}.res_units.{j}", h, d)
            h = self._conv(f"encoder.conv_blocks.{i}.conv", h, stride=s)
        if self.activate:
            h = F.elu(h)                                 # encoder.py:174-175
        return self._conv("projector.project", h)        # projector.py:52-54

    def quantize(self, z, return_margins=False):         # AudioDec.py:237-239 -> quantizer.py:42-44
        out = rvq_forward_index(z.transpose(2, 1), self.embeds, True, return_margins)
        idx = out[1]
        idx = idx.squeeze(1) if idx.shape[1] == 1 else idx   # vq_module.py:149 (B==1 only in the reference)
        return (idx, out[2]) if return_margins else idx

    def lookup(self, idx):                               # AudioDec.py:242-243
        if self.codebook is None:
            self.initial()
        return rvq_lookup(idx, self.codebook)

    def decode(self, zq):                                # AudioDec.py:246-247 -> decoder.py:142-148, :76-81
        self._ensure_batch(zq.shape[0])
        h = self._conv("decoder.conv1", zq.transpose(2, 1).to(self.dtype))
        for i, s in enumerate(self.p["dec_strides"]):
            n = f"decoder.conv_blocks.{i}.1" if self.activate else f"decoder.conv_blocks.{i}"
            if self.activate:
                h = F.elu(h)                             # decoder.py:207 conv_blocks[i][0]
            h, self.state[f"{n}.conv"] = causal_convtr1d_infer(
                h, self.sd[f"{n}.conv.deconv.weight"], self.sd.get(f"{n}.conv.deconv.bias"),
                h[:, :, :1] if self.offline else self.state[f"{n}.conv"], s)
            for j, d in enumerate((1, 3, 9)):
                h = self._res_unit(f"{n}.res_units.{j}", h, d)
        if self.activate:
            return torch.tanh(self._conv("decoder.conv2", F.elu(h)))      # decoder.py:209-211
        return self._conv("decoder.conv2", h)


    # -- non-streaming forward (codecTest.py:78-95): CausalConv1d.forward zero-pads on the left (conv_layer.py:148-151), which
    #    is inference() from an all-zero pad_buffer; CausalConvTranspose1d.forward replicates the first frame (:189-192)
    def _offline_call(self, fn, arg):
        self.reset_buffer()
        self.offline = True
        try:
            return fn(arg)
        finally:
            self.offline = False
            self.reset_buffer()

    def forward_encode(self, x):                         # encoder.py:131 + projector.py:49-50 (codecTest.py:84-85)
        return self._offline_call(self.encode, x)

    def forward_quantize(self, z):                       # quantizer.py:31-34 -> vq_module.py:119-134 (eval: same quantize as :136-149)
        return rvq_forward_index(z.transpose(2, 1), self.embeds)[0].transpose(2, 1)

    def forward_decode(self, zq):                        # decoder.py:135-140 (codecTest.py:94); zq (B,D,F) channels-first
        return self._offline_call(self.decode, zq.transpose(2, 1))


# --------------------------------------------------------------------------- HiFi-GAN vocoder (AD v1)
class HiFiGANOracle:
    """models/vocoder/HiFiGAN.py:222-305 (StreamGenerator) with MultiGroupConv1d blocks
    (models/vocoder/modules/multi_fusion.py:82-141, residual_block.py:23-105)."""

    def __init__(self, params, state_dict, dtype=torch.float32):
        """dtype: as SymADOracle's"""
        self.p = dict(params)
        self.dtype = dtype
        sd = {k: v.detach().clone().to(dtype) for k, v in state_dict.items()}
        self.w = {}
        for k in list(sd):
            if k.endswith("weight_g"):
                base = k[:-len("weight_g")]
                self.w[base + "weight"] = fold_weight_norm(sd[k], sd[base + "weight_v"])
            elif k.endswith(".weight") or k.endswith(".bias"):
                self.w[k] = sd[k]
        self.sd = sd
        self.mean, self.scale = sd.get("mean"), sd.get("scale")
        self.slope = self.p["nonlinear_activation_params"]["negative_slope"]
        self.offline = False
        self.state = OrderedDict()
        self.reset_buffer()

    def reset_buffer(self):                              # HiFiGAN.py:298-305
        self.state = OrderedDict((k[:-len(".pad_buffer")], torch.zeros_like(v))
                                 for k, v in self.sd.items() if k.endswith(".pad_buffer"))

    def set_batch(self, b):
        for k, v in self.state.items():
            if v.shape[0] != b:
                assert v.shape[0] == 1
                self.state[k] = v.repeat(b, 1, 1)

    def initial_decoder(self, c):                        # HiFiGAN.py:264-265
        self.decode(c)

    def to(self, device):
        """Move weights and causal state (bench.py's informational eager-GPU baseline: the same torch ops on a CUDA device)."""
        mv = lambda t: t.to(device) if torch.is_tensor(t) else t
        for name in ("sd", "w", "state"):
            d = getattr(self, name, None)
            if d is not None:
                for k in list(d):
                    d[k] = mv(d[k])
        for name in ("mean", "scale", "codebook"):
            if getattr(self, name, None) is not None:
                setattr(self, name, mv(getattr(self, name)))
        if getattr(self, "embeds", None) is not None:
            self.embeds = [mv(e) for e in self.embeds]
        return self

    def _conv(self, name, x, dilation=1, groups=1):
        y, self.state[name] = causal_conv1d_infer(
            x, self.w[f"{name}.conv.weight"], self.w.get(f"{name}.conv.bias"), self.state[name], 1, dilation, groups)
        return y

    def decode(self, c):                                 # HiFiGAN.py:268-296
        if next(iter(self.state.values())).shape[0] != c.shape[0]:
            self.set_batch(c.shape[0])
        c = c.to(self.dtype)
        if self.mean is not None:
            c = (c - self.mean) / self.scale             # :276-279
        c = self._conv("input_conv", c.transpose(2, 1))  # :282-284
        grp = self.p["groups"]
        for i, s in enumerate(self.p["upsample_scales"]):  # :287-291
            n = f"upsamples.{i}"
            c = F.leaky_relu(c, self.slope)
            c, self.state[n] = causal_convtr1d_infer(
                c, self.w[f"{n}.deconv.weight"], self.w.get(f"{n}.deconv.bias"),
                c[:, :, :1] if self.offline else self.state[n], s)
            if grp == 1 and len(self.p["resblock_kernel_sizes"]) > 1:
                # AD v0: MultiReceptiveField.inference (multi_fusion.py:73-79) over HiFiGANResidualBlock.inference
                # (residual_block.py:100-105)
                cs = 0.0
                for bk, dils in enumerate(self.p["resblock_dilations"]):
                    x = c
                    for j, d in enumerate(dils):
                        xt = self._conv(f"blocks.{i}.blocks.{bk}.convs1.{j}", F.leaky_relu(x, self.slope), d)
                        xt = self._conv(f"blocks.{i}.blocks.{bk}.convs2.{j}", F.leaky_relu(xt, self.slope), 1)
                        x = xt + x
                    cs = cs + x
                c = cs / len(self.p["resblock_dilations"])
                continue
            x = c.repeat(1, grp, 1)                      # multi_fusion.py:134
            for j, d in enumerate(self.p["resblock_dilations"][0]):   # :135-139
                xt = self._conv(f"blocks.{i}.convs1.{j}", F.leaky_relu(x, self.slope), d, grp)
                xt = self._conv(f"blocks.{i}.convs2.{j}", F.leaky_relu(xt, self.slope), 1, grp)
                x = xt + x
            c = F.conv1d(x, self.w[f"blocks.{i}.conv_out.weight"], None)   # :140
        c = self._conv("output_conv", F.leaky_relu(c, 0.01))   # :294-296 (nn.LeakyReLU() default slope, :116)
        return torch.tanh(c)

    def forward(self, c):                                # HiFiGAN.py:140-160 Generator.forward; c (B,in_channels,F) channels-first
        self.reset_buffer()
        self.offline = True
        try:
            return self.decode(c.transpose(2, 1))
        finally:
            self.offline = False
            self.reset_buffer()


# --------------------------------------------------------------------------- end-to-end helper
def hop_length(params):
    return math.prod(params["enc_strides"])              # utils/audiodec.py:58-62


class CodecOracle:
    """The three objects ``AudioDec`` holds after load_transmitter/load_receiver
    (bin/stream.py:56-77), warmed exactly the same way."""

    def __init__(self, enc_params, enc_sd, dec_params=None, dec_sd=None, receptive_length=8192):
        self.tx_encoder = SymADOracle(enc_params, enc_sd)
        self.tx_encoder.initial_encoder(receptive_length)            # stream.py:61
        self.rx_encoder = SymADOracle(enc_params, enc_sd)
        zq = self.rx_encoder.initial_encoder(receptive_length)       # stream.py:70
        if dec_sd is None:
            self.decoder = SymADOracle(enc_params, enc_sd)
        elif "input_conv.pad_buffer" in dec_sd:
            self.decoder = HiFiGANOracle(dec_params, dec_sd)
        else:
            self.decoder = SymADOracle(dec_params, dec_sd)
        self.decoder.initial_decoder(zq)                             # stream.py:76

    def run(self, x):
        """demoFile.py:58-61 on a (B,1,T) batch."""
        z = self.tx_encoder.encode(x)
        idx = self.tx_encoder.quantize(z)
        zq = self.rx_encoder.lookup(idx)
        y = self.decoder.decode(zq)
        return z, idx, zq, y
