"""Host-side mirrors of the reference's streaming generators, backed by the C-ABI library.

``SymADStreamGenerator`` stands in for ``models/autoencoder/AudioDec.py:166 StreamGenerator`` and
``HiFiGANStreamGenerator`` for ``models/vocoder/HiFiGAN.py:222 StreamGenerator``: same constructor
keywords (``config.yml`` ``generator_params``), same methods with the same tensor shapes
(``load_state_dict / eval / to / initial_encoder / initial_decoder / encode / quantize / lookup /
decode / reset_buffer``), so the objects can be returned from ``AudioCodec._load_encoder /
_load_decoder`` (bin/stream.py:38-45) unchanged.  All arithmetic happens in hand-written sm_90a
kernels (audiodec_b200/csrc); torch only provides device memory and the current stream.

Differences from the reference, all extensions:
  * batches: the reference's streaming state is (1,C,P) so only B=1 works (layers/conv_layer.py:144-146);
    here a batch of B independent streams is allowed.  A handle warmed with one stream replicates its
    state when first called with B>1.  ``quantize`` then returns (Nq,B,F) (what
    ``ResidualVQ.forward_index`` yields before its ``squeeze(1)``, vq_module.py:148-149) and ``lookup``
    returns (B,F,D).
  * there is no CPU path: ``.to('cpu')`` raises.
  * ``stream_state`` / ``load_stream_state`` move one stream's causal state out of and into any stream of a handle (of the same
    config and dtype, on any GPU); ``state_dict()`` returns the live state of every stream as the reference's pad_buffers.
  * ``set_activation_dtype(torch.bfloat16)`` on a decoder-only generator (``HiFiGANStreamGenerator``,
    ``SymADDecoderStreamGenerator``) keeps every activation, the causal state and the decode input / output in bf16 (the data
    layout and dtype contract of the reference's ``decoder.to(torch.bfloat16)``); plain ``.to(torch.bfloat16)`` rounds only the
    conv operands and keeps fp32 activations and fp32 I/O.  ``SymADDecoderStreamGenerator`` is the symAD decoder alone, the
    object the reference's receiver decodes with; a full ``SymADStreamGenerator`` stays fp32-grade.
  * ``SymADEncoderStreamGenerator`` is the symAD transmitter alone (encoder, projector and RVQ search), the reference's
    ``tx_encoder``.  Its ``.to(torch.bfloat16)`` runs the encoder's convs on bf16 operands with fp32 activations, state, x and z.
"""
from __future__ import annotations

import ctypes
import inspect

import numpy as np
import torch

from . import _lib


def _check(rc, handle):
    if rc != 0:
        raise RuntimeError("audiodec_b200: " + _lib.last_error(handle))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _fill(arr, values):
    for i, v in enumerate(values):
        arr[i] = int(v)


def varlen_layout(lengths, strides):
    """Frame counts and column offsets of a varlen batch: F_b = frames_for(T_b) (floor((t - 1) / s) + 1 per stride, conv_layer.py:153-156)
    and offsets[b] = sum_{i<b} F_i, B + 1 entries.  Utterance b's frames are columns [offsets[b], offsets[b + 1]) of the varlen z / zq;
    times the hop, the same offsets place its samples in the decoded waveform."""
    frames, offsets = [], [0]
    for t in lengths:
        t = int(t)
        for s in strides:
            t = (t - 1) // s + 1
        frames.append(t)
        offsets.append(offsets[-1] + t)
    return frames, offsets


def _int_array(values):
    values = [int(v) for v in values]
    return (ctypes.c_int * max(1, len(values)))(*values), len(values)


def _stream_ids(streams):
    """An int or an iterable of ints -> list of ints (the handle checks that they are distinct and in range)."""
    if isinstance(streams, int):
        return [streams]
    ids = list(streams)
    for s in ids:
        if isinstance(s, bool) or not isinstance(s, int):
            raise TypeError(f"audiodec_b200: stream ids must be ints, got {type(s).__name__}")
    return ids


def _check_state(state, n, elems, dtype, device):
    """An imported state: a (n, elems) tensor of the handle's state dtype on the handle's device, returned contiguous and 16-byte aligned."""
    if not isinstance(state, torch.Tensor):
        raise TypeError(f"audiodec_b200: load_stream_state: expected a tensor, got {type(state).__name__}")
    if state.device != device:
        raise RuntimeError(f"audiodec_b200: load_stream_state: the state is on {state.device}, the codec on {device}; move it with .to()")
    if state.dtype != dtype:
        raise ValueError(f"audiodec_b200: load_stream_state: the state is {state.dtype}, this handle's state is {dtype}")
    if tuple(state.shape) != (n, elems):
        raise ValueError(f"audiodec_b200: load_stream_state: expected ({n}, {elems}) for {n} streams, got {tuple(state.shape)}")
    state = state.contiguous()
    return state.clone() if state.data_ptr() % 16 else state


class _StreamGeneratorBase:
    """Common plumbing: deferred handle creation (weights arrive before the device is known, exactly
    like ``Generator(**params)`` -> ``load_state_dict`` -> ``.to(device)`` in the reference)."""

    def __init__(self):
        self._lib = _lib.load()
        self._cfg = _lib.AdecConfig()
        self._sd = None
        self._h = None
        self._device = None
        self._operand_mode = 0        # what .to(dtype) selected: 0 = fp32, 1 = bf16 conv operands
        self._act_bf16 = False        # decoders only (set_activation_dtype): bf16 activations, state and decode I/O = compute_dtype 2
        self._layout = None           # state_layout, read from the handle once

    # the decoder-only generators (HiFi-GAN vocoder, symAD decoder) and the symAD encoder-only generator have the bf16 modes; a full
    # symAD generator does not
    _bf16_modes = False

    # -- torch.nn.Module look-alikes ------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True):
        """Weights, stats, codebooks and pad_buffers as the reference's state dict names them.  A pad_buffer (1, C, P) is every stream's
        initial state; a batched one (B, C, P) with B > 1 (what state_dict() returns for B streams) gives stream b its row b: the handle
        gets B streams in `.to(device)`."""
        self._sd = {k: v.detach().to(torch.float32).cpu().contiguous() for k, v in state_dict.items()}
        return self

    def state_dict(self):
        """Every key as loaded, except the pad_buffers of the layers the handle runs: those are the live causal state of every stream,
        (n_streams, C, P) device tensors (fp32; bf16 with bf16 activations, as `.to(torch.bfloat16)` stores them in the reference), read
        in one launch.  `load_state_dict` of the result into a fresh generator resumes every stream exactly."""
        if self._sd is None:
            raise RuntimeError("load_state_dict must be called before state_dict")
        live = {}
        if self._h is not None and self.state_layout:
            n = self.n_streams
            st = self.stream_state(range(n))
            off = 0
            for key, c, p in self.state_layout:
                live[key] = st[:, off:off + c * p].view(n, c, p)
                off += c * p
        out = {k: live.pop(k, v) for k, v in self._sd.items()}
        out.update(live)
        return out

    def eval(self):
        return self

    def to(self, device):
        if isinstance(device, torch.dtype):
            return self._set_dtype(device)
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("audiodec_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        if self._sd is None:
            raise RuntimeError("load_state_dict must be called before .to(device)")
        if self._h is not None:
            if device.index not in (None, self._device.index):
                raise RuntimeError("handle already lives on " + str(self._device))
            return self
        index = device.index if device.index is not None else torch.cuda.current_device()
        self._device = torch.device("cuda", index)
        h = ctypes.c_void_p()
        rc = self._lib.adec_create(ctypes.byref(self._cfg), index, ctypes.byref(h))
        if rc != 0:
            raise RuntimeError("audiodec_b200: " + _lib.last_error(None))
        self._h = h
        for key, t in self._sd.items():
            shape = (ctypes.c_int64 * t.dim())(*t.shape)
            _check(self._lib.adec_set_tensor(h, key.encode(), _ptr(t), shape, t.dim()), h)
        _check(self._lib.adec_finalize(h), h)
        self._load_batched_pad_buffers()
        return self

    def _load_batched_pad_buffers(self):
        """(B, C, P) pad_buffers with B > 1: the handle (which started every stream from row 0) gets B streams, and stream b row b of
        each such buffer, in one import."""
        names = {key for key, _, _ in self.state_layout}
        rows = {k: v for k, v in self._sd.items() if k in names and v.dim() == 3 and v.size(0) > 1}
        if not rows:
            return
        sizes = {v.size(0) for v in rows.values()}
        if len(sizes) != 1:
            raise ValueError(f"audiodec_b200: load_state_dict: batched pad_buffers disagree on the number of streams {sorted(sizes)}")
        b = sizes.pop()
        self._batch(b)
        st = self.stream_state(range(b))
        off = 0
        for key, c, p in self.state_layout:
            if key in rows:
                if tuple(rows[key].shape) != (b, c, p):
                    raise ValueError(f"audiodec_b200: load_state_dict: {key} has shape {tuple(rows[key].shape)}, the handle runs {(b, c, p)}")
                st[:, off:off + c * p] = rows[key].reshape(b, c * p).to(self._device, st.dtype)
            off += c * p
        self.load_stream_state(range(b), st)

    def _set_dtype(self, dtype):
        """`module.to(torch.bfloat16)` of the reference: only the decoder-only generators (HiFi-GAN vocoder, symAD decoder) have a
        reduced-precision mode (bf16 conv operands, fp32 accumulation and fp32 activations in HBM); the encoder / projector / RVQ must
        stay fp32-grade for bit-identical indices."""
        if dtype == torch.float32:
            want = 0
        elif dtype == torch.bfloat16 and self._bf16_modes:
            want = 1
        else:
            raise NotImplementedError(f"{type(self).__name__} has no {dtype} mode (fp32 everywhere; bf16 for the decoder-only generators: "
                                      "HiFiGANStreamGenerator, SymADDecoderStreamGenerator, and the encoder-only SymADEncoderStreamGenerator)")
        mode = 2 if self._act_bf16 else want
        if self._h is not None and mode != self._cfg.compute_dtype:
            raise RuntimeError("set the compute dtype before .to(device): the weights are packed when the handle is created")
        self._operand_mode = want
        self._cfg.compute_dtype = mode
        return self

    def set_activation_dtype(self, dtype):
        """torch.bfloat16: every activation, the causal state, and decode's zq input and y output are bf16 (conv operands bf16, fp32
        accumulation, one rounding per stored value) - what the reference's `decoder.to(torch.bfloat16)` stores and returns.
        torch.float32: back to fp32 activations with the operand precision `.to(dtype)` chose.  Call before `.to(device)`; returns
        self, so `d.set_activation_dtype(torch.bfloat16).to(dev)` chains.  Decoder-only generators only."""
        if not self._bf16_modes:
            raise NotImplementedError(f"{type(self).__name__} keeps fp32 activations: the encoder, projector and RVQ must stay fp32-grade "
                                      "for bit-identical indices (bf16 activations are built for the decoder-only generators: "
                                      "HiFiGANStreamGenerator, SymADDecoderStreamGenerator)")
        if dtype not in (torch.float32, torch.bfloat16):
            raise NotImplementedError(f"{type(self).__name__} has no {dtype} activation mode (float32 or bfloat16)")
        if self._h is not None:
            raise RuntimeError("set the activation dtype before .to(device): the state and workspaces are laid out when the handle is created")
        self._act_bf16 = dtype == torch.bfloat16
        self._cfg.compute_dtype = 2 if self._act_bf16 else self._operand_mode
        return self

    def bfloat16(self):
        return self._set_dtype(torch.bfloat16)

    def float(self):
        return self._set_dtype(torch.float32)

    def __del__(self):
        try:
            if self._h is not None:
                self._lib.adec_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # -- helpers ------------------------------------------------------------------------------------
    def _ready(self):
        if self._h is None:
            raise RuntimeError("call .to('cuda:N') before using the codec")

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self._device).cuda_stream)

    def _in(self, t, dtype=torch.float32):
        if t.device != self._device:
            raise RuntimeError(f"input is on {t.device}, codec is on {self._device}")
        return t.to(dtype).contiguous()

    @staticmethod
    def _want(t, what, dim, size):
        """torch raises RuntimeError on a wrong feature dimension; the C ABI takes no D argument, so check here."""
        if t.dim() != 3 or t.size(dim) != size:
            raise RuntimeError(f"audiodec_b200: {what}: expected a 3-D tensor with size {size} in dim {dim}, got {tuple(t.shape)}")

    def _batch(self, b):
        n = self._lib.adec_n_streams(self._h)
        if n != b:
            _check(self._lib.adec_set_streams(self._h, b), self._h)

    @property
    def n_streams(self):
        self._ready()
        return self._lib.adec_n_streams(self._h)

    @property
    def launch_count(self):
        return int(self._lib.adec_launch_count(self._h)) if self._h is not None else 0

    def profile(self, enable=True):
        """start/stop per-launch CUDA-event timing (adec_profile)."""
        self._ready()
        _check(self._lib.adec_profile(self._h, int(enable)), self._h)

    def profile_report(self):
        """[(op name, ms, algorithmic bytes)] for every launch recorded since profile(True)."""
        self._ready()
        buf = ctypes.create_string_buffer(1 << 20)
        _check(self._lib.adec_profile_report(self._h, buf, len(buf)), self._h)
        rows = []
        for line in buf.value.decode().splitlines():
            name, ms, nbytes = line.split("\t")
            rows.append((name, float(ms), float(nbytes)))
        return rows

    def range_error(self):
        """True if an activation left the fp16-split range of the default conv engine since the last call (synchronises)."""
        self._ready()
        rc = self._lib.adec_range_error(self._h, self._stream())
        if rc < 0:
            raise RuntimeError("audiodec_b200: " + _lib.last_error(self._h))
        return bool(rc)

    def reset_buffer(self):
        """AudioDec.py:250-256 / HiFiGAN.py:298-305."""
        self._ready()
        _check(self._lib.adec_reset(self._h, self._stream()), self._h)

    # ---- stream slots: every stream of the handle (n_streams, see set_streams) is a slot with its own causal state
    def set_streams(self, n):
        """Resize the handle to n stream slots.  Existing streams keep their state; growing from one stream replicates its state."""
        self._ready()
        self._batch(int(n))

    def copy_stream_state(self, src, dst):
        """Copy stream `src`'s current causal state into stream(s) `dst` (an int or a list): a joining stream starts warm."""
        self._ready()
        dst = [dst] if isinstance(dst, int) else list(dst)
        arr, n = _int_array(dst)
        _check(self._lib.adec_copy_stream_state(self._h, int(src), arr, n, self._stream()), self._h)

    # ---- stream state out of and into the handle (adec_get_stream_state / adec_set_stream_state)
    @property
    def state_layout(self):
        """[(key, C, P)]: the reference pad_buffers the handle runs, in the order a stream's state vector holds them, each (C, P)
        channels-first."""
        self._ready()
        if self._layout is None:
            key, c, p = ctypes.c_char_p(), ctypes.c_int(), ctypes.c_int()
            out = []
            for i in range(self._lib.adec_state_entries(self._h)):
                _check(self._lib.adec_state_entry(self._h, i, ctypes.byref(key), ctypes.byref(c), ctypes.byref(p)), self._h)
                out.append((key.value.decode(), c.value, p.value))
            self._layout = out
        return self._layout

    @property
    def state_dtype(self):
        """dtype of the exported state: bf16 with bf16 activations, fp32 otherwise."""
        return torch.bfloat16 if self._act_bf16 else torch.float32

    def stream_state(self, streams):
        """The current causal state of `streams` (an int or a list of distinct ids) -> (n, S) device tensor, row i stream streams[i]'s
        state_layout entries one after the other.  Asynchronous on the current stream; the streams' state is left as it is."""
        self._ready()
        ids = _stream_ids(streams)
        arr, n = _int_array(ids)
        out = torch.empty(n, int(self._lib.adec_stream_state_elems(self._h)), device=self._device, dtype=self.state_dtype)
        _check(self._lib.adec_get_stream_state(self._h, arr, n, _ptr(out), self._stream()), self._h)
        return out

    def load_stream_state(self, streams, state, layout=None):
        """Import `state` (n, S), as stream_state returns it, into `streams`: stream streams[i] continues exactly as the exported stream
        would have.  `layout` (optional): the exporting handle's state_layout, checked against this handle's.  Streams not listed keep
        their state."""
        self._ready()
        ids = _stream_ids(streams)
        if layout is not None and [tuple(e) for e in layout] != [tuple(e) for e in self.state_layout]:
            raise ValueError(f"audiodec_b200: load_stream_state: the state was exported by a handle with another state layout "
                             f"({len(layout)} entries; this handle has {len(self.state_layout)})")
        state = _check_state(state, len(ids), int(self._lib.adec_stream_state_elems(self._h)), self.state_dtype, self._device)
        arr, n = _int_array(ids)
        _check(self._lib.adec_set_stream_state(self._h, arr, n, _ptr(state), self._stream()), self._h)

    # ---- decode plumbing shared by both generators
    def _fn(self, name):
        """The C entry point `name`, or its bf16 twin (`name`_bf16) when the handle has bf16 activations."""
        return getattr(self._lib, name + "_bf16" if self._act_bf16 else name)

    def _zq_dim(self):
        return getattr(self, "code_dim", None) or self.in_channels

    def _zq_in(self, zq):
        """zq on the codec's device, contiguous, in the decoder's activation dtype (bf16 with bf16 activations), 16-byte aligned."""
        zq = self._in(zq, torch.bfloat16 if self._act_bf16 else torch.float32)
        if self._act_bf16 and zq.data_ptr() % 16:
            zq = zq.clone()                  # the bf16 kernels read zq as 16-byte vectors: realign an offset view
        return zq

    def _decode(self, zq):
        """the streaming decode of zq (B,F,D) channels-last, checked by the caller -> y (B,1,F*hop)"""
        zq = self._zq_in(zq)
        b, f, _ = zq.shape
        self._batch(b)
        y = torch.empty(b, 1, f * self._lib.adec_hop_length(self._h), device=self._device, dtype=zq.dtype)
        _check(self._fn("adec_decode")(self._h, _ptr(zq), b, f, _ptr(y), self._stream()), self._h)
        return y

    def _decode_offline(self, zq):
        self._ready()
        self._want(zq, "decode_offline / forward", 1, self._zq_dim())
        zq_cl = self._zq_in(zq.transpose(1, 2))                     # the kernels' native channels-last (B,F,D)
        b, f, _ = zq_cl.shape
        y = torch.empty(b, 1, f * self._lib.adec_hop_length(self._h), device=self._device, dtype=zq_cl.dtype)
        _check(self._fn("adec_decode_offline")(self._h, _ptr(zq_cl), b, f, _ptr(y), self._stream()), self._h)
        return y

    def _decode_varlen(self, name, zq_cl, frames, *slots):
        """Decode zq_cl (sum F_b, D) channels-last as one varlen row space through entry point `name` (its stream array: `slots`) ->
        list of B waveforms (1, 1, F_b * hop), views of one output buffer."""
        zq_cl = self._zq_in(zq_cl)
        hop = self._lib.adec_hop_length(self._h)
        y = torch.empty(sum(frames) * hop, device=self._device, dtype=zq_cl.dtype)
        arr, b = _int_array(frames)
        _check(self._fn(name)(self._h, _ptr(zq_cl), arr, *slots, b, _ptr(y), self._stream()), self._h)
        out, o = [], 0
        for f in frames:
            out.append(y[o * hop:(o + f) * hop].view(1, 1, f * hop))
            o += f
        return out

    def _decode_offline_varlen(self, zq, frames):
        self._ready()
        self._want(zq, "decode_offline_varlen / forward_varlen", 1, self._zq_dim())
        frames = [int(f) for f in frames]
        if zq.size(0) != 1 or zq.size(2) != sum(frames):
            raise RuntimeError(f"audiodec_b200: decode_offline_varlen / forward_varlen: expected (1, D, {sum(frames)}) for frames summing to "
                               f"{sum(frames)}, got {tuple(zq.shape)}")
        return self._decode_varlen("adec_decode_offline_varlen", zq[0].transpose(0, 1), frames)

    def _decode_streams(self, zq, frames, streams):
        self._ready()
        d = self._zq_dim()
        frames = [int(f) for f in frames]
        if zq.dim() == 3 and zq.size(0) == 1:
            zq = zq[0]
        if zq.dim() != 2 or zq.size(0) != sum(frames) or zq.size(1) != d:
            raise RuntimeError(f"audiodec_b200: decode_streams: expected (1, {sum(frames)}, {d}) channels-last for frames summing to "
                               f"{sum(frames)}, got {tuple(zq.shape)}")
        if len(frames) != len(streams):
            raise RuntimeError(f"audiodec_b200: decode_streams: {len(frames)} frame counts for {len(streams)} streams")
        sarr, _ = _int_array(streams)
        return self._decode_varlen("adec_decode_streams", zq, frames, sarr)


def _symad_init(g, model_type, input_channels=1, output_channels=1, encode_channels=32, decode_channels=32, code_dim=64,
                codebook_num=8, codebook_size=1024, bias=True, enc_ratios=(2, 4, 8, 16), dec_ratios=(16, 8, 4, 2),
                enc_strides=(3, 4, 5, 5), dec_strides=(5, 5, 4, 3), mode="causal", codec="audiodec",
                projector="conv1d", quantier="residual_vq", nonlinear_activation="ELU",
                nonlinear_activation_params={}, use_weight_norm=False):
    """The config of a symAD generator (AudioDec.py:31-51 keywords) into g's adec_config, as a handle of `model_type`."""
    assert mode == "causal", f"Mode {mode} does not support streaming!"       # models/utils.py:13-15
    if codec not in ("audiodec", "activate_audiodec"):
        raise NotImplementedError(f"Codec ({codec}) is not supported!")          # AudioDec.py:53-60
    if projector != "conv1d" or quantier != "residual_vq":
        raise NotImplementedError("only projector='conv1d', quantier='residual_vq' are built")
    if nonlinear_activation != "ELU" or nonlinear_activation_params:
        raise NotImplementedError("only ELU(alpha=1) residual units are built")
    c = g._cfg
    c.model_type = model_type
    c.input_channels, c.output_channels = input_channels, output_channels
    c.encode_channels, c.decode_channels = encode_channels, decode_channels
    c.code_dim, c.codebook_num, c.codebook_size = code_dim, codebook_num, codebook_size
    c.bias = int(bias)
    c.n_enc, c.n_dec = len(enc_strides), len(dec_strides)
    _fill(c.enc_ratios, enc_ratios), _fill(c.enc_strides, enc_strides)
    _fill(c.dec_ratios, dec_ratios), _fill(c.dec_strides, dec_strides)
    c.use_weight_norm = int(use_weight_norm)
    c.codec_activate = int(codec == "activate_audiodec")
    g.input_channels = input_channels
    g.code_dim, g.codebook_num = code_dim, codebook_num
    g.enc_strides = tuple(enc_strides)


def _symad_signature(init):
    """Give a symAD generator's __init__(self, *args, **params) the explicit keywords of AudioDec.py's StreamGenerator (those of
    _symad_init), for inspect.signature and help()."""
    sig = inspect.signature(_symad_init)
    self_p = inspect.Parameter("self", inspect.Parameter.POSITIONAL_OR_KEYWORD)
    init.__signature__ = sig.replace(parameters=[self_p] + list(sig.parameters.values())[2:])
    return init


class _SymADTransmitter(_StreamGeneratorBase):
    """The transmitter side of a symAD generator, shared by the full generator and the encoder-only one: encode (streaming, offline,
    varlen, stream slots), quantize to indices / packed bytes, and pack.  With bf16 activations (the encoder-only generator's
    set_activation_dtype(torch.bfloat16)) x and z are bf16 on the device: fp32 inputs are cast there, and z comes back bf16."""

    @property
    def _act_dtype(self):
        return torch.bfloat16 if self._act_bf16 else torch.float32

    def _tx_in(self, t):
        """x or z on the codec's device, contiguous, in the activation dtype, 16-byte aligned (the bf16 kernels read whole vectors)"""
        t = self._in(t, self._act_dtype)
        return t.clone() if self._act_bf16 and t.data_ptr() % 16 else t

    def encode(self, x):
        """(B,1,T) float -> z (B,code_dim,F)   (AudioDec.py:228-234)"""
        self._ready()
        if x.dim() != 3:
            raise RuntimeError("encode expects (batch, channel, length)")
        if x.size(1) != self.input_channels:
            x = x.reshape(-1, self.input_channels, x.size(-1))
        x = self._tx_in(x)
        b, _, t = x.shape
        self._batch(b)
        f = self._lib.adec_frames_for(self._h, t)
        z = torch.empty(b, self.code_dim, f, device=self._device, dtype=self._act_dtype)
        _check(self._fn("adec_encode")(self._h, _ptr(x), b, t, _ptr(z), self._stream()), self._h)
        return z

    def quantize(self, z):
        """z (B,code_dim,F) -> idx int64 (Nq,F) for B==1 else (Nq,B,F)   (AudioDec.py:237-239)"""
        self._ready()
        self._want(z, "quantize", 1, self.code_dim)
        z = self._tx_in(z)
        b, _, f = z.shape
        idx = torch.empty(self.codebook_num, b, f, device=self._device, dtype=torch.int64)
        _check(self._fn("adec_quantize")(self._h, _ptr(z), b, f, _ptr(idx), self._stream()), self._h)
        return idx.squeeze(1) if b == 1 else idx

    def quantize_fused(self, z, want_idx=True, want_packed=False, want_zq=True):
        """quantize -> [pack] -> lookup in ONE launch (adec_quantize_ex): returns (idx or None, packed or None, zq or None) with the
        shapes of quantize() / pack() / lookup().  Bit-identical to the three separate calls."""
        self._ready()
        self._want(z, "quantize_fused", 1, self.code_dim)
        if want_zq and not hasattr(self, "lookup"):
            raise RuntimeError(f"audiodec_b200: quantize_fused: {type(self).__name__} has no lookup; pass want_zq=False")
        z = self._tx_in(z)
        b, _, f = z.shape
        idx = torch.empty(self.codebook_num, b, f, device=self._device, dtype=torch.int64) if want_idx else None
        packed = torch.empty(b, f, self.packed_frame_bytes(), device=self._device, dtype=torch.uint8) if want_packed else None
        zq = torch.empty(b, f, self.code_dim, device=self._device, dtype=torch.float32) if want_zq else None
        _check(self._fn("adec_quantize_ex")(self._h, _ptr(z), b, f, _ptr(idx) if want_idx else None, _ptr(packed) if want_packed else None,
                                          _ptr(zq) if want_zq else None, self._stream()), self._h)
        if b == 1:
            idx = idx.squeeze(1) if idx is not None else None
            packed = packed.squeeze(0) if packed is not None else None
        return idx, packed, zq

    # ---- non-streaming batch forward (SURVEY.md 8(f) rank 4; codecTest.py:78-95).  These calls discard the streaming state.
    def encode_offline(self, x):
        """x (B,1,T) -> z (B,code_dim,F): Encoder.forward + Projector.forward, zero left-pad (conv_layer.py:148-151)."""
        self._ready()
        if x.dim() != 3:
            raise RuntimeError("encode_offline expects (batch, channel, length)")
        if x.size(1) != self.input_channels:                 # same fold as encode(): every audio channel is its own batch row
            x = x.reshape(-1, self.input_channels, x.size(-1))
        x = self._tx_in(x)
        b, _, t = x.shape
        f = self._lib.adec_frames_for(self._h, t)
        z = torch.empty(b, self.code_dim, f, device=self._device, dtype=self._act_dtype)
        _check(self._fn("adec_encode_offline")(self._h, _ptr(x), b, t, _ptr(z), self._stream()), self._h)
        return z

    def encode_offline_varlen(self, xs):
        """Utterances of different lengths in one launch sequence: xs is a list of 1-D (T_b,) or (1, T_b) tensors.  Returns
        (z (1, code_dim, sum F_b), [F_b]); utterance b's frames are columns [sum_{i<b} F_i, +F_b) and equal encode_offline of that
        utterance alone.  z is quantize's B = 1 layout (and quantize_offline's), so one call quantizes the whole batch."""
        self._ready()
        if len(xs) == 0:
            raise RuntimeError("audiodec_b200: encode_offline_varlen: no utterances")
        return self._encode_varlen(self._fn("adec_encode_offline_varlen"), "encode_offline_varlen", "utterances", xs)

    def encode_streams(self, chunks, streams):
        """Advance streams[b] by chunks[b] (1-D (T_b,) or (1, T_b); lengths may differ) in one launch sequence.  Returns
        (z (1, code_dim, sum F_b), [F_b]) laid out like encode_offline_varlen; stream b's frames equal a B = 1 streaming encode of its
        chunk.  Streams not listed keep their state untouched."""
        self._ready()
        if len(chunks) != len(streams):
            raise RuntimeError(f"audiodec_b200: encode_streams: {len(chunks)} chunks for {len(streams)} streams")
        sarr, _ = _int_array(streams)
        return self._encode_varlen(self._fn("adec_encode_streams"), "encode_streams", "chunks", chunks, sarr)

    def _encode_varlen(self, fn, what, noun, xs, *slots):
        """Encode 1-D (T_b,) or (1, T_b) tensors concatenated into one varlen row space through `fn` (its stream array: `slots`) ->
        (z (1, code_dim, sum F_b), [F_b])."""
        flat = []
        for x in xs:
            x = x[0] if x.dim() == 2 and x.size(0) == 1 else x
            if x.dim() != 1:
                raise RuntimeError(f"audiodec_b200: {what}: expected 1-D (T,) or (1, T) {noun}, got {tuple(x.shape)}")
            flat.append(self._in(x, self._act_dtype))
        lengths = [x.numel() for x in flat]
        frames, offsets = varlen_layout(lengths, self.enc_strides)
        x = torch.cat(flat) if flat else torch.empty(0, device=self._device, dtype=self._act_dtype)
        z = torch.empty(1, self.code_dim, offsets[-1], device=self._device, dtype=self._act_dtype)
        arr, b = _int_array(lengths)
        _check(fn(self._h, _ptr(x), arr, *slots, b, _ptr(z), self._stream()), self._h)
        return z, frames

    # ---- index bitstream (SURVEY.md 8(f) rank 2; the reference queues the raw int64 tensor, bin/stream.py:224)
    def packed_frame_bytes(self):
        self._ready()
        return self._lib.adec_packed_frame_bytes(self._h)

    def pack(self, idx):
        """idx (Nq,F) -> uint8 (F,bytes); (Nq,B,F) -> (B,F,bytes): Nq x ceil(log2 N)-bit local indices per frame."""
        self._ready()
        idx = self._in(idx, torch.int64)
        two_d = idx.dim() == 2
        if two_d:
            idx = idx.unsqueeze(1)
        nq, b, f = idx.shape
        if nq != self.codebook_num:
            raise RuntimeError(f"audiodec_b200: pack: expected {self.codebook_num} index rows, got {nq}")
        out = torch.empty(b, f, self.packed_frame_bytes(), device=self._device, dtype=torch.uint8)
        _check(self._lib.adec_pack_indices(self._h, _ptr(idx), b, f, _ptr(out), self._stream()), self._h)
        return out.squeeze(0) if two_d else out

    def index_error(self):
        """True if lookup / pack / unpack met an out-of-range index since the last call (synchronises the stream)."""
        self._ready()
        rc = self._lib.adec_index_error(self._h, self._stream())
        if rc < 0:
            raise RuntimeError("audiodec_b200: " + _lib.last_error(self._h))
        return bool(rc)


class SymADStreamGenerator(_SymADTransmitter):
    """models/autoencoder/AudioDec.py:166-256."""

    @_symad_signature
    def __init__(self, *args, **params):
        super().__init__()
        _symad_init(self, _lib.MODEL_SYMAD, *args, **params)

    # -- streaming API ---------------------------------------------------------------------------------
    def initial_encoder(self, receptive_length, device):
        """AudioDec.py:216-221: push `receptive_length` zeros through encode/quantize/lookup."""
        self._ready()
        z = self.encode(torch.zeros(1, self.input_channels, receptive_length, device=self._device))
        return self.lookup(self.quantize(z))

    def initial_decoder(self, zq):
        self.decode(zq)                                                              # AudioDec.py:224-225

    def lookup_packed(self, packed, dtype=torch.float32):
        """uint8 (F,bytes) -> zq (1,F,D); (B,F,bytes) -> (B,F,D): lookup straight from the bitstream (unpack fused into lookup).
        dtype=torch.bfloat16: bf16 zq, the fp32 sum rounded once, equal to lookup_packed(packed).to(torch.bfloat16)."""
        self._ready()
        packed = self._in(packed, torch.uint8)
        if packed.dim() == 2:
            packed = packed.unsqueeze(0)
        b, f, nb = packed.shape
        if nb != self.packed_frame_bytes():
            raise RuntimeError(f"audiodec_b200: lookup_packed: expected {self.packed_frame_bytes()} bytes per frame, got {nb}")
        fn = self._lookup_fn("adec_lookup_packed", dtype)
        zq = torch.empty(b, f, self.code_dim, device=self._device, dtype=dtype)
        _check(fn(self._h, _ptr(packed), b, f, _ptr(zq), self._stream()), self._h)
        return zq

    def lookup_packed_conceal(self, packed, rows, anchors, dtype=torch.float32):
        """The packed lookup with loss concealment, in ONE launch (adec_lookup_packed_conceal): uint8 packed frames (F, bytes) or
        (1, F, bytes), and one descriptor per output row -> zq (1, R, D).  rows: R rows of (src, next, slot, j, den) ints (an (R, 5)
        array or a sequence of 5-tuples), checked before anything runs.  A real row (src >= 0) is lookup_packed's row of frame src and,
        with slot >= 0, stores its fp32 sum in anchors[slot].  A concealed row (src = -1) is fl(fl(fl(j / den) * fl(s_b - a)) + a) with
        s_b the sum of frame next and a = anchors[slot], or s_b with slot = -1.  anchors: a contiguous float32 (n_anchors, code_dim)
        device tensor, updated in place.  dtype=torch.bfloat16: bf16 zq, the fp32 result rounded once."""
        self._ready()
        packed = self._in(packed, torch.uint8)
        if packed.dim() == 3 and packed.size(0) == 1:
            packed = packed[0]
        if packed.dim() != 2 or packed.size(1) != self.packed_frame_bytes():
            raise RuntimeError(f"audiodec_b200: lookup_packed_conceal: expected (F, {self.packed_frame_bytes()}) packed frames, got "
                               f"{tuple(packed.shape)}")
        if not isinstance(anchors, torch.Tensor) or anchors.device != self._device or anchors.dtype != torch.float32 or \
                anchors.dim() != 2 or anchors.size(1) != self.code_dim or not anchors.is_contiguous():
            raise RuntimeError(f"audiodec_b200: lookup_packed_conceal: anchors must be a contiguous float32 (n, {self.code_dim}) tensor "
                               f"on {self._device}")
        desc = np.ascontiguousarray(rows, dtype=np.int32)
        if desc.ndim != 2 or desc.shape[1] != 5:
            raise ValueError(f"audiodec_b200: lookup_packed_conceal: rows must be (R, 5) (src, next, slot, j, den), got {desc.shape}")
        r = desc.shape[0]
        fn = self._lookup_fn("adec_lookup_packed_conceal", dtype)
        zq = torch.empty(1, r, self.code_dim, device=self._device, dtype=dtype)
        _check(fn(self._h, _ptr(packed), packed.size(0), desc.ctypes.data_as(ctypes.POINTER(_lib.AdecConcealRow)), r, _ptr(anchors),
                  anchors.size(0), _ptr(zq), self._stream()), self._h)
        return zq

    def lookup_packed_playout(self, packed, rows, anchors, targets, dtype=torch.float32):
        """The packed lookup of a receiver's playout clock, in ONE launch (adec_lookup_packed_playout): uint8 packed frames (F, bytes)
        or (1, F, bytes), F = 0 allowed, and one descriptor per output row -> zq (1, R, D).  rows: R rows of (src, next, target, slot,
        j, den) ints: an (R, 6) int32 array (it may be a page-locked buffer, which must then stay unchanged until the stream has run the
        call), or a sequence of 6-tuples; checked before anything runs.  A real row (src >= 0) and an interpolated row (src = -1,
        next >= 0) are lookup_packed_conceal's rows.  A fade row (src = next = -1) is t = targets[target] when j >= den or slot = -1,
        and otherwise fl(fl(fl(j / den) * fl(t - a)) + a) with a = anchors[slot].  anchors: a contiguous float32 (n_anchors, code_dim)
        device tensor, updated in place; targets: a contiguous float32 (n_targets, code_dim) device tensor.  dtype=torch.bfloat16: bf16
        zq, the fp32 result rounded once."""
        return self._lookup_playout("lookup_packed_playout", packed, rows, anchors, targets, dtype)

    def lookup_packed_timescale(self, packed, rows, anchors, targets, dtype=torch.float32):
        """The packed lookup of an adaptive playout clock, in ONE launch (adec_lookup_packed_timescale): lookup_packed_playout's
        arguments and rows, bit for bit, plus two row kinds that start from packed frame src of the same call (slot = -1) rather than
        an anchor, with s_x the fp32 sum of packed frame x.  A between row (src >= 0, next >= 0, target = -1, 1 <= j < den) is
        fl(fl(fl(j / den) * fl(s_next - s_src)) + s_src).  A frame-started fade (src >= 0, next = -1, target >= 0) is the fade row with
        a = s_src.  Both equal the anchor-read row of a later call, since a real row of frame src stores s_src as its anchor."""
        return self._lookup_playout("lookup_packed_timescale", packed, rows, anchors, targets, dtype)

    def _lookup_playout(self, what, packed, rows, anchors, targets, dtype):
        self._ready()
        packed = self._in(packed, torch.uint8)
        if packed.dim() == 3 and packed.size(0) == 1:
            packed = packed[0]
        if packed.dim() != 2 or packed.size(1) != self.packed_frame_bytes():
            raise RuntimeError(f"audiodec_b200: {what}: expected (F, {self.packed_frame_bytes()}) packed frames, got {tuple(packed.shape)}")
        for name, t in (("anchors", anchors), ("targets", targets)):
            if not isinstance(t, torch.Tensor) or t.device != self._device or t.dtype != torch.float32 or t.dim() != 2 or \
                    t.size(1) != self.code_dim or not t.is_contiguous():
                raise RuntimeError(f"audiodec_b200: {what}: {name} must be a contiguous float32 (n, {self.code_dim}) tensor on "
                                   f"{self._device}")
        if isinstance(rows, torch.Tensor):
            rows = rows.numpy()
        desc = np.ascontiguousarray(rows, dtype=np.int32)
        if desc.ndim != 2 or desc.shape[1] != 6:
            raise ValueError(f"audiodec_b200: {what}: rows must be (R, 6) (src, next, target, slot, j, den), got {desc.shape}")
        r = desc.shape[0]
        fn = self._lookup_fn("adec_" + what, dtype)
        zq = torch.empty(1, r, self.code_dim, device=self._device, dtype=dtype)
        _check(fn(self._h, _ptr(packed) if packed.size(0) else None, packed.size(0), ctypes.c_void_p(desc.ctypes.data), r, _ptr(anchors),
                  anchors.size(0), _ptr(targets), targets.size(0), _ptr(zq), self._stream()), self._h)
        return zq

    def silence_frame(self, receptive_length=8192):
        """The codec's silence frame, a (code_dim,) float32 device tensor: the lookup sum of the RVQ code of the last frame of
        encode_offline on `receptive_length` zeros (rounded up to a hop multiple), i.e. quantize_offline(encode_offline(zeros))[0][0, :, -1].
        A playout receiver fades toward it when a session's packets stop.  The encoder runs on a scratch encoder-only handle with this
        generator's config and weights (bit for bit this handle's encode in fp32), so no stream of this generator is touched."""
        self._ready()
        enc = SymADEncoderStreamGenerator.__new__(SymADEncoderStreamGenerator)
        _StreamGeneratorBase.__init__(enc)
        ctypes.memmove(ctypes.addressof(enc._cfg), ctypes.addressof(self._cfg), ctypes.sizeof(self._cfg))
        enc._cfg.model_type = _lib.MODEL_SYMAD_ENCODER
        enc.input_channels, enc.code_dim, enc.codebook_num, enc.enc_strides = \
            self.input_channels, self.code_dim, self.codebook_num, self.enc_strides
        enc._sd = self._sd
        enc.to(self._device)
        hop = self._lib.adec_hop_length(self._h)
        t = -(-receptive_length // hop) * hop
        idx = enc.quantize_offline(enc.encode_offline(torch.zeros(1, self.input_channels, t, device=self._device)))   # (Nq, 1, F)
        return self.lookup(idx[:, 0, -1:].contiguous())[0, 0]

    def _lookup_fn(self, name, dtype):
        if dtype not in (torch.float32, torch.bfloat16):
            raise NotImplementedError(f"audiodec_b200: {name[5:]}: zq is float32 or bfloat16, not {dtype}")
        return getattr(self._lib, name + "_bf16" if dtype == torch.bfloat16 else name)

    def lookup(self, idx, dtype=torch.float32):
        """idx (Nq,F) -> zq (1,F,D); (Nq,B,F) -> (B,F,D)   (AudioDec.py:242-243).  dtype=torch.bfloat16: bf16 zq, the fp32 sum
        rounded once, equal to lookup(idx).to(torch.bfloat16) (what a decoder with bf16 activations takes)."""
        self._ready()
        idx = self._in(idx, torch.int64)
        if idx.dim() == 2:
            idx = idx.unsqueeze(1)
        if idx.dim() != 3 or idx.size(0) != self.codebook_num:
            raise RuntimeError(f"audiodec_b200: lookup: expected ({self.codebook_num},F) or ({self.codebook_num},B,F) indices, got {tuple(idx.shape)}")
        _, b, f = idx.shape
        fn = self._lookup_fn("adec_lookup", dtype)
        zq = torch.empty(b, f, self.code_dim, device=self._device, dtype=dtype)
        _check(fn(self._h, _ptr(idx), b, f, _ptr(zq), self._stream()), self._h)
        return zq

    def decode_streams(self, zq, frames, streams):
        """Advance streams[b] by frames[b] frames of zq ((1, sum F_b, code_dim) or (sum F_b, code_dim) channels-last, as lookup
        returns it) in one launch sequence -> list of B waveforms (1, 1, F_b * hop), views of one output buffer, each equal to a
        B = 1 streaming decode of those frames.  Streams not listed keep their state untouched."""
        return self._decode_streams(zq, frames, streams)

    def quantize_offline(self, z):
        """z (B,code_dim,F) -> (zq (B,code_dim,F) channels-first like Quantizer.forward (quantizer.py:31-34), idx (Nq,B,F))."""
        self._ready()
        self._want(z, "quantize_offline", 1, self.code_dim)
        z = self._in(z)
        b, _, f = z.shape
        idx = torch.empty(self.codebook_num, b, f, device=self._device, dtype=torch.int64)
        _check(self._lib.adec_quantize(self._h, _ptr(z), b, f, _ptr(idx), self._stream()), self._h)
        zq = torch.empty(b, f, self.code_dim, device=self._device, dtype=torch.float32)
        _check(self._lib.adec_lookup(self._h, _ptr(idx), b, f, _ptr(zq), self._stream()), self._h)
        return zq.transpose(1, 2), idx

    def quantize_forward(self, z):
        """z (B,code_dim,F) -> (zq (B,code_dim,F) channels-first, idx (Nq,B,F)): Quantizer.forward's zq (quantizer.py:31-34), the
        sum over stages of r + (e - r) from 0. (vq_module.py:136-143), in one launch.  The indices equal quantize(); zq can differ from
        quantize_offline's codeword sum in the last bits.  The channels-last storage behind zq is what zq_moments reads."""
        self._ready()
        self._want(z, "quantize_forward", 1, self.code_dim)
        z = self._in(z)
        b, _, f = z.shape
        idx = torch.empty(self.codebook_num, b, f, device=self._device, dtype=torch.int64)
        zq = torch.empty(b, f, self.code_dim, device=self._device, dtype=torch.float32)
        _check(self._lib.adec_quantize_forward(self._h, _ptr(z), b, f, _ptr(idx), _ptr(zq), self._stream()), self._h)
        return zq.transpose(1, 2), idx

    def zq_moments(self, zq, frames):
        """Per-utterance moments of a varlen zq: zq (1, code_dim, sum F_b) as quantize_forward returns it for encode_offline_varlen's
        z (channels-last storage), or (sum F_b, code_dim) channels-last; utterance b holds frames[b] rows.  Returns fp64 device
        tensors (sum (B, code_dim), m2 (B, code_dim)): sum_f x and the corrected centred sum_f (x - T)^2 - (sum_f (x - T))^2 / F_b,
        T = sum / F_b, what StandardScaler.partial_fit computes for one utterance.  Deterministic, and independent of the batch
        around an utterance."""
        self._ready()
        if zq.dim() == 3 and zq.size(0) == 1 and zq.size(1) == self.code_dim:
            zq = zq[0].transpose(0, 1)                     # (sum F, D): a view of quantize_forward's channels-last storage
        if zq.dim() != 2 or zq.size(1) != self.code_dim:
            raise RuntimeError(f"audiodec_b200: zq_moments: expected (1, {self.code_dim}, F) or (F, {self.code_dim}), got {tuple(zq.shape)}")
        zq = self._in(zq)
        arr, b = _int_array(frames)
        if sum(int(f) for f in frames) != zq.size(0):
            raise RuntimeError(f"audiodec_b200: zq_moments: frames add up to {sum(int(f) for f in frames)}, zq has {zq.size(0)} rows")
        out = torch.empty(2, b, self.code_dim, device=self._device, dtype=torch.float64)
        _check(self._lib.adec_zq_moments(self._h, _ptr(zq), arr, b, _ptr(out[0]), _ptr(out[1]), self._stream()), self._h)
        return out[0], out[1]

    def decode_offline(self, zq):
        """zq (B,code_dim,F) channels-first (what Decoder.forward takes, decoder.py:135-140) -> y (B,1,F*hop); transposed convs
        replicate their first input frame (conv_layer.py:189-192)."""
        return self._decode_offline(zq)

    def decode_offline_varlen(self, zq, frames):
        """zq (1, code_dim, sum F_b) channels-first holding utterances of `frames` frames each (what encode_offline_varlen +
        quantize_offline give) -> list of B waveforms (1, 1, F_b * hop), views of one output buffer, each equal to decode_offline of
        that utterance alone."""
        return self._decode_offline_varlen(zq, frames)

    def unpack(self, packed):
        """uint8 (F,bytes) -> idx (Nq,F); (B,F,bytes) -> (Nq,B,F) int64 flat indices, ready for lookup()."""
        self._ready()
        packed = self._in(packed, torch.uint8)
        two_d = packed.dim() == 2
        if two_d:
            packed = packed.unsqueeze(0)
        b, f, nb = packed.shape
        if nb != self.packed_frame_bytes():
            raise RuntimeError(f"audiodec_b200: unpack: expected {self.packed_frame_bytes()} bytes per frame, got {nb}")
        idx = torch.empty(self.codebook_num, b, f, device=self._device, dtype=torch.int64)
        _check(self._lib.adec_unpack_indices(self._h, _ptr(packed), b, f, _ptr(idx), self._stream()), self._h)
        return idx.squeeze(1) if two_d else idx

    def decode(self, zq):
        """zq (B,F,D) channels-last -> y (B,1,F*hop)   (AudioDec.py:246-247)"""
        self._ready()
        self._want(zq, "decode", 2, self.code_dim)
        return self._decode(zq)



class SymADEncoderStreamGenerator(_SymADTransmitter):
    """The transmitter of a symAD StreamGenerator alone (models/autoencoder/AudioDec.py:216-239): what the reference's transmitter
    runs as its `tx_encoder` object (initial_encoder / encode / quantize, utils/audiodec.py:100-102).  Same constructor keywords as
    SymADStreamGenerator, and it loads the same state dict (the decoder keys are ignored).  In fp32 it encodes and quantizes what
    SymADStreamGenerator gives, bit for bit, in every call mode.  `.to(torch.bfloat16)` runs the encoder's and the projector's convs on
    bf16 operands (fp32 accumulation; the stem keeps fp32 weights), with fp32 x, activations, state and z, and the RVQ unchanged on
    that z; `set_activation_dtype(torch.bfloat16)` also keeps x, every activation, the causal state and z in bf16, as the reference's
    `tx_encoder.to(torch.bfloat16)` stores them (encode takes fp32 or bf16 x and returns bf16 z; the RVQ widens it exactly).  Both
    change some code indices.  It has no decode or lookup: a receiver needs a full generator's codebooks."""
    _bf16_modes = True

    @_symad_signature
    def __init__(self, *args, **params):
        super().__init__()
        _symad_init(self, _lib.MODEL_SYMAD_ENCODER, *args, **params)

    def initial_encoder(self, receptive_length, device):
        """AudioDec.py:216-221 without the lookup: push `receptive_length` zeros through encode and quantize (the transmitter's warm-up,
        bin/stream.py:49, which discards the result)."""
        self._ready()
        self.quantize(self.encode(torch.zeros(1, self.input_channels, receptive_length, device=self._device)))

    def quantize_offline(self, z):
        """z (B,code_dim,F) -> idx (Nq,B,F): the indices of Quantizer.forward (quantizer.py:31-34) without its zq, which needs the
        codebooks' lookup (a full generator's quantize_offline)."""
        self._ready()
        self._want(z, "quantize_offline", 1, self.code_dim)
        idx = self.quantize(z)
        return idx.unsqueeze(1) if idx.dim() == 2 else idx


class SymADDecoderStreamGenerator(_StreamGeneratorBase):
    """The decoder of a symAD StreamGenerator alone (models/autoencoder/AudioDec.py:224-256): what the reference's receiver runs as
    its `decoder` object (initial_decoder / decode, utils/audiodec.py:104-106; rx_encoder does the lookup).  Same constructor
    keywords as SymADStreamGenerator, and it loads the same state dict (the encoder, projector and quantizer keys are ignored).
    Decoding in fp32 gives what SymADStreamGenerator.decode gives, bit for bit.  Unlike the full generator it has the vocoder's
    bf16 modes: `.to(torch.bfloat16)` for bf16 conv operands with fp32 activations and I/O, `set_activation_dtype(torch.bfloat16)`
    for bf16 activations, causal state and decode I/O."""
    _bf16_modes = True

    @_symad_signature
    def __init__(self, *args, **params):
        super().__init__()
        _symad_init(self, _lib.MODEL_SYMAD_DECODER, *args, **params)

    def initial_decoder(self, zq):
        self.decode(zq)                                                              # AudioDec.py:224-225

    def decode(self, zq):
        """zq (B,F,code_dim) channels-last -> y (B,1,F*hop)   (AudioDec.py:246-247).  With bf16 activations zq may be bf16 or fp32
        (cast on the device) and y is bf16."""
        self._ready()
        self._want(zq, "decode", 2, self.code_dim)
        return self._decode(zq)

    def decode_offline(self, zq):
        """Decoder.forward (decoder.py:135-140): zq (B,code_dim,F) channels-first -> y (B,1,F*hop).  Discards the streaming state."""
        return self._decode_offline(zq)

    def decode_offline_varlen(self, zq, frames):
        """decode_offline over utterances of different lengths in one launch sequence: zq (1, code_dim, sum F_b) channels-first ->
        list of B waveforms (1, 1, F_b * hop), views of one output buffer, each equal to decode_offline of that utterance alone."""
        return self._decode_offline_varlen(zq, frames)

    def decode_streams(self, zq, frames, streams):
        """Advance streams[b] by frames[b] frames of zq ((1, sum F_b, code_dim) or (sum F_b, code_dim) channels-last) in one launch
        sequence -> list of B waveforms (1, 1, F_b * hop), each equal to a B = 1 streaming decode of those frames."""
        return self._decode_streams(zq, frames, streams)


class HiFiGANStreamGenerator(_StreamGeneratorBase):
    """models/vocoder/HiFiGAN.py:222-305 (AD v1: groups>1 and a single resblock kernel -> MultiGroupConv1d)."""
    _bf16_modes = True

    def __init__(self, in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=(8, 8, 2, 2),
                 upsample_kernel_sizes=(16, 16, 4, 4), resblock_kernel_sizes=(3, 7, 11),
                 resblock_dilations=[(1, 3, 5), (1, 3, 5), (1, 3, 5)], groups=1, bias=True, use_additional_convs=True,
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                 use_weight_norm=True, stats=None):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernel size must be odd number."               # HiFiGAN.py:73-75
        assert len(upsample_scales) == len(upsample_kernel_sizes)
        assert len(resblock_dilations) == len(resblock_kernel_sizes)
        multi_group = len(resblock_kernel_sizes) == 1 and groups > 1              # HiFiGAN.py:78-81
        if not multi_group:
            # MultiReceptiveField (AD v0): one residual block per kernel size, outputs averaged (multi_fusion.py:23-79)
            if groups != 1 or any(list(d) != list(resblock_dilations[0]) for d in resblock_dilations):
                raise NotImplementedError("MultiReceptiveField is built for groups=1 and identical dilation lists")
        if nonlinear_activation != "LeakyReLU" or not use_additional_convs or not bias:
            raise NotImplementedError("only LeakyReLU + additional convs + bias is built")
        c = self._cfg
        c.model_type = _lib.MODEL_HIFIGAN
        c.in_channels, c.out_channels, c.channels, c.kernel_size = in_channels, out_channels, channels, kernel_size
        c.n_up = len(upsample_scales)
        _fill(c.upsample_scales, upsample_scales), _fill(c.upsample_kernel_sizes, upsample_kernel_sizes)
        c.resblock_kernel_size = resblock_kernel_sizes[0]
        c.n_resblocks = 0 if multi_group else len(resblock_kernel_sizes)
        _fill(c.resblock_kernel_sizes, resblock_kernel_sizes)
        c.n_dil = len(resblock_dilations[0])
        _fill(c.resblock_dilations, resblock_dilations[0])
        c.groups = groups
        c.negative_slope = float(nonlinear_activation_params.get("negative_slope", 0.01))
        c.use_weight_norm = int(use_weight_norm)
        c.has_stats = int(stats is not None)       # mean/scale themselves come from the state dict (HiFiGAN.py:206-219)
        self.in_channels = in_channels

    def initial_decoder(self, c):
        self.decode(c)                                                                # HiFiGAN.py:264-265

    def decode(self, c):
        """zq (B,F,in_channels) channels-last -> y (B,1,F*prod(scales)) in (-1,1)   (HiFiGAN.py:268-296).  With bf16 activations
        zq may be bf16 or fp32 (cast on the device) and y is bf16."""
        self._ready()
        self._want(c, "decode", 2, self.in_channels)
        return self._decode(c)

    def forward(self, c):
        """Generator.forward (HiFiGAN.py:140-160), the non-streaming path: c (B,in_channels,F) channels-first -> y (B,1,F*hop).
        Discards the streaming state."""
        return self._decode_offline(c)

    __call__ = forward

    def forward_varlen(self, c, frames):
        """Generator.forward over utterances of different lengths in one launch sequence: c (1, in_channels, sum F_b) channels-first,
        utterance b at columns [sum_{i<b} F_i, +F_b) -> list of B waveforms (1, 1, F_b * hop), views of one output buffer (bf16 with
        bf16 activations), each equal to forward of that utterance alone."""
        return self._decode_offline_varlen(c, frames)

    def decode_streams(self, c, frames, streams):
        """Advance streams[b] by frames[b] frames of c ((1, sum F_b, in_channels) or (sum F_b, in_channels) channels-last) in one
        launch sequence -> list of B waveforms (1, 1, F_b * hop), views of one output buffer (bf16 with bf16 activations), each equal to
        a B = 1 streaming decode of those frames.  Streams not listed keep their state untouched."""
        return self._decode_streams(c, frames, streams)

class _StepGraph:
    """One graphed streaming step (adec_graph_*): static `input` / `output` tensors and the generators it runs.  Launching it is the
    eager call sequence it replaces, bit for bit: outputs, causal state, range / index flags and launch_count."""

    def __init__(self, kind, gens, state_gen, n_streams, size, wire, input, output):
        self._gens = gens
        for g in gens:
            g._ready()
        dev = gens[0]._device
        if any(g._device != dev for g in gens):
            raise RuntimeError(f"audiodec_b200: graph: the generators are on {[str(g._device) for g in gens]}; they must share one device")
        self._handles = [g._h.value for g in gens]
        self._state_gen, self._B = state_gen, n_streams
        self._kind, self._size, self._wire = kind, size, bool(wire)
        self._lib, self._device = gens[0]._lib, dev
        self._raw_in, self._raw_out = input, output
        self._g = None
        self._create()

    def _create(self):
        self._state_gen._batch(self._B)
        g = ctypes.c_void_p()
        a = self._gens[0]._h
        b = self._gens[1]._h if len(self._gens) > 1 else None
        _check(self._lib.adec_graph_create(self._kind, a, b, self._B, self._size, int(self._wire), _ptr(self._raw_in), _ptr(self._raw_out),
                                           ctypes.byref(g)), a)
        self._g = g

    def handles_current(self):
        """False once a generator's handle was replaced (.to() again) since the graph was made."""
        return [g._h.value if g._h is not None else None for g in self._gens] == self._handles

    def _check_handles(self):
        if not self.handles_current():
            raise RuntimeError("audiodec_b200: graph: a generator's handle was replaced (.to() again) since the graph was made; make a new graph")

    def __call__(self, x):
        """Copy x into `input` (unless x is `input`), launch the step on the current stream, return `output`.  Like torch.cuda.CUDAGraph,
        the output is a static tensor that the next call overwrites: clone it to keep it."""
        self._check_handles()
        if x is not self.input:
            if tuple(x.shape) != tuple(self.input.shape):
                raise RuntimeError(f"audiodec_b200: graph: expected input of shape {tuple(self.input.shape)}, got {tuple(x.shape)}")
            self.input.copy_(x)
        if self._state_gen.n_streams != self._B:         # what the eager call's _batch does; the launch re-captures if buffers moved
            self._state_gen._batch(self._B)
        a = self._gens[0]
        _check(self._lib.adec_graph_launch(self._g, a._stream()), a._h)
        return self.output

    def info(self):
        """{'kernels': kernels per step, 'programmatic_edges': PDL edges in the captured graph, 'instantiations': executables built}"""
        k, e, i = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _check(self._lib.adec_graph_info(self._g, ctypes.byref(k), ctypes.byref(e), ctypes.byref(i)), self._gens[0]._h)
        return {"kernels": k.value, "programmatic_edges": e.value, "instantiations": i.value}

    def __del__(self):
        try:
            if self._g is not None:
                self._lib.adec_graph_destroy(self._g)
                self._g = None
        except Exception:
            pass


class TransmitterGraph(_StepGraph):
    """tx_encoder.encode(x) -> tx_encoder.quantize(z) (tx_encoder: a full or encoder-only symAD generator) for n_streams streams of `chunk` samples as one CUDA graph launch; with wire,
    quantize_fused(z, want_idx=False, want_packed=True, want_zq=False) instead.  `input` is x (n_streams, 1, chunk), float32 (bf16 for a
    transmitter with bf16 activations, which also takes float32 x and casts it); `output`
    is what the eager calls return: indices (Nq, F) for one stream, (Nq, n_streams, F) otherwise, or with wire the packed bytes
    (F, bytes) / (n_streams, F, bytes).  The output is overwritten by the next call."""

    def __init__(self, tx_encoder, n_streams, chunk, wire=False):
        if not isinstance(tx_encoder, _SymADTransmitter):
            raise TypeError(f"audiodec_b200: TransmitterGraph needs a SymADStreamGenerator or SymADEncoderStreamGenerator (encoder, "
                            f"projector and RVQ), got {type(tx_encoder).__name__}")
        tx_encoder._ready()
        dev, b = tx_encoder._device, int(n_streams)
        f = tx_encoder._lib.adec_frames_for(tx_encoder._h, int(chunk))
        self.input = torch.zeros(b, tx_encoder.input_channels, int(chunk), device=dev, dtype=tx_encoder._act_dtype)
        if wire:
            raw = torch.empty(b, f, tx_encoder.packed_frame_bytes(), device=dev, dtype=torch.uint8)
            self.output = raw.squeeze(0) if b == 1 else raw
        else:
            raw = torch.empty(tx_encoder.codebook_num, b, f, device=dev, dtype=torch.int64)
            self.output = raw.squeeze(1) if b == 1 else raw
        super().__init__(_lib.GRAPH_TX, [tx_encoder], tx_encoder, b, int(chunk), wire, self.input, raw)


class ReceiverGraph(_StepGraph):
    """rx_encoder.lookup(idx) -> decoder.decode(zq) for n_streams streams of `frames` frames as one CUDA graph launch; with wire,
    rx_encoder.lookup_packed(packed) instead of lookup.  `decoder` is any decoder generator (symAD, symAD decoder-only or HiFi-GAN, fp32 or
    bf16).  `input` has the shape the transmitter's output has (indices or packed bytes); `output` is y (n_streams, 1, frames * hop),
    bf16 for a decoder with bf16 activations.  The output is overwritten by the next call."""

    def __init__(self, rx_encoder, decoder, n_streams, frames, wire=False):
        if not isinstance(rx_encoder, SymADStreamGenerator):
            raise TypeError(f"audiodec_b200: ReceiverGraph needs a SymADStreamGenerator as rx_encoder (its codebooks), got "
                            f"{type(rx_encoder).__name__}")
        if not isinstance(decoder, _StreamGeneratorBase):
            raise TypeError(f"audiodec_b200: ReceiverGraph needs a library decoder generator, got {type(decoder).__name__}")
        rx_encoder._ready(), decoder._ready()
        dev, b, f = rx_encoder._device, int(n_streams), int(frames)
        if wire:
            raw = torch.zeros(b, f, rx_encoder.packed_frame_bytes(), device=dev, dtype=torch.uint8)
            self.input = raw.squeeze(0) if b == 1 else raw
        else:
            raw = torch.zeros(rx_encoder.codebook_num, b, f, device=dev, dtype=torch.int64)
            self.input = raw.squeeze(1) if b == 1 else raw
        hop = decoder._lib.adec_hop_length(decoder._h)
        self.output = torch.empty(b, 1, f * hop, device=decoder._device, dtype=torch.bfloat16 if decoder._act_bf16 else torch.float32)
        super().__init__(_lib.GRAPH_RX, [rx_encoder, decoder], decoder, b, f, wire, raw, self.output)


def is_library_codec(tx_encoder, rx_encoder, decoder):
    """True when the three codec objects are this library's generators on a CUDA device, so a stream step can run as graphs."""
    return (isinstance(tx_encoder, _SymADTransmitter) and isinstance(rx_encoder, SymADStreamGenerator)
            and isinstance(decoder, _StreamGeneratorBase) and all(g._h is not None for g in (tx_encoder, rx_encoder, decoder)))


class OfflineCodec:
    """Mirror of codecTest.py's TestMain.encode / decode (codecTest.py:78-95): the non-streaming batch path.
    `encoder` is a SymADStreamGenerator, `decoder` a SymADStreamGenerator or HiFiGANStreamGenerator, both already on a
    CUDA device; they must not be the handles a live stream is using (offline calls reset the causal state)."""

    def __init__(self, encoder, decoder, multi_channel=False):
        if multi_channel and encoder.input_channels == 1:
            # codecTest.py:84-86 feeds (1,C,T) to a multi-channel generator; a mono generator would silently encode channel 0 only
            raise NotImplementedError("multi_channel=True needs a generator with input_channels > 1 (only mono generators are built)")
        self.encoder, self.decoder, self.multi_channel = encoder, decoder, multi_channel

    def encode(self, audio):
        """audio (T,C) float array -> zq (C,code_dim,F) (or (1,code_dim,F) when multi_channel)."""
        x = torch.as_tensor(audio, dtype=torch.float32).to(self.encoder._device)
        x = x.transpose(1, 0).unsqueeze(0) if self.multi_channel else x.transpose(1, 0).unsqueeze(1)
        zq, _ = self.encoder.quantize_offline(self.encoder.encode_offline(x))
        return zq

    def decode(self, zq):
        return self.decoder.forward(zq) if isinstance(self.decoder, HiFiGANStreamGenerator) else self.decoder.decode_offline(zq)

    def encode_many(self, audios):
        """encode() of every (T_i, C_i) array in `audios` through ONE varlen encode and quantize: each audio channel is an utterance.
        Returns [zq_i (C_i, code_dim, F_i)], equal to [encode(a) for a in audios]."""
        if self.multi_channel:
            raise NotImplementedError("encode_many runs one utterance per audio channel (multi_channel=False)")
        dev = self.encoder._device
        arrs = [torch.as_tensor(a, dtype=torch.float32) for a in audios]
        chans = [x.shape[1] for x in arrs]
        rows = torch.cat([x.transpose(1, 0).reshape(-1) for x in arrs]).to(dev)      # channel-major: one utterance per (file, channel)
        lengths = [x.shape[0] for x, c in zip(arrs, chans) for _ in range(c)]
        z, frames = self.encoder.encode_offline_varlen(list(torch.split(rows, lengths)))
        zq, _ = self.encoder.quantize_offline(z)                                       # (1, code_dim, sum F)
        cols = list(torch.split(zq[0], frames, dim=1))
        out, k = [], 0
        for c in chans:
            out.append(torch.stack(cols[k:k + c]))
            k += c
        return out

    def decode_many(self, zqs):
        """decode() of every zq_i (C_i, code_dim, F_i) through ONE varlen decode.  Returns [y_i (C_i, 1, F_i * hop)], equal to
        [decode(zq) for zq in zqs]."""
        chans = [zq.size(0) for zq in zqs]
        frames = [zq.size(2) for zq in zqs for _ in range(zq.size(0))]
        c = torch.cat([zq[i] for zq in zqs for i in range(zq.size(0))], dim=1).unsqueeze(0)
        fn = self.decoder.forward_varlen if isinstance(self.decoder, HiFiGANStreamGenerator) else self.decoder.decode_offline_varlen
        ys = fn(c, frames)
        out, k = [], 0
        for n in chans:
            out.append(torch.cat(ys[k:k + n]))
            k += n
        return out


def codec_host(encoder: SymADStreamGenerator, decoder, x_host: torch.Tensor, want_idx=True, reuse_buffers=False):
    """Whole path on HOST buffers through ``adec_codec_host`` (H2D + encode + quantize + lookup + decode +
    D2H), i.e. what demoFile.py:55-62 does around the four calls.  x_host: (B,1,T) float32 CPU tensor
    (pinned for full PCIe speed).  With reuse_buffers the returned tensors are views of cached pinned buffers that
    the next call overwrites.  Returns (idx (Nq,B,F) int64 CPU or None, y (B,1,F*hop) float32 CPU)."""
    encoder._ready(), decoder._ready()
    assert x_host.device.type == "cpu" and x_host.dtype == torch.float32 and x_host.is_contiguous()
    b, _, t = x_host.shape
    encoder._batch(b)
    if decoder is not encoder:
        decoder._batch(b)
    lib = encoder._lib
    f = lib.adec_frames_for(encoder._h, t)
    hop = lib.adec_hop_length(decoder._h)
    pin = x_host.is_pinned()
    # page-locked result buffers are expensive to create (cudaHostAlloc): keep one set per shape and hand out views;
    # pass reuse_buffers=False to get fresh tensors that the next call will not overwrite
    cache = encoder.__dict__.setdefault("_host_out", {})
    key = (b, f, hop, pin, want_idx)
    if reuse_buffers and key in cache:
        idx, y = cache[key]
    else:
        idx = torch.empty(encoder.codebook_num, b, f, dtype=torch.int64, pin_memory=pin) if want_idx else None
        y = torch.empty(b, 1, f * hop, dtype=torch.float32, pin_memory=pin)
        if reuse_buffers:
            cache.clear()
            cache[key] = (idx, y)
    _check(lib.adec_codec_host(encoder._h, decoder._h, _ptr(x_host), b, t, _ptr(idx) if want_idx else None,
                               _ptr(y), encoder._stream()), encoder._h)
    return idx, y
