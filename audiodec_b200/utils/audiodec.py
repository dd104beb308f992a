"""Drop-in for the reference's ``utils/audiodec.py``: ``AudioDec``, ``AudioDecStreamer``,
``assign_model`` with the same signatures, so ``demoFile.py`` / ``demoStream.py`` only change their
import line (see INTEGRATION.md).  The objects returned by ``_load_encoder`` / ``_load_decoder`` are the
CUDA-backed generators of ``audiodec_b200.codec`` instead of torch modules."""
from __future__ import annotations

import math
import os
from typing import Union

import torch

from audiodec_b200.bin.stream import AudioCodec, AudioCodecStreamer
from audiodec_b200.codec import HiFiGANStreamGenerator, ReceiverGraph, SymADStreamGenerator, TransmitterGraph, is_library_codec

_AUTOENCODER_TYPES = ("symAudioDec", "symAudioDecUniv")      # utils/audiodec.py:36,48
_VOCODER_TYPES = ("HiFiGAN", "UnivNet")                      # utils/audiodec.py:50


def _load_generator(cls, config, checkpoint):
    gen = cls(**config["generator_params"])
    gen.load_state_dict(torch.load(checkpoint, map_location="cpu")["model"]["generator"])
    return gen


class AudioDec(AudioCodec):
    def __init__(self, tx_device: str = "cpu", rx_device: str = "cpu", receptive_length: int = 8192):
        # 8192 >= the encoder's receptive field of 7209 samples (utils/audiodec.py:24)
        super().__init__(tx_device=tx_device, rx_device=rx_device, receptive_length=receptive_length)

    def _load_encoder(self, checkpoint):
        config = self._load_config(checkpoint)
        if config["model_type"] not in _AUTOENCODER_TYPES:
            raise NotImplementedError(f"Encoder type {config['model_type']} is not supported!")
        return _load_generator(SymADStreamGenerator, config, checkpoint)

    def _load_decoder(self, checkpoint):
        config = self._load_config(checkpoint)
        if config["model_type"] in _AUTOENCODER_TYPES:
            return _load_generator(SymADStreamGenerator, config, checkpoint)
        if config["model_type"] in _VOCODER_TYPES:
            return _load_generator(HiFiGANStreamGenerator, config, checkpoint)
        raise NotImplementedError(f"Decoder {config['model_type']} is not supported!")

    def get_hop_length(self, checkpoint):
        assert os.path.exists(checkpoint), f"{checkpoint} does not exist!"
        return math.prod(self._load_config(checkpoint)["generator_params"]["enc_strides"])


class AudioDecStreamer(AudioCodecStreamer):
    def __init__(self, input_device: Union[str, int], output_device: Union[str, int], input_channels: int = 1,
                 output_channels: int = 1, frame_size: int = 512, sample_rate: int = 48000, gain: int = 1.0,
                 max_latency: float = 0.1, tx_encoder=None, tx_device: str = "cpu", rx_encoder=None, decoder=None,
                 rx_device: str = "cpu"):
        super().__init__(input_device=input_device, output_device=output_device, input_channels=input_channels,
                         output_channels=output_channels, frame_size=frame_size, sample_rate=sample_rate, gain=gain,
                         max_latency=max_latency, tx_encoder=tx_encoder, tx_device=tx_device, rx_encoder=rx_encoder,
                         decoder=decoder, rx_device=rx_device)

    # On the library's generators each worker's step is one graph launch (TransmitterGraph / ReceiverGraph).  Both graphs are made
    # in _start_threads, on the calling thread, before the workers run: a capture must not overlap the other worker's device
    # synchronise.  A frame of another shape, or a generator whose handle was replaced, takes the eager calls.  The static output is
    # cloned before it goes into the queue: the other thread reads it after this thread's next launch.
    def _start_threads(self):
        if not self._threads_started:
            self._tx_graph = self._rx_graph = None
            if is_library_codec(self.tx_encoder, self.rx_encoder, self.decoder) and torch.device(self.tx_device).type == "cuda" \
                    and torch.device(self.rx_device).type == "cuda":
                frames = self.tx_encoder._lib.adec_frames_for(self.tx_encoder._h, self.frame_size)
                self._tx_graph = TransmitterGraph(self.tx_encoder, 1, self.frame_size)
                self._rx_graph = ReceiverGraph(self.rx_encoder, self.decoder, 1, frames)
        super()._start_threads()

    @staticmethod
    def _graph_for(graph, x):
        """the graph when x is its input's shape on its device and its generators keep their handles, else None"""
        if graph is None or tuple(x.shape) != tuple(graph.input.shape) or x.device != graph.input.device:
            return None
        return graph if graph.handles_current() else None

    def _encode(self, x):                       # utils/audiodec.py:100-102
        g = self._graph_for(getattr(self, "_tx_graph", None), x)
        if g is not None:
            return g(x).clone()
        return self.tx_encoder.quantize(self.tx_encoder.encode(x))

    def _decode(self, x):                       # utils/audiodec.py:104-106
        g = self._graph_for(getattr(self, "_rx_graph", None), x)
        if g is not None:
            return g(x).clone()
        return self.decoder.decode(self.rx_encoder.lookup(x))


# model name -> (sample rate, encoder dir, encoder steps, decoder dir, decoder steps); utils/audiodec.py:109-179
_AE, _VOC, _DN = "autoencoder", "vocoder", "denoise"
_MODELS = {
    "libritts_v1": (24000, (_AE, "symAD_libritts_24000_hop300", 500000), (_VOC, "AudioDec_v1_symAD_libritts_24000_hop300_clean", 500000)),
    "libritts_sym": (24000, (_AE, "symAD_libritts_24000_hop300", 500000), (_AE, "symAD_libritts_24000_hop300", 1000000)),
    "vctk_v1": (48000, (_AE, "symAD_vctk_48000_hop300", 200000), (_VOC, "AudioDec_v1_symAD_vctk_48000_hop300_clean", 500000)),
    "vctk_sym": (48000, (_AE, "symAD_vctk_48000_hop300", 200000), (_AE, "symAD_vctk_48000_hop300", 700000)),
    "vctk_v0": (48000, (_AE, "symAD_vctk_48000_hop300", 200000), (_VOC, "AudioDec_v0_symAD_vctk_48000_hop300_clean", 500000)),
    "vctk_v2": (48000, (_AE, "symAD_vctk_48000_hop300", 200000), (_VOC, "AudioDec_v2_symAD_vctk_48000_hop300_clean", 500000)),
    "vctk_denoise": (48000, (_DN, "symAD_vctk_48000_hop300", 200000), (_VOC, "AudioDec_v1_symAD_vctk_48000_hop300_clean", 500000)),
    "vctk_univ": (48000, (_AE, "symADuniv_vctk_48000_hop300", 500000), (_VOC, "AudioDec_v3_symADuniv_vctk_48000_hop300_clean", 500000)),
    "vctk_univ_sym": (48000, (_AE, "symADuniv_vctk_48000_hop300", 500000), (_AE, "symADuniv_vctk_48000_hop300", 1000000)),
    "vctk_activate_sym": (48000, (_AE, "symAAD_vctk_48000_hop300", 200000), (_AE, "symAAD_vctk_48000_hop300", 700000)),
    "vctk_c16h320_sym": (48000, (_AE, "symAD_c16_vctk_48000_hop320", 500000), (_AE, "symAD_c16_vctk_48000_hop320", 1000000)),
}


def assign_model(model):
    """name -> (sample_rate, encoder_checkpoint, decoder_checkpoint), cwd-relative like the reference."""
    if model not in _MODELS:
        raise NotImplementedError(f"Model {model} is not supported!")
    sr, enc, dec = _MODELS[model]
    path = lambda kind, tag, steps: os.path.join("exp", kind, tag, f"checkpoint-{steps}steps.pkl")
    return sr, path(*enc), path(*dec)
