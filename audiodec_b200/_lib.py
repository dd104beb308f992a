"""ctypes binding of the C ABI declared in include/audiodec_b200.h.

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no
CPU or PyTorch fallback: if the library is missing, or no CUDA device is usable, every entry point
raises."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ADEC_LIB_PATH") or os.path.join(_HERE, "lib", "libaudiodec_b200.so")   # override: A/B experiments only
MAX_STAGES = 8

c_int, c_float, c_void_p, c_char_p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_char_p
c_int64 = ctypes.c_int64
_I8 = c_int * MAX_STAGES


class AdecConfig(ctypes.Structure):
    """struct adec_config (include/audiodec_b200.h)."""
    _fields_ = [
        ("model_type", c_int),
        ("input_channels", c_int), ("output_channels", c_int), ("encode_channels", c_int), ("decode_channels", c_int),
        ("code_dim", c_int), ("codebook_num", c_int), ("codebook_size", c_int),
        ("n_enc", c_int), ("enc_ratios", _I8), ("enc_strides", _I8),
        ("n_dec", c_int), ("dec_ratios", _I8), ("dec_strides", _I8),
        ("bias", c_int),
        ("in_channels", c_int), ("out_channels", c_int), ("channels", c_int), ("kernel_size", c_int),
        ("n_up", c_int), ("upsample_scales", _I8), ("upsample_kernel_sizes", _I8),
        ("resblock_kernel_size", c_int),
        ("n_dil", c_int), ("resblock_dilations", _I8),
        ("groups", c_int),
        ("negative_slope", c_float),
        ("use_weight_norm", c_int),
        ("has_stats", c_int),
        ("codec_activate", c_int),
        ("n_resblocks", c_int), ("resblock_kernel_sizes", _I8),
        ("compute_dtype", c_int),
    ]


MODEL_SYMAD, MODEL_HIFIGAN, MODEL_SYMAD_DECODER, MODEL_SYMAD_ENCODER = 0, 1, 2, 3
GRAPH_TX, GRAPH_RX = 0, 1


class AdecTestOp(ctypes.Structure):
    """struct adec_test_op (include/audiodec_b200.h)."""
    _fields_ = [
        ("kind", c_int), ("Cin", c_int), ("Cout", c_int), ("K", c_int), ("stride", c_int), ("dil", c_int), ("groups", c_int),
        ("shared_in", c_int), ("pre_act", c_int), ("slope", c_float), ("out_nct", c_int), ("post_tanh", c_int),
        ("w", c_void_p), ("w2", c_void_p), ("bias", c_void_p), ("mean", c_void_p), ("scale", c_void_p),
        ("compute_dtype", c_int),
    ]


class AdecConcealRow(ctypes.Structure):
    """struct adec_conceal_row (include/audiodec_b200.h): one output row of adec_lookup_packed_conceal."""
    _fields_ = [("src", ctypes.c_int32), ("next", ctypes.c_int32), ("slot", ctypes.c_int32), ("j", ctypes.c_int32),
                ("den", ctypes.c_int32)]


class AdecPlayoutRow(ctypes.Structure):
    """struct adec_playout_row (include/audiodec_b200.h): one output row of adec_lookup_packed_playout / _timescale."""
    _fields_ = [("src", ctypes.c_int32), ("next", ctypes.c_int32), ("target", ctypes.c_int32), ("slot", ctypes.c_int32),
                ("j", ctypes.c_int32), ("den", ctypes.c_int32)]


TEST_CONV, TEST_RU, TEST_CONVTR, TEST_STEM, TEST_HEAD = 0, 1, 2, 3, 4
TEST_REC = 9

# name -> (restype, argtypes); every symbol include/audiodec_b200.h declares
SYMBOLS = {
    "adec_create": (c_int, [ctypes.POINTER(AdecConfig), c_int, ctypes.POINTER(c_void_p)]),
    "adec_destroy": (None, [c_void_p]),
    "adec_last_error": (c_char_p, [c_void_p]),
    "adec_set_tensor": (c_int, [c_void_p, c_char_p, c_void_p, ctypes.POINTER(c_int64), c_int]),
    "adec_finalize": (c_int, [c_void_p]),
    "adec_n_streams": (c_int, [c_void_p]),
    "adec_set_streams": (c_int, [c_void_p, c_int]),
    "adec_reset": (c_int, [c_void_p, c_void_p]),
    "adec_encode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_quantize": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_quantize_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "adec_quantize_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "adec_zq_moments": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p, c_void_p]),
    "adec_lookup": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_lookup_packed": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_lookup_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_lookup_packed_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_lookup_packed_conceal": (c_int, [c_void_p, c_void_p, c_int, ctypes.POINTER(AdecConcealRow), c_int, c_void_p, c_int, c_void_p,
                                           c_void_p]),
    "adec_lookup_packed_conceal_bf16": (c_int, [c_void_p, c_void_p, c_int, ctypes.POINTER(AdecConcealRow), c_int, c_void_p, c_int,
                                                c_void_p, c_void_p]),
    "adec_lookup_packed_playout": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                           c_void_p]),
    "adec_lookup_packed_playout_bf16": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                                                c_void_p, c_void_p]),
    "adec_lookup_packed_timescale": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                             c_void_p]),
    "adec_lookup_packed_timescale_bf16": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                                                  c_void_p, c_void_p]),
    "adec_graph_create": (c_int, [c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, ctypes.POINTER(c_void_p)]),
    "adec_graph_launch": (c_int, [c_void_p, c_void_p]),
    "adec_graph_info": (c_int, [c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "adec_graph_destroy": (c_int, [c_void_p]),
    "adec_decode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_encode_offline": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_decode_offline": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_decode_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_encode_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_encode_offline_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_encode_offline_varlen_bf16": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_encode_streams_bf16": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_quantize_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_quantize_ex_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "adec_decode_offline_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_encode_offline_varlen": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_decode_offline_varlen": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_decode_offline_varlen_bf16": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_encode_streams": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_decode_streams": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_decode_streams_bf16": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_copy_stream_state": (c_int, [c_void_p, c_int, ctypes.POINTER(c_int), c_int, c_void_p]),
    "adec_state_entries": (c_int, [c_void_p]),
    "adec_state_entry": (c_int, [c_void_p, c_int, ctypes.POINTER(c_char_p), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "adec_stream_state_elems": (c_int64, [c_void_p]),
    "adec_get_stream_state": (c_int, [c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_set_stream_state": (c_int, [c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_void_p]),
    "adec_frames_for": (c_int, [c_void_p, c_int]),
    "adec_hop_length": (c_int, [c_void_p]),
    "adec_codec_host": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "adec_packed_frame_bytes": (c_int, [c_void_p]),
    "adec_pack_indices": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_unpack_indices": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_index_error": (c_int, [c_void_p, c_void_p]),
    "adec_range_error": (c_int, [c_void_p, c_void_p]),
    "adec_launch_count": (c_int64, [c_void_p]),
    "adec_ktrace": (c_int, [c_void_p, ctypes.POINTER(ctypes.c_ulonglong), c_int]),
    "adec_probe_mma": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]),
    "adec_profile": (c_int, [c_void_p, c_int]),
    "adec_profile_report": (c_int, [c_void_p, c_char_p, c_int]),
    "adec_test_causal_conv": (c_int, [c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                      c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "adec_test_residual_unit": (c_int, [c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "adec_test_wgmma_columns": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "adec_test_causal_convtr": (c_int, [c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                        c_void_p, c_void_p]),
    "adec_test_vocoder_layer": (c_int, [c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                        c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "adec_test_conv_op": (c_int, [c_int, ctypes.POINTER(AdecTestOp), c_int, c_int, c_int, c_int, ctypes.POINTER(c_int),
                                  ctypes.POINTER(c_int), c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(c_int), c_int,
                                  ctypes.POINTER(c_int)]),
    "adec_record_launches": (c_int, [c_void_p, c_int]),
    "adec_launch_records": (c_int, [c_void_p, ctypes.POINTER(c_int), c_int]),
}

_lib = None


def load():
    """Load (once) and return the CDLL with argtypes set.  Raises if the extension was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build the CUDA extension first "
            "(python -c 'import __graft_entry__ as g; g.build()').  audiodec_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error(handle=None) -> str:
    msg = load().adec_last_error(handle)
    return msg.decode() if msg else ""
