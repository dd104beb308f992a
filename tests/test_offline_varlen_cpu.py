"""CPU checks of the varlen offline codec's host side: the bindings, the frame / offset arithmetic, and the batched codecTest.py's
refusals."""
import math
import os
import re
import subprocess
import sys

from audiodec_b200 import synthetic as S

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARLEN = ("adec_encode_offline_varlen", "adec_decode_offline_varlen", "adec_decode_offline_varlen_bf16")


def test_bindings_declare_the_varlen_entry_points():
    """The header declares them (so test_library_exports_every_declared_symbol checks the library exports them) and the binding
    table passes the lengths as a host int array."""
    import ctypes
    from audiodec_b200 import _lib
    hdr = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    declared = set(re.findall(r"\b(adec_[a-z_0-9]+)\s*\(", hdr))
    for name in VARLEN:
        assert name in declared and name in _lib.SYMBOLS
        assert _lib.SYMBOLS[name][1][2] is ctypes.POINTER(ctypes.c_int)
        assert hasattr(_lib.load(), name)


def test_frame_and_offset_arithmetic_matches_frames_for():
    """varlen_layout's F_b is frames_for(T_b) (floor((t - 1) / s) + 1 per stride = ceil(T / hop)) for every length up to 12 s at
    48 kHz, and its offsets are the running sums that place each utterance in z / zq (and, times the hop, in y)."""
    from audiodec_b200.codec import varlen_layout
    for params in (S.SYMAD_PARAMS, S.SYMAD_C16_PARAMS):
        strides = params["enc_strides"]
        hop = math.prod(strides)
        lengths = list(range(1, 12 * 48000 + 1))
        frames, offsets = varlen_layout(lengths, strides)
        assert frames == [-(-t // hop) for t in lengths]
        assert len(offsets) == len(lengths) + 1 and offsets[0] == 0
        assert all(offsets[i + 1] - offsets[i] == f for i, f in enumerate(frames[:5000]))
        assert offsets[-1] == sum(frames)
    assert varlen_layout([], (3, 4, 5, 5)) == ([], [0])


def _cli(*args):
    return subprocess.run([sys.executable, "-m", "audiodec_b200.codec_test", *args], cwd=REPO, capture_output=True, text=True)


def test_codec_test_cli_refuses_cpu_and_missing_inputs(tmp_path):
    r = _cli("--encoder", "e.pkl", "--decoder", "d.pkl", "--output_dir", str(tmp_path), "--cuda", "-1")
    assert r.returncode != 0 and "no CPU path" in r.stderr
    r = _cli("--encoder", str(tmp_path / "missing.pkl"), "--decoder", str(tmp_path / "missing.pkl"), "--output_dir", str(tmp_path))
    assert r.returncode != 0 and "does not exist" in r.stderr
    _, enc, dec = S.make_model_zoo(str(tmp_path / "zoo"), "vctk_sym")
    r = _cli("--encoder", enc, "--decoder", dec, "--output_dir", str(tmp_path), "--batch_seconds", "0")
    assert r.returncode != 0 and "batch_seconds" in r.stderr
    r = _cli("--encoder", enc, "--decoder", dec, "--output_dir", str(tmp_path))            # the config names no data folder
    assert r.returncode != 0 and "data" in r.stderr
    r = _cli("--encoder", enc, "--output_dir", str(tmp_path))
    assert r.returncode != 0 and "--decoder" in r.stderr
