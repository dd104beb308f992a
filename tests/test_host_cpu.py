"""CPU-only checks of the host side: the C-ABI library loads and exports every symbol the header
declares, config mirroring, the reference-facing API surface, error behaviour without a GPU, and the
multi-process (gloo, world_size 2) sharding logic."""
import ctypes
import os
import re
import socket
import subprocess
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from audiodec_b200 import _lib
    hdr = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    declared = set(re.findall(r"\b(adec_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.SYMBOLS), "python binding table and header disagree"
    _lib.load()


def test_config_struct_matches_header_field_order():
    from audiodec_b200 import _lib
    hdr = open(os.path.join(REPO, "include", "audiodec_b200.h")).read()
    body = hdr[hdr.index("typedef struct adec_config {"):hdr.index("} adec_config;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"\b(?:int|float)\s+([^;]+);", body)
    fields = []
    for group in names:
        for item in group.split(","):
            fields.append(re.sub(r"\[.*\]", "", item).strip())
    assert fields == [f[0] for f in _lib.AdecConfig._fields_]


def test_no_gpu_means_loud_failure(symad_sd):
    """There is no CPU fallback: without a usable CUDA device the product path raises."""
    from audiodec_b200 import synthetic as S
    from audiodec_b200.codec import SymADStreamGenerator
    g = SymADStreamGenerator(**S.SYMAD_PARAMS)
    g.load_state_dict(symad_sd)
    with pytest.raises(RuntimeError):
        g.to("cpu")
    with pytest.raises(RuntimeError):
        g.encode(torch.zeros(1, 1, 300))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no usable CUDA device|CUDA"):
            g.to("cuda:0")


def test_product_never_imports_oracle():
    pkg = os.path.join(REPO, "audiodec_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(root, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_unsupported_variants_raise_like_the_reference():
    from audiodec_b200.codec import HiFiGANStreamGenerator, SymADStreamGenerator
    with pytest.raises(NotImplementedError):
        SymADStreamGenerator(codec="unknown")
    SymADStreamGenerator(codec="activate_audiodec", use_weight_norm=True)      # symAAD is built
    HiFiGANStreamGenerator(in_channels=64, groups=1)                           # AD v0 (MultiReceptiveField) is built
    with pytest.raises(NotImplementedError):
        HiFiGANStreamGenerator(groups=1, resblock_dilations=[(1, 3, 5), (1, 3), (1, 3, 5)])
    with pytest.raises(AssertionError):
        SymADStreamGenerator(mode="noncausal")             # models/utils.py:13-15
    with pytest.raises(AssertionError):
        HiFiGANStreamGenerator(kernel_size=6)              # HiFiGAN.py:73


def test_audiodec_api_surface(tmp_path):
    from audiodec_b200 import synthetic as S
    from audiodec_b200.utils.audiodec import AudioDec, AudioDecStreamer, assign_model
    sr, enc, dec = assign_model("vctk_v1")
    assert sr == 48000 and enc.endswith("symAD_vctk_48000_hop300/checkpoint-200000steps.pkl")
    with pytest.raises(NotImplementedError):
        assign_model("nope")
    sr, enc, dec = S.make_model_zoo(str(tmp_path), "vctk_v1")
    a = AudioDec(tx_device="cuda:0", rx_device="cuda:0")
    assert a.receptive_length == 8192
    assert a.get_hop_length(enc) == 300
    tx = a._load_encoder(enc)            # builds the generator on the host; no GPU touched yet
    assert type(tx).__name__ == "SymADStreamGenerator"
    assert type(a._load_decoder(dec)).__name__ == "HiFiGANStreamGenerator"
    with pytest.raises(NotImplementedError):
        a._load_encoder(dec)             # a vocoder checkpoint is not an encoder (utils/audiodec.py:36-39)
    with pytest.raises(AssertionError):
        a.load_transmitter(str(tmp_path / "missing.pkl"))
    s = AudioDecStreamer(input_device=0, output_device=0, frame_size=1500, tx_encoder=None)
    assert s.frame_size == 1500 and s.frame_drops == 0


def test_shard_bounds():
    from audiodec_b200.shard import shard_bounds
    assert shard_bounds(512, 8) == [(64 * r, 64 * r + 64) for r in range(8)]
    assert shard_bounds(5, 2) == [(0, 3), (3, 5)]
    assert shard_bounds(1, 4) == [(0, 1), (1, 1), (1, 1), (1, 1)]
    for n in (0, 1, 7, 64, 511):
        b = shard_bounds(n, 8)
        assert b[0][0] == 0 and b[-1][1] == n and all(b[i][1] == b[i + 1][0] for i in range(7))


def _worker(rank, world, port, q):
    import torch.distributed as dist
    sys.path.insert(0, REPO)
    from audiodec_b200.shard import run_sharded
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    torch.manual_seed(0)
    x = torch.randn(5, 1, 600)          # 5 utterances over 2 ranks: ragged shards (3 + 2)

    def fake_codec(xs):                  # stands in for the GPU codec: any per-utterance function
        f = xs.shape[-1] // 300
        idx = (xs[:, 0, :f * 300].reshape(xs.shape[0], f, 300).sum(-1) * 100).long().unsqueeze(0).repeat(8, 1, 1)
        return idx, xs * 2.0

    idx, y, (lo, hi) = run_sharded(x, fake_codec, rank, world)
    ridx, ry = fake_codec(x)
    ok = torch.equal(idx, ridx) and torch.equal(y, ry) and (lo, hi) == ((0, 3) if rank == 0 else (3, 5))
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_sharded_equals_unsharded_gloo_world2():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = dict(q.get(timeout=120) for _ in range(2))
    [p.join(timeout=60) for p in procs]
    assert res == {0: True, 1: True}


def test_c_rvq_oracle_matches_torch_bitwise():
    """oracle/rvq_oracle.c (the plain-C spec the CUDA RVQ kernel mirrors) reproduces torch-CPU's distances
    and decisions bit-for-bit on random data (the summation orders in its header were found by probing)."""
    import numpy as np
    from oracle import audiodec_oracle as O
    from oracle import rvq_spec
    torch.manual_seed(5)
    nq, d, n, frames = 8, 64, 1024, 200
    embeds = [torch.randn(d, n) * 0.55 * 0.88 ** i for i in range(nq)]
    x = torch.randn(1, frames, d) * 0.6
    zq, idx = O.rvq_forward_index(x, embeds, True)
    oidx, ozq, od = rvq_spec.rvq_frames(x[0].numpy(), torch.stack(embeds).numpy(), dist=True)
    np.testing.assert_array_equal(oidx, idx.squeeze(1).numpy())
    fl = x.reshape(-1, d)
    dist0 = fl.pow(2).sum(1, keepdim=True) - 2 * fl @ embeds[0] + embeds[0].pow(2).sum(0, keepdim=True)
    same = (od[0] == dist0.numpy()).mean()
    assert same > 0.999, f"only {same:.4f} of the fp32 distances are bit-identical on this CPU"
    np.testing.assert_allclose(ozq, zq[0].numpy(), atol=1e-6)


def test_bench_reference_arm_prints_the_contract_line():
    """bench.py --impl reference runs on the host alone (oracle port) and prints ONE JSON line with the keys the
    driver reads; under torchrun only rank 0 prints."""
    import json
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--ref-utts", "1"]
    out = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["value"] > 0 and d["unit"] == "samples/s" and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert "workload" in d["config"] and "model" not in d["config"]
    # a non-zero rank exits 0 without printing
    out = subprocess.run(cmd, capture_output=True, text=True, env=dict(env, RANK="1", WORLD_SIZE="2"), timeout=600)
    assert out.returncode == 0 and not [l for l in out.stdout.splitlines() if l.startswith("{")]


def test_bench_cuda_arm_fails_loudly_without_a_gpu():
    out = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--steps", "1", "--warmup", "3", "--no-cpu-baseline"],
                         capture_output=True, text=True, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), timeout=600)
    assert out.returncode != 0
    assert not [l for l in out.stdout.splitlines() if l.startswith("{")]


def test_wav_io_pcm16_round_trip(tmp_path):
    """audiodec_b200/wavio.py: demoFile.py's sf.read(always_2d) / sf.write(PCM_16) conventions."""
    import numpy as np
    from audiodec_b200.wavio import read_wav, write_wav_pcm16
    p = str(tmp_path / "a.wav")
    x = np.stack([np.array([0.0, 0.5, -1.0, 1.0, 0.25], np.float32), np.array([0.1, -0.1, 0.0, 0.9, -0.9], np.float32)], axis=1)
    write_wav_pcm16(p, x, 48000)
    y, fs = read_wav(p)
    assert fs == 48000 and y.shape == (5, 2) and y.dtype == np.float32
    np.testing.assert_allclose(y, x, atol=5e-5)         # 32767 on write, 32768 on read, half an LSB of rounding
    from scipy.io import wavfile
    raw = wavfile.read(p)[1]
    assert raw.dtype == np.int16 and raw[:, 0].tolist() == [0, 16384, -32767, 32767, 8192]
    write_wav_pcm16(p, x[:, 0], 24000)                     # mono (T,) is written and read back as (T, 1)
    y1, fs1 = read_wav(p)
    assert fs1 == 24000 and y1.shape == (5, 1)


def test_demo_file_cli_refuses_cpu_and_missing_input(tmp_path):
    from audiodec_b200 import demo_file
    with pytest.raises(SystemExit):
        demo_file.main(["--model", "vctk_v1", "-i", "x.wav", "-o", "y.wav", "--cuda", "-1"])
    with pytest.raises(NotImplementedError):
        demo_file.main(["--model", "no_such_model", "-i", "x.wav", "-o", "y.wav"])
    with pytest.raises(ValueError):
        demo_file.main(["--model", "vctk_v1", "-i", str(tmp_path / "missing.wav"), "-o", "y.wav"])


def test_time_pairing_identity():
    """Design check for DESIGN.md section 8 item 1 (tools/pairing_math.py): the paired-weight GEMM over de-interleaved windows equals the
    dilated causal conv it replaces, for the dilations and kernel sizes of the symAD units and the HiFi-GAN blocks."""
    import importlib.util
    import numpy as np
    spec = importlib.util.spec_from_file_location("pairing_math", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "pairing_math.py"))
    pm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(pm)
    rng = np.random.default_rng(1)
    for (K, d, C, T) in ((7, 1, 16, 64), (7, 3, 16, 60), (7, 9, 16, 72), (11, 5, 8, 40)):
        W = rng.standard_normal((K, C, C)).astype(np.float32)
        xt = rng.standard_normal((T + (K - 1) * d, C)).astype(np.float32)
        np.testing.assert_allclose(pm.paired(xt, W, d), pm.direct(xt.astype(np.float64), W.astype(np.float64), d), atol=1e-9)
