"""Host-side logic of the product path that needs no GPU: wav ingest vs the oracle's reader,
CLI argument validation, rank sharding and the world_size-2 gloo exchange."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from nisqa_b200 import dist as nb_dist
from nisqa_b200 import wav
from oracle import librosa_compat as lb


def _write_pcm(path, data_bytes, tag, ch, sr, bits, extensible=False):
    ba = ch * bits // 8
    if extensible:
        fmt = struct.pack("<HHIIHHHHIH14s", 0xFFFE, ch, sr, sr * ba, ba, bits, 22, bits, 0, tag, b"\x00" * 14)
    else:
        fmt = struct.pack("<HHIIHH", tag, ch, sr, sr * ba, ba, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"LIST" + struct.pack("<I", 4) + b"abcd" \
        + b"data" + struct.pack("<I", len(data_bytes)) + data_bytes
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


def _as_float(x):
    return x.astype(np.float32) / np.float32(32768.0) if x.dtype == np.int16 else x


@pytest.mark.parametrize("kind", ["pcm16", "pcm16_stereo", "pcm24", "pcm32", "f32", "f64", "u8", "ext16", "alaw", "ulaw_stereo"])
def test_wav_reader_matches_oracle_loader(tmp_path, kind):
    rng = np.random.default_rng(1)
    p = str(tmp_path / (kind + ".wav"))
    n = 1000
    if kind in ("pcm16", "ext16"):
        d = rng.integers(-32768, 32767, n).astype("<i2")
        _write_pcm(p, d.tobytes(), 1, 1, 16000, 16, extensible=(kind == "ext16"))
    elif kind == "pcm16_stereo":
        d = rng.integers(-32768, 32767, (n, 2)).astype("<i2")
        _write_pcm(p, d.tobytes(), 1, 2, 44100, 16)
    elif kind == "pcm24":
        v = rng.integers(-(1 << 23), (1 << 23) - 1, n)
        b = bytearray()
        for x in v:
            b += int(x & 0xFFFFFF).to_bytes(3, "little")
        _write_pcm(p, bytes(b), 1, 1, 48000, 24)
    elif kind == "pcm32":
        d = rng.integers(-(1 << 31), (1 << 31) - 1, n).astype("<i4")
        _write_pcm(p, d.tobytes(), 1, 1, 48000, 32)
    elif kind == "alaw":
        _write_pcm(p, np.arange(n, dtype=np.int64).astype(np.uint8).tobytes(), 6, 1, 8000, 8)          # every code
    elif kind == "ulaw_stereo":
        _write_pcm(p, rng.integers(0, 256, (n, 2)).astype(np.uint8).tobytes(), 7, 2, 8000, 8)
    elif kind == "f32":
        _write_pcm(p, rng.standard_normal((n, 2)).astype("<f4").tobytes(), 3, 2, 22050, 32)
    elif kind == "f64":
        _write_pcm(p, rng.standard_normal(n).astype("<f8").tobytes(), 3, 1, 8000, 64)
    else:
        _write_pcm(p, rng.integers(0, 255, n).astype(np.uint8).tobytes(), 1, 1, 8000, 8)
    y_ref, sr_ref = lb.load(p, sr=None)
    y, sr = wav.read_wav(p)
    assert sr == sr_ref and y.ndim == 1
    np.testing.assert_array_equal(_as_float(y), y_ref)
    if kind in ("alaw", "ulaw_stereo"):
        # independent decoder: the standard library's G.711 tables
        audioop = pytest.importorskip("audioop")
        raw = open(p, "rb").read()[-n * (2 if kind == "ulaw_stereo" else 1):]
        lin = np.frombuffer((audioop.alaw2lin if kind == "alaw" else audioop.ulaw2lin)(raw, 2), dtype="<i2")
        want = lin.astype(np.float32) / np.float32(32768.0)
        if kind == "ulaw_stereo":
            want = np.mean(want.reshape(n, 2).T, axis=0)
        np.testing.assert_array_equal(_as_float(y), want)
    if kind in ("pcm16_stereo", "f32", "ulaw_stereo"):
        for ch in (0, 1):
            y2, _ = lb.load(p, sr=None, mono=False)
            yc, _ = wav.read_wav(p, ms_channel=ch)
            np.testing.assert_array_equal(_as_float(yc), y2[ch])
    if kind == "pcm16":
        assert y.dtype == np.int16           # mono PCM16 stays int16: the /32768 happens on the GPU


def test_unreadable_file_raises_value_error(tmp_path):
    p = tmp_path / "broken.wav"
    p.write_bytes(b"not a wav file at all")
    with pytest.raises(ValueError, match="Could not load file"):
        wav.read_wav(str(p))
    with pytest.raises(ValueError, match="Could not load file"):
        wav.read_wav(str(tmp_path / "missing.wav"))


def test_cli_argument_validation(monkeypatch):
    import importlib
    sys.path.insert(0, ROOT)
    rp = importlib.import_module("run_predict")
    a = rp.parse_args(["--mode", "predict_dir", "--pretrained_model", "w.tar", "--data_dir", "d", "--bs", "64", "--num_workers", "3"])
    assert a["tr_bs_val"] == 64 and a["tr_num_workers"] == 3 and a["output_dir"] is None
    a = rp.parse_args(["--mode", "predict_csv", "--pretrained_model", "w.tar", "--csv_file", "f.csv", "--csv_deg", "deg"])
    assert a["data_dir"] == ""
    with pytest.raises(ValueError):
        rp.parse_args(["--mode", "predict_file", "--pretrained_model", "w.tar"])
    with pytest.raises(ValueError):
        rp.parse_args(["--mode", "predict_dir", "--pretrained_model", "w.tar"])
    with pytest.raises(ValueError):
        rp.parse_args(["--mode", "predict_csv", "--pretrained_model", "w.tar", "--csv_file", "f.csv"])
    with pytest.raises(NotImplementedError):
        rp.parse_args(["--mode", "train", "--pretrained_model", "w.tar"])


def test_shard_rows_partition_and_balance():
    rng = np.random.default_rng(0)
    w = rng.uniform(2, 30, size=513)
    for world in (1, 2, 4, 8):
        shards = nb_dist.shard_rows(w, world)
        allrows = np.sort(np.concatenate(shards))
        np.testing.assert_array_equal(allrows, np.arange(513))
        loads = np.array([w[s].sum() for s in shards])
        assert loads.max() - loads.min() <= w.max() + 1e-9
        assert all(np.all(np.diff(s) > 0) for s in shards if len(s) > 1)
    g = np.zeros((2, 3, 5), np.float32)
    g[0, :3] = 1.0; g[1, :2] = 2.0
    out = nb_dist.scatter_rows(g, [np.array([0, 2, 4]), np.array([1, 3])], 5)
    np.testing.assert_array_equal(out[:, 0], [1, 2, 1, 2, 1])


def test_two_rank_gloo_exchange(tmp_path):
    """world_size-2 run of the N>1 host path on CPU (gloo): shard, 'score', all-gather."""
    script = tmp_path / "w.py"
    script.write_text(
        "import os, sys, numpy as np\n"
        "sys.path.insert(0, %r)\n"
        "import torch.distributed as dist\n"
        "from nisqa_b200 import dist as D\n"
        "rank, world, _ = D.init_process_group(backend='gloo')\n"
        "w = np.random.default_rng(3).uniform(1, 9, size=37)\n"
        "shards = D.shard_rows(w, world)\n"
        "local = np.stack([np.full(5, float(i), np.float32) + np.arange(5, dtype=np.float32) / 10 for i in shards[rank]])\n"
        "full = D.all_gather_scores(local, shards, 37)\n"
        "ref = np.arange(37, dtype=np.float32)[:, None] + np.arange(5, dtype=np.float32)[None, :] / 10\n"
        "assert full.shape == (37, 5) and np.array_equal(full, ref), full\n"
        "dist.barrier(); dist.destroy_process_group()\n"
        "open(os.path.join(%r, 'ok%%d' %% rank), 'w').write('ok')\n" % (ROOT, str(tmp_path)))
    port = 29500 + (os.getpid() % 2000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()


def test_two_rank_error_is_raised_on_every_rank(tmp_path):
    """A per-file ValueError fires on the one rank that owns the row; the N>1 path exchanges (ok, message) before the
    score gather so that EVERY rank raises the reference's error instead of blocking in the collective."""
    script = tmp_path / "w.py"
    script.write_text(
        "import os, sys, numpy as np, pandas as pd\n"
        "sys.path.insert(0, %r)\n"
        "from nisqa_b200 import dist as D, NISQA_lib as NL\n"
        "rank, world, _ = D.init_process_group(backend='gloo')\n"
        "def fake_rows(engine, ds, rows, bs, nw):\n"
        "    if 5 in [int(r) for r in rows]:\n"
        "        raise ValueError('Could not load file c5.wav')\n"
        "    return np.zeros((len(rows), 1), np.float32)\n"
        "NL._predict_rows = fake_rows\n"
        "class Eng: n_out = 1\n"
        "class Ds:\n"
        "    df = pd.DataFrame({'deg': ['c%%d.wav' %% i for i in range(9)]})\n"
        "    def __len__(self): return 9\n"
        "    def file_path(self, i): return '/nonexistent/c%%d.wav' %% i\n"
        "try:\n"
        "    NL._predict_all(Eng(), Ds(), 4, 0)\n"
        "    msg = 'no error'\n"
        "except ValueError as e:\n"
        "    msg = str(e)\n"
        "open(os.path.join(%r, 'msg%%d' %% rank), 'w').write(msg)\n"
        "import torch.distributed as dist\n"
        "dist.barrier(); dist.destroy_process_group()\n" % (ROOT, str(tmp_path)))
    port = 31500 + (os.getpid() % 2000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (tmp_path / "msg0").read_text() == (tmp_path / "msg1").read_text() == "Could not load file c5.wav"


def test_double_ended_rows_pair_up_on_the_host(tmp_path):
    """NISQA_DE host logic without a GPU (stub engine): a dataset row becomes the clip pair (degraded, reference) in that
    order, ``ms_channel`` applies to the degraded file only (lib:2136-2154), the pair's score is row 2p of the engine's
    output, and a too-short reference raises the reference's error naming the DEGRADED file (lib:2187-2192)."""
    import pandas as pd
    from nisqa_b200 import NISQA_lib as NL, engine as E, wav
    rng = np.random.default_rng(5)
    st = rng.integers(-3000, 3000, (4000, 2)).astype(np.int16)
    wav.write_wav_pcm16(str(tmp_path / "d0.wav"), st, 16000)                       # stereo degraded file
    wav.write_wav_pcm16(str(tmp_path / "r0.wav"), st, 16000)                       # stereo reference: always the mono mix
    wav.write_wav_pcm16(str(tmp_path / "d1.wav"), rng.integers(-3000, 3000, 5000).astype(np.int16), 16000)
    wav.write_wav_pcm16(str(tmp_path / "r1.wav"), rng.integers(-3000, 3000, 100).astype(np.int16), 16000)      # too short
    df = pd.DataFrame({"deg": ["d0.wav", "d1.wav"], "ref": ["r0.wav", "r1.wav"]})
    ds = NL.SpeechQualityDataset(df, data_dir=str(tmp_path), filename_column="deg", mos_column="predict_only",
                                 ms_sr=None, ms_channel=1, double_ended=True, filename_column_ref="ref",
                                 seg_length=15, ms_hop_length=0.01)
    with pytest.raises(KeyError):
        NL.SpeechQualityDataset(df, data_dir=str(tmp_path), filename_column="deg", mos_column="predict_only",
                                double_ended=True, filename_column_ref=None)       # predict_file / predict_dir (lib:2133)

    class StubEngine(object):
        n_out = 1
        seen = []

        def submit_pcm(self, clips, srs):
            self.seen.append([c.copy() for c in clips])
            n = len(clips)
            scores = np.full((n, 1), np.nan, np.float32)
            status = np.zeros(n, np.int32)
            for i, c in enumerate(clips):
                if c.shape[0] < 15 * 160:
                    status[i] = E.CLIP_TOO_SHORT
            scores[0::2, 0] = [float(np.abs(c.astype(np.float64)).sum() % 97) for c in clips[0::2]]
            return (None, scores, np.full(n, 3, np.int32), status)

        def wait(self, handle):
            return handle[1], handle[2], handle[3]

        def drain(self):
            pass

    eng = StubEngine()
    out = NL._predict_rows(eng, ds, np.array([0]), 4, 0)
    deg, ref = eng.seen[0]
    # channel pick on the degraded file (int16 -> float32 / 32768 because its partner in the call is float32)
    assert deg.dtype == np.float32 and np.array_equal(deg, st[:, 1].astype(np.float32) / np.float32(32768.0))
    mix = (st.astype(np.float32) / np.float32(32768.0)).mean(axis=1, dtype=np.float32)
    assert ref.dtype == np.float32 and np.allclose(ref, mix, atol=1e-7)            # mono mix on the reference
    assert out.shape == (1, 1) and np.isfinite(out[0, 0])
    with pytest.raises(ValueError) as ei:
        NL._predict_rows(eng, ds, np.array([0, 1]), 4, 0)
    assert "Sample too short" in str(ei.value) and str(ei.value).endswith("d1.wav")


def test_orderly_multi_rank_shutdown(tmp_path):
    """dist.shutdown (what run_predict.py calls last): barrier, engine close, barrier, process group destroyed - on
    two gloo ranks, and a no-op in a single process."""
    from nisqa_b200 import dist as D
    D.shutdown(None)                                             # single process: nothing to do
    script = tmp_path / "w.py"
    script.write_text(
        "import os, sys\n"
        "sys.path.insert(0, %r)\n"
        "import torch.distributed as dist\n"
        "from nisqa_b200 import dist as D\n"
        "rank, world, _ = D.init_process_group(backend='gloo')\n"
        "class Eng:\n"
        "    closed = False\n"
        "    def close(self): self.closed = True\n"
        "e = Eng(); D.shutdown(e)\n"
        "assert e.closed and not dist.is_initialized()\n"
        "open(os.path.join(%r, 'done%%d' %% rank), 'w').write('ok')\n" % (ROOT, str(tmp_path)))
    port = 33500 + (os.getpid() % 2000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert (tmp_path / "done0").exists() and (tmp_path / "done1").exists()


@pytest.mark.parametrize("kind", ["pcm16", "pcm16_stereo", "pcm24", "pcm32", "f32", "f64", "u8", "ext16", "alaw", "ulaw_stereo"])
def test_native_wav_reader_matches_oracle_loader(tmp_path, kind, built_lib):
    """csrc/wavio.cpp (nisqa_wav_probe / nisqa_wav_decode, host-only entry points of the C-ABI)."""
    rng = np.random.default_rng(2)
    p = str(tmp_path / (kind + ".wav"))
    n = 20011
    if kind in ("pcm16", "ext16"):
        _write_pcm(p, rng.integers(-32768, 32767, n).astype("<i2").tobytes(), 1, 1, 16000, 16, extensible=(kind == "ext16"))
    elif kind == "pcm16_stereo":
        _write_pcm(p, rng.integers(-32768, 32767, (n, 3)).astype("<i2").tobytes(), 1, 3, 44100, 16)
    elif kind == "pcm24":
        b = bytearray()
        for x in rng.integers(-(1 << 23), (1 << 23) - 1, n):
            b += int(x & 0xFFFFFF).to_bytes(3, "little")
        _write_pcm(p, bytes(b), 1, 1, 48000, 24)
    elif kind == "pcm32":
        _write_pcm(p, rng.integers(-(1 << 31), (1 << 31) - 1, n).astype("<i4").tobytes(), 1, 1, 48000, 32)
    elif kind == "alaw":
        _write_pcm(p, np.arange(n, dtype=np.int64).astype(np.uint8).tobytes(), 6, 1, 8000, 8)          # every code
    elif kind == "ulaw_stereo":
        _write_pcm(p, rng.integers(0, 256, (n, 2)).astype(np.uint8).tobytes(), 7, 2, 8000, 8)
    elif kind == "f32":
        _write_pcm(p, rng.standard_normal((n, 2)).astype("<f4").tobytes(), 3, 2, 22050, 32)
    elif kind == "f64":
        _write_pcm(p, rng.standard_normal(n).astype("<f8").tobytes(), 3, 1, 8000, 64)
    else:
        _write_pcm(p, rng.integers(0, 255, n).astype(np.uint8).tobytes(), 1, 1, 8000, 8)
    y_ref, sr_ref = lb.load(p, sr=None)
    y, sr = wav.read_wav_native(p)
    assert sr == sr_ref
    np.testing.assert_array_equal(_as_float(y), y_ref)
    y2, _ = lb.load(p, sr=None, mono=False)
    if y2.ndim > 1:
        for ch in range(y2.shape[0]):
            yc, _ = wav.read_wav_native(p, ms_channel=ch)
            np.testing.assert_array_equal(_as_float(yc), y2[ch])
    if kind == "pcm16":
        assert y.dtype == np.int16


def test_native_wav_reader_errors(tmp_path, built_lib):
    (tmp_path / "bad.wav").write_bytes(b"RIFFxxxxWAVEjunk")
    for name in ("bad.wav", "missing.wav"):
        with pytest.raises(ValueError, match="Could not load file"):
            wav.read_wav_native(str(tmp_path / name))


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the oracle port on the host cores) prints the contract's JSON line."""
    import json
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["unit"] == "clips/s" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["value"] == line["value"]


def test_bench_rooflines_replay_recorded_line():
    """bench.build_rooflines is a pure function of the per-kernel CUDA-event times: replaying a fixed bench line
    (tests/golden/bench_line_replay.json: synthetic kernel times, roofline entries computed from the algorithmic FLOP /
    byte counts) must reproduce its roofline entries, name the same dominant kernel, and carry the attention-FLOP
    roofline of SURVEY 8d(iii)."""
    import importlib.util
    import json
    spec = importlib.util.spec_from_file_location("nisqa_bench", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    rec = json.load(open(os.path.join(GOLDEN, "bench_line_replay.json")))
    peaks = {"hbm_gbs": rec["roofline"]["peak"], "bf16_tflops_sustained": rec["roofline_kernels"]["conv4"]["peak"],
             "bf16_tflops": 0.0, "source": "measured (MEASURED_PEAKS.json)"}
    traffic = {k: v["traffic"] for k, v in rec["roofline_kernels"].items()}
    roofs, dom = bench.build_rooflines(rec["kernel_ms_per_step"], peaks, rec["clocks"]["sm_max_mhz"], traffic, 480000)
    assert dom["kernel"] == rec["roofline"]["kernel"] == "frontend"
    fe_got, fe_want = roofs["frontend"], rec["roofline_kernels"]["frontend"]
    # round 2: the front-end is reported against the fp32 issue peak (`frac` = the recorded frac_fp32); the HBM view
    # the r01e line carried as `achieved` / `frac` is kept as hbm_gbs / hbm_frac
    assert fe_got["bound"] == "fp32-issue" and fe_got["unit"] == "TFLOP/s"
    assert abs(fe_got["achieved"] - fe_want["fft_tflops"]) <= 1e-9 and abs(fe_got["frac"] - fe_want["fft_tflops"] / fe_got["peak"]) <= 1e-12
    assert abs(fe_got["hbm_gbs"] - fe_want["achieved"]) <= 1e-6 and abs(fe_got["hbm_frac"] - fe_want["frac"]) <= 1e-12
    for k, want in rec["roofline_kernels"].items():
        if k == "frontend":
            continue
        got = roofs[k]
        for field in ("bound", "unit", "traffic"):
            assert got[field] == want[field], (k, field)
        for field in ("achieved", "peak", "frac", "kernel_ms"):
            assert abs(got[field] - want[field]) <= 1e-9 * max(1.0, abs(want[field])), (k, field)
        if "frac_executed" in want:
            assert abs(got["frac_executed"] - want["frac_executed"]) <= 1e-12
    for key in ("bound", "achieved", "peak", "unit", "frac", "traffic"):           # the contract's roofline object
        assert key in dom
    sa = roofs["sa_layer"]
    assert sa["unit"] == "TFLOP/s" and 0.0 < sa["frac"] < 1.0
    assert abs(sa["achieved"] - 31.2e6 * 64 / (rec["kernel_ms_per_step"]["sa_layer"] / 1e3) / 1e12) <= 1e-9
