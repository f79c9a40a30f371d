"""Recordings scored as a timeline of overlapping windows: nisqa_window_counts, nisqa_predict_device_windows,
Scorer.windows and run_predict.py --window_s / --window_hop_s.  CPU part: the window arithmetic against a NumPy
restatement of its definition, the refusals and the ABI.  GPU part: every window bit for bit what Scorer.__call__ gives
the same window cut out as a clip (int16 / float32, channel pick and mix, 22.05 / 48 / 96 kHz, ms_sr, several passes, a
batch against each recording alone), a sample against the oracle, and the CLI."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import resample as RS
from nisqa_b200 import synth, wav
from nisqa_b200.scorer import Scorer, window_geometry, window_times

gpu = pytest.mark.gpu
CKPTS = ["nisqa.tar", "nisqa_mos_only.tar", "nisqa_tts.tar"]


def _args(ckpt, **over):
    a = E.load_checkpoint(os.path.join(WEIGHTS, ckpt))[0]
    a.update(over)
    return a


def _cpu_scorer(ckpt, **over):
    s = Scorer.__new__(Scorer)
    s._configure(_args(ckpt, **over), torch.device("cpu"))
    return s


def _restate(args, T, rate, window_s, window_hop_s):
    """the definition: (W, H, window starts, ends, segment counts, statuses) of a recording of T samples at the model rate"""
    hop = int(rate * args["ms_hop_length"])
    W = int(round(window_s * rate))
    H = max(1, int(round(window_hop_s * rate / hop))) * hop
    K = 1 if T <= W else 1 + -(-(T - W) // H)
    k = np.arange(K, dtype=np.int64)
    start, end = k * H, np.minimum(k * H + W, T)
    n_wins = 1 + (end - start) // hop - (args["ms_seg_length"] - 1)
    sh = args["ms_seg_hop_length"]
    n_seg = np.where(n_wins < 1, 0, -(-n_wins // sh))
    status = np.where(n_wins < 1, E.CLIP_TOO_SHORT, np.where(n_seg > args["ms_max_segments"], E.CLIP_TOO_LONG, E.CLIP_OK))
    return W, H, start, end, n_seg, status


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("rate", [8000, 22050, 44100, 48000, 96000])
def test_window_counts_follow_the_definition(built_lib, rate):
    args = _args("nisqa.tar")
    cfg = E.config_from_args(args)
    hop = int(rate * args["ms_hop_length"])
    for window_s, window_hop_s in ((10.0, 10.0), (10.0, 5.0), (10.0, 1.0), (10.0, 0.01), (3.0, 0.37), (2.5, 2.4)):
        W, hf = window_geometry(args, rate, window_s, window_hop_s)
        for T in (1, hop * 3, W - 1, W, W + 1, 3 * W + 7, int(61.3 * rate)):
            W_, H, start, end, n_seg, status = _restate(args, T, rate, window_s, window_hop_s)
            assert (W, hf * hop) == (W_, H)
            got_seg, got_st = E.window_counts(cfg, T, rate, W, hf)
            np.testing.assert_array_equal(got_seg, n_seg, err_msg=str((rate, window_s, window_hop_s, T)))
            np.testing.assert_array_equal(got_st, status)
            assert np.all(status[:-1] == E.CLIP_OK)          # only the last window can be too short
            # each window alone: nisqa_segment_counts of the cut clip
            for k in {0, len(start) - 1}:
                assert E.segment_counts(cfg, int(end[k] - start[k]), rate)[1:] == (n_seg[k], status[k])
            t0, t1 = window_times(T, W, H, rate)
            np.testing.assert_array_equal(t0, start / rate)
            np.testing.assert_array_equal(t1, end / rate)


def test_window_counts_of_a_two_hour_recording(built_lib):
    args = _args("nisqa.tar")
    cfg = E.config_from_args(args)
    T = 2 * 3600 * 48000 + 123
    for window_hop_s in (1.0, 0.01):               # 1 s, and the hop of one mel frame
        W, H, start, end, n_seg, status = _restate(args, T, 48000, 10.0, window_hop_s)
        got_seg, got_st = E.window_counts(cfg, T, 48000, W, H // 480)
        assert got_seg.shape[0] == start.shape[0] == 1 + -(-(T - W) // H)
        np.testing.assert_array_equal(got_seg, n_seg)
        np.testing.assert_array_equal(got_st, status)


def test_refusals_name_the_argument(built_lib):
    x = torch.zeros(48000 * 70, dtype=torch.int16)
    sc = _cpu_scorer("nisqa.tar")
    with pytest.raises(ValueError, match="window_hop_s"):
        sc.windows(x, 48000, 5.0, 6.0)
    with pytest.raises(ValueError, match="window_s"):
        sc.windows(x, 48000, 60.0, 1.0)            # 1497 segments > ms_max_segments 1300
    with pytest.raises(ValueError, match="window_s"):
        sc.windows(x, 48000, 0.1, 0.1)             # not one segment
    for bad in (-1.0, 0, float("nan"), True, "10"):
        with pytest.raises(ValueError, match="window_s"):
            sc.windows(x, 48000, bad, 1.0)
        with pytest.raises(ValueError, match="window_hop_s"):
            sc.windows(x, 48000, 10.0, bad)
    with pytest.raises(ValueError, match="channel|lengths"):
        sc.windows(x[None], 48000, 10.0, 1.0, lengths=[0])
    de = _cpu_scorer("nisqa_mos_only.tar")
    de.double_ended = True                         # (what _configure sets for a NISQA_DE checkpoint)
    with pytest.raises(ValueError, match="NISQA_DE"):
        de.windows(x, 48000, 10.0, 1.0)
    cfg = E.config_from_args(_args("nisqa.tar"))
    k = ctypes.c_int64()
    lib = E.load_library()
    for window, hf in ((480000, 1001), (480000, 0), (48000 * 60, 100), (0, 1)):
        assert lib.nisqa_window_counts(ctypes.byref(cfg), 48000 * 70, 48000, window, hf, ctypes.byref(k), None, None, 0) \
            == -1


def test_cli_refusals_name_the_argument(monkeypatch):
    import run_predict
    from nisqa_b200.NISQA_model import nisqaModel
    base = ["--mode", "predict_dir", "--pretrained_model", "x.tar", "--data_dir", "d"]
    with pytest.raises(ValueError, match="window_hop_s"):
        run_predict.parse_args(base + ["--window_s", "10"])
    with pytest.raises(ValueError, match="window_s"):
        run_predict.parse_args(base + ["--window_hop_s", "1"])
    with pytest.raises(ValueError, match="window_s"):
        run_predict.parse_args(base + ["--window_s", "-2", "--window_hop_s", "1"])
    a = run_predict.parse_args(base + ["--window_s", "10", "--window_hop_s", "2.5"])
    assert (a["window_s"], a["window_hop_s"]) == (10.0, 2.5)
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("LOCAL_RANK", "0")
    with pytest.raises(ValueError, match="window_s"):
        nisqaModel({"mode": "predict_csv", "window_s": 10.0, "window_hop_s": 1.0, "csv_file": "/nonexistent.csv"})


def test_header_exports_and_binding_agree(built_lib):
    header = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    lib = E.load_library()
    for sym in ("nisqa_window_counts", "nisqa_predict_device_windows"):
        assert sym + "(" in header and sym in E.EXPORTS and hasattr(lib, sym)
    assert len(lib.nisqa_predict_device_windows.argtypes) == 10
    assert len(lib.nisqa_window_counts.argtypes) == 9
    assert "#define NISQA_B200_ABI_VERSION 4" in header


# ------------------------------------------------------------------ GPU
_CACHE = {}


def _recording(sec, sr=48000, seed=0):
    """int16 speech-like recording; ten minutes are built from a 61 s one with a gain that changes every second"""
    key = (sec, sr, seed)
    if key not in _CACHE:
        if sec <= 61:
            _CACHE[key] = synth.synth_speech_pcm16(2000 + seed, sec, sr)[:int(sec * sr)]
        else:
            base = _recording(61.0, sr, seed).astype(np.float32)
            n = int(sec * sr)
            x = np.resize(base, n)
            g = np.repeat(np.random.default_rng(seed).uniform(0.05, 1.0, n // sr + 1), sr)[:n]
            _CACHE[key] = np.clip(x * g, -32768, 32767).astype(np.int16)
    return _CACHE[key]


_SCORERS = {}


def _scorer(ckpt, **over):
    key = (ckpt, tuple(sorted(over.items())))
    if key not in _SCORERS:
        _SCORERS[key] = Scorer(os.path.join(WEIGHTS, ckpt), **over)
    return _SCORERS[key]


def _cut_scores(sc, x, T, W, H, rate, channel=None):
    """Scorer.__call__ on the windows of x ([T] or [C, T] CUDA tensor) cut out as clips (an overlapping strided view),
    the too-short last window left out"""
    K = 1 if T <= W else 1 + -(-(T - W) // H)
    span = (K - 1) * H + W
    xp = torch.zeros(x.shape[:-1] + (span,), dtype=x.dtype, device=x.device)
    xp[..., :T] = x[..., :T]
    view = xp.as_strided((K, W), (H, 1)) if x.dim() == 1 else xp.as_strided((K, x.shape[0], W), (H, span, 1))
    lens = [min(W, T - k * H) for k in range(K)]
    n_ok = K
    if E.segment_counts(sc.cfg, lens[-1], rate)[2] != E.CLIP_OK:
        n_ok -= 1
    if n_ok == 0:
        return np.zeros((0, len(sc.columns)), np.float32)
    return sc(view[:n_ok], rate, lengths=lens[:n_ok], channel=channel).cpu().numpy()


def _check_against_cut(sc, x, rate, window_s, window_hop_s, channel=None, cut_sc=None, cut_x=None, cut_rate=None):
    T = x.shape[-1]
    res = sc.windows(x if x.dim() == 1 else x[None], rate, window_s, window_hop_s, channel=channel)   # ([C, T]: one recording)
    got = res.scores.cpu().numpy()
    rate_m = cut_rate or rate
    W, hf = window_geometry(sc.args, rate_m, window_s, window_hop_s)
    H = hf * int(rate_m * sc.args["ms_hop_length"])
    Tm = (cut_x if cut_x is not None else x).shape[-1]
    want = _cut_scores(cut_sc or sc, cut_x if cut_x is not None else x, Tm, W, H, rate_m, channel)
    assert res.counts == [got.shape[0]]
    np.testing.assert_array_equal(got[:want.shape[0]], want, err_msg=str((rate, window_s, window_hop_s, channel)))
    assert np.isnan(got[want.shape[0]:]).all()
    assert np.all(res.status[want.shape[0]:] == E.CLIP_TOO_SHORT) and np.all(res.status[:want.shape[0]] == E.CLIP_OK)
    _, _, start, end, n_seg, status = _restate(sc.args, Tm, rate_m, window_s, window_hop_s)
    np.testing.assert_array_equal(res.t_start, start / rate_m)
    np.testing.assert_array_equal(res.t_end, end / rate_m)
    np.testing.assert_array_equal(res.n_segments, n_seg)
    return res


@gpu
@pytest.mark.parametrize("ckpt", CKPTS)
def test_windows_equal_the_cut_clips_bit_for_bit(built_lib, ckpt):
    sc = _scorer(ckpt)
    for sec in (3.0, 61.0, 600.0):
        x = torch.from_numpy(_recording(sec)).cuda()
        for window_hop_s in (10.0, 5.0, 1.0):
            _check_against_cut(sc, x, 48000, 10.0, window_hop_s)


@gpu
def test_other_inputs_equal_the_cut_clips(built_lib):
    sc = _scorer("nisqa.tar")
    st = np.stack([_recording(25.0, seed=1), _recording(25.0, seed=2)]).astype(np.float32) / 32768.0
    xs = torch.from_numpy(st).cuda()                                          # float32 stereo [2, T]
    for channel in (1, None):
        _check_against_cut(sc, xs, 48000, 10.0, 1.0, channel=channel)
    x22 = torch.from_numpy(_recording(25.0, 22050, seed=3)).cuda()            # 1 s is 100.2 frames of 220 samples
    _check_against_cut(sc, x22, 22050, 10.0, 1.0)
    x96 = torch.from_numpy(_recording(14.0, 96000, seed=4)).cuda()            # 1920-sample windows: frontend_kernel
    _check_against_cut(sc, x96, 96000, 10.0, 1.0)
    _check_against_cut(sc, x96.float() / 32768.0, 96000, 10.0, 3.33)          # an odd hop in frames: both pairings


@gpu
def test_ms_sr_passes_batches_and_short_last_window(built_lib):
    # ms_sr: the recording converted whole, then cut, equals cutting the host-converted recording
    x48 = _recording(25.0, 48000, seed=5)
    sr16 = _scorer("nisqa_mos_only.tar", ms_sr=16000)
    y16 = torch.from_numpy(RS.resample(x48, 48000, 16000)).cuda()
    _check_against_cut(sr16, torch.from_numpy(x48).cuda(), 48000, 10.0, 1.0, cut_sc=_scorer("nisqa_mos_only.tar"),
                       cut_x=y16, cut_rate=16000)
    # several passes equal one pass; a recording alone equals it in a batch
    sc = _scorer("nisqa.tar")
    small = _scorer("nisqa.tar", b200_max_chunk_segments=300)
    recs = [_recording(3.0, seed=6), _recording(61.0, seed=7), _recording(25.0, seed=8)]
    T = max(r.shape[0] for r in recs)
    xb = np.zeros((len(recs), T), np.int16)
    for i, r in enumerate(recs):
        xb[i, :r.shape[0]] = r
    xb = torch.from_numpy(xb).cuda()
    lens = [r.shape[0] for r in recs]
    one = sc.windows(xb, 48000, 10.0, 1.0, lengths=lens)
    many = small.windows(xb, 48000, 10.0, 1.0, lengths=lens)
    torch.cuda.synchronize()
    assert small.engine.lib.nisqa_stage_dump(small.engine.h, E.STAGE_MEL_DB, None, 0) < 0    # (it ran in passes)
    np.testing.assert_array_equal(one.scores.cpu().numpy(), many.scores.cpu().numpy())
    r0 = 0
    for i, n in enumerate(one.counts):
        alone = sc.windows(xb[i, :lens[i]], 48000, 10.0, 1.0)
        np.testing.assert_array_equal(alone.scores.cpu().numpy(), one.scores[r0:r0 + n].cpu().numpy())
        np.testing.assert_array_equal(alone.t_start, one.t_start[r0:r0 + n])
        r0 += n
    # a too-short last window: NaN and CLIP_TOO_SHORT, never an error
    xs = torch.from_numpy(_recording(20.05, seed=9)).cuda()
    res = _check_against_cut(sc, xs, 48000, 10.0, 10.0)
    assert res.status.tolist() == [E.CLIP_OK, E.CLIP_OK, E.CLIP_TOO_SHORT] and np.isnan(res.scores[2].cpu().numpy()).all()


@gpu
def test_sample_of_windows_against_the_oracle(built_lib):
    from oracle import nisqa_oracle as O
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    sc = _scorer("nisqa.tar")
    x = _recording(61.0, seed=10)
    res = sc.windows(torch.from_numpy(x).cuda(), 48000, 10.0, 5.0)
    got = res.scores.cpu().numpy()
    for k in (0, 6, len(got) - 1):
        a, b = int(round(res.t_start[k] * 48000)), int(round(res.t_end[k] * 48000))
        ref, n_seg, st = O.predict_pcm(args, sd, x[a:b].astype(np.float32) / 32768.0, 48000)
        assert st == 0 and n_seg == res.n_segments[k]
        np.testing.assert_allclose(got[k], ref, atol=1e-4, rtol=0)


@gpu
def test_cli_writes_windows_csv(built_lib, tmp_path):
    import pandas as pd
    import run_predict
    from nisqa_b200.NISQA_model import nisqaModel
    d = tmp_path / "wavs"
    d.mkdir()
    wav.write_wav_pcm16(str(d / "long.wav"), np.resize(_recording(61.0, seed=11), 48000 * 75), 48000)   # > ms_max_segments
    wav.write_wav_pcm16(str(d / "short.wav"), _recording(5.0, seed=12), 48000)
    out = tmp_path / "out"
    out.mkdir()
    argv = ["--mode", "predict_dir", "--pretrained_model", os.path.join(WEIGHTS, "nisqa.tar"), "--data_dir", str(d),
            "--output_dir", str(out), "--window_s", "10", "--window_hop_s", "5"]
    nisqaModel(run_predict.parse_args(argv)).predict()
    df = pd.read_csv(out / "NISQA_windows.csv")
    sc = _scorer("nisqa.tar")
    assert list(df.columns) == ["deg", "t_start", "t_end", "n_segments"] + sc.columns
    assert sorted(set(df["deg"])) == ["long.wav", "short.wav"]
    for f in ("long.wav", "short.wav"):
        y, sr = wav.read_wav(str(d / f), None)
        res = sc.windows(torch.from_numpy(y).cuda(), sr, 10.0, 5.0)
        rows = df[df["deg"] == f]
        assert len(rows) == res.counts[0] == (14 if f == "long.wav" else 1)
        np.testing.assert_array_equal(rows["t_start"].to_numpy(), res.t_start)
        np.testing.assert_array_equal(rows["t_end"].to_numpy(), res.t_end)
        np.testing.assert_array_equal(rows["n_segments"].to_numpy(), res.n_segments)
        np.testing.assert_array_equal(rows[sc.columns].to_numpy().astype(np.float32), res.scores.cpu().numpy())
