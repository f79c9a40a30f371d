"""Double-ended (NISQA_DE) recordings scored as a timeline of window pairs: nisqa_window_pair_counts,
nisqa_predict_device_window_pairs, Scorer.windows(..., reference=...) and run_predict.py --window_s with --csv_ref.
CPU part: the pair arithmetic against a NumPy restatement of its definition, the refusals and the ABI.  GPU part: every
pair bit for bit what Scorer.__call__ gives the two windows cut out as clips (int16 / float32, channel pick and mix,
16 / 22.05 / 48 kHz, odd and even hops, margins with clipped and empty reference windows, ms_sr), several passes, a batch
against each pair alone, the stream contract, a sample against the oracle, and the CLI."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import resample as RS
from nisqa_b200 import synth, wav
from nisqa_b200.scorer import Scorer, WindowPairs, Windows, window_geometry

gpu = pytest.mark.gpu
# the shape of the reference's train_nisqa_double_ended.yaml (AdaptCNN + self-attention, cosine, hard), and StandardCNN +
# a bidirectional LSTM td with Luong soft alignment and a fusion Linear
VARIANTS = ["de_cosine_hard", "std_fc20_lstm128bi_luong_soft_fd128"]


def _checkpoint(name):
    if name in VARIANTS[:1]:
        from oracle import variants as V
        bargs, bsd = E.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
        return V.de_checkpoint(name, bargs, bsd)
    from oracle import de_arch_variants as V
    base = V.DE_ARCH_VARIANTS[name][0]
    bargs, bsd = E.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.de_arch_checkpoint(name, bargs, bsd)


def _host_scorer(args):
    s = Scorer.__new__(Scorer)
    s._configure(args, torch.device("cpu"))
    s.engine = None
    return s


def _restate(args, T, T_ref, rate, window_s, window_hop_s, margin_s):
    """the definition: (W, H, M, degraded starts / ends, reference starts / ends, segment counts and statuses of both)"""
    hop = int(rate * args["ms_hop_length"])
    W = int(round(window_s * rate))
    H = max(1, int(round(window_hop_s * rate / hop))) * hop
    M = int(round(margin_s * rate / hop)) * hop
    K = 1 if T <= W else 1 + -(-(T - W) // H)
    k = np.arange(K, dtype=np.int64)
    d0, d1 = k * H, np.minimum(k * H + W, T)
    r0 = np.maximum(0, k * H - M)
    r1 = np.maximum(r0, np.minimum(T_ref, k * H + W + M))

    def counts(n):
        n_wins = np.where(n < 1, 0, 1 + n // hop - (args["ms_seg_length"] - 1))
        n_seg = np.where(n_wins < 1, 0, -(-n_wins // args["ms_seg_hop_length"]))
        st = np.where(n_wins < 1, E.CLIP_TOO_SHORT, np.where(n_seg > args["ms_max_segments"], E.CLIP_TOO_LONG, E.CLIP_OK))
        return n_seg, st
    return (W, H, M, d0, d1, r0, r1) + counts(d1 - d0) + counts(r1 - r0)


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("rate", [8000, 16000, 22050, 44100, 48000, 96000])
def test_pair_counts_follow_the_definition(built_lib, rate):
    args = _checkpoint("de_cosine_hard")[0]
    cfg = E.config_from_args(args)
    hop = int(rate * args["ms_hop_length"])
    for window_s, window_hop_s in ((10.0, 5.0), (10.0, 1.0), (3.0, 0.37)):
        W, hf = window_geometry(args, rate, window_s, window_hop_s)
        H = hf * hop
        for margin_frames in (0, 1, hf + 3):                     # none, one hop, more than the window hop
            M = margin_frames * hop
            for T in (W - 1, W, 3 * W + 7, int(31.3 * rate)):
                for T_ref in (1, M // 2 + 1, T // 3, T, T + 5 * W + 11):    # shorter than M, shorter, equal, longer
                    W_, H_, M_, d0, d1, r0, r1, ns, st, rns, rst = _restate(args, T, T_ref, rate, window_s, window_hop_s,
                                                                            M / rate)
                    assert (W_, H_, M_) == (W, H, M)
                    got = E.window_pair_counts(cfg, T, T_ref, rate, W, hf, margin_frames)
                    what = str((rate, window_s, window_hop_s, margin_frames, T, T_ref))
                    for g, w in zip(got, (ns, st, rns, rst)):
                        np.testing.assert_array_equal(g, w, err_msg=what)
                    # the degraded windows are those of nisqa_window_counts
                    for g, w in zip(got[:2], E.window_counts(cfg, T, rate, W, hf)):
                        np.testing.assert_array_equal(g, w)
                    # each reference window alone: nisqa_segment_counts of the cut clip
                    for k in {0, len(r0) - 1}:
                        assert E.segment_counts(cfg, int(r1[k] - r0[k]), rate)[1:] == (rns[k], rst[k])


def test_pair_counts_of_a_two_hour_pair(built_lib):
    args = _checkpoint("de_cosine_hard")[0]
    cfg = E.config_from_args(args)
    T, T_ref = 2 * 3600 * 48000 + 123, 2 * 3600 * 48000 - 48000 * 17
    for window_hop_s, margin_s in ((1.0, 0.5), (0.01, 0.0)):
        _, H, M, d0, _, _, _, ns, st, rns, rst = _restate(args, T, T_ref, 48000, 10.0, window_hop_s, margin_s)
        got = E.window_pair_counts(cfg, T, T_ref, 48000, 480000, H // 480, M // 480)
        assert got[0].shape[0] == d0.shape[0] == 1 + -(-(T - 480000) // H)
        for g, w in zip(got, (ns, st, rns, rst)):
            np.testing.assert_array_equal(g, w)
        assert rst[-1] == E.CLIP_TOO_SHORT                          # the reference ends 17 s before the recording


def test_refusals_name_the_argument(built_lib):
    de = _host_scorer(_checkpoint("de_cosine_hard")[0])
    se = _host_scorer(E.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))[0])
    x = torch.zeros(48000 * 70, dtype=torch.int16)
    r = torch.zeros(48000 * 65, dtype=torch.int16)
    # unchanged: a DE checkpoint without a reference
    with pytest.raises(ValueError, match="NISQA_DE"):
        de.windows(x, 48000, 10.0, 1.0)
    with pytest.raises(ValueError, match="reference"):
        se.windows(x, 48000, 10.0, 1.0, reference=r)
    with pytest.raises(ValueError, match="reference_margin_s"):
        se.windows(x, 48000, 10.0, 1.0, reference_margin_s=0.5)             # a margin without a reference
    with pytest.raises(ValueError, match="reference_margin_s"):
        de.windows(x, 48000, 10.0, 1.0, reference_margin_s=0.5)
    for bad in (-0.5, float("nan"), True, "1", None):
        with pytest.raises(ValueError, match="reference_margin_s"):
            de.windows(x, 48000, 10.0, 1.0, reference=r, reference_margin_s=bad)
    with pytest.raises(ValueError, match="reference_margin_s"):
        de.windows(x, 48000, 10.0, 1.0, reference=r, reference_margin_s=25.0)   # 60 s reference windows: > 1300 segments
    with pytest.raises(ValueError, match="reference_sample_rate"):
        de.windows(x, 48000, 10.0, 1.0, reference=r, reference_sample_rate=16000)
    with pytest.raises(ValueError, match="reference"):
        de.windows(x, 48000, 10.0, 1.0, reference=torch.zeros((2, 48000 * 65), dtype=torch.int16))
    with pytest.raises(ValueError, match="window_hop_s"):
        de.windows(x, 48000, 5.0, 6.0, reference=r)
    with pytest.raises(ValueError, match="window_s"):
        de.windows(x, 48000, 60.0, 1.0, reference=r)
    with pytest.raises(ValueError, match="reference_lengths"):
        de.windows(x, 48000, 10.0, 1.0, reference=r[None], reference_lengths=[0])
    # with ms_sr the reference may come at another rate (both converted whole)
    ms = _host_scorer(dict(_checkpoint("de_cosine_hard")[0], ms_sr=16000))
    with pytest.raises(ValueError, match="reference_margin_s"):
        ms.windows(x, 48000, 10.0, 1.0, reference=r, reference_sample_rate=22050, reference_margin_s=-1)
    cfg = E.config_from_args(_checkpoint("de_cosine_hard")[0])
    lib = E.load_library()
    k = ctypes.c_int64()
    for T, T_ref, window, hf, mf in ((48000 * 70, 48000, 480000, 1001, 0), (48000 * 70, 48000, 480000, 100, -1),
                                     (48000 * 70, 48000, 480000, 100, 3000), (48000 * 70, 0, 480000, 100, 0),
                                     (0, 48000, 480000, 100, 0)):
        assert lib.nisqa_window_pair_counts(ctypes.byref(cfg), T, T_ref, 48000, window, hf, mf, ctypes.byref(k), None,
                                            None, None, None, 0) == -1


def test_cli_refusals_name_the_argument():
    import run_predict
    base = ["--mode", "predict_csv", "--pretrained_model", "x.tar", "--csv_file", "f.csv", "--csv_deg", "deg"]
    with pytest.raises(ValueError, match="reference_margin_s"):
        run_predict.parse_args(base + ["--reference_margin_s", "0.5"])
    with pytest.raises(ValueError, match="reference_margin_s"):
        run_predict.parse_args(base + ["--window_s", "10", "--window_hop_s", "1", "--reference_margin_s", "-1"])
    a = run_predict.parse_args(base + ["--csv_ref", "ref", "--window_s", "10", "--window_hop_s", "1",
                                       "--reference_margin_s", "0.5"])
    assert (a["csv_ref"], a["reference_margin_s"]) == ("ref", 0.5)
    a = run_predict.parse_args(base)
    assert "csv_ref" not in a and "reference_margin_s" not in a        # (a checkpoint's csv_ref stays)


def test_header_exports_and_binding_agree(built_lib):
    header = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    lib = E.load_library()
    for sym in ("nisqa_window_pair_counts", "nisqa_predict_device_window_pairs"):
        assert sym + "(" in header and sym in E.EXPORTS and hasattr(lib, sym)
    assert len(lib.nisqa_predict_device_window_pairs.argtypes) == 14
    assert len(lib.nisqa_window_pair_counts.argtypes) == 13
    assert Windows._fields == ("scores", "counts", "t_start", "t_end", "n_segments", "status")
    assert WindowPairs._fields == Windows._fields + ("ref_t_start", "ref_t_end", "ref_n_segments", "ref_status")
    assert "#define NISQA_B200_ABI_VERSION 4" in header


# ------------------------------------------------------------------ GPU
_SCORERS = {}


def _scorer(name, tmp_path_factory, **over):
    key = (name, tuple(sorted(over.items())))
    if key not in _SCORERS:
        path = tmp_path_factory.getbasetemp() / (name + ".tar")
        if not path.exists():
            args, sd = _checkpoint(name)
            torch.save({"args": args, "model_state_dict": sd}, path)
        _SCORERS[key] = Scorer(str(path), **over)
    return _SCORERS[key]


def _pair(sec, sr, ref_sec=None, seed=0):
    """(degraded, reference) int16: the reference speech-like, the degraded one it delayed by 0.12 s, attenuated and
    noisy, cut to `sec` seconds"""
    ref = synth.synth_speech_pcm16(3000 + seed, ref_sec or sec, sr)[:int((ref_sec or sec) * sr)]
    n = int(sec * sr)
    d = np.zeros(n, np.float32)
    lag = int(0.12 * sr)
    src = ref[:max(0, n - lag)].astype(np.float32) * 0.7
    d[lag:lag + src.shape[0]] = src
    d += np.random.default_rng(seed).normal(0, 300, n).astype(np.float32)
    return np.clip(d, -32768, 32767).astype(np.int16), ref


def _cut_pairs(sc, x, r, rate, window_s, window_hop_s, margin_s, channel=None):
    """Scorer.__call__ on every window pair cut out of x / r ([T] or [C, T] CUDA tensors) as clips; NaN where either
    window is too short"""
    W, H, M, d0, d1, r0, r1, _, st, _, rst = _restate(sc.args, x.shape[-1], r.shape[-1], rate, window_s, window_hop_s,
                                                      margin_s)
    want = np.full((len(d0), len(sc.columns)), np.nan, np.float32)
    ok = np.nonzero((st == E.CLIP_OK) & (rst == E.CLIP_OK))[0]
    if ok.size:
        dx = torch.zeros((ok.size,) + tuple(x.shape[:-1]) + (W,), dtype=x.dtype, device=x.device)
        rx = torch.zeros((ok.size,) + tuple(r.shape[:-1]) + (W + 2 * M,), dtype=r.dtype, device=r.device)
        for j, k in enumerate(ok):
            dx[j, ..., :d1[k] - d0[k]] = x[..., d0[k]:d1[k]]
            rx[j, ..., :r1[k] - r0[k]] = r[..., r0[k]:r1[k]]
        want[ok] = sc(dx, rate, lengths=(d1 - d0)[ok], channel=channel, reference=rx,
                      reference_lengths=(r1 - r0)[ok]).cpu().numpy()
    return want, (d0, d1, r0, r1, st, rst)


def _check(sc, x, r, rate, window_s, window_hop_s, margin_s=0.0, channel=None, cut_sc=None, cut=None, cut_rate=None,
           ref_rate=None):
    """sc.windows on one recording pair against the cut-out pairs (of `cut` = (x, r) at cut_rate through cut_sc, when
    the recordings are converted first) -> the result"""
    one = lambda t: t if t.dim() == 1 else t[None]                          # noqa: E731  ([C, T]: one recording)
    res = sc.windows(one(x), rate, window_s, window_hop_s, channel=channel, reference=one(r),
                     reference_sample_rate=ref_rate, reference_margin_s=margin_s)
    rate_m = cut_rate or rate
    want, (d0, d1, r0, r1, st, rst) = _cut_pairs(cut_sc or sc, *(cut or (x, r)), rate_m, window_s, window_hop_s, margin_s,
                                                 channel)
    what = str((rate, window_s, window_hop_s, margin_s, channel))
    assert res.counts == [want.shape[0]]
    np.testing.assert_array_equal(res.scores.cpu().numpy(), want, err_msg=what)
    for got, w in ((res.t_start, d0), (res.t_end, d1), (res.ref_t_start, r0), (res.ref_t_end, r1)):
        np.testing.assert_array_equal(got, w / rate_m)
    np.testing.assert_array_equal(res.status, st)
    np.testing.assert_array_equal(res.ref_status, rst)
    return res


@gpu
@pytest.mark.parametrize("name", VARIANTS)
def test_pairs_equal_the_cut_pairs_bit_for_bit(built_lib, tmp_path_factory, name):
    sc = _scorer(name, tmp_path_factory)
    d, r = _pair(61.0, 48000, 63.0, seed=1)
    x, y = torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda()
    for window_hop_s in (5.0, 1.0):
        for margin_s in (0.0, 0.5):
            _check(sc, x, y, 48000, 10.0, window_hop_s, margin_s)


@gpu
def test_other_inputs_equal_the_cut_pairs(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    # float32 stereo: a channel of the degraded recording and its mono mix; the stereo reference is always mixed
    d1, r1 = _pair(25.0, 48000, seed=2)
    d2, r2 = _pair(25.0, 48000, seed=3)
    xs = torch.from_numpy(np.stack([d1, d2]).astype(np.float32) / 32768.0).cuda()
    ys = torch.from_numpy(np.stack([r1, r2]).astype(np.float32) / 32768.0).cuda()
    for channel in (1, None):
        _check(sc, xs, ys, 48000, 10.0, 1.0, 0.25, channel=channel)
    # 22.05 kHz: an odd hop in frames (333 of 220 samples) keeps both pairings; a margin longer than the hop
    d, r = _pair(40.0, 22050, 30.0, seed=4)
    _check(sc, torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda(), 22050, 10.0, 3.33, 4.0)
    # 16 kHz, an odd hop (101 frames); the reference ends early: edge-clipped, too-short and empty reference windows
    d, r = _pair(40.0, 16000, 14.0, seed=5)
    res = _check(sc, torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda(), 16000, 8.0, 1.01, 1.5)
    assert (res.ref_status == E.CLIP_TOO_SHORT).any() and (res.ref_status == E.CLIP_OK).any()
    assert (res.ref_t_end == res.ref_t_start).any()                          # empty reference windows
    assert np.isnan(res.scores.cpu().numpy()[res.ref_status != E.CLIP_OK]).all()
    # a reference shorter than the margin, and a degraded recording shorter than a window
    d, r = _pair(7.0, 16000, 1.2, seed=6)
    _check(sc, torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda(), 16000, 5.0, 1.0, 2.0)
    # a too-short last degraded window
    d, r = _pair(20.05, 48000, seed=7)
    res = _check(sc, torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda(), 48000, 10.0, 10.0)
    assert res.status.tolist() == [E.CLIP_OK, E.CLIP_OK, E.CLIP_TOO_SHORT]


@gpu
def test_ms_sr_converts_both_recordings_whole(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory, ms_sr=16000)
    d, _ = _pair(25.0, 48000, seed=8)
    r = synth.synth_speech_pcm16(3100, 27.0, 22050)
    d16, r16 = RS.resample(d, 48000, 16000), RS.resample(r, 22050, 16000)
    _check(sc, torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda(), 48000, 10.0, 1.0, 0.5, ref_rate=22050,
           cut_sc=_scorer("de_cosine_hard", tmp_path_factory),
           cut=(torch.from_numpy(d16).cuda(), torch.from_numpy(r16).cuda()), cut_rate=16000)


def _batch(recs):
    T = max(x.shape[0] for x in recs)
    b = np.zeros((len(recs), T), np.int16)
    for i, x in enumerate(recs):
        b[i, :x.shape[0]] = x
    return torch.from_numpy(b).cuda(), [x.shape[0] for x in recs]


@gpu
def test_passes_batches_and_alone(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    small = _scorer("de_cosine_hard", tmp_path_factory, b200_max_chunk_segments=300)
    pairs = [_pair(3.0, 48000, 4.0, seed=9), _pair(61.0, 48000, 50.0, seed=10), _pair(25.0, 48000, 31.0, seed=11)]
    xb, lens = _batch([p[0] for p in pairs])
    yb, rlens = _batch([p[1] for p in pairs])
    kw = dict(lengths=lens, reference=yb, reference_lengths=rlens, reference_margin_s=0.5)
    one = sc.windows(xb, 48000, 10.0, 1.0, **kw)
    many = small.windows(xb, 48000, 10.0, 1.0, **kw)
    torch.cuda.synchronize()
    assert small.engine.lib.nisqa_stage_dump(small.engine.h, E.STAGE_MEL_DB, None, 0) < 0    # (it ran in passes)
    np.testing.assert_array_equal(one.scores.cpu().numpy(), many.scores.cpu().numpy())
    r0 = 0
    for i, n in enumerate(one.counts):
        alone = sc.windows(xb[i, :lens[i]], 48000, 10.0, 1.0, reference=yb[i, :rlens[i]], reference_margin_s=0.5)
        np.testing.assert_array_equal(alone.scores.cpu().numpy(), one.scores[r0:r0 + n].cpu().numpy())
        for f in WindowPairs._fields[2:]:
            np.testing.assert_array_equal(getattr(alone, f), getattr(one, f)[r0:r0 + n])
        r0 += n


@gpu
def test_stream_order_without_a_host_wait(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    d, r = _pair(30.0, 48000, seed=12)
    src_x, src_y = torch.from_numpy(d).cuda(), torch.from_numpy(r).cuda()
    want = sc.windows(src_x, 48000, 10.0, 2.0, reference=src_y, reference_margin_s=0.3).scores.cpu().numpy()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(100_000_000)                      # a slow producer ...
        x, y = torch.empty_like(src_x), torch.empty_like(src_y)
        x.copy_(src_x)
        y.copy_(src_y)                                     # ... fills the input right before the call, no synchronise
        got = sc.windows(x, 48000, 10.0, 2.0, reference=y, reference_margin_s=0.3)
        assert not s.query()                               # returned while the stream still sleeps
        del x, y
        junk = [torch.full_like(src_y, 7) for _ in range(3)]       # reuses the freed input, on s
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.scores.cpu().numpy(), want)
    del junk


@gpu
def test_engine_refusals(built_lib, tmp_path_factory):
    de = _scorer("de_cosine_hard", tmp_path_factory)
    se = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    x = torch.zeros(48000 * 20, dtype=torch.int16, device="cuda")
    b = se._batch("wave", x, 48000, None, None)
    b16 = se._batch("reference", x, 16000, None, None)
    out = torch.empty(64, device="cuda")
    try:
        with pytest.raises(E.EngineError, match="NISQA_DE"):        # unchanged: no plain windows on a DE engine
            de.engine.predict_device_windows(0, b, out.data_ptr(), 64, 480000, 100)
        with pytest.raises(E.EngineError, match="double-ended"):
            se.engine.predict_device_window_pairs(0, b, b, out.data_ptr(), 64, 480000, 100, 0)
        with pytest.raises(E.EngineError, match="ref.sample_rate"):
            de.engine.predict_device_window_pairs(0, b, b16, out.data_ptr(), 64, 480000, 100, 0)
        with pytest.raises(E.EngineError, match="margin_frames"):
            de.engine.predict_device_window_pairs(0, b, b, out.data_ptr(), 64, 480000, 100, -1)
        with pytest.raises(E.EngineError, match="margin_frames"):
            de.engine.predict_device_window_pairs(0, b, b, out.data_ptr(), 64, 480000, 100, 3000)
        with pytest.raises(E.EngineError, match="n_rows"):
            de.engine.predict_device_window_pairs(0, b, b, out.data_ptr(), 2, 480000, 100, 0)
    finally:
        se.close()


@gpu
def test_sample_of_pairs_against_the_oracle(built_lib, tmp_path_factory):
    from oracle import de_arch_oracle as DO
    name = "std_fc20_lstm128bi_luong_soft_fd128"
    args, sd = _checkpoint(name)
    sc = _scorer(name, tmp_path_factory)
    d, r = _pair(40.0, 16000, 38.0, seed=13)
    res = sc.windows(torch.from_numpy(d).cuda(), 16000, 10.0, 5.0, reference=torch.from_numpy(r).cuda(),
                     reference_margin_s=0.5)
    got = res.scores.cpu().numpy()
    f = lambda a: a.astype(np.float32) / np.float32(32768.0)      # noqa: E731
    for k in (0, 3, len(got) - 1):
        a, b = (int(round(t * 16000)) for t in (res.t_start[k], res.t_end[k]))
        ra, rb = (int(round(t * 16000)) for t in (res.ref_t_start[k], res.ref_t_end[k]))
        want, (n1, n2), st = DO.predict_pcm_de(args, sd, f(d[a:b]), 16000, f(r[ra:rb]), 16000)
        assert st == 0 and (n1, n2) == (res.n_segments[k], res.ref_n_segments[k])
        np.testing.assert_allclose(got[k], want, atol=1e-4, rtol=0)


@gpu
def test_cli_writes_window_pairs_csv(built_lib, tmp_path_factory, tmp_path):
    import pandas as pd
    from nisqa_b200.NISQA_model import nisqaModel
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    rows = []
    for i, (sec, rsec) in enumerate(((61.0, 60.0), (6.0, 8.0))):
        d, r = _pair(sec, 48000, rsec, seed=20 + i)
        wav.write_wav_pcm16(str(tmp_path / ("deg%d.wav" % i)), d, 48000)
        wav.write_wav_pcm16(str(tmp_path / ("ref%d.wav" % i)), r, 48000)
        rows.append(("deg%d.wav" % i, "ref%d.wav" % i))
    pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(tmp_path / "files.csv", index=False)
    m = nisqaModel({"mode": "predict_csv", "pretrained_model": str(tmp_path_factory.getbasetemp() / "de_cosine_hard.tar"),
                    "csv_file": "files.csv", "csv_deg": "deg", "csv_ref": "ref", "data_dir": str(tmp_path),
                    "output_dir": str(tmp_path), "ms_channel": None, "tr_bs_val": 1, "tr_num_workers": 0,
                    "window_s": 10.0, "window_hop_s": 5.0, "reference_margin_s": 0.5})
    try:
        m.predict()
    finally:
        m.model.close()
    df = pd.read_csv(tmp_path / "NISQA_windows.csv")
    assert list(df.columns) == ["deg", "ref", "t_start", "t_end", "ref_t_start", "ref_t_end", "n_segments",
                                "ref_n_segments", "mos_pred"]
    for f, g in rows:
        y, sr = wav.read_wav(str(tmp_path / f), None)
        yr, _ = wav.read_wav(str(tmp_path / g), None)
        res = sc.windows(torch.from_numpy(y).cuda(), sr, 10.0, 5.0, reference=torch.from_numpy(yr).cuda(),
                         reference_margin_s=0.5)
        part = df[df["deg"] == f]
        assert len(part) == res.counts[0] and set(part["ref"]) == {g}
        for c in ("t_start", "t_end", "ref_t_start", "ref_t_end", "n_segments", "ref_n_segments"):
            np.testing.assert_array_equal(part[c].to_numpy(), getattr(res, c))
        np.testing.assert_array_equal(part["mos_pred"].to_numpy().astype(np.float32), res.scores.cpu().numpy()[:, 0])
