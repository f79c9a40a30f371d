"""Per-segment scores and pooling weights: nisqa_predict_device_batch_segments, Scorer.segments and
run_predict.py --segments.  CPU part: the oracle restatement and the identity score = sum_t a_t s_t on the golden of the
unmodified reference modules (oracle/make_segment_golden.py), the ABI, and the time columns.  GPU part: every golden
variant, bit identity of the clip scores with Scorer.__call__, ragged and multi-pass batches, the stream contract, the
too-small-buffer refusal and the CLI."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from nisqa_b200.scorer import Scorer
from oracle import segment_oracle as SO
from oracle import segment_variants as SV
from oracle import variants as V

gpu = pytest.mark.gpu
SEG_TOL = 1e-4
WEIGHTED = ("att", "avg", "last_step")        # the pooling modules whose clip score is sum_t a_t s_t


def _golden():
    return np.load(os.path.join(GOLDEN, "segments.npz"))


def _rows(z, name):
    return z[name + "/x"] if name + "/x" in z.files else z[str(z[name + "/x_from"]) + "/x"]


def _pcm(name, args):
    """(deg clips, rates, reference clips or None, their rates) the golden variant was scored on"""
    if args["model"] == "NISQA_DE":
        pairs = [V.de_pair_pcm(p) for p in SV.SEGMENT_DE_PAIRS]
        return [p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs], [p[3] for p in pairs]
    return [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in SV.SEGMENT_CLIPS], [c[2] for c in SV.SEGMENT_CLIPS], None, None


def _padded(clips):
    T = max(c.shape[0] for c in clips)
    x = np.zeros((len(clips), T), np.int16)
    for i, c in enumerate(clips):
        x[i, :c.shape[0]] = c
    return torch.from_numpy(x).cuda(), [c.shape[0] for c in clips]


def _scorer(name, tmp_path, **over):
    args, sd = SV.segment_checkpoint(name, WEIGHTS)
    path = os.path.join(str(tmp_path), name + ".tar")
    torch.save({"args": dict(args, **over), "model_state_dict": sd}, path)
    return Scorer(path), args


# ------------------------------------------------------------------ CPU
def test_oracle_restatement_matches_the_golden():
    z = _golden()
    for name in SV.SEGMENT_VARIANTS:
        args, sd = SV.segment_checkpoint(name, WEIGHTS)
        x, counts = _rows(z, name), z[name + "/counts"]
        r = 0
        for n in counts:
            s, w = SO.segment_scores(args, sd, torch.from_numpy(x[r:r + n]))
            np.testing.assert_allclose(s, z[name + "/seg_scores"][r:r + n], atol=5e-6, rtol=0, err_msg=name)
            np.testing.assert_allclose(w, z[name + "/seg_weights"][r:r + n], atol=5e-6, rtol=0, err_msg=name)
            assert np.array_equal(np.isnan(w), np.isnan(z[name + "/seg_weights"][r:r + n])), name
            r += n
        assert r == x.shape[0] == z[name + "/seg_scores"].shape[0]


def test_golden_weighted_sum_is_the_clip_score():
    z = _golden()
    checked = set()
    for name in SV.SEGMENT_VARIANTS:
        args, _ = SV.segment_checkpoint(name, WEIGHTS)
        s, w, sc = z[name + "/seg_scores"], z[name + "/seg_weights"], z[name + "/scores"]
        if args["pool"] not in WEIGHTED:
            assert np.isnan(w).all(), name
            continue
        checked.add(args["pool"] + ("_ff" if args.get("pool_att_h") else ""))
        r = 0
        for b, n in enumerate(z[name + "/counts"]):
            np.testing.assert_allclose((w[r:r + n] * s[r:r + n]).sum(0), sc[b], atol=1e-5, rtol=0, err_msg=name)
            r += n
    assert checked == {"att", "att_ff", "avg", "last_step"}


def test_segment_out_struct_header_and_exports(tmp_path, built_lib):
    src = tmp_path / "layout.c"
    fields = ["scores", "weights", "n_rows"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(nisqa_segment_out)'
                   + "".join(", offsetof(nisqa_segment_out, %s)" % f for f in fields) + ");return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [ctypes.sizeof(E.NisqaSegmentOut)] + [getattr(E.NisqaSegmentOut, f).offset for f in fields]
    header = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    assert "nisqa_predict_device_batch_segments(" in header
    assert "nisqa_predict_device_batch_segments" in E.EXPORTS
    assert hasattr(E.load_library(), "nisqa_predict_device_batch_segments")


@pytest.mark.parametrize("ckpt, n, sr", [("nisqa.tar", 48000 * 3 + 17, 48000), ("nisqa_tts.tar", 16000 * 2 + 5, 16000),
                                         ("nisqa.tar", 44100 * 5 + 3, 44100)])
def test_time_columns_follow_the_segment_arithmetic(built_lib, ckpt, n, sr):
    """t_start / t_end of Scorer.segments: the centres of each segment's first and last mel frame, the last one the
    clip's last frame that nisqa_segment_counts counts"""
    s = Scorer.__new__(Scorer)
    args = E.load_checkpoint(os.path.join(WEIGHTS, ckpt))[0]
    s._configure(args, torch.device("cpu"))
    n_frames, n_seg, st = E.segment_counts(s.cfg, n, sr)
    assert st == E.CLIP_OK
    hop = int(sr * args["ms_hop_length"])
    t = np.arange(n_seg)
    t_start = t * args["ms_seg_hop_length"] * hop / sr
    t_end = (t * args["ms_seg_hop_length"] + args["ms_seg_length"] - 1) * hop / sr
    # the first frame of the last segment + seg_length frames fit in the clip's frames; one more hop would not
    last = int(round(t_end[-1] * sr / hop))
    assert last <= n_frames - 1 and last + args["ms_seg_hop_length"] > n_frames - 1
    assert t_start[0] == 0.0 and np.all(np.diff(t_start) > 0)
    np.testing.assert_allclose(t_end - t_start, (args["ms_seg_length"] - 1) * hop / sr)


# ------------------------------------------------------------------ GPU
@gpu
@pytest.mark.parametrize("name", list(SV.SEGMENT_VARIANTS))
def test_every_golden_variant(built_lib, tmp_path, name):
    z = _golden()
    sc, args = _scorer(name, tmp_path)
    deg, srs, ref, ref_srs = _pcm(name, args)
    want_s, want_w = z[name + "/seg_scores"], z[name + "/seg_weights"]
    got_s, got_w, counts = [], [], []
    for i in range(len(deg)):          # (the clips have different rates: one call each)
        x, lens = _padded([deg[i]])
        kw = {}
        if ref is not None:
            kw["reference"], kw["reference_lengths"] = _padded([ref[i]])
            kw["reference_sample_rate"] = ref_srs[i]
        res = sc.segments(x, srs[i], lengths=lens, **kw)
        plain = sc(x, srs[i], lengths=lens, **kw)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(res.scores.cpu().numpy(), plain.cpu().numpy())
        np.testing.assert_allclose(res.scores.cpu().numpy()[0], z[name + "/scores"][i], atol=SEG_TOL, rtol=0)
        got_s.append(res.seg_scores.cpu().numpy())
        got_w.append(res.seg_weights.cpu().numpy())
        counts += res.counts
        s, w = got_s[-1], got_w[-1]
        if args["pool"] in WEIGHTED:
            np.testing.assert_allclose((w * s).sum(0), res.scores.cpu().numpy()[0], atol=2e-5, rtol=0)
            np.testing.assert_allclose(w.sum(0), 1.0, atol=1e-6, rtol=0)
    assert counts == z[name + "/counts"].tolist()
    got_s, got_w = np.concatenate(got_s), np.concatenate(got_w)
    np.testing.assert_allclose(got_s, want_s, atol=SEG_TOL, rtol=0)
    assert np.array_equal(np.isnan(got_w), np.isnan(want_w))
    np.testing.assert_allclose(np.nan_to_num(got_w), np.nan_to_num(want_w), atol=SEG_TOL, rtol=0)
    sc.close()


def _ragged_case(sc):
    """a one-segment clip between long clips, and a 1300-segment clip (ms_max_segments of nisqa.tar)"""
    from test_device_batch import _len_for_segments
    lens = [48000 * 7 + 11, _len_for_segments(sc.cfg, 1, 48000), 48000 * 4, _len_for_segments(sc.cfg, 1300, 48000)]
    T = max(lens)
    x = np.zeros((len(lens), T), np.int16)
    for i, n in enumerate(lens):
        x[i, :n] = synth.synth_speech_pcm16(1400 + i, n / 48000.0 + 0.01, 48000)[:n]
    return torch.from_numpy(x).cuda(), lens


@gpu
@pytest.mark.parametrize("ckpt", ["nisqa.tar", "nisqa_tts.tar"])
def test_ragged_multi_pass_and_alone_are_bit_identical(built_lib, ckpt):
    sc = Scorer(os.path.join(WEIGHTS, ckpt))
    small = Scorer(os.path.join(WEIGHTS, ckpt), b200_max_chunk_segments=700)
    x, lens = _ragged_case(sc)
    one = sc.segments(x, 48000, lengths=lens)
    many = small.segments(x, 48000, lengths=lens)
    torch.cuda.synchronize()
    assert small.engine.lib.nisqa_stage_dump(small.engine.h, E.STAGE_MEL_DB, None, 0) < 0    # (it really ran in passes)
    assert one.counts[1] == 1 and one.counts[3] == 1300 and sum(one.counts) == one.seg_scores.shape[0]
    for a, b in ((one.scores, many.scores), (one.seg_scores, many.seg_scores), (one.seg_weights, many.seg_weights)):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    r = 0
    for i, n in enumerate(one.counts):
        alone = sc.segments(x[i:i + 1], 48000, lengths=[lens[i]])
        torch.cuda.synchronize()
        np.testing.assert_array_equal(alone.seg_scores.cpu().numpy(), one.seg_scores[r:r + n].cpu().numpy())
        np.testing.assert_array_equal(alone.seg_weights.cpu().numpy(), one.seg_weights[r:r + n].cpu().numpy())
        np.testing.assert_array_equal(alone.scores.cpu().numpy(), one.scores[i:i + 1].cpu().numpy())
        r += n
    np.testing.assert_array_equal(one.t_start[r - 1300:], sc.segments(x[3:], 48000, lengths=lens[3:]).t_start)
    sc.close()
    small.close()


@gpu
def test_tts_plain_call_unchanged_by_a_segments_call(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa_tts.tar"))
    x = torch.from_numpy(np.stack([synth.synth_speech_pcm16(1500 + i, 3.0, 16000) for i in range(3)])).cuda()
    before = sc(x, 16000).cpu().numpy()
    sc.segments(x, 16000)
    after = sc(x, 16000).cpu().numpy()
    np.testing.assert_array_equal(before, after)
    with pytest.raises(E.EngineError, match="keep_td_out"):     # the option itself is unchanged
        sc.engine.stage_dump(E.STAGE_TD_OUT)
    sc.close()


@gpu
def test_double_ended_rows_and_ms_sr_times(built_lib, tmp_path):
    sc, args = _scorer("de_cosine_hard", tmp_path)
    deg, srs, ref, ref_srs = _pcm("de_cosine_hard", args)
    x, lens = _padded([deg[0], deg[0][:24000]])
    r, rlens = _padded([ref[0], ref[0]])
    res = sc.segments(x, srs[0], lengths=lens, reference=r, reference_lengths=rlens, reference_sample_rate=ref_srs[0])
    n_deg = [E.segment_counts(sc.cfg, n, srs[0])[1] for n in lens]
    assert res.counts == n_deg and res.seg_scores.shape[0] == sum(n_deg)
    sc.close()
    sc = Scorer(os.path.join(WEIGHTS, "nisqa_mos_only.tar"), ms_sr=16000)
    x = torch.from_numpy(synth.synth_speech_pcm16(1510, 2.0, 48000)[None]).cuda()
    res = sc.segments(x, 48000)
    hop = int(16000 * sc.args["ms_hop_length"])
    assert res.counts == [E.segment_counts(sc.cfg, 32000, 16000)[1]]
    np.testing.assert_array_equal(res.t_start, np.arange(res.counts[0]) * sc.args["ms_seg_hop_length"] * hop / 16000)
    sc.close()


@gpu
def test_segments_call_does_not_wait_and_input_frees_in_stream_order(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    B, T = 3, 48000 * 4
    src = torch.from_numpy(np.stack([synth.synth_speech_pcm16(1520 + i, 4.0, 48000)[:T] for i in range(B)])).cuda()
    want = sc.segments(src, 48000)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)
    got = sc.segments(src, 48000)
    assert not torch.cuda.current_stream().query()          # returned while the stream still sleeps
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.seg_scores.cpu().numpy(), want.seg_scores.cpu().numpy())
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        x = torch.empty_like(src)
        x.copy_(src)
        got = sc.segments(x, 48000)
        del x
        junk = [torch.full((B, T), 7, dtype=torch.int16, device="cuda") for _ in range(3)]
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.seg_weights.cpu().numpy(), want.seg_weights.cpu().numpy())
    del junk
    sc.close()


@gpu
def test_too_small_n_rows_is_refused_before_anything_is_enqueued(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    x = torch.from_numpy(np.stack([synth.synth_speech_pcm16(1530 + i, 2.0, 48000) for i in range(2)])).cuda()
    res = sc.segments(x, 48000)
    torch.cuda.synchronize()
    n = sum(res.counts)
    deg = E.device_batch(x.data_ptr(), E.FMT_S16, [x.shape[1]] * 2, 1, -1, x.shape[1], x.stride(0), 0, 48000)
    before = sc.engine.kernel_launches()
    with pytest.raises(E.EngineError, match="n_rows"):
        sc.engine.predict_device_batch_segments(torch.cuda.current_stream().cuda_stream, deg, res.scores.data_ptr(),
                                                res.seg_scores.data_ptr(), res.seg_weights.data_ptr(), n - 1)
    assert sc.engine.kernel_launches() == before
    sc.close()


@gpu
def test_cli_writes_segments_csv_and_leaves_results_unchanged(built_lib, tmp_path):
    import pandas as pd
    import run_predict
    from nisqa_b200.NISQA_model import nisqaModel
    d = tmp_path / "wavs"
    d.mkdir()
    for i, (sec, sr) in enumerate([(2.0, 48000), (1.1, 16000), (3.0, 48000)]):
        wav.write_wav_pcm16(str(d / ("c%d.wav" % i)), synth.synth_speech_pcm16(1540 + i, sec, sr), sr)
    outs = {}
    for seg in (False, True):
        o = tmp_path / ("out%d" % seg)
        o.mkdir()
        argv = ["--mode", "predict_dir", "--pretrained_model", os.path.join(WEIGHTS, "nisqa.tar"), "--data_dir", str(d),
                "--output_dir", str(o), "--bs", "2"] + (["--segments"] if seg else [])
        nisqaModel(run_predict.parse_args(argv)).predict()
        outs[seg] = o
    a = open(outs[False] / "NISQA_results.csv", "rb").read()
    assert a == open(outs[True] / "NISQA_results.csv", "rb").read()
    assert not (outs[False] / "NISQA_segments.csv").exists()
    seg = pd.read_csv(outs[True] / "NISQA_segments.csv")
    res = pd.read_csv(outs[True] / "NISQA_results.csv")
    cfg = E.config_from_args(E.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))[0])
    assert list(seg.columns) == ["deg", "segment", "t_start", "t_end", "mos_pred", "noi_pred", "dis_pred", "col_pred",
                                 "loud_pred", "mos_weight", "noi_weight", "dis_weight", "col_weight", "loud_weight"]
    for f in res["deg"]:
        n, sr = wav.read_wav(str(d / f), None)[0].shape[0], wav.read_wav(str(d / f), None)[1]
        rows = seg[seg["deg"] == f]
        assert len(rows) == E.segment_counts(cfg, n, sr)[1]
        mos = float(res[res["deg"] == f]["mos_pred"].iloc[0])
        assert abs(float((rows["mos_pred"] * rows["mos_weight"]).sum()) - mos) < 1e-4


def test_segments_refused_under_torchrun(monkeypatch):
    from nisqa_b200.NISQA_model import nisqaModel
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("LOCAL_RANK", "0")
    with pytest.raises(ValueError, match="segments"):
        nisqaModel({"mode": "predict_csv", "segments": True, "csv_file": "/nonexistent.csv"})
