"""Checkpoints trained with other Mel-spectrogram segment shapes (ms_n_mels x ms_seg_length): AdaptCNN at any accepted
shape (the separate conv1 + adaptive pool1 kernel), SkipCNN and DFF (fan_in = n_mels * seg_length, zero-padded to a
multiple of 64), behind self-attention, no td, or NISQA_DE's stack.

CPU: config_from_args accepts every accepted shape for every framewise model and fills n_mels / seg_len; it refuses the
shapes outside the kernels (and StandardCNN at any shape but 48 x 15, n_fft other than 4096), naming the value;
nisqa_segment_counts is bit-exact against the oracle for several segment lengths, at the too-short boundary too; the
oracle against the scores of the unmodified reference modules (tests/golden/variants_mel.npz, oracle/make_mel_golden.py).
GPU: every mel variant through the C ABI against the reference scores and the oracle (a one-segment and a 97-segment
clip, an 8 kHz clip - empty filters at 128 bands -, a 96 kHz clip - the front end's long-window kernel -, PCM16 and float
input), alone == in a batch, several passes == one pass; the filterbank and the MEL_DB dump against the oracle for every
band count; stage bounds from the engine's own dumps (tests/stage_ref.py); the tensor-core and FFMA conv paths against
each other; one 64-band checkpoint end to end through nisqaModel(mode='predict_dir').
"""
import os

import numpy as np
import pytest
import torch

import stage_ref as R
from conftest import GOLDEN, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from oracle import mel_variants as V
from oracle import nisqa_oracle as O
from oracle import td_pair_oracle as TO
from oracle.td_pair_variants import sa
from oracle.variants import de_pair_pcm

SCORE_TOL = 1e-4
MEL_TOL_DB = 1e-3
SR = 16000
N_MELS = (32, 40, 48, 64, 80, 96, 128)
SEG_LENS = (3, 9, 15, 21, 31)


def _variant(name):
    base = V.MEL_VARIANTS[name][0]
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.mel_checkpoint(name, args, sd)


def _args(ckpt, **over):
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    return dict(args, **over)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


# ------------------------------------------------------------------------------------------------------------ CPU
def _framewise_args():
    """args of every framewise model that takes other shapes: AdaptCNN with and without its Linear, SkipCNN raw and with
    its Linear, DFF - behind self-attention - and raw SkipCNN behind no td"""
    mos = _args("nisqa_mos_only.tar")
    return {"adapt": mos, "adapt_fc": dict(mos, cnn_fc_out_h=128), "skip": dict(mos, cnn_model="skip", cnn_fc_out_h=None),
            "skip_fc": dict(mos, cnn_model="skip", cnn_fc_out_h=256), "dff": dict(mos, cnn_model="dff", cnn_fc_out_h=256),
            "skip_td_skip": dict(mos, cnn_model="skip", cnn_fc_out_h=None, td="skip", td_2="skip", pool="avg", pool_att_h=None)}


def test_config_accepts_the_table():
    for kind, args in _framewise_args().items():
        for n_mels in N_MELS:
            for seg_len in SEG_LENS:
                c = E.config_from_args(dict(args, ms_n_mels=n_mels, ms_seg_length=seg_len))
                assert (c.n_fft, c.n_mels, c.seg_len) == (4096, n_mels, seg_len), kind
    for name in V.MEL_VARIANTS:
        args, _ = _variant(name)
        c = E.config_from_args(args)
        assert (c.n_mels, c.seg_len, c.seg_hop) == (args["ms_n_mels"], args["ms_seg_length"], args["ms_seg_hop_length"])
        assert c.double_ended == (1 if args["model"] == "NISQA_DE" else 0)
    # the shipped shape of StandardCNN still runs
    c = E.config_from_args(_args("nisqa_tts.tar"))
    assert (c.n_mels, c.seg_len) == (48, 15)


def test_config_refuses_shapes_outside_the_kernels():
    mos = _args("nisqa_mos_only.tar")
    tts = _args("nisqa_tts.tar")
    std_sa = dict(tts, cnn_fc_out_h=None, **sa("td", 64, 64), td_2="skip", pool="att", pool_att_h=128)
    for bad, what in ((dict(mos, ms_n_mels=50), "ms_n_mels=50"),
                      (dict(mos, ms_n_mels=256), "ms_n_mels=256"),
                      (dict(mos, ms_seg_length=2), "ms_seg_length=2"),
                      (dict(mos, ms_seg_length=33), "ms_seg_length=33"),
                      (dict(mos, ms_seg_length=20), "ms_seg_length=20.*odd"),
                      (dict(tts, ms_n_mels=64), r"ms_n_mels=64, ms_seg_length=15 with cnn_model='standard'.*output_height"),
                      (dict(tts, ms_seg_length=21), r"ms_n_mels=48, ms_seg_length=21 with cnn_model='standard'.*output_width"),
                      (dict(std_sa, ms_n_mels=64), r"ms_n_mels=64.*cnn_model='standard'"),
                      (dict(mos, ms_n_fft=2048), "ms_n_fft=2048")):
        with pytest.raises(NotImplementedError, match=what):
            E.config_from_args(bad)


def test_segment_counts_bit_exact_vs_oracle(built_lib):
    for seg_len in SEG_LENS:
        for seg_hop in (1, 2, 4):
            args = _args("nisqa_mos_only.tar", ms_seg_length=seg_len, ms_seg_hop_length=seg_hop)
            cfg = E.config_from_args(args)
            for sr in (8000, 16000, 48000):
                hop = int(sr * args["ms_hop_length"])
                # n_frames = 1 + n // hop: seg_len - 2 .. seg_len + 1 frames (the too-short boundary), and longer clips
                ns = [(f - 1) * hop + d for f in range(max(1, seg_len - 2), seg_len + 2) for d in (0, hop - 1)]
                ns = [n for n in ns if n > 0] + [12345, 3 * sr + 7]       # (an empty clip has no frames at all)
                for n in ns:
                    got = E.segment_counts(cfg, n, sr)
                    want = O.segment_counts(n, sr, args)
                    assert got == tuple(want), (seg_len, seg_hop, sr, n, got, want)
            # exactly at the boundary: seg_len - 1 frames is too short, seg_len frames is one segment
            hop = int(SR * args["ms_hop_length"])
            assert E.segment_counts(cfg, (seg_len - 2) * hop, SR)[1:] == (0, E.CLIP_TOO_SHORT)
            assert E.segment_counts(cfg, (seg_len - 1) * hop, SR)[1:] == (1, E.CLIP_OK)


def test_oracle_matches_reference_modules_on_the_mel_variants():
    g = np.load(os.path.join(GOLDEN, "variants_mel.npz"))
    assert sorted(g.files) == sorted(V.MEL_VARIANTS)
    for name in V.MEL_VARIANTS:
        args, sd = _variant(name)
        if args["model"] == "NISQA_DE":
            for i, pair in enumerate(V.MEL_DE_PAIRS):
                deg, srd, ref, srr = de_pair_pcm(pair)
                sc, _, st = O.predict_pcm_de(args, sd, _f32(deg), srd, _f32(ref), srr)
                assert st == O.STATUS_OK
                np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)
            continue
        for i, (seed, sec, sr) in enumerate(V.MEL_CLIPS):
            sc, _, st = TO.predict_pcm(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


def test_golden_scores_lie_in_the_mos_range():
    """every golden score lies where an absolute 1e-4 tolerance means something"""
    g = np.load(os.path.join(GOLDEN, "variants_mel.npz"))
    for name in g.files:
        n = len(V.MEL_DE_PAIRS) if name.startswith("de_") else len(V.MEL_CLIPS)
        assert g[name].shape == (n, 5 if name.startswith("dim_") else 1), name
        assert np.isfinite(g[name]).all() and g[name].min() >= -2.0 and g[name].max() <= 8.0, (name, g[name].tolist())


# ------------------------------------------------------------------------------------------------------------ GPU
def _pcm(args, n_seg, seed, sr=SR):
    """a clip of exactly n_seg segments"""
    hop = int(sr * args["ms_hop_length"])
    n = (args["ms_seg_length"] + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * hop
    y = synth.synth_speech_pcm16(seed, n / sr + 0.05, sr)[:n]
    assert O.segment_counts(n, sr, args)[1] == n_seg
    return y


def _engine(args, sd, **kw):
    eng = E.Engine(E.config_from_args(args, **kw), 0)
    eng.load_state_dict(sd)
    return eng


SINGLE = [n for n in V.MEL_VARIANTS if not n.startswith("de_")]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["pcm16", "f32"])
@pytest.mark.parametrize("name", SINGLE)
def test_mel_variant_through_the_c_abi(built_lib, name, fmt):
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_mel.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.MEL_CLIPS]
    srs = [c[2] for c in V.MEL_CLIPS]
    # one segment between long clips, 97 segments, 8 kHz (128 bands: empty filters), 96 kHz (windows over 1024 samples)
    extra = [_pcm(args, 1, 7), _pcm(args, 97, 8), synth.synth_speech_pcm16(9, 1.3, 8000), synth.synth_speech_pcm16(10, 0.6, 96000)]
    esr = [SR, SR, 8000, 96000]
    batch = pcm[:2] + extra[:1] + pcm[2:] + extra[1:]
    bsr = srs[:2] + esr[:1] + srs[2:] + esr[1:]
    if fmt == "f32":
        batch = [_f32(p) for p in batch]
    # (a window over 1024 samples - the 96 kHz clip - sends the whole pass through the long-window front-end kernel,
    # whose sums round differently: the bit-for-bit checks below run on the batch without it)
    same = [i for i, sr in enumerate(bsr) if sr != 96000]
    eng = _engine(args, sd)
    try:
        scores, nseg, status = eng.predict_pcm(batch, bsr)
        assert np.all(status == E.CLIP_OK), (name, status)
        ours = np.concatenate([scores[:2], scores[3:3 + len(pcm) - 2]])
        err = float(np.abs(ours - g).max())
        print("\n%s %s: max |engine - reference| %.3g" % (name, fmt, err))
        assert err <= SCORE_TOL, (name, err)
        worst = 0.0
        for i, (p, sr) in enumerate(zip(batch, bsr)):
            ref, ns, st = TO.predict_pcm(args, sd, p if fmt == "f32" else _f32(p), sr)
            assert st == O.STATUS_OK and ns == nseg[i], (name, i)
            worst = max(worst, float(np.abs(scores[i] - ref).max()))
        print("%s %s: max |engine - oracle| %.3g over segment counts %s" % (name, fmt, worst, nseg.tolist()))
        assert worst <= SCORE_TOL, (name, worst)
        batch, bsr = [batch[i] for i in same], [bsr[i] for i in same]
        scores, nseg, _ = eng.predict_pcm(batch, bsr)
        for i in range(len(batch)):                                      # alone == in the batch, bit for bit
            alone, _, _ = eng.predict_pcm(batch[i:i + 1], bsr[i:i + 1])
            np.testing.assert_array_equal(alone[0], scores[i])
    finally:
        eng.close()
    eng = _engine(args, sd, max_chunk_segments=120)                      # several internal passes == one pass
    try:
        multi, nseg2, _ = eng.predict_pcm(batch, bsr)
        np.testing.assert_array_equal(nseg2, nseg)
        np.testing.assert_array_equal(multi, scores)
    finally:
        eng.close()


@pytest.mark.gpu
def test_double_ended_mel_variant_through_the_c_abi(built_lib):
    name = "de_adapt_m64_s15"
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_mel.npz"))[name]
    clips, srs, refs = [], [], []
    for pair in V.MEL_DE_PAIRS:
        deg, srd, ref, srr = de_pair_pcm(pair)
        clips += [deg, ref]
        srs += [srd, srr]
        refs.append(O.predict_pcm_de(args, sd, _f32(deg), srd, _f32(ref), srr)[0])
    eng = _engine(args, sd)
    try:
        scores, _, status = eng.predict_pcm(clips, srs)
        assert np.all(status == E.CLIP_OK)
        got = scores[0::2]
        print("\n%s: max |engine - reference| %.3g, |engine - oracle| %.3g" % (
            name, float(np.abs(got - g).max()), float(np.abs(got - np.array(refs)).max())))
        assert np.abs(got - g).max() <= SCORE_TOL
        assert np.abs(got - np.array(refs)).max() <= SCORE_TOL
        alone, _, _ = eng.predict_pcm(clips[2:4], srs[2:4])                # a pair alone == in the batch
        np.testing.assert_array_equal(alone[0], scores[2])
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", N_MELS)
def test_filterbank_and_mel_db_against_the_oracle(built_lib, n_mels):
    from oracle import librosa_compat as lb
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    args = dict(args, ms_n_mels=n_mels)
    clips = [(1, 1.1, 48000), (2, 0.7, 16000), (3, 0.5, 8000), (4, 0.4, 96000), (5, 0.9, 44100)]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in clips]
    srs = [c[2] for c in clips]
    eng = _engine(args, sd)
    try:
        for sr in sorted(set(srs)):
            ref = lb.mel(sr, 4096, n_mels=n_mels, fmin=0.0, fmax=args["ms_fmax"], htk=False, norm="slaney")
            np.testing.assert_allclose(eng.mel_filterbank(sr), ref, rtol=0, atol=1e-7)
        for fmt in ("pcm16", "f32"):
            batch = pcm if fmt == "pcm16" else [_f32(p) for p in pcm]
            _, _, status = eng.predict_pcm(batch, srs)
            assert np.all(status == E.CLIP_OK)
            dump = eng.stage_dump(E.STAGE_MEL_DB)
            off = 0
            for p, sr in zip(pcm, srs):
                ref = np.asarray(O.mel_db(_f32(p), sr, args), dtype=np.float32)
                assert ref.shape[0] == n_mels
                got = dump[off:off + ref.size].reshape(ref.shape)
                off += ref.size
                err = float(np.abs(got - ref).max())
                assert err <= MEL_TOL_DB, (n_mels, sr, fmt, err)
            assert off == dump.size
    finally:
        eng.close()


def _stage_dumps(eng, args, lens, seed, stages):
    clips = [_pcm(args, n, seed + i) for i, n in enumerate(lens)]
    scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
    assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
    mel = eng.stage_dump(E.STAGE_MEL_DB)
    n_frames = [O.segment_counts(len(c), SR, args)[0] for c in clips]
    offs = np.concatenate([[0], np.cumsum(n_frames)]) * args["ms_n_mels"]
    seg = torch.cat([O.segments(mel[offs[i]:offs[i + 1]].reshape(args["ms_n_mels"], -1), args)
                     for i in range(len(clips))]).double()
    return seg, {k: torch.from_numpy(eng.stage_dump(st)).double() for k, st in stages.items()}


ADAPT_STAGES = {"pool1": (E.STAGE_POOL1, (16, 24, 7)), "pool2": (E.STAGE_POOL2, (32, 12, 5)), "conv3": (E.STAGE_CONV3, (64, 12, 5)),
                "pool3": (E.STAGE_POOL3, (64, 6, 3)), "conv5": (E.STAGE_CONV5, (64, 6, 3))}


@pytest.mark.gpu
@pytest.mark.parametrize("conv_tc", [1, 0])
@pytest.mark.parametrize("name", ["dim_adapt_m32_s11", "mos_adapt_m48_s21", "dim_adapt_fc128_m128_s21", "mos_adapt_m80_s31_hop2"])
def test_adapt_stages_against_float64(built_lib, name, conv_tc):
    """MEL_DB -> POOL1 (conv1 + adaptive pool1 of the runtime shape) and POOL1 -> ... -> CNN_FEAT against float64 from the
    engine's own dumps (bound TAU = 2^-18 times the magnitude of the stage's terms, tests/stage_ref.py)."""
    args, sd = _variant(name)
    lens = [1, 13, 97, 2, 40]
    N = sum(lens)
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        eng.set_option("conv_tc", conv_tc)
        eng.set_option("conv12", 1)              # (other shapes always take the separate conv1 kernel: pool1 is dumped)
        eng.load_state_dict(sd)
        stages = {k: v[0] for k, v in ADAPT_STAGES.items()}
        stages["cnn_feat"] = E.STAGE_CNN_FEAT
        seg, d = _stage_dumps(eng, args, lens, 500, stages)
    finally:
        eng.close()
    act = {k: d[k].reshape(N, *ADAPT_STAGES[k][1]) for k in ADAPT_STAGES}
    feat = d["cnn_feat"].reshape(N, -1)
    ratios = {}
    chain = [("mel", "pool1", 1), ("pool1", "pool2", 2), ("pool2", "conv3", 3), ("conv3", "pool3", 4), ("pool3", "conv5", 5),
             ("conv5", "cnn_feat", 6)]
    for src, dst, layer in chain:
        x = seg if src == "mel" else act[src]
        ref, err = R.conv_layer(sd, args, layer, x)
        if dst == "cnn_feat":            # (CNN_FEAT: conv6's 384 features, in front of AdaptCNN's Linear)
            ref, err = R.cnn_tail({k: v for k, v in sd.items() if not k.startswith("cnn.model.fc.")}, args, ref, err)
        got = feat if dst == "cnn_feat" else act[dst]
        ratios["%s->%s" % (src, dst)] = R.ratio(got, ref, err)
    print("\n%s conv_tc=%d max |got - ref| / bound: %s" % (name, conv_tc, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mos_skipcnn_skip_m40_s17_avg", "dim_skipcnn_fc256_m96_s31", "mos_dff_m64_s9"])
def test_ff_framewise_against_float64(built_lib, name):
    """SkipCNN / DFF: MEL_DB -> the framewise rows in float64.  Behind no td the rows are TD_OUT; behind self-attention
    the check runs through td's input Linear + LayerNorm (TD_IN)."""
    args, sd = _variant(name)
    lens = [1, 30, 97, 3]
    N = sum(lens)
    skip = args["td"] == "skip"
    eng = _engine(args, sd)
    try:
        seg, d = _stage_dumps(eng, args, lens, 700, {"rows": E.STAGE_TD_OUT if skip else E.STAGE_TD_IN})
    finally:
        eng.close()
    rows = d["rows"].reshape(N, -1)
    p = "cnn.model."
    bn = "bn." if args["cnn_model"] == "skip" else "bn1."
    a = float(sd[p + bn + "weight"]) / np.sqrt(float(sd[p + bn + "running_var"]) + 1e-5)
    c = float(sd[p + bn + "bias"]) - float(sd[p + bn + "running_mean"]) * a
    x = seg.reshape(N, -1) * a + c                    # x.view(-1, n_mels * seg_len) after BatchNorm2d(1)
    err = R.TAU * (seg.reshape(N, -1).abs() * abs(a) + abs(c))
    if args["cnn_model"] == "dff":
        for i in range(1, 5):
            b = p + "bn%d." % (i + 1)
            s = R._d(sd[b + "weight"]) / torch.sqrt(R._d(sd[b + "running_var"]) + 1e-5)
            w = R._d(sd[p + "lin%d.weight" % i]) * s[:, None]
            bias = (R._d(sd[p + "lin%d.bias" % i]) - R._d(sd[b + "running_mean"])) * s + R._d(sd[b + "bias"])
            x, err = R.linear(x, err, w, bias)
            x = torch.relu(x)                         # (1-Lipschitz: the bound carries over)
    elif p + "linear.weight" in sd:
        x, err = R.linear(x, err, sd[p + "linear.weight"], sd[p + "linear.bias"])
    if not skip:
        x, err = R.td_in(sd, x, err)
    assert rows.shape == x.shape
    r = R.ratio(rows, x, err)
    print("\n%s mel -> %s max |got - ref| / bound: %.3g" % (name, "td_out" if skip else "td_in", r))
    assert r <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mos_adapt_m64_s15", "dim_adapt_m32_s11"])
def test_conv_paths_agree_on_other_shapes(built_lib, name):
    """conv2..6 on the tensor cores (fp16 two-term split) against the fp32 FFMA kernels: fp32 noise apart"""
    args, sd = _variant(name)
    clips = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.MEL_CLIPS] + [_pcm(args, 97, 3)]
    srs = [c[2] for c in V.MEL_CLIPS] + [SR]
    out = {}
    for tc in (1, 0):
        eng = E.Engine(E.config_from_args(args), 0)
        try:
            eng.set_option("conv_tc", tc)
            eng.load_state_dict(sd)
            sc, _, _ = eng.predict_pcm(clips, srs)
            out[tc] = (sc, eng.stage_dump(E.STAGE_POOL1), eng.stage_dump(E.STAGE_CNN_FEAT))
        finally:
            eng.close()
    # the same conv1 kernel on both paths (the tensor-core path stores it as an fp16 hi / lo pair: about 2^-22 of the
    # value, and of the layer's scale for small values)
    np.testing.assert_allclose(out[1][1], out[0][1], rtol=2.0 ** -20, atol=2.0 ** -22 * float(np.abs(out[0][1]).max()))
    feat_err = float(np.abs(out[1][2] - out[0][2]).max() / max(1.0, np.abs(out[0][2]).max()))
    score_err = float(np.abs(out[1][0] - out[0][0]).max())
    print("\n%s: tc vs ffma: features %.3g (relative), scores %.3g" % (name, feat_err, score_err))
    assert feat_err <= 1e-5 and score_err <= 1e-5


@pytest.mark.gpu
def test_load_weights_refuses_a_linear_of_the_shipped_width(built_lib):
    """a SkipCNN Linear of the 48 x 15 fan_in does not load into a 40 x 15 engine"""
    args, sd = _variant("mos_skipcnn_m40_s15_sa")
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        with pytest.raises(E.EngineError, match=r"\(-3\).*time_dependency\.model\.linear\.weight"):
            eng.load_state_dict(dict(sd, **{"time_dependency.model.linear.weight": torch.zeros(64, 720)}))
    finally:
        eng.close()


@pytest.mark.gpu
def test_predict_dir_runs_a_64_band_checkpoint_end_to_end(built_lib, tmp_path):
    """A torch.save'd 64-band checkpoint scored through nisqaModel(mode='predict_dir') writes NISQA_results.csv with the
    Engine's scores."""
    import pandas as pd
    from nisqa_b200.NISQA_model import nisqaModel
    args, sd = _variant("mos_adapt_m64_s15")
    ck = str(tmp_path / "m64.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    d = tmp_path / "wavs"
    d.mkdir()
    out_dir = tmp_path / "out"
    out_dir.mkdir()
    pcm = {}
    for seed, sec, sr in V.MEL_CLIPS:
        fn = "m%03d.wav" % seed
        pcm[fn] = (synth.synth_speech_pcm16(seed, sec, sr), sr)
        wav.write_wav_pcm16(str(d / fn), *pcm[fn])
    nisqaModel({"mode": "predict_dir", "pretrained_model": ck, "data_dir": str(d), "output_dir": str(out_dir),
                "tr_bs_val": 2, "tr_num_workers": 0, "ms_channel": None}).predict()
    df = pd.read_csv(out_dir / "NISQA_results.csv")
    assert sorted(df["deg"]) == sorted(pcm)
    eng = _engine(args, sd)
    try:
        for _, row in df.iterrows():
            p, sr = pcm[row["deg"]]
            want, _, _ = eng.predict_pcm([p], [sr])
            np.testing.assert_allclose(row["mos_pred"], want[0, 0], rtol=0, atol=1e-5, err_msg=row["deg"])
    finally:
        eng.close()

