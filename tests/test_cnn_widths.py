"""AdaptCNN checkpoints trained with other channel counts: cnn_c_out_1 / cnn_c_out_2 / cnn_c_out_3 each 16, 32 or 64 (the
engine reads them from the conv / bn tensors), behind self-attention, no td, AdaptCNN's Linear, other Mel-spectrogram
shapes and NISQA_DE.

CPU: config_from_args accepts all 27 triples behind every framewise / td combination and refuses any other count (and
StandardCNN at anything but 16 / 32 / 64), naming the field and value; the oracle against the scores of the unmodified
reference modules (tests/golden/variants_cnn_width.npz, oracle/make_cnn_width_golden.py).
GPU: every width variant through the C ABI against the reference scores and the oracle (a one-segment and a 97-segment
clip, 8 kHz and 48 kHz clips, PCM16 and float input), alone == in a batch, several passes == one pass; all 27 triples
against the oracle on seeded weights; stage bounds from the engine's own dumps (tests/stage_ref.py); power-of-two
rescaling; weights of other channel counts reloaded into one engine == a fresh engine, and no stage dump of the previous
layout after such a reload; the refusals of nisqa_load_weights and of the FFMA path (conv_tc=0); one checkpoint end to
end through nisqaModel(mode='predict_dir').
"""
import os

import numpy as np
import pytest
import torch

import stage_ref as R
from conftest import GOLDEN, WEIGHTS
from rescale import rescale
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from oracle import cnn_width_variants as V
from oracle import nisqa_oracle as O
from oracle import td_pair_oracle as TO
from oracle.td_pair_variants import _pool, sa
from oracle.variants import de_pair_pcm

SCORE_TOL = 1e-4
SR = 16000


def _variant(name):
    base = V.CNN_WIDTH_VARIANTS[name][0]
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.cnn_width_checkpoint(name, args, sd)


def _args(ckpt, **over):
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    return dict(args, **over)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


def _oracle(args, sd, pcm, sr):
    with V.wide_cnn():
        return TO.predict_pcm(args, sd, pcm, sr)


def _oracle_de(args, sd, deg, srd, ref, srr):
    with V.wide_cnn():
        return O.predict_pcm_de(args, sd, deg, srd, ref, srr)


# ------------------------------------------------------------------------------------------------------------ CPU
def _adapt_args():
    """every AdaptCNN combination that takes other channel counts"""
    mos, dim = _args("nisqa_mos_only.tar"), _args("nisqa.tar")
    de, _ = _variant("de_c16_32_32")
    return {"sa": mos, "dim_sa": dim, "fc": dict(mos, cnn_fc_out_h=128), "sa_sa": dict(mos, **sa("td_2", 64, 64)),
            "skip": dict(mos, td="skip", td_2="skip", **_pool("avg")), "skip_sa": dict(mos, td="skip", **sa("td_2", 64, 64)),
            "mel": dict(mos, ms_n_mels=64, ms_seg_length=21), "de": de}


def test_config_accepts_every_triple():
    for kind, args in _adapt_args().items():
        for c1, c2, c3 in V.TRIPLES:
            c = E.config_from_args(dict(args, cnn_c_out_1=c1, cnn_c_out_2=c2, cnn_c_out_3=c3))
            assert c.cnn_kind == E.CNN_CONV, kind
    for name in V.CNN_WIDTH_VARIANTS:
        args, _ = _variant(name)
        E.config_from_args(args)


def test_config_refuses_other_counts_naming_them():
    for kind, args in _adapt_args().items():
        for i in (1, 2, 3):
            for bad in (8, 24, 48, 128):
                with pytest.raises(NotImplementedError, match=r"cnn_c_out_%d=%d: the engine runs AdaptCNN channel counts 16, 32 "
                                                              r"or 64" % (i, bad)):
                    E.config_from_args(dict(args, **{"cnn_c_out_%d" % i: bad}))
    # StandardCNN keeps its shipped counts
    tts = _args("nisqa_tts.tar")
    for i, bad in ((1, 32), (2, 16), (3, 32)):
        with pytest.raises(NotImplementedError, match=r"cnn_c_out_1/2/3=.*StandardCNN with 16, 32, 64"):
            E.config_from_args(dict(tts, **{"cnn_c_out_%d" % i: bad}))


def test_oracle_matches_reference_modules_on_the_width_variants():
    g = np.load(os.path.join(GOLDEN, "variants_cnn_width.npz"))
    assert sorted(g.files) == sorted(V.CNN_WIDTH_VARIANTS)
    for name in V.CNN_WIDTH_VARIANTS:
        args, sd = _variant(name)
        if args["model"] == "NISQA_DE":
            for i, pair in enumerate(V.WIDTH_DE_PAIRS):
                deg, srd, ref, srr = de_pair_pcm(pair)
                sc, _, st = _oracle_de(args, sd, _f32(deg), srd, _f32(ref), srr)
                assert st == O.STATUS_OK
                np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)
            continue
        for i, (seed, sec, sr) in enumerate(V.WIDTH_CLIPS):
            sc, _, st = _oracle(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


def test_width_oracle_is_the_shipped_oracle_at_the_shipped_widths():
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    x = O.segments(torch.from_numpy(np.asarray(O.mel_db(_f32(synth.synth_speech_pcm16(5, 1.5, SR)), SR, args))), args)
    with torch.no_grad():
        np.testing.assert_array_equal(V.adapt_cnn(sd, x, args).numpy(), O.adapt_cnn(sd, x, args).numpy())


def test_golden_scores_lie_in_the_mos_range():
    g = np.load(os.path.join(GOLDEN, "variants_cnn_width.npz"))
    for name in g.files:
        n = len(V.WIDTH_DE_PAIRS) if name.startswith("de_") else len(V.WIDTH_CLIPS)
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


SINGLE = [n for n in V.CNN_WIDTH_VARIANTS if not n.startswith("de_")]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["pcm16", "f32"])
@pytest.mark.parametrize("name", SINGLE)
def test_width_variant_through_the_c_abi(built_lib, name, fmt):
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_cnn_width.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.WIDTH_CLIPS]
    srs = [c[2] for c in V.WIDTH_CLIPS]
    # one segment between long clips, 97 segments, an 8 kHz and a 48 kHz clip
    extra = [_pcm(args, 1, 7), _pcm(args, 97, 8), synth.synth_speech_pcm16(9, 1.3, 8000), synth.synth_speech_pcm16(10, 0.8, 48000)]
    esr = [SR, SR, 8000, 48000]
    batch = pcm[:2] + extra[:1] + pcm[2:] + extra[1:]
    bsr = srs[:2] + esr[:1] + srs[2:] + esr[1:]
    if fmt == "f32":
        batch = [_f32(p) for p in batch]
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
            ref, ns, st = _oracle(args, sd, p if fmt == "f32" else _f32(p), sr)
            assert st == O.STATUS_OK and ns == nseg[i], (name, i)
            worst = max(worst, float(np.abs(scores[i] - ref).max()))
        print("%s %s: max |engine - oracle| %.3g over segment counts %s" % (name, fmt, worst, nseg.tolist()))
        assert worst <= SCORE_TOL, (name, worst)
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
def test_double_ended_width_variant_through_the_c_abi(built_lib):
    name = "de_c16_32_32"
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_cnn_width.npz"))[name]
    clips, srs, refs = [], [], []
    for pair in V.WIDTH_DE_PAIRS:
        deg, srd, ref, srr = de_pair_pcm(pair)
        clips += [deg, ref]
        srs += [srd, srr]
        refs.append(_oracle_de(args, sd, _f32(deg), srd, _f32(ref), srr)[0])
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
def test_every_triple_against_the_oracle(built_lib):
    """all 27 (c1, c2, c3) on seeded weights (nisqa_mos_only.tar's td and pooling), 1- and 40-segment clips and a 48 kHz one"""
    base_args, base_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    clips = [_pcm(base_args, 1, 21), _pcm(base_args, 40, 22), synth.synth_speech_pcm16(23, 1.1, 48000)]
    srs = [SR, SR, 48000]
    worst = {}
    for widths in V.TRIPLES:
        args, sd = V.triple_checkpoint(base_args, base_sd, widths)
        eng = _engine(args, sd)
        try:
            scores, _, status = eng.predict_pcm(clips, srs)
        finally:
            eng.close()
        assert np.all(status == E.CLIP_OK)
        ref = np.stack([_oracle(args, sd, _f32(p), sr)[0] for p, sr in zip(clips, srs)])
        worst[widths] = float(np.abs(scores - ref).max())
    print("\nmax |engine - oracle| per triple: %s" % worst)
    assert max(worst.values()) <= SCORE_TOL, worst


def _stage_dumps(eng, args, lens, seed, stages):
    clips = [_pcm(args, n, seed + i) for i, n in enumerate(lens)]
    scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
    assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
    return {k: torch.from_numpy(eng.stage_dump(st)).double() for k, st in stages.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("widths", [(16, 16, 16), (64, 32, 16), (16, 64, 32), (64, 64, 64), (32, 16, 64)])
def test_stages_against_float64(built_lib, widths):
    """POOL1 -> POOL2 -> CONV3 -> POOL3 -> CONV5 -> CNN_FEAT against float64 from the engine's own dumps (bound TAU =
    2^-18 times the magnitude of the stage's terms, tests/stage_ref.py).  A tile holds 1 (24 x 7 maps), 3 (12 x 5) or 9
    (6 x 3) consecutive segments of the pass, clips concatenated: nine batches of 165..173 segments leave every remainder
    of the last tile, 0..8 of 9 and 0..2 of 3."""
    base_args, base_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    args, sd = V.triple_checkpoint(base_args, base_sd, widths)
    c1, c2, c3 = widths
    shapes = {"pool1": (E.STAGE_POOL1, (c1, 24, 7)), "pool2": (E.STAGE_POOL2, (c2, 12, 5)), "conv3": (E.STAGE_CONV3, (c3, 12, 5)),
              "pool3": (E.STAGE_POOL3, (c3, 6, 3)), "conv5": (E.STAGE_CONV5, (c3, 6, 3))}
    chain = [("pool1", "pool2", 2), ("pool2", "conv3", 3), ("conv3", "pool3", 4), ("pool3", "conv5", 5), ("conv5", "cnn_feat", 6)]
    ratios = {"%s->%s" % (src, dst): 0.0 for src, dst, _ in chain}
    remainders = set()
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        eng.set_option("conv12", 0)              # (POOL1 lives in shared memory on the fused path)
        eng.load_state_dict(sd)
        stages = {k: v[0] for k, v in shapes.items()}
        stages["cnn_feat"] = E.STAGE_CNN_FEAT
        for extra in range(1, 10):
            lens = [1, 13, 97, 2, 40, 5, 6, extra]
            N = sum(lens)
            remainders.add(N % 9)
            d = _stage_dumps(eng, args, lens, 800 + 10 * extra, stages)
            act = {k: d[k].reshape(N, *shapes[k][1]) for k in shapes}
            feat = d["cnn_feat"].reshape(N, -1)
            assert feat.shape[1] == 6 * c3
            for src, dst, layer in chain:
                ref, err = R.conv_layer(sd, args, layer, act[src])
                if dst == "cnn_feat":
                    ref, err = R.cnn_tail({k: v for k, v in sd.items() if not k.startswith("cnn.model.fc.")}, args, ref, err)
                got = feat if dst == "cnn_feat" else act[dst]
                key = "%s->%s" % (src, dst)
                ratios[key] = max(ratios[key], R.ratio(got, ref, err))
    finally:
        eng.close()
    assert remainders == set(range(9))
    print("\n%s max |got - ref| / bound: %s" % (widths, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


@pytest.mark.gpu
def test_reloading_other_channel_counts_equals_a_fresh_engine(built_lib):
    """One engine, weights of other channel counts loaded one after the other (the plane pairs change their row width,
    and their zero rows / columns must be zero again): every load scores bit for bit like a fresh engine with those
    weights, on the fused conv1 + conv2 path and on the separate one."""
    base_args, base_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    clips = [_pcm(base_args, 1, 51), _pcm(base_args, 60, 52), synth.synth_speech_pcm16(53, 2.5, 48000), _pcm(base_args, 9, 54)]
    srs = [SR, SR, 48000, SR]
    seq = [None, (16, 16, 16), (64, 32, 16), (64, 64, 64), (16, 16, 16), None]      # None: the shipped weights
    ckpts = [(base_args, base_sd) if w is None else V.triple_checkpoint(base_args, base_sd, w) for w in seq]
    for conv12 in (1, 0):
        fresh = []
        for args, sd in ckpts:
            eng = E.Engine(E.config_from_args(args), 0)
            try:
                eng.set_option("conv12", conv12)
                eng.load_state_dict(sd)
                fresh.append(eng.predict_pcm(clips, srs)[0])
            finally:
                eng.close()
        eng = E.Engine(E.config_from_args(ckpts[0][0]), 0)
        try:
            eng.set_option("conv12", conv12)
            for i, (args, sd) in enumerate(ckpts):
                eng.load_state_dict(sd)
                got, _, status = eng.predict_pcm(clips, srs)
                assert np.all(status == E.CLIP_OK)
                np.testing.assert_array_equal(got, fresh[i], err_msg="load %d %s conv12=%d" % (i, seq[i], conv12))
        finally:
            eng.close()


@pytest.mark.gpu
def test_stage_dump_after_a_reload_of_other_channel_counts_is_refused(built_lib):
    """the last pass's maps were laid out for the previous channel counts: no dump of them through the new layout"""
    base_args, base_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    eng = E.Engine(E.config_from_args(base_args), 0)
    try:
        eng.set_option("conv12", 0)
        eng.load_state_dict(base_sd)
        eng.predict_pcm([_pcm(base_args, 5, 61)], [SR])
        assert eng.stage_dump(E.STAGE_POOL2).size == 5 * 32 * 12 * 5
        eng.load_state_dict(V.triple_checkpoint(base_args, base_sd, (16, 64, 64))[1])
        with pytest.raises(E.EngineError, match=r"\(-4\).*stage dump needs a predict call"):
            eng.stage_dump(E.STAGE_POOL2)
        eng.predict_pcm([_pcm(base_args, 5, 61)], [SR])
        assert eng.stage_dump(E.STAGE_POOL2).size == 5 * 64 * 12 * 5
    finally:
        eng.close()


@pytest.mark.gpu
def test_rescaled_batchnorm_leaves_the_scores_bit_identical(built_lib):
    """BatchNorm i times 2^k, its consumer times 2^-k: the fp16 split keeps every stored value, so the scores are
    bit-identical (64 / 32 / 16: 96 features, conv2 with one activation buffer)"""
    args, sd = _variant("mos_c64_32_16")
    clips = [_pcm(args, 1, 31), _pcm(args, 37, 32), synth.synth_speech_pcm16(33, 2.2, 48000)]
    srs = [SR, SR, 48000]
    eng = _engine(args, sd)
    try:
        base, _, _ = eng.predict_pcm(clips, srs)
        for layer in range(1, 7):
            for k in (-3, 5):
                eng.load_state_dict(rescale(sd, layer, k))
                got, _, _ = eng.predict_pcm(clips, srs)
                np.testing.assert_array_equal(got, base, err_msg="bn%d x 2^%d" % (layer, k))
    finally:
        eng.close()


@pytest.mark.gpu
def test_load_weights_names_the_tensor_it_refuses(built_lib):
    args, sd = _variant("mos_c16_64_32")
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        bad = dict(sd, **{"cnn.model.conv3.weight": torch.zeros(48, 64, 3, 3)})
        with pytest.raises(E.EngineError, match=r"\(-3\).*cnn\.model\.conv3\.weight: 48 output channels \(cnn_c_out_3\)"):
            eng.load_state_dict(bad)
        with pytest.raises(E.EngineError, match=r"\(-3\).*cnn\.model\.conv4\.weight"):
            eng.load_state_dict(dict(sd, **{"cnn.model.conv4.weight": torch.zeros(64, 32, 3, 3)}))
        with pytest.raises(E.EngineError, match=r"\(-3\).*time_dependency\.model\.linear\.weight"):
            eng.load_state_dict(dict(sd, **{"time_dependency.model.linear.weight": torch.zeros(64, 384)}))
    finally:
        eng.close()


@pytest.mark.gpu
def test_ffma_path_refuses_other_channel_counts(built_lib):
    """conv_tc=0 (the fp32 FFMA convolutions, kept for A/B) runs the shipped counts only and says so"""
    args, sd = _variant("mos_c16_16_16")
    eng = _engine(args, sd)
    try:
        eng.set_option("conv_tc", 0)
        with pytest.raises(E.EngineError, match=r"\(-4\).*conv_tc=0.*16 / 16 / 16"):
            eng.predict_pcm([_pcm(args, 3, 41)], [SR])
        eng.set_option("conv_tc", 1)
        _, _, status = eng.predict_pcm([_pcm(args, 3, 41)], [SR])
        assert status[0] == E.CLIP_OK
    finally:
        eng.close()


@pytest.mark.gpu
def test_predict_dir_runs_a_width_checkpoint_end_to_end(built_lib, tmp_path):
    import pandas as pd
    from nisqa_b200.NISQA_model import nisqaModel
    args, sd = _variant("mos_c16_64_32")
    ck = str(tmp_path / "w.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    d = tmp_path / "wavs"
    d.mkdir()
    out_dir = tmp_path / "out"
    out_dir.mkdir()
    pcm = {}
    for seed, sec, sr in V.WIDTH_CLIPS:
        fn = "w%03d.wav" % seed
        pcm[fn] = (synth.synth_speech_pcm16(seed, sec, sr), sr)
        wav.write_wav_pcm16(str(d / fn), *pcm[fn])
    nisqaModel({"mode": "predict_dir", "pretrained_model": ck, "data_dir": str(d), "output_dir": str(out_dir),
                "tr_bs_val": 2, "tr_num_workers": 0, "ms_channel": None}).predict()
    df = pd.read_csv(out_dir / "NISQA_results.csv")
    assert sorted(df["deg"]) == sorted(pcm)
    g = np.load(os.path.join(GOLDEN, "variants_cnn_width.npz"))["mos_c16_64_32"]
    eng = _engine(args, sd)
    try:
        for _, row in df.iterrows():
            p, sr = pcm[row["deg"]]
            want, _, _ = eng.predict_pcm([p], [sr])
            np.testing.assert_allclose(row["mos_pred"], want[0, 0], rtol=0, atol=1e-5, err_msg=row["deg"])
        assert np.abs(np.sort(df["mos_pred"].to_numpy()) - np.sort(g[:, 0])).max() <= SCORE_TOL
    finally:
        eng.close()
