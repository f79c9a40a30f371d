"""AdaptCNN checkpoints trained with other adaptive max-pool sizes: cnn_pool_1 / cnn_pool_2 / cnn_pool_3 (the engine takes
them through nisqa_set_cnn_pools, config_from_args attaches them as cfg.cnn_pools), behind self-attention, no td,
AdaptCNN's Linear, other Mel-spectrogram shapes and channel counts, and NISQA_DE.

CPU: config_from_args accepts every table entry and refuses out-of-bound pools, the fan-out bound and other AdaptCNN kernel
sizes, naming the field and value; the header and the binding carry nisqa_set_cnn_pools; the oracle against the scores of
the unmodified reference modules (tests/golden/variants_cnn_pool.npz, oracle/make_cnn_pool_golden.py).
GPU: every pool variant through the C ABI against the reference scores and the oracle (a one-segment and a 97-segment
clip, 8 kHz and 48 kHz clips, PCM16 and float input), alone == in a batch, several passes == one pass; the stage dumps'
shapes and float64 stage bounds (tests/stage_ref.py); one engine reloading other pools; the refusals of
nisqa_set_cnn_pools, nisqa_load_weights and the FFMA path (conv_tc=0); one checkpoint end to end through
nisqaModel(mode='predict_dir').
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import stage_ref as R
from conftest import GOLDEN, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from oracle import cnn_pool_variants as V
from oracle import cnn_width_variants as W
from oracle import nisqa_oracle as O
from oracle import td_pair_oracle as TO
from oracle.td_pair_variants import _pool, sa
from oracle.variants import de_pair_pcm

SCORE_TOL = 1e-4
SR = 16000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _variant(name):
    base = V.CNN_POOL_VARIANTS[name][0]
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.cnn_pool_checkpoint(name, args, sd)


def _args(ckpt, **over):
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    return dict(args, **over)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


def _oracle(args, sd, pcm, sr):
    with W.wide_cnn():
        return TO.predict_pcm(args, sd, pcm, sr)


def _oracle_de(args, sd, deg, srd, ref, srr):
    with W.wide_cnn():
        return O.predict_pcm_de(args, sd, deg, srd, ref, srr)


def _pools(args):
    return tuple(tuple(args["cnn_pool_%d" % i]) for i in (1, 2, 3))


# ------------------------------------------------------------------------------------------------------------ CPU
def test_config_accepts_every_variant_and_carries_its_pools():
    for name in V.CNN_POOL_VARIANTS:
        args, _ = _variant(name)
        c = E.config_from_args(args)
        assert c.cnn_kind == E.CNN_CONV, name
        assert c.cnn_pools == _pools(args), name
    # the shipped pools: nothing to attach
    for ck in ("nisqa.tar", "nisqa_mos_only.tar"):
        c = E.config_from_args(_args(ck))
        assert getattr(c, "cnn_pools", E.SHIPPED_POOLS) == E.SHIPPED_POOLS


def test_config_accepts_the_bounds_behind_every_td():
    mos = _args("nisqa_mos_only.tar")
    kinds = {"sa": mos, "fc": dict(mos, cnn_fc_out_h=128), "sa_sa": dict(mos, **sa("td_2", 64, 64)),
             "skip": dict(mos, td="skip", td_2="skip", **_pool("avg")), "skip_sa": dict(mos, td="skip", **sa("td_2", 64, 64)),
             "mel": dict(mos, ms_n_mels=64, ms_seg_length=21), "dim": _args("nisqa.tar")}
    edge = [([1, 1], [1, 1], [1, 1]), ([16, 14], [127, 1], [63, 1]), ([24, 7], [12, 5], [63, 3])]
    for kind, args in kinds.items():
        for p in edge:
            c = E.config_from_args(dict(args, cnn_pool_1=p[0], cnn_pool_2=p[1], cnn_pool_3=p[2]))
            assert c.cnn_pools == tuple(map(tuple, p)), (kind, p)


def test_config_refuses_out_of_bound_pools_naming_them():
    mos = _args("nisqa_mos_only.tar")
    for key in ("cnn_pool_1", "cnn_pool_2", "cnn_pool_3"):
        for bad in ([32, 7], [48, 7], [4, 15], [0, 3], [3, 0], [127, 2]):
            with pytest.raises(NotImplementedError, match=r"%s=\[%d, %d\]: the engine runs AdaptCNN pool sizes \[h, w\] with "
                                                          r"w <= 14 and \(h \+ 1\) \* \(w \+ 1\) <= 256" % ((key,) + tuple(bad))):
                E.config_from_args(dict(mos, **{key: bad}))
    for bad in ([6, 5], [6, 4], [2, 14]):
        with pytest.raises(NotImplementedError, match=r"cnn_pool_3=\[%d, %d\]: the engine runs pool_3 widths 1 to 3 "
                                                      r"\(conv6's kernel is 3 x pool_3\[1\]\)" % tuple(bad)):
            E.config_from_args(dict(mos, cnn_pool_3=bad))
    with pytest.raises(NotImplementedError, match=r"cnn_c_out_3=64, cnn_pool_3=\[65, 2\]: the engine runs up to 4096 framewise "
                                                  r"features \(cnn_c_out_3 \* cnn_pool_3\[0\] = 4160\)"):
        E.config_from_args(dict(mos, cnn_pool_3=[65, 2]))
    E.config_from_args(dict(mos, cnn_pool_3=[64, 2]))
    E.config_from_args(dict(mos, cnn_c_out_3=32, cnn_pool_3=[84, 1]))


def test_config_names_other_adapt_kernel_sizes():
    mos = _args("nisqa_mos_only.tar")
    for ks in (5, (5, 5), [3, 5]):
        with pytest.raises(NotImplementedError, match=re.escape("cnn_kernel_size=%r: the engine runs 3x3 convolutions" % (ks,))):
            E.config_from_args(dict(mos, cnn_kernel_size=ks))


def test_every_refusal_names_its_field():
    src = open(os.path.join(ROOT, "nisqa_b200", "engine.py")).read()
    assert "outside the shipped NISQA configurations" not in src


def test_header_declares_and_binding_exports_set_cnn_pools():
    hdr = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    assert "NISQA_API int  nisqa_set_cnn_pools(nisqa_engine* e, const int32_t pools[6]);" in hdr
    assert "nisqa_set_cnn_pools" in E.EXPORTS


def test_oracle_matches_reference_modules_on_the_pool_variants():
    g = np.load(os.path.join(GOLDEN, "variants_cnn_pool.npz"))
    assert sorted(g.files) == sorted(V.CNN_POOL_VARIANTS)
    for name in V.CNN_POOL_VARIANTS:
        args, sd = _variant(name)
        if args["model"] == "NISQA_DE":
            for i, pair in enumerate(V.POOL_DE_PAIRS):
                deg, srd, ref, srr = de_pair_pcm(pair)
                sc, _, st = _oracle_de(args, sd, _f32(deg), srd, _f32(ref), srr)
                assert st == O.STATUS_OK
                np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)
            continue
        for i, (seed, sec, sr) in enumerate(V.POOL_CLIPS):
            sc, _, st = _oracle(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


def test_golden_scores_lie_in_the_mos_range():
    g = np.load(os.path.join(GOLDEN, "variants_cnn_pool.npz"))
    for name in g.files:
        n = len(V.POOL_DE_PAIRS) if name.startswith("de_") else len(V.POOL_CLIPS)
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


SINGLE = [n for n in V.CNN_POOL_VARIANTS if not n.startswith("de_")]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["pcm16", "f32"])
@pytest.mark.parametrize("name", SINGLE)
def test_pool_variant_through_the_c_abi(built_lib, name, fmt):
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_cnn_pool.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.POOL_CLIPS]
    srs = [c[2] for c in V.POOL_CLIPS]
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
def test_double_ended_pool_variant_through_the_c_abi(built_lib):
    name = "de_p16x7_8x4_4x3"
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_cnn_pool.npz"))[name]
    clips, srs, refs = [], [], []
    for pair in V.POOL_DE_PAIRS:
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
@pytest.mark.parametrize("name", ["mos_p16x5_8x4_4x2", "mos_p24x7_12x5_6x1", "mos_p24x7_12x9_6x3", "mos_m128_p30x7_15x5_5x3",
                                  "mos_c16_32_32_p12x7_6x5_3x3"])
def test_stages_against_float64(built_lib, name):
    """POOL1 -> POOL2 -> CONV3 -> POOL3 -> CONV5 -> CNN_FEAT have the pools' shapes and stay within float64 bounds (TAU =
    2^-18 times the magnitude of the stage's terms, tests/stage_ref.py), over batches whose segment counts leave several
    remainders of the last tile"""
    args, sd = _variant(name)
    c1, c2, c3 = (args["cnn_c_out_%d" % i] for i in (1, 2, 3))
    (h1, w1), (h2, w2), (h3, w3) = _pools(args)
    shapes = {"pool1": (E.STAGE_POOL1, (c1, h1, w1)), "pool2": (E.STAGE_POOL2, (c2, h2, w2)), "conv3": (E.STAGE_CONV3, (c3, h2, w2)),
              "pool3": (E.STAGE_POOL3, (c3, h3, w3)), "conv5": (E.STAGE_CONV5, (c3, h3, w3))}
    chain = [("pool1", "pool2", 2), ("pool2", "conv3", 3), ("conv3", "pool3", 4), ("pool3", "conv5", 5), ("conv5", "cnn_feat", 6)]
    ratios = {"%s->%s" % (src, dst): 0.0 for src, dst, _ in chain}
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        eng.set_option("conv12", 0)
        eng.load_state_dict(sd)
        stages = {k: v[0] for k, v in shapes.items()}
        stages["cnn_feat"] = E.STAGE_CNN_FEAT
        for extra in range(1, 6):
            lens = [1, 13, 97, 2, 40, 5, extra]
            N = sum(lens)
            clips = [_pcm(args, n, 900 + 10 * extra + i) for i, n in enumerate(lens)]
            _, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
            assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
            d = {k: torch.from_numpy(eng.stage_dump(st)).double() for k, st in stages.items()}
            for k in shapes:
                assert d[k].numel() == N * int(np.prod(shapes[k][1])), k
            act = {k: d[k].reshape(N, *shapes[k][1]) for k in shapes}
            feat = d["cnn_feat"].reshape(N, -1)
            assert feat.shape[1] == c3 * h3
            for src, dst, layer in chain:
                ref, err = R.conv_layer(sd, args, layer, act[src])
                if dst == "cnn_feat":
                    ref, err = R.cnn_tail({k: v for k, v in sd.items() if not k.startswith("cnn.model.fc.")}, args, ref, err)
                got = feat if dst == "cnn_feat" else act[dst]
                key = "%s->%s" % (src, dst)
                ratios[key] = max(ratios[key], R.ratio(got, ref, err))
    finally:
        eng.close()
    print("\n%s max |got - ref| / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


@pytest.mark.gpu
def test_reloading_other_pools_matches_each_goldens(built_lib):
    """One engine loads pools [16, 5] [8, 4] [4, 2], then [24, 7] [12, 9] [6, 3], then the shipped nisqa_mos_only.tar, then
    the first again; a NISQA_DIM engine loads [24, 7] [12, 5] [12, 3], then the shipped nisqa.tar.  The plane pairs are
    cleared again whenever the maps move, so every load scores its own goldens (the shipped weights: the oracle)."""
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.POOL_CLIPS]
    srs = [c[2] for c in V.POOL_CLIPS]
    a1, sd1 = _variant("mos_p16x5_8x4_4x2")
    a2, sd2 = _variant("mos_p24x7_12x9_6x3")
    base_args, base_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    g = np.load(os.path.join(GOLDEN, "variants_cnn_pool.npz"))
    want_base = np.stack([_oracle(base_args, base_sd, _f32(p), sr)[0] for p, sr in zip(pcm, srs)])
    eng = E.Engine(E.config_from_args(a1), 0)
    try:
        for args, sd, want in ((a1, sd1, g["mos_p16x5_8x4_4x2"]), (a2, sd2, g["mos_p24x7_12x9_6x3"]),
                               (base_args, base_sd, want_base), (a1, sd1, g["mos_p16x5_8x4_4x2"])):
            eng.set_cnn_pools(_pools(args))
            eng.load_state_dict(sd)
            got, _, status = eng.predict_pcm(pcm, srs)
            assert np.all(status == E.CLIP_OK)
            assert np.abs(got - want).max() <= SCORE_TOL, (_pools(args), float(np.abs(got - want).max()))
    finally:
        eng.close()
    # NISQA_DIM: variant 3, then the shipped nisqa.tar
    a3, sd3 = _variant("dim_p24x7_12x5_12x3")
    dim_args, dim_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    want_dim = np.stack([_oracle(dim_args, dim_sd, _f32(p), sr)[0] for p, sr in zip(pcm, srs)])
    eng = E.Engine(E.config_from_args(a3), 0)
    try:
        for args, sd, want in ((a3, sd3, g["dim_p24x7_12x5_12x3"]), (dim_args, dim_sd, want_dim)):
            eng.set_cnn_pools(_pools(args))
            eng.load_state_dict(sd)
            got, _, _ = eng.predict_pcm(pcm, srs)
            assert np.abs(got - want).max() <= SCORE_TOL, _pools(args)
    finally:
        eng.close()


@pytest.mark.gpu
def test_stage_dump_after_a_reload_of_other_pools_is_refused(built_lib):
    base_args, base_sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    a1, sd1 = _variant("mos_p16x5_8x4_4x2")
    eng = E.Engine(E.config_from_args(base_args), 0)
    try:
        eng.set_option("conv12", 0)
        eng.load_state_dict(base_sd)
        eng.predict_pcm([_pcm(base_args, 5, 61)], [SR])
        assert eng.stage_dump(E.STAGE_POOL2).size == 5 * 32 * 12 * 5
        eng.set_cnn_pools(_pools(a1))
        eng.load_state_dict(sd1)
        with pytest.raises(E.EngineError, match=r"\(-4\).*stage dump needs a predict call"):
            eng.stage_dump(E.STAGE_POOL2)
        eng.predict_pcm([_pcm(base_args, 5, 61)], [SR])
        assert eng.stage_dump(E.STAGE_POOL2).size == 5 * 32 * 8 * 4
    finally:
        eng.close()


@pytest.mark.gpu
def test_refusals_name_the_field(built_lib):
    args, sd = _variant("mos_p16x5_8x4_4x2")
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        for bad, msg in (((32, 7, 12, 5, 6, 3), r"cnn_pool_1=\[32, 7\]: the engine runs AdaptCNN pool sizes"),
                         ((24, 7, 4, 15, 6, 3), r"cnn_pool_2=\[4, 15\]: the engine runs AdaptCNN pool sizes"),
                         ((24, 7, 12, 5, 6, 5), r"cnn_pool_3=\[6, 5\]: the engine runs pool_3 widths 1 to 3")):
            flat = (C.c_int32 * 6)(*bad)
            assert eng.lib.nisqa_set_cnn_pools(eng.h, flat) == -1
            assert re.search(msg, eng._err()), eng._err()
        # a conv6 of the wrong width: the weights were trained with another pool_3
        bad = dict(sd, **{"cnn.model.conv6.weight": torch.zeros(64, 64, 3, 3)})
        with pytest.raises(E.EngineError, match=r"\(-3\).*cnn\.model\.conv6\.weight"):
            eng.load_state_dict(bad)
        with pytest.raises(E.EngineError, match=r"\(-3\).*time_dependency\.model\.linear\.weight"):
            eng.load_state_dict(dict(sd, **{"time_dependency.model.linear.weight": torch.zeros(64, 384)}))
        eng.load_state_dict(sd)
        eng.set_option("conv_tc", 0)
        with pytest.raises(E.EngineError, match=r"\(-4\).*conv_tc=0.*\[16, 5\] \[8, 4\] \[4, 2\]"):
            eng.predict_pcm([_pcm(args, 3, 41)], [SR])
        eng.set_option("conv_tc", 1)
        _, _, status = eng.predict_pcm([_pcm(args, 3, 41)], [SR])
        assert status[0] == E.CLIP_OK
    finally:
        eng.close()


@pytest.mark.gpu
def test_predict_dir_runs_a_pool_checkpoint_end_to_end(built_lib, tmp_path):
    import pandas as pd
    from nisqa_b200.NISQA_model import nisqaModel
    name = "mos_p16x5_8x4_4x2"
    args, sd = _variant(name)
    ck = str(tmp_path / "p.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    d = tmp_path / "wavs"
    d.mkdir()
    out_dir = tmp_path / "out"
    out_dir.mkdir()
    pcm = {}
    for seed, sec, sr in V.POOL_CLIPS:
        fn = "p%03d.wav" % seed
        pcm[fn] = (synth.synth_speech_pcm16(seed, sec, sr), sr)
        wav.write_wav_pcm16(str(d / fn), *pcm[fn])
    nisqaModel({"mode": "predict_dir", "pretrained_model": ck, "data_dir": str(d), "output_dir": str(out_dir),
                "tr_bs_val": 2, "tr_num_workers": 0, "ms_channel": None}).predict()
    df = pd.read_csv(out_dir / "NISQA_results.csv")
    assert sorted(df["deg"]) == sorted(pcm)
    g = np.load(os.path.join(GOLDEN, "variants_cnn_pool.npz"))[name]
    assert np.abs(np.sort(df["mos_pred"].to_numpy()) - np.sort(g[:, 0])).max() <= SCORE_TOL
