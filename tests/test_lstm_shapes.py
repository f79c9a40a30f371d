"""StandardCNN + LSTM checkpoints of any accepted shape: td_lstm_h in {32, 64, 96, 128, 192, 256}, 1 to 4 layers,
either direction, cnn_fc_out_h 1..1024 or None, every pooling module, NISQA and NISQA_DIM.

CPU: the configuration accepts exactly that table (and refuses the rest, naming the value), and the oracle against the
scores of the unmodified reference modules (tests/golden/variants_lstm.npz, oracle/make_lstm_golden.py).
GPU: every LSTM variant through the C ABI against the reference scores and the oracle (one-segment, 97-segment,
1300-segment and too-short clips in the batch), alone == in a batch, several passes == one pass, the same scores
whatever NB / cluster grouping the batch size selects; and TD_OUT and the scores from the engine's CNN_FEAT dump against
float64 (tests/stage_ref_lstm.py) for H 32, 128 with two layers, 256, in both directions; nisqa_load_weights refusing
LSTM tensors of a shape the kernels do not implement (NISQA_ERR_WEIGHTS, naming the tensor).
"""
import itertools
import os

import numpy as np
import pytest
import torch

import stage_ref as R
import stage_ref_lstm as RL
from conftest import GOLDEN, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import lstm_oracle as LO
from oracle import lstm_variants as V
from oracle import nisqa_oracle as O

SCORE_TOL = 1e-4
SR = 16000


def _base():
    return O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_tts.tar"))


def _variant(name, over=None):
    args, sd = _base()
    return V.lstm_checkpoint(name, args, sd, over)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_config_accepts_the_table():
    args, _ = _base()
    pools = [("last_step_bi", None), ("last_step", None), ("avg", None), ("max", None), ("att", None), ("att", 128)]
    for h, nl, bi, fc, (pool, att_h), model in itertools.product(E.LSTM_H, (1, 2, 3, 4), (True, False), (1, 20, 100, 1024, None),
                                                                 pools, ("NISQA", "NISQA_DIM")):
        if pool == "last_step_bi" and not bi:
            continue
        c = E.config_from_args(dict(args, td_lstm_h=h, td_lstm_num_layers=nl, td_lstm_bidirectional=bi, cnn_fc_out_h=fc,
                                    pool=pool, pool_att_h=att_h, model=model))
        assert c.arch == E.ARCH_STD_LSTM_LASTBI and c.n_out == (5 if model == "NISQA_DIM" else 1)
        assert c.cnn_fc == 0 and c.sa_d_model == 0          # the LSTM's shape comes from the weights, not the config


def test_config_refuses_shapes_outside_the_kernels():
    args, _ = _base()
    sa, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    for bad, what in ((dict(args, td_lstm_h=48), "td_lstm_h=48"), (dict(args, td_lstm_h=512), "td_lstm_h=512"),
                      (dict(args, td_lstm_num_layers=5), "td_lstm_num_layers=5"),
                      (dict(args, td_lstm_num_layers=0), "td_lstm_num_layers=0"),
                      (dict(args, td_lstm_bidirectional=False), "last_step_bi"),
                      (dict(args, pool="att", pool_att_h=64), "pool_att_h=64"),
                      (dict(args, cnn_fc_out_h=2048), "cnn_fc_out_h=2048"),
                      (dict(args, td_2="lstm"), "td_2='lstm'"),
                      (dict(args, cnn_c_out_1=8), "cnn_c_out"),
                      (dict(args, cnn_kernel_size=(5, 5)), "cnn_kernel_size"),
                      (dict(sa, td="lstm", td_lstm_h=128, td_lstm_num_layers=1, td_lstm_bidirectional=True), "td='lstm'")):
        with pytest.raises(NotImplementedError, match=what):
            E.config_from_args(bad)


def test_oracle_matches_reference_modules_on_the_lstm_variants():
    g = np.load(os.path.join(GOLDEN, "variants_lstm.npz"))
    assert sorted(g.files) == sorted(V.LSTM_VARIANTS)
    for name in V.LSTM_VARIANTS:
        args, sd = _variant(name)
        for i, (seed, sec, sr) in enumerate(V.CLIPS):
            sc, _, st = LO.predict_pcm(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


# ------------------------------------------------------------------------------------------------------------ GPU
def _pcm(args, n_seg, seed):
    """a 16 kHz clip of exactly n_seg segments"""
    hop = int(SR * args["ms_hop_length"])
    n = (15 + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * hop
    y = synth.synth_speech_pcm16(seed, n / SR + 0.05, SR)[:n]
    assert O.segment_counts(n, SR, args)[1] == n_seg
    return y


def _engine(args, sd, **kw):
    eng = E.Engine(E.config_from_args(args, **kw), 0)
    eng.load_state_dict(sd)
    return eng


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.LSTM_VARIANTS))
def test_lstm_variant_through_the_c_abi(built_lib, name):
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_lstm.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.CLIPS]
    srs = [c[2] for c in V.CLIPS]
    # a one-segment clip between long clips, a too-short clip, 97 segments and, for H = 256, a 1300-segment clip
    short = synth.synth_speech_pcm16(6, 0.1, SR)
    extra = [_pcm(args, 1, 7), short, _pcm(args, 97, 8)] + ([_pcm(args, 1300, 9)] if args["td_lstm_h"] == 256 else [])
    batch = pcm[:2] + extra[:2] + pcm[2:] + extra[2:]
    bsr = srs[:2] + [SR, SR] + srs[2:] + [SR] * (len(extra) - 2)
    eng = _engine(args, sd)
    try:
        scores, nseg, status = eng.predict_pcm(batch, bsr)
        assert status[3] == E.CLIP_TOO_SHORT and np.all(np.isnan(scores[3])), name
        assert np.all(np.delete(status, 3) == E.CLIP_OK), name
        ours = np.concatenate([scores[:2], scores[4:5]])
        err = float(np.abs(ours - g).max())
        print("\n%s: max |engine - reference| %.3g" % (name, err))
        assert err <= SCORE_TOL, (name, err)
        worst = 0.0
        for i, (p, sr) in enumerate(zip(batch, bsr)):
            if i == 3:
                continue
            ref, ns, st = LO.predict_pcm(args, sd, _f32(p), sr)
            assert st == O.STATUS_OK and ns == nseg[i], (name, i)
            worst = max(worst, float(np.abs(scores[i] - ref).max()))
        print("%s: max |engine - oracle| %.3g over segment counts %s" % (name, worst, nseg.tolist()))
        assert worst <= SCORE_TOL, (name, worst)
        for i in (2, len(batch) - 1):                                    # alone == in the batch, bit for bit
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


# (variant, batch sizes): lstm_layer_kernel puts NB = 1, 2 or 4 sequences per CTA so that dirs x n_clips x C CTAs fit
# the 132 SMs - H 256 bidirectional (C = 4, 8 CTAs per clip): <= 16 clips NB 1, <= 33 NB 2, more NB 4; H 192
# unidirectional (C = 3): <= 44, <= 88; H 32 unidirectional (C = 1): <= 132, <= 264
@pytest.mark.gpu
@pytest.mark.parametrize("name,sizes", [("tts_h256_bi_fc100_max", (6, 30, 40)), ("tts_h192_l3_uni_fcnone_attff", (6, 80, 100)),
                                        ("tts_h32_uni_fc20_avg", (6, 200, 300))])
def test_scores_do_not_depend_on_the_grouping(built_lib, name, sizes):
    args, sd = _variant(name)
    rng = np.random.default_rng(11)
    lens = rng.integers(1, 60, max(sizes))
    pool = [_pcm(args, int(n), 200 + i) for i, n in enumerate(lens)]
    eng = _engine(args, sd)
    try:
        runs = [eng.predict_pcm(pool[:n], [SR] * n)[0] for n in sizes]
    finally:
        eng.close()
    for r in runs[1:]:
        np.testing.assert_array_equal(r[:sizes[0]], runs[0])
    for i in range(sizes[0]):
        ref, _, _ = LO.predict_pcm(args, sd, _f32(pool[i]), SR)
        assert float(np.abs(runs[0][i] - ref).max()) <= SCORE_TOL, (name, i)


# (H, layers, bidirectional, fc_out, pool, pool_att_h)
STAGE_SPECS = [(32, 1, False, 100, "att", 128), (32, 1, True, None, "last_step_bi", None),
               (128, 2, False, 20, "att", 128), (128, 2, True, 100, "last_step_bi", None),
               (256, 1, False, None, "att", 128), (256, 1, True, 20, "last_step_bi", None)]


@pytest.mark.gpu
@pytest.mark.parametrize("spec", STAGE_SPECS, ids=lambda s: "h%d_l%d_%s" % (s[0], s[1], "bi" if s[2] else "uni"))
def test_lstm_stages_against_float64(built_lib, spec):
    """TD_OUT from the engine's CNN_FEAT dump, and the scores from its TD_OUT dump, against float64 (bound TAU = 2^-18
    times the magnitude of the stage's terms, tests/stage_ref.py)."""
    H, nl, bi, fc, pool, att_h = spec
    name = "stage_h%d_l%d_%d" % (H, nl, bi)
    args, sd = _variant(name, {"td_lstm_h": H, "td_lstm_num_layers": nl, "td_lstm_bidirectional": bi, "cnn_fc_out_h": fc,
                               "pool": pool, "pool_att_h": att_h})
    lens = [1300 if H == 256 else 400, 1, 63, 97, 2]
    clips = [_pcm(args, n, 100 + i) for i, n in enumerate(lens)]
    eng = _engine(args, sd)
    try:
        scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
        assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
        N, D = sum(lens), (2 if bi else 1) * H
        feat = torch.from_numpy(eng.stage_dump(E.STAGE_CNN_FEAT)).double().reshape(N, -1)
        td_out = torch.from_numpy(eng.stage_dump(E.STAGE_TD_OUT)).double().reshape(N, D)
    finally:
        eng.close()
    assert feat.shape[1] == (fc or 768)
    starts = np.concatenate([[0], np.cumsum(lens)])
    xs = [feat[starts[i]:starts[i + 1]] for i in range(len(lens))]
    refs = RL.lstm_stack(sd, xs, [torch.zeros_like(x) for x in xs])
    ratios = {}
    for i, (ref, b) in enumerate(refs):
        y = td_out[starts[i]:starts[i + 1]]
        ratios["cnn_feat->td_out"] = max(ratios.get("cnn_feat->td_out", 0.0), R.ratio(y, ref, b))
        sref, sb = RL.pool_heads(sd, args, y, torch.zeros_like(y))
        ratios["td_out->scores"] = max(ratios.get("td_out->scores", 0.0), R.ratio(scores[i], sref, sb))
    print("\n%s max |got - ref| / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


@pytest.mark.gpu
def test_load_weights_refuses_lstm_tensors_outside_the_kernels(built_lib):
    """The LSTM's shape comes from the tensors: nisqa_load_weights refuses a shape the kernels do not implement with
    NISQA_ERR_WEIGHTS (-3) naming the tensor, and the engine still loads a good checkpoint afterwards."""
    args, sd = _base()
    p = "time_dependency.model.lstm."
    t = lambda *shape: torch.zeros(shape)      # noqa: E731
    no_reverse = {k: v for k, v in sd.items() if not k.endswith("_reverse")}
    five = dict(sd, **{p + "weight_hh_l%d" % l: t(512, 128) for l in range(1, 5)})
    for bad, tensor in ((dict(sd, **{p + "weight_hh_l0": t(192, 48)}), p + "weight_hh_l0"),
                        (five, p + "weight_hh_l4"),
                        (dict(sd, **{"cnn.model.fc_out.weight": t(2048, 768)}), "cnn.model.fc_out.weight"),
                        (no_reverse, p + "weight_hh_l0_reverse"),
                        (dict(sd, **{p + "weight_ih_l0": t(512, 21)}), p + "weight_ih_l0")):
        eng = E.Engine(E.config_from_args(args), 0)
        try:
            with pytest.raises(E.EngineError, match=r"\(-3\).*" + tensor.replace(".", r"\.")):
                eng.load_state_dict(bad)
            eng.load_state_dict(sd)
            scores, _, status = eng.predict_pcm([synth.synth_speech_pcm16(5, 1.0, SR)], [SR])
            assert status[0] == E.CLIP_OK and np.isfinite(scores).all()
        finally:
            eng.close()
