"""Checkpoints without a time-dependency model (td = 'skip'): the pooling module reads the framewise rows themselves
(pool_wide_kernel), or a self-attention td_2 - or, behind StandardCNN, an LSTM td_2 - reads them, for NISQA and NISQA_DIM.

CPU: the configuration (arch 4 / 5, cnn_kind, zeroed sa_*, td2_*) for every skip variant and the refusals, naming the
value; the header's new enum values and struct size equal the binding's; the oracle against the scores of the unmodified
reference modules (tests/golden/variants_td_skip.npz, oracle/make_td_skip_golden.py) and those scores in the MOS range.
GPU: every skip variant through the C ABI against the reference scores and the oracle (one-segment and 97-segment clips
in the batch, and for one StandardCNN variant a clip of exactly ms_max_segments), alone == in a batch, several passes ==
one pass; TD_OUT against the float64 framewise output and TD_OUT -> scores against float64 (tests/stage_ref_lstm.py);
nisqa_load_weights refusing a mis-shaped pooling tensor; and one skip checkpoint end to end through
nisqaModel(mode='predict_dir').
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import stage_ref as R
import stage_ref_lstm as RL
from conftest import GOLDEN, ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from oracle import nisqa_oracle as O
from oracle import td_pair_oracle as TO
from oracle import td_skip_variants as V
from oracle.td_pair_variants import TD_PAIR_CLIPS, lstm, sa

SCORE_TOL = 1e-4
SR = 16000
CNN_KIND = {"adapt": E.CNN_CONV, "standard": E.CNN_STANDARD, "skip": E.CNN_SKIP, None: E.CNN_SKIP, "dff": E.CNN_DFF}


def _variant(name):
    base = V.TD_SKIP_VARIANTS[name][0]
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.td_skip_checkpoint(name, args, sd)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(V.TD_SKIP_VARIANTS))
def test_config_fills_the_skip_variant(name):
    args, _ = _variant(name)
    c = E.config_from_args(args)
    td2 = args.get("td_2") or "skip"
    assert c.arch == (E.ARCH_SKIP_LSTM if td2 == "lstm" else E.ARCH_SKIP)
    assert c.n_out == (5 if args["model"] == "NISQA_DIM" else 1)
    assert c.cnn_kind == CNN_KIND[args["cnn_model"]]
    if args["cnn_model"] == "standard":
        assert c.cnn_fc == 0                    # StandardCNN's fc_out width comes from the weights
    else:
        assert c.cnn_fc == (args.get("cnn_fc_out_h") or 0)
    assert (c.sa_layers, c.sa_d_model, c.sa_ff, c.pos_enc) == (0, 0, 0, 0)
    if td2 == "self_att":
        assert (c.td2_layers, c.td2_d_model, c.td2_ff, c.td2_pos_enc) == (
            args["td_2_sa_num_layers"], args["td_2_sa_d_model"], args["td_2_sa_h"], int(bool(args["td_2_sa_pos_enc"])))
    else:
        assert (c.td2_layers, c.td2_d_model, c.td2_ff) == (0, 0, 0)


def test_config_refuses_skip_outside_the_kernels():
    adapt, _ = _variant("mos_adapt_skip_attff")
    skipcnn, _ = _variant("mos_skipcnn_skip_att")
    dff, _ = _variant("mos_dff_skip_avg")
    std, _ = _variant("mos_std_skip_max")
    std_lstm, _ = _variant("mos_std_fc20_skip_lstm128bi_lastbi")
    dim_sa, _ = _variant("dim_skipcnn_fc128_skip_sa128_att")
    dim_lstm, _ = _variant("dim_std_fc128_skip_lstm64bi_attff")
    nisqa, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    de = dict(nisqa, model="NISQA_DE", td="skip", de_align="dot", de_align_apply="soft", de_fuse="x/y/-", de_fuse_dim=None,
              **sa("td_2", 64, 64))
    for bad, what in ((dict(adapt, **lstm("td_2", 128)), "td_2='lstm' behind td='skip' and cnn_model='adapt'"),
                      (dict(skipcnn, **lstm("td_2", 128)), "td_2='lstm' behind td='skip' and cnn_model='skip'"),
                      (dict(dff, **lstm("td_2", 64)), "td_2='lstm' behind td='skip' and cnn_model='dff'"),
                      (dict(std, pool="last_step_bi"), "last_step_bi.*td='skip', td_2='skip'"),
                      (dict(adapt, td=None, pool="last_step_bi"), "last_step_bi.*td=None"),
                      (dict(std_lstm, td_2_lstm_bidirectional=False), "last_step_bi.*td_2_lstm_bidirectional=False"),
                      (dict(std_lstm, td_2_lstm_h=48), "td_2='lstm' with td_2_lstm_h=48"),
                      (de, "NISQA_DE with td='skip'"),
                      (dict(dim_sa, td_2_sa_d_model=64), r"td_2 fan_out 64 \(td_2_sa_d_model=64\) != td fan_out 128 \(td='skip': "
                                                         r"the framewise fan_out of cnn_model='skip', cnn_fc_out_h=128\)"),
                      (dict(dim_lstm, td_2_lstm_h=32), r"td_2 fan_out 64 \(td_2_lstm_h=32.*td fan_out 128 \(td='skip': "
                                                       r"the framewise fan_out of cnn_model='standard', cnn_fc_out_h=128\)"),
                      (dict(adapt, cnn_fc_out_h=100), "cnn_fc_out_h=100"),
                      (dict(dff, cnn_fc_out_h=200), "cnn_fc_out_h=200"),
                      (dict(std, cnn_kernel_size=5), "cnn_kernel_size=5"),
                      (dict(std, cnn_fc_out_h=2000), "cnn_fc_out_h=2000"),
                      (dict(adapt, td="conv"), "td='conv'")):
        with pytest.raises(NotImplementedError, match=what):
            E.config_from_args(bad)


def test_header_enums_equal_the_binding(tmp_path):
    src = tmp_path / "enums.c"
    names = ["NISQA_ARCH_SKIP", "NISQA_ARCH_SKIP_LSTM", "NISQA_B200_ABI_VERSION"]
    src.write_text('#include <stdio.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu' + " %d" * len(names)
                   + '\\n", sizeof(nisqa_config), ' + ", ".join(names) + ");return 0;}\n")
    exe = tmp_path / "enums"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [ctypes.sizeof(E.NisqaConfig), E.ARCH_SKIP, E.ARCH_SKIP_LSTM, E.ABI_VERSION]
    assert out[1:] == [4, 5, 4]


def test_oracle_matches_reference_modules_on_the_skip_variants():
    g = np.load(os.path.join(GOLDEN, "variants_td_skip.npz"))
    assert sorted(g.files) == sorted(V.TD_SKIP_VARIANTS)
    for name in V.TD_SKIP_VARIANTS:
        args, sd = _variant(name)
        for i, (seed, sec, sr) in enumerate(TD_PAIR_CLIPS):
            sc, _, st = TO.predict_pcm(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


def test_golden_scores_lie_in_the_mos_range():
    """the scaled score Linears keep every golden score where an absolute 1e-4 tolerance means something"""
    g = np.load(os.path.join(GOLDEN, "variants_td_skip.npz"))
    for name in g.files:
        assert g[name].shape == (len(TD_PAIR_CLIPS), 5 if name.startswith("dim_") else 1), name
        assert np.isfinite(g[name]).all() and g[name].min() >= -2.0 and g[name].max() <= 8.0, (name, g[name].tolist())


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


LONG_VARIANT = "dim_std_skip_attff"       # StandardCNN, five PoolAttFF heads: a clip of exactly ms_max_segments (6000)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.TD_SKIP_VARIANTS))
def test_td_skip_variant_through_the_c_abi(built_lib, name):
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_td_skip.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in TD_PAIR_CLIPS]
    srs = [c[2] for c in TD_PAIR_CLIPS]
    # a one-segment clip between long clips, 97 segments and, for one StandardCNN variant, ms_max_segments
    extra = [_pcm(args, 1, 7), _pcm(args, 97, 8)] + ([_pcm(args, args["ms_max_segments"], 9)] if name == LONG_VARIANT else [])
    batch = pcm[:2] + extra[:1] + pcm[2:] + extra[1:]
    bsr = srs[:2] + [SR] + srs[2:] + [SR] * (len(extra) - 1)
    eng = _engine(args, sd)
    try:
        scores, nseg, status = eng.predict_pcm(batch, bsr)
        assert np.all(status == E.CLIP_OK), name
        ours = np.concatenate([scores[:2], scores[3:3 + len(pcm) - 2]])
        err = float(np.abs(ours - g).max())
        print("\n%s: max |engine - reference| %.3g" % (name, err))
        assert err <= SCORE_TOL, (name, err)
        worst = 0.0
        for i, (p, sr) in enumerate(zip(batch, bsr)):
            ref, ns, st = TO.predict_pcm(args, sd, _f32(p), sr)
            assert st == O.STATUS_OK and ns == nseg[i], (name, i)
            worst = max(worst, float(np.abs(scores[i] - ref).max()))
        print("%s: max |engine - oracle| %.3g over segment counts %s" % (name, worst, nseg.tolist()))
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


POOL_VARIANTS = [n for n, (_, _, over) in V.TD_SKIP_VARIANTS.items() if over.get("td_2") == "skip"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", POOL_VARIANTS)
def test_td_skip_stages_against_float64(built_lib, name):
    """TD_OUT (the framewise rows the pooling module reads) against the float64 framewise output - the CNN_FEAT dump
    itself for conv6 features and fc_out, + the Linear for AdaptCNN's - and TD_OUT -> scores against float64 (bound
    TAU = 2^-18 times the magnitude of the stage's terms, tests/stage_ref.py)."""
    args, sd = _variant(name)
    lens = [400, 1, 63, 97, 2]
    clips = [_pcm(args, n, 100 + i) for i, n in enumerate(lens)]
    eng = _engine(args, sd)
    conv = args["cnn_model"] in ("adapt", "standard")
    try:
        scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
        assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
        N = sum(lens)
        dump = lambda st: torch.from_numpy(eng.stage_dump(st)).double().reshape(N, -1)      # noqa: E731
        td_out = dump(E.STAGE_TD_OUT)
        feat = dump(E.STAGE_CNN_FEAT) if conv else None
        for st in (E.STAGE_TD1_OUT, E.STAGE_TD_IN):                     # no td stage ran, no self-attention stack
            with pytest.raises(E.EngineError, match="not available"):
                eng.stage_dump(st)
    finally:
        eng.close()
    assert td_out.shape == (N, V.pooled_width(args))
    starts = np.concatenate([[0], np.cumsum(lens)])
    rows = lambda x, i: x[starts[i]:starts[i + 1]]          # noqa: E731
    zero = torch.zeros_like
    ratios = {}

    def add(k, got, ref, bound):
        ratios[k] = max(ratios.get(k, 0.0), R.ratio(got, ref, bound))
    if args["cnn_model"] == "adapt" and args.get("cnn_fc_out_h"):
        ref, b = R.linear(feat, zero(feat), sd["cnn.model.fc.weight"], sd["cnn.model.fc.bias"])
        add("cnn_feat->td_out", td_out, ref, b)
    elif conv:
        np.testing.assert_array_equal(td_out.numpy(), feat.numpy())   # the rows are the framewise output itself
    for i in range(len(lens)):
        y = rows(td_out, i)
        ref, b = RL.pool_heads(sd, args, y, zero(y))
        add("td_out->scores", scores[i], ref, b)
    print("\n%s max |got - ref| / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


@pytest.mark.gpu
def test_load_weights_refuses_a_misshaped_pooling_tensor(built_lib):
    for name, tensor, shape in (("mos_std_skip_max", "pool.model.linear.weight", (1, 767)),
                                ("dim_std_skip_attff", "pool_layers.1.model.linear1.weight", (128, 640)),
                                ("mos_skipcnn_skip_att", "pool.model.linear1.weight", (1, 768))):
        args, sd = _variant(name)
        eng = E.Engine(E.config_from_args(args), 0)
        try:
            with pytest.raises(E.EngineError, match=r"\(-3\).*" + tensor.replace(".", r"\.")):
                eng.load_state_dict(dict(sd, **{tensor: torch.zeros(*shape)}))
            eng.load_state_dict(sd)
            scores, _, status = eng.predict_pcm([synth.synth_speech_pcm16(5, 1.0, SR)], [SR])
            assert status[0] == E.CLIP_OK and np.isfinite(scores).all()
        finally:
            eng.close()


@pytest.mark.gpu
def test_predict_dir_runs_a_skip_checkpoint_end_to_end(built_lib, tmp_path):
    """A torch.save'd td='skip' checkpoint scored through nisqaModel(mode='predict_dir') gives the Engine's scores."""
    from nisqa_b200.NISQA_model import nisqaModel
    name = "mos_adapt_skip_attff"
    args, sd = _variant(name)
    ck = str(tmp_path / "skip.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    d = tmp_path / "wavs"; d.mkdir()
    pcm = {}
    for seed, sec, sr in TD_PAIR_CLIPS:
        fn = "s%03d.wav" % seed
        pcm[fn] = (synth.synth_speech_pcm16(seed, sec, sr), sr)
        wav.write_wav_pcm16(str(d / fn), *pcm[fn])
    df = nisqaModel({"mode": "predict_dir", "pretrained_model": ck, "data_dir": str(d), "output_dir": None, "tr_bs_val": 2,
                     "tr_num_workers": 0, "ms_channel": None}).predict()
    assert sorted(df["deg"]) == sorted(pcm)
    eng = _engine(args, sd)
    try:
        for _, row in df.iterrows():
            p, sr = pcm[row["deg"]]
            want, _, _ = eng.predict_pcm([p], [sr])
            np.testing.assert_allclose(row["mos_pred"], want[0, 0], rtol=0, atol=1e-6, err_msg=row["deg"])
    finally:
        eng.close()
