"""Time-dependency stages in any order the reference builds: StandardCNN in front of self-attention, an LSTM as td_2
behind self-attention or an LSTM, and self-attention as td_2 behind an LSTM, for NISQA and NISQA_DIM.

CPU: the configuration fills arch / cnn_kind / td2_* for every pair variant and refuses the rest, naming the value; the
header's new enum values equal the binding's; the oracle against the scores of the unmodified reference modules
(tests/golden/variants_td_pairs.npz, oracle/make_td_pair_golden.py).
GPU: every pair variant through the C ABI against the reference scores and the oracle (one-segment, 97-segment and, for
the cluster LSTMs, 1300-segment clips in the batch), alone == in a batch, several passes == one pass; the stages
CNN_FEAT -> TD_IN -> TD1_OUT -> TD_OUT -> scores against float64 (tests/stage_ref.py, tests/stage_ref_lstm.py) for
StandardCNN + self-attention, self-attention -> LSTM and LSTM -> self-attention; nisqa_load_weights refusing a
mis-shaped td_2 LSTM tensor; and one pairing end to end through nisqaModel(mode='predict_dir').
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
from oracle import td_pair_variants as V

SCORE_TOL = 1e-4
SR = 16000


def _variant(name, spec=None):
    base = (spec or V.TD_PAIR_VARIANTS[name])[0]
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.td_pair_checkpoint(name, args, sd, spec)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(V.TD_PAIR_VARIANTS))
def test_config_fills_the_pairing(name):
    args, _ = _variant(name)
    c = E.config_from_args(args)
    td_lstm, td2 = args["td"] == "lstm", args.get("td_2") or "skip"
    arch = {(False, "lstm"): E.ARCH_SA_LSTM, (True, "lstm"): E.ARCH_LSTM_LSTM}.get(
        (td_lstm, td2), E.ARCH_STD_LSTM_LASTBI if td_lstm else E.ARCH_ADAPT_SA_ATTFF)
    assert c.arch == arch and c.n_out == (5 if args["model"] == "NISQA_DIM" else 1)
    assert c.cnn_kind == (E.CNN_STANDARD if (args["cnn_model"], td_lstm) == ("standard", False) else
                          E.CNN_DFF if args["cnn_model"] == "dff" else E.CNN_CONV)
    if args["cnn_model"] == "standard":
        assert c.cnn_fc == 0                    # StandardCNN's fc_out width comes from the weights
    if td_lstm:
        assert (c.sa_layers, c.sa_d_model, c.pos_enc) == (0, 0, 0)
    else:
        assert (c.sa_layers, c.sa_d_model, c.sa_ff) == (args["td_sa_num_layers"], args["td_sa_d_model"], args["td_sa_h"])
    if td2 == "self_att":
        assert (c.td2_layers, c.td2_d_model, c.td2_ff, c.td2_pos_enc) == (
            args["td_2_sa_num_layers"], args["td_2_sa_d_model"], args["td_2_sa_h"], int(bool(args["td_2_sa_pos_enc"])))
    else:
        assert (c.td2_layers, c.td2_d_model, c.td2_ff) == (0, 0, 0)


def test_config_refuses_pairings_outside_the_kernels():
    sa_lstm, _ = _variant("mos_adapt_sa64_lstm128bi_lastbi")
    sa_sa, _ = _variant("mos_std_fc20_sa64pos_sa128_avg")
    lstm_lstm, _ = _variant("mos_std_lstm192bi_lstm64uni_last")
    dim_sa_lstm, _ = _variant("dim_adapt_sa64_lstm32bi_attff")
    dim_lstm_sa, _ = _variant("dim_std_lstm64bi_sa128_avg")
    nisqa, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    de = dict(nisqa, model="NISQA_DE", de_align="dot", de_align_apply="soft", de_fuse="x/y/-", de_fuse_dim=None,
              **V.lstm("td_2", 64))
    for bad, what in ((dict(sa_lstm, td_2_lstm_h=None), "td_2='lstm' with td_2_lstm_h=None"),
                      (dict(sa_lstm, td_2_lstm_h=48), "td_2='lstm' with td_2_lstm_h=48"),
                      (dict(lstm_lstm, td_2_lstm_num_layers=5), "td_2='lstm' with td_2_lstm_num_layers=5"),
                      (dict(sa_sa, pool="last_step_bi"), "last_step_bi.*td_2='self_att'"),
                      (dict(lstm_lstm, pool="last_step_bi"), "last_step_bi.*td_2_lstm_bidirectional=False"),
                      (dict(dim_sa_lstm, td_2_lstm_h=64), r"td_2 fan_out 128 \(td_2_lstm_h=64.*td fan_out 64 \(td_sa_d_model=64"),
                      (dict(dim_lstm_sa, td_2_sa_d_model=64), r"td_2 fan_out 64 \(td_2_sa_d_model=64\).*td fan_out 128 \(td_lstm_h=64"),
                      (de, "NISQA_DE with td_2='lstm'"),
                      (dict(nisqa, td="lstm", td_lstm_h=128, td_lstm_num_layers=1, td_lstm_bidirectional=True), "td='lstm'"),
                      (dict(sa_lstm, cnn_model="skip", td="lstm", td_lstm_h=128, td_lstm_num_layers=1), "td='lstm'")):
        with pytest.raises(NotImplementedError, match=what):
            E.config_from_args(bad)


def test_header_enums_equal_the_binding(tmp_path):
    src = tmp_path / "enums.c"
    names = ["NISQA_CNN_STANDARD", "NISQA_ARCH_ADAPT_SA_ATTFF", "NISQA_ARCH_STD_LSTM_LASTBI", "NISQA_ARCH_SA_LSTM",
             "NISQA_ARCH_LSTM_LSTM", "NISQA_STAGE_TD_IN", "NISQA_STAGE_TD_OUT", "NISQA_STAGE_TD1_OUT", "NISQA_STAGE_DE_FUSED"]
    src.write_text('#include <stdio.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu' + " %d" * len(names)
                   + '\\n", sizeof(nisqa_config), ' + ", ".join(names) + ");return 0;}\n")
    exe = tmp_path / "enums"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [ctypes.sizeof(E.NisqaConfig), E.CNN_STANDARD, E.ARCH_ADAPT_SA_ATTFF, E.ARCH_STD_LSTM_LASTBI, E.ARCH_SA_LSTM,
                   E.ARCH_LSTM_LSTM, E.STAGE_TD_IN, E.STAGE_TD_OUT, E.STAGE_TD1_OUT, E.STAGE_DE_FUSED]
    assert out[1:] == [3, 0, 1, 2, 3, 7, 8, 9, 10]


def test_oracle_matches_reference_modules_on_the_pair_variants():
    g = np.load(os.path.join(GOLDEN, "variants_td_pairs.npz"))
    assert sorted(g.files) == sorted(V.TD_PAIR_VARIANTS)
    for name in V.TD_PAIR_VARIANTS:
        args, sd = _variant(name)
        for i, (seed, sec, sr) in enumerate(V.TD_PAIR_CLIPS):
            sc, _, st = TO.predict_pcm(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
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


def _cluster(args):
    """an LSTM stage of H 192 / 256 (lstm_layer_kernel on clusters of CTAs)"""
    return any(args.get(s) == "lstm" and args[s + "_lstm_h"] >= 192 for s in ("td", "td_2"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.TD_PAIR_VARIANTS))
def test_td_pair_variant_through_the_c_abi(built_lib, name):
    args, sd = _variant(name)
    g = np.load(os.path.join(GOLDEN, "variants_td_pairs.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.TD_PAIR_CLIPS]
    srs = [c[2] for c in V.TD_PAIR_CLIPS]
    # a one-segment clip between long clips, 97 segments and, for the cluster LSTMs, a 1300-segment clip
    extra = [_pcm(args, 1, 7), _pcm(args, 97, 8)] + ([_pcm(args, 1300, 9)] if _cluster(args) else [])
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


# rows 1-3 of the new pairings: StandardCNN -> self-attention (with and without fc_out), self-attention -> LSTM,
# LSTM -> self-attention
STAGE_VARIANTS = ["mos_std_sa64_attff", "dim_std_fc100_sa128_l2_attff", "dim_adapt_sa64_lstm32bi_attff",
                  "mos_adapt_sa64_lstm128bi_lastbi", "mos_tts_sa64_attff", "dim_std_lstm64bi_sa128_avg"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", STAGE_VARIANTS)
def test_td_pair_stages_against_float64(built_lib, name):
    """Each stage from the engine's own dump of its input against float64 (bound TAU = 2^-18 times the magnitude of the
    stage's terms, tests/stage_ref.py): CNN_FEAT -> TD_IN / TD1_OUT -> TD_IN -> TD_OUT -> scores, as the pairing runs them."""
    args, sd = _variant(name)
    sd2 = TO.td2_state_dict(sd)
    lens = [400, 1, 63, 97, 2]
    clips = [_pcm(args, n, 100 + i) for i, n in enumerate(lens)]
    eng = _engine(args, sd)
    has2 = args.get("td_2") in ("self_att", "lstm")
    try:
        scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
        assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
        N = sum(lens)
        dump = lambda st: torch.from_numpy(eng.stage_dump(st)).double().reshape(N, -1)      # noqa: E731
        feat, td_in, td_out = dump(E.STAGE_CNN_FEAT), dump(E.STAGE_TD_IN), dump(E.STAGE_TD_OUT)
        td1 = dump(E.STAGE_TD1_OUT) if has2 else None
    finally:
        eng.close()
    starts = np.concatenate([[0], np.cumsum(lens)])
    rows = lambda x, i: x[starts[i]:starts[i + 1]]          # noqa: E731
    zero = torch.zeros_like
    ratios = {}

    def add(k, got, ref, bound):
        ratios[k] = max(ratios.get(k, 0.0), R.ratio(got, ref, bound))
    if args["td"] == "self_att":
        ref, b = R.td_in(sd, feat, zero(feat))
        add("cnn_feat->td_in", td_in, ref, b)
        sa_out = td1 if has2 else td_out
        for i in range(len(lens)):
            ref, b = R.sa_stack(sd, rows(td_in, i), zero(rows(td_in, i)))
            add("td_in->td1_out" if has2 else "td_in->td_out", rows(sa_out, i), ref, b)
        if args.get("td_2") == "lstm":
            xs = [rows(td1, i) for i in range(len(lens))]
            for i, (ref, b) in enumerate(RL.lstm_stack(sd2, xs, [zero(x) for x in xs])):
                add("td1_out->td_out", rows(td_out, i), ref, b)
    else:
        xs = [rows(feat, i) for i in range(len(lens))]
        for i, (ref, b) in enumerate(RL.lstm_stack(sd, xs, [zero(x) for x in xs])):
            add("cnn_feat->td1_out", rows(td1, i), ref, b)
        ref, b = R.td_in(sd2, td1, zero(td1))
        add("td1_out->td_in", td_in, ref, b)
        for i in range(len(lens)):
            ref, b = R.sa_stack(sd2, rows(td_in, i), zero(rows(td_in, i)))
            add("td_in->td_out", rows(td_out, i), ref, b)
    for i in range(len(lens)):
        y = rows(td_out, i)
        ref, b = RL.pool_heads(sd, args, y, zero(y))
        add("td_out->scores", scores[i], ref, b)
    print("\n%s max |got - ref| / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


@pytest.mark.gpu
def test_load_weights_refuses_a_misshaped_td2_lstm_tensor(built_lib):
    args, sd = _variant("mos_adapt_sa64_lstm128bi_lastbi")
    name = "time_dependency_2.model.lstm.weight_ih_l0"
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        with pytest.raises(E.EngineError, match=r"\(-3\).*" + name.replace(".", r"\.")):
            eng.load_state_dict(dict(sd, **{name: torch.zeros(512, 65)}))
        with pytest.raises(E.EngineError, match=r"\(-3\).*time_dependency_2\.model\.lstm\.weight_hh_l0"):
            eng.load_state_dict(dict(sd, **{"time_dependency_2.model.lstm.weight_hh_l0": torch.zeros(192, 48)}))
        eng.load_state_dict(sd)
        scores, _, status = eng.predict_pcm([synth.synth_speech_pcm16(5, 1.0, SR)], [SR])
        assert status[0] == E.CLIP_OK and np.isfinite(scores).all()
    finally:
        eng.close()


@pytest.mark.gpu
def test_predict_dir_runs_a_pairing_end_to_end(built_lib, tmp_path):
    """A torch.save'd checkpoint of a new pairing scored through nisqaModel(mode='predict_dir') gives the Engine's scores."""
    from nisqa_b200.NISQA_model import nisqaModel
    name = "mos_std_sa256_ff1024_lstm128bi_att"
    args, sd = _variant(name)
    ck = str(tmp_path / "pair.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    d = tmp_path / "wavs"; d.mkdir()
    pcm = {}
    for seed, sec, sr in V.TD_PAIR_CLIPS:
        fn = "p%03d.wav" % seed
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
