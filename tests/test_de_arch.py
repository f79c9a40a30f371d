"""NISQA_DE checkpoints with StandardCNN, SkipCNN or DFF in front of self-attention, and StandardCNN in front of an LSTM
td of any accepted shape: the alignment and fusion then run at the LSTM's fan_out W in {32, 64, 96, 128, 192, 256, 384,
512} (rows padded to 64 NC columns) instead of 64.

CPU: the configuration accepts every variant of oracle/de_arch_variants.py and the whole LSTM shape x alignment x
application x fusion grid, and keeps the refusals of what the engine does not run; the oracle matches the unmodified
reference NISQA_DE (oracle/de_arch_oracle.py against tests/golden/variants_de_arch.npz, oracle/make_de_arch_golden.py).
GPU: every variant through the C ABI against the golden and the oracle, with multi-block references, one-segment clips,
pairs of different lengths and a too-short reference; a pair alone == the same pair in the batch; several passes == one
pass; Scorer == predict_pcm; nisqaModel(mode='predict_csv', csv_ref=...).  And de_align_kernel's output
(NISQA_STAGE_DE_FUSED) from the engine's own td rows (NISQA_STAGE_TD1_OUT) against float64 (tests/stage_ref_de.py) at
W = 32, 96, 256 and 512 for every alignment method, hard and soft.
"""
import functools
import os

import numpy as np
import pytest
import torch

import stage_ref as R
import stage_ref_de as D
from conftest import GOLDEN, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import de_arch_oracle as DO
from oracle import de_arch_variants as V
from oracle import nisqa_oracle as O
from oracle import variants as VV
from oracle.td_pair_variants import lstm, sa

TOL = 1e-4
SR = 16000
ALIGNS = ["dot", "cosine", "distance", "luong", "bahd"]
APPLIES = ["hard", "soft"]
FUSES = ["x/y/-", "+/-", "x/y"]
DE_KEYS = dict(de_align="dot", de_align_apply="soft", de_fuse="x/y/-", de_fuse_dim=None)


@functools.lru_cache(maxsize=None)
def _base(ckpt):
    return O.load_checkpoint(os.path.join(WEIGHTS, ckpt))


def _variant(name, spec=None):
    base = (spec or V.DE_ARCH_VARIANTS[name])[0]
    bargs, bsd = _base(base)
    return V.de_arch_checkpoint(name, bargs, bsd, spec)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


def _pcm(args, n_seg, seed):
    """a 16 kHz clip of exactly n_seg segments"""
    n = (args["ms_seg_length"] + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * int(SR * args["ms_hop_length"])
    y = synth.synth_speech_pcm16(seed, n / SR + 0.05, SR)[:n]
    assert O.segment_counts(n, SR, args)[1] == n_seg
    return y


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(V.DE_ARCH_VARIANTS))
def test_config_accepts_the_variants(name):
    args, _ = _variant(name)
    c = E.config_from_args(args)
    assert (c.double_ended, c.n_out, c.td2_layers, c.td2_d_model) == (1, 1, 2, 64)
    assert c.arch == (E.ARCH_STD_LSTM_LASTBI if args["td"] == "lstm" else E.ARCH_ADAPT_SA_ATTFF)
    assert c.de_fuse_dim == (args.get("de_fuse_dim") or 0)


def test_config_accepts_the_lstm_grid():
    bargs, _ = _base("nisqa_tts.tar")
    de = dict(bargs, model="NISQA_DE", **sa("td_2", 64, 64, 2), pool="avg")
    n = 0
    for h in E.LSTM_H:
        for nl in range(1, E.LSTM_LAYERS_MAX + 1):
            for bi in (False, True):
                for fc in (None, 1, 20, 100, 1024):
                    for align in ALIGNS:
                        for apply in APPLIES:
                            for fuse in FUSES:
                                for fd in (None, 128):
                                    c = E.config_from_args(dict(de, **lstm("td", h, nl, bi), cnn_fc_out_h=fc, de_align=align,
                                                                de_align_apply=apply, de_fuse=fuse, de_fuse_dim=fd))
                                    assert (c.arch, c.double_ended, c.sa_layers, c.td2_layers) == (E.ARCH_STD_LSTM_LASTBI, 1, 0, 2)
                                    assert (c.de_align, c.de_align_apply, c.de_fuse, c.de_fuse_dim) == (
                                        E.DE_ALIGN[align], E.DE_APPLY[apply], E.DE_FUSE[fuse], fd or 0)
                                    n += 1
    assert n == len(E.LSTM_H) * E.LSTM_LAYERS_MAX * 2 * 5 * 5 * 2 * 3 * 2


def test_config_keeps_the_refusals():
    nisqa, _ = _base("nisqa.tar")
    tts, _ = _base("nisqa_tts.tar")
    de_sa = dict(nisqa, model="NISQA_DE", **sa("td_2", 64, 64, 2), **DE_KEYS)
    de_lstm = dict(tts, model="NISQA_DE", **sa("td_2", 64, 64, 2), **DE_KEYS, pool="avg")
    for bad, what in ((dict(de_sa, td="skip"), "NISQA_DE with td='skip'"),
                      (dict(de_sa, **lstm("td_2", 64)), "NISQA_DE with td_2='lstm'"),
                      (dict(de_sa, td_2="skip"), "NISQA_DE with td_2='skip'"),
                      (dict(de_sa, td_sa_d_model=128), "128"),
                      (dict(de_sa, td_2_sa_d_model=128), "128"),
                      (dict(de_lstm, td_2_sa_d_model=128), "128"),
                      (dict(de_lstm, cnn_model="standard", **sa("td", 128, 64)), "128"),
                      (dict(de_sa, de_align="none"), "de_align='none'"),
                      (dict(de_lstm, de_align="none"), "de_align='none'"),
                      (dict(de_sa, **lstm("td", 128)), "td='lstm'"),
                      (dict(de_sa, cnn_model="skip", cnn_fc_out_h=None, **lstm("td", 64)), "td='lstm'"),
                      (dict(de_sa, cnn_model="dff", cnn_fc_out_h=256, **lstm("td", 64)), "td='lstm'"),
                      (dict(de_lstm, td_lstm_h=48), "td_lstm_h=48"),
                      (dict(de_lstm, td_lstm_num_layers=5), "td_lstm_num_layers=5"),
                      (dict(de_lstm, pool="last_step_bi"), "last_step_bi"),
                      (dict(de_lstm, cnn_fc_out_h=2000), "cnn_fc_out_h=2000")):
        with pytest.raises(NotImplementedError, match=what):
            E.config_from_args(bad)


def test_oracle_matches_the_reference_golden():
    g = np.load(os.path.join(GOLDEN, "variants_de_arch.npz"))
    assert sorted(g.files) == sorted(V.DE_ARCH_VARIANTS)
    pairs = [VV.de_pair_pcm(p) for p in V.DE_ARCH_PAIRS]
    torch.set_num_threads(1)
    for name in V.DE_ARCH_VARIANTS:
        args, sd = _variant(name)
        got = []
        for deg, srd, ref, srr in pairs:
            sc, _, st = DO.predict_pcm_de(args, sd, _f32(deg), srd, _f32(ref), srr)
            assert st == O.STATUS_OK
            got.append(sc[0])
        d = float(np.abs(np.array(got) - g[name][:, 0]).max())
        assert d <= 5e-6, (name, d)


# ------------------------------------------------------------------------------------------------------------ GPU
def _gpu_batch(args):
    """-> (pairs [(deg, sr, ref, sr)], index of the pair with a too-short reference): the golden's pairs, a one-segment
    pair, a one-segment degraded clip against a three-key-block reference, a too-short reference, and a pair whose
    reference is shorter than its degraded clip"""
    pairs = [VV.de_pair_pcm(p) for p in V.DE_ARCH_PAIRS]
    pairs.append((_pcm(args, 1, 401), SR, _pcm(args, 1, 402), SR))
    pairs.append((_pcm(args, 1, 403), SR, _pcm(args, 150, 404), SR))
    short = len(pairs)
    pairs.append((_pcm(args, 40, 405), SR, np.zeros(100, np.int16), SR))
    pairs.append((_pcm(args, 130, 406), SR, _pcm(args, 65, 407), SR))
    return pairs, short


def _flat(pairs):
    clips, srs = [], []
    for deg, srd, ref, srr in pairs:
        clips += [deg, ref]; srs += [srd, srr]
    return clips, srs


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.DE_ARCH_VARIANTS))
def test_variant_through_the_c_abi(built_lib, name):
    g = np.load(os.path.join(GOLDEN, "variants_de_arch.npz"))[name][:, 0]
    args, sd = _variant(name)
    pairs, short = _gpu_batch(args)
    clips, srs = _flat(pairs)
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    try:
        scores, nseg, status = eng.predict_pcm(clips, srs)
        alone, nseg1, _ = eng.predict_pcm(clips[6:8], srs[6:8])          # the pair with the 8 s reference
    finally:
        eng.close()
    assert status[2 * short + 1] == E.CLIP_TOO_SHORT and (status == E.CLIP_OK).sum() == len(clips) - 1
    assert np.all(np.isnan(scores[1::2])) and np.isnan(scores[2 * short, 0])
    got = scores[0::2, 0]
    d = float(np.abs(got[:len(g)] - g).max())
    print("%s: max |engine - golden| %.3g" % (name, d))
    assert d <= TOL, (name, got[:len(g)], g)
    np.testing.assert_array_equal(alone[0], scores[6])
    np.testing.assert_array_equal(nseg1, nseg[6:8])
    for p, (deg, srd, ref, srr) in enumerate(pairs):
        if p == short:
            continue
        sc, ns, st = DO.predict_pcm_de(args, sd, _f32(deg), srd, _f32(ref), srr)
        assert st == O.STATUS_OK and ns == (nseg[2 * p], nseg[2 * p + 1]), (name, p)
        assert abs(float(got[p]) - float(sc[0])) <= TOL, (name, p, float(got[p]), float(sc[0]))
    eng = E.Engine(E.config_from_args(args, max_chunk_segments=120), 0)     # several passes == one pass
    eng.load_state_dict(sd)
    try:
        multi, nseg2, status2 = eng.predict_pcm(clips, srs)
    finally:
        eng.close()
    np.testing.assert_array_equal(nseg2, nseg)
    np.testing.assert_array_equal(status2, status)
    np.testing.assert_array_equal(multi, scores)


@pytest.mark.gpu
def test_lstm_variant_through_scorer_and_predict_csv(built_lib, tmp_path):
    import pandas as pd
    from nisqa_b200 import wav
    from nisqa_b200.NISQA_model import nisqaModel
    from nisqa_b200.scorer import Scorer
    name = "std_fc20_lstm128bi_luong_soft_fd128"
    args, sd = _variant(name)
    torch.save({"args": args, "model_state_dict": sd}, tmp_path / "de.tar")
    sc = Scorer(str(tmp_path / "de.tar"))
    try:
        deg, srd, ref, _ = VV.de_pair_pcm(V.DE_ARCH_PAIRS[0])
        n = min(len(deg), len(ref))
        d2 = torch.from_numpy(np.stack([deg[:n], deg[::-1][:n].copy()])).cuda()
        r2 = torch.from_numpy(np.stack([ref[:n], ref[::-1][:n].copy()])).cuda()
        got = sc(d2, srd, lengths=[n, n - 480], reference=r2).cpu().numpy()
        want = sc.engine.predict_pcm([deg[:n], ref[:n], deg[::-1][:n - 480].copy(), ref[::-1][:n].copy()], [srd] * 4)[0]
        np.testing.assert_array_equal(got, want[0::2])
    finally:
        sc.close()
    g = np.load(os.path.join(GOLDEN, "variants_de_arch.npz"))[name][:, 0]
    rows = []
    for i, pair in enumerate(V.DE_ARCH_PAIRS):
        deg, srd, ref, srr = VV.de_pair_pcm(pair)
        wav.write_wav_pcm16(str(tmp_path / ("deg%d.wav" % i)), deg, srd)
        wav.write_wav_pcm16(str(tmp_path / ("ref%d.wav" % i)), ref, srr)
        rows.append(("deg%d.wav" % i, "ref%d.wav" % i))
    pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(tmp_path / "files.csv", index=False)
    m = nisqaModel({"mode": "predict_csv", "pretrained_model": str(tmp_path / "de.tar"), "csv_file": "files.csv",
                    "csv_deg": "deg", "csv_ref": "ref", "data_dir": str(tmp_path), "output_dir": None, "ms_channel": None,
                    "tr_bs_val": 2, "tr_num_workers": 0})
    try:
        df = m.predict()
    finally:
        m.model.close()
    assert np.abs(df["mos_pred"].to_numpy() - g).max() <= TOL


# td's fan_out W -> the LSTM giving it
STAGE_W = {32: lstm("td", 32, 1, False), 96: lstm("td", 96, 1, False), 256: lstm("td", 128), 512: lstm("td", 256)}


def _stage_batch(args):
    """(degraded, reference) 16 kHz pairs in segments: 1 to 4 key blocks of 64 on either side, 1297 = 21 key blocks,
    and a too-short reference; -> (pairs, index of the too-short pair)"""
    counts = [(1, 1), (63, 65), (65, 130), (130, 64), (70, 1297)]
    pairs = [(_pcm(args, a, 500 + i), _pcm(args, b, 600 + i)) for i, (a, b) in enumerate(counts)]
    pairs.append((_pcm(args, 40, 520), np.zeros(100, np.int16)))
    return pairs, len(pairs) - 1


@pytest.mark.gpu
@pytest.mark.parametrize("W", list(STAGE_W))
def test_de_alignment_at_width_against_float64(built_lib, W):
    """td1_out -> de_fused from the engine's own dumps against float64 (stage_ref_de: soft rows within the first-order
    bound, hard rows the fp32 fusion with a reference step of the candidate set), every method, hard and soft.  The
    dump is the engine's padded layout: part p at column p round64(W), pad columns zero."""
    ld = (W + 63) // 64 * 64
    worst = {}
    for align in ALIGNS:
        fuse = FUSES[ALIGNS.index(align) % 3]              # every fusion mode, a different one per method
        for apply in APPLIES:
            over = dict(STAGE_W[W], **DE_KEYS, pool="avg")
            over.update(de_align=align, de_align_apply=apply, de_fuse=fuse)
            args, sd = _variant("stage_w%d_%s_%s" % (W, align, apply), ("nisqa_tts.tar", None, over))
            pairs, short = _stage_batch(args)
            clips = [c for p in pairs for c in p]
            eng = E.Engine(E.config_from_args(args), 0)
            eng.load_state_dict(sd)
            try:
                scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
                ok = status == E.CLIP_OK
                has_rows = np.repeat(ok[0::2] & ok[1::2], 2)
                N = int(nseg[has_rows].sum())
                td1 = torch.from_numpy(eng.stage_dump(E.STAGE_TD1_OUT)).double().reshape(N, W)
                fused = torch.from_numpy(eng.stage_dump(E.STAGE_DE_FUSED)).reshape(N, -1)
            finally:
                eng.close()
            nf = D.n_fused(args)
            assert fused.shape[1] == nf * ld
            parts = fused.reshape(N, nf, ld)
            assert not parts[:, :, W:].any()                         # pad columns zero
            compact = parts[:, :, :W].reshape(N, nf * W)
            assert np.isnan(scores[2 * short, 0]) and status[2 * short + 1] == E.CLIP_TOO_SHORT
            starts = np.concatenate([[0], np.cumsum(np.where(has_rows, nseg, 0))])
            rows = lambda t, c: t[starts[c]:starts[c + 1]]          # noqa: E731
            r, fr = 0.0, []
            for p in range(len(pairs)):
                if p == short:
                    continue
                assert not rows(fused, 2 * p + 1).any()              # reference rows stay zero
                x, y = rows(td1, 2 * p), rows(td1, 2 * p + 1)
                got = rows(compact, 2 * p)
                s, b = D.scores(args, sd, x, y)
                if apply == "hard":
                    bad, frac = D.check_hard(args, x, y, got, D.candidates(s, b))
                    assert bad is None, (W, align, p, bad)
                    fr.append((frac, x.shape[0]))
                else:
                    ref, bd = D.fuse(args, x, *D.soft_align(s, b, y))
                    r = max(r, R.ratio(got.double(), ref, bd))
            if apply == "hard":
                r = sum(f * n for f, n in fr) / sum(n for _, n in fr)
                assert r >= 0.5, (W, align, r)                        # most rows have one candidate
            else:
                assert r <= 1.0, (W, align, r)
            worst[(align, apply, fuse)] = r
    print("\nW %d: %s" % (W, ", ".join("%s/%s/%s %s %.3g" % (a, p, f, "one-candidate rows" if p == "hard" else "ratio", v)
                                        for (a, p, f), v in worst.items())))
