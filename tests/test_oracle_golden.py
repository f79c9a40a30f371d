"""Pins the oracle's model half to the UNMODIFIED reference modules: tests/golden/*.npz were
produced by oracle/make_golden.py running the reference's nisqaModel.predict() (reference
nisqa/NISQA_model.py:54-81) with forward hooks on model.cnn / model.time_dependency."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, WEIGHTS
from nisqa_b200 import synth
from oracle import nisqa_oracle as O

CASES = [("nisqa_48k_3s", "nisqa.tar"), ("nisqa_mixed", "nisqa.tar"), ("nisqa_48k_10s", "nisqa.tar"),
         ("mos_only_48k", "nisqa_mos_only.tar"), ("tts_16k", "nisqa_tts.tar")]


@pytest.mark.parametrize("name,ckpt", CASES)
def test_oracle_matches_reference_modules(name, ckpt):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    for i, (seed, sec, sr) in enumerate(zip(g["seeds"], g["seconds"], g["sr"])):
        pcm = synth.synth_speech_pcm16(int(seed), float(sec), int(sr))
        taps = {}
        sc, nseg, st = O.predict_pcm(args, sd, pcm.astype(np.float32) / 32768.0, int(sr), taps)
        assert st == O.STATUS_OK
        assert nseg == int(g["n_segments"][i])                        # bit-exact segment count
        assert taps["cnn_feat"].shape[0] == nseg
        np.testing.assert_allclose(taps["cnn_feat"].numpy(), g["cnn_%d" % i], rtol=0, atol=2e-5)
        np.testing.assert_allclose(taps["td_out"].numpy(), g["td_%d" % i], rtol=0, atol=2e-5)
        np.testing.assert_allclose(sc, g["scores"][i], rtol=0, atol=5e-6)
        if "mel_%d" % i in g:
            np.testing.assert_array_equal(taps["mel_db"], g["mel_%d" % i])


def _variant(name):
    from oracle import variants as V
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, V.VARIANTS[name][0]))
    return V.variant_checkpoint(name, args, sd)


def test_oracle_matches_reference_modules_on_the_variants():
    """SURVEY.md 8f.4: the other pooling modules and the positional encoding.  tests/golden/variants.npz holds the
    scores of the UNMODIFIED reference modules built with each variant's options and loaded (strict) with the seeded
    variant weights of oracle/variants.py (oracle/make_variant_golden.py)."""
    from oracle import variants as V
    g = np.load(os.path.join(GOLDEN, "variants.npz"))
    assert sorted(g.files) == sorted(V.VARIANTS)
    for name in V.VARIANTS:
        args, sd = _variant(name)
        for i, (seed, sec, sr) in enumerate(V.CLIPS):
            pcm = synth.synth_speech_pcm16(seed, sec, sr)
            sc, nseg, st = O.predict_pcm(args, sd, pcm.astype(np.float32) / 32768.0, sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


def test_oracle_matches_reference_double_ended_model():
    """SURVEY.md 8f.4: NISQA_DE (lib:272-424) - alignment (dot / cosine / distance, hard / soft), fusion (three modes),
    second self-attention stack (with and without positional encoding).  tests/golden/variants_de.npz holds the scores
    of the UNMODIFIED reference NISQA_DE run through nisqaModel(mode='predict_csv', csv_ref=...) in padded batches of
    two pairs (oracle/make_variant_golden.py); the oracle restates one pair at a time."""
    from oracle import variants as V
    g = np.load(os.path.join(GOLDEN, "variants_de.npz"))
    assert sorted(g.files) == sorted(V.DE_VARIANTS)
    bargs, bsd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    for name in V.DE_VARIANTS:
        args, sd = V.de_checkpoint(name, bargs, bsd)
        for i, pair in enumerate(V.DE_PAIRS):
            deg, srd, ref, srr = V.de_pair_pcm(pair)
            sc, _, st = O.predict_pcm_de(args, sd, deg.astype(np.float32) / 32768.0, srd, ref.astype(np.float32) / 32768.0, srr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


def test_reference_results_do_not_depend_on_batch_composition():
    """SURVEY.md 0.7: the per-clip (unpadded) oracle is equivalent to the padded batches."""
    g = np.load(os.path.join(GOLDEN, "nisqa_mixed.npz"))
    assert np.abs(g["scores"] - g["scores_bs8"]).max() < 2e-6


def test_segment_counts_formula():
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    assert O.segment_counts(480000, 48000, args) == (1001, 247, O.STATUS_OK)
    assert O.segment_counts(14 * 480 - 1, 48000, args)[2] == O.STATUS_TOO_SHORT     # 14 frames
    assert O.segment_counts(14 * 480, 48000, args) == (15, 1, O.STATUS_OK)
    # 1300 segments is the maximum: n_wins = 5197..5200 -> frames 5211..5214
    assert O.segment_counts((5214 - 1) * 480, 48000, args) == (5214, 1300, O.STATUS_OK)
    assert O.segment_counts((5215 - 1) * 480, 48000, args)[1:] == (1301, O.STATUS_TOO_LONG)
    targs, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_tts.tar"))
    assert O.segment_counts(160000, 16000, targs) == (1001, 987, O.STATUS_OK)
