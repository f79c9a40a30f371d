"""Checkpoints rescaled by powers of two (tests/rescale.py) compute the same function.

The oracle pins the premise on the CPU: its scores are bit-identical for every conv layer and k = +-12, +-24.  The
engine stores activations as fp16 pairs with a power-of-two scale per channel, chosen from that channel's folded
BatchNorm, and weights with one per layer, chosen from the weights (pack_weights), so its scores must be bit-identical
too - on every conv path - and within the usual 1e-4 of the oracle.  A fixed fp16 range would clamp or lose the lo half
instead.  tests/test_channel_rescale.py rescales channel by channel.
"""
import os

import numpy as np
import pytest
import torch

from conftest import WEIGHTS
from nisqa_b200 import synth
from oracle import nisqa_oracle as O
from rescale import rescale

KS = (-24, -12, 12, 24)
CASES = [("nisqa.tar", layer) for layer in range(1, 7)] + [("nisqa_tts.tar", layer) for layer in range(1, 6)]


def _clip(sr=16000):
    return synth.synth_speech_f32(77, 2.0, sr), sr


def test_rescale_is_exact_on_the_weights():
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    for layer in range(1, 7):
        back = rescale(rescale(sd, layer, 24), layer, -24)
        assert all(torch.equal(back[k], sd[k]) for k in sd)
        changed = [k for k in sd if not torch.equal(rescale(sd, layer, 12)[k], sd[k])]
        assert len(changed) == 3, changed                        # BN weight, BN bias, the consumer's weight


@pytest.mark.parametrize("ckpt", ["nisqa.tar", "nisqa_tts.tar"])
def test_oracle_scores_are_bit_identical_under_rescaling(ckpt):
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    y, sr = _clip()
    spec = O.mel_db(y, sr, args)
    base = O.forward_from_mel(args, sd, spec)
    for c, layer in CASES:
        if c != ckpt:
            continue
        for k in KS:
            np.testing.assert_array_equal(O.forward_from_mel(args, rescale(sd, layer, k), spec), base, err_msg=str((layer, k)))


PATHS = {"tc_fused": (1, 1), "tc_separate": (1, 0), "ffma": (0, 0)}      # (conv_tc, conv12)


@pytest.mark.gpu
@pytest.mark.parametrize("ckpt", ["nisqa.tar", "nisqa_tts.tar"])
def test_engine_scores_are_bit_identical_under_rescaling(built_lib, ckpt):
    from nisqa_b200 import engine as E
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    clips = [synth.synth_speech_pcm16(s, sec, 16000) for s, sec in ((81, 2.0), (82, 0.15), (83, 4.3))]
    ref = np.stack([O.predict_pcm(args, sd, c.astype(np.float32) / np.float32(32768.0), 16000)[0] for c in clips])
    eng = E.Engine(E.config_from_args(args), 0)
    worst = {}
    try:
        for path, (tc, c12) in PATHS.items():
            eng.set_option("conv_tc", tc)
            eng.set_option("conv12", c12)
            eng.load_state_dict(sd)
            base, _, st = eng.predict_pcm(clips, [16000] * 3)
            assert np.all(st == 0) and np.abs(base - ref).max() <= 1e-4
            for c, layer in CASES:
                if c != ckpt:
                    continue
                for k in KS:
                    eng.load_state_dict(rescale(sd, layer, k))
                    got, _, st = eng.predict_pcm(clips, [16000] * 3)
                    assert np.all(st == 0)
                    worst[(path, layer, k)] = float(np.abs(got - base).max())
                    assert np.abs(got - ref).max() <= 1e-4, (path, layer, k, float(np.abs(got - ref).max()))
                    np.testing.assert_array_equal(got, base, err_msg=str((path, layer, k)))
    finally:
        eng.close()
    print("max |score - unscaled score|:", {"%s L%d 2^%d" % key: v for key, v in worst.items() if v})
