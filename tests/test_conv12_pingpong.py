"""The ping-pong schedule of the fused conv1 + conv2 kernel (conv12_kernel, csrc/conv_split.cu): the CTA's i-th tile
goes to MMA warpgroup i & 1 and to A buffer i % 3, whose full / empty barriers wait on parity (i / 3) & 1.  Which
warpgroup gets a CTA's last tile, whether warpgroup 1 gets any, and how often each buffer's barriers change parity
depend on how many tiles a CTA gets, so the segment counts here are 1, 2 and n_sm k + r for k = 1 .. 7 and r = -1, 0, 1:
CTAs with 1 through 8 tiles, a warpgroup 1 with no tile, and every buffer's barriers through at least two phase changes.
Both CNN geometries (AdaptCNN: nisqa.tar, StandardCNN: nisqa_tts.tar).

Pass condition: pool2 (the fused kernel's output) and the scores are bit-identical to the separate conv1 / conv2
kernels (conv12 = 0).
"""
import os

import numpy as np
import pytest

from conftest import WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import nisqa_oracle as O
from test_conv12_pipeline import _n_sm, _samples_for, _segment_plan

pytestmark = pytest.mark.gpu


def _totals():
    n_sm = _n_sm()
    out = {1, 2}
    for k in range(1, 8):
        out |= {k * n_sm - 1, k * n_sm, k * n_sm + 1}
    return sorted(out)


@pytest.mark.parametrize("ckpt,sr", [("nisqa.tar", 48000), ("nisqa_tts.tar", 16000)], ids=["adapt", "standard"])
def test_pingpong_matches_separate_kernels_for_every_tile_count(built_lib, ckpt, sr):
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    cfg = E.config_from_args(args)
    eng = E.Engine(cfg, 0)
    try:
        eng.load_state_dict(sd)
        for total in _totals():
            plan = _segment_plan(total)
            pcm = [synth.synth_speech_pcm16(2000 + total + i, _samples_for(cfg, sr, n) / sr, sr)
                   for i, n in enumerate(plan)]
            out = {}
            for fused in (0, 1):
                eng.set_option("conv12", fused)
                scores, nseg, status = eng.predict_pcm(pcm, [sr] * len(pcm))
                out[fused] = (scores.copy(), nseg.copy(), status.copy(), eng.stage_dump(E.STAGE_POOL2))
            assert np.all(out[1][2] == 0)
            np.testing.assert_array_equal(out[1][1], np.asarray(plan, dtype=np.int32))
            for i in range(4):
                np.testing.assert_array_equal(out[1][i], out[0][i], err_msg="n_seg %d" % total)
    finally:
        eng.close()
