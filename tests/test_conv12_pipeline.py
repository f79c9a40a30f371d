"""The mel ring of the fused conv1 + conv2 kernel (conv12_kernel, csrc/conv_split.cu): one thread of the conv1 role
copies each segment's mel block into a ring of SpFused::MEL_R shared-memory slots two tiles ahead, and the persistent
CTAs walk the segments with a grid stride.  The ring's prologue, wrap-around and tail depend on how many tiles a CTA
gets, so the segment counts here give CTAs fewer tiles than the ring has slots, exactly that many, and more:
1, n_sm - 1, n_sm, n_sm + 1 and k n_sm - 1, k n_sm, k n_sm + 1 for k up to MEL_R + 1.  The clips mix long ones with
one-segment ones, and the last clip's last segment ends at the last mel frame of the pass (the end of the copied
range).  Both CNN geometries (AdaptCNN: nisqa.tar, StandardCNN: nisqa_tts.tar).

Pass condition: pool2 (the fused kernel's output) and the scores are bit-identical to the separate conv1 / conv2
kernels (conv12 = 0), which read the mel straight from global memory.
"""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import nisqa_oracle as O

pytestmark = pytest.mark.gpu

HEADER = os.path.join(ROOT, "nisqa_b200", "csrc", "conv_split.cuh")
SEG_LEN = 15


def _mel_ring_slots():
    return int(re.search(r"static constexpr int MEL_R = (\d+);", open(HEADER).read()).group(1))


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _samples_for(cfg, sr, n_seg):
    """The shortest clip with n_seg segments whose last segment ends at the clip's last frame."""
    want = SEG_LEN + cfg.seg_hop * (n_seg - 1)
    lo, hi = 1, 1
    while E.segment_counts(cfg, hi, sr)[0] < want:
        hi *= 2
    while lo < hi:                                   # n_frames is monotone in the sample count
        mid = (lo + hi) // 2
        if E.segment_counts(cfg, mid, sr)[0] < want:
            lo = mid + 1
        else:
            hi = mid
    n_frames, got, status = E.segment_counts(cfg, lo, sr)
    assert (n_frames, got, status) == (want, n_seg, 0), (n_seg, n_frames, got, status)
    return lo


def _segment_plan(total, long_seg=53):
    """Segments per clip summing to `total`: long clips separated by one-segment clips, then the remainder."""
    plan = []
    while total > 0:
        n = min(total, long_seg if len(plan) % 2 == 0 else 1)
        plan.append(n)
        total -= n
    return plan


@pytest.fixture(scope="module", params=[("nisqa.tar", 48000), ("nisqa_tts.tar", 16000)], ids=["adapt", "standard"])
def engine(request, built_lib):
    ckpt, sr = request.param
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    cfg = E.config_from_args(args)
    eng = E.Engine(cfg, 0)
    eng.load_state_dict(sd)
    yield eng, cfg, sr
    eng.close()


def _totals():
    n_sm, r = _n_sm(), _mel_ring_slots()
    out = {1, n_sm - 1, n_sm, n_sm + 1}
    for k in range(2, r + 2):
        out |= {k * n_sm - 1, k * n_sm, k * n_sm + 1}
    return sorted(out)


def test_fused_conv12_matches_separate_kernels_for_every_ring_fill(engine):
    eng, cfg, sr = engine
    for total in _totals():
        plan = _segment_plan(total)
        pcm = [synth.synth_speech_pcm16(1000 + total + i, _samples_for(cfg, sr, n) / sr, sr) for i, n in enumerate(plan)]
        srs = [sr] * len(pcm)
        out = {}
        try:
            for fused in (0, 1):
                eng.set_option("conv12", fused)
                scores, nseg, status = eng.predict_pcm(pcm, srs)
                out[fused] = (scores.copy(), nseg.copy(), status.copy(), eng.stage_dump(E.STAGE_POOL2))
        finally:
            eng.set_option("conv12", 1)
        assert np.all(out[1][2] == 0)
        np.testing.assert_array_equal(out[1][1], np.asarray(plan, dtype=np.int32))
        for i in range(4):
            np.testing.assert_array_equal(out[1][i], out[0][i], err_msg="n_seg %d" % total)
