"""Self-attention stacks wider than 64: td_sa_d_model / td_2_sa_d_model in {64, 128, 192, 256} and any feed-forward
width td_sa_h / td_2_sa_h (a multiple of 64 up to 4096), one head.

CPU: the configuration accepts exactly that range (and refuses the rest, naming the value), the C struct layout of the
new fields, and the oracle against the scores of the unmodified reference modules (tests/golden/variants_wide.npz,
oracle/make_wide_golden.py).
GPU: every wide variant through the C ABI against the reference scores and the oracle, alone == in a batch, several
passes == one pass; and the time-dependency stages on their own against float64 (tests/stage_ref.py) for
d_model 128, 192, 256 x feed-forward 64, 1024.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import stage_ref as R
from conftest import GOLDEN, ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import nisqa_oracle as O
from oracle import wide_variants as V

SCORE_TOL = 1e-4


def _wide(name, spec=None):
    base = (spec or V.WIDE_VARIANTS[name])[0]
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.wide_checkpoint(name, args, sd, spec)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(V.WIDE_VARIANTS))
def test_config_fills_the_widths(name):
    args, _ = _wide(name)
    c = E.config_from_args(args)
    assert (c.sa_d_model, c.sa_ff) == (args["td_sa_d_model"], args["td_sa_h"])
    if args.get("td_2") == "self_att":
        assert (c.td2_d_model, c.td2_ff) == (args["td_2_sa_d_model"], args["td_2_sa_h"])
    else:
        assert (c.td2_d_model, c.td2_ff) == (0, 0)


def test_config_refuses_widths_outside_the_kernels():
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    de = dict(args, model="NISQA_DE", td_2="self_att", td_2_sa_d_model=64, td_2_sa_nhead=1, td_2_sa_h=64, td_2_sa_num_layers=2,
              de_align="dot", de_align_apply="soft", de_fuse="x/y/-", de_fuse_dim=None)
    for bad, what in ((dict(args, td_sa_d_model=96), "96"), (dict(args, td_sa_d_model=320), "320"),
                      (dict(args, td_sa_h=100), "100"), (dict(args, td_sa_h=4160), "4160"),
                      (dict(args, td_sa_d_model=128, td_sa_nhead=2), "nhead"),
                      (dict(de, td_sa_d_model=128), "128"), (dict(de, td_2_sa_d_model=128), "128"),
                      (dict(args, td_2="self_att", td_2_sa_d_model=128, td_2_sa_nhead=1, td_2_sa_h=64, td_2_sa_num_layers=1), "128")):
        with pytest.raises(NotImplementedError, match=what):
            E.config_from_args(bad)
    c = E.config_from_args(dict(args, td_sa_d_model=256, td_sa_h=4096))
    assert (c.sa_d_model, c.sa_ff) == (256, 4096)
    assert E.config_from_args(dict(de, td_sa_h=512)).sa_ff == 512


def test_struct_layout_of_the_width_fields(tmp_path):
    src = tmp_path / "layout.c"
    fields = ["de_fuse_dim", "sa_d_model", "sa_ff", "td2_d_model", "td2_ff"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu %d'
                   + " %zu" * len(fields) + '\\n", sizeof(nisqa_config), NISQA_B200_ABI_VERSION'
                   + "".join(", offsetof(nisqa_config, %s)" % f for f in fields) + ");return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [ctypes.sizeof(E.NisqaConfig), E.ABI_VERSION] + [getattr(E.NisqaConfig, f).offset for f in fields]
    assert E.ABI_VERSION == 4


def test_oracle_matches_reference_modules_on_the_wide_variants():
    g = np.load(os.path.join(GOLDEN, "variants_wide.npz"))
    assert sorted(g.files) == sorted(V.WIDE_VARIANTS)
    for name in V.WIDE_VARIANTS:
        args, sd = _wide(name)
        for i, (seed, sec, sr) in enumerate(V.WIDE_CLIPS):
            sc, _, st = O.predict_pcm(args, sd, _f32(synth.synth_speech_pcm16(seed, sec, sr)), sr)
            assert st == O.STATUS_OK
            np.testing.assert_allclose(sc, g[name][i], rtol=0, atol=5e-6, err_msg=name)


# ------------------------------------------------------------------------------------------------------------ GPU
SR = 16000


def _pcm(args, n_seg, seed):
    """a 16 kHz clip of exactly n_seg segments"""
    hop = int(SR * args["ms_hop_length"])
    n = (15 + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * hop
    y = synth.synth_speech_pcm16(seed, n / SR + 0.05, SR)[:n]
    assert O.segment_counts(n, SR, args)[1] == n_seg
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.WIDE_VARIANTS))
def test_wide_variant_through_the_c_abi(built_lib, name):
    args, sd = _wide(name)
    g = np.load(os.path.join(GOLDEN, "variants_wide.npz"))[name]
    pcm = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in V.WIDE_CLIPS]
    srs = [c[2] for c in V.WIDE_CLIPS]
    # a one-segment (15-frame) clip between long clips, 97 segments (not a multiple of the key block of 64) and, for the
    # widest stack, a 1300-segment clip
    extra = [_pcm(args, 1, 7), _pcm(args, 97, 8)] + ([_pcm(args, 1300, 9)] if args["td_sa_d_model"] == 256 else [])
    batch = pcm[:2] + extra[:1] + pcm[2:] + extra[1:]
    bsr = srs[:2] + [SR] + srs[2:] + [SR] * (len(extra) - 1)
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        eng.load_state_dict(sd)
        scores, nseg, status = eng.predict_pcm(batch, bsr)
        assert np.all(status == E.CLIP_OK), name
        ours = np.concatenate([scores[:2], scores[3:3 + len(pcm) - 2]])
        err = float(np.abs(ours - g).max())
        print("\n%s: max |engine - reference| %.3g" % (name, err))
        assert err <= SCORE_TOL, (name, err)
        worst = 0.0
        for i, (p, sr) in enumerate(zip(batch, bsr)):
            ref, ns, st = O.predict_pcm(args, sd, _f32(p), sr)
            assert st == O.STATUS_OK and ns == nseg[i], (name, i)
            worst = max(worst, float(np.abs(scores[i] - ref).max()))
        print("%s: max |engine - oracle| %.3g over segment counts %s" % (name, worst, nseg.tolist()))
        assert worst <= SCORE_TOL, (name, worst)
        for i in (2, len(batch) - 1):                                    # alone == in the batch, bit for bit
            alone, _, _ = eng.predict_pcm(batch[i:i + 1], bsr[i:i + 1])
            np.testing.assert_array_equal(alone[0], scores[i])
    finally:
        eng.close()
    # several internal passes == one pass
    eng = E.Engine(E.config_from_args(args, max_chunk_segments=120), 0)
    try:
        eng.load_state_dict(sd)
        multi, nseg2, _ = eng.predict_pcm(batch, bsr)
        np.testing.assert_array_equal(nseg2, nseg)
        np.testing.assert_array_equal(multi, scores)
    finally:
        eng.close()


def _stage_spec(D, F):
    return ("nisqa.tar", None, {"td_sa_d_model": D, "td_sa_h": F})


@pytest.mark.gpu
@pytest.mark.parametrize("F", [64, 1024])
@pytest.mark.parametrize("D", [128, 192, 256])
def test_time_dependency_stages_against_float64(built_lib, D, F):
    """TD_IN, TD_OUT and the scores, each from the engine's own dump of the stage's input, against float64 (bound TAU =
    2^-18 times the magnitude of the stage's terms, tests/stage_ref.py)."""
    name = "stage_d%d_ff%d" % (D, F)
    args, sd = _wide(name, _stage_spec(D, F))
    lens = [1300, 1, 63, 64, 65, 129]
    clips = [_pcm(args, n, 100 + i) for i, n in enumerate(lens)]
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        eng.load_state_dict(sd)
        scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
        assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
        N = sum(lens)
        feat = torch.from_numpy(eng.stage_dump(E.STAGE_CNN_FEAT)).double().reshape(N, -1)
        td_in = torch.from_numpy(eng.stage_dump(E.STAGE_TD_IN)).double().reshape(N, D)
        td_out = torch.from_numpy(eng.stage_dump(E.STAGE_TD_OUT)).double().reshape(N, D)
    finally:
        eng.close()
    ratios = {}

    def add(k, got, ref, bound):
        ratios[k] = max(ratios.get(k, 0.0), R.ratio(got, ref, bound))
    ref, b = R.td_in(sd, feat, torch.zeros_like(feat))
    add("cnn_feat->td_in", td_in, ref, b)
    starts = np.concatenate([[0], np.cumsum(lens)])
    for i in range(len(lens)):
        x = td_in[starts[i]:starts[i + 1]]
        ref, b = R.sa_stack(sd, x, torch.zeros_like(x))
        add("td_in->td_out", td_out[starts[i]:starts[i + 1]], ref, b)
        y = td_out[starts[i]:starts[i + 1]]
        ref, b = R.pool_heads(sd, args, y, torch.zeros_like(y))
        add("td_out->scores", scores[i], ref, b)
    print("\nD %d F %d max |got - ref| / bound: %s" % (D, F, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios
