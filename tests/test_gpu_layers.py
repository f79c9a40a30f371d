"""Each kernel stage on its own against a float64 reference of that stage (tests/stage_ref.py), on an H100.

A check takes the engine's dump of a stage's input, computes that one stage in float64 on the host and compares the
engine's dump of the stage's output with it:

    |got - ref| <= bound,   bound = TAU * (magnitude of the stage's terms) (+ SPLIT |ref| for fp16 plane pairs)

TAU = 2^-18 is about 15x above what fp32 conv2d measures against float64 and about 30x below a two-term split with
one correction term dropped, so a fault confined to a few rows (a halo row, a tile's last segment, one K chunk)
fails here while the end-to-end tolerances of test_gpu_parity.py would let it through.  Every test prints the
measured max |got - ref| / bound per stage.

The batches are chosen where the kernels go wrong: totals of 1..12 segments (every remainder of the tile sizes G =
1, 3, 9, 12, and fewer tiles than SMs), and one long batch in which every CTA of every conv layer walks at least
four tiles (so every mbarrier phase flips several times), a one-segment clip sits between long clips (segments of
different clips share a tile), and the self-attention clips are 1, 63, 64, 65, 128, 129 and 1297..1300 segments
long; for the BiLSTM, batches that select 1, 2 and 4 clips per CTA.  Every conv check runs on the fused conv1+conv2
tensor-core path, the separate tensor-core kernels and the fp32 FFMA kernels.
"""
import os

import numpy as np
import pytest
import torch

import stage_ref as R
from conftest import WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import nisqa_oracle as O
from rescale import rescale

pytestmark = pytest.mark.gpu

SR = 16000
PATHS = {"tc_fused": (1, 1), "tc_separate": (1, 0), "ffma": (0, 0)}      # (conv_tc, conv12)
N_SM = 132
SUBSAMPLE = 17           # long batch: every 17th segment (coprime with every G) + each layer's last wave of tiles

CONV_STAGES = ["pool1", "pool2", "conv3", "pool3", "conv5"]
SHAPES = {"adapt": {"pool1": (16, 24, 7), "pool2": (32, 12, 5), "conv3": (64, 12, 5), "pool3": (64, 6, 3), "conv5": (64, 6, 3)},
          "standard": {"pool1": (16, 24, 8), "pool2": (32, 12, 4), "conv3": (64, 12, 4), "pool3": (64, 6, 2), "conv5": (64, 6, 2)}}
TILE_G = {"adapt": {1: 1, 2: 1, 3: 3, 4: 3, 5: 9, 6: 9}, "standard": {1: 1, 2: 1, 3: 3, 4: 3, 5: 12, 6: 12}}
DUMP = {"mel": E.STAGE_MEL_DB, "pool1": E.STAGE_POOL1, "pool2": E.STAGE_POOL2, "conv3": E.STAGE_CONV3,
        "pool3": E.STAGE_POOL3, "conv5": E.STAGE_CONV5, "cnn_feat": E.STAGE_CNN_FEAT, "td_in": E.STAGE_TD_IN,
        "td_out": E.STAGE_TD_OUT}


def _pcm(args, n_seg, seed):
    hop = int(SR * args["ms_hop_length"])
    n = (15 + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * hop
    y = synth.synth_speech_pcm16(seed, n / SR + 0.05, SR)[:n]
    assert O.segment_counts(n, SR, args)[1] == n_seg
    return y


def _batches(args):
    small = [[t] for t in range(1, 13)]
    if args["td"] == "self_att":
        # 5645 segments: 628 tiles of 9 = at least 4 per CTA of every layer
        long_ = [1300, 1, 1299, 63, 1298, 64, 1297, 65, 128, 129, 1]
        return small + [long_]
    # BiLSTM: <= 66 clips -> 1 clip per CTA, <= 132 -> 2, more -> 4; 140 clips, about 8100 segments (>= 4 tiles of 12)
    two = [1 + i % 5 for i in range(100)]
    four = [1000, 1, 999, 998, 997, 996, 995] + [1 + i % 17 for i in range(133)]
    return small + [two, four]


def _checkpoints():
    return ["nisqa.tar", "nisqa_tts.tar", "nisqa.tar@rescaled"]


def _load(name):
    ckpt, _, variant = name.partition("@")
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    if variant:                       # conv1 out by 2^16, conv4 out by 2^-16: outside the old fixed fp16 range
        sd = rescale(rescale(sd, 1, 16), 4, -16)
    return args, sd


def _subset(n, g):
    if n <= 12 * N_SM:
        return torch.arange(n)
    keep = set(range(0, n, SUBSAMPLE)) | set(range(max(0, n - g * N_SM), n))
    return torch.tensor(sorted(keep))


class Ratios(dict):
    def add(self, name, got, ref, bound):
        r = R.ratio(got, ref, bound)
        self[name] = max(self.get(name, 0.0), r)


def _check_call(eng, args, sd, path, lens, seed, ratios):
    kind = args["cnn_model"]
    clips = [_pcm(args, n, seed + i) for i, n in enumerate(lens)]
    scores, nseg, status = eng.predict_pcm(clips, [SR] * len(clips))
    assert np.all(status == E.CLIP_OK) and nseg.tolist() == lens
    N = int(sum(lens))
    fused = path == "tc_fused"
    names = ["mel"] + [s for s in CONV_STAGES if not (fused and s == "pool1")] + ["cnn_feat", "td_out"]
    if args["td"] == "self_att":
        names.append("td_in")
    d = {k: eng.stage_dump(DUMP[k]) for k in names}
    act = {k: torch.from_numpy(d[k]).double().reshape(N, *SHAPES[kind][k]) for k in CONV_STAGES if k in d}

    # ---- conv stages
    n_frames = [O.segment_counts(len(c), SR, args)[0] for c in clips]
    offs = np.concatenate([[0], np.cumsum(n_frames)]) * 48
    seg = torch.cat([O.segments(d["mel"][offs[i]:offs[i + 1]].reshape(48, -1), args) for i in range(len(clips))]).double()
    chain = [("mel", "pool1", [1]), ("pool1", "pool2", [2])] if not fused else [("mel", "pool2", [1, 2])]
    chain += [("pool2", "conv3", [3]), ("conv3", "pool3", [4]), ("pool3", "conv5", [5]), ("conv5", "cnn_feat", [6])]
    feat = torch.from_numpy(d["cnn_feat"]).double().reshape(N, -1)
    for src, dst, layers in chain:
        idx = _subset(N, TILE_G[kind][layers[-1]])
        x = seg[idx] if src == "mel" else act[src][idx]
        err = None
        for layer in layers:
            x, err = R.conv_layer(sd, args, layer, x, err)
        if dst == "cnn_feat":
            x, err = R.cnn_tail(sd, args, x, err)
            got = feat[idx]
        else:
            got = act[dst][idx]
        ratios.add("%s->%s" % (src, dst), got, x, err)

    # ---- time dependency and pooling, per clip
    starts = np.concatenate([[0], np.cumsum(lens)])
    zero = torch.zeros_like(feat)
    if args["td"] == "self_att":
        td_in = torch.from_numpy(d["td_in"]).double().reshape(N, 64)
        ref, b = R.td_in(sd, feat, zero)
        ratios.add("cnn_feat->td_in", td_in, ref, b)
        td_out = torch.from_numpy(d["td_out"]).double().reshape(N, 64)
        for i in range(len(clips)):
            x = td_in[starts[i]:starts[i + 1]]
            ref, b = R.sa_stack(sd, x, torch.zeros_like(x))
            ratios.add("td_in->td_out", td_out[starts[i]:starts[i + 1]], ref, b)
    else:
        td_out = torch.from_numpy(d["td_out"]).double().reshape(N, -1)
        outs = R.bilstm(sd, [feat[starts[i]:starts[i + 1]] for i in range(len(clips))])
        for i, (ref, b) in enumerate(outs):
            ratios.add("cnn_feat->td_out", td_out[starts[i]:starts[i + 1]], ref, b)
    for i in range(len(clips)):
        x = td_out[starts[i]:starts[i + 1]]
        ref, b = R.pool_heads(sd, args, x, torch.zeros_like(x))
        ratios.add("td_out->scores", scores[i], ref, b)


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("ckpt", _checkpoints())
def test_every_stage_against_float64(built_lib, ckpt, path):
    args, sd = _load(ckpt)
    eng = E.Engine(E.config_from_args(args), 0)
    ratios = Ratios()
    try:
        tc, c12 = PATHS[path]
        eng.set_option("conv_tc", tc)
        eng.set_option("conv12", c12)
        eng.set_option("keep_td_out", 1)
        eng.load_state_dict(sd)
        for j, lens in enumerate(_batches(args)):
            _check_call(eng, args, sd, path, lens, 1000 * (j + 1), ratios)
    finally:
        eng.close()
    print("\n%s %s max |got - ref| / bound: %s" % (ckpt, path, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios
