"""Checkpoints without a time-dependency model (td = 'skip', TimeDependency._skip, lib:839-895): the pooling module reads
the framewise rows themselves, or td_2 (self-attention, or an LSTM behind StandardCNN) reads them, for NISQA and
NISQA_DIM.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A skip variant is built by oracle/td_pair_variants.py's
``td_pair_checkpoint`` (its seeding, its framewise weights and its td_2 / pooling weights) on a shipped checkpoint or an
oracle/variants.py framewise model (a VARIANTS entry; for rows wider than any entry has, the SkipCNN of one with its
Linear re-seeded here at that width).  The score Linear of every head is then scaled by sqrt(64 / D), D the width of the
rows it reads, so that the scores stay in the MOS range at D = 384..2048 (oracle/make_td_skip_golden.py feeds these
checkpoints to the UNMODIFIED reference modules).
"""
import math

import numpy as np
import torch

from oracle.td_pair_variants import _pool, framewise_fan_out, fan_out, lstm, sa, td_pair_checkpoint
from oracle.variants import variant_checkpoint

SKIP = {"td": "skip"}

# name -> (base checkpoint, framewise parent: an oracle/variants.py VARIANTS name, (SkipCNN VARIANTS name, Linear width)
# or None, args overrides)
TD_SKIP_VARIANTS = {
    # AdaptCNN's 384 conv6 features (engine column order h*64 + c), PoolAttFF
    "mos_adapt_skip_attff": ("nisqa_mos_only.tar", None, dict(SKIP, td_2="skip", **_pool("att", 128))),
    # AdaptCNN + its Linear (cnn_fc_out_h 128), five PoolMax heads
    "dim_adapt_fc128_skip_max": ("nisqa.tar", "dim_adapt_fc", dict(SKIP, td_2="skip", **_pool("max"))),
    # StandardCNN's 768 conv6 features, PoolMax
    "mos_std_skip_max": ("nisqa_tts.tar", None, dict(SKIP, cnn_fc_out_h=None, td_2="skip", **_pool("max"))),
    # five PoolAttFF heads over 768-wide rows (StandardCNN, segment hop 1: the long-clip case of ms_max_segments 6000)
    "dim_std_skip_attff": ("nisqa_tts.tar", None, dict(SKIP, model="NISQA_DIM", cnn_fc_out_h=None, td_2="skip",
                                                        **_pool("att", 128))),
    # StandardCNN's fc_out at a width that is not a multiple of 64 (100, padded to 128), PoolLastStep
    "mos_std_fc100_skip_last": ("nisqa_tts.tar", None, dict(SKIP, cnn_fc_out_h=100, td_2="skip", **_pool("last_step"))),
    # raw SkipCNN (720 features, padded to 768), PoolAtt
    "mos_skipcnn_skip_att": ("nisqa_mos_only.tar", "mos_skip", dict(SKIP, td_2="skip", **_pool("att", None))),
    # SkipCNN's Linear at 2048: rows 2048 wide, five PoolAvg heads
    "dim_skipcnn_fc2048_skip_avg": ("nisqa.tar", ("dim_skip_fc", 2048), dict(SKIP, td_2="skip", **_pool("avg"))),
    # DFF (256), PoolAvg
    "mos_dff_skip_avg": ("nisqa_mos_only.tar", "mos_dff", dict(SKIP, td_2="skip", **_pool("avg"))),
    # td_2 = self-attention behind no td: AdaptCNN 384 -> d_model 128, PoolAttFF (logits fused into the stack)
    "mos_adapt_skip_sa128_attff": ("nisqa_mos_only.tar", None, dict(SKIP, **sa("td_2", 128, 256), **_pool("att", 128))),
    # NISQA_DIM: td_2's fan_out equals the framewise one (SkipCNN's Linear 128 -> d_model 128), PoolAtt
    "dim_skipcnn_fc128_skip_sa128_att": ("nisqa.tar", "dim_skip_fc", dict(SKIP, **sa("td_2", 128, 128, 2), **_pool("att", None))),
    # td_2 = LSTM behind no td (StandardCNN only): the shipped fc_out 20 -> BiLSTM 128, PoolLastStepBi
    "mos_std_fc20_skip_lstm128bi_lastbi": ("nisqa_tts.tar", None, dict(SKIP, **lstm("td_2", 128), **_pool("last_step_bi"))),
    # NISQA_DIM: fc_out 128 -> BiLSTM 64 (fan_out 128), five PoolAttFF heads
    "dim_std_fc128_skip_lstm64bi_attff": ("nisqa_tts.tar", None, dict(SKIP, model="NISQA_DIM", cnn_fc_out_h=128,
                                                                      **lstm("td_2", 64), **_pool("att", 128))),
}


def pooled_width(args):
    """width of the rows the pooling module reads"""
    return fan_out(args, "td_2", framewise_fan_out(args))


def td_skip_checkpoint(name, base_args, base_sd):
    """-> (args, state_dict) of a TD_SKIP_VARIANTS entry; base_args / base_sd are those of its base checkpoint."""
    base, parent, over = TD_SKIP_VARIANTS[name]
    if isinstance(parent, tuple):                 # SkipCNN with its Linear at a width no VARIANTS entry has
        parent, width = parent
        base_args, base_sd = variant_checkpoint(parent, base_args, base_sd)
        base_args = dict(base_args, cnn_fc_out_h=width)
        rng = np.random.default_rng(sum(map(ord, name)) + 3)
        # (half the scale of oracle/variants.py's Linears: SkipCNN's features have a large mean over time, and the
        # pooled scores must stay in the MOS range)
        base_sd = dict(base_sd, **{
            "cnn.model.linear.weight": torch.from_numpy((rng.standard_normal((width, 720)) * 0.5 / math.sqrt(720)).astype(np.float32)),
            "cnn.model.linear.bias": torch.from_numpy(rng.normal(0, 0.05, width).astype(np.float32))})
        parent = None
    args, sd = td_pair_checkpoint(name, base_args, base_sd, (base, parent, over))
    scale = math.sqrt(64.0 / pooled_width(args))
    heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    key = {"att": "linear3" if args.get("pool_att_h") else "linear2"}.get(args["pool"], "linear")
    for pf in heads:
        sd[pf + key + ".weight"] = sd[pf + key + ".weight"] * scale
    return args, sd
