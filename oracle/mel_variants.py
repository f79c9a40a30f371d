"""Checkpoints trained with other Mel-spectrogram segment shapes (ms_n_mels x ms_seg_length): AdaptCNN (any shape is
pooled to 24 x 7 by its first adaptive max-pool, lib:690-691), SkipCNN and DFF (fan_in = n_mels * seg_length,
lib:504-583), behind self-attention, no td, or NISQA_DE's stack.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A mel variant is an existing variant (a shipped checkpoint, an
oracle/variants.py VARIANTS / DE_VARIANTS entry) with ms_n_mels / ms_seg_length (and ms_seg_hop_length) switched.
AdaptCNN's weights do not depend on the input shape and are reused unchanged.  For SkipCNN / DFF, the first Linear - and,
where its input width changes, the Linear behind it - is re-seeded here at the new width (NumPy PCG64: the same here, in
oracle/make_mel_golden.py that feeds these checkpoints to the UNMODIFIED reference modules, and on the GPU box).  The
pooled score Linear of the td = 'skip' variant is scaled by sqrt(64 / D) as in oracle/td_skip_variants.py, so that every
score stays in the MOS range.
"""
import math

import numpy as np
import torch

from oracle.td_pair_variants import TD_PAIR_CLIPS, _pool
from oracle.variants import DE_PAIRS, de_checkpoint, variant_checkpoint

# name -> (base checkpoint, oracle/variants.py VARIANTS entry (or "de:" + a DE_VARIANTS entry) or None, args overrides,
#          re-seeded Linear widths {state-dict prefix: n_out} for SkipCNN / DFF)
MEL_VARIANTS = {
    # AdaptCNN, only ms_n_mels changed (nisqa_mos_only.tar's weights as they are)
    "mos_adapt_m64_s15": ("nisqa_mos_only.tar", None, dict(ms_n_mels=64), {}),
    # AdaptCNN, only ms_seg_length changed (the reference's segment_specs takes odd lengths only, lib:2253-2254)
    "mos_adapt_m48_s21": ("nisqa_mos_only.tar", None, dict(ms_seg_length=21), {}),
    # NISQA_DIM, fewer bands and shorter segments than the pool1 grid (H 32 < 48, W 11 < 15)
    "dim_adapt_m32_s11": ("nisqa.tar", None, dict(ms_n_mels=32, ms_seg_length=11), {}),
    # AdaptCNN + its Linear (cnn_fc_out_h 128), 128 bands: the front end's second band round, empty filters at 8 kHz
    "dim_adapt_fc128_m128_s21": ("nisqa.tar", "dim_adapt_fc", dict(ms_n_mels=128, ms_seg_length=21), {}),
    # 80 bands x 31 frames at segment hop 2
    "mos_adapt_m80_s31_hop2": ("nisqa_mos_only.tar", None, dict(ms_n_mels=80, ms_seg_length=31, ms_seg_hop_length=2), {}),
    # raw SkipCNN: 600 features (padded to 640) into self-attention
    "mos_skipcnn_m40_s15_sa": ("nisqa_mos_only.tar", "mos_skip", dict(ms_n_mels=40), {"time_dependency.model.linear.": 64}),
    # SkipCNN + Linear 256 over fan_in 2976 (padded to 3008), NISQA_DIM
    "dim_skipcnn_fc256_m96_s31": ("nisqa.tar", "dim_skip_fc", dict(ms_n_mels=96, ms_seg_length=31, cnn_fc_out_h=256),
                                  {"cnn.model.linear.": 256, "time_dependency.model.linear.": 64}),
    # DFF (256) over fan_in 576
    "mos_dff_m64_s9": ("nisqa_mos_only.tar", "mos_dff", dict(ms_n_mels=64, ms_seg_length=9), {"cnn.model.lin1.": 256}),
    # td = 'skip': raw SkipCNN rows (680, padded to 704) pooled directly by PoolAvg
    "mos_skipcnn_skip_m40_s17_avg": ("nisqa_mos_only.tar", "mos_skip", dict(ms_n_mels=40, ms_seg_length=17, td="skip",
                                                                          td_2="skip", **_pool("avg")), {}),
    # NISQA_DE: AdaptCNN at 64 x 15 on both signals
    "de_adapt_m64_s15": ("nisqa_mos_only.tar", "de:de_cosine_hard", dict(ms_n_mels=64), {}),
}
# the single-ended variants are scored on TD_PAIR_CLIPS, the NISQA_DE one on DE_PAIRS
MEL_CLIPS = TD_PAIR_CLIPS
MEL_DE_PAIRS = DE_PAIRS


def fan_in(args):
    """SkipCNN / DFF input width (lib:520 / 556)"""
    return int(args["ms_n_mels"]) * int(args["ms_seg_length"])


def mel_checkpoint(name, base_args, base_sd):
    """-> (args, state_dict) of a MEL_VARIANTS entry; base_args / base_sd are those of its base checkpoint."""
    _, parent, over, reseed = MEL_VARIANTS[name]
    if parent is None:
        args, sd = dict(base_args), dict(base_sd)
    elif parent.startswith("de:"):
        args, sd = de_checkpoint(parent[3:], base_args, base_sd)
    else:
        args, sd = variant_checkpoint(parent, base_args, base_sd)
    args = dict(args)
    args.update(over)
    sd = dict(sd)
    rng = np.random.default_rng(sum(map(ord, name)) + 11)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))      # noqa: E731
    n_in = fan_in(args)
    for prefix, n_out in reseed.items():
        # (SkipCNN's first Linear at half the scale of oracle/variants.py's: its features have a large mean over time)
        scale = 0.5 if prefix == "cnn.model.linear." else 1.0
        sd[prefix + "weight"] = t(rng.standard_normal((n_out, n_in)) * scale / math.sqrt(n_in))
        sd[prefix + "bias"] = t(rng.normal(0, 0.05, n_out))
        n_in = n_out
    if args.get("td") == "skip":
        # no time-dependency model: the pooling module reads the framewise rows (n_in wide), its score Linear scaled
        sd = {k: v for k, v in sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers."))}
        sd["pool.model.linear.weight"] = t(rng.standard_normal((1, n_in)) * 0.3 * math.sqrt(64.0 / n_in))
        sd["pool.model.linear.bias"] = t(rng.uniform(1.0, 4.0, 1))
    return args, sd
