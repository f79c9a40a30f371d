"""AdaptCNN checkpoints trained with other adaptive max-pool sizes (cnn_pool_1 / cnn_pool_2 / cnn_pool_3, lib:586-710), behind
self-attention, no td, AdaptCNN's Linear or NISQA_DE's stack, at the shipped and at other Mel-spectrogram shapes and
channel counts.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A pool variant is an existing checkpoint (a shipped one, an
oracle/variants.py VARIANTS / DE_VARIANTS entry) with its pools (and possibly its Mel shape or channel counts) switched: the
six conv / BN layers are seeded as in oracle/cnn_width_variants.py, conv6 then as (c3, c3, 3, pool_3[1]) (its kernel is
3 x pool_3[1], lib:623-625), and the Linear that reads the CNN's c3 * pool_3[0] features (AdaptCNN's cnn.model.fc, td's
input Linear, or the pooling module's Linear behind td = 'skip'), NumPy PCG64: the same here, in
oracle/make_cnn_pool_golden.py that feeds these checkpoints to the UNMODIFIED reference modules, and on the GPU box.

The oracle is oracle/cnn_width_variants.py's ``adapt_cnn`` (``wide_cnn()``): it already reads the pools from ``args`` and
conv6's kernel from its tensor.
"""
import math

import numpy as np
import torch

from oracle.cnn_width_variants import seed_cnn
from oracle.td_pair_variants import TD_PAIR_CLIPS, _pool
from oracle.variants import DE_PAIRS, de_checkpoint, variant_checkpoint

SHIPPED_POOLS = ([24, 7], [12, 5], [6, 3])

# name -> (base checkpoint, oracle/variants.py VARIANTS entry (or "de:" + a DE_VARIANTS entry) or None, args overrides,
#          (cnn_c_out_1, cnn_c_out_2, cnn_c_out_3), (cnn_pool_1, cnn_pool_2, cnn_pool_3))
CNN_POOL_VARIANTS = {
    # every layer off the shipped geometry, conv6 (3, 2), 256 features
    "mos_p16x5_8x4_4x2": ("nisqa_mos_only.tar", None, {}, (16, 32, 64), ([16, 5], [8, 4], [4, 2])),
    # only conv4's pooling and conv6 (3, 1) change: the shipped conv2 / conv3 instances run
    "mos_p24x7_12x5_6x1": ("nisqa_mos_only.tar", None, {}, (16, 32, 64), ([24, 7], [12, 5], [6, 1])),
    # NISQA_DIM's five heads, pool_3 3 wide at 12 rows: 768 features
    "dim_p24x7_12x5_12x3": ("nisqa.tar", None, {}, (16, 32, 64), ([24, 7], [12, 5], [12, 3])),
    # pool_2 wider than its 7-column input: upsampling windows
    "mos_p24x7_12x9_6x3": ("nisqa_mos_only.tar", None, {}, (16, 32, 64), ([24, 7], [12, 9], [6, 3])),
    # 32 bands x 11 frames
    "mos_m32_s11_p16x7_8x5_4x3": ("nisqa_mos_only.tar", None, dict(ms_n_mels=32, ms_seg_length=11), (16, 32, 64),
                                  ([16, 7], [8, 5], [4, 3])),
    # 128 bands: the largest conv2 tile under the bound, and a 15 -> 5 row reduction
    "mos_m128_p30x7_15x5_5x3": ("nisqa_mos_only.tar", None, dict(ms_n_mels=128), (16, 32, 64), ([30, 7], [15, 5], [5, 3])),
    # other channel counts: 96 features, padded to 128
    "mos_c16_32_32_p12x7_6x5_3x3": ("nisqa_mos_only.tar", None, {}, (16, 32, 32), ([12, 7], [6, 5], [3, 3])),
    # AdaptCNN's Linear (cnn_fc_out_h 128) over 512 features
    "dim_fc128_p20x6_10x4_8x2": ("nisqa.tar", "dim_adapt_fc", {}, (16, 32, 64), ([20, 6], [10, 4], [8, 2])),
    # td = 'skip': PoolAvg over the 192 framewise features
    "mos_skip_avg_p24x7_12x5_3x3": ("nisqa_mos_only.tar", None, dict(td="skip", td_2="skip", **_pool("avg")), (16, 32, 64),
                                    ([24, 7], [12, 5], [3, 3])),
    # NISQA_DE: the same CNN on both signals
    "de_p16x7_8x4_4x3": ("nisqa_mos_only.tar", "de:de_cosine_hard", {}, (16, 32, 64), ([16, 7], [8, 4], [4, 3])),
}
# the single-ended variants are scored on TD_PAIR_CLIPS, the NISQA_DE one on DE_PAIRS
POOL_CLIPS = TD_PAIR_CLIPS
POOL_DE_PAIRS = DE_PAIRS


def _t(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float32))


def pool_checkpoint(args, sd, widths, pools, rng):
    """(args, state_dict) of an AdaptCNN checkpoint re-seeded at widths (c1, c2, c3) and pools (pool_1, pool_2, pool_3):
    the CNN (conv6 as (c3, c3, 3, pool_3[1])) and the Linear that reads its c3 * pool_3[0] features."""
    args = dict(args, cnn_c_out_1=widths[0], cnn_c_out_2=widths[1], cnn_c_out_3=widths[2],
                cnn_pool_1=list(pools[0]), cnn_pool_2=list(pools[1]), cnn_pool_3=list(pools[2]))
    sd = dict(sd)
    seed_cnn(sd, widths, rng)
    c3, (h3, w3) = widths[2], pools[2]
    sd["cnn.model.conv6.weight"] = _t(rng.standard_normal((c3, c3, 3, w3)) * math.sqrt(2.0 / (3 * w3 * c3)))
    n_in = c3 * h3
    if args.get("cnn_fc_out_h"):
        h = int(args["cnn_fc_out_h"])
        sd["cnn.model.fc.weight"] = _t(rng.standard_normal((h, n_in)) / math.sqrt(n_in))
        sd["cnn.model.fc.bias"] = _t(rng.normal(0, 0.05, h))
    elif args.get("td") == "skip":
        # no time-dependency model: the pooling module reads the c3 * pool_3[0] features, its score Linear scaled
        sd = {k: v for k, v in sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers."))}
        heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
        for pf in heads:
            sd[pf + "linear.weight"] = _t(rng.standard_normal((1, n_in)) * 0.1 * math.sqrt(64.0 / n_in))
            sd[pf + "linear.bias"] = _t(rng.uniform(1.0, 4.0, 1))
    else:
        sd["time_dependency.model.linear.weight"] = _t(rng.standard_normal((64, n_in)) / math.sqrt(n_in))
    return args, sd


def cnn_pool_checkpoint(name, base_args, base_sd):
    """-> (args, state_dict) of a CNN_POOL_VARIANTS entry; base_args / base_sd are those of its base checkpoint."""
    _, parent, over, widths, pools = CNN_POOL_VARIANTS[name]
    if parent is None:
        args, sd = dict(base_args), dict(base_sd)
    elif parent.startswith("de:"):
        args, sd = de_checkpoint(parent[3:], base_args, base_sd)
    else:
        args, sd = variant_checkpoint(parent, base_args, base_sd)
    args = dict(args)
    args.update(over)
    return pool_checkpoint(args, sd, widths, pools, np.random.default_rng(sum(map(ord, name)) + 29))
