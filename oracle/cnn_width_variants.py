"""AdaptCNN checkpoints trained with other channel counts (cnn_c_out_1 / cnn_c_out_2 / cnn_c_out_3 in {16, 32, 64}, lib:653-710),
behind self-attention, no td, or NISQA_DE's stack, at the shipped and at another Mel-spectrogram shape.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A width variant is an existing checkpoint (a shipped one, an
oracle/variants.py VARIANTS / DE_VARIANTS entry) with cnn_c_out_1/2/3 switched: all six conv / BN layers are seeded at the
new widths, and so is the Linear that reads the CNN's 6 c3 features (AdaptCNN's cnn.model.fc, td's input Linear, or the
pooling module's Linear behind td = 'skip'), NumPy PCG64: the same here, in oracle/make_cnn_width_golden.py that feeds
these checkpoints to the UNMODIFIED reference modules, and on the GPU box.

``adapt_cnn`` is oracle/nisqa_oracle.py's AdaptCNN with the reference's reshape to c3 * pool_3[0] features (lib:706)
taken from the tensor instead of 64; ``wide_cnn()`` puts it in place of that module's for the oracle's predict functions.
"""
import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import nisqa_oracle as O
from oracle.td_pair_variants import TD_PAIR_CLIPS, _pool
from oracle.variants import DE_PAIRS, de_checkpoint, variant_checkpoint

CHANNELS = (16, 32, 64)
TRIPLES = [(a, b, c) for a in CHANNELS for b in CHANNELS for c in CHANNELS]

# name -> (base checkpoint, oracle/variants.py VARIANTS entry (or "de:" + a DE_VARIANTS entry) or None, args overrides,
#          (cnn_c_out_1, cnn_c_out_2, cnn_c_out_3))
CNN_WIDTH_VARIANTS = {
    # the narrowest: 96 features, padded to 128 in the engine
    "mos_c16_16_16": ("nisqa_mos_only.tar", None, {}, (16, 16, 16)),
    # conv2 64 -> 32 (one activation buffer beside the staging tile), 96 features
    "mos_c64_32_16": ("nisqa_mos_only.tar", None, {}, (64, 32, 16)),
    # conv3 64 -> 32
    "mos_c16_64_32": ("nisqa_mos_only.tar", None, {}, (16, 64, 32)),
    # the widest, NISQA_DIM's five heads
    "dim_c64_64_64": ("nisqa.tar", None, {}, (64, 64, 64)),
    # AdaptCNN's Linear (cnn_fc_out_h 128) over 192 features
    "dim_c32_32_32_fc128": ("nisqa.tar", "dim_adapt_fc", {}, (32, 32, 32)),
    # conv2 16 -> 64 at 48 x 15 (the separate conv1 kernel)
    "mos_c16_64_64": ("nisqa_mos_only.tar", None, {}, (16, 64, 64)),
    # conv1 + conv2 16 -> 16 in the fused kernel at 48 x 15
    "mos_c16_16_64": ("nisqa_mos_only.tar", None, {}, (16, 16, 64)),
    # another Mel-spectrogram shape (64 bands x 21 frames)
    "mos_c32_16_64_m64_s21": ("nisqa_mos_only.tar", None, dict(ms_n_mels=64, ms_seg_length=21), (32, 16, 64)),
    # td = 'skip': PoolAvg over the 96 framewise features
    "mos_c32_64_16_skip_avg": ("nisqa_mos_only.tar", None, dict(td="skip", td_2="skip", **_pool("avg")), (32, 64, 16)),
    # NISQA_DE: the same CNN on both signals
    "de_c16_32_32": ("nisqa_mos_only.tar", "de:de_cosine_hard", {}, (16, 32, 32)),
}
# the single-ended variants are scored on TD_PAIR_CLIPS, the NISQA_DE one on DE_PAIRS
WIDTH_CLIPS = TD_PAIR_CLIPS
WIDTH_DE_PAIRS = DE_PAIRS


def _t(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float32))


def seed_cnn(sd, widths, rng):
    """conv1..conv6 + bn1..bn6 of an AdaptCNN with output channels c1, c2, c3, c3, c3, c3 written into sd (He-scaled
    weights; conv1 scaled down to the mel dB range; BatchNorm statistics near unit scale)."""
    c1, c2, c3 = widths
    cins, couts = (1, c1, c2, c3, c3, c3), (c1, c2, c3, c3, c3, c3)
    for i in range(1, 7):
        ci, co = cins[i - 1], couts[i - 1]
        scale = math.sqrt(2.0 / (9 * ci)) / (30.0 if i == 1 else 1.0)
        sd["cnn.model.conv%d.weight" % i] = _t(rng.standard_normal((co, ci, 3, 3)) * scale)
        sd["cnn.model.conv%d.bias" % i] = _t(rng.normal(0, 0.05, co))
        b = "cnn.model.bn%d." % i
        sd[b + "weight"] = _t(rng.uniform(0.8, 1.2, co))
        sd[b + "bias"] = _t(rng.normal(0, 0.1, co))
        sd[b + "running_mean"] = _t(rng.normal(0, 0.2, co))
        sd[b + "running_var"] = _t(rng.uniform(0.5, 1.5, co))
        sd[b + "num_batches_tracked"] = torch.tensor(1)


def width_checkpoint(args, sd, widths, rng):
    """(args, state_dict) of an AdaptCNN checkpoint re-seeded at widths (c1, c2, c3): the CNN and the Linear that reads its
    6 c3 features."""
    args = dict(args, cnn_c_out_1=widths[0], cnn_c_out_2=widths[1], cnn_c_out_3=widths[2])
    sd = dict(sd)
    seed_cnn(sd, widths, rng)
    n_in = 6 * widths[2]
    if args.get("cnn_fc_out_h"):
        h = int(args["cnn_fc_out_h"])
        sd["cnn.model.fc.weight"] = _t(rng.standard_normal((h, n_in)) / math.sqrt(n_in))
        sd["cnn.model.fc.bias"] = _t(rng.normal(0, 0.05, h))
    elif args.get("td") == "skip":
        # no time-dependency model: the pooling module reads the 6 c3 features, its score Linear scaled
        sd = {k: v for k, v in sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers."))}
        heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
        for pf in heads:
            sd[pf + "linear.weight"] = _t(rng.standard_normal((1, n_in)) * 0.1 * math.sqrt(64.0 / n_in))
            sd[pf + "linear.bias"] = _t(rng.uniform(1.0, 4.0, 1))
    else:
        sd["time_dependency.model.linear.weight"] = _t(rng.standard_normal((64, n_in)) / math.sqrt(n_in))
    return args, sd


def cnn_width_checkpoint(name, base_args, base_sd):
    """-> (args, state_dict) of a CNN_WIDTH_VARIANTS entry; base_args / base_sd are those of its base checkpoint."""
    _, parent, over, widths = CNN_WIDTH_VARIANTS[name]
    if parent is None:
        args, sd = dict(base_args), dict(base_sd)
    elif parent.startswith("de:"):
        args, sd = de_checkpoint(parent[3:], base_args, base_sd)
    else:
        args, sd = variant_checkpoint(parent, base_args, base_sd)
    args = dict(args)
    args.update(over)
    return width_checkpoint(args, sd, widths, np.random.default_rng(sum(map(ord, name)) + 17))


def triple_checkpoint(base_args, base_sd, widths):
    """(args, state_dict) of nisqa_mos_only.tar re-seeded at any widths (c1, c2, c3)"""
    return width_checkpoint(base_args, base_sd, widths, np.random.default_rng(1000 + 100 * widths[0] + 10 * widths[1] + widths[2]))


# ------------------------------------------------------------------------------------------------------------ oracle
def adapt_cnn(sd, x, args, taps=None):
    """lib:688-710 at any channel counts (eval mode): nisqa_oracle.adapt_cnn with the c3 * pool_3[0] features of
    lib:706 read from conv6's output."""
    x = O._conv_bn_relu(sd, 1, x, (1, 1))
    x = F.adaptive_max_pool2d(x, output_size=tuple(args["cnn_pool_1"]))
    if taps is not None: taps["pool1"] = x
    x = O._conv_bn_relu(sd, 2, x, (1, 1))
    x = F.adaptive_max_pool2d(x, output_size=tuple(args["cnn_pool_2"]))
    if taps is not None: taps["pool2"] = x
    x = O._conv_bn_relu(sd, 3, x, (1, 1))
    if taps is not None: taps["conv3"] = x
    x = O._conv_bn_relu(sd, 4, x, (1, 1))
    x = F.adaptive_max_pool2d(x, output_size=tuple(args["cnn_pool_3"]))
    if taps is not None: taps["pool3"] = x
    x = O._conv_bn_relu(sd, 5, x, (1, 1))
    if taps is not None: taps["conv5"] = x
    x = O._conv_bn_relu(sd, 6, x, (1, 0))
    x = x.reshape(-1, x.shape[1] * args["cnn_pool_3"][0])
    if "cnn.model.fc.weight" in sd:
        x = F.linear(x, sd["cnn.model.fc.weight"], sd["cnn.model.fc.bias"])
    return x


@contextlib.contextmanager
def wide_cnn():
    """the oracle's predict functions (nisqa_oracle, td_pair_oracle) run ``adapt_cnn`` above while inside"""
    saved = O.adapt_cnn
    O.adapt_cnn = adapt_cnn
    try:
        yield
    finally:
        O.adapt_cnn = saved
