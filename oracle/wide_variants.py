"""Self-attention stacks wider than 64 reachable through user-trained checkpoints: td_sa_d_model / td_2_sa_d_model in
{64, 128, 192, 256} with any feed-forward width td_sa_h / td_2_sa_h (one head).

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A wide variant = a shipped checkpoint's args (or those of an
oracle/variants.py VARIANTS entry) with the widths switched + seeded weights for every self-attention stack and the
pooling head (NumPy PCG64: the same here, in oracle/make_wide_golden.py that feeds them to the UNMODIFIED reference
modules, and on the GPU box).
"""
import math

import numpy as np
import torch

from oracle.variants import CLIPS, positional_encoding, variant_checkpoint

# name -> (base checkpoint, oracle/variants.py VARIANTS entry whose framewise weights are reused or None, args overrides).
# The CNN (or the framewise model of the VARIANTS entry) comes from the base; every self-attention stack and the pooling
# head get seeded weights.
WIDE_VARIANTS = {
    "dim_sa_d128_ff256": ("nisqa.tar", None, {"td_sa_d_model": 128, "td_sa_h": 256}),
    "mos_sa_d256_ff1024_pos": ("nisqa_mos_only.tar", None, {"td_sa_d_model": 256, "td_sa_h": 1024, "td_sa_num_layers": 3,
                                                            "td_sa_pos_enc": True, "pool": "att", "pool_att_h": None}),
    "dim_sa_d192_max": ("nisqa.tar", None, {"td_sa_d_model": 192, "td_sa_h": 384, "pool": "max", "pool_att_h": None}),
    "mos_sa_d64_ff2048_avg": ("nisqa_mos_only.tar", None, {"td_sa_h": 2048, "pool": "avg", "pool_att_h": None}),
    # (NISQA only: NISQA_DIM sizes its pooling heads by the first stack, lib:247-253, so its td_2 keeps that width)
    "mos_td2_d128_to_d64": ("nisqa_mos_only.tar", None, {"td_sa_d_model": 128, "td_sa_h": 128, "td_2": "self_att", "td_2_sa_d_model": 64,
                                                         "td_2_sa_nhead": 1, "td_2_sa_h": 256, "td_2_sa_num_layers": 1,
                                                         "td_2_sa_pos_enc": None, "td_2_sa_dropout": 0.1}),
    "dim_adapt_fc128_d256_last": ("nisqa.tar", "dim_adapt_fc", {"td_sa_d_model": 256, "td_sa_h": 512, "pool": "last_step",
                                                                "pool_att_h": None}),
    "mos_dff_d128": ("nisqa_mos_only.tar", "mos_dff", {"td_sa_d_model": 128, "td_sa_h": 128}),
}
# the wide variants are scored on CLIPS plus a 12 s clip (297 segments: several key blocks of 64)
WIDE_CLIPS = CLIPS + [(74, 12.0, 48000)]


def sa_stack_weights(sd, prefix, args, key, in_dim, rng):
    """Seeded weights of one self-attention stack (args key prefix 'td_sa' or 'td_2_sa') written into sd under prefix:
    Linears scaled by 1/sqrt(fan_in), LayerNorm gamma about 1."""
    d, h = args[key + "_d_model"], args[key + "_h"]

    def put(k, shape, scale, offset=0.0):
        sd[prefix + k] = torch.from_numpy((rng.standard_normal(shape) * scale + offset).astype(np.float32))

    put("linear.weight", (d, in_dim), 1.0 / math.sqrt(in_dim)); put("linear.bias", (d,), 0.05)
    put("norm1.weight", (d,), 0.05, 1.0); put("norm1.bias", (d,), 0.05)
    for l in range(args[key + "_num_layers"]):
        q = "layers.%d." % l
        put(q + "self_attn.in_proj_weight", (3 * d, d), 1.0 / math.sqrt(d)); put(q + "self_attn.in_proj_bias", (3 * d,), 0.05)
        put(q + "self_attn.out_proj.weight", (d, d), 1.0 / math.sqrt(d)); put(q + "self_attn.out_proj.bias", (d,), 0.05)
        put(q + "linear1.weight", (h, d), 1.0 / math.sqrt(d)); put(q + "linear1.bias", (h,), 0.05)
        put(q + "linear2.weight", (d, h), 1.0 / math.sqrt(h)); put(q + "linear2.bias", (d,), 0.05)
        put(q + "norm1.weight", (d,), 0.05, 1.0); put(q + "norm1.bias", (d,), 0.05)
        put(q + "norm2.weight", (d,), 0.05, 1.0); put(q + "norm2.bias", (d,), 0.05)
    if args.get(key + "_pos_enc"):
        sd[prefix + "pos_encoder.pe"] = positional_encoding(d_model=d)


def wide_checkpoint(name, base_args, base_sd, spec=None):
    """-> (args, state_dict) of a WIDE_VARIANTS entry (or of `spec`, an entry of the same form, seeded by `name`);
    base_args / base_sd are those of its base checkpoint."""
    _, parent, over = spec or WIDE_VARIANTS[name]
    args, sd = variant_checkpoint(parent, base_args, base_sd) if parent else (dict(base_args), dict(base_sd))
    args = dict(args)
    args.update(over)
    sd = {k: v for k, v in sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers."))}
    rng = np.random.default_rng(sum(map(ord, name)) + 3)
    if args["cnn_model"] == "adapt":
        in_dim = args.get("cnn_fc_out_h") or 64 * args["cnn_pool_3"][0]
    else:
        in_dim = args.get("cnn_fc_out_h") or 720
    sa_stack_weights(sd, "time_dependency.model.", args, "td_sa", in_dim, rng)
    d = args["td_sa_d_model"]
    if args.get("td_2") == "self_att":
        sa_stack_weights(sd, "time_dependency_2.model.", args, "td_2_sa", d, rng)
        d = args["td_2_sa_d_model"]
    heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    for pf in heads:
        def lin(key, n_out, n_in, scale, bias):
            sd[pf + key + ".weight"] = torch.from_numpy((rng.standard_normal((n_out, n_in)) * scale).astype(np.float32))
            sd[pf + key + ".bias"] = torch.from_numpy(bias(n_out).astype(np.float32))
        score_bias = lambda n: rng.uniform(1.0, 4.0, n)      # noqa: E731  (scores in the MOS range)
        small_bias = lambda n: rng.normal(0, 0.05, n)        # noqa: E731
        if args["pool"] == "att" and args.get("pool_att_h"):
            lin("linear1", 128, d, 1.0 / math.sqrt(d), small_bias)
            lin("linear2", 1, 128, 1.0 / math.sqrt(128), small_bias)
            lin("linear3", 1, d, 0.15, score_bias)
        elif args["pool"] == "att":
            lin("linear1", 1, d, 1.0 / math.sqrt(d), small_bias)
            lin("linear2", 1, d, 0.15, score_bias)
        else:
            lin("linear", 1, d, 0.15, score_bias)
    return args, sd
