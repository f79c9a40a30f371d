"""Double-ended (NISQA_DE, reference lib:272-424) checkpoints with the other framewise and time-dependency models the
reference builds for it: StandardCNN, SkipCNN or DFF in front of self-attention, and StandardCNN in front of an LSTM td
of any accepted shape.  The alignment and fusion then run at the LSTM's fan_out W = dirs * td_lstm_h (32 .. 512)
instead of 64 (q_dim = y_dim = time_dependency.fan_out, lib:404-410).

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A variant = a shipped checkpoint's args (or those of an
oracle/variants.py VARIANTS entry, for SkipCNN / DFF weights) switched to NISQA_DE + its framewise weights (StandardCNN:
a seeded fc_out unless it keeps the shipped 20-wide one) + seeded weights for td, the alignment, lin_fusion, td_2 and the
pooling head (NumPy PCG64: the same here, in oracle/make_de_arch_golden.py that feeds them to the UNMODIFIED reference
NISQA_DE, and on the GPU box).
"""
import math

import numpy as np
import torch

from oracle.td_pair_variants import fan_out, framewise_fan_out, lstm, lstm_weights, sa
from oracle.variants import DE_PAIRS, variant_checkpoint
from oracle.wide_variants import sa_stack_weights


def _de(align, apply, fuse, fuse_dim=None):
    return {"de_align": align, "de_align_apply": apply, "de_fuse": fuse, "de_fuse_dim": fuse_dim}


def _pool(pool, att_h=None):
    return {"pool": pool, "pool_att_h": att_h, "pool_att_dropout": 0.1 if pool == "att" else None}


# name -> (base checkpoint, oracle/variants.py VARIANTS entry whose framewise weights are reused or None, args overrides).
# Together: every framewise model in front of self-attention; LSTM fan_outs W = 32, 96, 128, 256, 384 and 512 with
# cnn_fc_out_h None, 20 and 100; every alignment method at a W != 64; hard and soft; every fusion mode; de_fuse_dim;
# five pooling modules.
DE_ARCH_VARIANTS = {
    "std_fc20_sa64_cosine_soft": ("nisqa_tts.tar", None, dict(**sa("td", 64, 64), **_de("cosine", "soft", "x/y/-"),
                                                              **_pool("att", 128))),
    "std_fcnone_sa64_luong_hard": ("nisqa_tts.tar", None, dict(cnn_fc_out_h=None, **sa("td", 64, 64, 2),
                                                               **_de("luong", "hard", "+/-"), **_pool("avg"))),
    "skip_fc128_sa64_bahd_soft": ("nisqa.tar", "dim_skip_fc", dict(**sa("td", 64, 128), **_de("bahd", "soft", "x/y"),
                                                                   **_pool("max"))),
    "dff_sa64_dot_hard": ("nisqa_mos_only.tar", "mos_dff", dict(**sa("td", 64, 64), **_de("dot", "hard", "x/y/-"),
                                                                **_pool("att", None))),
    "std_fc20_lstm32uni_dot_soft": ("nisqa_tts.tar", None, dict(**lstm("td", 32, 1, False), **_de("dot", "soft", "x/y/-"),
                                                                **_pool("att", 128))),
    "std_fcnone_lstm96uni_distance_soft": ("nisqa_tts.tar", None, dict(cnn_fc_out_h=None, **lstm("td", 96, 1, False),
                                                                       **_de("distance", "soft", "+/-"), **_pool("avg"))),
    "std_fc100_lstm64bi_cosine_hard": ("nisqa_tts.tar", None, dict(cnn_fc_out_h=100, **lstm("td", 64),
                                                                   **_de("cosine", "hard", "x/y"), **_pool("last_step"))),
    "std_fc20_lstm128bi_luong_soft_fd128": ("nisqa_tts.tar", None, dict(**lstm("td", 128), **_de("luong", "soft", "x/y/-", 128),
                                                                        **_pool("att", 128))),
    "std_fcnone_lstm192bi_l3_bahd_soft": ("nisqa_tts.tar", None, dict(cnn_fc_out_h=None, **lstm("td", 192, 3),
                                                                      **_de("bahd", "soft", "+/-"), **_pool("max"))),
    "std_fc100_lstm256bi_l2_distance_hard_fd64": ("nisqa_tts.tar", None, dict(cnn_fc_out_h=100, **lstm("td", 256, 2),
                                                                              **_de("distance", "hard", "x/y/-", 64),
                                                                              **_pool("att", None))),
    "std_fc20_lstm256bi_l2_dot_soft": ("nisqa_tts.tar", None, dict(**lstm("td", 256, 2), **_de("dot", "soft", "x/y"),
                                                                   **_pool("att", 128))),
}
# (degraded, reference) pairs the variants are scored on: oracle/variants.py DE_PAIRS plus a 2.5 s degraded clip against
# an unrelated 8 s reference (797 segments at 48 kHz: 13 key blocks of 64)
DE_ARCH_PAIRS = DE_PAIRS + [((85, 2.5, 48000), (86, 8.0, 48000))]


def de_arch_checkpoint(name, base_args, base_sd, spec=None):
    """-> (args, state_dict) of a DE_ARCH_VARIANTS entry (or of `spec`, an entry of the same form, seeded by `name`);
    base_args / base_sd are those of its base checkpoint."""
    _, parent, over = spec or DE_ARCH_VARIANTS[name]
    args, sd = variant_checkpoint(parent, base_args, base_sd) if parent else (dict(base_args), dict(base_sd))
    args = dict(args)
    args.update({"model": "NISQA_DE", "td_lstm_dropout": 0, **sa("td_2", 64, 64, 2), "td_2_lstm_h": None,
                 "td_2_lstm_num_layers": None, "td_2_lstm_dropout": None, "td_2_lstm_bidirectional": None})
    args.update(over)
    sd = {k: v for k, v in sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers.", "align.", "fuse."))}
    rng = np.random.default_rng(sum(map(ord, name)) + 11)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))      # noqa: E731
    if args["cnn_model"] == "standard" and args.get("cnn_fc_out_h") != 20:
        sd = {k: v for k, v in sd.items() if not k.startswith("cnn.model.fc_out.")}
        fc = args.get("cnn_fc_out_h")
        if fc:
            sd["cnn.model.fc_out.weight"] = t(rng.standard_normal((fc, 768)) / math.sqrt(768))
            sd["cnn.model.fc_out.bias"] = t(rng.normal(0, 0.05, fc))
    d = framewise_fan_out(args)
    if args["td"] == "self_att":
        sa_stack_weights(sd, "time_dependency.model.", args, "td_sa", d, rng)
    else:
        lstm_weights(sd, "time_dependency.model.lstm.", args, "td_lstm", d, rng)
    W = fan_out(args, "td", d)
    put = lambda key, shape, scale: sd.__setitem__(key, t(rng.standard_normal(shape) * scale))      # noqa: E731
    if args["de_align"] == "luong":             # AttLuong: W = Linear(y_dim -> q_dim) (lib:1348-1351)
        put("align.att.W.weight", (W, W), 1.0 / math.sqrt(W)); put("align.att.W.bias", (W,), 0.05)
    if args["de_align"] == "bahd":              # AttBahdanau, att_dim 128 (lib:1329-1337)
        put("align.att.Wq.weight", (128, W), 1.0 / math.sqrt(W)); put("align.att.Wq.bias", (128,), 0.05)
        put("align.att.Wy.weight", (128, W), 1.0 / math.sqrt(W)); put("align.att.Wy.bias", (128,), 0.05)
        put("align.att.v.weight", (1, 128), 0.3); put("align.att.v.bias", (1,), 0.05)
    fdim = (3 if args["de_fuse"] == "x/y/-" else 2) * W
    if args.get("de_fuse_dim"):                 # Fusion.lin_fusion (lib:1399-1401)
        put("fuse.lin_fusion.weight", (args["de_fuse_dim"], fdim), 1.0 / math.sqrt(fdim))
        put("fuse.lin_fusion.bias", (args["de_fuse_dim"],), 0.05)
        fdim = args["de_fuse_dim"]
    sa_stack_weights(sd, "time_dependency_2.model.", args, "td_2_sa", fdim, rng)
    pf = "pool.model."
    D = args["td_2_sa_d_model"]
    lin = lambda key, n_out, n_in, scale: put(pf + key + ".weight", (n_out, n_in), scale)           # noqa: E731
    if args["pool"] == "att" and args.get("pool_att_h"):
        lin("linear1", 128, D, 1.0 / math.sqrt(D)); put(pf + "linear1.bias", (128,), 0.05)
        lin("linear2", 1, 128, 1.0 / math.sqrt(128)); put(pf + "linear2.bias", (1,), 0.05)
        lin("linear3", 1, D, 0.3); sd[pf + "linear3.bias"] = t(rng.uniform(1.0, 4.0, 1))
    elif args["pool"] == "att":
        lin("linear1", 1, D, 1.0 / math.sqrt(D)); put(pf + "linear1.bias", (1,), 0.05)
        lin("linear2", 1, D, 0.3); sd[pf + "linear2.bias"] = t(rng.uniform(1.0, 4.0, 1))
    else:
        lin("linear", 1, D, 0.3); sd[pf + "linear.bias"] = t(rng.uniform(1.0, 4.0, 1))
    return args, sd
