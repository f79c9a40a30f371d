"""Checkpoints whose td and td_2 pair the time-dependency models in the orders the reference builds beyond the shipped
ones (TimeDependency, lib:839-895, used for both stages by NISQA / NISQA_DIM, lib:84-141, 200-268): StandardCNN in front of
self-attention, an LSTM as td_2 behind self-attention or an LSTM, and self-attention as td_2 behind an LSTM.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A pair variant = a shipped checkpoint's args (or those of an
oracle/variants.py VARIANTS entry) with td / td_2 / pooling switched + its framewise weights (StandardCNN: a seeded fc_out
unless it keeps the shipped 20-wide one) + seeded weights for td, td_2 and the pooling heads (NumPy PCG64: the same here,
in oracle/make_td_pair_golden.py that feeds them to the UNMODIFIED reference modules, and on the GPU box).
"""
import math

import numpy as np
import torch

from oracle.variants import CLIPS, variant_checkpoint
from oracle.wide_variants import sa_stack_weights


def sa(stage, d, h, layers=1, pos_enc=False):
    """args of a one-head self-attention stage ('td' / 'td_2')"""
    return {stage: "self_att", stage + "_sa_d_model": d, stage + "_sa_nhead": 1, stage + "_sa_h": h,
            stage + "_sa_num_layers": layers, stage + "_sa_pos_enc": pos_enc, stage + "_sa_dropout": 0.1}


def lstm(stage, h, layers=1, bi=True):
    """args of an LSTM stage ('td' / 'td_2')"""
    return {stage: "lstm", stage + "_lstm_h": h, stage + "_lstm_num_layers": layers, stage + "_lstm_bidirectional": bi,
            stage + "_lstm_dropout": 0}


def _pool(pool, att_h=None):
    return {"pool": pool, "pool_att_h": att_h, "pool_att_dropout": 0.1 if pool == "att" else None}


# name -> (base checkpoint, oracle/variants.py VARIANTS entry whose framewise weights are reused or None, args overrides)
TD_PAIR_VARIANTS = {
    "mos_std_sa64_attff": ("nisqa_tts.tar", None, dict(cnn_fc_out_h=None, **sa("td", 64, 64), td_2="skip", **_pool("att", 128))),
    "dim_std_fc100_sa128_l2_attff": ("nisqa_tts.tar", None, dict(model="NISQA_DIM", cnn_fc_out_h=100, **sa("td", 128, 256, 2),
                                                                 td_2="skip", **_pool("att", 128))),
    # (the positional encoding buffer holds 3000 steps, lib:1042-1062: ms_max_segments must not exceed it)
    "mos_std_fc20_sa64pos_sa128_avg": ("nisqa_tts.tar", None, dict(ms_max_segments=1300, **sa("td", 64, 64, 1, True),
                                                                   **sa("td_2", 128, 128), **_pool("avg"))),
    "mos_adapt_sa64_lstm128bi_lastbi": ("nisqa_mos_only.tar", None, dict(**lstm("td_2", 128), **_pool("last_step_bi"))),
    "dim_adapt_sa64_lstm32bi_attff": ("nisqa.tar", None, dict(**lstm("td_2", 32), **_pool("att", 128))),
    "mos_dff_sa128_lstm96uni_l2_max": ("nisqa_mos_only.tar", "mos_dff", dict(**sa("td", 128, 128), **lstm("td_2", 96, 2, False),
                                                                             **_pool("max"))),
    "mos_tts_sa64_attff": ("nisqa_tts.tar", None, dict(**sa("td_2", 64, 64), **_pool("att", 128))),
    "dim_std_lstm64bi_sa128_avg": ("nisqa_tts.tar", None, dict(model="NISQA_DIM", td_lstm_h=64, **sa("td_2", 128, 256),
                                                               **_pool("avg"))),
    "mos_std_lstm192bi_lstm64uni_last": ("nisqa_tts.tar", None, dict(td_lstm_h=192, **lstm("td_2", 64, 1, False),
                                                                     **_pool("last_step"))),
    "mos_std_lstm32uni_l2_lstm256bi_lastbi": ("nisqa_tts.tar", None, dict(td_lstm_h=32, td_lstm_num_layers=2,
                                                                          td_lstm_bidirectional=False, **lstm("td_2", 256),
                                                                          **_pool("last_step_bi"))),
    "mos_std_sa256_ff1024_lstm128bi_att": ("nisqa_tts.tar", None, dict(**sa("td", 256, 1024), **lstm("td_2", 128),
                                                                       **_pool("att", None))),
}
# the pair variants are scored on CLIPS plus a 12 s clip (297 segments)
TD_PAIR_CLIPS = CLIPS + [(74, 12.0, 48000)]


def framewise_fan_out(args):
    """width of the framewise model's output rows (Framewise.fan_out, lib:428-836)"""
    if args["cnn_model"] == "adapt":
        return args.get("cnn_fc_out_h") or 64 * args["cnn_pool_3"][0]
    if args["cnn_model"] == "standard":
        return args.get("cnn_fc_out_h") or 768
    if args["cnn_model"] == "dff":
        return args.get("cnn_fc_out_h") or 4096
    return args.get("cnn_fc_out_h") or 720


def fan_out(args, stage, in_dim):
    """TimeDependency.fan_out of stage 'td' / 'td_2' fed in_dim-wide rows (lib:867-885)"""
    if args.get(stage) == "self_att":
        return args[stage + "_sa_d_model"]
    if args.get(stage) == "lstm":
        return (2 if args[stage + "_lstm_bidirectional"] else 1) * args[stage + "_lstm_h"]
    return in_dim


def lstm_weights(sd, prefix, args, key, in_dim, rng):
    """Seeded weights of an nn.LSTM (args key prefix 'td_lstm' / 'td_2_lstm') under prefix, in nn.LSTM's own range"""
    H, dirs = args[key + "_h"], 2 if args[key + "_bidirectional"] else 1
    k = 1.0 / math.sqrt(H)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))      # noqa: E731
    for l in range(args[key + "_num_layers"]):
        n_in = in_dim if l == 0 else dirs * H
        for d in range(dirs):
            sfx = "_l%d%s" % (l, "_reverse" if d else "")
            sd[prefix + "weight_ih" + sfx] = t(rng.uniform(-k, k, (4 * H, n_in)))
            sd[prefix + "weight_hh" + sfx] = t(rng.uniform(-k, k, (4 * H, H)))
            sd[prefix + "bias_ih" + sfx] = t(rng.uniform(-k, k, 4 * H))
            sd[prefix + "bias_hh" + sfx] = t(rng.uniform(-k, k, 4 * H))


def td_pair_checkpoint(name, base_args, base_sd, spec=None):
    """-> (args, state_dict) of a TD_PAIR_VARIANTS entry (or of `spec`, an entry of the same form, seeded by `name`);
    base_args / base_sd are those of its base checkpoint."""
    _, parent, over = spec or TD_PAIR_VARIANTS[name]
    args, sd = variant_checkpoint(parent, base_args, base_sd) if parent else (dict(base_args), dict(base_sd))
    args = dict(args)
    args.update(over)
    sd = {k: v for k, v in sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers."))}
    rng = np.random.default_rng(sum(map(ord, name)) + 7)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))      # noqa: E731
    if args["cnn_model"] == "standard" and args.get("cnn_fc_out_h") != 20:
        sd = {k: v for k, v in sd.items() if not k.startswith("cnn.model.fc_out.")}
        fc = args.get("cnn_fc_out_h")
        if fc:
            sd["cnn.model.fc_out.weight"] = t(rng.standard_normal((fc, 768)) / math.sqrt(768))
            sd["cnn.model.fc_out.bias"] = t(rng.normal(0, 0.05, fc))
    d = framewise_fan_out(args)
    fans = []
    for stage, prefix in (("td", "time_dependency.model."), ("td_2", "time_dependency_2.model.")):
        if args.get(stage) == "self_att":
            sa_stack_weights(sd, prefix, args, stage + "_sa", d, rng)
        elif args.get(stage) == "lstm":
            lstm_weights(sd, prefix + "lstm.", args, stage + "_lstm", d, rng)
        d = fan_out(args, stage, d)
        fans.append(d)
    heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    d = fans[0] if args["model"] == "NISQA_DIM" else fans[1]        # lib:130-135 / 247-253
    for pf in heads:
        def lin(key, n_out, n_in, scale, bias):
            sd[pf + key + ".weight"] = t(rng.standard_normal((n_out, n_in)) * scale)
            sd[pf + key + ".bias"] = t(bias(n_out))
        score_bias = lambda n: rng.uniform(1.0, 4.0, n)      # noqa: E731  (scores in the MOS range)
        small_bias = lambda n: rng.normal(0, 0.05, n)        # noqa: E731
        if args["pool"] == "att" and args.get("pool_att_h"):
            lin("linear1", 128, d, 1.0 / math.sqrt(d), small_bias)
            lin("linear2", 1, 128, 1.0 / math.sqrt(128), small_bias)
            lin("linear3", 1, d, 0.3, score_bias)
        elif args["pool"] == "att":
            lin("linear1", 1, d, 1.0 / math.sqrt(d), small_bias)
            lin("linear2", 1, d, 0.3, score_bias)
        else:
            lin("linear", 1, d, 0.3, score_bias)
    return args, sd
