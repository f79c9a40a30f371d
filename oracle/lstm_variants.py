"""StandardCNN + LSTM checkpoints of other shapes reachable through user-trained checkpoints (reference
config/train_nisqa_cnn_lstm_avg.yaml): td_lstm_h in {32, 64, 96, 128, 192, 256}, 1 to 4 layers, either direction,
cnn_fc_out_h of any width or None, every pooling module, NISQA and NISQA_DIM.

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  An LSTM variant = nisqa_tts.tar's args with the shape switched +
its StandardCNN convolutions + seeded weights for fc_out (unless it keeps the shipped 20-wide one), every LSTM layer and
the pooling heads (NumPy PCG64: the same here, in oracle/make_lstm_golden.py that feeds them to the UNMODIFIED reference
modules, and on the GPU box).
"""
import math

import numpy as np
import torch

from oracle.variants import CLIPS  # noqa: F401  (the clips every LSTM variant is scored on)

# name -> args overrides of nisqa_tts.tar.  Together: every H class (32, 64, 96, 128 with 2 layers, 192 with 3 layers,
# 256), both directions, fc_out 20 / 100 / None, every pooling module, and three NISQA_DIM models.
LSTM_VARIANTS = {
    "tts_h32_uni_fc20_avg": {"td_lstm_h": 32, "td_lstm_bidirectional": False, "pool": "avg"},
    "tts_h96_bi_fc100_att": {"td_lstm_h": 96, "cnn_fc_out_h": 100, "pool": "att", "pool_att_h": None},
    "tts_h128_l2_bi_lastbi": {"td_lstm_num_layers": 2},
    "tts_h192_l3_uni_fcnone_attff": {"td_lstm_h": 192, "td_lstm_num_layers": 3, "td_lstm_bidirectional": False,
                                     "cnn_fc_out_h": None, "pool": "att", "pool_att_h": 128},
    "tts_h256_bi_fc100_max": {"td_lstm_h": 256, "cnn_fc_out_h": 100, "pool": "max"},
    "dim_h64_l2_uni_fc20_last": {"model": "NISQA_DIM", "td_lstm_h": 64, "td_lstm_num_layers": 2,
                                 "td_lstm_bidirectional": False, "pool": "last_step"},
    "dim_h96_uni_fcnone_attff": {"model": "NISQA_DIM", "td_lstm_h": 96, "td_lstm_bidirectional": False,
                                 "cnn_fc_out_h": None, "pool": "att", "pool_att_h": 128},
    "dim_h256_bi_fc100_lastbi": {"model": "NISQA_DIM", "td_lstm_h": 256, "cnn_fc_out_h": 100},
}


def lstm_checkpoint(name, base_args, base_sd, over=None):
    """-> (args, state_dict) of an LSTM_VARIANTS entry (or of `over`, overrides of the same form, seeded by `name`);
    base_args / base_sd are nisqa_tts.tar's."""
    args = dict(base_args)
    args.update(over if over is not None else LSTM_VARIANTS[name])
    args["td_lstm_dropout"] = 0
    if args.get("pool_att_h"):
        args["pool_att_dropout"] = 0.1          # (nisqa_tts.tar's args leave it None; eval mode ignores it)
    sd = {k: v for k, v in base_sd.items() if not k.startswith(("time_dependency", "pool.", "pool_layers."))}
    rng = np.random.default_rng(sum(map(ord, name)) + 5)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))      # noqa: E731
    fc = args.get("cnn_fc_out_h")
    if fc != 20:
        sd = {k: v for k, v in sd.items() if not k.startswith("cnn.model.fc_out.")}
        if fc:
            sd["cnn.model.fc_out.weight"] = t(rng.standard_normal((fc, 768)) / math.sqrt(768))
            sd["cnn.model.fc_out.bias"] = t(rng.normal(0, 0.05, fc))
    H, dirs = args["td_lstm_h"], 2 if args["td_lstm_bidirectional"] else 1
    k = 1.0 / math.sqrt(H)                      # nn.LSTM's own initialisation range
    p = "time_dependency.model.lstm."
    for l in range(args["td_lstm_num_layers"]):
        n_in = (fc or 768) if l == 0 else dirs * H
        for d in range(dirs):
            sfx = "_l%d%s" % (l, "_reverse" if d else "")
            sd[p + "weight_ih" + sfx] = t(rng.uniform(-k, k, (4 * H, n_in)))
            sd[p + "weight_hh" + sfx] = t(rng.uniform(-k, k, (4 * H, H)))
            sd[p + "bias_ih" + sfx] = t(rng.uniform(-k, k, 4 * H))
            sd[p + "bias_hh" + sfx] = t(rng.uniform(-k, k, 4 * H))
    D = dirs * H
    heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    for pf in heads:
        def lin(key, n_out, n_in, scale, bias):
            sd[pf + key + ".weight"] = t(rng.standard_normal((n_out, n_in)) * scale)
            sd[pf + key + ".bias"] = t(bias(n_out))
        score_bias = lambda n: rng.uniform(1.0, 4.0, n)      # noqa: E731  (scores in the MOS range)
        small_bias = lambda n: rng.normal(0, 0.05, n)        # noqa: E731
        if args["pool"] == "att" and args.get("pool_att_h"):
            lin("linear1", 128, D, 1.0 / math.sqrt(D), small_bias)
            lin("linear2", 1, 128, 1.0 / math.sqrt(128), small_bias)
            lin("linear3", 1, D, 0.3, score_bias)
        elif args["pool"] == "att":
            lin("linear1", 1, D, 1.0 / math.sqrt(D), small_bias)
            lin("linear2", 1, D, 0.3, score_bias)
        else:
            lin("linear", 1, D, 0.3, score_bias)
    return args, sd
