"""CPU oracle for StandardCNN + LSTM checkpoints of any accepted shape (oracle/lstm_variants.py): a stacked LSTM of
any width, depth and direction and every pooling module, for NISQA and NISQA_DIM.

TEST INFRASTRUCTURE ONLY, like oracle/nisqa_oracle.py, whose front end, StandardCNN and pooling functions it reuses
unchanged (``lib`` = nisqa/NISQA_lib.py).  The shipped one-layer BiLSTM still goes through ``nisqa_oracle.bilstm``.
Pinned against the unmodified reference modules by tests/golden/variants_lstm.npz (oracle/make_lstm_golden.py).
"""
import numpy as np
import torch

from oracle import nisqa_oracle as O

P = "time_dependency.model.lstm."


def lstm_shape(sd):
    """(H, layers, dirs) from the checkpoint's tensors."""
    layers = 0
    while P + "weight_hh_l%d" % layers in sd:
        layers += 1
    return sd[P + "weight_hh_l0"].shape[1], layers, 2 if P + "weight_hh_l0_reverse" in sd else 1


def lstm(sd, feats):
    """nn.LSTM (lib:898-943) for ONE clip: layer l + 1 reads layer l's outputs (both directions side by side); each
    direction runs over the clip's own steps, the reverse one from its last step.  PyTorch gate order i, f, g, o."""
    H, layers, dirs = lstm_shape(sd)
    if (layers, dirs) == (1, 2):
        return O.bilstm(sd, feats)
    S = feats.shape[0]
    x = feats
    for l in range(layers):
        outs = []
        for d in range(dirs):
            sfx = "_l%d%s" % (l, "_reverse" if d else "")
            w_ih, w_hh = sd[P + "weight_ih" + sfx], sd[P + "weight_hh" + sfx]
            gx = x @ w_ih.t() + (sd[P + "bias_ih" + sfx] + sd[P + "bias_hh" + sfx])
            h, c = torch.zeros(H), torch.zeros(H)
            out = torch.zeros(S, H)
            for t in (range(S - 1, -1, -1) if d else range(S)):
                g = gx[t] + w_hh @ h
                i, f, gg, o = g[:H], g[H:2 * H], g[2 * H:3 * H], g[3 * H:]
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
                h = torch.sigmoid(o) * torch.tanh(c)
                out[t] = h
            outs.append(out)
        x = torch.cat(outs, dim=1)
    return x


def pool(args, sd, x):
    """The pooling module of every head (order mos, noi, dis, col, loud for NISQA_DIM, lib:255-266)."""
    prefixes = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    outs = []
    for pf in prefixes:
        if args["pool"] == "att":
            outs.append(O.pool_attff(sd, pf, x) if args.get("pool_att_h") else O.pool_att(sd, pf, x))
        elif args["pool"] == "last_step_bi":
            outs.append(O.pool_last_step_bi(sd, pf, x))
        else:
            outs.append({"avg": O.pool_avg, "max": O.pool_max, "last_step": O.pool_last_step}[args["pool"]](sd, pf, x))
    return torch.cat(outs)


def forward_from_mel(args, sd, spec, taps=None):
    """mel dB [n_mels, F] -> scores [1] or [5]."""
    if args["cnn_model"] != "standard" or args["td"] != "lstm" or args.get("td_2") not in (None, "skip"):
        raise NotImplementedError("lstm oracle: StandardCNN + LSTM, no td_2")
    x = O.segments(spec, args)
    with torch.no_grad():
        feats = O.standard_cnn(sd, x, args)
        if taps is not None: taps["cnn_feat"] = feats
        td = lstm(sd, feats)
        if taps is not None: taps["td_out"] = td
        return pool(args, sd, td).numpy()


def predict_pcm(args, sd, y, sr, taps=None):
    """float32 mono samples -> (scores, n_segments, status) for one clip."""
    y = np.ascontiguousarray(y, dtype=np.float32)
    _, n_seg, status = O.segment_counts(y.shape[0], sr, args)
    n_out = 5 if args["model"] == "NISQA_DIM" else 1
    if status != O.STATUS_OK:
        return np.full(n_out, np.nan, dtype=np.float32), n_seg, status
    return forward_from_mel(args, sd, O.mel_db(y, sr, args), taps).astype(np.float32), n_seg, O.STATUS_OK
