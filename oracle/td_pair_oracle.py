"""CPU oracle for checkpoints whose td and td_2 are any pair of self-attention and LSTM stages (oracle/td_pair_variants.py):
framewise model -> td -> td_2 -> pooling, for NISQA and NISQA_DIM.

TEST INFRASTRUCTURE ONLY, like oracle/nisqa_oracle.py and oracle/lstm_oracle.py, whose framewise models,
``self_attention``, ``lstm`` and ``pool`` it reuses unchanged.  Those read the ``time_dependency.model.`` prefix, so td_2
runs on the state dict with its ``time_dependency_2.`` keys remapped onto it.  Pinned against the unmodified reference
modules by tests/golden/variants_td_pairs.npz (oracle/make_td_pair_golden.py).
"""
import numpy as np
import torch

from oracle import lstm_oracle as LO
from oracle import nisqa_oracle as O


def td2_state_dict(sd):
    """time_dependency_2.* renamed to time_dependency.* (only those keys)"""
    return {k.replace("time_dependency_2.", "time_dependency.", 1): v for k, v in sd.items() if k.startswith("time_dependency_2.")}


def framewise(args, sd, x):
    if args["cnn_model"] == "adapt":
        return O.adapt_cnn(sd, x, args)
    if args["cnn_model"] == "standard":
        return O.standard_cnn(sd, x, args)
    if args["cnn_model"] in (None, "skip"):
        return O.skip_cnn(sd, x)
    if args["cnn_model"] == "dff":
        return O.dff(sd, x)
    raise NotImplementedError(args["cnn_model"])


def stage(args, key, sd, x):
    """one time-dependency stage ('td' / 'td_2', its weights under time_dependency.model.) for ONE clip"""
    if args.get(key) == "self_att":
        return O.self_attention(sd, x, pos_enc=bool(args.get(key + "_sa_pos_enc")))
    if args.get(key) == "lstm":
        return LO.lstm(sd, x)
    if args.get(key) in (None, "skip"):
        return x
    raise NotImplementedError(args.get(key))


def forward_from_mel(args, sd, spec, taps=None):
    """mel dB [n_mels, F] -> scores [1] or [5]."""
    x = O.segments(spec, args)
    with torch.no_grad():
        feats = framewise(args, sd, x)
        if taps is not None: taps["cnn_feat"] = feats
        td = stage(args, "td", sd, feats)
        if taps is not None: taps["td1_out"] = td
        td = stage(args, "td_2", td2_state_dict(sd), td)
        if taps is not None: taps["td_out"] = td
        return LO.pool(args, sd, td).numpy()


def predict_pcm(args, sd, y, sr, taps=None):
    """float32 mono samples -> (scores, n_segments, status) for one clip."""
    y = np.ascontiguousarray(y, dtype=np.float32)
    _, n_seg, status = O.segment_counts(y.shape[0], sr, args)
    n_out = 5 if args["model"] == "NISQA_DIM" else 1
    if status != O.STATUS_OK:
        return np.full(n_out, np.nan, dtype=np.float32), n_seg, status
    return forward_from_mel(args, sd, O.mel_db(y, sr, args), taps).astype(np.float32), n_seg, O.STATUS_OK
