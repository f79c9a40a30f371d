"""Architecture variants reachable through user-trained checkpoints (SURVEY.md 8f.4) for which the reference ships
no weights: the other pooling modules (PoolAtt / PoolAvg / PoolMax / PoolLastStep, reference lib:1117-1225) and the
positional encoding of the self-attention block (lib:1042-1062).

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  A variant checkpoint = a shipped checkpoint's args with the
variant's options switched + its state_dict with the pooling head replaced by deterministic seeded weights (NumPy
PCG64: the same here, in the golden generator that feeds them to the UNMODIFIED reference modules, and on the GPU box).
"""
import math

import numpy as np
import torch

# name -> (base checkpoint, args overrides)
VARIANTS = {
    "dim_pool_avg": ("nisqa.tar", {"pool": "avg", "pool_att_h": None}),
    "dim_pool_max": ("nisqa.tar", {"pool": "max", "pool_att_h": None}),
    "dim_pool_last_step": ("nisqa.tar", {"pool": "last_step", "pool_att_h": None}),
    "dim_pool_att": ("nisqa.tar", {"pool": "att", "pool_att_h": None}),
    "dim_pos_enc": ("nisqa.tar", {"td_sa_pos_enc": True}),
    "mos_pool_att_pos_enc": ("nisqa_mos_only.tar", {"pool": "att", "pool_att_h": None, "td_sa_pos_enc": True}),
    "tts_pool_avg": ("nisqa_tts.tar", {"pool": "avg"}),
    "tts_pool_max": ("nisqa_tts.tar", {"pool": "max"}),
    "tts_pool_last_step": ("nisqa_tts.tar", {"pool": "last_step"}),
    # td_2 = 'self_att': a second self-attention stack behind the first (lib:114-141, 236-268), seeded weights
    "dim_td2_sa": ("nisqa.tar", {"td_2": "self_att", "td_2_sa_d_model": 64, "td_2_sa_nhead": 1, "td_2_sa_h": 64,
                                 "td_2_sa_num_layers": 2, "td_2_sa_pos_enc": None, "td_2_sa_dropout": 0.1}),
    "mos_td2_sa_pos_enc": ("nisqa_mos_only.tar", {"td_2": "self_att", "td_2_sa_d_model": 64, "td_2_sa_nhead": 1, "td_2_sa_h": 64,
                                                  "td_2_sa_num_layers": 1, "td_2_sa_pos_enc": True, "td_2_sa_dropout": 0.1}),
    # framewise models without convolutions (lib:504-583): seeded weights for the framewise module and the first Linear
    "mos_skip": ("nisqa_mos_only.tar", {"cnn_model": "skip", "cnn_fc_out_h": None}),
    "dim_skip_fc": ("nisqa.tar", {"cnn_model": "skip", "cnn_fc_out_h": 128}),
    "mos_dff": ("nisqa_mos_only.tar", {"cnn_model": "dff", "cnn_fc_out_h": 256}),
    # AdaptCNN with its optional Linear behind conv6 (lib:682-684): seeded fc and first Linear of the stack
    "dim_adapt_fc": ("nisqa.tar", {"cnn_fc_out_h": 128}),
}
# double-ended variants (NISQA_DE, reference lib:272-424): nisqa_mos_only.tar's CNN, first self-attention stack and
# PoolAttFF head (identical shapes) + seeded weights for time_dependency_2 (input width 192 or 128)
DE_VARIANTS = {
    "de_cosine_hard": {"de_align": "cosine", "de_align_apply": "hard", "de_fuse": "x/y/-"},        # config/train_nisqa_double_ended.yaml
    "de_dot_soft": {"de_align": "dot", "de_align_apply": "soft", "de_fuse": "+/-"},
    "de_distance_soft_xy": {"de_align": "distance", "de_align_apply": "soft", "de_fuse": "x/y", "td_2_sa_pos_enc": True,
                            "td_2_sa_num_layers": 1},
    "de_dot_hard": {"de_align": "dot", "de_align_apply": "hard", "de_fuse": "x/y"},
    # the alignment modules with learned weights (seeded): AttLuong (lib:1344-1357), AttBahdanau (lib:1325-1342)
    "de_luong_soft": {"de_align": "luong", "de_align_apply": "soft", "de_fuse": "x/y/-"},
    "de_luong_hard": {"de_align": "luong", "de_align_apply": "hard", "de_fuse": "+/-"},
    "de_bahd_soft": {"de_align": "bahd", "de_align_apply": "soft", "de_fuse": "x/y/-"},
    # Fusion with its optional Linear (de_fuse_dim, lib:1399-1401)
    "de_cosine_soft_fuse_dim": {"de_align": "cosine", "de_align_apply": "soft", "de_fuse": "x/y/-", "de_fuse_dim": 64},
}
# (degraded, reference) pairs: (seed, seconds, sample rate) each; the degraded signal of pair 0 / 1 is derived from its
# reference (delay + noise + clipping: what a double-ended model is for), pair 2 has unrelated signals of other lengths
DE_PAIRS = [((81, 2.4, 48000), (81, 2.4, 48000)), ((82, 1.3, 16000), (82, 1.5, 16000)), ((83, 3.1, 44100), (84, 2.0, 48000))]


def de_pair_pcm(pair):
    """-> (deg int16, sr_deg, ref int16, sr_ref) of one DE_PAIRS entry."""
    from nisqa_b200 import synth
    (sd_, secd, srd), (sr_, secr, srr) = pair
    ref = synth.synth_speech_pcm16(sr_, secr, srr)
    if sd_ == sr_ and srd == srr:
        rng = np.random.default_rng(1000 + sd_)
        n = int(secd * srd)
        x = np.roll(ref.astype(np.float32), int(0.013 * srd))[:n] if n <= len(ref) else np.resize(ref.astype(np.float32), n)
        x = x * 1.6 + rng.standard_normal(n).astype(np.float32) * 250.0
        deg = np.clip(x, -9000, 9000).astype(np.int16)
    else:
        deg = synth.synth_speech_pcm16(sd_, secd, srd)
    return deg, srd, ref, srr


def td2_weights(sd, args, in_dim, rng):
    """Seeded weights of a time_dependency_2 self-attention stack (input width in_dim) written into sd."""
    def put(key, shape, scale, offset=0.0):
        sd["time_dependency_2.model." + key] = torch.from_numpy((rng.standard_normal(shape) * scale + offset).astype(np.float32))

    put("linear.weight", (64, in_dim), 1.0 / math.sqrt(in_dim)); put("linear.bias", (64,), 0.05)
    put("norm1.weight", (64,), 0.05, 1.0); put("norm1.bias", (64,), 0.05)
    for l in range(args["td_2_sa_num_layers"]):
        q = "layers.%d." % l
        put(q + "self_attn.in_proj_weight", (192, 64), 0.125); put(q + "self_attn.in_proj_bias", (192,), 0.05)
        put(q + "self_attn.out_proj.weight", (64, 64), 0.125); put(q + "self_attn.out_proj.bias", (64,), 0.05)
        put(q + "linear1.weight", (64, 64), 0.125); put(q + "linear1.bias", (64,), 0.05)
        put(q + "linear2.weight", (64, 64), 0.125); put(q + "linear2.bias", (64,), 0.05)
        put(q + "norm1.weight", (64,), 0.05, 1.0); put(q + "norm1.bias", (64,), 0.05)
        put(q + "norm2.weight", (64,), 0.05, 1.0); put(q + "norm2.bias", (64,), 0.05)
    if args.get("td_2_sa_pos_enc"):
        sd["time_dependency_2.model.pos_encoder.pe"] = positional_encoding()


def de_checkpoint(name, base_args, base_sd, over=None):
    """-> (args, state_dict) of a double-ended variant built on nisqa_mos_only.tar: a DE_VARIANTS entry, or `over` (an
    entry of the same form, seeded by `name`)."""
    over = DE_VARIANTS[name] if over is None else over
    args = dict(base_args)
    args.update({"model": "NISQA_DE", "td_2": "self_att", "td_2_sa_d_model": 64, "td_2_sa_nhead": 1, "td_2_sa_pos_enc": None,
                 "td_2_sa_num_layers": 2, "td_2_sa_h": 64, "td_2_sa_dropout": 0.1, "td_2_lstm_h": None,
                 "td_2_lstm_num_layers": None, "td_2_lstm_dropout": None, "td_2_lstm_bidirectional": None,
                 "de_fuse_dim": None})
    args.update(over)
    sd = {k: v for k, v in base_sd.items()}
    fdim = 192 if args["de_fuse"] == "x/y/-" else 128
    rng = np.random.default_rng(sum(map(ord, name)))
    if args.get("de_fuse_dim"):
        d = args["de_fuse_dim"]
        sd["fuse.lin_fusion.weight"] = torch.from_numpy((rng.standard_normal((d, fdim)) / math.sqrt(fdim)).astype(np.float32))
        sd["fuse.lin_fusion.bias"] = torch.from_numpy(rng.normal(0, 0.05, d).astype(np.float32))
        fdim = d
    td2_weights(sd, args, fdim, rng)

    def put(key, shape, scale):
        sd["align.att." + key] = torch.from_numpy((rng.standard_normal(shape) * scale).astype(np.float32))
    if args["de_align"] == "luong":
        put("W.weight", (64, 64), 0.125); put("W.bias", (64,), 0.05)
    if args["de_align"] == "bahd":
        put("Wq.weight", (128, 64), 0.125); put("Wq.bias", (128,), 0.05)
        put("Wy.weight", (128, 64), 0.125); put("Wy.bias", (128,), 0.05)
        put("v.weight", (1, 128), 0.3); put("v.bias", (1,), 0.05)
    return args, sd


# clips every variant is scored on: (seed, seconds, sample rate)
CLIPS = [(71, 2.0, 48000), (72, 0.9, 16000), (73, 3.7, 44100)]


def positional_encoding(d_model=64, max_len=3000):
    """The registered buffer of PositionalEncoding.__init__ (reference lib:1051-1058: the PyTorch tutorial formula,
    same torch ops so that the values are the ones the reference module builds)."""
    pe = torch.zeros(max_len, d_model)
    position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-math.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.unsqueeze(0).transpose(0, 1).contiguous()


def variant_checkpoint(name, base_args, base_sd):
    """-> (args, state_dict) of the variant."""
    _, over = VARIANTS[name]
    args = dict(base_args)
    args.update(over)
    sd = {k: v for k, v in base_sd.items()}
    pool_changed = "pool" in over
    if pool_changed:
        sd = {k: v for k, v in sd.items() if not (k.startswith("pool.") or k.startswith("pool_layers."))}
        d = 256 if args["td"] == "lstm" else 64
        heads = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
        rng = np.random.default_rng(sum(map(ord, name)))
        for pf in heads:
            def lin(key):
                sd[pf + key + ".weight"] = torch.from_numpy((rng.standard_normal((1, d)) * 0.15).astype(np.float32))
                sd[pf + key + ".bias"] = torch.from_numpy(rng.uniform(1.0, 4.0, 1).astype(np.float32))
            if args["pool"] == "att":
                lin("linear1")
                lin("linear2")
            else:
                lin("linear")
    if args.get("td_sa_pos_enc"):
        sd["time_dependency.model.pos_encoder.pe"] = positional_encoding()
    if args.get("td_2") == "self_att":
        td2_weights(sd, args, 64, np.random.default_rng(sum(map(ord, name))))
    if args.get("cnn_model") == "adapt" and args.get("cnn_fc_out_h"):
        rng = np.random.default_rng(sum(map(ord, name)) + 2)
        h = args["cnn_fc_out_h"]
        sd["cnn.model.fc.weight"] = torch.from_numpy((rng.standard_normal((h, 384)) / math.sqrt(384)).astype(np.float32))
        sd["cnn.model.fc.bias"] = torch.from_numpy(rng.normal(0, 0.05, h).astype(np.float32))
        sd["time_dependency.model.linear.weight"] = torch.from_numpy((rng.standard_normal((64, h)) / math.sqrt(h)).astype(np.float32))
    if args.get("cnn_model") in ("skip", "dff"):
        rng = np.random.default_rng(sum(map(ord, name)) + 1)
        sd = {k: v for k, v in sd.items() if not k.startswith("cnn.")}
        t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))

        def bn(prefix, n):      # running statistics in the range the data really has (mel dB / unit-scale activations)
            sd[prefix + "weight"] = t(rng.uniform(0.8, 1.2, n)); sd[prefix + "bias"] = t(rng.normal(0, 0.1, n))
            sd[prefix + "running_mean"] = t(rng.normal(0, 0.2, n)); sd[prefix + "running_var"] = t(rng.uniform(0.5, 1.5, n))
            sd[prefix + "num_batches_tracked"] = torch.tensor(1)

        def lin(prefix, n_out, n_in):
            sd[prefix + "weight"] = t(rng.standard_normal((n_out, n_in)) / math.sqrt(n_in)); sd[prefix + "bias"] = t(rng.normal(0, 0.05, n_out))
        h = args.get("cnn_fc_out_h")
        if args["cnn_model"] == "skip":
            bn("cnn.model.bn.", 1)
            sd["cnn.model.bn.running_mean"] = t([-35.0]); sd["cnn.model.bn.running_var"] = t([400.0])
            if h:
                lin("cnn.model.linear.", h, 720)
            fan = h or 720
        else:
            bn("cnn.model.bn1.", 1)
            sd["cnn.model.bn1.running_mean"] = t([-35.0]); sd["cnn.model.bn1.running_var"] = t([400.0])
            lin("cnn.model.lin1.", h, 720)
            for i in (2, 3, 4):
                lin("cnn.model.lin%d." % i, h, h)
            for i in (2, 3, 4, 5):
                bn("cnn.model.bn%d." % i, h)
            fan = h
        sd["time_dependency.model.linear.weight"] = t(rng.standard_normal((64, fan)) / math.sqrt(fan))
    return args, sd
