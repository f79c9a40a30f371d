"""Checkpoints whose per-segment scores and pooling weights tests/golden/segments.npz holds (oracle/make_segment_golden.py).

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  Every entry is a shipped checkpoint or an entry of one of the
existing variant registries, so the weights are the ones the other goldens were made from.  Together they cover every
pooling module behind self-attention (the shipped PoolAttFF, PoolAtt, PoolAvg, PoolMax, PoolLastStep), every pooling
module behind an LSTM (the shipped BiLSTM shape with PoolLastStepBi, PoolAvg, PoolMax, PoolLastStep; stacked LSTMs with
PoolAtt, PoolAttFF and PoolLastStepBi), td = 'skip' (the wide-row pooling, PoolAttFF and PoolAtt), a td_2 stack,
NISQA_DE and an ms_sr checkpoint.
"""
import os

from oracle import lstm_variants, td_skip_variants, variants

# name -> (base checkpoint, registry, registry entry, args overrides)
SEGMENT_VARIANTS = {
    "nisqa": ("nisqa.tar", None, None, None),
    "mos_only": ("nisqa_mos_only.tar", None, None, None),
    "tts": ("nisqa_tts.tar", None, None, None),
    "dim_pool_att": ("nisqa.tar", "variants", "dim_pool_att", None),
    "dim_pool_avg": ("nisqa.tar", "variants", "dim_pool_avg", None),
    "dim_pool_max": ("nisqa.tar", "variants", "dim_pool_max", None),
    "dim_pool_last_step": ("nisqa.tar", "variants", "dim_pool_last_step", None),
    "tts_pool_avg": ("nisqa_tts.tar", "variants", "tts_pool_avg", None),
    "tts_pool_max": ("nisqa_tts.tar", "variants", "tts_pool_max", None),
    "tts_pool_last_step": ("nisqa_tts.tar", "variants", "tts_pool_last_step", None),
    "tts_h96_bi_fc100_att": ("nisqa_tts.tar", "lstm", "tts_h96_bi_fc100_att", None),
    "dim_h96_uni_fcnone_attff": ("nisqa_tts.tar", "lstm", "dim_h96_uni_fcnone_attff", None),
    "tts_h128_l2_bi_lastbi": ("nisqa_tts.tar", "lstm", "tts_h128_l2_bi_lastbi", None),
    "mos_adapt_skip_attff": ("nisqa_mos_only.tar", "td_skip", "mos_adapt_skip_attff", None),
    "mos_skipcnn_skip_att": ("nisqa_mos_only.tar", "td_skip", "mos_skipcnn_skip_att", None),
    "dim_td2_sa": ("nisqa.tar", "variants", "dim_td2_sa", None),
    "de_cosine_hard": ("nisqa_mos_only.tar", "de", "de_cosine_hard", None),
    "mos_only_ms_sr16k": ("nisqa_mos_only.tar", None, None, {"ms_sr": 16000}),
}
# the clips (seed, seconds, rate) every single-ended variant is scored on, and NISQA_DE's (degraded, reference) pairs
# (short: the golden keeps every row the pooling modules read, up to 720 floats wide)
SEGMENT_CLIPS = [(71, 1.2, 48000), (72, 0.9, 16000)]
SEGMENT_DE_PAIRS = variants.DE_PAIRS[:2]


def segment_checkpoint(name, weights_dir):
    """-> (args, state_dict) of a SEGMENT_VARIANTS entry, its base checkpoint read from weights_dir"""
    import torch
    base, registry, entry, over = SEGMENT_VARIANTS[name]
    ck = torch.load(os.path.join(weights_dir, base), map_location="cpu", weights_only=False)
    args, sd = dict(ck["args"]), ck["model_state_dict"]
    if registry == "variants":
        args, sd = variants.variant_checkpoint(entry, args, sd)
    elif registry == "lstm":
        args, sd = lstm_variants.lstm_checkpoint(entry, args, sd)
    elif registry == "td_skip":
        args, sd = td_skip_variants.td_skip_checkpoint(entry, args, sd)
    elif registry == "de":
        args, sd = variants.de_checkpoint(entry, args, sd)
    args.update(over or {})
    return args, sd
