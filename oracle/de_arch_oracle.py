"""CPU oracle for double-ended (NISQA_DE) checkpoints with the other framewise and time-dependency models
(oracle/de_arch_variants.py): AdaptCNN, StandardCNN, SkipCNN or DFF, then a self-attention or LSTM td, on both signals;
alignment and fusion at td's fan_out; a self-attention td_2; the pooling module.

TEST INFRASTRUCTURE ONLY, like oracle/nisqa_oracle.py, whose front end, ``de_align`` and ``de_fuse`` it reuses
unchanged, and oracle/td_pair_oracle.py, whose ``framewise``, ``stage`` and ``td2_state_dict`` run the framewise model
and the time-dependency stages (``lib`` = nisqa/NISQA_lib.py).  Pinned against the unmodified reference NISQA_DE by
tests/golden/variants_de_arch.npz (oracle/make_de_arch_golden.py).
"""
import numpy as np
import torch

from oracle import lstm_oracle as LO
from oracle import nisqa_oracle as O
from oracle import td_pair_oracle as TP


def forward_from_mel(args, sd, spec, spec_ref, taps=None):
    """NISQA_DE.forward (lib:404-424) for one (degraded, reference) pair of mel dB spectrograms -> score [1]."""
    if args.get("td") not in ("self_att", "lstm") or args.get("td_2") != "self_att":
        raise NotImplementedError("de_arch oracle: NISQA_DE with a self-attention or LSTM td and a self-attention td_2")
    with torch.no_grad():
        x, y = (TP.stage(args, "td", sd, TP.framewise(args, sd, O.segments(sp, args))) for sp in (spec, spec_ref))
        y_al = O.de_align(args, x, y, sd)
        if taps is not None: taps["de_x"], taps["de_y"], taps["de_y_aligned"] = x, y, y_al
        td2 = TP.stage(args, "td_2", TP.td2_state_dict(sd), O.de_fuse(args, x, y_al, sd))
        if taps is not None: taps["td2_out"] = td2
        return LO.pool(args, sd, td2).numpy()


def predict_pcm_de(args, sd, y_deg, sr_deg, y_ref, sr_ref, taps=None):
    """(degraded, reference) float32 mono samples -> (score [1], (n_seg_deg, n_seg_ref), status) for one double-ended
    row (lib:2132-2214 + lib:1420-1439)."""
    y_deg = np.ascontiguousarray(y_deg, dtype=np.float32)
    y_ref = np.ascontiguousarray(y_ref, dtype=np.float32)
    _, n1, st1 = O.segment_counts(y_deg.shape[0], sr_deg, args)
    _, n2, st2 = O.segment_counts(y_ref.shape[0], sr_ref, args)
    if st1 != O.STATUS_OK or st2 != O.STATUS_OK:
        return np.full(1, np.nan, dtype=np.float32), (n1, n2), (st1 if st1 != O.STATUS_OK else st2)
    score = forward_from_mel(args, sd, O.mel_db(y_deg, sr_deg, args), O.mel_db(y_ref, sr_ref, args), taps)
    return score.astype(np.float32), (n1, n2), O.STATUS_OK
