"""tests/golden/alignment.npz from the UNMODIFIED reference NISQA_DE's Alignment module (runs only in the build container).

    python -m oracle.make_alignment_golden       # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

For every entry of oracle/variants.py DE_VARIANTS (all five alignment modules, hard and soft) and a few of
oracle/de_arch_variants.py DE_ARCH_VARIANTS (LSTM tds of W = 512, 384 and 128: soft CTAs of several column groups) a
temporary checkpoint is scored by the reference's own ``nisqaModel(args).predict()`` with ``csv_ref`` on ALIGN_PAIRS
(one pair per batch).  A forward hook on ``model.align`` takes its inputs ``(query, y, n_wins_y)``, calls the module's
own ``att``, masks and softmaxes exactly as ``Alignment.forward`` does (lib:1279-1285), and stores per pair, for the
degraded clip's Sx steps (a pre-hook on the model reads n_wins) and the reference's Sy:
    <name>/<p>/scores  : float32 [Sx, Sy] the masked attention scores (AttBahdanau: with v's bias)
    <name>/<p>/idx     : int64 [Sx] ApplyHardAttention.idx (hard variants)
    <name>/<p>/ref_seg, weight, centroid, peak : the four values of include/nisqa_b200.h nisqa_alignment_out, from the
                         float32 scores and softmax (first maximal score; its softmax weight; sum_j a_ij j; its score)
Front end: oracle/librosa_compat.py (see oracle/make_golden.py for why).
"""
import os
import sys
import tempfile

import numpy as np
import torch

from oracle.build_ref import reference_dir

REF = reference_dir()     # the reference checkout ($NISQA_REFERENCE_DIR); exits with a message when absent
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import de_arch_variants, librosa_compat, variants  # noqa: E402
from nisqa_b200 import wav  # noqa: E402

# DE_PAIRS 1 and 2 (short clips; other rates), and a pair whose reference spans two 64-step key blocks at every
# checkpoint's segment hop (mos_only: 52 x 77 steps; the tts-based LSTM variants: 205 x 305)
ALIGN_PAIRS = variants.DE_PAIRS[1:] + [((87, 2.2, 16000), (87, 3.2, 16000))]
ARCH = ["std_fc20_lstm256bi_l2_dot_soft", "std_fcnone_lstm192bi_l3_bahd_soft", "std_fc100_lstm64bi_cosine_hard"]
# the LSTM variants (segment hop 1) on the shorter pairs only: their score matrices grow with the square of the steps
ARCH_PAIRS = [variants.DE_PAIRS[1], ((88, 0.8, 16000), (88, 1.2, 16000))]


def checkpoints():
    """-> [(name, args, state_dict, pairs)] of the golden's variants"""
    out = []
    for name in variants.DE_VARIANTS:
        ck = torch.load(os.path.join(REF, "weights", "nisqa_mos_only.tar"), map_location="cpu", weights_only=False)
        args, sd = variants.de_checkpoint(name, ck["args"], ck["model_state_dict"])
        out.append((name, args, sd, ALIGN_PAIRS))
    for name in ARCH:
        base = de_arch_variants.DE_ARCH_VARIANTS[name][0]
        ck = torch.load(os.path.join(REF, "weights", base), map_location="cpu", weights_only=False)
        args, sd = de_arch_variants.de_arch_checkpoint(name, ck["args"], ck["model_state_dict"])
        out.append((name, args, sd, ARCH_PAIRS))
    return out


def main():
    librosa_compat.install()
    sys.path.insert(0, REF)
    from nisqa.NISQA_model import nisqaModel
    import pandas as pd
    import torch.nn.functional as F
    torch.set_num_threads(1)              # (one thread: the same float32 sums on every build machine)
    out = {}
    for name, args, sd, pairs in checkpoints():
        with tempfile.TemporaryDirectory() as td:
            rows = []
            for i, pair in enumerate(pairs):
                deg, srd, ref, srr = variants.de_pair_pcm(pair)
                wav.write_wav_pcm16(os.path.join(td, "deg%d.wav" % i), deg, srd)
                wav.write_wav_pcm16(os.path.join(td, "ref%d.wav" % i), ref, srr)
                rows.append(("deg%d.wav" % i, "ref%d.wav" % i))
            pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(os.path.join(td, "files.csv"), index=False)
            ckpt_path = os.path.join(td, name + ".tar")
            torch.save({"args": args, "model_state_dict": sd}, ckpt_path)
            m = nisqaModel({"mode": "predict_csv", "pretrained_model": ckpt_path, "csv_file": "files.csv", "csv_deg": "deg",
                            "csv_ref": "ref", "data_dir": td, "output_dir": None, "num_workers": 0, "bs": 1, "ms_channel": None,
                            "tr_bs_val": 1, "tr_num_workers": 0, "tr_device": "cpu"})
            seen, n_wins = [], []

            def pre(module, inputs):
                n_wins.append(inputs[1])

            def hook(module, inputs, output):
                query, y, n_wins_y = inputs
                att, _ = module.att(query, y)
                module._mask_attention(att, y, n_wins_y)
                a = F.softmax(att, dim=2)
                sx, sy = int(n_wins[-1][0, 0]), int(n_wins_y[0])
                s, a = att[0, :sx, :sy].detach(), a[0, :sx, :sy].detach()
                r = {"scores": s.numpy().astype(np.float32)}
                if args["de_align_apply"] == "hard":
                    r["idx"] = module.apply_att.idx[0, :sx].numpy().astype(np.int64)
                j = (s == s.max(1, keepdim=True)[0]).to(torch.float32).argmax(1)
                rr = torch.arange(sx)
                r["ref_seg"] = j.numpy().astype(np.int32)
                r["weight"] = a[rr, j].numpy().astype(np.float32)
                r["centroid"] = (a @ torch.arange(sy, dtype=torch.float32)).numpy().astype(np.float32)
                r["peak"] = s[rr, j].numpy().astype(np.float32)
                seen.append(r)
            h1 = m.model.register_forward_pre_hook(pre)
            h2 = m.model.align.register_forward_hook(hook)
            m.predict()
            h1.remove(); h2.remove()
            assert len(seen) == len(pairs), (name, len(seen))
            for p, r in enumerate(seen):
                for k, v in r.items():
                    out["%s/%d/%s" % (name, p, k)] = v
            print(name, [r["scores"].shape for r in seen])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "alignment.npz"), **out)


if __name__ == "__main__":
    main()
