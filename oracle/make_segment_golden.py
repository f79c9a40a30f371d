"""tests/golden/segments.npz from the UNMODIFIED reference modules (runs only in the build container).

    python -m oracle.make_segment_golden          # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

For every entry of oracle/segment_variants.py a temporary checkpoint ({'args', 'model_state_dict'}) is written and scored
by the reference's own ``nisqaModel(args).predict()`` (strict ``load_state_dict``, as the other generators) on
``SEGMENT_CLIPS`` (NISQA_DE: ``SEGMENT_DE_PAIRS`` with ``csv_ref``).  A forward pre-hook on each pooling module keeps
the padded rows [B, T, D] it reads and n_wins.  Then, per clip and segment t, the reference's own pooling module is
called on the one-row sequence x[b:b+1, t:t+1] with n_wins = 1: the segment score.  The weights come from that module's
own layers: the attention logits of linear1 (PoolAtt) or linear2(activation(linear1)) (PoolAttFF), masked to the clip's
n_wins and softmaxed over the padded time axis as the module does; PoolAvg 1 / n_wins, PoolLastStep one at n_wins - 1,
PoolMax and PoolLastStepBi NaN.  Front end: oracle/librosa_compat.py (see oracle/make_golden.py for why).

Per variant the archive holds <name>/x (the rows of every clip, concatenated, float32; or /x_from, the name of an
earlier variant with the same rows), /seg_scores and /seg_weights [N, n_heads], /counts [B] and /scores [B, n_heads]
(the reference's clip scores).
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

from oracle import librosa_compat, segment_variants as SV, variants  # noqa: E402
from nisqa_b200 import synth, wav  # noqa: E402


def _weights(mod, x, n_wins, kind):
    """the pooling module's weight of every step of x [B, T, D] -> [B, T] (NaN where no weight exists)"""
    B, T, _ = x.shape
    mask = torch.arange(T)[None, :] < n_wins[:, None].to(torch.long)
    if kind == "PoolAtt":
        att = mod.linear1(x).transpose(2, 1)
    elif kind == "PoolAttFF":
        att = mod.linear2(mod.dropout(mod.activation(mod.linear1(x)))).transpose(2, 1)
    elif kind == "PoolAvg":
        return torch.where(mask, 1.0 / n_wins[:, None].to(x.dtype), torch.zeros(()))
    elif kind == "PoolLastStep":
        return (torch.arange(T)[None, :] == (n_wins[:, None].to(torch.long) - 1)).to(x.dtype)
    else:
        return torch.full((B, T), float("nan"))
    att[~mask.unsqueeze(1)] = float("-Inf")
    return torch.softmax(att, dim=2)[:, 0, :]


def main():
    librosa_compat.install()
    sys.path.insert(0, REF)
    from nisqa.NISQA_model import nisqaModel
    import pandas as pd
    torch.set_num_threads(1)              # (one thread: the same float32 sums on every build machine)
    out = {}
    for name in SV.SEGMENT_VARIANTS:
        args, sd = SV.segment_checkpoint(name, os.path.join(REF, "weights"))
        de = args["model"] == "NISQA_DE"
        with tempfile.TemporaryDirectory() as td:
            if de:
                rows = []
                for i, pair in enumerate(SV.SEGMENT_DE_PAIRS):
                    deg, srd, ref, srr = variants.de_pair_pcm(pair)
                    wav.write_wav_pcm16(os.path.join(td, "deg%d.wav" % i), deg, srd)
                    wav.write_wav_pcm16(os.path.join(td, "ref%d.wav" % i), ref, srr)
                    rows.append(("deg%d.wav" % i, "ref%d.wav" % i))
                pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(os.path.join(td, "files.csv"), index=False)
            else:
                files = []
                for seed, sec, sr in SV.SEGMENT_CLIPS:
                    fn = "v%03d.wav" % seed
                    wav.write_wav_pcm16(os.path.join(td, fn), synth.synth_speech_pcm16(seed, sec, sr), sr)
                    files.append(fn)
                pd.DataFrame({"deg": files}).to_csv(os.path.join(td, "files.csv"), index=False)
            ckpt_path = os.path.join(td, name + ".tar")
            torch.save({"args": args, "model_state_dict": sd}, ckpt_path)
            m = nisqaModel({"mode": "predict_csv", "pretrained_model": ckpt_path, "csv_file": "files.csv", "csv_deg": "deg",
                            "csv_ref": "ref" if de else None, "data_dir": td, "output_dir": None, "num_workers": 0,
                            "bs": 4, "ms_channel": None, "tr_bs_val": 4, "tr_num_workers": 0, "tr_device": "cpu"})
            heads = list(m.model.pool_layers) if args["model"] == "NISQA_DIM" else [m.model.pool]
            seen = [[] for _ in heads]
            hooks = [h.register_forward_pre_hook(lambda mod, inp, k=k: seen[k].append((inp[0].detach().clone(),
                                                                                         inp[1].detach().clone())))
                     for k, h in enumerate(heads)]
            df = m.predict()
            for h in hooks:
                h.remove()
            cols = [c for c in ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"] if c in df]
            xs, counts, s_all, w_all = [], [], [], []
            with torch.no_grad():
                for k, head in enumerate(heads):
                    mod, kind = head.model, type(head.model).__name__
                    s_k, w_k = [], []
                    for x, n_wins in seen[k]:
                        w = _weights(mod, x.clone(), n_wins, kind)
                        for b in range(x.shape[0]):
                            n = int(n_wins[b])
                            for t in range(n):
                                s_k.append(float(head(x[b:b + 1, t:t + 1].clone(), torch.ones(1, dtype=n_wins.dtype))[0, 0]))
                            w_k.extend(w[b, :n].tolist())
                            if k == 0:
                                xs.append(x[b, :n].numpy())
                                counts.append(n)
                    s_all.append(s_k)
                    w_all.append(w_k)
            x = np.concatenate(xs).astype(np.float32)
            same = [k[:-2] for k in out if k.endswith("/x") and np.array_equal(out[k], x)]
            if same:
                out[name + "/x_from"] = np.array(same[0])      # (variants that change the pooling module only)
            else:
                out[name + "/x"] = x
            out[name + "/seg_scores"] = np.array(s_all, dtype=np.float64).T
            out[name + "/seg_weights"] = np.array(w_all, dtype=np.float64).T
            out[name + "/counts"] = np.array(counts, dtype=np.int64)
            out[name + "/scores"] = df[cols].to_numpy().astype(np.float64)
            print(name, counts, out[name + "/scores"].reshape(-1).tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "segments.npz"), **out)


if __name__ == "__main__":
    main()
