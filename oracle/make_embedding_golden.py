"""tests/golden/embeddings.npz from the UNMODIFIED reference modules (runs only in the build container).

    python -m oracle.make_embedding_golden        # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

The checkpoints and clips are those of oracle/make_segment_golden.py (oracle/segment_variants.py: SEGMENT_VARIANTS on
SEGMENT_CLIPS, NISQA_DE on SEGMENT_DE_PAIRS), so the pooled vectors here tie to the rows tests/golden/segments.npz holds.
Each is scored by the reference's own ``nisqaModel(args).predict()``.  A forward pre-hook on each pooling head's last
Linear (PoolAttFF linear3, PoolAtt linear2, every other module's linear: lib:1099-1225) keeps that Linear's input, the
pooled vector.  Front end: oracle/librosa_compat.py (see oracle/make_golden.py for why).

Per variant the archive holds <name>/pooled float32 [B, n_heads, width] and <name>/scores float64 [B, n_heads] (the
reference's clip scores).
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

LAST_LINEAR = {"PoolAttFF": "linear3", "PoolAtt": "linear2"}      # every other module: "linear"


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
            hooks = []
            for k, h in enumerate(heads):
                lin = getattr(h.model, LAST_LINEAR.get(type(h.model).__name__, "linear"))
                hooks.append(lin.register_forward_pre_hook(lambda mod, inp, k=k: seen[k].append(inp[0].detach().clone())))
            df = m.predict()
            for h in hooks:
                h.remove()
            cols = [c for c in ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"] if c in df]
            pooled = np.stack([torch.cat(s).numpy() for s in seen], axis=1).astype(np.float32)
            out[name + "/pooled"] = pooled
            out[name + "/scores"] = df[cols].to_numpy().astype(np.float64)
            print(name, pooled.shape, out[name + "/scores"].reshape(-1).tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "embeddings.npz"), **out)


if __name__ == "__main__":
    main()
