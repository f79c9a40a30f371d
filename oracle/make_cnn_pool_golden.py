"""tests/golden/variants_cnn_pool.npz from the UNMODIFIED reference modules (runs only in the build container).

    python -m oracle.make_cnn_pool_golden          # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

For every entry of oracle/cnn_pool_variants.py a temporary checkpoint ({'args', 'model_state_dict'}) is written and scored by
the reference's own ``nisqaModel(args).predict()`` (strict ``load_state_dict`` into the reference's NISQA / NISQA_DIM /
NISQA_DE built with the variant's cnn_pool_1/2/3 - a wrong key or shape fails right here) on the clips of ``POOL_CLIPS``
(NISQA_DE: the pairs of ``POOL_DE_PAIRS``).  Front end: oracle/librosa_compat.py (see oracle/make_golden.py for why).
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

from oracle import cnn_pool_variants as V, librosa_compat  # noqa: E402
from oracle.variants import de_pair_pcm  # noqa: E402
from nisqa_b200 import synth, wav  # noqa: E402


def main():
    librosa_compat.install()
    sys.path.insert(0, REF)
    from nisqa.NISQA_model import nisqaModel
    import pandas as pd
    torch.set_num_threads(1)              # (one thread: the same float32 sums on every build machine)
    out = {}
    for name, (base, _, _, _, _) in V.CNN_POOL_VARIANTS.items():
        ck = torch.load(os.path.join(REF, "weights", base), map_location="cpu", weights_only=False)
        args, sd = V.cnn_pool_checkpoint(name, ck["args"], ck["model_state_dict"])
        de = args["model"] == "NISQA_DE"
        with tempfile.TemporaryDirectory() as td:
            if de:
                rows = []
                for i, pair in enumerate(V.POOL_DE_PAIRS):
                    deg, srd, ref, srr = de_pair_pcm(pair)
                    wav.write_wav_pcm16(os.path.join(td, "deg%d.wav" % i), deg, srd)
                    wav.write_wav_pcm16(os.path.join(td, "ref%d.wav" % i), ref, srr)
                    rows.append(("deg%d.wav" % i, "ref%d.wav" % i))
                pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(os.path.join(td, "files.csv"), index=False)
            else:
                files = []
                for seed, sec, sr in V.POOL_CLIPS:
                    fn = "v%03d.wav" % seed
                    wav.write_wav_pcm16(os.path.join(td, fn), synth.synth_speech_pcm16(seed, sec, sr), sr)
                    files.append(fn)
                pd.DataFrame({"deg": files}).to_csv(os.path.join(td, "files.csv"), index=False)
            ckpt_path = os.path.join(td, name + ".tar")
            torch.save({"args": args, "model_state_dict": sd}, ckpt_path)
            opts = {"mode": "predict_csv", "pretrained_model": ckpt_path, "csv_file": "files.csv", "csv_deg": "deg",
                    "data_dir": td, "output_dir": None, "num_workers": 0, "bs": 4, "ms_channel": None,
                    "tr_bs_val": 4, "tr_num_workers": 0, "tr_device": "cpu"}
            if de:
                opts["csv_ref"] = "ref"
            df = nisqaModel(opts).predict()
            cols = [c for c in ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"] if c in df]
            out[name] = df[cols].to_numpy().astype(np.float64)
            print(name, out[name].tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "variants_cnn_pool.npz"), **out)


if __name__ == "__main__":
    main()
