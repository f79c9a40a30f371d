"""tests/golden/variants_td_skip.npz from the UNMODIFIED reference modules (runs only in the build container).

    python -m oracle.make_td_skip_golden         # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

For every entry of oracle/td_skip_variants.py a temporary checkpoint ({'args', 'model_state_dict'}) is written and scored
by the reference's own ``nisqaModel(args).predict()`` (strict ``load_state_dict`` into the reference's NISQA / NISQA_DIM
built with td = 'skip' and the variant's td_2 - a wrong key or shape fails right here) on the clips of
``td_pair_variants.TD_PAIR_CLIPS``.  Front end: oracle/librosa_compat.py (see oracle/make_golden.py for why).
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

from oracle import librosa_compat, td_skip_variants  # noqa: E402
from oracle.td_pair_variants import TD_PAIR_CLIPS  # noqa: E402
from nisqa_b200 import synth, wav  # noqa: E402


def main():
    librosa_compat.install()
    sys.path.insert(0, REF)
    from nisqa.NISQA_model import nisqaModel
    import pandas as pd
    torch.set_num_threads(1)              # (one thread: the same float32 sums on every build machine)
    out = {}
    for name, (base, _, _) in td_skip_variants.TD_SKIP_VARIANTS.items():
        ck = torch.load(os.path.join(REF, "weights", base), map_location="cpu", weights_only=False)
        args, sd = td_skip_variants.td_skip_checkpoint(name, ck["args"], ck["model_state_dict"])
        with tempfile.TemporaryDirectory() as td:
            files = []
            for seed, sec, sr in TD_PAIR_CLIPS:
                fn = "v%03d.wav" % seed
                wav.write_wav_pcm16(os.path.join(td, fn), synth.synth_speech_pcm16(seed, sec, sr), sr)
                files.append(fn)
            pd.DataFrame({"deg": files}).to_csv(os.path.join(td, "files.csv"), index=False)
            ckpt_path = os.path.join(td, name + ".tar")
            torch.save({"args": args, "model_state_dict": sd}, ckpt_path)
            m = nisqaModel({"mode": "predict_csv", "pretrained_model": ckpt_path, "csv_file": "files.csv", "csv_deg": "deg",
                            "data_dir": td, "output_dir": None, "num_workers": 0, "bs": 4, "ms_channel": None,
                            "tr_bs_val": 4, "tr_num_workers": 0, "tr_device": "cpu"})
            df = m.predict()
            cols = [c for c in ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"] if c in df]
            out[name] = df[cols].to_numpy().astype(np.float64)
            print(name, out[name].tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "variants_td_skip.npz"), **out)


if __name__ == "__main__":
    main()
