"""Generate tests/golden/*.npz from the UNMODIFIED reference (runs only in the build container).

    python -m oracle.make_golden            # needs the reference checkout ($NISQA_REFERENCE_DIR, read-only)

The reference package is imported as-is from $NISQA_REFERENCE_DIR with ``librosa`` replaced by
``oracle/librosa_compat.py`` (real librosa 0.8.1 is not installable offline - the front-end
half therefore stays "parity unpinned") and a ``matplotlib.pyplot`` stub.  Everything
downstream of the mel-dB tensor - ``segment_specs``, ``SpeechQualityDataset``, the
``NISQA``/``NISQA_DIM`` torch modules, ``predict_mos``/``predict_dim`` and
``nisqaModel.predict()`` - is the reference's own code, and its outputs are what the golden
files hold.  Inputs are regenerated from seeds by ``nisqa_b200/synth.py`` so the fixtures stay
small.
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

from oracle import librosa_compat  # noqa: E402
from nisqa_b200 import synth, wav  # noqa: E402

# (name, checkpoint, [(seed, seconds, sr)], keep_mel)
CASES = [
    ("nisqa_48k_3s", "nisqa.tar", [(1, 3.0, 48000)], True),
    ("nisqa_mixed", "nisqa.tar", [(2, 1.37, 48000), (3, 2.0, 16000), (4, 2.5, 44100),
                                  (5, 0.1875, 8000), (6, 1.0, 22050), (7, 4.21, 48000)], True),
    ("nisqa_48k_10s", "nisqa.tar", [(0, 10.0, 48000)], False),
    ("mos_only_48k", "nisqa_mos_only.tar", [(8, 2.2, 48000), (9, 1.0, 32000)], False),
    ("tts_16k", "nisqa_tts.tar", [(10, 2.0, 16000), (11, 1.3, 48000), (12, 0.9, 22050)], True),
]


def _import_reference():
    librosa_compat.install()
    sys.path.insert(0, REF)
    from nisqa.NISQA_model import nisqaModel  # noqa
    import nisqa.NISQA_lib as NL  # noqa
    return nisqaModel, NL


def main():
    nisqaModel, NL = _import_reference()
    torch.manual_seed(0)
    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    for name, ckpt, clips, keep_mel in CASES:
        with tempfile.TemporaryDirectory() as td:
            files = []
            for (seed, seconds, sr) in clips:
                pcm = synth.synth_speech_pcm16(seed, seconds, sr)
                fn = "c%03d.wav" % seed
                wav.write_wav_pcm16(os.path.join(td, fn), pcm, sr)
                files.append(fn)
            import pandas as pd
            pd.DataFrame({"deg": files}).to_csv(os.path.join(td, "files.csv"), index=False)
            args = {"mode": "predict_csv", "pretrained_model": os.path.join(REF, "weights", ckpt),
                    "csv_file": "files.csv", "csv_deg": "deg", "data_dir": td, "output_dir": None,
                    "num_workers": 0, "bs": 4, "ms_channel": None, "tr_bs_val": 4,
                    "tr_num_workers": 0, "tr_device": "cpu"}
            m = nisqaModel(args)
            taps = {}

            def hook_cnn(mod, inp, out):
                taps["cnn"] = out.detach().clone()

            def hook_td(mod, inp, out):
                taps["td"] = out[0].detach().clone()

            h1 = m.model.cnn.register_forward_hook(hook_cnn)
            h2 = m.model.time_dependency.register_forward_hook(hook_td)
            df = m.predict()
            h1.remove(); h2.remove()
            cols = [c for c in ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"] if c in df]
            scores = df[cols].to_numpy().astype(np.float64)
            save = {"scores": scores, "seeds": np.array([c[0] for c in clips]),
                    "seconds": np.array([c[1] for c in clips]), "sr": np.array([c[2] for c in clips])}
            n_wins = []
            for i in range(len(clips)):
                x, y, (idx, nw) = m.ds_val[i]
                n_wins.append(int(nw))
                if keep_mel:
                    spec = m.ds_val._load_spec(i)
                    save["mel_%d" % i] = np.asarray(spec, dtype=np.float32)
            save["n_segments"] = np.array(n_wins, dtype=np.int64)
            # per-clip module outputs from the single batch the reference ran (bs=4 >= #clips
            # except the 6-clip case, where the hooks hold the LAST batch -> rerun with bs=8)
            if len(clips) > 4:
                args2 = dict(args); args2["bs"] = 8; args2["tr_bs_val"] = 8
                m2 = nisqaModel(args2)
                h1 = m2.model.cnn.register_forward_hook(hook_cnn)
                h2 = m2.model.time_dependency.register_forward_hook(hook_td)
                df2 = m2.predict()
                h1.remove(); h2.remove()
                save["scores_bs8"] = df2[cols].to_numpy().astype(np.float64)
            for i, nw in enumerate(n_wins):
                save["cnn_%d" % i] = taps["cnn"][i, :nw].numpy().astype(np.float32)
                save["td_%d" % i] = taps["td"][i, :nw].numpy().astype(np.float32)
            np.savez_compressed(os.path.join(out_dir, name + ".npz"), **save)
            print(name, "->", scores.tolist(), n_wins)


if __name__ == "__main__":
    main()
