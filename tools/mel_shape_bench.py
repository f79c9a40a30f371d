"""Time checkpoints trained with other Mel-spectrogram segment shapes (ms_n_mels x ms_seg_length) on the bench's size:
64 x 10 s 48 kHz clips.  Device times of the engine's scopes come from its CUDA-event timers (nisqa_set_profiling):
"frontend" (PCM -> mel dB), "conv1" (the separate conv1 + adaptive pool1 kernel; "conv12" on the fused 48 x 15 path),
"conv2_6" (conv2..conv6), "framewise" (SkipCNN's / DFF's seg_feats + Linear layers, AdaptCNN's Linear), "td" (the
self-attention stack) and "pool".  The AdaptCNN shapes run nisqa_mos_only.tar's weights with ms_n_mels / ms_seg_length
switched (its weights do not depend on them); SkipCNN / DFF run seeded weights (oracle/mel_variants.py).  Prints the
card's name and power limit, then one JSON line per shape (median over --reps calls).

    python tools/mel_shape_bench.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nisqa_b200 import engine as E  # noqa: E402
from nisqa_b200 import synth  # noqa: E402
from oracle import mel_variants as V  # noqa: E402
from oracle import nisqa_oracle as O  # noqa: E402

GROUPS = {"frontend": ("frontend",), "conv1": ("conv1", "conv12"), "conv2_6": ("conv2", "conv3", "conv4", "conv5", "conv6"),
          "framewise": ("framewise",), "td": ("lin_ln", "sa_layer"), "pool": ("pool",)}
# label -> (base checkpoint, MEL_VARIANTS entry for seeded SkipCNN / DFF weights or None, args overrides)
SHAPES = {
    "adapt 48x15": ("nisqa_mos_only.tar", None, {}),
    "adapt 32x15": ("nisqa_mos_only.tar", None, dict(ms_n_mels=32)),
    "adapt 64x15": ("nisqa_mos_only.tar", None, dict(ms_n_mels=64)),
    "adapt 128x21": ("nisqa_mos_only.tar", None, dict(ms_n_mels=128, ms_seg_length=21)),
    "adapt 48x31": ("nisqa_mos_only.tar", None, dict(ms_seg_length=31)),
    "skipcnn fc256 96x31": ("nisqa.tar", "dim_skipcnn_fc256_m96_s31", {}),
    "dff 64x9": ("nisqa_mos_only.tar", "mos_dff_m64_s9", {}),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--clips", type=int, default=64)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    pcm = [synth.synth_speech_pcm16(1000 + i % 4, 10.0, 48000) for i in range(a.clips)]
    srs = [48000] * a.clips
    for label, (base, variant, over) in SHAPES.items():
        args, sd = O.load_checkpoint(os.path.join(ROOT, "weights", base))
        if variant:
            args, sd = V.mel_checkpoint(variant, args, sd)
        args = dict(args, **over)
        eng = E.Engine(E.config_from_args(args), 0)
        scopes = [s for g in GROUPS.values() for s in g]
        try:
            eng.load_state_dict(sd)
            eng.set_profiling(True)
            ms = {s: [] for s in scopes}
            for r in range(a.reps + 3):
                _, nseg, status = eng.predict_pcm(pcm, srs)
                if r >= 3:
                    for s in scopes:
                        ms[s].append(max(eng.group_ms(s), 0.0))       # (a negative time: the variant has no such scope)
            assert (status == E.CLIP_OK).all()
        finally:
            eng.close()
        row = {"shape": label, "model": args["model"], "seg_hop": args["ms_seg_hop_length"], "clips": a.clips,
               "segments": int(nseg.sum())}
        for g, members in GROUPS.items():
            t = float(np.median([sum(ms[s][i] for s in members) for i in range(a.reps)]))
            row[g + "_ms"] = round(t, 4) if t > 0 else None
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
