"""Time the time-dependency stages of every pairing oracle/td_pair_variants.py covers (StandardCNN + self-attention,
self-attention -> LSTM, LSTM -> self-attention, LSTM -> LSTM) on the bench's size: 64 x 10 s 48 kHz clips (247 segments
each), seeded weights.  Device times of the engine's scopes come from its CUDA-event timers (nisqa_set_profiling):
"lin_ln" (Linear + LayerNorm + QKV of layer 0 of each self-attention stack), "sa_layer" (its encoder layers), "fc_out"
(StandardCNN's fc_out), "lstm" (input projection + recurrence of every LSTM layer) and "pool".  Prints the card's name and
power limit, then one JSON line per variant (median over --reps calls).

    python tools/td_pair_bench.py [--reps 10]
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
from oracle import nisqa_oracle as O  # noqa: E402
from oracle import td_pair_variants as V  # noqa: E402

SCOPES = ("lin_ln", "sa_layer", "fc_out", "lstm", "pool")


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
    for name, (base, _, _) in V.TD_PAIR_VARIANTS.items():
        base_args, base_sd = O.load_checkpoint(os.path.join(ROOT, "weights", base))
        args, sd = V.td_pair_checkpoint(name, base_args, base_sd)
        eng = E.Engine(E.config_from_args(args), 0)
        try:
            eng.load_state_dict(sd)
            eng.set_profiling(True)
            ms = {g: [] for g in SCOPES}
            for r in range(a.reps + 3):
                _, nseg, status = eng.predict_pcm(pcm, srs)
                if r >= 3:
                    for g in SCOPES:
                        ms[g].append(eng.group_ms(g))
            assert (status == E.CLIP_OK).all()
        finally:
            eng.close()
        row = {"variant": name, "clips": a.clips, "segments": int(nseg.sum())}
        for g in SCOPES:
            v = float(np.median(ms[g]))
            row[g + "_ms"] = round(v, 4) if v >= 0 else None          # (None: the pairing has no such scope)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
