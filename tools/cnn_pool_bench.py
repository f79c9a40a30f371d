"""Time AdaptCNN checkpoints trained with other adaptive max-pool sizes (cnn_pool_1 / cnn_pool_2 / cnn_pool_3) on the bench's
size: 64 x 10 s 48 kHz clips.  Device times of the engine's scopes come from its CUDA-event timers (nisqa_set_profiling):
"conv1" (the separate conv1 + pool1 kernel, or "conv12", the fused conv1 + conv2 kernel), "conv2_6" (conv2..conv6;
conv3..conv6 behind conv12) and "td" (the self-attention stack).  Every entry of oracle/cnn_pool_variants.py runs on its
seeded weights (NISQA_DE: the degraded and the reference clip of 32 pairs); "shipped" runs nisqa_mos_only.tar.
Prints the card's name and power limit, then one JSON line per entry (median over --reps calls).

    python tools/cnn_pool_bench.py [--reps 10] [--variants mos_p16x5_8x4_4x2 ...]
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
from oracle import cnn_pool_variants as V  # noqa: E402
from oracle import nisqa_oracle as O  # noqa: E402

GROUPS = {"conv1": ("conv1", "conv12"), "conv2_6": ("conv2", "conv3", "conv4", "conv5", "conv6"), "td": ("lin_ln", "sa_layer")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--variants", nargs="*", default=None, help="entries of CNN_POOL_VARIANTS (default: all, and 'shipped')")
    a = ap.parse_args()
    names = a.variants or ["shipped"] + list(V.CNN_POOL_VARIANTS)
    print(json.dumps({"card": card()}), flush=True)
    pcm = [synth.synth_speech_pcm16(1000 + i % 4, 10.0, 48000) for i in range(a.clips)]
    srs = [48000] * a.clips
    for name in names:
        if name == "shipped":
            args, sd = O.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_mos_only.tar"))
        else:
            base_args, base_sd = O.load_checkpoint(os.path.join(ROOT, "weights", V.CNN_POOL_VARIANTS[name][0]))
            args, sd = V.cnn_pool_checkpoint(name, base_args, base_sd)
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
                        ms[s].append(max(eng.group_ms(s), 0.0))       # (a negative time: the entry has no such scope)
            assert (status == E.CLIP_OK).all()
        finally:
            eng.close()
        pools = [list(args["cnn_pool_%d" % i]) for i in (1, 2, 3)]
        row = {"variant": name, "pools": pools, "n_mels": args["ms_n_mels"], "clips": a.clips, "segments": int(nseg.sum()),
               "fused_conv12": ms["conv12"][0] > 0}
        for g, members in GROUPS.items():
            t = float(np.median([sum(ms[s][i] for s in members) for i in range(a.reps)]))
            row[g + "_ms"] = round(t, 4) if t > 0 else None
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
