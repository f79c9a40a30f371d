"""Time the checkpoints without a time-dependency model (td = 'skip', oracle/td_skip_variants.py) on the bench's size:
64 x 10 s 48 kHz clips, seeded weights.  Device times of the engine's scopes come from its CUDA-event timers
(nisqa_set_profiling): "framewise" is the framewise model after the front end (conv1..conv6, StandardCNN's fc_out,
AdaptCNN's / SkipCNN's / DFF's Linear layers), "pool" the pooling module (with PoolAttFF's hidden GEMM and logits, or
PoolAtt's logits, when the rows go straight to it) and "td2" a td_2 stage when one runs.  For the pool scope of the
variants without td_2 it also prints the bytes of framewise rows pooled (n_seg x D x 4, each read once by
pool_wide_kernel) and those bytes over the scope's time.  Prints the card's name and power limit, then one JSON line
per variant (median over --reps calls).

    python tools/td_skip_bench.py [--reps 10]
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
from oracle import td_skip_variants as V  # noqa: E402

FRAMEWISE = ("conv12", "conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "fc_out", "framewise")
TD2 = ("lin_ln", "sa_layer", "lstm")


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
    for name, (base, _, _) in V.TD_SKIP_VARIANTS.items():
        base_args, base_sd = O.load_checkpoint(os.path.join(ROOT, "weights", base))
        args, sd = V.td_skip_checkpoint(name, base_args, base_sd)
        eng = E.Engine(E.config_from_args(args), 0)
        groups = FRAMEWISE + TD2 + ("pool",)
        try:
            eng.load_state_dict(sd)
            eng.set_profiling(True)
            ms = {g: [] for g in groups}
            for r in range(a.reps + 3):
                _, nseg, status = eng.predict_pcm(pcm, srs)
                if r >= 3:
                    for g in groups:
                        ms[g].append(max(eng.group_ms(g), 0.0))       # (a negative time: the variant has no such scope)
            assert (status == E.CLIP_OK).all()
        finally:
            eng.close()
        n_seg = int(nseg.sum())
        fw = float(np.median([sum(ms[g][i] for g in FRAMEWISE) for i in range(a.reps)]))
        td2 = float(np.median([sum(ms[g][i] for g in TD2) for i in range(a.reps)]))
        pool = float(np.median(ms["pool"]))
        row = {"variant": name, "clips": a.clips, "segments": n_seg, "pool_module": args["pool"],
               "framewise_ms": round(fw, 4), "td2_ms": round(td2, 4) if td2 > 0 else None, "pool_ms": round(pool, 4)}
        if args.get("td_2") == "skip":
            nbytes = n_seg * V.pooled_width(args) * 4
            row["pooled_bytes"] = nbytes
            row["pool_GB_per_s"] = round(nbytes / (pool * 1e-3) / 1e9, 1) if pool > 0 else None
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
