"""Time the self-attention kernels per width: td_in (Linear + LayerNorm + QKV of layer 0, group "lin_ln") and the two
encoder layers (group "sa_layer") on 64 x 10 s 48 kHz clips (247 segments each), for d_model D in {64, 128, 192, 256} x
feed-forward width F in {64, 4D}, nisqa.tar's CNN and seeded self-attention / PoolAttFF weights (oracle/wide_variants.py).
Device times come from the engine's CUDA-event timers (nisqa_set_profiling).  Prints one JSON line per configuration.

    python tools/td_width_bench.py [--reps 20]

FLOPs are counted from the shapes, per row (segment) of a clip with S segments:
    Linear 384 -> D: 2 384 D;  per layer: QKV 6 D^2, out_proj 2 D^2, FFN 4 D F, q k^T + P V 4 S D;  PoolAttFF logits:
    5 heads x 2 128 D
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nisqa_b200 import engine as E  # noqa: E402
from nisqa_b200 import synth  # noqa: E402
from oracle import nisqa_oracle as O  # noqa: E402
from oracle import wide_variants as V  # noqa: E402


def flops(D, F, layers, seg_counts, heads=5):
    S = np.asarray(seg_counts, dtype=np.float64)
    per_row = 2 * 384 * D + layers * (6 * D * D + 2 * D * D + 4 * D * F) + heads * 2 * 128 * D
    return float((S * per_row + layers * 4 * S * S * D).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--clips", type=int, default=64)
    a = ap.parse_args()
    base_args, base_sd = O.load_checkpoint(os.path.join(ROOT, "weights", "nisqa.tar"))
    pcm = [synth.synth_speech_pcm16(1000 + i % 4, 10.0, 48000) for i in range(a.clips)]
    srs = [48000] * a.clips
    for D in (64, 128, 192, 256):
        for F in (64, 4 * D):
            args, sd = V.wide_checkpoint("td_width_d%d_ff%d" % (D, F), base_args, base_sd, ("nisqa.tar", None, {"td_sa_d_model": D, "td_sa_h": F}))
            eng = E.Engine(E.config_from_args(args), 0)
            try:
                eng.load_state_dict(sd)
                eng.set_profiling(True)
                ms = {"lin_ln": [], "sa_layer": []}
                for r in range(a.reps + 3):
                    _, nseg, status = eng.predict_pcm(pcm, srs)
                    if r >= 3:
                        for g in ms:
                            ms[g].append(eng.group_ms(g))
                assert (status == E.CLIP_OK).all()
            finally:
                eng.close()
            lin, sa = float(np.median(ms["lin_ln"])), float(np.median(ms["sa_layer"]))
            fl = flops(D, F, args["td_sa_num_layers"], nseg)
            print(json.dumps({"d_model": D, "ff": F, "clips": a.clips, "segments": int(nseg.sum()),
                              "lin_ln_ms": round(lin, 4), "sa_layer_ms": round(sa, 4), "td_ms": round(lin + sa, 4),
                              "gflop": round(fl / 1e9, 3), "tflops": round(fl / ((lin + sa) * 1e-3) / 1e12, 2)}), flush=True)


if __name__ == "__main__":
    main()
