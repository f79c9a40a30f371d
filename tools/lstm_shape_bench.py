"""Time the StandardCNN + LSTM time-dependency block per LSTM shape: fc_out (group "fc_out"), the input projections and
recurrences of every layer (group "lstm") and the pooling module (group "pool") on 64 x 10 s 16 kHz clips (987 segments,
so 987 serial steps per layer), for td_lstm_h H in {32, 64, 96, 128, 192, 256}, one bidirectional layer, fc_out 100 and
PoolAvg - every one of them on the stacked path (tile-GEMM input projection + lstm_layer_kernel; H 192 / 256 on
clusters of 3 / 4 CTAs) - plus nisqa_tts.tar's own shape (fc_out 20: linear_rows_kernel<20> + lstm_batched_kernel).
Each line names the path it ran (the rule of pack_lstm_model in csrc/engine.cu).
nisqa_tts.tar's CNN with seeded LSTM and pooling weights (oracle/lstm_variants.py).  Device times come from the engine's
CUDA-event timers (nisqa_set_profiling).  Prints the card and its power limit, then one JSON line per configuration;
`step_us` is the "lstm" time divided by the serial steps.

    python tools/lstm_shape_bench.py [--reps 20] [--layers 1]
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
from oracle import lstm_variants as V  # noqa: E402
from oracle import nisqa_oracle as O  # noqa: E402


def card():
    """(name, power limit) of device 0, read with a query of nvidia-smi (nothing is changed)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


def path(args):
    """The LSTM path the engine selects for these args (pack_lstm_model): nisqa_tts.tar's shape keeps lstm_batched_kernel"""
    shipped = (args.get("cnn_fc_out_h") == 20 and args["td_lstm_h"] == 128 and args["td_lstm_num_layers"] == 1
               and bool(args["td_lstm_bidirectional"]) and args["model"] == "NISQA" and args["pool"] != "att")
    return "linear_rows_kernel<20> + lstm_batched_kernel" if shipped else "linear_tile_kernel + lstm_layer_kernel"


def time_groups(args, sd, pcm, srs, reps):
    eng = E.Engine(E.config_from_args(args), 0)
    try:
        eng.load_state_dict(sd)
        eng.set_profiling(True)
        ms = {"fc_out": [], "lstm": [], "pool": []}
        for r in range(reps + 3):
            _, nseg, status = eng.predict_pcm(pcm, srs)
            if r >= 3:
                for g in ms:
                    ms[g].append(eng.group_ms(g))
        assert (status == E.CLIP_OK).all()
    finally:
        eng.close()
    return {g: float(np.median(v)) for g, v in ms.items()}, nseg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--layers", type=int, default=1)
    a = ap.parse_args()
    name, limit = card()
    print(json.dumps({"card": name, "power_limit": limit}), flush=True)
    base_args, base_sd = O.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_tts.tar"))
    pcm = [synth.synth_speech_pcm16(1000 + i % 4, 10.0, 16000) for i in range(a.clips)]
    srs = [16000] * a.clips
    ms, nseg = time_groups(base_args, base_sd, pcm, srs, a.reps)
    steps = int(nseg.max())
    print(json.dumps({"shape": "nisqa_tts.tar (H 128, 1 layer, bidirectional, fc_out 20)", "path": path(base_args), "clips": a.clips,
                      "steps": steps, **{k + "_ms": round(v, 4) for k, v in ms.items()},
                      "step_us": round(ms["lstm"] * 1e3 / steps, 3)}), flush=True)
    for H in E.LSTM_H:
        over = {"td_lstm_h": H, "td_lstm_num_layers": a.layers, "td_lstm_bidirectional": True, "cnn_fc_out_h": 100,
                "pool": "avg"}
        args, sd = V.lstm_checkpoint("lstm_bench_h%d" % H, base_args, base_sd, over)
        assert path(args) == "linear_tile_kernel + lstm_layer_kernel"
        ms, nseg = time_groups(args, sd, pcm, srs, a.reps)
        print(json.dumps({"H": H, "layers": a.layers, "fc_out": 100, "path": path(args), "cluster": max(1, H // 64) if H > 128 else 1, "clips": a.clips,
                          "steps": steps, **{k + "_ms": round(v, 4) for k, v in ms.items()},
                          "step_us": round(ms["lstm"] * 1e3 / (steps * a.layers), 3)}), flush=True)


if __name__ == "__main__":
    main()
