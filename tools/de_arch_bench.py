"""Throughput of double-ended (NISQA_DE) models: the shipped shape (AdaptCNN + 64-wide self-attention,
oracle/variants.py de_cosine_hard) next to StandardCNN -> BiLSTM128 (alignment and fusion at W = 256) and StandardCNN ->
BiLSTM256 (W = 512) from oracle/de_arch_variants.py, seeded weights.  Batches of --pairs (degraded, reference) pairs of
10 s 48 kHz clips (494 segments per pair at the shipped shape's segment hop of 4, 1974 at nisqa_tts.tar's hop of 1).
pairs/s: host clock around synchronous predict_pcm calls (median over --reps after 3 warm-up calls), profiling off;
de_align_ms: the engine's CUDA-event timer of its "de_align" scope (the projections / norms, de_align_kernel and
lin_fusion) in separate profiled calls.  Prints the card's name and power limit, then one JSON line per variant.

    python tools/de_arch_bench.py [--reps 10] [--pairs 64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nisqa_b200 import engine as E  # noqa: E402
from nisqa_b200 import synth  # noqa: E402
from oracle import de_arch_variants as DV  # noqa: E402
from oracle import nisqa_oracle as O  # noqa: E402
from oracle import variants as V  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def checkpoints():
    bargs, bsd = O.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_mos_only.tar"))
    yield "shipped_adapt_sa64_cosine_hard", V.de_checkpoint("de_cosine_hard", bargs, bsd)
    targs, tsd = O.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_tts.tar"))
    for name in ("std_fc20_lstm128bi_luong_soft_fd128", "std_fc20_lstm256bi_l2_dot_soft"):
        yield name, DV.de_arch_checkpoint(name, targs, tsd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--pairs", type=int, default=64)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    clips = []
    for i in range(a.pairs):
        clips += [synth.synth_speech_pcm16(1000 + i % 4, 10.0, 48000), synth.synth_speech_pcm16(2000 + i % 3, 10.0, 48000)]
    srs = [48000] * len(clips)
    for name, (args, sd) in checkpoints():
        eng = E.Engine(E.config_from_args(args), 0)
        try:
            eng.load_state_dict(sd)
            secs = []
            for r in range(a.reps + 3):
                t0 = time.perf_counter()
                _, nseg, status = eng.predict_pcm(clips, srs)
                if r >= 3:
                    secs.append(time.perf_counter() - t0)
            assert (status == E.CLIP_OK).all()
            eng.set_profiling(True)
            ms = []
            for _ in range(3):
                eng.predict_pcm(clips, srs)
                ms.append(eng.group_ms("de_align"))
        finally:
            eng.close()
        print(json.dumps({"variant": name, "pairs": a.pairs, "segments": int(nseg.sum()),
                          "pairs_per_s": round(a.pairs / float(np.median(secs)), 1),
                          "de_align_ms": round(float(np.median(ms)), 4)}), flush=True)


if __name__ == "__main__":
    main()
