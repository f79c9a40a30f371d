"""What the quality embeddings cost: Scorer.embed (nisqa_predict_device_batch_embeddings), with and without the
per-segment rows, against Scorer.__call__ (nisqa_predict_device_batch) on the same batch resident in HBM, 64 x 10 s clips
at 48 kHz, for nisqa.tar and nisqa_tts.tar (the shipped BiLSTM then also stores its per-step outputs, which the
embeddings kernel reads).

The three calls alternate, --rounds times each, every round --iters calls followed by one device synchronise; clips/s
per round (min / median / max).  Checks first that every call gives the same clip scores bit for bit.  Prints the card's
name and power limit, then one JSON line per checkpoint.

    python tools/embed_bench.py [--clips 64] [--seconds 10] [--iters 30] [--rounds 7]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from device_batch_bench import card  # noqa: E402
from nisqa_b200 import synth  # noqa: E402
from nisqa_b200.scorer import Scorer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sr, B = 48000, a.clips
    T = int(a.seconds * sr)
    x = torch.from_numpy(np.stack([synth.synth_speech_pcm16(100 + i, T / sr + 0.01, sr)[:T] for i in range(B)])).cuda()
    print("card: %s" % card())
    for ckpt in ("nisqa.tar", "nisqa_tts.tar"):
        sc = Scorer(os.path.join(ROOT, "weights", ckpt))
        plain = sc(x, sr)
        emb = sc.embed(x, sr, rows=True)
        pooled_only = sc.embed(x, sr)
        torch.cuda.synchronize()
        assert torch.equal(plain, emb.scores) and torch.equal(plain, pooled_only.scores), "embed changed the clip scores"
        arms = {"plain": lambda: sc(x, sr), "embed": lambda: sc.embed(x, sr), "embed_rows": lambda: sc.embed(x, sr, rows=True)}
        rates = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                f()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    f()
                torch.cuda.synchronize()
                rates[k].append(B * a.iters / (time.perf_counter() - t0))
        res = {k: {"min": min(v), "median": float(np.median(v)), "max": max(v)} for k, v in rates.items()}
        res["width"] = int(emb.rows.shape[1])
        res["segments_per_call"] = int(sum(emb.counts))
        res["row_bytes_per_call"] = int(emb.rows.numel() * 4)
        for k in ("embed", "embed_rows"):
            res[k + "_median_overhead_pct"] = 100.0 * (res["plain"]["median"] / res[k]["median"] - 1.0)
        print(json.dumps({"checkpoint": ckpt, "clips": B, "seconds": a.seconds, "unit": "clips/s", **res}))
        sc.close()


if __name__ == "__main__":
    main()
