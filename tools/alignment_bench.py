"""What reporting NISQA_DE's time alignment costs: the alignment call (nisqa_predict_device_batch_alignment,
de_align_kernel's alignment instances) against the plain call (nisqa_predict_device_batch) on the same pairs.  64 pairs of 10 s
clips at 48 kHz in HBM (the degraded clip: its reference delayed by 0.12 s, attenuated and noisy), for de_cosine_hard
(the shape of train_nisqa_double_ended.yaml) and de_dot_soft, the checkpoints the tests build from nisqa_mos_only.tar.

The two arms alternate, --rounds times each, every round --iters calls of the whole batch followed by one device
synchronise.  The arms are the engine calls into preallocated outputs (Scorer.align's host time columns wait for the
call, so they are not part of the timed loop).  Pairs/s per round (min / median / max) and the alignment call's extra
time as a share of the plain call's (from the medians).  Checks first that both arms give the same scores bit for bit.  --plain_only times the plain arm
alone and needs nothing the plain call does not, so that a copy of this file run from a checkout of an older commit
(its own package and library: that library lacks the alignment entry points, which this package binds) times that
build's plain call in the same session.  Prints the card's name and power limit, then one JSON line per checkpoint.

    python tools/alignment_bench.py [--pairs 64] [--seconds 10] [--iters 5] [--rounds 7] [--plain_only]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from device_batch_bench import card  # noqa: E402
from nisqa_b200 import engine as E  # noqa: E402
from nisqa_b200 import synth  # noqa: E402
from nisqa_b200.scorer import Scorer  # noqa: E402
from oracle import variants as V  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--plain_only", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sr, B = 48000, a.pairs
    T = int(a.seconds * sr)
    base = [synth.synth_speech_pcm16(300 + i, 6.01, sr)[:6 * sr] for i in range(8)]     # (tiled: synthesis is slow)
    rng = np.random.default_rng(0)
    ref = np.stack([np.resize(np.concatenate([base[j] for j in rng.permutation(8)]), T) for _ in range(B)])
    lag = int(0.12 * sr)
    deg = np.zeros_like(ref, dtype=np.float32)
    deg[:, lag:] = ref[:, :T - lag] * 0.7
    deg = np.clip(deg + rng.normal(0, 300, deg.shape), -32768, 32767).astype(np.int16)
    x, y = torch.from_numpy(deg).cuda(), torch.from_numpy(ref).cuda()
    bargs, bsd = E.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_mos_only.tar"))
    print("card: %s" % card())
    for name in ("de_cosine_hard", "de_dot_soft"):
        args, sd = V.de_checkpoint(name, bargs, bsd)
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, name + ".tar")
            torch.save({"args": args, "model_state_dict": sd}, path)
            sc = Scorer(path)
        # the engine calls themselves, into preallocated outputs (Scorer.align also copies ref_seg and centroid to the
        # host for its time columns, which waits for the call)
        deg, ref = sc._batch("wave", x, sr, None, None), sc._batch("reference", y, sr, None, None)
        stream = sc._stream()
        scores = torch.empty((2 * B, 1), device="cuda")
        arms = {"plain": lambda: sc.engine.predict_device_batch(stream, deg, scores.data_ptr(), ref=ref)}
        if not a.plain_only:
            res = sc.align(x, sr, y)
            al, al_rows = sc._alignment_buffers(int(sum(res.counts)))        # (al_rows: the arrays al points into)
            arms["alignment"] = lambda: sc.engine.predict_device_batch_alignment(stream, deg, ref, scores.data_ptr(), al)
            assert torch.equal(res.scores.view(torch.int32), sc(x, sr, reference=y).view(torch.int32))
            delay = float(np.median(res.delay_s[np.isfinite(res.delay_s)]))
        for f in arms.values():                                   # warm-up of every shape the rounds use
            f()
        torch.cuda.synchronize()
        rates = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    f()
                torch.cuda.synchronize()
                rates[k].append(a.iters * B / (time.perf_counter() - t0))
        out = {"checkpoint": name, "pairs": B, "seconds": a.seconds, "sample_rate": sr}
        for k, r in rates.items():
            out[k + "_pairs_per_s"] = {"min": min(r), "median": float(np.median(r)), "max": max(r)}
        if not a.plain_only:
            p, q = out["plain_pairs_per_s"]["median"], out["alignment_pairs_per_s"]["median"]
            out["alignment_extra_time_share"] = p / q - 1.0
            out["median_delay_s"] = delay
        print(json.dumps(out))
        sc.close()


if __name__ == "__main__":
    main()
