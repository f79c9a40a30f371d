"""What scoring windows of recordings costs: Scorer.windows (nisqa_predict_device_windows: each recording span packed
once, each interior mel frame pair computed once) against Scorer.__call__ on the same windows cut out as clips (the
overlapping `unfold` view of each recording, one call per recording, so every window's PCM is packed and its mel frames
computed again), and against one Scorer.__call__ on a contiguous copy of all those windows (the same work in one call).  64 recordings of 60 s at 48 kHz in HBM, nisqa.tar, 10 s windows at 5 s and 1 s hops.

The two arms alternate, --rounds times each, every round --iters calls of each arm's whole batch followed by one device
synchronise; windows/s per round (min / median / max).  Then one profiled round of each arm gives the "frontend" and
"ingest" kernel-group times (CUDA events on the engine's lanes; the profiled calls run on one lane).  Checks first that
both arms give the same scores bit for bit.  Prints the card's name and power limit, then one JSON line per hop.

    python tools/window_bench.py [--recordings 64] [--seconds 60] [--iters 3] [--rounds 7]
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
    ap.add_argument("--recordings", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--window_s", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sr, B = 48000, a.recordings
    T = int(a.seconds * sr)
    base = [synth.synth_speech_pcm16(300 + i, 6.01, sr)[:6 * sr] for i in range(8)]     # (tiled: synthesis is slow)
    rng = np.random.default_rng(0)
    x = np.stack([np.resize(np.concatenate([base[j] for j in rng.permutation(8)]), T) for _ in range(B)])
    x = torch.from_numpy(x).cuda()
    sc = Scorer(os.path.join(ROOT, "weights", "nisqa.tar"))
    W = int(round(a.window_s * sr))
    print("card: %s" % card())
    for hop_s in (5.0, 1.0):
        H = int(round(hop_s * 100)) * 480
        views = [x[b].unfold(-1, W, H) for b in range(B)]           # T - W is a multiple of H: every window is whole
        K = views[0].shape[0]

        def windows():
            return sc.windows(x, sr, a.window_s, hop_s).scores

        def cut():
            return [sc(v, sr) for v in views]

        flat = torch.cat(views)                                        # (a copy: the windows as B K contiguous clips)

        def cut_one_call():
            return sc(flat, sr)

        got, want = windows(), torch.cat(cut())
        torch.cuda.synchronize()
        assert torch.equal(got, want), "windows differ from the cut clips"
        assert torch.equal(got, cut_one_call())
        arms = {"windows": windows, "cut_clips": cut, "cut_clips_one_call": cut_one_call}
        rates = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                f()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    f()
                torch.cuda.synchronize()
                rates[k].append(B * K * a.iters / (time.perf_counter() - t0))
        res = {k: {"min": min(v), "median": float(np.median(v)), "max": max(v)} for k, v in rates.items()}
        res["median_saving_pct"] = 100.0 * (1.0 - res["cut_clips"]["median"] / res["windows"]["median"])
        res["median_saving_vs_one_call_pct"] = 100.0 * (1.0 - res["cut_clips_one_call"]["median"] / res["windows"]["median"])
        scopes = {}
        sc.engine.set_profiling(True)
        for k, f in arms.items():
            ms = {"frontend": 0.0, "ingest": 0.0}
            if k != "cut_clips":
                f()
                ms = {g: max(0.0, sc.engine.group_ms(g)) for g in ms}
            else:
                for v in views:                 # (each call's timers are its own: summed over the batch)
                    sc(v, sr)
                    for g in ms:
                        ms[g] += max(0.0, sc.engine.group_ms(g))
            scopes[k] = {g + "_ms": v for g, v in ms.items()}
        sc.engine.set_profiling(False)
        print(json.dumps({"checkpoint": "nisqa.tar", "recordings": B, "seconds": a.seconds, "window_s": a.window_s,
                          "window_hop_s": hop_s, "windows_per_recording": K, "unit": "windows/s", **res,
                          "scopes_per_batch": scopes}))
    sc.close()


if __name__ == "__main__":
    main()
