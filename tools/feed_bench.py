"""What scoring live feeds costs: Scorer.feed (nisqa_feed_push: each chunk appended to its feed's device ring, each
interior mel frame pair computed once as its samples arrive, each window scored as it completes) against the two ways a
caller had before.  256 feeds of 20 s at 48 kHz in HBM, nisqa.tar, 10 s windows at 1 s and 0.1 s hops, pushes of 0.1 s
and 1 s.

  feed         : the recordings pushed chunk by chunk.  The first 10 s (no window completes before) run untimed; the
                 rest is timed: windows/s over all those pushes (one device synchronise at the end), and the device time
                 per push (CUDA events on the caller's stream, the interval between consecutive pushes' ends)
  per_window   : the same windows scored as they complete by Scorer.__call__ from a sample buffer (a view of the
                 recording), one call per window index completed by a push (all feeds' windows of that index)
  windows      : Scorer.windows on the finished recordings (one call, every window of the 20 s)

Windows/s of each arm (min / median / max over --rounds alternating rounds), then one profiled round of each gives the
"frontend" and "ingest" kernel-group times (CUDA events on the engine's lanes; profiled calls run on one lane and
synchronise).  Checks first that the feed's rows equal Scorer.windows bit for bit.  Prints the card's name and power
limit, then one JSON line per (hop, push).

    python tools/feed_bench.py [--feeds 256] [--seconds 20] [--rounds 5]
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
    ap.add_argument("--feeds", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--window_s", type=float, default=10.0)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sr, B = 48000, a.feeds
    T = int(a.seconds * sr)
    W = int(round(a.window_s * sr))
    base = [synth.synth_speech_pcm16(300 + i, 6.01, sr)[:6 * sr] for i in range(8)]     # (tiled: synthesis is slow)
    rng = np.random.default_rng(0)
    x = np.stack([np.resize(np.concatenate([base[j] for j in rng.permutation(8)]), T) for _ in range(B)])
    x = torch.from_numpy(x).cuda()
    sc = Scorer(os.path.join(ROOT, "weights", "nisqa.tar"))
    eng = sc.engine
    print("card: %s" % card())
    for hop_s in (1.0, 0.1):
        H = int(round(hop_s * 100)) * 480
        for push_s in (0.1, 1.0):
            c = int(round(push_s * sr))
            warm = W // c * c                   # pushes before the first window completes run untimed
            n_timed = (T - warm) // c
            K = 1 + (T - W) // H                # T - W is a multiple of H: every window is whole

            def feed(profile_ms=None):
                fd = sc.feed(B, sr, a.window_s, hop_s, max_push_s=push_s)
                rows = []
                for t in range(0, warm, c):
                    rows.append(fd.push(x[:, t:t + c]).scores)
                torch.cuda.synchronize()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(n_timed + 1)]
                ev[0].record()
                t0 = time.perf_counter()
                for i in range(n_timed):
                    t = warm + i * c
                    end = [True] * B if t + c >= T else None
                    rows.append(fd.push(x[:, t:t + c], end=end).scores)
                    ev[i + 1].record()
                    if profile_ms is not None:
                        for g in profile_ms:
                            profile_ms[g] += max(0.0, eng.group_ms(g))
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                fd.close()
                per_push = [ev[i].elapsed_time(ev[i + 1]) for i in range(n_timed)]
                return torch.cat(rows), dt, per_push

            # the window indices each push completes (every feed alike): window k once t < k H + W <= t + c
            emitted = [[k for k in range(K) if t < k * H + W <= t + c] for t in range(0, warm + n_timed * c, c)]
            starts = emitted[warm // c:]

            def per_window(profile_ms=None):
                out = []
                for ks in starts:
                    for k in ks:
                        out.append(sc(x[:, k * H:k * H + W], sr))
                        if profile_ms is not None:
                            for g in profile_ms:
                                profile_ms[g] += max(0.0, eng.group_ms(g))
                return out

            def windows(profile_ms=None):
                r = sc.windows(x, sr, a.window_s, hop_s).scores
                if profile_ms is not None:
                    for g in profile_ms:
                        profile_ms[g] += max(0.0, eng.group_ms(g))
                return r

            got, _, _ = feed()
            want = windows().view(B, K, -1)
            # the feed's rows come push by push, by feed then window: their places in recording order
            order = torch.tensor([b * K + k for ks in emitted for b in range(B) for k in ks])
            assert got.shape[0] == order.shape[0] == B * K
            inv = torch.empty(B * K, dtype=torch.long)
            inv[order] = torch.arange(B * K)
            assert torch.equal(got[inv.cuda()].view(B, K, -1), want), "feed rows differ from Scorer.windows"
            rates = {"feed": [], "per_window": [], "windows": []}
            per_push_ms = []
            n_timed_windows = B * sum(len(ks) for ks in starts)
            for _ in range(a.rounds):
                _, dt, pp = feed()
                rates["feed"].append(n_timed_windows / dt)
                per_push_ms += pp
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                per_window()
                torch.cuda.synchronize()
                rates["per_window"].append(n_timed_windows / (time.perf_counter() - t0))
                t0 = time.perf_counter()
                windows()
                torch.cuda.synchronize()
                rates["windows"].append(B * K / (time.perf_counter() - t0))
            res = {k: {"min": min(v), "median": float(np.median(v)), "max": max(v)} for k, v in rates.items()}
            res["per_push_device_ms"] = {"min": min(per_push_ms), "median": float(np.median(per_push_ms)),
                                         "max": max(per_push_ms)}
            scopes = {}
            eng.set_profiling(True)
            for k, f in (("feed", feed), ("per_window", per_window), ("windows", windows)):
                ms = {"frontend": 0.0, "ingest": 0.0}
                f(profile_ms=ms)
                scopes[k] = {g + "_ms": v for g, v in ms.items()}
            eng.set_profiling(False)
            print(json.dumps({"checkpoint": "nisqa.tar", "feeds": B, "seconds": a.seconds, "window_s": a.window_s,
                              "window_hop_s": hop_s, "push_s": push_s, "timed_pushes": n_timed,
                              "timed_windows": n_timed_windows, "windows_per_recording": K, "unit": "windows/s", **res,
                              "scopes": scopes,
                              "scopes_note": "feed / per_window: the timed pushes; windows: the whole recordings"}),
                  flush=True)
    sc.close()


if __name__ == "__main__":
    main()
