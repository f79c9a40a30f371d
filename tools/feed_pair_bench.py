"""What scoring live double-ended (NISQA_DE) feeds costs: Scorer.feed(..., reference=True) (nisqa_feed_pair_push: each
side's chunk appended to its device ring, each interior mel frame pair of either side computed once as its samples
arrive, each window pair scored as both its windows complete) against the two ways a caller had before.  64 to 256 pair
feeds of 20 s at 48 kHz in HBM, de_cosine_hard (oracle/variants.py, from the shipped weights), 10 s windows at 1 s and
0.1 s hops, pushes of 0.1 s and 1 s, reference margins of 0 and 0.5 s.

  feed      : both recordings pushed chunk by chunk, side by side.  The pushes before the first pair completes run
              untimed; the rest is timed: pairs/s over all those pushes (one device synchronise at the end), and the
              device time per push (CUDA events on the caller's stream, the interval between consecutive pushes' ends)
  per_pair  : the same pairs scored as they complete by Scorer.__call__ on views of both recordings, one call per pair
              index completed by a push (all feeds' pairs of that index)
  windows   : Scorer.windows(..., reference=) on the finished recordings (one call, every pair of the 20 s)

Pairs/s of each arm (min / median / max over --rounds alternating rounds), then one profiled round of each gives the
"frontend" and "ingest" kernel-group times.  Checks first that the three arms agree bit for bit.  Prints the card's name
and power limit, then one JSON line per (hop, push, margin).

    python tools/feed_pair_bench.py [--feeds 256] [--seconds 20] [--rounds 5]
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
from nisqa_b200 import engine as E, synth  # noqa: E402
from nisqa_b200.scorer import Scorer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--feeds", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--window_s", type=float, default=10.0)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--hops", default="1.0,0.1")
    ap.add_argument("--pushes", default="0.1,1.0")
    ap.add_argument("--margins", default="0.0,0.5")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from oracle import variants as V
    bargs, bsd = E.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_mos_only.tar"))
    args, sd = V.de_checkpoint("de_cosine_hard", bargs, bsd)
    path = os.path.join(tempfile.mkdtemp(), "de_cosine_hard.tar")
    torch.save({"args": args, "model_state_dict": sd}, path)
    sr, B = 48000, a.feeds
    T = int(a.seconds * sr)
    W = int(round(a.window_s * sr))
    base = [synth.synth_speech_pcm16(300 + i, 6.01, sr)[:6 * sr] for i in range(8)]     # (tiled: synthesis is slow)
    rng = np.random.default_rng(0)
    y = np.stack([np.resize(np.concatenate([base[j] for j in rng.permutation(8)]), T) for _ in range(B)])
    lag = int(0.12 * sr)                      # the degraded side: the reference delayed, attenuated and noisy
    x = np.zeros_like(y, dtype=np.float32)
    x[:, lag:] = y[:, :T - lag] * 0.7
    x += rng.normal(0, 300, x.shape).astype(np.float32)
    x = torch.from_numpy(np.clip(x, -32768, 32767).astype(np.int16)).cuda()
    y = torch.from_numpy(y).cuda()
    sc = Scorer(path)
    eng = sc.engine
    print("card: %s" % card())
    for hop_s in (float(v) for v in a.hops.split(",")):
        H = int(round(hop_s * 100)) * 480
        for push_s in (float(v) for v in a.pushes.split(",")):
            c = int(round(push_s * sr))
            for margin_s in (float(v) for v in a.margins.split(",")):
                M = int(round(margin_s * 100)) * 480
                warm = (W + M) // c * c                 # pushes before the first pair completes run untimed
                n_push = -(-T // c)
                n_timed = n_push - warm // c
                K = 1 + (T - W) // H                    # T - W is a multiple of H: every degraded window is whole
                # the pair indices each push completes (every feed alike): pair k once k H + W + M <= t + c, the rest
                # with the ending push
                emitted = [[k for k in range(K) if t < k * H + W + M <= t + c or (t + c >= T and k * H + W + M > t + c)]
                           for t in range(0, n_push * c, c)]
                starts = emitted[warm // c:]

                def feed(profile_ms=None):
                    fd = sc.feed(B, sr, a.window_s, hop_s, max_push_s=push_s, reference=True, reference_margin_s=margin_s)
                    rows = []
                    for t in range(0, warm, c):
                        rows.append(fd.push(x[:, t:t + c], y[:, t:t + c]).scores)
                    torch.cuda.synchronize()
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n_timed + 1)]
                    ev[0].record()
                    t0 = time.perf_counter()
                    for i in range(n_timed):
                        t = warm + i * c
                        end = [True] * B if t + c >= T else None
                        rows.append(fd.push(x[:, t:t + c], y[:, t:t + c], end=end).scores)
                        ev[i + 1].record()
                        if profile_ms is not None:
                            for g in profile_ms:
                                profile_ms[g] += max(0.0, eng.group_ms(g))
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    fd.close()
                    return torch.cat(rows), dt, [ev[i].elapsed_time(ev[i + 1]) for i in range(n_timed)]

                def per_pair(profile_ms=None):
                    out = []
                    for ks in starts:
                        for k in ks:
                            r0, r1 = max(0, k * H - M), min(T, k * H + W + M)
                            out.append(sc(x[:, k * H:k * H + W], sr, reference=y[:, r0:r1]))
                            if profile_ms is not None:
                                for g in profile_ms:
                                    profile_ms[g] += max(0.0, eng.group_ms(g))
                    return out

                def windows(profile_ms=None):
                    r = sc.windows(x, sr, a.window_s, hop_s, reference=y, reference_margin_s=margin_s).scores
                    if profile_ms is not None:
                        for g in profile_ms:
                            profile_ms[g] += max(0.0, eng.group_ms(g))
                    return r

                got, _, _ = feed()
                want = windows().view(B, K, -1)
                order = torch.tensor([b * K + k for ks in emitted for b in range(B) for k in ks])
                assert got.shape[0] == order.shape[0] == B * K
                inv = torch.empty(B * K, dtype=torch.long)
                inv[order] = torch.arange(B * K)
                assert torch.equal(got[inv.cuda()].view(B, K, -1), want), "pair feed rows differ from Scorer.windows"
                pp = per_pair()
                n0 = sum(len(ks) for ks in emitted[:warm // c])
                for i, k in enumerate(k for ks in starts for k in ks):
                    assert torch.equal(pp[i], want[:, k]), "per-pair calls differ from Scorer.windows"
                assert n0 + len(pp) == K
                rates = {"feed": [], "per_pair": [], "windows": []}
                per_push_ms = []
                n_timed_pairs = B * sum(len(ks) for ks in starts)
                for _ in range(a.rounds):
                    _, dt, pms = feed()
                    rates["feed"].append(n_timed_pairs / dt)
                    per_push_ms += pms
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    per_pair()
                    torch.cuda.synchronize()
                    rates["per_pair"].append(n_timed_pairs / (time.perf_counter() - t0))
                    t0 = time.perf_counter()
                    windows()
                    torch.cuda.synchronize()
                    rates["windows"].append(B * K / (time.perf_counter() - t0))
                res = {k: {"min": min(v), "median": float(np.median(v)), "max": max(v)} for k, v in rates.items()}
                res["per_push_device_ms"] = {"min": min(per_push_ms), "median": float(np.median(per_push_ms)),
                                             "max": max(per_push_ms)}
                scopes = {}
                eng.set_profiling(True)
                for k, f in (("feed", feed), ("per_pair", per_pair), ("windows", windows)):
                    ms = {"frontend": 0.0, "ingest": 0.0}
                    f(profile_ms=ms)
                    scopes[k] = {g + "_ms": v for g, v in ms.items()}
                eng.set_profiling(False)
                print(json.dumps({"checkpoint": "de_cosine_hard", "feeds": B, "seconds": a.seconds,
                                  "window_s": a.window_s, "window_hop_s": hop_s, "push_s": push_s,
                                  "reference_margin_s": margin_s, "timed_pushes": n_timed, "timed_pairs": n_timed_pairs,
                                  "pairs_per_recording": K, "unit": "pairs/s", **res, "scopes": scopes,
                                  "scopes_note": "feed / per_pair: the timed pushes; windows: the whole recordings"}),
                      flush=True)
    sc.close()


if __name__ == "__main__":
    main()
