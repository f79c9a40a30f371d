"""What scoring window pairs of double-ended (NISQA_DE) recordings costs: Scorer.windows(..., reference=...)
(nisqa_predict_device_window_pairs: each span of either recording packed once, each interior mel frame pair computed
once) against one Scorer.__call__ on a contiguous copy of the same pairs cut out as clips (the same work in one call,
every window's PCM packed and its mel frames computed again).  64 pairs of 60 s recordings at 48 kHz in HBM, the
double-ended checkpoint the tests build from nisqa_mos_only.tar (the shape of train_nisqa_double_ended.yaml: AdaptCNN,
self-attention, cosine alignment), 10 s windows at 5 s and 1 s hops, reference margins of 0 and 0.5 s.

The two arms alternate, --rounds times each, every round --iters calls of each arm's whole batch followed by one device
synchronise; window pairs/s per round (min / median / max).  Then one profiled round of each arm gives the "frontend"
and "ingest" kernel-group times (CUDA events on the engine's lanes; the profiled calls run on one lane).  Checks first
that both arms give the same scores bit for bit.  Prints the card's name and power limit, then one JSON line per
(hop, margin).

    python tools/window_pair_bench.py [--recordings 64] [--seconds 60] [--iters 3] [--rounds 7]
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
    ref = np.stack([np.resize(np.concatenate([base[j] for j in rng.permutation(8)]), T) for _ in range(B)])
    lag = int(0.12 * sr)                       # the degraded signal: the reference delayed, attenuated and noisy
    deg = np.zeros_like(ref, dtype=np.float32)
    deg[:, lag:] = ref[:, :T - lag] * 0.7
    deg = np.clip(deg + rng.normal(0, 300, deg.shape), -32768, 32767).astype(np.int16)
    x, y = torch.from_numpy(deg).cuda(), torch.from_numpy(ref).cuda()
    bargs, bsd = E.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_mos_only.tar"))
    args, sd = V.de_checkpoint("de_cosine_hard", bargs, bsd)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "de_cosine_hard.tar")
        torch.save({"args": args, "model_state_dict": sd}, path)
        sc = Scorer(path)
    W = int(round(a.window_s * sr))
    print("card: %s" % card())
    for hop_s in (5.0, 1.0):
        for margin_s in (0.0, 0.5):
            H, M = int(round(hop_s * 100)) * 480, int(round(margin_s * 100)) * 480
            K = 1 + (T - W) // H                                      # T - W is a multiple of H: every window is whole
            flat_deg = torch.cat([x[b].unfold(-1, W, H) for b in range(B)])
            flat_ref = torch.zeros((B * K, W + 2 * M), dtype=y.dtype, device=y.device)
            ref_len = []
            for b in range(B):                                        # (a copy: the pairs as B K contiguous clips)
                for k in range(K):
                    r0, r1 = max(0, k * H - M), min(T, k * H + W + M)
                    flat_ref[b * K + k, :r1 - r0] = y[b, r0:r1]
                    ref_len.append(r1 - r0)

            def pairs():
                return sc.windows(x, sr, a.window_s, hop_s, reference=y, reference_margin_s=margin_s).scores

            def cut_one_call():
                return sc(flat_deg, sr, reference=flat_ref, reference_lengths=ref_len)

            got, want = pairs(), cut_one_call()
            torch.cuda.synchronize()
            assert torch.equal(got, want), "window pairs differ from the cut pairs"
            arms = {"window_pairs": pairs, "cut_pairs_one_call": cut_one_call}
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
            res["median_saving_pct"] = 100.0 * (1.0 - res["cut_pairs_one_call"]["median"] / res["window_pairs"]["median"])
            scopes = {}
            sc.engine.set_profiling(True)
            for k, f in arms.items():
                f()
                scopes[k] = {g + "_ms": max(0.0, sc.engine.group_ms(g)) for g in ("frontend", "ingest")}
            sc.engine.set_profiling(False)
            print(json.dumps({"checkpoint": "de_cosine_hard (nisqa_mos_only.tar)", "recordings": B, "seconds": a.seconds,
                              "window_s": a.window_s, "window_hop_s": hop_s, "reference_margin_s": margin_s,
                              "pairs_per_recording": K, "unit": "window pairs/s", **res, "scopes_per_batch": scopes}))
            del flat_deg, flat_ref
    sc.close()


if __name__ == "__main__":
    main()
