"""What computing each NISQA_DE reference once buys when many degraded clips share it: the shared-reference call
(nisqa_predict_device_batch_shared_ref) against nisqa_predict_device_batch on the replicated reference batch.  B pairs of
10 s clips at 48 kHz in HBM, M conditions per reference (B / M distinct references; the degraded clip of a condition: its
reference delayed, attenuated and noisy), for de_cosine_hard and an LSTM-td NISQA_DE variant.  At M = 1 the shared call
is also timed against the existing call on the same pairs (what the indirection costs).

Every round times --iters calls of each arm, the arms alternating, each round ended by one device synchronise.  Checks
first that the arms give the same scores bit for bit.  Pairs/s per arm (min / median / max over the rounds), the speed-up
of the medians and each arm's front-end and cnn/td group times (nisqa_group_ms, one profiled call).  Prints the card's
name and power limit, then one JSON line per (checkpoint, M).

    python tools/shared_ref_bench.py [--pairs 256] [--seconds 10] [--conditions 1,4,16,64] [--iters 3] [--rounds 5]
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
from oracle import de_arch_variants as DV  # noqa: E402
from oracle import variants as V  # noqa: E402

CHECKPOINTS = ("de_cosine_hard", "std_fc100_lstm64bi_cosine_hard")
GROUPS = ("frontend", "cnn", "td")


def _checkpoint(name):
    if name in V.DE_VARIANTS:
        return V.de_checkpoint(name, *E.load_checkpoint(os.path.join(ROOT, "weights", "nisqa_mos_only.tar")))
    return DV.de_arch_checkpoint(name, *E.load_checkpoint(os.path.join(ROOT, "weights", DV.DE_ARCH_VARIANTS[name][0])))


def _groups(sc, f):
    sc.engine.set_profiling(1)
    f()
    torch.cuda.synchronize()
    g = {k: float(sc.engine.group_ms(k)) for k in GROUPS}
    sc.engine.set_profiling(0)
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--conditions", default="1,4,16,64")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sr, B = 48000, a.pairs
    T = int(a.seconds * sr)
    base = [synth.synth_speech_pcm16(300 + i, 6.01, sr)[:6 * sr] for i in range(8)]     # (tiled: synthesis is slow)
    rng = np.random.default_rng(0)
    src = np.stack([np.resize(np.concatenate([base[j] for j in rng.permutation(8)]), T) for _ in range(B)])
    print("card: %s" % card())
    for name in CHECKPOINTS:
        args, sd = _checkpoint(name)
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, name + ".tar")
            torch.save({"args": args, "model_state_dict": sd}, path)
            sc = Scorer(path)
        stream = sc._stream()
        for M in [int(m) for m in a.conditions.split(",")]:
            U = B // M
            idx = np.repeat(np.arange(U), M).astype(np.int32)
            ref = src[:U]
            lag = (int(0.03 * sr) * (1 + np.arange(B) % 5))
            deg = np.zeros((B, T), np.float32)
            for p in range(B):
                deg[p, lag[p]:] = ref[idx[p], :T - lag[p]] * (0.5 + 0.1 * (p % M % 5))
            deg = np.clip(deg + rng.normal(0, 300, deg.shape), -32768, 32767).astype(np.int16)
            x, y = torch.from_numpy(deg).cuda(), torch.from_numpy(ref).cuda()
            yr = y[torch.from_numpy(idx.astype(np.int64)).cuda()].contiguous()
            dg, rf, rr = (sc._batch("wave", x, sr, None, None), sc._batch("reference", y, sr, None, None),
                          sc._batch("reference", yr, sr, None, None))
            s_shared = torch.empty((B, 1), device="cuda")
            s_rep = torch.empty((2 * B, 1), device="cuda")
            arms = {"shared": lambda: sc.engine.predict_device_batch_shared_ref(stream, dg, rf, idx, s_shared.data_ptr()),
                    "replicated": lambda: sc.engine.predict_device_batch(stream, dg, s_rep.data_ptr(), ref=rr)}
            for f in arms.values():                                   # warm-up of every shape the rounds use
                f()
            torch.cuda.synchronize()
            assert torch.equal(s_shared.view(torch.int32), s_rep[0::2].view(torch.int32)), (name, M)
            groups = {k: _groups(sc, f) for k, f in arms.items()}
            rates = {k: [] for k in arms}
            for _ in range(a.rounds):
                for k, f in arms.items():
                    t0 = time.perf_counter()
                    for _ in range(a.iters):
                        f()
                    torch.cuda.synchronize()
                    rates[k].append(a.iters * B / (time.perf_counter() - t0))
            out = {"checkpoint": name, "pairs": B, "conditions": M, "references": U, "seconds": a.seconds,
                   "sample_rate": sr}
            for k, r in rates.items():
                out[k + "_pairs_per_s"] = {"min": min(r), "median": float(np.median(r)), "max": max(r)}
                out[k + "_group_ms"] = groups[k]
            out["speedup_median"] = out["shared_pairs_per_s"]["median"] / out["replicated_pairs_per_s"]["median"]
            print(json.dumps(out), flush=True)
            del x, y, yr
        sc.close()


if __name__ == "__main__":
    main()
