"""nisqa_predict_device_batch against nisqa_predict_pcm_device on the same batch resident in HBM (64 x 10 s at 48 kHz,
nisqa.tar): what the ingest kernel (strided [B, C, T] -> packed mono PCM) and the stream handshake cost.

Two inputs: int16 mono (the ingest copies it as int16), and float32 stereo (the ingest mixes it to mono; the packed
arm gets the same mix precomputed, so both arms score identical samples).  The arms alternate, --rounds times each, every
round --iters calls followed by one device synchronise; clips/s per round (min / median / max).  A third arm rotates
the device-batch calls over three CUDA streams: calls on one stream run one after the other (each waits for the work
before it on that stream), calls on separate streams may overlap like the engine's own lanes do.  Checks that all arms
give the same scores bit for bit first.  Prints the card's name and power limit, then one JSON line per input.

    python tools/device_batch_bench.py [--clips 64] [--seconds 10] [--iters 30] [--rounds 7]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nisqa_b200 import engine as E  # noqa: E402
from nisqa_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


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
    T = int(a.seconds * sr) // 16 * 16                     # packed offsets i * T keep the engine's 16-sample alignment
    args, sd = E.load_checkpoint(os.path.join(ROOT, "weights", "nisqa.tar"))
    eng = E.engine_from_checkpoint(args, sd, 0)
    pcm = np.stack([synth.synth_speech_pcm16(100 + i, T / sr + 0.01, sr)[:T] for i in range(B)])
    s16 = torch.from_numpy(pcm).cuda()
    f = s16.float() / 32768.0
    stereo = torch.stack([f, torch.roll(f, 4801, dims=1)], dim=1).contiguous()          # [B, 2, T] float32
    mono = ((stereo[:, 0] + stereo[:, 1]) / 2).contiguous()                               # the ingest's mix rule for 2 channels
    n_out = eng.n_out
    offs, ns, srs = np.arange(B, dtype=np.int64) * T, np.full(B, T, np.int64), np.full(B, sr, np.int32)
    out_a = torch.empty((B, n_out), device="cuda")
    out_b = torch.empty((B, n_out), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    side = [torch.cuda.Stream() for _ in range(3)]
    out_3 = [torch.empty((B, n_out), device="cuda") for _ in range(3)]
    print("card: %s" % card())
    for name, packed, fmt, batch_t, ch in (("int16_mono", s16, E.FMT_S16, s16.unsqueeze(1), -1),
                                          ("float32_stereo", mono, E.FMT_F32, stereo, -1)):
        batch = E.device_batch(batch_t.data_ptr(), E.FMT_S16 if batch_t.dtype == torch.int16 else E.FMT_F32, ns,
                               batch_t.shape[1], ch, T, batch_t.stride(0), batch_t.stride(1), sr)

        def arm_packed():
            eng.predict_pcm_device(packed.data_ptr(), offs, ns, srs, fmt, out_a.data_ptr(), sync=False)

        def arm_batch():
            eng.predict_device_batch(stream, batch, out_b.data_ptr())

        calls = [0]

        def arm_batch_3():
            k = calls[0] % 3
            calls[0] += 1
            eng.predict_device_batch(side[k].cuda_stream, batch, out_3[k].data_ptr())

        for fn in (arm_packed, arm_batch, arm_batch_3, arm_batch_3, arm_batch_3):     # warm-up: module loads, buffer sizes
            fn(); fn()
        torch.cuda.synchronize()
        assert torch.equal(out_a, out_b) and all(torch.equal(out_a, o) for o in out_3), "the entry points disagree on %s" % name
        rates = {"pcm_device": [], "device_batch": [], "device_batch_3_streams": []}
        for _ in range(a.rounds):
            for key, fn in (("pcm_device", arm_packed), ("device_batch", arm_batch), ("device_batch_3_streams", arm_batch_3)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    fn()
                torch.cuda.synchronize()
                rates[key].append(B * a.iters / (time.perf_counter() - t0))
        summary = {k: {"min": round(min(v)), "median": round(float(np.median(v))), "max": round(max(v))} for k, v in rates.items()}
        p, d = summary["pcm_device"], summary["device_batch"]
        overlap = d["max"] >= p["min"] and p["max"] >= d["min"]
        print(json.dumps({"input": name, "clips": B, "seconds": T / sr, "iters": a.iters, "rounds": a.rounds,
                          "clips_per_s": summary, "median_ratio": round(d["median"] / p["median"], 4),
                          "median_ratio_3_streams": round(summary["device_batch_3_streams"]["median"] / p["median"], 4),
                          "ranges_overlap": overlap, "card": card()}))
    eng.close()


if __name__ == "__main__":
    main()
