#!/bin/bash
# GPU-box memory / race / init check of every kernel on the default path (SURVEY.md section 5: the reference has no
# sanitizer story; this is ours): compute-sanitizer memcheck over __graft_entry__.smoke() (nisqa.tar, two
# short clips at 48 / 16 kHz: front-end, conv1, the five wgmma conv layers with their bulk copies /
# mbarriers, self-attention, pooling), over a 96 kHz clip (frontend_kernel, the front end for windows over 1024
# samples), over a short nisqa_tts.tar call (StandardCNN, BiLSTM) and over device-batch
# calls (the ingest kernel, with and without ms_sr, one segments call, one embeddings call, two windows calls, a live feed and a live pair feed); racecheck over the double-ended alignment's multi-block path.
#   bash tools/sanitize.sh TAG
TAG=${1:-rXX}
OUT=gpurun_out
mkdir -p $OUT
cat > /tmp/san_run.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np
import __graft_entry__ as g
g.smoke()
from nisqa_b200 import engine as E, synth
from oracle import nisqa_oracle as O
args, sd = O.load_checkpoint(os.path.join("weights", "nisqa.tar"))
eng = E.Engine(E.config_from_args(args), 0); eng.load_state_dict(sd)
x = synth.synth_speech_pcm16(15, 0.7, 96000)
sc = eng.predict_pcm([x], [96000])[0]
ref, _, _ = O.predict_pcm(args, sd, x.astype(np.float32) / 32768.0, 96000)
assert float(np.abs(sc[0] - ref).max()) <= 1e-4
print("96 kHz ok", sc.tolist())
eng.close()
args, sd = O.load_checkpoint(os.path.join("weights", "nisqa_tts.tar"))
eng = E.Engine(E.config_from_args(args, max_chunk_segments=64), 0); eng.load_state_dict(sd)   # two passes: shrinking planes
sc, ns, st = eng.predict_pcm([synth.synth_speech_pcm16(7, 0.6, 16000), synth.synth_speech_pcm16(8, 0.3, 16000)], [16000, 16000])
ref, _, _ = O.predict_pcm(args, sd, synth.synth_speech_pcm16(7, 0.6, 16000).astype(np.float32) / 32768.0, 16000)
assert abs(float(sc[0, 0]) - float(ref[0])) <= 1e-4
print("tts ok", sc.tolist())
eng.close()
# round-2 kernels: double-ended model (de_align, td_in with 192 inputs, second stack), td_2 behind the first stack,
# device resampler (both directions), conv12 with the padded mel ring
from oracle import variants as V
bargs, bsd = O.load_checkpoint(os.path.join("weights", "nisqa_mos_only.tar"))
for name in ("de_cosine_hard", "de_distance_soft_xy"):
    a2, s2 = V.de_checkpoint(name, bargs, bsd)
    e2 = E.Engine(E.config_from_args(a2), 0); e2.load_state_dict(s2)
    d, srd, r, srr = V.de_pair_pcm(V.DE_PAIRS[1])
    got = e2.predict_pcm([d, r], [srd, srr])[0]
    ref = O.predict_pcm_de(a2, s2, d.astype(np.float32) / 32768.0, srd, r.astype(np.float32) / 32768.0, srr)[0]
    assert abs(float(got[0, 0]) - float(ref[0])) <= 5e-4, (name, got, ref)
    # a reference of 130 steps (three key blocks, the last with 2 keys) behind a 70-step degraded clip
    d2, r2 = synth.synth_speech_pcm16(13, 2.9, 16000), synth.synth_speech_pcm16(14, 5.3, 16000)
    assert e2.predict_pcm([d2, r2], [16000, 16000])[1].tolist() == [70, 130]
    e2.close()
a3, s3 = V.variant_checkpoint("mos_td2_sa_pos_enc", bargs, bsd)
e3 = E.Engine(E.config_from_args(a3), 0); e3.load_state_dict(s3)
x = synth.synth_speech_pcm16(9, 0.8, 16000)
print("td2", e3.predict_pcm([x], [16000])[0].tolist())
from nisqa_b200 import resample as RS
for so, sn in ((48000, 16000), (16000, 44100)):
    xs = synth.synth_speech_pcm16(10, 0.25, so)
    assert np.array_equal(e3.resample_device(xs, so, sn), RS.resample(xs, so, sn))
print("resample ok", e3.predict_pcm_resampled([x, synth.synth_speech_pcm16(11, 0.5, 48000)], [16000, 48000], 16000)[0].tolist())
e3.close()
# device-batch ingest (csrc/ingest.cu): int16 channel pick, float32 mix of strided channels, ms_sr into a conversion slot
import torch
from nisqa_b200.scorer import Scorer
w = torch.from_numpy(np.stack([synth.synth_speech_pcm16(12 + c, 0.7, 48000) for c in range(2)])[None]).cuda()   # [1, 2, T]
s4 = Scorer(os.path.join("weights", "nisqa.tar"))
print("ingest", s4(w, 48000, channel=1).tolist(), s4(w.float() / 32768, 48000).tolist())
seg = s4.segments(w, 48000, channel=0)      # segment_scores_kernel (PoolAttFF logits of the last td_sa layer)
print("segments", seg.counts, seg.seg_weights.sum(0).tolist())
emb = s4.embed(w, 48000, channel=0, rows=True)    # pool_embed_kernel (rows in the reference's order)
print("embeddings", emb.counts, emb.pooled.shape, emb.rows.shape)
s4.close()
s5 = Scorer(os.path.join("weights", "nisqa_mos_only.tar"), ms_sr=16000)
print("ingest ms_sr", s5(w[0], 48000, lengths=[30000, w.shape[-1]]).tolist())
s5.close()
# windows of a recording (ingest_span_kernel, frontend_windows_kernel: shared and edge pairs, both pairings): 25 s at a
# 3.33 s hop (an odd number of frames), and 96 kHz windows (the generic front-end arithmetic)
s6 = Scorer(os.path.join("weights", "nisqa.tar"))
r = torch.from_numpy(synth.synth_speech_pcm16(16, 25.0, 48000)).cuda()
print("windows", s6.windows(r, 48000, 10.0, 3.33).scores.tolist())
print("windows 96 kHz", s6.windows(torch.from_numpy(synth.synth_speech_pcm16(17, 12.0, 96000)).cuda(), 96000, 10.0, 1.0).scores.tolist())
# live feeds (ingest_feed_kernel, frontend_feed_kernel, feed_rows_kernel, and frontend_windows_kernel's edge pairs over
# the rings): two feeds of 12.5 s and 3 s at a 3.33 s hop (both pairings) in 0.7 s pushes, ring wrap and mirror included
fd = s6.feed(2, 48000, 10.0, 3.33, max_push_s=0.7)
n, T = 33600, 600000
for t in range(0, T, n):
    m = [min(n, T - t), min(n, max(0, 144000 - t))]
    out = fd.push(torch.stack([r[t:t + n], r[t:t + n]]), lengths=m, end=[t + n >= T, t < 144000 <= t + n])
    print("feed", out.scores.tolist())
fd.close()
s6.close()
# live pair feeds (both sources' rings in one allocation, the reference's offset geometry and mirror of W + 2M, the
# front-clipped reference windows as one-window spans over the ring): one pair of 16 s / 15.5 s at 16 kHz with a 1.5 s
# margin (two front-clipped windows), 0.5 s pushes and the reference 1 s behind (the maximal skew), so both rings wrap;
# the ending push emits end-clipped reference windows
import tempfile
a7, s7 = V.de_checkpoint("de_cosine_hard", bargs, bsd)
p7 = os.path.join(tempfile.mkdtemp(), "de.tar")
torch.save({"args": a7, "model_state_dict": s7}, p7)
s8 = Scorer(p7)
d8 = torch.from_numpy(synth.synth_speech_pcm16(18, 16.0, 16000)).cuda()
fp = s8.feed(1, 16000, 5.0, 1.0, max_push_s=0.5, reference=True, reference_margin_s=1.5, max_skew_s=1.0)
n, Td, Tr = 8000, 256000, 248000
for t in range(0, Td + n, n):
    a, b = min(n, max(0, Td - t)), min(n, max(0, Tr - (t - 16000))) if t >= 16000 else 0
    out = fp.push(d8[None, t:t + n], d8[None, max(0, t - 16000):max(0, t - 16000) + n], lengths=[a], reference_lengths=[b],
                  end=[t + n >= Td + n])
    print("pair feed", out.scores.tolist())
fp.close()
s8.close()
PY
timeout 400 compute-sanitizer --tool memcheck --error-exitcode 7 --log-file $OUT/${TAG}_memcheck.log python /tmp/san_run.py > $OUT/${TAG}_memcheck_stdout.log 2>&1
echo "memcheck exit $?"
tail -5 $OUT/${TAG}_memcheck.log; tail -3 $OUT/${TAG}_memcheck_stdout.log
# shared-memory hazards of de_align_kernel's key-block loop (Yb / Yn / Yp / YK reused across blocks): one soft and one
# hard call whose reference spans three key blocks
cat > /tmp/san_de.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
from nisqa_b200 import engine as E, synth
from oracle import nisqa_oracle as O, variants as V
bargs, bsd = O.load_checkpoint(os.path.join("weights", "nisqa_mos_only.tar"))
d, r = synth.synth_speech_pcm16(13, 2.9, 16000), synth.synth_speech_pcm16(14, 5.3, 16000)
for name, over in (("de_luong_soft", None), ("de_bahd_hard", {"de_align": "bahd", "de_align_apply": "hard", "de_fuse": "+/-"})):
    a, s = V.de_checkpoint(name, bargs, bsd, over)
    e = E.Engine(E.config_from_args(a), 0); e.load_state_dict(s)
    print(name, e.predict_pcm([d, r], [16000, 16000])[:2])
    e.close()
PY
timeout 300 compute-sanitizer --tool racecheck --error-exitcode 7 --log-file $OUT/${TAG}_de_racecheck.log python /tmp/san_de.py > $OUT/${TAG}_de_racecheck_stdout.log 2>&1
echo "de racecheck exit $?"
tail -4 $OUT/${TAG}_de_racecheck.log; tail -2 $OUT/${TAG}_de_racecheck_stdout.log
# frontend_pp_kernel with a hop over 512 (ms_hop_length = ms_win_length = 20 ms at 32 kHz: hop = win = 640): the input
# stage's reads must stay inside the sample slot, clear of the FFT planes the other warps write; PCM16 and float32
cat > /tmp/san_fe.py <<'PY'
import os, sys
sys.path.insert(0, os.getcwd())
from nisqa_b200 import engine as E, synth
from oracle import nisqa_oracle as O
args, sd = O.load_checkpoint(os.path.join("weights", "nisqa_mos_only.tar"))
e = E.Engine(E.config_from_args(dict(args, ms_hop_length=0.02, ms_win_length=0.02)), 0); e.load_state_dict(sd)
x = synth.synth_speech_pcm16(19, 1.3, 32000)
print("hop 640", e.predict_pcm([x], [32000])[0].tolist(), e.predict_pcm([x.astype("float32") / 32768], [32000])[0].tolist())
e.close()
PY
for tool in racecheck memcheck; do
  timeout 300 compute-sanitizer --tool $tool --error-exitcode 7 --log-file $OUT/${TAG}_fe_hop640_$tool.log python /tmp/san_fe.py > $OUT/${TAG}_fe_hop640_${tool}_stdout.log 2>&1
  echo "fe hop 640 $tool exit $?"
  tail -4 $OUT/${TAG}_fe_hop640_$tool.log; tail -1 $OUT/${TAG}_fe_hop640_${tool}_stdout.log
done
# shared-memory hazards (racecheck) and uninitialised device reads (initcheck) of the whole run (RACE=1)
[ -z "$RACE" ] && exit 0
timeout 400 compute-sanitizer --tool racecheck --error-exitcode 7 --log-file $OUT/${TAG}_racecheck.log python /tmp/san_run.py > $OUT/${TAG}_racecheck_stdout.log 2>&1
echo "racecheck exit $?"
tail -4 $OUT/${TAG}_racecheck.log
timeout 280 compute-sanitizer --tool initcheck --error-exitcode 7 --log-file $OUT/${TAG}_initcheck.log python /tmp/san_run.py > $OUT/${TAG}_initcheck_stdout.log 2>&1
echo "initcheck exit $?"
tail -4 $OUT/${TAG}_initcheck.log
