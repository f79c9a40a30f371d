"""nisqa_predict_device_batch and nisqa_b200.scorer.Scorer: waveforms already on the GPU, scored in the caller's CUDA
stream order.  CPU part: the ABI struct layout and every argument refusal of Scorer (host code, before any launch).
GPU part: bit-for-bit parity with the host entry points, strided and multi-channel input against the file ingest,
ms_sr, NISQA_DE, and the stream contract (ordering, no host synchronisation, errors before anything is enqueued)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from nisqa_b200.scorer import Scorer

SCORE_TOL = 1e-4


def _host_scorer(args):
    """A Scorer's host side alone (no engine, no GPU): argument checks on CPU tensors"""
    s = Scorer.__new__(Scorer)
    s._configure(args, torch.device("cpu"))
    s.engine = None
    return s


def _args(ckpt):
    return E.load_checkpoint(os.path.join(WEIGHTS, ckpt))[0]


def _de_args():
    from oracle import variants as V
    bargs, bsd = E.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    return V.de_checkpoint("de_cosine_hard", bargs, bsd)


def _len_for_segments(cfg, n_seg, sr):
    """the shortest clip length with n_seg segments"""
    lo, hi = 1, 1 << 28
    while lo < hi:
        mid = (lo + hi) // 2
        if E.segment_counts(cfg, mid, sr)[1] >= n_seg:
            hi = mid
        else:
            lo = mid + 1
    assert E.segment_counts(cfg, lo, sr)[1:] == (n_seg, E.CLIP_OK)
    return lo


# ------------------------------------------------------------------ CPU
def test_device_batch_struct_layout_matches_header(tmp_path):
    src = tmp_path / "layout.c"
    fields = ["data", "sample_fmt", "n_clips", "n_channels", "channel", "length", "clip_stride", "channel_stride",
              "n_samples", "sample_rate"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(nisqa_device_batch)'
                   + "".join(", offsetof(nisqa_device_batch, %s)" % f for f in fields) + ");return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    import ctypes
    assert out == [ctypes.sizeof(E.NisqaDeviceBatch)] + [getattr(E.NisqaDeviceBatch, f).offset for f in fields]


def test_scorer_refuses_bad_arguments(built_lib):
    s = _host_scorer(_args("nisqa.tar"))
    assert s.columns == ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"]
    assert _host_scorer(_args("nisqa_tts.tar")).columns == ["mos_pred"]
    x = torch.zeros(2, 2, 48000)
    with pytest.raises(TypeError, match="wave"):
        s(np.zeros(48000, np.float32), 48000)
    for dt in (torch.float64, torch.float16, torch.int32):
        with pytest.raises(TypeError, match="wave: dtype"):
            s(x.to(dt), 48000)
    with pytest.raises(ValueError, match="wave: on meta"):
        s(torch.zeros(2, 48000, device="meta"), 48000)
    with pytest.raises(ValueError, match="wave: shape"):
        s(x[None], 48000)
    with pytest.raises(ValueError, match="contiguous"):
        s(x[:, :, ::2], 48000)
    with pytest.raises(ValueError, match="sample_rate"):
        s(x, 0)
    with pytest.raises(TypeError, match="lengths: host"):
        s(x, 48000, lengths=torch.tensor([48000, 48000], device="meta"))
    with pytest.raises(ValueError, match="lengths: 1 entries"):
        s(x, 48000, lengths=[48000])
    with pytest.raises(ValueError, match=r"lengths\[1\] = 48001"):
        s(x, 48000, lengths=[48000, 48001])
    with pytest.raises(TypeError, match="lengths"):
        s(x, 48000, lengths=[0.5, 1.0])
    with pytest.raises(ValueError, match="channel: 2 is out of range"):
        s(x, 48000, channel=2)
    with pytest.raises(ValueError, match="channel: -1"):
        s(x, 48000, channel=-1)
    with pytest.raises(ValueError, match="reference: only a double-ended"):
        s(x, 48000, reference=x)
    de = _host_scorer(_de_args()[0])
    with pytest.raises(ValueError, match="reference: a double-ended"):
        de(x, 48000)
    with pytest.raises(ValueError, match="reference: 1 clips for 2"):
        de(x, 48000, reference=x[:1])


def test_scorer_raises_too_short_and_too_long_before_any_launch(built_lib):
    args = _args("nisqa.tar")
    s = _host_scorer(args)
    x = torch.zeros(3, 48000 * 53, dtype=torch.int16)
    with pytest.raises(ValueError, match=r"^Sample too short\. Only 2 windows available but seg_length=15\. "
                                         r"Consider zero padding the audio sample\. File: wave\[1\]$"):
        s(x, 48000, lengths=[48000, 480, 48000])
    n_seg = E.segment_counts(s.cfg, 48000 * 53, 48000)[1]
    with pytest.raises(ValueError, match=r"^n_wins %d > max_length 1300 --- wave\[2\]\. Increase max window length "
                                         r"ms_max_segments!$" % n_seg):
        s(x, 48000, lengths=[48000, 48000, 48000 * 53])
    # after ms_sr the converted length counts
    with pytest.raises(ValueError, match=r"Only 4 windows .* File: wave\[0\]"):
        _host_scorer(dict(args, ms_sr=16000))(x, 48000, lengths=[480 * 3, 48000, 48000])
    de = _host_scorer(_de_args()[0])
    with pytest.raises(ValueError, match=r"File: reference\[0\]"):
        de(x[:1], 48000, lengths=[48000], reference=x[:1], reference_lengths=[100])


# ------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


def _ragged(cfg, sr, seed):
    """clips of 1, 97 and 1300 segments and two ordinary ones, int16, and their lengths"""
    lens = [_len_for_segments(cfg, 1, sr), 2 * sr + 333, _len_for_segments(cfg, 97, sr),
            _len_for_segments(cfg, 1300, sr), sr + 17]
    T = max(lens) + 5
    clips = [synth.synth_speech_pcm16(seed + i, T / sr + 0.01, sr)[:T] for i in range(len(lens))]
    return np.stack(clips), lens


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


@gpu
@pytest.mark.parametrize("ckpt", ["nisqa.tar", "nisqa_mos_only.tar", "nisqa_tts.tar"])
def test_scorer_equals_host_entry_point_bit_for_bit(built_lib, ckpt):
    path = os.path.join(WEIGHTS, ckpt)
    sc = Scorer(path)
    sr = 48000
    pcm, lens = _ragged(sc.cfg, sr, 4000)
    for x in (pcm, _f32(pcm)):
        host, nseg, status = sc.engine.predict_pcm([x[i, :n] for i, n in enumerate(lens)], [sr] * len(lens))
        assert np.all(status == E.CLIP_OK) and list(nseg[[0, 2, 3]]) == [1, 97, 1300]
        got = sc(torch.from_numpy(x).cuda(), sr, lengths=lens)
        assert got.dtype == torch.float32 and got.shape == (len(lens), len(sc.columns)) and got.is_cuda
        np.testing.assert_array_equal(got.cpu().numpy(), host)
        # one clip, [T]
        np.testing.assert_array_equal(sc(torch.from_numpy(x[1, :lens[1]]).cuda(), sr).cpu().numpy(), host[1:2])
    # the same call split into several internal passes
    split = Scorer(path, b200_max_chunk_segments=600)
    np.testing.assert_array_equal(split(torch.from_numpy(pcm).cuda(), sr, lengths=lens).cpu().numpy(),
                                  split.engine.predict_pcm([pcm[i, :n] for i, n in enumerate(lens)], [sr] * len(lens))[0])
    sc.close(); split.close()


@gpu
def test_strided_views_equal_their_contiguous_copies(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    B, T = 3, 48000 * 2
    big = torch.from_numpy(_f32(np.stack([synth.synth_speech_pcm16(700 + i, 2.5, 48000)[:T + 999] for i in range(B)]))).cuda()
    view = big[:, 555:555 + T]                                          # clip stride T + 999
    assert not view.is_contiguous()
    np.testing.assert_array_equal(sc(view, 48000).cpu().numpy(), sc(view.contiguous(), 48000).cpu().numpy())
    cbt = torch.stack([big[:, :T], big[:, 999:999 + T]]).cuda()            # [C, B, T]
    bct = cbt.transpose(0, 1)                                           # [B, C, T]: clip stride T, channel stride B T
    assert not bct.is_contiguous()
    for ch in (None, 1):
        np.testing.assert_array_equal(sc(bct, 48000, channel=ch).cpu().numpy(),
                                      sc(bct.contiguous(), 48000, channel=ch).cpu().numpy())
    sc.close()


@gpu
def test_multichannel_equals_the_file_ingest(built_lib, tmp_path):
    from nisqa_b200.NISQA_model import nisqaModel
    path = os.path.join(WEIGHTS, "nisqa.tar")
    sc = Scorer(path)
    sr, n = 48000, int(2.3 * 48000)
    chans = np.stack([synth.synth_speech_pcm16(800 + c, 2.3, sr)[:n] for c in range(4)], axis=1)     # [n, 4]
    cases = [("s16_2ch.wav", chans[:, :2], wav.write_wav_pcm16), ("f32_4ch.wav", _f32(chans) * 0.7, wav.write_wav_f32)]
    for name, data, writer in cases:
        writer(str(tmp_path / name), data, sr)
        t = torch.from_numpy(np.ascontiguousarray(data.T)[None]).cuda()     # [1, C, T]
        for ch in (None, 1):
            df = nisqaModel({"mode": "predict_file", "pretrained_model": path, "deg": str(tmp_path / name),
                             "output_dir": None, "tr_bs_val": 1, "tr_num_workers": 0, "ms_channel": ch}).predict()
            want = df[sc.columns].to_numpy(dtype=np.float32)
            np.testing.assert_array_equal(sc(t, sr, channel=ch).cpu().numpy(), want, err_msg="%s %r" % (name, ch))
    sc.close()


@gpu
def test_ms_sr_checkpoint_equals_predict_pcm_resampled(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa_mos_only.tar"), ms_sr=16000)
    sr, lens = 48000, [48000 * 2 + 7, 48000 * 3, 30001]
    pcm = np.stack([synth.synth_speech_pcm16(900 + i, 3.1, sr)[:max(lens)] for i in range(3)])
    for x in (pcm, _f32(pcm)):
        want, nseg, _ = sc.engine.predict_pcm_resampled([x[i, :n] for i, n in enumerate(lens)], [sr] * 3, 16000)
        np.testing.assert_array_equal(sc(torch.from_numpy(x).cuda(), sr, lengths=lens).cpu().numpy(), want)
    # stereo int16, mixed before the conversion, as the file ingest does
    st = torch.from_numpy(np.stack([pcm, pcm[::-1].copy()], axis=1)).cuda()
    mixed = (_f32(pcm) + _f32(pcm[::-1].copy())) / np.float32(2)
    want = sc.engine.predict_pcm_resampled([mixed[i, :n] for i, n in enumerate(lens)], [sr] * 3, 16000)[0]
    np.testing.assert_array_equal(sc(st, sr, lengths=lens).cpu().numpy(), want)
    sc.close()


@gpu
def test_double_ended_pairs(built_lib, tmp_path):
    from oracle import nisqa_oracle as O
    from oracle import variants as V
    args, sd = _de_args()
    torch.save({"args": args, "model_state_dict": sd}, tmp_path / "de.tar")
    sc = Scorer(str(tmp_path / "de.tar"))
    for pair in V.DE_PAIRS:
        deg, srd, ref, srr = V.de_pair_pcm(pair)
        want, _, _ = sc.engine.predict_pcm([deg, ref], [srd, srr])
        got = sc(torch.from_numpy(deg).cuda(), srd, reference=torch.from_numpy(ref).cuda(), reference_sample_rate=srr)
        assert got.shape == (1, 1)
        np.testing.assert_array_equal(got.cpu().numpy(), want[0:1])
        sc_o, _, _ = O.predict_pcm_de(args, sd, _f32(deg), srd, _f32(ref), srr)
        assert abs(float(got[0, 0]) - sc_o[0]) <= 5 * SCORE_TOL           # the hard-alignment bound of test_gpu_parity
    # two pairs in one batch (same rates), the reference as float32 and stereo: mixed to mono
    deg, srd, ref, _ = V.de_pair_pcm(V.DE_PAIRS[0])
    n = min(len(deg), len(ref))
    d2 = torch.from_numpy(np.stack([deg[:n], deg[::-1][:n].copy()])).cuda()
    r2 = torch.from_numpy(np.stack([np.stack([_f32(ref[:n])] * 2), np.stack([_f32(ref[:n]), _f32(deg[:n])])])).cuda()
    got = sc(d2, srd, lengths=[n, n - 100], reference=r2).cpu().numpy()
    mix = (_f32(ref[:n]) + _f32(deg[:n])) / np.float32(2)
    want = sc.engine.predict_pcm([_f32(deg[:n]), _f32(ref[:n]), _f32(deg[::-1][:n - 100].copy()), mix], [srd] * 4)[0]
    np.testing.assert_array_equal(got, want[0::2])
    sc.close()


@gpu
def test_stream_order_input_freed_and_reused(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    B, T = 4, 48000 * 4
    src = torch.from_numpy(_f32(np.stack([synth.synth_speech_pcm16(950 + i, 4.0, 48000)[:T] for i in range(B)]))).cuda()
    want = sc(src, 48000)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)                      # a slow producer ...
        x = torch.empty_like(src)
        x.copy_(src)                                       # ... fills the input right before the call, no synchronise
        got = sc(x, 48000)
        del x                                              # freed at once: its memory goes back to s's pool
        junk = [torch.full((B, T), 7.0, device="cuda") for _ in range(3)]      # reuses it, on s
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy(), want.cpu().numpy())
    del junk
    sc.close()


@gpu
def test_call_does_not_wait_for_the_gpu(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    x = torch.from_numpy(_f32(np.stack([synth.synth_speech_pcm16(960 + i, 3.0, 48000) for i in range(3)]))).cuda()
    want = sc(x, 48000).cpu().numpy()                      # (also sizes every buffer: no allocation below)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)                         # ~50 ms of GPU time on the current stream
    got = sc(x, 48000)
    assert not torch.cuda.current_stream().query()         # returned while the stream still sleeps
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    sc.close()


@gpu
def test_errors_are_raised_before_anything_is_enqueued(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    x = torch.zeros(2, 48000 * 53, dtype=torch.int16, device="cuda")
    sc(x[:, :48000], 48000)
    before = sc.engine.kernel_launches()
    with pytest.raises(ValueError, match="Sample too short"):
        sc(x, 48000, lengths=[48000, 100])
    with pytest.raises(ValueError, match="n_wins"):
        sc(x, 48000)
    assert sc.engine.kernel_launches() == before
    # the C entry point refuses what the wrapper would: a length beyond the array
    b = E.device_batch(x.data_ptr(), E.FMT_S16, [48000 * 54], 1, -1, 48000 * 53, x.stride(0), 0, 48000)
    out = torch.empty((1, 5), device="cuda")
    with pytest.raises(E.EngineError, match="n_samples"):
        sc.engine.predict_device_batch(torch.cuda.current_stream().cuda_stream, b, out.data_ptr())
    sc.close()


_FRESH_MS_SR = r"""
import os, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from nisqa_b200 import engine as E, synth
from nisqa_b200.scorer import Scorer
path = os.path.join(sys.argv[1], "weights", "nisqa_mos_only.tar")
x = np.stack([synth.synth_speech_pcm16(970 + i, 2.0, 16000) for i in range(2)])
# audio already at ms_sr, first thing in the process: the interpolation table has never been set
got = Scorer(path, ms_sr=16000)(torch.from_numpy(x).cuda(), 16000).cpu().numpy()
args, sd = E.load_checkpoint(path, {"ms_sr": 16000})
eng = E.engine_from_checkpoint(args, sd)
out = torch.empty((2, 1), device="cuda")
eng.predict_device_batch(0, E.device_batch(torch.from_numpy(x).cuda().data_ptr(), E.FMT_S16, [x.shape[1]] * 2, 1, -1,
                                           x.shape[1], x.shape[1], 0, 16000), out.data_ptr(), target_sr=16000)
torch.cuda.synchronize()
want = eng.predict_pcm_resampled(list(x), [16000, 16000], 16000)[0]
assert np.array_equal(got, want) and np.array_equal(out.cpu().numpy(), want), (got, out, want)
print("fresh ms_sr ok")
"""


@gpu
def test_ms_sr_at_the_target_rate_in_a_fresh_process(built_lib, tmp_path):
    """Scorer and Engine.predict_device_batch with ms_sr set the resampler's table themselves, also for audio that is
    already at ms_sr (no conversion needed) and nothing else ran before in the process"""
    script = tmp_path / "fresh.py"
    script.write_text(_FRESH_MS_SR)
    r = subprocess.run([sys.executable, str(script), ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "fresh ms_sr ok" in r.stdout, r.stdout + r.stderr


@gpu
def test_ms_sr_calls_do_not_wait_for_the_gpu(built_lib):
    """Two ms_sr calls in a row behind a sleeping stream: the conversion buffers rotate, so neither call waits"""
    sc = Scorer(os.path.join(WEIGHTS, "nisqa_mos_only.tar"), ms_sr=16000)
    x = torch.from_numpy(_f32(np.stack([synth.synth_speech_pcm16(980 + i, 3.0, 48000) for i in range(3)]))).cuda()
    want = [sc(x, 48000).cpu().numpy(), sc(x[:2], 48000).cpu().numpy()]     # (sizes both conversion slots)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)                         # ~50 ms of GPU time on the current stream
    got = [sc(x, 48000), sc(x[:2], 48000)]
    assert not torch.cuda.current_stream().query()         # both returned while the stream still sleeps
    torch.cuda.synchronize()
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g.cpu().numpy(), w)
    sc.close()
