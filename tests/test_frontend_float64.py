"""The front end's mel dB rows (csrc/frontend.cu) against a float64 STFT at every kernel instance, rate, STFT geometry and
signal edge, with the per-element bound and the precision statistic of tests/stage_ref_frontend.py.

CPU: the float64 reference + clamp is the oracle's operation (oracle.nisqa_oracle.mel_db, within the oracle's own
float32 rounding) on every rate, geometry and signal of the GPU battery; the float32 restatement of the pipelined
kernel sits within 1/8 of both limits, and its fp16-table, bf16-sample and shifted-frame variants fail by 8x or more.
GPU: every call runs in one pass and checks every element of its MEL_DB dump (and that the dump has no extra rows):
the 28 clip-path instances (frontend_pp_kernel / frontend_kernel x int16 / float32 x 7 band counts) on a battery of
edge signals; 4 kHz .. 204.8 kHz with fmax 20 kHz and 8 kHz (frontend_kernel at Q = 1 .. 4); STFT geometries from
checkpoint args (a hop over 512 on the pipelined kernel); a mixed-rate pass; fe_ppc 1, 2, 3, 8 bit for bit; device
input at every misalignment, bit for bit with the host call.
"""
import os

import numpy as np
import pytest

import stage_ref_frontend as F
from conftest import WEIGHTS
from nisqa_b200 import synth
from oracle import librosa_compat as lb
from oracle import nisqa_oracle as O

N_MELS = (32, 40, 48, 64, 80, 96, 128)
RATES = (4000, 8000, 11025, 22050, 44100, 48000, 51200, 51250, 96000, 120000, 192000, 204800)
FMAXES = (20000, 8000)                  # nisqa.tar / nisqa_mos_only.tar, nisqa_tts.tar
GEOMETRIES = (((0.01, 0.025), 48000), ((0.015, 0.02), 48000), ((0.02, 0.02), 32000), ((0.005, 0.02), 16000))
SPAN_MAX = 1536                         # frontend.cu kSpanMax
U = 2.0 ** -24


def _args(**over):
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    return dict(args, **over)


def fe_kernel(args, srs):
    """the clip path's choice for a pass (launch_frontend_mels): the pipelined kernel when every clip has win <= 1024
    and hop + win <= 1536, else frontend_kernel at Q = max ceil(win / 1024)"""
    geo = [F.hop_win(sr, args) for sr in srs]
    Q = max((w + 1023) // 1024 for _, w in geo)
    return "pp" if Q == 1 and max(h + w for h, w in geo) <= SPAN_MAX else "generic Q=%d" % Q


def _clip16(v):
    return np.clip(np.round(v), -32768, 32767).astype(np.int16)


def battery(sr, args, long_clip=False):
    """(name, int16 clip) of the edge signals at rate sr; frame counts odd and even, the 15-frame minimum (shorter than
    the 2048-sample reflect pad below 22 kHz: repeated reflection) and, with long_clip, ms_max_segments segments"""
    hop, _ = F.hop_win(sr, args)
    rng = np.random.default_rng(sr)
    n_even, n_odd = 37 * hop + hop // 3, 40 * hop + 1            # 38 and 41 frames
    t = np.arange(n_odd) / sr
    out = [("speech", synth.synth_speech_pcm16(11, n_even / sr + 0.05, sr)[:n_even]),
           ("min_frames", synth.synth_speech_pcm16(12, 14 * hop / sr + 0.05, sr)[:14 * hop]),
           ("noise", _clip16(rng.normal(0.0, 8000.0, n_odd))),
           ("tone_bin", _clip16(16000 * np.sin(2 * np.pi * 93 * sr / 4096 * t))),
           ("tone_off", _clip16(16000 * np.sin(2 * np.pi * 93.37 * sr / 4096 * t[:n_even]))),
           ("dc", _clip16(8192 + rng.normal(0.0, 30.0, n_even))),
           ("nyquist", np.where(np.arange(n_odd) % 2 == 0, 32767, -32768).astype(np.int16))]
    imp = np.zeros(n_even, np.int16)
    imp[0], imp[-1] = 32767, -32768
    dur = n_odd / sr
    out += [("impulses", imp),
            ("chirp", _clip16(20000 * np.sin(np.pi * (sr / 2) * t * t / dur))),
            ("silence", np.zeros(n_odd, np.int16)),
            ("dither", rng.integers(-1, 2, n_even).astype(np.int16))]
    loud = _clip16(synth.synth_speech_pcm16(13, n_odd / sr + 0.05, sr)[:n_odd] * 1e-3)
    loud[-2 * hop:] = _clip16(rng.normal(0.0, 12000.0, 2 * hop))
    out.append(("loud_end", loud))
    if long_clip:
        n = (args["ms_seg_length"] - 1 + (args["ms_max_segments"] - 1) * args["ms_seg_hop_length"]) * hop + hop - 1
        y = synth.synth_speech_pcm16(14, n / sr + 0.05, sr)[:n]
        assert O.segment_counts(n, sr, args)[1:] == (args["ms_max_segments"], O.STATUS_OK)
        out.append(("max_segments", y))
    return out


def _f32(y):
    return y.astype(np.float32) / np.float32(32768.0)


_REF = {}


def reference(y, sr, args, fb):
    """mel_ref, cached: a test checks each clip in both formats and several passes"""
    hop, win = F.hop_win(sr, args)
    key = (y.tobytes().__hash__(), y.size, sr, hop, win, fb.tobytes().__hash__())
    if key not in _REF:
        if len(_REF) > 64:
            _REF.clear()
        _REF[key] = F.mel_ref(y, sr, args, fb)
    return _REF[key]


# ------------------------------------------------------------------------------------------------------------ CPU
def _oracle_tolerance(M, fb):
    """the oracle's own float32 rounding, in dB: complex64 spectrum and |.| (2 u), the float32 product over the band's
    nnz non-negative terms ((nnz + 2) u of the band) and log10 / the clamp (a few ulp)"""
    nnz = (np.asarray(fb) != 0).sum(1)
    rel = (nnz + 4) * U
    tol = 10.0 / np.log(10.0) * 2.0 * rel[:, None] * np.ones_like(M)
    return tol + tol.max() + 8 * np.spacing(np.float32(100.0))


def test_reference_is_the_oracle_operation():
    worst = 0.0
    cases = [(sr, fmax, _args(ms_fmax=fmax)) for sr in RATES for fmax in FMAXES]
    cases += [(sr, 20000, _args(ms_hop_length=h, ms_win_length=w)) for (h, w), sr in GEOMETRIES]
    for sr, fmax, args in cases:
        fb = lb.mel(sr, 4096, n_mels=48, fmin=0.0, fmax=fmax, htk=False, norm="slaney")
        sigs = battery(sr, args, long_clip=(sr == 8000 and fmax == 8000))
        for name, y in sigs:
            M, L, Wn = F.mel_ref(y, sr, args, fb)
            want = np.asarray(O.mel_db(_f32(y), sr, args), dtype=np.float64)
            assert want.shape == M.shape == (48, 1 + y.size // F.hop_win(sr, args)[0]), (sr, name)
            err = np.abs(F.ref_db(M) - want)
            tol = _oracle_tolerance(M, fb)
            assert (err <= tol).all(), (sr, fmax, name, float(err.max()), float((err / tol).max()))
            worst = max(worst, float((err / tol).max()))
    print("\nfloat64 reference vs the oracle: max |diff| / the oracle's float32 rounding %.3g" % worst)


EMU_RATES = (8000, 16000, 48000)


def _emu_signals(sr, args):
    b = dict(battery(sr, args))
    return [(k, b[k]) for k in ("speech", "noise", "tone_bin", "tone_off")]


def _emu_figures(**variant):
    """max tier-1 ratio and tier-2 RMS of emulate_pp over the calibration signals (int16 and float32)"""
    args = _args()
    r1, diffs = 0.0, []
    for sr in EMU_RATES:
        fb = lb.mel(sr, 4096, n_mels=48, fmin=0.0, fmax=args["ms_fmax"], htk=False, norm="slaney")
        for name, y in _emu_signals(sr, args):
            M, L, Wn = F.mel_ref(y, sr, args, fb)
            for x in (y, _f32(y)):
                got = F.emulate_pp(x, sr, args, fb, **variant)
                r1 = max(r1, F.tier1_ratio(got, M, L, Wn))
                diffs.append(F.tier2_diffs(got, M, L, Wn))
    return r1, F.rms(diffs)


def test_fp32_restatement_sits_well_inside_both_limits():
    r1, r2 = _emu_figures()
    print("\nfloat32 restatement of frontend_pp_kernel: max tier-1 ratio %.3g, tier-2 RMS %.3g dB (limit %.3g dB)"
          % (r1, r2, F.TIER2_DB))
    assert r1 <= 1 / 8
    assert r2 <= F.TIER2_DB / 8
    # the limit is 8x the restatement's RMS rounded up to a power of two: no looser
    assert F.TIER2_DB < 16 * r2


@pytest.mark.parametrize("variant", ["fp16_tables", "bf16_samples", "late_b"])
def test_the_bound_rejects_a_lower_precision_or_shifted_kernel(variant):
    r1, r2 = _emu_figures(**{variant: True})
    print("\n%s: max tier-1 ratio %.3g, tier-2 RMS / limit %.3g" % (variant, r1, r2 / F.TIER2_DB))
    if variant == "late_b":
        assert r1 >= 8
    else:
        assert r2 >= 8 * F.TIER2_DB


def test_selection_rule_reaches_every_kernel_shape():
    """the rates and geometries below select what the GPU tests say they do"""
    a = _args()
    assert fe_kernel(a, [48000, 16000, 8000]) == "pp"
    assert fe_kernel(a, [51200]) == "pp" and fe_kernel(a, [51250]) == "generic Q=2"
    assert fe_kernel(a, [48000, 96000]) == "generic Q=2"
    assert [fe_kernel(a, [sr]) for sr in (120000, 192000, 204800)] == ["generic Q=3", "generic Q=4", "generic Q=4"]
    assert F.hop_win(204800, a)[1] == 4096
    assert [fe_kernel(_args(ms_hop_length=h, ms_win_length=w), [sr]) for (h, w), sr in GEOMETRIES] == \
        ["generic Q=2", "generic Q=1", "pp", "pp"]
    assert F.hop_win(32000, _args(ms_hop_length=0.02, ms_win_length=0.02)) == (640, 640)


# ------------------------------------------------------------------------------------------------------------ GPU
def _engine(args):
    from nisqa_b200 import engine as E
    _, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    return eng


class Groups(object):
    """tier-1 ratios and tier-2 differences per group (kernel x format x rate)"""

    def __init__(self):
        self.r1, self.d2 = {}, {}

    def add(self, key, r1, d2):
        self.r1[key] = max(self.r1.get(key, 0.0), r1)
        self.d2.setdefault(key, []).append(d2)

    def report(self, title):
        print("\n" + title)
        bad = []
        for key in sorted(self.r1, key=str):
            r2 = F.rms(self.d2[key])
            print("  %-32s max tier-1 ratio %.3g  tier-2 RMS %.3g dB" % (" ".join(map(str, key)), self.r1[key], r2))
            if r2 > F.TIER2_DB:
                bad.append((key, r2))
        assert not bad, ("tier-2 RMS over %.3g dB" % F.TIER2_DB, bad)


def check_dump(eng, args, clips, srs, dump, groups, kernel, fmt):
    """every element of a pass's MEL_DB dump within tier 1, no extra rows; tier-2 differences to the groups"""
    assert fe_kernel(args, srs) == kernel
    off, fbs = 0, {}
    for y, sr in zip(clips, srs):
        if sr not in fbs:
            fbs[sr] = eng.mel_filterbank(sr)
        M, L, Wn = reference(y, sr, args, fbs[sr])
        got = dump[off:off + M.size].reshape(M.shape)
        off += M.size
        r1 = F.tier1_ratio(got, M, L, Wn)
        assert r1 <= 1.0, (kernel, fmt, sr, r1)
        groups.add((kernel, fmt, sr), r1, F.tier2_diffs(got, M, L, Wn))
    assert off == dump.size, (off, dump.size)


def check_call(eng, args, clips, srs, groups, kernel, fmt):
    """one pass over int16 clips (fmt "f32": as float32) checked by check_dump"""
    from nisqa_b200 import engine as E
    batch = [_f32(y) for y in clips] if fmt == "f32" else clips
    _, _, status = eng.predict_pcm(batch, srs)
    assert np.all(status == E.CLIP_OK), status
    check_dump(eng, args, clips, srs, eng.stage_dump(E.STAGE_MEL_DB), groups, kernel, fmt)


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", N_MELS)
def test_every_clip_path_instance_against_float64(built_lib, n_mels):
    """frontend_pp_kernel<T, n_mels> (a pass of 8 / 16 / 48 kHz clips) and frontend_kernel<T, n_mels> (the same clips
    with a 96 kHz clip in the pass: Q = 2) for T = int16 and float32: 4 of the 28 instances per band count"""
    args = _args(ms_n_mels=n_mels)
    groups = Groups()
    sigs = [(y, sr) for sr in (8000, 16000, 48000) for _, y in battery(sr, args, long_clip=(sr == 16000))]
    hi = [(y, 96000) for _, y in battery(96000, args)[:4]]
    covered = set()
    eng = _engine(args)
    try:
        for fmt in ("pcm16", "f32"):
            for kernel, part in (("pp", sigs), ("generic Q=2", sigs[::3] + hi)):
                clips, srs = [c for c, _ in part], [s for _, s in part]
                check_call(eng, args, clips, srs, groups, kernel, fmt)
                covered.add((kernel, fmt, n_mels))
    finally:
        eng.close()
    groups.report("%d bands:" % n_mels)
    assert len(covered) == 4


def test_the_instances_are_the_engine_band_counts():
    """7 band counts x 2 kernels x 2 formats: the 28 clip-path instances test_every_clip_path_instance covers"""
    from nisqa_b200 import engine as E
    for m in N_MELS:
        E.config_from_args(_args(ms_n_mels=m))
    with pytest.raises(NotImplementedError):
        E.config_from_args(_args(ms_n_mels=56))


def _ulp_distance(a, b):
    """max distance in float32 steps (-0 and +0 are the same point)"""
    def ordered(v):
        i = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return int(np.abs(ordered(a) - ordered(b)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("fmax", FMAXES)
def test_rates_against_float64(built_lib, fmax):
    """4 kHz .. 204.8 kHz: the pipelined kernel up to 51.2 kHz (its span limit exactly), frontend_kernel from 51.25 kHz
    (Q = 2) to 204.8 kHz (Q = 4, win == n_fft); the filterbank against librosa's in float32 ulps"""
    args = _args(ms_fmax=fmax)
    groups = Groups()
    ulps = {}
    eng = _engine(args)
    try:
        for sr in RATES:
            fb = eng.mel_filterbank(sr)
            ref = lb.mel(sr, 4096, n_mels=48, fmin=0.0, fmax=fmax, htk=False, norm="slaney")
            ulps[sr] = _ulp_distance(fb, ref)
            b = dict(battery(sr, args))
            clips = [b[k] for k in ("speech", "min_frames", "noise", "chirp", "nyquist", "loud_end")]
            for fmt in ("pcm16", "f32"):
                check_call(eng, args, clips, [sr] * len(clips), groups, fe_kernel(args, [sr]), fmt)
    finally:
        eng.close()
    print("\nfmax %d: filterbank vs librosa, max float32 ulp distance per rate: %s" % (fmax, ulps))
    groups.report("fmax %d:" % fmax)
    assert max(ulps.values()) <= 1, ulps


@pytest.mark.gpu
@pytest.mark.parametrize("geometry", GEOMETRIES, ids=["h10_w25_48k", "h15_w20_48k", "h20_w20_32k", "h5_w20_16k"])
def test_stft_geometry_from_args_against_float64(built_lib, geometry):
    """ms_hop_length / ms_win_length other than 10 / 20 ms: frontend_kernel at Q = 2 and Q = 1 (hop + win > 1536),
    the pipelined kernel with hop == win == 640 (over 512) and with a 5 ms hop"""
    (h, w), sr = geometry
    args = _args(ms_hop_length=h, ms_win_length=w)
    groups = Groups()
    b = dict(battery(sr, args))
    clips = [b[k] for k in ("speech", "min_frames", "noise", "tone_off", "impulses", "loud_end", "nyquist")]
    eng = _engine(args)
    try:
        for fmt in ("pcm16", "f32"):
            check_call(eng, args, clips, [sr] * len(clips), groups, fe_kernel(args, [sr]), fmt)
    finally:
        eng.close()
    groups.report("hop %g s, win %g s at %d Hz (%s):" % (h, w, sr, fe_kernel(args, [sr])))


@pytest.mark.gpu
def test_mixed_rate_pass_against_float64(built_lib):
    """a 48 kHz clip and a 96 kHz clip in one call: both through frontend_kernel at Q = 2"""
    args = _args()
    groups = Groups()
    clips = [synth.synth_speech_pcm16(21, 1.3, 48000), synth.synth_speech_pcm16(22, 0.9, 96000)]
    eng = _engine(args)
    try:
        for fmt in ("pcm16", "f32"):
            check_call(eng, args, clips, [48000, 96000], groups, "generic Q=2", fmt)
    finally:
        eng.close()
    groups.report("48 kHz + 96 kHz in one pass:")
    assert {k[2] for k in groups.r1} == {48000, 96000}


@pytest.mark.gpu
def test_pairs_per_cta_do_not_change_a_row(built_lib):
    """fe_ppc 1 (no prefetch), 2 (the default), 3 and 8 (the ring turns over, the last CTA of a clip takes the
    remainder): bit-identical rows for pair counts 24 (no remainder), 25 and 23"""
    from nisqa_b200 import engine as E
    args = _args()
    sr = 48000
    hop, _ = F.hop_win(sr, args)
    clips = [synth.synth_speech_pcm16(30 + i, (2 * p - 1) * hop / sr + 0.05, sr)[:(2 * p - 1) * hop]
             for i, p in enumerate((24, 25, 23))]
    clips.append(_clip16(np.random.default_rng(5).normal(0.0, 8000.0, 2 * 24 * hop - hop)))
    assert [(1 + y.size // hop + 1) // 2 for y in clips] == [24, 25, 23, 24]
    groups = Groups()
    eng = _engine(args)
    try:
        for fmt in ("pcm16", "f32"):
            rows = {}
            for ppc in (1, 2, 3, 8, 0):
                eng.set_option("fe_ppc", ppc)
                batch = [_f32(y) for y in clips] if fmt == "f32" else clips
                eng.predict_pcm(batch, [sr] * len(clips))
                rows[ppc] = eng.stage_dump(E.STAGE_MEL_DB)
            for ppc in (1, 3, 8, 0):
                np.testing.assert_array_equal(rows[ppc], rows[2], err_msg="fe_ppc=%d %s" % (ppc, fmt))
            eng.set_option("fe_ppc", 8)
            check_call(eng, args, clips, [sr] * len(clips), groups, "pp", fmt)
            eng.set_option("fe_ppc", 0)
    finally:
        eng.close()
    groups.report("fe_ppc = 8:")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["pcm16", "f32"])
def test_misaligned_device_input_equals_the_host_call(built_lib, fmt):
    """predict_pcm_device with clips at every element offset mod 16 bytes (8 int16 / 4 float32 residues), the gaps
    between them full scale (int16) or NaN (float32): scores and mel rows bit-identical to the host call, every row
    within tier 1 (no neighbouring sample leaks into a frame)"""
    import torch
    from nisqa_b200 import engine as E
    args = _args()
    sr = 48000
    n_res = 8 if fmt == "pcm16" else 4
    clips = [synth.synth_speech_pcm16(40 + i, 0.45 + 0.13 * i, sr) for i in range(n_res)]
    batch = clips if fmt == "pcm16" else [_f32(y) for y in clips]
    offs, pos = [], 64
    for i, y in enumerate(batch):
        pos = (pos + 2 * n_res) // n_res * n_res + i                 # residue i, at least one residue block of gap
        offs.append(pos)
        pos += y.size
    buf = np.empty(pos + 64, batch[0].dtype)
    if fmt == "pcm16":
        buf[:] = np.where(np.arange(buf.size) % 2 == 0, 32767, -32768).astype(np.int16)
    else:
        buf[:] = np.nan
    for o, y in zip(offs, batch):
        buf[o:o + y.size] = y
    assert sorted(o % n_res for o in offs) == list(range(n_res))
    eng = _engine(args)
    try:
        s_host, n_host, _ = eng.predict_pcm(batch, [sr] * len(batch))
        d_host = eng.stage_dump(E.STAGE_MEL_DB)
        d = torch.from_numpy(buf).cuda()
        out = torch.full((len(batch), 1), float("nan"), dtype=torch.float32, device="cuda")
        nseg, status = eng.predict_pcm_device(d.data_ptr(), offs, [y.size for y in batch], [sr] * len(batch),
                                              E.FMT_S16 if fmt == "pcm16" else E.FMT_F32, out.data_ptr(), sync=True)
        assert np.all(status == E.CLIP_OK)
        d_dev = eng.stage_dump(E.STAGE_MEL_DB)
        np.testing.assert_array_equal(nseg, n_host)
        np.testing.assert_array_equal(out.cpu().numpy(), s_host)
        np.testing.assert_array_equal(d_dev, d_host)
        groups = Groups()
        check_dump(eng, args, clips, [sr] * len(clips), d_dev, groups, "pp", fmt)
    finally:
        eng.close()
    groups.report("device input at every misalignment (%s):" % fmt)
