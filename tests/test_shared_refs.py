"""NISQA_DE pairs whose references repeat: nisqa_predict_device_batch_shared_ref, nisqa_submit_pcm_pairs,
Scorer(..., reference_index=) and predict_csv's per-batch reference sharing.

CPU: the header against the ctypes bindings, every Scorer refusal of reference_index (a stand-in engine), the
predict_csv batch plan (a stand-in engine that echoes its inputs).  GPU: bit identity with the replicated call across
every DE variant and the LSTM-td variants, several passes, work done once (stage dumps), statuses, the stream contract
and the CLI."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import de_arch_variants as DV
from oracle import nisqa_oracle as O
from oracle import variants as V

SR = 16000
LSTM_TD = [k for k in DV.DE_ARCH_VARIANTS if "lstm" in k]


# ------------------------------------------------------------------------------------------------------------ CPU
def test_header_prototypes_match_the_bindings(tmp_path):
    """gcc against the header: the two prototypes (assigned to pointers of the bound signature), the unchanged structs
    and ABI version 4"""
    src, exe = tmp_path / "p.c", tmp_path / "p"
    src.write_text(r'''#include <stdio.h>
#include "nisqa_b200.h"
int main(void) {
  int (*a)(nisqa_engine*, void*, const nisqa_device_batch*, const nisqa_device_batch*, const int32_t*, int32_t, float*,
           const nisqa_segment_out*, const nisqa_embedding_out*, const nisqa_alignment_out*, int32_t*, int32_t*, int32_t*,
           int32_t*) = nisqa_predict_device_batch_shared_ref;
  int (*b)(nisqa_engine*, int, const void* const*, const int64_t*, const int32_t*, int, const void* const*, const int64_t*,
           const int32_t*, const int32_t*, int, float*, int32_t*, int32_t*, int32_t*, int32_t*, int64_t*) = nisqa_submit_pcm_pairs;
  printf("%d %zu %zu %zu %zu %zu %d\n", NISQA_B200_ABI_VERSION, sizeof(nisqa_config), sizeof(nisqa_device_batch),
         sizeof(nisqa_segment_out), sizeof(nisqa_embedding_out), sizeof(nisqa_alignment_out), a != 0 && b != 0);
  return 0;
}
''')
    subprocess.run(["gcc", "-Werror=incompatible-pointer-types", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                    "-Wl,--unresolved-symbols=ignore-all"], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [4, C.sizeof(E.NisqaConfig), C.sizeof(E.NisqaDeviceBatch), C.sizeof(E.NisqaSegmentOut),
                   C.sizeof(E.NisqaEmbeddingOut), C.sizeof(E.NisqaAlignmentOut), 1]
    assert {"nisqa_predict_device_batch_shared_ref", "nisqa_submit_pcm_pairs"} <= set(E.EXPORTS)
    lib = E.load_library() if os.path.exists(os.path.join(ROOT, "nisqa_b200", "libnisqa_b200.so")) else None
    if lib is not None:
        assert len(lib.nisqa_predict_device_batch_shared_ref.argtypes) == 14
        assert len(lib.nisqa_submit_pcm_pairs.argtypes) == 17


class _NoEngine(object):
    """a stand-in engine: any call reaching it fails the test"""
    def __getattr__(self, name):
        raise AssertionError("the engine was reached: " + name)


def _host_scorer(double_ended=True):
    from nisqa_b200.scorer import Scorer
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    if double_ended:
        args = dict(args, model="NISQA_DE", de_align="dot", de_align_apply="hard", de_fuse="x/y/-", td_2="self_att",
                    td_2_sa_d_model=64, td_2_sa_nhead=1, td_2_sa_h=64, td_2_sa_num_layers=1, td_2_sa_pos_enc=None,
                    td_2_sa_dropout=0.1, ms_sr=None)
    sc = Scorer.__new__(Scorer)
    sc._configure(args, torch.device("cpu"))
    sc.engine = _NoEngine()
    sc._stream = lambda: 0
    return sc


def test_scorer_refusals_before_the_engine():
    sc = _host_scorer()
    deg, ref = torch.zeros(4, 16000, dtype=torch.int16), torch.zeros(2, 16000, dtype=torch.int16)
    for method in (sc.__call__, sc.segments, sc.embed):
        with pytest.raises(ValueError, match=r"reference_index: 3 entries for 4 clips"):
            method(deg, SR, reference=ref, reference_index=[0, 1, 0])
        with pytest.raises(ValueError, match=r"reference_index\[2\] = 2: not within 0 \.\. 1"):
            method(deg, SR, reference=ref, reference_index=[0, 1, 2, 0])
        with pytest.raises(ValueError, match=r"reference_index\[0\] = -1"):
            method(deg, SR, reference=ref, reference_index=np.array([-1, 0, 0, 0]))
        with pytest.raises(TypeError, match="reference_index: one int per clip"):
            method(deg, SR, reference=ref, reference_index=[0.0, 1.0, 0.0, 1.0])
        with pytest.raises(TypeError, match="reference_index: host integers"):
            method(deg, SR, reference=ref, reference_index=torch.zeros(4, dtype=torch.int64, device="meta"))
    with pytest.raises(ValueError, match=r"reference_index\[2\] = 5"):
        sc.align(deg, SR, ref, reference_index=torch.tensor([0, 1, 5, 0]))
    # a reference too short for the checkpoint: named only when a clip names it
    refs = torch.zeros(3, 16000, dtype=torch.int16)
    with pytest.raises(ValueError, match=r"reference\[2\].*too short|too short.*reference\[2\]"):
        sc(deg, SR, reference=refs, reference_lengths=[16000, 16000, 100], reference_index=[0, 2, 1, 1])
    with pytest.raises(AssertionError, match="the engine was reached"):
        sc(deg, SR, reference=refs, reference_lengths=[16000, 16000, 100], reference_index=[0, 1, 1, 0])
    # without reference_index the clip-count refusal stands
    with pytest.raises(ValueError, match="reference: 2 clips for 4 clips of wave"):
        sc(deg, SR, reference=ref)
    # windows, align(window_s=) and feeds refuse it
    with pytest.raises(ValueError, match="reference_index: windows"):
        sc.windows(deg[:2], SR, 1.0, 0.5, reference=ref, reference_index=[0, 1])
    with pytest.raises(ValueError, match=r"reference_index: align\(window_s=...\)"):
        sc.align(deg[:2], SR, ref, window_s=1.0, window_hop_s=0.5, reference_index=[0, 1])
    with pytest.raises(ValueError, match="reference_index: feed"):
        sc.feed(2, SR, 1.0, 0.5, reference=True, reference_index=[0, 1])
    # a single-ended checkpoint
    se = _host_scorer(double_ended=False)
    with pytest.raises(ValueError, match="reference_index: only a double-ended"):
        se(deg, SR, reference_index=[0, 0, 0, 0])
    with pytest.raises(ValueError, match="reference_index: only a double-ended"):
        se.embed(deg, SR, reference_index=[0, 0, 0, 0])


class _EchoEngine(object):
    """predict_csv's engine: pair p's score is its degraded clip's first sample * 1000 + its reference's first sample"""
    n_out = 1

    def __init__(self):
        self.calls = []

    def submit_pcm_pairs(self, clips, srs, refs, ref_srs, ref_index):
        self.calls.append(([int(c[0]) for c in clips], [int(r[0]) for r in refs], list(ref_index)))
        s = np.array([[float(c[0]) * 1000 + float(refs[u][0])] for c, u in zip(clips, ref_index)], np.float32)
        n = np.zeros(len(clips), np.int32)
        return (None, s, n + 5, n, np.zeros(len(refs), np.int32) + 5, np.zeros(len(refs), np.int32))

    def submit_pcm(self, clips, srs):        # (a batch whose references are all distinct: the clip pairs)
        degs, refs = clips[0::2], clips[1::2]
        h = self.submit_pcm_pairs(degs, srs[0::2], refs, srs[1::2], list(range(len(refs))))
        s = np.full((len(clips), 1), np.nan, np.float32)
        s[0::2] = h[1]
        return (None, s, np.zeros(len(clips), np.int32) + 5, np.zeros(len(clips), np.int32))

    def wait(self, h):
        return h[1], h[2], h[3]

    def drain(self):
        pass


def test_predict_csv_batch_plan(tmp_path, monkeypatch):
    import pandas as pd
    from nisqa_b200 import NISQA_lib as L
    from nisqa_b200 import wav
    # 3 references x 7 conditions, rows interleaved: reference of row i is i % 3, degraded file i holds sample value i
    rows = []
    for u in range(3):
        wav.write_wav_pcm16(str(tmp_path / ("r%d.wav" % u)), np.full(1600, 100 + u, np.int16), SR)
    for i in range(21):
        wav.write_wav_pcm16(str(tmp_path / ("d%d.wav" % i)), np.full(1600, i, np.int16), SR)
        rows.append(("d%d.wav" % i, "r%d.wav" % (i % 3)))
    df = pd.DataFrame(rows, columns=["deg", "ref"])
    ds = L.SpeechQualityDataset(df, data_dir=str(tmp_path), filename_column="deg", mos_column="predict_only",
                                double_ended=True, filename_column_ref="ref", ms_sr=None)
    decoded = []
    real = L.read_wav
    monkeypatch.setattr(L, "read_wav", lambda p, ch=None: (decoded.append(os.path.basename(p)), real(p, ch))[1])
    eng = _EchoEngine()
    out = L._predict_rows(eng, ds, np.arange(21, dtype=np.int64), 4, 0)
    # results in CSV order
    np.testing.assert_array_equal(out[:, 0], [i * 1000 + 100 + i % 3 for i in range(21)])
    # rows regrouped by reference (stable: CSV order within a reference), each distinct reference decoded once a batch
    order = [i for u in range(3) for i in range(21) if i % 3 == u]
    assert [d for c in eng.calls for d in c[0]] == order
    for degs, refs, idx in eng.calls:
        assert len(set(refs)) == len(refs) and [refs[u] - 100 for u in idx] == [d % 3 for d in degs]
    # 6 batches of 4 rows: each reference's 7 rows cross a batch boundary, so 8 reference decodes instead of 21
    assert [len(c[1]) for c in eng.calls] == [1, 2, 1, 2, 1, 1]
    assert len([d for d in decoded if d.startswith("r")]) == 8


# ------------------------------------------------------------------------------------------------------------ GPU
@functools.lru_cache(maxsize=None)
def _base(name):
    return O.load_checkpoint(os.path.join(WEIGHTS, name))


def _checkpoint(name):
    if name in V.DE_VARIANTS:
        return V.de_checkpoint(name, *_base("nisqa_mos_only.tar"))
    return DV.de_arch_checkpoint(name, *_base(DV.DE_ARCH_VARIANTS[name][0]))


def _scorer(name, tmp_path, **over):
    from nisqa_b200.scorer import Scorer
    args, sd = _checkpoint(name)
    path = str(tmp_path / (name + ".tar"))
    torch.save({"args": args, "model_state_dict": sd}, path)
    return Scorer(path, **over), args


def _wave(seed, seconds, sr, n_ch=1, f32=False):
    ch = [synth.synth_speech_pcm16(seed + 17 * c, seconds, sr) for c in range(n_ch)]
    x = torch.from_numpy(np.stack(ch))
    return (x.float() / 32768.0 if f32 else x)


def _batch(waves, f32=False):
    """-> [B, C, T] CUDA tensor (zero padded) and the lengths"""
    lens = [w.shape[-1] for w in waves]
    C_ = waves[0].shape[0]
    x = torch.zeros(len(waves), C_, max(lens), dtype=torch.float32 if f32 else torch.int16)
    for i, w in enumerate(waves):
        x[i, :, :lens[i]] = w
    return x.cuda(), lens


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _case(seed, n_pairs, n_refs, unused=(), f32=False, ref_sr=SR, n_ch=1):
    """n_pairs degraded clips (n_ch channels) and n_refs references at ref_sr, references named out of order and
    repeated; the references in `unused` are named by no pair"""
    rng = np.random.default_rng(seed)
    named = [u for u in range(n_refs) if u not in unused]
    idx = np.array([named[k] for k in rng.integers(0, len(named), n_pairs)], np.int64)
    deg = [_wave(1000 * seed + p, float(rng.uniform(1.0, 3.5)), SR, n_ch, f32) for p in range(n_pairs)]
    ref = [_wave(1000 * seed + 500 + u, float(rng.uniform(1.0, 4.0)), ref_sr, 1, f32) for u in range(n_refs)]
    (xd, ld), (xr, lr) = _batch(deg, f32), _batch(ref, f32)
    return xd, ld, xr, lr, idx


def _assert_shared_equals_replicated(sc, xd, ld, xr, lr, idx, ref_sr=SR, channel=None, embed=True):
    kw = dict(lengths=ld, channel=channel, reference_sample_rate=ref_sr)
    rep_x, rep_l = xr[torch.from_numpy(idx).cuda()], [lr[u] for u in idx]
    a = sc(xd, SR, reference=xr, reference_lengths=lr, reference_index=idx, **kw)
    b = sc(xd, SR, reference=rep_x, reference_lengths=rep_l, **kw)
    assert a.shape == b.shape and torch.equal(_bits(a), _bits(b))
    sa = sc.segments(xd, SR, reference=xr, reference_lengths=lr, reference_index=idx, **kw)
    sb = sc.segments(xd, SR, reference=rep_x, reference_lengths=rep_l, **kw)
    for f in ("scores", "seg_scores", "seg_weights"):
        assert torch.equal(_bits(getattr(sa, f)), _bits(getattr(sb, f))), f
    assert sa.counts == sb.counts
    if embed:
        ea = sc.embed(xd, SR, reference=xr, reference_lengths=lr, reference_index=idx, rows=True, **kw)
        eb = sc.embed(xd, SR, reference=rep_x, reference_lengths=rep_l, rows=True, **kw)
        for f in ("scores", "pooled", "rows"):
            assert getattr(ea, f).shape == getattr(eb, f).shape and torch.equal(_bits(getattr(ea, f)), _bits(getattr(eb, f))), f
    aa = sc.align(xd, SR, xr, reference_lengths=lr, reference_index=idx, **kw)
    ab = sc.align(xd, SR, rep_x, reference_lengths=rep_l, **kw)
    for f in ("scores", "ref_seg", "weight", "centroid", "peak"):
        assert torch.equal(_bits(getattr(aa, f)), _bits(getattr(ab, f))), f
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.DE_VARIANTS) + LSTM_TD)
def test_bit_identity_with_the_replicated_call(built_lib, tmp_path, name):
    sc, _ = _scorer(name, tmp_path)
    try:
        for k, (n_pairs, n_refs, unused) in enumerate([(12, 4, (2,)), (40, 1, ()), (9, 6, (0, 5))]):
            xd, ld, xr, lr, idx = _case(7 + k, n_pairs, n_refs, unused)
            _assert_shared_equals_replicated(sc, xd, ld, xr, lr, idx, embed=k != 1)
    finally:
        sc.close()


@pytest.mark.gpu
def test_formats_channels_rates_and_ms_sr(built_lib, tmp_path):
    sc, _ = _scorer("de_cosine_hard", tmp_path)
    try:
        xd, ld, xr, lr, idx = _case(21, 10, 3, f32=True)
        _assert_shared_equals_replicated(sc, xd, ld, xr, lr, idx)
        xd, ld, xr, lr, idx = _case(22, 10, 3, n_ch=2)                  # a channel pick on the degraded side
        _assert_shared_equals_replicated(sc, xd, ld, xr, lr, idx, channel=1)
        xd, ld, xr, lr, idx = _case(23, 10, 3, ref_sr=48000)            # references at another rate
        _assert_shared_equals_replicated(sc, xd, ld, xr, lr, idx, ref_sr=48000)
    finally:
        sc.close()
    sc, _ = _scorer("de_dot_soft", tmp_path, ms_sr=16000)
    try:
        xd, ld, xr, lr, idx = _case(24, 10, 3, ref_sr=22050, unused=(1,))
        _assert_shared_equals_replicated(sc, xd, ld, xr, lr, idx, ref_sr=22050)
    finally:
        sc.close()


@pytest.mark.gpu
def test_passes_equal_one_pass(built_lib, tmp_path):
    xd, ld, xr, lr, _ = _case(31, 30, 2)
    idx = np.array([0] * 24 + [1] * 6)
    one, _ = _scorer("de_luong_soft", tmp_path)
    try:
        a = one(xd, SR, lengths=ld, reference=xr, reference_lengths=lr, reference_index=idx)
        e1 = one.embed(xd, SR, lengths=ld, reference=xr, reference_lengths=lr, reference_index=idx)
        assert one.engine.lib.nisqa_stage_dump(one.engine.h, E.STAGE_TD1_OUT, None, 0) > 0     # (one pass)
    finally:
        one.close()
    n_seg = O.segment_counts(lr[0], SR, _checkpoint("de_luong_soft")[0])[1]
    many, _ = _scorer("de_luong_soft", tmp_path, b200_max_chunk_segments=n_seg + 5 * 120)
    try:
        b = many(xd, SR, lengths=ld, reference=xr, reference_lengths=lr, reference_index=idx)
        e2 = many.embed(xd, SR, lengths=ld, reference=xr, reference_lengths=lr, reference_index=idx)
        assert E.EngineError is not None and many.engine.lib.nisqa_stage_dump(many.engine.h, E.STAGE_TD1_OUT, None, 0) < 0
    finally:
        many.close()
    assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(e1.pooled), _bits(e2.pooled))


@pytest.mark.gpu
def test_each_reference_is_computed_once(built_lib, tmp_path):
    sc, args = _scorer("de_cosine_hard", tmp_path)
    try:
        xd, ld, xr, lr, _ = _case(41, 8, 3)
        idx = np.array([2, 0, 2, 2, 0, 2, 0, 2])                     # reference 1 unused
        sc(xd, SR, lengths=ld, reference=xr, reference_lengths=lr, reference_index=idx)
        dumps = {st: sc.engine.stage_dump(st) for st in (E.STAGE_CNN_FEAT, E.STAGE_TD1_OUT)}
        nd = [O.segment_counts(n, SR, args)[1] for n in ld]
        nr = [O.segment_counts(n, SR, args)[1] for n in lr]
        rows = sum(nd) + nr[0] + nr[2]
        # the replicated call: every pair's reference rows, in pair order
        rep = sc(xd, SR, lengths=ld, reference=xr[torch.from_numpy(idx).cuda()], reference_lengths=[lr[u] for u in idx])
        for st, d in dumps.items():
            full = sc.engine.stage_dump(st)
            width = full.size // (sum(nd) + sum(nr[u] for u in idx))
            assert d.size == rows * width
            d, full = d.reshape(rows, width), full.reshape(-1, width)
            at, at_full, seen = 0, 0, set()
            for p, u in enumerate(idx):       # slot order: pair p's degraded rows, then its reference's if new
                np.testing.assert_array_equal(d[at:at + nd[p]], full[at_full:at_full + nd[p]])
                at, at_full = at + nd[p], at_full + nd[p]
                if u not in seen:
                    np.testing.assert_array_equal(d[at:at + nr[u]], full[at_full:at_full + nr[u]])
                    at += nr[u]
                    seen.add(u)
                at_full += nr[u]
            assert at == rows
        assert rep.shape[0] == 8
    finally:
        sc.close()


@pytest.mark.gpu
def test_statuses(built_lib, tmp_path):
    sc, args = _scorer("de_dot_hard", tmp_path)
    try:
        xd, ld, xr, lr, _ = _case(51, 9, 3)
        lr[1] = 100                                                    # too short, shared by 5 pairs
        ld[7] = 120                                                    # a too-short degraded clip, reference 0
        idx = np.array([1, 0, 1, 1, 2, 1, 0, 0, 1])
        deg = E.device_batch(xd.data_ptr(), E.FMT_S16, np.array(ld, np.int64), 1, -1, xd.shape[-1], xd.stride(0),
                             xd.stride(1), SR)
        ref = E.device_batch(xr.data_ptr(), E.FMT_S16, np.array(lr, np.int64), 1, -1, xr.shape[-1], xr.stride(0),
                             xr.stride(1), SR)
        out = torch.full((9, 1), 7.0, device="cuda")
        nseg, status, rnseg, rstatus = sc.engine.predict_device_batch_shared_ref(0, deg, ref, idx, out.data_ptr())
        torch.cuda.synchronize()
        nan = torch.isnan(out[:, 0]).cpu().numpy()
        assert nan.tolist() == [u == 1 or p == 7 for p, u in enumerate(idx)]
        assert rstatus.tolist() == [E.CLIP_OK, E.CLIP_TOO_SHORT, E.CLIP_OK]
        assert status.tolist() == [E.CLIP_TOO_SHORT if p == 7 else E.CLIP_OK for p in range(9)]
        assert rnseg[1] == O.segment_counts(100, SR, args)[1] and nseg[0] == O.segment_counts(ld[0], SR, args)[1]
        with pytest.raises(ValueError, match=r"reference\[1\]"):
            sc(xd, SR, reference=xr, reference_lengths=lr, reference_index=idx)
        # engine refusals, nothing enqueued
        for bad, msg in (([0] * 8 + [3], r"ref_index\[8\] = 3"), ([0] * 8 + [-1], r"ref_index\[8\] = -1")):
            with pytest.raises(E.EngineError, match=msg):
                sc.engine.predict_device_batch_shared_ref(0, deg, ref, np.array(bad), out.data_ptr())
        with pytest.raises(E.EngineError, match="ref_index: null argument"):
            sc.engine.predict_device_batch_shared_ref(0, deg, ref, None, out.data_ptr())
        none = E.device_batch(xr.data_ptr(), E.FMT_S16, np.zeros(0, np.int64), 1, -1, xr.shape[-1], xr.stride(0),
                              xr.stride(1), SR)
        with pytest.raises(E.EngineError, match="ref: no reference clip"):
            sc.engine.predict_device_batch_shared_ref(0, deg, none, idx, out.data_ptr())
        t = torch.full((4,), 3.0, device="cuda")
        with pytest.raises(E.EngineError, match="seg->n_rows = 4"):
            sc.engine.predict_device_batch_shared_ref(0, deg, ref, idx, out.data_ptr(),
                                                      E.NisqaSegmentOut(t.data_ptr(), t.data_ptr(), 4))
        torch.cuda.synchronize()
        assert (t == 3.0).all()
    finally:
        sc.close()
    args, sd = _base("nisqa_mos_only.tar")
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    try:
        with pytest.raises(E.EngineError, match="ref_index: only a double-ended"):
            eng.predict_device_batch_shared_ref(0, deg, ref, idx, out.data_ptr())
        with pytest.raises(E.EngineError, match="ref_index: only a double-ended"):
            eng.submit_pcm_pairs([np.zeros(16000, np.int16)], [SR], [np.zeros(16000, np.int16)], [SR], [0])
    finally:
        eng.close()


@pytest.mark.gpu
def test_stream_contract(built_lib, tmp_path):
    sc, _ = _scorer("de_luong_hard", tmp_path)
    try:
        xd, ld, xr, lr, idx = _case(61, 12, 3)
        want = sc(xd, SR, lengths=ld, reference=xr, reference_lengths=lr, reference_index=idx)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            torch.cuda._sleep(20000000)                     # the inputs are written late in the stream's order
            xd2, xr2 = xd.clone(), xr.clone()
            got = sc(xd2, SR, lengths=ld, reference=xr2, reference_lengths=lr, reference_index=idx)
            del xd2, xr2                                    # freed and overwritten in stream order right after the call
            junk = torch.full_like(xd, 1234), torch.full_like(xr, -77)
            first = got.clone()
        torch.cuda.synchronize()
        assert torch.equal(_bits(first), _bits(want)) and junk[0].shape == xd.shape
    finally:
        sc.close()


@pytest.mark.gpu
def test_cli_predict_csv(built_lib, tmp_path):
    import pandas as pd
    import run_predict
    from nisqa_b200 import wav
    from nisqa_b200.NISQA_model import nisqaModel
    args, sd = _checkpoint("de_cosine_hard")
    ck = str(tmp_path / "de.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    rows, pairs = [], []
    for u in range(3):
        ref = synth.synth_speech_pcm16(70 + u, 2.5, SR)
        wav.write_wav_pcm16(str(tmp_path / ("r%d.wav" % u)), ref, SR)
    for i in range(21):
        u = (i * 2) % 3
        ref = synth.synth_speech_pcm16(70 + u, 2.5, SR)
        d = np.clip(np.roll(ref, 97 * i).astype(np.float32) * (0.5 + 0.05 * i), -32768, 32767).astype(np.int16)
        wav.write_wav_pcm16(str(tmp_path / ("d%d.wav" % i)), d, SR)
        rows.append(("d%d.wav" % i, "r%d.wav" % u))
        pairs.append((d, ref))
    pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(tmp_path / "t.csv", index=False)

    def run(csv, out):
        out.mkdir()
        a = run_predict.parse_args(["--mode", "predict_csv", "--pretrained_model", ck, "--csv_file", str(csv), "--csv_deg",
                                    "deg", "--csv_ref", "ref", "--data_dir", str(tmp_path), "--bs", "4", "--output_dir",
                                    str(out)])
        nisqaModel(a).predict()
        return pd.read_csv(out / "NISQA_results.csv")
    df = run(tmp_path / "t.csv", tmp_path / "o")
    assert df.deg.tolist() == [r[0] for r in rows]
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    try:
        clips = [c for p in pairs for c in p]
        want, _, _ = eng.wait(eng.submit_pcm(clips, [SR] * len(clips)))
    finally:
        eng.close()
    # (the CSV's decimal text of each float64 column value returns the engine's float32 score exactly)
    got = df.mos_pred.to_numpy(np.float64).astype(np.float32)
    np.testing.assert_array_equal(got.view(np.int32), want[0::2, 0].view(np.int32))
    # a too-short shared reference names the first affected row's degraded file in CSV order
    wav.write_wav_pcm16(str(tmp_path / "r1.wav"), np.zeros(200, np.int16), SR)
    first = next(r[0] for r in rows if r[1] == "r1.wav")
    with pytest.raises(ValueError) as err:
        run(tmp_path / "t.csv", tmp_path / "o2")
    assert os.path.join(str(tmp_path), first) in str(err.value)
