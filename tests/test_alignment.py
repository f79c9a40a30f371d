"""NISQA_DE's time alignment as an output (nisqa_predict_device_batch_alignment,
nisqa_predict_device_window_pairs_alignment, Scorer.align, run_predict.py --alignment).

CPU: the nisqa_alignment_out layout against gcc, the time and delay columns of Scorer.align for mixed-rate pairs and for
window pairs with a margin (on a stand-in engine that writes known rows), the CLI refusals, and the float64
restatement (oracle/alignment_oracle.py) on hand-made score rows.
GPU: every alignment variant against float64 from the engine's own TD1_OUT dump (tests/stage_ref_de.py bounds), hard
rows against the fused rows, identity pairs, unchanged scores, batching and passes, window pairs against the clip-pair
call on the cut-out windows, the refusals, the stream contract and the CLI.
"""
import ctypes as C
import functools
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import stage_ref_de as D
from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import alignment_oracle as AO
from oracle import de_arch_variants as DV
from oracle import nisqa_oracle as O
from oracle import variants as V

SR = 16000
# LSTM td variants: W = 512 (8 column chunks: soft CTAs in two blockIdx.y groups), 384 (Bahdanau, two groups), 128
ARCH = ["std_fc20_lstm256bi_l2_dot_soft", "std_fcnone_lstm192bi_l3_bahd_soft", "std_fc100_lstm64bi_cosine_hard"]


# ------------------------------------------------------------------------------------------------------------ CPU
def test_struct_layout_matches_the_header(tmp_path):
    src, exe = tmp_path / "l.c", tmp_path / "l"
    fields = [f for f, _ in E.NisqaAlignmentOut._fields_]
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(nisqa_alignment_out)'
                   + "".join(", offsetof(nisqa_alignment_out, %s)" % f for f in fields) + ");return 0;}\n")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(E.NisqaAlignmentOut)] + [getattr(E.NisqaAlignmentOut, f).offset for f in fields]


def test_stats_of_hand_made_rows():
    s = torch.tensor([[1.0, 3.0, 3.0, 0.0], [0.0, 0.0, 0.0, 0.0], [-2.0, -1.0, -5.0, -1.0]], dtype=torch.float64)
    ref_seg, w, c, peak = AO.stats(s)
    assert ref_seg.tolist() == [1, 0, 1]                       # the first maximal score
    e = torch.exp(s - s.max(1, keepdim=True)[0])
    np.testing.assert_allclose(w, 1 / e.sum(1), rtol=1e-15)
    np.testing.assert_allclose(c, (e * torch.arange(4.0, dtype=torch.float64)).sum(1) / e.sum(1), rtol=1e-15)
    assert peak.tolist() == [3.0, 0.0, -1.0]


class _FakeEngine(object):
    """writes ref_seg = 2 i + 1 and centroid = i + 0.5 for row i of an alignment call"""
    def _fill(self, al):
        n = al.n_rows
        if n:
            i = torch.arange(n, dtype=torch.float64)
            for ptr, v, dt in ((al.ref_seg, 2 * i + 1, C.c_int32), (al.centroid, i + 0.5, C.c_float)):
                arr = (dt * n).from_address(ptr)
                arr[:] = [int(x) if dt is C.c_int32 else float(x) for x in v.tolist()]

    def predict_device_batch_alignment(self, stream, deg, ref, scores_ptr, al, target_sr=0):
        self._fill(al)

    def predict_device_window_pairs_alignment(self, stream, deg, ref, scores_ptr, n_rows, W, hop_frames, margin_frames, al,
                                              target_sr=0):
        self._fill(al)


def _host_scorer(ms_sr=None):
    """a NISQA_DE Scorer on the CPU (tensors on the host, the stand-in engine): only the host arithmetic runs"""
    from nisqa_b200.scorer import Scorer
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    args = dict(args, model="NISQA_DE", de_align="dot", de_align_apply="hard", de_fuse="x/y/-", td_2="self_att",
                td_2_sa_d_model=64, td_2_sa_nhead=1, td_2_sa_h=64, td_2_sa_num_layers=1, td_2_sa_pos_enc=None,
                td_2_sa_dropout=0.1, ms_sr=ms_sr)
    sc = Scorer.__new__(Scorer)
    sc._configure(args, torch.device("cpu"))
    sc.engine = _FakeEngine()
    sc._stream = lambda: 0
    return sc


def test_times_of_mixed_rate_pairs():
    sc = _host_scorer()
    deg, ref = torch.zeros(2, 48000, dtype=torch.int16), torch.zeros(2, 22050, dtype=torch.int16)
    res = sc.align(deg, 48000, ref, lengths=[48000, 24000], reference_sample_rate=22050)
    a = sc.args
    counts = [O.segment_counts(n, 48000, a)[1] for n in (48000, 24000)]
    assert res.counts == counts and res.ref_seg.shape[0] == sum(counts)
    i = np.concatenate([np.arange(c) for c in counts]).astype(np.float64)
    r = np.arange(sum(counts), dtype=np.float64)
    step, ref_step = 4 * 480 / 48000, 4 * 220 / 22050          # seg_hop * int(sr * 0.01) / sr on each side
    np.testing.assert_allclose(res.t_start, i * step, rtol=0, atol=1e-12)
    np.testing.assert_allclose(res.ref_t_start, (2 * r + 1) * ref_step, rtol=0, atol=1e-12)
    np.testing.assert_allclose(res.delay_s, (2 * r + 1) * ref_step - i * step, rtol=0, atol=1e-12)
    np.testing.assert_allclose(res.centroid_delay_s, (r + 0.5) * ref_step - i * step, rtol=0, atol=1e-12)


def test_times_of_window_pairs_with_a_margin():
    sc = _host_scorer()
    T, T_ref, rate = 16000 * 7, 16000 * 5, 16000
    res = sc.align(torch.zeros(1, T, dtype=torch.int16), rate, torch.zeros(1, T_ref, dtype=torch.int16), window_s=3.0,
                   window_hop_s=1.0, reference_margin_s=0.5)
    W, H, M = 48000, 16000, 8000
    K = 1 + -(-(T - W) // H)
    assert res.pair_counts == [K] and len(res.counts) == K
    ok = res.pair_status == E.CLIP_OK
    assert res.counts == np.where(ok, res.pair_n_segments, 0).tolist()
    k = res.window.astype(np.int64)
    i = np.concatenate([np.arange(c) for c in res.counts]).astype(np.float64)
    r = np.arange(len(k), dtype=np.float64)
    step = 4 * 160 / rate
    np.testing.assert_allclose(res.t_start, k * H / rate + i * step, rtol=0, atol=1e-12)
    r0 = np.maximum(0, k * H - M) / rate
    np.testing.assert_allclose(res.ref_t_start, r0 + (2 * r + 1) * step, rtol=0, atol=1e-12)
    np.testing.assert_allclose(res.delay_s, r0 + (2 * r + 1) * step - (k * H / rate + i * step), rtol=0, atol=1e-12)
    np.testing.assert_allclose(res.centroid_delay_s, r0 + (r + 0.5) * step - (k * H / rate + i * step), rtol=0, atol=1e-12)
    assert (res.pair_ref_t_start == np.maximum(0, np.arange(K) * H - M) / rate).all()


def test_single_ended_and_argument_refusals():
    sc = _host_scorer()
    sc.double_ended = False
    with pytest.raises(ValueError, match="only a double-ended"):
        sc.align(torch.zeros(1, 16000, dtype=torch.int16), 16000, torch.zeros(1, 16000, dtype=torch.int16))
    sc = _host_scorer()
    with pytest.raises(ValueError, match="reference_margin_s"):
        sc.align(torch.zeros(1, 16000, dtype=torch.int16), 16000, torch.zeros(1, 16000, dtype=torch.int16),
                 reference_margin_s=0.5)
    with pytest.raises(ValueError, match="too short"):
        sc.align(torch.zeros(1, 100, dtype=torch.int16), 16000, torch.zeros(1, 16000, dtype=torch.int16))


def test_cli_refusals(monkeypatch):
    import run_predict
    from nisqa_b200 import NISQA_model as NM
    args = run_predict.parse_args(["--mode", "predict_file", "--pretrained_model", os.path.join(WEIGHTS, "nisqa.tar"),
                                   "--deg", "x.wav", "--alignment"])
    assert args["alignment"] is True
    monkeypatch.setattr(NM.nb_dist, "env_world", lambda: (0, 2, 0))
    with pytest.raises(ValueError, match="alignment: NISQA_alignment.csv is written by a single process"):
        NM.nisqaModel(dict(args))
    monkeypatch.setattr(NM.nb_dist, "env_world", lambda: (0, 1, 0))
    monkeypatch.setattr(NM.nisqaModel, "_getDevice", lambda self: setattr(self, "dev", torch.device("cpu")))
    monkeypatch.setattr(NM, "engine_from_checkpoint", lambda a, sd, device=0: None)
    with pytest.raises(ValueError, match="alignment: a single-ended checkpoint"):
        NM.nisqaModel(dict(args))


# ------------------------------------------------------------------------------------------------------------ GPU
@functools.lru_cache(maxsize=None)
def _base(name):
    return O.load_checkpoint(os.path.join(WEIGHTS, name))


def _checkpoint(name):
    if name in V.DE_VARIANTS:
        return V.de_checkpoint(name, *_base("nisqa_mos_only.tar"))
    return DV.de_arch_checkpoint(name, *_base(DV.DE_ARCH_VARIANTS[name][0]))


def _pcm(args, n_seg, seed):
    n = (15 + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * int(SR * args["ms_hop_length"])
    y = synth.synth_speech_pcm16(seed, n / SR + 0.05, SR)[:n]
    assert O.segment_counts(n, SR, args)[1] == n_seg
    return y


def _derived(ref, seed, n):
    rng = np.random.default_rng(seed)
    x = np.roll(ref.astype(np.float32), int(0.013 * SR))[:n]
    x = x * 1.6 + rng.standard_normal(len(x)).astype(np.float32) * 250.0
    return np.clip(x, -9000, 9000).astype(np.int16)


def _pairs(args):
    """-> (pairs [(deg, ref)] int16 16 kHz, index of the pair with a too-short reference): one-segment clips, references
    of one and of several 64-key blocks, a degraded clip derived from a three-block reference"""
    pairs = [(_pcm(args, a, 700 + i), _pcm(args, b, 800 + i)) for i, (a, b) in enumerate([(1, 1), (1, 130), (65, 63),
                                                                                         (64, 200)])]
    ref = _pcm(args, 150, 810)
    pairs.append((_derived(ref, 811, len(ref) * 2 // 3), ref))
    short = len(pairs)
    pairs.append((_pcm(args, 40, 812), np.zeros(100, np.int16)))
    return pairs, short


def _batch(clips):
    lens = [len(c) for c in clips]
    x = torch.zeros(len(clips), max(lens), dtype=torch.int16)
    for i, c in enumerate(clips):
        x[i, :len(c)] = torch.from_numpy(c)
    x = x.cuda()
    return x, E.device_batch(x.data_ptr(), E.FMT_S16, np.array(lens, np.int64), 1, -1, x.shape[1], x.stride(0), 0, SR)


class _Run(object):
    """one engine, its device batch calls and its dumps"""
    def __init__(self, args, sd, max_chunk_segments=0):
        self.args = args
        self.eng = E.Engine(E.config_from_args(args, max_chunk_segments=max_chunk_segments), 0)
        self.eng.load_state_dict(sd)

    def call(self, pairs, align=True, stream=0):
        xd, deg = _batch([p[0] for p in pairs])
        xr, ref = _batch([p[1] for p in pairs])
        scores = torch.empty(2 * len(pairs), 1, device="cuda")
        if not align:
            nseg, status = self.eng.predict_device_batch(stream, deg, scores.data_ptr(), ref=ref)
            torch.cuda.synchronize()
            return scores.cpu().numpy(), nseg, status
        counts = [O.segment_counts(len(d), SR, self.args)[1:] for d, _ in pairs]
        n = int(sum(c for c, st in counts if st == O.STATUS_OK))             # the rows: every OK degraded clip's segments
        outs = (torch.full((n,), 7, dtype=torch.int32, device="cuda"),) + tuple(
            torch.full((n,), 7.0, device="cuda") for _ in range(3))
        al = E.NisqaAlignmentOut(*[t.data_ptr() for t in outs], n)
        nseg, status = self.eng.predict_device_batch_alignment(stream, deg, ref, scores.data_ptr(), al)
        torch.cuda.synchronize()
        return scores.cpu().numpy(), nseg, status, [t.cpu() for t in outs]

    def close(self):
        self.eng.close()


def _row_bounds(args, sd, x, y):
    """float64 (s, row bound b_i = max_j b_ij) of one pair from td's dumped rows; s includes AttBahdanau's v bias"""
    s, b = D.scores(args, sd, x, y)
    if args["de_align"] == "bahd":
        s = s + float(sd["align.att.v.bias"])
    return s, b


def _check_rows(args, sd, x, y, got, sy):
    """the engine's four values of one pair's rows against float64 with bounds derived from the score bound b"""
    s, b = _row_bounds(args, sd, x, y)
    ref_seg, w, c, peak = (t.double() for t in got)
    cand = D.candidates(s, b)
    rows = torch.arange(x.shape[0])
    j = ref_seg.long()
    assert bool(cand[rows, j].all()), "ref_seg outside the candidates"
    bi = b.max(1)[0]
    eps = (sy + 16) * 2.0 ** -23                              # fp32 sums over the keys, exp and division
    assert bool(((peak - s[rows, j]).abs() <= b[rows, j] + 4 * 2.0 ** -24 * s[rows, j].abs() + 1e-30).all()), "peak"
    w_ref = 1.0 / torch.exp(s - s[rows, j][:, None]).sum(1)  # the weight of the engine's pick
    lo, hi = w_ref * torch.exp(-2 * bi) * (1 - eps), w_ref * torch.exp(2 * bi) * (1 + eps)
    assert bool(((w >= lo) & (w <= hi)).all()), ("weight", float((w / w_ref - 1).abs().max()))
    a = torch.softmax(s, 1)
    c_ref = a @ torch.arange(s.shape[1], dtype=torch.float64)
    tol = (torch.exp(2 * bi) * (1 + eps) ** 2 - 1) * c_ref + eps
    assert bool(((c - c_ref).abs() <= tol).all()), ("centroid", float(((c - c_ref).abs() / tol).max()))
    return float((cand.sum(1) == 1).double().mean())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(V.DE_VARIANTS) + ARCH)
def test_alignment_against_float64(built_lib, name):
    args, sd = _checkpoint(name)
    pairs, short = _pairs(args)
    run = _Run(args, sd)
    try:
        plain, nseg0, status0 = run.call(pairs, align=False)
        scores, nseg, status, got = run.call(pairs)
        ok = status == E.CLIP_OK
        has_rows = np.repeat(ok[0::2] & ok[1::2], 2)
        N = int(nseg[has_rows].sum())
        td1 = torch.from_numpy(run.eng.stage_dump(E.STAGE_TD1_OUT)).reshape(N, -1)
        fused = torch.from_numpy(run.eng.stage_dump(E.STAGE_DE_FUSED)).reshape(N, -1)
        alone = run.call(pairs[4:5])                       # the pair with a derived degraded clip, alone
    finally:
        run.close()
    np.testing.assert_array_equal(scores.view(np.int32), plain.view(np.int32))   # the scores of the plain call
    assert (nseg == nseg0).all() and (status == status0).all()
    W = td1.shape[1]
    starts = np.concatenate([[0], np.cumsum(np.where(has_rows, nseg, 0))])
    out_rows = np.concatenate([[0], np.cumsum(nseg[0::2])])              # every OK degraded clip has rows
    hard = args["de_align_apply"] == "hard"
    one = []
    for p in range(len(pairs)):
        r = slice(out_rows[p], out_rows[p + 1])
        if p == short:
            assert (got[0][r] == -1).all() and all(torch.isnan(t[r]).all() for t in got[1:])
            continue
        x, y = td1[starts[2 * p]:starts[2 * p + 1]].double(), td1[starts[2 * p + 1]:starts[2 * p + 2]].double()
        one.append(_check_rows(args, sd, x, y, [t[r] for t in got], y.shape[0]))
        if hard and args["de_fuse"] in ("x/y/-", "x/y"):    # y_al is stored as it is: the reference row ref_seg, bit for bit
            ld = (W + 63) // 64 * 64
            y_al = fused[starts[2 * p]:starts[2 * p + 1], ld:ld + W]
            assert torch.equal(y_al.view(torch.int32), td1[starts[2 * p + 1]:starts[2 * p + 2]][got[0][r].long()].view(torch.int32))
    print("\n%s: rows with one candidate %.3f" % (name, np.mean(one)))
    r = slice(out_rows[4], out_rows[5])
    for a, b in zip(alone[3], got):                          # a pair alone == the pair in the batch
        assert torch.equal(a.view(torch.int32), b[r].view(torch.int32))
    np.testing.assert_array_equal(alone[0][0], scores[8])
    run = _Run(args, sd, max_chunk_segments=200)            # several passes == one pass
    try:
        multi = run.call(pairs)
    finally:
        run.close()
    np.testing.assert_array_equal(multi[0], scores)         # (a pass of NaN pairs alone writes another NaN pattern)
    for a, b in zip(multi[3], got):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("align", ["distance", "cosine"])
def test_identity_pairs(built_lib, align):
    args, sd = V.de_checkpoint("ident_" + align, *_base("nisqa_mos_only.tar"),
                               {"de_align": align, "de_align_apply": "hard", "de_fuse": "x/y/-"})
    y = _pcm(args, 130, 901).copy()
    y[:SR] = 0                                              # a silent second: repeated rows
    run = _Run(args, sd)
    try:
        _, nseg, status, got = run.call([(y, y)])
        td1 = torch.from_numpy(run.eng.stage_dump(E.STAGE_TD1_OUT)).reshape(2 * int(nseg[0]), -1)
    finally:
        run.close()
    n = int(nseg[0])
    x = td1[:n]
    first = [int((x == x[i]).all(1).nonzero()[0]) for i in range(n)]
    if align == "distance":
        assert got[0].tolist() == first
        assert (got[3] == 0).all()
    else:
        assert float((got[3] - 1).abs().max()) <= 1e-5


def _scorer(name, tmp_path, **over):
    from nisqa_b200.scorer import Scorer
    args, sd = _checkpoint(name)
    path = str(tmp_path / (name + ".tar"))
    torch.save({"args": args, "model_state_dict": sd}, path)
    return Scorer(path, **over), args


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["de_cosine_hard", "de_dot_soft"])
def test_window_pairs_equal_the_cut_out_pairs(built_lib, tmp_path, name):
    sc, args = _scorer(name, tmp_path)
    try:
        T, T_ref = 16000 * 9 + 123, 16000 * 7 + 45
        deg = torch.from_numpy(synth.synth_speech_pcm16(31, T / SR, SR)[:T].copy()).cuda()
        ref = torch.from_numpy(synth.synth_speech_pcm16(32, T_ref / SR, SR)[:T_ref].copy()).cuda()
        res = sc.align(deg[None], SR, ref[None], window_s=4.0, window_hop_s=1.5, reference_margin_s=0.7)
        win = sc.windows(deg[None], SR, 4.0, 1.5, reference=ref[None], reference_margin_s=0.7)
        assert torch.equal(res.scores.view(torch.int32), win.scores.view(torch.int32))
        r0 = 0
        for k in range(len(res.counts)):
            a, b = int(round(win.t_start[k] * SR)), int(round(win.t_end[k] * SR))
            c, d = int(round(win.ref_t_start[k] * SR)), int(round(win.ref_t_end[k] * SR))
            n = res.counts[k]
            if win.status[k] != E.CLIP_OK:
                assert n == 0
                continue
            if win.ref_status[k] != E.CLIP_OK:
                assert (res.ref_seg[r0:r0 + n] == -1).all() and torch.isnan(res.weight[r0:r0 + n]).all()
                r0 += n
                continue
            one = sc.align(deg[a:b][None], SR, ref[c:d][None])
            for f in ("ref_seg", "weight", "centroid", "peak"):
                assert torch.equal(getattr(res, f)[r0:r0 + n].view(torch.int32), getattr(one, f).view(torch.int32)), (k, f)
            np.testing.assert_allclose(res.delay_s[r0:r0 + n], one.delay_s + (c - a) / SR, rtol=0, atol=1e-9)
            r0 += n
        assert r0 == res.ref_seg.shape[0]
    finally:
        sc.close()


@pytest.mark.gpu
def test_scores_equal_call_and_stream_contract(built_lib, tmp_path):
    sc, args = _scorer("de_luong_hard", tmp_path)
    try:
        pairs, short = _pairs(args)
        pairs = pairs[:short]
        xd, _ = _batch([p[0] for p in pairs])
        xr, _ = _batch([p[1] for p in pairs])
        lens, rlens = [len(p[0]) for p in pairs], [len(p[1]) for p in pairs]
        plain = sc(xd, SR, lengths=lens, reference=xr, reference_lengths=rlens)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            torch.cuda._sleep(20000000)                     # the inputs are written late in the stream's order
            xd2, xr2 = xd.clone(), xr.clone()
            res = sc.align(xd2, SR, xr2, lengths=lens, reference_lengths=rlens)
        torch.cuda.synchronize()
        assert torch.equal(res.scores.view(torch.int32), plain.view(torch.int32))
        again = sc.align(xd, SR, xr, lengths=lens, reference_lengths=rlens)
        for f in ("ref_seg", "weight", "centroid", "peak"):
            assert torch.equal(getattr(res, f).view(torch.int32), getattr(again, f).view(torch.int32))
    finally:
        sc.close()


@pytest.mark.gpu
def test_engine_refusals(built_lib):
    """every refusal of both entry points returns NISQA_ERR_INVALID with nothing enqueued: the outputs keep their values"""
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    y = _pcm(args, 10, 5)
    x, deg = _batch([y])
    t = torch.full((64,), 3.0, device="cuda")
    ok = E.NisqaAlignmentOut(t.data_ptr(), t.data_ptr(), t.data_ptr(), t.data_ptr(), 64)
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    try:
        with pytest.raises(E.EngineError, match="only a double-ended"):
            eng.predict_device_batch_alignment(0, deg, deg, t.data_ptr(), ok)
        with pytest.raises(E.EngineError, match="only a double-ended"):
            eng.predict_device_window_pairs_alignment(0, deg, deg, t.data_ptr(), 1, len(y), 10, 0, ok)
    finally:
        eng.close()
    args, sd = _checkpoint("de_dot_hard")
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    lib = eng.lib
    try:
        null = "al: null argument"
        rc = lib.nisqa_predict_device_batch_alignment(eng.h, None, C.byref(deg[0]), C.byref(deg[0]), 0,
                                                      C.c_void_p(t.data_ptr()), None, None, None)
        assert rc == -1 and null in eng._err()          # NISQA_ERR_INVALID
        rc = lib.nisqa_predict_device_window_pairs_alignment(eng.h, None, C.byref(deg[0]), C.byref(deg[0]), 0, len(y), 10, 0,
                                                             C.c_void_p(t.data_ptr()), 1, None, None, None, None, None)
        assert rc == -1 and null in eng._err()          # NISQA_ERR_INVALID
        for bad, msg in ((E.NisqaAlignmentOut(t.data_ptr(), None, t.data_ptr(), t.data_ptr(), 64), "null ref_seg"),
                         (E.NisqaAlignmentOut(t.data_ptr(), t.data_ptr(), t.data_ptr(), t.data_ptr(), 9), "al->n_rows = 9")):
            with pytest.raises(E.EngineError, match=msg):
                eng.predict_device_batch_alignment(0, deg, deg, t.data_ptr(), bad)
            with pytest.raises(E.EngineError, match=msg):
                eng.predict_device_window_pairs_alignment(0, deg, deg, t.data_ptr(), 1, len(y), 10, 0, bad)
        torch.cuda.synchronize()
        assert (t == 3.0).all()                               # nothing was enqueued
    finally:
        eng.close()


@pytest.mark.gpu
def test_cli_writes_the_alignment_csv(built_lib, tmp_path):
    import pandas as pd
    import run_predict
    from nisqa_b200 import wav
    from nisqa_b200.NISQA_model import nisqaModel
    args, sd = _checkpoint("de_cosine_hard")
    ck = str(tmp_path / "de.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    rows = []
    for i, sr in enumerate((16000, 48000)):
        ref = synth.synth_speech_pcm16(60 + i, 3.0, sr)
        wav.write_wav_pcm16(str(tmp_path / ("r%d.wav" % i)), ref, sr)
        wav.write_wav_pcm16(str(tmp_path / ("d%d.wav" % i)), np.roll(ref, sr // 10), sr)
        rows.append(("d%d.wav" % i, "r%d.wav" % i))
    pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(tmp_path / "t.csv", index=False)
    outs = []
    for extra in ([], ["--alignment"]):
        out = tmp_path / ("o%d" % len(outs))
        out.mkdir()
        a = run_predict.parse_args(["--mode", "predict_csv", "--pretrained_model", ck, "--csv_file", str(tmp_path / "t.csv"),
                                    "--csv_deg", "deg", "--csv_ref", "ref", "--data_dir", str(tmp_path), "--bs", "2",
                                    "--output_dir", str(out)] + extra)
        m = nisqaModel(a)
        m.predict()
        outs.append(out)
    assert (outs[0] / "NISQA_results.csv").read_bytes() == (outs[1] / "NISQA_results.csv").read_bytes()
    df = pd.read_csv(outs[1] / "NISQA_alignment.csv")
    assert list(df.columns) == ["deg", "ref", "seg", "t_start", "ref_seg", "ref_t_start", "delay_s", "weight",
                                "centroid_delay_s", "peak"]
    for i, sr in enumerate((16000, 48000)):
        d = df[df.deg == "d%d.wav" % i]
        n = O.segment_counts(3 * sr, sr, args)[1]
        assert d.seg.tolist() == list(range(n)) and d.ref_seg.between(0, n - 1).all()
        step = args["ms_seg_hop_length"] * int(sr * args["ms_hop_length"]) / sr
        np.testing.assert_allclose(d.t_start, np.arange(n) * step, rtol=0, atol=1e-9)
        np.testing.assert_allclose(d.ref_t_start, d.ref_seg * step, rtol=0, atol=1e-9)
        np.testing.assert_allclose(d.delay_s, d.ref_t_start - d.t_start, rtol=0, atol=1e-9)
        assert (d.weight > 0).all() and (d.weight <= 1).all() and (d.peak <= 1 + 1e-5).all()


@pytest.mark.gpu
def test_cli_writes_the_alignment_csv_of_window_pairs(built_lib, tmp_path):
    """--alignment with --window_s: one row per segment of every window pair's degraded window, at absolute positions;
    NISQA_windows.csv unchanged"""
    import pandas as pd
    import run_predict
    from nisqa_b200 import wav
    from nisqa_b200.NISQA_model import nisqaModel
    args, sd = _checkpoint("de_dot_soft")
    ck = str(tmp_path / "de.tar")
    torch.save({"args": args, "model_state_dict": sd}, ck)
    rows = []
    for i, (sec, ref_sec) in enumerate(((7.3, 6.0), (7.0, 2.0))):      # (pair 1: empty reference windows from k = 3)
        ref = synth.synth_speech_pcm16(70 + i, ref_sec, SR)
        wav.write_wav_pcm16(str(tmp_path / ("r%d.wav" % i)), ref, SR)
        wav.write_wav_pcm16(str(tmp_path / ("d%d.wav" % i)), synth.synth_speech_pcm16(80 + i, sec, SR), SR)
        rows.append(("d%d.wav" % i, "r%d.wav" % i))
    pd.DataFrame(rows, columns=["deg", "ref"]).to_csv(tmp_path / "t.csv", index=False)
    outs = []
    for extra in ([], ["--alignment"]):
        out = tmp_path / ("o%d" % len(outs))
        out.mkdir()
        a = run_predict.parse_args(["--mode", "predict_csv", "--pretrained_model", ck, "--csv_file", str(tmp_path / "t.csv"),
                                    "--csv_deg", "deg", "--csv_ref", "ref", "--data_dir", str(tmp_path), "--output_dir",
                                    str(out), "--window_s", "3", "--window_hop_s", "1", "--reference_margin_s", "0.5"] + extra)
        nisqaModel(a).predict()
        outs.append(out)
    assert (outs[0] / "NISQA_windows.csv").read_bytes() == (outs[1] / "NISQA_windows.csv").read_bytes()
    assert not (outs[0] / "NISQA_alignment.csv").exists()
    win = pd.read_csv(outs[1] / "NISQA_windows.csv")
    df = pd.read_csv(outs[1] / "NISQA_alignment.csv")
    assert list(df.columns) == ["deg", "ref", "window", "win_t_start", "win_ref_t_start", "seg", "t_start", "ref_seg",
                                "ref_t_start", "delay_s", "weight", "centroid_delay_s", "peak"]
    step = args["ms_seg_hop_length"] * int(SR * args["ms_hop_length"]) / SR
    empty = 0
    for f in ("d0.wav", "d1.wav"):
        w, d = win[win.deg == f].reset_index(drop=True), df[df.deg == f]
        for k in range(len(w)):
            r = d[d.window == k]
            if not np.isfinite(w.mos_pred[k]) and len(r) == 0:
                continue                                       # (a too-short degraded window: no rows)
            assert r.seg.tolist() == list(range(int(w.n_segments[k])))
            np.testing.assert_allclose(r.win_t_start, w.t_start[k], rtol=0, atol=1e-9)
            np.testing.assert_allclose(r.win_ref_t_start, w.ref_t_start[k], rtol=0, atol=1e-9)
            np.testing.assert_allclose(r.t_start, w.t_start[k] + r.seg * step, rtol=0, atol=1e-9)
            if not np.isfinite(w.mos_pred[k]):                 # a too-short or empty reference window: -1 / NaN rows
                assert (r.ref_seg == -1).all() and r.weight.isna().all() and r.delay_s.isna().all()
                empty += 1
                continue
            assert r.ref_seg.between(0, int(w.ref_n_segments[k]) - 1).all()
            np.testing.assert_allclose(r.ref_t_start, w.ref_t_start[k] + r.ref_seg * step, rtol=0, atol=1e-9)
            np.testing.assert_allclose(r.delay_s, r.ref_t_start - r.t_start, rtol=0, atol=1e-9)
    assert empty > 0


# ------------------------------------------------------------------------------------- the reference golden
GOLDEN_FILE = os.path.join(ROOT, "tests", "golden", "alignment.npz")


def _golden():
    g = np.load(GOLDEN_FILE)
    out = {}
    for k in g.files:
        name, p, f = k.split("/")
        out.setdefault(name, {}).setdefault(int(p), {})[f] = g[k]
    return out


def _golden_pairs(name):
    """the pairs oracle/make_alignment_golden.py scored for the variant"""
    pairs = V.DE_PAIRS[1:] + [((87, 2.2, 16000), (87, 3.2, 16000))]
    arch = [V.DE_PAIRS[1], ((88, 0.8, 16000), (88, 1.2, 16000))]
    return [V.de_pair_pcm(p) for p in (pairs if name in V.DE_VARIANTS else arch)]


def _against_golden(gp, ref_seg, weight, centroid, peak, delta):
    """the four values of one pair against the golden's, with delta bounding |score - golden score|: ref_seg exact wherever
    the golden's best score leads every other by more than 2 delta, else one of the keys within 2 delta of it; weight
    and centroid within the factor e^(+-2 delta) (each softmax weight moves by at most that), peak within delta.
    -> the largest |difference| / bound"""
    s = torch.from_numpy(gp["scores"]).double()
    top = s.max(1, keepdim=True)[0]
    cand = s >= top - 2 * delta
    rows = torch.arange(s.shape[0])
    j = torch.as_tensor(np.asarray(ref_seg)).long()
    assert bool(cand[rows, j].all()), "ref_seg outside the keys within 2 delta of the golden's best"
    clear = cand.sum(1) == 1
    assert bool((j[clear] == torch.from_numpy(gp["ref_seg"]).long()[clear]).all())
    g = 2.0 ** -22                                         # the golden's own float32 rounding of the four values
    f = math.expm1(2 * delta)
    w_g, c_g, p_g = (torch.from_numpy(gp[k]).double() for k in ("weight", "centroid", "peak"))
    w_ref = torch.where(clear, w_g, 1.0 / torch.exp(s - s[rows, j][:, None]).sum(1))   # (a near tie: the engine's pick)
    worst = 0.0
    for got, ref, bound in ((weight, w_ref, f * w_ref + g), (centroid, c_g, f * c_g + g * s.shape[1]),
                            (peak, s[rows, j], delta + g * s[rows, j].abs())):
        d = (torch.as_tensor(np.asarray(got)).double() - ref).abs() / bound
        worst = max(worst, float(d.max()))
    return worst


@pytest.mark.parametrize("name", sorted(_golden()))
def test_golden_matches_the_oracle_restatement(name):
    """The reference's own Alignment module (tests/golden/alignment.npz) against oracle/alignment_oracle.py in float64 on
    the oracle's td rows: the scores within delta = 2^-16 max(1, max |s|) (float32 rows and sums), the four values
    as _against_golden bounds them; hard variants' ApplyHardAttention.idx is the golden's first maximal score."""
    from oracle import de_arch_oracle as DO
    gold = _golden()[name]
    args, sd = _checkpoint(name)
    fwd = O.predict_pcm_de if name in V.DE_VARIANTS else DO.predict_pcm_de
    for p, (deg, srd, ref, srr) in enumerate(_golden_pairs(name)):
        gp = gold[p]
        taps = {}
        fwd(args, sd, deg.astype(np.float32) / 32768, srd, ref.astype(np.float32) / 32768, srr, taps)
        s = AO.scores(args, taps["de_x"], taps["de_y"], sd)
        sg = torch.from_numpy(gp["scores"]).double()
        assert s.shape == sg.shape, (name, p)
        delta = 2.0 ** -16 * max(1.0, float(sg.abs().max()))
        assert float((s - sg).abs().max()) <= delta, (name, p)
        r = _against_golden(gp, *AO.stats(s), delta)
        assert r <= 1.0, (name, p, r)
        if "idx" in gp:
            sg32 = torch.from_numpy(gp["scores"])
            first = (sg32 == sg32.max(1, keepdim=True)[0]).to(torch.float32).argmax(1).numpy()
            assert (gp["idx"] == first).all() and (gp["idx"] == gp["ref_seg"]).all(), (name, p)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_golden()))
def test_engine_against_the_reference_golden(built_lib, name):
    """the engine's alignment of the golden's pairs (each at its own rates) against the reference module's"""
    gold = _golden()[name]
    args, sd = _checkpoint(name)
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    worst = 0.0
    try:
        for p, (deg, srd, ref, srr) in enumerate(_golden_pairs(name)):
            gp = gold[p]
            sx = gp["scores"].shape[0]
            xd, bd = _batch([deg])
            xr, br = _batch([ref])
            bd[0].sample_rate, br[0].sample_rate = srd, srr
            scores = torch.empty(2, 1, device="cuda")
            outs = (torch.empty(sx, dtype=torch.int32, device="cuda"),) + tuple(torch.empty(sx, device="cuda") for _ in range(3))
            nseg, status = eng.predict_device_batch_alignment(0, bd, br, scores.data_ptr(),
                                                              E.NisqaAlignmentOut(*[t.data_ptr() for t in outs], sx))
            torch.cuda.synchronize()
            assert tuple(nseg) == gp["scores"].shape and (status == E.CLIP_OK).all(), (name, p)
            # the engine's fp32 scores and the reference's differ by their rounding and the front ends' (oracle/
            # librosa_compat.py against the engine's mel): 2^-14 max(1, max |s|)
            delta = 2.0 ** -14 * max(1.0, float(np.abs(gp["scores"]).max()))
            worst = max(worst, _against_golden(gp, *[t.cpu() for t in outs], delta))
    finally:
        eng.close()
    print("\n%s: max |engine - golden| / bound %.3g" % (name, worst))
    assert worst <= 1.0, (name, worst)
