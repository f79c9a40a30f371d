"""Live double-ended (NISQA_DE) feeds: nisqa_feed_pair_rows, nisqa_feed_pair_create / push and Scorer.feed(...,
reference=True).  CPU part: the pairs each push emits against a NumPy restatement of the window-pair definition on the
concatenated recordings (independent random chunkings of both sides within the skew bound: empty, 1-sample and max_push
pushes, skew at +-max_skew; 8 to 96 kHz; odd and even hops and margins in frames; margins of 0, one hop and more than the
window hop; references shorter than the margin, shorter than, equal to and longer than the recording, empty; ends and
slot reuse), the ring bound, the refusals and the ABI.  GPU part: every pair bit for bit what Scorer.windows(...,
reference=) gives on the whole recordings (both DE checkpoints, int16 / float32, channel pick and mix, a stereo reference,
16 / 22.05 / 48 kHz, ms_sr, front-clipped windows and both pairings, ring wrap at maximal skew both ways, several
passes, slot reuse, a side stream, two feed objects interleaved), empty references, a sample against the oracle, and the
engine's own refusals."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from nisqa_b200.scorer import FeedPairRows, FeedPairs, FeedRows, Scorer, window_geometry

gpu = pytest.mark.gpu
# the checkpoints of test_window_pairs.py: the reference's train_nisqa_double_ended.yaml shape (AdaptCNN + self-attention,
# cosine, hard) and StandardCNN + a bidirectional LSTM td with Luong soft alignment and a fusion Linear
VARIANTS = ["de_cosine_hard", "std_fc20_lstm128bi_luong_soft_fd128"]


def _checkpoint(name):
    if name in VARIANTS[:1]:
        from oracle import variants as V
        bargs, bsd = E.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
        return V.de_checkpoint(name, bargs, bsd)
    from oracle import de_arch_variants as V
    base = V.DE_ARCH_VARIANTS[name][0]
    bargs, bsd = E.load_checkpoint(os.path.join(WEIGHTS, base))
    return V.de_arch_checkpoint(name, bargs, bsd)


_ARGS = {}


def _de_args():
    if "de" not in _ARGS:
        _ARGS["de"] = _checkpoint("de_cosine_hard")[0]
    return _ARGS["de"]


def _host_scorer(args):
    s = Scorer.__new__(Scorer)
    s._configure(args, torch.device("cpu"))
    s.engine = None
    return s


def _definition(args, T, T_ref, rate, W, H, M):
    """the definition on the concatenated recordings: pair index, degraded / reference window bounds, segment counts and
    statuses of both windows (no pair when T == 0)"""
    hop = int(rate * args["ms_hop_length"])
    K = 0 if T == 0 else 1 if T <= W else 1 + -(-(T - W) // H)
    k = np.arange(K, dtype=np.int64)
    d0, d1 = k * H, np.minimum(k * H + W, T)
    r0 = np.maximum(0, k * H - M)
    r1 = np.maximum(r0, np.minimum(T_ref, k * H + W + M))

    def counts(n):
        n_wins = np.where(n < 1, 0, 1 + n // hop - (args["ms_seg_length"] - 1))
        n_seg = np.where(n_wins < 1, 0, -(-n_wins // args["ms_seg_hop_length"]))
        st = np.where(n_wins < 1, E.CLIP_TOO_SHORT, np.where(n_seg > args["ms_max_segments"], E.CLIP_TOO_LONG, E.CLIP_OK))
        return n_seg, st
    return (k, d0, d1, r0, r1) + counts(d1 - d0) + counts(r1 - r0)


def _plan(pairs, rng, max_push, max_skew):
    """independent random chunkings of both sides of recording pairs [(T, T_ref), ...] per feed, played back to back,
    within the skew bound: [(n_samples, ref_n_samples, end)] pushes.  A side gets 0, 1, max_push or any number of samples,
    and often as many as puts the skew at exactly +max_skew or -max_skew; a feed ends with the push that completes both
    sides"""
    B = len(pairs)
    left = [list(p) for p in pairs]
    pos = [[0, 0] for _ in range(B)]
    pushes = []
    while any(left):
        ns, rns, ends = np.zeros(B, np.int64), np.zeros(B, np.int64), np.zeros(B, np.uint8)
        for b in range(B):
            if not left[b]:
                continue
            T, Tr = left[b][0]
            pd, pr = pos[b]
            hi_d = min(max_push, T - pd)
            c = (0, 1, max_push, int(rng.integers(0, max_push + 1)), int(rng.integers(0, max(2, max_push // 10))))
            nd = min(c[rng.integers(0, 5)], hi_d)
            lo = max(0, pd + nd - pr - max_skew)
            hi = min(max_push, Tr - pr, pd + nd - pr + max_skew)
            if lo > hi:
                nd = 0
                lo, hi = max(0, pd - pr - max_skew), min(max_push, Tr - pr, pd - pr + max_skew)
            nr = (lo, hi, int(rng.integers(lo, hi + 1)), min(max(lo, 1), hi))[rng.integers(0, 4)]
            ns[b], rns[b] = nd, nr
            pos[b] = [pd + nd, pr + nr]
            if pos[b] == [T, Tr]:
                ends[b] = 1
                left[b].pop(0)
                pos[b] = [0, 0]
        pushes.append((ns, rns, ends))
    return pushes


# ------------------------------------------------------------------ CPU
def _rings(W, max_push, M, max_skew):
    """the ring lengths nisqa_feed_pair_create allocates (degraded, reference)"""
    return W + max_push + M + max_skew, W + max_push + M + max(M, max_skew)


@pytest.mark.parametrize("rate", [8000, 16000, 22050, 44100, 48000, 96000])
def test_pair_rows_follow_the_definition(built_lib, rate):
    args = _de_args()
    cfg = E.config_from_args(args)
    hop = int(rate * args["ms_hop_length"])
    rng = np.random.default_rng(rate)
    for window_s, window_hop_s in ((10.0, 1.0), (3.0, 0.37), (3.0, 2.9)):
        W, hf = window_geometry(args, rate, window_s, window_hop_s)
        H = hf * hop
        for mf in (0, 1, 2, hf + 3):                  # none, one hop (odd), even, more than the window hop
            M = mf * hop
            for max_push, max_skew in ((1 + W // 7, W // 5), (W, 0), (W // 3, 2 * W)):
                # references shorter than the margin, shorter than, equal to and longer than the recording, empty ones
                # and empty recordings; feed b plays its pairs back to back (slot reuse)
                cand = [(W - 1, max(1, M // 2)), (3 * W + 7, 2 * W), (W, W), (2 * W + 11, 2 * W + 11 + max_skew),
                        (int(2.3 * W), 0), (0, 1), (1, 1)]
                pairs = [[p for p in cand[i::3] if abs(p[0] - p[1]) <= max_skew] for i in range(3)]
                R_d, R_r = _rings(W, max_push, M, max_skew)
                held, rheld = np.zeros(3, np.int64), np.zeros(3, np.int64)
                got = [[] for _ in range(3)]
                cur = [[] for _ in range(3)]
                for ns, rns, ends in _plan(pairs, rng, max_push, max_skew):
                    feed, index, nseg, st, rnseg, rst = E.feed_pair_rows(cfg, rate, W, hf, mf, held, rheld, ns, rns, ends)
                    assert np.all(np.diff(feed) >= 0)
                    T, Tr = held + ns, rheld + rns
                    assert np.all(np.abs(T - Tr) <= max_skew)
                    for f, k, a, b, c, d in zip(feed, index, nseg, st, rnseg, rst):
                        cur[f].append((k, a, b, c, d, held[f], rheld[f], T[f], Tr[f], bool(ends[f])))
                    for f in range(3):             # no pair of this push reads a ring position this push overwrites
                        ks = index[feed == f]
                        if ks.size and ns[f]:
                            assert T[f] - 1 - ks.min() * H < R_d
                        if ks.size and rns[f]:
                            assert Tr[f] - 1 - max(0, ks.min() * H - M) < R_r
                    for b in np.nonzero(ends)[0]:
                        got[b].append(cur[b])
                        cur[b] = []
                    held, rheld = np.where(ends.astype(bool), 0, T), np.where(ends.astype(bool), 0, Tr)
                what = str((rate, window_s, window_hop_s, mf, max_push, max_skew))
                for b in range(3):
                    assert len(got[b]) == len(pairs[b]), what
                    for (T, Tr), rows in zip(pairs[b], got[b]):
                        k, _, _, _, _, ns_, st_, rns_, rst_ = _definition(args, T, Tr, rate, W, H, M)
                        for j, want in enumerate((k, ns_, st_, rns_, rst_)):
                            np.testing.assert_array_equal([r[j] for r in rows], want, err_msg=what)
                        for kk, _, _, _, _, hd, hr, ad, ar, ended in rows:
                            # the first push after which both sides are complete, or the ending push
                            assert not (hd >= kk * H + W and hr >= kk * H + W + M), what
                            assert ended or (ad >= kk * H + W and ar >= kk * H + W + M), what


def test_rows_of_empty_ended_and_one_sample_pushes(built_lib):
    args = _de_args()
    cfg = E.config_from_args(args)
    W, hf = window_geometry(args, 48000, 10.0, 1.0)
    mf, M, z = 50, 24000, np.zeros(2, np.int64)
    assert E.feed_pair_rows(cfg, 48000, W, hf, mf, z, z, z, z, None)[0].shape == (0,)
    assert E.feed_pair_rows(cfg, 48000, W, hf, mf, z, z, z, z, [1, 1])[0].shape == (0,)     # ended with no sample
    held, rheld = np.array([W - 1, W], np.int64), np.array([W + M, W + M - 1], np.int64)
    feed, index = E.feed_pair_rows(cfg, 48000, W, hf, mf, held, rheld, np.array([1, 0]), np.array([0, 0]))[:2]
    assert feed.tolist() == [0] and index.tolist() == [0]                # the degraded side was the slower one
    feed, index = E.feed_pair_rows(cfg, 48000, W, hf, mf, held, rheld, np.array([0, 0]), np.array([0, 1]))[:2]
    assert feed.tolist() == [1] and index.tolist() == [0]                # the reference side was
    # Tr == 0 at end: every pair of the degraded recording, NaN references (CLIP_TOO_SHORT)
    r = E.feed_pair_rows(cfg, 48000, W, hf, mf, np.array([3 * W]), np.array([0]), np.array([0]), np.array([0]), [1])
    assert r[1].tolist() == list(range(21)) and (r[5] == E.CLIP_TOO_SHORT).all() and (r[3] == E.CLIP_OK).all()
    # Td == 0 at end: none
    r = E.feed_pair_rows(cfg, 48000, W, hf, mf, np.array([0]), np.array([500]), np.array([0]), np.array([7]), [1])
    assert r[0].shape == (0,)


def _fake_feed(sc, **kw):
    class _Eng(object):
        def feed_pair_create(self, *a):
            return 1

        def feed_pair_push(self, *a):
            raise AssertionError("a refused push reached the engine")
    sc.engine = _Eng()
    return sc.feed(3, 48000, 10.0, 1.0, reference=True, **kw)


def test_refusals_name_the_argument(built_lib):
    de = _host_scorer(_de_args())
    se = _host_scorer(E.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))[0])
    with pytest.raises(ValueError, match="NISQA_DE"):                  # unchanged: a DE checkpoint without reference=
        de.feed(4, 48000, 10.0, 1.0)
    with pytest.raises(ValueError, match="reference"):
        se.feed(4, 48000, 10.0, 1.0, reference=True)
    with pytest.raises(ValueError, match="reference_margin_s"):
        se.feed(4, 48000, 10.0, 1.0, reference_margin_s=0.5)
    with pytest.raises(ValueError, match="reference_margin_s"):
        de.feed(4, 48000, 10.0, 1.0, reference_margin_s=0.5)           # a margin without reference=True
    with pytest.raises(ValueError, match="max_skew_s"):
        se.feed(4, 48000, 10.0, 1.0, max_skew_s=1.0)
    with pytest.raises(TypeError, match="reference"):
        de.feed(4, 48000, 10.0, 1.0, reference=1)
    for bad in (-0.5, float("nan"), True, "1", None):
        with pytest.raises(ValueError, match="reference_margin_s"):
            de.feed(4, 48000, 10.0, 1.0, reference=True, reference_margin_s=bad)
    for bad in (-0.5, float("nan"), True, "1"):
        with pytest.raises(ValueError, match="max_skew_s"):
            de.feed(4, 48000, 10.0, 1.0, reference=True, max_skew_s=bad)
    with pytest.raises(ValueError, match="reference_margin_s"):
        de.feed(4, 48000, 10.0, 1.0, reference=True, reference_margin_s=25.0)    # 60 s reference windows
    # what Scorer.feed refuses
    for bad in (0, 65536, 2.0, True):
        with pytest.raises(ValueError, match="n_feeds"):
            de.feed(bad, 48000, 10.0, 1.0, reference=True)
    with pytest.raises(ValueError, match="sample_rate"):
        de.feed(4, 0, 10.0, 1.0, reference=True)
    with pytest.raises(ValueError, match="window_hop_s"):
        de.feed(4, 48000, 5.0, 6.0, reference=True)
    with pytest.raises(ValueError, match="window_s"):
        de.feed(4, 48000, 60.0, 1.0, reference=True)
    with pytest.raises(ValueError, match="max_push_s"):
        de.feed(4, 48000, 10.0, 1.0, reference=True, max_push_s=0)
    with pytest.raises(TypeError, match="channel"):
        de.feed(4, 48000, 10.0, 1.0, reference=True, channel="left")
    ms = _host_scorer(dict(_de_args(), ms_sr=16000))
    with pytest.raises(ValueError, match="sample_rate.*ms_sr"):
        ms.feed(4, 48000, 10.0, 1.0, reference=True)
    # push: checked before anything reaches the engine
    fd = _fake_feed(_host_scorer(_de_args()), max_push_s=0.5, max_skew_s=0.25, reference_margin_s=0.5)
    assert isinstance(fd, FeedPairs) and (fd.max_push, fd.max_skew, fd.margin) == (24000, 12000, 24000)
    assert _fake_feed(_host_scorer(_de_args()), max_push_s=0.5).max_skew == 24000            # default: max_push_s
    x = torch.zeros((3, 30000), dtype=torch.int16)
    with pytest.raises(ValueError, match="reference"):
        fd.push(x[:, :100], x[:2, :100])                            # 2 feeds for 3
    with pytest.raises(ValueError, match="wave"):
        fd.push(x[:2, :100], x[:, :100])
    with pytest.raises(ValueError, match="reference_lengths"):
        fd.push(x[:, :100], x)                                      # 30000 samples > max_push
    with pytest.raises(ValueError, match="lengths"):
        fd.push(x, x[:, :100])
    with pytest.raises(ValueError, match="reference_lengths"):
        fd.push(x[:, :100], x[:, :100], reference_lengths=[1, -1, 0])
    with pytest.raises(ValueError, match="reference_lengths"):
        fd.push(x[:, :100], x[:, :0], reference_lengths=[1, 0, 0])
    with pytest.raises(ValueError, match="end"):
        fd.push(x[:, :100], x[:, :100], end=[True, False])
    with pytest.raises(TypeError, match="reference"):
        fd.push(x[:, :100], x[:, :100].double())
    with pytest.raises(ValueError, match="lengths / reference_lengths"):
        fd.push(x[:, :24000], x[:, :0])                             # skew 24000 > 12000
    fd.held[:], fd.ref_held[:] = [20000, 0, 0], [10000, 0, 0]       # (the state pushes would leave: skew +10000)
    fd._fmt = E.FMT_S16
    with pytest.raises(ValueError, match="lengths / reference_lengths"):
        fd.push(x[:, :3000], x[:, :0], lengths=[3000, 0, 0], end=[True, False, False])    # before the end's reset
    with pytest.raises(ValueError, match="lengths / reference_lengths"):
        fd.push(x[:, :0], x[:, :23000], reference_lengths=[23000, 0, 0])    # -13000
    # one format for both sides while a feed holds samples on either side
    with pytest.raises(ValueError, match="wave / reference.*int16"):
        fd.push(x[:, :100], x[:, :100].float())
    with pytest.raises(ValueError, match="wave / reference.*int16"):
        fd.push(x[:, :100], torch.zeros((3, 2, 100), dtype=torch.int16))   # a stereo reference is mixed: float32
    fd.held[:], fd.ref_held[:] = 0, [0, 0, 7]
    with pytest.raises(ValueError, match="wave / reference.*int16"):
        fd.push(x[:, :100].float(), x[:, :0])


def test_header_exports_and_binding_agree(built_lib):
    header = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    lib = E.load_library()
    syms = ("nisqa_feed_pair_create", "nisqa_feed_pair_rows", "nisqa_feed_pair_push")
    for sym in syms:
        assert sym + "(" in header and sym in E.EXPORTS and hasattr(lib, sym)
    assert [len(getattr(lib, s).argtypes) for s in syms] == [9, 19, 13]
    assert FeedPairRows._fields == FeedRows._fields + ("ref_t_start", "ref_t_end", "ref_n_segments", "ref_status")
    assert "#define NISQA_B200_ABI_VERSION 4" in header
    cfg = E.config_from_args(_de_args())
    n = ctypes.c_int64()
    z = (ctypes.c_int64 * 1)(0)
    neg = (ctypes.c_int64 * 1)(-1)
    for window, hf, mf, rheld in ((480000, 1001, 0, z), (480000, 100, -1, z), (480000, 100, 3000, z), (0, 1, 0, z),
                                  (480000, 100, 0, neg)):
        assert lib.nisqa_feed_pair_rows(ctypes.byref(cfg), 48000, window, hf, mf, 1, z, rheld, z, z, None,
                                        ctypes.byref(n), None, None, None, None, None, None, 0) == -1


# ------------------------------------------------------------------ GPU
_SCORERS = {}


@pytest.fixture(scope="module", autouse=True)
def _close_scorers():
    """the engines of this module hold their pass workspaces: freed for the modules after it"""
    yield
    for sc in _SCORERS.values():
        sc.close()
    _SCORERS.clear()


def _scorer(name, tmp_path_factory, **over):
    key = (name, tuple(sorted(over.items())))
    if key not in _SCORERS:
        path = tmp_path_factory.getbasetemp() / (name + ".tar")
        if not path.exists():
            args, sd = _checkpoint(name)
            torch.save({"args": args, "model_state_dict": sd}, path)
        _SCORERS[key] = Scorer(str(path), **over)
    return _SCORERS[key]


def _pair(sec, sr, ref_sec=None, seed=0):
    """(degraded, reference) int16 as test_window_pairs.py makes them: the degraded one the reference delayed by 0.12 s,
    attenuated and noisy"""
    rs = sec if ref_sec is None else ref_sec
    ref = synth.synth_speech_pcm16(3000 + seed, max(rs, 0.5), sr)[:int(rs * sr)]
    n = int(sec * sr)
    d = np.zeros(n, np.float32)
    lag = int(0.12 * sr)
    src = ref[:max(0, n - lag)].astype(np.float32) * 0.7
    d[lag:lag + src.shape[0]] = src
    d += np.random.default_rng(seed).normal(0, 300, n).astype(np.float32)
    return np.clip(d, -32768, 32767).astype(np.int16), ref


class _Player(object):
    """pushes the recording pairs recs[b] (lists of ([T] or [C, T], [T_ref] or [C, T_ref]) CUDA tensor pairs, played back
    to back) to a pair feed object and collects each feed's rows, recording pair by recording pair"""

    def __init__(self, fd, recs):
        self.fd, self.queue = fd, [list(r) for r in recs]
        B = len(recs)
        self.pos, self.cur, self.out = [[0, 0] for _ in range(B)], [[] for _ in range(B)], [[] for _ in range(B)]
        self.x0 = next(q[0] for q in self.queue if q)

    def _chunk(self, side, ns):
        B = len(self.queue)
        t = self.x0[side]
        c = torch.zeros((B,) + tuple(t.shape[:-1]) + (max(int(ns.max()), 1),), dtype=t.dtype, device=t.device)
        for b in range(B):
            if ns[b]:
                p = self.pos[b][side]
                c[b, ..., :ns[b]] = self.queue[b][0][side][..., p:p + ns[b]]
        return c

    def push(self, ns, rns, ends):
        r = self.fd.push(self._chunk(0, ns), self._chunk(1, rns), lengths=ns, reference_lengths=rns, end=ends)
        for i, f in enumerate(r.feed):
            self.cur[f].append((r.scores[i],) + tuple(getattr(r, n)[i] for n in FeedPairRows._fields[2:]))
        for b in range(len(self.queue)):
            self.pos[b][0] += int(ns[b])
            self.pos[b][1] += int(rns[b])
            if ends[b]:
                self.out[b].append(self.cur[b])
                self.cur[b] = []
                self.queue[b].pop(0)
                self.pos[b] = [0, 0]

    def result(self):
        """per feed, per recording pair: (scores, index, t_start, ..., ref_status) of its rows"""
        torch.cuda.synchronize()
        res = []
        for b in range(len(self.out)):
            res.append([])
            for rows in self.out[b]:
                sc = torch.stack([r[0] for r in rows]).cpu().numpy() if rows else np.zeros((0, 1), np.float32)
                res[b].append((sc,) + tuple(np.array([r[j] for r in rows]) for j in range(1, 10)))
        return res


def _replay(fd, recs, pushes):
    pl = _Player(fd, recs)
    for ns, rns, ends in pushes:
        pl.push(ns, rns, ends)
    return pl.result()


def _check(sc, recs, rate, window_s, window_hop_s, margin_s, seed, channel=None, max_push_s=2.0, max_skew_s=None,
           pushes=None):
    """every feed's pairs, recording pair by recording pair, equal Scorer.windows(..., reference=) on the whole
    recordings -> the rows"""
    rng = np.random.default_rng(seed)
    fd = sc.feed(len(recs), rate, window_s, window_hop_s, channel=channel, max_push_s=max_push_s, reference=True,
                 reference_margin_s=margin_s, max_skew_s=max_skew_s)
    try:
        if pushes is None:
            pushes = _plan([[(x.shape[-1], r.shape[-1]) for x, r in rr] for rr in recs], rng, fd.max_push, fd.max_skew)
        got = _replay(fd, recs, pushes)
    finally:
        fd.close()
    for b, rr in enumerate(recs):
        for (x, r), rows in zip(rr, got[b]):
            one = lambda t: t if t.dim() == 1 else t[None]        # noqa: E731
            w = sc.windows(one(x), rate, window_s, window_hop_s, channel=channel, reference=one(r),
                           reference_margin_s=margin_s)
            what = str((rate, window_s, window_hop_s, margin_s, channel, x.shape, r.shape))
            assert w.counts == [len(rows[1])], what
            np.testing.assert_array_equal(rows[1], np.arange(len(rows[1])), err_msg=what)
            np.testing.assert_array_equal(rows[0], w.scores.cpu().numpy(), err_msg=what)
            for j, f in enumerate(FeedPairRows._fields[3:]):
                np.testing.assert_array_equal(rows[2 + j], getattr(w, f), err_msg=what + " " + f)
    return got


def _cuda(*a):
    return tuple(torch.from_numpy(x).cuda() for x in a)


@gpu
@pytest.mark.parametrize("name", VARIANTS)
def test_pair_feeds_equal_window_pairs_bit_for_bit(built_lib, tmp_path_factory, name):
    sc = _scorer(name, tmp_path_factory)
    recs = [[_cuda(*_pair(sec, 48000, rsec, seed=i))] for i, (sec, rsec) in enumerate(((25.0, 26.0), (61.0, 60.0),
                                                                                        (8.0, 9.5)))]
    # 100 frames and a margin of 50 (even / even: one pairing), 333 (odd) frames and 25 (odd)
    _check(sc, recs, 48000, 10.0, 1.0, 0.5, seed=1, max_push_s=2.0, max_skew_s=2.0)
    if name == VARIANTS[0]:
        _check(sc, recs, 48000, 10.0, 3.33, 0.25, seed=2, max_push_s=2.0, max_skew_s=2.0)
        _check(sc, recs, 48000, 10.0, 1.0, 0.0, seed=3, max_push_s=2.0, max_skew_s=2.0)


@gpu
def test_other_inputs_equal_window_pairs(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    d1, r1 = _pair(22.0, 48000, seed=4)
    d2, r2 = _pair(22.0, 48000, seed=5)
    xs = torch.from_numpy(np.stack([d1, d2]).astype(np.float32) / 32768.0).cuda()      # float32 stereo
    ys16 = torch.from_numpy(np.stack([r1, r2])).cuda()                                   # int16 stereo reference
    for channel in (1, None):                # a degraded channel and its mix; the stereo reference forces float32
        _check(sc, [[(xs, ys16)], [(xs[:, :500000].contiguous(), ys16[:, :520000].contiguous())]], 48000, 10.0, 1.0, 0.5,
               seed=6, channel=channel)
    st16 = torch.from_numpy(np.stack([d1, d2])).cuda()
    _check(sc, [[(st16, torch.from_numpy(r1).cuda())]], 48000, 10.0, 1.0, 0.3, seed=7, channel=0)   # int16 rings
    # 16 kHz: an even hop (100 frames) with an odd margin (5 frames: the uniform windows pair odd frames), and a margin
    # longer than the hop (150 frames: two front-clipped windows)
    d, r = _pair(30.0, 16000, 28.0, seed=8)
    for margin_s in (0.05, 1.5):
        _check(sc, [[_cuda(d, r)]], 16000, 8.0, 1.0, margin_s, seed=9)
    # 22.05 kHz: an odd hop (37 frames: both pairings), an odd margin, and a margin longer than the hop
    d, r = _pair(20.0, 22050, 23.0, seed=10)
    for margin_s in (0.07, 0.9):
        _check(sc, [[_cuda(d, r)], [_cuda(d[:150000], r[:140000])]], 22050, 5.0, 0.37, margin_s, seed=11, max_skew_s=3.0)
    # references shorter than the margin and shorter than a window: clipped, too-short and empty reference windows
    d, r = _pair(20.0, 16000, 1.2, seed=12)
    got = _check(sc, [[_cuda(d, r)]], 16000, 5.0, 1.0, 2.0, seed=13, max_push_s=20.0, max_skew_s=20.0)
    assert (got[0][0][9] == E.CLIP_TOO_SHORT).any() and (got[0][0][9] == E.CLIP_OK).any()


@gpu
def test_ms_sr_checkpoint_fed_at_ms_sr(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory, ms_sr=16000)
    d, r = _pair(25.0, 16000, 24.0, seed=14)
    f = lambda a: torch.from_numpy(a.astype(np.float32) / 32768.0).cuda()    # noqa: E731  (windows convert to float32)
    _check(sc, [[(f(d), f(r))]], 16000, 10.0, 1.0, 0.5, seed=15)


@gpu
def test_ring_wrap_at_maximal_skew(built_lib, tmp_path_factory):
    # pushes of exactly max_push, one side max_skew ahead of the other for the whole recording, then the other way round;
    # both rings wrap many times (max_push 0.5 s, max_skew 1 s: rings of 12 s + 2 M)
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    rate, mp, sk = 16000, 8000, 16000
    d, r = _pair(47.0, rate, 47.0, seed=16)
    T = d.shape[0]
    for lead in (0, 1):                      # 0: the degraded side leads by max_skew, 1: the reference side
        pushes, pos = [], [0, 0]
        while pos != [T, T]:
            n = [0, 0]
            n[lead] = min(mp, T - pos[lead])
            ahead = pos[lead] + n[lead]              # the other side follows max_skew behind, then catches up
            n[1 - lead] = min(mp, T - pos[1 - lead], T if ahead == T else max(0, ahead - sk - pos[1 - lead]))
            pos = [pos[0] + n[0], pos[1] + n[1]]
            pushes.append((np.array([n[0]]), np.array([n[1]]), np.array([int(pos == [T, T])], np.uint8)))
        assert max(abs(sum(int(p[0][0]) for p in pushes[:i]) - sum(int(p[1][0]) for p in pushes[:i]))
                   for i in range(len(pushes) + 1)) == sk
        for margin_s in (0.0, 0.5):
            _check(sc, [[_cuda(d, r)]], rate, 10.0, 1.0, margin_s, seed=0, max_push_s=0.5, max_skew_s=1.0, pushes=pushes)


@gpu
def test_passes_ends_and_slot_reuse(built_lib, tmp_path_factory):
    small = _scorer("de_cosine_hard", tmp_path_factory, b200_max_chunk_segments=600)
    x, y = _cuda(*_pair(40.0, 48000, 41.0, seed=17))
    fd = small.feed(1, 48000, 10.0, 1.0, max_push_s=41.0, reference=True, reference_margin_s=0.5, max_skew_s=1.0)
    rr = fd.push(x[None], y[None], end=[True])
    torch.cuda.synchronize()
    fd.close()
    assert small.engine.lib.nisqa_stage_dump(small.engine.h, E.STAGE_MEL_DB, None, 0) < 0      # (it ran in passes)
    w = small.windows(x, 48000, 10.0, 1.0, reference=y, reference_margin_s=0.5)
    np.testing.assert_array_equal(rr.scores.cpu().numpy(), w.scores.cpu().numpy())
    # several recording pairs per feed, ending with T_ref < T and T_ref > T
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    recs = [[_cuda(*_pair(s, 48000, rs, seed=18 + i)) for i, (s, rs) in enumerate(((17.0, 15.5), (3.0, 4.0), (24.0, 25.0)))],
            [_cuda(*_pair(s, 48000, rs, seed=22 + i)) for i, (s, rs) in enumerate(((12.5, 13.0), (31.0, 29.5)))]]
    _check(sc, recs, 48000, 10.0, 1.0, 0.5, seed=19)
    _check(sc, recs, 48000, 10.0, 3.33, 1.3, seed=20)


@gpu
def test_empty_reference_scores_nan(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    x, y = _cuda(*_pair(12.0, 48000, seed=23))
    fd = sc.feed(2, 48000, 10.0, 1.0, max_push_s=12.0, reference=True, reference_margin_s=0.5, max_skew_s=12.0)
    try:
        both = torch.stack([x, x])
        r = fd.push(both, torch.stack([y, y]), lengths=[x.shape[0], x.shape[0]], reference_lengths=[0, y.shape[0]],
                    end=[True, True])
        torch.cuda.synchronize()
    finally:
        fd.close()
    a = r.feed == 0
    assert r.index[a].tolist() == list(range(3))                       # 12 s: windows at 0, 1 and 2 s
    assert (r.ref_status[a] == E.CLIP_TOO_SHORT).all() and (r.ref_n_segments[a] == 0).all()
    assert (r.status[a] == E.CLIP_OK).all() and np.isnan(r.scores.cpu().numpy()[a]).all()
    np.testing.assert_array_equal(r.ref_t_end[a], r.ref_t_start[a])
    w = sc.windows(x, 48000, 10.0, 1.0, reference=y, reference_margin_s=0.5)
    np.testing.assert_array_equal(r.scores.cpu().numpy()[~a], w.scores.cpu().numpy())


@gpu
def test_stream_order_and_interleaved_feeds(built_lib, tmp_path_factory):
    sc = _scorer("de_cosine_hard", tmp_path_factory)
    recs = [[_cuda(*_pair(s, 48000, rs, seed=30 + i))] for i, (s, rs) in enumerate(((23.0, 24.0), (17.0, 16.0)))]
    pushes = _plan([[(r[0][0].shape[-1], r[0][1].shape[-1])] for r in recs], np.random.default_rng(21), 48000, 48000)

    def run(hop_s, stream=None):
        fd = sc.feed(2, 48000, 10.0, hop_s, max_push_s=1.0, reference=True, reference_margin_s=0.5)
        try:
            if stream is None:
                return _replay(fd, recs, pushes)
            with torch.cuda.stream(stream):
                return _replay(fd, recs, pushes)
        finally:
            fd.close()

    def same(a, b):
        for fa, fb in zip(a, b):
            for ra, rb in zip(fa, fb):
                for u, v in zip(ra, rb):
                    np.testing.assert_array_equal(u, v)

    alone = [run(1.0), run(5.0)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    same(run(1.0, s), alone[0])                              # queued back to back on a side stream, no host wait
    fa = sc.feed(2, 48000, 10.0, 1.0, max_push_s=1.0, reference=True, reference_margin_s=0.5)
    fb = sc.feed(2, 48000, 10.0, 5.0, max_push_s=1.0, reference=True, reference_margin_s=0.5)
    try:
        pa, pb = _Player(fa, recs), _Player(fb, recs)
        for ns, rns, ends in pushes:
            pa.push(ns, rns, ends)
            pb.push(ns, rns, ends)
        same(pa.result(), alone[0])
        same(pb.result(), alone[1])
    finally:
        fa.close()
        fb.close()


@gpu
def test_sample_of_pairs_against_the_oracle(built_lib, tmp_path_factory):
    from oracle import de_arch_oracle as DO
    name = "std_fc20_lstm128bi_luong_soft_fd128"
    args, sd = _checkpoint(name)
    sc = _scorer(name, tmp_path_factory)
    d, r = _pair(30.0, 16000, 29.0, seed=40)
    got = _check(sc, [[_cuda(d, r)]], 16000, 10.0, 5.0, 0.5, seed=41)[0][0]
    scores, t0, t1, rt0, rt1 = got[0], got[2], got[3], got[6], got[7]
    f = lambda a: a.astype(np.float32) / np.float32(32768.0)      # noqa: E731
    for k in (0, len(scores) - 1):
        a, b = (int(round(t * 16000)) for t in (t0[k], t1[k]))
        ra, rb = (int(round(t * 16000)) for t in (rt0[k], rt1[k]))
        want, _, st = DO.predict_pcm_de(args, sd, f(d[a:b]), 16000, f(r[ra:rb]), 16000)
        assert st == 0
        np.testing.assert_allclose(scores[k], want, atol=1e-4, rtol=0)


@gpu
def test_engine_refusals_name_the_argument(built_lib, tmp_path_factory):
    de = _scorer("de_cosine_hard", tmp_path_factory)
    se = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    eng = de.engine
    try:
        with pytest.raises(E.EngineError, match="NISQA_DE"):          # unchanged: no single-ended feeds on a DE engine
            eng.feed_create(2, 48000, 480000, 100, 48000)
        with pytest.raises(E.EngineError, match="double-ended"):
            se.engine.feed_pair_create(2, 48000, 480000, 100, 0, 48000, 48000)
        with pytest.raises(E.EngineError, match="margin_frames"):
            eng.feed_pair_create(2, 48000, 480000, 100, -1, 48000, 48000)
        with pytest.raises(E.EngineError, match="margin_frames"):
            eng.feed_pair_create(2, 48000, 480000, 100, 3000, 48000, 48000)
        with pytest.raises(E.EngineError, match="max_skew"):
            eng.feed_pair_create(2, 48000, 480000, 100, 0, 48000, -1)
        with pytest.raises(E.EngineError, match="max_push"):
            eng.feed_pair_create(2, 48000, 480000, 100, 0, 0, 48000)
        with pytest.raises(E.EngineError, match="n_feeds"):
            eng.feed_pair_create(0, 48000, 480000, 100, 0, 48000, 48000)
        h = eng.feed_pair_create(2, 48000, 480000, 100, 50, 48000, 24000)
        hs = se.engine.feed_create(2, 48000, 480000, 100, 48000)
        x = torch.zeros((3, 1, 96000), dtype=torch.int16, device="cuda")
        out = torch.empty((8, 1), device="cuda")
        stream = torch.cuda.current_stream().cuda_stream

        def batch(n, ns, fmt=E.FMT_S16, rate=48000, data=x):
            b = E.device_batch(data.data_ptr(), fmt, ns, data.shape[1], -1, data.shape[2], data.stride(0), data.stride(1),
                               rate)
            b[0].n_clips = n
            return b

        def push(ns, rns, rows=8, end=None, **kw):
            return eng.feed_pair_push(h, stream, batch(2, ns), batch(kw.pop("rn", 2), rns, **kw), end, out.data_ptr(), rows)

        try:
            with pytest.raises(E.EngineError, match="nisqa_feed_pair_push"):
                eng.feed_push(h, stream, batch(2, [10, 10]), None, out.data_ptr(), 8)
            with pytest.raises(E.EngineError, match="nisqa_feed_push"):
                se.engine.feed_pair_push(hs, stream, batch(2, [10, 10]), batch(2, [10, 10]), None, out.data_ptr(), 8)
            with pytest.raises(E.EngineError, match="ref.n_clips"):
                push([10, 10], [10, 10, 10], rn=3)
            with pytest.raises(E.EngineError, match="ref.sample_rate"):
                push([10, 10], [10, 10], rate=16000)
            with pytest.raises(E.EngineError, match="ref.n_samples"):
                push([10, 10], [48001, 10])
            with pytest.raises(E.EngineError, match="deg.n_samples.*max_skew"):
                push([30000, 0], [0, 0])                              # 30000 apart > max_skew 24000
            push([24000, 0], [0, 0])
            with pytest.raises(E.EngineError, match="max_skew"):
                push([1, 0], [0, 0], end=np.array([1, 0], np.uint8))        # measured before the end's reset
            with pytest.raises(E.EngineError, match="sample_fmt"):
                push([10, 10], [10, 10], fmt=E.FMT_F32, data=x.float())     # the feeds hold int16 samples
            for _ in range(19):                                             # (the refused pushes changed nothing)
                push([24000, 0], [24000, 0], rows=0)
            push([0, 0], [24000, 0], rows=0)                                # 480000 degraded, 480000 reference samples
            with pytest.raises(E.EngineError, match="n_rows"):             # 480000 + M reference: the first pair
                push([0, 0], [24000, 0], rows=0)
            f, k = push([0, 0], [24000, 0], rows=1)[:2]
            assert f.tolist() == [0] and k.tolist() == [0]
            torch.cuda.synchronize()
            # rings of W + max_push + M + max_skew and W + max_push + M + max(M, max_skew) samples, mirrors of W and W + 2M
            assert eng.feed_device_bytes(h) >= 2 * 4 * ((480000 + 48000 + 24000 + 24000 + 480000) +
                                                        (480000 + 48000 + 24000 + 24000 + 528000))
        finally:
            eng.feed_destroy(h)
            se.engine.feed_destroy(hs)
    finally:
        se.close()
