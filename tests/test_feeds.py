"""Live feeds: nisqa_feed_rows, nisqa_feed_create / push / destroy and Scorer.feed.  CPU part: the rows each push emits
against a NumPy restatement of the window definition on the concatenated recording (random chunkings, 1-sample and
empty pushes, pushes of exactly max_push, ends and slot reuse, 8 to 96 kHz, odd and even hops in frames), the refusals
and the ABI.  GPU part: the rows of every feed bit for bit what Scorer.windows gives on the whole recording (int16 /
float32, channel pick and mix, 22.05 / 48 / 96 kHz, several passes, a too-short last window, slot reuse, pushes queued
on a side stream, two feed objects interleaved), a sample against the oracle, and the engine's own refusals."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from nisqa_b200.scorer import Feed, Scorer, window_geometry

gpu = pytest.mark.gpu
CKPTS = ["nisqa.tar", "nisqa_mos_only.tar", "nisqa_tts.tar"]


def _args(ckpt, **over):
    a = E.load_checkpoint(os.path.join(WEIGHTS, ckpt))[0]
    a.update(over)
    return a


def _cpu_scorer(ckpt, **over):
    s = Scorer.__new__(Scorer)
    s._configure(_args(ckpt, **over), torch.device("cpu"))
    return s


def _definition(args, T, rate, W, H):
    """window index, segment count and status of the windows of a recording of T samples (the definition)"""
    hop = int(rate * args["ms_hop_length"])
    K = 1 if T <= W else 1 + -(-(T - W) // H)
    k = np.arange(K, dtype=np.int64)
    n_wins = 1 + (np.minimum(k * H + W, T) - k * H) // hop - (args["ms_seg_length"] - 1)
    sh = args["ms_seg_hop_length"]
    n_seg = np.where(n_wins < 1, 0, -(-n_wins // sh))
    status = np.where(n_wins < 1, E.CLIP_TOO_SHORT, np.where(n_seg > args["ms_max_segments"], E.CLIP_TOO_LONG, E.CLIP_OK))
    return k, n_seg, status


def _plan(lengths, rng, max_push, recordings_per_feed=1):
    """a random chunking of recordings of the given lengths per feed: [(n_samples, end)] pushes.  Chunks of 0, 1, exactly
    max_push or any number of samples; feed b plays recordings_per_feed recordings back to back (slot reuse)"""
    B = len(lengths)
    left = [list(lengths[b]) if isinstance(lengths[b], (list, tuple)) else [lengths[b]] * recordings_per_feed
            for b in range(B)]
    pos = [0] * B
    pushes = []
    while any(left):
        ns, ends = np.zeros(B, np.int64), np.zeros(B, np.uint8)
        for b in range(B):
            if not left[b]:
                continue
            rem = left[b][0] - pos[b]
            c = rng.integers(0, 5)
            n = (0, 1, max_push, int(rng.integers(1, max_push + 1)), int(rng.integers(1, max(2, max_push // 10))))[c]
            ns[b] = min(n, rem)
            pos[b] += ns[b]
            if pos[b] == left[b][0]:
                ends[b] = 1
                left[b].pop(0)
                pos[b] = 0
        pushes.append((ns, ends))
    return pushes


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("rate", [8000, 22050, 44100, 48000, 96000])
def test_rows_per_push_follow_the_window_definition(built_lib, rate):
    args = _args("nisqa.tar")
    cfg = E.config_from_args(args)
    hop = int(rate * args["ms_hop_length"])
    rng = np.random.default_rng(rate)
    for window_s, window_hop_s in ((10.0, 1.0), (10.0, 0.37), (3.0, 2.9), (2.5, 0.01)):
        W, hf = window_geometry(args, rate, window_s, window_hop_s)
        H = hf * hop
        for max_push in (1 + W // 7, W):
            lengths = [[1, hop * 3, W - 1, W], [W + 1, 3 * W + 7], [int(4.3 * W) + 11]]
            held = np.zeros(3, np.int64)
            got = [[] for _ in range(3)]           # per feed: per recording (index, n_seg, status, emitted at held)
            cur = [[] for _ in range(3)]
            for ns, ends in _plan(lengths, rng, max_push):
                feed, index, n_seg, status = E.feed_rows(cfg, rate, W, hf, held, ns, ends)
                assert np.all(np.diff(feed) >= 0)
                T = held + ns
                for f, k, s, z in zip(feed, index, n_seg, status):
                    cur[f].append((k, s, z, T[f], bool(ends[f])))
                for b in np.nonzero(ends)[0]:
                    got[b].append(cur[b])
                    cur[b] = []
                held = np.where(ends.astype(bool), 0, T)
            for b in range(3):
                assert len(got[b]) == len(lengths[b])
                for T, rows in zip(lengths[b], got[b]):
                    k, n_seg, status = _definition(args, T, rate, W, H)
                    what = str((rate, window_s, window_hop_s, max_push, T))
                    np.testing.assert_array_equal([r[0] for r in rows], k, err_msg=what)
                    np.testing.assert_array_equal([r[1] for r in rows], n_seg, err_msg=what)
                    np.testing.assert_array_equal([r[2] for r in rows], status, err_msg=what)
                    for kk, _, _, at, ended in rows:      # the first push after which the feed holds k H + W samples
                        assert at >= kk * H + W or ended, what


def test_rows_of_empty_and_one_sample_pushes(built_lib):
    args = _args("nisqa.tar")
    cfg = E.config_from_args(args)
    W, hf = window_geometry(args, 48000, 10.0, 1.0)
    z = np.zeros(2, np.int64)
    assert E.feed_rows(cfg, 48000, W, hf, z, z, None)[0].shape == (0,)
    assert E.feed_rows(cfg, 48000, W, hf, z, z, [1, 1])[0].shape == (0,)       # an ended feed with no sample: no row
    held = np.array([W - 1, W - 2], np.int64)
    feed, index, _, _ = E.feed_rows(cfg, 48000, W, hf, held, np.array([1, 1]), None)
    assert feed.tolist() == [0] and index.tolist() == [0]
    feed, index, n_seg, status = E.feed_rows(cfg, 48000, W, hf, held, np.array([0, 0]), [0, 1])
    assert feed.tolist() == [1] and index.tolist() == [0] and status.tolist() == [E.CLIP_OK]


def _fake_feed(sc, n_feeds, rate, window_s, window_hop_s, channel=None, max_push_s=None):
    class _Eng(object):
        def feed_create(self, *a):
            return 1

        def feed_push(self, *a):
            raise AssertionError("a refused push reached the engine")
    sc.engine = _Eng()
    return sc.feed(n_feeds, rate, window_s, window_hop_s, channel=channel, max_push_s=max_push_s)


def test_refusals_name_the_argument(built_lib):
    sc = _cpu_scorer("nisqa.tar")
    sc.engine = None
    for bad in (0, -1, 65536, 2.0, True):
        with pytest.raises(ValueError, match="n_feeds"):
            sc.feed(bad, 48000, 10.0, 1.0)
    for bad in (0, -8000, 48000.0):
        with pytest.raises(ValueError, match="sample_rate"):
            sc.feed(4, bad, 10.0, 1.0)
    with pytest.raises(ValueError, match="window_hop_s"):
        sc.feed(4, 48000, 5.0, 6.0)
    with pytest.raises(ValueError, match="window_s"):
        sc.feed(4, 48000, 60.0, 1.0)              # 1497 segments > ms_max_segments 1300
    with pytest.raises(ValueError, match="window_s"):
        sc.feed(4, 48000, 0.1, 0.1)               # not one segment
    for bad in (-1.0, 0, float("nan"), True, "10"):
        with pytest.raises(ValueError, match="window_s"):
            sc.feed(4, 48000, bad, 1.0)
        with pytest.raises(ValueError, match="window_hop_s"):
            sc.feed(4, 48000, 10.0, bad)
        with pytest.raises(ValueError, match="max_push_s"):
            sc.feed(4, 48000, 10.0, 1.0, max_push_s=bad)
    with pytest.raises(TypeError, match="channel"):
        sc.feed(4, 48000, 10.0, 1.0, channel="left")
    ms = _cpu_scorer("nisqa_mos_only.tar", ms_sr=16000)
    ms.engine = None
    with pytest.raises(ValueError, match="sample_rate.*ms_sr"):
        ms.feed(4, 48000, 10.0, 1.0)
    de = _cpu_scorer("nisqa_mos_only.tar")
    de.double_ended = True                         # (what _configure sets for a NISQA_DE checkpoint)
    with pytest.raises(ValueError, match="NISQA_DE"):
        de.feed(4, 48000, 10.0, 1.0)
    # push: checked before anything reaches the engine
    fd = _fake_feed(_cpu_scorer("nisqa.tar"), 3, 48000, 10.0, 1.0, max_push_s=0.5)
    assert isinstance(fd, Feed) and fd.max_push == 24000
    x = torch.zeros((3, 30000), dtype=torch.int16)
    with pytest.raises(ValueError, match="wave"):
        fd.push(x[:2])                             # 2 feeds for 3
    with pytest.raises(ValueError, match="lengths"):
        fd.push(x)                                 # 30000 samples > max_push
    with pytest.raises(ValueError, match="lengths"):
        fd.push(x, lengths=[1, -1, 0])
    with pytest.raises(ValueError, match="lengths"):
        fd.push(x[:, :0], lengths=[1, 0, 0])
    with pytest.raises(ValueError, match="end"):
        fd.push(x[:, :100], end=[True, False])
    with pytest.raises(TypeError, match="wave"):
        fd.push(x.double())
    with pytest.raises(ValueError, match="channel"):
        _fake_feed(_cpu_scorer("nisqa.tar"), 3, 48000, 10.0, 1.0, channel=2).push(x[:, None, :100])
    # a format holds while a feed holds samples (the fake engine records nothing: set the state a push would leave)
    fd.held[:] = [5, 0, 0]
    fd._fmt = E.FMT_S16
    with pytest.raises(ValueError, match="wave.*int16"):
        fd.push(x[:, :100].float())


def test_header_exports_and_binding_agree(built_lib):
    header = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    lib = E.load_library()
    syms = ("nisqa_feed_create", "nisqa_feed_rows", "nisqa_feed_push", "nisqa_feed_device_bytes", "nisqa_feed_destroy")
    for sym in syms:
        assert sym + "(" in header and sym in E.EXPORTS and hasattr(lib, sym)
    assert [len(getattr(lib, s).argtypes) for s in syms] == [7, 14, 10, 1, 1]
    assert "typedef struct nisqa_feed nisqa_feed;" in header
    assert "#define NISQA_B200_ABI_VERSION 4" in header
    cfg = E.config_from_args(_args("nisqa.tar"))
    n = ctypes.c_int64()
    z = (ctypes.c_int64 * 1)(0)
    for window, hf in ((480000, 1001), (480000, 0), (48000 * 60, 100), (0, 1)):
        assert lib.nisqa_feed_rows(ctypes.byref(cfg), 48000, window, hf, 1, z, z, None, ctypes.byref(n),
                                   None, None, None, None, 0) == -1


# ------------------------------------------------------------------ GPU
_CACHE = {}


def _recording(sec, sr=48000, seed=0):
    """int16 speech-like recording; longer than 61 s: a 61 s one repeated with a gain that changes every second"""
    key = (sec, sr, seed)
    if key not in _CACHE:
        if sec <= 61:
            _CACHE[key] = synth.synth_speech_pcm16(3000 + seed, sec, sr)[:int(sec * sr)]
        else:
            base = _recording(61.0, sr, seed).astype(np.float32)
            n = int(sec * sr)
            g = np.repeat(np.random.default_rng(seed).uniform(0.05, 1.0, n // sr + 1), sr)[:n]
            _CACHE[key] = np.clip(np.resize(base, n) * g, -32768, 32767).astype(np.int16)
    return _CACHE[key]


_SCORERS = {}


@pytest.fixture(scope="module", autouse=True)
def _close_scorers():
    """the engines of this module hold their pass workspaces: freed for the modules after it"""
    yield
    for sc in _SCORERS.values():
        sc.close()
    _SCORERS.clear()


def _scorer(ckpt, **over):
    key = (ckpt, tuple(sorted(over.items())))
    if key not in _SCORERS:
        _SCORERS[key] = Scorer(os.path.join(WEIGHTS, ckpt), **over)
    return _SCORERS[key]


class _Player(object):
    """pushes the recordings recs[b] (lists of [T] or [C, T] CUDA tensors, played back to back) to a feed object chunk by
    chunk and collects each feed's rows, recording by recording"""

    def __init__(self, fd, recs):
        self.fd, self.queue = fd, [list(r) for r in recs]
        B = len(recs)
        self.pos, self.cur, self.out = [0] * B, [[] for _ in range(B)], [[] for _ in range(B)]

    def push(self, ns, ends, sync=False):
        B = len(self.queue)
        x0 = next(q[0] for q in self.queue if q)
        Tc = max(int(ns.max()), 1)
        chunk = torch.zeros((B,) + tuple(x0.shape[:-1]) + (Tc,), dtype=x0.dtype, device=x0.device)
        for b in range(B):
            if ns[b]:
                chunk[b, ..., :ns[b]] = self.queue[b][0][..., self.pos[b]:self.pos[b] + ns[b]]
        r = self.fd.push(chunk, lengths=ns, end=ends)
        if sync:
            torch.cuda.synchronize()
        for i, f in enumerate(r.feed):
            self.cur[f].append((r.scores[i], r.index[i], r.t_start[i], r.t_end[i], r.n_segments[i], r.status[i]))
        for b in range(B):
            self.pos[b] += int(ns[b])
            if ends[b]:
                self.out[b].append(self.cur[b])
                self.cur[b] = []
                self.queue[b].pop(0)
                self.pos[b] = 0

    def result(self):
        """per feed, per recording: (scores, index, t_start, t_end, n_segments, status) of its rows"""
        torch.cuda.synchronize()
        res = []
        for b in range(len(self.out)):
            res.append([])
            for rows in self.out[b]:
                sc = torch.stack([r[0] for r in rows]).cpu().numpy() if rows else np.zeros((0, 1), np.float32)
                res[b].append((sc,) + tuple(np.array([r[j] for r in rows]) for j in range(1, 6)))
        return res


def _replay(fd, recs, pushes, sync=False):
    pl = _Player(fd, recs)
    for ns, ends in pushes:
        pl.push(ns, ends, sync)
    return pl.result()


def _check_feeds(sc, recs, rate, window_s, window_hop_s, seed, channel=None, max_push_s=2.0):
    """every feed's rows, recording by recording, equal Scorer.windows on the whole recording"""
    rng = np.random.default_rng(seed)
    fd = sc.feed(len(recs), rate, window_s, window_hop_s, channel=channel, max_push_s=max_push_s)
    try:
        pushes = _plan([[r.shape[-1] for r in rr] for rr in recs], rng, fd.max_push)
        got = _replay(fd, recs, pushes)
    finally:
        fd.close()
    for b, rr in enumerate(recs):
        for x, (scores, index, t0, t1, nseg, status) in zip(rr, got[b]):
            w = sc.windows(x if x.dim() == 1 else x[None], rate, window_s, window_hop_s, channel=channel)
            what = str((rate, window_s, window_hop_s, channel, x.shape))
            assert w.counts == [len(index)], what
            np.testing.assert_array_equal(index, np.arange(len(index)), err_msg=what)
            np.testing.assert_array_equal(scores, w.scores.cpu().numpy(), err_msg=what)
            np.testing.assert_array_equal(t0, w.t_start, err_msg=what)
            np.testing.assert_array_equal(t1, w.t_end, err_msg=what)
            np.testing.assert_array_equal(nseg, w.n_segments, err_msg=what)
            np.testing.assert_array_equal(status, w.status, err_msg=what)
    return got


@gpu
@pytest.mark.parametrize("ckpt", CKPTS)
def test_feeds_equal_windows_bit_for_bit(built_lib, ckpt):
    sc = _scorer(ckpt)
    recs = [[torch.from_numpy(_recording(sec, seed=i)).cuda()] for i, sec in enumerate((3.0, 61.0, 150.0))]
    for i, window_hop_s in enumerate((1.0, 5.0, 3.33)):            # 100, 500 and 333 (odd) frames
        _check_feeds(sc, recs, 48000, 10.0, window_hop_s, seed=i, max_push_s=4.0)


@gpu
def test_other_inputs_equal_windows(built_lib):
    sc = _scorer("nisqa.tar")
    st = torch.from_numpy(np.stack([_recording(25.0, seed=11), _recording(25.0, seed=12)]).astype(np.float32) / 32768.0)
    st = st.cuda()                                                            # float32 stereo [2, T]
    for channel in (1, None):
        _check_feeds(sc, [[st], [st[:, :400000].contiguous()]], 48000, 10.0, 1.0, seed=3, channel=channel)
    st16 = torch.from_numpy(np.stack([_recording(14.0, seed=13), _recording(14.0, seed=14)])).cuda()
    _check_feeds(sc, [[st16]], 48000, 10.0, 1.0, seed=4, channel=0)           # int16, a channel picked: int16 rings
    x22 = torch.from_numpy(_recording(25.0, 22050, seed=15)).cuda()
    _check_feeds(sc, [[x22], [x22[:300000]]], 22050, 10.0, 1.0, seed=5)
    _check_feeds(sc, [[x22.float() / 32768.0]], 22050, 10.0, 0.37, seed=6)   # 37 frames: both pairings
    x96 = torch.from_numpy(_recording(14.0, 96000, seed=16)).cuda()          # 1920-sample windows: frontend_kernel
    _check_feeds(sc, [[x96], [x96[:1000000]]], 96000, 10.0, 1.0, seed=7)
    _check_feeds(sc, [[x96.float() / 32768.0]], 96000, 10.0, 3.33, seed=8)
    # a too-short last window: NaN and CLIP_TOO_SHORT
    xs = torch.from_numpy(_recording(20.05, seed=17)).cuda()
    got = _check_feeds(sc, [[xs]], 48000, 10.0, 10.0, seed=9)
    assert got[0][0][5].tolist() == [E.CLIP_OK, E.CLIP_OK, E.CLIP_TOO_SHORT] and np.isnan(got[0][0][0][2]).all()


@gpu
def test_passes_and_slot_reuse(built_lib):
    # one push completing many windows, each pass holding one window (b200_max_chunk_segments)
    small = _scorer("nisqa.tar", b200_max_chunk_segments=300)
    x = torch.from_numpy(_recording(61.0, seed=21)).cuda()
    fd = small.feed(1, 48000, 10.0, 1.0, max_push_s=61.0)
    r = fd.push(x[None], end=[True])
    torch.cuda.synchronize()
    fd.close()
    assert small.engine.lib.nisqa_stage_dump(small.engine.h, E.STAGE_MEL_DB, None, 0) < 0     # (it ran in passes)
    w = small.windows(x, 48000, 10.0, 1.0)
    np.testing.assert_array_equal(r.scores.cpu().numpy(), w.scores.cpu().numpy())
    assert r.index.tolist() == list(range(w.counts[0]))
    # a slot reused after end scores each recording as Scorer.windows does
    sc = _scorer("nisqa.tar")
    recs = [[torch.from_numpy(_recording(sec, seed=22 + i)).cuda() for i, sec in enumerate((17.0, 3.0, 31.0))],
            [torch.from_numpy(_recording(sec, seed=30 + i)).cuda() for i, sec in enumerate((12.5, 40.0))]]
    _check_feeds(sc, recs, 48000, 10.0, 1.0, seed=10)
    _check_feeds(sc, recs, 48000, 10.0, 3.33, seed=11)


@gpu
def test_stream_order_and_interleaved_feeds(built_lib):
    sc = _scorer("nisqa.tar")
    recs = [[torch.from_numpy(_recording(sec, seed=40 + i)).cuda()] for i, sec in enumerate((23.0, 37.0, 8.0))]
    pushes = _plan([[r[0].shape[-1]] for r in recs], np.random.default_rng(12), 48000)

    def run(sync, stream=None):
        fd = sc.feed(3, 48000, 10.0, 1.0, max_push_s=1.0)
        try:
            if stream is None:
                return _replay(fd, recs, pushes, sync=sync)
            with torch.cuda.stream(stream):
                return _replay(fd, recs, pushes, sync=sync)
        finally:
            fd.close()

    def same(a, b):
        for fa, fb in zip(a, b):
            for ra, rb in zip(fa, fb):
                for u, v in zip(ra, rb):
                    np.testing.assert_array_equal(u, v)

    ref = run(True)
    same(run(False, torch.cuda.Stream()), ref)              # queued back to back on a side stream, no host sync
    # two feed objects on one scorer, their pushes interleaved, against each alone
    alone = []
    for hop_s in (1.0, 5.0):
        fd = sc.feed(3, 48000, 10.0, hop_s, max_push_s=1.0)
        alone.append(_replay(fd, recs, pushes))
        fd.close()
    fa, fb = sc.feed(3, 48000, 10.0, 1.0, max_push_s=1.0), sc.feed(3, 48000, 10.0, 5.0, max_push_s=1.0)
    try:
        pa, pb = _Player(fa, recs), _Player(fb, recs)
        for ns, ends in pushes:
            pa.push(ns, ends)
            pb.push(ns, ends)
        same(pa.result(), alone[0])
        same(pb.result(), alone[1])
    finally:
        fa.close()
        fb.close()


@gpu
def test_sample_of_feed_windows_against_the_oracle(built_lib):
    from oracle import nisqa_oracle as O
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    sc = _scorer("nisqa.tar")
    x = _recording(61.0, seed=50)
    got = _check_feeds(sc, [[torch.from_numpy(x).cuda()]], 48000, 10.0, 5.0, seed=13)
    scores, index, t0, t1, nseg, status = got[0][0]
    for k in (0, 6, len(index) - 1):
        a, b = int(round(t0[k] * 48000)), int(round(t1[k] * 48000))
        ref, n_seg, st = O.predict_pcm(args, sd, x[a:b].astype(np.float32) / 32768.0, 48000)
        assert st == 0 and n_seg == nseg[k]
        np.testing.assert_allclose(scores[k], ref, atol=1e-4, rtol=0)


@gpu
def test_engine_refusals_name_the_argument(built_lib):
    sc = _scorer("nisqa.tar")
    eng = sc.engine
    with pytest.raises(E.EngineError, match="n_feeds"):
        eng.feed_create(0, 48000, 480000, 100, 48000)
    with pytest.raises(E.EngineError, match="hop_frames"):
        eng.feed_create(2, 48000, 480000, 1001, 48000)
    with pytest.raises(E.EngineError, match="max_push"):
        eng.feed_create(2, 48000, 480000, 100, 0)
    h = eng.feed_create(2, 48000, 480000, 100, 48000)
    x = torch.zeros((3, 1, 96000), dtype=torch.int16, device="cuda")
    out = torch.empty((8, 1), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def push(n, ns, fmt=E.FMT_S16, rate=48000, ch=-1, rows=8, end=None, data=x):
        b = E.device_batch(data.data_ptr(), fmt, ns, data.shape[1], ch, data.shape[2], data.stride(0), data.stride(1), rate)
        b[0].n_clips = n
        return eng.feed_push(h, stream, b, end, out.data_ptr(), rows)

    try:
        with pytest.raises(E.EngineError, match="chunk.n_clips"):
            push(3, [10, 10, 10])
        with pytest.raises(E.EngineError, match="chunk.sample_rate"):
            push(2, [10, 10], rate=16000)
        with pytest.raises(E.EngineError, match="chunk.n_samples"):
            push(2, [48001, 10])
        with pytest.raises(E.EngineError, match="chunk.n_samples"):
            push(2, [-1, 10])
        with pytest.raises(E.EngineError, match="chunk.sample_fmt"):
            push(2, [10, 10], fmt=7)
        with pytest.raises(E.EngineError, match="chunk.channel"):
            push(2, [10, 10], ch=5, data=torch.zeros((2, 2, 100), dtype=torch.int16, device="cuda"))
        push(2, [48000, 0])
        with pytest.raises(E.EngineError, match="chunk.sample_fmt"):
            push(2, [10, 10], fmt=E.FMT_F32, data=x.float())          # the feeds hold int16 samples
        for _ in range(8):
            push(2, [48000, 0])
        push(2, [47999, 0])                                           # one sample short of the first window
        with pytest.raises(E.EngineError, match="n_rows"):
            push(2, [1, 0], rows=0)
        f, k, _, _ = push(2, [1, 0], rows=1)                          # (the refused pushes changed nothing)
        assert f.tolist() == [0] and k.tolist() == [0]
        f, k, _, st = push(2, [1, 0], rows=1, end=np.array([1, 1], np.uint8))
        assert f.tolist() == [0] and k.tolist() == [1] and st.tolist() == [E.CLIP_OK]     # [48000, 480001)
        push(2, [10, 10], fmt=E.FMT_F32, data=x.float())             # every feed ended: another format may start
        torch.cuda.synchronize()
        assert eng.feed_device_bytes(h) >= 2 * (2 * 480000 + 48000) * 4
    finally:
        eng.feed_destroy(h)
