"""``Scorer``: NISQA scores of waveforms that are already on the GPU, in the caller's CUDA stream order.

    scorer = Scorer("weights/nisqa.tar")
    scores = scorer(wave, 48000)            # wave: [T], [B, T] or [B, C, T] int16 / float32 CUDA tensor
    dict(zip(scorer.columns, scores[0].tolist()))

The audio never leaves the device: the engine packs it with its own ingest kernel (``nisqa_predict_device_batch``)
and the scores come back as a CUDA tensor, written in the order of ``torch.cuda.current_stream()``.  Nothing waits for
the GPU: ``wave`` may be freed or reused in stream order as soon as the call returns.

``scorer.segments(wave, 48000)`` also returns where in each clip the quality drops: every segment's score and pooling
weight (``nisqa_predict_device_batch_segments``) with its time span.

``scorer.embed(wave, 48000)`` returns the representation behind the scores: each pooling head's pooled vector, the
input of its last Linear, and optionally every segment's row (``nisqa_predict_device_batch_embeddings``).

``scorer.windows(wave, 48000, 10.0, 1.0)`` scores recordings of any length as a timeline: every 10 s window at a 1 s hop,
each scored as the clip cut out of the recording would be (``nisqa_predict_device_windows``).  A NISQA_DE checkpoint
scores window pairs of a recording and its reference: ``scorer.windows(wave, 48000, 10.0, 1.0, reference=ref)``
(``nisqa_predict_device_window_pairs``).

``scorer.align(wave, 48000, ref)`` reports a NISQA_DE checkpoint's time alignment: for every degraded segment the
reference segment it matched, how sharp the match is, and the delay in seconds (``nisqa_predict_device_batch_alignment``;
with ``window_s`` of window pairs, ``nisqa_predict_device_window_pairs_alignment``).

``scorer.feed(256, 48000, 10.0, 1.0)`` scores live sources as their audio arrives: ``feed.push(chunk)`` appends a chunk to
every source and returns the windows it completed, with the scores ``windows`` gives on the whole recording
(``nisqa_feed_push``).  A NISQA_DE checkpoint scores live (degraded, reference) pairs:
``scorer.feed(256, 48000, 10.0, 1.0, reference=True)`` and ``feed.push(chunk, ref_chunk)`` (``nisqa_feed_pair_push``).
"""
import collections
import numbers

import numpy as np
import torch

from . import engine as E

DIM_COLUMNS = ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"]     # NISQA_DIM's outputs (lib:1461-1465)


# Scorer.segments: scores [B, n_cols] (as Scorer.__call__), seg_scores / seg_weights [N, n_cols] CUDA tensors (the rows of
# clip b follow those of the clips before it, counts[b] of them), t_start / t_end float64 [N] seconds
Segments = collections.namedtuple("Segments", ["scores", "seg_scores", "seg_weights", "counts", "t_start", "t_end"])
# Scorer.embed: scores [B, n_cols] (as Scorer.__call__), pooled [B, n_cols, width] CUDA tensor (head h's pooled vector),
# rows [N, width] CUDA tensor or None (the rows of clip b follow those of the clips before it, counts[b] of them)
Embeddings = collections.namedtuple("Embeddings", ["scores", "pooled", "rows", "counts"])
# Scorer.windows: scores [N, n_cols] CUDA tensor (the windows of recording b follow those of the recordings before it,
# counts[b] of them); t_start / t_end float64 [N] seconds, n_segments / status int32 [N] host arrays
Windows = collections.namedtuple("Windows", ["scores", "counts", "t_start", "t_end", "n_segments", "status"])
# Scorer.windows with a reference (NISQA_DE): scores [N, n_cols] CUDA tensor, one row per window pair (the pairs of
# recording b follow those of the recordings before it, counts[b] of them); the degraded windows' t_start / t_end float64
# [N] seconds and n_segments / status int32 [N], and the same of the reference windows (ref_*), host arrays
WindowPairs = collections.namedtuple("WindowPairs", ["scores", "counts", "t_start", "t_end", "n_segments", "status",
                                                     "ref_t_start", "ref_t_end", "ref_n_segments", "ref_status"])
# Scorer.align: scores [B, n_cols] (as Scorer.__call__); ref_seg int32, weight / centroid / peak float32 [N] CUDA tensors
# (the rows of clip b follow those of the clips before it, counts[b] of them); t_start / ref_t_start / delay_s /
# centroid_delay_s float64 [N] host arrays, seconds
Alignment = collections.namedtuple("Alignment", ["scores", "ref_seg", "weight", "centroid", "peak", "counts", "t_start",
                                                 "ref_t_start", "delay_s", "centroid_delay_s"])
# Scorer.align with window_s: the fields of Alignment (scores, counts: of the window pairs, counts[k] rows of pair k),
# window int64 [N] (the row's pair), and the pair columns of WindowPairs, one entry per pair, as pair_* (pair_counts:
# pairs per recording)
AlignmentWindows = collections.namedtuple("AlignmentWindows", Alignment._fields + ("window",) + tuple(
    "pair_" + f for f in WindowPairs._fields[1:]))
# Feed.push: scores [N, n_cols] CUDA tensor of the windows the push completed, by feed then window index; feed int32 [N],
# index int64 [N] (window k of the feed's current recording), t_start / t_end float64 [N] seconds, n_segments / status
# int32 [N] host arrays
FeedRows = collections.namedtuple("FeedRows", ["scores", "feed", "index", "t_start", "t_end", "n_segments", "status"])
# FeedPairs.push: the fields of FeedRows for the window pairs the push completed (one score row per pair; t_start / t_end,
# n_segments / status of the degraded windows), and ref_t_start / ref_t_end float64 [N] seconds, ref_n_segments /
# ref_status int32 [N] of the reference windows, host arrays
FeedPairRows = collections.namedtuple("FeedPairRows", FeedRows._fields + ("ref_t_start", "ref_t_end", "ref_n_segments",
                                                                          "ref_status"))


def window_geometry(args, rate, window_s, window_hop_s):
    """(W, hop_frames) of windows of ``window_s`` seconds at a hop of ``window_hop_s`` seconds at the model rate ``rate``:
    W = round(window_s rate) samples, a hop of max(1, round(window_hop_s rate / hop)) mel frames of hop = int(rate
    ms_hop_length) samples, so that every window starts on a mel frame of the recording"""
    for name, v in (("window_s", window_s), ("window_hop_s", window_hop_s)):
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not np.isfinite(v) or v <= 0:
            raise ValueError("%s: a positive number of seconds, not %r" % (name, v))
    hop = int(rate * args["ms_hop_length"])
    W = int(round(window_s * rate))
    hop_frames = max(1, int(round(window_hop_s * rate / hop)))
    if W < 1:
        raise ValueError("window_s=%r: no sample at %d Hz" % (window_s, rate))
    if hop_frames * hop > W:
        raise ValueError("window_hop_s=%r: a hop of %d samples (%d mel frames of %d) is longer than the window of %d samples "
                         "(window_s=%r) at %d Hz" % (window_hop_s, hop_frames * hop, hop_frames, hop, W, window_s, rate))
    return W, hop_frames


def window_times(T, W, H, rate):
    """(t_start, t_end) in seconds of the windows of a recording of T samples at the model rate"""
    K = 1 if T <= W else 1 + -(-(T - W) // H)
    k = np.arange(K, dtype=np.int64)
    return k * H / rate, np.minimum(k * H + W, T) / rate


class Scorer(object):
    """A checkpoint loaded onto one GPU.  ``overrides`` update the checkpoint's args like the caller's dict of
    ``nisqaModel`` (e.g. ``ms_sr``, ``b200_max_chunk_segments``)."""

    def __init__(self, pretrained_model, device=None, **overrides):
        if not torch.cuda.is_available():
            raise RuntimeError("no CUDA device available: the engine has no CPU fallback")
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ValueError("device: the engine runs on a CUDA device, not %r" % (device,))
        args, state_dict = E.load_checkpoint(pretrained_model, overrides)
        self._configure(args, torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device()))
        self.engine = E.engine_from_checkpoint(args, state_dict, device=self.device.index)

    def _configure(self, args, device):
        """The host side of a scorer: what its arguments are checked against"""
        self.args, self.device = args, device
        self.cfg = E.config_from_args(args, max_chunk_segments=args.get("b200_max_chunk_segments", 0))
        self.double_ended = args["model"] == "NISQA_DE"
        self.columns = list(DIM_COLUMNS) if args["model"] == "NISQA_DIM" else ["mos_pred"]
        self.target_sr = int(args["ms_sr"]) if args.get("ms_sr") else 0

    def close(self):
        self.engine.close()

    def __call__(self, wave, sample_rate, lengths=None, channel=None, reference=None, reference_lengths=None,
                 reference_sample_rate=None, reference_index=None):
        """Scores of a batch -> float32 [B, len(columns)] on ``wave.device``.

        wave        : [T], [B, T] or [B, C, T] int16 / float32 CUDA tensor on the scorer's device, any batch and channel
                      strides, samples contiguous
        sample_rate : of every clip
        lengths     : host ints, samples of each clip (default T)
        channel     : None = the mono mix (mean over channels, as the file ingest), else that channel
        reference   : NISQA_DE only: the reference clips, one per clip of ``wave``, always mixed to mono; with their own
                      ``reference_lengths`` and ``reference_sample_rate`` (default: ``sample_rate``)
        reference_index : NISQA_DE only, references shared by several clips (a sweep of conditions over one source):
                      host ints, one per clip of ``wave``, naming its clip of ``reference``, which then holds any number
                      U >= 1 of clips.  Each reference is computed once per engine pass and every pair scores bit for
                      bit what ``reference[reference_index]`` gives; a reference no clip names is not read.
        A clip too short or too long for the checkpoint raises the file ingest's ValueError before anything is enqueued.
        """
        deg, ref, _, idx = self._arguments(wave, sample_rate, lengths, channel, reference, reference_lengths,
                                           reference_sample_rate, reference_index)
        out = self._scores_buffer(deg, ref, idx)
        if out.shape[0] and idx is not None:
            self.engine.predict_device_batch_shared_ref(self._stream(), deg, ref, idx, out.data_ptr(), target_sr=self.target_sr)
        elif out.shape[0]:
            self.engine.predict_device_batch(self._stream(), deg, out.data_ptr(), ref=ref, target_sr=self.target_sr)
        return self._clip_rows(out, ref, idx)

    def segments(self, wave, sample_rate, lengths=None, channel=None, reference=None, reference_lengths=None,
                 reference_sample_rate=None, reference_index=None):
        """Scores of a batch and of every segment of its clips -> :data:`Segments`.  Takes the arguments of
        ``__call__`` and checks them alike.

        scores      : float32 [B, len(columns)], the values ``__call__`` returns
        seg_scores  : float32 [N, len(columns)] CUDA tensor: each pooling head applied to the segment alone (its last
                      Linear of the segment's time-dependency output row)
        seg_weights : float32 [N, len(columns)] CUDA tensor: the head's pooling weight of the segment (attention: its
                      softmax weight; avg: 1 / n_seg; last_step: 1 at the last segment; max, last_step_bi: NaN).  Where
                      defined, a clip's score is the weighted sum of its segments' scores
        counts      : host list of B ints, the segments of each clip (its rows follow those of the clips before it)
        t_start, t_end : float64 [N] host arrays, seconds: the centres of the segment's first and last mel frame
        NISQA_DE: rows for the degraded clips only.
        """
        deg, ref, counts, idx = self._arguments(wave, sample_rate, lengths, channel, reference, reference_lengths,
                                                reference_sample_rate, reference_index)
        out = self._scores_buffer(deg, ref, idx)
        n_rows = int(sum(counts))
        seg_s = torch.empty((n_rows, len(self.columns)), dtype=torch.float32, device=self.device)
        seg_w = torch.empty_like(seg_s)
        if out.shape[0] and idx is not None:
            so = E.NisqaSegmentOut(scores=seg_s.data_ptr() or None, weights=seg_w.data_ptr() or None, n_rows=n_rows)
            self.engine.predict_device_batch_shared_ref(self._stream(), deg, ref, idx, out.data_ptr(), so,
                                                        target_sr=self.target_sr)
        elif out.shape[0]:
            self.engine.predict_device_batch_segments(self._stream(), deg, out.data_ptr(), seg_s.data_ptr(), seg_w.data_ptr(),
                                                      n_rows, ref=ref, target_sr=self.target_sr)
        rate = self.target_sr or deg[0].sample_rate
        a = self.args
        hop = int(rate * a["ms_hop_length"])                  # (int)(sr * hop_s), as the engine's front end
        t = np.concatenate([np.arange(c, dtype=np.float64) for c in counts]) if counts else np.zeros(0)
        t_start = t * a["ms_seg_hop_length"] * hop / rate
        t_end = (t * a["ms_seg_hop_length"] + a["ms_seg_length"] - 1) * hop / rate
        return Segments(self._clip_rows(out, ref, idx), seg_s, seg_w, list(counts), t_start, t_end)

    def windows(self, wave, sample_rate, window_s, window_hop_s, lengths=None, channel=None, reference=None,
                reference_lengths=None, reference_sample_rate=None, reference_margin_s=0.0, reference_index=None):
        """Every recording of a batch scored as a timeline of overlapping windows -> :data:`Windows`, or with a
        ``reference`` (NISQA_DE) as a timeline of window pairs -> :data:`WindowPairs`.  Takes the arguments of
        ``__call__`` and checks them alike, but accepts recordings of any length.

        window_s     : window length in seconds at the model rate (``ms_sr`` when set, else ``sample_rate``):
                       W = round(window_s rate) samples; its segment count must fit ``ms_max_segments``
        window_hop_s : hop between window starts, rounded to whole mel frames (at least one); at most the window
        Window k of a recording of T samples covers samples [k H, min(k H + W, T)) and scores exactly what that cut-out
        clip scores through ``__call__``.  Only the last window can be shorter than W; if it is too short for the
        checkpoint its scores are NaN and its status is CLIP_TOO_SHORT.
        scores       : float32 [N, len(columns)] CUDA tensor, the windows of recording b after those of the ones before it
        counts       : host list of B ints, windows per recording
        t_start, t_end : float64 [N] host arrays, seconds at the model rate
        n_segments, status : int32 [N] host arrays

        reference          : NISQA_DE only: one reference recording per recording of ``wave``, of any length, always
                             mixed to mono; with its own ``reference_lengths`` and ``reference_sample_rate`` (default
                             ``sample_rate``; without ``ms_sr`` it must equal ``sample_rate``)
        reference_margin_s : widens each reference window by M = round(reference_margin_s rate / hop) hop samples on
                             either side (default 0), so that the alignment finds delayed content near a window's edge
        Pair k scores exactly what ``__call__`` gives the degraded window k and the reference window [max(0, k H - M),
        min(T_ref, k H + W + M)) cut out as clips.  A pair whose degraded or reference window is too short (or empty:
        k H - M >= T_ref) scores NaN; ``status`` and ``ref_status`` tell which.
        ``reference_index`` (shared references) is refused: window pairs take one reference recording per recording.
        """
        _refuse_reference_index(reference_index, "windows")
        return self._windows(wave, sample_rate, window_s, window_hop_s, lengths, channel, reference, reference_lengths,
                             reference_sample_rate, reference_margin_s, None)

    def _windows(self, wave, sample_rate, window_s, window_hop_s, lengths, channel, reference, reference_lengths,
                 reference_sample_rate, reference_margin_s, alignment):
        """windows(); alignment (window pairs only): None, or alignment(n_segments, status) of the pairs -> the
        NisqaAlignmentOut the call also writes"""
        from . import resample as RS
        m = reference_margin_s
        if isinstance(m, bool) or not isinstance(m, numbers.Real) or not np.isfinite(m) or m < 0:
            raise ValueError("reference_margin_s: a non-negative number of seconds, not %r" % (m,))
        if reference is None:
            if m != 0:
                raise ValueError("reference_margin_s=%r: a margin widens reference windows; pass reference= (NISQA_DE)" % (m,))
            if self.double_ended:
                raise ValueError("windows: a double-ended (NISQA_DE) checkpoint scores window pairs of a recording and its "
                                 "reference: pass reference=")
        elif not self.double_ended:
            raise ValueError("reference: only a double-ended (NISQA_DE) checkpoint takes reference clips")
        deg = self._batch("wave", wave, sample_rate, lengths, channel)
        sr = deg[0].sample_rate
        ref = None
        if reference is not None:
            ref = self._batch("reference", reference, sample_rate if reference_sample_rate is None else reference_sample_rate,
                              reference_lengths, None)
            if ref[0].n_clips != deg[0].n_clips:
                raise ValueError("reference: %d recordings for %d recordings of wave" % (ref[0].n_clips, deg[0].n_clips))
            if not self.target_sr and ref[0].sample_rate != sr:
                raise ValueError("reference_sample_rate: %d Hz for wave at %d Hz; without ms_sr both recordings' windows "
                                 "run at one rate" % (ref[0].sample_rate, sr))
        rate = self.target_sr or sr
        W, hop_frames = window_geometry(self.args, rate, window_s, window_hop_s)
        hop = int(rate * self.args["ms_hop_length"])
        H = hop_frames * hop
        a = self.args
        _, n_seg, status = E.segment_counts(self.cfg, W, rate)
        if status != E.CLIP_OK:
            err = E.clip_status_error(status, "window_s=%r (%d samples at %d Hz)" % (window_s, W, rate), W, rate, n_seg,
                                      a["ms_hop_length"], a["ms_seg_length"], a["ms_max_segments"])
            raise ValueError("window_s: " + str(err))
        margin_frames = int(round(m * rate / hop))
        M = margin_frames * hop
        if ref is not None:
            _, n_seg, status = E.segment_counts(self.cfg, W + 2 * M, rate)
            if status != E.CLIP_OK:
                raise ValueError("reference_margin_s=%r: reference windows of %d samples (W + 2 x %d) have %d segments > "
                                 "ms_max_segments %d" % (m, W + 2 * M, M, n_seg, a["ms_max_segments"]))
        model_len = lambda n, r: int(n) if rate == r else RS.out_len(int(n), r, rate)      # noqa: E731
        counts, parts = [], []
        for b, n in enumerate(deg[1]):
            T = model_len(n, sr)
            t0, t1 = window_times(T, W, H, rate)
            if ref is None:
                cols = E.window_counts(self.cfg, T, rate, W, hop_frames)
            else:
                T_ref = model_len(ref[1][b], ref[0].sample_rate)
                cols = E.window_pair_counts(self.cfg, T, T_ref, rate, W, hop_frames, margin_frames)
                k = np.arange(len(t0), dtype=np.int64)
                r0 = np.maximum(0, k * H - M)
                r1 = np.maximum(r0, np.minimum(T_ref, k * H + W + M))
                cols = cols[:2] + (r0 / rate, r1 / rate) + cols[2:]
            counts.append(len(t0))
            parts.append((t0, t1) + tuple(cols))
        N = int(sum(counts))
        out = torch.empty((N, len(self.columns)), dtype=torch.float32, device=self.device)
        types = (np.float64, np.float64, np.int32, np.int32) * (1 if ref is None else 2)
        cols = [np.concatenate([p[i] for p in parts]).astype(t) if parts else np.zeros(0, t) for i, t in enumerate(types)]
        if N and ref is None:
            self.engine.predict_device_windows(self._stream(), deg, out.data_ptr(), N, W, hop_frames, target_sr=self.target_sr)
        elif N and alignment is None:
            self.engine.predict_device_window_pairs(self._stream(), deg, ref, out.data_ptr(), N, W, hop_frames, margin_frames,
                                                    target_sr=self.target_sr)
        elif N:
            self.engine.predict_device_window_pairs_alignment(self._stream(), deg, ref, out.data_ptr(), N, W, hop_frames,
                                                              margin_frames, alignment(cols[2], cols[3]),
                                                              target_sr=self.target_sr)
        return Windows(out, counts, *cols) if ref is None else WindowPairs(out, counts, *cols)

    def align(self, wave, sample_rate, reference, lengths=None, channel=None, reference_lengths=None,
              reference_sample_rate=None, window_s=None, window_hop_s=None, reference_margin_s=0.0, reference_index=None):
        """NISQA_DE's time alignment of every degraded segment -> :data:`Alignment`, or with ``window_s`` of every segment
        of each window pair's degraded window -> :data:`AlignmentWindows`.  Takes the arguments of ``__call__`` (of
        ``windows`` with a ``window_s``) and checks them alike; a single-ended checkpoint raises ValueError.

        scores        : the values ``__call__`` (``windows(..., reference=)``) returns
        ref_seg       : int32 [N] CUDA tensor, the reference segment with the first maximal alignment score (under hard
                        application: the one the model fused); -1 where the pair scores NaN
        weight        : float32 [N] CUDA tensor, that segment's softmax weight: how sharp the match is
        centroid      : float32 [N] CUDA tensor, the softmax-weighted reference segment position
        peak          : float32 [N] CUDA tensor, the maximal score as the alignment module computes it (cosine: the
                        cosine similarity)
        counts        : host list, the rows of each clip (window mode: of each pair)
        t_start       : float64 [N] seconds, the degraded segment's start in its recording
        ref_t_start   : float64 [N] seconds, the start of reference segment ref_seg in the reference recording
        delay_s       : ref_t_start - t_start;  centroid_delay_s: the centroid's position in seconds minus t_start
        Segment i starts i * ms_seg_hop_length * hop / rate seconds into its clip, each side at its own model rate and hop;
        window mode adds k H / rate on the degraded side and max(0, k H - M) / rate on the reference side of pair k.
        reference_index : clip mode only, as in ``__call__`` (shared references)
        """
        if not self.double_ended:
            raise ValueError("align: only a double-ended (NISQA_DE) checkpoint aligns a reference to the degraded signal")
        if window_s is not None or window_hop_s is not None:
            _refuse_reference_index(reference_index, "align(window_s=...)")
            return self._align_windows(wave, sample_rate, reference, lengths, channel, reference_lengths,
                                       reference_sample_rate, window_s, window_hop_s, reference_margin_s)
        if reference_margin_s != 0:
            raise ValueError("reference_margin_s=%r: a margin widens reference windows; pass window_s and window_hop_s"
                             % (reference_margin_s,))
        deg, ref, counts, idx = self._arguments(wave, sample_rate, lengths, channel, reference, reference_lengths,
                                                reference_sample_rate, reference_index)
        out = self._scores_buffer(deg, ref, idx)
        n_rows = int(sum(counts))
        al, outs = self._alignment_buffers(n_rows)
        if out.shape[0] and idx is not None:
            self.engine.predict_device_batch_shared_ref(self._stream(), deg, ref, idx, out.data_ptr(), al,
                                                        target_sr=self.target_sr)
        elif out.shape[0]:
            self.engine.predict_device_batch_alignment(self._stream(), deg, ref, out.data_ptr(), al, target_sr=self.target_sr)
        i = np.concatenate([np.arange(c, dtype=np.float64) for c in counts]) if counts else np.zeros(0)
        z = np.zeros(n_rows)
        cols = self._alignment_times(outs, i, deg[0].sample_rate, ref[0].sample_rate, z, z)
        return Alignment(self._clip_rows(out, ref, idx), *outs, list(counts), *cols)

    def _align_windows(self, wave, sample_rate, reference, lengths, channel, reference_lengths, reference_sample_rate,
                       window_s, window_hop_s, reference_margin_s):
        made = []

        def buffers(n_segments, status):            # the rows: every segment of each pair's OK degraded window
            counts = np.where(status == E.CLIP_OK, n_segments, 0).astype(np.int64)
            made.append((counts,) + self._alignment_buffers(int(counts.sum())))
            return made[0][1]
        pairs = self._windows(wave, sample_rate, window_s, window_hop_s, lengths, channel, reference, reference_lengths,
                              reference_sample_rate, reference_margin_s, buffers)
        if not made:                                 # (no pair: nothing was enqueued)
            buffers(pairs.n_segments, pairs.status)
        counts, _, outs = made[0]
        n_rows = int(counts.sum())
        window = np.repeat(np.arange(len(counts), dtype=np.int64), counts)
        i = np.concatenate([np.arange(c, dtype=np.float64) for c in counts]) if n_rows else np.zeros(0)
        rate = self.target_sr or int(sample_rate)
        cols = self._alignment_times(outs, i, rate, rate, pairs.t_start[window], pairs.ref_t_start[window])
        return AlignmentWindows(pairs.scores, *outs, counts.tolist(), *cols, window, *pairs[1:])

    def _alignment_buffers(self, n_rows):
        outs = (torch.empty(n_rows, dtype=torch.int32, device=self.device),) + tuple(
            torch.empty(n_rows, dtype=torch.float32, device=self.device) for _ in range(3))
        al = E.NisqaAlignmentOut(*[t.data_ptr() or None for t in outs], n_rows)
        return al, outs

    def _alignment_times(self, outs, i, sr, ref_sr, off, ref_off):
        """-> (t_start, ref_t_start, delay_s, centroid_delay_s) of the rows: segment i of the degraded side starts at
        off + i seg_hop hop / rate, reference segment j at ref_off + j seg_hop ref_hop / ref_rate (each side at its own
        model rate and hop).  Waits for the alignment (a device-to-host copy of ref_seg and centroid)."""
        a = self.args
        rate, ref_rate = self.target_sr or int(sr), self.target_sr or int(ref_sr)
        step = a["ms_seg_hop_length"] * int(rate * a["ms_hop_length"]) / rate
        ref_step = a["ms_seg_hop_length"] * int(ref_rate * a["ms_hop_length"]) / ref_rate
        j = outs[0].cpu().numpy().astype(np.float64)
        j[j < 0] = np.nan
        cen = outs[2].cpu().numpy().astype(np.float64)
        t_start = off + i * step
        ref_t_start = ref_off + j * ref_step
        return t_start, ref_t_start, ref_t_start - t_start, ref_off + cen * ref_step - t_start

    def feed(self, n_feeds, sample_rate, window_s, window_hop_s, channel=None, max_push_s=None, reference=None,
             reference_margin_s=0.0, max_skew_s=None, reference_index=None):
        """A :class:`Feed` of ``n_feeds`` live recordings at ``sample_rate``, scored as the windows of :meth:`windows`
        (``window_s``, ``window_hop_s``, checked alike) as soon as each window is complete.  ``channel`` applies to every
        push (None: the mono mix); ``max_push_s`` (default ``window_s``) is the longest chunk one push may append to one
        feed, which sizes the feed's device rings.  A checkpoint with ``ms_sr`` takes feeds at that rate only.

        NISQA_DE: ``reference=True`` returns :class:`FeedPairs`, ``n_feeds`` live (degraded, reference) recording pairs
        scored as the window pairs of ``windows(..., reference=, reference_margin_s=)`` as soon as both windows of a pair
        are complete; ``channel`` applies to the degraded side, the reference is always the mono mix.  ``max_skew_s``
        (default ``max_push_s``) is the most a feed's two sides may differ in length after any push: pairs wait for the
        slower side, so the rings hold the faster side's backlog (device memory grows with it).  Recordings whose two
        sides end further apart than that need a larger ``max_skew_s``."""
        m = reference_margin_s
        _refuse_reference_index(reference_index, "feed")
        if reference is not None and not isinstance(reference, bool):
            raise TypeError("reference: True (NISQA_DE: live (degraded, reference) pairs) or None, not %r" % (reference,))
        if isinstance(m, bool) or not isinstance(m, numbers.Real) or not np.isfinite(m) or m < 0:
            raise ValueError("reference_margin_s: a non-negative number of seconds, not %r" % (m,))
        if not reference:
            if m != 0:
                raise ValueError("reference_margin_s=%r: a margin widens reference windows; pass reference=True "
                                 "(NISQA_DE)" % (m,))
            if max_skew_s is not None:
                raise ValueError("max_skew_s=%r: the skew of a feed's two sides; pass reference=True (NISQA_DE)"
                                 % (max_skew_s,))
            if self.double_ended:
                raise ValueError("feed: a double-ended (NISQA_DE) checkpoint scores (wave, reference) pairs, not live "
                                 "feeds; pass reference=True")
        elif not self.double_ended:
            raise ValueError("reference: only a double-ended (NISQA_DE) checkpoint scores live (degraded, reference) pairs")
        if isinstance(n_feeds, bool) or not isinstance(n_feeds, numbers.Integral) or not 1 <= n_feeds <= 65535:
            raise ValueError("n_feeds: an int within 1 .. 65535, not %r" % (n_feeds,))
        if isinstance(sample_rate, bool) or not isinstance(sample_rate, numbers.Integral) or sample_rate <= 0:
            raise ValueError("sample_rate must be a positive int, not %r" % (sample_rate,))
        if self.target_sr and sample_rate != self.target_sr:
            raise ValueError("sample_rate: %d Hz, but the checkpoint resamples to ms_sr=%d; a feed takes audio at ms_sr"
                             % (sample_rate, self.target_sr))
        if channel is not None and (isinstance(channel, bool) or not isinstance(channel, numbers.Integral) or channel < 0):
            raise TypeError("channel: a non-negative int or None, not %r" % (channel,))
        W, hop_frames = window_geometry(self.args, sample_rate, window_s, window_hop_s)
        a = self.args
        _, n_seg, status = E.segment_counts(self.cfg, W, sample_rate)
        if status != E.CLIP_OK:
            err = E.clip_status_error(status, "window_s=%r (%d samples at %d Hz)" % (window_s, W, sample_rate), W,
                                      sample_rate, n_seg, a["ms_hop_length"], a["ms_seg_length"], a["ms_max_segments"])
            raise ValueError("window_s: " + str(err))
        if max_push_s is None:
            max_push_s = window_s
        if isinstance(max_push_s, bool) or not isinstance(max_push_s, numbers.Real) or not np.isfinite(max_push_s) \
                or max_push_s <= 0 or int(round(max_push_s * sample_rate)) < 1:
            raise ValueError("max_push_s: a positive number of seconds (at least one sample), not %r" % (max_push_s,))
        max_push = int(round(max_push_s * sample_rate))
        if not reference:
            return Feed(self, int(n_feeds), int(sample_rate), W, hop_frames, channel, max_push)
        hop = int(sample_rate * a["ms_hop_length"])
        margin_frames = int(round(m * sample_rate / hop))
        M = margin_frames * hop
        _, n_seg, status = E.segment_counts(self.cfg, W + 2 * M, sample_rate)
        if status != E.CLIP_OK:
            raise ValueError("reference_margin_s=%r: reference windows of %d samples (W + 2 x %d) have %d segments > "
                             "ms_max_segments %d" % (m, W + 2 * M, M, n_seg, a["ms_max_segments"]))
        if max_skew_s is None:
            max_skew = max_push
        elif isinstance(max_skew_s, bool) or not isinstance(max_skew_s, numbers.Real) or not np.isfinite(max_skew_s) \
                or max_skew_s < 0:
            raise ValueError("max_skew_s: a non-negative number of seconds, not %r" % (max_skew_s,))
        else:
            max_skew = int(round(max_skew_s * sample_rate))
        return FeedPairs(self, int(n_feeds), int(sample_rate), W, hop_frames, channel, max_push, margin_frames, max_skew)

    def embed(self, wave, sample_rate, lengths=None, channel=None, reference=None, reference_lengths=None,
              reference_sample_rate=None, rows=False, reference_index=None):
        """Scores of a batch and the representation behind them -> :data:`Embeddings`.  Takes the arguments of
        ``__call__`` and checks them alike.

        scores : float32 [B, len(columns)], the values ``__call__`` returns
        pooled : float32 [B, len(columns), width] CUDA tensor: the input of each pooling head's last Linear (attention:
                 the softmax-weighted sum of the rows; avg: their mean; max: their column-wise max; last_step: the last
                 row; last_step_bi: the last row's forward half and the first row's backward half), so that a head's
                 score is pooled[b, h] @ w + b of that Linear.  NaN for a clip whose score is NaN
        rows   : float32 [N, width] CUDA tensor of every segment's row the pooling module reads, in the reference's
                 column order (``rows=True``), else None
        counts : host list of B ints, the segments of each clip (its rows follow those of the clips before it)
        NISQA_DE: one pooled vector per pair, rows for the degraded clips only.
        """
        deg, ref, counts, idx = self._arguments(wave, sample_rate, lengths, channel, reference, reference_lengths,
                                                reference_sample_rate, reference_index)
        out = self._scores_buffer(deg, ref, idx)
        width = self.engine.embedding_width()
        pooled = torch.empty((out.shape[0], len(self.columns), width), dtype=torch.float32, device=self.device)
        n_rows = int(sum(counts))
        seg_rows = torch.empty((n_rows, width), dtype=torch.float32, device=self.device) if rows else None
        if out.shape[0] and idx is not None:
            eo = E.NisqaEmbeddingOut(pooled=pooled.data_ptr() or None, rows=seg_rows.data_ptr() if rows else None,
                                     n_rows=n_rows)
            self.engine.predict_device_batch_shared_ref(self._stream(), deg, ref, idx, out.data_ptr(), eo,
                                                        target_sr=self.target_sr)
        elif out.shape[0]:
            self.engine.predict_device_batch_embeddings(self._stream(), deg, out.data_ptr(), pooled.data_ptr(),
                                                        seg_rows.data_ptr() if rows else 0, n_rows, ref=ref,
                                                        target_sr=self.target_sr)
        return Embeddings(self._clip_rows(out, ref, idx), self._clip_rows(pooled, ref, idx), seg_rows, list(counts))

    # ------------------------------------------------------------------ shared by __call__, segments and embed
    def _arguments(self, wave, sample_rate, lengths, channel, reference, reference_lengths, reference_sample_rate,
                   reference_index=None):
        """-> (deg, ref or None, segment counts of wave's clips, reference_index as int32 or None) after every check,
        before anything is enqueued"""
        if reference_index is not None and not self.double_ended:
            raise ValueError("reference_index: only a double-ended (NISQA_DE) checkpoint pairs clips with references")
        if self.double_ended and reference is None:
            raise ValueError("reference: a double-ended (NISQA_DE) checkpoint scores (wave, reference) pairs")
        if not self.double_ended and reference is not None:
            raise ValueError("reference: only a double-ended (NISQA_DE) checkpoint takes reference clips")
        deg = self._batch("wave", wave, sample_rate, lengths, channel)
        ref = None
        if reference is not None:
            ref = self._batch("reference", reference, sample_rate if reference_sample_rate is None else reference_sample_rate,
                              reference_lengths, None)
            if reference_index is None and ref[0].n_clips != deg[0].n_clips:
                raise ValueError("reference: %d clips for %d clips of wave" % (ref[0].n_clips, deg[0].n_clips))
        idx = None
        if reference_index is not None:
            idx = _host_ints("reference_index", reference_index, deg[0].n_clips)
            bad = np.nonzero((idx < 0) | (idx >= ref[0].n_clips))[0]
            if bad.size:
                raise ValueError("reference_index[%d] = %d: not within 0 .. %d (the clips of reference)"
                                 % (bad[0], idx[bad[0]], ref[0].n_clips - 1))
            idx = idx.astype(np.int32)
        counts = self._check_segments("wave", deg[1], deg[0].sample_rate)
        if ref is not None:      # (shared references: the ones some clip names)
            self._check_segments("reference", ref[1], ref[0].sample_rate, None if idx is None else np.unique(idx))
        return deg, ref, counts, idx

    def _scores_buffer(self, deg, ref, idx=None):
        n = deg[0].n_clips * (2 if ref is not None and idx is None else 1)
        return torch.empty((n, len(self.columns)), dtype=torch.float32, device=self.device)

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    @staticmethod
    def _clip_rows(out, ref, idx=None):
        # (NISQA_DE: row 2p holds pair p's score, row 2p + 1 is the reference clip's NaN row; shared references: compact)
        return out[0::2].contiguous() if ref is not None and idx is None else out

    # ------------------------------------------------------------------ arguments
    def _batch(self, name, x, sample_rate, lengths, channel, min_len=1):
        """-> engine.device_batch(...) of one batch argument, after the argument checks (lengths >= min_len)"""
        if not isinstance(x, torch.Tensor):
            raise TypeError("%s: a torch.Tensor on the GPU, not %s" % (name, type(x).__name__))
        if x.dtype not in (torch.int16, torch.float32):
            raise TypeError("%s: dtype %s; the engine reads int16 or float32 samples (convert with .float())" % (name, x.dtype))
        if x.device != self.device:
            raise ValueError("%s: on %s, the scorer runs on %s" % (name, x.device, self.device))
        if x.dim() not in (1, 2, 3):
            raise ValueError("%s: shape %s; expected [T], [B, T] or [B, C, T]" % (name, tuple(x.shape)))
        if isinstance(sample_rate, bool) or not isinstance(sample_rate, numbers.Integral) or sample_rate <= 0:
            raise ValueError("%s: sample_rate must be a positive int, not %r" % (name, sample_rate))
        x3 = x.reshape(1, 1, -1) if x.dim() == 1 else x.unsqueeze(1) if x.dim() == 2 else x
        B, C, T = x3.shape
        if T < 1:
            raise ValueError("%s: no samples" % name)
        if T > 1 and x3.stride(2) != 1:
            raise ValueError("%s: samples must be contiguous (stride 1 along the last dimension, got %d)" % (name, x3.stride(2)))
        if channel is None:
            ch = -1
        elif isinstance(channel, bool) or not isinstance(channel, numbers.Integral):
            raise TypeError("channel: an int or None, not %r" % (channel,))
        elif not 0 <= channel < C:
            raise ValueError("channel: %d is out of range for %d channel(s)" % (channel, C))
        else:
            ch = int(channel)
        what = "reference_lengths" if name == "reference" else "lengths"
        if lengths is None:
            ns = np.full(B, T, dtype=np.int64)
        else:
            ns = _host_ints(what, lengths, B)
            bad = np.nonzero((ns < min_len) | (ns > T))[0]
            if bad.size:
                raise ValueError("%s[%d] = %d: not within %d .. %d samples" % (what, bad[0], ns[bad[0]], min_len, T))
        fmt = E.FMT_S16 if x.dtype == torch.int16 else E.FMT_F32
        return E.device_batch(x3.data_ptr(), fmt, ns, C, ch, T, x3.stride(0), x3.stride(1), int(sample_rate))

    def _check_segments(self, name, n_samples, sample_rate, which=None):
        """The file ingest's too-short / too-long errors (NISQA_lib._raise_for_status), on the host, before any launch,
        for every clip or the clips ``which`` names.  Returns each clip's segment count."""
        from . import resample as RS
        rate = self.target_sr or sample_rate
        a = self.args
        counts = []
        for i, n in enumerate(n_samples):
            if which is not None and i not in which:
                counts.append(0)
                continue
            n = int(n) if rate == sample_rate else RS.out_len(int(n), sample_rate, rate)
            _, n_seg, status = E.segment_counts(self.cfg, n, rate)
            err = E.clip_status_error(status, "%s[%d]" % (name, i), n, rate, n_seg, a["ms_hop_length"], a["ms_seg_length"],
                                      a["ms_max_segments"])
            if err is not None:
                raise err
            counts.append(n_seg)
        return counts


def _host_ints(what, x, B):
    """-> int64 [B] of a host-integer argument (a list, NumPy array or CPU tensor; ``lengths``, ``reference_index``)"""
    if isinstance(x, torch.Tensor) and x.device.type != "cpu":
        raise TypeError("%s: host integers (a list, NumPy array or CPU tensor), not a CUDA tensor" % what)
    a = np.asarray(x.tolist() if isinstance(x, torch.Tensor) else x)
    if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
        raise TypeError("%s: one int per clip" % what)
    a = a.astype(np.int64)
    if a.shape[0] != B:
        raise ValueError("%s: %d entries for %d clips" % (what, a.shape[0], B))
    return a


def _refuse_reference_index(reference_index, where):
    if reference_index is not None:
        raise ValueError("reference_index: %s takes one reference recording per recording; shared references are for "
                         "clip pairs (__call__, segments, embed, align)" % where)


class Feed(object):
    """Live recordings scored window by window as their samples arrive (``Scorer.feed``).  Holds device rings of
    ``device_bytes`` bytes until ``close()``.  Pushes are ordered on ``torch.cuda.current_stream()`` at each call; the
    feed runs them in push order whatever streams they come from."""

    def __init__(self, scorer, n_feeds, sample_rate, W, hop_frames, channel, max_push):
        self.scorer, self.n_feeds, self.sample_rate, self.channel, self.max_push = scorer, n_feeds, sample_rate, channel, max_push
        self.window, self.hop_frames = W, hop_frames
        self.hop = hop_frames * int(sample_rate * scorer.args["ms_hop_length"])
        self.held = np.zeros(n_feeds, np.int64)          # samples of each feed's current recording
        self._fmt = None                                  # the format the feeds' samples are held in
        self._h = self._create()

    def _create(self):
        return self.scorer.engine.feed_create(self.n_feeds, self.sample_rate, self.window, self.hop_frames, self.max_push)

    @property
    def device_bytes(self):
        return self.scorer.engine.feed_device_bytes(self._h)

    def close(self):
        if self._h is not None:
            self.scorer.engine.feed_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push(self, wave, lengths=None, end=None):
        """Append a chunk to every feed and score the windows it completes -> :data:`FeedRows`.

        wave    : [B, T] or [B, C, T] int16 / float32 CUDA tensor, B = n_feeds (a [T] tensor for one feed), T >= 0
        lengths : host ints, the samples of each feed's chunk, 0 .. T and at most max_push_s (default T)
        end     : host bools, one per feed: the feed's recording ends after this chunk; its remaining windows are scored
                  as ``Scorer.windows`` scores the last ones (the last may be short: NaN, CLIP_TOO_SHORT) and the next
                  sample pushed to it starts a new recording
        Window k of a feed is emitted by the first push after which the feed holds k H + W samples of its recording,
        with the scores ``Scorer.windows`` gives that window of the whole recording, bit for bit.
        """
        deg = self._chunk("wave", wave, lengths, self.channel)
        ends = self._ends(end)
        b, ns = deg
        self._check_format(self._format(b), ns.sum() > 0, self.held.sum() > 0, "wave")
        eng = self.scorer.engine
        feed, index, _, _ = E.feed_rows(self.scorer.cfg, self.sample_rate, self.window, self.hop_frames, self.held, ns, ends)
        N = feed.shape[0]
        out = torch.empty((N, len(self.scorer.columns)), dtype=torch.float32, device=self.scorer.device)
        f2, i2, nseg, status = eng.feed_push(self._h, self.scorer._stream(), deg, ends, out.data_ptr(), N)
        T = self.held + ns
        t_start = index * self.hop / self.sample_rate
        t_end = np.minimum(index * self.hop + self.window, T[feed]) / self.sample_rate
        if ns.sum() > 0:
            self._fmt = self._format(b)
        self.held = np.where(ends.astype(bool), 0, T)
        return FeedRows(out, f2, i2, t_start, t_end, nseg, status)

    # ------------------------------------------------------------------ shared by Feed.push and FeedPairs.push
    def _chunk(self, name, wave, lengths, channel):
        """-> engine.device_batch(...) of one chunk argument (``wave`` or ``reference``), after its checks"""
        if self._h is None:
            raise ValueError("push: the feed is closed")
        what = "reference_lengths" if name == "reference" else "lengths"
        if isinstance(wave, torch.Tensor) and wave.shape[-1] == 0:
            if lengths is not None and np.any(np.asarray(lengths) != 0):
                raise ValueError("%s: a chunk of 0 samples holds no sample" % what)
            wave = torch.zeros(tuple(wave.shape[:-1]) + (1,), dtype=wave.dtype, device=wave.device)
            lengths = [0] * (wave.shape[0] if wave.dim() > 1 else 1)
        batch = self.scorer._batch(name, wave, self.sample_rate, lengths, channel, min_len=0)
        b, ns = batch
        if b.n_clips != self.n_feeds:
            raise ValueError("%s: %d feeds (clips) in the chunk for a feed object of %d feeds" % (name, b.n_clips, self.n_feeds))
        over = np.nonzero(ns > self.max_push)[0]
        if over.size:
            raise ValueError("%s[%d] = %d: more than max_push_s (%d samples)" % (what, over[0], ns[over[0]], self.max_push))
        return batch

    def _ends(self, end):
        if end is None:
            return np.zeros(self.n_feeds, np.uint8)
        ends = np.asarray(end.tolist() if isinstance(end, torch.Tensor) else end)
        if ends.shape != (self.n_feeds,) or not (ends.dtype == np.bool_ or np.issubdtype(ends.dtype, np.integer)):
            raise ValueError("end: one bool per feed (%d), not %r" % (self.n_feeds, end))
        return ends.astype(bool).astype(np.uint8)

    @staticmethod
    def _format(b):
        """the ring format of a chunk: mono int16 (one channel, or one picked) or float32 (float32 or mixed)"""
        return E.FMT_S16 if b.sample_fmt == E.FMT_S16 and (b.n_channels == 1 or b.channel >= 0) else E.FMT_F32

    def _check_format(self, fmt, pushes, holds, name):
        if pushes and holds and fmt != self._fmt:
            raise ValueError("%s: %s samples, but the feeds hold %s ones until every feed has ended" % (
                name, "mono int16" if fmt == E.FMT_S16 else "float32 (or mixed)",
                "mono int16" if self._fmt == E.FMT_S16 else "float32 (or mixed)"))


class FeedPairs(Feed):
    """Live (degraded, reference) recording pairs of a NISQA_DE checkpoint scored window pair by window pair as both
    sides' samples arrive (``Scorer.feed(..., reference=True)``).  Closes, reports ``device_bytes`` and orders its pushes
    as :class:`Feed`."""

    def __init__(self, scorer, n_feeds, sample_rate, W, hop_frames, channel, max_push, margin_frames, max_skew):
        self.margin_frames, self.max_skew = margin_frames, max_skew
        self.margin = margin_frames * int(sample_rate * scorer.args["ms_hop_length"])
        self.ref_held = np.zeros(n_feeds, np.int64)      # reference samples of each feed's current recording pair
        super(FeedPairs, self).__init__(scorer, n_feeds, sample_rate, W, hop_frames, channel, max_push)

    def _create(self):
        return self.scorer.engine.feed_pair_create(self.n_feeds, self.sample_rate, self.window, self.hop_frames,
                                                   self.margin_frames, self.max_push, self.max_skew)

    def push(self, wave, reference, lengths=None, reference_lengths=None, end=None):
        """Append a degraded and a reference chunk to every feed and score the window pairs they complete ->
        :data:`FeedPairRows`.

        wave, lengths      : the degraded chunks, as :meth:`Feed.push` (the feed's ``channel`` applies)
        reference          : the reference chunks, [B, T] or [B, C, T] int16 / float32 CUDA tensor (always mixed to mono),
                             with their own ``reference_lengths``; either side may bring 0 samples
        end                : host bools, one per feed: both recordings of the feed end after this push; its remaining
                             pairs are scored as ``Scorer.windows(..., reference=)`` scores the last ones of the final
                             lengths (a reference window that is empty scores NaN with ``ref_status`` CLIP_TOO_SHORT), and
                             the next sample on either side starts a new pair of recordings
        Pair k of a feed is emitted by the first push after which the feed holds k H + W degraded and k H + W + M
        reference samples, with the scores ``Scorer.windows(..., reference=, reference_margin_s=)`` gives that pair of
        the whole recordings, bit for bit.  Both sides share one sample format (float32 if either is float32 or mixed),
        which holds until every feed has ended; after a push, a feed's two lengths may differ by at most max_skew_s.
        """
        deg = self._chunk("wave", wave, lengths, self.channel)
        ref = self._chunk("reference", reference, reference_lengths, None)
        ends = self._ends(end)
        (b, ns), (rb, rns) = deg, ref
        T, T_ref = self.held + ns, self.ref_held + rns
        skew = np.nonzero(np.abs(T - T_ref) > self.max_skew)[0]
        if skew.size:
            i = skew[0]
            raise ValueError("lengths / reference_lengths: feed %d would hold %d degraded and %d reference samples, more "
                             "than max_skew_s (%d samples) apart" % (i, T[i], T_ref[i], self.max_skew))
        fmt = E.FMT_F32 if E.FMT_F32 in (self._format(b), self._format(rb)) else E.FMT_S16
        pushes = ns.sum() + rns.sum() > 0
        self._check_format(fmt, pushes, self.held.sum() + self.ref_held.sum() > 0, "wave / reference")
        eng = self.scorer.engine
        feed, index = E.feed_pair_rows(self.scorer.cfg, self.sample_rate, self.window, self.hop_frames, self.margin_frames,
                                       self.held, self.ref_held, ns, rns, ends)[:2]
        N = feed.shape[0]
        out = torch.empty((N, len(self.scorer.columns)), dtype=torch.float32, device=self.scorer.device)
        rows = eng.feed_pair_push(self._h, self.scorer._stream(), deg, ref, ends, out.data_ptr(), N)
        kH, W, M, rate = index * self.hop, self.window, self.margin, self.sample_rate
        r0 = np.maximum(0, kH - M)
        r1 = np.maximum(r0, np.minimum(T_ref[feed], kH + W + M))
        if pushes:
            self._fmt = fmt
        self.held = np.where(ends.astype(bool), 0, T)
        self.ref_held = np.where(ends.astype(bool), 0, T_ref)
        return FeedPairRows(out, rows[0], rows[1], kH / rate, np.minimum(kH + W, T[feed]) / rate, rows[2], rows[3],
                            r0 / rate, r1 / rate, rows[4], rows[5])
