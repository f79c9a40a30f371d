"""Host-side mirror of the reference's predict seam (reference nisqa/NISQA_lib.py:1420-1467,
2052-2236) with the hot path replaced by the engine.

Same names, argument meaning and error behaviour as the reference so that
``nisqaModel.predict()`` reads the same:

* :func:`predict_dim` / :func:`predict_mos` take ``(model, ds, bs, dev, num_workers)``, return
  ``(y_hat, y)`` and add ``mos_pred`` (+ ``noi_pred, dis_pred, col_pred, loud_pred``) to
  ``ds.df`` in dataset row order; ``predict_mos`` stores float64, ``predict_dim`` float32.
* ``model`` is an :class:`nisqa_b200.engine.Engine` instead of an ``nn.Module``; one batch of
  ``bs`` clips becomes ONE C-ABI call (wav decode -> PCM pointers -> scores), there is no
  padded ``[bs, 1300, 1, 48, 15]`` tensor and no DataLoader.  ``num_workers`` sizes the thread pool
  that drives the native wav reader (csrc/wavio.cpp) straight into pinned batch buffers while the
  GPU works on earlier batches.
* errors are the reference's ``ValueError``s: unreadable file (lib:2305-2306), clip shorter
  than ``seg_length`` frames (lib:2258-2263), more than ``ms_max_segments`` segments
  (lib:2276-2277) - a single bad file aborts the run, like the reference.
* under ``torchrun`` (WORLD_SIZE > 1) the rows are sharded over the ranks and the scores are
  all-gathered once (``nisqa_b200/dist.py``); every rank ends up with the full table.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import dist as nb_dist
from . import engine as nb_engine
from . import resample as nb_resample
from .wav import decode_batch, decode_wav_into, probe_batch, read_wav


class SpeechQualityDataset(object):
    """Predict-only subset of the reference Dataset (lib:2052-2236): holds the table of files
    and the front-end parameters; ``load_pcm(index)`` replaces ``__getitem__`` (no mel, no
    segment tensor on the host)."""

    def __init__(self, df, df_con=None, data_dir="", folder_column="", filename_column="filename",
                 mos_column="MOS", seg_length=15, max_length=None, to_memory=False,
                 to_memory_workers=0, transform=None, seg_hop_length=1, ms_n_fft=1024,
                 ms_hop_length=80, ms_win_length=170, ms_n_mels=32, ms_sr=48e3, ms_fmax=16e3,
                 ms_channel=None, double_ended=False, filename_column_ref=None, dim=False):
        if double_ended and filename_column_ref is None:
            # the reference indexes df[None] here (lib:2133) - predict_file / predict_dir have no reference column
            raise KeyError(filename_column_ref)
        if mos_column != "predict_only":
            raise NotImplementedError("only predict_only datasets are on the engine path")
        if transform is not None or to_memory:
            raise NotImplementedError("transform / to_memory are training-side options")
        self.df = df
        self.df_con = df_con
        self.data_dir = data_dir
        self.filename_column = filename_column
        self.mos_column = mos_column
        self.seg_length = seg_length
        self.seg_hop_length = seg_hop_length
        self.max_length = max_length
        self.ms_n_fft, self.ms_hop_length, self.ms_win_length = ms_n_fft, ms_hop_length, ms_win_length
        self.ms_n_mels, self.ms_sr, self.ms_fmax = ms_n_mels, ms_sr, ms_fmax
        self.ms_channel = ms_channel
        self.double_ended = bool(double_ended)
        self.filename_column_ref = filename_column_ref
        self._paths = None
        self.dim = dim

    def __len__(self):
        return len(self.df)

    def file_path(self, index):
        # (the column is read once: a pandas scalar lookup per file costs more than decoding a short clip)
        if self._paths is None or len(self._paths) != len(self.df):
            self._paths = [os.path.join(self.data_dir, f) for f in self.df[self.filename_column].tolist()]
        return self._paths[index]

    def file_path_ref(self, index):
        """Reference signal of a double-ended row (lib:2132-2134)."""
        return os.path.join(self.data_dir, self.df[self.filename_column_ref].iloc[index])

    def target_sr(self):
        """``ms_sr`` of the checkpoint as an int, or None (= every file at its native rate, lib:2300)."""
        return None if self.ms_sr is None else int(self.ms_sr)

    def load_pcm(self, index):
        """-> (int16|float32 mono samples, sample_rate); ValueError('Could not load file ..').  With
        ``ms_sr`` set the clip is converted to that rate (lb.load(path, sr=ms_sr), lib:2300-2304)."""
        y, sr = read_wav(self.file_path(index), self.ms_channel)
        target = self.target_sr()
        if target is not None and sr != target:
            try:
                y, sr = nb_resample.resample(y, sr, target), target
            except Exception:
                raise ValueError("Could not load file {}".format(self.file_path(index)))
        return y, sr


def _raise_for_status(ds, engine, index, n_samples, sr, n_seg, status):
    err = nb_engine.clip_status_error(status, ds.file_path(index), n_samples, sr, n_seg, ds.ms_hop_length, ds.seg_length,
                                      ds.max_length)
    if err is not None:
        raise err


class _PinnedPool(object):
    """Grow-only ring of pinned host buffers: a batch is decoded straight into one of them (native
    reader, csrc/wavio.cpp), clips back to back at the engine's 16-sample alignment, so the whole
    batch travels to the GPU as ONE asynchronous copy."""

    def __init__(self, n):
        self.bufs = [None] * n

    def get(self, slot, nbytes):
        import torch
        cur = self.bufs[slot]
        if cur is None or cur.numel() < nbytes:
            cur = torch.empty(max(int(nbytes * 1.25), 1 << 20), dtype=torch.uint8).pin_memory()
            self.bufs[slot] = cur
        return cur.numpy()


def _load_batch(ds, batch, pool, slot, n_threads):
    """wav files of one batch -> (list of 1-D views into a pinned buffer, sample rates).  Two native
    calls per batch (probe, decode), each spread over ``n_threads`` C++ threads."""
    paths = [ds.file_path(int(i)) for i in batch]
    sr, nf, kind, arr = probe_batch(paths, ds.ms_channel, n_threads)
    target = ds.target_sr()
    if target is not None and bool((sr != target).any()) and os.environ.get("NISQA_RESAMPLE", "device") == "host":
        return _load_batch_resampled(ds, paths, sr, nf, target, pool, slot, n_threads)     # host threads (A/B, tests)
    dtype = np.int16 if not kind.any() else np.float32
    offs = np.zeros(len(paths), np.int64)
    if len(paths) > 1:
        offs[1:] = np.cumsum((nf[:-1] + 15) // 16 * 16)
    total = int(offs[-1] + (nf[-1] + 15) // 16 * 16) if len(paths) else 0
    nbytes = max(total, 16) * np.dtype(dtype).itemsize
    buf = pool.get(slot, nbytes)[:nbytes].view(dtype)
    decode_batch(arr, len(paths), buf, offs, nf, ds.ms_channel, n_threads, paths)
    clips = [buf[int(o):int(o) + int(n)] for o, n in zip(offs, nf)]
    return clips, [int(x) for x in sr]


def _load_batch_resampled(ds, paths, sr, nf, target, pool, slot, n_threads):
    """``ms_sr`` checkpoints (lib:2300-2304): every clip is decoded to float32 (mono mix / channel pick first, as
    librosa does) and converted to ``target`` Hz straight into the pinned batch buffer; one native decode + one
    native resample call per file, spread over ``n_threads`` threads (ctypes releases the GIL)."""
    n_out = np.array([nb_resample.out_len(int(n), int(s), target) for n, s in zip(nf, sr)], np.int64)
    offs = np.zeros(len(paths), np.int64)
    if len(paths) > 1:
        offs[1:] = np.cumsum((n_out[:-1] + 15) // 16 * 16)
    total = int(offs[-1] + (n_out[-1] + 15) // 16 * 16) if len(paths) else 0
    buf = pool.get(slot, max(total, 16) * 4)[:max(total, 16) * 4].view(np.float32)

    def one(i):
        dst = buf[int(offs[i]):int(offs[i]) + int(n_out[i])]
        if int(sr[i]) == target:
            decode_wav_into(paths[i], dst, ds.ms_channel)
            return
        tmp = np.empty(int(nf[i]), np.float32)
        decode_wav_into(paths[i], tmp, ds.ms_channel)
        try:
            nb_resample.resample(tmp, int(sr[i]), target, out=dst)
        except Exception:
            raise ValueError("Could not load file {}".format(paths[i]))

    if n_threads > 1 and len(paths) > 1:
        with ThreadPoolExecutor(max_workers=n_threads) as ex:
            list(ex.map(one, range(len(paths))))
    else:
        for i in range(len(paths)):
            one(i)
    clips = [buf[int(o):int(o) + int(n)] for o, n in zip(offs, n_out)]
    return clips, [target] * len(paths)


def _load_batch_de(ds, batch):
    """Double-ended rows (lib:2132-2156): the degraded files (``ms_channel`` applies) and each distinct reference file of
    the batch once (always the mono mix: the reference call passes no ``ms_channel``, lib:2146-2154), in the order the
    rows first name them; ``ms_sr`` converts each decoded file once.  -> (degraded clips, their rates, reference clips,
    their rates, ref_index: each row's reference).  Mixed sample formats go through float32 (submit_pcm_pairs)."""
    target = ds.target_sr()

    def load(path, ch):
        y, sr = read_wav(path, ch)
        if target is not None and sr != target:
            try:
                y, sr = nb_resample.resample(y, sr, target), target
            except Exception:
                raise ValueError("Could not load file {}".format(path))
        return np.ascontiguousarray(y), int(sr)

    clips, srs, refs, ref_srs, ref_index, seen = [], [], [], [], [], {}
    for i in batch:
        y, sr = load(ds.file_path(int(i)), ds.ms_channel)
        clips.append(y)
        srs.append(sr)
        path = ds.file_path_ref(int(i))
        if path not in seen:
            seen[path] = len(refs)
            y, sr = load(path, None)
            refs.append(y)
            ref_srs.append(sr)
        ref_index.append(seen[path])
    return clips, srs, refs, ref_srs, ref_index


def _predict_rows(engine, ds, rows, bs, num_workers):
    """Scores for the given dataset rows (in that order) through the C-ABI, bs clips per call.
    Pipeline: decode batch b+1 (thread pool, native reader -> pinned memory) while the engine has up
    to five earlier batches in flight (H2D on the copy stream, kernels on rotating compute lanes)."""
    n_out = engine.n_out
    out = np.empty((len(rows), n_out), dtype=np.float32)
    bs = max(1, int(bs))
    batches = [rows[i:i + bs] for i in range(0, len(rows), bs)]
    # native decode threads per batch; three batches are decoded concurrently (DEPTH), so more than half of the CPUs the
    # process is granted per batch only oversubscribes them
    n_threads = max(1, min(int(num_workers) if num_workers else 1, max(1, nb_dist.usable_cpus() // 2)))

    de = getattr(ds, "double_ended", False)
    order = np.arange(len(rows))
    if de:
        # a double-ended row is a (degraded, reference) pair; rows that share a reference file (a condition sweep) are
        # submitted next to each other, so that a batch decodes, uploads and computes that reference once.  The stable
        # sort keeps CSV order among them; the scores go back to the given row order.
        order = np.argsort(np.array([ds.file_path_ref(int(i)) for i in rows], dtype=object), kind="stable")
        batches = [np.asarray(rows)[order[i:i + bs]] for i in range(0, len(rows), bs)]

    def finish(job):
        handle, batch, clips, srs, pos, shared = job
        scores, nseg, status = engine.wait(handle)
        # (the reference names the degraded file for either signal, lib:2187-2192)
        if shared:      # one score per pair; the references' statuses come apart
            refs, ref_srs, ref_index = shared
            ref_nseg, ref_status = handle[4], handle[5]
            for j, st in enumerate(status):
                u = ref_index[j]
                if st != nb_engine.CLIP_OK:
                    _raise_for_status(ds, engine, int(batch[j]), clips[j].shape[0], srs[j], int(nseg[j]), int(st))
                if ref_status[u] != nb_engine.CLIP_OK:
                    _raise_for_status(ds, engine, int(batch[j]), refs[u].shape[0], ref_srs[u], int(ref_nseg[u]),
                                      int(ref_status[u]))
            out[order[pos:pos + len(batch)]] = scores
            return
        per_row = 2 if de else 1          # (a double-ended row: the clips of its (degraded, reference) pair)
        for j, st in enumerate(status):
            if st != nb_engine.CLIP_OK:
                _raise_for_status(ds, engine, int(batch[j // per_row]), clips[j].shape[0], srs[j], int(nseg[j]), int(st))
        out[order[pos:pos + len(batch)]] = scores[::per_row]

    DEPTH = 3                         # batches being decoded ahead of the GPU
    FLIGHT = 5                        # submissions kept in flight on the engine (it has 6 staging slots)
    pool = _PinnedPool(FLIGHT + DEPTH + 1)
    in_flight = []                    # batches whose kernels are running while later ones are decoded
    try:
        with ThreadPoolExecutor(max_workers=DEPTH) as feeder:
            pending = []
            nxt = 0

            def top_up():
                nonlocal nxt
                while nxt < len(batches) and len(pending) < DEPTH:
                    if de:
                        pending.append(feeder.submit(_load_batch_de, ds, batches[nxt]))
                    else:
                        pending.append(feeder.submit(_load_batch, ds, batches[nxt], pool, nxt % len(pool.bufs), n_threads))
                    nxt += 1

            top_up()
            pos = 0
            for b, batch in enumerate(batches):
                shared = None
                if de:
                    clips, srs, refs, ref_srs, ref_index = pending.pop(0).result()
                    if len(refs) < len(clips):      # a reference repeats: computed once per engine pass
                        shared = (refs, ref_srs, ref_index)
                    else:                           # every reference once: the (degraded, reference) clip pairs
                        clips = [c for j, u in enumerate(ref_index) for c in (clips[j], refs[u])]
                        srs = [r for j, u in enumerate(ref_index) for r in (srs[j], ref_srs[u])]
                        if any(c.dtype != clips[0].dtype for c in clips):
                            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0)
                                     for c in clips]
                else:
                    clips, srs = pending.pop(0).result()
                target = ds.target_sr()
                if shared:
                    handle = engine.submit_pcm_pairs(clips, srs, refs, ref_srs, ref_index)
                elif target is not None and not de and any(sr != target for sr in srs):
                    # ms_sr checkpoint (lib:2300-2304): the clips travel at their native rates and are converted on
                    # the device (csrc/resample_gpu.cu), where the predict path picks them up - one synchronous call
                    handle = (None,) + tuple(engine.predict_pcm_resampled(clips, srs, target))
                    srs = [target] * len(srs)
                else:
                    handle = engine.submit_pcm(clips, srs)      # asynchronous: H2D + kernels enqueued
                in_flight.append((handle, batch, clips, srs, pos, shared))
                pos += len(batch)
                if len(in_flight) >= FLIGHT:
                    finish(in_flight.pop(0))
                top_up()                                        # a pinned slot is recycled only after its batch finished
            while in_flight:
                finish(in_flight.pop(0))
    except BaseException:
        # a bad file (pending.result()) or a too short / too long clip (finish()) unwinds the loop while earlier
        # submissions still hold raw pointers into `in_flight`'s score arrays and the pinned PCM buffers: make the
        # engine forget them before those buffers are released (the reference simply raises, lib:2305-2306)
        engine.drain()
        raise
    return out


def _predict_all(engine, ds, bs, num_workers):
    n = len(ds)
    rank, world, _ = nb_dist.env_world()
    if world > 1:
        import torch.distributed as tdist
        if not tdist.is_initialized():
            nb_dist.init_process_group()
        sizes = []
        for i in range(n):
            try:
                sizes.append(os.path.getsize(ds.file_path(i)))
            except OSError:
                sizes.append(0)
        shards = nb_dist.shard_rows(sizes, world)
        # a per-file ValueError (unreadable / too short / too long) fires on the one rank that owns the row; the
        # others would block in the score gather.  Exchange (ok, message) first and raise the same error everywhere
        # (the reference is single-process and simply raises, lib:2258-2263, 2276-2277, 2305-2306).
        local, failure = None, None
        try:
            local = _predict_rows(engine, ds, shards[rank], bs, num_workers)
        except ValueError as exc:
            failure = str(exc)
        reports = [None] * world
        tdist.all_gather_object(reports, failure)
        for msg in reports:                 # lowest rank first: every rank raises the same message
            if msg is not None:
                raise ValueError(msg)
        return nb_dist.all_gather_scores(local, shards, n, engine=engine)
    return _predict_rows(engine, ds, np.arange(n, dtype=np.int64), bs, num_workers)


def predict_mos(model, ds, bs, dev, num_workers=0):
    """MOS-only models (reference lib:1420-1439): adds ``mos_pred`` (float64) to ``ds.df``."""
    y_hat = _predict_all(model, ds, bs, num_workers)[:, :1].reshape(-1, 1)
    y = np.full((len(ds), 1), np.nan, dtype=np.float32)          # predict_only labels (lib:2224-2225)
    ds.df["mos_pred"] = y_hat.astype(dtype=float)
    return y_hat, y


def predict_dim(model, ds, bs, dev, num_workers=0):
    """NISQA_DIM models (reference lib:1441-1467): adds the five ``*_pred`` columns (float32)."""
    y_hat = _predict_all(model, ds, bs, num_workers)
    y = np.full((len(ds), 5), np.nan, dtype=np.float32)          # predict_only labels (lib:2217-2219)
    ds.df["mos_pred"] = y_hat[:, 0].reshape(-1, 1)
    ds.df["noi_pred"] = y_hat[:, 1].reshape(-1, 1)
    ds.df["dis_pred"] = y_hat[:, 2].reshape(-1, 1)
    ds.df["col_pred"] = y_hat[:, 3].reshape(-1, 1)
    ds.df["loud_pred"] = y_hat[:, 4].reshape(-1, 1)
    return y_hat, y
