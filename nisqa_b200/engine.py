"""ctypes binding of libnisqa_b200.so (include/nisqa_b200.h) - the only way Python reaches the
CUDA hot path.  PyTorch / NumPy arrays are used as containers only: the library receives raw
pointers and sizes.

There is no CPU fallback: if the shared library is missing or no CUDA device is usable,
constructing an :class:`Engine` raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnisqa_b200.so")

ABI_VERSION = 3
MAX_IN_FLIGHT = 6          # staging slots of the engine (nisqa_submit_pcm)
ARCH_ADAPT_SA_ATTFF, ARCH_STD_LSTM_LASTBI = 0, 1
FMT_S16, FMT_F32 = 0, 1
CLIP_OK, CLIP_TOO_SHORT, CLIP_TOO_LONG = 0, 1, 2
POOL_ATT_FF, POOL_ATT, POOL_AVG, POOL_MAX, POOL_LAST_STEP, POOL_LAST_STEP_BI = range(6)
# NISQA_DE options (enum nisqa_de_align / nisqa_de_apply / nisqa_de_fuse)
CNN_CONV, CNN_SKIP, CNN_DFF = 0, 1, 2
DE_ALIGN = {"dot": 1, "cosine": 2, "distance": 3, "luong": 4, "bahd": 5}
DE_APPLY = {"hard": 0, "soft": 1}
DE_FUSE = {"x/y/-": 0, "+/-": 1, "x/y": 2}
(STAGE_MEL_DB, STAGE_POOL1, STAGE_POOL2, STAGE_CONV3, STAGE_POOL3, STAGE_CONV5, STAGE_CNN_FEAT,
 STAGE_TD_IN, STAGE_TD_OUT) = range(9)

# every symbol include/nisqa_b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "nisqa_create", "nisqa_destroy", "nisqa_last_error", "nisqa_load_weights",
    "nisqa_predict_pcm", "nisqa_predict_pcm_device", "nisqa_stage_dump", "nisqa_segment_counts",
    "nisqa_mel_filterbank", "nisqa_gather_nccl", "nisqa_nccl_unique_id", "nisqa_nccl_init",
    "nisqa_kernel_launches", "nisqa_stream", "nisqa_set_profiling", "nisqa_group_ms", "nisqa_set_option",
    "nisqa_submit_pcm", "nisqa_wait", "nisqa_drain", "nisqa_join", "nisqa_set_gather_target",
    "nisqa_wav_probe", "nisqa_wav_decode", "nisqa_wav_probe_batch", "nisqa_wav_decode_batch",
    "nisqa_resample_set_filter", "nisqa_resample_out_len", "nisqa_resample_f32",
    "nisqa_resample_device", "nisqa_predict_pcm_resampled",
]


class NisqaConfig(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("arch", C.c_int32), ("n_out", C.c_int32),
                ("n_fft", C.c_int32), ("n_mels", C.c_int32), ("seg_len", C.c_int32),
                ("seg_hop", C.c_int32), ("max_segments", C.c_int32), ("hop_s", C.c_double),
                ("win_s", C.c_double), ("fmax", C.c_double), ("sa_layers", C.c_int32),
                ("max_chunk_segments", C.c_int32), ("pool", C.c_int32), ("pos_enc", C.c_int32),
                ("double_ended", C.c_int32), ("de_align", C.c_int32), ("de_align_apply", C.c_int32),
                ("de_fuse", C.c_int32), ("td2_layers", C.c_int32), ("td2_pos_enc", C.c_int32),
                ("cnn_kind", C.c_int32), ("cnn_fc", C.c_int32), ("de_fuse_dim", C.c_int32)]


class NisqaTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("ndim", C.c_int32),
                ("dims", C.c_int64 * 4)]


class EngineError(RuntimeError):
    pass


_lib = None


def load_library(path=None):
    """dlopen the engine.  Raises if it has not been built (python -m nisqa_b200.build)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("NISQA_LIB") or LIB_PATH          # NISQA_LIB: a variant build for A/B measurements
    if not os.path.exists(p):
        raise EngineError(
            "libnisqa_b200.so is missing (%s): build it with `python -m nisqa_b200.build`; "
            "there is no CPU fallback" % p)
    lib = C.CDLL(p)
    vp, i32p, i64p, f32p = C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_float)
    lib.nisqa_create.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(NisqaConfig)]
    lib.nisqa_create.restype = C.c_int
    lib.nisqa_destroy.argtypes = [vp]
    lib.nisqa_destroy.restype = None
    lib.nisqa_last_error.argtypes = [vp]
    lib.nisqa_last_error.restype = C.c_char_p
    lib.nisqa_load_weights.argtypes = [vp, C.POINTER(NisqaTensor), C.c_int]
    lib.nisqa_load_weights.restype = C.c_int
    lib.nisqa_predict_pcm.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, f32p, i32p, i32p]
    lib.nisqa_predict_pcm.restype = C.c_int
    lib.nisqa_submit_pcm.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, f32p, i32p, i32p, i64p]
    lib.nisqa_submit_pcm.restype = C.c_int
    lib.nisqa_wav_probe.argtypes = [C.c_char_p, C.c_int32, i32p, i64p, i32p, i32p]
    lib.nisqa_wav_probe.restype = C.c_int
    lib.nisqa_wav_decode.argtypes = [C.c_char_p, C.c_int32, C.c_int32, vp, C.c_int64]
    lib.nisqa_wav_decode.restype = C.c_int64
    cpp = C.POINTER(C.c_char_p)
    lib.nisqa_wav_probe_batch.argtypes = [C.c_int, cpp, C.c_int32, C.c_int, i32p, i64p, i32p, i32p]
    lib.nisqa_wav_probe_batch.restype = C.c_int
    lib.nisqa_wav_decode_batch.argtypes = [C.c_int, cpp, C.c_int32, C.c_int32, vp, i64p, i64p, C.c_int, i32p]
    lib.nisqa_wav_decode_batch.restype = C.c_int
    lib.nisqa_resample_set_filter.argtypes = [C.POINTER(C.c_double), C.c_int64, C.c_int32]
    lib.nisqa_resample_set_filter.restype = C.c_int
    lib.nisqa_resample_out_len.argtypes = [C.c_int64, C.c_int32, C.c_int32]
    lib.nisqa_resample_out_len.restype = C.c_int64
    lib.nisqa_resample_f32.argtypes = [f32p, C.c_int64, C.c_int32, C.c_int32, f32p, C.c_int64]
    lib.nisqa_resample_f32.restype = C.c_int64
    lib.nisqa_resample_device.argtypes = [vp, vp, C.c_int64, C.c_int, C.c_int32, C.c_int32, f32p, C.c_int64]
    lib.nisqa_resample_device.restype = C.c_int
    lib.nisqa_predict_pcm_resampled.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, C.c_int32, f32p, i32p, i32p]
    lib.nisqa_predict_pcm_resampled.restype = C.c_int
    lib.nisqa_set_gather_target.argtypes = [vp, vp, C.c_int]
    lib.nisqa_set_gather_target.restype = C.c_int
    lib.nisqa_join.argtypes = [vp]
    lib.nisqa_join.restype = C.c_int
    lib.nisqa_wait.argtypes = [vp, C.c_int64]
    lib.nisqa_wait.restype = C.c_int
    lib.nisqa_drain.argtypes = [vp]
    lib.nisqa_drain.restype = C.c_int
    lib.nisqa_predict_pcm_device.argtypes = [vp, C.c_int, vp, i64p, i64p, i32p, C.c_int, vp, i32p, i32p, C.c_int]
    lib.nisqa_predict_pcm_device.restype = C.c_int
    lib.nisqa_stage_dump.argtypes = [vp, C.c_int, f32p, C.c_int64]
    lib.nisqa_stage_dump.restype = C.c_int64
    lib.nisqa_segment_counts.argtypes = [C.POINTER(NisqaConfig), C.c_int64, C.c_int32, i32p, i32p, i32p]
    lib.nisqa_segment_counts.restype = C.c_int
    lib.nisqa_mel_filterbank.argtypes = [vp, C.c_int32, f32p, C.c_int64]
    lib.nisqa_mel_filterbank.restype = C.c_int
    lib.nisqa_gather_nccl.argtypes = [vp, vp, vp, C.c_int, vp]
    lib.nisqa_gather_nccl.restype = C.c_int
    lib.nisqa_nccl_unique_id.argtypes = [vp, vp]
    lib.nisqa_nccl_unique_id.restype = C.c_int
    lib.nisqa_nccl_init.argtypes = [vp, C.c_int, C.c_int, vp]
    lib.nisqa_nccl_init.restype = C.c_int
    lib.nisqa_kernel_launches.argtypes = [vp]
    lib.nisqa_kernel_launches.restype = C.c_int64
    lib.nisqa_stream.argtypes = [vp]
    lib.nisqa_stream.restype = vp
    lib.nisqa_set_profiling.argtypes = [vp, C.c_int]
    lib.nisqa_set_profiling.restype = C.c_int
    lib.nisqa_set_option.argtypes = [vp, C.c_char_p, C.c_int]
    lib.nisqa_set_option.restype = C.c_int
    lib.nisqa_group_ms.argtypes = [vp, C.c_char_p]
    lib.nisqa_group_ms.restype = C.c_double
    if path is None:
        _lib = lib
    return lib


def config_from_args(args, max_chunk_segments=0):
    """Checkpoint ``args`` (reference model:941-942) -> nisqa_config.  Refuses anything the
    kernels do not implement (no fallback)."""
    cnn, td, pool = args.get("cnn_model"), args.get("td"), args.get("pool")
    if args.get("model") not in ("NISQA", "NISQA_DIM", "NISQA_DE"):
        raise NotImplementedError("Model not available in the engine: %r" % args.get("model"))
    de = args.get("model") == "NISQA_DE"
    pool_mode = {"avg": POOL_AVG, "max": POOL_MAX, "last_step": POOL_LAST_STEP, "last_step_bi": POOL_LAST_STEP_BI}.get(pool)
    if pool == "att":
        if args.get("pool_att_h") == 128:
            pool_mode = POOL_ATT_FF
        elif args.get("pool_att_h") in (None, 0):
            pool_mode = POOL_ATT
        else:
            raise NotImplementedError("pool_att_h=%r is not implemented by the engine (128 or None)" % args.get("pool_att_h"))
    if pool_mode is None:
        raise NotImplementedError("Pool option not available in the engine: %r" % pool)
    cnn_kind, cnn_fc = CNN_CONV, 0
    if (cnn, td) == ("adapt", "self_att") and pool_mode != POOL_LAST_STEP_BI:
        arch = ARCH_ADAPT_SA_ATTFF
        ok = (list(args["cnn_pool_1"]) == [24, 7] and list(args["cnn_pool_2"]) == [12, 5]
              and list(args["cnn_pool_3"]) == [6, 3]
              and args["td_sa_d_model"] == 64 and args["td_sa_nhead"] == 1 and args["td_sa_h"] == 64)
        cnn_fc = int(args.get("cnn_fc_out_h") or 0)           # optional Linear behind conv6 (lib:682-684)
        if cnn_fc % 64 != 0:
            raise NotImplementedError("cnn_fc_out_h=%d: the engine needs a multiple of 64" % cnn_fc)
    elif cnn in (None, "skip", "dff") and td == "self_att" and pool_mode != POOL_LAST_STEP_BI:
        # framewise models without convolutions (lib:504-583) in front of the self-attention stack
        arch = ARCH_ADAPT_SA_ATTFF
        cnn_kind = CNN_DFF if cnn == "dff" else CNN_SKIP
        cnn_fc = int(args.get("cnn_fc_out_h") or 0)
        if cnn_kind == CNN_DFF and cnn_fc == 0:
            cnn_fc = 4096                                   # DFF's default hidden width (lib:544)
        if cnn_fc % 64 != 0:
            raise NotImplementedError("cnn_fc_out_h=%d: the engine needs a multiple of 64" % cnn_fc)
        ok = args["td_sa_d_model"] == 64 and args["td_sa_nhead"] == 1 and args["td_sa_h"] == 64
    elif (cnn, td) == ("standard", "lstm") and pool_mode in (POOL_LAST_STEP_BI, POOL_AVG, POOL_MAX, POOL_LAST_STEP):
        arch = ARCH_STD_LSTM_LASTBI
        ok = (args.get("cnn_fc_out_h") == 20 and args["td_lstm_h"] == 128
              and args["td_lstm_num_layers"] == 1 and bool(args["td_lstm_bidirectional"])
              and args["model"] == "NISQA")
    else:
        raise NotImplementedError(
            "architecture cnn=%r td=%r pool=%r is not implemented by the engine" % (cnn, td, pool))
    ks = args.get("cnn_kernel_size")
    ok = ok and (ks == 3 or tuple(ks) == (3, 3))
    if de:
        # double-ended model (reference lib:272-424, config/train_nisqa_double_ended.yaml): AdaptCNN + self-attention on
        # both signals, alignment without learned weights, fusion without the optional Linear, td_2 = self-attention
        if arch != ARCH_ADAPT_SA_ATTFF:
            raise NotImplementedError("NISQA_DE is implemented for cnn_model='adapt', td='self_att'")
        if args.get("de_align") not in DE_ALIGN:
            raise NotImplementedError("de_align=%r is not implemented by the engine (dot, cosine, distance, luong, bahd)" % (args.get("de_align"),))
        if args.get("de_align_apply") not in DE_APPLY or args.get("de_fuse") not in DE_FUSE:
            raise NotImplementedError("de_align_apply / de_fuse option not available: %r / %r" % (args.get("de_align_apply"), args.get("de_fuse")))
        if args.get("de_fuse_dim") and int(args["de_fuse_dim"]) % 64 != 0:
            raise NotImplementedError("de_fuse_dim=%r: the engine needs a multiple of 64" % (args.get("de_fuse_dim"),))
        ok = ok and args.get("td_2") == "self_att" and args.get("td_2_sa_d_model") == 64 and args.get("td_2_sa_nhead") == 1 \
            and args.get("td_2_sa_h") == 64
    elif args.get("td_2") == "self_att":
        # a second self-attention stack behind the first one (lib:114-141, 236-268)
        ok = ok and arch == ARCH_ADAPT_SA_ATTFF and args.get("td_2_sa_d_model") == 64 and args.get("td_2_sa_nhead") == 1 \
            and args.get("td_2_sa_h") == 64
    else:
        ok = ok and args.get("td_2") in (None, "skip")
    ok = ok and (cnn_kind != CNN_CONV or (args["cnn_c_out_1"], args["cnn_c_out_2"], args["cnn_c_out_3"]) == (16, 32, 64))
    ok = ok and args["ms_n_fft"] == 4096 and args["ms_n_mels"] == 48 and args["ms_seg_length"] == 15
    if not ok:
        raise NotImplementedError("checkpoint hyper-parameters outside the shipped NISQA configurations")
    # ms_sr != None: the ingest converts every clip to that rate (nisqa_b200/resample.py) before the engine sees it
    cfg = NisqaConfig()
    cfg.abi_version = ABI_VERSION
    cfg.arch = arch
    cfg.n_out = 5 if args["model"] == "NISQA_DIM" else 1
    cfg.n_fft, cfg.n_mels, cfg.seg_len = 4096, 48, 15
    cfg.seg_hop = int(args["ms_seg_hop_length"])
    cfg.max_segments = int(args["ms_max_segments"]) if args.get("ms_max_segments") else 0
    cfg.hop_s, cfg.win_s = float(args["ms_hop_length"]), float(args["ms_win_length"])
    cfg.fmax = float(args["ms_fmax"])
    cfg.sa_layers = int(args["td_sa_num_layers"]) if arch == ARCH_ADAPT_SA_ATTFF else 0
    # NISQA_MAX_CHUNK: experiment knob (segments per internal pass) for A/B runs of the pass size
    cfg.max_chunk_segments = int(max_chunk_segments) or int(os.environ.get("NISQA_MAX_CHUNK", "0"))
    cfg.pool = pool_mode
    cfg.pos_enc = 1 if (arch == ARCH_ADAPT_SA_ATTFF and args.get("td_sa_pos_enc")) else 0
    cfg.cnn_kind, cfg.cnn_fc = cnn_kind, cnn_fc
    if args.get("td_2") == "self_att":
        cfg.td2_layers = int(args["td_2_sa_num_layers"])
        cfg.td2_pos_enc = 1 if args.get("td_2_sa_pos_enc") else 0
    if de:
        cfg.double_ended = 1
        cfg.de_fuse_dim = int(args.get("de_fuse_dim") or 0)
        cfg.de_align, cfg.de_align_apply, cfg.de_fuse = DE_ALIGN[args["de_align"]], DE_APPLY[args["de_align_apply"]], DE_FUSE[args["de_fuse"]]
    return cfg


def segment_counts(cfg, n_samples, sample_rate):
    """(n_frames, n_segments, status) - pure host arithmetic inside the library."""
    lib = load_library()
    a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
    rc = lib.nisqa_segment_counts(C.byref(cfg), int(n_samples), int(sample_rate), C.byref(a), C.byref(b), C.byref(c))
    if rc != 0:
        raise EngineError("nisqa_segment_counts failed (%d)" % rc)
    return a.value, b.value, c.value


class Engine(object):
    """One engine per GPU (rank)."""

    def __init__(self, cfg, device=0):
        self.lib = load_library()
        self.cfg = cfg
        self.n_out = cfg.n_out
        self.h = C.c_void_p()
        rc = self.lib.nisqa_create(C.byref(self.h), int(device), C.byref(cfg))
        if rc != 0:
            msg = self._err()
            if self.h:
                self.lib.nisqa_destroy(self.h)
                self.h = C.c_void_p()
            raise EngineError("nisqa_create failed (%d): %s" % (rc, msg))
        self.device = int(device)

    def _err(self):
        m = self.lib.nisqa_last_error(self.h)
        return m.decode() if m else ""

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError("%s failed (%d): %s" % (what, rc, self._err()))

    def drain(self):
        """Abandon the submissions in flight (their buffers may be freed afterwards)."""
        if getattr(self, "h", None):
            self.lib.nisqa_drain(self.h)

    def close(self):
        if getattr(self, "h", None):
            self.lib.nisqa_drain(self.h)
            self.lib.nisqa_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, state_dict):
        """state_dict: name -> torch.Tensor | ndarray, straight from the checkpoint."""
        keep, arr = [], (NisqaTensor * len(state_dict))()
        n = 0
        for name, t in state_dict.items():
            a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            if a.dtype != np.float32 or a.ndim > 4:
                continue                          # num_batches_tracked (int64) is not consumed
            a = np.ascontiguousarray(a)
            nm = name.encode()
            keep.append((a, nm))
            arr[n].name = nm
            arr[n].data = a.ctypes.data_as(C.POINTER(C.c_float))
            arr[n].ndim = a.ndim
            for d in range(a.ndim):
                arr[n].dims[d] = a.shape[d]
            n += 1
        self._check(self.lib.nisqa_load_weights(self.h, arr, n), "nisqa_load_weights")

    # ------------------------------------------------------------------ predict
    def predict_pcm(self, clips, sample_rates):
        """clips: list of 1-D contiguous int16 (all) or float32 (all) host arrays.
        Returns (scores [n, n_out] float32, n_segments int32[n], status int32[n])."""
        n = len(clips)
        if n == 0:
            return (np.zeros((0, self.n_out), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32))
        dt = clips[0].dtype
        if any(c.dtype != dt for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
            dt = np.dtype(np.float32)
        if dt == np.int16:
            fmt = FMT_S16
        elif dt == np.float32:
            fmt = FMT_F32
        else:
            raise ValueError("clips must be int16 or float32")
        clips = [np.ascontiguousarray(c) for c in clips]
        ptrs = (C.c_void_p * n)(*[c.ctypes.data for c in clips])
        ns = np.array([c.shape[0] for c in clips], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)),
            sr.ctypes.data_as(C.POINTER(C.c_int32)), fmt,
            scores.ctypes.data_as(C.POINTER(C.c_float)), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)))
        self._check(rc, "nisqa_predict_pcm")
        return scores, nseg, status

    def resample_device(self, x, sr_orig, sr_new):
        """One int16 / float32 clip converted on the device (csrc/resample_gpu.cu) -> float32 at sr_new."""
        from . import resample as _rs
        n_out = _rs.out_len(x.shape[0], sr_orig, sr_new)              # (also sets the interpolation table once)
        x = np.ascontiguousarray(x)
        fmt = FMT_S16 if x.dtype == np.int16 else FMT_F32
        if fmt == FMT_F32 and x.dtype != np.float32:
            raise ValueError("clips must be int16 or float32")
        y = np.empty(max(n_out, 1), dtype=np.float32)
        got = self.lib.nisqa_resample_device(self.h, x.ctypes.data, x.shape[0], fmt, int(sr_orig), int(sr_new),
                                             y.ctypes.data_as(C.POINTER(C.c_float)), y.shape[0])
        if got < 0:
            self._check(got, "nisqa_resample_device")
        return y[:got]

    def predict_pcm_resampled(self, clips, sample_rates, target_sr):
        """predict_pcm for checkpoints with ``ms_sr``: clips at their own rates are converted to ``target_sr`` on the
        device and scored there.  Synchronous.  Returns (scores, n_segments, status)."""
        from . import resample as _rs
        _rs.out_len(1, 1, 1)                                          # the interpolation table is set once
        n = len(clips)
        if n == 0:
            return (np.zeros((0, self.n_out), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32))
        dt = clips[0].dtype
        if any(c.dtype != dt for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
            dt = np.dtype(np.float32)
        if dt not in (np.dtype(np.int16), np.dtype(np.float32)):
            raise ValueError("clips must be int16 or float32")
        clips = [np.ascontiguousarray(c) for c in clips]
        ptrs = (C.c_void_p * n)(*[c.ctypes.data for c in clips])
        ns = np.array([c.shape[0] for c in clips], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm_resampled(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)), sr.ctypes.data_as(C.POINTER(C.c_int32)),
            FMT_S16 if dt == np.int16 else FMT_F32, int(target_sr), scores.ctypes.data_as(C.POINTER(C.c_float)),
            nseg.ctypes.data_as(C.POINTER(C.c_int32)), status.ctypes.data_as(C.POINTER(C.c_int32)))
        self._check(rc, "nisqa_predict_pcm_resampled")
        return scores, nseg, status

    def submit_pcm(self, clips, sample_rates):
        """Asynchronous predict_pcm: returns a handle; ``wait(handle)`` -> (scores, n_segments, status).
        Up to six submissions are in flight (H2D of the next batch overlaps this batch's kernels)."""
        n = len(clips)
        dt = clips[0].dtype if n else np.dtype(np.int16)
        if any(c.dtype != dt for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
            dt = np.dtype(np.float32)
        if dt not in (np.dtype(np.int16), np.dtype(np.float32)):
            raise ValueError("clips must be int16 or float32")
        fmt = FMT_S16 if dt == np.int16 else FMT_F32
        clips = [np.ascontiguousarray(c) for c in clips]
        ptrs = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in clips])
        ns = np.array([c.shape[0] for c in clips], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        ticket = C.c_int64(0)
        rc = self.lib.nisqa_submit_pcm(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)), sr.ctypes.data_as(C.POINTER(C.c_int32)),
            fmt, scores.ctypes.data_as(C.POINTER(C.c_float)), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(ticket))
        self._check(rc, "nisqa_submit_pcm")
        return (ticket.value, scores, nseg, status, clips, ptrs, ns, sr)      # keeps the buffers alive

    def wait(self, handle):
        if handle[0] is not None:             # (None: a synchronous call's results wrapped as a handle)
            self._check(self.lib.nisqa_wait(self.h, handle[0]), "nisqa_wait")
        return handle[1], handle[2], handle[3]

    def submit_pcm_ptrs(self, ptrs, n_samples, sample_rates, fmt, scores_out, nseg, status):
        """Raw-pointer asynchronous variant (bench e2e).  Returns the ticket."""
        ticket = C.c_int64(0)
        rc = self.lib.nisqa_submit_pcm(
            self.h, len(n_samples), ptrs, n_samples.ctypes.data_as(C.POINTER(C.c_int64)),
            sample_rates.ctypes.data_as(C.POINTER(C.c_int32)), fmt,
            scores_out.ctypes.data_as(C.POINTER(C.c_float)), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(ticket))
        self._check(rc, "nisqa_submit_pcm")
        return ticket.value

    def wait_ticket(self, ticket):
        self._check(self.lib.nisqa_wait(self.h, int(ticket)), "nisqa_wait")

    def predict_pcm_ptrs(self, ptrs, n_samples, sample_rates, fmt, scores_out):
        """Raw-pointer variant (bench e2e: pinned host buffers).  ptrs: ctypes array of void*."""
        n = len(n_samples)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm(
            self.h, n, ptrs, n_samples.ctypes.data_as(C.POINTER(C.c_int64)),
            sample_rates.ctypes.data_as(C.POINTER(C.c_int32)), fmt,
            scores_out.ctypes.data_as(C.POINTER(C.c_float)),
            nseg.ctypes.data_as(C.POINTER(C.c_int32)), status.ctypes.data_as(C.POINTER(C.c_int32)))
        self._check(rc, "nisqa_predict_pcm")
        return nseg, status

    def predict_pcm_device(self, pcm_dev_ptr, offsets, n_samples, sample_rates, fmt, scores_dev_ptr, sync=True):
        """Packed PCM already in device memory (bench 'inputs resident in HBM' figure)."""
        n = len(n_samples)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n_samples = np.ascontiguousarray(n_samples, dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm_device(
            self.h, n, C.c_void_p(pcm_dev_ptr), offsets.ctypes.data_as(C.POINTER(C.c_int64)),
            n_samples.ctypes.data_as(C.POINTER(C.c_int64)), sr.ctypes.data_as(C.POINTER(C.c_int32)),
            fmt, C.c_void_p(scores_dev_ptr), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)), 1 if sync else 0)
        self._check(rc, "nisqa_predict_pcm_device")
        return nseg, status

    # ------------------------------------------------------------------ introspection
    def stage_dump(self, stage):
        n = self.lib.nisqa_stage_dump(self.h, int(stage), None, 0)
        if n < 0:
            raise EngineError("nisqa_stage_dump failed (%d): %s" % (n, self._err()))
        out = np.empty(int(n), dtype=np.float32)
        if n:
            m = self.lib.nisqa_stage_dump(self.h, int(stage), out.ctypes.data_as(C.POINTER(C.c_float)), n)
            if m < 0:
                raise EngineError("nisqa_stage_dump failed (%d): %s" % (m, self._err()))
        return out

    def mel_filterbank(self, sample_rate):
        out = np.empty((self.cfg.n_mels, self.cfg.n_fft // 2 + 1), dtype=np.float32)
        self._check(self.lib.nisqa_mel_filterbank(self.h, int(sample_rate),
                                                  out.ctypes.data_as(C.POINTER(C.c_float)), out.size),
                    "nisqa_mel_filterbank")
        return out

    def kernel_launches(self):
        return int(self.lib.nisqa_kernel_launches(self.h))

    def stream(self):
        return self.lib.nisqa_stream(self.h)

    def join(self):
        self._check(self.lib.nisqa_join(self.h), "nisqa_join")

    def set_profiling(self, on):
        self._check(self.lib.nisqa_set_profiling(self.h, 1 if on else 0), "nisqa_set_profiling")

    def set_option(self, name, value):
        self._check(self.lib.nisqa_set_option(self.h, name.encode(), int(value)), "nisqa_set_option")

    def group_ms(self, group):
        return float(self.lib.nisqa_group_ms(self.h, group.encode()))

    # ------------------------------------------------------------------ multi-GPU exchange
    def nccl_unique_id(self):
        buf = (C.c_char * 128)()
        self._check(self.lib.nisqa_nccl_unique_id(self.h, buf), "nisqa_nccl_unique_id")
        return bytes(buf)

    def nccl_init(self, world, rank, uid):
        buf = (C.c_char * 128).from_buffer_copy(uid)
        self._check(self.lib.nisqa_nccl_init(self.h, int(world), int(rank), buf), "nisqa_nccl_init")

    def set_gather_target(self, global_dev_ptr, rows):
        self._check(self.lib.nisqa_set_gather_target(self.h, C.c_void_p(global_dev_ptr), int(rows)), "nisqa_set_gather_target")

    def gather_nccl(self, local_dev_ptr, max_rows, global_dev_ptr, comm=None):
        self._check(self.lib.nisqa_gather_nccl(self.h, C.c_void_p(comm), C.c_void_p(local_dev_ptr),
                                               int(max_rows), C.c_void_p(global_dev_ptr)),
                    "nisqa_gather_nccl")
