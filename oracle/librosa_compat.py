"""CPU restatement of the four librosa-0.8.1 entry points the NISQA front-end calls.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is on the product path: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl
reference`` legs may import it, and only as the checker / the thing timed as the
CPU baseline.

PARITY UNPINNED (front-end half).  The arithmetic restated here lives in a
third-party dependency that is not vendored in the reference project:
``librosa==0.8.1`` (reference ``env.yml:16``; with ``numpy==1.20.3`` FFT,
``scipy=1.7.3`` ``get_window``, ``libsndfile=1.0.31``).  It cannot be installed in
this environment and the reference ships no golden vectors / tests for this
boundary, so this file restates the *published* librosa 0.8.1 algorithm and is
anchored on the reference's own call sites:

* ``lb.load``                      -> reference ``nisqa/NISQA_lib.py:2298-2306``
* ``lb.feature.melspectrogram``    -> reference ``nisqa/NISQA_lib.py:2311-2328``
* ``lb.core.amplitude_to_db``      -> reference ``nisqa/NISQA_lib.py:2330``

Independent cross-checks (``tests/test_oracle_frontend.py``): the filterbank
against ``torchaudio.functional.melscale_fbanks`` and
``transformers.audio_utils.mel_filter_bank``; the STFT against ``torch.stft`` in
float64; the window against ``scipy.signal.get_window``; the whole chain (STFT, mel, dB, clamp)
against ``transformers.audio_utils.spectrogram`` + ``amplitude_to_db`` to 1e-5 dB.

librosa 0.8.1 functions restated (module :: function):
  core/audio.py    :: load, to_mono
  core/spectrum.py :: stft, _spectrogram, amplitude_to_db, power_to_db
  feature/spectral.py :: melspectrogram
  filters.py       :: mel, get_window
  core/convert.py  :: hz_to_mel, mel_to_hz, mel_frequencies, fft_frequencies
  util/utils.py    :: pad_center, frame
"""
import struct
import sys
import types

import numpy as np

__version__ = "0.8.1-restated"


# --------------------------------------------------------------------------- load
def _g711_expand(codes, alaw):
    """ITU-T G.711 expansion of 8-bit codes to 16-bit linear samples (the tables of libsndfile's alaw.c / ulaw.c)."""
    c = codes.astype(np.int32)
    if alaw:
        c = c ^ 0x55
        t = (c & 0x0F) << 4
        seg = (c & 0x70) >> 4
        t = np.where(seg == 0, t + 8, np.where(seg == 1, t + 0x108, (t + 0x108) << np.maximum(seg - 1, 0)))
        return np.where(c & 0x80, t, -t)
    c = ~c & 0xFF
    t = (((c & 0x0F) << 3) + 0x84) << ((c & 0x70) >> 4)
    return np.where(c & 0x80, 0x84 - t, t - 0x84)


def _read_wav(path):
    """RIFF/WAVE reader with libsndfile's float conversion rules.

    PCM u8 -> (v-128)/128, PCM16 -> v/32768, PCM24 -> v/2**23, PCM32 -> v/2**31,
    IEEE float32/float64 -> as is (cast to float32), G.711 A-law / mu-law (tags 6 / 7) -> the 16-bit
    expansion / 32768 (libsndfile alaw.c / ulaw.c).  Returns (y[n, ch] float32, sr).
    """
    with open(path, "rb") as f:
        data = f.read()
    if len(data) < 12 or data[0:4] != b"RIFF" or data[8:12] != b"WAVE":
        raise ValueError("not a RIFF/WAVE file")
    pos = 12
    fmt = None
    payload = None
    while pos + 8 <= len(data):
        cid = data[pos:pos + 4]
        csz = struct.unpack("<I", data[pos + 4:pos + 8])[0]
        body = data[pos + 8:pos + 8 + csz]
        if cid == b"fmt ":
            tag, ch, sr, _br, _ba, bits = struct.unpack("<HHIIHH", body[:16])
            if tag == 0xFFFE and len(body) >= 26:  # WAVE_FORMAT_EXTENSIBLE
                tag = struct.unpack("<H", body[24:26])[0]
            fmt = (tag, ch, sr, bits)
        elif cid == b"data":
            payload = body
        pos += 8 + csz + (csz & 1)
    if fmt is None or payload is None:
        raise ValueError("missing fmt/data chunk")
    tag, ch, sr, bits = fmt
    if tag == 1:
        if bits == 8:
            y = (np.frombuffer(payload, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
        elif bits == 16:
            y = np.frombuffer(payload[:len(payload) // 2 * 2], dtype="<i2").astype(np.float32) / 32768.0
        elif bits == 24:
            raw = np.frombuffer(payload[:len(payload) // 3 * 3], dtype=np.uint8).reshape(-1, 3)
            v = (raw[:, 0].astype(np.int32) | (raw[:, 1].astype(np.int32) << 8)
                 | (raw[:, 2].astype(np.int32) << 16))
            v = np.where(v >= (1 << 23), v - (1 << 24), v)
            y = v.astype(np.float32) / np.float32(1 << 23)
        elif bits == 32:
            y = (np.frombuffer(payload[:len(payload) // 4 * 4], dtype="<i4").astype(np.float64)
                 / 2147483648.0).astype(np.float32)
        else:
            raise ValueError("unsupported PCM width %d" % bits)
    elif tag in (6, 7) and bits == 8:
        y = _g711_expand(np.frombuffer(payload, dtype=np.uint8), alaw=(tag == 6)).astype(np.float32) / 32768.0
    elif tag == 3:
        if bits == 32:
            y = np.frombuffer(payload[:len(payload) // 4 * 4], dtype="<f4").astype(np.float32)
        elif bits == 64:
            y = np.frombuffer(payload[:len(payload) // 8 * 8], dtype="<f8").astype(np.float32)
        else:
            raise ValueError("unsupported float width %d" % bits)
    else:
        raise ValueError("unsupported WAVE format tag %d" % tag)
    n = (y.shape[0] // ch) * ch
    return y[:n].reshape(-1, ch), int(sr)


def to_mono(y):
    """librosa.core.audio.to_mono: mean over the channel axis (float32 in, float32 out)."""
    if y.ndim > 1:
        y = np.mean(y, axis=0)
    return y


def load(path, sr=22050, mono=True, offset=0.0, duration=None, dtype=np.float32,
         res_type="kaiser_best"):
    """librosa.core.audio.load as used at reference lib:2300/2304 (sr=None, offset=0)."""
    y, sr_native = _read_wav(path)
    y = y.T  # soundfile gives [n, ch]; librosa transposes to [ch, n]
    if y.shape[0] == 1:
        y = y[0]
    if mono:
        y = to_mono(y)
    if sr is not None:
        y = resample(y, sr_native, sr, res_type=res_type)
    else:
        sr = sr_native
    return np.ascontiguousarray(y, dtype=dtype), sr


# ----------------------------------------------------------------------- resample
# librosa 0.8.1 core/audio.py::resample -> resampy (0.2.2) core.py::resample / interpn.py::resample_f with the
# 'kaiser_best' filter.  resampy is a further third-party dependency that is not vendored (PARITY UNPINNED, like
# the rest of this file); restated from its published algorithm.  Its data/kaiser_best.npz is the output of
# filters.sinc_window(num_zeros=64, precision=9, rolloff=0.9475937167399596) with a Kaiser window of
# beta=14.769656459379492 (the parameters stated in resampy's filters.py docstring) and is regenerated here.
_KAISER_BEST = dict(num_zeros=64, precision=9, rolloff=0.9475937167399596, beta=14.769656459379492)
_filter_cache = {}


def sinc_window(num_zeros, precision, rolloff, beta):
    """resampy.filters.sinc_window with window = scipy.signal.kaiser(., beta): right half of a windowed sinc,
    2**precision samples per zero crossing.  -> (half_window float64 [n + 1], samples per zero crossing)."""
    from scipy.signal.windows import kaiser
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = kaiser(2 * n + 1, beta)[n:]
    return taper * sinc_win, num_bits


def resampy_resample(x, sr_orig, sr_new):
    """resampy.resample(x, sr_orig, sr_new, filter='kaiser_best') for 1-D float32 x: band-limited sinc
    interpolation (J. O. Smith) with linear interpolation between filter table entries.  The reference loop runs
    per output sample t over the left wing (taps i = 0.. towards the past) and then the right wing (taps k), adding
    weight (float64) * x (float32) into the float32 output EVERY iteration; here the same additions are done in
    the same order, vectorised over t."""
    if sr_orig <= 0 or sr_new <= 0:
        raise ValueError("invalid sample rate")
    x = np.asarray(x, dtype=np.float32)
    sample_ratio = float(sr_new) / sr_orig
    n_out = int(x.shape[0] * sample_ratio)
    if n_out < 1:
        raise ValueError("Input signal length is too small to resample")
    if "kb" not in _filter_cache:
        _filter_cache["kb"] = sinc_window(**_KAISER_BEST)
    interp_win, num_table = _filter_cache["kb"]
    interp_win = interp_win.copy()
    if sample_ratio < 1:
        interp_win *= sample_ratio
    interp_delta = np.zeros_like(interp_win)
    interp_delta[:-1] = np.diff(interp_win)
    scale = min(1.0, sample_ratio)
    time_increment = 1.0 / sample_ratio
    index_step = int(scale * num_table)
    nwin, n_orig = interp_win.shape[0], x.shape[0]
    # time_register += time_increment, starting from 0.0 (sequential float64 additions)
    steps = np.full(n_out, time_increment)
    steps[0] = 0.0
    time_register = np.cumsum(steps)
    n = time_register.astype(np.int64)
    y = np.zeros(n_out, dtype=np.float32)
    for wing in (0, 1):
        frac = scale * (time_register - n)
        if wing:
            frac = scale - frac
        index_frac = frac * num_table
        offset = index_frac.astype(np.int64)
        eta = index_frac - offset
        if wing == 0:
            count = np.minimum(n + 1, (nwin - offset) // index_step)
        else:
            count = np.minimum(n_orig - n - 1, (nwin - offset) // index_step)
        for i in range(int(count.max()) if n_out else 0):
            live = np.nonzero(count > i)[0]
            idx = offset[live] + i * index_step
            weight = interp_win[idx] + eta[live] * interp_delta[idx]
            src = n[live] - i if wing == 0 else n[live] + i + 1
            y[live] = (y[live].astype(np.float64) + weight * x[src].astype(np.float64)).astype(np.float32)
    return y


def fix_length(data, size):
    """librosa.util.fix_length on the last axis: trim, or pad with zeros."""
    n = data.shape[-1]
    if n > size:
        return data[..., :size]
    if n < size:
        return np.pad(data, [(0, 0)] * (data.ndim - 1) + [(0, size - n)], mode="constant")
    return data


def resample(y, orig_sr, target_sr, res_type="kaiser_best", fix=True, scale=False):
    """librosa.core.audio.resample (0.8.1) for mono or [ch, n] float32 input."""
    if orig_sr == target_sr:
        return y
    if res_type != "kaiser_best":
        raise NotImplementedError("only res_type='kaiser_best' (librosa.load's default) is restated")
    ratio = float(target_sr) / orig_sr
    n_samples = int(np.ceil(y.shape[-1] * ratio))
    if y.ndim == 1:
        y_hat = resampy_resample(y, orig_sr, target_sr)
    else:
        y_hat = np.stack([resampy_resample(c, orig_sr, target_sr) for c in y])
    if fix:
        y_hat = fix_length(y_hat, n_samples)
    if scale:
        y_hat = y_hat / np.sqrt(ratio)
    return np.ascontiguousarray(y_hat, dtype=y.dtype)


# ------------------------------------------------------------------------ convert
def fft_frequencies(sr=22050, n_fft=2048):
    return np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)


def hz_to_mel(frequencies, htk=False):
    frequencies = np.asanyarray(frequencies)
    if htk:
        return 2595.0 * np.log10(1.0 + frequencies / 700.0)
    f_min = 0.0
    f_sp = 200.0 / 3
    mels = (frequencies - f_min) / f_sp
    min_log_hz = 1000.0
    min_log_mel = (min_log_hz - f_min) / f_sp
    logstep = np.log(6.4) / 27.0
    if frequencies.ndim:
        log_t = frequencies >= min_log_hz
        mels[log_t] = min_log_mel + np.log(frequencies[log_t] / min_log_hz) / logstep
    elif frequencies >= min_log_hz:
        mels = min_log_mel + np.log(frequencies / min_log_hz) / logstep
    return mels


def mel_to_hz(mels, htk=False):
    mels = np.asanyarray(mels)
    if htk:
        return 700.0 * (10.0 ** (mels / 2595.0) - 1.0)
    f_min = 0.0
    f_sp = 200.0 / 3
    freqs = f_min + f_sp * mels
    min_log_hz = 1000.0
    min_log_mel = (min_log_hz - f_min) / f_sp
    logstep = np.log(6.4) / 27.0
    if mels.ndim:
        log_t = mels >= min_log_mel
        freqs[log_t] = min_log_hz * np.exp(logstep * (mels[log_t] - min_log_mel))
    elif mels >= min_log_mel:
        freqs = min_log_hz * np.exp(logstep * (mels - min_log_mel))
    return freqs


def mel_frequencies(n_mels=128, fmin=0.0, fmax=11025.0, htk=False):
    min_mel = hz_to_mel(fmin, htk=htk)
    max_mel = hz_to_mel(fmax, htk=htk)
    mels = np.linspace(min_mel, max_mel, n_mels)
    return mel_to_hz(mels, htk=htk)


# ------------------------------------------------------------------------ filters
def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm="slaney",
        dtype=np.float32):
    """librosa.filters.mel (0.8.1): float32 triangular bank, Slaney area normalisation."""
    if fmax is None:
        fmax = float(sr) / 2
    n_mels = int(n_mels)
    weights = np.zeros((n_mels, int(1 + n_fft // 2)), dtype=dtype)
    fftfreqs = fft_frequencies(sr=sr, n_fft=n_fft)
    mel_f = mel_frequencies(n_mels + 2, fmin=fmin, fmax=fmax, htk=htk)
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    if norm == "slaney":
        enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
        # librosa does `weights *= enorm[:, np.newaxis]` on the float32 array: the product is
        # formed in float64 from the already-float32-rounded triangle and rounded back.
        weights[...] = (weights.astype(np.float64) * enorm[:, np.newaxis]).astype(dtype)
    return weights


def get_window(window, Nx, fftbins=True):
    """scipy.signal.get_window('hann', Nx, fftbins=True): periodic Hann, float64."""
    if window not in ("hann", "hanning"):
        raise NotImplementedError(window)
    if Nx == 1:
        return np.ones(1)
    M = Nx + 1 if fftbins else Nx
    n = np.arange(0, M)
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / (M - 1))
    return w[:Nx] if fftbins else w


def pad_center(data, size):
    n = data.shape[-1]
    lpad = int((size - n) // 2)
    if lpad < 0:
        raise ValueError("Target size ({:d}) must be at least input size ({:d})".format(size, n))
    return np.pad(data, [(lpad, int(size - n - lpad))], mode="constant")


def frame(x, frame_length, hop_length):
    n_frames = 1 + (x.shape[-1] - frame_length) // hop_length
    strides = (x.itemsize, hop_length * x.itemsize)
    return np.lib.stride_tricks.as_strided(x, shape=(frame_length, n_frames), strides=strides)


# ----------------------------------------------------------------------- spectrum
def stft(y, n_fft=2048, hop_length=None, win_length=None, window="hann", center=True,
         dtype=None, pad_mode="reflect"):
    """librosa.core.spectrum.stft (0.8.1): float64 rfft of (float64 window x float32 frame),
    stored as complex64."""
    if win_length is None:
        win_length = n_fft
    if hop_length is None:
        hop_length = int(win_length // 4)
    fft_window = get_window(window, win_length, fftbins=True)
    fft_window = pad_center(fft_window, n_fft).reshape((-1, 1))
    if center:
        y = np.pad(y, int(n_fft // 2), mode=pad_mode)
    y = np.ascontiguousarray(y)
    y_frames = frame(y, frame_length=n_fft, hop_length=hop_length)
    if dtype is None:
        dtype = np.complex64 if y.dtype == np.float32 else np.complex128
    stft_matrix = np.empty((int(1 + n_fft // 2), y_frames.shape[1]), dtype=dtype, order="F")
    max_mem_block = 2 ** 8 * 2 ** 10
    n_columns = max(max_mem_block // (stft_matrix.shape[0] * stft_matrix.itemsize), 1)
    for bl_s in range(0, stft_matrix.shape[1], n_columns):
        bl_t = min(bl_s + n_columns, stft_matrix.shape[1])
        stft_matrix[:, bl_s:bl_t] = np.fft.rfft(fft_window * y_frames[:, bl_s:bl_t], axis=0)
    return stft_matrix


def _spectrogram(y=None, S=None, n_fft=2048, hop_length=512, power=1, win_length=None,
                 window="hann", center=True, pad_mode="reflect"):
    if S is not None:
        n_fft = 2 * (S.shape[0] - 1)
    else:
        S = np.abs(stft(y, n_fft=n_fft, hop_length=hop_length, win_length=win_length,
                        center=center, window=window, pad_mode=pad_mode)) ** power
    return S, n_fft


def melspectrogram(y=None, sr=22050, S=None, n_fft=2048, hop_length=512, win_length=None,
                   window="hann", center=True, pad_mode="reflect", power=2.0, **kwargs):
    S, n_fft = _spectrogram(y=y, S=S, n_fft=n_fft, hop_length=hop_length, power=power,
                            win_length=win_length, window=window, center=center,
                            pad_mode=pad_mode)
    mel_basis = mel(sr, n_fft, **kwargs)
    return np.dot(mel_basis, S)


def power_to_db(S, ref=1.0, amin=1e-10, top_db=80.0):
    S = np.asarray(S)
    magnitude = S
    ref_value = np.abs(ref)
    log_spec = 10.0 * np.log10(np.maximum(amin, magnitude))
    log_spec -= 10.0 * np.log10(np.maximum(amin, ref_value))
    if top_db is not None:
        log_spec = np.maximum(log_spec, log_spec.max() - top_db)
    return log_spec


def amplitude_to_db(S, ref=1.0, amin=1e-5, top_db=80.0):
    S = np.asarray(S)
    magnitude = np.abs(S)
    ref_value = np.abs(ref)
    power = np.square(magnitude, out=magnitude)
    return power_to_db(power, ref=ref_value ** 2, amin=amin ** 2, top_db=top_db)


# ---------------------------------------------------------------- module install
def install():
    """Register this restatement as ``librosa`` (plus a ``matplotlib.pyplot`` stub) so that
    the reference package imports unmodified (reference lib:10, lib:13).  Used only by the
    golden-vector generator and the reference-plumbing tests in THIS container."""
    me = sys.modules[__name__]
    lb = types.ModuleType("librosa")
    lb.load = load
    lb.__version__ = __version__
    feat = types.ModuleType("librosa.feature")
    feat.melspectrogram = melspectrogram
    core = types.ModuleType("librosa.core")
    core.amplitude_to_db = amplitude_to_db
    core.load = load
    core.stft = stft
    filt = types.ModuleType("librosa.filters")
    filt.mel = mel
    lb.feature, lb.core, lb.filters = feat, core, filt
    lb.stft = stft
    lb.amplitude_to_db = amplitude_to_db
    lb._restated_by = me
    sys.modules.setdefault("librosa", lb)
    sys.modules.setdefault("librosa.feature", feat)
    sys.modules.setdefault("librosa.core", core)
    sys.modules.setdefault("librosa.filters", filt)
    if "matplotlib" not in sys.modules:
        try:
            import matplotlib.pyplot  # noqa: F401
        except Exception:
            mpl = types.ModuleType("matplotlib")
            plt = types.ModuleType("matplotlib.pyplot")
            mpl.pyplot = plt
            sys.modules["matplotlib"] = mpl
            sys.modules["matplotlib.pyplot"] = plt
    return lb
