"""Float64 reference of the front end (PCM -> mel dB, csrc/frontend.cu) with a per-element bound, and a float32 NumPy
restatement of the pipelined kernel's dataflow that calibrates the bound.

mel_ref restates librosa 0.8.1's melspectrogram(power=1) in float64, independently of the kernel's index arithmetic:
np.pad(reflect, n_fft / 2), frames of n_fft at `hop`, the float64 periodic Hann of `win` pad_center'ed, rfft, |X|, and
the band sums with the engine's own float32 filterbank promoted to float64.  It returns the band magnitudes M[b, t], the
L1 mass of each windowed frame L[t] = sum_n |h[n] x_t[n]| and the L1 norm of each filterbank row ||W_b||_1.

Tier 1 (a bound that always holds).  The kernel transforms two real frames packed as one complex sequence z = a + i b
(frames 2p and 2p + 1 of a clip; an odd clip's last frame is packed with itself), so every spectrum value it forms is
a sum of terms whose moduli add up to at most Lp[t] = L[t] + L[partner].  The transform is a window x twiddle product,
twelve radix-2 butterfly levels with three twiddle multiplications (two 32-point passes around the W_1024 table), and
the pair unpack: about 13 rounding stages plus the roundings of the window and twiddle tables, each adding at most ~3u
(u = 2^-24) of the terms' mass.  So |X_got[k] - X[k]| <= 45 u Lp[t] in the worst case; the band sum with non-negative
weights carries it as 45 u Lp[t] ||W_b||_1.  sqrt.approx (2 ulp), the per-lane FMA chain, the warp reduction and the
squaring are relative to the band itself.  With TAU = 2^-17 = 128 u:

    |M_got[b, t] - M[b, t]| <= dM[b, t] = TAU Lp[t] ||W_b||_1 + TAU M[b, t]

[M - dM, M + dM] maps to a dB interval through 10 log10(max(m^2, 1e-8)) at both ends (monotone), widened by a few ulp
of the dB value for log10f.  The top_db clamp is then applied on intervals: the clip maximum lies in [max lo, max hi],
so every dumped value lies in [max(lo, max_lo - 80), max(hi, max_hi - 80)], widened by the rounding of the threshold.
That covers the -80 dB floor, empty bands above Nyquist and clamped bands without special cases.  The tier-1 ratio of
an element is its distance from the clamped float64 value over the distance to the interval's edge on its side
(<= 1: inside).

Tier 2 (precision).  Tier 1 is a worst case and loose for loud bands: it does not separate fp32 from fp16 tables.  The
RMS of dB_got - dB_ref over the entries within NEAR_DB of their frame's loudest band (clear of the clamp, and whose
band is not below the transform's absolute rounding floor: Lp ||W_b||_1 / M <= KAPPA_MAX = 2^10, where speech, noise,
tones and chirps stay under ~600 while window leakage alone reaches 10^5 and more) does:
TIER2_DB is 8x the RMS of the float32 restatement below (emulate_pp) on speech, noise and tones at 8, 16 and 48 kHz,
rounded up to a power of two.  fp16 tables (2^-11 per entry) or bf16 samples put it 8x or more above the limit.

emulate_pp restates frontend_pp_kernel in float32, operation by operation (FMA through float64, one rounding): the
fused window x residue-twiddle table, two in-register 32-point DIT FFTs with the W_1024 twiddle between them, the pair
unpack, |.| per bin, the CSR band sums (per lane FMA chains, then the warp's butterfly reduction), dB and the clamp.
It is CPU only, like test_plane_layout.py's layout emulation; its variants (fp16 tables, bf16 samples, frame B read
one sample late) are what the bound has to reject.
"""
import numpy as np

N_FFT = 4096
TAU = 2.0 ** -17
TIER2_DB = 2.0 ** -17
NEAR_DB = 30.0
KAPPA_MAX = 2.0 ** 10
TOP_DB = 80.0


def hop_win(sr, args):
    """lib:2308-2309 (int() truncation of sr * seconds), as the engine's plan_clip"""
    return int(sr * args["ms_hop_length"]), int(sr * args["ms_win_length"])


def samples64(y):
    """int16 PCM -> v / 32768 (libsndfile), float32 as is; float64"""
    y = np.asarray(y)
    return y.astype(np.float64) / 32768.0 if y.dtype == np.int16 else y.astype(np.float64)


def hann64(win):
    """scipy.signal.get_window('hann', win, fftbins=True) in float64"""
    if win == 1:
        return np.ones(1)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win) / win)


def mel_ref(y, sr, args, fb):
    """float64 melspectrogram(power=1) of clip y with filterbank fb [n_mels, 2049] -> (M [n_mels, T], L [T],
    ||W_b||_1 [n_mels])"""
    hop, win = hop_win(sr, args)
    x = np.pad(samples64(y), N_FFT // 2, mode="reflect")
    T = 1 + (x.shape[0] - N_FFT) // hop
    lpad = (N_FFT - win) // 2
    h = hann64(win)
    W = np.asarray(fb, dtype=np.float64)
    M = np.empty((W.shape[0], T))
    L = np.empty(T)
    for t0 in range(0, T, 256):
        t1 = min(T, t0 + 256)
        idx = (np.arange(t0, t1) * hop)[:, None] + lpad + np.arange(win)[None, :]
        fr = x[idx] * h[None, :]                               # the window's support of each frame
        L[t0:t1] = np.abs(fr).sum(1)
        full = np.zeros((t1 - t0, N_FFT))
        full[:, lpad:lpad + win] = fr
        M[:, t0:t1] = W @ np.abs(np.fft.rfft(full, axis=1)).T
    return M, L, np.abs(W).sum(1)


def db64(m):
    return 10.0 * np.log10(np.maximum(np.square(np.maximum(m, 0.0)), 1e-8))


def _ulp32(v):
    return np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


def ref_db(M):
    """the float64 dB rows with the top_db clamp"""
    d = db64(M)
    return np.maximum(d, d.max() - TOP_DB)


def pair_mass(L):
    """Lp[t] = L[t] + L[partner of t]: frames 2p and 2p + 1 share a transform, a lone last frame pairs with itself"""
    T = L.shape[0]
    partner = np.arange(T) ^ 1
    partner[partner >= T] = T - 1
    return L + L[partner]


def interval(M, L, Wn):
    """per-element [lo, hi] of the clamped dB value the kernel may produce (tier 1)"""
    dM = TAU * pair_mass(L)[None, :] * Wn[:, None] + TAU * M
    lo, hi = db64(M - dM), db64(M + dM)
    lo = lo - 4 * _ulp32(np.maximum(np.abs(lo), 1.0))
    hi = hi + 4 * _ulp32(np.maximum(np.abs(hi), 1.0))
    thr_lo, thr_hi = lo.max() - TOP_DB, hi.max() - TOP_DB
    pad = 2 * _ulp32(np.array(max(abs(thr_lo), abs(thr_hi), TOP_DB)))
    return np.maximum(lo, thr_lo - pad), np.maximum(hi, thr_hi + pad)


def tier1_ratio(got, M, L, Wn):
    """max over the clip of |got - ref| / (distance from ref to the interval's edge on that side); <= 1 holds"""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == M.shape, (got.shape, M.shape)
    assert np.isfinite(got).all()
    lo, hi = interval(M, L, Wn)
    ref = np.clip(ref_db(M), lo, hi)
    up = (got - ref) / np.maximum(hi - ref, 1e-300)
    dn = (ref - got) / np.maximum(ref - lo, 1e-300)
    return float(np.maximum(up, dn).max())


def tier2_diffs(got, M, L, Wn):
    """got - dB_ref over the entries within NEAR_DB of their frame's loudest band, clear of the -80 dB floor and the
    clamp, and above the transform's absolute rounding floor (Lp ||W_b||_1 <= KAPPA_MAX M: not a band that only
    holds the window's leakage, such as a 24 kHz tone seen by bands below 20 kHz); tier 2 takes the RMS over a group"""
    d = db64(M)
    keep = (d >= d.max(0, keepdims=True) - NEAR_DB) & (d > d.max() - TOP_DB + 1.0) & (d > -TOP_DB + 1.0)
    keep &= pair_mass(L)[None, :] * Wn[:, None] <= KAPPA_MAX * M
    return (np.asarray(got, dtype=np.float64) - d)[keep]


def rms(v):
    v = np.concatenate([np.ravel(x) for x in v]) if isinstance(v, (list, tuple)) else np.ravel(v)
    return float(np.sqrt(np.mean(np.square(v)))) if v.size else 0.0


# ------------------------------------------------------------------ float32 restatement of frontend_pp_kernel
f32 = np.float32


def _fma(a, b, c):
    """fmaf: the exact product (two float32 fit in a float64) plus c, rounded once"""
    return (a.astype(np.float64) * np.asarray(b, dtype=np.float64) + c.astype(np.float64)).astype(f32)


def _rev5(i):
    return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4)


REV5 = np.array([_rev5(i) for i in range(32)])
_W32 = [(f32(np.cos(2 * np.pi * k / 32)), f32(-np.sin(2 * np.pi * k / 32))) for k in range(16)]


def _fft32(xr, xi):
    """fft32 of frontend.cu on [32, ...] float32 arrays (position axis first, input in bit-reversed order); in place"""
    for half in (1, 2, 4, 8, 16):
        for base in range(0, 32, 2 * half):
            for j in range(half):
                k = j * (16 // half)
                a, b = base + j, base + j + half
                ar, ai, br, bi = xr[a].copy(), xi[a].copy(), xr[b].copy(), xi[b].copy()
                if k == 0:
                    xr[a], xi[a], xr[b], xi[b] = ar + br, ai + bi, ar - br, ai - bi
                elif k == 8:
                    xr[a], xi[a], xr[b], xi[b] = ar + bi, ai - br, ar - bi, ai + br
                else:
                    wx, wy = _W32[k]
                    ox = _fma(br, wx, _fma(bi, -wy, ar))
                    oy = _fma(bi, wx, _fma(br, wy, ai))
                    xr[a], xi[a] = ox, oy
                    xr[b], xi[b] = _fma(ar, 2.0, -ox), _fma(ai, 2.0, -oy)


def wtab_table(win):
    """engine build_fb: wtab[r][n] = float32(window[n]) * e^{-2 pi i r n / 4096} (0 for n >= win), [4, 1024] x 2"""
    n = np.arange(1024)
    wf = np.zeros(1024, f32)
    wf[:min(win, 1024)] = hann64(win)[:1024].astype(f32)
    a = -2.0 * np.pi * ((np.arange(4)[:, None] * n[None, :]) & 4095) / 4096.0
    return (wf.astype(np.float64) * np.cos(a)).astype(f32), (wf.astype(np.float64) * np.sin(a)).astype(f32)


def tw2_table():
    """engine nisqa_create: tw2[q][lane] = W_1024^(lane q), [32 q, 32 lane] x 2"""
    k = (4 * np.arange(32)[:, None] * np.arange(32)[None, :]) & 4095
    a = -2.0 * np.pi * k / 4096.0
    return np.cos(a).astype(f32), np.sin(a).astype(f32)


def csr_bands(fb):
    """engine build_fb: each band's non-zero run of bins, zero-padded to a multiple of 32 -> (first bin [n_mels],
    weights [n_mels, iters, 32])"""
    fb = np.asarray(fb, dtype=f32)
    rows, k0s = [], []
    for w in fb:
        nz = np.nonzero(w)[0]
        k0 = int(nz[0]) if nz.size else 0
        r = w[k0:int(nz[-1]) + 1] if nz.size else np.zeros(0, f32)
        rows.append(np.concatenate([r, np.zeros(-len(r) % 32, f32)]))
        k0s.append(k0)
    it = max(1, max(len(r) // 32 for r in rows))
    wts = np.zeros((fb.shape[0], it, 32), f32)
    for b, r in enumerate(rows):
        wts[b, :len(r) // 32] = r.reshape(-1, 32)
    return np.array(k0s), wts


def _bf16(v):
    b = np.ascontiguousarray(v, dtype=f32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(f32)


def emulate_pp(y, sr, args, fb, fp16_tables=False, bf16_samples=False, late_b=False):
    """frontend_pp_kernel's mel dB rows of clip y (int16: raw integers and the 2^-30 power scale; float32 as is) with
    the top_db clamp, [n_mels, T] float32.  Variants: fp16_tables (wtab and tw2 rounded to fp16), bf16_samples (every
    sample rounded to bf16), late_b (frame B of each pair read one sample late)."""
    hop, win = hop_win(sr, args)
    assert win <= 1024 and hop + win <= 1536, "the pipelined kernel's geometry"
    y = np.asarray(y)
    pscale = f32(2.0 ** -30) if y.dtype == np.int16 else f32(1.0)
    ys = y.astype(f32)
    if bf16_samples:
        ys = _bf16(ys)
    n = y.shape[0]
    T = 1 + n // hop
    P = (T + 1) // 2
    s0 = (N_FFT - win) // 2 - N_FFT // 2
    wr, wi = wtab_table(win)
    tr, ti = tw2_table()
    if fp16_tables:
        wr, wi, tr, ti = (t.astype(np.float16).astype(f32) for t in (wr, wi, tr, ti))

    def sample(i):                                             # y over numpy's reflect padding (any depth)
        period = 2 * n - 2 if n > 1 else 1
        m = np.mod(i, period)
        return ys[np.where(m < n, m, period - m)] if n > 1 else ys[np.zeros_like(i)]

    a = s0 + 2 * np.arange(P) * hop
    validB = 2 * np.arange(P) + 1 < T
    nn = np.arange(1024)
    sa = sample(a[:, None] + nn[None, :])                      # [P, 1024]
    sb = sample(a[:, None] + np.where(validB, hop + (1 if late_b else 0), 0)[:, None] + nn[None, :])
    # input stage: x = (sa, sb) * wtab[r][n]: fmaf(sa, wt.x, -(sb wt.y)), fmaf(sa, wt.y, sb wt.x) -> [P, 4, 1024]
    sa, sb = sa[:, None, :], sb[:, None, :]
    xr = _fma(sa, wr[None], -(sb * wi[None]))
    xi = _fma(sa, wi[None], (sb * wr[None]).astype(f32))
    # n = lane + 32 j -> [j, P, 4, lane], positions in bit-reversed order
    xr = np.moveaxis(xr.reshape(P, 4, 32, 32), 2, 0)[REV5].copy()
    xi = np.moveaxis(xi.reshape(P, 4, 32, 32), 2, 0)[REV5].copy()
    _fft32(xr, xi)                                             # A_lane[q] at position q
    vr = _fma(xr, tr[:, None, None, :], -(xi * ti[:, None, None, :]).astype(f32))
    vi = _fma(xr, ti[:, None, None, :], (xi * tr[:, None, None, :]).astype(f32))
    vr[0], vi[0] = xr[0], xi[0]
    # transpose: new lane = q, position rev5(old lane)
    xr = np.moveaxis(vr, (0, 3), (3, 0))[REV5].copy()
    xi = np.moveaxis(vi, (0, 3), (3, 0))[REV5].copy()
    _fft32(xr, xi)                                             # Z_r[q + 32 p] at position p, lane q
    Zr = np.moveaxis(xr, 0, 2).reshape(P, 4, 1024)             # [P, r, m]
    Zi = np.moveaxis(xi, 0, 2).reshape(P, 4, 1024)
    Zr = np.swapaxes(Zr, 1, 2).reshape(P, N_FFT)               # bin k = 4 m + r
    Zi = np.swapaxes(Zi, 1, 2).reshape(P, N_FFT)
    kk = (N_FFT - np.arange(N_FFT)) & (N_FFT - 1)
    ar, ai = Zr + Zr[:, kk], Zi - Zi[:, kk]
    br, bi = Zi + Zi[:, kk], Zr - Zr[:, kk]
    ma = np.sqrt(_fma(ar, ar, (ai * ai).astype(f32)))
    mb = np.sqrt(_fma(br, br, (bi * bi).astype(f32)))
    mags = np.stack([ma, mb], 1)                               # [P, 2 frames, 4096]
    k0, wts = csr_bands(fb)
    bins = np.minimum(k0[:, None, None] + 32 * np.arange(wts.shape[1])[None, :, None] + np.arange(32)[None, None, :],
                      N_FFT - 1)
    acc = np.zeros((P, 2, wts.shape[0], 32), f32)
    for it in range(wts.shape[1]):
        acc = _fma(mags[:, :, bins[:, it, :]], wts[None, None, :, it, :], acc)
    for d in (16, 8, 4, 2, 1):                                 # the warp's butterfly reduction
        acc = acc[..., :d] + acc[..., d:2 * d]
    sv = f32(0.5) * acc[..., 0]                                # [P, 2, n_mels]
    p = (sv * sv) * pscale
    dbv = (f32(10.0) * np.log10(np.maximum(p, f32(1e-8)).astype(np.float64)).astype(f32)).astype(f32)
    rows = dbv.reshape(2 * P, -1)[:T]                          # frame 2p + f
    thr = f32(rows.max() - f32(TOP_DB))
    return np.maximum(rows, thr).T.copy()
