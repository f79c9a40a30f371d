"""Float64 reference of the double-ended model's alignment and fusion (NISQA_DE, reference lib:1228-1417), with the
first-order bound of tests/stage_ref.py (whose helpers it reuses).  Inputs are td's output rows of one pair as the
engine dumped them (NISQA_STAGE_TD1_OUT), so they carry no error.

Scores (Alignment, lib:1274-1357) and their bounds:
    dot       x . y                                        TAU sum |x| |y|
    cosine    x . y / (max(|x|, 1e-8) max(|y|, 1e-8))      the dot bound scaled by the norms + 2 TAU |s| (the two norms)
    distance  -mean |x - y|                                TAU sum (|x| + |y|) / 64
    luong     x . (W y + b)                                the key projection's bound, root-sum-square through x
    bahd      v . tanh(Wq x + bq + Wy y + by)              the projections' bounds through tanh' <= 1, + TAU sum |v| |t|
              (v.bias shifts every score of a row alike: softmax and argmax drop it, and so does the engine)
Soft application: softmax_rows, then matmul(p, ep, y, 0).  Hard application picks ONE reference row: any j of
    C_i = { j : s[i, j] + b[i, j] >= max_k (s[i, k] - b[i, k]) }
is a pick a correct fp32 evaluation may make, and no other j is, so the engine's row must be the fp32 fusion of x_i
with y_j, bit for bit, for some j in C_i.  Fusion copies x exactly; x +- y_al is `add` with its bound.
"""
import torch

import stage_ref as R
from stage_ref import TAU, _d

EPS_COS = 1e-8
BAHD_ROWS = 32              # query rows per block of the [rows, Sy, 128] Bahdanau tensor


def n_fused(args):
    return 3 if args["de_fuse"] == "x/y/-" else 2


def scores(args, sd, x, y):
    """attention scores [Sx, Sy] of degraded rows x [Sx, 64] against reference rows y [Sy, 64] (float64) -> (s, bound)"""
    m = args["de_align"]
    zx, zy = torch.zeros_like(x), torch.zeros_like(y)
    if m in ("dot", "cosine"):
        s, b = R.matmul(x, zx, y.t(), zy.t())
        if m == "cosine":
            n = x.norm(dim=1).clamp_min(EPS_COS)[:, None] * y.norm(dim=1).clamp_min(EPS_COS)[None, :]
            s = s / n
            b = b / n + 2 * TAU * s.abs()
        return s, b
    if m == "distance":
        s = -torch.cdist(x, y, p=1) / x.shape[1]
        return s, TAU * (x.abs().sum(1)[:, None] + y.abs().sum(1)[None, :]) / x.shape[1]
    if m == "luong":
        yp, eyp = R.linear(y, zy, sd["align.att.W.weight"], sd["align.att.W.bias"])
        return R.matmul(x, zx, yp.t(), eyp.t())
    if m == "bahd":
        xq, exq = R.linear(x, zx, sd["align.att.Wq.weight"], sd["align.att.Wq.bias"])
        yk, eyk = R.linear(y, zy, sd["align.att.Wy.weight"], sd["align.att.Wy.bias"])
        v = _d(sd["align.att.v.weight"]).reshape(-1)
        av = v.abs()
        s = torch.empty(x.shape[0], y.shape[0], dtype=torch.float64)
        b = torch.empty_like(s)
        carried = (exq @ av)[:, None] + (eyk @ av)[None, :]
        for i0 in range(0, x.shape[0], BAHD_ROWS):
            a = xq[i0:i0 + BAHD_ROWS, None, :] + yk[None, :, :]
            t = torch.tanh(a)
            s[i0:i0 + BAHD_ROWS] = t @ v
            b[i0:i0 + BAHD_ROWS] = carried[i0:i0 + BAHD_ROWS] + TAU * ((a.abs() + t.abs()) @ av)
        return s, b
    raise NotImplementedError(m)


def candidates(s, b):
    """[Sx, Sy] bool: the reference steps a correct fp32 argmax of each row may pick"""
    return (s + b) >= (s - b).max(1, keepdim=True)[0]


def soft_align(s, b, y):
    """softmax over the reference steps, then the weighted sum of y -> (y_al, bound)"""
    p, ep = R.softmax_rows(s, b)
    return R.matmul(p, ep, y, torch.zeros_like(y))


def fuse(args, x, y_al, e_al):
    """Fusion (lib:1402-1413) of float64 rows -> ([Sx, 64 nf], bound); the x columns are exact copies"""
    z = torch.zeros_like(x)
    mode = args["de_fuse"]
    diff = R.add(x, z, -y_al, e_al)
    if mode == "x/y/-":
        parts = [(x, z), (y_al, e_al), diff]
    elif mode == "+/-":
        parts = [R.add(x, z, y_al, e_al), diff]
    elif mode == "x/y":
        parts = [(x, z), (y_al, e_al)]
    else:
        raise NotImplementedError(mode)
    return torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1)


def fuse_f32(args, x, y):
    """Fusion of float32 rows, each term rounded once as fp32 arithmetic rounds it (the hard-alignment rows)"""
    mode = args["de_fuse"]
    if mode == "x/y/-":
        return torch.cat((x, y, x - y), -1)
    if mode == "+/-":
        return torch.cat((x + y, x - y), -1)
    if mode == "x/y":
        return torch.cat((x, y), -1)
    raise NotImplementedError(mode)


def check_hard(args, x, y, got, cand):
    """Every fused row got[i] must be fuse_f32(x_i, y_j) bit for bit for some j in C_i.  -> (first failing row or None,
    fraction of rows with a single candidate)"""
    x32, y32 = x.float(), y.float()
    got = torch.as_tensor(got).float().reshape(x.shape[0], -1)
    for i in range(x.shape[0]):
        js = cand[i].nonzero().reshape(-1)
        rows = fuse_f32(args, x32[i].expand(len(js), -1), y32[js])
        if not (rows.view(torch.int32) == got[i].view(torch.int32)).all(1).any():
            return i, None
    return None, float((cand.sum(1) == 1).double().mean())


def lin_fusion(sd, fused):
    """Fusion.lin_fusion (de_fuse_dim, lib:1414-1415) of the dumped fused rows"""
    return R.linear(fused, torch.zeros_like(fused), sd["fuse.lin_fusion.weight"], sd["fuse.lin_fusion.bias"])
