"""Float64 restatement of NISQA_DE's alignment (reference lib:1228-1357) for the alignment outputs: the score matrix of
one pair, as ``oracle.nisqa_oracle.de_align`` computes it before its softmax, and the four values the engine reports per
degraded step (include/nisqa_b200.h nisqa_alignment_out).

TEST INFRASTRUCTURE ONLY (like the rest of oracle/).  Pinned against the unmodified reference modules by
tests/golden/alignment.npz (oracle/make_alignment_golden.py).
"""
import torch
import torch.nn.functional as F


def scores(args, x, y, sd):
    """Alignment.forward's att_score (lib:1279-1282) of ONE pair in float64, no padding so no mask: s [Sx, Sy] of degraded
    rows x [Sx, d] against reference rows y [Sy, d] - AttDot, AttCosine (eps 1e-8 per norm), AttDistance (default
    norms), AttLuong x . (W y + b), AttBahdanau v . tanh(Wq x + bq + Wy y + by) + v's bias."""
    x, y = torch.as_tensor(x).double(), torch.as_tensor(y).double()
    w = {k: v.double() for k, v in (sd or {}).items() if k.startswith("align.")}
    method = args["de_align"]
    if method == "dot":
        return x @ y.t()
    if method == "cosine":
        return (x @ y.t()) / (x.norm(dim=1).clamp_min(1e-8)[:, None] * y.norm(dim=1).clamp_min(1e-8)[None, :])
    if method == "distance":
        return -torch.cdist(x, y, p=1) / x.shape[1]
    if method == "luong":
        return x @ F.linear(y, w["align.att.W.weight"], w["align.att.W.bias"]).t()
    if method == "bahd":
        xq = F.linear(x, w["align.att.Wq.weight"], w["align.att.Wq.bias"])
        yk = F.linear(y, w["align.att.Wy.weight"], w["align.att.Wy.bias"])
        v, vb = w["align.att.v.weight"].reshape(-1), w["align.att.v.bias"].reshape(())
        return torch.stack([torch.tanh(xq[i][None, :] + yk) @ v for i in range(x.shape[0])]) + vb
    raise NotImplementedError(method)


def stats(s):
    """The alignment of each degraded step from its score row s [Sx, Sy] -> float64 (ref_seg = the first maximal s_ij,
    weight = softmax_j(s_ij) at ref_seg, centroid = sum_j softmax_j(s_ij) j, peak = s_i,ref_seg)."""
    s = torch.as_tensor(s).double()
    a = torch.softmax(s, dim=1)
    ref_seg = (s == s.max(1, keepdim=True)[0]).double().argmax(1)
    rows = torch.arange(s.shape[0])
    return ref_seg, a[rows, ref_seg], a @ torch.arange(s.shape[1], dtype=torch.float64), s[rows, ref_seg]
