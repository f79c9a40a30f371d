"""Float64 references of single engine stages, each with a first-order bound on what fp32 arithmetic may add.

Every function takes float64 values together with an elementwise bound on the error they already carry (zero for a
stage dump: a plane dump is hi + lo summed in fp32, which is exact, so a reference that starts from a dump starts from
the very values the kernel read) and returns the float64 result of the operation plus the bound of its output:

    bound_out = (error carried in, propagated to first order) + TAU * (magnitude of the operation's terms)

The magnitude of a dot product is sum |x| |w| (+ |b|); LayerNorm scales it by |gamma| / sigma, softmax by the
probabilities.  A convolution stage starts from a dump and propagates nothing (or, conv1 into conv2 on the fused
path, through |w|).  Multi-operation stages (the attention stack, the BiLSTM, the pooling heads) carry their errors
through each product norm-wise, as root-sum-squares (sqrt(err^2 |w|^2)): a worst-case |w| propagation compounds the
row sums of every Linear and is loose by orders of magnitude after a few layers or LSTM steps.

fp32 accumulation of n terms stays far below n 2^-24 of the magnitude, so TAU = 2^-18 (about 15x above fp32
conv2d) holds for every correct kernel here, while a kernel that loses a correction term of the fp16 split (2^-12 of
the magnitude) or misplaces a row is far outside it.  A value written as an fp16 hi / lo pair adds SPLIT = 2^-22 of
itself.
"""
import math

import torch
import torch.nn.functional as F

TAU = 2.0 ** -18
SPLIT = 2.0 ** -22
EPS = 1e-5


def _d(t):
    return torch.as_tensor(t).double()


# ------------------------------------------------------------------------------------------------------------ CNN
def fold_bn(sd, i):
    """conv i + eval-mode BatchNorm i as one convolution (float64)."""
    p = "cnn.model."
    s = _d(sd[p + "bn%d.weight" % i]) / torch.sqrt(_d(sd[p + "bn%d.running_var" % i]) + EPS)
    w = _d(sd[p + "conv%d.weight" % i]) * s[:, None, None, None]
    b = (_d(sd[p + "conv%d.bias" % i]) - _d(sd[p + "bn%d.running_mean" % i])) * s + _d(sd[p + "bn%d.bias" % i])
    return w, b


def cnn_layers(args):
    """(padding, pool, split output) of conv1..conv6; pool maps an NCHW tensor (values or bounds: both >= 0 after
    ReLU) to the pooled one."""
    if args["cnn_model"] == "adapt":
        def ap(size):
            return lambda t: F.adaptive_max_pool2d(t, tuple(size))
        return {1: ((1, 1), ap(args["cnn_pool_1"]), True), 2: ((1, 1), ap(args["cnn_pool_2"]), True),
                3: ((1, 1), None, True), 4: ((1, 1), ap(args["cnn_pool_3"]), True), 5: ((1, 1), None, True),
                6: ((1, 0), None, False)}
    first = lambda t: F.max_pool2d(t, 2, stride=2, padding=(0, 1))      # noqa: E731
    mp = lambda t: F.max_pool2d(t, 2, stride=2)                           # noqa: E731
    return {1: (1, first, True), 2: (1, mp, True), 3: (1, None, True), 4: (1, mp, True), 5: (1, None, True),
            6: (1, None, False)}


def conv_layer(sd, args, i, x, err=None):
    """conv i + BN + ReLU (+ pool) of NCHW float64 x -> (ref, bound).  The bound is the carried error through |w|,
    TAU (sum |x| |w_folded| + |b|), max-pooled like the values, plus SPLIT |ref| where the kernel stores fp16 pairs."""
    w, b = fold_bn(sd, i)
    return conv_stage(x, err, w, b, *cnn_layers(args)[i])


def conv_stage(x, err, w, b, pad, pool, split):
    """relu(conv2d(x, w) + b) (+ pool) of float64 NCHW x with the bound of conv_layer."""
    y = F.relu(F.conv2d(x, w, b, padding=pad))
    bound = TAU * F.conv2d(x.abs(), w.abs(), b.abs(), padding=pad)
    if err is not None:
        bound = bound + F.conv2d(err, w.abs(), None, padding=pad)
    if pool is not None:
        y, bound = pool(y), pool(bound)
    if split:
        bound = bound + SPLIT * y
    return y, bound


def cnn_tail(sd, args, y, err):
    """conv6 output NCHW -> the engine's cnn_feat rows (the reference's reshape, + fc / fc_out when present)."""
    n = y.shape[0]
    y, err = y.reshape(n, -1), err.reshape(n, -1)
    for key in ("cnn.model.fc", "cnn.model.fc_out"):
        if key + ".weight" in sd:
            y, err = linear(y, err, sd[key + ".weight"], sd[key + ".bias"])
    return y, err


# --------------------------------------------------------------------------------------------- time dependency
def _rss(err, w):
    """carried error of a product: root-sum-square over the terms of each dot product"""
    return torch.sqrt((err * err) @ (w * w))


def linear(x, err, w, b):
    w, b = _d(w), _d(b)
    y = x @ w.t() + b
    bound = _rss(err, w.t()) + TAU * (x.abs() @ w.abs().t() + b.abs())
    return y, bound


def layer_norm(x, err, g, b):
    """First order: d xhat = (dx - mean dx) / sigma - xhat mean(xhat dx) / sigma."""
    g, b = _d(g), _d(b)
    mu = x.mean(-1, keepdim=True)
    sig = torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + EPS)
    xh = (x - mu) / sig
    y = xh * g + b
    erms = torch.sqrt((err * err).mean(-1, keepdim=True))
    bound = g.abs() / sig * (err + erms + xh.abs() * erms) + TAU * (y.abs() + b.abs())
    return y, bound


def add(a, ea, b, eb):
    y = a + b
    return y, ea + eb + TAU * (a.abs() + b.abs())


def softmax_rows(s, es):
    """softmax over the last dim; d p_i = p_i (d s_i - sum_j p_j d s_j)."""
    p = torch.softmax(s, dim=-1)
    return p, p * (es + (p * es).sum(-1, keepdim=True)) + TAU * p


def matmul(a, ea, b, eb):
    y = a @ b
    return y, _rss(ea, b) + _rss(eb.t(), a.t()).t() + TAU * (a.abs() @ b.abs())


def td_in(sd, x, err, prefix="time_dependency.model."):
    """SelfAttention's Linear + LayerNorm (lib:988-990) of one or more clips' cnn_feat rows."""
    y, e = linear(x, err, sd[prefix + "linear.weight"], sd[prefix + "linear.bias"])
    return layer_norm(y, e, sd[prefix + "norm1.weight"], sd[prefix + "norm1.bias"])


def sa_stack(sd, x, err, prefix="time_dependency.model."):
    """The encoder layers of ONE clip (post-norm, one head, lib:1025-1040)."""
    n_layers = len({k.split(".")[3] for k in sd if k.startswith(prefix + "layers.")})
    for l in range(n_layers):
        q = prefix + "layers.%d." % l
        d = x.shape[-1]
        w_in, b_in = _d(sd[q + "self_attn.in_proj_weight"]), _d(sd[q + "self_attn.in_proj_bias"])
        scale = torch.ones(3 * d, dtype=torch.float64)
        scale[:d] = 1.0 / math.sqrt(d)                                   # exact power of two, folded into W_q
        qkv, eqkv = linear(x, err, w_in * scale[:, None], b_in * scale)
        qq, kk, vv = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        eq, ek, ev = eqkv[:, :d], eqkv[:, d:2 * d], eqkv[:, 2 * d:]
        s, es = matmul(qq, eq, kk.t(), ek.t())
        p, ep = softmax_rows(s, es)
        o, eo = matmul(p, ep, vv, ev)
        sa, esa = linear(o, eo, sd[q + "self_attn.out_proj.weight"], sd[q + "self_attn.out_proj.bias"])
        x, err = layer_norm(*add(x, err, sa, esa), sd[q + "norm1.weight"], sd[q + "norm1.bias"])
        h, eh = linear(x, err, sd[q + "linear1.weight"], sd[q + "linear1.bias"])
        h = F.relu(h)
        ff, eff = linear(h, eh, sd[q + "linear2.weight"], sd[q + "linear2.bias"])
        x, err = layer_norm(*add(x, err, ff, eff), sd[q + "norm2.weight"], sd[q + "norm2.bias"])
    return x, err


def bilstm(sd, clips):
    """1-layer BiLSTM (lib:925-943) of a list of [S_i, 20] float64 inputs (no carried error) -> list of
    ([S_i, 2H] ref, bound); clips run side by side, each direction from the clip's own ends."""
    p = "time_dependency.model.lstm."
    n, T = len(clips), max(c.shape[0] for c in clips)
    lens = torch.tensor([c.shape[0] for c in clips])
    outs = []
    for sfx, rev in (("", False), ("_reverse", True)):
        w_ih, w_hh = _d(sd[p + "weight_ih_l0" + sfx]), _d(sd[p + "weight_hh_l0" + sfx])
        b = _d(sd[p + "bias_ih_l0" + sfx]) + _d(sd[p + "bias_hh_l0" + sfx])
        H = w_hh.shape[1]
        X = torch.zeros(n, T, clips[0].shape[1], dtype=torch.float64)
        for i, c in enumerate(clips):
            X[i, :c.shape[0]] = c.flip(0) if rev else c
        gx = X @ w_ih.t() + b
        mx = X.abs() @ w_ih.t().abs() + b.abs()
        h = torch.zeros(n, H, dtype=torch.float64)
        c = torch.zeros_like(h)
        eh, ec = torch.zeros_like(h), torch.zeros_like(h)
        Y, EY = torch.zeros(n, T, H, dtype=torch.float64), torch.zeros(n, T, H, dtype=torch.float64)
        for t in range(T):
            g = gx[:, t] + h @ w_hh.t()
            eg = _rss(eh, w_hh.t()) + TAU * (mx[:, t] + h.abs() @ w_hh.t().abs())
            sg = torch.sigmoid(g)
            tg = torch.tanh(g)
            esg = sg * (1 - sg) * eg + TAU * sg                          # sigmoid' <= 1/4
            etg = (1 - tg * tg) * eg + TAU * tg.abs()
            i_, f_, g_, o_ = (slice(k * H, (k + 1) * H) for k in range(4))
            cn = sg[:, f_] * c + sg[:, i_] * tg[:, g_]
            ecn = (c.abs() * esg[:, f_] + sg[:, f_] * ec + tg[:, g_].abs() * esg[:, i_] + sg[:, i_] * etg[:, g_]
                   + TAU * (sg[:, f_] * c.abs() + sg[:, i_] * tg[:, g_].abs()))
            tc = torch.tanh(cn)
            hn = sg[:, o_] * tc
            ehn = tc.abs() * esg[:, o_] + sg[:, o_] * (1 - tc * tc) * ecn + TAU * hn.abs()
            live = (t < lens)[:, None]
            h, c = torch.where(live, hn, h), torch.where(live, cn, c)
            eh, ec = torch.where(live, ehn, eh), torch.where(live, ecn, ec)
            Y[:, t], EY[:, t] = h, eh
        for i, L in enumerate(lens.tolist()):
            y, e = Y[i, :L], EY[i, :L]
            outs.append((y.flip(0), e.flip(0)) if rev else (y, e))
    return [(torch.cat((outs[i][0], outs[n + i][0]), 1), torch.cat((outs[i][1], outs[n + i][1]), 1)) for i in range(n)]


# --------------------------------------------------------------------------------------------------- pooling
def pool_heads(sd, args, x, err):
    """td_out of ONE clip -> (scores [n_out], bound): PoolAttFF (x5 for NISQA_DIM) or PoolLastStepBi."""
    prefixes = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    ys, es = [], []
    for pf in prefixes:
        if args["pool"] == "att" and args.get("pool_att_h"):
            a, ea = linear(x, err, sd[pf + "linear1.weight"], sd[pf + "linear1.bias"])
            a, ea = linear(F.relu(a), ea, sd[pf + "linear2.weight"], sd[pf + "linear2.bias"])     # [S, 1]
            p, ep = softmax_rows(a.t(), ea.t())                                                   # [1, S]
            v, ev = matmul(p, ep, x, err)
            y, e = linear(v, ev, sd[pf + "linear3.weight"], sd[pf + "linear3.bias"])
        elif args["pool"] == "last_step_bi":
            H = x.shape[1] // 2
            v = torch.cat((x[-1, :H], x[0, H:]))[None, :]
            ev = torch.cat((err[-1, :H], err[0, H:]))[None, :]
            y, e = linear(v, ev, sd[pf + "linear.weight"], sd[pf + "linear.bias"])
        else:
            raise NotImplementedError(args["pool"])
        ys.append(y.reshape(-1))
        es.append(e.reshape(-1))
    return torch.cat(ys), torch.cat(es)


def ratio(got, ref, bound):
    """max |got - ref| / bound (the check passes at <= 1)."""
    got = torch.as_tensor(got).double().reshape(ref.shape)
    return float(((got - ref).abs() / bound.clamp_min(1e-300)).max())
