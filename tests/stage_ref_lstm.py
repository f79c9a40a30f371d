"""Float64 reference of a stacked LSTM of any width, depth and direction, with the first-order bound of tests/stage_ref.py
(whose helpers it reuses): each layer's input error, carried in from the layer below, enters the gate pre-activations
through |W_ih|; the recurrent error goes root-sum-square through W_hh as in stage_ref.bilstm; TAU bounds what fp32 adds to
each operation.  Also the pooling modules stage_ref.pool_heads does not cover (PoolAtt, PoolAvg, PoolMax, PoolLastStep).
"""
import torch

import stage_ref as R
from stage_ref import TAU, _d, _rss

P = "time_dependency.model.lstm."


def lstm_layer(sd, sfx, clips, errs, rev):
    """One direction of one layer over a list of [S_i, in] float64 inputs and their bounds -> list of ([S_i, H], bound)."""
    w_ih, w_hh = _d(sd[P + "weight_ih" + sfx]), _d(sd[P + "weight_hh" + sfx])
    b = _d(sd[P + "bias_ih" + sfx]) + _d(sd[P + "bias_hh" + sfx])
    H = w_hh.shape[1]
    n, T = len(clips), max(c.shape[0] for c in clips)
    lens = torch.tensor([c.shape[0] for c in clips])
    X = torch.zeros(n, T, clips[0].shape[1], dtype=torch.float64)
    EX = torch.zeros_like(X)
    for i, (c, e) in enumerate(zip(clips, errs)):
        X[i, :c.shape[0]] = c.flip(0) if rev else c
        EX[i, :c.shape[0]] = e.flip(0) if rev else e
    gx = X @ w_ih.t() + b
    mx = X.abs() @ w_ih.t().abs() + b.abs()
    ex = EX @ w_ih.t().abs()
    h = torch.zeros(n, H, dtype=torch.float64)
    c = torch.zeros_like(h)
    eh, ec = torch.zeros_like(h), torch.zeros_like(h)
    Y, EY = torch.zeros(n, T, H, dtype=torch.float64), torch.zeros(n, T, H, dtype=torch.float64)
    for t in range(T):
        g = gx[:, t] + h @ w_hh.t()
        eg = ex[:, t] + _rss(eh, w_hh.t()) + TAU * (mx[:, t] + h.abs() @ w_hh.t().abs())
        sg, tg = torch.sigmoid(g), torch.tanh(g)
        esg = sg * (1 - sg) * eg + TAU * sg
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
    out = []
    for i, L in enumerate(lens.tolist()):
        y, e = Y[i, :L], EY[i, :L]
        out.append((y.flip(0), e.flip(0)) if rev else (y, e))
    return out


def lstm_stack(sd, clips, errs):
    """Every layer of the checkpoint's LSTM over a list of clips' input rows -> list of ([S_i, dirs H], bound)."""
    layers = 0
    while P + "weight_hh_l%d" % layers in sd:
        layers += 1
    dirs = 2 if P + "weight_hh_l0_reverse" in sd else 1
    for l in range(layers):
        per_dir = [lstm_layer(sd, "_l%d%s" % (l, "_reverse" if d else ""), clips, errs, d == 1) for d in range(dirs)]
        clips = [torch.cat([per_dir[d][i][0] for d in range(dirs)], 1) for i in range(len(clips))]
        errs = [torch.cat([per_dir[d][i][1] for d in range(dirs)], 1) for i in range(len(clips))]
    return list(zip(clips, errs))


def pool_heads(sd, args, x, err):
    """td_out of ONE clip -> (scores [n_out], bound) for every pooling module."""
    if args["pool"] == "last_step_bi" or (args["pool"] == "att" and args.get("pool_att_h")):
        return R.pool_heads(sd, args, x, err)
    prefixes = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    ys, es = [], []
    for pf in prefixes:
        if args["pool"] == "att":
            a, ea = R.linear(x, err, sd[pf + "linear1.weight"], sd[pf + "linear1.bias"])
            p, ep = R.softmax_rows(a.t(), ea.t())
            v, ev = R.matmul(p, ep, x, err)
            y, e = R.linear(v, ev, sd[pf + "linear2.weight"], sd[pf + "linear2.bias"])
        else:
            if args["pool"] == "avg":
                v = x.mean(0, keepdim=True)
                ev = err.mean(0, keepdim=True) + TAU * x.abs().mean(0, keepdim=True)
            elif args["pool"] == "max":
                v = x.max(0, keepdim=True)[0]
                ev = err.max(0, keepdim=True)[0]
            elif args["pool"] == "last_step":
                v, ev = x[-1:], err[-1:]
            else:
                raise NotImplementedError(args["pool"])
            y, e = R.linear(v, ev, sd[pf + "linear.weight"], sd[pf + "linear.bias"])
        ys.append(y.reshape(-1))
        es.append(e.reshape(-1))
    return torch.cat(ys), torch.cat(es)
