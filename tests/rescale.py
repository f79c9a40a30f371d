"""Power-of-two rescaling of a checkpoint that leaves the network's function unchanged.

BatchNorm i's weight and bias times 2^k scale conv layer i's output by 2^k; ReLU and max-pooling commute with a
positive scale, so dividing the weights of the next layer by 2^k restores its input exactly (conv i+1 for i < 6, the
Linear behind the CNN for i = 6).  All factors are powers of two, so every fp32 product of the rescaled network is the
original one times a power of two, and the oracle's scores are bit-identical.

The same holds channel by channel (rescale_channels): BatchNorm i's channel c times 2^k_c, input channel c of its
consumer times 2^-k_c.  The engine stores each channel of the activations at its own power-of-two scale, taken from its
own folded BatchNorm (pack_weights), so a rescaled checkpoint leaves every stored fp16 value unchanged either way.
"""
import torch


def _next_linear(sd):
    for key in ("cnn.model.fc.weight", "cnn.model.fc_out.weight", "time_dependency.model.linear.weight"):
        if key in sd:
            return [key]
    return [k for k in sd if k.startswith("time_dependency.model.lstm.weight_ih_l0")]


def rescale(sd, layer, k):
    """Copy of state dict `sd` with BatchNorm `layer` (1..6) scaled by 2^k and its consumer by 2^-k."""
    out = dict(sd)
    p = "cnn.model."
    for name in ("bn%d.weight" % layer, "bn%d.bias" % layer):
        out[p + name] = torch.ldexp(sd[p + name], torch.tensor(k))
    nxt = [p + "conv%d.weight" % (layer + 1)] if layer < 6 else _next_linear(sd)
    for name in nxt:
        out[name] = torch.ldexp(sd[name], torch.tensor(-k))
    return out


def rescale_channels(sd, layer, ks):
    """Copy of state dict `sd` with channel c of BatchNorm `layer` (1..6) scaled by 2^ks[c] and input channel c of its
    consumer by 2^-ks[c]: conv layer+1, or for layer 6 the features c * hw + pos (the CNN output flattened channel-major,
    hw positions per channel) of the Linear or LSTM behind the CNN."""
    out = dict(sd)
    p = "cnn.model."
    ks = torch.as_tensor(ks, dtype=torch.int32)
    for name in ("bn%d.weight" % layer, "bn%d.bias" % layer):
        assert sd[p + name].shape == ks.shape, (name, tuple(sd[p + name].shape), tuple(ks.shape))
        out[p + name] = torch.ldexp(sd[p + name], ks)
    if layer < 6:
        w = sd[p + "conv%d.weight" % (layer + 1)]
        out[p + "conv%d.weight" % (layer + 1)] = torch.ldexp(w, -ks[None, :, None, None])
        return out
    for name in _next_linear(sd):
        w = sd[name]
        hw = w.shape[1] // ks.numel()
        assert hw * ks.numel() == w.shape[1], (name, tuple(w.shape))
        out[name] = torch.ldexp(w, -ks.repeat_interleave(hw)[None, :])
    return out
