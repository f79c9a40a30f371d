"""CPU oracle of the per-segment scores and pooling weights (include/nisqa_b200.h nisqa_segment_out,
nisqa_predict_device_batch_segments, Scorer.segments).

TEST INFRASTRUCTURE ONLY, like the rest of oracle/.  A restatement of the definition from the checkpoint's own pooling
tensors (``lib`` = nisqa/NISQA_lib.py, lib:1099-1225), pinned against the unmodified reference pooling modules by
tests/golden/segments.npz (oracle/make_segment_golden.py).
"""
import numpy as np
import torch
import torch.nn.functional as F


def segment_scores(args, sd, x):
    """Per-segment scores and pooling weights of one clip: x [S, D], the rows the pooling module reads -> (scores
    [S, n_heads], weights [S, n_heads]) float32.  A segment's score is the module applied to x[t:t+1], i.e. its last
    Linear of x_t; its weight is the attention softmax weight (att), 1 / S (avg), [t == S - 1] (last_step) or NaN (max,
    last_step_bi)."""
    prefixes = ["pool_layers.%d.model." % i for i in range(5)] if args["model"] == "NISQA_DIM" else ["pool.model."]
    pool, S = args["pool"], x.shape[0]
    scores, weights = [], []
    with torch.no_grad():
        for pf in prefixes:
            if pool == "att":
                last = pf + ("linear3" if args.get("pool_att_h") else "linear2")
                a = F.linear(x, sd[pf + "linear1.weight"], sd[pf + "linear1.bias"])
                if args.get("pool_att_h"):
                    a = F.linear(F.relu(a), sd[pf + "linear2.weight"], sd[pf + "linear2.bias"])
                w = torch.softmax(a[:, 0], dim=0)
            else:
                last = pf + "linear"
                w = {"avg": torch.full((S,), 1.0 / S), "last_step": (torch.arange(S) == S - 1).float()}.get(
                    pool, torch.full((S,), float("nan")))
            scores.append(F.linear(x, sd[last + ".weight"], sd[last + ".bias"])[:, 0])
            weights.append(w)
    return torch.stack(scores, 1).numpy().astype(np.float32), torch.stack(weights, 1).numpy().astype(np.float32)
