"""The double-ended model's alignment and fusion (de_align_kernel, csrc/td_tiled.cu) against float64
(tests/stage_ref_de.py), with reference clips longer than one 64-step key block.

The kernel walks the reference clip's steps in blocks of 64 keys: a double-buffered key tile, an online max / sum for
soft attention, the first maximal score of a block for hard attention (a later block replaces it only with a strictly
greater one), per-block key norms (cosine) and per-block key projections (Luong, Bahdanau).  All of that only runs
from the second key block on.

CPU: the float64 reference against oracle.nisqa_oracle.de_align / de_fuse in float64; a float32 emulation of the
kernel's blocked schedule passes the check, and each of a list of faults in that schedule fails it.  Inputs are td
output rows the oracle computes for synthetic clips, not random rows.
GPU: ten alignment / application / fusion variants through the C ABI, stage by stage from the engine's own dumps
(TD_IN -> TD1_OUT -> DE_FUSED -> TD_OUT -> scores), against the oracle's scores, and several passes == one pass.
"""
import functools
import math
import os

import numpy as np
import pytest
import torch

import stage_ref as R
import stage_ref_de as D
from conftest import WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth
from oracle import nisqa_oracle as O
from oracle import variants as V

SR = 16000
KB = 64                   # keys per block of de_align_kernel
ALIGNS = ["dot", "cosine", "distance", "luong", "bahd"]
FUSES = ["x/y/-", "+/-", "x/y"]
# (degraded, reference) step counts of the CPU checks: every one of 1, 63, 64, 65, 130 and 1297 on both sides
CPU_PAIRS = [(1, 1), (1, 130), (63, 65), (64, 64), (65, 63), (130, 1297), (1297, 130)]


@functools.lru_cache(maxsize=None)
def _base():
    return O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))


def _checkpoint(name, over):
    bargs, bsd = _base()
    return V.de_checkpoint(name, bargs, bsd, over)


def _n_samples(args, n_seg):
    return (15 + (n_seg - 1) * args["ms_seg_hop_length"] - 1) * int(SR * args["ms_hop_length"])


def _pcm(args, n_seg, seed):
    """a 16 kHz clip of exactly n_seg segments"""
    n = _n_samples(args, n_seg)
    y = synth.synth_speech_pcm16(seed, n / SR + 0.05, SR)[:n]
    assert O.segment_counts(n, SR, args)[1] == n_seg
    return y


def _silent_start(args, n_seg, seed, silence_s):
    """a clip of exactly n_seg segments whose first silence_s seconds are digital silence: identical td rows"""
    y = _pcm(args, n_seg, seed).copy()
    y[:int(silence_s * SR)] = 0
    return y


def _degrade(ref, seed, n=None):
    """delay + gain + noise + clipping of a reference clip (as oracle.variants.de_pair_pcm does): clear alignment peaks"""
    rng = np.random.default_rng(seed)
    x = np.roll(ref.astype(np.float32), int(0.013 * SR))[:n or len(ref)]
    x = x * 1.6 + rng.standard_normal(len(x)).astype(np.float32) * 250.0
    return np.clip(x, -9000, 9000).astype(np.int16)


def _f32(pcm):
    return pcm.astype(np.float32) / np.float32(32768.0)


@functools.lru_cache(maxsize=None)
def _td_rows():
    """td output rows (oracle, float32) of a 1297-step reference clip that starts with 3.5 s of digital silence (its
    silent steps span key blocks 0 and 1) and of a degraded clip derived from it"""
    args, sd = _base()
    ref = _silent_start(args, 1297, 31, 3.5)
    deg = _degrade(ref, 32)
    out = []
    with torch.no_grad():
        for pcm in (deg, ref):
            feats = O.adapt_cnn(sd, O.segments(O.mel_db(_f32(pcm), SR, args), args), args)
            out.append(O.self_attention(sd, feats))
    return out


def _pair_rows(sx, sy):
    """float64 (x, y): the last sx degraded and the last sy reference rows (the aligned tails)"""
    x, y = _td_rows()
    return x[-sx:].double(), y[-sy:].double()


def _sd64(sd):
    return {k: v.double() for k, v in sd.items() if k.startswith(("align.", "fuse."))}


def _check(args, sd, x, y, got):
    """max |got - ref| / bound of the fused rows (soft), or 0 / inf for hard rows inside / outside their candidates"""
    s, b = D.scores(args, sd, x, y)
    if args["de_align_apply"] == "hard":
        bad, _ = D.check_hard(args, x, y, got, D.candidates(s, b))
        return 0.0 if bad is None else math.inf
    ref, bound = D.fuse(args, x, *D.soft_align(s, b, y))
    return R.ratio(got, ref, bound)


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("align", ALIGNS)
def test_float64_reference_equals_the_oracle(align):
    """stage_ref_de in float64 == oracle de_align / de_fuse (+ lin_fusion) in float64, every application and fusion"""
    for apply in ("hard", "soft"):
        for fuse in FUSES + ["fuse_dim"]:
            over = {"de_align": align, "de_align_apply": apply, "de_fuse": "x/y/-" if fuse == "fuse_dim" else fuse}
            if fuse == "fuse_dim":
                over["de_fuse_dim"] = 64
            name = "cpu_%s_%s_%s" % (align, apply, fuse)
            args, sd = _checkpoint(name, over)
            sd64 = _sd64(sd)
            for sx, sy in CPU_PAIRS:
                x, y = _pair_rows(sx, sy)
                s, b = D.scores(args, sd, x, y)
                y_or = O.de_align(args, x, y, sd64)
                if apply == "soft":
                    y_al, e_al = D.soft_align(s, b, y)
                    rows = torch.ones(sx, dtype=torch.bool)
                else:
                    cand = D.candidates(s, b)
                    rows = cand.sum(1) == 1
                    y_al, e_al = y[cand.double().argmax(1)], torch.zeros_like(x)
                    assert rows.double().mean() >= 0.5, (name, sx, sy)
                tol = 1e-12 * float(y.abs().max())
                np.testing.assert_allclose(y_al[rows], y_or[rows], rtol=0, atol=tol, err_msg=name)
                f_ref, _ = D.fuse(args, x, y_al, e_al)
                if args.get("de_fuse_dim"):
                    f_ref, _ = D.lin_fusion(sd, f_ref)
                f_or = O.de_fuse(args, x, y_or, sd64)
                np.testing.assert_allclose(f_ref[rows], f_or[rows], rtol=0, atol=10 * tol, err_msg=name)


def _score32(args, sd, X, Y, fault):
    """fp32 scores [64, 64] of one query tile against one key tile (zero rows beyond the clips)"""
    m = args["de_align"]
    if m in ("dot", "cosine"):
        return X @ Y.t()
    if m == "distance":
        return -torch.cdist(X, Y, p=1) / 64
    if m == "luong":
        yp = Y @ sd["align.att.W.weight"].t()
        if fault != "key_bias":
            yp = yp + sd["align.att.W.bias"]
        return X @ yp.t()
    xq = X @ sd["align.att.Wq.weight"].t() + sd["align.att.Wq.bias"]
    yk = Y @ sd["align.att.Wy.weight"].t()
    if fault != "key_bias":
        yk = yk + sd["align.att.Wy.bias"]
    return torch.tanh(xq[:, None, :] + yk[None, :, :]) @ sd["align.att.v.weight"].reshape(-1)


def _inv_norm(T):
    return 1.0 / T.norm(dim=1).clamp_min(D.EPS_COS)


def emulate(args, sd, x, y, fault=None):
    """float32 model of de_align_kernel's schedule for one pair -> fused rows [Sx, 64 nf].  Query tiles of 64 rows;
    key blocks of 64 zero-padded rows with the padding keys masked; soft: online max / sum with the rescale of l and o
    whenever the running max rises; hard: the first maximal score of each block, replaced only by a strictly greater
    score of a later block.  `fault` injects one mistake (FAULTS)."""
    x32, y32 = x.float(), y.float()
    sx, sy = x32.shape[0], y32.shape[0]
    n_kb = (sy + KB - 1) // KB
    ypad = torch.zeros(n_kb * KB, 64)
    ypad[:sy] = y32
    blocks = [ypad[kb * KB:(kb + 1) * KB] for kb in range(n_kb)]
    hard = args["de_align_apply"] == "hard"
    out = []
    for q0 in range(0, sx, KB):
        src = q0 + KB if fault == "query_tile" else q0
        X = torch.zeros(KB, 64)
        rows = x32[src:src + KB]
        X[:rows.shape[0]] = rows
        m = torch.full((KB,), -math.inf)
        l, o = torch.zeros(KB), torch.zeros(KB, 64)
        best = torch.zeros(KB, dtype=torch.long)
        for kb in range(n_kb):
            j0 = kb * KB
            Y = blocks[kb - 1] if fault == "stale_keys" and kb > 0 else blocks[kb]
            s = _score32(args, sd, X, Y, fault)
            if args["de_align"] == "cosine":
                ry = _inv_norm(blocks[kb - 1] if fault == "norm_slot" and kb > 0 else Y)
                s = s * _inv_norm(X)[:, None] * ry[None, :]
            if fault != "unmasked_padding":
                s = s.masked_fill(torch.arange(KB)[None, :] >= sy - j0, -math.inf)
            if hard:
                bv, bi = s.max(1)                                  # (the first maximal score of the block)
                bi = bi + (0 if fault == "drop_j0" else j0)
                upd = bv > m
                m, best = torch.where(upd, bv, m), torch.where(upd, bi, best)
            else:
                mn = torch.maximum(m, s.max(1)[0])
                sc = torch.ones(KB) if fault == "no_rescale" else torch.exp(m - mn)
                p = torch.exp(s - mn[:, None])
                l = l * sc + p.sum(1)
                o = o * sc[:, None] + p @ Y
                m = mn
        y_al = ypad[best] if hard else o / l[:, None]
        out.append(D.fuse_f32(args, X, y_al)[:min(KB, sx - q0)])
    return torch.cat(out)


# mutation -> the alignment methods it applies to, and the applications
FAULTS = {
    "no_rescale": (ALIGNS, ["soft"]),                    # o and l keep their scale when the running max rises
    "stale_keys": (ALIGNS, ["hard", "soft"]),            # block kb reads block kb - 1's keys
    "unmasked_padding": (ALIGNS, ["hard", "soft"]),      # the last block's zero padding keys take part
    "norm_slot": (["cosine"], ["hard", "soft"]),         # the key norms of the other slot (the previous block)
    "drop_j0": (ALIGNS, ["hard"]),                       # the block-local key index is taken as the global one
    "key_bias": (["luong", "bahd"], ["hard", "soft"]),   # W y (Luong) / Wy y (Bahdanau) without the key-side bias
    "query_tile": (ALIGNS, ["hard", "soft"]),            # the degraded rows of the next query tile
}
# (fault, align, apply) the check cannot see on any input, and why
INVISIBLE = {
    # x . (W y + b) = x . W y + x . b: the bias term is the same for every key of a row, and softmax and argmax drop it
    ("key_bias", "luong", "hard"): "x . b shifts every score of a row alike",
    ("key_bias", "luong", "soft"): "x . b shifts every score of a row alike",
}
# (fault, align, apply) these inputs cannot show although other inputs could, and why
NOT_ON_THESE_INPUTS = {
    # A padding key is a zero row.  Hard attention only notices it where it would be the row's maximum, soft attention
    # where its weight exp(score - max) is not negligible.  The td rows are LayerNorm outputs: every row has a real key
    # scoring far above the zero key for these methods (the Luong zero key scores x . b, which does win, and the soft
    # cosine / distance / Bahdanau weights of the zero key are large: those cases are caught).
    ("unmasked_padding", "dot", "hard"): "the zero key scores 0, below every row's best dot product",
    ("unmasked_padding", "dot", "soft"): "the zero key's weight exp(0 - max) is far below the bound",
    ("unmasked_padding", "cosine", "hard"): "the zero key scores 0, below every row's best cosine",
    ("unmasked_padding", "distance", "hard"): "every row has a key closer than mean |x| (the zero key's distance)",
    ("unmasked_padding", "bahd", "hard"): "the zero key's v . tanh(Wq x + bq + by) is below every row's best score",
}
MUTATION_PAIRS = [(p[0], p[1]) for p in CPU_PAIRS if p[1] > KB]       # every one with more than one key block


def _mode_args(align, apply, fuse="x/y/-"):
    return _checkpoint("cpu_%s_%s_%s" % (align, apply, fuse), {"de_align": align, "de_align_apply": apply, "de_fuse": fuse})


@pytest.mark.parametrize("align", ALIGNS)
def test_blocked_fp32_schedule_passes_the_check(align):
    """The kernel's schedule in float32 is inside the bound (soft) or picks a candidate (hard) for every fusion; so
    does the fp32 oracle's softmax + argmax."""
    worst = {}
    for apply in ("hard", "soft"):
        for fuse in FUSES:
            args, sd = _mode_args(align, apply, fuse)
            for sx, sy in CPU_PAIRS:
                x, y = _pair_rows(sx, sy)
                r = _check(args, sd, x, y, emulate(args, sd, x, y))
                worst[apply] = max(worst.get(apply, 0.0), r)
                assert r <= 1.0, (align, apply, fuse, sx, sy, r)
            if apply == "hard" and fuse == "x/y":
                for sx, sy in CPU_PAIRS:
                    x, y = _pair_rows(sx, sy)
                    y_or = O.de_align(args, x.float(), y.float(), sd)
                    assert _check(args, sd, x, y, torch.cat((x.float(), y_or), 1)) == 0.0, (align, sx, sy)
    print("\n%s: emulation max ratio %s" % (align, worst))


@pytest.mark.parametrize("fault", list(FAULTS))
def test_blocked_fp32_schedule_with_a_fault_fails_the_check(fault):
    aligns, applies = FAULTS[fault]
    for align in aligns:
        for apply in applies:
            args, sd = _mode_args(align, apply)
            rs = []
            for sx, sy in MUTATION_PAIRS:
                x, y = _pair_rows(sx, sy)
                rs.append(_check(args, sd, x, y, emulate(args, sd, x, y, fault)))
            key = (fault, align, apply)
            print("%s %s %s: ratios %s" % (fault, align, apply, ["%.3g" % r for r in rs]))
            if key in INVISIBLE or key in NOT_ON_THESE_INPUTS:
                assert max(rs) <= 1.0, (key, rs)         # (documented as not visible here: keep the list true)
            else:
                assert max(rs) > 1.0, (key, rs)


def test_luong_key_bias_shifts_each_row_alike():
    """why INVISIBLE lists the Luong key bias: x . b is one constant per degraded row"""
    for (fault, align, apply) in list(INVISIBLE) + list(NOT_ON_THESE_INPUTS):
        assert align in FAULTS[fault][0] and apply in FAULTS[fault][1]
    args, sd = _mode_args("luong", "soft")
    x, y = _pair_rows(130, 1297)
    s = D.scores(args, sd, x, y)[0]
    sd0 = dict(sd, **{"align.att.W.bias": torch.zeros(64)})
    s0 = D.scores(args, sd0, x, y)[0]
    shift = s - s0                                      # x . b: constant along each row
    assert float((shift - shift[:, :1]).abs().max()) <= 1e-12 * float(shift.abs().max())


# ------------------------------------------------------------------------------------------------------------ GPU
GPU_VARIANTS = dict(V.DE_VARIANTS)
GPU_VARIANTS["de_distance_hard"] = {"de_align": "distance", "de_align_apply": "hard", "de_fuse": "x/y/-"}
GPU_VARIANTS["de_bahd_hard"] = {"de_align": "bahd", "de_align_apply": "hard", "de_fuse": "+/-"}


def _gpu_batch(args):
    """-> list of (deg, ref) int16 16 kHz pairs, and the index of the pair whose reference is too short"""
    pairs = [(_pcm(args, a, 200 + i), _pcm(args, b, 300 + i)) for i, (a, b) in enumerate(
        [(1, 1), (1, 129), (129, 1), (64, 64), (65, 63), (63, 65)])]
    ref128 = _pcm(args, 128, 310)
    pairs.append((_degrade(ref128, 311), ref128))
    ref_long = _silent_start(args, 1297, 312, 3.5)                    # 21 key blocks; silent steps in blocks 0 and 1
    pairs.append((_degrade(ref_long, 313, _n_samples(args, 200)), ref_long))
    short = len(pairs)
    pairs.append((_pcm(args, 40, 314), np.zeros(100, np.int16)))
    pairs.append((_pcm(args, 700, 315), _pcm(args, 130, 316)))
    return pairs, short


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_VARIANTS))
def test_de_alignment_stages_against_float64(built_lib, name):
    """TD_IN -> TD1_OUT -> DE_FUSED -> TD_OUT -> scores from the engine's own dumps, each against float64 (bound TAU =
    2^-18 times the magnitude of the stage's terms); scores against the oracle; several passes == one pass."""
    args, sd = _checkpoint(name, GPU_VARIANTS[name])
    pairs, short = _gpu_batch(args)
    clips = [c for p in pairs for c in p]
    srs = [SR] * len(clips)
    hard = args["de_align_apply"] == "hard"
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    try:
        scores, nseg, status = eng.predict_pcm(clips, srs)
        ok = status == E.CLIP_OK
        assert status[2 * short + 1] == E.CLIP_TOO_SHORT and ok.sum() == len(clips) - 1
        has_rows = np.repeat(ok[0::2] & ok[1::2], 2)            # a pair with a clip the engine skips has no rows
        N = int(nseg[has_rows].sum())
        dump = lambda st: torch.from_numpy(eng.stage_dump(st)).double().reshape(N, -1)      # noqa: E731
        td_in, td1, fused, td_out = (dump(s) for s in (E.STAGE_TD_IN, E.STAGE_TD1_OUT, E.STAGE_DE_FUSED, E.STAGE_TD_OUT))
        alone, nseg1, _ = eng.predict_pcm(clips[14:16], srs[14:16])        # the (200, 1297) pair alone
        np.testing.assert_array_equal(alone[0], scores[14])
        np.testing.assert_array_equal(nseg1, nseg[14:16])
    finally:
        eng.close()
    assert fused.shape[1] == 64 * D.n_fused(args)
    rows_of = np.where(has_rows, nseg, 0)
    starts = np.concatenate([[0], np.cumsum(rows_of)])
    rows = lambda t, c: t[starts[c]:starts[c + 1]]          # noqa: E731
    zero = torch.zeros_like
    ratios, unique = {}, []

    def add(k, got, ref, bound):
        ratios[k] = max(ratios.get(k, 0.0), R.ratio(got, ref, bound))
    for c in range(len(clips)):
        if has_rows[c]:
            ref, b = R.sa_stack(sd, rows(td_in, c), zero(rows(td_in, c)))
            add("td_in->td1_out", rows(td1, c), ref, b)
        if c % 2:
            assert not rows(fused, c).any(), (name, c)          # reference rows stay zero
    pf = "time_dependency_2.model."
    for p in range(len(pairs)):
        if p == short:
            continue
        x, y = rows(td1, 2 * p), rows(td1, 2 * p + 1)
        got = rows(fused, 2 * p)
        s, b = D.scores(args, sd, x, y)
        if hard:
            bad, frac = D.check_hard(args, x, y, got, D.candidates(s, b))
            assert bad is None, (name, p, bad)
            unique.append((frac, x.shape[0]))
        else:
            ref, bd = D.fuse(args, x, *D.soft_align(s, b, y))
            add("td1_out->de_fused", got, ref, bd)
        f, ef = got, zero(got)
        if args.get("de_fuse_dim"):
            f, ef = D.lin_fusion(sd, f)
        h, eh = R.td_in(sd, f, ef, prefix=pf)
        if args.get("td_2_sa_pos_enc"):
            pe = sd[pf + "pos_encoder.pe"][:h.shape[0], 0, :].double()
            h, eh = R.add(h, eh, pe, zero(pe))
        ref, bd = R.sa_stack(sd, h, eh, prefix=pf)
        add("de_fused->td_out", rows(td_out, 2 * p), ref, bd)
        y_out = rows(td_out, 2 * p)
        ref, bd = R.pool_heads(sd, args, y_out, zero(y_out))
        add("td_out->scores", scores[2 * p], ref, bd)
    msg = "\n%s max |got - ref| / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items()))
    if hard:
        frac = sum(f * n for f, n in unique) / sum(n for _, n in unique)
        msg += "; hard rows with one candidate: %.3f" % frac
    print(msg)
    assert all(r <= 1.0 for r in ratios.values()), ratios
    if hard:
        assert frac >= 0.5, frac
    assert np.all(np.isnan(scores[1::2])) and np.isnan(scores[2 * short, 0])
    # the oracle on the pairs up to 5.3 s (the others only add runtime)
    tol = 5e-4 if hard else 1e-4
    worst = 0.0
    for p, (deg, ref) in enumerate(pairs):
        if p == short or max(nseg[2 * p], nseg[2 * p + 1]) > 129:
            continue
        sc, ns, st = O.predict_pcm_de(args, sd, _f32(deg), SR, _f32(ref), SR)
        assert st == O.STATUS_OK and ns == (nseg[2 * p], nseg[2 * p + 1]), (name, p)
        worst = max(worst, abs(float(scores[2 * p, 0]) - float(sc[0])))
    print("%s: max |engine - oracle| %.3g" % (name, worst))
    assert worst <= tol, (name, worst)
    eng = E.Engine(E.config_from_args(args, max_chunk_segments=256), 0)     # pairs in separate passes == one pass
    eng.load_state_dict(sd)
    try:
        multi, nseg2, status2 = eng.predict_pcm(clips, srs)
    finally:
        eng.close()
    np.testing.assert_array_equal(nseg2, nseg)
    np.testing.assert_array_equal(status2, status)
    np.testing.assert_array_equal(multi, scores)


@pytest.mark.gpu
def test_de_fused_is_not_available_for_a_single_ended_model(built_lib):
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_mos_only.tar"))
    eng = E.Engine(E.config_from_args(args), 0)
    eng.load_state_dict(sd)
    try:
        eng.predict_pcm([synth.synth_speech_pcm16(5, 1.0, SR)], [SR])
        with pytest.raises(E.EngineError, match="stage not available"):
            eng.stage_dump(E.STAGE_DE_FUSED)
    finally:
        eng.close()
