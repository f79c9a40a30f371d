"""Checkpoints rescaled channel by channel (tests/rescale.py rescale_channels) compute the same function, and the
engine computes it bit for bit.

BatchNorm i's channel c times 2^k_c and input channel c of its consumer times 2^-k_c: ReLU, max-pooling and adaptive
max-pooling commute with a positive scale per channel, so the oracle's scores are bit-identical (CPU, every layer).  The
tensor-core conv path stores each channel's activations as fp16 pairs of v 2^-e_c, e_c taken from that channel's own
folded BatchNorm, and folds 2^-e_c into the producing layer's weights and 2^e_c into the consuming layer's, so every
stored fp16 value, every packed weight and every scale is unchanged by such a rescaling: the engine's scores are
bit-identical on every conv path (GPU), and each stage stays inside the float64 bound of tests/stage_ref.py at spreads
of 2^+-12 and 2^+-24 between the channels of a layer.  One exponent per layer, from the layer's largest channel,
stores a channel far below it with a fixed absolute error instead (tests/test_plane_layout.py emulates that).
"""
import os

import numpy as np
import pytest

from conftest import WEIGHTS
from nisqa_b200 import synth
from oracle import cnn_pool_variants as PV
from oracle import cnn_width_variants as WV
from oracle import de_arch_oracle as DO
from oracle import de_arch_variants as DV
from oracle import mel_variants as MV
from oracle import nisqa_oracle as O
from oracle import td_pair_oracle as TO
from oracle.variants import de_pair_pcm
from rescale import rescale_channels

SR = 16000
TOL = 1e-4
SHIPPED = ["nisqa.tar", "nisqa_tts.tar"]
VARIANTS = {"width": ("mos_c16_64_32", WV.CNN_WIDTH_VARIANTS, WV.cnn_width_checkpoint),
            "pool": ("mos_p16x5_8x4_4x2", PV.CNN_POOL_VARIANTS, PV.cnn_pool_checkpoint),
            "mel": ("mos_adapt_m64_s15", MV.MEL_VARIANTS, MV.mel_checkpoint)}
DE_VARIANT = "std_fc20_sa64_cosine_soft"          # NISQA_DE behind StandardCNN


def _checkpoint(name):
    if name in SHIPPED:
        return O.load_checkpoint(os.path.join(WEIGHTS, name))
    if name == DE_VARIANT:
        base = DV.DE_ARCH_VARIANTS[name][0]
        return DV.de_arch_checkpoint(name, *O.load_checkpoint(os.path.join(WEIGHTS, base)))
    vname, table, make = VARIANTS[name]
    return make(vname, *O.load_checkpoint(os.path.join(WEIGHTS, table[vname][0])))


def exponent_vectors(n, layer, spread=24):
    """seeded per-channel exponents spanning [-spread, spread], and one channel at +spread with the rest at 0"""
    rng = np.random.default_rng(100 * layer + n)
    ks = rng.integers(-spread, spread + 1, n)
    ks[rng.permutation(n)[:2]] = (-spread, spread)
    one = np.zeros(n, np.int64)
    one[rng.integers(n)] = spread
    return [ks, one]


def _channels(sd, layer):
    return sd["cnn.model.bn%d.weight" % layer].numel()


def rescale_every_layer(sd, spread, seed):
    """every BatchNorm 1..6 rescaled channel by channel at once, exponents spanning [-spread, spread]"""
    rng = np.random.default_rng(seed)
    for layer in range(1, 7):
        n = _channels(sd, layer)
        ks = rng.integers(-spread, spread + 1, n)
        ks[rng.permutation(n)[:2]] = (-spread, spread)
        sd = rescale_channels(sd, layer, ks)
    return sd


def test_rescale_channels_is_exact_and_touches_what_it_should():
    args, sd = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa_tts.tar"))
    for layer in range(1, 7):
        for ks in exponent_vectors(_channels(sd, layer), layer):
            fwd = rescale_channels(sd, layer, ks)
            back = rescale_channels(fwd, layer, -ks)
            assert all(np.array_equal(back[k].numpy(), sd[k].numpy()) for k in sd)
            changed = sorted(k for k in sd if not np.array_equal(fwd[k].numpy(), sd[k].numpy()))
            consumer = "cnn.model.conv%d.weight" % (layer + 1) if layer < 6 else "cnn.model.fc_out.weight"
            assert changed == sorted(["cnn.model.bn%d.weight" % layer, "cnn.model.bn%d.bias" % layer, consumer]), changed
    # layer 6: feature c * hw + pos of fc_out (64 channels x 6 x 2 positions) divided by 2^ks[c]
    ks = np.arange(64) % 7 - 3
    w = rescale_channels(sd, 6, ks)["cnn.model.fc_out.weight"].double()
    want = sd["cnn.model.fc_out.weight"].double().numpy() * np.ldexp(1.0, -np.repeat(ks, 12))[None, :]
    assert np.array_equal(w.numpy(), want)


def _oracle_scores(name, args, sd, spec):
    if name in SHIPPED:
        return O.forward_from_mel(args, sd, spec)
    with WV.wide_cnn():
        return TO.forward_from_mel(args, sd, spec)


@pytest.mark.parametrize("name", SHIPPED + list(VARIANTS))
def test_oracle_scores_are_bit_identical_under_channel_rescaling(name):
    args, sd = _checkpoint(name)
    spec = O.mel_db(synth.synth_speech_f32(77, 2.0, SR), SR, args)
    base = _oracle_scores(name, args, sd, spec)
    for layer in range(1, 7):
        for ks in exponent_vectors(_channels(sd, layer), layer):
            got = _oracle_scores(name, args, rescale_channels(sd, layer, ks), spec)
            np.testing.assert_array_equal(got, base, err_msg=str((layer, ks.tolist())))


# ------------------------------------------------------------------------------------------------------------ GPU
PATHS = {"tc_fused": (1, 1), "tc_separate": (1, 0), "ffma": (0, 0)}      # (conv_tc, conv12)


def _clips(name):
    """(pcm clips, rates, float32 oracle scores): three clips, or for NISQA_DE three (degraded, reference) pairs"""
    args, sd = _checkpoint(name)
    if name == DE_VARIANT:
        clips, srs, ref = [], [], []
        for pair in DV.DE_ARCH_PAIRS[:3]:
            deg, srd, r, srr = de_pair_pcm(pair)
            clips += [deg, r]
            srs += [srd, srr]
            ref.append(DO.predict_pcm_de(args, sd, deg.astype(np.float32) / np.float32(32768.0), srd,
                                         r.astype(np.float32) / np.float32(32768.0), srr)[0])
        return clips, srs, np.stack(ref)
    clips = [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in ((81, 2.0, SR), (82, 0.15, SR), (83, 4.3, 48000))]
    srs = [SR, SR, 48000]
    ref = []
    for c, sr in zip(clips, srs):
        y = c.astype(np.float32) / np.float32(32768.0)
        if name in SHIPPED:
            ref.append(O.predict_pcm(args, sd, y, sr)[0])
        else:
            with WV.wide_cnn():
                ref.append(TO.predict_pcm(args, sd, y, sr)[0])
    return clips, srs, np.stack(ref)


def _check_bit_identity(name, paths):
    from nisqa_b200 import engine as E
    args, sd = _checkpoint(name)
    clips, srs, ref = _clips(name)
    scored = slice(0, None, 2) if name == DE_VARIANT else slice(None)
    eng = E.Engine(E.config_from_args(args), 0)
    worst = 0.0
    try:
        for path in paths:
            tc, c12 = PATHS[path]
            eng.set_option("conv_tc", tc)
            eng.set_option("conv12", c12)
            eng.load_state_dict(sd)
            base, _, st = eng.predict_pcm(clips, srs)
            assert np.all(st == 0)
            base = base[scored]
            assert np.abs(base - ref).max() <= TOL, (path, float(np.abs(base - ref).max()))
            for layer in range(1, 7):
                for ks in exponent_vectors(_channels(sd, layer), layer):
                    eng.load_state_dict(rescale_channels(sd, layer, ks))
                    got, _, st = eng.predict_pcm(clips, srs)
                    assert np.all(st == 0)
                    got = got[scored]
                    worst = max(worst, float(np.abs(got - ref).max()))
                    np.testing.assert_array_equal(got, base, err_msg="%s %s bn%d x 2^%s" % (name, path, layer, ks.tolist()))
    finally:
        eng.close()
    print("\n%s %s: max |score - oracle| under channel rescaling %.3g" % (name, "/".join(paths), worst))
    assert worst <= TOL


@pytest.mark.gpu
@pytest.mark.parametrize("ckpt", SHIPPED)
def test_engine_scores_are_bit_identical_under_channel_rescaling(built_lib, ckpt):
    _check_bit_identity(ckpt, list(PATHS))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VARIANTS) + [DE_VARIANT])
def test_variant_scores_are_bit_identical_under_channel_rescaling(built_lib, name):
    _check_bit_identity(name, ["tc_fused"])


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("spread", [12, 24])
@pytest.mark.parametrize("ckpt", SHIPPED)
def test_every_stage_against_float64_under_channel_rescaling(built_lib, ckpt, spread, path):
    """tests/test_gpu_layers.py's stage checks, from the engine's own dumps, on a checkpoint whose every BatchNorm is
    rescaled channel by channel; the batches of 1..12 segments leave every remainder of the last tile of every layer"""
    import test_gpu_layers as L
    from nisqa_b200 import engine as E
    args, sd = _checkpoint(ckpt)
    sd = rescale_every_layer(sd, spread, seed=spread)
    eng = E.Engine(E.config_from_args(args), 0)
    ratios = L.Ratios()
    try:
        tc, c12 = PATHS[path]
        eng.set_option("conv_tc", tc)
        eng.set_option("conv12", c12)
        eng.set_option("keep_td_out", 1)
        eng.load_state_dict(sd)
        for n_seg in range(1, 13):
            L._check_call(eng, args, sd, path, [n_seg], 1000 * n_seg, ratios)
    finally:
        eng.close()
    print("\n%s 2^+-%d %s max |got - ref| / bound: %s" % (ckpt, spread, path, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios
