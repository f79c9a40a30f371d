"""Quality embeddings: nisqa_predict_device_batch_embeddings, Scorer.embed and run_predict.py --embeddings.  CPU part:
the golden of the unmodified reference modules (oracle/make_embedding_golden.py) against the checkpoints' last Linears
and against the rows and weights of tests/golden/segments.npz, the ABI, and the CLI refusals.  GPU part: every golden
variant, the kernel's arithmetic on long clips against float64, ragged and multi-pass batches, NISQA_DE, the stream
contract, the too-small-buffer refusal and the CLI."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, WEIGHTS
from nisqa_b200 import engine as E
from nisqa_b200 import synth, wav
from nisqa_b200.scorer import Scorer
from oracle import segment_variants as SV
from oracle import variants as V

gpu = pytest.mark.gpu
WEIGHTED = ("att", "avg")          # pooled = sum_t a_t x_t with the segments call's weights


def _golden():
    return np.load(os.path.join(GOLDEN, "embeddings.npz"))


def _segments():
    return np.load(os.path.join(GOLDEN, "segments.npz"))


def _seg_rows(z, name):
    return z[name + "/x"] if name + "/x" in z.files else z[str(z[name + "/x_from"]) + "/x"]


def _head_params(args, sd):
    """each head's pooling tensors as float64 numpy: [(last Linear w [D], b, attention logit function or None)]"""
    n = 5 if args["model"] == "NISQA_DIM" else 1
    pool, att_h = args["pool"], args.get("pool_att_h")
    out = []
    for h in range(n):
        p = "pool_layers.%d.model." % h if n == 5 else "pool.model."
        t = lambda k: sd[p + k].double().numpy()         # noqa: E731
        if pool == "att" and att_h:
            w1, b1, w2, b2 = t("linear1.weight"), t("linear1.bias"), t("linear2.weight")[0], t("linear2.bias")[0]
            out.append((t("linear3.weight")[0], t("linear3.bias")[0],
                        lambda x, w1=w1, b1=b1, w2=w2, b2=b2: np.maximum(x @ w1.T + b1, 0) @ w2 + b2))
        elif pool == "att":
            a1, a1b = t("linear1.weight")[0], t("linear1.bias")[0]
            out.append((t("linear2.weight")[0], t("linear2.bias")[0], lambda x, a1=a1, a1b=a1b: x @ a1 + a1b))
        else:
            out.append((t("linear.weight")[0], t("linear.bias")[0], None))
    return out


def _pool64(args, heads, x):
    """float64 pooled vectors [n_heads, D] of one clip's rows x [S, D] and the scale each element's error is relative to"""
    x = x.astype(np.float64)
    pool, out, scale = args["pool"], [], []
    for _, _, logit in heads:
        if pool == "att":
            l = logit(x)
            a = np.exp(l - l.max())
            a /= a.sum()
            out.append(a @ x)
            scale.append(a @ np.abs(x))
        elif pool == "avg":
            out.append(x.sum(0) / x.shape[0])
            scale.append(np.abs(x).sum(0) / x.shape[0])
        elif pool == "max":
            out.append(x.max(0))
        elif pool == "last_step":
            out.append(x[-1])
        else:
            half = x.shape[1] // 2
            out.append(np.concatenate([x[-1, :half], x[0, half:]]))
        if pool not in WEIGHTED:
            scale.append(np.abs(out[-1]))
    return np.stack(out), np.stack(scale)


def _scorer(name, tmp_path, **over):
    args, sd = SV.segment_checkpoint(name, WEIGHTS)
    path = os.path.join(str(tmp_path), name + ".tar")
    torch.save({"args": dict(args, **over), "model_state_dict": sd}, path)
    return Scorer(path), args, sd


def _pcm(args):
    if args["model"] == "NISQA_DE":
        pairs = [V.de_pair_pcm(p) for p in SV.SEGMENT_DE_PAIRS]
        return [p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs], [p[3] for p in pairs]
    return [synth.synth_speech_pcm16(s, sec, sr) for s, sec, sr in SV.SEGMENT_CLIPS], [c[2] for c in SV.SEGMENT_CLIPS], None, None


def _padded(clips):
    T = max(c.shape[0] for c in clips)
    x = np.zeros((len(clips), T), np.int16)
    for i, c in enumerate(clips):
        x[i, :c.shape[0]] = c
    return torch.from_numpy(x).cuda(), [c.shape[0] for c in clips]


# ------------------------------------------------------------------ CPU
def test_golden_pooled_through_the_last_linear_is_the_score():
    z = _golden()
    for name in SV.SEGMENT_VARIANTS:
        args, sd = SV.segment_checkpoint(name, WEIGHTS)
        pooled, scores = z[name + "/pooled"].astype(np.float64), z[name + "/scores"]
        heads = _head_params(args, sd)
        assert pooled.shape[:2] == scores.shape == (len(scores), len(heads)), name
        got = np.stack([pooled[:, h] @ w + b for h, (w, b, _) in enumerate(heads)], axis=1)
        np.testing.assert_allclose(got, scores, atol=1e-5, rtol=0, err_msg=name)
        np.testing.assert_array_equal(scores, _segments()[name + "/scores"])


def test_golden_ties_to_the_segment_rows_and_weights():
    z, s = _golden(), _segments()
    seen = set()
    for name in SV.SEGMENT_VARIANTS:
        args, _ = SV.segment_checkpoint(name, WEIGHTS)
        x, counts, w = _seg_rows(s, name).astype(np.float64), s[name + "/counts"], s[name + "/seg_weights"]
        pooled = z[name + "/pooled"]
        assert pooled.shape == (len(counts), w.shape[1], x.shape[1]), name
        seen.add(args["pool"])
        r = 0
        for b, n in enumerate(counts):
            xb = x[r:r + n]
            for h in range(w.shape[1]):
                if args["pool"] in WEIGHTED:
                    np.testing.assert_allclose(w[r:r + n, h] @ xb, pooled[b, h], atol=1e-5, rtol=0, err_msg=name)
                else:
                    want = {"max": xb.max(0), "last_step": xb[-1],
                            "last_step_bi": np.concatenate([xb[-1, :xb.shape[1] // 2], xb[0, xb.shape[1] // 2:]])}
                    np.testing.assert_array_equal(pooled[b, h], want[args["pool"]].astype(np.float32), err_msg=name)
            r += n
    assert seen == {"att", "avg", "max", "last_step", "last_step_bi"}


def test_embedding_out_struct_header_and_exports(tmp_path, built_lib):
    src = tmp_path / "layout.c"
    fields = ["pooled", "rows", "n_rows"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nisqa_b200.h"\nint main(void){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(nisqa_embedding_out)'
                   + "".join(", offsetof(nisqa_embedding_out, %s)" % f for f in fields) + ");return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [ctypes.sizeof(E.NisqaEmbeddingOut)] + [getattr(E.NisqaEmbeddingOut, f).offset for f in fields]
    header = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    lib = E.load_library()
    for sym in ("nisqa_embedding_width", "nisqa_predict_device_batch_embeddings"):
        assert sym + "(" in header and sym in E.EXPORTS and hasattr(lib, sym)


def test_embeddings_refused_under_torchrun(monkeypatch):
    from nisqa_b200.NISQA_model import nisqaModel
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("LOCAL_RANK", "0")
    with pytest.raises(ValueError, match="embeddings"):
        nisqaModel({"mode": "predict_csv", "embeddings": True, "csv_file": "/nonexistent.csv"})


def test_embeddings_refused_in_windows_mode():
    from nisqa_b200.NISQA_model import nisqaModel
    with pytest.raises(ValueError, match="embeddings"):
        nisqaModel({"mode": "predict_csv", "embeddings": True, "window_s": 10.0, "window_hop_s": 1.0,
                    "csv_file": "/nonexistent.csv"})


# ------------------------------------------------------------------ GPU
@gpu
@pytest.mark.parametrize("name", list(SV.SEGMENT_VARIANTS))
def test_every_golden_variant(built_lib, tmp_path, name):
    z, s = _golden(), _segments()
    sc, args, sd = _scorer(name, tmp_path)
    heads = _head_params(args, sd)
    deg, srs, ref, ref_srs = _pcm(args)
    want_x = _seg_rows(s, name)
    tol = 1e-4 * max(1.0, float(np.abs(want_x).max()))
    got_p, got_x, counts = [], [], []
    for i in range(len(deg)):          # (the clips have different rates: one call each)
        x, lens = _padded([deg[i]])
        kw = {}
        if ref is not None:
            kw["reference"], kw["reference_lengths"] = _padded([ref[i]])
            kw["reference_sample_rate"] = ref_srs[i]
        res = sc.embed(x, srs[i], lengths=lens, rows=True, **kw)
        plain = sc(x, srs[i], lengths=lens, **kw)
        torch.cuda.synchronize()
        scores = res.scores.cpu().numpy()
        np.testing.assert_array_equal(scores, plain.cpu().numpy())
        p = res.pooled.cpu().numpy()
        assert p.shape == (1, len(sc.columns), sc.engine.embedding_width())
        lin = np.stack([p[:, h].astype(np.float64) @ w + b for h, (w, b, _) in enumerate(heads)], axis=1)
        np.testing.assert_allclose(lin, scores, atol=2e-5, rtol=0)
        got_p.append(p)
        got_x.append(res.rows.cpu().numpy())
        counts += res.counts
    assert counts == s[name + "/counts"].tolist()
    np.testing.assert_allclose(np.concatenate(got_p), z[name + "/pooled"], atol=tol, rtol=0)
    np.testing.assert_allclose(np.concatenate(got_x), want_x, atol=tol, rtol=0)
    sc.close()


def _ragged_case(sc, n_segs=(1, 63, 64, 65, 97, 1300)):
    """clips of n_segs segments, each beside a long clip (48 kHz)"""
    from test_device_batch import _len_for_segments
    lens = []
    for n in n_segs:
        lens += [48000 * 7 + 11, _len_for_segments(sc.cfg, n, 48000)]
    x = np.zeros((len(lens), max(lens)), np.int16)
    for i, n in enumerate(lens):
        x[i, :n] = synth.synth_speech_pcm16(1600 + i, n / 48000.0 + 0.01, 48000)[:n]
    return torch.from_numpy(x).cuda(), lens


@gpu
@pytest.mark.parametrize("name", ["nisqa", "dim_pool_att", "dim_pool_avg", "dim_pool_max", "dim_pool_last_step", "tts",
                                  "mos_adapt_skip_attff"])
def test_long_clips_against_float64(built_lib, tmp_path, name):
    """pooled recomputed in float64 from the call's own rows and the module's weights"""
    sc, args, sd = _scorer(name, tmp_path)
    heads = _head_params(args, sd)
    x, lens = _ragged_case(sc)
    res = sc.embed(x, 48000, lengths=lens, rows=True)
    torch.cuda.synchronize()
    pooled, rows = res.pooled.cpu().numpy(), res.rows.cpu().numpy()
    assert sorted(set(res.counts)) == sorted({E.segment_counts(sc.cfg, 48000 * 7 + 11, 48000)[1], 1, 63, 64, 65, 97, 1300})
    r = 0
    for b, n in enumerate(res.counts):
        want, scale = _pool64(args, heads, rows[r:r + n])
        if args["pool"] in WEIGHTED:
            assert np.all(np.abs(pooled[b] - want) <= 1e-5 * scale + 1e-30), (name, n)
        else:
            np.testing.assert_array_equal(pooled[b], want.astype(np.float32))
        r += n
    assert r == rows.shape[0]
    sc.close()


@gpu
@pytest.mark.parametrize("ckpt", ["nisqa.tar", "nisqa_tts.tar"])
def test_ragged_multi_pass_and_alone_are_bit_identical(built_lib, ckpt):
    sc = Scorer(os.path.join(WEIGHTS, ckpt))
    small = Scorer(os.path.join(WEIGHTS, ckpt), b200_max_chunk_segments=700)
    x, lens = _ragged_case(sc, (1, 1300))
    one = sc.embed(x, 48000, lengths=lens, rows=True)
    many = small.embed(x, 48000, lengths=lens, rows=True)
    torch.cuda.synchronize()
    assert small.engine.lib.nisqa_stage_dump(small.engine.h, E.STAGE_MEL_DB, None, 0) < 0    # (it really ran in passes)
    for a, b in ((one.scores, many.scores), (one.pooled, many.pooled), (one.rows, many.rows)):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    r = 0
    for i, n in enumerate(one.counts):
        alone = sc.embed(x[i:i + 1], 48000, lengths=[lens[i]], rows=True)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(alone.pooled.cpu().numpy(), one.pooled[i:i + 1].cpu().numpy())
        np.testing.assert_array_equal(alone.rows.cpu().numpy(), one.rows[r:r + n].cpu().numpy())
        np.testing.assert_array_equal(alone.scores.cpu().numpy(), one.scores[i:i + 1].cpu().numpy())
        r += n
    without = sc.embed(x, 48000, lengths=lens)
    torch.cuda.synchronize()
    assert without.rows is None
    np.testing.assert_array_equal(without.pooled.cpu().numpy(), one.pooled.cpu().numpy())
    sc.close()
    small.close()


@gpu
def test_tts_plain_call_unchanged_by_an_embeddings_call(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa_tts.tar"))
    x = torch.from_numpy(np.stack([synth.synth_speech_pcm16(1650 + i, 3.0, 16000) for i in range(3)])).cuda()
    before = sc(x, 16000).cpu().numpy()
    sc.embed(x, 16000, rows=True)
    after = sc(x, 16000).cpu().numpy()
    np.testing.assert_array_equal(before, after)
    with pytest.raises(E.EngineError, match="keep_td_out"):     # the option itself is unchanged
        sc.engine.stage_dump(E.STAGE_TD_OUT)
    sc.close()


@gpu
def test_double_ended_rows_and_unusable_reference(built_lib, tmp_path):
    sc, args, _ = _scorer("de_cosine_hard", tmp_path)
    deg, srs, ref, ref_srs = _pcm(args)
    x, lens = _padded([deg[0], deg[0][:24000]])
    r, rlens = _padded([ref[0], ref[0]])
    res = sc.embed(x, srs[0], lengths=lens, reference=r, reference_lengths=rlens, reference_sample_rate=ref_srs[0],
                   rows=True)
    torch.cuda.synchronize()
    n_deg = [E.segment_counts(sc.cfg, n, srs[0])[1] for n in lens]
    assert res.counts == n_deg and res.rows.shape[0] == sum(n_deg) and res.pooled.shape[0] == 2
    assert np.isfinite(res.pooled.cpu().numpy()).all() and np.isfinite(res.rows.cpu().numpy()).all()
    # a pair whose reference is too short scores NaN: NaN pooled vectors and NaN rows (the engine call: Scorer refuses it)
    short = E.segment_counts(sc.cfg, 100, ref_srs[0])[2]
    assert short != E.CLIP_OK
    rlens2 = [rlens[0], 100]
    deg_b = E.device_batch(x.data_ptr(), E.FMT_S16, lens, 1, -1, x.shape[1], x.stride(0), 0, srs[0])
    ref_b = E.device_batch(r.data_ptr(), E.FMT_S16, rlens2, 1, -1, r.shape[1], r.stride(0), 0, ref_srs[0])
    W = sc.engine.embedding_width()
    scores = torch.empty((4, 1), device="cuda")
    pooled = torch.empty((4, 1, W), device="cuda")
    rows = torch.empty((sum(n_deg), W), device="cuda")
    sc.engine.predict_device_batch_embeddings(torch.cuda.current_stream().cuda_stream, deg_b, scores.data_ptr(),
                                              pooled.data_ptr(), rows.data_ptr(), rows.shape[0], ref=ref_b)
    torch.cuda.synchronize()
    p, rw = pooled.cpu().numpy(), rows.cpu().numpy()
    np.testing.assert_array_equal(p[0], res.pooled.cpu().numpy()[0])
    np.testing.assert_array_equal(rw[:n_deg[0]], res.rows.cpu().numpy()[:n_deg[0]])
    assert np.isnan(p[1]).all() and np.isnan(p[2]).all() and np.isnan(p[3]).all()
    assert np.isnan(rw[n_deg[0]:]).all() and np.isnan(scores.cpu().numpy()[2, 0])
    sc.close()


@gpu
def test_embeddings_call_does_not_wait_and_input_frees_in_stream_order(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    B, T = 3, 48000 * 4
    src = torch.from_numpy(np.stack([synth.synth_speech_pcm16(1660 + i, 4.0, 48000)[:T] for i in range(B)])).cuda()
    want = sc.embed(src, 48000, rows=True)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)
    got = sc.embed(src, 48000, rows=True)
    assert not torch.cuda.current_stream().query()          # returned while the stream still sleeps
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.pooled.cpu().numpy(), want.pooled.cpu().numpy())
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        x = torch.empty_like(src)
        x.copy_(src)
        got = sc.embed(x, 48000, rows=True)
        del x
        junk = [torch.full((B, T), 7, dtype=torch.int16, device="cuda") for _ in range(3)]
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.pooled.cpu().numpy(), want.pooled.cpu().numpy())
    np.testing.assert_array_equal(got.rows.cpu().numpy(), want.rows.cpu().numpy())
    del junk
    sc.close()


@gpu
def test_bad_outputs_are_refused_before_anything_is_enqueued(built_lib):
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    x = torch.from_numpy(np.stack([synth.synth_speech_pcm16(1670 + i, 2.0, 48000) for i in range(2)])).cuda()
    res = sc.embed(x, 48000, rows=True)
    torch.cuda.synchronize()
    n = sum(res.counts)
    deg = E.device_batch(x.data_ptr(), E.FMT_S16, [x.shape[1]] * 2, 1, -1, x.shape[1], x.stride(0), 0, 48000)
    st = torch.cuda.current_stream().cuda_stream
    before = sc.engine.kernel_launches()
    with pytest.raises(E.EngineError, match="n_rows"):
        sc.engine.predict_device_batch_embeddings(st, deg, res.scores.data_ptr(), res.pooled.data_ptr(),
                                                  res.rows.data_ptr(), n - 1)
    with pytest.raises(E.EngineError, match="pooled"):
        sc.engine.predict_device_batch_embeddings(st, deg, res.scores.data_ptr(), 0, res.rows.data_ptr(), n)
    assert sc.engine.kernel_launches() == before
    sc.close()


@gpu
def test_cli_writes_embeddings_npz_and_leaves_results_unchanged(built_lib, tmp_path):
    import run_predict
    from nisqa_b200.NISQA_model import nisqaModel
    d = tmp_path / "wavs"
    d.mkdir()
    for i, (sec, sr) in enumerate([(2.0, 48000), (1.1, 16000), (3.0, 48000)]):
        wav.write_wav_pcm16(str(d / ("c%d.wav" % i)), synth.synth_speech_pcm16(1680 + i, sec, sr), sr)
    outs = {}
    for emb in (False, True):
        o = tmp_path / ("out%d" % emb)
        o.mkdir()
        argv = ["--mode", "predict_dir", "--pretrained_model", os.path.join(WEIGHTS, "nisqa.tar"), "--data_dir", str(d),
                "--output_dir", str(o), "--bs", "2"] + (["--embeddings"] if emb else [])
        nisqaModel(run_predict.parse_args(argv)).predict()
        outs[emb] = o
    assert open(outs[False] / "NISQA_results.csv", "rb").read() == open(outs[True] / "NISQA_results.csv", "rb").read()
    assert not (outs[False] / "NISQA_embeddings.npz").exists()
    z = np.load(outs[True] / "NISQA_embeddings.npz")
    assert sorted(z.files) == ["files", "heads", "pooled"]
    assert z["heads"].tolist() == ["mos_pred", "noi_pred", "dis_pred", "col_pred", "loud_pred"]
    sc = Scorer(os.path.join(WEIGHTS, "nisqa.tar"))
    assert z["pooled"].dtype == np.float32 and z["pooled"].shape == (3, 5, sc.engine.embedding_width())
    for k, f in enumerate(z["files"].tolist()):
        y, sr = wav.read_wav(str(d / f), None)
        got = sc.embed(torch.from_numpy(y[None]).cuda(), sr).pooled.cpu().numpy()
        np.testing.assert_array_equal(z["pooled"][k], got[0])
    sc.close()
