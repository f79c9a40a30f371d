"""CPU-side checks of the C-ABI boundary: the library builds for sm_90a, loads, exports every
symbol include/nisqa_b200.h declares, its pure-host entry points agree with the oracle, and the
product path fails loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT, WEIGHTS
from nisqa_b200 import engine as E
from oracle import nisqa_oracle as O


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "nisqa_b200.h")).read()
    return sorted(set(re.findall(r"NISQA_API[^;(]*?\b(nisqa_\w+)\s*\(", txt)))


def test_library_exports_every_declared_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    names = _declared_symbols()
    assert len(names) >= 16
    for n in names:
        assert hasattr(lib, n), "missing export " + n
    assert sorted(E.EXPORTS) == names          # the ctypes binding covers the whole header


def test_struct_layout_matches_header(tmp_path):
    """The ctypes structs mirror the C structs: sizes and offsets printed by a gcc-compiled
    program that includes the header."""
    import subprocess
    src = tmp_path / "layout.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "nisqa_b200.h"\n'
        'int main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(nisqa_config), offsetof(nisqa_config, hop_s),'
        ' offsetof(nisqa_config, fmax), offsetof(nisqa_config, max_chunk_segments), sizeof(nisqa_tensor),'
        ' offsetof(nisqa_tensor, ndim), offsetof(nisqa_tensor, dims), offsetof(nisqa_config, double_ended),'
        ' offsetof(nisqa_config, td2_pos_enc));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    got = [ctypes.sizeof(E.NisqaConfig), E.NisqaConfig.hop_s.offset, E.NisqaConfig.fmax.offset,
           E.NisqaConfig.max_chunk_segments.offset, ctypes.sizeof(E.NisqaTensor),
           E.NisqaTensor.ndim.offset, E.NisqaTensor.dims.offset, E.NisqaConfig.double_ended.offset,
           E.NisqaConfig.td2_pos_enc.offset]
    assert [int(x) for x in out] == got


@pytest.mark.parametrize("ckpt", ["nisqa.tar", "nisqa_tts.tar"])
def test_segment_counts_bit_exact_vs_oracle(built_lib, ckpt):
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, ckpt))
    cfg = E.config_from_args(args)
    rng = np.random.default_rng(0)
    rates = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000]
    for sr in rates:
        lens = list(rng.integers(1, 60 * sr, size=40)) + [1, 13 * int(sr * 0.01), 14 * int(sr * 0.01),
                                                           14 * int(sr * 0.01) - 1, 10 * sr, 52 * sr, 53 * sr]
        for n in lens:
            got = E.segment_counts(cfg, int(n), sr)
            ref = O.segment_counts(int(n), sr, args)
            if ref[2] == O.STATUS_TOO_SHORT:
                assert got[2] == E.CLIP_TOO_SHORT
            else:
                assert got == ref, (sr, n, got, ref)


def test_config_refuses_unknown_architectures():
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    for k, v in (("pool", "last_step_bi"), ("pool_att_h", 64), ("td", "lstm"), ("cnn_model", "resnet"), ("model", "NISQA_DE"),
                 ("td_sa_nhead", 4), ("cnn_fc_out_h", 100), ("td_2", "lstm"), ("cnn_c_out_1", 8)):
        bad = dict(args); bad[k] = v
        with pytest.raises(NotImplementedError):
            E.config_from_args(bad)
    # ms_sr is an ingest parameter (clips are converted to that rate before the engine sees them, 8f.2)
    assert E.config_from_args(dict(args, ms_sr=16000)).n_out == 5
    # the other pooling modules and the positional encoding are implemented (SURVEY.md 8f.4)
    assert E.config_from_args(dict(args, pool="avg")).pool == E.POOL_AVG
    assert E.config_from_args(dict(args, pool="att", pool_att_h=None, td_sa_pos_enc=True)).pos_enc == 1
    # ... and so are the framewise models without convolutions, td_2 and the double-ended model
    c = E.config_from_args(dict(args, cnn_model="dff", cnn_fc_out_h=None))
    assert (c.cnn_kind, c.cnn_fc) == (E.CNN_DFF, 4096)
    assert E.config_from_args(dict(args, cnn_model="skip", cnn_fc_out_h=None)).cnn_kind == E.CNN_SKIP
    de = dict(args, model="NISQA_DE", td_2="self_att", td_2_sa_d_model=64, td_2_sa_nhead=1, td_2_sa_h=64, td_2_sa_num_layers=2,
              de_align="bahd", de_align_apply="soft", de_fuse="x/y/-", de_fuse_dim=None)
    c = E.config_from_args(de)
    assert (c.double_ended, c.de_align, c.td2_layers, c.n_out) == (1, 5, 2, 1)
    assert E.config_from_args(dict(de, de_fuse_dim=64)).de_fuse_dim == 64
    assert E.config_from_args(dict(args, cnn_fc_out_h=128)).cnn_fc == 128         # AdaptCNN's optional Linear
    for k, v in (("de_align", "none"), ("de_fuse_dim", 100), ("td_2", "skip")):
        with pytest.raises(NotImplementedError):
            E.config_from_args(dict(de, **{k: v}))


def test_no_cpu_fallback(built_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for the GPU-less container")
    args, _ = O.load_checkpoint(os.path.join(WEIGHTS, "nisqa.tar"))
    with pytest.raises(E.EngineError):
        E.Engine(E.config_from_args(args), 0)
    from nisqa_b200.NISQA_model import nisqaModel
    with pytest.raises(RuntimeError):
        nisqaModel({"mode": "predict_file", "pretrained_model": os.path.join(WEIGHTS, "nisqa.tar"),
                    "deg": "x.wav", "output_dir": None, "tr_bs_val": 1, "tr_num_workers": 0, "ms_channel": None})


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "nisqa_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f
    assert "oracle" not in open(os.path.join(ROOT, "run_predict.py")).read()
