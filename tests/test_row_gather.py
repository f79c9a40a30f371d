"""The gathered GEMM rows of the tensor-core conv kernels (csrc/conv_split.cu): GEMM row m of a tile is the m-th
interior output position of the tile's segments in (segment, h, w) order (conv6 of the AdaptCNN: one column), and its
taps are read around that position's plane row.  gemm_row (csrc/conv_split.cuh) is restated here and checked for every
SpCfg instance declared in csrc/conv_split.cuh and for the run-time geometries of the AdaptCNN pool variants
(oracle/cnn_pool_variants.py) and of the corners of the accepted pools:

  * the kept rows hit every output position of a tile's live segments exactly once, inside the 256-row staging tile,
    so every staging row the epilogue's store reads has been written (full and short last tiles),
  * every tap of every GEMM row, the rows past the kept ones included, stays inside the copied rows,
  * on the NumPy plane emulation of tests/test_plane_layout.py, the gathered GEMM gives exactly the conv's values at
    the kept rows (and, for 3 x 3 taps with padding 1, the full 256-row GEMM's).

No GPU: the kernels' results on the device are tests/test_gpu_layers.py's and test_conv_paths_agree's job.
"""
import os
import re

import numpy as np
import pytest

from oracle.cnn_pool_variants import CNN_POOL_VARIANTS, SHIPPED_POOLS
from test_plane_layout import Geom, implicit_gemm, pack_planes, tile_matrix

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nisqa_b200", "csrc", "conv_split.cuh")


def _instances():
    """name -> (H, W, CIN, COUT, CENTER) of every `using SpConvX = SpCfg<...>;` in conv_split.cuh."""
    src = open(HEADER).read()
    out = {}
    for name, args in re.findall(r"using\s+(SpConv\w+)\s*=\s*SpCfg<([^>]*)>;", src):
        a = [x.strip() for x in args.split(",")]
        H, W, CIN, COUT = (int(x) for x in a[:4])
        center = len(a) > 7 and a[7] == "true"
        out[name] = (H, W, CIN, COUT, center)
    return out


INSTANCES = _instances()


def _rt_maps():
    """(H, W, conv6) of every run-time geometry layer the pool variants run (launch_conv_split: an AdaptCNN layer whose
    input map or output pooling differs from the shipped), plus the corners of the accepted pools: w = 1 and w = 14,
    (h + 1) (w + 1) = 256, and pool_3 widths 1, 2 and 3."""
    maps = set()
    shipped = [v for hw in SHIPPED_POOLS for v in hw]
    for entry in CNN_POOL_VARIANTS.values():
        p = [v for hw in entry[4] for v in hw]
        for layer, k0, k1 in ((2, 0, 4), (3, 2, 4), (4, 2, 6), (5, 4, 6), (6, 4, 6)):
            if p[k0:k1] != shipped[k0:k1]:
                i = 0 if layer == 2 else 2 if layer <= 4 else 4
                maps.add((p[i], p[i + 1], layer == 6))
    for h, w in ((127, 1), (16, 14), (63, 3), (31, 7), (1, 1), (1, 14)):
        maps.add((h, w, False))
    for h, w in ((127, 1), (84, 2), (63, 3), (1, 1), (1, 2), (1, 3)):
        maps.add((h, w, True))
    return sorted(maps)


class Rows(object):
    """gemm_row (conv_split.cuh) on one layer's geometry: KW output columns per row from plane column X0, taps 3 x KX
    at row offsets (t // KX - 1) P + t % KX - PADX; `cols` are the output columns the layer computes."""

    def __init__(self, H, W, CIN, KW, X0, KX, PADX, cols):
        self.g = Geom(H, W, CIN)
        self.KW, self.X0, self.KX, self.PADX, self.cols = KW, X0, KX, PADX, list(cols)
        self.SEG_ROWS = H * KW
        self.KEPT = self.g.G * self.SEG_ROWS
        self.NBLK = (self.KEPT + 63) // 64

    def gemm_row(self, m):
        if m >= self.KEPT:
            return 0
        s, q = divmod(m, self.SEG_ROWS)
        h, w = divmod(q, self.KW)
        return s * self.g.BLK + (h + 1) * self.g.P + w + self.X0

    def taps(self):
        return [(t // self.KX, t % self.KX, (t // self.KX - 1) * self.g.P + (t % self.KX - self.PADX))
                for t in range(3 * self.KX)]


def _compile_time(name):
    H, W, CIN, _, center = INSTANCES[name]
    # conv6 of the AdaptCNN: the padded 3 x 3 conv evaluated at its centre column only
    return Rows(H, W, CIN, 1 if center else W, 2 if center else 1, 3, 1, [1] if center else range(W))


def _run_time(H, W, conv6):
    # conv6: kernel (3, W), padding (1, 0): one output column; conv2..conv5: 3 x 3, padding 1
    return Rows(H, W, 16, 1, 1, W, 0, [0]) if conv6 else Rows(H, W, 16, W, 1, 3, 1, range(W))


CASES = {n: (lambda n=n: _compile_time(n)) for n in INSTANCES}
CASES.update({"rt_conv%s_%dx%d" % ("6" if c6 else "2_5", H, W): (lambda a=(H, W, c6): _run_time(*a))
              for H, W, c6 in _rt_maps()})
COUT = {n: INSTANCES[n][3] for n in INSTANCES}


def test_every_instance_is_found():
    assert set(INSTANCES) == {"SpConv%d%s" % (i, k) for i in range(2, 7) for k in "AS"}
    # the m64 blocks a tile issues: three everywhere, one for the centre-column conv6 of the AdaptCNN
    assert {n: _compile_time(n).NBLK for n in INSTANCES} == {n: (1 if n == "SpConv6A" else 3) for n in INSTANCES}


@pytest.mark.parametrize("name", sorted(CASES))
def test_kept_rows_cover_every_output_position_once(name):
    R = CASES[name]()
    g = R.g
    for live in range(1, g.G + 1):                   # segments of the tile below n_seg: short last tiles too
        staged = [R.gemm_row(m) for m in range(64 * R.NBLK) if m < R.KEPT and m // R.SEG_ROWS < live]
        want = [s * g.BLK + (h + 1) * g.P + (c + 1) for s in range(live) for h in range(g.H) for c in R.cols]
        assert sorted(staged) == sorted(want) and len(set(staged)) == len(staged)
        assert max(staged) < 256                     # rows of the staging tile


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_tap_stays_inside_the_copied_rows(name):
    R = CASES[name]()
    g = R.g
    for m in range(256):                             # conv12_kernel runs all four blocks of conv2
        for _, _, off in R.taps():
            assert 0 <= g.HALO + R.gemm_row(m) + off < g.AROWS, (m, off)


@pytest.mark.parametrize("name", sorted(CASES))
def test_gathered_gemm_equals_the_full_gemm_at_the_kept_rows(name):
    R = CASES[name]()
    g = R.g
    H, W, CIN = g.H, g.W, g.C
    rng = np.random.default_rng(H * 1000 + W * 10 + CIN)
    n_seg = g.G + 1                                  # the second tile holds one segment
    # small integers: every product and sum is exact in float64, so the GEMMs and the conv must agree bit for bit
    x = rng.integers(0, 9, (n_seg, H, W, CIN)).astype(np.float32)
    wgt = rng.integers(-4, 5, (COUT.get(name, 16), CIN, 3, R.KX)).astype(np.float64)
    hi_p, lo_p = pack_planes(x, g)
    for seg0 in range(0, n_seg, g.G):
        X = tile_matrix(hi_p, lo_p, g, seg0)
        rows = np.array([g.HALO + R.gemm_row(m) for m in range(64 * R.NBLK)])
        gathered = np.zeros((64 * R.NBLK, wgt.shape[0]))
        for ky, kx, off in R.taps():
            gathered += X[rows + off] @ wgt[:, :, ky, kx].T
        kept = [R.gemm_row(m) for m in range(R.KEPT)]
        if R.KX == 3 and R.PADX == 1:
            full = implicit_gemm(X, wgt, g)          # D[n] for tile rows n = 0..255
            np.testing.assert_array_equal(gathered[:R.KEPT], full[kept])
        live = min(g.G, n_seg - seg0)
        for m in range(R.KEPT):
            s, q = divmod(m, R.SEG_ROWS)
            h, w = divmod(q, R.KW)
            if s < live:                             # the planes hold x: the GEMM is the conv of x at (h, cols[w])
                xs = np.pad(x[seg0 + s].astype(np.float64), ((1, 1), (R.PADX, R.PADX), (0, 0)))
                c = R.cols[w]
                want = np.einsum("yxc,ocyx->o", xs[h:h + 3, c:c + R.KX], wgt)
                np.testing.assert_array_equal(gathered[m], want)
