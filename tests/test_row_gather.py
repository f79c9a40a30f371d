"""The gathered GEMM rows of the tensor-core conv kernels (csrc/conv_split.cu): GEMM row m of a tile is the m-th
interior output position of the tile's segments in (segment, h, w) order (conv6 of the AdaptCNN: the centre column
only), and its nine taps are read around that position's plane row.  SpCfg::gemm_row is restated here and checked
for every SpCfg instance declared in csrc/conv_split.cuh:

  * the kept rows hit every output position of a tile's live segments exactly once, so every staging row the
    epilogue's store reads has been written (full and short last tiles),
  * every tap of every GEMM row, the rows past the kept ones included, stays inside the AROWS copied rows,
  * on the NumPy plane emulation of tests/test_plane_layout.py, the gathered GEMM gives exactly the full 256-row
    GEMM's values at the kept rows.

No GPU: the kernels' results on the device are tests/test_gpu_layers.py's and test_conv_paths_agree's job.
"""
import os
import re

import numpy as np
import pytest

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


class Rows(object):
    """SpCfg's GEMM-row map (conv_split.cuh) on the geometry of one instance."""

    def __init__(self, H, W, CIN, center):
        self.g = Geom(H, W, CIN)
        self.center = center
        self.KW = 1 if center else W
        self.SEG_ROWS = H * self.KW
        self.KEPT = self.g.G * self.SEG_ROWS
        self.NBLK = (self.KEPT + 63) // 64

    def gemm_row(self, m):
        if m >= self.KEPT:
            return 0
        s, q = divmod(m, self.SEG_ROWS)
        h, w = divmod(q, self.KW)
        return s * self.g.BLK + (h + 1) * self.g.P + (2 if self.center else w + 1)


def test_every_instance_is_found():
    assert set(INSTANCES) == {"SpConv%d%s" % (i, k) for i in range(2, 7) for k in "AS"}
    # the m64 blocks a tile issues: three everywhere, one for the centre-column conv6 of the AdaptCNN
    assert {n: Rows(H, W, CIN, c).NBLK for n, (H, W, CIN, _, c) in INSTANCES.items()} == \
        {n: (1 if n == "SpConv6A" else 3) for n in INSTANCES}


@pytest.mark.parametrize("name", sorted(INSTANCES))
def test_kept_rows_cover_every_output_position_once(name):
    H, W, CIN, _, center = INSTANCES[name]
    R = Rows(H, W, CIN, center)
    g = R.g
    for live in range(1, g.G + 1):                   # segments of the tile below n_seg: short last tiles too
        staged = [R.gemm_row(m) for m in range(64 * R.NBLK) if m < R.KEPT and m // R.SEG_ROWS < live]
        cols = [1] if center else range(W)           # conv6A: only the centre column is read by the store
        want = [s * g.BLK + (h + 1) * g.P + (w + 1) for s in range(live) for h in range(H) for w in cols]
        assert sorted(staged) == sorted(want) and len(set(staged)) == len(staged)


@pytest.mark.parametrize("name", sorted(INSTANCES))
def test_every_tap_stays_inside_the_copied_rows(name):
    H, W, CIN, _, center = INSTANCES[name]
    R = Rows(H, W, CIN, center)
    g = R.g
    offs = [(t // 3 - 1) * g.P + (t % 3 - 1) for t in range(9)]
    for m in range(256):                             # conv12_kernel runs all four blocks of conv2
        for off in offs:
            assert 0 <= g.HALO + R.gemm_row(m) + off < g.AROWS, (m, off)


@pytest.mark.parametrize("name", sorted(INSTANCES))
def test_gathered_gemm_equals_the_full_gemm_at_the_kept_rows(name):
    H, W, CIN, COUT, center = INSTANCES[name]
    R = Rows(H, W, CIN, center)
    g = R.g
    rng = np.random.default_rng(H * 1000 + W * 10 + CIN)
    n_seg = g.G + 1                                  # the second tile holds one segment
    # small integers: every product and sum is exact in float64, so the two GEMMs must agree bit for bit
    x = rng.integers(0, 9, (n_seg, H, W, CIN)).astype(np.float32)
    wgt = rng.integers(-4, 5, (COUT, CIN, 3, 3)).astype(np.float64)
    hi_p, lo_p = pack_planes(x, g)
    for seg0 in range(0, n_seg, g.G):
        X = tile_matrix(hi_p, lo_p, g, seg0)
        full = implicit_gemm(X, wgt, g)              # D[n] for tile rows n = 0..255
        rows = np.array([g.HALO + R.gemm_row(m) for m in range(64 * R.NBLK)])
        gathered = np.zeros((64 * R.NBLK, COUT))
        for t in range(9):
            off = (t // 3 - 1) * g.P + (t % 3 - 1)
            gathered += X[rows + off] @ wgt[:, :, t // 3, t % 3].T
        kept = [R.gemm_row(m) for m in range(R.KEPT)]
        np.testing.assert_array_equal(gathered[:R.KEPT], full[kept])
        live = min(g.G, n_seg - seg0)
        for m in range(R.KEPT):
            s, q = divmod(m, R.SEG_ROWS)
            h, w = divmod(q, R.KW)
            if s < live:                             # the planes hold x: the GEMM is the conv of x at (h, w)
                xs = np.pad(x[seg0 + s].astype(np.float64), ((1, 1), (1, 1), (0, 0)))
                wc = 1 if center else w
                want = np.einsum("yxc,ocyx->o", xs[h:h + 3, wc:wc + 3], wgt)
                np.testing.assert_array_equal(gathered[m], want)
