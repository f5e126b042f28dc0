"""The grid-index reference (tests/grid_index_reference.py) on the CPU: it reproduces the reference's hashgrid_naive golden and
the C oracle's hash grid, its corner rows stay inside their level for every (resolution, bitwidth) the host accepts, its bitmask
builders agree with a direct construction, and its prune rules agree with the golden of the reference class and with torch."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O

import grid_index_reference as GR
import octree_reference as OR

f32 = np.float32


def _coords(rng, n):
    c = rng.uniform(-1.0, 1.0, (n, 3)).astype(f32)
    c[:16] = np.sign(c[:16])                                           # corners / faces
    return c


def test_reference_reproduces_hashgrid_naive(golden_dir):
    """wisp.ops.grid.hashgrid_naive (the reference's pure-torch blend) at the golden's tolerance: the naive version clamps in
    float and blends in another order (ops/grid.py:16-75)."""
    g = np.load(os.path.join(golden_dir, "hashgrid_naive.npz"))
    res, bw = [int(r) for r in g["resolutions"]], int(g["codebook_bitwidth"])
    emu, cen, rad = GR.hashgrid_fwd(g["coords"], g["table"], res, bw)
    np.testing.assert_allclose(emu, g["feats"], atol=2e-6, rtol=1e-4)
    assert (np.abs(emu - cen) <= rad).all()


@pytest.mark.parametrize("bw,F,res", [(9, 2, [4, 7, 13, 24, 40]), (12, 4, [2, 8, 15, 16, 17, 32]), (14, 8, [16, 25, 26, 64]),
                                      (18, 6, [16, 63, 64, 65, 300])])
def test_reference_matches_oracle(bw, F, res):
    """The C oracle (wo_hashgrid_fwd / _bwd, the restatement of the reference kernel) bit for bit on the forward and inside the
    float64 interval on the backward; the corner rows are the oracle's."""
    rng = np.random.default_rng(bw)
    begin = GR.table_layout(res, bw)
    assert np.array_equal(begin, O.table_layout(res, bw))
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    coords = _coords(rng, 4000)
    ref, corners = O.hashgrid_fwd(coords, table, res, bw, return_corners=True)
    emu, cen, rad = GR.hashgrid_fwd(coords, table, res, bw)
    assert np.array_equal(emu.view(np.uint32), ref.view(np.uint32))
    assert (np.abs(emu.astype(np.float64) - cen) <= rad).all()
    for l, r in enumerate(res):
        rows, _ = GR.corners(coords, r, bw)
        assert np.array_equal(rows, corners[:, l])
    go = rng.standard_normal(ref.shape).astype(f32)
    go[::3] = 0.0
    gt = O.hashgrid_bwd(coords, go, table.shape[0], res, bw)
    c, r, k = GR.hashgrid_bwd(coords, go, np.zeros_like(table), res, bw)
    assert (np.abs(gt - c) <= r).all()
    assert (gt[k == 0] == 0).all()


def test_corner_rows_stay_inside_their_level():
    """Every (res, bitwidth) the host accepts (2 <= res < 2^20, 2^bitwidth a positive int32): the rows of the extreme cells (a
    coordinate at -inf, -1, 0, just below +1, +1, +inf and NaN on each axis) lie inside [0, min(res^3, 2^bw)).  Rows are monotone
    in the cell on dense levels and masked on hashed ones, so these cells bound every coordinate.  The unclamped arithmetic of the
    reference kernel leaves its level exactly on the dense levels with res >= 258 (bitwidth >= 25): fl(res - 1 - 1e-5) == res - 1
    there and the +1 corner of the last cell is row res on that axis."""
    ext = np.array([-np.inf, -1.0, 0.0, np.nextafter(f32(1), f32(0)), 1.0, np.inf, np.nan], f32)
    coords = np.stack(np.meshgrid(ext, ext, ext, indexing="ij"), -1).reshape(-1, 3)
    outside_before = set()
    for bw in range(0, 31):
        dense_max = max((r for r in range(2, 1024) if GR.is_dense(r, bw)), default=1)
        hashed = sorted({r for r in (dense_max + 1, dense_max + 2, 257, 258, 1023, 1024, 4096, (1 << 20) - 1) if r > dense_max})
        for res in list(range(2, dense_max + 1)) + hashed:
            n = GR.level_rows(res, bw)
            rows, cf = GR.corners(coords, res, bw)
            assert rows.min() >= 0 and rows.max() < n, (res, bw)
            old, cf_old = GR.corners(coords, res, bw, top_clamp=False)
            assert np.array_equal(cf, cf_old)
            if old.max() >= n:
                outside_before.add((res, bw))
                assert (cf[old != rows] == 0).all()                   # the moved corners carry no weight
    expected = {(r, bw) for bw in range(25, 31) for r in range(258, 1024) if GR.is_dense(r, bw)}
    assert outside_before == expected
    print(f"GRIDINDEX corner rows: {len(expected)} (res, bitwidth) pairs left their level before the clamp: res 258..1023 on "
          f"dense levels of bitwidth 25..30, e.g. {min(expected)}, {max(expected)}; none after")


def test_clamp_bound_rounds_to_res_minus_one_from_258():
    for res in range(2, 4096):
        assert (GR.clamp_hi(res) == res - 1) == (res >= 258), res


@pytest.mark.parametrize("name", ["lego6", "corner_lo4", "corner_hi5", "dense3", "checker4", "random8", "lines9", "faces5"])
def test_bitmask_builders(name):
    """The bit and coarse builders against a direct construction: set membership per cell and a brute-force 26-neighbourhood."""
    pts, level = OR.octree_points(name)
    bits = GR.build_bits(pts, level)
    n = 1 << level
    occ = np.zeros((n, n, n), bool)
    occ[pts[:, 0], pts[:, 1], pts[:, 2]] = True
    flat = np.unpackbits(bits.view(np.uint8), bitorder="little")[:n ** 3].astype(bool)
    assert np.array_equal(flat.reshape(n, n, n), occ)
    for cl in range(1, level):
        m = 1 << cl
        cocc = occ.reshape(m, n // m, m, n // m, m, n // m).any((1, 3, 5))
        want = np.zeros_like(cocc)
        for x, y, z in np.argwhere(cocc):
            want[max(x - 1, 0):x + 2, max(y - 1, 0):y + 2, max(z - 1, 0):z + 2] = True
        got = np.unpackbits(GR.build_coarse(pts, level, cl).view(np.uint8), bitorder="little")[:m ** 3].astype(bool)
        assert np.array_equal(got.reshape(m, m, m), want), cl


def test_prune_samples_and_update_reproduce_the_reference_class(golden_dir):
    """tests/golden/prune.npz: the probe points of the reference class's explicit u give the density the reference recorded
    (through the oracle), and the update rule gives its occupancy and surviving cells."""
    g = np.load(os.path.join(golden_dir, "prune.npz"))
    spc = O.octree_to_spc(g["octree"])
    level = int(g["level"])
    pts = spc.points[spc.pyramid[1, level]:spc.pyramid[1, level] + spc.pyramid[0, level]]
    s = GR.prune_samples(pts, level, g["u"])
    ref = ((torch.from_numpy(pts.astype(np.int64)).float() + torch.from_numpy(g["u"])) / 2.0 ** level) * 2.0 - 1.0
    assert np.array_equal(s, ref.numpy())
    occ, keep = GR.prune_update(g["density"], g["occupancy0"], float(g["decay"]), float(g["min_density"]))
    np.testing.assert_allclose(occ, g["occupancy1"], atol=2e-5, rtol=0)
    assert np.array_equal(keep, g["keep"])


def test_prune_update_nan_and_edges_follow_torch():
    """occupancy = torch.stack([density, occupancy * decay], -1).max(-1)[0]; keep = occupancy > min_density (nerf.py:186-198):
    a NaN from either side propagates and prunes the cell."""
    nan, inf = float("nan"), float("inf")
    dens = np.array([nan, 0.3, inf, -inf, -inf, 0.01, 0.2, nan, 0.5, 0.0], f32)
    occ0 = np.array([0.9, nan, 0.1, 0.9, 0.0, 0.01, 0.3, nan, 0.5, 0.0], f32)
    for decay in (0.0, 0.6, 1.0):
        for md in (0.01, 0.5):
            occ, keep = GR.prune_update(dens, occ0, decay, md)
            t = torch.stack([torch.from_numpy(dens), torch.from_numpy(occ0) * decay], -1).max(-1)[0]
            assert np.array_equal(np.isnan(occ), t.isnan().numpy())
            assert np.array_equal(occ[~np.isnan(occ)], t.numpy()[~np.isnan(occ)])
            assert np.array_equal(keep, (t > md).numpy())
            assert not keep[np.isnan(occ)].any()
    occ, keep = GR.prune_update(np.array([0.01], f32), np.zeros(1, f32), 0.5, 0.01)   # equal to min_density: not kept
    assert not keep[0]


def test_prune_stream_is_the_ray_jitter():
    """The counter-based u of wb_prune_samples is wb_jitter(wb_ray_key(seed, cell), axis): the marcher's stream with cells for rays."""
    u = GR.prune_stream(7, 100)
    assert u.shape == (100, 5) and (u >= 0).all() and (u < 1).all()
    assert np.array_equal(u, OR.jitter_stream(7, 100, 8)[:, :5])
