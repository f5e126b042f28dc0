"""CPU tests: the oracle (oracle/wisp_oracle.c) against the fixtures produced by the UNMODIFIED reference
Python (oracle/make_golden.py).  These pin the oracle before it is used to judge the CUDA path."""
import glob
import os

import numpy as np
import pytest

from oracle import oracle as O
from golden_util import load_case

CASES = ["rf_trace_cat", "rf_trace_sum", "rf_trace_noview"]


def test_hashgrid_against_reference_naive(golden_dir):
    """wisp.ops.grid.hashgrid_naive (ops/grid.py:16-75) vs wo_hashgrid_fwd.  fp32 tolerance of the reference's own
    unit test for one trilinear blend (tests/core/test_grid_interpolation.py:50-53): atol 1e-6 / rtol 1e-4
    (atol widened to 2e-6: the naive version clamps in float, the kernel in double)."""
    g = np.load(os.path.join(golden_dir, "hashgrid_naive.npz"))
    feats = O.hashgrid_fwd(g["coords"], g["table"], [int(r) for r in g["resolutions"]], int(g["codebook_bitwidth"]))
    np.testing.assert_allclose(feats, g["feats"], atol=2e-6, rtol=1e-4)


@pytest.mark.parametrize("name", CASES)
def test_raymarch_bit_exact(golden_dir, name):
    """OctreeAS._raymarch_ray executed by the reference Python: indices bit-exact, floats bit-exact."""
    g, nef, spc = load_case(os.path.join(golden_dir, name + ".npz"))
    mr = O.raymarch_ray(spc, g["origins"], g["dirs"], float(g["near"]), float(g["far"]), int(g["n_steps"]), jitter_arr=g["jitter"])
    assert np.array_equal(mr["ridx"], g["mr_ridx"])
    assert np.array_equal(mr["boundary"], g["mr_boundary"])
    assert np.array_equal(mr["samples"], g["mr_samples"])
    assert np.array_equal(mr["depth_samples"], g["mr_depth"])
    assert np.array_equal(mr["deltas"], g["mr_deltas"])


@pytest.mark.parametrize("name", CASES)
def test_trace_forward(golden_dir, name):
    g, nef, spc = load_case(os.path.join(golden_dir, name + ".npz"))
    f = O.rf_trace_fwd(spc, nef, g["origins"], g["dirs"], float(g["near"]), float(g["far"]), int(g["n_steps"]), bg=g["bg"], jitter_arr=g["jitter"])
    assert f["num_samples"] == int(g["num_samples"])
    assert np.array_equal(f["hit"], g["hit"])
    np.testing.assert_allclose(f["rgb"], g["rgb"], atol=1e-5, rtol=0)
    np.testing.assert_allclose(f["alpha"], g["alpha"], atol=1e-5, rtol=0)
    np.testing.assert_allclose(f["depth"], g["depth"], atol=5e-5, rtol=0)


@pytest.mark.parametrize("name", CASES)
def test_trace_backward(golden_dir, name):
    """Gradients: reference autograd (torch) through the reference glue vs the oracle's hand-written backward."""
    g, nef, spc = load_case(os.path.join(golden_dir, name + ".npz"))
    st = O.rf_step(spc, nef, g["origins"], g["dirs"], float(g["near"]), float(g["far"]), int(g["n_steps"]), g["target"],
                   loss=str(g["loss_type"]), bg=g["bg"], jitter_arr=g["jitter"])
    assert abs(st["loss"] - float(g["loss"])) < 1e-6
    for key, ref in (("table", g["g_table"]), ("dens", g["g_dens"]), ("col", g["g_col"])):
        scale = max(np.abs(ref).max(), 1e-12)
        assert np.abs(st[key] - ref).max() <= 1e-4 * scale + 1e-9, key


def test_backward_api_matches_step(golden_dir):
    g, nef, spc = load_case(os.path.join(golden_dir, "rf_trace_cat.npz"))
    R = g["origins"].shape[0]
    st = O.rf_step(spc, nef, g["origins"], g["dirs"], 0.0, 10.0, int(g["n_steps"]), g["target"], bg=g["bg"], jitter_arr=g["jitter"])
    grgb = (st["rgb"] - g["target"]) / (3 * R)
    b = O.rf_trace_bwd(spc, nef, g["origins"], g["dirs"], 0.0, 10.0, int(g["n_steps"]), grgb, bg=g["bg"], jitter_arr=g["jitter"])
    np.testing.assert_allclose(b["table"], st["table"], atol=1e-9)
    np.testing.assert_allclose(b["col"], st["col"], atol=1e-8)


def test_spc_dense_and_points():
    spc = O.octree_to_spc(O.dense_octree(3))
    assert spc.max_level == 3
    assert spc.pyramid[0].tolist() == [1, 8, 64, 512, 0]
    assert spc.pyramid[1].tolist() == [0, 1, 9, 73, 585]
    # Morton order, child c = 4x+2y+z
    assert spc.points[1:9].tolist() == [[0, 0, 0], [0, 0, 1], [0, 1, 0], [0, 1, 1], [1, 0, 0], [1, 0, 1], [1, 1, 0], [1, 1, 1]]
    pts = O.lego_like_points(5)
    s2 = O.octree_to_spc(O.points_to_octree(pts, 5))
    lvl = s2.points[s2.pyramid[1, 5]: s2.pyramid[1, 5] + s2.pyramid[0, 5]]
    assert set(map(tuple, lvl.tolist())) == set(map(tuple, pts.tolist()))


def test_query_edges():
    spc = O.octree_to_spc(O.dense_octree(2))
    c = np.array([[-1.0, -1.0, -1.0], [1.0, 0.0, 0.0], [0.999999, 0.0, 0.0], [-1.0000001, 0, 0], [0.0, 0.0, 0.0],
                  [np.nextafter(np.float32(0), np.float32(-1)), 0, 0]], dtype=np.float32)
    p = O.query(spc, c)
    assert p[0] >= 0 and p[1] == -1 and p[2] >= 0 and p[3] == -1 and p[4] >= 0
    wp = O.query(spc, c, with_parents=True)
    assert wp.shape == (6, 3) and wp[0, 0] == 0 and wp[1].tolist() == [-1, -1, -1]
    # the cell just below 0 differs from the cell at 0 along x
    assert p[5] != p[4]


def test_jitter_stream_properties():
    v = np.array([O.jitter(3, r, s) for r in range(8) for s in range(64)], dtype=np.float32)
    assert v.min() >= 0.0 and v.max() < 1.0
    assert abs(v.mean() - 0.5) < 0.06
    assert len(np.unique(v)) > 500


def test_raymarch_voxel_uniform_golden(golden_dir):
    """OctreeAS._raymarch_voxel / _raymarch_uniform run by the reference Python vs the oracle restatement: bit-exact."""
    g = np.load(os.path.join(golden_dir, "raymarch_nuggets.npz"))
    spc = O.octree_to_spc(g["octree"])
    rt = O.raytrace(spc, g["origins"], g["dirs"], int(g["level"]))
    assert np.array_equal(rt["ridx"], g["nug_ridx"]) and np.array_equal(rt["pidx"], g["nug_pidx"]) and np.array_equal(rt["depth"], g["nug_depth"])
    mv = O.raymarch_voxel(spc, g["origins"], g["dirs"], int(g["n_voxel"]), int(g["level"]), jitter_arr=g["jitter"])
    for k, ref in (("ridx", "v_ridx"), ("samples", "v_samples"), ("depth_samples", "v_depth"), ("deltas", "v_deltas"), ("boundary", "v_boundary")):
        assert np.array_equal(mv[k], g[ref]), k
    mu = O.raymarch_uniform(spc, g["origins"], g["dirs"], int(g["n_uniform"]), int(g["level"]))
    for k, ref in (("ridx", "u_ridx"), ("samples", "u_samples"), ("depth_samples", "u_depth"), ("deltas", "u_deltas"), ("boundary", "u_boundary")):
        assert np.array_equal(mu[k], g[ref]), k


def test_raytrace_against_brute_force():
    """Nugget set == all occupied level cells whose slab intersection is positive and in front of the origin; entry depths
    non-decreasing along each ray; the root level (AABB tracing, triplanar_grid.py:145-150) gives at most one nugget per ray."""
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(4), 4))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 24, 24, 30.0)
    o = np.concatenate([o, np.array([[0.05, 0.02, -0.03], [0.3, 0.3, 0.3]], np.float32)])       # origins inside the volume
    d = np.concatenate([d, np.array([[0.0, 0.0, 1.0], [-0.57735, -0.57735, -0.57735]], np.float32)])
    rt = O.raytrace(spc, o, d)
    lvl = spc.points[spc.pyramid[1, 4]: spc.pyramid[1, 4] + spc.pyramid[0, 4]].astype(np.int64)
    size = np.float32(2.0 / 16)
    for r in list(range(0, o.shape[0], 11)) + [o.shape[0] - 2, o.shape[0] - 1]:
        lo = (lvl.astype(np.float32) * size - np.float32(1.0)); hi = lo + size
        with np.errstate(divide="ignore", invalid="ignore"):
            ta, tb = (lo - o[r]) / d[r], (hi - o[r]) / d[r]
            te = np.where(d[r] != 0, np.minimum(ta, tb), -np.inf).max(1); tx = np.where(d[r] != 0, np.maximum(ta, tb), np.inf).min(1)
        inside_zero = np.all((d[r] != 0) | ((o[r] >= lo) & (o[r] < hi)), axis=1)
        hit = (tx > np.maximum(te, 0)) & inside_zero
        mine = rt["pidx"][rt["ridx"] == r] - spc.pyramid[1, 4]
        assert set(mine.tolist()) == set(np.nonzero(hit)[0].tolist()), r
        dd = rt["depth"][rt["ridx"] == r]
        assert (np.diff(dd[:, 0]) >= 0).all() and (dd[:, 1] > dd[:, 0]).all() and (dd[:, 0] >= 0).all()
    root = O.raytrace(spc, o, d, 0)
    assert root["counts"].max() == 1 and (root["pidx"] == 0).all()


SHAPES = [dict(num_lods=8, feature_dim=4, codebook_bitwidth=14, min_res=8, max_res=128, hidden_dim=32, multiscale="cat", view_freq=4, bias=True),
          dict(num_lods=6, feature_dim=8, codebook_bitwidth=12, min_res=8, max_res=96, hidden_dim=64, multiscale="sum", view_freq=2, bias=False),
          dict(num_lods=12, feature_dim=2, codebook_bitwidth=15, min_res=16, max_res=256, hidden_dim=48, multiscale="cat", view_freq=3, bias=True),
          dict(num_lods=4, feature_dim=2, codebook_bitwidth=10, min_res=4, max_res=32, hidden_dim=16, multiscale="sum", view_freq=1, bias=True)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda c: f"F{c['feature_dim']}{c['multiscale']}L{c['num_lods']}h{c['hidden_dim']}")
def test_oracle_step_vs_torch_twin_other_shapes(shape):
    """The shapes the GPU suite uses beyond the golden fixtures (feature widths 4 / 8, 'sum', 48-wide decoders, no bias):
    the C oracle's hand-written forward + backward against the op-for-op torch twin differentiated by autograd."""
    import torch
    from oracle import torch_twin as T
    rng = np.random.default_rng(2)
    nef = O.make_nef(feature_std=0.3, seed=11, **shape)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(4), 4))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 12, 12, 30.0)
    n = 48
    jit = rng.random((o.shape[0], n), dtype=np.float32)
    tgt = rng.random((o.shape[0], 3), dtype=np.float32)
    st = O.rf_step(spc, nef, o, d, 0.0, 8.0, n, tgt, loss="huber", bg=(1, 1, 1), jitter_arr=jit)
    p = T.TwinParams(nef)
    rgb, _, _, _, mr = T.trace(p, spc, o, d, 0.0, 8.0, n, jit, (1.0, 1.0, 1.0))
    loss = torch.nn.functional.smooth_l1_loss(rgb, torch.from_numpy(tgt), reduction='none').mean()
    loss.backward()
    assert st["num_samples"] == int(mr["ridx"].shape[0]) > 100
    np.testing.assert_allclose(st["rgb"], rgb.detach().numpy(), atol=2e-6)
    assert abs(st["loss"] - float(loss.detach())) < 1e-6
    gt, gd, gc = p.packed_grads()
    for got, ref, nm in ((st["table"], gt, "table"), (st["dens"], gd, "dens"), (st["col"], gc, "col")):
        scale = max(np.abs(ref).max(), 1e-12)
        assert np.abs(got - ref).max() <= 2e-4 * scale + 1e-9, (nm, np.abs(got - ref).max(), scale)


def test_sdf_trace_restatement_matches_reference_tracer(golden_dir):
    """oracle.octree_grid.sdf_trace (numpy restatement of packed_sdf_tracer.py:78-174) against the RenderBuffer the reference's
    own PackedSDFTracer produced (tests/golden/sdf_octree.npz, oracle/make_golden.py:gen_sdf)."""
    from oracle import octree_grid as OG
    g = np.load(os.path.join(golden_dir, "sdf_octree.npz"))
    spc = O.octree_to_spc(g["octree"])
    _, pyr, tr, _ = OG.make_trilinear_spc(spc)
    case = dict(spc=spc, trinkets=tr, pyramid_dual=pyr, active_lods=[3, 4, 5], feats=[g[f"sum_feat{i}"] for i in range(3)], multiscale="sum",
                W=[g["sum_W0"], g["sum_W1"]], b=[g["sum_b0"], g["sum_b1"]], origins=g["origins"], dirs=g["dirs"])
    out = OG.sdf_trace(case, num_steps=24, step_size=0.8, min_dis=1e-3, lod_idx=2, dist_max=6.0)
    assert np.array_equal(out["hit"], g["t_hit"]) and g["t_hit"].sum() > 20
    for k, tol in (("depth", 2e-5), ("xyz", 2e-6), ("normal", 2e-4), ("rgb", 1e-4), ("alpha", 0.0)):
        assert np.abs(out[k] - g["t_" + k]).max() <= tol, k


def test_prune_density_probe_matches_reference_class(golden_dir):
    """The density the reference NeuralRadianceField returned at prune()'s probe points (tests/golden/prune.npz) == oracle nef_rgba."""
    g, onef, spc = load_case(os.path.join(golden_dir, "prune.npz"))
    lvl = int(g["level"])
    pts = spc.points[spc.pyramid[1, lvl]: spc.pyramid[1, lvl] + spc.pyramid[0, lvl]].astype(np.float32)
    smp = ((pts + g["u"]) / np.float32(2 ** lvl) * np.float32(2.0) - np.float32(1.0)).astype(np.float32)
    _, dens = O.nef_rgba(onef, smp, np.zeros_like(smp) + 0.5)
    np.testing.assert_allclose(dens[:, 0], g["density"], atol=2e-6)
    occ = np.maximum(dens[:, 0], g["occupancy0"] * np.float32(g["decay"]))
    np.testing.assert_allclose(occ, g["occupancy1"], atol=2e-6)
    assert np.array_equal(O.points_to_octree(pts[g["keep"]].astype(np.int16), lvl), g["new_octree"])


def test_look_at_rays_matches_reference_source(golden_dir):
    """oracle.look_at_rays == _look_at of the reference's offline renderer (tests/golden/raygen.npz, generated from the unmodified source)."""
    g = np.load(os.path.join(golden_dir, "raygen.npz"))
    for n in ("square", "wide", "tall"):
        a = g[n + "_args"]
        o, d = O.look_at_rays(list(a[:3]), list(a[3:6]), int(a[6]), int(a[7]), float(a[8]))
        assert np.abs(o - g[n + "_origins"]).max() == 0.0 and np.abs(d - g[n + "_dirs"]).max() <= 5e-7, n
