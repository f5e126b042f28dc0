"""The selection mirror of tests/test_gpu_tc_shape_family.py follows the source: its geometry is the TcShapeNerf64 line of wb_shade_tc.cu
and its shared-memory constants are wb_shade_tc.cu's, so an edit of the shape moves the family test with it instead of leaving it on a
stale copy.  The mirror's verdicts on a few known decoders are checked without a GPU."""
import os
import re

from test_gpu_tc_decoders import CASES, SIZE_CASE, Case
import test_gpu_tc_shape_family as F

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kaolin-wisp_b200", "csrc", "wb_shade_tc.cu")


def _source():
    with open(SRC) as f:
        return f.read()


def test_mirror_geometry_is_the_source_shape():
    m = re.findall(r"^using\s+TcShapeNerf64\s*=\s*TcShape<\s*(\d+)\s*,\s*(\d+)\s*,\s*TcList<([\d,\s]+)>\s*,\s*TcList<([\d,\s]+)>\s*>\s*;",
                   _source(), re.M)
    assert len(m) == 1, m
    nd, nc, kp, np_ = m[0]
    ints = lambda s: tuple(int(v) for v in s.split(","))
    assert (int(nd), int(nc), ints(kp), ints(np_)) == (F.NERF64_ND, F.NERF64_NC, F.NERF64_KP, F.NERF64_NP)


def test_mirror_constants_are_the_source_constants():
    src = _source()
    assert re.search(r"constexpr int TC_SMEM_MAX = 227 \* 1024 - 1024;", src) and F.TC_SMEM_MAX == 227 * 1024 - 1024
    assert re.search(r"constexpr int TC_ROWS = 64;", src) and re.search(r"constexpr int TC_SLAB = TC_ROWS \* 16;", src)
    assert F.TC_SLAB == 64 * 16
    assert re.search(r"constexpr int TC_SCR_LD = 33;", src) and F.TC_SCR_BYTES == (64 * 33 * 4 + 15) // 16 * 16
    assert re.search(r"constexpr int TC_FWD_GROUPS = 2;", src)
    # the selection functions the mirror restates
    assert "return m.maxw <= 64 && grid_kind == 0 && per_sm == 3 && TcShapeNerf64::matches(m);" in src
    assert "return nef->grid_kind == 0 && nef->feature_dim == 2 && nef->multiscale == 0 && planes <= 16 && m.groups > 1;" in src


def test_mirror_on_known_decoders():
    byname = {c.name: c for c in CASES}
    assert F.nerf64_expected(SIZE_CASE, 0) == 1 and F.nerf64_expected(SIZE_CASE, 1) == 1
    assert F.nerf64_expected(byname["race_L13_pos"], 0) == 1 and F.nerf64_expected(byname["race_L13_pos"], 1) == 1
    for name in ("w64_L16", "w128", "unequal", "cat_lod_F2", "w16"):
        assert F.nerf64_expected(byname[name], 0) == 0 and F.nerf64_expected(byname[name], 1) == 0, name
    # the family shape's forward runs three CTAs per SM at any of its members' real widths
    assert F.fwd_per_sm(F.NERF64_KP, F.NERF64_NP) == 3
    # members named in tests/test_gpu_tc_shape_family.py: their padded geometry, and the route the mirror predicts
    for c, fwd, bwd in F.MEMBERS:
        assert (F.nerf64_expected(c, 0), F.nerf64_expected(c, 1)) == (fwd, bwd), c.name
    dout1 = Case("dout1", [64], [64, 64], dout=1, view=(3, 5), L=16)
    assert F.padded_dims(dout1)[2:] == (F.NERF64_KP, F.NERF64_NP) and F.nerf64_expected(dout1, 0) == 0


def test_sweep_reaches_every_class():
    """The seeded sweep holds members of every class (the GPU test then checks that the library agrees with the mirror on them)."""
    import numpy as np
    rng = np.random.default_rng(F.SWEEP_SEED)
    found = {k: 0 for k in F.FAMILY_CLASSES}
    for i in range(F.SWEEP_N):
        c = F._sweep_case(rng, i)
        f0, f1 = F.nerf64_expected(c, 0), F.nerf64_expected(c, 1)
        for k, (fused, pred) in F.FAMILY_CLASSES.items():
            if (f1 if fused else (f0 and not f1)) and pred(c):
                found[k] += 1
    assert all(found.values()), found
