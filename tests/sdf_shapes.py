"""Field shapes and sample points shared by the NeuralSDF kernel tests (tests/test_gpu_sdf_kernels.py) and the tightness check of
their reference (tests/test_sdf_reference.py)."""
import numpy as np

from oracle import octree_grid as OG
from oracle import sdf_reference as S

_CASES = {}


def case_of(level, num_lods, F, multiscale):
    key = (level, num_lods, F, multiscale)
    if key not in _CASES:
        _CASES[key] = OG.make_sdf_case(level=level, num_lods=num_lods, feature_dim=F, hidden_dim=8, multiscale=multiscale, res=24, seed=11,
                                       feature_std=0.05)
    return _CASES[key]


# name: (level, num_lods, F, multiscale, pos_mode, pos_freq, hidden, layers, half)
SHAPES = {
    "config3":       (6, 4, 16, "sum", 1, 0, 128, 1, True),    # <16,1>: the app/nglod shape
    "fast_h1":       (5, 3, 16, "sum", 1, 0, 1, 1, True),      # <16,1>, H % 4 tail only
    "fast_h3":       (5, 3, 16, "sum", 1, 0, 3, 1, True),
    "fast_h30":      (5, 3, 16, "sum", 1, 0, 30, 1, True),     # 28 units in quads + a 2-unit tail
    "fast_fp32":     (5, 3, 16, "sum", 1, 0, 32, 1, False),    # half_features = False
    "fast_1lod":     (5, 1, 16, "sum", 1, 0, 32, 1, True),     # num_lods = 1
    "sum_pos3":      (5, 3, 16, "sum", 3, 2, 32, 1, True),     # <0,0> at the dispatch boundary: embedded position
    "cat_id":        (5, 3, 16, "cat", 1, 0, 32, 1, True),     # <0,0> at the dispatch boundary: 'cat'
    "widest":        (5, 3, 23, "cat", 3, 10, 128, 1, True),   # <0,0>: in 132, H 128 (205 KB of shared memory in training)
    "f64_pos2":      (5, 3, 64, "sum", 2, 1, 32, 1, True),     # F above WB_X_MAX_F, no raw position
    "f1_base0":      (5, 6, 1, "cat", 0, 0, 16, 1, True),      # every octree level, the root cell included
    "l2_h64":        (5, 3, 8, "cat", 3, 2, 64, 2, True),      # eval / trace only from here on
    "l3_h128":       (5, 3, 23, "cat", 3, 10, 128, 3, True),   # in 132: 200 720 B, the largest image that fits
    "l4_h124":       (5, 3, 16, "sum", 1, 0, 124, 4, True),    # in 19: 196 928 B
    "l4_h4":         (5, 3, 16, "sum", 1, 0, 4, 4, True),
}
TRAINABLE = [k for k, v in SHAPES.items() if v[7] == 1]


def make_field(name, seed=0):
    level, nl, F, ms, pm, pf, H, layers, half = SHAPES[name]
    case = case_of(level, nl, F, ms)
    rng = np.random.default_rng(seed)
    feats = [(rng.standard_normal(f.shape) * 0.05).astype(np.float32) for f in case["feats"]]
    pd = S.Field(case["spc"], case["trinkets"], feats, 0, ms, [], [], pm, pf).pos_dim
    Ws, bs = S.random_decoder(rng, pd + (F if ms == "sum" else F * nl), pm, H, layers, scale=0.2)
    return S.Field(case["spc"], case["trinkets"], feats, case["active_lods"][0], ms, Ws, bs, pm, pf, half), case


def points(case, n, seed=1, coarse_level=2):
    """Near-surface points, uniform points in [-1.1, 1.1]^3 (outside the octree too), points on cell faces / edges / corners of the
    finest and of a coarse level (dyadic coordinates), coordinates exactly +-1, and duplicates."""
    rng = np.random.default_rng(seed)
    spc, L = case["spc"], case["level"]
    ipts = spc.points[spc.pyramid[1, L]: spc.pyramid[1, L] + spc.pyramid[0, L]].astype(np.int64)
    pts = ipts.astype(np.float32)
    k = max(n // 6, 1)
    near = (pts[rng.integers(0, pts.shape[0], k)] + rng.random((k, 3)).astype(np.float32)) / (2.0 ** (L - 1)) - 1.0
    uni = rng.uniform(-1.1, 1.1, (k, 3))
    def dyadic(level, m):
        c = ipts[rng.integers(0, pts.shape[0], m)] >> (L - level)
        off = rng.integers(0, 2, (m, 3)).astype(np.float64) * rng.integers(0, 2, (m, 1))       # corners, edges, faces
        frac = np.where(rng.random((m, 3)) < 0.5, off, rng.random((m, 3)))
        return (c + frac) / 2.0 ** (level - 1) - 1.0
    ones = rng.choice([-1.0, 1.0], (k, 3)) * (rng.random((k, 3)) < 0.5) + rng.uniform(-1, 1, (k, 3)) * (rng.random((k, 3)) >= 0.5)
    ones[:, 0] = rng.choice([-1.0, 1.0], k)
    dup = np.repeat(near[:1], k, 0)
    c = np.concatenate([near, uni, dyadic(L, k), dyadic(coarse_level, k), ones, dup]).astype(np.float32)
    c = np.concatenate([c, near[rng.integers(0, k, max(n - c.shape[0], 0))]]).astype(np.float32)
    c = c[rng.permutation(c.shape[0])[:n]]
    gt = ((np.abs(c).sum(-1) - 0.5) / np.sqrt(3.0)).astype(np.float32)
    return c, gt
