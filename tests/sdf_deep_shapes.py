"""Decoders with 2 to 4 hidden layers that wb_sdf_train trains natively, shared by tests/test_gpu_sdf_train_deep.py and the CPU
checks of their reference (tests/test_sdf_train_deep_cpu.py).  Same tuple layout and sample points as tests/sdf_shapes.py."""
import numpy as np

from oracle import sdf_reference as S
from sdf_shapes import SHAPES, case_of, points      # noqa: F401  (points: re-exported for the tests)

# name: (level, num_lods, F, multiscale, pos_mode, pos_freq, hidden, layers, half)
DEEP_SHAPES = {
    "l2_h128": (6, 4, 16, "sum", 1, 0, 128, 2, True),     # the app/nglod octree shape with num_layers = 2 (64-sample tiles)
    "l2_h64":  SHAPES["l2_h64"],                          # 'cat' + positional embedding with the input, in 39
    "l4_h4":   SHAPES["l4_h4"],
    "cat_l3":  (5, 3, 8, "cat", 3, 2, 64, 3, True),       # 'cat' + positional embedding, three hidden layers
}


def make_field(name, seed=0):
    level, nl, F, ms, pm, pf, H, layers, half = DEEP_SHAPES[name]
    case = case_of(level, nl, F, ms)
    rng = np.random.default_rng(seed)
    feats = [(rng.standard_normal(f.shape) * 0.05).astype(np.float32) for f in case["feats"]]
    pd = S.Field(case["spc"], case["trinkets"], feats, 0, ms, [], [], pm, pf).pos_dim
    Ws, bs = S.random_decoder(rng, pd + (F if ms == "sum" else F * nl), pm, H, layers, scale=0.2)
    return S.Field(case["spc"], case["trinkets"], feats, case["active_lods"][0], ms, Ws, bs, pm, pf, half), case


def tile_of(field, limit=227 * 1024, threads=256):
    """The sample tile wb_sdf_train picks for a decoder with more than one hidden layer (csrc/wb_sdf_train.cu, sdf_train_plan),
    or None when it does not fit."""
    H, nh, in_dim = field.Ws[0].shape[0], len(field.Ws) - 1, field.Ws[0].shape[1]
    in_pad = (in_dim + 3) & ~3
    img = (H * in_pad + H + (nh - 1) * (H * H + H) + H + 4 + 3) & ~3
    stride = lambda n: ((n + 31) & ~31) + 4
    row = stride(in_pad) + nh * stride(H) + 1
    for t in (128, 96, 64, 32):
        if (2 * img + t * row + 2 * (threads // 32)) * 4 <= limit:
            return t
    return None
