"""The tensor-core decoder launches pick the kernel instances compiled for the app/nerf geometry (TcShapeNerf64 in wb_shade_tc.cu)
exactly for decoders of that geometry: the bench-shaped decoder of test_gpu_tc_decoders.py (SIZE_CASE) and race_L13_pos run them;
other widths and embeddings keep the run-time instances.  The geometry is the padded one, so the shaped instances serve a family of
decoders: tests/test_gpu_tc_shape_family.py sweeps the selection against a mirror of it, checks members of that family inside the
interval reference and runs the shaped kernels at coordinate, run and tile edges."""
import ctypes as C

import pytest
import torch

from test_gpu_tc_decoders import CASES, SIZE_CASE, Setup

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def shaped(s, backward):
    v = C.c_int32(-1)
    s.L.wb_rf_tc_shaped(s.desc, backward, C.addressof(v))
    return v.value


@pytest.mark.parametrize("name, expect", [
    ("sizes", 1),             # app/nerf: density 32 -> 64 -> 16, colour 42 -> 64 -> 64 -> 3
    ("race_L13_pos", 1),      # 26 features + 3 position-embedding ones pad to the same 32
    ("w64_L16", 0),           # view embedding of 6 frequencies: colour input 54 -> Kp 64
    ("w128", 0),
    ("unequal", 0),
])
def test_shape_instance_selection(W, name, expect):
    case = SIZE_CASE if name == "sizes" else next(c for c in CASES if c.name == name)
    s = Setup(W, case)
    assert shaped(s, 0) == expect
    assert shaped(s, 1) == expect
