"""CPU tests of the SPC render path's host side: SPCField's colour sources against the reference class (through tests/golden/spc_trace.npz
everywhere, and the unmodified class itself where the reference checkout is present), PackedSPCTracer's channel negotiation against
the reference's BaseTracer and install() on the real PackedSPCTracer."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import wisp_b200 as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "spc_trace.npz")
REF = "/root/reference/wisp"


def _features(z, name, src):
    if src == "rgba":
        return {"colors": torch.from_numpy(z[f"{name}_colors"])}
    if src == "normals":
        return {"normals": torch.from_numpy(z[f"{name}_normals"])}
    return None


@pytest.mark.parametrize("name", ["octa5", "rand7"])
@pytest.mark.parametrize("src", ["rgba", "normals", "coords"])
def test_colour_sources_match_the_reference_golden(name, src):
    """The mirror derives the colours the reference's SPCField derived (spc_field.py:69-114), values and dtype, and rgba() gathers
    the finest level's rows like the reference's (spc_field.py:130-147)."""
    z = np.load(GOLDEN)
    nef = W.SPCField(torch.from_numpy(z[f"{name}_octree"]), features_dict=_features(z, name, src), device="cpu")
    exp = z[f"{name}_{src}_field_colors"]
    assert nef.colors.numpy().dtype == exp.dtype and np.array_equal(nef.colors.numpy(), exp)
    blas = nef.grid.blas
    assert blas.max_level == int(z[f"{name}_level"]) and nef.grid.num_lods == 0 and nef.get_supported_channels() == {"rgb"}
    off = int(blas.pyramid[1, blas.max_level])
    idx = torch.tensor([off, off + 3, off + exp.shape[0] - 1])
    rgb = nef(ridx_hit=idx, channels="rgb")
    assert rgb.shape == (3, 1, 3) and np.array_equal(rgb[:, 0].numpy(), exp[[0, 3, exp.shape[0] - 1], :3])


def test_no_cpu_fallback():
    """Both routes of the tracer need the device: the native one (f32 colours) and the reference body (lod_idx below the finest)."""
    z = np.load(GOLDEN)
    nef = W.SPCField(torch.from_numpy(z["octa5_octree"]), features_dict=_features(z, "octa5", "rgba"), device="cpu")
    rays = W.Rays(torch.from_numpy(z["octa5_origins"]), torch.from_numpy(z["octa5_dirs"]))
    for lod in (None, 3):
        with pytest.raises(W.WispB200Error):
            W.PackedSPCTracer()(nef, rays, lod_idx=lod)


_NEGOTIATION = r"""
import torch
def negotiation(Tracer, tag):
    '''(result, message) of forward() for each channel request against a field that has / lacks "rgb".'''
    class Rec(Tracer):
        def trace(self, nef, rays, channels, extra_channels, lod_idx=None):
            return (sorted(channels), sorted(extra_channels), lod_idx)
    class Nef:
        def __init__(self, ch): self.ch = ch
        def get_supported_channels(self): return set(self.ch)
    t = Rec()
    out = []
    for ch, req, kw in (({"rgb"}, None, {}), ({"rgb"}, "depth", {}), ({"rgb", "normal"}, ["rgb", "normal"], {"lod_idx": 2}),
                        ({"rgb"}, ["normal"], {}), ({"density"}, None, {}), ({"rgb"}, {"hit", "alpha"}, {"lod_idx": None})):
        try:
            out.append(("ok", t(Nef(ch), None, req, **kw)))
        except Exception as e:
            out.append(("raise", str(e).replace(tag, "TRACER")))
    assert t.bg_color == (0.0, 0.0, 0.0) and t.get_supported_channels() == {"depth", "hit", "rgb", "alpha"} and t.get_required_nef_channels() == {"rgb"}
    return out
"""


def test_channel_negotiation_matches_the_mirror_base_tracer():
    ns = {}
    exec(_NEGOTIATION, ns)
    got = ns["negotiation"](W.PackedSPCTracer, "X")
    assert got[0] == ("ok", (["alpha", "depth", "hit", "rgb"], [], None))
    assert got[1] == ("ok", (["depth"], [], None)) and got[2] == ("ok", (["normal", "rgb"], ["normal"], 2))
    assert got[3][0] == "raise" and "{'normal'} are not supported" in got[3][1]
    assert got[4][0] == "raise" and "does not output the required channels {'rgb'}" in got[4][1]
    assert got[5] == ("ok", (["alpha", "hit"], [], None))


def _run_reference(code):
    r = subprocess.run([sys.executable, "-c", code.replace("ROOT", repr(ROOT))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


@pytest.mark.skipif(not os.path.isdir(REF), reason="needs the reference checkout")
def test_against_the_reference_classes():
    """The UNMODIFIED reference SPCField / PackedSPCTracer (imported on CPU through oracle/ref_import.py, in a subprocess: the stubs are
    process-wide): the mirror's colours equal the reference's for every source and normal dtype (float64 and float16 included), the
    channel negotiation gives the same results and exception texts (class names aside), install() patches PackedSPCTracer.trace with
    the same signature and runs the mirror's body, the patched trace has no CPU fallback, and uninstall() restores the original."""
    _run_reference(_NEGOTIATION + r"""
import inspect, sys, warnings
warnings.filterwarnings("ignore")
sys.path.insert(0, ROOT)
import numpy as np
from oracle import ref_import, oracle as O
ref_import.install()
from wisp.core import Rays, RenderBuffer
from wisp.models.nefs import SPCField
from wisp.tracers import PackedSPCTracer
import wisp_b200 as W
from wisp_b200 import install as I
pts = np.argwhere(np.random.default_rng(0).random((16, 16, 16)) < 0.1).astype(np.int16)
octree = torch.from_numpy(O.points_to_octree(pts, 4))
M = pts.shape[0]
g = torch.Generator().manual_seed(0)
sources = [{"colors": torch.randint(0, 256, (M, 4), dtype=torch.uint8, generator=g)}, {"colors": torch.rand(M * 4, generator=g) * 255},
           {"normals": torch.randn(M, 3, generator=g)}, {"normals": torch.randn(M, 3, generator=g, dtype=torch.float64)},
           {"normals": torch.randn(M, 3, generator=g).half()}, None, {}]
for f in sources:
    a, b = SPCField(octree, features_dict=f, device="cpu"), W.SPCField(octree, features_dict=f, device="cpu")
    assert a.colors.dtype == b.colors.dtype and a.colors.shape == b.colors.shape and torch.equal(a.colors, b.colors), f
    assert (a.normals is None) == (b.normals is None) and a.get_supported_channels() == b.get_supported_channels()
    idx = torch.arange(int(a.grid.blas.pyramid[1, 4]), int(a.grid.blas.pyramid[1, 5]))
    assert torch.equal(a(ridx_hit=idx, channels="rgb"), b(ridx_hit=idx, channels="rgb"))
assert negotiation(PackedSPCTracer, "PackedSPCTracer") == negotiation(W.PackedSPCTracer, "PackedSPCTracer")
orig = PackedSPCTracer.trace
assert I.install() is True
assert PackedSPCTracer.trace is not orig and PackedSPCTracer.trace.__name__ == "trace"
assert list(inspect.signature(PackedSPCTracer.trace).parameters) == list(inspect.signature(orig).parameters)
nef = SPCField(octree, features_dict=sources[0], device="cpu")
rays = Rays(origins=torch.zeros(4, 3), dirs=torch.ones(4, 3))
x = torch.zeros(4, 3)
rb = W.RenderBuffer(depth=x[:, :1], hit=x[:, 0] > 0, rgb=x, alpha=x[:, 1:2])
calls = []
mirror = W.tracers.PackedSPCTracer.trace
W.tracers.PackedSPCTracer.trace = lambda self, *a: calls.append((self, a)) or rb
try:
    t = PackedSPCTracer()
    out = t(nef, rays, lod_idx=3)
finally:
    W.tracers.PackedSPCTracer.trace = mirror
assert len(calls) == 1 and calls[0][0] is t and calls[0][1][0] is nef and calls[0][1][1] is rays and calls[0][1][4] == 3
assert isinstance(out, RenderBuffer) and all(getattr(out, c) is getattr(rb, c) for c in ("depth", "hit", "rgb", "alpha"))
for lod in (None, 3):
    try:
        PackedSPCTracer()(nef, rays, lod_idx=lod)
        raise SystemExit("trace on CPU tensors must raise")
    except W.WispB200Error:
        pass
I.uninstall()
assert PackedSPCTracer.trace is orig
print("OK")
""")
