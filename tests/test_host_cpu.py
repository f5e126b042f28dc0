"""CPU tests of the product's host side: the C-ABI library loads and exports every symbol include/wispb200.h declares,
the ctypes struct layouts match the header, the host-side SPC builder matches the oracle, and compute entry points
refuse to run without an H100 (no CPU fallback)."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
import torch

import wisp_b200 as W
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "wispb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(wb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = W._cabi.lib()
    names = header_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"libwispb200.so does not export {n}"
    assert sorted(W._cabi.EXPORTS) == names


def test_struct_layouts_match_header(tmp_path):
    """Compile include/wispb200.h with the C compiler and compare sizeof/offsetof of EVERY descriptor struct with the ctypes mirrors."""
    import subprocess
    A = W._cabi
    structs = {"wb_nef_desc": A.NefDesc, "wb_rays": A.RaysDesc, "wb_octree": A.OctreeDesc, "wb_sdf_desc": A.SdfDesc, "wb_sdf_state": A.SdfState,
               "wb_adam_segment": A.AdamSegment}
    lines, mine = [], []
    for cname, cls in structs.items():
        lines.append(f'printf("%zu\\n", sizeof({cname}));'); mine.append(C.sizeof(cls))
        for fname, _ in cls._fields_:
            lines.append(f'printf("%zu\\n", offsetof({cname}, {fname}));'); mine.append(getattr(cls, fname).offset)
    src = tmp_path / "lay.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wispb200.h"\nint main(void){ ' + " ".join(lines) + ' return 0; }')
    exe = tmp_path / "lay"
    subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert mine == vals


def test_no_cpu_fallback():
    o = W.OctreeAS.make_dense(2, device="cpu")
    with pytest.raises(W._cabi.WispB200Error):
        o.query(torch.zeros(3, 3))
    g = W.HashGrid.from_geometric(o, 2, 4, 'cat', 0.1, 0.0, 10, 4, 32)
    with pytest.raises(W._cabi.WispB200Error):
        g.interpolate(torch.zeros(3, 3), 3)
    with pytest.raises(W._cabi.WispB200Error):
        o.raymarch(W.Rays(torch.zeros(2, 3), torch.ones(2, 3), 0.0, 1.0), 'ray', 8)


def test_host_spc_builder_matches_oracle():
    pts = O.lego_like_points(5)
    oct_t = W.spc.points_to_octree(torch.from_numpy(pts), 5)
    assert np.array_equal(oct_t.numpy(), O.points_to_octree(pts, 5))
    ref = O.octree_to_spc(oct_t.numpy())
    points, pyramid, prefix = W.spc.octree_to_spc(oct_t)
    assert np.array_equal(points.numpy(), ref.points) and np.array_equal(pyramid.numpy(), ref.pyramid) and np.array_equal(prefix.numpy(), ref.prefix)
    assert np.array_equal(W.spc.create_dense_octree(3).numpy(), O.dense_octree(3))


def test_nef_mirror_matches_reference_names_and_shapes():
    o = W.OctreeAS.make_dense(2, device="cpu")
    g = W.HashGrid.from_geometric(o, feature_dim=2, num_lods=16, multiscale_type='cat', feature_std=1e-9, codebook_bitwidth=19,
                                  min_grid_res=16, max_grid_res=512)
    assert g.resolutions == [16, 20, 25, 32, 40, 50, 64, 80, 101, 128, 161, 203, 256, 322, 406, 512]      # SURVEY.md section 8
    assert g.codebook.feats.shape == (5217937, 2)
    nef = W.NeuralRadianceField(g, view_embedder='positional', view_multires=4, hidden_dim=64, num_layers=1, bias=True)
    names = dict(nef.named_parameters())
    assert names["decoder_density.layers.0.weight"].shape == (64, 32) and names["decoder_density.lout.weight"].shape == (16, 64)
    assert names["decoder_color.layers.0.weight"].shape == (64, 42) and names["decoder_color.lout.weight"].shape == (3, 64)
    assert "grid.codebook.feats" in names
    assert sum(p.numel() for n, p in names.items() if n.startswith("decoder_density")) == 3152
    assert sum(p.numel() for n, p in names.items() if n.startswith("decoder_color")) == 7107
    assert float(nef.decoder_density.lout.bias[0]) == 1.0
    spec = nef.fused_spec()
    assert spec.view_mode == 3 and spec.dens_dims == [32, 64, 16] and spec.col_dims == [42, 64, 64, 3]
    # view_embedder='none' still feeds ray_d (include_input=True), nerf.py:105-106,116-119
    nef2 = W.NeuralRadianceField(g, view_embedder='none', hidden_dim=16)
    assert nef2.view_embed_dim == 3 and nef2.fused_spec().view_mode == 1


def test_tracer_channel_negotiation_errors():
    o = W.OctreeAS.make_dense(2, device="cpu")
    g = W.HashGrid.from_geometric(o, 2, 4, 'cat', 0.1, 0.0, 10, 4, 32)
    nef = W.NeuralRadianceField(g, hidden_dim=16)
    tr = W.PackedRFTracer()
    assert tr.get_supported_channels() == {"depth", "hit", "rgb", "alpha"} and tr.get_required_nef_channels() == {"rgb", "density"}
    with pytest.raises(Exception, match="not supported"):
        tr(nef, rays=W.Rays(torch.zeros(1, 3), torch.ones(1, 3)), channels=["rgb", "normals"])
    assert tr.get_prev_num_samples() is None


def test_host_prefetcher_cpu_passthrough():
    """HostPrefetcher keeps order and arity; on a CPU 'device' it degenerates to plain .to() (no stream)."""
    import torch
    from wisp_b200.parallel import HostPrefetcher
    batches = [(torch.full((3,), float(i)), torch.full((2, 2), float(-i))) for i in range(4)]
    got = list(HostPrefetcher(batches, "cpu"))
    assert len(got) == 4
    for i, (a, b) in enumerate(got):
        assert float(a[0]) == i and float(b[0, 0]) == -i
    assert list(HostPrefetcher([], "cpu")) == []


def test_precision_support_query_is_host_side():
    """wb_rf_precision_supported answers without a device: the 64-wide app/nerf decoders fit the tensor-core path forward
    and backward, so do 128-wide ones of the same depth; deeper decoders fit forward only (their backward stays on the fp32 kernels)."""
    import wisp_b200 as W
    from wisp_b200 import ops
    ans = {}
    for hidden, layers in ((64, 1), (128, 1), (64, 2)):
        blas = W.OctreeAS.make_dense(3, device='cpu')
        grid = W.HashGrid.from_geometric(blas, feature_dim=2, num_lods=16, multiscale_type='cat', feature_std=1e-4, codebook_bitwidth=19,
                                         min_grid_res=16, max_grid_res=512)
        nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=4, hidden_dim=hidden, num_layers=layers, bias=True)
        spec = nef.fused_spec()
        ans[(hidden, layers)] = (ops.precision_supported(spec, nef, 1, False), ops.precision_supported(spec, nef, 1, True),
                                 ops.precision_supported(spec, nef, 0, True))
    assert ans[(64, 1)] == (True, True, True)
    assert ans[(128, 1)] == (True, True, True) and ans[(64, 2)] == (True, False, True)      # hidden 128: one-group tensor-core backward


def test_bucketed_capacities():
    """Per-sample buffers are carved from capacities with at most 1/8 slack that repeat across nearby sample counts, and the
    capacity in force never shrinks (one stable size per training run: no cudaMalloc when S crosses a bucket boundary)."""
    from wisp_b200 import ops
    b = ops._bucket_raw
    assert b(0) == 0 and b(1) == 1 << 16 and b((1 << 16) + 1) == 2 << 16
    for S in (15_592_267, 15_667_821, 12_191_426, 333_000_000, 70_001):
        assert S <= b(S) <= S * 1.125 + (1 << 16)
    assert b(15_592_267) == b(15_667_821)
    old = ops._CAP_FLOOR
    try:
        ops._CAP_FLOOR = 0
        c0 = ops._bucket(15_000_000)
        assert 15_000_000 <= c0 <= 15_000_000 * 1.2
        assert {ops._bucket(s) for s in range(12_000_000, 15_900_000, 100_003)} == {c0}     # smaller and slightly larger batches reuse it
        c1 = ops._bucket(20_000_000)
        assert c1 >= 20_000_000 and ops._bucket(15_000_000) == c1                            # grows, never shrinks
        assert ops.reserve_samples(30_000_000) >= 30_000_000 and ops._bucket(1) >= 30_000_000
        assert ops._bucket(0) == 0
    finally:
        ops._CAP_FLOOR = old


def test_nugget_capacities_and_bench_shapes():
    """Raytrace outputs come from their own high-water capacity (a render loop over many cameras must not reach cudaMalloc), and
    bench.py's --config 1 / --hidden-dim select the documented shapes."""
    import importlib.util
    import torch
    from wisp_b200 import ops
    old = ops._NUG_FLOOR
    try:
        ops._NUG_FLOOR = 0
        a = ops._empty_n(1_000_000, (2,), torch.float32, "cpu")
        cap = ops._NUG_FLOOR
        assert a.shape == (1_000_000, 2) and 1_000_000 <= cap <= 1_400_000
        assert ops._empty_n(1_100_000, (), torch.int32, "cpu").shape == (1_100_000,) and ops._NUG_FLOOR == cap       # within the headroom: same capacity
        assert ops._empty_n(0, (2,), torch.float32, "cpu").shape == (0, 2)
        assert ops.reserve_nuggets(5_000_000) >= 5_000_000 and ops._empty_n(10, (), torch.int32, "cpu").untyped_storage().nbytes() >= 5_000_000 * 4
    finally:
        ops._NUG_FLOOR = old
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("wb_bench", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec); spec.loader.exec_module(bench)
    import sys
    argv = sys.argv
    try:
        sys.argv = ["bench.py", "--config", "1"]
        a1 = bench.parse()
        assert a1.res == 256 and bench.nef_shape(a1) == (8, 32) and "256^2" in bench.metric_name(a1)
        sys.argv = ["bench.py", "--hidden-dim", "128"]
        a2 = bench.parse()
        assert a2.res == 1024 and bench.nef_shape(a2) == (16, 128) and bench.metric_name(a2) == bench.METRIC
        assert "hidden-128" in bench.workload_config(a2)["workload"]
        sys.argv = ["bench.py"]
        assert "2-layer-64" in bench.workload_config(bench.parse())["workload"]
    finally:
        sys.argv = argv


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` needs no GPU: it times the CPU oracle on a bounded sample and prints ONE JSON line carrying
    the contract keys with impl = reference, zero-byte e2e and a cpu_baseline that repeats the line's value."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                          "--cpu-sample-rays", "256"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-500:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "e2e", "cpu_baseline"):
        assert key in d, key
    assert d["impl"] == "reference" and d["unit"] == "rays/s" and d["value"] > 0 and d["steps"] == 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert "workload" in d["config"]
    # ranks other than 0 of a torchrun launch print nothing and exit 0
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out1 = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                          capture_output=True, text=True, timeout=300, env=env)
    assert out1.returncode == 0 and out1.stdout.strip() == ""


@pytest.mark.skipif(not os.path.isdir("/root/reference/wisp"), reason="needs the reference checkout (build container only)")
def test_install_patches_the_real_wisp_classes():
    """wisp_b200.install.install() against the UNMODIFIED reference classes (imported on CPU through oracle/ref_import.py, in a
    subprocess because the import stubs are process-wide): every patched method keeps its signature, the tracer keeps the
    attributes other wisp code reads and survives copy.deepcopy, ops.nef_spec / ops.sdf_field read the reference's own
    NeuralRadianceField / NeuralSDF objects, unsupported configurations are declined (-> original method), deep decoders
    under autocast resolve to the fp32 kernels, ops.octree_tensors caches one handle per octree on either OctreeAS, the grid
    and SDF-tracer patches run the mirror classes' methods, and uninstall() restores the originals."""
    import subprocess
    code = r"""
import copy, inspect, sys, warnings
warnings.filterwarnings("ignore")
sys.path.insert(0, ROOT)
import torch
from oracle import ref_import, oracle as O
ref_import.install()
import wisp.ops.grid as grid_ops
from wisp.accelstructs import OctreeAS
from wisp.models.grids import HashGrid, OctreeGrid, TriplanarGrid
from wisp.models.nefs import NeuralRadianceField, NeuralSDF
from wisp.tracers import PackedRFTracer, PackedSDFTracer
targets = [(OctreeAS, n) for n in ("query", "raytrace", "_raymarch_ray", "_raymarch_voxel", "_raymarch_uniform")] + \
          [(TriplanarGrid, "interpolate"), (OctreeGrid, "interpolate"), (PackedRFTracer, "trace"), (PackedSDFTracer, "trace"),
           (NeuralSDF, "sdf"), (NeuralRadianceField, "prune"), (grid_ops, "hashgrid")]
before = {(c.__name__, n): getattr(c, n) for c, n in targets}
import wisp_b200 as W
from wisp_b200 import install as I, ops
assert I.install() is True
for c, n in targets:
    new, old = getattr(c, n), before[(c.__name__, n)]
    assert new is not old, (c, n)
    assert list(inspect.signature(new).parameters) == list(inspect.signature(old).parameters), (c, n)
    assert new.__name__ == n
tracer = PackedRFTracer(raymarch_type='ray', num_steps=16, bg_color=(0.0, 0.0, 0.0))
t2 = copy.deepcopy(tracer)
assert t2.num_steps == 16 and t2.raymarch_type == 'ray' and hasattr(t2, "bg_color") and t2.get_prev_num_samples() is None
assert tracer.get_supported_channels() == {"depth", "hit", "rgb", "alpha"}
blas = OctreeAS(torch.from_numpy(O.dense_octree(3)))
hg = HashGrid.from_geometric(blas, feature_dim=2, num_lods=4, multiscale_type='cat', feature_std=0.1, codebook_bitwidth=10, min_grid_res=4, max_grid_res=32)
nef = NeuralRadianceField(hg, view_embedder='positional', view_multires=4, hidden_dim=64, num_layers=1, bias=True)
spec = ops.nef_spec(nef, 3)
assert spec is not None and spec.kind == "hash" and spec.view_mode == 3 and spec.view_freq == 4 and spec.pos_mode == 0
assert spec.dens_dims == [8, 64, 16] and spec.col_dims == [42, 64, 64, 3] and spec.has_bias and spec.resolutions == [int(r) for r in hg.resolutions]
assert ops.precision_supported(spec, nef, 1, True)
wide = NeuralRadianceField(hg, view_embedder='positional', view_multires=4, hidden_dim=128, num_layers=1, bias=False)
sw = ops.nef_spec(wide, 3)
assert sw is not None and not sw.has_bias and ops.precision_supported(sw, wide, 1, False) and ops.precision_supported(sw, wide, 1, True)
deep = NeuralRadianceField(hg, view_embedder='positional', view_multires=4, hidden_dim=128, num_layers=2, bias=True)
assert ops.precision_supported(ops.nef_spec(deep, 3), deep, 1, False) and not ops.precision_supported(ops.nef_spec(deep, 3), deep, 1, True)
# the precision rule of both tracers and MultiviewStep: an explicit precision is literal, None follows autocast where supported
sd = ops.nef_spec(deep, 3)
assert [ops.resolve_precision(None, s, n, True) for s, n in ((spec, nef), (sw, wide), (sd, deep))] == [0, 0, 0]
torch.set_autocast_enabled("cuda", True)
try:
    assert [ops.resolve_precision(None, s, n, b) for s, n, b in ((spec, nef, True), (sw, wide, True), (sd, deep, True), (sd, deep, False))] == [1, 1, 0, 1]
    assert ops.resolve_precision(0, spec, nef, True) == 0 and ops.resolve_precision(1, sd, deep, True) == 1
finally:
    torch.set_autocast_enabled("cuda", False)
ident = NeuralRadianceField(hg, view_embedder='none', pos_embedder='positional', pos_multires=3, position_input=True, hidden_dim=32)
si = ops.nef_spec(ident, 3)
assert si.view_mode == 1 and si.pos_mode == 3 and si.pos_freq == 3 and si.dens_dims[0] == 8 + 3 + 18
nef.view_embedder = torch.nn.Linear(3, 27)                      # something the native path does not know (cf. 'tcnn')
assert ops.nef_spec(nef, 3) is None
tg = TriplanarGrid(blas, feature_dim=4, log_base_resolution=3, num_lods=2, multiscale_type='sum', feature_std=0.1)
st = ops.nef_spec(NeuralRadianceField(tg, view_embedder='positional', view_multires=4, hidden_dim=32), 1)
assert st.kind == "triplanar" and st.feature_dim == 12 and st.resolutions == [8, 16] and ops.raymarch_level(tg, 1) == 0
og = OctreeGrid(blas, feature_dim=8, num_lods=2, multiscale_type='cat', feature_std=0.1)
so = ops.nef_spec(NeuralRadianceField(og, view_embedder='positional', view_multires=4, hidden_dim=32), 1)
assert so.kind == "octree" and so.base_lod == og.base_lod == 2 and so.dens_dims[0] == 16 and ops.raymarch_level(og, 1) == 2
assert ops.raymarch_level(hg, 3) == 3
sdf = NeuralSDF(OctreeGrid(blas, feature_dim=16, num_lods=2, multiscale_type='sum', feature_std=0.1), pos_embedder='none', position_input=True, hidden_dim=128, num_layers=1)
fd = ops.sdf_field(sdf)
assert fd is not None and fd[0].hidden_dim == 128 and fd[0].feature_dim == 16 and fd[0].pos_mode == 1 and fd[0].multiscale == 1
assert ops.sdf_field(NeuralSDF(hg, pos_embedder='none', position_input=True, hidden_dim=32)) is None       # SDF over a hash grid: phase-by-phase route
# one octree handle for the reference's and the mirror's OctreeAS: cached on the BLAS, rebuilt when the octree tensor is replaced
mb = W.OctreeAS(torch.from_numpy(O.dense_octree(3)))
for b in (blas, mb):
    t = ops.octree_tensors(b)
    assert ops.octree_tensors(b) is t and t.prefix.dtype == t.pyramid.dtype == torch.int32
    b.octree = b.octree.clone()
    t2 = ops.octree_tensors(b)
    assert t2 is not t and ops.octree_tensors(b) is t2
assert mb.tensors() is t2
mb.to("cpu")
assert mb.tensors() is not t2
# the grid and SDF-tracer patches run the mirror classes' methods; the triplanar fall-back (non-'reflection' padding) stays
from wisp.core import Rays, RenderBuffer
x = torch.zeros(4, 3)
rb = W.RenderBuffer(rgb=x, alpha=x[:, :1], depth=x[:, :1], hit=x[:, 0] > 0, xyz=x, normal=x)
calls = []
def recorder(name, result):
    def fn(self, *a):
        calls.append((name, self, a))
        return result
    return fn
mirror = (W.grids.TriplanarGrid.interpolate, W.grids.OctreeGrid.interpolate, W.tracers.PackedSDFTracer.trace)
W.grids.TriplanarGrid.interpolate, W.grids.OctreeGrid.interpolate = recorder("tri", x), recorder("oct", x)
W.tracers.PackedSDFTracer.trace = recorder("sdf", rb)
try:
    st_ = PackedSDFTracer()
    assert tg.interpolate(x, 1) is x and og.interpolate(x, 1) is x
    out = st_.trace(sdf, Rays(origins=x, dirs=x), {"rgb"}, set(), 1, 8, 0.5, 1e-3)
    tg.features[1].padding_mode = 'zeros'
    assert tg.interpolate(x, 1) is not x and len(calls) == 3
    tg.features[1].padding_mode = 'reflection'
finally:
    W.grids.TriplanarGrid.interpolate, W.grids.OctreeGrid.interpolate, W.tracers.PackedSDFTracer.trace = mirror
assert [c[0] for c in calls] == ["tri", "oct", "sdf"] and calls[0][1] is tg and calls[1][1] is og and calls[2][1] is st_
assert all(c[2][0] is x and c[2][1] == 1 for c in calls[:2])
assert calls[2][2][0] is sdf and calls[2][2][2] == {"rgb"} and calls[2][2][3:] == (set(), 1, 8, 0.5, 1e-3)
assert isinstance(out, RenderBuffer) and all(getattr(out, c) is getattr(rb, c) for c in ("rgb", "alpha", "depth", "hit", "xyz", "normal"))
# the real mirror bodies on the reference grids (no `half_features` on its OctreeGrid) get as far as the device check
for g in (tg, og):
    try:
        g.interpolate(x, 1)
        raise SystemExit("interpolate on CPU tensors must raise")
    except W.WispB200Error:
        pass
# no CPU fallback behind the patches either
try:
    blas.query(torch.zeros(4, 3))
    raise SystemExit("query on CPU tensors must raise")
except W.WispB200Error:
    pass
I.uninstall()
for c, n in targets:
    assert getattr(c, n) is before[(c.__name__, n)], (c, n)
print("INSTALL-OK")
"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code.replace("ROOT", repr(root))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "INSTALL-OK" in r.stdout, (r.stdout[-500:], r.stderr[-1500:])
