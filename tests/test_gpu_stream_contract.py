"""Every stream-taking entry point keeps to the stream it is given (include/wispb200.h, Conventions), for every case of
tests/stream_cases.py:

- side stream, gated: the real inputs are copied in and the call is made on a fresh stream that first sleeps, over buffers that hold
  a valid second input set (the poison).  The call must return while the stream is still busy (no host synchronisation) and, after
  the sleep, give the default-stream result: a launch that escaped to another stream runs at once, on the poison, and changes it.
  Each case must be sensitive: the same call on the poison gives another result.
- graph capture: the call captured into a CUDA graph over the same static buffers, replayed on the poison set, gives what an eager
  call on the poison gives.
- two host threads calling entry points that share kernel instances in other configurations, at the same time (ctypes releases the
  GIL), get what the same calls give one after the other.
- a second device, when there is one: the same calls on cuda:1 between two runs on cuda:0 give the same bits.
"""
import threading

import pytest
import torch

import stream_cases as SC

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 200_000_000          # ~0.12 s of GPU time on the side stream: the host enqueues the copies and the call long before it ends

# Entry points the driver refuses to capture into a CUDA graph, and why (include/wispb200.h, Conventions, says the same).
GRAPH_REFUSED = {}


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


_BUILT = {}


ALL_CASES = {**SC.CASES, **SC.EXTRA_CASES}


def built(name):
    if name not in _BUILT:
        _BUILT[name] = ALL_CASES[name]()
        torch.cuda.synchronize()
    return _BUILT[name]


def load(b, vals):
    for k, v in vals.items():
        b.bufs[k].copy_(v)


def snap(b):
    return {k: b.bufs[k].clone() for k in b.outputs}


def eager(b, vals):
    load(b, vals)
    b.call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return snap(b)


def _bits(t):
    return t.contiguous().view(torch.uint8)


def mismatch(b, want, got):
    """Outputs of `got` that differ from `want` beyond their tolerance -> [(name, description)]."""
    bad = []
    for k, tol in b.outputs.items():
        w, g = want[k], got[k]
        if tol is None:
            if not torch.equal(_bits(w), _bits(g)):
                bad.append((k, f"{int((_bits(w) != _bits(g)).sum())} bytes differ"))
        else:
            top = float(w.double().abs().max()) if w.numel() else 0.0
            err = float((g.double() - w.double()).abs().max()) if w.numel() else 0.0
            if not (err <= tol * max(top, 1e-30)):
                bad.append((k, f"max|diff| {err:.3e} > {tol:g} * max|ref| {top:.3e}"))
    return bad


def initial_outputs(b):
    return {k: b.real[k].clone() for k in b.outputs}


@pytest.mark.parametrize("name", sorted(ALL_CASES))
def test_side_stream_gated(W, name):
    b = built(name)
    ref = eager(b, b.real)
    # sensitivity: what a launch that ran on the poison (or, for calls without device inputs, did not run after the re-initialisation)
    # would leave must differ from the reference
    other = initial_outputs(b) if b.host_inputs else eager(b, b.poison)
    assert mismatch(b, ref, other), f"{name}: the poison set gives the reference result; the gate would prove nothing"

    load(b, b.poison)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        load(b, b.real)
        b.call(s.cuda_stream)
        busy = not s.query()
        got = snap(b)               # on s: work the call forked elsewhere and did not join back to s is not waited for
    torch.cuda.synchronize()
    assert busy, f"{name}: the side stream had drained when the call returned (a host synchronisation, or a sleep too short)"
    bad = mismatch(b, ref, got)
    assert not bad, f"{name}: the call on a gated side stream differs from the default-stream call: {bad}"
    print(f"STREAM {name}: gated side stream == default stream ({len(b.outputs)} outputs)")


@pytest.mark.parametrize("name", sorted(ALL_CASES))
def test_graph_capture(W, name):
    b = built(name)
    want = eager(b, b.poison)
    load(b, b.real)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(g):
            b.call(torch.cuda.current_stream().cuda_stream)
        refused = None
    except Exception as e:           # noqa: BLE001 -- the driver's or the library's refusal, reported below
        refused = e
    torch.cuda.synchronize()
    if name in GRAPH_REFUSED:
        assert refused is not None, f"{name} is listed as refusing capture but was captured: update GRAPH_REFUSED and the header"
        print(f"GRAPH {name}: refused as expected ({GRAPH_REFUSED[name]})")
        return
    assert refused is None, f"{name}: capture failed: {refused!r}"
    load(b, b.poison)
    g.replay()
    torch.cuda.synchronize()
    bad = mismatch(b, want, snap(b))
    assert not bad, f"{name}: graph replay on the poison set differs from the eager call: {bad}"
    print(f"GRAPH {name}: replay == eager")


def _concurrent_pairs():
    """(what, builder of thread 0's call, builder of thread 1's call): calls sharing kernel instances in different configurations.
    The precision-0 widths stop at 128: a 256-wide decoder needs more than the 227 KB of shared memory of an SM, and wb_rf_shade_fwd
    refuses it ("decoder too large for shared memory")."""
    return [
        ("precision-0 shade fwd+bwd, 16 vs 128 wide", lambda: SC.p0_shade_case(16), lambda: SC.p0_shade_case(128, seed=1)),
        ("chunked precision-1 backward, two data sets", lambda: SC.chunked_bwd_case(0), lambda: SC.chunked_bwd_case(1)),
        ("wb_image_train, hidden 16 vs 128", lambda: SC.image_train_case(16), lambda: SC.image_train_case(128)),
        ("wb_sdf_train_tc, two field shapes", lambda: SC.sdf_train_tc_case("config3"), lambda: SC.sdf_train_tc_case("cat_id")),
        ("wb_mesh_sdf, two meshes", lambda: SC.CASES["wb_mesh_sdf"](), lambda: SC.CASES["wb_mesh_sdf"]()),
    ]


def test_two_host_threads(W):
    pairs = [(what, f0(), f1()) for what, f0, f1 in _concurrent_pairs()]
    # thread 1 runs the mesh case on its poison set: another mesh, same shapes
    vals = [[b0.real, b1.poison if what.startswith("wb_mesh_sdf") else b1.real] for what, b0, b1 in pairs]
    serial = [[eager(b, v) for b, v in zip((b0, b1), vs)] for (_, b0, b1), vs in zip(pairs, vals)]
    for (_, b0, b1), vs in zip(pairs, vals):
        load(b0, vs[0]); load(b1, vs[1])
    torch.cuda.synchronize()
    dev = torch.cuda.current_device()
    barrier = threading.Barrier(2)
    errors = []

    def run(i):
        try:
            torch.cuda.set_device(dev)
            s = torch.cuda.Stream()
            barrier.wait()
            for _, *bs in pairs:
                bs[i].call(s.cuda_stream)
            s.synchronize()
        except Exception as e:          # noqa: BLE001 -- reported on the main thread
            errors.append((i, repr(e)))
            barrier.abort()

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for (what, b0, b1), ref in zip(pairs, serial):
        for i, b in enumerate((b0, b1)):
            bad = mismatch(b, ref[i], snap(b))
            assert not bad, f"{what}, thread {i}: concurrent call differs from the serial one: {bad}"
        print(f"THREADS {what}: both threads == serial")


# entries whose dynamic shared memory exceeds the default 48 KB (per-device function attributes), and the chunked backward
# (per-device side stream)
SECOND_DEVICE = ["wb_rf_shade_fwd", "wb_rf_shade_bwd", "wb_rf_decoder_bwd", "wb_sdf_eval", "wb_sdf_train", "wb_sdf_train_tc", "wb_sdf_trace",
                 "wb_image_eval", "wb_image_train", "wb_codebook_rows_bwd"]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second CUDA device")
def test_second_device(W):
    def run_on(dev, make):
        with torch.cuda.device(dev):
            b = make()
            out = eager(b, b.real)
            return b, {k: v.cpu() for k, v in out.items()}
    makers = [(n, SC.CASES[n]) for n in SECOND_DEVICE] + [("chunked backward", SC.chunked_bwd_case)]
    for name, make in makers:
        b, first = run_on(0, make)
        _, other = run_on(1, make)
        _, again = run_on(0, make)
        # bit-exact outputs bit for bit, atomically accumulated ones within their summation-order tolerance
        for got in (other, again):
            bad = mismatch(b, first, got)
            assert not bad, (name, bad)
        print(f"DEVICE {name}: cuda:0 == cuda:1 == cuda:0")


# ---- public routes under `with torch.cuda.stream(s)` ---------------------------------------------------------------------------
# Each route builds a fresh model and its inputs (the same every time), runs on the default stream for the reference, then runs again
# on a side stream that first sleeps: the inputs (rays, coordinates, targets, and the parameters for prune) hold a valid second set
# until the side stream copies the real ones in after the sleep.  Anything the route enqueues elsewhere -- its own side streams, a
# per-stream cache, a host read between stages -- that is not ordered after the side stream sees the second set.  Forward outputs and
# sample counts must match bit for bit; gradients and updated parameters within the atomic-order tolerance of their kernels' tests.
ROUTE_TOL = 1e-5            # fp32 atomics (tests/test_gpu_sdf_step.py compares its gradients at 1e-4 of their max across routes)
ROUTE_TOL_TC = 1e-4


def _dev(a, dtype=None):
    t = torch.as_tensor(a)
    return (t.to(dtype) if dtype is not None else t).cuda().contiguous()


def _route(build, run, tol):
    """build() -> (state, {name: (destination tensor, real value, other value)}); run(state) -> {name: tensor};
    tol: {output name: None (bit-exact) or relative tolerance}, default None."""
    st, ins = build()
    with torch.no_grad():
        for dst, real, _ in ins.values():
            dst.copy_(real)
    ref = {k: v.detach().clone() for k, v in run(st).items()}
    torch.cuda.synchronize()
    st, ins = build()
    with torch.no_grad():
        for dst, _, other in ins.values():
            dst.copy_(other)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        with torch.no_grad():
            for dst, real, _ in ins.values():
                dst.copy_(real)
        got = {k: v.detach().clone() for k, v in run(st).items()}
    torch.cuda.synchronize()
    bad = []
    for k, w in ref.items():
        t = tol.get(k)
        g = got[k]
        if t is None:
            if not torch.equal(_bits(w), _bits(g)):
                bad.append((k, "differs"))
        elif w.numel():
            err, top = float((g.double() - w.double()).abs().max()), float(w.double().abs().max())
            if not err <= t * max(top, 1e-30):
                bad.append((k, f"max|diff| {err:.3e} > {t:g} * {top:.3e}"))
    assert not bad, bad
    return ref


def _rays_pair(res, seed):
    from oracle import oracle as O
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], res, res, 30.0)
    o2, d2 = O.look_at_rays([2.5, 1.2, -2.8], [0.1, 0, 0], res, res, 30.0)
    g = torch.Generator().manual_seed(seed)
    tgt, tgt2 = torch.rand(res * res, 3, generator=g), torch.rand(res * res, 3, generator=g)
    return (_dev(o), _dev(d), _dev(tgt)), (_dev(o2), _dev(d2), _dev(tgt2))


def _nerf(W):
    from oracle import oracle as O
    from gpu_util import nef_from_oracle
    onef = O.make_nef(num_lods=8, codebook_bitwidth=14, min_res=8, max_res=128, hidden_dim=64, feature_std=0.3, seed=1)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(5), 5))
    return nef_from_oracle(onef, spc)[0]


def _grads(mod, tol):
    out = {}
    for n, p in mod.named_parameters():
        if p.grad is not None:
            out["grad." + n] = p.grad
            tol["grad." + n] = tol["_grad"]
    return out


@pytest.mark.parametrize("precision", [0, 1])
def test_route_pipeline_forward_backward(W, precision):
    real, other = _rays_pair(40, 1)
    tol = {"_grad": ROUTE_TOL if precision == 0 else ROUTE_TOL_TC}

    def build():
        nef = _nerf(W)
        tr = W.PackedRFTracer('ray', 128, bg_color=(1.0, 1.0, 1.0)); tr.precision = precision; tr.seed = 21
        bufs = [torch.empty_like(t) for t in real]
        return (W.Pipeline(nef, tr), nef, tr, bufs), {f"in{i}": (b, r, x) for i, (b, r, x) in enumerate(zip(bufs, real, other))}

    def run(st):
        pipe, nef, tr, (o, d, tgt) = st
        rb = pipe(rays=W.Rays(o, d, 0.0, 10.0), channels=["rgb"])
        ((rb.rgb - tgt) ** 2).mean().backward()
        return {"rgb": rb.rgb, "samples": torch.tensor([tr.get_prev_num_samples()]), **_grads(nef, tol)}
    ref = _route(build, run, tol)
    assert int(ref["samples"]) > 0
    print(f"ROUTE Pipeline precision {precision}: side stream == default stream ({int(ref['samples'])} samples)")


def test_route_multiview_step_next_rays(W):
    real, other = _rays_pair(40, 2)
    real2, other2 = _rays_pair(40, 3)

    def build():
        nef = _nerf(W)
        tr = W.PackedRFTracer('ray', 128, bg_color=(1.0, 1.0, 1.0)); tr.precision = 1
        ms = W.MultiviewStep(W.Pipeline(nef, tr), lr=1e-3, eps=1e-8)
        assert ms.fused
        bufs = [torch.empty_like(t) for t in real + real2]
        vals = list(zip(bufs, real + real2, other + other2))
        return (ms, nef, bufs), {f"in{i}": v for i, v in enumerate(vals)}

    def run(st):
        ms, nef, (o, d, tgt, o2, d2, tgt2) = st
        r1, r2 = W.Rays(o, d, 0.0, 10.0), W.Rays(o2, d2, 0.0, 10.0)
        l1 = ms.step(r1, tgt, seed=21, next_rays=r2, next_seed=22)          # premarches r2 on the tracer's side stream
        l2 = ms.step(r2, tgt2, seed=22)
        return {"loss1": l1.reshape(1), "loss2": l2.reshape(1), **{"param." + n: p for n, p in nef.named_parameters()}}
    tol = {"loss1": ROUTE_TOL_TC, "loss2": ROUTE_TOL_TC}
    tol.update({"param." + n: ROUTE_TOL_TC for n, _ in _nerf(W).named_parameters()})
    _route(build, run, tol)
    print("ROUTE MultiviewStep.step(next_rays=...): side stream == default stream")


def _sdf_coords(n, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, 3, generator=g) * 2.1 - 1.05
    return _dev(c), _dev(((c.abs().sum(-1, keepdim=True) - 0.5) / 3 ** 0.5))


@pytest.mark.parametrize("kind", ["octree", "hash"])
def test_route_sdf_step(W, kind):
    from test_gpu_sdf_step import _field

    def build():
        if kind == "octree":
            nef, _ = _field(W, "sum4")
        else:
            nef, case = _field(W, "sum4")
            torch.manual_seed(0)
            grid = W.HashGrid.from_geometric(nef.grid.blas, feature_dim=8, num_lods=4, multiscale_type="cat", feature_std=0.01,
                                             codebook_bitwidth=14, min_grid_res=16, max_grid_res=256)
            nef = W.NeuralSDF(grid, pos_embedder="none", position_input=True, hidden_dim=64, num_layers=1).cuda()
        step = W.SDFStep(W.Pipeline(nef))
        assert step.fused
        (c, g), (c2, g2) = _sdf_coords(8192, 1), _sdf_coords(8192, 2)
        bc, bg = torch.empty_like(c), torch.empty_like(g)
        return (step, nef, bc, bg), {"c": (bc, c, c2), "g": (bg, g, g2)}

    def run(st):
        step, nef, c, g = st
        loss = step.step(c, g)
        return {"loss": loss.reshape(1), **{"param." + n: p for n, p in nef.named_parameters()}}
    st, _ = build()
    tol = {"loss": ROUTE_TOL, **{"param." + n: ROUTE_TOL for n, _ in st[1].named_parameters()}}
    _route(build, run, tol)
    print(f"ROUTE SDFStep ({kind}): side stream == default stream")


def test_route_image_step(W):
    from test_gpu_image import make_field

    def build():
        nef = make_field(W, F=2, L=8, bw=14, max_res=256, H=64, seed=0)
        step = W.ImageStep(W.Pipeline(nef))
        g = torch.Generator().manual_seed(4)
        vals = [torch.rand(4096, 2, generator=g).cuda() * 2 - 1, torch.rand(4096, 3, generator=g).cuda()]
        oth = [torch.rand(4096, 2, generator=g).cuda() * 2 - 1, torch.rand(4096, 3, generator=g).cuda()]
        bufs = [torch.empty_like(t) for t in vals]
        return (step, nef, bufs), {f"in{i}": v for i, v in enumerate(zip(bufs, vals, oth))}

    def run(st):
        step, nef, (c, rgb) = st
        loss = step.step(c, rgb)
        return {"loss": loss.reshape(1), **{"param." + n: p for n, p in nef.named_parameters()}}
    st, _ = build()
    tol = {"loss": ROUTE_TOL, **{"param." + n: ROUTE_TOL for n, _ in st[1].named_parameters()}}
    _route(build, run, tol)
    print("ROUTE ImageStep: side stream == default stream")


@pytest.mark.parametrize("route", ["persistent", "phase"])
def test_route_packed_sdf_tracer(W, route):
    from test_gpu_sdf_tracer import _case, _config3, _frame, _sdf_like
    o, d = _frame(64, 0.75)
    o2, d2 = _frame(64, 0.6)

    def build():
        if route == "persistent":
            _, nef = _config3()
        else:
            case = _case()
            torch.manual_seed(0)
            grid = W.HashGrid.from_geometric(W.OctreeAS(_dev(case["octree"])), feature_dim=8, num_lods=4, multiscale_type="cat",
                                             feature_std=0.01, codebook_bitwidth=14, min_grid_res=16, max_grid_res=256)
            nef = _sdf_like(W.NeuralSDF(grid, pos_embedder="none", position_input=True, hidden_dim=64, num_layers=1).cuda(), 64)
        fd = W.ops.sdf_field(nef)
        assert fd is not None and (fd[1] is not None) == (route == "persistent")
        bo, bd = torch.empty_like(_dev(o)), torch.empty_like(_dev(d))
        return (nef, bo, bd), {"o": (bo, _dev(o), _dev(o2)), "d": (bd, _dev(d), _dev(d2))}

    def run(st):
        nef, bo, bd = st
        tracer = W.PackedSDFTracer(num_steps=32, step_size=0.8, min_dis=1e-3)
        rb = tracer(nef, rays=W.Rays(bo, bd, dist_min=0.0, dist_max=6.0), lod_idx=nef.grid.num_lods - 1 if route == "persistent" else 3,
                    channels=["depth", "hit", "xyz", "normal", "rgb", "alpha"])
        return {k: getattr(rb, k) for k in ("depth", "hit", "xyz", "normal", "rgb", "alpha")}
    # normal / rgb: finite differences through the torch decoder (autograd on), a cuBLAS GEMM whose kernel choice may follow the stream
    ref = _route(build, run, {"normal": ROUTE_TOL, "rgb": ROUTE_TOL})
    assert int(ref["hit"].sum()) > 0
    print(f"ROUTE PackedSDFTracer ({route}): side stream == default stream ({int(ref['hit'].sum())} hits)")


def test_route_packed_spc_tracer(W):
    import numpy as np
    from test_gpu_spc_trace import GOLDEN, golden_field
    z = np.load(GOLDEN)

    def build():
        nef, rays = golden_field(W, z, "octa5", "rgba")
        o, d = rays.origins, rays.dirs
        bo, bd = torch.empty_like(o), torch.empty_like(d)
        return (nef, bo, bd), {"o": (bo, o, torch.flip(o, [0])), "d": (bd, d, torch.flip(d, [0]))}

    def run(st):
        nef, bo, bd = st
        rb = W.PackedSPCTracer()(nef, W.Rays(bo, bd))
        return {k: getattr(rb, k) for k in ("depth", "hit", "rgb", "alpha")}
    _route(build, run, {})
    print("ROUTE PackedSPCTracer: side stream == default stream")


def _mesh(seed, T=300):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(3 * T, 3, generator=g) * 1.6 - 0.8
    return _dev(V), _dev(torch.arange(3 * T).reshape(T, 3), torch.int64)


def test_route_compute_sdf_and_mesh_to_octree(W):
    (V, F), (V2, _) = _mesh(1), _mesh(2)
    g = torch.Generator().manual_seed(3)
    P, P2 = _dev(torch.rand(5000, 3, generator=g, dtype=torch.float64) * 2 - 1), _dev(torch.rand(5000, 3, generator=g, dtype=torch.float64) * 2 - 1)

    def build():
        bv, bp = torch.empty_like(V), torch.empty_like(P)
        return (bv, bp), {"V": (bv, V, V2), "P": (bp, P, P2)}

    def run(st):
        bv, bp = st
        return {"sdf": W.compute_sdf(bv.double(), F, bp), "octree": W.mesh_to_octree(bv, F, 5, 10 ** 5, seed=9)}
    _route(build, run, {})
    print("ROUTE compute_sdf, mesh_to_octree: side stream == default stream")


def test_route_prune(W):
    def build():
        nef = _nerf(W)
        t = nef.grid.codebook.feats
        g = torch.Generator().manual_seed(8)
        return nef, {"table": (t, t.detach().clone(), (torch.randn(t.shape, generator=g) * 0.3).cuda())}

    def run(nef):
        nef.prune(seed=5)
        return {"occupancy": nef.grid.occupancy, "octree": nef.grid.blas.octree}
    _route(build, run, {})
    print("ROUTE NeuralRadianceField.prune: side stream == default stream")
