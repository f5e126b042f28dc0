"""One case per stream-taking entry point of the C ABI (include/wispb200.h): every prototype whose last parameter is `wb_stream s`.

A case builds, on the device, the static buffers one call reads and writes, two VALID value sets for them of the same shapes (the
real set and the "poison": another seed, other rays, other table values; accumulate-into outputs zeroed as part of the set), and the
call itself over those buffers.  tests/test_gpu_stream_contract.py runs each call gated behind a sleep on a side stream and inside a
CUDA graph; a launch that escapes the caller's stream runs on the poison and changes the result.

Nothing here touches CUDA at import: tests/test_stream_contract_cpu.py checks the registry against the header on a machine
without a GPU.  Shared constants (octrees, their prefix sums and points) are the same in both sets: every call also reads an input
that differs.

Buffer naming: `outputs` maps each compared buffer to None (must match bit for bit) or to a relative tolerance (max |a - b| over
max |reference|) for buffers accumulated with atomics, whose summation order is free.
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, Dict, Optional

# Relative tolerances (max |a - b| / max |reference|) of atomically accumulated fp32 outputs: the summation order of float atomics
# is free, which moves a sum by a few ulps of its largest partial sums.  The precision-1 table gradient adds fp16-rounded dL/dfeat
# values; tests/test_gpu_tc_decoders.py compares such sums at 3e-2 across schedules, here the schedule is the same and only the
# atomic order moves.
ATOMIC = 1e-5
ATOMIC_TC = 1e-4


@dataclass
class Built:
    bufs: Dict[str, "object"]                     # name -> static device tensor the call reads or writes
    real: Dict[str, "object"]                     # name -> value of the real set (every key of bufs that is not a shared constant)
    poison: Dict[str, "object"]                   # name -> value of the poison set, same shapes
    outputs: Dict[str, Optional[float]]           # compared buffers: None = bit-exact, float = relative tolerance
    call: Callable[[int], None]                   # call(stream handle): one call of the entry point on that stream
    host_inputs: bool = False                     # the call reads no device input: an escaped launch is caught by the re-initialised
                                                  # outputs (the sensitivity check compares with those instead of the poison result)
    keep: list = field(default_factory=list)      # descriptors and host arrays the call's pointers live in


CASES: Dict[str, Callable] = {}


def case(name):
    def deco(fn):
        assert name not in CASES, name
        CASES[name] = fn
        return fn
    return deco


# ------------------------------------------------------------------------------------------------------------------------------
# shared helpers (device work only inside builders)
# ------------------------------------------------------------------------------------------------------------------------------
def _t():
    import torch
    return torch


def _A():
    import wisp_b200
    return wisp_b200._cabi


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _pp(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _split(bufs, sets):
    """sets: name -> (real value, poison value); the static buffer is a clone of the real value."""
    for k, (r, _) in sets.items():
        bufs[k] = r.clone()
    return {k: v[0] for k, v in sets.items()}, {k: v[1] for k, v in sets.items()}


def _rays(R, seed, dev="cuda"):
    """Rays from a sphere of radius 2.5 towards points inside [-0.7, 0.7]^3: most cross the octree scenes below."""
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g)
    o = o / o.norm(dim=1, keepdim=True) * 2.5
    tgt = (torch.rand(R, 3, generator=g) * 1.4 - 0.7)
    d = tgt - o
    d = d / d.norm(dim=1, keepdim=True)
    return o.float().to(dev).contiguous(), d.float().to(dev).contiguous()


def _rays_desc(o, d, near=0.0, far=6.0):
    r = _A().RaysDesc()
    r.origins, r.dirs, r.num_rays, r.dist_min, r.dist_max, r.near_v, r.far_v = o.data_ptr(), d.data_ptr(), o.shape[0], near, far, None, None
    return r


_OCT = {}
OCT_LEVEL = 5


def _octree():
    """A sparse level-5 octree (a shell plus scattered cells) with its dense bitmask and coarse mask, built once per process."""
    if "oct" not in _OCT:
        torch = _t()
        import wisp_b200 as W
        from wisp_b200 import ops
        g = torch.Generator().manual_seed(7)
        n = 2 ** OCT_LEVEL
        ijk = torch.stack(torch.meshgrid(*[torch.arange(n)] * 3, indexing="ij"), -1).reshape(-1, 3)
        c = (ijk.float() + 0.5) / n * 2 - 1
        r = c.norm(dim=1)
        keep = ((r > 0.45) & (r < 0.65)) | (torch.rand(ijk.shape[0], generator=g) < 0.05)
        blas = W.OctreeAS.from_quantized_points(ijk[keep].short().cuda(), OCT_LEVEL)
        oct = ops.octree_tensors(blas)
        oct.ensure_bits(OCT_LEVEL)
        _OCT["oct"], _OCT["blas"] = oct, blas
    return _OCT["oct"]


def _level_points(oct, level):
    s, c = int(oct.pyramid[1, level]), int(oct.pyramid[0, level])
    return oct.points[s:s + c].contiguous()


def _scan(counts):
    torch = _t()
    A = _A(); L = A.lib()
    n = counts.shape[0]
    off = torch.empty(n + 1, dtype=torch.int64, device=counts.device)
    wsb = int(L.wb_scan_workspace_bytes(n))
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=counts.device)
    L.wb_scan_counts(_p(counts), n, _p(off), _p(ws), wsb, 0)
    torch.cuda.synchronize()
    return off


R_OCT = 384
MARCH_N = 32


def _march_set(oct, seed):
    """count -> scan of the ray marcher for one ray set: rays, hitmask, offsets."""
    torch = _t()
    A = _A(); L = A.lib()
    o, d = _rays(R_OCT, seed)
    rays = _rays_desc(o, d)
    words = (MARCH_N + 31) // 32
    hm = torch.zeros(R_OCT, words, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(R_OCT, dtype=torch.int32, device="cuda")
    L.wb_raymarch_ray_count(oct.desc(), OCT_LEVEL, rays, MARCH_N, None, 3, _p(hm), _p(cnt), 0)
    return dict(o=o, d=d, hm=hm, off=_scan(cnt), cnt=cnt)


def _trace_set(oct, seed):
    """raytrace count -> scan -> fill for one ray set: rays, counts, offsets, nuggets."""
    torch = _t()
    A = _A(); L = A.lib()
    o, d = _rays(R_OCT, seed)
    rays = _rays_desc(o, d)
    cnt = torch.zeros(R_OCT, dtype=torch.int32, device="cuda")
    L.wb_raytrace_count(oct.desc(), OCT_LEVEL, rays, _p(cnt), 0)
    off = _scan(cnt)
    Ng = int(off[-1])
    ridx = torch.zeros(Ng, dtype=torch.int32, device="cuda"); pidx = torch.zeros_like(ridx)
    depth = torch.zeros(Ng, 2, dtype=torch.float32, device="cuda")
    L.wb_raytrace_fill(oct.desc(), OCT_LEVEL, rays, _p(off), _p(ridx), _p(pidx), _p(depth), 0)
    torch.cuda.synchronize()
    return dict(o=o, d=d, cnt=cnt, off=off, ridx=ridx, pidx=pidx, depth=depth, Ng=Ng)


def _outs(sets, names, shape_dtype, poison_fill=3):
    """Pure outputs: zeros in the real set, `poison_fill` in the poison set."""
    torch = _t()
    for n in names:
        shape, dt = shape_dtype[n]
        sets[n] = (torch.zeros(shape, dtype=dt, device="cuda"), torch.full(shape, poison_fill, dtype=dt, device="cuda"))


# ------------------------------------------------------------------------------------------------------------------------------
# SPC helpers, marcher, raytrace
# ------------------------------------------------------------------------------------------------------------------------------
COARSE_LEVEL = 4


def _bits_case(coarse):
    torch = _t()
    oct = _octree()
    lp = _level_points(oct, OCT_LEVEL)
    g = torch.Generator().manual_seed(11)
    # the poison: as many cells, all in one corner (the dilated coarse mask of the scene covers nearly every coarse cell)
    lp2 = torch.randint(0, 2 ** (OCT_LEVEL - 2), lp.shape, generator=g).short().cuda()
    words = (8 ** (COARSE_LEVEL if coarse else OCT_LEVEL) + 31) // 32
    sets = {"pts": (lp, lp2), "bits": (torch.zeros(words, dtype=torch.int32, device="cuda"),) * 2}
    bufs = {}
    real, poison = _split(bufs, sets)
    A = _A(); L = A.lib(); n = lp.shape[0]
    if coarse:
        call = lambda s: L.wb_octree_build_coarse(_p(bufs["pts"]), n, OCT_LEVEL, COARSE_LEVEL, _p(bufs["bits"]), s)
    else:
        call = lambda s: L.wb_octree_build_bits(_p(bufs["pts"]), n, OCT_LEVEL, _p(bufs["bits"]), s)
    return Built(bufs, real, poison, {"bits": None}, call)


@case("wb_octree_build_bits")
def _c_bits():
    return _bits_case(False)


@case("wb_octree_build_coarse")
def _c_coarse():
    return _bits_case(True)


@case("wb_query")
def _c_query():
    torch = _t()
    oct = _octree(); L = _A().lib()
    N = 4096
    g = torch.Generator().manual_seed(5)
    sets = {"x": ((torch.rand(N, 3, generator=g) * 2.2 - 1.1).cuda(), (torch.rand(N, 3, generator=g) * 2.2 - 1.1).cuda())}
    _outs(sets, ["out"], {"out": ((N, OCT_LEVEL + 1), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    od = oct.desc()
    return Built(bufs, real, poison, {"out": None},
                 lambda s: L.wb_query(od, _p(bufs["x"]), N, OCT_LEVEL, 1, _p(bufs["out"]), s), keep=[od])


@case("wb_raymarch_ray_count")
def _c_ray_count():
    torch = _t()
    oct = _octree(); L = _A().lib()
    r0, r1 = _rays(R_OCT, 1), _rays(R_OCT, 2)
    sets = {"o": (r0[0], r1[0]), "d": (r0[1], r1[1])}
    _outs(sets, ["hm", "cnt"], {"hm": ((R_OCT, 1), torch.int32), "cnt": ((R_OCT,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    od, rays = oct.desc(), _rays_desc(bufs["o"], bufs["d"])
    return Built(bufs, real, poison, {"hm": None, "cnt": None},
                 lambda s: L.wb_raymarch_ray_count(od, OCT_LEVEL, rays, MARCH_N, None, 3, _p(bufs["hm"]), _p(bufs["cnt"]), s), keep=[od, rays])


@case("wb_scan_counts")
def _c_scan():
    torch = _t()
    L = _A().lib()
    R = 300_000                      # several chunks: all three scan kernels run
    g = torch.Generator().manual_seed(3)
    wsb = int(L.wb_scan_workspace_bytes(R))
    sets = {"cnt": (torch.randint(0, 40, (R,), generator=g, dtype=torch.int32).cuda(), torch.randint(0, 40, (R,), generator=g, dtype=torch.int32).cuda()),
            "ws": (torch.zeros(wsb, dtype=torch.uint8, device="cuda"), torch.full((wsb,), 1, dtype=torch.uint8, device="cuda"))}
    _outs(sets, ["off"], {"off": ((R + 1,), torch.int64)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"off": None},
                 lambda s: L.wb_scan_counts(_p(bufs["cnt"]), R, _p(bufs["off"]), _p(bufs["ws"]), wsb, s))


def _fill_sets(sa, sb, keys):
    return {k: (sa[k], sb[k]) for k in keys}


@case("wb_raymarch_ray_fill")
def _c_ray_fill():
    torch = _t()
    oct = _octree(); L = _A().lib()
    a, b = _march_set(oct, 1), _march_set(oct, 2)
    cap = max(int(a["off"][-1]), int(b["off"][-1]), 1)
    sets = _fill_sets(a, b, ["o", "d", "hm", "off"])
    _outs(sets, ["ridx", "x", "depth", "deltas", "bnd"],
          {"ridx": ((cap,), torch.int64), "x": ((cap, 3), torch.float32), "depth": ((cap, 1), torch.float32),
           "deltas": ((cap, 1), torch.float32), "bnd": ((cap,), torch.uint8)})
    bufs = {}
    real, poison = _split(bufs, sets)
    rays = _rays_desc(bufs["o"], bufs["d"])
    return Built(bufs, real, poison, dict.fromkeys(["ridx", "x", "depth", "deltas", "bnd"]),
                 lambda s: L.wb_raymarch_ray_fill(rays, MARCH_N, None, 3, _p(bufs["hm"]), _p(bufs["off"]), _p(bufs["ridx"]), _p(bufs["x"]),
                                                  _p(bufs["depth"]), _p(bufs["deltas"]), _p(bufs["bnd"]), s), keep=[rays])


@case("wb_rf_march_fill")
def _c_rf_march_fill():
    torch = _t()
    oct = _octree(); L = _A().lib()
    a, b = _march_set(oct, 1), _march_set(oct, 2)
    cap = max(int(a["off"][-1]), int(b["off"][-1]), 1)
    sets = _fill_sets(a, b, ["o", "d", "hm", "off"])
    _outs(sets, ["t", "dt", "ray"], {"t": ((cap,), torch.float32), "dt": ((cap,), torch.float32), "ray": ((cap,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    rays = _rays_desc(bufs["o"], bufs["d"])
    return Built(bufs, real, poison, dict.fromkeys(["t", "dt", "ray"]),
                 lambda s: L.wb_rf_march_fill(rays, MARCH_N, None, 3, _p(bufs["hm"]), _p(bufs["off"]), _p(bufs["t"]), _p(bufs["dt"]),
                                              _p(bufs["ray"]), s), keep=[rays])


def _rt_count_case(cached):
    torch = _t()
    oct = _octree(); A = _A(); L = A.lib()
    r0, r1 = _rays(R_OCT, 1), _rays(R_OCT, 2)
    sets = {"o": (r0[0], r1[0]), "d": (r0[1], r1[1])}
    K = 4
    shapes = {"cnt": ((R_OCT,), torch.int32)}
    if cached:
        shapes["cache"] = ((int(L.wb_raytrace_cache_bytes(R_OCT, K)),), torch.uint8)
    _outs(sets, list(shapes), shapes)
    bufs = {}
    real, poison = _split(bufs, sets)
    od, rays = oct.desc(), _rays_desc(bufs["o"], bufs["d"])
    if cached:
        call = lambda s: L.wb_raytrace_count_cached(od, OCT_LEVEL, rays, _p(bufs["cnt"]), _p(bufs["cache"]), K, s)
    else:
        call = lambda s: L.wb_raytrace_count(od, OCT_LEVEL, rays, _p(bufs["cnt"]), s)
    return Built(bufs, real, poison, {"cnt": None}, call, keep=[od, rays])


@case("wb_raytrace_count")
def _c_rt_count():
    return _rt_count_case(False)


@case("wb_raytrace_count_cached")
def _c_rt_count_cached():
    return _rt_count_case(True)


def _rt_fill_case(cached):
    torch = _t()
    oct = _octree(); A = _A(); L = A.lib()
    a, b = _trace_set(oct, 1), _trace_set(oct, 2)
    cap = max(a["Ng"], b["Ng"], 1)
    K = 4
    sets = _fill_sets(a, b, ["o", "d", "off"])
    if cached:
        cb = int(L.wb_raytrace_cache_bytes(R_OCT, K))
        for st in (a, b):                       # the cache the count pass leaves for this ray set
            st["cache"] = torch.zeros(cb, dtype=torch.uint8, device="cuda")
            L.wb_raytrace_count_cached(oct.desc(), OCT_LEVEL, _rays_desc(st["o"], st["d"]), _p(torch.zeros_like(st["cnt"])), _p(st["cache"]), K, 0)
        sets["cache"] = (a["cache"], b["cache"])
    _outs(sets, ["ridx", "pidx", "depth"], {"ridx": ((cap,), torch.int32), "pidx": ((cap,), torch.int32), "depth": ((cap, 2), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    od, rays = oct.desc(), _rays_desc(bufs["o"], bufs["d"])
    if cached:
        call = lambda s: L.wb_raytrace_fill_cached(od, OCT_LEVEL, rays, _p(bufs["off"]), _p(bufs["cache"]), K, _p(bufs["ridx"]), _p(bufs["pidx"]),
                                                   _p(bufs["depth"]), s)
    else:
        call = lambda s: L.wb_raytrace_fill(od, OCT_LEVEL, rays, _p(bufs["off"]), _p(bufs["ridx"]), _p(bufs["pidx"]), _p(bufs["depth"]), s)
    return Built(bufs, real, poison, dict.fromkeys(["ridx", "pidx", "depth"]), call, keep=[od, rays])


@case("wb_raytrace_fill")
def _c_rt_fill():
    return _rt_fill_case(False)


@case("wb_raytrace_fill_cached")
def _c_rt_fill_cached():
    return _rt_fill_case(True)


def _nugget_sets():
    """Two raytrace results cut to the same nugget count (a prefix of each ray-ordered list is itself a valid nugget list), with the
    per-ray nugget offsets of the cut lists."""
    torch = _t()
    oct = _octree()
    a, b = _trace_set(oct, 1), _trace_set(oct, 2)
    Ng = min(a["Ng"], b["Ng"])
    for st in (a, b):
        st["ridx"], st["depth"] = st["ridx"][:Ng].contiguous(), st["depth"][:Ng].contiguous()
        cnt = torch.bincount(st["ridx"].long(), minlength=R_OCT)
        st["roff"] = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), cnt.cumsum(0)])
    return a, b, Ng


@case("wb_raymarch_voxel_fill")
def _c_voxel_fill():
    torch = _t()
    L = _A().lib()
    a, b, Ng = _nugget_sets()
    n = 4
    S = Ng * n
    sets = _fill_sets(a, b, ["o", "d", "ridx", "depth"])
    _outs(sets, ["sridx", "x", "sd", "dl", "bnd", "rr"],
          {"sridx": ((S,), torch.int64), "x": ((S, 3), torch.float32), "sd": ((S, 1), torch.float32), "dl": ((S, 1), torch.float32),
           "bnd": ((S,), torch.uint8), "rr": ((S,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    rays = _rays_desc(bufs["o"], bufs["d"])
    return Built(bufs, real, poison, dict.fromkeys(["sridx", "x", "sd", "dl", "bnd", "rr"]),
                 lambda s: L.wb_raymarch_voxel_fill(rays, _p(bufs["ridx"]), _p(bufs["depth"]), Ng, n, None, 9, _p(bufs["sridx"]), _p(bufs["x"]),
                                                    _p(bufs["sd"]), _p(bufs["dl"]), _p(bufs["bnd"]), _p(bufs["rr"]), s), keep=[rays])


UNIFORM_SCALE = 10


@case("wb_raymarch_uniform_count")
def _c_uniform_count():
    torch = _t()
    L = _A().lib()
    a, b, Ng = _nugget_sets()
    sets = _fill_sets(a, b, ["depth"])
    _outs(sets, ["cnt"], {"cnt": ((Ng,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"cnt": None},
                 lambda s: L.wb_raymarch_uniform_count(_p(bufs["depth"]), Ng, UNIFORM_SCALE, _p(bufs["cnt"]), s))


@case("wb_raymarch_uniform_fill")
def _c_uniform_fill():
    torch = _t()
    L = _A().lib()
    a, b, Ng = _nugget_sets()
    for st in (a, b):
        cnt = torch.zeros(Ng, dtype=torch.int32, device="cuda")
        L.wb_raymarch_uniform_count(_p(st["depth"]), Ng, UNIFORM_SCALE, _p(cnt), 0)
        st["soff"] = _scan(cnt)
    cap = max(int(a["soff"][-1]), int(b["soff"][-1]), 1)
    sets = _fill_sets(a, b, ["o", "d", "ridx", "depth", "soff", "roff"])
    _outs(sets, ["sridx", "x", "sd", "dl", "bnd", "rr"],
          {"sridx": ((cap,), torch.int64), "x": ((cap, 3), torch.float32), "sd": ((cap, 1), torch.float32), "dl": ((cap, 1), torch.float32),
           "bnd": ((cap,), torch.uint8), "rr": ((cap,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    rays = _rays_desc(bufs["o"], bufs["d"])
    return Built(bufs, real, poison, dict.fromkeys(["sridx", "x", "sd", "dl", "bnd", "rr"]),
                 lambda s: L.wb_raymarch_uniform_fill(rays, _p(bufs["ridx"]), _p(bufs["depth"]), Ng, UNIFORM_SCALE, _p(bufs["soff"]), _p(bufs["roff"]),
                                                      _p(bufs["sridx"]), _p(bufs["x"]), _p(bufs["sd"]), _p(bufs["dl"]), _p(bufs["bnd"]), _p(bufs["rr"]), s),
                 keep=[rays])


@case("wb_find_depth_bound")
def _c_find_depth_bound():
    torch = _t()
    L = _A().lib()
    a, b, Ng = _nugget_sets()
    for k, st in (("a", a), ("b", b)):
        starts = st["roff"][:-1]
        has = st["roff"][1:] > starts
        st["curr"] = torch.where(has, starts, torch.full_like(starts, -1)).int().contiguous()
        g = torch.Generator(device="cuda").manual_seed(4 if k == "a" else 5)
        st["q"] = (torch.rand(R_OCT, 1, device="cuda", generator=g) * 5.0).contiguous()
    sets = _fill_sets(a, b, ["q", "curr", "depth"])
    _outs(sets, ["out"], {"out": ((R_OCT,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"out": None},
                 lambda s: L.wb_find_depth_bound(_p(bufs["q"]), _p(bufs["curr"]), _p(bufs["depth"]), R_OCT, Ng, _p(bufs["out"]), s))


@case("wb_spc_trace")
def _c_spc_trace():
    torch = _t()
    oct = _octree(); L = _A().lib()
    r0, r1 = _rays(R_OCT, 1), _rays(R_OCT, 2)
    npts = int(oct.pyramid[0, OCT_LEVEL])
    off = int(oct.pyramid[1, OCT_LEVEL])
    g = torch.Generator().manual_seed(8)
    sets = {"o": (r0[0], r1[0]), "d": (r0[1], r1[1]),
            "col": (torch.rand(npts, 4, generator=g).cuda(), torch.rand(npts, 4, generator=g).cuda())}
    _outs(sets, ["depth", "hit", "rgb", "alpha"], {"depth": ((R_OCT,), torch.float32), "hit": ((R_OCT,), torch.uint8),
                                                         "rgb": ((R_OCT, 3), torch.float32), "alpha": ((R_OCT,), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    od, rays = oct.desc(), _rays_desc(bufs["o"], bufs["d"])
    return Built(bufs, real, poison, dict.fromkeys(["depth", "hit", "rgb", "alpha"]),
                 lambda s: L.wb_spc_trace(od, OCT_LEVEL, rays, _p(bufs["col"]), 4, off, _p(bufs["depth"]), _p(bufs["hit"]), _p(bufs["rgb"]),
                                          _p(bufs["alpha"]), s), keep=[od, rays])


# ------------------------------------------------------------------------------------------------------------------------------
# prune
# ------------------------------------------------------------------------------------------------------------------------------
@case("wb_prune_samples")
def _c_prune_samples():
    torch = _t()
    oct = _octree(); L = _A().lib()
    pts = _level_points(oct, OCT_LEVEL)
    N = pts.shape[0]
    g = torch.Generator().manual_seed(12)
    sets = {"pts": (pts, torch.randint(0, 2 ** OCT_LEVEL, (N, 3), generator=g).short().cuda()),
            "u": (torch.rand(N, 3, generator=g).cuda(), torch.rand(N, 3, generator=g).cuda())}
    _outs(sets, ["x", "dirs", "t", "ray"], {"x": ((N, 3), torch.float32), "dirs": ((N, 3), torch.float32), "t": ((N,), torch.float32),
                                                   "ray": ((N,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, dict.fromkeys(["x", "dirs", "t", "ray"]),
                 lambda s: L.wb_prune_samples(_p(bufs["pts"]), N, OCT_LEVEL, _p(bufs["u"]), 0, _p(bufs["x"]), _p(bufs["dirs"]), _p(bufs["t"]),
                                              _p(bufs["ray"]), s))


@case("wb_prune_update")
def _c_prune_update():
    torch = _t()
    L = _A().lib()
    N = 5000
    g = torch.Generator().manual_seed(13)
    sets = {"sh": (torch.rand(N, 4, generator=g).cuda() * 0.02, torch.rand(N, 4, generator=g).cuda() * 0.02),
            "occ": (torch.rand(N, generator=g).cuda() * 0.02, torch.rand(N, generator=g).cuda() * 0.02)}
    _outs(sets, ["keep"], {"keep": ((N,), torch.uint8)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"occ": None, "keep": None},
                 lambda s: L.wb_prune_update(_p(bufs["sh"]), N, 0.7, 0.01, _p(bufs["occ"]), _p(bufs["keep"]), s))


# ------------------------------------------------------------------------------------------------------------------------------
# hash grid, radiance-field shading (the Setup of tests/test_gpu_tc_decoders.py, seeds 0 and 1)
# ------------------------------------------------------------------------------------------------------------------------------
def _tc_setups(name="w64", **kw):
    import wisp_b200 as W
    from test_gpu_tc_decoders import Case, Setup
    base = dict(dens_hidden=[64], col_hidden=[64, 64], view=(3, 4), L=16, S=3000, R=200)
    base.update(kw)
    return Setup(W, Case(name, **base, seed=0)), Setup(W, Case(name, **base, seed=1))


def _nef_sets(a, b):
    """The parameter / ray / sample buffers of two Setups; the static buffers are a's own tensors (its descriptors point at them)."""
    return {"table": (a.t_table, b.t_table), "fd": (a.t_fd, b.t_fd), "fc": (a.t_fc, b.t_fc),
            "o": (a.rkeep[0], b.rkeep[0]), "d": (a.rkeep[1], b.rkeep[1]),
            "rt": (a.t_rec_t, b.t_rec_t), "rr": (a.t_rec_ray, b.t_rec_ray)}


def _adopt(a, sets, outs=()):
    """bufs = a's tensors for the shared keys (a's descriptors point at them), fresh clones for the rest."""
    bufs = {"table": a.t_table, "fd": a.t_fd, "fc": a.t_fc, "o": a.rkeep[0], "d": a.rkeep[1], "rt": a.t_rec_t, "rr": a.t_rec_ray}
    bufs = {k: v for k, v in bufs.items() if k in sets}
    real = {k: v[0].clone() for k, v in sets.items()}
    poison = {k: v[1] for k, v in sets.items()}
    for k, (r, _) in sets.items():
        if k not in bufs:
            bufs[k] = r.clone()
    return bufs, real, poison


def _g_shaded(S, seed):
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(S, 4, generator=g) * 1e-2).cuda()


def _hg_coords(N, seed):
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(N, 3, generator=g) * 2 - 1).cuda()


@case("wb_hashgrid_fwd")
def _c_hashgrid_fwd():
    torch = _t()
    a, b = _tc_setups()
    N = 3000
    sets = {"table": (a.t_table, b.t_table), "x": (_hg_coords(N, 1), _hg_coords(N, 2))}
    _outs(sets, ["feats"], {"feats": ((N, a.c.L * a.c.F), torch.float32)})
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"feats": None}, lambda s: L.wb_hashgrid_fwd(_p(bufs["x"]), N, a.desc, _p(bufs["feats"]), s), keep=[a, b])


@case("wb_hashgrid_bwd")
def _c_hashgrid_bwd():
    torch = _t()
    a, b = _tc_setups()
    N = 3000
    W_ = a.c.L * a.c.F
    g = torch.Generator().manual_seed(3)
    sets = {"x": (_hg_coords(N, 1), _hg_coords(N, 2)), "gf": (torch.randn(N, W_, generator=g).cuda(), torch.randn(N, W_, generator=g).cuda()),
            "gt": (torch.zeros_like(a.t_table), torch.zeros_like(a.t_table))}
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"gt": ATOMIC}, lambda s: L.wb_hashgrid_bwd(_p(bufs["x"]), N, a.desc, _p(bufs["gf"]), _p(bufs["gt"]), s),
                 keep=[a, b])


@case("wb_rf_pack_params")
def _c_pack():
    torch = _t()
    a, b = _tc_setups()
    sets = {"fd": (a.t_fd, b.t_fd), "fc": (a.t_fc, b.t_fc)}
    _outs(sets, ["blob"], {"blob": (tuple(a.blob.shape), torch.float32)})
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"blob": None}, lambda s: L.wb_rf_pack_params(a.desc, 1, _p(bufs["blob"]), s), keep=[a, b])


def _fwd_state(st, precision=1):
    """blob (packed for `precision`), the forward's saved rows and the per-ray rows of one Setup."""
    torch = _t()
    A = st.A; L = st.L
    blob = torch.empty(int(L.wb_rf_param_blob_floats(st.desc, precision)), dtype=torch.float32, device="cuda")
    L.wb_rf_pack_params(st.desc, precision, _p(blob), 0)
    shaded = torch.zeros(st.S, 4, device="cuda")
    feat = torch.zeros_like(st.feat); ws = torch.zeros_like(st.ws)
    L.wb_rf_shade_fwd(st.desc, _p(blob), precision, st.rays, _p(st.t_rec_t), _p(st.t_rec_ray), st.S, _p(shaded),
                      _p(feat) if precision else None, _p(ws) if precision else None, 0)
    torch.cuda.synchronize()
    return blob, feat, ws, shaded


@case("wb_rf_shade_fwd")
def _c_shade_fwd():
    torch = _t()
    a, b = _tc_setups()
    sets = _nef_sets(a, b)
    sets["blob"] = (_fwd_state(a)[0], _fwd_state(b)[0])
    _outs(sets, ["sh", "feat", "ws"], {"sh": ((a.S, 4), torch.float32), "feat": (tuple(a.feat.shape), torch.uint8),
                                             "ws": (tuple(a.ws.shape), torch.uint8)})
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"sh": None, "feat": None},
                 lambda s: L.wb_rf_shade_fwd(a.desc, _p(bufs["blob"]), 1, a.rays, _p(bufs["rt"]), _p(bufs["rr"]), a.S, _p(bufs["sh"]), _p(bufs["feat"]),
                                             _p(bufs["ws"]), s), keep=[a, b])


def _bwd_sets(a, b):
    torch = _t()
    sa, sb = _fwd_state(a), _fwd_state(b)
    sets = _nef_sets(a, b)
    sets["blob"], sets["feat"], sets["ws"] = (sa[0], sb[0]), (sa[1], sb[1]), (sa[2], sb[2])
    sets["g"] = (_g_shaded(a.S, 1), _g_shaded(a.S, 2))
    sets["scale"] = (torch.tensor([256.0], device="cuda"), torch.tensor([512.0], device="cuda"))
    for k, t in (("gd", a.t_fd), ("gc", a.t_fc), ("gt", a.t_table)):
        sets[k] = (torch.zeros_like(t), torch.zeros_like(t))
    return sets


@case("wb_rf_shade_bwd")
def _c_shade_bwd():
    a, b = _tc_setups()
    sets = _bwd_sets(a, b)
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"gd": ATOMIC_TC, "gc": ATOMIC_TC, "gt": ATOMIC_TC},
                 lambda s: L.wb_rf_shade_bwd(a.desc, _p(bufs["blob"]), 1, a.rays, _p(bufs["rt"]), _p(bufs["rr"]), a.S, _p(bufs["g"]), _p(bufs["scale"]),
                                             _p(bufs["feat"]), _p(bufs["ws"]), _p(bufs["gt"]), _p(bufs["gd"]), _p(bufs["gc"]), s), keep=[a, b])


@case("wb_rf_decoder_bwd")
def _c_decoder_bwd():
    a, b = _tc_setups()
    sets = _bwd_sets(a, b)
    del sets["gt"]
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"gd": ATOMIC_TC, "gc": ATOMIC_TC},
                 lambda s: L.wb_rf_decoder_bwd(a.desc, _p(bufs["blob"]), a.rays, _p(bufs["rt"]), _p(bufs["rr"]), a.S, _p(bufs["g"]), _p(bufs["scale"]),
                                               _p(bufs["feat"]), _p(bufs["ws"]), _p(bufs["gd"]), _p(bufs["gc"]), s), keep=[a, b])


@case("wb_rf_table_scatter")
def _c_table_scatter():
    torch = _t()
    a, b = _tc_setups()
    sets = _bwd_sets(a, b)
    for st, i in ((a, 0), (b, 1)):        # the dL/dfeat planes the decoder backward leaves in the workspace
        gd, gc = torch.zeros_like(st.t_fd), torch.zeros_like(st.t_fc)
        st.L.wb_rf_decoder_bwd(st.desc, _p(sets["blob"][i]), st.rays, _p(st.t_rec_t), _p(st.t_rec_ray), st.S, _p(sets["g"][i]), _p(sets["scale"][i]),
                               _p(sets["feat"][i]), _p(sets["ws"][i]), _p(gd), _p(gc), 0)
    torch.cuda.synchronize()
    sets = {k: sets[k] for k in ("o", "d", "rt", "rr", "scale", "ws", "gt")}
    bufs, real, poison = _adopt(a, sets)
    L = a.L
    return Built(bufs, real, poison, {"gt": ATOMIC_TC},
                 lambda s: L.wb_rf_table_scatter(a.desc, a.rays, _p(bufs["rt"]), _p(bufs["rr"]), a.S, _p(bufs["scale"]), _p(bufs["ws"]), _p(bufs["gt"]), s),
                 keep=[a, b])


@case("wb_rf_loss_scale")
def _c_loss_scale():
    torch = _t()
    L = _A().lib()
    sets = {"am": (torch.tensor([0.37], device="cuda"), torch.tensor([5.0e-4], device="cuda"))}
    _outs(sets, ["scale"], {"scale": ((1,), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"scale": None}, lambda s: L.wb_rf_loss_scale(_p(bufs["am"]), _p(bufs["scale"]), s))


# ------------------------------------------------------------------------------------------------------------------------------
# compositing
# ------------------------------------------------------------------------------------------------------------------------------
R_COMP = 500


def _comp_set(seed):
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    S = 2500                                  # the same sample count in both sets, spread unevenly over the rays (some get none)
    cnt = torch.bincount(torch.randint(0, R_COMP, (S,), generator=g) // 3 * 3, minlength=R_COMP)
    off = torch.cat([torch.zeros(1, dtype=torch.int64), cnt.cumsum(0)])
    depth = torch.zeros(S, 1)
    for r in range(R_COMP):
        n = int(cnt[r])
        if n:
            depth[int(off[r]):int(off[r + 1]), 0] = torch.sort(torch.rand(n, generator=g) * 4)[0]
    sh = torch.rand(S, 4, generator=g); sh[:, 3] *= 8
    return dict(sh=sh.cuda(), depth=depth.cuda(), deltas=(torch.rand(S, 1, generator=g) * 0.1).cuda(), off=off.cuda(),
                grgb=torch.randn(R_COMP, 3, generator=g).cuda(), gdep=torch.randn(R_COMP, 1, generator=g).cuda(),
                galp=torch.randn(R_COMP, 1, generator=g).cuda(), tgt=torch.rand(R_COMP, 3, generator=g).cuda(),
                rgb=torch.rand(R_COMP, 3, generator=g).cuda())


BG = (C.c_float * 3)(0.25, 0.5, 1.0)


@case("wb_composite_fwd")
def _c_comp_fwd():
    torch = _t()
    L = _A().lib()
    a, b = _comp_set(1), _comp_set(2)
    sets = _fill_sets(a, b, ["sh", "depth", "deltas", "off"])
    _outs(sets, ["rgb", "dout", "alpha", "hit"], {"rgb": ((R_COMP, 3), torch.float32), "dout": ((R_COMP, 1), torch.float32),
                                                        "alpha": ((R_COMP, 1), torch.float32), "hit": ((R_COMP,), torch.uint8)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, dict.fromkeys(["rgb", "dout", "alpha", "hit"]),
                 lambda s: L.wb_composite_fwd(_p(bufs["sh"]), _p(bufs["depth"]), _p(bufs["deltas"]), _p(bufs["off"]), R_COMP, BG, _p(bufs["rgb"]),
                                              _p(bufs["dout"]), _p(bufs["alpha"]), _p(bufs["hit"]), s))


@case("wb_composite_bwd")
def _c_comp_bwd():
    torch = _t()
    L = _A().lib()
    a, b = _comp_set(1), _comp_set(2)
    sets = _fill_sets(a, b, ["sh", "depth", "deltas", "off", "grgb", "gdep", "galp"])
    sets["absmax"] = (torch.zeros(1, device="cuda"),) * 2
    S = a["sh"].shape[0]
    _outs(sets, ["gsh"], {"gsh": ((S, 4), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"gsh": None, "absmax": None},
                 lambda s: L.wb_composite_bwd(_p(bufs["sh"]), _p(bufs["depth"]), _p(bufs["deltas"]), _p(bufs["off"]), R_COMP, BG, _p(bufs["grgb"]),
                                              _p(bufs["gdep"]), _p(bufs["galp"]), _p(bufs["gsh"]), _p(bufs["absmax"]), s))


@case("wb_composite_bwd_loss")
def _c_comp_bwd_loss():
    torch = _t()
    L = _A().lib()
    a, b = _comp_set(1), _comp_set(2)
    sets = _fill_sets(a, b, ["sh", "depth", "deltas", "off", "rgb", "tgt"])
    sets["absmax"] = (torch.zeros(1, device="cuda"),) * 2
    sets["loss"] = (torch.zeros(1, device="cuda"),) * 2
    S = a["sh"].shape[0]
    _outs(sets, ["gsh"], {"gsh": ((S, 4), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"gsh": None, "absmax": None, "loss": ATOMIC},
                 lambda s: L.wb_composite_bwd_loss(_p(bufs["sh"]), _p(bufs["depth"]), _p(bufs["deltas"]), _p(bufs["off"]), R_COMP, BG, _p(bufs["rgb"]),
                                                   _p(bufs["tgt"]), 2, 1.0 / (3 * R_COMP), _p(bufs["gsh"]), _p(bufs["absmax"]), _p(bufs["loss"]), s))


# ------------------------------------------------------------------------------------------------------------------------------
# triplanar and octree grids
# ------------------------------------------------------------------------------------------------------------------------------
TRI_RES = [8, 16]
TRI_FDIM = 4


def _planes(seed, layout=0):
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    out = []
    for r in TRI_RES:
        for _ in range(3):
            shape = (1, TRI_FDIM, r + 1, r + 1) if layout == 0 else (r + 1, r + 1, TRI_FDIM)
            out.append(torch.randn(*shape, generator=g).cuda())
    return out


@case("wb_triplane_fwd")
def _c_tri_fwd():
    torch = _t()
    L = _A().lib()
    N = 3000
    pa, pb = _planes(1), _planes(2)
    sets = {f"p{i}": (x, y) for i, (x, y) in enumerate(zip(pa, pb))}
    sets["x"] = (_hg_coords(N, 1), _hg_coords(N, 2))
    nl = len(TRI_RES)
    _outs(sets, ["f"], {"f": ((N, nl, 3, TRI_FDIM), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    res = (C.c_int32 * nl)(*TRI_RES)
    planes = _pp([bufs[f"p{i}"] for i in range(3 * nl)])
    return Built(bufs, real, poison, {"f": None},
                 lambda s: L.wb_triplane_fwd(_p(bufs["x"]), N, nl, TRI_FDIM, res, planes, _p(bufs["f"]), s), keep=[res, planes])


@case("wb_triplane_bwd")
def _c_tri_bwd():
    torch = _t()
    L = _A().lib()
    N = 3000
    nl = len(TRI_RES)
    pa = _planes(1)
    g = torch.Generator().manual_seed(6)
    sets = {f"p{i}": (x, x) for i, x in enumerate(pa)}
    sets.update({f"g{i}": (torch.zeros_like(x), torch.zeros_like(x)) for i, x in enumerate(pa)})
    sets["x"] = (_hg_coords(N, 1), _hg_coords(N, 2))
    sets["gf"] = (torch.randn(N, nl, 3, TRI_FDIM, generator=g).cuda(), torch.randn(N, nl, 3, TRI_FDIM, generator=g).cuda())
    bufs = {}
    real, poison = _split(bufs, sets)
    res = (C.c_int32 * nl)(*TRI_RES)
    planes = _pp([bufs[f"p{i}"] for i in range(3 * nl)])
    grads = _pp([bufs[f"g{i}"] for i in range(3 * nl)])
    return Built(bufs, real, poison, {f"g{i}": ATOMIC for i in range(3 * nl)},
                 lambda s: L.wb_triplane_bwd(_p(bufs["x"]), N, nl, TRI_FDIM, res, planes, _p(bufs["gf"]), grads, s), keep=[res, planes, grads])


@case("wb_triplane_relayout")
def _c_tri_relayout():
    torch = _t()
    L = _A().lib()
    pa, pb = _planes(1), _planes(2)
    n = len(pa)
    sets = {f"p{i}": (x, y) for i, (x, y) in enumerate(zip(pa, pb))}
    _outs(sets, [f"q{i}" for i in range(n)], {f"q{i}": ((x.shape[2], x.shape[3], TRI_FDIM), torch.float32) for i, x in enumerate(pa)})
    bufs = {}
    real, poison = _split(bufs, sets)
    src, dst = _pp([bufs[f"p{i}"] for i in range(n)]), _pp([bufs[f"q{i}"] for i in range(n)])
    sizes = (C.c_int32 * n)(*[x.shape[2] for x in pa])
    return Built(bufs, real, poison, {f"q{i}": None for i in range(n)},
                 lambda s: L.wb_triplane_relayout(src, dst, sizes, n, TRI_FDIM, 1, s), keep=[src, dst, sizes])


def _sdf_nef(shape="cat_id", seed=0):
    """A NeuralSDF(OctreeGrid) of tests/sdf_shapes.py (seed: other features and decoder, same shapes) and its wb_sdf_field tuple."""
    from sdf_shapes import make_field
    from gpu_util import sdf_nef_from_case
    from wisp_b200 import ops
    f, case_ = make_field(shape, seed=seed)
    c = dict(case_)
    c["feats"] = f.feats
    c["W"], c["b"] = f.Ws, f.bs
    c["hidden_dim"] = f.Ws[0].shape[0]
    nef = sdf_nef_from_case(c)
    nef.grid.half_features = f.half
    return nef, ops.sdf_field(nef)


def _sdf_pair(shape="cat_id"):
    na, fa = _sdf_nef(shape, 0)
    nb, fb = _sdf_nef(shape, 1)
    d, oct, keep = fa
    sets = {f"f{i}": (x, y) for i, (x, y) in enumerate(zip(keep[1], fb[2][1]))}
    sets["params"] = (keep[2], fb[2][2])
    bufs = {f"f{i}": x for i, x in enumerate(keep[1])}
    bufs["params"] = keep[2]
    return d, oct, sets, bufs, [na, nb, fa, fb]


@case("wb_octree_interp_fwd")
def _c_oct_fwd():
    torch = _t()
    L = _A().lib()
    d, oct, sets, bufs, keep = _sdf_pair()
    nl = d.num_lods
    N = 3000
    sets = {k: v for k, v in sets.items() if k != "params"}
    sets["x"] = (_hg_coords(N, 1), _hg_coords(N, 2))
    _outs(sets, ["out"], {"out": ((N, nl * d.feature_dim), torch.float32)})
    real = {k: v[0].clone() for k, v in sets.items()}; poison = {k: v[1] for k, v in sets.items()}
    for k in ("x", "out"):
        bufs[k] = real[k].clone()
    od = oct.desc()
    return Built(bufs, real, poison, {"out": None},
                 lambda s: L.wb_octree_interp_fwd(od, _p(oct.points), C.c_void_p(d.trinkets), _p(bufs["x"]), N, d.feature_dim, d.base_lod, nl, 0,
                                                  d.half_round, d.feats, _p(bufs["out"]), s), keep=keep + [od])


@case("wb_octree_interp_bwd")
def _c_oct_bwd():
    torch = _t()
    L = _A().lib()
    d, oct, sets, bufs, keep = _sdf_pair()
    nl = d.num_lods
    N = 3000
    g = torch.Generator().manual_seed(2)
    feats = [bufs[f"f{i}"] for i in range(nl)]
    sets = {f"g{i}": (torch.zeros_like(f), torch.zeros_like(f)) for i, f in enumerate(feats)}
    sets["x"] = (_hg_coords(N, 1), _hg_coords(N, 2))
    sets["go"] = (torch.randn(N, nl * d.feature_dim, generator=g).cuda(), torch.randn(N, nl * d.feature_dim, generator=g).cuda())
    bufs = {}
    real, poison = _split(bufs, sets)
    grads = _pp([bufs[f"g{i}"] for i in range(nl)])
    od = oct.desc()
    return Built(bufs, real, poison, {f"g{i}": ATOMIC for i in range(nl)},
                 lambda s: L.wb_octree_interp_bwd(od, _p(oct.points), C.c_void_p(d.trinkets), _p(bufs["x"]), N, d.feature_dim, d.base_lod, nl, 0,
                                                  d.feats, _p(bufs["go"]), grads, s), keep=keep + [od, grads])


# ------------------------------------------------------------------------------------------------------------------------------
# NeuralSDF
# ------------------------------------------------------------------------------------------------------------------------------
@case("wb_sdf_eval")
def _c_sdf_eval():
    torch = _t()
    L = _A().lib()
    d, oct, sets, bufs, keep = _sdf_pair("config3")
    N = 4000
    sets["x"] = (_hg_coords(N, 1), _hg_coords(N, 2))
    _outs(sets, ["sdf"], {"sdf": ((N,), torch.float32)})
    real = {k: v[0].clone() for k, v in sets.items()}; poison = {k: v[1] for k, v in sets.items()}
    for k in ("x", "sdf"):
        bufs[k] = real[k].clone()
    od = oct.desc()
    return Built(bufs, real, poison, {"sdf": None},
                 lambda s: L.wb_sdf_eval(od, d, d.num_lods - 1, _p(bufs["x"]), N, _p(bufs["sdf"]), s), keep=keep + [od])


def _sdf_train_case(tc, shape="config3", N=4096):
    torch = _t()
    L = _A().lib()
    d, oct, sets, bufs, keep = _sdf_pair(shape)
    nl = d.num_lods
    g = torch.Generator().manual_seed(9)
    feats = [bufs[f"f{i}"] for i in range(nl)]
    sets["x"] = (_hg_coords(N, 1), _hg_coords(N, 2))
    sets["gt"] = ((torch.rand(N, generator=g) * 0.2 - 0.1).cuda(), (torch.rand(N, generator=g) * 0.2 - 0.1).cuda())
    sets.update({f"g{i}": (torch.zeros_like(f), torch.zeros_like(f)) for i, f in enumerate(feats)})
    sets["gp"] = (torch.zeros_like(bufs["params"]), torch.zeros_like(bufs["params"]))
    sets["loss"] = (torch.zeros(1, device="cuda"),) * 2
    real = {k: v[0].clone() for k, v in sets.items()}; poison = {k: v[1] for k, v in sets.items()}
    for k in real:
        if k not in bufs:
            bufs[k] = real[k].clone()
    grads = _pp([bufs[f"g{i}"] for i in range(nl)])
    od = oct.desc()
    fn = L.wb_sdf_train_tc if tc else L.wb_sdf_train
    outs = {f"g{i}": ATOMIC for i in range(nl)}
    outs.update(gp=ATOMIC, loss=ATOMIC)
    return Built(bufs, real, poison, outs,
                 lambda s: fn(od, d, nl - 1, _p(bufs["x"]), _p(bufs["gt"]), N, 1.0 / N, grads, _p(bufs["gp"]), _p(bufs["loss"]), s),
                 keep=keep + [od, grads])


@case("wb_sdf_train")
def _c_sdf_train():
    return _sdf_train_case(False)


@case("wb_sdf_train_tc")
def _c_sdf_train_tc():
    return _sdf_train_case(True)


def _sdf_trace_sets(nef_shape="config3"):
    """Two ray sets traced through the octree of the SDF field at its finest active level, cut to one nugget count."""
    torch = _t()
    A = _A(); L = A.lib()
    d, oct, sets, bufs, keep = _sdf_pair(nef_shape)
    level = d.base_lod + d.num_lods - 1
    R = 256
    out = []
    for seed in (1, 2):
        o, dd = _rays(R, seed)
        cnt = torch.zeros(R, dtype=torch.int32, device="cuda")
        rays = _rays_desc(o, dd)
        L.wb_raytrace_count(oct.desc(), level, rays, _p(cnt), 0)
        off = _scan(cnt)
        Ng = int(off[-1])
        ridx = torch.zeros(max(Ng, 1), dtype=torch.int32, device="cuda"); pidx = torch.zeros_like(ridx)
        dep = torch.zeros(max(Ng, 1), 2, device="cuda")
        L.wb_raytrace_fill(oct.desc(), level, rays, _p(off), _p(ridx), _p(pidx), _p(dep), 0)
        torch.cuda.synchronize()
        out.append(dict(o=o, d=dd, ridx=ridx, dep=dep, Ng=Ng))
    Ng = min(o_["Ng"] for o_ in out)
    for st in out:
        st["dep"] = st["dep"][:Ng].contiguous()
        c = torch.bincount(st["ridx"][:Ng].long(), minlength=R)
        st["off"] = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), c.cumsum(0)])
    return d, oct, sets, bufs, keep, out, R, Ng


def _sdf_state_bufs(R, steps):
    torch = _t()
    A = _A(); L = A.lib()
    wsb = int(L.wb_scan_workspace_bytes(R))
    shapes = {"flags": ((R,), torch.int32), "pack_off": ((R + 1,), torch.int64), "scan_ws": ((max(wsb, 1),), torch.uint8),
              "pack_ray": ((R,), torch.int32), "t": ((R,), torch.float32), "dist": ((R,), torch.float32), "dist_prev": ((R,), torch.float32),
              "x": ((3 * R,), torch.float32), "cursor0": ((R,), torch.int32), "cursor1": ((R,), torch.int32), "state": ((R,), torch.uint8),
              "iterflags": ((2 * steps + 4,), torch.int32)}
    return shapes, wsb


def _state_desc(bufs, wsb):
    s = _A().SdfState()
    for k in ("flags", "pack_off", "scan_ws", "pack_ray", "t", "dist", "dist_prev", "x", "cursor0", "cursor1", "state", "iterflags"):
        setattr(s, k, bufs["st_" + k].data_ptr())
    s.scan_ws_bytes = wsb
    return s


SDF_STEPS = 32


@case("wb_sdf_trace")
def _c_sdf_trace():
    torch = _t()
    L = _A().lib()
    d, oct, sets, bufs, keep, tr, R, Ng = _sdf_trace_sets()
    sets.update(_fill_sets(tr[0], tr[1], ["o", "d", "dep", "off"]))
    shapes, wsb = _sdf_state_bufs(R, SDF_STEPS)
    # the state is scratch the call initialises: zeros in both sets (valid indices whatever a stray launch reads)
    for k, (shp, dt) in shapes.items():
        sets["st_" + k] = (torch.zeros(shp, dtype=dt, device="cuda"),) * 2
    outs = {"xyz": ((R, 3), torch.float32), "depth": ((R, 1), torch.float32), "hit": ((R,), torch.uint8), "normal": ((R, 3), torch.float32),
            "rgb": ((R, 3), torch.float32), "alpha": ((R, 1), torch.float32)}
    _outs(sets, list(outs), outs)
    real = {k: v[0].clone() for k, v in sets.items()}; poison = {k: v[1] for k, v in sets.items()}
    for k in real:
        if k not in bufs:
            bufs[k] = real[k].clone()
    st = _state_desc(bufs, wsb)
    od, rays = oct.desc(), _rays_desc(bufs["o"], bufs["d"], 0.0, 6.0)
    return Built(bufs, real, poison, dict.fromkeys(outs),
                 lambda s: L.wb_sdf_trace(od, d, d.num_lods - 1, rays, _p(bufs["dep"]), Ng, _p(bufs["off"]), SDF_STEPS, 0.8, 1e-3, 1, st,
                                          _p(bufs["xyz"]), _p(bufs["depth"]), _p(bufs["hit"]), _p(bufs["normal"]), _p(bufs["rgb"]), _p(bufs["alpha"]), s),
                 keep=keep + [od, rays, st])


@case("wb_sdf_phase")
def _c_sdf_phase():
    """Phase 0 (pack list: the flag kernel, the three scan kernels and the phase kernel) then phase 1 (initial state) of the
    phase-by-phase route: the state they write is compared."""
    torch = _t()
    L = _A().lib()
    d, oct, sets, bufs, keep, tr, R, Ng = _sdf_trace_sets()
    sets = _fill_sets(tr[0], tr[1], ["o", "d", "dep", "off"])
    shapes, wsb = _sdf_state_bufs(R, SDF_STEPS)
    for k, (shp, dt) in shapes.items():
        sets["st_" + k] = (torch.zeros(shp, dtype=dt, device="cuda"),) * 2
    bufs = {}
    real, poison = _split(bufs, sets)
    st = _state_desc(bufs, wsb)
    rays = _rays_desc(bufs["o"], bufs["d"], 0.0, 6.0)

    def call(s):
        for ph in (0, 1):
            L.wb_sdf_phase(ph, rays, _p(bufs["dep"]), Ng, _p(bufs["off"]), SDF_STEPS, 0, 1e-3, st, None, None, None, None, s)
    return Built(bufs, real, poison, {"st_flags": None, "st_pack_off": None, "st_pack_ray": None, "st_t": None, "st_x": None, "st_cursor0": None,
                                      "st_state": None}, call, keep=keep + [rays, st])


# ------------------------------------------------------------------------------------------------------------------------------
# codebook, optimisers, ray generation, the wgmma self-test
# ------------------------------------------------------------------------------------------------------------------------------
CB_ROWS, CB_K, CB_F = 3000, 64, 8


@case("wb_codebook_rows_fwd")
def _c_cb_fwd():
    torch = _t()
    L = _A().lib()
    g = torch.Generator().manual_seed(4)
    sets = {"lg": (torch.randn(CB_ROWS, CB_K, generator=g).cuda(), torch.randn(CB_ROWS, CB_K, generator=g).cuda()),
            "dc": (torch.randn(CB_K, CB_F, generator=g).cuda(), torch.randn(CB_K, CB_F, generator=g).cuda())}
    _outs(sets, ["E", "am"], {"E": ((CB_ROWS, CB_F), torch.float32), "am": ((CB_ROWS,), torch.int32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"E": None, "am": None},
                 lambda s: L.wb_codebook_rows_fwd(_p(bufs["lg"]), _p(bufs["dc"]), CB_ROWS, CB_K, CB_F, 1, _p(bufs["E"]), _p(bufs["am"]), s))


@case("wb_codebook_rows_bwd")
def _c_cb_bwd():
    torch = _t()
    L = _A().lib()
    g = torch.Generator().manual_seed(4)
    K, F = 1024, 16                             # (K*F + 256) * 4 bytes of shared memory: above the default 48 KB
    sets = {"lg": (torch.randn(CB_ROWS, K, generator=g).cuda(), torch.randn(CB_ROWS, K, generator=g).cuda()),
            "dc": (torch.randn(K, F, generator=g).cuda(), torch.randn(K, F, generator=g).cuda()),
            "dE": (torch.randn(CB_ROWS, F, generator=g).cuda(), torch.randn(CB_ROWS, F, generator=g).cuda()),
            "gl": (torch.zeros(CB_ROWS, K, device="cuda"),) * 2, "gd": (torch.zeros(K, F, device="cuda"),) * 2}
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"gl": None, "gd": ATOMIC},
                 lambda s: L.wb_codebook_rows_bwd(_p(bufs["lg"]), _p(bufs["dc"]), _p(bufs["dE"]), CB_ROWS, K, F, _p(bufs["gl"]), _p(bufs["gd"]), s))


def _optim_case(kind):
    torch = _t()
    A = _A(); L = A.lib()
    g = torch.Generator().manual_seed(21)
    sizes = [1000, 37, 4096]
    names = ["param", "grad", "s1", "s2"]
    sets = {}
    for i, n in enumerate(sizes):
        for nm in names:
            mk = lambda: (torch.rand(n, generator=g) if nm in ("s2",) else torch.randn(n, generator=g)).cuda()
            sets[f"{nm}{i}"] = (mk(), mk())
    bufs = {}
    real, poison = _split(bufs, sets)
    if kind == "rmsprop":
        segs = (A.RMSpropSegment * len(sizes))()
        for i, n in enumerate(sizes):
            segs[i].param, segs[i].grad, segs[i].square_avg, segs[i].momentum_buffer = (bufs[f"{k}{i}"].data_ptr() for k in ("param", "grad", "s2", "s1"))
            segs[i].numel, segs[i].lr, segs[i].weight_decay = n, 1e-2, 0.01 * i
        call = lambda s: L.wb_rmsprop_step(segs, len(sizes), 0.99, 1e-8, 0.9, 0.5, 1, s)
    else:
        segs = (A.AdamSegment * len(sizes))()
        for i, n in enumerate(sizes):
            segs[i].param, segs[i].grad, segs[i].exp_avg, segs[i].exp_avg_sq = (bufs[f"{k}{i}"].data_ptr() for k in names)
            segs[i].numel, segs[i].lr, segs[i].weight_decay = n, 1e-2, 0.01 * i
        fn = L.wb_adam_step if kind == "adam" else L.wb_adamw_step
        call = lambda s: fn(segs, len(sizes), 0.9, 0.999, 1e-8, 3, 0.5, 1, s)
    return Built(bufs, real, poison, {k: None for k in sets}, call, keep=[segs])


@case("wb_adam_step")
def _c_adam():
    return _optim_case("adam")


@case("wb_adamw_step")
def _c_adamw():
    return _optim_case("adamw")


@case("wb_rmsprop_step")
def _c_rmsprop():
    return _optim_case("rmsprop")


RG_H, RG_W = 96, 128


@case("wb_raygen_lookat")
def _c_raygen_lookat():
    torch = _t()
    L = _A().lib()
    sets = {}
    _outs(sets, ["o", "d"], {"o": ((RG_H * RG_W, 3), torch.float32), "d": ((RG_H * RG_W, 3), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    f3 = lambda *v: (C.c_float * 3)(*v)
    org, view, right, up = f3(0.0, 1.0, 4.0), f3(0.0, -0.242535, -0.970143), f3(1.0, 0.0, 0.0), f3(0.0, 0.970143, -0.242535)
    return Built(bufs, real, poison, {"o": None, "d": None},
                 lambda s: L.wb_raygen_lookat(org, view, right, up, 0.4, RG_H, RG_W, 0, _p(bufs["o"]), _p(bufs["d"]), s),
                 host_inputs=True, keep=[org, view, right, up])


@case("wb_raygen_pinhole")
def _c_raygen_pinhole():
    torch = _t()
    L = _A().lib()
    sets = {}
    _outs(sets, ["o", "d"], {"o": ((RG_H * RG_W, 3), torch.float32), "d": ((RG_H * RG_W, 3), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    pos = (C.c_float * 3)(0.5, 1.0, 3.0)
    rot = (C.c_float * 9)(1, 0, 0, 0, 0.8, -0.6, 0, 0.6, 0.8)
    return Built(bufs, real, poison, {"o": None, "d": None},
                 lambda s: L.wb_raygen_pinhole(pos, rot, 0.0, 0.0, 0.4, 0.3, RG_H, RG_W, RG_H, RG_W, _p(bufs["o"]), _p(bufs["d"]), s),
                 host_inputs=True, keep=[pos, rot])


@case("wb_tc_selftest")
def _c_tc_selftest():
    """mode 0, N = K = 64: operand images of random fp16 values (any byte image of finite fp16 values is a valid operand)."""
    torch = _t()
    L = _A().lib()
    N, K = 64, 64
    g = torch.Generator().manual_seed(31)
    a_n, b_n = 128 * K, N * K
    mk = lambda n: (torch.rand(n, generator=g) * 2 - 1).half().cuda().view(torch.uint8)
    sets = {"a": (mk(a_n), mk(a_n)), "b": (mk(b_n), mk(b_n))}
    _outs(sets, ["D"], {"D": ((128, N), torch.float32)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"D": None},
                 lambda s: L.wb_tc_selftest(_p(bufs["a"]), 2 * a_n, _p(bufs["b"]), 2 * b_n, _p(bufs["D"]), N, K, 0, s))


# ------------------------------------------------------------------------------------------------------------------------------
# app/image: 2-D hash grid and the image field (make_field of tests/test_gpu_image.py, seeds 0 and 1)
# ------------------------------------------------------------------------------------------------------------------------------
def _image_pair(H=64, F=2, L_=8):
    import wisp_b200 as W
    from wisp_b200 import ops
    from test_gpu_image import make_field
    na = make_field(W, F=F, L=L_, bw=14, max_res=256, H=H, seed=0)
    nb = make_field(W, F=F, L=L_, bw=14, max_res=256, H=H, seed=1)
    fa, fb = ops.image_field(na), ops.image_field(nb)
    return na, nb, fa, fb


def _coords2(N, seed):
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(N, 2, generator=g) * 2 - 1).cuda()


@case("wb_hashgrid2d_fwd")
def _c_hg2_fwd():
    torch = _t()
    L = _A().lib()
    na, nb, fa, fb = _image_pair()
    N = 3000
    bufs = {"table": fa[3][0].detach()}
    sets = {"table": (fa[3][0].detach(), fb[3][0].detach()), "x": (_coords2(N, 1), _coords2(N, 2))}
    _outs(sets, ["f"], {"f": ((N, fa[0].num_lods * fa[0].feature_dim), torch.float32)})
    real = {k: v[0].clone() for k, v in sets.items()}; poison = {k: v[1] for k, v in sets.items()}
    for k in ("x", "f"):
        bufs[k] = real[k].clone()
    return Built(bufs, real, poison, {"f": None}, lambda s: L.wb_hashgrid2d_fwd(_p(bufs["x"]), N, fa[0], _p(bufs["f"]), s), keep=[na, nb, fa, fb])


@case("wb_hashgrid2d_bwd")
def _c_hg2_bwd():
    torch = _t()
    L = _A().lib()
    na, nb, fa, fb = _image_pair()
    N = 3000
    Wd = fa[0].num_lods * fa[0].feature_dim
    g = torch.Generator().manual_seed(3)
    t = fa[3][0]
    sets = {"x": (_coords2(N, 1), _coords2(N, 2)), "gf": (torch.randn(N, Wd, generator=g).cuda(), torch.randn(N, Wd, generator=g).cuda()),
            "gt": (torch.zeros_like(t.detach()),) * 2}
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"gt": ATOMIC}, lambda s: L.wb_hashgrid2d_bwd(_p(bufs["x"]), N, fa[0], _p(bufs["gf"]), _p(bufs["gt"]), s),
                 keep=[na, nb, fa, fb])


def _image_sets(fa, fb):
    sets = {"table": (fa[3][0].detach(), fb[3][0].detach())}
    for i in range(4):
        sets[f"w{i}"] = (fa[3][1 + i].detach(), fb[3][1 + i].detach())
    bufs = {"table": fa[3][0].detach()}
    bufs.update({f"w{i}": fa[3][1 + i].detach() for i in range(4)})
    return sets, bufs


def _image_case(train, H=64, N=3000):
    torch = _t()
    L = _A().lib()
    na, nb, fa, fb = _image_pair(H=H)
    sets, bufs = _image_sets(fa, fb)
    sets["x"] = (_coords2(N, 1), _coords2(N, 2))
    desc, Hd, ptrs = fa[0], fa[1], fa[2]
    lod = desc.num_lods - 1
    if train:
        g = torch.Generator().manual_seed(5)
        npar = sum(int(t.numel()) for t in fa[3][1:])
        sets["gt"] = (torch.rand(N, 3, generator=g).cuda(), torch.rand(N, 3, generator=g).cuda())
        sets["gtab"] = (torch.zeros_like(fa[3][0].detach()),) * 2
        sets["gp"] = (torch.zeros(npar, device="cuda"),) * 2
        sets["loss"] = (torch.zeros(1, device="cuda"),) * 2
        outs = {"gtab": ATOMIC, "gp": ATOMIC, "loss": ATOMIC}
    else:
        _outs(sets, ["rgb"], {"rgb": ((N, 3), torch.float32)})
        outs = {"rgb": None}
    real = {k: v[0].clone() for k, v in sets.items()}; poison = {k: v[1] for k, v in sets.items()}
    for k in real:
        if k not in bufs:
            bufs[k] = real[k].clone()
    if train:
        call = lambda s: L.wb_image_train(desc, Hd, ptrs, lod, _p(bufs["x"]), _p(bufs["gt"]), N, 1.0 / (3 * N), _p(bufs["gtab"]), _p(bufs["gp"]),
                                          _p(bufs["loss"]), s)
    else:
        call = lambda s: L.wb_image_eval(desc, Hd, ptrs, lod, _p(bufs["x"]), N, _p(bufs["rgb"]), s)
    return Built(bufs, real, poison, outs, call, keep=[na, nb, fa, fb])


@case("wb_image_eval")
def _c_image_eval():
    return _image_case(False)


@case("wb_image_train")
def _c_image_train():
    return _image_case(True)


# ------------------------------------------------------------------------------------------------------------------------------
# meshes
# ------------------------------------------------------------------------------------------------------------------------------
MESH_T = 600


def _tris(seed, dtype):
    torch = _t()
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(MESH_T, 1, 3, generator=g, dtype=torch.float64) * 1.4 - 0.7
    return (c + (torch.rand(MESH_T, 3, 3, generator=g, dtype=torch.float64) - 0.5) * 0.3).reshape(MESH_T, 9).to(dtype).cuda()


@case("wb_mesh_sdf")
def _c_mesh_sdf():
    torch = _t()
    L = _A().lib()
    N = 2000
    wsb = int(L.wb_mesh_sdf_workspace_bytes(MESH_T))
    g = torch.Generator().manual_seed(17)
    sets = {"tris": (_tris(1, torch.float64), _tris(2, torch.float64)),
            "pts": ((torch.rand(N, 3, generator=g, dtype=torch.float64) * 2 - 1).cuda(), (torch.rand(N, 3, generator=g, dtype=torch.float64) * 2 - 1).cuda()),
            "ws": (torch.zeros(wsb, dtype=torch.uint8, device="cuda"),) * 2}
    _outs(sets, ["out"], {"out": ((N,), torch.float64)})
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"out": None},
                 lambda s: L.wb_mesh_sdf(_p(bufs["tris"]), MESH_T, _p(bufs["pts"]), N, _p(bufs["ws"]), wsb, _p(bufs["out"]), s))


@case("wb_mesh_octree_bits")
def _c_mesh_octree():
    torch = _t()
    L = _A().lib()
    level = 6
    sets = {}
    for k, seed in (("a", 1), ("b", 2)):
        tr = _tris(seed, torch.float32)
        v = tr.double().reshape(-1, 3, 3)
        area = torch.linalg.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]).norm(dim=1) * 0.5
        cdf = torch.zeros(MESH_T + 1, dtype=torch.float64, device="cuda"); cdf[1:] = area.cumsum(0)
        sets.setdefault("tris", []).append(tr); sets.setdefault("cdf", []).append(cdf)
    sets = {k: tuple(v) for k, v in sets.items()}
    sets["bits"] = (torch.zeros((8 ** level + 31) // 32, dtype=torch.int32, device="cuda"),) * 2
    bufs = {}
    real, poison = _split(bufs, sets)
    return Built(bufs, real, poison, {"bits": None},
                 lambda s: L.wb_mesh_octree_bits(_p(bufs["tris"]), _p(bufs["cdf"]), MESH_T, 200_000, level, 5, _p(bufs["bits"]), s))


# ------------------------------------------------------------------------------------------------------------------------------
# configurations for the concurrent-caller checks (not registry entries: the same entry points at other shapes)
# ------------------------------------------------------------------------------------------------------------------------------
def p0_shade_case(width, S=6000, R=300, seed=0):
    """Precision-0 wb_rf_shade_fwd then wb_rf_shade_bwd over a hash grid with `width`-wide decoders (one hidden density layer, two
    hidden colour layers): the shade kernel instances are shared by every width, their dynamic shared memory is not."""
    import numpy as np
    import torch
    from oracle import oracle as O
    from wisp_b200 import ops
    A = _A(); L = A.lib()
    rng = np.random.default_rng(500 + seed)
    Lh, F, bw = 8, 2, 12
    res = O.geometric_resolutions(Lh, 4, 64)
    begin = [int(b) for b in O.table_layout(res, bw)]
    dens = [Lh * F, width, 16]
    col = [15 + 27, width, width, 3]
    mk = lambda dims: np.concatenate([np.concatenate([(rng.uniform(-1, 1, (o, i)) / np.sqrt(i)).ravel(), rng.uniform(-0.1, 0.1, o)])
                                      for i, o in zip(dims[:-1], dims[1:])]).astype(np.float32)
    table = torch.from_numpy((rng.standard_normal((begin[-1], F)) * 0.5).astype(np.float32)).cuda()
    fd, fc = torch.from_numpy(mk(dens)).cuda(), torch.from_numpy(mk(col)).cuda()
    spec = ops.NefSpec(resolutions=res, begin_idxes=begin, codebook_size=2 ** bw, feature_dim=F, multiscale="cat", lod_idx=Lh, pos_mode=0,
                       pos_freq=0, view_mode=3, view_freq=4, has_bias=True, dens_dims=dens, col_dims=col)
    desc, dkeep = spec.desc([table], fd, fc)
    o = torch.from_numpy(rng.uniform(-0.4, 0.4, (R, 3)).astype(np.float32)).cuda()
    d = torch.nn.functional.normalize(torch.from_numpy(rng.standard_normal((R, 3)).astype(np.float32)), dim=1).cuda()
    rr = torch.from_numpy(np.sort(rng.integers(0, R, S)).astype(np.int32)).cuda()
    rt = torch.from_numpy(rng.uniform(0.0, 0.5, S).astype(np.float32)).cuda()
    blob = torch.empty(int(L.wb_rf_param_blob_floats(desc, 0)), dtype=torch.float32, device="cuda")
    L.wb_rf_pack_params(desc, 0, _p(blob), 0)
    g = torch.from_numpy((rng.standard_normal((S, 4)) * 1e-2).astype(np.float32)).cuda()
    bufs = dict(table=table, fd=fd, fc=fc, o=o, d=d, rr=rr, rt=rt, blob=blob, g=g, sh=torch.zeros(S, 4, device="cuda"),
                gt=torch.zeros_like(table), gd=torch.zeros_like(fd), gc=torch.zeros_like(fc))
    real = {k: bufs[k].clone() for k in ("sh", "gt", "gd", "gc")}
    rays = _rays_desc(o, d, 0.0, 1.0)

    def call(s):
        L.wb_rf_shade_fwd(desc, _p(blob), 0, rays, _p(rt), _p(rr), S, _p(bufs["sh"]), None, None, s)
        L.wb_rf_shade_bwd(desc, _p(blob), 0, rays, _p(rt), _p(rr), S, _p(g), None, None, None, _p(bufs["gt"]), _p(bufs["gd"]), _p(bufs["gc"]), s)
    return Built(bufs, real, real, {"sh": None, "gt": ATOMIC, "gd": ATOMIC, "gc": ATOMIC}, call, keep=[desc, dkeep, rays])


def chunked_bwd_case(seed=0):
    """The precision-1 backward that splits its samples into chunks and scatters the table gradient of each chunk on the library's
    side stream: the 128-wide, S = 2^20 + 4097 case of tests/test_gpu_tc_decoders.py::test_chunked_backward_matches_two_stages."""
    import wisp_b200 as W
    from test_gpu_tc_decoders import Case, Setup
    torch = _t()
    a = Setup(W, Case("chunked", [128], [128, 128], view=(3, 4), L=16, S=(1 << 20) + 4097, R=5000, seed=seed))
    blob, feat, ws, _ = _fwd_state(a)
    scale = torch.tensor([256.0], device="cuda")
    # the poison: other incoming gradients (the saved forward rows and the workspace are this field's)
    sets = {"g": (_g_shaded(a.S, 10 + seed), _g_shaded(a.S, 20 + seed)), "ws": (ws, ws)}
    for k, t in (("gt", a.t_table), ("gd", a.t_fd), ("gc", a.t_fc)):
        sets[k] = (torch.zeros_like(t),) * 2
    bufs = {}
    real, poison = _split(bufs, sets)
    call = lambda s: a.L.wb_rf_shade_bwd(a.desc, _p(blob), 1, a.rays, _p(a.t_rec_t), _p(a.t_rec_ray), a.S, _p(bufs["g"]), _p(scale), _p(feat),
                                         _p(bufs["ws"]), _p(bufs["gt"]), _p(bufs["gd"]), _p(bufs["gc"]), s)
    return Built(bufs, real, poison, {"gt": ATOMIC_TC, "gd": ATOMIC_TC, "gc": ATOMIC_TC}, call, keep=[a, blob, feat, scale])


# Configurations of registry entry points that the gated and graph checks run besides CASES: the chunked backward is the only call
# that forks work onto the library's side stream (a captured call runs it on the caller's stream alone).
EXTRA_CASES = {"wb_rf_shade_bwd[chunked]": chunked_bwd_case}


def image_train_case(hidden):
    return _image_case(True, H=hidden)


def sdf_train_tc_case(shape):
    return _sdf_train_case(True, shape)
