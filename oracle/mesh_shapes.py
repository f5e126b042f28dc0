"""Procedural, seeded meshes and point sets for the mesh-SDF checks (TEST INFRASTRUCTURE, numpy only).

Used by oracle/make_ref_golden_mesh.py (the reference kernel's golden), tests/test_mesh_sdf_reference_cpu.py,
tests/test_gpu_mesh_sdf.py and tools/bench_mesh_sdf.py.  Meshes are (V f64 [#V, 3], F int64 [#F, 3]) in wisp's [-1, 1] cube."""
from __future__ import annotations

import numpy as np

NEAR_STD = 1.0 / 128        # sample_near_surface: samples + randn * variance, with the variance the SDF datasets pass


def icosphere(subdiv: int, radius: float = 1.0):
    """Icosahedron subdivided `subdiv` times and projected on the sphere: 20 * 4^subdiv triangles, outward winding."""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    V = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    F = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
                  [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], np.int64)
    V /= np.linalg.norm(V, axis=1, keepdims=True)
    for _ in range(subdiv):
        e = np.sort(np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]), axis=1)
        uniq, inv = np.unique(e, axis=0, return_inverse=True)
        mid = V[uniq[:, 0]] + V[uniq[:, 1]]
        mid /= np.linalg.norm(mid, axis=1, keepdims=True)
        ab, bc, ca = inv.reshape(3, -1) + V.shape[0]
        a, b, c = F.T
        V = np.concatenate([V, mid])
        F = np.concatenate([np.stack([a, ab, ca], 1), np.stack([b, bc, ab], 1), np.stack([c, ca, bc], 1), np.stack([ab, bc, ca], 1)])
    return V * radius, F


def noisy_sphere(subdiv: int, seed: int = 0, radius: float = 0.7):
    """An icosphere with a smooth seeded radial bump field and a little per-vertex noise."""
    V, F = icosphere(subdiv)
    rng = np.random.default_rng(seed)
    k = rng.normal(size=(6, 3)) * 3.0
    ph = rng.uniform(0, 2 * np.pi, 6)
    r = 1.0 + 0.06 * np.sin(V @ k.T + ph).sum(1) / 3.0 + 0.002 * rng.standard_normal(V.shape[0])
    return V * (radius * r)[:, None], F


def torus(nu: int = 32, nv: int = 16, R: float = 0.55, r: float = 0.2):
    """Closed torus around z, 2 nu nv triangles, outward winding."""
    u, v = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    V = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    F = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return V, F


def cube(h: float = 0.5):
    """Axis-aligned cube [-h, h]^3: 12 triangles, two per face sharing the face's diagonal."""
    V = np.array([[x, y, z] for x in (-h, h) for y in (-h, h) for z in (-h, h)], np.float64)
    F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                  [1, 5, 7], [1, 7, 3]], np.int64)
    return V, F


def open_mesh():
    """An icosphere (1280 triangles) with its cap above z = 0.35 removed: a mesh with a boundary."""
    V, F = icosphere(3, 0.6)
    return V, F[V[F][:, :, 2].mean(1) <= 0.35 * 0.6]


def surface_points(V, F, n: int, rng):
    """Area-weighted uniform points on the surface (sample_surface)."""
    T = V[F]
    area = np.linalg.norm(np.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0]), axis=1)
    f = rng.choice(F.shape[0], n, p=area / area.sum())
    r1, r2 = np.sqrt(rng.uniform(size=n)), rng.uniform(size=n)
    return T[f, 0] * (1 - r1)[:, None] + T[f, 1] * (r1 * (1 - r2))[:, None] + T[f, 2] * (r1 * r2)[:, None]


def near_points(V, F, n: int, rng):
    return surface_points(V, F, n, rng) + rng.standard_normal((n, 3)) * NEAR_STD


def uniform_points(n: int, rng, lo: float = -1.1, hi: float = 1.1):
    return rng.uniform(lo, hi, (n, 3))


def feature_points(V, F, n: int, rng):
    """n points on vertices, n on edges (seeded parameter) and n inside faces (seeded barycentric)."""
    T = V[F]
    pv = V[rng.integers(0, V.shape[0], n)]
    f, k, s = rng.integers(0, F.shape[0], n), rng.integers(0, 3, n), rng.uniform(size=n)[:, None]
    pe = T[f, k] * (1 - s) + T[f, (k + 1) % 3] * s
    f = rng.integers(0, F.shape[0], n)
    b = rng.dirichlet((1.0, 1.0, 1.0), n)
    pf = (T[f] * b[:, :, None]).sum(1)
    return np.concatenate([pv, pe, pf])


def dataset_points(V, F, n: int, rng):
    """Points drawn as the SDF datasets draw them (point_sample with sample_mode ['rand', 'near', 'near', 'trace', 'trace']):
    uniform in [-1, 1]^3, near-surface, and surface points, in the proportions 1 : 2 : 2."""
    k = n // 5
    return np.concatenate([uniform_points(n - 4 * k, rng, -1.0, 1.0), near_points(V, F, 2 * k, rng), surface_points(V, F, 2 * k, rng)])


# The golden's cases: name -> (mesh, number of near / uniform / feature points)
def golden_cases():
    return {
        "icosphere": (icosphere(3, 0.6), (3000, 2000, 500)),
        "torus": (torus(), (3000, 2000, 500)),
        "cube": (cube(), (3000, 2000, 500)),
        "open": (open_mesh(), (3000, 2000, 500)),
        "noisy_sphere": (noisy_sphere(5, seed=3), (12000, 6000, 2000)),
    }


def golden_points(name: str, V, F, counts, seed: int):
    rng = np.random.default_rng(seed)
    n_near, n_uni, n_feat = counts
    return np.concatenate([near_points(V, F, n_near, rng), uniform_points(n_uni, rng), feature_points(V, F, n_feat, rng)])
