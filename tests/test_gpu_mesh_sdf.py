"""wisp_b200.compute_sdf (wb_mesh_sdf) on the H100 against the reference's own kernel (tests/golden/ref_mesh_sdf.npz, recorded by
oracle/make_ref_golden_mesh.py) and against the numpy restatement of its rule (tests/mesh_sdf_reference.py)."""
import os

import numpy as np
import pytest
import torch

import mesh_sdf_reference as R
from oracle import mesh_shapes as MS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["icosphere", "torus", "cube", "open", "noisy_sphere"]
MAX_PAIRS = 10 ** 7          # restatement pairs per check


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    torch.cuda.set_device(0)
    return wisp_b200


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "ref_mesh_sdf.npz"))


def sdf(W, V, F, P, **kw):
    out = W.compute_sdf(torch.as_tensor(V), torch.as_tensor(F, dtype=torch.int64), torch.as_tensor(P), **kw)
    torch.cuda.synchronize()
    assert out.dtype == torch.float64 and out.is_cuda and out.shape == (P.shape[0], 1)
    return out[:, 0].cpu().numpy()


def against_restatement(got, V, F, P):
    ref = R.mesh_sdf(V[F].reshape(-1, 9), P)
    both_inf = np.isinf(got) & np.isinf(ref["sdf"]) & (np.sign(got) == np.sign(ref["sdf"]))
    err = np.where(both_inf, 0.0, np.abs(np.abs(got) - np.abs(ref["sdf"])))
    bad = ~(err <= ref["tol"])
    assert not bad.any(), (int(bad.sum()), got[bad][:5], ref["sdf"][bad][:5], ref["tol"][bad][:5])
    ok = ref["sign_ok"]
    assert np.array_equal(got[ok] < 0, ref["inside"][ok]), int(((got < 0) != ref["inside"])[ok].sum())
    return ref


def subsample(n, T, seed):
    k = max(1, min(n, MAX_PAIRS // max(T, 1)))
    return np.sort(np.random.default_rng(seed).choice(n, k, replace=False))


@pytest.mark.parametrize("case", CASES)
def test_golden_reference_kernel(W, golden, case):
    """Bit-identical distances on >= 99.9 % of the points, every other one inside the restatement's bound; the sign equal to the
    reference kernel's on every point whose sign the restatement calls unambiguous: every point where the signs differ is ambiguous,
    and so is every sign difference between the restatement and the golden on a seeded subsample."""
    V, F, P, gold = (golden[f"{case}_{k}"] for k in ("V", "F", "points", "sdf"))
    F, gold = F.astype(np.int64), gold.astype(np.float64)
    got = sdf(W, V, F, P)
    same = np.abs(got) == np.abs(gold)
    assert same.mean() >= 0.999, same.mean()
    diff = np.nonzero(~same)[0]
    if diff.size:
        ref = R.mesh_sdf(V[F].reshape(-1, 9), P[diff])
        assert np.all(np.abs(np.abs(got[diff]) - np.abs(gold[diff])) <= ref["tol"]), (got[diff][:5], gold[diff][:5], ref["tol"][:5])
    sign_diff = np.nonzero((got < 0) != (gold < 0))[0]
    if sign_diff.size:
        assert not R.mesh_sdf(V[F].reshape(-1, 9), P[sign_diff])["sign_ok"].any()
    idx = subsample(P.shape[0], F.shape[0], 7)
    ref = R.mesh_sdf(V[F].reshape(-1, 9), P[idx])
    ok = ref["sign_ok"]
    assert np.array_equal(got[idx][ok] < 0, gold[idx][ok] < 0)
    assert np.array_equal(ref["inside"][ok], gold[idx][ok] < 0)          # the restatement reads the reference's sign rule right
    print(f"{case}: {P.shape[0]} points, distance bit-identical {same.mean():.6f}, sign differs on {sign_diff.size} (all ambiguous), "
          f"sign checked on {int(ok.sum())} unambiguous of {idx.size}")


def test_empty_and_single_triangle(W):
    P = np.random.default_rng(1).uniform(-1, 1, (300, 3))
    assert np.all(sdf(W, np.zeros((0, 3)), np.zeros((0, 3), np.int64), P) == np.inf)
    V = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.1], [0.1, 0.6, -0.2]])
    against_restatement(sdf(W, V, np.array([[0, 1, 2]]), P), V, np.array([[0, 1, 2]]), P)


def test_duplicate_and_degenerate_triangles(W):
    V, F = MS.icosphere(2, 0.7)
    extra_v = np.array([[0.125, 0.125, 0.125], [0.25, 0.25, 0.25], [0.5, 0.5, 0.5], [0.25, -0.125, 0.0]])     # exactly collinear
    n = V.shape[0]
    V = np.concatenate([V, extra_v])
    F = np.concatenate([F, F[:40], [[n, n + 1, n + 2], [n + 3, n + 3, n + 3], [n, n, n + 1]]])      # duplicates, collinear, point, sliver
    P = np.concatenate([MS.near_points(V, F, 1500, np.random.default_rng(2)), extra_v, (extra_v[:3] + extra_v[1:4]) / 2])
    against_restatement(sdf(W, V, F, P), V, F, P)


def test_centre_of_icosphere_and_far_points(W):
    """The centre is equidistant from every triangle (the distance search cannot prune); points 10^3 away."""
    V, F = MS.icosphere(4, 0.8)
    rng = np.random.default_rng(3)
    far = rng.normal(size=(200, 3))
    far = 1e3 * far / np.linalg.norm(far, axis=1, keepdims=True)
    P = np.concatenate([np.zeros((1, 3)), far, MS.near_points(V, F, 100, rng)])
    got = sdf(W, V, F, P)
    against_restatement(got, V, F, P)
    assert 0.7 < abs(got[0]) <= 0.8


def test_nan_coordinates_and_sizes(W):
    V, F = MS.torus()
    rng = np.random.default_rng(4)
    P = MS.near_points(V, F, 50, rng)
    P[::7, rng.integers(0, 3)] = np.nan
    got = sdf(W, V, F, P)
    assert np.all(got[np.isnan(P).any(1)] == np.inf)
    against_restatement(got, V, F, P)
    assert sdf(W, V, F, np.zeros((0, 3))).shape == (0,)
    against_restatement(sdf(W, V, F, P[1:2]), V, F, P[1:2])
    big = MS.dataset_points(V, F, 2 ** 20 + 3, rng)
    got = sdf(W, V, F, big)
    idx = np.concatenate([subsample(big.shape[0], F.shape[0], 5)[:4000], [big.shape[0] - 1]])
    against_restatement(got[idx], V, F, big[idx])
    assert np.array_equal(got[idx], sdf(W, V, F, big[idx]))


def test_large_mesh(W):
    V, F = MS.torus(316, 316, 0.55, 0.25)
    V = V + np.random.default_rng(6).normal(scale=2e-4, size=V.shape)
    assert 1.9e5 < F.shape[0] < 2.1e5
    P = MS.dataset_points(V, F, 200000, np.random.default_rng(7))
    got = sdf(W, V, F, P)
    assert np.all(np.isfinite(got))
    idx = np.sort(np.random.default_rng(8).choice(P.shape[0], 512, replace=False))
    against_restatement(got[idx], V, F, P[idx])


def test_dtypes_devices_split_size(W):
    V, F = MS.noisy_sphere(3, seed=1)
    P = MS.dataset_points(V, F, 5000, np.random.default_rng(9))
    V32, P32 = V.astype(np.float32), P.astype(np.float32)
    Ft = torch.from_numpy(F)
    a = W.compute_sdf(torch.from_numpy(V32), Ft, torch.from_numpy(P32))                      # host float32, as the datasets pass
    b = W.compute_sdf(torch.from_numpy(V32).double().cuda(), Ft.cuda(), torch.from_numpy(P32).double().cuda())
    c = W.compute_sdf(torch.from_numpy(V32).cuda(), Ft.int().cuda(), torch.from_numpy(P32).cuda(), split_size=777)
    torch.cuda.synchronize()
    for t in (a, b, c):
        assert t.dtype == torch.float64 and t.is_cuda and t.shape == (P.shape[0], 1)
    assert torch.equal(a, b) and torch.equal(a, c)
    assert np.array_equal(np.signbit(a.cpu().numpy()), np.signbit(b.cpu().numpy()))


def test_launch_count(W):
    """wb_mesh_sdf: bounds, Morton codes, the radix sort (counted once), the Karras split, the refit and the query -- 6 launches for
    T >= 2, 5 for T = 1 (no internal node), 1 for T = 0 (the query alone), none for N = 0."""
    V, F = MS.cube()
    P = torch.zeros(10, 3, dtype=torch.float64, device="cuda")
    for f, n, expect in ((F, 10, 6), (F[:1], 10, 5), (F[:0], 10, 1), (F, 0, 0)):
        before = W._cabi.launch_count()
        W.compute_sdf(torch.from_numpy(V), torch.from_numpy(f), P[:n])
        assert W._cabi.launch_count() - before == expect
