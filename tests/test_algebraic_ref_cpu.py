"""The weighted DLT (csrc/algebraic.cu) against a high-precision reference, on the CPU through the kernels' own per-item code.

Reference:
- A is built from float32 rows formed exactly as the kernels form them: (P[2] * x - P[0]) * c with one float32 rounding per
  operation (numpy does not fuse), then widened.  Forward and backward are therefore compared on the same A.
- Forward: the eigenvector of A^T A for its smallest eigenvalue (the right singular vector of A for its smallest singular
  value), solved by mpmath at 50 digits; squaring the condition number costs nothing at that precision.
- Backward: central differences of that forward in the direction each input moves A: d x moves row 2v by c P[2], d y row 2v+1,
  d c both rows by the unweighted rows.  Independent of the perturbation formula the kernel applies.
- Bars per element, from the solve's conditioning: the kernel forms A^T A and rotates it in float64, an error bounded
  componentwise by eta * d_i * d_j (d = column norms of A, eta = (2V + 400) 2^-53: the 2V-term sums and at most 16 sweeps of
  6 rotations).  That moves the eigenvector u towards e_k by eta (d.|e_k|)(d.|u|) / |lambda_0 - lambda_k|, and X = u[0:3] / u[3]
  by that over |u[3]|; plus the float32 rounding of the output.  Gradients: the same relative error, taken over all eigenpair
  gaps, times the magnitude of the terms each element sums, plus its float32 rounding.
The GPU launches of the same scenes are in tests/test_gpu_algebraic_ref.py."""
import math

import mpmath
import numpy as np
import pytest
import torch

from lt_b200 import capi, testing

F32 = np.float32
ULP32 = 2.0 ** -23              # one float32 ulp, relative: the rounding of each output and then some
EPS64 = 2.0 ** -53
MP_DPS = 50
FD_STEP = "1e-18"


# ---- scenes -----------------------------------------------------------------------------------------------------------

def ring(V, step_deg=None, image_size=384):
    """(V, 3, 4) float32 projections: `make_cameras`' ring (90 degrees apart at V = 4), or V cameras step_deg apart on it."""
    if step_deg is None:
        cams = testing.make_cameras(V, image_size=image_size)
    else:
        cams = [testing.make_cameras(1, image_size=image_size, phase=0.3 + math.radians(step_deg) * v)[0] for v in range(V)]
    return np.stack([c.projection for c in cams]).astype(F32)


def confidences(kind, B, V, J, rng):
    if kind is None:
        return None
    if kind == "rand":
        return (rng.rand(B, V, J) + 0.1).astype(F32)
    if kind == "zero_view":                           # view 1 has confidence 0
        c = (rng.rand(B, V, J) + 0.1).astype(F32)
        c[:, 1] = 0
        return c
    if kind == "tiny":
        return np.full((B, V, J), 1e-6, F32)
    if kind == "zero":                                # A = 0: every eigenvalue ties
        return np.zeros((B, V, J), F32)
    if kind.startswith("graded"):                     # "graded1e-4": view 0 at 1, the others at 1e-4
        c = np.full((B, V, J), float(kind[6:]), F32)
        c[:, 0] = 1
        return c
    raise ValueError(kind)


def make_scene(V, B=1, J=4, noise=2.0, step_deg=None, image_size=384, far=False, conf="rand", seed=0):
    """-> proj (B, V, 3, 4), kp2d (B, V, J, 2), conf (B, V, J) or None, grad_out (B, J, 3), all float32 numpy.  Points
    ~ N(0, 300^2) + (0, 0, 900) mm (far: ~1e5 mm away), projected and given `noise` px of Gaussian noise."""
    rng = np.random.RandomState(seed)
    P = np.repeat(ring(V, step_deg, image_size)[None], B, axis=0)
    X = rng.randn(B, J, 3) * 300 + [0, 0, 900]
    if far:
        X = X + [6e4, -8e4, 0]
    uvw = np.einsum("bvij,bkj->bvki", P.astype(np.float64), np.concatenate([X, np.ones((B, J, 1))], -1))
    kp = (uvw[..., :2] / uvw[..., 2:3] + rng.randn(B, V, J, 2) * noise).astype(F32)
    g = rng.randn(B, J, 3).astype(F32)
    return P, kp, confidences(conf, B, V, J, rng), g


def scene_id(s):
    return "-".join("%s=%s" % kv for kv in sorted(s.items()))


# (V, conf) on the 90-degree ring, 2 px and noise-free; then the geometry edges; then the confidence edges on V = 4
SCENES = ([dict(V=V, noise=n, conf=c) for V in (2, 3, 4, 8) for n in (0.0, 2.0) for c in (None, "rand")]
          + [dict(V=V, step_deg=d, noise=n, conf=c) for V in (2, 4) for d in (1.0, 0.1) for n in (0.0, 2.0) for c in (None, "rand")]
          + [dict(V=4, far=True, conf=c) for c in (None, "rand")]
          + [dict(V=4, image_size=1000, conf=c) for c in (None, "rand")]
          + [dict(V=4, conf=c) for c in ("graded1e-2", "graded1e-3", "graded1e-4", "graded1e-5", "graded1e-6", "zero_view", "tiny")])


# ---- reference --------------------------------------------------------------------------------------------------------

def dlt_rows32(P, kp, cf):
    """Weighted and unweighted DLT rows of one item as the kernels round them: P (V, 3, 4), kp (V, 2), cf (V,) float32 or None
    -> A (2V, 4) and U (2V, 4) float64 (row 2v from x, 2v+1 from y)."""
    V = P.shape[0]
    c = np.ones(V, F32) if cf is None else cf.astype(F32)
    u0 = P[:, 2] * kp[:, 0:1] - P[:, 0]
    u1 = P[:, 2] * kp[:, 1:2] - P[:, 1]
    U = np.stack([u0, u1], 1).reshape(2 * V, 4)
    A = np.stack([u0 * c[:, None], u1 * c[:, None]], 1).reshape(2 * V, 4)
    assert A.dtype == F32 and U.dtype == F32
    return A.astype(np.float64), U.astype(np.float64)


def mp_eigen(A):
    """Eigenpairs of A^T A, ascending, at MP_DPS digits: (lam [4] mpf, E 4x4 mp.matrix, columns normalised)."""
    with mpmath.workdps(MP_DPS):
        Am = A if isinstance(A, mpmath.matrix) else mpmath.matrix(A.tolist())
        lam, E = mpmath.eigsy(Am.T * Am)
        order = sorted(range(4), key=lambda k: lam[k])
        return [lam[k] for k in order], mpmath.matrix([[E[r, k] for k in order] for r in range(4)])


def mp_point(A):
    with mpmath.workdps(MP_DPS):
        _, E = mp_eigen(A)
        return [E[i, 0] / E[3, 0] for i in range(3)]


def dlt_reference(P, kp, cf):
    """One item: X (3,) float64 from the 50-digit solve, and what the bars need."""
    A, U = dlt_rows32(P, kp, cf)
    with mpmath.workdps(MP_DPS):
        lam, E = mp_eigen(A)
        X = np.array([float(E[i, 0] / E[3, 0]) for i in range(3)])
    return dict(A=A, U=U, X=X, lam=np.array([float(v) for v in lam]), E=np.array(E.tolist(), dtype=np.float64))


def eta(V):
    return (2 * V + 400) * EPS64


def spreads(ref):
    """s_k = d . |e_k| with d the column norms of A: the componentwise error bound of A^T A, seen along e_k."""
    A = ref["A"]
    return np.sqrt((A * A).sum(0)) @ np.abs(ref["E"])


def eigvec_err(ref):
    """First-order bound (4,) of the kernel's error in u = e_0."""
    lam, E, s = ref["lam"], ref["E"], spreads(ref)
    du = sum(np.abs(E[:, k]) * s[k] * s[0] / max(abs(lam[0] - lam[k]), 1e-300) for k in range(1, 4))
    return eta(ref["A"].shape[0] // 2) * du


def forward_bar(ref):
    """Per-coordinate bar of X (see the module docstring)."""
    X, u3, du = ref["X"], abs(ref["E"][3, 0]), eigvec_err(ref)
    return (du[:3] + np.abs(X) * du[3]) / u3


def grad_reference(P, kp, cf, g):
    """Central differences of the 50-digit forward: (grad_kp (V, 2), grad_conf (V,) or None) of g . X."""
    V = P.shape[0]
    A, U = dlt_rows32(P, kp, cf)
    c = np.ones(V) if cf is None else cf.astype(np.float64)
    gk, gc = np.zeros((V, 2)), (None if cf is None else np.zeros(V))
    with mpmath.workdps(MP_DPS):
        h = mpmath.mpf(FD_STEP)
        Am = mpmath.matrix(A.tolist())

        def directional(rows_dirs):
            res = []
            for sign in (1, -1):
                Ah = Am.copy()
                for r, dvec in rows_dirs:
                    for col in range(4):
                        Ah[r, col] += sign * h * mpmath.mpf(float(dvec[col]))
                res.append(mp_point(Ah))
            return float(sum(mpmath.mpf(float(g[i])) * (res[0][i] - res[1][i]) for i in range(3)) / (2 * h))

        for v in range(V):
            p2 = P[v, 2].astype(np.float64)
            gk[v, 0] = directional([(2 * v, c[v] * p2)])
            gk[v, 1] = directional([(2 * v + 1, c[v] * p2)])
            if cf is not None:
                gc[v] = directional([(2 * v, U[2 * v]), (2 * v + 1, U[2 * v + 1])])
    return gk, gc


def grad_bars(P, kp, cf, g, ref):
    """Per-element bars of grad_kp (V, 2) and grad_conf (V,): rho x (magnitude of the terms the kernel sums) + float32 rounding
    of the result (added by the caller, which knows the value)."""
    A, U, lam, E = ref["A"], ref["U"], ref["lam"], ref["E"]
    V = P.shape[0]
    s = spreads(ref)
    u = E[:, 0]
    # relative error of the eigen-system as the gradient uses it: every pair's rotation and both eigenvalues against their gap,
    # and u[3], which gu divides by; x 4 for the first-order terms adding up
    rho = eta(V) * max((s[j] * s[k] + s[j] ** 2 + s[k] ** 2) / max(abs(lam[j] - lam[k]), 1e-300)
                       for j in range(4) for k in range(j + 1, 4))
    rho = 4 * (rho + eigvec_err(ref)[3] / abs(u[3]))
    iw = 1.0 / abs(u[3])
    gu = np.abs(np.concatenate([g.astype(np.float64) * iw, [np.abs(g.astype(np.float64) * u[:3]).sum() * iw * iw]]))
    wabs = sum((gu @ np.abs(E[:, k])) / max(abs(lam[0] - lam[k]), 1e-300) * np.abs(E[:, k]) for k in range(1, 4))
    ua = np.abs(u)
    c = np.ones(V) if cf is None else np.abs(cf.astype(np.float64))
    bk, bc = np.zeros((V, 2)), np.zeros(V)
    for v in range(V):
        p2 = np.abs(P[v, 2].astype(np.float64))
        tot_c = 0.0
        for r in range(2):
            a = np.abs(A[2 * v + r])
            t = (a @ wabs) * ua + (a @ ua) * wabs          # |row r of G_A|, termwise
            bk[v, r] = c[v] * (t @ p2)
            tot_c += t @ np.abs(U[2 * v + r])
        bc[v] = tot_c
    return rho * bk, rho * bc


def err_over_bar(got, want, bar):
    """Worst |got - want| / (bar + one float32 ulp of want)."""
    return float(np.max(np.abs(np.asarray(got, np.float64) - want) / (bar + ULP32 * np.abs(want) + 1e-30)))


# ---- host hooks -------------------------------------------------------------------------------------------------------

def host_forward(P, kp, conf):
    out = torch.full((kp.shape[0], kp.shape[2], 3), float("nan"))
    capi.triangulate_dlt_host(torch.from_numpy(P), torch.from_numpy(kp), None if conf is None else torch.from_numpy(conf), out)
    return out.numpy()


def host_backward(P, kp, conf, g):
    gk = torch.full(kp.shape, float("nan"))
    gc = None if conf is None else torch.full(conf.shape, float("nan"))
    capi.triangulate_dlt_bwd_host(torch.from_numpy(P), torch.from_numpy(kp), None if conf is None else torch.from_numpy(conf),
                                  torch.from_numpy(g), gk, gc)
    return gk.numpy(), None if gc is None else gc.numpy()


def item(P, kp, conf, b, j):
    return P[b], kp[b, :, j], None if conf is None else conf[b, :, j]


def check_forward(P, kp, conf, got):
    """Worst err/bar over every item of a scene (got: (B, J, 3))."""
    worst = 0.0
    for b in range(kp.shape[0]):
        for j in range(kp.shape[2]):
            ref = dlt_reference(*item(P, kp, conf, b, j))
            worst = max(worst, err_over_bar(got[b, j], ref["X"], forward_bar(ref)))
    return worst


def check_backward(P, kp, conf, g, gk, gc, items):
    """Worst err/bar of the gradients over `items` [(b, j)] (the mpmath differences are the cost: 6V solves per item)."""
    worst = 0.0
    for b, j in items:
        Pi, kpi, cfi = item(P, kp, conf, b, j)
        ref = dlt_reference(Pi, kpi, cfi)
        wk, wc = grad_reference(Pi, kpi, cfi, g[b, j])
        bk, bc = grad_bars(Pi, kpi, cfi, g[b, j], ref)
        worst = max(worst, err_over_bar(gk[b, :, j], wk, bk))
        if conf is not None:
            worst = max(worst, err_over_bar(gc[b, :, j], wc, bc))
    return worst


@pytest.mark.parametrize("scene", SCENES, ids=scene_id)
def test_dlt_forward_item_code_vs_high_precision(scene):
    P, kp, conf, _ = make_scene(B=2, J=4, seed=1, **scene)
    got = host_forward(P, kp, conf)
    assert np.isfinite(got).all()
    worst = check_forward(P, kp, conf, got)
    print("dlt forward (host) %s: worst err/bar %.3g" % (scene_id(scene), worst))
    assert worst <= 1.0


@pytest.mark.parametrize("scene", SCENES, ids=scene_id)
def test_dlt_backward_item_code_vs_high_precision(scene):
    P, kp, conf, g = make_scene(B=1, J=3, seed=2, **scene)
    gk, gc = host_backward(P, kp, conf, g)
    assert np.isfinite(gk).all() and (gc is None or np.isfinite(gc).all())
    worst = check_backward(P, kp, conf, g, gk, gc, [(0, j) for j in range(3)])
    print("dlt backward (host) %s: worst err/bar %.3g" % (scene_id(scene), worst))
    assert worst <= 1.0


def test_dlt_backward_keeps_the_main_term_on_graded_confidences():
    """Confidences (1, 1e-4, 1e-4, 1e-4): the eigenvalues of A^T A are ~6e-6, 5.6e-3, 2.7e5 and 4.9e11.  A tie threshold scaled
    by the largest eigenvalue (1e-12 x 4.9e11) dropped the 5.6e-3 gap, the term with the largest weight, and the gradient came
    out wrong by ~1x its maximum."""
    P, kp, conf, g = make_scene(V=4, B=1, J=1, seed=0, conf="graded1e-4")
    ref = dlt_reference(*item(P, kp, conf, 0, 0))
    assert ref["lam"][1] < 1e-12 * ref["lam"][3] < ref["lam"][2]
    gk, gc = host_backward(P, kp, conf, g)
    wk, wc = grad_reference(*item(P, kp, conf, 0, 0), g[0, 0])
    e = max(np.abs(gk[0, :, 0] - wk).max() / np.abs(wk).max(), np.abs(gc[0, :, 0] - wc).max() / np.abs(wc).max())
    print("graded confidences: max|err| / max|grad| = %.3g" % e)
    assert e <= 1e-5


def test_dlt_backward_is_zero_on_an_exact_tie():
    """All confidences zero: A = 0, every eigenvalue ties with the smallest, every term is dropped: the gradient is exactly 0."""
    P, kp, conf, g = make_scene(V=3, B=1, J=2, seed=3, conf="zero")
    gk, gc = host_backward(P, kp, conf, g)
    assert np.isfinite(gk).all() and np.isfinite(gc).all()
    assert not gk.any() and not gc.any()


def point_at_infinity_scene(V=3, seed=4):
    """Item 0 sees the direction (1, 0, 0, 0) in every view: column 0 of every P is (200, 100, 1) x 2^k and the key point is
    (200, 100), so column 0 of A is exactly 0 and u = (1, 0, 0, 0) exactly (u[3] = 0).  Item 1 is an ordinary point."""
    P, kp, conf, g = make_scene(V=V, B=1, J=2, seed=seed, conf="rand")
    P[0, :, :, 0] = np.array([200.0, 100.0, 1.0], F32) * (2.0 ** np.arange(V, dtype=F32))[:, None]
    X = np.array([100.0, -200.0, 900.0, 1.0])
    uvw = np.einsum("vij,j->vi", P[0].astype(np.float64), X)
    kp[0, :, 1] = (uvw[:, :2] / uvw[:, 2:3]).astype(F32)
    kp[0, :, 0] = [200.0, 100.0]
    return P, kp, conf, g


def test_dlt_point_at_infinity_is_pinned():
    """u[3] = 0: the forward divides by zero like the reference's dehomogenisation, (+inf, nan, nan); its backward divides by u[3]
    too, so every gradient of that item is NaN.  The other item is unaffected."""
    P, kp, conf, g = point_at_infinity_scene()
    out = host_forward(P, kp, conf)
    assert out[0, 0, 0] == np.inf and np.isnan(out[0, 0, 1:]).all()
    assert np.isfinite(out[0, 1]).all()
    gk, gc = host_backward(P, kp, conf, g)
    assert np.isnan(gk[0, :, 0]).all() and np.isnan(gc[0, :, 0]).all()
    assert np.isfinite(gk[0, :, 1]).all() and np.isfinite(gc[0, :, 1]).all()


def test_reference_rows_are_the_float32_rows():
    """The reference forms each entry with three float32 roundings, not with one fused multiply-subtract: on this scene the two
    differ, so a fused kernel would not reproduce the reference's A."""
    P, kp, conf, _ = make_scene(V=4, B=1, J=8, seed=5)
    p2, p0, x, c = P[0, :, 2][:, None], P[0, :, 0][:, None], kp[0, :, :, 0][..., None], conf[0][..., None]   # (V, J, 4)
    unfused = (np.float32(1) * (p2 * x) - p0) * c
    fused = (p2.astype(np.float64) * x - p0).astype(F32) * c          # the float64 product is exact: one rounding, as an FMA
    for j in range(8):
        A, _ = dlt_rows32(P[0], kp[0, :, j], conf[0, :, j])
        assert np.array_equal(A[0::2], unfused[:, j].astype(np.float64))
    assert (fused != unfused).mean() > 0.1
