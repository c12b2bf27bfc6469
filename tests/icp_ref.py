"""A float64 restatement of one ICP step (numpy only), for tests that check the device solves in isolation.

Given the correspondence pairs (first = dst index, second = src index), the current transform T and the pivots, each
function returns the next transform the way the reference's estimators define it (transform_estimation.hpp):
  - p2p_step: estimateTransformPointToPointMetric - Kabsch on the centred pairs, numpy SVD, reflection fixed on U's
    LAST column;
  - combined_step: estimateTransformCombinedMetric / the symmetric metric, one Gauss-Newton step - the normal
    equations from eq_vecs and a = [(d + s) x n; n], solved in float64, then the atan / AngleAxis update,
    Translation(dst_mean) * . * Translation(-T src_mean);
and both finish like ICP's iteration: rotation() (SVD, reflection fixed on U's FIRST column), then compose with T.
The pairs are an input: the tests take them from the product and check them against the oracle separately, so a
difference here is a difference of the solve.
"""
import numpy as np

# la::polar_rotation (solve_core.hpp) runs when det(sigma) > POLAR_DET_RATIO |sigma|_F^3; the Jacobi SVD otherwise
POLAR_DET_RATIO = 1e-6


def det_ratio(sigma):
    """det(sigma) / |sigma|_F^3: the quantity polar_rotation's acceptance test compares with POLAR_DET_RATIO."""
    sigma = np.asarray(sigma, np.float64)
    f2 = float((sigma * sigma).sum())
    return float(np.linalg.det(sigma)) / (f2 * np.sqrt(f2)) if f2 > 0 else 0.0


def polar_accepts(sigma):
    """True when la::nearest_rotation(sigma) takes the Newton polar iteration, False when it takes the Jacobi SVD
    (the same test as polar_rotation's entry, in float64)."""
    sigma = np.asarray(sigma, np.float64)
    f2 = float((sigma * sigma).sum())
    if not (0.0 < f2 < 1e300):
        return False
    d0 = (sigma[0, 0] * (sigma[1, 1] * sigma[2, 2] - sigma[1, 2] * sigma[2, 1]) -
          sigma[0, 1] * (sigma[1, 0] * sigma[2, 2] - sigma[1, 2] * sigma[2, 0]) +
          sigma[0, 2] * (sigma[1, 0] * sigma[2, 1] - sigma[1, 1] * sigma[2, 0]))
    return bool(d0 > POLAR_DET_RATIO * f2 * np.sqrt(f2))


def apply(T, pts):
    T = np.asarray(T, np.float64)
    return np.asarray(pts, np.float64) @ T[:3, :3].T + T[:3, 3]


def apply_f32(T, pts):
    """q = R p + t in float32 with the product's contract order (solve_core.hpp apply_point): the points the
    device accumulates are these fp32 values."""
    T = np.asarray(T, np.float32)
    p = np.asarray(pts, np.float32).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        out = np.stack([(T[r, 0] * p[:, 0] + (T[r, 1] * p[:, 1] + T[r, 2] * p[:, 2])) + T[r, 3] for r in range(3)], 1)
    return out.astype(np.float32)


def identity():
    return np.hstack([np.eye(3), np.zeros((3, 1))])


def kabsch_rotation(sigma):
    """U V^T of sigma with the Kabsch reflection rule (last column of U)."""
    U, _, Vt = np.linalg.svd(np.asarray(sigma, np.float64))
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        U[:, 2] = -U[:, 2]
    return U @ Vt


def rotation(L):
    """LinearTransform::rotation(): U V^T with the reflection fixed on the FIRST column of U."""
    U, _, Vt = np.linalg.svd(np.asarray(L, np.float64))
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        U[:, 0] = -U[:, 0]
    return U @ Vt


def compose(A, B):
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    out = np.zeros((3, 4))
    out[:, :3] = A[:, :3] @ B[:, :3]
    out[:, 3] = A[:, :3] @ B[:, 3] + A[:, 3]
    return out


def kabsch(d, q):
    """estimateTransformPointToPointMetric on matched rows d[i] <-> q[i] (float64). Returns (T 3x4, sigma); no
    pairs -> identity, sigma = 0."""
    d, q = np.asarray(d, np.float64).reshape(-1, 3), np.asarray(q, np.float64).reshape(-1, 3)
    if len(d) == 0:
        return identity(), np.zeros((3, 3))
    mud, muq = d.mean(0), q.mean(0)
    sigma = (d - mud).T @ (q - muq) / len(d)
    R = kabsch_rotation(sigma)
    return np.hstack([R, (mud - R @ muq)[:, None]]), sigma


def finish(Titer, T):
    """ICP's iteration epilogue: rotation() on the update's linear part, then update * T."""
    Tr = np.asarray(Titer, np.float64).copy()
    Tr[:, :3] = rotation(Tr[:, :3])
    return compose(Tr, T)


def p2p_step(dst, src, T, first, second):
    """One point-to-point ICP iteration from the pairs. Returns (T_next, info) with info = dict(sigma, polar)."""
    q = apply_f32(T, np.asarray(src)[second])
    Titer, sigma = kabsch(np.asarray(dst, np.float64)[first], q)
    return finish(Titer, T), dict(sigma=sigma, polar=polar_accepts(sigma), n=len(first))


def normal_equations(d, s, w_pt, w_pl, n=None):
    """AtA (6x6) and Atb of the combined metric's Gauss-Newton step on centred matched rows d (destination minus
    dst_mean), s (transformed source minus T src_mean) and normals n (dst normals, or the symmetric metric's sum), as
    transform_estimation.hpp:298-343 builds them, in float64."""
    d, s = np.asarray(d, np.float64).reshape(-1, 3), np.asarray(s, np.float64).reshape(-1, 3)
    v, e = d + s, d - s
    A, b = np.zeros((6, 6)), np.zeros(6)
    if w_pt > 0:
        # E = [[v]x ; I]: E E^T = [[|v|^2 I - v v^T, [v]x], [-[v]x, I]], E e = [v x e ; e]
        vv = (v * v).sum()
        A[:3, :3] += w_pt * (vv * np.eye(3) - v.T @ v)
        sv = v.sum(0)
        vx = np.array([[0, -sv[2], sv[1]], [sv[2], 0, -sv[0]], [-sv[1], sv[0], 0]])
        A[:3, 3:] += w_pt * vx
        A[3:, :3] -= w_pt * vx
        A[3:, 3:] += w_pt * len(v) * np.eye(3)
        b[:3] += w_pt * np.cross(v, e).sum(0)
        b[3:] += w_pt * e.sum(0)
    if w_pl > 0:
        n = np.asarray(n, np.float64).reshape(-1, 3)
        a = np.hstack([np.cross(v, n), n])
        r = (n * e).sum(1)
        A += w_pl * a.T @ a
        b += w_pl * a.T @ r
    return A, b


def gauss_newton_update(x, Tin=None):
    """T_out = Ra * Translation(cos(theta) v) * Ra * T_in from d_theta = x (transform_estimation.hpp:346-357)."""
    x = np.asarray(x, np.float64)
    Tin = identity() if Tin is None else np.asarray(Tin, np.float64)
    na = np.linalg.norm(x[:3])
    theta = np.arctan(na)
    ax = x[:3] / na if na > 0 else np.zeros(3)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    Ra = np.cos(theta) * np.eye(3) + np.sin(theta) * K + (1 - np.cos(theta)) * np.outer(ax, ax)
    out = np.zeros((3, 4))
    out[:, :3] = Ra @ Ra @ Tin[:, :3]
    out[:, 3] = Ra @ (Ra @ Tin[:, 3] + np.cos(theta) * x[3:])
    return out


def combined_step(dst, dst_n, src, T, first, second, w_pt, w_pl, dst_mean, src_mean, src_n=None):
    """One combined-metric (or, with src_n, symmetric-metric) ICP iteration with one Gauss-Newton step, from the
    pairs and the pivots (dst_mean, src_mean: the means the product uses, float32). Returns (T_next, info) with
    info = dict(A, b, cond = 2-norm condition number of AtA)."""
    T = np.asarray(T, np.float64)
    dm = np.asarray(dst_mean, np.float32)
    sm = apply_f32(T, np.asarray(src_mean, np.float32)[None])[0]
    q = apply_f32(T, np.asarray(src)[second]).astype(np.float64)
    d = np.asarray(dst, np.float64)[first] - dm
    s = q - sm
    nrm = None
    if w_pl > 0:
        nrm = np.asarray(dst_n, np.float64)[first]
        if src_n is not None:
            nrm = nrm + np.asarray(src_n, np.float64)[second] @ T[:, :3].T
    if len(first) == 0 or not (w_pt > 0 or w_pl > 0):
        return compose(identity(), T), dict(A=np.zeros((6, 6)), b=np.zeros(6), cond=1.0)
    A, b = normal_equations(d, s, w_pt, w_pl, nrm)
    x = np.linalg.solve(A, b)
    Titer = gauss_newton_update(x)
    Titer[:, 3] = Titer[:, 3] - Titer[:, :3] @ sm.astype(np.float64) + dm.astype(np.float64)  # un-centre (:365)
    return finish(Titer, T), dict(A=A, b=b, cond=float(np.linalg.cond(A)))


def finite_rows(pts):
    return np.isfinite(np.asarray(pts, np.float64)).all(1)
