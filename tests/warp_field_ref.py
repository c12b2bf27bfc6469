"""A float64 statement of the dense warp-field normal equations that scales to 10^6 points: the system the oracle
assembles (oracle.warp_field.system: the data blocks B_i, the right-hand side g and the arc couplings c_e) written as

    A = blockdiag(B_i) + sum_e c_e (.) L_e,   L_e the graph Laplacian of arc e = (lo, hi), one per unknown u,

without Python loops over points or arcs. `matrix()` forms A as a scipy.sparse matrix (for the small cases of the CPU
pins); `matvec()` applies it without forming it, so that a device solution on 10^5-10^6 points can be judged by its
true relative residual |A x - g| / |g| in float64."""
import numpy as np
import scipy.sparse as sp

_IU = np.triu_indices(6)  # (row, col) of the 21 upper-triangle entries, row-major: the order of B_i


class NormalSystem:
    """The normal equations of one Gauss-Newton step, from the dict of oracle.warp_field.system()."""

    def __init__(self, sysd):
        self.B = np.asarray(sysd["B"], np.float64)
        self.n = self.B.shape[0]
        self.g = np.asarray(sysd["g"], np.float64).reshape(-1)
        self.c = np.asarray(sysd["arc_c"], np.float64).reshape(-1, 6)
        self.lo = np.asarray(sysd["lo"], np.int64)
        self.hi = np.asarray(sysd["hi"], np.int64)
        full = np.zeros((self.n, 6, 6))
        full[:, _IU[0], _IU[1]] = self.B
        full[:, _IU[1], _IU[0]] = self.B
        self.blocks = full

    def matrix(self):
        """A as a (6n, 6n) scipy.sparse CSR matrix (duplicate arcs summed, as in A = J^T J)."""
        n, m = self.n, self.lo.shape[0]
        base = 6 * np.arange(n)
        r_blk = (base[:, None, None] + np.arange(6)[None, :, None]).repeat(6, 2).reshape(-1)
        c_blk = (base[:, None, None] + np.arange(6)[None, None, :]).repeat(6, 1).reshape(-1)
        u = np.arange(6)
        lo = (6 * self.lo[:, None] + u).reshape(-1)
        hi = (6 * self.hi[:, None] + u).reshape(-1)
        c = self.c.reshape(-1)
        rows = np.concatenate([r_blk, lo, hi, lo, hi])
        cols = np.concatenate([c_blk, lo, hi, hi, lo])
        vals = np.concatenate([self.blocks.reshape(-1), c, c, -c, -c])
        assert rows.shape[0] == 36 * n + 24 * m
        return sp.coo_matrix((vals, (rows, cols)), shape=(6 * n, 6 * n)).tocsr()

    def matvec(self, x):
        """A x in float64 without forming A: B_i x_i + sum over the arcs e at i of c_e (.) (x_i - x_other(e))."""
        x = np.asarray(x, np.float64).reshape(self.n, 6)
        q = np.einsum("nrc,nc->nr", self.blocks, x)
        if self.lo.shape[0]:
            d = self.c * (x[self.lo] - x[self.hi])  # the lower end gets +d, the upper end -d
            for u in range(6):
                q[:, u] += np.bincount(self.lo, d[:, u], self.n) - np.bincount(self.hi, d[:, u], self.n)
        return q.reshape(-1)

    def true_rel_residual(self, x):
        """|A x - g| / |g| in float64 (0 when g = 0 and A x = 0)."""
        r = np.linalg.norm(self.matvec(x) - self.g)
        gn = np.linalg.norm(self.g)
        return float(r / gn) if gn > 0 else float(r)


def system(wf, dst, dst_n, src, first, second, nbhd, x=None, **kw):
    """NormalSystem at the unknowns x (n, 6) (zero by default); kw as oracle.warp_field.system."""
    n = np.asarray(src).reshape(-1, 3).shape[0]
    x = np.zeros((n, 6)) if x is None else np.asarray(x, np.float64).reshape(n, 6)
    return NormalSystem(wf.system(dst, dst_n, src, first, second, nbhd, x, **kw))
