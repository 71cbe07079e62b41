"""NumPy prototype of the device algorithm (design validation; mirrors run_sweep of gpy_b200/csrc/gpx_api.cu step by step).

Unified in-place sweep on one n x n buffer S (column-major on device):
  lower triangle : A -> L      (Cholesky factor)
  upper triangle : 0 -> U=L^-T (inverse factor, transposed), diagonal tiles of U kept in a strip
Every trailing update has the single form  S[r,c] -= P[r] @ P[c].T  (NT GEMM), and the final
K^-1 = U @ U.T restricted to k >= max(r,c) is again NT.
"""
import numpy as np

T = 4  # base tile (128 on device)


def base_sweep(tile):
    """Scalar unified sweep on a T x T tile held 'in registers': returns (L_dd lower, W_dd = L_dd^-1 lower, ok)."""
    S = tile.copy()
    n = S.shape[0]
    S[np.triu_indices(n, 1)] = 0.0  # V = 0
    ldiag = np.zeros(n)
    for j in range(n):
        a = S[j, j]
        if not (a > 0):
            return None, None, False
        l = np.sqrt(a); ldiag[j] = l; inv = 1.0 / l
        p = S[:, j] * inv
        p[j] = inv
        for col in range(j + 1, n):
            for row in range(n):
                if row >= col or row <= j:
                    S[row, col] -= p[row] * p[col]
        S[:, j] = np.where(np.arange(n) == j, S[j, j], p)
    L = np.tril(S, -1) + np.diag(ldiag)
    W = np.triu(S, 1).T + np.diag(1.0 / ldiag)
    return L, W, True


def sweep(S, n, step, Dinv, DinvT, off, level):
    """Factor-and-invert the n x n block S (view) in place. step = panel width at this level (multiple of T).
    Dinv/DinvT: dict tile_index -> T x T inverse diagonal tiles (global tile index = off//T + local)."""
    nt = n // T
    if step == T:
        for d in range(nt):
            sl = slice(d * T, (d + 1) * T)
            L, W, ok = base_sweep(S[sl, sl])
            assert ok
            S[sl, sl] = np.tril(L) + np.triu(S[sl, sl], 1) * 0
            g = off // T + d
            Dinv[g] = W; DinvT[g] = W.T.copy()
            # panel op, in place (K depth = one tile): P[r] = S[r,d] @ W^T for r != d
            for r in range(nt):
                if r == d: continue
                rs = slice(r * T, (r + 1) * T)
                S[rs, sl] = S[rs, sl] @ W.T
            # update: tiles (r,c), c>d, (r>=c or r<=d); operand row-tile d is DinvT
            def P(r):
                return DinvT[g] if r == d else S[r * T:(r + 1) * T, sl]
            for c in range(d + 1, nt):
                for r in list(range(0, d + 1)) + list(range(c, nt)):
                    rs = slice(r * T, (r + 1) * T); cs = slice(c * T, (c + 1) * T)
                    S[rs, cs] -= P(r) @ P(c).T
        return
    nb = n // step
    for k in range(nb):
        o = k * step
        blk = S[o:o + step, o:o + step]
        sweep(blk, step, T if level == 1 else step // 2, Dinv, DinvT, off + o, level - 1)
        # assemble Linv_kk (lower, dense) = transpose of block-upper part + Dinv diagonal tiles
        Tm = np.triu(blk, 0).T.copy()
        for d in range(step // T):
            g = (off + o) // T + d
            Tm[d * T:(d + 1) * T, d * T:(d + 1) * T] = Dinv[g]
        # panel op out-of-place into P (n x step); rows of the diagonal block get Linv_kk^T
        Pbuf = np.zeros((n, step))
        rows = np.r_[0:o, o + step:n]
        Pbuf[rows] = S[rows, o:o + step] @ Tm.T
        Pbuf[o:o + step] = Tm.T
        S[rows, o:o + step] = Pbuf[rows]          # copy back (memcpy2D on device)
        # unified trailing update, tile granularity T
        k1 = (o + step) // T; ntl = n // T
        for c in range(k1, ntl):
            for r in list(range(0, k1)) + list(range(c, ntl)):
                rs = slice(r * T, (r + 1) * T); cs = slice(c * T, (c + 1) * T)
                S[rs, cs] -= Pbuf[rs] @ Pbuf[cs].T


def run(n=32, step=8, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (n, 3))
    d2 = ((X[:, None] - X[None]) ** 2).sum(-1)
    K = np.exp(-0.5 * d2 / 3.0) + 0.01 * np.eye(n)
    S = np.tril(K)  # lower = A, upper = 0
    Dinv, DinvT = {}, {}
    sweep(S, n, step, Dinv, DinvT, 0, 1)
    nt = n // T
    L = np.tril(S)
    # swap diagonal tiles: U diag tiles <- DinvT
    U = np.triu(S, 1)
    for d in range(nt):
        sl = slice(d * T, (d + 1) * T)
        U[sl, sl] = DinvT[d]
    Lref = np.linalg.cholesky(K)
    print("L err", np.abs(L - Lref).max(), " U err", np.abs(U - np.linalg.inv(Lref).T).max())
    # LAUUM with restricted k-range, tile-wise
    Kinv = np.zeros_like(K)
    for r in range(nt):
        for c in range(r + 1):
            rs = slice(r * T, (r + 1) * T); cs = slice(c * T, (c + 1) * T)
            ks = slice(r * T, n)
            Kinv[rs, cs] = U[rs, ks] @ U[cs, ks].T
    Kinv = np.tril(Kinv) + np.tril(Kinv, -1).T
    print("Kinv err", np.abs(Kinv - np.linalg.inv(K)).max() / np.abs(np.linalg.inv(K)).max())
    y = rng.standard_normal(n)
    t = U.T @ y; alpha = U @ t
    print("alpha err", np.abs(alpha - np.linalg.solve(K, y)).max())


if __name__ == "__main__":
    run(32, 8); run(64, 16); run(48, 16)
