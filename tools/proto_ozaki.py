"""Numerical prototype (CPU, NumPy) of the digit-split kernel: the N^3 GEMMs of the factor-and-invert sweep computed by an
Ozaki split on INT8 tensor cores (wgmma s8 x s8 -> s32, exact int32 accumulation) instead of fp64 DMMA.

  * each row of an operand is scaled by a power of two to (-1, 1) and cut into S signed 7-bit digits (int8),
  * C = A B^T = sum_{s+t <= S+1} 2^(e_i + f_j - 7(s+t)) * (D_s^A D_t^B^T), every digit product accumulated EXACTLY
    (emulated with integer-valued fp64 here, exact below 2^53; on the device |digit| <= 127 and k <= 2^17 keeps the sum inside int32),
  * the per-(s+t) groups are converted and added in fp64, smallest magnitude first.

What this answers before any device code is written: how many digits S the exact-GP evaluation needs to stay inside the
tolerances of BASELINE.json (|dLML| <= 1e-8, gradient 1e-6 relative) when ONLY the outer panel / trailing-update / U U^T
products go through the split (the 128-wide diagonal blocks stay fp64, as they would on DMMA), and how many int8 GEMMs
that costs (S(S+1)/2 slice pairs).

    python tools/proto_ozaki.py [N] [NB]
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gpy_oracle as o  # noqa: E402

BITS = 7


def split_rows(A, S):
    """-> (digits [S][m][k] integer-valued with |d| <= 127, exponents e[m]) such that A = 2^e * sum_s d_s 2^(-7 s) + O(2^(-7S))."""
    amax = np.abs(A).max(axis=1)
    e = np.where(amax > 0, np.floor(np.log2(np.where(amax > 0, amax, 1.0))) + 1, 0).astype(np.int64)
    r = np.ldexp(A, (-e)[:, None].astype(np.int32))          # |r| < 1, exact (power-of-two scaling)
    digs = []
    for _ in range(S):
        r = r * 128.0                                         # exact
        d = np.trunc(r)                                       # |d| <= 127
        r = r - d                                             # exact, same sign as before, |r| < 1
        digs.append(d)                                        # kept as float64: all integer sums below stay < 2^53 (exact)
    return digs, e


def ozaki_nt(A, B, S):
    """C = A @ B.T through the int8 split with S digits per operand and slice pairs s + t <= S + 1."""
    dA, eA = split_rows(A, S)
    dB, eB = split_rows(B, S)
    C = np.zeros((A.shape[0], B.shape[0]))
    for g in range(S + 1, 1, -1):                             # groups by s + t = g, smallest magnitude first
        acc = np.zeros((A.shape[0], B.shape[0]))              # integer-valued, |acc| <= 127^2 k S < 2^53: exact in fp64
        for s in range(1, S + 1):
            t = g - s
            if 1 <= t <= S:
                acc += dA[s - 1] @ dB[t - 1].T                # exact integer GEMM (int32-safe per pair on the device)
        C += np.ldexp(acc, -BITS * g)
    return np.ldexp(C, (eA[:, None] + eB[None, :]).astype(np.int32))


def pairs(S):
    return sum(1 for s in range(1, S + 1) for t in range(1, S + 1) if s + t <= S + 1)


def evaluate(X, Y, var, ls, noise, NB, mm, mmU=None):
    """One exact-GP evaluation with the blocked factor-and-invert sweep; every outer product goes through mm(A, B) = A B^T
    (mm: the Cholesky part = rows at / below the block, which feeds log|K| and alpha; mmU: the inverse part = rows above
    the block and K^-1 = U U^T, which only feeds the gradients)."""
    mmU = mm if mmU is None else mmU
    N, D = X.shape
    Xs = X / ls
    sq = (Xs ** 2).sum(1)
    r2 = np.maximum(sq[:, None] + sq[None, :] - 2 * Xs @ Xs.T, 0.0)
    np.fill_diagonal(r2, 0.0)
    K = var * np.exp(-0.5 * r2)
    S = np.tril(K + (noise + 1e-8) * np.eye(N))               # lower = Ky, upper = 0 -> U
    logdet = 0.0
    ldiag = np.zeros(N)
    for o_ in range(0, N, NB):
        sl = slice(o_, o_ + NB)
        Lkk = np.linalg.cholesky(S[sl, sl] + np.tril(S[sl, sl], -1).T)      # diagonal block: stays fp64
        Linv = np.linalg.inv(Lkk)
        logdet += 2 * np.log(np.diag(Lkk)).sum()
        ldiag[sl] = np.diag(Lkk)
        P = np.zeros((N, NB))
        rows = np.r_[0:o_, o_ + NB:N]
        if o_ > 0:
            P[:o_] = mmU(S[:o_, sl], Linv)                    # panel, rows above: finished block column of U
        if o_ + NB < N:
            P[o_ + NB:] = mm(S[o_ + NB:, sl], Linv)           # panel, rows below: Cholesky panel
        P[sl] = Linv.T
        S[rows, sl] = P[rows]
        S[sl, sl] = np.tril(Lkk, -1) + np.triu(Linv.T)
        k1 = o_ + NB
        if k1 < N:
            upd = np.vstack([mmU(P[:k1], P[k1:]), mm(P[k1:], P[k1:])])   # trailing update: inverse part | Cholesky part
            cols = np.arange(k1, N)
            rr = np.arange(N)[:, None]
            mask = (rr < k1) | (rr >= cols[None, :] - (cols[None, :] % 1))   # rows [0,k1) U [c, N): element granularity
            S[:, k1:] -= np.where(mask, upd, 0.0)
    U = np.triu(S)                                            # L^-T
    from scipy.linalg import solve_triangular
    L = np.tril(S, -1) + np.diag(ldiag)
    t = solve_triangular(L, Y, lower=True)                    # the quadratic form of the bound from the Cholesky part only
    alpha = U @ (U.T @ Y)                                     # alpha (gradients) from the inverse part
    Kinv = mmU(U, U)                                          # U U^T
    lml = 0.5 * (-N * Y.shape[1] * np.log(2 * np.pi) - Y.shape[1] * logdet - float((t * t).sum()))
    dL = 0.5 * (alpha @ alpha.T - Y.shape[1] * Kinv)
    dvar = (K * dL).sum() / var
    dls = np.array([(-(K * dL) * -((Xs[:, q][:, None] - Xs[None, :, q]) ** 2)).sum() / ls[q] for q in range(D)])
    return lml, np.concatenate([[dvar], dls, [np.trace(dL)]])


def main():
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 768
    NB = int(sys.argv[2]) if len(sys.argv) > 2 else 128
    D = 8
    X, Y = o.synthetic(N, D)
    var, ls, noise = o.theta_bench(D, True)
    lml0, g0, _ = o.eval_lml_grad(X, Y, "rbf", True, var, ls, noise)
    lml, g = evaluate(X, Y, var, ls, noise, NB, lambda A, B: A @ B.T)
    print("N=%d NB=%d  blocked sweep in fp64:        |dLML| %.2e  grad rel %.2e" % (N, NB, abs(lml - lml0), np.max(np.abs(g - g0) / np.abs(g0))))
    for S in (5, 6, 7, 8, 9):
        lml, g = evaluate(X, Y, var, ls, noise, NB, lambda A, B: ozaki_nt(A, B, S))
        print("  int8 split, %d digits (%2d slice-pair GEMMs): |dLML| %.2e  grad rel %.2e" % (
            S, pairs(S), abs(lml - lml0), np.max(np.abs(g - g0) / np.abs(g0))))
    for (SL, SU) in ((8, 5), (8, 6), (9, 6)):
        lml, g = evaluate(X, Y, var, ls, noise, NB, lambda A, B: ozaki_nt(A, B, SL), lambda A, B: ozaki_nt(A, B, SU))
        print("  mixed: Cholesky part %d digits, inverse part + U U^T %d digits (flop-weighted %.1f slice-pair GEMMs): "
              "|dLML| %.2e  grad rel %.2e" % (SL, SU, (pairs(SL) + 2 * pairs(SU)) / 3.0, abs(lml - lml0),
                                             np.max(np.abs(g - g0) / np.abs(g0))))
    # plain GEMM accuracy on the operand type of the update (a panel of the sweep has rows of very different scale)
    rng = np.random.default_rng(0)
    A = rng.standard_normal((256, 1024)) * np.exp(rng.uniform(-8, 8, (256, 1)))
    B = rng.standard_normal((256, 1024)) * np.exp(rng.uniform(-8, 8, (256, 1)))
    ref = (A.astype(np.longdouble) @ B.T.astype(np.longdouble))
    den = (np.abs(A) @ np.abs(B).T)
    print("GEMM 256x256x1024, rows scaled over e^+-8: max |err| / (|A||B|^T):  fp64 %.2e" % float(np.max(np.abs(A @ B.T - ref) / den)), end="")
    for S in (7, 8, 9):
        print("  S=%d %.2e" % (S, float(np.max(np.abs(ozaki_nt(A, B, S) - ref) / den))), end="")
    print()


if __name__ == "__main__":
    main()
