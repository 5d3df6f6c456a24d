"""The schedule of `ba_solve_cam_dsm` (ic_gvins_b200/csrc/ba_split.cuh), restated in numpy and checked against a dense solve.

Not a test of the CUDA code (tests/test_ba_gpu.py compares the kernel with the oracle through the C ABI): this pins the ALGORITHM the kernel
implements -- the tile layout (tile row T on CTA T mod 4, strictly-lower tiles, replicated diagonal tiles), the right-looking panel loop with the
panel column all-gathered into every CTA, the right-hand side carried as an augmented row, and the distributed backward substitution whose
partial sums travel point to point -- and the invariant its back-substitution mbarrier relies on:
  * every tile row of the backward substitution receives exactly three partial-sum messages, counting the local arrivals that stand in for
    senders that do not exist (the mbarrier's arrival count is 3).
A schedule that violates it would not give wrong numbers on the GPU, it would hang a cluster (the kernel bounds its waits and raises the
handle's error word instead).  Reference for what is solved: Ceres' DENSE_SCHUR reduced camera system of IG/ic_gvins.cc:1130-1239 at 20
keyframes (n = 15 K + 7 = 307).
"""
import numpy as np
import pytest

CL = 4


def tile_off(cr, m):  # tiles ahead of local tile row m (T = cr + 4 m) in a CTA's tile store: dsm_tile_off
    return m * cr + 2 * m * (m - 1)


def solve_dsm(S, rhs):
    N = S.shape[0]
    NR = N + 1
    nt, npan, Tn, rn = (NR + 7) // 8, (N + 7) // 8, N >> 3, N & 7
    aug = np.zeros((nt * 8, nt * 8))
    aug[:N, :N] = np.tril(S)
    aug[N, :N] = rhs
    tiles = [dict() for _ in range(CL)]
    for cr in range(CL):
        for m, T in enumerate(range(cr, nt, CL)):
            for tc in range(T):
                tiles[cr][tile_off(cr, m) + tc] = aug[8 * T:8 * T + 8, 8 * tc:8 * tc + 8].copy()
        assert sorted(tiles[cr]) == list(range(len(tiles[cr])))  # the offsets tile the store densely
    dg = [[np.tril(aug[8 * T:8 * T + 8, 8 * T:8 * T + 8]).copy() for T in range(nt)] for _ in range(CL)]
    P = [np.zeros((2, nt, 8, 8)) for _ in range(CL)]
    y, dinv = np.zeros(nt * 8), np.zeros(nt * 8)
    Lf = None
    for J in range(npan):
        nb = min(8, N - 8 * J)
        for cr in range(CL):  # trailing update of panel J - 1, then the (redundant) factorisation of the diagonal tile
            PJ = P[cr][(J - 1) & 1]
            if J > 0:
                Jp = J - 1
                dg[cr][J] -= PJ[J] @ PJ[J].T
                m_lo, m_hi = (Jp + 2 - cr + CL - 1) // CL, ((nt - 1 - cr) // CL if cr < nt else -1)
                for m in range(m_lo, m_hi + 1):
                    T = cr + CL * m
                    for tc in range(Jp + 1, T):
                        tiles[cr][tile_off(cr, m) + tc] -= PJ[T] @ PJ[tc].T
                for T in range(Jp + 2, nt):
                    dg[cr][T] -= PJ[T] @ PJ[T].T
            Ld = np.eye(8)
            Ld[:nb, :nb] = np.tril(dg[cr][J][:nb, :nb])
            Lc = np.linalg.cholesky(Ld + np.tril(Ld, -1).T)
            dg[cr][J][:nb, :nb] = np.tril(Lc[:nb, :nb])  # the right-hand-side row below the block stays
            Lf = Lc
            if cr == 0:
                dinv[8 * J:8 * J + nb] = 1.0 / np.diag(Lc)[:nb]
        for cr in range(CL):  # row solves; every solved row goes to all four CTAs
            m0 = (J + 1 - cr + CL - 1) // CL
            nloc = (nt - 1 - (cr + CL * m0)) // CL + 1 if cr + CL * m0 < nt else 0
            for m in range(m0, m0 + nloc):
                T = cr + CL * m
                x = np.linalg.solve(Lf, tiles[cr][tile_off(cr, m) + J].T).T
                tiles[cr][tile_off(cr, m) + J] = x
                for q in range(CL):
                    P[q][J & 1][T] = x
        if Tn > J:
            y[8 * J:8 * J + 8] = P[0][J & 1][Tn][rn]
    if rn > 0:  # the right-hand-side row shares the last diagonal tile with the last rn columns
        x = np.zeros(8)
        for c in range(rn):
            x[c] = (dg[0][Tn][rn, c] - x[:c] @ dg[0][Tn][c, :c]) * dinv[8 * Tn + c]
            y[8 * Tn + c] = x[c]
    contrib = [np.zeros(nt * 8) for _ in range(CL)]
    inbox = [np.zeros((CL, 8)) for _ in range(CL)]
    got = np.zeros(npan, int)
    xs = np.zeros(nt * 8)
    for T in range(npan - 1, -1, -1):
        cr, nbT, m = T % CL, min(8, N - 8 * T), T // CL
        got[T] += max(0, 3 - (npan - 1 - T))  # local arrivals for the senders that do not exist
        assert got[T] == 3
        v = np.zeros(8)
        v[:nbT] = y[8 * T:8 * T + nbT] - contrib[cr][8 * T:8 * T + nbT]
        for q in range(CL):
            if q != cr:
                v[:nbT] -= inbox[cr][q][:nbT]
        for r in range(7, -1, -1):
            xr = v[r] * dinv[8 * T + r]
            v[r] = xr
            v[:r] -= dg[cr][T][r, :r] * xr
        xs[8 * T:8 * T + 8] = v
        for col in range(8 * T):
            contrib[cr][col] += tiles[cr][tile_off(cr, m) + (col >> 3)][:, col & 7] @ v
        for k in (1, 2, 3):  # final on this CTA: its next own tile row is T - 4
            if T - k >= 0:
                assert (T - k) % CL != cr
                inbox[(T - k) % CL][cr] = contrib[cr][8 * (T - k):8 * (T - k) + 8].copy()
                got[T - k] += 1
    return xs[:N]


@pytest.mark.parametrize("N", [307, 157, 337, 37, 22, 64, 56, 16, 9, 8, 7])
def test_schedule_solves_the_system(N):
    rng = np.random.default_rng(N)
    A = rng.standard_normal((N, N + 20))
    S = A @ A.T + N * np.eye(N)
    rhs = rng.standard_normal(N)
    x = solve_dsm(S, rhs)
    ref = np.linalg.solve(S, rhs)
    assert np.abs(x - ref).max() <= 1e-12 * np.abs(ref).max()
