"""The windows that take the marginalization to the edges of its four eigensolver kernels, built and checked on the CPU oracle.

icg_ba_marginalize eigendecomposes two blocks per window: Hmm (n = m rows: pose_0, mix_0 and the landmarks anchored in node 0) and the
Schur complement Hp (n = r rows: the remained pose / mix blocks, ext, td).  One kernel per stage serves the whole batch, chosen by the
batch's largest block (ba_keyframe.cu, marginalize_body):
    n <= 118: marg_jacobi_cta (one CTA);  n <= 160: marg_jacobi_pair (2-CTA cluster);  n <= 320: marg_jacobi_cluster (8-CTA cluster);
    n <= 512: marg_jacobi (global memory);  above 512 the call is refused.
Every kernel pads n to even (round-robin ordering), so the sweep takes both parities on both sides of each limit.

This file restates that rule (select_kernel), builds the sweep's windows (sized_window) and the windows whose Schur complement has a
designed spectrum around the pseudo-inverse cut EPS = 1e-8 (designed_window), and checks on the oracle that each window has the (m, r)
it is meant to have and that the designed eigenvalues fall on the intended side of EPS.  tests/test_marg_sizes_gpu.py runs the same
windows through the device kernels."""
import copy

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa

EPS = 1e-8
LIMITS = {"cta": 118, "pair": 160, "cluster": 320, "global": 512}
ENVS = ((), ("ICG_MARG_PAIR_JACOBI",), ("ICG_MARG_CLUSTER_JACOBI",), ("ICG_MARG_GLOBAL_JACOBI",))

# (m, r) of the sweep.  m: node 0's 15 state rows + the landmarks anchored in it (K = 10); r: the remained blocks, set by a synthetic
# previous prior.  With ext and td present r = 7 + 6 a + 9 b = 1 (mod 3): 118 and 160 are reachable, 320 is not (319 / 322 are).
M_SWEEP = [(m, 64) for m in (15, 16, 117, 118, 119, 120, 159, 160, 161, 162, 319, 320, 321, 322, 511, 512)]
R_SWEEP = [(75, r) for r in (115, 118, 121, 124, 157, 160, 163, 166, 316, 319, 322, 325, 472)]
SWEEP = M_SWEEP + R_SWEEP
REJECTED = (513, 64)
# the designed-spectrum windows: one r per kernel class (m = 40 + 15 on the one-CTA kernel)
DESIGNED_R = (100, 151, 292, 436)


def select_kernel(n, env=()):
    """the kernel marginalize_body launches for a stage whose batch maximum is n, under the ICG_MARG_* variables in env (H100: the 8-CTA
    cluster can always be placed)"""
    glob = "ICG_MARG_GLOBAL_JACOBI" in env
    if n <= LIMITS["cluster"] and not glob and ("ICG_MARG_CLUSTER_JACOBI" in env or n > LIMITS["pair"]):
        return "cluster"
    if n <= LIMITS["cta"] and not glob and "ICG_MARG_PAIR_JACOBI" not in env:
        return "cta"
    if n <= LIMITS["pair"] and not glob:
        return "pair"
    return "global"


def kernel_runs(m, r):
    """{(kernel of the Hmm stage, kernel of the Hp stage): env} over the variable settings that give distinct pairs; the default first"""
    out = {}
    for env in ENVS:
        out.setdefault((select_kernel(m, env), select_kernel(r, env)), env)
    return out


# ------------------------------------------------------------------------------------------------ window construction
_GEN = {}


def generated(olib, K, L, seed, **kw):
    """a fresh copy of make_window(n_ref=1): every landmark is anchored in node 0 (generated once per module)"""
    key = (K, L, seed, tuple(sorted(kw.items())))
    if key not in _GEN:
        _GEN[key] = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=K, L=L, seed=seed, n_ref=1, **kw)
    return copy.deepcopy(_GEN[key])


def keep_landmarks(prob, n_lm, max_obs=None):
    """clear f_active on every factor of the landmarks after the first n_lm observed ones (and, with max_obs, on every factor observed in a
    node > max_obs): node 0 then carries exactly n_lm landmarks into the marginalization, m = 15 + n_lm"""
    observed = np.unique(prob["f_lm"])
    assert observed.size >= n_lm, (observed.size, n_lm)
    keep = np.isin(prob["f_lm"], observed[:n_lm])
    if max_obs is not None:
        keep &= prob["f_obs"] <= max_obs
    prob["f_active"] = keep.astype(np.uint8)
    return prob


def remained_by_factors(prob):
    """the pose / mix nodes (>= 1) the marginalized factors reach: observers of node 0's active factors, and node 1 through IMU factor 0"""
    act = (prob["f_active"] != 0) & (prob["f_ref"] == 0)
    return set(prob["f_obs"][act].tolist()) | {1}, {1}


def split_rows(need, free_pose, free_mix):
    """6 a + 9 b = need with a <= free_pose, b <= free_mix (fewest mix blocks)"""
    for b in range(0, free_mix + 1):
        if need - 9 * b >= 0 and (need - 9 * b) % 6 == 0 and (need - 9 * b) // 6 <= free_pose:
            return (need - 9 * b) // 6, b
    raise ValueError(f"{need} rows cannot be made of the free blocks")


def set_prior(prob, truth, blocks, rng, designed=None):
    """a previous prior over `blocks` ([(type, node)], type 0 pose, 1 mix, 2 ext, 3 td).  The blocks listed in `designed` (a set of
    (type, node)) get the square root J_b handed in designed[...]; the others J0 = (3 I + small upper-triangular coupling) diag(scale), well
    conditioned, around the true values (window_prior of tests/test_marg_large_gpu.py).  The designed blocks' x0 are the window's current
    values, so that their part of the prior enters as H = J_b^T J_b, b = -J_b^T e_b exactly."""
    size = {0: 6, 1: 9, 2: 6, 3: 1}
    scl = {0: [10.0] * 6, 1: [5.0] * 3 + [2000.0] * 3 + [500.0] * 3, 2: [50.0] * 6, 3: [100.0]}
    dset = designed["blocks"] if designed else set()
    cols_wc, cols_d, scale, x0 = [], [], [], []
    col = 0
    pose, mix = prob["pose"].reshape(-1, 7), prob["mix"].reshape(-1, 9)
    for t, nd in blocks:
        idx = list(range(col, col + size[t]))
        (cols_d if (t, nd) in dset else cols_wc).extend(idx)
        scale += scl[t]
        col += size[t]
        src = pose if (t, nd) in dset else truth["pose"]
        if t == 0:
            x0.append(src[nd])
        elif t == 1:
            x0.append((mix if (t, nd) in dset else truth["mix"])[nd])
        elif t == 2:
            x0.append(truth["ext"][:7])
        else:
            x0.append([0.0])
    r = col
    J0, e0 = np.zeros((r, r)), np.zeros(r)
    nw = len(cols_wc)
    A = 3.0 * np.eye(nw) + np.triu(rng.normal(0, 0.5 / np.sqrt(nw), (nw, nw)), 1)
    J0[np.ix_(cols_wc, cols_wc)] = A * np.asarray(scale)[cols_wc][None, :]
    e0[cols_wc] = rng.normal(0, 0.1, nw)
    if designed:
        J0[np.ix_(cols_d, cols_d)] = designed["J"]
        e0[cols_d] = designed["e"]
    prob.update(marg_r=r, marg_nblocks=len(blocks), marg_block_type=np.array([t for t, _ in blocks], np.int32),
                marg_block_node=np.array([nd for _, nd in blocks], np.int32), marg_x0=np.concatenate(x0), marg_J0=J0.reshape(-1).copy(),
                marg_e0=e0)
    return prob


def node_order(blocks):
    """blocks in the order of the remained columns (node-major pose, mix; then ext, td), node 0 first"""
    return sorted(blocks, key=lambda b: (b[0] >= 2, b[1] if b[0] < 2 else 0, b[0]))


def sized_window(olib, m, r, seed=0):
    """a window whose marginalization of node 0 has exactly m marginalized and r remained rows.  m <= 120 on a K = 32 window (so that
    the prior can reach r = 15 * 31 + 7 = 472), larger m on K = 10 with up to 540 landmarks; r through a prior over node 0, the blocks
    the factors reach, ext, td and as many further pose / mix blocks as r asks for"""
    K, L = (32, 140) if m <= 120 else (10, 540)
    prob, truth = generated(olib, K, L, 7100 + seed)
    keep_landmarks(prob, m - 15)
    poses, mixes = remained_by_factors(prob)
    free_pose = [k for k in range(1, K) if k not in poses]
    free_mix = [k for k in range(1, K) if k not in mixes]
    a, b = split_rows(r - 7 - 6 * len(poses) - 9 * len(mixes), len(free_pose), len(free_mix))
    blocks = [(0, 0), (1, 0)] + [(0, k) for k in sorted(poses) + free_pose[:a]] + [(1, k) for k in sorted(mixes) + free_mix[:b]] + [(2, 0), (3, 0)]
    return set_prior(prob, truth, node_order(blocks), np.random.default_rng(7200 + 1000 * seed + m + r))


def designed_spectrum(n, rng):
    """eigenvalues of the low and the high sub-block of the designed block (n >= 44).  Low sub-block (scale 10, so the rounding of every
    FP64 step on it is ~1e-15, far below 1e-3 EPS): 3 exact zeros, 1e-12, two at 0.5 EPS, 0.8 EPS, 1.25 EPS, two at 2 EPS, a 10-fold
    eigenvalue 1.0, fill log-uniform in [1e-3, 10].  0.8 EPS and 1.25 EPS tell a cut moved by a factor 1.5 either way.  High sub-block:
    1e6 and fill log-uniform in [1e2, 1e6]."""
    n_lo = n // 2
    lo = np.concatenate([[0.0] * 3, [1e-12], [0.5 * EPS] * 2, [0.8 * EPS, 1.25 * EPS], [2 * EPS] * 2, [1.0] * 10])
    lo = np.concatenate([lo, 10.0 ** rng.uniform(-3, 1, n_lo - lo.size)])
    hi = np.concatenate([[1e6], 10.0 ** rng.uniform(2, 6, n - n_lo - 1)])
    return lo, hi


def random_orthogonal(n, rng):
    q, rr = np.linalg.qr(rng.normal(size=(n, n)))
    return q * np.sign(np.diag(rr))[None, :]


def designed_window(olib, r, seed=0):
    """K = 32, 40 landmarks on node 0 (m = 55), their factors limited to observers 1..3.  The previous prior is block diagonal: a well
    conditioned part over node 0..3's pose / mix, ext and td (everything the node-0 factors reach), and a designed part over pose / mix
    blocks of nodes >= 4, which no marginalized factor touches: no Schur term reaches those columns, so Hp restricted to them is
    J_b^T J_b = Q diag(lambda) Q^T exactly, Q = blockdiag(Q_lo, Q_hi) random orthogonal (Q_lo over the first half of the designed
    columns, Q_hi over the rest).  Returns (prob, info): info["cols"] are the designed columns of Hp, info["lam"] / info["Q"] the designed
    eigenpairs (columns of Q), info["bp"] = -J_b^T e_b."""
    K = 32
    prob, truth = generated(olib, K, 140, 7300 + seed)
    keep_landmarks(prob, 40, max_obs=3)
    wc = [(t, k) for k in range(4) for t in (0, 1)]
    n_b = r - 15 * 3 - 7
    a, b = split_rows(n_b, K - 4, K - 4)
    dblocks = [(0, k) for k in range(4, 4 + a)] + [(1, k) for k in range(4, 4 + b)]
    blocks = node_order(wc + dblocks + [(2, 0), (3, 0)])
    rng = np.random.default_rng(7400 + seed + r)
    lo, hi = designed_spectrum(n_b, rng)
    n_lo = lo.size
    Q = np.zeros((n_b, n_b))
    Q[:n_lo, :n_lo] = random_orthogonal(n_lo, rng)
    Q[n_lo:, n_lo:] = random_orthogonal(n_b - n_lo, rng)
    lam = np.concatenate([lo, hi])
    J = (Q * np.sqrt(lam)[None, :]) @ Q.T
    e = rng.normal(0, 1.0, n_b)
    set_prior(prob, truth, blocks, rng, designed=dict(blocks=set(dblocks), J=J, e=e))
    # the designed columns of Hp: remained order = blocks without node 0, sizes 6 / 9 / 6 / 1
    size = {0: 6, 1: 9, 2: 6, 3: 1}
    cols, col = [], 0
    for t, nd in blocks:
        if nd == 0 and t < 2:
            continue
        if (t, nd) in set(dblocks):
            cols.extend(range(col, col + size[t]))
        col += size[t]
    assert col == r and len(cols) == n_b
    return prob, dict(cols=np.array(cols), lam=lam, Q=Q, bp=-J.T @ e, scale=lam.max())


def check_designed(g, info, tol=1e-9, ascending=True):
    """the prior g (J0, e0, bp of a marginalization of a designed_window) against the designed spectrum: the designed block's J0 rows are
    exactly its eigenvalues above EPS, rows and e0 entries dropped at EPS are exactly zero, J0^T J0 and J0^T e0 on the block equal the
    kept part of the designed spectrum to tol of the block scale, rows in ascending order (the device's order; the oracle's two-sided
    Jacobi leaves them unsorted: ascending=False)"""
    J0, e0, D = g["J0"], g["e0"], info["cols"]
    r = J0.shape[0]
    other = np.setdiff1d(np.arange(r), D)
    lam, Q = info["lam"], info["Q"]
    kept = lam > EPS
    on_d = np.any(J0[:, D] != 0, axis=1)
    on_o = np.any(J0[:, other] != 0, axis=1)
    assert not np.any(on_d & on_o), "a row mixes the designed block with the rest"
    assert on_d.sum() == kept.sum(), (int(on_d.sum()), int(kept.sum()))
    zero = ~on_d & ~on_o
    assert np.all(e0[zero] == 0), "an e0 entry of a dropped row is not exactly 0"
    rn = (J0 ** 2).sum(axis=1)
    if ascending:
        assert np.all(np.diff(rn) >= -tol * np.maximum(rn[1:], rn[:-1])), "rows not in ascending order"
    # the designed rows carry the kept eigenvalues themselves
    got = np.sort(rn[on_d])
    want = np.sort(lam[kept])
    assert np.all(np.abs(got - want) <= 1e-6 * want + 1e-14), np.abs(got - want).max()
    Hk = (Q[:, kept] * lam[kept]) @ Q[:, kept].T
    Pk = Q[:, kept] @ Q[:, kept].T
    JJ = J0[:, D].T @ J0[:, D]
    Je = J0[:, D].T @ e0
    bscale = np.abs(info["bp"]).max()
    dJ = np.abs(JJ - Hk).max() / info["scale"]
    de = np.abs(Je + Pk @ info["bp"]).max() / bscale
    db = np.abs(g["bp"][D] - info["bp"]).max() / bscale
    assert dJ < tol and de < tol and db < tol, (dJ, de, db)
    return dJ, de


# ------------------------------------------------------------------------------------------------ tests (CPU)
@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


def test_selection_rule_classes():
    """the kernels each n can be forced onto: every kernel takes every n up to its limit, nothing above"""
    order = ["cta", "pair", "cluster", "global"]
    for n in range(1, 513):
        runs = {select_kernel(n, env) for env in ENVS}
        assert runs == {k for k in order if n <= LIMITS[k]}, n
        assert select_kernel(n) == next(k for k in order if n <= LIMITS[k])


def test_sweep_reaches_both_parities_on_both_sides_of_every_limit():
    ns = {n for mr in SWEEP for n in mr}
    for k, lim in LIMITS.items():
        below = [n for n in ns if lim - 4 <= n <= lim]
        assert {n % 2 for n in below} == {0, 1} and lim in ns, (k, sorted(below))
        if k != "global":
            above = [n for n in ns if lim < n <= lim + 6]
            assert {n % 2 for n in above} == {0, 1}, (k, sorted(above))
    assert REJECTED[0] == LIMITS["global"] + 1
    assert any(n > LIMITS["cluster"] for _, n in R_SWEEP)
    # both directions of a batch whose two stages take different kernel classes
    assert any(select_kernel(m) == "cta" and select_kernel(r) == "global" for m, r in SWEEP)
    assert any(select_kernel(m) == "global" and select_kernel(r) == "cta" for m, r in SWEEP)
    assert [select_kernel(r) for r in DESIGNED_R] == ["cta", "pair", "cluster", "global"]


@pytest.mark.parametrize("m,r", SWEEP + [REJECTED])
def test_sweep_window_has_its_size(olib, m, r):
    p = sized_window(olib, m, r)
    o = oa.ba_marginalize(olib, copy.deepcopy(p), 1)
    assert (o["m"], o["r"]) == (m, r)
    assert np.all(np.isfinite(o["J0"])) and np.all(np.isfinite(o["e0"]))


@pytest.mark.parametrize("r", DESIGNED_R)
def test_oracle_splits_the_designed_spectrum_at_eps(olib, r):
    p, info = designed_window(olib, r)
    o = oa.ba_marginalize(olib, copy.deepcopy(p), 1)
    assert (o["m"], o["r"]) == (55, r)
    # Hp restricted to the designed columns is the designed matrix, decoupled from the rest
    D = info["cols"]
    other = np.setdiff1d(np.arange(r), D)
    H = (info["Q"] * info["lam"]) @ info["Q"].T
    assert np.abs(o["Hp"][np.ix_(D, D)] - H).max() < 1e-9 * info["scale"]
    assert np.all(o["Hp"][np.ix_(D, other)] == 0)
    check_designed(o, info, ascending=False)
