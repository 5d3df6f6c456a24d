"""CPU: the IMU preintegration entry by entry against a high-precision restatement (tests/preint_mp.py), at the edges of the sweep there:
1 to 2001 rows, 100 / 200 / 400 Hz, short first and last samples, a repeated timestamp, jittered dt, zero rotation, a 180 deg/s turn, large
start biases, the Earth form at latitudes 0 / 30.5 / 80 deg and the Normal form, and a 100 s bias correlation time.

Both the product's host core (icg_imu_preintegrate, the scalar core the device kernels share bit for bit) and the oracle's
icgo_preintegrate are held to the same per-entry rule, so that an error in either -- including one that would move host and device
together -- shows in the small blocks of the covariance, not only in its largest entry:
  covariance   |dC_ij| <= TOL_COV sqrt(C_ii C_jj) where C_ii, C_jj > 0; elsewhere relative to the 3 x 3 block's max; zero blocks exactly 0
  J            per 3 x 3 block, |dJ| <= TOL_J * max |block|; blocks that are 0 exactly 0
  head, end    per group (dp, dv, dq, s1, ...), |d| <= TOL_HEAD * max |group|; the copied start biases, gravity and iewn bit for bit
  exact zeros  the blocks that are 0 in exact arithmetic (p, v, att, bg, ba = 0..4): J's strict lower block triangle, J(att, ba),
               J(bg, ba), the off-diagonals of J(bg, bg) / J(ba, ba); covariance (att, ba), (bg, ba), their transposes and the
               off-diagonals of (bg, bg) / (ba, ba) -- all exactly 0.0, in both forms"""
import numpy as np
import pytest

from tests import oracle_api as oa
from tests import preint_mp as pm

# about 10x the worst ratios measured over mp_sweep() (98 intervals; the host core and the oracle gave the same worst cases): covariance
# 8.7e-15 (201 rows, the turn at latitude 0), J 4.8e-15, head 3.3e-15, end state 1.3e-15
TOL_COV, TOL_J, TOL_HEAD = 1e-13, 5e-14, 5e-14

J_ZERO = [(i, j) for i in range(5) for j in range(5) if i > j] + [(2, 4), (3, 4)]
C_ZERO = [(2, 4), (4, 2), (3, 4), (4, 3)]
HEAD_GROUPS = [(0, 1), (1, 4), (4, 7), (7, 11), (23, 24), (24, 27)]  # delta_time, dp, dv, dq, s0, s1; [11, 23) is copied
END_GROUPS = [(0, 3), (3, 7), (7, 10)]


def _group_ratio(got, ref, groups, floors=None):
    worst = 0.0
    for g, (a, b) in enumerate(groups):
        mx = max(np.abs(ref[a:b]).max(), floors[g] if floors else 0.0)
        if mx > 0:
            worst = max(worst, float(np.abs(got[a:b] - ref[a:b]).max() / mx))
    return worst


def ratios(blob, end, ref):
    """the worst ratio of each per-entry rule (the exact parts are exact_parts').  The end position and velocity are scaled by at least the
    size of the terms they sum, |v| T + |g| T^2 and |g| T: standing still, velocity increments of size |g| dt cancel to ~0."""
    head, J, Cv, e = ref
    T, g = head[0], float(np.linalg.norm(head[17:20]))
    floors = (float(np.linalg.norm(e[7:10])) * T + g * T * T, 1.0, g * T)
    gJ, gC = blob[27:252].reshape(15, 15), blob[252:477].reshape(15, 15)
    d = np.sqrt(np.maximum(np.diag(Cv), 0.0))
    m = np.outer(d > 0, d > 0)
    cov = float((np.abs(gC - Cv)[m] / np.outer(d, d)[m]).max()) if m.any() else 0.0
    # beside a zero diagonal entry (the p rows after one sample: C(p, v) = 0.5 dt^2 G(v, v)), relative to the largest entry of the 3 x 3 block
    bmax = np.kron(np.abs(Cv).reshape(5, 3, 5, 3).max(axis=(1, 3)), np.ones((3, 3)))
    o = ~m & (bmax > 0)
    cov = max(cov, float((np.abs(gC - Cv)[o] / bmax[o]).max()) if o.any() else 0.0)
    jac = 0.0
    for i in range(5):
        for j in range(5):
            r, q = blk(J, i, j), blk(gJ, i, j)
            if np.abs(r).max() > 0:
                jac = max(jac, float(np.abs(q - r).max() / np.abs(r).max()))
    return dict(cov=cov, jac=jac, head=_group_ratio(blob[:27], head, HEAD_GROUPS), end=_group_ratio(end, e, END_GROUPS, floors))


def blk(M, i, j):
    return M[3 * i:3 * i + 3, 3 * j:3 * j + 3]


def offdiag(M):
    return M[~np.eye(3, dtype=bool)]


def exact_parts(blob, end, ref, case):
    """every entry the rules above hold exactly"""
    head, J, Cv, e = ref
    gJ, gC = blob[27:252].reshape(15, 15), blob[252:477].reshape(15, 15)
    for M, name in ((J, "restatement J"), (gJ, "J")):
        for i, j in J_ZERO:
            assert not blk(M, i, j).any(), (case, name, i, j)
        for i in (3, 4):
            assert not offdiag(blk(M, i, i)).any(), (case, name, i)
    for M, name in ((Cv, "restatement covariance"), (gC, "covariance")):
        for i, j in C_ZERO:
            assert not blk(M, i, j).any(), (case, name, i, j)
        for i in (3, 4):
            assert not offdiag(blk(M, i, i)).any(), (case, name, i)
    for i in range(5):
        for j in range(5):
            if not blk(Cv, i, j).any():
                assert not blk(gC, i, j).any(), (case, "covariance block", i, j)
    for i in range(5):
        for j in range(5):
            if not blk(J, i, j).any():
                assert not blk(gJ, i, j).any(), (case, "J block", i, j)
    assert np.array_equal(blob[11:23], head[11:23]), case  # start biases, gravity, iewn: copied
    for got, ref_, groups in ((blob[:27], head, HEAD_GROUPS), (end, e, END_GROUPS)):
        for a, b in groups:
            if not ref_[a:b].any():
                assert not got[a:b].any(), (case, a, b)
    assert blob[477] == (1.0 if case.iewn is None else 0.0) and blob[478] == 0 and blob[479] == 0, case


def check(blob, end, case):
    ref = pm.preintegrate(*case.args)
    exact_parts(blob, end, ref, case)
    r = ratios(blob, end, ref)
    assert r["cov"] <= TOL_COV and r["jac"] <= TOL_J and r["head"] <= TOL_HEAD and r["end"] <= TOL_HEAD, (case, r)


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def host():
    """the product's host core; it needs the built library, which loads without a GPU"""
    try:
        from ic_gvins_b200._lib import IcgError, lib
        lib()
    except (IcgError, OSError) as e:
        pytest.skip(f"libicgvins_b200.so cannot be loaded here ({e}); the host core is compared on machines where it can")
    from ic_gvins_b200.ba import imu_preintegrate
    return imu_preintegrate


MP = pm.mp_sweep()
ALL = pm.sweep()


@pytest.mark.parametrize("case", MP, ids=[c.name for c in MP])
def test_host_core_against_the_restatement(host, case):
    blob, end = host(*case.args)
    check(blob, end, case)


@pytest.mark.parametrize("case", MP, ids=[c.name for c in MP])
def test_oracle_against_the_restatement(olib, case):
    blob, _, end = oa.preintegrate(olib, *case.args)
    check(blob, end, case)


def test_host_core_against_the_oracle_on_the_whole_sweep(host, olib):
    """the intervals too long for the restatement (up to 2001 rows, 20 s at 100 Hz): the host core against the oracle by the same rules"""
    for case in ALL:
        blob, end = host(*case.args)
        bo, _, eo = oa.preintegrate(olib, *case.args)
        ref = (bo[:27], bo[27:252].reshape(15, 15), bo[252:477].reshape(15, 15), eo)
        exact_parts(blob, end, ref, case)
        r = ratios(blob, end, ref)
        assert r["cov"] <= TOL_COV and r["jac"] <= TOL_J and r["head"] <= TOL_HEAD and r["end"] <= TOL_HEAD, (case, r)


def test_the_sweep_reaches_every_edge():
    tags = [c.tags for c in ALL]
    for key, values in (("n", pm.ROWS), ("rate", pm.RATES), ("timing", pm.TIMINGS), ("motion", pm.MOTIONS), ("form", pm.FORMS)):
        assert {t[key] for t in tags} == set(values), key
    for n in pm.ROWS:
        assert {t["timing"] for t in tags if t["n"] == n} == set(pm.TIMINGS), n
        assert {t["form"] for t in tags if t["n"] == n} == set(pm.FORMS), n
        assert {t["corr100"] for t in tags if t["n"] == n} == {False, True}, n
    for c in ALL:
        assert len(c.imu) == c.tags["n"], c
        dt = c.imu[1:, 0]
        if c.tags["timing"] == "repeat" and c.tags["n"] >= 3:
            assert (dt == 0).sum() == 1, c
        else:
            assert (dt > 0).all(), c
        if c.tags["timing"] == "frac_ends" and c.tags["n"] >= 3:
            assert np.isclose(dt[0], 0.3 / c.tags["rate"]) and np.isclose(dt[-1], 0.7 / c.tags["rate"]), c
        if c.tags["motion"] == "stationary":  # rotvec2q's zero-angle branch on every sample
            assert c.iewn is None and not c.state16[10:16].any() and not c.imu[:, 1:4].any(), c
    turn = [c for c in ALL if c.tags["motion"] == "turn" and c.tags["n"] == 2001]
    assert all(np.abs(c.imu[1:, 3] / c.imu[1:, 0]).max() > 3.0 for c in turn)  # rad/s
    assert {m for t in tags for m in [t["motion"]] if t["n"] in (1, 2, 3)} == set(pm.MOTIONS)
    assert 20 <= len(MP) <= 100 and sum(c.tags["n"] for c in MP) < 3500


def test_noise_scale_draws_the_same_random_numbers():
    """imu_samples(noise_scale=0) consumes the generator as the default does, so the windows the other tests build stay bit for bit"""
    from datagen import synth_ba
    a, b = np.random.default_rng(3), np.random.default_rng(3)
    x = synth_ba.imu_samples(0.0, 0.1, 200.0, a, np.zeros(3), np.zeros(3))
    y = synth_ba.imu_samples(0.0, 0.1, 200.0, b, np.zeros(3), np.zeros(3), noise_scale=0.0)
    assert a.bit_generator.state == b.bit_generator.state and not np.array_equal(x, y)
    z = synth_ba.imu_samples(0.0, 0.1, 200.0, np.random.default_rng(3), np.zeros(3), np.zeros(3), noise_scale=1.0)
    assert np.array_equal(x, z)
