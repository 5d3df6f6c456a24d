"""GPU: the warp-per-interval preintegration (preint.cu) at the edges of tests/preint_mp.py's sweep, on its three front ends.

Every device blob, end state and node row must equal the host core's (icg_imu_preintegrate: the same sums in the same order, built with
-fmad=false) bit for bit; the host core is held to the high-precision restatement in test_preint_edges.py, and the device blobs are
held to it here too, by the same per-entry rule.
  batch     preint_batch_kernel: each interval alone, in launches of 1, 2, 3 and 33 intervals, and in one launch of ~4000 intervals of
            1 to 2001 rows, where each must equal its solo call (the two warps of a CTA do not see each other)
  resident  preint_resident_kernel: the gate exactly at 6 sigma (closed) and one ulp above (open) in its own sum order; 1-, 2- and 3-row
            intervals, -1 exactly where icg_ba_upload refuses the blob, the factor kept and the others reintegrated; 1001 rows
  slide     preint_slide_kernel: every factor of a window as one ICG_SLIDE_CHAIN with Normal and Earth items mixed, items of 2 and 2001
            rows, 11 aligned GNSS fixes (3 * 11 > 32 lanes: the alignment loop wraps), a one-item window in the same launch"""
import copy
import math

import numpy as np
import pytest

from datagen import synth_ba
from datagen.slide_window import build_next
from tests import preint_mp as pm
from tests.test_post_solve_gpu import make
from tests.test_preint_edges import check as check_mp
from tests.test_reintegration_gpu import earth_iewn, solver_for, state16, window
from tests.test_slide_gpu import PARAMS, handle
from tests.test_slide_integrate_gpu import CHAIN, host_twin, integ_for, intervals

pytestmark = pytest.mark.gpu
IMU = 480
NOISE5 = synth_ba.NOISE5
ALL = pm.sweep()


@pytest.fixture(scope="module")
def olib(oracle):
    from tests import oracle_api as oa
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def geom():
    from ic_gvins_b200.geom import Geometry
    g = Geometry()
    yield g
    g.close()


def host(*args):
    from ic_gvins_b200.ba import imu_preintegrate
    return imu_preintegrate(*args)


def groups(cases):
    """the cases by (form, noise): a batch launch takes one iewn and one noise5"""
    out = {}
    for c in cases:
        out.setdefault((c.tags["form"], c.tags["corr100"]), []).append(c)
    return out


def batch(geom, cases, iewn=False):
    """one launch; iewn=False: the cases' own (one form per launch)"""
    iw = cases[0].iewn if iewn is False else iewn
    return geom.imu_preintegrate_batch(np.array([c.state16 for c in cases]), iw, synth_ba.GRAVITY, cases[0].noise5, [c.imu for c in cases])


# ---------------------------------------------------------------------------------------------- batch
def test_batch_solo_and_in_launches_of_1_2_3_33_bitwise(geom):
    for key, cs in groups(ALL).items():
        solo = []
        for c in cs:
            b, e = batch(geom, [c])
            hb, he = host(*c.args)
            assert np.array_equal(b[0], hb) and np.array_equal(e[0], he), c
            solo.append((b[0], e[0]))
        for size in (2, 3, 33):
            for i in range(0, len(cs), size):
                b, e = batch(geom, cs[i:i + size])
                for j in range(len(b)):
                    assert np.array_equal(b[j], solo[i + j][0]) and np.array_equal(e[j], solo[i + j][1]), (size, cs[i + j])


def test_one_launch_of_4000_mixed_lengths_equals_solo_calls(geom):
    """every sweep interval in the Earth form at 30.5 deg, 30 times over in a shuffled order: 4001 intervals of 1 to 2001 rows side by side,
    the last CTA with one idle warp"""
    iw = pm.iewn_at(30.5)
    solo = []
    for c in ALL:
        b, e = geom.imu_preintegrate_batch(c.state16[None], iw, synth_ba.GRAVITY, NOISE5, [c.imu])
        hb, he = host(c.state16, iw, synth_ba.GRAVITY, NOISE5, c.imu)
        assert np.array_equal(b[0], hb) and np.array_equal(e[0], he), c
        solo.append((b[0], e[0]))
    idx = np.random.default_rng(7).permutation(np.tile(np.arange(len(ALL)), 30))[:4001]
    cs = [ALL[i] for i in idx]
    assert {c.tags["n"] for c in cs} == set(pm.ROWS)
    b, e = geom.imu_preintegrate_batch(np.array([c.state16 for c in cs]), iw, synth_ba.GRAVITY, NOISE5, [c.imu for c in cs])
    for k, i in enumerate(idx):
        assert np.array_equal(b[k], solo[i][0]) and np.array_equal(e[k], solo[i][1]), (k, ALL[i])


def test_batch_against_the_restatement(geom):
    for key, cs in groups(pm.mp_sweep()).items():
        b, e = batch(geom, cs)
        for k, c in enumerate(cs):
            check_mp(b[k], e[k], c)


# ---------------------------------------------------------------------------------------------- resident
SG, SA = 6 * NOISE5[2], 6 * NOISE5[3]


def norm3(x, y, z):
    return math.sqrt(x * x + y * y + z * z)  # the gate's order: (x^2 + y^2) + z^2, then sqrt (no FMA, as preint.cu is built)


def knife(b, thr, above, seed):
    """mix biases m with all three offsets b - m non-zero whose norm, in the gate's order, is exactly thr (above: the next double up), and
    in the other association, x^2 + (y^2 + z^2), is not: a gate that summed in another order would land on the other side"""
    rng = np.random.default_rng(seed)
    want = np.nextafter(thr, np.inf) if above else thr
    for _ in range(10000):
        u = rng.normal(size=3)
        g = u / np.linalg.norm(u) * thr
        for step in range(-40, 41):
            gz = g[2] + step * np.spacing(g[2])
            m = np.array([b[0] - g[0], b[1] - g[1], b[2] - gz])
            d = b - m
            if d.all() and norm3(*d) == want and math.sqrt(d[0] * d[0] + (d[1] * d[1] + d[2] * d[2])) != want:
                return m
    raise AssertionError("no offset lands on the threshold")


def test_resident_gate_exactly_at_6_sigma(olib):
    prob, rows = window(olib, 1301, K=10, L=60)
    mix, blobs = prob["mix"].reshape(10, 9), prob["imu_blob"].reshape(-1, IMU)
    # factor: (gyro on the threshold, above it), (accel on the threshold, above it); the other offset far below its threshold
    plan = {0: (False, None), 1: (True, None), 2: (None, False), 3: (None, True), 4: (False, False), 5: (True, False), 6: (False, True)}
    for k, (gy, ac) in plan.items():
        mix[k, 3:6] = blobs[k, 11:14] if gy is None else knife(blobs[k, 11:14], SG, gy, 10 * k)
        mix[k, 6:9] = blobs[k, 14:17] if ac is None else knife(blobs[k, 14:17], SA, ac, 10 * k + 1)
    for k in (7, 8):
        mix[k, 3:9] = blobs[k, 11:17]
    want = np.array([0, 1, 0, 1, 0, 1, 1, 0, 0], np.int8)
    s = solver_for([prob])
    try:
        s.upload([prob])
        before = prob["imu_blob"].copy()
        out = s.reintegrate([prob], NOISE5, np.zeros(3), [rows])[0]
    finally:
        s.close()
    assert np.array_equal(out["status"], want), out["status"]
    pose = prob["pose"].reshape(10, 7)
    for k in range(9):
        if want[k]:
            st = state16(pose[k], mix[k])
            hb, he = host(st, earth_iewn(np.zeros(3), pose[k, :3]), synth_ba.GRAVITY, NOISE5, rows[k])
            assert np.array_equal(out["blobs"][k], hb) and np.array_equal(out["end_states"][k], he), k
        else:
            assert np.array_equal(prob["imu_blob"].reshape(-1, IMU)[k], before.reshape(-1, IMU)[k]), k


def upload_refuses(prob, k, blob):
    """icg_ba_upload of prob with factor k's blob replaced: False (taken) or True (refused as not positive definite)"""
    from ic_gvins_b200._lib import IcgError
    q = copy.deepcopy(prob)
    q["imu_blob"].reshape(-1, IMU)[k] = blob
    u = solver_for([q])
    try:
        u.upload([q])
        return False
    except IcgError as e:
        assert f"IMU factor {k} has a non positive-definite covariance" in str(e), str(e)
        return True
    finally:
        u.close()


@pytest.mark.parametrize("earth", [True, False], ids=["earth", "normal"])
def test_resident_short_and_long_intervals(olib, earth):
    """factors 1, 2, 3: 1-, 2- and 3-row intervals; factor 5: 1001 rows; every gate open"""
    from ic_gvins_b200._lib import IcgError
    K = 8
    prob, rows = window(olib, 1311 + earth, K=K, L=60, earth=earth, lin=lambda k: (np.full(3, 9 * NOISE5[2]), np.zeros(3)))
    mix, pose = prob["mix"].reshape(K, 9), prob["pose"].reshape(K, 7)
    rng = np.random.default_rng(1320)
    for k, n in ((1, 1), (2, 2), (3, 3), (5, 1001)):
        rows[k] = synth_ba.imu_samples(0.5 * k, 0.5 * k + (n - 1) / 200.0, 200.0, rng, mix[k, 3:6], mix[k, 6:9], earth=earth)
        assert len(rows[k]) == n
    station = np.array([0.52, 1.99, 30.0])
    hosts, refused = [], []
    for k in range(K - 1):
        iw = earth_iewn(station, pose[k, :3]) if earth else None
        hosts.append(host(state16(pose[k], mix[k]), iw, synth_ba.GRAVITY, NOISE5, rows[k]))
        refused.append(upload_refuses(prob, k, hosts[-1][0]))
    assert refused[1] and not any(refused[4:])
    s = solver_for([prob])
    try:
        s.upload([prob])
        before = prob["imu_blob"].copy()
        try:
            out = s.reintegrate([prob], NOISE5, station, [rows])[0]
            assert not any(refused)
        except IcgError as e:
            assert any(refused) and "not positive definite" in str(e)
            out = e.results[0]
    finally:
        s.close()
    assert np.array_equal(out["status"], np.where(refused, -1, 1).astype(np.int8)), out["status"]
    assert out["count"] == K - 1
    for k in range(K - 1):
        if refused[k]:
            assert np.array_equal(prob["imu_blob"].reshape(-1, IMU)[k], before.reshape(-1, IMU)[k]), k
            assert np.array_equal(out["end_states"][k], hosts[k][1]), k
        else:
            assert np.array_equal(out["blobs"][k], hosts[k][0]) and np.array_equal(out["end_states"][k], hosts[k][1]), k
            assert np.array_equal(prob["imu_blob"].reshape(-1, IMU)[k], hosts[k][0]), k


# ---------------------------------------------------------------------------------------------- slide
def chain_window(olib, seed, K, lengths, normal):
    """window of K nodes and its next window: nodes K - 2 and K - 1 kept, K - 2 new nodes, every new factor integrated (the first from node
    K - 1, the rest ICG_SLIDE_CHAIN), item k of lengths[k] rows in the form normal[k]; every new GNSS fix aligned by node K - 1's velocity"""
    p = make(olib, seed=seed, K=K, L=60, n_ref=K)
    up, nxt, carry = build_next(p, seed + 1, drop=tuple(range(K - 2)), n_new=K - 2)
    m = nxt["n_imu"]
    assert m == K - 1 and carry["imu_src"][0] == K - 2 and (carry["imu_src"][1:] < 0).all()
    rng = np.random.default_rng(seed + 2)
    mix = p["mix"].reshape(K, 9)[K - 1]
    rows = {}
    for k, n in enumerate(lengths):
        t0 = 0.5 * (K - 1 + k)
        rows[k + 1] = synth_ba.imu_samples(t0, t0 + (n - 1) / 200.0, 200.0, rng, mix[3:6], mix[6:9], earth=not normal[k])
    g = integ_for(nxt, carry, {k: (K - 1 if k == 1 else CHAIN) for k in range(1, m)}, rows, normal=np.array([False] + list(normal), bool))
    free = np.nonzero(carry["gnss_src"] < 0)[0]
    g["gnss_node"][free] = K - 1
    g["gnss_dt"][free] = np.linspace(-0.045, 0.04, len(free))
    return p, nxt, carry, g


def one_item_window(olib, seed):
    p = make(olib, seed=seed, K=6, L=60)
    up, nxt, carry = build_next(p, seed + 1)
    k = nxt["n_imu"] - 1
    return p, nxt, carry, integ_for(nxt, carry, {k: p["K"] - 1}, {k: intervals(p, p["K"] - 1, 1, seed + 2)[0]})


def solved(probs, K):
    s1, s2 = handle(n=len(probs), K=K, L=120, F=1500), handle(n=len(probs), K=K, L=120, F=1500)
    q = copy.deepcopy(probs)
    s1.gvins_optimization_batch(probs, 20)
    s2.gvins_optimization_batch(q, 20)
    return s1, s2


def test_slide_chain_of_every_factor_with_wrapped_alignment_beside_a_one_item_window(olib):
    """window 0: 11 chained items, Normal and Earth alternating, 33 to 2001 rows, 11 aligned fixes; window 1: one item"""
    lengths = [101, 2001, 33, 201, 101, 1001, 41, 101, 2001, 65, 101]
    normal = [k % 2 == 1 for k in range(11)]
    w0 = chain_window(olib, 1401, 13, lengths, normal)
    w1 = one_item_window(olib, 1411)
    assert (w0[3]["gnss_node"] >= 0).sum() == 11
    s1, s2 = solved([w0[0], w1[0]], 13)
    try:
        nx = [copy.deepcopy(w[1]) for w in (w0, w1)]
        station = np.array([0.53, 1.99, 25.0])
        outs = s1.slide_integrate(nx, [w0[2], w1[2]], [w0[3], w1[3]], NOISE5, station, False)
        twins = [host_twin(w[0], w[1], w[2], w[3], o, station) for w, o in zip((w0, w1), outs)]
        s2.slide(twins, [w0[2], w1[2]], False)
        for w, (o, b) in enumerate(zip(outs, twins)):
            assert (o["status"][np.asarray([s != -1 for s in (w0, w1)[w][3]["imu_from"]])] == 1).all(), w
            for k in np.nonzero(o["status"] == 1)[0]:
                assert np.array_equal(o["blobs"][k], b["imu_blob"].reshape(-1, IMU)[k]), (w, k)
        s1.download(), s2.download()  # the gathered node rows
        for a, b in zip(nx, twins):
            for key in ("pose", "mix"):
                assert np.array_equal(a[key], b[key]), key
        # the aligned fixes stay on the device: the solves see them, so the two handles agree only if all 11 moved as the twin's did
        assert not np.array_equal(twins[0]["gnss_blh"], w0[1]["gnss_blh"])
        s1.run_gvins(20), s2.run_gvins(20)
        assert s1.gvins_optimization_end(nx) == s2.gvins_optimization_end(twins)
        for a, b in zip(nx, twins):
            for key in PARAMS:
                assert np.array_equal(a[key], b[key]), key
    finally:
        s1.close(), s2.close()


def test_slide_chain_through_2_row_items(olib):
    """a chain of 9 items with 2-row items in it: the call is refused (their covariance is not positive definite), and every blob and end
    state it returns -- the items after the short ones start from their end states -- equals the host chain"""
    from ic_gvins_b200._lib import IcgError
    lengths = [101, 2, 2001, 33, 2, 101, 3, 201, 101]
    normal = [k in (1, 2, 5, 8) for k in range(9)]
    w0 = chain_window(olib, 1421, 11, lengths, normal)
    w1 = one_item_window(olib, 1431)
    s1, s2 = solved([w0[0], w1[0]], 11)
    try:
        nx = [copy.deepcopy(w[1]) for w in (w0, w1)]
        with pytest.raises(IcgError, match="not positive definite") as e:
            s1.slide_integrate(nx, [w0[2], w1[2]], [w0[3], w1[3]], NOISE5, np.zeros(3), False)
        outs = e.value.results
    finally:
        s1.close(), s2.close()
    p = w0[0]
    st = state16(p["pose"].reshape(-1, 7)[-1], p["mix"].reshape(-1, 9)[-1])
    refused = []
    for k, n in enumerate(lengths):
        iw = None if normal[k] else earth_iewn(np.zeros(3), st[:3])
        hb, he = host(st, iw, synth_ba.GRAVITY, NOISE5, w0[3]["imu_rows"][k + 1])
        assert np.array_equal(outs[0]["blobs"][k + 1], hb) and np.array_equal(outs[0]["end_states"][k + 1], he), k
        refused.append(upload_refuses(p, 0, hb))
        st = state16(he[:7], np.r_[he[7:10], st[10:16]])
    assert np.array_equal(outs[0]["status"], np.r_[0, np.where(refused, -1, 1)].astype(np.int8)), outs[0]["status"]
    assert refused[1] and refused[4] and not refused[2]
    assert outs[1]["status"][-1] == 1
