"""GPU: icg_ba_slide_integrate_resident.  Each case slides one handle with the new IMU factors, node rows and aligned GNSS fixes integrated on
the device, and slides a twin handle that went through the same calls with the same rows computed on the host (icg_imu_preintegrate from
the downloaded start states, the alignment in numpy) through icg_ba_slide_resident.  Blobs, node rows, the two-pass solve, a resident
marginalization and a restarted solve must then be the same bits; the integrated blobs must match the oracle's preintegration."""
import copy

import numpy as np
import pytest

from datagen import synth_ba
from datagen.slide_window import build_next
from tests import oracle_api as oa
from tests.test_marg_large_gpu import make as make_large
from tests.test_post_solve_gpu import make
from tests.test_reintegration_gpu import STATION, earth_iewn, state16
from tests.test_slide_gpu import PARAMS, chain, handle

pytestmark = pytest.mark.gpu

IMU = 480
NOISE5 = synth_ba.NOISE5
CHAIN, ROW = -2, -3


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def cam():
    from ic_gvins_b200.camera import Camera
    from tests.test_post_solve_gpu import CAMD
    return Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])


def intervals(p, k0, n, seed, earth=True):
    """n consecutive fresh IMU intervals of 0.5 s at 200 Hz from node k0's time (the synthetic windows put node k at 0.5 k)"""
    rng = np.random.default_rng(seed)
    mix = p["mix"].reshape(p["K"], 9)[min(k0, p["K"] - 1)]
    return [synth_ba.imu_samples(0.5 * (k0 + j), 0.5 * (k0 + j + 1), 200.0, rng, mix[3:6], mix[6:9], earth=earth) for j in range(n)]


def integ_for(nxt, carry, sources, rows, normal=False, state=None, align=None):
    """the integrate dict: sources = {new factor: imu_from}, rows = {new factor: rows}; every integrated factor's end node is flagged;
    align = (new fix, old node, dt)"""
    m, K = nxt["n_imu"], nxt["K"]
    g = dict(imu_from=np.full(m, -1, np.int32), imu_rows=[None] * m, gravity=synth_ba.GRAVITY, normal=normal,
             node_from_imu=np.zeros(K, np.uint8), gnss_node=np.full(nxt["n_gnss"], -1, np.int32), gnss_dt=np.zeros(nxt["n_gnss"]))
    for k, s in sources.items():
        assert carry["imu_src"][k] < 0
        g["imu_from"][k], g["imu_rows"][k] = s, rows[k]
        if carry["node_src"][k + 1] < 0:
            g["node_from_imu"][k + 1] = 1
    if state is not None:
        g["state16"] = state
    if align is not None:
        q, node, dt = align
        assert carry["gnss_src"][q] < 0
        g["gnss_node"][q], g["gnss_dt"][q] = node, dt
    return g


def host_twin(p, nxt, carry, g, out, station):
    """the next window with every row the call integrates computed on the host, from p's (downloaded) states"""
    from ic_gvins_b200.ba import imu_preintegrate
    q = copy.deepcopy(nxt)
    K = p["K"]
    pose, mix = p["pose"].reshape(K, 7), p["mix"].reshape(K, 9)
    blobs, qp, qm = q["imu_blob"].reshape(-1, IMU), q["pose"].reshape(-1, 7), q["mix"].reshape(-1, 9)
    normal = np.broadcast_to(np.asarray(g["normal"], bool), (q["n_imu"],))
    end = st = None
    for k, src in enumerate(g["imu_from"]):
        if carry["imu_src"][k] >= 0 or src == -1:
            continue
        if src >= 0:
            st = state16(pose[src], mix[src])
        elif src == CHAIN:
            st = state16(end[:7], np.r_[end[7:10], st[10:16]])
        else:
            st = np.asarray(g["state16"][k], np.float64)
        iw = None
        if not normal[k]:
            iw = out["blobs"][k, 20:23]
            assert np.abs(iw - earth_iewn(station, st[:3])).max() <= 1e-15 * np.abs(iw).max()
        blobs[k], end = imu_preintegrate(st, iw, synth_ba.GRAVITY, NOISE5, g["imu_rows"][k])
        assert np.array_equal(end, out["end_states"][k]), k
        if g["node_from_imu"][k + 1] and carry["node_src"][k + 1] < 0:
            qp[k + 1], qm[k + 1] = end[:7], np.r_[end[7:10], st[10:16]]
    blh = q["gnss_blh"].reshape(-1, 3)
    for f, node in enumerate(g["gnss_node"]):
        if node >= 0 and carry["gnss_src"][f] < 0:
            blh[f] = blh[f] + mix[node, :3] * g["gnss_dt"][f]
    return q


def oracle_check(olib, got, st, rows, iw):
    bo = oa.preintegrate(olib, st, iw, synth_ba.GRAVITY, NOISE5, rows)[0]
    assert np.abs(got[:27] - bo[:27]).max() <= 1e-12 * max(1.0, np.abs(bo[:27]).max())
    assert np.abs(got[27:252] - bo[27:252]).max() <= 1e-12 * np.abs(bo[27:252]).max()
    assert np.abs(got[252:477] - bo[252:477]).max() <= 1e-10 * np.abs(bo[252:477]).max()


def compare(s1, s2, a, b, n_iter=20, marg=True):
    """the solve, a resident marginalization and a restarted solve of the two handles, bitwise"""
    for s in (s1, s2):
        s.run_gvins(n_iter)
    assert s1.gvins_optimization_end([a]) == s2.gvins_optimization_end([b])
    for k in PARAMS:
        assert np.array_equal(a[k], b[k]), k
    if marg:
        m1, m2 = s1.marginalize([a], 1, resident=True)[0], s2.marginalize([b], 1, resident=True)[0]
        assert m1["m"] == m2["m"] and m1["r"] == m2["r"]
        for k in ("J0", "e0", "Hp", "bp"):
            assert np.array_equal(m1[k], m2[k]), k
    for s in (s1, s2):
        s.run_gvins(n_iter, restart=True)
    assert s1.gvins_optimization_end([a]) == s2.gvins_optimization_end([b])
    for k in PARAMS:
        assert np.array_equal(a[k], b[k]), k


def twin(s1, s2, p, nxt, carry, g, prior, station=np.zeros(3), n_iter=20):
    """slide s1 with the integration and s2 with the host twin; compare blobs, node rows and GNSS rows, then the solves.  Returns (out, twin)"""
    a = copy.deepcopy(nxt)
    out = s1.slide_integrate([a], [carry], [g], NOISE5, station, prior)[0]
    b = host_twin(p, nxt, carry, g, out, station)
    s2.slide([b], [carry], prior)
    done = np.nonzero(out["status"] == 1)[0]
    assert list(done) == [k for k, s in enumerate(g["imu_from"]) if s != -1 and carry["imu_src"][k] < 0]
    assert not out["status"][out["status"] != 1].any()
    for k in done:
        assert np.array_equal(out["blobs"][k], b["imu_blob"].reshape(-1, IMU)[k]), k
    s1.download(), s2.download()  # the gathered node rows
    assert np.array_equal(a["pose"], b["pose"]) and np.array_equal(a["mix"], b["mix"])
    assert not np.isnan(a["pose"]).any() and not np.isnan(a["mix"]).any()
    compare(s1, s2, a, b, n_iter)
    return out, b


def new_keyframe_case(p, seed, **kw):
    """drop node 0, one new keyframe node integrated from the last old node (addNewTimeNode)"""
    up, nxt, carry = build_next(p, seed, **kw)
    k = nxt["n_imu"] - 1
    return nxt, carry, {k: p["K"] - 1}, {k: intervals(p, p["K"] - 1, 1, seed)[0]}


@pytest.mark.parametrize("dt", [-0.04, 0.03], ids=["align_back", "align_forward"])
def test_new_keyframe_after_the_cfg3_chain(olib, cam, dt):
    """solve, culling, culled marginalization, then the next window with the new keyframe node integrated on the device and its GNSS fix
    aligned by the old last node's velocity (each branch of insertNewGnssTimeNode's alignment)"""
    p1 = make(olib, outliers=25, seed=901, K=10, L=300)
    p2 = copy.deepcopy(p1)
    s1, s2 = handle(), handle()
    try:
        mg, bad_lm, bad_f = chain(p1, s1, cam, 902, 10)
        chain(p2, s2, cam, 902, 10)
        for k in PARAMS:
            assert np.array_equal(p1[k], p2[k])
        nxt, carry, src, rows = new_keyframe_case(p1, 903, prior=mg, drop_lm=bad_lm, drop_f=bad_f)
        g = integ_for(nxt, carry, src, rows, align=(nxt["n_gnss"] - 1, p1["K"] - 1, dt))
        out, b = twin(s1, s2, p1, nxt, carry, g, True, STATION)
        k = nxt["n_imu"] - 1
        st = state16(p1["pose"].reshape(-1, 7)[-1], p1["mix"].reshape(-1, 9)[-1])
        oracle_check(olib, out["blobs"][k], st, rows[k], earth_iewn(STATION, st[:3]))
        assert not np.array_equal(b["gnss_blh"].reshape(-1, 3)[-1], nxt["gnss_blh"].reshape(-1, 3)[-1])
    finally:
        s1.close(), s2.close()




def solved_pair(p, **kw):
    """two handles that solved the same window; p is left with the solved states"""
    s1, s2 = handle(**kw), handle(**kw)
    q = copy.deepcopy(p)
    s1.gvins_optimization_batch([p], 20)
    s2.gvins_optimization_batch([q], 20)
    for k in PARAMS:
        assert np.array_equal(p[k], q[k])
    return s1, s2


@pytest.mark.parametrize("normal", [False, True], ids=["earth", "normal"])
def test_merged_middle_node(olib, normal):
    """removeUnusedTimeNode: node 5 leaves and factors 4 and 5 merge, replayed from factor 4's start state over its rows and factor 5's
    without their first row (ICG_SLIDE_ROW); the merged blob is the oracle's preintegration of that concatenated series.  A new keyframe
    node follows (NODE)."""
    p = make(olib, seed=911, K=8, L=120)
    s1, s2 = solved_pair(p, K=10)
    try:
        up, nxt, carry = build_next(p, 912, drop=(5,), n_new=1)
        assert list(carry["imu_src"]) == [0, 1, 2, 3, -1, 6, -1]
        r4, r5 = intervals(p, 4, 2, 913, earth=not normal)
        merged = np.concatenate([r4, r5[1:]])
        state = np.zeros((nxt["n_imu"], 16))
        state[4] = np.concatenate([p["pose"].reshape(-1, 7)[4], p["mix"].reshape(-1, 9)[4]])  # the state factor 4 began from, as given
        rows = {4: merged, 6: intervals(p, 7, 1, 914, earth=not normal)[0]}
        g = integ_for(nxt, carry, {4: ROW, 6: 7}, rows, normal=normal, state=state)
        assert g["node_from_imu"].tolist() == [0] * 7 + [1]
        out, _ = twin(s1, s2, p, nxt, carry, g, False)
        oracle_check(olib, out["blobs"][4], state[4], merged, None if normal else earth_iewn(np.zeros(3), state[4][:3]))
        assert out["blobs"][4][477] == (1.0 if normal else 0.0)
    finally:
        s1.close(), s2.close()


@pytest.mark.parametrize("normal", [False, True], ids=["earth", "normal"])
def test_gnss_insertion_with_a_tail_of_recreated_nodes(olib, normal):
    """insertNewGnssTimeNode's insertion: a node at the fix from the last old node (NODE), then two nodes re-created, each from the state
    the previous interval propagated (ICG_SLIDE_CHAIN)"""
    p = make(olib, seed=921, K=8, L=120)
    s1, s2 = solved_pair(p, K=10)
    try:
        up, nxt, carry = build_next(p, 922, drop=(0,), n_new=3)
        m = nxt["n_imu"]
        iv = intervals(p, 7, 3, 923, earth=not normal)
        g = integ_for(nxt, carry, {m - 3: 7, m - 2: CHAIN, m - 1: CHAIN}, {m - 3: iv[0], m - 2: iv[1], m - 1: iv[2]}, normal=normal)
        assert g["node_from_imu"][-3:].all() and not g["node_from_imu"][:-3].any()
        out, _ = twin(s1, s2, p, nxt, carry, g, False)
        st = state16(p["pose"].reshape(-1, 7)[7], p["mix"].reshape(-1, 9)[7])
        for k in range(m - 3, m):  # each interval against the oracle from the state the one before it ended in
            oracle_check(olib, out["blobs"][k], st, iv[k - m + 3], None if normal else earth_iewn(np.zeros(3), st[:3]))
            e = out["end_states"][k]
            st = state16(e[:7], np.r_[e[7:10], st[10:16]])
    finally:
        s1.close(), s2.close()


def test_reintegrated_blobs_carried_beside_a_new_one(olib):
    from tests.test_reintegration_gpu import window
    p, rows = window(olib, 931, K=10, L=120, lin=lambda k: (np.full(3, 9 * NOISE5[2]), np.zeros(3)))
    q = copy.deepcopy(p)
    s1, s2 = handle(), handle()
    try:
        for s, x in ((s1, p), (s2, q)):
            s.gvins_optimization_batch([x], 20)
            assert (s.reintegrate([x], NOISE5, np.zeros(3), [rows])[0]["status"] == 1).all()
        mg = s1.marginalize([p], 1, resident=True)[0]
        s2.marginalize([q], 1, resident=True)
        nxt, carry, src, rw = new_keyframe_case(p, 932, prior=mg)
        assert (carry["imu_src"] >= 0).sum() == 8
        twin(s1, s2, p, nxt, carry, integ_for(nxt, carry, src, rw), True)
    finally:
        s1.close(), s2.close()


def test_cfg4_split_pipeline(olib, cam):
    p1 = make_large(olib, K=20, L=2000, seed=2042, n_ref=20, prior=True)
    p2 = copy.deepcopy(p1)
    kw = dict(K=20, L=2000, F=12000, R=292)
    s1, s2 = handle(**kw), handle(**kw)
    try:
        mg, bad_lm, bad_f = chain(p1, s1, cam, 941, 20)
        chain(p2, s2, cam, 941, 20)
        nxt, carry, src, rows = new_keyframe_case(p1, 942, prior=mg, drop_lm=bad_lm, drop_f=bad_f)
        twin(s1, s2, p1, nxt, carry, integ_for(nxt, carry, src, rows), True, n_iter=12)
    finally:
        s1.close(), s2.close()


def mixed_cases(olib):
    """three windows of different sizes and kinds of integration: a new keyframe with an aligned fix, a merge, a GNSS tail in the Normal form"""
    probs = [make(olib, seed=951, K=8, L=150), make(olib, seed=952, K=6, L=80), make(olib, seed=953, K=7, L=120)]
    return probs


def next_for(w, p):
    if w == 0:
        nxt, carry, src, rows = new_keyframe_case(p, 961)
        return nxt, carry, integ_for(nxt, carry, src, rows, align=(nxt["n_gnss"] - 1, p["K"] - 1, -0.02))
    if w == 1:
        up, nxt, carry = build_next(p, 962, drop=(3,), n_new=1)
        r2, r3 = intervals(p, 2, 2, 963)
        state = np.zeros((nxt["n_imu"], 16))
        state[2] = np.concatenate([p["pose"].reshape(-1, 7)[2], p["mix"].reshape(-1, 9)[2]])
        rows = {2: np.concatenate([r2, r3[1:]]), nxt["n_imu"] - 1: intervals(p, p["K"] - 1, 1, 964)[0]}
        return nxt, carry, integ_for(nxt, carry, {2: ROW, nxt["n_imu"] - 1: p["K"] - 1}, rows, state=state)
    up, nxt, carry = build_next(p, 965, drop=(0,), n_new=2)
    m = nxt["n_imu"]
    iv = intervals(p, p["K"] - 1, 2, 966, earth=False)
    return nxt, carry, integ_for(nxt, carry, {m - 2: p["K"] - 1, m - 1: CHAIN}, {m - 2: iv[0], m - 1: iv[1]}, normal=True)


def test_mixed_batch_equals_per_window_calls(olib):
    from ic_gvins_b200.ba import WindowSolver
    probs = mixed_cases(olib)
    s = WindowSolver(max_windows=3, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=160)
    try:
        s.gvins_optimization_batch(probs, 20)
        cases = [next_for(w, p) for w, p in enumerate(probs)]
        nx = [copy.deepcopy(c[0]) for c in cases]
        outs = s.slide_integrate(nx, [c[1] for c in cases], [c[2] for c in cases], NOISE5, STATION, False)
        s.run_gvins(20)
        batch = s.gvins_optimization_end(nx)
    finally:
        s.close()
    for w, p in enumerate(mixed_cases(olib)):
        one = handle(K=10)
        try:
            one.gvins_optimization_batch([p], 20)
            nxt, carry, g = next_for(w, p)
            o = one.slide_integrate([nxt], [carry], [g], NOISE5, STATION, False)[0]
            for k in ("status", "blobs", "end_states"):
                assert np.array_equal(o[k], outs[w][k]), (w, k)
            one.run_gvins(20)
            assert one.gvins_optimization_end([nxt])[0] == batch[w]
        finally:
            one.close()
        for k in PARAMS:
            assert np.array_equal(nxt[k], nx[w][k]), (w, k)


def test_rejections_leave_the_handle_as_it_was(olib):
    from ic_gvins_b200 import IcgError
    p = make(olib, seed=971, K=8, L=120)
    s = handle(K=10)

    def state():
        s.run_gvins(20, restart=True)
        q = copy.deepcopy(p)
        return s.gvins_optimization_end([q]), [q[k].copy() for k in PARAMS]

    def same(a, b):
        assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))

    def reject(nxt, carry, g, match):
        with pytest.raises(IcgError, match=match):
            s.slide_integrate([copy.deepcopy(nxt)], [carry], [g], NOISE5, np.zeros(3), False)
        same(base, state())

    try:
        s.gvins_optimization_batch([p], 20)
        base = state()
        nxt, carry, src, rows = new_keyframe_case(p, 972)
        k = nxt["n_imu"] - 1
        good = integ_for(nxt, carry, src, rows, align=(nxt["n_gnss"] - 1, p["K"] - 1, -0.02))
        g = copy.deepcopy(good)
        g["imu_from"][k] = CHAIN  # factor k - 1 is carried, not integrated
        reject(nxt, carry, g, "ICG_SLIDE_CHAIN")
        g = copy.deepcopy(good)
        g["imu_from"][k] = p["K"]
        reject(nxt, carry, g, "imu_from.*out of range")
        g = copy.deepcopy(good)
        g["gnss_node"][-1] = p["K"]
        reject(nxt, carry, g, "gnss_node.*out of range")
        g = copy.deepcopy(good)
        off = np.zeros(nxt["n_imu"] + 1, np.int32)
        off[k + 1:] = len(rows[k])
        g.update(imu=rows[k], imu_off=off.copy())
        g["imu_off"][k + 1] = g["imu_off"][k]
        reject(nxt, carry, g, "at least one row")
        g = copy.deepcopy(good)
        g["imu_from"][k] = -1
        reject(nxt, carry, g, "node_from_imu")
        g = copy.deepcopy(good)
        flat = rows[k].copy()
        flat[:, 0] = 0.0  # every sample of zero length: the covariance stays zero (finite, not positive definite)
        g["imu_rows"][k] = flat
        with pytest.raises(IcgError, match="not positive definite") as e:
            s.slide_integrate([copy.deepcopy(nxt)], [carry], [g], NOISE5, np.zeros(3), False)
        assert e.value.results[0]["status"][k] == -1
        same(base, state())
        s.slide_integrate([copy.deepcopy(nxt)], [carry], [good], NOISE5, np.zeros(3), False)  # the handle still takes a good call
    finally:
        s.close()
