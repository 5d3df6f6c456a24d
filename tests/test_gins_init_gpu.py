"""GPU: icg_ins_gins_initialize (ic_gvins_b200.ins.InsWindow.gins_initialize, csrc/ins.cu + preint.cu) against the CPU restatement of
gvinsInitialization (tests/gins_init_oracle.cpp) and the BA oracle's preintegration of the restatement's series.

Exact: statuses, has_zero_velocity, n_series, window counts, rows and state times, the biases (bg = mean(dtheta) rate is the same sums in
the same order on both sides), the priors' standard deviations.
Roll / pitch / heading: each is one asin / atan / atan2 of an operand both sides form bit for bit.  The CUDA Math API bounds these at 2 ulp
in double precision, glibc at 1 ulp, so the two results are at most 3 ulp of the angle apart: the bound is 4 ulp of each angle (relative,
so a levelled roll of 1e-2 rad is held to 4 ulp of 1e-2, not of pi).
q = euler2quaternion(initatt): each component is a product of three half-angle sines / cosines (2 ulp each on CUDA, 1 on glibc) summed in
two Hamilton products (4 roundings), all of magnitude <= 1, so 16 ulp of 1 (1.8e-15) covers the libm and rounding terms; an angle that is
d apart moves a component by at most d / 2, so QTOL = 1.8e-15 + sum_i 2 ulp(angle_i).  p = last_blh - q antlever: a rotation error of
2 QTOL moves q antlever by at most 2 QTOL |antlever|, plus 4 ulp of |p| for the products and the subtraction.
The window after the call: the TOL of tests/test_ins_gpu.py (5e-14 of each group's scale).  The first node's blob: the 1e-12 (head,
Jacobian) / 1e-10 (covariance) of the preintegration tests, and its end state within TOL.  The first GINS window built from these outputs
and solved: the tolerances of tests/test_ba_gpu.py's gvinsInitializationOptimization case."""
import math

import numpy as np
import pytest

from datagen import synth_ba
from tests import gins_init_oracle as go
from tests import oracle_api as oa
from tests.test_ins_gpu import TOL, _same_window, _state_err
from tests.test_ba_gpu import _compare_solution
from tests.test_oracle_gins_init import GYR_BIAS_STD, RATE, _knife, init, moving, still

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not go.HAVE_CXX, reason="no host C++ compiler for the INS restatement")]
ROUND_Q = 16 * 1.1102230246251565e-16  # 16 ulp of 1
NOISE5 = synth_ba.NOISE5
STATION = np.zeros(3)
B = 296
BRANCHES = ("time0", "rows19", "still", "short", "after_back", "moving", "dual", "on_row")


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


def _cfg(s):
    return {"with_earth": (s // len(BRANCHES)) % 2 == 0, "gravity": synth_ba.GRAVITY}


def _scenario(s):
    """rows and initialization input of stream s: branch s % 8, Earth / Normal form alternating every 8 streams"""
    b = BRANCHES[s % len(BRANCHES)]
    t0 = 10.0 + 0.013 * s
    earth = _cfg(s)["with_earth"]
    r = still(t0, t0 + 3.0, seed=s) if b == "still" else moving(t0, t0 + 3.0, seed=s, earth=earth)
    last, gnss = t0 + 1.0023, t0 + 2.0023
    g = init(last, gnss)
    if b == "time0":
        g = init(0.0, gnss)
    elif b == "rows19":
        g = init(r[200, 0], r[220, 0])
    elif b == "short":
        g = init(last, gnss, disp=(0.2, 0.3, 0.0))
    elif b == "after_back":
        g = init(t0 + 2.5, t0 + 3.5)
    elif b == "dual":
        g = init(last, gnss, disp=(0.0, 0.0, 0.0), last_yaw_valid=1, last_yaw=0.01 * s - 1.5)
    elif b == "on_row":  # both ends exactly on rows: no interpolation at either end
        g = init(r[201, 0], r[401, 0])
    g["antlever"] = (0.1 + 1e-3 * s, -0.2, 0.3)
    return r, g


def _setup(n, streams):
    from ic_gvins_b200.ins import InsWindow
    d, o = InsWindow(n), go.OracleGins(n)
    rows, inits = [], []
    for s in streams:
        r, g = _scenario(s)
        rows.append(r), inits.append(g)
    cfg = [_cfg(s) for s in streams]
    d.push(rows, cfg)
    assert o.push(rows, cfg) == 0
    return d, o, rows, inits, cfg


def _check_outputs(got, ref, cfg_d, cfg_o, olib, inits):
    cfg_lever = [g["antlever"] for g in inits]
    for k in ("status", "has_zero_velocity"):
        np.testing.assert_array_equal(got[k], ref[k])
    np.testing.assert_array_equal(got["bg"], ref["bg"])
    assert (np.abs(got["initatt"] - ref["initatt"]) <= 4 * np.spacing(np.abs(ref["initatt"]))).all()
    ok = got["status"] == 1
    np.testing.assert_array_equal(got["n_series"][ok], ref["n_series"][ok])
    for s in np.nonzero(ok)[0]:
        x, xo = got["state17"][s, 0], ref["state17"][s]
        assert x[0] == xo[0]
        np.testing.assert_array_equal(x[8:17], xo[8:17])
        qtol = ROUND_Q + 2 * np.spacing(np.abs(ref["initatt"][s])).sum()
        assert np.abs(x[4:8] - xo[4:8]).max() <= qtol
        lever = np.linalg.norm(cfg_lever[s])
        assert np.abs(x[1:4] - xo[1:4]).max() <= 2 * qtol * lever + 4 * np.spacing(np.abs(xo[1:4]).max())
        np.testing.assert_array_equal(got["pose_prior"][s], x[1:8]), np.testing.assert_array_equal(got["mix_prior"][s], x[8:17])
        np.testing.assert_array_equal(got["pose_prior_std"][s], ref["pose_prior_std"][s])
        np.testing.assert_array_equal(got["mix_prior_std"][s], ref["mix_prior_std"][s])
        assert cfg_d[s]["gravity"] == cfg_o[s]["gravity"]
        if cfg_o[s]["with_earth"]:
            assert np.abs(np.array(cfg_d[s]["iewn"]) - cfg_o[s]["iewn"]).max() <= 1e-19  # |iewn| = 7.3e-5: a few of its ulps
        # the first GNSS node's factor: the oracle's preintegration of the restatement's series from stateFromData(state17[0])
        st16 = xo[1:17].copy()
        st16[3:7] /= math.sqrt(sum(v * v for v in st16[3:7]))
        iw = go.earth_iewn(STATION, st16[:3]) if cfg_o[s]["with_earth"] else None
        bo, _, end = oa.preintegrate(olib, st16, iw, np.array([0, 0, cfg_o[s]["gravity"][2]]), NOISE5, ref["series"][s][:, 1:])
        b = got["imu_blob"][s]
        assert np.abs(b[:27] - bo[:27]).max() <= 1e-12 * max(1.0, np.abs(bo[:27]).max()), s
        assert np.abs(b[27:252] - bo[27:252]).max() <= 1e-12 * np.abs(bo[27:252]).max(), s
        assert np.abs(b[252:477] - bo[252:477]).max() <= 1e-10 * np.abs(bo[252:477]).max(), s
        np.testing.assert_array_equal(b[477:], bo[477:])
        x1 = got["state17"][s, 1]
        assert x1[0] == ref_gnss_time(ref, s)
        np.testing.assert_array_equal(x1[11:17], xo[11:17])
        e1 = np.concatenate([[x1[0]], end, x1[11:17]])
        assert _state_err(x1[None], e1[None]) <= TOL, s
    not_ok = ~ok
    assert not got["state17"][not_ok].any() and not got["imu_blob"][not_ok].any()


def ref_gnss_time(ref, s):
    return ref["series"][s][-1, 0]  # getImuSeriesFromTo sets the last row's time to gnss_time


def _windows(d, n):
    return [d.window(s) for s in range(n)]


def test_b296_every_branch_both_forms(olib):
    streams = list(range(B))
    d, o, rows, inits, cfg = _setup(B, streams)
    sel = np.array([s % 37 != 36 for s in streams], np.uint8)
    before = _windows(d, B)
    got, cfg_d = d.gins_initialize(inits, cfg, NOISE5, STATION, sel=sel)
    ref, cfg_o = o.gins_initialize(inits, cfg, GYR_BIAS_STD, sel=sel)
    expect = {"time0": -1, "rows19": -2, "still": -3, "short": -4, "after_back": -5, "moving": 1, "dual": 1, "on_row": 1}
    for s in streams:
        assert got["status"][s] == (expect[BRANCHES[s % 8]] if sel[s] else 0), s
    _check_outputs(got, ref, cfg_d, cfg_o, olib, inits)
    for s in streams:
        if got["status"][s] == 1:
            _same_window(d, o, s)
        else:  # unselected and rejected streams: the window bitwise as it was
            imu, st = d.window(s)
            np.testing.assert_array_equal(imu, before[s][0]), np.testing.assert_array_equal(st, before[s][1])
    # a zero-velocity stream, then motion: the levelled roll / pitch are kept
    zv = [s for s in streams if got["status"][s] == -3]
    more = [moving(rows[k][-1, 0] + 1 / RATE, rows[k][-1, 0] + 3.0, seed=500 + k) if k in zv else np.zeros((0, 8)) for k in streams]
    d.push(more, cfg)
    assert o.push(more, cfg) == 0
    inits2 = [init(m[0, 0] + 1.0023, m[0, 0] + 2.0023) if len(m) else inits[k] for k, m in enumerate(more)]
    sel2 = np.array([k in zv for k in streams], np.uint8)
    got2, cfg_d2 = d.gins_initialize(inits2, cfg, NOISE5, STATION, sel=sel2)
    ref2, cfg_o2 = o.gins_initialize(inits2, cfg, GYR_BIAS_STD, sel=sel2)
    assert all(got2["status"][k] == 1 for k in zv)
    for k in zv:
        np.testing.assert_array_equal(got2["initatt"][k, :2], got["initatt"][k, :2])
        np.testing.assert_array_equal(got2["mix_prior_std"][k, 3:6], GYR_BIAS_STD * 3)
        _same_window(d, o, k)
    _check_outputs(got2, ref2, cfg_d2, cfg_o2, olib, inits2)
    # initialized streams then take the mechanized path of icg_ins_push
    done = [k for k in streams if got["status"][k] == 1 or got2["status"][k] == 1]
    cfg_now = [cfg_d2[k] if got2["status"][k] == 1 else cfg_d[k] for k in streams]
    cfg_now_o = [cfg_o2[k] if got2["status"][k] == 1 else cfg_o[k] for k in streams]
    tail = [moving(d.window(k)[0][-1, 0] + 1 / RATE, d.window(k)[0][-1, 0] + 0.5, seed=900 + k) if k in done else np.zeros((0, 8))
            for k in streams]
    d.push(tail, cfg_now)
    assert o.push(tail, cfg_now_o) == 0
    for k in done:
        _same_window(d, o, k)
        assert d.window(k)[1][-1, 1:8].any()  # mechanized: the new rows carry states


def test_batch_equals_single_streams(olib):
    streams = list(range(0, B, 5))
    d, _, _, inits, cfg = _setup(len(streams), streams)
    got, cfg_d = d.gins_initialize(inits, cfg, NOISE5, STATION)
    d1, _, _, _, _ = _setup(len(streams), streams)
    for k in range(len(streams)):
        sel = np.zeros(len(streams), np.uint8)
        sel[k] = 1
        one, cfg1 = d1.gins_initialize(inits, cfg, NOISE5, STATION, sel=sel)
        for key in got:
            np.testing.assert_array_equal(one[key][k], got[key][k]), key
        assert cfg1[k] == cfg_d[k]
    for k in range(len(streams)):
        a, b = d.window(k), d1.window(k)
        np.testing.assert_array_equal(a[0], b[0]), np.testing.assert_array_equal(a[1], b[1])


def test_rejects_mechanized_and_bad_arguments():
    from ic_gvins_b200 import IcgError
    streams = [5, 6]
    d, _, _, inits, cfg = _setup(2, streams)
    got, cfg_d = d.gins_initialize(inits, cfg, NOISE5, STATION)
    assert list(got["status"]) == [1, 1]
    before = _windows(d, 2)
    with pytest.raises(IcgError, match="already mechanized"):
        d.gins_initialize(inits, cfg, NOISE5, STATION, sel=[0, 1])
    with pytest.raises(IcgError):
        d.gins_initialize(inits, cfg, NOISE5, STATION, reserved=-1)
    # the C ABI's own checks: a configuration whose form is neither 0 nor 1, and missing arrays (the wrapper never passes either)
    import ctypes as C
    from ic_gvins_b200._lib import GinsInit, GinsInitOut, InsConfig, lib
    from ic_gvins_b200.ins import _configs
    d2, _, _, inits2, cfg2 = _setup(2, [5, 6])
    c = _configs(cfg2, 2)
    arr, res = (GinsInit * 2)(), (GinsInitOut * 2)()
    for k, g in enumerate(inits2):
        arr[k].gnss_time, arr[k].last_time, arr[k].gravity, arr[k].imudatarate = g["gnss_time"], g["last_time"], g["gravity"], g["imudatarate"]
    nz, stn = np.ascontiguousarray(NOISE5, np.float64), np.zeros(3)
    c[1].with_earth = 2
    assert lib().icg_ins_gins_initialize(d2._h, 2, c, None, arr, C.c_void_p(nz.ctypes.data), C.c_void_p(stn.ctypes.data), 2, res) != 0
    c[1].with_earth = 0
    for args in ((c, None, arr, None, C.c_void_p(stn.ctypes.data), res), (c, None, None, C.c_void_p(nz.ctypes.data), C.c_void_p(stn.ctypes.data), res),
                 (c, None, arr, C.c_void_p(nz.ctypes.data), C.c_void_p(stn.ctypes.data), None), (None, None, arr, C.c_void_p(nz.ctypes.data), C.c_void_p(stn.ctypes.data), res)):
        assert lib().icg_ins_gins_initialize(d2._h, 2, *args[:5], 2, args[5]) != 0
    for k in range(2):  # nothing was initialized by the refused calls
        assert not d2.window(k)[1][:, 1:].any()
    for k in range(2):
        np.testing.assert_array_equal(d.window(k)[1], before[k][1])


def test_knife_edges_on_the_device(olib):
    """the zero-velocity thresholds at their knife edge (the last amplitude below each and the next double, for a gyroscope and an
    accelerometer column of each threshold) and the window ends one ulp inside, as streams of one batch: statuses as the restatement's"""
    rows, inits, expect = [], [], []
    for col, thr in ((2, 0.002), (4, 0.002), (5, 0.1), (7, 0.1)):
        r = still(10.0, 12.0, noise=(0.0, 0.0))
        inside = (r[:, 0] > 10.5) & (r[:, 0] < 11.5)
        for vals, status in zip(_knife(col, thr, r[inside, col]), (-3, 1)):
            rr = r.copy()
            rr[inside, col] = vals
            rows.append(rr), inits.append(init(10.5, 11.5)), expect.append(status)
    r = moving(10.0, 13.0)
    t = r[:, 0]
    for g, status in ((init(t[200], t[220]), -2), (init(t[200], t[221]), 1), (init(np.nextafter(t[200], 0), t[220]), 1),
                      (init(t[200], np.nextafter(t[220], 99)), 1)):
        rows.append(r), inits.append(g), expect.append(status)
    from ic_gvins_b200.ins import InsWindow
    n = len(rows)
    cfg = [{"with_earth": k % 2 == 0, "gravity": synth_ba.GRAVITY} for k in range(n)]
    d, o = InsWindow(n), go.OracleGins(n)
    d.push(rows, cfg)
    assert o.push(rows, cfg) == 0
    got, cfg_d = d.gins_initialize(inits, cfg, NOISE5, STATION)
    ref, cfg_o = o.gins_initialize(inits, cfg, GYR_BIAS_STD)
    assert list(got["status"]) == expect == list(ref["status"])
    _check_outputs(got, ref, cfg_d, cfg_o, olib, inits)
    for k in range(n):
        if got["status"][k] == 1:
            _same_window(d, o, k)


def _gnss_on_trajectory(t, lever):
    p, _, _, psi = synth_ba.trajectory(t)
    return tuple(p + synth_ba.q_mat(synth_ba.q_yaw(psi)) @ np.asarray(lever))


def _first_window(out, s, g, blob, pn):
    """GVINS::gvinsInitializationOptimization's window (IG/ic_gvins.cc:694-722) after gvinsInitialization: the two states, the GNSS fixes
    at both nodes (Huber), the first node's IMU factor, ImuErrorFactor and the first-window priors; no landmarks"""
    x = out["state17"][s]
    return dict(
        K=2, L=0, F=0, pose=np.concatenate([x[0, 1:8], x[1, 1:8]]), mix=np.concatenate([x[0, 8:17], x[1, 8:17]]),
        ext=np.array([0, 0, 0, 0, 0, 0, 1.0, 0]), invdepth=np.zeros(0), ext_const=1, td_const=1,
        f_lm=np.zeros(0, np.int32), f_ref=np.zeros(0, np.int32), f_obs=np.zeros(0, np.int32), f_const=np.zeros(0), f_active=np.zeros(0, np.uint8),
        reproj_std=1.0, reproj_huber=1, n_imu=1, imu_blob=np.array(blob, np.float64), pn=np.array(pn, np.float64).reshape(-1),
        pn_off=np.array([0, np.asarray(pn).reshape(-1, 4).shape[0]], np.int32), has_imu_error=1,
        has_pose_prior=1, pose_prior=out["pose_prior"][s].copy(), pose_prior_std=out["pose_prior_std"][s].copy(),
        has_mix_prior=1, mix_prior=out["mix_prior"][s].copy(), mix_prior_std=out["mix_prior_std"][s].copy(),
        n_gnss=2, gnss_node=np.array([0, 1], np.int32), gnss_blh=np.array([*g["last_blh"], *g["gnss_blh"]]),
        gnss_std=np.array([*g["last_std"], *g["gnss_std"]]), lever=np.array(g["antlever"], np.float64), gnss_huber=1,
        marg_r=0, marg_nblocks=0, marg_block_type=np.zeros(0, np.int32), marg_block_node=np.zeros(0, np.int32),
        marg_x0=np.zeros(0), marg_J0=np.zeros(0), marg_e0=np.zeros(0))


def test_chain_redo_and_first_gins_window(olib):
    """The reference's next steps after gvinsInitialization returns true, on both sides:
      * isoptimized_ (:302-306): the next sample is pushed and the window redone from statedatalist_.back() = state17[1] (:272-280);
      * gvinsInitializationOptimization's first window built from the outputs -- both states, GNSS at both nodes, the IMU blob, the pose /
        mix priors -- solved with 50 iterations and L = F = 0, against the oracle solve of the window the restatement gives (its state17[0],
        its series preintegrated by the BA oracle, the same GNSS and priors), with test_ba_gpu.py's tolerances for that shape."""
    from ic_gvins_b200.ba import WindowSolver
    streams = [5, 6, 7, 13, 14, 15]  # moving, dual-antenna yaw, both ends on rows; Earth and Normal form
    rows, inits = [], []
    for s in streams:
        r, g = _scenario(s)
        lever = g["antlever"]
        g["last_blh"], g["gnss_blh"] = _gnss_on_trajectory(g["last_time"], lever), _gnss_on_trajectory(g["gnss_time"], lever)
        g["last_std"], g["gnss_std"] = (0.05, 0.05, 0.1), (0.06, 0.06, 0.12)
        rows.append(r), inits.append(g)
    cfg = [_cfg(s) for s in streams]
    n = len(streams)
    from ic_gvins_b200.ins import InsWindow
    d, o = InsWindow(n), go.OracleGins(n)
    d.push(rows, cfg)
    assert o.push(rows, cfg) == 0
    got, cfg_d = d.gins_initialize(inits, cfg, NOISE5, STATION)
    ref, cfg_o = o.gins_initialize(inits, cfg, GYR_BIAS_STD)
    assert (got["status"] == 1).all() and (ref["status"] == 1).all()
    # the restatement's state17[1] and blob: the BA oracle's preintegration of its series
    ref_x1, ref_blob, ref_pn = [], [], []
    for k in range(n):
        xo = ref["state17"][k]
        st16 = xo[1:17].copy()
        st16[3:7] /= math.sqrt(sum(v * v for v in st16[3:7]))
        iw = go.earth_iewn(STATION, st16[:3]) if cfg_o[k]["with_earth"] else None
        bo, pn, end = oa.preintegrate(olib, st16, iw, np.array([0, 0, cfg_o[k]["gravity"][2]]), NOISE5, ref["series"][k][:, 1:])
        ref_x1.append(np.concatenate([[inits[k]["gnss_time"]], end, xo[11:17]])), ref_blob.append(bo), ref_pn.append(pn)
    ref_x1 = np.array(ref_x1)
    # isoptimized_: push the next samples, redo from state17[1]
    tail = [moving(r[-1, 0] + 1 / RATE, r[-1, 0] + 0.3, seed=700 + k) for k, r in enumerate(rows)]
    d.push(tail, cfg_d)
    assert o.push(tail, cfg_o) == 0
    np.testing.assert_array_equal(d.redo(got["state17"][:, 1], cfg_d), o.redo(ref_x1, cfg_o))
    for k in range(n):
        _same_window(d, o, k)
    # the first GINS window, solved
    solver = WindowSolver(max_windows=1, max_K=4, max_L=0, max_F=0, max_gnss=8, max_marg_r=0)
    try:
        for k in range(n):
            ref_out = dict(ref, state17=np.stack([ref["state17"], ref_x1], axis=1))
            pg = _first_window(got, k, inits[k], got["imu_blob"][k], ref_pn[k])
            po = _first_window(ref_out, k, inits[k], ref_blob[k], ref_pn[k])
            so = oa.ba_solve(olib, po, 50)
            sg = solver.solve(pg, 50)[0]
            assert sg["iterations"] == so["iterations"] and sg["termination"] == so["termination"], (k, sg, so)
            assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-7 * so["final_cost"], k
            _compare_solution(pg, po)
    finally:
        solver.close()
