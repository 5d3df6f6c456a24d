"""GPU: the series cut of the INS windows (ins_cut_kernel, csrc/ins.cu) as the window solver's sample store receives it
(icg_ba_imu_samples_from_ins, read back with icg_ba_imu_samples), against getImuSeriesFromTo of the std::deque restatement
(tests/ins_series_oracle.cpp): rows bitwise, row counts exact.  Every node time is the end of one interval and the start of the next, so
each case below is met at both ends: a time on a sample, each isNeedInterpolation case (-1, 1, 2), one-ulp knife edges on both sides of
MINIMUM_TIME_INTERVAL from either sample, and both ends inside one sample interval; on rings wrapped past their capacity, in the Earth and
the Normal form."""
import numpy as np
import pytest

from datagen import synth_ba
from tests import ins_series_oracle as so
from tests import oracle_api as oa
from tests.test_oracle_gins_init import moving

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not so.HAVE_CXX, reason="no host C++ compiler for the INS restatement")]
NOISE5 = synth_ba.NOISE5
MIN_DT = 1e-4  # MISC::MINIMUM_TIME_INTERVAL
K = 6


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
    return {"with_earth": s % 2 == 0, "gravity": synth_ba.GRAVITY}


def _times(T, i):
    """node time cases around sample i of row times T"""
    a, b = T[i], T[i + 1]
    lo, hi = a + MIN_DT, b - MIN_DT
    return [a, a + 0.5 * MIN_DT, b - 0.5 * MIN_DT, 0.5 * (a + b), lo, np.nextafter(lo, 0), np.nextafter(lo, 99), hi, np.nextafter(hi, 0),
            np.nextafter(hi, 99)]


def _node_times(T, w):
    """K increasing node times of window w: node j near sample 40 + 45 j, each taking a case in turn; window 3 starts with both ends of
    its first interval inside one sample interval"""
    out = []
    for j in range(K):
        c = _times(T, 40 + 45 * j + (w % 5))
        out.append(c[(w + 3 * j) % len(c)])
    if w % 7 == 3:
        i = 40 + (w % 5)
        out[0], out[1] = T[i] + 0.0004, T[i] + 0.0031
    return np.array(out)


def _setup(n_streams, olib):
    """INS windows (device and restatement) of n_streams streams: odd streams get 1.5 capacities of rows, so their rings wrap; then a
    redo near the front mechanizes every stream; a solver with n_streams uploaded windows of K nodes"""
    from ic_gvins_b200.ba import WindowSolver
    from ic_gvins_b200.ins import InsWindow
    d, o = InsWindow(n_streams), so.OracleSeries(n_streams)
    rows = []
    for s in range(n_streams):
        t0 = 10.0 + 0.0013 * s
        r = moving(t0 - (2.6 if s % 2 else 0.0), t0 + 3.9, seed=s, earth=_cfg(s)["with_earth"])
        rows.append(r)
    cfg = [_cfg(s) for s in range(n_streams)]
    d.push(rows, cfg)
    assert o.push(rows, cfg) == 0
    win = [d.window(s)[0][:, 0] for s in range(n_streams)]
    st = np.zeros((n_streams, 17))
    st[:, 7] = 1
    st[:, 0] = [w[2] + 0.001 for w in win]
    np.testing.assert_array_equal(d.redo(st, cfg), o.redo(st, cfg))
    prob, _ = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=K, L=20, seed=5)
    solver = WindowSolver(max_windows=n_streams, max_K=K, max_L=20, max_F=max(1, prob["F"]), max_gnss=8, max_marg_r=1)
    solver.upload([prob] * n_streams)
    return d, o, solver, [d.window(s)[0][:, 0] for s in range(n_streams)]


def test_cut_equals_the_restatement(olib):
    n = 24
    d, o, s, T = _setup(n, olib)
    try:
        times = [_node_times(T[w], w) for w in range(n)]
        s.imu_samples_from_ins(d, list(range(n)), times)
        for w in range(n):
            got = s.imu_samples(w)
            assert len(got) == K - 1
            for k in range(K - 1):
                ref = o.series(w, times[w][k], times[w][k + 1])
                assert ref is not None, (w, k)
                assert got[k].shape == ref.shape, (w, k, got[k].shape, ref.shape)
                np.testing.assert_array_equal(got[k], ref, err_msg=f"window {w} factor {k}")
        assert all(len(T[w]) == 999 for w in range(1, n, 2))  # odd streams: 1000 rows of a wrapped ring, less the one the redo pruned
    finally:
        s.close(), d.close()


def test_interval_the_window_cannot_serve(olib):
    from ic_gvins_b200 import IcgError
    d, o, s, T = _setup(2, olib)
    try:
        good = [_node_times(T[w], w) for w in range(2)]
        s.imu_samples_from_ins(d, [0, 1], good)
        before = [s.imu_samples(w) for w in range(2)]
        for bad in (T[1][-1], T[1][-1] + 1.0, T[1][0] - 0.5):  # at the back (index 0), after it, before the front
            t = good[1].copy()
            if bad < T[1][0]:
                t[0] = bad
            else:
                t[-1] = bad
            assert o.series(1, t[0], t[1]) is None or o.series(1, t[-2], t[-1]) is None
            with pytest.raises(IcgError, match="window 1 IMU factor .* cannot serve"):
                s.imu_samples_from_ins(d, [0, 1], [good[0], t])
            for w in range(2):  # the store as it was
                for a, b in zip(s.imu_samples(w), before[w]):
                    np.testing.assert_array_equal(a, b)
        with pytest.raises(IcgError, match="not less than"):
            s.imu_samples_from_ins(d, [0, 1], [good[0], good[1][::-1].copy()])
        with pytest.raises(IcgError, match="out of range or not mechanized"):
            s.imu_samples_from_ins(d, [0, 5], good)
    finally:
        s.close(), d.close()


def test_seed_after_gins_initialization(olib):
    """the K = 2 GINS window seeded right after icg_ins_gins_initialize: its factor's rows are the initialization's own first-interval
    series, with its n_series rows"""
    from ic_gvins_b200.ba import WindowSolver
    from tests.test_gins_init_gpu import STATION, _first_window, _setup as gins_setup
    from tests.test_oracle_gins_init import GYR_BIAS_STD
    streams = [5, 6, 13, 14]
    d, o, _, inits, cfg = gins_setup(len(streams), streams)
    got, _ = d.gins_initialize(inits, cfg, NOISE5, STATION)
    ref, _ = o.gins_initialize(inits, cfg, GYR_BIAS_STD)
    assert (got["status"] == 1).all()
    solver = WindowSolver(max_windows=len(streams), max_K=2, max_L=0, max_F=0, max_gnss=8, max_marg_r=0)
    try:
        for g in inits:
            g["last_std"], g["gnss_std"] = (0.05, 0.05, 0.1), (0.06, 0.06, 0.12)
        wins = [_first_window(got, k, inits[k], got["imu_blob"][k], np.zeros((2, 4))) for k in range(len(streams))]
        solver.upload(wins)
        solver.imu_samples_from_ins(d, list(range(len(streams))), [[g["last_time"], g["gnss_time"]] for g in inits])
        for k in range(len(streams)):
            rows = solver.imu_samples(k)[0]
            assert rows.shape[0] == got["n_series"][k] == ref["n_series"][k]
            np.testing.assert_array_equal(rows, ref["series"][k][:, 1:])
    finally:
        solver.close(), d.close()
