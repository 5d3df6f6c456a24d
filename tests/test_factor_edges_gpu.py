"""GPU: every device factor evaluator, entry by entry, against the high-precision restatement (tests/factors_mp.py) on the edge sweep of
tests/test_factor_edges.py, with the same per-entry bounds: icg_ba_reproj_evaluate (the quaternion form), icg_ba_reproj_evaluate_frames
(the node-frame form ba_lin_vis and ba_cost run: node_frame rotation matrices, R^T for each quaternion inverse), icg_ba_imu_evaluate,
icg_ba_gnss_evaluate, icg_ba_pose_prior_evaluate, icg_ba_mix_prior_evaluate, icg_ba_imu_error_evaluate and icg_ba_marg_factor_evaluate;
and per window, the reprojection and GNSS costs of icg_ba_residual_costs against the restatement's 0.5 |r|^2.

Off the unit sphere the two reprojection forms are different functions: the reference (and the quaternion form) rotate by
q^-1 = conj(q) / |q|^2, the frame form by R(q)^T, which differ by 2 (|q|^2 - 1) (R^T - I) v.  tests/test_factor_edges.py pins that exact
gap per point (FRAME_GAP: at most 0.09 eps E for 1 to 4 ulp per component), and test_frame_form_gap reports the device's measured
frame-minus-quaternion difference per point; both are far inside C_REPROJ eps E, so the frame-form test cannot resolve them."""
import numpy as np
import pytest

from tests import factors_mp as fm
from tests import oracle_api as oa
from tests.test_factor_edges import (C_IMU, C_REPROJ, C_SMALL, HUBER_WINDOWS, check, huber_window, imu_ref, reproj_ref,
                                     residual_cost_ratios, window_cost)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def solver():
    from ic_gvins_b200.ba import WindowSolver
    s = WindowSolver(max_windows=1, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=64)
    yield s
    s.close()


@pytest.fixture(scope="module")
def prob(olib):
    return fm.window(lambda *a: oa.preintegrate(olib, *a), K=10, L=60, seed=11, with_priors=True)[0]


@pytest.fixture(autouse=True)
def _dps():
    import mpmath
    with mpmath.workdps(fm.DPS):
        yield


@pytest.mark.parametrize("frames", [False, True], ids=["quaternion_form", "frame_form"])
def test_reprojection(solver, prob, frames):
    worst = 0.0
    for p in fm.sweep_reprojection(prob):
        r, J = solver.reproj_evaluate(*p.args, frames=frames)
        worst = max(worst, *check(r, J, *reproj_ref(p.args), C_REPROJ, p))
    print(f"reprojection {'frame' if frames else 'quaternion'} form: worst error / (eps E) = {worst:.3g}")


def test_frame_form_gap(solver, prob):
    """the device's frame-form residual minus its quaternion-form residual, per point, in units of eps E (printed), within the bound"""
    from tests.test_factor_edges import frame_gap
    for p in fm.sweep_reprojection(prob):
        rq, _ = solver.reproj_evaluate(*p.args)
        rf, _ = solver.reproj_evaluate(*p.args, frames=True)
        e = fm.vals(reproj_ref(p.args)[0])[1]
        g = float((np.abs(rf - rq) / (fm.EPS * e)).max())
        print(f"frame - quaternion form: {g:.3g} eps E (exact gap {frame_gap(p):.3g})  {p.why}")
        assert g <= C_REPROJ, (p, g)


def test_gnss_and_priors(solver, prob):
    worst = 0.0
    for p in fm.sweep_gnss(prob):
        r, J = solver.gnss_evaluate(*p.args)
        worst = max(worst, *check(r, [J], *fm.gnss(*[fm.xs(x) for x in p.args]), C_SMALL, p))
    for p in fm.sweep_pose_prior(prob):
        r, J = solver.pose_prior_evaluate(*p.args)
        worst = max(worst, *check(r, [J], *fm.pose_prior(*[fm.xs(x) for x in p.args]), C_SMALL, p))
    for p in fm.sweep_mix(prob):
        r, J = solver.mix_prior_evaluate(*p.args)
        worst = max(worst, *check(r, [J], *fm.mix_prior(*[fm.xs(x) for x in p.args]), C_SMALL, p))
        r, J = solver.imu_error_evaluate(p.args[0])
        worst = max(worst, *check(r, [J], *fm.imu_error(fm.xs(p.args[0])), C_SMALL, p))
    print(f"GNSS / pose prior / mix prior / ImuErrorFactor: worst error / (eps E) = {worst:.3g}")


def test_imu(olib, solver):
    prep = lambda *a: oa.preintegrate(olib, *a)
    worst = 0.0
    for why, n, form, lat, far, db in fm.IMU_POINTS:
        blob, pn, p0, m0, p1, m1 = fm.interval(prep, n, form, lat, far, db, seed=n + int(lat))
        r, J = solver.imu_evaluate(blob, p0, m0, p1, m1)
        worst = max(worst, *check(r, J, *imu_ref(blob, pn, p0, m0, p1, m1), C_IMU, why))
    print(f"IMU: worst error / (eps E) = {worst:.3g}")
    from ic_gvins_b200 import IcgError
    blob, _, p0, m0, p1, m1 = fm.interval(prep, 3, "earth", seed=3)
    with pytest.raises(IcgError, match="not positive definite"):  # the singular covariance of test_three_row_interval_has_no_square_root_information
        solver.imu_evaluate(blob, p0, m0, p1, m1)


def test_marginalization(solver, prob):
    worst = 0.0
    for p in fm.sweep_marginalization(prob, np.random.default_rng(5)):
        types, params, x0, J0, e0 = p.args
        r, Js = solver.marg_factor_evaluate(types, params, x0, J0, e0)
        ref_r, ref_J = fm.marginalization(types, [fm.xs(q) for q in params], fm.xs(x0), [fm.xs(row) for row in J0], fm.xs(e0))
        worst = max(worst, *check(r, Js, ref_r, ref_J, C_SMALL, p))
    print(f"marginalization factor: worst error / (eps E) = {worst:.3g}")


def test_residual_costs(solver, prob):
    """icg_ba_residual_costs (the quaternion form, without the loss) per factor of a whole window: record slots map back to factor ids"""
    wr, wg = residual_cost_ratios(*solver.residual_costs(prob), prob)
    print(f"icg_ba_residual_costs: worst error / (eps E) = {wr:.3g} (reprojection), {wg:.3g} (GNSS)")
    assert wr <= C_REPROJ and wg <= C_SMALL


def test_huber_through_the_window_cost(solver, prob):
    """The device applies the loss inline in ba_lin_vis / ba_lin_cam (huber() of ba_math.cuh, then the sqrt(rho') scaling); no evaluator
    returns one factor's corrected residual.  The window solve's initial cost is the sum of every factor's 0.5 rho: it is held to the
    restated total with each loss on and off, the GNSS fixes on both sides of the knee (the per-factor knee points are held on the oracle)."""
    worst = 0.0
    for flags in HUBER_WINDOWS:
        p = huber_window(prob, *flags)
        ref = window_cost(p)
        s = solver.solve(p, 1)[0]
        worst = max(worst, abs(s["initial_cost"] - float(ref.v)) / (fm.EPS * float(ref.e)))
    print(f"window initial cost with and without the loss: worst error / (eps E) = {worst:.3g}")
    assert worst <= C_SMALL
