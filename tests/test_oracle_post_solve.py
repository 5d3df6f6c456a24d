"""CPU: hand cases for every branch of the post-solve map update and outlier culling restated in tests/post_solve_oracle.py
(updateParametersFromOptimizer, gvinsOutlierCulling and the factor set of gvinsMarginalization after it, IG/ic_gvins.cc:1035-1389, 1558-1609)."""
import math

import numpy as np
import pytest

from tests import post_solve_oracle as po

CAM = dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0, skew=0.0)
STD = 1.0


def rotz(deg):
    a = math.radians(deg)
    return np.array([0.0, 0.0, math.sin(a / 2), math.cos(a / 2)])


def window(K=4, ext=None, invdepth=(0.1,)):
    pose = np.zeros((K, 7))
    pose[:, 0] = np.arange(K) * 0.5  # moving along x, identity attitude
    pose[:, 6] = 1.0
    e = np.array([0, 0, 0, 0, 0, 0, 1.0, 0.003]) if ext is None else np.asarray(ext, float)
    return dict(K=K, L=len(invdepth), F=0, pose=pose.reshape(-1), ext=e, invdepth=np.array(invdepth, float))


def inputs(ref_node, ref_kp, obs, **kw):
    """obs: per landmark a list of (node, (u, v)) in list order"""
    off = np.cumsum([0] + [len(o) for o in obs]).astype(np.int32)
    flat = [x for o in obs for x in o]
    ci = dict(R_bc=np.eye(3), t_bc=np.zeros(3), td_bc=0.001, estimate_ext=1, estimate_td=1, lm_ref_node=np.array(ref_node, np.int32),
              lm_ref_kp=np.array(ref_kp, np.float32).reshape(-1, 2), obs_off=off, obs_node=np.array([n for n, _ in flat], np.int32),
              obs_kp=np.array([kp for _, kp in flat], np.float32).reshape(-1, 2), obs_factor=np.full(len(flat), -1, np.int32))
    ci.update(kw)
    return ci


def project(prob, node, pw):
    """exact keypoint of pw in node (identity extrinsic)"""
    P = list(np.eye(3).reshape(-1)) + list(np.asarray(prob["pose"]).reshape(-1, 7)[node, :3])
    x, y, z = po.world2cam(P, pw)
    return tuple(float(v) for v in po.cam2pixel(CAM, x, y, z))


def pw_of(prob, ref, kp, invdepth):
    x, y = po.pixel2cam(CAM, np.float32(kp[0]), np.float32(kp[1]))
    d = 1.0 / invdepth
    return np.array([x * d, y * d, d]) + np.asarray(prob["pose"]).reshape(-1, 7)[ref, :3]


# ---------------------------------------------------------------------------------------------- extrinsic / td
@pytest.mark.parametrize("dt,deg,accepted", [(0.1, 1.0, 1), (1.5, 0.0, 0), (0.0, 12.0, 0), (0.0, 9.9, 1)])
def test_extrinsic_gate(dt, deg, accepted):
    """1 m / 5 deg gate; dr is |vec(q)| in degrees = sin(theta / 2) * 180 / pi, so a 9.9 deg rotation passes and 12 deg does not"""
    ext = np.concatenate([[dt, 0, 0], rotz(deg), [0.004]])
    prob = window(ext=ext, invdepth=())
    r = po.update_and_cull(prob, CAM, STD, inputs([], np.zeros((0, 2)), []))
    assert r["ext_accepted"] == accepted
    R = np.array(po.unit_quat_to_rot(ext[3:7])).reshape(3, 3)
    if accepted:
        assert np.allclose(r["R_bc_out"], R, atol=1e-15) and np.allclose(r["t_bc_out"], ext[:3])
    else:
        assert np.array_equal(r["R_bc_out"], np.eye(3)) and np.array_equal(r["t_bc_out"], np.zeros(3))
    assert r["td_bc_out"] == 0.004
    # camera poses use the gated extrinsic: R_c = R(q) R_bc, t_c = p + R(q) t_bc
    Rbc, tbc = r["R_bc_out"], r["t_bc_out"]
    for k in range(prob["K"]):
        assert np.allclose(r["cam_pose"][k, :9].reshape(3, 3), Rbc, atol=1e-15)
        assert np.allclose(r["cam_pose"][k, 9:], prob["pose"].reshape(-1, 7)[k, :3] + tbc, atol=1e-15)


def test_estimate_flags_off():
    ext = np.concatenate([[0.1, 0, 0], rotz(1.0), [0.004]])
    prob = window(ext=ext, invdepth=())
    r = po.update_and_cull(prob, CAM, STD, inputs([], np.zeros((0, 2)), [], estimate_ext=0, estimate_td=0, t_bc=np.array([0.01, 0, 0])))
    assert r["ext_accepted"] == -1 and r["td_bc_out"] == 0.001
    assert np.array_equal(r["R_bc_out"], np.eye(3)) and np.array_equal(r["t_bc_out"], [0.01, 0, 0])


def test_unnormalised_quaternions_are_normalised():
    ext = np.concatenate([[0.1, 0, 0], 3.0 * rotz(2.0), [0.0]])
    prob = window(ext=ext, invdepth=())
    prob["pose"].reshape(-1, 7)[1, 3:] = 2.0 * rotz(30.0)
    r = po.update_and_cull(prob, CAM, STD, inputs([], np.zeros((0, 2)), []))
    assert r["ext_accepted"] == 1
    Rq = np.array(po.unit_quat_to_rot(rotz(30.0))).reshape(3, 3)
    Re = np.array(po.unit_quat_to_rot(rotz(2.0))).reshape(3, 3)
    assert np.allclose(r["cam_pose"][1, :9].reshape(3, 3), Rq @ Re, atol=1e-14)


# ---------------------------------------------------------------------------------------------- culling
def scene(errs, ref_pos, rho=0.1, ref=0, K=4):
    """one landmark seen from nodes 0..K-1 (node `ref` is the reference); errs[i] = pixel error added to the i-th NON-reference
    observation; the reference observation sits at list position ref_pos"""
    prob = window(K=K, invdepth=(rho,))
    kp0 = (330.0, 250.0)
    pw = pw_of(prob, ref, kp0, 0.1)
    others = [k for k in range(K) if k != ref][:len(errs)]
    obs = [(k, (project(prob, k, pw)[0] + e, project(prob, k, pw)[1])) for k, e in zip(others, errs)]
    obs.insert(ref_pos, (ref, kp0))
    return prob, inputs([ref], [kp0], [obs])


def test_all_good():
    prob, ci = scene([0.0, 0.0, 0.0], 0)
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert r["lm_outlier"][0] == 0 and not r["obs_outlier"].any() and list(r["counts"]) == [0, 0, 0, 0, 0]
    assert np.allclose(r["lm_pw"][0], pw_of(prob, 0, (330.0, 250.0), 0.1), rtol=1e-15) and r["lm_depth"][0] == 10.0


def test_feature_outlier_only():
    prob, ci = scene([0.0, 5.0, 0.0], 0)
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert list(r["obs_outlier"]) == [0, 0, 1, 0] and r["lm_outlier"][0] == 0 and list(r["counts"]) == [0, 1, 0, 0, 0]


def test_reference_fails_after_others_double_counts_into_num2():
    """list order [node 1 good, node 0 = reference (moved away: fails), node 2 (not visited)]: reason 1, then < 2 good -> reason 2 too"""
    prob, ci = scene([0.0, 0.0], 1)
    ci["lm_ref_kp"] = ci["lm_ref_kp"].copy()
    ci["obs_kp"][1] = [400.0, 250.0]  # the reference observation's keyPoint() disagrees with pw
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert list(r["obs_outlier"]) == [0, 1, 0]  # node 2 after the break: neither checked nor flagged
    assert r["lm_outlier"][0] == 1 | 2 and list(r["counts"]) == [2, 0, 1, 1, 0]


def test_reference_fails_first_breaks():
    prob, ci = scene([0.0, 9.0], 0)
    ci["obs_kp"][0] = [400.0, 250.0]
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert list(r["obs_outlier"]) == [1, 0, 0]  # the bad node-2 observation is never checked
    assert r["lm_outlier"][0] == 1 | 2 and list(r["counts"]) == [2, 0, 1, 1, 0]


def test_reference_fails_after_two_high_errors_double_counts_into_num3():
    prob, ci = scene([2.0, 2.5], 2)
    ci["obs_kp"][2] = [400.0, 250.0]
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert list(r["obs_outlier"]) == [0, 0, 1]
    assert r["lm_outlier"][0] == 1 | 4 and list(r["counts"]) == [2, 0, 1, 0, 1]


def test_fewer_than_two_good():
    prob, ci = scene([5.0, 6.0], 0)
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert list(r["obs_outlier"]) == [0, 1, 1] and r["lm_outlier"][0] == 2 and list(r["counts"]) == [1, 2, 0, 1, 0]


def test_mean_above_std():
    prob, ci = scene([2.0, 2.0], 0)
    r = po.update_and_cull(prob, CAM, 1.2, ci)  # mean (0 + 2 + 2) / 3 > 1.2, each error <= 3.6
    assert not r["obs_outlier"].any() and r["lm_outlier"][0] == 4 and list(r["counts"]) == [1, 0, 0, 0, 1]
    r = po.update_and_cull(prob, CAM, 2.0, ci)  # mean (0 + 2 + 2) / 3 <= 2
    assert r["lm_outlier"][0] == 0


@pytest.mark.parametrize("rho", [-0.1, 0.0])
def test_non_positive_inverse_depth(rho):
    """1 / rho without a clamp: a negative depth puts the point behind every camera, a zero one gives inf / NaN coordinates; both fail
    the depth test at the reference observation and never enter the error sum"""
    prob, ci = scene([0.0, 0.0], 0, rho=rho)
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert r["lm_depth"][0] == (1.0 / rho if rho else math.inf)
    assert r["lm_outlier"][0] == 1 | 2 and list(r["obs_outlier"]) == [1, 0, 0] and list(r["counts"]) == [2, 0, 1, 1, 0]


def test_landmark_without_factor_rows():
    """only the reference observation (no factor row): pw is still updated; one good observation -> reason 2"""
    prob = window(invdepth=(0.2, 0.1))
    ci = inputs([1, 0], [(300.0, 200.0), (330.0, 250.0)], [[(1, (300.0, 200.0))], []])
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert np.allclose(r["lm_pw"][0], pw_of(prob, 1, (300.0, 200.0), 0.2), rtol=1e-15)
    assert list(r["lm_outlier"]) == [2, 2] and list(r["counts"]) == [2, 0, 0, 2, 0]


def test_outlier_flags_of_several_landmarks_accumulate():
    p1, c1 = scene([0.0, 5.0, 0.0], 0)
    r1 = po.update_and_cull(p1, CAM, STD, c1)
    p2, c2 = scene([5.0, 6.0], 0)
    r2 = po.update_and_cull(p2, CAM, STD, c2)
    prob = window(invdepth=(0.1, 0.1))
    n1 = len(c1["obs_node"])
    ci = inputs([0, 0], [(330.0, 250.0)] * 2, [list(zip(c1["obs_node"], map(tuple, c1["obs_kp"]))), list(zip(c2["obs_node"], map(tuple, c2["obs_kp"])))])
    r = po.update_and_cull(prob, CAM, STD, ci)
    assert np.array_equal(r["obs_outlier"][:n1], r1["obs_outlier"]) and np.array_equal(r["obs_outlier"][n1:], r2["obs_outlier"])
    assert np.array_equal(r["counts"], r1["counts"] + r2["counts"])


# ---------------------------------------------------------------------------------------------- factor set of the marginalization
def test_culled_factor_mask():
    """landmark 0: node-2 observation is a feature outlier (its factor goes, the others stay; the chi-square-removed row stays);
    landmark 1: reference observation flagged (all its factors go); landmark 2: a culling outlier; node 3 left the map"""
    prob = dict(K=4, L=3, F=7, f_lm=np.array([0, 0, 0, 1, 1, 2, 0], np.int32), f_obs=np.array([1, 2, 3, 1, 2, 1, 3], np.int32),
                f_active=np.array([0, 1, 1, 1, 1, 1, 1], np.uint8))
    prob["f_obs"][6] = 3
    ci = dict(lm_ref_node=np.array([0, 0, 0]), obs_off=np.array([0, 3, 6, 8]), obs_node=np.array([1, 0, 2, 0, 1, 2, 0, 1]),
              obs_factor=np.array([0, -1, 1, -1, 3, 4, -1, 5]))
    res = dict(lm_outlier=np.array([0, 0, 2], np.uint8), obs_outlier=np.array([0, 0, 1, 1, 0, 0, 0, 0], np.uint8))
    m = po.culled_factor_mask(prob, ci, res, [1, 1, 1, 1])
    assert list(m) == [1, 0, 1, 0, 0, 0, 1]  # row 0 was removed by chi2 and stays; row 2 has no listed observation and stays
    m = po.culled_factor_mask(prob, ci, res, [1, 1, 1, 0])
    assert list(m) == [1, 0, 0, 0, 0, 0, 0]
