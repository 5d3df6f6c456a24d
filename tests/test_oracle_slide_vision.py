"""CPU: the numpy restatement of the next window's vision half (tests/slide_vision_oracle.py), one hand case per rule."""
import numpy as np
import pytest

from tests import slide_vision_oracle as so

CAM = dict(fx=400.0, fy=400.0, cx=320.0, cy=240.0, skew=0.0)


def window():
    """old window: 4 nodes, 4 landmarks; landmark l has reference node ref[l]; factor rows carry their index in pts0[0]"""
    f_lm = np.array([0, 0, 1, 1, 2, 3], np.int32)
    f_ref = np.array([0, 0, 1, 1, 1, 2], np.int32)
    f_obs = np.array([1, 2, 2, 3, 3, 3], np.int32)
    fc = np.zeros((6, 14))
    fc[:, 0] = np.arange(6)
    fc[:, 12] = 0.5
    old = dict(K=4, L=4, F=6, invdepth=np.array([0.5, 0.25, 0.2, 0.1]), f_lm=f_lm, f_ref=f_ref, f_obs=f_obs, f_const=fc)
    # observations: the reference one (factor -1) and one per factor
    obs_factor = np.array([-1, 0, 1, -1, 2, 3, -1, 4, -1, 5], np.int32)
    cull = dict(lm_ref_node=np.array([0, 1, 1, 2], np.int32), obs_off=np.array([0, 3, 6, 8, 10], np.int32), obs_factor=obs_factor,
                lm_outlier=np.zeros(4, np.uint8), obs_outlier=np.zeros(10, np.uint8))
    vis = dict(num_marg=1, node_in_map=np.ones(4, np.uint8), node_td=np.array([0.0, 0.01, 0.02, 0.03]), cur_node=3, frames={}, obs=[], new=[])
    return old, cull, [1, 2, 3, -1], vis


def run(old, cull, node_src, vis):
    return so.build(old, cull, node_src, vis, CAM)


def test_marginalized_anchor_removes_the_landmark():
    o = run(*window())
    assert o["lm_src"].tolist() == [1, 2, 3]  # landmark 0 is anchored in node 0
    assert o["f_src"].tolist() == [2, 3, 4, 5] and o["f_lm"].tolist() == [0, 0, 1, 2]
    assert o["f_ref"].tolist() == [0, 0, 0, 1] and o["f_obs"].tolist() == [1, 2, 2, 2]


def test_outlier_landmark_and_outlier_observation():
    old, cull, ns, vis = window()
    cull["lm_outlier"][2] = 1
    cull["obs_outlier"][5] = 1  # factor 3
    o = run(old, cull, ns, vis)
    assert o["lm_src"].tolist() == [1, 3] and o["f_src"].tolist() == [2, 5]


def test_reference_keyframe_not_in_the_map():
    old, cull, ns, vis = window()
    vis["node_in_map"][2] = 0
    o = run(old, cull, ns, vis)
    assert o["lm_src"].tolist() == [1, 2]  # landmark 3's reference node left the map
    assert o["f_src"].tolist() == [3, 4]   # factor 2 was observed in node 2 too


def test_nan_and_zero_inverse_depth():
    old, cull, ns, vis = window()
    old["invdepth"][1] = np.nan
    old["invdepth"][2] = 0.0
    o = run(old, cull, ns, vis)
    assert o["nan_dropped"] == 1 and o["lm_src"].tolist() == [-1, 3]
    assert o["invdepth"][0] == 0.1


def test_chi2_removed_factors_come_back_and_unlisted_ones_do_not():
    old, cull, ns, vis = window()
    cull["obs_factor"][7] = -1  # factor 4 is no longer listed by the culling
    o = run(old, cull, ns, vis)
    assert o["f_src"].tolist() == [2, 3, 5]


def test_new_observations_skip_the_reference_node_and_unknown_points():
    old, cull, ns, vis = window()
    xy, v = np.float32([330.0, 250.0]), (1.0, 2.0)
    vis["obs"] = [(3, 3, xy, v), (1, 0, xy, v), (-1, 3, xy, v), (2, 1, xy, v)]  # landmark 1's reference node is next node 0
    o = run(old, cull, ns, vis)
    assert o["f_src"].tolist() == [2, 3, 4, -1, 5, -1]
    assert o["f_obs"][[3, 5]].tolist() == [1, 3]
    row = o["f_const"][-1]
    assert row[0] == 5 and row[3:6].tolist() == [10 / 400, 10 / 400, 1.0] and row[9:12].tolist() == [1.0, 2.0, 0.0]
    assert row[12] == 0.5 and row[13] == 0.03


def test_two_new_keyframes_and_new_map_points():
    old, cull, ns, vis = window()
    xy, v = np.float32([320.0, 240.0]), (0.0, 0.0)
    vis["obs"] = [(2, 3, xy, v), (2, 1, xy, v)]
    vis["frames"] = {7: 1, 9: 3}
    vis["new"] = [dict(depth=4.0, ref_xy=xy, vel_ref=(1, 1), ref_id=7, cur_xy=xy, vel_cur=(2, 2)),
                  dict(depth=5.0, ref_xy=xy, vel_ref=(1, 1), ref_id=9, cur_xy=xy, vel_cur=(2, 2))]
    o = run(old, cull, ns, vis)
    assert o["L"] == 5 and o["invdepth"][3:].tolist() == [0.25, 0.2]
    # landmark 2 observed in both new keyframes, in node order; the second new point is anchored in the current node: no factor
    assert o["f_lm"].tolist() == [0, 0, 1, 1, 1, 2, 3] and o["f_obs"].tolist() == [1, 2, 2, 1, 3, 2, 3]
    with pytest.raises(ValueError, match="frame table"):
        vis["new"][0]["ref_id"] = 8
        run(old, cull, ns, vis)


def test_duplicate_observation_is_rejected():
    old, cull, ns, vis = window()
    xy, v = np.float32([320.0, 240.0]), (0.0, 0.0)
    vis["obs"] = [(1, 3, xy, v), (1, 3, xy, v)]
    with pytest.raises(ValueError, match="two observations"):
        run(old, cull, ns, vis)


def test_empty_window():
    old = dict(K=2, L=0, F=0, invdepth=np.zeros(0), f_lm=np.zeros(0, np.int32), f_ref=np.zeros(0, np.int32), f_obs=np.zeros(0, np.int32),
               f_const=np.zeros(0))
    cull = dict(lm_ref_node=np.zeros(0, np.int32), obs_off=np.zeros(1, np.int32), obs_factor=np.zeros(0, np.int32), lm_outlier=np.zeros(0, np.uint8),
                obs_outlier=np.zeros(0, np.uint8))
    vis = dict(num_marg=1, node_in_map=np.ones(2, np.uint8), node_td=np.zeros(2), cur_node=1, frames={}, obs=[], new=[])
    o = so.build(old, cull, [1, -1], vis, CAM)
    assert o["L"] == 0 and o["F"] == 0


def test_observation_in_a_node_the_slide_removes():
    old, cull, ns, vis = window()
    ns = [1, 3, -1]  # node 2 leaves the window although it is still flagged in the map
    vis["node_td"] = vis["node_td"][:3]
    vis["cur_node"] = 2
    o = run(old, cull, ns, vis)
    assert o["lm_src"].tolist() == [1, 2] and o["f_src"].tolist() == [3, 4]


def test_factorless_landmark_takes_a_new_observation_through_its_resident_row():
    old, cull, ns, vis = window()
    cull["obs_outlier"][7] = 1  # landmark 2's only factor is culled: it stays in the window without factors
    xy, v = np.float32([320.0, 240.0]), (0.0, 0.0)
    old["lm_ref"] = so.reference_rows(old)
    o = run(old, cull, ns, dict(vis, obs=[(2, 3, xy, v)]))
    assert o["f_src"].tolist() == [2, 3, -1, 5] and o["f_const"][2][0] == 4  # pts0 from the row the landmark kept
    old["lm_ref"][2] = np.nan  # unknown row: rejected
    with pytest.raises(ValueError, match="reference row"):
        run(old, cull, ns, dict(vis, obs=[(2, 3, xy, v)]))
