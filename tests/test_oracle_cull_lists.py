"""The list rule of icg_ba_update_and_cull_built against the reference's object graph (tests/cull_lists_oracle.py): over seeded sequences of
keyframes -- culling flags, the marginalized keyframe's removeKeyFrame(frame, true), a second-new keyframe's removeKeyFrame(frame, false),
tracked observations and new map points -- the walk gvinsOutlierCulling makes at every keyframe equals the rule applied to the previous
keyframe's lists, entry for entry."""
import numpy as np
import pytest

from tests.cull_lists_oracle import Graph, next_lists


def lists_of(g, nodes, lms, factors):
    """the culling's lists of a window as the host gathers them from the graph (:1058-1069)"""
    node_of = {fid: k for k, fid in enumerate(nodes)}
    fidx = {pf: f for f, pf in enumerate(factors)}
    out = dict(lm_ref_node=[], lm_ref_kp=[], obs_off=[0], obs_node=[], obs_factor=[], obs_kp=[])
    for pid in lms:
        p = g.points[pid]
        out["lm_ref_node"].append(node_of[p["ref"]]), out["lm_ref_kp"].append(p["ref_kp"])
        for ft in g.walk(pid):
            out["obs_node"].append(node_of[ft["frame"]]), out["obs_kp"].append(ft["kp"])
            out["obs_factor"].append(-1 if ft["frame"] == p["ref"] else fidx[(pid, ft["frame"])])
        out["obs_off"].append(len(out["obs_node"]))
    return dict(n_obs=len(out["obs_node"]), lm_ref_node=np.array(out["lm_ref_node"], np.int32), obs_off=np.array(out["obs_off"], np.int32),
                obs_node=np.array(out["obs_node"], np.int32), obs_factor=np.array(out["obs_factor"], np.int32),
                lm_ref_kp=np.array(out["lm_ref_kp"], np.float32).reshape(-1, 2), obs_kp=np.array(out["obs_kp"], np.float32).reshape(-1, 2))


def window_factors(g, lms):
    """addReprojectionFactors on a window built from the graph: every walked observation outside the reference frame"""
    return [(pid, ft["frame"]) for pid in lms for ft in g.walk(pid) if ft["frame"] != g.points[pid]["ref"]]


def run(seed, n_kf=8, K=7, n_pts=60, p_flag=0.12, p_drop=0.05):
    rng = np.random.default_rng(seed)
    kp = lambda: rng.uniform([0, 0], [1280, 720]).astype(np.float32)
    g = Graph()
    nodes = list(range(K))
    for fid in nodes:
        g.add_frame(fid)
    next_fid, next_pid = K, 0
    for _ in range(n_pts):
        r = int(rng.integers(0, K - 1))
        g.new_point(next_pid, nodes[r], kp(), nodes[r + 1], kp())
        for k in range(r + 2, K):
            if rng.random() < 0.6:
                g.observe(next_pid, nodes[k], kp())
        next_pid += 1
    lms = list(range(n_pts))
    factors = window_factors(g, lms)
    lists = lists_of(g, nodes, lms, factors)
    stops = 0
    for _ in range(n_kf):
        # the culling: its walk flags features; a flagged reference observation makes the landmark an outlier and stops the walk
        flags = np.zeros(lists["n_obs"], np.uint8)
        for li, pid in enumerate(lms):
            p, walked = g.points[pid], g.walk(pid)
            o0 = lists["obs_off"][li]
            out = False
            for i, ft in enumerate(walked):
                if rng.random() < p_flag:
                    ft["outlier"] = True
                    flags[o0 + i] = 1
                    if ft["frame"] == p["ref"]:
                        out = True
                        stops += i + 1 < len(walked)
                        break
            if out or rng.random() < p_drop:
                p["outlier"] = True
        fkeep = np.zeros(len(factors), bool)
        for o, f in enumerate(lists["obs_factor"]):
            if f >= 0:
                fkeep[f] = flags[o] == 0
        # gvinsRemoveAllSecondNewFrame, then the marginalization's removeKeyFrame(frame, true)
        if len(nodes) >= K and rng.random() < 0.5:
            g.remove_keyframe(nodes[int(rng.integers(1, len(nodes) - 1))], False)
        g.remove_keyframe(nodes[0], True)
        kept = [fid for fid in nodes if g.frames[fid]["in_map"]]
        onode = np.array([kept.index(fid) if fid in kept else -1 for fid in nodes])
        cur = next_fid
        next_fid += 1
        g.add_frame(cur)
        nxt_nodes = kept + [cur]
        cur_node = len(kept)
        # the next window: carried landmarks with their surviving factors and new observations, then the new map points
        carried = [li for li, pid in enumerate(lms) if not g.points[pid]["outlier"] and g.frames[g.points[pid]["ref"]]["in_map"]]
        new_obs_xy = {}
        for li in carried:
            if rng.random() < 0.5:
                xy = kp()
                g.observe(lms[li], cur, xy)  # tracking.cc:437
                new_obs_xy[(li, cur_node)] = xy
        new_points = []
        for j in range(int(rng.integers(2, 7))):
            r = int(rng.integers(0, len(kept)))
            ref_xy, cur_xy = kp(), kp()
            g.new_point(next_pid, kept[r], ref_xy, cur, cur_xy)
            new_points.append(dict(pid=next_pid, ref_node=r, ref_xy=ref_xy, cur_xy=cur_xy))
            next_pid += 1
        nxt = dict(lm_origin=[], f_src=[], f_lm=[], f_obs=[])
        nfac = []
        for li in carried:
            lnew = len(nxt["lm_origin"])
            nxt["lm_origin"].append(li)
            for f, (pid, fr) in enumerate(factors):
                if pid == lms[li] and fkeep[f] and g.frames[fr]["in_map"]:
                    nxt["f_src"].append(f), nxt["f_lm"].append(lnew), nxt["f_obs"].append(kept.index(fr)), nfac.append((pid, fr))
            if (li, cur_node) in new_obs_xy:
                nxt["f_src"].append(-1), nxt["f_lm"].append(lnew), nxt["f_obs"].append(cur_node), nfac.append((lms[li], cur))
        for j, p in enumerate(new_points):
            lnew = len(nxt["lm_origin"])
            nxt["lm_origin"].append(-(j + 1))
            nxt["f_src"].append(-1), nxt["f_lm"].append(lnew), nxt["f_obs"].append(cur_node), nfac.append((p["pid"], cur))
        built = next_lists(lists, flags, onode, nxt, new_obs_xy, new_points, cur_node)
        nlms = [lms[li] for li in carried] + [p["pid"] for p in new_points]
        assert nfac == window_factors(g, nlms)  # the next window's factors are addReprojectionFactors' on the graph
        walked = lists_of(g, nxt_nodes, nlms, nfac)
        for k in ("n_obs", "lm_ref_node", "obs_off", "obs_node", "obs_factor"):
            assert np.array_equal(built[k], walked[k]), k
        for k in ("lm_ref_kp", "obs_kp"):
            assert built[k].tobytes() == walked[k].tobytes(), k
        assert built["n_obs"] == len(nlms) + len(nfac)
        lists, lms, factors, nodes = built, nlms, nfac, nxt_nodes
    return stops


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5])
def test_walk_equals_the_rule_at_every_keyframe(seed):
    run(seed)


def test_observations_after_a_reason_1_stop():
    """a flagged reference observation stops the walk before later entries: those stay listed (flag 0) and the landmark goes"""
    assert sum(run(s, p_flag=0.3) for s in range(10, 14)) > 0


def test_rule_on_a_hand_built_window():
    """two landmarks, one reference-node flag, a factor the slide drops, a new observation and a new point with and without a factor"""
    prev = dict(lm_ref_node=np.array([0, 1], np.int32), lm_ref_kp=np.array([[1, 2], [3, 4]], np.float32), obs_off=np.array([0, 3, 5], np.int32),
                obs_node=np.array([1, 0, 2, 1, 2], np.int32), obs_factor=np.array([0, -1, 1, -1, 2], np.int32),
                obs_kp=np.arange(10, dtype=np.float32).reshape(5, 2))
    flags = np.array([0, 0, 1, 0, 0], np.uint8)
    onode = np.array([0, 1, 2])
    nxt = dict(lm_origin=[0, 1, -1, -2], f_src=[0, 2, -1, -1], f_lm=[0, 1, 1, 2], f_obs=[1, 2, 3, 3])
    pts = [dict(ref_node=1, ref_xy=[5, 6], cur_xy=[7, 8]), dict(ref_node=3, ref_xy=[9, 10], cur_xy=[11, 12])]
    r = next_lists(prev, flags, onode, nxt, {(1, 3): [20, 21]}, pts, 3)
    assert r["obs_off"].tolist() == [0, 2, 5, 7, 8] and r["n_obs"] == 8
    assert r["obs_node"].tolist() == [1, 0, 1, 2, 3, 3, 1, 3]
    assert r["obs_factor"].tolist() == [0, -1, -1, 1, 2, 3, -1, -1]
    assert r["lm_ref_node"].tolist() == [0, 1, 1, 3]
