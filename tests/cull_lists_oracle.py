"""numpy restatement of the next culling's observation lists that icg_ba_slide_vision_resident builds on the device (the list rule of
icg_ba_update_and_cull_built, include/icgvins_b200.h), and of the reference's object graph those lists summarise: MapPoint::observations_
appended at tracking.cc:437 (a tracked frame), :771 and :778 (a new point's current, then reference frame), feature outlier flags set by the
culling's walk (IG/ic_gvins.cc:1061-1091), Map::removeKeyFrame(frame, true / false) (tracking/map.cc:89-125) and the keyframes in the map."""
import numpy as np


def next_lists(prev, obs_outlier, onode, nxt, new_obs_xy, new_points, cur_node):
    """The list rule.  prev: the last culling's lists (lm_ref_node, lm_ref_kp, obs_off, obs_node, obs_kp, obs_factor) and obs_outlier its
    flags; onode: old node -> next node (-1: gone); nxt: the next window's lm_origin (old landmark, or -(j + 1) for new point j), f_src,
    f_lm, f_obs; new_obs_xy: {(old landmark, next node): undis_xy} of the new observations; new_points[j]: dict ref_node (next node), ref_xy,
    cur_xy.  Returns the next lists as the device writes them (n_obs included)."""
    fmap = {int(s): f for f, s in enumerate(nxt["f_src"]) if s >= 0}
    f_lm, f_src, f_obs = (np.asarray(nxt[k]) for k in ("f_lm", "f_src", "f_obs"))
    out = dict(lm_ref_node=[], lm_ref_kp=[], obs_off=[0], obs_node=[], obs_factor=[], obs_kp=[])

    def entry(node, f, xy):
        out["obs_node"].append(int(node)), out["obs_factor"].append(int(f)), out["obs_kp"].append(np.asarray(xy, np.float32))

    for li, org in enumerate(nxt["lm_origin"]):
        if org >= 0:
            r = int(prev["lm_ref_node"][org])
            out["lm_ref_node"].append(int(onode[r])), out["lm_ref_kp"].append(np.asarray(prev["lm_ref_kp"][org], np.float32))
            for o in range(prev["obs_off"][org], prev["obs_off"][org + 1]):
                f, k = int(prev["obs_factor"][o]), int(prev["obs_node"][o])
                if obs_outlier[o] or onode[k] < 0:
                    continue
                if f >= 0 and f in fmap:
                    entry(onode[k], fmap[f], prev["obs_kp"][o])
                elif f == -1 and k == r:
                    entry(onode[k], -1, prev["obs_kp"][o])
            for f in np.nonzero((f_lm == li) & (f_src < 0))[0]:  # the new observations, in node order as the factors are
                entry(f_obs[f], f, new_obs_xy[(int(org), int(f_obs[f]))])
        else:
            p = new_points[-org - 1]
            out["lm_ref_node"].append(int(p["ref_node"])), out["lm_ref_kp"].append(np.asarray(p["ref_xy"], np.float32))
            if p["ref_node"] != cur_node:
                entry(cur_node, int(np.nonzero(f_lm == li)[0][0]), p["cur_xy"])
            entry(p["ref_node"], -1, p["ref_xy"])
        out["obs_off"].append(len(out["obs_node"]))
    L = len(out["lm_ref_node"])
    return dict(n_obs=len(out["obs_node"]), lm_ref_node=np.array(out["lm_ref_node"], np.int32), obs_off=np.array(out["obs_off"], np.int32),
                obs_node=np.array(out["obs_node"], np.int32), obs_factor=np.array(out["obs_factor"], np.int32),
                lm_ref_kp=np.array(out["lm_ref_kp"], np.float32).reshape(L, 2), obs_kp=np.array(out["obs_kp"], np.float32).reshape(-1, 2))


class Graph:
    """The reference's map objects, as far as the culling's walk reads them."""

    def __init__(self):
        self.frames = {}  # frame id -> {"kf", "in_map"}
        self.points = {}  # point id -> {"ref", "ref_kp", "obs": [feature], "outlier"}

    def add_frame(self, fid):
        self.frames[fid] = dict(kf=True, in_map=True)

    def observe(self, pid, fid, kp):  # MapPoint::addObservation: observations_.push_back
        self.points[pid]["obs"].append(dict(frame=fid, kp=np.asarray(kp, np.float32), outlier=False, alive=True))

    def new_point(self, pid, ref, ref_kp, cur, cur_kp):  # tracking.cc:771, then :778
        self.points[pid] = dict(ref=ref, ref_kp=np.asarray(ref_kp, np.float32), obs=[], outlier=False)
        self.observe(pid, cur, cur_kp)
        self.observe(pid, ref, ref_kp)

    def remove_keyframe(self, fid, remove_points):  # Map::removeKeyFrame
        if remove_points:
            for p in self.points.values():
                if p["ref"] == fid and not p["outlier"]:
                    p["obs"] = []  # removeAllObservations
                    p["outlier"] = True
            for p in self.points.values():  # frame->clearFeatures(): the weak observations expire
                for f in p["obs"]:
                    if f["frame"] == fid:
                        f["alive"] = False
        self.frames[fid]["in_map"] = False

    def walk(self, pid):
        """the observations gvinsOutlierCulling visits (:1061-1069)"""
        return [f for f in self.points[pid]["obs"] if f["alive"] and not f["outlier"] and self.frames[f["frame"]]["kf"] and self.frames[f["frame"]]["in_map"]]
