"""numpy restatement of the next window's vision half: GVINS::addReprojectionParameters + addReprojectionFactors (IG/ic_gvins.cc:1697-1837) on
the map after the culling and Map::removeKeyFrame(frame, true) (tracking/map.cc:89-125), in the fixed order icg_ba_slide_vision_resident
documents (include/icgvins_b200.h).  The reference iterates an unordered_map; this order only permutes rows."""
import numpy as np

DEFAULT_INVDEPTH = 1.0 / 10.0  # 1 / MapPoint::DEFAULT_DEPTH


def pixel2cam(cam, xy):
    """Camera::pixel2cam (camera.cc:126-130) of a float32 keypoint, as (x, y, 1)"""
    u, v = float(np.float32(xy[0])), float(np.float32(xy[1]))
    y = (v - cam["cy"]) / cam["fy"]
    x = (u - cam["cx"] - cam.get("skew", 0.0) * y) / cam["fx"]
    return [x, y, 1.0]


def carried_invdepth(rho):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.float64(1.0) / (np.float64(1.0) / np.float64(rho))


def reference_rows(old):
    """the rows icg_ba_upload keeps: each landmark's first factor's pts0, vel0, td0, NaN for a landmark without factors"""
    rows = np.full((old["L"], 7), np.nan)
    fc = np.asarray(old["f_const"], np.float64).reshape(-1, 14)
    for f in range(old["F"] - 1, -1, -1):
        rows[old["f_lm"][f]] = np.r_[fc[f, 0:3], fc[f, 6:9], fc[f, 12]]
    return rows


def build(old, cull, node_src, vis, cam):
    """old: the window the handle holds (K, L, F, invdepth as the solve left it, f_lm, f_ref, f_obs, f_const); cull: lm_ref_node, obs_off,
    obs_factor, lm_outlier, obs_outlier; node_src: the slide's next node -> old node map; vis: num_marg, node_in_map, node_td, cur_node,
    frames ({frame id: next node}), obs (list of (old landmark or -1, next node, undis_xy, vel2)), new (list of dicts depth, ref_xy, vel_ref,
    ref_id, cur_xy, vel_cur).  old["lm_ref"] (L x 7) are the handle's reference rows (default: reference_rows(old), what an upload keeps).
    Returns the next window's L, F, lm_src, lm_origin, invdepth, f_lm, f_ref, f_obs, f_src, f_const (every row), lm_ref (its reference rows),
    nan_flags (old L + new points) and nan_dropped.  Raises ValueError where the call returns ICG_EINVAL."""
    oK, oL, oF = old["K"], old["L"], old["F"]
    f_lm, f_ref, f_obs = (np.asarray(old[k]) for k in ("f_lm", "f_ref", "f_obs"))
    fc = np.asarray(old["f_const"], np.float64).reshape(-1, 14)
    lref = old["lm_ref"] if old.get("lm_ref") is not None else reference_rows(old)
    onode = np.full(oK, -1)
    for j, i in enumerate(node_src):
        if vis["num_marg"] <= i < oK and vis["node_in_map"][i]:
            onode[i] = j
    # a factor survives only through an observation the culling listed and did not flag
    fkeep = np.zeros(oF, bool)
    for o, f in enumerate(cull["obs_factor"]):
        if f < -1 or f >= oF:
            raise ValueError("obs_factor names no factor of the old window")
        if f >= 0:
            fkeep[f] = cull["obs_outlier"][o] == 0
    ref = np.asarray(cull["lm_ref_node"])
    nan_dropped = 0
    nan_flags = np.zeros(oL + len(vis["new"]), np.uint8)
    keep = np.zeros(oL, bool)
    for l in range(oL):
        ok = cull["lm_outlier"][l] == 0 and 0 <= ref[l] < oK and onode[ref[l]] >= 0
        nan = np.isnan(carried_invdepth(old["invdepth"][l]))
        keep[l] = ok and not nan
        nan_flags[l] = ok and nan
        nan_dropped += ok and nan
    new_obs = {}  # landmark -> {node: (xy, vel)}
    for l, node, xy, vel in vis["obs"]:
        if not 0 <= node < len(vis["node_td"]):
            raise ValueError("a node is out of range")
        if l < -1 or l >= oL:
            raise ValueError("obs_lm is out of range")
        if l < 0 or not keep[l] or onode[ref[l]] == node:
            continue
        d = new_obs.setdefault(l, {})
        if node in d:
            raise ValueError("two observations of one landmark in one node")
        d[node] = (xy, vel)
    out = dict(lm_src=[], lm_origin=[], lm_ref=[], invdepth=[], f_lm=[], f_ref=[], f_obs=[], f_src=[], f_const=[])

    def factor(li, r, o, src, row):
        out["f_lm"].append(li), out["f_ref"].append(r), out["f_obs"].append(o), out["f_src"].append(src), out["f_const"].append(row)

    for l in range(oL):
        if not keep[l]:
            continue
        li = len(out["lm_src"])
        v = carried_invdepth(old["invdepth"][l])
        out["lm_src"].append(-1 if v == 0 else l)
        out["lm_origin"].append(l), out["lm_ref"].append(lref[l])
        out["invdepth"].append(DEFAULT_INVDEPTH if v == 0 else v)
        mine = np.nonzero(f_lm == l)[0]
        for f in mine:
            if fkeep[f] and onode[f_obs[f]] >= 0:
                factor(li, onode[ref[l]], onode[f_obs[f]], int(f), fc[f].copy())
        if l in new_obs:
            r0 = lref[l]
            if np.isnan(r0[0]):
                raise ValueError("a landmark whose reference row is unknown takes a new observation")
            for node in sorted(new_obs[l]):
                xy, vel = new_obs[l][node]
                row = np.r_[r0[0:3], pixel2cam(cam, xy), r0[3:6], vel[0], vel[1], 0.0, r0[6], vis["node_td"][node]]
                factor(li, onode[ref[l]], node, -1, row)
    cur = vis["cur_node"]
    for j, p in enumerate(vis["new"]):
        if p["ref_id"] not in vis["frames"]:
            raise ValueError("a reference frame id is not in the frame table")
        r = vis["frames"][p["ref_id"]]
        with np.errstate(divide="ignore"):
            v = np.float64(1.0) / np.float64(p["depth"])
        if np.isnan(v):
            nan_dropped += 1
            nan_flags[oL + j] = 1
            continue
        li = len(out["lm_src"])
        out["lm_src"].append(-1)
        out["lm_origin"].append(-(j + 1))
        out["lm_ref"].append(np.r_[pixel2cam(cam, p["ref_xy"]), p["vel_ref"][0], p["vel_ref"][1], 0.0, vis["node_td"][r]])
        out["invdepth"].append(DEFAULT_INVDEPTH if v == 0 else v)
        if r != cur:
            row = np.r_[pixel2cam(cam, p["ref_xy"]), pixel2cam(cam, p["cur_xy"]), p["vel_ref"][0], p["vel_ref"][1], 0.0, p["vel_cur"][0], p["vel_cur"][1],
                        0.0, vis["node_td"][r], vis["node_td"][cur]]
            factor(li, r, cur, -1, row)
    res = dict(L=len(out["lm_src"]), F=len(out["f_src"]), nan_dropped=int(nan_dropped), nan_flags=nan_flags,
               lm_src=np.array(out["lm_src"], np.int32), lm_origin=np.array(out["lm_origin"], np.int32),
               lm_ref=np.array(out["lm_ref"], np.float64).reshape(-1, 7), invdepth=np.array(out["invdepth"], np.float64),
               f_lm=np.array(out["f_lm"], np.int32), f_ref=np.array(out["f_ref"], np.int32), f_obs=np.array(out["f_obs"], np.int32),
               f_src=np.array(out["f_src"], np.int32), f_const=np.array(out["f_const"], np.float64).reshape(-1, 14))
    return res
