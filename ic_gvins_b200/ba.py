"""Host-side mirror of the reference's window-solve seam (IG/ic_gvins.cc:1130-1239): `WindowSolver` plays the role of
`ceres::Problem` + `ceres::Solver::Solve`, `gvins_optimization()` restates the two-pass protocol of
GVINS::gvinsOptimization (solve N/4 -> chi-square culling -> solve N - N/4).  All arithmetic runs in libicgvins_b200.so.
"""
from __future__ import annotations

import copy
import ctypes as C

import numpy as np

from ._lib import (BaPrior, BaProblem, BaSummary, CullLists, CullWindow, InsCut, Linearization, ReintWindow, SlideIns, SlideIntegrate, SlideVision, Structure,
                   SlideWindow, check, f32p, f64p, i8p, i32p, i64p, lib, u8p, vp)
from .camera import CameraStruct

IMU_BLOB = 480

_CULL_IN = dict(lm_ref_node=(np.int32, i32p), lm_ref_kp=(np.float32, f32p), obs_off=(np.int32, i32p), obs_node=(np.int32, i32p),
                obs_kp=(np.float32, f32p), obs_factor=(np.int32, i32p))


def _cull_ext(s: CullWindow, ci: dict) -> None:
    """The extrinsic inputs of one icg_ba_cull_window from those of `ci` (R_bc, t_bc; td_bc, estimate_ext, estimate_td default 0, 1, 1)."""
    for k in ("R_bc", "t_bc"):
        getattr(s, k)[:] = [float(x) for x in np.asarray(ci[k], np.float64).reshape(-1)]
    s.td_bc, s.estimate_ext, s.estimate_td = float(ci.get("td_bc", 0.0)), int(ci.get("estimate_ext", 1)), int(ci.get("estimate_td", 1))


def _cull_outputs(s: CullWindow, ci: dict, K: int, L: int, n_obs: int) -> None:
    """Add the culling's output arrays to `ci` and point `s` at them."""
    ci.update(cam_pose=np.zeros((K, 12)), lm_pw=np.zeros((L, 3)), lm_depth=np.zeros(L), lm_outlier=np.zeros(L, np.uint8), obs_outlier=np.zeros(n_obs, np.uint8))
    s.cam_pose, s.lm_pw, s.lm_depth = (ci[k].ctypes.data_as(f64p) for k in ("cam_pose", "lm_pw", "lm_depth"))
    s.lm_outlier, s.obs_outlier = ci["lm_outlier"].ctypes.data_as(u8p), ci["obs_outlier"].ctypes.data_as(u8p)


def cull_struct(prob: dict, ci: dict) -> CullWindow:
    """The icg_ba_cull_window of one window over the arrays of `ci` (made contiguous in place; output arrays are added to it)."""
    s = CullWindow()
    L = int(prob["L"])
    _cull_ext(s, ci)
    for k, (dt, pt) in _CULL_IN.items():
        if ci.get(k) is None:
            continue
        a = np.ascontiguousarray(ci[k], dtype=dt)
        ci[k] = a
        setattr(s, k, a.ctypes.data_as(pt) if a.size else pt())
    n_obs = int(ci["obs_off"][L]) if L > 0 and ci.get("obs_off") is not None else len(ci.get("obs_outlier", ()))
    _cull_outputs(s, ci, int(prob["K"]), L, n_obs)
    return s


_ARR = dict(pose=np.float64, mix=np.float64, ext=np.float64, invdepth=np.float64, f_lm=np.int32, f_ref=np.int32, f_obs=np.int32,
            f_const=np.float64, f_active=np.uint8, imu_blob=np.float64, pose_prior=np.float64, pose_prior_std=np.float64,
            mix_prior=np.float64, mix_prior_std=np.float64, gnss_node=np.int32, gnss_blh=np.float64, gnss_std=np.float64,
            marg_block_type=np.int32, marg_block_node=np.int32, marg_x0=np.float64, marg_J0=np.float64, marg_e0=np.float64)
_PTR = {np.float64: f64p, np.int32: i32p, np.uint8: u8p}
_SCAL = ["K", "L", "F", "ext_const", "td_const", "reproj_std", "reproj_huber", "n_imu", "has_imu_error", "has_pose_prior",
         "has_mix_prior", "n_gnss", "gnss_huber", "marg_r", "marg_nblocks"]


def to_struct(prob: dict) -> BaProblem:
    """Build the C struct over the dict's numpy arrays IN PLACE (arrays are made contiguous inside the dict so that the
    solve's in/out parameter updates are visible to the caller)."""
    s = BaProblem()
    for k, dt in _ARR.items():
        a = np.ascontiguousarray(prob[k], dtype=dt)
        prob[k] = a
        ptr_t = _PTR[dt]
        setattr(s, k, a.ctypes.data_as(ptr_t) if a.size else ptr_t())
    for k in _SCAL:
        setattr(s, k, prob[k])
    for i in range(3):
        s.lever[i] = float(prob["lever"][i])
    return s


def shard_window(prob: dict, rank: int, world: int) -> dict:
    """Landmark shard `rank` of `world` of one window problem (SURVEY.md 8e): block partition of the landmarks, each landmark keeps
    all of its reprojection factors (the per-landmark loop at IG/ic_gvins.cc:1777-1834); the camera-side problem is replicated.
    Returns a new dict whose `invdepth`, `f_*` arrays are the local slices (landmark indices remapped) plus `lm_lo`, `lm_hi`
    (global landmark range) and `f_index` (global factor indices) for merging results back."""
    L, F = prob["L"], prob["F"]
    lo, hi = (L * rank) // world, (L * (rank + 1)) // world
    f_lm = np.asarray(prob["f_lm"])
    sel = np.nonzero((f_lm >= lo) & (f_lm < hi))[0]
    out = dict(prob)
    out.update(L=hi - lo, F=len(sel), invdepth=np.array(prob["invdepth"][lo:hi], np.float64),
               f_lm=(f_lm[sel] - lo).astype(np.int32), f_ref=np.asarray(prob["f_ref"])[sel].astype(np.int32),
               f_obs=np.asarray(prob["f_obs"])[sel].astype(np.int32),
               f_const=np.asarray(prob["f_const"], np.float64).reshape(-1, 14)[sel].reshape(-1).copy(),
               f_active=np.asarray(prob["f_active"], np.uint8)[sel].copy(), lm_lo=lo, lm_hi=hi, f_index=sel)
    for k in ("pose", "mix", "ext", "gnss_std"):
        out[k] = np.array(prob[k], copy=True)
    return out


def merge_shard(prob: dict, shard: dict) -> None:
    """Write a solved shard's landmark results back into the full problem dict (camera-side blocks are identical on all shards)."""
    prob["invdepth"][shard["lm_lo"]:shard["lm_hi"]] = shard["invdepth"]
    prob["f_active"][shard["f_index"]] = shard["f_active"]
    for k in ("pose", "mix", "ext", "gnss_std"):
        prob[k][...] = shard[k]


def shard_cull_inputs(ci: dict, shard: dict) -> dict:
    """The culling inputs of one landmark shard (what each rank passes to update_and_cull on a sharded handle) from those of the whole
    window: the shard's landmarks and their observation lists, `obs_factor` renumbered to the shard's factors (-1 stays -1)."""
    lo, hi = shard["lm_lo"], shard["lm_hi"]
    off = np.asarray(ci["obs_off"], np.int32)
    o0, o1 = int(off[lo]), int(off[hi])
    out = dict(ci, lm_ref_node=np.array(ci["lm_ref_node"][lo:hi], np.int32), lm_ref_kp=np.array(ci["lm_ref_kp"][lo:hi], np.float32),
               obs_off=(off[lo:hi + 1] - o0).astype(np.int32), obs_node=np.array(ci["obs_node"][o0:o1], np.int32),
               obs_kp=np.array(ci["obs_kp"][o0:o1], np.float32))
    if ci.get("obs_factor") is not None:
        local = np.full(max(1, int(np.max(shard["f_index"], initial=-1)) + 1), -1, np.int32)
        local[shard["f_index"]] = np.arange(len(shard["f_index"]), dtype=np.int32)
        f = np.asarray(ci["obs_factor"][o0:o1], np.int32)
        out["obs_factor"] = np.where(f >= 0, local[np.clip(f, 0, len(local) - 1)], -1).astype(np.int32)
    return out


def shard_vision_inputs(vision: dict, shard: dict, cull_shard: dict) -> dict:
    """The vision inputs of one landmark shard (what each rank passes to shard_slide_vision) from those of the whole window: obs_lm remapped
    on the device to the shard's old rows (-1 outside [lm_lo, lm_hi)), obs_factor the shard's (shard_cull_inputs' output, `cull_shard`).
    Every other entry, the new map points included, is the whole window's.  Returns once the remap is done on torch's current stream (the
    handle reads it on its own)."""
    lo, hi = int(shard["lm_lo"]), int(shard["lm_hi"])
    out = dict(vision, obs_factor=cull_shard.get("obs_factor"))
    lm = vision.get("obs_lm")
    if lm is not None:
        import torch
        out["obs_lm"] = torch.where((lm >= lo) & (lm < hi), lm - lo, torch.full_like(lm, -1))
        torch.cuda.current_stream(lm.device).synchronize()
    return out


def merge_cull_shard(full: dict, shard: dict, shard_out: dict) -> None:
    """Write one shard's culling results (update_and_cull on a sharded handle) into the whole window's result dict `full`: lm_pw, lm_depth,
    lm_outlier over the shard's landmark range, obs_outlier over its observations.  Camera outputs and counts are the same on every rank."""
    lo, hi = shard["lm_lo"], shard["lm_hi"]
    off = full["obs_off"]
    for k in ("lm_pw", "lm_depth", "lm_outlier"):
        full[k][lo:hi] = shard_out[k]
    full["obs_outlier"][off[lo]:off[hi]] = shard_out["obs_outlier"]


def shard_next(nxt: dict, carry: dict, prev_shards, new_rank):
    """Per-rank shard slides from a whole-window slide.  nxt / carry: the next whole window and its whole-window carry maps (lm_src and f_src
    name rows of the old whole window); prev_shards: the old window's shards in rank order, with lm_lo / lm_hi / f_index as shard_window gives
    them; new_rank[l] (L entries): the rank of next landmark l where lm_src[l] < 0, -1 or the old rank where it is carried.  A carried
    landmark stays on the rank that held it (ValueError when new_rank names another).  Returns (the next whole window reordered
    rank-major -- each rank's landmarks contiguous, in next's order within the rank, factors landmark by landmark --, its carry maps,
    [(shard, shard-local carry)] per rank), each shard with lm_lo / lm_hi / f_index into the reordered window, so that shard_cull_inputs
    and merge_cull_shard keep working.  Every shard owns its arrays: a call that writes one rank's rows in place (reintegrate() writing
    imu_blob, a solve writing the parameters) changes no other rank's shard and not the returned whole window."""
    world = len(prev_shards)
    lm_src, f_src = np.asarray(carry["lm_src"]), np.asarray(carry["f_src"])
    L = int(nxt["L"])
    old_rank = np.full(max(1, max(int(s["lm_hi"]) for s in prev_shards)), -1, np.int64)
    for r, s in enumerate(prev_shards):
        old_rank[s["lm_lo"]:s["lm_hi"]] = r
    rank = np.asarray(new_rank, np.int64).copy() if L else np.zeros(0, np.int64)
    for l in np.nonzero(lm_src >= 0)[0]:
        r0 = int(old_rank[lm_src[l]])
        if int(new_rank[l]) not in (-1, r0):
            raise ValueError(f"landmark {l} is carried from rank {r0} but assigned to rank {int(new_rank[l])}")
        rank[l] = r0
    if ((rank < 0) | (rank >= world)).any():
        raise ValueError("every new landmark needs a rank in [0, world)")
    order = np.argsort(rank, kind="stable")  # rank-major, next's order within a rank
    new_of = np.empty(L, np.int64)
    new_of[order] = np.arange(L)
    f_lm = np.asarray(nxt["f_lm"], np.int64)
    fo = np.argsort(new_of[f_lm], kind="stable")  # factors landmark by landmark, next's order within a landmark
    whole = copy.deepcopy(nxt)
    whole.update(invdepth=np.asarray(nxt["invdepth"], np.float64)[order].copy(), f_lm=new_of[f_lm][fo].astype(np.int32),
                 f_ref=np.asarray(nxt["f_ref"])[fo].astype(np.int32), f_obs=np.asarray(nxt["f_obs"])[fo].astype(np.int32),
                 f_const=np.asarray(nxt["f_const"], np.float64).reshape(-1, 14)[fo].reshape(-1).copy(),
                 f_active=np.asarray(nxt["f_active"], np.uint8)[fo].copy())
    wcarry = dict(carry, lm_src=lm_src[order].astype(np.int32), f_src=f_src[fo].astype(np.int32))
    counts = np.bincount(rank, minlength=world) if L else np.zeros(world, np.int64)
    out = []
    for r in range(world):
        lo = int(counts[:r].sum())
        hi = lo + int(counts[r])
        sel = np.nonzero((whole["f_lm"] >= lo) & (whole["f_lm"] < hi))[0]
        sh = {k: np.array(v, copy=True) if isinstance(v, np.ndarray) else copy.deepcopy(v) for k, v in whole.items()}
        sh.update(L=hi - lo, F=len(sel), invdepth=whole["invdepth"][lo:hi].copy(), f_lm=(whole["f_lm"][sel] - lo).astype(np.int32),
                  f_ref=whole["f_ref"][sel].copy(), f_obs=whole["f_obs"][sel].copy(),
                  f_const=whole["f_const"].reshape(-1, 14)[sel].reshape(-1).copy(), f_active=whole["f_active"][sel].copy(), lm_lo=lo, lm_hi=hi,
                  f_index=sel)
        old = prev_shards[r]
        old_f = np.full(max(1, int(np.max(old["f_index"], initial=-1)) + 1), -1, np.int64)
        old_f[old["f_index"]] = np.arange(len(old["f_index"]))
        lsrc = wcarry["lm_src"][lo:hi].astype(np.int64)
        fsrc = wcarry["f_src"][sel].astype(np.int64)
        fl = np.where(fsrc >= 0, old_f[np.clip(fsrc, 0, len(old_f) - 1)], -1)
        if ((fsrc >= 0) & (fl < 0)).any():
            raise ValueError(f"rank {r}: a carried factor is not in the old shard of its landmark")
        sc = dict(carry, lm_src=np.where(lsrc >= 0, lsrc - int(old["lm_lo"]), -1).astype(np.int32), f_src=fl.astype(np.int32))
        out.append((sh, sc))
    return whole, wcarry, out


def connect_shards(solver: "WindowSolver", rank: int, world: int, transport: str, dist) -> None:
    """Join `solver` to the landmark-shard group of `world` processes (one per GPU) over peer memory (transport "p2p": each rank stores
    its reduction operand into the window owner's buffer over NVLink; the only transport).  `dist` is an initialised torch.distributed
    module (any backend): it only carries the rendezvous blobs, the CUDA IPC handles of the exchange buffers."""
    if transport != "p2p":
        raise ValueError(f"unknown landmark-shard transport {transport!r} (only 'p2p')")
    mine = solver.shard_export(rank, world)
    blobs = [None] * world
    dist.all_gather_object(blobs, mine)
    solver.shard_connect(blobs)
    dist.barrier()


def imu_preintegrate(state16, iewn, gravity, noise5, imu):
    """B3 host-side propagation in the product library (PreintegrationEarth::integrationProcess, preintegration_earth.cc:205-303)."""
    imu = np.ascontiguousarray(imu, np.float64)
    n = imu.shape[0]
    blob = np.zeros(IMU_BLOB)
    end = np.zeros(10)
    st, g, nz = (np.ascontiguousarray(x, np.float64) for x in (state16, gravity, noise5))
    iw = np.ascontiguousarray(iewn, np.float64) if iewn is not None else None  # None: PreintegrationNormal (iswithearth false)
    check(lib().icg_imu_preintegrate(vp(st.ctypes.data), vp(iw.ctypes.data) if iw is not None else None, vp(g.ctypes.data), vp(nz.ctypes.data),
                                     vp(imu.ctypes.data), n, vp(blob.ctypes.data), vp(end.ctypes.data)), "icg_imu_preintegrate")
    return blob, end


def _arg(keep: list, a, dtype, ptr):
    """`a` as a contiguous `dtype` array, cast to `ptr`.  The array goes into `keep`, which the caller holds until the C call returns."""
    a = np.ascontiguousarray(a, dtype)
    keep.append(a)
    return a.ctypes.data_as(ptr)


def _problems(problems):
    """The icg_ba_problem array over the problem dicts (to_struct: their arrays are made contiguous in place)."""
    return (BaProblem * len(problems))(*[to_struct(p) for p in problems])


def _summary(s: BaSummary) -> dict:
    return dict(iterations=s.iterations, num_successful_steps=s.num_successful_steps, termination=s.termination,
                initial_cost=s.initial_cost, final_cost=s.final_cost, final_radius=s.final_radius)


def _two_pass(summ, culled, n: int) -> list:
    """One gvinsOptimization result per window from the two summaries and two counts per window of icg_ba_gvins_optimization[_end]."""
    return [dict(pass1=_summary(summ[2 * w]), pass2=_summary(summ[2 * w + 1]), reproj_removed=culled[2 * w], gnss_reweighted=culled[2 * w + 1])
            for w in range(n)]


def _flags(flag, n: int) -> list:
    """Per-window 0 / 1 flags from one flag for all n windows or one per window."""
    return [1 if f else 0 for f in ([flag] * n if np.isscalar(flag) else flag)]


def _cam(camera) -> CameraStruct:
    """The icg_camera of a camera.Camera or CameraStruct."""
    return camera.c if hasattr(camera, "c") else camera


_CARRY = ("node_src", "lm_src", "f_src", "imu_src", "gnss_src")
_VISION_CARRY = ("node_src", "imu_src", "gnss_src")  # a vision slide builds lm_src / f_src itself


def _slide_carry(carry, n: int, prior_from_marg, keep: list, keys=_CARRY):
    """The icg_ba_slide_window array of n windows from their carry dicts: the maps of `keys` a dict holds (a missing or None map carries
    nothing of its kind) and the prior_from_marg flag (one, or one per window)."""
    cw = (SlideWindow * n)()
    for w, (c, f) in enumerate(zip(carry, _flags(prior_from_marg, n))):
        for k in keys:
            if c.get(k) is not None:
                setattr(cw[w], k, _arg(keep, c[k], np.int32, i32p))
        cw[w].prior_from_marg = f
    return cw


def _noise_station(noise5, station, keep: list):
    """The noise5 and station3 pointers of a reintegration or an integrating slide (noise5 None: zeros)."""
    return _arg(keep, np.zeros(5) if noise5 is None else noise5, np.float64, vp), _arg(keep, station, np.float64, vp)


def _imu_rows(rows, m: int):
    """The rows (n x 7) and offsets (m + 1) of m factors from one (k, 7) row array per factor, None for a factor without rows."""
    rows = [np.zeros((0, 7)) if r is None else np.asarray(r, np.float64).reshape(-1, 7) for r in rows]
    off = np.zeros(m + 1, np.int32)
    off[1:] = np.cumsum([len(r) for r in rows])
    return (np.concatenate(rows, axis=0) if rows else np.zeros((0, 7))), off


def _point_outputs(s, o: dict) -> None:
    """Point an icg_ba_slide_integrate or icg_ba_reint_window at the status, blobs and end_states arrays of `o`."""
    s.status, s.blob_out, s.end_state10 = o["status"].ctypes.data_as(i8p), o["blobs"].ctypes.data_as(f64p), o["end_states"].ctypes.data_as(f64p)


def _integ_struct(s, g, m, keep, with_rows=True):
    """fill one icg_ba_slide_integrate from an `integrate` dict of WindowSolver.slide_integrate (m = next n_imu; with_rows False: imu /
    imu_off stay NULL, the rows come from the device)"""
    if g.get("imu_from") is not None:
        s.imu_from = _arg(keep, g["imu_from"], np.int32, i32p)
        if not with_rows:
            pass
        elif "imu_off" in g:
            s.imu, s.imu_off = _arg(keep, g["imu"], np.float64, f64p), _arg(keep, g["imu_off"], np.int32, i32p)
        else:
            imu, off = _imu_rows(g["imu_rows"], m)
            s.imu, s.imu_off = _arg(keep, imu, np.float64, f64p), _arg(keep, off, np.int32, i32p)
        s.gravity3 = _arg(keep, np.broadcast_to(np.asarray(g["gravity"], np.float64), (m, 3)), np.float64, f64p)
        s.normal = _arg(keep, np.broadcast_to(np.asarray(g.get("normal", False), np.uint8), (m,)), np.uint8, u8p)
        if g.get("state16") is not None:
            s.state16 = _arg(keep, g["state16"], np.float64, f64p)
    if g.get("node_from_imu") is not None:
        s.node_from_imu = _arg(keep, g["node_from_imu"], np.uint8, u8p)
    if g.get("gnss_node") is not None:
        s.gnss_node, s.gnss_dt = _arg(keep, g["gnss_node"], np.int32, i32p), _arg(keep, g["gnss_dt"], np.float64, f64p)


def _integ_array(next_problems, integrate, keep: list):
    """The icg_ba_slide_integrate array of the `integrate` dicts (a None entry integrates nothing in its window)."""
    iw = (SlideIntegrate * len(next_problems))()
    for w, (p, g) in enumerate(zip(next_problems, integrate)):
        if g:
            _integ_struct(iw[w], g, int(p["n_imu"]), keep)
    return iw


def _dev(t):
    return None if t is None else vp(t.data_ptr() if hasattr(t, "data_ptr") else int(t))


_LEAN_ROWS = ("lm_src", "lm_origin", "f_src", "f_lm", "f_ref", "f_obs")


def _vision_struct(next_problems, vision, Lc: int, Fc: int, keep: list, rows: bool = True):
    """The icg_ba_slide_vision array of the `vision` dicts (WindowSolver.slide_vision) and the host rows the call builds into, sized to a
    handle of Lc landmarks and Fc factors (rows False: no invdepth / f_const, which the call then leaves on the device).  Empties the vision
    rows of next_problems, which the call does not read."""
    vw = (SlideVision * len(next_problems))()
    outs = []
    for w, (p, v) in enumerate(zip(next_problems, vision)):
        if rows:
            o = dict(lm_src=np.zeros(Lc, np.int32), lm_origin=np.zeros(Lc, np.int32), nan_flags=np.zeros(Lc + int(v.get("n_new", 0)), np.uint8), f_src=np.zeros(Fc, np.int32), f_lm=np.zeros(Fc, np.int32), f_ref=np.zeros(Fc, np.int32),
                     f_obs=np.zeros(Fc, np.int32), invdepth=np.zeros(Lc), f_const=np.zeros((Fc, 14)))
        else:
            o = {k: np.empty(Fc if k.startswith("f_") else Lc, np.int32) for k in _LEAN_ROWS}
            o["nan_flags"] = np.zeros(Lc + int(v.get("n_new", 0)), np.uint8)
        outs.append(o)
        p.update(L=0, F=0, invdepth=np.zeros(0), f_lm=np.zeros(0, np.int32), f_ref=np.zeros(0, np.int32), f_obs=np.zeros(0, np.int32),
                 f_const=np.zeros(0), f_active=np.zeros(0, np.uint8))
        s = vw[w]
        s.num_marg = int(v["num_marg"])
        s.node_in_map = _arg(keep, v["node_in_map"], np.uint8, u8p)
        if v.get("obs_factor") is not None and len(v["obs_factor"]):
            s.obs_factor = _arg(keep, v["obs_factor"], np.int32, i32p)
        cs = _cam(v["camera"])
        s.cam[:] = [float(getattr(cs, k)) for k, _ in CameraStruct._fields_]
        s.node_td = _arg(keep, v["node_td"], np.float64, f64p)
        s.cur_node = int(v["cur_node"])
        frames = v.get("frames", {})
        s.n_frames = len(frames)
        s.frame_id = _arg(keep, np.array(list(frames.keys()), np.int64), np.int64, i64p)
        s.frame_node = _arg(keep, np.array(list(frames.values()), np.int32), np.int32, i32p)
        s.n_obs, s.n_in = int(v.get("n_obs", 0)), int(v.get("n_in", 0))
        s.dev_n, s.obs_src, s.obs_lm, s.obs_node = (_dev(v.get(k)) for k in ("dev_n", "obs_src", "obs_lm", "obs_node"))
        s.obs_undis_xy, s.obs_vel = _dev(v.get("obs_undis_xy")), _dev(v.get("obs_vel"))
        s.n_new = int(v.get("n_new", 0))
        s.dev_new_n = _dev(v.get("dev_new_n"))
        s.new_depth, s.new_vel_ref, s.new_vel_cur = (_dev(v.get(k)) for k in ("new_depth", "new_vel_ref", "new_vel_cur"))
        s.new_ref_undis_xy, s.new_cur_undis_xy, s.new_ref_frame_id = (_dev(v.get(k)) for k in ("new_ref_undis_xy", "new_cur_undis_xy", "new_ref_frame_id"))
        s.lm_src, s.f_src, s.f_lm, s.f_ref, s.f_obs = (o[k].ctypes.data_as(i32p) for k in ("lm_src", "f_src", "f_lm", "f_ref", "f_obs"))
        if rows:
            s.invdepth, s.f_const = o["invdepth"].ctypes.data_as(f64p), o["f_const"].ctypes.data_as(f64p)
        s.lm_origin, s.nan_flags = o["lm_origin"].ctypes.data_as(i32p), o["nan_flags"].ctypes.data_as(u8p)
    return vw, outs


def _vision_results(next_problems, carry, vw, outs) -> list:
    """slide_vision()'s dicts from the rows a successful call built; writes the built window into next_problems and its lm_src / f_src
    into carry."""
    res = []
    for w, (p, c, o) in enumerate(zip(next_problems, carry, outs)):
        L, F = int(vw[w].L), int(vw[w].F)
        if "f_const" not in o:
            # rows=False: what the rest of the keyframe cycle reads on the host.  invdepth is the buffer a later download fills
            r = dict(L=L, F=F, nan_dropped=int(vw[w].nan_dropped), nan_flags=o["nan_flags"], **{k: o[k][:F if k.startswith("f_") else L] for k in _LEAN_ROWS})
            res.append(r)
            p.update(L=L, F=F, invdepth=np.zeros(L), f_lm=r["f_lm"], f_ref=r["f_ref"], f_obs=r["f_obs"], f_const=np.zeros(0), f_active=np.ones(F, np.uint8))
            c["lm_src"], c["f_src"] = r["lm_src"], r["f_src"]
            continue
        r = dict(L=L, F=F, nan_dropped=int(vw[w].nan_dropped), lm_src=o["lm_src"][:L].copy(), lm_origin=o["lm_origin"][:L].copy(),
                 nan_flags=o["nan_flags"], invdepth=o["invdepth"][:L].copy(),
                 f_src=o["f_src"][:F].copy(), f_lm=o["f_lm"][:F].copy(), f_ref=o["f_ref"][:F].copy(), f_obs=o["f_obs"][:F].copy(),
                 f_const=o["f_const"][:F].copy())
        res.append(r)
        fcn = r["f_const"].copy()
        fcn[r["f_src"] >= 0] = np.nan
        p.update(L=L, F=F, invdepth=r["invdepth"].copy(), f_lm=r["f_lm"].copy(), f_ref=r["f_ref"].copy(), f_obs=r["f_obs"].copy(),
                 f_const=fcn.reshape(-1), f_active=np.ones(F, np.uint8))
        c["lm_src"], c["f_src"] = r["lm_src"].copy(), r["f_src"].copy()
    return res


class WindowSolver:
    """Batched sliding-window solver handle (one per optimization thread / GPU)."""

    def __init__(self, max_windows=1, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=160, device=0, stream=None):
        self._h = vp()
        self.max_L, self.max_F, self.max_K = max_L, max_F, max_K
        check(lib().icg_ba_create(C.byref(self._h), max_windows, max_K, max_L, max_F, max_gnss, max_marg_r, device,
                                  vp(stream) if stream else None), "icg_ba_create")

    def close(self):
        if getattr(self, "_h", None):
            lib().icg_ba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def shard_export(self, rank: int, world: int) -> bytes:
        """Allocate this rank's peer-memory exchange buffer for a group of `world` ranks; returns the blob the other ranks need."""
        buf = (C.c_uint8 * 128)()
        check(lib().icg_ba_shard_export(self._h, rank, world, buf), "icg_ba_shard_export")
        return bytes(buf)

    def shard_connect(self, blobs) -> None:
        """blobs: the `world` export blobs in rank order."""
        raw = b"".join(blobs)
        buf = (C.c_uint8 * len(raw)).from_buffer_copy(raw)
        check(lib().icg_ba_shard_connect(self._h, buf), "icg_ba_shard_connect")

    def shard_leave(self) -> None:
        """Leave the landmark-shard group: the handle solves whole windows on its own GPU again, like a fresh handle of its capacities."""
        check(lib().icg_ba_shard_leave(self._h), "icg_ba_shard_leave")

    def solve(self, problems, max_num_iterations: int):
        """ceres::Solver::Solve on a list of problem dicts (updated in place).  Returns a list of summaries."""
        if isinstance(problems, dict):
            problems = [problems]
        n = len(problems)
        arr = _problems(problems)
        summ = (BaSummary * n)()
        check(lib().icg_ba_solve(self._h, n, arr, max_num_iterations, summ), "icg_ba_solve")
        return [_summary(s) for s in summ]

    def solve_structs(self, arr, n, max_num_iterations, summ):
        check(lib().icg_ba_solve(self._h, n, arr, max_num_iterations, summ), "icg_ba_solve")

    # -- device-resident stages
    def upload(self, problems):
        n = len(problems)
        self._keep = _problems(problems)
        self._n = n
        check(lib().icg_ba_upload(self._h, n, self._keep), "icg_ba_upload")

    def run(self, max_num_iterations: int, restart: bool = False):
        check(lib().icg_ba_run(self._h, max_num_iterations, 1 if restart else 0), "icg_ba_run")

    def download(self, write_back: bool = True):
        summ = (BaSummary * self._n)()
        check(lib().icg_ba_download(self._h, self._n, self._keep if write_back else None, summ), "icg_ba_download")
        return [_summary(s) for s in summ]

    def sync(self):
        check(lib().icg_ba_sync(self._h), "icg_ba_sync")

    def peek_linearization(self, w: int) -> dict:
        """Window w's system as the last linearisation and Schur complement left it (icg_ba_peek_linearization; a test read-out).  Mp: a
        dict (reference node, observing node) -> packed upper 20x20; A_W: (L, 6K + 8) by landmark id; Hs: (NCV, NCV) lower triangle."""
        K, L, F = self.max_K, max(1, self.max_L), max(1, self.max_F)
        NCV, N, PM = 6 * K + 7, 15 * K + 7, K * (K - 1)
        a = dict(pair_ro=np.zeros(PM, np.int32), Mp=np.zeros(PM * 210), A_W=np.zeros(L * (NCV + 1)), h_l=np.zeros(L), g_l=np.zeros(L),
                 H_c=np.zeros(N * N), g_c=np.zeros(N), costf=np.zeros(F), scale_l=np.zeros(L), Hs=np.zeros(NCV * NCV), visv=np.zeros(3 * NCV))
        s = Linearization()
        for name, arr in a.items():
            setattr(s, name, arr.ctypes.data_as(i32p if arr.dtype == np.int32 else f64p))
        check(lib().icg_ba_peek_linearization(self._h, w, C.byref(s)), "icg_ba_peek_linearization")
        K, L, F, P = s.K, s.L, s.F, s.n_pairs
        NCV, N = 6 * K + 7, 15 * K + 7
        ro, Mp = a["pair_ro"][:P], a["Mp"][:P * 210].reshape(P, 210)
        return dict(K=K, L=L, F=F, lin_buf=s.lin_buf, radius=s.radius, Mp={(int(v) >> 8, int(v) & 255): Mp[p].copy() for p, v in enumerate(ro)},
                    A_W=a["A_W"][:L * (NCV + 1)].reshape(L, NCV + 1), h_l=a["h_l"][:L], g_l=a["g_l"][:L], scale_l=a["scale_l"][:L],
                    H_c=a["H_c"][:N * N].reshape(N, N), g_c=a["g_c"][:N], costf=a["costf"][:F], Hs=a["Hs"][:NCV * NCV].reshape(NCV, NCV),
                    visv=a["visv"][:3 * NCV].reshape(3, NCV))

    def peek_structure(self, w: int) -> dict:
        """Window w's structure tables (icg_ba_peek_structure; a test read-out), in the window's sizes: lm_perm, lm_off, f_meta_s (F x 4),
        vb_lm0 (runs + 1), ref_nrun, part_off, pair_ro, vis_ord, npairs, f_active."""
        K, L, F = self.max_K, self.max_L, self.max_F
        PM = K * (K - 1)
        a = dict(lm_perm=np.zeros(L, np.int32), lm_off=np.zeros(L + 1, np.int32), f_meta_s=np.zeros(4 * F, np.int32), vb_lm0=np.zeros(L + F + 2, np.int32),
                 ref_nrun=np.zeros(K, np.int32), part_off=np.zeros(PM + 1, np.int32), pair_ro=np.zeros(PM, np.int32), vis_ord=np.zeros(F, np.int32),
                 f_active=np.zeros(F, np.uint8))
        s = Structure()
        for name, arr in a.items():
            setattr(s, name, arr.ctypes.data_as(u8p if arr.dtype == np.uint8 else i32p))
        check(lib().icg_ba_peek_structure(self._h, w, C.byref(s)), "icg_ba_peek_structure")
        L, F, R, P = s.L, s.F, s.n_runs, s.npairs
        return dict(lm_perm=a["lm_perm"][:L], lm_off=a["lm_off"][:L + 1], f_meta_s=a["f_meta_s"][:4 * F].reshape(F, 4), vb_lm0=a["vb_lm0"][:R + 1],
                    ref_nrun=a["ref_nrun"][:s.K], part_off=a["part_off"][:P + 1], pair_ro=a["pair_ro"][:P], vis_ord=a["vis_ord"][:F],
                    npairs=np.array([P]), f_active=a["f_active"][:F])

    def residual_costs(self, prob):
        s = to_struct(prob)
        rc = np.zeros(prob["F"])
        gc = np.zeros(prob["n_gnss"])
        check(lib().icg_ba_residual_costs(self._h, C.byref(s), vp(rc.ctypes.data), vp(gc.ctypes.data) if gc.size else None),
              "icg_ba_residual_costs")
        return rc, gc

    def gvins_optimization_batch(self, problems, num_iterations=20):
        """GVINS::gvinsOptimization on a list of windows in one device-resident call (icg_ba_gvins_optimization)."""
        n = len(problems)
        arr = _problems(problems)
        summ = (BaSummary * (2 * n))()
        culled = (C.c_int32 * (2 * n))()
        check(lib().icg_ba_gvins_optimization(self._h, n, arr, num_iterations, summ, culled), "icg_ba_gvins_optimization")
        return _two_pass(summ, culled, n)

    def run_gvins(self, num_iterations: int = 20, restart: bool = False):
        check(lib().icg_ba_run_gvins(self._h, num_iterations, 1 if restart else 0), "icg_ba_run_gvins")

    def gvins_optimization(self, prob, num_iterations=20):
        """GVINS::gvinsOptimization (IG/ic_gvins.cc:1130-1239): pass 1 (N/4 iterations, Huber on GNSS + reprojection),
        GNSS chi2 re-weighting (:1241-1267), reprojection chi2 removal (:1269-1297), pass 2 (N - N/4, GNSS without loss)."""
        first = num_iterations // 4
        second = num_iterations - first
        prob["gnss_huber"] = 1
        s1 = self.solve(prob, first)[0]
        rc, gc = self.residual_costs(prob)
        gnss_std = prob["gnss_std"].reshape(-1, 3)
        n_gnss_out = 0
        for g in range(prob["n_gnss"]):
            chi2 = 2.0 * gc[g]
            if chi2 > 7.815:
                gnss_std[g] *= np.sqrt(chi2 / 7.815)
                n_gnss_out += 1
        prob["gnss_std"] = gnss_std.reshape(-1)
        act = prob["f_active"]
        out = (2.0 * rc > 5.991) & (act != 0)
        act[out] = 0
        prob["gnss_huber"] = 0
        s2 = self.solve(prob, second)[0]
        return dict(pass1=s1, pass2=s2, reproj_removed=int(out.sum()), gnss_reweighted=n_gnss_out)

    def marginalize(self, problems, num_marg=1, want_schur=True, resident=False, culled=None, node_in_map=None):
        """MarginalizationInfo::marginalization as GVINS::gvinsMarginalization drives it (IG/ic_gvins.cc:1412-1640) on a list of
        windows: removes the `num_marg` oldest nodes + the landmarks anchored in them.  Returns one dict per window with the new
        prior in the layout the problem dict's marg_* entries use (node indices already shifted).  resident=True: the windows are the
        ones this handle has just solved (icg_ba_marginalize_resident: nothing is uploaded again).  culled (resident only): the list
        update_and_cull returned, with `obs_factor` in each dict; the factor set is then the map after the culling
        (icg_ba_marginalize_resident_culled), node_in_map[w] (K flags) naming the keyframes still in the map (all of them when None).
        Any handle marginalizes (cfg-4 windows included); a window whose marginalized or remained block exceeds 512 rows raises IcgError
        (ICG_EUNSUPPORTED) before anything runs.  To consume its own prior, a handle of max_K nodes needs max_marg_r >= 15 (max_K - 1) + 7.
        On a landmark-sharded handle (resident only) the call is collective: every rank passes its shard dicts (and, with culled=, its own
        update_and_cull results); window w's prior is returned on rank w mod world, the other ranks get m = r = 0 and empty arrays."""
        if isinstance(problems, dict):
            problems = [problems]
        call = self.marg_prepare(problems, num_marg, want_schur)
        if culled is None:
            self.marg_run(call, resident)
        else:
            if not resident:
                raise ValueError("culled= applies to the resident marginalization")
            if node_in_map is None:
                node_in_map = [np.ones(p["K"], np.uint8) for p in problems]
            nim = [np.ascontiguousarray(m, np.uint8) for m in node_in_map]
            keep = [dict(c) for c in culled]
            cw = (CullWindow * len(problems))(*[cull_struct(p, c) for p, c in zip(problems, keep)])
            for w, (c, k) in enumerate(zip(culled, keep)):  # the culling's flags, as that call returned them
                k["flags"] = [np.ascontiguousarray(c["lm_outlier"], np.uint8), np.ascontiguousarray(c["obs_outlier"], np.uint8)]
                cw[w].lm_outlier, cw[w].obs_outlier = (a.ctypes.data_as(u8p) for a in k["flags"])
            ptrs = (vp * len(nim))(*[vp(m.ctypes.data) for m in nim])
            check(lib().icg_ba_marginalize_resident_culled(self._h, call["n"], call["arr"], vp(call["nm"].ctypes.data), cw, ptrs, call["pri"]),
                  "icg_ba_marginalize_resident_culled")
        return self.marg_collect(call)

    def marginalize_built(self, problems, num_marg=1, node_in_map=None, want_schur=True):
        """marginalize(resident=True, culled=...) after update_and_cull_built(), with the factor set and the column map built on the device
        (icg_ba_marginalize_built): the problem dicts need their camera side only (f_lm, f_ref, f_obs, f_active and invdepth may be empty).
        node_in_map[w] (K flags) names the keyframes still in the map (all of them when None).  Returns marginalize()'s dicts, bit for bit the
        ones marginalize(resident=True, culled=...) returns on the same culling; single-GPU handles only."""
        if isinstance(problems, dict):
            problems = [problems]
        if node_in_map is None:
            node_in_map = [np.ones(p["K"], np.uint8) for p in problems]
        call = self.marg_prepare(problems, num_marg, want_schur)
        nim = [np.ascontiguousarray(m, np.uint8) for m in node_in_map]
        ptrs = (vp * len(nim))(*[vp(m.ctypes.data) for m in nim])
        check(lib().icg_ba_marginalize_built(self._h, call["n"], call["arr"], vp(call["nm"].ctypes.data), ptrs, call["pri"]), "icg_ba_marginalize_built")
        return self.marg_collect(call)

    def update_and_cull(self, problems, camera, std, cull_inputs):
        """updateParametersFromOptimizer + gvinsOutlierCulling (IG/ic_gvins.cc:1299-1389, 1035-1128) on the windows this handle has just
        solved (icg_ba_update_and_cull_resident).  camera: a camera.Camera or CameraStruct; std: reprojection_error_std_.  cull_inputs: one
        dict per window with R_bc (3x3), t_bc, td_bc, estimate_ext, estimate_td, lm_ref_node (L), lm_ref_kp (L x 2), obs_off (L + 1),
        obs_node, obs_kp (x 2) and optionally obs_factor.  Returns one dict per window: the inputs plus R_bc_out, t_bc_out, td_bc_out,
        ext_accepted, cam_pose (K x 12), lm_pw (L x 3), lm_depth, lm_outlier, obs_outlier and counts (5).  On a landmark-sharded handle every
        rank calls with its shard dicts and shard_cull_inputs(); the counts are the window's totals on every rank, the landmark outputs cover the
        shard (merge_cull_shard writes them into the whole window's)."""
        if isinstance(problems, dict):
            problems, cull_inputs = [problems], [cull_inputs]
        n = len(problems)
        arr = _problems(problems)
        outs = [dict(c) for c in cull_inputs]
        cw = (CullWindow * n)(*[cull_struct(p, c) for p, c in zip(problems, outs)])
        check(lib().icg_ba_update_and_cull_resident(self._h, n, arr, C.byref(_cam(camera)), float(std), cw), "icg_ba_update_and_cull_resident")
        for c, s in zip(outs, cw):
            c.update(R_bc_out=np.array(s.R_bc_out[:]).reshape(3, 3), t_bc_out=np.array(s.t_bc_out[:]), td_bc_out=s.td_bc_out, ext_accepted=s.ext_accepted,
                     counts=np.array(s.counts[:], np.int32))
        return outs

    def update_and_cull_built(self, problems, camera, std, ext_inputs):
        """update_and_cull() on the observation lists the last slide_vision() built on the device (icg_ba_update_and_cull_built): nothing
        but the extrinsic inputs goes up.  ext_inputs: one dict per window with R_bc (3x3), t_bc, td_bc, estimate_ext, estimate_td.  Returns
        update_and_cull()'s dicts with the list keys the culling walked filled in (lm_ref_node, lm_ref_kp, obs_off, obs_node, obs_kp,
        obs_factor, and n_obs), so that marginalize(culled=...) takes them unchanged; slide_vision() may then omit obs_factor, and
        marginalize(culled=...) takes dicts without the four integer lists (the culling's own are used)."""
        return self._cull_built("icg_ba_update_and_cull_built", problems, camera, std, ext_inputs)

    def shard_update_and_cull_built(self, problems, camera, std, ext_inputs):
        """update_and_cull_built() on a landmark-sharded handle (icg_ba_shard_update_and_cull_built), a collective call: every rank passes its
        shard dicts and the same ext_inputs, and culls on the lists its last shard_slide_vision() built.  Returns the rank's dicts as the sharded
        update_and_cull() does (landmark outputs over the shard, counts the window's totals) with the rank's shard-local lists, without
        obs_factor: marginalize(culled=...) and shard_vision_inputs() / shard_slide_vision() take them unchanged, and each rank's own culling
        supplies obs_factor.  A rejection on any rank raises IcgError on every rank, with every handle unchanged."""
        outs = self._cull_built("icg_ba_shard_update_and_cull_built", problems, camera, std, ext_inputs)
        for o in outs:
            o.pop("obs_factor")
        return outs

    def _cull_built(self, fn, problems, camera, std, ext_inputs):
        if isinstance(problems, dict):
            problems, ext_inputs = [problems], [ext_inputs]
        n = len(problems)
        arr = _problems(problems)
        outs, cw, cl = [], (CullWindow * n)(), (CullLists * n)()
        cap = self.max_L + self.max_F
        for w, (p, e) in enumerate(zip(problems, ext_inputs)):
            K, L = int(p["K"]), int(p["L"])
            o = {k: e[k] for k in ("R_bc", "t_bc", "td_bc", "estimate_ext", "estimate_td") if k in e}
            o.update(lm_ref_node=np.zeros(L, np.int32), obs_off=np.zeros(L + 1, np.int32), obs_node=np.zeros(cap, np.int32), obs_factor=np.zeros(cap, np.int32),
                     lm_ref_kp=np.zeros((L, 2), np.float32), obs_kp=np.zeros((cap, 2), np.float32))
            outs.append(o)
            _cull_ext(cw[w], e)
            _cull_outputs(cw[w], o, K, L, cap)
            for k in ("lm_ref_node", "obs_off", "obs_node", "obs_factor"):
                setattr(cl[w], k, o[k].ctypes.data_as(i32p))
            cl[w].lm_ref_kp, cl[w].obs_kp = o["lm_ref_kp"].ctypes.data_as(f32p), o["obs_kp"].ctypes.data_as(f32p)
        check(getattr(lib(), fn)(self._h, n, arr, C.byref(_cam(camera)), float(std), cw, cl), fn)
        for o, s, c in zip(outs, cw, cl):
            no = int(c.n_obs)
            for k in ("obs_node", "obs_factor", "obs_kp", "obs_outlier"):
                o[k] = o[k][:no].copy()
            o.update(n_obs=no, R_bc_out=np.array(s.R_bc_out[:]).reshape(3, 3), t_bc_out=np.array(s.t_bc_out[:]), td_bc_out=s.td_bc_out,
                     ext_accepted=s.ext_accepted, counts=np.array(s.counts[:], np.int32))
        return outs

    def reintegrate(self, problems, noise5, station, imu_rows, reintegrate=None):
        return self._reintegrate("icg_ba_reintegrate_resident", problems, noise5, station, imu_rows, reintegrate)

    def shard_reintegrate(self, problems, noise5, station, imu_rows, reintegrate=None):
        """reintegrate() on a landmark-sharded handle (icg_ba_shard_reintegrate_resident), a collective call: every rank passes its shard dicts
        and the same IMU rows, and every rank reintegrates the same factors, bit for bit."""
        return self._reintegrate("icg_ba_shard_reintegrate_resident", problems, noise5, station, imu_rows, reintegrate)

    def reintegrate_stored(self, problems, noise5, station=(0.0, 0.0, 0.0), reintegrate=None):
        """reintegrate() with every factor's rows from the handle's sample store (icg_ba_reintegrate_stored_resident): filled by
        imu_samples_from_ins() or slide_ins(), and not replaced by an upload or another slide since."""
        if isinstance(problems, dict):
            problems = [problems]
        return self._reintegrate("icg_ba_reintegrate_stored_resident", problems, noise5, station, [None] * len(problems), reintegrate, stored=True)

    def _reintegrate(self, fn, problems, noise5, station, imu_rows, reintegrate=None, stored=False):
        """GVINS::doReintegration (IG/ic_gvins.cc:1680-1695) on the windows this handle has just solved (icg_ba_reintegrate_resident).  noise5 =
        gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time; station = parameters_->station (the reference leaves it at (0, 0, 0));
        imu_rows[w] = the n_imu row arrays (m_k, 7) of window w's factors (None for a window left alone); reintegrate: per-window flags
        (None = all).  Returns one dict per window: status (n_imu int8: 1 reintegrated, 0 gate closed, -1 not positive definite), count,
        end_states (n_imu x 10, zero where the gate was closed) and blobs (n_imu x 480: the window's blobs with the reintegrated ones
        replaced).  The reintegrated blobs are written into problem["imu_blob"], as the reference mutates preintegrationlist_.  A factor with
        status -1 raises IcgError after the call; the exception's `results` holds the dicts."""
        if isinstance(problems, dict):
            problems, imu_rows = [problems], [imu_rows]
        n = len(problems)
        flags = _flags(True if reintegrate is None else reintegrate, n)
        arr = _problems(problems)
        io = (ReintWindow * n)()
        outs, keep = [], []
        for w, p in enumerate(problems):
            m = int(p["n_imu"])
            o = dict(status=np.zeros(m, np.int8), count=0, end_states=np.zeros((m, 10)),
                     blobs=np.array(np.asarray(p["imu_blob"], np.float64)[:m * IMU_BLOB].reshape(m, IMU_BLOB), copy=True))
            outs.append(o)
            io[w].reintegrate = flags[w] if m > 0 else 0
            _point_outputs(io[w], o)
            if io[w].reintegrate and not stored:
                imu, off = _imu_rows(imu_rows[w], m)
                io[w].imu, io[w].imu_off = _arg(keep, imu, np.float64, f64p), _arg(keep, off, np.int32, i32p)
        nz, stn = _noise_station(noise5, station, keep)
        rc = getattr(lib(), fn)(self._h, n, arr, nz, stn, io)
        for w, (p, o) in enumerate(zip(problems, outs)):
            o["count"] = int(io[w].count)
            if (o["status"] == 1).any():
                p["imu_blob"].reshape(-1, IMU_BLOB)[:len(o["status"])][o["status"] == 1] = o["blobs"][o["status"] == 1]
        check(rc, fn, outs)
        return outs

    def slide(self, next_problems, carry, prior_from_marg=True):
        self._slide("icg_ba_slide_resident", next_problems, carry, prior_from_marg)

    def shard_slide(self, next_problems, carry, prior_from_marg=True):
        """slide() on a landmark-sharded handle (icg_ba_shard_slide_resident), a collective call: every rank passes its next shards and their
        shard-local carry maps (shard_next builds both); window w's prior comes from the last sharded marginalization on its owner."""
        self._slide("icg_ba_shard_slide_resident", next_problems, carry, prior_from_marg)

    def _slide(self, fn, next_problems, carry, prior_from_marg=True):
        """The next keyframe's windows from the ones this handle holds (icg_ba_slide_resident): rows whose source is carried stay on the device,
        the rest are read from `next_problems` (dicts as upload() takes them; carried value rows may be stale).  carry: one dict per window
        with int32 arrays node_src (K), lm_src (L), f_src (F), imu_src (n_imu), gnss_src (n_gnss) -- old row or -1; a missing key carries
        nothing of that kind.  prior_from_marg (one flag, or one per window): the prior is the one the last resident marginalization left.
        Follow with run_gvins() and gvins_optimization_end(next_problems)."""
        n = len(next_problems)
        keep = []
        arr, cw = _problems(next_problems), _slide_carry(carry, n, prior_from_marg, keep)
        check(getattr(lib(), fn)(self._h, n, arr, cw), fn)
        self._keep, self._n = arr, n

    def slide_integrate(self, next_problems, carry, integrate, noise5, station=(0.0, 0.0, 0.0), prior_from_marg=True):
        return self._slide_integrate("icg_ba_slide_integrate_resident", next_problems, carry, integrate, noise5, station, prior_from_marg)

    def shard_slide_integrate(self, next_problems, carry, integrate, noise5, station=(0.0, 0.0, 0.0), prior_from_marg=True):
        """slide_integrate() on a landmark-sharded handle (icg_ba_shard_slide_integrate_resident), a collective call: as shard_slide, with the
        same `integrate` dicts on every rank; every rank integrates the same rows from its replicated states."""
        return self._slide_integrate("icg_ba_shard_slide_integrate_resident", next_problems, carry, integrate, noise5, station, prior_from_marg)

    def _slide_integrate(self, fn, next_problems, carry, integrate, noise5, station=(0.0, 0.0, 0.0), prior_from_marg=True):
        """slide() whose new IMU factors, new node rows and aligned GNSS fixes are computed on the device from the states this handle holds
        (icg_ba_slide_integrate_resident: the host halves of addNewTimeNode, removeUnusedTimeNode and insertNewGnssTimeNode, IG/ic_gvins.cc:754-928).
        Only rows that `carry` leaves to next_problems are read.  integrate: one dict per window (None: nothing integrated) with
          imu_from       n_imu int32: -1 next's blob, i >= 0 from old node i's state, SLIDE_CHAIN from the previous factor's end, SLIDE_ROW from state16
          imu_rows       n_imu entries: the (m, 7) rows (dt, dtheta, dvel) of an integrated factor, None otherwise
                         (or `imu` + `imu_off` as the C call takes them)
          gravity        3, or n_imu x 3;  normal: one flag or n_imu (PreintegrationNormal; default Earth);  state16: n_imu x 16 (SLIDE_ROW)
          node_from_imu  K flags: node j is the end state of integrated factor j - 1
          gnss_node, gnss_dt  n_gnss: old node whose velocity moves the fix by dt (-1: none)
        noise5 = gyr_arw, acc_vrw, gyr_bias_std, acc_bias_std, corr_time; station = parameters_->station.  Returns one dict per window: status
        (n_imu int8: 1 integrated, 0 not, -1 not positive definite), blobs (n_imu x 480) and end_states (n_imu x 10), zero where status is 0.
        A rejected call raises IcgError with the handle unchanged; after the integration its `results` holds the dicts."""
        n = len(next_problems)
        keep = []
        arr, cw = _problems(next_problems), _slide_carry(carry, n, prior_from_marg, keep)
        iw = _integ_array(next_problems, integrate, keep)
        outs = []
        for w, p in enumerate(next_problems):
            m = int(p["n_imu"])
            outs.append(dict(status=np.zeros(m, np.int8), blobs=np.zeros((m, IMU_BLOB)), end_states=np.zeros((m, 10))))
            _point_outputs(iw[w], outs[w])
        nz, stn = _noise_station(noise5, station, keep)
        check(getattr(lib(), fn)(self._h, n, arr, cw, iw, nz, stn), fn, outs)
        self._keep, self._n = arr, n
        return outs

    def imu_samples_from_ins(self, ins, streams, node_times) -> None:
        """Seeds the handle's IMU sample store (icg_ba_imu_samples_from_ins): factor k of resident window w gets getImuSeriesFromTo(
        node_times[w][k], node_times[w][k + 1]) cut from stream streams[w] of `ins` (an ins.InsWindow on this handle's device).  Call it right
        after the upload of windows whose INS windows still cover their spans."""
        n = len(streams)
        cut = (InsCut * n)()
        keep = []
        for w in range(n):
            cut[w].stream, cut[w].node_time = int(streams[w]), _arg(keep, node_times[w], np.float64, f64p)
        check(lib().icg_ba_imu_samples_from_ins(self._h, ins._h, n, cut), "icg_ba_imu_samples_from_ins")

    def imu_samples(self, w: int):
        """The stored rows of resident window w (icg_ba_imu_samples): a list with one (m, 7) array per IMU factor, None for a factor without
        samples."""
        # the call writes the window's n_imu + 1 offsets: room for the most a window of this handle holds, the rest left at a sentinel
        off = np.full(self.max_K + 1, np.iinfo(np.int32).min, np.int32)
        check(lib().icg_ba_imu_samples(self._h, int(w), 0, vp(off.ctypes.data), None), "icg_ba_imu_samples")
        m = int(np.nonzero(off != np.iinfo(np.int32).min)[0][-1])
        total = int(off[m])
        rows = np.zeros((total, 7))
        if total:
            check(lib().icg_ba_imu_samples(self._h, int(w), total, vp(off.ctypes.data), vp(rows.ctypes.data)), "icg_ba_imu_samples")
        out = []
        for k in range(m):
            if off[k] < 0:
                out.append(None)
                continue
            end = next((int(off[j]) for j in range(k + 1, m + 1) if off[j] >= 0), total)
            out.append(rows[off[k]:end].copy())
        return out

    def slide_ins(self, next_problems, carry, integrate, ins, streams, node_times, merge_src, noise5, station=(0.0, 0.0, 0.0), vision=None,
                  prior_from_marg=True):
        """slide_integrate() (vision given: slide_vision() with `integrate`) whose integrated factors' rows come from the device
        (icg_ba_slide_ins_resident): NODE / SLIDE_CHAIN factor k of window w is cut from stream streams[w] of `ins` over node_times[w][k] ..
        node_times[w][k + 1] (next K entries); a SLIDE_ROW factor k is old factors merge_src[w][k] and merge_src[w][k] + 1 of the sample store;
        carried factors keep their stored rows.  `integrate` dicts as slide_integrate takes them, without imu_rows / imu / imu_off.  Returns
        slide_integrate()'s dicts (vision: slide_vision()'s), each with n_rows (every new factor's stored rows, -1: none).  Status -2 marks a
        factor whose interval the INS window cannot serve (the call raises IcgError, the handle unchanged)."""
        fn = "icg_ba_slide_ins_resident"
        if vision is not None and integrate is not None and noise5 is None:
            raise ValueError(f"{fn}: integrate needs noise5")
        n = len(next_problems)
        keep = []
        vw, built = (None, None) if vision is None else _vision_struct(next_problems, vision, self.max_L, self.max_F, keep)
        arr = _problems(next_problems)
        cw = _slide_carry(carry, n, prior_from_marg, keep, _CARRY if vision is None else _VISION_CARRY)
        io = (SlideIns * n)()
        outs = []
        for w, p in enumerate(next_problems):
            m = int(p["n_imu"])
            outs.append(dict(status=np.zeros(m, np.int8), blobs=np.zeros((m, IMU_BLOB)), end_states=np.zeros((m, 10)), n_rows=np.full(m, -1, np.int32)))
            if integrate is not None and integrate[w]:
                _integ_struct(io[w].integ, integrate[w], m, keep, with_rows=False)
            _point_outputs(io[w].integ, outs[w])
            io[w].stream = int(streams[w])
            if node_times[w] is not None:
                io[w].node_time = _arg(keep, node_times[w], np.float64, f64p)
            if merge_src is not None and merge_src[w] is not None:
                io[w].merge_src = _arg(keep, merge_src[w], np.int32, i32p)
            io[w].n_rows = outs[w]["n_rows"].ctypes.data_as(i32p)
        nz, stn = _noise_station(noise5, station, keep)
        check(lib().icg_ba_slide_ins_resident(self._h, ins._h, n, arr, cw, io, nz, stn, vw), fn, outs)
        if vision is not None:
            outs = [dict(r, **o) for r, o in zip(_vision_results(next_problems, carry, vw, built), outs)]
        self._keep, self._n = arr, n
        return outs

    def slide_vision(self, next_problems, carry, vision, integrate=None, noise5=None, station=(0.0, 0.0, 0.0), prior_from_marg=True, rows=True):
        return self._slide_vision("icg_ba_slide_vision_resident", next_problems, carry, vision, integrate, noise5, station, prior_from_marg, rows)

    def shard_slide_vision(self, next_problems, carry, vision, integrate=None, noise5=None, station=(0.0, 0.0, 0.0), prior_from_marg=True,
                           rows=True):
        """slide_vision() on a landmark-sharded handle (icg_ba_shard_slide_vision_resident), a collective call: every rank passes its next shards
        (camera side as shard_slide takes it), their carry maps (node / IMU / GNSS) and its own vision dicts (shard_vision_inputs); new map
        point j of window w is built on rank (j + w) % world.  Returns the rank's shard as slide_vision does (lm_src / f_src shard-local,
        lm_origin: old shard-local landmark or -(j + 1) for global new point j, nan_flags: old shard L + every new point, set on its own rank)."""
        return self._slide_vision("icg_ba_shard_slide_vision_resident", next_problems, carry, vision, integrate, noise5, station, prior_from_marg, rows)

    def _slide_vision(self, fn, next_problems, carry, vision, integrate=None, noise5=None, station=(0.0, 0.0, 0.0), prior_from_marg=True, rows=True):
        """slide() (integrate given: slide_integrate()) whose vision rows are built on the device (icg_ba_slide_vision_resident):
        addReprojectionParameters + addReprojectionFactors on the culled window this handle holds plus the new keyframes' observations.  The
        last update_and_cull() of these windows must be current.  next_problems' L, F, invdepth, f_lm / f_ref / f_obs / f_const, f_active and
        carry's lm_src / f_src are not read; they are written into next_problems / carry (carried f_const rows as NaN, as slide() never reads
        them).  vision: one dict per window with
          num_marg, node_in_map (old K), obs_factor (the culling's), camera (camera.Camera or CameraStruct), node_td (next K), cur_node,
          frames ({frame id: next node}) for the new points' reference frames;
          tracked observations as DEVICE tensors (torch): obs_lm, obs_node (optional: cur_node), obs_undis_xy (float32 x 2), obs_vel (x 2),
            obs_src (optional, with n_in) and dev_n (optional int32 device count), n_obs (count, or the list's length with dev_n);
          new map points as DEVICE tensors: new_depth, new_ref_undis_xy, new_vel_ref, new_ref_frame_id (int64), new_cur_undis_xy,
            new_vel_cur, n_new and optionally dev_new_n.
        Returns one dict per window: L, F, nan_dropped, nan_flags (old L + n_new entries first: 1 where a landmark or new point was dropped
        for a NaN inverse depth), lm_origin (old landmark, or -(j + 1) for new point j), lm_src, f_src, f_lm, f_ref, f_obs, invdepth and f_const (the new factors' rows, f_src = -1;
        the others zero).  rows=False returns only what the rest of the keyframe cycle reads on the host (L, F, nan_dropped, nan_flags,
        lm_origin, lm_src, f_src, f_lm, f_ref, f_obs, sized to L and F): the inverse depths and factor constants stay on the device, and
        next_problems gets f_const empty and invdepth as a buffer for the next download.  A rejected call raises IcgError with the handle
        unchanged."""
        if integrate is not None and noise5 is None:
            raise ValueError(f"{fn}: integrate needs noise5")
        n = len(next_problems)
        keep = []
        vw, built = _vision_struct(next_problems, vision, self.max_L, self.max_F, keep, rows)
        arr, cw = _problems(next_problems), _slide_carry(carry, n, prior_from_marg, keep, _VISION_CARRY)
        iw, nz, stn = None, None, None
        if integrate is not None:
            iw = _integ_array(next_problems, integrate, keep)
            nz, stn = _noise_station(noise5, station, keep)
        check(getattr(lib(), fn)(self._h, n, arr, cw, iw, nz, stn, vw), fn)
        res = _vision_results(next_problems, carry, vw, built)
        self._keep, self._n = arr, n
        return res

    def gvins_optimization_end(self, problems):
        """icg_ba_gvins_optimization_end after run_gvins(): synchronises, writes the parameters, f_active and gnss_std back into the problem
        dicts and returns the two-pass results in the layout of gvins_optimization_batch."""
        n = len(problems)
        arr = _problems(problems)
        summ = (BaSummary * (2 * n))()
        culled = (C.c_int32 * (2 * n))()
        check(lib().icg_ba_gvins_optimization_end(self._h, n, arr, summ, culled), "icg_ba_gvins_optimization_end")
        return _two_pass(summ, culled, n)

    def marg_prepare(self, problems, num_marg=1, want_schur=True):
        """The argument block of one icg_ba_marginalize call (struct array over the problems' host arrays + caller-allocated output arrays):
        what a C++ caller keeps alive across keyframes.  marg_run issues the call, marg_collect turns the outputs into dicts."""
        n = len(problems)
        nm = np.full(n, num_marg, np.int32) if np.isscalar(num_marg) else np.ascontiguousarray(num_marg, np.int32)
        arr = _problems(problems)
        pri = (BaPrior * n)()
        bufs = []
        for w, p in enumerate(problems):
            rcap = 15 * p["K"] + 7
            b = dict(bt=np.zeros(2 * p["K"] + 2, np.int32), bn=np.zeros(2 * p["K"] + 2, np.int32), x0=np.zeros(16 * p["K"] + 8),
                     J0=np.zeros(rcap * rcap), e0=np.zeros(rcap))
            if want_schur:
                b.update(Hp=np.zeros(rcap * rcap), bp=np.zeros(rcap))
            bufs.append(b)
            pri[w].rcap = rcap
            pri[w].block_type, pri[w].block_node = b["bt"].ctypes.data_as(i32p), b["bn"].ctypes.data_as(i32p)
            pri[w].x0, pri[w].J0, pri[w].e0 = b["x0"].ctypes.data_as(f64p), b["J0"].ctypes.data_as(f64p), b["e0"].ctypes.data_as(f64p)
            if want_schur:
                pri[w].Hp, pri[w].bp = b["Hp"].ctypes.data_as(f64p), b["bp"].ctypes.data_as(f64p)
        return dict(n=n, nm=nm, arr=arr, pri=pri, bufs=bufs, want_schur=want_schur, problems=problems)

    def marg_run(self, call, resident=False):
        fn = lib().icg_ba_marginalize_resident if resident else lib().icg_ba_marginalize
        check(fn(self._h, call["n"], call["arr"], vp(call["nm"].ctypes.data), call["pri"]), "icg_ba_marginalize")

    def marg_collect(self, call):
        out = []
        gs = {0: 7, 1: 9, 2: 7, 3: 1}
        pri, want_schur = call["pri"], call["want_schur"]
        for w, b in enumerate(call["bufs"]):
            r, nb = pri[w].r, pri[w].nblocks
            nx = sum(gs[int(t)] for t in b["bt"][:nb])
            out.append(dict(m=pri[w].m, r=r, block_type=b["bt"][:nb].copy(), block_node=b["bn"][:nb].copy(), x0=b["x0"][:nx].copy(),
                            J0=b["J0"][:r * r].reshape(r, r).copy(), e0=b["e0"][:r].copy(),
                            Hp=b["Hp"][:r * r].reshape(r, r).copy() if want_schur else None, bp=b["bp"][:r].copy() if want_schur else None))
        return out

    # -- single-factor Evaluate (Ceres CostFunction contract), computed on the device
    def reproj_evaluate(self, pose0, pose1, ext, invdepth, td, const14, std, want_jac=True, frames=False):
        """frames=True: the node-frame form of ba_lin_vis / ba_cost (icg_ba_reproj_evaluate_frames)"""
        a = [np.ascontiguousarray(x, np.float64) for x in (pose0, pose1, ext, np.atleast_1d(invdepth), np.atleast_1d(td), const14)]
        r = np.zeros(2)
        Js = [np.zeros((2, 7)), np.zeros((2, 7)), np.zeros((2, 7)), np.zeros((2, 1)), np.zeros((2, 1))]
        jp = (vp * 5)(*[vp(j.ctypes.data) for j in Js])
        name = "icg_ba_reproj_evaluate_frames" if frames else "icg_ba_reproj_evaluate"
        check(getattr(lib(), name)(self._h, *[vp(x.ctypes.data) for x in a], float(std), vp(r.ctypes.data), jp if want_jac else None), name)
        return r, Js

    def gnss_evaluate(self, pose, blh, std3, lever):
        a = [np.ascontiguousarray(x, np.float64) for x in (pose, blh, std3, lever)]
        r, J = np.zeros(3), np.zeros((3, 7))
        jp = (vp * 1)(vp(J.ctypes.data))
        check(lib().icg_ba_gnss_evaluate(self._h, *[vp(x.ctypes.data) for x in a], vp(r.ctypes.data), jp), "icg_ba_gnss_evaluate")
        return r, J

    def pose_prior_evaluate(self, pose, prior7, std6):
        a = [np.ascontiguousarray(x, np.float64) for x in (pose, prior7, std6)]
        r, J = np.zeros(6), np.zeros((6, 7))
        jp = (vp * 1)(vp(J.ctypes.data))
        check(lib().icg_ba_pose_prior_evaluate(self._h, *[vp(x.ctypes.data) for x in a], vp(r.ctypes.data), jp), "icg_ba_pose_prior_evaluate")
        return r, J

    def mix_prior_evaluate(self, mix, prior9, std9):
        a = [np.ascontiguousarray(x, np.float64) for x in (mix, prior9, std9)]
        r, J = np.zeros(9), np.zeros((9, 9))
        jp = (vp * 1)(vp(J.ctypes.data))
        check(lib().icg_ba_mix_prior_evaluate(self._h, *[vp(x.ctypes.data) for x in a], vp(r.ctypes.data), jp), "icg_ba_mix_prior_evaluate")
        return r, J

    def imu_error_evaluate(self, mix):
        m = np.ascontiguousarray(mix, np.float64)
        r, J = np.zeros(6), np.zeros((6, 9))
        jp = (vp * 1)(vp(J.ctypes.data))
        check(lib().icg_ba_imu_error_evaluate(self._h, vp(m.ctypes.data), vp(r.ctypes.data), jp), "icg_ba_imu_error_evaluate")
        return r, J

    def marg_factor_evaluate(self, block_type, params, x0, J0, e0):
        """MarginalizationFactor::Evaluate: params = list of the remained blocks' current values (global sizes)."""
        bt = np.ascontiguousarray(block_type, np.int32)
        ps = [np.ascontiguousarray(x, np.float64) for x in params]
        x0, J0, e0 = (np.ascontiguousarray(x, np.float64) for x in (x0, J0, e0))
        r = len(e0)
        gs = {0: 7, 1: 9, 2: 7, 3: 1}
        res = np.zeros(r)
        Js = [np.zeros((r, gs[int(t)])) for t in bt]
        pp = (vp * len(ps))(*[vp(x.ctypes.data) for x in ps])
        jp = (vp * len(Js))(*[vp(x.ctypes.data) for x in Js])
        check(lib().icg_ba_marg_factor_evaluate(self._h, r, len(bt), vp(bt.ctypes.data), pp, vp(x0.ctypes.data), vp(J0.ctypes.data), vp(e0.ctypes.data),
                                                vp(res.ctypes.data), jp), "icg_ba_marg_factor_evaluate")
        return res, Js

    def imu_evaluate(self, blob, pose0, mix0, pose1, mix1, want_jac=True):
        a = [np.ascontiguousarray(x, np.float64) for x in (blob, pose0, mix0, pose1, mix1)]
        r = np.zeros(15)
        Js = [np.zeros((15, 7)), np.zeros((15, 9)), np.zeros((15, 7)), np.zeros((15, 9))]
        jp = (vp * 4)(*[vp(j.ctypes.data) for j in Js])
        check(lib().icg_ba_imu_evaluate(self._h, *[vp(x.ctypes.data) for x in a], vp(r.ctypes.data), jp if want_jac else None),
              "icg_ba_imu_evaluate")
        return r, Js
