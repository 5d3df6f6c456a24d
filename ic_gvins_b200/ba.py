"""Host-side mirror of the reference's window-solve seam (IG/ic_gvins.cc:1130-1239): `WindowSolver` plays the role of
`ceres::Problem` + `ceres::Solver::Solve`, `gvins_optimization()` restates the two-pass protocol of
GVINS::gvinsOptimization (solve N/4 -> chi-square culling -> solve N - N/4).  All arithmetic runs in libicgvins_b200.so.
"""
from __future__ import annotations

import copy
import ctypes as C

import numpy as np

from ._lib import check, lib, vp

IMU_BLOB = 480
dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)
bp = C.POINTER(C.c_uint8)


class BaProblem(C.Structure):
    """ctypes image of `icg_ba_problem` (include/icgvins_b200.h)."""
    _fields_ = [
        ("K", C.c_int32), ("L", C.c_int32), ("F", C.c_int32),
        ("pose", dp), ("mix", dp), ("ext", dp), ("invdepth", dp),
        ("ext_const", C.c_int32), ("td_const", C.c_int32),
        ("f_lm", ip), ("f_ref", ip), ("f_obs", ip), ("f_const", dp), ("f_active", bp),
        ("reproj_std", C.c_double), ("reproj_huber", C.c_int32),
        ("n_imu", C.c_int32), ("imu_blob", dp), ("has_imu_error", C.c_int32),
        ("has_pose_prior", C.c_int32), ("pose_prior", dp), ("pose_prior_std", dp),
        ("has_mix_prior", C.c_int32), ("mix_prior", dp), ("mix_prior_std", dp),
        ("n_gnss", C.c_int32), ("gnss_node", ip), ("gnss_blh", dp), ("gnss_std", dp), ("lever", C.c_double * 3),
        ("gnss_huber", C.c_int32),
        ("marg_r", C.c_int32), ("marg_nblocks", C.c_int32), ("marg_block_type", ip), ("marg_block_node", ip),
        ("marg_x0", dp), ("marg_J0", dp), ("marg_e0", dp),
    ]


class BaPrior(C.Structure):
    """ctypes image of `icg_ba_prior`."""
    _fields_ = [("m", C.c_int32), ("r", C.c_int32), ("nblocks", C.c_int32), ("rcap", C.c_int32), ("block_type", ip), ("block_node", ip),
                ("x0", dp), ("J0", dp), ("e0", dp), ("Hp", dp), ("bp", dp)]


class BaSummary(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("num_successful_steps", C.c_int32), ("termination", C.c_int32), ("reserved", C.c_int32),
                ("initial_cost", C.c_double), ("final_cost", C.c_double), ("final_radius", C.c_double)]


fp = C.POINTER(C.c_float)


class CullWindow(C.Structure):
    """ctypes image of `icg_ba_cull_window`."""
    _fields_ = [("R_bc", C.c_double * 9), ("t_bc", C.c_double * 3), ("td_bc", C.c_double), ("estimate_ext", C.c_int32), ("estimate_td", C.c_int32),
                ("lm_ref_node", ip), ("lm_ref_kp", fp), ("obs_off", ip), ("obs_node", ip), ("obs_kp", fp), ("obs_factor", ip),
                ("R_bc_out", C.c_double * 9), ("t_bc_out", C.c_double * 3), ("td_bc_out", C.c_double), ("ext_accepted", C.c_int32),
                ("cam_pose", dp), ("lm_pw", dp), ("lm_depth", dp), ("lm_outlier", bp), ("obs_outlier", bp), ("counts", C.c_int32 * 5)]


class ReintWindow(C.Structure):
    """ctypes image of `icg_ba_reint_window`."""
    _fields_ = [("reintegrate", C.c_int32), ("imu", dp), ("imu_off", ip), ("status", C.POINTER(C.c_int8)), ("blob_out", dp), ("end_state10", dp),
                ("count", C.c_int32)]


_CULL_IN = dict(lm_ref_node=(np.int32, ip), lm_ref_kp=(np.float32, fp), obs_off=(np.int32, ip), obs_node=(np.int32, ip), obs_kp=(np.float32, fp),
                obs_factor=(np.int32, ip))


def cull_struct(prob: dict, ci: dict) -> CullWindow:
    """The icg_ba_cull_window of one window over the arrays of `ci` (made contiguous in place; output arrays are added to it)."""
    s = CullWindow()
    K, L = int(prob["K"]), int(prob["L"])
    for k, v in zip(("R_bc", "t_bc"), (np.asarray(ci["R_bc"], np.float64).reshape(-1), np.asarray(ci["t_bc"], np.float64).reshape(-1))):
        getattr(s, k)[:] = [float(x) for x in v]
    s.td_bc, s.estimate_ext, s.estimate_td = float(ci.get("td_bc", 0.0)), int(ci.get("estimate_ext", 1)), int(ci.get("estimate_td", 1))
    for k, (dt, pt) in _CULL_IN.items():
        if ci.get(k) is None:
            continue
        a = np.ascontiguousarray(ci[k], dtype=dt)
        ci[k] = a
        setattr(s, k, a.ctypes.data_as(pt) if a.size else pt())
    n_obs = int(ci["obs_off"][L]) if L > 0 else 0
    ci.update(cam_pose=np.zeros((K, 12)), lm_pw=np.zeros((L, 3)), lm_depth=np.zeros(L), lm_outlier=np.zeros(L, np.uint8), obs_outlier=np.zeros(n_obs, np.uint8))
    s.cam_pose, s.lm_pw, s.lm_depth = (ci[k].ctypes.data_as(dp) for k in ("cam_pose", "lm_pw", "lm_depth"))
    s.lm_outlier, s.obs_outlier = ci["lm_outlier"].ctypes.data_as(bp), ci["obs_outlier"].ctypes.data_as(bp)
    return s


_ARR = dict(pose=np.float64, mix=np.float64, ext=np.float64, invdepth=np.float64, f_lm=np.int32, f_ref=np.int32, f_obs=np.int32,
            f_const=np.float64, f_active=np.uint8, imu_blob=np.float64, pose_prior=np.float64, pose_prior_std=np.float64,
            mix_prior=np.float64, mix_prior_std=np.float64, gnss_node=np.int32, gnss_blh=np.float64, gnss_std=np.float64,
            marg_block_type=np.int32, marg_block_node=np.int32, marg_x0=np.float64, marg_J0=np.float64, marg_e0=np.float64)
_SCAL = ["K", "L", "F", "ext_const", "td_const", "reproj_std", "reproj_huber", "n_imu", "has_imu_error", "has_pose_prior",
         "has_mix_prior", "n_gnss", "gnss_huber", "marg_r", "marg_nblocks"]


def to_struct(prob: dict) -> BaProblem:
    """Build the C struct over the dict's numpy arrays IN PLACE (arrays are made contiguous inside the dict so that the
    solve's in/out parameter updates are visible to the caller)."""
    s = BaProblem()
    for k, dt in _ARR.items():
        a = np.ascontiguousarray(prob[k], dtype=dt)
        prob[k] = a
        ptr_t = dp if dt == np.float64 else ip if dt == np.int32 else bp
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


def _integ_struct(s, g, m, arg, with_rows=True):
    """fill one icg_ba_slide_integrate from an `integrate` dict of WindowSolver.slide_integrate (m = next n_imu; with_rows False: imu /
    imu_off stay NULL, the rows come from the device)"""
    from ._lib import u8p
    if g.get("imu_from") is not None:
        s.imu_from = arg(g["imu_from"], np.int32, ip)
        if not with_rows:
            pass
        elif "imu_off" in g:
            s.imu, s.imu_off = arg(g["imu"], np.float64, dp), arg(g["imu_off"], np.int32, ip)
        else:
            rows = [np.zeros((0, 7)) if r is None else np.asarray(r, np.float64).reshape(-1, 7) for r in g["imu_rows"]]
            off = np.zeros(m + 1, np.int32)
            off[1:] = np.cumsum([len(r) for r in rows])
            imu = np.concatenate(rows, axis=0) if rows else np.zeros((0, 7))
            s.imu, s.imu_off = arg(imu, np.float64, dp), arg(off, np.int32, ip)
        s.gravity3 = arg(np.broadcast_to(np.asarray(g["gravity"], np.float64), (m, 3)), np.float64, dp)
        s.normal = arg(np.broadcast_to(np.asarray(g.get("normal", False), np.uint8), (m,)), np.uint8, u8p)
        if g.get("state16") is not None:
            s.state16 = arg(g["state16"], np.float64, dp)
    if g.get("node_from_imu") is not None:
        s.node_from_imu = arg(g["node_from_imu"], np.uint8, u8p)
    if g.get("gnss_node") is not None:
        s.gnss_node, s.gnss_dt = arg(g["gnss_node"], np.int32, ip), arg(g["gnss_dt"], np.float64, dp)


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
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
        summ = (BaSummary * n)()
        check(lib().icg_ba_solve(self._h, n, arr, max_num_iterations, summ), "icg_ba_solve")
        return [dict(iterations=s.iterations, num_successful_steps=s.num_successful_steps, termination=s.termination,
                     initial_cost=s.initial_cost, final_cost=s.final_cost, final_radius=s.final_radius) for s in summ]

    def solve_structs(self, arr, n, max_num_iterations, summ):
        check(lib().icg_ba_solve(self._h, n, arr, max_num_iterations, summ), "icg_ba_solve")

    # -- device-resident stages
    def upload(self, problems):
        n = len(problems)
        self._keep = (BaProblem * n)(*[to_struct(p) for p in problems])
        self._n = n
        check(lib().icg_ba_upload(self._h, n, self._keep), "icg_ba_upload")

    def run(self, max_num_iterations: int, restart: bool = False):
        check(lib().icg_ba_run(self._h, max_num_iterations, 1 if restart else 0), "icg_ba_run")

    def download(self, write_back: bool = True):
        summ = (BaSummary * self._n)()
        check(lib().icg_ba_download(self._h, self._n, self._keep if write_back else None, summ), "icg_ba_download")
        return [dict(iterations=s.iterations, num_successful_steps=s.num_successful_steps, termination=s.termination,
                     initial_cost=s.initial_cost, final_cost=s.final_cost, final_radius=s.final_radius) for s in summ]

    def sync(self):
        check(lib().icg_ba_sync(self._h), "icg_ba_sync")

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
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
        summ = (BaSummary * (2 * n))()
        culled = (C.c_int32 * (2 * n))()
        check(lib().icg_ba_gvins_optimization(self._h, n, arr, num_iterations, summ, culled), "icg_ba_gvins_optimization")
        f = lambda s: dict(iterations=s.iterations, num_successful_steps=s.num_successful_steps, termination=s.termination,
                           initial_cost=s.initial_cost, final_cost=s.final_cost, final_radius=s.final_radius)
        return [dict(pass1=f(summ[2 * w]), pass2=f(summ[2 * w + 1]), reproj_removed=culled[2 * w], gnss_reweighted=culled[2 * w + 1])
                for w in range(n)]

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
                cw[w].lm_outlier, cw[w].obs_outlier = (a.ctypes.data_as(bp) for a in k["flags"])
            ptrs = (vp * len(nim))(*[vp(m.ctypes.data) for m in nim])
            check(lib().icg_ba_marginalize_resident_culled(self._h, call["n"], call["arr"], vp(call["nm"].ctypes.data), cw, ptrs, call["pri"]),
                  "icg_ba_marginalize_resident_culled")
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
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
        outs = [dict(c) for c in cull_inputs]
        cw = (CullWindow * n)(*[cull_struct(p, c) for p, c in zip(problems, outs)])
        cam = camera.c if hasattr(camera, "c") else camera
        check(lib().icg_ba_update_and_cull_resident(self._h, n, arr, C.byref(cam), float(std), cw), "icg_ba_update_and_cull_resident")
        for c, s in zip(outs, cw):
            c.update(R_bc_out=np.array(s.R_bc_out[:]).reshape(3, 3), t_bc_out=np.array(s.t_bc_out[:]), td_bc_out=s.td_bc_out, ext_accepted=s.ext_accepted,
                     counts=np.array(s.counts[:], np.int32))
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
        from ._lib import IcgError
        if isinstance(problems, dict):
            problems, imu_rows = [problems], [imu_rows]
        n = len(problems)
        flags = [1] * n if reintegrate is None else [int(bool(x)) for x in reintegrate]
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
        io = (ReintWindow * n)()
        outs, keep = [], []
        for w, p in enumerate(problems):
            m = int(p["n_imu"])
            o = dict(status=np.zeros(m, np.int8), count=0, end_states=np.zeros((m, 10)),
                     blobs=np.array(np.asarray(p["imu_blob"], np.float64)[:m * IMU_BLOB].reshape(m, IMU_BLOB), copy=True))
            outs.append(o)
            io[w].reintegrate = flags[w] if m > 0 else 0
            io[w].status, io[w].blob_out = o["status"].ctypes.data_as(C.POINTER(C.c_int8)), o["blobs"].ctypes.data_as(dp)
            io[w].end_state10 = o["end_states"].ctypes.data_as(dp)
            if io[w].reintegrate and not stored:
                rows = [np.asarray(x, np.float64).reshape(-1, 7) for x in imu_rows[w]]
                off = np.zeros(m + 1, np.int32)
                off[1:] = np.cumsum([len(x) for x in rows])
                imu = np.ascontiguousarray(np.concatenate(rows, axis=0)) if rows else np.zeros((0, 7))
                keep.append((imu, off))
                io[w].imu, io[w].imu_off = imu.ctypes.data_as(dp), off.ctypes.data_as(ip)
        nz = np.ascontiguousarray(noise5, np.float64)
        stn = np.ascontiguousarray(station, np.float64)
        rc = getattr(lib(), fn)(self._h, n, arr, vp(nz.ctypes.data), vp(stn.ctypes.data), io)
        for w, (p, o) in enumerate(zip(problems, outs)):
            o["count"] = int(io[w].count)
            if (o["status"] == 1).any():
                p["imu_blob"].reshape(-1, IMU_BLOB)[:len(o["status"])][o["status"] == 1] = o["blobs"][o["status"] == 1]
        if rc != 0:
            err = IcgError(f"{fn} failed with code {rc}: {lib().icg_last_error().decode('utf-8', 'replace')}")
            err.code, err.results = rc, outs
            raise err
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
        from ._lib import SlideWindow
        n = len(next_problems)
        flags = [prior_from_marg] * n if np.isscalar(prior_from_marg) else list(prior_from_marg)
        arr = (BaProblem * n)(*[to_struct(p) for p in next_problems])
        cw = (SlideWindow * n)()
        keep = []
        for w, c in enumerate(carry):
            for k in ("node_src", "lm_src", "f_src", "imu_src", "gnss_src"):
                if c.get(k) is None:
                    continue
                a = np.ascontiguousarray(c[k], np.int32)
                keep.append(a)
                setattr(cw[w], k, a.ctypes.data_as(ip))
            cw[w].prior_from_marg = 1 if flags[w] else 0
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
        from ._lib import IcgError, SlideIntegrate, SlideWindow, u8p
        n = len(next_problems)
        flags = [prior_from_marg] * n if np.isscalar(prior_from_marg) else list(prior_from_marg)
        arr = (BaProblem * n)(*[to_struct(p) for p in next_problems])
        cw = (SlideWindow * n)()
        iw = (SlideIntegrate * n)()
        keep, outs = [], []

        def arg(a, dtype, ptr):
            a = np.ascontiguousarray(a, dtype)
            keep.append(a)
            return a.ctypes.data_as(ptr)

        for w, (p, c, g) in enumerate(zip(next_problems, carry, integrate)):
            for k in ("node_src", "lm_src", "f_src", "imu_src", "gnss_src"):
                if c.get(k) is not None:
                    setattr(cw[w], k, arg(c[k], np.int32, ip))
            cw[w].prior_from_marg = 1 if flags[w] else 0
            m = int(p["n_imu"])
            o = dict(status=np.zeros(m, np.int8), blobs=np.zeros((m, IMU_BLOB)), end_states=np.zeros((m, 10)))
            outs.append(o)
            iw[w].status, iw[w].blob_out = o["status"].ctypes.data_as(C.POINTER(C.c_int8)), o["blobs"].ctypes.data_as(dp)
            iw[w].end_state10 = o["end_states"].ctypes.data_as(dp)
            if g:
                _integ_struct(iw[w], g, m, arg)
        nz = np.ascontiguousarray(noise5, np.float64)
        stn = np.ascontiguousarray(station, np.float64)
        rc = getattr(lib(), fn)(self._h, n, arr, cw, iw, vp(nz.ctypes.data), vp(stn.ctypes.data))
        if rc != 0:
            err = IcgError(f"{fn} failed with code {rc}: {lib().icg_last_error().decode('utf-8', 'replace')}")
            err.code, err.results = rc, outs
            raise err
        self._keep, self._n = arr, n
        return outs

    def imu_samples_from_ins(self, ins, streams, node_times) -> None:
        """Seeds the handle's IMU sample store (icg_ba_imu_samples_from_ins): factor k of resident window w gets getImuSeriesFromTo(
        node_times[w][k], node_times[w][k + 1]) cut from stream streams[w] of `ins` (an ins.InsWindow on this handle's device).  Call it right
        after the upload of windows whose INS windows still cover their spans."""
        from ._lib import InsCut
        n = len(streams)
        cut = (InsCut * n)()
        keep = []
        for w in range(n):
            t = np.ascontiguousarray(node_times[w], np.float64)
            keep.append(t)
            cut[w].stream, cut[w].node_time = int(streams[w]), t.ctypes.data_as(dp)
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
        from ._lib import IcgError, SlideIns, SlideIntegrate
        fn = "icg_ba_slide_ins_resident"
        n = len(next_problems)
        keep = []
        n_rows = [np.full(int(p["n_imu"]), -1, np.int32) for p in next_problems]
        statuses = [np.zeros(int(p["n_imu"]), np.int8) for p in next_problems]
        blobs = [np.zeros((int(p["n_imu"]), IMU_BLOB)) for p in next_problems]
        ends = [np.zeros((int(p["n_imu"]), 10)) for p in next_problems]

        def arg(a, dtype, ptr):
            a = np.ascontiguousarray(a, dtype)
            keep.append(a)
            return a.ctypes.data_as(ptr)

        def call(arr, cw, iw, nz, stn, vw):
            io = (SlideIns * n)()
            for w, p in enumerate(next_problems):
                m = int(p["n_imu"])
                if iw is not None:
                    io[w].integ = iw[w]
                elif integrate is not None and integrate[w]:
                    _integ_struct(io[w].integ, integrate[w], m, arg, with_rows=False)
                g = io[w].integ
                g.status, g.blob_out = statuses[w].ctypes.data_as(C.POINTER(C.c_int8)), blobs[w].ctypes.data_as(dp)
                g.end_state10 = ends[w].ctypes.data_as(dp)
                io[w].stream = int(streams[w])
                if node_times[w] is not None:
                    io[w].node_time = arg(node_times[w], np.float64, dp)
                if merge_src is not None and merge_src[w] is not None:
                    io[w].merge_src = arg(merge_src[w], np.int32, ip)
                io[w].n_rows = n_rows[w].ctypes.data_as(ip)
            return lib().icg_ba_slide_ins_resident(self._h, ins._h, n, arr, cw, io, vp(nz.ctypes.data), vp(stn.ctypes.data), vw)

        def results():
            return [dict(status=statuses[w], blobs=blobs[w], end_states=ends[w], n_rows=n_rows[w]) for w in range(n)]

        if vision is not None:
            try:
                res = self._slide_vision(fn, next_problems, carry, vision, integrate, noise5, station, prior_from_marg, call=call)
            except IcgError as e:
                e.results = results()
                raise
            for w, r in enumerate(res):
                r.update(results()[w])
            return res
        from ._lib import SlideWindow
        flags = [prior_from_marg] * n if np.isscalar(prior_from_marg) else list(prior_from_marg)
        arr = (BaProblem * n)(*[to_struct(p) for p in next_problems])
        cw = (SlideWindow * n)()
        for w, c in enumerate(carry):
            for k in ("node_src", "lm_src", "f_src", "imu_src", "gnss_src"):
                if c.get(k) is not None:
                    setattr(cw[w], k, arg(c[k], np.int32, ip))
            cw[w].prior_from_marg = 1 if flags[w] else 0
        nz = np.ascontiguousarray(noise5, np.float64)
        stn = np.ascontiguousarray(station, np.float64)
        rc = call(arr, cw, None, nz, stn, None)
        if rc != 0:
            err = IcgError(f"{fn} failed with code {rc}: {lib().icg_last_error().decode('utf-8', 'replace')}")
            err.code, err.results = rc, results()
            raise err
        self._keep, self._n = arr, n
        return results()

    def slide_vision(self, next_problems, carry, vision, integrate=None, noise5=None, station=(0.0, 0.0, 0.0), prior_from_marg=True):
        return self._slide_vision("icg_ba_slide_vision_resident", next_problems, carry, vision, integrate, noise5, station, prior_from_marg)

    def shard_slide_vision(self, next_problems, carry, vision, integrate=None, noise5=None, station=(0.0, 0.0, 0.0), prior_from_marg=True):
        """slide_vision() on a landmark-sharded handle (icg_ba_shard_slide_vision_resident), a collective call: every rank passes its next shards
        (camera side as shard_slide takes it), their carry maps (node / IMU / GNSS) and its own vision dicts (shard_vision_inputs); new map
        point j of window w is built on rank (j + w) % world.  Returns the rank's shard as slide_vision does (lm_src / f_src shard-local,
        lm_origin: old shard-local landmark or -(j + 1) for global new point j, nan_flags: old shard L + every new point, set on its own rank)."""
        return self._slide_vision("icg_ba_shard_slide_vision_resident", next_problems, carry, vision, integrate, noise5, station, prior_from_marg)

    def _slide_vision(self, fn, next_problems, carry, vision, integrate=None, noise5=None, station=(0.0, 0.0, 0.0), prior_from_marg=True,
                      call=None):
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
        the others zero).  A rejected call raises IcgError with the handle unchanged."""
        from ._lib import IcgError, SlideIntegrate, SlideVision, SlideWindow
        from .camera import CameraStruct
        if integrate is not None and noise5 is None:
            raise ValueError(f"{fn}: integrate needs noise5")
        n = len(next_problems)
        flags = [prior_from_marg] * n if np.isscalar(prior_from_marg) else list(prior_from_marg)
        Lc, Fc = self.max_L, self.max_F
        outs = []
        for p, v in zip(next_problems, vision):  # the built rows land here, sized to the handle's capacity until the call returns
            o = dict(lm_src=np.zeros(Lc, np.int32), lm_origin=np.zeros(Lc, np.int32), nan_flags=np.zeros(Lc + int(v.get("n_new", 0)), np.uint8), f_src=np.zeros(Fc, np.int32), f_lm=np.zeros(Fc, np.int32), f_ref=np.zeros(Fc, np.int32),
                     f_obs=np.zeros(Fc, np.int32), invdepth=np.zeros(Lc), f_const=np.zeros((Fc, 14)))
            outs.append(o)
            p.update(L=0, F=0, invdepth=np.zeros(0), f_lm=np.zeros(0, np.int32), f_ref=np.zeros(0, np.int32), f_obs=np.zeros(0, np.int32),
                     f_const=np.zeros(0), f_active=np.zeros(0, np.uint8))
        arr = (BaProblem * n)(*[to_struct(p) for p in next_problems])
        cw = (SlideWindow * n)()
        vw = (SlideVision * n)()
        iw = (SlideIntegrate * n)() if integrate is not None else None
        keep = []

        def arg(a, dtype, ptr):
            a = np.ascontiguousarray(a, dtype)
            keep.append(a)
            return a.ctypes.data_as(ptr)

        def dev(t):
            return None if t is None else vp(t.data_ptr() if hasattr(t, "data_ptr") else int(t))

        for w, (p, c, v) in enumerate(zip(next_problems, carry, vision)):
            for k in ("node_src", "imu_src", "gnss_src"):
                if c.get(k) is not None:
                    setattr(cw[w], k, arg(c[k], np.int32, ip))
            cw[w].prior_from_marg = 1 if flags[w] else 0
            if iw is not None and integrate[w]:
                _integ_struct(iw[w], integrate[w], int(p["n_imu"]), arg, with_rows=call is None)
            s = vw[w]
            s.num_marg = int(v["num_marg"])
            s.node_in_map = arg(v["node_in_map"], np.uint8, bp)
            if v.get("obs_factor") is not None and len(v["obs_factor"]):
                s.obs_factor = arg(v["obs_factor"], np.int32, ip)
            cam = v["camera"]
            cs = cam.c if hasattr(cam, "c") else cam
            s.cam[:] = [float(getattr(cs, k)) for k, _ in CameraStruct._fields_]
            s.node_td = arg(v["node_td"], np.float64, dp)
            s.cur_node = int(v["cur_node"])
            frames = v.get("frames", {})
            s.n_frames = len(frames)
            s.frame_id = arg(np.array(list(frames.keys()), np.int64), np.int64, C.POINTER(C.c_int64))
            s.frame_node = arg(np.array(list(frames.values()), np.int32), np.int32, ip)
            s.n_obs, s.n_in = int(v.get("n_obs", 0)), int(v.get("n_in", 0))
            s.dev_n, s.obs_src, s.obs_lm, s.obs_node = (dev(v.get(k)) for k in ("dev_n", "obs_src", "obs_lm", "obs_node"))
            s.obs_undis_xy, s.obs_vel = dev(v.get("obs_undis_xy")), dev(v.get("obs_vel"))
            s.n_new = int(v.get("n_new", 0))
            s.dev_new_n = dev(v.get("dev_new_n"))
            s.new_depth, s.new_vel_ref, s.new_vel_cur = (dev(v.get(k)) for k in ("new_depth", "new_vel_ref", "new_vel_cur"))
            s.new_ref_undis_xy, s.new_cur_undis_xy, s.new_ref_frame_id = (dev(v.get(k)) for k in ("new_ref_undis_xy", "new_cur_undis_xy", "new_ref_frame_id"))
            o = outs[w]
            s.lm_src, s.f_src, s.f_lm, s.f_ref, s.f_obs = (o[k].ctypes.data_as(ip) for k in ("lm_src", "f_src", "f_lm", "f_ref", "f_obs"))
            s.invdepth, s.f_const = o["invdepth"].ctypes.data_as(dp), o["f_const"].ctypes.data_as(dp)
            s.lm_origin, s.nan_flags = o["lm_origin"].ctypes.data_as(ip), o["nan_flags"].ctypes.data_as(bp)
        nz = np.ascontiguousarray(noise5 if noise5 is not None else np.zeros(5), np.float64)
        stn = np.ascontiguousarray(station, np.float64)
        if call is not None:  # slide_ins: the INS form of the call, from the same structs
            rc = call(arr, cw, iw, nz, stn, vw)
        else:
            rc = getattr(lib(), fn)(self._h, n, arr, cw, None if iw is None else iw, vp(nz.ctypes.data) if iw is not None else None,
                                    vp(stn.ctypes.data) if iw is not None else None, vw)
        if rc != 0:
            err = IcgError(f"{fn} failed with code {rc}: {lib().icg_last_error().decode('utf-8', 'replace')}")
            err.code = rc
            raise err
        res = []
        for w, (p, c, o) in enumerate(zip(next_problems, carry, outs)):
            L, F = int(vw[w].L), int(vw[w].F)
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
        self._keep, self._n = arr, n
        return res

    def gvins_optimization_end(self, problems):
        """icg_ba_gvins_optimization_end after run_gvins(): synchronises, writes the parameters, f_active and gnss_std back into the problem
        dicts and returns the two-pass results in the layout of gvins_optimization_batch."""
        n = len(problems)
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
        summ = (BaSummary * (2 * n))()
        culled = (C.c_int32 * (2 * n))()
        check(lib().icg_ba_gvins_optimization_end(self._h, n, arr, summ, culled), "icg_ba_gvins_optimization_end")
        f = lambda s: dict(iterations=s.iterations, num_successful_steps=s.num_successful_steps, termination=s.termination,
                           initial_cost=s.initial_cost, final_cost=s.final_cost, final_radius=s.final_radius)
        return [dict(pass1=f(summ[2 * w]), pass2=f(summ[2 * w + 1]), reproj_removed=culled[2 * w], gnss_reweighted=culled[2 * w + 1])
                for w in range(n)]

    def marg_prepare(self, problems, num_marg=1, want_schur=True):
        """The argument block of one icg_ba_marginalize call (struct array over the problems' host arrays + caller-allocated output arrays):
        what a C++ caller keeps alive across keyframes.  marg_run issues the call, marg_collect turns the outputs into dicts."""
        n = len(problems)
        nm = np.full(n, num_marg, np.int32) if np.isscalar(num_marg) else np.ascontiguousarray(num_marg, np.int32)
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
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
            pri[w].block_type, pri[w].block_node = b["bt"].ctypes.data_as(ip), b["bn"].ctypes.data_as(ip)
            pri[w].x0, pri[w].J0, pri[w].e0 = b["x0"].ctypes.data_as(dp), b["J0"].ctypes.data_as(dp), b["e0"].ctypes.data_as(dp)
            if want_schur:
                pri[w].Hp, pri[w].bp = b["Hp"].ctypes.data_as(dp), b["bp"].ctypes.data_as(dp)
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
