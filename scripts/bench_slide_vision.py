"""Times icg_ba_slide_vision_resident against the slide it replaces, on B windows that have just been solved, culled and marginalized.

  host rows : icg_ba_slide_resident with the vision rows already built on the host (the restatement in tests/slide_vision_oracle.py builds
              them; that build is numpy and is not timed: a C++ integrator's own graph walk takes its place)
  device    : icg_ba_slide_vision_resident from the same culled windows and the same new keyframe observations in device memory, through the
              default binding (every built row back on the host, capacity-sized arrays)
  lean      : the same call through slide_vision(rows=False): only what the rest of the keyframe cycle reads on the host comes back

Per repetition the handle is restored outside the timed region (upload, solve, culling, culled marginalization).  Wall time from the call to a
device synchronise (CUDA events around it too), the kernel's time from torch.profiler in a separate pass, and the bytes each path moves
computed from the array shapes.  Prints one JSON line.

    python scripts/bench_slide_vision.py --cfg 3 --windows 296
    python scripts/bench_slide_vision.py --cfg 4 --windows 128
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_DISTINCT = 4


def card(torch):
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    return torch.cuda.get_device_name(0), plim


def cull_lists(p, fx, cx, cy):
    """the culling's observation lists: every factor's observation plus the reference one, keypoints from the factor constants"""
    fc = p["f_const"].reshape(-1, 14)
    L = p["L"]
    ref = np.zeros(L, np.int32)
    rkp = np.tile(np.array([[cx, cy]], np.float32), (L, 1))
    lists = [[] for _ in range(L)]
    px = lambda q: (np.float32(fx * q[0] / q[2] + cx), np.float32(fx * q[1] / q[2] + cy))
    for f in range(p["F"]):
        l = p["f_lm"][f]
        ref[l], rkp[l] = p["f_ref"][f], px(fc[f, 0:3])
        lists[l].append((int(p["f_obs"][f]), px(fc[f, 3:6]), f))
    off, node, kp, fac = [0], [], [], []
    for l in range(L):
        for o in lists[l] + [(int(ref[l]), tuple(rkp[l]), -1)]:
            node.append(o[0]), kp.append(o[1]), fac.append(o[2])
        off.append(len(node))
    from tests.post_solve_oracle import unit_quat_to_rot
    return dict(R_bc=np.array(unit_quat_to_rot(p["ext"][3:7])).reshape(3, 3), t_bc=p["ext"][:3].copy(), td_bc=float(p["ext"][7]), estimate_ext=0, estimate_td=0, lm_ref_node=ref, lm_ref_kp=rkp,
                obs_off=np.array(off, np.int32), obs_node=np.array(node, np.int32), obs_kp=np.array(kp, np.float32).reshape(-1, 2),
                obs_factor=np.array(fac, np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3, choices=(3, 4))
    ap.add_argument("--windows", type=int, default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_slide_vision.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from datagen.slide_window import build_next
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate
    from ic_gvins_b200.camera import CameraStruct
    from tests import slide_vision_oracle as so
    cfg3 = args.cfg == 3
    B = args.windows or (296 if cfg3 else 128)
    K, L, iters = (10, 300, 20) if cfg3 else (20, 2000, 12)
    gpu, plim = card(torch)
    fx, cx, cy = synth_ba.F_PIX, 640.0, 280.0
    cam = CameraStruct(fx, fx, cx, cy, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    camd = dict(fx=fx, fy=fx, cx=cx, cy=cy, skew=0.0)

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    kw = dict(K=K, L=L) if cfg3 else dict(K=K, L=L, n_ref=K)
    base = [synth_ba.make_window(pre, seed=9500 + i, **kw)[0] for i in range(min(N_DISTINCT, B))]
    probs0 = [copy.deepcopy(base[i % len(base)]) for i in range(B)]
    F = max(p["F"] for p in probs0) + 512
    s = WindowSolver(max_windows=B, max_K=K, max_L=L + 64, max_F=F, max_gnss=16, max_marg_r=15 * (K - 1) + 7)

    def restore():
        solved = copy.deepcopy(probs0)
        s.upload(solved)
        s.run_gvins(iters)
        s.gvins_optimization_end(solved)
        gs = s.update_and_cull(solved, cam, 1.5, [cull_lists(p, fx, cx, cy) for p in solved])
        mg = s.marginalize(solved, 1, resident=True, culled=gs)
        torch.cuda.synchronize()
        return solved, gs, mg

    solved, gs, mg = restore()
    rng = np.random.default_rng(9600)
    cases = []
    n_obs_tot = n_new_tot = 0
    for w, (p, g, m) in enumerate(zip(solved, gs, mg)):
        _, nxt, carry = build_next(p, 9700 + w, drop=(0,), n_new=1, prior=m)
        cur = nxt["K"] - 1
        lms = rng.choice(np.unique(p["f_lm"]), size=min(200 if cfg3 else 600, p["L"]), replace=False)
        xy = rng.uniform([100, 60], [1180, 500], (len(lms), 2)).astype(np.float32)
        vel = rng.normal(0, 5, (len(lms), 2))
        nn = 30 if cfg3 else 100
        new = dict(depth=rng.uniform(2, 40, nn), ref_xy=rng.uniform([100, 60], [1180, 500], (nn, 2)).astype(np.float32), vel_ref=rng.normal(0, 5, (nn, 2)),
                   ref_id=np.array([1000 + cur - 1 - j % 3 for j in range(nn)], np.int64), cur_xy=rng.uniform([100, 60], [1180, 500], (nn, 2)).astype(np.float32),
                   vel_cur=rng.normal(0, 5, (nn, 2)))
        td = np.zeros(nxt["K"])
        frames = {1000 + k: k for k in range(nxt["K"])}
        vis_h = dict(num_marg=1, node_in_map=np.ones(p["K"], np.uint8), node_td=td, cur_node=cur, frames=frames,
                     obs=[(int(l), cur, xy[i], vel[i]) for i, l in enumerate(lms)],
                     new=[dict(depth=new["depth"][j], ref_xy=new["ref_xy"][j], vel_ref=new["vel_ref"][j], ref_id=int(new["ref_id"][j]),
                               cur_xy=new["cur_xy"][j], vel_cur=new["vel_cur"][j]) for j in range(nn)])
        o = so.build(p, g, carry["node_src"], vis_h, camd)
        q, c = copy.deepcopy(nxt), copy.deepcopy(carry)
        q.update(L=o["L"], F=o["F"], invdepth=o["invdepth"], f_lm=o["f_lm"], f_ref=o["f_ref"], f_obs=o["f_obs"], f_const=o["f_const"].reshape(-1),
                 f_active=np.ones(o["F"], np.uint8))
        c.update(lm_src=o["lm_src"], f_src=o["f_src"])
        d = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a, dt)).cuda()
        vis_d = dict(num_marg=1, node_in_map=np.ones(p["K"], np.uint8), obs_factor=g["obs_factor"], camera=cam, node_td=td, cur_node=cur, frames=frames,
                     n_obs=len(lms), obs_lm=d(lms, np.int32), obs_node=d(np.full(len(lms), cur), np.int32), obs_undis_xy=d(xy, np.float32),
                     obs_vel=d(vel, np.float64), n_new=nn, new_depth=d(new["depth"], np.float64), new_ref_undis_xy=d(new["ref_xy"], np.float32),
                     new_vel_ref=d(new["vel_ref"], np.float64), new_ref_frame_id=d(new["ref_id"], np.int64), new_cur_undis_xy=d(new["cur_xy"], np.float32),
                     new_vel_cur=d(new["vel_cur"], np.float64))
        cases.append((nxt, carry, q, c, vis_d, o))
        n_obs_tot += len(lms)
        n_new_tot += nn

    def host():
        s.slide([copy.deepcopy(x[2]) for x in cases], [x[3] for x in cases], True)

    def device(rows=True):
        s.slide_vision([copy.deepcopy(x[0]) for x in cases], [copy.deepcopy(x[1]) for x in cases], [x[4] for x in cases], rows=rows)

    times = {"host_rows": [], "device": [], "lean": []}
    ev = {"host_rows": [], "device": [], "lean": []}
    for rep in range(args.reps + 1):
        for name, fn in (("host_rows", host), ("device", device), ("lean", lambda: device(False))):
            restore()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if rep:
                times[name].append(1e3 * (time.perf_counter() - t0))
                ev[name].append(e0.elapsed_time(e1))
    restore()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device()
        torch.cuda.synchronize()
    kern = {e.key: e.device_time_total / max(1, e.count) / 1e3 for e in prof.key_averages()
            if any(k in e.key for k in ("ba_vision_build", "ba_pack_structure", "ba_slide_gather", "ba_lm_ref_fill"))}
    # bytes from the shapes.  The vision call copies back per window [counts | slot -> factor table (bound Fb = F + n_obs + n_new)] and each row
    # array a caller asks for at its bound (Lb = L + n_new landmarks, Fb factors, n_obs + n_new new factor rows); the host-rows slide uploads
    # the structure tables at the handle's capacities, which the vision call writes on the device
    Lb = sum(p["L"] + nn for p, nn in zip(solved, [len(x[4]["new_depth"]) for x in cases]))
    Fb = sum(p["F"] for p in solved) + n_obs_tot + n_new_tot
    Nb = n_obs_tot + n_new_tot
    counts = 4 * 11 * B
    d2h_lean = counts + 4 * Fb + 4 * (2 * Lb + 4 * Fb) + Lb
    d2h_default = d2h_lean + 8 * Lb + 112 * Nb
    Kc, Lc, Fc = K, L + 64, F
    nvb = (Fc + 127 - Kc) // (128 - Kc) + Lc // 128 + 4 + Kc
    PM = Kc * (Kc - 1)
    h2d_tables = B * (16 * Fc + 4 * nvb + 4 * (Lc + 1) + 4 * Lc + 4 * Kc + 4 * (PM + 1) + 4 * PM + 4 * Fc + 4 + Fc)
    F_tot = sum(x[5]["F"] for x in cases)
    L_tot = sum(x[5]["L"] for x in cases)
    new_f = sum(int((x[5]["f_src"] < 0).sum()) for x in cases)
    out = dict(metric=f"slide_vision cfg-{args.cfg}", windows=B, gpu=gpu, power_limit_w=plim, reps=args.reps,
               host_rows_ms_median=statistics.median(times["host_rows"]), device_ms_median=statistics.median(times["device"]),
               lean_ms_median=statistics.median(times["lean"]), host_rows_event_ms_median=statistics.median(ev["host_rows"]),
               device_event_ms_median=statistics.median(ev["device"]), lean_event_ms_median=statistics.median(ev["lean"]),
               kernel_ms=kern, tracked_obs=n_obs_tot, new_points=n_new_tot, next_L=L_tot, next_F=F_tot, new_factors=new_f,
               bytes_h2d_vision_inputs=int(4 * sum(len(x[4]["obs_factor"]) for x in cases)),
               bytes_d2h_device=int(d2h_default), bytes_d2h_lean=int(d2h_lean), bytes_h2d_structure_tables_host_rows=int(h2d_tables),
               bytes_h2d_host_rows_vision=int(8 * (L_tot - sum(int((x[5]["lm_src"] >= 0).sum()) for x in cases)) + 112 * new_f))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
