#!/usr/bin/env python
"""Cost of the culling on the lists the vision slide builds on the device (icg_ba_update_and_cull_built) against the culling on host lists
(icg_ba_update_and_cull_resident) on one H100, for B resident windows: cfg 3 (K = 10, L = 300, B = 296) and cfg 4 (K = 20, L = 2000, B = 64).

    python scripts/bench_cull_built.py [--reps 20] [--warmup 3]

One JSON line per configuration:
  * the two cullings, alternated rep by rep, host clock around each synchronous call, medians.  The host-list culling is fed the very lists the
    built one walked (they are equal by tests/test_cull_built_gpu.py), so the two calls do the same kernel work;
  * ba_vision_build's kernel time (with the list emission) from a torch.profiler run of a vision slide.  The whole slide before and after the
    emission is timed by scripts/bench_slide_vision.py, run on this tree and on a tree without the emission;
  * bytes crossing PCIe per call for the lists, computed from shapes: the host-list culling's list upload plus the slide's obs_factor,
    against the built culling's download of the four integer lists (the C call with NULL keypoint outputs;
    icg_ba_marginalize_resident_culled reads the integer lists on the host), and the download of the Python binding, which also returns the
    keypoints.
The gather the host does today (the walk over observations()) is not part of either call and is not timed.  The card name and power limit
are read in the same run.  Writes nothing to the source tree.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LISTS = ("lm_ref_node", "lm_ref_kp", "obs_off", "obs_node", "obs_kp", "obs_factor")


def run(B, K, L, F, R, reps, warmup):
    import torch
    from datagen import synth_ba
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate
    from ic_gvins_b200.camera import Camera
    from tests import slide_vision_oracle as so
    from tests.test_post_solve_gpu import CAMD, STD, cull_inputs
    from tests.test_slide_vision_gpu import Keyframe

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    base = [synth_ba.make_window(pre, K=K, L=L, seed=7000 + i, n_ref=K)[0] for i in range(min(8, B))]
    probs = [copy.deepcopy(base[w % len(base)]) for w in range(B)]
    cam = Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0] * 4)
    s = WindowSolver(max_windows=B, max_K=K, max_L=L, max_F=F, max_gnss=16, max_marg_r=R)
    try:
        s.gvins_optimization_batch(probs, 20)
        cis = [cull_inputs(p, p["ext"].copy(), 7100 + w, bad_kp=20) for w, p in enumerate(probs)]
        gs = s.update_and_cull(probs, cam, STD, cis)
        mgs = s.marginalize(probs, 1, resident=True, culled=gs)
        kfs = [Keyframe(p, g, mg, so.reference_rows(p), 7200 + w, n_new=20, n_obs=L // 5) for w, (p, g, mg) in enumerate(zip(probs, gs, mgs))]
        nxt, carry = [copy.deepcopy(k.nxt) for k in kfs], [copy.deepcopy(k.carry) for k in kfs]
        vis = [k.device() for k in kfs]
        s.slide_vision(nxt, carry, vis)
        s.run_gvins(20)
        s.gvins_optimization_end(nxt)
        exts = [{k: c[k] for k in ("R_bc", "t_bc", "td_bc", "estimate_ext", "estimate_td")} for c in cis]
        built = s.update_and_cull_built(nxt, cam, STD, exts)
        host_in = [dict(e, **{k: b[k] for k in LISTS}) for e, b in zip(exts, built)]
        th, tb = [], []
        for i in range(warmup + reps):
            t0 = time.perf_counter()
            s.update_and_cull(nxt, cam, STD, host_in)
            t1 = time.perf_counter()
            s.update_and_cull_built(nxt, cam, STD, exts)
            t2 = time.perf_counter()
            if i >= warmup:
                th.append((t1 - t0) * 1e3), tb.append((t2 - t1) * 1e3)
        n_obs = sum(b["n_obs"] for b in built)
        nL = sum(p["L"] for p in nxt)
        host_bytes = 4 * nL + 4 * (nL + B) + 4 * n_obs + 8 * nL + 8 * n_obs + 4 * n_obs  # lists up, plus the slide's obs_factor
        built_bytes = 4 * nL + 4 * (nL + B) + 8 * n_obs  # the four integer lists down
        python_bytes = built_bytes + 8 * nL + 8 * n_obs  # and the keypoints the binding returns
        # ba_vision_build's kernel time: one more culling and slide under the profiler
        gs2 = s.update_and_cull_built(nxt, cam, STD, exts)
        mgs2 = s.marginalize(nxt, 1, resident=True, culled=gs2)
        refs = [so.reference_rows(p) for p in nxt]
        kfs2 = [Keyframe(p, g, mg, rf, 7300 + w, n_new=20, n_obs=L // 5) for w, (p, g, mg, rf) in enumerate(zip(nxt, gs2, mgs2, refs))]
        v2 = [k.device() for k in kfs2]
        for v in v2:
            v.pop("obs_factor")
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.slide_vision([copy.deepcopy(k.nxt) for k in kfs2], [copy.deepcopy(k.carry) for k in kfs2], v2)
            torch.cuda.synchronize()
        kern = sum(e.device_time for e in prof.events() if "ba_vision_build" in e.name) / 1e3
        return dict(windows=B, K=K, L=L, n_obs_per_window=n_obs / B, host_list_cull_ms=float(np.median(th)), built_cull_ms=float(np.median(tb)),
                    ba_vision_build_kernel_ms=kern, host_list_bytes_up=host_bytes, built_list_bytes_down=built_bytes,
                    built_list_bytes_down_python=python_bytes)
    finally:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_cull_built.py: no CUDA device; the product path has no CPU fallback")
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        plim = "unknown"
    card = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=plim)
    for B, K, L, F, R in ((296, 10, 300, 2700, 160), (64, 20, 2000, 12000, 292)):
        print(json.dumps(dict(card, **run(B, K, L, F, R, args.reps, args.warmup))), flush=True)


if __name__ == "__main__":
    main()
