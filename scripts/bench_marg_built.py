#!/usr/bin/env python
"""Cost of the marginalization whose factor set and column map are built on the device (icg_ba_marginalize_built) against
icg_ba_marginalize_resident_culled with NULL lists (the factor set and the column map built on the host from the culling's host copy of the
lists and the problem's f_lm / f_ref / f_obs) on one H100, for B resident windows after the same culling on the built lists: cfg 3 (K = 10,
L = 300, B = 296) and cfg 4 (K = 20, L = 2000, B = 128, on a max_K = 20 handle).

    python scripts/bench_marg_built.py [--reps 20] [--warmup 3]

One JSON line per configuration:
  * the two calls, alternated rep by rep on the same culled windows, host clock around each synchronous call, medians;
  * bytes each call moves H2D and D2H, computed from the shapes: the host-list call's column map (8 + 2 max_K + max_L ints) and factor mask
    (max_F bytes) up per window, against the built call's 120-byte window record up and its 8 + 2 max_K ints down; the prior's D2H is the
    same for both and is counted separately;
  * the card name and power limit, read in the same run.
Whether the keyframe cycle is faster end to end is not measured.  Writes nothing to the source tree.
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


def run(B, K, L, F, R, reps, warmup):
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
        s.slide_vision(nxt, carry, [k.device() for k in kfs])
        s.run_gvins(20)
        s.gvins_optimization_end(nxt)
        exts = [{k: c[k] for k in ("R_bc", "t_bc", "td_bc", "estimate_ext", "estimate_td")} for c in cis]
        built = s.update_and_cull_built(nxt, cam, STD, exts)
        bare = [{k: v for k, v in g.items() if k not in ("lm_ref_node", "obs_off", "obs_node", "obs_factor")} for g in built]
        lean = [dict(p, invdepth=np.zeros(0), f_lm=np.zeros(0, np.int32), f_ref=np.zeros(0, np.int32), f_obs=np.zeros(0, np.int32),
                     f_const=np.zeros(0), f_active=np.zeros(0, np.uint8)) for p in nxt]
        th, tb = [], []
        for i in range(warmup + reps):
            t0 = time.perf_counter()
            mh = s.marginalize(nxt, 1, resident=True, culled=bare)
            t1 = time.perf_counter()
            mb = s.marginalize_built(lean, 1)
            t2 = time.perf_counter()
            if i >= warmup:
                th.append((t1 - t0) * 1e3), tb.append((t2 - t1) * 1e3)
        same = all(x["m"] == y["m"] and x["r"] == y["r"] and x["J0"].tobytes() == y["J0"].tobytes() and x["e0"].tobytes() == y["e0"].tobytes()
                   for x, y in zip(mh, mb))
        host_up = B * (4 * (8 + 2 * K + L) + F)
        built_up, built_down = B * 120, B * 4 * (8 + 2 * K)
        prior_down = sum(8 * (2 * x["r"] * x["r"] + 2 * x["r"]) for x in mb)  # J0, e0, Hp, bp (used prefix of each window's slot)
        return dict(windows=B, K=K, L=L, F_cap=F, m_max=max(x["m"] for x in mb), r_max=max(x["r"] for x in mb), outputs_bitwise_equal=same,
                    host_list_marg_ms=float(np.median(th)), built_marg_ms=float(np.median(tb)), host_list_bytes_h2d=host_up, host_list_bytes_d2h=0,
                    built_bytes_h2d=built_up, built_bytes_d2h=built_down, prior_bytes_d2h_both=prior_down)
    finally:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_marg_built.py: no CUDA device; the product path has no CPU fallback")
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        plim = "unknown"
    card = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=plim)
    for B, K, L, F, R in ((296, 10, 300, 2700, 160), (128, 20, 2000, 12000, 292)):
        print(json.dumps(dict(card, **run(B, K, L, F, R, args.reps, args.warmup))), flush=True)


if __name__ == "__main__":
    main()
