#!/usr/bin/env python
"""Cost of the post-solve map update + outlier culling (icg_ba_update_and_cull_resident) and of the marginalization of the culled map
(icg_ba_marginalize_resident_culled) on one H100, for B resident cfg-3 windows (K = 10, L = 300) right after icg_ba_gvins_optimization.

    python scripts/bench_post_solve.py [--windows 296] [--reps 20] [--warmup 3]

One JSON line:
  * the cull call: CUDA events on the handle's stream around the synchronous call (host packing of the observation lists, one H2D, the
    kernel, one D2H, the copies into the caller's arrays), and the host clock around it; ba_update_cull's kernel time from a separate
    torch.profiler run;
  * the culled resident marginalization against the existing resident marginalization (host clock around the synchronous calls);
  * as an order-of-magnitude reference, the same update + culling done on the host by the scalar numpy restatement
    (tests/post_solve_oracle.py) on downloaded arrays, timed on a few windows and scaled to B.
Windows: 16 distinct synthetic windows with 20 pixel outliers in their factor rows and 20 displaced keypoints in their observation lists,
repeated to fill the batch.  The card name and power limit are read in the same run.  Writes nothing to the source tree.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=296)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-windows", type=int, default=4)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_post_solve.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate
    from ic_gvins_b200.camera import Camera
    from tests import post_solve_oracle as po
    from tests.test_post_solve_gpu import CAMD, STD, cull_inputs

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    B = args.windows
    base = []
    for i in range(min(16, B)):
        p = synth_ba.make_window(pre, K=10, L=300, seed=5000 + i)[0]
        rng = np.random.default_rng(6000 + i)
        rows = rng.choice(p["F"], size=20, replace=False)
        p["f_const"].reshape(-1, 14)[rows, 3] += rng.choice([-1, 1], 20) * rng.uniform(3, 40, 20) / synth_ba.F_PIX
        base.append(p)
    probs = [copy.deepcopy(base[i % len(base)]) for i in range(B)]
    ext0 = [p["ext"].copy() for p in probs]
    dev = torch.device("cuda:0")
    cs = torch.cuda.Stream(dev)  # the handle runs on this stream, so that the events bracket its work
    torch.cuda.set_stream(cs)
    s = WindowSolver(max_windows=B, max_K=10, max_L=300, max_F=max(p["F"] for p in probs), max_gnss=8, max_marg_r=160, stream=cs.cuda_stream)
    s.gvins_optimization_batch(probs, 20)
    cis = [cull_inputs(p, e, 7000 + (i % len(base)), bad_kp=20) for i, (p, e) in enumerate(zip(probs, ext0))]
    cam = Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0] * 4)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        t_ev = t_host = 0.0
        for _ in range(args.reps):
            ev[0].record(cs)
            t0 = time.perf_counter()
            fn()
            t1 = time.perf_counter()
            ev[1].record(cs)
            torch.cuda.synchronize()
            t_ev += ev[0].elapsed_time(ev[1])
            t_host += (t1 - t0) * 1e3
        return t_ev / args.reps, t_host / args.reps

    out = {}
    cull = lambda: out.__setitem__("g", s.update_and_cull(probs, cam, STD, cis))
    ms_cull_ev, ms_cull_host = timed(cull)
    g = out["g"]
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            cull()
        torch.cuda.synchronize()
    kern_us = sum(float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))) for e in prof.key_averages() if "ba_update_cull" in e.key) / 5
    _, ms_marg = timed(lambda: s.marginalize(probs, 1, resident=True))
    _, ms_marg_culled = timed(lambda: s.marginalize(probs, 1, resident=True, culled=g))
    # host reference: the scalar numpy restatement on downloaded arrays (a few windows, scaled to B)
    nh = min(args.host_windows, B)
    t0 = time.perf_counter()
    for i in range(nh):
        po.update_and_cull(probs[i], CAMD, STD, cis[i])
    ms_host_per_window = (time.perf_counter() - t0) * 1e3 / nh
    n_obs = int(sum(int(c["obs_off"][-1]) for c in cis))
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    line = {"metric": "post-solve update + outlier culling on the device, windows/s", "value": B / (ms_cull_ev / 1e3), "unit": "windows/s",
            "windows": B, "observations": n_obs, "cull_ms_per_call_events": ms_cull_ev, "cull_ms_per_call_host": ms_cull_host,
            "ba_update_cull_kernel_us": round(kern_us, 1), "marginalize_resident_ms": ms_marg, "marginalize_resident_culled_ms": ms_marg_culled,
            "host_numpy_ms_per_window": ms_host_per_window, "host_numpy_ms_scaled_to_B": ms_host_per_window * B,
            "counts_sum": np.sum([x["counts"] for x in g], axis=0).tolist(), "ext_accepted": int(sum(x["ext_accepted"] == 1 for x in g)),
            "gpu": torch.cuda.get_device_name(dev), "power_limit_w": plim}
    print(json.dumps(line))
    s.close()


if __name__ == "__main__":
    main()
