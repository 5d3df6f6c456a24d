#!/usr/bin/env python
"""Cost of the resident marginalization (icg_ba_marginalize_resident) of cfg-4 windows (K = 20, L = 2000) on one H100, per eigensolver kernel.

    python scripts/bench_marg_large.py [--windows 64] [--windows3 128] [--reps 10] [--warmup 2]

Workloads (a few distinct synthetic windows repeated to fill the batch, solved once with icg_ba_gvins_optimization, then marginalized
repeatedly; the marginalization leaves the handle as it found it):
  * cfg 4 windows carrying a 292-row prior over nodes 0..18, the extrinsic and td (the span a sliding window's prior reaches after a few
    slides; tests/test_marg_large_gpu.py: window_prior), so that Hp has r = 277 rows (the 8-CTA cluster kernel):
      default anchoring (landmark j in node j mod 5): m ~ 410 (Hmm on the global-memory kernel);
      anchors spread over 19 nodes (n_ref = 20): m ~ 120 (Hmm on the cluster pair);
  each with the default dispatch and with ICG_MARG_GLOBAL_JACOBI=1 (both blocks on the global-memory kernel);
  * cfg 3 (K = 10, L = 300): the default dispatch (one CTA / cluster pair) against ICG_MARG_CLUSTER_JACOBI=1 (both blocks on the cluster).
Each variant: the host clock around the synchronous call (it ends in a stream synchronise and the copies into the caller's arrays); the
variants of one workload alternate rep by rep.  Medians over the reps, and windows/s from the median.  The card name and power limit are read
in the same run.  One JSON line.  Writes nothing to the source tree.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=64, help="cfg-4 windows per batch")
    ap.add_argument("--windows3", type=int, default=128, help="cfg-3 windows per batch")
    ap.add_argument("--distinct", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_marg_large.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate
    from tests.test_marg_large_gpu import window_prior

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    def batch(n, d, prior=False, **kw):
        base = []
        for i in range(min(d, n)):
            p, truth = synth_ba.make_window(pre, seed=8000 + i, **kw)
            base.append(window_prior(p, truth, 9000 + i) if prior else p)
        return [copy.deepcopy(base[i % len(base)]) for i in range(n)]

    def timed(s, probs, variants):
        """variants: {name: env var or None}; returns {name: (median ms, all ms, m max, r max)}"""
        def call(env):
            if env:
                os.environ[env] = "1"
            try:
                t0 = time.perf_counter()
                out = s.marginalize(probs, 1, resident=True)
                return (time.perf_counter() - t0) * 1e3, out
            finally:
                if env:
                    del os.environ[env]
        for _ in range(args.warmup):
            for env in variants.values():
                call(env)
        ts = {k: [] for k in variants}
        dims = {}
        for _ in range(args.reps):
            for k, env in variants.items():
                t, out = call(env)
                ts[k].append(t)
                dims[k] = (max(o["m"] for o in out), max(o["r"] for o in out))
        return {k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3),
                        windows_per_s=round(len(probs) / (statistics.median(v) / 1e3), 1), m_max=dims[k][0], r_max=dims[k][1])
                for k, v in ts.items()}

    res = {}
    B4 = args.windows
    w4 = {"default_anchors": batch(B4, args.distinct, prior=True, K=20, L=2000),
          "spread_anchors": batch(B4, args.distinct, prior=True, K=20, L=2000, n_ref=20)}
    s = WindowSolver(max_windows=B4, max_K=20, max_L=2000, max_F=max(p["F"] for v in w4.values() for p in v), max_gnss=16, max_marg_r=292)
    for name, probs in w4.items():
        s.gvins_optimization_batch(probs, 20)
        res["cfg4_" + name] = timed(s, probs, {"default": None, "global": "ICG_MARG_GLOBAL_JACOBI"})
    s.close()
    B3 = args.windows3
    p3 = batch(B3, args.distinct, K=10, L=300)
    s = WindowSolver(max_windows=B3, max_K=10, max_L=300, max_F=max(p["F"] for p in p3), max_gnss=16, max_marg_r=160)
    s.gvins_optimization_batch(p3, 20)
    res["cfg3"] = timed(s, p3, {"default": None, "cluster": "ICG_MARG_CLUSTER_JACOBI"})
    s.close()
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True,
                           text=True, timeout=10).stdout.strip()
    except Exception:
        q = None
    line = {"metric": "resident marginalization of cfg-4 windows, windows/s (default dispatch, default anchoring)",
            "value": res["cfg4_default_anchors"]["default"]["windows_per_s"], "unit": "windows/s", "windows_cfg4": B4, "windows_cfg3": B3,
            "reps": args.reps, "results": res, "gpu": torch.cuda.get_device_name(0), "power_limit_w,max_sm_clock_mhz": q}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
