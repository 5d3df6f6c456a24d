#!/usr/bin/env python
"""Cost of starting the next keyframe's solve on B resident windows: (a) the full re-pack and upload (icg_ba_gvins_optimization_begin / _end
on the next windows) against (b) icg_ba_slide_resident + icg_ba_run_gvins + _end, on the same next windows.

    python scripts/bench_slide.py [--windows 296] [--reps 20] [--warmup 3]        # cfg 3: K = 10, L = 300 (fused single-GPU pipeline)
    python scripts/bench_slide.py --cfg4 [--windows 128]                          # cfg 4: K = 20, L = 2000, max_marg_r = 292 (split pipeline)

Every window is solved (icg_ba_gvins_optimization) and marginalized on the device (icg_ba_marginalize_resident, num_marg = 1); its next
window drops node 0 with the landmarks anchored there, adds one node (IMU factor, GNSS fix), re-anchors one landmark and adds three that
observe the new node (datagen/slide_window.py).  Before every repetition of (b) the handle is put back into that state, outside the timing.
The C entry points are called on struct arrays built outside the timing, as a C++ caller keeps them.  One JSON line:
  * per call: the upload or the slide alone, and the whole step (upload or slide, both passes, write-back), as CUDA events on the handle's
    stream and as a host clock that ends in a synchronise;
  * the H2D bytes of both paths, computed from the array shapes;
  * ba_slide_gather and ba_slide_prior kernel times from a separate torch.profiler run;
  * whether the two paths' outputs (summaries, parameters, f_active, gnss_std) are np.array_equal;
  * the card name and power limit, read in the same run.
Writes nothing to the source tree.
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

N_DISTINCT = 8
PARAMS = ("pose", "mix", "ext", "invdepth", "f_active", "gnss_std")


def card(torch, dev):
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    return torch.cuda.get_device_name(dev), plim


def make_windows(B, K, L, n_ref):
    from datagen import synth_ba
    from ic_gvins_b200.ba import imu_preintegrate

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    kw = dict(n_ref=n_ref) if n_ref else {}
    base = [synth_ba.make_window(pre, K=K, L=L, seed=8100 + i, **kw)[0] for i in range(min(N_DISTINCT, B))]
    return [copy.deepcopy(base[i % len(base)]) for i in range(B)]


def h2d_bytes(caps, nxt, carries, slide):
    """bytes icg_ba_upload (slide = False) or icg_ba_slide_resident (slide = True) moves host -> device for these next windows"""
    K, L, F, G, R, NVB = caps
    PM = K * (K - 1)
    n = len(nxt)
    structure = n * (64 + 64 + F + 16 * F + 4 * NVB + 4 * (L + 1) + 4 * L + 4 * K + 4 * (PM + 1) + 4 * PM + 4 * F + 4 + 4 * G + 24 + 56 + 48 + 72 + 72
                     + 2 * 4 * 72 + 8 * 72 * 9)
    if not slide:
        return structure + n * (56 * K + 72 * K + 8 * L + 112 * F + 8 * 480 * K + 8 * 225 * K + 48 * G + 8 * R * R + 8 * R + 8)
    al = lambda b: (b + 15) & ~15
    maps = sum(q["K"] + q["L"] + q["F"] + q["n_imu"] + q["n_gnss"] for q in nxt)
    vals = 0
    for q, c in zip(nxt, carries):
        vals += 16 * int((c["node_src"] < 0).sum()) + int((c["lm_src"] < 0).sum()) + 14 * int((c["f_src"] < 0).sum())
        vals += 705 * int((c["imu_src"] < 0).sum()) + 6 * int((c["gnss_src"] < 0).sum())
    return structure + al(48 * n) + al(4 * maps) + 8 * vals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=None)
    ap.add_argument("--cfg4", action="store_true")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_slide.py: no CUDA device; the product path has no CPU fallback")
    import ctypes as C

    from datagen.slide_window import build_next
    from ic_gvins_b200._lib import BaProblem, BaSummary, SlideWindow, check, lib
    from ic_gvins_b200.ba import WindowSolver, to_struct
    K, L, R, n_ref, iters = (20, 2000, 292, 20, 12) if args.cfg4 else (10, 300, 160, 0, 20)
    B = args.windows or (128 if args.cfg4 else 296)
    dev = torch.device("cuda:0")
    cs = torch.cuda.Stream(dev)
    torch.cuda.set_stream(cs)
    gpu, plim = card(torch, dev)
    probs0 = make_windows(B, K, L, n_ref)
    F = max(p["F"] for p in probs0) + 64
    s = WindowSolver(max_windows=B, max_K=K, max_L=L, max_F=F, max_gnss=16, max_marg_r=R, stream=cs.cuda_stream)
    solved = copy.deepcopy(probs0)
    s.gvins_optimization_batch(solved, iters)
    marg = s.marginalize(solved, 1, resident=True)
    nxt = [build_next(p, 9000 + w, prior=m) for w, (p, m) in enumerate(zip(solved, marg))]
    up0, slid0, carries = [x[0] for x in nxt], [x[1] for x in nxt], [x[2] for x in nxt]

    def restore():  # the handle right after the solve and the resident marginalization of the current windows
        s.upload(copy.deepcopy(probs0))
        s.run_gvins(iters)
        s.sync()
        s.marginalize(solved, 1, resident=True)

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn, before):
        for _ in range(args.warmup):
            before()
            fn()
        torch.cuda.synchronize()
        t_ev = t_host = 0.0
        for _ in range(args.reps):
            before()
            torch.cuda.synchronize()
            ev[0].record(cs)
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            ev[1].record(cs)
            torch.cuda.synchronize()
            t_ev += ev[0].elapsed_time(ev[1])
            t_host += (t1 - t0) * 1e3
        return t_ev / args.reps, t_host / args.reps

    # the C calls on struct arrays built outside the timing (what a C++ caller keeps across keyframes): the times are the library's
    L_ = lib()
    cw = (SlideWindow * B)()
    for w, c in enumerate(carries):
        for k in ("node_src", "lm_src", "f_src", "imu_src", "gnss_src"):
            setattr(cw[w], k, c[k].ctypes.data_as(C.POINTER(C.c_int32)))
        cw[w].prior_from_marg = 1
    summ, culled = (BaSummary * (2 * B))(), (C.c_int32 * (2 * B))()
    out = {}

    def fresh(src):  # untimed: the handle's state before the step and a fresh copy of the next windows (the step writes its results into it)
        def f():
            restore()
            out["q"] = copy.deepcopy(src)
            out["arr"] = (BaProblem * B)(*[to_struct(q) for q in out["q"]])
        return f

    results = lambda: [(x.iterations, x.num_successful_steps, x.termination, x.initial_cost, x.final_cost, x.final_radius) for x in summ]

    def step_a():
        check(L_.icg_ba_gvins_optimization(s._h, B, out["arr"], iters, summ, culled), "icg_ba_gvins_optimization")
        out["a"] = (out["q"], results(), list(culled))

    def step_b():
        check(L_.icg_ba_slide_resident(s._h, B, out["arr"], cw), "icg_ba_slide_resident")
        check(L_.icg_ba_run_gvins(s._h, iters, 0), "icg_ba_run_gvins")
        check(L_.icg_ba_gvins_optimization_end(s._h, B, out["arr"], summ, culled), "icg_ba_gvins_optimization_end")
        out["b"] = (out["q"], results(), list(culled))

    upload_ms = timed(lambda: check(L_.icg_ba_upload(s._h, B, out["arr"]), "icg_ba_upload"), fresh(up0))
    step_a_ms = timed(step_a, fresh(up0))
    slide_ms = timed(lambda: check(L_.icg_ba_slide_resident(s._h, B, out["arr"], cw), "icg_ba_slide_resident"), fresh(slid0))
    step_b_ms = timed(step_b, fresh(slid0))
    qa, ra, ca = out["a"]
    qb, rb, cb = out["b"]
    equal = ra == rb and ca == cb and all(np.array_equal(x[k], y[k]) for x, y in zip(qa, qb) for k in PARAMS)
    # kernel times, profiled in a run of their own
    from torch.profiler import ProfilerActivity, profile
    restore()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.slide(copy.deepcopy(slid0), carries, True)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for name in ("ba_slide_gather", "ba_slide_prior"):
            if name in e.key:
                kern[name + "_us"] = round(float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))), 1)
    NVB = (F + 127 - K) // (128 - K) + L // 128 + 4 + K
    caps = (K, L, F, 16, R, NVB)
    line = {"metric": "next-window start, slide vs re-upload (ms per call, B windows)", "cfg": 4 if args.cfg4 else 3, "windows": B,
            "upload_ms_events": upload_ms[0], "upload_ms_host": upload_ms[1], "slide_ms_events": slide_ms[0], "slide_ms_host": slide_ms[1],
            "step_upload_ms_events": step_a_ms[0], "step_upload_ms_host": step_a_ms[1], "step_slide_ms_events": step_b_ms[0],
            "step_slide_ms_host": step_b_ms[1], "h2d_bytes_upload": h2d_bytes(caps, up0, carries, False),
            "h2d_bytes_slide": h2d_bytes(caps, up0, carries, True), **kern, "outputs_array_equal": bool(equal), "gpu": gpu, "power_limit_w": plim}
    print(json.dumps(line))
    s.close()


if __name__ == "__main__":
    main()
