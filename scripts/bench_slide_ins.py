#!/usr/bin/env python
"""One keyframe of B resident windows whose IMU samples live in device INS windows, by two routes on the same inputs:

  host    every stream's INS window downloaded (icg_ins_window), the new interval cut on the host (getImuSeriesFromTo in numpy), then
          icg_ba_slide_integrate_resident with those rows and icg_ba_reintegrate_resident with every factor's rows the host keeps
  device  icg_ba_slide_ins_resident (the new interval cut on the device, the carried factors' rows kept in the handle's store), then
          icg_ba_reintegrate_stored_resident

    python scripts/bench_slide_ins.py [--windows 296] [--reps 10] [--warmup 2]

Cfg-3 windows (K = 10, L = 300) are solved and marginalized on the device; each next window drops node 0 and adds one node joined by one
new interval of 0.5 s of 200 Hz samples.  The handle is put back into that state (and its sample store seeded) before every repetition,
outside the timing, and the two routes alternate.  Both routes must leave the same blobs and the same reintegration results, which is
checked, and the device store must hold the host's rows.  One JSON line: the median wall time of each route up to a device synchronise
(Python wrappers included on both sides), and the card name and power limit read in the same run.  Writes nothing to the source tree.
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

N_DISTINCT = 8
MIN_DT = 1e-4  # MISC::MINIMUM_TIME_INTERVAL


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=10).stdout.strip()
    except Exception:
        q = None
    return q


def window_index(T, t):
    """MISC::getInsWindowIndex: the first entry whose time is greater than t; 0 before the front or at / after the back"""
    if len(T) == 0 or T[0] > t or T[-1] <= t:
        return 0
    return int(np.searchsorted(T, t, side="right"))


def need(a, b, t):
    if a[0] < t and b[0] > t:
        return -1 if t - a[0] < MIN_DT else 1 if b[0] - t < MIN_DT else 2
    return 0


def split(row, t):
    scale = (row[0] - t) / row[1]
    first, second = row.copy(), row.copy()
    first[0], first[1], first[2:] = t, row[1] - (row[0] - t), row[2:] * (1 - scale)
    second[0], second[1], second[2:] = row[0], row[0] - t, row[2:] * scale
    return first, second


def series(W, start, end):
    """MISC::getImuSeriesFromTo on window rows W (n x 8): rows (dt, dtheta, dvel)"""
    T = W[:, 0]
    i_s, i_e = window_index(T, start), window_index(T, end)
    assert i_s and i_e
    out = []
    c = need(W[i_s - 1], W[i_s], start)
    if c == -1:
        out += [W[i_s - 1], W[i_s]]
    elif c == 1:
        out += [W[i_s]]
    elif c == 2:
        out += list(split(W[i_s], start))
    out += [W[k] for k in range(i_s + 1, i_e - 1)]
    c = need(W[i_e - 1], W[i_e], end)
    if c == -1:
        out += [W[i_e - 1]]
    elif c == 1:
        out += [W[i_e - 1], W[i_e]]
    elif c == 2:
        out += [W[i_e - 1], split(W[i_e], end)[0]]
    return np.ascontiguousarray(np.array(out)[:, 1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=296)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_slide_ins.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from datagen.slide_window import build_next
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate
    from ic_gvins_b200.ins import InsWindow
    B, K, L, iters = args.windows, 10, 300, 20
    gpu = card()

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    # INS windows: 200 Hz rows 10.0 .. 15.5 s per stream, mechanized by a redo near the front
    ins = InsWindow(B, capacity=2000)
    cfg = [{"with_earth": w % 2 == 0, "gravity": synth_ba.GRAVITY} for w in range(B)]
    rng = np.random.default_rng(9400)
    rows8 = []
    for w in range(B):
        r = synth_ba.imu_samples(10.0, 15.5, 200.0, rng, np.zeros(3), np.zeros(3), earth=cfg[w]["with_earth"])
        rows8.append(np.concatenate([(10.0 + 0.005 * np.arange(len(r)))[:, None], r], axis=1))
    ins.push([r[:1000] for r in rows8], cfg)  # a window that was never redone keeps its newest 1000 rows
    st = np.zeros((B, 17))
    st[:, 7], st[:, 0] = 1, 10.011
    assert (ins.redo(st, cfg) == 1).all()
    ins.push([r[1000:] for r in rows8], cfg)
    t_old = 10.0507 + 0.5 * np.arange(K)
    t_new = np.r_[t_old[1:], t_old[-1] + 0.5]
    host_rows = [[series(ins.window(w)[0], t_old[k], t_old[k + 1]) for k in range(K - 1)] for w in range(B)]  # kept by the host route

    base = [synth_ba.make_window(pre, K=K, L=L, seed=8300 + i)[0] for i in range(min(N_DISTINCT, B))]
    probs0 = [copy.deepcopy(base[i % len(base)]) for i in range(B)]
    F = max(p["F"] for p in probs0) + 64
    s = WindowSolver(max_windows=B, max_K=K, max_L=L, max_F=F, max_gnss=16, max_marg_r=160)
    solved = copy.deepcopy(probs0)
    s.gvins_optimization_batch(solved, iters)
    marg = s.marginalize(solved, 1, resident=True)
    built = [build_next(p, 9100 + w, prior=m) for w, (p, m) in enumerate(zip(solved, marg))]
    nxt, carries = [x[1] for x in built], [x[2] for x in built]
    k_new = K - 2
    src = np.full(K - 1, -1, np.int32)
    src[k_new] = K - 1
    node = np.zeros(K, np.uint8)
    node[K - 1] = 1
    nz = synth_ba.NOISE5
    streams = list(range(B))

    def restore():  # the handle right after the solve and the resident marginalization, its store seeded from the INS windows
        s.upload(copy.deepcopy(probs0))
        s.run_gvins(iters)
        s.sync()
        s.marginalize(solved, 1, resident=True)
        s.imu_samples_from_ins(ins, streams, [t_old] * B)
        torch.cuda.synchronize()

    out = {}

    def host():
        new = [series(ins.window(w)[0], t_new[k_new], t_new[k_new + 1]) for w in range(B)]
        integ = [dict(imu_from=src, imu_rows=[None] * k_new + [new[w]], gravity=synth_ba.GRAVITY, normal=not cfg[w]["with_earth"],
                      node_from_imu=node) for w in range(B)]
        q = copy.deepcopy(nxt)
        sl = s.slide_integrate(q, carries, integ, nz)
        reint = s.reintegrate(q, nz, np.zeros(3), [host_rows[w][1:] + [new[w]] for w in range(B)])
        torch.cuda.synchronize()
        out["host"] = (sl, reint, new)

    def device():
        integ = [dict(imu_from=src, gravity=synth_ba.GRAVITY, normal=not cfg[w]["with_earth"], node_from_imu=node) for w in range(B)]
        q = copy.deepcopy(nxt)
        sl = s.slide_ins(q, carries, integ, ins, streams, [t_new] * B, None, nz)
        reint = s.reintegrate_stored(q, nz)
        torch.cuda.synchronize()
        out["device"] = (sl, reint)

    times = {"host": [], "device": []}
    for r in range(args.warmup + args.reps):
        for name, fn in (("host", host), ("device", device)) if r % 2 == 0 else (("device", device), ("host", host)):
            restore()
            t0 = time.perf_counter()
            fn()
            t = (time.perf_counter() - t0) * 1e3
            if r >= args.warmup:
                times[name].append(t)
            if name == "device":
                out["store"] = [s.imu_samples(w) for w in (0, B - 1)]
    (hs, hr, new), (ds, dr) = out["host"], out["device"]
    # equal_nan: the reintegration's blob arrays start from next's blobs, whose carried rows are NaN (the slide never reads them)
    equal = all(np.array_equal(a[k], b[k], equal_nan=True) for a, b in zip(hs, ds) for k in ("status", "blobs", "end_states"))
    equal = equal and all(np.array_equal(a[k], b[k], equal_nan=True) for a, b in zip(hr, dr) for k in ("status", "blobs", "end_states"))
    for i, w in enumerate((0, B - 1)):
        stored = out["store"][i]
        equal = equal and all(np.array_equal(stored[k], host_rows[w][k + 1]) for k in range(K - 2)) and np.array_equal(stored[k_new], new[w])
    line = {"metric": "new keyframe slide + reintegration, host-cut rows vs device store (ms per call, B windows, median)", "cfg": 3,
            "windows": B, "K": K, "imu_rate_hz": 200, "host_route_ms": statistics.median(times["host"]),
            "device_route_ms": statistics.median(times["device"]), "reps": args.reps, "outputs_array_equal": bool(equal),
            "reintegrated_factors": int(sum((x["status"] == 1).sum() for x in dr)), "gpu_name_power_limit": gpu}
    print(json.dumps(line))
    s.close(), ins.close()


if __name__ == "__main__":
    main()
