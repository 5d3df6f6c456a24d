#!/usr/bin/env python
"""Cost of doReintegration on the device (icg_ba_reintegrate_resident) for B resident cfg-3 windows (K = 10, L = 300) right after
icg_ba_gvins_optimization, and of the plain batch propagation (icg_geom_imu_preintegrate_batch) on the same intervals.

    python scripts/bench_reintegration.py [--windows 296] [--reps 10] [--warmup 2]
    python scripts/bench_reintegration.py --batch-only --dump DIR [--reps 10]

Every window has 9 intervals of 100 samples at 200 Hz; its factors are linearised 8 gyro-bias sigmas away from the node biases, so that
every gate opens after the solve.  One JSON line:
  * the call with every gate open (the handle re-uploaded and re-solved before each repetition, outside the timing) and with every gate
    closed (the call right after one that reintegrated everything): CUDA events on the handle's stream and the host clock around the
    synchronous call;
  * preint_resident_kernel's time from a separate torch.profiler run;
  * icg_geom_imu_preintegrate_batch on the same B x 9 intervals (states from the solved windows), events + host clock, and its kernel time;
  * as an order of magnitude, the host icg_imu_preintegrate loop on a few windows, scaled to B;
  * multiply-adds per interval counted from the shapes: the dense 15 x 15 products of the scalar core and the ones the warp kernel keeps
    (phi's structural zeros left out);
  * the card name and power limit, read in the same run.
--batch-only uses the existing API only (Geometry.imu_preintegrate_batch), so that the same script measures an earlier tree; with --dump it
writes the batch's blobs and end states to DIR/batch_outputs.npz.  Writes nothing to the source tree.
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

N_DISTINCT = 16
SAMPLES = 100


def card(torch, dev):
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    return torch.cuda.get_device_name(dev), plim


def make_windows(B):
    """B cfg-3 windows (16 distinct ones repeated) and their IMU rows; deterministic, host preintegration of this library"""
    from datagen import synth_ba
    from ic_gvins_b200.ba import imu_preintegrate

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    base = []
    for i in range(min(N_DISTINCT, B)):
        p = synth_ba.make_window(pre, K=10, L=300, seed=8000 + i)[0]
        rng = np.random.default_rng(9000 + i)
        pose, mix, blobs, rows = p["pose"].reshape(10, 7), p["mix"].reshape(10, 9), p["imu_blob"].reshape(9, 480), []
        for k in range(9):
            imu = synth_ba.imu_samples(0.5 * k, 0.5 * k + SAMPLES / 200.0, 200.0, rng, mix[k, 3:6], mix[k, 6:9])
            st = np.concatenate([pose[k], mix[k]])
            st[10] += 8 * synth_ba.NOISE5[2]
            blobs[k] = imu_preintegrate(st, synth_ba.IEWN, synth_ba.GRAVITY, synth_ba.NOISE5, imu)[0]
            rows.append(imu)
        base.append((p, rows))
    probs = [copy.deepcopy(base[i % len(base)][0]) for i in range(B)]
    rows = [base[i % len(base)][1] for i in range(B)]
    return probs, rows


def batch_inputs(probs, rows):
    from datagen import synth_ba
    st = []
    for p in probs:
        pose, mix = p["pose"].reshape(p["K"], 7), p["mix"].reshape(p["K"], 9)
        for k in range(p["n_imu"]):
            q = pose[k, 3:7] / np.sqrt(np.sum(pose[k, 3:7] ** 2))
            st.append(np.concatenate([pose[k, :3], q, mix[k]]))
    return np.array(st), synth_ba.IEWN, [r for rw in rows for r in rw]


def timed(torch, cs, fn, reps, warmup, before=None):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(warmup):
        if before:
            before()
        fn()
    torch.cuda.synchronize()
    t_ev = t_host = 0.0
    for _ in range(reps):
        if before:
            before()
            torch.cuda.synchronize()
        ev[0].record(cs)
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        ev[1].record(cs)
        torch.cuda.synchronize()
        t_ev += ev[0].elapsed_time(ev[1])
        t_host += (t1 - t0) * 1e3
    return t_ev / reps, t_host / reps


def kernel_us(torch, fn, name, n=3):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    return sum(float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))) for e in prof.key_averages() if name in e.key) / n


def macs_per_interval():
    """multiply-adds of one sample's covariance / Jacobian update, times SAMPLES: the scalar core's dense products (phi jac, phi G, phi cov,
    cov' phi^T, G phi^T: 15^3 each; G = gt noise gt^T: 225 x 12 products of three) and the warp kernel's (phi's 45 non-zeros per column)"""
    nnz = 3 * 2 + 3 * 7 + 3 * 4 + 6 * 1
    dense = 5 * 15 ** 3 + 225 * 12 * 2
    sparse = 5 * nnz * 15 + 9 * 3 * 2
    return dense * SAMPLES, sparse * SAMPLES


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=296)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-windows", type=int, default=2)
    ap.add_argument("--batch-only", action="store_true")
    ap.add_argument("--dump", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_reintegration.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from ic_gvins_b200.geom import Geometry
    B = args.windows
    dev = torch.device("cuda:0")
    cs = torch.cuda.Stream(dev)
    torch.cuda.set_stream(cs)
    probs, rows = make_windows(B)
    gpu, plim = card(torch, dev)
    g = Geometry(stream=cs.cuda_stream)
    line = {"windows": B, "intervals": B * 9, "samples_per_interval": SAMPLES}

    if args.batch_only:  # the existing API only: the uploaded (unsolved) states
        st, iw, rl = batch_inputs(probs, rows)
        res = {}
        ms_ev, ms_host = timed(torch, cs, lambda: res.__setitem__("o", g.imu_preintegrate_batch(st, iw, synth_ba.GRAVITY, synth_ba.NOISE5, rl)),
                               args.reps, args.warmup)
        if args.dump:
            os.makedirs(args.dump, exist_ok=True)
            np.savez(os.path.join(args.dump, "batch_outputs.npz"), blobs=res["o"][0], ends=res["o"][1])
        line.update(metric="icg_geom_imu_preintegrate_batch, intervals/s", value=B * 9 / (ms_ev / 1e3), unit="intervals/s",
                    batch_ms_events=ms_ev, batch_ms_host=ms_host, gpu=gpu, power_limit_w=plim)
        print(json.dumps(line))
        g.close()
        return

    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate
    s = WindowSolver(max_windows=B, max_K=10, max_L=300, max_F=max(p["F"] for p in probs), max_gnss=8, max_marg_r=160, stream=cs.cuda_stream)
    s.gvins_optimization_batch(probs, 20)
    blobs0 = [p["imu_blob"].copy() for p in probs]
    solved = copy.deepcopy(probs)
    out = {}

    def restore():  # the factors as the solve saw them, re-solved from the same start: every gate open again
        for p, b in zip(probs, blobs0):
            p["imu_blob"][...] = b
        s.upload(probs)
        s.run_gvins(20, restart=True)

    call = lambda: out.__setitem__("o", s.reintegrate(probs, synth_ba.NOISE5, np.zeros(3), rows))
    ms_open_ev, ms_open_host = timed(torch, cs, call, args.reps, args.warmup, before=restore)
    opened = int(sum(o["count"] for o in out["o"]))
    ms_closed_ev, ms_closed_host = timed(torch, cs, call, args.reps, args.warmup)
    closed = int(sum(o["count"] for o in out["o"]))
    restore()
    kern_open = kernel_us(torch, call, "preint_resident_kernel", 1)
    # the plain batch on the same intervals, states from the solved windows
    st, iw, rl = batch_inputs(solved, rows)
    res = {}
    ms_b_ev, ms_b_host = timed(torch, cs, lambda: res.__setitem__("o", g.imu_preintegrate_batch(st, iw, synth_ba.GRAVITY, synth_ba.NOISE5, rl)),
                               args.reps, args.warmup)
    kern_batch = kernel_us(torch, lambda: g.imu_preintegrate_batch(st, iw, synth_ba.GRAVITY, synth_ba.NOISE5, rl), "preint_batch_kernel")
    # host reference: icg_imu_preintegrate interval by interval on a few windows, scaled to B
    nh = min(args.host_windows, B)
    t0 = time.perf_counter()
    for i in range(nh * 9):
        imu_preintegrate(st[i], iw, synth_ba.GRAVITY, synth_ba.NOISE5, rl[i])
    ms_host_window = (time.perf_counter() - t0) * 1e3 / nh
    dense, sparse = macs_per_interval()
    line.update(metric="doReintegration on the device, windows/s (every gate open)", value=B / (ms_open_ev / 1e3), unit="windows/s",
                reintegrated_open=opened, reintegrated_closed=closed, call_open_ms_events=ms_open_ev, call_open_ms_host=ms_open_host,
                call_closed_ms_events=ms_closed_ev, call_closed_ms_host=ms_closed_host, preint_resident_kernel_us=round(kern_open, 1),
                batch_ms_events=ms_b_ev, batch_ms_host=ms_b_host, preint_batch_kernel_us=round(kern_batch, 1),
                host_icg_imu_preintegrate_ms_per_window=ms_host_window, host_icg_imu_preintegrate_ms_scaled_to_B=ms_host_window * B,
                mac_per_interval_dense=dense, mac_per_interval_kernel=sparse, gpu=gpu, power_limit_w=plim)
    print(json.dumps(line))
    s.close()
    g.close()


if __name__ == "__main__":
    main()
