#!/usr/bin/env python
"""The new keyframe's IMU factor of B resident windows, preintegrated on the host or on the device, on the same inputs:

  host    icg_imu_preintegrate of the B new intervals on host threads (from the node states the solve wrote back), the blobs and node rows
          written into the next windows, then icg_ba_slide_resident
  device  icg_ba_slide_integrate_resident (the interval from the resident last node, the new node from its end state)

    python scripts/bench_slide_integrate.py [--windows 296] [--reps 10] [--warmup 2]

Cfg-3 windows (K = 10, L = 300) are solved and marginalized on the device; each next window drops node 0 and adds one node joined by one
new interval of 0.5 s at 200 Hz (101 samples) (datagen/slide_window.py).  The handle is put back into that state before every repetition,
outside the timing, and the two paths alternate.  The host path is handed the Earth-rate vectors the device computed (the only input it
would otherwise have to form itself), so both paths produce the same bits, which is checked.  One JSON line: the median wall time of
each call up to a device synchronise, the host preintegration alone, and the card name and power limit read in the same run.  Writes
nothing to the source tree.
"""
from __future__ import annotations

import argparse
import copy
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_DISTINCT = 8


def card(torch, dev):
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    return torch.cuda.get_device_name(dev), plim


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=296)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_slide_integrate.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from datagen.slide_window import build_next
    from ic_gvins_b200._lib import BaProblem, SlideIntegrate, SlideWindow, check, lib, u8p
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate, to_struct
    B, K, L, iters = args.windows, 10, 300, 20
    dev = torch.device("cuda:0")
    cs = torch.cuda.Stream(dev)
    torch.cuda.set_stream(cs)
    gpu, plim = card(torch, dev)

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    base = [synth_ba.make_window(pre, K=K, L=L, seed=8300 + i)[0] for i in range(min(N_DISTINCT, B))]
    probs0 = [copy.deepcopy(base[i % len(base)]) for i in range(B)]
    F = max(p["F"] for p in probs0) + 64
    s = WindowSolver(max_windows=B, max_K=K, max_L=L, max_F=F, max_gnss=16, max_marg_r=160, stream=cs.cuda_stream)
    solved = copy.deepcopy(probs0)
    s.gvins_optimization_batch(solved, iters)
    marg = s.marginalize(solved, 1, resident=True)
    built = [build_next(p, 9100 + w, prior=m) for w, (p, m) in enumerate(zip(solved, marg))]
    nxt, carries = [x[1] for x in built], [x[2] for x in built]
    rng = np.random.default_rng(9300)
    rows = [np.ascontiguousarray(synth_ba.imu_samples(0.5 * (K - 1), 0.5 * K, 200.0, rng, p["mix"][-9:][3:6], p["mix"][-9:][6:9]))
            for p in solved]
    k_new = K - 2  # the factor that joins the old last node (new node K - 2) and the new node K - 1
    starts = []
    for p in solved:
        pose, mix = p["pose"].reshape(K, 7)[K - 1], p["mix"].reshape(K, 9)[K - 1]
        x, y, z, w = pose[3:7]
        n = np.sqrt(((x * x + y * y) + z * z) + w * w)
        starts.append(np.concatenate([pose[:3], [x / n, y / n, z / n, w / n], mix]))

    def restore():  # the handle right after the solve and the resident marginalization of the current windows
        s.upload(copy.deepcopy(probs0))
        s.run_gvins(iters)
        s.sync()
        s.marginalize(solved, 1, resident=True)

    L_ = lib()
    cw = (SlideWindow * B)()
    keep = []  # the arrays the struct arrays point into
    for w, c in enumerate(carries):
        for k in ("node_src", "lm_src", "f_src", "imu_src", "gnss_src"):
            setattr(cw[w], k, c[k].ctypes.data_as(C.POINTER(C.c_int32)))
        cw[w].prior_from_marg = 1
    # the device path's arguments
    iw = (SlideIntegrate * B)()
    dev_blobs = np.zeros((B, K - 1, 480))
    status = np.zeros((B, K - 1), np.int8)
    for w in range(B):
        src = np.full(K - 1, -1, np.int32)
        src[k_new] = K - 1
        off = np.zeros(K, np.int32)
        off[k_new + 1:] = len(rows[w])
        node = np.zeros(K, np.uint8)
        node[K - 1] = 1
        grav = np.tile(synth_ba.GRAVITY, (K - 1, 1))
        keep += [src, off, node, grav]
        iw[w].imu_from, iw[w].imu_off = src.ctypes.data_as(C.POINTER(C.c_int32)), off.ctypes.data_as(C.POINTER(C.c_int32))
        iw[w].imu, iw[w].gravity3 = rows[w].ctypes.data_as(C.POINTER(C.c_double)), grav.ctypes.data_as(C.POINTER(C.c_double))
        iw[w].node_from_imu = node.ctypes.data_as(u8p)
        iw[w].status, iw[w].blob_out = status[w].ctypes.data_as(C.POINTER(C.c_int8)), dev_blobs[w].ctypes.data_as(C.POINTER(C.c_double))
    nz = np.ascontiguousarray(synth_ba.NOISE5)
    stn = np.zeros(3)
    out = {}

    def fresh():
        restore()
        out["q"] = copy.deepcopy(nxt)
        out["arr"] = (BaProblem * B)(*[to_struct(q) for q in out["q"]])

    def device():
        check(L_.icg_ba_slide_integrate_resident(s._h, B, out["arr"], cw, iw, nz.ctypes.data, stn.ctypes.data), "icg_ba_slide_integrate_resident")
        torch.cuda.synchronize()

    fresh()
    device()
    assert (status[:, k_new] == 1).all()
    iewn = [np.ascontiguousarray(dev_blobs[w, k_new, 20:23]) for w in range(B)]
    ends = np.zeros((B, 10))
    pool = ThreadPoolExecutor(max_workers=max(1, min(16, os.cpu_count() or 1)))

    def host_one(w):
        q = out["q"][w]
        blob = q["imu_blob"].reshape(-1, 480)[k_new]
        check(L_.icg_imu_preintegrate(starts[w].ctypes.data, iewn[w].ctypes.data, synth_ba.GRAVITY.ctypes.data, nz.ctypes.data, rows[w].ctypes.data,
                                      len(rows[w]), blob.ctypes.data, ends[w].ctypes.data), "icg_imu_preintegrate")
        q["pose"].reshape(K, 7)[K - 1] = ends[w, :7]
        q["mix"].reshape(K, 9)[K - 1] = np.r_[ends[w, 7:10], starts[w][10:16]]

    host_pre = []

    def host():
        t0 = time.perf_counter()
        list(pool.map(host_one, range(B)))
        host_pre.append((time.perf_counter() - t0) * 1e3)
        check(L_.icg_ba_slide_resident(s._h, B, out["arr"], cw), "icg_ba_slide_resident")
        torch.cuda.synchronize()

    times = {"host": [], "device": []}
    for r in range(args.warmup + args.reps):
        for name, fn in (("host", host), ("device", device)) if r % 2 == 0 else (("device", device), ("host", host)):
            fresh()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            t = (time.perf_counter() - t0) * 1e3
            if r >= args.warmup:
                times[name].append(t)
            check(L_.icg_ba_download(s._h, B, out["arr"], None), "icg_ba_download")  # the gathered node rows, into out["q"]
            out[name] = [(q["pose"].copy(), q["mix"].copy()) for q in out["q"]]
            if name == "host":
                out["host_blobs"] = np.array([q["imu_blob"].reshape(-1, 480)[k_new] for q in out["q"]])
    equal = np.array_equal(out["host_blobs"], dev_blobs[:, k_new]) and all(
        np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(out["host"], out["device"]))
    pool.shutdown()
    line = {"metric": "new keyframe interval + slide, host preintegration vs device (ms per call, B windows, median)", "cfg": 3, "windows": B,
            "samples_per_interval": len(rows[0]), "host_path_ms": statistics.median(times["host"]),
            "device_path_ms": statistics.median(times["device"]), "host_preintegration_ms": statistics.median(host_pre[args.warmup:]),
            "host_threads": pool._max_workers, "reps": args.reps, "outputs_array_equal": bool(equal), "gpu": gpu, "power_limit_w": plim}
    print(json.dumps(line))
    s.close()


if __name__ == "__main__":
    main()
