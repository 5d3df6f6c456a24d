#!/usr/bin/env python
"""Cost of starting B streams' GNSS/INS states (gvinsInitialization, IG/ic_gvins.cc:584-692) on the device, against the route a B-stream
user had before icg_ins_gins_initialize existed.

    python scripts/bench_gins_init.py [--streams 296] [--reps 7]

Each stream holds 3 s of 200 Hz IMU rows (an unmechanized window) and one GNSS interval of 1 s inside it; half the streams use the Earth
form, half the Normal form.  Per repetition, on fresh windows:
  * device:  one icg_ins_gins_initialize call for all B streams (synchronous: the host clock around it is the whole cost);
  * host route, each segment timed on its own: icg_ins_window per stream (a synchronous download); the zero-velocity test, alignment,
    constructPrior and getImuSeriesFromTo on the host (the CPU restatement, tests/gins_init_oracle.cpp, one core, fed all downloaded
    windows at once -- it also redoes its own copy of each window, so this segment is an upper bound); icg_ins_redo for the B streams;
    the first node's preintegration of each series with the product's host core (icg_imu_preintegrate).  host_route_ms is their sum.
One JSON line with the medians, the card name and power limit read in the same run.  Writes nothing to the source tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(torch, dev):
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    return torch.cuda.get_device_name(dev), plim


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=296)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_gins_init: no CUDA device")
    from datagen import synth_ba
    from ic_gvins_b200.ba import imu_preintegrate
    from ic_gvins_b200.ins import InsWindow
    from tests import gins_init_oracle as go
    from tests.test_oracle_gins_init import GYR_BIAS_STD, init, moving

    B = a.streams
    cfg = [{"with_earth": s % 2 == 0, "gravity": synth_ba.GRAVITY} for s in range(B)]
    rows = [moving(10.0 + 0.013 * s, 13.0 + 0.013 * s, seed=s, earth=cfg[s]["with_earth"]) for s in range(B)]
    inits = [init(11.0023 + 0.013 * s, 12.0023 + 0.013 * s) for s in range(B)]
    noise5, station = synth_ba.NOISE5, np.zeros(3)

    def fresh():
        d = InsWindow(B)
        d.push(rows, cfg)
        d.sync()
        return d

    seg = {k: [] for k in ("device_call", "download", "restatement", "redo", "preintegration")}
    statuses = None
    for rep in range(a.reps + 1):
        d = fresh()
        t0 = time.perf_counter()
        out, _ = d.gins_initialize(inits, cfg, noise5, station)
        t1 = time.perf_counter()
        d.close()
        statuses = out["status"]
        d = fresh()
        t2 = time.perf_counter()
        windows = [d.window(s)[0] for s in range(B)]  # one synchronous download per stream
        t3 = time.perf_counter()
        o = go.OracleGins(B)
        o.push(windows, cfg)
        ref, cfg_o = o.gins_initialize(inits, cfg, GYR_BIAS_STD)
        t4 = time.perf_counter()
        d.redo(ref["state17"], cfg_o)
        t5 = time.perf_counter()
        for s in range(B):
            x = ref["state17"][s, 1:17].copy()
            x[3:7] /= np.linalg.norm(x[3:7])
            iw = go.earth_iewn(station, x[:3]) if cfg[s]["with_earth"] else None
            imu_preintegrate(x, iw, np.array([0, 0, synth_ba.GRAVITY[2]]), noise5, ref["series"][s][:, 1:])
        t6 = time.perf_counter()
        d.close()
        o.close()
        if rep:  # repetition 0 loads modules and compiles the restatement
            for k, v in zip(seg, (t1 - t0, t3 - t2, t4 - t3, t5 - t4, t6 - t5)):
                seg[k].append(v)
    med = {f"{k}_ms": 1e3 * float(np.median(v)) for k, v in seg.items()}
    host = sum(med[f"{k}_ms"] for k in ("download", "restatement", "redo", "preintegration"))
    name, plim = card(torch, 0)
    print(json.dumps({"bench": "gins_init", "streams": B, "initialized": int((statuses == 1).sum()), **med, "host_route_ms": host,
                      "reps": a.reps, "gpu": name, "power_limit_w": plim}))


if __name__ == "__main__":
    main()
