#!/usr/bin/env python
"""Cost of the device INS windows (ic_gvins_b200.ins) for B streams at the rates the reference runs: 200 Hz IMU, 10 Hz frames.

    python scripts/bench_ins.py [--streams 296] [--frames 200] [--warmup 20] [--redo-every 5] [--redo-samples 150]

Per frame every stream pushes its 20 new samples (icg_ins_push) and takes one prior camera pose (icg_ins_camera_pose with a host copy, the
form the tracking call's host parameters need); every --redo-every frames (a keyframe) each window is redone from an optimized state
--redo-samples samples back (icg_ins_redo, reserved 2).  Half the streams use the Earth form, half the Normal form.  One JSON line:
  * device time per frame and per redo from CUDA events on the handle's stream, and the host clock around the same synchronous calls;
  * beside them, the host time of the CPU restatement (tests/ins_oracle.cpp, std::deque windows, one core) over the same inputs;
  * the largest difference of the final windows between the two, per group scale;
  * the card name and power limit, read in the same run.
Writes nothing to the source tree (the restatement compiles into a temporary directory).
"""
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

RATE, PER_FRAME = 200.0, 20


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
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--redo-every", type=int, default=5)
    ap.add_argument("--redo-samples", type=int, default=150)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ins: no CUDA device")
    from ic_gvins_b200.ins import InsWindow
    from tests import ins_oracle as io
    from tests.test_oracle_ins import EARTH, NORMAL, POSE_B_C, rows8, state_at

    B, F = a.streams, a.warmup + a.frames
    cfg = [EARTH if s % 2 == 0 else NORMAL for s in range(B)]
    n_rows = 200 + PER_FRAME * F + 1
    rows = [rows8(0.013 * s, 0.013 * s + (n_rows - 1) / RATE, RATE, earth=cfg[s]["with_earth"], seed=s) for s in range(B)]
    c7 = io.cfg7(cfg, B)

    stream = torch.cuda.current_stream()
    d = InsWindow(B, 4000, 0, stream.cuda_stream)
    o = io.OracleIns(B, 4000)
    # initialization: one second of samples, then the first redo switches every stream to per-sample mechanization
    init = [r[:200] for r in rows]
    st = np.array([state_at(r[50, 0]) for r in rows])
    st[:, 0] = [r[50, 0] + 0.0021 for r in rows]
    d.push(init, cfg)
    o.push(init, cfg)
    assert (d.redo(st, cfg) == 1).all() and (o.redo(st, cfg) == 1).all()

    def packed(f):
        part = [r[200 + PER_FRAME * f:200 + PER_FRAME * (f + 1)] for r in rows]
        off = np.arange(B + 1, dtype=np.int32) * PER_FRAME
        return part, off, np.ascontiguousarray(np.concatenate(part))

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t_frame, t_redo, h_frame, h_redo, o_frame, o_redo = [], [], [], [], [], []
    bc = np.ascontiguousarray(np.repeat(POSE_B_C[None], B, axis=0))
    dev_pose = torch.zeros((B, 12), dtype=torch.float64, device="cuda")
    for f in range(F):
        part, off, imu = packed(f)
        last = imu[PER_FRAME - 1::PER_FRAME, 0]
        stamp = last - 0.0037  # a frame between two samples
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        ev[0].record(stream)
        d.push(part, cfg)
        hp, found, _ = d.camera_pose(stamp, bc, dev_pose)
        ev[1].record(stream)
        h1 = time.perf_counter()
        o0 = time.perf_counter()
        o.push_packed(c7, off, imu)
        po, fo = o.camera_pose(stamp, bc)
        o1 = time.perf_counter()
        assert (found == fo).all() and (found == 1).all()
        redo = (f + 1) % a.redo_every == 0
        if redo:
            node = np.array([state_at(t) for t in last])
            node[:, 0] = last - a.redo_samples / RATE + 0.0021
            torch.cuda.synchronize()
            h2 = time.perf_counter()
            ev[2].record(stream)
            sd = d.redo(node, cfg)
            ev[3].record(stream)
            h3 = time.perf_counter()
            o2 = time.perf_counter()
            so = o.redo(node, cfg)
            o3 = time.perf_counter()
            assert (sd == so).all() and (sd == 1).all()
        torch.cuda.synchronize()
        if f >= a.warmup:
            t_frame.append(ev[0].elapsed_time(ev[1])), h_frame.append(1e3 * (h1 - h0)), o_frame.append(1e3 * (o1 - o0))
            if redo:
                t_redo.append(ev[2].elapsed_time(ev[3])), h_redo.append(1e3 * (h3 - h2)), o_redo.append(1e3 * (o3 - o2))
    worst = 0.0
    for s in range(0, B, 7):
        xd, xo = d.window(s)[1], o.window(s)[1]
        assert xd.shape == xo.shape
        sp = np.maximum(np.linalg.norm(xo[:, 1:4], axis=1), 1.0)[:, None]
        sv = np.maximum(np.linalg.norm(xo[:, 8:11], axis=1), 1.0)[:, None]
        worst = max(worst, float((np.abs(xd[:, 1:4] - xo[:, 1:4]) / sp).max()), float(np.abs(xd[:, 4:8] - xo[:, 4:8]).max()),
                    float((np.abs(xd[:, 8:11] - xo[:, 8:11]) / sv).max()))
    gpu, plim = card(torch, 0)
    med = lambda v: float(np.median(v)) if v else None  # noqa: E731
    print(json.dumps(dict(streams=B, frames=a.frames, imu_hz=RATE, frame_hz=RATE / PER_FRAME, redo_every=a.redo_every, redo_samples=a.redo_samples,
                          frame_ms_events=med(t_frame), frame_ms_host=med(h_frame), redo_ms_events=med(t_redo), redo_ms_host=med(h_redo),
                          oracle_frame_ms_host_1core=med(o_frame), oracle_redo_ms_host_1core=med(o_redo), n_redo=len(t_redo),
                          max_state_diff=worst, gpu=gpu, power_limit_w=plim)))
    d.close()


if __name__ == "__main__":
    main()
