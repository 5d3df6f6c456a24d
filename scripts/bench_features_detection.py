#!/usr/bin/env python
"""Throughput of featuresDetection driven by the point lists (icg_detect_features_dev, IG/tracking/tracking.cc:579-685) on one H100.

    python scripts/bench_features_detection.py [--streams 296] [--reps 20] [--warmup 3]

B synthetic 1280x560 streams: frame 0 and frame 1 of every stream sit in KLT slots; 300 points per stream are tracked 0 -> 1 with the fused
forward/backward LK (icg_klt_track_batch_dev).  One call = gate + block counts + occupancy mask (radius 40) + goodFeaturesToTrack +
cornerSubPix of the deficits + shift to frame coordinates for all B frames at once:
  * main: list B = the first 200 tracked points of each stream with their LK status (the gate passes, blocks have deficits), list A empty,
    ismask = 1;
  * gated: all 300 points of each stream without status (300 > 295: the gate skips every frame) -- what a skipped frame costs.
The occupancy kernel's own device time comes from a torch.profiler run of its own, after the timed runs.  Prints one JSON line with the card
name and power limit.  Writes nothing to the source tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, NPTS, NB = 1280, 560, 300, 200


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=296)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_features_detection.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_klt as synth
    from ic_gvins_b200 import lib
    from ic_gvins_b200.detect import Detector, block_rois
    from ic_gvins_b200.klt import KltTracker

    B, dev = args.streams, torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    st = synth.KltStream(W, H, NPTS, 1234)
    f0, f1 = st.frame(0), st.frame(1)
    trk = KltTracker(W, H, n_slots=2 * B, max_points=B * NPTS, stream=stream.cuda_stream)
    for b in range(B):  # slot b: frame 0 of stream b, slot B + b: its frame 1
        trk.upload(b, f0, build=True)
        trk.upload(B + b, f1, build=True)
    trk.sync()
    rng = np.random.Generator(np.random.PCG64(7))
    p0 = np.tile(st.points(0).astype(np.float32), (B, 1))
    init = (np.tile(st.points(1), (B, 1)) + rng.normal(0.0, 1.0, (B * NPTS, 2))).astype(np.float32)
    slots = np.stack([np.repeat(np.arange(B), NPTS), np.repeat(np.arange(B, 2 * B), NPTS)], axis=1).astype(np.int32)
    d_p0, d_init, d_slots = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (p0, init, slots))
    d_fwd = torch.empty((B * NPTS, 2), dtype=torch.float32, device=dev)
    d_bwd = torch.empty((B * NPTS, 2), dtype=torch.float32, device=dev)
    d_st = torch.empty((B * NPTS,), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    trk.track_batch_dev(B * NPTS, d_slots.data_ptr(), d_p0.data_ptr(), d_init.data_ptr(), d_fwd.data_ptr(), d_bwd.data_ptr(), d_st.data_ptr(), 1)

    rois, quota, _, _ = block_rois(W, H, NPTS)
    det = Detector(W, H, max_blocks=B * len(rois), max_corners_per_block=32, max_roi_pixels=213 * 186, stream=stream.cuda_stream)
    q0, q1, pitch = C.c_void_p(), C.c_void_p(), C.c_int()
    lib().icg_klt_slot_level0(trk._h, B, C.byref(q0), C.byref(pitch))
    lib().icg_klt_slot_level0(trk._h, B + 1, C.byref(q1), C.byref(pitch))
    img0, fstride = q0.value, q1.value - q0.value
    with torch.cuda.stream(stream):
        l_xy = d_fwd.view(B, NPTS, 2)[:, :NB].contiguous()
        l_st = d_st.view(B, NPTS)[:, :NB].contiguous()
    out_xy = torch.empty((B, len(rois) * quota, 2), dtype=torch.float32, device=dev)
    out_n = torch.empty((B,), dtype=torch.int32, device=dev)
    no_feat, ism = np.zeros(B + 1, np.int32), np.ones(B, np.uint8)

    def call(xy, status, n_per):
        det.features_detection_dev(B, img0, pitch.value, fstride, 0, 0, no_feat, xy.data_ptr(), status.data_ptr() if status is not None else 0,
                                   np.arange(B + 1, dtype=np.int32) * n_per, out_xy.data_ptr(), out_n.data_ptr(), ismask=ism, max_features=NPTS)

    def timed(xy, status, n_per):
        for _ in range(args.warmup):
            call(xy, status, n_per)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(args.reps):
            call(xy, status, n_per)
        b.record(stream)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.reps

    ms = timed(l_xy, l_st, NB)
    n = out_n.cpu().numpy()
    ms_gated = timed(d_fwd, None, NPTS)
    n_gated = out_n.cpu().numpy()
    occ_us = None
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call(l_xy, l_st, NB)
        torch.cuda.synchronize()
    occ = [e for e in prof.key_averages() if "detect_occupancy" in e.key]
    if occ:
        occ_us = sum(float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))) for e in occ) / 5  # 5 calls, one launch each
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    line = {"metric": "featuresDetection from point lists, frames/s", "value": B / (ms / 1e3), "unit": "frames/s", "frames_per_call": B,
            "ms_per_call": ms, "frames_detected": int((n >= 0).sum()), "corners_per_frame": float(n[n >= 0].mean()) if (n >= 0).any() else 0.0,
            "occupancy_kernel_us_per_call": occ_us, "gated_ms_per_call": ms_gated, "gated_frames_per_s": B / (ms_gated / 1e3),
            "gated_frames": int((n_gated == -1).sum()), "gpu": torch.cuda.get_device_name(dev), "power_limit_w": plim}
    print(json.dumps(line))
    det.close()
    trk.close()


if __name__ == "__main__":
    main()
