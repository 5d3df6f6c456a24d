#!/usr/bin/env python
"""Throughput of Tracking::triangulation on the device (icg_klt_triangulate_dev, IG/tracking/tracking.cc:690-798) on one H100.

    python scripts/bench_triangulation.py [--streams 296] [--reps 20] [--warmup 3]

Two measurements, one JSON line:
  * the call alone: B streams of 200 reference points with 10-entry keyframe tables, from the scene of tests/test_triangulation_gpu.py
    (a known mix of resets, out-of-window points, low parallax, outliers and new map points; the counts are reported).  The lists are
    compacted in place, so each timed call is preceded by an untimed restore of the lists; CUDA events bracket the call alone;
  * chained after icg_klt_track_frames_dev: the tracking step on 200 reference points of 1280x560 synthetic frames per stream, then the
    triangulation reading the live counts from dev_n_out on the device; events bracket the pair, and the tracking step alone.
Per-kernel device time comes from a separate torch.profiler run.  The card name and its power limit are read in the same run.  Writes
nothing to the source tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, NREF = 1280, 560, 200


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=296)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_triangulation.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_klt as synth
    from ic_gvins_b200.klt import _SPEC, _TRI_NEW_SPEC, REF_IN, REF_OUT, TRI_LIST, KltTracker, track_frame_params
    from ic_gvins_b200.klt import TriFrameStruct, tri_keyframes
    from tests.test_triangulation_gpu import Ry, kf_rows, make_stream, struct

    B, dev = args.streams, torch.device("cuda", 0)
    cs = torch.cuda.Stream(device=dev)
    trk = KltTracker(W, H, n_slots=2 * B, max_points=B * NREF, stream=cs.cuda_stream)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn, before=None):
        for _ in range(args.warmup):
            if before:
                before()
            fn()
        torch.cuda.synchronize()
        total = 0.0
        for _ in range(args.reps):
            if before:
                before()
            ev[0].record(cs)
            fn()
            ev[1].record(cs)
            torch.cuda.synchronize()
            total += ev[0].elapsed_time(ev[1])
        return total / args.reps

    def kernels(fn, before=None, names=("tri_kernel",)):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                if before:
                    before()
                fn()
            torch.cuda.synchronize()
        out = {}
        for e in prof.key_averages():
            for k in names:
                if k in e.key:
                    out[k] = out.get(k, 0.0) + float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))) / 5
        return {k: round(v, 1) for k, v in out.items()}

    # ---- the call alone on the mixed scene
    rng = np.random.default_rng(2026)
    cases = [make_stream(rng, NREF, window_normal=s % 2 == 0, std=1.5) for s in range(B)]
    off = np.arange(B + 1, dtype=np.int32) * NREF
    pristine = {}
    for k in TRI_LIST:
        dt, col = _SPEC[k]
        arr = np.concatenate([np.asarray(c[2][k], dt).reshape(NREF, col) for c in cases]) if k != "src" else np.zeros((B * NREF, 1), dt)
        pristine[k] = torch.from_numpy(np.ascontiguousarray(arr)).to(dev)
    lt = {k: v.clone() for k, v in pristine.items()}
    nt = {k: torch.zeros((B * NREF, c), dtype=getattr(torch, np.dtype(dt).name), device=dev) for k, (dt, c) in _TRI_NEW_SPEC.items()}
    counts = torch.zeros((B, 5), dtype=torch.int32, device=dev)
    params = (TriFrameStruct * B)(*[struct(c[0]) for c in cases])  # built once: the timed call is the library call
    kf_off = np.concatenate([[0], np.cumsum([len(c[1]) for c in cases])]).astype(np.int32)
    rows = tri_keyframes([r for c in cases for r in kf_rows(c[1])])
    lp, npt = {k: v.data_ptr() for k, v in lt.items()}, {k: v.data_ptr() for k, v in nt.items()}
    torch.cuda.synchronize()

    def restore():
        with torch.cuda.stream(cs):
            for k in TRI_LIST:
                lt[k].copy_(pristine[k])

    def call():
        trk.triangulate_dev(params, kf_off, rows, off, 0, 1, lp, npt, counts.data_ptr())

    ms_alone = timed(call, restore)
    cnt = counts.cpu().numpy()
    kern_alone = kernels(call, restore)

    # ---- chained after the tracking step
    st = synth.KltStream(W, H, NREF, 1234)
    f0, f1 = st.frame(0), st.frame(1)
    for b in range(B):
        trk.upload(b, f0, build=True)
        trk.upload(B + b, f1, build=True)
    trk.sync()
    p0 = st.points(0).astype(np.float32)[:NREF]
    # reference frames 7 (frame_ref_), 6, 5 (out of the map) and 8 (newer: reset); rotated keyframes give the parallax to triangulate
    one = dict(new_xy=p0, ref_xy=p0, ref_frame_id=np.tile(np.array([7, 6, 5, 8], np.int64), NREF // 4), velocity_ref=np.zeros((NREF, 2)))
    rt = {}
    for k in REF_IN + REF_OUT:
        dt, col = _SPEC[k]
        rt[k] = (torch.from_numpy(np.ascontiguousarray(np.tile(np.asarray(one[k], dt).reshape(NREF, col), (B, 1)))).to(dev) if k in one
                 else torch.zeros((B * NREF, col), dtype=getattr(torch, np.dtype(dt).name), device=dev))
    rp = {k: v.data_ptr() for k, v in rt.items()}
    I3 = np.eye(3)
    tparams = [track_frame_params(b, B + b, cases[0][0]["intrinsic"], cases[0][0]["distortion"], I3, I3, I3,
                                  np.zeros(3), 0.05, 7, 1.0) for b in range(B)]
    moff = np.zeros(B + 1, np.int32)
    n_out = torch.zeros(2 * B, dtype=torch.int32, device=dev)
    par = torch.zeros(2 * B, dtype=torch.float64, device=dev)
    par_n = torch.zeros(2 * B, dtype=torch.int32, device=dev)
    src = torch.zeros(B * NREF, dtype=torch.int32, device=dev)
    tri_kf = {fid: (Ry(0.03 * (j + 1)), np.array([-0.2 * j - 0.1, 0.0, 0.02 * j]), fid != 5) for j, fid in enumerate(range(7, -3, -1))}
    P = dict(cases[0][0], R_cur=I3, t_cur=np.array([0.6, 0.0, 0.05]), cur_id=9, ref_id=7, window_normal=True, triangulate=True)
    cparams = (TriFrameStruct * B)(*([struct(P)] * B))
    ckf_off = np.arange(B + 1, dtype=np.int32) * len(tri_kf)
    crows = tri_keyframes(kf_rows(tri_kf) * B)
    clp = dict({k: rp[k] for k in ("ref_out_xy", "ref_frame_id_out", "cur_xy", "velocity_ref_out", "velocity")}, src=src.data_ptr())
    torch.cuda.synchronize()

    def track():
        trk.track_frames_dev(tparams, moff, None, off, rp, n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())

    def chained():
        track()
        trk.triangulate_dev(cparams, ckf_off, crows, off, n_out.data_ptr() + 4, 2, clp, npt, counts.data_ptr())

    ms_track = timed(track)
    ms_chain = timed(chained)
    ccnt = counts.cpu().numpy()
    kern_chain = kernels(chained, names=("tri_kernel", "track_post_kernel", "klt_track_kernel", "geom_ransac_batch_kernel"))
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    line = {"metric": "Tracking::triangulation on the device, streams/s", "value": B / (ms_alone / 1e3), "unit": "streams/s", "streams_per_call": B,
            "points_per_stream": NREF, "keyframes_per_stream": 10, "ms_per_call": ms_alone, "kernel_us_per_call": kern_alone,
            "counts_sum": dict(zip(("kept", "succeeded", "outlier", "reset", "outtime"), cnt.sum(0).tolist())),
            "chained_ms_per_call": ms_chain, "track_step_ms_per_call": ms_track, "chained_kernel_us_per_call": kern_chain,
            "chained_counts_sum": dict(zip(("kept", "succeeded", "outlier", "reset", "outtime"), ccnt.sum(0).tolist())),
            "gpu": torch.cuda.get_device_name(dev), "power_limit_w": plim}
    print(json.dumps(line))
    trk.close()


if __name__ == "__main__":
    main()
