#!/usr/bin/env python
"""Throughput of trackMappoint + trackReferenceFrame on the device (icg_klt_track_frames_dev, IG/tracking/tracking.cc:351-574) on one H100.

    python scripts/bench_track_frame.py [--streams 296] [--reps 20] [--warmup 3]

B synthetic 1280x560 streams: frame 0 and frame 1 of every stream sit in KLT slots; per stream 200 reference-list points and 100 map points
(pw back-projected at depth 4 from their frame-1 positions) of the synthetic stream, identity attitudes.  One call = prediction + one
forward/backward LK launch over both lists of all streams + compaction / velocities / parallax + batched RANSAC + final compaction.
Reported:
  * ms per call and frames/s (CUDA events, profiler off);
  * per-kernel device time per call from a torch.profiler run of its own (track_predict, klt_track, track_post, geom_ransac_batch,
    track_compact);
  * the RANSAC's serial subset draw: icg_geom_find_fundamental_mat_ransac_batch on the same survivor sets with its clock64 statistics
    (subsets drawn, share of the set's cycles spent drawing);
  * the same work as a caller does it without this call: icg_klt_track_batch_dev on host-predicted points, D2H, then per stream the host
    undistortion and icg_geom_find_fundamental_mat_ransac (synchronous, one call per stream; Python glue included).
Prints one JSON line with the card name and power limit.  Writes nothing to the source tree.
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

W, H, NREF, NMAP = 1280, 560, 200, 100
INTR = [460.0, 455.0, 640.0, 280.0, 0.0]
DIST = [-0.05, 0.01, 1e-4, -2e-5, 0.0]
KERNELS = ("track_predict_kernel", "klt_track_kernel", "track_post_kernel", "geom_ransac_batch_kernel", "track_compact_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=296)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_frame.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_klt as synth
    from ic_gvins_b200.camera import Camera
    from ic_gvins_b200.geom import Geometry
    from ic_gvins_b200.klt import MAP_IN, MAP_OUT, REF_IN, REF_OUT, _SPEC, KltTracker, track_frame_params

    B, dev = args.streams, torch.device("cuda", 0)
    cs = torch.cuda.Stream(device=dev)
    st = synth.KltStream(W, H, NREF + NMAP, 1234)
    f0, f1 = st.frame(0), st.frame(1)
    trk = KltTracker(W, H, n_slots=2 * B, max_points=B * (NREF + NMAP), stream=cs.cuda_stream)
    for b in range(B):
        trk.upload(b, f0, build=True)
        trk.upload(B + b, f1, build=True)
    trk.sync()
    cam = Camera(INTR, DIST)
    p0, p1 = st.points(0).astype(np.float32), st.points(1).astype(np.float32)
    und1 = cam.undistortPoints(p1[:NMAP])
    pw = cam.pixel2cam(und1) * 4.0
    one = dict(prev_xy=p0[:NMAP], prev_undis_xy=cam.undistortPoints(p0[:NMAP]), pw=pw, ref_kp_xy=cam.undistortPoints(p0[:NMAP]),
               new_xy=p0[NMAP:], ref_xy=p0[NMAP:], ref_frame_id=np.full(NREF, 7, np.int64), velocity_ref=np.zeros((NREF, 2)))
    ten = {}
    for names, n in ((MAP_IN + MAP_OUT, NMAP), (REF_IN + REF_OUT, NREF)):
        for k in names:
            dt, col = _SPEC[k]
            key = ("m_" if n == NMAP else "r_") + k
            if k in one:
                ten[key] = torch.from_numpy(np.ascontiguousarray(np.tile(np.asarray(one[k], dt).reshape(n, col), (B, 1)))).to(dev)
            else:
                ten[key] = torch.zeros((B * n, col), dtype=getattr(torch, np.dtype(dt).name), device=dev)
    mp = {k: ten["m_" + k].data_ptr() for k in MAP_IN + MAP_OUT}
    rp = {k: ten["r_" + k].data_ptr() for k in REF_IN + REF_OUT}
    I3 = np.eye(3)
    params = [track_frame_params(b, B + b, INTR, DIST, I3, I3, I3, np.zeros(3), 0.05, 7, 1.0) for b in range(B)]
    moff, roff = np.arange(B + 1, dtype=np.int32) * NMAP, np.arange(B + 1, dtype=np.int32) * NREF
    n_out = torch.zeros(2 * B, dtype=torch.int32, device=dev)
    par = torch.zeros(2 * B, dtype=torch.float64, device=dev)
    par_n = torch.zeros(2 * B, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()

    def call():
        trk.track_frames_dev(params, moff, mp, roff, rp, n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())

    for _ in range(args.warmup):
        call()
    torch.cuda.synchronize()
    a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(cs)
    for _ in range(args.reps):
        call()
    b_.record(cs)
    torch.cuda.synchronize()
    ms = a.elapsed_time(b_) / args.reps
    no, pn = n_out.cpu().numpy(), par_n.cpu().numpy()

    # ---- per-kernel device time (separate profiled run)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                kern[k] = kern.get(k, 0.0) + float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))) / 5

    # ---- the RANSAC on the same survivor sets, with its draw statistics
    geom = Geometry(stream=cs.cuda_stream)
    new_und = cam.undistortPoints(p0[NMAP:])
    # the RANSAC input of one stream (LK survivors before the RANSAC), from the host LK; every stream has the same content
    tb = KltTracker(W, H, n_slots=4, max_points=NREF)
    init = cam.distortPoints(cam.undistortPoints(p0[NMAP:]))
    q, _, s1 = tb.track_fb(f0, f1, p0[NMAP:], init)
    tb.close()
    k1 = s1 != 0
    set1 = new_und[k1], cam.undistortPoints(q[k1])
    S = B
    P1 = torch.from_numpy(np.ascontiguousarray(np.tile(set1[0], (S, 1)))).to(dev)
    P2 = torch.from_numpy(np.ascontiguousarray(np.tile(set1[1], (S, 1)))).to(dev)
    off = np.arange(S + 1, dtype=np.int32) * len(set1[0])
    mask = torch.zeros(len(set1[0]) * S, dtype=torch.uint8, device=dev)
    ninl = torch.zeros(S, dtype=torch.int32, device=dev)
    stats = torch.zeros((S, 3), dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    for _ in range(2):
        geom.findFundamentalMat_batch_dev(off, P1.data_ptr(), P2.data_ptr(), mask.data_ptr(), ninl.data_ptr(), thresholds=[1.0] * S,
                                          dev_stats=stats.data_ptr())
    torch.cuda.synchronize()
    a.record(cs)
    for _ in range(args.reps):
        geom.findFundamentalMat_batch_dev(off, P1.data_ptr(), P2.data_ptr(), mask.data_ptr(), ninl.data_ptr(), thresholds=[1.0] * S,
                                          dev_stats=stats.data_ptr())
    b_.record(cs)
    torch.cuda.synchronize()
    ransac_ms = a.elapsed_time(b_) / args.reps
    stt = stats.cpu().numpy()

    # ---- the same work without this call: LK batch on host-predicted points, D2H, per-stream host undistortion + RANSAC
    map_pred = cam.distortPoints(cam.world2pixel(pw, I3, np.zeros(3)))
    pts0 = np.tile(np.concatenate([p0[:NMAP], p0[NMAP:]]), (B, 1)).astype(np.float32)
    slots = np.stack([np.repeat(np.arange(B), NMAP + NREF), np.repeat(np.arange(B, 2 * B), NMAP + NREF)], 1).astype(np.int32)
    d_p0, d_slots = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (pts0, slots))
    d_fwd = torch.empty((B * (NMAP + NREF), 2), dtype=torch.float32, device=dev)
    d_st = torch.empty((B * (NMAP + NREF),), dtype=torch.uint8, device=dev)

    def baseline():
        init = np.tile(np.concatenate([map_pred, cam.distortPoints(cam.undistortPoints(p0[NMAP:]))]), (B, 1)).astype(np.float32)
        d_init = torch.from_numpy(init).to(dev)
        torch.cuda.synchronize()
        trk.track_batch_dev(B * (NMAP + NREF), d_slots.data_ptr(), d_p0.data_ptr(), d_init.data_ptr(), d_fwd.data_ptr(), 0, d_st.data_ptr(), 1)
        trk.sync()
        fw, sv = d_fwd.cpu().numpy().reshape(B, -1, 2), d_st.cpu().numpy().reshape(B, -1)
        for s in range(B):
            km, kr = sv[s, :NMAP] != 0, sv[s, NMAP:] != 0
            cam.undistortPoints(fw[s, :NMAP][km])
            cu_s = cam.undistortPoints(fw[s, NMAP:][kr])
            nu_s = cam.undistortPoints(p0[NMAP:][kr])
            if len(cu_s) >= 15:
                geom.findFundamentalMat(nu_s, cu_s, 1.0, 0.99)

    baseline()
    t0 = time.perf_counter()
    nb = max(2, args.reps // 5)
    for _ in range(nb):
        baseline()
    base_ms = (time.perf_counter() - t0) * 1e3 / nb
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        plim = None
    line = {"metric": "trackMappoint + trackReferenceFrame on the device, frames/s", "value": B / (ms / 1e3), "unit": "frames/s",
            "frames_per_call": B, "ms_per_call": ms, "map_survivors_mean": float(no[0::2].mean()), "ref_survivors_mean": float(no[1::2].mean()),
            "parallax_counts_mean": [float(pn[0::2].mean()), float(pn[1::2].mean())],
            "kernel_us_per_call": {k: round(v, 1) for k, v in kern.items()},
            "ransac_batch_ms_same_sets": ransac_ms, "ransac_pairs_per_set": int(len(set1[0])), "ransac_subsets_drawn_mean": float(stt[:, 0].mean()),
            "ransac_draw_share_of_cycles": float(stt[:, 1].sum() / max(1, stt[:, 2].sum())),
            "baseline_ms_per_step": base_ms, "baseline_note": "icg_klt_track_batch_dev + D2H + per-stream host undistortion and icg_geom_find_fundamental_mat_ransac, Python glue",
            "gpu": torch.cuda.get_device_name(dev), "power_limit_w": plim}
    print(json.dumps(line))
    geom.close()
    trk.close()


if __name__ == "__main__":
    main()
