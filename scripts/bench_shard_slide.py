#!/usr/bin/env python
"""Cost of one keyframe step of a landmark-sharded group: the next windows with one new keyframe interval, for B resident cfg-4 windows
(K = 20, L = 2000, max_marg_r = 292) on two in-process ranks sharing one GPU.

    python scripts/bench_shard_slide.py [--windows 128] [--reps 5] [--iters 4]

Every repetition starts from the same state, set up outside the timed region: the shards uploaded, the sharded culling and the culled
resident marginalization run (each window's prior on its owner).  Then, timed with the host clock around work that ends in a synchronise,
alternating:
  (a) host   what a sharded user had to do before: the owner's prior handed to every rank's next shards, the states downloaded, the new
             interval (101 samples) preintegrated on the host (icg_imu_preintegrate) with its new node row, icg_ba_upload on every rank;
  (b) device icg_ba_shard_slide_integrate_resident on both ranks.
The next windows' structure (build_next, shard_next) is made once, outside the timing; both paths go through the Python wrappers, which
build the argument structs on every call.  H2D value bytes are computed from the shapes.  A separate torch.profiler run of (b) gives the
kernel times of ba_slide_gather, ba_slide_prior, preint_slide_kernel and ba_xsum.  The card name and power limit are read in the same run.
Prints one JSON line; writes nothing to the source tree.  What this script does NOT do, and why:
  * Output check.  The two paths are not compared after run_gvins: a two-rank sharded solve of 128 cfg-4 windows cannot run on one GPU in
    one process (a rank's kernels that wait for the other's flags occupy the device).  After one run of each path the sharded resident
    marginalization of the next windows -- which reads their parameters, blobs and square-root information, GNSS rows and the prior on the
    device -- must give np.array_equal priors on the owners.  The solve after the slide is compared bitwise in tests/test_shard_slide_gpu.py.
  * Independence.  In that check the host path preintegrates with the Earth rate taken from the device path's blobs (the numpy restatement
    of Earth::iewn is not pinned to the last bit), so the check covers everything but that rate; the timed host runs use the numpy rate.
  * One process per GPU.  Not measured: the script has no per-GPU mode ("one_process_per_gpu" says so in the output).
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("ba_slide_gather", "ba_slide_prior", "preint_slide_kernel", "ba_xsum")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=4)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_slide.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    from datagen.slide_window import build_next
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate, shard_cull_inputs, shard_next, shard_window
    from ic_gvins_b200.camera import Camera
    from tests.test_post_solve_gpu import CAMD, STD, cull_inputs
    from tests.test_reintegration_gpu import earth_iewn, state16

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    B, G, K, L, R = args.windows, 2, 20, 2000, 292
    nb = min(8, B)
    base = [synth_ba.make_window(pre, K=K, L=L, seed=7300 + i)[0] for i in range(nb)]
    shards = [[shard_window(base[w % nb], r, G) for w in range(B)] for r in range(G)]
    caps = [dict(L=max(s["L"] for s in shards[r]) + 8, F=max(s["F"] for s in shards[r]) + 64) for r in range(G)]
    ranks = [WindowSolver(max_windows=B, max_K=K, max_L=caps[r]["L"], max_F=caps[r]["F"], max_gnss=16, max_marg_r=R) for r in range(G)]
    blobs = [ranks[r].shard_export(r, G) for r in range(G)]
    for s in ranks:
        s.shard_connect(blobs)
    cam = Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])
    cis = [cull_inputs(p, p["ext"].copy(), 7400 + i, bad_kp=20) for i, p in enumerate(base)]

    def on_ranks(fn):
        out, errs = [None] * G, []

        def body(r):
            try:
                out[r] = fn(r)
            except Exception as e:  # noqa: BLE001
                errs.append((r, repr(e)))
        th = [threading.Thread(target=body, args=(r,)) for r in range(G)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if errs:
            raise RuntimeError(errs)
        return out

    held = {}

    def setup():
        """the shards uploaded, culled and marginalized (sharded): the state both paths start from; returns every window's prior"""
        sh = [[copy.deepcopy(s) for s in shards[r]] for r in range(G)]
        held["sh"] = sh

        def rank(r):
            ranks[r].upload(sh[r])
            g = ranks[r].update_and_cull(sh[r], cam, STD, [shard_cull_inputs(cis[w % nb], sh[r][w]) for w in range(B)])
            return ranks[r].marginalize(sh[r], 1, resident=True, culled=g)
        pri = on_ranks(rank)
        torch.cuda.synchronize()
        return [pri[w % G][w] for w in range(B)]

    priors = setup()
    # the next windows of the distinct bases (the repeated windows' priors are the same): node 0 dropped, one new node whose interval and
    # node row are integrated from the last old node
    nexts = []
    for i in range(nb):
        p = base[i]
        up, stale, carry = build_next(p, 7500 + i, prior=priors[i])
        k = up["n_imu"] - 1
        rng = np.random.default_rng(7600 + i)
        mix = p["mix"].reshape(K, 9)[K - 1]
        rows = synth_ba.imu_samples(0.5 * (K - 1), 0.5 * K, 200.0, rng, mix[3:6], mix[6:9])
        g = dict(imu_from=np.full(up["n_imu"], -1, np.int32), imu_rows=[None] * up["n_imu"], gravity=synth_ba.GRAVITY,
                 node_from_imu=np.zeros(up["K"], np.uint8))
        g["imu_from"][k], g["imu_rows"][k], g["node_from_imu"][k + 1] = K - 1, rows, 1
        nr = np.where(carry["lm_src"] < 0, np.arange(up["L"]) % G, -1)
        sa = shard_next(stale, carry, [shards[r][i] for r in range(G)], nr)[2]
        su = shard_next(up, carry, [shards[r][i] for r in range(G)], nr)
        nexts.append(dict(up=up, carry=carry, g=g, k=k, rows=rows, nr=nr, sa=sa, whole_up=su[0], su=su[2]))
    n_samples = int(nexts[0]["rows"].shape[0])
    flags = [True] * B

    def path_device():
        parts = [[copy.deepcopy(nexts[w % nb]["sa"][r]) for w in range(B)] for r in range(G)]
        t0 = time.perf_counter()
        outs = on_ranks(lambda r: ranks[r].shard_slide_integrate([x[0] for x in parts[r]], [x[1] for x in parts[r]], [nexts[w % nb]["g"] for w in range(B)],
                                                         synth_ba.NOISE5, np.zeros(3), flags))
        for s in ranks:
            s.sync()
        path_device.outs = outs
        return (time.perf_counter() - t0) * 1e3, [[x[0] for x in parts[r]] for r in range(G)]

    def path_host(iewn=None):
        """iewn: per window, the Earth rate to preintegrate with (None: Earth::iewn of the start position, restated in numpy)"""
        parts = [[copy.deepcopy(nexts[w % nb]["su"][r][0]) for w in range(B)] for r in range(G)]
        cur = held["sh"][0]  # rank 0's dicts: its download writes the resident states into them
        t0 = time.perf_counter()
        for w in range(B):  # the owner's prior, as its marginalization returned it on the host, handed to every rank
            for r in range(G):
                parts[r][w]["marg_J0"][:] = priors[w]["J0"].reshape(-1)
                parts[r][w]["marg_e0"][:] = priors[w]["e0"]
        ranks[0].download()  # the states the interval starts from (replicated: one rank's)
        for w in range(B):
            c = nexts[w % nb]
            pose, mix = cur[w]["pose"].reshape(K, 7), cur[w]["mix"].reshape(K, 9)
            st = state16(pose[K - 1], mix[K - 1])
            iw = earth_iewn(np.zeros(3), st[:3]) if iewn is None else iewn[w]
            blob, end = imu_preintegrate(st, iw, synth_ba.GRAVITY, synth_ba.NOISE5, c["rows"])
            for r in range(G):
                parts[r][w]["imu_blob"].reshape(-1, 480)[c["k"]] = blob
                parts[r][w]["pose"].reshape(-1, 7)[c["k"] + 1] = end[:7]
                parts[r][w]["mix"].reshape(-1, 9)[c["k"] + 1] = np.r_[end[7:10], st[10:16]]
        on_ranks(lambda r: ranks[r].upload(parts[r]))
        for s in ranks:
            s.sync()
        return (time.perf_counter() - t0) * 1e3, parts

    times = dict(host=[], device=[])
    for rep in range(args.reps + 1):  # the first round warms up (first launches, staging and workspace allocations)
        for name, fn in (("host", path_host), ("device", path_device)):
            priors[:] = setup()
            ms, _ = fn()
            if rep:
                times[name].append(ms)
    # outputs: one run of each path from the same state, then the sharded resident marginalization of the next windows (it reads their
    # parameters, IMU blobs and square-root information, GNSS rows and the prior's normal equations on the device); every prior, on its owner.
    # A two-rank sharded solve of a batch this large cannot run on one GPU in one process, so run_gvins is not part of this check.
    # The host path takes the device's Earth rate here (the numpy restatement of Earth::iewn is not pinned to the last bit)
    res = {}
    for name, fn in (("device", path_device), ("host", lambda: path_host([path_device.outs[0][w]["blobs"][nexts[w % nb]["k"], 20:23] for w in range(B)]))):
        priors[:] = setup()
        _, nxt = fn()
        out = on_ranks(lambda r: ranks[r].marginalize(nxt[r], 1, resident=True))
        res[name] = [out[w % G][w] for w in range(B)]
    equal = all(np.array_equal(a[k], b[k]) for a, b in zip(res["host"], res["device"]) for k in ("J0", "e0", "Hp", "bp"))
    # kernel times of (b), in a run of its own
    setup()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        path_device()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        for kn in KERNELS:
            if kn in ev.key:
                t = getattr(ev, "self_device_time_total", None)
                if t is None:
                    t = getattr(ev, "self_cuda_time_total", 0.0)
                kern[kn] = kern.get(kn, 0.0) + float(t) / 1e3
    # H2D value bytes from the shapes (doubles of the next shards each path sends; integer structure of both paths not counted)
    h2d = dict(host=0, device=0)
    for w in range(B):
        c = nexts[w % nb]
        for r in range(G):
            s, sc = c["su"][r]
            h2d["host"] += 8 * (16 * s["K"] + s["L"] + 14 * s["F"] + 480 * s["n_imu"] + 6 * s["n_gnss"] + s["marg_r"] ** 2 + s["marg_r"]
                                + len(s["marg_x0"]))
            new = lambda m: int((np.asarray(m) < 0).sum())
            h2d["device"] += 8 * (16 * (new(sc["node_src"]) - 1) + new(sc["lm_src"]) + 14 * new(sc["f_src"]) + 705 * (new(sc["imu_src"]) - 1)
                                  + 6 * new(sc["gnss_src"]) + 7 * n_samples)
    for s in ranks:
        s.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(bench="shard_slide", windows=B, K=K, L=L, max_marg_r=R, ranks=G, interval_samples=n_samples, reps=args.reps,
                          gpu=smi.splitlines()[0] if smi else "?", median_ms={k: float(np.median(v)) for k, v in times.items()},
                          min_ms={k: float(np.min(v)) for k, v in times.items()}, h2d_value_bytes=h2d, kernel_ms=kern, outputs_equal=bool(equal),
                          one_process_per_gpu="not measured")))


if __name__ == "__main__":
    main()
