"""Times icg_ba_shard_update_and_cull_built against the sharded culling it replaces, on two in-process landmark-shard ranks of one GPU, on B
windows that have just slid with icg_ba_shard_slide_vision_resident (which built each rank's next culling lists on the device).

  built     : icg_ba_shard_update_and_cull_built on every rank; only the extrinsic inputs go up
  host lists: icg_ba_update_and_cull_resident on every rank, fed the same shard lists already built (what a host hands over after its walk)
  host work : what the built call removes from the host, timed on the CPU on its own line: the numpy list restatement of every whole window
              (tests/cull_lists_oracle.next_lists) plus the cut of its lists into the ranks' shards.  A C++ integrator's own graph walk would
              take its place
  bytes     : per rank and keyframe, the list bytes each route uploads (host lists: lm_ref_node, lm_ref_kp, obs_off, obs_node, obs_kp for the
              culling, obs_factor for the next vision slide; built: none)
  kernel    : ba_vision_build per launch (it emits the lists on shards now), from torch.profiler in a separate pass

The culling leaves the windows as they are, so the two routes alternate on the same slid group.  Wall time from the calls to a device
synchronise.  The ranks run in threads on cuda:0, so the peer exchanges never cross NVLink here.  Prints two JSON lines.

    python scripts/bench_shard_cull_built.py --cfg 3 --windows 296
    python scripts/bench_shard_cull_built.py --cfg 4 --windows 128
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

N_DISTINCT = 4
WORLD = 2
LISTS = ("lm_ref_node", "lm_ref_kp", "obs_off", "obs_node", "obs_kp", "obs_factor")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3, choices=(3, 4))
    ap.add_argument("--windows", type=int, default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_cull_built.py: no CUDA device; the product path has no CPU fallback")
    from bench_slide_vision import card, cull_lists
    from datagen import synth_ba
    from datagen.slide_window import build_next
    from ic_gvins_b200.ba import WindowSolver, imu_preintegrate, merge_cull_shard, shard_cull_inputs, shard_vision_inputs, shard_window
    from ic_gvins_b200.camera import CameraStruct
    from tests import shard_vision_oracle as sv
    from tests import slide_vision_oracle as so
    from tests.cull_lists_oracle import next_lists
    from tests.test_cull_built_gpu import ext_of
    from tests.test_shard_cull_lists_oracle import cut
    from tests.test_shard_post_solve_gpu import run_ranks
    cfg3 = args.cfg == 3
    B = args.windows or (296 if cfg3 else 128)
    K, L = (10, 300) if cfg3 else (20, 2000)
    gpu, plim = card(torch)
    fx, cx, cy = synth_ba.F_PIX, 640.0, 280.0
    cam = CameraStruct(fx, fx, cx, cy, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    camd = dict(fx=fx, fy=fx, cx=cx, cy=cy, skew=0.0)

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    kw = dict(K=K, L=L) if cfg3 else dict(K=K, L=L, n_ref=K)
    base = [synth_ba.make_window(pre, seed=9500 + i, **kw)[0] for i in range(min(N_DISTINCT, B))]
    probs0 = [copy.deepcopy(base[i % len(base)]) for i in range(B)]
    shards0 = [[shard_window(p, r, WORLD) for p in probs0] for r in range(WORLD)]
    cis = [cull_lists(p, fx, cx, cy) for p in probs0]
    sci = [[shard_cull_inputs(ci, sh) for ci, sh in zip(cis, shards0[r])] for r in range(WORLD)]
    S = [WindowSolver(max_windows=B, max_K=K, max_L=max(s["L"] for s in shards0[r]) + 64, max_F=max(s["F"] for s in shards0[r]) + 512, max_gnss=16,
                      max_marg_r=15 * (K - 1) + 7) for r in range(WORLD)]
    blobs = [S[r].shard_export(r, WORLD) for r in range(WORLD)]
    for s in S:
        s.shard_connect(blobs)

    def restore():
        def rank(r):
            sh = copy.deepcopy(shards0[r])
            S[r].upload(sh)
            g = S[r].update_and_cull(sh, cam, 1.5, sci[r])
            return sh, g, S[r].marginalize(sh, 1, resident=True, culled=g)
        out = run_ranks(WORLD, rank)
        torch.cuda.synchronize()
        return out

    st = restore()
    sh = [x[0] for x in st]
    gr = [x[1] for x in st]
    rng = np.random.default_rng(9600)
    cases, whole_in = [], []
    n_obs_tot = n_new_tot = 0
    for w, p0 in enumerate(probs0):
        p = copy.deepcopy(p0)  # the whole window and its culling
        for r in range(WORLD):
            s_ = sh[r][w]
            p["invdepth"][s_["lm_lo"]:s_["lm_hi"]] = s_["invdepth"]
            p["f_active"][s_["f_index"]] = s_["f_active"]
        for k in ("pose", "mix", "ext", "gnss_std"):
            p[k] = sh[0][w][k].copy()
        g = dict(cis[w], lm_pw=np.zeros((p["L"], 3)), lm_depth=np.zeros(p["L"]), lm_outlier=np.zeros(p["L"], np.uint8),
                 obs_outlier=np.zeros(len(cis[w]["obs_node"]), np.uint8))
        for r in range(WORLD):
            merge_cull_shard(g, sh[r][w], gr[r][w])
        prior = st[w % WORLD][2][w]
        _, nxt, carry = build_next(p, 9700 + w, drop=(0,), n_new=1, prior=prior)
        cur = nxt["K"] - 1
        lms = rng.choice(np.unique(p["f_lm"]), size=min(200 if cfg3 else 600, p["L"]), replace=False)
        xy = rng.uniform([100, 60], [1180, 500], (len(lms), 2)).astype(np.float32)
        vel = rng.normal(0, 5, (len(lms), 2))
        nn = 30 if cfg3 else 100
        new = dict(depth=rng.uniform(2, 40, nn), ref_xy=rng.uniform([100, 60], [1180, 500], (nn, 2)).astype(np.float32), vel_ref=rng.normal(0, 5, (nn, 2)),
                   ref_id=np.array([1000 + cur - 1 - j % 3 for j in range(nn)], np.int64), cur_xy=rng.uniform([100, 60], [1180, 500], (nn, 2)).astype(np.float32),
                   vel_cur=rng.normal(0, 5, (nn, 2)))
        td = np.zeros(nxt["K"])
        frames = {1000 + k: k for k in range(nxt["K"])}
        vis_h = dict(num_marg=1, node_in_map=np.ones(p["K"], np.uint8), node_td=td, cur_node=cur, frames=frames,
                     obs=[(int(l), cur, xy[i], vel[i]) for i, l in enumerate(lms)],
                     new=[dict(depth=new["depth"][j], ref_xy=new["ref_xy"][j], vel_ref=new["vel_ref"][j], ref_id=int(new["ref_id"][j]),
                               cur_xy=new["cur_xy"][j], vel_cur=new["vel_cur"][j]) for j in range(nn)])
        d = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a, dt)).cuda()  # noqa: E731
        vis_d = dict(num_marg=1, node_in_map=np.ones(p["K"], np.uint8), camera=cam, node_td=td, cur_node=cur, frames=frames,
                     n_obs=len(lms), obs_lm=d(lms, np.int32), obs_node=d(np.full(len(lms), cur), np.int32), obs_undis_xy=d(xy, np.float32),
                     obs_vel=d(vel, np.float64), n_new=nn, new_depth=d(new["depth"], np.float64), new_ref_undis_xy=d(new["ref_xy"], np.float32),
                     new_vel_ref=d(new["vel_ref"], np.float64), new_ref_frame_id=d(new["ref_id"], np.int64), new_cur_undis_xy=d(new["cur_xy"], np.float32),
                     new_vel_cur=d(new["vel_cur"], np.float64))
        whole_in.append((p, g, carry, vis_h, nxt, w))
        cases.append((nxt, {k: v for k, v in carry.items() if k not in ("lm_src", "f_src")}, [shard_vision_inputs(vis_d, sh[r][w], gr[r][w]) for r in range(WORLD)]))
        n_obs_tot += len(lms)
        n_new_tot += nn


    # the slide that builds the lists, and the whole-window restatement the host would otherwise make (not timed)
    nxt_r = [[copy.deepcopy(x[0]) for x in cases] for _ in range(WORLD)]
    res = run_ranks(WORLD, lambda r: S[r].shard_slide_vision(nxt_r[r], [copy.deepcopy(x[1]) for x in cases], [x[2][r] for x in cases]))
    torch.cuda.synchronize()
    wholes = []
    for p, g, carry, vis_h, nxt, w in whole_in:
        o = so.build(p, g, carry["node_src"], vis_h, camd)
        onode = np.full(p["K"], -1)
        for j, i in enumerate(carry["node_src"]):
            if 1 <= i < p["K"]:
                onode[i] = j
        xy = {(l, nd): q for l, nd, q, _ in vis_h["obs"]}
        pts = [dict(ref_node=vis_h["frames"][q["ref_id"]], ref_xy=q["ref_xy"], cur_xy=q["cur_xy"]) for q in vis_h["new"]]
        prev = [sh[r][w] for r in range(WORLD)]
        order = sv.rank_order(o, prev, w)
        new_of = np.empty(o["L"], np.int64)
        new_of[order] = np.arange(o["L"])
        pos = np.empty(o["F"], np.int64)
        pos[np.argsort(new_of[o["f_lm"]], kind="stable")] = np.arange(o["F"])
        wholes.append((g, onode, o, xy, pts, nxt["K"] - 1, order, pos, [res[r][w]["L"] for r in range(WORLD)]))

    def host_work():
        for g, onode, o, xy, pts, cur, order, pos, Ls in wholes:
            wl = next_lists(g, g["obs_outlier"], onode, o, xy, pts, cur)
            lo = 0
            for r in range(WORLD):
                cut(wl, order[lo:lo + Ls[r]], pos)
                lo += Ls[r]

    t0 = time.perf_counter()
    host_work()
    host_work_ms = 1e3 * (time.perf_counter() - t0)
    exts = [ext_of(p) for p in nxt_r[0]]
    lists = run_ranks(WORLD, lambda r: S[r]._cull_built("icg_ba_shard_update_and_cull_built", nxt_r[r], cam, 1.5, exts))
    host_in = [[dict(e, **{k: lists[r][w][k] for k in LISTS}) for w, e in enumerate(exts)] for r in range(WORLD)]
    up_bytes = [sum(12 * len(x["lm_ref_node"]) + 4 * len(x["obs_off"]) + 16 * int(x["n_obs"]) for x in lists[r]) for r in range(WORLD)]

    def built():
        run_ranks(WORLD, lambda r: S[r].shard_update_and_cull_built(nxt_r[r], cam, 1.5, exts))

    def host_lists():
        run_ranks(WORLD, lambda r: S[r].update_and_cull(nxt_r[r], cam, 1.5, host_in[r]))

    times = {"built": [], "host_lists": []}
    for rep in range(args.reps + 1):
        for name, fn in (("host_lists", host_lists), ("built", built)):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if rep:
                times[name].append(1e3 * (time.perf_counter() - t0))
    restore()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_ranks(WORLD, lambda r: S[r].shard_slide_vision([copy.deepcopy(x[0]) for x in cases], [copy.deepcopy(x[1]) for x in cases],
                                                           [x[2][r] for x in cases]))
        torch.cuda.synchronize()
    kern = {e.key: e.device_time_total / max(1, e.count) / 1e3 for e in prof.key_averages() if "ba_vision_build" in e.key}
    for s in S:
        s.close()
    out = dict(metric=f"shard_update_and_cull_built cfg-{args.cfg}", windows=B, world=WORLD, gpu=gpu, power_limit_w=plim, reps=args.reps,
               built_ms_median=statistics.median(times["built"]), host_lists_ms_median=statistics.median(times["host_lists"]),
               list_bytes_uploaded_per_rank_host_lists=up_bytes, list_bytes_uploaded_per_rank_built=[0] * WORLD,
               list_entries_per_rank=[sum(int(x["n_obs"]) for x in lists[r]) for r in range(WORLD)],
               vision_build_ms_per_launch_with_lists=kern)
    print(json.dumps(out))
    print(json.dumps(dict(metric=f"shard_update_and_cull_built cfg-{args.cfg} host work it removes (list restatement + shard cut, CPU)",
                          host_work_ms=host_work_ms)))


if __name__ == "__main__":
    main()
