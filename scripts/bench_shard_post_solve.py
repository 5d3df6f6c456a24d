#!/usr/bin/env python
"""Cost of the post-solve culling + culled marginalization (icg_ba_update_and_cull_resident, icg_ba_marginalize_resident_culled) on
landmark-sharded handles, for B resident cfg-4 windows (K = 20, L = 2000).  The windows are solved once on an unsharded handle
(icg_ba_gvins_optimization) and their shards uploaded to the ranks: a two-rank sharded solve of a batch this large cannot run on ONE GPU in
one process (the kernels of one rank that wait for the other's flags occupy the device), and the solve is not what is timed here.

    python scripts/bench_shard_post_solve.py [--windows 128] [--reps 7] [--iters 4]

Three ways to get the same priors, timed with the host clock around the synchronous C calls, in alternating repetitions.  The argument
structs are built once, outside the timed region, as a C++ caller keeps them across keyframes (the Python wrappers rebuild them on every
call, and the in-process ranks would then serialise on the interpreter lock):
  * sharded   two ranks on ONE GPU (two handles of this process, one host thread each, peer memory over plain pointers): cull + culled
              marginalization on the shards, each window's prior formed on its owner;
  * twin      one unsharded handle that holds the merged windows: cull + culled marginalization;
  * replaced  what a sharded user had to do before: download both shards, merge them on the host, upload the whole windows to an unsharded
              handle, cull and marginalize there.
Also the bytes of each rank's marginalization export region.  Windows: 8 distinct synthetic windows repeated to fill the batch.  The card
name and power limit are read in the same run.  Prints one JSON line; writes nothing to the source tree.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=128)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=4)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_post_solve.py: no CUDA device; the product path has no CPU fallback")
    from datagen import synth_ba
    import ctypes as C
    from ic_gvins_b200._lib import BaProblem, BaSummary, CullWindow, check, lib, vp
    from ic_gvins_b200.ba import WindowSolver, cull_struct, imu_preintegrate, merge_shard, shard_cull_inputs, shard_window, to_struct
    from ic_gvins_b200.camera import Camera
    from tests.test_post_solve_gpu import CAMD, STD, cull_inputs

    def pre(st, iewn, g, nz, imu):
        blob, end = imu_preintegrate(st, iewn, g, nz, imu)
        return blob, np.zeros((imu.shape[0] - 1, 4)), end

    B, G, K, L = args.windows, 2, 20, 2000
    base = []
    for i in range(min(8, B)):
        p = synth_ba.make_window(pre, K=K, L=L, seed=7000 + i)[0]
        rng = np.random.default_rng(7100 + i)
        rows = rng.choice(p["F"], size=30, replace=False)
        p["f_const"].reshape(-1, 14)[rows, 3] += rng.choice([-1, 1], 30) * rng.uniform(3, 40, 30) / synth_ba.F_PIX
        base.append(p)
    probs = [copy.deepcopy(base[w % len(base)]) for w in range(B)]
    ext0 = [p["ext"].copy() for p in probs]
    Fmax = max(p["F"] for p in probs)
    single = WindowSolver(max_windows=B, max_K=K, max_L=L, max_F=Fmax, max_gnss=16, max_marg_r=292)
    single.gvins_optimization_batch(probs, args.iters)  # the solved windows, written back into probs
    shards = [[shard_window(p, r, G) for p in probs] for r in range(G)]
    caps = [dict(L=max(1, max(s["L"] for s in shards[r])), F=max(1, max(s["F"] for s in shards[r]))) for r in range(G)]
    ranks = [WindowSolver(max_windows=B, max_K=K, max_L=caps[r]["L"], max_F=caps[r]["F"], max_gnss=16, max_marg_r=292) for r in range(G)]
    blobs = [ranks[r].shard_export(r, G) for r in range(G)]
    for s in ranks:
        s.shard_connect(blobs)

    def on_ranks(fn):
        errs = []

        def body(r):
            try:
                fn(r)
            except Exception as e:  # noqa: BLE001
                errs.append((r, repr(e)))
        th = [threading.Thread(target=body, args=(r,)) for r in range(G)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if errs:
            raise RuntimeError(errs)

    for r in range(G):
        ranks[r].upload(shards[r])
    merged = probs
    cam = Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])
    cis = [cull_inputs(p, e, 7200 + w % len(base), bad_kp=20) for w, (p, e) in enumerate(zip(merged, ext0))]
    sci = [[shard_cull_inputs(cis[w], shards[r][w]) for w in range(B)] for r in range(G)]
    twin = WindowSolver(max_windows=B, max_K=K, max_L=L, max_F=Fmax, max_gnss=16, max_marg_r=292)
    twin.upload(merged)

    def post_solve_call(solver, problems, cull_in):
        """the two C calls of one handle over argument structs built here once"""
        n = len(problems)
        arr = (BaProblem * n)(*[to_struct(p) for p in problems])
        keep = [dict(c) for c in cull_in]
        cw = (CullWindow * n)(*[cull_struct(p, c) for p, c in zip(problems, keep)])
        call = solver.marg_prepare(problems, 1)
        nim = [np.ones(p["K"], np.uint8) for p in problems]
        ptrs = (vp * n)(*[vp(m.ctypes.data) for m in nim])

        def run():
            check(lib().icg_ba_update_and_cull_resident(solver._h, n, arr, C.byref(cam.c), float(STD), cw), "icg_ba_update_and_cull_resident")
            check(lib().icg_ba_marginalize_resident_culled(solver._h, n, call["arr"], vp(call["nm"].ctypes.data), cw, ptrs, call["pri"]),
                  "icg_ba_marginalize_resident_culled")
        run.keep = (arr, keep, cw, call, nim, ptrs)
        return run

    rank_calls = [post_solve_call(ranks[r], shards[r], sci[r]) for r in range(G)]
    twin_call = post_solve_call(twin, merged, cis)
    # the replaced path: download targets per rank, the whole windows the merge writes into in place, the unsharded handle's calls on them
    dl = [[dict(sh, **{k: np.array(sh[k], copy=True) for k in ("pose", "mix", "ext", "invdepth", "f_active", "gnss_std")}) for sh in shards[r]]
          for r in range(G)]
    dl_arr = [(BaProblem * B)(*[to_struct(p) for p in dl[r]]) for r in range(G)]
    full = [dict(p, **{k: np.array(p[k], copy=True) for k in ("pose", "mix", "ext", "invdepth", "f_active", "gnss_std")}) for p in probs]
    full_arr = (BaProblem * B)(*[to_struct(p) for p in full])
    single_call = post_solve_call(single, full, cis)

    def sharded():
        on_ranks(lambda r: rank_calls[r]())

    def on_twin():
        twin_call()

    def replaced():
        summ = (BaSummary * B)()
        for r in range(G):  # download both shards into the host arrays
            check(lib().icg_ba_download(ranks[r]._h, B, dl_arr[r], summ), "icg_ba_download")
        for w in range(B):
            for r in range(G):
                merge_shard(full[w], dl[r][w])
        check(lib().icg_ba_upload(single._h, B, full_arr), "icg_ba_upload")
        single_call()

    fns = dict(sharded=sharded, twin=on_twin, replaced=replaced)
    for f in fns.values():  # warm-up: first launches, staging and workspace allocations
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(args.reps):
        for k, f in fns.items():
            t0 = time.perf_counter()
            f()
            times[k].append((time.perf_counter() - t0) * 1e3)
    for s in ranks + [twin, single]:
        s.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    exp_bytes = [8 * (2 * B + B * caps[r]["F"] * 16) for r in range(G)]
    print(json.dumps(dict(bench="shard_post_solve", windows=B, K=K, L=L, ranks=G, reps=args.reps, gpu=smi.splitlines()[0] if smi else "?",
                          median_ms={k: float(np.median(v)) for k, v in times.items()}, min_ms={k: float(np.min(v)) for k, v in times.items()},
                          export_region_bytes_per_rank=exp_bytes, shard_max_F=[c["F"] for c in caps])))


if __name__ == "__main__":
    main()
