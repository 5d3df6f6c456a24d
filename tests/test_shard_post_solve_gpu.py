"""GPU: the post-solve culling (icg_ba_update_and_cull_resident) and the resident marginalization (icg_ba_marginalize_resident[_culled]) on
landmark-sharded handles.  The ranks are `world` handles on cuda:0 of this process, connected with plain pointers, one host thread per rank
(the in-process harness of tests/test_ba_gpu.py).  Each sharded result is compared bit for bit with an unsharded twin handle that holds the
merged solved values: the camera outputs and counters on every rank, the landmark outputs merged by shard range, and every window's prior
on its owner (rank w mod world).  A spawn test repeats the comparison with one process per GPU where the box has two or more."""
import copy
import ctypes as C
import os
import socket
import threading

import numpy as np
import pytest

from tests import oracle_api as oa
from tests.test_post_solve_gpu import CAMD, STD, cull_inputs, make, olib  # noqa: F401  (olib: fixture)

pytestmark = pytest.mark.gpu

PRIOR_KEYS = ("block_type", "block_node", "x0", "J0", "e0", "Hp", "bp")
CAM_KEYS = ("R_bc_out", "t_bc_out", "cam_pose", "counts")
LM_KEYS = ("lm_pw", "lm_depth", "lm_outlier", "obs_outlier")


def run_ranks(world, fn):
    out, errs = [None] * world, []

    def body(r):
        try:
            out[r] = fn(r)
        except Exception as e:  # noqa: BLE001
            errs.append((r, repr(e)))
    th = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(300)
    assert not errs, errs
    return out


def marg_landmarks_last(prob, nm):
    """the same window with the landmarks anchored in the removed nodes renumbered to the end (factors listed landmark by landmark): with
    two ranks every one of them lives on rank 1"""
    f_lm, f_ref = np.asarray(prob["f_lm"]), np.asarray(prob["f_ref"])
    L = prob["L"]
    ref = np.full(L, 99)
    ref[f_lm] = f_ref
    order = np.argsort(ref < nm, kind="stable")
    new_of = np.empty(L, np.int64)
    new_of[order] = np.arange(L)
    fo = np.argsort(new_of[f_lm], kind="stable")
    q = copy.deepcopy(prob)
    q.update(invdepth=np.asarray(prob["invdepth"])[order].copy(), f_lm=new_of[f_lm][fo].astype(np.int32), f_ref=f_ref[fo].astype(np.int32),
             f_obs=np.asarray(prob["f_obs"])[fo].astype(np.int32), f_const=prob["f_const"].reshape(-1, 14)[fo].reshape(-1).copy(),
             f_active=np.asarray(prob["f_active"])[fo].copy())
    return q


def flag_reference_observations(ci, nm, count):
    """move the reference keypoint of `count` landmarks anchored in the removed nodes: the culling flags the reference observation and
    the whole landmark leaves the culled marginalization"""
    done = 0
    for l in range(len(ci["lm_ref_node"])):
        if ci["lm_ref_node"][l] >= nm or done == count:
            continue
        for o in range(ci["obs_off"][l], ci["obs_off"][l + 1]):
            if ci["obs_factor"][o] < 0:
                ci["obs_kp"][o, 0] += 12.0
                done += 1
    assert done == count


def marginalize_nan(solver, probs, nm):
    """the plain resident marginalization with every output array filled with NaN first (non-owner arrays must stay so)"""
    from ic_gvins_b200._lib import check, lib
    from ic_gvins_b200.ba import vp
    call = solver.marg_prepare(probs, nm)
    for b in call["bufs"]:
        for k in ("x0", "J0", "e0", "Hp", "bp"):
            b[k][:] = np.nan
        b["bt"][:], b["bn"][:] = -7, -7
    check(lib().icg_ba_marginalize_resident(solver._h, call["n"], call["arr"], vp(call["nm"].ctypes.data), call["pri"]), "icg_ba_marginalize_resident")
    return solver.marg_collect(call), call


def solve_sharded(probs, world, K, iters, max_marg_r):
    from ic_gvins_b200.ba import WindowSolver, shard_window
    n = len(probs)
    shards = [[shard_window(p, r, world) for p in probs] for r in range(world)]
    solvers = [WindowSolver(max_windows=n, max_K=K, max_L=max(1, max(s["L"] for s in shards[r])), max_F=max(1, max(s["F"] for s in shards[r])),
                            max_gnss=16, max_marg_r=max_marg_r) for r in range(world)]
    blobs = [solvers[r].shard_export(r, world) for r in range(world)]
    for sv in solvers:
        sv.shard_connect(blobs)
    run_ranks(world, lambda r: solvers[r].gvins_optimization_batch(shards[r], iters))
    merged = []
    for w, p in enumerate(probs):
        full = copy.deepcopy(p)
        for r in range(world):
            sh = shards[r][w]
            full["invdepth"][sh["lm_lo"]:sh["lm_hi"]] = sh["invdepth"]
            full["f_active"][sh["f_index"]] = sh["f_active"]
        for key in ("pose", "mix", "ext", "gnss_std"):
            full[key] = shards[0][w][key].copy()
        merged.append(full)
    return solvers, shards, merged


def post_solve_twin(probs, world, K, L, nm, iters=12, max_marg_r=160, ref_flags=0, seed=0):
    """solve sharded, then cull + culled marginalization + plain marginalization on the ranks and on the twin; compare everything"""
    from ic_gvins_b200.ba import WindowSolver, merge_cull_shard, shard_cull_inputs
    n = len(probs)
    ext0 = [p["ext"].copy() for p in probs]
    solvers, shards, merged = solve_sharded(probs, world, K, iters, max_marg_r)
    try:
        cis = [cull_inputs(p, e, seed + w, bad_kp=20) for w, (p, e) in enumerate(zip(merged, ext0))]
        if ref_flags:
            for ci in cis:
                if len(ci["lm_ref_node"]):
                    flag_reference_observations(ci, nm, ref_flags)
        nim = [np.ones(p["K"], np.uint8) for p in probs]
        nim[-1][-2] = 0
        sci = [[shard_cull_inputs(cis[w], shards[r][w]) for w in range(n)] for r in range(world)]

        def rank(r):
            g = solvers[r].update_and_cull(shards[r], cam_struct(), STD, sci[r])
            mc = solvers[r].marginalize(shards[r], nm, resident=True, culled=g, node_in_map=nim)
            mp, call = marginalize_nan(solvers[r], shards[r], nm)
            for w, buf in enumerate(call["bufs"]):  # a non-owner's output arrays are not written
                if w % world != r:
                    assert all(np.isnan(buf[k]).all() for k in ("x0", "J0", "e0", "Hp", "bp")) and (buf["bt"] == -7).all(), (w, r)
                    assert call["pri"][w].nblocks == 0
            return g, mc, mp
        res = run_ranks(world, rank)
    finally:
        for sv in solvers:
            sv.close()
    twin = WindowSolver(max_windows=n, max_K=K, max_L=max(1, L), max_F=max(1, max(p["F"] for p in merged)), max_gnss=16, max_marg_r=max_marg_r)
    try:
        twin.upload(merged)
        gt = twin.update_and_cull(merged, cam_struct(), STD, cis)
        mct = twin.marginalize(merged, nm, resident=True, culled=gt, node_in_map=nim)
        mpt = twin.marginalize(merged, nm, resident=True)
    finally:
        twin.close()
    for w in range(n):
        full = {k: np.zeros_like(gt[w][k]) for k in LM_KEYS}
        full["obs_off"] = gt[w]["obs_off"]
        for r in range(world):
            g = res[r][0][w]
            for k in CAM_KEYS:
                assert np.array_equal(g[k], gt[w][k]), (w, r, k)
            assert g["ext_accepted"] == gt[w]["ext_accepted"] and g["td_bc_out"] == gt[w]["td_bc_out"]
            merge_cull_shard(full, shards[r][w], g)
        for k in LM_KEYS:
            assert np.array_equal(full[k], gt[w][k], equal_nan=gt[w][k].dtype.kind == "f"), (w, k)
        for r in range(world):
            for got, want in ((res[r][1][w], mct[w]), (res[r][2][w], mpt[w])):
                if r == w % world:
                    assert got["m"] == want["m"] > 0 and got["r"] == want["r"], (w, r)
                    for key in PRIOR_KEYS:
                        assert np.array_equal(got[key], want[key]), (w, r, key)
                else:
                    assert got["m"] == 0 and got["r"] == 0 and len(got["block_type"]) == 0, (w, r)
    return gt, mct, res


_CAM = {}


def cam_struct():
    if "c" not in _CAM:
        from ic_gvins_b200.camera import Camera
        _CAM["c"] = Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])
    return _CAM["c"]


@pytest.mark.parametrize("world", [2, 3])
def test_cfg3_twin_equality(olib, world):
    n = 2 * world + 1
    probs = [make(olib, outliers=20, seed=400 + w, K=10, L=300, with_marg=(w % 2 == 1)) for w in range(n)]
    gt, mct, _ = post_solve_twin(probs, world, 10, 300, 1, seed=500, ref_flags=2)
    assert sum(int(g["counts"][2]) for g in gt) >= len(gt)  # reference observations were flagged in every window


def test_cfg4_split_pipeline_with_prior(olib):
    probs = [make(olib, outliers=30, seed=430 + w, K=20, L=2000, with_marg=(w % 2 == 0)) for w in range(4)]
    assert probs[0]["marg_r"] > 0  # the handle carries a prior into the marginalization
    post_solve_twin(probs, 2, 20, 2000, 1, iters=8, max_marg_r=292, seed=530)


def test_edges_num_marg_2_empty_shard_and_marginalized_landmarks_off_the_owner(olib):
    """num_marg = 2; window 0 (owned by rank 0) has every marginalized landmark on rank 1; window 1 has no landmark at all (every shard
    L = 0, every export empty); window 2 has 3 landmarks (rank 0's shard is empty of marginalized rows in some windows)"""
    base = [make(olib, outliers=10, seed=460 + w, K=8, L=L) for w, L in enumerate((200, 0, 3, 150))]
    probs = [marg_landmarks_last(base[0], 2)] + base[1:]
    p0 = probs[0]
    marg_lm = np.unique(p0["f_lm"][p0["f_ref"] < 2])
    assert len(marg_lm) and marg_lm.min() >= p0["L"] // 2  # rank 1's block: the owner (rank 0) exports no row of window 0
    post_solve_twin(probs, 2, 8, 200, 2, iters=8, seed=560, ref_flags=1)


def test_unchanged_calls_still_rejected_and_resolve_is_unaffected(olib):
    from ic_gvins_b200 import IcgError
    probs = [make(olib, outliers=10, seed=480 + w, K=10, L=300) for w in range(4)]

    def chain(reject):
        solvers, shards, _ = solve_sharded(copy.deepcopy(probs), 2, 10, 12, 160)
        try:
            def rank(r):
                s, sh = solvers[r], shards[r]
                if reject:
                    with pytest.raises(IcgError, match="landmark-sharded"):
                        s.marginalize(sh, 1)
                    with pytest.raises(IcgError, match="landmark-sharded"):
                        s.reintegrate(sh, np.ones(5), np.zeros(3), [None] * len(sh), reintegrate=[0] * len(sh))
                    with pytest.raises(IcgError, match="landmark-sharded"):
                        s.slide(sh, [{} for _ in sh])
                    with pytest.raises(IcgError, match="landmark-sharded"):
                        s.slide_integrate(sh, [{} for _ in sh], [None] * len(sh), np.ones(5))
                s.run_gvins(12, restart=True)
                s.gvins_optimization_end(sh)
                return [{k: p[k].copy() for k in ("pose", "mix", "ext", "invdepth", "f_active")} for p in sh]
            return run_ranks(2, rank)
        finally:
            for sv in solvers:
                sv.close()
    a, b = chain(True), chain(False)
    for ra, rb in zip(a, b):
        for wa, wb in zip(ra, rb):
            for k in wa:
                assert np.array_equal(wa[k], wb[k]), k


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import oracle
        from datagen import synth_ba
        from ic_gvins_b200.ba import WindowSolver, connect_shards, shard_cull_inputs, shard_window
        from ic_gvins_b200.camera import Camera
        olib_ = C.CDLL(oracle.build())
        oa.declare(olib_)
        oa.declare_ba(olib_)
        n = 2 * world
        probs = [synth_ba.make_window(lambda *a: oa.preintegrate(olib_, *a), K=10, L=300, seed=2200 + w, with_marg=(w % 2 == 1))[0] for w in range(n)]
        ext0 = [p["ext"].copy() for p in probs]
        shards = [shard_window(p, rank, world) for p in probs]
        s = WindowSolver(max_windows=n, max_K=10, max_L=max(1, max(sh["L"] for sh in shards)), max_F=max(1, max(sh["F"] for sh in shards)),
                         max_gnss=16, max_marg_r=160, device=rank)
        connect_shards(s, rank, world, "p2p", dist)
        s.gvins_optimization_batch(shards, 12)
        parts = [None] * world
        dist.all_gather_object(parts, [(sh["lm_lo"], sh["lm_hi"], sh["invdepth"], sh["f_index"], sh["f_active"]) for sh in shards])
        merged = []
        for w, p in enumerate(probs):
            full = copy.deepcopy(p)
            for lo, hi, rho, fi, act in (parts[r][w] for r in range(world)):
                full["invdepth"][lo:hi], full["f_active"][fi] = rho, act
            for key in ("pose", "mix", "ext", "gnss_std"):
                full[key] = shards[w][key].copy()
            merged.append(full)
        cam_ = Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])
        cis = [cull_inputs(p, e, 2300 + w, bad_kp=20) for w, (p, e) in enumerate(zip(merged, ext0))]
        g = s.update_and_cull(shards, cam_, STD, [shard_cull_inputs(ci, sh) for ci, sh in zip(cis, shards)])
        mc = s.marginalize(shards, 1, resident=True, culled=g)
        s.close()
        outs = [None] * world
        dist.all_gather_object(outs, ([{k: x[k] for k in CAM_KEYS + LM_KEYS + ("ext_accepted", "td_bc_out")} for x in g], mc, shards))
        if rank == 0:
            with torch.cuda.device(0):
                twin = WindowSolver(max_windows=n, max_K=10, max_L=300, max_F=max(p["F"] for p in merged), max_gnss=16, max_marg_r=160, device=0)
                twin.upload(merged)
                gt = twin.update_and_cull(merged, cam_, STD, cis)
                mct = twin.marginalize(merged, 1, resident=True, culled=gt)
                twin.close()
            from ic_gvins_b200.ba import merge_cull_shard
            for w in range(n):
                full = {k: np.zeros_like(gt[w][k]) for k in LM_KEYS}
                full["obs_off"] = gt[w]["obs_off"]
                for r in range(world):
                    gr = outs[r][0][w]
                    for k in CAM_KEYS:
                        assert np.array_equal(gr[k], gt[w][k]), (w, r, k)
                    assert gr["ext_accepted"] == gt[w]["ext_accepted"] and gr["td_bc_out"] == gt[w]["td_bc_out"], (w, r)
                    merge_cull_shard(full, outs[r][2][w], gr)
                for k in LM_KEYS:
                    assert np.array_equal(full[k], gt[w][k], equal_nan=gt[w][k].dtype.kind == "f"), (w, k)
                got = outs[w % world][1][w]
                assert got["m"] == mct[w]["m"] > 0
                for key in PRIOR_KEYS:
                    assert np.array_equal(got[key], mct[w][key]), (w, key)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + repr(e) + "\n" + traceback.format_exc()))


@pytest.mark.skipif(_ngpu() < 2, reason="needs two or more GPUs")
def test_multi_gpu_twin_equality():
    import torch.multiprocessing as mp
    world = 2
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    try:
        res = dict(q.get(timeout=600) for _ in range(world))
    finally:
        for p in ps:
            p.join(60)
            if p.is_alive():
                p.kill()
    assert all(v == "ok" for v in res.values()), res
