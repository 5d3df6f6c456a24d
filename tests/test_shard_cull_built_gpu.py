"""GPU: icg_ba_shard_update_and_cull_built.  The ranks are in-process handles on cuda:0.  Group A slides with
icg_ba_shard_slide_vision_resident, which also writes each rank's next culling lists on the device, then culls on those lists and passes NULL
lists to the culled marginalization and a NULL obs_factor to the next vision slide; twin group B makes the same calls but culls on host lists
through the sharded icg_ba_update_and_cull_resident.  Each rank's built lists must equal the per-rank list rule (tests/cull_lists_oracle.py on
the rank's own shard) exactly, the lists merged rank-major must be an unsharded handle's built lists, and the two groups must give the same
bits: culling outputs, the owners' priors, the next slide and the solves after it."""
import copy
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import shard_vision_oracle as sv
from tests import slide_vision_oracle as so
from tests.cull_lists_oracle import next_lists
from tests.test_cull_built_gpu import ext_of
from tests.test_post_solve_gpu import STD, make, olib  # noqa: F401  (olib: fixture)
from tests.test_shard_post_solve_gpu import CAM_KEYS, LM_KEYS, PRIOR_KEYS, cam_struct, run_ranks
from tests.test_shard_slide_gpu import PARAMS, close, merge, post_solve
from tests.test_shard_slide_vision_gpu import group, whole_cull
from tests.test_slide_vision_gpu import Keyframe, host_twin

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LISTS = ("lm_ref_node", "lm_ref_kp", "obs_off", "obs_node", "obs_kp", "obs_factor")
INT_LISTS = ("lm_ref_node", "obs_off", "obs_node", "obs_factor")


def rank_rule(prev, res, kf, sh):
    """the list rule on one rank: its last culling `prev` (shard-local lists and flags), its built shard `res` (lm_origin, f_src, f_lm, f_obs)
    and the keyframe's observations of its own landmarks"""
    lo, hi = int(sh["lm_lo"]), int(sh["lm_hi"])
    onode = np.full(kf.K_old, -1)
    for j, i in enumerate(kf.carry["node_src"]):
        if 1 <= i < kf.K_old and kf.in_map[i]:
            onode[i] = j
    xy = {(l - lo, nd): kf.xy[i] for i, (l, nd) in enumerate(kf.obs) if lo <= l < hi}
    pts = [dict(ref_node=kf.frames[int(kf.new["ref_id"][j])], ref_xy=kf.new["ref_xy"][j], cur_xy=kf.new["cur_xy"][j]) for j in range(len(kf.new["depth"]))]
    return next_lists(prev, prev["obs_outlier"], onode, res, xy, pts, kf.cur)


def merged_lists(ranks, shards_w):
    """the whole window's lists from the ranks' shard-local ones: rank-major, factor ids mapped through each shard's f_index"""
    out = {k: [] for k in LISTS}
    off, base = [np.zeros(1, np.int64)], 0
    for g, sh in zip(ranks, shards_w):
        f, fi = np.asarray(g["obs_factor"], np.int64), np.asarray(sh["f_index"], np.int64)
        out["obs_factor"].append(np.where(f >= 0, fi[np.clip(f, 0, max(len(fi) - 1, 0))] if len(fi) else -1, -1))
        for k in ("lm_ref_node", "lm_ref_kp", "obs_node", "obs_kp"):
            out[k].append(np.asarray(g[k]))
        off.append(np.asarray(g["obs_off"][1:], np.int64) + base)
        base += int(g["obs_off"][-1])
    r = {k: np.concatenate(v) for k, v in out.items() if k != "obs_off"}
    r.update(obs_off=np.concatenate(off).astype(np.int32), obs_factor=r["obs_factor"].astype(np.int32), lm_ref_node=r["lm_ref_node"].astype(np.int32),
             obs_node=r["obs_node"].astype(np.int32), lm_ref_kp=r["lm_ref_kp"].astype(np.float32).reshape(-1, 2),
             obs_kp=r["obs_kp"].astype(np.float32).reshape(-1, 2), n_obs=base)
    return r


def same_lists(x, y, keys=LISTS):
    for k in keys:
        assert np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes(), k


def built(S, r, shards, exts):
    """rank r's built culling with obs_factor kept (shard_update_and_cull_built's dicts without it are derived from these)"""
    return S[r]._cull_built("icg_ba_shard_update_and_cull_built", shards, cam_struct(), STD, exts)


def bare(gs):
    return [{k: v for k, v in g.items() if k not in INT_LISTS} for g in gs]


def chain(probs, world, K, R, iters, seed, n_kf, twin=True):
    """n_kf keyframes: the first culls on host lists in both groups; from the second on A culls on its built lists with NULL lists after it"""
    from ic_gvins_b200.ba import WindowSolver, shard_next, shard_vision_inputs
    n = len(probs)
    A, sa, ma = group(copy.deepcopy(probs), world, K, iters, R)
    B, sb, _ = group(copy.deepcopy(probs), world, K, iters, R)
    try:
        refs = [so.reference_rows(p) for p in ma]
        want = None
        for c in range(n_kf + 1):
            if c == 0:
                ga, pa, cis = post_solve(A, sa, ma, world, seed)
                gb, pb, _ = post_solve(B, sb, ma, world, seed)
                gw = [whole_cull(cis[w], [ga[r][w] for r in range(world)], [sa[r][w] for r in range(world)]) for w in range(n)]
            else:
                exts = [ext_of(p) for p in sa[0]]
                full = run_ranks(world, lambda r: built(A, r, sa[r], exts))
                gb = run_ranks(world, lambda r: B[r].update_and_cull(sb[r], cam_struct(), STD, [dict(e, **{k: want[r][w][k] for k in LISTS})
                                                                                               for w, e in enumerate(exts)]))
                for r in range(world):
                    for w in range(n):
                        assert full[r][w]["n_obs"] == want[r][w]["n_obs"] == sa[r][w]["L"] + sa[r][w]["F"], (c, r, w)
                        same_lists(full[r][w], want[r][w])
                        for k in CAM_KEYS + LM_KEYS:
                            assert np.array_equal(full[r][w][k], gb[r][w][k]), (c, r, w, k)
                        assert full[r][w]["td_bc_out"] == gb[r][w]["td_bc_out"] and full[r][w]["ext_accepted"] == gb[r][w]["ext_accepted"]
                ga = [[dict(g) for g in rg] for rg in full]
                for rg in ga:
                    for g in rg:
                        g.pop("obs_factor")  # what shard_update_and_cull_built returns
                pa = run_ranks(world, lambda r: A[r].marginalize(sa[r], 1, resident=True, culled=bare(ga[r])))
                pb = run_ranks(world, lambda r: B[r].marginalize(sb[r], 1, resident=True, culled=gb[r]))
                for r in range(world):
                    for w in range(r, n, world):
                        for k in PRIOR_KEYS:
                            assert np.array_equal(pa[r][w][k], pb[r][w][k]), (c, r, w, k)
                gw = [whole_cull(merged_lists([gb[r][w] for r in range(world)], [sb[r][w] for r in range(world)]), [gb[r][w] for r in range(world)],
                                 [sb[r][w] for r in range(world)]) for w in range(n)]
            if c == n_kf:
                break
            kfs = [Keyframe(ma[w], gw[w], pa[w % world][w], refs[w], seed + 100 * c + w) for w in range(n)]
            os_ = [kf.oracle(ma[w], refs[w]) for w, kf in enumerate(kfs)]
            vis = [kf.device() for kf in kfs]
            na = [[copy.deepcopy(kf.nxt) for kf in kfs] for _ in range(world)]
            nb = copy.deepcopy(na)
            ca = [[{k: v for k, v in kf.carry.items() if k not in ("lm_src", "f_src")} for kf in kfs] for _ in range(world)]
            cb = copy.deepcopy(ca)
            va = [[shard_vision_inputs(vis[w], sa[r][w], ga[r][w]) for w in range(n)] for r in range(world)]
            vb = [[shard_vision_inputs(vis[w], sb[r][w], gb[r][w]) for w in range(n)] for r in range(world)]
            if c > 0:
                assert all(v["obs_factor"] is None for rv in va for v in rv)
            ra = run_ranks(world, lambda r: A[r].shard_slide_vision(na[r], ca[r], va[r]))
            rb = run_ranks(world, lambda r: B[r].shard_slide_vision(nb[r], cb[r], vb[r]))
            wholes = []
            for w, (kf, o) in enumerate(zip(kfs, os_)):
                prev = [sa[r][w] for r in range(world)]
                q, cq = host_twin(kf.nxt, kf.carry, o)
                wb, _, parts = shard_next(q, cq, prev, sv.new_rank(o, prev, w))
                wholes.append(wb)
                for r in range(world):
                    for k in ra[r][w]:
                        assert np.array_equal(ra[r][w][k], rb[r][w][k]), (c, r, w, k)
                    for x in (na[r][w], nb[r][w]):
                        x.update(lm_lo=parts[r][0]["lm_lo"], lm_hi=parts[r][0]["lm_hi"], f_index=parts[r][0]["f_index"])
            # every rank's built lists: the list rule on the rank's own shard
            want = [[rank_rule(gb[r][w], ra[r][w], kfs[w], sb[r][w]) for w in range(n)] for r in range(world)]
            if twin and c == 0:  # merged rank-major through f_index: what an unsharded handle builds on the merged window, reordered
                T = WindowSolver(max_windows=n, max_K=K, max_L=max(max(p["L"] for p in ma), max(o["L"] for o in os_)),
                                 max_F=max(max(p["F"] for p in ma), max(o["F"] for o in os_)), max_gnss=16, max_marg_r=R)
                try:
                    T.upload([copy.deepcopy(p) for p in ma])
                    gt = T.update_and_cull(ma, cam_struct(), STD, cis)
                    T.marginalize(ma, 1, resident=True, culled=gt)
                    tn = [copy.deepcopy(kf.nxt) for kf in kfs]
                    rt = T.slide_vision(tn, [copy.deepcopy(kf.carry) for kf in kfs], vis)
                    gt = T.update_and_cull_built(tn, cam_struct(), STD, [ext_of(p) for p in tn])
                finally:
                    T.close()
                for w in range(n):
                    prev = [sa[r][w] for r in range(world)]
                    order = sv.rank_order(rt[w], prev, w)
                    new_of = np.empty(len(order), np.int64)
                    new_of[order] = np.arange(len(order))
                    pos = np.empty(rt[w]["F"], np.int64)  # unsharded factor -> its row in the rank-major window
                    pos[np.argsort(new_of[rt[w]["f_lm"]], kind="stable")] = np.arange(rt[w]["F"])
                    m = merged_lists([want[r][w] for r in range(world)], [na[r][w] for r in range(world)])
                    off = gt[w]["obs_off"]
                    idx = np.concatenate([np.arange(off[l], off[l + 1]) for l in order]).astype(np.int64)
                    f = gt[w]["obs_factor"][idx]
                    t = dict(lm_ref_node=gt[w]["lm_ref_node"][order], lm_ref_kp=gt[w]["lm_ref_kp"][order], obs_node=gt[w]["obs_node"][idx],
                             obs_kp=gt[w]["obs_kp"][idx], obs_factor=np.where(f >= 0, pos[np.maximum(f, 0)], -1).astype(np.int32),
                             obs_off=np.r_[0, np.cumsum(np.diff(off)[order])].astype(np.int32))
                    same_lists(m, t)
            for grp in (A, B):
                run_ranks(world, lambda r: grp[r].run_gvins(20))
            assert run_ranks(world, lambda r: A[r].gvins_optimization_end(na[r])) == run_ranks(world, lambda r: B[r].gvins_optimization_end(nb[r]))
            for r in range(world):
                for w in range(n):
                    for k in PARAMS:
                        assert np.array_equal(na[r][w][k], nb[r][w][k]), (c, r, w, k)
            refs = [o["lm_ref"][sv.rank_order(o, [sa[r][w] for r in range(world)], w)] for w, o in enumerate(os_)]
            sa, sb = na, nb
            ma = [merge([nb[r][w] for r in range(world)], wholes[w], blobs=False) for w in range(n)]
        return A, B, sa, ga
    except BaseException:
        close(A, B)
        raise


def mixed(olib, seed):
    return [make(olib, outliers=25, seed=seed, K=10, L=300), make(olib, outliers=10, seed=seed + 1, K=8, L=150),
            make(olib, outliers=25, seed=seed + 2, K=10, L=200)]


@pytest.mark.parametrize("world", [2, 3])
def test_cfg3_mixed_batch_three_keyframes_with_null_lists(olib, world):
    """three keyframes on a mixed cfg-3 batch: built culling, culled marginalization with NULL lists, vision slide with NULL obs_factor"""
    A, B, _, _ = chain(mixed(olib, 5100 + 10 * world), world, 10, 160, 12, 5150 + world, 3)
    close(A, B)


def test_cfg4_split_pipeline(olib):
    from tests.test_marg_large_gpu import make as make_large
    probs = [make_large(olib, K=20, L=2000, seed=5200 + w, n_ref=20, prior=True) for w in range(2)]
    A, B, _, _ = chain(probs, 2, 20, 292, 8, 5210, 1, twin=False)
    close(A, B)


def test_contract(olib):
    """before any vision slide; a rejection on one rank (every rank ICG_EINVAL, every handle unchanged, the corrected retry succeeds); non-NULL
    list inputs; a rejected vision slide keeps the lists current; after shard_slide and shard_slide_integrate they are gone"""
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200.ba import shard_next, shard_vision_inputs
    from tests.test_slide_integrate_gpu import NOISE5
    world, n = 2, 2
    probs = [make(olib, outliers=25, seed=5300 + w, K=10, L=300) for w in range(n)]
    A, sa, ma = group(copy.deepcopy(probs), world, 10, 12, 160, extra_L=(0, 400), extra_F=(256, 800))
    try:
        def reject(args, match):
            def rank(r):
                with pytest.raises(IcgError, match=match[r]) as e:
                    A[r].shard_update_and_cull_built(*args(r))
                assert e.value.code == -1  # ICG_EINVAL
            run_ranks(world, rank)

        exts = [ext_of(p) for p in sa[0]]
        reject(lambda r: (sa[r], cam_struct(), STD, exts), ["no built lists", "no built lists"])
        ga, pa, cis = post_solve(A, sa, ma, world, 5310)
        gw = [whole_cull(cis[w], [ga[r][w] for r in range(world)], [sa[r][w] for r in range(world)]) for w in range(n)]
        kfs = [Keyframe(ma[w], gw[w], pa[w % world][w], so.reference_rows(ma[w]), 5320 + w) for w in range(n)]
        na = [[copy.deepcopy(kf.nxt) for kf in kfs] for _ in range(world)]
        ca = [[{k: v for k, v in kf.carry.items() if k not in ("lm_src", "f_src")} for kf in kfs] for _ in range(world)]
        vis = [kf.device() for kf in kfs]
        res = run_ranks(world, lambda r: A[r].shard_slide_vision(na[r], ca[r], [shard_vision_inputs(vis[w], sa[r][w], ga[r][w]) for w in range(n)]))
        want = [[rank_rule(ga[r][w], res[r][w], kfs[w], sa[r][w]) for w in range(n)] for r in range(world)]
        for w, kf in enumerate(kfs):
            prev = [sa[r][w] for r in range(world)]
            o = kf.oracle(ma[w], so.reference_rows(ma[w]))
            parts = shard_next(*host_twin(kf.nxt, kf.carry, o), prev, sv.new_rank(o, prev, w))[2]
            for r in range(world):
                na[r][w].update(lm_lo=parts[r][0]["lm_lo"], lm_hi=parts[r][0]["lm_hi"], f_index=parts[r][0]["f_index"])
        run_ranks(world, lambda r: A[r].run_gvins(20))
        run_ranks(world, lambda r: A[r].gvins_optimization_end(na[r]))
        exts = [ext_of(p) for p in na[0]]
        # lists current for these windows on rank 0 only: rank 1 names one window fewer
        reject(lambda r: (na[r][:n - r], cam_struct(), STD, exts[:n - r]), ["rank 1 .*rejected", "holds 2 uploaded windows"])
        # the extrinsic inputs differ between the ranks
        reject(lambda r: (na[r], cam_struct(), STD, [dict(e, td_bc=e["td_bc"] + r) for e in exts]), ["camera sides differ"] * 2)
        g1 = run_ranks(world, lambda r: built(A, r, na[r], exts))  # the corrected retry
        for r in range(world):
            for w in range(n):
                same_lists(g1[r][w], want[r][w])
        # non-NULL list inputs on rank 0: rejected before the agreement, every handle unchanged (the NULL lists below are this culling's)
        def rank_lists(r):
            import ctypes as C
            from ic_gvins_b200._lib import BaProblem, CullLists, CullWindow, lib
            from ic_gvins_b200.ba import cull_struct, to_struct
            arr = (BaProblem * n)(*[to_struct(p) for p in na[r]])
            keep = [dict(e, obs_factor=np.zeros(3, np.int32)) if (r, w) == (0, 1) else dict(e) for w, e in enumerate(exts)]
            cw = (CullWindow * n)(*[cull_struct(p, ci) for p, ci in zip(na[r], keep)])
            flags = [np.zeros(A[r].max_L + A[r].max_F, np.uint8) for _ in range(n)]
            for w in range(n):
                cw[w].obs_outlier = flags[w].ctypes.data_as(C.POINTER(C.c_uint8))
            rc = lib().icg_ba_shard_update_and_cull_built(A[r]._h, n, arr, C.byref(cam_struct().c if hasattr(cam_struct(), 'c') else cam_struct()), float(STD), cw, (CullLists * n)())
            return rc, lib().icg_last_error().decode()
        out = run_ranks(world, rank_lists)
        assert out[0][0] == out[1][0] == -1 and "inputs must be NULL" in out[0][1] and "rank 0" in out[1][1], out
        bare_g = [[{k: v for k, v in g.items() if k not in INT_LISTS} for g in rg] for rg in g1]
        run_ranks(world, lambda r: A[r].marginalize(na[r], 1, resident=True, culled=bare_g[r]))
        # a vision slide rejected on every rank (rank 0 has no room for window 0's new points) keeps the lists current
        big = Keyframe(ma[0], gw[0], pa[0][0], so.reference_rows(ma[0]), 5330, n_new=2 * A[0].max_L)
        bv = [big.device(), vis[1]]

        def slide_rejected(r):
            with pytest.raises(IcgError) as e:
                strip = [{k: v for k, v in kf.carry.items() if k not in ("lm_src", "f_src")} for kf in (big, kfs[1])]
                A[r].shard_slide_vision([copy.deepcopy(big.nxt), copy.deepcopy(kfs[1].nxt)], strip,
                                        [shard_vision_inputs(bv[w], na[r][w], {}) for w in range(n)])
            assert e.value.code == -1
        run_ranks(world, slide_rejected)
        g2 = run_ranks(world, lambda r: built(A, r, na[r], exts))
        for r in range(world):
            for w in range(n):
                same_lists(g2[r][w], want[r][w])
                for k in CAM_KEYS + LM_KEYS:
                    assert np.array_equal(g2[r][w][k], g1[r][w][k]), (r, w, k)
        # another slide ends them: the window onto itself, every row carried
        same = [[dict(node_src=np.arange(p["K"], dtype=np.int32), lm_src=np.arange(p["L"], dtype=np.int32), f_src=np.arange(p["F"], dtype=np.int32),
                      imu_src=np.arange(p["n_imu"], dtype=np.int32), gnss_src=np.arange(p["n_gnss"], dtype=np.int32)) for p in na[r]] for r in range(world)]
        run_ranks(world, lambda r: A[r].shard_slide(copy.deepcopy(na[r]), same[r], False))
        reject(lambda r: (na[r], cam_struct(), STD, exts), ["no built lists", "no built lists"])
        run_ranks(world, lambda r: A[r].shard_slide_integrate(copy.deepcopy(na[r]), same[r], [{}] * n, NOISE5, prior_from_marg=False))
        reject(lambda r: (na[r], cam_struct(), STD, exts), ["no built lists", "no built lists"])
    finally:
        close(A)
    # outside a shard group
    from ic_gvins_b200.ba import WindowSolver
    one = WindowSolver(max_windows=1, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=160)
    try:
        p = copy.deepcopy(probs[0])
        one.gvins_optimization_batch([p], 8)
        with pytest.raises(IcgError, match="not in a landmark-shard group.*icg_ba_update_and_cull_built") as e:
            one.shard_update_and_cull_built([p], cam_struct(), STD, [ext_of(p)])
        assert e.value.code == -1
    finally:
        one.close()


SHIM = r'''
#include <cstdio>
#include "ic_gvins_b200/host/icg_shims.hpp"
// links and runs WindowSolver::shardUpdateAndCullBuilt: outside a shard group it must throw, naming the call
int main() {
    icg_b200::WindowSolver s(10, 300, 2700);
    icg_ba_problem p{};
    icg_camera cam{};
    icg_ba_cull_window io{};
    icg_ba_cull_lists lists{};
    try {
        s.shardUpdateAndCullBuilt(p, cam, 1.0, io, &lists);
    } catch (const std::exception &e) {
        printf("%s\n", e.what());
        return 0;
    }
    return 1;
}
'''


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_shim_shard_update_and_cull_built_runs():
    """the C++ member compiles, links against the library and reaches the call"""
    lib = os.path.join(ROOT, "ic_gvins_b200", "libicgvins_b200.so")
    tmp = tempfile.mkdtemp()
    try:
        src, exe = os.path.join(tmp, "t.cpp"), os.path.join(tmp, "t")
        with open(src, "w") as f:
            f.write(SHIM)
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, src, "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "icg_ba_shard_update_and_cull_built" in r.stdout and "not in a landmark-shard group" in r.stdout
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
