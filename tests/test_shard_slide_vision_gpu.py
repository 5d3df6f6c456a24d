"""GPU: icg_ba_shard_slide_vision_resident.  The ranks are in-process handles on cuda:0 (run_ranks).  Group A solves, culls and marginalizes
landmark-sharded windows, then slides with each rank building its own next shard on the device (shard_slide_vision); group B, the same ranks
through the same calls, takes the host path: the whole-window numpy restatement (tests/slide_vision_oracle.py), shard_next with the new-point
rule, and shard_slide[_integrate].  Each rank's built shard must equal shard_next's exactly (inverse depths and new factor rows bit for bit),
and the per-rank restatement (tests/shard_vision_oracle.py) in lm_origin and nan_flags; in the first keyframe also shard_next of the
unsharded slide_vision on one handle holding the merged window.  After the slide, both passes, the next sharded culling and culled
marginalization (the owner's prior) must give the same bits in A and B."""
import copy

import numpy as np
import pytest

from tests import shard_vision_oracle as sv
from tests import slide_vision_oracle as so
from tests.test_post_solve_gpu import STD, make, olib  # noqa: F401  (olib: fixture)
from tests.test_shard_post_solve_gpu import CAM_KEYS, LM_KEYS, PRIOR_KEYS, cam_struct, run_ranks
from tests.test_shard_slide_gpu import PARAMS, STATION0, close, merge, post_solve
from tests.test_slide_integrate_gpu import NOISE5, integ_for, intervals
from tests.test_slide_vision_gpu import CAM, Keyframe, dev, host_twin

pytestmark = pytest.mark.gpu


def group(probs, world, K, iters, R, extra_L=16, extra_F=256):
    """solve_sharded with room in each rank's capacities (extra_L / extra_F: one value, or one per rank) for the next shards"""
    from ic_gvins_b200.ba import WindowSolver, shard_window
    n = len(probs)
    xl = [extra_L] * world if np.isscalar(extra_L) else list(extra_L)
    xf = [extra_F] * world if np.isscalar(extra_F) else list(extra_F)
    shards = [[shard_window(p, r, world) for p in probs] for r in range(world)]
    S = [WindowSolver(max_windows=n, max_K=K, max_L=max(1, max(s["L"] for s in shards[r]) + xl[r]), max_F=max(1, max(s["F"] for s in shards[r]) + xf[r]),
                      max_gnss=16, max_marg_r=R) for r in range(world)]
    blobs = [S[r].shard_export(r, world) for r in range(world)]
    for s in S:
        s.shard_connect(blobs)
    run_ranks(world, lambda r: S[r].gvins_optimization_batch(shards[r], iters))
    merged = [merge([shards[r][w] for r in range(world)], p, blobs=False) for w, p in enumerate(probs)]
    return S, shards, merged


def whole_cull(ci, ranks_out, shards_w):
    """the whole window's culling (inputs and flags) from the ranks' results"""
    from ic_gvins_b200.ba import merge_cull_shard
    L, no = len(ci["lm_ref_node"]), int(ci["obs_off"][-1])
    full = dict(ci, lm_pw=np.zeros((L, 3)), lm_depth=np.zeros(L), lm_outlier=np.zeros(L, np.uint8), obs_outlier=np.zeros(no, np.uint8))
    for g, sh in zip(ranks_out, shards_w):
        merge_cull_shard(full, sh, g)
    return full


def oracle_vis(kf):
    n = kf.new
    return dict(num_marg=1, node_in_map=kf.in_map, node_td=kf.node_td, cur_node=kf.cur, frames=kf.frames,
                obs=[(l, nd, kf.xy[i], kf.vel[i]) for i, (l, nd) in enumerate(kf.obs)],
                new=[dict(depth=n["depth"][j], ref_xy=n["ref_xy"][j], vel_ref=n["vel_ref"][j], ref_id=int(n["ref_id"][j]), cur_xy=n["cur_xy"][j],
                          vel_cur=n["vel_cur"][j]) for j in range(len(n["depth"]))])


def check_shard(res, sh, sc, rb=None):
    """one rank's built shard (shard_slide_vision's result) against shard_next's shard and carry, and the per-rank restatement rb"""
    assert (res["L"], res["F"]) == (sh["L"], sh["F"])
    for k in ("invdepth", "f_lm", "f_ref", "f_obs"):
        assert np.array_equal(res[k], sh[k]), k
    assert np.array_equal(res["lm_src"], sc["lm_src"]) and np.array_equal(res["f_src"], sc["f_src"])
    new = res["f_src"] < 0
    assert np.array_equal(res["f_const"][new], sh["f_const"].reshape(-1, 14)[new])
    if rb is not None:
        assert np.array_equal(res["lm_origin"], rb["lm_origin"]) and res["nan_dropped"] == rb["nan_dropped"]
        assert np.array_equal(res["nan_flags"][:len(rb["nan_flags"])], rb["nan_flags"])


def cycle(probs, world, K, R, iters, seed, n_kf, integrate=False, handoff=False, twin=True, n_new=7):
    """n_kf keyframes of sharded solve -> culling -> culled marginalization -> slide: A on the device, B on the host path.  Returns the
    built results of the last keyframe per rank."""
    from ic_gvins_b200.ba import WindowSolver, shard_next, shard_vision_inputs
    n = len(probs)
    A, sa, ma = group(copy.deepcopy(probs), world, K, iters, R)
    B, sb, mb = group(copy.deepcopy(probs), world, K, iters, R)
    try:
        refs = [so.reference_rows(p) for p in ma]
        for c in range(n_kf + 1):
            ga, pa, cis = post_solve(A, sa, ma, world, seed + 100 * c)
            gb, pb, _ = post_solve(B, sb, ma, world, seed + 100 * c)
            for r in range(world):
                for w in range(n):
                    for k in CAM_KEYS + LM_KEYS:
                        assert np.array_equal(ga[r][w][k], gb[r][w][k], equal_nan=ga[r][w][k].dtype.kind == "f"), (c, r, w, k)
                    if r == w % world:
                        for k in PRIOR_KEYS:
                            assert np.array_equal(pa[r][w][k], pb[r][w][k]), (c, r, w, k)
            if c == n_kf:
                break
            kfs, wholes, vis, parts, igs, prevs = [], [], [], [], [], []
            for w in range(n):
                prev = [sa[r][w] for r in range(world)]
                prevs.append(prev)
                g = whole_cull(cis[w], [ga[r][w] for r in range(world)], prev)
                kf = Keyframe(ma[w], g, pa[w % world][w], refs[w], seed + 100 * c + w, n_new=n_new)
                o = kf.oracle(ma[w], refs[w])
                q, cq = host_twin(kf.nxt, kf.carry, o)
                wb, _, pts = shard_next(q, cq, [sb[r][w] for r in range(world)], sv.new_rank(o, prev, w))
                kfs.append((kf, o, g)), wholes.append(wb), parts.append(pts)
                vis.append(kf.device())
                if integrate:
                    k = kf.nxt["n_imu"] - 1
                    igs.append(integ_for(kf.nxt, kf.carry, {k: ma[w]["K"] - 1}, {k: intervals(ma[w], ma[w]["K"] - 1, 1, seed + 100 * c + w)[0]}))
            if handoff:
                vis = [handoff_vis(kf, v, seed + w) for w, ((kf, _, _), v) in enumerate(zip(kfs, vis))]
            na = [[copy.deepcopy(kf.nxt) for kf, _, _ in kfs] for _ in range(world)]
            ca = [[{k: v for k, v in kf.carry.items() if k not in ("lm_src", "f_src")} for kf, _, _ in kfs] for _ in range(world)]
            va = [[shard_vision_inputs(vis[w], sa[r][w], ga[r][w]) for w in range(n)] for r in range(world)]
            res = run_ranks(world, lambda r: A[r].shard_slide_vision(na[r], ca[r], va[r], igs if integrate else None, NOISE5 if integrate else None))
            for r in range(world):
                for w in range(n):
                    kf, o, _ = kfs[w]
                    sh = sa[r][w]
                    rb = sv.build_rank(dict(sh, lm_ref=refs[w][sh["lm_lo"]:sh["lm_hi"]]), ga[r][w], kf.carry["node_src"],
                                       dict(oracle_vis(kf), obs=sv.shard_obs(oracle_vis(kf)["obs"], sh)), CAM, r, world, w)
                    check_shard(res[r][w], parts[w][r][0], parts[w][r][1], rb)
                    na[r][w].update(lm_lo=parts[w][r][0]["lm_lo"], lm_hi=parts[w][r][0]["lm_hi"], f_index=parts[w][r][0]["f_index"])
            assert sum(res[r][w]["L"] for r in range(world) for w in range(n)) == sum(kf[1]["L"] for kf in kfs)
            if twin and c == 0:  # the unsharded call on the merged window, reordered by shard_next, is what the ranks built
                T = WindowSolver(max_windows=n, max_K=K, max_L=max(max(p["L"] for p in ma), max(kf[1]["L"] for kf in kfs)),
                                 max_F=max(max(p["F"] for p in ma), max(kf[1]["F"] for kf in kfs)), max_gnss=16, max_marg_r=R)
                try:
                    T.upload([copy.deepcopy(p) for p in ma])
                    gt = T.update_and_cull(ma, cam_struct(), STD, cis)
                    T.marginalize(ma, 1, resident=True, culled=gt)
                    rt = T.slide_vision([copy.deepcopy(kf.nxt) for kf, _, _ in kfs], [copy.deepcopy(kf.carry) for kf, _, _ in kfs], vis,
                                        igs if integrate else None, NOISE5 if integrate else None)
                finally:
                    T.close()
                for w, (kf, o, _) in enumerate(kfs):
                    q, cq = host_twin(kf.nxt, kf.carry, rt[w])
                    pts = shard_next(q, cq, [sa[r][w] for r in range(world)], sv.new_rank(rt[w], [sa[r][w] for r in range(world)], w))[2]
                    for r in range(world):
                        check_shard(res[r][w], pts[r][0], pts[r][1])
            nb = [[parts[w][r][0] for w in range(n)] for r in range(world)]
            cb = [[parts[w][r][1] for w in range(n)] for r in range(world)]
            if integrate:
                run_ranks(world, lambda r: B[r].shard_slide_integrate(nb[r], cb[r], igs, NOISE5, STATION0, True))
            else:
                run_ranks(world, lambda r: B[r].shard_slide(nb[r], cb[r], True))
            for grp in (A, B):
                run_ranks(world, lambda r: grp[r].run_gvins(20))
            sum_a = run_ranks(world, lambda r: A[r].gvins_optimization_end(na[r]))
            sum_b = run_ranks(world, lambda r: B[r].gvins_optimization_end(nb[r]))
            assert sum_a == sum_b
            for r in range(world):
                for w in range(n):
                    for k in PARAMS:
                        assert np.array_equal(na[r][w][k], nb[r][w][k]), (c, r, w, k)
                    assert not np.isnan(na[r][w]["invdepth"]).any()
            refs = [o["lm_ref"][sv.rank_order(o, prevs[w], w)] for w, (_, o, _) in enumerate(kfs)]  # the reference rows the slides carried
            sa, sb = na, nb
            ma = [merge([nb[r][w] for r in range(world)], wholes[w], blobs=False) for w in range(n)]
        return res
    finally:
        close(A, B)


def handoff_vis(kf, v, seed):
    """the tracked list behind a src indirection with its count on the device, the new points in a longer buffer with a device count"""
    rng = np.random.default_rng(seed)
    m = len(kf.obs)
    n_in = m + 25
    src = np.sort(rng.choice(n_in, size=m, replace=False)).astype(np.int32)
    lm_in, node_in = np.full(n_in, -1, np.int32), np.full(n_in, 77, np.int32)
    lm_in[src], node_in[src] = [x[0] for x in kf.obs], [x[1] for x in kf.obs]
    cap = m + 40
    xy, vel = np.zeros((cap, 2), np.float32), np.zeros((cap, 2))
    xy[:m], vel[:m] = kf.xy, kf.vel
    nn = len(kf.new["depth"])
    ncap = nn + 9
    pad = lambda a, dt: dev(np.concatenate([np.asarray(a, dt), np.zeros((ncap - nn,) + np.asarray(a).shape[1:], dt)]), dt)  # noqa: E731
    counts = dev([0, m, 0, 0, 0, 0, nn, 0, 0, 0], np.int32)
    return dict(v, n_obs=cap, n_in=n_in, obs_src=dev(src, np.int32), dev_n=counts[1:], obs_lm=dev(lm_in, np.int32), obs_node=dev(node_in, np.int32),
                obs_undis_xy=dev(xy, np.float32), obs_vel=dev(vel, np.float64), n_new=ncap, dev_new_n=counts[6:],
                new_depth=pad(kf.new["depth"], np.float64), new_ref_undis_xy=pad(kf.new["ref_xy"], np.float32),
                new_vel_ref=pad(kf.new["vel_ref"], np.float64), new_ref_frame_id=pad(kf.new["ref_id"], np.int64),
                new_cur_undis_xy=pad(kf.new["cur_xy"], np.float32), new_vel_cur=pad(kf.new["vel_cur"], np.float64))


@pytest.mark.parametrize("world", [2, 3])
def test_cfg3_two_keyframes(olib, world):
    """two keyframes on 2 * world cfg-3 windows: the second slide starts from shards the first one built"""
    probs = [make(olib, outliers=25, seed=3400 + w, K=10, L=300) for w in range(2 * world)]
    cycle(probs, world, 10, 160, 12, 3410 + world, 2)


def test_integrating_slide(olib):
    """with integ: the new keyframe's IMU factor integrated on every rank, against icg_ba_shard_slide_integrate_resident"""
    probs = [make(olib, outliers=25, seed=3500 + w, K=10, L=300) for w in range(3)]
    cycle(probs, 2, 10, 160, 12, 3510, 1, integrate=True)


def test_cfg4_split_pipeline(olib):
    from tests.test_marg_large_gpu import make as make_large
    probs = [make_large(olib, K=20, L=2000, seed=3600 + w, n_ref=20, prior=True) for w in range(2)]
    cycle(probs, 2, 20, 292, 8, 3610, 1)


def test_device_handoff_through_src_and_device_counts(olib):
    """the tracked list behind obs_src with its count on the device, the new points in a longer buffer with a device count"""
    probs = [make(olib, outliers=25, seed=3700 + w, K=10, L=300) for w in range(3)]
    cycle(probs, 2, 10, 160, 12, 3710, 1, handoff=True)


def test_rejections_on_every_rank_leave_the_group_unchanged(olib):
    """over capacity on the rank that receives the new points only, different device counts on the ranks, no current culling on one rank:
    every rank returns ICG_EINVAL, and the good call that follows still matches the host path"""
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200.ba import WindowSolver, shard_next, shard_vision_inputs
    world, n = 2, 2
    probs = [make(olib, outliers=25, seed=3800 + w, K=10, L=300) for w in range(n)]
    grp = dict(extra_L=(0, 400), extra_F=(256, 800))  # rank 0 has no room for more landmarks than its old shard holds
    A, sa, ma = group(copy.deepcopy(probs), world, 10, 12, 160, **grp)
    B, sb, _ = group(copy.deepcopy(probs), world, 10, 12, 160, **grp)
    try:
        def cull_both():
            ga, pa, cis = post_solve(A, sa, ma, world, 3810)
            post_solve(B, sb, ma, world, 3810)
            gs = [whole_cull(cis[w], [ga[r][w] for r in range(world)], [sa[r][w] for r in range(world)]) for w in range(n)]
            return ga, pa, gs

        def keyframes(pa, gs, n_new=7):
            return [Keyframe(ma[w], gs[w], pa[w % world][w], so.reference_rows(ma[w]), 3820 + w, n_new=n_new if w == 0 else 7) for w in range(n)]

        def call(kfs, ga, vis_of):
            na = [[copy.deepcopy(kf.nxt) for kf in kfs] for _ in range(world)]
            ca = [[{k: v for k, v in kf.carry.items() if k not in ("lm_src", "f_src")} for kf in kfs] for _ in range(world)]
            return na, run_ranks(world, lambda r: A[r].shard_slide_vision(na[r], ca[r], vis_of(r)))

        def reject(kfs, ga, vis_of, match):
            def rank(r):
                na = [copy.deepcopy(kf.nxt) for kf in kfs]
                ca = [{k: v for k, v in kf.carry.items() if k not in ("lm_src", "f_src")} for kf in kfs]
                with pytest.raises(IcgError, match=match[r]) as e:
                    A[r].shard_slide_vision(na, ca, vis_of(r))
                assert e.value.code == -1  # ICG_EINVAL
            run_ranks(world, rank)

        ga, pa, gs = cull_both()
        kfs = keyframes(pa, gs)
        dv = [kf.device() for kf in kfs]
        # 1. window 0's 2 * max_L new points: rank 0 (even points) overflows its capacity, rank 1 (odd points) has room
        big = keyframes(pa, gs, n_new=2 * A[0].max_L)
        bv = [kf.device() for kf in big]
        reject(big, ga, lambda r: [shard_vision_inputs(bv[w], sa[r][w], ga[r][w]) for w in range(n)], ["the handle holds", "rank 0 .*rejected"])
        # 2. the ranks read different new-point counts on the device
        nn = len(kfs[1].new["depth"])
        cnt = [dev([nn], np.int32), dev([nn - 1], np.int32)]
        reject(kfs, ga, lambda r: [dict(shard_vision_inputs(dv[w], sa[r][w], ga[r][w]), dev_new_n=cnt[r] if w == 1 else None) for w in range(n)],
               ["camera sides differ", "camera sides differ"])
        # 3. no current culling on rank 1 (an upload since; the twin group takes the same upload)
        A[1].upload(sa[1]), B[1].upload(sb[1])
        reject(kfs, ga, lambda r: [shard_vision_inputs(dv[w], sa[r][w], ga[r][w]) for w in range(n)], ["rank 1 .*rejected", "no culling"])
        # the good call: culling and culled marginalization again on both groups, then A against B's host path
        ga, pa, gs = cull_both()
        kfs = keyframes(pa, gs)
        dv = [kf.device() for kf in kfs]
        na, res = call(kfs, ga, lambda r: [shard_vision_inputs(dv[w], sa[r][w], ga[r][w]) for w in range(n)])
        nb = [[None] * n for _ in range(world)]
        cb = [[None] * n for _ in range(world)]
        for w, kf in enumerate(kfs):
            o = kf.oracle(ma[w], so.reference_rows(ma[w]))
            q, cq = host_twin(kf.nxt, kf.carry, o)
            pts = shard_next(q, cq, [sb[r][w] for r in range(world)], sv.new_rank(o, [sa[r][w] for r in range(world)], w))[2]
            for r in range(world):
                check_shard(res[r][w], pts[r][0], pts[r][1])
                nb[r][w], cb[r][w] = pts[r]
        run_ranks(world, lambda r: B[r].shard_slide(nb[r], cb[r], True))
        for g in (A, B):
            run_ranks(world, lambda r: g[r].run_gvins(20))
        assert run_ranks(world, lambda r: A[r].gvins_optimization_end(na[r])) == run_ranks(world, lambda r: B[r].gvins_optimization_end(nb[r]))
        for r in range(world):
            for w in range(n):
                for k in PARAMS:
                    assert np.array_equal(na[r][w][k], nb[r][w][k]), (r, w, k)
    finally:
        close(A, B)
    # outside a shard group
    one = WindowSolver(max_windows=1, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=160)
    try:
        p = copy.deepcopy(probs[0])
        one.gvins_optimization_batch([p], 8)
        with pytest.raises(IcgError, match="not in a landmark-shard group.*icg_ba_slide_vision_resident") as e:
            one.shard_slide_vision([p], [{}], [dict(num_marg=1, node_in_map=np.ones(10, np.uint8), camera=cam_struct(), node_td=np.zeros(10), cur_node=9)])
        assert e.value.code == -1
    finally:
        one.close()
