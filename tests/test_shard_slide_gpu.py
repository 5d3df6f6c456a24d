"""GPU: the reintegration and the slides of landmark-sharded handles (icg_ba_shard_reintegrate_resident, icg_ba_shard_slide[_integrate]_resident).
The ranks are in-process handles on cuda:0 (run_ranks of test_shard_post_solve_gpu).  Group A slides on the device; group B, the same ranks
after the same calls, takes the host path: icg_imu_preintegrate from the downloaded states, the owner's J0 / e0 handed to every rank and
icg_ba_upload of the next shards.  Every comparison is bitwise.  Carried value rows of every next shard are NaN, so a read of one shows."""
import copy

import numpy as np
import pytest

from datagen.slide_window import build_next
from tests.test_post_solve_gpu import STD, cull_inputs, make, olib  # noqa: F401  (olib: fixture)
from tests.test_reintegration_gpu import NOISE5, window
from tests.test_shard_post_solve_gpu import LM_KEYS, CAM_KEYS, PRIOR_KEYS, cam_struct, run_ranks, solve_sharded
from tests.test_slide_integrate_gpu import host_twin, integ_for, intervals

pytestmark = pytest.mark.gpu

PARAMS = ("pose", "mix", "ext", "invdepth", "f_active", "gnss_std")
STATION0 = np.zeros(3)


def post_solve(solvers, shards, merged, world, seed, nm=1):
    """culling + culled marginalization on every rank; returns (per-rank cull results, per-rank priors, whole-window cull inputs)"""
    from ic_gvins_b200.ba import shard_cull_inputs
    cis = [cull_inputs(p, p["ext"].copy(), seed + w, bad_kp=20) for w, p in enumerate(merged)]
    sci = [[shard_cull_inputs(cis[w], shards[r][w]) for w in range(len(merged))] for r in range(world)]

    def rank(r):
        g = solvers[r].update_and_cull(shards[r], cam_struct(), STD, sci[r])
        return g, solvers[r].marginalize(shards[r], nm, resident=True, culled=g)
    res = run_ranks(world, rank)
    return [x[0] for x in res], [x[1] for x in res], cis


def merge(shards_w, like, blobs=True):
    """the whole window from its shards (lm_lo / lm_hi / f_index into `like`), the solved camera side from rank 0 (and its IMU blobs)"""
    full = copy.deepcopy(like)
    for sh in shards_w:
        full["invdepth"][sh["lm_lo"]:sh["lm_hi"]] = sh["invdepth"]
        full["f_active"][sh["f_index"]] = sh["f_active"]
    for k in ("pose", "mix", "ext", "gnss_std") + (("imu_blob",) if blobs else ()):
        full[k] = np.array(shards_w[0][k], copy=True)
    return full


def close(*groups):
    for g in groups:
        for s in g:
            s.close()


def next_case(p, w, world, seed, prior, integrate, drop_lm=()):
    """build_next of window p (node 0 dropped, one new node, one landmark re-anchored, new landmarks round-robin) and its integration: the
    new interval from the last old node (NODE) with its new node row, the new GNSS fix aligned by that node's velocity"""
    up, stale, carry = build_next(p, seed, prior=prior, drop_lm=drop_lm)
    new = np.nonzero(carry["lm_src"] < 0)[0]
    new_rank = np.full(up["L"], -1)
    new_rank[new] = (np.arange(len(new)) + w) % world
    g = None
    if integrate:
        k = up["n_imu"] - 1
        g = integ_for(up, carry, {k: p["K"] - 1}, {k: intervals(p, p["K"] - 1, 1, seed)[0]}, align=(up["n_gnss"] - 1, p["K"] - 1, -0.03))
    return up, stale, carry, new_rank, g


def slide_twin(olib, probs, world, K, L, R, iters, seed, integrate=True, reint_rows=None, from_marg=None, no_prior=(), rank_of_new=None,
               empty_rank0=()):
    """group A and group B through solve, culling, culled marginalization (and the sharded reintegration), then A's sharded slide against
    B's host path, then both passes, a second culling and culled marginalization; A's result also against an unsharded twin holding the
    merged rank-major window"""
    from ic_gvins_b200.ba import WindowSolver, shard_next
    n = len(probs)
    A, sa, ma = solve_sharded(copy.deepcopy(probs), world, K, iters, R)
    B, sb, mb = solve_sharded(copy.deepcopy(probs), world, K, iters, R)
    try:
        ga, pa, _ = post_solve(A, sa, ma, world, seed)
        gb, pb, _ = post_solve(B, sb, mb, world, seed)
        if reint_rows is not None:
            flags = [w != 1 for w in range(n)]  # window 1 left alone
            ra = run_ranks(world, lambda r: A[r].shard_reintegrate(sa[r], NOISE5, STATION0, reint_rows, flags))
            rb = run_ranks(world, lambda r: B[r].shard_reintegrate(sb[r], NOISE5, STATION0, reint_rows, flags))
            one = WindowSolver(max_windows=n, max_K=K, max_L=L, max_F=max(p["F"] for p in ma), max_gnss=16, max_marg_r=R)
            try:
                one.upload([copy.deepcopy(p) for p in ma])
                ro = one.reintegrate([copy.deepcopy(p) for p in ma], NOISE5, STATION0, reint_rows, flags)
            finally:
                one.close()
            assert sum(o["count"] for o in ro) > 0 and ro[1]["count"] == 0
            for r in range(world):
                for w in range(n):
                    for k in ("status", "blobs", "end_states"):
                        assert np.array_equal(ra[r][w][k], ro[w][k]) and np.array_equal(rb[r][w][k], ro[w][k]), (r, w, k)
        cases, parts_a, parts_b, wholes = [], [], [], []  # wholes: the rank-major next windows with every value filled in
        for w in range(n):
            whole = merge([sa[r][w] for r in range(world)], ma[w])
            prior = None if w in no_prior else pa[w % world][w]
            drop = range(sa[0][w]["lm_lo"], sa[0][w]["lm_hi"]) if w in empty_rank0 else ()  # rank 0 keeps none of its landmarks
            up, stale, carry, new_rank, g = next_case(whole, w, world, seed + 10 * w, prior, integrate, drop)
            if rank_of_new is not None:
                new_rank[carry["lm_src"] < 0] = rank_of_new
            fm = True if from_marg is None else from_marg[w]
            if prior is not None and not fm:
                stale.update(marg_J0=up["marg_J0"].copy(), marg_e0=up["marg_e0"].copy())
            pts = shard_next(stale, carry, [sa[r][w] for r in range(world)], new_rank)[2]
            cases.append((whole, up, carry, new_rank, g, fm and prior is not None))
            parts_a.append(pts)
        flags = [c[5] for c in cases]
        if integrate:
            outs = run_ranks(world, lambda r: A[r].shard_slide_integrate([parts_a[w][r][0] for w in range(n)], [parts_a[w][r][1] for w in range(n)],
                                                                        [c[4] for c in cases], NOISE5, STATION0, flags))
            for r in range(1, world):
                for w in range(n):
                    for k in ("status", "blobs", "end_states"):
                        assert np.array_equal(outs[r][w][k], outs[0][w][k]), (r, w, k)
        else:
            run_ranks(world, lambda r: A[r].shard_slide([parts_a[w][r][0] for w in range(n)], [parts_a[w][r][1] for w in range(n)], flags))
        for w, (whole, up, carry, new_rank, g, _) in enumerate(cases):
            q = host_twin(whole, up, carry, g, outs[0][w], STATION0) if integrate else up
            wb, _, pts = shard_next(q, carry, [sb[r][w] for r in range(world)], new_rank)
            parts_b.append(pts)
            wholes.append(wb)
        next_a = [[parts_a[w][r][0] for w in range(n)] for r in range(world)]
        next_b = [[parts_b[w][r][0] for w in range(n)] for r in range(world)]
        run_ranks(world, lambda r: B[r].upload(next_b[r]))
        for grp in (A, B):
            run_ranks(world, lambda r: grp[r].run_gvins(20))
        sum_a = run_ranks(world, lambda r: A[r].gvins_optimization_end(next_a[r]))
        sum_b = run_ranks(world, lambda r: B[r].gvins_optimization_end(next_b[r]))
        assert sum_a == sum_b
        for r in range(world):
            for w in range(n):
                for k in PARAMS:
                    assert np.array_equal(next_a[r][w][k], next_b[r][w][k]), (r, w, k)
                assert not np.isnan(next_a[r][w]["invdepth"]).any() and not np.isnan(next_a[r][w]["pose"]).any()
        merged = [merge([next_a[r][w] for r in range(world)], wholes[w], blobs=False) for w in range(n)]
        for r in range(world):
            for w in empty_rank0:
                if r == 0:
                    assert next_a[r][w]["L"] == 0 and next_a[r][w]["F"] == 0
        # second culling + culled marginalization: A against B (priors on the owners), and A against an unsharded twin
        ga2, pa2, cis2 = post_solve(A, next_a, merged, world, seed + 500)
        gb2, pb2, _ = post_solve(B, next_b, merged, world, seed + 500)
        twin = WindowSolver(max_windows=n, max_K=K, max_L=max(1, max(p["L"] for p in merged)), max_F=max(1, max(p["F"] for p in merged)),
                            max_gnss=16, max_marg_r=R)
        try:
            twin.upload(merged)
            gt = twin.update_and_cull(merged, cam_struct(), STD, cis2)
            mt = twin.marginalize(merged, 1, resident=True, culled=gt)
        finally:
            twin.close()
        from ic_gvins_b200.ba import merge_cull_shard
        for w in range(n):
            full = {k: np.zeros_like(gt[w][k]) for k in LM_KEYS}
            full["obs_off"] = gt[w]["obs_off"]
            for r in range(world):
                for k in CAM_KEYS:
                    assert np.array_equal(ga2[r][w][k], gt[w][k]) and np.array_equal(gb2[r][w][k], gt[w][k]), (w, r, k)
                merge_cull_shard(full, next_a[r][w], ga2[r][w])
                if r == w % world:
                    for key in PRIOR_KEYS:
                        assert np.array_equal(pa2[r][w][key], mt[w][key]) and np.array_equal(pb2[r][w][key], mt[w][key]), (w, r, key)
            for k in LM_KEYS:
                assert np.array_equal(full[k], gt[w][k], equal_nan=gt[w][k].dtype.kind == "f"), (w, k)
        return cases
    finally:
        close(A, B)


@pytest.mark.parametrize("world", [2, 3])
def test_cfg3_chain(olib, world):
    """solve, culling, culled marginalization, reintegration (gates open in the even windows, window 1 left alone), the integrating slide to
    the next keyframe, both passes; window 0 takes its prior from next (prior_from_marg = 0), window 2 has none"""
    from tests.test_reintegration_gpu import NOISE5 as N5
    n = 2 * world
    made = [window(olib, 600 + w, K=10, L=300, lin=(lambda k: (np.full(3, 9 * N5[2]), np.zeros(3))) if w % 2 == 0 else None) for w in range(n)]
    probs, rows = [m[0] for m in made], [m[1] for m in made]
    slide_twin(olib, probs, world, 10, 300, 160, 12, 610, reint_rows=rows, from_marg=[w != 0 for w in range(n)], no_prior=(2,))


def test_cfg4_split_pipeline_slide(olib):
    from tests.test_marg_large_gpu import make as make_large
    probs = [make_large(olib, K=20, L=2000, seed=2042 + w, n_ref=20, prior=True) for w in range(2)]
    slide_twin(olib, probs, 2, 20, 2000, 292, 8, 640, integrate=False)


def test_every_new_landmark_on_one_rank_and_an_empty_shard(olib):
    """rank 1 takes every new landmark; in window 1 rank 0 keeps none of its landmarks, so its next shard is empty (L = 0)"""
    probs = [make(olib, outliers=10, seed=650 + w, K=8, L=L) for w, L in enumerate((150, 40, 120))]
    slide_twin(olib, probs, 2, 8, 150, 160, 8, 660, rank_of_new=1, empty_rank0=(1,))


def test_merged_interval_and_gnss_insertion(olib):
    """ICG_SLIDE_ROW (a middle node dropped, its two factors merged) in one window, a GNSS insertion with re-created nodes (NODE, CHAIN) in
    the other, on the sharded slide against the host path"""
    from ic_gvins_b200.ba import shard_next
    from tests.test_slide_integrate_gpu import CHAIN, ROW
    world = 2
    probs = [make(olib, seed=670 + w, K=8, L=120) for w in range(2)]
    A, sa, ma = solve_sharded(copy.deepcopy(probs), world, 10, 12, 160)
    B, sb, mb = solve_sharded(copy.deepcopy(probs), world, 10, 12, 160)
    try:
        cases = []
        for w in range(2):
            p = merge([sa[r][w] for r in range(world)], ma[w])
            if w == 0:
                up, stale, carry = build_next(p, 671, drop=(5,), n_new=1, drop_lm=range(0, 120, 6))  # room in the shards' capacity
                r4, r5 = intervals(p, 4, 2, 672)
                state = np.zeros((up["n_imu"], 16))
                state[4] = np.concatenate([p["pose"].reshape(-1, 7)[4], p["mix"].reshape(-1, 9)[4]])
                g = integ_for(up, carry, {4: ROW, 6: 7}, {4: np.concatenate([r4, r5[1:]]), 6: intervals(p, 7, 1, 673)[0]}, state=state)
            else:
                up, stale, carry = build_next(p, 674, drop=(0,), n_new=3, drop_lm=range(0, 120, 6))
                m = up["n_imu"]
                iv = intervals(p, 7, 3, 675)
                g = integ_for(up, carry, {m - 3: 7, m - 2: CHAIN, m - 1: CHAIN}, {m - 3: iv[0], m - 2: iv[1], m - 1: iv[2]})
            nr = np.where(carry["lm_src"] < 0, np.arange(up["L"]) % world, -1)
            cases.append((p, up, stale, carry, g, nr))
        pa = [shard_next(c[2], c[3], [sa[r][w] for r in range(world)], c[5])[2] for w, c in enumerate(cases)]
        outs = run_ranks(world, lambda r: A[r].shard_slide_integrate([pa[w][r][0] for w in range(2)], [pa[w][r][1] for w in range(2)],
                                                                    [c[4] for c in cases], NOISE5, STATION0, False))
        pb = [shard_next(host_twin(c[0], c[1], c[3], c[4], outs[0][w], STATION0), c[3], [sb[r][w] for r in range(world)], c[5])[2]
              for w, c in enumerate(cases)]
        na = [[pa[w][r][0] for w in range(2)] for r in range(world)]
        nb = [[pb[w][r][0] for w in range(2)] for r in range(world)]
        run_ranks(world, lambda r: B[r].upload(nb[r]))
        for grp, nx in ((A, na), (B, nb)):
            run_ranks(world, lambda r: grp[r].run_gvins(20, restart=False))
        sa2 = run_ranks(world, lambda r: A[r].gvins_optimization_end(na[r]))
        sb2 = run_ranks(world, lambda r: B[r].gvins_optimization_end(nb[r]))
        assert sa2 == sb2
        for r in range(world):
            for w in range(2):
                for k in PARAMS:
                    assert np.array_equal(na[r][w][k], nb[r][w][k]), (r, w, k)
    finally:
        close(A, B)


def test_rejections_on_every_rank_leave_the_group_unchanged(olib):
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200.ba import WindowSolver, shard_next
    world, n = 2, 2
    probs = [make(olib, outliers=10, seed=680 + w, K=8, L=120) for w in range(n)]
    S, sh, mg = solve_sharded(copy.deepcopy(probs), world, 10, 12, 160)

    def state():
        def rank(r):
            S[r].run_gvins(12, restart=True)
            q = copy.deepcopy(sh[r])
            return S[r].gvins_optimization_end(q), [[x[k].copy() for k in PARAMS] for x in q]
        return run_ranks(world, rank)

    def same(a, b):
        for x, y in zip(a, b):
            assert x[0] == y[0]
            for u, v in zip(x[1], y[1]):
                assert all(np.array_equal(s, t) for s, t in zip(u, v))

    try:
        base = state()
        priors = [None] * n
        cases = []
        for w in range(n):
            p = merge([sh[r][w] for r in range(world)], mg[w])
            up, stale, carry, nr, g = next_case(p, w, world, 690 + w, None, True)
            cases.append((up, stale, carry, nr, g))

        def parts():
            return [shard_next(c[1], c[2], [sh[r][w] for r in range(world)], c[3])[2] for w, c in enumerate(cases)]

        def reject(mutate, match, flags=False, integ=None, g_all=None):
            pts = parts()
            per = [[copy.deepcopy(pts[w][r]) for w in range(n)] for r in range(world)]
            mutate(per)

            def rank(r):
                with pytest.raises(IcgError, match=match[r] if isinstance(match, (list, tuple)) else match):
                    if g_all is not None:
                        S[r].shard_slide_integrate([x[0] for x in per[r]], [x[1] for x in per[r]], g_all, NOISE5, STATION0, flags)
                    else:
                        S[r].shard_slide([x[0] for x in per[r]], [x[1] for x in per[r]], flags)
            run_ranks(world, rank)
            same(base, state())

        # prior_from_marg = 1 with no sharded resident marginalization since the upload
        reject(lambda per: None, "no sharded resident marginalization", flags=True)
        # one rank's lm_src out of range: that rank names its error, the other names the rejecting rank
        def bad_lm(per):
            per[1][0][1]["lm_src"] = per[1][0][1]["lm_src"].copy()
            per[1][0][1]["lm_src"][0] = 10 ** 6
        reject(bad_lm, ["rank 1 .*rejected", "lm_src.*out of range"])
        # node_src differ between the ranks
        def bad_node(per):
            per[1][1][1]["node_src"] = per[1][1][1]["node_src"].copy()
            per[1][1][1]["node_src"][1] = per[1][1][1]["node_src"][2]
        reject(bad_node, "camera sides differ")
        # an integrated covariance that is not positive definite (every rank integrates the same flat rows)
        gs = copy.deepcopy([c[4] for c in cases])
        k = cases[0][0]["n_imu"] - 1
        gs[0]["imu_rows"][k] = gs[0]["imu_rows"][k].copy()
        gs[0]["imu_rows"][k][:, 0] = 0.0
        reject(lambda per: None, "not positive definite", g_all=gs)
        # marg_r not the owner's r, after a sharded marginalization
        _, pr, _ = post_solve(S, sh, mg, world, 695)
        for w in range(n):
            priors[w] = pr[w % world][w]
            assert priors[w]["r"] > 0

        def wrong_r(per):
            # a self-consistent prior that is not the owner's: its last block (td, one column) left out.  Only the owner's record of its
            # marginalization catches it; rank 1 learns of it through the agreement
            pr0 = priors[0]
            assert pr0["block_type"][-1] == 3
            rr = pr0["r"] - 1
            for r in range(world):
                per[r][0][0].update(marg_r=rr, marg_nblocks=len(pr0["block_type"]) - 1, marg_block_type=pr0["block_type"][:-1].copy(),
                                    marg_block_node=pr0["block_node"][:-1].copy(), marg_x0=pr0["x0"][:-1].copy(), marg_J0=np.zeros(rr * rr),
                                    marg_e0=np.zeros(rr))
        reject(wrong_r, ["marg_r=", "rank 0 .*rejected"], flags=[True, False])
    finally:
        close(S)
    # each new call on an unsharded handle
    one = WindowSolver(max_windows=1, max_K=10, max_L=300, max_F=2700, max_gnss=16, max_marg_r=160)
    try:
        p = copy.deepcopy(probs[0])
        one.gvins_optimization_batch([p], 8)
        with pytest.raises(IcgError, match="not in a landmark-shard group.*icg_ba_reintegrate_resident"):
            one.shard_reintegrate([p], NOISE5, STATION0, [None], reintegrate=[0])
        with pytest.raises(IcgError, match="not in a landmark-shard group.*icg_ba_slide_resident"):
            one.shard_slide([p], [{}], False)
        with pytest.raises(IcgError, match="not in a landmark-shard group.*icg_ba_slide_integrate_resident"):
            one.shard_slide_integrate([p], [{}], [None], NOISE5)
    finally:
        one.close()


# ------------------------------------------------------------------------------------------------------- one process per rank
class ThreadGather:
    """all_gather_object among the threads of run_ranks (the in-process stand-in of torch.distributed's)"""

    def __init__(self, world):
        import threading
        self.bar, self.slots = threading.Barrier(world, timeout=300), [None] * world

    def __call__(self, rank, obj):
        self.bar.wait()  # the previous round's readers are done
        self.slots[rank] = obj
        self.bar.wait()
        return list(self.slots)


def chain_rank(olib, rank, world, gather, device=0, seed=2600):
    """rank `rank`'s part of the cfg-3 chain, written against an all-gather only, so that it runs the same as in-process threads and as one
    process per GPU: groups A and B (same capacities) through the sharded solve, culling, culled marginalization and reintegration; A takes
    the integrating slide, B the host path (host preintegration, the owner's prior on every rank, icg_ba_upload); both passes; a second
    culling and culled marginalization.  A against B bitwise on every rank; the reintegration and the second culling and marginalization
    also against an unsharded twin on rank 0."""
    from ic_gvins_b200.ba import WindowSolver, merge_cull_shard, shard_cull_inputs, shard_next, shard_window
    n = 2 * world
    lin = lambda k: (np.full(3, 9 * NOISE5[2]), np.zeros(3))  # noqa: E731  (gates open)
    made = [window(olib, seed + w, K=10, L=300, lin=lin if w % 2 == 0 else None) for w in range(n)]
    probs, rows = [m[0] for m in made], [m[1] for m in made]
    shards_all = [[shard_window(p, r, world) for p in probs] for r in range(world)]
    cam = cam_struct()

    def group():
        mine = [copy.deepcopy(s) for s in shards_all[rank]]
        s = WindowSolver(max_windows=n, max_K=10, max_L=max(1, max(x["L"] for x in mine)) + 16, max_F=max(1, max(x["F"] for x in mine)) + 256,
                         max_gnss=16, max_marg_r=160, device=device)
        s.shard_connect(gather(rank, s.shard_export(rank, world)))
        gather(rank, None)  # every rank connected
        return s, mine

    def whole_windows(shards, likes):
        parts = gather(rank, [(x["lm_lo"], x["lm_hi"], x["invdepth"], x["f_index"], x["f_active"]) for x in shards])
        out = []
        for w, like in enumerate(likes):
            full = copy.deepcopy(like)
            for lo, hi, rho, fi, act in (parts[r][w] for r in range(world)):
                full["invdepth"][lo:hi], full["f_active"][fi] = rho, act
            for k in ("pose", "mix", "ext", "gnss_std", "imu_blob"):
                full[k] = np.array(shards[w][k], copy=True)
            out.append(full)
        return out

    def cull_marg(s, shards, wholes, cis):
        g = s.update_and_cull(shards, cam, STD, [shard_cull_inputs(ci, x) for ci, x in zip(cis, shards)])
        return g, s.marginalize(shards, 1, resident=True, culled=g)

    def sync():  # one group's work is done on every rank before the other group's starts (in-process ranks share one GPU)
        gather(rank, None)

    (A, sa), (B, sb) = group(), group()
    try:
        A.gvins_optimization_batch(sa, 12)
        sync()
        B.gvins_optimization_batch(sb, 12)
        for x, y in zip(sa, sb):
            assert all(np.array_equal(x[k], y[k]) for k in PARAMS)
        merged = whole_windows(sa, probs)
        cis = [cull_inputs(p, p["ext"].copy(), seed + 50 + w, bad_kp=20) for w, p in enumerate(merged)]
        ga, pa = cull_marg(A, sa, merged, cis)
        sync()
        gb, pb = cull_marg(B, sb, merged, cis)
        allp = gather(rank, pa)
        prior = [allp[w % world][w] for w in range(n)]
        flags = [w != 1 for w in range(n)]  # window 1 left alone
        ra = A.shard_reintegrate(sa, NOISE5, STATION0, rows, flags)
        sync()
        rb = B.shard_reintegrate(sb, NOISE5, STATION0, rows, flags)
        for x, y in zip(ra, rb):
            assert all(np.array_equal(x[k], y[k]) for k in ("status", "blobs", "end_states"))
        all_ra = gather(rank, ra)
        if rank == 0:
            one = WindowSolver(max_windows=n, max_K=10, max_L=300, max_F=max(p["F"] for p in merged), max_gnss=16, max_marg_r=160, device=device)
            try:
                one.upload([copy.deepcopy(p) for p in merged])
                ro = one.reintegrate([copy.deepcopy(p) for p in merged], NOISE5, STATION0, rows, flags)
            finally:
                one.close()
            assert sum(o["count"] for o in ro) > 0 and ro[1]["count"] == 0
            for r in range(world):
                for w in range(n):
                    assert all(np.array_equal(all_ra[r][w][k], ro[w][k]) for k in ("status", "blobs", "end_states")), (r, w)
        wholes = whole_windows(sa, merged)  # the reintegrated blobs
        cases, na, ca = [], [], []
        for w in range(n):
            up, stale, carry, new_rank, g = next_case(wholes[w], w, world, seed + 100 + 10 * w, None if w == 2 else prior[w], True)
            fm = w not in (0, 2)  # window 0 takes its prior from next (prior_from_marg = 0), window 2 has none
            if w == 0:
                stale.update(marg_J0=up["marg_J0"].copy(), marg_e0=up["marg_e0"].copy())
            part = shard_next(stale, carry, [shards_all[r][w] for r in range(world)], new_rank)[2][rank]
            na.append(part[0]), ca.append(part[1])
            cases.append((up, carry, new_rank, g, fm))
        outs = A.shard_slide_integrate(na, ca, [c[3] for c in cases], NOISE5, STATION0, [c[4] for c in cases])
        all_outs = gather(rank, outs)
        for r in range(world):
            for w in range(n):
                assert all(np.array_equal(all_outs[r][w][k], outs[w][k]) for k in ("status", "blobs", "end_states")), (r, w)
        nb, likes = [], []
        for w, (up, carry, new_rank, g, _) in enumerate(cases):
            q = host_twin(wholes[w], up, carry, g, outs[w], STATION0)
            wb, _, parts = shard_next(q, carry, [shards_all[r][w] for r in range(world)], new_rank)
            nb.append(parts[rank][0]), likes.append(wb)
        B.upload(nb)
        A.run_gvins(20)
        sum_a = A.gvins_optimization_end(na)
        sync()
        B.run_gvins(20)
        sum_b = B.gvins_optimization_end(nb)
        assert sum_a == sum_b
        for w in range(n):
            assert all(np.array_equal(na[w][k], nb[w][k]) for k in PARAMS), w
            assert not np.isnan(na[w]["invdepth"]).any() and not np.isnan(na[w]["pose"]).any()
        merged2 = whole_windows(na, likes)
        for w in range(n):  # the camera side with every value (A's carried rows were NaN on the host)
            for k in ("imu_blob", "gnss_blh", "marg_J0", "marg_e0"):
                merged2[w][k] = likes[w][k]
        cis2 = [cull_inputs(p, p["ext"].copy(), seed + 500 + w, bad_kp=20) for w, p in enumerate(merged2)]
        g2a, p2a = cull_marg(A, na, merged2, cis2)
        sync()
        g2b, p2b = cull_marg(B, nb, merged2, cis2)
        for w in range(n):
            assert all(np.array_equal(g2a[w][k], g2b[w][k], equal_nan=g2a[w][k].dtype.kind == "f") for k in CAM_KEYS + LM_KEYS), w
            assert all(np.array_equal(p2a[w][k], p2b[w][k]) for k in PRIOR_KEYS), w
        all2 = gather(rank, (g2a, p2a, [(x["lm_lo"], x["lm_hi"], x["f_index"]) for x in na]))
        if rank == 0:  # the merged rank-major windows on an unsharded twin
            twin = WindowSolver(max_windows=n, max_K=10, max_L=max(p["L"] for p in merged2), max_F=max(p["F"] for p in merged2), max_gnss=16,
                                max_marg_r=160, device=device)
            try:
                twin.upload(merged2)
                gt = twin.update_and_cull(merged2, cam, STD, cis2)
                mt = twin.marginalize(merged2, 1, resident=True, culled=gt)
            finally:
                twin.close()
            for w in range(n):
                full = {k: np.zeros_like(gt[w][k]) for k in LM_KEYS}
                full["obs_off"] = gt[w]["obs_off"]
                for r in range(world):
                    g, pr, lims = all2[r][0][w], all2[r][1][w], all2[r][2][w]
                    assert all(np.array_equal(g[k], gt[w][k]) for k in CAM_KEYS), (w, r)
                    merge_cull_shard(full, dict(lm_lo=lims[0], lm_hi=lims[1], f_index=lims[2]), g)
                    if r == w % world:
                        assert all(np.array_equal(pr[k], mt[w][k]) for k in PRIOR_KEYS), (w, r)
                assert all(np.array_equal(full[k], gt[w][k], equal_nan=gt[w][k].dtype.kind == "f") for k in LM_KEYS), w
        gather(rank, None)
        return "ok"
    finally:
        A.close(), B.close()


def test_chain_rank_code_on_in_process_ranks(olib):
    """the per-rank chain of the spawn test below, on two in-process ranks of cuda:0"""
    gather = ThreadGather(2)
    assert run_ranks(2, lambda r: chain_rank(olib, r, 2, gather)) == ["ok", "ok"]


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _worker(rank, world, port, q):
    try:
        import ctypes as C
        import os
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import oracle
        from tests import oracle_api as oa
        olib_ = C.CDLL(oracle.build())
        oa.declare(olib_)
        oa.declare_ba(olib_)

        def gather(r, obj):
            out = [None] * world
            dist.all_gather_object(out, obj)
            return out
        res = chain_rank(olib_, rank, world, gather, device=rank)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, res))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + repr(e) + "\n" + traceback.format_exc()))


@pytest.mark.skipif(_ngpu() < 2, reason="needs two or more GPUs")
def test_multi_gpu_chain():
    """the cfg-3 chain with one process per GPU: the exchange buffers over CUDA IPC, each owner's gather handle in its own process"""
    import socket
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
        res = dict(q.get(timeout=900) for _ in range(world))
    finally:
        for p in ps:
            p.join(60)
            if p.is_alive():
                p.kill()
    assert all(v == "ok" for v in res.values()), res
