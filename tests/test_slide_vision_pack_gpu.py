"""GPU: the structure tables of icg_ba_slide_vision_resident's windows, packed on the device (ba_pack_structure).  After a vision slide every
window's tables (icg_ba_peek_structure) must equal, table by table, those of a twin handle that slid to the same windows with the rows the
vision call returned, packed on the host (icg_ba_slide_resident / icg_ba_slide_integrate_resident).  Also: a window the host packing rejects
is rejected with its message and leaves the handle as it was; the lean binding (rows=False) drives the whole keyframe cycle to the same bits
as the default one."""
import copy

import numpy as np
import pytest

from tests import slide_vision_oracle as so
from tests.test_cull_built_gpu import check_cull, check_priors, ext_of
from tests.test_marg_large_gpu import make as make_large
from tests.test_post_solve_gpu import STD, make
from tests.test_slide_gpu import PARAMS, handle
from tests.test_slide_integrate_gpu import NOISE5, integ_for, intervals
from tests.test_slide_vision_gpu import Keyframe, cam, compare_all, host_twin, olib, solve_cull_marg  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu

TABLES = ("lm_perm", "lm_off", "f_meta_s", "vb_lm0", "ref_nrun", "part_off", "pair_ro", "vis_ord", "npairs", "f_active")


def same_structure(s1, s2, n):
    for w in range(n):
        x, y = s1.peek_structure(w), s2.peek_structure(w)
        for k in TABLES:
            assert np.array_equal(x[k], y[k]), (w, k)


def twin_case(olib, cam, probs, kw, seed, out_of_map=(), n_new=7, integrate=False):
    """one keyframe: handle 1 slides with the vision rows built on the device, handle 2 with the same rows through the host packing.
    Returns the structures of handle 1"""
    p1, p2 = probs, copy.deepcopy(probs)
    s1, s2 = handle(n=len(probs), **kw), handle(n=len(probs), **kw)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch(x, 20)
        refs = [so.reference_rows(p) for p in p1]
        gs, mgs = solve_cull_marg(p1, s1, cam, seed)
        solve_cull_marg(p2, s2, cam, seed)
        kfs = [Keyframe(p, g, mg, rf, seed + w, n_new=n_new, out_of_map=out_of_map) for w, (p, g, mg, rf) in enumerate(zip(p1, gs, mgs, refs))]
        a, ca = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
        if integrate:
            ig = []
            for w, (kf, p) in enumerate(zip(kfs, p1)):
                k = kf.nxt["n_imu"] - 1
                ig.append(integ_for(kf.nxt, kf.carry, {k: p["K"] - 1}, {k: intervals(p, p["K"] - 1, 1, seed + 100 + w)[0]}))
            r = s1.slide_vision(a, ca, [kf.device() for kf in kfs], ig, NOISE5)
        else:
            r = s1.slide_vision(a, ca, [kf.device() for kf in kfs])
        twins = [host_twin(kf.nxt, kf.carry, x) for kf, x in zip(kfs, r)]
        b, cb = [t[0] for t in twins], [t[1] for t in twins]
        if integrate:
            s2.slide_integrate(b, cb, ig, NOISE5)
        else:
            s2.slide(b, cb, True)
        same_structure(s1, s2, len(probs))
        st = [s1.peek_structure(w) for w in range(len(probs))]
        compare_all(s1, s2, a, b)
        return st, r
    finally:
        s1.close(), s2.close()


def test_mixed_batch(olib, cam):
    probs = [make(olib, outliers=25, seed=3101, K=10, L=300), make(olib, outliers=10, seed=3102, K=8, L=150),
             make(olib, outliers=10, seed=3103, K=7, L=120)]
    twin_case(olib, cam, probs, dict(K=10), 3110)


def test_integrating_slide(olib, cam):
    twin_case(olib, cam, [make(olib, outliers=25, seed=3151, K=10, L=300)], dict(K=10), 3160, integrate=True)


def test_cfg4_window_several_runs_per_reference_node(olib, cam):
    """a cfg-4 window (split pipeline): 2000 landmarks over 20 reference nodes, so a reference node's landmarks take several runs"""
    st, _ = twin_case(olib, cam, [make_large(olib, K=20, L=2000, seed=3201, n_ref=20, prior=True)], dict(K=20, L=2000, F=12000, R=292), 3210)
    assert st[0]["ref_nrun"].max() > 1


def test_factorless_landmarks_last(olib, cam):
    """nodes 2, 3 and 5 leave the map: landmarks lose every factor and are placed after the others, in one run of their own"""
    st, r = twin_case(olib, cam, [make(olib, outliers=25, seed=3301, K=10, L=300)], dict(K=10), 3310, out_of_map=(2, 3, 5))
    x = st[0]
    counts = np.diff(x["lm_off"])
    bare = np.nonzero(counts == 0)[0]
    assert len(bare) > 0 and bare[0] == len(counts) - len(bare)
    assert np.array_equal(np.sort(x["lm_perm"][bare]), np.setdiff1d(np.arange(r[0]["L"]), r[0]["f_lm"]))


def test_window_without_factors(olib, cam):
    """every old node out of the map and no new point: no landmark is carried, L = F = 0 next to a full window"""
    probs = [make(olib, outliers=10, seed=3401, K=8, L=150), make(olib, outliers=10, seed=3402, K=8, L=150)]
    p1, p2 = probs, copy.deepcopy(probs)
    s1, s2 = handle(n=2, K=10), handle(n=2, K=10)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch(x, 20)
        refs = [so.reference_rows(p) for p in p1]
        gs, mgs = solve_cull_marg(p1, s1, cam, 3410)
        solve_cull_marg(p2, s2, cam, 3410)
        kfs = [Keyframe(p1[0], gs[0], mgs[0], refs[0], 3411, n_new=0, out_of_map=tuple(range(p1[0]["K"]))),
               Keyframe(p1[1], gs[1], mgs[1], refs[1], 3412)]
        a, ca = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
        r = s1.slide_vision(a, ca, [kf.device() for kf in kfs])
        assert r[0]["L"] == 0 and r[0]["F"] == 0 and r[1]["F"] > 0
        twins = [host_twin(kf.nxt, kf.carry, x) for kf, x in zip(kfs, r)]
        b, cb = [t[0] for t in twins], [t[1] for t in twins]
        s2.slide(b, cb, True)
        same_structure(s1, s2, 2)
        assert s1.peek_structure(0)["npairs"][0] == 0
        compare_all(s1, s2, a, b)
    finally:
        s1.close(), s2.close()


def test_packing_rejection_leaves_the_handle_as_it_was(olib, cam):
    """a new observation of a carried landmark in a node where one of its carried factors already observes it: the build takes it, the
    packing rejects the window with icg_ba_upload's message, before anything is committed.  (The packing's other two checks, a landmark of
    more than 128 factors and a run table overflow, cannot be reached: a landmark has at most one factor per node of max_K <= 32, and the
    run table is sized for the handle's max_L and max_F.)"""
    from ic_gvins_b200 import IcgError
    p1 = make(olib, outliers=25, seed=3501, K=10, L=300)
    p2 = copy.deepcopy(p1)
    s1, s2 = handle(), handle()
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch([x], 20)
        gs, mgs = solve_cull_marg([p1], s1, cam, 3510)
        solve_cull_marg([p2], s2, cam, 3510)
        ref = so.reference_rows(p1)
        kf = Keyframe(p1, gs[0], mgs[0], ref, 3511)
        o = kf.oracle(p1, ref)
        # a carried landmark with a carried factor: a new observation of it in that factor's (next) node
        f = next(f for f in range(o["F"]) if o["f_src"][f] >= 0 and o["lm_origin"][o["f_lm"][f]] >= 0 and not np.isnan(ref[o["lm_origin"][o["f_lm"][f]], 0]))
        lm, node = int(o["lm_origin"][o["f_lm"][f]]), int(o["f_obs"][f])
        bad = kf.device()
        bad["obs_lm"][0], bad["obs_node"][0] = lm, node
        before = s1.peek_structure(0)
        with pytest.raises(IcgError, match="icg_ba_upload: window 0 factor .*: landmark .* has two reference nodes or two observations in node") as e:
            s1.slide_vision([copy.deepcopy(kf.nxt)], [copy.deepcopy(kf.carry)], [bad])
        assert e.value.code == -1  # ICG_EINVAL
        after = s1.peek_structure(0)
        for k in TABLES:
            assert np.array_equal(before[k], after[k]), k
        # the restarted solve and the built culling are those of the twin, which never made the call
        q1, q2 = copy.deepcopy(p1), copy.deepcopy(p2)
        for s in (s1, s2):
            s.run_gvins(20, restart=True)
        assert s1.gvins_optimization_end([q1]) == s2.gvins_optimization_end([q2])
        for k in PARAMS:
            assert np.array_equal(q1[k], q2[k]), k
        # a good call afterwards still matches the twin
        gs1, mgs1 = solve_cull_marg([p1], s1, cam, 3520)
        gs2, _ = solve_cull_marg([p2], s2, cam, 3520)
        check_cull(gs1[0], gs2[0])
        kf = Keyframe(p1, gs1[0], mgs1[0], ref, 3521)
        a, ca = copy.deepcopy(kf.nxt), copy.deepcopy(kf.carry)
        r = s1.slide_vision([a], [ca], [kf.device()])
        b, cb = host_twin(kf.nxt, kf.carry, r[0])
        s2.slide([b], [cb], True)
        same_structure(s1, s2, 1)
        compare_all(s1, s2, [a], [b])
    finally:
        s1.close(), s2.close()


def test_lean_binding_through_the_cycle(olib, cam):
    """three keyframes of vision slide -> run_gvins -> built culling -> culled marginalization, handle 1 with rows=False, handle 2 with the
    default binding: every summary, solution, culling output, prior and structure table bitwise equal"""
    probs = [make(olib, outliers=25, seed=3601, K=10, L=300), make(olib, outliers=25, seed=3602, K=9, L=200)]
    p1, p2 = probs, copy.deepcopy(probs)
    s1, s2 = handle(n=2, K=10), handle(n=2, K=10)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch(x, 20)
        refs = [so.reference_rows(p) for p in p1]
        gs, mgs = solve_cull_marg(p1, s1, cam, 3610)
        solve_cull_marg(p2, s2, cam, 3610)
        for c in range(3):
            # the keyframes are drawn from the default binding's windows, which hold the host rows the lean ones leave on the device
            kfs = [Keyframe(p, g, mg, rf, 3620 + 10 * c + w) for w, (p, g, mg, rf) in enumerate(zip(p2, gs, mgs, refs))]
            os_ = [kf.oracle(p, rf) for kf, p, rf in zip(kfs, p2, refs)]
            a, ca = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
            b, cb = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
            v1, v2 = [kf.device() for kf in kfs], [kf.device() for kf in kfs]
            if c > 0:
                for v in v1 + v2:
                    v.pop("obs_factor")
            r1, r2 = s1.slide_vision(a, ca, v1, rows=False), s2.slide_vision(b, cb, v2)
            for x, y in zip(r1, r2):
                assert "invdepth" not in x and "f_const" not in x
                for k in ("L", "F", "nan_dropped"):
                    assert x[k] == y[k], k
                for k in ("lm_src", "lm_origin", "nan_flags", "f_src", "f_lm", "f_ref", "f_obs"):
                    assert np.array_equal(x[k], y[k]), k
                assert len(x["lm_src"]) == x["L"] and len(x["f_lm"]) == x["F"]
            same_structure(s1, s2, 2)
            for s in (s1, s2):
                s.run_gvins(20)
            assert s1.gvins_optimization_end(a) == s2.gvins_optimization_end(b)
            for x, y in zip(a, b):
                for k in PARAMS:
                    assert np.array_equal(x[k], y[k]), k
            exts = [ext_of(p) for p in a]
            gs, hs = s1.update_and_cull_built(a, cam, STD, exts), s2.update_and_cull_built(b, cam, STD, exts)
            for g, h in zip(gs, hs):
                check_cull(g, h)
            bare = [{k: v for k, v in g.items() if k not in ("lm_ref_node", "obs_off", "obs_node", "obs_factor")} for g in gs]
            mgs = s1.marginalize(a, 1, resident=True, culled=bare)
            check_priors(mgs, s2.marginalize(b, 1, resident=True, culled=[{k: v for k, v in h.items() if k not in ("lm_ref_node", "obs_off", "obs_node", "obs_factor")} for h in hs]))
            p1, p2 = a, b
            refs = [o["lm_ref"] for o in os_]
    finally:
        s1.close(), s2.close()
