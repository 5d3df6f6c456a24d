"""GPU: icg_ba_update_and_cull_built.  A handle slides with icg_ba_slide_vision_resident, which also writes the next culling's observation
lists on the device, then culls on those lists; a twin handle makes the same calls but culls on host lists that the numpy list rule
(tests/cull_lists_oracle.py) builds from the previous lists.  The built lists must equal the rule's exactly, and the two handles must give the
same bits: culling outputs, the marginalization's prior, the next slide and the solves after it."""
import copy
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import slide_vision_oracle as so
from tests.cull_lists_oracle import next_lists
from tests.test_marg_large_gpu import make as make_large
from tests.test_post_solve_gpu import STD, cull_inputs, make
from tests.test_slide_gpu import handle
from tests.test_slide_vision_gpu import Keyframe, cam, check_built, compare_all, olib, solve_cull_marg  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LISTS = ("lm_ref_node", "lm_ref_kp", "obs_off", "obs_node", "obs_kp", "obs_factor")


def ext_of(p):
    c = cull_inputs(dict(p, L=0, F=0), p["ext"].copy(), 0)
    return {k: c[k] for k in ("R_bc", "t_bc", "td_bc", "estimate_ext", "estimate_td")}


def restate(kf, g, o):
    """the rule's next lists from the culling `g` (its lists and flags), the slide's restated window `o` and the keyframe's observations"""
    K_old = kf.K_old
    onode = np.full(K_old, -1)
    for j, i in enumerate(kf.carry["node_src"]):
        if 1 <= i < K_old and kf.in_map[i]:
            onode[i] = j
    new_obs_xy = {(l, nd): kf.xy[i] for i, (l, nd) in enumerate(kf.obs) if l >= 0}
    pts = [dict(ref_node=kf.frames[int(kf.new["ref_id"][j])], ref_xy=kf.new["ref_xy"][j], cur_xy=kf.new["cur_xy"][j]) for j in range(len(kf.new["depth"]))]
    return next_lists(g, g["obs_outlier"], onode, o, new_obs_xy, pts, kf.cur)


def check_lists(got, want, L, F):
    assert got["n_obs"] == want["n_obs"] == L + F
    for k in LISTS:
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k


def check_cull(x, y):
    for k in ("R_bc_out", "t_bc_out", "cam_pose", "lm_pw", "lm_depth", "lm_outlier", "obs_outlier", "counts"):
        assert np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes(), k
    assert x["td_bc_out"] == y["td_bc_out"] and x["ext_accepted"] == y["ext_accepted"]


def check_priors(m1, m2):
    for x, y in zip(m1, m2):
        assert x["m"] == y["m"] and x["r"] == y["r"]
        for k in ("J0", "e0", "Hp", "bp"):
            assert np.array_equal(x[k], y[k]), k


def chain(olib, cam, probs, kw, seed, n_cycles):
    """n_cycles keyframes; from the second one on, handle 1 culls on its built lists and passes NULL lists to the culled marginalization and
    the next vision slide, handle 2 culls on the restated host lists"""
    p1, p2 = probs, copy.deepcopy(probs)
    s1, s2 = handle(n=len(probs), **kw), handle(n=len(probs), **kw)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch(x, 20)
        refs = [so.reference_rows(p) for p in p1]
        full, want = None, None
        for c in range(n_cycles):
            if c == 0:
                gs, mgs = solve_cull_marg(p1, s1, cam, seed, full)
                solve_cull_marg(p2, s2, cam, seed, full)
            else:
                exts = [ext_of(p) for p in p1]
                gs = s1.update_and_cull_built(p1, cam, STD, exts)
                hs = s2.update_and_cull(p2, cam, STD, [dict(e, **{k: w[k] for k in LISTS}) for e, w in zip(exts, want)])
                for g, h, w, p in zip(gs, hs, want, p1):
                    check_lists(g, w, p["L"], p["F"])
                    check_cull(g, h)
                bare = [{k: v for k, v in g.items() if k not in ("lm_ref_node", "obs_off", "obs_node", "obs_factor")} for g in gs]
                mgs = s1.marginalize(p1, 1, resident=True, culled=bare)
                check_priors(mgs, s2.marginalize(p2, 1, resident=True, culled=hs))
            kfs = [Keyframe(p, g, mg, rf, seed + 10 * c + w) for w, (p, g, mg, rf) in enumerate(zip(p1, gs, mgs, refs))]
            os_ = [kf.oracle(p, rf) for kf, p, rf in zip(kfs, p1, refs)]
            a, ca = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
            b, cb = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
            v1 = [kf.device() for kf in kfs]
            if c > 0:
                for v in v1:
                    v.pop("obs_factor")
            r1, r2 = s1.slide_vision(a, ca, v1), s2.slide_vision(b, cb, [kf.device() for kf in kfs])
            for x, y, o in zip(r1, r2, os_):
                check_built(x, o), check_built(y, o)
            want = [restate(kf, g, o) for kf, g, o in zip(kfs, gs, os_)]
            compare_all(s1, s2, a, b)
            p1, p2 = a, b
            refs = [o["lm_ref"] for o in os_]
            full = [x["f_const"].copy() for x in b]
        return s1, s2, p1, p2, want
    except BaseException:
        s1.close(), s2.close()
        raise


def finish(s1, s2, p1, p2, want, cam):
    """a last built culling against the twin's host-list culling"""
    try:
        exts = [ext_of(p) for p in p1]
        gs = s1.update_and_cull_built(p1, cam, STD, exts)
        hs = s2.update_and_cull(p2, cam, STD, [dict(e, **{k: w[k] for k in LISTS}) for e, w in zip(exts, want)])
        for g, h, w, p in zip(gs, hs, want, p1):
            check_lists(g, w, p["L"], p["F"])
            check_cull(g, h)
    finally:
        s1.close(), s2.close()


def test_mixed_batch_built_lists_and_twin(olib, cam):
    probs = [make(olib, outliers=25, seed=2101, K=10, L=300), make(olib, outliers=10, seed=2102, K=8, L=150),
             make(olib, outliers=10, seed=2103, K=7, L=120)]
    finish(*chain(olib, cam, probs, dict(K=10), 2110, 1), cam)


def test_cfg4_window(olib, cam):
    finish(*chain(olib, cam, [make_large(olib, K=20, L=2000, seed=2201, n_ref=20, prior=True)], dict(K=20, L=2000, F=12000, R=292), 2210, 1), cam)


def test_three_keyframe_chain_with_null_lists(olib, cam):
    """solve -> built culling -> culled marginalization with NULL lists -> vision slide with NULL obs_factor, three times, against the twin"""
    probs = [make(olib, outliers=25, seed=2301, K=10, L=300), make(olib, outliers=25, seed=2302, K=9, L=200)]
    finish(*chain(olib, cam, probs, dict(K=10), 2310, 3), cam)


def test_contract(olib, cam):
    from ic_gvins_b200 import IcgError
    from tests.test_slide_vision_gpu import host_twin
    p1 = make(olib, outliers=25, seed=2401, K=10, L=300)
    p0, p2 = copy.deepcopy(p1), copy.deepcopy(p1)
    s1, s2 = handle(n=2), handle(n=2)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch([x], 20)
        with pytest.raises(IcgError, match="no built lists") as e:  # before any vision slide
            s1.update_and_cull_built([p1], cam, STD, [ext_of(p1)])
        assert e.value.code == -1  # ICG_EINVAL
        gs, mgs = solve_cull_marg([p1], s1, cam, 2410, None)
        solve_cull_marg([p2], s2, cam, 2410, None)
        ref = so.reference_rows(p1)
        kf = Keyframe(p1, gs[0], mgs[0], ref, 2411)
        o = kf.oracle(p1, ref)
        want = restate(kf, gs[0], o)
        a, ca = copy.deepcopy(kf.nxt), copy.deepcopy(kf.carry)
        s1.slide_vision([a], [ca], [kf.device()])
        b, cb = host_twin(kf.nxt, kf.carry, o)
        s2.slide([b], [cb], True)
        s1.run_gvins(20), s2.run_gvins(20)
        s1.gvins_optimization_end([a]), s2.gvins_optimization_end([b])
        # another window count: the built lists are only ever current for the uploaded count, so the window-count check of every resident
        # call rejects it before the lists are looked at
        with pytest.raises(IcgError, match="holds 1 uploaded windows") as e:
            s1.update_and_cull_built([a, a], cam, STD, [ext_of(a)] * 2)
        assert e.value.code == -1
        ext = ext_of(a)
        g = s1.update_and_cull_built([a], cam, STD, [ext])[0]
        h = s2.update_and_cull([b], cam, STD, [dict(ext, **{k: want[k] for k in LISTS})])[0]
        check_lists(g, want, a["L"], a["F"])
        check_cull(g, h)
        # a vision slide rejected after its kernel wrote the other list buffer keeps these lists current
        bare = {k: v for k, v in g.items() if k not in ("lm_ref_node", "obs_off", "obs_node", "obs_factor")}
        mg = s1.marginalize([a], 1, resident=True, culled=[bare])
        check_priors(mg, s2.marginalize([b], 1, resident=True, culled=[h]))
        big = Keyframe(a, g, mg[0], o["lm_ref"], 2412, n_new=400)
        v = big.device()
        v.pop("obs_factor")
        with pytest.raises(IcgError, match="the handle holds"):
            s1.slide_vision([copy.deepcopy(big.nxt)], [copy.deepcopy(big.carry)], [v])
        g2 = s1.update_and_cull_built([a], cam, STD, [ext])[0]
        check_lists(g2, want, a["L"], a["F"])
        check_cull(g2, h)
        s1.upload([p0])  # an upload ends them
        with pytest.raises(IcgError, match="no built lists"):
            s1.update_and_cull_built([p0], cam, STD, [ext_of(p0)])
    finally:
        s1.close(), s2.close()


def test_other_slides_end_the_built_lists(olib, cam):
    """a built culling after icg_ba_slide_resident or icg_ba_slide_integrate_resident is ICG_EINVAL; on a landmark-sharded handle
    ICG_EUNSUPPORTED"""
    from ic_gvins_b200 import IcgError
    from tests.test_slide_integrate_gpu import NOISE5
    p = make(olib, outliers=25, seed=2501, K=10, L=300)
    s = handle()
    try:
        s.gvins_optimization_batch([p], 20)
        ref = so.reference_rows(p)
        for i, other in enumerate((lambda q, c: s.slide([q], [c], False), lambda q, c: s.slide_integrate([q], [c], [{}], NOISE5, prior_from_marg=False))):
            gs, mgs = solve_cull_marg([p], s, cam, 2510 + 10 * i, None)
            kf = Keyframe(p, gs[0], mgs[0], ref, 2511 + 10 * i)
            o = kf.oracle(p, ref)
            a = copy.deepcopy(kf.nxt)
            s.slide_vision([a], [copy.deepcopy(kf.carry)], [kf.device()])
            s.run_gvins(20)
            s.gvins_optimization_end([a])
            same = dict(node_src=np.arange(a["K"], dtype=np.int32), lm_src=np.arange(a["L"], dtype=np.int32), f_src=np.arange(a["F"], dtype=np.int32),
                        imu_src=np.arange(a["n_imu"], dtype=np.int32), gnss_src=np.arange(a["n_gnss"], dtype=np.int32))
            other(copy.deepcopy(a), same)  # the window onto itself, every row carried
            with pytest.raises(IcgError, match="no built lists"):
                s.update_and_cull_built([a], cam, STD, [ext_of(a)])
            s.run_gvins(20)
            s.gvins_optimization_end([a])
            p, ref = a, o["lm_ref"]
        s.shard_export(0, 2)
        with pytest.raises(IcgError, match="landmark-sharded") as e:
            s.update_and_cull_built([p], cam, STD, [ext_of(p)])
        assert e.value.code == -4  # ICG_EUNSUPPORTED
        s.shard_leave()
    finally:
        s.close()


SHIM = r'''
#include <cstdio>
#include <vector>
#include "ic_gvins_b200/host/icg_shims.hpp"
// links and runs WindowSolver::updateAndCullBuilt: on a handle without built lists it must throw, naming the call
int main() {
    icg_b200::WindowSolver s(10, 300, 2700);
    icg_ba_problem p{};
    icg_camera cam{};
    icg_ba_cull_window io{};
    icg_ba_cull_lists lists{};
    try {
        s.updateAndCullBuilt(p, cam, 1.0, io, &lists);
    } catch (const std::exception &e) {
        printf("%s\n", e.what());
        return 0;
    }
    return 1;
}
'''


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_shim_update_and_cull_built_runs():
    """the C++ member compiles, links against the library and reaches the call (which rejects a handle holding no windows)"""
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
        assert "icg_ba_update_and_cull_built" in r.stdout
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def test_lists_longer_than_the_handle_are_refused(olib, cam):
    """host lists that name every entry twice (not shaped as the reference builds them, but accepted by the culling and the slide) grow
    built lists longer than max_L + max_F: the built culling refuses them before writing any caller array; the slide itself is unchanged"""
    from ic_gvins_b200 import IcgError
    p = make(olib, outliers=25, seed=2701, K=10, L=300)
    s = handle(F=p["F"] + 100)
    try:
        s.gvins_optimization_batch([p], 20)
        ci = cull_inputs(p, p["ext"].copy(), 2710)
        off = ci["obs_off"]
        idx = np.concatenate([np.r_[np.arange(off[l], off[l + 1]), np.arange(off[l], off[l + 1])] for l in range(p["L"])]).astype(np.int64)
        dup = dict(ci, obs_off=(2 * off).astype(np.int32), obs_node=ci["obs_node"][idx], obs_kp=ci["obs_kp"][idx], obs_factor=ci["obs_factor"][idx])
        g = s.update_and_cull([p], cam, STD, [dup])[0]
        mg = s.marginalize([p], 1, resident=True, culled=[g])
        kf = Keyframe(p, g, mg[0], so.reference_rows(p), 2711)
        o = kf.oracle(p, so.reference_rows(p))
        want = restate(kf, g, o)
        assert want["n_obs"] > s.max_L + s.max_F
        a = copy.deepcopy(kf.nxt)
        check_built(s.slide_vision([a], [copy.deepcopy(kf.carry)], [kf.device()])[0], o)
        s.run_gvins(20)
        s.gvins_optimization_end([a])
        with pytest.raises(IcgError, match="more than max_L \\+ max_F") as e:
            s.update_and_cull_built([a], cam, STD, [ext_of(a)])
        assert e.value.code == -1
    finally:
        s.close()


def test_slide_ins_vision_form_makes_the_lists_current_and_its_plain_form_ends_them(olib, cam):
    """icg_ba_slide_ins_resident with vis builds the lists like icg_ba_slide_vision_resident (against the twin's host-list culling of the
    restated lists); without vis it ends them like every other slide"""
    from datagen import synth_ba
    from datagen.slide_window import build_next
    from ic_gvins_b200 import IcgError
    from tests import ins_series_oracle as iso
    if not iso.HAVE_CXX:
        pytest.skip("no host C++ compiler for the INS restatement")
    from tests.test_slide_gpu import PARAMS
    from tests.test_slide_ins_gpu import ins_pair, node_times
    from tests.test_slide_integrate_gpu import integ_for
    from tests.test_slide_vision_gpu import host_twin
    p1 = make(olib, outliers=10, seed=2801, K=8, L=120)
    p2 = copy.deepcopy(p1)
    s1, s2 = handle(), handle()
    d, o = ins_pair(1)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch([x], 20)
        t = node_times(8)
        s1.imu_samples_from_ins(d, [0], [t])
        gs, mgs = solve_cull_marg([p1], s1, cam, 2810, None)
        solve_cull_marg([p2], s2, cam, 2810, None)
        ref = so.reference_rows(p1)
        kf = Keyframe(p1, gs[0], mgs[0], ref, 2811)
        ov = kf.oracle(p1, ref)
        want = restate(kf, gs[0], ov)
        a = copy.deepcopy(kf.nxt)
        b, cb = host_twin(kf.nxt, kf.carry, ov)
        t1 = np.r_[t[1:], t[-1] + 0.5]
        m = kf.nxt["n_imu"]
        ig = integ_for(kf.nxt, kf.carry, {m - 1: p1["K"] - 1}, {m - 1: o.series(0, t1[m - 1], t1[m])})
        s1.slide_ins([a], [copy.deepcopy(kf.carry)], [dict(ig, imu_rows=None)], d, [0], [t1], None, synth_ba.NOISE5, vision=[kf.device()])
        s2.slide_integrate([b], [cb], [ig], synth_ba.NOISE5)
        compare_all(s1, s2, [a], [b])
        ext = ext_of(a)
        g = s1.update_and_cull_built([a], cam, STD, [ext])[0]
        h = s2.update_and_cull([b], cam, STD, [dict(ext, **{k: want[k] for k in LISTS})])[0]
        check_lists(g, want, a["L"], a["F"])
        check_cull(g, h)
        full = dict(b, **{k: a[k] for k in PARAMS})
        _, n0, c0 = build_next(full, 2812, drop=(0,), n_new=1)
        t_a = np.r_[t1[1:], t1[-1] + 0.5]
        mm = n0["n_imu"]
        g0 = integ_for(n0, c0, {mm - 1: 7}, {mm - 1: o.series(0, t_a[mm - 1], t_a[mm])})
        s1.slide_ins([copy.deepcopy(n0)], [c0], [dict(g0, imu_rows=None)], d, [0], [t_a], None, synth_ba.NOISE5, prior_from_marg=False)
        with pytest.raises(IcgError, match="no built lists"):
            s1.update_and_cull_built([n0], cam, STD, [ext_of(n0)])
    finally:
        s1.close(), s2.close(), d.close()
