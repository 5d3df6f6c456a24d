"""GPU: icg_ba_marginalize_built.  Twin handles go through the same keyframe cycle (vision slide -> two-pass solve -> culling on the built
lists); handle A then marginalizes with icg_ba_marginalize_resident_culled on the host lists the culling returned, handle B with
icg_ba_marginalize_built on problems that hold only their camera side.  The priors must be equal bit for bit, and so must everything the
next slide and solve compute from them."""
import copy
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import slide_vision_oracle as so
from tests.test_cull_built_gpu import check_cull, ext_of
from tests.test_marg_large_gpu import make as make_large
from tests.test_post_solve_gpu import STD, make
from tests.test_slide_gpu import PARAMS, handle
from tests.test_slide_vision_gpu import Keyframe, cam, olib, solve_cull_marg  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def lean(p):
    """the camera side of a problem dict: no landmark or factor row"""
    return dict(p, invdepth=np.zeros(0), f_lm=np.zeros(0, np.int32), f_ref=np.zeros(0, np.int32), f_obs=np.zeros(0, np.int32),
                f_const=np.zeros(0), f_active=np.zeros(0, np.uint8))


def check_same(ma, mb):
    for x, y in zip(ma, mb):
        assert x["m"] == y["m"] and x["r"] == y["r"]
        for k in ("block_type", "block_node", "x0", "J0", "e0", "Hp", "bp"):
            assert np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes(), k


def both(sa, sb, pa, pb, ga, num_marg, nim):
    ma = sa.marginalize(pa, num_marg, resident=True, culled=ga, node_in_map=nim)
    mb = sb.marginalize_built([lean(p) for p in pb], num_marg, node_in_map=nim)
    check_same(ma, mb)
    return ma


def twin(olib, cam, probs, kw, seed, n_cycles, lean_b=False, extra=None):
    """n_cycles keyframes on twin handles; at each one, after the built culling, A's host-list marginalization against B's built one (first
    with num_marg alternating 1 / 2 and a node out of the map, then with num_marg 1, the prior the next slide consumes).  lean_b: B slides
    with rows=False and keeps no factor row.  extra(sa, sb, pa, pb, ga): more checks on the culled windows of the last keyframe."""
    pa, pb = probs, copy.deepcopy(probs)
    n = len(probs)
    sa, sb = handle(n=n, **kw), handle(n=n, **kw)
    try:
        for s, x in ((sa, pa), (sb, pb)):
            s.gvins_optimization_batch(x, 20)
        gs, mgs = solve_cull_marg(pa, sa, cam, seed, None)
        solve_cull_marg(pb, sb, cam, seed, None)
        refs = [so.reference_rows(p) for p in pa]
        for c in range(n_cycles):
            kfs = [Keyframe(p, g, mg, rf, seed + 10 * c + w) for w, (p, g, mg, rf) in enumerate(zip(pa, gs, mgs, refs))]
            os_ = [kf.oracle(p, rf) for kf, p, rf in zip(kfs, pa, refs)]
            a, ca = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
            b, cb = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.carry) for kf in kfs]
            va, vb = [kf.device() for kf in kfs], [kf.device() for kf in kfs]
            if c > 0:  # the built culling's own lists
                for v in va + vb:
                    v.pop("obs_factor")
            sa.slide_vision(a, ca, va)
            sb.slide_vision(b, cb, vb, rows=not lean_b)
            if lean_b:  # invdepth: the buffer the download fills
                b = [dict(lean(q), invdepth=np.zeros(q["L"])) for q in b]
                for x in cb:
                    x.pop("f_src", None), x.pop("lm_src", None)
            for s in (sa, sb):
                s.run_gvins(20)
            assert sa.gvins_optimization_end(a) == sb.gvins_optimization_end(b)
            for x, y in zip(a, b):
                for k in PARAMS:
                    if not (lean_b and k == "f_active"):
                        assert np.array_equal(x[k], y[k]), k
            exts = [ext_of(p) for p in a]
            ga = sa.update_and_cull_built(a, cam, STD, exts)
            gb = sb.update_and_cull_built(b, cam, STD, exts)
            for x, y in zip(ga, gb):
                check_cull(x, y)
            nim = [np.ones(p["K"], np.uint8) for p in a]
            nim[0][2] = 0  # gvinsRemoveAllSecondNewFrame took node 2 of window 0 out of the map
            both(sa, sb, a, b, ga, np.array([1 + w % 2 for w in range(n)], np.int32), nim)
            if extra is not None and c == n_cycles - 1:
                extra(sa, sb, a, b, ga)
            mgs = both(sa, sb, a, b, ga, 1, None)
            pa, pb, gs = a, b, ga
            refs = [o["lm_ref"] for o in os_]
        # the slide that consumes the last prior, and its two-pass solve
        kfs = [Keyframe(p, g, mg, rf, seed + 999 + w) for w, (p, g, mg, rf) in enumerate(zip(pa, gs, mgs, refs))]
        a, b = [copy.deepcopy(kf.nxt) for kf in kfs], [copy.deepcopy(kf.nxt) for kf in kfs]
        va, vb = [kf.device() for kf in kfs], [kf.device() for kf in kfs]
        for v in va + vb:
            v.pop("obs_factor")
        sa.slide_vision(a, [copy.deepcopy(kf.carry) for kf in kfs], va)
        sb.slide_vision(b, [copy.deepcopy(kf.carry) for kf in kfs], vb)
        for s in (sa, sb):
            s.run_gvins(20)
        assert sa.gvins_optimization_end(a) == sb.gvins_optimization_end(b)
        for x, y in zip(a, b):
            for k in PARAMS:
                assert np.array_equal(x[k], y[k]), k
        return gs
    finally:
        sa.close(), sb.close()


def special_cases(cam):
    def run(sa, sb, pa, pb, ga):
        # the reference observations name no factor (obs_factor -1)
        assert all((g["obs_factor"] == -1).any() for g in ga)
        # every landmark an outlier (a culling std no error passes), each through an outlier observation in its reference node: only the
        # camera side is marginalized
        exts = [ext_of(p) for p in pa]
        ta = sa.update_and_cull_built(pa, cam, 1e-12, exts)
        sb.update_and_cull_built(pb, cam, 1e-12, exts)
        assert all((t["lm_outlier"] != 0).all() for t in ta)
        t = ta[0]
        assert any(t["obs_outlier"][o] and t["obs_node"][o] == t["lm_ref_node"][l] for l in range(len(t["lm_ref_node"]))
                   for o in range(t["obs_off"][l], t["obs_off"][l + 1]))
        m = both(sa, sb, pa, pb, ta, 1, None)
        assert all(x["m"] <= 15 for x in m)
        # the culling of the chain again (the built lists are still current)
        for x, y in zip(sa.update_and_cull_built(pa, cam, STD, exts), ga):
            check_cull(x, y)
        sb.update_and_cull_built(pb, cam, STD, exts)
    return run


def test_mixed_batch(olib, cam):
    """24 cfg-3 windows of different sizes; num_marg 1 and 2; a node out of the map; every landmark an outlier; reason-1 landmarks"""
    probs = [make(olib, outliers=25, seed=3101 + w, K=10 - w % 4, L=300 - 40 * (w % 4)) for w in range(24)]
    twin(olib, cam, probs, dict(K=10), 3110, 1, extra=special_cases(cam))


def test_cfg4_window(olib, cam):
    """a cfg-4 window on a max_K = 20 handle: m above the one-CTA eigensolver's 118 rows; a block above 512 rows is refused, then a retry
    equals the twin"""
    from ic_gvins_b200 import IcgError

    def big(sa, sb, pa, pb, ga):
        with pytest.raises(IcgError, match="exceeds the 512 rows") as e:
            sb.marginalize_built([lean(p) for p in pb], 12)
        assert e.value.code == -4  # ICG_EUNSUPPORTED
        m = both(sa, sb, pa, pb, ga, 2, None)
        assert m[0]["m"] > 118

    twin(olib, cam, [make_large(olib, K=20, L=2000, seed=3201, n_ref=20, prior=True)], dict(K=20, L=2000, F=12000, R=292), 3210, 1, extra=big)


def test_three_keyframe_chain_without_factor_rows(olib, cam):
    """three keyframes; B slides with rows=False and keeps no factor row: every prior and every solve equals A's host-list chain"""
    probs = [make(olib, outliers=25, seed=3301, K=10, L=300), make(olib, outliers=25, seed=3302, K=9, L=200)]
    twin(olib, cam, probs, dict(K=10), 3310, 3, lean_b=True)


def test_contract(olib, cam):
    """each rejected call leaves the handle as it was: the retry succeeds and equals the twin's host-list marginalization"""
    from ic_gvins_b200 import IcgError
    from ic_gvins_b200._lib import lib
    from ic_gvins_b200.ba import vp
    pa = make(olib, outliers=25, seed=3401, K=10, L=300)
    pb = copy.deepcopy(pa)
    sa, sb = handle(n=2), handle(n=2)

    def reject(match, code=-1, **kw):
        with pytest.raises(IcgError, match=match) as e:
            sb.marginalize_built([lean(pb)], **kw)
        assert e.value.code == code

    try:
        for s, x in ((sa, pa), (sb, pb)):
            s.gvins_optimization_batch([x], 20)
        reject("no culling of these 1 windows")
        gs, mgs = solve_cull_marg([pa], sa, cam, 3410, None)
        solve_cull_marg([pb], sb, cam, 3410, None)
        reject("walked host lists")
        kf = Keyframe(pa, gs[0], mgs[0], so.reference_rows(pa), 3411)
        a, b = copy.deepcopy(kf.nxt), copy.deepcopy(kf.nxt)
        sa.slide_vision([a], [copy.deepcopy(kf.carry)], [kf.device()])
        sb.slide_vision([b], [copy.deepcopy(kf.carry)], [kf.device()])
        pb = b
        reject("no culling of these 1 windows")  # the slide ended the culling
        for s in (sa, sb):
            s.run_gvins(20)
        assert sa.gvins_optimization_end([a]) == sb.gvins_optimization_end([b])
        ga = sa.update_and_cull_built([a], cam, STD, [ext_of(a)])
        sb.update_and_cull_built([b], cam, STD, [ext_of(b)])
        with pytest.raises(IcgError, match="holds 1 uploaded windows"):
            sb.marginalize_built([lean(b), lean(b)])
        reject("out of range", num_marg=b["K"])
        call = sb.marg_prepare([lean(b)], 1)
        call["pri"][0].rcap = 15 * (b["K"] - 1) + 6  # one row short
        in_map = np.ones(b["K"], np.uint8)
        ptrs = (vp * 1)(vp(in_map.ctypes.data))
        assert lib().icg_ba_marginalize_built(sb._h, 1, call["arr"], vp(call["nm"].ctypes.data), ptrs, call["pri"]) == -1
        # the retry equals the twin, and its prior is the resident one: the next slide consumes it on both handles alike
        mg = sa.marginalize([a], 1, resident=True, culled=ga)
        check_same(mg, sb.marginalize_built([lean(b)], 1))
        kf2 = Keyframe(a, ga[0], mg[0], kf.oracle(pa, so.reference_rows(pa))["lm_ref"], 3412)
        a2, b2 = copy.deepcopy(kf2.nxt), copy.deepcopy(kf2.nxt)
        v1, v2 = kf2.device(), kf2.device()
        v1.pop("obs_factor"), v2.pop("obs_factor")
        sa.slide_vision([a2], [copy.deepcopy(kf2.carry)], [v1])
        sb.slide_vision([b2], [copy.deepcopy(kf2.carry)], [v2])
        for s in (sa, sb):
            s.run_gvins(20)
        assert sa.gvins_optimization_end([a2]) == sb.gvins_optimization_end([b2])
        for k in PARAMS:
            assert np.array_equal(a2[k], b2[k]), k
    finally:
        sa.close(), sb.close()
    # a two-rank landmark-shard group in this process: refused, naming the route that works there
    s0, s1 = handle(), handle()
    try:
        blobs = [s0.shard_export(0, 2), s1.shard_export(1, 2)]
        s0.shard_connect(blobs), s1.shard_connect(blobs)
        with pytest.raises(IcgError, match="icg_ba_marginalize_resident_culled and NULL lists") as e:
            s0.marginalize_built([lean(pa)])
        assert e.value.code == -4
    finally:
        s0.close(), s1.close()


SHIM = r'''
#include <cstdio>
#include <vector>
#include "ic_gvins_b200/host/icg_shims.hpp"
// links and runs WindowSolver::marginalizeBuilt: on a handle without windows it must throw, naming the call
int main() {
    icg_b200::WindowSolver s(10, 300, 2700);
    icg_ba_problem p{};
    p.K = 10;
    std::vector<uint8_t> in_map(10, 1);
    try {
        s.marginalizeBuilt(p, 1, in_map.data());
    } catch (const std::exception &e) {
        printf("%s\n", e.what());
        return 0;
    }
    return 1;
}
'''


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_shim_marginalize_built_runs():
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
        assert "icg_ba_marginalize_built" in r.stdout
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
