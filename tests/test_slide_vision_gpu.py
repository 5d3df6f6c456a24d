"""GPU: icg_ba_slide_vision_resident.  A handle solves, culls and marginalizes perturbed windows, then slides with the vision rows built on the
device from the culled windows, tracked observations and new map points held in device memory; a twin handle goes through the same calls and
slides (icg_ba_slide_resident, or icg_ba_slide_integrate_resident with the same integration) with the same windows built on the host by the
numpy restatement (tests/slide_vision_oracle.py).  The built structure must equal the restatement exactly, the inverse depths and new factor
rows bit for bit, and the two handles must then give the same bits in the two-pass solve, a resident marginalization and a restarted solve."""
import copy

import numpy as np
import pytest

from datagen.slide_window import build_next
from tests import oracle_api as oa
from tests import slide_vision_oracle as so
from tests.test_marg_large_gpu import make as make_large
from tests.test_post_solve_gpu import CAMD, STD, cull_inputs, make
from tests.test_slide_gpu import PARAMS, handle
from tests.test_slide_integrate_gpu import NOISE5, integ_for, intervals

pytestmark = pytest.mark.gpu

CAM = dict(fx=CAMD["fx"], fy=CAMD["fy"], cx=CAMD["cx"], cy=CAMD["cy"], skew=0.0)


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def cam():
    from ic_gvins_b200.camera import Camera
    return Camera([CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"]], [0.0, 0.0, 0.0, 0.0])


def cam_struct():
    from ic_gvins_b200.camera import CameraStruct
    return CameraStruct(CAMD["fx"], CAMD["fy"], CAMD["cx"], CAMD["cy"], 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)


def dev(a, dt):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dt)).cuda()


def solve_cull_marg(probs, s, cam, seed, full_fc=None):
    """the culling and the culled marginalization of every window the handle has just solved; full_fc[w]: the window's f_const with every row (the
    culling inputs are drawn from it)"""
    cis = []
    for w, p in enumerate(probs):
        q = dict(p, f_const=full_fc[w]) if full_fc else p
        cis.append(cull_inputs(q, p["ext"].copy(), seed + w, bad_kp=20))
    gs = s.update_and_cull(probs, cam, STD, cis)
    mgs = s.marginalize(probs, 1, resident=True, culled=gs)
    return gs, mgs


class Keyframe:
    """one new keyframe of one window: the next camera side (node 0 marginalized, one new node, the prior from the marginalization) and the
    new observations: tracked points of carried, culled and unknown landmarks (landmarks with a known reference row, factor-less ones
    included), one in its landmark's reference node, and new map points anchored in three earlier nodes"""

    def __init__(self, p, g, mg, lm_ref, seed, n_new=7, n_obs=60, out_of_map=()):
        rng = np.random.default_rng(seed)
        _, self.nxt, self.carry = build_next(p, seed, drop=(0,), n_new=1)
        for k, v in (("marg_r", mg["r"]), ("marg_nblocks", len(mg["block_type"])), ("marg_block_type", mg["block_type"]),
                     ("marg_block_node", mg["block_node"]), ("marg_x0", mg["x0"]), ("marg_J0", mg["J0"].reshape(-1).copy()), ("marg_e0", mg["e0"].copy())):
            self.nxt[k] = v
        K2 = self.nxt["K"]
        self.cur = K2 - 1
        known = np.nonzero(~np.isnan(lm_ref[:, 0]))[0]
        lms = rng.choice(known, size=min(n_obs, len(known)), replace=False)
        self.obs = [(int(l), self.cur) for l in lms] + [(-1, self.cur), (-1, self.cur)]
        ref = g["lm_ref_node"]
        l0 = next(l for l in range(p["L"]) if ref[l] >= 1)
        self.obs.append((int(l0), int(ref[l0]) - 1))  # in its reference node: skipped
        m = len(self.obs)
        self.xy = rng.uniform([100, 60], [1180, 500], (m, 2)).astype(np.float32)
        self.vel = rng.normal(0, 5, (m, 2))
        self.frames = {1000 + k: k for k in range(K2)}
        self.new = dict(depth=rng.uniform(2, 40, n_new), ref_xy=rng.uniform([100, 60], [1180, 500], (n_new, 2)).astype(np.float32),
                        vel_ref=rng.normal(0, 5, (n_new, 2)), ref_id=np.array([1000 + (self.cur - 1 - j % 3) for j in range(n_new)], np.int64),
                        cur_xy=rng.uniform([100, 60], [1180, 500], (n_new, 2)).astype(np.float32), vel_cur=rng.normal(0, 5, (n_new, 2)))
        self.node_td = rng.normal(0, 1e-3, K2)
        self.K_old, self.g = p["K"], g
        self.in_map = np.ones(p["K"], np.uint8)
        self.in_map[list(out_of_map)] = 0  # gvinsRemoveAllSecondNewFrame: factors observed there drop, their landmarks may stay factor-less

    def device(self):
        o, n = self.obs, self.new
        return dict(num_marg=1, node_in_map=self.in_map, obs_factor=self.g["obs_factor"], camera=cam_struct(), node_td=self.node_td,
                    cur_node=self.cur, frames=self.frames, n_obs=len(o), obs_lm=dev([x[0] for x in o], np.int32), obs_node=dev([x[1] for x in o], np.int32),
                    obs_undis_xy=dev(self.xy, np.float32), obs_vel=dev(self.vel, np.float64), n_new=len(n["depth"]), new_depth=dev(n["depth"], np.float64),
                    new_ref_undis_xy=dev(n["ref_xy"], np.float32), new_vel_ref=dev(n["vel_ref"], np.float64), new_ref_frame_id=dev(n["ref_id"], np.int64),
                    new_cur_undis_xy=dev(n["cur_xy"], np.float32), new_vel_cur=dev(n["vel_cur"], np.float64))

    def oracle(self, p, lm_ref):
        n = self.new
        vis = dict(num_marg=1, node_in_map=self.in_map, node_td=self.node_td, cur_node=self.cur, frames=self.frames,
                   obs=[(l, nd, self.xy[i], self.vel[i]) for i, (l, nd) in enumerate(self.obs)],
                   new=[dict(depth=n["depth"][j], ref_xy=n["ref_xy"][j], vel_ref=n["vel_ref"][j], ref_id=int(n["ref_id"][j]), cur_xy=n["cur_xy"][j],
                             vel_cur=n["vel_cur"][j]) for j in range(len(n["depth"]))])
        return so.build(dict(p, lm_ref=lm_ref), self.g, self.carry["node_src"], vis, CAM)


def host_twin(nxt, carry, o):
    q, c = copy.deepcopy(nxt), copy.deepcopy(carry)
    q.update(L=o["L"], F=o["F"], invdepth=o["invdepth"].copy(), f_lm=o["f_lm"], f_ref=o["f_ref"], f_obs=o["f_obs"], f_const=o["f_const"].reshape(-1).copy(),
             f_active=np.ones(o["F"], np.uint8))
    c.update(lm_src=o["lm_src"], f_src=o["f_src"])
    return q, c


def check_built(r, o):
    for k in ("L", "F", "nan_dropped"):
        assert r[k] == o[k], k
    for k in ("lm_src", "lm_origin", "f_src", "f_lm", "f_ref", "f_obs", "invdepth"):
        assert np.array_equal(r[k], o[k]), k
    assert np.array_equal(r["nan_flags"][:len(o["nan_flags"])], o["nan_flags"])
    new_rows = o["f_src"] < 0
    assert np.array_equal(r["f_const"][new_rows], o["f_const"][new_rows])


def compare_all(s1, s2, a, b, n_iter=20):
    """the two-pass solve, a resident marginalization and a restarted solve of the two handles, bitwise"""
    for s in (s1, s2):
        s.run_gvins(n_iter)
    assert s1.gvins_optimization_end(a) == s2.gvins_optimization_end(b)
    for x, y in zip(a, b):
        for k in PARAMS:
            assert np.array_equal(x[k], y[k]), k
    m1, m2 = s1.marginalize(a, 1, resident=True), s2.marginalize(b, 1, resident=True)
    for x, y in zip(m1, m2):
        assert x["m"] == y["m"] and x["r"] == y["r"]
        for k in ("J0", "e0", "Hp", "bp"):
            assert np.array_equal(x[k], y[k]), k
    for s in (s1, s2):
        s.run_gvins(n_iter, restart=True)
    assert s1.gvins_optimization_end(a) == s2.gvins_optimization_end(b)
    for x, y in zip(a, b):
        for k in PARAMS:
            assert np.array_equal(x[k], y[k]), k


def cycle(olib, cam, probs, kw, seed, n_cycles, integrate=False):
    """returns how many new factors went to landmarks that had no factor in the window they came from"""
    """n_cycles keyframes of solve -> culling -> culled marginalization -> slide on B windows, device-built against host-built at every step"""
    p1, p2 = probs, copy.deepcopy(probs)
    s1, s2 = handle(n=len(probs), **kw), handle(n=len(probs), **kw)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch(x, 20)
        refs = [so.reference_rows(p) for p in p1]
        full, factorless = None, 0
        for c in range(n_cycles):
            gs, mgs = solve_cull_marg(p1, s1, cam, seed + 10 * c, full)
            solve_cull_marg(p2, s2, cam, seed + 10 * c, full)
            kfs = [Keyframe(p, g, mg, rf, seed + 10 * c + w, out_of_map=(2, 3, 5) if c == 0 and n_cycles > 1 else ()) for w, (p, g, mg, rf) in enumerate(zip(p1, gs, mgs, refs))]
            os_ = [kf.oracle(p, rf) for kf, p, rf in zip(kfs, p1, refs)]
            a = [copy.deepcopy(kf.nxt) for kf in kfs]
            ca = [copy.deepcopy(kf.carry) for kf in kfs]
            twins = [host_twin(kf.nxt, kf.carry, o) for kf, o in zip(kfs, os_)]
            b, cb = [t[0] for t in twins], [t[1] for t in twins]
            if integrate:
                ig = []
                for w, (kf, p) in enumerate(zip(kfs, p1)):
                    k = kf.nxt["n_imu"] - 1
                    ig.append(integ_for(kf.nxt, kf.carry, {k: p["K"] - 1}, {k: intervals(p, p["K"] - 1, 1, seed + 100 * c + w)[0]}))
                r = s1.slide_vision(a, ca, [kf.device() for kf in kfs], ig, NOISE5)
                s2.slide_integrate(b, cb, ig, NOISE5)
            else:
                r = s1.slide_vision(a, ca, [kf.device() for kf in kfs])
                s2.slide(b, cb, True)
            for x, o, p in zip(r, os_, p1):
                check_built(x, o)
                bare = np.setdiff1d(np.arange(p["L"]), p["f_lm"])
                factorless += int(np.isin(o["lm_origin"][o["f_lm"][o["f_src"] < 0]], bare).sum())
            compare_all(s1, s2, a, b)
            p1, p2 = a, b
            refs = [o["lm_ref"] for o in os_]
            full = [x["f_const"].copy() for x in b]
            for x, y in zip(p1, full):  # the twin's rows are the full rows the device window holds
                x["f_const"] = y.copy()
        return factorless
    finally:
        s1.close(), s2.close()


def test_mixed_batch(olib, cam):
    """three windows of different sizes in one call; each built window equals the restatement and the handle the host-built twin"""
    probs = [make(olib, outliers=25, seed=1101, K=10, L=300), make(olib, outliers=10, seed=1102, K=8, L=150),
             make(olib, outliers=10, seed=1103, K=7, L=120)]
    cycle(olib, cam, probs, dict(K=10), 1110, 1)
    assert any((x["f_active"] == 0).any() for x in probs)  # the chi-square pass removed factors; the built windows (oracle-equal) restore them


def test_cycle_of_three_keyframes(olib, cam):
    """three keyframes of solve -> culling -> culled marginalization -> vision slide on two windows: the second and third slides start from a
    window a vision slide built, and every new observation takes its pts0 / vel0 / td0 from the reference rows the earlier slides carried
    (the first keyframe takes nodes 2, 3 and 5 out of the map, so many landmarks lose factors there)"""
    probs = [make(olib, outliers=25, seed=1201, K=10, L=300), make(olib, outliers=25, seed=1202, K=9, L=200)]
    cycle(olib, cam, probs, dict(K=10), 1210, 3)


def test_integrating_slide(olib, cam):
    """the call with integ: the new keyframe's IMU factor integrated on the device, against icg_ba_slide_integrate_resident"""
    cycle(olib, cam, [make(olib, outliers=25, seed=1301, K=10, L=300)], dict(K=10), 1310, 2, integrate=True)


def test_cfg4_window(olib, cam):
    cycle(olib, cam, [make_large(olib, K=20, L=2000, seed=1401, n_ref=20, prior=True)], dict(K=20, L=2000, F=12000, R=292), 1410, 1)


def test_device_handoff_through_src_and_device_counts(olib, cam):
    """the tracked list compacted with a src indirection and its count on the device (icg_klt_track_frames_dev's map list), the new points
    in a longer buffer with their count on the device (icg_klt_triangulate_dev's dev_counts): the same window as the direct arrays"""
    p = make(olib, outliers=25, seed=1501, K=10, L=300)
    s = handle()
    try:
        s.gvins_optimization_batch([p], 20)
        gs, mgs = solve_cull_marg([p], s, cam, 1510, None)
        kf = Keyframe(p, gs[0], mgs[0], so.reference_rows(p), 1511)
        o = kf.oracle(p, so.reference_rows(p))
        rng = np.random.default_rng(1512)
        m = len(kf.obs)
        n_in = m + 25  # the input list: the survivors at scattered positions, dropped points between them
        src = np.sort(rng.choice(n_in, size=m, replace=False)).astype(np.int32)
        lm_in, node_in = np.full(n_in, -1, np.int32), np.full(n_in, 77, np.int32)  # node 77: out of range, never read for a dropped point
        lm_in[src], node_in[src] = [x[0] for x in kf.obs], [x[1] for x in kf.obs]
        cap = m + 40
        xy, vel = np.zeros((cap, 2), np.float32), np.zeros((cap, 2))
        xy[:m], vel[:m] = kf.xy, kf.vel
        v = kf.device()
        nn = len(kf.new["depth"])
        ncap = nn + 9
        pad = lambda a, dt: dev(np.concatenate([np.asarray(a, dt), np.zeros((ncap - nn,) + np.asarray(a).shape[1:], dt)]), dt)
        counts = dev([0, m, 0, 0, 0, 0, nn, 0, 0, 0], np.int32)  # dev_n_out + 2 s and dev_counts + 5 s + 1 of stream 0
        v.update(n_obs=cap, n_in=n_in, obs_src=dev(src, np.int32), dev_n=counts[1:], obs_lm=dev(lm_in, np.int32), obs_node=dev(node_in, np.int32),
                 obs_undis_xy=dev(xy, np.float32), obs_vel=dev(vel, np.float64), n_new=ncap, dev_new_n=counts[6:],
                 new_depth=pad(kf.new["depth"], np.float64), new_ref_undis_xy=pad(kf.new["ref_xy"], np.float32), new_vel_ref=pad(kf.new["vel_ref"], np.float64),
                 new_ref_frame_id=pad(kf.new["ref_id"], np.int64), new_cur_undis_xy=pad(kf.new["cur_xy"], np.float32),
                 new_vel_cur=pad(kf.new["vel_cur"], np.float64))
        r = s.slide_vision([copy.deepcopy(kf.nxt)], [copy.deepcopy(kf.carry)], [v])[0]
        check_built(r, o)
    finally:
        s.close()


def test_rejections_leave_the_handle_as_it_was(olib, cam):
    from ic_gvins_b200 import IcgError
    p1 = make(olib, outliers=25, seed=1601, K=10, L=300)
    p2 = copy.deepcopy(p1)
    s1, s2 = handle(L=320), handle(L=320)
    try:
        for s, x in ((s1, p1), (s2, p2)):
            s.gvins_optimization_batch([x], 20)
        gs, mgs = solve_cull_marg([p1], s1, cam, 1610, None)
        solve_cull_marg([p2], s2, cam, 1610, None)
        ref = so.reference_rows(p1)
        big = Keyframe(p1, gs[0], mgs[0], ref, 1611, n_new=120)  # more landmarks than max_L = 320
        assert big.oracle(p1, ref)["L"] > 320
        kf = Keyframe(p1, gs[0], mgs[0], ref, 1612)

        def reject(v, match):
            with pytest.raises(IcgError, match=match):
                s1.slide_vision([copy.deepcopy(kf.nxt)], [copy.deepcopy(kf.carry)], [v])

        reject(big.device(), "the handle holds")
        reject(dict(kf.device(), frames={k: n for k, n in kf.frames.items() if k != 1000 + kf.cur - 1}), "frame table")
        o = kf.oracle(p1, ref)
        lnew = next(int(o["lm_origin"][o["f_lm"][f]]) for f in np.nonzero(o["f_src"] < 0)[0] if o["lm_origin"][o["f_lm"][f]] >= 0)
        dup = kf.device()
        dup["obs_lm"][0], dup["obs_lm"][1] = lnew, lnew
        reject(dup, "two observations")
        reject(dict(kf.device(), obs_node=dev([77] * len(kf.obs), np.int32)), "node is out of range")
        # the culling state, the reference rows and the window survived: the good call still matches the twin
        a, ca = copy.deepcopy(kf.nxt), copy.deepcopy(kf.carry)
        check_built(s1.slide_vision([a], [ca], [kf.device()])[0], o)
        b, cb = host_twin(kf.nxt, kf.carry, o)
        s2.slide([b], [cb], True)
        compare_all(s1, s2, [a], [b])
    finally:
        s1.close(), s2.close()


def test_needs_a_current_culling_and_an_unsharded_handle(olib):
    from ic_gvins_b200 import IcgError
    p = make(olib, seed=1701, K=8, L=100)
    s = handle(K=10)
    try:
        s.gvins_optimization_batch([p], 20)
        nxt, carry = build_next(p, 1702, drop=(0,), n_new=1)[1:]
        vis = dict(num_marg=1, node_in_map=np.ones(p["K"], np.uint8), camera=cam_struct(), node_td=np.zeros(nxt["K"]), cur_node=nxt["K"] - 1)
        with pytest.raises(IcgError, match="no culling"):
            s.slide_vision([nxt], [carry], [vis])
        s.shard_export(0, 2)
        with pytest.raises(IcgError, match="landmark-sharded") as e:
            s.slide_vision([nxt], [carry], [vis])
        assert e.value.code == -4  # ICG_EUNSUPPORTED
        s.shard_leave()
    finally:
        s.close()
