"""The window's normal equations and reduced camera system on the device, entry by entry, against the high-precision assembly of
tests/lin_system_mp.py: every array WindowSolver.peek_linearization reads out after icg_ba_run(h, 0, restart=1) -- the per-pair Gram
matrices, A_W, h_l, g_l, the per-factor costs and the Jacobi scaling of ba_lin_vis, H_c and g_c of ba_lin_cam, Hs and the vision vectors of
ba_schur_dmma -- within its bound.  The windows sit at the kernels' edges, restated from the code below; each test prints its worst
error-to-bound ratio per kernel.  Then bitwise checks that need no reference: capacities, the other windows of a batch and the candidate
path (at_cand = 1) do not change a bit of the system."""
import copy
import os
import re

import numpy as np
import pytest

from datagen import synth_ba
from tests import lin_system_mp as lm
from tests import oracle_api as oa
from tests.test_ba_sizes_gpu import lin_vis_runs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RADIUS0 = 1e4


def _const(path, name):
    return int(re.search(rf"\b{name}\s*=\s*(\d+)", open(os.path.join(ROOT, "ic_gvins_b200", "csrc", path)).read()).group(1))


SCHUR_RCH, SCHUR_PASS, BA_SPLIT_W = _const("ba_dev.cuh", "SCHUR_RCH"), _const("ba_dev.cuh", "SCHUR_PASS"), _const("ba_dev.cuh", "BA_SPLIT_W")
LV_THREADS = int(re.search(r"__launch_bounds__\((\d+), \d+\) ba_lin_vis\(", open(os.path.join(ROOT, "ic_gvins_b200", "csrc", "ba.cu")).read()).group(1))
CAM_THREADS_1RANK = int(re.search(r"cam_threads\(const icg_ba \*h\) \{ return h->D.world >= 4 \? CAM_THREADS : (\d+);",
                                  open(os.path.join(ROOT, "ic_gvins_b200", "csrc", "ba_handle.cu")).read()).group(1))


def schur_passes(K):
    """ba_schur_dmma's passes at K: NCA = roundup4(NCV + 1), T2 = ceil(NCA / 16) super-tile rows, nsuper = T2 (T2 + 1) / 2 upper super-tiles,
    SCHUR_PASS of them per pass"""
    NCA = 4 * ((6 * K + 7 + 1 + 3) // 4)
    T2 = (NCA + 15) // 16
    return (T2 * (T2 + 1) // 2 + SCHUR_PASS - 1) // SCHUR_PASS


def schur_split_rows(L):
    """landmark rows of each of ba_schur_dmma's BA_SPLIT_W cluster CTAs: nsteps = ceil(L / 4) k-steps, split k takes rows
    [4 floor(nsteps k / W), min(L, 4 floor(nsteps (k + 1) / W))), staged in chunks of SCHUR_RCH rows"""
    nsteps = (L + 3) // 4
    return [min(L, 4 * (nsteps * (k + 1) // BA_SPLIT_W)) - 4 * (nsteps * k // BA_SPLIT_W) for k in range(BA_SPLIT_W)]


# ---------------------------------------------------------------------------------------------------------------------------------- windows
def _trim(prob, plan):
    """keep, per (reference node, observations) of plan, one landmark of that reference node with at least that many factors, cut to its
    first ones; landmark ids follow the plan"""
    nobs = np.bincount(prob["f_lm"], minlength=prob["L"])
    ref = np.full(prob["L"], -1)
    ref[prob["f_lm"]] = prob["f_ref"]
    used, keep, fk = set(), [], []
    for r, n in plan:
        l = next(l for l in range(prob["L"]) if l not in used and ref[l] == r and nobs[l] >= n)
        used.add(l)
        keep.append(l)
        fk += list(np.flatnonzero(prob["f_lm"] == l)[:n])
    fk = np.array(fk, int)
    new_id = np.full(prob["L"], -1)
    new_id[keep] = np.arange(len(keep))
    prob.update(L=len(keep), F=len(fk), invdepth=prob["invdepth"][keep].copy(), f_lm=new_id[prob["f_lm"][fk]].astype(np.int32),
                f_ref=prob["f_ref"][fk].copy(), f_obs=prob["f_obs"][fk].copy(), f_const=prob["f_const"].reshape(-1, 14)[fk].reshape(-1).copy(),
                f_active=np.ones(len(fk), np.uint8))
    return prob


def _extra_gnss(prob, n):
    """n GNSS fixes in all: the window's fixes repeated on their nodes with other offsets (several fixes per node)"""
    g = prob["n_gnss"]
    idx = np.arange(n) % g
    blh = prob["gnss_blh"].reshape(-1, 3)[idx] + np.linspace(-0.3, 0.3, n)[:, None]
    prob.update(n_gnss=n, gnss_node=prob["gnss_node"][idx].astype(np.int32), gnss_blh=blh.reshape(-1).copy(),
                gnss_std=prob["gnss_std"].reshape(-1, 3)[idx].reshape(-1).copy())
    return prob


def _inactive(prob, frac_every, whole_lm=None):
    prob["f_active"][::frac_every] = 0
    if whole_lm is not None:
        prob["f_active"][prob["f_lm"] == whole_lm] = 0
    return prob


def _cap_obs(prob, n):
    """every landmark's first n factors only (a window of many landmarks at a small reference cost)"""
    fk = np.concatenate([np.flatnonzero(prob["f_lm"] == l)[:n] for l in range(prob["L"])]).astype(int)
    fk.sort()
    prob.update(F=len(fk), f_lm=prob["f_lm"][fk].copy(), f_ref=prob["f_ref"][fk].copy(), f_obs=prob["f_obs"][fk].copy(),
                f_const=prob["f_const"].reshape(-1, 14)[fk].reshape(-1).copy(), f_active=np.ones(len(fk), np.uint8))
    return prob


def _no_factor_landmark(prob):
    """one more landmark, without factors (h_l = 0: the min_diagonal clamp decides phi_l)"""
    prob.update(L=prob["L"] + 1, invdepth=np.append(prob["invdepth"], 0.05))
    return prob


def _make(olib, edit=None, **kw):
    prob = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), **kw)[0]
    return edit(prob) if edit else prob


def _long_runs(olib):
    """K = 14: node 0 anchors 9 landmarks of 13 factors and one of 11 (a run of exactly 128 record slots), then one of 5 (a second run of
    node 0); node 1 anchors 9 of 12, one of 11 and one of 8 (127 slots); node 2 one landmark of 1 factor (a run of 1); nodes 3 .. 13 none"""
    plan = [(0, 13)] * 9 + [(0, 11), (0, 5)] + [(1, 12)] * 9 + [(1, 11), (1, 8)] + [(2, 1)]
    prob = _make(olib, K=14, L=240, seed=7014, n_ref=3, full_visibility=True, dt_node=0.1, pixel_noise=2.0)
    return _trim(prob, plan)


WINDOWS = {
    # name: (why, builder)
    "K2-L3": ("K = 2 (the smallest NCA), L = 3 < 4 (cluster CTAs with empty landmark splits, L mod 4 = 3), both priors",
              lambda o: _make(o, K=2, L=3, seed=9002, n_ref=1, with_priors=True)),
    "K6-L5": ("K = 6: 5 IMU factors = one round of the 5 warps; L mod 4 = 1; a marginalization prior of every block type",
              lambda o: _make(o, K=6, L=5, seed=9006, with_marg=True)),
    "K7-L6": ("K = 7: 6 IMU factors, one past a round; L mod 4 = 2; no GNSS; the Normal preintegration; no ImuErrorFactor",
              lambda o: _make(o, lambda p: p.update(n_gnss=0, gnss_node=np.zeros(0, np.int32), gnss_blh=np.zeros(0), gnss_std=np.zeros(0),
                                                          has_imu_error=0) or p, K=7, L=6, seed=9007, earth=False)),
    "K11-L79": ("K = 11: 10 IMU factors = two rounds; L mod 4 = 3 with 20 rows per Schur split; ext_const and td_const; reproj_huber off; "
                "pose prior only",
                lambda o: _make(o, lambda p: p.update(ext_const=1, td_const=1, reproj_huber=0, has_mix_prior=0) or p,
                                K=11, L=79, seed=9011, with_priors=True)),
    "K12-L81": ("K = 12: the last single-pass Schur, 11 IMU factors; L mod 4 = 1 with a short last split; 16 GNSS fixes (several per node) "
                "with Huber; "
                "mix prior only", lambda o: _make(o, lambda p: _extra_gnss(p, 16).update(has_pose_prior=0) or p,
                                                  K=12, L=81, seed=9012, with_priors=True, pixel_noise=2.0)),
    "K13-L160": ("K = 13: the first two-pass Schur; L mod 4 = 0; every 7th factor inactive, landmark 3's factors all inactive, one "
                 "landmark without factors", lambda o: _make(o, lambda p: _no_factor_landmark(_inactive(p, 7, whole_lm=3)),
                                                             K=13, L=159, seed=9013, with_marg=True)),
    "K14-runs": ("K = 14 (the largest ba_solve window): runs of exactly 128, 127 and 1 record slots, node 0 with two runs, runs observed "
                 "from 13 nodes (more than ba_lin_vis's warps), nodes without landmarks, factors on both sides of the Huber knee", _long_runs),
    # ba_schur_dmma's row chunks: rows per cluster split (schur_split_rows) at SCHUR_RCH - 1, SCHUR_RCH, SCHUR_RCH + 1 (a second chunk of one
    # row) and 2 SCHUR_RCH (two full chunks, restaged and accumulated) + 1 (a third chunk of one row); at most 2 factors per landmark
    "K3-L319": ("L = 319: splits of 80, 80, 80 and 79 = SCHUR_RCH - 1 rows (one chunk each)",
                lambda o: _make(o, lambda p: _cap_obs(p, 2), K=3, L=319, seed=9103)),
    "K4-L321": ("L = 321: splits of 80, 80, 80 and 81 = SCHUR_RCH + 1 rows (a second chunk of one row)",
                lambda o: _make(o, lambda p: _cap_obs(p, 2), K=4, L=321, seed=9104)),
    "K13-L641": ("K = 13 (two passes), L = 641: splits of 160 = 2 SCHUR_RCH rows (two full chunks) and 161 (a third chunk of one row)",
                 lambda o: _make(o, lambda p: _cap_obs(p, 2), K=13, L=641, seed=9113, n_ref=12)),
}
HANDLE = dict(max_windows=4, max_K=14, max_L=700, max_F=1600, max_gnss=16, max_marg_r=64)


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def windows(olib):
    made = {}

    def get(name):
        if name not in made:
            made[name] = WINDOWS[name][1](olib)
            made[name]["why"] = WINDOWS[name][0]
        return copy.deepcopy(made[name])
    return get


# ---------------------------------------------------------------------------------------------------------------------------------- CPU
def test_the_windows_reach_every_edge(windows):
    """each edge the module docstring names is in the data (restated from the code, so a moved constant shows here)"""
    ws = {n: windows(n) for n in WINDOWS}
    assert CAM_THREADS_1RANK == 160
    warps = CAM_THREADS_1RANK // 32
    assert {ws[n]["n_imu"] for n in ws} >= {warps, warps + 1, 2 * warps, 2 * warps + 1}
    Ls = {ws[n]["L"] for n in ws}
    assert min(Ls) < 4 and {L % 4 for L in Ls} == {0, 1, 2, 3}
    split_rows = [r for L in Ls for r in schur_split_rows(L)]
    assert 0 in split_rows                                                   # a cluster CTA without landmarks
    assert {SCHUR_RCH - 1, SCHUR_RCH, SCHUR_RCH + 1, 2 * SCHUR_RCH, 2 * SCHUR_RCH + 1} <= set(split_rows)
    assert schur_split_rows(641) == [2 * SCHUR_RCH] * 3 + [2 * SCHUR_RCH + 1] and schur_passes(ws["K13-L641"]["K"]) == 2
    assert schur_passes(12) == 1 and schur_passes(13) == 2 and {12, 13, 2, 14} <= {ws[n]["K"] for n in ws}
    runs = lin_vis_runs(ws["K14-runs"])
    assert {128, 127, 1} <= set(runs)
    p = ws["K14-runs"]
    ref = np.full(p["L"], -1)
    ref[p["f_lm"]] = p["f_ref"]
    assert sum(1 for k in range(p["K"]) if not (ref == k).any()) >= 3
    pair_counts = np.bincount(p["f_ref"] * p["K"] + p["f_obs"])
    assert 1 in pair_counts and any(c % 2 == 1 and c > 1 for c in pair_counts)
    assert max(len(set(p["f_obs"][p["f_ref"] == r])) for r in range(p["K"])) > LV_THREADS // 32
    m = ws["K13-L160"]
    assert (m["f_active"] == 0).any() and not m["f_active"][m["f_lm"] == 3].any() and m["L"] - 1 not in set(m["f_lm"])
    assert ws["K6-L5"]["marg_r"] > 0 and set(ws["K6-L5"]["marg_block_type"]) == {0, 1, 2, 3}
    assert ws["K12-L81"]["n_gnss"] == HANDLE["max_gnss"] and ws["K7-L6"]["n_gnss"] == 0
    assert {ws[n]["has_imu_error"] for n in ws} == {0, 1} and {ws[n]["has_pose_prior"] for n in ws} == {0, 1}
    assert {ws[n]["has_mix_prior"] for n in ws} == {0, 1}
    assert all(ws[n]["L"] <= HANDLE["max_L"] and ws[n]["F"] <= HANDLE["max_F"] for n in ws)


# ---------------------------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def solver():
    from ic_gvins_b200.ba import WindowSolver
    s = WindowSolver(**HANDLE)
    yield s
    s.close()


def system_at_x(s, probs):
    """upload, one linearisation and one Schur complement (icg_ba_run(h, 0, restart=1)), the read-out of every window"""
    s.upload(probs)
    s.run(0, restart=True)
    return [s.peek_linearization(w) for w in range(len(probs))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WINDOWS))
def test_system_matches_the_high_precision_assembly(windows, solver, name):
    prob = windows(name)
    dev = system_at_x(solver, [prob])[0]
    assert dev["radius"] == RADIUS0 and (dev["K"], dev["L"], dev["F"]) == (prob["K"], prob["L"], prob["F"])
    vis, cam = lm.factors(prob)
    if name == "K14-runs":  # Huber on and off per factor: factors on both sides of the knee
        assert any(v.sq > 1 for v in vis) and any(v.sq <= 1 for v in vis)
    ref = lm.assemble(prob, vis, cam, dev["radius"])
    rs = lm.ratios(dev, ref)
    per_kernel = {k: max(v for a, v in rs.items() if lm.KERNEL_OF[a] == k) for k in lm.CONST}
    print(f"{name}: worst error / bound", {k: f"{v:.2e}" for k, v in per_kernel.items()}, {a: f"{v:.1e}" for a, v in rs.items()})
    assert max(rs.values()) <= 1.0, (prob["why"], rs)


COMPARED = ("Mp", "A_W", "h_l", "g_l", "H_c", "g_c", "costf", "scale_l", "Hs", "visv")


def assert_same(a, b, keys=COMPARED, what=""):
    for k in keys:
        if k == "Mp":
            assert a[k].keys() == b[k].keys(), what
            assert all(np.array_equal(a[k][p], b[k][p]) for p in a[k]), (what, k)
        else:
            assert np.array_equal(a[k], b[k]), (what, k)


@pytest.mark.gpu
def test_system_is_independent_of_the_capacity(windows, solver):
    from ic_gvins_b200.ba import WindowSolver
    other = WindowSolver(max_windows=2, max_K=13, max_L=170, max_F=900, max_gnss=12, max_marg_r=40)
    try:
        for name in ("K2-L3", "K6-L5", "K11-L79", "K13-L160"):
            assert_same(system_at_x(solver, [windows(name)])[0], system_at_x(other, [windows(name)])[0], what=name)
    finally:
        other.close()


@pytest.mark.gpu
def test_system_is_independent_of_the_other_windows(windows, solver):
    names = ["K13-L160", "K7-L6", "K14-runs", "K2-L3"]
    batch = system_at_x(solver, [windows(n) for n in names])
    for n, b in zip(names, batch):
        assert_same(b, system_at_x(solver, [windows(n)])[0], what=n)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["K6-L5", "K12-L81", "K14-runs"])
def test_candidate_linearisation_equals_a_fresh_one(windows, solver, name):
    """one accepted step: the buffer the window uses now (the candidate's, at_cand = 1) is bitwise the linearisation at x of a fresh upload
    of the accepted parameters (what does not depend on the radius or on the first linearisation's scaling)"""
    prob = windows(name)
    solver.upload([prob])
    solver.run(1, restart=True)
    summ = solver.download()[0]
    assert summ["num_successful_steps"] == 1
    dev = solver.peek_linearization(0)
    assert dev["lin_buf"] == 1
    # download(write_back=True) above wrote the accepted parameters into prob's arrays (the uploaded structs point at them)
    fresh = system_at_x(solver, [prob])[0]
    assert fresh["lin_buf"] == 0
    assert_same(dev, fresh, keys=("Mp", "A_W", "h_l", "g_l", "H_c", "g_c", "costf"), what=name)


@pytest.mark.gpu
def test_read_out_needs_a_linearisation(windows, solver):
    """after an upload and before any run the buffers do not hold the uploaded windows' system: the read-out refuses"""
    from ic_gvins_b200 import IcgError
    solver.upload([windows("K2-L3")])
    with pytest.raises(IcgError, match="no icg_ba_run"):
        solver.peek_linearization(0)
    solver.run(0, restart=True)
    assert solver.peek_linearization(0)["K"] == 2
