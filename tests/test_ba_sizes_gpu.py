"""The window solve across the max_K range icg_ba_create accepts (2 .. 32), against the CPU oracle (FP64 dense Schur + Cholesky).

The reduced camera system (n = 15 K + 7 columns) is solved by one of three kernels, chosen from the handle's capacity max_K:
    ba_solve           max_K  2 .. 14   one CTA, packed system in shared memory
    ba_solve_cam_dsm   max_K 15 .. 23   4-CTA cluster, 8 x 8 tiles in distributed shared memory (tile row T on CTA T mod 4)
    ba_solve_cam       max_K 24 .. 32   cluster, packed system in L2
Every kernel takes its strides from the capacity and its extent from the window, so each handle here solves windows of several sizes,
chosen where the layouts turn: the first and last max_K of each kernel, n = 0 mod 8 (the right-hand-side row opens a panel), every owner
CTA of ba_solve_cam_dsm's last tile row, its right-hand-side row at both ends of a tile, and the longest rows its staging admits.  Tracks
reach over the whole window (landmarks anchored in nodes 0 .. K - 2) and, at K = 32, over 31 nodes with lin_vis runs of 128 factors."""
import copy

import numpy as np
import pytest

from datagen import synth_ba
from tests import oracle_api as oa
from tests.test_ba_gpu import _compare_solution, oracle_two_pass, rel_err

SOLVE_KERNELS = ("ba_solve", "ba_solve_cam_dsm", "ba_solve_cam")


def solve_kernel(max_K: int) -> str:
    """The kernel that solves the reduced camera system of a max_K handle.  Restates ba_create_body in csrc/ba_handle.cu (ba_solve while
    its vectors and the packed augmented system fit 220 KB of one CTA) and split_setup there (with dsm_smem_doubles of csrc/ba_dev.cuh:
    ba_solve_cam_dsm while one CTA's share of the tiles fits 227 KB and a row is at most 11 staging chunks of 32)."""
    N = 15 * max_K + 7
    NS = (N + 3) & ~3
    if 8 * (40 + 5 * NS) + 8 * ((N + 1) * (N + 2) // 2) <= 220 * 1024:
        return "ba_solve"
    nt = (N + 1 + 7) // 8
    mx = max(sum(range(cr, nt, 4)) for cr in range(4))
    dsm = 8 * (40 + 8 * nt * 8 + 64 + 8 + 8 * 4 + 8 + 8 + nt * 64 * 3 + mx * 64)
    return "ba_solve_cam_dsm" if dsm <= 227 * 1024 and N <= 32 * 11 else "ba_solve_cam"


def dsm_layout(K: int):
    """(n, n & 7, owner CTA of the last tile row) of a K-node window in ba_solve_cam_dsm: the augmented right-hand-side row is row n, in
    tile row n >> 3 at row n & 7 (ba_solve_cam_dsm, csrc/ba_split.cuh), and tile row T lives on CTA T mod 4."""
    N = 15 * K + 7
    return N, N & 7, (N >> 3) % 4


def lin_vis_runs(prob):
    """Record slots of every ba_lin_vis run of a window, in run order.  Restates pack_window of csrc/ba_handle.cu: landmarks ordered by
    reference node (stable by id, landmarks without factors last), then greedy runs of whole landmarks of one reference node within 128
    slots, one slot per factor."""
    L, K = prob["L"], prob["K"]
    nobs = np.bincount(prob["f_lm"], minlength=L)
    ref = np.full(L, K)
    ref[prob["f_lm"]] = prob["f_ref"]
    order = np.argsort(ref, kind="stable")
    runs, l0 = [], 0
    while l0 < L:
        l1, slots = l0, 0
        while l1 < L and ref[order[l1]] == ref[order[l0]] and slots + nobs[order[l1]] <= 128:
            slots += nobs[order[l1]]
            l1 += 1
        assert l1 > l0, "a landmark with more than 128 factors"
        runs.append(int(slots))
        l0 = l1
    return runs


# Windows: synth_ba.make_window arguments (+ ext_const).  Landmarks anchored in nodes 0 .. K - 2 (n_ref = K - 1) couple every pose column.
WINDOWS = {
    "K2": dict(K=2, L=120, seed=3102, n_ref=1, with_priors=True),
    "K7": dict(K=7, L=200, seed=3107, n_ref=6, ext_const=True),
    "K10": dict(K=10, L=300, seed=3110, n_ref=9, with_priors=True),
    "K13": dict(K=13, L=300, seed=3113, n_ref=12, with_marg=True),
    "K14": dict(K=14, L=300, seed=3114, n_ref=13),
    "K15": dict(K=15, L=300, seed=3115, n_ref=14, with_marg=True, with_priors=True),
    "K16": dict(K=16, L=300, seed=3116, n_ref=15, ext_const=True),
    "K17": dict(K=17, L=300, seed=3117, n_ref=16, with_marg=True),
    "K21": dict(K=21, L=300, seed=3121, n_ref=20),
    "K23": dict(K=23, L=300, seed=3123, n_ref=22, with_priors=True, ext_const=True),
    "K24": dict(K=24, L=300, seed=3124, n_ref=23, with_marg=True),
    "K25": dict(K=25, L=300, seed=3125, n_ref=24, with_priors=True),
    "K31": dict(K=31, L=300, seed=3131, n_ref=30, with_marg=True, ext_const=True),
    # long tracks: nodes 0.1 s apart, every landmark seen to the end of the window -- landmarks with 31 observations, 128-slot runs
    "K32": dict(K=32, L=400, seed=5, n_ref=31, full_visibility=True, dt_node=0.1),
}

# Handles by max_K (max_gnss = 16, max_marg_r = 64) and the windows each solves.  10 and 24 are only used as the second capacity of a kernel.
HANDLES = {
    2: dict(max_windows=1, max_L=120, max_F=200),
    10: dict(max_windows=4, max_L=300, max_F=2700),
    14: dict(max_windows=4, max_L=300, max_F=1500),
    15: dict(max_windows=1, max_L=300, max_F=1500),
    23: dict(max_windows=5, max_L=300, max_F=1500),
    24: dict(max_windows=1, max_L=300, max_F=1500),
    32: dict(max_windows=5, max_L=400, max_F=6000),
}
SWEEP = {
    2: ("K2",),
    14: ("K2", "K7", "K13", "K14"),
    15: ("K15",),
    23: ("K10", "K16", "K17", "K21", "K23"),
    32: ("K2", "K14", "K25", "K31", "K32"),
}
POINTS = [(mk, name) for mk, names in SWEEP.items() for name in names]
# the same window on two handles of one kernel: bit-identical results
CAPACITY = [("K2", 2, 14), ("K10", 10, 14), ("K15", 15, 23), ("K24", 24, 32)]
# Largest relative gap of a first LM step's parameter increments to the oracle's, per group (below).  Measured on an H100 80GB HBM3
# (700 W power limit): at most 3.9e-11 over the sweep (ba_solve 3.9e-11, ba_solve_cam_dsm 2.9e-11, ba_solve_cam 3.9e-11).  A 1e-7
# relative error in the last 8 right-hand-side entries of ba_solve_cam_dsm's factorisation shows here as a 1e-7 gap, while the
# 20-iteration comparison does not see it.
ONE_STEP_REL = 1e-9


def _ids(points):
    return [f"maxK{mk}-{name}" for mk, name in points]


# ---------------------------------------------------------------------------------------------------------------------------------- CPU
def test_solve_kernel_ranges_and_sweep_ends():
    kernels = [solve_kernel(k) for k in range(2, 33)]
    assert kernels == ["ba_solve"] * 13 + ["ba_solve_cam_dsm"] * 9 + ["ba_solve_cam"] * 9
    for kernel in SOLVE_KERNELS:
        ks = [k for k in range(2, 33) if solve_kernel(k) == kernel]
        assert ks[0] in HANDLES and ks[-1] in HANDLES, kernel   # 2 and 14, 15 and 23, 24 and 32
    for mk, names in SWEEP.items():
        for name in names:
            assert WINDOWS[name]["K"] <= mk
    for name, a, b in CAPACITY:
        assert solve_kernel(a) == solve_kernel(b) and WINDOWS[name]["K"] <= min(a, b)


def test_sweep_covers_the_layout_turns():
    Ks = {mk: [WINDOWS[n]["K"] for n in SWEEP[mk]] for mk in SWEEP}
    # ba_solve: the largest window it accepts, and n = 0 mod 8 (the right-hand-side row opens a new 8-column panel)
    assert 14 in Ks[14] and any((15 * K + 7) % 8 == 0 for K in Ks[14])
    # ba_solve_cam_dsm: every owner CTA of the last tile row, the right-hand-side row first (rn = 0) and last (rn = 7) in its tile, the
    # longest row the staging admits (n = 352 = 11 x 32), and windows smaller than the handle
    dsm = [dsm_layout(K) for K in Ks[15] + Ks[23]]
    assert {o for _, _, o in dsm} == {0, 1, 2, 3}
    assert {0, 7} <= {rn for _, rn, _ in dsm}
    assert 352 in [n for n, _, _ in dsm] and min(Ks[23]) < 23
    # ba_solve_cam: the largest window, n = 0 mod 8, and windows far below the capacity
    assert 32 in Ks[32] and any((15 * K + 7) % 8 == 0 for K in Ks[32]) and min(Ks[32]) == 2


def test_long_track_window_has_full_runs(olib):
    """dt_node = 0.1 at K = 32: landmarks observed by every later node and lin_vis runs that fill all 128 record slots."""
    prob = _window(olib, "K32")
    runs = lin_vis_runs(prob)
    nobs = np.bincount(prob["f_lm"], minlength=prob["L"])
    assert prob["F"] == 5291 and sum(runs) == prob["F"]
    assert int((nobs == 31).sum()) == 7 and runs.count(128) == 3


def test_eight_observation_window_is_all_full_runs(olib):
    prob = _eight_observation_window(olib)
    runs = lin_vis_runs(prob)
    assert prob["L"] % 16 == 0 and prob["F"] == 8 * prob["L"] and runs == [128] * (prob["L"] // 16)
    assert np.all(np.bincount(prob["f_lm"], minlength=prob["L"]) == 8) and np.all(prob["f_ref"] == 0)


def test_lin_vis_runs_restates_the_greedy_packing():
    """Hand-built window: landmarks of reference 1 listed before those of reference 0, one landmark without factors, a landmark that
    does not fit the open run."""
    nobs = {0: (1, 100), 1: (0, 60), 2: (1, 20), 3: (0, 70), 4: (1, 9), 5: (None, 0), 6: (0, 1)}
    f_lm, f_ref = [], []
    for l, (r, n) in nobs.items():
        f_lm += [l] * n
        f_ref += [r] * n
    prob = dict(K=2, L=len(nobs), f_lm=np.array(f_lm), f_ref=np.array(f_ref))
    # reference 0 in id order 1, 3, 6: 60 | 70 + 1; reference 1: 100 + 20 | 9; then the landmark without factors
    assert lin_vis_runs(prob) == [60, 71, 120, 9, 0]


# ---------------------------------------------------------------------------------------------------------------------------------- windows
def _window(olib, name):
    kw = dict(WINDOWS[name])
    ext_const = kw.pop("ext_const", False)
    prob, _ = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), **kw)
    if ext_const:
        prob["ext_const"], prob["td_const"] = 1, 1
    return prob


def _eight_observation_window(olib):
    """K = 10, all landmarks anchored in node 0 and seen to the end of the window; landmarks with fewer than 8 observations dropped, the
    others cut to their first 8, and a multiple of 16 of them kept: every lin_vis run holds 16 landmarks, 128 factors."""
    prob, _ = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=10, L=400, seed=2040, n_ref=1, full_visibility=True)
    nobs = np.bincount(prob["f_lm"], minlength=prob["L"])
    keep = np.flatnonzero(nobs >= 8)
    keep = keep[:len(keep) // 16 * 16]
    new_id = np.full(prob["L"], -1)
    new_id[keep] = np.arange(len(keep))
    taken = np.zeros(prob["L"], int)
    fk = []
    for f, l in enumerate(prob["f_lm"]):
        if new_id[l] >= 0 and taken[l] < 8:
            fk.append(f)
            taken[l] += 1
    fk = np.array(fk)
    prob.update(L=len(keep), F=len(fk), invdepth=prob["invdepth"][keep].copy(), f_lm=new_id[prob["f_lm"][fk]].astype(np.int32),
                f_ref=prob["f_ref"][fk].copy(), f_obs=prob["f_obs"][fk].copy(),
                f_const=prob["f_const"].reshape(-1, 14)[fk].reshape(-1).copy(), f_active=np.ones(len(fk), np.uint8))
    return prob


# ---------------------------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def windows(olib):
    made = {}

    def get(name):
        if name not in made:
            made[name] = _window(olib, name)
        return copy.deepcopy(made[name])
    return get


@pytest.fixture(scope="module")
def handles():
    from ic_gvins_b200.ba import WindowSolver
    made = {}

    def get(max_K):
        if max_K not in made:
            made[max_K] = WindowSolver(max_K=max_K, max_gnss=16, max_marg_r=64, **HANDLES[max_K])
        return made[max_K]
    yield get
    for s in made.values():
        s.close()


def _assert_oracle_contract(sg, so, pg, po):
    assert sg["iterations"] == so["iterations"] and sg["num_successful_steps"] == so["num_successful_steps"], (sg, so)
    assert sg["termination"] == so["termination"]
    assert abs(sg["initial_cost"] - so["initial_cost"]) <= 1e-9 * so["initial_cost"]
    assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-7 * so["final_cost"]
    _compare_solution(pg, po)


def _increments(p, p0):
    """A step's parameter increments by group: positions, quaternions, velocities, gyro / accelerometer biases, inverse depths, extrinsic
    translation / rotation, time offset."""
    dp = (p["pose"] - p0["pose"]).reshape(-1, 7)
    dm = (p["mix"] - p0["mix"]).reshape(-1, 9)
    de = p["ext"] - p0["ext"]
    return dict(position=dp[:, :3], rotation=dp[:, 3:], velocity=dm[:, :3], gyro_bias=dm[:, 3:6], accel_bias=dm[:, 6:],
                invdepth=p["invdepth"] - p0["invdepth"], ext_translation=de[:3], ext_rotation=de[3:7], td=de[7:])


@pytest.mark.gpu
@pytest.mark.parametrize("max_K,name", POINTS, ids=_ids(POINTS))
def test_window_solve_matches_oracle(olib, windows, handles, max_K, name):
    """20 LM iterations: same trajectory as the oracle, solution within 1e-6 relative per group."""
    prob = windows(name)
    if name == "K32":   # the long-track case is really in the data
        assert 128 in lin_vis_runs(prob) and np.bincount(prob["f_lm"]).max() == prob["K"] - 1
    pg, po = copy.deepcopy(prob), copy.deepcopy(prob)
    so = oa.ba_solve(olib, po, 20)
    sg = handles(max_K).solve(pg, 20)[0]
    _assert_oracle_contract(sg, so, pg, po)


@pytest.mark.gpu
@pytest.mark.parametrize("max_K,name", POINTS, ids=_ids(POINTS))
def test_first_step_matches_oracle(olib, windows, handles, max_K, name):
    """One LM iteration, accepted: the parameter increments within 1e-9 relative of the oracle's, group by group.  Twenty iterations would
    correct a small error in one step; a single step shows it."""
    prob = windows(name)
    pg, po = copy.deepcopy(prob), copy.deepcopy(prob)
    so = oa.ba_solve(olib, po, 1)
    sg = handles(max_K).solve(pg, 1)[0]
    assert so["num_successful_steps"] == sg["num_successful_steps"] == 1 and sg["iterations"] == so["iterations"] == 1
    assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-7 * so["final_cost"]
    dg, do = _increments(pg, prob), _increments(po, prob)
    gaps = {}
    for group, ref in do.items():
        if ref.size == 0 or not np.any(ref):   # constant blocks stay put
            assert not np.any(dg[group]), group
            continue
        gaps[group] = rel_err(dg[group], ref)
    worst = max(gaps, key=gaps.get)
    print(f"first step {solve_kernel(max_K)} max_K={max_K} {name}: largest gap {gaps[worst]:.2e} ({worst})")
    assert gaps[worst] <= ONE_STEP_REL, gaps


@pytest.mark.gpu
@pytest.mark.parametrize("max_K", [14, 23, 32])
def test_mixed_size_batch_equals_single_windows(windows, handles, max_K):
    """All of a handle's windows, of different sizes, in one call == the same windows solved one at a time on that handle (bitwise)."""
    s = handles(max_K)
    probs = [windows(name) for name in SWEEP[max_K]]
    single, out_single = [], []
    for p in probs:
        q = copy.deepcopy(p)
        out_single.append(s.solve(q, 10)[0])
        single.append(q)
    batch = copy.deepcopy(probs)
    out_batch = s.solve(batch, 10)
    assert out_batch == out_single
    for a, b, name in zip(batch, single, SWEEP[max_K]):
        for key in ("pose", "mix", "invdepth", "ext"):
            assert np.array_equal(a[key], b[key]), (name, key)


@pytest.mark.gpu
@pytest.mark.parametrize("name,cap_a,cap_b", CAPACITY, ids=[f"{n}-maxK{a}-maxK{b}" for n, a, b in CAPACITY])
def test_solve_is_independent_of_the_capacity(olib, windows, handles, name, cap_a, cap_b):
    """The same window on two handles of one kernel whose max_K differ: capacities set strides and buffer sizes, never the order of a sum,
    so the results are bit-identical (and match the oracle)."""
    prob = windows(name)
    pa, pb, po = copy.deepcopy(prob), copy.deepcopy(prob), copy.deepcopy(prob)
    sa = handles(cap_a).solve(pa, 20)[0]
    sb = handles(cap_b).solve(pb, 20)[0]
    assert sa == sb
    for key in ("pose", "mix", "invdepth", "ext"):
        assert np.array_equal(pa[key], pb[key]), key
    _assert_oracle_contract(sa, oa.ba_solve(olib, po, 20), pa, po)


def _outliers(prob, fa, fb):
    fc = prob["f_const"].reshape(-1, 14)
    fc[fa, 3] += 0.2        # gross visual outliers
    fc[fb, 4] -= 0.15
    prob["gnss_blh"][3:6] += np.array([1.0, -0.8, 0.5])   # a GNSS outlier on the second fix


def _assert_two_pass_matches_oracle(olib, s, prob, fa, fb):
    _outliers(prob, fa, fb)
    pg, po = copy.deepcopy(prob), copy.deepcopy(prob)
    info = s.gvins_optimization_batch([pg], 20)[0]
    s1, s2, out = oracle_two_pass(olib, po)
    assert info["pass1"]["iterations"] == s1["iterations"] and info["pass2"]["iterations"] == s2["iterations"]
    assert info["reproj_removed"] == int(out.sum()) and out[fa] and out[fb]
    assert np.array_equal(pg["f_active"], po["f_active"])
    assert rel_err(pg["gnss_std"], po["gnss_std"]) <= 1e-9
    _compare_solution(pg, po)


@pytest.mark.gpu
def test_full_runs_on_the_production_handle(olib, handles):
    """max_K = 10: every landmark has exactly 8 observations, so every ba_lin_vis run fills its 128 record slots (every thread holds a
    record).  A 20-iteration solve and the two-pass gvinsOptimization protocol against the oracle."""
    prob = _eight_observation_window(olib)
    assert set(lin_vis_runs(prob)) == {128}
    s = handles(10)
    pg, po = copy.deepcopy(prob), copy.deepcopy(prob)
    so = oa.ba_solve(olib, po, 20)
    sg = s.solve(pg, 20)[0]
    _assert_oracle_contract(sg, so, pg, po)
    _assert_two_pass_matches_oracle(olib, s, prob, 10, 500)


@pytest.mark.gpu
def test_long_track_two_pass_matches_oracle(olib, windows, handles):
    """The two-pass gvinsOptimization protocol on the K = 32 long-track window (ba_solve_cam), with gross outliers."""
    _assert_two_pass_matches_oracle(olib, handles(32), windows("K32"), 10, 5000)
