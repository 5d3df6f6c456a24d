"""CPU: the high-precision assembly of a window's normal equations and reduced camera system (tests/lin_system_mp.py) against an
independent float64 dense J^T J and Schur elimination built from the oracle's factor evaluations, and the evidence that its bounds reject
the mistakes a linearisation or Schur kernel could plausibly make: each mutation below moves some entry by at least 100 times its bound.
Every mutation but one changes the reference's inputs (the factors it sums, their loss, the pair records, the damping, the parameters); a
6x6 off-diagonal block transposed is a mistake of the output's layout, so it is applied to the assembled H_c and Hs."""
import copy

import numpy as np
import pytest

from datagen import synth_ba
from tests import lin_system_mp as lm
from tests import oracle_api as oa
from tests.test_oracle_lm_step import dense_system

RADIUS0 = 1e4  # Ceres' initial_trust_region_radius: the radius of the first Schur complement
MUTATION_MARGIN = 100.0


@pytest.fixture(scope="module")
def olib(oracle):
    oa.declare_ba(oracle)
    return oracle


@pytest.fixture(scope="module")
def case(olib):
    """K = 4, 24 landmarks, pixel noise of 2 px (some factors above the Huber knee), factor 5 inactive"""
    prob = synth_ba.make_window(lambda *a: oa.preintegrate(olib, *a), K=4, L=24, seed=41, pixel_noise=2.0)[0]
    prob["f_active"][5] = 0
    vis, cam = lm.factors(prob)
    return prob, vis, cam, lm.assemble(prob, vis, cam, RADIUS0)


def dense_in_window_layout(olib, prob):
    """the oracle's dense (J, r) with columns permuted to [pose 6K | ext 6 | td 1 | mix 9K | rho L]"""
    K, L = prob["K"], prob["L"]
    r, J, _ = dense_system(olib, prob)
    perm = [15 * k + c for k in range(K) for c in range(6)] + list(range(15 * K, 15 * K + 7)) + \
           [15 * k + 6 + c for k in range(K) for c in range(9)] + list(range(15 * K + 7, 15 * K + 7 + L))
    return r, J[:, perm]


def test_assembly_matches_the_dense_float64_system(olib, case):
    prob, vis, cam, ref = case
    K = prob["K"]
    NCV, N = 6 * K + 7, 15 * K + 7
    r, J = dense_in_window_layout(olib, prob)
    H, g = J.T @ J, J.T @ r
    Hc, HcE = ref["H_c"]
    Hv, HvE = ref["H_vis"]
    worst = {}
    # the camera block: H_c + H_vis (both triangles)
    Hcam, HcamE = Hc.copy(), HcE + np.abs(Hc)
    Hcam[:NCV, :NCV] += Hv[:NCV, :NCV]
    HcamE[:NCV, :NCV] += HvE[:NCV, :NCV] + np.abs(Hv[:NCV, :NCV])
    worst["H"] = lm.ratio(H[:N, :N], Hcam, HcamE, 1.0)
    # the landmark terms and coupling rows
    worst["h_l"] = lm.ratio(np.diag(H)[N:], *ref["h_l"], 1.0)
    worst["A_W"] = lm.ratio(H[N:, :NCV], ref["A_W"][0][:, :NCV], ref["A_W"][1][:, :NCV], 1.0)
    worst["g_l"] = lm.ratio(g[N:], *ref["g_l"], 1.0)
    # the gradient: g_c + g_vis
    gv, gvE = np.zeros(N), np.zeros(N)
    gv[:NCV], gvE[:NCV] = Hv[:NCV, NCV], HvE[:NCV, NCV]
    gc, gcE = ref["g_c"]
    worst["g"] = lm.ratio(g[:N], gc + gv, gcE + gvE + np.abs(gc + gv), 1.0)
    # the reduced camera system (vision rows): dense Schur elimination with the float64 phi
    hl = np.diag(H)[N:]
    s = 1.0 / (1.0 + np.sqrt(hl))
    hs = s * s * hl
    phi = s * s / (hs + np.clip(hs, lm.MIN_DIAG, lm.MAX_DIAG) / RADIUS0)
    W = H[N:, :NCV]
    Hs_dense = H[:NCV, :NCV] - W.T @ (phi[:, None] * W)
    worst["Hs"] = lm.ratio(np.tril(Hs_dense), *ref["Hs"], 1.0)
    print("dense float64 against the assembly, worst error / bound:", {k: f"{v:.2e}" for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


def separation(mut, ref):
    """the largest |mutated - reference| / (c eps bound) over every array of the system"""
    out = 0.0
    for name, entry in ref.items():
        if name in ("phi", "H_vis"):
            continue
        val, bnd = (entry, None) if isinstance(entry, dict) else entry
        if name == "Mp":
            for k in set(val) | set(mut[name]):
                if k not in val or k not in mut[name]:
                    return float("inf")
                out = max(out, lm.ratio(mut[name][k][0], *val[k], 1.0))
        elif name == "costf":
            out = max(out, max(lm.ratio(mut[name][f][0], *val[f], 1.0) for f in set(val) & set(mut[name])))
        else:
            out = max(out, lm.ratio(mut[name][0], val, bnd, 1.0))
    return out


def test_mutations_break_the_bound(olib, case):
    prob, vis, cam, ref = case
    inactive = int(np.flatnonzero(prob["f_active"] == 0)[0])
    above = [v for v in vis if v.sq > 1.0]
    assert above, "the window must have a factor above the Huber knee"
    key = (vis[0].ref, vis[0].obs)
    other = next(v for v in vis if v.ref != key[0])  # a record of another reference node's run
    muts = {
        "one factor dropped": lambda: lm.assemble(prob, vis[1:], cam, RADIUS0),
        "an inactive factor counted": lambda: lm.assemble(prob, vis + [lm.vis_factor(prob, inactive)], cam, RADIUS0),
        "Huber scaling skipped on one factor": lambda: lm.assemble(
            prob, [lm.vis_factor(prob, v.f, huber=False) if v is above[0] else v for v in vis], cam, RADIUS0),
        "one Gram partial counted twice": lambda: lm.assemble(prob, vis, cam, RADIUS0, dup_rows=key),
        "one Gram partial from the wrong run": lambda: lm.assemble(prob, vis, cam, RADIUS0, wrong_rows=(key, other)),
        "D_l^2 omitted": lambda: lm.assemble(prob, vis, cam, RADIUS0, no_d2=True),
        "the other linearisation buffer's parameters": lambda: _at_candidate(olib, prob),
    }
    seps = {}
    for why, make in muts.items():
        seps[why] = separation(make(), ref)
    # a 6x6 off-diagonal block transposed: (pose 0, pose 1) of H_c and of Hs (IMU factor 0 couples them)
    for name in ("H_c", "Hs"):
        val = ref[name][0].copy()
        b = val[6:12, 0:6].copy()
        val[6:12, 0:6] = b.T
        if name == "H_c":
            val[0:6, 6:12] = b
        seps[f"{name} block (pose 1, pose 0) transposed"] = lm.ratio(val, *ref[name], 1.0)
    print("mutation / bound:", {k: f"{v:.1e}" for k, v in seps.items()})
    assert all(s >= MUTATION_MARGIN for s in seps.values()), seps


def _at_candidate(olib, prob):
    """the system at the parameters one oracle LM step away (what the other linearisation buffer holds after a step)"""
    p = copy.deepcopy(prob)
    s = oa.ba_solve(olib, p, 1)
    assert s["num_successful_steps"] == 1
    vis, cam = lm.factors(p)
    return lm.assemble(p, vis, cam, RADIUS0)
