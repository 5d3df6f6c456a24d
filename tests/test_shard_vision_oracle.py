"""CPU: the per-rank restatement of the sharded vision slide (tests/shard_vision_oracle.py) against shard_next of the whole-window restatement
(tests/slide_vision_oracle.py): every rank's next shard, built from its own old shard, culling and shard-local observations plus the new-point
rule, must be exactly the rank's part of the whole window reordered rank-major."""
import numpy as np
import pytest

from tests import shard_vision_oracle as sv
from tests import slide_vision_oracle as so

CAM = dict(fx=400.0, fy=400.0, cx=320.0, cy=240.0, skew=0.0)
K = 6


def window(seed, L, zero=(), nan=(), n_new=6):
    """a whole old window of K nodes (node 0 leaves, one node arrives), its culling and the new keyframe's observations: two tracked nodes,
    unknown points, and new map points anchored in three nodes (one in the current node: no factor)"""
    rng = np.random.default_rng(seed)
    ref = rng.integers(1, K - 1, L)
    ref[: max(1, L // 6)] = 0  # anchored in the marginalized node: dropped
    f_lm, f_ref, f_obs = [], [], []
    for l in range(L):
        for k in sorted(rng.choice([k for k in range(K) if k != ref[l]], size=int(rng.integers(1, 4)), replace=False)):
            f_lm.append(l), f_ref.append(ref[l]), f_obs.append(k)
    F = len(f_lm)
    fc = rng.normal(0, 1, (F, 14))
    invd = rng.uniform(0.05, 1.0, L)
    invd[list(zero)], invd[list(nan)] = 0.0, np.nan
    old = dict(K=K, L=L, F=F, invdepth=invd, f_lm=np.array(f_lm, np.int32), f_ref=np.array(f_ref, np.int32), f_obs=np.array(f_obs, np.int32),
               f_const=fc.reshape(-1), f_active=np.ones(F, np.uint8), pose=np.zeros(7 * K), mix=np.zeros(9 * K), ext=np.zeros(8), gnss_std=np.zeros(3))
    off, node, fac = [0], [], []
    for l in range(L):
        obs = [(int(ref[l]), -1)] + [(int(f_obs[f]), f) for f in range(F) if f_lm[f] == l]
        for i in rng.permutation(len(obs)):
            node.append(obs[i][0]), fac.append(obs[i][1])
        off.append(len(node))
    no = len(node)
    lm_out = (rng.random(L) < 0.1).astype(np.uint8)
    lm_out[list(zero) + list(nan)] = 0
    cull = dict(lm_ref_node=ref.astype(np.int32), lm_ref_kp=np.zeros((L, 2), np.float32), obs_off=np.array(off, np.int32),
                obs_node=np.array(node, np.int32), obs_kp=np.zeros((no, 2), np.float32), obs_factor=np.array(fac, np.int32), lm_outlier=lm_out,
                obs_outlier=(rng.random(no) < 0.1).astype(np.uint8))
    cur = K - 1
    obs = []
    for nd in (cur - 1, cur):  # next node cur - 1 is old node K - 1
        for l in rng.choice(L, size=min(L, 5), replace=False):
            obs.append((int(l), nd, rng.uniform(100, 500, 2).astype(np.float32), rng.normal(0, 5, 2)))
        obs.append((-1, nd, np.float32([320, 240]), (0.0, 0.0)))
    new = [dict(depth=float(rng.uniform(2, 40)) if j != 3 else np.nan, ref_xy=rng.uniform(100, 500, 2).astype(np.float32), vel_ref=rng.normal(0, 5, 2),
                ref_id=100 + (cur - j % 3), cur_xy=rng.uniform(100, 500, 2).astype(np.float32), vel_cur=rng.normal(0, 5, 2)) for j in range(n_new)]
    vis = dict(num_marg=1, node_in_map=np.ones(K, np.uint8), node_td=rng.normal(0, 1e-3, K), cur_node=cur, frames={100 + k: k for k in range(K)},
               obs=obs, new=new)
    node_src = list(range(1, K)) + [-1]
    return old, cull, node_src, vis


def split(prob, bounds):
    """the shards of `prob` over the landmark ranges bounds[r] .. bounds[r + 1] (shard_window's dicts, at any bounds)"""
    from ic_gvins_b200.ba import shard_window
    f_lm = np.asarray(prob["f_lm"])
    out = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        s = shard_window(prob, 0, 1)
        sel = np.nonzero((f_lm >= lo) & (f_lm < hi))[0]
        s.update(L=hi - lo, F=len(sel), invdepth=prob["invdepth"][lo:hi].copy(), f_lm=(f_lm[sel] - lo).astype(np.int32), f_ref=prob["f_ref"][sel],
                 f_obs=prob["f_obs"][sel], f_const=prob["f_const"].reshape(-1, 14)[sel].reshape(-1).copy(), f_active=prob["f_active"][sel], lm_lo=lo,
                 lm_hi=hi, f_index=sel)
        out.append(s)
    return out


def check(old, cull, node_src, vis, bounds, w):
    from ic_gvins_b200.ba import shard_next
    world = len(bounds) - 1
    prev = split(old, bounds)
    whole = so.build(old, cull, node_src, vis, CAM)
    nxt = dict(old, L=whole["L"], F=whole["F"], invdepth=whole["invdepth"], f_lm=whole["f_lm"], f_ref=whole["f_ref"], f_obs=whole["f_obs"],
               f_const=whole["f_const"].reshape(-1), f_active=np.ones(whole["F"], np.uint8))
    nr = sv.new_rank(whole, prev, w)
    _, wcarry, parts = shard_next(nxt, dict(node_src=np.array(node_src, np.int32), lm_src=whole["lm_src"], f_src=whole["f_src"]), prev, nr)
    origins, flags_new = [], np.zeros(len(vis["new"]), np.uint8)
    for r in range(world):
        sh, sc = parts[r]
        b = sv.build_rank(prev[r], sv.shard_cull(cull, prev[r]), node_src, dict(vis, obs=sv.shard_obs(vis["obs"], prev[r])), CAM, r, world, w)
        assert (b["L"], b["F"]) == (sh["L"], sh["F"]), r
        for k in ("invdepth", "f_lm", "f_ref", "f_obs"):
            assert np.array_equal(b[k], sh[k]), (r, k)
        assert np.array_equal(b["f_const"].reshape(-1), sh["f_const"]), r
        assert np.array_equal(b["lm_src"], sc["lm_src"]) and np.array_equal(b["f_src"], sc["f_src"]), r
        lo = prev[r]["lm_lo"]
        origins.append(np.where(b["lm_origin"] >= 0, b["lm_origin"] + lo, b["lm_origin"]))
        assert np.array_equal(b["nan_flags"][:prev[r]["L"]], whole["nan_flags"][lo:prev[r]["lm_hi"]]), r
        assert not (flags_new & b["nan_flags"][prev[r]["L"]:]).any(), r  # a new point is flagged on one rank only
        flags_new |= b["nan_flags"][prev[r]["L"]:]
    assert np.array_equal(flags_new, whole["nan_flags"][old["L"]:])
    order = sv.rank_order(whole, prev, w)
    assert np.array_equal(np.concatenate(origins), whole["lm_origin"][order])
    assert sum(p[0]["L"] for p in parts) == whole["L"] and np.array_equal(wcarry["lm_src"], whole["lm_src"][order])
    return whole, parts


@pytest.mark.parametrize("world", [2, 3])
def test_ranks_build_shard_next_of_the_whole_window(world):
    for w in range(2 * world):
        old, cull, ns, vis = window(3000 + w, 40)
        whole, parts = check(old, cull, ns, vis, [40 * r // world for r in range(world + 1)], w)
        assert (whole["lm_origin"] < 0).sum() >= 3 and whole["nan_flags"][old["L"]:].any()
        assert (whole["f_src"] < 0).sum() > (whole["lm_origin"] < 0).sum()  # tracked observations of carried landmarks


@pytest.mark.parametrize("world", [2, 3])
def test_rank_with_an_empty_old_shard(world):
    """rank 0 held no landmark: its next shard holds only its new points"""
    old, cull, ns, vis = window(3100 + world, 30)
    whole, parts = check(old, cull, ns, vis, [0, 0] + [30 * r // (world - 1) for r in range(1, world)], 1)
    assert parts[0][0]["L"] > 0 and (parts[0][1]["lm_src"] < 0).all()


@pytest.mark.parametrize("world", [2, 3])
def test_window_without_new_points(world):
    old, cull, ns, vis = window(3200 + world, 36, n_new=0)
    whole, parts = check(old, cull, ns, vis, [36 * r // world for r in range(world + 1)], 0)
    assert (whole["lm_origin"] >= 0).all()


@pytest.mark.parametrize("world", [2, 3])
def test_zero_depth_carried_landmark_stays_on_its_rank(world):
    """a zero inverse depth stages the landmark as a new row (lm_src -1) on the rank that held it; a NaN one is dropped and flagged there"""
    L = 36
    zero = [L - 2, L // 2, 7]
    old, cull, ns, vis = window(3300 + world, L, zero=zero, nan=[L - 5])
    whole, parts = check(old, cull, ns, vis, [L * r // world for r in range(world + 1)], 1)
    staged = np.nonzero((whole["lm_src"] < 0) & (whole["lm_origin"] >= 0))[0]
    assert len(staged) >= 2 and (whole["invdepth"][staged] == so.DEFAULT_INVDEPTH).all()
    assert whole["nan_flags"][L - 5] == 1
