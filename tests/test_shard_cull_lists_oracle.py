"""CPU: the list rule of icg_ba_shard_update_and_cull_built.  Over seeded keyframe sequences at world 2 and 3, each rank's next culling lists
-- the list rule (tests/cull_lists_oracle.next_lists) applied to the rank's own old shard lists and its own next shard (the per-rank vision
restatement, tests/shard_vision_oracle.build_rank) -- must equal the rank's cut of the whole window's lists: the landmarks shard_next puts on
the rank, their entries in order, factor ids renumbered to the rank's shard."""
import numpy as np
import pytest

from tests import shard_vision_oracle as sv
from tests import slide_vision_oracle as so
from tests.cull_lists_oracle import next_lists
from tests.test_shard_vision_oracle import CAM, K, split, window

LISTS = ("lm_ref_node", "obs_off", "obs_node", "obs_factor", "lm_ref_kp", "obs_kp")


def onode_of(node_src, vis, oK):
    onode = np.full(oK, -1)
    for j, i in enumerate(node_src):
        if vis["num_marg"] <= i < oK and vis["node_in_map"][i]:
            onode[i] = j
    return onode


def points(vis):
    return [dict(ref_node=vis["frames"][p["ref_id"]], ref_xy=p["ref_xy"], cur_xy=p["cur_xy"]) for p in vis["new"]]


def cut(lists, lms, fmap):
    """the lists of landmarks lms (in that order) of `lists`, factor f renumbered to fmap[f] (-1 stays -1)"""
    off = lists["obs_off"]
    idx = np.concatenate([np.arange(off[l], off[l + 1]) for l in lms]).astype(np.int64) if len(lms) else np.zeros(0, np.int64)
    f = lists["obs_factor"][idx]
    n = np.array([off[l + 1] - off[l] for l in lms], np.int64)
    return dict(n_obs=len(idx), lm_ref_node=lists["lm_ref_node"][lms].astype(np.int32), lm_ref_kp=lists["lm_ref_kp"][lms].reshape(-1, 2),
                obs_off=np.r_[0, np.cumsum(n)].astype(np.int32), obs_node=lists["obs_node"][idx].astype(np.int32),
                obs_factor=np.where(f >= 0, fmap[np.maximum(f, 0)], -1).astype(np.int32), obs_kp=lists["obs_kp"][idx].reshape(-1, 2))


def keyframe(old, cull, prev, node_src, vis, w, rng):
    """one keyframe: the whole window's next lists cut per rank against each rank's own rule.  Returns the next whole window in rank-major order
    (with its reference rows), its shards and its culling (the whole next lists with fresh flags)"""
    from ic_gvins_b200.ba import shard_next
    world = len(prev)
    whole = so.build(old, cull, node_src, vis, CAM)
    onode = onode_of(node_src, vis, old["K"])
    cur = vis["cur_node"]
    xy = {(l, nd): p for l, nd, p, _ in vis["obs"] if l >= 0}
    wl = next_lists(cull, cull["obs_outlier"], onode, whole, xy, points(vis), cur)
    nxt = dict(old, L=whole["L"], F=whole["F"], invdepth=whole["invdepth"], f_lm=whole["f_lm"], f_ref=whole["f_ref"], f_obs=whole["f_obs"],
               f_const=whole["f_const"].reshape(-1), f_active=np.ones(whole["F"], np.uint8))
    wr, _, parts = shard_next(nxt, dict(node_src=np.array(node_src, np.int32), lm_src=whole["lm_src"], f_src=whole["f_src"]), prev,
                              sv.new_rank(whole, prev, w))
    order = sv.rank_order(whole, prev, w)
    new_of = np.empty(whole["L"], np.int64)
    new_of[order] = np.arange(whole["L"])
    pos = np.empty(whole["F"], np.int64)  # whole factor -> its row in the rank-major window
    pos[np.argsort(new_of[whole["f_lm"]], kind="stable")] = np.arange(whole["F"])
    got = []
    for r in range(world):
        sh = prev[r]
        lo, hi = int(sh["lm_lo"]), int(sh["lm_hi"])
        sc = sv.shard_cull(cull, sh)
        rb = sv.build_rank(dict(sh, lm_ref=old["lm_ref"][lo:hi]), sc, node_src, dict(vis, obs=sv.shard_obs(vis["obs"], sh)), CAM, r, world, w)
        rl = next_lists(sc, sc["obs_outlier"], onode, rb, {(l - lo, nd): p for (l, nd), p in xy.items() if lo <= l < hi}, points(vis), cur)
        part = parts[r][0]
        local = np.full(max(1, whole["F"]), -1, np.int64)
        local[part["f_index"]] = np.arange(len(part["f_index"]))
        want = cut(wl, order[part["lm_lo"]:part["lm_hi"]], local[pos] if whole["F"] else local)
        assert rl["n_obs"] == want["n_obs"] and len(rl["lm_ref_node"]) == rb["L"], r
        for k in LISTS:
            assert np.asarray(rl[k]).tobytes() == np.asarray(want[k]).tobytes(), (r, k)
        got.append(rl)
    # the next keyframe's culling: the whole lists in rank-major order, flags drawn afresh
    lists = cut(wl, order, pos if whole["F"] else np.zeros(1, np.int64))
    lists.update(lm_outlier=(rng.random(whole["L"]) < 0.08).astype(np.uint8), obs_outlier=(rng.random(lists["n_obs"]) < 0.1).astype(np.uint8))
    wr["lm_ref"] = whole["lm_ref"][order]
    return wr, [p[0] for p in parts], lists, got, whole


def next_vis(rng, L, n_new):
    """the new keyframe's observations of a window of L landmarks (tests/test_shard_vision_oracle.window's shape)"""
    cur = K - 1
    obs = []
    for nd in (cur - 1, cur):
        for l in rng.choice(L, size=min(L, 5), replace=False):
            obs.append((int(l), nd, rng.uniform(100, 500, 2).astype(np.float32), rng.normal(0, 5, 2)))
        obs.append((-1, nd, np.float32([320, 240]), (0.0, 0.0)))
    new = [dict(depth=float(rng.uniform(2, 40)), ref_xy=rng.uniform(100, 500, 2).astype(np.float32), vel_ref=rng.normal(0, 5, 2),
                ref_id=100 + (cur - j % 3), cur_xy=rng.uniform(100, 500, 2).astype(np.float32), vel_cur=rng.normal(0, 5, 2)) for j in range(n_new)]
    return dict(num_marg=1, node_in_map=np.ones(K, np.uint8), node_td=rng.normal(0, 1e-3, K), cur_node=cur, frames={100 + k: k for k in range(K)},
                obs=obs, new=new)


def sequence(seed, world, L, bounds=None, n_kf=3, zero=(), n_new=6, all_dropped=()):
    """n_kf keyframes from a seeded window; the old window's keypoints are random, landmarks all_dropped have every factor flagged"""
    rng = np.random.default_rng(seed)
    old, cull, ns, vis = window(seed, L, zero=zero, n_new=n_new)
    cull["lm_ref_kp"] = rng.uniform(0, 640, (L, 2)).astype(np.float32)
    cull["obs_kp"] = rng.uniform(0, 640, (len(cull["obs_node"]), 2)).astype(np.float32)
    for l in all_dropped:
        o0, o1 = cull["obs_off"][l], cull["obs_off"][l + 1]
        cull["obs_outlier"][o0:o1] = cull["obs_factor"][o0:o1] >= 0
        cull["lm_ref_node"][l], cull["lm_outlier"][l] = 2, 0
    old["lm_ref"] = so.reference_rows(old)
    prev = split(old, bounds if bounds is not None else [L * r // world for r in range(world + 1)])
    out = []
    for c in range(n_kf):
        w = (seed + c) % (2 * world)
        old, prev, cull, got, whole = keyframe(old, cull, prev, ns, vis, w, rng)
        out.append((got, whole))
        vis = next_vis(rng, old["L"], n_new)
    return out


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("seed", [4000, 4001, 4002])
def test_rank_lists_are_the_shard_cut_of_the_whole_lists(world, seed):
    for got, whole in sequence(seed, world, 40):
        assert sum(len(g["lm_ref_node"]) for g in got) == whole["L"]
        assert sum((g["obs_factor"] >= 0).sum() for g in got) > 0


@pytest.mark.parametrize("world", [2, 3])
def test_empty_old_shard(world):
    """rank 0 holds no landmark of the first old window: its first lists are its new points' only"""
    got, _ = sequence(4100 + world, world, 30, bounds=[0, 0] + [30 * r // (world - 1) for r in range(1, world)], n_kf=2)[0]
    assert len(got[0]["lm_ref_node"]) > 0 and (got[0]["obs_factor"][got[0]["obs_node"] != K - 1] == -1).all()


@pytest.mark.parametrize("world", [2, 3])
def test_rank_without_new_points(world):
    """one new point per keyframe: every other rank lists only its carried landmarks"""
    for got, whole in sequence(4200 + world, world, 36, n_new=1):
        assert sum(len(g["lm_ref_node"]) for g in got) == whole["L"]
        assert sum(len(g["lm_ref_node"]) > 0 for g in got) == world  # a rank without a new point still lists its carried landmarks


@pytest.mark.parametrize("world", [2, 3])
def test_zero_depth_carried_landmark(world):
    """a carried landmark staged for a zero inverse depth keeps its list on its own rank"""
    L = 36
    (got, whole), *_ = sequence(4300 + world, world, L, zero=[L - 2, L // 2, 7])
    staged = (whole["lm_src"] < 0) & (whole["lm_origin"] >= 0)
    assert staged.sum() >= 2


@pytest.mark.parametrize("world", [2, 3])
def test_landmark_whose_factors_were_all_dropped(world):
    """every factor of landmarks 5 and 30 flagged: each is carried with its reference observation alone (plus any new one)"""
    L = 36
    (got, whole), *_ = sequence(4400 + world, world, L, all_dropped=[5, 30])
    for l in (5, 30):
        li = int(np.nonzero(whole["lm_origin"] == l)[0][0])
        assert not (whole["f_src"][whole["f_lm"] == li] >= 0).any()
