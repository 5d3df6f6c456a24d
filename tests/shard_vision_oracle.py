"""numpy restatement of icg_ba_shard_slide_vision_resident on one rank: the rules of slide_vision_oracle.build on the rank's old shard, then the
new-point rule (new map point j of window w lives on rank (j + w) % world).  new_rank() gives the rank of every landmark of a whole-window build,
so that shard_next of that build is what the ranks build on their own."""
import numpy as np

from tests import slide_vision_oracle as so


def build_rank(old, cull, node_src, vis, cam, rank, world, w):
    """old / cull: the rank's old shard and its culling (shard-local f_lm and obs_factor); vis as so.build takes it, with every observation's
    landmark shard-local (-1 for a point the rank does not hold) and every new map point.  Returns so.build's dict for the rank's next shard:
    its carried landmarks, then its own new points; lm_origin -(j + 1) with the global creation index j; nan_flags old shard L + every new
    point, set for a new point on its own rank only."""
    r = so.build(old, cull, node_src, vis, cam)
    org = r["lm_origin"]
    keep = (org >= 0) | ((-org - 1 + w) % world == rank)
    new_of = np.cumsum(keep) - 1
    fk = keep[r["f_lm"]]
    flags = r["nan_flags"].copy()
    j = np.arange(len(vis["new"]))
    flags[old["L"]:][(j + w) % world != rank] = 0
    return dict(r, L=int(keep.sum()), F=int(fk.sum()), lm_src=r["lm_src"][keep], lm_origin=org[keep], lm_ref=r["lm_ref"][keep],
                invdepth=r["invdepth"][keep], f_lm=new_of[r["f_lm"][fk]].astype(np.int32), f_ref=r["f_ref"][fk], f_obs=r["f_obs"][fk],
                f_src=r["f_src"][fk], f_const=r["f_const"][fk], nan_flags=flags, nan_dropped=int(flags.sum()))


def new_rank(built, prev_shards, w):
    """shard_next's new_rank for a whole-window build: -1 for a carried landmark, the old rank for one staged for a zero depth (lm_src -1,
    lm_origin >= 0), (j + w) % world for new map point j"""
    world = len(prev_shards)
    old_rank = np.zeros(max(1, max(int(s["lm_hi"]) for s in prev_shards)), np.int64)
    for r, s in enumerate(prev_shards):
        old_rank[s["lm_lo"]:s["lm_hi"]] = r
    org = np.asarray(built["lm_origin"], np.int64)
    return np.where(built["lm_src"] >= 0, -1, np.where(org >= 0, old_rank[np.maximum(org, 0)], (-org - 1 + w) % world))


def rank_order(built, prev_shards, w):
    """the permutation that writes a whole-window build rank-major, as shard_next does (next's order within a rank)"""
    rank = new_rank(built, prev_shards, w)
    src = np.asarray(built["lm_src"])
    for r, s in enumerate(prev_shards):
        rank[(src >= s["lm_lo"]) & (src < s["lm_hi"])] = r
    return np.argsort(rank, kind="stable")


def shard_obs(obs, shard):
    """so.build's observation list with its landmarks remapped to the shard's old rows (-1 outside [lm_lo, lm_hi))"""
    lo, hi = int(shard["lm_lo"]), int(shard["lm_hi"])
    return [(l - lo if lo <= l < hi else -1, node, xy, vel) for l, node, xy, vel in obs]


def shard_cull(cull, shard):
    """so.build's culling dict of one shard of the whole window's (shard_cull_inputs' lists plus the shard's slices of the two flag arrays)"""
    from ic_gvins_b200.ba import shard_cull_inputs
    lo, hi = int(shard["lm_lo"]), int(shard["lm_hi"])
    off = np.asarray(cull["obs_off"])
    out = shard_cull_inputs(cull, shard)
    out.update(lm_outlier=np.asarray(cull["lm_outlier"])[lo:hi], obs_outlier=np.asarray(cull["obs_outlier"])[off[lo]:off[hi]])
    return out
