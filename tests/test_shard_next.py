"""CPU: shard_next, the per-rank shard slides of a whole-window slide, on a hand-made window: carried landmarks stay on their rank, the next
window is rank-major with its factors landmark by landmark, and every shard's carry maps name rows of the same rank's old shard."""
import numpy as np
import pytest

from ic_gvins_b200.ba import shard_next, shard_window


def window(L, f_lm, f_ref, f_obs, base):
    F = len(f_lm)
    return dict(L=L, F=F, K=4, imu_blob=np.arange(3 * 480, dtype=np.float64), invdepth=base + np.arange(L, dtype=np.float64),
                f_lm=np.array(f_lm, np.int32), f_ref=np.array(f_ref, np.int32), f_obs=np.array(f_obs, np.int32), f_const=(base + np.arange(14 * F, dtype=np.float64)), f_active=np.ones(F, np.uint8),
                pose=np.zeros(28), mix=np.zeros(36), ext=np.zeros(8), gnss_std=np.zeros(3))


def case():
    old = window(6, [0, 0, 1, 2, 3, 3, 4, 5], [0, 0, 1, 1, 0, 0, 2, 2], [1, 2, 2, 3, 1, 2, 3, 3], 100.0)
    prev = [shard_window(old, r, 2) for r in range(2)]  # rank 0: landmarks 0-2 (factors 0-3), rank 1: 3-5 (factors 4-7)
    # next: l0 = old 4 (rank 1), l1 new, l2 = old 1 (rank 0), l3 new, l4 = old 0 (rank 0); factors shuffled, two of them new
    nxt = window(5, [2, 0, 4, 1, 3, 4, 2], [0, 1, 0, 2, 2, 0, 0], [1, 2, 1, 3, 3, 2, 2], 200.0)
    carry = dict(node_src=np.arange(4, dtype=np.int32), lm_src=np.array([4, -1, 1, -1, 0], np.int32),
                 f_src=np.array([2, 6, 0, -1, -1, 1, -1], np.int32))
    return old, prev, nxt, carry


def test_rank_major_order_and_shard_local_maps():
    old, prev, nxt, carry = case()
    whole, wcarry, parts = shard_next(nxt, carry, prev, np.array([-1, 0, -1, 1, -1]))
    order = [1, 2, 4, 0, 3]  # rank 0: l1 (new), l2, l4; rank 1: l0, l3 (new)
    assert np.array_equal(whole["invdepth"], nxt["invdepth"][order])
    assert (np.diff(whole["f_lm"]) >= 0).all()
    assert np.array_equal(wcarry["lm_src"], carry["lm_src"][order])
    # the factors of each landmark keep next's order; every factor keeps its row values
    new_of = np.argsort(order)
    for f in range(whole["F"]):
        src = [g for g in range(nxt["F"]) if new_of[nxt["f_lm"][g]] == whole["f_lm"][f]]
        assert any(np.array_equal(whole["f_const"].reshape(-1, 14)[f], nxt["f_const"].reshape(-1, 14)[g]) for g in src)
    (s0, c0), (s1, c1) = parts
    assert (s0["lm_lo"], s0["lm_hi"], s1["lm_lo"], s1["lm_hi"]) == (0, 3, 3, 5)
    assert np.array_equal(c0["lm_src"], [-1, 1, 0]) and np.array_equal(c1["lm_src"], [1, -1])  # old 4 is rank 1's landmark 1
    for (sh, sc), pv in zip(parts, prev):
        assert (np.diff(sh["f_lm"]) >= 0).all()
        assert np.array_equal(sh["invdepth"], whole["invdepth"][sh["lm_lo"]:sh["lm_hi"]])
        assert np.array_equal(sh["f_const"].reshape(-1, 14), whole["f_const"].reshape(-1, 14)[sh["f_index"]])
        for f in range(sh["F"]):  # a carried factor names the same factor of the same rank's old shard
            g = wcarry["f_src"][sh["f_index"][f]]
            assert (sc["f_src"][f] < 0) == (g < 0)
            if g >= 0:
                assert pv["f_index"][sc["f_src"][f]] == g
                assert pv["f_lm"][sc["f_src"][f]] + pv["lm_lo"] == carry["lm_src"][order][sh["f_lm"][f] + sh["lm_lo"]]
        assert np.array_equal(sc["node_src"], carry["node_src"])
    for k in ("pose", "mix", "imu_blob", "invdepth", "f_const"):  # every shard owns its arrays
        assert all(not np.shares_memory(s0[k], x[k]) for x in (s1, whole)), k


def test_every_new_landmark_on_one_rank_and_an_empty_shard():
    old, prev, nxt, carry = case()
    carry = dict(carry, lm_src=np.array([-1, -1, 1, -1, 0], np.int32), f_src=np.array([2, -1, 0, -1, -1, 1, -1], np.int32))
    _, _, parts = shard_next(nxt, carry, prev, np.array([0, 0, -1, 0, -1]))
    assert parts[0][0]["L"] == 5 and parts[1][0]["L"] == 0 and parts[1][0]["F"] == 0


def test_rank_change_is_rejected():
    old, prev, nxt, carry = case()
    with pytest.raises(ValueError, match="carried from rank 1"):
        shard_next(nxt, carry, prev, np.array([0, 0, -1, 1, -1]))
