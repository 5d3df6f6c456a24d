"""The next sliding window of a solved window, with the maps icg_ba_slide_resident takes (which rows of the next window carry over from
the old one): shared by tests/test_slide_gpu.py and scripts/bench_slide.py."""
import copy

import numpy as np

IMU = 480


def build_next(p, seed, *, drop=(0,), n_new=1, drop_lm=(), drop_f=(), n_reanchor=1, n_new_lm=3, prior=None, keep_prior=False):
    """The next window of `p` (the window as the last solve left it on the host: optimised parameters, re-weighted gnss_std, reintegrated
    blobs) and its carry maps.  Nodes `drop` leave (the IMU factors around a middle one merge into a new blob), `n_new` nodes arrive with an
    IMU factor and a GNSS fix each; landmarks `drop_lm`, those anchored in a dropped node and factors `drop_f` leave; `n_reanchor` landmarks
    come back as new ones (new inverse depth, their factors new); `n_new_lm` new landmarks observe the newest node.  The prior is `prior` (a
    marginalize() result), p's own (keep_prior) or none.  Factor rows are shuffled.  Returns (upload twin with every value filled in, the
    same window with NaN in every carried value row, carry)."""
    rng = np.random.default_rng(seed)
    K, L = p["K"], p["L"]
    pose, mix = p["pose"].reshape(K, 7), p["mix"].reshape(K, 9)
    kept = [k for k in range(K) if k not in drop]
    node_src = np.array(kept + [-1] * n_new, np.int32)
    K2 = len(node_src)
    new_of = {k: i for i, k in enumerate(kept)}
    pose2 = np.concatenate([pose[kept]] + [(pose[kept[-1]] + np.r_[0.4 * (j + 1), 0, 0, 0, 0, 0, 0])[None] for j in range(n_new)]).reshape(-1)
    mix2 = np.concatenate([mix[kept]] + [mix[kept[-1]][None]] * n_new).reshape(-1)
    blobs = p["imu_blob"].reshape(-1, IMU)
    imu_src, blob2 = [], []
    for j in range(K2 - 1):
        a, b = node_src[j], node_src[j + 1]
        if a >= 0 and b == a + 1 and a < p["n_imu"]:
            imu_src.append(a)
            blob2.append(blobs[a])
        else:  # a merged factor or one that joins a new node: a new blob (any valid one)
            imu_src.append(-1)
            blob2.append(blobs[min(max(a, 0), p["n_imu"] - 1)] if a < 0 or a >= p["n_imu"] else blobs[a])
    gn, blh, gstd = p["gnss_node"], p["gnss_blh"].reshape(-1, 3), p["gnss_std"].reshape(-1, 3)
    gsel = [g for g in range(p["n_gnss"]) if gn[g] in new_of]
    gnss_src = gsel + [-1] * n_new
    gnode2 = [new_of[gn[g]] for g in gsel] + [len(kept) + j for j in range(n_new)]
    blh2 = np.concatenate([blh[gsel]] + [blh[gsel[-1] if gsel else 0][None] + 1e-6 * (j + 1) for j in range(n_new)])
    gstd2 = np.concatenate([gstd[gsel]] + [np.array([[0.5, 0.5, 1.0]])] * n_new)
    f_lm, f_ref, f_obs, fc = p["f_lm"], p["f_ref"], p["f_obs"], p["f_const"].reshape(-1, 14)
    refof = np.full(L, -1)
    refof[f_lm] = f_ref
    lm_keep = [l for l in range(L) if l not in set(drop_lm) and (refof[l] < 0 or refof[l] in new_of)]
    with_f = [l for l in lm_keep if refof[l] >= 0]
    reanchor = set(rng.choice(with_f, size=min(n_reanchor, len(with_f)), replace=False).tolist()) if n_reanchor else set()
    lm_new_of = {l: i for i, l in enumerate(lm_keep)}
    lm_src = [-1 if l in reanchor else l for l in lm_keep]
    rho = p["invdepth"]
    rho2 = [rho[l] * 1.25 if l in reanchor else 1.0 / (1.0 / rho[l]) for l in lm_keep]
    rows = []  # (landmark, ref, obs, const, source)
    gone = set(drop_f)
    for f in range(p["F"]):
        l = f_lm[f]
        if f in gone or l not in lm_new_of or f_ref[f] not in new_of or f_obs[f] not in new_of:
            continue
        rows.append((lm_new_of[l], new_of[f_ref[f]], new_of[f_obs[f]], fc[f], -1 if l in reanchor else f))
    newest = K2 - 1
    src = [r for r in rows if r[4] >= 0]
    for j in range(n_new_lm):  # a copy of a carried landmark's factors plus an observation in the newest node
        base = src[(7 * j) % len(src)][0]
        facs = [r for r in src if r[0] == base]
        l2 = len(lm_src)
        lm_src.append(-1)
        rho2.append(rho2[base] * 0.9)
        rows += [(l2, r[1], r[2], r[3], -1) for r in facs]
        if newest != facs[0][1] and all(r[2] != newest for r in facs):
            rows.append((l2, facs[0][1], newest, facs[0][3], -1))
    order = rng.permutation(len(rows))
    rows = [rows[i] for i in order]
    q = copy.deepcopy(p)
    q.update(K=K2, pose=pose2, mix=mix2, L=len(lm_src), invdepth=np.array(rho2), F=len(rows),
             f_lm=np.array([r[0] for r in rows], np.int32), f_ref=np.array([r[1] for r in rows], np.int32),
             f_obs=np.array([r[2] for r in rows], np.int32), f_const=np.array([r[3] for r in rows]).reshape(-1),
             f_active=np.ones(len(rows), np.uint8), n_imu=K2 - 1, imu_blob=np.array(blob2).reshape(-1),
             n_gnss=len(gnode2), gnss_node=np.array(gnode2, np.int32), gnss_blh=blh2.reshape(-1), gnss_std=gstd2.reshape(-1), gnss_huber=1)
    if prior is not None:
        q.update(marg_r=prior["r"], marg_nblocks=len(prior["block_type"]), marg_block_type=prior["block_type"], marg_block_node=prior["block_node"],
                 marg_x0=prior["x0"], marg_J0=prior["J0"].reshape(-1).copy(), marg_e0=prior["e0"].copy())
    elif not keep_prior:
        q.update(marg_r=0, marg_nblocks=0, marg_block_type=np.zeros(0, np.int32), marg_block_node=np.zeros(0, np.int32), marg_x0=np.zeros(0),
                 marg_J0=np.zeros(0), marg_e0=np.zeros(0))
    carry = dict(node_src=node_src, lm_src=np.array(lm_src, np.int32), f_src=np.array([r[4] for r in rows], np.int32),
                 imu_src=np.array(imu_src, np.int32), gnss_src=np.array(gnss_src, np.int32))
    stale = copy.deepcopy(q)  # what the slide must not read
    stale["pose"].reshape(K2, 7)[node_src >= 0] = np.nan
    stale["mix"].reshape(K2, 9)[node_src >= 0] = np.nan
    stale["invdepth"][carry["lm_src"] >= 0] = np.nan
    stale["f_const"].reshape(-1, 14)[carry["f_src"] >= 0] = np.nan
    stale["imu_blob"].reshape(-1, IMU)[carry["imu_src"] >= 0] = np.nan
    stale["gnss_blh"].reshape(-1, 3)[carry["gnss_src"] >= 0] = np.nan
    stale["gnss_std"].reshape(-1, 3)[carry["gnss_src"] >= 0] = np.nan
    if prior is not None:
        stale["marg_J0"][:], stale["marg_e0"][:] = np.nan, np.nan
    return q, stale, carry
