"""Stream-level parity of the triangulation step: the 200-frame stream of tests/test_stream_track_gpu.py with the stand-in for triangulation
replaced by Tracking::triangulation (IG/tracking/tracking.cc:690-798) on every 10th frame (the keyframes).

The camera has fx = fy and no distortion, and its poses come from synth_klt.ego_motion: the frames are views of a fronto-parallel textured plane
at depth DEPTH, where image translation is camera translation in the plane, scale is motion along the optical axis and in-plane rotation is
roll about the principal point (640, 280), so each frame's similarity is exactly a camera motion.  The cv2 arm runs tests/tracking_oracle.py
(cv2 LK, cv2.findFundamentalMat) and tests/triangulation_oracle.py (numpy SVD); the CUDA arm chains icg_klt_track_frames_dev ->
icg_klt_triangulate_dev on the device, the live counts read from dev_n_out.  The map holds the last 10 keyframes; once it is full
window_normal is set and points whose reference keyframe has left it are dropped.  In this scene every point is triangulated or lost before
its keyframe leaves a 10-keyframe window, so the test prints the out-of-window count rather than requiring it; the branch itself is pinned by
tests/test_oracle_triangulation.py and tests/test_triangulation_gpu.py.  Feature-ID lists must be identical after every frame under the knife-edge
allowance of test_stream_track_gpu.py; every map point the device creates must match the numpy triangulation of the device's own lists to 1e-9
relative."""
import math

import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import oracle_api as oa
from tests import tracking_oracle as to
from tests import triangulation_oracle as tri
from tests.test_stream_gpu import H, MAXF, NFRAMES, W, Cv2Arm, make_mask, occupancy
from tests.test_stream_track_gpu import add_new, apply, new_state

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")

F = 460.0
INTR, DIST, DEPTH = [F, F, W / 2.0, H / 2.0, 0.0], [0.0, 0.0, 0.0, 0.0, 0.0], 5.0
WINDOW, KF_EVERY = 10, 10


def Rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def pose(t):
    """camera-to-world (R, position) whose view of the plane z = DEPTH is frame t's similarity: D - Z = D / s, R^T = roll(rot),
    (Cx, Cy) = -(D / (s f)) roll(-rot) (tx, ty)"""
    tx, ty, rot, sc = synth.ego_motion(t)
    c, s = math.cos(-rot), math.sin(-rot)
    k = -DEPTH / (sc * F)
    return Rz(-rot), np.array([k * (c * tx - s * ty), k * (s * tx + c * ty), DEPTH * (1.0 - 1.0 / sc)])


def lists(st):
    nm = len(st["mid"])
    ml = dict(prev_xy=st["mpts"], prev_undis_xy=st["mpts"], pw=st["mpw"], ref_kp_xy=np.full((nm, 2), np.nan, np.float32)) if nm else None
    rl = dict(new_xy=st["rpts"], ref_xy=st["rref"], ref_frame_id=st["rfid"], velocity_ref=st["rvel"]) if len(st["rid"]) else None
    return ml, rl


def apply_tri(st, lo, new):
    """reduce the reference list by the triangulation's kept points and append the new map points in creation order"""
    rid = st["rid"]
    st["mid"] = st["mid"] + [rid[k] for k in np.asarray(new["src"], np.int64).reshape(-1)]
    st["mpts"] = np.concatenate([st["mpts"], np.asarray(new["cur_xy"], np.float32).reshape(-1, 2)])
    st["mpw"] = np.concatenate([st["mpw"], np.asarray(new["pw"], np.float64).reshape(-1, 3)])
    st["rid"] = [rid[k] for k in np.asarray(lo["src"], np.int64).reshape(-1)]
    st["rpts"] = np.asarray(lo["cur_xy"], np.float32).reshape(-1, 2)
    st["rref"] = np.asarray(lo["ref_out_xy"], np.float32).reshape(-1, 2)
    st["rfid"] = np.asarray(lo["ref_frame_id_out"], np.int64).reshape(-1)
    st["rvel"] = np.asarray(lo["velocity_ref_out"], np.float64).reshape(-1, 2)


def tri_params(t, keyframes):
    R, c = pose(t)
    window = keyframes[-WINDOW:]
    P = dict(intrinsic=INTR, distortion=DIST, R_cur=R, t_cur=c, cur_id=t, ref_id=keyframes[-1], window_normal=len(keyframes) >= WINDOW,
             reprojection_error_std=1.5)
    kfs = {k: (pose(k)[0], pose(k)[1], k in window) for k in keyframes}
    return P, kfs


class ChainArm:
    """icg_klt_track_frames_dev, then on keyframes icg_klt_triangulate_dev reading the live counts from dev_n_out, on torch's stream"""

    def __init__(self):
        from ic_gvins_b200.clahe import Clahe
        from ic_gvins_b200.detect import Detector
        from ic_gvins_b200.klt import KltTracker
        self.stream = torch.cuda.Stream()  # the handle's stream: the copy below is ordered between the two calls without a host sync
        self.clahe, self.det = Clahe(W, H, 3.0, (21, 21)), Detector(W, H, 32, 64)
        self.klt = KltTracker(W, H, n_slots=2, max_points=2 * MAXF, stream=self.stream.cuda_stream)

    def close(self):
        self.clahe.close(), self.klt.close(), self.det.close()

    def step(self, t, img, P, ml, rl, tri_case):
        """returns (map_out, ref_out) of the tracking step and, on keyframes, (ref list given to the triangulation, list_out, new, counts)"""
        from ic_gvins_b200.klt import _SPEC, _TRI_NEW_SPEC, MAP_IN, MAP_OUT, REF_IN, REF_OUT, TRI_NEW, track_frame_params
        self.klt.upload(t % 2, img)
        keep_alive, offs, ptrs = [], [], []
        for lst, names_in, names_out in ((ml, MAP_IN, MAP_OUT), (rl, REF_IN, REF_OUT)):
            n = len(lst[names_in[0]]) if lst else 0
            tens = {}
            for k in names_in + names_out:
                dt, col = _SPEC[k]
                a = np.ascontiguousarray(np.asarray(lst[k], dt).reshape(n, col)) if (lst and k in names_in) else np.zeros((max(n, 1), col), dt)
                tens[k] = torch.from_numpy(a).cuda()
            keep_alive.append(tens)
            offs.append([0, n])
            ptrs.append({k: v.data_ptr() for k, v in tens.items()} if n else None)
        n_out = torch.zeros(2, dtype=torch.int32, device="cuda")
        par = torch.zeros(2, dtype=torch.float64, device="cuda")
        par_n = torch.zeros(2, dtype=torch.int32, device="cuda")
        p = track_frame_params((t - 1) % 2, t % 2, P["intrinsic"], P["distortion"], P["R_pre"], P["R_cur"], P["R_ref"], P["t_cur"], P["dt"],
                               P["ref_id"], P["fm_threshold"])
        N = max(offs[1][1], 1)
        src = torch.zeros(N, dtype=torch.int32, device="cuda")
        nt = {k: torch.zeros((N, c), dtype=getattr(torch, np.dtype(dt).name), device="cuda") for k, (dt, c) in _TRI_NEW_SPEC.items()}
        counts = torch.zeros(5, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()  # inputs were written on torch's default stream
        self.klt.track_frames_dev([p], offs[0], ptrs[0], offs[1], ptrs[1], n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())
        tri_out = None
        if tri_case is not None:
            TP, kfs = tri_case
            rt = keep_alive[1]
            names = ("ref_out_xy", "ref_frame_id_out", "cur_xy", "velocity_ref_out", "velocity")
            with torch.cuda.stream(self.stream):
                given = {k: rt[k].clone() for k in names}  # stream-ordered copy of the tracking step's lists, for the numpy check
            from tests.test_triangulation_gpu import kf_rows, struct
            has = offs[1][1] > 0
            self.klt.triangulate_dev([struct(TP)], [0, len(kfs)], kf_rows(kfs), offs[1], n_out.data_ptr() + 4, 2,
                                     dict({k: rt[k].data_ptr() for k in names}, src=src.data_ptr()) if has else None,
                                     {k: v.data_ptr() for k, v in nt.items()} if has else None, counts.data_ptr())
            tri_out = (given, rt, src, nt, counts)
        self.klt.sync()
        no = n_out.cpu().numpy()
        out = []
        for (tens, names_out), k_out in zip(((keep_alive[0], MAP_OUT), (keep_alive[1], REF_OUT)), no):
            out.append({k: tens[k].cpu().numpy()[:k_out] for k in names_out if k not in ("fwd_xy", "fwd_undis_xy", "keep")})
        mo, ro = out[0] if ml else {}, out[1] if rl else {}
        if tri_out is None:
            return mo, ro, None
        given, rt, src, nt, counts = tri_out
        c = counts.cpu().numpy()
        k_ref = int(no[1]) if rl else 0
        if rl:
            for k in ("ref_out_xy", "cur_xy", "ref_frame_id_out", "velocity_ref_out", "velocity"):  # the lists as the triangulation read them
                ro[k] = given[k].cpu().numpy()[:k_ref]
            ro["ref_frame_id_out"] = ro["ref_frame_id_out"].reshape(-1)
        kk, mm = max(int(c[0]), 0), max(int(c[1]), 0)
        lo = {k: rt[k].cpu().numpy()[:kk] for k in ("ref_out_xy", "cur_xy", "ref_frame_id_out", "velocity_ref_out")}
        lo["src"] = src.cpu().numpy()[:kk]
        new = {k: nt[k].cpu().numpy()[:mm] for k in TRI_NEW}
        new["src"], new["depth"], new["ref_frame_id"] = new["src"].reshape(-1), new["depth"].reshape(-1), new["ref_frame_id"].reshape(-1)
        if c[0] < 0:  # an empty list: nothing changes
            lo = dict(ref_out_xy=ro.get("ref_out_xy", np.zeros((0, 2), np.float32)), cur_xy=ro.get("cur_xy", np.zeros((0, 2), np.float32)),
                      ref_frame_id_out=ro.get("ref_frame_id_out", np.zeros(0, np.int64)), velocity_ref_out=ro.get("velocity_ref_out", np.zeros((0, 2))),
                      src=np.arange(k_ref, dtype=np.int32))
        return mo, ro, (lo, new, c)

    def detect(self, img, feat, new, n_ref, ismask):
        return self.det.features_detection_points(img, feat, new, n_ref=n_ref, ismask=ismask, max_features=MAXF)


def tri_lists(ro):
    return {k: ro[k] for k in ("ref_out_xy", "ref_frame_id_out", "cur_xy", "velocity_ref_out", "velocity")} if ro and len(ro.get("cur_xy", [])) else None


def test_200_frame_stream_with_device_triangulation_matches_cv2(oracle):
    oa.declare_detect(oracle)
    from ic_gvins_b200.detect import block_rois
    rois, quota, min_dist, grid = block_rois(W, H, MAXF)
    stream = synth.KltStream(W, H, MAXF, 1234)
    cv, gpu = Cv2Arm(oracle), ChainArm()
    margins = {}

    def lk_cv2(a, b, p, init):
        fwd, good, margin = cv.track(a, b, np.asarray(p, np.float32).reshape(-1, 2), np.asarray(init, np.float32).reshape(-1, 2))
        margins.setdefault("m", []).append(margin)
        return fwd, good
    try:
        S = [new_state(), new_state()]
        for s in S:
            s["mpw"] = np.zeros((0, 3))
        prev = [None, None]
        keyframes = [0]
        resyncs, n_detect, kf_made, n_kf, worst_pw, n_pw = 0, 0, 0, 0, 0.0, 0
        branches = np.zeros(5, np.int64)
        for t in range(NFRAMES):
            raw = stream.frame(t)
            imgs = [cv.preprocess(raw), gpu.clahe.apply(raw)]
            assert np.array_equal(imgs[0], imgs[1]), f"frame {t}: CLAHE differs"
            is_kf = t > 0 and t % KF_EVERY == 0
            if t > 0:
                margins.clear()
                (Rp, _), (Rc, tc), (Rr, _) = pose(t - 1), pose(t), pose(keyframes[-1])
                P = dict(intrinsic=INTR, distortion=DIST, R_pre=Rp, R_cur=Rc, R_ref=Rr, t_cur=tc, dt=0.1, ref_id=keyframes[-1], fm_threshold=1.0)
                tri_case = tri_params(t, keyframes) if is_kf else None
                ml, rl = lists(S[0])
                mo, ro, _, _, _ = to.track_frame(lk_cv2, prev[0], imgs[0], P, ml, rl, ransac=to.cv2_ransac(cv2))
                res0 = (mo, ro, tri.triangulation(tri_case[0], tri_case[1], tri_lists(ro)) if is_kf else None)
                ml, rl = lists(S[1])
                res1 = gpu.step(t, imgs[1], P, ml, rl, tri_case)
                if is_kf:
                    n_kf += 1
                    lo, new, c = res1[2]
                    # the device's map points against the numpy triangulation of the device's own lists
                    want = tri.triangulation(tri_case[0], tri_case[1], tri_lists(res1[1]))
                    both = np.intersect1d(new["src"], want[1]["src"])
                    if len(both):
                        a = new["pw"][np.searchsorted(new["src"], both)]
                        b = want[1]["pw"][np.searchsorted(want[1]["src"], both)]
                        rel = float(np.abs(a - b).max() / np.abs(b).max())
                        assert rel <= 1e-9, f"frame {t}: pw differs from the numpy triangulation by {rel:.2e}"
                        worst_pw, n_pw = max(worst_pw, rel), n_pw + len(both)
                    if c[0] >= 0:
                        got_st = np.zeros(len(want[3]), np.int32)
                        got_st[lo["src"]], got_st[new["src"]] = 1, 2
                        for k in np.nonzero(got_st != want[3])[0]:
                            assert tri.knife_edge(want[4][k]), f"frame {t}: triangulation decision of point {k} differs off a knife edge"
                    branches += np.maximum(c, 0)
                    kf_made += int(c[1] > 0)
                before = [(list(s["mid"]), list(s["rid"])) for s in S]
                for s, (mo, ro, tr) in zip(S, (res0, res1)):
                    if mo:
                        s["mpw"] = s["mpw"][np.asarray(mo["src"], np.int64).reshape(-1)]
                    apply(s, mo, ro)
                    if tr is not None:
                        apply_tri(s, tr[0], tr[1])
                if (S[0]["mid"], S[0]["rid"]) != (S[1]["mid"], S[1]["rid"]):
                    diff = (set(S[0]["mid"]) ^ set(S[1]["mid"])) | (set(S[0]["rid"]) ^ set(S[1]["rid"]))
                    allm = np.concatenate(margins["m"]) if margins.get("m") else np.zeros(0)
                    ids = before[0][0] + before[0][1]
                    worst = max(float(allm[ids.index(i)]) if i in ids and ids.index(i) < len(allm) else np.inf for i in diff)
                    assert worst <= 5e-3, f"frame {t}: feature IDs differ ({sorted(diff)}) and the decision was not on a knife edge ({worst:.3e} px)"
                    resyncs += 1
                    assert resyncs <= 2, "too many knife-edge re-synchronisations"
                    S[1] = {k: (list(v) if isinstance(v, list) else (v.copy() if hasattr(v, "copy") else v)) for k, v in S[0].items()}
                if is_kf:
                    keyframes.append(t)
            else:
                gpu.klt.upload(0, imgs[1])
                gpu.klt.sync()
            feats = [s["mpts"] if len(s["mid"]) else np.zeros((0, 2), np.float32) for s in S]  # no distortion: keyPoint() == distortedKeyPoint()
            d0 = None
            if len(S[0]["mid"]) + len(S[0]["rid"]) <= MAXF - 5:
                allp = np.concatenate([feats[0], S[0]["rpts"]])
                want = [quota - c for c in occupancy(allp, grid)]
                mask = make_mask(allp, min_dist) if t > 0 else np.full((H, W), 255, np.uint8)
                blocks = cv.detect(imgs[0], rois, want, min_dist, mask)
                nw = [p + np.array([x0, y0], np.float32) for (x0, y0, _, _), p in zip(rois, blocks) if len(p)]
                d0 = np.concatenate(nw, axis=0) if nw else np.zeros((0, 2), np.float32)
            d1 = gpu.detect(imgs[1], feats[1], S[1]["rpts"], len(S[1]["rid"]), t > 0)
            assert (d0 is None) == (d1 is None), f"frame {t}: the gate decided differently"
            if d0 is not None:
                n_detect += 1
                assert d0.shape == d1.shape, f"frame {t}: {len(d0)} vs {len(d1)} new corners"
                if len(d0):
                    assert np.abs(d0 - d1).max() <= 1e-3, f"frame {t}: new corners differ by {np.abs(d0 - d1).max():.2e} px"
                add_new(S[0], d0, t)
                add_new(S[1], d1, t)
            prev = imgs
            assert S[0]["mid"] == S[1]["mid"] and S[0]["rid"] == S[1]["rid"] and S[0]["next_id"] == S[1]["next_id"], f"frame {t}: ID lists differ"
        assert kf_made * 2 >= n_kf, f"map points on only {kf_made} of {n_kf} keyframes"
        assert branches[1] > 0 and branches[3] > 0, branches  # new map points and resets; see the module docstring for out-of-window points
        print(f"triangulation stream parity: {NFRAMES} frames, {n_kf} keyframes ({kf_made} with new map points), {S[0]['next_id']} feature IDs, "
              f"{len(S[0]['mid'])} map points at the end, branches (kept, succeeded, outlier, reset, outtime) = {branches.tolist()}, "
              f"{n_pw} map points checked (worst pw {worst_pw:.1e}), knife-edge re-syncs = {resyncs}")
    finally:
        gpu.close()
