"""Stream-level parity of the tracking step: the 200-frame cfg-2 stream of tests/test_stream_gpu.py, where the CUDA arm makes ONE
icg_klt_track_frames_dev call per frame (trackMappoint + trackReferenceFrame, IG/tracking/tracking.cc:351-574, with the reference's own pose
prediction under identity attitudes) and detects from the returned point lists, while the cv2 arm restates both steps with cv2 and numpy
(tests/tracking_oracle.py: cv2.calcOpticalFlowPyrLK x 2, cv2.findFundamentalMat) and builds the occupancy mask with cv2.circle.  Part of every
list is a map list: every 10 frames the points detected at least 10 frames earlier become map points, with pw back-projected from their
previous position at a fixed depth.  The feature-ID lists must be identical after every frame; the knife-edge allowance is that of
test_stream_points_gpu.py (a tracking decision within 5e-3 px of a gate may flip; the CUDA arm is then re-synchronised, at most twice)."""
import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import oracle_api as oa
from tests import tracking_oracle as to
from tests.test_stream_gpu import H, MAXF, NFRAMES, W, Cv2Arm, make_mask, occupancy

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")

INTR, DIST, DEPTH = [460.0, 455.0, 640.0, 280.0, 0.0], [0.0, 0.0, 0.0, 0.0, 0.0], 5.0
I3 = np.eye(3)


def new_state():
    return dict(mid=[], mpts=np.zeros((0, 2), np.float32), rid=[], rpts=np.zeros((0, 2), np.float32), rref=np.zeros((0, 2), np.float32),
                rfid=np.zeros(0, np.int64), rvel=np.zeros((0, 2)), next_id=0)


def lists(st, cam):
    """the map list (pw at DEPTH behind the previous position: identity attitudes make world2pixel predict the previous position) and the
    reference list of one arm's state"""
    nm = len(st["mid"])
    pc = to.cref.pixel2cam(cam, to.cref.undistort_points(cam, st["mpts"])) if nm else np.zeros((0, 3))
    rk = to.cref.undistort_points(cam, st["mpts"]) if nm else np.zeros((0, 2), np.float32)
    if nm:
        rk[1::2] = np.nan
    ml = dict(prev_xy=st["mpts"], prev_undis_xy=to.cref.undistort_points(cam, st["mpts"]), pw=pc * DEPTH, ref_kp_xy=rk) if nm else None
    rl = dict(new_xy=st["rpts"], ref_xy=st["rref"], ref_frame_id=st["rfid"], velocity_ref=st["rvel"]) if len(st["rid"]) else None
    return ml, rl


def apply(st, mo, ro):
    """reduce the state by the step's outputs (src indices), as Tracking does with mappoint_matched_ / pts2d_ref_frame_"""
    if mo:
        st["mid"] = [st["mid"][k] for k in np.asarray(mo["src"], np.int64).reshape(-1)]
        st["mpts"] = np.asarray(mo["cur_xy"], np.float32).reshape(-1, 2)
    if ro:
        src = np.asarray(ro["src"], np.int64).reshape(-1)
        st["rid"] = [st["rid"][k] for k in src]
        st["rpts"] = np.asarray(ro["cur_xy"], np.float32).reshape(-1, 2)
        st["rref"] = np.asarray(ro["ref_out_xy"], np.float32).reshape(-1, 2)
        st["rfid"] = np.asarray(ro["ref_frame_id_out"], np.int64).reshape(-1)
        st["rvel"] = np.asarray(ro["velocity_ref_out"], np.float64).reshape(-1, 2)


def promote(st, t):
    """points detected at least 10 frames ago join the map list (a stand-in for triangulation)"""
    old = st["rfid"] <= t - 10
    if old.any():
        st["mid"] = st["mid"] + [i for i, o in zip(st["rid"], old) if o]
        st["mpts"] = np.concatenate([st["mpts"], st["rpts"][old]])
        st["rid"] = [i for i, o in zip(st["rid"], old) if not o]
        for k in ("rpts", "rref", "rfid", "rvel"):
            st[k] = st[k][~old]


def add_new(st, new, t):
    st["rid"] = st["rid"] + list(range(st["next_id"], st["next_id"] + len(new)))
    st["next_id"] += len(new)
    new = np.asarray(new, np.float32).reshape(-1, 2)
    st["rpts"] = np.concatenate([st["rpts"], new])
    st["rref"] = np.concatenate([st["rref"], new])
    st["rfid"] = np.concatenate([st["rfid"], np.full(len(new), t, np.int64)])
    st["rvel"] = np.concatenate([st["rvel"], np.zeros((len(new), 2))])


class TrackArm:
    """one icg_klt_track_frames_dev call per frame on device-resident lists, detection from the returned lists"""

    def __init__(self):
        from ic_gvins_b200.clahe import Clahe
        from ic_gvins_b200.detect import Detector
        from ic_gvins_b200.klt import KltTracker
        self.clahe, self.klt, self.det = Clahe(W, H, 3.0, (21, 21)), KltTracker(W, H, n_slots=2, max_points=2 * MAXF), Detector(W, H, 32, 64)

    def close(self):
        self.clahe.close(), self.klt.close(), self.det.close()

    def step(self, t, img, P, ml, rl):
        from ic_gvins_b200.klt import MAP_IN, MAP_OUT, REF_IN, REF_OUT, _SPEC, track_frame_params
        self.klt.upload(t % 2, img)
        self.klt.sync()
        out, keep_alive = [], []
        offs, ptrs = [], []
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
        torch.cuda.synchronize()
        p = track_frame_params((t - 1) % 2, t % 2, P["intrinsic"], P["distortion"], I3, I3, I3, np.zeros(3), P["dt"], P["ref_id"], P["fm_threshold"])
        self.klt.track_frames_dev([p], offs[0], ptrs[0], offs[1], ptrs[1], n_out.data_ptr(), par.data_ptr(), par_n.data_ptr())
        self.klt.sync()
        no = n_out.cpu().numpy()
        for (tens, names_out), k_out in zip(((keep_alive[0], MAP_OUT), (keep_alive[1], REF_OUT)), no):
            out.append({k: tens[k].cpu().numpy()[:k_out] for k in names_out if k not in ("fwd_xy", "fwd_undis_xy", "keep")})
        return out[0] if ml else {}, out[1] if rl else {}

    def detect(self, img, feat, new, n_ref, ismask):
        return self.det.features_detection_points(img, feat, new, n_ref=n_ref, ismask=ismask, max_features=MAXF)


def test_200_frame_stream_with_the_device_tracking_step_matches_cv2(oracle):
    oa.declare_detect(oracle)
    from ic_gvins_b200.detect import block_rois
    rois, quota, min_dist, grid = block_rois(W, H, MAXF)
    stream = synth.KltStream(W, H, MAXF, 1234)
    cam = to.cam_dict(INTR, DIST)
    cv, gpu = Cv2Arm(oracle), TrackArm()
    margins = {}

    def lk_cv2(a, b, p, init):
        fwd, good, margin = cv.track(a, b, np.asarray(p, np.float32).reshape(-1, 2), np.asarray(init, np.float32).reshape(-1, 2))
        margins.setdefault("m", []).append(margin)
        return fwd, good
    try:
        S = [new_state(), new_state()]
        prev = [None, None]
        resyncs, n_detect, n_map_max = 0, 0, 0
        for t in range(NFRAMES):
            raw = stream.frame(t)
            imgs = [cv.preprocess(raw), gpu.clahe.apply(raw)]
            assert np.array_equal(imgs[0], imgs[1]), f"frame {t}: CLAHE differs"
            P = dict(intrinsic=INTR, distortion=DIST, R_pre=I3, R_cur=I3, R_ref=I3, t_cur=np.zeros(3), dt=0.1, ref_id=(t // 10) * 10, fm_threshold=1.0)
            results = []
            if t > 0:
                margins.clear()
                ml, rl = lists(S[0], cam)
                mo, ro, n_out, _, _ = to.track_frame(lk_cv2, prev[0], imgs[0], P, ml, rl, ransac=to.cv2_ransac(cv2))
                results.append((mo, ro))
                ml, rl = lists(S[1], cam)
                results.append(gpu.step(t, imgs[1], P, ml, rl))
                before = [(list(s["mid"]), list(s["rid"])) for s in S]
                for s, (mo, ro) in zip(S, results):
                    apply(s, mo, ro)
                if (S[0]["mid"], S[0]["rid"]) != (S[1]["mid"], S[1]["rid"]):
                    diff = (set(S[0]["mid"]) ^ set(S[1]["mid"])) | (set(S[0]["rid"]) ^ set(S[1]["rid"]))
                    allm = np.concatenate(margins["m"]) if margins.get("m") else np.zeros(0)
                    ids = before[0][0] + before[0][1]
                    worst = max(float(allm[ids.index(i)]) if i in ids and ids.index(i) < len(allm) else np.inf for i in diff)
                    assert worst <= 5e-3, f"frame {t}: feature IDs differ ({sorted(diff)}) and the decision was not on a knife edge ({worst:.3e} px)"
                    resyncs += 1
                    assert resyncs <= 2, "too many knife-edge re-synchronisations"
                    S[1] = {k: (list(v) if isinstance(v, list) else (v.copy() if hasattr(v, "copy") else v)) for k, v in S[0].items()}
            else:
                gpu.klt.upload(0, imgs[1])  # slot t % 2 holds frame t
            if t % 10 == 0 and t > 0:
                for s in S:
                    promote(s, t)
            n_map_max = max(n_map_max, len(S[0]["mid"]))
            # featuresDetection (tracking.cc:576-685): feat = the tracked map points' keyPoint(), new = pts2d_new_, n_ref = |pts2d_ref_|
            feats = [to.cref.undistort_points(cam, s["mpts"]) if len(s["mid"]) else np.zeros((0, 2), np.float32) for s in S]
            d0 = None
            if len(S[0]["mid"]) + len(S[0]["rid"]) <= MAXF - 5:
                allp = np.concatenate([feats[0], S[0]["rpts"]])
                want = [quota - c for c in occupancy(allp, grid)]
                mask = make_mask(allp, min_dist) if t > 0 else np.full((H, W), 255, np.uint8)
                blocks = cv.detect(imgs[0], rois, want, min_dist, mask)
                new = [p + np.array([x0, y0], np.float32) for (x0, y0, _, _), p in zip(rois, blocks) if len(p)]
                d0 = np.concatenate(new, axis=0) if new else np.zeros((0, 2), np.float32)
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
        assert n_detect >= 10 and S[0]["next_id"] > MAXF and n_map_max > 20, "the stream must lose and re-detect features and carry map points"
        print(f"tracking-step stream parity: {NFRAMES} frames, {S[0]['next_id']} feature IDs, {n_detect} detection passes, up to {n_map_max} map "
              f"points, knife-edge re-syncs = {resyncs}")
    finally:
        gpu.close()
