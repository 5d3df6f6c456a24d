"""Stream-level parity with detection driven by the point lists: the 200-frame cfg-2 stream of tests/test_stream_gpu.py, whose cv2 arm
builds the occupancy mask with cv2.circle and counts the blocks in Python, while the CUDA arm hands its own tracked points to
icg_detect_features (IG/tracking/tracking.cc:579-685 in one call: gate, counts, mask, detection, shift).  The feature-ID lists must be
identical after every frame, with the same knife-edge allowance as the cv2-mask test (a tracking decision within 5e-3 px of a gate may
flip; the CUDA arm is then re-synchronised, at most twice)."""
import numpy as np
import pytest

from datagen import synth_klt as synth
from tests import oracle_api as oa
from tests.test_stream_gpu import H, MAXF, NFRAMES, W, Cv2Arm, GpuArm, flow_prediction, make_mask, occupancy

pytestmark = pytest.mark.gpu


class PointListArm(GpuArm):
    def detect_points(self, img, pts, ismask):
        # every tracked point is in pts2d_new_ (list B) and pts2d_ref_ (n_ref); no map-point features in this stream
        return self.det.features_detection_points(img, np.zeros((0, 2), np.float32), pts, n_ref=len(pts), ismask=ismask, max_features=MAXF)


def test_200_frame_stream_point_list_detection_matches_cv2(oracle):
    oa.declare_detect(oracle)
    from ic_gvins_b200.detect import block_rois
    rois, quota, min_dist, grid = block_rois(W, H, MAXF)
    stream = synth.KltStream(W, H, MAXF, 1234)
    cv, gpu = Cv2Arm(oracle), PointListArm()
    arms = [cv, gpu]
    try:
        state = [dict(ids=[], pts=np.zeros((0, 2), np.float32), next_id=0, prev=None) for _ in arms]
        resyncs, n_detect, n_skip = 0, 0, 0
        for t in range(NFRAMES):
            raw = stream.frame(t)
            imgs = [arm.preprocess(raw) for arm in arms]
            assert np.array_equal(imgs[0], imgs[1]), f"frame {t}: CLAHE differs"
            margins = None
            for k_arm, (arm, st, img) in enumerate(zip(arms, state, imgs)):
                if t > 0 and len(st["ids"]):
                    rng = np.random.Generator(np.random.PCG64(977 + t))  # same noise for both arms
                    pred = flow_prediction(st["pts"], t, rng)
                    fwd, good, margin = arm.track(st["prev"], img, st["pts"], pred)
                    if k_arm == 0:
                        margins = margin
                    keep = good != 0
                    st["ids"] = [i for i, k in zip(st["ids"], keep) if k]         # reduceVector (tracking.cc:831-839)
                    st["pts"] = fwd[keep]
            if t > 0 and state[0]["ids"] != state[1]["ids"]:
                diff = set(state[0]["ids"]) ^ set(state[1]["ids"])
                worst = max(float(margins[state[0]["_before"].index(i)]) for i in diff)
                assert worst <= 5e-3, f"frame {t}: feature IDs differ ({sorted(diff)}) and the decision was not on a knife edge (margin {worst:.3e} px)"
                resyncs += 1
                assert resyncs <= 2, "too many knife-edge re-synchronisations"
                state[1]["ids"], state[1]["pts"] = list(state[0]["ids"]), state[0]["pts"].copy()
            # cv2 arm: the gate, counts and mask on the host (tracking.cc:579-620), then block detection
            st = state[0]
            st["det"] = None
            if len(st["ids"]) <= MAXF - 5:
                want = [quota - c for c in occupancy(st["pts"], grid)]
                mask = make_mask(st["pts"], min_dist) if t > 0 else np.full((H, W), 255, np.uint8)
                blocks = cv.detect(imgs[0], rois, want, min_dist, mask)
                new = [p + np.array([x0, y0], np.float32) for (x0, y0, _, _), p in zip(rois, blocks) if len(p)]
                st["det"] = np.concatenate(new, axis=0) if new else np.zeros((0, 2), np.float32)
            # CUDA arm: its own point list is the only input of detection (ismask = frame > 0)
            sg = state[1]
            sg["det"] = gpu.detect_points(imgs[1], sg["pts"], t > 0)
            for s_, img in zip(state, imgs):
                if s_["det"] is not None:
                    new = s_["det"]
                    s_["ids"] = s_["ids"] + list(range(s_["next_id"], s_["next_id"] + len(new)))
                    s_["next_id"] += len(new)
                    s_["pts"] = np.concatenate([s_["pts"], new.astype(np.float32)], axis=0)
                s_["prev"] = img
                s_["_before"] = list(s_["ids"])
            d0, d1 = state[0]["det"], state[1]["det"]
            assert (d0 is None) == (d1 is None), f"frame {t}: the gate decided differently"
            if d0 is None:
                n_skip += 1
            else:
                n_detect += 1
                assert d0.shape == d1.shape, f"frame {t}: {len(d0)} vs {len(d1)} new corners"
                if len(d0):
                    assert np.abs(d0 - d1).max() <= 1e-3, f"frame {t}: new corners differ by {np.abs(d0 - d1).max():.2e} px"
            assert state[0]["ids"] == state[1]["ids"] and state[0]["next_id"] == state[1]["next_id"], f"frame {t}: ID lists differ after detection"
        assert n_detect >= 10 and state[0]["next_id"] > MAXF, "the stream must lose and re-detect features"
        print(f"point-list stream parity: {NFRAMES} frames, {state[0]['next_id']} feature IDs issued, {n_detect} detection passes, {n_skip} gated, "
              f"knife-edge re-syncs = {resyncs}")
    finally:
        gpu.close()
