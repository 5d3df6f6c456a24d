"""CPU: the restatement of trackMappoint / trackReferenceFrame in tests/tracking_oracle.py, pinned by hand cases for every rule of
IG/tracking/tracking.cc:351-574 and against a live-cv2 restatement (cv2.calcOpticalFlowPyrLK x 2, cv2.findFundamentalMat) on frame pairs of
the synthetic stream."""
import numpy as np
import pytest

from datagen import synth_klt as synth
from oracle import camera_ref as cref
from tests import oracle_api as oa
from tests import tracking_oracle as to

INTR = [460.0, 455.0, 640.0, 280.0, 0.0]
DIST = [-0.28, 0.07, 2e-4, 1e-5, 0.0]
I3 = np.eye(3)


def Rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def params(**kw):
    P = dict(intrinsic=INTR, distortion=DIST, R_pre=I3, R_cur=I3, R_ref=I3, t_cur=np.zeros(3), dt=0.1, ref_id=7, fm_threshold=1.0)
    P.update(kw)
    return P


def fake_lk(status):
    """LK stand-in: the forward position is the prediction, the gate is `status`"""
    return lambda a, b, p, init: (np.asarray(init, np.float32).reshape(-1, 2).copy(), np.asarray(status, np.uint8))


def test_prediction_pieces():
    cam = to.cam_dict(INTR, DIST)
    # world2pixel: the optical axis lands on the principal point, a point at depth 2 with x = 1 on cx + fx / 2
    px = to.world2pixel(cam, [[0, 0, 1.0], [1.0, 0, 2.0]], I3, np.zeros(3))
    assert np.array_equal(px, np.array([[640, 280], [640 + 230, 280]], np.float32))
    # the map prediction adds the distortion of Camera::distortPoints
    assert np.array_equal(to.predict_map(cam, [[0.3, -0.1, 1.5]], I3, np.zeros(3)), cref.distort_points(cam, to.world2pixel(cam, [[0.3, -0.1, 1.5]], I3, np.zeros(3))))
    # the reference prediction with R_cur == R_pre is undistort -> distort: back on the input where the five fixed-point iterations of
    # cv::undistortPoints converge (the centre of this strongly distorted lens)
    rng = np.random.default_rng(3)
    pts = rng.uniform([440, 180], [840, 380], (50, 2)).astype(np.float32)
    back = to.predict_ref(cam, pts, Rz(0.01), Rz(0.01))
    assert np.abs(back - pts).max() < 2e-3
    # a yaw of the camera between the frames shifts the prediction sideways by about fx * angle near the centre
    sh = to.predict_ref(cam, np.array([[640, 280]], np.float32), I3, Rz(0.01))
    assert abs(float(sh[0, 1]) - 280) < 1e-3 and abs(abs(float(sh[0, 0]) - 640)) < 1e-3
    cv2 = pytest.importorskip("cv2")
    K = np.array([[INTR[0], INTR[4], INTR[2]], [0, INTR[1], INTR[3]], [0, 0, 1]])
    ref = cv2.undistortPoints(pts.reshape(-1, 1, 2), K, np.array(DIST), P=K).reshape(-1, 2)
    assert np.abs(cref.undistort_points(cam, pts) - ref).max() <= 1e-3


def test_compaction_velocity_ref_rule_and_parallax():
    rng = np.random.default_rng(5)
    n = 10
    new = rng.uniform([200, 100], [1000, 400], (n, 2)).astype(np.float32)
    ref = (new + rng.normal(0, 3, (n, 2))).astype(np.float32)
    ids = np.array([7, 8, 6, 7, 9, 7, 5, 8, 7, 7], np.int64)
    vref = rng.normal(0, 1, (n, 2))
    st = np.array([1, 1, 0, 1, 1, 0, 1, 1, 1, 0], np.uint8)
    P = params(R_cur=Rz(0.02))
    mo, ro, n_out, par, par_n = to.track_frame(fake_lk(st), None, None, P, None, dict(new_xy=new, ref_xy=ref, ref_frame_id=ids, velocity_ref=vref))
    keep = st != 0
    assert n_out[1] == keep.sum() < 15  # fewer than 15 survivors: no RANSAC, all kept
    assert np.array_equal(ro["src"], np.nonzero(keep)[0]) and np.array_equal(ro["ref_frame_id_out"], ids[keep])
    assert np.array_equal(ro["ref_out_xy"], ref[keep])
    newer = ids[keep] > 7
    assert np.array_equal(ro["velocity_ref_out"][newer], ro["velocity"][newer])
    assert np.array_equal(ro["velocity_ref_out"][~newer], vref[keep][~newer])
    same = ids[keep] == 7
    assert par_n[1] == same.sum() == 3 and par[1] > 0
    assert par_n[0] == -1 and n_out[0] == 0  # no map list: parallax_map_ kept


def test_early_return_rules():
    pw = np.array([[0.1, 0.0, 2.0], [0.0, 0.1, 3.0]])
    lists = dict(prev_xy=np.array([[600, 300], [650, 250]], np.float32), prev_undis_xy=np.array([[600, 300], [650, 250]], np.float32), pw=pw,
                 ref_kp_xy=np.array([[600, 301], [np.nan, np.nan]], np.float32))
    # a map list the gate empties: parallax_map_ = counts = 0 (:410-419)
    _, _, n_out, par, par_n = to.track_frame(fake_lk([0, 0]), None, None, params(), lists, None)
    assert n_out[0] == 0 and par_n[0] == 0 and par[0] == 0.0
    # survivors, one with a frame_ref_ feature
    _, _, n_out, par, par_n = to.track_frame(fake_lk([1, 1]), None, None, params(), lists, None)
    assert n_out[0] == 2 and par_n[0] == 1 and par[0] > 0
    # a reference list the gate empties returns before the parallax (:513-517): -1
    r = dict(new_xy=np.array([[600, 300]], np.float32), ref_xy=np.array([[600, 300]], np.float32), ref_frame_id=np.array([7]), velocity_ref=np.zeros((1, 2)))
    _, ro, n_out, _, par_n = to.track_frame(fake_lk([0]), None, None, params(), None, r)
    assert n_out[1] == 0 and par_n[1] == -1 and ro["keep"].tolist() == [0]


@pytest.mark.parametrize("n_keep", [14, 15])
def test_ransac_applies_from_15_survivors(n_keep):
    rng = np.random.default_rng(n_keep)
    n = 16
    new = rng.uniform([200, 100], [1000, 400], (n, 2)).astype(np.float32)
    st = np.zeros(n, np.uint8)
    st[:n_keep] = 1
    calls = []

    def ransac(p1, p2, thr):
        calls.append(len(p1))
        m = np.ones(len(p1), bool)
        m[3] = False
        return m
    _, ro, n_out, _, _ = to.track_frame(fake_lk(st), None, None, params(), None,
                                        dict(new_xy=new, ref_xy=new, ref_frame_id=np.full(n, 7), velocity_ref=np.zeros((n, 2))), ransac=ransac)
    if n_keep < 15:
        assert calls == [] and n_out[1] == 14
    else:
        assert calls == [15] and n_out[1] == 14 and 3 not in ro["src"].tolist() and ro["keep"][3] == 0


def test_whole_step_matches_live_cv2_restatement(oracle):
    cv2 = pytest.importorskip("cv2")
    W, H = 1280, 560
    stream = synth.KltStream(W, H, 300, 1234)
    lk_oracle = lambda a, b, p, init: oa.track_fb(oracle, a, b, p, init)[::2]  # noqa: E731
    for t in (1, 7, 23):
        a, b = stream.frame(t - 1), stream.frame(t)
        p0 = stream.points(t - 1).astype(np.float32)
        cam = to.cam_dict(INTR, [0, 0, 0, 0, 0])
        nm = 100
        pw = np.concatenate([cref.pixel2cam(cam, stream.points(t)[:nm].astype(np.float32))[:, :2] * 4.0, np.full((nm, 1), 4.0)], 1)
        ml = dict(prev_xy=p0[:nm], prev_undis_xy=p0[:nm], pw=pw, ref_kp_xy=p0[:nm])
        ids = np.where(np.arange(300 - nm) % 3 == 0, 7, 8).astype(np.int64)
        rl = dict(new_xy=p0[nm:], ref_xy=p0[nm:], ref_frame_id=ids, velocity_ref=np.zeros((300 - nm, 2)))
        P = params(distortion=[0, 0, 0, 0, 0])
        got = to.track_frame(lk_oracle, a, b, P, ml, rl)
        want = to.track_frame(to.cv2_lk_fb(cv2), a, b, P, ml, rl, ransac=to.cv2_ransac(cv2))
        for k in (0, 1):
            assert np.array_equal(got[k]["keep"], want[k]["keep"]), (t, k)
            assert np.abs(got[k]["cur_xy"] - want[k]["cur_xy"]).max() <= 1e-3
        assert np.array_equal(got[2], want[2]) and np.array_equal(got[4], want[4])
        assert np.allclose(got[3], want[3], rtol=0, atol=1e-3)
        assert got[2][0] > 80 and got[2][1] > 150
