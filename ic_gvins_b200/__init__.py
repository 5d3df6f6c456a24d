"""ic_gvins_b200 -- H100-native (sm_90a) hot paths of i2Nav-WHU/IC-GVINS behind a C ABI.

Host-side mirror (Python, over ctypes) of the reference call sites:
  klt.calcOpticalFlowPyrLK / klt.KltTracker   <- cv::calcOpticalFlowPyrLK as used by Tracking (tracking.cc:385-403)
  detect.goodFeaturesToTrack / cornerSubPix     <- Tracking::featuresDetection (tracking.cc:576-688)
  clahe.Clahe                                   <- cv::CLAHE as Tracking::preprocessing applies it (tracking.cc:62,141)
  camera.Camera / findFundamentalMat /
    triangulatePoints / calculate_histogram     <- Camera (camera.cc:72-150), cv::findFundamentalMat (tracking.cc:547),
                                                   Tracking::triangulatePoint (:796-808), calculateHistigram (:88-104)  [host functions]
  ba.WindowSolver (.solve / .gvins_optimization / .marginalize)
                                                <- GVINS::gvinsOptimization + ceres::Solver::Solve (ic_gvins.cc:1130-1239),
                                                   MarginalizationInfo::marginalization via gvinsMarginalization (:1412-1640)
  ins.InsWindow                                 <- ins_window_: runFusion's mechanization, redoInsMechanization, getCameraPoseFromInsWindow
                                                   (ic_gvins.cc:249-293, misc.cc:30-286) for B streams on the device
The product path is the CUDA library only; importing this package never touches oracle/.
"""
from ._lib import IcgError, LIB_PATH, lib  # noqa: F401

__all__ = ["IcgError", "LIB_PATH", "lib"]
