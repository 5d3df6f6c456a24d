// klt_handle.cuh -- the KLT handle (struct icg_klt) and the pyramid geometry it owns, shared by klt.cu (pyramids, LK) and track.cu
// (Tracking::trackMappoint / trackReferenceFrame on the handle's slots and stream).
#pragma once
#include <vector>

#include "common.cuh"

namespace icg {

constexpr int KLT_WIN     = 21;
constexpr int KLT_LEVELS  = 4;  // maxLevel 3 (IG/tracking/tracking.h:113)
constexpr int KLT_BOXW    = 48; // TMA box width in bytes: the innermost TMA coordinate must be 16-byte aligned
                                // (measured: UTMALDG raises "illegal instruction" otherwise), so windows start at
                                // x & ~15 and over-fetch: 15 + 24 <= 48
constexpr int KLT_BOXH_J  = 32; // search-window rows (22 needed + 10 slack)
constexpr int KLT_BOXH_I  = 24; // template-window rows (21 + 1 bilinear + 2 Scharr)
constexpr int KLT_MARGIN  = 5;  // search window slack kept on the low side when (re-)centring
constexpr int KLT_PAD     = 48; // reflect-101 padding stored around every pyramid plane: any TMA box the tracker can ask for
                                // (x in [-41, W+42], y in [-26, H+26]) stays inside the plane, so no border patching is needed
constexpr int KLT_WPB     = 4;  // warps per block
constexpr int KLT_PXL     = 14; // template pixels per lane: ceil(441 / 32)

struct KltLevel {
    const uint8_t *base;  // padded plane origin of slot 0; pixel (x, y) of slot s lives at base + s*slot_stride + (y+PAD)*pitch + x+PAD
    int W, H, pitch;      // logical size, padded row pitch (multiple of 16)
    size_t slot_stride;
};

struct KltMaps {
    CUtensorMap mj[KLT_LEVELS];  // box 48 x 32 x 1 (search window)
    CUtensorMap mi[KLT_LEVELS];  // box 48 x 24 x 1 (template window)
};

struct TrackScratch;
void track_scratch_free(TrackScratch *t);  // track.cu

}  // namespace icg

struct icg_klt {
    int W, H, n_slots, max_pts, device;
    int n_levels;  // pyramid levels cv::buildOpticalFlowPyramid builds for this size at maxLevel KLT_LEVELS - 1 (<= KLT_LEVELS)
    cudaStream_t stream;
    bool own_stream;
    icg::KltLevel lv[icg::KLT_LEVELS];
    uint8_t *planes[icg::KLT_LEVELS];
    icg::KltMaps maps;
    // device scratch for the host-pointer API
    int32_t *d_slots;
    float *d_prev, *d_init, *d_fwd, *d_bwd, *d_err;
    uint8_t *d_status;
    // pinned staging
    uint8_t *h_stage;
    size_t h_stage_bytes;
    // content-addressed cache for the host-pointer API: hash -> slot
    std::vector<uint64_t> slot_hash;
    std::vector<uint64_t> slot_age;
    uint64_t age;
    // linear device staging of the batched frame upload (icg_klt_upload_batch)
    uint8_t *d_upstage = nullptr;
    size_t d_upstage_bytes = 0;
    // scratch of icg_klt_track_frames_dev / icg_klt_track_frame (track.cu), allocated on first use
    icg::TrackScratch *track = nullptr;
};

