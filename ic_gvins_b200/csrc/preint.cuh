// preint.cuh -- the IMU propagation of PreintegrationEarth / PreintegrationNormal on the device, one warp per interval (preint.cu), and its
// three front ends: the plain batch of icg_geom_imu_preintegrate_batch (geom.cu: states from the caller), the reintegration of the factors
// an icg_ba handle holds (ba.cu: icg_ba_reintegrate_resident, doReintegration of IG/ic_gvins.cc:1680-1695) and the new factors of a slide
// (ba.cu: icg_ba_slide_integrate_resident, addNewTimeNode / removeUnusedTimeNode / insertNewGnssTimeNode, :754-928).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace icg {

constexpr int PREINT_WARPS = 2;  // intervals (warps) per CTA

struct PreintBatch {  // all DEVICE pointers; interval k = rows off[k] .. off[k + 1] of imu
    int n;
    const double *state16;  // n x 16
    const double *iewn3;    // 3 shared, NULL: PreintegrationNormal
    const double *gravity3, *noise5, *imu;
    const int *off;
    double *blobs, *ends;   // n x ICG_IMU_BLOB_DOUBLES, n x 10 (ends may be NULL)
};

struct ReintItem {  // one factor of a window the caller asked to reintegrate
    int win, fac;    // window, factor (joins nodes fac and fac + 1)
    int row0, nrow;  // its rows in the staged IMU rows (row0 = the sample at its start)
};
struct PreintResident {
    int n;                    // items
    const ReintItem *item;    // DEVICE
    const double *imu;        // DEVICE, staged rows of every item
    const double *pose, *mix; // the handle's parameters, capacity-strided by window: K x 7, K x 9
    double *blob, *U;         // the handle's factors: K x ICG_IMU_BLOB_DOUBLES, K x 225 per window
    int K;                    // the handle's max_K
    double noise5[5], station[3];
    int8_t *status;           // per item: 1 reintegrated, 0 gate closed, -1 not positive definite (factor kept)
    double *ends;             // per item x 10: end state where status != 0
    double *out_blob;         // compact: the status-1 blobs in completion order ...
    int *out_item;            // ... and the item each one belongs to
    int *counter;             // number of status-1 items (zero before the launch)
};

// icg_ba_slide_integrate_resident (ba.cu): the new factors of the next windows, integrated from the handle's states into the slide's staged
// value rows (ba_slide.cuh), which ba_slide_gather then reads as if they had come from the host
struct SlideItem {    // one integrated factor, in factor order within its window
    int src;          // >= 0: old node; ICG_SLIDE_CHAIN; ICG_SLIDE_ROW
    int row0, nrow;   // its staged IMU rows
    int state;        // ICG_SLIDE_ROW: first double of its staged state16
    int blob;         // value offset of its staged blob (the square-root information follows at + ICG_IMU_BLOB_DOUBLES)
    int node;         // value offset of the staged node row (pose 7 | mix 9) it defines, or -1
    int normal;
    double grav[3];
};
struct SlideAlign {   // one aligned GNSS fix
    int blh;          // value offset of its staged blh
    int node;         // old node whose velocity moves it
    double dt;
};
struct SlideIntWin {  // the work of one window: one warp
    int win, item0, n_item, align0, n_align;
};
struct PreintSlide {
    int n;                          // windows with work
    const SlideIntWin *win;         // DEVICE, all below too
    const SlideItem *item;
    const SlideAlign *align;
    const double *imu, *state;      // staged rows, staged ICG_SLIDE_ROW states
    const double *pose, *mix;       // the handle's (old) parameters, K x 7, K x 9 per window
    int K;                          // the handle's max_K
    double *val;                    // the slide's staged value rows
    double noise5[5], station[3];
    int8_t *status;                 // per item: 1, or -1 when the covariance is not positive definite
    double *ends;                   // per item x 10
    double *out_blob;               // per item x ICG_IMU_BLOB_DOUBLES, or NULL
};

// icg_ins_gins_initialize (ins.cu): the first GNSS time node's factor of each stream gvinsInitialization initialized, from its state17[0]
// as a slide's ICG_SLIDE_ROW item starts (stateFromData's q.normalize() added, as for an old node), into blob and end_state10
struct PreintGins {
    int n;                      // streams
    const int32_t *status;      // DEVICE, all below too: per stream; only status 1 is integrated
    const double *state17;      // per stream: time, p, q_xyzw, v, bg, ba
    const double *gravity;      // per stream: g, the preintegration's gravity (0, 0, g)
    const int32_t *earth;       // per stream: PreintegrationEarth (iewn = Earth::iewn(station, p)) or PreintegrationNormal
    const double *imu;          // per stream: rows (dt, dtheta[3], dvel[3]), max_rows apart
    const int32_t *nrow;
    int max_rows;
    double noise5[5], station[3];
    double *blob, *ends;        // per stream x ICG_IMU_BLOB_DOUBLES, x 10
};

cudaError_t preint_batch_launch(const PreintBatch &a, cudaStream_t stream);
cudaError_t preint_gins_launch(const PreintGins &a, cudaStream_t stream);
cudaError_t preint_resident_launch(const PreintResident &a, cudaStream_t stream);
cudaError_t preint_slide_launch(const PreintSlide &a, cudaStream_t stream);
// loads the resident and slide kernels (a shard group loads every kernel its calls launch when it is set up)
cudaError_t preload_preint_resident();

}  // namespace icg
