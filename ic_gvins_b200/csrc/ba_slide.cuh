// ba_slide.cuh -- the slide of B resident windows to the next keyframe's windows (icg_ba_slide_resident): the interface between the handle
// (ba.cu: validation, the structure tables, staging, copies) and the kernels (ba_slide.cu, built without FMA contraction so that the prior's
// normal equations are the sums icg_ba_upload forms on the host, bit for bit).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace icg {

constexpr int SLIDE_NODE = 16;  // staged doubles per new node: pose 7 | mix 9
constexpr int SLIDE_IMU = 705;  // per new IMU factor: blob 480 | U 225
constexpr int SLIDE_GNSS = 6;   // per new GNSS fix: blh 3 | std 3

// One window of the slide, as staged.  Every map entry m of a destination row: m >= 0 is the row of the OLD window it carries, m < 0 a staged
// row that starts at value offset -(m + 1) (doubles, relative to SlideArgs::val).
struct SlideWin {
    int K, L, F, n_imu, n_gnss;                         // next window's sizes
    int node_map, lm_map, slot_map, imu_map, gnss_map;  // first entry of each map in SlideArgs::map (slot_map: by record slot)
    int r, from_marg;  // prior rows (0: none); 1: J0 / e0 from the marginalization workspace, 0: staged at j0 / e0
    int j0, e0;        // value offsets of the staged J0 (r x r row-major) and e0 (from_marg = 0)
    int slot;          // from_marg = 1: the window's slot of the workspace, or -1: no source here (H0, b0, c0 are written as zeros)
    int vis;           // 1: lm_map / slot_map are in SlideArgs::vmap, their rows m < 0 start at -(m + 1) of vlm / vfc (the vision build's)
};

struct SlideArgs {
    const SlideWin *win;
    const int *map;
    const double *val;
    const int *vmap;          // vision windows: landmark and record-slot maps written on the device (ba_pack_structure)
    const double *vlm, *vfc;  // and the rows their entries m < 0 name: the built inverse depths, the new factors' constants
    int K, L, F, G, R;  // capacities: the handle's arrays are strided by them per window
    // the old window (copies of the handle's arrays at the same strides; old_fc is the f_const_s buffer the slide swaps out) -> the handle
    const double *old_pose, *old_mix, *old_rho, *old_fc, *old_blob, *old_U, *old_blh, *old_std;
    double *pose, *mix, *rho, *fc, *blob, *U, *blh, *std;
    // prior: the marginalization workspace (J0 r x r at slot mrcap^2, e0 at slot mrcap) -> the handle's H0 (r x r at w R^2), b0, c0
    const double *mJ0, *me0;
    int mrcap;
    double *H0, *b0, *c0;
};

// ba_slide_gather: the value rows of the next windows, carried from the old copies or staged;  ba_slide_prior: H0 = J0^T J0, b0 = J0^T e0,
// c0 = e0.e0 of every window with a prior, in the order of icg_ba_upload's host loop.  Both on `stream`, batched over the windows; max_elems is
// the largest window's destination doubles of the gather (16 K + L + 14 F + 705 n_imu + 6 n_gnss), max_r its largest prior.
cudaError_t launch_slide(const SlideArgs &a, int n_windows, int max_elems, int max_r, cudaStream_t stream);
// loads both kernels (a shard group loads every kernel its calls launch when it is set up)
cudaError_t preload_slide();

}  // namespace icg
