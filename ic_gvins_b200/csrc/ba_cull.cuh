// ba_cull.cuh -- the post-solve map update and outlier culling of GVINS::gvinsOptimization (IG/ic_gvins.cc:1232-1236) for the windows an
// icg_ba handle holds: the interface between the handle (ba.cu: validation, staging, copies) and the kernel (ba_cull.cu, built without FMA
// contraction so that its sums are the fixed-order sums the numpy restatement in tests/post_solve_oracle.py computes).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/icgvins_b200.h"

namespace icg {

constexpr int CULL_THREADS = 128;
constexpr int CULL_MAX_NODES = 32;  // = the handle's max_K limit

struct CullWin {  // one window's inputs, as staged
    double R_bc[9], t_bc[3], td_bc;
    int K, L, estimate_ext, estimate_td;
    int lm0;   // first landmark of the window in the staged landmark arrays (lm_ref_node, lm_ref_kp, outputs)
    int off0;  // first entry of the window's obs_off (L + 1 entries, relative to obs0)
    int obs0;  // first observation of the window in the staged observation arrays
    int node0; // first node of the window in cam_pose
};
struct CullSrc {  // where the culling's lists sit: lm_ref_node, obs_off, obs_node, obs_factor, lm_ref_kp, obs_kp
    const int *ref, *off, *node, *fac;
    const float *rkp, *kp;
};
struct CullOut {  // one window's scalar outputs
    double R_bc[9], t_bc[3], td_bc;
    int ext_accepted, counts[5];
};
struct CullArgs {
    icg_camera cam;
    double std;
    const double *pose, *ext, *rho;  // the handle's parameters (capacity-strided by window)
    int pose_stride, rho_stride;     // doubles per window: 7 max_K, max_L
    const CullWin *win;
    const int *lm_ref_node, *obs_off, *obs_node;
    const float *lm_ref_kp, *obs_kp;
    CullOut *out;
    double *cam_pose, *lm_pw, *lm_depth;
    uint8_t *lm_outlier, *obs_outlier;
};

// one CTA of CULL_THREADS per window, on `stream`
cudaError_t launch_update_cull(const CullArgs &a, int n_windows, cudaStream_t stream);
// loads the kernel into the current context (landmark-shard groups load every kernel up front: ba.cu, preload_group_kernels)
cudaError_t preload_update_cull();

}  // namespace icg
