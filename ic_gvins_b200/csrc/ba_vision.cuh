// ba_vision.cuh -- the vision half of the next window (icg_ba_slide_vision_resident and its sharded form): GVINS::addReprojectionParameters +
// addReprojectionFactors (IG/ic_gvins.cc:1697-1837) after Map::removeKeyFrame(frame, true) (tracking/map.cc:89-125), built on the device from
// the culled window the handle holds and the new keyframes' observations.  The interface between the handle (ba.cu: validation, staging,
// the slide) and the kernel (ba_vision.cu, built without FMA contraction so that pixel2cam is the host's sub-then-divide).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/icgvins_b200.h"

namespace icg {

constexpr int VIS_THREADS = 256;
constexpr int VIS_MAX_NODES = 32;   // = the handle's max_K limit (one bit per node in the per-landmark masks)
constexpr int VIS_MAX_FRAMES = 64;  // frame id -> node table entries

// one window, as staged.  Old-window arrays are the handle's (capacity-strided) and the last culling's staging; new-keyframe arrays are the
// caller's DEVICE pointers.  Every output and scratch offset is in elements of its own array.
struct VisWin {
    icg_camera cam;
    double node_td[VIS_MAX_NODES];     // next-window node -> timeDelay()
    int8_t onode[VIS_MAX_NODES];       // old node -> next node, -1: marginalized, removed or not in the map
    int64_t frame_id[VIS_MAX_FRAMES];  // frame table of the new map points' reference frames
    int frame_node[VIS_MAX_FRAMES];
    int oK, oL, oF, nK, n_frames, cur_node;
    int cull_lm0, cull_off0, cull_obs0, n_cull_obs;  // the window's slices of the last culling's lists and flags
    const int *obs_factor;                            // the window's obs_factor (n_cull_obs entries): the caller's, staged, or the built lists'
    // tracked observations: k < count (*dev_n when given, else n_obs), j = src ? src[k] : k (j < n_in); lm = obs_lm[j], node = obs_node[j]
    // (obs_node NULL: cur_node); undis_xy / vel at k
    int n_obs, n_in;
    const int *dev_n, *src, *obs_node, *obs_lm;
    const float *obs_xy;
    const double *obs_vel;
    // new map points: j < count (*dev_new_n when given, else n_new)
    int n_new;
    const int *dev_new_n;
    const double *new_depth, *new_vel_ref, *new_vel_cur;
    const float *new_ref_xy, *new_cur_xy;
    const int64_t *new_ref_frame;
    // bounds: next landmarks Lb = oL + n_new, next factors Fb = oF + n_obs + n_new, new factors Nb = n_obs + n_new
    int lm_out, f_out, nf_out, scr;  // offsets of the window's output rows (Lb, Fb, Nb) and int scratch
    int lst_obs;                     // the next culling's lists: first entry of the window's observations (Ob = n_cull_obs + n_obs + 2 n_new)
    int pscr;                        // ba_pack_structure's int scratch (5 Lb + Fb + oF + NVB)
};

// per window: [L, F, new factors, error code, error index, landmarks dropped for a NaN inverse depth, the observation count and the new-point
// count the kernel read (a landmark shard's ranks must read the same), the entries of the next culling's lists (0 when they are not emitted),
// the landmark and observing node of a VIS_EPACK_DUP factor]
constexpr int VIS_COUNTS = 11;
// VIS_EPACK_*: ba_pack_structure's rejections, the checks of icg_ba_upload's packing the build does not make (error index: the factor of a
// landmark with two reference nodes or two observations in one node; the landmark that starts a run of more than 128 factors or that the run
// table has no room for)
enum VisError {
    VIS_OK = 0, VIS_EOBS_FACTOR = 1, VIS_ECOUNT = 2, VIS_ESRC = 3, VIS_ENODE = 4, VIS_ELM = 5, VIS_EDUP = 6, VIS_EFRAME = 7, VIS_EROW = 8,
    VIS_EPACK_DUP = 9, VIS_EPACK_LM128 = 10, VIS_EPACK_RUNS = 11
};

struct VisArgs {
    const VisWin *win;
    int K, L, F;      // the handle's capacities (strides of its arrays)
    int rank, world;  // landmark shards: new map point j of window w is built on rank (j + w) mod world only (one GPU: 0, 1)
    // the window the handle holds
    const double *rho;
    const int *f_meta_s, *lm_off, *lm_perm;
    const double *lm_ref;  // per landmark: its reference row pts0[3] | vel0[3] | td0 (NaN: unknown), capacity-strided (7 L per window)
    // the last culling: its lists (the host lists it staged, or the lists the last slide built) and its flags
    const int *lm_ref_node, *obs_off, *obs_node;
    const float *lm_ref_kp, *obs_kp;
    const uint8_t *lm_outlier, *obs_outlier;
    // outputs: counts (VIS_COUNTS per window), per next landmark lm_src, its origin (old landmark, or -(j + 1) for new map point j) and
    // invdepth, per old landmark and new map point a NaN-drop flag (Lb bytes), per next factor f_lm / f_ref / f_obs / f_src, per new factor
    // its 14 constants (the new factors in factor order); lm_ref_next: the next window's reference rows (capacity-strided, as lm_ref)
    int *counts, *lm_src, *lm_org, *f_lm, *f_ref, *f_obs, *f_src;
    uint8_t *lm_nan;
    double *invdepth, *f_new, *lm_ref_next;
    int *scratch;
    // the next culling's lists (NULL: not emitted); on a landmark shard the rank's next shard's, in its numbering.  Per window, in
    // next-landmark order: l_ref / l_rkp at lm_out (Lb), l_off at lm_out + w (Lb + 1), l_node / l_fac / l_kp at lst_obs (Ob); keypoints 2
    // floats each
    int *l_ref, *l_off, *l_node, *l_fac;
    float *l_rkp, *l_kp;
};

cudaError_t launch_vision(const VisArgs &a, int n_windows, cudaStream_t stream);

// The structure tables of the built windows, as icg_ba_upload packs them (ba_handle.cu, pack_window), into second buffers at the handle's
// strides.  The slide makes them the handle's once every check has passed.
struct PackTables {
    int *f_meta_s, *vb_lm0, *lm_off, *lm_perm, *ref_nrun, *part_off, *pair_ro, *vis_ord, *npairs;
    uint8_t *f_active;
};

struct PackArgs {
    const VisWin *win;
    int K, L, F, NVB;   // the handle's capacities and run-table stride
    int *counts;        // ba_vision_build's (L, F and its error code are read; a packing error is written there)
    const int *lm_src, *f_lm, *f_ref, *f_obs, *f_src;  // ba_vision_build's rows
    const int *old_meta;                                // the handle's f_meta_s: the old window's slot -> factor table
    PackTables out;
    // per window: the slot -> factor table at f_out (the host's copy); the slide's maps, landmarks at lm_out, record slots at nL + f_out:
    // m >= 0 the old landmark / slot carried, m < 0 the row at -(m + 1) of ba_vision_build's invdepth / f_new (doubles)
    int *fidx, *map;
    int nL;
    int *scratch;
};

// ba_pack_structure, one CTA per window, after ba_vision_build on the same stream; a window the build rejected or that exceeds the handle is
// skipped
cudaError_t launch_pack(const PackArgs &a, int n_windows, cudaStream_t stream);

}  // namespace icg
