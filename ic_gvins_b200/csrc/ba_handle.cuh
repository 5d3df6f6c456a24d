// ba_handle.cuh -- the host side of the window solve's handle, shared by ba_handle.cu (lifecycle and the solve) and ba_keyframe.cu (the
// resident keyframe cycle).  Host code only: the kernels are reached through ba_dev.cuh.
#pragma once
#include <string.h>

#include <algorithm>
#include <vector>

#include "ba_cull.cuh"
#include "ba_dev.cuh"
#include "ba_vision.cuh"
#include "geom_core.cuh"

// ---- IMU sqrt information  U = LLT(cov^-1).matrixL().transpose(): the shared core of geom_core.cuh, so that the reintegration kernel
//      (preint.cu) writes the same U into the handle as the upload
inline bool host_imu_sqrt_info(const double *cov, double *U) {
    double work[675];
    return icg::gc::imu_sqrt_info(cov, U, work);
}

// pinned host staging + device array, released with its owner
template <typename T>
struct HostDev {
    T *h = nullptr, *d = nullptr;
    size_t n = 0;
    HostDev() = default;
    HostDev(const HostDev &) = delete;
    HostDev &operator=(const HostDev &) = delete;
    ~HostDev() { release(); }
    int alloc(size_t count) {  // n: the count of a completed allocation (0 before and after a failed one)
        if (cudaMallocHost(&h, sizeof(T) * count) != cudaSuccess) return ICG_ENOMEM;
        if (cudaMalloc(&d, sizeof(T) * count) != cudaSuccess) return ICG_ENOMEM;
        memset(h, 0, sizeof(T) * count);
        n = count;
        return ICG_OK;
    }
    void release() {
        if (h) cudaFreeHost(h);
        if (d) cudaFree(d);
        h = d = nullptr, n = 0;
    }
    cudaError_t up(cudaStream_t s, size_t count = 0) { return cudaMemcpyAsync(d, h, sizeof(T) * (count ? count : n), cudaMemcpyHostToDevice, s); }
    cudaError_t down(cudaStream_t s, size_t count = 0) { return cudaMemcpyAsync(h, d, sizeof(T) * (count ? count : n), cudaMemcpyDeviceToHost, s); }
};

// Byte offsets of consecutive slices of one staging buffer, each slice starting 16-byte aligned.  end: the end of the last slice; size():
// that end padded to 16 bytes
struct Layout {
    size_t end = 0;
    size_t size() const { return (end + 15) & ~(size_t) 15; }
    size_t take(size_t bytes) {
        const size_t o = size();
        end = o + bytes;
        return o;
    }
};

struct icg_ba {
    icg::BaCaps C;
    icg::BaDev D;
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t stream_cam = nullptr;  // the camera-only factors are linearised concurrently with the vision chain
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool own_stream = false;
    int nblk_vis = 0;
    int cur_windows = 0;
    size_t smem_cam, smem_solve, smem_schur;
    int ld_schur;
    int use_global_S;
    HostDev<icg::WinDims> dims;
    HostDev<icg::LmState> st;
    HostDev<double> pose, mix, ext, rho, imu_blob, imu_U, gnss_blh, gnss_std, lever, pose_prior, pose_prior_sinfo, mix_prior, mix_prior_std, marg_x0,
        marg_H0, marg_b0, marg_c0;
    HostDev<int> f_meta_s, vb_lm0, ref_nrun;  // lm_fidx: host-side packing helper only (record slot -> factor id)
    HostDev<double> f_const_s;
    HostDev<int> lm_off, lm_perm, lm_fidx, gnss_node, marg_type, marg_node, part_off, pair_ro, vis_ord, npairs;
    HostDev<uint8_t> f_active;
    std::vector<void *> dev_only;
    HostDev<double> scratch;  // single-factor evaluation
    HostDev<icg::LmState> st_save;   // pass-1 LM state of the two-pass protocol
    HostDev<int> cull_counters; // per window: reprojection factors removed, GNSS fixes re-weighted
    // split pipeline (ba_split.cuh): exchange buffer of this rank, peers' buffers opened through CUDA IPC, epoch counter of the flags
    double *xbuf = nullptr;
    size_t xbuf_doubles = 0;
    int x_world = 0;
    void *ipc_opened[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    unsigned long long epoch = 0;
    size_t smem_solve_cam = 0, smem_step_lm = 0;
    bool solve_cam_dsm = false;      // the packed system fits the cluster's shared memory: ba_solve_cam_dsm (max_K <= 23)
    size_t smem_solve_cam_dsm = 0;
    // in-situ stage timing (ICG_BA_PROFILE=1): events between the kernels of the LM sequence on the main stream, read back in
    // icg_ba_sync / icg_ba_download and printed by icg_ba_destroy (warm caches, real launch gaps -- unlike an ncu replay)
    bool prof = false;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int> prof_tag;
    size_t prof_used = 0;
    int prof_skip = 1;  // LM sequences to discard first (lazy module loading puts a one-off multi-ms cost on every kernel's first launch)
    double prof_ms[16] = {0};
    long prof_cnt[16] = {0};
    // marginalization workspace (allocated on the first icg_ba_marginalize call).  The parts sized by the marginalized block (H0, b0, G1,
    // V1, lam1, Z) follow the largest batch seen so far: marg_nw windows at the strides M.n0cap / M.mcap, grown on demand
    bool marg_ready = false;
    icg::MargDev M{};
    int marg_nw = 0;
    int marg_cluster_ok = -1;  // -1 not checked yet; 1: an 8-CTA marg_jacobi_cluster with its largest shared memory can be scheduled
    HostDev<int> marg_map;
    HostDev<double> marg_oJ0, marg_oe0, marg_oHp, marg_obp;
    HostDev<uint8_t> marg_fmask;  // factor set of icg_ba_marginalize_resident_culled (ba_lin_vis reads it in place of f_active)
    HostDev<unsigned char> marg_sel;  // icg_ba_marginalize_built's staging [MargSelWin | headers and block tables], grown on demand
    int *marg_ftab = nullptr;         // its device scratch (marg_select_built: NW x max_F ints), allocated on first use
    HostDev<unsigned char> cull;   // post-solve update + culling: staging [inputs | outputs], grown on demand
    HostDev<unsigned char> vis;    // icg_ba_slide_vision_resident's staging, grown on demand
    HostDev<unsigned char> reint;  // the reintegration's staging, grown on demand
    // ---- the keyframe cycle's results, each current from its one writer until it ends; a call rejected before that point leaves it as it
    //      was.  "Replaced": end_results, which icg_ba_upload calls after its argument check, and every slide once all its checks have passed
    void end_results() { culled.n = 0, built.n = 0, prior.n = 0, store.valid = false; }
    // the linearisation buffers hold the last single-GPU LM sequence's system (icg_ba_peek_linearization): made current by icg_ba_run /
    // icg_ba_run_gvins; ended by pack_windows (an upload, a slide) and at the start of every culling, marginalization and reintegration launch
    bool lin_ready = false;
    // the last culling (sharded: of the rank's shard; icg_ba_slide_vision_resident, icg_ba_marginalize_resident_culled): made current by a
    // successful cull_run; ended at cull_run's start and when replaced.  Window w's slices: win[w], nobs[w] observations.  Lists: dev (the
    // culling's staging with fac NULL, or the built lists), host (the built lists' host copies, else NULL); flags: the culling's staging
    struct CullResult {
        int n = 0;  // windows (0: none)
        std::vector<icg::CullWin> win;
        std::vector<int> nobs;
        icg::CullSrc dev{};
        const uint8_t *lm_outlier = nullptr, *obs_outlier = nullptr;
        icg::CullSrc host{};
    } culled;
    // the next culling's lists, built by icg_ba_slide_vision_resident (sharded: the rank's next shard's) into buf[cur ^ 1]: made current at
    // the end of vision_body, after its slide's commit; ended when replaced and by a shard export.  Each buffer is [lm_ref_node | obs_off |
    // obs_node | obs_factor | lm_ref_kp | obs_kp] at at[], sized by the slide's bounds (nL landmarks, nO observations); window w's slices are
    // win[w], with nobs[w] entries.  dev() / host(): the current buffer's lists / their host copies (a culling on them writes those)
    struct BuiltLists {
        struct At { size_t ref, off, node, fac, rkp, kp, end; };
        HostDev<unsigned char> buf[2];
        At at[2] = {};
        int cur = 0, n = 0;  // n: windows (0: none)
        size_t nL = 0, nO = 0;
        std::vector<icg::CullWin> win;
        std::vector<int> nobs;
        icg::CullSrc dev() const { return slices(buf[cur].d); }
        icg::CullSrc host() const { return slices(buf[cur].h); }
        icg::CullSrc slices(const unsigned char *p) const {
            const At &a = at[cur];
            return {(const int *) (p + a.ref), (const int *) (p + a.off), (const int *) (p + a.node), (const int *) (p + a.fac),
                    (const float *) (p + a.rkp), (const float *) (p + a.kp)};
        }
    } built;
    // the last resident marginalization, while its workspace (marg_oJ0 / marg_oe0) is the prior of the windows the handle holds (a slide's
    // prior_from_marg reads it): made current by prior_commit; ended by every marginalization before it writes the workspace, and when
    // replaced.  m, r, nb: every window's m, r and remained blocks.  sharded: a shard group's; window w's prior is then in the workspace of
    // mx_h (slot (w - rank) / world) on its owner, and the windows another rank owns keep m = r = nb = 0
    struct ResidentPrior {
        int n = 0;  // windows (0: none)
        bool sharded = false;
        std::vector<int> m, r, nb;
    } prior;
    // every IMU factor's samples (imu_buffer_): rows (dt, dtheta[3], dvel[3]) window after window, factor after factor, in d[cur].  store_build
    // cuts the next store from the INS windows into the other buffer; store_commit makes it current when icg_ba_imu_samples_from_ins or
    // icg_ba_slide_ins_resident (after its slide) commits.  Ended when replaced
    struct SampleStore {
        double *d[2] = {nullptr, nullptr};
        size_t cap[2] = {0, 0};  // rows
        int cur = 0;
        bool valid = false;
        std::vector<std::vector<int>> row0, nrow;  // per window and factor: first row, row count (-1: the factor has no samples)
        HostDev<unsigned char> stage;              // [cut jobs | row counts | statuses | gather segments], grown on demand
        double *cut = nullptr;                     // the series cut out of the INS windows, before the gather
        size_t cut_cap = 0;                        // rows
    } store;
    // icg_ba_slide_resident: staging (grown on demand), the copy of the old value rows, the second f_const_s buffer
    HostDev<unsigned char> slide;
    double *slide_old = nullptr, *fc_alt = nullptr;
    // icg_ba_slide_vision_resident: the structure tables ba_pack_structure writes (one allocation at f_meta_s, the handle's capacities and
    // strides), copied into the handle's when the slide commits
    icg::PackTables pack{};
    // every landmark's reference row pts0[3] | vel0[3] | td0 (NaN: unknown), 7 doubles at w L + l, and the buffer the next slide writes: set by
    // icg_ba_upload from the landmark's first factor, carried by every slide, read by icg_ba_slide_vision_resident
    double *lm_ref = nullptr, *lm_ref_alt = nullptr;
    cudaEvent_t slide_ev = nullptr;  // recorded after the staging's H2D
    cudaEvent_t ins_ev = nullptr;    // recorded on the INS handle's stream, waited on by this one (the sample store's cuts)
    // post-solve calls of a shard group (world > 1): integer exchanges so far (slot parity), epoch of the last marginalization export, the
    // exchange's device word, the export's slot lists, the owner's gathered rows with their tables, and the handle the owner uploads its
    // gathered windows to (created on first use, recreated when a batch needs more landmarks, factors or windows)
    unsigned long long xs_calls = 0, exp_epoch = 0;
    HostDev<int> xs_v, mx_sel, mx_row;
    HostDev<long long> mx_heads, mx_idx;
    double *mx_rows = nullptr;
    size_t mx_rows_cap = 0;
    icg_ba *mx_h = nullptr;
    // buffers a shard group's call outgrew.  Freeing synchronises the device, and between handles of one process that would wait for a
    // peer's kernel spinning on this rank's flags: they are freed when the group is left or the handle destroyed
    std::vector<void *> retired_d, retired_h;
    std::vector<icg_ba *> retired_mx;
};

// The launch configuration of grid CTAs of block threads in clusters of cx CTAs along x (cudaLaunchKernelEx, cluster occupancy queries)
struct ClusterLaunch {
    cudaLaunchConfig_t cfg{};
    cudaLaunchAttribute at[1];
    ClusterLaunch(unsigned grid, unsigned block, size_t smem, cudaStream_t s, unsigned cx) {
        cfg.gridDim = dim3(grid), cfg.blockDim = dim3(block), cfg.dynamicSmemBytes = smem, cfg.stream = s;
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = cx, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
        cfg.attrs = at, cfg.numAttrs = 1;
    }
    ClusterLaunch(const ClusterLaunch &) = delete;  // cfg points into at
};

// ---- shared by ba_handle.cu and ba_keyframe.cu
int dmalloc(icg_ba *h, double **p, size_t n);
cudaError_t launch_lm_ref_fill(icg_ba *h, int n, const icg::SlideWin *win, const int *map, const double *old, double *out);
int pack_windows(icg_ba *h, int n, const icg_ba_problem *P, bool values, bool vision = true);
int upload_structure(icg_ba *h, int n, bool vision = true);
int keep_pristine(icg_ba *h, int n);
void retire(icg_ba *h, void *d, void *hp);
// shard groups (world > 1, ba_split.cuh); fn: the calling entry point, for the error messages
int shard_timed_out(icg_ba *h, const char *what);
int shard_xsum(icg_ba *h, int *v, int stride, int n, int nv, int op);
int shard_xmax(icg_ba *h, int *v3, const char *fn);
int shard_agree(icg_ba *h, bool rejected, int fp, const char *fn);

// b holds at least count elements: a buffer that is too small is retired and replaced by one 1.25 times the request.  No synchronisation:
// the caller waits for earlier work on the old buffer where it needs to (in a shard group a wait here could block on a peer's kernel)
template <typename T>
int hd_reserve(icg_ba *h, HostDev<T> &b, size_t count, const char *fn) {
    if (b.d && b.n >= count) return ICG_OK;
    retire(h, b.d, b.h);  // earlier launches may still use the old buffers
    b.d = b.h = nullptr, b.n = 0;
    const size_t cap = std::max<size_t>(16, count + count / 4);
    if (b.alloc(cap) != ICG_OK) {
        icg::set_error("%s: staging allocation of %zu bytes failed", fn, sizeof(T) * cap);
        return ICG_ENOMEM;
    }
    return ICG_OK;
}
