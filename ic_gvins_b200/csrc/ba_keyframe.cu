// ba_keyframe.cu -- host side of the resident keyframe cycle on a window-solve handle (ba_handle.cuh): after the solve, the windows stay on
// the device for the map update and outlier culling (ba_cull.cu), the reintegration of their IMU factors (preint.cu), the marginalization
// (ba_marg.cuh) and the slide to the next keyframe's windows (ba_slide.cu, ba_vision.cu), on one GPU or across a landmark-shard group.
#include <functional>
#include <memory>
#include <string>
#include <thread>

#include "ba_handle.cuh"
#include "ba_vision.cuh"
#include "ins_handle.cuh"
#include "preint.cuh"

using namespace icg;

namespace {
// 31-bit fingerprint of the arguments a collective call requires to be the same on every rank (FNV-1a over 64-bit words)
struct ArgPrint {
    uint64_t v = 1469598103934665603ull;
    void bytes(const void *p, size_t n) {
        const unsigned char *c = (const unsigned char *) p;
        size_t i = 0;
        for (uint64_t x; i + 8 <= n; i += 8) memcpy(&x, c + i, 8), v = (v ^ x) * 1099511628211ull;
        for (; i < n; i++) v = (v ^ c[i]) * 1099511628211ull;
    }
    template <typename T>
    void arr(const T *p, long long count) {
        if (p && count > 0) bytes(p, sizeof(T) * (size_t) count);
    }
    void num(long long x) { bytes(&x, sizeof(x)); }
    int get() const { return (int) ((v ^ (v >> 31) ^ (v >> 62)) & 0x7fffffff); }
};
}  // namespace

// ---- marginalization (B10)
constexpr int MARG_MAXN = 512;  // rows of the largest block an eigensolver takes (marg_jacobi: RPL = 16 rows per lane)

// The parts of the workspace that do not depend on the batch: the structure map, the outputs (rcap = N per window), the Jacobi workspace
// of Hp (n = r <= N) and the saved flags
static int marg_alloc(icg_ba *h) {
    if (h->marg_ready) return ICG_OK;
    const BaCaps &C = h->C;
    MargDev &M = h->M;
    const size_t NW = C.NW;
    M.rcap = C.N, M.mcap = 0, M.n0cap = 0;
    M.map_stride = MARG_MAP_HDR + 2 * C.K + C.L;
    if (h->marg_map.alloc(NW * M.map_stride) != ICG_OK || h->marg_oJ0.alloc(NW * (size_t) M.rcap * M.rcap) != ICG_OK || h->marg_oe0.alloc(NW * M.rcap) != ICG_OK ||
        h->marg_oHp.alloc(NW * (size_t) M.rcap * M.rcap) != ICG_OK || h->marg_obp.alloc(NW * M.rcap) != ICG_OK || h->marg_fmask.alloc(NW * C.F) != ICG_OK) {
        set_error("icg_ba_marginalize: workspace allocation failed");
        return ICG_ENOMEM;
    }
    M.map = h->marg_map.d, M.J0 = h->marg_oJ0.d, M.e0 = h->marg_oe0.d, M.Hp = h->marg_oHp.d, M.bp = h->marg_obp.d;
    int rc = ICG_OK;
    double *fl = nullptr;
#define DM(ptr, count) \
    if (rc == ICG_OK) rc = dmalloc(h, &ptr, count);
    DM(M.G2, NW * (size_t) M.rcap * M.rcap) DM(M.V2, NW * (size_t) M.rcap * M.rcap) DM(M.lam2, NW * M.rcap) DM(fl, NW * 2)
#undef DM
    if (rc != ICG_OK) return rc;
    M.flags = (int *) fl;
    const size_t smem = sizeof(double) * (8 * 480 + 2 * (size_t) C.R) + sizeof(int) * (size_t) C.R + 64;
    ICG_CUDA(raise_dynamic_smem((const void *) marg_assemble, (size_t) (smem)));
    h->marg_ready = true;
    return ICG_OK;
}

// The parts sized by the marginalized block: H0 / b0 (n0 = m + r), G1 / V1 / lam1 (m), Z (m (rcap + 1)) for n windows.  They grow to the
// batch's maxima when a batch needs more than the last allocation (strides only: the kernels index window w's slot by them and touch the
// n0^2 / m^2 leading entries, so the results do not depend on them).
static int marg_grow(icg_ba *h, int n, int max_m, int max_n0) {
    MargDev &M = h->M;
    if (n <= h->marg_nw && max_m <= M.mcap && max_n0 <= M.n0cap) return ICG_OK;
    const int nw = std::max(n, h->marg_nw), mcap = std::max(max_m, M.mcap), n0cap = std::max(max_n0, M.n0cap);
    ICG_CUDA(cudaStreamSynchronize(h->stream));  // earlier launches on the handle's stream may still read the old buffers
    for (double **p : {&M.H0, &M.b0, &M.G1, &M.V1, &M.lam1, &M.Z}) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    h->marg_nw = 0, M.mcap = 0, M.n0cap = 0;
    const size_t NW = nw;
    const size_t count[6] = {NW * n0cap * n0cap, NW * n0cap, NW * mcap * mcap, NW * mcap * mcap, NW * mcap, NW * mcap * (M.rcap + 1)};
    double **ptr[6] = {&M.H0, &M.b0, &M.G1, &M.V1, &M.lam1, &M.Z};
    for (int k = 0; k < 6; k++) {
        if (cudaMalloc(ptr[k], sizeof(double) * std::max<size_t>(1, count[k])) != cudaSuccess) {
            *ptr[k] = nullptr;
            set_error("icg_ba_marginalize: workspace allocation of %zu doubles failed (%d windows, m <= %d, m + r <= %d)", count[k], nw, mcap, n0cap);
            return ICG_ENOMEM;
        }
        ICG_CUDA(cudaMemsetAsync(*ptr[k], 0, sizeof(double) * std::max<size_t>(1, count[k]), h->stream));
    }
    h->marg_nw = nw, M.mcap = mcap, M.n0cap = n0cap;
    return ICG_OK;
}

// a resident marginalization succeeded: its record of windows first, first + step, ... (step > 1: those a shard group's rank owns)
static void prior_commit(icg_ba *h, int n, const icg_ba_prior *out, int first, int step) {
    icg_ba::ResidentPrior &P = h->prior;
    P.m.assign(n, 0), P.r.assign(n, 0), P.nb.assign(n, 0);
    for (int w = first; w < n; w += step) P.m[w] = out[w].m, P.r[w] = out[w].r, P.nb[w] = out[w].nblocks;
    P.n = n, P.sharded = step > 1;
}

// The blocks the camera-side factors of the marginalization touch (MarginalizationInfo::addResidualBlockInfo, marginalization_info.h:103-121):
// the preintegration factors k < num_marg (factor k joins node k and node k + 1), GNSS at the removed nodes, the first-window priors and the
// previous prior's blocks.  tp / tm: K flags each, set (never cleared) here; ext / td: the previous prior names them
static void marg_camera_touched(const icg_ba_problem &p, int nm, char *tp, char *tm, bool *ext, bool *td) {
    for (int k = 0; k < nm && k < p.n_imu; k++) tp[k] = tm[k] = tp[k + 1] = tm[k + 1] = 1;
    for (int g = 0; g < p.n_gnss; g++)
        if (p.gnss_node[g] < nm) tp[p.gnss_node[g]] = 1;
    if (p.has_pose_prior) tp[0] = 1;
    if (p.has_mix_prior) tm[0] = 1;
    for (int b = 0; b < p.marg_nblocks && p.marg_r > 0; b++) {
        const int t = p.marg_block_type[b], nd = p.marg_block_node[b];
        if (t == 0) tp[nd] = 1;
        else if (t == 1) tm[nd] = 1;
        else if (t == 2) *ext = true;
        else *td = true;
    }
}

// num_marg and the output arrays of window w (every entry point checks them before anything is written)
static bool marg_out_ok(const icg_ba_problem &p, int nm, const icg_ba_prior &o) {
    return nm >= 1 && nm < p.K && o.block_type && o.block_node && o.x0 && o.J0 && o.e0 && o.rcap >= 15 * (p.K - nm) + 7;
}

static int marg_solve(icg_ba *h, int n, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out, bool resident,
                      const uint8_t *const *fmask, const std::function<int(int *)> *agree, bool dev_structure);

// fmask (resident only, may be NULL): per window, the factor set to marginalize in place of the problem's activity (F bytes each); it reaches
// ba_lin_vis through a copy of the device view, so the handle's own f_active is never written.
// agree (may be NULL): called once the structure is known, with {largest m, largest r, 1 if a window is rejected} of this batch; it returns
// the values the eigensolver kernels are chosen by (the owner of a shard group's windows takes the group's maxima, so that it runs the
// kernels an unsharded handle holding the whole batch runs).  It is called on the rejection path too, so that no peer is left waiting.
static int marginalize_body(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out, bool resident,
                            const uint8_t *const *fmask = nullptr, const std::function<int(int *)> *agree = nullptr) {
    if (!h || !problems || !num_marg || !out || n_windows < 1 || n_windows > h->C.NW) {
        set_error("icg_ba_marginalize: bad arguments");
        return ICG_EINVAL;
    }
    if (h->D.world > 1) {
        set_error("icg_ba_marginalize: not available on a landmark-sharded handle (icg_ba_shard_leave first)");
        return ICG_EUNSUPPORTED;
    }
    int rc = ICG_OK;
    h->prior.n = 0;  // the workspace is about to be overwritten: it is the resident prior again only if this call is resident and succeeds
    h->lin_ready = false;  // its linearisation takes the buffer the window uses
    if (resident) {
        // the windows of the last upload / solve are still on the device (parameters at their optimised values, factor activity and GNSS
        // weights as the two-pass solve left them): `problems` is read for the structure and for x0 only
        if (h->cur_windows != n_windows) {
            set_error("icg_ba_marginalize_resident: the handle holds %d uploaded windows, the call names %d", h->cur_windows, n_windows);
            return ICG_EINVAL;
        }
        ICG_CUDA(cudaSetDevice(h->device));
    } else {
        rc = icg_ba_upload(h, n_windows, problems);
        if (rc != ICG_OK) return rc;
    }
    rc = marg_alloc(h);
    if (rc != ICG_OK) return rc;
    const BaCaps &C = h->C;
    MargDev &M = h->M;
    const int n = n_windows;
    // ---- updateParameterBlocksIndex (marginalization_info.h:228-251) on the host: structure only.  The reference iterates
    //      unordered_maps (implementation-defined order inside each group); here: marginalized = [pose_k, mix_k (k < num_marg),
    //      landmarks ascending], remained = [pose_k, mix_k (k >= num_marg, only blocks some factor touches), ext, td].
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const int nm = num_marg[w];
        icg_ba_prior &o = out[w];
        if (!marg_out_ok(p, nm, o)) {
            set_error("icg_ba_marginalize: window %d: num_marg=%d out of range or output arrays missing / too small (rcap=%d)", w, nm, o.rcap);
            return ICG_EINVAL;
        }
        int *map = h->marg_map.h + (size_t) w * M.map_stride;
        int *pose_col = map + MARG_MAP_HDR, *mix_col = pose_col + C.K, *lm_col = mix_col + C.K;
        std::vector<char> tp(p.K, 0), tm(p.K, 0), tl(p.L, 0);
        const uint8_t *act = fmask ? fmask[w] : p.f_active;
        if (fmask) memcpy(h->marg_fmask.h + (size_t) w * C.F, act, p.F);
        bool any_vis = false;
        for (int f = 0; f < p.F; f++) {
            if ((act && !act[f]) || p.f_ref[f] >= nm) continue;
            tl[p.f_lm[f]] = 1, tp[p.f_obs[f]] = 1, any_vis = true;
        }
        bool has_ext = any_vis, has_td = any_vis;
        // a block exists in the marginalization problem only if some factor touches it (MarginalizationInfo::addResidualBlockInfo,
        // marginalization_info.h:103-121): removed nodes without any factor get no columns
        for (int f = 0; f < p.F; f++)
            if (!(act && !act[f]) && p.f_ref[f] < nm) tp[p.f_ref[f]] = 1;
        marg_camera_touched(p, nm, tp.data(), tm.data(), &has_ext, &has_td);
        int idx = 0;
        for (int k = 0; k < C.K; k++) pose_col[k] = mix_col[k] = -1;
        for (int k = 0; k < nm; k++) {
            if (tp[k]) pose_col[k] = idx, idx += 6;
            if (tm[k]) mix_col[k] = idx, idx += 9;
        }
        for (int l = 0; l < C.L; l++) lm_col[l] = -1;
        for (int l = 0; l < p.L; l++)
            if (tl[l]) lm_col[l] = idx++;
        const int m = idx;
        int nb = 0, xo = 0;
        for (int k = nm; k < p.K; k++) {
            if (tp[k]) pose_col[k] = idx, idx += 6, o.block_type[nb] = 0, o.block_node[nb++] = k - nm, xo += 7;
            if (tm[k]) mix_col[k] = idx, idx += 9, o.block_type[nb] = 1, o.block_node[nb++] = k - nm, xo += 9;
        }
        int ext_col = -1, td_col = -1;
        if (has_ext) ext_col = idx, idx += 6, o.block_type[nb] = 2, o.block_node[nb++] = 0, xo += 7;
        if (has_td) td_col = idx, idx += 1, o.block_type[nb] = 3, o.block_node[nb++] = 0, xo += 1;
        // a reprojection factor always carries ext and td columns; give them (unused) columns when only camera factors exist
        if (ext_col < 0) ext_col = 0;
        if (td_col < 0) td_col = 0;
        map[0] = m, map[1] = idx - m, map[2] = idx, map[3] = nm, map[4] = ext_col, map[5] = td_col, map[6] = map[7] = 0;
        o.m = m, o.r = idx - m, o.nblocks = nb;
        // checked before anything is launched: a rejected call leaves the device state of the handle as it was
        if (m > MARG_MAXN || idx - m > MARG_MAXN) {
            if (agree) {
                int mx[3] = {0, 0, 1};
                (*agree)(mx);
            }
            set_error("icg_ba_marginalize: window %d: %s=%d exceeds the %d rows of the largest eigensolver kernel", w, m > MARG_MAXN ? "m" : "r",
                      m > MARG_MAXN ? m : idx - m, MARG_MAXN);
            return ICG_EUNSUPPORTED;
        }
    }
    return marg_solve(h, n, problems, num_marg, out, resident, fmask, agree, false);
}

// The launch sequence of every marginalization once the batch's structure is known: out[w]'s m, r, nblocks and block tables, and the column
// map -- in marg_map's host half (and the factor set in marg_fmask's when fmask is given), uploaded here, or already on the device
// (dev_structure: marg_select_built wrote both).  Then the eigensolver kernels the batch's largest blocks select, the prior's D2H and the
// write-back into out, x0 from problems' camera side.
static int marg_solve(icg_ba *h, int n, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out, bool resident,
                      const uint8_t *const *fmask, const std::function<int(int *)> *agree, bool dev_structure) {
    const BaCaps &C = h->C;
    MargDev &M = h->M;
    int rc = ICG_OK;
    int max_m = 0, max_r = 0, max_n0 = 0;
    for (int w = 0; w < n; w++) max_m = std::max(max_m, out[w].m), max_r = std::max(max_r, out[w].r), max_n0 = std::max(max_n0, out[w].m + out[w].r);
    int sel_m = max_m, sel_r = max_r;  // what the eigensolver kernels are chosen by
    if (agree) {
        int mx[3] = {max_m, max_r, 0};
        rc = (*agree)(mx);
        if (rc != ICG_OK) return rc;
        if (mx[2]) {
            set_error("icg_ba_marginalize_resident: a window owned by another rank of the shard group was rejected (see that rank's error)");
            return ICG_EUNSUPPORTED;
        }
        sel_m = mx[0], sel_r = mx[1];
    }
    rc = marg_grow(h, n, max_m, max_n0);
    if (rc != ICG_OK) return rc;
    cudaStream_t s = h->stream;
    if (h->marg_cluster_ok < 0) {  // once per handle: can an 8-CTA marg_jacobi_cluster with the largest shared-memory slices be placed at all?
        const size_t csm = marg_cluster_smem(MARG_CLUSTER_MAXN);
        ICG_CUDA(raise_dynamic_smem((const void *) marg_jacobi_cluster, csm));
        const ClusterLaunch L(MARG_CLUSTER_CTAS, MARG_CLUSTER_THREADS, csm, s, MARG_CLUSTER_CTAS);
        int nclusters = 0;
        h->marg_cluster_ok = cudaOccupancyMaxActiveClusters(&nclusters, marg_jacobi_cluster, &L.cfg) == cudaSuccess && nclusters > 0 ? 1 : 0;
        cudaGetLastError();  // a refused query is an answer (the global kernel takes those blocks), not an error of this call
    }
    if (!dev_structure) ICG_CUDA(h->marg_map.up(s, (size_t) n * M.map_stride));
    BaDev D = h->D;
    if (fmask || dev_structure) {
        if (!dev_structure) ICG_CUDA(h->marg_fmask.up(s, (size_t) n * C.F));
        D.f_active = h->marg_fmask.d;
    }
    const size_t smem = sizeof(double) * (8 * 480 + 2 * (size_t) C.R) + sizeof(int) * (size_t) C.R + 64;
    marg_prepare<<<(n + 127) / 128, 128, 0, s>>>(D, M, n, 0);
    ba_lin_vis<<<dim3(C.NVB - 2, n), 128, LV_SMEM, s>>>(C, D, 0);
    marg_assemble<<<n, 256, smem, s>>>(C, D, M);
    // eigendecompositions: one kernel per stage serves the whole batch, chosen by the batch's largest block --
    //   n <= MARG_CTA_MAXN: one CTA;  n <= MARG_PAIR_MAXN: cluster pair;  n <= MARG_CLUSTER_MAXN: 8-CTA cluster;  otherwise: global memory.
    // ICG_MARG_GLOBAL_JACOBI forces the global kernel, ICG_MARG_PAIR_JACOBI skips the one-CTA kernel, ICG_MARG_CLUSTER_JACOBI takes the
    // 8-CTA cluster for any n it supports.
    auto jacobi = [&](int which, int nmax) -> int {
        const bool cluster_ok = nmax <= MARG_CLUSTER_MAXN && h->marg_cluster_ok == 1;
        if (cluster_ok && !getenv("ICG_MARG_GLOBAL_JACOBI") && (getenv("ICG_MARG_CLUSTER_JACOBI") || nmax > MARG_PAIR_MAXN)) {
            const size_t smem = marg_cluster_smem(nmax);
            const ClusterLaunch L((unsigned) (MARG_CLUSTER_CTAS * n), MARG_CLUSTER_THREADS, smem, s, MARG_CLUSTER_CTAS);
            ICG_CUDA(cudaLaunchKernelEx(&L.cfg, marg_jacobi_cluster, M, which));
        } else if (nmax <= MARG_CTA_MAXN && !getenv("ICG_MARG_GLOBAL_JACOBI") && !getenv("ICG_MARG_PAIR_JACOBI")) {
            const size_t smem = sizeof(double) * 2 * (size_t) nmax * nmax;
            ICG_CUDA(raise_dynamic_smem((const void *) marg_jacobi_cta, smem));
            marg_jacobi_cta<<<n, MARG_CTA_THREADS, smem, s>>>(M, which);
        } else if (nmax <= MARG_PAIR_MAXN && !getenv("ICG_MARG_GLOBAL_JACOBI")) {
            const size_t smem = sizeof(double) * ((size_t) nmax * nmax + 2 * (size_t) (nmax + 2));
            const ClusterLaunch L((unsigned) (2 * n), MARG_THREADS, smem, s, 2);
            ICG_CUDA(raise_dynamic_smem((const void *) marg_jacobi_pair, (size_t) (smem)));
            ICG_CUDA(cudaLaunchKernelEx(&L.cfg, marg_jacobi_pair, M, which));
        } else {
            marg_jacobi<<<n, MARG_THREADS, 0, s>>>(M, which);
        }
        return ICG_OK;
    };
    rc = jacobi(0, sel_m);
    if (rc != ICG_OK) return rc;
    marg_schur<<<n, MARG_THREADS, 0, s>>>(M);
    rc = jacobi(1, sel_r);
    if (rc != ICG_OK) return rc;
    marg_finish<<<n, MARG_THREADS, 0, s>>>(M);
    marg_prepare<<<(n + 127) / 128, 128, 0, s>>>(D, M, n, 1);
    ICG_CHECK_LAUNCH();
    count_launch(9);
    // D2H: every window's r x r result sits at the start of its rcap^2 slot -- move the used prefix of each slot only (one strided copy)
    {
        const size_t pitch = sizeof(double) * (size_t) M.rcap * M.rcap, used = sizeof(double) * (size_t) max_r * max_r;
        bool want_Hp = false;
        for (int w = 0; w < n; w++) want_Hp = want_Hp || out[w].Hp != nullptr;
        if (used) ICG_CUDA(cudaMemcpy2DAsync(h->marg_oJ0.h, pitch, h->marg_oJ0.d, pitch, used, (size_t) n, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(h->marg_oe0.down(s, (size_t) n * M.rcap));
        if (want_Hp && used) ICG_CUDA(cudaMemcpy2DAsync(h->marg_oHp.h, pitch, h->marg_oHp.d, pitch, used, (size_t) n, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(h->marg_obp.down(s, (size_t) n * M.rcap));
    }
    ICG_CUDA(cudaStreamSynchronize(s));
    auto write_back = [&](int w) {
        const icg_ba_problem &p = problems[w];
        icg_ba_prior &o = out[w];
        const int nm = num_marg[w], r = o.r;
        // preMarginalization copies the parameter data of every block: x0 of the remained blocks (marginalization_info.h:270-283)
        int xo = 0;
        for (int b = 0; b < o.nblocks; b++) {
            const int t = o.block_type[b], nd = o.block_node[b] + nm;
            const double *src = t == 0 ? p.pose + 7 * nd : t == 1 ? p.mix + 9 * nd : t == 2 ? p.ext : p.ext + 7;
            const int gs = t == 1 ? 9 : t == 3 ? 1 : 7;
            memcpy(o.x0 + xo, src, sizeof(double) * gs);
            xo += gs;
        }
        if (o.m <= 0) return;
        memcpy(o.J0, h->marg_oJ0.h + (size_t) w * M.rcap * M.rcap, sizeof(double) * (size_t) r * r);
        memcpy(o.e0, h->marg_oe0.h + (size_t) w * M.rcap, sizeof(double) * r);
        if (o.Hp) memcpy(o.Hp, h->marg_oHp.h + (size_t) w * M.rcap * M.rcap, sizeof(double) * (size_t) r * r);
        if (o.bp) memcpy(o.bp, h->marg_obp.h + (size_t) w * M.rcap, sizeof(double) * r);
    };
    {   // the copies into the caller's arrays are memcpy-bound (r^2 doubles per window): a few host threads, like the packing of icg_ba_upload
        const int nthreads = std::max(1, std::min({n / 8, 8, (int) std::thread::hardware_concurrency()}));
        auto worker = [&](int t) {
            for (int w = t; w < n; w += nthreads) write_back(w);
        };
        std::vector<std::thread> th;
        for (int t = 1; t < nthreads; t++) th.emplace_back(worker, t);
        worker(0);
        for (auto &x : th) x.join();
    }
    if (resident) prior_commit(h, n, out, 0, 1);  // icg_ba_slide_resident(prior_from_marg = 1) takes this prior from the workspace
    return ICG_OK;
}

// The resident marginalization on a landmark-sharded handle, a collective call: every rank exports the rows of its factors with
// f_ref < num_marg (ba_marg_export); the owner of window w (w mod world) gathers the world exports of w in rank order -- global landmark
// order, since the landmarks are block-partitioned and each rank lists its factors landmark by landmark --, packs the gathered windows' integer
// structure into a handle of its own (nothing of their values goes through the host: ba_marg_fill copies the gathered rows and the shard
// handle's resident camera side on the device), and runs the single-GPU marginalization there.  That handle packs the
// gathered window exactly as an unsharded handle packs the marginalized part of the whole window (runs, Gram partials and pairs of the
// reference nodes < num_marg depend on those landmarks only), so the prior is the unsharded one, bit for bit.
static int marginalize_sharded(icg_ba *h, int n, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out, const uint8_t *const *fmask,
                               const char *fn) {
    const BaCaps &C = h->C;
    const int G = h->D.world, R = h->D.rank;
    if (!problems || !num_marg || !out || n < 1 || n > C.NW) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->cur_windows != n) {
        set_error("%s: the handle holds %d uploaded windows, the call names %d", fn, h->cur_windows, n);
        return ICG_EINVAL;
    }
    for (int r = 0; r < G; r++)
        if (!h->D.S.peer[r]) {
            set_error("%s: peer %d is not connected (icg_ba_shard_connect)", fn, r);
            return ICG_EINVAL;
        }
    // every check before anything is launched: a rank that returns here leaves its peers to the bounded waits
    size_t n_sel = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const WinDims &d = h->dims.h[w];
        const icg_ba_prior &o = out[w];
        if (p.K != d.K || p.L != d.L || p.F != d.F || (p.F > 0 && (!p.f_lm || !p.f_ref || !p.f_obs))) {
            set_error("%s: window %d does not describe the uploaded shard (K=%d L=%d F=%d)", fn, w, p.K, p.L, p.F);
            return ICG_EINVAL;
        }
        if (num_marg[w] < 1 || num_marg[w] >= p.K || !o.block_type || !o.block_node || !o.x0 || !o.J0 || !o.e0 || o.rcap < 15 * (p.K - num_marg[w]) + 7) {
            set_error("%s: window %d: num_marg=%d out of range or output arrays missing / too small (rcap=%d)", fn, w, num_marg[w], o.rcap);
            return ICG_EINVAL;
        }
        for (int f = 0; f < p.F; f++) {
            if (f > 0 && p.f_lm[f] < p.f_lm[f - 1]) {
                set_error("%s: window %d factor %d: a landmark-sharded window must list its factors landmark by landmark (f_lm non-decreasing)", fn, w, f);
                return ICG_EINVAL;
            }
            n_sel += p.f_ref[f] < num_marg[w];
        }
    }
    ICG_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    int rc = marg_alloc(h);  // marg_fmask: the culled factor set the export reads
    if (rc != ICG_OK) return rc;
    if ((rc = hd_reserve(h, h->mx_sel, n_sel + n + 1, fn)) != ICG_OK) return rc;
    int *sel = h->mx_sel.h, *sel_off = sel + n_sel;
    {   // the record slots of the exported factors, in factor order (the inverse of the packing's slot -> factor table)
        size_t at = 0;
        std::vector<int> slot_of;
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = problems[w];
            slot_of.assign(p.F, 0);
            const int *fidx = h->lm_fidx.h + (size_t) w * C.F;
            for (int q = 0; q < p.F; q++) slot_of[fidx[q]] = q;
            sel_off[w] = (int) at;
            for (int f = 0; f < p.F; f++)
                if (p.f_ref[f] < num_marg[w]) sel[at++] = slot_of[f];
            if (fmask) memcpy(h->marg_fmask.h + (size_t) w * C.F, fmask[w], p.F);
        }
        sel_off[n] = (int) at;
    }
    ICG_CUDA(h->mx_sel.up(s, n_sel + n + 1));
    if (fmask) ICG_CUDA(h->marg_fmask.up(s, (size_t) n * C.F));
    const unsigned long long epoch = ++h->epoch;
    ba_marg_export<<<n, 128, 0, s>>>(C, h->D, h->mx_sel.d, h->mx_sel.d + n_sel, fmask ? h->marg_fmask.d : nullptr, h->exp_epoch);
    ba_xflag<<<1, 32, 0, s>>>(h->D, XF_EXPORT, epoch);
    h->exp_epoch = epoch;
    count_launch(2);
    const int n_own = R < n ? (n - R + G - 1) / G : 0;
    std::vector<int> row0(n_own + 1, 0);
    if (n_own > 0) {
        if ((rc = hd_reserve(h, h->mx_heads, 2 * (size_t) n_own * G, fn)) != ICG_OK) return rc;
        ba_marg_heads<<<1, 256, 0, s>>>(C, h->D, n_own, h->mx_heads.d, epoch);
        ICG_CUDA(h->mx_heads.down(s, 2 * (size_t) n_own * G));
        ICG_CUDA(cudaStreamSynchronize(s));
        if ((rc = shard_timed_out(h, fn)) != ICG_OK) return rc;
        if ((rc = hd_reserve(h, h->mx_row, (size_t) n_own * G + n_own + 1, fn)) != ICG_OK) return rc;
        size_t tot = 0;
        for (int e = 0; e < n_own * G; e++) {
            if (e % G == 0) row0[e / G] = (int) tot;
            h->mx_row.h[e] = (int) tot;
            tot += (size_t) h->mx_heads.h[2 * e + 1];
        }
        row0[n_own] = (int) tot;
        if (tot > (size_t) INT32_MAX / MEXP_ROW) {
            set_error("%s: %zu gathered factors exceed the gather buffer's index range", fn, tot);
            return ICG_EINVAL;
        }
        if (tot * MEXP_ROW > h->mx_rows_cap) {
            retire(h, h->mx_rows, nullptr), h->mx_rows = nullptr;
            h->mx_rows_cap = 0;
            const size_t cap = (tot + tot / 4) * MEXP_ROW;
            if (cudaMalloc(&h->mx_rows, sizeof(double) * cap) != cudaSuccess) {
                set_error("%s: gather buffer allocation of %zu doubles failed", fn, cap);
                return ICG_ENOMEM;
            }
            h->mx_rows_cap = cap;
        }
        if ((rc = hd_reserve(h, h->mx_idx, std::max<size_t>(1, tot), fn)) != ICG_OK) return rc;
        memcpy(h->mx_row.h + (size_t) n_own * G, row0.data(), sizeof(int) * (n_own + 1));
        ICG_CUDA(h->mx_row.up(s, (size_t) n_own * G + n_own + 1));
        ba_marg_gather<<<dim3(n_own, G), 256, 0, s>>>(C, h->D, h->mx_heads.d, h->mx_row.d, h->mx_rows);
        count_launch(2);
        if (tot) ICG_CUDA(cudaMemcpy2DAsync(h->mx_idx.h, sizeof(long long), h->mx_rows, sizeof(double) * MEXP_ROW, sizeof(long long), tot, cudaMemcpyDeviceToHost, s));
    }
    ba_xflag<<<1, 32, 0, s>>>(h->D, XF_DONE, epoch);  // this rank's reads of the exports are enqueued: the exporters may reuse their regions
    ICG_CHECK_LAUNCH();
    count_launch();
    for (int w = 0; w < n; w++)
        if (w % G != R) out[w].m = out[w].r = out[w].nblocks = 0;
    h->prior.n = 0;  // the workspace is about to be overwritten: the sharded slide's prior again only if this call succeeds
    // on success: the record icg_ba_shard_slide[_integrate]_resident checks (every rank: a sharded resident marginalization of these n
    // windows; the owner: each owned window's m, r, nblocks)
    auto record = [&]() { prior_commit(h, n, out, R, G); return ICG_OK; };
    // an owner that fails from here joins the group's agreement on the eigensolver sizes with a rejection, so that no peer waits for it
    auto reject = [&](int code) {
        int mx[3] = {0, 0, 1};
        shard_xmax(h, mx, fn);
        return code;
    };
    if (n_own == 0) {
        int mx[3] = {0, 0, 0};
        rc = shard_xmax(h, mx, fn);
        if (rc != ICG_OK) return rc;
        if (mx[2]) {
            set_error("%s: a window owned by another rank of the shard group was rejected (see that rank's error)", fn);
            return ICG_EUNSUPPORTED;
        }
        return record();
    }
    ICG_CUDA(cudaStreamSynchronize(s));
    if ((rc = shard_timed_out(h, fn)) != ICG_OK) return rc;
    // the gathered windows, structure on the host (values follow on the device): landmarks renumbered densely in (rank, shard landmark) order
    std::vector<icg_ba_problem> gp(n_own);
    std::vector<std::vector<int32_t>> g_lm(n_own), g_ref(n_own), g_obs(n_own);
    std::vector<std::vector<uint8_t>> g_act(n_own);
    int max_L = 1, max_F = 1;
    for (int j = 0; j < n_own; j++) {
        const int w = R + j * G, F = row0[j + 1] - row0[j];
        const icg_ba_problem &p = problems[w];
        g_lm[j].resize(F), g_ref[j].resize(F), g_obs[j].resize(F), g_act[j].resize(F);
        int L = 0, last_r = -1, last_l = -1;
        for (int r = 0, i = 0; r < G; r++)
            for (long long k = 0; k < h->mx_heads.h[2 * ((size_t) j * G + r) + 1]; k++, i++) {
                const unsigned long long x = (unsigned long long) h->mx_idx.h[row0[j] + i];
                const int l = (int) (x & 0xffffffffu), hi = (int) (x >> 32), ref = hi & 255, obs = (hi >> 8) & 255;
                if (r != last_r || l != last_l) L++, last_r = r, last_l = l;
                if (ref >= num_marg[w] || obs >= p.K) {
                    set_error("%s: window %d: gathered factor %d names nodes %d / %d (the ranks' windows differ)", fn, w, i, ref, obs);
                    return reject(ICG_EINVAL);
                }
                g_lm[j][i] = L - 1, g_ref[j][i] = ref, g_obs[j][i] = obs, g_act[j][i] = (uint8_t) ((hi >> 16) & 1);
            }
        icg_ba_problem &q = gp[j];
        q = p;
        q.L = L, q.F = F;
        q.f_lm = g_lm[j].data(), q.f_ref = g_ref[j].data(), q.f_obs = g_obs[j].data(), q.f_active = g_act[j].data();
        max_L = std::max(max_L, L), max_F = std::max(max_F, F);
    }
    double unread = 0;  // the structure-only packing checks these pointers but reads no value: ba_marg_fill writes them on the device
    for (auto &q : gp) q.invdepth = &unread, q.f_const = &unread;
    icg_ba *&mh = h->mx_h;
    if (mh && (mh->C.NW < n_own || mh->C.L < max_L || mh->C.F < max_F)) {
        max_L = std::max(max_L, mh->C.L), max_F = std::max(max_F, mh->C.F);
        h->retired_mx.push_back(mh), mh = nullptr;
    }
    if (!mh) {
        const int nw = std::max(n_own, (C.NW + G - 1) / G);
        rc = icg_ba_create(&mh, nw, C.K, max_L + max_L / 4, max_F + max_F / 4, C.G, C.R, h->device, (void *) s);
        if (rc != ICG_OK) {
            mh = nullptr;
            return reject(rc);
        }
    }
    // structure only (landmark positions, record slots, lin_vis runs, Gram partials, pairs; the small camera-side tables): the same packing
    // icg_ba_upload does, so the sums match an unsharded handle's.  Every value comes from the device: the gathered rows, and the shard
    // handle's resident camera side (parameters, IMU blobs and square-root information, GNSS, the carried prior's normal equations).
    rc = pack_windows(mh, n_own, gp.data(), false);
    if (rc == ICG_OK) rc = upload_structure(mh, n_own);
    if (rc != ICG_OK) return reject(rc);
    mh->cur_windows = n_own, mh->end_results();
    ICG_CUDA(mh->lm_fidx.up(s, (size_t) n_own * mh->C.F));
    ba_marg_fill<<<n_own, 128, 0, s>>>(mh->C, mh->D, C, h->D, h->mx_rows, h->mx_row.d + (size_t) n_own * G, mh->lm_fidx.d);
    ICG_CHECK_LAUNCH();
    count_launch();
    std::vector<int32_t> nm(n_own);
    std::vector<icg_ba_prior> po(n_own);
    for (int j = 0; j < n_own; j++) nm[j] = num_marg[R + j * G], po[j] = out[R + j * G];
    const std::function<int(int *)> agree = [h, fn](int *mx) { return shard_xmax(h, mx, fn); };
    rc = marginalize_body(mh, n_own, gp.data(), nm.data(), po.data(), true, nullptr, &agree);
    for (int j = 0; j < n_own; j++) out[R + j * G].m = po[j].m, out[R + j * G].r = po[j].r, out[R + j * G].nblocks = po[j].nblocks;
    return rc == ICG_OK ? record() : rc;
}

// ---- post-solve map update + outlier culling (ba_cull.cu)
static int resident_single_rank(icg_ba *h, int n_windows, const icg_ba_problem *problems, const char *what, bool sharded_ok = false) {
    if (!h || !problems || n_windows < 1) {
        set_error("%s: bad arguments", what);
        return ICG_EINVAL;
    }
    if (h->D.world > 1 && !sharded_ok) {  // the reintegration and the slides: their collective forms are icg_ba_shard_*
        set_error("%s: not available on a landmark-sharded handle (the group calls icg_ba_shard_%s; or icg_ba_shard_leave first)", what, what + 7);
        return ICG_EUNSUPPORTED;
    }
    if (h->cur_windows != n_windows) {
        set_error("%s: the handle holds %d uploaded windows, the call names %d", what, h->cur_windows, n_windows);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

// Every IMU factor's rows already on the device (the handle's sample store, or the next one a slide builds): factor k of window w is rows
// row0[w][k] .. + nrow[w][k] of d (nrow -1: no samples)
struct FactorRows {
    const double *d;
    const std::vector<std::vector<int>> &row0, &nrow;
};

// ---- doReintegration (IG/ic_gvins.cc:1680-1695) on the resident IMU factors (preint.cu)
// fr: the rows are the store's (icg_ba_reintegrate_stored_resident), io's imu / imu_off are not read
// sharded (icg_ba_shard_reintegrate_resident): every rank runs the same reintegration on its replicated states, after the group agreed
static int reint_body(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3, icg_ba_reint_window *io,
                      const char *fn, bool sharded, const FactorRows *fr = nullptr) {
    const int n = n_windows;
    // validation first: nothing is launched on bad input
    size_t n_items = 0, n_rows = 0;
    auto validate = [&]() -> int {
        int rc = resident_single_rank(h, n_windows, problems, fn, sharded);
        if (rc != ICG_OK) return rc;
        if (!noise5 || !station3 || !io) {
            set_error("%s: bad arguments", fn);
            return ICG_EINVAL;
        }
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = problems[w];
            const icg_ba_reint_window &c = io[w];
            if (p.K < 2 || p.K > h->C.K || p.n_imu < 0 || p.n_imu > p.K - 1) {
                set_error("%s: window %d: sizes out of range", fn, w);
                return ICG_EINVAL;
            }
            if (!c.reintegrate || p.n_imu == 0) continue;
            if ((!fr && (!c.imu || !c.imu_off)) || !c.status || !c.blob_out) {
                set_error("%s: window %d: arrays missing", fn, w);
                return ICG_EINVAL;
            }
            if (fr) {
                for (int k = 0; k < p.n_imu; k++)
                    if (k >= (int) fr->nrow[w].size() || fr->nrow[w][k] < 1) {
                        set_error("%s: window %d IMU factor %d has no samples in the store", fn, w, k);
                        return ICG_EINVAL;
                    }
                n_items += p.n_imu;
                continue;
            }
            if (c.imu_off[0] < 0) {
                set_error("%s: window %d: imu_off[0] is negative", fn, w);
                return ICG_EINVAL;
            }
            for (int k = 0; k < p.n_imu; k++)
                if (c.imu_off[k + 1] - c.imu_off[k] < 1) {
                    set_error("%s: window %d factor %d: imu_off must give every interval at least one row", fn, w, k);
                    return ICG_EINVAL;
                }
            n_items += p.n_imu, n_rows += (size_t) (c.imu_off[p.n_imu] - c.imu_off[0]);
        }
        if (n_items > INT32_MAX / 8 || n_rows > INT32_MAX / 8) {
            set_error("%s: too many factors or IMU rows in one call", fn);
            return ICG_EINVAL;
        }
        return ICG_OK;
    };
    int rc = validate();
    if (sharded) {  // every argument is camera side: the sizes, the flags, the rows, noise and station
        ArgPrint fp;
        fp.num(n);
        for (int w = 0; rc == ICG_OK && w < n; w++) {
            const icg_ba_problem &p = problems[w];
            const icg_ba_reint_window &c = io[w];
            const bool on = c.reintegrate && p.n_imu > 0;
            fp.num(p.K), fp.num(p.n_imu), fp.num(on);
            if (!on) continue;
            fp.arr(c.imu_off, p.n_imu + 1);
            fp.arr(c.imu + 7 * (size_t) c.imu_off[0], 7LL * (c.imu_off[p.n_imu] - c.imu_off[0]));
        }
        if (rc == ICG_OK) fp.arr(noise5, 5), fp.arr(station3, 3);
        rc = shard_agree(h, rc != ICG_OK, fp.get(), fn);
    }
    if (rc != ICG_OK) return rc;
    const BaCaps &C = h->C;
    for (int w = 0; w < n; w++) io[w].count = 0;
    if (n_items == 0) return ICG_OK;
    // staging: inputs [items | rows | counter (0)] go up in one copy; [counter | status | ends | out_item] come back in one copy, then the
    // status-1 blobs, compacted on the device
    Layout lay;
    const size_t i_item = lay.take(sizeof(ReintItem) * n_items), i_rows = lay.take(56 * n_rows), o_cnt = lay.take(sizeof(int));
    const size_t o_status = lay.take(n_items), o_ends = lay.take(80 * n_items), o_item = lay.take(4 * n_items),
                 o_blob = lay.take(sizeof(double) * ICG_IMU_BLOB_DOUBLES * n_items);
    ICG_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (lay.size() > h->reint.n) ICG_CUDA(cudaStreamSynchronize(s));
    if ((rc = hd_reserve(h, h->reint, lay.size(), fn)) != ICG_OK) return rc;  // a shard group keeps the old one: freeing would wait for a peer's kernel
    unsigned char *H = h->reint.h, *Dv = h->reint.d;
    ReintItem *items = (ReintItem *) (H + i_item);
    std::vector<int> first(n, -1);  // first item of each reintegrated window
    {
        size_t it = 0, row = 0;
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = problems[w];
            const icg_ba_reint_window &c = io[w];
            if (!c.reintegrate || p.n_imu == 0) continue;
            first[w] = (int) it;
            if (fr) {
                for (int k = 0; k < p.n_imu; k++, it++) items[it] = ReintItem{w, k, fr->row0[w][k], fr->nrow[w][k]};
                continue;
            }
            const int r0 = c.imu_off[0], nr = c.imu_off[p.n_imu] - r0;
            memcpy(H + i_rows + 56 * row, c.imu + 7 * (size_t) r0, 56 * (size_t) nr);
            for (int k = 0; k < p.n_imu; k++, it++)
                items[it] = ReintItem{w, k, (int) row + c.imu_off[k] - r0, c.imu_off[k + 1] - c.imu_off[k]};
            row += nr;
        }
    }
    *(int *) (H + o_cnt) = 0;
    ICG_CUDA(cudaMemcpyAsync(Dv, H, o_status, cudaMemcpyHostToDevice, s));
    PreintResident a;
    a.n = (int) n_items, a.item = (const ReintItem *) (Dv + i_item), a.imu = fr ? fr->d : (const double *) (Dv + i_rows);
    a.pose = h->D.pose, a.mix = h->D.mix, a.blob = h->D.imu_blob, a.U = h->D.imu_U, a.K = C.K;
    for (int k = 0; k < 5; k++) a.noise5[k] = noise5[k];
    for (int k = 0; k < 3; k++) a.station[k] = station3[k];
    a.status = (int8_t *) (Dv + o_status), a.ends = (double *) (Dv + o_ends), a.out_blob = (double *) (Dv + o_blob), a.out_item = (int *) (Dv + o_item);
    a.counter = (int *) (Dv + o_cnt);
    h->lin_ready = false;  // the reintegrated factors are not those of the last linearisation
    ICG_CUDA(preint_resident_launch(a, s));
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(H + o_cnt, Dv + o_cnt, o_blob - o_cnt, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    const int n_done = *(const int *) (H + o_cnt);
    if (n_done < 0 || (size_t) n_done > n_items) {
        set_error("%s: inconsistent completion count %d", fn, n_done);
        return ICG_ECUDA;
    }
    if (n_done > 0) {
        ICG_CUDA(cudaMemcpyAsync(H + o_blob, Dv + o_blob, sizeof(double) * ICG_IMU_BLOB_DOUBLES * (size_t) n_done, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(cudaStreamSynchronize(s));
    }
    const int8_t *st = (const int8_t *) (H + o_status);
    const double *ends = (const double *) (H + o_ends);
    for (int q = 0; q < n_done; q++) {
        const ReintItem &it = items[((const int *) (H + o_item))[q]];
        memcpy(io[it.win].blob_out + (size_t) ICG_IMU_BLOB_DOUBLES * it.fac, H + o_blob + sizeof(double) * ICG_IMU_BLOB_DOUBLES * (size_t) q,
               sizeof(double) * ICG_IMU_BLOB_DOUBLES);
    }
    int bad_w = -1, bad_k = -1;
    for (int w = 0; w < n; w++) {
        if (first[w] < 0) continue;
        icg_ba_reint_window &c = io[w];
        for (int k = 0; k < problems[w].n_imu; k++) {
            const int q = first[w] + k;
            c.status[k] = st[q];
            if (st[q] != 0) {
                c.count++;
                if (c.end_state10) memcpy(c.end_state10 + 10 * (size_t) k, ends + 10 * (size_t) q, 80);
            }
            if (st[q] < 0 && bad_w < 0) bad_w = w, bad_k = k;
        }
    }
    if (bad_w >= 0) {
        set_error("%s: window %d IMU factor %d: the reintegrated covariance is not positive definite (the factor was kept)", fn, bad_w, bad_k);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

// a collective call of a shard group: the entry points below take the sharded form of their plain counterpart's body
static int shard_group_only(icg_ba *h, const char *fn, const char *plain) {
    if (!h) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->D.world < 2) {
        set_error("%s: the handle is not in a landmark-shard group (call %s)", fn, plain);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

// What vision_body hands slide_body for windows built on the device: the outcome of ba_pack_structure (a rejection is reported where the
// host packing would report it), and the maps and rows the gather reads there (PackArgs::map)
struct VisSlide {
    int rc = ICG_OK;
    std::string err;
    const int *map = nullptr;
    const double *invdepth = nullptr, *f_new = nullptr;
    std::vector<int> lm_at, slot_at;  // per window: its first landmark / record-slot entry of map
};

// ---- the next keyframe's windows from the resident ones (ba_slide.cu): the structure is packed on the host as icg_ba_upload packs it, the
//      values of the carried rows never leave the device.  With `integ`, the new factors, node rows and aligned fixes it names are computed on
//      the device (preint.cu) into the staged value rows before the gather reads them.
//
// sharded (icg_ba_shard_slide[_integrate]_resident, a collective call): the same checks, plus landmark-by-landmark factor lists and the owner's
// check of its own prior; then one agreement of the group (shard_agree: every rank's verdict and a fingerprint of the camera side) before any
// rank writes its device, and with `integ` a second one on the integration's outcome.  A rank that rejects joins the agreement all the same
// (fail below), so its peers never wait for it.  The owner of window w forms its prior from the workspace of mx_h; the other ranks get zeros.
// vs: the windows vision_body built, whose vision structure ba_pack_structure packed into h->pack and whose new vision rows the gather reads
// on the device (vision_body has also written their reference rows into lm_ref_alt); seed (sharded): vision_body's fingerprint of
// its own arguments, which the agreement's fingerprint continues; fr (icg_ba_slide_ins_resident): the integrated factors' rows are the next
// sample store's, integ's imu / imu_off are not read
static int slide_body(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                      const double *noise5, const double *station3, const char *fn, bool sharded, const VisSlide *vs = nullptr,
                      const ArgPrint *seed = nullptr, const FactorRows *fr = nullptr) {
    bool joined = false;  // sharded: this rank has joined the agreement of the call
    std::vector<WinDims> old_dims;
    std::vector<std::vector<int>> old_slot;
    // a rejected call leaves the handle as it was: the packing below rewrites the host tables later calls read (dims, which restore_params
    // uploads, and the slot table of the next slide), so they go back on failure; nothing reaches the device before every check has passed
    auto fail = [&](int code) {
        if (!old_dims.empty()) {
            memcpy(h->dims.h, old_dims.data(), sizeof(WinDims) * n);
            for (int w = 0; w < (int) old_slot.size(); w++) {
                int *fidx = h->lm_fidx.h + (size_t) w * h->C.F;
                for (int f = 0; f < old_dims[w].F; f++) fidx[old_slot[w][f]] = f;
            }
        }
        // sharded: a rank that rejects before the agreement joins it with its rejection, and returns ICG_EINVAL as its peers do (its own
        // message says why); only a failed exchange (a peer did not make the call) returns that error instead
        if (sharded && !joined) joined = true, code = shard_agree(h, true, 0, fn);
        return code;
    };
    // a CUDA error before the agreement is this rank's rejection like any other
    auto cuda_fail = [&](cudaError_t e, const char *what) {
        set_error("%s: %s failed: %s", fn, what, cudaGetErrorString(e));
        return fail(ICG_ECUDA);
    };
    int rc = resident_single_rank(h, n, next, fn, sharded);
    if (rc != ICG_OK) return fail(rc);
    if (!carry || (integ && (!noise5 || !station3))) {
        set_error("%s: bad arguments", fn);
        return fail(ICG_EINVAL);
    }
    if (cudaError_t e = cudaSetDevice(h->device)) return cuda_fail(e, "cudaSetDevice");
    const BaCaps &C = h->C;
    const size_t NW = C.NW;
    const int G = h->D.world, R = h->D.rank;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = next[w];
        // (the vision build lists each landmark's factors together, landmarks in order: next's f_lm is NULL there)
        if (sharded)
            for (int f = 1; p.f_lm && f < p.F; f++)
                if (p.f_lm[f] < p.f_lm[f - 1]) {
                    set_error("%s: window %d factor %d: a landmark-sharded window must list its factors landmark by landmark (f_lm non-decreasing)", fn, w, f);
                    return fail(ICG_EINVAL);
                }
        if (!carry[w].prior_from_marg) continue;
        if (h->prior.n != n || h->prior.sharded != sharded) {
            set_error("%s: window %d takes its prior from the marginalization, but no %sresident marginalization of these %d windows "
                      "ran since the last upload or slide", fn, w, sharded ? "sharded " : "", n);
            return fail(ICG_EINVAL);
        }
        if (sharded && w % G != R) continue;  // the owner holds the window's m, r and nblocks
        if (h->prior.m[w] <= 0 || p.marg_r != h->prior.r[w] || p.marg_nblocks != h->prior.nb[w]) {
            set_error("%s: window %d: marg_r=%d / marg_nblocks=%d, but the resident marginalization left m=%d, r=%d / nblocks=%d", fn, w,
                      p.marg_r, p.marg_nblocks, h->prior.m[w], h->prior.r[w], h->prior.nb[w]);
            return fail(ICG_EINVAL);
        }
    }
    // the device buffers of the first slide: the old value rows at the handle's strides, the second f_const_s
    const size_t o_mix = NW * C.K * 7, o_rho = o_mix + NW * C.K * 9, o_blob = o_rho + NW * C.L, o_U = o_blob + NW * C.K * ICG_IMU_BLOB_DOUBLES,
                 o_blh = o_U + NW * C.K * 225, o_std = o_blh + NW * C.G * 3, n_old = o_std + NW * C.G * 3;
    if (!h->slide_old && (cudaMalloc(&h->slide_old, sizeof(double) * n_old) != cudaSuccess ||
                          cudaMalloc(&h->fc_alt, sizeof(double) * NW * C.F * 14) != cudaSuccess)) {
        if (h->slide_old) cudaFree(h->slide_old), h->slide_old = nullptr;
        set_error("%s: allocation of the slide buffers failed", fn);
        return fail(ICG_ENOMEM);
    }
    // the old windows: sizes, and every factor's record slot (the inverse of the last packing's slot -> factor table; built windows: the
    // device's slot maps)
    old_dims.assign(h->dims.h, h->dims.h + n);
    old_slot.resize(vs ? 0 : n);
    for (int w = 0; w < (int) old_slot.size(); w++) {
        old_slot[w].resize(old_dims[w].F);
        const int *fidx = h->lm_fidx.h + (size_t) w * C.F;
        for (int q = 0; q < old_dims[w].F; q++) old_slot[w][fidx[q]] = q;
    }
    rc = pack_windows(h, n, next, false, !vs);
    if (rc == ICG_OK && vs && vs->rc != ICG_OK) set_error("%s", vs->err.c_str()), rc = vs->rc;
    if (rc != ICG_OK) return fail(rc);
    // the maps: range checks, sizes of the staging
    std::vector<SlideWin> wins(n);
    std::vector<size_t> vbase(n);  // first staged value of each window
    size_t n_map = 0, n_val = 0;
    int max_elems = 0, max_r = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const WinDims &od = old_dims[w];
        const int32_t *maps[5] = {c.node_src, c.lm_src, c.f_src, c.imu_src, c.gnss_src};
        const int cnt[5] = {p.K, p.L, p.F, p.n_imu, p.n_gnss}, lim[5] = {od.K, od.L, od.F, od.n_imu, od.n_gnss}, width[5] = {SLIDE_NODE, 1, 14, SLIDE_IMU, SLIDE_GNSS};
        static const char *names[5] = {"node_src", "lm_src", "f_src", "imu_src", "gnss_src"};
        vbase[w] = n_val;
        for (int t = 0; t < 5; t++)
            for (int i = 0; maps[t] && i < cnt[t] && !(vs && (t == 1 || t == 2)); i++) {
                if (maps[t][i] < -1 || maps[t][i] >= lim[t]) {
                    set_error("%s: window %d: %s[%d] = %d is out of range of the old window (%d)", fn, w, names[t], i, maps[t][i], lim[t]);
                    return fail(ICG_EINVAL);
                }
                if (maps[t][i] >= 0) continue;
                n_val += width[t];
            }
        for (int t = 0; t < 5; t++)
            if (!maps[t] && !(vs && (t == 1 || t == 2))) n_val += (size_t) width[t] * cnt[t];
        SlideWin &W = wins[w];
        W.K = p.K, W.L = p.L, W.F = p.F, W.n_imu = p.n_imu, W.n_gnss = p.n_gnss;
        if (vs) {
            W.vis = 1, W.lm_map = vs->lm_at[w], W.slot_map = vs->slot_at[w];
            W.node_map = (int) n_map, W.imu_map = W.node_map + p.K, W.gnss_map = W.imu_map + p.n_imu;
        } else {
            W.node_map = (int) n_map, W.lm_map = W.node_map + p.K, W.slot_map = W.lm_map + p.L, W.imu_map = W.slot_map + p.F, W.gnss_map = W.imu_map + p.n_imu;
        }
        n_map = (size_t) W.gnss_map + p.n_gnss;
        W.r = p.marg_r, W.from_marg = c.prior_from_marg != 0, W.j0 = W.e0 = 0;
        W.slot = !sharded ? w : w % G == R ? (w - R) / G : -1;
        if (W.r > 0 && !W.from_marg) n_val += (size_t) W.r * W.r + W.r;
        max_elems = std::max(max_elems, SLIDE_NODE * p.K + p.L + 14 * p.F + SLIDE_IMU * p.n_imu + SLIDE_GNSS * p.n_gnss);
        max_r = std::max(max_r, W.r);
    }
    // the integration's arrays (only rows the carry maps leave to next are read): every check before anything is staged
    std::vector<std::vector<int>> item_of(integ ? n : 0);  // per window and new factor: its item, or -1
    std::vector<int> iwin_of(integ ? n : 0, -1);           // per window: its entry of iwins, or -1
    std::vector<SlideIntWin> iwins;                         // the windows with device work, one warp each
    std::vector<size_t> row_base(integ ? n : 0), state_base(integ ? n : 0);
    size_t n_item = 0, n_align = 0, n_row = 0, n_state = 0;
    bool want_blob = false;
    for (int w = 0; integ && w < n; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const icg_ba_slide_integrate &g = integ[w];
        const int oK = old_dims[w].K;
        std::vector<int> &io = item_of[w];
        io.assign(p.n_imu, -1);
        const size_t item0 = n_item, align0 = n_align;
        row_base[w] = n_row, state_base[w] = n_state;
        for (int k = 0; g.imu_from && k < p.n_imu; k++) {
            const int src = g.imu_from[k];
            if ((c.imu_src && c.imu_src[k] >= 0) || src == -1) continue;
            if (src >= oK || (src < 0 && src != ICG_SLIDE_CHAIN && src != ICG_SLIDE_ROW)) {
                set_error("%s: window %d: imu_from[%d] = %d is out of range of the old window (%d)", fn, w, k, src, oK);
                return fail(ICG_EINVAL);
            }
            if (src == ICG_SLIDE_CHAIN && (k == 0 || io[k - 1] < 0)) {
                set_error("%s: window %d: imu_from[%d] is ICG_SLIDE_CHAIN, but no integrated factor precedes it", fn, w, k);
                return fail(ICG_EINVAL);
            }
            if (!g.gravity3 || (!fr && (!g.imu || !g.imu_off)) || (src == ICG_SLIDE_ROW && !g.state16)) {
                set_error("%s: window %d: arrays missing", fn, w);
                return fail(ICG_EINVAL);
            }
            if (fr ? fr->nrow[w][k] < 1 : g.imu_off[k] < 0 || (long long) g.imu_off[k + 1] - g.imu_off[k] < 1) {
                set_error("%s: window %d factor %d: imu_off must give every integrated interval at least one row", fn, w, k);
                return fail(ICG_EINVAL);
            }
            io[k] = (int) n_item++;
            if (!fr) n_row += (size_t) (g.imu_off[k + 1] - g.imu_off[k]);
            n_state += src == ICG_SLIDE_ROW;
        }
        for (int j = 0; g.node_from_imu && j < p.K; j++) {
            if ((c.node_src && c.node_src[j] >= 0) || !g.node_from_imu[j]) continue;
            if (j == 0 || j - 1 >= p.n_imu || io[j - 1] < 0) {
                set_error("%s: window %d: node_from_imu[%d] is set, but factor %d is not integrated", fn, w, j, j - 1);
                return fail(ICG_EINVAL);
            }
        }
        for (int q = 0; g.gnss_node && q < p.n_gnss; q++) {
            if ((c.gnss_src && c.gnss_src[q] >= 0) || g.gnss_node[q] == -1) continue;
            if (g.gnss_node[q] < -1 || g.gnss_node[q] >= oK) {
                set_error("%s: window %d: gnss_node[%d] = %d is out of range of the old window (%d)", fn, w, q, g.gnss_node[q], oK);
                return fail(ICG_EINVAL);
            }
            if (!g.gnss_dt) {
                set_error("%s: window %d: arrays missing", fn, w);
                return fail(ICG_EINVAL);
            }
            n_align++;
        }
        if (n_item == item0 && n_align == align0) continue;
        iwin_of[w] = (int) iwins.size();
        iwins.push_back(SlideIntWin{w, (int) item0, (int) (n_item - item0), (int) align0, (int) (n_align - align0)});
        want_blob = want_blob || (g.blob_out && n_item > item0);
    }
    if (n_val >= (size_t) INT32_MAX || n_map >= (size_t) INT32_MAX || n_row >= (size_t) INT32_MAX / 8 || n_item >= (size_t) INT32_MAX / 8) {
        set_error("%s: too many new value rows in one call", fn);
        return fail(ICG_EINVAL);
    }
    // staging: [windows | maps | new value rows] in one pinned buffer, one H2D; with device work also [its windows | items | alignments |
    // IMU rows | ICG_SLIDE_ROW states] (up to in_end) and the outputs that come back, [status | end states | blobs]
    Layout lay;
    lay.take(sizeof(SlideWin) * n);
    const size_t b_map = lay.take(sizeof(int) * n_map), b_val = lay.take(sizeof(double) * n_val);
    size_t b_iw = 0, b_item = 0, b_align = 0, b_rows = 0, b_state = 0, b_status = 0, b_ends = 0, b_blob = 0;
    if (!iwins.empty()) {
        b_iw = lay.take(sizeof(SlideIntWin) * iwins.size()), b_item = lay.take(sizeof(SlideItem) * n_item), b_align = lay.take(sizeof(SlideAlign) * n_align);
        b_rows = lay.take(56 * n_row), b_state = lay.take(128 * n_state);
    }
    const size_t in_end = lay.end;
    if (!iwins.empty()) {
        b_status = lay.take(n_item), b_ends = lay.take(80 * n_item);
        if (want_blob) b_blob = lay.take(sizeof(double) * ICG_IMU_BLOB_DOUBLES * n_item);
    }
    const size_t total = lay.end;
    cudaStream_t s = h->stream;
    if (total > h->slide.n) {
        if (cudaError_t e = cudaStreamSynchronize(s)) return cuda_fail(e, "cudaStreamSynchronize");  // an earlier slide's copy may read the old buffer
    } else if (h->slide_ev) {
        // the previous slide's H2D has left the pinned buffer before it is rewritten
        if (cudaError_t e = cudaEventSynchronize(h->slide_ev)) return cuda_fail(e, "cudaEventSynchronize");
    }
    if ((rc = hd_reserve(h, h->slide, total, fn)) != ICG_OK) return fail(rc);  // a shard group keeps the old one: freeing would wait for a peer's kernel
    if (!h->slide_ev)
        if (cudaError_t e = cudaEventCreateWithFlags(&h->slide_ev, cudaEventDisableTiming)) return cuda_fail(e, "cudaEventCreateWithFlags");
    int *map = (int *) (h->slide.h + b_map);
    double *val = (double *) (h->slide.h + b_val);
    SlideItem *items = (SlideItem *) (h->slide.h + b_item);
    SlideAlign *aligns = (SlideAlign *) (h->slide.h + b_align);
    double *rows = (double *) (h->slide.h + b_rows), *states = (double *) (h->slide.h + b_state);
    // per window: its slices of the maps, the values and the integration's inputs are disjoint, so the windows are staged on a few host
    // threads, as pack_windows packs them (the square-root information of every new blob is a 15 x 15 factorisation).  A row the device
    // computes gets its value slot here and is written there.
    auto stage_window = [&](int w, std::string &err) -> int {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const icg_ba_slide_integrate *g = integ && iwin_of[w] >= 0 ? &integ[w] : nullptr;
        SlideWin &W = wins[w];
        int vo = (int) vbase[w];
        auto stage = [&](const double *src, int count) {
            const int at = vo;
            memcpy(val + vo, src, sizeof(double) * count);
            vo += count;
            return -(at + 1);
        };
        std::vector<int> node_at(g ? p.K + 1 : 0, -1);  // value offset of a node row the device writes
        for (int k = 0; k < p.K; k++) {
            if (c.node_src && c.node_src[k] >= 0) {
                map[W.node_map + k] = c.node_src[k];
                continue;
            }
            if (g && g->node_from_imu && g->node_from_imu[k]) {
                node_at[k] = vo, map[W.node_map + k] = -(vo + 1), vo += SLIDE_NODE;
                continue;
            }
            map[W.node_map + k] = stage(p.pose + 7 * (size_t) k, 7);
            stage(p.mix + 9 * (size_t) k, 9);
        }
        for (int l = 0; !vs && l < p.L; l++) map[W.lm_map + l] = c.lm_src && c.lm_src[l] >= 0 ? c.lm_src[l] : stage(p.invdepth + l, 1);
        const int *fidx = h->lm_fidx.h + (size_t) w * C.F;  // the new packing's slot -> factor table
        for (int q = 0; !vs && q < p.F; q++) {
            const int f = fidx[q];
            map[W.slot_map + q] = c.f_src && c.f_src[f] >= 0 ? old_slot[w][c.f_src[f]] : stage(p.f_const + 14 * (size_t) f, 14);
        }
        size_t row_at = g ? row_base[w] : 0, state_at = g ? state_base[w] : 0;
        for (int k = 0; k < p.n_imu; k++) {
            if (c.imu_src && c.imu_src[k] >= 0) {
                map[W.imu_map + k] = c.imu_src[k];
                continue;
            }
            if (g && item_of[w][k] >= 0) {
                SlideItem &it = items[item_of[w][k]];
                it.src = g->imu_from[k], it.state = -1, it.blob = vo, it.node = node_at[k + 1];
                it.normal = g->normal && g->normal[k] ? 1 : 0;
                for (int i = 0; i < 3; i++) it.grav[i] = g->gravity3[3 * (size_t) k + i];
                if (fr) {
                    it.row0 = fr->row0[w][k], it.nrow = fr->nrow[w][k];
                } else {
                    const int r0 = g->imu_off[k], nr = g->imu_off[k + 1] - r0;
                    it.row0 = (int) row_at, it.nrow = nr;
                    memcpy(rows + 7 * row_at, g->imu + 7 * (size_t) r0, 56 * (size_t) nr);
                    row_at += nr;
                }
                if (it.src == ICG_SLIDE_ROW) {
                    memcpy(states + 16 * state_at, g->state16 + 16 * (size_t) k, 128);
                    it.state = (int) (16 * state_at++);
                }
                map[W.imu_map + k] = -(vo + 1), vo += SLIDE_IMU;
                continue;
            }
            const double *b = p.imu_blob + (size_t) k * ICG_IMU_BLOB_DOUBLES;
            map[W.imu_map + k] = stage(b, ICG_IMU_BLOB_DOUBLES);
            if (!host_imu_sqrt_info(b + 252, val + vo)) {
                char eb[256];
                snprintf(eb, sizeof(eb), "%s: window %d IMU factor %d has a non positive-definite covariance", fn, w, k);
                err = eb;
                return ICG_EINVAL;
            }
            vo += 225;
        }
        int align_at = g ? iwins[iwin_of[w]].align0 : 0;
        for (int q = 0; q < p.n_gnss; q++) {
            if (c.gnss_src && c.gnss_src[q] >= 0) {
                map[W.gnss_map + q] = c.gnss_src[q];
                continue;
            }
            map[W.gnss_map + q] = stage(p.gnss_blh + 3 * (size_t) q, 3);
            stage(p.gnss_std + 3 * (size_t) q, 3);
            if (g && g->gnss_node && g->gnss_node[q] >= 0) aligns[align_at++] = SlideAlign{-(map[W.gnss_map + q] + 1), g->gnss_node[q], g->gnss_dt[q]};
        }
        if (W.r > 0 && !W.from_marg) {
            W.j0 = -(stage(p.marg_J0, W.r * W.r) + 1);
            W.e0 = -(stage(p.marg_e0, W.r) + 1);
        }
        return ICG_OK;
    };
    {
        const int nthreads = std::max(1, std::min({n / 4, 16, (int) std::thread::hardware_concurrency()}));
        std::vector<int> rcs(nthreads, ICG_OK);
        std::vector<std::string> errs(nthreads);
        auto worker = [&](int t) {
            for (int w = t; w < n && rcs[t] == ICG_OK; w += nthreads) rcs[t] = stage_window(w, errs[t]);
        };
        std::vector<std::thread> th;
        for (int t = 1; t < nthreads; t++) th.emplace_back(worker, t);
        worker(0);
        for (auto &x : th) x.join();
        for (int t = 0; t < nthreads; t++)
            if (rcs[t] != ICG_OK) {
                set_error("%s", errs[t].c_str());
                return fail(rcs[t]);
            }
    }
    if (sharded) {
        ArgPrint fp = seed ? *seed : ArgPrint();
        fp.num(n);
        if (integ) fp.arr(noise5, 5), fp.arr(station3, 3);
        for (int w = 0; w < n; w++) {
            const icg_ba_problem &p = next[w];
            const icg_ba_slide_window &c = carry[w];
            const icg_ba_slide_integrate *g = integ ? &integ[w] : nullptr;
            fp.num(p.K), fp.num(p.n_imu), fp.num(p.n_gnss), fp.num(c.prior_from_marg), fp.num(p.marg_r), fp.num(p.marg_nblocks);
            // the flags and camera-side values the structure packing reads from next
            fp.arr(p.ext, 8), fp.num(p.ext_const), fp.num(p.td_const), fp.arr(&p.reproj_std, 1), fp.num(p.reproj_huber), fp.num(p.gnss_huber);
            fp.num(p.has_imu_error), fp.arr(p.lever, 3), fp.num(p.has_pose_prior), fp.num(p.has_mix_prior);
            if (p.has_pose_prior) fp.arr(p.pose_prior, 7), fp.arr(p.pose_prior_std, 6);
            if (p.has_mix_prior) fp.arr(p.mix_prior, 9), fp.arr(p.mix_prior_std, 9);
            fp.num(!c.node_src), fp.num(!c.imu_src), fp.num(!c.gnss_src);
            fp.arr(c.node_src, p.K), fp.arr(c.imu_src, p.n_imu), fp.arr(c.gnss_src, p.n_gnss), fp.arr(p.gnss_node, p.n_gnss);
            for (int k = 0; k < p.K; k++) {
                if (c.node_src && c.node_src[k] >= 0) continue;
                if (g && g->node_from_imu && g->node_from_imu[k]) fp.num(-1);
                else fp.arr(p.pose + 7 * (size_t) k, 7), fp.arr(p.mix + 9 * (size_t) k, 9);
            }
            for (int k = 0; k < p.n_imu; k++) {
                if (c.imu_src && c.imu_src[k] >= 0) continue;
                const int q = g ? item_of[w][k] : -1;
                if (q < 0) {
                    fp.arr(p.imu_blob + (size_t) k * ICG_IMU_BLOB_DOUBLES, ICG_IMU_BLOB_DOUBLES);
                    continue;
                }
                fp.num(g->imu_from[k]), fp.arr(g->gravity3 + 3 * (size_t) k, 3), fp.num(g->normal && g->normal[k]);
                fp.arr(g->imu + 7 * (size_t) g->imu_off[k], 7LL * (g->imu_off[k + 1] - g->imu_off[k]));
                if (g->imu_from[k] == ICG_SLIDE_ROW) fp.arr(g->state16 + 16 * (size_t) k, 16);
            }
            for (int q = 0; q < p.n_gnss; q++) {
                if (c.gnss_src && c.gnss_src[q] >= 0) continue;
                fp.arr(p.gnss_blh + 3 * (size_t) q, 3), fp.arr(p.gnss_std + 3 * (size_t) q, 3);
                if (g && g->gnss_node) fp.num(g->gnss_node[q]), fp.arr(g->gnss_node[q] >= 0 ? g->gnss_dt + q : nullptr, 1);
            }
            if (p.marg_r > 0) {
                long long nx = 0;
                for (int b = 0; p.marg_block_type && b < p.marg_nblocks; b++) nx += p.marg_block_type[b] == 1 ? 9 : p.marg_block_type[b] == 3 ? 1 : 7;
                fp.arr(p.marg_block_type, p.marg_nblocks), fp.arr(p.marg_block_node, p.marg_nblocks), fp.arr(p.marg_x0, nx);
                if (!c.prior_from_marg) fp.arr(p.marg_J0, (long long) p.marg_r * p.marg_r), fp.arr(p.marg_e0, p.marg_r);
            }
        }
        joined = true;
        if ((rc = shard_agree(h, false, fp.get(), fn)) != ICG_OK) return fail(rc);
    }
    memcpy(h->slide.h, wins.data(), sizeof(SlideWin) * n);
    if (integ) {
        // the device work writes the staging only; a covariance that is not positive definite is known after it, so the call waits for it.
        // Sharded: the ranks integrate the same rows from the same states; the outcome is agreed on all the same before the device is written
        int irc = ICG_OK;
        if (!iwins.empty()) {
            memcpy(h->slide.h + b_iw, iwins.data(), sizeof(SlideIntWin) * iwins.size());
            PreintSlide a;
            a.n = (int) iwins.size(), a.win = (const SlideIntWin *) (h->slide.d + b_iw), a.item = (const SlideItem *) (h->slide.d + b_item);
            a.align = (const SlideAlign *) (h->slide.d + b_align), a.imu = fr ? fr->d : (const double *) (h->slide.d + b_rows);
            a.state = (const double *) (h->slide.d + b_state), a.pose = h->D.pose, a.mix = h->D.mix, a.K = C.K, a.val = (double *) (h->slide.d + b_val);
            for (int k = 0; k < 5; k++) a.noise5[k] = noise5[k];
            for (int k = 0; k < 3; k++) a.station[k] = station3[k];
            a.status = (int8_t *) (h->slide.d + b_status), a.ends = (double *) (h->slide.d + b_ends);
            a.out_blob = want_blob ? (double *) (h->slide.d + b_blob) : nullptr;
            cudaError_t e = cudaMemcpyAsync(h->slide.d, h->slide.h, in_end, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = preint_slide_launch(a, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(h->slide.h + b_status, h->slide.d + b_status, total - b_status, cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
            if (e != cudaSuccess) {
                set_error("%s: the integration on the device failed: %s", fn, cudaGetErrorString(e));
                irc = ICG_ECUDA;
            }
            count_launch();
        }
        const int8_t *st = (const int8_t *) (h->slide.h + b_status);
        const double *ends = (const double *) (h->slide.h + b_ends), *blobs = (const double *) (h->slide.h + b_blob);
        int bad_w = -1, bad_k = -1;
        for (int w = 0; irc == ICG_OK && w < n; w++) {
            const icg_ba_slide_integrate &g = integ[w];
            for (int k = 0; k < next[w].n_imu; k++) {
                const int q = item_of[w][k];
                if (g.status) g.status[k] = q >= 0 ? st[q] : 0;
                if (q < 0) continue;
                if (g.end_state10) memcpy(g.end_state10 + 10 * (size_t) k, ends + 10 * (size_t) q, 80);
                if (g.blob_out) memcpy(g.blob_out + (size_t) ICG_IMU_BLOB_DOUBLES * k, blobs + (size_t) ICG_IMU_BLOB_DOUBLES * q, 8 * ICG_IMU_BLOB_DOUBLES);
                if (st[q] < 0 && bad_w < 0) bad_w = w, bad_k = k;
            }
        }
        if (bad_w >= 0) {
            set_error("%s: window %d IMU factor %d: the integrated covariance is not positive definite", fn, bad_w, bad_k);
            irc = ICG_EINVAL;
        }
        if (sharded) irc = shard_agree(h, irc != ICG_OK, 0, fn);  // a rank's own rejection or a peer's: ICG_EINVAL on every rank
        if (irc != ICG_OK) return fail(irc);
    }
    // every check has passed: from here on the device is written
    h->end_results();
    if (iwins.empty()) ICG_CUDA(cudaMemcpyAsync(h->slide.d, h->slide.h, in_end, cudaMemcpyHostToDevice, s));
    ICG_CUDA(cudaEventRecord(h->slide_ev, s));
    rc = upload_structure(h, n, !vs);
    if (rc != ICG_OK) return rc;
    BaDev &D = h->D;
    if (vs) {
        const size_t nn = (size_t) n, PM = (size_t) C.K * (C.K - 1);
        const PackTables &T = h->pack;
        auto take = [&](void *dst, const void *src, size_t bytes) { return cudaMemcpyAsync(dst, src, nn * bytes, cudaMemcpyDeviceToDevice, s); };
        ICG_CUDA(take(D.f_meta_s, T.f_meta_s, 16 * (size_t) C.F));
        ICG_CUDA(take(D.vb_lm0, T.vb_lm0, 4 * (size_t) C.NVB));
        ICG_CUDA(take(D.lm_off, T.lm_off, 4 * ((size_t) C.L + 1)));
        ICG_CUDA(take(D.lm_perm, T.lm_perm, 4 * (size_t) C.L));
        ICG_CUDA(take(D.ref_nrun, T.ref_nrun, 4 * (size_t) C.K));
        ICG_CUDA(take(D.part_off, T.part_off, 4 * (PM + 1)));
        ICG_CUDA(take(D.pair_ro, T.pair_ro, 4 * PM));
        ICG_CUDA(take(D.vis_ord, T.vis_ord, 4 * (size_t) C.F));
        ICG_CUDA(take(D.npairs, T.npairs, 4));
        ICG_CUDA(take(D.f_active, T.f_active, C.F));
    }
    double *old = h->slide_old;
    const size_t nn = (size_t) n;
    auto d2d = [&](double *dst, const double *src, size_t count) { return cudaMemcpyAsync(dst, src, sizeof(double) * count, cudaMemcpyDeviceToDevice, s); };
    ICG_CUDA(d2d(old, D.pose, nn * C.K * 7));
    ICG_CUDA(d2d(old + o_mix, D.mix, nn * C.K * 9));
    ICG_CUDA(d2d(old + o_rho, D.rho, nn * C.L));
    ICG_CUDA(d2d(old + o_blob, D.imu_blob, nn * C.K * ICG_IMU_BLOB_DOUBLES));
    ICG_CUDA(d2d(old + o_U, D.imu_U, nn * C.K * 225));
    ICG_CUDA(d2d(old + o_blh, D.gnss_blh, nn * C.G * 3));
    ICG_CUDA(d2d(old + o_std, D.gnss_std, nn * C.G * 3));
    SlideArgs a;
    a.win = (const SlideWin *) h->slide.d, a.map = (const int *) (h->slide.d + b_map), a.val = (const double *) (h->slide.d + b_val);
    a.vmap = vs ? vs->map : nullptr, a.vlm = vs ? vs->invdepth : nullptr, a.vfc = vs ? vs->f_new : nullptr;
    a.K = C.K, a.L = C.L, a.F = C.F, a.G = C.G, a.R = C.R;
    a.old_pose = old, a.old_mix = old + o_mix, a.old_rho = old + o_rho, a.old_fc = D.f_const_s, a.old_blob = old + o_blob, a.old_U = old + o_U;
    a.old_blh = old + o_blh, a.old_std = old + o_std;
    a.pose = D.pose, a.mix = D.mix, a.rho = D.rho, a.fc = h->fc_alt, a.blob = D.imu_blob, a.U = D.imu_U, a.blh = D.gnss_blh, a.std = D.gnss_std;
    const icg_ba *mw = sharded ? h->mx_h : h;  // the marginalization's workspace (sharded: the owner's gather handle; none on a rank owning no window)
    a.mJ0 = mw ? mw->M.J0 : nullptr, a.me0 = mw ? mw->M.e0 : nullptr, a.mrcap = mw ? mw->M.rcap : 0;
    a.H0 = D.marg_H0, a.b0 = D.marg_b0, a.c0 = D.marg_c0;
    ICG_CUDA(launch_slide(a, n, max_elems, max_r, s));
    count_launch(2);
    std::swap(h->f_const_s.d, h->fc_alt);  // the gathered record constants become the handle's
    D.f_const_s = h->f_const_s.d;
    if (!vs) ICG_CUDA(launch_lm_ref_fill(h, n, a.win, a.map, h->lm_ref, h->lm_ref_alt));
    std::swap(h->lm_ref, h->lm_ref_alt);
    rc = keep_pristine(h, n);
    if (rc != ICG_OK) return rc;
    h->cur_windows = n;
    return ICG_OK;
}

// ---- the vision half of the next windows built on the device (ba_vision.cu), then the slide of those windows (slide_body).
//
// sharded (icg_ba_shard_slide_vision_resident, a collective call): each rank builds its next shard from its own old shard, its own culling and
// its shard-local obs_lm; new map point j of window w is built on rank (j + w) mod world only.  The vision arguments every rank must share and
// the two counts the kernel read on the device seed slide_body's fingerprint, so the group still agrees once; a rank that rejects before
// slide_body joins that agreement with its rejection, as slide_body's own checks do.  The kernel also writes the next culling's lists (the
// rank's next shard's, sharded); they become current only when slide_body has committed.
static int vision_body(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                       const double *noise5, const double *station3, icg_ba_slide_vision *vis, const char *fn, bool sharded,
                       const FactorRows *fr = nullptr) {
    auto reject = [&](int code) { return sharded ? shard_agree(h, true, 0, fn) : code; };
    auto cuda_fail = [&](cudaError_t e, const char *what) {
        set_error("%s: %s failed: %s", fn, what, cudaGetErrorString(e));
        return reject(ICG_ECUDA);
    };
    int rc = resident_single_rank(h, n, next, fn, sharded);
    if (rc != ICG_OK) return reject(rc);
    if (!carry || !vis || (integ && (!noise5 || !station3))) {
        set_error("%s: bad arguments", fn);
        return reject(ICG_EINVAL);
    }
    const icg_ba::CullResult &cul = h->culled;
    if (cul.n != n) {
        set_error("%s: no culling of these %d windows is current (icg_ba_update_and_cull_resident, with no upload or slide since)", fn, n);
        return reject(ICG_EINVAL);
    }
    if (cudaError_t e = cudaSetDevice(h->device)) return cuda_fail(e, "cudaSetDevice");
    const BaCaps &C = h->C;
    std::vector<VisWin> wins(n);
    std::vector<long long> ofac_at(n, -1);  // the window's first entry in the staged obs_factor, -1: the built lists' (vis[w].obs_factor NULL)
    ArgPrint fp;  // sharded: what every rank must pass alike, then the counts its kernel read
    size_t n_ofac = 0, n_lm = 0, n_f = 0, n_nf = 0, n_scr = 0, n_lo = 0, n_pscr = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_vision &v = vis[w];
        const WinDims &od = h->dims.h[w];
        const CullWin &cw = cul.win[w];
        const int nco = cul.nobs[w];
        bool bad = p.K < 2 || p.K > C.K || v.num_marg < 0 || v.num_marg > od.K || !v.node_in_map || !v.node_td || v.cur_node < 0 || v.cur_node >= p.K ||
                   v.n_frames < 0 || v.n_frames > VIS_MAX_FRAMES || (v.n_frames > 0 && (!v.frame_id || !v.frame_node)) || v.n_obs < 0 || v.n_new < 0 ||
                   (v.obs_src && v.n_in < 0) || (v.n_obs > 0 && (!v.obs_lm || !v.obs_undis_xy || !v.obs_vel)) ||
                   (v.n_new > 0 && (!v.new_depth || !v.new_vel_ref || !v.new_vel_cur || !v.new_ref_undis_xy || !v.new_cur_undis_xy || !v.new_ref_frame_id)) ||
                   (nco > 0 && !v.obs_factor && !cul.dev.fac) || cw.K != od.K || cw.L != od.L;
        for (int e = 0; !bad && e < v.n_frames; e++) bad = v.frame_node[e] < 0 || v.frame_node[e] >= p.K;
        if (bad) {
            set_error("%s: window %d: arguments out of range or arrays missing", fn, w);
            return reject(ICG_EINVAL);
        }
        if (sharded) {
            fp.num(v.num_marg), fp.arr(v.node_in_map, od.K), fp.arr(&v.cam, 1), fp.arr(v.node_td, p.K), fp.num(v.cur_node), fp.num(v.n_frames);
            fp.arr(v.frame_id, v.n_frames), fp.arr(v.frame_node, v.n_frames), fp.num(v.n_obs), fp.num(v.n_new);
        }
        VisWin &W = wins[w];
        memset(&W, 0, sizeof(W));
        W.cam = v.cam;
        memcpy(W.node_td, v.node_td, sizeof(double) * p.K);
        memset(W.onode, -1, sizeof(W.onode));
        const int32_t *ns = carry[w].node_src;
        for (int j = 0; ns && j < p.K; j++)
            if (ns[j] >= v.num_marg && ns[j] < od.K && v.node_in_map[ns[j]]) W.onode[ns[j]] = (int8_t) j;
        for (int e = 0; e < v.n_frames; e++) W.frame_id[e] = v.frame_id[e], W.frame_node[e] = v.frame_node[e];
        W.oK = od.K, W.oL = od.L, W.oF = od.F, W.nK = p.K, W.n_frames = v.n_frames, W.cur_node = v.cur_node;
        W.cull_lm0 = cw.lm0, W.cull_off0 = cw.off0, W.cull_obs0 = cw.obs0, W.n_cull_obs = nco;
        if (v.obs_factor) ofac_at[w] = (long long) n_ofac, n_ofac += nco;
        W.n_obs = v.n_obs, W.n_in = v.obs_src ? v.n_in : v.n_obs, W.dev_n = v.dev_n, W.src = v.obs_src, W.obs_node = v.obs_node, W.obs_lm = v.obs_lm;
        W.obs_xy = v.obs_undis_xy, W.obs_vel = v.obs_vel;
        W.n_new = v.n_new, W.dev_new_n = v.dev_new_n, W.new_depth = v.new_depth, W.new_vel_ref = v.new_vel_ref, W.new_vel_cur = v.new_vel_cur;
        W.new_ref_xy = v.new_ref_undis_xy, W.new_cur_xy = v.new_cur_undis_xy, W.new_ref_frame = v.new_ref_frame_id;
        W.lm_out = (int) n_lm, W.f_out = (int) n_f, W.nf_out = (int) n_nf, W.scr = (int) n_scr, W.lst_obs = (int) n_lo, W.pscr = (int) n_pscr;
        n_pscr += 5 * ((size_t) od.L + v.n_new) + 2 * (size_t) od.F + v.n_obs + v.n_new + C.NVB;  // ba_pack_structure's
        n_lm += (size_t) od.L + v.n_new, n_f += (size_t) od.F + v.n_obs + v.n_new, n_nf += (size_t) v.n_obs + v.n_new;
        n_scr += (size_t) od.F + 3 * (size_t) od.L + 5 * ((size_t) od.L + v.n_new) + v.n_new;  // ba_vision_build's scratch
        n_scr += (size_t) od.F + od.L + v.n_new, n_lo += (size_t) nco + v.n_obs + 2 * (size_t) v.n_new;  // and the lists'
        if (n_ofac >= INT32_MAX / 2 || n_f >= INT32_MAX / 16 || n_scr >= INT32_MAX / 2 || n_lo >= INT32_MAX / 4 || n_pscr >= INT32_MAX / 2) {
            set_error("%s: too many rows in one call", fn);
            return reject(ICG_EINVAL);
        }
    }
    // staging: inputs [windows | obs_factor], outputs [counts | slot -> factor tables] (always copied back), [lm_src | lm_org | f_lm | f_ref |
    // f_obs | f_src | invdepth | new factor rows | NaN flags] (each copied back when a caller asks for it), then the slide's maps and the
    // kernels' scratch (never copied)
    Layout lay;
    const size_t b_win = lay.take(sizeof(VisWin) * n), b_ofac = lay.take(4 * n_ofac), in_end = lay.size();
    const size_t b_cnt = lay.take(4 * VIS_COUNTS * (size_t) n), b_fidx = lay.take(4 * n_f), cnt_end = lay.end;
    const size_t b_lms = lay.take(4 * n_lm), b_org = lay.take(4 * n_lm), b_flm = lay.take(4 * n_f), b_fref = lay.take(4 * n_f), b_fobs = lay.take(4 * n_f),
                 b_fsrc = lay.take(4 * n_f), b_invd = lay.take(8 * n_lm), b_fnew = lay.take(112 * n_nf), b_nan = lay.take(n_lm);
    const size_t b_map = lay.take(4 * (n_lm + n_f)), b_scr = lay.take(4 * n_scr), b_pscr = lay.take(4 * n_pscr);
    cudaStream_t s = h->stream;
    if (lay.size() > h->vis.n)
        if (cudaError_t e = cudaStreamSynchronize(s)) return cuda_fail(e, "cudaStreamSynchronize");
    if ((rc = hd_reserve(h, h->vis, lay.size(), fn)) != ICG_OK) return reject(rc);
    // the packed tables' buffer, at the handle's capacities (the first call allocates it)
    PackTables &T = h->pack;
    if (!T.f_meta_s) {
        const size_t NW = C.NW, PM = (size_t) C.K * (C.K - 1);
        const size_t ints = NW * (4 * (size_t) C.F + C.NVB + 2 * (size_t) C.L + 1 + C.K + 2 * PM + 1 + C.F + 1);
        if (cudaMalloc(&T.f_meta_s, 4 * ints + NW * C.F) != cudaSuccess) {
            T.f_meta_s = nullptr;
            set_error("%s: allocation of the packed structure tables failed", fn);
            return reject(ICG_ENOMEM);
        }
        T.vb_lm0 = T.f_meta_s + NW * 4 * C.F, T.lm_off = T.vb_lm0 + NW * C.NVB, T.lm_perm = T.lm_off + NW * (C.L + 1), T.ref_nrun = T.lm_perm + NW * C.L;
        T.part_off = T.ref_nrun + NW * C.K, T.pair_ro = T.part_off + NW * (PM + 1), T.vis_ord = T.pair_ro + NW * PM, T.npairs = T.vis_ord + NW * C.F;
        T.f_active = (uint8_t *) (T.npairs + NW);
    }
    // the next culling's lists (sharded: the rank's next shard's) go to the buffer that is not current
    const int nb = h->built.cur ^ 1;
    icg_ba::BuiltLists::At at{};
    {
        Layout ll;
        at.ref = ll.take(4 * n_lm), at.off = ll.take(4 * (n_lm + n)), at.node = ll.take(4 * n_lo), at.fac = ll.take(4 * n_lo);
        at.rkp = ll.take(8 * n_lm), at.kp = ll.take(8 * n_lo), at.end = ll.size();
        if ((rc = hd_reserve(h, h->built.buf[nb], at.end, fn)) != ICG_OK) return reject(rc);
    }
    unsigned char *H = h->vis.h, *Dv = h->vis.d;
    for (int w = 0; w < n; w++) {
        wins[w].obs_factor = ofac_at[w] >= 0 ? (const int *) (Dv + b_ofac) + ofac_at[w] : cul.dev.fac + cul.win[w].obs0;
        if (ofac_at[w] >= 0 && wins[w].n_cull_obs > 0) memcpy(H + b_ofac + 4 * (size_t) ofac_at[w], vis[w].obs_factor, 4 * (size_t) wins[w].n_cull_obs);
    }
    memcpy(H + b_win, wins.data(), sizeof(VisWin) * n);
    VisArgs a;
    a.win = (const VisWin *) (Dv + b_win), a.K = C.K, a.L = C.L, a.F = C.F;
    a.rank = sharded ? h->D.rank : 0, a.world = sharded ? h->D.world : 1;
    a.rho = h->D.rho, a.lm_ref = h->lm_ref, a.lm_ref_next = h->lm_ref_alt, a.f_meta_s = h->D.f_meta_s, a.lm_off = h->D.lm_off, a.lm_perm = h->D.lm_perm;
    a.lm_ref_node = cul.dev.ref, a.obs_off = cul.dev.off, a.obs_node = cul.dev.node, a.lm_ref_kp = cul.dev.rkp, a.obs_kp = cul.dev.kp;
    a.lm_outlier = cul.lm_outlier, a.obs_outlier = cul.obs_outlier;
    a.counts = (int *) (Dv + b_cnt), a.lm_src = (int *) (Dv + b_lms), a.lm_org = (int *) (Dv + b_org), a.lm_nan = Dv + b_nan, a.f_lm = (int *) (Dv + b_flm), a.f_ref = (int *) (Dv + b_fref);
    a.f_obs = (int *) (Dv + b_fobs), a.f_src = (int *) (Dv + b_fsrc), a.invdepth = (double *) (Dv + b_invd), a.f_new = (double *) (Dv + b_fnew);
    a.scratch = (int *) (Dv + b_scr);
    unsigned char *Dl = h->built.buf[nb].d;
    a.l_ref = (int *) (Dl + at.ref), a.l_off = (int *) (Dl + at.off), a.l_node = (int *) (Dl + at.node), a.l_fac = (int *) (Dl + at.fac);
    a.l_rkp = (float *) (Dl + at.rkp), a.l_kp = (float *) (Dl + at.kp);
    PackArgs pa;
    pa.win = a.win, pa.K = C.K, pa.L = C.L, pa.F = C.F, pa.NVB = C.NVB, pa.counts = a.counts;
    pa.lm_src = a.lm_src, pa.f_lm = a.f_lm, pa.f_ref = a.f_ref, pa.f_obs = a.f_obs, pa.f_src = a.f_src, pa.old_meta = h->D.f_meta_s, pa.out = T;
    pa.fidx = (int *) (Dv + b_fidx), pa.map = (int *) (Dv + b_map), pa.nL = (int) n_lm, pa.scratch = (int *) (Dv + b_pscr);
    // the rows a caller asks for come back; the rest stay on the device, where the slide reads them
    bool want[9] = {};
    for (int w = 0; w < n; w++) {
        const icg_ba_slide_vision &v = vis[w];
        const bool wv[9] = {v.lm_src != nullptr, v.lm_origin != nullptr, v.f_lm != nullptr, v.f_ref != nullptr, v.f_obs != nullptr,
                            v.f_src != nullptr || v.f_const != nullptr, v.invdepth != nullptr, v.f_const != nullptr, v.nan_flags != nullptr};
        for (int i = 0; i < 9; i++) want[i] = want[i] || wv[i];
    }
    const size_t row_at[10] = {b_lms, b_org, b_flm, b_fref, b_fobs, b_fsrc, b_invd, b_fnew, b_nan, b_nan + n_lm};
    cudaError_t e = cudaMemcpyAsync(Dv, H, in_end, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(Dv + b_cnt, 0, 4 * VIS_COUNTS * (size_t) n, s);
    if (e == cudaSuccess && (e = launch_vision(a, n, s)) == cudaSuccess) count_launch();
    if (e == cudaSuccess && (e = launch_pack(pa, n, s)) == cudaSuccess) count_launch();
    if (e == cudaSuccess) e = cudaMemcpyAsync(H + b_cnt, Dv + b_cnt, cnt_end - b_cnt, cudaMemcpyDeviceToHost, s);
    for (int i = 0; i < 9; i++)
        if (e == cudaSuccess && want[i]) e = cudaMemcpyAsync(H + row_at[i], Dv + row_at[i], row_at[i + 1] - row_at[i], cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return cuda_fail(e, "the build on the device");
    // the built windows: every check, then the slide of next with these vision rows
    static const char *what[] = {"", "obs_factor names no factor of the old window", "a device count is outside its list", "obs_src is out of range",
                                 "a node is out of range", "obs_lm is out of range", "two observations of one landmark in one node",
                                 "a reference frame id is not in the frame table", "a landmark whose reference row is unknown takes a new observation"};
    std::vector<icg_ba_problem> nx(next, next + n);
    std::vector<icg_ba_slide_window> cr(carry, carry + n);
    VisSlide vs;
    vs.map = pa.map, vs.invdepth = a.invdepth, vs.f_new = a.f_new;
    vs.lm_at.resize(n), vs.slot_at.resize(n);
    const int *cnt = (const int *) (H + b_cnt);
    for (int w = 0; w < n; w++) {
        const int *c = cnt + VIS_COUNTS * w;
        if (c[3] >= VIS_EPACK_DUP) {
            // the host packing's checks: reported as icg_ba_upload's packing reports them, at the point of the slide where it runs
            if (vs.rc != ICG_OK) continue;
            char eb[256];
            if (c[3] == VIS_EPACK_DUP)
                snprintf(eb, sizeof(eb), "icg_ba_upload: window %d factor %d: landmark %d has two reference nodes or two observations in node %d", w, c[4], c[9], c[10]);
            else
                snprintf(eb, sizeof(eb), "icg_ba_upload: window %d: landmark %d has more than 128 factors or the run table overflows", w, c[4]);
            vs.rc = ICG_EINVAL, vs.err = eb;
        } else if (c[3] != 0) {
            set_error("%s: window %d: %s (entry %d)", fn, w, c[3] > 0 && c[3] <= VIS_EROW ? what[c[3]] : "?", c[4]);
            return reject(ICG_EINVAL);
        }
        if (c[0] > C.L || c[1] > C.F) {
            set_error("%s: window %d: the next window has %d landmarks and %d factors, the handle holds %d / %d", fn, w, c[0], c[1], C.L, C.F);
            return reject(ICG_EINVAL);
        }
        if (sharded) fp.num(c[6]), fp.num(c[7]);
    }
    for (int w = 0; w < n; w++) {
        const int *c = cnt + VIS_COUNTS * w;
        const VisWin &W = wins[w];
        icg_ba_slide_vision &v = vis[w];
        icg_ba_problem &p = nx[w];
        const int L = c[0], F = c[1];
        // the vision half of the next window stays on the device: slide_body reads sizes only
        p.L = L, p.F = F, p.invdepth = nullptr, p.f_active = nullptr, p.f_lm = p.f_ref = p.f_obs = nullptr, p.f_const = nullptr;
        cr[w].lm_src = cr[w].f_src = nullptr;
        vs.lm_at[w] = W.lm_out, vs.slot_at[w] = (int) n_lm + W.f_out;
        v.L = L, v.F = F, v.nan_dropped = c[5];
        const int *f_src = (const int *) (H + b_fsrc) + W.f_out;
        if (v.f_const) {
            const double *rows = (const double *) (H + b_fnew) + 14 * (size_t) W.nf_out;
            for (int f = 0, t = 0; f < F; f++)
                if (f_src[f] < 0) memcpy(v.f_const + 14 * (size_t) f, rows + 14 * (size_t) t++, 112);
        }
        if (v.lm_src) memcpy(v.lm_src, (int *) (H + b_lms) + W.lm_out, 4 * (size_t) L);
        if (v.lm_origin) memcpy(v.lm_origin, (int *) (H + b_org) + W.lm_out, 4 * (size_t) L);
        if (v.nan_flags) memcpy(v.nan_flags, H + b_nan + W.lm_out, (size_t) W.oL + W.n_new);
        if (v.f_src) memcpy(v.f_src, f_src, 4 * (size_t) F);
        if (v.f_lm) memcpy(v.f_lm, (int *) (H + b_flm) + W.f_out, 4 * (size_t) F);
        if (v.f_ref) memcpy(v.f_ref, (int *) (H + b_fref) + W.f_out, 4 * (size_t) F);
        if (v.f_obs) memcpy(v.f_obs, (int *) (H + b_fobs) + W.f_out, 4 * (size_t) F);
        if (v.invdepth) memcpy(v.invdepth, (double *) (H + b_invd) + W.lm_out, 8 * (size_t) L);
    }
    std::vector<CullWin> lw(n);
    std::vector<int> lnobs(n);
    for (int w = 0; w < n; w++) {
        const int *c = cnt + VIS_COUNTS * w;
        lw[w].K = next[w].K, lw[w].L = c[0], lw[w].lm0 = wins[w].lm_out, lw[w].off0 = wins[w].lm_out + w, lw[w].obs0 = wins[w].lst_obs, lnobs[w] = c[8];
    }
    rc = slide_body(h, n, nx.data(), cr.data(), integ, noise5, station3, fn, sharded, &vs, sharded ? &fp : nullptr, fr);
    if (rc != ICG_OK) return rc;  // sharded: the group's agreement inside slide_body has committed every rank's slide, or none
    // the host's copy of the slot -> factor tables (the next plain slide's old slots, the sharded marginalization's export)
    for (int w = 0; w < n; w++)
        memcpy(h->lm_fidx.h + (size_t) w * C.F, (const int *) (H + b_fidx) + wins[w].f_out, 4 * (size_t) h->dims.h[w].F);
    icg_ba::BuiltLists &B = h->built;
    B.cur = nb, B.at[nb] = at, B.n = n, B.nL = n_lm, B.nO = n_lo, B.win = std::move(lw), B.nobs = std::move(lnobs);
    return ICG_OK;
}

// ---- the per-factor IMU sample store (icg_ba_imu_samples_from_ins, icg_ba_slide_ins_resident, icg_ba_reintegrate_stored_resident)
struct StoreSeg {  // rows src_row .. + n of the cut rows (src 0) or of the current store (src 1) to row dst of the next store
    int src, row, dst, n;
};

// one segment per warp, the lanes over its doubles
__global__ void __launch_bounds__(128) ba_store_gather_kernel(int n_seg, const StoreSeg *seg, const double *cut, const double *cur, double *next) {
    const int g = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (g >= n_seg) return;
    const StoreSeg S = seg[g];
    const double *src = (S.src ? cur : cut) + 7 * (size_t) S.row;
    double *dst = next + 7 * (size_t) S.dst;
    for (int i = threadIdx.x & 31; i < 7 * S.n; i += 32) dst[i] = src[i];
}

enum { STORE_NONE, STORE_CUT, STORE_OLD, STORE_MERGE };
struct StoreSrc {  // where a factor of the next store takes its rows from
    int kind;      // STORE_CUT: getImuSeriesFromTo(t0, t1) of INS stream `stream`; STORE_OLD: old factor a's rows; STORE_MERGE: old factor a's
    int a, stream; // rows, then old factor a + 1's without its first (removeUnusedTimeNode's addNewImu loop); STORE_NONE: no samples
    double t0, t1;
};

static int grow_rows(double *&d, size_t &cap, size_t rows, cudaStream_t s, const char *fn) {
    if (rows <= cap) return ICG_OK;
    ICG_CUDA(cudaStreamSynchronize(s));
    if (d) cudaFree(d);
    d = nullptr, cap = 0;
    const size_t c = std::max<size_t>(64, rows + rows / 4);
    if (cudaMalloc(&d, 56 * c) != cudaSuccess) {
        set_error("%s: allocation of %zu IMU rows failed", fn, c);
        return ICG_ENOMEM;
    }
    cap = c;
    return ICG_OK;
}

// The next store from src (per window and factor) into d[1 - cur] and its tables into row0 / nrow; the current store, its tables and the
// INS windows are not changed.  The cut runs on this handle's stream after the work queued on the INS handle's stream, and has completed
// when this returns.  Jobs the INS windows cannot serve are listed in bad (window, factor), with ICG_EINVAL naming the first.
static int store_build(icg_ba *h, const icg_ins *ins, const std::vector<std::vector<StoreSrc>> &src, const char *fn, std::vector<std::vector<int>> &row0,
                       std::vector<std::vector<int>> &nrow, std::vector<std::pair<int, int>> &bad) {
    icg_ba::SampleStore &S = h->store;
    const int n = (int) src.size();
    std::vector<InsCutJob> jobs;
    std::vector<std::pair<int, int>> job_of;
    size_t cut_rows = 0, n_fac = 0;
    for (int w = 0; w < n; w++)
        for (int k = 0; k < (int) src[w].size(); k++) {
            n_fac++;
            const StoreSrc &q = src[w][k];
            if (q.kind != STORE_CUT) continue;
            jobs.push_back(InsCutJob{q.t0, q.t1, q.stream, ins->head[q.stream], ins->count[q.stream], (int) std::min<size_t>(cut_rows, INT32_MAX)});
            job_of.push_back({w, k});
            cut_rows += (size_t) ins->count[q.stream] + 2;  // getImuSeriesFromTo's bound
        }
    if (cut_rows >= (size_t) INT32_MAX / 8 || n_fac >= (size_t) INT32_MAX / 8) {
        set_error("%s: too many IMU rows in one call", fn);
        return ICG_EINVAL;
    }
    const size_t nj = jobs.size();
    Layout lay;
    const size_t b_job = lay.take(sizeof(InsCutJob) * nj), b_n = lay.take(4 * nj), b_st = lay.take(4 * nj), b_seg = lay.take(sizeof(StoreSeg) * 2 * n_fac);
    cudaStream_t s = h->stream;
    int rc = hd_reserve(h, S.stage, lay.size(), fn);  // every call of the store synchronises before it returns: the old one is idle
    if (rc != ICG_OK) return rc;
    if ((rc = grow_rows(S.cut, S.cut_cap, cut_rows, s, fn)) != ICG_OK) return rc;
    unsigned char *H = S.stage.h, *Dv = S.stage.d;
    const int32_t *got_n = (const int32_t *) (H + b_n), *got_st = (const int32_t *) (H + b_st);
    if (nj > 0) {
        memcpy(H + b_job, jobs.data(), sizeof(InsCutJob) * nj);
        ICG_CUDA(cudaMemcpyAsync(Dv, H, b_n, cudaMemcpyHostToDevice, s));
        if (!h->ins_ev) ICG_CUDA(cudaEventCreateWithFlags(&h->ins_ev, cudaEventDisableTiming));
        ICG_CUDA(cudaEventRecord(h->ins_ev, ins->stream));  // the pushes and redos queued on the INS handle come first
        ICG_CUDA(cudaStreamWaitEvent(s, h->ins_ev, 0));
        ICG_CUDA(ins_cut_launch(ins, (int) nj, (const InsCutJob *) Dv, S.cut, (int32_t *) (Dv + b_n), (int32_t *) (Dv + b_st), s));
        ICG_CUDA(cudaMemcpyAsync(H + b_n, Dv + b_n, b_seg - b_n, cudaMemcpyDeviceToHost, s));
        ICG_CUDA(cudaStreamSynchronize(s));
        for (size_t q = 0; q < nj; q++)
            if (got_st[q] != 1) bad.push_back(job_of[q]);
        if (!bad.empty()) {
            const InsCutJob &J = jobs[std::find(job_of.begin(), job_of.end(), bad[0]) - job_of.begin()];
            set_error("%s: window %d IMU factor %d: the INS window of stream %d cannot serve the interval %.17g .. %.17g", fn, bad[0].first,
                      bad[0].second, J.stream, J.t0, J.t1);
            return ICG_EINVAL;
        }
    }
    // the next store's layout, window after window, factor after factor
    std::vector<StoreSeg> segs;
    row0.assign(n, {}), nrow.assign(n, {});
    size_t total = 0, q = 0;
    for (int w = 0; w < n; w++) {
        row0[w].assign(src[w].size(), -1), nrow[w].assign(src[w].size(), -1);
        for (int k = 0; k < (int) src[w].size(); k++) {
            const StoreSrc &f = src[w][k];
            const int at = (int) total;
            int m = -1;
            if (f.kind == STORE_CUT) {
                m = got_n[q];
                segs.push_back(StoreSeg{0, jobs[q++].out, at, m});
            } else if (f.kind == STORE_OLD && S.nrow[w][f.a] >= 0) {
                m = S.nrow[w][f.a];
                segs.push_back(StoreSeg{1, S.row0[w][f.a], at, m});
            } else if (f.kind == STORE_MERGE) {
                const int na = S.nrow[w][f.a], nb = S.nrow[w][f.a + 1];
                segs.push_back(StoreSeg{1, S.row0[w][f.a], at, na});
                if (nb > 1) segs.push_back(StoreSeg{1, S.row0[w][f.a + 1] + 1, at + na, nb - 1});
                m = na + nb - 1;
            }
            if (m < 0) continue;
            row0[w][k] = at, nrow[w][k] = m;
            total += (size_t) m;
        }
    }
    if (total >= (size_t) INT32_MAX / 8) {
        set_error("%s: too many IMU rows in one call", fn);
        return ICG_EINVAL;
    }
    const int nx = 1 - S.cur;
    if ((rc = grow_rows(S.d[nx], S.cap[nx], total, s, fn)) != ICG_OK) return rc;
    if (segs.empty()) return ICG_OK;
    memcpy(H + b_seg, segs.data(), sizeof(StoreSeg) * segs.size());
    ICG_CUDA(cudaMemcpyAsync(Dv + b_seg, H + b_seg, sizeof(StoreSeg) * segs.size(), cudaMemcpyHostToDevice, s));
    ba_store_gather_kernel<<<(unsigned) ((segs.size() + 3) / 4), 128, 0, s>>>((int) segs.size(), (const StoreSeg *) (Dv + b_seg), S.cut, S.d[S.cur],
                                                                             S.d[nx]);
    ICG_CHECK_LAUNCH();
    count_launch();
    return ICG_OK;
}

static void store_commit(icg_ba *h, std::vector<std::vector<int>> &row0, std::vector<std::vector<int>> &nrow) {
    h->store.cur = 1 - h->store.cur;
    h->store.row0.swap(row0), h->store.nrow.swap(nrow);
    h->store.valid = true;
}

// the checks every call that cuts from the INS windows shares
static int store_ins_ok(icg_ba *h, const icg_ins *ins, int n_windows, const char *fn) {
    if (!h || !ins || n_windows < 1) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->D.world > 1) {
        set_error("%s: not available on a landmark-sharded handle", fn);
        return ICG_EUNSUPPORTED;
    }
    if (ins->device != h->device) {
        set_error("%s: the INS windows are on device %d, the solver on device %d", fn, ins->device, h->device);
        return ICG_EINVAL;
    }
    if (h->cur_windows != n_windows) {
        set_error("%s: the handle holds %d uploaded windows, the call names %d", fn, h->cur_windows, n_windows);
        return ICG_EINVAL;
    }
    return ICG_OK;
}

// stream in range and mechanized, K node times increasing
static int cut_window_ok(const icg_ins *ins, int w, int stream, const double *node_time, int K, const char *fn) {
    if (stream < 0 || stream >= ins->max_streams || !ins->mech[stream]) {
        set_error("%s: window %d: INS stream %d is out of range or not mechanized", fn, w, stream);
        return ICG_EINVAL;
    }
    if (!node_time) {
        set_error("%s: window %d: arrays missing", fn, w);
        return ICG_EINVAL;
    }
    for (int j = 0; j + 1 < K; j++)
        if (!(node_time[j] < node_time[j + 1])) {
            set_error("%s: window %d: node_time[%d] = %.17g is not less than node_time[%d] = %.17g", fn, w, j, node_time[j], j + 1, node_time[j + 1]);
            return ICG_EINVAL;
        }
    return ICG_OK;
}


// ---- the culling (ba_cull.cu) of both entries: staging [windows | host lists] in, [windows | cam_pose | lm_pw | lm_depth | lm_outlier |
//      obs_outlier] out, one launch, one synchronisation, the outputs into io.  win[w]'s slices index the lists and the outputs alike.
//      built: the current built lists (nL landmarks, nO observations), copied back to the host with the outputs (with their keypoints
//      when want_kp); NULL: io's host lists, staged here.  Makes the culling current.
static int cull_run(icg_ba *h, int n, const icg_ba_problem *problems, const icg_camera *cam, double std, icg_ba_cull_window *io,
                    const std::vector<CullWin> &win, const std::vector<int> &nobs, size_t nL, size_t nO, size_t nK,
                    const icg_ba::BuiltLists *built, bool want_kp, const char *fn) {
    const BaCaps &C = h->C;
    const size_t sL = built ? 0 : nL, sO = built ? 0 : nO;  // the host lists' staging
    Layout lay;
    const size_t i_win = lay.take(sizeof(CullWin) * n), i_ref = lay.take(4 * sL), i_off = lay.take(4 * (sL + (built ? 0 : n))), i_node = lay.take(4 * sO),
                 i_rkp = lay.take(8 * sL), i_kp = lay.take(8 * sO);
    const size_t in_bytes = lay.size();
    const size_t o_win = lay.take(sizeof(CullOut) * n), o_pose = lay.take(96 * nK), o_pw = lay.take(24 * nL), o_depth = lay.take(8 * nL),
                 o_lmo = lay.take(nL), o_obso = lay.take(nO);
    const size_t out_bytes = lay.size() - in_bytes;
    h->culled.n = 0;  // the staging is rewritten (or replaced) from here
    h->lin_ready = false;  // parameters and factor activity change
    ICG_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    if (lay.size() > h->cull.n) ICG_CUDA(cudaStreamSynchronize(s));
    int rc = hd_reserve(h, h->cull, lay.size(), fn);
    if (rc != ICG_OK) return rc;
    unsigned char *H = h->cull.h, *Dv = h->cull.d;
    memcpy(H + i_win, win.data(), sizeof(CullWin) * n);
    for (int w = 0; !built && w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const icg_ba_cull_window &c = io[w];
        const CullWin &W = win[w];
        if (p.L == 0) {
            ((int *) (H + i_off))[W.off0] = 0;
            continue;
        }
        const int no = c.obs_off[p.L];
        memcpy(H + i_ref + 4 * (size_t) W.lm0, c.lm_ref_node, 4 * (size_t) p.L);
        memcpy(H + i_off + 4 * (size_t) W.off0, c.obs_off, 4 * ((size_t) p.L + 1));
        memcpy(H + i_rkp + 8 * (size_t) W.lm0, c.lm_ref_kp, 8 * (size_t) p.L);
        if (no > 0) memcpy(H + i_node + 4 * (size_t) W.obs0, c.obs_node, 4 * (size_t) no), memcpy(H + i_kp + 8 * (size_t) W.obs0, c.obs_kp, 8 * (size_t) no);
    }
    ICG_CUDA(cudaMemcpyAsync(Dv, H, in_bytes, cudaMemcpyHostToDevice, s));
    const CullSrc src = built ? built->dev()
                              : CullSrc{(const int *) (Dv + i_ref), (const int *) (Dv + i_off), (const int *) (Dv + i_node), nullptr,
                                        (const float *) (Dv + i_rkp), (const float *) (Dv + i_kp)};
    CullArgs a;
    a.cam = *cam, a.std = std;
    a.pose = h->D.pose, a.ext = h->D.ext, a.rho = h->D.rho, a.pose_stride = C.K * 7, a.rho_stride = C.L;
    a.win = (const CullWin *) (Dv + i_win), a.lm_ref_node = src.ref, a.obs_off = src.off, a.obs_node = src.node, a.lm_ref_kp = src.rkp, a.obs_kp = src.kp;
    a.out = (CullOut *) (Dv + o_win), a.cam_pose = (double *) (Dv + o_pose), a.lm_pw = (double *) (Dv + o_pw), a.lm_depth = (double *) (Dv + o_depth);
    a.lm_outlier = Dv + o_lmo, a.obs_outlier = Dv + o_obso;
    ICG_CUDA(launch_update_cull(a, n, s));
    count_launch();
    if (h->D.world > 1) {  // landmark shards: every rank's counters become the window's totals (the other outputs are the camera side or its shard's)
        rc = shard_xsum(h, (int *) (Dv + o_win + offsetof(CullOut, counts)), (int) (sizeof(CullOut) / sizeof(int)), n, 5, 0);
        if (rc != ICG_OK) return rc;
    }
    ICG_CUDA(cudaMemcpyAsync(H + in_bytes, Dv + in_bytes, out_bytes, cudaMemcpyDeviceToHost, s));
    if (built) {  // the integer lists on the host (icg_ba_marginalize_resident_culled's NULL lists read them there), the keypoints if asked
        const HostDev<unsigned char> &lb = built->buf[built->cur];
        const icg_ba::BuiltLists::At &at = built->at[built->cur];
        ICG_CUDA(cudaMemcpyAsync(lb.h, lb.d, want_kp ? at.end : at.rkp, cudaMemcpyDeviceToHost, s));
    }
    ICG_CUDA(cudaStreamSynchronize(s));
    if (h->D.world > 1 && (rc = shard_timed_out(h, fn)) != ICG_OK) return rc;
    h->culled = {n, win, nobs, src, Dv + o_lmo, Dv + o_obso, built ? built->host() : CullSrc{}};
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        icg_ba_cull_window &c = io[w];
        const CullWin &W = win[w];
        const CullOut &O = ((const CullOut *) (H + o_win))[w];
        memcpy(c.R_bc_out, O.R_bc, sizeof(c.R_bc_out)), memcpy(c.t_bc_out, O.t_bc, sizeof(c.t_bc_out));
        c.td_bc_out = O.td_bc, c.ext_accepted = O.ext_accepted;
        memcpy(c.counts, O.counts, sizeof(c.counts));
        memcpy(c.cam_pose, H + o_pose + 96 * (size_t) W.node0, 96 * (size_t) p.K);
        if (p.L == 0) continue;
        memcpy(c.lm_pw, H + o_pw + 24 * (size_t) W.lm0, 24 * (size_t) p.L);
        memcpy(c.lm_depth, H + o_depth + 8 * (size_t) W.lm0, 8 * (size_t) p.L);
        memcpy(c.lm_outlier, H + o_lmo + W.lm0, p.L);
        if (nobs[w] > 0) memcpy(c.obs_outlier, H + o_obso + W.obs0, nobs[w]);
    }
    return ICG_OK;
}

// ---- the culling on the lists the last vision slide built (icg_ba_update_and_cull_built and its collective form).  sharded
//      (icg_ba_shard_update_and_cull_built): each rank's lists are its shard's; every rank runs the checks of the plain call, then the group
//      agrees once (every rank's verdict and a fingerprint of what every rank must pass alike) before cull_run writes anything or exchanges
//      its counters, so that a rejection on any rank leaves every handle as it was, the last culling included.
static int cull_built_body(icg_ba *h, int n, const icg_ba_problem *problems, const icg_camera *cam, double reprojection_error_std,
                           icg_ba_cull_window *io, icg_ba_cull_lists *lists, const char *fn, bool sharded) {
    auto reject = [&](int code) { return sharded ? shard_agree(h, true, 0, fn) : code; };
    // built.n is 0 or the uploaded count, so a call over another window count fails here already
    int rc = resident_single_rank(h, n, problems, fn, sharded);
    if (rc != ICG_OK) return reject(rc);
    if (!cam || !io) {
        set_error("%s: bad arguments", fn);
        return reject(ICG_EINVAL);
    }
    if (h->built.n != n) {
        set_error("%s: no built lists of these %d windows are current (%s, with no upload or other slide since)", fn, n,
                  sharded ? "icg_ba_shard_slide_vision_resident" : "icg_ba_slide_vision_resident");
        return reject(ICG_EINVAL);
    }
    const BaCaps &C = h->C;
    std::vector<CullWin> win(n);
    size_t nK = 0;
    ArgPrint fp;  // sharded: the camera side, which every rank must pass alike
    fp.num(n), fp.arr(cam, 1), fp.arr(&reprojection_error_std, 1);
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const icg_ba_cull_window &c = io[w];
        const CullWin &lw = h->built.win[w];
        const int no = h->built.nobs[w];
        // the caller's observation arrays hold max_L + max_F entries: lists not shaped as the reference builds them (an entry listed twice
        // in the host lists the slide carried) can be longer
        if (no > C.L + C.F) {
            set_error("%s: window %d: the built lists hold %d observations, more than max_L + max_F = %d", fn, w, no, C.L + C.F);
            return reject(ICG_EINVAL);
        }
        if (p.K != lw.K || p.L != lw.L || p.K > C.K || !c.cam_pose || (p.L > 0 && (!c.lm_pw || !c.lm_depth || !c.lm_outlier)) || (no > 0 && !c.obs_outlier)) {
            set_error("%s: window %d: sizes differ from the built lists' (K %d, L %d) or arrays missing", fn, w, lw.K, lw.L);
            return reject(ICG_EINVAL);
        }
        if (c.lm_ref_node || c.lm_ref_kp || c.obs_off || c.obs_node || c.obs_kp || c.obs_factor) {
            set_error("%s: window %d: the lists are the built ones; their inputs must be NULL", fn, w);
            return reject(ICG_EINVAL);
        }
        CullWin &W = win[w];
        memcpy(W.R_bc, c.R_bc, sizeof(W.R_bc)), memcpy(W.t_bc, c.t_bc, sizeof(W.t_bc));
        W.td_bc = c.td_bc, W.K = p.K, W.L = p.L, W.estimate_ext = c.estimate_ext != 0, W.estimate_td = c.estimate_td != 0;
        W.lm0 = lw.lm0, W.off0 = lw.off0, W.obs0 = lw.obs0, W.node0 = (int) nK;
        nK += p.K;
        fp.num(p.K), fp.arr(c.R_bc, 9), fp.arr(c.t_bc, 3), fp.arr(&c.td_bc, 1), fp.num(W.estimate_ext), fp.num(W.estimate_td);
    }
    if (sharded && (rc = shard_agree(h, false, fp.get(), fn)) != ICG_OK) return rc;
    bool want_kp = false;
    for (int w = 0; lists && w < n; w++) want_kp = want_kp || lists[w].lm_ref_kp || lists[w].obs_kp;
    const icg_ba::BuiltLists &B = h->built;
    rc = cull_run(h, n, problems, cam, reprojection_error_std, io, win, B.nobs, B.nL, B.nO, nK, &B, want_kp, fn);
    if (rc != ICG_OK) return rc;
    const CullSrc hl = B.host();
    for (int w = 0; lists && w < n; w++) {
        const int L = problems[w].L, no = B.nobs[w];
        const CullWin &W = win[w];
        icg_ba_cull_lists &o = lists[w];
        o.n_obs = no;
        if (o.lm_ref_node) memcpy(o.lm_ref_node, hl.ref + W.lm0, 4 * (size_t) L);
        if (o.obs_off) memcpy(o.obs_off, hl.off + W.off0, 4 * ((size_t) L + 1));
        if (o.obs_node) memcpy(o.obs_node, hl.node + W.obs0, 4 * (size_t) no);
        if (o.obs_factor) memcpy(o.obs_factor, hl.fac + W.obs0, 4 * (size_t) no);
        if (o.lm_ref_kp) memcpy(o.lm_ref_kp, hl.rkp + 2 * (size_t) W.lm0, 8 * (size_t) L);
        if (o.obs_kp) memcpy(o.obs_kp, hl.kp + 2 * (size_t) W.obs0, 8 * (size_t) no);
    }
    return ICG_OK;
}

extern "C" {

int icg_ba_marginalize(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out) {
    return marginalize_body(h, n_windows, problems, num_marg, out, false);
}

int icg_ba_marginalize_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, icg_ba_prior *out) {
    if (h && h->D.world > 1) return marginalize_sharded(h, n_windows, problems, num_marg, out, nullptr, "icg_ba_marginalize_resident");
    return marginalize_body(h, n_windows, problems, num_marg, out, true);
}

int icg_ba_update_and_cull_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const icg_camera *cam, double reprojection_error_std,
                                    icg_ba_cull_window *io) {
    static const char *fn = "icg_ba_update_and_cull_resident";
    int rc = resident_single_rank(h, n_windows, problems, fn, true);
    if (rc != ICG_OK) return rc;
    if (!cam || !io) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    const BaCaps &C = h->C;
    const int n = n_windows;
    std::vector<CullWin> win(n);
    std::vector<int> nobs(n);
    size_t nL = 0, nO = 0, nK = 0;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const icg_ba_cull_window &c = io[w];
        if (p.K < 2 || p.K > C.K || p.L < 0 || p.L > C.L || !c.cam_pose ||
            (p.L > 0 && (!c.lm_ref_node || !c.lm_ref_kp || !c.obs_off || !c.lm_pw || !c.lm_depth || !c.lm_outlier))) {
            set_error("%s: window %d: sizes out of range or arrays missing", fn, w);
            return ICG_EINVAL;
        }
        const int no = p.L > 0 ? c.obs_off[p.L] : 0;
        if (p.L > 0 && (c.obs_off[0] != 0 || no < 0 || no > INT32_MAX - (int64_t) nO || (no > 0 && (!c.obs_node || !c.obs_kp || !c.obs_outlier)))) {
            set_error("%s: window %d: obs_off must start at 0 and observation arrays must be given", fn, w);
            return ICG_EINVAL;
        }
        for (int l = 0; l < p.L; l++) {
            if (c.obs_off[l + 1] < c.obs_off[l] || c.lm_ref_node[l] < 0 || c.lm_ref_node[l] >= p.K) {
                set_error("%s: window %d landmark %d: obs_off not monotone or reference node out of range", fn, w, l);
                return ICG_EINVAL;
            }
        }
        for (int o = 0; o < no; o++)
            if (c.obs_node[o] < 0 || c.obs_node[o] >= p.K) {
                set_error("%s: window %d observation %d: node %d out of range", fn, w, o, c.obs_node[o]);
                return ICG_EINVAL;
            }
        CullWin &W = win[w];
        memcpy(W.R_bc, c.R_bc, sizeof(W.R_bc)), memcpy(W.t_bc, c.t_bc, sizeof(W.t_bc));
        W.td_bc = c.td_bc, W.K = p.K, W.L = p.L, W.estimate_ext = c.estimate_ext != 0, W.estimate_td = c.estimate_td != 0;
        W.lm0 = (int) nL, W.off0 = (int) (nL + w), W.obs0 = (int) nO, W.node0 = (int) nK;
        nobs[w] = no;
        nL += p.L, nO += no, nK += p.K;
    }
    return cull_run(h, n, problems, cam, reprojection_error_std, io, win, nobs, nL, nO, nK, nullptr, false, fn);
}

int icg_ba_update_and_cull_built(icg_ba *h, int n_windows, const icg_ba_problem *problems, const icg_camera *cam, double reprojection_error_std,
                                 icg_ba_cull_window *io, icg_ba_cull_lists *lists) {
    static const char *fn = "icg_ba_update_and_cull_built";
    if (h && h->D.world > 1) {
        set_error("%s: not available on a landmark-sharded handle (its group calls icg_ba_shard_update_and_cull_built)", fn);
        return ICG_EUNSUPPORTED;
    }
    return cull_built_body(h, n_windows, problems, cam, reprojection_error_std, io, lists, fn, false);
}

int icg_ba_shard_update_and_cull_built(icg_ba *h, int n_windows, const icg_ba_problem *problems, const icg_camera *cam, double reprojection_error_std,
                                       icg_ba_cull_window *io, icg_ba_cull_lists *lists) {
    const char *fn = "icg_ba_shard_update_and_cull_built";
    const int rc = shard_group_only(h, fn, "icg_ba_update_and_cull_built");
    return rc != ICG_OK ? rc : cull_built_body(h, n_windows, problems, cam, reprojection_error_std, io, lists, fn, true);
}
int icg_ba_reintegrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                icg_ba_reint_window *io) {
    return reint_body(h, n_windows, problems, noise5, station3, io, "icg_ba_reintegrate_resident", false);
}

int icg_ba_shard_reintegrate_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                      icg_ba_reint_window *io) {
    const char *fn = "icg_ba_shard_reintegrate_resident";
    const int rc = shard_group_only(h, fn, "icg_ba_reintegrate_resident");
    return rc != ICG_OK ? rc : reint_body(h, n_windows, problems, noise5, station3, io, fn, true);
}

int icg_ba_marginalize_resident_culled(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg,
                                       const icg_ba_cull_window *culled, const uint8_t *const *node_in_map, icg_ba_prior *out) {
    int rc = resident_single_rank(h, n_windows, problems, "icg_ba_marginalize_resident_culled", true);
    if (rc != ICG_OK) return rc;
    if (!culled || !node_in_map) {
        set_error("icg_ba_marginalize_resident_culled: bad arguments");
        return ICG_EINVAL;
    }
    // the factor set of gvinsMarginalization (IG/ic_gvins.cc:1558-1609) from the culling's flags: on the host, beside the structure loop
    // of marginalize_body, which reads the factor set on the host as well
    std::vector<std::vector<uint8_t>> masks(n_windows);
    std::vector<const uint8_t *> mp(n_windows);
    // a NULL list after a built culling is that culling's own (its host copy)
    const icg_ba::CullResult &cul = h->culled;
    const bool built = cul.n == n_windows && cul.host.ref;
    for (int w = 0; w < n_windows; w++) {
        const icg_ba_problem &p = problems[w];
        icg_ba_cull_window c = culled[w];
        if (!c.lm_ref_node || !c.obs_off || !c.obs_node || !c.obs_factor) {
            const CullWin *bw = built ? &cul.win[w] : nullptr;
            if (p.L > 0 && (!bw || bw->L != p.L || bw->K != p.K)) {
                set_error("icg_ba_marginalize_resident_culled: window %d: lists missing, and no built culling of these windows is current", w);
                return ICG_EINVAL;
            }
            if (bw) {
                if (!c.lm_ref_node) c.lm_ref_node = cul.host.ref + bw->lm0;
                if (!c.obs_off) c.obs_off = cul.host.off + bw->off0;
                if (!c.obs_node) c.obs_node = cul.host.node + bw->obs0;
                if (!c.obs_factor) c.obs_factor = cul.host.fac + bw->obs0;
            }
        }
        if (!node_in_map[w] || (p.L > 0 && (!c.lm_ref_node || !c.obs_off || !c.lm_outlier)) || p.K > h->C.K || p.L > h->C.L || p.F > h->C.F ||
            (p.L > 0 && c.obs_off[p.L] > 0 && (!c.obs_node || !c.obs_factor || !c.obs_outlier))) {
            set_error("icg_ba_marginalize_resident_culled: window %d: arrays missing", w);
            return ICG_EINVAL;
        }
        std::vector<uint8_t> &m = masks[w];
        m.assign(p.F, 1);
        std::vector<uint8_t> lm_bad(p.L, 0);
        for (int l = 0; l < p.L; l++) {
            lm_bad[l] = c.lm_outlier[l] != 0;
            for (int o = c.obs_off[l]; o < c.obs_off[l + 1]; o++) {
                const int f = c.obs_factor[o], k = c.obs_node[o];
                if (f < -1 || f >= p.F || (f >= 0 && (p.f_lm[f] != l || p.f_obs[f] != k))) {
                    set_error("icg_ba_marginalize_resident_culled: window %d landmark %d: observation %d names factor %d of another landmark or node", w, l, o, f);
                    return ICG_EINVAL;
                }
                if (!c.obs_outlier[o]) continue;
                if (k == c.lm_ref_node[l]) lm_bad[l] = 1;
                if (f >= 0) m[f] = 0;
            }
        }
        for (int f = 0; f < p.F; f++)
            if (lm_bad[p.f_lm[f]] || !node_in_map[w][p.f_obs[f]]) m[f] = 0;
        mp[w] = m.data();
    }
    if (h->D.world > 1) return marginalize_sharded(h, n_windows, problems, num_marg, out, mp.data(), "icg_ba_marginalize_resident_culled");
    return marginalize_body(h, n_windows, problems, num_marg, out, true, mp.data());
}

int icg_ba_marginalize_built(icg_ba *h, int n_windows, const icg_ba_problem *problems, const int32_t *num_marg, const uint8_t *const *node_in_map,
                             icg_ba_prior *out) {
    static const char *fn = "icg_ba_marginalize_built";
    if (h && h->D.world > 1) {
        set_error("%s: not available on a landmark-sharded handle (its group marginalizes with icg_ba_marginalize_resident_culled and NULL lists "
                  "after icg_ba_shard_update_and_cull_built)", fn);
        return ICG_EUNSUPPORTED;
    }
    int rc = resident_single_rank(h, n_windows, problems, fn);
    if (rc != ICG_OK) return rc;
    if (!num_marg || !node_in_map || !out) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    const icg_ba::CullResult &cul = h->culled;
    if (cul.n != n_windows) {
        set_error("%s: no culling of these %d windows is current (icg_ba_update_and_cull_built, with no upload or slide since)", fn, n_windows);
        return ICG_EINVAL;
    }
    if (!cul.host.ref) {
        set_error("%s: the current culling walked host lists (icg_ba_update_and_cull_resident); this call needs a culling on the built lists "
                  "(icg_ba_update_and_cull_built)", fn);
        return ICG_EINVAL;
    }
    const BaCaps &C = h->C;
    const int n = n_windows;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const CullWin &W = cul.win[w];
        if (p.K != W.K || p.L != W.L || !node_in_map[w]) {
            set_error("%s: window %d: sizes differ from the culled window's (K %d, L %d) or node_in_map missing", fn, w, W.K, W.L);
            return ICG_EINVAL;
        }
        if (!marg_out_ok(p, num_marg[w], out[w])) {
            set_error("%s: window %d: num_marg=%d out of range or output arrays missing / too small (rcap=%d)", fn, w, num_marg[w], out[w].rcap);
            return ICG_EINVAL;
        }
    }
    ICG_CUDA(cudaSetDevice(h->device));
    if ((rc = marg_alloc(h)) != ICG_OK) return rc;
    if (!h->marg_ftab) {
        if (cudaMalloc(&h->marg_ftab, sizeof(int) * (size_t) C.NW * std::max(1, C.F)) != cudaSuccess) {
            h->marg_ftab = nullptr;
            set_error("%s: scratch allocation failed", fn);
            return ICG_ENOMEM;
        }
        h->dev_only.push_back(h->marg_ftab);
    }
    // staging [MargSelWin x n | per window MARG_SEL_HDR + 2 max_K ints out]: the camera side up, the headers and block tables down
    const int so = MARG_SEL_HDR + 2 * C.K;
    Layout lay;
    const size_t i_win = lay.take(sizeof(MargSelWin) * n), i_out = lay.take(sizeof(int) * (size_t) n * so);
    if ((rc = hd_reserve(h, h->marg_sel, lay.size(), fn)) != ICG_OK) return rc;
    unsigned char *H = h->marg_sel.h, *Dv = h->marg_sel.d;
    for (int w = 0; w < n; w++) {
        const icg_ba_problem &p = problems[w];
        const CullWin &cw = cul.win[w];
        MargSelWin &W = ((MargSelWin *) (H + i_win))[w];
        memset(&W, 0, sizeof(W));
        W.lm0 = cw.lm0, W.off0 = cw.off0, W.obs0 = cw.obs0, W.num_marg = num_marg[w];
        char tp[BA_MAX_NODES] = {}, tm[BA_MAX_NODES] = {};
        bool ext = false, td = false;
        marg_camera_touched(p, num_marg[w], tp, tm, &ext, &td);
        for (int k = 0; k < p.K; k++) W.tp[k] = tp[k], W.tm[k] = tm[k], W.in_map[k] = node_in_map[w][k] != 0;
        W.ext = ext, W.td = td;
    }
    cudaStream_t s = h->stream;
    ICG_CUDA(cudaMemcpyAsync(Dv + i_win, H + i_win, sizeof(MargSelWin) * n, cudaMemcpyHostToDevice, s));
    MargSelArgs a;
    a.win = (const MargSelWin *) (Dv + i_win);
    a.ref = cul.dev.ref, a.off = cul.dev.off, a.node = cul.dev.node, a.fac = cul.dev.fac;
    a.lm_outlier = cul.lm_outlier, a.obs_outlier = cul.obs_outlier;
    a.fmask = h->marg_fmask.d, a.ftab = h->marg_ftab, a.out = (int *) (Dv + i_out);
    marg_select_built<<<n, MARG_SEL_THREADS, 0, s>>>(C, h->D, h->M, a);
    ICG_CHECK_LAUNCH();
    count_launch();
    ICG_CUDA(cudaMemcpyAsync(H + i_out, Dv + i_out, sizeof(int) * (size_t) n * so, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    // every check before the marginalization kernels: a rejected call leaves the culling, the built lists and the resident prior current
    const int *hdr = (const int *) (H + i_out);
    for (int w = 0; w < n; w++)
        if (hdr[(size_t) w * so + 3] > 0) {
            set_error("%s: window %d: %d observations of the built lists name a factor outside [-1, F) or one of another landmark or node", fn, w,
                      hdr[(size_t) w * so + 3]);
            return ICG_EINVAL;
        }
    for (int w = 0; w < n; w++) {
        const int *o = hdr + (size_t) w * so, m = o[0], r = o[1];
        if (m > MARG_MAXN || r > MARG_MAXN) {
            set_error("%s: window %d: %s=%d exceeds the %d rows of the largest eigensolver kernel", fn, w, m > MARG_MAXN ? "m" : "r", m > MARG_MAXN ? m : r,
                      MARG_MAXN);
            return ICG_EUNSUPPORTED;
        }
    }
    for (int w = 0; w < n; w++) {
        const int *o = hdr + (size_t) w * so;
        icg_ba_prior &q = out[w];
        q.m = o[0], q.r = o[1], q.nblocks = o[2];
        for (int b = 0; b < q.nblocks; b++) q.block_type[b] = o[MARG_SEL_HDR + b] & 3, q.block_node[b] = o[MARG_SEL_HDR + b] >> 2;
    }
    h->prior.n = 0;  // the workspace is about to be overwritten
    h->lin_ready = false;  // the linearisation takes the buffer the window uses
    return marg_solve(h, n, problems, num_marg, out, true, nullptr, nullptr, true);
}

int icg_ba_slide_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry) {
    return slide_body(h, n, next, carry, nullptr, nullptr, nullptr, "icg_ba_slide_resident", false);
}

int icg_ba_slide_integrate_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                                    const double *noise5, const double *station3) {
    if (!integ) {
        set_error("icg_ba_slide_integrate_resident: bad arguments");
        return ICG_EINVAL;
    }
    return slide_body(h, n, next, carry, integ, noise5, station3, "icg_ba_slide_integrate_resident", false);
}

int icg_ba_slide_vision_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry, const icg_ba_slide_integrate *integ,
                                 const double *noise5, const double *station3, icg_ba_slide_vision *vis) {
    static const char *fn = "icg_ba_slide_vision_resident";
    if (h && h->D.world > 1) {
        set_error("%s: not available on a landmark-sharded handle (its group calls icg_ba_shard_slide_vision_resident)", fn);
        return ICG_EUNSUPPORTED;
    }
    return vision_body(h, n, next, carry, integ, noise5, station3, vis, fn, false);
}

int icg_ba_shard_slide_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry) {
    const char *fn = "icg_ba_shard_slide_resident";
    const int rc = shard_group_only(h, fn, "icg_ba_slide_resident");
    return rc != ICG_OK ? rc : slide_body(h, n, next, carry, nullptr, nullptr, nullptr, fn, true);
}

int icg_ba_shard_slide_integrate_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                          const icg_ba_slide_integrate *integ, const double *noise5, const double *station3) {
    const char *fn = "icg_ba_shard_slide_integrate_resident";
    int rc = shard_group_only(h, fn, "icg_ba_slide_integrate_resident");
    if (rc != ICG_OK) return rc;
    if (!integ) {  // still a collective call: the rank joins the agreement with its rejection
        set_error("%s: bad arguments", fn);
        shard_agree(h, true, 0, fn);
        return ICG_EINVAL;
    }
    return slide_body(h, n, next, carry, integ, noise5, station3, fn, true);
}

int icg_ba_shard_slide_vision_resident(icg_ba *h, int n, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                                       const icg_ba_slide_integrate *integ, const double *noise5, const double *station3, icg_ba_slide_vision *vis) {
    const char *fn = "icg_ba_shard_slide_vision_resident";
    const int rc = shard_group_only(h, fn, "icg_ba_slide_vision_resident");
    return rc != ICG_OK ? rc : vision_body(h, n, next, carry, integ, noise5, station3, vis, fn, true);
}

int icg_ba_imu_samples_from_ins(icg_ba *h, icg_ins *ins, int n_windows, const icg_ba_ins_cut *cut) {
    static const char *fn = "icg_ba_imu_samples_from_ins";
    int rc = store_ins_ok(h, ins, n_windows, fn);
    if (rc != ICG_OK) return rc;
    if (!cut) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    std::vector<std::vector<StoreSrc>> src(n_windows);
    for (int w = 0; w < n_windows; w++) {
        const WinDims &d = h->dims.h[w];
        if ((rc = cut_window_ok(ins, w, cut[w].stream, cut[w].node_time, d.K, fn)) != ICG_OK) return rc;
        for (int k = 0; k < d.n_imu; k++) src[w].push_back(StoreSrc{STORE_CUT, 0, cut[w].stream, cut[w].node_time[k], cut[w].node_time[k + 1]});
    }
    ICG_CUDA(cudaSetDevice(h->device));
    std::vector<std::vector<int>> row0, nrow;
    std::vector<std::pair<int, int>> bad;
    if ((rc = store_build(h, ins, src, fn, row0, nrow, bad)) != ICG_OK) return rc;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    store_commit(h, row0, nrow);
    return ICG_OK;
}

int icg_ba_slide_ins_resident(icg_ba *h, icg_ins *ins, int n_windows, const icg_ba_problem *next, const icg_ba_slide_window *carry,
                              const icg_ba_slide_ins *io, const double *noise5, const double *station3, icg_ba_slide_vision *vis) {
    static const char *fn = "icg_ba_slide_ins_resident";
    int rc = store_ins_ok(h, ins, n_windows, fn);
    if (rc != ICG_OK) return rc;
    if (!next || !carry || !io || !noise5 || !station3) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    // each new factor's rows: carried, cut from the INS window, merged from two old factors, or none (a blob read from next)
    std::vector<std::vector<StoreSrc>> src(n_windows);
    for (int w = 0; w < n_windows; w++) {
        const icg_ba_problem &p = next[w];
        const icg_ba_slide_window &c = carry[w];
        const icg_ba_slide_ins &g = io[w];
        const int on = h->dims.h[w].n_imu;
        if (g.integ.imu || g.integ.imu_off) {
            set_error("%s: window %d: integ.imu and integ.imu_off must be NULL (the rows are cut from the INS window)", fn, w);
            return ICG_EINVAL;
        }
        if (p.K < 2 || p.K > h->C.K || p.n_imu < 0 || p.n_imu > p.K - 1) {
            set_error("%s: window %d: sizes out of range", fn, w);
            return ICG_EINVAL;
        }
        bool cuts = false;
        for (int k = 0; k < p.n_imu; k++) {
            StoreSrc f = {STORE_NONE, 0, g.stream, 0, 0};
            const int from = g.integ.imu_from ? g.integ.imu_from[k] : -1;
            if (c.imu_src && c.imu_src[k] >= 0) {
                if (c.imu_src[k] >= on) {
                    set_error("%s: window %d: imu_src[%d] = %d is out of range of the old window (%d)", fn, w, k, c.imu_src[k], on);
                    return ICG_EINVAL;
                }
                if (h->store.valid) f.kind = STORE_OLD, f.a = c.imu_src[k];
            } else if (from == ICG_SLIDE_ROW) {
                const int a = g.merge_src ? g.merge_src[k] : -1;
                if (a < 0 || a + 1 >= on || !h->store.valid || h->store.nrow[w][a] < 1 || h->store.nrow[w][a + 1] < 1) {
                    set_error("%s: window %d factor %d: merge_src must name old factors a and a + 1 that both hold samples", fn, w, k);
                    return ICG_EINVAL;
                }
                f.kind = STORE_MERGE, f.a = a;
            } else if (from >= 0 || from == ICG_SLIDE_CHAIN) {
                f.kind = STORE_CUT, cuts = true;
            } else if (from != -1) {
                set_error("%s: window %d: imu_from[%d] = %d is not a source", fn, w, k, from);
                return ICG_EINVAL;
            }
            src[w].push_back(f);
        }
        if (cuts && (rc = cut_window_ok(ins, w, g.stream, g.node_time, p.K, fn)) != ICG_OK) return rc;
        for (int k = 0; k < p.n_imu; k++)
            if (src[w][k].kind == STORE_CUT) src[w][k].t0 = g.node_time[k], src[w][k].t1 = g.node_time[k + 1];
    }
    ICG_CUDA(cudaSetDevice(h->device));
    std::vector<std::vector<int>> row0, nrow;
    std::vector<std::pair<int, int>> bad;
    rc = store_build(h, ins, src, fn, row0, nrow, bad);
    if (!bad.empty()) {  // status -2 where the INS window cannot serve the interval
        for (int w = 0; w < n_windows; w++)
            if (io[w].integ.status) memset(io[w].integ.status, 0, (size_t) next[w].n_imu);
        for (const auto &b : bad)
            if (io[b.first].integ.status) io[b.first].integ.status[b.second] = -2;
    }
    if (rc != ICG_OK) return rc;
    std::vector<icg_ba_slide_integrate> integ(n_windows);
    for (int w = 0; w < n_windows; w++) integ[w] = io[w].integ;
    const FactorRows fr = {h->store.d[1 - h->store.cur], row0, nrow};
    rc = vis ? vision_body(h, n_windows, next, carry, integ.data(), noise5, station3, vis, fn, false, &fr)
             : slide_body(h, n_windows, next, carry, integ.data(), noise5, station3, fn, false, nullptr, nullptr, &fr);
    if (rc != ICG_OK) return rc;
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    for (int w = 0; w < n_windows; w++)
        if (io[w].n_rows) memcpy(io[w].n_rows, nrow[w].data(), sizeof(int) * nrow[w].size());
    store_commit(h, row0, nrow);
    return ICG_OK;
}

int icg_ba_reintegrate_stored_resident(icg_ba *h, int n_windows, const icg_ba_problem *problems, const double *noise5, const double *station3,
                                       icg_ba_reint_window *io) {
    static const char *fn = "icg_ba_reintegrate_stored_resident";
    int rc = resident_single_rank(h, n_windows, problems, fn);
    if (rc != ICG_OK) return rc;
    if (!io) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (!h->store.valid) {
        set_error("%s: the handle holds no IMU samples (an upload or a slide other than icg_ba_slide_ins_resident replaced the windows since "
                  "the last icg_ba_imu_samples_from_ins)", fn);
        return ICG_EINVAL;
    }
    for (int w = 0; w < n_windows; w++)
        if (io[w].imu || io[w].imu_off) {
            set_error("%s: window %d: imu and imu_off must be NULL (the rows are the store's)", fn, w);
            return ICG_EINVAL;
        }
    const FactorRows fr = {h->store.d[h->store.cur], h->store.row0, h->store.nrow};
    return reint_body(h, n_windows, problems, noise5, station3, io, fn, false, &fr);
}

int icg_ba_imu_samples(icg_ba *h, int window, int cap_rows, int32_t *off, double *rows) {
    static const char *fn = "icg_ba_imu_samples";
    if (!h || window < 0 || window >= h->cur_windows || cap_rows < 0 || !off || (cap_rows > 0 && !rows)) {
        set_error("%s: bad arguments", fn);
        return ICG_EINVAL;
    }
    if (h->D.world > 1) {
        set_error("%s: not available on a landmark-sharded handle", fn);
        return ICG_EUNSUPPORTED;
    }
    if (!h->store.valid) {
        set_error("%s: the handle holds no IMU samples", fn);
        return ICG_EINVAL;
    }
    const std::vector<int> &r0 = h->store.row0[window], &nr = h->store.nrow[window];
    int first = -1, total = 0;
    for (size_t k = 0; k < nr.size(); k++) {
        off[k] = nr[k] < 0 ? -1 : total;
        if (nr[k] < 0) continue;
        if (first < 0) first = r0[k];
        total += nr[k];
    }
    off[nr.size()] = total;
    const int m = std::min(total, cap_rows);
    if (m == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaMemcpyAsync(rows, h->store.d[h->store.cur] + 7 * (size_t) first, 56 * (size_t) m, cudaMemcpyDeviceToHost, h->stream));
    ICG_CUDA(cudaStreamSynchronize(h->stream));
    return ICG_OK;
}

}  // extern "C"
