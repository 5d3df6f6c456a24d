// ba_slide.cu -- the device half of icg_ba_slide_resident (ba_slide.cuh).  Built with -fmad=false: ba_slide_prior's products and sums must each
// be rounded on their own, as the host loop of icg_ba_upload rounds them (x86-64 baseline: no FMA), so that a slid window's prior normal
// equations are the uploaded window's bit for bit.  The intrinsics below say the same thing explicitly.
#include "ba_slide.cuh"

namespace icg {

constexpr int SLIDE_THREADS = 256;

// One grid-stride pass per window (blockIdx.y) over the flattened destination rows [nodes 16 | landmarks 1 | record slots 14 | IMU factors 705 |
// GNSS fixes 6]: every destination double is written once, from the old copy or from the staged row.
__global__ void __launch_bounds__(SLIDE_THREADS) ba_slide_gather(SlideArgs a) {
    const int w = blockIdx.y;
    const SlideWin W = a.win[w];
    const int n0 = W.K * SLIDE_NODE, n1 = n0 + W.L, n2 = n1 + W.F * 14, n3 = n2 + W.n_imu * SLIDE_IMU, n4 = n3 + W.n_gnss * SLIDE_GNSS;
    const size_t wK = (size_t) w * a.K, wL = (size_t) w * a.L, wF = (size_t) w * a.F, wG = (size_t) w * a.G;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += gridDim.x * blockDim.x) {
        if (e < n0) {
            const int k = e / SLIDE_NODE, c = e % SLIDE_NODE, m = a.map[W.node_map + k];
            if (c < 7)
                a.pose[(wK + k) * 7 + c] = m >= 0 ? a.old_pose[(wK + m) * 7 + c] : a.val[-(m + 1) + c];
            else
                a.mix[(wK + k) * 9 + c - 7] = m >= 0 ? a.old_mix[(wK + m) * 9 + c - 7] : a.val[-(m + 1) + c];
        } else if (e < n1) {
            // updateParametersFromOptimizer stores depth = 1 / invdepth, the next addReprojectionParameters invdepth = 1 / depth
            const int l = e - n0, m = (W.vis ? a.vmap : a.map)[W.lm_map + l];
            a.rho[wL + l] = m >= 0 ? __ddiv_rn(1.0, __ddiv_rn(1.0, a.old_rho[wL + m])) : (W.vis ? a.vlm : a.val)[-(m + 1)];
        } else if (e < n2) {
            const int q = (e - n1) / 14, c = (e - n1) % 14, m = (W.vis ? a.vmap : a.map)[W.slot_map + q];
            a.fc[(wF + q) * 14 + c] = m >= 0 ? a.old_fc[(wF + m) * 14 + c] : (W.vis ? a.vfc : a.val)[-(m + 1) + c];
        } else if (e < n3) {
            const int k = (e - n2) / SLIDE_IMU, c = (e - n2) % SLIDE_IMU, m = a.map[W.imu_map + k];
            if (c < 480)
                a.blob[(wK + k) * 480 + c] = m >= 0 ? a.old_blob[(wK + m) * 480 + c] : a.val[-(m + 1) + c];
            else
                a.U[(wK + k) * 225 + c - 480] = m >= 0 ? a.old_U[(wK + m) * 225 + c - 480] : a.val[-(m + 1) + c];
        } else {
            const int g = (e - n3) / SLIDE_GNSS, c = (e - n3) % SLIDE_GNSS, m = a.map[W.gnss_map + g];
            if (c < 3)
                a.blh[(wG + g) * 3 + c] = m >= 0 ? a.old_blh[(wG + m) * 3 + c] : a.val[-(m + 1) + c];
            else
                a.std[(wG + g) * 3 + c - 3] = m >= 0 ? a.old_std[(wG + m) * 3 + c - 3] : a.val[-(m + 1) + c];
        }
    }
}

// Thread per entry of [H0 (r x r, upper triangle computed, mirrored) | b0 (r) | c0]: the serial k loop of icg_ba_upload, k ascending, every
// product and every sum rounded (no contraction, no reordering), so the result is the host's bit for bit.  Adjacent threads take adjacent j:
// the J0[k][j] loads coalesce, J0[k][i] is a broadcast.
__global__ void __launch_bounds__(SLIDE_THREADS) ba_slide_prior(SlideArgs a) {
    const int w = blockIdx.y;
    const SlideWin W = a.win[w];
    const int r = W.r;
    if (r <= 0) return;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e > r * r + r) return;
    // a window without a source (slot -1) sums nothing: its rows become zeros
    const bool src = !W.from_marg || W.slot >= 0;
    const int nk = src ? r : 0;
    const double *J0 = !W.from_marg ? a.val + W.j0 : src ? a.mJ0 + (size_t) W.slot * a.mrcap * a.mrcap : nullptr;
    const double *e0 = !W.from_marg ? a.val + W.e0 : src ? a.me0 + (size_t) W.slot * a.mrcap : nullptr;
    double s = 0;
    if (e < r * r) {
        const int i = e / r, j = e % r;
        if (j < i) return;
        for (int k = 0; k < nk; k++) s = __dadd_rn(s, __dmul_rn(J0[(size_t) k * r + i], J0[(size_t) k * r + j]));
        double *H0 = a.H0 + (size_t) w * a.R * a.R;
        H0[(size_t) i * r + j] = s, H0[(size_t) j * r + i] = s;
    } else if (e < r * r + r) {
        const int i = e - r * r;
        for (int k = 0; k < nk; k++) s = __dadd_rn(s, __dmul_rn(J0[(size_t) k * r + i], e0[k]));
        a.b0[(size_t) w * a.R + i] = s;
    } else {
        for (int k = 0; k < nk; k++) s = __dadd_rn(s, __dmul_rn(e0[k], e0[k]));
        a.c0[w] = s;
    }
}

cudaError_t preload_slide() {
    cudaFuncAttributes attr;
    cudaError_t e = cudaFuncGetAttributes(&attr, ba_slide_gather);
    return e == cudaSuccess ? cudaFuncGetAttributes(&attr, ba_slide_prior) : e;
}

cudaError_t launch_slide(const SlideArgs &a, int n_windows, int max_elems, int max_r, cudaStream_t stream) {
    if (max_elems > 0) {
        const int gx = (max_elems + SLIDE_THREADS - 1) / SLIDE_THREADS;
        ba_slide_gather<<<dim3(gx < 128 ? gx : 128, n_windows), SLIDE_THREADS, 0, stream>>>(a);
    }
    if (max_r > 0) ba_slide_prior<<<dim3((max_r * max_r + max_r + SLIDE_THREADS) / SLIDE_THREADS, n_windows), SLIDE_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace icg
