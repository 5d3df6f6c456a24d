// preint.cu -- PreintegrationEarth / PreintegrationNormal propagation (IG/preintegration/preintegration_earth.cc:205-338,
// preintegration_normal.cc:195-232) with one warp per interval.
//
//   every lane   the per-sample scalar chain of gc::preint_sample (bias compensation, dvfb, dtheta, the quaternion updates, cbb0), redundantly,
//                so that no lane waits for another's scalars
//   shared       jacobian_, covariance_, G = gt noise gt^T, phi's non-zero entries row by row, phi cov and phi G of this interval
//   lanes        the 15 x 15 products dealt out by output entry (entry lane + 32 t), __syncwarp between the phases
//
// Every entry is the sum of gc::preintegrate_core over k ascending, with the terms whose phi factor is a structural zero left out: such a
// term is +-0 when the other factor is finite, a sum that starts at +0 never becomes -0, and x + (+-0) == x, so for finite inputs the result
// is the scalar core's bit for bit (the file is built with -fmad=false, as geom.cu was).  phi's pattern (rows -> columns, ascending):
//   rows 0-2   i (I), i + 3 (dt I)
//   rows 3-5   i (I), 6..8 (cbb0 [cvl]x), 12..14 (dt cbb0)
//   rows 6-8   6..8 (I - [cth]x), i + 3 (-dt I)
//   rows 9-14  i ((1 - dt / corr) I)
// G is zero except its (3, 3) block (cbb0 diag(noise) cbb0^T) and the diagonal of rows 6-14, which does not change over the interval.
#include <math.h>

#include "geom_core.cuh"
#include "preint.cuh"

namespace icg {
namespace {

constexpr int PH_NZ = 7;                            // phi's widest row
constexpr int SM_PHI = 0, SM_J = 15 * PH_NZ, SM_C = SM_J + 225, SM_G = SM_C + 225, SM_PC = SM_G + 225, SM_PG = SM_PC + 225;
constexpr int SM_WARP = SM_PG + 225;                // doubles of shared memory per warp; G | PC | PG (675) is the sqrt-information workspace

__device__ __forceinline__ double sel9(const bam::M3 &m, int e) {  // m.m[e] without a dynamically indexed register array
    double v = m.m[0];
#pragma unroll
    for (int q = 1; q < 9; q++)
        if (q == e) v = m.m[q];
    return v;
}

// phi's column list (s_k) and row lengths (s_nz), shared by the CTA
__device__ void phi_pattern(signed char *s_k, signed char *s_nz) {
    const int i = threadIdx.x;
    if (i >= 15) return;
    signed char *k = s_k + i * PH_NZ;
    if (i < 3) {
        k[0] = i, k[1] = i + 3, s_nz[i] = 2;
    } else if (i < 6) {
        k[0] = i, k[1] = 6, k[2] = 7, k[3] = 8, k[4] = 12, k[5] = 13, k[6] = 14, s_nz[i] = 7;
    } else if (i < 9) {
        k[0] = 6, k[1] = 7, k[2] = 8, k[3] = i + 3, s_nz[i] = 4;
    } else {
        k[0] = i, s_nz[i] = 1;
    }
}

// one warp: propagate n rows of imu from the state S was begun with; leaves jacobian_ in sm + SM_J, covariance_ in sm + SM_C
__device__ void propagate(gc::PreintScalar &S, const double *noise5, const double *imu, int n, double *sm, const signed char *s_k, const signed char *s_nz,
                          int lane) {
    using namespace bam;
    double *phv = sm + SM_PHI, *J = sm + SM_J, *Cv = sm + SM_C, *G = sm + SM_G, *PC = sm + SM_PC, *PG = sm + SM_PG;
    double noise[12];
    gc::preint_noise(noise5, noise);
    const double corr = noise5[4];
    for (int e = lane; e < 225; e += 32) {
        const int i = e / 15, j = e - 15 * i;
        J[e] = i == j ? 1.0 : 0.0, Cv[e] = 0, G[e] = 0;
    }
    for (int e = lane; e < 15 * PH_NZ; e += 32) phv[e] = (e < 6 * PH_NZ && e % PH_NZ == 0) ? 1.0 : 0.0;  // the identity entries of rows 0-5
    __syncwarp();
    if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 3; r++) {
            G[(6 + r) * 16] = 0.0 + -1.0 * noise[r] * -1.0;  // gt(6, 0) = -I
            G[(9 + r) * 16] = 0.0 + 1.0 * noise[6 + r] * 1.0;
            G[(12 + r) * 16] = 0.0 + 1.0 * noise[9 + r] * 1.0;
        }
    }
    for (int s = 1; s < n; s++) {
        double dt;
        V3 cth, cvl;
        M3 cbb0;
        gc::preint_sample(S, imu + 7 * (size_t) (s - 1), imu + 7 * (size_t) s, dt, cth, cvl, cbb0);
        // this sample's entries of phi and of G's (3, 3) block, as preintegrate_core builds them
        {
            const int l = lane;
            if (l < 9) {
                const M3 P = mul(cbb0, skew(cvl));
                phv[(3 + l / 3) * PH_NZ + 1 + l % 3] = sel9(P, l);
                M3 Gb;
#pragma unroll
                for (int r = 0; r < 3; r++)
#pragma unroll
                    for (int c = 0; c < 3; c++) {
                        double a = 0;
#pragma unroll
                        for (int q = 0; q < 3; q++) a += cbb0.m[3 * r + q] * noise[3 + q] * cbb0.m[3 * c + q];
                        Gb.m[3 * r + c] = a;
                    }
                G[(3 + l / 3) * 15 + 3 + l % 3] = sel9(Gb, l);
            } else if (l < 18) {
                phv[(3 + (l - 9) / 3) * PH_NZ + 4 + (l - 9) % 3] = sel9(scale(dt, cbb0), l - 9);
            } else if (l < 27) {
                phv[(6 + (l - 18) / 3) * PH_NZ + (l - 18) % 3] = sel9(sub(ident(), skew(cth)), l - 18);
            } else if (l == 27) {
                const double d = dt * 1.0, md = -dt * 1.0;  // scale(dt, I), scale(-dt, I)
#pragma unroll
                for (int r = 0; r < 3; r++) phv[r * PH_NZ + 1] = d, phv[(6 + r) * PH_NZ + 3] = md;
            } else if (l == 28) {
                const double f = (1 - dt / corr) * 1.0;
#pragma unroll
                for (int r = 9; r < 15; r++) phv[r * PH_NZ] = f;
            }
        }
        __syncwarp();
        // phase 1: jacobian_ = phi jacobian_ (kept in registers until every lane has read the old one), PG = phi G, PC = phi covariance_
        double jn[8];
#pragma unroll
        for (int t = 0; t < 8; t++) {
            const int e = lane + 32 * t;
            jn[t] = 0;
            if (e < 225) {
                const int i = e / 15, j = e - 15 * i, nz = s_nz[i];
                double aj = 0, ag = 0, ac = 0;
                for (int q = 0; q < nz; q++) {
                    const int k = s_k[i * PH_NZ + q];
                    const double ph = phv[i * PH_NZ + q];
                    aj += ph * J[k * 15 + j], ag += ph * G[k * 15 + j], ac += ph * Cv[k * 15 + j];
                }
                jn[t] = aj, PG[e] = ag, PC[e] = ac;
            }
        }
        __syncwarp();
#pragma unroll
        for (int t = 0; t < 8; t++) {
            const int e = lane + 32 * t;
            if (e < 225) J[e] = jn[t];
        }
        // phase 2: covariance_ = PC phi^T + 0.5 dt (PG + G phi^T), entry (i, j) on lane (15 j + i) mod 32 so that a round shares phi's rows j
        for (int t = 0; t < 8; t++) {
            const int e = lane + 32 * t;
            if (e < 225) {
                const int j = e / 15, i = e - 15 * j, nz = s_nz[j];
                double a = 0, gpt = 0;
                for (int q = 0; q < nz; q++) {
                    const int k = s_k[j * PH_NZ + q];
                    const double ph = phv[j * PH_NZ + q];
                    a += PC[i * 15 + k] * ph, gpt += G[i * 15 + k] * ph;
                }
                Cv[i * 15 + j] = a + 0.5 * dt * (PG[i * 15 + j] + gpt);
            }
        }
        __syncwarp();
    }
}

// stateFromData's q.normalize() (preintegration_base.cc:115-125) on state16's q_xyzw, in place
__device__ __forceinline__ void start_q_normalize(double *st) {
    const double qx = st[3], qy = st[4], qz = st[5], qw = st[6], qn = sqrt(qx * qx + qy * qy + qz * qz + qw * qw);
    st[3] = qx / qn, st[4] = qy / qn, st[5] = qz / qn, st[6] = qw / qn;
}

// resetState: iewn_ = Earth::iewn(station, p) at the start position (preintegration_earth.cc:305-324), the Earth form's only
__device__ __forceinline__ void start_iewn(const double *stn, const double *st, double *iw) {
    const bam::V3 v = gc::earth_iewn(stn, bam::mk(st[0], st[1], st[2]));
    iw[0] = v.x, iw[1] = v.y, iw[2] = v.z;
}

__device__ void write_matrices(const double *sm, double *blob, int lane) {
    for (int e = lane; e < 225; e += 32) blob[27 + e] = sm[SM_J + e], blob[252 + e] = sm[SM_C + e];
}

__global__ void __launch_bounds__(PREINT_WARPS * 32) preint_batch_kernel(PreintBatch A) {
    __shared__ double s_m[PREINT_WARPS * SM_WARP];
    __shared__ signed char s_k[15 * PH_NZ], s_nz[16];
    phi_pattern(s_k, s_nz);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, k = blockIdx.x * PREINT_WARPS + warp;
    if (k >= A.n) return;
    double *sm = s_m + warp * SM_WARP;
    double st[16];
#pragma unroll
    for (int i = 0; i < 16; i++) st[i] = A.state16[16 * (size_t) k + i];
    gc::PreintScalar S;
    gc::preint_begin(S, st, A.iewn3, A.gravity3);
    propagate(S, A.noise5, A.imu + 7 * (size_t) A.off[k], A.off[k + 1] - A.off[k], sm, s_k, s_nz, lane);
    double *blob = A.blobs + (size_t) ICG_IMU_BLOB_DOUBLES * k;
    write_matrices(sm, blob, lane);
    if (lane == 0) gc::preint_head(S, st, A.gravity3, blob, A.ends ? A.ends + 10 * (size_t) k : nullptr);
}

__global__ void __launch_bounds__(PREINT_WARPS * 32) preint_resident_kernel(PreintResident A) {
    __shared__ double s_m[PREINT_WARPS * SM_WARP];
    __shared__ signed char s_k[15 * PH_NZ], s_nz[16];
    phi_pattern(s_k, s_nz);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, k = blockIdx.x * PREINT_WARPS + warp;
    if (k >= A.n) return;
    double *sm = s_m + warp * SM_WARP;
    const ReintItem it = A.item[k];
    const size_t node = (size_t) it.win * A.K + it.fac;
    const double *pose = A.pose + 7 * node, *mix = A.mix + 9 * node;
    double *hb = A.blob + (size_t) ICG_IMU_BLOB_DOUBLES * node;
    double nz5[5], st[16], grav[3], iw[3], stn[3];
#pragma unroll
    for (int i = 0; i < 5; i++) nz5[i] = A.noise5[i];
    // doReintegration's gate: |deltaState().bg - state.bg| > 6 gyr_bias_std or |deltaState().ba - state.ba| > 6 acc_bias_std
    const double gx = hb[11] - mix[3], gy = hb[12] - mix[4], gz = hb[13] - mix[5];
    const double ax = hb[14] - mix[6], ay = hb[15] - mix[7], az = hb[16] - mix[8];
    const bool open = sqrt(gx * gx + gy * gy + gz * gz) > 6 * nz5[2] || sqrt(ax * ax + ay * ay + az * az) > 6 * nz5[3];
    if (!open) {
        if (lane == 0) A.status[k] = 0;
        return;
    }
    // stateFromData(statedatalist_[fac]) with q.normalize() (preintegration_base.cc:115-125); the factor's own form and gravity
#pragma unroll
    for (int i = 0; i < 7; i++) st[i] = pose[i];
    start_q_normalize(st);
#pragma unroll
    for (int i = 0; i < 9; i++) st[7 + i] = mix[i];
#pragma unroll
    for (int i = 0; i < 3; i++) grav[i] = hb[17 + i], stn[i] = A.station[i];
    const bool normal = hb[477] != 0.0;
    if (!normal) start_iewn(stn, st, iw);  // at the new start position
    gc::PreintScalar S;
    gc::preint_begin(S, st, normal ? nullptr : iw, grav);
    propagate(S, nz5, A.imu + 7 * (size_t) it.row0, it.nrow, sm, s_k, s_nz, lane);
    // the factor's square-root information from the new covariance (lane 0; written into the handle only when it exists)
    int ok = 0;
    if (lane == 0) ok = gc::imu_sqrt_info(sm + SM_C, A.U + 225 * node, sm + SM_G) ? 1 : 0;
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if (lane == 0) {
        A.status[k] = ok ? 1 : -1;
        double *e = A.ends + 10 * (size_t) k;
        e[0] = S.cur_p.x, e[1] = S.cur_p.y, e[2] = S.cur_p.z, e[3] = S.cur_q.x, e[4] = S.cur_q.y, e[5] = S.cur_q.z, e[6] = S.cur_q.w;
        e[7] = S.cur_v.x, e[8] = S.cur_v.y, e[9] = S.cur_v.z;
    }
    if (!ok) return;
    int pos = 0;
    if (lane == 0) pos = atomicAdd(A.counter, 1);
    pos = __shfl_sync(0xffffffffu, pos, 0);
    double *ob = A.out_blob + (size_t) ICG_IMU_BLOB_DOUBLES * pos;
    write_matrices(sm, ob, lane);
    write_matrices(sm, hb, lane);
    if (lane == 0) {
        A.out_item[pos] = k;
        gc::preint_head(S, st, grav, ob, nullptr);
        gc::preint_head(S, st, grav, hb, nullptr);
    }
}

// One warp per window: the aligned GNSS fixes, then the integrated factors in order, so that an ICG_SLIDE_CHAIN factor starts from the state
// the previous iteration left in st.  Everything goes into the staged value rows; the handle itself is only read.
__global__ void __launch_bounds__(PREINT_WARPS * 32) preint_slide_kernel(PreintSlide A) {
    __shared__ double s_m[PREINT_WARPS * SM_WARP];
    __shared__ signed char s_k[15 * PH_NZ], s_nz[16];
    phi_pattern(s_k, s_nz);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q = blockIdx.x * PREINT_WARPS + warp;
    if (q >= A.n) return;
    double *sm = s_m + warp * SM_WARP;
    const SlideIntWin W = A.win[q];
    const size_t base = (size_t) W.win * A.K;
    // insertNewGnssTimeNode's alignment: blh[c] -= mix[c] * dt / += mix[c] * dt (ic_gvins.cc:836-838, 850-852), with the sign in dt
    for (int e = lane; e < 3 * W.n_align; e += 32) {
        const SlideAlign g = A.align[W.align0 + e / 3];
        const int c = e % 3;
        double *b = A.val + g.blh + c;
        *b = __dadd_rn(*b, __dmul_rn(A.mix[(base + g.node) * 9 + c], g.dt));
    }
    double nz5[5], stn[3], st[16], iw[3];
#pragma unroll
    for (int i = 0; i < 5; i++) nz5[i] = A.noise5[i];
#pragma unroll
    for (int i = 0; i < 3; i++) stn[i] = A.station[i];
#pragma unroll
    for (int i = 0; i < 16; i++) st[i] = 0;
    for (int t = 0; t < W.n_item; t++) {
        const int k = W.item0 + t;
        const SlideItem it = A.item[k];
        if (it.src == ICG_SLIDE_ROW) {
#pragma unroll
            for (int i = 0; i < 16; i++) st[i] = A.state[it.state + i];
        } else {
            // stateFromData (preintegration_base.cc:115-125) of an old node, or of the stateToData(currentState()) st holds (ICG_SLIDE_CHAIN)
            if (it.src >= 0) {
                const double *pose = A.pose + 7 * (base + it.src), *mix = A.mix + 9 * (base + it.src);
#pragma unroll
                for (int i = 0; i < 7; i++) st[i] = pose[i];
#pragma unroll
                for (int i = 0; i < 9; i++) st[7 + i] = mix[i];
            }
            start_q_normalize(st);
        }
        if (!it.normal) start_iewn(stn, st, iw);
        gc::PreintScalar S;
        gc::preint_begin(S, st, it.normal ? nullptr : iw, it.grav);
        propagate(S, nz5, A.imu + 7 * (size_t) it.row0, it.nrow, sm, s_k, s_nz, lane);
        double *blob = A.val + it.blob;
        int ok = 0;
        if (lane == 0) ok = gc::imu_sqrt_info(sm + SM_C, blob + ICG_IMU_BLOB_DOUBLES, sm + SM_G) ? 1 : 0;
        ok = __shfl_sync(0xffffffffu, ok, 0);
        double *ob = A.out_blob ? A.out_blob + (size_t) ICG_IMU_BLOB_DOUBLES * k : nullptr;
        write_matrices(sm, blob, lane);
        if (ob) write_matrices(sm, ob, lane);
        if (lane == 0) {
            A.status[k] = ok ? 1 : -1;
            gc::preint_head(S, st, it.grav, blob, A.ends + 10 * (size_t) k);
            if (ob) gc::preint_head(S, st, it.grav, ob, nullptr);
        }
        // stateToData(currentState()): p, q, v propagated, bg / ba of the start state -- the new node's row and the next CHAIN's start
        st[0] = S.cur_p.x, st[1] = S.cur_p.y, st[2] = S.cur_p.z, st[3] = S.cur_q.x, st[4] = S.cur_q.y, st[5] = S.cur_q.z, st[6] = S.cur_q.w;
        st[7] = S.cur_v.x, st[8] = S.cur_v.y, st[9] = S.cur_v.z;
        if (it.node >= 0 && lane == 0) {
#pragma unroll
            for (int i = 0; i < 16; i++) A.val[it.node + i] = st[i];
        }
        __syncwarp();  // the next factor's propagate rewrites the shared matrices the lanes have just read
    }
}

__global__ void __launch_bounds__(PREINT_WARPS * 32) preint_gins_kernel(PreintGins A) {
    __shared__ double s_m[PREINT_WARPS * SM_WARP];
    __shared__ signed char s_k[15 * PH_NZ], s_nz[16];
    phi_pattern(s_k, s_nz);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, k = blockIdx.x * PREINT_WARPS + warp;
    if (k >= A.n || A.status[k] != 1) return;
    double *sm = s_m + warp * SM_WARP;
    const double *x = A.state17 + 17 * (size_t) k;
    double nz5[5], stn[3], st[16], iw[3], grav[3] = {0, 0, A.gravity[k]};
#pragma unroll
    for (int i = 0; i < 5; i++) nz5[i] = A.noise5[i];
#pragma unroll
    for (int i = 0; i < 3; i++) stn[i] = A.station[i];
#pragma unroll
    for (int i = 0; i < 16; i++) st[i] = x[1 + i];
    start_q_normalize(st);
    const bool normal = A.earth[k] == 0;
    if (!normal) start_iewn(stn, st, iw);
    gc::PreintScalar S;
    gc::preint_begin(S, st, normal ? nullptr : iw, grav);
    propagate(S, nz5, A.imu + 7 * (size_t) A.max_rows * k, A.nrow[k], sm, s_k, s_nz, lane);
    double *blob = A.blob + (size_t) ICG_IMU_BLOB_DOUBLES * k;
    write_matrices(sm, blob, lane);
    if (lane == 0) gc::preint_head(S, st, grav, blob, A.ends + 10 * (size_t) k);
}

}  // namespace

cudaError_t preint_gins_launch(const PreintGins &a, cudaStream_t stream) {
    if (a.n <= 0) return cudaSuccess;
    preint_gins_kernel<<<(a.n + PREINT_WARPS - 1) / PREINT_WARPS, PREINT_WARPS * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t preint_batch_launch(const PreintBatch &a, cudaStream_t stream) {
    if (a.n <= 0) return cudaSuccess;
    preint_batch_kernel<<<(a.n + PREINT_WARPS - 1) / PREINT_WARPS, PREINT_WARPS * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t preint_resident_launch(const PreintResident &a, cudaStream_t stream) {
    if (a.n <= 0) return cudaSuccess;
    preint_resident_kernel<<<(a.n + PREINT_WARPS - 1) / PREINT_WARPS, PREINT_WARPS * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t preint_slide_launch(const PreintSlide &a, cudaStream_t stream) {
    if (a.n <= 0) return cudaSuccess;
    preint_slide_kernel<<<(a.n + PREINT_WARPS - 1) / PREINT_WARPS, PREINT_WARPS * 32, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t preload_preint_resident() {
    cudaFuncAttributes attr;
    cudaError_t e = cudaFuncGetAttributes(&attr, preint_resident_kernel);
    return e == cudaSuccess ? cudaFuncGetAttributes(&attr, preint_slide_kernel) : e;
}

}  // namespace icg
