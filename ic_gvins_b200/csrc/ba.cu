// ba.cu -- Path B: batched sliding-window factor-graph solve on sm_90a.
//
// Replaces `ceres::Solver::Solve` (LEVENBERG_MARQUARDT + DENSE_SCHUR, IG/ic_gvins.cc:1143-1146,1183,1217) and the
// per-factor `CostFunction::Evaluate` calls Ceres drives (IG/factors/*.h, IG/preintegration/*.h) for MANY independent
// windows at once (throughput mode: one window per stream).  Ceres is an un-vendored dependency of the reference; the
// trust-region loop restated here follows its published algorithm and the defaults the reference leaves untouched.
//
// Device-resident LM: the host only enqueues a fixed kernel sequence per iteration; every decision (step validity,
// accept/reject, radius update, convergence) is taken on the device in per-window LM state.
//
// Per window: n = 15K+7 camera-side columns laid out [pose_0..pose_{K-1} (6 each) | extrinsic 6 | td 1 | mix_0..mix_{K-1} (9 each)];
// the vision factors only touch the first NCV = 6K+7 ("vision columns").  Landmarks (inverse depths) are eliminated:
//   lin_vis    : CTA / run of landmarks of one reference node: thread / reprojection factor -> residual, local Jacobians, Huber
//                correction -> record in shared memory; per (reference node, observing node) pair the 20x20 Gram matrix of the run's
//                records on the FP64 tensor cores (DMMA.8x8x4), summed over the node's runs in run order;
//                lanes / landmark -> h_l, g_l and the dense coupling row w_l (A_W, landmark-major)
//   schur_dmma : cluster of 4 CTAs / window: sum_l phi_l w_l w_l^T with phi_l = s_l^2 / (s_l^2 h_l + D_l^2) on the FP64 tensor cores, one
//                landmark split per CTA, the partials summed over DSMEM; epilogue: one-writer-per-entry gather of the pair Gram matrices
//                into the vision part of H_cc and g_c -> Hs = H_c + H_vis - Schur term and the solve's vision vectors (or the split
//                pipeline's export payload)
//   lin_cam    : one CTA / window (second stream, beside the vision chain) -> IMU preintegration, GNSS, bias, prior and
//                marginalization factors -> H_c, g_c
//   solve      : one CTA / window -> Jacobi scaling, LM diagonal, S = s(H - Schur)s + D^2, packed Cholesky in shared memory
//                (panel updates on DMMA), triangular solves, landmark back-substitution, model cost change, candidate x (+) delta
//   single GPU : lin_vis + lin_cam at the candidate, into the window's second linearisation buffer (its costs are the candidate cost)
//   cost       : candidate cost (all factors, residuals only) of the split pipeline;   accept : Ceres step acceptance + radius update
//   ba_lm.cuh  : that trust-region policy (LM diagonal, termination, iteration commit, step decision), shared with ba_split.cuh
//   ba_marg.cuh: sliding-window marginalization (MarginalizationInfo) on the same device-resident linearisation
// Kernels only: the host side is ba_handle.cu (lifecycle, the solve) and ba_keyframe.cu (the resident keyframe cycle), through ba_dev.cuh.
#include <cooperative_groups.h>
#include <math.h>
#include <string.h>

#include "ba_dev.cuh"
#include "geom_core.cuh"

namespace icg {
using namespace bam;
namespace cg = cooperative_groups;

constexpr int BA_CHOL_NB = 8;   // Cholesky block width

// window w's part of linearisation buffer b
__device__ __forceinline__ double *lin_Mp(const BaCaps &C, const BaDev &D, int b, int w) { return D.Mp[b] + (size_t) w * C.K * (C.K - 1) * 210; }
__device__ __forceinline__ double *lin_AW(const BaCaps &C, const BaDev &D, int b, int w) { return D.AW[b] + (size_t) w * C.LP * C.NCA; }
__device__ __forceinline__ double *lin_costf(const BaCaps &C, const BaDev &D, int b, int w) { return D.costf[b] + (size_t) w * C.F; }
__device__ __forceinline__ double *lin_hl(const BaCaps &C, const BaDev &D, int b, int w) { return D.hl[b] + (size_t) w * C.L; }
__device__ __forceinline__ double *lin_gl(const BaCaps &C, const BaDev &D, int b, int w) { return D.gl[b] + (size_t) w * C.L; }
__device__ __forceinline__ double *lin_Hc(const BaCaps &C, const BaDev &D, int b, int w) { return D.Hc[b] + (size_t) w * C.NS * C.NS; }
__device__ __forceinline__ double *lin_gc(const BaCaps &C, const BaDev &D, int b, int w) { return D.gc[b] + (size_t) w * C.NS; }

__device__ __forceinline__ int col_pose(int k) { return 6 * k; }
__device__ __forceinline__ int col_ext(int K) { return 6 * K; }
__device__ __forceinline__ int col_td(int K) { return 6 * K + 6; }
__device__ __forceinline__ int col_mix(int K, int k) { return 6 * K + 7 + 9 * k; }

__device__ __forceinline__ double block_sum(double v, double *s_red);
__device__ __forceinline__ double block_max(double v, double *s_red);
}  // namespace icg
#include "ba_lm.cuh"  // the trust-region policy (over the column layout and block_sum above)
namespace icg {

// ------------------------------------------------------------------------------------------------ lin_vis (+ landmark rows)
__device__ __forceinline__ int jc_off(int a) { return a < 18 ? (a / 6) * 12 + (a % 6) : 36 + 2 * (a - 18); }  // row 0 offset in a record
__device__ __forceinline__ int jc_row1(int a) { return a < 18 ? 6 : 1; }                                           // + this for row 1
__device__ __forceinline__ int tri20(int la, int lb) {  // index of (la <= lb) in the packed upper 20x20
    return la * 20 - la * (la - 1) / 2 + (lb - la);
}
__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// One CTA linearises a run of WHOLE landmarks of ONE reference node (<= 128 reprojection factors; the host packs the runs at upload).
//  phase 1: thread / factor, in record slot order -> residual, local Jacobians, Huber correction -> 40-double record
//           [Ji 12 | Jj 12 | Je 12 | Jt 2 | r 2] + [j_rho 2 | observing node | reference node], staged in shared memory;
//  phase 2: the Gram matrices of the run.  Within a (reference node, observing node) pair every factor has the same 19 camera-side columns
//           [ref pose 6 | obs pose 6 | extrinsic 6 | td 1] (+ the residual as a 20th column), so the pair's contribution is the dense
//           20x20 Gram matrix X^T X of its stacked 2x20 rows: one warp per observing node of the run, 4 rows (2 factors) per DMMA.8x8x4
//           k-step.  With the m8n8k4 fragment layout (A: lane -> (row lane/4, k lane%4); B: lane -> (k lane%4, col lane/4)) the A and
//           B operands of X^T X are the SAME register: lane loads X[k = lane%4][8 t + lane/4] for the three column tiles t and issues
//           the six upper-triangular tile products.  The packed result is the run's partial of that pair (D.gpart);
//  phase 3: eight lanes per landmark reduce its records, straight from shared memory, to h_l, g_l and the coupling row
//           w_l[c] = sum_f J_f[:, c]^T j_rho,f of A_W (landmark-major [l][NCA]: zeroed, then the <= 13 + 6 n_obs non-zeros).  All
//           factors of a landmark share the reference node, the extrinsic and td (accumulated); each observing node appears once
//           (written directly; icg_ba_upload checks it);
//  phase 4: the last run of the reference node to arrive (arrival counter) sums the node's partials of every pair in run order -> Mp.
//           No floating-point atomics: the result does not depend on which CTA arrives last, nor on the other windows of the batch.
// The Jacobians never leave the SM: per factor only the cost is stored.
// at_cand = 0: at x (windows that need a linearisation) into buffer lin_buf; at_cand = 1: at the candidate of a valid step into buffer
// 1 - lin_buf (its per-factor costs are the candidate cost ba_accept tests).
__global__ void __launch_bounds__(128, 4) ba_lin_vis(BaCaps C, BaDev D, int at_cand) {
    extern __shared__ double lv_sm[];
    __shared__ int s_ord[128], s_gbeg[BA_MAX_NODES], s_gend[BA_MAX_NODES], s_last, s_p0, s_np;
    double (*s_rec)[LV_LD] = (double (*)[LV_LD]) lv_sm;
    double (*s_frame)[NODE_FRAME_LD] = (double (*)[NODE_FRAME_LD]) (lv_sm + 128 * LV_LD);
    const int w = blockIdx.y;
    const LmState &st = D.st[w];
    if (st.done || !(at_cand ? st.step_valid : st.need_lin)) return;
    const int b = at_cand ? 1 - st.lin_buf : st.lin_buf;
    const double *pose = at_cand ? D.pose_c : D.pose, *xext = at_cand ? D.ext_c : D.ext, *rho = at_cand ? D.rho_c : D.rho;
    const int *vb = D.vb_lm0 + (size_t) w * C.NVB;
    if ((int) blockIdx.x >= vb[C.NVB - 1]) return;  // last entry = number of runs of this window
    const WinDims dm = D.dims[w];
    const int tid = threadIdx.x;
    const int *off = D.lm_off + (size_t) w * (C.L + 1);
    const int pA = vb[blockIdx.x], pB = vb[blockIdx.x + 1];  // landmark positions of the run
    const int s0 = off[pA], nslot = off[pB] - s0;
    // ---- phase 0: the window's K + 1 node frames (rotation matrix | position of every pose and of the extrinsic), once per CTA
    if (tid <= dm.K) node_frame(tid < dm.K ? pose + ((size_t) w * C.K + tid) * 7 : xext + (size_t) w * 8, s_frame[tid]);
    if (tid < BA_MAX_NODES) s_gbeg[tid] = s_gend[tid] = 0;
    if (tid == 0) s_np = 0;
    __syncthreads();
    // ---- phase 1
    if (tid < nslot) {
        const int q = s0 + tid;
        double r[2], Ji[12], Jj[12], Je[12], Jr[2], Jt[2], cost = 0;
        const int4 meta = ((const int4 *) D.f_meta_s)[(size_t) w * C.F + q];  // (landmark, reference node, observing node, factor id)
        const int i = meta.y, j = meta.z, f = meta.w;
        if (D.f_active[(size_t) w * C.F + f] != 0) {
            const double *ext = xext + (size_t) w * 8;
            reproj_eval_frames(s_frame[i], s_frame[j], s_frame[dm.K], rho[(size_t) w * C.L + meta.x], ext[7],
                               D.f_const_s + ((size_t) w * C.F + q) * 14, dm.reproj_sinv, true, r, Ji, Jj, Je, Jr, Jt);
            if (dm.ext_const)
                for (int k = 0; k < 12; k++) Je[k] = 0;
            if (dm.td_const) Jt[0] = Jt[1] = 0;
            double sq = r[0] * r[0] + r[1] * r[1], sc = 1.0;
            if (dm.reproj_huber)
                huber(sq, cost, sc);
            else
                cost = 0.5 * sq;
            if (sc != 1.0) {
                for (int k = 0; k < 12; k++) Ji[k] *= sc, Jj[k] *= sc, Je[k] *= sc;
                Jr[0] *= sc, Jr[1] *= sc, Jt[0] *= sc, Jt[1] *= sc, r[0] *= sc, r[1] *= sc;
            }
        } else {
            for (int k = 0; k < 12; k++) Ji[k] = Jj[k] = Je[k] = 0;
            Jr[0] = Jr[1] = Jt[0] = Jt[1] = r[0] = r[1] = 0;
        }
        lin_costf(C, D, b, w)[f] = cost;
        double *sr = s_rec[tid];
#pragma unroll
        for (int k = 0; k < 12; k++) sr[k] = Ji[k], sr[12 + k] = Jj[k], sr[24 + k] = Je[k];
        sr[36] = Jt[0], sr[37] = Jt[1], sr[38] = r[0], sr[39] = r[1];
        sr[40] = Jr[0], sr[41] = Jr[1], sr[42] = (double) j, sr[43] = (double) i;
    }
    __syncthreads();
    // ---- phase 2
    const int lane = tid & 31, warp = tid >> 5;
    if (nslot > 0) {
        if (tid < nslot) {  // slots [s_gbeg[o], s_gend[o]) of s_ord observe from node o
            const int *ord = D.vis_ord + (size_t) w * C.F + s0;
            const int v = ord[tid], ob = (int) s_rec[v & 255][42];
            s_ord[tid] = v;
            if (tid == 0 || (int) s_rec[ord[tid - 1] & 255][42] != ob) s_gbeg[ob] = tid;
            if (tid == nslot - 1 || (int) s_rec[ord[tid + 1] & 255][42] != ob) s_gend[ob] = tid + 1;
        }
        __syncthreads();
        const int kk = lane & 3, g = lane >> 2;  // k index inside the step (factor kk/2, residual row kk%2), column inside the tile
        int o[3];
#pragma unroll
        for (int t = 0; t < 3; t++) {
            const int a = 8 * t + g;
            o[t] = a < 20 ? jc_off(a) + (kk & 1) * jc_row1(a) : -1;
        }
        for (int ob = warp; ob < dm.K; ob += 4) {
            const int beg = s_gbeg[ob], end = s_gend[ob];
            if (beg == end) continue;
            double c00[2] = {0, 0}, c01[2] = {0, 0}, c02[2] = {0, 0}, c11[2] = {0, 0}, c12[2] = {0, 0}, c22[2] = {0, 0};
            constexpr int UNR = 2;  // k-steps in flight (4 factors)
            for (int base = beg; base < end; base += 2 * UNR) {
                double x[UNR][3];
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const int q = base + 2 * u + (kk >> 1);
                    const bool ok = q < end;
                    const double *rec = s_rec[ok ? s_ord[q] & 255 : 0];
#pragma unroll
                    for (int t = 0; t < 3; t++) x[u][t] = (ok && o[t] >= 0) ? rec[o[t]] : 0.0;
                }
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    dmma884(c00[0], c00[1], x[u][0], x[u][0]);
                    dmma884(c01[0], c01[1], x[u][0], x[u][1]);
                    dmma884(c02[0], c02[1], x[u][0], x[u][2]);
                    dmma884(c11[0], c11[1], x[u][1], x[u][1]);
                    dmma884(c12[0], c12[1], x[u][1], x[u][2]);
                    dmma884(c22[0], c22[1], x[u][2], x[u][2]);
                }
            }
            // C fragment: lane holds (row lane/4, cols 2 (lane%4) + {0,1}) of each 8x8 tile
            double *pp = D.gpart + ((size_t) w * C.GQ + (s_ord[beg] >> 8)) * 210;
            auto put = [&](int ti, int tj, const double *c) {
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int la = 8 * ti + g, lb = 8 * tj + 2 * kk + e;
                    if (la <= lb && lb < 20) pp[tri20(la, lb)] = c[e];
                }
            };
            put(0, 0, c00), put(0, 1, c01), put(0, 2, c02), put(1, 1, c11), put(1, 2, c12), put(2, 2, c22);
        }
        __threadfence();  // the partials are visible device-wide before this run is counted (phase 4)
    }
    // ---- phase 3
    const int *perm = D.lm_perm + (size_t) w * C.L;
    const int K = dm.K, NCV = 6 * K + 7, NCA = 4 * ((NCV + 1 + 3) / 4);
    const int grp = tid >> 3, sl = tid & 7;
    int o0[3], o1[3];
#pragma unroll
    for (int t = 0; t < 3; t++) {
        const int c = sl + 8 * t;  // 0..23; 19 -> residual pair (g_l); 20 -> h_l from j_rho; > 20 unused
        o0[t] = c < 19 ? jc_off(c) : 38, o1[t] = c < 19 ? o0[t] + jc_row1(c) : 39;
    }
    for (int pl = pA + grp; pl < pB; pl += 16) {
        const int l = perm[pl], f0 = off[pl] - s0, nf = off[pl + 1] - off[pl];
        double *row = lin_AW(C, D, b, w) + (size_t) l * C.NCA;
        for (int c = sl; c < NCA; c += 8) row[c] = 0.0;
        __syncwarp(0xffu << (tid & 24));  // the landmark's eight lanes: zeros land before the values
        double acc[3] = {0, 0, 0};
        for (int q = 0; q < nf; q++) {
            const double *rec = s_rec[f0 + q];
            const double r0 = rec[40], r1 = rec[41];
            const int ob = (int) rec[42];
#pragma unroll
            for (int t = 0; t < 3; t++) {
                const int c = sl + 8 * t;
                if (c == 20) {
                    acc[t] += r0 * r0 + r1 * r1;
                } else if (c < 20) {
                    const double v = rec[o0[t]] * r0 + rec[o1[t]] * r1;
                    if (c >= 6 && c < 12)
                        row[col_pose(ob) + c - 6] = v;
                    else
                        acc[t] += v;
                }
            }
        }
        const int ref = nf > 0 ? (int) s_rec[f0][43] : 0;
#pragma unroll
        for (int t = 0; t < 3; t++) {
            const int c = sl + 8 * t;
            if (nf > 0) {
                if (c < 6) row[col_pose(ref) + c] = acc[t];
                else if (c >= 12 && c < 18) row[col_ext(K) + c - 12] = acc[t];
                else if (c == 18) row[col_td(K)] = acc[t];
            }
            if (c == 19) {
                row[NCV] = acc[t];
                lin_gl(C, D, b, w)[l] = acc[t];
            } else if (c == 20) {
                lin_hl(C, D, b, w)[l] = acc[t];
                if (st.first) D.scale_l[(size_t) w * C.L + l] = 1.0 / (1.0 + sqrt(acc[t]));  // jacobi_scaling, once (iteration 0)
            }
        }
    }
    // ---- phase 4
    if (nslot == 0) return;  // a run of landmarks without factors: no pair
    const int rn = (int) s_rec[0][43];
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(D.vis_cnt + (size_t) w * C.K + rn, 1) == D.ref_nrun[(size_t) w * C.K + rn] - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) D.vis_cnt[(size_t) w * C.K + rn] = 0;
    const int PM = C.K * (C.K - 1), P = D.npairs[w];
    const int *pro = D.pair_ro + (size_t) w * PM, *poff = D.part_off + (size_t) w * (PM + 1);
    for (int p = tid; p < P; p += 128)  // the node's pairs are consecutive (pairs are ordered by reference node)
        if ((pro[p] >> 8) == rn) {
            atomicAdd(&s_np, 1);
            if (p == 0 || (pro[p - 1] >> 8) != rn) s_p0 = p;
        }
    __syncthreads();
    const double *part = D.gpart + (size_t) w * C.GQ * 210;
    double *Mp = lin_Mp(C, D, b, w);
    for (int p = s_p0 + warp; p < s_p0 + s_np; p += 4) {  // warp / pair: the 7 entries of a lane in flight together
        const int k0 = poff[p], k1 = poff[p + 1];
        double acc[7];
#pragma unroll
        for (int j = 0; j < 7; j++) acc[j] = lane + 32 * j < 210 ? __ldcg(part + (size_t) k0 * 210 + lane + 32 * j) : 0.0;
        for (int k = k0 + 1; k < k1; k++) {
            double v[7];
#pragma unroll
            for (int j = 0; j < 7; j++) v[j] = lane + 32 * j < 210 ? __ldcg(part + (size_t) k * 210 + lane + 32 * j) : 0.0;
#pragma unroll
            for (int j = 0; j < 7; j++) acc[j] += v[j];
        }
#pragma unroll
        for (int j = 0; j < 7; j++)
            if (lane + 32 * j < 210) Mp[(size_t) p * 210 + lane + 32 * j] = acc[j];
    }
}

// ------------------------------------------------------------------------------------------------ pair_gram: vision part of H_cc, g_c
// ba_lin_vis leaves one packed 20x20 Gram matrix per (reference node, observing node) pair in Mp; the epilogue of ba_schur_dmma gathers
// them (thread / output entry) into the symmetric (NCV+1)^2 matrix [H_vis g_vis; g_vis^T r^T r].  No atomics: every output has one writer.

// gather of one entry (A <= B) of the symmetric (NCV+1)^2 matrix [H_vis g_vis; g_vis^T r^T r] from the per-pair Gram matrices: the groups
// that touch both of its blocks
__device__ __forceinline__ void gram2_slots(const BaCaps &C, const BaDev &D, int w, int K, short *s_slot) {
    const int PM = C.K * (C.K - 1), P = D.npairs[w];
    const int *pro = D.pair_ro + (size_t) w * PM;
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) s_slot[e] = -1;
    __syncthreads();
    for (int p = threadIdx.x; p < P; p += blockDim.x) s_slot[(pro[p] >> 8) * K + (pro[p] & 255)] = (short) p;
    __syncthreads();
}
__device__ __forceinline__ double gram2_entry(const BaCaps &C, const BaDev &D, int buf, int w, int K, const short *s_slot, int A, int B) {
    const int P = D.npairs[w];
    const double *Mp = lin_Mp(C, D, buf, w);
    const int bA = A < 6 * K ? A / 6 : K, bB = B < 6 * K ? B / 6 : K;
    const int a = A - 6 * bA, b = B - 6 * bB;  // offsets inside the block (global block: 0..7 = ext 6, td, residual)
    const int ga = 12 + a, gb = 12 + b;          // local column of a global-block column
    double sum = 0;
    if (bA == K) {  // (global, global): every group
        // up to K (K - 1) groups: sixteen loads in flight and four partial sums in a fixed order, group p into sum p mod 4 (these 36 entries
        // are the tail of the epilogue: a serial sum is 90 dependent L2 round trips)
        const int idx = tri20(ga, gb);
        double s4[4] = {0, 0, 0, 0};
        int p = 0;
        for (; p + 16 <= P; p += 16) {
            double v[16];
#pragma unroll
            for (int u = 0; u < 16; u++) v[u] = Mp[(size_t) (p + u) * 210 + idx];
#pragma unroll
            for (int u = 0; u < 16; u++) s4[u & 3] += v[u];
        }
        for (; p < P; p++) s4[p & 3] += Mp[(size_t) p * 210 + idx];
        sum = (s4[0] + s4[1]) + (s4[2] + s4[3]);
    } else if (bB == K || bB == bA) {  // (pose, global) or the pose's diagonal block
        const int i1 = tri20(a, bB == K ? gb : b), i2 = tri20(6 + a, bB == K ? gb : 6 + b);
        // 16 loads in flight; same summation order as a serial loop (a missing pair or o >= K adds +0.0, which leaves a sum that started
        // at +0.0 unchanged)
        for (int o0 = 0; o0 < K; o0 += 8) {
            double v1[8], v2[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int o = o0 + u;
                const int p1 = o < K ? s_slot[bA * K + o] : -1, p2 = o < K ? s_slot[o * K + bA] : -1;  // bA as reference node / as observing node
                v1[u] = p1 >= 0 ? Mp[(size_t) p1 * 210 + i1] : 0.0;
                v2[u] = p2 >= 0 ? Mp[(size_t) p2 * 210 + i2] : 0.0;
            }
#pragma unroll
            for (int u = 0; u < 8; u++) sum += v1[u], sum += v2[u];
        }
    } else {  // two different poses: the (bA -> bB) and (bB -> bA) groups
        const int p1 = s_slot[bA * K + bB], p2 = s_slot[bB * K + bA];
        if (p1 >= 0) sum += Mp[(size_t) p1 * 210 + tri20(a, 6 + b)];
        if (p2 >= 0) sum += Mp[(size_t) p2 * 210 + tri20(b, 6 + a)];
    }
    return sum;
}

// ------------------------------------------------------------------------------------------------ Schur term + reduced camera system
__device__ __forceinline__ double *x_inbox(const BaDev &D, int peer, int w, int from);  // ba_split.cuh
__device__ __forceinline__ int tri_idx(int A, int B, int ncv);

// Entry (A <= B <= NCV) of the vision Gram matrix (cj, gathered here from Mp) and of the Schur term (cw): stores what the solve of the
// pipeline that drives the handle reads.
//   single GPU (fused pipeline): Hs = H_c + (cj - cw) on the vision rows (lower triangle) and D.visv = [diag H_vis | g_vis | W phi g_l];
//   split pipeline: [tri(H_vis - Schur) | diag H_vis | g_vis | W phi g_l] straight into the owner's inbox (P2P stores; ba_signal publishes
//                   them, the owner's ba_reduce sums the ranks).
__device__ __forceinline__ void schur_store(const BaCaps &C, const BaDev &D, int buf, int w, int K, const short *s_slot, int A, int B, double cw) {
    const int NCV = 6 * K + 7;
    if (A == NCV) return;  // the r^T r corner: no solve reads it
    const size_t e = (size_t) w * C.NS * C.NS + (size_t) B * C.NS + A;
    const double hc = !D.S.split && B < NCV ? lin_Hc(C, D, buf, w)[(size_t) B * C.NS + A] : 0.0;  // in flight during the gather
    const double cj = gram2_entry(C, D, buf, w, K, s_slot, A, B);
    if (D.S.split) {
        double *P = x_inbox(D, w % D.world, w, D.rank);
        const int TRI = NCV * (NCV + 1) / 2;
        if (B < NCV) {
            P[tri_idx(A, B, NCV)] = cj - cw;
            if (A == B) P[TRI + A] = cj;
        } else {
            P[TRI + NCV + A] = cj;       // g_vis
            P[TRI + 2 * NCV + A] = cw;   // W phi g_l
        }
    } else {
        double *V = D.visv + (size_t) w * 3 * C.NCV;
        if (B < NCV) {
            D.Hs[e] = hc + (cj - cw);
            if (A == B) V[A] = cj;
        } else {
            V[NCV + A] = cj, V[2 * NCV + A] = cw;
        }
    }
}

// the scalars of the split payload: vision cost, sum rho^2 and max |g_l| over this rank's factors and landmarks (one CTA)
__device__ __forceinline__ void schur_scalars(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, double *s_red) {
    const int tid = threadIdx.x;
    double c = 0, q = 0, gm = 0;
    const double *costf = lin_costf(C, D, 0, w), *gl = lin_gl(C, D, 0, w);  // the split pipeline uses buffer 0 only
    for (int f = tid; f < dm.F; f += 256) c += costf[f];
    for (int l = tid; l < dm.L; l += 256) {
        const double r = D.rho[(size_t) w * C.L + l];
        q += r * r;
        gm = fmax(gm, fabs(gl[l]));
    }
    c = block_sum(c, s_red);
    q = block_sum(q, s_red);
    gm = block_max(gm, s_red);
    if (tid != 0) return;
    const int NCV = 6 * dm.K + 7, TRI = NCV * (NCV + 1) / 2;
    double *P = x_inbox(D, w % D.world, w, D.rank);
    P[TRI + 3 * NCV] = c, P[TRI + 3 * NCV + 1] = q, P[TRI + 3 * NCV + 2] = gm;
}

// Schur SYRK on the FP64 tensor cores: the sum over the window's landmarks of phi_l w_l w_l^T, with
// phi_l = s_l^2 / (s_l^2 h_l + clamp(s_l^2 h_l) / radius) the LM-damped landmark pivot.  DMMA.8x8x4 with k = 4 landmarks per step; as in
// ba_lin_vis's Gram phase the A and B fragments of X^T X share one layout: lane reads A_W[l0 + lane%4][8 t + lane/4].  The CTA stages its
// landmark rows (and phi) in shared memory once per pass -- leading dimension = 8 mod 16 doubles, so a fragment read is the minimal
// two wavefronts -- and every warp accumulates two 16x16 super-tiles (2x2 DMMA tiles each) of the upper triangle per pass.
// One thread-block CLUSTER of BA_SPLIT_W CTAs per window: CTA k accumulates the partial of landmark split k.  After each pass (16
// super-tiles) every CTA puts its partials in shared memory over its staging rows, which the pass no longer needs; after a cluster barrier
// each CTA owns a quarter of the pass's super-tiles, sums the BA_SPLIT_W partials of an entry over DSMEM in split order starting from 0.0
// (deterministic) and hands the entry to schur_store.  The partials never leave the cluster.
__global__ void __cluster_dims__(BA_SPLIT_W, 1, 1) __launch_bounds__(256) ba_schur_dmma(BaCaps C, BaDev D, int ld) {
    extern __shared__ double sA[];  // [SCHUR_RCH][ld] rows, then phi[SCHUR_RCH]; between passes: [SCHUR_PASS][256] partials
    __shared__ short s_slot[32 * 32];
    __shared__ double s_red[40];
    cg::cluster_group cluster = cg::this_cluster();
    const int w = blockIdx.y, split = blockIdx.x;  // cluster rank = split
    const LmState &st = D.st[w];
    if (st.done) return;  // per window: the whole cluster leaves
    const WinDims dm = D.dims[w];
    const int NCV = 6 * dm.K + 7, NCA = 4 * ((NCV + 1 + 3) / 4);
    const int T2 = (NCA + 15) / 16, nsuper = T2 * (T2 + 1) / 2;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, kk = lane & 3;
    double *sphi = sA + (size_t) SCHUR_RCH * ld;
    const int b = st.lin_buf;
    const double *A = lin_AW(C, D, b, w), *hl = lin_hl(C, D, b, w);
    const double radius = st.radius;
    const int nsteps = (dm.L + 3) / 4;
    const int r_beg = 4 * (int) ((long long) nsteps * split / BA_SPLIT_W), r_end = min(dm.L, 4 * (int) ((long long) nsteps * (split + 1) / BA_SPLIT_W));
    const int npass = (nsuper + SCHUR_PASS - 1) / SCHUR_PASS;
    gram2_slots(C, D, w, dm.K, s_slot);
    for (int pass = 0; pass < npass; pass++) {
        if (pass > 0) cluster.barrier_wait();  // the peers have read this CTA's partials of the previous pass: its staging rows are free
        int si[2], sj[2];
        bool on[2];
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
            const int su = (2 * pass + h2) * 8 + warp;
            on[h2] = su < nsuper;
            int a = 0, e = on[h2] ? su : 0;
            while (e >= T2 - a) e -= T2 - a, a++;
            si[h2] = a, sj[h2] = a + e;
        }
        double acc[2][4][2];
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++)
#pragma unroll
            for (int q = 0; q < 4; q++) acc[h2][q][0] = acc[h2][q][1] = 0;
        for (int r0 = r_beg; r0 < r_end; r0 += SCHUR_RCH) {
            const int nr = min(SCHUR_RCH, r_end - r0), nr4 = (nr + 3) & ~3;
            __syncthreads();
            for (int rb = warp; rb < nr4; rb += 8 * 4) {  // warp stages rows rb, rb + 8, rb + 16, rb + 24: 4 rows x 3 column chunks in flight
                double v[4][3];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int rr = rb + 8 * u;
#pragma unroll
                    for (int cchunk = 0; cchunk < 3; cchunk++) {
                        const int c = lane + 32 * cchunk;
                        v[u][cchunk] = (rr < nr && c < NCA) ? A[(size_t) (r0 + rr) * C.NCA + c] : 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int rr = rb + 8 * u;
#pragma unroll
                    for (int cchunk = 0; cchunk < 3; cchunk++) {
                        const int c = lane + 32 * cchunk;
                        if (rr < nr4 && c < ld) sA[(size_t) rr * ld + c] = v[u][cchunk];
                    }
                }
                for (int c = lane + 96; c < ld; c += 32)  // wider rows (K > 12): remaining columns
                    for (int u = 0; u < 4; u++) {
                        const int rr = rb + 8 * u;
                        if (rr < nr4) sA[(size_t) rr * ld + c] = (rr < nr && c < NCA) ? A[(size_t) (r0 + rr) * C.NCA + c] : 0.0;
                    }
            }
            for (int rr = tid; rr < nr4; rr += 256) {
                double ph = 0;
                if (rr < nr) {
                    const int l = r0 + rr;
                    const double sl = D.scale_l[(size_t) w * C.L + l], hs = sl * sl * hl[l];
                    ph = sl * sl / (hs + lm_d2(hs, radius));
                }
                sphi[rr] = ph;
            }
            __syncthreads();
            for (int ks = 0; ks < nr4 / 4; ks++) {
                const double *row = sA + (size_t) (4 * ks + kk) * ld;
                const double ph = sphi[4 * ks + kk];
#pragma unroll
                for (int h2 = 0; h2 < 2; h2++) {
                    if (!on[h2]) continue;
                    const double xb0 = row[16 * sj[h2] + g], xb1 = row[16 * sj[h2] + 8 + g];
                    const double a0 = row[16 * si[h2] + g] * ph, a1 = row[16 * si[h2] + 8 + g] * ph;
                    dmma884(acc[h2][0][0], acc[h2][0][1], a0, xb0);
                    dmma884(acc[h2][1][0], acc[h2][1][1], a0, xb1);
                    dmma884(acc[h2][2][0], acc[h2][2][1], a1, xb0);
                    dmma884(acc[h2][3][0], acc[h2][3][1], a1, xb1);
                }
            }
        }
        __syncthreads();  // every warp is done with the staged rows
        // super-tile (2 pass + h2) * 8 + warp -> slot h2 * 8 + warp, in C-fragment order: position 64 q + 32 e + lane holds (row g, col
        // 2 kk + e) of DMMA tile q (conflict-free stores, and reads below)
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
            if (!on[h2]) continue;
#pragma unroll
            for (int q = 0; q < 4; q++)
#pragma unroll
                for (int e = 0; e < 2; e++) sA[(h2 * 8 + warp) * 256 + 64 * q + 32 * e + lane] = acc[h2][q][e];
        }
        cluster.sync();  // every split's partials of this pass are in place
        // CTA `split` owns slots split, split + 4, ...; thread tid owns position tid of each
        const int nslot = min(SCHUR_PASS, nsuper - SCHUR_PASS * pass);
        double cw[SCHUR_PASS / BA_SPLIT_W];
#pragma unroll
        for (int j = 0; j < SCHUR_PASS / BA_SPLIT_W; j++) {
            const int sl = split + BA_SPLIT_W * j;
            double p[BA_SPLIT_W];
#pragma unroll
            for (int k = 0; k < BA_SPLIT_W; k++) p[k] = sl < nslot ? cluster.map_shared_rank(sA, k)[sl * 256 + tid] : 0.0;
            cw[j] = 0;
#pragma unroll
            for (int k = 0; k < BA_SPLIT_W; k++) cw[j] += p[k];
        }
        cluster.barrier_arrive();  // done reading the peers (the matching wait comes before this CTA's shared memory is reused or released)
        const int q = tid >> 6, r_in = 8 * (q >> 1) + ((tid & 31) >> 2), c_in = 8 * (q & 1) + 2 * (tid & 3) + ((tid >> 5) & 1);
#pragma unroll
        for (int j = 0; j < SCHUR_PASS / BA_SPLIT_W; j++) {
            const int sl = split + BA_SPLIT_W * j;
            if (sl >= nslot) break;
            int a = 0, e = SCHUR_PASS * pass + sl;
            while (e >= T2 - a) e -= T2 - a, a++;
            const int r = 16 * a + r_in, cc = 16 * (a + e) + c_in;
            if (r <= cc && cc <= NCV) schur_store(C, D, b, w, dm.K, s_slot, r, cc, cw[j]);
        }
    }
    if (split == 0 && D.S.split) schur_scalars(C, D, w, dm, s_red);
    cluster.barrier_wait();  // no CTA leaves while a peer may still read its shared memory
}

// ------------------------------------------------------------------------------------------------ camera-only factors
constexpr double IMU_GB_STD = 7200 / 3600.0 * 3.14159265358979323846 / 180.0;  // IG/preintegration/imu_error_factor.h:89-91
constexpr double IMU_AB_STD = 2.0e4 * 1.0e-5;

// one warp evaluates one IMU factor: whitened residual rw[15] and (optionally) whitened local Jacobian Jw[15x30] in shared memory
__device__ void imu_factor_warp(const double *blob, const double *U, const double *pose0, const double *mix0, const double *pose1,
                                const double *mix1, bool want_j, double *rw, double *Jw, int lane) {
    __shared__ ImuMid s_mid[16];
    double *raw_r = rw + 15;  // scratch behind rw (caller provides 30 doubles)
    const int wslot = (threadIdx.x >> 5) & 15;
    if (want_j)
        for (int e = lane; e < 450; e += 32) Jw[e] = 0;
    __syncwarp();
    if (lane == 0) {
        ImuMid M;
        imu_residual_raw(blob, pose0, mix0, pose1, mix1, raw_r, M);
        if (want_j) imu_jacobian_raw(blob, M, Jw);
        s_mid[wslot] = M;
    }
    __syncwarp();
    // whitening by the upper-triangular sqrt information: out[i] = sum_{k >= i} U[i][k] in[k]  (in place, rows ascending)
    if (want_j && lane < 30) {
        for (int i = 0; i < 15; i++) {
            double s = 0;
            for (int k = i; k < 15; k++) s += U[i * 15 + k] * Jw[k * 30 + lane];
            Jw[i * 30 + lane] = s;
        }
    }
    if (lane < 15) {
        double s = 0;
        for (int k = lane; k < 15; k++) s += U[lane * 15 + k] * raw_r[k];
        rw[lane] = s;
    }
    __syncwarp();
}

// marginalization prior (IG/factors/marginalization_factor.h:47-101): dx of every remained block
__device__ void marg_dx(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, const double *pose, const double *mix, const double *ext, double *dx,
                        int *colmap, int tid, int nthreads) {
    const int *type = D.marg_type + (size_t) w * BA_MARG_MAXB, *node = D.marg_node + (size_t) w * BA_MARG_MAXB;
    const double *x0 = D.marg_x0 + (size_t) w * BA_MARG_MAXB * 9;
    if (tid == 0) {
        int col = 0, xo = 0;
        for (int b = 0; b < dm.marg_nb; b++) {
            int t = type[b], nd = node[b];
            if (t == 0 || t == 2) {
                const double *x = t == 0 ? pose + nd * 7 : ext;
                const double *xl = x0 + xo;
                Q dq = qmul(qinv(pose_q(xl)), pose_q(x));
                V3 a = 2.0 * qv(dq);
                if (dq.w < 0) a = -a;
                for (int k = 0; k < 3; k++) dx[col + k] = x[k] - xl[k];
                dx[col + 3] = a.x, dx[col + 4] = a.y, dx[col + 5] = a.z;
                int base = t == 0 ? col_pose(nd) : col_ext(dm.K);
                for (int k = 0; k < 6; k++) colmap[col + k] = (t == 2 && dm.ext_const) ? -1 : base + k;
                col += 6, xo += 7;
            } else if (t == 1) {
                for (int k = 0; k < 9; k++) dx[col + k] = mix[nd * 9 + k] - x0[xo + k], colmap[col + k] = col_mix(dm.K, nd) + k;
                col += 9, xo += 9;
            } else {
                dx[col] = ext[7] - x0[xo];
                colmap[col] = dm.td_const ? -1 : col_td(dm.K);
                col += 1, xo += 1;
            }
        }
    }
}

// cost of all camera-only factors at (pose, mix, ext); optionally the linearisation (H_c, g_c of buffer b).  One CTA (256 threads).
// smem: per IMU factor 30 + 450 doubles; GNSS 3 + 18 each; misc.
// x += v on a global accumulator whose value the thread does not need back: one fire-and-forget reduction at the L2 (RED.ADD.F64) instead of a
// load -> add -> store chain (a dependent L2 round trip per entry: measured 50 k of ba_lin_cam's 123 k cycles in the IMU block accumulation).
// Every entry has ONE writer per phase and the phases are separated by block barriers, so the summation order is fixed (deterministic).
__device__ __forceinline__ void red_add(double *p, double v) { asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }

__device__ double cam_factors(const BaCaps &C, const BaDev &D, int w, const WinDims &dm, const double *pose, const double *mix, const double *ext,
                              bool lin, int b, double *smem) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int K = dm.K, N = 15 * K + 7;
    double *Hc = lin_Hc(C, D, b, w), *gc = lin_gc(C, D, b, w);
    double *s_imu = smem;                              // n_imu * 480
    double *s_gnss = s_imu + (size_t) C.K * 480;       // G * 24 : r[3] J[18] cost scale
    double *s_misc = s_gnss + (size_t) C.G * 24;       // pose prior r[6] J[36] | mix prior r[9] | marg dx[R] y[R] | costs
    double *s_pp = s_misc, *s_mp = s_misc + 48, *s_dx = s_mp + 16, *s_y = s_dx + C.R, *s_cost = s_y + C.R;
    int *s_colmap = (int *) (s_cost + 8);
    __shared__ double s_total;
#ifdef ICG_BA_PHASE_CLOCKS
    unsigned long long cclk = D.clk ? clock64() : 0ull;  // profiling build: phase clocks of the linearising call, window 0
#define CAM_CLK(k)                                                 \
    if (D.clk && lin && w == 0 && tid == 0) {                      \
        const unsigned long long t_ = clock64();                   \
        atomicAdd(&D.clk[16 + (k)], t_ - cclk), atomicAdd(&D.clk[24 + (k)], 1ull); \
        cclk = t_;                                                 \
    }
#else
#define CAM_CLK(k)
#endif
    // ---- phase 1: evaluate
    for (int k = warp; k < dm.n_imu; k += nwarps)
        imu_factor_warp(D.imu_blob + ((size_t) w * C.K + k) * ICG_IMU_BLOB_DOUBLES, D.imu_U + ((size_t) w * C.K + k) * 225, pose + k * 7, mix + k * 9,
                        pose + (k + 1) * 7, mix + (k + 1) * 9, lin, s_imu + (size_t) k * 480, s_imu + (size_t) k * 480 + 30, lane);
    if (tid < dm.n_gnss) {
        const int nd = D.gnss_node[(size_t) w * C.G + tid];
        double *o = s_gnss + tid * 24;
        gnss_eval(pose + nd * 7, D.gnss_blh + ((size_t) w * C.G + tid) * 3, D.gnss_std + ((size_t) w * C.G + tid) * 3, D.lever + (size_t) w * 3, lin, o, o + 3);
        double sq = o[0] * o[0] + o[1] * o[1] + o[2] * o[2], cost, sc = 1.0;
        if (dm.gnss_huber)
            huber(sq, cost, sc);
        else
            cost = 0.5 * sq;
        if (sc != 1.0) {
            for (int e = 0; e < 3; e++) o[e] *= sc;
            if (lin)
                for (int e = 0; e < 18; e++) o[3 + e] *= sc;
        }
        o[21] = cost;
    }
    if (tid == 64 && dm.has_pose_prior) pose_prior_eval(pose, D.pose_prior + (size_t) w * 7, D.pose_prior_sinfo + (size_t) w * 6, lin, s_pp, s_pp + 6);
    if (tid == 96 && dm.has_mix_prior)
        for (int k = 0; k < 9; k++) s_mp[k] = (mix[k] - D.mix_prior[(size_t) w * 9 + k]) / D.mix_prior_std[(size_t) w * 9 + k];
    if (dm.marg_r > 0) marg_dx(C, D, w, dm, pose, mix, ext, s_dx, s_colmap, tid, blockDim.x);
    __syncthreads();
    CAM_CLK(0)  // factor evaluation
    const double *H0 = D.marg_H0 + (size_t) w * C.R * C.R, *b0 = D.marg_b0 + (size_t) w * C.R;
    if (dm.marg_r > 0) {
        for (int i = tid; i < dm.marg_r; i += blockDim.x) {
            double s = 0;
            for (int k = 0; k < dm.marg_r; k++) s += H0[(size_t) i * dm.marg_r + k] * s_dx[k];
            s_y[i] = s;
        }
    }
    __syncthreads();
    // ---- cost (single thread, fixed order -> deterministic)
    if (tid == 0) {
        double c = 0;
        for (int k = 0; k < dm.n_imu; k++) {
            const double *r = s_imu + (size_t) k * 480;
            double sq = 0;
            for (int e = 0; e < 15; e++) sq += r[e] * r[e];
            c += 0.5 * sq;
        }
        for (int g = 0; g < dm.n_gnss; g++) c += s_gnss[g * 24 + 21];
        if (dm.has_imu_error) {
            const double *m = mix + dm.n_imu * 9;
            double sq = 0;
            for (int e = 0; e < 3; e++) sq += (m[3 + e] / IMU_GB_STD) * (m[3 + e] / IMU_GB_STD) + (m[6 + e] / IMU_AB_STD) * (m[6 + e] / IMU_AB_STD);
            c += 0.5 * sq;
        }
        if (dm.has_pose_prior) {
            double sq = 0;
            for (int e = 0; e < 6; e++) sq += s_pp[e] * s_pp[e];
            c += 0.5 * sq;
        }
        if (dm.has_mix_prior) {
            double sq = 0;
            for (int e = 0; e < 9; e++) sq += s_mp[e] * s_mp[e];
            c += 0.5 * sq;
        }
        if (dm.marg_r > 0) {
            // 0.5 |e0 + J0 dx|^2 = 0.5 (e0.e0 + 2 b0.dx + dx.H0.dx)
            double q = D.marg_c0[w];
            for (int i = 0; i < dm.marg_r; i++) q += (2.0 * b0[i] + s_y[i]) * s_dx[i];
            c += 0.5 * q;
        }
        s_total = c;
    }
    if (!lin) {
        __syncthreads();
        return s_total;
    }
    CAM_CLK(1)  // prior product + cost
    // ---- phase 2: H_c = sum J^T J, g_c = sum J^T r   (every entry has exactly one writer per round -> deterministic)
    for (int e = tid; e < N * C.NS; e += blockDim.x) Hc[e] = 0;
    for (int e = tid; e < N; e += blockDim.x) gc[e] = 0;
    __syncthreads();
    CAM_CLK(2)  // zero H_c
    if (dm.marg_r > 0) {
        const int r = dm.marg_r;
        for (int e = tid; e < r * r; e += blockDim.x) {
            int i = e / r, j = e - i * r;
            int ci = s_colmap[i], cj = s_colmap[j];
            if (ci >= 0 && cj >= 0) Hc[(size_t) ci * C.NS + cj] = H0[e];
        }
        for (int i = tid; i < r; i += blockDim.x)
            if (s_colmap[i] >= 0) gc[s_colmap[i]] = b0[i] + s_y[i];
    }
    __syncthreads();
    CAM_CLK(3)  // prior blocks
    for (int parity = 0; parity < 2; parity++) {  // IMU factors k and k+2 touch disjoint nodes
        const int nf = (dm.n_imu - parity + 1) / 2;
        for (int e = tid; e < nf * 930; e += blockDim.x) {
            const int k = parity + 2 * (e / 930), q = e % 930;
            const double *rw = s_imu + (size_t) k * 480, *Jw = rw + 30;
            auto gcol = [&](int c) { return c < 6 ? col_pose(k) + c : c < 15 ? col_mix(K, k) + c - 6 : c < 21 ? col_pose(k + 1) + c - 15 : col_mix(K, k + 1) + c - 21; };
            if (q < 900) {
                int a = q / 30, b = q - a * 30;
                double s = 0;
                for (int m = 0; m < 15; m++) s += Jw[m * 30 + a] * Jw[m * 30 + b];
                red_add(&Hc[(size_t) gcol(a) * C.NS + gcol(b)], s);
            } else {
                int a = q - 900;
                double s = 0;
                for (int m = 0; m < 15; m++) s += Jw[m * 30 + a] * rw[m];
                red_add(&gc[gcol(a)], s);
            }
        }
        __syncthreads();
    }
    CAM_CLK(4)  // IMU J^T J
    // pose-diagonal blocks: GNSS + pose prior; mix-diagonal: bias-magnitude factor + mix prior
    for (int e = tid; e < K * 42; e += blockDim.x) {
        const int k = e / 42, q = e % 42;
        double s = 0;
        if (q < 36) {
            const int a = q / 6, b = q % 6;
            for (int g = 0; g < dm.n_gnss; g++)
                if (D.gnss_node[(size_t) w * C.G + g] == k) {
                    const double *J = s_gnss + g * 24 + 3;
                    s += J[a] * J[b] + J[6 + a] * J[6 + b] + J[12 + a] * J[12 + b];
                }
            if (k == 0 && dm.has_pose_prior)
                for (int m = 0; m < 6; m++) s += s_pp[6 + m * 6 + a] * s_pp[6 + m * 6 + b];
            red_add(&Hc[(size_t) (col_pose(k) + a) * C.NS + col_pose(k) + b], s);
        } else {
            const int a = q - 36;
            for (int g = 0; g < dm.n_gnss; g++)
                if (D.gnss_node[(size_t) w * C.G + g] == k) {
                    const double *o = s_gnss + g * 24;
                    s += o[3 + a] * o[0] + o[9 + a] * o[1] + o[15 + a] * o[2];
                }
            if (k == 0 && dm.has_pose_prior)
                for (int m = 0; m < 6; m++) s += s_pp[6 + m * 6 + a] * s_pp[m];
            red_add(&gc[col_pose(k) + a], s);
        }
    }
    if (tid < 9) {
        if (dm.has_imu_error && tid >= 3) {
            const int k = dm.n_imu;
            const double sd = tid < 6 ? IMU_GB_STD : IMU_AB_STD;
            Hc[(size_t) (col_mix(K, k) + tid) * C.NS + col_mix(K, k) + tid] += 1.0 / (sd * sd);
            gc[col_mix(K, k) + tid] += mix[k * 9 + tid] / (sd * sd);
        }
    }
    __syncthreads();
    if (tid < 9 && dm.has_mix_prior) {
        const double sd = D.mix_prior_std[(size_t) w * 9 + tid];
        Hc[(size_t) (col_mix(K, 0) + tid) * C.NS + col_mix(K, 0) + tid] += 1.0 / (sd * sd);
        gc[col_mix(K, 0) + tid] += s_mp[tid] / sd;
    }
    __syncthreads();
    CAM_CLK(5)  // GNSS / prior diagonal blocks
#undef CAM_CLK
    return s_total;
}

// at_cand: as ba_lin_vis
__global__ void __launch_bounds__(CAM_THREADS) ba_lin_cam(BaCaps C, BaDev D, int at_cand) {
    extern __shared__ double smem[];
    const int w = blockIdx.x;
    LmState &st = D.st[w];
    if (st.done || !(at_cand ? st.step_valid : st.need_lin)) return;
    if (D.S.split && (w % D.world) != D.rank) return;  // split pipeline: the window's owner handles the camera-only factors
    const WinDims dm = D.dims[w];
    const int b = at_cand ? 1 - st.lin_buf : st.lin_buf;
    const double *pose = at_cand ? D.pose_c : D.pose, *mix = at_cand ? D.mix_c : D.mix, *ext = at_cand ? D.ext_c : D.ext;
    double c = cam_factors(C, D, w, dm, pose + (size_t) w * C.K * 7, mix + (size_t) w * C.K * 9, ext + (size_t) w * 8, true, b, smem);
    if (threadIdx.x == 0) st.cost_cam[b] = c;
}

// ------------------------------------------------------------------------------------------------ solve (one CTA per window)

__device__ __forceinline__ double block_sum(double v, double *s_red) {
    // deterministic block reduction (fixed tree)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    double t = 0;
    if (tid == 0) {
        for (int k = 0; k < (int) (blockDim.x >> 5); k++) t += s_red[k];
        s_red[32] = t;
    }
    __syncthreads();
    return s_red[32];
}
__device__ __forceinline__ double block_max(double v, double *s_red) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    if (tid == 0) {
        double t = 0;
        for (int k = 0; k < (int) (blockDim.x >> 5); k++) t = fmax(t, s_red[k]);
        s_red[32] = t;
    }
    __syncthreads();
    return s_red[32];
}

__global__ void __launch_bounds__(SOLVE_THREADS, 2) ba_solve(BaCaps C, BaDev D) {
    extern __shared__ double sm[];
    const int w = blockIdx.x, tid = threadIdx.x;
    LmState &st = D.st[w];
    if (st.done) return;
    // phase clocks (profiling BUILD only, -DICG_BA_PHASE_CLOCKS: the instrumentation perturbs register allocation): thread 0 of window 0 adds
    // the SM cycles since the previous mark
#ifdef ICG_BA_PHASE_CLOCKS
    unsigned long long clk_prev = D.clk ? clock64() : 0ull;
#define SOLVE_CLK(k)                                              \
    if (D.clk && w == 0 && tid == 0) {                            \
        const unsigned long long t_ = clock64();                  \
        atomicAdd(&D.clk[k], t_ - clk_prev), atomicAdd(&D.clk[8 + (k)], 1ull); \
        clk_prev = t_;                                            \
    }
#define SOLVE_CLK_NOW() (D.clk ? clock64() : 0ull)
#define SOLVE_CLK_ADD(k, t0)                                      \
    if (D.clk && w == 0 && tid == 0) atomicAdd(&D.clk[k], clock64() - (t0)), atomicAdd(&D.clk[8 + (k)], 1ull);
#else
#define SOLVE_CLK(k)
#define SOLVE_CLK_NOW() 0ull
#define SOLVE_CLK_ADD(k, t0)
#endif
    const WinDims dm = D.dims[w];
    const int K = dm.K, L = dm.L, NCV = 6 * K + 7, N = 15 * K + 7;
    const int f_first = st.first, f_fresh = st.fresh_lin, f_last = st.last_success, f_iter = st.iter;
    const double f_gmax_old = st.gmax;
    (void) f_gmax_old;
    // shared layout: vectors first, packed matrix last
    double *s_red = sm;                 // 40
    double *s_scale = s_red + 40;       // N
    double *s_g = s_scale + C.NS;       // N   full camera gradient (unscaled)
    double *s_rhs = s_g + C.NS;         // N   -> step' (scaled space)
    double *s_d2 = s_rhs + C.NS;        // N
    double *s_diag = s_d2 + C.NS;       // N   Cholesky diagonal
    // packed lower triangle, N + 1 rows, ALWAYS in shared memory (systems that do not fit are driven by the split pipeline, ba_solve_cam): a
    // pointer that could also be global made every access a generic LD / ST (longer latency, long-scoreboard tracked)
    double *S = s_diag + C.NS;
    const int b = st.lin_buf;
    const double *Hc = lin_Hc(C, D, b, w), *gcam = lin_gc(C, D, b, w), *Hs = D.Hs + (size_t) w * C.NS * C.NS;
    // Vision vectors [diag H_vis | g_vis | W phi g_l] (a < NCV), as ba_schur_dmma's epilogue wrote them.
    const double *V = D.visv + (size_t) (3 * C.NCV) * w;
    if (tid == 0 && st.need_lin) st.need_lin = 0;      // the linearisation kernels of this iteration have run (stream order)
    double *scale_c = D.scale_c + (size_t) w * C.NS;
    const double *hl = lin_hl(C, D, b, w), *gl = lin_gl(C, D, b, w), *scale_l = D.scale_l + (size_t) w * C.L;

    // ---- after a fresh linearisation: total cost, gradient, (first time) Jacobi scaling
    for (int a = tid; a < N; a += SOLVE_THREADS) {
        double g = gcam[a];
        if (a < NCV) g += V[NCV + a];
        s_g[a] = g;
        if (f_first) {
            double h = Hc[(size_t) a * C.NS + a] + (a < NCV ? V[a] : 0.0);
            scale_c[a] = 1.0 / (1.0 + sqrt(h));
        }
    }
    __syncthreads();
    for (int a = tid; a < N; a += SOLVE_THREADS) s_scale[a] = scale_c[a];
    double gmax_now = st.gmax;
    if (f_fresh) {
        double cs = 0, gq = 0;
        const double *costf = lin_costf(C, D, b, w);
        for (int f = tid; f < dm.F; f += SOLVE_THREADS) cs += costf[f];
        for (int l = tid; l < L; l += SOLVE_THREADS) gq = fmax(gq, fabs(gl[l]));
        const double c = block_sum(cs, s_red), gml = block_max(gq, s_red);
        double gm = 0;
        for (int a = tid; a < N; a += SOLVE_THREADS) gm = fmax(gm, fabs(s_g[a]));
        gm = fmax(block_max(gm, s_red), gml);
        gmax_now = gm;
        if (tid == 0) {
            st.x_cost = c + st.cost_cam[b];
            st.gmax = gm;
            if (f_first) st.initial_cost = st.x_cost;
            st.fresh_lin = 0;
        }
        __syncthreads();
    }
    if (f_first) {
        __syncthreads();
        if (tid == 0) st.first = 0;
    }
    {
        const int term = lm_term(f_iter, st.max_iter, f_last, gmax_now, st.radius);
        if (term) {
            __syncthreads();
            if (tid == 0) st.done = term, st.step_valid = 0;
            return;
        }
    }
    __syncthreads();
    if (tid == 0) st.iter++;
    const double radius = st.radius;
    SOLVE_CLK(0)  // gradient, cost, termination tests

    // ---- assemble S' = s (H - Schur) s + D^2 (packed lower), rhs' = -s (g - W phi g_l)
    // The reduced camera matrix (Hs, row i contiguous) goes global -> packed shared rows with 8-byte cp.async: every element of
    // the lower triangle is in flight at once (one L2 round trip for the whole matrix instead of one per row and warp), the vector part below
    // overlaps the copy, and the Jacobi scaling + LM diagonal are applied in place afterwards.
    constexpr bool async_fill = true;
    if (async_fill) {
        for (int i = tid >> 5; i < N; i += SOLVE_THREADS / 32) {
            const double *src = (i < NCV ? Hs : Hc) + (size_t) i * C.NS;
            const unsigned dst = (unsigned) __cvta_generic_to_shared(S + i * (i + 1) / 2);
            for (int j = tid & 31; j <= i; j += 32)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst + 8u * j), "l"(src + j) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (int a = tid; a < N; a += SOLVE_THREADS) {
        double h = Hc[(size_t) a * C.NS + a] + (a < NCV ? V[a] : 0.0);
        double hs = s_scale[a] * s_scale[a] * h;
        s_d2[a] = lm_d2(hs, radius);
        double gw = a < NCV ? V[2 * NCV + a] : 0.0;
        s_rhs[a] = -s_scale[a] * (s_g[a] - gw);
    }
    if (async_fill) asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    if (async_fill) {
        for (int i = tid >> 5; i < N; i += SOLVE_THREADS / 32) {
            double *row = S + i * (i + 1) / 2;
            const double si = s_scale[i];
            for (int j = tid & 31; j <= i; j += 32) {
                double v = si * s_scale[j] * row[j];
                if (i == j) v += s_d2[i];
                row[j] = v;
            }
        }
    } else {
        for (int i = tid >> 5; i < N; i += SOLVE_THREADS / 32) {
            // one warp per row; all global loads of the row are issued before the first store (memory-level parallelism)
            constexpr int MAXQ = 16;  // N <= 512
            double hv[MAXQ];
            const int nq = i / 32 + 1;
#pragma unroll
            for (int q = 0; q < MAXQ; q++) {
                const int j = (tid & 31) + 32 * q;
                hv[q] = 0;
                if (q < nq && j <= i) hv[q] = (i < NCV ? Hs : Hc)[(size_t) i * C.NS + j];  // Hs: H_c + vision Gram - Schur (vision rows); row i contiguous
            }
#pragma unroll
            for (int q = 0; q < MAXQ; q++) {
                const int j = (tid & 31) + 32 * q;
                if (q < nq && j <= i) {
                    double v = s_scale[i] * s_scale[j] * hv[q];
                    if (i == j) v += s_d2[i];
                    S[i * (i + 1) / 2 + j] = v;
                }
            }
        }
    }
    // augmented row N = rhs': the factorisation then leaves y = L^-1 rhs' in it (forward substitution for free)
    for (int a = tid; a < N; a += SOLVE_THREADS) S[N * (N + 1) / 2 + a] = s_rhs[a];
    __syncthreads();
    SOLVE_CLK(1)  // assembly
    // ---- blocked left-looking Cholesky on the packed lower triangle (two barriers per 8 columns); failure -> invalid step.
    // Per panel J (columns J0 .. J0 + 7):
    //   (1) panel update with all previous columns on the FP64 tensor cores, S[J0:, J0:J0+8] -= L[J0:, :J0] L[J0:J0+8, :J0]^T, one warp per
    //       8-row tile (A fragment = L[i0 + g][k0 + kk], B fragment = L[J0 + g][k0 + kk], DMMA.8x8x4, J0 % 8 == 0).  WARP 0 takes the
    //       diagonal tile alone and FACTORS it straight away (in registers: the 8-column pivot chain, ~8 x (DFMA + rsqrt + DMUL) = 600 cycles of
    //       pure latency) while warps 1..7 are still updating the tiles below -- the chain hides behind their tensor-core work.  (The
    //       previous version let every thread factor the block redundantly to save a barrier: measured, a barrier costs ~30 cycles here,
    //       the redundant factorisation ~3 000 issue slots per panel -- 58 % of the kernel.)
    //   (2) barrier; every row below the block (and the augmented rhs row) is solved against the factored block by its own thread; barrier.
    // 1/sqrt(d) comes from rsqrt (one dependent op per column instead of sqrt + divide); the row solve multiplies by it.
    __shared__ int s_fail;
    if (tid == 0) s_fail = 0;
    __syncthreads();
    const int NR = N + 1;
    for (int J0 = 0; J0 < N; J0 += BA_CHOL_NB) {
        const int nb = min(BA_CHOL_NB, N - J0);
        const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, kk = lane & 3;
        const int ntile = (NR - J0 + 7) / 8;
        const unsigned long long pc0 = SOLVE_CLK_NOW();  // profiling: warp 0's own work / the row-solve phase of this panel
        (void) pc0;
        const int cb = J0 + g;                                     // row of L that is the B operand's column
        const double *rb = S + (cb < NR ? cb * (cb + 1) / 2 : 0);
        const bool okb = cb < NR;
        if (warp == 0) {
            if (J0 > 0) {  // diagonal tile: rows J0 + g; four accumulator chains over the k range
                const double *ra = rb;
                double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                int k0 = 0;
                for (; k0 + 16 <= J0; k0 += 16) {
                    const double x0 = okb ? ra[k0 + kk] : 0.0, x1 = okb ? ra[k0 + 4 + kk] : 0.0, x2 = okb ? ra[k0 + 8 + kk] : 0.0, x3 = okb ? ra[k0 + 12 + kk] : 0.0;
                    dmma884(acc[0], acc[1], x0, x0);
                    dmma884(acc[2], acc[3], x1, x1);
                    dmma884(acc[4], acc[5], x2, x2);
                    dmma884(acc[6], acc[7], x3, x3);
                }
                for (; k0 + 8 <= J0; k0 += 8) {
                    const double x0 = okb ? ra[k0 + kk] : 0.0, x1 = okb ? ra[k0 + 4 + kk] : 0.0;
                    dmma884(acc[0], acc[1], x0, x0);
                    dmma884(acc[2], acc[3], x1, x1);
                }
                const double c0 = (acc[0] + acc[2]) + (acc[4] + acc[6]), c1 = (acc[1] + acc[3]) + (acc[5] + acc[7]);
                const int i = J0 + g;
                if (i < NR) {
                    const int ca = J0 + 2 * kk;
                    if (ca < J0 + nb && ca <= i) S[i * (i + 1) / 2 + ca] -= c0;
                    if (ca + 1 < J0 + nb && ca + 1 <= i) S[i * (i + 1) / 2 + ca + 1] -= c1;
                }
                __syncwarp();
            }
            // factor the nb x nb diagonal block: every lane of warp 0 runs the same register code on broadcast loads (no divergence, no
            // shuffles on the chain); lane a writes row a of L_JJ and its pivot reciprocal back
            double Ld[BA_CHOL_NB][BA_CHOL_NB], dinv[BA_CHOL_NB];
            bool bad = false;
#pragma unroll
            for (int a = 0; a < BA_CHOL_NB; a++)
#pragma unroll
                for (int b = 0; b < BA_CHOL_NB; b++) Ld[a][b] = (a < nb && b <= a) ? S[(J0 + a) * (J0 + a + 1) / 2 + J0 + b] : (a == b ? 1.0 : 0.0);
#pragma unroll
            for (int j = 0; j < BA_CHOL_NB; j++) {
                double d = Ld[j][j];
#pragma unroll
                for (int k = 0; k < j; k++) d -= Ld[j][k] * Ld[j][k];
                if (!(d > 0.0) || !isfinite(d)) bad = true;
                const double di = rsqrt(d);
                dinv[j] = di;
                Ld[j][j] = d * di;
#pragma unroll
                for (int a = j + 1; a < BA_CHOL_NB; a++) {
                    double sum = Ld[a][j];
#pragma unroll
                    for (int k = 0; k < j; k++) sum -= Ld[a][k] * Ld[j][k];
                    Ld[a][j] = sum * di;
                }
            }
            __syncwarp();  // every lane has read the unfactored block
            if (bad && lane == 0) s_fail = 1;
#pragma unroll
            for (int a2 = 0; a2 < BA_CHOL_NB; a2++) {
                // every lane holds the whole factor: entry (a2, b) is stored by ONE lane under a predicate -- statically indexed registers and no
                // divergent code.  ("lane a writes row a" was compiled into a switch on the lane, eight serial paths, several times slower in
                // ba_solve_cam_dsm's phase clocks than this form.)
                double *ri = S + (J0 + a2) * (J0 + a2 + 1) / 2 + J0;
#pragma unroll
                for (int b = 0; b <= a2; b++)
                    if (lane == ((a2 * 8 + b) & 31) && a2 < nb) ri[b] = Ld[a2][b];
                if (lane == 8 + a2 && a2 < nb) s_diag[J0 + a2] = dinv[a2];
            }
            SOLVE_CLK_ADD(6, pc0)
        } else if (J0 > 0 && warp != 4) {
            // tiles 1 .. ntile-1 over warps 1, 2, 3, 5, 6, 7, up to four row tiles per warp in flight (they share the B fragment): N = 157 gives
            // <= 19 such tiles, so the whole panel update is ONE round of the k loop, and eight independent DMMA chains hide the tensor-pipe
            // latency.  Warp 4 sits out: it shares warp 0's scheduler and FP64 pipe (warp id mod 4), and every DMMA holds that pipe for 16
            // cycles -- measured, warp 0's 130-operation pivot chain took 3 600 cycles per panel queuing behind warp 4's tiles.
            constexpr int TPW = 4, NWARP = 6;
            const int wslot = warp < 4 ? warp - 1 : warp - 2;  // 0..5
            for (int t0 = 1 + wslot; t0 < ntile; t0 += TPW * NWARP) {
                const double *ra[TPW];
                bool oka[TPW];
                double acc[TPW][4];
#pragma unroll
                for (int u = 0; u < TPW; u++) {
                    const int ia = J0 + 8 * (t0 + u * NWARP) + g;
                    oka[u] = (t0 + u * NWARP) < ntile && ia < NR;
                    ra[u] = S + (oka[u] ? ia * (ia + 1) / 2 : 0);
                    acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0;
                }
                for (int k0 = 0; k0 + 8 <= J0; k0 += 8) {
                    const double b0 = okb ? rb[k0 + kk] : 0.0, b1 = okb ? rb[k0 + 4 + kk] : 0.0;
                    double a0[TPW], a1[TPW];
#pragma unroll
                    for (int u = 0; u < TPW; u++) a0[u] = oka[u] ? ra[u][k0 + kk] : 0.0, a1[u] = oka[u] ? ra[u][k0 + 4 + kk] : 0.0;
#pragma unroll
                    for (int u = 0; u < TPW; u++) {
                        dmma884(acc[u][0], acc[u][1], a0[u], b0);
                        dmma884(acc[u][2], acc[u][3], a1[u], b1);
                    }
                }
#pragma unroll
                for (int u = 0; u < TPW; u++) {
                    const double c0 = acc[u][0] + acc[u][2], c1 = acc[u][1] + acc[u][3];
                    const int i = J0 + 8 * (t0 + u * NWARP) + g;
                    if (oka[u]) {
                        const int ca = J0 + 2 * kk;
                        if (ca < J0 + nb && ca <= i) S[i * (i + 1) / 2 + ca] -= c0;
                        if (ca + 1 < J0 + nb && ca + 1 <= i) S[i * (i + 1) / 2 + ca + 1] -= c1;
                    }
                }
            }
        }
        __syncthreads();
        const unsigned long long pc1 = SOLVE_CLK_NOW();
        (void) pc1;
        if (s_fail) break;
        // rows below the block (incl. the augmented rhs row): solve against the factored block, one row per thread.  L_JJ and the pivot
        // reciprocals are read from shared memory as the chain needs them (every thread reads the same address: broadcast, off the
        // dependent chain) instead of being staged in 36 + 8 registers
        for (int i = J0 + nb + tid; i < NR; i += SOLVE_THREADS) {
            double *ri = S + i * (i + 1) / 2 + J0;
            double x[BA_CHOL_NB];
#pragma unroll
            for (int c = 0; c < BA_CHOL_NB; c++) x[c] = c < nb ? ri[c] : 0.0;
#pragma unroll
            for (int c = 0; c < BA_CHOL_NB; c++) {
                if (c < nb) {
                    const double *lc = S + (J0 + c) * (J0 + c + 1) / 2 + J0;
                    double sum = x[c];
#pragma unroll
                    for (int k = 0; k < c; k++) sum -= x[k] * lc[k];
                    x[c] = sum * s_diag[J0 + c];
                }
            }
#pragma unroll
            for (int c = 0; c < BA_CHOL_NB; c++)
                if (c < nb) ri[c] = x[c];
        }
        __syncthreads();
        SOLVE_CLK_ADD(7, pc1)
    }
    __syncthreads();
    bool valid = !s_fail;
    SOLVE_CLK(2)  // Cholesky
    // ---- backward substitution L^T x = y, blocked by the factorisation's 8-column panels, last panel first:
    //   (a) warp 0 solves the panel's 8 x 8 triangle L_JJ^T x_J = y_J in registers (every lane the same code on broadcast loads; the
    //       dependent chain is 8 x (DFMA + DMUL));
    //   (b) barrier; every thread i < J0 applies the panel to its own entry, y_i -= sum_c L[J0 + c][i] x_{J0 + c} -- row J0 + c of the
    //       packed triangle is contiguous in i, so the reads are coalesced; barrier.
    // Same operations in the same order as a column-by-column substitution (c descending), on 256 threads instead of one warp:
    // measured 185 cycles per COLUMN for the single-warp form (29 k cycles at N = 157), about 400 cycles per PANEL for this one.
    if (valid) {
        double *y = S + N * (N + 1) / 2;
        const int lane = tid & 31;
        for (int J0 = ((N - 1) / BA_CHOL_NB) * BA_CHOL_NB; J0 >= 0; J0 -= BA_CHOL_NB) {
            const int nb = min(BA_CHOL_NB, N - J0);
            if (tid < 32) {
                double x[BA_CHOL_NB];
#pragma unroll
                for (int c = BA_CHOL_NB - 1; c >= 0; c--) {
                    x[c] = 0.0;
                    if (c < nb) {
                        double sum = y[J0 + c];
#pragma unroll
                        for (int k = BA_CHOL_NB - 1; k > c; k--)
                            if (k < nb) sum -= S[(J0 + k) * (J0 + k + 1) / 2 + J0 + c] * x[k];
                        x[c] = sum * s_diag[J0 + c];
                    }
                }
#pragma unroll
                for (int c = 0; c < BA_CHOL_NB; c++)
                    if (c == lane && c < nb) s_rhs[J0 + c] = x[c];
            }
            __syncthreads();
            for (int i = tid; i < J0; i += SOLVE_THREADS) {
                double acc = y[i];
#pragma unroll
                for (int c = BA_CHOL_NB - 1; c >= 0; c--)
                    if (c < nb) acc -= S[(J0 + c) * (J0 + c + 1) / 2 + i] * s_rhs[J0 + c];
                y[i] = acc;
            }
            __syncthreads();
        }
    }
    __syncthreads();
    SOLVE_CLK(3)  // camera back-substitution
    // ---- landmark back-substitution + model cost change  (-1/2 step'.g' + 1/2 step'.D^2 step', exact identity of
    //      Ceres' -(J' step)^T (r + J' step / 2) for the damped normal-equation solution)
    double *step_l = D.step_l + (size_t) w * C.L;
    const double *AW = lin_AW(C, D, b, w);  // landmark-major
    double part = 0;
    bool finite = true;
    double *R2 = D.red2 + (size_t) w * 4;
    if (!valid) {
        // Cholesky breakdown: the step is invalid; ba_accept applies HandleInvalidStep
        if (tid == 0) {
            st.chol_ok = 0, st.step_valid = 0;
            R2[0] = 0, R2[1] = 0, R2[2] = 1;
        }
        return;
    }
    for (int a = tid; a < N; a += SOLVE_THREADS) {
        double sp = s_rhs[a];
        finite = finite && isfinite(sp);
        part += -0.5 * sp * (s_scale[a] * s_g[a]) + 0.5 * s_d2[a] * sp * sp;
    }
    // landmark back-substitution: one warp per landmark, the coupling row is read coalesced (two landmarks in flight per warp)
    double *s_sx = s_diag;  // s_diag is dead after the back-substitution: scaled camera step s_c * step'_c
    __syncthreads();
    for (int a = tid; a < NCV; a += SOLVE_THREADS) s_sx[a] = s_scale[a] * s_rhs[a];
    __syncthreads();
    {
        const int lane = tid & 31, warp = tid >> 5;
        constexpr int LB = 8;  // landmarks in flight per warp (the coupling rows come from L2: 24 loads per lane outstanding)
        // after the transposing reduction below, lane holds the dot product of landmark l0 + lu; its per-landmark scalars are loaded at the top
        // of the round, together with the coupling rows (one L2 round trip per round instead of two)
        const int lu = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
        for (int l0 = LB * warp; l0 < L; l0 += LB * (SOLVE_THREADS / 32)) {
            const int l = l0 + lu;
            const bool lok = l < L;
            const double sl = lok ? scale_l[l] : 0.0, hh = lok ? hl[l] : 0.0, gg = lok ? gl[l] : 0.0;
            double d[LB];
#pragma unroll
            for (int u = 0; u < LB; u++) d[u] = 0;
            for (int c = lane; c < NCV; c += 32) {
                const double sx = s_sx[c];
#pragma unroll
                for (int u = 0; u < LB; u++) d[u] += (l0 + u < L ? AW[(size_t) (l0 + u) * C.NCA + c] : 0.0) * sx;
            }
            const double hs = sl * sl * hh, d2 = lm_d2(hs, radius), den = hs + d2, sg = sl * gg;
            // transposing butterfly: 8 values x 32 lanes -> 1 value per lane in 4 + 2 + 1 + 1 + 1 exchanges (a plain butterfly needs 8 x 5)
            double e4[4], e2[2];
            {
                const bool hi = lane & 16;
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const double keep = hi ? d[u + 4] : d[u], send = hi ? d[u] : d[u + 4];
                    e4[u] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
                }
            }
            {
                const bool hi = lane & 8;
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const double keep = hi ? e4[u + 2] : e4[u], send = hi ? e4[u] : e4[u + 2];
                    e2[u] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
                }
            }
            double mine;
            {
                const bool hi = lane & 4;
                const double keep = hi ? e2[1] : e2[0], send = hi ? e2[0] : e2[1];
                mine = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            mine += __shfl_xor_sync(0xffffffffu, mine, 2);
            mine += __shfl_xor_sync(0xffffffffu, mine, 1);
            if ((lane & 3) == 0 && lok) {
                double sp = (-sg - sl * mine) / den;
                finite = finite && isfinite(sp);
                step_l[l] = sp;
                part += -0.5 * sp * sg + 0.5 * d2 * sp * sp;
            }
        }
    }
    __syncthreads();
    SOLVE_CLK(4)  // landmark back-substitution
    const double mcc = block_sum(part, s_red);
    const double nfin = block_sum(finite ? 0.0 : 1.0, s_red);
    // ---- candidate point x (+) delta, delta = step' * scale; |x - x_cand|^2 over active blocks
    const double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8, *rho = D.rho + (size_t) w * C.L;
    double *pose_c = D.pose_c + (size_t) w * C.K * 7, *mix_c = D.mix_c + (size_t) w * C.K * 9, *ext_c = D.ext_c + (size_t) w * 8, *rho_c = D.rho_c + (size_t) w * C.L;
    double sn = 0;
    for (int k = tid; k <= K; k += SOLVE_THREADS) {  // K poses + the extrinsic
        const bool is_ext = (k == K);
        const double *x = is_ext ? ext : pose + k * 7;
        double *xc = is_ext ? ext_c : pose_c + k * 7;
        if (is_ext && dm.ext_const) {
            for (int e = 0; e < 7; e++) xc[e] = x[e];
        } else {
            const int c0 = is_ext ? col_ext(K) : col_pose(k);
            double d[6];
            for (int e = 0; e < 6; e++) d[e] = s_rhs[c0 + e] * s_scale[c0 + e];
            pose_plus(x, d, xc);
            for (int e = 0; e < 7; e++) sn += (x[e] - xc[e]) * (x[e] - xc[e]);
        }
    }
    for (int e = tid; e < K * 9; e += SOLVE_THREADS) {
        int k = e / 9, q = e - 9 * k, c = col_mix(K, k) + q;
        double v = mix[e] + s_rhs[c] * s_scale[c];
        mix_c[e] = v;
        sn += (mix[e] - v) * (mix[e] - v);
    }
    if (tid == 0) {
        if (dm.td_const) {
            ext_c[7] = ext[7];
        } else {
            double v = ext[7] + s_rhs[col_td(K)] * s_scale[col_td(K)];
            ext_c[7] = v;
            sn += (ext[7] - v) * (ext[7] - v);
        }
    }
    for (int l = tid; l < L; l += SOLVE_THREADS) {
        double v = rho[l] + step_l[l] * scale_l[l];
        rho_c[l] = v;
        sn += (rho[l] - v) * (rho[l] - v);
    }
    sn = block_sum(sn, s_red);
    if (tid == 0) {
        st.chol_ok = 1, st.step_valid = 1;  // provisional: ba_accept validates with the reduced model cost change
        R2[0] = mcc, R2[1] = sn, R2[2] = nfin;
    }
    SOLVE_CLK(5)  // candidate point, reductions
#undef SOLVE_CLK
#undef SOLVE_CLK_NOW
#undef SOLVE_CLK_ADD
}

// ------------------------------------------------------------------------------------------------ candidate cost (split pipeline)
// The single-GPU pipeline takes the candidate cost from the linearisation at the candidate instead (ba_accept).
// camera-only factors at the candidate point (one CTA per window; runs beside the vision blocks on the handle's second stream)
__global__ void __launch_bounds__(CAM_THREADS) ba_cost_cam(BaCaps C, BaDev D, int nblk_vis) {
    extern __shared__ double smem[];
    const int w = blockIdx.x;
    const LmState &st = D.st[w];
    if (st.done || !st.step_valid) return;
    if (D.S.split && (w % D.world) != D.rank) return;
    const WinDims dm = D.dims[w];
    double c = cam_factors(C, D, w, dm, D.pose_c + (size_t) w * C.K * 7, D.mix_c + (size_t) w * C.K * 9, D.ext_c + (size_t) w * 8, false, 0, smem);
    if (threadIdx.x == 0) D.cost_part[(size_t) w * (nblk_vis + 1) + nblk_vis] = c;
}
__global__ void __launch_bounds__(256) ba_cost(BaCaps C, BaDev D, int nblk_vis) {
    __shared__ double s_red[40];
    const int w = blockIdx.y;
    const LmState &st = D.st[w];
    if (st.done || !st.step_valid) return;
    const WinDims dm = D.dims[w];
    const double *pose = D.pose_c + (size_t) w * C.K * 7, *ext = D.ext_c + (size_t) w * 8, *rho = D.rho_c + (size_t) w * C.L;
    double *part = D.cost_part + (size_t) w * (nblk_vis + 1);
    const int q = blockIdx.x * 256 + threadIdx.x;  // record slot (landmark-CSR order): the slot-ordered copies are the only factor data on the device
    __shared__ double s_frame[BA_MAX_NODES + 1][NODE_FRAME_LD];  // node frames of the candidate point (see ba_lin_vis)
    if ((int) threadIdx.x <= dm.K) node_frame((int) threadIdx.x < dm.K ? pose + threadIdx.x * 7 : ext, s_frame[threadIdx.x]);
    __syncthreads();
    double cost = 0;
    int4 meta = make_int4(0, 0, 0, 0);
    if (q < dm.F) meta = ((const int4 *) D.f_meta_s)[(size_t) w * C.F + q];  // (landmark, reference node, observing node, factor id)
    if (q < dm.F && D.f_active[(size_t) w * C.F + meta.w]) {
        double r[2];
        reproj_eval_frames(s_frame[meta.y], s_frame[meta.z], s_frame[dm.K], rho[meta.x], ext[7], D.f_const_s + ((size_t) w * C.F + q) * 14, dm.reproj_sinv,
                           false, r, nullptr, nullptr, nullptr, nullptr, nullptr);
        double sq = r[0] * r[0] + r[1] * r[1], sc;
        if (dm.reproj_huber)
            huber(sq, cost, sc);
        else
            cost = 0.5 * sq;
    }
    cost = block_sum(cost, s_red);
    if (threadIdx.x == 0) part[blockIdx.x] = cost;
}

// ------------------------------------------------------------------------------------------------ accept / reject
__global__ void __launch_bounds__(128) ba_accept(BaCaps C, BaDev D) {
    __shared__ int s_accept;
    __shared__ double s_camsq, s_rhosq;
    __shared__ double s_red[40];
    const int w = blockIdx.x, tid = threadIdx.x;
    LmState &st = D.st[w];
    if (st.done) return;
    const WinDims dm = D.dims[w];
    const double *R2 = D.red2 + (size_t) w * 4;
    // |x|^2 of the camera-side blocks and of the landmarks
    {
        const double s = lm_cam_sq(C, D, w, dm, s_red);
        double q = 0;  // |rho|^2
        for (int l = tid; l < dm.L; l += 128) q += D.rho[(size_t) w * C.L + l] * D.rho[(size_t) w * C.L + l];
        q = block_sum(q, s_red);
        if (tid == 0) s_camsq = s, s_rhosq = q;
    }
    // The candidate cost from the linearisation at the candidate (buffer 1 - lin_buf), summed in ba_cost's order -- per 256 record slots
    // block_sum's tree (warp k sums slots [32 k, 32 k + 32) of the block, then the eight warp sums in order), the blocks in order, then the
    // camera-only cost -- so that every decision below matches the sum of ba_cost's partials bit for bit.
    // s_warp (dynamic, 8 per 256 slots): the sums of the 32-slot groups; warp k of this CTA reduces groups k, k + 4, ... with no barrier in
    // between, so that the loads of several groups are in flight together.
    extern __shared__ double s_warp[];
    const int lane = tid & 31, warp = tid >> 5, ngrp = (dm.F + 31) / 32;
    if (st.step_valid) {
        const double *costf = lin_costf(C, D, 1 - st.lin_buf, w);
        const int4 *meta = (const int4 *) D.f_meta_s + (size_t) w * C.F;  // (landmark, reference node, observing node, factor id) per slot
#pragma unroll 4
        for (int g = warp; g < ngrp; g += 4) {
            const int q = 32 * g + lane;
            double v = q < dm.F ? costf[meta[q].w] : 0.0;  // lin_vis leaves 0 for an inactive factor
            for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
            if (lane == 0) s_warp[g] = v;
        }
    }
    __syncthreads();
    if (tid == 0) {
        const double mcc = R2[0], sn = R2[1], nfin = R2[2];
        double cand = 0;
        if (st.step_valid) {
            for (int g0 = 0; g0 < ngrp; g0 += 8) {
                double t = 0;
                for (int k = 0; k < 8; k++) t += g0 + k < ngrp ? s_warp[g0 + k] : 0.0;
                cand += t;
            }
            cand += st.cost_cam[1 - st.lin_buf];
        }
        s_accept = lm_decide(st, mcc, sn, nfin, s_camsq + s_rhosq, cand);
        if (s_accept) st.lin_buf ^= 1;  // the candidate's linearisation is now the one at x
    }
    __syncthreads();
    if (s_accept) lm_take_cand(C, D, w, dm);
}

// ------------------------------------------------------------------------------------------------ LM state reset (device side)
__global__ void ba_reset_state(BaDev D, LmState *save, int n, int max_iter) {
    int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n) return;
    if (save) save[w] = D.st[w];
    LmState st;
    memset(&st, 0, sizeof(st));
    st.radius = 1e4, st.decrease_factor = 2.0;  // Ceres initial_trust_region_radius
    st.need_lin = 1, st.fresh_lin = 1, st.first = 1, st.last_success = 1, st.max_iter = max_iter;
    D.st[w] = st;
}

// The outlier pass between the two solves of GVINS::gvinsOptimization (IG/ic_gvins.cc:1196-1207):
//   gnssOutlierCullingByChi2 (:1241-1267): chi2 = 2 cost > 7.815 -> std *= sqrt(chi2 / 7.815)
//   removeReprojectionFactorsByChi2 (:1269-1297): chi2 = 2 cost > 5.991 -> RemoveResidualBlock
//   GNSS factors re-added without loss function (:1202-1207)
__global__ void __launch_bounds__(128) ba_chi2_cull(BaCaps C, BaDev D, int *counters) {
    const int w = blockIdx.y;
    WinDims &dm = D.dims[w];
    const int t = blockIdx.x * 128 + threadIdx.x;
    const double *pose = D.pose + (size_t) w * C.K * 7, *ext = D.ext + (size_t) w * 8, *rho = D.rho + (size_t) w * C.L;
    int4 meta = make_int4(0, 0, 0, 0);
    if (t < dm.F) meta = ((const int4 *) D.f_meta_s)[(size_t) w * C.F + t];  // record slot t
    if (t < dm.F && D.f_active[(size_t) w * C.F + meta.w]) {
        double r[2];
        reproj_eval(pose + meta.y * 7, pose + meta.z * 7, ext, rho[meta.x], ext[7], D.f_const_s + ((size_t) w * C.F + t) * 14, dm.reproj_sinv, false, r, nullptr,
                    nullptr, nullptr, nullptr, nullptr);
        if ((r[0] * r[0] + r[1] * r[1]) > 5.991) {
            D.f_active[(size_t) w * C.F + meta.w] = 0;
            atomicAdd(&counters[2 * w], 1);
        }
    }
    if (t < dm.n_gnss) {
        double r[3];
        double *sd = D.gnss_std + ((size_t) w * C.G + t) * 3;
        gnss_eval(pose + D.gnss_node[(size_t) w * C.G + t] * 7, D.gnss_blh + ((size_t) w * C.G + t) * 3, sd, D.lever + (size_t) w * 3, false, r, nullptr);
        double chi2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
        if (chi2 > 7.815) {
            double sc = sqrt(chi2 / 7.815);
            sd[0] *= sc, sd[1] *= sc, sd[2] *= sc;
            atomicAdd(&counters[2 * w + 1], 1);
        }
    }
}
__global__ void ba_set_gnss_huber(BaDev D, int n, int v) {
    int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w < n) D.dims[w].gnss_huber = v;
}

// ------------------------------------------------------------------------------------------------ utility kernels
__global__ void ba_residual_costs_kernel(BaCaps C, BaDev D, double *reproj_cost, double *gnss_cost) {
    const int w = 0;
    const WinDims dm = D.dims[w];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const double *pose = D.pose, *ext = D.ext, *rho = D.rho;
    if (t < dm.F) {
        double r[2];
        const int4 meta = ((const int4 *) D.f_meta_s)[t];  // record slot t -> (landmark, reference node, observing node, factor id)
        reproj_eval(pose + meta.y * 7, pose + meta.z * 7, ext, rho[meta.x], ext[7], D.f_const_s + (size_t) t * 14, dm.reproj_sinv, false, r, nullptr, nullptr,
                    nullptr, nullptr, nullptr);
        reproj_cost[meta.w] = 0.5 * (r[0] * r[0] + r[1] * r[1]);  // EvaluateResidualBlock(id, false, &cost, ...) (IG/ic_gvins.cc:1278)
    }
    if (t < dm.n_gnss) {
        double r[3];
        gnss_eval(pose + D.gnss_node[t] * 7, D.gnss_blh + t * 3, D.gnss_std + t * 3, D.lever, false, r, nullptr);
        gnss_cost[t] = 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    }
}

__global__ void ba_reproj_eval_kernel(const double *in /* 7+7+8+1+1+14+1 */, double *out /* 2 + 14+14+14+2+2 */) {
    double r[2], Ji[12], Jj[12], Je[12], Jr[2], Jt[2];
    reproj_eval(in, in + 7, in + 14, in[22], in[23], in + 24, 1.0 / in[38], true, r, Ji, Jj, Je, Jr, Jt);
    out[0] = r[0], out[1] = r[1];
    double *o = out + 2;
    const double *src[3] = {Ji, Jj, Je};
    for (int b = 0; b < 3; b++)
        for (int rr = 0; rr < 2; rr++) {
            for (int c = 0; c < 6; c++) o[b * 14 + rr * 7 + c] = src[b][rr * 6 + c];
            o[b * 14 + rr * 7 + 6] = 0.0;  // the quaternion-w column of the global Jacobian is zero (reprojection_factor.h:103,114,131)
        }
    o[42] = Jr[0], o[43] = Jr[1], o[44] = Jt[0], o[45] = Jt[1];
}

__global__ void ba_imu_eval_kernel(const double *blob, const double *U, const double *x /* 7 9 7 9 */, double *out /* 15 + 450 */) {
    __shared__ double s_buf[480];
    imu_factor_warp(blob, U, x, x + 7, x + 16, x + 23, true, s_buf, s_buf + 30, threadIdx.x);
    for (int e = threadIdx.x; e < 15; e += 32) out[e] = s_buf[e];
    for (int e = threadIdx.x; e < 450; e += 32) out[15 + e] = s_buf[30 + e];
}

// GnssFactor / ImuPosePriorFactor / ImuMixPriorFactor / ImuErrorFactor (kind 0..3), one thread; in / out layouts in the callers below
__global__ void ba_small_factor_eval_kernel(int kind, const double *in, double *out) {
    if (kind == 0) {         // in: pose7 blh3 std3 lever3 -> r[3], J local 3x6
        gnss_eval(in, in + 7, in + 10, in + 13, true, out, out + 3);
    } else if (kind == 1) {  // in: pose7 prior7 sinfo6 -> r[6], J local 6x6
        pose_prior_eval(in, in + 7, in + 14, true, out, out + 6);
    } else if (kind == 2) {  // in: mix9 prior9 std9 -> r[9], diag J[9]   (ImuMixPriorFactor, imu_mix_prior_factor.h:40-75)
        for (int k = 0; k < 9; k++) out[k] = (in[k] - in[9 + k]) / in[18 + k], out[9 + k] = 1.0 / in[18 + k];
    } else {                 // in: mix9 -> r[6], diag J[6]                (ImuErrorFactor, imu_error_factor.h:45-91)
        for (int k = 0; k < 3; k++) {
            out[k] = in[3 + k] / IMU_GB_STD, out[3 + k] = in[6 + k] / IMU_AB_STD;
            out[6 + k] = 1.0 / IMU_GB_STD, out[9 + k] = 1.0 / IMU_AB_STD;
        }
    }
}

// MarginalizationFactor::Evaluate (IG/factors/marginalization_factor.h:47-101): e = e0 + J0 dx with dx the local difference of every
// remained block to its linearisation point (quaternion blocks: 2 vec(q0^-1 q), sign-fixed).  One CTA; thread per residual row.
// in: [r, nb, types[nb], x (global sizes, concatenated), x0 (same), e0[r], J0[r*r]] as doubles; out: residuals[r]
__global__ void ba_marg_factor_eval_kernel(const double *in, double *out) {
    extern __shared__ double s_dx[];
    const int r = (int) in[0], nb = (int) in[1];
    const double *types = in + 2;
    int tot = 0;
    for (int b = 0; b < nb; b++) tot += ((int) types[b] == 1) ? 9 : ((int) types[b] == 3) ? 1 : 7;
    const double *x = types + nb, *x0 = x + tot, *e0 = x0 + tot, *J0 = e0 + r;
    if (threadIdx.x == 0) {
        int col = 0, xo = 0;
        for (int b = 0; b < nb; b++) {
            const int t = (int) types[b];
            if (t == 0 || t == 2) {
                Q dq = qmul(qinv(pose_q(x0 + xo)), pose_q(x + xo));
                V3 a = 2.0 * qv(dq);
                if (dq.w < 0) a = -a;
                for (int k = 0; k < 3; k++) s_dx[col + k] = x[xo + k] - x0[xo + k];
                s_dx[col + 3] = a.x, s_dx[col + 4] = a.y, s_dx[col + 5] = a.z;
                col += 6, xo += 7;
            } else {
                const int g = t == 1 ? 9 : 1;
                for (int k = 0; k < g; k++) s_dx[col + k] = x[xo + k] - x0[xo + k];
                col += g, xo += g;
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < r; i += blockDim.x) {
        double sum = e0[i];
        for (int k = 0; k < r; k++) sum += J0[(size_t) i * r + k] * s_dx[k];
        out[i] = sum;
    }
}

// Every landmark's reference row (pts0, vel0, td0 of its factors' constants) into out: the old row of the landmark a slide carries (win / map:
// the slide's staging), otherwise its first factor's (record slot order), otherwise NaN.  One thread per landmark position, blockIdx.y = window.
__global__ void ba_lm_ref_fill(const WinDims *dims, const SlideWin *win, const int *map, const double *old, const double *fc, const int *lm_off,
                               const int *lm_perm, double *out, int Lc, int Fc) {
    const int w = blockIdx.y, L = dims[w].L;
    const size_t wL = (size_t) w * Lc;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < L; p += gridDim.x * blockDim.x) {
        const int l = lm_perm[wL + p], m = win ? map[win[w].lm_map + l] : -1;
        const int q0 = lm_off[(size_t) w * (Lc + 1) + p], q1 = lm_off[(size_t) w * (Lc + 1) + p + 1];
        double *r = out + (wL + l) * 7;
        if (m >= 0) {
            for (int c = 0; c < 7; c++) r[c] = old[(wL + m) * 7 + c];
        } else if (q1 > q0) {
            const double *f = fc + ((size_t) w * Fc + q0) * 14;
            r[0] = f[0], r[1] = f[1], r[2] = f[2], r[3] = f[6], r[4] = f[7], r[5] = f[8], r[6] = f[12];
        } else {
            for (int c = 0; c < 7; c++) r[c] = __longlong_as_double(0x7ff8000000000000LL);
        }
    }
}

}  // namespace icg

#include "ba_split.cuh"
#include "ba_marg.cuh"
