// ba_marg.cuh -- sliding-window marginalization on the device (SURVEY.md 8a row B10).  Included by ba.cu (it reuses the factor
// kernels and the handle of the window solve).
//
// Replaces MarginalizationInfo::marginalization (IG/factors/marginalization_info.h:73-101: preMarginalization :253-285,
// constructEquation :195-226, schurElimination :170-193, linearization :153-168) as GVINS::gvinsMarginalization drives it
// (IG/ic_gvins.cc:1412-1640): the num_marg oldest nodes (pose + mix) and the inverse depths anchored in them are removed; the
// factors that touch them (previous prior, GNSS, preintegration, first-window priors, reprojection factors of those landmarks -- all
// WITHOUT loss function, ic_gvins.cc:1499,1510,1532,1543,1605) are linearised at the current estimate; the new prior is
// J0 = S^1/2 V^T, e0 = -S^-1/2 V^T bp of the Schur complement Hp = Hrr - Hrm Hmm^+ Hmr (eigen-pseudo-inverse, EPS 1e-8).
//
// Device plan (batched over windows, one CTA per window per stage):
//   lin_vis                         (the solve's own kernel, loss + constant-block masks switched off) -> per-landmark coupling
//                                    rows (lin_vis phase 3), per-(ref,obs) 20x20 Gram matrices
//   marg_assemble                   dense H0, b0 in the [marginalized | remained] column order (one writer per entry per stage)
//   marg_jacobi(Hmm)                one-sided (Hestenes) Jacobi: columns of G = Hmm V orthogonalised by plane rotations, one warp per
//                                    column pair, round-robin ordering; lambda_i = v_i . g_i
//   marg_schur                      Z = Lambda^-1/2 V^T [Hmr | bm];  Hp = Hrr - Z^T Z, bp = br - Z^T z_b
//   marg_jacobi(Hp) + marg_finish   J0, e0 (rows sorted by ascending eigenvalue, as Eigen::SelfAdjointEigenSolver returns them)
// Eigen's SelfAdjointEigenSolver (tridiagonal QR) is un-vendored; Jacobi gives the same decomposition up to rounding and the
// prior only enters through J0^T J0, J0^T e0.
#pragma once

namespace icg {

constexpr double MARG_EPS = 1e-8;  // MarginalizationInfo::EPS (marginalization_info.h:256)
__global__ void marg_prepare(BaDev D, MargDev M, int n, int restore) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n) return;
    WinDims &d = D.dims[w];
    int *f = M.flags + 4 * w;
    if (!restore) {
        f[0] = d.reproj_huber, f[1] = d.ext_const, f[2] = d.td_const;
        d.reproj_huber = 0, d.ext_const = 0, d.td_const = 0;  // ResidualBlockInfo asks for every Jacobian and has no loss function
        LmState &st = D.st[w];
        f[3] = st.done;
        st.done = 0, st.need_lin = 1;
    } else {
        d.reproj_huber = f[0], d.ext_const = f[1], d.td_const = f[2];
        D.st[w].done = f[3], D.st[w].need_lin = 0;
    }
}

// The structure of icg_ba_marginalize_built, one CTA per window: the factor set gvinsMarginalization builds from the culling (IG/ic_gvins.cc:
// 1558-1609) into a.fmask, and updateParameterBlocksIndex's column map (marginalization_info.h:228-251) into M.map, from the slot table, the
// built lists and the culling's flags -- the rules of the host loops of icg_ba_marginalize_resident_culled and marginalize_body (ba_keyframe.cu):
//   a landmark is bad when lm_outlier is set or an outlier observation lies in its reference node; an outlier observation drops its factor;
//   a factor of a bad landmark or observed at a node out of the map drops; every other factor is in the set (the chi-square activity plays
//   no part).  Touched: the landmark, observing and reference node of every factor in the set with f_ref < num_marg, OR the camera side's
//   flags the host staged.  Columns [pose_k, mix_k (k < num_marg), touched landmarks ascending | pose_k, mix_k (k >= num_marg), ext, td].
// An observation whose factor is outside [-1, F) or is not a factor of its landmark and node is counted in out[3] (the host then rejects
// the call).  lm_col serves as the landmark flags first: 1 bad, 2 touched (a touched landmark is never bad: its factors are in the set).
__global__ void __launch_bounds__(MARG_SEL_THREADS) marg_select_built(BaCaps C, BaDev D, MargDev M, MargSelArgs a) {
    __shared__ int s_tp[BA_MAX_NODES], s_tm[BA_MAX_NODES], s_warp[MARG_SEL_THREADS / 32], s_bad, s_vis, s_base;
    const int w = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const WinDims dm = D.dims[w];
    const MargSelWin &W = a.win[w];
    const int K = dm.K, L = dm.L, F = dm.F, nm = W.num_marg;
    int *map = M.map + (size_t) w * M.map_stride;
    int *pose_col = map + MARG_MAP_HDR, *mix_col = pose_col + C.K, *lm_col = mix_col + C.K;
    uint8_t *mask = a.fmask + (size_t) w * C.F;
    int *ftab = a.ftab + (size_t) w * C.F;
    const int4 *meta = (const int4 *) D.f_meta_s + (size_t) w * C.F;  // (landmark, reference node, observing node, factor id) per slot
    const int *off = a.off + W.off0;
    for (int f = tid; f < F; f += blockDim.x) mask[f] = 1;
    for (int q = tid; q < F; q += blockDim.x) {
        const int4 mt = meta[q];
        ftab[mt.w] = mt.x * BA_MAX_NODES + mt.z;
    }
    for (int l = tid; l < C.L; l += blockDim.x) lm_col[l] = l < L && a.lm_outlier[W.lm0 + l] ? 1 : 0;
    for (int k = tid; k < BA_MAX_NODES; k += blockDim.x) s_tp[k] = k < K && W.tp[k], s_tm[k] = k < K && W.tm[k];
    if (tid == 0) s_bad = 0, s_vis = 0;
    __syncthreads();
    // the observations, landmark by landmark (a thread owns its landmark's flag and the factors of its observations)
    for (int l = tid; l < L; l += blockDim.x) {
        const int ref = a.ref[W.lm0 + l], ob = W.obs0 + off[l], oe = W.obs0 + off[l + 1];
        int bad = 0, invalid = 0;
        for (int o = ob; o < oe; o++) {
            const int f = a.fac[o], k = a.node[o];
            if (f < -1 || f >= F || (f >= 0 && ftab[f] != l * BA_MAX_NODES + k)) {
                invalid++;
                continue;
            }
            if (!a.obs_outlier[o]) continue;
            if (k == ref) bad = 1;
            if (f >= 0) mask[f] = 0;
        }
        if (bad) lm_col[l] = 1;
        if (invalid) atomicAdd(&s_bad, invalid);
    }
    __syncthreads();
    for (int q = tid; q < F; q += blockDim.x) {
        const int4 mt = meta[q];
        if (lm_col[mt.x] == 1 || !W.in_map[mt.z]) mask[mt.w] = 0;
    }
    __syncthreads();
    // touched blocks (every writer of an entry stores the same value)
    for (int q = tid; q < F; q += blockDim.x) {
        const int4 mt = meta[q];
        if (!mask[mt.w] || mt.y >= nm) continue;
        lm_col[mt.x] = 2, s_tp[mt.z] = 1, s_tp[mt.y] = 1, s_vis = 1;
    }
    __syncthreads();
    if (tid == 0) {
        int idx = 0;
        for (int k = 0; k < nm; k++) {
            if (s_tp[k]) idx += 6;
            if (s_tm[k]) idx += 9;
        }
        s_base = idx;
    }
    __syncthreads();
    // landmark columns: an exclusive prefix count of the touched landmarks in ascending id, chunk by chunk
    for (int l0 = 0; l0 < C.L; l0 += blockDim.x) {
        const int l = l0 + tid;
        const int t = l < L && lm_col[l] == 2;
        int incl = t;
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        int before = s_base;
        for (int v = 0; v < warp; v++) before += s_warp[v];
        if (l < C.L) lm_col[l] = t ? before + incl - 1 : -1;
        __syncthreads();
        if (tid == blockDim.x - 1) s_base = before + incl;
        __syncthreads();
    }
    if (tid != 0) return;
    int idx = 0;
    for (int k = 0; k < C.K; k++) pose_col[k] = mix_col[k] = -1;
    for (int k = 0; k < nm; k++) {
        if (s_tp[k]) pose_col[k] = idx, idx += 6;
        if (s_tm[k]) mix_col[k] = idx, idx += 9;
    }
    idx = s_base;
    const int m = idx;
    int *out = a.out + (size_t) w * (MARG_SEL_HDR + 2 * C.K), *blk = out + MARG_SEL_HDR;
    int nb = 0;
    for (int k = nm; k < K; k++) {
        if (s_tp[k]) pose_col[k] = idx, idx += 6, blk[nb++] = 0 | (k - nm) << 2;
        if (s_tm[k]) mix_col[k] = idx, idx += 9, blk[nb++] = 1 | (k - nm) << 2;
    }
    int ext_col = -1, td_col = -1;
    if (W.ext || s_vis) ext_col = idx, idx += 6, blk[nb++] = 2;
    if (W.td || s_vis) td_col = idx, idx += 1, blk[nb++] = 3;
    // a reprojection factor always carries ext and td columns; give them (unused) columns when only camera factors exist
    if (ext_col < 0) ext_col = 0;
    if (td_col < 0) td_col = 0;
    map[0] = m, map[1] = idx - m, map[2] = idx, map[3] = nm, map[4] = ext_col, map[5] = td_col, map[6] = map[7] = 0;
    out[0] = m, out[1] = idx - m, out[2] = nb, out[3] = s_bad, out[4] = out[5] = out[6] = out[7] = 0;
}

// H0, b0 of constructEquation.  One CTA per window; every stage has one writer per entry, stages are separated by barriers.
__global__ void __launch_bounds__(256) marg_assemble(BaCaps C, BaDev D, MargDev M) {
    extern __shared__ double smem[];
    const int w = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const WinDims dm = D.dims[w];
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], n0 = map[2], nm = map[3], ext_col = map[4], td_col = map[5];
    if (m <= 0) return;
    const int *pose_col = map + MARG_MAP_HDR, *mix_col = pose_col + C.K, *lm_col = mix_col + C.K;
    double *H0 = M.H0 + (size_t) w * M.n0cap * M.n0cap, *b0 = M.b0 + (size_t) w * M.n0cap;
    const double *pose = D.pose + (size_t) w * C.K * 7, *mix = D.mix + (size_t) w * C.K * 9, *ext = D.ext + (size_t) w * 8;
    const int K = dm.K, NCV = 6 * K + 7;
    for (int e = tid; e < n0 * n0; e += blockDim.x) H0[e] = 0;
    for (int e = tid; e < n0; e += blockDim.x) b0[e] = 0;
    double *s_imu = smem;            // 480 per warp slot (8 slots)
    double *s_dx = s_imu + 8 * 480;  // R
    double *s_y = s_dx + C.R;        // R
    int *s_cm = (int *) (s_y + C.R); // R
    __syncthreads();
    // ---- previous prior (MarginalizationFactor, marginalization_factor.h:47-101): J = J0, e = e0 + J0 dx
    if (dm.marg_r > 0) {
        const int r = dm.marg_r;
        if (tid == 0) {
            const int *type = D.marg_type + (size_t) w * BA_MARG_MAXB, *node = D.marg_node + (size_t) w * BA_MARG_MAXB;
            const double *x0 = D.marg_x0 + (size_t) w * BA_MARG_MAXB * 9;
            int col = 0, xo = 0;
            for (int b = 0; b < dm.marg_nb; b++) {
                const int t = type[b], nd = node[b];
                if (t == 0 || t == 2) {
                    const double *x = t == 0 ? pose + nd * 7 : ext, *xl = x0 + xo;
                    Q dq = qmul(qinv(pose_q(xl)), pose_q(x));
                    V3 a = 2.0 * qv(dq);
                    if (dq.w < 0) a = -a;
                    for (int k = 0; k < 3; k++) s_dx[col + k] = x[k] - xl[k];
                    s_dx[col + 3] = a.x, s_dx[col + 4] = a.y, s_dx[col + 5] = a.z;
                    const int base = t == 0 ? pose_col[nd] : ext_col;
                    for (int k = 0; k < 6; k++) s_cm[col + k] = base + k;
                    col += 6, xo += 7;
                } else if (t == 1) {
                    for (int k = 0; k < 9; k++) s_dx[col + k] = mix[nd * 9 + k] - x0[xo + k], s_cm[col + k] = mix_col[nd] + k;
                    col += 9, xo += 9;
                } else {
                    s_dx[col] = ext[7] - x0[xo], s_cm[col] = td_col;
                    col += 1, xo += 1;
                }
            }
        }
        __syncthreads();
        const double *Hq = D.marg_H0 + (size_t) w * C.R * C.R, *bq = D.marg_b0 + (size_t) w * C.R;
        for (int i = tid; i < r; i += blockDim.x) {
            double s = 0;
            for (int k = 0; k < r; k++) s += Hq[(size_t) i * r + k] * s_dx[k];
            s_y[i] = s;
        }
        __syncthreads();
        for (int e = tid; e < r * r; e += blockDim.x) {
            const int i = e / r, j = e - i * r;
            H0[(size_t) s_cm[i] * n0 + s_cm[j]] = Hq[e];
        }
        for (int i = tid; i < r; i += blockDim.x) b0[s_cm[i]] = -(bq[i] + s_y[i]);  // b = -J^T e = -(J0^T e0 + J0^T J0 dx)
        __syncthreads();
    }
    // ---- preintegration factors k < num_marg (ic_gvins.cc:1520-1538), one at a time (they share node k+1 / k)
    for (int k = 0; k < nm && k < dm.n_imu; k++) {
        double *rw = s_imu, *Jw = s_imu + 30;
        if (warp == 0)
            imu_factor_warp(D.imu_blob + ((size_t) w * C.K + k) * ICG_IMU_BLOB_DOUBLES, D.imu_U + ((size_t) w * C.K + k) * 225, pose + k * 7, mix + k * 9,
                            pose + (k + 1) * 7, mix + (k + 1) * 9, true, rw, Jw, lane);
        __syncthreads();
        auto gcol = [&](int c) { return c < 6 ? pose_col[k] + c : c < 15 ? mix_col[k] + c - 6 : c < 21 ? pose_col[k + 1] + c - 15 : mix_col[k + 1] + c - 21; };
        for (int e = tid; e < 930; e += blockDim.x) {
            if (e < 900) {
                const int a = e / 30, b = e - a * 30;
                double s = 0;
                for (int q = 0; q < 15; q++) s += Jw[q * 30 + a] * Jw[q * 30 + b];
                H0[(size_t) gcol(a) * n0 + gcol(b)] += s;
            } else {
                const int a = e - 900;
                double s = 0;
                for (int q = 0; q < 15; q++) s += Jw[q * 30 + a] * rw[q];
                b0[gcol(a)] -= s;
            }
        }
        __syncthreads();
    }
    // ---- GNSS at the removed nodes (:1505-1516), first-window priors (:1542-1554): pose / mix diagonal blocks, thread per entry
    for (int e = tid; e < nm * 42; e += blockDim.x) {
        const int k = e / 42, q = e % 42;
        if (k >= K || pose_col[k] < 0) continue;  // a removed node no factor touches has no columns
        double s = 0;
        const int a = q < 36 ? q / 6 : q - 36, b = q % 6;
        for (int g = 0; g < dm.n_gnss; g++) {
            if (D.gnss_node[(size_t) w * C.G + g] != k) continue;
            double r3[3], J[18];
            gnss_eval(pose + k * 7, D.gnss_blh + ((size_t) w * C.G + g) * 3, D.gnss_std + ((size_t) w * C.G + g) * 3, D.lever + (size_t) w * 3, true, r3, J);
            if (q < 36)
                s += J[a] * J[b] + J[6 + a] * J[6 + b] + J[12 + a] * J[12 + b];
            else
                s += J[a] * r3[0] + J[6 + a] * r3[1] + J[12 + a] * r3[2];
        }
        if (k == 0 && dm.has_pose_prior) {
            double r6[6], J[36];
            pose_prior_eval(pose, D.pose_prior + (size_t) w * 7, D.pose_prior_sinfo + (size_t) w * 6, true, r6, J);
            for (int q6 = 0; q6 < 6; q6++) s += q < 36 ? J[q6 * 6 + a] * J[q6 * 6 + b] : J[q6 * 6 + a] * r6[q6];
        }
        if (q < 36)
            H0[(size_t) (pose_col[k] + a) * n0 + pose_col[k] + b] += s;
        else
            b0[pose_col[k] + a] -= s;
    }
    if (tid < 9 && dm.has_mix_prior) {  // ImuMixPriorFactor (imu_mix_prior_factor.h:40-75): r = (mix - prior) / std
        const double sd = D.mix_prior_std[(size_t) w * 9 + tid];
        H0[(size_t) (mix_col[0] + tid) * n0 + mix_col[0] + tid] += 1.0 / (sd * sd);
        b0[mix_col[0] + tid] -= (mix[tid] - D.mix_prior[(size_t) w * 9 + tid]) / (sd * sd);
    }
    __syncthreads();
    // ---- reprojection factors of the landmarks anchored in the removed nodes (:1559-1611): camera-side part from the per-pair
    //      Gram matrices (columns [ref 6 | obs 6 | ext 6 | td | residual]); pairs in sequence, thread per entry
    {
        const int PM = C.K * (C.K - 1), P = D.npairs[w];
        const int *pro = D.pair_ro + (size_t) w * PM;
        const double *Mp = lin_Mp(C, D, D.st[w].lin_buf, w);
        int la = 0, lb = 0;
        if (tid < 210) {
            int e = tid;
            while (e >= 20 - la) e -= 20 - la, la++;
            lb = la + e;
        }
        for (int p = 0; p < P; p++) {
            const int ref = pro[p] >> 8, obs = pro[p] & 255;
            // uniform over the CTA.  A node without columns has no marginalized factor, so the pair's Gram matrix is zero: a pair whose
            // factors were all left out of the factor set (culled landmarks, a keyframe gone from the map) adds nothing and is skipped
            if (ref >= nm || pose_col[ref] < 0 || pose_col[obs] < 0) continue;
            if (tid < 210) {
                auto gcol = [&](int c) { return c < 6 ? pose_col[ref] + c : c < 12 ? pose_col[obs] + c - 6 : c < 18 ? ext_col + c - 12 : td_col; };
                const double v = Mp[(size_t) p * 210 + tid];
                if (lb < 19) {
                    const int ca = gcol(la), cb = gcol(lb);
                    H0[(size_t) ca * n0 + cb] += v;
                    if (ca != cb) H0[(size_t) cb * n0 + ca] += v;
                } else if (la < 19) {
                    b0[gcol(la)] -= v;
                }
            }
            __syncthreads();
        }
    }
    // ---- landmark rows: h_l on the diagonal, coupling row w_l, g_l  (thread per (landmark, vision column))
    const int buf = D.st[w].lin_buf;  // the linearisation ba_lin_vis just made at x
    const double *AW = lin_AW(C, D, buf, w), *hl = lin_hl(C, D, buf, w);
    for (int e = tid; e < dm.L * (NCV + 1); e += blockDim.x) {
        const int l = e / (NCV + 1), c = e - l * (NCV + 1);
        const int cl = lm_col[l];
        if (cl < 0) continue;
        const double v = AW[(size_t) l * C.NCA + c];
        if (c == NCV) {
            H0[(size_t) cl * n0 + cl] = hl[l];
            b0[cl] = -v;
        } else {
            const int mc = c < 6 * K ? (pose_col[c / 6] < 0 ? -1 : pose_col[c / 6] + c % 6) : c < 6 * K + 6 ? ext_col + c - 6 * K : td_col;
            if (mc >= 0) H0[(size_t) cl * n0 + mc] = v, H0[(size_t) mc * n0 + cl] = v;
        }
    }
}

// Plane rotation that orthogonalises two columns with squared norms al, be and inner product ga (one-sided Jacobi / Hestenes):
// tan(2 theta) = 2 ga / (be - al), smaller root.  Returns false (c, s untouched) when the pair is orthogonal to rounding level,
// |ga| <= 1e-15 sqrt(al be) (tested squared: no square root).  The scalar chain sits on the critical path of every round-robin step and
// every lane of the warp executes it, so it is written with reciprocals and one rsqrt (a general FP64 divide or sqrt is a 20-30
// instruction sequence on this part): 2 reciprocals, 1 sqrt, 1 rsqrt instead of 3 divisions and 3 square roots.
__device__ __forceinline__ bool jacobi_rotation(double al, double be, double ga, double &c, double &s) {
    if (ga == 0.0 || ga * ga <= 1e-30 * (al * be)) return false;
    const double zeta = (be - al) * (0.5 / ga);
    if (!(fabs(zeta) < 1e300)) return false;  // denormal inner product: nothing to rotate
    const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    c = rsqrt(1.0 + t * t), s = c * t;
    return true;
}

// One-sided Jacobi eigensolver of a symmetric n x n block (rows/cols [off, off+n) of src, leading dimension lds; the block is
// symmetrised as 0.5 (A + A^T) like schurElimination does).  G (= A V) and V are column-major n x n in global memory (L2).
// One warp per column pair, round-robin (circle) ordering: the n/2 pairs of a step are disjoint, a barrier separates steps.
__global__ void __launch_bounds__(MARG_THREADS) marg_jacobi(MargDev M, int which) {
    __shared__ int s_rot[2];
    const int w = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = MARG_THREADS / 32;
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], r = map[1], n0 = map[2];
    if (m <= 0) return;
    const int n = which == 0 ? m : r;
    const double *src = which == 0 ? M.H0 + (size_t) w * M.n0cap * M.n0cap : M.Hp + (size_t) w * M.rcap * M.rcap;
    const int lds = which == 0 ? n0 : r;
    double *G = which == 0 ? M.G1 + (size_t) w * M.mcap * M.mcap : M.G2 + (size_t) w * M.rcap * M.rcap;
    double *V = which == 0 ? M.V1 + (size_t) w * M.mcap * M.mcap : M.V2 + (size_t) w * M.rcap * M.rcap;
    double *lam = which == 0 ? M.lam1 + (size_t) w * M.mcap : M.lam2 + (size_t) w * M.rcap;
    for (int e = tid; e < n * n; e += MARG_THREADS) {
        const int j = e / n, i = e - j * n;  // column j, row i
        G[e] = 0.5 * (src[(size_t) i * lds + j] + src[(size_t) j * lds + i]);
        V[e] = i == j ? 1.0 : 0.0;
    }
    if (tid < 2) s_rot[tid] = 0;
    __syncthreads();
    const int ne = (n + 1) & ~1, half = ne / 2;
    constexpr int RPL = 16;  // rows per lane held in registers: n <= 512
    for (int sweep = 0; sweep < 40; sweep++) {
        for (int step = 0; step < ne - 1; step++) {
            for (int i = warp; i < half; i += nwarps) {
                int p = i == 0 ? ne - 1 : (step + i) % (ne - 1);
                int q = (step + ne - 1 - i) % (ne - 1);
                if (p >= n || q >= n) continue;
                if (p > q) {
                    const int t = p;
                    p = q, q = t;
                }
                double *gp = G + (size_t) p * n, *gq = G + (size_t) q * n, *vp = V + (size_t) p * n, *vq = V + (size_t) q * n;
                double a[RPL], b[RPL];
                double al = 0, be = 0, ga = 0, c, s;
#pragma unroll
                for (int k = 0; k < RPL; k++) {
                    const int row = lane + 32 * k;
                    a[k] = row < n ? gp[row] : 0.0;
                    b[k] = row < n ? gq[row] : 0.0;
                    al += a[k] * a[k], be += b[k] * b[k], ga += a[k] * b[k];
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    al += __shfl_xor_sync(0xffffffffu, al, o);
                    be += __shfl_xor_sync(0xffffffffu, be, o);
                    ga += __shfl_xor_sync(0xffffffffu, ga, o);
                }
                if (!jacobi_rotation(al, be, ga, c, s)) continue;
#pragma unroll
                for (int k = 0; k < RPL; k++) {
                    const int row = lane + 32 * k;
                    if (row < n) {
                        gp[row] = c * a[k] - s * b[k];
                        gq[row] = s * a[k] + c * b[k];
                        const double x = vp[row], y = vq[row];
                        vp[row] = c * x - s * y;
                        vq[row] = s * x + c * y;
                    }
                }
                if (lane == 0) s_rot[sweep & 1] = 1;
            }
            __syncthreads();
        }
        const int any = s_rot[sweep & 1];
        __syncthreads();
        if (tid == 0) s_rot[(sweep + 1) & 1] = 0;
        __syncthreads();
        if (!any) break;
    }
    // lambda_i = v_i . (A v_i) = v_i . g_i  (signed: a negative rounding-level eigenvalue must fail the > EPS test like Eigen's)
    for (int j = warp; j < n; j += nwarps) {
        double s = 0;
        for (int row = lane; row < n; row += 32) s += V[(size_t) j * n + row] * G[(size_t) j * n + row];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) lam[j] = s;
    }
}

// The same eigensolver for blocks that fit on chip (n <= MARG_PAIR_MAXN): a CLUSTER OF TWO CTAs per window.  CTA 0 keeps G = A V (column-major,
// n^2 doubles) in its shared memory, generates the plane rotations of a round-robin step (one warp per column pair: three dot products, then
// the rotation of the pair) and writes the step's (c, s) list into CTA 1's shared memory (DSMEM stores); CTA 1 keeps V in its shared memory and
// applies the list while CTA 0 already works on the next step (two record slots, one cluster barrier per step).  No L2 round trip sits on
// the rotation loop any more (the global-memory kernel above pays two per rotation); same rotation formula, ordering and stopping rule, so
// the decomposition is the same up to rounding.  lambda_i = v_i . g_i is formed by CTA 1 reading G over DSMEM once at the end.
__global__ void __launch_bounds__(MARG_THREADS) marg_jacobi_pair(MargDev M, int which) {
    extern __shared__ double sm_mat[];  // CTA 0: G; CTA 1: V   (n x n, column-major), then the two rotation-record slots (CTA 1)
    cg::cluster_group cluster = cg::this_cluster();
    const int cr = (int) cluster.block_rank();
    const int w = blockIdx.x / 2, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = MARG_THREADS / 32;
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], r = map[1], n0 = map[2];
    if (m <= 0) return;  // uniform over the cluster
    const int n = which == 0 ? m : r;
    const double *src = which == 0 ? M.H0 + (size_t) w * M.n0cap * M.n0cap : M.Hp + (size_t) w * M.rcap * M.rcap;
    const int lds = which == 0 ? n0 : r;
    double *Vout = which == 0 ? M.V1 + (size_t) w * M.mcap * M.mcap : M.V2 + (size_t) w * M.rcap * M.rcap;
    double *lam = which == 0 ? M.lam1 + (size_t) w * M.mcap : M.lam2 + (size_t) w * M.rcap;
    const int ne = (n + 1) & ~1, half = ne / 2;
    double *mat = sm_mat;
    double *rec = sm_mat + (size_t) n * n;  // [2][half][2] (c, s); c = 2 marks "no rotation"
    __shared__ int s_any[2];
    if (cr == 0) {
        for (int e = tid; e < n * n; e += MARG_THREADS) {
            const int j = e / n, i = e - j * n;
            mat[e] = 0.5 * (src[(size_t) i * lds + j] + src[(size_t) j * lds + i]);
        }
    } else {
        for (int e = tid; e < n * n; e += MARG_THREADS) mat[e] = (e / n) == (e % n) ? 1.0 : 0.0;
    }
    if (tid < 2) s_any[tid] = 0;
    // CTA 0 addresses the record slots and the "any rotation" word of CTA 1
    double *rec_remote = cluster.map_shared_rank(rec, 1);
    int *any_remote = cluster.map_shared_rank(s_any, 1);
    cluster.sync();
    constexpr int RPL = 5;  // rows per lane: n <= 160
    int pending = -1, pending_slot = 0;  // step (and record slot) CTA 1 still has to apply
    int gstep = 0;                       // steps executed so far over all sweeps: the record slots alternate on it (ne - 1 is odd)
    bool stop = false;
    for (int sweep = 0; sweep < 40 && !stop; sweep++) {
        for (int step = 0; step < ne - 1; step++, gstep++) {
            const int slot = gstep & 1;
            if (cr == 0) {
                for (int i = warp; i < half; i += nwarps) {
                    int p = i == 0 ? ne - 1 : (step + i) % (ne - 1);
                    int q = (step + ne - 1 - i) % (ne - 1);
                    double c = 2.0, sn = 0.0;
                    if (p < n && q < n) {
                        if (p > q) {
                            const int t = p;
                            p = q, q = t;
                        }
                        double *gp = mat + (size_t) p * n, *gq = mat + (size_t) q * n;
                        double a[RPL], b[RPL], al = 0, be = 0, ga = 0;
#pragma unroll
                        for (int k = 0; k < RPL; k++) {
                            const int row = lane + 32 * k;
                            a[k] = row < n ? gp[row] : 0.0;
                            b[k] = row < n ? gq[row] : 0.0;
                            al += a[k] * a[k], be += b[k] * b[k], ga += a[k] * b[k];
                        }
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) {
                            al += __shfl_xor_sync(0xffffffffu, al, o);
                            be += __shfl_xor_sync(0xffffffffu, be, o);
                            ga += __shfl_xor_sync(0xffffffffu, ga, o);
                        }
                        if (jacobi_rotation(al, be, ga, c, sn)) {
#pragma unroll
                            for (int k = 0; k < RPL; k++) {
                                const int row = lane + 32 * k;
                                if (row < n) {
                                    gp[row] = c * a[k] - sn * b[k];
                                    gq[row] = sn * a[k] + c * b[k];
                                }
                            }
                        }
                    }
                    if (lane == 0) {
                        rec_remote[((size_t) slot * half + i) * 2] = c, rec_remote[((size_t) slot * half + i) * 2 + 1] = sn;
                        if (c != 2.0) any_remote[sweep & 1] = 1;
                    }
                }
            } else if (pending >= 0) {
                // apply the previous step's rotations to V (its record was completed before the last cluster barrier)
                const int pstep = pending, pslot = pending_slot;
                for (int i = warp; i < half; i += nwarps) {
                    const double c = rec[((size_t) pslot * half + i) * 2], sn = rec[((size_t) pslot * half + i) * 2 + 1];
                    if (c == 2.0) continue;
                    int p = i == 0 ? ne - 1 : (pstep + i) % (ne - 1);
                    int q = (pstep + ne - 1 - i) % (ne - 1);
                    if (p > q) {
                        const int t = p;
                        p = q, q = t;
                    }
                    double *vp = mat + (size_t) p * n, *vq = mat + (size_t) q * n;
#pragma unroll
                    for (int k = 0; k < RPL; k++) {
                        const int row = lane + 32 * k;
                        if (row < n) {
                            const double x = vp[row], y = vq[row];
                            vp[row] = c * x - sn * y;
                            vq[row] = sn * x + c * y;
                        }
                    }
                }
            }
            cluster.sync();  // record of `step` complete and visible in CTA 1; CTA 1 done with the slot CTA 0 writes next
            pending = step, pending_slot = slot;
        }
        // end of sweep: both CTAs read the same flag (it lives in CTA 1; CTA 0 reads it over DSMEM)
        const int any = cr == 0 ? *((volatile int *) any_remote + (sweep & 1)) : *((volatile int *) s_any + (sweep & 1));
        cluster.sync();
        if (cr == 1 && tid == 0) s_any[(sweep + 1) & 1] = 0;
        cluster.sync();
        if (!any) stop = true;
    }
    // flush: the record of the last executed step has not been applied yet
    if (cr == 1 && pending >= 0) {
        const int pstep = pending, pslot = pending_slot;
        for (int i = warp; i < half; i += nwarps) {
            const double c = rec[((size_t) pslot * half + i) * 2], sn = rec[((size_t) pslot * half + i) * 2 + 1];
            if (c == 2.0) continue;
            int p = i == 0 ? ne - 1 : (pstep + i) % (ne - 1);
            int q = (pstep + ne - 1 - i) % (ne - 1);
            if (p > q) {
                const int t = p;
                p = q, q = t;
            }
            double *vp = mat + (size_t) p * n, *vq = mat + (size_t) q * n;
            for (int row = lane; row < n; row += 32) {
                const double x = vp[row], y = vq[row];
                vp[row] = c * x - sn * y;
                vq[row] = sn * x + c * y;
            }
        }
    }
    __syncthreads();
    // ---- results (CTA 1): V to global (column-major n x n), lambda_j = v_j . g_j with g_j read from CTA 0 over DSMEM
    const double *G_remote = cluster.map_shared_rank(sm_mat, 0);
    if (cr == 1) {
        for (int e = tid; e < n * n; e += MARG_THREADS) Vout[e] = mat[e];
        for (int j = warp; j < n; j += nwarps) {
            double s2 = 0;
            for (int row = lane; row < n; row += 32) s2 += mat[(size_t) j * n + row] * G_remote[(size_t) j * n + row];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            if (lane == 0) lam[j] = s2;
        }
    }
    cluster.sync();  // CTA 0's shared memory must stay alive until CTA 1 has read G
}

// The same eigensolver for the sizes the sliding window actually produces (n <= MARG_CTA_MAXN: marginalising one keyframe of a 10-frame window
// gives m = 15 + its landmarks and r <= 70): ONE CTA per window with G = A V and V both in shared memory, eight lanes per column pair (four pairs
// per warp share the warp-wide scalar chain; all n/2 pairs of a round-robin step run in one round), one block barrier per step.  Against the
// cluster-pair kernel: no cluster barrier on the step, and the grid needs half the CTAs.
__global__ void __launch_bounds__(MARG_CTA_THREADS) marg_jacobi_cta(MargDev M, int which) {
    extern __shared__ double sm_mat[];  // G | V (n x n each, column-major)
    __shared__ int s_any[2];
    const int w = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, sub = lane >> 3, sl = lane & 7;
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], r = map[1], n0 = map[2];
    if (m <= 0) return;
    const int n = which == 0 ? m : r;
    const double *src = which == 0 ? M.H0 + (size_t) w * M.n0cap * M.n0cap : M.Hp + (size_t) w * M.rcap * M.rcap;
    const int lds = which == 0 ? n0 : r;
    double *Vout = which == 0 ? M.V1 + (size_t) w * M.mcap * M.mcap : M.V2 + (size_t) w * M.rcap * M.rcap;
    double *lam = which == 0 ? M.lam1 + (size_t) w * M.mcap : M.lam2 + (size_t) w * M.rcap;
    double *G = sm_mat, *V = sm_mat + (size_t) n * n;
    for (int e = tid; e < n * n; e += MARG_CTA_THREADS) {
        const int j = e / n, i = e - j * n;
        G[e] = 0.5 * (src[(size_t) i * lds + j] + src[(size_t) j * lds + i]);
        V[e] = i == j ? 1.0 : 0.0;
    }
    if (tid < 2) s_any[tid] = 0;
    __syncthreads();
    const int ne = (n + 1) & ~1, half = ne / 2;
    const int i = warp * 4 + sub;                 // pair slot of this eight-lane group
    const unsigned gmask = 0xFFu << (8 * sub);
    constexpr int RPL = 15;                       // rows per lane: n <= 120
    for (int sweep = 0; sweep < 40; sweep++) {
        for (int step = 0; step < ne - 1; step++) {
            if (i < half) {
                int p = i == 0 ? ne - 1 : (step + i) % (ne - 1);
                int q = (step + ne - 1 - i) % (ne - 1);
                if (p < n && q < n) {
                    if (p > q) {
                        const int t = p;
                        p = q, q = t;
                    }
                    double *gp = G + (size_t) p * n, *gq = G + (size_t) q * n;
                    double a[RPL], b[RPL], al = 0, be = 0, ga = 0, c, s;
#pragma unroll
                    for (int k = 0; k < RPL; k++) {
                        const int row = sl + 8 * k;
                        a[k] = row < n ? gp[row] : 0.0;
                        b[k] = row < n ? gq[row] : 0.0;
                        al += a[k] * a[k], be += b[k] * b[k], ga += a[k] * b[k];
                    }
#pragma unroll
                    for (int o = 4; o > 0; o >>= 1) {
                        al += __shfl_xor_sync(gmask, al, o);
                        be += __shfl_xor_sync(gmask, be, o);
                        ga += __shfl_xor_sync(gmask, ga, o);
                    }
                    if (jacobi_rotation(al, be, ga, c, s)) {
                        double *vp = V + (size_t) p * n, *vq = V + (size_t) q * n;
#pragma unroll
                        for (int k = 0; k < RPL; k++) {
                            const int row = sl + 8 * k;
                            if (row < n) {
                                gp[row] = c * a[k] - s * b[k];
                                gq[row] = s * a[k] + c * b[k];
                                const double x = vp[row], y = vq[row];
                                vp[row] = c * x - s * y;
                                vq[row] = s * x + c * y;
                            }
                        }
                        if (sl == 0) s_any[sweep & 1] = 1;
                    }
                }
            }
            __syncthreads();
        }
        const int any = s_any[sweep & 1];
        __syncthreads();
        if (tid == 0) s_any[(sweep + 1) & 1] = 0;
        __syncthreads();
        if (!any) break;
    }
    for (int e = tid; e < n * n; e += MARG_CTA_THREADS) Vout[e] = V[e];
    for (int j = warp; j < n; j += MARG_CTA_THREADS / 32) {
        double s2 = 0;
        for (int row = lane; row < n; row += 32) s2 += V[(size_t) j * n + row] * G[(size_t) j * n + row];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        if (lane == 0) lam[j] = s2;
    }
}

// The same eigensolver for MARG_PAIR_MAXN < n <= MARG_CLUSTER_MAXN (a cfg-4 window's remained block, r = 15 * 19 + 7 = 292): a CLUSTER OF
// EIGHT CTAs per window, G and V distributed over their shared memory by rows.  CTA k holds rows [k R8, (k + 1) R8), R8 = ceil(n / 8) <= 40,
// of every column of G and of V (column-major inside the slice): 2 * 40 * 320 doubles = 204.8 KB at n = 320, plus the partial-sum slots.
// A round-robin step:
//   1. four lanes per column pair form the pair's three partial dot products (al, be, ga) over the CTA's rows, into a local slot;
//   2. one cluster barrier;
//   3. every CTA reads the eight CTAs' slots over DSMEM and sums them in rank order 0..7, so every CTA gets the same (al, be, ga), the same
//      rotation and the same "any rotation this sweep" decision (the sweep loop exits uniformly with no broadcast);
//   4. every CTA rotates its own rows of G and V; a block barrier separates them from the next step's partials.
// The slots are double-buffered by step parity: a slot is rewritten two steps later, after every CTA has passed the barrier that follows its
// reads, so one cluster barrier per step is enough.  lambda_j = v_j . g_j is summed from rank-ordered per-CTA partials.
__global__ void __launch_bounds__(MARG_CLUSTER_THREADS) marg_jacobi_cluster(MargDev M, int which) {
    extern __shared__ double sm_mat[];  // G slice | V slice (n columns of R8 rows each) | partial slots [2][MARG_CLUSTER_SLOT]
    __shared__ int s_any[2];
    cg::cluster_group cluster = cg::this_cluster();
    const int cr = (int) cluster.block_rank();
    const int w = blockIdx.x / MARG_CLUSTER_CTAS, tid = threadIdx.x, lane = tid & 31, sl = lane & 3;
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], r = map[1], n0 = map[2];
    if (m <= 0) return;  // uniform over the cluster
    const int n = which == 0 ? m : r;
    const double *src = which == 0 ? M.H0 + (size_t) w * M.n0cap * M.n0cap : M.Hp + (size_t) w * M.rcap * M.rcap;
    const int lds = which == 0 ? n0 : r;
    double *Vout = which == 0 ? M.V1 + (size_t) w * M.mcap * M.mcap : M.V2 + (size_t) w * M.rcap * M.rcap;
    double *lam = which == 0 ? M.lam1 + (size_t) w * M.mcap : M.lam2 + (size_t) w * M.rcap;
    const int R8 = marg_cluster_rows(n), r0 = cr * R8;
    double *G = sm_mat, *V = sm_mat + (size_t) R8 * n, *slot = V + (size_t) R8 * n;
    for (int e = tid; e < R8 * n; e += MARG_CLUSTER_THREADS) {
        const int j = e / R8, i = r0 + (e - j * R8);  // column j, row i (rows past n are zero: they add nothing to any sum)
        G[e] = i < n ? 0.5 * (src[(size_t) i * lds + j] + src[(size_t) j * lds + i]) : 0.0;
        V[e] = i == j ? 1.0 : 0.0;
    }
    if (tid < 2) s_any[tid] = 0;
    // this lane's two remote slots in the rank-ordered sum: ranks 2 sl and 2 sl + 1
    const double *slot_a = cluster.map_shared_rank(slot, 2 * sl), *slot_b = cluster.map_shared_rank(slot, 2 * sl + 1);
    cluster.sync();
    const int ne = (n + 1) & ~1, half = ne / 2;
    const int i = tid >> 2;                                  // pair slot of this four-lane group
    const unsigned gmask = 0xFu << (lane & ~3);
    constexpr int RPL = (MARG_CLUSTER_MAXN / MARG_CLUSTER_CTAS + 3) / 4;  // rows per lane: R8 <= 40
    int gstep = 0;                                           // steps over all sweeps: the slot parity (ne - 1 is odd)
    for (int sweep = 0; sweep < 40; sweep++) {
        for (int step = 0; step < ne - 1; step++, gstep++) {
            const int buf = gstep & 1;
            int p = i == 0 ? ne - 1 : (step + i) % (ne - 1);
            int q = (step + ne - 1 - i) % (ne - 1);
            const bool active = i < half && p < n && q < n;  // uniform over the four lanes
            if (p > q) {
                const int t = p;
                p = q, q = t;
            }
            double *gp = G + (size_t) p * R8, *gq = G + (size_t) q * R8;
            if (active) {
                double al = 0, be = 0, ga = 0;
#pragma unroll
                for (int k = 0; k < RPL; k++) {
                    const int row = sl + 4 * k;
                    const double a = row < R8 ? gp[row] : 0.0, b = row < R8 ? gq[row] : 0.0;
                    al += a * a, be += b * b, ga += a * b;
                }
#pragma unroll
                for (int o = 2; o > 0; o >>= 1) {
                    al += __shfl_xor_sync(gmask, al, o);
                    be += __shfl_xor_sync(gmask, be, o);
                    ga += __shfl_xor_sync(gmask, ga, o);
                }
                if (sl == 0) {
                    double *s = slot + (size_t) buf * MARG_CLUSTER_SLOT + 3 * i;
                    s[0] = al, s[1] = be, s[2] = ga;
                }
            }
            cluster.sync();  // every CTA's partials of this step are in place
            if (active) {
                const size_t o = (size_t) buf * MARG_CLUSTER_SLOT + 3 * i;
                const double xa[3] = {slot_a[o], slot_a[o + 1], slot_a[o + 2]}, xb[3] = {slot_b[o], slot_b[o + 1], slot_b[o + 2]};
                double t3[3] = {0, 0, 0};
#pragma unroll
                for (int rk = 0; rk < MARG_CLUSTER_CTAS; rk++) {
                    const int src_lane = (lane & ~3) | (rk >> 1);
#pragma unroll
                    for (int c = 0; c < 3; c++) t3[c] += __shfl_sync(gmask, (rk & 1) ? xb[c] : xa[c], src_lane);
                }
                double c, s;
                if (jacobi_rotation(t3[0], t3[1], t3[2], c, s)) {
                    double *vp = V + (size_t) p * R8, *vq = V + (size_t) q * R8;
#pragma unroll
                    for (int k = 0; k < RPL; k++) {
                        const int row = sl + 4 * k;
                        if (row < R8) {
                            const double a = gp[row], b = gq[row];
                            gp[row] = c * a - s * b;
                            gq[row] = s * a + c * b;
                            const double x = vp[row], y = vq[row];
                            vp[row] = c * x - s * y;
                            vq[row] = s * x + c * y;
                        }
                    }
                    if (sl == 0) s_any[sweep & 1] = 1;
                }
            }
            __syncthreads();  // this step's rotations land before the next step's partials read the columns
        }
        const int any = s_any[sweep & 1];  // the same value in every CTA of the cluster
        if (tid == 0) s_any[(sweep + 1) & 1] = 0;
        if (!any) break;
    }
    // ---- results: this CTA's rows of V; lambda_j from the eight CTAs' partials of v_j . g_j, summed in rank order
    for (int e = tid; e < R8 * n; e += MARG_CLUSTER_THREADS) {
        const int j = e / R8, il = e - j * R8;
        if (r0 + il < n) Vout[(size_t) j * n + r0 + il] = V[e];
    }
    cluster.sync();  // the other CTAs have read this CTA's slots of the last step: the slot area is free
    for (int j = tid; j < n; j += MARG_CLUSTER_THREADS) {
        double s = 0;
        for (int il = 0; il < R8; il++) s += V[(size_t) j * R8 + il] * G[(size_t) j * R8 + il];
        slot[j] = s;  // n <= 2 * MARG_CLUSTER_SLOT
    }
    cluster.sync();
    for (int j = cr + MARG_CLUSTER_CTAS * tid; j < n; j += MARG_CLUSTER_CTAS * MARG_CLUSTER_THREADS) {
        double s = 0;
        for (int rk = 0; rk < MARG_CLUSTER_CTAS; rk++) s += cluster.map_shared_rank(slot, rk)[j];
        lam[j] = s;
    }
    cluster.sync();  // every CTA's shared memory stays alive until the others have read its partials
}

// Hp = Hrr - Hrm Hmm^+ Hmr, bp = br - Hrm Hmm^+ bm with Hmm^+ = V diag(1/lambda > EPS) V^T  (schurElimination)
__global__ void __launch_bounds__(MARG_THREADS) marg_schur(MargDev M) {
    const int w = blockIdx.x, tid = threadIdx.x;
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], r = map[1], n0 = map[2];
    if (m <= 0) return;
    const double *H0 = M.H0 + (size_t) w * M.n0cap * M.n0cap, *b0 = M.b0 + (size_t) w * M.n0cap;
    const double *V = M.V1 + (size_t) w * M.mcap * M.mcap, *lam = M.lam1 + (size_t) w * M.mcap;
    double *Z = M.Z + (size_t) w * M.mcap * (M.rcap + 1);
    double *Hp = M.Hp + (size_t) w * M.rcap * M.rcap, *bp = M.bp + (size_t) w * M.rcap;
    const int ldz = r + 1;
    // Z[i][j] = lambda_i^-1/2 * sum_k V[k][i] * [Hmr | bm][k][j]
    for (int e = tid; e < m * ldz; e += MARG_THREADS) {
        const int i = e / ldz, j = e - i * ldz;
        double s = 0;
        if (lam[i] > MARG_EPS) {
            const double *vi = V + (size_t) i * m;
            if (j < r)
                for (int k = 0; k < m; k++) s += vi[k] * H0[(size_t) k * n0 + m + j];
            else
                for (int k = 0; k < m; k++) s += vi[k] * b0[k];
            s *= sqrt(1.0 / lam[i]);
        }
        Z[e] = s;
    }
    __syncthreads();
    for (int e = tid; e < r * ldz; e += MARG_THREADS) {
        const int a = e / ldz, b = e - a * ldz;
        double s = 0;
        for (int i = 0; i < m; i++) s += Z[(size_t) i * ldz + a] * Z[(size_t) i * ldz + b];
        if (b < r)
            Hp[(size_t) a * r + b] = H0[(size_t) (m + a) * n0 + m + b] - s;
        else
            bp[a] = b0[m + a] - s;
    }
}

// linearization: J0 = S^1/2 V^T, e0 = -S^-1/2 V^T bp, rows in ascending eigenvalue order
__global__ void __launch_bounds__(MARG_THREADS) marg_finish(MargDev M) {
    const int w = blockIdx.x, tid = threadIdx.x;
    const int *map = M.map + (size_t) w * M.map_stride;
    const int m = map[0], r = map[1];
    if (m <= 0) return;
    const double *V = M.V2 + (size_t) w * M.rcap * M.rcap, *lam = M.lam2 + (size_t) w * M.rcap, *bp = M.bp + (size_t) w * M.rcap;
    double *J0 = M.J0 + (size_t) w * M.rcap * M.rcap, *e0 = M.e0 + (size_t) w * M.rcap;
    for (int k = tid; k < r; k += MARG_THREADS) {
        int rank = 0;
        for (int j = 0; j < r; j++) rank += (lam[j] < lam[k] || (lam[j] == lam[k] && j < k)) ? 1 : 0;
        const double s = lam[k] > MARG_EPS ? lam[k] : 0.0, si = lam[k] > MARG_EPS ? 1.0 / lam[k] : 0.0;
        const double ss = sqrt(s), ssi = sqrt(si);
        double d = 0;
        for (int j = 0; j < r; j++) {
            const double v = V[(size_t) k * r + j];
            J0[(size_t) rank * r + j] = ss * v;
            d += v * -bp[j];
        }
        e0[rank] = ssi * d;
    }
}

}  // namespace icg
