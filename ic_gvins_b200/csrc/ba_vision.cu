// ba_vision.cu -- the device half of icg_ba_slide_vision_resident (ba_vision.cuh).  One CTA per window: the structure of one window is small
// (a few thousand landmarks and factors) and windows are independent, as in the slide's gather.  Built with -fmad=false: pixel2cam is a
// subtract and a divide on the host, and must stay so here.
#include <cub/block/block_scan.cuh>

#include "ba_vision.cuh"
#include "geom_core.cuh"

namespace icg {

namespace {

using Scan = cub::BlockScan<int, VIS_THREADS>;

// in-place exclusive prefix sum of a[0 .. n) by the whole CTA (each thread a contiguous chunk, one block scan of the chunk sums); returns the total
__device__ int block_exscan(int *a, int n, Scan::TempStorage &tmp) {
    const int chunk = (n + VIS_THREADS - 1) / VIS_THREADS, b = threadIdx.x * chunk, e = min(n, b + chunk);
    int s = 0;
    for (int i = b; i < e; i++) s += a[i];
    int base, total;
    Scan(tmp).ExclusiveSum(s, base, total);
    for (int i = b; i < e; i++) {
        const int v = a[i];
        a[i] = base, base += v;
    }
    __syncthreads();
    return total;
}

__device__ void fail(int *cnt, int code, int idx) {
    if (atomicCAS(cnt + 3, 0, code) == 0) cnt[4] = idx;
}

__device__ double carried_invdepth(double rho) { return __ddiv_rn(1.0, __ddiv_rn(1.0, rho)); }

__device__ void cam_point(const icg_camera &c, float u, float v, double *p) {
    gc::pixel2cam(c, u, v, p[0], p[1]);
    p[2] = 1.0;
}

// an entry of the last culling's list is kept in the next one (step 4): not flagged, in a next node, naming a carried factor or, with no
// factor, in the landmark's reference node
__device__ __forceinline__ bool listed(int f, int k, uint8_t flagged, int8_t next_node, int ref, int oF, const int *fmap) {
    if (flagged != 0 || next_node < 0) return false;
    return f >= 0 ? f < oF && fmap[f] >= 0 : f == -1 && k == ref;
}

__device__ __forceinline__ void list_entry(int *node, int *fac, float *kp, int e, int nd, int f, const float *xy) {
    node[e] = nd, fac[e] = f, kp[2 * e] = xy[0], kp[2 * e + 1] = xy[1];
}

}  // namespace

// Rules (include/icgvins_b200.h, icg_ba_slide_vision_resident): landmark l of the old window is carried when it is not a culling outlier, its
// reference node is usable (in the map, not marginalized, kept by the slide) and 1 / (1 / rho) is not NaN; its old factors survive when their
// observation is listed by the culling and not an outlier and their observing node is usable; its new observations follow in node order.  New map
// points follow the carried landmarks in creation order, each with one factor from its reference node to the current node.  On a landmark shard
// the old window is the rank's shard and only the rank's new points are kept; the numbering below is then the shard's.  The kernel then writes
// the next culling's lists (step 4, the list rule of icg_ba_update_and_cull_built).  The rule is local to each landmark, so on a shard step 4
// needs nothing else: keep covers the rank's carried landmarks and its own new points, fmap maps its old shard factors to next shard rows,
// and node indices are the replicated camera side's.
__global__ void __launch_bounds__(VIS_THREADS) ba_vision_build(VisArgs a) {
    __shared__ Scan::TempStorage tmp;
    __shared__ int s_nobs, s_nnew;
    const int w = blockIdx.x, t = threadIdx.x;
    const VisWin &W = a.win[w];
    const int oK = W.oK, oL = W.oL, oF = W.oF;
    int *cnt = a.counts + (size_t) w * VIS_COUNTS;
    const size_t wL = (size_t) w * a.L, wF = (size_t) w * a.F;
    const int *meta = a.f_meta_s + wF * 4, *off = a.lm_off + (size_t) w * (a.L + 1), *perm = a.lm_perm + wL;
    const double *rho = a.rho + wL;
    const int *ref_node = a.lm_ref_node + W.cull_lm0;
    const uint8_t *lm_out = a.lm_outlier + W.cull_lm0, *obs_out = a.obs_outlier + W.cull_obs0;
    const int *ofac = W.obs_factor;
    if (t == 0) {
        int n = W.dev_n ? *W.dev_n : W.n_obs, m = W.dev_new_n ? *W.dev_new_n : W.n_new;
        cnt[6] = n, cnt[7] = m;
        if (n < 0 || n > W.n_obs) fail(cnt, VIS_ECOUNT, n), n = 0;
        if (m < 0 || m > W.n_new) fail(cnt, VIS_ECOUNT, m), m = 0;
        s_nobs = n, s_nnew = m;
    }
    // scratch (vis_scratch_ints): fkeep (oF) | pos_of (oL) | mask (oL) | nkeep (oL) | keep, nn, lidx, fbase, nbase (oL + n_new each) | ref node
    // of each new point (n_new); with the lists: | next factor row of each old factor, -1: dropped (oF) | list entries per landmark (oL + n_new)
    const int NA = oL + W.n_new;
    int *fkeep = a.scratch + W.scr, *pos_of = fkeep + oF, *mask = pos_of + oL, *nkeep = mask + oL;
    int *keep = nkeep + oL, *nn = keep + NA, *lidx = nn + NA, *fbase = lidx + NA, *nbase = fbase + NA, *new_ref = nbase + NA;
    const double *lref = a.lm_ref + wL * 7;
    double *lref_next = a.lm_ref_next + wL * 7;
    uint8_t *lm_nan = a.lm_nan + W.lm_out;
    for (int q = t; q < oF; q += VIS_THREADS) {
        fkeep[q] = 0;
        if (a.l_off) new_ref[W.n_new + q] = -1;  // fmap, step 4
    }
    for (int p = t; p < oL; p += VIS_THREADS) pos_of[perm[p]] = p, mask[perm[p]] = 0;
    __syncthreads();
    const int nobs = s_nobs, nnew = s_nnew;
    // 1. flags: the factors the culling's observations keep, the carried landmarks, the new points' reference nodes
    for (int o = t; o < W.n_cull_obs; o += VIS_THREADS) {
        const int f = ofac[o];
        if (f < -1 || f >= oF) fail(cnt, VIS_EOBS_FACTOR, o);
        else if (f >= 0) fkeep[f] = obs_out[o] == 0;
    }
    int nan_drops = 0;
    for (int l = t; l < oL; l += VIS_THREADS) {
        const int r = ref_node[l];
        const bool nan = isnan(carried_invdepth(rho[l]));
        const bool k = lm_out[l] == 0 && r >= 0 && r < oK && W.onode[r] >= 0;
        keep[l] = k && !nan;
        lm_nan[l] = k && nan;
        nan_drops += k && nan;
    }
    for (int j = t; j < NA - oL; j += VIS_THREADS) {
        keep[oL + j] = 0, lm_nan[oL + j] = 0;
        if (j >= nnew) {
            new_ref[j] = -1;
            continue;
        }
        const int64_t id = W.new_ref_frame[j];
        int node = -1;
        for (int e = 0; e < W.n_frames; e++)
            if (W.frame_id[e] == id) node = W.frame_node[e];
        if (node < 0) fail(cnt, VIS_EFRAME, j);
        new_ref[j] = node;
        // landmark shards: new point j of window w lives on rank (j + w) mod world only (world 1: every point)
        const bool nan = isnan(__ddiv_rn(1.0, W.new_depth[j])), mine = node >= 0 && (j + w) % a.world == a.rank;
        keep[oL + j] = mine && !nan;
        lm_nan[oL + j] = mine && nan;
        nan_drops += mine && nan;
    }
    __syncthreads();
    // the new observations: one bit per (landmark, next node); a second observation of a landmark in one node is an error
    for (int k = t; k < nobs; k += VIS_THREADS) {
        const int j = W.src ? W.src[k] : k;
        if (j < 0 || j >= W.n_in) {
            fail(cnt, VIS_ESRC, k);
            continue;
        }
        const int l = W.obs_lm[j], node = W.obs_node ? W.obs_node[j] : W.cur_node;
        if (node < 0 || node >= W.nK) fail(cnt, VIS_ENODE, k);
        else if (l < -1 || l >= oL) fail(cnt, VIS_ELM, k);
        else if (l >= 0 && keep[l] && W.onode[ref_node[l]] != node && (atomicOr((unsigned *) mask + l, 1u << node) >> node) & 1u) fail(cnt, VIS_EDUP, k);
    }
    __syncthreads();
    // 2. counts per landmark (factors, new factors) and the three dense numberings
    for (int i = t; i < NA; i += VIS_THREADS) {
        int s = 0, m = 0;
        if (i < oL && keep[i]) {
            const int p = pos_of[i];
            for (int q = off[p]; q < off[p + 1]; q++) s += fkeep[meta[4 * q + 3]] && W.onode[meta[4 * q + 2]] >= 0;
            m = __popc(mask[i]);
            if (m > 0 && isnan(lref[(size_t) i * 7])) fail(cnt, VIS_EROW, i);
            nkeep[i] = s;
        } else if (i >= oL && keep[i]) {
            m = new_ref[i - oL] != W.cur_node;
        }
        nn[i] = m, lidx[i] = keep[i], fbase[i] = s + m, nbase[i] = m;
    }
    __syncthreads();
    const int L = block_exscan(lidx, NA, tmp), F = block_exscan(fbase, NA, tmp), N = block_exscan(nbase, NA, tmp);
    {
        int before;
        Scan(tmp).ExclusiveSum(nan_drops, before, nan_drops);
    }
    if (t == 0) cnt[0] = L, cnt[1] = F, cnt[2] = N, cnt[5] = nan_drops;
    // 3. the rows: carried landmarks and factors, new map points with their factor
    int *lm_src = a.lm_src + W.lm_out, *lm_org = a.lm_org + W.lm_out, *f_lm = a.f_lm + W.f_out, *f_ref = a.f_ref + W.f_out, *f_obs = a.f_obs + W.f_out, *f_src = a.f_src + W.f_out;
    double *invd = a.invdepth + W.lm_out, *fnew = a.f_new + (size_t) W.nf_out * 14;
    for (int i = t; i < NA; i += VIS_THREADS) {
        if (!keep[i]) continue;
        const int li = lidx[i];
        int fo = fbase[i];
        double *row = li < a.L ? lref_next + (size_t) li * 7 : nullptr;  // a window beyond the handle's capacity is rejected afterwards
        if (i < oL) {
            const double v = carried_invdepth(rho[i]);
            lm_src[li] = v == 0.0 ? -1 : i;  // addReprojectionFactors: 0 -> 1 / MapPoint::DEFAULT_DEPTH, staged as a new row
            lm_org[li] = i;
            invd[li] = v == 0.0 ? 0.1 : v;
            for (int c = 0; row && c < 7; c++) row[c] = lref[(size_t) i * 7 + c];
            const int p = pos_of[i], r = W.onode[ref_node[i]];
            for (int q = off[p]; q < off[p + 1]; q++) {
                const int f = meta[4 * q + 3], ob = W.onode[meta[4 * q + 2]];
                if (!fkeep[f] || ob < 0) continue;
                f_lm[fo] = li, f_ref[fo] = r, f_obs[fo] = ob, f_src[fo] = f;
                if (a.l_off) new_ref[W.n_new + f] = fo;
                fo++;
            }
        } else {
            const int j = i - oL;
            const double v = __ddiv_rn(1.0, W.new_depth[j]);
            const int r = new_ref[j];
            lm_src[li] = -1, lm_org[li] = -(j + 1);
            invd[li] = v == 0.0 ? 0.1 : v;
            if (row) {
                cam_point(W.cam, W.new_ref_xy[2 * j], W.new_ref_xy[2 * j + 1], row);
                row[3] = W.new_vel_ref[2 * j], row[4] = W.new_vel_ref[2 * j + 1], row[5] = 0.0, row[6] = W.node_td[r];
            }
            if (nn[i] == 0) continue;
            f_lm[fo] = li, f_ref[fo] = r, f_obs[fo] = W.cur_node, f_src[fo] = -1;
            double *c = fnew + (size_t) nbase[i] * 14;
            cam_point(W.cam, W.new_ref_xy[2 * j], W.new_ref_xy[2 * j + 1], c);
            cam_point(W.cam, W.new_cur_xy[2 * j], W.new_cur_xy[2 * j + 1], c + 3);
            c[6] = W.new_vel_ref[2 * j], c[7] = W.new_vel_ref[2 * j + 1], c[8] = 0.0;
            c[9] = W.new_vel_cur[2 * j], c[10] = W.new_vel_cur[2 * j + 1], c[11] = 0.0;
            c[12] = W.node_td[r], c[13] = W.node_td[W.cur_node];
        }
    }
    // the new observations of carried landmarks, after the landmark's surviving old factors, in node order, with the landmark's resident
    // reference row (pts0, vel0, td0)
    for (int k = t; k < nobs; k += VIS_THREADS) {
        const int j = W.src ? W.src[k] : k;
        if (j < 0 || j >= W.n_in) continue;
        const int l = W.obs_lm[j], node = W.obs_node ? W.obs_node[j] : W.cur_node;
        if (node < 0 || node >= W.nK || l < 0 || l >= oL || !keep[l] || W.onode[ref_node[l]] == node) continue;
        const double *r0 = lref + (size_t) l * 7;
        if (isnan(r0[0])) continue;
        const int rank = __popc(mask[l] & ((1u << node) - 1u));
        const int fo = fbase[l] + nkeep[l] + rank;
        f_lm[fo] = lidx[l], f_ref[fo] = W.onode[ref_node[l]], f_obs[fo] = node, f_src[fo] = -1;
        double *c = fnew + (size_t) (nbase[l] + rank) * 14;
        c[0] = r0[0], c[1] = r0[1], c[2] = r0[2];
        cam_point(W.cam, W.obs_xy[2 * k], W.obs_xy[2 * k + 1], c + 3);
        c[6] = r0[3], c[7] = r0[4], c[8] = r0[5];
        c[9] = W.obs_vel[2 * k], c[10] = W.obs_vel[2 * k + 1], c[11] = 0.0;
        c[12] = r0[6], c[13] = W.node_td[node];
    }
    if (!a.l_off) return;
    __syncthreads();
    const int *fmap = new_ref + W.n_new;
    int *lcnt = new_ref + W.n_new + oF;
    // 4. the next culling's lists, landmark by landmark in next-row order: a carried landmark's entries of the last culling's list that are not
    // flagged, lie in a next node and name a carried factor (or no factor, in the reference node), then its new observations in node order;
    // a new map point's creation observation (when it has a factor) and its reference observation
    const int *ooff = a.obs_off + W.cull_off0, *o_node = a.obs_node + W.cull_obs0;
    const float *o_kp = a.obs_kp + 2 * (size_t) W.cull_obs0, *o_rkp = a.lm_ref_kp + 2 * (size_t) W.cull_lm0;
    for (int i = t; i < NA; i += VIS_THREADS) {
        int c = 0;
        if (i < oL && keep[i]) {
            const int r = ref_node[i];
            for (int o = ooff[i]; o < ooff[i + 1]; o++) c += listed(ofac[o], o_node[o], obs_out[o], W.onode[o_node[o]], r, oF, fmap);
            c += nn[i];
        } else if (keep[i]) {
            c = 1 + nn[i];
        }
        lcnt[i] = c;
    }
    __syncthreads();
    const int n_list = block_exscan(lcnt, NA, tmp);
    int *l_ref = a.l_ref + W.lm_out, *l_off = a.l_off + W.lm_out + w, *l_node = a.l_node + W.lst_obs, *l_fac = a.l_fac + W.lst_obs;
    float *l_rkp = a.l_rkp + 2 * (size_t) W.lm_out, *l_kp = a.l_kp + 2 * (size_t) W.lst_obs;
    if (t == 0) cnt[8] = n_list, l_off[L] = n_list;
    for (int i = t; i < NA; i += VIS_THREADS) {
        if (!keep[i]) continue;
        const int li = lidx[i];
        int e = lcnt[i];
        l_off[li] = e;
        if (i < oL) {
            const int r = ref_node[i];
            l_ref[li] = W.onode[r], l_rkp[2 * li] = o_rkp[2 * i], l_rkp[2 * li + 1] = o_rkp[2 * i + 1];
            for (int o = ooff[i]; o < ooff[i + 1]; o++)
                if (listed(ofac[o], o_node[o], obs_out[o], W.onode[o_node[o]], r, oF, fmap))
                    list_entry(l_node, l_fac, l_kp, e++, W.onode[o_node[o]], ofac[o] >= 0 ? fmap[ofac[o]] : -1, o_kp + 2 * o);
        } else {
            const int j = i - oL;
            l_ref[li] = new_ref[j], l_rkp[2 * li] = W.new_ref_xy[2 * j], l_rkp[2 * li + 1] = W.new_ref_xy[2 * j + 1];
            if (nn[i]) list_entry(l_node, l_fac, l_kp, e++, W.cur_node, fbase[i], W.new_cur_xy + 2 * j);
            list_entry(l_node, l_fac, l_kp, e, new_ref[j], -1, W.new_ref_xy + 2 * j);
        }
    }
    // a carried landmark's new observations end its list (its segment ends where the next one's starts)
    for (int k = t; k < nobs; k += VIS_THREADS) {
        const int j = W.src ? W.src[k] : k;
        if (j < 0 || j >= W.n_in) continue;
        const int l = W.obs_lm[j], node = W.obs_node ? W.obs_node[j] : W.cur_node;
        if (node < 0 || node >= W.nK || l < 0 || l >= oL || !keep[l] || W.onode[ref_node[l]] == node || isnan(lref[(size_t) l * 7])) continue;
        const int rank = __popc(mask[l] & ((1u << node) - 1u));
        const int end = l + 1 < NA ? lcnt[l + 1] : n_list;
        list_entry(l_node, l_fac, l_kp, end - nn[l] + rank, node, fbase[l] + nkeep[l] + rank, W.obs_xy + 2 * k);
    }
}

cudaError_t launch_vision(const VisArgs &a, int n_windows, cudaStream_t stream) {
    ba_vision_build<<<n_windows, VIS_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

// pack_window's tables (ba_handle.cu) of one built window, in its orders.  Landmark positions: a stable counting sort by reference node (no
// factor: last), placed by warp 0 in id order, 32 landmarks a step (__match_any_sync ranks the lanes of one key).  Record slots: factor order
// within each landmark, placed by warp 0 the same way.  lin_vis runs: the greedy scan is sequential, one thread (L <= max_L steps).  Pairs in
// key order ref K + obs; a run's Gram partials and its slots ordered by observing node: a warp per run, lane k for observing node k.
constexpr int NO_FACTOR = 0x7fffffff;

__global__ void __launch_bounds__(VIS_THREADS) ba_pack_structure(PackArgs a) {
    __shared__ Scan::TempStorage tmp;
    __shared__ int s_pair[VIS_MAX_NODES * VIS_MAX_NODES];  // (ref K + obs) -> pair, -1: none
    __shared__ int s_part[VIS_MAX_NODES * VIS_MAX_NODES];  // pair -> its partials, then its first partial
    __shared__ int s_bin[VIS_MAX_NODES + 1];
    __shared__ int s_bad, s_nrun;
    const int w = blockIdx.x, t = threadIdx.x, lane = t & 31;
    const VisWin &W = a.win[w];
    int *cnt = a.counts + (size_t) w * VIS_COUNTS;
    const int L = cnt[0], F = cnt[1], K = W.nK;
    if (cnt[3] != 0 || L > a.L || F > a.F) return;
    const int *flm = a.f_lm + W.f_out, *fref = a.f_ref + W.f_out, *fobs = a.f_obs + W.f_out, *fsrc = a.f_src + W.f_out, *lms = a.lm_src + W.lm_out;
    const size_t wL = (size_t) w * a.L, wF = (size_t) w * a.F, PM = (size_t) a.K * (a.K - 1);
    const PackTables &T = a.out;
    int *perm = T.lm_perm + wL, *off = T.lm_off + w * (a.L + 1), *meta = T.f_meta_s + wF * 4, *vb = T.vb_lm0 + (size_t) w * a.NVB;
    int *nrun_of = T.ref_nrun + (size_t) w * a.K, *poff = T.part_off + w * (PM + 1), *pro = T.pair_ro + w * PM, *ord = T.vis_ord + wF;
    uint8_t *act = T.f_active + wF;
    int *fidx = a.fidx + W.f_out, *lmap = a.map + W.lm_out, *smap = a.map + a.nL + W.f_out;
    // scratch: factors per landmark, first factor per landmark, position of each landmark, reference key by position (K: no factor), cursor
    // per landmark (K by id first), new-factor rank (F), old slot of each old factor (oF), observing nodes of each run (NVB)
    int *nf = a.scratch + W.pscr, *first = nf + L, *pos_of = first + L, *key = pos_of + L, *cur = key + L, *newt = cur + L, *oslot = newt + F,
        *seen = oslot + W.oF;
    const int *ometa = a.old_meta + wF * 4;
    __syncthreads();  // every thread has read cnt before any writes it
    for (int l = t; l < L; l += VIS_THREADS) nf[l] = 0, first[l] = NO_FACTOR;
    for (int i = t; i < K * K; i += VIS_THREADS) s_pair[i] = -1;
    for (int i = t; i <= K; i += VIS_THREADS) s_bin[i] = 0;
    for (int i = t; i < a.K; i += VIS_THREADS) nrun_of[i] = 0;
    for (int q = t; q < W.oF; q += VIS_THREADS) oslot[ometa[4 * q + 3]] = q;
    if (t == 0) s_bad = NO_FACTOR;
    __syncthreads();
    for (int f = t; f < F; f += VIS_THREADS) {
        const int l = flm[f];
        atomicAdd(nf + l, 1), atomicMin(first + l, f);
        s_pair[fref[f] * K + fobs[f]] = 0;
        act[f] = 1;
        newt[f] = fsrc[f] < 0;
    }
    for (int l = t; l < L; l += VIS_THREADS) lmap[l] = lms[l] >= 0 ? lms[l] : -(W.lm_out + l + 1);
    __syncthreads();
    // 1. landmark positions: by reference node, stable by id, landmarks without factors last
    for (int l = t; l < L; l += VIS_THREADS) {
        const int k = nf[l] ? fref[first[l]] : K;
        cur[l] = k;
        atomicAdd(s_bin + k, 1);
    }
    __syncthreads();
    if (t == 0)
        for (int k = 0, s = 0; k <= K; k++) {
            const int c = s_bin[k];
            s_bin[k] = s, s += c;
        }
    __syncthreads();
    if (t < 32) {
        for (int b = 0; b < L; b += 32) {
            const int l = b + lane, k = l < L ? cur[l] : -1;
            const unsigned peers = __match_any_sync(~0u, k), below = peers & ((1u << lane) - 1u);
            if (l < L) {
                const int p = s_bin[k] + __popc(below);
                perm[p] = l, pos_of[l] = p, key[p] = k;
            }
            __syncwarp();
            if (l < L && below == 0) s_bin[k] += __popc(peers);
            __syncwarp();
        }
    }
    __syncthreads();
    // 2. CSR by position, and the rank of every new factor among the new factors (its row of f_new)
    for (int p = t; p < L; p += VIS_THREADS) off[p] = nf[perm[p]];
    __syncthreads();
    block_exscan(off, L, tmp);
    block_exscan(newt, F, tmp);
    if (t == 0) off[L] = F;
    for (int l = t; l < L; l += VIS_THREADS) cur[l] = off[pos_of[l]];
    __syncthreads();
    // 3. record slots in factor order within each landmark; the slot's row of the slide (old slot, or the new factor's constants)
    if (t < 32) {
        for (int b = 0; b < F; b += 32) {
            const int f = b + lane, l = f < F ? flm[f] : -1;
            const unsigned peers = __match_any_sync(~0u, l), below = peers & ((1u << lane) - 1u);
            if (f < F) {
                const int q = cur[l] + __popc(below);
                meta[4 * q] = l, meta[4 * q + 1] = fref[f], meta[4 * q + 2] = fobs[f], meta[4 * q + 3] = f;
                fidx[q] = f;
                smap[q] = fsrc[f] >= 0 ? oslot[fsrc[f]] : -(14 * (W.nf_out + newt[f]) + 1);
            }
            __syncwarp();
            if (f < F && below == 0) cur[l] += __popc(peers);
            __syncwarp();
        }
    }
    __syncthreads();
    // a landmark has one reference node and at most one observation per node: the first factor that breaks it, in factor order
    for (int p = t; p < L; p += VIS_THREADS) {
        unsigned obs = 0u;
        for (int q = off[p]; q < off[p + 1]; q++) {
            const int o = meta[4 * q + 2];
            if (meta[4 * q + 1] != key[p] || (obs >> o) & 1u) {
                atomicMin(&s_bad, meta[4 * q + 3]);
                break;
            }
            obs |= 1u << o;
        }
    }
    __syncthreads();
    if (s_bad != NO_FACTOR) {
        if (t == 0) cnt[3] = VIS_EPACK_DUP, cnt[4] = s_bad, cnt[9] = flm[s_bad], cnt[10] = fobs[s_bad];
        return;
    }
    // 4. lin_vis runs: whole landmarks of one reference node, <= 128 record slots each
    if (t == 0) {
        int nrun = 0, l0 = 0, err = 0;
        while (l0 < L) {
            const int ref = key[l0];
            int l1 = l0;
            while (l1 < L && key[l1] == ref && off[l1 + 1] - off[l0] <= 128) l1++;
            if (l1 == l0 || nrun >= a.NVB - 2) {
                err = l1 == l0 ? VIS_EPACK_LM128 : VIS_EPACK_RUNS;
                break;
            }
            if (ref < K) nrun_of[ref]++;
            vb[nrun++] = l0;
            l0 = l1;
        }
        if (err) {
            cnt[3] = err, cnt[4] = perm[l0];
            nrun = -1;
        } else {
            vb[nrun] = L, vb[a.NVB - 1] = nrun;
        }
        s_nrun = nrun;
    }
    // 5. pairs in key order
    const int KK = K * K;
    {
        const int chunk = (KK + VIS_THREADS - 1) / VIS_THREADS, b = t * chunk, e = min(KK, b + chunk);
        int c = 0;
        for (int i = b; i < e; i++) c += s_pair[i] == 0;
        int base, P;
        Scan(tmp).ExclusiveSum(c, base, P);
        for (int i = b; i < e; i++)
            if (s_pair[i] == 0) s_pair[i] = base, pro[base] = ((i / K) << 8) | (i % K), base++;
        for (int i = t; i < P; i += VIS_THREADS) s_part[i] = 0;
        if (t == 0) T.npairs[w] = P;
    }
    __syncthreads();
    const int nrun = s_nrun;
    if (nrun < 0) return;
    // 6. each run's observing nodes; a pair's partials: one per run of its reference node that observes from its node
    for (int r = t; r < nrun; r += VIS_THREADS) {
        unsigned s = 0u;
        for (int q = off[vb[r]]; q < off[vb[r + 1]]; q++) s |= 1u << meta[4 * q + 2];
        seen[r] = (int) s;
        const int ref = key[vb[r]];
        for (unsigned m = s; m; m &= m - 1) atomicAdd(s_part + s_pair[ref * K + __ffs(m) - 1], 1);
    }
    __syncthreads();
    {
        const int P = T.npairs[w], total = block_exscan(s_part, P, tmp);
        for (int i = t; i < P; i += VIS_THREADS) poff[i] = s_part[i];
        if (t == 0) poff[P] = total;
    }
    __syncthreads();
    // 7. vis_ord: warp per run, lane k counts the run's slots observed from node k; their Gram partial is the pair's first plus the earlier
    // runs of the same reference node that observe from k
    for (int r = t >> 5; r < nrun; r += VIS_THREADS / 32) {
        const int q0 = off[vb[r]], q1 = off[vb[r + 1]];
        if (q0 == q1) continue;
        const int ref = meta[4 * q0 + 1];
        int c = 0;
        for (int q = q0; q < q1; q++) c += meta[4 * q + 2] == lane;
        int incl = c;
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(~0u, incl, d);
            if (lane >= d) incl += v;
        }
        int at = q0 + incl - c;
        if (c == 0) continue;
        int pidx = s_part[s_pair[ref * K + lane]];
        for (int r2 = r - 1; r2 >= 0 && key[vb[r2]] == ref; r2--) pidx += (seen[r2] >> lane) & 1;
        for (int q = q0; q < q1; q++)
            if (meta[4 * q + 2] == lane) ord[at++] = (q - q0) | (pidx << 8);
    }
}

cudaError_t launch_pack(const PackArgs &a, int n_windows, cudaStream_t stream) {
    ba_pack_structure<<<n_windows, VIS_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace icg
