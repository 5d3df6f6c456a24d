// detect.cu -- Path A, detection leg: Shi-Tomasi block detection + sub-pixel refinement for sm_90a.
//
// Replaces the tbb::parallel_for body of Tracking::featuresDetection (IG/tracking/tracking.cc:627-656):
//     cv::goodFeaturesToTrack(block_image, out, n, 0.01, track_min_pixel_distance_, block_mask)      (:647)
//     cv::cornerSubPix(block_image, out, Size(5,5), Size(-1,-1), TermCriteria(COUNT+EPS, 20, 0.01))    (:651)
// for ALL blocks of a frame in one call.  OpenCV is an un-vendored dependency of the reference; the arithmetic restated here
// (SURVEY.md Appendix A.4 / A.5, float sequences matched bit-for-bit against cv2 4.13.0) is pinned by oracle/detect_ref.c and
// tests/golden/detect_golden.npz.  ROI semantics as in C++: the Sobel derivative of a block reads the frame's pixels beyond
// the block edge, the 3x3 covariance box filter reflects at the block edge, getRectSubPix replicates at the block edge.
//
// Kernels (all HBM/L2 streaming or tiny):  detect_eig (min-eigenvalue map + masked per-block maximum),
// detect_nms (threshold, 3x3 non-maximum suppression, candidate list), detect_select (CTA per block: bitonic sort by
// (value desc, address desc) + greedy min-distance grid), detect_subpix (warp per corner).  detect_eig and detect_nms return at once for
// a block whose max_corners is <= 0.  The point-list entry (icg_detect_features[_dev], tracking.cc:579-685) adds detect_occupancy (gate,
// per-block deficits, occupancy mask plane) before them and detect_compact (frame coordinates, block order) after them.  Compile with -fmad=false; the two
// fused multiply-adds OpenCV's AVX2 Sobel performs are written explicitly with __fmaf_rn.
#include <math.h>
#include <string.h>

#include <vector>

#include "common.cuh"

namespace icg {

constexpr int DET_MAX_CAND = 16384;  // candidates per block after NMS (sorted in 128 KB of dynamic shared memory)
constexpr int DET_CELL_CAP = 4;      // accepted corners per min-distance grid cell (cell = round(minDistance) -> at most 4)
constexpr int DET_MAX_CELLS = 1024;

struct DetRect {
    int x, y, w, h;
};

struct DetArgs {
    const uint8_t *img;
    const uint8_t *mask;  // may be null
    int W, H, pitch;
    int n_blocks, cap;    // cap = corner capacity per block in the outputs
    int roi_cap;          // eig plane capacity per block (floats)
    const DetRect *rois;
    const int *max_corners;
    float *eig;                 // [n_blocks][roi_cap]
    unsigned int *maxkey;       // [n_blocks] order-preserving key of the masked maximum
    unsigned long long *cand;   // [n_blocks][DET_MAX_CAND]
    int *ncand;                 // [n_blocks]
    float *out_xy;              // [n_blocks][cap][2]
    int *out_n;                 // [n_blocks]
    int *overflow;
    double quality, min_distance;
    // batched frames: block b belongs to frame b / bpf, whose image starts frame * img_stride bytes further and whose mask (row pitch
    // mask_pitch) frame * mask_stride bytes further
    size_t img_stride, mask_stride;
    int bpf, mask_pitch;
};
// kernel prologue: point the by-value argument copy at the block's frame
#define DET_FRAME(A, b)                                           \
    do {                                                          \
        const size_t f_ = (size_t) ((b) / (A).bpf);                  \
        (A).img += f_ * (A).img_stride;                           \
        if ((A).mask) (A).mask += f_ * (A).mask_stride;           \
    } while (0)

__device__ __forceinline__ int refl(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
    return p;
}
__device__ __forceinline__ unsigned int float_key(float v) {  // monotonic float -> uint
    unsigned int b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned int k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// cv::Sobel(..., CV_32F, ksize 3, scale = 1/(4*3*255)) at frame pixel (x, y): reflect-101 at the FRAME border only
// fma_row: OpenCV's AVX2 u8->f32 row filter covers 32 pixels per iteration with FMA; the last (roi_width % 32) columns of a row
// take the scalar loop, which rounds every product and sum separately (measured against cv2 4.13.0).
__device__ __forceinline__ void sobel_at(const DetArgs &A, int x, int y, bool fma_row, float &dx, float &dy) {
    const float s = (float) (1.0 / (4 * 3 * 255.0)), s2 = (float) (2.0 * (1.0 / (4 * 3 * 255.0)));
    const int xm = refl(x - 1, A.W), xp = refl(x + 1, A.W), ym = refl(y - 1, A.H), yp = refl(y + 1, A.H);
    const uint8_t *r0 = A.img + (size_t) ym * A.pitch, *r1 = A.img + (size_t) y * A.pitch, *r2 = A.img + (size_t) yp * A.pitch;
    const float a00 = r0[xm], a01 = r0[x], a02 = r0[xp], a10 = r1[xm], a12 = r1[xp], a20 = r2[xm], a21 = r2[x], a22 = r2[xp];
    const float top = a02 - a00, mid = a12 - a10, bot = a22 - a20;
    dx = __fmaf_rn(top + bot, s, s2 * mid);                                  // SymmColumnFilter: fma(S0 + S2, f1, f0 * S1)
    float rowm, rowp;
    if (fma_row) {
        rowm = __fmaf_rn(a02, s, __fmaf_rn(a01, s2, s * a00));  // RowVec: s*L, fma(C, 2s, .), fma(R, s, .)
        rowp = __fmaf_rn(a22, s, __fmaf_rn(a21, s2, s * a20));
    } else {
        rowm = (s * a00 + s2 * a01) + s * a02;
        rowp = (s * a20 + s2 * a21) + s * a22;
    }
    dy = rowp - rowm;
}

// ------------------------------------------------------------------------------------------------ eig map
constexpr int ET_W = 32, ET_H = 16;
__global__ void __launch_bounds__(256) detect_eig(DetArgs A) {
    __shared__ float s_xx[ET_H + 2][ET_W + 2], s_xy[ET_H + 2][ET_W + 2], s_yy[ET_H + 2][ET_W + 2];
    __shared__ unsigned int s_max;
    const int b = blockIdx.z;
    if (A.max_corners[b] <= 0) return;  // no deficit: detect_select returns 0 corners whatever the map holds
    DET_FRAME(A, b);
    const DetRect R = A.rois[b];
    const int tx0 = blockIdx.x * ET_W, ty0 = blockIdx.y * ET_H;
    if (tx0 >= R.w || ty0 >= R.h) return;
    const int tid = threadIdx.x;
    if (tid == 0) s_max = 0;
    for (int e = tid; e < (ET_H + 2) * (ET_W + 2); e += 256) {
        const int cy = e / (ET_W + 2), cx = e - cy * (ET_W + 2);
        // covariance cell (tx0 + cx - 1, ty0 + cy - 1) in ROI coordinates, reflect-101 at the ROI edge (boxFilter on the ROI-sized cov Mat)
        const int rx = refl(tx0 + cx - 1, R.w), ry = refl(ty0 + cy - 1, R.h);
        float dx, dy;
        sobel_at(A, R.x + rx, R.y + ry, rx < (R.w & ~31), dx, dy);
        s_xx[cy][cx] = dx * dx, s_xy[cy][cx] = dx * dy, s_yy[cy][cx] = dy * dy;
    }
    __syncthreads();
    unsigned int lmax = 0;
    for (int e = tid; e < ET_W * ET_H; e += 256) {
        const int py = e / ET_W, px = e - py * ET_W;
        const int x = tx0 + px, y = ty0 + py;
        if (x >= R.w || y >= R.h) continue;
        double sa = 0, sb = 0, sc = 0;  // unnormalised 3x3 box sums accumulated in f64, rounded once to f32
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int i = 0; i < 3; i++) sa += (double) s_xx[py + j][px + i], sb += (double) s_xy[py + j][px + i], sc += (double) s_yy[py + j][px + i];
        const float a = (float) sa * 0.5f, bb = (float) sb, c = (float) sc * 0.5f;
        const float ev = (a + c) - sqrtf((a - c) * (a - c) + bb * bb);
        A.eig[(size_t) b * A.roi_cap + (size_t) y * R.w + x] = ev;
        if (!A.mask || A.mask[(size_t) (R.y + y) * A.mask_pitch + R.x + x]) lmax = max(lmax, float_key(ev));
    }
    for (int o = 16; o > 0; o >>= 1) lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    if ((tid & 31) == 0 && lmax) atomicMax(&s_max, lmax);
    __syncthreads();
    if (tid == 0 && s_max) atomicMax(&A.maxkey[b], s_max);
}

// ------------------------------------------------------------------------------------------------ threshold + NMS
__global__ void __launch_bounds__(256) detect_nms(DetArgs A) {
    const int b = blockIdx.z;
    if (A.max_corners[b] <= 0) return;  // as in detect_eig: no candidates are needed
    DET_FRAME(A, b);
    const DetRect R = A.rois[b];
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x < 1 || y < 1 || x >= R.w - 1 || y >= R.h - 1) return;
    const unsigned int mk = A.maxkey[b];
    const double maxVal = mk ? (double) key_float(mk) : 0.0;  // minMaxLoc over the mask (0 when the mask is empty)
    const float thr = (float) (maxVal * A.quality);           // threshold(eig, eig, maxVal * qualityLevel, 0, THRESH_TOZERO)
    const float *E = A.eig + (size_t) b * A.roi_cap;
    const float val = E[(size_t) y * R.w + x];
    if (!(val > thr)) return;
    float mx = val;  // dilate 3x3 of the thresholded map: a neighbour above val is necessarily above thr
#pragma unroll
    for (int j = -1; j <= 1; j++)
#pragma unroll
        for (int i = -1; i <= 1; i++) mx = fmaxf(mx, E[(size_t) (y + j) * R.w + x + i]);
    if (val != mx) return;
    if (A.mask && !A.mask[(size_t) (R.y + y) * A.mask_pitch + R.x + x]) return;
    const int slot = atomicAdd(&A.ncand[b], 1);
    if (slot >= DET_MAX_CAND) {
        *A.overflow = 1;
        return;
    }
    // sort key: value descending, then linear address descending (goodFeaturesToTrack's greaterThanPtr); val > 0 here or thr < 0
    A.cand[(size_t) b * DET_MAX_CAND + slot] = ((unsigned long long) float_key(val) << 32) | (unsigned int) (y * R.w + x);
}

// ------------------------------------------------------------------------------------------------ sort + greedy min-distance selection
__global__ void __launch_bounds__(1024) detect_select(DetArgs A) {
    extern __shared__ unsigned long long s_key[];  // DET_MAX_CAND keys
    __shared__ float s_gx[DET_MAX_CELLS][DET_CELL_CAP], s_gy[DET_MAX_CELLS][DET_CELL_CAP];
    __shared__ unsigned char s_gn[DET_MAX_CELLS];
    const int b = blockIdx.x, tid = threadIdx.x;
    DET_FRAME(A, b);
    const DetRect R = A.rois[b];
    int n = min(A.ncand[b], DET_MAX_CAND);
    int npow = 1;
    while (npow < n) npow <<= 1;
    for (int i = tid; i < npow; i += 1024) s_key[i] = i < n ? A.cand[(size_t) b * DET_MAX_CAND + i] : 0ull;
    __syncthreads();
    // bitonic sort, descending
    for (int k = 2; k <= npow; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < npow; i += 1024) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = s_key[i], c = s_key[ixj];
                    const bool desc = (i & k) == 0;
                    if (desc ? a < c : a > c) s_key[i] = c, s_key[ixj] = a;
                }
            }
            __syncthreads();
        }
    // greedy acceptance with the min-distance cell grid (sequential by definition; a few hundred candidates are examined)
    const int max_corners = min(A.max_corners[b], A.cap);
    if (tid == 0) {
        int n_out = 0;
        float *out = A.out_xy + (size_t) b * A.cap * 2;
        if (max_corners > 0) {
            if (A.min_distance >= 1) {
                const int cell = (int) rint(A.min_distance);
                const int gw = (R.w + cell - 1) / cell, gh = (R.h + cell - 1) / cell;
                const double md2 = A.min_distance * A.min_distance;
                if (gw * gh > DET_MAX_CELLS) {
                    *A.overflow = 2;
                } else {
                    for (int c = 0; c < gw * gh; c++) s_gn[c] = 0;
                    for (int i = 0; i < n; i++) {
                        const int addr = (int) (s_key[i] & 0xffffffffu);
                        const int y = addr / R.w, x = addr - y * R.w;
                        const int xc = x / cell, yc = y / cell;
                        const int x1 = max(0, xc - 1), y1 = max(0, yc - 1), x2 = min(gw - 1, xc + 1), y2 = min(gh - 1, yc + 1);
                        bool good = true;
                        for (int yy = y1; yy <= y2 && good; yy++)
                            for (int xx = x1; xx <= x2 && good; xx++) {
                                const int c = yy * gw + xx;
                                for (int k = 0; k < s_gn[c]; k++) {
                                    const float dx = (float) x - s_gx[c][k], dy = (float) y - s_gy[c][k];
                                    if ((double) (dx * dx + dy * dy) < md2) {
                                        good = false;
                                        break;
                                    }
                                }
                            }
                        if (!good) continue;
                        const int c = yc * gw + xc;
                        if (s_gn[c] < DET_CELL_CAP) {
                            s_gx[c][s_gn[c]] = (float) x, s_gy[c][s_gn[c]] = (float) y, s_gn[c]++;
                        } else {
                            *A.overflow = 3;  // more than 4 corners in one cell is geometrically impossible for cell = round(minDistance)
                        }
                        out[2 * n_out] = (float) x, out[2 * n_out + 1] = (float) y;
                        if (++n_out == max_corners) break;
                    }
                }
            } else {
                for (int i = 0; i < n && n_out < max_corners; i++) {
                    const int addr = (int) (s_key[i] & 0xffffffffu);
                    out[2 * n_out] = (float) (addr % R.w), out[2 * n_out + 1] = (float) (addr / R.w);
                    n_out++;
                }
            }
        }
        A.out_n[b] = n_out;
    }
}

// ------------------------------------------------------------------------------------------------ cornerSubPix (warp per corner)
__global__ void __launch_bounds__(128) detect_subpix(DetArgs A, int half_win, int max_iter, double eps2) {
    __shared__ float s_sub[4][13 * 13];
    __shared__ float s_mask[11 * 11];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y;
    DET_FRAME(A, b);
    const int p = blockIdx.x * 4 + warp;
    if (half_win != 5) return;  // the only window the reference uses (tracking.cc:623)
    for (int e = threadIdx.x; e < 121; e += 128) {
        const int i = e / 11, j = e - 11 * i;
        const float ty = (float) (i - 5) / 5, tx = (float) (j - 5) / 5;
        s_mask[e] = expf(-ty * ty) * expf(-tx * tx);
    }
    __syncthreads();
    if (p >= A.out_n[b]) return;
    const DetRect R = A.rois[b];
    const uint8_t *roi = A.img + (size_t) R.y * A.pitch + R.x;
    float *xy = A.out_xy + ((size_t) b * A.cap + p) * 2;
    const float cTx = xy[0], cTy = xy[1];
    float cIx = cTx, cIy = cTy;
    float *sub = s_sub[warp];
    int iter = 0;
    float err = 0.f;
    do {
        // getRectSubPix(src, Size(13, 13), cI, ..., CV_32F): bilinear, replicate at the ROI edge
        const float cx = cIx - 6.f, cy = cIy - 6.f;
        const int ipx = __float2int_rd(cx), ipy = __float2int_rd(cy);
        const float a = cx - (float) ipx, bq = cy - (float) ipy;
        const float a11 = (1.f - a) * (1.f - bq), a12 = a * (1.f - bq), a21 = (1.f - a) * bq, a22 = a * bq;
        __syncwarp();
        for (int e = lane; e < 169; e += 32) {
            const int yy = e / 13, xx = e - 13 * yy;
            const int X0 = min(max(ipx + xx, 0), R.w - 1), X1 = min(max(ipx + xx + 1, 0), R.w - 1);
            const int Y0 = min(max(ipy + yy, 0), R.h - 1), Y1 = min(max(ipy + yy + 1, 0), R.h - 1);
            sub[e] = (float) roi[(size_t) Y0 * A.pitch + X0] * a11 + (float) roi[(size_t) Y0 * A.pitch + X1] * a12 + (float) roi[(size_t) Y1 * A.pitch + X0] * a21 +
                     (float) roi[(size_t) Y1 * A.pitch + X1] * a22;
        }
        __syncwarp();
        double sa = 0, sb = 0, sc = 0, sb1 = 0, sb2 = 0;
        for (int e = lane; e < 121; e += 32) {
            const int i = e / 11, j = e - 11 * i;
            const double m = s_mask[e];
            const float *sp = sub + (i + 1) * 13 + (j + 1);
            const double tgx = (double) (sp[1] - sp[-1]), tgy = (double) (sp[13] - sp[-13]);
            const double gxx = tgx * tgx * m, gxy = tgx * tgy * m, gyy = tgy * tgy * m;
            const double px = j - 5, py = i - 5;
            sa += gxx, sb += gxy, sc += gyy;
            sb1 += gxx * px + gxy * py;
            sb2 += gxy * px + gyy * py;
        }
        for (int o = 16; o > 0; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o), sb += __shfl_xor_sync(0xffffffffu, sb, o), sc += __shfl_xor_sync(0xffffffffu, sc, o);
            sb1 += __shfl_xor_sync(0xffffffffu, sb1, o), sb2 += __shfl_xor_sync(0xffffffffu, sb2, o);
        }
        const double det = sa * sc - sb * sb;
        if (fabs(det) <= 2.220446049250313e-16 * 2.220446049250313e-16) break;
        const double scale = 1.0 / det;
        const float nx = (float) ((double) cIx + sc * scale * sb1 - sb * scale * sb2), ny = (float) ((double) cIy - sb * scale * sb1 + sa * scale * sb2);
        err = (nx - cIx) * (nx - cIx) + (ny - cIy) * (ny - cIy);
        cIx = nx, cIy = ny;
        if (cIx < 0 || cIx >= (float) R.w || cIy < 0 || cIy >= (float) R.h) break;
    } while (++iter < max_iter && (double) err > eps2);
    if (fabsf(cIx - cTx) > (float) half_win || fabsf(cIy - cTy) > (float) half_win) cIx = cTx, cIy = cTy;
    if (lane == 0) xy[0] = cIx, xy[1] = cIy;
}

// ------------------------------------------------------------------------------------------------ featuresDetection from point lists
// Tracking::featuresDetection before its block loop (IG/tracking/tracking.cc:579-620): the gate, the per-block counts of the existing
// points and the occupancy mask, for every frame of a call.  List A = the frame's map-point features (undistorted keyPoint()), list B =
// pts2d_new_ (distorted).  A point whose status byte is 0 is neither counted nor masked.
constexpr int DET_OCC_MAX_BLOCKS = 1024;  // blocks per frame (the grid of a 6400 x 6400 frame)

struct OccArgs {
    const float *a_xy, *b_xy;           // point lists (x, y) of all frames
    const uint8_t *a_st, *b_st;         // per-point status or null
    const int *a_off, *b_off;           // [n_frames + 1] each
    const int *n_ref;                   // [n_frames]; < 0: the number of valid points of list B
    const int *ismask;                  // [n_frames]
    uint8_t *mask;                      // frame f's plane at mask + f * mask_stride, row pitch mask_pitch
    size_t mask_stride;
    int mask_pitch, W, H, rows_per_cta;
    int cols, nb, bw, bh, quota, radius, gate_max;  // gate_max = max_features - 5
    int *max_corners;                   // [n_frames * nb] out: quota - count, 0 for a skipped frame
    int *skipped;                       // [n_frames] out: 1 when the gate skipped the frame
};

__device__ __forceinline__ bool occ_valid(const uint8_t *st, int i) { return !st || st[i]; }

__device__ __forceinline__ int block_reduce_add(int v, int *s_acc) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // every thread has read the previous result
    if (threadIdx.x == 0) *s_acc = 0;
    __syncthreads();
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(s_acc, v);
    __syncthreads();
    return *s_acc;
}

// block index of a point as tracking.cc:598-605 computes it: int(x / (float) bw), int(y / (float) bh) in IEEE float32, truncation toward
// zero, row * cols + col (a col == cols aliases into the next row).  -1 for an index outside [0, nb), where the reference writes past its
// array.  Quotients are clamped before the conversion; a clamped value lies outside the grid either way.
__device__ __forceinline__ int occ_block(float x, float y, const OccArgs &O) {
    const float qx = fminf(fmaxf(__fdiv_rn(x, (float) O.bw), -1e9f), 1e9f), qy = fminf(fmaxf(__fdiv_rn(y, (float) O.bh), -1e9f), 1e9f);
    if (qx != qx || qy != qy) return -1;
    const long long k = (long long) __float2int_rz(qy) * O.cols + __float2int_rz(qx);
    return k >= 0 && k < O.nb ? (int) k : -1;
}

// cv::Point(pt) = cvRound of each coordinate (round half to even); false for a centre whose disc of radius r misses rows [y0, y1) or the
// frame's columns (a centre beyond +-2^30 or NaN misses everything)
__device__ __forceinline__ bool occ_centre(float px, float py, int y0, int y1, const OccArgs &O, int2 &c) {
    const long long cx = __float2ll_rn(px), cy = __float2ll_rn(py), r = O.radius;
    if (cx < -(1ll << 30) || cx > (1ll << 30) || cy < -(1ll << 30) || cy > (1ll << 30)) return false;
    if (cy + r < y0 || cy - r > y1 - 1 || cx + r < 0 || cx - r >= O.W) return false;
    c = make_int2((int) cx, (int) cy);
    return true;
}

// cv::circle(mask, c, radius, 0, FILLED): the pixels with (x - cx)^2 + (y - cy)^2 <= radius^2, clipped to rows [y0, y1) and the frame.
// One warp per centre, lanes along the row; racing zero-stores into shared memory are order-independent.
__device__ __forceinline__ void occ_disc(int2 c, int y0, int y1, const OccArgs &O, uint8_t *s_rows, int lane) {
    const long long cx = c.x, cy = c.y, r = O.radius;
    const long long ya = max((long long) y0, cy - r), yb = min((long long) y1 - 1, cy + r);
    for (long long y = ya; y <= yb; y++) {
        const long long v = r * r - (y - cy) * (y - cy);
        long long d = (long long) sqrt((double) v);
        while (d * d > v) d--;
        while ((d + 1) * (d + 1) <= v) d++;
        const int xa = (int) max(0ll, cx - d), xb = (int) min((long long) O.W - 1, cx + d);
        uint8_t *row = s_rows + (size_t) (y - y0) * O.mask_pitch;
        for (int x = xa + lane; x <= xb; x += 32) row[x] = 0;
    }
}

// grid (ceil(H / rows_per_cta), n_frames) x 256; dynamic shared memory rows_per_cta * mask_pitch bytes.  Every CTA of a frame evaluates the
// gate; CTA 0 also counts and writes the frame's deficits; the others write rows [y0, y1) of the mask (a skipped frame's mask is not written).
__global__ void __launch_bounds__(256) detect_occupancy(OccArgs O) {
    extern __shared__ __align__(16) uint8_t s_rows[];
    __shared__ int s_cnt[DET_OCC_MAX_BLOCKS];
    __shared__ int s_acc;
    const int f = blockIdx.y, tid = threadIdx.x;
    const int a0 = O.a_off[f], a1 = O.a_off[f + 1], b0 = O.b_off[f], b1 = O.b_off[f + 1];
    int va = 0, vb = 0;
    for (int i = a0 + tid; i < a1; i += 256) va += occ_valid(O.a_st, i);
    for (int i = b0 + tid; i < b1; i += 256) vb += occ_valid(O.b_st, i);
    const int n_a = block_reduce_add(va, &s_acc);
    const int n_b = block_reduce_add(vb, &s_acc);
    const int n_ref = O.n_ref[f] >= 0 ? O.n_ref[f] : n_b;
    const bool skip = n_a + n_ref > O.gate_max;  // tracking.cc:579-582
    if (blockIdx.x == 0) {
        for (int k = tid; k < O.nb; k += 256) s_cnt[k] = 0;
        __syncthreads();
        if (!skip) {
            for (int i = a0 + tid; i < a1; i += 256)
                if (occ_valid(O.a_st, i)) {
                    const int k = occ_block(O.a_xy[2 * i], O.a_xy[2 * i + 1], O);
                    if (k >= 0) atomicAdd(&s_cnt[k], 1);
                }
            for (int i = b0 + tid; i < b1; i += 256)
                if (occ_valid(O.b_st, i)) {
                    const int k = occ_block(O.b_xy[2 * i], O.b_xy[2 * i + 1], O);
                    if (k >= 0) atomicAdd(&s_cnt[k], 1);
                }
        }
        __syncthreads();
        for (int k = tid; k < O.nb; k += 256) O.max_corners[f * O.nb + k] = skip ? 0 : O.quota - s_cnt[k];  // tracking.cc:629
        if (tid == 0) O.skipped[f] = skip;
    }
    if (skip) return;
    const int y0 = blockIdx.x * O.rows_per_cta, y1 = min(O.H, y0 + O.rows_per_cta);
    if (y0 >= y1) return;
    const int n16 = (y1 - y0) * O.mask_pitch / 16;
    uint4 *s16 = reinterpret_cast<uint4 *>(s_rows);
    for (int e = tid; e < n16; e += 256) s16[e] = make_uint4(~0u, ~0u, ~0u, ~0u);
    __syncthreads();
    if (O.ismask[f]) {
        // 256 points at a time: one coalesced load per thread keeps the valid centres whose disc reaches the band, then a warp per centre
        __shared__ int2 s_c[256];
        __shared__ int s_nc;
        const int warp = tid >> 5, lane = tid & 31, na = a1 - a0, n = na + (b1 - b0);
        for (int base = 0; base < n; base += 256) {
            if (tid == 0) s_nc = 0;
            __syncthreads();
            const int i = base + tid;
            int2 c;
            if (i < n) {
                const bool in_a = i < na;
                const int j = in_a ? a0 + i : b0 + (i - na);
                const float *xy = in_a ? O.a_xy : O.b_xy;
                if (occ_valid(in_a ? O.a_st : O.b_st, j) && occ_centre(xy[2 * j], xy[2 * j + 1], y0, y1, O, c)) s_c[atomicAdd(&s_nc, 1)] = c;
            }
            __syncthreads();
            for (int k = warp; k < s_nc; k += 8) occ_disc(s_c[k], y0, y1, O, s_rows, lane);
            __syncthreads();
        }
    }
    uint4 *g16 = reinterpret_cast<uint4 *>(O.mask + f * O.mask_stride + (size_t) y0 * O.mask_pitch);
    for (int e = tid; e < n16; e += 256) g16[e] = s16[e];
}

// tracking.cc:669-675: the corners of frame f in block order, shifted to frame coordinates in float32, at out_xy + f * nb * quota * 2;
// out_n[f] = their number, -1 when the gate skipped the frame, -2 when a block exceeded an internal capacity (the overflow flag).
__global__ void __launch_bounds__(256) detect_compact(DetArgs A, const int *skipped, int nb, int quota, float *out_xy, int *out_n) {
    __shared__ int s_off[DET_OCC_MAX_BLOCKS + 1];
    const int f = blockIdx.x, tid = threadIdx.x;
    if (skipped[f] || *A.overflow) {
        if (tid == 0) out_n[f] = skipped[f] ? -1 : -2;
        return;
    }
    if (tid == 0) {
        int n = 0;
        for (int k = 0; k < nb; k++) s_off[k] = n, n += A.out_n[f * nb + k];
        s_off[nb] = n;
        out_n[f] = n;
    }
    __syncthreads();
    float *dst = out_xy + (size_t) f * nb * quota * 2;
    const int warp = tid >> 5, lane = tid & 31;
    for (int k = warp; k < nb; k += 8) {
        const int b = f * nb + k, n = s_off[k + 1] - s_off[k];
        const DetRect R = A.rois[b];
        const float *src = A.out_xy + (size_t) b * A.cap * 2;
        for (int i = lane; i < n; i += 32) {
            dst[2 * (s_off[k] + i)] = (float) R.x + src[2 * i];
            dst[2 * (s_off[k] + i) + 1] = (float) R.y + src[2 * i + 1];
        }
    }
}

}  // namespace icg

// ======================================================================================================= C ABI
using namespace icg;

struct icg_detect {
    int W, H, pitch, max_blocks, cap, roi_cap, device;
    cudaStream_t stream;
    bool own_stream;
    uint8_t *d_img, *d_mask;
    DetRect *d_rois;
    int *d_maxc, *d_ncand, *d_out_n, *d_overflow;
    unsigned int *d_maxkey;
    float *d_eig, *d_out_xy;
    unsigned long long *d_cand;
    // pinned staging
    uint8_t *h_stage;
    size_t h_stage_bytes;
    // featuresDetection from point lists (allocated on first use): one occupancy mask plane per frame the handle's max_blocks allows,
    // per-frame parameters, the per-frame gate, the host call's point lists and outputs
    uint8_t *d_planes;
    int n_planes;
    int *d_fpar, *d_skipped, *d_fout_n;
    float *d_fout_xy, *d_pts;
    size_t pts_cap;
    // an asynchronous call's H2D copies from h_stage complete at stage_ev; the next writer of h_stage waits for it
    cudaEvent_t stage_ev;
    bool stage_pending;
};

extern "C" {

int icg_detect_create(icg_detect **out, int width, int height, int max_blocks, int max_corners_per_block, int max_roi_pixels, int device, void *stream) {
    if (!out || width < 16 || height < 16 || max_blocks < 1 || max_corners_per_block < 1 || max_roi_pixels < 9) {
        set_error("icg_detect_create: bad arguments");
        return ICG_EINVAL;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("icg_detect_create: no CUDA device (this library has no CPU fallback)");
        return ICG_ENODEVICE;
    }
    if (device < 0 || device >= ndev) {
        set_error("icg_detect_create: device %d out of range", device);
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ICG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("icg_detect_create: device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        return ICG_ENODEVICE;
    }
    icg_detect *h = new icg_detect();
    h->W = width, h->H = height, h->pitch = (width + 15) & ~15, h->max_blocks = max_blocks, h->cap = max_corners_per_block, h->roi_cap = max_roi_pixels;
    h->device = device;
    h->own_stream = stream == nullptr;
    if (stream)
        h->stream = (cudaStream_t) stream;
    else
        ICG_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    ICG_CUDA(cudaMalloc(&h->d_img, (size_t) h->pitch * height));
    ICG_CUDA(cudaMalloc(&h->d_mask, (size_t) h->pitch * height));
    ICG_CUDA(cudaMalloc(&h->d_rois, sizeof(DetRect) * max_blocks));
    ICG_CUDA(cudaMalloc(&h->d_maxc, sizeof(int) * max_blocks));
    ICG_CUDA(cudaMalloc(&h->d_ncand, sizeof(int) * (2 * max_blocks + 2)));
    h->d_out_n = h->d_ncand + max_blocks;
    h->d_overflow = h->d_ncand + 2 * max_blocks;
    ICG_CUDA(cudaMalloc(&h->d_maxkey, sizeof(unsigned int) * max_blocks));
    ICG_CUDA(cudaMalloc(&h->d_eig, sizeof(float) * (size_t) max_blocks * max_roi_pixels));
    ICG_CUDA(cudaMalloc(&h->d_out_xy, sizeof(float) * 2 * (size_t) max_blocks * max_corners_per_block));
    ICG_CUDA(cudaMalloc(&h->d_cand, sizeof(unsigned long long) * (size_t) max_blocks * DET_MAX_CAND));
    h->h_stage_bytes = sizeof(DetRect) * max_blocks + sizeof(int) * (3 * max_blocks + 4) + sizeof(float) * 2 * (size_t) max_blocks * max_corners_per_block;
    ICG_CUDA(cudaMallocHost(&h->h_stage, h->h_stage_bytes));
    ICG_CUDA(raise_dynamic_smem((const void *) detect_select, (size_t) ((sizeof(unsigned long long) * DET_MAX_CAND))));
    *out = h;
    return ICG_OK;
}

void icg_detect_destroy(icg_detect *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    cudaFree(h->d_img), cudaFree(h->d_mask), cudaFree(h->d_rois), cudaFree(h->d_maxc), cudaFree(h->d_ncand), cudaFree(h->d_maxkey), cudaFree(h->d_eig);
    cudaFree(h->d_out_xy), cudaFree(h->d_cand);
    cudaFree(h->d_planes), cudaFree(h->d_fpar), cudaFree(h->d_fout_xy), cudaFree(h->d_pts);
    if (h->stage_ev) cudaEventDestroy(h->stage_ev);
    cudaFreeHost(h->h_stage);
    if (h->own_stream) cudaStreamDestroy(h->stream);
    delete h;
}

// goodFeaturesToTrack on every block: eig map, threshold + NMS, sort + greedy min-distance selection
static void launch_select(const DetArgs &A, int n_blocks, int maxw, int maxh, cudaStream_t s) {
    detect_eig<<<dim3((maxw + ET_W - 1) / ET_W, (maxh + ET_H - 1) / ET_H, n_blocks), 256, 0, s>>>(A);
    detect_nms<<<dim3((maxw + 31) / 32, (maxh + 7) / 8, n_blocks), 256, 0, s>>>(A);
    detect_select<<<n_blocks, 1024, sizeof(unsigned long long) * DET_MAX_CAND, s>>>(A);
    count_launch(3);
}
// cornerSubPix(win (5,5), zeroZone (-1,-1), COUNT+EPS 20 / 0.01): eps squared (IG/tracking/tracking.cc:623-625,651)
static void launch_subpix(const DetArgs &A, int n_blocks, cudaStream_t s) {
    detect_subpix<<<dim3((A.cap + 3) / 4, n_blocks), 128, 0, s>>>(A, 5, 20, 0.01 * 0.01);
    count_launch();
}

static int stage_acquire(icg_detect *h) {
    if (h->stage_pending) ICG_CUDA(cudaEventSynchronize(h->stage_ev));
    h->stage_pending = false;
    return ICG_OK;
}

static int run_detect(icg_detect *h, const uint8_t *d_img, const uint8_t *d_mask, int n_blocks, const icg_rect *rois, const int32_t *max_corners, double quality,
                      double min_distance, int do_select, int do_subpix, int n_given, float *out_xy, int32_t *out_n, int pitch = 0, size_t frame_stride = 0,
                      int n_frames = 1) {
    // n_frames > 1: `rois` (n_blocks of them) apply to every frame; device block index = frame * n_blocks + roi
    const int rois_per_frame = n_blocks;
    n_blocks *= n_frames;
    if (int rc = stage_acquire(h)) return rc;
    DetRect *hr = (DetRect *) h->h_stage;
    int *hm = (int *) (hr + h->max_blocks);
    int *hn = hm + h->max_blocks;          // out_n (also input counts when !do_select)
    int *hov = hn + 2 * h->max_blocks;      // overflow flag
    float *hxy = (float *) (hov + 4);
    int maxw = 0, maxh = 0;
    for (int b = 0; b < n_blocks; b++) {
        const icg_rect &r = rois[b % rois_per_frame];
        if (r.w < 3 || r.h < 3 || r.x < 0 || r.y < 0 || r.x + r.w > h->W || r.y + r.h > h->H || (size_t) r.w * r.h > (size_t) h->roi_cap) {
            set_error("icg_detect: block %d ROI (%d,%d,%d,%d) outside the %dx%d frame or larger than max_roi_pixels", b, r.x, r.y, r.w, r.h, h->W, h->H);
            return ICG_EINVAL;
        }
        hr[b] = DetRect{r.x, r.y, r.w, r.h};
        hm[b] = max_corners ? max_corners[b] : h->cap;
        maxw = std::max(maxw, r.w), maxh = std::max(maxh, r.h);
    }
    cudaStream_t s = h->stream;
    ICG_CUDA(cudaMemcpyAsync(h->d_rois, hr, sizeof(DetRect) * n_blocks, cudaMemcpyHostToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(h->d_maxc, hm, sizeof(int) * n_blocks, cudaMemcpyHostToDevice, s));
    ICG_CUDA(cudaMemsetAsync(h->d_ncand, 0, sizeof(int) * (2 * h->max_blocks + 2), s));
    ICG_CUDA(cudaMemsetAsync(h->d_maxkey, 0, sizeof(unsigned int) * h->max_blocks, s));
    DetArgs A;
    A.img = d_img, A.mask = d_mask, A.W = h->W, A.H = h->H, A.pitch = pitch ? pitch : h->pitch, A.n_blocks = n_blocks, A.cap = h->cap, A.roi_cap = h->roi_cap;
    A.img_stride = frame_stride, A.bpf = rois_per_frame, A.mask_stride = frame_stride, A.mask_pitch = A.pitch;
    A.rois = h->d_rois, A.max_corners = h->d_maxc, A.eig = h->d_eig, A.maxkey = h->d_maxkey, A.cand = h->d_cand, A.ncand = h->d_ncand;
    A.out_xy = h->d_out_xy, A.out_n = h->d_out_n, A.overflow = h->d_overflow, A.quality = quality, A.min_distance = min_distance;
    if (do_select) {
        launch_select(A, n_blocks, maxw, maxh, s);
    } else {
        // corners supplied by the caller (cv::cornerSubPix drop-in): out_xy holds n_given points of block 0
        memcpy(hxy, out_xy, sizeof(float) * 2 * n_given);
        hn[0] = n_given;
        ICG_CUDA(cudaMemcpyAsync(h->d_out_xy, hxy, sizeof(float) * 2 * n_given, cudaMemcpyHostToDevice, s));
        ICG_CUDA(cudaMemcpyAsync(h->d_out_n, hn, sizeof(int), cudaMemcpyHostToDevice, s));
    }
    if (do_subpix) launch_subpix(A, n_blocks, s);
    ICG_CHECK_LAUNCH();
    ICG_CUDA(cudaMemcpyAsync(hn, h->d_out_n, sizeof(int) * n_blocks, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaMemcpyAsync(hov, h->d_overflow, sizeof(int), cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaMemcpyAsync(hxy, h->d_out_xy, sizeof(float) * 2 * (size_t) n_blocks * h->cap, cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    if (*hov) {
        set_error("icg_detect: internal capacity exceeded (code %d: 1 = more than %d NMS candidates in a block, 2 = min-distance grid too fine, 3 = cell overflow)", *hov,
                  DET_MAX_CAND);
        return ICG_EUNSUPPORTED;
    }
    for (int b = 0; b < n_blocks; b++) {
        if (out_n) out_n[b] = hn[b];
        memcpy(out_xy + (size_t) b * h->cap * 2, hxy + (size_t) b * h->cap * 2, sizeof(float) * 2 * hn[b]);
    }
    return ICG_OK;
}

int icg_detect_blocks(icg_detect *h, const uint8_t *img, const uint8_t *mask, int stride, int n_blocks, const icg_rect *rois, const int32_t *max_corners,
                      double quality, double min_distance, int do_subpix, float *out_xy, int32_t *out_n) {
    if (!h || !img || !rois || !out_xy || !out_n || n_blocks < 1 || n_blocks > h->max_blocks || stride < h->W) {
        set_error("icg_detect_blocks: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaMemcpy2DAsync(h->d_img, h->pitch, img, stride, h->W, h->H, cudaMemcpyHostToDevice, h->stream));
    if (mask) ICG_CUDA(cudaMemcpy2DAsync(h->d_mask, h->pitch, mask, stride, h->W, h->H, cudaMemcpyHostToDevice, h->stream));
    return run_detect(h, h->d_img, mask ? h->d_mask : nullptr, n_blocks, rois, max_corners, quality, min_distance, 1, do_subpix, 0, out_xy, out_n);
}

int icg_detect_blocks_dev(icg_detect *h, int n_frames, const uint8_t *dev_img, int pitch, size_t frame_stride, const uint8_t *dev_mask, int n_blocks,
                          const icg_rect *rois, const int32_t *max_corners, double quality, double min_distance, int do_subpix, float *out_xy, int32_t *out_n) {
    if (!h || !dev_img || !rois || !out_xy || !out_n || n_frames < 1 || n_blocks < 1 || (long long) n_frames * n_blocks > h->max_blocks || pitch < h->W) {
        set_error("icg_detect_blocks_dev: bad arguments (n_frames * n_blocks must be <= max_blocks of the handle)");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    return run_detect(h, dev_img, dev_mask, n_blocks, rois, max_corners, quality, min_distance, 1, do_subpix, 0, out_xy, out_n, pitch, frame_stride, n_frames);
}

// ------------------------------------------------------------------------------------------------ featuresDetection from point lists
// The block grid of Tracking::Tracking (IG/tracking/tracking.cc:66-85) for a W x H frame and track_max_features_ = max_features.
struct FeatGrid {
    int cols, rows, bw, bh, nb, quota, min_dist;
};
static bool feat_grid(int W, int H, int max_features, FeatGrid &g) {
    g.cols = (int) lround(W / 200.0), g.rows = (int) lround(H / 200.0);
    if (g.cols < 1 || g.rows < 1 || max_features < 1) return false;
    g.bw = W / g.cols, g.bh = H / g.rows, g.nb = g.cols * g.rows;
    g.quota = (int) lround((double) max_features / (double) g.nb);
    if (g.quota < 1) return false;
    g.min_dist = (int) round(200.0 / sqrt(g.quota * 1.5));
    return true;
}

// one-time allocation of the feature path's buffers; the mask planes are sized for the max_blocks / nb frames a call can hold
static int features_alloc(icg_detect *h, int nb) {
    if (!h->d_planes) {
        const int n_planes = h->max_blocks / nb;
        const size_t plane = (size_t) h->pitch * h->H;
        if (cudaMalloc(&h->d_planes, plane * n_planes) != cudaSuccess) {
            cudaGetLastError();
            h->d_planes = nullptr;
            set_error("icg_detect_features: cannot allocate %d occupancy mask planes (%zu bytes)", n_planes, plane * n_planes);
            return ICG_ENOMEM;
        }
        h->n_planes = n_planes;
    }
    if (!h->d_fpar) {
        ICG_CUDA(cudaMalloc(&h->d_fpar, sizeof(int) * (size_t) (6 * h->max_blocks + 2)));
        h->d_skipped = h->d_fpar + 4 * h->max_blocks + 2;
        h->d_fout_n = h->d_skipped + h->max_blocks;
    }
    if (!h->d_fout_xy) ICG_CUDA(cudaMalloc(&h->d_fout_xy, sizeof(float) * 2 * (size_t) h->max_blocks * h->cap));
    if (!h->stage_ev) ICG_CUDA(cudaEventCreateWithFlags(&h->stage_ev, cudaEventDisableTiming));
    return ICG_OK;
}

static bool offsets_ok(const int32_t *off, int n) {
    if (!off || off[0] < 0) return false;
    for (int f = 0; f < n; f++)
        if (off[f + 1] < off[f]) return false;
    return true;
}

// gate + counts + mask (detect_occupancy) -> the existing block detection with the deficits as max_corners and the planes as mask ->
// detect_compact.  Asynchronous: the per-frame parameters go through h_stage, fenced by stage_ev.
static int run_features(icg_detect *h, int n_frames, const uint8_t *d_img, int pitch, size_t frame_stride, const float *a_xy, const uint8_t *a_st,
                        const int32_t *a_off, const float *b_xy, const uint8_t *b_st, const int32_t *b_off, const int32_t *n_ref, const uint8_t *ismask,
                        int max_features, float *out_xy, int32_t *out_n) {
    FeatGrid g;
    if (!feat_grid(h->W, h->H, max_features, g)) {
        set_error("icg_detect_features: no block grid for a %dx%d frame and max_features %d", h->W, h->H, max_features);
        return ICG_EINVAL;
    }
    if (g.quota > h->cap) {
        set_error("icg_detect_features: per-block quota %d exceeds max_corners_per_block %d of the handle", g.quota, h->cap);
        return ICG_EINVAL;
    }
    if ((long long) n_frames * g.nb > h->max_blocks || g.nb > DET_OCC_MAX_BLOCKS) {
        set_error("icg_detect_features: %d frames x %d blocks exceed max_blocks %d of the handle", n_frames, g.nb, h->max_blocks);
        return ICG_EINVAL;
    }
    if (!offsets_ok(a_off, n_frames) || !offsets_ok(b_off, n_frames)) {
        set_error("icg_detect_features: point-list offsets must start at >= 0 and be non-decreasing");
        return ICG_EINVAL;
    }
    if ((a_off[n_frames] > 0 && !a_xy) || (b_off[n_frames] > 0 && !b_xy)) {
        set_error("icg_detect_features: a non-empty point list without coordinates");
        return ICG_EINVAL;
    }
    const int n_blocks = n_frames * g.nb;
    int maxw = 0, maxh = 0;
    std::vector<DetRect> rois(g.nb);
    for (int k = 0; k < g.nb; k++) {  // tracking.cc:631-645: every block but the last is shrunk by 5 px
        const int c = k % g.cols, r = k / g.cols, shrink = k != g.nb - 1 ? 5 : 0;
        rois[k] = DetRect{c * g.bw, r * g.bh, g.bw - shrink, g.bh - shrink};
        if (rois[k].w < 3 || rois[k].h < 3 || (size_t) rois[k].w * rois[k].h > (size_t) h->roi_cap) {
            set_error("icg_detect_features: block %d (%dx%d) is smaller than 3x3 or larger than max_roi_pixels %d", k, rois[k].w, rois[k].h, h->roi_cap);
            return ICG_EINVAL;
        }
        maxw = std::max(maxw, rois[k].w), maxh = std::max(maxh, rois[k].h);
    }
    if (int rc = features_alloc(h, g.nb)) return rc;
    if (int rc = stage_acquire(h)) return rc;
    DetRect *hr = (DetRect *) h->h_stage;
    int *hp = (int *) (hr + h->max_blocks);  // [a_off n+1][b_off n+1][n_ref n][ismask n]: 4 * max_blocks + 2 ints fit the staging buffer
    for (int b = 0; b < n_blocks; b++) hr[b] = rois[b % g.nb];
    for (int f = 0; f <= n_frames; f++) hp[f] = a_off[f], hp[n_frames + 1 + f] = b_off[f];
    for (int f = 0; f < n_frames; f++) hp[2 * n_frames + 2 + f] = n_ref ? n_ref[f] : -1, hp[3 * n_frames + 2 + f] = ismask ? ismask[f] != 0 : 1;
    cudaStream_t s = h->stream;
    ICG_CUDA(cudaMemcpyAsync(h->d_rois, hr, sizeof(DetRect) * n_blocks, cudaMemcpyHostToDevice, s));
    ICG_CUDA(cudaMemcpyAsync(h->d_fpar, hp, sizeof(int) * (4 * n_frames + 2), cudaMemcpyHostToDevice, s));
    ICG_CUDA(cudaEventRecord(h->stage_ev, s));
    h->stage_pending = true;
    ICG_CUDA(cudaMemsetAsync(h->d_ncand, 0, sizeof(int) * (2 * h->max_blocks + 2), s));
    ICG_CUDA(cudaMemsetAsync(h->d_maxkey, 0, sizeof(unsigned int) * h->max_blocks, s));

    OccArgs O;
    O.a_xy = a_xy, O.b_xy = b_xy, O.a_st = a_st, O.b_st = b_st;
    O.a_off = h->d_fpar, O.b_off = h->d_fpar + n_frames + 1, O.n_ref = h->d_fpar + 2 * n_frames + 2, O.ismask = h->d_fpar + 3 * n_frames + 2;
    O.mask = h->d_planes, O.mask_stride = (size_t) h->pitch * h->H, O.mask_pitch = h->pitch, O.W = h->W, O.H = h->H;
    O.rows_per_cta = std::max(1, std::min(16, 16384 / h->pitch));
    O.cols = g.cols, O.nb = g.nb, O.bw = g.bw, O.bh = g.bh, O.quota = g.quota, O.radius = g.min_dist, O.gate_max = max_features - 5;
    O.max_corners = h->d_maxc, O.skipped = h->d_skipped;
    const size_t smem = (size_t) O.rows_per_cta * h->pitch;
    if (smem > 48 * 1024) ICG_CUDA(raise_dynamic_smem((const void *) detect_occupancy, smem));
    detect_occupancy<<<dim3((h->H + O.rows_per_cta - 1) / O.rows_per_cta, n_frames), 256, smem, s>>>(O);
    count_launch();

    DetArgs A;
    A.img = d_img, A.mask = h->d_planes, A.W = h->W, A.H = h->H, A.pitch = pitch, A.n_blocks = n_blocks, A.cap = h->cap, A.roi_cap = h->roi_cap;
    A.img_stride = frame_stride, A.bpf = g.nb, A.mask_stride = O.mask_stride, A.mask_pitch = h->pitch;
    A.rois = h->d_rois, A.max_corners = h->d_maxc, A.eig = h->d_eig, A.maxkey = h->d_maxkey, A.cand = h->d_cand, A.ncand = h->d_ncand;
    A.out_xy = h->d_out_xy, A.out_n = h->d_out_n, A.overflow = h->d_overflow, A.quality = 0.01, A.min_distance = (double) g.min_dist;  // tracking.cc:647
    launch_select(A, n_blocks, maxw, maxh, s);
    launch_subpix(A, n_blocks, s);
    detect_compact<<<n_frames, 256, 0, s>>>(A, h->d_skipped, g.nb, g.quota, out_xy, out_n);
    count_launch();
    ICG_CHECK_LAUNCH();
    return ICG_OK;
}

int icg_detect_features(icg_detect *h, const uint8_t *img, int stride, const float *feat_xy, int n_feat, const float *new_xy, int n_new, int n_ref, int ismask,
                        int max_features, float *out_xy, int32_t *out_n) {
    if (!h || !img || !out_xy || !out_n || stride < h->W || n_feat < 0 || n_new < 0 || (n_feat && !feat_xy) || (n_new && !new_xy)) {
        set_error("icg_detect_features: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaStreamSynchronize(h->stream));  // the point buffer may be reallocated below
    const size_t n_pts = (size_t) n_feat + n_new;
    if (n_pts > h->pts_cap) {
        cudaFree(h->d_pts);
        h->d_pts = nullptr, h->pts_cap = 0;
        ICG_CUDA(cudaMalloc(&h->d_pts, sizeof(float) * 2 * std::max<size_t>(n_pts, 1024)));
        h->pts_cap = std::max<size_t>(n_pts, 1024);
    }
    cudaStream_t s = h->stream;
    ICG_CUDA(cudaMemcpy2DAsync(h->d_img, h->pitch, img, stride, h->W, h->H, cudaMemcpyHostToDevice, s));
    if (n_feat) ICG_CUDA(cudaMemcpyAsync(h->d_pts, feat_xy, sizeof(float) * 2 * n_feat, cudaMemcpyHostToDevice, s));
    if (n_new) ICG_CUDA(cudaMemcpyAsync(h->d_pts + 2 * (size_t) n_feat, new_xy, sizeof(float) * 2 * n_new, cudaMemcpyHostToDevice, s));
    const int32_t a_off[2] = {0, n_feat}, b_off[2] = {0, n_new}, nr = n_ref;
    const uint8_t im = ismask != 0;
    FeatGrid g;
    if (feat_grid(h->W, h->H, max_features, g) && g.nb <= h->max_blocks) {  // the output buffers below must exist before they are passed
        if (int rc = features_alloc(h, g.nb)) return rc;
    }
    if (int rc = run_features(h, 1, h->d_img, h->pitch, 0, h->d_pts, nullptr, a_off, h->d_pts + 2 * (size_t) n_feat, nullptr, b_off, &nr, &im, max_features,
                              h->d_fout_xy, h->d_fout_n))
        return rc;
    int32_t n = 0;
    ICG_CUDA(cudaMemcpyAsync(&n, h->d_fout_n, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    ICG_CUDA(cudaStreamSynchronize(s));
    if (n == -2) {
        set_error("icg_detect_features: internal capacity exceeded (more than %d NMS candidates in a block, or a min-distance grid too fine)", DET_MAX_CAND);
        return ICG_EUNSUPPORTED;
    }
    if (n > 0) ICG_CUDA(cudaMemcpy(out_xy, h->d_fout_xy, sizeof(float) * 2 * n, cudaMemcpyDeviceToHost));
    *out_n = n;
    return ICG_OK;
}

int icg_detect_features_dev(icg_detect *h, int n_frames, const uint8_t *dev_img, int pitch, size_t frame_stride, const float *dev_feat_xy,
                            const uint8_t *dev_feat_status, const int32_t *feat_off, const float *dev_new_xy, const uint8_t *dev_new_status,
                            const int32_t *new_off, const int32_t *n_ref, const uint8_t *ismask, int max_features, float *dev_out_xy, int32_t *dev_out_n) {
    if (!h || !dev_img || !dev_out_xy || !dev_out_n || n_frames < 1 || pitch < h->W || !feat_off || !new_off) {
        set_error("icg_detect_features_dev: bad arguments");
        return ICG_EINVAL;
    }
    ICG_CUDA(cudaSetDevice(h->device));
    return run_features(h, n_frames, dev_img, pitch, frame_stride, dev_feat_xy, dev_feat_status, feat_off, dev_new_xy, dev_new_status, new_off, n_ref,
                        ismask, max_features, dev_out_xy, dev_out_n);
}

int icg_detect_mask_dev(icg_detect *h, int frame, void **dev_ptr, int *pitch) {
    if (!h || !dev_ptr || !pitch || !h->d_planes || frame < 0 || frame >= h->n_planes) {
        set_error("icg_detect_mask_dev: bad arguments (no icg_detect_features call yet, or frame out of range)");
        return ICG_EINVAL;
    }
    *dev_ptr = h->d_planes + (size_t) frame * h->pitch * h->H;
    *pitch = h->pitch;
    return ICG_OK;
}

int icg_corner_subpix(icg_detect *h, const uint8_t *img, int stride, float *corners_xy, int n) {
    if (!h || !img || !corners_xy || n < 0 || n > h->cap || stride < h->W) {
        set_error("icg_corner_subpix: bad arguments (n must be <= max_corners_per_block of the handle)");
        return ICG_EINVAL;
    }
    if (n == 0) return ICG_OK;
    ICG_CUDA(cudaSetDevice(h->device));
    ICG_CUDA(cudaMemcpy2DAsync(h->d_img, h->pitch, img, stride, h->W, h->H, cudaMemcpyHostToDevice, h->stream));
    icg_rect full = {0, 0, h->W, h->H};
    int32_t cnt = 0;
    if ((size_t) h->W * h->H > (size_t) h->roi_cap) {
        // the eig plane is not needed for sub-pixel refinement; only the ROI geometry is
    }
    // run_detect validates roi_cap against w*h; sub-pixel refinement does not touch the eig plane, so bypass that check
    int saved = h->roi_cap;
    h->roi_cap = h->W * h->H;
    int rc = run_detect(h, h->d_img, nullptr, 1, &full, nullptr, 0.0, 0.0, 0, 1, n, corners_xy, &cnt);
    h->roi_cap = saved;
    return rc;
}

}  // extern "C"
