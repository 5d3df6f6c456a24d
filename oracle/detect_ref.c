/*
 * oracle/detect_ref.c -- CPU restatement (TEST INFRASTRUCTURE ONLY) of the OpenCV routines behind
 * Tracking::featuresDetection (ic_gvins/ic_gvins/tracking/tracking.cc:576-688):
 *
 *   cv::goodFeaturesToTrack(block_image, out, n, 0.01, track_min_pixel_distance_, block_mask)     tracking.cc:647
 *   cv::cornerSubPix(block_image, out, Size(5,5), Size(-1,-1), TermCriteria(COUNT+EPS, 20, 0.01))   tracking.cc:651
 *
 * block_image / block_mask are ROI views of the frame (tracking.cc:644-645).  OpenCV (un-vendored; pinned here to
 * opencv-python-headless 4.13.0) evaluates the Sobel derivative of an ROI with the PARENT image's pixels beyond the ROI
 * edge, but box-filters the (ROI-sized, freshly allocated) covariance image with reflect-101 at the ROI edge;
 * cornerSubPix samples the ROI alone, through getRectSubPix's edge rule (icgo_rect_subpix: replicate, except at the
 * top-right corner).  The min-eigenvalue maps and corner lists are bit-exact against cv2 and getRectSubPix patches are
 * bit-exact; sub-pixel positions agree to 1e-3 px (tests/golden/make_detect_golden.py, make_detect_edges_golden.py,
 * SURVEY.md Appendix A.4/A.5).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline int reflect101i(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
    return p;
}

/* cv::Sobel(src, CV_32F, 1, 0, 3, scale) / (0, 1): scale = 1 / (4 * 3 * 255) folded into the smoothing kernel [s, 2s, s].
 * dx = fmaf(top + bot, s, 2s * mid)          (column pass, top/mid/bot = exact horizontal differences)
 * dy = row(y+1) - row(y-1), row = fmaf(R, s, fmaf(C, 2s, s * L))   (row pass on the u8 source)                     */
static inline float pix(const uint8_t *img, int W, int H, int stride, int x, int y) {
    return (float) img[(size_t) reflect101i(y, H) * stride + reflect101i(x, W)];
}
/* fma_row: OpenCV's AVX2 row filter (u8 -> f32) handles 32 pixels per iteration with FMA; the remaining (roi_width % 32)
 * columns of every row go through the scalar loop, which rounds each product and sum separately (measured against cv2). */
static void sobel_at(const uint8_t *img, int W, int H, int stride, int x, int y, int fma_row, float *dx, float *dy) {
    const float s = (float) (1.0 / (4 * 3 * 255.0)), s2 = (float) (2.0 * (1.0 / (4 * 3 * 255.0)));
    float top = pix(img, W, H, stride, x + 1, y - 1) - pix(img, W, H, stride, x - 1, y - 1);
    float mid = pix(img, W, H, stride, x + 1, y) - pix(img, W, H, stride, x - 1, y);
    float bot = pix(img, W, H, stride, x + 1, y + 1) - pix(img, W, H, stride, x - 1, y + 1);
    *dx = fmaf(top + bot, s, s2 * mid);
    float lm = pix(img, W, H, stride, x - 1, y - 1), cm = pix(img, W, H, stride, x, y - 1), rm = pix(img, W, H, stride, x + 1, y - 1);
    float lp = pix(img, W, H, stride, x - 1, y + 1), cp = pix(img, W, H, stride, x, y + 1), rp = pix(img, W, H, stride, x + 1, y + 1);
    float rowm, rowp;
    if (fma_row) {
        rowm = fmaf(rm, s, fmaf(cm, s2, s * lm));
        rowp = fmaf(rp, s, fmaf(cp, s2, s * lp));
    } else {
        rowm = (s * lm + s2 * cm) + s * rm;
        rowp = (s * lp + s2 * cp) + s * rp;
    }
    *dy = rowp - rowm;
}

/* cv::cornerMinEigenVal(roi, eig, blockSize 3, ksize 3) for the ROI (x0, y0, w, h) of the W x H frame. */
void icgo_min_eig_roi(const uint8_t *img, int W, int H, int stride, int x0, int y0, int w, int h, float *eig /* h*w */) {
    float *xx = (float *) malloc(sizeof(float) * (size_t) w * h), *xy = (float *) malloc(sizeof(float) * (size_t) w * h),
          *yy = (float *) malloc(sizeof(float) * (size_t) w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float dx, dy;
            sobel_at(img, W, H, stride, x0 + x, y0 + y, x < (w & ~31), &dx, &dy);
            xx[(size_t) y * w + x] = dx * dx;
            xy[(size_t) y * w + x] = dx * dy;
            yy[(size_t) y * w + x] = dy * dy;
        }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            double sa = 0, sb = 0, sc = 0; /* unnormalised 3x3 box, f64 accumulation, reflect-101 at the ROI edge */
            for (int j = -1; j <= 1; j++)
                for (int i = -1; i <= 1; i++) {
                    size_t o = (size_t) reflect101i(y + j, h) * w + reflect101i(x + i, w);
                    sa += xx[o], sb += xy[o], sc += yy[o];
                }
            float a = (float) sa * 0.5f, b = (float) sb, c = (float) sc * 0.5f;
            eig[(size_t) y * w + x] = (float) ((a + c) - sqrtf((a - c) * (a - c) + b * b));
        }
    free(xx), free(xy), free(yy);
}

typedef struct {
    float v;
    int addr;
} cand_t;
static int cand_cmp(const void *pa, const void *pb) {
    const cand_t *a = (const cand_t *) pa, *b = (const cand_t *) pb;
    if (a->v > b->v) return -1;
    if (a->v < b->v) return 1;
    return a->addr > b->addr ? -1 : (a->addr < b->addr ? 1 : 0); /* greaterThanPtr: ties by address, descending */
}

/* cv::goodFeaturesToTrack tail on a precomputed eig map of the ROI (w x h); mask = ROI view (stride mstride) or NULL.
 * Returns the number of corners written to out_xy (ROI-local coordinates, acceptance order). */
int icgo_good_features_from_eig(const float *eig_in, int w, int h, const uint8_t *mask, int mstride, int max_corners, double quality, double min_distance,
                                float *out_xy) {
    float *eig = (float *) malloc(sizeof(float) * (size_t) w * h);
    memcpy(eig, eig_in, sizeof(float) * (size_t) w * h);
    double maxVal = 0; /* minMaxLoc(eig, 0, &maxVal, 0, 0, mask) */
    int any = 0;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++)
            if (!mask || mask[(size_t) y * mstride + x]) {
                if (!any || eig[(size_t) y * w + x] > maxVal) maxVal = eig[(size_t) y * w + x], any = 1;
            }
    if (!any) maxVal = 0;
    const float thr = (float) (maxVal * quality); /* threshold(eig, eig, maxVal*quality, 0, THRESH_TOZERO) */
    for (size_t i = 0; i < (size_t) w * h; i++)
        if (!(eig[i] > thr)) eig[i] = 0;
    cand_t *cand = (cand_t *) malloc(sizeof(cand_t) * (size_t) w * h);
    int nc = 0;
    for (int y = 1; y < h - 1; y++)
        for (int x = 1; x < w - 1; x++) {
            float val = eig[(size_t) y * w + x];
            if (val == 0) continue;
            float mx = val; /* dilate 3x3 */
            for (int j = -1; j <= 1; j++)
                for (int i = -1; i <= 1; i++) {
                    float v = eig[(size_t) (y + j) * w + x + i];
                    if (v > mx) mx = v;
                }
            if (val == mx && (!mask || mask[(size_t) y * mstride + x])) cand[nc].v = val, cand[nc].addr = y * w + x, nc++;
        }
    qsort(cand, nc, sizeof(cand_t), cand_cmp);
    int n_out = 0;
    if (min_distance >= 1) {
        const int cell = (int) lrint(min_distance);
        const int gw = (w + cell - 1) / cell, gh = (h + cell - 1) / cell;
        const double md2 = min_distance * min_distance;
        int *cnt = (int *) calloc((size_t) gw * gh, sizeof(int));
        float *gpts = (float *) malloc(sizeof(float) * 2 * (size_t) gw * gh * 64);
        for (int i = 0; i < nc; i++) {
            int y = cand[i].addr / w, x = cand[i].addr - y * w;
            int xc = x / cell, yc = y / cell;
            int x1 = xc - 1 < 0 ? 0 : xc - 1, y1 = yc - 1 < 0 ? 0 : yc - 1, x2 = xc + 1 > gw - 1 ? gw - 1 : xc + 1, y2 = yc + 1 > gh - 1 ? gh - 1 : yc + 1;
            int good = 1;
            for (int yy = y1; yy <= y2 && good; yy++)
                for (int xx = x1; xx <= x2 && good; xx++)
                    for (int k = 0; k < cnt[yy * gw + xx]; k++) {
                        float dx = (float) x - gpts[((size_t) (yy * gw + xx) * 64 + k) * 2], dy = (float) y - gpts[((size_t) (yy * gw + xx) * 64 + k) * 2 + 1];
                        if (dx * dx + dy * dy < md2) {
                            good = 0;
                            break;
                        }
                    }
            if (good) {
                int c = yc * gw + xc;
                if (cnt[c] < 64) gpts[((size_t) c * 64 + cnt[c]) * 2] = (float) x, gpts[((size_t) c * 64 + cnt[c]) * 2 + 1] = (float) y, cnt[c]++;
                out_xy[2 * n_out] = (float) x, out_xy[2 * n_out + 1] = (float) y;
                n_out++;
                if (max_corners > 0 && n_out == max_corners) break;
            }
        }
        free(cnt), free(gpts);
    } else {
        for (int i = 0; i < nc; i++) {
            int y = cand[i].addr / w, x = cand[i].addr - y * w;
            out_xy[2 * n_out] = (float) x, out_xy[2 * n_out + 1] = (float) y;
            n_out++;
            if (max_corners > 0 && n_out == max_corners) break;
        }
    }
    free(cand), free(eig);
    return n_out;
}

/* cv::getRectSubPix(src, Size(n, n), (cx, cy), patch, CV_32F) of the w x h u8 image src (row stride `stride`), centres inside
 * the image.  Window pixel (i, j) samples src at (ipx + j + a, ipy + i + b), (ipx, ipy) = floor of the window's top-left corner
 * (cx, cy) - (n - 1) / 2 and (a, b) its fraction.  The float sequence below matches cv2 4.13.0 bit for bit, inside the image
 * and at its edges (tests/golden/make_detect_edges_golden.py):
 *  - both sample columns x, x + 1 and both sample rows y, y + 1 in the image: (s00 * a11 + s01 * a12) + (s10 * a21 + s11 * a22);
 *  - window rows above the image or at / below its last row (the row clamped to [0, h - 1]): fmaf(s01, a, s00 * (1 - a));
 *  - a column left of 0 or at / right of w - 1: (1 - b) * src(c, Y0) + b * src(c, Y1) of one edge column c, which is 0 on the
 *    left and w - 1 on the right, except in window rows above the image (ipy + i < 0), where cv2 reads column w - 2 on the
 *    right: it does not replicate at the top-right corner. */
void icgo_rect_subpix(const uint8_t *src, int w, int h, int stride, float cx, float cy, int n, float *dst) {
    const float x0 = cx - (n - 1) * 0.5f, y0 = cy - (n - 1) * 0.5f;
    const int ipx = (int) floorf(x0), ipy = (int) floorf(y0);
    const float a = x0 - ipx, b = y0 - ipy;
    const float a11 = (1.f - a) * (1.f - b), a12 = a * (1.f - b), a21 = (1.f - a) * b, a22 = a * b, b1 = 1.f - b, b2 = b;
    for (int i = 0; i < n; i++) {
        const int y = ipy + i, Y0 = y < 0 ? 0 : (y > h - 1 ? h - 1 : y), Y1 = y + 1 < 0 ? 0 : (y + 1 > h - 1 ? h - 1 : y + 1);
        const uint8_t *r0 = src + (size_t) Y0 * stride, *r1 = src + (size_t) Y1 * stride;
        for (int j = 0; j < n; j++) {
            const int x = ipx + j;
            if (x < 0 || x >= w - 1) {
                const int c = x < 0 ? 0 : (y < 0 ? w - 2 : w - 1);
                dst[i * n + j] = (float) r0[c] * b1 + (float) r1[c] * b2;
            } else if (Y0 == Y1) {
                dst[i * n + j] = fmaf((float) r0[x + 1], a, (float) r0[x] * (1.f - a));
            } else {
                dst[i * n + j] = ((float) r0[x] * a11 + (float) r0[x + 1] * a12) + ((float) r1[x] * a21 + (float) r1[x + 1] * a22);
            }
        }
    }
}

/* cv::cornerSubPix(roi, corners, win (5,5), zeroZone (-1,-1), (COUNT+EPS, max_iter, eps)) on the ROI (x0,y0,w,h):
 * cornerSubPix reads nothing outside its input, so the ROI behaves as a w x h image sampled by icgo_rect_subpix.  An iterate
 * outside the ROI ends the loop and is discarded: the corner keeps the last iterate inside it.  corners in ROI-local
 * coordinates, refined in place. */
void icgo_corner_subpix_roi(const uint8_t *img, int W, int H, int stride, int x0, int y0, int w, int h, float *xy, int n, int half_win, int max_iter, double eps) {
    (void) W, (void) H;
    const int win_w = 2 * half_win + 1, sw = win_w + 2;
    float *maskw = (float *) malloc(sizeof(float) * win_w * win_w), *sub = (float *) malloc(sizeof(float) * sw * sw);
    float *mx = (float *) malloc(sizeof(float) * win_w);
    for (int i = 0; i < win_w; i++) {
        float t = (float) (i - half_win) / half_win;
        mx[i] = expf(-t * t);
    }
    for (int i = 0; i < win_w; i++)
        for (int j = 0; j < win_w; j++) maskw[i * win_w + j] = mx[i] * mx[j]; /* mask[i][j] = vy * vx */
    if (max_iter < 0) max_iter = 0;
    if (max_iter > 100) max_iter = 100;
    if (eps < 0) eps = 0;
    const double eps2 = eps * eps;
    const uint8_t *roi = img + (size_t) y0 * stride + x0;
    for (int p = 0; p < n; p++) {
        float cTx = xy[2 * p], cTy = xy[2 * p + 1], cIx = cTx, cIy = cTy;
        int iter = 0;
        double err = 0;
        do {
            icgo_rect_subpix(roi, w, h, stride, cIx, cIy, sw, sub);
            double A = 0, Bm = 0, Cc = 0, bb1 = 0, bb2 = 0;
            for (int i = 0; i < win_w; i++) {
                double py = i - half_win;
                for (int j = 0; j < win_w; j++) {
                    double m = maskw[i * win_w + j];
                    const float *sp = sub + (i + 1) * sw + (j + 1);
                    double tgx = sp[1] - sp[-1], tgy = sp[sw] - sp[-sw];
                    double gxx = tgx * tgx * m, gxy = tgx * tgy * m, gyy = tgy * tgy * m;
                    double px = j - half_win;
                    A += gxx, Bm += gxy, Cc += gyy;
                    bb1 += gxx * px + gxy * py;
                    bb2 += gxy * px + gyy * py;
                }
            }
            double det = A * Cc - Bm * Bm;
            if (fabs(det) <= DBL_EPSILON * DBL_EPSILON) break;
            double scale = 1.0 / det;
            float nx = (float) (cIx + Cc * scale * bb1 - Bm * scale * bb2), ny = (float) (cIy - Bm * scale * bb1 + A * scale * bb2);
            err = (nx - cIx) * (nx - cIx) + (ny - cIy) * (ny - cIy); /* float arithmetic, as in cornersubpix.cpp */
            if (nx < 0 || nx >= w || ny < 0 || ny >= h) break;
            cIx = nx, cIy = ny;
        } while (++iter < max_iter && err > eps2);
        if (fabsf(cIx - cTx) > half_win || fabsf(cIy - cTy) > half_win) cIx = cTx, cIy = cTy;
        xy[2 * p] = cIx, xy[2 * p + 1] = cIy;
    }
    free(maskw), free(sub), free(mx);
}

/* One block of Tracking::featuresDetection (tracking.cc:627-656): goodFeaturesToTrack + cornerSubPix on an ROI. */
int icgo_detect_block(const uint8_t *img, const uint8_t *mask, int W, int H, int stride, int x0, int y0, int w, int h, int max_corners, double quality,
                      double min_distance, float *out_xy) {
    float *eig = (float *) malloc(sizeof(float) * (size_t) w * h);
    icgo_min_eig_roi(img, W, H, stride, x0, y0, w, h, eig);
    int n = icgo_good_features_from_eig(eig, w, h, mask ? mask + (size_t) y0 * stride + x0 : NULL, stride, max_corners, quality, min_distance, out_xy);
    free(eig);
    if (n > 0) icgo_corner_subpix_roi(img, W, H, stride, x0, y0, w, h, out_xy, n, 5, 20, 0.01);
    return n;
}
