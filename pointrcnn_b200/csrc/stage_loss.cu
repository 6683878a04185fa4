// stage_loss.cu -- the RPN and RCNN training losses (lib/net/train_functions.py:55-209 get_rpn_loss / get_rcnn_loss,
// lib/utils/loss_utils.py:7-233) and their gradients, for either stage through one forward and one backward entry:
//   forward   row pass     one thread per row: the classification term of every row and, for the foreground rows, every
//                          get_reg_loss term; float64 sums per CTA into a fixed grid of partial rows
//             final pass   one CTA: the partials summed in a fixed order, divided by the reference's normalisers, written
//                          as the loss vector (terms + the normalisers the backward reads)
//   backward  one CTA per 128 rows: d cls per row, d reg of the foreground rows built in shared memory and written densely
//             (zero rows included); the per-row derivatives are recomputed from the saved inputs
// No float atomics: the same inputs give the same bits.  The per-row arithmetic is fp32 in the order of the torch mirror
// (pointrcnn_b200/train/losses.py), with explicit _rn intrinsics where a bin label depends on it, and the derivatives are
// those torch autograd derives for that mirror, including its kinks (saturated BCE, clamp_min / abs at a logit of 0,
// min / max ties in the Dice loss).
#include <math_constants.h>

#include "common.cuh"

namespace prb {

constexpr int kSlThreads = 256;
constexpr int kSlMaxParts = 1024;     // partial-sum rows of the row pass (the grid never depends on the device)
constexpr int kSlTile = 128;          // rows per CTA of the backward
constexpr int kSlMaxK = 16;           // classes of the CrossEntropy variant
constexpr int kSlMaxCols = 256;       // regression channels

// float64 accumulators of the row pass
enum { A_POS, A_NEG, A_CLS, A_DMIN, A_DMAX, A_NPOS, A_NVALID, A_NFG, A_XB, A_ZB, A_XR, A_ZR, A_YB, A_YR, A_YO, A_RB, A_RR, A_SIZE,
       kSlAcc };
// per-term gradient scales of the backward
enum { K_CLS, K_POS, K_NEG, K_DMIN, K_DMAX, K_XB, K_ZB, K_XR, K_ZR, K_YB, K_YR, K_YO, K_RB, K_RR, K_SIZE, K_N };

struct SlCfg {
    int cls_loss, K, C, nloc, ny, nhb, xz_fine, y_by_bin, ry_fine, lab64, valid64;
    int off_y, off_ry, off_size;
    float alpha, alpha1, gamma, fg_weight, w_cls, w_reg;
    float loc_scope, loc_hi, loc_bin, loc_half;
    float y_scope, y_hi, y_bin, y_half;
    float per, per_half;
};

__device__ __forceinline__ long long sl_ld(const void *p, int is64, int i) {
    return is64 ? reinterpret_cast<const long long *>(p)[i] : (long long)reinterpret_cast<const int *>(p)[i];
}
__device__ __forceinline__ float sl_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
// Python's float %: the sign of the divisor
__device__ __forceinline__ float sl_pymod(float a, float b) {
    float m = fmodf(a, b);
    if (m != 0.f && ((b < 0.f) != (m < 0.f))) m += b;
    return m;
}
__device__ __forceinline__ float sl_smooth_l1(float d) {
    const float z = fabsf(d);
    return z < 1.f ? 0.5f * z * z : z - 0.5f;
}
// F.smooth_l1_loss backward (beta 1): the quadratic branch up to and including |d| = 1
__device__ __forceinline__ float sl_smooth_l1_grad(float d) { return d < -1.f ? -1.f : (d > 1.f ? 1.f : d); }

// -log_softmax(x)[y] over n logits (cross_entropy of one row); lse = max + log(sum exp(x - max))
__device__ __forceinline__ float sl_ce(const float *x, int n, int y, float &mx, float &ls) {
    mx = x[0];
    for (int k = 1; k < n; ++k) mx = fmaxf(mx, x[k]);
    float s = 0.f;
    for (int k = 0; k < n; ++k) s += expf(x[k] - mx);
    ls = logf(s);
    return -((x[y] - mx) - ls);
}
// its gradient, scaled by g, into d[0..n)
__device__ __forceinline__ void sl_ce_grad(const float *x, int n, int y, float g, float *d) {
    float mx, ls;
    sl_ce(x, n, y, mx, ls);
    for (int k = 0; k < n; ++k) d[k] = g * (expf((x[k] - mx) - ls) - (k == y ? 1.f : 0.f));
}

// the bin label and the residual target of one shifted coordinate: floor(shift / bin), (shift - (bin*b + half)) / half'
__device__ __forceinline__ int sl_bin(float shift, float bin, float half, float res_div, float &res) {
    const int b = (int)floorf(__fdiv_rn(shift, bin));
    res = __fdiv_rn(__fsub_rn(shift, __fadd_rn(__fmul_rn((float)b, bin), half)), res_div);
    return b;
}

struct SlLab {
    int xb, zb, yb, rb;
    float xr, zr, yr, y, rr, sz[3];
};

// get_reg_loss's labels of one foreground row (loss_utils.py:87-233)
__device__ __forceinline__ void sl_labels(const SlCfg &c, const float *lab, const float *anc, SlLab &L) {
    const float xs = fminf(fmaxf(__fadd_rn(lab[0], c.loc_scope), 0.f), c.loc_hi);
    const float zs = fminf(fmaxf(__fadd_rn(lab[2], c.loc_scope), 0.f), c.loc_hi);
    L.xb = sl_bin(xs, c.loc_bin, c.loc_half, c.loc_bin, L.xr);
    L.zb = sl_bin(zs, c.loc_bin, c.loc_half, c.loc_bin, L.zr);
    L.y = lab[1];
    L.yb = 0;
    L.yr = 0.f;
    if (c.y_by_bin) {
        const float ys = fminf(fmaxf(__fadd_rn(lab[1], c.y_scope), 0.f), c.y_hi);
        L.yb = sl_bin(ys, c.y_bin, c.y_half, c.y_bin, L.yr);
    }
    const float two_pi = (float)(2.0 * CUDART_PI);
    float shift;
    if (c.ry_fine) {       // fold into [0, pi): the opposite heading is the same box
        float r = sl_pymod(lab[6], two_pi);
        if (r > (float)(CUDART_PI * 0.5) && r < (float)(CUDART_PI * 1.5)) r = sl_pymod(__fadd_rn(r, (float)CUDART_PI), two_pi);
        shift = __fsub_rn(sl_pymod(__fadd_rn(r, (float)(CUDART_PI * 0.5)), two_pi), (float)(CUDART_PI * 0.25));
        shift = fminf(fmaxf(shift, 1e-3f), (float)(CUDART_PI * 0.5 - 1e-3));
    } else {
        shift = sl_pymod(__fadd_rn(sl_pymod(lab[6], two_pi), c.per_half), two_pi);
    }
    L.rb = sl_bin(shift, c.per, c.per_half, c.per_half, L.rr);
#pragma unroll
    for (int q = 0; q < 3; ++q) L.sz[q] = __fdiv_rn(__fsub_rn(lab[3 + q], anc[q]), anc[q]);
}

struct SlPtrs {
    const float *cls, *reg, *reg_label, *mean_size, *anchor_boxes, *ce_weight;
    const void *label, *valid;
};

__device__ __forceinline__ const float *sl_anchor(const SlPtrs &p, int i) {
    return p.anchor_boxes ? p.anchor_boxes + (size_t)i * 7 + 3 : p.mean_size;
}

template <int NW>
__device__ __forceinline__ void sl_block_sum(double (&a)[kSlAcc], double (*s_red)[kSlAcc]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < kSlAcc; ++j) {
        double v = a[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) s_red[warp][j] = v;
    }
    __syncthreads();
    if (threadIdx.x < kSlAcc) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < NW; ++w) v += s_red[w][threadIdx.x];
        a[0] = v;        // thread j < kSlAcc holds the CTA's sum of accumulator j in a[0]
    }
}

__global__ void __launch_bounds__(kSlThreads) stage_loss_rows_kernel(int rows, SlCfg c, SlPtrs p, double *__restrict__ parts) {
    __shared__ double s_red[kSlThreads / 32][kSlAcc];
    double a[kSlAcc];
#pragma unroll
    for (int j = 0; j < kSlAcc; ++j) a[j] = 0.0;
    for (int i = blockIdx.x * kSlThreads + threadIdx.x; i < rows; i += gridDim.x * kSlThreads) {
        const long long lab = sl_ld(p.label, c.lab64, i);
        const bool pos = lab > 0, valid = lab >= 0;
        a[A_NPOS] += pos;
        a[A_NVALID] += valid;
        if (c.cls_loss == PRB_LOSS_CE) {
            if (valid && lab < c.K) {
                float mx, ls;
                const float l = sl_ce(p.cls + (size_t)i * c.K, c.K, (int)lab, mx, ls);
                a[A_CLS] += (double)((p.ce_weight ? p.ce_weight[lab] : 1.f) * l);
            }
        } else {
            const float x = p.cls[i], t = pos ? 1.f : 0.f;
            if (c.cls_loss == PRB_LOSS_FOCAL) {
                if (valid) {
                    const float ce = fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
                    const float pr = sl_sigmoid(x);
                    const float b = 1.f - (t * pr + (1.f - t) * (1.f - pr));
                    const float mod = c.gamma == 0.f ? 1.f : (c.gamma == 2.f ? b * b : powf(b, c.gamma));
                    const float f = mod * (pos ? c.alpha : c.alpha1) * ce;
                    if (pos) a[A_POS] += (double)f;
                    else a[A_NEG] += (double)f;
                }
            } else if (c.cls_loss == PRB_LOSS_BCE) {
                if (valid) {
                    const float pr = sl_sigmoid(x);
                    const float l = (t - 1.f) * fmaxf(log1pf(-pr), -100.f) - t * fmaxf(logf(pr), -100.f);
                    a[A_CLS] += (double)(l * (pos ? c.fg_weight : 1.f));
                }
            } else {   // Dice: min / max of p and the label over the rows whose label is not -1
                if (lab != -1) {
                    const float pr = sl_sigmoid(x), tl = (float)lab;
                    a[A_DMIN] += (double)fminf(pr, tl);
                    a[A_DMAX] += (double)fmaxf(pr, tl);
                }
            }
        }
        const bool fg = p.valid ? sl_ld(p.valid, c.valid64, i) > 0 : pos;
        if (!fg) continue;
        a[A_NFG] += 1.0;
        SlLab L;
        sl_labels(c, p.reg_label + (size_t)i * 7, sl_anchor(p, i), L);
        const float *x = p.reg + (size_t)i * c.C;
        float mx, ls;
        a[A_XB] += (double)sl_ce(x, c.nloc, L.xb, mx, ls);
        a[A_ZB] += (double)sl_ce(x + c.nloc, c.nloc, L.zb, mx, ls);
        if (c.xz_fine) {
            a[A_XR] += (double)sl_smooth_l1(__fsub_rn(x[2 * c.nloc + L.xb], L.xr));
            a[A_ZR] += (double)sl_smooth_l1(__fsub_rn(x[3 * c.nloc + L.zb], L.zr));
        }
        if (c.y_by_bin) {
            a[A_YB] += (double)sl_ce(x + c.off_y, c.ny, L.yb, mx, ls);
            a[A_YR] += (double)sl_smooth_l1(__fsub_rn(x[c.off_y + c.ny + L.yb], L.yr));
        } else {
            a[A_YO] += (double)sl_smooth_l1(__fsub_rn(x[c.off_y], L.y));
        }
        a[A_RB] += (double)sl_ce(x + c.off_ry, c.nhb, L.rb, mx, ls);
        a[A_RR] += (double)sl_smooth_l1(__fsub_rn(x[c.off_ry + c.nhb + L.rb], L.rr));
#pragma unroll
        for (int q = 0; q < 3; ++q) a[A_SIZE] += (double)sl_smooth_l1(__fsub_rn(x[c.off_size + q], L.sz[q]));
    }
    sl_block_sum<kSlThreads / 32>(a, s_red);
    if (threadIdx.x < kSlAcc) parts[(size_t)blockIdx.x * kSlAcc + threadIdx.x] = a[0];
}

__global__ void __launch_bounds__(kSlThreads) stage_loss_final_kernel(int nparts, SlCfg c, const double *__restrict__ parts,
                                                                      float *__restrict__ total, float *__restrict__ out) {
    __shared__ double s_red[kSlThreads / 32][kSlAcc];
    __shared__ double s_sum[kSlAcc];
    double a[kSlAcc];
#pragma unroll
    for (int j = 0; j < kSlAcc; ++j) a[j] = 0.0;
    for (int b = threadIdx.x; b < nparts; b += kSlThreads) {
#pragma unroll
        for (int j = 0; j < kSlAcc; ++j) a[j] += parts[(size_t)b * kSlAcc + j];
    }
    sl_block_sum<kSlThreads / 32>(a, s_red);
    if (threadIdx.x < kSlAcc) s_sum[threadIdx.x] = a[0];
    __syncthreads();
    if (threadIdx.x != 0) return;
    const double *s = s_sum;
    const double P = fmax(s[A_NPOS], 1.0), V = fmax(s[A_NVALID], 1.0), F = s[A_NFG];
    double cls, norm = V, cpos = 0.0, cneg = 0.0;
    if (c.cls_loss == PRB_LOSS_FOCAL) {
        cpos = s[A_POS] / P;
        cneg = s[A_NEG] / P;
        cls = (s[A_POS] + s[A_NEG]) / P;
        norm = P;
    } else if (c.cls_loss == PRB_LOSS_DICE) {
        norm = fmax(s[A_DMAX], 1.0);
        cls = 1.0 - s[A_DMIN] / norm;
    } else {
        cls = s[A_CLS] / V;
    }
    auto mean = [&](int j, double n) { return F > 0.0 ? s[j] / n : 0.0; };
    const double xb = mean(A_XB, F), zb = mean(A_ZB, F), xr = mean(A_XR, F), zr = mean(A_ZR, F), yb = mean(A_YB, F),
                 yr = mean(A_YR, F), yo = mean(A_YO, F), rb = mean(A_RB, F), rr = mean(A_RR, F), size = mean(A_SIZE, 3.0 * F);
    const double loc = xb + zb + (c.xz_fine ? xr + zr : 0.0) + (c.y_by_bin ? yb + yr : yo), ang = rb + rr;
    const double reg = loc + ang + 3.0 * size;
    const double v[PRB_SL_TERMS] = {cls, reg, xb, zb, xr, zr, yb, yr, yo, rb, rr, loc, ang, size, cpos, cneg, norm, F, s[A_DMIN], s[A_DMAX]};
#pragma unroll
    for (int j = 0; j < PRB_SL_TERMS; ++j) out[j] = (float)v[j];
    *total = (float)(cls * c.w_cls + reg * c.w_reg);
}

__global__ void __launch_bounds__(kSlTile) stage_loss_backward_kernel(int rows, SlCfg c, SlPtrs p, const float *__restrict__ terms,
                                                                      const float *__restrict__ g_total, const float *__restrict__ g_terms,
                                                                      float *__restrict__ d_cls, float *__restrict__ d_reg) {
    extern __shared__ __align__(16) float s_tile[];          // kSlTile x C
    __shared__ float s_k[K_N];
    const int r0 = blockIdx.x * kSlTile, n = min(kSlTile, rows - r0), tid = threadIdx.x;
    for (int e = tid; e < n * c.C; e += kSlTile) s_tile[e] = 0.f;
    if (tid == 0) {   // the upstream gradient of every atomic term (its own, plus what flows in through the sums it is part of),
                      // over its normaliser
        auto gv = [&](int j) { return g_terms ? g_terms[j] : 0.f; };
        const float gt = g_total ? *g_total : 0.f;
        const float c_cls = gv(PRB_SL_CLS) + gt * c.w_cls, c_reg = gv(PRB_SL_REG) + gt * c.w_reg;
        const float c_loc = gv(PRB_SL_LOC) + c_reg, c_ang = gv(PRB_SL_ANGLE) + c_reg, c_size = gv(PRB_SL_SIZE) + 3.f * c_reg;
        const float norm = terms[PRB_SL_NORM], F = terms[PRB_SL_NFG], f = F > 0.f ? F : 1.f;
        s_k[K_CLS] = c_cls / norm;
        s_k[K_POS] = (c_cls + gv(PRB_SL_CLS_POS)) / norm;
        s_k[K_NEG] = (c_cls + gv(PRB_SL_CLS_NEG)) / norm;
        s_k[K_DMIN] = -c_cls / norm;
        s_k[K_DMAX] = terms[PRB_SL_DMAX] >= 1.f ? c_cls * (terms[PRB_SL_DMIN] / (norm * norm)) : 0.f;   // clamp(., min=1)
        s_k[K_XB] = (gv(PRB_SL_X_BIN) + c_loc) / f;
        s_k[K_ZB] = (gv(PRB_SL_Z_BIN) + c_loc) / f;
        s_k[K_XR] = (gv(PRB_SL_X_RES) + c_loc) / f;
        s_k[K_ZR] = (gv(PRB_SL_Z_RES) + c_loc) / f;
        s_k[K_YB] = (gv(PRB_SL_Y_BIN) + c_loc) / f;
        s_k[K_YR] = (gv(PRB_SL_Y_RES) + c_loc) / f;
        s_k[K_YO] = (gv(PRB_SL_Y_OFFSET) + c_loc) / f;
        s_k[K_RB] = (gv(PRB_SL_RY_BIN) + c_ang) / f;
        s_k[K_RR] = (gv(PRB_SL_RY_RES) + c_ang) / f;
        s_k[K_SIZE] = c_size / (3.f * f);
    }
    __syncthreads();
    const int i = r0 + tid;
    if (tid < n) {
        const long long lab = sl_ld(p.label, c.lab64, i);
        const bool pos = lab > 0, valid = lab >= 0;
        if (c.cls_loss == PRB_LOSS_CE) {
            float *d = d_cls + (size_t)i * c.K;
            if (valid && lab < c.K) {
                const float w = p.ce_weight ? p.ce_weight[lab] : 1.f;
                sl_ce_grad(p.cls + (size_t)i * c.K, c.K, (int)lab, s_k[K_CLS] * w, d);
            } else {
                for (int k = 0; k < c.K; ++k) d[k] = 0.f;
            }
        } else {
            const float x = p.cls[i], t = pos ? 1.f : 0.f, pr = sl_sigmoid(x), dp = (1.f - pr) * pr;
            float d = 0.f;
            if (c.cls_loss == PRB_LOSS_FOCAL) {
                if (valid) {
                    const float e = expf(-fabsf(x));
                    const float ce = fmaxf(x, 0.f) - x * t + log1pf(e);
                    // clamp_min passes the gradient at 0, abs has a zero subgradient there
                    const float dce = (x >= 0.f ? 1.f : 0.f) - t - (x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f)) * (e / (1.f + e));
                    const float b = 1.f - (t * pr + (1.f - t) * (1.f - pr));
                    const float mod = c.gamma == 0.f ? 1.f : (c.gamma == 2.f ? b * b : powf(b, c.gamma));
                    const float dmod = c.gamma == 0.f ? 0.f : -(c.gamma == 2.f ? 2.f * b : c.gamma * powf(b, c.gamma - 1.f)) * (2.f * t - 1.f) * dp;
                    const float g = pos ? s_k[K_POS] : s_k[K_NEG];
                    d = g * (pos ? c.alpha : c.alpha1) * (dmod * ce + mod * dce);
                }
            } else if (c.cls_loss == PRB_LOSS_BCE) {
                if (valid) {      // binary_cross_entropy's backward (its 1e-12 floor), then sigmoid's: 0 where p saturates
                    const float g = s_k[K_CLS] * (pr - t) / fmaxf((1.f - pr) * pr, 1e-12f) * (pos ? c.fg_weight : 1.f);
                    d = g * dp;
                }
            } else if (lab != -1) {     // Dice: minimum / maximum split the gradient at a tie
                const float tl = (float)lab;
                const float dmin = pr < tl ? 1.f : (pr == tl ? 0.5f : 0.f), dmax = pr > tl ? 1.f : (pr == tl ? 0.5f : 0.f);
                d = (s_k[K_DMIN] * dmin + s_k[K_DMAX] * dmax) * dp;
            }
            d_cls[i] = d;
        }
        const bool fg = p.valid ? sl_ld(p.valid, c.valid64, i) > 0 : pos;
        if (fg) {
            SlLab L;
            sl_labels(c, p.reg_label + (size_t)i * 7, sl_anchor(p, i), L);
            const float *x = p.reg + (size_t)i * c.C;
            float *d = s_tile + (size_t)tid * c.C;
            sl_ce_grad(x, c.nloc, L.xb, s_k[K_XB], d);
            sl_ce_grad(x + c.nloc, c.nloc, L.zb, s_k[K_ZB], d + c.nloc);
            if (c.xz_fine) {
                d[2 * c.nloc + L.xb] = s_k[K_XR] * sl_smooth_l1_grad(__fsub_rn(x[2 * c.nloc + L.xb], L.xr));
                d[3 * c.nloc + L.zb] = s_k[K_ZR] * sl_smooth_l1_grad(__fsub_rn(x[3 * c.nloc + L.zb], L.zr));
            }
            if (c.y_by_bin) {
                sl_ce_grad(x + c.off_y, c.ny, L.yb, s_k[K_YB], d + c.off_y);
                d[c.off_y + c.ny + L.yb] = s_k[K_YR] * sl_smooth_l1_grad(__fsub_rn(x[c.off_y + c.ny + L.yb], L.yr));
            } else {
                d[c.off_y] = s_k[K_YO] * sl_smooth_l1_grad(__fsub_rn(x[c.off_y], L.y));
            }
            sl_ce_grad(x + c.off_ry, c.nhb, L.rb, s_k[K_RB], d + c.off_ry);
            d[c.off_ry + c.nhb + L.rb] = s_k[K_RR] * sl_smooth_l1_grad(__fsub_rn(x[c.off_ry + c.nhb + L.rb], L.rr));
#pragma unroll
            for (int q = 0; q < 3; ++q)
                d[c.off_size + q] = s_k[K_SIZE] * sl_smooth_l1_grad(__fsub_rn(x[c.off_size + q], L.sz[q]));
        }
    }
    __syncthreads();
    float *o = d_reg + (size_t)r0 * c.C;
    for (int e = tid; e < n * c.C; e += kSlTile) o[e] = s_tile[e];
}

// the launch configuration of one call, checked against the options (get_reg_loss's width assert)
int sl_config(const prb_stage_loss_desc *d, int rows, int reg_cols, int label_bytes, int valid_bytes, SlCfg &c) {
    PRB_REQUIRE(d, "stage_loss: NULL descriptor");
    PRB_REQUIRE(rows >= 0 && rows < (1 << 24), "stage_loss: %d rows not in 0..2^24", rows);
    PRB_REQUIRE(d->cls_loss >= PRB_LOSS_FOCAL && d->cls_loss <= PRB_LOSS_CE, "stage_loss: classification loss code %d", d->cls_loss);
    PRB_REQUIRE(d->cls_loss == PRB_LOSS_CE ? (d->num_class >= 2 && d->num_class <= kSlMaxK) : d->num_class == 1,
                "stage_loss: %d classification columns for loss code %d (1 for the sigmoid losses, 2..%d for CrossEntropy)",
                d->num_class, d->cls_loss, kSlMaxK);
    PRB_REQUIRE(label_bytes == 4 || label_bytes == 8, "stage_loss: labels must be int32 or int64 (%d bytes)", label_bytes);
    PRB_REQUIRE(valid_bytes == 0 || valid_bytes == 4 || valid_bytes == 8, "stage_loss: the foreground mask must be int32 or int64");
    PRB_REQUIRE(d->loc_scope > 0 && d->loc_bin_size > 0 && d->num_head_bin > 0 && (!d->y_by_bin || (d->loc_y_scope > 0 && d->loc_y_bin_size > 0)),
                "stage_loss: scopes, bin sizes and NUM_HEAD_BIN must be positive");
    c.cls_loss = d->cls_loss;
    c.K = d->num_class;
    c.nloc = (int)(d->loc_scope / d->loc_bin_size) * 2;
    c.ny = d->y_by_bin ? (int)(d->loc_y_scope / d->loc_y_bin_size) * 2 : 0;
    c.nhb = d->num_head_bin;
    c.xz_fine = d->xz_fine != 0;
    c.y_by_bin = d->y_by_bin != 0;
    c.ry_fine = d->ry_fine != 0;
    c.lab64 = label_bytes == 8;
    c.valid64 = valid_bytes == 8;
    PRB_REQUIRE(c.nloc >= 1 && (!c.y_by_bin || c.ny >= 1), "stage_loss: no location bin (scope / bin size < 1)");
    c.off_y = (c.xz_fine ? 4 : 2) * c.nloc;
    c.off_ry = c.off_y + (c.y_by_bin ? 2 * c.ny : 1);
    c.off_size = c.off_ry + 2 * c.nhb;
    c.C = c.off_size + 3;
    PRB_REQUIRE(reg_cols == c.C, "stage_loss: %d regression channels, the options imply %d", reg_cols, c.C);
    PRB_REQUIRE(c.C <= kSlMaxCols, "stage_loss: %d regression channels > %d", c.C, kSlMaxCols);
    c.alpha = (float)d->focal_alpha;
    c.alpha1 = (float)(1.0 - d->focal_alpha);
    c.gamma = (float)d->focal_gamma;
    c.fg_weight = (float)d->fg_weight;
    c.w_cls = (float)d->loss_weight_cls;
    c.w_reg = (float)d->loss_weight_reg;
    // the Python scalars of the mirror, each rounded to fp32 once as torch does
    c.loc_scope = (float)d->loc_scope;
    c.loc_hi = (float)(d->loc_scope * 2 - 1e-3);
    c.loc_bin = (float)d->loc_bin_size;
    c.loc_half = (float)(d->loc_bin_size / 2);
    c.y_scope = (float)d->loc_y_scope;
    c.y_hi = (float)(d->loc_y_scope * 2 - 1e-3);
    c.y_bin = (float)d->loc_y_bin_size;
    c.y_half = (float)(d->loc_y_bin_size / 2);
    const double per = (c.ry_fine ? CUDART_PI / 2 : 2 * CUDART_PI) / d->num_head_bin;
    c.per = (float)per;
    c.per_half = (float)(per / 2);
    return 0;
}

int sl_parts(int rows) { return min(max(ceil_div(rows, kSlThreads), 1), kSlMaxParts); }

}  // namespace prb

using namespace prb;

extern "C" size_t prb_stage_loss_workspace_bytes(int rows) { return (size_t)sl_parts(rows) * kSlAcc * sizeof(double); }

extern "C" int prb_stage_loss_forward(const prb_stage_loss_desc *desc, int rows, int reg_cols, const float *cls, const float *reg,
                                      const void *cls_label, int label_bytes, const void *fg_mask, int fg_mask_bytes,
                                      const float *reg_label, const float *mean_size, const float *anchor_boxes,
                                      const float *ce_weight, float *total, float *terms, void *workspace, size_t workspace_bytes,
                                      void *stream) {
    SlCfg c;
    if (int rc = sl_config(desc, rows, reg_cols, label_bytes, fg_mask ? fg_mask_bytes : 0, c)) return rc;
    PRB_REQUIRE(total && terms && workspace && (rows == 0 || (cls && reg && cls_label && reg_label && (anchor_boxes || mean_size))),
                "stage_loss_forward: bad arguments");
    PRB_REQUIRE(workspace_bytes >= prb_stage_loss_workspace_bytes(rows), "stage_loss_forward: workspace of %zu bytes < %zu",
                workspace_bytes, prb_stage_loss_workspace_bytes(rows));
    const SlPtrs p{cls, reg, reg_label, mean_size, anchor_boxes, ce_weight, cls_label, fg_mask};
    const int parts = sl_parts(rows);
    double *ws = reinterpret_cast<double *>(workspace);
    stage_loss_rows_kernel<<<parts, kSlThreads, 0, (cudaStream_t)stream>>>(rows, c, p, ws);
    if (int rc = check_launch("stage_loss_rows_kernel")) return rc;
    stage_loss_final_kernel<<<1, kSlThreads, 0, (cudaStream_t)stream>>>(parts, c, ws, total, terms);
    return check_launch("stage_loss_final_kernel");
}

extern "C" int prb_stage_loss_backward(const prb_stage_loss_desc *desc, int rows, int reg_cols, const float *cls, const float *reg,
                                       const void *cls_label, int label_bytes, const void *fg_mask, int fg_mask_bytes,
                                       const float *reg_label, const float *mean_size, const float *anchor_boxes,
                                       const float *ce_weight, const float *terms, const float *grad_total,
                                       const float *grad_terms, float *d_cls, float *d_reg, void *stream) {
    SlCfg c;
    if (int rc = sl_config(desc, rows, reg_cols, label_bytes, fg_mask ? fg_mask_bytes : 0, c)) return rc;
    PRB_REQUIRE(terms && (rows == 0 || (cls && reg && cls_label && reg_label && (anchor_boxes || mean_size) && d_cls && d_reg)),
                "stage_loss_backward: bad arguments");
    if (rows == 0) return 0;
    const SlPtrs p{cls, reg, reg_label, mean_size, anchor_boxes, ce_weight, cls_label, fg_mask};
    const size_t smem = (size_t)kSlTile * c.C * sizeof(float);
    PRB_CUDA(cudaFuncSetAttribute(stage_loss_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    stage_loss_backward_kernel<<<ceil_div(rows, kSlTile), kSlTile, smem, (cudaStream_t)stream>>>(rows, c, p, terms, grad_total, grad_terms,
                                                                                                  d_cls, d_reg);
    return check_launch("stage_loss_backward_kernel");
}
