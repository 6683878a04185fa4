// rcnn_sample.cu -- RoI sampling, jitter and targets of offline RCNN training (lib/datasets/kitti_rcnn_dataset.py:876-1077,
// get_rcnn_training_sample_batch with sample_bg_inds and aug_roi_by_noise_batch) for a batch of scenes, around the existing
// 3D-IoU matrix and RoI pooling launches:
//   prb_boxes_iou3d -> sample (this file) -> prb_roipool3d_ws (two passes) -> targets (this file)
//   sample   one CTA per scene: IoU reductions, the fg / easy bg / hard bg candidate lists, the four branches, then one
//            thread per sampled RoI runs the jitter loop with the 3D IoU computed inline (iou3d_dev.cuh's iou3d_pair)
//   targets  one CTA per sampled RoI: stage-2 data augmentation of the pooled points and both boxes, labels from the
//            pre-augmentation IoU, canonical transform
// Random draws are counter-based hashes keyed by (seed, scene, stage, roi, try, slot): the same distribution as the
// reference's np.random stream, not the same stream.  oracle/rcnn_offline.py restates the keys, and the jitter arithmetic
// below uses explicit _rn intrinsics so that an fp32 numpy restatement matches it bit for bit.
#include <math_constants.h>

#include "common.cuh"
#include "iou3d_dev.cuh"

namespace prb {

constexpr int kRsThreads = 128;
constexpr int kRsMaxRois = 4096;       // proposals per scene
constexpr int kRsMaxGt = 256;          // GT boxes per scene
constexpr int kRsMaxRows = 1024;       // ROI_PER_IMAGE
constexpr int kRtThreads = 128;
constexpr int POLY_SLOTS_RS = 16;    // an intersection polygon has at most 8 + 8 vertices
constexpr uint32_t kSaltFg = 0x3c6ef372u, kSaltBg = 0xa54ff53au, kSaltJitter = 0x510e527fu, kSaltAug = 0x9b05688cu;

// key of one draw: stage salt, output row (or fg-list position), try, slot
__device__ __forceinline__ uint32_t rs_key(uint32_t seed, int scene, uint32_t salt, int row, int t, int slot) {
    return draw_key(seed, (uint32_t)scene, ((uint32_t)row << 12) | ((uint32_t)t << 6) | (uint32_t)slot, salt);
}
// uniform in [0, 1) on a 2^-24 grid (exact in fp32)
__device__ __forceinline__ float rs_u01(uint32_t h) { return (float)(h >> 8) * 5.9604644775390625e-08f; }
// floor(u * n) in integers
__device__ __forceinline__ int rs_pick(uint32_t h, int n) { return (int)(((unsigned long long)(h >> 8) * (unsigned)n) >> 24); }

// appends, in index order, every i < n with pred(i) to out[base..]; returns the new length (CTA-uniform)
template <class Pred>
__device__ __forceinline__ int rs_append(int n, Pred pred, const int *vals, int *out, int base, int *s_wc) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = kRsThreads / 32;
    for (int c0 = 0; c0 < n; c0 += kRsThreads) {
        const int i = c0 + tid;
        const bool in = i < n && pred(i);
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_wc[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
            before += w < warp ? s_wc[w] : 0;
            total += s_wc[w];
        }
        if (in) out[base + before + __popc(m & ((1u << lane) - 1u))] = vals ? vals[i] : i;
        base += total;
        __syncthreads();
    }
    return base;
}

// random_aug_box3d (kitti_rcnn_dataset.py:746-788); method 0 single, 1 multiple, 2 normal
__device__ __forceinline__ void rs_jitter(const float *src, float *o, int method, uint32_t seed, int scene, int row, int t) {
    auto u = [&](int slot) { return rs_u01(rs_key(seed, scene, kSaltJitter, row, t, slot)); };
    if (method == 2) {
        const float sd[6] = {0.3f, 0.2f, 0.3f, 0.25f, 0.15f, 0.5f};
#pragma unroll
        for (int p = 0; p < 3; ++p) {       // Box-Muller: slots 2+2p, 3+2p -> two standard normals
            const float r = sqrtf(-2.0f * logf(1.0f - u(2 + 2 * p)));
            float sn, cs;
            sincospif(2.0f * u(3 + 2 * p), &sn, &cs);
            o[2 * p] = __fadd_rn(src[2 * p], __fmul_rn(__fmul_rn(r, cs), sd[2 * p]));
            o[2 * p + 1] = __fadd_rn(src[2 * p + 1], __fmul_rn(__fmul_rn(r, sn), sd[2 * p + 1]));
        }
        o[6] = __fadd_rn(src[6], __fmul_rn(__fmul_rn(__fsub_rn(u(8), 0.5f), 2.0f), (float)(CUDART_PI / 12.0)));
        return;
    }
    float pos_r, hwl_r, ang_r;
    if (method == 1) {
        const int idx = rs_pick(rs_key(seed, scene, kSaltJitter, row, t, 1), 5);
        pos_r = idx == 0 ? 0.2f : idx == 1 ? 0.3f : idx == 2 ? 0.5f : idx == 3 ? 0.8f : 1.0f;
        hwl_r = idx == 0 ? 0.1f : 0.15f;
        ang_r = idx <= 1 ? (float)(CUDART_PI / 12.0) : idx == 2 ? (float)(CUDART_PI / 9.0) : idx == 3 ? (float)(CUDART_PI / 6.0)
                                                                                                  : (float)(CUDART_PI / 3.0);
    } else {   // single: shift U(-0.5, 0.5), scale 1 + U(-0.15, 0.15), angle U(-pi/12, pi/12)
        pos_r = 0.5f;
        hwl_r = 0.15f;
        ang_r = (float)(CUDART_PI / 12.0);
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const float d = __fmul_rn(__fsub_rn(u(2 + q), 0.5f), 2.0f);              // exact: U(-1, 1)
        o[q] = __fadd_rn(src[q], __fmul_rn(d, pos_r));
        const float e = __fmul_rn(__fsub_rn(u(5 + q), 0.5f), 2.0f);
        o[3 + q] = __fmul_rn(src[3 + q], __fadd_rn(__fmul_rn(e, hwl_r), 1.0f));
    }
    o[6] = __fadd_rn(src[6], __fmul_rn(__fmul_rn(__fsub_rn(u(8), 0.5f), 2.0f), ang_r));
}

struct RsCfg {
    int R, fg_quota, method, fg_aug_times;
    float reg_fg, cls_fg, cls_bg, cls_bg_lo, extra_width;
    double hard_ratio;
    uint32_t seed;
};

__global__ void __launch_bounds__(kRsThreads) rcnn_sample_kernel(
    int m, int g, RsCfg cf, const float *__restrict__ iou, const float *__restrict__ rois, const int *__restrict__ roi_count,
    const float *__restrict__ gts, const int *__restrict__ gt_count, float *__restrict__ rois_out, float *__restrict__ gt_out,
    float *__restrict__ iou_out, float *__restrict__ pool_boxes, int *__restrict__ sel, int *__restrict__ status) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    float *s_maxov = reinterpret_cast<float *>(s_raw);        // m
    int *s_gtas = reinterpret_cast<int *>(s_maxov + m);       // m
    int *s_fg = s_gtas + m;                                   // m + g
    uint32_t *s_key = reinterpret_cast<uint32_t *>(s_fg + m + g);   // m + g
    int *s_easy = reinterpret_cast<int *>(s_key + m + g);     // m
    int *s_hard = s_easy + m;                                 // m
    int *s_roias = s_hard + m;                                // g
    __shared__ int s_src[kRsMaxRows];
    __shared__ int s_wc[kRsThreads / 32];
    __shared__ float s_poly[3 * POLY_SLOTS_RS * kRsThreads];
    const int scene = blockIdx.x, tid = threadIdx.x, R = cf.R;
    const int n = min(roi_count[scene], m), ng = min(gt_count[scene], g);
    const float fg_thresh = fminf(cf.reg_fg, cf.cls_fg);

    int st = 0, fg_rows = 0, hard_rows = 0, fg_num = 0, nh = 0, ne = 0;
    bool fg_only = false;
    if (n == 0 || ng == 0) {
        st = 2;
    } else {
        // max_overlaps / gt_assignment, max_iou_of_gt / roi_assignment: numpy's first-max argmax
        const float *I = iou + (size_t)scene * m * g;
        for (int i = tid; i < n; i += kRsThreads) {
            float best = I[(size_t)i * g];
            int arg = 0;
            for (int j = 1; j < ng; ++j) {
                const float v = I[(size_t)i * g + j];
                if (v > best) { best = v; arg = j; }
            }
            s_maxov[i] = best;
            s_gtas[i] = arg;
        }
        for (int j = tid; j < ng; j += kRsThreads) {
            float best = I[j];
            int arg = 0;
            for (int i = 1; i < n; ++i) {
                const float v = I[(size_t)i * g + j];
                if (v > best) { best = v; arg = i; }
            }
            s_roias[j] = best > 0.f ? arg : -1;
        }
        __syncthreads();
        // fg: over the threshold in index order, then roi_assignment in GT order (duplicates kept); easy / hard bg
        fg_num = rs_append(n, [&](int i) { return s_maxov[i] >= fg_thresh; }, nullptr, s_fg, 0, s_wc);
        fg_num = rs_append(ng, [&](int j) { return s_roias[j] >= 0; }, s_roias, s_fg, fg_num, s_wc);
        ne = rs_append(n, [&](int i) { return s_maxov[i] < cf.cls_bg_lo; }, nullptr, s_easy, 0, s_wc);
        nh = rs_append(n, [&](int i) { return s_maxov[i] < cf.cls_bg && s_maxov[i] >= cf.cls_bg_lo; }, nullptr, s_hard, 0, s_wc);
        const int bg_num = ne + nh;
        if (fg_num > 0 && bg_num > 0) fg_rows = min(cf.fg_quota, fg_num);
        else if (fg_num > 0) { fg_rows = R; fg_only = true; }
        else if (bg_num > 0) fg_rows = 0;
        else st = 1;                                          // the reference stops in pdb here
        const int bg_rows = R - fg_rows;
        hard_rows = (nh > 0 && ne > 0) ? (int)((double)bg_rows * cf.hard_ratio) : (nh > 0 ? bg_rows : 0);
    }
    if (tid == 0) status[scene] = st;
    if (st == 0) {
        if (fg_rows > 0 && !fg_only) {
            // fg without replacement: the fg_rows smallest keys (ties by position), in key order
            for (int e = tid; e < fg_num; e += kRsThreads) s_key[e] = draw_key(cf.seed, (uint32_t)scene, (uint32_t)e, kSaltFg);
            __syncthreads();
            for (int e = tid; e < fg_num; e += kRsThreads) {
                const uint32_t k = s_key[e];
                int rank = 0;
                for (int f = 0; f < fg_num; ++f) {
                    const uint32_t kf = s_key[f];
                    rank += (kf < k) | ((kf == k) & (f < e));
                }
                if (rank < fg_rows) s_src[rank] = s_fg[e];
            }
        } else if (fg_only) {
            for (int r = tid; r < R; r += kRsThreads) s_src[r] = s_fg[rs_pick(rs_key(cf.seed, scene, kSaltBg, r, 0, 0), fg_num)];
        }
        // bg with replacement: hard rows first, then easy rows
        for (int r = fg_rows + tid; r < R; r += kRsThreads) {
            const uint32_t h = rs_key(cf.seed, scene, kSaltBg, r, 0, 0);
            s_src[r] = r - fg_rows < hard_rows ? s_hard[rs_pick(h, nh)] : s_easy[rs_pick(h, ne)];
        }
        __syncthreads();
    }
    // the jitter loop (aug_roi_by_noise_batch), one thread per sampled RoI
    const float pos_thresh = fg_thresh;
    float *px = s_poly + tid, *py = px + POLY_SLOTS_RS * kRsThreads, *pa = py + POLY_SLOTS_RS * kRsThreads;
    for (int r = tid; r < R; r += kRsThreads) {
        const size_t o = (size_t)scene * R + r;
        float box[7], gt[7];
        float temp_iou = 0.f;
        int cnt = 0, src = -1, ga = -1;
        if (st == 0) {
            src = s_src[r];
            ga = s_gtas[src];
            float s[7];
#pragma unroll
            for (int q = 0; q < 7; ++q) {
                s[q] = rois[((size_t)scene * m + src) * 7 + q];
                gt[q] = gts[((size_t)scene * g + ga) * 7 + q];
                box[q] = s[q];
            }
            const int times = r < fg_rows ? cf.fg_aug_times : 1;
            while (temp_iou < pos_thresh && cnt < times) {
                if (rs_u01(rs_key(cf.seed, scene, kSaltJitter, r, cnt, 0)) < 0.2f) {
#pragma unroll
                    for (int q = 0; q < 7; ++q) box[q] = s[q];
                } else {
                    rs_jitter(s, box, cf.method, cf.seed, scene, r, cnt);
                }
                temp_iou = iou3d_pair(box, gt, px, py, pa, kRsThreads);
                ++cnt;
            }
        } else {
#pragma unroll
            for (int q = 0; q < 7; ++q) box[q] = gt[q] = 0.f;
        }
#pragma unroll
        for (int q = 0; q < 7; ++q) {
            rois_out[o * 7 + q] = box[q];
            gt_out[o * 7 + q] = gt[q];
        }
        iou_out[o] = temp_iou;
        // enlarge_box3d (kitti_utils.py:150-160); an ignored row gets negative sizes, which no point is inside
        float pb[7];
        if (st == 0) {
            const float w2 = __fmul_rn(cf.extra_width, 2.0f);
            pb[0] = box[0]; pb[1] = __fadd_rn(box[1], cf.extra_width); pb[2] = box[2];
            pb[3] = __fadd_rn(box[3], w2); pb[4] = __fadd_rn(box[4], w2); pb[5] = __fadd_rn(box[5], w2); pb[6] = box[6];
        } else {
            pb[0] = pb[1] = pb[2] = pb[6] = 0.f;
            pb[3] = pb[4] = pb[5] = -1.f;
        }
#pragma unroll
        for (int q = 0; q < 7; ++q) pool_boxes[o * 7 + q] = pb[q];
        sel[o * 3] = src;
        sel[o * 3 + 1] = ga;
        sel[o * 3 + 2] = cnt;
    }
}

// rotate_pc_along_y on one (x, z) pair
__device__ __forceinline__ void rt_rot(float &x, float &z, float c, float s) {
    const float nx = x * c - z * s, nz = x * s + z * c;
    x = nx;
    z = nz;
}
__device__ __forceinline__ float rt_sign(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// rotate_box3d_along_y (kitti_rcnn_dataset.py:396-406): the observation angle is kept
__device__ __forceinline__ void rt_rotate_box(float *b, float c, float s) {
    const float beta0 = atan2f(b[2], b[0]);
    const float alpha = -rt_sign(beta0) * (float)(CUDART_PI / 2.0) + beta0 + b[6];
    rt_rot(b[0], b[2], c, s);
    const float beta1 = atan2f(b[2], b[0]);
    b[6] = rt_sign(beta1) * (float)(CUDART_PI / 2.0) + alpha - beta1;
}

struct RtCfg {
    int aug, rotation, scaling, flip;
    float rot_range, flip_prob, reg_fg, cls_fg, cls_bg;
    uint32_t seed;
};

// one CTA per sampled RoI k = scene * R + r
__global__ void __launch_bounds__(kRtThreads) rcnn_targets_kernel(
    int R, int S, int W, RtCfg cf, float *__restrict__ rows, float *__restrict__ rois, float *__restrict__ gts,
    const float *__restrict__ iou, const int *__restrict__ empty, float *__restrict__ gt_ct, int *__restrict__ cls_label,
    int *__restrict__ reg_valid) {
    const int k = blockIdx.x, scene = k / R, r = k - scene * R, tid = threadIdx.x;
    float rb[7], gb[7];
#pragma unroll
    for (int q = 0; q < 7; ++q) { rb[q] = rois[(size_t)k * 7 + q]; gb[q] = gts[(size_t)k * 7 + q]; }
    __syncthreads();          // every thread has read the boxes before thread 0 overwrites them with the augmented ones
    // data_augmentation(mustaug=True, stage=2): three aug_enable draws, rotation and scaling always, flip by aug_enable[2]
    float ac = 1.f, as = 0.f, sc = 1.f;
    bool rot = false, scale = false, flip = false;
    if (cf.aug) {
        auto u = [&](int slot) { return rs_u01(rs_key(cf.seed, scene, kSaltAug, r, 0, slot)); };
        const float lo = -(float)CUDART_PI / cf.rot_range;
        rot = cf.rotation;
        scale = cf.scaling;
        flip = cf.flip && __fsub_rn(1.0f, u(2)) < cf.flip_prob;
        if (rot) {
            const float angle = __fadd_rn(lo, __fmul_rn(__fmul_rn(lo, -2.0f), u(3)));
            sincosf(angle, &as, &ac);
            rt_rotate_box(rb, ac, as);
            rt_rotate_box(gb, ac, as);
        }
        if (scale) {
            sc = __fadd_rn(0.95f, __fmul_rn(0.1f, u(4)));
#pragma unroll
            for (int q = 0; q < 6; ++q) { rb[q] *= sc; gb[q] *= sc; }
        }
        if (flip) {
            rb[0] = -rb[0]; gb[0] = -gb[0];
            rb[6] = rt_sign(rb[6]) * (float)CUDART_PI - rb[6];
            gb[6] = rt_sign(gb[6]) * (float)CUDART_PI - gb[6];
        }
    }
    // canonical_transform_batch (:685-704): roi_ry = ry mod 2 pi (Python's sign rule)
    const float two_pi = (float)(2.0 * CUDART_PI);
    float roi_ry = fmodf(rb[6], two_pi);
    if (roi_ry < 0.f) roi_ry += two_pi;
    float cc, cs;
    sincosf(roi_ry, &cs, &cc);
    float *p = rows + (size_t)k * S * W;
    for (int i = tid; i < S; i += kRtThreads) {
        float x = p[(size_t)i * W], y = p[(size_t)i * W + 1], z = p[(size_t)i * W + 2];
        if (rot) rt_rot(x, z, ac, as);
        if (scale) { x *= sc; y *= sc; z *= sc; }
        if (flip) x = -x;
        x -= rb[0]; y -= rb[1]; z -= rb[2];
        rt_rot(x, z, cc, cs);
        p[(size_t)i * W] = x; p[(size_t)i * W + 1] = y; p[(size_t)i * W + 2] = z;
    }
    if (tid == 0) {
        float c[7];
#pragma unroll
        for (int q = 0; q < 7; ++q) c[q] = gb[q];
        c[0] -= rb[0]; c[1] -= rb[1]; c[2] -= rb[2];
        rt_rot(c[0], c[2], cc, cs);
        c[6] -= roi_ry;
#pragma unroll
        for (int q = 0; q < 7; ++q) {
            gt_ct[(size_t)k * 7 + q] = c[q];
            rois[(size_t)k * 7 + q] = rb[q];
            gts[(size_t)k * 7 + q] = gb[q];
        }
        // labels from the IoU before augmentation
        const float v = iou[k];
        const bool valid = empty[k] == 0;
        int cls = v > cf.cls_fg ? 1 : 0;
        if ((v > cf.cls_bg && v < cf.cls_fg) || !valid) cls = -1;
        cls_label[k] = cls;
        reg_valid[k] = (v > cf.reg_fg && valid) ? 1 : 0;
    }
}

}  // namespace prb

using namespace prb;

extern "C" int prb_rcnn_sample_rois(int b, int m, int g, const float *iou, const float *rois, const int *roi_count, const float *gt_boxes,
                                    const int *gt_count, int roi_per_image, int fg_per_image, float reg_fg_thresh, float cls_fg_thresh,
                                    float cls_bg_thresh, float cls_bg_thresh_lo, double hard_bg_ratio, int aug_method, int fg_aug_times,
                                    float pool_extra_width, unsigned seed, float *rois_out, float *gt_out, float *iou_out,
                                    float *pool_boxes, int *sel, int *status, void *stream) {
    PRB_REQUIRE(b > 0 && m >= 0 && g >= 0 && roi_count && gt_count && rois_out && gt_out && iou_out && pool_boxes && sel && status &&
                    (m == 0 || rois) && (g == 0 || gt_boxes) && (m == 0 || g == 0 || iou),
                "rcnn_sample_rois: bad arguments");
    PRB_REQUIRE(m <= kRsMaxRois, "rcnn_sample_rois: %d proposals per scene > %d", m, kRsMaxRois);
    PRB_REQUIRE(g <= kRsMaxGt, "rcnn_sample_rois: %d GT boxes per scene > %d", g, kRsMaxGt);
    PRB_REQUIRE(roi_per_image > 0 && roi_per_image <= kRsMaxRows, "rcnn_sample_rois: ROI_PER_IMAGE %d not in 1..%d", roi_per_image,
                kRsMaxRows);
    PRB_REQUIRE(fg_per_image >= 0 && fg_per_image <= roi_per_image && fg_aug_times >= 1 && fg_aug_times < 64,
                "rcnn_sample_rois: fg quota %d or fg aug times %d out of range", fg_per_image, fg_aug_times);
    PRB_REQUIRE(aug_method >= 0 && aug_method <= 2, "rcnn_sample_rois: REG_AUG_METHOD code %d not in 0..2", aug_method);
    PRB_REQUIRE(hard_bg_ratio >= 0.0 && hard_bg_ratio <= 1.0, "rcnn_sample_rois: HARD_BG_RATIO %g not in [0, 1]", hard_bg_ratio);
    RsCfg cf{roi_per_image, fg_per_image, aug_method, fg_aug_times, reg_fg_thresh, cls_fg_thresh, cls_bg_thresh, cls_bg_thresh_lo,
             pool_extra_width, hard_bg_ratio, seed};
    const size_t smem = (size_t)(6 * m + 3 * g) * 4;
    PRB_CUDA(cudaFuncSetAttribute(rcnn_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(smem > 0 ? smem : 4)));
    rcnn_sample_kernel<<<b, kRsThreads, smem, (cudaStream_t)stream>>>(m, g, cf, iou, rois, roi_count, gt_boxes, gt_count, rois_out,
                                                                       gt_out, iou_out, pool_boxes, sel, status);
    return check_launch("rcnn_sample_kernel");
}

extern "C" int prb_rcnn_roi_targets(int b, int roi_per_image, int S, int W, float *rows, float *rois, float *gt_boxes,
                                    const float *iou, const int *empty_flag, int aug_data, int aug_rotation, int aug_scaling,
                                    int aug_flip, float aug_rot_range, float flip_prob, float reg_fg_thresh, float cls_fg_thresh,
                                    float cls_bg_thresh, unsigned seed, float *gt_boxes_ct, int *cls_label, int *reg_valid_mask,
                                    void *stream) {
    PRB_REQUIRE(b > 0 && roi_per_image > 0 && S > 0 && W >= 3 && rows && rois && gt_boxes && iou && empty_flag && gt_boxes_ct &&
                    cls_label && reg_valid_mask,
                "rcnn_roi_targets: bad arguments");
    PRB_REQUIRE(!aug_data || !aug_rotation || aug_rot_range > 0.f, "rcnn_roi_targets: AUG_ROT_RANGE must be > 0");
    PRB_REQUIRE((long)b * roi_per_image <= 0x7fffffffL, "rcnn_roi_targets: too many RoIs");
    RtCfg cf{aug_data != 0, aug_rotation != 0, aug_scaling != 0, aug_flip != 0, aug_rot_range, flip_prob, reg_fg_thresh, cls_fg_thresh,
             cls_bg_thresh, seed};
    rcnn_targets_kernel<<<b * roi_per_image, kRtThreads, 0, (cudaStream_t)stream>>>(roi_per_image, S, W, cf, rows, rois, gt_boxes, iou,
                                                                                      empty_flag, gt_boxes_ct, cls_label, reg_valid_mask);
    return check_launch("rcnn_targets_kernel");
}
