// eval_stats.cu -- the statistics of tools/eval_rcnn.py's evaluation loops for a batch of scenes: box recall at several
// IoU thresholds (with every box's max IoU over the GT), the RPN segmentation IoU and the RCNN classification accuracy.
// The reference computes them one scene at a time with a boxes_iou3d_gpu call per box set and about a dozen `.item()`
// host round trips; here each is one launch per batch, one CTA per scene, with integer counts, so the results do not
// depend on scheduling.
#include <math_constants.h>

#include "common.cuh"
#include "iou3d_dev.cuh"

namespace prb {

constexpr int kEsThreads = 128;
constexpr int kEsMaxBoxes = 512;       // the TRAIN post-NMS proposal count
constexpr int kEsMaxThresh = 16;
constexpr int POLY_SLOTS_ES = 16;      // an intersection polygon has at most 8 + 8 vertices
constexpr int kEsMaxPoints = 16384;    // every count stays exact in fp32

struct EsThresh {
    int n;
    float t[kEsMaxThresh];
};

// order-preserving map of a float onto int (for atomicMax in shared memory); -0 sorts just below +0
__device__ __forceinline__ int es_key(float v) {
    const int i = __float_as_int(v);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float es_val(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

__device__ __forceinline__ int es_block_sum(int v, int *s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    int total = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) total += s_red[w];
    return total;
}

// one CTA per scene: every (real box, real GT) pair once, the row and column maxima in shared memory
__global__ void __launch_bounds__(kEsThreads) eval_box_recall_kernel(int m, int g, const float *__restrict__ boxes,
                                                                     const int *__restrict__ box_count, const float *__restrict__ gt,
                                                                     const int *__restrict__ gt_count, EsThresh th,
                                                                     unsigned long long *__restrict__ recalled,
                                                                     unsigned long long *__restrict__ gt_total,
                                                                     float *__restrict__ box_max_iou) {
    extern __shared__ int s_gt_max[];             // g
    __shared__ int s_row_max[kEsMaxBoxes];
    __shared__ float s_poly[3 * POLY_SLOTS_ES * kEsThreads];
    __shared__ int s_hits[kEsMaxThresh];
    const int scene = blockIdx.x, tid = threadIdx.x;
    const int n = box_count ? min(max(box_count[scene], 0), m) : m;
    const int ng = min(max(gt_count[scene], 0), g);
    const int neg = es_key(-CUDART_INF_F);
    for (int i = tid; i < n; i += kEsThreads) s_row_max[i] = neg;
    for (int j = tid; j < ng; j += kEsThreads) s_gt_max[j] = neg;
    if (tid < th.n) s_hits[tid] = 0;
    __syncthreads();

    float *px = s_poly + tid, *py = px + POLY_SLOTS_ES * kEsThreads, *pa = py + POLY_SLOTS_ES * kEsThreads;
    const float *B = boxes + (size_t)scene * m * 7, *G = gt + (size_t)scene * g * 7;
    const int pairs = n * ng;
    for (int p = tid; p < pairs; p += kEsThreads) {
        const int i = p / ng, j = p - i * ng;
        float a[7], b[7];
#pragma unroll
        for (int q = 0; q < 7; ++q) { a[q] = B[i * 7 + q]; b[q] = G[j * 7 + q]; }
        const int k = es_key(iou3d_pair(a, b, px, py, pa, kEsThreads));
        atomicMax(&s_row_max[i], k);
        atomicMax(&s_gt_max[j], k);
    }
    __syncthreads();

    if (box_max_iou) {
        float *out = box_max_iou + (size_t)scene * m;
        for (int i = tid; i < m; i += kEsThreads) out[i] = (i < n && ng > 0) ? es_val(s_row_max[i]) : 0.f;
    }
    if (recalled) {
        for (int j = tid; j < ng; j += kEsThreads) {
            const float v = es_val(s_gt_max[j]);           // -inf when the scene has no real box
#pragma unroll
            for (int t = 0; t < kEsMaxThresh; ++t)          // constant indices: the thresholds stay in the parameter bank
                if (t < th.n && v > th.t[t]) atomicAdd(&s_hits[t], 1);
        }
        __syncthreads();
        if (tid < th.n && s_hits[tid]) atomicAdd(&recalled[tid], (unsigned long long)s_hits[tid]);
    }
    if (gt_total && tid == 0 && ng > 0) atomicAdd(gt_total, (unsigned long long)ng);
}

__global__ void __launch_bounds__(256) eval_seg_iou_kernel(int n, const int *__restrict__ pred, const int *__restrict__ label,
                                                           float *__restrict__ iou) {
    __shared__ int s_red[8];
    const int scene = blockIdx.x;
    const int *P = pred + (size_t)scene * n, *L = label + (size_t)scene * n;
    int fg = 0, pos = 0, correct = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int p = P[i], l = L[i];
        fg += l > 0;
        pos += p > 0;
        correct += (p == l) & (l > 0);
    }
    fg = es_block_sum(fg, s_red);
    pos = es_block_sum(pos, s_red);
    correct = es_block_sum(correct, s_red);
    if (threadIdx.x == 0) {
        // fg_mask.sum().float() + (seg > 0).sum().float() - correct, clamp(min=1), one division: exact counts in fp32
        const float uni = __fsub_rn(__fadd_rn((float)fg, (float)pos), (float)correct);
        iou[scene] = __fdiv_rn((float)correct, fmaxf(uni, 1.f));
    }
}

__global__ void __launch_bounds__(256) eval_cls_acc_kernel(int m, const int *__restrict__ box_count, const int *__restrict__ pred_cls,
                                                           const float *__restrict__ gt_iou, float cls_fg, float cls_bg,
                                                           float refined_thresh, float *__restrict__ acc,
                                                           float *__restrict__ acc_refined) {
    __shared__ int s_red[8];
    const int scene = blockIdx.x;
    const int n = box_count ? min(max(box_count[scene], 0), m) : m;
    const int *P = pred_cls + (size_t)scene * m;
    const float *I = gt_iou + (size_t)scene * m;
    int eq_valid = 0, valid = 0, eq_refined = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int p = P[i];
        const float v = I[i];
        const int va = (v >= cls_fg) | (v <= cls_bg);
        valid += va;
        eq_valid += (p == (int)(v > cls_fg)) & va;
        eq_refined += p == (int)(v >= refined_thresh);
    }
    eq_valid = es_block_sum(eq_valid, s_red);
    valid = es_block_sum(valid, s_red);
    eq_refined = es_block_sum(eq_refined, s_red);
    if (threadIdx.x == 0) {
        acc[scene] = __fdiv_rn((float)eq_valid, fmaxf((float)valid, 1.f));
        // `sum / max(count, 1.0)` with a Python divisor: torch's CUDA division multiplies by the fp32 reciprocal
        acc_refined[scene] = __fmul_rn((float)eq_refined, __fdiv_rn(1.f, (float)max(n, 1)));
    }
}

}  // namespace prb

using namespace prb;

extern "C" int prb_eval_box_recall(int b, int m, const float *boxes, const int *box_count, int g, const float *gt, const int *gt_count,
                                   int n_thresh, const float *thresh, long long *recalled, long long *gt_total, float *box_max_iou,
                                   void *stream) {
    PRB_REQUIRE(b >= 0 && m >= 0 && g >= 0 && gt_count && (m == 0 || boxes) && (g == 0 || gt), "eval_box_recall: bad arguments");
    PRB_REQUIRE(m <= kEsMaxBoxes, "eval_box_recall: %d boxes per scene > %d", m, kEsMaxBoxes);
    PRB_REQUIRE(!recalled || (n_thresh >= 0 && n_thresh <= kEsMaxThresh && (n_thresh == 0 || thresh)),
                "eval_box_recall: %d thresholds (at most %d)", n_thresh, kEsMaxThresh);
    if (b == 0) return 0;
    EsThresh th{};
    th.n = recalled ? n_thresh : 0;
    for (int t = 0; t < th.n; ++t) th.t[t] = thresh[t];
    const size_t smem = (size_t)g * sizeof(int);
    int dev = 0, optin = 0;
    PRB_CUDA(cudaGetDevice(&dev));
    PRB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const size_t static_smem = sizeof(int) * (kEsMaxBoxes + kEsMaxThresh) + sizeof(float) * 3 * POLY_SLOTS_ES * kEsThreads;
    PRB_REQUIRE(smem + static_smem <= (size_t)optin, "eval_box_recall: %d GT boxes per scene do not fit in shared memory", g);
    if (smem > 48 * 1024 - static_smem)
        PRB_CUDA(cudaFuncSetAttribute(eval_box_recall_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    eval_box_recall_kernel<<<b, kEsThreads, smem, (cudaStream_t)stream>>>(m, g, boxes, box_count, gt, gt_count, th,
                                                                          (unsigned long long *)recalled,
                                                                          (unsigned long long *)gt_total, box_max_iou);
    return check_launch("eval_box_recall_kernel");
}

extern "C" int prb_eval_seg_iou(int b, int n, const int *pred, const int *label, float *iou, void *stream) {
    PRB_REQUIRE(b >= 0 && n >= 0 && iou && (n == 0 || (pred && label)), "eval_seg_iou: bad arguments");
    PRB_REQUIRE(n <= kEsMaxPoints, "eval_seg_iou: %d points per scene > %d", n, kEsMaxPoints);
    if (b == 0) return 0;
    eval_seg_iou_kernel<<<b, 256, 0, (cudaStream_t)stream>>>(n, pred, label, iou);
    return check_launch("eval_seg_iou_kernel");
}

extern "C" int prb_eval_cls_acc(int b, int m, const int *box_count, const int *pred_cls, const float *gt_iou, float cls_fg,
                                float cls_bg, float refined_thresh, float *acc, float *acc_refined, void *stream) {
    PRB_REQUIRE(b >= 0 && m >= 0 && acc && acc_refined && (m == 0 || (pred_cls && gt_iou)), "eval_cls_acc: bad arguments");
    PRB_REQUIRE(m <= (1 << 24), "eval_cls_acc: %d RoIs per scene", m);
    if (b == 0) return 0;
    eval_cls_acc_kernel<<<b, 256, 0, (cudaStream_t)stream>>>(m, box_count, pred_cls, gt_iou, cls_fg, cls_bg, refined_thresh, acc,
                                                             acc_refined);
    return check_launch("eval_cls_acc_kernel");
}
