// kitti_eval.cu -- the KITTI AP metric of tools/kitti_object_eval_python/eval.py:608-678 (get_official_eval_result),
// evaluated on the device for a whole split.
//
// The annotations of every image sit in two row tables (ground truth and detections, kEvalCols doubles per row, ragged by
// per-image offsets).  The stages follow eval.py's:
//   filter      kitti_common.filter_annos_low_score (optional): the detections scoring >= score_thresh, in row order
//   overlaps    calculate_iou_partly, per image a (dt x gt) matrix of the three metrics (:335-409)
//   clean       clean_data per (class, difficulty): ignored_gt, ignored_dt, number of valid GT (:28-81)
//   pass 1      compute_statistics_jit(compute_fp=False): the TP scores that are threshold candidates (:156-273)
//   thresholds  get_thresholds on the sorted TP scores (:8-25)
//   pass 2      fused_compute_statistics: tp / fp / fn / similarity per threshold (:285-332)
//   finish      recall, precision, orientation similarity and their suffix maxima (:532-542)
// A config is one (metric, class, difficulty, overlap set); the official table has two overlap sets per class
// (get_official_eval_result), the COCO-style one ten (get_coco_eval_result, eval.py:681-740).  The overlaps do not depend on
// the configs and are computed once.  Each (image, config) is one warp: the GT loop stays
// sequential as in the reference, and the loop over detections is a warp reduction whose tie rule gives what the
// sequential loop gives.  tp / fp / fn are integers; the similarity is summed per image in GT order and over images in
// image order, so a result is the same, bit for bit, from run to run.
#include <math_constants.h>

#include "iou3d_dev.cuh"

namespace prb {

constexpr int kEvalCols = 16;
enum { C_X1 = 0, C_Y1, C_X2, C_Y2, C_ALPHA, C_TRUNC, C_OCC, C_L, C_H, C_W, C_X, C_Y, C_Z, C_RY, C_SCORE, C_CLS };
constexpr int kSamplePts = 41;
constexpr int kMaxDetPerImage = 1024;     // one assignment bit per lane and 32 detections
constexpr int kMaxEvalClasses = 8;
constexpr int kMaxOverlapSets = 10;       // get_coco_eval_result's ten overlap thresholds per class
constexpr int kCodeDontCare = 5;          // class codes: 0 car, 1 pedestrian, 2 cyclist, 3 van, 4 person_sitting, 5 DontCare
constexpr int kOutPerThr = 8;             // tp, fp, fn, similarity, recall, precision, aos, threshold

struct EvalCfg {
    int nc;                                                 // evaluated classes
    int ns;                                                 // overlap sets
    int cls[kMaxEvalClasses];                               // their indices (0..2)
    double min_ov[kMaxOverlapSets][3][kMaxEvalClasses];     // [overlap set][metric][class]
};

struct ConfigId {
    int metric, c, diff, k;
};
// config q = ((metric * nc + c) * 3 + diff) * ns + k: the metric-0 configs come first
__device__ __forceinline__ ConfigId config_of(int q, int nc, int ns) {
    ConfigId r;
    r.k = q % ns;
    r.diff = (q / ns) % 3;
    r.c = (q / (3 * ns)) % nc;
    r.metric = q / (3 * ns * nc);
    return r;
}

// image_box_overlap (eval.py:85-111) for one (dt, gt) pair in double, without contractions: criterion -1 = IoU,
// 0 = intersection over the dt box's area
__device__ __forceinline__ double image_overlap(const double *a, const double *b, bool iou) {
    const double iw = __dsub_rn(fmin(a[C_X2], b[C_X2]), fmax(a[C_X1], b[C_X1]));
    if (!(iw > 0.0)) return 0.0;
    const double ih = __dsub_rn(fmin(a[C_Y2], b[C_Y2]), fmax(a[C_Y1], b[C_Y1]));
    if (!(ih > 0.0)) return 0.0;
    const double area_a = __dmul_rn(__dsub_rn(a[C_X2], a[C_X1]), __dsub_rn(a[C_Y2], a[C_Y1]));
    const double inter = __dmul_rn(iw, ih);
    double ua = area_a;
    if (iou) ua = __dsub_rn(__dadd_rn(area_a, __dmul_rn(__dsub_rn(b[C_X2], b[C_X1]), __dsub_rn(b[C_Y2], b[C_Y1]))), inter);
    return __ddiv_rn(inter, ua);
}

// the camera-frame BEV box (x, z, l, w, ry) in fp32 as rotate_iou_gpu_eval takes it, as the iou3d overlap's
// [x - l/2, z - w/2, x + l/2, z + w/2, ry]
__device__ __forceinline__ void bev_pre(const double *r, BoxPre &p, float &area) {
    const float x = (float)r[C_X], z = (float)r[C_Z], l = (float)r[C_L], w = (float)r[C_W];
    const float box[5] = {__fsub_rn(x, l * 0.5f), __fsub_rn(z, w * 0.5f), __fadd_rn(x, l * 0.5f), __fadd_rn(z, w * 0.5f), (float)r[C_RY]};
    box_pre(box, p);
    area = __fmul_rn(l, w);
}

// ------------------------------------------------------------------------------------------------ filter
// filter_annos_low_score (kitti_common.py:190-201) in front of the other stages: the detections of image img with
// score >= thresh, in row order, to the same rows of dt_f, and their number to count_f.  The rows after them, up to the
// image's range, are zeroed.  A stable compaction leaves the assignment order and the AOS decision (the first image that
// still has detections) as evaluating the filtered annotations gives them.  One warp per image.
__global__ void __launch_bounds__(128) eval_filter_kernel(int n_img, double thresh, const double *__restrict__ dt,
                                                          const int *__restrict__ dt_off, const int *__restrict__ dt_count,
                                                          double *__restrict__ dt_f, int *__restrict__ count_f) {
    const int img = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (img >= n_img) return;
    const int d0 = dt_off[img], cap = dt_off[img + 1] - d0;
    const int nd = min(dt_count[img], min(cap, kMaxDetPerImage));
    const double *src = dt + (size_t)d0 * kEvalCols;
    double *dst = dt_f + (size_t)d0 * kEvalCols;
    int n = 0;
    for (int j0 = 0; j0 < nd; j0 += 32) {
        const int j = j0 + lane;
        const bool keep = j < nd && src[(size_t)j * kEvalCols + C_SCORE] >= thresh;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        // the kept rows of these 32 in order, each copied by lanes 0..15, one field per lane
        for (unsigned b = bal; b; b &= b - 1) {
            const int s = __ffs(b) - 1;
            if (lane < kEvalCols) dst[(size_t)n * kEvalCols + lane] = src[(size_t)(j0 + s) * kEvalCols + lane];
            ++n;
        }
    }
    for (size_t e = (size_t)n * kEvalCols + lane; e < (size_t)cap * kEvalCols; e += 32) dst[e] = 0.0;
    if (lane == 0) count_f[img] = n;
}

// ------------------------------------------------------------------------------------------------ overlaps
// one CTA per image; ov (3, n_pairs): metric m of (dt j, gt i) at m * n_pairs + pair_off[img] + j * ng + i
__global__ void __launch_bounds__(128, 4) eval_overlaps_kernel(const double *__restrict__ gt, const int *__restrict__ gt_off,
                                                             const double *__restrict__ dt, const int *__restrict__ dt_off,
                                                             const int *__restrict__ dt_count,
                                                             const long long *__restrict__ pair_off, long long n_pairs,
                                                             double *__restrict__ ov) {
    __shared__ float s_px[POLY_SLOTS * 128], s_py[POLY_SLOTS * 128], s_pa[POLY_SLOTS * 128];
    const int img = blockIdx.x;
    const int g0 = gt_off[img], ng = gt_off[img + 1] - g0;
    const int d0 = dt_off[img], nd = min(dt_count[img], min(dt_off[img + 1] - d0, kMaxDetPerImage));
    double *o = ov + pair_off[img];
    for (int e = threadIdx.x; e < nd * ng; e += 128) {
        const int j = e / ng, i = e - j * ng;
        const double *a = dt + (size_t)(d0 + j) * kEvalCols, *b = gt + (size_t)(g0 + i) * kEvalCols;
        const size_t at = (size_t)j * ng + i;
        o[at] = image_overlap(a, b, true);
        BoxPre A, B;
        float area_a, area_b;
        bev_pre(a, A, area_a);
        bev_pre(b, B, area_b);
        const float inter = box_overlap(A, B, s_px + threadIdx.x, s_py + threadIdx.x, s_pa + threadIdx.x, 128);
        // rotate_iou_gpu_eval's fp32 IoU (criterion -1)
        o[n_pairs + at] = (double)__fdiv_rn(inter, __fsub_rn(__fadd_rn(area_b, area_a), inter));
        // d3_box_overlap_kernel (eval.py:120-145): height range [y - h, y] and the volumes l*h*w in double on top of the fp32
        // BEV intersection, stored into the reference's fp32 matrix
        double v = 0.0;
        if (inter > 0.f) {
            const double iw = __dsub_rn(fmin(a[C_Y], b[C_Y]), fmax(__dsub_rn(a[C_Y], a[C_H]), __dsub_rn(b[C_Y], b[C_H])));
            if (iw > 0.0) {
                const double va = __dmul_rn(__dmul_rn(a[C_L], a[C_H]), a[C_W]), vb = __dmul_rn(__dmul_rn(b[C_L], b[C_H]), b[C_W]);
                const double inc = __dmul_rn(iw, (double)inter);
                v = (double)(float)__ddiv_rn(inc, __dsub_rn(__dadd_rn(va, vb), inc));
            }
        }
        o[2 * n_pairs + at] = v;
    }
}

// ------------------------------------------------------------------------------------------------ clean
__device__ __forceinline__ double min_height(int d) { return d == 0 ? 40.0 : 25.0; }

// blockIdx.y = class * 3 + difficulty; rows of both tables.  ig_gt / ig_dt (3 nc, rows) int8, nvalid (3 nc)
__global__ void __launch_bounds__(256) eval_clean_kernel(EvalCfg cfg, const double *__restrict__ gt, int n_gt,
                                                          const double *__restrict__ dt, int n_dt, signed char *__restrict__ ig_gt,
                                                          signed char *__restrict__ ig_dt, int *__restrict__ nvalid) {
    const int cl = blockIdx.y, cls = cfg.cls[cl / 3], diff = cl % 3;
    const int r = blockIdx.x * 256 + threadIdx.x;
    if (r < n_gt) {
        const double *g = gt + (size_t)r * kEvalCols;
        const int code = (int)g[C_CLS];
        const int vc = code == cls ? 1 : ((cls == 1 && code == 4) || (cls == 0 && code == 3)) ? 0 : -1;
        const double max_trunc = diff == 0 ? 0.15 : (diff == 1 ? 0.3 : 0.5);
        const bool ignore = g[C_OCC] > (double)diff || g[C_TRUNC] > max_trunc || __dsub_rn(g[C_Y2], g[C_Y1]) <= min_height(diff);
        const int ig = (vc == 1 && !ignore) ? 0 : ((vc == 0 || (ignore && vc == 1)) ? 1 : -1);
        ig_gt[(size_t)cl * n_gt + r] = (signed char)ig;
        if (ig == 0) atomicAdd(&nvalid[cl], 1);
    }
    if (r < n_dt) {
        const double *d = dt + (size_t)r * kEvalCols;
        const double h = fabs(__dsub_rn(d[C_Y2], d[C_Y1]));
        ig_dt[(size_t)cl * n_dt + r] = (signed char)(h < min_height(diff) ? 1 : ((int)d[C_CLS] == cls ? 0 : -1));
    }
}

// ------------------------------------------------------------------------------------------------ matching
struct ImageView {
    int g0, ng, d0, nd;
    const double *ov;               // this image's (dt x gt) matrix of the config's metric
    const signed char *igg, *igd;   // clean flags of the config's (class, difficulty)
};

__device__ __forceinline__ ImageView image_view(int img, int metric, int cl, const int *gt_off, const int *dt_off, const int *dt_count,
                                                const long long *pair_off, const double *ov, long long n_pairs,
                                                const signed char *ig_gt, int n_gt, const signed char *ig_dt, int n_dt) {
    ImageView v;
    v.g0 = gt_off[img];
    v.ng = gt_off[img + 1] - v.g0;
    v.d0 = dt_off[img];
    v.nd = min(dt_count[img], min(dt_off[img + 1] - v.d0, kMaxDetPerImage));
    v.ov = ov + metric * n_pairs + pair_off[img];
    v.igg = ig_gt + (size_t)cl * n_gt + v.g0;
    v.igd = ig_dt + (size_t)cl * n_dt + v.d0;
    return v;
}

// pass 1 (compute_fp=False): per GT, among the unassigned detections with ignored_det != -1 and overlap > min_overlap,
// the highest score wins (lowest index on ties: the reference compares `>` against NO_DETECTION = -1e7).  A TP's score
// is appended to its config's candidate list (the order does not matter: the list is sorted next).
__global__ void __launch_bounds__(256) eval_pass1_kernel(EvalCfg cfg, int n_img, int nconf, const double *__restrict__ dt,
                                                          const int *__restrict__ gt_off, const int *__restrict__ dt_off,
                                                          const int *__restrict__ dt_count, const long long *__restrict__ pair_off,
                                                          const double *__restrict__ ov, long long n_pairs,
                                                          const signed char *__restrict__ ig_gt, int n_gt,
                                                          const signed char *__restrict__ ig_dt, int n_dt, int *__restrict__ tp_count,
                                                          double *__restrict__ tp_scores, int score_stride) {
    const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (w >= n_img * nconf) return;
    const int q = w / n_img, img = w - q * n_img;
    const ConfigId id = config_of(q, cfg.nc, cfg.ns);
    const double mo = cfg.min_ov[id.k][id.metric][id.c];
    const ImageView v = image_view(img, id.metric, id.c * 3 + id.diff, gt_off, dt_off, dt_count, pair_off, ov, n_pairs, ig_gt, n_gt, ig_dt, n_dt);
    unsigned assigned = 0;      // bit s: detection lane + 32 s
    for (int i = 0; i < v.ng; ++i) {
        const int ig = v.igg[i];
        if (ig == -1) continue;
        double best = -10000000.0;
        int bj = 0x7fffffff;
        for (int s = 0, j = lane; j < v.nd; ++s, j += 32) {
            if (v.igd[j] == -1 || ((assigned >> s) & 1u)) continue;
            const double sc = dt[(size_t)(v.d0 + j) * kEvalCols + C_SCORE];
            if (v.ov[(size_t)j * v.ng + i] > mo && sc > best) { best = sc; bj = j; }
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, d);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, d);
            if (ob > best || (ob == best && oj < bj)) { best = ob; bj = oj; }
        }
        if (bj == 0x7fffffff) continue;
        if (lane == 0 && ig == 0 && v.igd[bj] == 0) {
            const int p = atomicAdd(&tp_count[q], 1);
            tp_scores[(size_t)q * score_stride + p] = best;
        }
        if ((bj & 31) == lane) assigned |= 1u << (bj >> 5);
    }
}

// one CTA per config: sort the TP scores in descending order (bitonic, in place in global memory, padded with -inf to a
// power of two) and pick get_thresholds' ranks.  With the recall fixed between two picks, "take rank i" is monotone in i
// (both rounded differences are monotone in the rounded recalls), so each pick is a binary search; the last rank is
// always taken.  Same picks as the sequential loop, in the same double arithmetic.
__global__ void __launch_bounds__(512) eval_thresholds_kernel(int nc, int ns, const int *__restrict__ nvalid, const int *__restrict__ tp_count,
                                                               double *__restrict__ tp_scores, int score_stride, double *__restrict__ thr,
                                                               int *__restrict__ nthr) {
    const int q = blockIdx.x, tid = threadIdx.x;
    const ConfigId id = config_of(q, nc, ns);
    const int n = tp_count[q];
    double *s = tp_scores + (size_t)q * score_stride;
    int pad = 1;
    while (pad < n) pad <<= 1;
    for (int e = n + tid; e < pad; e += 512) s[e] = -CUDART_INF;
    __syncthreads();
    for (int k = 2; k <= pad; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int e = tid; e < pad; e += 512) {
                const int p = e ^ j;
                if (p > e) {
                    const bool desc = (e & k) == 0;
                    const double a = s[e], b = s[p];
                    if (desc ? a < b : a > b) { s[e] = b; s[p] = a; }
                }
            }
            __syncthreads();
        }
    }
    if (tid != 0) return;
    const double num_gt = (double)nvalid[id.c * 3 + id.diff];
    double cur = 0.0;
    int cnt = 0;
    for (int i = 0; i < n && cnt < kSamplePts;) {
        int lo = i, hi = n - 1;     // first rank in [i, n-2] the loop takes, else n-1
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            const double l = (double)(mid + 1) / num_gt, r = (double)(mid + 2) / num_gt;
            if (!((r - cur) < (cur - l))) hi = mid; else lo = mid + 1;
        }
        thr[q * kSamplePts + cnt++] = s[lo];
        cur += 1.0 / 40.0;
        i = lo + 1;
    }
    nthr[q] = cnt;
}

// pass 2 (compute_fp=True), per (image, config), every threshold: detections with score < thresh are skipped.  Per GT,
// among the remaining candidates (overlap > min_overlap, unassigned, ignored_det != -1) the one with ignored_det == 0 and
// the largest overlap wins (lowest index on ties), else the lowest-index one with ignored_det == 1 -- eval.py:198-223's
// rule, as min_overlap > 0.  fp = unassigned detections with ignored_det == 0, minus (metric 0) those whose
// intersection over their own area with a DontCare box exceeds min_overlap.
__global__ void __launch_bounds__(256, 2) eval_pass2_kernel(EvalCfg cfg, int n_img, int nconf, const double *__restrict__ gt,
                                                          const double *__restrict__ dt, const int *__restrict__ gt_off,
                                                          const int *__restrict__ dt_off, const int *__restrict__ dt_count,
                                                          const long long *__restrict__ pair_off, const double *__restrict__ ov,
                                                          long long n_pairs, const signed char *__restrict__ ig_gt, int n_gt,
                                                          const signed char *__restrict__ ig_dt, int n_dt, const double *__restrict__ thr,
                                                          const int *__restrict__ nthr, int *__restrict__ pr, double *__restrict__ sim_img) {
    const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (w >= n_img * nconf) return;
    const int q = w / n_img, img = w - q * n_img;
    const ConfigId id = config_of(q, cfg.nc, cfg.ns);
    const double mo = cfg.min_ov[id.k][id.metric][id.c];
    const ImageView v = image_view(img, id.metric, id.c * 3 + id.diff, gt_off, dt_off, dt_count, pair_off, ov, n_pairs, ig_gt, n_gt, ig_dt, n_dt);
    // per lane: its detections' eligibility for the DontCare rule (metric 0), independent of the threshold
    unsigned near_dc = 0;
    if (id.metric == 0) {
        for (int s = 0, j = lane; j < v.nd; ++s, j += 32) {
            const double *a = dt + (size_t)(v.d0 + j) * kEvalCols;
            for (int i = 0; i < v.ng; ++i) {
                const double *b = gt + (size_t)(v.g0 + i) * kEvalCols;
                if ((int)b[C_CLS] == kCodeDontCare && image_overlap(a, b, false) > mo) { near_dc |= 1u << s; break; }
            }
        }
    }
    const int nt = nthr[q];
    for (int t = 0; t < nt; ++t) {
        const double th = thr[q * kSamplePts + t];
        unsigned usable = 0, assigned = 0, ig0 = 0;
        for (int s = 0, j = lane; j < v.nd; ++s, j += 32) {
            const int f = v.igd[j];
            if (f != -1 && !(dt[(size_t)(v.d0 + j) * kEvalCols + C_SCORE] < th)) usable |= 1u << s;
            if (f == 0) ig0 |= 1u << s;
        }
        int tp = 0, fn = 0;
        double sim = 0.0;
        for (int i = 0; i < v.ng; ++i) {
            const int ig = v.igg[i];
            if (ig == -1) continue;
            double bo = -1.0;
            int bj = 0x7fffffff, b1 = 0x7fffffff;
            for (int s = 0, j = lane; j < v.nd; ++s, j += 32) {
                if (!((usable & ~assigned) >> s & 1u)) continue;
                const double o = v.ov[(size_t)j * v.ng + i];
                if (!(o > mo)) continue;
                if ((ig0 >> s) & 1u) {
                    if (o > bo) { bo = o; bj = j; }
                } else if (b1 == 0x7fffffff) {
                    b1 = j;
                }
            }
#pragma unroll
            for (int d = 16; d; d >>= 1) {
                const double ob = __shfl_xor_sync(0xffffffffu, bo, d);
                const int oj = __shfl_xor_sync(0xffffffffu, bj, d);
                if (ob > bo || (ob == bo && oj < bj)) { bo = ob; bj = oj; }
                b1 = min(b1, __shfl_xor_sync(0xffffffffu, b1, d));
            }
            const int det = bj != 0x7fffffff ? bj : b1;
            if (det == 0x7fffffff) {
                if (ig == 0) ++fn;
                continue;
            }
            if (ig == 0 && bj != 0x7fffffff) {
                ++tp;
                if (id.metric == 0) {
                    const double delta = __dsub_rn(gt[(size_t)(v.g0 + i) * kEvalCols + C_ALPHA], dt[(size_t)(v.d0 + det) * kEvalCols + C_ALPHA]);
                    // (1 + cos(delta)) / 2; cospi needs no slow-path argument reduction (cos's is a call that spills
                    // here), and rounding delta / pi moves a term by ~1e-16
                    sim = __dadd_rn(sim, __dadd_rn(1.0, cospi(delta * 0.31830988618379067)) / 2.0);
                }
            }
            if ((det & 31) == lane) assigned |= 1u << (det >> 5);
        }
        const unsigned left = usable & ~assigned & ig0;
        int fp = __popc(left) - (id.metric == 0 ? __popc(left & near_dc) : 0);
#pragma unroll
        for (int d = 16; d; d >>= 1) fp += __shfl_xor_sync(0xffffffffu, fp, d);
        if (lane == 0) {
            int *p = pr + ((size_t)q * kSamplePts + t) * 3;
            if (tp) atomicAdd(p, tp);
            if (fp) atomicAdd(p + 1, fp);
            if (fn) atomicAdd(p + 2, fn);
            if (id.metric == 0) sim_img[((size_t)q * kSamplePts + t) * n_img + img] = (tp > 0 || fp > 0) ? sim : 0.0;
        }
    }
}

// np.max semantics: a NaN anywhere in the slice gives NaN
__device__ __forceinline__ double nan_max(double a, double b) { return (isnan(a) || isnan(b)) ? CUDART_NAN : fmax(a, b); }

// one CTA per config, one thread per threshold: the similarity summed over images in image order, the rates in double,
// suffix maxima over the thresholds.  out (nconf, 41, kOutPerThr), then the AOS flag (eval.py:636-641: the first
// detection annotation with rows decides; AOS unless its first alpha is -10), then nthr (nconf)
__global__ void __launch_bounds__(64) eval_finish_kernel(int nc, int ns, int n_img, const int *__restrict__ pr, const double *__restrict__ sim_img,
                                                          const double *__restrict__ thr, const int *__restrict__ nthr,
                                                          const double *__restrict__ dt, const int *__restrict__ dt_off,
                                                          const int *__restrict__ dt_count, int nconf, double *__restrict__ out) {
    __shared__ double s_v[3][kSamplePts];
    const int q = blockIdx.x, t = threadIdx.x;
    const ConfigId id = config_of(q, nc, ns);
    const int nt = nthr[q];
    double *o = out + (size_t)q * kSamplePts * kOutPerThr;
    if (t < kSamplePts) {
        const int *p = pr + ((size_t)q * kSamplePts + t) * 3;
        const double tp = p[0], fp = p[1], fn = p[2];
        double sim = 0.0;
        if (id.metric == 0 && t < nt)
            for (int img = 0; img < n_img; ++img) sim = __dadd_rn(sim, sim_img[((size_t)q * kSamplePts + t) * n_img + img]);
        const bool on = t < nt;
        s_v[0][t] = on ? tp / (tp + fn) : 0.0;
        s_v[1][t] = on ? tp / (tp + fp) : 0.0;
        s_v[2][t] = on ? sim / (tp + fp) : 0.0;
        o[t * kOutPerThr + 0] = tp; o[t * kOutPerThr + 1] = fp; o[t * kOutPerThr + 2] = fn; o[t * kOutPerThr + 3] = sim;
        o[t * kOutPerThr + 7] = on ? thr[q * kSamplePts + t] : 0.0;
    }
    __syncthreads();
    if (t < 3) {
        double m = s_v[t][kSamplePts - 1];
        for (int i = kSamplePts - 1; i >= 0; --i) {
            m = i == kSamplePts - 1 ? m : nan_max(s_v[t][i], m);
            o[i * kOutPerThr + 4 + t] = i < nt ? m : s_v[t][i];
        }
    }
    if (q == 0 && t == 0) {
        double aos = 0.0;
        for (int img = 0; img < n_img; ++img)
            if (dt_count[img] > 0) {
                aos = dt[(size_t)dt_off[img] * kEvalCols + C_ALPHA] != -10.0 ? 1.0 : 0.0;
                break;
            }
        out[(size_t)nconf * kSamplePts * kOutPerThr] = aos;
    }
    if (t == 0) out[(size_t)nconf * kSamplePts * kOutPerThr + 1 + q] = nt;
}

// ------------------------------------------------------------------------------------------------ in-memory detections
// the rows save_kitti_format writes (valid and selected, in row order) of scene k go to image slot[k]'s rows, each field
// quantised to the text's "%.4f" when `rounding`: rint((double)f * 1e4) / 1e4 is exact arithmetic up to the final
// division, so it is the double that parsing the text gives.  One warp per scene.
__device__ __forceinline__ double q4(float f, int rounding) { return rounding ? rint((double)f * 1e4) / 1e4 : (double)f; }

__global__ void __launch_bounds__(128, 4) eval_add_detections_kernel(int b, int m, const float *__restrict__ boxes3d, const float *__restrict__ scores,
                                                                   const float *__restrict__ img_boxes, const float *__restrict__ alpha,
                                                                   const int *__restrict__ valid, const int *__restrict__ select,
                                                                   const int *__restrict__ slot, int rounding, int code, double *__restrict__ dt,
                                                                   const int *__restrict__ dt_off, int *__restrict__ dt_count) {
    const int k = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (k >= b) return;
    const int img = slot[k];
    const int d0 = dt_off[img], cap = dt_off[img + 1] - d0;
    int n = 0;
    for (int j0 = 0; j0 < m; j0 += 32) {
        const int j = j0 + lane;
        const size_t r = (size_t)k * m + j;
        const bool keep = j < m && valid[r] != 0 && select[r] != 0;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        const int pos = n + __popc(bal & ((1u << lane) - 1u));
        if (keep && pos < cap) {
            const float *q = boxes3d + r * 7, *ib = img_boxes + r * 4;
            double *d = dt + (size_t)(d0 + pos) * kEvalCols;
            d[C_X1] = q4(ib[0], rounding); d[C_Y1] = q4(ib[1], rounding); d[C_X2] = q4(ib[2], rounding); d[C_Y2] = q4(ib[3], rounding);
            d[C_ALPHA] = q4(alpha[r], rounding);
            d[C_TRUNC] = -1.0; d[C_OCC] = -1.0;
            d[C_L] = q4(q[5], rounding); d[C_H] = q4(q[3], rounding); d[C_W] = q4(q[4], rounding);
            d[C_X] = q4(q[0], rounding); d[C_Y] = q4(q[1], rounding); d[C_Z] = q4(q[2], rounding);
            d[C_RY] = q4(q[6], rounding);
            d[C_SCORE] = q4(scores[r], rounding);
            d[C_CLS] = (double)code;
        }
        n += __popc(bal);
    }
    if (lane == 0) dt_count[img] = min(n, cap);
}

// ------------------------------------------------------------------------------------------------ workspace
struct EvalWs {
    size_t ig_gt, ig_dt, ints, n_ints, nvalid, tp_count, nthr, pr, tp_scores, thr, sim, dt_f, count_f, total;
    int score_stride;
};

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// `filter`: room for the score-filtered detection table and counts, after everything else
static EvalWs eval_ws(int n_img, int n_gt, int n_dt, int nc, int ns, bool filter) {
    EvalWs w;
    const int ncl = 3 * nc, nconf = 9 * ns * nc;
    int pad = 1;
    while (pad < n_gt) pad <<= 1;
    w.score_stride = pad;
    size_t off = 0;
    w.ig_gt = off; off = align256(off + (size_t)ncl * n_gt);
    w.ig_dt = off; off = align256(off + (size_t)ncl * n_dt);
    w.ints = off;
    w.nvalid = 0;
    w.tp_count = ncl;
    w.nthr = ncl + nconf;
    w.pr = ncl + 2 * (size_t)nconf;
    w.n_ints = w.pr + (size_t)nconf * kSamplePts * 3;
    off = align256(off + w.n_ints * sizeof(int));
    w.tp_scores = off; off = align256(off + (size_t)nconf * pad * sizeof(double));
    w.thr = off; off = align256(off + (size_t)nconf * kSamplePts * sizeof(double));
    w.sim = off; off = align256(off + (size_t)3 * ns * nc * kSamplePts * n_img * sizeof(double));    // the metric-0 configs
    w.dt_f = off; off = filter ? align256(off + (size_t)n_dt * kEvalCols * sizeof(double)) : off;
    w.count_f = off; off = filter ? align256(off + (size_t)n_img * sizeof(int)) : off;
    w.total = off;
    return w;
}

}  // namespace prb

using namespace prb;

extern "C" size_t prb_kitti_eval_workspace_bytes(int n_img, int n_gt, int n_dt, int num_classes) {
    if (n_img < 1 || n_gt < 0 || n_dt < 0 || num_classes < 1 || num_classes > kMaxEvalClasses) return 0;
    return eval_ws(n_img, n_gt, n_dt, num_classes, 2, false).total;
}

extern "C" size_t prb_kitti_eval_sets_workspace_bytes(int n_img, int n_gt, int n_dt, int num_classes, int num_sets) {
    if (n_img < 1 || n_gt < 0 || n_dt < 0 || num_classes < 1 || num_classes > kMaxEvalClasses || num_sets < 1 || num_sets > kMaxOverlapSets)
        return 0;
    return eval_ws(n_img, n_gt, n_dt, num_classes, num_sets, true).total;
}

extern "C" int prb_kitti_eval_sets(int n_img, int num_classes, const int *classes, int num_sets, const double *min_overlaps,
                                   double score_thresh, const double *gt, const int *gt_off, int n_gt, const double *dt,
                                   const int *dt_off, const int *dt_count, int n_dt, int max_det, const long long *pair_off,
                                   long long n_pairs, double *overlaps, double *out, void *workspace, size_t workspace_bytes,
                                   void *stream) {
    PRB_REQUIRE(n_img >= 1 && n_gt >= 0 && n_dt >= 0 && n_pairs >= 0 && classes && min_overlaps && gt_off && dt_off && dt_count &&
                    pair_off && out && (n_pairs == 0 || overlaps) && (n_gt == 0 || gt) && (n_dt == 0 || dt),
                "kitti_eval: bad arguments");
    PRB_REQUIRE(num_classes >= 1 && num_classes <= kMaxEvalClasses, "kitti_eval: %d classes (1..%d)", num_classes, kMaxEvalClasses);
    PRB_REQUIRE(num_sets >= 1 && num_sets <= kMaxOverlapSets, "kitti_eval: %d overlap sets (1..%d)", num_sets, kMaxOverlapSets);
    PRB_REQUIRE(max_det >= 0 && max_det <= kMaxDetPerImage, "kitti_eval: %d detection rows per image > %d", max_det, kMaxDetPerImage);
    PRB_REQUIRE((long long)n_img * 9 * num_sets * num_classes <= 0x7fffffffLL / 32, "kitti_eval: %d images is too many", n_img);
    EvalCfg cfg;
    cfg.nc = num_classes;
    cfg.ns = num_sets;
    for (int c = 0; c < num_classes; ++c) {
        PRB_REQUIRE(classes[c] >= 0 && classes[c] <= 2, "kitti_eval: class %d is not 0 (Car), 1 (Pedestrian) or 2 (Cyclist)", classes[c]);
        cfg.cls[c] = classes[c];
        for (int k = 0; k < num_sets; ++k)
            for (int m = 0; m < 3; ++m) {
                const double v = min_overlaps[(k * 3 + m) * num_classes + c];
                PRB_REQUIRE(v > 0.0 && v < 1.0, "kitti_eval: min_overlap %g outside (0, 1)", v);
                cfg.min_ov[k][m][c] = v;
            }
    }
    // the reference's rule (evaluate.py:22): a threshold filters only when it is > 0
    const bool filter = score_thresh > 0.0;
    const EvalWs w = eval_ws(n_img, n_gt, n_dt, num_classes, num_sets, filter);
    PRB_REQUIRE(workspace && workspace_bytes >= w.total, "kitti_eval: workspace of %zu bytes < %zu", workspace_bytes, w.total);
    const int nconf = 9 * num_sets * num_classes, ncl = 3 * num_classes;
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    signed char *ig_gt = (signed char *)(ws + w.ig_gt), *ig_dt = (signed char *)(ws + w.ig_dt);
    int *ints = (int *)(ws + w.ints);
    int *nvalid = ints + w.nvalid, *tp_count = ints + w.tp_count, *nthr = ints + w.nthr, *pr = ints + w.pr;
    double *tp_scores = (double *)(ws + w.tp_scores), *thr = (double *)(ws + w.thr), *sim = (double *)(ws + w.sim);
    PRB_CUDA(cudaMemsetAsync(ints, 0, w.n_ints * sizeof(int), st));

    if (filter) {
        double *dt_f = (double *)(ws + w.dt_f);
        int *count_f = (int *)(ws + w.count_f);
        eval_filter_kernel<<<ceil_div(n_img, 4), 128, 0, st>>>(n_img, score_thresh, dt, dt_off, dt_count, dt_f, count_f);
        if (int rc = check_launch("eval_filter_kernel")) return rc;
        dt = dt_f;
        dt_count = count_f;
    }
    eval_overlaps_kernel<<<n_img, 128, 0, st>>>(gt, gt_off, dt, dt_off, dt_count, pair_off, n_pairs, overlaps);
    if (int rc = check_launch("eval_overlaps_kernel")) return rc;
    const int rows = max(1, max(n_gt, n_dt));
    eval_clean_kernel<<<dim3(ceil_div(rows, 256), ncl), 256, 0, st>>>(cfg, gt, n_gt, dt, n_dt, ig_gt, ig_dt, nvalid);
    if (int rc = check_launch("eval_clean_kernel")) return rc;
    const int warps = n_img * nconf;
    eval_pass1_kernel<<<ceil_div(warps, 8), 256, 0, st>>>(cfg, n_img, nconf, dt, gt_off, dt_off, dt_count, pair_off, overlaps, n_pairs, ig_gt,
                                                          n_gt, ig_dt, n_dt, tp_count, tp_scores, w.score_stride);
    if (int rc = check_launch("eval_pass1_kernel")) return rc;
    eval_thresholds_kernel<<<nconf, 512, 0, st>>>(num_classes, num_sets, nvalid, tp_count, tp_scores, w.score_stride, thr, nthr);
    if (int rc = check_launch("eval_thresholds_kernel")) return rc;
    eval_pass2_kernel<<<ceil_div(warps, 8), 256, 0, st>>>(cfg, n_img, nconf, gt, dt, gt_off, dt_off, dt_count, pair_off, overlaps, n_pairs,
                                                          ig_gt, n_gt, ig_dt, n_dt, thr, nthr, pr, sim);
    if (int rc = check_launch("eval_pass2_kernel")) return rc;
    eval_finish_kernel<<<nconf, 64, 0, st>>>(num_classes, num_sets, n_img, pr, sim, thr, nthr, dt, dt_off, dt_count, nconf, out);
    return check_launch("eval_finish_kernel");
}

extern "C" int prb_kitti_eval(int n_img, int num_classes, const int *classes, const double *min_overlaps, const double *gt,
                              const int *gt_off, int n_gt, const double *dt, const int *dt_off, const int *dt_count, int n_dt,
                              int max_det, const long long *pair_off, long long n_pairs, double *overlaps, double *out,
                              void *workspace, size_t workspace_bytes, void *stream) {
    return prb_kitti_eval_sets(n_img, num_classes, classes, 2, min_overlaps, -1.0, gt, gt_off, n_gt, dt, dt_off, dt_count, n_dt, max_det,
                               pair_off, n_pairs, overlaps, out, workspace, workspace_bytes, stream);
}

extern "C" int prb_kitti_eval_add_detections(int b, int m, const float *boxes3d, const float *scores, const float *img_boxes,
                                             const float *alpha, const int *valid, const int *select, const int *slot, int text_rounding,
                                             int class_code, double *dt, const int *dt_off, int *dt_count, void *stream) {
    PRB_REQUIRE(b >= 0 && m >= 0 && slot && dt_off && dt_count && (b * m == 0 || (boxes3d && scores && img_boxes && alpha && valid && select && dt)),
                "kitti_eval_add_detections: bad arguments");
    if (b == 0) return 0;
    eval_add_detections_kernel<<<ceil_div(b, 4), 128, 0, (cudaStream_t)stream>>>(b, m, boxes3d, scores, img_boxes, alpha, valid, select, slot,
                                                                                text_rounding, class_code, dt, dt_off, dt_count);
    return check_launch("eval_add_detections_kernel");
}
