// kitti_io.cu -- the two ends of the hot path (SURVEY.md 8(f) rank 4), batched on the device:
//
//   input side   lib/datasets/kitti_rcnn_dataset.py:246-394 (get_rpn_sample + generate_rpn_training_labels):
//                lidar -> rectified camera frame, image / range validity, the 16384-point draw (all far points + a
//                random subset of the near ones, shuffled), augmentation of the drawn points, per-point RPN labels;
//   output side  tools/eval_rcnn.py:69-94 (save_kitti_format): 3D boxes -> image boxes, validity, alpha, text lines.
//
// The reference does this per scene in numpy on the host (Delaunay triangulations for the labels, one text file per
// scene); at several thousand scenes per second and GPU that is the bottleneck of a real run.  Here a batch of raw
// scans is prepared by four launches with no host round trip: the result is the (B, npoints, 3|4) network input and
// the labels, already in HBM.
#include <math_constants.h>
#include <stdio.h>
#include <string.h>

#include "common.cuh"

namespace prb {

// ---------------------------------------------------------------------------------------------------- prepare
// per scene: M (4x3, rect = [x y z 1] . M, the reference's V2C^T . R0^T computed by the caller in fp32), P2 (3x4),
// image height, width, then the optional range box (x0,x1,y0,y1,z0,z1) -- 32 floats
constexpr int kCalibFloats = 32;

__device__ __forceinline__ int scene_of(const int *__restrict__ offsets, int b, int i) {
    int lo = 0, hi = b;                 // offsets[lo] <= i < offsets[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (offsets[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) kitti_prepare_kernel(int b, int total, const int *__restrict__ offsets,
                                                             const float *__restrict__ lidar, int stride,
                                                             const float *__restrict__ calib, int use_range,
                                                             float *__restrict__ rect, unsigned char *__restrict__ flags,
                                                             int *__restrict__ counts) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    const bool inb = i < total;
    const int s = inb ? scene_of(offsets, b, i) : -1;
    bool ok = false, near = true;
    if (inb) {
        const float *c = calib + (size_t)s * kCalibFloats;
        const float x = lidar[(size_t)i * stride], y = lidar[(size_t)i * stride + 1], z = lidar[(size_t)i * stride + 2];
        float r[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) r[k] = __fmaf_rn(z, c[6 + k], __fmaf_rn(y, c[3 + k], __fmul_rn(x, c[k]))) + c[9 + k];
        const float *P = c + 12;
        float h[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            h[k] = __fmaf_rn(r[2], P[k * 4 + 2], __fmaf_rn(r[1], P[k * 4 + 1], __fmul_rn(r[0], P[k * 4]))) + P[k * 4 + 3];
        const float u = __fdiv_rn(h[0], r[2]), v = __fdiv_rn(h[1], r[2]);     // the reference divides by the rect depth
        const float depth = h[2] - P[11];
        const float H = c[24], W = c[25];
        ok = u >= 0.f && u < W && v >= 0.f && v < H && depth >= 0.f;
        if (use_range) ok = ok && r[0] >= c[26] && r[0] <= c[27] && r[1] >= c[28] && r[1] <= c[29] && r[2] >= c[30] && r[2] <= c[31];
        near = r[2] < 40.0f;
        rect[(size_t)i * 3] = r[0]; rect[(size_t)i * 3 + 1] = r[1]; rect[(size_t)i * 3 + 2] = r[2];
        flags[i] = (unsigned char)((ok ? 1 : 0) | (near ? 2 : 0));
    }
    if (counts) {
        // one atomic per warp and scene (a warp nearly always lies inside one scene): per-point atomics on the 2*b counters
        // serialise the whole kernel
        const unsigned grp = __match_any_sync(0xffffffffu, s);
        const unsigned okm = __ballot_sync(0xffffffffu, ok) & grp;
        const unsigned farm = __ballot_sync(0xffffffffu, ok && !near) & grp;
        if (inb && (threadIdx.x & 31) == __ffs(grp) - 1) {
            if (okm) atomicAdd(&counts[s * 2], __popc(okm));
            if (farm) atomicAdd(&counts[s * 2 + 1], __popc(farm));
        }
    }
}

// ---------------------------------------------------------------------------------------------------- draw
// block-wide exclusive scan of one int per thread (1024 threads); returns the exclusive prefix, total in *sum
__device__ __forceinline__ int block_excl_scan(int v, int *s_warp, int *sum) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
    }
    __syncthreads();
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = s_warp[lane];
        int winc = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, winc, d);
            if (lane >= d) winc += o;
        }
        s_warp[lane] = winc - w;
        if (lane == 31) s_warp[32] = winc;
    }
    __syncthreads();
    *sum = s_warp[32];
    return s_warp[warp] + inc - v;
}

// One CTA per scene.  pool / base as in kitti_rcnn_dataset.py:285-303:
//   nv >  npoints: base = valid far points, pool = valid near points, need = npoints - |base|
//   nv <= npoints: base = all valid points, pool = all valid points,  need = npoints - nv   (extra copies)
// `need` pool members are chosen without replacement (the `need` smallest 32-bit hash keys, ties by index), then
// base + chosen are put in a random order (bitonic sort by a second, independent key).  choice[] holds indices into
// the scene's RAW points.  Deviations from the reference, both where its np.random.choice would raise: more far
// points than npoints -> the draw is taken from all valid points; fewer than npoints/2 valid points -> extra copies
// cycle through the valid points.  status[scene]: 0 ok, 1 no valid point (choice = 0, rows zero).
__global__ void __launch_bounds__(1024) kitti_draw_kernel(int b, const int *__restrict__ offsets,
                                                           const unsigned char *__restrict__ flags, int npoints, int npad,
                                                           uint32_t seed, int *__restrict__ cand, int *__restrict__ choice,
                                                           int *__restrict__ status) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    uint32_t *s_key = reinterpret_cast<uint32_t *>(s_raw);            // npad sort keys
    int *s_idx = reinterpret_cast<int *>(s_raw + (size_t)npad * 4);   // npad payloads
    __shared__ int s_hist[256];
    __shared__ int s_warp[33];
    __shared__ int s_cnt[4];
    const int scene = blockIdx.x, tid = threadIdx.x;
    const int beg = offsets[scene], n = offsets[scene + 1] - beg;
    const unsigned char *f = flags + beg;
    int *cnd = cand + beg;      // compacted raw indices of the valid points, in index order

    // 1. compact the valid points (4 consecutive points per thread and scan step); count the far ones
    int nv = 0, far_mine = 0;
    for (int base = 0; base < n; base += 4096) {
        const int i0 = base + tid * 4;
        int okq[4], c = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int fl = i0 + q < n ? f[i0 + q] : 0;
            okq[q] = fl & 1;
            c += okq[q];
            far_mine += (fl & 1) && !(fl & 2);
        }
        int tot;
        int pos = nv + block_excl_scan(c, s_warp, &tot);
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (okq[q]) cnd[pos++] = i0 + q;
        nv += tot;
    }
    int nfar;
    (void)block_excl_scan(far_mine, s_warp, &nfar);
    __syncthreads();
    int *ch = choice + (size_t)scene * npoints;
    if (nv == 0) {
        for (int e = tid; e < npoints; e += 1024) ch[e] = 0;
        if (tid == 0 && status) status[scene] = 1;
        return;
    }
    if (tid == 0 && status) status[scene] = 0;
    // pool / base
    const bool sub = nv > npoints;                   // subsample
    const bool far_base = sub && nfar < npoints;     // base = far points, pool = near points
    const int nbase = sub ? (far_base ? nfar : 0) : nv;
    const int npool = sub ? (far_base ? nv - nfar : nv) : nv;
    int need = npoints - nbase;
    const int cycles = need / npool;                 // > 0 only when nv < npoints / 2 (whole extra copies)
    need -= cycles * npool;

    // 2. radix select: threshold key T such that exactly `need` pool members have (key, position) below it
    auto in_pool = [&](int i) { return !far_base || (f[i] & 2); };
    uint32_t prefix = 0;
    int remaining = need;        // how many still to take among the keys matching the prefix
    if (need > 0) {
        for (int pass = 3; pass >= 0; --pass) {
            if (tid < 256) s_hist[tid] = 0;
            __syncthreads();
            const uint32_t mask = pass == 3 ? 0u : (0xffffffffu << ((pass + 1) * 8));
            for (int e = tid; e < nv; e += 1024) {
                const int i = cnd[e];
                if (!in_pool(i)) continue;
                const uint32_t k = draw_key(seed, scene, i, 0x51ed27u);
                if ((k & mask) == (prefix & mask)) atomicAdd(&s_hist[(k >> (pass * 8)) & 255], 1);
            }
            __syncthreads();
            if (tid == 0) {
                int acc = 0, bin = 0;
                for (; bin < 256; ++bin) {
                    if (acc + s_hist[bin] >= remaining) break;
                    acc += s_hist[bin];
                }
                if (bin > 255) bin = 255;
                s_cnt[0] = bin; s_cnt[1] = acc;
            }
            __syncthreads();
            prefix |= (uint32_t)s_cnt[0] << (pass * 8);
            remaining -= s_cnt[1];
            __syncthreads();
        }
    }
    // keys < prefix are taken, keys == prefix: the first `remaining` in index order

    // 3. emit base + chosen (+ whole extra copies) into the sort buffers, 4 consecutive candidates per thread and scan step
    int out = 0, eq_seen = 0;
    for (int base = 0; base < nv; base += 4096) {
        const int e0 = base + tid * 4;
        int iq[4], takeq[4], eqq[4], eqs = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            iq[q] = 0; takeq[q] = 0; eqq[q] = 0;
            if (e0 + q < nv) {
                const int i = cnd[e0 + q];
                iq[q] = i;
                const bool pool = in_pool(i);
                const bool isbase = sub ? (far_base && !pool) : true;
                takeq[q] = isbase ? 1 : 0;
                if (pool && need > 0) {
                    const uint32_t k = draw_key(seed, scene, i, 0x51ed27u);
                    if (k < prefix) takeq[q] += 1;
                    else if (k == prefix) eqq[q] = 1;
                }
                if (pool) takeq[q] += cycles;
            }
            eqs += eqq[q];
        }
        int tot;
        int eqpos = eq_seen + block_excl_scan(eqs, s_warp, &tot);
        eq_seen += tot;
        int ts = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (eqq[q] && eqpos++ < remaining) takeq[q] += 1;
            ts += takeq[q];
        }
        int o = out + block_excl_scan(ts, s_warp, &tot);
#pragma unroll
        for (int q = 0; q < 4; ++q)
            for (int t = 0; t < takeq[q]; ++t, ++o)
                if (o < npoints) {
                    s_key[o] = draw_key(seed, scene, iq[q], 0xa511e9b3u + (uint32_t)t);
                    s_idx[o] = iq[q];
                }
        out += tot;
    }
    __syncthreads();
    for (int e = out + tid; e < npad; e += 1024) { s_key[e] = 0xffffffffu; s_idx[e] = 0x7fffffff; }
    if (out < npoints) {       // cannot happen (counts add up); keep the rows defined
        for (int e = out + tid; e < npoints; e += 1024) { s_key[e] = 0xfffffffeu; s_idx[e] = cnd[0]; }
    }
    __syncthreads();

    // 4. random order: bitonic sort by (key, idx)
    for (int k = 2; k <= npad; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int e = tid; e < npad; e += 1024) {
                const int p = e ^ j;
                if (p > e) {
                    const bool up = (e & k) == 0;
                    const uint32_t ka = s_key[e], kb = s_key[p];
                    const int ia = s_idx[e], ib = s_idx[p];
                    const bool gt = ka > kb || (ka == kb && ia > ib);
                    if (gt == up) { s_key[e] = kb; s_key[p] = ka; s_idx[e] = ib; s_idx[p] = ia; }
                }
            }
            __syncthreads();
        }
    }
    for (int e = tid; e < npoints; e += 1024) ch[e] = s_idx[e];
}

// gather the drawn points, intensity - 0.5, and the per-scene augmentation (rotation about y, scaling, x flip) in the
// reference's order (kitti_rcnn_dataset.py:526-568; rotate_pc_along_y: [x z] . [[c,-s],[s,c]]^T)
// aug (b,4) DOUBLE: cos, sin, scale, flip (0/1); nullptr = none.  The rotation is evaluated in fp64 and rounded once, as
// numpy does for a float32 array times a float64 matrix; the scale is a float32 multiply (numpy's weak-scalar rule).
__global__ void __launch_bounds__(256) kitti_gather_kernel(int b, int npoints, const int *__restrict__ offsets,
                                                            const float *__restrict__ rect, const float *__restrict__ lidar,
                                                            int stride, const int *__restrict__ choice,
                                                            const double *__restrict__ aug, const int *__restrict__ status,
                                                            int channels, float *__restrict__ pts_input,
                                                            float *__restrict__ pts_rect_out, float *__restrict__ intensity_out) {
    const int scene = blockIdx.y, e = blockIdx.x * 256 + threadIdx.x;
    if (e >= npoints) return;
    const int n = offsets[scene + 1] - offsets[scene];
    const size_t o = (size_t)scene * npoints + e;
    float x = 0.f, y = 0.f, z = 0.f, it = 0.f;
    if (n > 0 && !(status && status[scene] != 0)) {      // scenes without a valid point: zero rows
        const size_t i = (size_t)offsets[scene] + choice[o];
        x = rect[i * 3]; y = rect[i * 3 + 1]; z = rect[i * 3 + 2];
        it = stride > 3 ? lidar[i * stride + 3] - 0.5f : 0.f;
    }
    if (aug) {
        const double c = aug[scene * 4], s = aug[scene * 4 + 1];
        const float sc = (float)aug[scene * 4 + 2];
        if (c != 1.0 || s != 0.0) {
            const float nx = (float)__dadd_rn(__dmul_rn((double)x, c), __dmul_rn((double)z, -s));
            const float nz = (float)__dadd_rn(__dmul_rn((double)x, s), __dmul_rn((double)z, c));
            x = nx; z = nz;
        }
        if (sc != 1.f) { x = __fmul_rn(x, sc); y = __fmul_rn(y, sc); z = __fmul_rn(z, sc); }
        if (aug[scene * 4 + 3] != 0.0) x = -x;
    }
    if (pts_rect_out) { pts_rect_out[o * 3] = x; pts_rect_out[o * 3 + 1] = y; pts_rect_out[o * 3 + 2] = z; }
    if (intensity_out) intensity_out[o] = it;
    if (pts_input) {
        float *d = pts_input + o * channels;
        d[0] = x; d[1] = y; d[2] = z;
        if (channels > 3) d[3] = it;
    }
}

// ---------------------------------------------------------------------------------------------------- labels
// generate_rpn_training_labels (kitti_rcnn_dataset.py:355-391): boxes visited in order, later boxes overwrite.
// Inside test in the box frame (x_c = dx cos - dz sin, z_c = dx sin + dz cos from boxes3d_to_corners3d's rotation,
// kitti_utils.py:66-101) instead of a Delaunay triangulation of the 8 corners: same set up to points on a face.
__device__ __forceinline__ bool in_box(float px, float py, float pz, float cx, float cy, float cz, float h, float w, float l,
                                       float cosr, float sinr) {
    const float dy = py - cy;                      // box y is the bottom face; the body extends to cy - h
    if (dy > 0.f || dy < -h) return false;
    const float dx = px - cx, dz = pz - cz;
    const float xc = dx * cosr - dz * sinr, zc = dx * sinr + dz * cosr;
    return fabsf(xc) <= l * 0.5f && fabsf(zc) <= w * 0.5f;
}

constexpr int kMaxGt = 128;

__global__ void __launch_bounds__(256) rpn_labels_kernel(int n, int g, const float *__restrict__ pts,
                                                          const float *__restrict__ gt, const int *__restrict__ gt_count,
                                                          float extra, int *__restrict__ cls, float *__restrict__ reg) {
    __shared__ float s_gt[kMaxGt][9];
    const int scene = blockIdx.y;
    int ng = gt_count ? min(gt_count[scene], g) : g;
    for (int k = threadIdx.x; k < ng; k += 256) {
        const float *q = gt + ((size_t)scene * g + k) * 7;
#pragma unroll
        for (int c = 0; c < 7; ++c) s_gt[k][c] = q[c];
        float sn, cs;
        sincosf(q[6], &sn, &cs);
        s_gt[k][7] = cs; s_gt[k][8] = sn;
    }
    __syncthreads();
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    const float *p = pts + ((size_t)scene * n + j) * 3;
    const float px = p[0], py = p[1], pz = p[2];
    int c = 0;
    float r[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < ng; ++k) {
        const float *q = s_gt[k];
        if (!gt_count && q[3] == 0.f && q[4] == 0.f && q[5] == 0.f) continue;     // zero rows of a padded batch
        const bool fg = in_box(px, py, pz, q[0], q[1], q[2], q[3], q[4], q[5], q[7], q[8]);
        const bool big = in_box(px, py, pz, q[0], q[1] + extra, q[2], q[3] + 2.f * extra, q[4] + 2.f * extra,
                                q[5] + 2.f * extra, q[7], q[8]);
        if (fg) {
            c = 1;
            r[0] = __fsub_rn(q[0], px);
            r[1] = __fsub_rn(__fsub_rn(q[1], __fmul_rn(q[3], 0.5f)), py);
            r[2] = __fsub_rn(q[2], pz);
            r[3] = q[3]; r[4] = q[4]; r[5] = q[5]; r[6] = q[6];
        }
        if (fg != big) c = -1;
    }
    cls[(size_t)scene * n + j] = c;
    float *d = reg + ((size_t)scene * n + j) * 7;
#pragma unroll
    for (int k = 0; k < 7; ++k) d[k] = r[k];
}

// ---------------------------------------------------------------------------------------------------- output
// save_kitti_format (eval_rcnn.py:69-94): corners in fp32 (kitti_utils.py:66-101), projection in fp64 like the
// reference's np.matmul of a float64 homogeneous array (calibration.py:106-124)
// per_scene > 0: box i belongs to scene i / per_scene with its own P2 (12 floats) and image size hw (2 floats)
__global__ void __launch_bounds__(128) kitti_image_boxes_kernel(int n, const float *__restrict__ boxes,
                                                                 const float *__restrict__ P2_all, int per_scene,
                                                                 const float *__restrict__ hw_all, float img_h, float img_w,
                                                                 float *__restrict__ img_boxes, float *__restrict__ alpha,
                                                                 int *__restrict__ valid) {
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    const int scene = per_scene > 0 ? i / per_scene : 0;
    const float *P2 = P2_all + (size_t)scene * 12;
    if (hw_all) { img_h = hw_all[scene * 2]; img_w = hw_all[scene * 2 + 1]; }
    const float *q = boxes + (size_t)i * 7;
    const float x = q[0], y = q[1], z = q[2], h = q[3], w = q[4], l = q[5], ry = q[6];
    const float cs = cosf(ry), sn = sinf(ry);
    const float hl = l / 2.f, hw = w / 2.f;
    const float xs[4] = {hl, hl, -hl, -hl}, zs[4] = {hw, -hw, -hw, hw};
    double x1 = CUDART_INF, y1 = CUDART_INF, x2 = -CUDART_INF, y2 = -CUDART_INF;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float xc = xs[k & 3], zc = zs[k & 3], yc = k < 4 ? 0.f : -h;
        // [xc yc zc] . [[cos,0,-sin],[0,1,0],[sin,0,cos]]
        const float rx = __fadd_rn(__fmul_rn(xc, cs), __fmul_rn(zc, sn));
        const float rz = __fadd_rn(__fmul_rn(xc, -sn), __fmul_rn(zc, cs));
        const double X = (double)__fadd_rn(x, rx), Y = (double)__fadd_rn(y, yc), Z = (double)__fadd_rn(z, rz);
        const double pu = X * (double)P2[0] + Y * (double)P2[1] + Z * (double)P2[2] + (double)P2[3];
        const double pv = X * (double)P2[4] + Y * (double)P2[5] + Z * (double)P2[6] + (double)P2[7];
        const double pw = X * (double)P2[8] + Y * (double)P2[9] + Z * (double)P2[10] + (double)P2[11];
        const double u = pu / pw, v = pv / pw;
        x1 = fmin(x1, u); x2 = fmax(x2, u); y1 = fmin(y1, v); y2 = fmax(y2, v);
    }
    const double W1 = (double)img_w - 1.0, H1 = (double)img_h - 1.0;
    x1 = fmin(fmax(x1, 0.0), W1); x2 = fmin(fmax(x2, 0.0), W1);
    y1 = fmin(fmax(y1, 0.0), H1); y2 = fmin(fmax(y2, 0.0), H1);
    img_boxes[i * 4] = (float)x1; img_boxes[i * 4 + 1] = (float)y1; img_boxes[i * 4 + 2] = (float)x2; img_boxes[i * 4 + 3] = (float)y2;
    valid[i] = ((x2 - x1) < (double)img_w * 0.8 && (y2 - y1) < (double)img_h * 0.8) ? 1 : 0;
    const float beta = atan2f(z, x);
    const double sg = beta > 0.f ? 1.0 : (beta < 0.f ? -1.0 : 0.0);
    alpha[i] = (float)(-sg * 3.141592653589793 / 2.0 + (double)beta + (double)ry);
}

}  // namespace prb

using namespace prb;

extern "C" int prb_kitti_prepare_points(int b, int total, const int *offsets, const float *lidar, int stride, const float *calib,
                                        int use_range, float *rect, unsigned char *flags, int *counts, void *stream) {
    PRB_REQUIRE(b > 0 && total >= 0 && offsets && lidar && calib && rect && flags && stride >= 3, "kitti_prepare_points: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (counts) PRB_CUDA(cudaMemsetAsync(counts, 0, (size_t)b * 2 * sizeof(int), st));
    if (total == 0) return 0;
    kitti_prepare_kernel<<<ceil_div(total, 256), 256, 0, st>>>(b, total, offsets, lidar, stride, calib, use_range, rect, flags, counts);
    return check_launch("kitti_prepare_kernel");
}

static int draw_pad(int npoints) {
    int p = 32;
    while (p < npoints) p <<= 1;
    return p;
}

extern "C" int prb_kitti_draw_points(int b, int total, const int *offsets, const unsigned char *flags, int npoints, unsigned seed,
                                     int *cand_scratch, int *choice, int *status, void *stream) {
    PRB_REQUIRE(b > 0 && offsets && flags && choice && cand_scratch && npoints > 0, "kitti_draw_points: bad arguments");
    PRB_REQUIRE(npoints <= 16384, "kitti_draw_points: npoints %d > 16384 (one shared-memory sort per scene)", npoints);
    (void)total;
    const int npad = draw_pad(npoints);
    const size_t smem = (size_t)npad * 8;
    if (smem > 40 * 1024) PRB_CUDA(cudaFuncSetAttribute(kitti_draw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kitti_draw_kernel<<<b, 1024, smem, (cudaStream_t)stream>>>(b, offsets, flags, npoints, npad, seed, cand_scratch, choice, status);
    return check_launch("kitti_draw_kernel");
}

extern "C" int prb_kitti_gather_points(int b, int npoints, const int *offsets, const float *rect, const float *lidar, int stride,
                                       const int *choice, const double *aug, const int *status, int channels, float *pts_input,
                                       float *pts_rect, float *intensity, void *stream) {
    PRB_REQUIRE(b > 0 && npoints > 0 && offsets && rect && lidar && choice && (channels == 3 || channels == 4), "kitti_gather_points: bad arguments");
    kitti_gather_kernel<<<dim3(ceil_div(npoints, 256), b), 256, 0, (cudaStream_t)stream>>>(b, npoints, offsets, rect, lidar, stride, choice,
                                                                                         aug, status, channels, pts_input, pts_rect, intensity);
    return check_launch("kitti_gather_kernel");
}

extern "C" int prb_rpn_training_labels(int b, int n, int g, const float *pts_rect, const float *gt_boxes3d, const int *gt_count,
                                       float extra_width, int *cls_label, float *reg_label, void *stream) {
    PRB_REQUIRE(b > 0 && n > 0 && g >= 0 && pts_rect && cls_label && reg_label && (g == 0 || gt_boxes3d), "rpn_training_labels: bad arguments");
    PRB_REQUIRE(g <= kMaxGt, "rpn_training_labels: %d boxes per scene > %d", g, kMaxGt);
    rpn_labels_kernel<<<dim3(ceil_div(n, 256), b), 256, 0, (cudaStream_t)stream>>>(n, g, pts_rect, gt_boxes3d, gt_count, extra_width, cls_label,
                                                                                 reg_label);
    return check_launch("rpn_labels_kernel");
}

extern "C" int prb_kitti_image_boxes(int n, const float *boxes3d, const float *P2, float img_h, float img_w, float *img_boxes,
                                     float *alpha, int *valid, void *stream) {
    PRB_REQUIRE(n >= 0 && P2 && (n == 0 || (boxes3d && img_boxes && alpha && valid)), "kitti_image_boxes: bad arguments");
    if (n == 0) return 0;
    kitti_image_boxes_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(n, boxes3d, P2, 0, nullptr, img_h, img_w, img_boxes, alpha,
                                                                               valid);
    return check_launch("kitti_image_boxes_kernel");
}

extern "C" int prb_kitti_image_boxes_batch(int b, int m, const float *boxes3d, const float *P2, const float *img_hw, float *img_boxes,
                                           float *alpha, int *valid, void *stream) {
    PRB_REQUIRE(b >= 0 && m >= 0 && P2 && img_hw && (b * m == 0 || (boxes3d && img_boxes && alpha && valid)), "kitti_image_boxes_batch: bad arguments");
    if (b * m == 0) return 0;
    kitti_image_boxes_kernel<<<ceil_div(b * m, 128), 128, 0, (cudaStream_t)stream>>>(b * m, boxes3d, P2, m, img_hw, 0.f, 0.f, img_boxes, alpha,
                                                                                   valid);
    return check_launch("kitti_image_boxes_kernel");
}

// host: the text of one KITTI result file (eval_rcnn.py:85-94).  All pointers are HOST arrays.  Returns the number of
// bytes the text needs (excluding the terminator); nothing is written past `cap`.
extern "C" size_t prb_kitti_format_detections(const char *cls_name, int n, const float *boxes3d, const float *img_boxes,
                                              const float *alpha, const float *scores, const int *valid, char *buf, size_t cap) {
    size_t used = 0;
    for (int k = 0; k < n; ++k) {
        if (valid && !valid[k]) continue;
        const float *q = boxes3d + (size_t)k * 7, *ib = img_boxes + (size_t)k * 4;
        char line[512];
        const int len = snprintf(line, sizeof line, "%s -1 -1 %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f\n", cls_name,
                                 (double)alpha[k], (double)ib[0], (double)ib[1], (double)ib[2], (double)ib[3], (double)q[3], (double)q[4],
                                 (double)q[5], (double)q[0], (double)q[1], (double)q[2], (double)q[6], (double)scores[k]);
        if (len < 0) continue;
        if (buf && used + (size_t)len < cap) memcpy(buf + used, line, (size_t)len);
        used += (size_t)len;
    }
    if (buf && cap) buf[used < cap ? used : cap - 1] = 0;
    return used;
}
