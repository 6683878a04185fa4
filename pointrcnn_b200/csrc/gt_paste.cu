// gt_paste.cu -- GT-paste augmentation of the batched RPN input (lib/datasets/kitti_rcnn_dataset.py:273-282, 408-511,
// apply_gt_aug_to_one_scene), the two device stages between kitti_prepare_points and kitti_draw_points.
//
// Every random draw of the reference's paste loop comes before any collision test, and its candidate counter counts
// a candidate before that test: the candidate list (which database entries reach the test, and their moved boxes)
// depends on the database, the road plane and the random stream only.  The host draws it; the device does the two
// data-dependent parts:
//   select  one CTA per scene walks its candidates in order; each candidate's enlarged box is tested against every
//           current box in parallel (the scene's collision boxes, enlarged, plus the candidates accepted so far), an
//           accepted one joins the CTA's shared list.  Writes the per-candidate placement, per-scene counts and the
//           compacted label boxes [caller's GT rows | accepted candidates' rows].
//   paste   builds the post-paste ragged cloud in the layout the draw and gather stages read: each scene's raw
//           segment with the valid bit cleared on points inside an accepted box (h + 2), then the accepted entries'
//           points moved onto the road plane, in acceptance order.
// Buffers are sized by a bound the host knows (raw points + the points of every candidate): nothing is read back.
#include "common.cuh"
#include "iou3d_dev.cuh"

namespace prb {

constexpr int kPasteMaxCand = 128;     // candidates per scene
constexpr int kPasteMaxRows = 128;     // caller's GT + candidate rows: prb_rpn_training_labels' box limit
constexpr int kSelectThreads = 128;

// a box of the collision test: w and l enlarged by 0.5 (apply_gt_aug_to_one_scene), BEV rectangle
// [x-l/2, z-w/2, x+l/2, z+w/2, ry] for box_overlap (the rotation convention of boxes3d_to_corners3d), and the height
// range [-y, -(y-h)] get_iou3d reads from the corners (y points down)
struct CollBox {
    BoxPre bev;
    float lo, hi, vol;
};

__device__ __forceinline__ void coll_box(const float *__restrict__ q, CollBox &c) {
    const float y = q[1], h = q[3];
    const float enlarged[7] = {q[0], y, q[2], h, q[4] + 0.5f, q[5] + 0.5f, q[6]};
    float bev[5];
    box7_to_bev(enlarged, bev);
    box_pre(bev, c.bev);
    c.lo = -y;
    c.hi = -(y - h);
    c.vol = (c.bev.x2 - c.bev.x1) * (c.bev.y2 - c.bev.y1) * (c.hi - c.lo);
}

// 3D IoU >= 1e-8 (kitti_rcnn_dataset.py:479-480); px / py / pa: the thread's polygon scratch column
__device__ __forceinline__ bool collides(const CollBox &a, const CollBox &b, float *px, float *py, float *pa) {
    const float oh = fminf(a.hi, b.hi) - fmaxf(a.lo, b.lo);
    if (!(oh > 0.f)) return false;
    const float ov = box_overlap(a.bev, b.bev, px, py, pa, kSelectThreads) * oh;
    return ov / (a.vol + b.vol - ov) >= 1e-8f;
}

// cand_boxes (b,k,7): moved (not enlarged) boxes; cand_first (b*k+1): exclusive prefix of the candidates' point counts
__global__ void __launch_bounds__(kSelectThreads) gt_paste_select_kernel(
    int k, int m, int g, const float *__restrict__ cand_boxes, const int *__restrict__ cand_count, const int *__restrict__ cand_first,
    const float *__restrict__ coll_boxes, const int *__restrict__ coll_count, const float *__restrict__ gt_rows,
    const int *__restrict__ gt_count, const float *__restrict__ cand_rows, int *__restrict__ place, int *__restrict__ stats,
    float *__restrict__ gt_out, int *__restrict__ gt_count_out, int *__restrict__ counts) {
    // shared memory: polygon scratch (3 x POLY_SLOTS x kSelectThreads), then m collision boxes + up to k accepted candidates
    extern __shared__ float s_dyn[];
    CollBox *s_cur = reinterpret_cast<CollBox *>(s_dyn + 3 * POLY_SLOTS * kSelectThreads);
    __shared__ int s_acc[kPasteMaxCand];                      // candidate index of the r-th accepted one
    const int scene = blockIdx.x, tid = threadIdx.x;
    float *px = s_dyn + tid, *py = px + POLY_SLOTS * kSelectThreads, *pa = py + POLY_SLOTS * kSelectThreads;
    const int nm = min(coll_count[scene], m), nc = min(cand_count[scene], k);
    for (int q = tid; q < nm; q += kSelectThreads) coll_box(coll_boxes + ((size_t)scene * m + q) * 7, s_cur[q]);
    for (int j = nc + tid; j < k; j += kSelectThreads) place[(size_t)scene * k + j] = -1;
    __syncthreads();
    int ncur = nm, nacc = 0, npts = 0;          // CTA-uniform
    for (int j = 0; j < nc; ++j) {
        const int c = scene * k + j;
        CollBox cb;
        coll_box(cand_boxes + (size_t)c * 7, cb);
        bool hit = false;
        for (int q = tid; q < ncur && !hit; q += kSelectThreads) hit = collides(cb, s_cur[q], px, py, pa);
        if (__syncthreads_or(hit)) {
            if (tid == 0) place[c] = -1;
            continue;
        }
        if (tid == 0) {
            s_cur[ncur] = cb;
            s_acc[nacc] = j;
            place[c] = npts;
        }
        ++ncur;
        ++nacc;
        npts += cand_first[c + 1] - cand_first[c];
        __syncthreads();                        // the new box is read by the next candidate's test
    }
    if (tid == 0) {
        stats[scene * 2] = nacc;
        stats[scene * 2 + 1] = npts;
        if (counts) { counts[scene * 2] = 0; counts[scene * 2 + 1] = 0; }
    }
    if (gt_out) {
        const int ng = gt_count ? min(gt_count[scene], g) : g;
        const int width = g + k;
        float *o = gt_out + (size_t)scene * width * 7;
        for (int e = tid; e < width * 7; e += kSelectThreads) {
            const int r = e / 7, col = e - r * 7;
            float v = 0.f;
            if (r < ng) v = gt_rows[((size_t)scene * g + r) * 7 + col];
            else if (r < ng + nacc) v = cand_rows[((size_t)scene * k + s_acc[r - ng]) * 7 + col];
            o[e] = v;
        }
        if (tid == 0) gt_count_out[scene] = ng + nacc;
    }
}

// pts_in_boxes3d_cpu's predicate (roipool3d.cpp:82-95): fp32 differences and rotation, cos / sin and the half sizes in
// double, as the host compiler evaluates it (no contraction)
struct PasteBox {
    float cx, cy, cz, cosa, sina;
    double half_h, half_l, half_w;
};

__device__ __forceinline__ PasteBox paste_box(const float *__restrict__ bx) {
    PasteBox c;
    const float h = bx[3] + 2.0f;               // enlarged_box3d[3] += 2: remove the points above and below the object
    c.cx = bx[0];
    c.cz = bx[2];
    c.half_h = (double)h / 2.0;
    c.half_l = (double)bx[5] / 2.0;
    c.half_w = (double)bx[4] / 2.0;
    c.cy = (float)((double)bx[1] - c.half_h);
    c.cosa = (float)cos((double)bx[6]);
    c.sina = (float)sin((double)bx[6]);
    return c;
}

__device__ __forceinline__ bool paste_in_box(const PasteBox &c, float x, float y, float z) {
    const float dx = __fsub_rn(x, c.cx), dz = __fsub_rn(z, c.cz);
    if (fabsf(dx) > 10.0f || (double)fabsf(__fsub_rn(y, c.cy)) > c.half_h || fabsf(dz) > 10.0f) return false;
    const float x_rot = __fadd_rn(__fmul_rn(dx, c.cosa), __fmul_rn(dz, -c.sina));
    const float z_rot = __fadd_rn(__fmul_rn(dx, c.sina), __fmul_rn(dz, c.cosa));
    return ((double)x_rot >= -c.half_l) & ((double)x_rot <= c.half_l) & ((double)z_rot >= -c.half_w) &
           ((double)z_rot <= c.half_w);
}

// largest i in [0, n) with a[i] <= v (a ascending, a[0] <= v)
__device__ __forceinline__ int last_le(const int *__restrict__ a, int n, int v) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] <= v) lo = mid; else hi = mid;
    }
    return lo;
}

// threads [0, total) copy raw point i; threads [total, total + cand_total) copy candidate point t = i - total if its
// candidate was accepted.  points_out (.,4): rect x, y, z, intensity (the gather stage's lidar operand, stride 4).
__global__ void __launch_bounds__(256) gt_paste_points_kernel(
    int b, int total, int k, int cand_total, const int *__restrict__ offsets, const float *__restrict__ rect,
    const float *__restrict__ lidar, int stride, const unsigned char *__restrict__ flags, const float *__restrict__ cand_boxes,
    const int *__restrict__ cand_first, const int *__restrict__ cand_src, const double *__restrict__ moves,
    const int *__restrict__ place, const int *__restrict__ stats, const float *__restrict__ db_points, int *__restrict__ offsets_out,
    float *__restrict__ rect_out, float *__restrict__ points_out, unsigned char *__restrict__ flags_out, int *__restrict__ counts) {
    extern __shared__ int s_noff[];             // b + 1 post-paste scene offsets
    __shared__ PasteBox s_box[kPasteMaxCand];   // accepted boxes of the block's first scene
    __shared__ int s_ok[kPasteMaxCand];
    const int tid = threadIdx.x, i0 = blockIdx.x * 256, i = i0 + tid;
    if (tid == 0) {
        int acc = 0;
        for (int s = 0; s < b; ++s) {
            s_noff[s] = acc;
            acc += offsets[s + 1] - offsets[s] + stats[s * 2 + 1];
        }
        s_noff[b] = acc;
    }
    const int s0 = i0 < total ? last_le(offsets, b, i0) : -1;
    if (s0 >= 0 && tid < k) {
        const int c = s0 * k + tid;
        s_ok[tid] = place[c] >= 0;
        if (s_ok[tid]) s_box[tid] = paste_box(cand_boxes + (size_t)c * 7);
    }
    __syncthreads();
    if (blockIdx.x == 0)
        for (int s = tid; s <= b; s += 256) offsets_out[s] = s_noff[s];

    int s = -1;
    bool ok = false, near = false;
    if (i < total) {
        s = last_le(offsets, b, i);
        const unsigned char fl = flags[i];
        const float x = rect[(size_t)i * 3], y = rect[(size_t)i * 3 + 1], z = rect[(size_t)i * 3 + 2];
        ok = fl & 1;
        near = fl & 2;
        if (ok) {
            for (int j = 0; j < k && ok; ++j) {
                if (s == s0) {
                    if (s_ok[j] && paste_in_box(s_box[j], x, y, z)) ok = false;
                } else if (place[s * k + j] >= 0 && paste_in_box(paste_box(cand_boxes + ((size_t)s * k + j) * 7), x, y, z)) {
                    ok = false;
                }
            }
        }
        const size_t o = (size_t)s_noff[s] + (i - offsets[s]);
        rect_out[o * 3] = x; rect_out[o * 3 + 1] = y; rect_out[o * 3 + 2] = z;
        float4 p = make_float4(x, y, z, stride > 3 ? lidar[(size_t)i * stride + 3] : 0.f);
        reinterpret_cast<float4 *>(points_out)[o] = p;
        flags_out[o] = (unsigned char)((ok ? 1 : 0) | (near ? 2 : 0));
    } else if (i - total < cand_total) {
        const int t = i - total;
        const int c = last_le(cand_first, b * k, t);
        const int pl = place[c];
        if (pl >= 0) {
            s = c / k;
            const int r = t - cand_first[c];
            const float4 q = reinterpret_cast<const float4 *>(db_points)[cand_src[c] + r];
            const float y = (float)((double)q.y - moves[c]);    // numpy: float32 -= float64 scalar computes in float64
            const size_t o = (size_t)s_noff[s] + (offsets[s + 1] - offsets[s]) + pl + r;
            rect_out[o * 3] = q.x; rect_out[o * 3 + 1] = y; rect_out[o * 3 + 2] = q.z;
            reinterpret_cast<float4 *>(points_out)[o] = make_float4(q.x, y, q.z, q.w);
            ok = true;
            near = q.z < 40.0f;
            flags_out[o] = (unsigned char)(1 | (near ? 2 : 0));
        }
    }
    // per-scene valid / valid far counts: one atomic per warp and scene, as in kitti_prepare_kernel
    const unsigned grp = __match_any_sync(0xffffffffu, s);
    const unsigned okm = __ballot_sync(0xffffffffu, ok) & grp;
    const unsigned farm = __ballot_sync(0xffffffffu, ok && !near) & grp;
    if (s >= 0 && (tid & 31) == __ffs(grp) - 1) {
        if (okm) atomicAdd(&counts[s * 2], __popc(okm));
        if (farm) atomicAdd(&counts[s * 2 + 1], __popc(farm));
    }
}

}  // namespace prb

using namespace prb;

extern "C" int prb_gt_paste_select(int b, int k, int m, int g, const float *cand_boxes, const int *cand_count, const int *cand_first,
                                   const float *coll_boxes, const int *coll_count, const float *gt_rows, const int *gt_count,
                                   const float *cand_rows, int *place, int *stats, float *gt_out, int *gt_count_out, int *counts,
                                   void *stream) {
    PRB_REQUIRE(b > 0 && k >= 0 && m >= 0 && g >= 0 && cand_count && cand_first && coll_count && place && stats &&
                    (k == 0 || cand_boxes) && (m == 0 || coll_boxes),
                "gt_paste_select: bad arguments");
    PRB_REQUIRE(k <= kPasteMaxCand, "gt_paste_select: %d candidates per scene > %d", k, kPasteMaxCand);
    PRB_REQUIRE(m <= 1024, "gt_paste_select: %d collision boxes per scene > 1024", m);
    PRB_REQUIRE(!gt_out || (gt_count_out && (g == 0 || gt_rows) && (k == 0 || cand_rows)), "gt_paste_select: label rows need gt_rows, "
                "cand_rows and gt_count_out");
    PRB_REQUIRE(!gt_out || g + k <= kPasteMaxRows, "gt_paste_select: %d GT + %d candidate rows > %d", g, k, kPasteMaxRows);
    // polygon scratch (24 KB) and 76 bytes per box: m = 1024, k = 128 need 110 KB (above 40 KB: s_acc shares the default 48)
    const size_t smem = (size_t)3 * POLY_SLOTS * kSelectThreads * sizeof(float) + (size_t)(m + k) * sizeof(CollBox);
    if (smem > 40 * 1024) PRB_CUDA(cudaFuncSetAttribute(gt_paste_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gt_paste_select_kernel<<<b, kSelectThreads, smem, (cudaStream_t)stream>>>(k, m, g, cand_boxes, cand_count, cand_first, coll_boxes,
                                                                              coll_count, gt_rows, gt_count, cand_rows, place, stats, gt_out,
                                                                              gt_count_out, counts);
    return check_launch("gt_paste_select_kernel");
}

extern "C" int prb_gt_paste_points(int b, int total, int k, int cand_total, const int *offsets, const float *rect, const float *lidar,
                                   int stride, const unsigned char *flags, const float *cand_boxes, const int *cand_first,
                                   const int *cand_src, const double *moves, const int *place, const int *stats, const float *db_points,
                                   int *offsets_out, float *rect_out, float *points_out, unsigned char *flags_out, int *counts,
                                   void *stream) {
    PRB_REQUIRE(b > 0 && total >= 0 && k >= 0 && cand_total >= 0 && offsets && place && stats && cand_first && offsets_out && counts &&
                    (total == 0 || (rect && lidar && flags && stride >= 3)) && (cand_total == 0 || (cand_boxes && cand_src && moves && db_points)) &&
                    (total + cand_total == 0 || (rect_out && points_out && flags_out)),
                "gt_paste_points: bad arguments");
    PRB_REQUIRE(k <= kPasteMaxCand, "gt_paste_points: %d candidates per scene > %d", k, kPasteMaxCand);
    PRB_REQUIRE((reinterpret_cast<uintptr_t>(points_out) | reinterpret_cast<uintptr_t>(db_points)) % 16 == 0,
                "gt_paste_points: points_out and db_points must be 16-byte aligned");
    const int n = total + cand_total;
    const size_t smem = (size_t)(b + 1) * sizeof(int);
    if (smem > 40 * 1024) PRB_CUDA(cudaFuncSetAttribute(gt_paste_points_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gt_paste_points_kernel<<<ceil_div(n > 0 ? n : 1, 256), 256, smem, (cudaStream_t)stream>>>(
        b, total, k, cand_total, offsets, rect, lidar, stride, flags, cand_boxes, cand_first, cand_src, moves, place, stats, db_points,
        offsets_out, rect_out, points_out, flags_out, counts);
    return check_launch("gt_paste_points_kernel");
}
