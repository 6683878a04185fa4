// iou3d_dev.cuh -- device functions of the rotated / axis-aligned BEV IoU, shared by iou3d.cu (matrices, bitmask
// NMS) and proposal.cu (top-k greedy NMS inside the RPN proposal kernel).
//
// The overlap arithmetic IS the spec (keep masks are compared bit-exactly with lib/utils/iou3d/src/iou3d_kernel.cu:
// 34-221): corners rotated about the box centre, 4x4 edge intersections (bbox reject, straddle test, line solve with
// an EPS fallback), corners of one box inside the other (MARGIN 1e-5), centroid, bubble sort by atan2f, fan area / 2.0.
//
// Measured behaviour (tests/test_cpu_iou_geometry.py, tests/test_gpu_iou_geometry.py): the fixed MARGIN is below a few
// fp32 ulps at KITTI far range (one ulp is 7.6e-6 at 64 m), so a box's own corners, rotated there and back, can fall
// outside it: IoU(a, a) < 1, down to 0, for some boxes at z 60-80 m, as in the reference.  Near-parallel and
// near-duplicate pairs are ill-conditioned the same way, and their polygon can reach 16 vertices (the scratch size).
// Every consumer inherits this: NMS (matrix, bitmask, proposal), the fused 3D IoU, RoI sampling, recall statistics,
// GT-paste collisions and the KITTI overlaps.
#pragma once
#include "common.cuh"

namespace prb {

struct P2 {
    float x, y;
};
__device__ __forceinline__ P2 mk(float x, float y) { P2 p; p.x = x; p.y = y; return p; }

__device__ __forceinline__ float cross2(const P2 &a, const P2 &b) { return a.x * b.y - a.y * b.x; }
__device__ __forceinline__ float cross3(const P2 &p1, const P2 &p2, const P2 &p0) {
    return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}
__device__ __forceinline__ int rect_cross(const P2 &p1, const P2 &p2, const P2 &q1, const P2 &q2) {
    return min(p1.x, p2.x) <= max(q1.x, q2.x) && min(q1.x, q2.x) <= max(p1.x, p2.x) &&
           min(p1.y, p2.y) <= max(q1.y, q2.y) && min(q1.y, q2.y) <= max(p1.y, p2.y);
}
// The rotation of in_box2d and rot_center with the contraction the reference's SASS shows (nvcc 12.9 -O2, iou3d_kernel.cu):
// x' = fma(dx, cos, dy * sin) + c.x and y' = fma(dy, cos, -(dx * sin)) + c.y.  Left to the compiler, the inlined copies
// here fused the other product of y' in in_box2d_pre, which flips the inside test of near-boundary corners.
__device__ __forceinline__ P2 rot_about(float dx, float dy, float cx, float cy, float angle_cos, float angle_sin) {
    return mk(__fadd_rn(__fmaf_rn(dx, angle_cos, __fmul_rn(dy, angle_sin)), cx),
              __fadd_rn(__fmaf_rn(dy, angle_cos, -__fmul_rn(dx, angle_sin)), cy));
}
__device__ __forceinline__ int in_box2d(const float *box, const P2 &p) {
    const float MARGIN = 1e-5;
    float center_x = (box[0] + box[2]) / 2;
    float center_y = (box[1] + box[3]) / 2;
    float angle_cos = cos(-box[4]), angle_sin = sin(-box[4]);
    const P2 r = rot_about(__fsub_rn(p.x, center_x), __fsub_rn(p.y, center_y), center_x, center_y, angle_cos, angle_sin);
    return (r.x > box[0] - MARGIN && r.x < box[2] + MARGIN && r.y > box[1] - MARGIN && r.y < box[3] + MARGIN);
}
__device__ __forceinline__ int seg_intersection(const P2 &p1, const P2 &p0, const P2 &q1, const P2 &q0, P2 &ans) {
    const float EPS = 1e-8;
    if (rect_cross(p0, p1, q0, q1) == 0) return 0;
    float s1 = cross3(q0, p1, p0);
    float s2 = cross3(p1, q1, p0);
    float s3 = cross3(p0, q1, q0);
    float s4 = cross3(q1, p1, q0);
    if (!(s1 * s2 > 0 && s3 * s4 > 0)) return 0;
    float s5 = cross3(q1, p1, p0);
    if (fabs(s5 - s1) > EPS) {
        ans.x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        ans.y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        float D = a0 * b1 - a1 * b0;
        ans.x = (b0 * c1 - b1 * c0) / D;
        ans.y = (a1 * c0 - a0 * c1) / D;
    }
    return 1;
}
__device__ __forceinline__ void rot_center(const P2 &c, const float angle_cos, const float angle_sin, P2 &p) {
    p = rot_about(__fsub_rn(p.x, c.x), __fsub_rn(p.y, c.y), c.x, c.y, angle_cos, angle_sin);
}
__device__ __forceinline__ int angle_gt(const P2 &a, const P2 &b, const P2 &c) {
    return atan2(a.y - c.y, a.x - c.x) > atan2(b.y - c.y, b.x - c.x);
}

// rotated-rectangle intersection area of two [x1,y1,x2,y2,ry] boxes
__device__ inline float box_overlap(const float *box_a, const float *box_b) {
    float a_x1 = box_a[0], a_y1 = box_a[1], a_x2 = box_a[2], a_y2 = box_a[3], a_angle = box_a[4];
    float b_x1 = box_b[0], b_y1 = box_b[1], b_x2 = box_b[2], b_y2 = box_b[3], b_angle = box_b[4];
    P2 center_a = mk((a_x1 + a_x2) / 2, (a_y1 + a_y2) / 2);
    P2 center_b = mk((b_x1 + b_x2) / 2, (b_y1 + b_y2) / 2);
    P2 ca[5], cb[5];
    ca[0] = mk(a_x1, a_y1); ca[1] = mk(a_x2, a_y1); ca[2] = mk(a_x2, a_y2); ca[3] = mk(a_x1, a_y2);
    cb[0] = mk(b_x1, b_y1); cb[1] = mk(b_x2, b_y1); cb[2] = mk(b_x2, b_y2); cb[3] = mk(b_x1, b_y2);
    float a_angle_cos = cos(a_angle), a_angle_sin = sin(a_angle);
    float b_angle_cos = cos(b_angle), b_angle_sin = sin(b_angle);
    for (int k = 0; k < 4; k++) {
        rot_center(center_a, a_angle_cos, a_angle_sin, ca[k]);
        rot_center(center_b, b_angle_cos, b_angle_sin, cb[k]);
    }
    ca[4] = ca[0];
    cb[4] = cb[0];

    P2 cp[16];
    P2 poly_center = mk(0, 0);
    int cnt = 0;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            if (seg_intersection(ca[i + 1], ca[i], cb[j + 1], cb[j], cp[cnt])) {
                poly_center = mk(poly_center.x + cp[cnt].x, poly_center.y + cp[cnt].y);
                cnt++;
            }
    for (int k = 0; k < 4; k++) {
        if (in_box2d(box_a, cb[k])) {
            poly_center = mk(poly_center.x + cb[k].x, poly_center.y + cb[k].y);
            cp[cnt] = cb[k];
            cnt++;
        }
        if (in_box2d(box_b, ca[k])) {
            poly_center = mk(poly_center.x + ca[k].x, poly_center.y + ca[k].y);
            cp[cnt] = ca[k];
            cnt++;
        }
    }
    poly_center.x /= cnt;
    poly_center.y /= cnt;

    P2 t;
    for (int j = 0; j < cnt - 1; j++)
        for (int i = 0; i < cnt - j - 1; i++)
            if (angle_gt(cp[i], cp[i + 1], poly_center)) {
                t = cp[i];
                cp[i] = cp[i + 1];
                cp[i + 1] = t;
            }

    float area = 0;
    for (int k = 0; k < cnt - 1; k++)
        area += cross2(mk(cp[k].x - cp[0].x, cp[k].y - cp[0].y), mk(cp[k + 1].x - cp[0].x, cp[k + 1].y - cp[0].y));
    return fabs(area) / 2.0;
}

__device__ __forceinline__ float iou_bev(const float *box_a, const float *box_b) {
    const float EPS = 1e-8;
    float sa = (box_a[2] - box_a[0]) * (box_a[3] - box_a[1]);
    float sb = (box_b[2] - box_b[0]) * (box_b[3] - box_b[1]);
    float s_overlap = box_overlap(box_a, box_b);
    return s_overlap / fmaxf(sa + sb - s_overlap, EPS);
}

__device__ __forceinline__ float iou_normal(const float *a, const float *b) {
    const float EPS = 1e-8;
    float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    float width = fmaxf(right - left, 0.f), height = fmaxf(bottom - top, 0.f);
    float interS = width * height;
    float Sa = (a[2] - a[0]) * (a[3] - a[1]);
    float Sb = (b[2] - b[0]) * (b[3] - b[1]);
    return interS / fmaxf(Sa + Sb - interS, EPS);
}

// ---------------------------------------------------------------------------------------------- per-box precompute
// box_overlap above recomputes, for EVERY PAIR, the four rotated corners of both boxes (2 sincos) and calls in_box2d eight
// times (8 x cos(-ry), sin(-ry)), and its bubble sort calls atan2f twice per comparison: ~20 sincosf + up to ~200 atan2f per
// pair, with the intersection polygon `cp[16]` in local memory.  BoxPre holds what depends on ONE box only -- centre,
// cos / sin of its heading, rotated corners -- computed once per box per tile (the same expressions, so the same bits:
// cosf is even and sinf odd on the device, `sin(-a)` is replaced by `-sin(a)`), the polygon lives in a caller-provided
// (shared-memory) scratch column, and the polar angles are computed once per polygon vertex.  The comparisons, the
// centroid and the fan area see the same floats in the same order as box_overlap, hence bit-identical results
// (tests/test_gpu_ops.py compares masks / matrices with the reference kernel by torch.equal).
struct BoxPre {
    float x1, y1, x2, y2;      // axis-aligned extent before rotation
    float cx, cy, c, s;        // centre, cos(ry), sin(ry)
    P2 k[4];                   // rotated corners
};

__device__ __forceinline__ void box_pre(const float *box, BoxPre &b) {
    b.x1 = box[0]; b.y1 = box[1]; b.x2 = box[2]; b.y2 = box[3];
    const float ang = box[4];
    b.cx = (b.x1 + b.x2) / 2;
    b.cy = (b.y1 + b.y2) / 2;
    b.c = cos(ang);
    b.s = sin(ang);
    const P2 ctr = mk(b.cx, b.cy);
    b.k[0] = mk(b.x1, b.y1); b.k[1] = mk(b.x2, b.y1); b.k[2] = mk(b.x2, b.y2); b.k[3] = mk(b.x1, b.y2);
#pragma unroll
    for (int q = 0; q < 4; ++q) rot_center(ctr, b.c, b.s, b.k[q]);
}

// in_box2d with the box's precomputed centre and cos(-ry) = c, sin(-ry) = -s
__device__ __forceinline__ int in_box2d_pre(const BoxPre &b, const P2 &p) {
    const float MARGIN = 1e-5;
    const P2 r = rot_about(__fsub_rn(p.x, b.cx), __fsub_rn(p.y, b.cy), b.cx, b.cy, b.c, -b.s);
    return (r.x > b.x1 - MARGIN && r.x < b.x2 + MARGIN && r.y > b.y1 - MARGIN && r.y < b.y2 + MARGIN);
}

// rotated-rectangle intersection area from two precomputed boxes.  px / py / pa: scratch for up to 16 polygon vertices
// (x, y, polar angle), element i at [i * stride] (e.g. a shared-memory column per thread: no local memory)
__device__ inline float box_overlap_pre(const BoxPre &A, const BoxPre &B, float *px, float *py, float *pa, int stride) {
    float sum_x = 0.f, sum_y = 0.f;
    int cnt = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            P2 ans;
            if (seg_intersection(A.k[(i + 1) & 3], A.k[i], B.k[(j + 1) & 3], B.k[j], ans)) {
                sum_x = sum_x + ans.x; sum_y = sum_y + ans.y;
                px[cnt * stride] = ans.x; py[cnt * stride] = ans.y;
                cnt++;
            }
        }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        if (in_box2d_pre(A, B.k[q])) {
            sum_x = sum_x + B.k[q].x; sum_y = sum_y + B.k[q].y;
            px[cnt * stride] = B.k[q].x; py[cnt * stride] = B.k[q].y;
            cnt++;
        }
        if (in_box2d_pre(B, A.k[q])) {
            sum_x = sum_x + A.k[q].x; sum_y = sum_y + A.k[q].y;
            px[cnt * stride] = A.k[q].x; py[cnt * stride] = A.k[q].y;
            cnt++;
        }
    }
    if (cnt < 3) {
        // fewer than three vertices: the fan below has no triangle (cnt = 0 divides by zero in the reference and then
        // loops over nothing: area 0 as well)
        return 0.f;
    }
    const float ctr_x = sum_x / cnt, ctr_y = sum_y / cnt;
    for (int i = 0; i < cnt; ++i) pa[i * stride] = atan2(py[i * stride] - ctr_y, px[i * stride] - ctr_x);
    // the reference's bubble sort (swap when strictly greater): same comparisons on the same angles
    for (int j = 0; j < cnt - 1; j++)
        for (int i = 0; i < cnt - j - 1; i++) {
            const float a0 = pa[i * stride], a1 = pa[(i + 1) * stride];
            if (a0 > a1) {
                pa[i * stride] = a1; pa[(i + 1) * stride] = a0;
                float t = px[i * stride]; px[i * stride] = px[(i + 1) * stride]; px[(i + 1) * stride] = t;
                t = py[i * stride]; py[i * stride] = py[(i + 1) * stride]; py[(i + 1) * stride] = t;
            }
        }
    float area = 0;
    const float x0 = px[0], y0 = py[0];
    for (int q = 0; q < cnt - 1; q++)
        area += cross2(mk(px[q * stride] - x0, py[q * stride] - y0), mk(px[(q + 1) * stride] - x0, py[(q + 1) * stride] - y0));
    return fabs(area) / 2.0;
}

__device__ __forceinline__ float iou_bev_pre(const BoxPre &A, const BoxPre &B, float *px, float *py, float *pa, int stride) {
    const float EPS = 1e-8;
    float sa = (A.x2 - A.x1) * (A.y2 - A.y1);
    float sb = (B.x2 - B.x1) * (B.y2 - B.y1);
    float s_overlap = box_overlap_pre(A, B, px, py, pa, stride);
    return s_overlap / fmaxf(sa + sb - s_overlap, EPS);
}

// ---------------------------------------------------------------------------------------------- fused 3D IoU of one pair
// iou3d_utils.boxes_iou3d_gpu's op sequence for [x,y,z,h,w,l,ry] boxes, every torch op one fp32 rounding (iou3d.cu's
// iou3d_kernel, rcnn_sample.cu's jitter loop)
// torch.max / torch.min / torch.clamp propagate a NaN operand, fmaxf / fminf drop it: a NaN height or size must give a
// NaN IoU, as boxes_iou3d_gpu does, not ov3d / 1e-7
__device__ __forceinline__ float nan_max(float x, float y) { return x != x ? x : (y != y ? y : fmaxf(x, y)); }
__device__ __forceinline__ float nan_min(float x, float y) { return x != x ? x : (y != y ? y : fminf(x, y)); }
__device__ __forceinline__ void box7_to_bev(const float *b, float *bev) {
    const float half_l = __fmul_rn(b[5], 0.5f), half_w = __fmul_rn(b[4], 0.5f);
    bev[0] = __fsub_rn(b[0], half_l); bev[1] = __fsub_rn(b[2], half_w);
    bev[2] = __fadd_rn(b[0], half_l); bev[3] = __fadd_rn(b[2], half_w);
    bev[4] = b[6];
}
__device__ __forceinline__ float iou3d_pair(const float *a, const float *b, float *px, float *py, float *pa, int stride) {
    float abev[5], bbev[5];
    box7_to_bev(a, abev);
    box7_to_bev(b, bbev);
    BoxPre A, Bp;
    box_pre(abev, A);
    box_pre(bbev, Bp);
    const float ov_bev = box_overlap_pre(A, Bp, px, py, pa, stride);
    const float a_min = __fsub_rn(a[1], a[3]), b_min = __fsub_rn(b[1], b[3]);       // y - h .. y (y points down)
    const float ov_h = nan_max(__fsub_rn(nan_min(a[1], b[1]), nan_max(a_min, b_min)), 0.f);
    const float ov3d = __fmul_rn(ov_bev, ov_h);
    const float va = __fmul_rn(__fmul_rn(a[3], a[4]), a[5]), vb = __fmul_rn(__fmul_rn(b[3], b[4]), b[5]);
    return __fdiv_rn(ov3d, nan_max(__fsub_rn(__fadd_rn(va, vb), ov3d), 1e-7f));
}

}  // namespace prb
