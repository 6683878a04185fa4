/*
 * oracle/pointops_oracle.c -- CPU restatement of PointRCNN's point-cloud operator path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under pointrcnn_b200/ may import, link or call this
 * file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs use it, as the checker / the timed CPU baseline.
 *
 * Every function restates one reference CUDA kernel (paths relative to /root/reference):
 *   orc_fps                 pointnet2_lib/pointnet2/src/sampling_gpu.cu:86-209, cuda_utils.h:10-14
 *   orc_gather(+grad)       pointnet2_lib/pointnet2/src/sampling_gpu.cu:8-24, 46-63
 *   orc_ball_query          pointnet2_lib/pointnet2/src/ball_query_gpu.cu:9-45
 *   orc_group(+grad)        pointnet2_lib/pointnet2/src/group_points_gpu.cu:47-66, 8-25
 *   orc_three_nn            pointnet2_lib/pointnet2/src/interpolate_gpu.cu:9-52
 *   orc_three_interpolate   pointnet2_lib/pointnet2/src/interpolate_gpu.cu:77-97 (grad :120-142)
 *   orc_pt_in_box3d         lib/utils/roipool3d/src/roipool3d_kernel.cu:14-28
 *   orc_roipool3d           lib/utils/roipool3d/src/roipool3d_kernel.cu:97-194 (== roipool3d.cpp:127-195)
 *   orc_box_overlap         lib/utils/iou3d/src/iou3d_kernel.cu:34-212
 *   orc_box_overlap_pairs   the same for aligned pairs, with the polygon vertex count and planted mistakes
 *   orc_iou_bev/normal      lib/utils/iou3d/src/iou3d_kernel.cu:214-221, 295-303
 *   orc_nms_mask / orc_nms  lib/utils/iou3d/src/iou3d_kernel.cu:250-348 + iou3d.cpp:100-116
 *
 * Arithmetic contract: fp32 everywhere the kernels are fp32, with the FMA contraction the
 * reference's SASS shows for the three distance kernels (nvcc 12.9 -O2):
 *     d = fmaf(dz, dz, fmaf(dx, dx, dy * dy))
 * so FPS / ball-query / three_nn indices are bit-exact against the GPU.  This file must be
 * compiled with -ffp-contract=off so that gcc adds no contraction of its own.
 * Transcendentals (cosf/sinf/atan2f) come from the host libm here and from libdevice on
 * the GPU, so roipool3d flags and box overlaps agree with the GPU up to those ulps: tests
 * compare them bit-exactly against oracle/_ref (the reference kernels themselves) on the
 * GPU and with a stated tolerance / borderline filter against this file.
 *
 * Parity pin: the reference ships no golden vectors (SURVEY.md section 4).  This oracle is
 * pinned against outputs of the reference's own kernels (oracle/_ref, run on a GPU through
 * gpurun) committed under tests/golden/ by oracle/make_golden.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API __attribute__((visibility("default")))

/* squared distance with the reference's SASS contraction order */
static inline float dist2_ref(float ax, float ay, float az, float bx, float by, float bz) {
    float dx = ax - bx, dy = ay - by, dz = az - bz;
    float t = dy * dy;
    t = fmaf(dx, dx, t);
    return fmaf(dz, dz, t);
}

/* the squared distance above for n aligned pairs, so tests can certify fp32 boundary placements */
ORC_API void orc_dist2(int n, const float *a, const float *b, float *out) {
    for (int i = 0; i < n; ++i) out[i] = dist2_ref(a[i * 3], a[i * 3 + 1], a[i * 3 + 2], b[i * 3], b[i * 3 + 1], b[i * 3 + 2]);
}

/* cuda_utils.h:10-14 : largest power of two <= min(n, 1024), at least 1 */
ORC_API int orc_opt_n_threads(int work_size) {
    int pow_2 = (int)(log((double)work_size) / log(2.0));
    int t = 1 << pow_2;
    if (t > 1024) t = 1024;
    if (t < 1) t = 1;
    return t;
}

/* ---------------------------------------------------------------------------------------
 * FPS: literal simulation of the S-thread block (strided scan + shared-memory tree) so the
 * tie-break is the reference's by construction.  temp is read-modify-written like the kernel.
 * ------------------------------------------------------------------------------------- */
ORC_API void orc_fps(int b, int n, int m, const float *xyz, float *temp, int *idx) {
    if (m <= 0) return;
    const int S = orc_opt_n_threads(n);
#pragma omp parallel for schedule(dynamic, 1)
    for (int bi = 0; bi < b; ++bi) {
        const float *p = xyz + (size_t)bi * n * 3;
        float *tmp = temp + (size_t)bi * n;
        int *out = idx + (size_t)bi * m;
        float *dists = (float *)malloc(sizeof(float) * S);
        int *dists_i = (int *)malloc(sizeof(int) * S);
        int old = 0;
        out[0] = 0;
        for (int j = 1; j < m; ++j) {
            const float x1 = p[old * 3 + 0], y1 = p[old * 3 + 1], z1 = p[old * 3 + 2];
            for (int tid = 0; tid < S; ++tid) {
                int besti = 0;
                float best = -1.0f;
                for (int k = tid; k < n; k += S) {
                    /* (x2-x1)^2 + (y2-y1)^2 + (z2-z1)^2 in the kernel's contraction order */
                    float d = dist2_ref(p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2], x1, y1, z1);
                    float d2 = fminf(d, tmp[k]);
                    tmp[k] = d2;
                    besti = d2 > best ? k : besti;
                    best = d2 > best ? d2 : best;
                }
                dists[tid] = best;
                dists_i[tid] = besti;
            }
            for (int stride = S / 2; stride >= 1; stride >>= 1) {
                for (int tid = 0; tid < stride; ++tid) {
                    float v1 = dists[tid], v2 = dists[tid + stride];
                    int i1 = dists_i[tid], i2 = dists_i[tid + stride];
                    dists[tid] = fmaxf(v1, v2);
                    dists_i[tid] = v2 > v1 ? i2 : i1;
                }
            }
            old = dists_i[0];
            out[j] = old;
        }
        free(dists);
        free(dists_i);
    }
}

ORC_API void orc_gather(int b, int c, int n, int m, const float *points, const int *idx, float *out) {
#pragma omp parallel for collapse(2)
    for (int bi = 0; bi < b; ++bi)
        for (int ci = 0; ci < c; ++ci) {
            const float *src = points + ((size_t)bi * c + ci) * n;
            const int *ix = idx + (size_t)bi * m;
            float *dst = out + ((size_t)bi * c + ci) * m;
            for (int j = 0; j < m; ++j) dst[j] = src[ix[j]];
        }
}

ORC_API void orc_gather_grad(int b, int c, int n, int m, const float *grad_out, const int *idx,
                             float *grad_points) {
#pragma omp parallel for collapse(2)
    for (int bi = 0; bi < b; ++bi)
        for (int ci = 0; ci < c; ++ci) {
            const float *g = grad_out + ((size_t)bi * c + ci) * m;
            const int *ix = idx + (size_t)bi * m;
            float *dst = grad_points + ((size_t)bi * c + ci) * n;
            for (int j = 0; j < m; ++j) dst[ix[j]] += g[j];
        }
}

ORC_API void orc_ball_query(int b, int n, int m, float radius, int nsample, const float *new_xyz,
                            const float *xyz, int *idx) {
    const float radius2 = radius * radius;
#pragma omp parallel for collapse(2) schedule(static)
    for (int bi = 0; bi < b; ++bi)
        for (int j = 0; j < m; ++j) {
            const float *c = new_xyz + ((size_t)bi * m + j) * 3;
            const float *p = xyz + (size_t)bi * n * 3;
            int *o = idx + ((size_t)bi * m + j) * nsample;
            int cnt = 0;
            for (int k = 0; k < n; ++k) {
                float d2 = dist2_ref(c[0], c[1], c[2], p[k * 3], p[k * 3 + 1], p[k * 3 + 2]);
                if (d2 < radius2) {
                    if (cnt == 0)
                        for (int l = 0; l < nsample; ++l) o[l] = k;
                    o[cnt] = k;
                    ++cnt;
                    if (cnt >= nsample) break;
                }
            }
        }
}

ORC_API void orc_group(int b, int c, int n, int npoints, int nsample, const float *points,
                       const int *idx, float *out) {
#pragma omp parallel for collapse(2)
    for (int bi = 0; bi < b; ++bi)
        for (int ci = 0; ci < c; ++ci) {
            const float *src = points + ((size_t)bi * c + ci) * n;
            const int *ix = idx + (size_t)bi * npoints * nsample;
            float *dst = out + ((size_t)bi * c + ci) * npoints * nsample;
            for (size_t t = 0; t < (size_t)npoints * nsample; ++t) dst[t] = src[ix[t]];
        }
}

ORC_API void orc_group_grad(int b, int c, int n, int npoints, int nsample, const float *grad_out,
                            const int *idx, float *grad_points) {
#pragma omp parallel for collapse(2)
    for (int bi = 0; bi < b; ++bi)
        for (int ci = 0; ci < c; ++ci) {
            const float *g = grad_out + ((size_t)bi * c + ci) * npoints * nsample;
            const int *ix = idx + (size_t)bi * npoints * nsample;
            float *dst = grad_points + ((size_t)bi * c + ci) * n;
            for (size_t t = 0; t < (size_t)npoints * nsample; ++t) dst[ix[t]] += g[t];
        }
}

ORC_API void orc_three_nn(int b, int n, int m, const float *unknown, const float *known,
                          float *dist2, int *idx) {
#pragma omp parallel for collapse(2) schedule(static)
    for (int bi = 0; bi < b; ++bi)
        for (int j = 0; j < n; ++j) {
            const float *u = unknown + ((size_t)bi * n + j) * 3;
            const float *kn = known + (size_t)bi * m * 3;
            double best1 = 1e40, best2 = 1e40, best3 = 1e40;
            int besti1 = 0, besti2 = 0, besti3 = 0;
            for (int k = 0; k < m; ++k) {
                float d = dist2_ref(u[0], u[1], u[2], kn[k * 3], kn[k * 3 + 1], kn[k * 3 + 2]);
                if (d < best1) {
                    best3 = best2; besti3 = besti2;
                    best2 = best1; besti2 = besti1;
                    best1 = d; besti1 = k;
                } else if (d < best2) {
                    best3 = best2; besti3 = besti2;
                    best2 = d; besti2 = k;
                } else if (d < best3) {
                    best3 = d; besti3 = k;
                }
            }
            float *od = dist2 + ((size_t)bi * n + j) * 3;
            int *oi = idx + ((size_t)bi * n + j) * 3;
            od[0] = (float)best1; od[1] = (float)best2; od[2] = (float)best3;
            oi[0] = besti1; oi[1] = besti2; oi[2] = besti3;
        }
}

/* out = w0*p0 + w1*p1 + w2*p2 ; reference SASS (nvcc 12.9 -O2): FMUL(w1,p1) -> FFMA(w0,p0,.) -> FFMA(w2,p2,.) */
ORC_API void orc_three_interpolate(int b, int c, int m, int n, const float *points, const int *idx,
                                   const float *weight, float *out) {
#pragma omp parallel for collapse(2)
    for (int bi = 0; bi < b; ++bi)
        for (int ci = 0; ci < c; ++ci) {
            const float *src = points + ((size_t)bi * c + ci) * m;
            float *dst = out + ((size_t)bi * c + ci) * n;
            for (int j = 0; j < n; ++j) {
                const int *ix = idx + ((size_t)bi * n + j) * 3;
                const float *w = weight + ((size_t)bi * n + j) * 3;
                float t = w[1] * src[ix[1]];
                t = fmaf(w[0], src[ix[0]], t);
                dst[j] = fmaf(w[2], src[ix[2]], t);
            }
        }
}

ORC_API void orc_three_interpolate_grad(int b, int c, int n, int m, const float *grad_out,
                                        const int *idx, const float *weight, float *grad_points) {
#pragma omp parallel for collapse(2)
    for (int bi = 0; bi < b; ++bi)
        for (int ci = 0; ci < c; ++ci) {
            const float *g = grad_out + ((size_t)bi * c + ci) * n;
            float *dst = grad_points + ((size_t)bi * c + ci) * m;
            for (int j = 0; j < n; ++j) {
                const int *ix = idx + ((size_t)bi * n + j) * 3;
                const float *w = weight + ((size_t)bi * n + j) * 3;
                dst[ix[0]] += g[j] * w[0];
                dst[ix[1]] += g[j] * w[1];
                dst[ix[2]] += g[j] * w[2];
            }
        }
}

/* ---------------------------------------------------------------------------------------
 * roipool3d
 * ------------------------------------------------------------------------------------- */
ORC_API int orc_pt_in_box3d(float x, float y, float z, float cx, float bottom_y, float cz, float h,
                            float w, float l, float angle) {
    const float max_dis = 10.0f;
    float x_rot, z_rot, cosa, sina, cy;
    cy = (float)(bottom_y - h / 2.0); /* double arithmetic, stored to float */
    if ((fabsf(x - cx) > max_dis) || (fabsf(y - cy) > h / 2.0) || (fabsf(z - cz) > max_dis)) return 0;
    cosa = cosf(angle);
    sina = sinf(angle);
    /* reference SASS (assign_pts_to_box3d, nvcc 12.9 -O2):
     *   x_rot = FFMA(dx, cosa, -(FMUL(dz, sina)));  z_rot = FFMA(dz, cosa, FMUL(dx, sina)) */
    float dx = x - cx, dz = z - cz;
    x_rot = fmaf(dx, cosa, -(dz * sina));
    z_rot = fmaf(dz, cosa, dx * sina);
    return (x_rot >= -l / 2.0) & (x_rot <= l / 2.0) & (z_rot >= -w / 2.0) & (z_rot <= w / 2.0);
}

ORC_API void orc_pts_in_boxes3d(int n, int m, const float *pts, const float *boxes, int64_t *flag) {
#pragma omp parallel for
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j)
            flag[(size_t)i * n + j] =
                orc_pt_in_box3d(pts[j * 3], pts[j * 3 + 1], pts[j * 3 + 2], boxes[i * 7], boxes[i * 7 + 1],
                                boxes[i * 7 + 2], boxes[i * 7 + 3], boxes[i * 7 + 4], boxes[i * 7 + 5],
                                boxes[i * 7 + 6]);
}

/* pooled (B,M,S,3+C) and empty (B,M) must be zero-filled by the caller (roipool3d_utils.py:21-23) */
ORC_API void orc_roipool3d(int B, int N, int M, int C, int S, const float *xyz, const float *boxes3d,
                           const float *pts_feature, float *pooled, int *empty_flag) {
    const int W = 3 + C;
#pragma omp parallel for collapse(2) schedule(dynamic, 4)
    for (int bi = 0; bi < B; ++bi)
        for (int mi = 0; mi < M; ++mi) {
            const float *bx = boxes3d + ((size_t)bi * M + mi) * 7;
            const float *p = xyz + (size_t)bi * N * 3;
            const float *f = pts_feature + (size_t)bi * N * C;
            float *dst = pooled + ((size_t)bi * M + mi) * S * W;
            int cnt = 0;
            for (int k = 0; k < N && cnt < S; ++k) {
                if (orc_pt_in_box3d(p[k * 3], p[k * 3 + 1], p[k * 3 + 2], bx[0], bx[1], bx[2], bx[3], bx[4],
                                    bx[5], bx[6])) {
                    float *row = dst + (size_t)cnt * W;
                    row[0] = p[k * 3]; row[1] = p[k * 3 + 1]; row[2] = p[k * 3 + 2];
                    memcpy(row + 3, f + (size_t)k * C, sizeof(float) * C);
                    ++cnt;
                }
            }
            if (cnt == 0) {
                empty_flag[(size_t)bi * M + mi] = 1;
            } else if (cnt < S) {
                for (int k = cnt; k < S; ++k)
                    memcpy(dst + (size_t)k * W, dst + (size_t)(k % cnt) * W, sizeof(float) * W);
            }
        }
}

/* ---------------------------------------------------------------------------------------
 * iou3d : rotated BEV overlap, following iou3d_kernel.cu:34-212 statement by statement.
 * ------------------------------------------------------------------------------------- */
typedef struct { float x, y; } pt2;

static inline float cross2(pt2 a, pt2 b) { return a.x * b.y - a.y * b.x; }
static inline float cross3(pt2 p1, pt2 p2, pt2 p0) {
    return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}
static inline int rect_cross(pt2 p1, pt2 p2, pt2 q1, pt2 q2) {
    return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
           fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}
static inline int in_box2d(const float *box, pt2 p) {
    const float MARGIN = 1e-5f;
    float center_x = (box[0] + box[2]) / 2, center_y = (box[1] + box[3]) / 2;
    float angle_cos = cosf(-box[4]), angle_sin = sinf(-box[4]);
    float rot_x = (p.x - center_x) * angle_cos + (p.y - center_y) * angle_sin + center_x;
    float rot_y = -(p.x - center_x) * angle_sin + (p.y - center_y) * angle_cos + center_y;
    return (rot_x > box[0] - MARGIN && rot_x < box[2] + MARGIN && rot_y > box[1] - MARGIN &&
            rot_y < box[3] + MARGIN);
}
static inline int seg_intersection(pt2 p1, pt2 p0, pt2 q1, pt2 q0, pt2 *ans) {
    const float EPS = 1e-8f;
    if (rect_cross(p0, p1, q0, q1) == 0) return 0;
    float s1 = cross3(q0, p1, p0);
    float s2 = cross3(p1, q1, p0);
    float s3 = cross3(p0, q1, q0);
    float s4 = cross3(q1, p1, q0);
    if (!(s1 * s2 > 0 && s3 * s4 > 0)) return 0;
    float s5 = cross3(q1, p1, p0);
    if (fabsf(s5 - s1) > EPS) {
        ans->x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        ans->y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        float D = a0 * b1 - a1 * b0;
        ans->x = (b0 * c1 - b1 * c0) / D;
        ans->y = (a1 * c0 - a0 * c1) / D;
    }
    return 1;
}
static inline void rot_center(pt2 c, float ca, float sa, pt2 *p) {
    float nx = (p->x - c.x) * ca + (p->y - c.y) * sa + c.x;
    float ny = -(p->x - c.x) * sa + (p->y - c.y) * ca + c.y;
    p->x = nx; p->y = ny;
}

/* The overlap with a planted mistake, for tests that show their error bound catches one (tests/iou_reference.py):
 * mutant 0 = the reference; 1 = the last corner of box b is never tested; 2 = sin of the heading negated;
 * 3 = the sort comparison reversed; 4 = the bubble sort stops one pass early.  *cnt: polygon vertex count.  The
 * reference and the device kernels hold 16 vertices (cp[16], POLY_SLOTS); crossings and corners are counted separately,
 * so rounding alone does not bound the count by 16 (at most 16 + 8), and cp[24] lets this restatement report a larger
 * count instead of overflowing.  For every count up to 16 it computes what cp[16] does. */
static float box_overlap_impl(const float *box_a, const float *box_b, int mutant, int *cnt_out) {
    float a_x1 = box_a[0], a_y1 = box_a[1], a_x2 = box_a[2], a_y2 = box_a[3], a_angle = box_a[4];
    float b_x1 = box_b[0], b_y1 = box_b[1], b_x2 = box_b[2], b_y2 = box_b[3], b_angle = box_b[4];
    pt2 center_a = {(a_x1 + a_x2) / 2, (a_y1 + a_y2) / 2};
    pt2 center_b = {(b_x1 + b_x2) / 2, (b_y1 + b_y2) / 2};
    pt2 ca[5] = {{a_x1, a_y1}, {a_x2, a_y1}, {a_x2, a_y2}, {a_x1, a_y2}, {0, 0}};
    pt2 cb[5] = {{b_x1, b_y1}, {b_x2, b_y1}, {b_x2, b_y2}, {b_x1, b_y2}, {0, 0}};
    float a_cos = cosf(a_angle), a_sin = sinf(a_angle);
    float b_cos = cosf(b_angle), b_sin = sinf(b_angle);
    if (mutant == 2) { a_sin = -a_sin; b_sin = -b_sin; }
    for (int k = 0; k < 4; ++k) {
        rot_center(center_a, a_cos, a_sin, &ca[k]);
        rot_center(center_b, b_cos, b_sin, &cb[k]);
    }
    ca[4] = ca[0];
    cb[4] = cb[0];
    pt2 cp[24];
    pt2 pc = {0, 0};
    int cnt = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            if (seg_intersection(ca[i + 1], ca[i], cb[j + 1], cb[j], &cp[cnt])) {
                pc.x = pc.x + cp[cnt].x; pc.y = pc.y + cp[cnt].y;
                ++cnt;
            }
    for (int k = 0; k < 4; ++k) {
        if (!(mutant == 1 && k == 3) && in_box2d(box_a, cb[k])) {
            pc.x = pc.x + cb[k].x; pc.y = pc.y + cb[k].y;
            cp[cnt++] = cb[k];
        }
        if (in_box2d(box_b, ca[k])) {
            pc.x = pc.x + ca[k].x; pc.y = pc.y + ca[k].y;
            cp[cnt++] = ca[k];
        }
    }
    if (cnt_out) *cnt_out = cnt;
    pc.x /= cnt;
    pc.y /= cnt;
    for (int j = 0; j < cnt - 1 - (mutant == 4); ++j)
        for (int i = 0; i < cnt - j - 1; ++i) {
            float t0 = atan2f(cp[i].y - pc.y, cp[i].x - pc.x), t1 = atan2f(cp[i + 1].y - pc.y, cp[i + 1].x - pc.x);
            if (mutant == 3 ? t0 < t1 : t0 > t1) {
                pt2 t = cp[i]; cp[i] = cp[i + 1]; cp[i + 1] = t;
            }
        }
    float area = 0;
    for (int k = 0; k < cnt - 1; ++k) {
        pt2 u = {cp[k].x - cp[0].x, cp[k].y - cp[0].y};
        pt2 v = {cp[k + 1].x - cp[0].x, cp[k + 1].y - cp[0].y};
        area += cross2(u, v);
    }
    return (float)(fabsf(area) / 2.0);
}

ORC_API float orc_box_overlap(const float *box_a, const float *box_b) { return box_overlap_impl(box_a, box_b, 0, NULL); }

/* aligned pairs: out[k] = overlap(a[k], b[k]) (with the planted mistake `mutant`, see above), cnt[k] its polygon
 * vertex count (cnt may be NULL) */
ORC_API void orc_box_overlap_pairs(int n, const float *a, const float *b, int mutant, float *out, int *cnt) {
#pragma omp parallel for schedule(static, 256)
    for (int k = 0; k < n; ++k)
        out[k] = box_overlap_impl(a + (size_t)k * 5, b + (size_t)k * 5, mutant, cnt ? cnt + k : NULL);
}

ORC_API float orc_iou_bev(const float *a, const float *b) {
    float sa = (a[2] - a[0]) * (a[3] - a[1]);
    float sb = (b[2] - b[0]) * (b[3] - b[1]);
    float s = orc_box_overlap(a, b);
    return s / fmaxf(sa + sb - s, 1e-8f);
}

ORC_API float orc_iou_normal(const float *a, const float *b) {
    float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    float width = fmaxf(right - left, 0.f), height = fmaxf(bottom - top, 0.f);
    float interS = width * height;
    float Sa = (a[2] - a[0]) * (a[3] - a[1]);
    float Sb = (b[2] - b[0]) * (b[3] - b[1]);
    return interS / fmaxf(Sa + Sb - interS, 1e-8f);
}

ORC_API void orc_boxes_overlap_bev(int na, const float *a, int nb, const float *b, float *out) {
#pragma omp parallel for schedule(dynamic, 8)
    for (int i = 0; i < na; ++i)
        for (int j = 0; j < nb; ++j) out[(size_t)i * nb + j] = orc_box_overlap(a + i * 5, b + j * 5);
}

ORC_API void orc_boxes_iou_bev(int na, const float *a, int nb, const float *b, float *out) {
#pragma omp parallel for schedule(dynamic, 8)
    for (int i = 0; i < na; ++i)
        for (int j = 0; j < nb; ++j) out[(size_t)i * nb + j] = orc_iou_bev(a + i * 5, b + j * 5);
}

/* full (N x col_blocks) suppression mask exactly as nms_kernel / nms_normal_kernel write it */
ORC_API void orc_nms_mask(const float *boxes, int n, float thresh, int normal, uint64_t *mask) {
    const int cb = (n + 63) / 64;
#pragma omp parallel for schedule(dynamic, 8)
    for (int i = 0; i < n; ++i)
        for (int c = 0; c < cb; ++c) {
            uint64_t t = 0;
            int start = (i / 64 == c) ? (i % 64) + 1 : 0;
            int csz = n - c * 64 < 64 ? n - c * 64 : 64;
            for (int j = start; j < csz; ++j) {
                const float *bj = boxes + (size_t)(c * 64 + j) * 5;
                float v = normal ? orc_iou_normal(boxes + (size_t)i * 5, bj) : orc_iou_bev(boxes + (size_t)i * 5, bj);
                if (v > thresh) t |= 1ULL << j;
            }
            mask[(size_t)i * cb + c] = t;
        }
}

/* host greedy scan, iou3d.cpp:100-116 */
ORC_API int orc_nms_scan(const uint64_t *mask, int n, int64_t *keep) {
    const int cb = (n + 63) / 64;
    uint64_t *remv = (uint64_t *)calloc(cb > 0 ? cb : 1, sizeof(uint64_t));
    int num = 0;
    for (int i = 0; i < n; ++i) {
        int nblock = i / 64, inblock = i % 64;
        if (!(remv[nblock] & (1ULL << inblock))) {
            keep[num++] = i;
            const uint64_t *p = mask + (size_t)i * cb;
            for (int j = nblock; j < cb; ++j) remv[j] |= p[j];
        }
    }
    free(remv);
    return num;
}

ORC_API int orc_nms(const float *boxes, int n, float thresh, int normal, int64_t *keep) {
    const int cb = (n + 63) / 64;
    uint64_t *mask = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(n > 0 ? n : 1) * (cb > 0 ? cb : 1));
    orc_nms_mask(boxes, n, thresh, normal, mask);
    int num = orc_nms_scan(mask, n, keep);
    free(mask);
    return num;
}

ORC_API int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
