// roipool3d.cu -- RoI point pooling (+ optional canonical transform) in one pass per box.
//
// Replaces roipool3d_gpu (lib/utils/roipool3d/src/roipool3d.cpp:48-79) -> roipool3dLauncher
// (roipool3d_kernel.cu:209-237: assign_pts_to_box3d, get_pooled_idx, roipool3d_forward, two
// cudaMalloc/cudaFree and a (B,N,M) int scratch per call) and, when asked, the canonical transform the
// caller applies right after (lib/net/rcnn_net.py:146-152, lib/utils/kitti_utils.py:45-63).
//
// Semantics (the spec): a point is inside a box iff pt_in_box3d (roipool3d_kernel.cu:14-28) says so;
// per box the first S inside points in point-index order are copied as rows [x,y,z,features...];
// 0 < cnt < S pads slot k with slot k % cnt; cnt == 0 sets empty_flag and leaves the rows untouched.
//
// Here: one CTA per (scene, box).  Per-box constants (cy, cos, sin, half sizes) are computed once; the
// CTA streams the scene's xyz 256 points at a time, compacts hits in index order with ballot + a
// warp-count prefix, stops at S hits, then copies the S rows as one flat, fully coalesced stream.
// The predicate keeps the reference's arithmetic: double for cy / the h,l,w half sizes and their
// compares, fp32 FMA shape of the rotation as in the reference's SASS
//   x_rot = fma(dx, cosa, -(dz*sina)),  z_rot = fma(dz, cosa, dx*sina).
#include <math_constants.h>

#include "common.cuh"

namespace prb {

constexpr int RP_THREADS = 256;
constexpr int RP_WARPS = RP_THREADS / 32;

struct BoxConst {
    float cx, cy, cz, cosa, sina;
    double half_h, half_l, half_w;
};

__device__ __forceinline__ BoxConst make_box(const float *bx) {
    BoxConst c;
    const float h = bx[3], w = bx[4], l = bx[5], angle = bx[6];
    c.cx = bx[0];
    c.cz = bx[2];
    c.half_h = (double)h / 2.0;
    c.half_l = (double)l / 2.0;
    c.half_w = (double)w / 2.0;
    c.cy = (float)((double)bx[1] - c.half_h);  // cy = bottom_y - h / 2.0, double then stored to float
    c.cosa = cosf(angle);
    c.sina = sinf(angle);
    return c;
}

__device__ __forceinline__ bool pt_in_box(const BoxConst &c, float x, float y, float z) {
    const float dx = x - c.cx, dz = z - c.cz;
    if (fabsf(dx) > 10.0f || (double)fabsf(y - c.cy) > c.half_h || fabsf(dz) > 10.0f) return false;
    const float x_rot = __fmaf_rn(dx, c.cosa, -__fmul_rn(dz, c.sina));
    const float z_rot = __fmaf_rn(dz, c.cosa, __fmul_rn(dx, c.sina));
    return ((double)x_rot >= -c.half_l) & ((double)x_rot <= c.half_l) & ((double)z_rot >= -c.half_w) &
           ((double)z_rot <= c.half_w);
}

// ------------------------------------------------------------------------------------------------ one-pass form (prb_roipool3d: no scratch)
__global__ void __launch_bounds__(RP_THREADS) roipool3d_kernel(int N, int M, int C, int S, const float *__restrict__ xyz,
                                                               const float *__restrict__ boxes3d,
                                                               const float *__restrict__ pts_feature,
                                                               float *__restrict__ pooled, int *__restrict__ empty_flag,
                                                               const float *__restrict__ rois) {
    extern __shared__ int s_idx[];  // S selected point indices
    __shared__ int s_wcnt[RP_WARPS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int box = blockIdx.x, scene = blockIdx.y;
    const BoxConst bc = make_box(boxes3d + ((size_t)scene * M + box) * 7);
    const float *pts = xyz + (size_t)scene * N * 3;

    int cnt = 0;  // uniform across the CTA
    for (int k0 = 0; k0 < N && cnt < S; k0 += RP_THREADS) {
        const int k = k0 + tid;
        bool in = false;
        if (k < N) in = pt_in_box(bc, pts[(size_t)k * 3], pts[(size_t)k * 3 + 1], pts[(size_t)k * 3 + 2]);
        const unsigned hits = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_wcnt[warp] = __popc(hits);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < RP_WARPS; ++w) {
            const int c = s_wcnt[w];
            before += w < warp ? c : 0;
            total += c;
        }
        const int pos = cnt + before + __popc(hits & ((1u << lane) - 1));
        if (in && pos < S) s_idx[pos] = k;
        cnt = min(S, cnt + total);
        __syncthreads();
    }
    if (cnt == 0) {
        if (tid == 0) empty_flag[(size_t)scene * M + box] = 1;
        if (rois) {   // the reference applies the canonical transform to the (zero) rows of empty boxes as well
            const float *r = rois + ((size_t)scene * M + box) * 7;
            const float c = cosf(r[6]), s = sinf(r[6]);
            const float x = 0.f - r[0], y = 0.f - r[1], z = 0.f - r[2];
            const float ex = __fmaf_rn(x, c, -__fmul_rn(z, s)), ez = __fmaf_rn(x, s, __fmul_rn(z, c));
            const int W = 3 + C;
            float *dst = pooled + ((size_t)scene * M + box) * (size_t)S * W;
            for (int row = tid; row < S; row += RP_THREADS) { dst[(size_t)row * W] = ex; dst[(size_t)row * W + 1] = y; dst[(size_t)row * W + 2] = ez; }
        }
        return;
    }

    // canonical transform constants (rcnn_net.py:146-152): xyz -= roi centre, rotate (x,z) by roi ry
    float rcx = 0.f, rcy = 0.f, rcz = 0.f, rcos = 1.f, rsin = 0.f;
    if (rois) {
        const float *r = rois + ((size_t)scene * M + box) * 7;
        rcx = r[0]; rcy = r[1]; rcz = r[2];
        rcos = cosf(r[6]); rsin = sinf(r[6]);
    }
    const int W = 3 + C;
    const float *feat = pts_feature + (size_t)scene * N * C;
    float *dst = pooled + ((size_t)scene * M + box) * (size_t)S * W;
    // warp per row, lanes along the row: both the feature read and the pooled write are coalesced
    for (int row = warp; row < S; row += RP_WARPS) {
        const int k = s_idx[row < cnt ? row : row % cnt];
        float *o = dst + (size_t)row * W;
        if (lane < 3) {
            float v;
            if (rois) {
                const float x = pts[(size_t)k * 3] - rcx, y = pts[(size_t)k * 3 + 1] - rcy, z = pts[(size_t)k * 3 + 2] - rcz;
                // [x z] @ [[cos,-sin],[sin,cos]]^T : x' = x*cos - z*sin, z' = x*sin + z*cos
                v = lane == 0 ? __fmaf_rn(x, rcos, -__fmul_rn(z, rsin)) : (lane == 1 ? y : __fmaf_rn(x, rsin, __fmul_rn(z, rcos)));
            } else {
                v = pts[(size_t)k * 3 + lane];
            }
            o[lane] = v;
        }
        const float *f = feat + (size_t)k * C;
        for (int j = lane; j < C; j += 32) o[3 + j] = __ldg(f + j);
    }
}


// ------------------------------------------------------------------------------------------------ two-pass form
// Pass A (assign) writes each box's first S inside points in index order -> idx (B,M,S) int32 + cnt (B,M) in caller
// scratch: binned (below) for scenes of at most RG_MAX_POINTS points, exhaustive for larger ones.
// Pass B (copy): one CTA per box streams the S x (3+C) output as ONE flat array with 128-bit stores (rows are
// 532 bytes at C4, so row-aligned stores are 4 bytes per lane).  Empty boxes set the flag and, when asked, zero their
// rows, so the caller need not pre-zero the 558 MB output.
//
// Pass A, exhaustive: one CTA per (scene, tile of RA_BOXES boxes).  The scene's points are read ONCE per tile (the
// reference and the one-pass kernel above re-read all N points for every box).  Warp w owns the contiguous point range
// [w*N/8, (w+1)*N/8): it appends the hits of every box to its own ordered list in shared memory (ballot + popc prefix, no
// CTA barrier inside the scan); the lists are then concatenated in warp order, which IS point-index order, and cut at S.
constexpr int RA_BOXES = 4;
constexpr int RA_WARPS = 8;
constexpr int RA_UNROLL = 4;     // points per lane per step: 12 coordinate loads in flight per lane

__global__ void __launch_bounds__(32 * RA_WARPS) roipool3d_assign_kernel(int N, int M, int S, const float *__restrict__ xyz,
                                                                        const float *__restrict__ boxes3d,
                                                                        int *__restrict__ idx_out, int *__restrict__ cnt_out) {
    extern __shared__ int s_list[];      // [RA_BOXES][RA_WARPS][S]
    __shared__ int s_cnt[RA_BOXES][RA_WARPS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int box0 = blockIdx.x * RA_BOXES, scene = blockIdx.y;
    const int nb = min(RA_BOXES, M - box0);
    BoxConst bc[RA_BOXES];
#pragma unroll
    for (int b = 0; b < RA_BOXES; ++b) bc[b] = make_box(boxes3d + ((size_t)scene * M + box0 + (b < nb ? b : 0)) * 7);
    const float *pts = xyz + (size_t)scene * N * 3;
    const int per = (N + RA_WARPS - 1) / RA_WARPS;
    const int lo = warp * per, hi = min(N, lo + per);
    int cnt[RA_BOXES];
#pragma unroll
    for (int b = 0; b < RA_BOXES; ++b) cnt[b] = 0;
    for (int k0 = lo; k0 < hi; k0 += 32 * RA_UNROLL) {
        float x[RA_UNROLL], y[RA_UNROLL], z[RA_UNROLL];
#pragma unroll
        for (int j = 0; j < RA_UNROLL; ++j) {          // all loads of the step first
            const int k = k0 + 32 * j + lane;
            x[j] = y[j] = z[j] = 0.f;
            if (k < hi) { x[j] = __ldg(pts + (size_t)k * 3); y[j] = __ldg(pts + (size_t)k * 3 + 1); z[j] = __ldg(pts + (size_t)k * 3 + 2); }
        }
#pragma unroll
        for (int j = 0; j < RA_UNROLL; ++j) {          // then the tests, in point order
            const int k = k0 + 32 * j + lane;
            const bool ok = k < hi;
#pragma unroll
            for (int b = 0; b < RA_BOXES; ++b) {
                const bool in = ok && b < nb && pt_in_box(bc[b], x[j], y[j], z[j]);
                const unsigned hits = __ballot_sync(0xffffffffu, in);
                if (hits) {
                    const int pos = cnt[b] + __popc(hits & ((1u << lane) - 1));
                    if (in && pos < S) s_list[((size_t)b * RA_WARPS + warp) * S + pos] = k;
                    cnt[b] = min(S, cnt[b] + __popc(hits));
                }
            }
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int b = 0; b < RA_BOXES; ++b) s_cnt[b][warp] = cnt[b];
    }
    __syncthreads();
    // concatenate the per-warp lists (warp order = point order), cut at S
    for (int b = 0; b < nb; ++b) {
        int off = 0;
        for (int w = 0; w < RA_WARPS; ++w) {
            const int c = s_cnt[b][w];
            const int take = min(c, S - off);
            int *dst = idx_out + ((size_t)scene * M + box0 + b) * S + off;
            for (int j = tid; j < take; j += 32 * RA_WARPS) dst[j] = s_list[((size_t)b * RA_WARPS + w) * S + j];
            off += take;
            if (off >= S) break;
        }
        if (tid == 0) cnt_out[(size_t)scene * M + box0 + b] = off;
    }
}

// Pass A, binned (scenes of at most RG_MAX_POINTS points): the exhaustive pass above tests every point against every box
// (B*N*M = 33.5 M predicates at C4, ~100 us).  Here the scene's points are first bucketed into an RG x RG grid over their
// x-z bounding box (one CTA per scene: bounds, histogram, scan, scatter -> a point permutation grouped by cell, cells
// row-major in z), and a box only tests the points of the cells its footprint touches.  Index ORDER is restored by a
// bitmap: hits set bit k of an N-bit shared-memory bitmap, one warp then walks the bitmap word by word (popc prefix) and
// emits the first S set bits -- exactly "the first S inside points in point-index order" (roipool3d_kernel.cu:81-110).
// Exactness: the predicate is the same pt_in_box; the footprint is conservative -- an inside point has
// |x - cx| <= min(10, |cos| l/2 + |sin| w/2) (+ rounding, covered by the margin), likewise z, and the cell function is
// monotone, so cell(x) lies in [cell(cx - ex), cell(cx + ex)].
constexpr int RG = 64;
constexpr int RG_CELLS = RG * RG;
constexpr int RG_MAX_POINTS = 262144;     // bitmap of 32 KB
constexpr int RG_THREADS = 1024;

struct SceneGrid { float x0, z0, invx, invz; };

__device__ __forceinline__ int grid_cell(float v, float v0, float inv) {
    // NaN -> 0 (fmaxf returns the non-NaN operand); never out of range
    return (int)fminf(fmaxf((v - v0) * inv, 0.f), (float)(RG - 1));
}

__global__ void __launch_bounds__(RG_THREADS) roipool3d_bin_kernel(int N, const float *__restrict__ xyz, int *__restrict__ sorted_idx,
                                                                  int *__restrict__ cell_start, SceneGrid *__restrict__ grids) {
    __shared__ int s_hist[RG_CELLS];
    __shared__ float s_red[4][RG_THREADS / 32];
    __shared__ int s_wsum[RG_THREADS / 32];
    __shared__ SceneGrid s_g;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, scene = blockIdx.x;
    const float *pts = xyz + (size_t)scene * N * 3;
    int *sorted = sorted_idx + (size_t)scene * N;
    int *cstart = cell_start + (size_t)scene * (RG_CELLS + 1);
    // bounds of the finite x / z coordinates
    float xlo = CUDART_INF_F, xhi = -CUDART_INF_F, zlo = CUDART_INF_F, zhi = -CUDART_INF_F;
    for (int k = tid; k < N; k += RG_THREADS) {
        const float x = pts[(size_t)k * 3], z = pts[(size_t)k * 3 + 2];
        if (fabsf(x) <= 3.0e38f) { xlo = fminf(xlo, x); xhi = fmaxf(xhi, x); }
        if (fabsf(z) <= 3.0e38f) { zlo = fminf(zlo, z); zhi = fmaxf(zhi, z); }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        xlo = fminf(xlo, __shfl_xor_sync(0xffffffffu, xlo, o)); xhi = fmaxf(xhi, __shfl_xor_sync(0xffffffffu, xhi, o));
        zlo = fminf(zlo, __shfl_xor_sync(0xffffffffu, zlo, o)); zhi = fmaxf(zhi, __shfl_xor_sync(0xffffffffu, zhi, o));
    }
    if (lane == 0) { s_red[0][warp] = xlo; s_red[1][warp] = xhi; s_red[2][warp] = zlo; s_red[3][warp] = zhi; }
    for (int i = tid; i < RG_CELLS; i += RG_THREADS) s_hist[i] = 0;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < RG_THREADS / 32; ++w) {
            xlo = fminf(xlo, s_red[0][w]); xhi = fmaxf(xhi, s_red[1][w]); zlo = fminf(zlo, s_red[2][w]); zhi = fmaxf(zhi, s_red[3][w]);
        }
        SceneGrid g;
        g.x0 = xlo <= xhi ? xlo : 0.f;
        g.z0 = zlo <= zhi ? zlo : 0.f;
        const float dx = xlo <= xhi ? xhi - xlo : 0.f, dz = zlo <= zhi ? zhi - zlo : 0.f;
        g.invx = dx > 1e-20f && dx < 3.0e38f ? (float)RG / dx : 0.f;
        g.invz = dz > 1e-20f && dz < 3.0e38f ? (float)RG / dz : 0.f;
        s_g = g;
        grids[scene] = g;
    }
    __syncthreads();
    const SceneGrid g = s_g;
    for (int k = tid; k < N; k += RG_THREADS) {
        const int c = grid_cell(pts[(size_t)k * 3 + 2], g.z0, g.invz) * RG + grid_cell(pts[(size_t)k * 3], g.x0, g.invx);
        atomicAdd(&s_hist[c], 1);
    }
    __syncthreads();
    // exclusive scan of the RG_CELLS counts: 4 per thread, warp scan, scan of the warp sums
    constexpr int PER = RG_CELLS / RG_THREADS;
    int v[PER], sum = 0;
#pragma unroll
    for (int i = 0; i < PER; ++i) { v[i] = s_hist[tid * PER + i]; sum += v[i]; }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = s_wsum[lane];
        int wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
        s_wsum[lane] = wi - w;
    }
    __syncthreads();
    int run = s_wsum[warp] + incl - sum;
#pragma unroll
    for (int i = 0; i < PER; ++i) { s_hist[tid * PER + i] = run; cstart[tid * PER + i] = run; run += v[i]; }
    if (tid == RG_THREADS - 1) cstart[RG_CELLS] = run;
    __syncthreads();
    for (int k = tid; k < N; k += RG_THREADS) {
        const int c = grid_cell(pts[(size_t)k * 3 + 2], g.z0, g.invz) * RG + grid_cell(pts[(size_t)k * 3], g.x0, g.invx);
        sorted[atomicAdd(&s_hist[c], 1)] = k;          // order inside a cell is irrelevant: the bitmap restores index order
    }
}

// One CTA per (scene, box): set the bit of every inside point in s_bits (N bits), then warp 0 walks the bitmap and writes
// the first S set bits -- "the first S inside points in point-index order" -- and their count.
constexpr int RGA_THREADS = 128;
__global__ void __launch_bounds__(RGA_THREADS) roipool3d_assign_grid_kernel(int N, int M, int S, const float *__restrict__ xyz,
                                                                           const float *__restrict__ boxes3d,
                                                                           const int *__restrict__ sorted_idx,
                                                                           const int *__restrict__ cell_start,
                                                                           const SceneGrid *__restrict__ grids,
                                                                           int *__restrict__ idx_out, int *__restrict__ cnt_out) {
    extern __shared__ unsigned int s_bits[];          // ceil(N / 32) words
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int box = blockIdx.x, scene = blockIdx.y;
    const size_t bi = (size_t)scene * M + box;
    const float *pts = xyz + (size_t)scene * N * 3;
    const int *sorted = sorted_idx + (size_t)scene * N;
    const int *cstart = cell_start + (size_t)scene * (RG_CELLS + 1);
    const SceneGrid g = grids[scene];
    const int nwords = (N + 31) >> 5;
    for (int i = tid; i < nwords; i += RGA_THREADS) s_bits[i] = 0u;
    const BoxConst bc = make_box(boxes3d + bi * 7);
    // conservative x-z footprint of the predicate (see above); NaN / Inf boxes degrade to "every cell" or "cell 0", both safe
    const float hl = (float)bc.half_l, hw = (float)bc.half_w, ac = fabsf(bc.cosa), as = fabsf(bc.sina);
    float ex = fminf(__fmaf_rn(ac, hl, as * hw), 10.f), ez = fminf(__fmaf_rn(as, hl, ac * hw), 10.f);
    ex = ex * 1.0001f + 1e-3f + 1e-6f * fabsf(bc.cx);
    ez = ez * 1.0001f + 1e-3f + 1e-6f * fabsf(bc.cz);
    int xc0 = grid_cell(bc.cx - ex, g.x0, g.invx), xc1 = grid_cell(bc.cx + ex, g.x0, g.invx);
    int zc0 = grid_cell(bc.cz - ez, g.z0, g.invz), zc1 = grid_cell(bc.cz + ez, g.z0, g.invz);
    if (!(ex == ex) || !(ez == ez) || !(bc.cx == bc.cx) || !(bc.cz == bc.cz)) { xc0 = zc0 = 0; xc1 = zc1 = RG - 1; }
    if (xc0 > xc1) { const int t = xc0; xc0 = xc1; xc1 = t; }
    if (zc0 > zc1) { const int t = zc0; zc0 = zc1; zc1 = t; }
    __syncthreads();
    // a z-row of the footprint is one contiguous span of the permutation
    for (int zc = zc0 + warp; zc <= zc1; zc += RGA_THREADS / 32) {
        const int lo = cstart[zc * RG + xc0], hi = cstart[zc * RG + xc1 + 1];
        for (int e = lo + lane; e < hi; e += 32) {
            const int k = sorted[e];
            if (pt_in_box(bc, pts[(size_t)k * 3], pts[(size_t)k * 3 + 1], pts[(size_t)k * 3 + 2]))
                atomicOr(&s_bits[k >> 5], 1u << (k & 31));
        }
    }
    __syncthreads();
    if (warp != 0) return;
    int *list = idx_out + bi * S;
    int run = 0;
    for (int w0 = 0; w0 < nwords && run < S; w0 += 32) {
        unsigned word = w0 + lane < nwords ? s_bits[w0 + lane] : 0u;
        const int c = __popc(word);
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        int pos = run + incl - c;
        const int base = (w0 + lane) << 5;
        while (word && pos < S) {
            const int b = __ffs(word) - 1;
            word &= word - 1;
            list[pos++] = base + b;
        }
        run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) cnt_out[bi] = min(run, S);
}

// Pass B.  A box usually holds far fewer than S points, so its S output rows are `cnt` distinct rows repeated cyclically:
// flat, the output IS the cnt x (3+C) source block repeated -- out[e] = block[e mod (cnt*(3+C))].  The block is staged in
// shared memory once (coalesced row reads, canonical transform applied there) and streamed out with 128-bit stores;
// boxes with more points than the staging area holds take the direct paths below.
constexpr int RB_STAGE_FLOATS = 12 * 1024;   // 48 KB: 92 rows of 133 floats.  Data dependent: a smaller area suits boxes that
                                             // hold a few points, 48 KB the ~60 points per enlarged RoI of the RCNN stage

__global__ void __launch_bounds__(RP_THREADS) roipool3d_copy_kernel(int N, int M, int C, int S, const float *__restrict__ xyz,
                                                                    const float *__restrict__ pts_feature,
                                                                    const int *__restrict__ idx_in, const int *__restrict__ cnt_in,
                                                                    float *__restrict__ pooled, int *__restrict__ empty_flag,
                                                                    const float *__restrict__ rois, int zero_fill) {
    extern __shared__ float s_blk[];          // RB_STAGE_FLOATS floats, then S ints (the direct paths' index list)
    int *s_idx = reinterpret_cast<int *>(s_blk + RB_STAGE_FLOATS);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int box = blockIdx.x, scene = blockIdx.y;
    const size_t bi = (size_t)scene * M + box;
    const int cnt = cnt_in[bi];
    const int W = 3 + C;
    const long total = (long)S * W;
    float *dst = pooled + bi * (size_t)total;
    const bool vec = (total & 3) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
    // canonical transform constants (rcnn_net.py:146-152): xyz -= roi centre, rotate (x,z) by roi ry
    float rcx = 0.f, rcy = 0.f, rcz = 0.f, rcos = 1.f, rsin = 0.f;
    if (rois) {
        const float *r = rois + bi * 7;
        rcx = r[0]; rcy = r[1]; rcz = r[2];
        rcos = cosf(r[6]); rsin = sinf(r[6]);
    }
    auto canon = [&](float px, float py, float pz, int col) -> float {
        const float x = px - rcx, y = py - rcy, z = pz - rcz;
        // [x z] @ [[cos,-sin],[sin,cos]]^T : x' = x*cos - z*sin, z' = x*sin + z*cos
        return col == 0 ? __fmaf_rn(x, rcos, -__fmul_rn(z, rsin)) : (col == 1 ? y : __fmaf_rn(x, rsin, __fmul_rn(z, rcos)));
    };
    if (cnt == 0) {
        if (tid == 0) empty_flag[bi] = 1;
        // The reference leaves the rows of an empty box zero -- and then applies the canonical transform to those zeros too
        // (rcnn_net.py:146-152 runs over every RoI).  With the transform fused, an empty box's xyz columns get the
        // transformed origin; without it the rows are zero-filled on request or left to the caller's memset.
        if (rois) {
            const float ex = canon(0.f, 0.f, 0.f, 0), ey = canon(0.f, 0.f, 0.f, 1), ez = canon(0.f, 0.f, 0.f, 2);
            for (long e = tid; e < total; e += RP_THREADS) { const int c = (int)(e % W); dst[e] = c == 0 ? ex : (c == 1 ? ey : (c == 2 ? ez : 0.f)); }
        } else if (zero_fill) {
            if (vec) for (long e = 4L * tid; e < total; e += 4L * RP_THREADS) *reinterpret_cast<float4 *>(dst + e) = make_float4(0.f, 0.f, 0.f, 0.f);
            else for (long e = tid; e < total; e += RP_THREADS) dst[e] = 0.f;
        }
        return;
    }
    const float *pts = xyz + (size_t)scene * N * 3;
    const float *feat = pts_feature + (size_t)scene * N * C;
    const int *idx = idx_in + bi * S;
    if ((long)cnt * W <= RB_STAGE_FLOATS && vec) {
        // ---- stage the cnt distinct rows (warp per row, lanes along the row), then stream the block cyclically
        for (int j = warp; j < cnt; j += RP_WARPS) {
            const int k = idx[j];
            float *row = s_blk + (size_t)j * W;
            if (lane < 3) {
                const float px = __ldg(pts + (size_t)k * 3), py = __ldg(pts + (size_t)k * 3 + 1), pz = __ldg(pts + (size_t)k * 3 + 2);
                row[lane] = rois ? canon(px, py, pz, lane) : (lane == 0 ? px : (lane == 1 ? py : pz));
            }
            const float *f = feat + (size_t)k * C;
            for (int c = lane; c < C; c += 32) row[3 + c] = __ldg(f + c);
        }
        __syncthreads();
        const int P = cnt * W;                       // period of the output, in floats
        const int step = (4 * RP_THREADS) % P;
        int m = (4 * tid) % P;
        for (long e = 4L * tid; e < total; e += 4L * RP_THREADS) {
            float4 v;
            if (m + 3 < P) {
                v = make_float4(s_blk[m], s_blk[m + 1], s_blk[m + 2], s_blk[m + 3]);
            } else {                                 // the unit wraps around the end of the block
                float t[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) { int mm = m + q; if (mm >= P) mm -= P; t[q] = s_blk[mm]; }
                v = make_float4(t[0], t[1], t[2], t[3]);
            }
            *reinterpret_cast<float4 *>(dst + e) = v;
            m += step;
            if (m >= P) m -= P;
        }
        return;
    }
    // ---- direct paths: many points in the box (or an unaligned output)
    for (int j = tid; j < S; j += RP_THREADS) s_idx[j] = idx[j < cnt ? j : j % cnt];
    __syncthreads();
    auto value = [&](int row, int col) -> float {
        const int k = s_idx[row];
        if (col >= 3) return __ldg(feat + (size_t)k * C + (col - 3));
        if (!rois) return __ldg(pts + (size_t)k * 3 + col);
        return canon(__ldg(pts + (size_t)k * 3), __ldg(pts + (size_t)k * 3 + 1), __ldg(pts + (size_t)k * 3 + 2), col);
    };
    if (vec && W <= RB_STAGE_FLOATS / 2) {
        // ---- chunked staging (boxes with more distinct rows than the staging area holds: the regime of real RoIs, ~60 and
        // more points per enlarged box): the output is produced in pieces of CH rows -- gather the piece's rows into shared
        // memory (warp per row, coalesced), stream the piece out with 128-bit stores -- instead of assembling every float4
        // from four scalar loads through L1.  Pieces are cut at multiples of 4 floats, so a piece needs one row more than
        // its length.
        const int CH = RB_STAGE_FLOATS / W - 1;                 // whole rows per piece (>= 1)
        const long piece = ((long)CH * W) & ~3L;
        for (long f0 = 0; f0 < total; f0 += piece) {
            const long f1 = f0 + piece < total ? f0 + piece : total;
            const int r0 = (int)(f0 / W), r1 = (int)((f1 - 1) / W);
            __syncthreads();                                     // the previous piece has been streamed out
            for (int j = r0 + warp; j <= r1; j += RP_WARPS) {
                const int k = s_idx[j];
                float *row = s_blk + (size_t)(j - r0) * W;
                if (lane < 3) {
                    const float px = __ldg(pts + (size_t)k * 3), py = __ldg(pts + (size_t)k * 3 + 1), pz = __ldg(pts + (size_t)k * 3 + 2);
                    row[lane] = rois ? canon(px, py, pz, lane) : (lane == 0 ? px : (lane == 1 ? py : pz));
                }
                const float *f = feat + (size_t)k * C;
                for (int c = lane; c < C; c += 32) row[3 + c] = __ldg(f + c);
            }
            __syncthreads();
            const float *src = s_blk - (size_t)r0 * W;           // src[e] is output element e of this box
            for (long e = f0 + 4L * tid; e < f1; e += 4L * RP_THREADS)
                *reinterpret_cast<float4 *>(dst + e) = make_float4(src[e], src[e + 1], src[e + 2], src[e + 3]);
        }
    } else if (vec) {
        // rows wider than half the staging area: sources through L1.  Thread t owns float4 units t, t + T, ...: (row, col)
        // of the unit's first float advance by a constant stride
        const int step = 4 * RP_THREADS;
        const int d_row = step / W, d_col = step % W;
        int row = 4 * tid / W, col = 4 * tid % W;
        for (long e = 4L * tid; e < total; e += step) {
            float v[4];
            int r = row, c = col;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                v[q] = value(r, c);
                if (++c == W) { c = 0; ++r; }
            }
            *reinterpret_cast<float4 *>(dst + e) = make_float4(v[0], v[1], v[2], v[3]);
            row += d_row; col += d_col;
            if (col >= W) { col -= W; ++row; }
        }
    } else {
        for (long e = tid; e < total; e += RP_THREADS) dst[e] = value((int)(e / W), (int)(e % W));
    }
}

}  // namespace prb

using namespace prb;

// scratch: idx (B,M,S) + cnt (B,M) + the binned pass's point permutation (B,N), cell offsets (B, RG*RG+1) and grid parameters
extern "C" size_t prb_roipool3d_workspace_bytes(int B, int N, int M, int S) {
    return ((size_t)B * M * S + (size_t)B * M + (size_t)B * N + (size_t)B * (RG_CELLS + 1) + 4 * (size_t)B + 64) * sizeof(int) + 256;
}

// two-pass form with caller scratch; zero_fill_empty != 0: rows of empty boxes are zeroed by the kernel (the caller may
// pass an uninitialised `pooled`), 0: they are left untouched like the reference (caller pre-zeroes)
extern "C" int prb_roipool3d_ws(int B, int N, int M, int C, int S, const float *xyz, const float *boxes3d,
                                const float *pts_feature, float *pooled, int *empty_flag, const float *rois_canonical,
                                int zero_fill_empty, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(B >= 0 && N >= 0 && M >= 0 && C >= 0 && S > 0 && xyz && boxes3d && pooled && empty_flag && (C == 0 || pts_feature),
                "roipool3d: bad arguments");
    if (B == 0 || M == 0) return 0;
    PRB_REQUIRE(workspace && workspace_bytes >= prb_roipool3d_workspace_bytes(B, N, M, S), "roipool3d: workspace too small");
    // The largest S the entry accepts: 3200 up to 65536 points, 1600 above.  The exhaustive pass A keeps RA_BOXES x RA_WARPS
    // x S int indices in shared memory, so it takes S <= 1600 within the 200 KB; the binned pass has no limit of its own.
    PRB_REQUIRE(S <= (N <= 65536 ? 3200 : 1600), "roipool3d: sampled_pts_num %d too large", S);
    int *idx = reinterpret_cast<int *>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    int *cnt = idx + (size_t)B * M * S;
    cudaStream_t st = (cudaStream_t)stream;
    if (N <= RG_MAX_POINTS) {
        int *sorted = cnt + (size_t)B * M;
        int *cstart = sorted + (size_t)B * N;
        SceneGrid *grids = reinterpret_cast<SceneGrid *>(((uintptr_t)(cstart + (size_t)B * (RG_CELLS + 1)) + 15) & ~(uintptr_t)15);
        roipool3d_bin_kernel<<<B, RG_THREADS, 0, st>>>(N, xyz, sorted, cstart, grids);
        if (int rc = check_launch("roipool3d_bin_kernel")) return rc;
        const size_t smem_bits = (size_t)((N + 31) / 32) * sizeof(unsigned int);
        roipool3d_assign_grid_kernel<<<dim3(M, B), RGA_THREADS, smem_bits, st>>>(N, M, S, xyz, boxes3d, sorted, cstart, grids, idx, cnt);
        if (int rc = check_launch("roipool3d_assign_grid_kernel")) return rc;
    } else {
        const size_t smem_a = (size_t)RA_BOXES * RA_WARPS * S * sizeof(int);
        if (smem_a > 48 * 1024)
            PRB_CUDA(cudaFuncSetAttribute(roipool3d_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_a));
        roipool3d_assign_kernel<<<dim3(ceil_div(M, RA_BOXES), B), 32 * RA_WARPS, smem_a, st>>>(N, M, S, xyz, boxes3d, idx, cnt);
        if (int rc = check_launch("roipool3d_assign_kernel")) return rc;
    }
    const size_t smem_b = (size_t)RB_STAGE_FLOATS * sizeof(float) + (size_t)S * sizeof(int);
    if (smem_b > 48 * 1024)
        PRB_CUDA(cudaFuncSetAttribute(roipool3d_copy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_b));
    roipool3d_copy_kernel<<<dim3(M, B), RP_THREADS, smem_b, st>>>(N, M, C, S, xyz, pts_feature, idx, cnt, pooled, empty_flag,
                                                                 rois_canonical, zero_fill_empty);
    return check_launch("roipool3d_copy_kernel");
}

extern "C" int prb_roipool3d(int B, int N, int M, int C, int S, const float *xyz, const float *boxes3d,
                             const float *pts_feature, float *pooled, int *empty_flag, const float *rois_canonical,
                             void *stream) {
    PRB_REQUIRE(B >= 0 && N >= 0 && M >= 0 && C >= 0 && S > 0 && xyz && boxes3d && pooled && empty_flag && (C == 0 || pts_feature),
                "roipool3d: bad arguments");
    if (B == 0 || M == 0) return 0;
    PRB_REQUIRE((size_t)S * sizeof(int) <= 200 * 1024, "roipool3d: sampled_pts_num %d too large", S);
    size_t smem = (size_t)S * sizeof(int);
    if (smem > 48 * 1024)
        PRB_CUDA(cudaFuncSetAttribute(roipool3d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(M, B);
    roipool3d_kernel<<<grid, RP_THREADS, smem, (cudaStream_t)stream>>>(N, M, C, S, xyz, boxes3d, pts_feature, pooled,
                                                                      empty_flag, rois_canonical);
    return check_launch("roipool3d_kernel");
}
