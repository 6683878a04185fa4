// ball_group.cu -- ball query, point grouping / gathering (+ their backward scatters), layout change.
//
// Replaces (paths relative to the reference tree):
//   ball_query_wrapper_fast       pointnet2_lib/pointnet2/src/ball_query.cpp:14-25 -> ball_query_gpu.cu:9-67
//   group_points_wrapper_fast     group_points.cpp:25-36 -> group_points_gpu.cu:47-86 (grad :8-44)
//   gather_points_wrapper_fast    sampling.cpp:11-33 -> sampling_gpu.cu:8-83
//
// Ball query semantics (the spec): for each centre scan the points in INDEX order, collect the first
// nsample with d2 < r*r (strict, fp32 r*r), pad the remaining slots with the first hit, leave the row
// untouched when nothing hits.  Here: one warp per centre tests 32 points per step; ballot + popc
// prefix keeps index order; the scene's points are staged through shared memory as SoA tiles shared by
// all the warps of the CTA; a second radius over the same centres rides along for free (MSG layers).
#include <stdint.h>

#include "rev_index.cuh"

namespace prb {

constexpr int BQ_THREADS = 256;
constexpr int BQ_WARPS = BQ_THREADS / 32;
constexpr int BQ_CPW = 4;                 // centres per warp
constexpr int BQ_TILE = 2048;             // points per shared-memory tile

template <int NR>
struct BqParams {
    int b, n, m;
    float r2[NR];
    int ns[NR];
    int *idx[NR];
    const float *new_xyz, *xyz;
};

template <int NR>
__global__ void __launch_bounds__(BQ_THREADS) ball_query_kernel(const BqParams<NR> p) {
    __shared__ float sx[BQ_TILE], sy[BQ_TILE], sz[BQ_TILE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.y;
    const int c0 = (blockIdx.x * BQ_WARPS + warp) * BQ_CPW;
    const float *xyz = p.xyz + (size_t)scene * p.n * 3;

    float cx[BQ_CPW], cy[BQ_CPW], cz[BQ_CPW];
    int cnt[BQ_CPW][NR], first[BQ_CPW][NR];
    bool live[BQ_CPW];
#pragma unroll
    for (int c = 0; c < BQ_CPW; ++c) {
        int ci = c0 + c;
        live[c] = ci < p.m;
        const float *q = p.new_xyz + ((size_t)scene * p.m + (live[c] ? ci : 0)) * 3;
        cx[c] = q[0]; cy[c] = q[1]; cz[c] = q[2];
#pragma unroll
        for (int r = 0; r < NR; ++r) { cnt[c][r] = 0; first[c][r] = 0; }
    }

    for (int t0 = 0; t0 < p.n; t0 += BQ_TILE) {
        const int tn = min(BQ_TILE, p.n - t0);
        bool warp_busy = false;
#pragma unroll
        for (int c = 0; c < BQ_CPW; ++c) {
            bool need = false;
#pragma unroll
            for (int r = 0; r < NR; ++r) need |= cnt[c][r] < p.ns[r];
            live[c] = live[c] && need;
            warp_busy |= live[c];
        }
        // barrier: previous tile fully consumed; early exit once every centre of the CTA is full
        if (!__syncthreads_or(warp_busy)) break;
        for (int i = tid; i < tn; i += BQ_THREADS) {
            sx[i] = xyz[(size_t)(t0 + i) * 3 + 0];
            sy[i] = xyz[(size_t)(t0 + i) * 3 + 1];
            sz[i] = xyz[(size_t)(t0 + i) * 3 + 2];
        }
        __syncthreads();
        if (!warp_busy) continue;  // uniform per warp; the CTA-level barriers stay matched
        float rmax = p.r2[0];
#pragma unroll
        for (int r = 1; r < NR; ++r) rmax = fmaxf(rmax, p.r2[r]);
        for (int i0 = 0; i0 < tn; i0 += 32) {
            const int i = i0 + lane;
            const bool in = i < tn;
            const float x = in ? sx[i] : 0.f, y = in ? sy[i] : 0.f, z = in ? sz[i] : 0.f;
            // pass 1: distances to the warp's live centres, ONE vote for "anything inside the largest ball?"
            // (LiDAR-like scenes: almost every 32-point step has no hit at all)
            float d2[BQ_CPW];
            bool any_hit = false;
#pragma unroll
            for (int c = 0; c < BQ_CPW; ++c) {
                // reference: d2 = (new_x-x)^2 + (new_y-y)^2 + (new_z-z)^2 in its SASS contraction order
                d2[c] = dist2_ref(cx[c] - x, cy[c] - y, cz[c] - z);
                any_hit |= live[c] && d2[c] < rmax;
            }
            if (!__any_sync(0xffffffffu, in && any_hit)) continue;
            // pass 2: ordered compaction of the hits
#pragma unroll
            for (int c = 0; c < BQ_CPW; ++c) {
                if (!live[c]) continue;
#pragma unroll
                for (int r = 0; r < NR; ++r) {
                    const unsigned hits = __ballot_sync(0xffffffffu, in && d2[c] < p.r2[r]);
                    if (hits == 0 || cnt[c][r] >= p.ns[r]) continue;
                    if (cnt[c][r] == 0) first[c][r] = t0 + i0 + __ffs(hits) - 1;
                    const int pos = cnt[c][r] + __popc(hits & ((1u << lane) - 1));
                    if (((hits >> lane) & 1u) && pos < p.ns[r])
                        p.idx[r][((size_t)scene * p.m + c0 + c) * p.ns[r] + pos] = t0 + i;
                    cnt[c][r] = min(p.ns[r], cnt[c][r] + __popc(hits));
                }
            }
        }
    }
    // pad with the first hit (the reference pre-fills all slots on the first hit)
#pragma unroll
    for (int c = 0; c < BQ_CPW; ++c) {
        if (c0 + c >= p.m) continue;
#pragma unroll
        for (int r = 0; r < NR; ++r) {
            if (cnt[c][r] == 0) continue;
            for (int s = cnt[c][r] + lane; s < p.ns[r]; s += 32)
                p.idx[r][((size_t)scene * p.m + c0 + c) * p.ns[r] + s] = first[c][r];
        }
    }
}

// out[b,c,j] = points[b,c,idx[b,j]] for a flat list of L = npoints*nsample indices per scene.
// One CTA owns a block of channels of one scene, so the (C_blk x N) source rows stay L1-resident
// while the index list streams through; writes are coalesced along j.
constexpr int GP_THREADS = 256;
constexpr int GP_CH = 8;

__global__ void __launch_bounds__(GP_THREADS) group_points_kernel(int c, int n, long L, const float *__restrict__ points,
                                                                  const int *__restrict__ idx, float *__restrict__ out) {
    const int scene = blockIdx.z, cb = blockIdx.y * GP_CH;
    const int nch = min(GP_CH, c - cb);
    const float *src = points + ((size_t)scene * c + cb) * n;
    const int *ix = idx + (size_t)scene * L;
    float *dst = out + ((size_t)scene * c + cb) * L;
    for (long j = (long)blockIdx.x * GP_THREADS + threadIdx.x; j < L; j += (long)gridDim.x * GP_THREADS) {
        const int k = ix[j];
#pragma unroll
        for (int ch = 0; ch < GP_CH; ++ch)
            if (ch < nch) dst[(size_t)ch * L + j] = __ldg(src + (size_t)ch * n + k);
    }
}

__global__ void __launch_bounds__(GP_THREADS) group_points_grad_kernel(int c, int n, long L, const float *__restrict__ grad_out,
                                                                       const int *__restrict__ idx, float *__restrict__ grad_points) {
    const int scene = blockIdx.z, cb = blockIdx.y * GP_CH;
    const int nch = min(GP_CH, c - cb);
    const float *g = grad_out + ((size_t)scene * c + cb) * L;
    const int *ix = idx + (size_t)scene * L;
    float *dst = grad_points + ((size_t)scene * c + cb) * n;
    for (long j = (long)blockIdx.x * GP_THREADS + threadIdx.x; j < L; j += (long)gridDim.x * GP_THREADS) {
        const int k = ix[j];
#pragma unroll
        for (int ch = 0; ch < GP_CH; ++ch)
            if (ch < nch) atomicAdd(dst + (size_t)ch * n + k, g[(size_t)ch * L + j]);
    }
}

// bfloat16 grouping (the same copy): each thread moves V consecutive references of its channel block.  V = 8 reads
// their indices as two 16-byte loads and writes each channel's 8 values as one 16-byte store (the launcher picks it when L
// is a multiple of 8 and idx / out are 16-byte aligned); V = 1 is the element-wise form for every other layout.
template <int V>
__global__ void __launch_bounds__(GP_THREADS) group_points_bf16_kernel(int c, int n, long L, const __nv_bfloat16 *__restrict__ points,
                                                                       const int *__restrict__ idx, __nv_bfloat16 *__restrict__ out) {
    const int scene = blockIdx.z, cb = blockIdx.y * GP_CH;
    const int nch = min(GP_CH, c - cb);
    const __nv_bfloat16 *src = points + ((size_t)scene * c + cb) * n;
    const int *ix = idx + (size_t)scene * L;
    __nv_bfloat16 *dst = out + ((size_t)scene * c + cb) * L;
    for (long j = ((long)blockIdx.x * GP_THREADS + threadIdx.x) * V; j < L; j += (long)gridDim.x * GP_THREADS * V) {
        int k[V];
        if constexpr (V == 8) {
            const int4 a = *reinterpret_cast<const int4 *>(ix + j), b = *reinterpret_cast<const int4 *>(ix + j + 4);
            k[0] = a.x; k[1] = a.y; k[2] = a.z; k[3] = a.w; k[4] = b.x; k[5] = b.y; k[6] = b.z; k[7] = b.w;
        } else {
            k[0] = ix[j];
        }
#pragma unroll
        for (int ch = 0; ch < GP_CH; ++ch) {
            if (ch >= nch) continue;
            const __nv_bfloat16 *row = src + (size_t)ch * n;
            if constexpr (V == 8) {
                __align__(16) __nv_bfloat16 v[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = __ldg(row + k[i]);
                *reinterpret_cast<uint4 *>(dst + (size_t)ch * L + j) = *reinterpret_cast<const uint4 *>(v);
            } else {
                dst[(size_t)ch * L + j] = __ldg(row + k[0]);
            }
        }
    }
}

// the atomic bfloat16 gradient, first pass: every reference adds its value, converted exactly, into fp32 sums (b, c, n)
__global__ void __launch_bounds__(GP_THREADS) group_points_grad_bf16_kernel(int c, int n, long L, const __nv_bfloat16 *__restrict__ grad_out,
                                                                            const int *__restrict__ idx, float *__restrict__ sums) {
    const int scene = blockIdx.z, cb = blockIdx.y * GP_CH;
    const int nch = min(GP_CH, c - cb);
    const __nv_bfloat16 *g = grad_out + ((size_t)scene * c + cb) * L;
    const int *ix = idx + (size_t)scene * L;
    float *dst = sums + ((size_t)scene * c + cb) * n;
    for (long j = (long)blockIdx.x * GP_THREADS + threadIdx.x; j < L; j += (long)gridDim.x * GP_THREADS) {
        const int k = ix[j];
#pragma unroll
        for (int ch = 0; ch < GP_CH; ++ch)
            if (ch < nch) atomicAdd(dst + (size_t)ch * n + k, __bfloat162float(g[(size_t)ch * L + j]));
    }
}

// (B,C,N) -> (B,N,C) through a 32x33 shared tile
__global__ void transpose_bcn_bnc_kernel(int c, int n, const float *__restrict__ in, float *__restrict__ out) {
    __shared__ float tile[32][33];
    const int scene = blockIdx.z;
    const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const float *src = in + (size_t)scene * c * n;
    float *dst = out + (size_t)scene * c * n;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int cc = c0 + i, nn = n0 + threadIdx.x;
        if (cc < c && nn < n) tile[i][threadIdx.x] = src[(size_t)cc * n + nn];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int nn = n0 + i, cc = c0 + threadIdx.x;
        if (cc < c && nn < n) dst[(size_t)nn * c + cc] = tile[threadIdx.x][i];
    }
}

static dim3 gp_grid(int b, int c, long L) {
    long bx = (L + GP_THREADS - 1) / GP_THREADS;
    if (bx > 1024) bx = 1024;
    if (bx < 1) bx = 1;
    return dim3((unsigned)bx, (unsigned)ceil_div(c, GP_CH), (unsigned)b);
}

}  // namespace prb

using namespace prb;

extern "C" int prb_ball_query(int b, int n, int m, float radius, int nsample, const float *new_xyz,
                              const float *xyz, int *idx, void *stream) {
    PRB_REQUIRE(b >= 0 && n >= 0 && m >= 0 && nsample > 0 && new_xyz && xyz && idx, "ball_query: bad arguments");
    if (b == 0 || m == 0) return 0;
    BqParams<1> p;
    p.b = b; p.n = n; p.m = m;
    p.r2[0] = radius * radius;  // fp32 product, as ball_query_gpu.cu:23
    p.ns[0] = nsample; p.idx[0] = idx; p.new_xyz = new_xyz; p.xyz = xyz;
    dim3 grid(ceil_div(m, BQ_WARPS * BQ_CPW), b);
    ball_query_kernel<1><<<grid, BQ_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("ball_query_kernel<1>");
}

extern "C" int prb_ball_query_msg2(int b, int n, int m, float radius0, int nsample0, float radius1, int nsample1,
                                   const float *new_xyz, const float *xyz, int *idx0, int *idx1, void *stream) {
    PRB_REQUIRE(b >= 0 && n >= 0 && m >= 0 && nsample0 > 0 && nsample1 > 0 && new_xyz && xyz && idx0 && idx1,
                "ball_query_msg2: bad arguments");
    if (b == 0 || m == 0) return 0;
    BqParams<2> p;
    p.b = b; p.n = n; p.m = m;
    p.r2[0] = radius0 * radius0; p.r2[1] = radius1 * radius1;
    p.ns[0] = nsample0; p.ns[1] = nsample1;
    p.idx[0] = idx0; p.idx[1] = idx1; p.new_xyz = new_xyz; p.xyz = xyz;
    dim3 grid(ceil_div(m, BQ_WARPS * BQ_CPW), b);
    ball_query_kernel<2><<<grid, BQ_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("ball_query_kernel<2>");
}

extern "C" int prb_group_points(int b, int c, int n, int npoints, int nsample, const float *points, const int *idx,
                                float *out, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n > 0 && points && idx && out, "group_points: bad arguments");
    long L = (long)npoints * nsample;
    if (b == 0 || c == 0 || L == 0) return 0;
    group_points_kernel<<<gp_grid(b, c, L), GP_THREADS, 0, (cudaStream_t)stream>>>(c, n, L, points, idx, out);
    return check_launch("group_points_kernel");
}

extern "C" int prb_group_points_grad(int b, int c, int n, int npoints, int nsample, const float *grad_out,
                                     const int *idx, float *grad_points, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n > 0 && grad_out && idx && grad_points, "group_points_grad: bad arguments");
    long L = (long)npoints * nsample;
    if (b == 0 || c == 0 || L == 0) return 0;
    group_points_grad_kernel<<<gp_grid(b, c, L), GP_THREADS, 0, (cudaStream_t)stream>>>(c, n, L, grad_out, idx, grad_points);
    return check_launch("group_points_grad_kernel");
}

// the ordered gradient: grad_points[b, c, j] += the sum of grad_out over the references of point j in increasing flat
// index, through the reverse index of idx (rev_index.cuh)
extern "C" size_t prb_group_points_grad_workspace_bytes(int b, int n, int npoints, int nsample) {
    const long L = (long)npoints * nsample;
    if (b <= 0 || n <= 0 || npoints <= 0 || nsample <= 0 || !rev_index_fits(b, L, n)) return 0;
    return rev_index_bytes(b, (int)L, n);
}

extern "C" int prb_group_points_grad_ws(int b, int c, int n, int npoints, int nsample, const float *grad_out, const int *idx,
                                        float *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n >= 0 && npoints >= 0 && nsample > 0, "group_points_grad_ws: bad dimensions");
    const long L = (long)npoints * nsample;
    if (b == 0 || c == 0 || n == 0 || L == 0) return 0;
    PRB_REQUIRE(rev_index_fits(b, L, n), "group_points_grad_ws: %d x %ld references over %d points", b, L, n);
    PRB_REQUIRE(grad_out && idx && grad_points && workspace, "group_points_grad_ws: bad arguments");
    const size_t need = rev_index_bytes(b, (int)L, n);
    PRB_REQUIRE(workspace_bytes >= need, "group_points_grad_ws: workspace of %zu bytes < %zu", workspace_bytes, need);
    const RevIndex R = rev_index_at(b, (int)L, n, workspace);
    const cudaStream_t s = (cudaStream_t)stream;
    if (int rc = rev_index_build(R, idx, s)) return rc;
    return seg_sum(R, SEG_GROUP, c, grad_out, nullptr, true, grad_points, s);
}

// gather == grouping with nsample = 1
extern "C" int prb_gather_points(int b, int c, int n, int npoints, const float *points, const int *idx, float *out,
                                 void *stream) {
    return prb_group_points(b, c, n, npoints, 1, points, idx, out, stream);
}
extern "C" int prb_gather_points_grad(int b, int c, int n, int npoints, const float *grad_out, const int *idx,
                                      float *grad_points, void *stream) {
    return prb_group_points_grad(b, c, n, npoints, 1, grad_out, idx, grad_points, stream);
}
extern "C" size_t prb_gather_points_grad_workspace_bytes(int b, int n, int npoints) {
    return prb_group_points_grad_workspace_bytes(b, n, npoints, 1);
}
extern "C" int prb_gather_points_grad_ws(int b, int c, int n, int npoints, const float *grad_out, const int *idx, float *grad_points,
                                         void *workspace, size_t workspace_bytes, void *stream) {
    return prb_group_points_grad_ws(b, c, n, npoints, 1, grad_out, idx, grad_points, workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------ bfloat16 grouping / gather (include/pointrcnn_b200.h)
extern "C" int prb_group_points_bf16(int b, int c, int n, int npoints, int nsample, const uint16_t *points, const int *idx, uint16_t *out,
                                     void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n > 0 && npoints >= 0 && nsample > 0 && points && idx && out, "group_points_bf16: bad arguments");
    const long L = (long)npoints * nsample;
    if (b == 0 || c == 0 || L == 0) return 0;
    const auto *p = reinterpret_cast<const __nv_bfloat16 *>(points);
    auto *o = reinterpret_cast<__nv_bfloat16 *>(out);
    const cudaStream_t s = (cudaStream_t)stream;
    if (L % 8 == 0 && (((uintptr_t)idx | (uintptr_t)out) & 15) == 0) {
        group_points_bf16_kernel<8><<<gp_grid(b, c, L / 8), GP_THREADS, 0, s>>>(c, n, L, p, idx, o);
        return check_launch("group_points_bf16_kernel<8>");
    }
    group_points_bf16_kernel<1><<<gp_grid(b, c, L), GP_THREADS, 0, s>>>(c, n, L, p, idx, o);
    return check_launch("group_points_bf16_kernel<1>");
}

extern "C" size_t prb_group_points_grad_bf16_workspace_bytes(int b, int c, int n) {
    if (b <= 0 || c <= 0 || n <= 0) return 0;
    return (size_t)b * c * n * sizeof(float);
}

extern "C" int prb_group_points_grad_bf16(int b, int c, int n, int npoints, int nsample, const uint16_t *grad_out, const int *idx,
                                          uint16_t *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n > 0 && npoints >= 0 && nsample > 0, "group_points_grad_bf16: bad dimensions");
    const long L = (long)npoints * nsample;
    if (b == 0 || c == 0) return 0;
    PRB_REQUIRE(grad_out && idx && grad_points && workspace, "group_points_grad_bf16: bad arguments");
    const size_t need = prb_group_points_grad_bf16_workspace_bytes(b, c, n);
    PRB_REQUIRE(workspace_bytes >= need, "group_points_grad_bf16: workspace of %zu bytes < %zu", workspace_bytes, need);
    const cudaStream_t s = (cudaStream_t)stream;
    float *sums = static_cast<float *>(workspace);
    PRB_CUDA(cudaMemsetAsync(sums, 0, need, s));
    if (L > 0) {
        group_points_grad_bf16_kernel<<<gp_grid(b, c, L), GP_THREADS, 0, s>>>(c, n, L, reinterpret_cast<const __nv_bfloat16 *>(grad_out),
                                                                               idx, sums);
        if (int rc = check_launch("group_points_grad_bf16_kernel")) return rc;
    }
    return round_bf16((size_t)b * c * n, sums, grad_points, s);
}

extern "C" int prb_group_points_grad_bf16_ws(int b, int c, int n, int npoints, int nsample, const uint16_t *grad_out, const int *idx,
                                             uint16_t *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n >= 0 && npoints >= 0 && nsample > 0, "group_points_grad_bf16_ws: bad dimensions");
    const long L = (long)npoints * nsample;
    if (b == 0 || c == 0 || n == 0) return 0;
    PRB_REQUIRE(grad_points, "group_points_grad_bf16_ws: bad arguments");
    const cudaStream_t s = (cudaStream_t)stream;
    if (L == 0) {   // no reference: every sum is +0
        PRB_CUDA(cudaMemsetAsync(grad_points, 0, (size_t)b * c * n * sizeof(uint16_t), s));
        return 0;
    }
    PRB_REQUIRE(rev_index_fits(b, L, n), "group_points_grad_bf16_ws: %d x %ld references over %d points", b, L, n);
    PRB_REQUIRE(grad_out && idx && workspace, "group_points_grad_bf16_ws: bad arguments");
    const size_t need = rev_index_bytes(b, (int)L, n);
    PRB_REQUIRE(workspace_bytes >= need, "group_points_grad_bf16_ws: workspace of %zu bytes < %zu", workspace_bytes, need);
    const RevIndex R = rev_index_at(b, (int)L, n, workspace);
    if (int rc = rev_index_build(R, idx, s)) return rc;
    return seg_sum_bf16(R, SEG_GROUP, c, reinterpret_cast<const __nv_bfloat16 *>(grad_out), nullptr,
                        reinterpret_cast<__nv_bfloat16 *>(grad_points), s);
}

extern "C" int prb_gather_points_bf16(int b, int c, int n, int npoints, const uint16_t *points, const int *idx, uint16_t *out, void *stream) {
    return prb_group_points_bf16(b, c, n, npoints, 1, points, idx, out, stream);
}
extern "C" int prb_gather_points_grad_bf16(int b, int c, int n, int npoints, const uint16_t *grad_out, const int *idx, uint16_t *grad_points,
                                           void *workspace, size_t workspace_bytes, void *stream) {
    return prb_group_points_grad_bf16(b, c, n, npoints, 1, grad_out, idx, grad_points, workspace, workspace_bytes, stream);
}
extern "C" int prb_gather_points_grad_bf16_ws(int b, int c, int n, int npoints, const uint16_t *grad_out, const int *idx,
                                              uint16_t *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    return prb_group_points_grad_bf16_ws(b, c, n, npoints, 1, grad_out, idx, grad_points, workspace, workspace_bytes, stream);
}

extern "C" int prb_transpose_bcn_to_bnc(int b, int c, int n, const float *in, float *out, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n >= 0 && in && out, "transpose: bad arguments");
    if (b == 0 || c == 0 || n == 0) return 0;
    dim3 grid(ceil_div(n, 32), ceil_div(c, 32), b), block(32, 8);
    transpose_bcn_bnc_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(c, n, in, out);
    return check_launch("transpose_bcn_bnc_kernel");
}
