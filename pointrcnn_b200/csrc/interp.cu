// interp.cu -- three nearest neighbours (+ inverse-distance weights) and 3-point interpolation.
//
// Replaces three_nn_wrapper_fast / three_interpolate_wrapper_fast / three_interpolate_grad_wrapper_fast
// (pointnet2_lib/pointnet2/src/interpolate.cpp:14-54 -> interpolate_gpu.cu:9-161) and the weight
// arithmetic of pointnet2_modules.py:140-142.
//
// three_nn semantics (the spec): scan the known points in index order, keep the three smallest d2 with
// a strict '<' cascade (earlier index wins ties).  The reference holds the bests as doubles initialised
// to 1e40 and compares the fp32 distance against them; every fp32 value converts exactly, so an fp32
// cascade initialised to +inf takes the same branches and (float)1e40 == +inf is what it stores when
// fewer than three points exist.
#include <math_constants.h>
#include <stdint.h>

#include "rev_index.cuh"

namespace prb {

constexpr int NN_THREADS = 256;
constexpr int NN_UPT = 2;        // unknown points per thread
constexpr int NN_TILE = 1024;    // known points per shared tile

__global__ void __launch_bounds__(NN_THREADS) three_nn_kernel(int n, int m, const float *__restrict__ unknown,
                                                              const float *__restrict__ known, float *__restrict__ dist2,
                                                              int *__restrict__ idx, float *__restrict__ weight) {
    __shared__ float4 sk[NN_TILE];
    const int scene = blockIdx.y;
    const int u0 = (blockIdx.x * NN_THREADS + threadIdx.x) * NN_UPT;
    const float *kn = known + (size_t)scene * m * 3;
    float ux[NN_UPT], uy[NN_UPT], uz[NN_UPT], b1[NN_UPT], b2[NN_UPT], b3[NN_UPT];
    int i1[NN_UPT], i2[NN_UPT], i3[NN_UPT];
#pragma unroll
    for (int u = 0; u < NN_UPT; ++u) {
        int ui = min(u0 + u, n - 1);
        const float *q = unknown + ((size_t)scene * n + ui) * 3;
        ux[u] = q[0]; uy[u] = q[1]; uz[u] = q[2];
        b1[u] = b2[u] = b3[u] = CUDART_INF_F;
        i1[u] = i2[u] = i3[u] = 0;
    }
    for (int t0 = 0; t0 < m; t0 += NN_TILE) {
        const int tn = min(NN_TILE, m - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < tn; i += NN_THREADS)
            sk[i] = make_float4(kn[(size_t)(t0 + i) * 3], kn[(size_t)(t0 + i) * 3 + 1], kn[(size_t)(t0 + i) * 3 + 2], 0.f);
        __syncthreads();
#pragma unroll 4
        for (int i = 0; i < tn; ++i) {
            const float4 k = sk[i];
#pragma unroll
            for (int u = 0; u < NN_UPT; ++u) {
                const float d = dist2_ref(ux[u] - k.x, uy[u] - k.y, uz[u] - k.z);
                if (d < b3[u]) {
                    const int kk = t0 + i;
                    if (d < b1[u]) {
                        b3[u] = b2[u]; i3[u] = i2[u];
                        b2[u] = b1[u]; i2[u] = i1[u];
                        b1[u] = d; i1[u] = kk;
                    } else if (d < b2[u]) {
                        b3[u] = b2[u]; i3[u] = i2[u];
                        b2[u] = d; i2[u] = kk;
                    } else {
                        b3[u] = d; i3[u] = kk;
                    }
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < NN_UPT; ++u) {
        if (u0 + u >= n) continue;
        const size_t o = ((size_t)scene * n + u0 + u) * 3;
        dist2[o] = b1[u]; dist2[o + 1] = b2[u]; dist2[o + 2] = b3[u];
        idx[o] = i1[u]; idx[o + 1] = i2[u]; idx[o + 2] = i3[u];
        if (weight) {
            // dist = sqrt(d2); r = 1/(dist + 1e-8); w = r / (r0 + r1 + r2)   (torch fp32 elementwise ops,
            // torch.sum over 3 elements accumulates left to right)
            const float r0 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(b1[u]), 1e-8f));
            const float r1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(b2[u]), 1e-8f));
            const float r2 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(b3[u]), 1e-8f));
            const float norm = __fadd_rn(__fadd_rn(r0, r1), r2);
            weight[o] = __fdiv_rn(r0, norm); weight[o + 1] = __fdiv_rn(r1, norm); weight[o + 2] = __fdiv_rn(r2, norm);
        }
    }
}

// out[b,c,j] = w0*p[c,i0] + w1*p[c,i1] + w2*p[c,i2]; one CTA owns a block of channels of one scene
// (rows stay L1-resident); reference contraction (its SASS): FMUL(w1,p1) -> FFMA(w0,p0,.) -> FFMA(w2,p2,.)
constexpr int TI_THREADS = 256;
constexpr int TI_CH = 8;

__global__ void __launch_bounds__(TI_THREADS) three_interpolate_kernel(int c, int m, int n, const float *__restrict__ points,
                                                                       const int *__restrict__ idx, const float *__restrict__ weight,
                                                                       float *__restrict__ out) {
    const int scene = blockIdx.z, cb = blockIdx.y * TI_CH;
    const int nch = min(TI_CH, c - cb);
    const float *src = points + ((size_t)scene * c + cb) * m;
    float *dst = out + ((size_t)scene * c + cb) * n;
    for (int j = blockIdx.x * TI_THREADS + threadIdx.x; j < n; j += gridDim.x * TI_THREADS) {
        const size_t o = ((size_t)scene * n + j) * 3;
        const int k0 = idx[o], k1 = idx[o + 1], k2 = idx[o + 2];
        const float w0 = weight[o], w1 = weight[o + 1], w2 = weight[o + 2];
#pragma unroll
        for (int ch = 0; ch < TI_CH; ++ch)
            if (ch < nch) {
                const float *row = src + (size_t)ch * m;
                dst[(size_t)ch * n + j] =
                    __fmaf_rn(w2, __ldg(row + k2), __fmaf_rn(w0, __ldg(row + k0), __fmul_rn(w1, __ldg(row + k1))));
            }
    }
}

__global__ void __launch_bounds__(TI_THREADS) three_interpolate_grad_kernel(int c, int n, int m, const float *__restrict__ grad_out,
                                                                            const int *__restrict__ idx, const float *__restrict__ weight,
                                                                            float *__restrict__ grad_points) {
    const int scene = blockIdx.z, cb = blockIdx.y * TI_CH;
    const int nch = min(TI_CH, c - cb);
    const float *g = grad_out + ((size_t)scene * c + cb) * n;
    float *dst = grad_points + ((size_t)scene * c + cb) * m;
    for (int j = blockIdx.x * TI_THREADS + threadIdx.x; j < n; j += gridDim.x * TI_THREADS) {
        const size_t o = ((size_t)scene * n + j) * 3;
        const int k0 = idx[o], k1 = idx[o + 1], k2 = idx[o + 2];
        const float w0 = weight[o], w1 = weight[o + 1], w2 = weight[o + 2];
#pragma unroll
        for (int ch = 0; ch < TI_CH; ++ch)
            if (ch < nch) {
                const float gv = g[(size_t)ch * n + j];
                float *row = dst + (size_t)ch * m;
                atomicAdd(row + k0, gv * w0);
                atomicAdd(row + k1, gv * w1);
                atomicAdd(row + k2, gv * w2);
            }
    }
}

// bfloat16 interpolation: the fp32 kernel's arithmetic on the exactly converted values, rounded once to bfloat16.  Each
// thread computes V consecutive output points of its channel block; V = 8 reads their taps and weights as 16-byte loads and
// writes each channel's 8 values as one 16-byte store (the launcher picks it when n is a multiple of 8 and idx / weight / out
// are 16-byte aligned).
template <int V>
__global__ void __launch_bounds__(TI_THREADS) three_interpolate_bf16_kernel(int c, int m, int n, const __nv_bfloat16 *__restrict__ points,
                                                                            const int *__restrict__ idx, const float *__restrict__ weight,
                                                                            __nv_bfloat16 *__restrict__ out) {
    const int scene = blockIdx.z, cb = blockIdx.y * TI_CH;
    const int nch = min(TI_CH, c - cb);
    const __nv_bfloat16 *src = points + ((size_t)scene * c + cb) * m;
    __nv_bfloat16 *dst = out + ((size_t)scene * c + cb) * n;
    for (int j = (blockIdx.x * TI_THREADS + threadIdx.x) * V; j < n; j += gridDim.x * TI_THREADS * V) {
        const size_t o = ((size_t)scene * n + j) * 3;
        int k[3 * V];
        float w[3 * V];
        if constexpr (V == 8) {
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                const int4 a = reinterpret_cast<const int4 *>(idx + o)[i];
                const float4 b = reinterpret_cast<const float4 *>(weight + o)[i];
                k[4 * i] = a.x; k[4 * i + 1] = a.y; k[4 * i + 2] = a.z; k[4 * i + 3] = a.w;
                w[4 * i] = b.x; w[4 * i + 1] = b.y; w[4 * i + 2] = b.z; w[4 * i + 3] = b.w;
            }
        } else {
#pragma unroll
            for (int t = 0; t < 3; ++t) { k[t] = idx[o + t]; w[t] = weight[o + t]; }
        }
#pragma unroll
        for (int ch = 0; ch < TI_CH; ++ch) {
            if (ch >= nch) continue;
            const __nv_bfloat16 *row = src + (size_t)ch * m;
            __align__(16) __nv_bfloat16 v[V];
#pragma unroll
            for (int i = 0; i < V; ++i) {
                const float p0 = __bfloat162float(__ldg(row + k[3 * i])), p1 = __bfloat162float(__ldg(row + k[3 * i + 1])),
                            p2 = __bfloat162float(__ldg(row + k[3 * i + 2]));
                v[i] = __float2bfloat16_rn(__fmaf_rn(w[3 * i + 2], p2, __fmaf_rn(w[3 * i], p0, __fmul_rn(w[3 * i + 1], p1))));
            }
            if constexpr (V == 8)
                *reinterpret_cast<uint4 *>(dst + (size_t)ch * n + j) = *reinterpret_cast<const uint4 *>(v);
            else
                dst[(size_t)ch * n + j] = v[0];
        }
    }
}

// the atomic bfloat16 gradient, first pass: the fp32 kernel's products and float atomics into fp32 sums (b, c, m)
__global__ void __launch_bounds__(TI_THREADS) three_interpolate_grad_bf16_kernel(int c, int n, int m, const __nv_bfloat16 *__restrict__ grad_out,
                                                                                 const int *__restrict__ idx, const float *__restrict__ weight,
                                                                                 float *__restrict__ sums) {
    const int scene = blockIdx.z, cb = blockIdx.y * TI_CH;
    const int nch = min(TI_CH, c - cb);
    const __nv_bfloat16 *g = grad_out + ((size_t)scene * c + cb) * n;
    float *dst = sums + ((size_t)scene * c + cb) * m;
    for (int j = blockIdx.x * TI_THREADS + threadIdx.x; j < n; j += gridDim.x * TI_THREADS) {
        const size_t o = ((size_t)scene * n + j) * 3;
        const int k0 = idx[o], k1 = idx[o + 1], k2 = idx[o + 2];
        const float w0 = weight[o], w1 = weight[o + 1], w2 = weight[o + 2];
#pragma unroll
        for (int ch = 0; ch < TI_CH; ++ch)
            if (ch < nch) {
                const float gv = __bfloat162float(g[(size_t)ch * n + j]);
                float *row = dst + (size_t)ch * m;
                atomicAdd(row + k0, __fmul_rn(gv, w0));
                atomicAdd(row + k1, __fmul_rn(gv, w1));
                atomicAdd(row + k2, __fmul_rn(gv, w2));
            }
    }
}

}  // namespace prb

using namespace prb;

extern "C" int prb_three_nn(int b, int n, int m, const float *unknown, const float *known, float *dist2, int *idx,
                            float *weight, void *stream) {
    PRB_REQUIRE(b >= 0 && n >= 0 && m >= 0 && unknown && known && dist2 && idx, "three_nn: bad arguments");
    if (b == 0 || n == 0) return 0;
    dim3 grid(ceil_div(n, NN_THREADS * NN_UPT), b);
    three_nn_kernel<<<grid, NN_THREADS, 0, (cudaStream_t)stream>>>(n, m, unknown, known, dist2, idx, weight);
    return check_launch("three_nn_kernel");
}

extern "C" int prb_three_interpolate(int b, int c, int m, int n, const float *points, const int *idx,
                                     const float *weight, float *out, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && m > 0 && n >= 0 && points && idx && weight && out, "three_interpolate: bad arguments");
    if (b == 0 || c == 0 || n == 0) return 0;
    dim3 grid(min(ceil_div(n, TI_THREADS), 64), ceil_div(c, TI_CH), b);
    three_interpolate_kernel<<<grid, TI_THREADS, 0, (cudaStream_t)stream>>>(c, m, n, points, idx, weight, out);
    return check_launch("three_interpolate_kernel");
}

extern "C" int prb_three_interpolate_grad(int b, int c, int n, int m, const float *grad_out, const int *idx,
                                          const float *weight, float *grad_points, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && m > 0 && n >= 0 && grad_out && idx && weight && grad_points,
                "three_interpolate_grad: bad arguments");
    if (b == 0 || c == 0 || n == 0) return 0;
    dim3 grid(min(ceil_div(n, TI_THREADS), 64), ceil_div(c, TI_CH), b);
    three_interpolate_grad_kernel<<<grid, TI_THREADS, 0, (cudaStream_t)stream>>>(c, n, m, grad_out, idx, weight, grad_points);
    return check_launch("three_interpolate_grad_kernel");
}

// the ordered gradient: grad_points[b, c, k] += the sum of grad_out * weight over the taps q = 3 i + t naming known point k,
// in increasing q, through the reverse index of idx (rev_index.cuh)
extern "C" size_t prb_three_interpolate_grad_workspace_bytes(int b, int n, int m) {
    if (b <= 0 || n <= 0 || m <= 0 || !rev_index_fits(b, 3L * n, m)) return 0;
    return rev_index_bytes(b, 3 * n, m);
}

extern "C" int prb_three_interpolate_grad_ws(int b, int c, int n, int m, const float *grad_out, const int *idx, const float *weight,
                                             float *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n >= 0 && m >= 0, "three_interpolate_grad_ws: bad dimensions");
    if (b == 0 || c == 0 || n == 0 || m == 0) return 0;
    PRB_REQUIRE(rev_index_fits(b, 3L * n, m), "three_interpolate_grad_ws: %d x %d rows over %d points", b, n, m);
    PRB_REQUIRE(grad_out && idx && weight && grad_points && workspace, "three_interpolate_grad_ws: bad arguments");
    const size_t need = rev_index_bytes(b, 3 * n, m);
    PRB_REQUIRE(workspace_bytes >= need, "three_interpolate_grad_ws: workspace of %zu bytes < %zu", workspace_bytes, need);
    const RevIndex R = rev_index_at(b, 3 * n, m, workspace);
    const cudaStream_t s = (cudaStream_t)stream;
    if (int rc = rev_index_build(R, idx, s)) return rc;
    return seg_sum(R, SEG_TAPS, c, grad_out, weight, true, grad_points, s);
}

// ------------------------------------------------------------------ bfloat16 interpolation (include/pointrcnn_b200.h)
extern "C" int prb_three_interpolate_bf16(int b, int c, int m, int n, const uint16_t *points, const int *idx, const float *weight,
                                          uint16_t *out, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && m > 0 && n >= 0 && points && idx && weight && out, "three_interpolate_bf16: bad arguments");
    if (b == 0 || c == 0 || n == 0) return 0;
    const auto *p = reinterpret_cast<const __nv_bfloat16 *>(points);
    auto *o = reinterpret_cast<__nv_bfloat16 *>(out);
    const cudaStream_t s = (cudaStream_t)stream;
    if (n % 8 == 0 && (((uintptr_t)idx | (uintptr_t)weight | (uintptr_t)out) & 15) == 0) {
        dim3 grid(min(ceil_div(n / 8, TI_THREADS), 64), ceil_div(c, TI_CH), b);
        three_interpolate_bf16_kernel<8><<<grid, TI_THREADS, 0, s>>>(c, m, n, p, idx, weight, o);
        return check_launch("three_interpolate_bf16_kernel<8>");
    }
    dim3 grid(min(ceil_div(n, TI_THREADS), 64), ceil_div(c, TI_CH), b);
    three_interpolate_bf16_kernel<1><<<grid, TI_THREADS, 0, s>>>(c, m, n, p, idx, weight, o);
    return check_launch("three_interpolate_bf16_kernel<1>");
}

extern "C" size_t prb_three_interpolate_grad_bf16_workspace_bytes(int b, int c, int m) {
    if (b <= 0 || c <= 0 || m <= 0) return 0;
    return (size_t)b * c * m * sizeof(float);
}

extern "C" int prb_three_interpolate_grad_bf16(int b, int c, int n, int m, const uint16_t *grad_out, const int *idx, const float *weight,
                                               uint16_t *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && m > 0 && n >= 0, "three_interpolate_grad_bf16: bad dimensions");
    if (b == 0 || c == 0) return 0;
    PRB_REQUIRE(grad_out && idx && weight && grad_points && workspace, "three_interpolate_grad_bf16: bad arguments");
    const size_t need = prb_three_interpolate_grad_bf16_workspace_bytes(b, c, m);
    PRB_REQUIRE(workspace_bytes >= need, "three_interpolate_grad_bf16: workspace of %zu bytes < %zu", workspace_bytes, need);
    const cudaStream_t s = (cudaStream_t)stream;
    float *sums = static_cast<float *>(workspace);
    PRB_CUDA(cudaMemsetAsync(sums, 0, need, s));
    if (n > 0) {
        dim3 grid(min(ceil_div(n, TI_THREADS), 64), ceil_div(c, TI_CH), b);
        three_interpolate_grad_bf16_kernel<<<grid, TI_THREADS, 0, s>>>(c, n, m, reinterpret_cast<const __nv_bfloat16 *>(grad_out), idx, weight,
                                                                       sums);
        if (int rc = check_launch("three_interpolate_grad_bf16_kernel")) return rc;
    }
    return round_bf16((size_t)b * c * m, sums, grad_points, s);
}

extern "C" int prb_three_interpolate_grad_bf16_ws(int b, int c, int n, int m, const uint16_t *grad_out, const int *idx, const float *weight,
                                                  uint16_t *grad_points, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && c >= 0 && n >= 0 && m >= 0, "three_interpolate_grad_bf16_ws: bad dimensions");
    if (b == 0 || c == 0 || m == 0) return 0;
    PRB_REQUIRE(grad_points, "three_interpolate_grad_bf16_ws: bad arguments");
    const cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) {   // no tap: every sum is +0
        PRB_CUDA(cudaMemsetAsync(grad_points, 0, (size_t)b * c * m * sizeof(uint16_t), s));
        return 0;
    }
    PRB_REQUIRE(rev_index_fits(b, 3L * n, m), "three_interpolate_grad_bf16_ws: %d x %d rows over %d points", b, n, m);
    PRB_REQUIRE(grad_out && idx && weight && workspace, "three_interpolate_grad_bf16_ws: bad arguments");
    const size_t need = rev_index_bytes(b, 3 * n, m);
    PRB_REQUIRE(workspace_bytes >= need, "three_interpolate_grad_bf16_ws: workspace of %zu bytes < %zu", workspace_bytes, need);
    const RevIndex R = rev_index_at(b, 3 * n, m, workspace);
    if (int rc = rev_index_build(R, idx, s)) return rc;
    return seg_sum_bf16(R, SEG_TAPS, c, reinterpret_cast<const __nv_bfloat16 *>(grad_out), weight, reinterpret_cast<__nv_bfloat16 *>(grad_points), s);
}
