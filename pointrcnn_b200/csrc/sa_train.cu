// sa_train.cu -- training-mode forward and backward of one SA scale's grouped SharedMLP + max-pool
// (pointnet2_modules.py: QueryAndGroup(use_xyz) -> [1x1 conv -> BatchNorm2d (batch statistics) | conv + bias -> ReLU] x L ->
// max_pool2d over the samples), for autograd.
//
// Rows are r = (b * npoint + p) * nsample + s; A_0 is the row QueryAndGroup builds, [xyz[idx] - centre | feats_pm[idx]].
// Every layer keeps its pre-activation Z_l = A_l W_l^T (rows x C_l, fp32, bias excluded) and a per-channel affine (a, b)
// with y_l = relu(a * Z_l + b): BN a = gamma * invstd, b = beta - mean * a; no BN a = 1, b = bias.
//   forward   per layer: GEMM (A built on load: the gather for layer 0, relu(a Z + b) of the previous layer otherwise) that
//             stores Z and per-CTA float64 column sums of z and z^2; a finalise launch (mean, biased variance, running
//             statistics, a, b); then one max-pool launch that records the chosen sample of every (group, channel)
//   backward  per layer, last to first: the BN statistics sum(g), sum(g * xhat) (last layer: over the chosen rows only;
//             inner layers: in the epilogue of the GEMM that produced their dA), a finalise launch (dgamma, dbeta / dbias),
//             dA = dZ W (skipped for layer 0 without a feature gradient; layer 0 scatters into d features with atomics),
//             dW = dZ^T A as per-CTA partials over row ranges, reduced in a fixed order
// dZ = a (g - sum(g)/n - xhat sum(g xhat)/n) (no BN: dZ = g) is formed on load.  GEMMs are mma.sync m16n8k8 TF32 with fp32
// accumulation.  No float atomics except the feature scatter: parameter gradients, outputs and running statistics are the
// same bits on every call with the same inputs.
#include <algorithm>

#include "mlp_dev.cuh"

namespace prb {

constexpr int kStMaxC = 512;        // widest layer; also the stride of the per-layer statistics rows
constexpr int kStThreads = 256;
constexpr int kStBK = 32;           // K per shared-memory stage
constexpr int kStRowTile = 128;     // rows per CTA of the row-parallel GEMMs
constexpr int kStColTile = 64;      // output channels per CTA
constexpr int kStWCtas = 528;       // CTAs a weight-gradient GEMM aims for (fixes its row split; never read from the device)
constexpr int kStMaxParts = 1024;   // partial rows of the last layer's statistics pass
// rows of the per-layer statistics block (float, kStMaxC apart)
enum { ST_MEAN, ST_INVSTD, ST_A, ST_B, ST_ROWS };

struct StGeom {
    int b, n, npoint, ns, log_ns, c_feat, rows;
    const float *xyz, *centres, *feats_pm;
    const int *idx;
};

// one layer as the loaders see it
struct StLayer {
    int c;
    const float *z;        // (rows, c)
    const float *st;       // ST_ROWS x kStMaxC
};

// the gradient side of one layer
struct StGrad {
    int c, bn;
    const float *z, *st;
    const float *g;                 // inner layer: (rows, c) dA masked by the ReLU; nullptr: the last layer, read from gout
    const float *gout;              // (b, out_stride_c, npoint)
    const unsigned char *chosen;    // (b * npoint, c)
    int out_stride_c, out_c_off;
    const float *mg;                // 2 x kStMaxC: sum(g) / n, sum(g xhat) / n
};

__device__ __forceinline__ float st_a0(const StGeom &G, int r, int k) {
    if (r >= G.rows || k >= 3 + G.c_feat) return 0.f;
    const int grp = r >> G.log_ns;
    const size_t src = (size_t)(grp / G.npoint) * G.n + G.idx[r];
    if (k < 3) return G.xyz[src * 3 + k] - G.centres[(size_t)grp * 3 + k];
    return G.feats_pm[src * G.c_feat + (k - 3)];
}

// ReLU that passes NaN through, as torch.relu does (fmaxf alone returns 0 for NaN); finite results keep fmaxf's bits
__device__ __forceinline__ float st_relu(float x) { return isnan(x) ? x : fmaxf(x, 0.f); }

__device__ __forceinline__ float st_act(const StGeom &G, const StLayer &P, int r, int k) {
    if (r >= G.rows || k >= P.c) return 0.f;
    return st_relu(fmaf(P.st[ST_A * kStMaxC + k], P.z[(size_t)r * P.c + k], P.st[ST_B * kStMaxC + k]));
}

__device__ __forceinline__ float st_dz(const StGeom &G, const StGrad &L, int r, int c) {
    if (r >= G.rows || c >= L.c) return 0.f;
    const float z = L.z[(size_t)r * L.c + c];
    float g;
    if (L.g) {
        g = L.g[(size_t)r * L.c + c];
    } else {
        const int grp = r >> G.log_ns;
        g = 0.f;
        if ((int)L.chosen[(size_t)grp * L.c + c] == (r & (G.ns - 1)) &&
            fmaf(L.st[ST_A * kStMaxC + c], z, L.st[ST_B * kStMaxC + c]) > 0.f) {
            const int bb = grp / G.npoint, p = grp - bb * G.npoint;
            g = L.gout[((size_t)bb * L.out_stride_c + L.out_c_off + c) * G.npoint + p];
        }
    }
    if (!L.bn) return g;
    const float xhat = (z - L.st[ST_MEAN * kStMaxC + c]) * L.st[ST_INVSTD * kStMaxC + c];
    return L.st[ST_A * kStMaxC + c] * (g - L.mg[c] - xhat * L.mg[kStMaxC + c]);
}

// ------------------------------------------------------------------------------------------------ tensor-core tile
// BM x BN outputs per CTA, 8 warps of 32 x (BN / WN).  Operands live in shared memory in the orientation they are read
// from global memory: A as [m][k] (A_KMAJ = false) or [k][m], B as [n][k] (B_KMAJ = false) or [k][n]; the paddings make
// every fragment load conflict-free.
template <int BM, int BN, bool A_KMAJ, bool B_KMAJ>
struct StTile {
    static constexpr int WM = BM / 32, WN = 8 / WM, WNC = BN / WN, NI = WNC / 8;
    static constexpr int SA = A_KMAJ ? BM + 8 : kStBK + 4;
    static constexpr int SB = B_KMAJ ? BN + 8 : kStBK + 4;
    static constexpr int A_FLOATS = (A_KMAJ ? kStBK : BM) * SA;
    static constexpr int B_FLOATS = (B_KMAJ ? kStBK : BN) * SB;

    __device__ static float a(const float *s, int m, int k) { return A_KMAJ ? s[k * SA + m] : s[m * SA + k]; }
    __device__ static float b(const float *s, int k, int n) { return B_KMAJ ? s[k * SB + n] : s[n * SB + k]; }

    __device__ static void mma(const float *sA, const float *sB, float (&acc)[2][NI][4]) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const int g = lane >> 2, t = lane & 3;
        const int m0 = (warp % WM) * 32, n0 = (warp / WM) * WNC;
#pragma unroll
        for (int kk = 0; kk < kStBK; kk += 8) {
            uint32_t af[2][4], bf[NI][2];
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                const int m = m0 + mi * 16 + g;
                af[mi][0] = __float_as_uint(a(sA, m, kk + t));
                af[mi][1] = __float_as_uint(a(sA, m + 8, kk + t));
                af[mi][2] = __float_as_uint(a(sA, m, kk + t + 4));
                af[mi][3] = __float_as_uint(a(sA, m + 8, kk + t + 4));
            }
#pragma unroll
            for (int ni = 0; ni < NI; ++ni) {
                const int n = n0 + ni * 8 + g;
                bf[ni][0] = __float_as_uint(b(sB, kk + t, n));
                bf[ni][1] = __float_as_uint(b(sB, kk + t + 4, n));
            }
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int ni = 0; ni < NI; ++ni)
                    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                                 "{%0,%1,%2,%3};"
                                 : "+f"(acc[mi][ni][0]), "+f"(acc[mi][ni][1]), "+f"(acc[mi][ni][2]), "+f"(acc[mi][ni][3])
                                 : "r"(af[mi][0]), "r"(af[mi][1]), "r"(af[mi][2]), "r"(af[mi][3]), "r"(bf[ni][0]), "r"(bf[ni][1]));
        }
    }

    // (local row, local column) of accumulator element e of fragment (mi, ni)
    __device__ static int row(int mi, int e) { return ((threadIdx.x >> 5) % WM) * 32 + mi * 16 + ((threadIdx.x & 31) >> 2) + (e >> 1) * 8; }
    __device__ static int col(int ni, int e) { return ((threadIdx.x >> 5) / WM) * WNC + ni * 8 + (threadIdx.x & 3) * 2 + (e & 1); }
};

// s[row * stride + col] = tf32(f(row, col)) for an SR x SC tile; a warp covers 32 consecutive columns of one source row
template <int SR, int SC, typename F>
__device__ __forceinline__ void st_fill(float *s, int stride, F f) {
    static_assert((SR * SC) % kStThreads == 0, "tile");
#pragma unroll
    for (int i = 0; i < SR * SC / kStThreads; ++i) {
        const int e = threadIdx.x + i * kStThreads, r = e / SC, c = e % SC;
        s[r * stride + c] = to_tf32(f(r, c));
    }
}

// per-column float64 sums of v and v * w over the CTA's rows, in a fixed order, into part[c * T + tile]
template <class Tl>
__device__ __forceinline__ void st_col_sums(const double (&s1)[Tl::NI][2], const double (&s2)[Tl::NI][2], double (*red)[2][64],
                                            int n0, int c_lim, int T, int tile, double *p1, double *p2) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int ni = 0; ni < Tl::NI; ++ni)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            double a = s1[ni][j], b = s2[ni][j];
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                a += __shfl_xor_sync(0xffffffffu, a, o);
                b += __shfl_xor_sync(0xffffffffu, b, o);
            }
            if (lane < 4) {
                const int c = Tl::col(ni, j);
                red[warp % Tl::WM][0][c] = a;
                red[warp % Tl::WM][1][c] = b;
            }
        }
    __syncthreads();
    if (threadIdx.x < 64 && n0 + (int)threadIdx.x < c_lim) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int w = 0; w < Tl::WM; ++w) {
            a += red[w][0][threadIdx.x];
            b += red[w][1][threadIdx.x];
        }
        p1[(size_t)(n0 + threadIdx.x) * T + tile] = a;
        p2[(size_t)(n0 + threadIdx.x) * T + tile] = b;
    }
}

using StRowsTile = StTile<kStRowTile, kStColTile, false, false>;   // forward: A [row][k], B = W [n][k]
using StDaTile = StTile<kStRowTile, kStColTile, false, true>;      // dA: A = dZ [row][k], B = W [k][n]
using StDwTile = StTile<64, 64, true, true>;                       // dW: A = dZ [row][m], B = A_l [row][n]

// Z_l = A_l W_l^T; with BN also the column sums of z and z^2 of this row tile
template <bool L0>
__global__ void __launch_bounds__(kStThreads) sa_train_fwd_gemm(StGeom G, StLayer P, const float *__restrict__ W, int cin, int cout,
                                                                float *__restrict__ z, int bn, int T, double *p1, double *p2) {
    using Tl = StRowsTile;
    __shared__ __align__(16) float sA[Tl::A_FLOATS];
    __shared__ __align__(16) float sB[Tl::B_FLOATS];
    __shared__ double red[Tl::WM][2][64];
    const int r0 = blockIdx.x * kStRowTile, n0 = blockIdx.y * kStColTile;
    float acc[2][Tl::NI][4] = {};
    for (int k0 = 0; k0 < cin; k0 += kStBK) {
        st_fill<kStRowTile, kStBK>(sA, Tl::SA, [&](int r, int k) { return L0 ? st_a0(G, r0 + r, k0 + k) : st_act(G, P, r0 + r, k0 + k); });
        st_fill<kStColTile, kStBK>(sB, Tl::SB, [&](int n, int k) {
            return (n0 + n < cout && k0 + k < cin) ? W[(size_t)(n0 + n) * cin + k0 + k] : 0.f;
        });
        __syncthreads();
        Tl::mma(sA, sB, acc);
        __syncthreads();
    }
    double s1[Tl::NI][2] = {}, s2[Tl::NI][2] = {};
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < Tl::NI; ++ni)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = r0 + Tl::row(mi, e), c = n0 + Tl::col(ni, e);
                const float v = acc[mi][ni][e];          // rows past the end read zeros: v == 0
                if (r < G.rows && c < cout) z[(size_t)r * cout + c] = v;
                s1[ni][e & 1] += (double)v;
                s2[ni][e & 1] += (double)v * (double)v;
            }
    if (bn) st_col_sums<Tl>(s1, s2, red, n0, cout, T, blockIdx.x, p1, p2);
}

// per channel: the partials in a fixed order -> mean / invstd / a / b; running statistics as BatchNorm2d.train() updates them
__global__ void __launch_bounds__(kStThreads) sa_train_bn_finalise(int T, const double *p1, const double *p2, long n, int bn, double eps,
                                                                   double momentum, const float *gamma, const float *beta, const float *bias,
                                                                   float *rmean, float *rvar, long long *nbt, float *st) {
    __shared__ double s[2][kStThreads];
    const int c = blockIdx.x;
    if (!bn) {
        if (threadIdx.x == 0) {
            st[ST_MEAN * kStMaxC + c] = 0.f;
            st[ST_INVSTD * kStMaxC + c] = 1.f;
            st[ST_A * kStMaxC + c] = 1.f;
            st[ST_B * kStMaxC + c] = bias ? bias[c] : 0.f;
        }
        return;
    }
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < T; i += kStThreads) {
        a += p1[(size_t)c * T + i];
        b += p2[(size_t)c * T + i];
    }
    s[0][threadIdx.x] = a;
    s[1][threadIdx.x] = b;
    __syncthreads();
    for (int o = kStThreads / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            s[0][threadIdx.x] += s[0][threadIdx.x + o];
            s[1][threadIdx.x] += s[1][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double mean = s[0][0] / n;
        // clamp the cancellation below zero only: a NaN variance stays NaN, as in torch
        double var = s[1][0] / n - mean * mean;
        if (var < 0.0) var = 0.0;
        const double invstd = 1.0 / sqrt(var + eps);
        const double ga = gamma ? gamma[c] : 1.0, be = beta ? beta[c] : 0.0;
        st[ST_MEAN * kStMaxC + c] = (float)mean;
        st[ST_INVSTD * kStMaxC + c] = (float)invstd;
        st[ST_A * kStMaxC + c] = (float)(ga * invstd);
        st[ST_B * kStMaxC + c] = (float)(be - mean * ga * invstd);
        if (rmean) rmean[c] = (float)((1.0 - momentum) * rmean[c] + momentum * mean);
        if (rvar) rvar[c] = (float)((1.0 - momentum) * rvar[c] + momentum * var * ((double)n / (double)(n - 1)));
        if (nbt && c == 0) *nbt += 1;
    }
}

// y = relu(max_s (a z + b)) per (group, channel) -> out (b, out_stride_c, npoint) and out_pm (b, npoint, out_stride_c) at
// out_c_off; the first maximal sample is recorded.  A NaN sample wins, as in ATen's max-pool (the last NaN is recorded);
// the backward's "a z + b > 0" test then drops its gradient, as torch's ReLU backward does.
__global__ void __launch_bounds__(kStThreads) sa_train_pool(StGeom G, StLayer L, float *out, float *out_pm, int out_stride_c, int out_c_off,
                                                            unsigned char *chosen) {
    const long e = (long)blockIdx.x * kStThreads + threadIdx.x;
    const long groups = (long)G.b * G.npoint;
    if (e >= groups * L.c) return;
    const int grp = (int)(e / L.c), c = (int)(e - (long)grp * L.c);
    const float a = L.st[ST_A * kStMaxC + c], b = L.st[ST_B * kStMaxC + c];
    const float *z = L.z + (size_t)grp * G.ns * L.c + c;
    float best = fmaf(a, z[0], b);
    int arg = 0;
    for (int s = 1; s < G.ns; ++s) {
        const float v = fmaf(a, z[(size_t)s * L.c], b);
        if (v > best || isnan(v)) {
            best = v;
            arg = s;
        }
    }
    const float y = st_relu(best);
    const int bb = grp / G.npoint, p = grp - bb * G.npoint;
    out[((size_t)bb * out_stride_c + out_c_off + c) * G.npoint + p] = y;
    if (out_pm) out_pm[(size_t)grp * out_stride_c + out_c_off + c] = y;
    chosen[e] = (unsigned char)arg;
}

// the last layer's BN backward sums over the chosen rows: part[c * P + blockIdx.x]
__global__ void __launch_bounds__(kStThreads) sa_train_last_stats(StGeom G, StGrad L, int groups_per_part, double *p1, double *p2) {
    const int P = gridDim.x, groups = G.b * G.npoint;
    const int g0 = blockIdx.x * groups_per_part, g1 = min(groups, g0 + groups_per_part);
    for (int c = threadIdx.x; c < L.c; c += kStThreads) {
        const float a = L.st[ST_A * kStMaxC + c], b = L.st[ST_B * kStMaxC + c];
        const float mean = L.st[ST_MEAN * kStMaxC + c], invstd = L.st[ST_INVSTD * kStMaxC + c];
        double s1 = 0.0, s2 = 0.0;
        for (int grp = g0; grp < g1; ++grp) {
            const int r = grp * G.ns + L.chosen[(size_t)grp * L.c + c];
            const float z = L.z[(size_t)r * L.c + c];
            if (fmaf(a, z, b) > 0.f) {
                const int bb = grp / G.npoint, p = grp - bb * G.npoint;
                const float g = L.gout[((size_t)bb * L.out_stride_c + L.out_c_off + c) * G.npoint + p];
                s1 += g;
                s2 += (double)g * (double)((z - mean) * invstd);
            }
        }
        p1[(size_t)c * P + blockIdx.x] = s1;
        p2[(size_t)c * P + blockIdx.x] = s2;
    }
}

// per channel: sum(g), sum(g xhat) in a fixed order -> dgamma, dbeta (BN) or dbias, and the two means dZ reads
__global__ void __launch_bounds__(kStThreads) sa_train_grad_finalise(int T, const double *p1, const double *p2, long n, int bn, float *dgamma,
                                                                     float *dbeta, float *dbias, float *mg) {
    __shared__ double s[2][kStThreads];
    const int c = blockIdx.x;
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < T; i += kStThreads) {
        a += p1[(size_t)c * T + i];
        b += p2[(size_t)c * T + i];
    }
    s[0][threadIdx.x] = a;
    s[1][threadIdx.x] = b;
    __syncthreads();
    for (int o = kStThreads / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            s[0][threadIdx.x] += s[0][threadIdx.x + o];
            s[1][threadIdx.x] += s[1][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (bn) {
            if (dgamma) dgamma[c] = (float)s[1][0];
            if (dbeta) dbeta[c] = (float)s[0][0];
        } else if (dbias) {
            dbias[c] = (float)s[0][0];
        }
        mg[c] = (float)(s[0][0] / n);
        mg[kStMaxC + c] = (float)(s[1][0] / n);
    }
}

// dA_l = dZ_l W_l.  TO_FEATS (layer 0): the feature columns are scattered into grad_feats (b, c_feat, n).  Otherwise the
// result is masked by the previous layer's ReLU and stored as its g, with that layer's BN sums of g and g xhat.
template <bool TO_FEATS>
__global__ void __launch_bounds__(kStThreads) sa_train_da_gemm(StGeom G, StGrad L, const float *__restrict__ W, int cin, StLayer P,
                                                               float *__restrict__ gprev, int T, double *p1, double *p2, float *grad_feats) {
    using Tl = StDaTile;
    __shared__ __align__(16) float sA[Tl::A_FLOATS];
    __shared__ __align__(16) float sB[Tl::B_FLOATS];
    __shared__ double red[Tl::WM][2][64];
    const int r0 = blockIdx.x * kStRowTile, n0 = blockIdx.y * kStColTile;
    float acc[2][Tl::NI][4] = {};
    for (int k0 = 0; k0 < L.c; k0 += kStBK) {
        st_fill<kStRowTile, kStBK>(sA, Tl::SA, [&](int r, int k) { return st_dz(G, L, r0 + r, k0 + k); });
        st_fill<kStBK, kStColTile>(sB, Tl::SB, [&](int k, int n) {
            return (k0 + k < L.c && n0 + n < cin) ? W[(size_t)(k0 + k) * cin + n0 + n] : 0.f;
        });
        __syncthreads();
        Tl::mma(sA, sB, acc);
        __syncthreads();
    }
    double s1[Tl::NI][2] = {}, s2[Tl::NI][2] = {};
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < Tl::NI; ++ni)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = r0 + Tl::row(mi, e), c = n0 + Tl::col(ni, e);
                if (r >= G.rows || c >= cin) continue;
                const float v = acc[mi][ni][e];
                if (TO_FEATS) {
                    if (c >= 3) {
                        const int bb = (r >> G.log_ns) / G.npoint;
                        atomicAdd(grad_feats + ((size_t)bb * G.c_feat + (c - 3)) * G.n + G.idx[r], v);
                    }
                } else {
                    const float zp = P.z[(size_t)r * cin + c];
                    const float g = fmaf(P.st[ST_A * kStMaxC + c], zp, P.st[ST_B * kStMaxC + c]) > 0.f ? v : 0.f;
                    gprev[(size_t)r * cin + c] = g;
                    s1[ni][e & 1] += (double)g;
                    s2[ni][e & 1] += (double)g * (double)((zp - P.st[ST_MEAN * kStMaxC + c]) * P.st[ST_INVSTD * kStMaxC + c]);
                }
            }
    if (!TO_FEATS) st_col_sums<Tl>(s1, s2, red, n0, cin, T, blockIdx.x, p1, p2);
}

// partial dW_l = dZ_l^T A_l over the rows [blockIdx.z * chunk, +chunk) -> part[blockIdx.z][cout][cin]
template <bool L0>
__global__ void __launch_bounds__(kStThreads) sa_train_dw_gemm(StGeom G, StGrad L, StLayer P, int cin, int chunk, float *__restrict__ part) {
    using Tl = StDwTile;
    __shared__ __align__(16) float sA[Tl::A_FLOATS];
    __shared__ __align__(16) float sB[Tl::B_FLOATS];
    const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
    const int q0 = blockIdx.z * chunk, q1 = min(G.rows, q0 + chunk);
    float acc[2][Tl::NI][4] = {};
    for (int k0 = q0; k0 < q1; k0 += kStBK) {
        st_fill<kStBK, 64>(sA, Tl::SA, [&](int k, int m) { return k0 + k < q1 ? st_dz(G, L, k0 + k, m0 + m) : 0.f; });
        st_fill<kStBK, 64>(sB, Tl::SB, [&](int k, int n) {
            if (k0 + k >= q1) return 0.f;
            return L0 ? st_a0(G, k0 + k, n0 + n) : st_act(G, P, k0 + k, n0 + n);
        });
        __syncthreads();
        Tl::mma(sA, sB, acc);
        __syncthreads();
    }
    float *o = part + (size_t)blockIdx.z * L.c * cin;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < Tl::NI; ++ni)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = m0 + Tl::row(mi, e), n = n0 + Tl::col(ni, e);
                if (m < L.c && n < cin) o[(size_t)m * cin + n] = acc[mi][ni][e];
            }
}

__global__ void __launch_bounds__(kStThreads) sa_train_dw_reduce(int parts, int count, const float *part, float *dw) {
    const int e = blockIdx.x * kStThreads + threadIdx.x;
    if (e >= count) return;
    double s = 0.0;
    for (int p = 0; p < parts; ++p) s += part[(size_t)p * count + e];
    dw[e] = (float)s;
}

// ------------------------------------------------------------------------------------------------ host side
struct StPlan {
    int L, cin[3], cout[3];
    long rows;
    int T;                 // row tiles of the row-parallel GEMMs
    int P, gpp;            // parts / groups per part of the last layer's statistics pass
    int wparts[3], wchunk[3];
    size_t off_p1, off_p2, off_mg, off_wpart, off_g0, off_g1;
    size_t fwd_total, total;   // the forward reads only the statistics partials; the backward the whole layout
};

inline size_t st_align(size_t x) { return (x + 255) & ~(size_t)255; }

int st_plan(const prb_sa_train_desc *d, int b, int npoint, int ns, int c_feat, StPlan &p) {
    PRB_REQUIRE(d, "sa_train: NULL descriptor");
    PRB_REQUIRE(d->num_layers >= 1 && d->num_layers <= 3, "sa_train: %d layers (1..3)", d->num_layers);
    PRB_REQUIRE(b >= 1 && npoint >= 1 && ns >= 1 && ns <= 128 && (ns & (ns - 1)) == 0, "sa_train: nsample %d must be a power of two <= 128", ns);
    PRB_REQUIRE(c_feat >= 0 && d->c_in == 3 + c_feat, "sa_train: layer 0 reads %d channels, the rows have 3 + %d", d->c_in, c_feat);
    const long rows = (long)b * npoint * ns;
    PRB_REQUIRE(rows < (1L << 30), "sa_train: %ld rows", rows);
    p.L = d->num_layers;
    p.rows = rows;
    int cmax = 0, cinner = 0;
    for (int l = 0; l < p.L; ++l) {
        p.cin[l] = l ? d->c_out[l - 1] : d->c_in;
        p.cout[l] = d->c_out[l];
        PRB_REQUIRE(p.cout[l] >= 1 && p.cout[l] <= kStMaxC, "sa_train: layer %d has %d channels (1..%d)", l, p.cout[l], kStMaxC);
        PRB_REQUIRE(p.cin[l] <= kStMaxC + 3, "sa_train: layer %d reads %d channels", l, p.cin[l]);
        cmax = max(cmax, p.cout[l]);
        if (l + 1 < p.L) cinner = max(cinner, p.cout[l]);
    }
    p.T = ceil_div((int)rows, kStRowTile);
    const int groups = b * npoint;
    p.P = min(max(ceil_div(groups, 32), 1), kStMaxParts);
    p.gpp = ceil_div(groups, p.P);
    p.P = ceil_div(groups, p.gpp);
    size_t wpart = 0;
    for (int l = 0; l < p.L; ++l) {
        const int tiles = ceil_div(p.cout[l], 64) * ceil_div(p.cin[l], 64);
        int parts = min(ceil_div(kStWCtas, tiles), ceil_div((int)rows, 256));
        parts = max(parts, 1);
        p.wchunk[l] = ceil_div(ceil_div((int)rows, parts), kStBK) * kStBK;
        p.wparts[l] = ceil_div((int)rows, p.wchunk[l]);
        wpart = std::max(wpart, (size_t)p.wparts[l] * p.cout[l] * p.cin[l]);
    }
    const size_t nparts = (size_t)cmax * max(p.T, p.P);
    p.off_p1 = 0;
    p.off_p2 = st_align(p.off_p1 + nparts * sizeof(double));
    p.off_mg = st_align(p.off_p2 + nparts * sizeof(double));
    p.fwd_total = p.off_mg;
    p.off_wpart = st_align(p.off_mg + 2 * kStMaxC * sizeof(float));
    p.off_g0 = st_align(p.off_wpart + wpart * sizeof(float));
    p.off_g1 = st_align(p.off_g0 + (size_t)rows * cinner * sizeof(float));
    p.total = st_align(p.off_g1 + (size_t)rows * cinner * sizeof(float));
    return 0;
}

StGeom st_geom(int b, int n, int npoint, int ns, int c_feat, long rows, const float *xyz, const float *new_xyz, const float *feats_pm,
               const int *idx) {
    StGeom G;
    G.b = b; G.n = n; G.npoint = npoint; G.ns = ns; G.c_feat = c_feat; G.rows = (int)rows;
    G.log_ns = 0;
    while ((1 << G.log_ns) < ns) ++G.log_ns;
    G.xyz = xyz; G.centres = new_xyz; G.feats_pm = feats_pm; G.idx = idx;
    return G;
}

}  // namespace prb

using namespace prb;

extern "C" size_t prb_sa_train_workspace_bytes(int b, int npoint, int nsample, int c_feat, const prb_sa_train_desc *desc, int backward) {
    StPlan p;
    if (st_plan(desc, b, npoint, nsample, c_feat, p)) return 0;
    return backward ? p.total : p.fwd_total;
}

extern "C" int prb_sa_train_forward(const prb_sa_train_desc *desc, int b, int n, int npoint, int nsample, int c_feat, const float *xyz,
                                    const float *new_xyz, const float *feats_pm, const int *idx, float *const *z, float *stats,
                                    unsigned char *chosen, float *out, float *out_pm, int out_stride_c, int out_c_off, void *workspace,
                                    size_t workspace_bytes, void *stream) {
    StPlan p;
    if (int rc = st_plan(desc, b, npoint, nsample, c_feat, p)) return rc;
    PRB_REQUIRE(xyz && new_xyz && idx && z && stats && chosen && out && (c_feat == 0 || feats_pm) && workspace, "sa_train_forward: bad arguments");
    PRB_REQUIRE(workspace_bytes >= p.fwd_total, "sa_train_forward: workspace of %zu bytes < %zu", workspace_bytes, p.fwd_total);
    PRB_REQUIRE(out_c_off >= 0 && out_c_off + p.cout[p.L - 1] <= out_stride_c, "sa_train_forward: channels %d..%d outside %d", out_c_off,
                out_c_off + p.cout[p.L - 1], out_stride_c);
    PRB_REQUIRE(!desc->bn || p.rows > 1, "sa_train_forward: batch statistics need more than one value per channel");
    const cudaStream_t s = (cudaStream_t)stream;
    char *ws = reinterpret_cast<char *>(workspace);
    double *p1 = reinterpret_cast<double *>(ws + p.off_p1), *p2 = reinterpret_cast<double *>(ws + p.off_p2);
    const StGeom G = st_geom(b, n, npoint, nsample, c_feat, p.rows, xyz, new_xyz, feats_pm, idx);
    StLayer prev{0, nullptr, nullptr};
    for (int l = 0; l < p.L; ++l) {
        PRB_REQUIRE(z[l] && desc->weight[l], "sa_train_forward: layer %d: no Z buffer or weight", l);
        const dim3 grid(p.T, ceil_div(p.cout[l], kStColTile));
        if (l == 0)
            sa_train_fwd_gemm<true><<<grid, kStThreads, 0, s>>>(G, prev, desc->weight[l], p.cin[l], p.cout[l], z[l], desc->bn, p.T, p1, p2);
        else
            sa_train_fwd_gemm<false><<<grid, kStThreads, 0, s>>>(G, prev, desc->weight[l], p.cin[l], p.cout[l], z[l], desc->bn, p.T, p1, p2);
        if (int rc = check_launch("sa_train_fwd_gemm")) return rc;
        float *st = stats + (size_t)l * ST_ROWS * kStMaxC;
        sa_train_bn_finalise<<<p.cout[l], kStThreads, 0, s>>>(p.T, p1, p2, p.rows, desc->bn, desc->eps, desc->momentum, desc->gamma[l],
                                                              desc->beta[l], desc->bias[l], desc->running_mean[l], desc->running_var[l],
                                                              desc->num_batches_tracked[l], st);
        if (int rc = check_launch("sa_train_bn_finalise")) return rc;
        prev = StLayer{p.cout[l], z[l], st};
    }
    const long items = (long)b * npoint * prev.c;
    sa_train_pool<<<(unsigned)((items + kStThreads - 1) / kStThreads), kStThreads, 0, s>>>(G, prev, out, out_pm, out_stride_c, out_c_off, chosen);
    return check_launch("sa_train_pool");
}

extern "C" int prb_sa_train_backward(const prb_sa_train_desc *desc, int b, int n, int npoint, int nsample, int c_feat, const float *xyz,
                                     const float *new_xyz, const float *feats_pm, const int *idx, const float *const *z,
                                     const float *stats, const unsigned char *chosen, const float *grad_out, int out_stride_c,
                                     int out_c_off, float *const *grad_weight, float *const *grad_bias, float *const *grad_gamma,
                                     float *const *grad_beta, float *grad_feats, void *workspace, size_t workspace_bytes, void *stream) {
    StPlan p;
    if (int rc = st_plan(desc, b, npoint, nsample, c_feat, p)) return rc;
    PRB_REQUIRE(xyz && new_xyz && idx && z && stats && chosen && grad_out && grad_weight && (c_feat == 0 || feats_pm) && workspace,
                "sa_train_backward: bad arguments");
    PRB_REQUIRE(workspace_bytes >= p.total, "sa_train_backward: workspace of %zu bytes < %zu", workspace_bytes, p.total);
    PRB_REQUIRE(out_c_off >= 0 && out_c_off + p.cout[p.L - 1] <= out_stride_c, "sa_train_backward: channels %d..%d outside %d", out_c_off,
                out_c_off + p.cout[p.L - 1], out_stride_c);
    const cudaStream_t s = (cudaStream_t)stream;
    char *ws = reinterpret_cast<char *>(workspace);
    double *p1 = reinterpret_cast<double *>(ws + p.off_p1), *p2 = reinterpret_cast<double *>(ws + p.off_p2);
    float *mg = reinterpret_cast<float *>(ws + p.off_mg), *wpart = reinterpret_cast<float *>(ws + p.off_wpart);
    float *gbuf[2] = {reinterpret_cast<float *>(ws + p.off_g0), reinterpret_cast<float *>(ws + p.off_g1)};
    const StGeom G = st_geom(b, n, npoint, nsample, c_feat, p.rows, xyz, new_xyz, feats_pm, idx);
    const float *g_in = nullptr;      // g of the current layer (nullptr: the last layer, from grad_out)
    int nparts = p.P;                 // partial rows of the current layer's statistics
    for (int l = p.L - 1; l >= 0; --l) {
        const float *st = stats + (size_t)l * ST_ROWS * kStMaxC;
        const StGrad Lg{p.cout[l], desc->bn, z[l], st, g_in, grad_out, chosen, out_stride_c, out_c_off, mg};
        if (l == p.L - 1) {
            sa_train_last_stats<<<p.P, kStThreads, 0, s>>>(G, Lg, p.gpp, p1, p2);
            if (int rc = check_launch("sa_train_last_stats")) return rc;
        }
        sa_train_grad_finalise<<<p.cout[l], kStThreads, 0, s>>>(nparts, p1, p2, p.rows, desc->bn, grad_gamma ? grad_gamma[l] : nullptr,
                                                                grad_beta ? grad_beta[l] : nullptr, grad_bias ? grad_bias[l] : nullptr, mg);
        if (int rc = check_launch("sa_train_grad_finalise")) return rc;
        // dW first: it reads this layer's g, which the dA launch below does not overwrite (it writes the other buffer)
        const StLayer prev = l ? StLayer{p.cout[l - 1], z[l - 1], stats + (size_t)(l - 1) * ST_ROWS * kStMaxC} : StLayer{0, nullptr, nullptr};
        const dim3 wgrid(ceil_div(p.cout[l], 64), ceil_div(p.cin[l], 64), p.wparts[l]);
        if (l == 0)
            sa_train_dw_gemm<true><<<wgrid, kStThreads, 0, s>>>(G, Lg, prev, p.cin[l], p.wchunk[l], wpart);
        else
            sa_train_dw_gemm<false><<<wgrid, kStThreads, 0, s>>>(G, Lg, prev, p.cin[l], p.wchunk[l], wpart);
        if (int rc = check_launch("sa_train_dw_gemm")) return rc;
        PRB_REQUIRE(grad_weight[l], "sa_train_backward: layer %d: no weight gradient", l);
        const int count = p.cout[l] * p.cin[l];
        sa_train_dw_reduce<<<ceil_div(count, kStThreads), kStThreads, 0, s>>>(p.wparts[l], count, wpart, grad_weight[l]);
        if (int rc = check_launch("sa_train_dw_reduce")) return rc;
        const dim3 agrid(p.T, ceil_div(p.cin[l], kStColTile));
        if (l > 0) {
            float *g_out = gbuf[(l - 1) & 1];
            sa_train_da_gemm<false><<<agrid, kStThreads, 0, s>>>(G, Lg, desc->weight[l], p.cin[l], prev, g_out, p.T, p1, p2, nullptr);
            if (int rc = check_launch("sa_train_da_gemm")) return rc;
            g_in = g_out;
            nparts = p.T;
        } else if (grad_feats && c_feat > 0) {
            sa_train_da_gemm<true><<<agrid, kStThreads, 0, s>>>(G, Lg, desc->weight[0], p.cin[0], prev, nullptr, p.T, nullptr, nullptr,
                                                                 grad_feats);
            if (int rc = check_launch("sa_train_da_gemm")) return rc;
        }
    }
    return 0;
}
