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
//             dA = dZ W (skipped for layer 0 without a feature gradient; layer 0 scatters into d features with atomics, or in
//             the ordered backward stages them for a per-point sum over the reverse index of idx),
//             dW = dZ^T A as per-CTA partials over row ranges, reduced in a fixed order
// dZ = a (g - sum(g)/n - xhat sum(g xhat)/n) (no BN: dZ = g) is formed on load.  GEMMs are mma.sync m16n8k8 TF32 with fp32
// accumulation.  No float atomics except the feature scatter of prb_sa_train_backward: parameter gradients, outputs and
// running statistics are the same bits on every call with the same inputs, and so is the feature gradient of
// prb_sa_train_backward_det, which stages layer 0's feature columns and sums them per point over a reverse index of idx.
#include <algorithm>

#include "mlp_dev.cuh"
#include "rev_index.cuh"

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

__device__ __forceinline__ float st_act(int rows, const StLayer &P, int r, int k) {
    if (r >= rows || k >= P.c) return 0.f;
    return st_relu(fmaf(P.st[ST_A * kStMaxC + k], P.z[(size_t)r * P.c + k], P.st[ST_B * kStMaxC + k]));
}

// dZ from g (the upstream gradient of y, ReLU mask applied) and the pre-activation z
__device__ __forceinline__ float st_dz_bn(const StGrad &L, int c, float z, float g) {
    if (!L.bn) return g;
    const float xhat = (z - L.st[ST_MEAN * kStMaxC + c]) * L.st[ST_INVSTD * kStMaxC + c];
    return L.st[ST_A * kStMaxC + c] * (g - L.mg[c] - xhat * L.mg[kStMaxC + c]);
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
    return st_dz_bn(L, c, z, g);
}

// ------------------------------------------------------------------------------------------------ row sources
// The GEMM kernels stage their row operands through one of these: s(r, k) is row r, column k, and 0 outside the operand.
struct SaA0Src {      // SA layer 0: the grouped row
    StGeom G;
    __device__ float operator()(int r, int k) const { return st_a0(G, r, k); }
};
struct ActSrc {       // relu(a Z + b) of a layer
    int rows;
    StLayer P;
    __device__ float operator()(int r, int k) const { return st_act(rows, P, r, k); }
};
struct SaDzSrc {      // SA dZ; the last layer's g comes through the pooled choice
    StGeom G;
    StGrad L;
    __device__ float operator()(int r, int c) const { return st_dz(G, L, r, c); }
};
struct DzSrc {        // dZ of a layer whose g is materialised (rows, c)
    int rows;
    StGrad L;
    __device__ float operator()(int r, int c) const {
        if (r >= rows || c >= L.c) return 0.f;
        const size_t e = (size_t)r * L.c + c;
        return st_dz_bn(L, c, L.z[e], L.g[e]);
    }
};
struct MatSrc {       // a dense row-major matrix
    int rows, cols, ld;
    const float *p;
    __device__ float operator()(int r, int k) const { return (r < rows && k < cols) ? p[(size_t)r * ld + k] : 0.f; }
};

// FP module: unknown row r = b * n + i takes three taps idx[r][t] (known points of its scene) with weights w[r][t]
struct FpGeom {
    int rows, n, m, ci, cs;
    const int *idx;
    const float *w;
    const float *known_pm;    // (b, m, ci)
    const float *skip;        // (b, cs, n)
};

// sum_t w_t x[b * m + idx_t][k] for row-major x of width ld, in three_interpolate's order
__device__ __forceinline__ float fp_taps(const FpGeom &F, int r, const float *x, int ld, int k) {
    const int *id = F.idx + (size_t)r * 3;
    const float *w = F.w + (size_t)r * 3;
    const float *base = x + (size_t)(r / F.n) * F.m * ld + k;
    return fmaf(w[2], base[(size_t)id[2] * ld], fmaf(w[0], base[(size_t)id[0] * ld], w[1] * base[(size_t)id[1] * ld]));
}

__device__ __forceinline__ float fp_skip(const FpGeom &F, int r, int k) {
    const int b = r / F.n;
    return F.skip[((size_t)b * F.cs + k) * F.n + (r - b * F.n)];
}

struct FpSkipSrc {    // FP skip columns alone
    FpGeom F;
    __device__ float operator()(int r, int k) const { return (r < F.rows && k < F.cs) ? fp_skip(F, r, k) : 0.f; }
};

// what the forward GEMM adds to its accumulator before storing Z
struct NoAdd {
    static constexpr bool kOn = false;
    __device__ float operator()(int, int) const { return 0.f; }
};
struct FpTapAdd {     // FP layer 0: the three-tap sum of the projected known rows (b * m, c1)
    static constexpr bool kOn = true;
    FpGeom F;
    const float *proj;
    int c1;
    __device__ float operator()(int r, int c) const { return fp_taps(F, r, proj, c1, c); }
};

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

// Z_l = A_l W_l^T (+ add(r, c)); with BN also the column sums of z and z^2 of this row tile.  W is (cout, cin) with row
// pitch ldw (a column block of a wider weight).
template <class Src, class Add>
__global__ void __launch_bounds__(kStThreads) sa_train_fwd_gemm(Src A, Add add, int rows, const float *__restrict__ W, int ldw, int cin,
                                                                int cout, float *__restrict__ z, int bn, int T, double *p1, double *p2) {
    using Tl = StRowsTile;
    __shared__ __align__(16) float sA[Tl::A_FLOATS];
    __shared__ __align__(16) float sB[Tl::B_FLOATS];
    __shared__ double red[Tl::WM][2][64];
    const int r0 = blockIdx.x * kStRowTile, n0 = blockIdx.y * kStColTile;
    float acc[2][Tl::NI][4] = {};
    for (int k0 = 0; k0 < cin; k0 += kStBK) {
        st_fill<kStRowTile, kStBK>(sA, Tl::SA, [&](int r, int k) { return A(r0 + r, k0 + k); });
        st_fill<kStColTile, kStBK>(sB, Tl::SB, [&](int n, int k) {
            return (n0 + n < cout && k0 + k < cin) ? W[(size_t)(n0 + n) * ldw + k0 + k] : 0.f;
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
                float v = acc[mi][ni][e];                // rows past the end read zeros: v == 0
                if constexpr (Add::kOn) {
                    if (r < rows && c < cout) v += add(r, c);
                }
                if (r < rows && c < cout) z[(size_t)r * cout + c] = v;
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

// what the dA GEMM does with each output element (r, c) = v
struct DaScatterFeats {     // SA layer 0: the feature columns are scattered into grad_feats (b, c_feat, n)
    static constexpr bool kSums = false;
    StGeom G;
    float *grad_feats;
    __device__ void operator()(int r, int c, float v, float &, float &) const {
        if (c >= 3) {
            const int bb = (r >> G.log_ns) / G.npoint;
            atomicAdd(grad_feats + ((size_t)bb * G.c_feat + (c - 3)) * G.n + G.idx[r], v);
        }
    }
};
struct DaStageFeats {       // SA layer 0, ordered: the feature columns are stored (rows, c_feat) for the gather-sum
    static constexpr bool kSums = false;
    int c_feat;
    float *stage;
    __device__ void operator()(int r, int c, float v, float &, float &) const {
        if (c >= 3) stage[(size_t)r * c_feat + (c - 3)] = v;
    }
};
struct DaMasked {           // inner layer: masked by the previous layer's ReLU, stored as its g; g and xhat feed its BN sums
    static constexpr bool kSums = true;
    StLayer P;
    float *gprev;
    __device__ void operator()(int r, int c, float v, float &g, float &xhat) const {
        const float zp = P.z[(size_t)r * P.c + c];
        g = fmaf(P.st[ST_A * kStMaxC + c], zp, P.st[ST_B * kStMaxC + c]) > 0.f ? v : 0.f;
        gprev[(size_t)r * P.c + c] = g;
        xhat = (zp - P.st[ST_MEAN * kStMaxC + c]) * P.st[ST_INVSTD * kStMaxC + c];
    }
};
struct DaChannelMajor {     // FP input gradients: row r = b * n + i of a (b, c, n) tensor
    static constexpr bool kSums = false;
    float *out;
    int n, c;
    __device__ void operator()(int r, int k, float v, float &, float &) const {
        const int b = r / n;
        out[((size_t)b * c + k) * n + (r - b * n)] = v;
    }
};

// dA = dZ W for dZ (rows, K) staged through A and W (K, cin) with row pitch ldw; epi consumes the result
template <class Src, class Epi>
__global__ void __launch_bounds__(kStThreads) sa_train_da_gemm(Src A, Epi epi, int rows, int K, const float *__restrict__ W, int ldw, int cin,
                                                               int T, double *p1, double *p2) {
    using Tl = StDaTile;
    __shared__ __align__(16) float sA[Tl::A_FLOATS];
    __shared__ __align__(16) float sB[Tl::B_FLOATS];
    __shared__ double red[Tl::WM][2][64];
    const int r0 = blockIdx.x * kStRowTile, n0 = blockIdx.y * kStColTile;
    float acc[2][Tl::NI][4] = {};
    for (int k0 = 0; k0 < K; k0 += kStBK) {
        st_fill<kStRowTile, kStBK>(sA, Tl::SA, [&](int r, int k) { return A(r0 + r, k0 + k); });
        st_fill<kStBK, kStColTile>(sB, Tl::SB, [&](int k, int n) {
            return (k0 + k < K && n0 + n < cin) ? W[(size_t)(k0 + k) * ldw + n0 + n] : 0.f;
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
                if (r >= rows || c >= cin) continue;
                float g, xhat;
                epi(r, c, acc[mi][ni][e], g, xhat);
                if constexpr (Epi::kSums) {
                    s1[ni][e & 1] += (double)g;
                    s2[ni][e & 1] += (double)g * (double)xhat;
                }
            }
    if constexpr (Epi::kSums) st_col_sums<Tl>(s1, s2, red, n0, cin, T, blockIdx.x, p1, p2);
}

// partial dW = dZ^T A over the rows [blockIdx.z * chunk, +chunk) -> part[blockIdx.z][cout][cin]; dZ (rows, cout) staged
// through D, A (rows, cin) through S
template <class SrcD, class SrcA>
__global__ void __launch_bounds__(kStThreads) sa_train_dw_gemm(SrcD D, SrcA S, int rows, int cout, int cin, int chunk,
                                                               float *__restrict__ part) {
    using Tl = StDwTile;
    __shared__ __align__(16) float sA[Tl::A_FLOATS];
    __shared__ __align__(16) float sB[Tl::B_FLOATS];
    const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
    const int q0 = blockIdx.z * chunk, q1 = min(rows, q0 + chunk);
    float acc[2][Tl::NI][4] = {};
    for (int k0 = q0; k0 < q1; k0 += kStBK) {
        st_fill<kStBK, 64>(sA, Tl::SA, [&](int k, int m) { return k0 + k < q1 ? D(k0 + k, m0 + m) : 0.f; });
        st_fill<kStBK, 64>(sB, Tl::SB, [&](int k, int n) { return k0 + k < q1 ? S(k0 + k, n0 + n) : 0.f; });
        __syncthreads();
        Tl::mma(sA, sB, acc);
        __syncthreads();
    }
    float *o = part + (size_t)blockIdx.z * cout * cin;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < Tl::NI; ++ni)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = m0 + Tl::row(mi, e), n = n0 + Tl::col(ni, e);
                if (m < cout && n < cin) o[(size_t)m * cin + n] = acc[mi][ni][e];
            }
}

// dw[m * ld + n] = the partials [parts][cout][ncol] summed in part order (count = cout * ncol)
__global__ void __launch_bounds__(kStThreads) sa_train_dw_reduce(int parts, int count, int ncol, int ld, const float *part, float *dw) {
    const int e = blockIdx.x * kStThreads + threadIdx.x;
    if (e >= count) return;
    double s = 0.0;
    for (int p = 0; p < parts; ++p) s += part[(size_t)p * count + e];
    dw[(size_t)(e / ncol) * ld + e % ncol] = (float)s;
}

// ------------------------------------------------------------------------------------------------ FP module
// Training-mode forward and backward of one PointnetFPModule's three_interpolate + cat + SharedMLP (no pool), rows
// r = b * n + i.  The inner layers are the SA kernels above with the row sources ActSrc / DzSrc.  Layer 0 reads
// [I F | S] with I the (rows x b m) three-tap interpolation, F the known features (point-major), S the skip features
// (channel-major); W_0 = [Wi | Ws].
//   forward  P = F Wi^T over the b m known rows, then Z_0 = S Ws^T + (three-tap sum of P) in one GEMM that also writes the
//            BN column sums
//   backward G = I^T dZ_0 from a reverse index of the taps (no float atomics), then dWi = G^T F, dF = G Wi,
//            dWs = dZ_0^T S, dS = dZ_0 Ws
// y_L = relu(a Z_L + b) -> out (b, c, n) and optionally its point-major twin (b, n, c), through a 32 x 32 tile
__global__ void __launch_bounds__(kStThreads) fp_train_out(int rows, int n, StLayer L, float *out, float *out_pm) {
    __shared__ float t[32][33];
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int i = ty; i < 32; i += kStThreads / 32) {
        const int r = r0 + i, c = c0 + tx;
        if (r < rows && c < L.c) {
            const float y = st_act(rows, L, r, c);
            t[i][tx] = y;
            if (out_pm) out_pm[(size_t)r * L.c + c] = y;
        }
    }
    __syncthreads();
    for (int i = ty; i < 32; i += kStThreads / 32) {
        const int c = c0 + i, r = r0 + tx;
        if (r < rows && c < L.c) {
            const int b = r / n;
            out[((size_t)b * L.c + c) * n + (r - b * n)] = t[tx][i];
        }
    }
}

// the last layer: g = grad_out (b, c, n) where a z + b > 0, stored (rows, c) for the GEMMs, and the BN sums of g and
// g xhat over each 128-row tile, in row order -> part[c * gridDim.x + blockIdx.x]
__global__ void __launch_bounds__(kStThreads) fp_train_last_grad(int rows, int n, StGrad L, float *g, double *p1, double *p2) {
    __shared__ float sg[32][kStRowTile + 1], sx[32][kStRowTile + 1];
    const int r0 = blockIdx.x * kStRowTile, c0 = blockIdx.y * 32;
    for (int e = threadIdx.x; e < 32 * kStRowTile; e += kStThreads) {
        const int cl = e / kStRowTile, rl = e % kStRowTile, r = r0 + rl, c = c0 + cl;
        float v = 0.f;
        if (r < rows && c < L.c) {
            const int b = r / n;
            v = L.gout[((size_t)b * L.c + c) * n + (r - b * n)];
        }
        sg[cl][rl] = v;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 32 * kStRowTile; e += kStThreads) {
        const int rl = e / 32, cl = e % 32, r = r0 + rl, c = c0 + cl;
        float v = 0.f, xhat = 0.f;
        if (r < rows && c < L.c) {
            const float z = L.z[(size_t)r * L.c + c];
            v = fmaf(L.st[ST_A * kStMaxC + c], z, L.st[ST_B * kStMaxC + c]) > 0.f ? sg[cl][rl] : 0.f;
            xhat = (z - L.st[ST_MEAN * kStMaxC + c]) * L.st[ST_INVSTD * kStMaxC + c];
            g[(size_t)r * L.c + c] = v;
        }
        sg[cl][rl] = v;
        sx[cl][rl] = xhat;
    }
    __syncthreads();
    const int c = c0 + (int)threadIdx.x;
    if (threadIdx.x < 32 && c < L.c) {
        double s1 = 0.0, s2 = 0.0;
        for (int rl = 0; rl < kStRowTile; ++rl) {
            s1 += (double)sg[threadIdx.x][rl];
            s2 += (double)sg[threadIdx.x][rl] * (double)sx[threadIdx.x][rl];
        }
        p1[(size_t)c * gridDim.x + blockIdx.x] = s1;
        p2[(size_t)c * gridDim.x + blockIdx.x] = s2;
    }
}

// G = I^T dZ_0 (b m, c1): per known point the sum over its references in list order, one warp per point
__global__ void __launch_bounds__(kStThreads) fp_train_gather_g(int K, const int *off, const int *list, const float *w, DzSrc D, float *G) {
    const int j = blockIdx.x * (kStThreads / 32) + (threadIdx.x >> 5);
    if (j >= K) return;
    const int e0 = off[j], e1 = off[j + 1];
    for (int c = threadIdx.x & 31; c < D.L.c; c += 32) {
        float acc = 0.f;
        for (int e = e0; e < e1; ++e) {
            const int q = list[e];
            acc = fmaf(w[q], D(q / 3, c), acc);
        }
        G[(size_t)j * D.L.c + c] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ host side
// row split of a weight-gradient GEMM over `rows` rows: about kStWCtas CTAs, chunks a multiple of kStBK
inline void st_wsplit(int rows, int cout, int cin, int &chunk, int &parts) {
    const int tiles = ceil_div(cout, 64) * ceil_div(cin, 64);
    parts = max(min(ceil_div(kStWCtas, tiles), ceil_div(rows, 256)), 1);
    chunk = ceil_div(ceil_div(rows, parts), kStBK) * kStBK;
    parts = ceil_div(rows, chunk);
}

// the offset of `bytes` placed at `at`; `at` moves past them to the next 256-byte boundary
inline size_t st_take(size_t &at, size_t bytes) {
    const size_t off = at;
    at = (at + bytes + 255) & ~(size_t)255;
    return off;
}

template <class T>
T *st_at(void *ws, size_t off) { return reinterpret_cast<T *>(static_cast<char *>(ws) + off); }

// The layer stack of an SA scale or an FP module: its widths, the row tiles and weight-gradient row splits of the layer
// GEMMs, and the workspace both modules lay out.  The forward reads only the statistics partials and the module's own
// forward scratch after them (fwd_total); the backward the whole layout.
struct StackPlan {
    int L, cin[3], cout[3];
    int rows, T;                  // rows of the layer GEMMs, their row tiles
    int wparts[3], wchunk[3];     // dW row splits over those rows (FP: index 0 is Ws's)
    size_t off_p1, off_p2, off_mg, off_wpart, off_g0, off_g1;
    size_t fwd_total, total;
    // the gradient buffer g of layer l (every layer but SA's last)
    float *g(void *ws, int l) const { return st_at<float>(ws, l & 1 ? off_g1 : off_g0); }
};

// The descriptor checks both modules share (1..3 layers, each 1..kStMaxC channels), the widths, and the row tiles and
// dW row splits of layers 1.. over `rows` rows; layer 0's split is the module's.
int st_stack(const prb_sa_train_desc *d, const char *who, int rows, StackPlan &p) {
    PRB_REQUIRE(d, "%s: NULL descriptor", who);
    PRB_REQUIRE(d->num_layers >= 1 && d->num_layers <= 3, "%s: %d layers (1..3)", who, d->num_layers);
    p.L = d->num_layers;
    p.rows = rows;
    p.T = ceil_div(rows, kStRowTile);
    for (int l = 0; l < p.L; ++l) {
        p.cin[l] = l ? d->c_out[l - 1] : d->c_in;
        p.cout[l] = d->c_out[l];
        PRB_REQUIRE(p.cout[l] >= 1 && p.cout[l] <= kStMaxC, "%s: layer %d has %d channels (1..%d)", who, l, p.cout[l], kStMaxC);
        if (l) st_wsplit(rows, p.cout[l], p.cin[l], p.wchunk[l], p.wparts[l]);
    }
    return 0;
}

// The shared layout: the statistics partials p1 / p2 (nparts float64 each), then `fwd_extra` bytes of the module's forward
// scratch at the returned offset; for the backward mg, the dW partials (the largest of layer 0's wpart0 floats and those of
// layers 1..) and the gradient buffers g0 / g1 of rows x gw floats each.
size_t st_layout(StackPlan &p, size_t nparts, size_t fwd_extra, size_t wpart0, int gw) {
    size_t wpart = wpart0;
    for (int l = 1; l < p.L; ++l) wpart = std::max(wpart, (size_t)p.wparts[l] * p.cout[l] * p.cin[l]);
    size_t at = 0;
    p.off_p1 = st_take(at, nparts * sizeof(double));
    p.off_p2 = st_take(at, nparts * sizeof(double));
    const size_t off_extra = st_take(at, fwd_extra);
    p.fwd_total = at;
    p.off_mg = st_take(at, 2 * kStMaxC * sizeof(float));
    p.off_wpart = st_take(at, wpart * sizeof(float));
    p.off_g0 = st_take(at, (size_t)p.rows * gw * sizeof(float));
    p.off_g1 = st_take(at, (size_t)p.rows * gw * sizeof(float));
    p.total = at;
    return off_extra;
}

// every layer's Z buffer and weight, and with grad_weight its weight gradient, before an entry launches anything
int st_check_layers(const StackPlan &p, const prb_sa_train_desc *d, const char *who, const float *const *z, float *const *grad_weight) {
    for (int l = 0; l < p.L; ++l) {
        PRB_REQUIRE(z[l] && d->weight[l], "%s: layer %d: no Z buffer or weight", who, l);
        PRB_REQUIRE(!grad_weight || grad_weight[l], "%s: layer %d: no weight gradient", who, l);
    }
    return 0;
}

// The forward's layer loop, once the module's layer-0 GEMM has stored Z_0 and its statistics partials: every layer has its
// statistics finalised, and layers 1.. run the GEMM over relu(a Z + b) of the layer before.  `top` receives the last layer.
int st_forward(const StackPlan &p, const prb_sa_train_desc *d, float *const *z, float *stats, void *ws, cudaStream_t s, StLayer &top) {
    double *p1 = st_at<double>(ws, p.off_p1), *p2 = st_at<double>(ws, p.off_p2);
    for (int l = 0; l < p.L; ++l) {
        if (l > 0) {
            sa_train_fwd_gemm<<<dim3(p.T, ceil_div(p.cout[l], kStColTile)), kStThreads, 0, s>>>(ActSrc{p.rows, top}, NoAdd{}, p.rows, d->weight[l],
                                                                                               p.cin[l], p.cin[l], p.cout[l], z[l], d->bn, p.T, p1, p2);
            if (int rc = check_launch("sa_train_fwd_gemm")) return rc;
        }
        float *st = stats + (size_t)l * ST_ROWS * kStMaxC;
        sa_train_bn_finalise<<<p.cout[l], kStThreads, 0, s>>>(p.T, p1, p2, p.rows, d->bn, d->eps, d->momentum, d->gamma[l], d->beta[l], d->bias[l],
                                                              d->running_mean[l], d->running_var[l], d->num_batches_tracked[l], st);
        if (int rc = check_launch("sa_train_bn_finalise")) return rc;
        top = StLayer{p.cout[l], z[l], st};
    }
    return 0;
}

// The backward's layer loop, last layer to first, once the module has written the last layer's statistics partials
// (nparts_last per channel; T for every other layer).  dz(l) stages layer l's dZ.  Every layer has dgamma / dbeta or dbias
// finalised; layers 1.. then run dW = dZ^T A over the layer before's relu(a Z + b), and dA = dZ W masked by that layer's
// ReLU into its g buffer, with its BN sums.  Layer 0's weight and input gradients are the module's.
template <class Dz>
int st_backward(const StackPlan &p, const prb_sa_train_desc *d, Dz dz, int nparts_last, const float *const *z, const float *stats,
                float *const *grad_weight, float *const *grad_bias, float *const *grad_gamma, float *const *grad_beta, void *ws,
                cudaStream_t s) {
    double *p1 = st_at<double>(ws, p.off_p1), *p2 = st_at<double>(ws, p.off_p2);
    float *mg = st_at<float>(ws, p.off_mg), *wpart = st_at<float>(ws, p.off_wpart);
    for (int l = p.L - 1; l >= 0; --l) {
        sa_train_grad_finalise<<<p.cout[l], kStThreads, 0, s>>>(l == p.L - 1 ? nparts_last : p.T, p1, p2, p.rows, d->bn,
                                                                grad_gamma ? grad_gamma[l] : nullptr, grad_beta ? grad_beta[l] : nullptr,
                                                                grad_bias ? grad_bias[l] : nullptr, mg);
        if (int rc = check_launch("sa_train_grad_finalise")) return rc;
        if (l == 0) break;
        // dW first: it reads this layer's g, which the dA launch below does not overwrite (it writes the other buffer)
        const auto D = dz(l);
        const StLayer prev{p.cout[l - 1], z[l - 1], stats + (size_t)(l - 1) * ST_ROWS * kStMaxC};
        sa_train_dw_gemm<<<dim3(ceil_div(p.cout[l], 64), ceil_div(p.cin[l], 64), p.wparts[l]), kStThreads, 0, s>>>(
            D, ActSrc{p.rows, prev}, p.rows, p.cout[l], p.cin[l], p.wchunk[l], wpart);
        if (int rc = check_launch("sa_train_dw_gemm")) return rc;
        const int count = p.cout[l] * p.cin[l];
        sa_train_dw_reduce<<<ceil_div(count, kStThreads), kStThreads, 0, s>>>(p.wparts[l], count, p.cin[l], p.cin[l], wpart, grad_weight[l]);
        if (int rc = check_launch("sa_train_dw_reduce")) return rc;
        sa_train_da_gemm<<<dim3(p.T, ceil_div(p.cin[l], kStColTile)), kStThreads, 0, s>>>(D, DaMasked{prev, p.g(ws, l - 1)}, p.rows, p.cout[l],
                                                                                          d->weight[l], p.cin[l], p.cin[l], p.T, p1, p2);
        if (int rc = check_launch("sa_train_da_gemm")) return rc;
    }
    return 0;
}

struct StPlan : StackPlan {
    int P, gpp;            // parts / groups per part of the last layer's statistics pass
    size_t off_stage, off_rev, det_total;   // the ordered backward's scratch after `total` (st_det_layout)
};

int st_plan(const prb_sa_train_desc *d, int b, int npoint, int ns, int c_feat, StPlan &p) {
    PRB_REQUIRE(b >= 1 && npoint >= 1 && ns >= 1 && ns <= 128 && (ns & (ns - 1)) == 0, "sa_train: nsample %d must be a power of two <= 128", ns);
    const long rows = (long)b * npoint * ns;
    PRB_REQUIRE(rows < (1L << 30), "sa_train: %ld rows", rows);
    if (int rc = st_stack(d, "sa_train", (int)rows, p)) return rc;
    PRB_REQUIRE(c_feat >= 0 && d->c_in == 3 + c_feat, "sa_train: layer 0 reads %d channels, the rows have 3 + %d", d->c_in, c_feat);
    PRB_REQUIRE(d->c_in <= kStMaxC + 3, "sa_train: layer 0 reads %d channels", d->c_in);
    st_wsplit(p.rows, p.cout[0], p.cin[0], p.wchunk[0], p.wparts[0]);
    const int groups = b * npoint;
    p.P = min(max(ceil_div(groups, 32), 1), kStMaxParts);
    p.gpp = ceil_div(groups, p.P);
    p.P = ceil_div(groups, p.gpp);
    // the partials serve the last layer's statistics pass too; the g buffers only the inner layers
    const int cmax = *std::max_element(p.cout, p.cout + p.L);
    const int cinner = p.L > 1 ? *std::max_element(p.cout, p.cout + p.L - 1) : 0;
    st_layout(p, (size_t)cmax * max(p.T, p.P), 0, (size_t)p.wparts[0] * p.cout[0] * p.cin[0], cinner);
    return 0;
}

// the ordered backward: the staged layer-0 feature gradient (rows, c_feat) and the reverse index of idx over the n points
int st_det_layout(StPlan &p, int b, int n, int npoint, int ns, int c_feat) {
    PRB_REQUIRE(n >= 1 && rev_index_fits(b, (long)npoint * ns, n), "sa_train: %d scenes of %d points", b, n);
    size_t at = p.total;
    p.off_stage = st_take(at, (size_t)p.rows * c_feat * sizeof(float));
    p.off_rev = st_take(at, rev_index_bytes(b, npoint * ns, n));
    p.det_total = at;
    return 0;
}

StGeom st_geom(int b, int n, int npoint, int ns, int c_feat, int rows, const float *xyz, const float *new_xyz, const float *feats_pm,
               const int *idx) {
    StGeom G;
    G.b = b; G.n = n; G.npoint = npoint; G.ns = ns; G.c_feat = c_feat; G.rows = rows;
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
    if (int rc = st_check_layers(p, desc, "sa_train_forward", z, nullptr)) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    double *p1 = st_at<double>(workspace, p.off_p1), *p2 = st_at<double>(workspace, p.off_p2);
    const StGeom G = st_geom(b, n, npoint, nsample, c_feat, p.rows, xyz, new_xyz, feats_pm, idx);
    sa_train_fwd_gemm<<<dim3(p.T, ceil_div(p.cout[0], kStColTile)), kStThreads, 0, s>>>(SaA0Src{G}, NoAdd{}, p.rows, desc->weight[0], p.cin[0],
                                                                                       p.cin[0], p.cout[0], z[0], desc->bn, p.T, p1, p2);
    if (int rc = check_launch("sa_train_fwd_gemm")) return rc;
    StLayer top{};
    if (int rc = st_forward(p, desc, z, stats, workspace, s, top)) return rc;
    const long items = (long)b * npoint * top.c;
    sa_train_pool<<<(unsigned)((items + kStThreads - 1) / kStThreads), kStThreads, 0, s>>>(G, top, out, out_pm, out_stride_c, out_c_off, chosen);
    return check_launch("sa_train_pool");
}

namespace prb {

int sa_train_backward(bool ordered, const prb_sa_train_desc *desc, int b, int n, int npoint, int nsample, int c_feat, const float *xyz,
                      const float *new_xyz, const float *feats_pm, const int *idx, const float *const *z, const float *stats,
                      const unsigned char *chosen, const float *grad_out, int out_stride_c, int out_c_off, float *const *grad_weight,
                      float *const *grad_bias, float *const *grad_gamma, float *const *grad_beta, float *grad_feats, void *workspace,
                      size_t workspace_bytes, void *stream) {
    StPlan p;
    if (int rc = st_plan(desc, b, npoint, nsample, c_feat, p)) return rc;
    if (ordered) {
        if (int rc = st_det_layout(p, b, n, npoint, nsample, c_feat)) return rc;
    }
    const size_t need = ordered ? p.det_total : p.total;
    PRB_REQUIRE(xyz && new_xyz && idx && z && stats && chosen && grad_out && grad_weight && (c_feat == 0 || feats_pm) && workspace,
                "sa_train_backward: bad arguments");
    PRB_REQUIRE(workspace_bytes >= need, "sa_train_backward: workspace of %zu bytes < %zu", workspace_bytes, need);
    PRB_REQUIRE(out_c_off >= 0 && out_c_off + p.cout[p.L - 1] <= out_stride_c, "sa_train_backward: channels %d..%d outside %d", out_c_off,
                out_c_off + p.cout[p.L - 1], out_stride_c);
    if (int rc = st_check_layers(p, desc, "sa_train_backward", z, grad_weight)) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    double *p1 = st_at<double>(workspace, p.off_p1), *p2 = st_at<double>(workspace, p.off_p2);
    float *mg = st_at<float>(workspace, p.off_mg), *wpart = st_at<float>(workspace, p.off_wpart);
    const StGeom G = st_geom(b, n, npoint, nsample, c_feat, p.rows, xyz, new_xyz, feats_pm, idx);
    // the last layer's g comes from grad_out through the pooled choice
    auto dz = [&](int l) {
        return SaDzSrc{G, StGrad{p.cout[l], desc->bn, z[l], stats + (size_t)l * ST_ROWS * kStMaxC, l == p.L - 1 ? nullptr : p.g(workspace, l),
                                 grad_out, chosen, out_stride_c, out_c_off, mg}};
    };
    sa_train_last_stats<<<p.P, kStThreads, 0, s>>>(G, dz(p.L - 1).L, p.gpp, p1, p2);
    if (int rc = check_launch("sa_train_last_stats")) return rc;
    if (int rc = st_backward(p, desc, dz, p.P, z, stats, grad_weight, grad_bias, grad_gamma, grad_beta, workspace, s)) return rc;
    // layer 0: dW over the grouped rows; dA only for the feature columns, scattered into grad_feats (ordered: staged, then
    // summed per point over the reverse index of idx)
    sa_train_dw_gemm<<<dim3(ceil_div(p.cout[0], 64), ceil_div(p.cin[0], 64), p.wparts[0]), kStThreads, 0, s>>>(dz(0), SaA0Src{G}, p.rows, p.cout[0],
                                                                                                            p.cin[0], p.wchunk[0], wpart);
    if (int rc = check_launch("sa_train_dw_gemm")) return rc;
    const int count = p.cout[0] * p.cin[0];
    sa_train_dw_reduce<<<ceil_div(count, kStThreads), kStThreads, 0, s>>>(p.wparts[0], count, p.cin[0], p.cin[0], wpart, grad_weight[0]);
    if (int rc = check_launch("sa_train_dw_reduce")) return rc;
    if (!grad_feats || c_feat == 0) return 0;
    const dim3 grid(p.T, ceil_div(p.cin[0], kStColTile));
    if (!ordered) {
        sa_train_da_gemm<<<grid, kStThreads, 0, s>>>(dz(0), DaScatterFeats{G, grad_feats}, p.rows, p.cout[0], desc->weight[0], p.cin[0], p.cin[0],
                                                     p.T, nullptr, nullptr);
        return check_launch("sa_train_da_gemm");
    }
    float *stage = st_at<float>(workspace, p.off_stage);
    const RevIndex R = rev_index_at(b, npoint * nsample, n, st_at<void>(workspace, p.off_rev));
    if (int rc = rev_index_build(R, idx, s)) return rc;
    sa_train_da_gemm<<<grid, kStThreads, 0, s>>>(dz(0), DaStageFeats{c_feat, stage}, p.rows, p.cout[0], desc->weight[0], p.cin[0], p.cin[0],
                                                 p.T, nullptr, nullptr);
    if (int rc = check_launch("sa_train_da_gemm")) return rc;
    return seg_sum(R, SEG_ROWS, c_feat, stage, nullptr, false, grad_feats, s);
}

}  // namespace prb

extern "C" int prb_sa_train_backward(const prb_sa_train_desc *desc, int b, int n, int npoint, int nsample, int c_feat, const float *xyz,
                                     const float *new_xyz, const float *feats_pm, const int *idx, const float *const *z,
                                     const float *stats, const unsigned char *chosen, const float *grad_out, int out_stride_c,
                                     int out_c_off, float *const *grad_weight, float *const *grad_bias, float *const *grad_gamma,
                                     float *const *grad_beta, float *grad_feats, void *workspace, size_t workspace_bytes, void *stream) {
    return sa_train_backward(false, desc, b, n, npoint, nsample, c_feat, xyz, new_xyz, feats_pm, idx, z, stats, chosen, grad_out, out_stride_c,
                             out_c_off, grad_weight, grad_bias, grad_gamma, grad_beta, grad_feats, workspace, workspace_bytes, stream);
}

extern "C" size_t prb_sa_train_det_workspace_bytes(int b, int n, int npoint, int nsample, int c_feat, const prb_sa_train_desc *desc) {
    StPlan p;
    if (st_plan(desc, b, npoint, nsample, c_feat, p) || st_det_layout(p, b, n, npoint, nsample, c_feat)) return 0;
    return p.det_total;
}

extern "C" int prb_sa_train_backward_det(const prb_sa_train_desc *desc, int b, int n, int npoint, int nsample, int c_feat, const float *xyz,
                                         const float *new_xyz, const float *feats_pm, const int *idx, const float *const *z,
                                         const float *stats, const unsigned char *chosen, const float *grad_out, int out_stride_c,
                                         int out_c_off, float *const *grad_weight, float *const *grad_bias, float *const *grad_gamma,
                                         float *const *grad_beta, float *grad_feats, void *workspace, size_t workspace_bytes, void *stream) {
    return sa_train_backward(true, desc, b, n, npoint, nsample, c_feat, xyz, new_xyz, feats_pm, idx, z, stats, chosen, grad_out, out_stride_c,
                             out_c_off, grad_weight, grad_bias, grad_gamma, grad_beta, grad_feats, workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------------------------------------ FP module, host side
namespace prb {

constexpr int kFpMaxIn = 2048;     // widest layer-0 input (interpolated + skip channels)

struct FpPlan : StackPlan {
    int krows, KT;              // b m known rows, their row tiles
    int wparts_i, wchunk_i;     // dWi over the known rows
    size_t off_proj, off_rev;
};

int fp_plan(const prb_sa_train_desc *d, int b, int n, int m, int ci, int cs, FpPlan &p) {
    PRB_REQUIRE(b >= 1 && n >= 1 && m >= 1, "fp_train: b %d, n %d, m %d", b, n, m);
    PRB_REQUIRE(3L * b * n < (1L << 30) && (long)b * m < (1L << 30), "fp_train: %d x %d rows", b, n);
    if (int rc = st_stack(d, "fp_train", b * n, p)) return rc;
    PRB_REQUIRE(ci >= 1 && cs >= 0 && d->c_in == ci + cs && d->c_in <= kFpMaxIn, "fp_train: layer 0 reads %d channels, not %d + %d (at most %d)",
                d->c_in, ci, cs, kFpMaxIn);
    p.krows = b * m;
    p.KT = ceil_div(p.krows, kStRowTile);
    st_wsplit(p.rows, p.cout[0], max(cs, 1), p.wchunk[0], p.wparts[0]);
    st_wsplit(p.krows, p.cout[0], ci, p.wchunk_i, p.wparts_i);
    const int cmax = *std::max_element(p.cout, p.cout + p.L);
    const size_t wpart0 = std::max((size_t)p.wparts[0] * p.cout[0] * cs, (size_t)p.wparts_i * p.cout[0] * ci);
    // proj: the forward's P = F Wi^T, the backward's G = I^T dZ_0
    p.off_proj = st_layout(p, (size_t)cmax * p.T, (size_t)p.krows * p.cout[0] * sizeof(float), wpart0, cmax);
    size_t at = p.total;
    p.off_rev = st_take(at, rev_index_bytes(b, 3 * n, m));
    p.total = at;
    return 0;
}

}  // namespace prb

extern "C" size_t prb_fp_train_workspace_bytes(int b, int n, int m, int c_interp, int c_skip, const prb_sa_train_desc *desc, int backward) {
    FpPlan p;
    if (fp_plan(desc, b, n, m, c_interp, c_skip, p)) return 0;
    return backward ? p.total : p.fwd_total;
}

extern "C" int prb_fp_train_forward(const prb_sa_train_desc *desc, int b, int n, int m, int c_interp, int c_skip, const int *idx,
                                    const float *weight, const float *known_pm, const float *skip, float *const *z, float *stats, float *out,
                                    float *out_pm, void *workspace, size_t workspace_bytes, void *stream) {
    FpPlan p;
    if (int rc = fp_plan(desc, b, n, m, c_interp, c_skip, p)) return rc;
    PRB_REQUIRE(idx && weight && known_pm && (c_skip == 0 || skip) && z && stats && out && workspace, "fp_train_forward: bad arguments");
    PRB_REQUIRE(workspace_bytes >= p.fwd_total, "fp_train_forward: workspace of %zu bytes < %zu", workspace_bytes, p.fwd_total);
    PRB_REQUIRE(!desc->bn || p.rows > 1, "fp_train_forward: batch statistics need more than one value per channel");
    if (int rc = st_check_layers(p, desc, "fp_train_forward", z, nullptr)) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    double *p1 = st_at<double>(workspace, p.off_p1), *p2 = st_at<double>(workspace, p.off_p2);
    float *proj = st_at<float>(workspace, p.off_proj);
    const FpGeom F{p.rows, n, m, c_interp, c_skip, idx, weight, known_pm, skip};
    const float *W = desc->weight[0];
    const int cols = ceil_div(p.cout[0], kStColTile);
    sa_train_fwd_gemm<<<dim3(p.KT, cols), kStThreads, 0, s>>>(MatSrc{p.krows, c_interp, c_interp, known_pm}, NoAdd{}, p.krows, W, p.cin[0], c_interp,
                                                              p.cout[0], proj, 0, 0, nullptr, nullptr);
    if (int rc = check_launch("sa_train_fwd_gemm")) return rc;
    sa_train_fwd_gemm<<<dim3(p.T, cols), kStThreads, 0, s>>>(FpSkipSrc{F}, FpTapAdd{F, proj, p.cout[0]}, p.rows, W + c_interp, p.cin[0], c_skip,
                                                             p.cout[0], z[0], desc->bn, p.T, p1, p2);
    if (int rc = check_launch("sa_train_fwd_gemm")) return rc;
    StLayer top{};
    if (int rc = st_forward(p, desc, z, stats, workspace, s, top)) return rc;
    fp_train_out<<<dim3(ceil_div(p.rows, 32), ceil_div(top.c, 32)), kStThreads, 0, s>>>(p.rows, n, top, out, out_pm);
    return check_launch("fp_train_out");
}

extern "C" int prb_fp_train_backward(const prb_sa_train_desc *desc, int b, int n, int m, int c_interp, int c_skip, const int *idx,
                                     const float *weight, const float *known_pm, const float *skip, const float *const *z, const float *stats,
                                     const float *grad_out, float *const *grad_weight, float *const *grad_bias, float *const *grad_gamma,
                                     float *const *grad_beta, float *grad_known, float *grad_skip, void *workspace, size_t workspace_bytes,
                                     void *stream) {
    FpPlan p;
    if (int rc = fp_plan(desc, b, n, m, c_interp, c_skip, p)) return rc;
    PRB_REQUIRE(idx && weight && known_pm && (c_skip == 0 || skip) && z && stats && grad_out && grad_weight && workspace,
                "fp_train_backward: bad arguments");
    PRB_REQUIRE(workspace_bytes >= p.total, "fp_train_backward: workspace of %zu bytes < %zu", workspace_bytes, p.total);
    if (int rc = st_check_layers(p, desc, "fp_train_backward", z, grad_weight)) return rc;
    const cudaStream_t s = (cudaStream_t)stream;
    double *p1 = st_at<double>(workspace, p.off_p1), *p2 = st_at<double>(workspace, p.off_p2);
    float *mg = st_at<float>(workspace, p.off_mg), *wpart = st_at<float>(workspace, p.off_wpart);
    float *G = st_at<float>(workspace, p.off_proj);
    const RevIndex R = rev_index_at(b, 3 * n, m, st_at<void>(workspace, p.off_rev));
    const FpGeom F{p.rows, n, m, c_interp, c_skip, idx, weight, known_pm, skip};
    const int last = p.L - 1;

    // the reverse index depends only on the taps: build it first
    if (int rc = rev_index_build(R, idx, s)) return rc;

    const StGrad Lg{p.cout[last], desc->bn, z[last], stats + (size_t)last * ST_ROWS * kStMaxC, nullptr, grad_out, nullptr, p.cout[last], 0, mg};
    fp_train_last_grad<<<dim3(p.T, ceil_div(p.cout[last], 32)), kStThreads, 0, s>>>(p.rows, n, Lg, p.g(workspace, last), p1, p2);
    if (int rc = check_launch("fp_train_last_grad")) return rc;
    auto dz = [&](int l) {
        return DzSrc{p.rows, StGrad{p.cout[l], desc->bn, z[l], stats + (size_t)l * ST_ROWS * kStMaxC, p.g(workspace, l), nullptr, nullptr, p.cout[l],
                                    0, mg}};
    };
    if (int rc = st_backward(p, desc, dz, p.T, z, stats, grad_weight, grad_bias, grad_gamma, grad_beta, workspace, s)) return rc;

    const int c1 = p.cout[0], cin0 = p.cin[0];
    const float *W0 = desc->weight[0];
    const DzSrc D = dz(0);
    fp_train_gather_g<<<ceil_div(p.krows, kStThreads / 32), kStThreads, 0, s>>>(p.krows, R.off, R.list, weight, D, G);
    if (int rc = check_launch("fp_train_gather_g")) return rc;
    const MatSrc Gs{p.krows, c1, c1, G};
    // dWi = G^T F
    sa_train_dw_gemm<<<dim3(ceil_div(c1, 64), ceil_div(c_interp, 64), p.wparts_i), kStThreads, 0, s>>>(
        Gs, MatSrc{p.krows, c_interp, c_interp, known_pm}, p.krows, c1, c_interp, p.wchunk_i, wpart);
    if (int rc = check_launch("sa_train_dw_gemm")) return rc;
    sa_train_dw_reduce<<<ceil_div(c1 * c_interp, kStThreads), kStThreads, 0, s>>>(p.wparts_i, c1 * c_interp, c_interp, cin0, wpart,
                                                                                  grad_weight[0]);
    if (int rc = check_launch("sa_train_dw_reduce")) return rc;
    if (c_skip > 0) {
        // dWs = dZ_0^T S
        sa_train_dw_gemm<<<dim3(ceil_div(c1, 64), ceil_div(c_skip, 64), p.wparts[0]), kStThreads, 0, s>>>(D, FpSkipSrc{F}, p.rows, c1, c_skip,
                                                                                                       p.wchunk[0], wpart);
        if (int rc = check_launch("sa_train_dw_gemm")) return rc;
        sa_train_dw_reduce<<<ceil_div(c1 * c_skip, kStThreads), kStThreads, 0, s>>>(p.wparts[0], c1 * c_skip, c_skip, cin0, wpart,
                                                                                    grad_weight[0] + c_interp);
        if (int rc = check_launch("sa_train_dw_reduce")) return rc;
    }
    if (grad_known) {
        // dF = G Wi -> (b, c_interp, m)
        sa_train_da_gemm<<<dim3(p.KT, ceil_div(c_interp, kStColTile)), kStThreads, 0, s>>>(Gs, DaChannelMajor{grad_known, m, c_interp}, p.krows,
                                                                                           c1, W0, cin0, c_interp, 0, nullptr, nullptr);
        if (int rc = check_launch("sa_train_da_gemm")) return rc;
    }
    if (grad_skip && c_skip > 0) {
        // dS = dZ_0 Ws -> (b, c_skip, n)
        sa_train_da_gemm<<<dim3(p.T, ceil_div(c_skip, kStColTile)), kStThreads, 0, s>>>(D, DaChannelMajor{grad_skip, n, c_skip}, p.rows, c1,
                                                                                        W0 + c_interp, cin0, c_skip, 0, nullptr, nullptr);
        if (int rc = check_launch("sa_train_da_gemm")) return rc;
    }
    return 0;
}
