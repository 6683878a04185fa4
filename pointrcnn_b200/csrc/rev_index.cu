// rev_index.cu -- reverse index of a reference list and the fixed-order gather-sum over it; see rev_index.cuh.
#include <algorithm>
#include <type_traits>

#include "rev_index.cuh"

namespace prb {

constexpr int kRiThreads = 256;
constexpr int kScanItems = 4 * kRiThreads;   // counts per block of the offset scan

__global__ void __launch_bounds__(kRiThreads) rev_count(RevIndex R, const int *__restrict__ idx) {
    const int q = blockIdx.x * kRiThreads + threadIdx.x;
    if (q >= R.b * R.L) return;
    const int k = idx[q];
    if ((unsigned)k < (unsigned)R.n) atomicAdd(R.cnt + (q / R.L) * R.n + k, 1);
}

// exclusive prefix of v over the block; total receives the block's sum
__device__ __forceinline__ int ri_block_scan(int v, int &total) {
    __shared__ int ws[kRiThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) ws[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < kRiThreads / 32 ? ws[lane] : 0;
#pragma unroll
        for (int o = 1; o < kRiThreads / 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < kRiThreads / 32) ws[lane] = w;
    }
    __syncthreads();
    const int before = warp ? ws[warp - 1] : 0;
    total = ws[kRiThreads / 32 - 1];
    __syncthreads();
    return before + x - v;
}

// off[i] = the prefix of cnt within its block of kScanItems; tot[block] = the block's sum
__global__ void __launch_bounds__(kRiThreads) rev_scan_local(int K, const int *cnt, int *off, int *tot) {
    const int base = blockIdx.x * kScanItems + threadIdx.x * 4;
    int v[4], s = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[i] = base + i < K ? cnt[base + i] : 0;
        s += v[i];
    }
    int total;
    int x = ri_block_scan(s, total);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (base + i < K) off[base + i] = x;
        x += v[i];
    }
    if (threadIdx.x == 0) tot[blockIdx.x] = total;
}

// one block: tot -> its exclusive prefix; off[K] = the sum of all counts
__global__ void __launch_bounds__(kRiThreads) rev_scan_blocks(int nb, int *tot, int *off_end) {
    int carry = 0;
    for (int b0 = 0; b0 < nb; b0 += kRiThreads) {
        const int i = b0 + (int)threadIdx.x;
        const int v = i < nb ? tot[i] : 0;
        int total;
        const int x = ri_block_scan(v, total);
        if (i < nb) tot[i] = carry + x;
        carry += total;
    }
    if (threadIdx.x == 0) *off_end = carry;
}

__global__ void __launch_bounds__(kRiThreads) rev_scan_add(int K, const int *tot, int *off) {
    const int i = blockIdx.x * kRiThreads + threadIdx.x;
    if (i < K) off[i] += tot[i / kScanItems];
}

// each reference into a free slot of its source (cnt counts down to 0)
__global__ void __launch_bounds__(kRiThreads) rev_fill(RevIndex R, const int *__restrict__ idx) {
    const int q = blockIdx.x * kRiThreads + threadIdx.x;
    if (q >= R.b * R.L) return;
    const int k = idx[q];
    if ((unsigned)k >= (unsigned)R.n) return;
    const int j = (q / R.L) * R.n + k;
    R.list[R.off[j] + atomicSub(R.cnt + j, 1) - 1] = q;
}

// every source's references in increasing order (heapsort: bounded work however many references share a source)
__global__ void __launch_bounds__(kRiThreads) rev_sort(int K, const int *off, int *list) {
    const int j = blockIdx.x * kRiThreads + threadIdx.x;
    if (j >= K) return;
    int *a = list + off[j];
    const int len = off[j + 1] - off[j];
    auto sift = [a](int root, int end) {
        for (;;) {
            int ch = 2 * root + 1;
            if (ch >= end) return;
            if (ch + 1 < end && a[ch + 1] > a[ch]) ++ch;
            if (a[root] >= a[ch]) return;
            const int t = a[root];
            a[root] = a[ch];
            a[ch] = t;
            root = ch;
        }
    };
    for (int i = len / 2 - 1; i >= 0; --i) sift(i, len);
    for (int e = len - 1; e > 0; --e) {
        const int t = a[0];
        a[0] = a[e];
        a[e] = t;
        sift(0, e);
    }
}

__device__ __forceinline__ float seg_load(const float *p) { return __ldg(p); }
__device__ __forceinline__ float seg_load(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }

// one thread per (source, block of kSegCh channels); grid (sources / kRiThreads, channel blocks, scenes).  T: the value
// and output type (float: out = out + acc or acc; bfloat16: out = acc rounded once)
template <int KIND, typename T>
__global__ void __launch_bounds__(kRiThreads) seg_sum_kernel(RevIndex R, int c, const T *__restrict__ g, const float *__restrict__ w,
                                                             int accumulate, T *__restrict__ out) {
    const int s = blockIdx.z, cb = blockIdx.y * kSegCh, j = blockIdx.x * kRiThreads + threadIdx.x;
    if (j >= R.n) return;
    const int nch = min(kSegCh, c - cb);
    const int src = s * R.n + j;
    const int e0 = R.off[src], e1 = R.off[src + 1];
    float acc[kSegCh];
#pragma unroll
    for (int ch = 0; ch < kSegCh; ++ch) acc[ch] = 0.f;
    for (int e = e0; e < e1; ++e) {
        const int q = R.list[e], l = q - s * R.L;
        if constexpr (KIND == SEG_GROUP) {
            const T *gv = g + ((size_t)s * c + cb) * R.L + l;
#pragma unroll
            for (int ch = 0; ch < kSegCh; ++ch)
                if (ch < nch) acc[ch] = __fadd_rn(acc[ch], seg_load(gv + (size_t)ch * R.L));
        } else if constexpr (KIND == SEG_TAPS) {
            const int rows = R.L / 3;
            const T *gv = g + ((size_t)s * c + cb) * rows + l / 3;
            const float wq = __ldg(w + q);
#pragma unroll
            for (int ch = 0; ch < kSegCh; ++ch)
                if (ch < nch) acc[ch] = __fadd_rn(acc[ch], __fmul_rn(seg_load(gv + (size_t)ch * rows), wq));
        } else {
            const T *gv = g + (size_t)q * c + cb;
#pragma unroll
            for (int ch = 0; ch < kSegCh; ++ch)
                if (ch < nch) acc[ch] = __fadd_rn(acc[ch], seg_load(gv + ch));
        }
    }
    T *o = out + ((size_t)s * c + cb) * R.n + j;
#pragma unroll
    for (int ch = 0; ch < kSegCh; ++ch) {
        if (ch >= nch) continue;
        if constexpr (std::is_same_v<T, float>)
            o[(size_t)ch * R.n] = accumulate ? __fadd_rn(o[(size_t)ch * R.n], acc[ch]) : acc[ch];
        else
            o[(size_t)ch * R.n] = __float2bfloat16_rn(acc[ch]);
    }
}

// the offset of `bytes` placed at `at`; `at` moves past them to the next 256-byte boundary
static size_t ri_take(size_t &at, size_t bytes) {
    const size_t off = at;
    at = (at + bytes + 255) & ~(size_t)255;
    return off;
}

struct RiLayout {
    size_t cnt, off, tot, list, total;
};

static RiLayout ri_layout(int b, int L, int n) {
    const int K = b * n;
    RiLayout r;
    size_t at = 0;
    r.cnt = ri_take(at, (size_t)K * sizeof(int));
    r.off = ri_take(at, (size_t)(K + 1) * sizeof(int));
    r.tot = ri_take(at, (size_t)max(ceil_div(K, kScanItems), 1) * sizeof(int));
    r.list = ri_take(at, (size_t)b * L * sizeof(int));
    r.total = at;
    return r;
}

bool rev_index_fits(long b, long L, long n) {
    return b >= 0 && L >= 0 && n >= 0 && b * L < (1L << 31) && b * n < (1L << 31) - 1;
}

size_t rev_index_bytes(int b, int L, int n) { return ri_layout(b, L, n).total; }

RevIndex rev_index_at(int b, int L, int n, void *ws) {
    const RiLayout r = ri_layout(b, L, n);
    char *p = static_cast<char *>(ws);
    return RevIndex{b, L, n, reinterpret_cast<int *>(p + r.cnt), reinterpret_cast<int *>(p + r.off), reinterpret_cast<int *>(p + r.tot),
                    reinterpret_cast<int *>(p + r.list)};
}

int rev_index_build(const RevIndex &R, const int *idx, cudaStream_t s) {
    const int K = R.b * R.n, Q = R.b * R.L;
    if (cudaMemsetAsync(R.cnt, 0, (size_t)K * sizeof(int), s) != cudaSuccess) return check_launch("rev_index: memset");
    const int qblocks = max(ceil_div(Q, kRiThreads), 1), kblocks = max(ceil_div(K, kRiThreads), 1);
    const int scan_blocks = max(ceil_div(K, kScanItems), 1);
    rev_count<<<qblocks, kRiThreads, 0, s>>>(R, idx);
    if (int rc = check_launch("rev_count")) return rc;
    rev_scan_local<<<scan_blocks, kRiThreads, 0, s>>>(K, R.cnt, R.off, R.tot);
    if (int rc = check_launch("rev_scan_local")) return rc;
    rev_scan_blocks<<<1, kRiThreads, 0, s>>>(ceil_div(K, kScanItems), R.tot, R.off + K);
    if (int rc = check_launch("rev_scan_blocks")) return rc;
    rev_scan_add<<<kblocks, kRiThreads, 0, s>>>(K, R.tot, R.off);
    if (int rc = check_launch("rev_scan_add")) return rc;
    rev_fill<<<qblocks, kRiThreads, 0, s>>>(R, idx);
    if (int rc = check_launch("rev_fill")) return rc;
    rev_sort<<<kblocks, kRiThreads, 0, s>>>(K, R.off, R.list);
    return check_launch("rev_sort");
}

template <typename T>
static int seg_sum_launch(const RevIndex &R, int kind, int c, const T *g, const float *w, bool accumulate, T *out, cudaStream_t s) {
    const dim3 grid(ceil_div(R.n, kRiThreads), ceil_div(c, kSegCh), R.b);
    switch (kind) {
    case SEG_GROUP:
        seg_sum_kernel<SEG_GROUP, T><<<grid, kRiThreads, 0, s>>>(R, c, g, w, accumulate, out);
        return check_launch("seg_sum_kernel<SEG_GROUP>");
    case SEG_TAPS:
        seg_sum_kernel<SEG_TAPS, T><<<grid, kRiThreads, 0, s>>>(R, c, g, w, accumulate, out);
        return check_launch("seg_sum_kernel<SEG_TAPS>");
    default:
        seg_sum_kernel<SEG_ROWS, T><<<grid, kRiThreads, 0, s>>>(R, c, g, w, accumulate, out);
        return check_launch("seg_sum_kernel<SEG_ROWS>");
    }
}

int seg_sum(const RevIndex &R, int kind, int c, const float *g, const float *w, bool accumulate, float *out, cudaStream_t s) {
    return seg_sum_launch(R, kind, c, g, w, accumulate, out, s);
}

int seg_sum_bf16(const RevIndex &R, int kind, int c, const __nv_bfloat16 *g, const float *w, __nv_bfloat16 *out, cudaStream_t s) {
    return seg_sum_launch(R, kind, c, g, w, false, out, s);
}

__global__ void __launch_bounds__(kRiThreads) round_bf16_kernel(size_t count, const float *__restrict__ in, __nv_bfloat16 *__restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * kRiThreads + threadIdx.x; i < count; i += (size_t)gridDim.x * kRiThreads)
        out[i] = __float2bfloat16_rn(in[i]);
}

int round_bf16(size_t count, const float *in, void *out, cudaStream_t s) {
    if (count == 0) return 0;
    const unsigned blocks = (unsigned)std::min<size_t>((count + kRiThreads - 1) / kRiThreads, 4096);
    round_bf16_kernel<<<blocks, kRiThreads, 0, s>>>(count, in, static_cast<__nv_bfloat16 *>(out));
    return check_launch("round_bf16_kernel");
}

}  // namespace prb
