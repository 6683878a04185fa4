// grid.cu -- hash-grid accelerated ball query and 3-NN search with exact reference semantics.
//
// The reference scans ALL n points for every query (ball_query_gpu.cu:9-45, interpolate_gpu.cu:9-52): O(m*n)
// distance evaluations, 143 M + 72 M per RPN scene.  LiDAR scenes are sparse at the scale of the query radius, so a
// uniform hash grid visits ~10-40 candidates instead of 16384 -- but the OUTPUT contract is order dependent:
//   ball query : the first nsample hits in point-INDEX order, padded with the first hit
//   three_nn   : the three smallest d2, earlier index wins ties (strict '<' cascade in index order)
// Both are reproduced exactly from an unordered candidate set:
//   ball query : all in-range candidates of the 27 neighbouring cells are collected, then ranked by index
//                (rank = number of hits with a smaller index); rank k < nsample goes to slot k.
//   three_nn   : lexicographic (d2, idx) insertion == the reference's index-order strict-'<' cascade.
// The distance arithmetic is the reference's (dist2_ref), so every in/out decision is bit-identical.
// Coverage guarantee: cells are indexed in double precision with edge h = r_max*(1+1e-4); a point within the radius
// differs by less than one cell per axis, so the 3x3x3 block holds every hit.  three_nn accepts the block result only
// if its third distance is below (0.9999 h)^2, i.e. nothing outside the block can be closer or tie.
// Whatever the grid cannot answer safely (more than CAP candidates in dense clouds, a third neighbour farther than
// one cell) goes to an overflow list that the brute-force kernels of ball_group.cu / interp.cu process afterwards --
// dense clouds are exactly where their early exit is fast.
#include <math_constants.h>

#include "common.cuh"

namespace prb {

constexpr int GR_THREADS = 256;
constexpr int GR_WARPS = GR_THREADS / 32;
constexpr int BQ_CAP = 128;   // candidates per centre handled on the grid path

struct GridView {
    int table_size;           // power of two
    const int *heads;         // (b, table_size) first node of every hash bucket's list, -1 = empty
    const float4 *nodes;      // (b, n) {x, y, z, next index as int bits}, node i = point i
    const double *inv_h;      // (b) 1 / cell edge
};

__device__ __forceinline__ int cell_coord(float v, double inv_h) { return (int)floor((double)v * inv_h); }
__device__ __forceinline__ unsigned cell_hash(int cx, int cy, int cz, int mask) {
    unsigned h = (unsigned)cx * 73856093u ^ (unsigned)cy * 19349663u ^ (unsigned)cz * 83492791u;
    h ^= h >> 15;
    return h & (unsigned)mask;
}

// ---------------------------------------------------------------- build
// per-scene cell edge from the bounding box and the point count (three_nn): h = 1.6 * cbrt(volume / m), with every
// extent clamped from below so that flat or degenerate clouds still get a sane edge
__global__ void __launch_bounds__(256) grid_cell_from_bbox_kernel(int n, const float *__restrict__ xyz, double factor,
                                                                  double *__restrict__ inv_h, float *__restrict__ h_out) {
    __shared__ float s_lo[3][8], s_hi[3][8];
    const int scene = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *p = xyz + (size_t)scene * n * 3;
    float lo[3] = {CUDART_INF_F, CUDART_INF_F, CUDART_INF_F}, hi[3] = {-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F};
    for (int i = tid; i < n; i += 256)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = p[(size_t)i * 3 + a];
            if (isfinite(v)) { lo[a] = fminf(lo[a], v); hi[a] = fmaxf(hi[a], v); }
        }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        for (int o = 16; o; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        if (lane == 0) { s_lo[a][warp] = lo[a]; s_hi[a][warp] = hi[a]; }
    }
    __syncthreads();
    if (tid == 0) {
        double ext[3], emax = 0.0;
        for (int a = 0; a < 3; ++a) {
            float l = s_lo[a][0], h = s_hi[a][0];
            for (int w = 1; w < 8; ++w) { l = fminf(l, s_lo[a][w]); h = fmaxf(h, s_hi[a][w]); }
            ext[a] = (h >= l) ? (double)h - (double)l : 0.0;
            emax = fmax(emax, ext[a]);
        }
        if (!(emax > 0.0)) emax = 1.0;
        double vol = 1.0;
        for (int a = 0; a < 3; ++a) vol *= fmax(ext[a], emax * 0.02);
        double h = factor * cbrt(vol / (double)(n > 0 ? n : 1));
        h = fmax(h, emax * 1e-4);
        inv_h[scene] = 1.0 / h;
        h_out[scene] = (float)h;
    }
}

__global__ void grid_set_cell_kernel(int b, double h, double *__restrict__ inv_h, float *__restrict__ h_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < b) { inv_h[i] = 1.0 / h; h_out[i] = (float)h; }
}

__global__ void __launch_bounds__(256) grid_insert_kernel(int n, int table_size, const float *__restrict__ xyz,
                                                          const double *__restrict__ inv_h, int *__restrict__ heads,
                                                          float4 *__restrict__ nodes) {
    const int scene = blockIdx.y;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float *p = xyz + ((size_t)scene * n + i) * 3;
    const double ih = inv_h[scene];
    const unsigned hsh = cell_hash(cell_coord(p[0], ih), cell_coord(p[1], ih), cell_coord(p[2], ih), table_size - 1);
    const int nxt = atomicExch(heads + (size_t)scene * table_size + hsh, i);
    nodes[(size_t)scene * n + i] = make_float4(p[0], p[1], p[2], __int_as_float(nxt));
}

// prb_options.nn_sort_queries (off by default): one CTA per scene counts the 3-NN queries of every hash bucket in shared
// memory, scans, and scatters the queries grouped by bucket, so that a warp of three_nn_grid_kernel holds queries of one
// or two cells.  Measured: the sort costs what the locality saves.  Order inside a bucket is arbitrary (atomics) and
// does not matter: every query's answer is its own.
constexpr int GB_THREADS = 1024;
constexpr int GB_MAX_TABLE = 32768;      // 128 KB of shared counters

__global__ void __launch_bounds__(GB_THREADS) grid_build_csr_kernel(int n, int table_size, const float *__restrict__ xyz,
                                                                   const double *__restrict__ inv_h, int2 *__restrict__ range,
                                                                   float4 *__restrict__ nodes) {
    extern __shared__ int s_cnt[];          // table_size counters, then cursors
    __shared__ int s_wsum[GB_THREADS / 32];
    const int scene = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *pts = xyz + (size_t)scene * n * 3;
    const double ih = inv_h[scene];
    const int mask = table_size - 1;
    for (int i = tid; i < table_size; i += GB_THREADS) s_cnt[i] = 0;
    __syncthreads();
    for (int k = tid; k < n; k += GB_THREADS) {
        const float *q = pts + (size_t)k * 3;
        atomicAdd(&s_cnt[cell_hash(cell_coord(q[0], ih), cell_coord(q[1], ih), cell_coord(q[2], ih), mask)], 1);
    }
    __syncthreads();
    const int per = table_size / GB_THREADS;             // table_size is a power of two >= 1024
    const int base = tid * per;
    int sum = 0;
    for (int i = 0; i < per; ++i) sum += s_cnt[base + i];
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const int w = s_wsum[lane];
        int wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
        s_wsum[lane] = wi - w;
    }
    __syncthreads();
    int run = s_wsum[warp] + incl - sum;
    int2 *rg = range + (size_t)scene * table_size;
    for (int i = 0; i < per; ++i) {
        const int c = s_cnt[base + i];
        rg[base + i] = make_int2(run, run + c);
        s_cnt[base + i] = run;
        run += c;
    }
    __syncthreads();
    float4 *nd = nodes + (size_t)scene * n;
    for (int k = tid; k < n; k += GB_THREADS) {
        const float *q = pts + (size_t)k * 3;
        const float x = q[0], y = q[1], z = q[2];
        const int pos = atomicAdd(&s_cnt[cell_hash(cell_coord(x, ih), cell_coord(y, ih), cell_coord(z, ih), mask)], 1);
        nd[pos] = make_float4(x, y, z, __int_as_float(k));
    }
}

// ---------------------------------------------------------------- ball query on the grid
template <int NR>
struct GridBqParams {
    int b, n, m;
    float r2[NR];
    int ns[NR];
    int *idx[NR];
    const float *new_xyz, *xyz;
    GridView g;
    int *overflow;      // [0] = count, [1..] = (scene*m + centre) of centres left to the brute-force kernel
};

template <int NR>
__global__ void __launch_bounds__(GR_THREADS) ball_query_grid_kernel(const GridBqParams<NR> p) {
    __shared__ int s_cand[GR_WARPS][BQ_CAP];
    __shared__ int s_cnt[GR_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int scene = blockIdx.y;
    const int centre = blockIdx.x * GR_WARPS + warp;
    if (centre >= p.m) return;                       // whole warp
    const float *q = p.new_xyz + ((size_t)scene * p.m + centre) * 3;
    const float cx = q[0], cy = q[1], cz = q[2];
    const float *xyz = p.xyz + (size_t)scene * p.n * 3;
    const float4 *nodes = p.g.nodes + (size_t)scene * p.n;
    const double ih = p.g.inv_h[scene];
    float rmax = p.r2[0];
#pragma unroll
    for (int r = 1; r < NR; ++r) rmax = fmaxf(rmax, p.r2[r]);

    if (lane == 0) s_cnt[warp] = 0;
    __syncwarp();
    // lane l < 27 owns neighbour cell l; duplicates of a hash bucket are walked once (lowest lane keeps it)
    int j = -1;
    if (lane < 27) {
        const int bx = cell_coord(cx, ih) + lane % 3 - 1, by = cell_coord(cy, ih) + (lane / 3) % 3 - 1, bz = cell_coord(cz, ih) + lane / 9 - 1;
        const unsigned hsh = cell_hash(bx, by, bz, p.g.table_size - 1);
        const unsigned same = __match_any_sync(0x07ffffffu, hsh);
        if ((int)(__ffs(same) - 1) == lane) j = p.g.heads[(size_t)scene * p.g.table_size + hsh];
    }
    int walked = 0;
    bool over = false;
    while (j >= 0) {
        const float4 nd = __ldg(nodes + j);
        const float d2 = dist2_ref(cx - nd.x, cy - nd.y, cz - nd.z);
        if (d2 < rmax) {
            const int pos = atomicAdd(&s_cnt[warp], 1);
            if (pos < BQ_CAP) s_cand[warp][pos] = j;
        }
        j = __float_as_int(nd.w);
        if (++walked > 4 * BQ_CAP) { over = true; break; }     // pathological bucket: leave it to the scan kernel
    }
    __syncwarp();
    const int cnt = s_cnt[warp];
    if (__any_sync(0xffffffffu, over) || cnt > BQ_CAP) {
        if (lane == 0) p.overflow[1 + atomicAdd(p.overflow, 1)] = scene * p.m + centre;
        return;
    }
    // rank the hits of each radius by point index; slot k takes the hit of rank k, the tail repeats rank 0
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        int *out = p.idx[r] + ((size_t)scene * p.m + centre) * p.ns[r];
        if (cnt <= 32) {
            // the common case (ncu: one 32-candidate chunk per centre, where the all-pairs ranking below costs ~245
            // instructions per radius): a 15-stage bitonic sort of the hit indices across the warp; lane k then HOLDS rank k
            int v = 0x7fffffff;
            if (lane < cnt) {
                const int k = s_cand[warp][lane];
                const float d2 = dist2_ref(cx - xyz[(size_t)k * 3], cy - xyz[(size_t)k * 3 + 1], cz - xyz[(size_t)k * 3 + 2]);
                if (d2 < p.r2[r]) v = k;
            }
#pragma unroll
            for (int k = 2; k <= 32; k <<= 1)
#pragma unroll
                for (int j = k >> 1; j > 0; j >>= 1) {
                    const int o = __shfl_xor_sync(0xffffffffu, v, j);
                    const bool keep_min = ((lane & k) == 0) == ((lane & j) == 0);
                    v = keep_min ? min(v, o) : max(v, o);
                }
            const int nh = __popc(__ballot_sync(0xffffffffu, v != 0x7fffffff));
            const int first = __shfl_sync(0xffffffffu, v, 0);
            if (lane < nh && lane < p.ns[r]) out[lane] = v;
            if (nh > 0)
                for (int sl = nh + lane; sl < p.ns[r]; sl += 32) out[sl] = first;
            continue;
        }
        int nh = 0, first = 0x7fffffff;
        for (int c0 = 0; c0 < cnt; c0 += 32) {
            const int c = c0 + lane;
            int me = -1;
            if (c < cnt) {
                const int k = s_cand[warp][c];
                const float d2 = dist2_ref(cx - xyz[(size_t)k * 3], cy - xyz[(size_t)k * 3 + 1], cz - xyz[(size_t)k * 3 + 2]);
                if (d2 < p.r2[r]) me = k;
            }
            // rank of my hit among ALL hits of this radius
            int rank = 0;
            for (int e0 = 0; e0 < cnt; e0 += 32) {
                const int e = e0 + lane;
                int other = -1;
                if (e < cnt) {
                    const int k = s_cand[warp][e];
                    const float d2 = dist2_ref(cx - xyz[(size_t)k * 3], cy - xyz[(size_t)k * 3 + 1], cz - xyz[(size_t)k * 3 + 2]);
                    if (d2 < p.r2[r]) other = k;
                }
                for (int t = 0; t < 32; ++t) {
                    const int o = __shfl_sync(0xffffffffu, other, t);
                    rank += (o >= 0 && o < me) ? 1 : 0;
                }
            }
            if (me >= 0 && rank < p.ns[r]) out[rank] = me;
            const unsigned hm = __ballot_sync(0xffffffffu, me >= 0);
            nh += __popc(hm);
            const int lo = __reduce_min_sync(0xffffffffu, me >= 0 ? me : 0x7fffffff);
            first = min(first, lo);
        }
        if (nh > 0)
            for (int s = nh + lane; s < p.ns[r]; s += 32) out[s] = first;
    }
}

// brute-force scan for the centres on the overflow list (same code path as ball_query_kernel, one warp per centre)
template <int NR>
__global__ void __launch_bounds__(GR_THREADS) ball_query_overflow_kernel(const GridBqParams<NR> p) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int total = p.overflow[0];
    for (int item = blockIdx.x * GR_WARPS + warp; item < total; item += gridDim.x * GR_WARPS) {
        const int id = p.overflow[1 + item];
        const int scene = id / p.m, centre = id - scene * p.m;
        const float *q = p.new_xyz + (size_t)id * 3;
        const float cx = q[0], cy = q[1], cz = q[2];
        const float *xyz = p.xyz + (size_t)scene * p.n * 3;
        int cnt[NR], first[NR];
#pragma unroll
        for (int r = 0; r < NR; ++r) { cnt[r] = 0; first[r] = 0; }
        for (int i0 = 0; i0 < p.n; i0 += 32) {
            bool need = false;
#pragma unroll
            for (int r = 0; r < NR; ++r) need |= cnt[r] < p.ns[r];
            if (!need) break;
            const int i = i0 + lane;
            const bool in = i < p.n;
            float d2 = CUDART_INF_F;
            if (in) d2 = dist2_ref(cx - xyz[(size_t)i * 3], cy - xyz[(size_t)i * 3 + 1], cz - xyz[(size_t)i * 3 + 2]);
#pragma unroll
            for (int r = 0; r < NR; ++r) {
                const unsigned hits = __ballot_sync(0xffffffffu, in && d2 < p.r2[r]);
                if (hits == 0 || cnt[r] >= p.ns[r]) continue;
                if (cnt[r] == 0) first[r] = i0 + __ffs(hits) - 1;
                const int pos = cnt[r] + __popc(hits & ((1u << lane) - 1));
                if (((hits >> lane) & 1u) && pos < p.ns[r]) p.idx[r][((size_t)scene * p.m + centre) * p.ns[r] + pos] = i;
                cnt[r] = min(p.ns[r], cnt[r] + __popc(hits));
            }
        }
#pragma unroll
        for (int r = 0; r < NR; ++r)
            if (cnt[r] > 0)
                for (int s = cnt[r] + lane; s < p.ns[r]; s += 32) p.idx[r][((size_t)scene * p.m + centre) * p.ns[r] + s] = first[r];
    }
}

// ---------------------------------------------------------------- three_nn on the grid
struct GridNnParams {
    int b, n, m;
    const float *unknown, *known;
    float *dist2, *weight;
    int *idx;
    GridView g;
    const float *h;     // (b) cell edge
    int *overflow;      // [0] = count, [1..] = scene*n + unknown index
    const float4 *qnodes;   // optional: the queries grouped by hash bucket, {x, y, z, query index} (see prb_three_nn_grid)
};

__device__ __forceinline__ void nn_insert(float d, int k, float &b1, float &b2, float &b3, int &i1, int &i2, int &i3) {
    // lexicographic (d2, idx) order == the reference's strict '<' cascade over ascending indices
    if (k == i1 || k == i2 || k == i3) return;     // the same point reached through a colliding hash bucket
    if (d < b1 || (d == b1 && k < i1)) {
        b3 = b2; i3 = i2; b2 = b1; i2 = i1; b1 = d; i1 = k;
    } else if (d < b2 || (d == b2 && k < i2)) {
        b3 = b2; i3 = i2; b2 = d; i2 = k;
    } else if (d < b3 || (d == b3 && k < i3)) {
        b3 = d; i3 = k;
    }
}

__device__ __forceinline__ void nn_store(const GridNnParams &p, size_t o, float b1, float b2, float b3, int i1, int i2, int i3) {
    p.dist2[o] = b1; p.dist2[o + 1] = b2; p.dist2[o + 2] = b3;
    p.idx[o] = i1; p.idx[o + 1] = i2; p.idx[o + 2] = i3;
    if (p.weight) {
        const float r0 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(b1), 1e-8f));
        const float r1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(b2), 1e-8f));
        const float r2 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(b3), 1e-8f));
        const float norm = __fadd_rn(__fadd_rn(r0, r1), r2);
        p.weight[o] = __fdiv_rn(r0, norm); p.weight[o + 1] = __fdiv_rn(r1, norm); p.weight[o + 2] = __fdiv_rn(r2, norm);
    }
}

__global__ void __launch_bounds__(GR_THREADS) three_nn_grid_kernel(const GridNnParams p) {
    const int scene = blockIdx.y;
    const int t_ = blockIdx.x * GR_THREADS + threadIdx.x;
    if (t_ >= p.n) return;
    int u = t_;
    float ux, uy, uz;
    if (p.qnodes) {          // queries in cell order: the lanes of a warp walk the same few buckets (L1 hits instead of L2 sectors)
        const float4 qn = __ldg(p.qnodes + (size_t)scene * p.n + t_);
        ux = qn.x; uy = qn.y; uz = qn.z; u = __float_as_int(qn.w);
    } else {
        const float *q = p.unknown + ((size_t)scene * p.n + u) * 3;
        ux = q[0]; uy = q[1]; uz = q[2];
    }
    const float4 *nodes = p.g.nodes + (size_t)scene * p.m;
    const int *heads = p.g.heads + (size_t)scene * p.g.table_size;
    const double ih = p.g.inv_h[scene];
    const int cx = cell_coord(ux, ih), cy = cell_coord(uy, ih), cz = cell_coord(uz, ih);
    float b1 = CUDART_INF_F, b2 = CUDART_INF_F, b3 = CUDART_INF_F;
    int i1 = -1, i2 = -1, i3 = -1;
    int walked = 0;
    bool over = false;
    // a bucket reached twice (hash collision between neighbour cells) is harmless: nn_insert ignores a point that is
    // already in the list, and a point that was evicted cannot re-enter (everything kept is lexicographically smaller).
    // All 27 bucket heads are fetched up front (independent loads); the cells are then walked centre-out and a cell
    // whose nearest face is farther than the current third distance is skipped (its points can neither beat nor tie
    // it: the per-axis gaps are shrunk by 0.999 so that rounding on either side cannot make the bound optimistic).
    // The 27 unrolled walks diverge, and that helps: the diverged lane groups of a warp cover each other's dependent L2
    // loads, where one convergent cursor loop per lane measured slower.
    int hd[27];
#pragma unroll
    for (int c = 0; c < 27; ++c)
        hd[c] = __ldg(heads + cell_hash(cx + c % 3 - 1, cy + (c / 3) % 3 - 1, cz + c / 9 - 1, p.g.table_size - 1));
    float gap[3][3];
    {
        const double hd_ = 1.0 / ih;
        const double f[3] = {(double)ux - (double)cx * hd_, (double)uy - (double)cy * hd_, (double)uz - (double)cz * hd_};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float lo = (float)fmax(f[a] - 1e-9, 0.0) * 0.999f, hi = (float)fmax(hd_ - f[a] - 1e-9, 0.0) * 0.999f;
            gap[a][0] = lo * lo; gap[a][1] = 0.f; gap[a][2] = hi * hi;
        }
    }
    // visiting order: centre, 6 faces, 12 edges, 8 corners (cell c = (oz+1)*9 + (oy+1)*3 + (ox+1))
    constexpr int kOrder[27] = {13, 12, 14, 10, 16, 4, 22, 9, 11, 15, 17, 3, 5, 21, 23, 1, 7, 19, 25, 0, 2, 6, 8, 18, 20, 24, 26};
#pragma unroll
    for (int t = 0; t < 27; ++t) {
        const int c = kOrder[t];
        const float lb = gap[0][c % 3] + gap[1][(c / 3) % 3] + gap[2][c / 9];
        if (lb > b3) continue;
        for (int j = hd[c]; j >= 0 && !over;) {
            const float4 nd = __ldg(nodes + j);
            const float d = dist2_ref(ux - nd.x, uy - nd.y, uz - nd.z);
            nn_insert(d, j, b1, b2, b3, i1, i2, i3);
            j = __float_as_int(nd.w);
            if (++walked > 2048) over = true;
        }
    }
    const float hb = p.h[scene] * 0.9999f;
    if (over || !(b3 < hb * hb)) {   // something outside the 3x3x3 block could be closer (or tie): brute force decides
        p.overflow[1 + atomicAdd(p.overflow, 1)] = scene * p.n + u;
        return;
    }
    nn_store(p, ((size_t)scene * p.n + u) * 3, b1, b2, b3, i1, i2, i3);
}

// The reference starts its cascade at 1e40 (double), so only a finite distance ever enters: an inf (or NaN) distance
// must not take an empty slot through the index tie-break, or a query at infinity would list points 0, 1, 2 instead of
// the reference's 0, 0, 0.
__device__ __forceinline__ void nn_insert_lex(float d, int k, float &b1, float &b2, float &b3, int &i1, int &i2, int &i3) {
    if (!(d < CUDART_INF_F)) return;
    if (d < b1 || (d == b1 && k < i1)) {
        b3 = b2; i3 = i2; b2 = b1; i2 = i1; b1 = d; i1 = k;
    } else if (d < b2 || (d == b2 && k < i2)) {
        b3 = b2; i3 = i2; b2 = d; i2 = k;
    } else if (d < b3 || (d == b3 && k < i3)) {
        b3 = d; i3 = k;
    }
}

// brute force for the queries the grid could not certify: one CTA per query (a single warp walking thousands of
// points is a 40-80 us dependency chain that the whole level then waits for).  Every thread keeps the lexicographic
// top-3 of its strided share, warps merge with shuffles, warp 0 merges the 8 warp lists (the top-3 of a union does
// not depend on the visiting order).
__global__ void __launch_bounds__(GR_THREADS) three_nn_overflow_kernel(const GridNnParams p) {
    __shared__ float s_d[GR_WARPS][3];
    __shared__ int s_i[GR_WARPS][3];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int total = p.overflow[0];
    const int BIG = 0x7fffffff;
    for (int item = blockIdx.x; item < total; item += gridDim.x) {
        const int id = p.overflow[1 + item];
        const int scene = id / p.n;
        const float *q = p.unknown + (size_t)id * 3;
        const float ux = q[0], uy = q[1], uz = q[2];
        const float *kn = p.known + (size_t)scene * p.m * 3;
        float b1 = CUDART_INF_F, b2 = CUDART_INF_F, b3 = CUDART_INF_F;
        int i1 = BIG, i2 = BIG, i3 = BIG;
        int k = tid;
        for (; k + 3 * GR_THREADS < p.m; k += 4 * GR_THREADS) {     // four independent loads in flight per thread
            float d[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const float *c = kn + (size_t)(k + t * GR_THREADS) * 3;
                d[t] = dist2_ref(ux - c[0], uy - c[1], uz - c[2]);
            }
#pragma unroll
            for (int t = 0; t < 4; ++t) nn_insert_lex(d[t], k + t * GR_THREADS, b1, b2, b3, i1, i2, i3);
        }
        for (; k < p.m; k += GR_THREADS)
            nn_insert_lex(dist2_ref(ux - kn[(size_t)k * 3], uy - kn[(size_t)k * 3 + 1], uz - kn[(size_t)k * 3 + 2]), k, b1, b2, b3, i1, i2, i3);
        for (int o = 16; o; o >>= 1) {
            const float e1 = __shfl_xor_sync(0xffffffffu, b1, o), e2 = __shfl_xor_sync(0xffffffffu, b2, o), e3 = __shfl_xor_sync(0xffffffffu, b3, o);
            const int j1 = __shfl_xor_sync(0xffffffffu, i1, o), j2 = __shfl_xor_sync(0xffffffffu, i2, o), j3 = __shfl_xor_sync(0xffffffffu, i3, o);
            if (j1 != BIG) nn_insert_lex(e1, j1, b1, b2, b3, i1, i2, i3);
            if (j2 != BIG) nn_insert_lex(e2, j2, b1, b2, b3, i1, i2, i3);
            if (j3 != BIG) nn_insert_lex(e3, j3, b1, b2, b3, i1, i2, i3);
        }
        __syncthreads();      // the previous item's readers are done with the staging arrays
        if (lane == 0) { s_d[warp][0] = b1; s_d[warp][1] = b2; s_d[warp][2] = b3; s_i[warp][0] = i1; s_i[warp][1] = i2; s_i[warp][2] = i3; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < GR_WARPS; ++w)
                for (int t = 0; t < 3; ++t)
                    if (s_i[w][t] != BIG) nn_insert_lex(s_d[w][t], s_i[w][t], b1, b2, b3, i1, i2, i3);
            // fewer than three known points: the reference leaves index 0 / distance 1e40 (-> inf)
            nn_store(p, (size_t)id * 3, b1, b2, b3, i1 == BIG ? 0 : i1, i2 == BIG ? 0 : i2, i3 == BIG ? 0 : i3);
        }
    }
}

static int table_size_for(int n) {
    int t = 1024;
    while (t < 2 * n) t <<= 1;
    return t;
}

struct GridWs {
    int table;
    double *inv_h;      // (b)
    float *h;           // (b)
    float4 *nodes;      // (b, n_points)
    int *heads;         // (b, table)
    float4 *qnodes;     // (b, n_queries) the queries grouped by bucket (nn_sort_queries)
    int2 *qrange;       // (b, table) their runs
    int *overflow;      // count + up to b * n_queries entries
    size_t bytes;       // from ws to the end of the overflow list
};

// The one layout of the grid workspace.  carve(nullptr, ...) measures it, so the size the caller allocates and the
// regions carved from it cannot disagree.
static GridWs carve(void *ws, int b, int n_points, int n_queries) {
    GridWs g;
    g.table = table_size_for(n_points);
    const uintptr_t base = (uintptr_t)ws;
    uintptr_t c = (base + 255) & ~(uintptr_t)255;
    g.inv_h = (double *)c; c += (((size_t)b * 8 + 255) & ~(size_t)255);
    g.h = (float *)c; c += (((size_t)b * 4 + 255) & ~(size_t)255);
    g.nodes = (float4 *)c; c += (size_t)b * n_points * 16;
    g.heads = (int *)c; c += (size_t)b * g.table * 4;
    g.qnodes = (float4 *)c; c += (size_t)b * n_queries * 16;
    g.qrange = (int2 *)c; c += (size_t)b * g.table * 8;
    g.overflow = (int *)c; c += ((size_t)b * n_queries + 64) * 4;
    g.bytes = c - base;
    return g;
}

static GridView view_of(const GridWs &w) { return GridView{w.table, w.heads, w.nodes, w.inv_h}; }

// hash the points of every scene into the table: one linked list per bucket
static int build_grid(int b, int n, const float *xyz, const GridWs &w, cudaStream_t st) {
    grid_insert_kernel<<<dim3(ceil_div(n, 256), b), 256, 0, st>>>(n, w.table, xyz, w.inv_h, w.heads, w.nodes);
    return check_launch("grid_insert_kernel");
}

}  // namespace prb

using namespace prb;

extern "C" {

// the layout plus the slack that aligns it on any base
PRB_API size_t prb_grid_workspace_bytes(int b, int n_points, int n_queries) { return carve(nullptr, b, n_points, n_queries).bytes + 255; }

// ball query for one or two radii through the hash grid; same outputs as prb_ball_query / prb_ball_query_msg2
PRB_API int prb_ball_query_grid(int b, int n, int m, int nr, const float *radius, const int *nsample, const float *new_xyz,
                                const float *xyz, int *const *idx, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && n >= 0 && m >= 0 && (nr == 1 || nr == 2) && radius && nsample && new_xyz && xyz && idx && workspace,
                "ball_query_grid: bad arguments");
    if (b == 0 || m == 0) return 0;
    PRB_REQUIRE(workspace_bytes >= prb_grid_workspace_bytes(b, n, m), "ball_query_grid: workspace too small");
    PRB_REQUIRE((long)b * m < 0x7fffffffL && (long)b * n < 0x7fffffffL, "ball_query_grid: too many points");
    cudaStream_t st = (cudaStream_t)stream;
    GridWs w = carve(workspace, b, n, m);
    float rmax = radius[0];
    for (int r = 1; r < nr; ++r) rmax = radius[r] > rmax ? radius[r] : rmax;
    PRB_REQUIRE(rmax > 0.f, "ball_query_grid: radius must be positive");
    PRB_CUDA(cudaMemsetAsync(w.heads, 0xff, (size_t)b * w.table * 4, st));
    PRB_CUDA(cudaMemsetAsync(w.overflow, 0, 4, st));
    grid_set_cell_kernel<<<ceil_div(b, 128), 128, 0, st>>>(b, (double)rmax * 1.0001, w.inv_h, w.h);
    if (int rc = check_launch("grid_set_cell_kernel")) return rc;
    if (int rc = build_grid(b, n, xyz, w, st)) return rc;
    const dim3 grid(ceil_div(m, GR_WARPS), b);
    const int ogrid = 2 * num_sms();
    if (nr == 1) {
        GridBqParams<1> p;
        p.b = b; p.n = n; p.m = m; p.r2[0] = radius[0] * radius[0]; p.ns[0] = nsample[0]; p.idx[0] = idx[0];
        p.new_xyz = new_xyz; p.xyz = xyz; p.g = view_of(w); p.overflow = w.overflow;
        ball_query_grid_kernel<1><<<grid, GR_THREADS, 0, st>>>(p);
        if (int rc = check_launch("ball_query_grid_kernel<1>")) return rc;
        ball_query_overflow_kernel<1><<<ogrid, GR_THREADS, 0, st>>>(p);
        return check_launch("ball_query_overflow_kernel<1>");
    }
    GridBqParams<2> p;
    p.b = b; p.n = n; p.m = m;
    for (int r = 0; r < 2; ++r) { p.r2[r] = radius[r] * radius[r]; p.ns[r] = nsample[r]; p.idx[r] = idx[r]; }
    p.new_xyz = new_xyz; p.xyz = xyz; p.g = view_of(w); p.overflow = w.overflow;
    ball_query_grid_kernel<2><<<grid, GR_THREADS, 0, st>>>(p);
    if (int rc = check_launch("ball_query_grid_kernel<2>")) return rc;
    ball_query_overflow_kernel<2><<<ogrid, GR_THREADS, 0, st>>>(p);
    return check_launch("ball_query_overflow_kernel<2>");
}

// three_nn (+ optional weights) through the hash grid; same outputs as prb_three_nn
PRB_API int prb_three_nn_grid(int b, int n, int m, const float *unknown, const float *known, float *dist2, int *idx, float *weight,
                              void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && n >= 0 && m >= 0 && unknown && known && dist2 && idx && workspace, "three_nn_grid: bad arguments");
    if (b == 0 || n == 0) return 0;
    if (m < 3) return prb_three_nn(b, n, m, unknown, known, dist2, idx, weight, stream);
    PRB_REQUIRE(workspace_bytes >= prb_grid_workspace_bytes(b, m, n), "three_nn_grid: workspace too small");
    PRB_REQUIRE((long)b * m < 0x7fffffffL && (long)b * n < 0x7fffffffL, "three_nn_grid: too many points");
    cudaStream_t st = (cudaStream_t)stream;
    GridWs w = carve(workspace, b, m, n);
    PRB_CUDA(cudaMemsetAsync(w.heads, 0xff, (size_t)b * w.table * 4, st));
    PRB_CUDA(cudaMemsetAsync(w.overflow, 0, 4, st));
    // cell edge = 1.6 x mean point spacing.  A query is certified only if its third neighbour is closer than one
    // cell, everything else falls back to the exhaustive scan; the centre-out walk skips cells beyond the current
    // third distance.
    grid_cell_from_bbox_kernel<<<b, 256, 0, st>>>(m, known, 1.6, w.inv_h, w.h);
    if (int rc = check_launch("grid_cell_from_bbox_kernel")) return rc;
    if (int rc = build_grid(b, m, known, w, st)) return rc;
    GridNnParams p;
    p.b = b; p.n = n; p.m = m; p.unknown = unknown; p.known = known; p.dist2 = dist2; p.weight = weight; p.idx = idx;
    p.g = view_of(w); p.h = w.h; p.overflow = w.overflow;
    p.qnodes = nullptr;
    if (w.table <= GB_MAX_TABLE && opts().nn_sort_queries) {
        const size_t smem = (size_t)w.table * sizeof(int);
        if (smem > 48 * 1024)
            PRB_CUDA(cudaFuncSetAttribute(grid_build_csr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        grid_build_csr_kernel<<<b, GB_THREADS, smem, st>>>(n, w.table, unknown, w.inv_h, w.qrange, w.qnodes);
        if (int rc = check_launch("grid_build_csr_kernel(queries)")) return rc;
        p.qnodes = w.qnodes;
    }
    three_nn_grid_kernel<<<dim3(ceil_div(n, GR_THREADS), b), GR_THREADS, 0, st>>>(p);
    if (int rc = check_launch("three_nn_grid_kernel")) return rc;
    three_nn_overflow_kernel<<<4 * num_sms(), GR_THREADS, 0, st>>>(p);
    if (int rc = check_launch("three_nn_overflow_kernel")) return rc;
    return 0;
}

}  // extern "C"
