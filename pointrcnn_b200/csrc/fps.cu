// fps.cu -- furthest point sampling for sm_90a: register-resident, cluster-parallel.
//
// Replaces furthest_point_sampling_wrapper (pointnet2_lib/pointnet2/src/sampling.cpp:36-46 ->
// sampling_gpu.cu:93-253) and the gather_operation that follows it (pointnet2_modules.py:32-35).
//
// What the reference computes (the spec): idx[0]=0; every round updates temp[k]=min(temp[k],
// |p_k - p_last|^2) for all k and picks argmax_k temp[k].  Among equal maxima its S-thread strided
// scan + shared-memory tree picks the point with the smallest "rank"
//      rank(k) = bitrev_log2(S)(k mod S) * ceil(n/S) + k div S,   S = 2^floor(log2(min(n,1024)))
// (thread k mod S keeps its lowest k on ties; the tree keeps the lower slot on ties, i.e. compares
// thread ids LSB-first).  That rule is an observable part of the output (RoI-pooled inputs are full
// of duplicates), so it is reproduced exactly -- but not by copying the tree:
//
// Design: points are laid out in RANK order.  Thread g of a scene owns ranks [g*PPT,(g+1)*PPT) with
// xyz and the running min-distance in registers, so "lowest position wins" IS the tie rule at every
// level: strict '>' inside a thread, lowest lane inside a warp (redux.max + ballot + ffs), lowest
// warp inside a CTA, lowest CTA inside a cluster.  One __syncthreads per round.  A scene is spread
// over a thread-block cluster of CS CTAs (CS*THREADS*PPT >= n): each CTA's winner -- distance, rank AND
// coordinates, 32 bytes -- goes to every peer with two st.async stores that complete a transaction count on the
// peer's mbarrier (no cluster barrier in the loop).  A CTA mirrors only its OWN points in shared memory (<= 96 KB); the
// winner's coordinates travel with the message.  new_xyz is emitted on the fly.
#include <limits.h>
#include <math_constants.h>

#include "common.cuh"

namespace prb {

struct FpsParams {
    int b, n, m;
    int S, logS, Q;      // reference block size, its log2, ceil(n/S)
    const float *xyz;    // (b,n,3)
    float *temp;         // (b,n)
    int *idx;            // (b,m)
    float *new_xyz;      // (b,m,3) or nullptr
    const int *todo;     // (b) or nullptr: scenes whose entry is 0 are already answered (ordered-input shortcut below)
};

__device__ __forceinline__ int rank_to_k(int r, int S, int logS, int Q) {
    int brev = r / Q, q = r - brev * Q;
    if (brev >= S) return INT_MAX;
    int t = logS ? (int)(__brev((unsigned)brev) >> (32 - logS)) : 0;
    return q * S + t;
}
__device__ __forceinline__ int k_to_rank(int k, int S, int logS, int Q) {
    int t = k & (S - 1);
    int rv = logS == 0 ? 0 : (int)(__brev((unsigned)t) >> (32 - logS));
    return rv * Q + (k >> logS);
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_addr, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(cta));
    return r;
}
// ---- cluster exchange primitives
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity)
        : "memory");
}
// 16-byte store into a peer CTA's shared memory that completes 16 tx-bytes on the peer's mbarrier.
__device__ __forceinline__ void st_async_v4(uint32_t remote_addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t remote_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(remote_addr),
                 "r"(a), "r"(b), "r"(c), "r"(d), "r"(remote_bar)
                 : "memory");
}

constexpr int kMaxWarps = 32;
constexpr int kMaxCluster = 8;

// one exchanged winner: 32 bytes = two 16-byte st.async: {dist bits, rank, x, y} {z, -, -, -}
struct __align__(16) FpsMsg {
    int dist_bits;
    int rank;
    float x, y;
    float z;
    int pad[3];
};

template <int THREADS, int PPT, int CS>
__global__ void __launch_bounds__(THREADS, 1) fps_rank_kernel(const FpsParams p) {
    constexpr int W = THREADS / 32;
    constexpr int CAP = THREADS * PPT;               // ranks owned by this CTA
    extern __shared__ __align__(16) float s_pts[];   // xyz of MY ranks (3 floats per rank)
    __shared__ int2 s_wkey[2][kMaxWarps];            // per-warp (dist bits, rank), double buffered
    __shared__ FpsMsg s_slot[2][kMaxCluster];        // per-CTA winners (cluster exchange), double buffered
    __shared__ __align__(8) uint64_t s_bar[2];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int crank = CS > 1 ? (int)cluster_ctarank() : 0;
    const int scene = blockIdx.x / CS;
    if (p.todo && p.todo[scene] == 0) return;        // the whole cluster of a scene leaves together, before any barrier
    const int n = p.n, m = p.m, S = p.S, logS = p.logS, Q = p.Q;
    const float *xyz = p.xyz + (size_t)scene * n * 3;
    float *temp = p.temp + (size_t)scene * n;
    int *idx = p.idx + (size_t)scene * m;
    float *new_xyz = p.new_xyz ? p.new_xyz + (size_t)scene * m * 3 : nullptr;

    if (CS > 1 && tid == 0) {
        mbar_init(smem_u32(&s_bar[0]), 1);
        mbar_init(smem_u32(&s_bar[1]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }

    // my PPT consecutive ranks: coordinates + running min distance in registers, coordinates mirrored in shared
    // memory so that the CTA's winner can be looked up by rank
    const int g = crank * THREADS + tid;
    float px[PPT], py[PPT], pz[PPT], pd[PPT];
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
        int k = rank_to_k(g * PPT + i, S, logS, Q);
        if (k < n) {
            px[i] = xyz[k * 3 + 0];
            py[i] = xyz[k * 3 + 1];
            pz[i] = xyz[k * 3 + 2];
            pd[i] = temp[k];
        } else {  // hole in the rank space: can never win (real distances are >= 0)
            px[i] = py[i] = pz[i] = 0.f;
            pd[i] = -1.f;
        }
        s_pts[(tid * PPT + i) * 3 + 0] = px[i];
        s_pts[(tid * PPT + i) * 3 + 1] = py[i];
        s_pts[(tid * PPT + i) * 3 + 2] = pz[i];
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();

    // round 0: idx[0] = 0 (rank 0 == point 0)
    float cx = xyz[0], cy = xyz[1], cz = xyz[2];
    const bool writer = (tid == 0 && crank == 0);
    if (writer) {
        idx[0] = 0;  // holds RANKS until the fix-up pass below
        if (new_xyz) { new_xyz[0] = cx; new_xyz[1] = cy; new_xyz[2] = cz; }
    }
    uint32_t phase0 = 0, phase1 = 0;

    for (int j = 1; j < m; ++j) {
        const int par = j & 1;
        if (CS > 1 && tid == 0) mbar_arrive_expect_tx(smem_u32(&s_bar[par]), CS * 32);
        float best = -1.f;
        int bslot = 0;
#pragma unroll
        for (int i = 0; i < PPT; ++i) {
            float d = dist2_ref(px[i] - cx, py[i] - cy, pz[i] - cz);
            d = fminf(d, pd[i]);
            pd[i] = d;
            if (d > best) { best = d; bslot = i; }
        }
        // warp arg-max: distances are >= 0 (or -1 for holes), so their bit patterns order as signed ints
        // (two REDUX ops per level: max distance, then min rank among the ties -- ranks grow with lane and warp, so
        //  this is "lowest position wins"; measured 72-82 cycles per level against 121 for redux + vote + ffs + shfl)
        int vb = __float_as_int(best);
        int wm = __reduce_max_sync(0xffffffffu, vb);
        int wr = (int)__reduce_min_sync(0xffffffffu, vb == wm ? (unsigned)(g * PPT + bslot) : 0xffffffffu);
        if (lane == 0) s_wkey[par][warp] = make_int2(wm, wr);
        __syncthreads();

        // CTA-level winner (lowest warp wins ties)
        int2 kv = lane < W ? s_wkey[par][lane] : make_int2(INT_MIN, 0);
        int cm = __reduce_max_sync(0xffffffffu, kv.x);
        int r = (int)__reduce_min_sync(0xffffffffu, kv.x == cm ? (unsigned)kv.y : 0xffffffffu);   // winning rank, uniform in the CTA

        if (CS == 1) {
            cx = s_pts[r * 3 + 0]; cy = s_pts[r * 3 + 1]; cz = s_pts[r * 3 + 2];
        } else {
            // my CTA's winner (with its coordinates) goes to every CTA of the cluster: two 16-byte st.async per peer
            if (warp == 0 && lane < CS) {
                const int lr = r - crank * CAP;
                const float wx = s_pts[lr * 3 + 0], wy = s_pts[lr * 3 + 1], wz = s_pts[lr * 3 + 2];
                const uint32_t dst = map_to_cta(smem_u32(&s_slot[par][crank]), lane);
                const uint32_t bar = map_to_cta(smem_u32(&s_bar[par]), lane);
                st_async_v4(dst, (uint32_t)cm, (uint32_t)r, __float_as_uint(wx), __float_as_uint(wy), bar);
                st_async_v4(dst + 16, __float_as_uint(wz), 0u, 0u, 0u, bar);
            }
            mbar_wait_cluster(smem_u32(&s_bar[par]), par ? phase1 : phase0);
            if (par) phase1 ^= 1; else phase0 ^= 1;
            const int kx = lane < CS ? s_slot[par][lane].dist_bits : INT_MIN;
            const int gm = __reduce_max_sync(0xffffffffu, kx);
            const unsigned b3 = __ballot_sync(0xffffffffu, kx == gm);
            const FpsMsg &win = s_slot[par][__ffs(b3) - 1];      // lowest CTA wins ties: broadcast LDS
            r = win.rank;
            cx = win.x; cy = win.y; cz = win.z;
        }
        if (writer) {
            idx[j] = r;
            if (new_xyz) { new_xyz[j * 3 + 0] = cx; new_xyz[j * 3 + 1] = cy; new_xyz[j * 3 + 2] = cz; }
        }
    }

    // write back the running minimum distances (the reference leaves them in temp)
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
        int k = rank_to_k(g * PPT + i, S, logS, Q);
        if (k < n) temp[k] = pd[i];
    }
    // ranks -> point indices (same CTA wrote them; __syncthreads orders the global accesses)
    __syncthreads();
    if (crank == 0)
        for (int j = tid; j < m; j += THREADS) idx[j] = rank_to_k(idx[j], S, logS, Q);
    if (CS > 1) cluster_sync_all();
}

// Any n: distances stay in global memory (temp), points are visited in the reference's strided order;
// the tie rule is applied as (max distance, then min rank) with two redux ops per level.
__global__ void __launch_bounds__(1024, 1) fps_generic_kernel(const FpsParams p) {
    __shared__ int s_val[2][32];
    __shared__ unsigned s_rank[2][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.x, n = p.n, m = p.m, S = p.S, logS = p.logS, Q = p.Q;
    if (p.todo && p.todo[scene] == 0) return;
    const int W = blockDim.x / 32;  // blockDim.x = max(S, 32)
    const float *xyz = p.xyz + (size_t)scene * n * 3;
    float *temp = p.temp + (size_t)scene * n;
    int *idx = p.idx + (size_t)scene * m;
    float *new_xyz = p.new_xyz ? p.new_xyz + (size_t)scene * m * 3 : nullptr;
    int old = 0;
    if (tid == 0) idx[0] = 0;
    for (int j = 0; j < m; ++j) {
        float cx = xyz[old * 3], cy = xyz[old * 3 + 1], cz = xyz[old * 3 + 2];
        if (tid == 0 && new_xyz) { new_xyz[j * 3] = cx; new_xyz[j * 3 + 1] = cy; new_xyz[j * 3 + 2] = cz; }
        if (j == m - 1) break;
        float best = -1.f;
        int besti = 0;
        for (int k = tid; k < n && tid < S; k += S) {  // thread tid plays reference thread tid
            float d = dist2_ref(xyz[k * 3] - cx, xyz[k * 3 + 1] - cy, xyz[k * 3 + 2] - cz);
            d = fminf(d, temp[k]);
            temp[k] = d;
            if (d > best) { best = d; besti = k; }
        }
        unsigned rank = (unsigned)k_to_rank(besti, S, logS, Q);
        int vb = __float_as_int(best);
        int wm = __reduce_max_sync(0xffffffffu, vb);
        unsigned wr = __reduce_min_sync(0xffffffffu, vb == wm ? rank : 0xffffffffu);
        const int par = j & 1;
        if (lane == 0) { s_val[par][warp] = wm; s_rank[par][warp] = wr; }
        __syncthreads();
        int v = lane < W ? s_val[par][lane] : INT_MIN;
        unsigned rk = lane < W ? s_rank[par][lane] : 0xffffffffu;
        int cm = __reduce_max_sync(0xffffffffu, v);
        unsigned cr = __reduce_min_sync(0xffffffffu, v == cm ? rk : 0xffffffffu);
        old = rank_to_k((int)cr, S, logS, Q);
        if (tid == 0) idx[j + 1] = old;
    }
}

template <int THREADS, int PPT, int CS>
static int launch_rank(const FpsParams &p, cudaStream_t stream) {
    auto kern = fps_rank_kernel<THREADS, PPT, CS>;
    constexpr size_t smem = (size_t)THREADS * PPT * 3 * sizeof(float);   // the CTA's slice of the scene
    // static shared memory counts against the 48 KB default too
    if (smem + 2048 > 48 * 1024) PRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.b * CS);
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CS;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    PRB_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
    return check_launch("fps_rank_kernel");
}

// the (CS, threads, ppt) triples fps_run's configuration reaches, one line per cluster size
static int dispatch_rank(const FpsParams &p, int cs, int threads, int ppt, cudaStream_t st) {
#define PRB_FPS_CASE(C, T, P) \
    if (cs == C && threads == T && ppt == P) return launch_rank<T, P, C>(p, st);
    PRB_FPS_CASE(1, 128, 1) PRB_FPS_CASE(1, 128, 2) PRB_FPS_CASE(1, 128, 4) PRB_FPS_CASE(1, 256, 4)
    PRB_FPS_CASE(1, 512, 4) PRB_FPS_CASE(1, 512, 8) PRB_FPS_CASE(1, 512, 16)
    PRB_FPS_CASE(2, 512, 8) PRB_FPS_CASE(2, 512, 16)
    PRB_FPS_CASE(4, 512, 4) PRB_FPS_CASE(4, 512, 8) PRB_FPS_CASE(4, 512, 16)
    PRB_FPS_CASE(8, 256, 4) PRB_FPS_CASE(8, 512, 4) PRB_FPS_CASE(8, 512, 8) PRB_FPS_CASE(8, 512, 16)
#undef PRB_FPS_CASE
    set_error("fps: no kernel instance for cs=%d threads=%d ppt=%d", cs, threads, ppt);
    return -1;
}

// ------------------------------------------------------------------------------------------------------------
// Pruned FPS (n in (4096, 16384]): one CTA per scene, exact.
//
// A round only changes temp[k] where |p_k - p_last|^2 < temp[k], i.e. inside the new sample's Voronoi cell (~n/j
// points in round j).  Points are pre-sorted into spatially compact GROUPS of 32 (k-d ordered cells, counting sort
// in fps_sort_kernel); every group caches its box and its best (temp, rank).  A group whose box is provably
// farther from the new sample than its cached maximum cannot change and is skipped, so a round costs one box test
// per group plus the few groups around the sample -- and the fixed reduction latency -- instead of n updates.
// Exactness: a skipped update is a no-op of the reference (fminf(d, temp) == temp), the box test is conservative
// (0.9999 safety factor against fp32 rounding of either side), and the winner is still (max temp, then min rank).
//
// Layout: group g = slot * 16 + warp (neighbouring groups go to different warps); lane l of warp w keeps temp and
// rank of point l of its NS groups in registers (static indexing: the slot loop is unrolled and predicated on the
// ballot of the box tests, where lane j tests slot j); coordinates live in shared memory as three planes.
constexpr int kPrunedWarps = 16;

struct FpsSorted {
    float *sx, *sy, *sz, *st;   // (b, np) sorted coordinates and running min distance (pads: st = -1)
    int *srank;                 // (b, np) reference rank of the sorted point (pads: 0xffff)
    int np;                     // padded points per scene = 16 warps x NS slots x 32
};

constexpr int kSortBits = 13;
constexpr int kSortBins = 1 << kSortBits;

__global__ void __launch_bounds__(1024, 1) fps_sort_kernel(const FpsParams p, const FpsSorted s) {
    __shared__ unsigned s_cnt[kSortBins];
    __shared__ float s_red[6][32];
    __shared__ unsigned s_scan[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.x, n = p.n, np = s.np;
    if (p.todo && p.todo[scene] == 0) return;
    const float *xyz = p.xyz + (size_t)scene * n * 3;
    const float *temp = p.temp + (size_t)scene * n;
    float *sx = s.sx + (size_t)scene * np, *sy = s.sy + (size_t)scene * np, *sz = s.sz + (size_t)scene * np;
    float *st = s.st + (size_t)scene * np;
    int *srank = s.srank + (size_t)scene * np;

    for (int i = tid; i < kSortBins; i += 1024) s_cnt[i] = 0;
    // scene box
    float lo[3] = {CUDART_INF_F, CUDART_INF_F, CUDART_INF_F}, hi[3] = {-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F};
    for (int k = tid; k < n; k += 1024) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = xyz[k * 3 + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        if (lane == 0) { s_red[a][warp] = lo[a]; s_red[3 + a][warp] = hi[a]; }
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = s_red[a][0]; hi[a] = s_red[3 + a][0];
        for (int w = 1; w < 32; ++w) { lo[a] = fminf(lo[a], s_red[a][w]); hi[a] = fmaxf(hi[a], s_red[3 + a][w]); }
    }
    // k-d style bit allocation: every split halves the currently longest cell edge
    float edge[3];
    int bits[3] = {0, 0, 0};
    unsigned order = 0;   // 2 bits per split, first split in the low bits
#pragma unroll
    for (int a = 0; a < 3; ++a) { edge[a] = hi[a] - lo[a]; if (!(edge[a] > 0.f) || !(edge[a] < CUDART_INF_F)) edge[a] = 0.f; }
    for (int sidx = 0; sidx < kSortBits; ++sidx) {
        int a = 0;
        if (edge[1] > edge[a]) a = 1;
        if (edge[2] > edge[a]) a = 2;
        order |= (unsigned)a << (2 * sidx);
        edge[a] *= 0.5f;
        bits[a] += 1;
    }
    float inv[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float ext = hi[a] - lo[a];
        inv[a] = (ext > 0.f && ext < CUDART_INF_F) ? (float)(1 << bits[a]) / ext : 0.f;
    }
    // bit of the quantised coordinate each split looks at (4 bits per split)
    unsigned long long shifts = 0;
    {
        int rem0 = bits[0], rem1 = bits[1], rem2 = bits[2];
        for (int sidx = 0; sidx < kSortBits; ++sidx) {
            const int a = (order >> (2 * sidx)) & 3;
            int sh;
            if (a == 0) sh = --rem0; else if (a == 1) sh = --rem1; else sh = --rem2;
            shifts |= (unsigned long long)sh << (4 * sidx);
        }
    }
    const float lo0 = lo[0], lo1 = lo[1], lo2 = lo[2], inv0 = inv[0], inv1 = inv[1], inv2 = inv[2];
    const int top0 = (1 << bits[0]) - 1, top1 = (1 << bits[1]) - 1, top2 = (1 << bits[2]) - 1;
    auto quant = [](float c, float l, float iv, int top) -> int {
        const float f = (c - l) * iv;
        const int v = (f > 0.f) ? (int)fminf(f, 65535.f) : 0;   // NaN -> 0
        return v > top ? top : v;
    };
    auto key_of = [&](float x, float y, float z) -> unsigned {
        const int q0 = quant(x, lo0, inv0, top0), q1 = quant(y, lo1, inv1, top1), q2 = quant(z, lo2, inv2, top2);
        unsigned key = 0;
#pragma unroll
        for (int sidx = 0; sidx < kSortBits; ++sidx) {
            const int a = (order >> (2 * sidx)) & 3;
            const int sh = (int)((shifts >> (4 * sidx)) & 15ull);
            const int q = a == 0 ? q0 : (a == 1 ? q1 : q2);
            key = (key << 1) | ((unsigned)(q >> sh) & 1u);
        }
        return key;
    };
    __syncthreads();
    for (int k = tid; k < n; k += 1024) atomicAdd(&s_cnt[key_of(xyz[k * 3], xyz[k * 3 + 1], xyz[k * 3 + 2])], 1u);
    __syncthreads();
    // exclusive scan of the histogram: 8 consecutive bins per thread
    {
        constexpr int PER = kSortBins / 1024;
        unsigned loc[PER], sum = 0;
#pragma unroll
        for (int i = 0; i < PER; ++i) { loc[i] = s_cnt[tid * PER + i]; sum += loc[i]; }
        unsigned inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) s_scan[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            unsigned v = s_scan[lane], iv = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                unsigned u = __shfl_up_sync(0xffffffffu, iv, o);
                if (lane >= o) iv += u;
            }
            s_scan[lane] = iv - v;
        }
        __syncthreads();
        unsigned run = s_scan[warp] + inc - sum;
#pragma unroll
        for (int i = 0; i < PER; ++i) { s_cnt[tid * PER + i] = run; run += loc[i]; }
    }
    __syncthreads();
    for (int k = tid; k < n; k += 1024) {
        const float x = xyz[k * 3], y = xyz[k * 3 + 1], z = xyz[k * 3 + 2];
        const unsigned pos = atomicAdd(&s_cnt[key_of(x, y, z)], 1u);
        sx[pos] = x; sy[pos] = y; sz[pos] = z;
        st[pos] = temp[k];
        srank[pos] = k_to_rank(k, p.S, p.logS, p.Q);
    }
    __syncthreads();   // CTA-scope visibility of the scatter above
    for (int i = n + tid; i < np; i += 1024) {   // pads sit on the last sorted point and can never win
        sx[i] = sx[n - 1]; sy[i] = sy[n - 1]; sz[i] = sz[n - 1];
        st[i] = -1.f;
        srank[i] = 0xffff;
    }
}

// Warp-wide float max / min as one integer REDUX: sm_90 has no float redux, but the map below is an order-preserving
// involution from floats to signed ints (negative floats get their magnitude bits flipped), so the integer extremum
// maps back to the float extremum exactly.
__device__ __forceinline__ int float_order_key(float v) {
    const int i = __float_as_int(v);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float float_from_order_key(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }
__device__ __forceinline__ float redux_max_f32(float v) {
    return float_from_order_key(__reduce_max_sync(0xffffffffu, float_order_key(v)));
}
__device__ __forceinline__ float redux_min_f32(float v) {
    return float_from_order_key(__reduce_min_sync(0xffffffffu, float_order_key(v)));
}

// one slot of the pruned round: update my point of group (J, warp), refresh the group's cached best.
// The best is a (value, payload) pair reduced with two CREDUX ops: payload = (0x3fff - rank) << 5 | lane, so the
// larger payload is the smaller rank and names the lane that holds the point (no vote / ffs / shuffle).
#define PRB_FPS_SLOT(J)                                                                                      \
    case J: {                                                                                                \
        const int P = (((J) * W + warp) << 5) + lane;                                                        \
        const float v = fminf(dist2_ref(px[P] - cx, py[P] - cy, pz[P] - cz), t[(J) < NS ? (J) : 0]);         \
        t[(J) < NS ? (J) : 0] = v;                                                                           \
        const float mx = redux_max_f32(v);                                                                   \
        const unsigned mp = __reduce_max_sync(0xffffffffu, v == mx ? pay[(J) < NS ? (J) : 0] : 0u);          \
        if (lane == (J)) { gval = mx; gpay = mp; }                                                           \
    } break;

// W warps x NS slots per lane cover the W * NS groups of a scene: NS = 32 for 16384 points, 16 for 8192.
template <int NS>
__global__ void __launch_bounds__(32 * kPrunedWarps, 1) fps_pruned_kernel(const FpsParams p, const FpsSorted s) {
    constexpr int W = kPrunedWarps;
    constexpr int NP = W * NS * 32;
    extern __shared__ __align__(16) float s_pl[];       // three planes of NP floats
    __shared__ uint2 s_w[2][W];                         // per-warp winner {temp bits, (0x3fff - rank) << 14 | position}
    float *px = s_pl, *py = s_pl + NP, *pz = s_pl + 2 * NP;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.x, n = p.n, m = p.m;
    if (p.todo && p.todo[scene] == 0) return;
    const float *xyz = p.xyz + (size_t)scene * n * 3;
    float *temp = p.temp + (size_t)scene * n;
    int *idx = p.idx + (size_t)scene * m;
    float *new_xyz = p.new_xyz ? p.new_xyz + (size_t)scene * m * 3 : nullptr;
    {
        const float4 *gx = reinterpret_cast<const float4 *>(s.sx + (size_t)scene * NP);
        const float4 *gy = reinterpret_cast<const float4 *>(s.sy + (size_t)scene * NP);
        const float4 *gz = reinterpret_cast<const float4 *>(s.sz + (size_t)scene * NP);
        for (int i = tid; i < NP / 4; i += 32 * W) {
            reinterpret_cast<float4 *>(px)[i] = gx[i];
            reinterpret_cast<float4 *>(py)[i] = gy[i];
            reinterpret_cast<float4 *>(pz)[i] = gz[i];
        }
    }
    __syncthreads();
    // registers: running min distance and tie-break payload of my point in each of the warp's NS groups; lane j
    // also owns the box and the cached best of slot j
    float t[NS];
    unsigned pay[NS];
    float lox = 0.f, loy = 0.f, loz = 0.f, hix = 0.f, hiy = 0.f, hiz = 0.f, gval = -1.f;
    unsigned gpay = 0u;
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        const int P = ((j * W + warp) << 5) + lane;
        t[j] = s.st[(size_t)scene * NP + P];
        pay[j] = ((0x3fffu - ((unsigned)s.srank[(size_t)scene * NP + P] & 0x3fffu)) << 5) | (unsigned)lane;
        const float x = px[P], y = py[P], z = pz[P];
        const float ax = redux_min_f32(x), ay = redux_min_f32(y), az = redux_min_f32(z);
        const float bx = redux_max_f32(x), by = redux_max_f32(y), bz = redux_max_f32(z);
        const float mx = redux_max_f32(t[j]);
        const unsigned mp = __reduce_max_sync(0xffffffffu, t[j] == mx ? pay[j] : 0u);
        if (lane == j) { lox = ax; loy = ay; loz = az; hix = bx; hiy = by; hiz = bz; gval = mx; gpay = mp; }
    }

    float cx = xyz[0], cy = xyz[1], cz = xyz[2];
    if (tid == 0) {
        idx[0] = 0;   // ranks until the fix-up pass below (rank 0 == point 0)
        if (new_xyz) { new_xyz[0] = cx; new_xyz[1] = cy; new_xyz[2] = cz; }
    }
    const unsigned my_group_base = (unsigned)((lane * W + warp) << 5);
    for (int round = 1; round < m; ++round) {
        const int par = round & 1;
        // box test of my slot
        const float ex = fmaxf(fmaxf(lox - cx, cx - hix), 0.f);
        const float ey = fmaxf(fmaxf(loy - cy, cy - hiy), 0.f);
        const float ez = fmaxf(fmaxf(loz - cz, cz - hiz), 0.f);
        const float lb = ex * ex + ey * ey + ez * ez;
        const bool untouched = (lb * 0.9999f >= gval) && (lb > 1e-30f);
        unsigned mask = __ballot_sync(0xffffffffu, lane < NS && !untouched);
        while (mask) {                       // warp-uniform walk over the touched slots, highest first
            const int j = 31 - __clz(mask);
            mask &= ~(1u << j);
            switch (j) {
                PRB_FPS_SLOT(0) PRB_FPS_SLOT(1) PRB_FPS_SLOT(2) PRB_FPS_SLOT(3) PRB_FPS_SLOT(4) PRB_FPS_SLOT(5) PRB_FPS_SLOT(6)
                PRB_FPS_SLOT(7) PRB_FPS_SLOT(8) PRB_FPS_SLOT(9) PRB_FPS_SLOT(10) PRB_FPS_SLOT(11) PRB_FPS_SLOT(12)
                PRB_FPS_SLOT(13) PRB_FPS_SLOT(14) PRB_FPS_SLOT(15) PRB_FPS_SLOT(16) PRB_FPS_SLOT(17) PRB_FPS_SLOT(18)
                PRB_FPS_SLOT(19) PRB_FPS_SLOT(20) PRB_FPS_SLOT(21) PRB_FPS_SLOT(22) PRB_FPS_SLOT(23) PRB_FPS_SLOT(24)
                PRB_FPS_SLOT(25) PRB_FPS_SLOT(26) PRB_FPS_SLOT(27) PRB_FPS_SLOT(28) PRB_FPS_SLOT(29) PRB_FPS_SLOT(30)
                PRB_FPS_SLOT(31)
            }
        }
        // warp winner over its slots, then CTA winner: (max temp, then min rank) as (value, payload) maxima
        const float wm = redux_max_f32(gval);
        const unsigned cand = ((gpay >> 5) << 14) | (my_group_base + (gpay & 31u));
        const unsigned wp = __reduce_max_sync(0xffffffffu, gval == wm ? cand : 0u);
        if (lane == 0) s_w[par][warp] = make_uint2(__float_as_uint(wm), wp);
        __syncthreads();
        const uint2 kv = lane < W ? s_w[par][lane] : make_uint2(__float_as_uint(-1.f), 0u);
        const float cm = redux_max_f32(__uint_as_float(kv.x));
        const unsigned cp = __reduce_max_sync(0xffffffffu, __uint_as_float(kv.x) == cm ? kv.y : 0u);
        const unsigned pos = cp & 0x3fffu;
        cx = px[pos]; cy = py[pos]; cz = pz[pos];
        if (tid == 0) {
            idx[round] = (int)(0x3fffu - (cp >> 14));
            if (new_xyz) { new_xyz[round * 3 + 0] = cx; new_xyz[round * 3 + 1] = cy; new_xyz[round * 3 + 2] = cz; }
        }
    }
    // running minimum distances back to the reference's temp (pads sit past n in the sorted order), ranks -> indices
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        const int P = ((j * W + warp) << 5) + lane;
        if (P < n) {
            const int k = rank_to_k((int)(0x3fffu - (pay[j] >> 5)), p.S, p.logS, p.Q);
            if (k < n) temp[k] = t[j];
        }
    }
    __syncthreads();
    for (int j = tid; j < m; j += 32 * W) idx[j] = rank_to_k(idx[j], p.S, p.logS, p.Q);
}
#undef PRB_FPS_SLOT

}  // namespace prb

using namespace prb;

// pruned path: slots per lane for n points (0 = not applicable)
static int pruned_slots(int n) {
    if (n > 16384) return 0;
    if (n > 8192) return 32;
    if (n > 4096) return 16;
    return 0;
}

template <int NS>
static int launch_pruned(const FpsParams &p, const FpsSorted &s, cudaStream_t st) {
    const size_t smem = (size_t)3 * kPrunedWarps * NS * 32 * sizeof(float);
    if (smem + 1024 > 48 * 1024)
        PRB_CUDA(cudaFuncSetAttribute(fps_pruned_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fps_sort_kernel<<<p.b, 1024, 0, st>>>(p, s);
    if (int rc = check_launch("fps_sort_kernel")) return rc;
    fps_pruned_kernel<NS><<<p.b, 32 * kPrunedWarps, smem, st>>>(p, s);
    return check_launch("fps_pruned_kernel");
}

extern "C" size_t prb_fps_workspace_bytes(int b, int n) {
    const int ns = pruned_slots(n);
    return ns ? (size_t)b * kPrunedWarps * ns * 32 * 5 * sizeof(float) + 256 : 0;
}

extern "C" int prb_furthest_point_sampling(int b, int n, int m, const float *xyz, float *temp, int *idx,
                                           float *new_xyz, void *stream) {
    return prb_furthest_point_sampling_ws(b, n, m, xyz, temp, idx, new_xyz, nullptr, 0, stream);
}

static int fps_run(int b, int n, int m, const float *xyz, float *temp, int *idx, float *new_xyz, void *workspace,
                   size_t workspace_bytes, void *stream, const int *todo);

extern "C" int prb_furthest_point_sampling_ws(int b, int n, int m, const float *xyz, float *temp, int *idx,
                                              float *new_xyz, void *workspace, size_t workspace_bytes, void *stream) {
    return fps_run(b, n, m, xyz, temp, idx, new_xyz, workspace, workspace_bytes, stream, nullptr);
}

static int fps_run(int b, int n, int m, const float *xyz, float *temp, int *idx, float *new_xyz, void *workspace,
                   size_t workspace_bytes, void *stream, const int *todo) {
    PRB_REQUIRE(b >= 0 && n > 0 && xyz && temp && idx, "fps: bad arguments (b=%d n=%d)", b, n);
    if (m <= 0 || b == 0) return 0;  // reference kernel returns immediately for m <= 0
    cudaStream_t st = (cudaStream_t)stream;
    FpsParams p;
    p.b = b; p.n = n; p.m = m; p.todo = todo;
    int logS = 0;
    while ((2 << logS) <= n && logS < 10) ++logS;  // S = 2^floor(log2(min(n,1024))), cuda_utils.h:10-14
    p.S = 1 << logS; p.logS = logS; p.Q = ceil_div(n, p.S);
    p.xyz = xyz; p.temp = temp; p.idx = idx; p.new_xyz = new_xyz;
    const int n_pad = p.S * p.Q;

    // exact pruned kernel (one CTA per scene) when the caller lent scratch memory
    if (const int ns = pruned_slots(n); ns && workspace && m > 1) {
        const size_t np = (size_t)kPrunedWarps * ns * 32;
        PRB_REQUIRE(workspace_bytes >= (size_t)b * np * 5 * sizeof(float) + 256, "fps: workspace of %zu bytes is too small", workspace_bytes);
        FpsSorted s;
        float *w = reinterpret_cast<float *>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
        s.sx = w; s.sy = w + b * np; s.sz = w + 2 * b * np; s.st = w + 3 * b * np;
        s.srank = reinterpret_cast<int *>(w + 4 * b * np);
        s.np = (int)np;
        return ns == 16 ? launch_pruned<16>(p, s, st) : launch_pruned<32>(p, s, st);
    }

    // configuration: cluster size, threads per CTA, points per thread
    // A cluster of CS CTAs per scene cuts the per-round compute CS-fold; each CTA mirrors only its own slice of the
    // scene in shared memory (<= 96 KB); large batches use smaller clusters so that CTAs do not start sharing SMs.
    int cs = 1;
    if (n_pad >= 8192) {
        cs = (long)b * 8 <= num_sms() / 2 ? 8 : 4;
        while (cs > 1 && (long)b * cs > 2L * num_sms()) cs >>= 1;
    }
    while (cs < 8 && ceil_div(n_pad, cs) > 8192) cs <<= 1;  // keep the register-resident path
    const int P = ceil_div(n_pad, cs);
    if (P > 8192) {                                          // more than 65536 points
        fps_generic_kernel<<<b, p.S < 32 ? 32 : p.S, 0, st>>>(p);
        return check_launch("fps_generic_kernel");
    }
    int threads = 128;
    while (threads < 512 && threads * 4 < P) threads <<= 1;
    int ppt = 1;
    while (threads * ppt < P) ppt <<= 1;
    return dispatch_rank(p, cs, threads, ppt, st);
}

// ------------------------------------------------------------------------------------------------------------
// Ordered-input shortcut.
//
// The four sampling levels of a PointNet++ encoder are nested: level l+1 samples from the OUTPUT of level l, which
// lists its points in the order FPS picked them, starting at the same point 0.  Pick k of level l maximises the
// running min-distance over ALL points of level l-1; it belongs to the sampled subset, the subset's running
// distances are the same fp32 numbers (same operands, same order), so it is also the maximum over the subset:
// FPS(level-l output, m) = (0, 1, ..., m-1) -- unless two points tie for a maximum, where the reference's
// position-dependent tie rule may choose differently in the two levels.
//
// Nothing is assumed about where xyz came from.  The shortcut is taken per scene only after it is PROVEN for that
// scene: with r_j(k) = min(temp0[j], min_{i<k} |p_j - p_i|^2) (the reference's running distance of point j when
// pick k is chosen if the picks so far were 0..k-1) and v_k = r_k(k),
//      FPS(xyz, m) = iota(m)   <=   for all k in [1, m), for all j != k:  r_j(k) < v_k,  or  r_j(k) == v_k and rank(k) < rank(j)
// by induction over k (rank = the reference's tie rule, which the sampling kernels implement: equal maxima go to the smaller rank).  The check is n*m distance evaluations with no serial
// dependence between points (one thread per j, a running minimum over k) instead of m dependent arg-max rounds:
// 16 x (4096 -> 1024) takes ~20 us against ~400 us.  Scenes that fail the check (ties, duplicates, NaN, or simply an
// input that is not in FPS order) keep todo[scene] = 1 and are sampled by the ordinary kernels, launched right after
// with the todo list (their CTAs of proven scenes return at once): no host round trip, capturable in a CUDA graph.
// Outputs of a proven scene are written exactly as the kernels would: idx = iota, new_xyz = xyz[:m],
// temp[j] = r_j(m-1).

namespace prb {

// v[k] = r_k(k) for k < m.  Four lanes share one k (i strided by 4), 32 k per CTA.
__global__ void __launch_bounds__(128) fps_prefix_v_kernel(int n, int m, const float *__restrict__ xyz_all,
                                                            const float *__restrict__ temp_all, float *__restrict__ v_all,
                                                            int *__restrict__ todo) {
    __shared__ float4 s_p[256];
    const int scene = blockIdx.y, tid = threadIdx.x;
    const float *xyz = xyz_all + (size_t)scene * n * 3;
    if (blockIdx.x == 0 && tid == 0) todo[scene] = 0;   // raised by the check kernel, which runs after this one
    const int k = blockIdx.x * 32 + (tid >> 2), sub = tid & 3;
    const int kmax = min(m, blockIdx.x * 32 + 32);      // picks < kmax are needed by this CTA
    float px = 0.f, py = 0.f, pz = 0.f, r = CUDART_INF_F;
    if (k < m) {
        px = xyz[k * 3]; py = xyz[k * 3 + 1]; pz = xyz[k * 3 + 2];
        if (sub == 0) r = temp_all[(size_t)scene * n + k];
    }
    for (int base = 0; base < kmax; base += 256) {
        __syncthreads();
        for (int e = tid; e < 256 && base + e < kmax; e += 128)
            s_p[e] = make_float4(xyz[(base + e) * 3], xyz[(base + e) * 3 + 1], xyz[(base + e) * 3 + 2], 0.f);
        __syncthreads();
        const int hi = min(256, k - base);               // picks i < k only
#pragma unroll 4
        for (int e = sub; e < hi; e += 4) {
            const float4 c = s_p[e];
            r = fminf(r, dist2_ref(px - c.x, py - c.y, pz - c.z));
        }
    }
    r = fminf(r, __shfl_xor_sync(0xffffffffu, r, 1));
    r = fminf(r, __shfl_xor_sync(0xffffffffu, r, 2));
    if (k < m && sub == 0) v_all[(size_t)scene * m + k] = r;
}

// thread j walks k = 1 .. m-1 with its running minimum and compares it with v_k.  r_j(k) < v_k is the common case; an exact
// tie (r_j(k) == v_k: ~2 % of uniform 4096-point levels hold one, always between consecutive picks) is settled the way the
// sampling kernels settle it -- the smaller reference rank wins -- so pick k stands iff rank(k) < rank(j); anything else
// (r_j(k) > v_k, NaN, a lost tie) leaves the scene to the kernels.
__global__ void __launch_bounds__(256) fps_prefix_check_kernel(int n, int m, const float *__restrict__ xyz_all,
                                                                const float *__restrict__ temp_all,
                                                                const float *__restrict__ v_all, float *__restrict__ rtemp_all,
                                                                int *__restrict__ todo, int S, int logS, int Q) {
    __shared__ float4 s_c[256];                          // (x, y, z of pick k-1, v_k)
    const int scene = blockIdx.y, tid = threadIdx.x;
    const float *xyz = xyz_all + (size_t)scene * n * 3;
    const float *v = v_all + (size_t)scene * m;
    const int j = blockIdx.x * 256 + tid;
    float px = 0.f, py = 0.f, pz = 0.f, r = -1.f;        // threads past n: r = -1 is below every v_k >= 0
    if (j < n) {
        px = xyz[j * 3]; py = xyz[j * 3 + 1]; pz = xyz[j * 3 + 2];
        r = temp_all[(size_t)scene * n + j];
    }
    bool bad = false;
    for (int base = 1; base < m; base += 256) {
        __syncthreads();
        {
            const int k = base + tid;
            if (k < m) s_c[tid] = make_float4(xyz[(k - 1) * 3], xyz[(k - 1) * 3 + 1], xyz[(k - 1) * 3 + 2], v[k]);
        }
        __syncthreads();
        const int cnt = min(256, m - base);
        const float r0 = r;
        bool any = false;
#pragma unroll 8
        for (int e = 0; e < cnt; ++e) {                  // branch-free: 4096 x 1024 of these per scene at level 2
            const float4 c = s_c[e];
            r = fminf(r, dist2_ref(px - c.x, py - c.y, pz - c.z));
            any |= !(r < c.w);
        }
        if (any) {                                       // rare: my own round (k == j), a tie, or a failed proof -- replay the chunk
            float rr = r0;
            for (int e = 0; e < cnt; ++e) {
                const float4 c = s_c[e];
                rr = fminf(rr, dist2_ref(px - c.x, py - c.y, pz - c.z));
                const int k = base + e;
                if (!(rr < c.w) && k != j && (!(rr <= c.w) || k_to_rank(j, S, logS, Q) < k_to_rank(k, S, logS, Q))) bad = true;
            }
        }
    }
    if (j < n) {
        rtemp_all[(size_t)scene * n + j] = r;
        if (bad) todo[scene] = 1;
    }
}

__global__ void __launch_bounds__(256) fps_prefix_emit_kernel(int n, int m, const float *__restrict__ xyz_all,
                                                               const float *__restrict__ rtemp_all,
                                                               const int *__restrict__ todo, float *__restrict__ temp_all,
                                                               int *__restrict__ idx_all, float *__restrict__ new_xyz_all) {
    const int scene = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
    if (todo[scene] != 0 || j >= n) return;
    temp_all[(size_t)scene * n + j] = rtemp_all[(size_t)scene * n + j];
    if (j < m) {
        idx_all[(size_t)scene * m + j] = j;
        if (new_xyz_all) {
            const float *s = xyz_all + ((size_t)scene * n + j) * 3;
            float *d = new_xyz_all + ((size_t)scene * m + j) * 3;
            d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
        }
    }
}

}  // namespace prb

static size_t ordered_header_bytes(int b, int n, int m) {
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    return up((size_t)b * sizeof(int)) + up((size_t)b * m * sizeof(float)) + up((size_t)b * n * sizeof(float));
}

extern "C" size_t prb_fps_ordered_workspace_bytes(int b, int n, int m) {
    if (b <= 0 || n <= 0 || m <= 0) return 0;
    return ordered_header_bytes(b, n, m) + prb_fps_workspace_bytes(b, n) + 256;
}

extern "C" int prb_furthest_point_sampling_ordered_ws(int b, int n, int m, const float *xyz, float *temp, int *idx,
                                                      float *new_xyz, int *todo_out, void *workspace, size_t workspace_bytes,
                                                      void *stream) {
    PRB_REQUIRE(b >= 0 && n > 0 && xyz && temp && idx, "fps: bad arguments (b=%d n=%d)", b, n);
    if (m <= 0 || b == 0) return 0;
    if (m > n || m < 2)   // nothing to prove / not a prefix: the ordinary path
        return fps_run(b, n, m, xyz, temp, idx, new_xyz, workspace, workspace_bytes, stream, nullptr);
    PRB_REQUIRE(workspace && workspace_bytes >= prb_fps_ordered_workspace_bytes(b, n, m), "fps (ordered): workspace of %zu bytes is too small",
                workspace_bytes);
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    char *w = reinterpret_cast<char *>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    int *todo = reinterpret_cast<int *>(w);                              w += up((size_t)b * sizeof(int));
    float *v = reinterpret_cast<float *>(w);                             w += up((size_t)b * m * sizeof(float));
    float *rtemp = reinterpret_cast<float *>(w);                         w += up((size_t)b * n * sizeof(float));
    const size_t rest = workspace_bytes - (size_t)(w - reinterpret_cast<char *>(workspace));
    cudaStream_t st = (cudaStream_t)stream;
    fps_prefix_v_kernel<<<dim3(ceil_div(m, 32), b), 128, 0, st>>>(n, m, xyz, temp, v, todo);
    if (int rc = check_launch("fps_prefix_v_kernel")) return rc;
    int logS = 0;
    while ((2 << logS) <= n && logS < 10) ++logS;       // the sampling kernels' tie rule: reference rank of a point (fps_run)
    fps_prefix_check_kernel<<<dim3(ceil_div(n, 256), b), 256, 0, st>>>(n, m, xyz, temp, v, rtemp, todo, 1 << logS, logS, ceil_div(n, 1 << logS));
    if (int rc = check_launch("fps_prefix_check_kernel")) return rc;
    fps_prefix_emit_kernel<<<dim3(ceil_div(n, 256), b), 256, 0, st>>>(n, m, xyz, rtemp, todo, temp, idx, new_xyz);
    if (int rc = check_launch("fps_prefix_emit_kernel")) return rc;
    if (todo_out) PRB_CUDA(cudaMemcpyAsync(todo_out, todo, (size_t)b * sizeof(int), cudaMemcpyDeviceToDevice, st));
    return fps_run(b, n, m, xyz, temp, idx, new_xyz, w, rest, stream, todo);
}
