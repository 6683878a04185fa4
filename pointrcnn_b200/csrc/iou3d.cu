// iou3d.cu -- rotated BEV overlap / IoU matrices and bitmask NMS with an on-device greedy scan.
//
// Replaces boxes_overlap_bev_gpu / boxes_iou_bev_gpu / nms_gpu / nms_normal_gpu
// (lib/utils/iou3d/src/iou3d.cpp:31-170 -> iou3d_kernel.cu:223-387).
//
// The overlap arithmetic IS the spec (keep masks are compared bit-exactly): corners rotated about the
// box centre, 4x4 edge intersections (bbox reject, straddle test, line solve with an EPS fallback),
// corners of one box inside the other (MARGIN 1e-5), centroid, bubble sort by atan2f, fan area / 2.0
// (iou3d_kernel.cu:34-212).  What changes is everything around it:
//   * NMS computes only the upper-triangle 64x64 tiles (the scan never reads the others),
//   * the suppression mask never leaves the device: one CTA runs the greedy scan 64 boxes at a time
//     (serial resolve on the diagonal word, then a parallel OR of the kept rows into the remaining
//     columns) and emits the kept indices + count; no cudaMalloc, no 5 MB D2H, no host loop,
//   * everything runs on the caller's stream.
#include "common.cuh"
#include "iou3d_dev.cuh"

namespace prb {

// ---------------------------------------------------------------- pairwise matrices
// 16 x 16 pairs per CTA; the 32 boxes of the tile are precomputed once (BoxPre: centre, cos/sin, rotated corners), the
// intersection polygon of each pair lives in a shared-memory column of its thread (no local memory).
constexpr int PM_T = 16;
// the reference's cp[16].  The algorithm counts edge crossings and corners separately, so with rounding it can count more
// than the 8 vertices an exact intersection has: near-parallel and near-duplicate pairs reach exactly 16 in the
// CPU oracle (tests/test_cpu_iou_geometry.py); none of the generated pairs exceeds it, but no proof bounds the count by 16
constexpr int POLY_SLOTS = 16;
template <bool IOU>
__global__ void __launch_bounds__(PM_T * PM_T) pair_matrix_kernel(int num_a, const float *__restrict__ boxes_a, int num_b,
                                                                  const float *__restrict__ boxes_b, float *__restrict__ out) {
    extern __shared__ float s_poly[];                     // 3 x POLY_SLOTS x 256 floats
    __shared__ BoxPre sa[PM_T], sb[PM_T];
    const int a0 = blockIdx.y * PM_T, b0 = blockIdx.x * PM_T;
    const int t = threadIdx.y * PM_T + threadIdx.x;
    if (t < PM_T) {
        if (a0 + t < num_a) box_pre(boxes_a + (size_t)(a0 + t) * 5, sa[t]);
    } else if (t < 2 * PM_T) {
        if (b0 + t - PM_T < num_b) box_pre(boxes_b + (size_t)(b0 + t - PM_T) * 5, sb[t - PM_T]);
    }
    __syncthreads();
    const int ai = a0 + threadIdx.y, bi = b0 + threadIdx.x;
    if (ai >= num_a || bi >= num_b) return;
    constexpr int NT = PM_T * PM_T;
    float *px = s_poly + t, *py = px + POLY_SLOTS * NT, *pa = py + POLY_SLOTS * NT;
    out[(size_t)ai * num_b + bi] = IOU ? iou_bev_pre(sa[threadIdx.y], sb[threadIdx.x], px, py, pa, NT)
                                       : box_overlap_pre(sa[threadIdx.y], sb[threadIdx.x], px, py, pa, NT);
}

// ---------------------------------------------------------------- NMS mask (upper-triangle tiles)
// One CTA of 8 warps per RT x 64 tile (RT rows, one 64-column mask word per row).  Warp w takes rows w, w+8, ...; lane l tests
// columns l and l+32 of the row and two ballots assemble the 64-bit mask word (the reference and the round-1 kernel: one
// thread per row, 64 pairs in sequence).  Rotated: the boxes of the tile are precomputed once; axis-aligned: plain extents.
// RT = 64 for the cheap axis-aligned test.  RT = 8 for the rotated test (one row per warp, two polygon clippings per
// thread): with 64-row tiles a thread clipped 16 polygons in sequence and N = 1000 gave only 136 busy CTAs;
// short tiles trade 72 box precomputations per 512 pairs for 8x the CTAs.
constexpr int NM_THREADS = 256;
template <bool NORMAL, int RT>
__global__ void __launch_bounds__(NM_THREADS) nms_mask_kernel(int n, float thresh, const float *__restrict__ boxes,
                                                              unsigned long long *__restrict__ mask) {
    extern __shared__ float s_poly[];                     // rotated only: 3 x POLY_SLOTS x 256 floats
    __shared__ BoxPre cpre[NORMAL ? 1 : 64], rpre[NORMAL ? 1 : RT];
    __shared__ float cbx[NORMAL ? 64 * 5 : 1], rbx[NORMAL ? RT * 5 : 1];
    const int col_blk = blockIdx.x;
    const int row0 = blockIdx.y * RT, col0 = col_blk * 64;
    const int col_blocks = ceil_div(n, 64);
    const int row_size = min(n - row0, RT), col_size = min(n - col0, 64);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (row0 >= col0 + 64) {  // every row lies behind every column: never read by the scan; keep the buffer defined
        if (tid < row_size) mask[(size_t)(row0 + tid) * col_blocks + col_blk] = 0ull;
        return;
    }
    if (NORMAL) {
        for (int i = tid; i < col_size * 5; i += NM_THREADS) cbx[i] = boxes[(size_t)col0 * 5 + i];
        for (int i = tid; i < row_size * 5; i += NM_THREADS) rbx[i] = boxes[(size_t)row0 * 5 + i];
    } else {
        if (tid < col_size) box_pre(boxes + (size_t)(col0 + tid) * 5, cpre[tid]);
        else if (tid >= 64 && tid - 64 < row_size) box_pre(boxes + (size_t)(row0 + tid - 64) * 5, rpre[tid - 64]);
    }
    __syncthreads();
    float *px = s_poly + tid, *py = px + POLY_SLOTS * NM_THREADS, *pa = py + POLY_SLOTS * NM_THREADS;
    for (int r = warp; r < row_size; r += NM_THREADS / 32) {
        const int start = row0 + r + 1 - col0;                      // only columns behind the row (<= 0 above the diagonal)
        bool hit[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = lane + 32 * h;
            hit[h] = false;
            if (c >= start && c < col_size) {
                const float v = NORMAL ? iou_normal(rbx + r * 5, cbx + c * 5) : iou_bev_pre(rpre[r], cpre[c], px, py, pa, NM_THREADS);
                hit[h] = v > thresh;
            }
        }
        const unsigned lo = __ballot_sync(0xffffffffu, hit[0]), hi = __ballot_sync(0xffffffffu, hit[1]);
        if (lane == 0) mask[(size_t)(row0 + r) * col_blocks + col_blk] = ((unsigned long long)hi << 32) | lo;
    }
}

// ---------------------------------------------------------------- greedy scan on the device
// Same recurrence as the host loop of iou3d.cpp:100-116: box i is kept iff bit i of remv is clear;
// a kept box ORs its mask row into remv (columns >= its own block).
// One CTA walks the 64-box blocks in order.  The 64 mask rows of the NEXT block are prefetched into shared memory
// with cp.async while the current block is resolved (serial pass over its diagonal word by one thread, then a
// parallel OR of the kept rows into the remaining columns, all from shared memory).
constexpr int SCAN_THREADS = 256;
__device__ __forceinline__ void scan_cp_async8(uint32_t dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
__global__ void __launch_bounds__(SCAN_THREADS) nms_scan_kernel(int n, const unsigned long long *__restrict__ mask,
                                                                long long *__restrict__ keep, int *__restrict__ num_out) {
    extern __shared__ unsigned long long s_dyn[];   // remv[cb] then two row tiles of 64 x cb words
    __shared__ unsigned long long s_kept;
    __shared__ int s_num;
    const int tid = threadIdx.x;
    const int cb = ceil_div(n, 64);
    unsigned long long *s_remv = s_dyn;
    unsigned long long *s_tile[2] = {s_dyn + cb, s_dyn + cb + (size_t)64 * cb};
    for (int j = tid; j < cb; j += SCAN_THREADS) s_remv[j] = 0ull;
    if (tid == 0) s_num = 0;
    auto prefetch = [&](int bi, int buf) {   // rows bi*64.., columns bi..cb-1 (the only ones the scan reads)
        const int rows = min(64, n - bi * 64), cols = cb - bi;
        for (int e = tid; e < rows * cols; e += SCAN_THREADS) {
            const int t = e / cols, j = bi + e - t * cols;
            scan_cp_async8((uint32_t)__cvta_generic_to_shared(s_tile[buf] + (size_t)t * cb + j), mask + (size_t)(bi * 64 + t) * cb + j);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if (cb > 0) prefetch(0, 0);
    for (int bi = 0; bi < cb; ++bi) {
        const int buf = bi & 1;
        if (bi + 1 < cb) {
            prefetch(bi + 1, buf ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const unsigned long long *tile = s_tile[buf];
        const int lim = min(64, n - bi * 64);
        if (tid < 32) {
            // The block's 64 boxes are resolved by ONE WARP as a fixed point instead of a 64-step serial walk: with d_t = row t's
            // diagonal word (bits > t only), the greedy answer is the unique K with  K = alive & ~OR_{t in K} d_t.  Iterating
            // K <- alive & ~OR_{t in K} d_t from K = alive fixes bit b after at most b rounds (bit b depends on bits < b only),
            // i.e. after (longest suppression chain + 1) rounds -- 2 to 4 for real box sets -- of two selects and two REDUX.OR.
            const int lane = tid;
            const unsigned long long valid = lim == 64 ? ~0ull : ((1ull << lim) - 1ull);
            const unsigned long long dlo = lane < lim ? tile[(size_t)lane * cb + bi] : 0ull;
            const unsigned long long dhi = lane + 32 < lim ? tile[(size_t)(lane + 32) * cb + bi] : 0ull;
            const unsigned long long alive = ~s_remv[bi] & valid;
            unsigned long long kept = alive, prev;
            do {
                prev = kept;
                const unsigned long long x = (((kept >> lane) & 1ull) ? dlo : 0ull) | (((kept >> (lane + 32)) & 1ull) ? dhi : 0ull);
                const unsigned lo = __reduce_or_sync(0xffffffffu, (unsigned)x);
                const unsigned hi = __reduce_or_sync(0xffffffffu, (unsigned)(x >> 32));
                kept = alive & ~(((unsigned long long)hi << 32) | lo);
            } while (kept != prev);
            const int num = s_num;
            if ((kept >> lane) & 1ull) keep[num + __popcll(kept & ((1ull << lane) - 1ull))] = (long long)bi * 64 + lane;
            if ((kept >> (lane + 32)) & 1ull) keep[num + __popcll(kept & ((1ull << (lane + 32)) - 1ull))] = (long long)bi * 64 + lane + 32;
            __syncwarp();
            if (lane == 0) { s_num = num + __popcll(kept); s_kept = kept; }
        }
        __syncthreads();
        const unsigned long long kept = s_kept;
        for (int j = bi + 1 + tid; j < cb; j += SCAN_THREADS) {
            unsigned long long acc = s_remv[j];
            for (unsigned long long k = kept; k; k &= k - 1ull)          // kept rows only
                acc |= tile[(size_t)(__ffsll((long long)k) - 1) * cb + j];
            s_remv[j] = acc;
        }
        __syncthreads();   // tile[buf] is overwritten by the prefetch of block bi+2
    }
    if (tid == 0) *num_out = s_num;
}

// fallback for very large n (the prefetched tiles no longer fit shared memory): same recurrence, mask rows read
// straight from global memory
__global__ void __launch_bounds__(SCAN_THREADS) nms_scan_global_kernel(int n, const unsigned long long *__restrict__ mask,
                                                                       long long *__restrict__ keep, int *__restrict__ num_out) {
    extern __shared__ unsigned long long s_remv[];  // col_blocks words
    __shared__ unsigned long long s_diag[64];
    __shared__ unsigned long long s_kept;
    __shared__ int s_num;
    const int tid = threadIdx.x;
    const int cb = ceil_div(n, 64);
    for (int j = tid; j < cb; j += SCAN_THREADS) s_remv[j] = 0ull;
    if (tid == 0) s_num = 0;
    __syncthreads();
    for (int bi = 0; bi < cb; ++bi) {
        if (tid < 64) { const int i = bi * 64 + tid; s_diag[tid] = i < n ? mask[(size_t)i * cb + bi] : 0ull; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long cur = s_remv[bi], kept = 0ull;
            const int lim = min(64, n - bi * 64);
            const unsigned long long valid = lim == 64 ? ~0ull : ((1ull << lim) - 1ull);
            unsigned long long alive = ~cur & valid;
            int num = s_num;
            while (alive) {
                const int t = __ffsll((long long)alive) - 1;
                kept |= 1ull << t;
                keep[num++] = (long long)bi * 64 + t;
                cur |= s_diag[t];
                alive = ~cur & valid & ~((2ull << t) - 1ull);
            }
            s_num = num;
            s_kept = kept;
        }
        __syncthreads();
        const unsigned long long kept = s_kept;
        for (int j = bi + 1 + tid; j < cb; j += SCAN_THREADS) {
            unsigned long long acc = s_remv[j];
#pragma unroll 8
            for (int t = 0; t < 64; ++t)
                if ((kept >> t) & 1ull) acc |= mask[(size_t)(bi * 64 + t) * cb + j];
            s_remv[j] = acc;
        }
        __syncthreads();
    }
    if (tid == 0) *num_out = s_num;
}

// ---------------------------------------------------------------- fused 3D IoU (boxes_iou3d_gpu in one launch)
// lib/utils/iou3d/iou3d_utils.py:21-53 runs: 2 x boxes3d_to_bev (kitti_utils.py:134-147), the overlap kernel, ~12 small
// torch kernels for the height overlap / volumes / division -- and lib/rpn/proposal_target_layer.py calls that once per
// scene for (RoIs x GTs) and up to 10 times per RoI for single pairs (:104, :232).  Here one thread per pair does all of
// it; every torch op of the reference is one fp32 rounding here too (explicit _rn intrinsics: no FMA contraction), so
// the values equal the reference's op sequence on its own overlap kernel bit for bit.
//   mode 0: matrix, out[s][i][j] = iou(a[s][i], b[s][j]) for s < batch; mode 1: aligned pairs, out[k] = iou(a[k], b[k])
// (the per-pair arithmetic, box7_to_bev / iou3d_pair, is in iou3d_dev.cuh)
__global__ void __launch_bounds__(128) iou3d_kernel(int mode, int batch, int na, int nb, const float *__restrict__ boxes_a,
                                                    const float *__restrict__ boxes_b, float *__restrict__ out) {
    __shared__ float s_poly[3 * POLY_SLOTS * 128];
    float *px = s_poly + threadIdx.x, *py = px + POLY_SLOTS * 128, *pa = py + POLY_SLOTS * 128;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    float a[7], b[7];
    if (mode == 1) {
        if (t >= na) return;
#pragma unroll
        for (int q = 0; q < 7; ++q) { a[q] = boxes_a[t * 7 + q]; b[q] = boxes_b[t * 7 + q]; }
        out[t] = iou3d_pair(a, b, px, py, pa, 128);
        return;
    }
    const long per = (long)na * nb;
    if (t >= per * batch) return;
    const long s = t / per, e = t - s * per;
    const long i = e / nb, j = e - i * nb;
#pragma unroll
    for (int q = 0; q < 7; ++q) { a[q] = boxes_a[(s * na + i) * 7 + q]; b[q] = boxes_b[(s * nb + j) * 7 + q]; }
    out[t] = iou3d_pair(a, b, px, py, pa, 128);
}

}  // namespace prb

using namespace prb;

extern "C" int prb_boxes_iou3d(int batch, int na, const float *boxes_a, int nb, const float *boxes_b, float *out, void *stream) {
    PRB_REQUIRE(batch >= 0 && na >= 0 && nb >= 0 && boxes_a && boxes_b && out, "boxes_iou3d: bad arguments");
    const long total = (long)batch * na * nb;
    if (total == 0) return 0;
    iou3d_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>(0, batch, na, nb, boxes_a, boxes_b, out);
    return check_launch("iou3d_kernel");
}
extern "C" int prb_boxes_iou3d_aligned(int n, const float *boxes_a, const float *boxes_b, float *out, void *stream) {
    PRB_REQUIRE(n >= 0 && boxes_a && boxes_b && out, "boxes_iou3d_aligned: bad arguments");
    if (n == 0) return 0;
    iou3d_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(1, 1, n, 1, boxes_a, boxes_b, out);
    return check_launch("iou3d_kernel");
}

static int pair_matrix(bool iou, int na, const float *a, int nb, const float *b, float *out, void *stream) {
    PRB_REQUIRE(na >= 0 && nb >= 0 && a && b && out, "boxes matrix: bad arguments");
    if (na == 0 || nb == 0) return 0;
    dim3 grid(ceil_div(nb, PM_T), ceil_div(na, PM_T)), block(PM_T, PM_T);
    const size_t smem = (size_t)3 * POLY_SLOTS * PM_T * PM_T * sizeof(float);      // 48 KB
    if (iou) {
        PRB_CUDA(cudaFuncSetAttribute(pair_matrix_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        pair_matrix_kernel<true><<<grid, block, smem, (cudaStream_t)stream>>>(na, a, nb, b, out);
    } else {
        PRB_CUDA(cudaFuncSetAttribute(pair_matrix_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        pair_matrix_kernel<false><<<grid, block, smem, (cudaStream_t)stream>>>(na, a, nb, b, out);
    }
    return check_launch("pair_matrix_kernel");
}

extern "C" int prb_boxes_overlap_bev(int na, const float *a, int nb, const float *b, float *out, void *stream) {
    return pair_matrix(false, na, a, nb, b, out, stream);
}
extern "C" int prb_boxes_iou_bev(int na, const float *a, int nb, const float *b, float *out, void *stream) {
    return pair_matrix(true, na, a, nb, b, out, stream);
}

extern "C" int prb_nms_mask(const float *boxes, int n, float thresh, int normal, unsigned long long *mask, void *stream) {
    PRB_REQUIRE(n >= 0 && boxes && mask, "nms_mask: bad arguments");
    if (n == 0) return 0;
    const int cb = ceil_div(n, 64);
    if (normal) {
        nms_mask_kernel<true, 64><<<dim3(cb, cb), NM_THREADS, 0, (cudaStream_t)stream>>>(n, thresh, boxes, mask);
    } else {
        constexpr int RT = 8;
        const size_t smem = (size_t)3 * POLY_SLOTS * NM_THREADS * sizeof(float);    // 48 KB of polygon scratch
        PRB_CUDA(cudaFuncSetAttribute(nms_mask_kernel<false, RT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        nms_mask_kernel<false, RT><<<dim3(cb, ceil_div(n, RT)), NM_THREADS, smem, (cudaStream_t)stream>>>(n, thresh, boxes, mask);
    }
    return check_launch("nms_mask_kernel");
}

extern "C" size_t prb_nms_workspace_bytes(int n) {
    if (n <= 0) return 256;
    const size_t cb = (size_t)ceil_div(n, 64);
    return (size_t)n * cb * 8 + (size_t)n * 8 + 256;
}

extern "C" int prb_nms_device(const float *boxes, int n, float thresh, int normal, long long *keep_dev, int *num_dev,
                              void *workspace, void *stream) {
    PRB_REQUIRE(n >= 0 && keep_dev && num_dev && workspace && (n == 0 || boxes), "nms: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        PRB_CUDA(cudaMemsetAsync(num_dev, 0, sizeof(int), st));
        return 0;
    }
    unsigned long long *mask = (unsigned long long *)workspace;
    int rc = prb_nms_mask(boxes, n, thresh, normal, mask, stream);
    if (rc) return rc;
    const size_t cbs = (size_t)ceil_div(n, 64);
    const size_t smem = (cbs + 2 * 64 * cbs) * 8;   // remv + two prefetched row tiles
    if (smem > 220 * 1024) {                        // > ~13.6k boxes: rows straight from global memory
        const size_t smem_g = cbs * 8;
        PRB_REQUIRE(smem_g <= 200 * 1024, "nms: %d boxes exceed the single-CTA scan capacity", n);
        if (smem_g > 48 * 1024) PRB_CUDA(cudaFuncSetAttribute(nms_scan_global_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g));
        nms_scan_global_kernel<<<1, SCAN_THREADS, smem_g, st>>>(n, mask, keep_dev, num_dev);
        return check_launch("nms_scan_global_kernel");
    }
    if (smem > 48 * 1024) PRB_CUDA(cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    nms_scan_kernel<<<1, SCAN_THREADS, smem, st>>>(n, mask, keep_dev, num_dev);
    return check_launch("nms_scan_kernel");
}

extern "C" int prb_nms_host(const float *boxes, int n, float thresh, int normal, long long *keep_host, int *num_out,
                            void *workspace, void *stream) {
    PRB_REQUIRE(n >= 0 && keep_host && num_out && workspace, "nms: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    *num_out = 0;
    if (n == 0) return 0;
    const size_t cb = (size_t)ceil_div(n, 64);
    char *ws = (char *)workspace;
    long long *keep_dev = (long long *)(ws + (size_t)n * cb * 8);
    int *num_dev = (int *)(ws + (size_t)n * cb * 8 + (size_t)n * 8);
    int rc = prb_nms_device(boxes, n, thresh, normal, keep_dev, num_dev, workspace, stream);
    if (rc) return rc;
    // like the reference (iou3d.cpp:105-116) only keep_host[0 .. num_out) is written: count first, then that many indices
    PRB_CUDA(cudaMemcpyAsync(num_out, num_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
    PRB_CUDA(cudaStreamSynchronize(st));
    if (*num_out > 0) {
        PRB_CUDA(cudaMemcpyAsync(keep_host, keep_dev, (size_t)*num_out * 8, cudaMemcpyDeviceToHost, st));
        PRB_CUDA(cudaStreamSynchronize(st));
    }
    return 0;
}
