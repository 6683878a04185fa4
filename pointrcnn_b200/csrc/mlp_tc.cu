// mlp_tc.cu -- the per-group / per-point shared MLP as a wgmma (Hopper tensor core) layer chain.
//
// Replaces, for eval-mode forward, everything between the ball query and the next level's features:
//   grouping_operation x2 + cat + SharedMLP (Conv2d 1x1 -> BN -> ReLU) x L + max_pool2d
//     (pointnet2_lib/pointnet2/pointnet2_utils.py:249-257, pointnet2_modules.py:40-52, pytorch_utils.py:5-101)
//   three_interpolate + cat + SharedMLP x L
//     (pointnet2_modules.py:144-156)
// The reference materialises every (B,C,npoint,nsample) tensor in HBM between ~10 library kernels per
// scale; here a 64-row tile never leaves the SM between its gather and its pooled output.
//
// Two kernels run a fused launch (layers of a chain at most 256 wide); they share the tile stages -- the row lookup, the
// layer-0 gather, the inner-layer epilogue and the final epilogues -- issue the same MMA sequence per K chunk, and give
// bit-identical outputs.  launch_chain picks one by shape:
//   resident   every layer <= 128 wide; input / output one of SA -> max-pool, FP -> FP, rows -> rows; the packed weight
//              image at most half of a CTA's shared memory; prb_options.mlp_resident != 0 (the default).
//   streaming  every other fused launch.
// A layer wider than 256 runs alone on a third kernel, mlp_wide_kernel, as a dense GEMM over rows in global memory
// (see there), with the same K order, k8 steps and epilogues.
//
// Resident kernel (mlp_resident_kernel; persistent CTAs of nwg warpgroups, no producer warp): at CTA start one thread
// loads the segment's whole packed image with cp.async.bulk on one mbarrier, which every warpgroup waits on once.  Each
// warpgroup then runs its own 64-row tiles (strided over the grid; the tiles of a pooled SA centre stay together)
// through every layer at full width -- one m64n(np)k8 instruction per K=8 step -- in a private work region (layer-0 A
// slots -> activations -> per-warp pool maxima), synchronising only on its own named barrier, so one warpgroup's
// gather and epilogues overlap another's MMAs.  Where every layer is at most 64 wide, a warpgroup runs tiles 2u and
// 2u + 1 together: two row tables and work regions, two MMAs on the same B descriptor per K step in one commit group,
// and one drain, barrier and epilogue pass per layer for the 128 rows -- the serial steps of a narrow tile are short, so
// the pair halves their count per row.  The B operand of chunk kc of layer l is the image at the layer's offset
// + kc * np * 128 bytes.  Warpgroups per CTA and CTAs per SM are the pair the occupancy calculator allows the most
// warpgroups per SM for (registers: 128 for 32-wide pairs and single tiles, 168 for 64-wide pairs).
//
// Streaming kernel (mlp_chain_kernel; persistent CTAs over 64-row tiles; rows = (centre, sample) pairs or points):
//   warpgroups 0, 1  gather layer 0's A operand chunk by chunk (32 K-columns = one 128-byte swizzle row) into a
//                    ring of three shared-memory slots, issue wgmma tf32 with fp32 register accumulators -- the
//                    layer's output columns are split between the two warpgroups, and each warpgroup covers its
//                    nsub * 32 columns with ONE m64n(32 nsub)k8 instruction per K=8 step, so the A slice is read
//                    from shared memory once per step -- and run the epilogues: layer l < L-1 writes
//                    relu(acc + shift) as tf32 into the resident activation buffer (the next layer's A operand, all
//                    of its K chunks), the last layer pools / stores.
//                    A chunk's MMAs are one commit group and stay in flight: the warpgroup waits for the previous
//                    chunk's group only (wgmma_wait<1>), then releases that chunk's weight stage and gathers the
//                    next chunk while the current one runs.  The whole layer is drained before its epilogue.
//   warp 8           weight producer: one thread streams pre-packed weight chunks (already in the K-major
//                    SWIZZLE_128B image, see prb_mlp_pack_weights) with cp.async.bulk + mbarrier transaction counts.
// Where the widest layer is 129-256 wide and a three-stage weight ring still fits beside two work regions (the SA3
// chains of the RPN), a CTA runs tiles 2u and 2u + 1 together (T = 2): warpgroup s gathers tile s's row table and layer-0
// chunks (all of a chunk's loads in flight at once), then each warpgroup issues two MMAs on the same B descriptor per K step for its column half of both tiles, and
// the two tiles share every drain, barrier and epilogue pass.  The producer streams each chunk once per pair, so the L2
// weight traffic halves.  The 128 accumulators per thread need more than the 168 registers 9 warps allow, so there the
// producer is a whole warpgroup that hands its registers to the MMA warpgroups (setmaxnreg).  launch_chain holds the
// per-launch timings the rule follows.
// Chains with a layer wider than 256, or whose activation buffer and weight stages do not fit in shared memory, are split
// into several launches by the host wrapper (rows materialised in between).
// Precision: operands are rounded to TF32 (cvt.rn), products accumulate in fp32 -- the same contract as the
// reference's cuDNN convolutions under torch's default allow_tf32=True (SURVEY.md 8c).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <string.h>

#include <vector>

#include "mlp_dev.cuh"

namespace prb {

// ------------------------------------------------------------------------------------------------ kernel
// element l of a per-layer parameter array, by selects: indexing the kernel parameter with a runtime l would copy
// the array to local memory
template <typename T>
__device__ __forceinline__ T per_layer(const T (&a)[MAX_LAYERS], int l) {
    static_assert(MAX_LAYERS == 3, "per_layer: one select per layer");
    return l == 0 ? a[0] : l == 1 ? a[1] : a[2];
}

// The MMAs of one K chunk over a warpgroup's nsub * 32 output columns, for T 64-row tiles that share the B operand: per
// K=8 step, one m64n(32*NSUB)k8 instruction per tile, KSTEPS steps in K order, straight-line.  nsub and ksteps are
// warp-uniform and select the sequence before the first wgmma, so no predicate sits between wgmma_fence and wgmma_commit
// (a divergent one makes ptxas serialise every wgmma behind its own arrive / wait).
template <int NSUB, int KSTEPS, int NS, int T>
__device__ __forceinline__ void mma_steps(float (&acc)[T][16 * NS], const uint64_t (&adesc)[T], uint64_t bdesc,
                                          uint32_t accumulate) {
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks)
#pragma unroll
        for (int s = 0; s < T; ++s)
            wgmma_tf32<NSUB, NS>(acc[s], adesc[s] + (uint64_t)(2 * ks), bdesc + (uint64_t)(2 * ks), ks > 0 ? 1u : accumulate);
}
template <int NSUB, int NS, int T>
__device__ __forceinline__ void mma_chunk_n(float (&acc)[T][16 * NS], int ksteps, const uint64_t (&adesc)[T], uint64_t bdesc,
                                            uint32_t accumulate) {
    static_assert(KC / 8 == 4, "mma_chunk_n: one case per K=8 step of a chunk");
    switch (ksteps) {   // fewer than 4 only for the last chunk of a layer-0 segment (the rest of the chunk is padding)
        case 1: mma_steps<NSUB, 1, NS, T>(acc, adesc, bdesc, accumulate); break;
        case 2: mma_steps<NSUB, 2, NS, T>(acc, adesc, bdesc, accumulate); break;
        case 3: mma_steps<NSUB, 3, NS, T>(acc, adesc, bdesc, accumulate); break;
        default: mma_steps<NSUB, 4, NS, T>(acc, adesc, bdesc, accumulate); break;
    }
}
template <int NS, int T>
__device__ __forceinline__ void mma_chunk(float (&acc)[T][16 * NS], int nsub, int ksteps, const uint64_t (&adesc)[T],
                                          uint64_t bdesc, uint32_t accumulate) {
    // both are warp-uniform already; the broadcast keeps ptxas from losing track of that under register pressure
    nsub = __shfl_sync(0xffffffffu, nsub, 0);
    ksteps = __shfl_sync(0xffffffffu, ksteps, 0);
    switch (nsub) {
        case 1: mma_chunk_n<1, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 2: if constexpr (NS >= 2) mma_chunk_n<2, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 3: if constexpr (NS >= 3) mma_chunk_n<3, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 4: if constexpr (NS >= 4) mma_chunk_n<4, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 5: if constexpr (NS >= 5) mma_chunk_n<5, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 6: if constexpr (NS >= 6) mma_chunk_n<6, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 7: if constexpr (NS >= 7) mma_chunk_n<7, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        case 8: if constexpr (NS >= 8) mma_chunk_n<8, NS, T>(acc, ksteps, adesc, bdesc, accumulate); break;
        default: break;   // the warpgroup owns no columns of this layer (np = 32: all of them go to warpgroup 0)
    }
}

// ------------------------------------------------------------------------------------------------ tile stages
// The stages of a tile that do not depend on how the weights reach shared memory, shared by both kernels.  NT is the
// number of threads that run a stage together (the streaming kernel's two warpgroups: 256; one resident warpgroup: 128),
// t the thread's index among them.

// the tile's source rows (threads t < TM)
__device__ __forceinline__ void load_tile_rows(const ChainParams &p, int tile, int t, TileRows &M) {
    if (t >= TM) return;
    const long R = (long)tile * TM + t;
    const bool valid = R < p.total_rows;
    int src[3] = {0, 0, 0};
    float aux[3] = {0.f, 0.f, 0.f};
    if (p.mode_in == IN_SA) {
        const long pr = valid ? (R >> p.log_ns) : 0;      // global centre index (nsample is a power of two)
        const int scene = (int)(pr / p.npoint);
        src[0] = scene * p.n + (valid ? __ldg(p.idx + R) : 0);
#pragma unroll
        for (int q = 0; q < 3; ++q) aux[q] = __ldg(p.new_xyz + (size_t)pr * 3 + q);
    } else if (p.mode_in == IN_FP) {
        const long rr = valid ? R : 0;
        const int scene = (int)(rr / p.n);
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            src[q] = scene * p.m + __ldg(p.idx + (size_t)rr * 3 + q);
            aux[q] = __ldg(p.weight + (size_t)rr * 3 + q);
        }
    }
    M.valid[t] = valid;
#pragma unroll
    for (int q = 0; q < 3; ++q) { M.src[t][q] = src[q]; M.aux[t][q] = aux[q]; }
}

// gather K chunk kc of the tile's layer-0 input rows, rounded to tf32, into the A chunk at A; returns the K=8 steps that
// hold data (the rest of the chunk is padding).  STEPS: row steps of a point-major segment whose loads are in flight
// together (TM / (STEPS * NT / 8) dependent batches per chunk)
template <int NT, int STEPS = 2>
__device__ __forceinline__ int gather_chunk(const ChainParams &p, int tile, int kc, int t, const TileRows &M, uint8_t *A) {
    static_assert(NT == 128 || NT == 256, "gather_chunk: one or two warpgroups");
    int c = kc, seg = 0;
    if (p.nseg > 1 && c >= p.seg_chunks[0]) { c -= p.seg_chunks[0]; seg = 1; }
    const int k0 = c * KC;                         // first column of this chunk inside its segment
    const int width = seg ? p.seg_width[1] : p.seg_width[0];
    const int ksteps = (min(KC, width - k0) + 7) >> 3;
    const bool rows_seg = (p.mode_in == IN_DIRECT) || (p.mode_in == IN_SA && seg == 0 && p.c_feat > 5) ||
                          (p.mode_in == IN_FP && seg == 0);
    if (rows_seg) {
        // point-major sources: 8 threads cover one row's 128 bytes, NT threads NT/8 rows per step, STEPS steps in flight
        constexpr int RS = NT / 8;
        static_assert(TM % (STEPS * RS) == 0, "gather_chunk: whole batches of rows");
        const int j8 = t & 7, kk = k0 + 4 * j8;
#pragma unroll 1
        for (int r0 = 0; r0 < TM; r0 += STEPS * RS) {
            float4 v[STEPS];
            if (p.mode_in == IN_FP) {
                const int C = p.c_known;
                const bool vec = (C & 3) == 0;
#pragma unroll
                for (int i = 0; i < STEPS; ++i) {
                    const int rr = r0 + (t >> 3) + RS * i;
                    float4 t0 = make_float4(0.f, 0.f, 0.f, 0.f), t1 = t0, t2 = t0;
                    const float w0 = M.aux[rr][0], w1 = M.aux[rr][1], w2 = M.aux[rr][2];
                    if (M.valid[rr] && kk < width) {
                        const float *s0 = p.known_pm + (size_t)M.src[rr][0] * C + kk;
                        const float *s1 = p.known_pm + (size_t)M.src[rr][1] * C + kk;
                        const float *s2 = p.known_pm + (size_t)M.src[rr][2] * C + kk;
                        if (vec) {
                            t0 = __ldg((const float4 *)s0); t1 = __ldg((const float4 *)s1); t2 = __ldg((const float4 *)s2);
                        } else {
                            float a0[4], a1[4], a2[4];
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const bool in = kk + q < width;
                                a0[q] = in ? __ldg(s0 + q) : 0.f; a1[q] = in ? __ldg(s1 + q) : 0.f; a2[q] = in ? __ldg(s2 + q) : 0.f;
                            }
                            t0 = make_float4(a0[0], a0[1], a0[2], a0[3]);
                            t1 = make_float4(a1[0], a1[1], a1[2], a1[3]);
                            t2 = make_float4(a2[0], a2[1], a2[2], a2[3]);
                        }
                    }
                    // same contraction as three_interpolate (reference SASS): fma(w2,p2, fma(w0,p0, w1*p1))
                    v[i].x = __fmaf_rn(w2, t2.x, __fmaf_rn(w0, t0.x, __fmul_rn(w1, t1.x)));
                    v[i].y = __fmaf_rn(w2, t2.y, __fmaf_rn(w0, t0.y, __fmul_rn(w1, t1.y)));
                    v[i].z = __fmaf_rn(w2, t2.z, __fmaf_rn(w0, t0.z, __fmul_rn(w1, t1.z)));
                    v[i].w = __fmaf_rn(w2, t2.w, __fmaf_rn(w0, t0.w, __fmul_rn(w1, t1.w)));
                }
            } else {
                const float *srcb = p.mode_in == IN_DIRECT ? (seg ? p.x2_rows : p.x_rows) : p.feats_pm;
                const int pitch = p.mode_in == IN_DIRECT ? (seg ? p.x2_pitch : p.x_pitch) : p.c_feat;
                // a 128-bit load only where the whole group of 4 columns lies inside the segment: a direct-rows segment may
                // be narrower than its pitch, and the columns past it must not be read (0 * NaN would reach the output)
                const bool vec = (pitch & 3) == 0 && (reinterpret_cast<uintptr_t>(srcb) & 15) == 0 && kk + 4 <= width;
#pragma unroll
                for (int i = 0; i < STEPS; ++i) {
                    const int rr = r0 + (t >> 3) + RS * i;
                    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (M.valid[rr] && kk < width) {
                        const size_t row = p.mode_in == IN_DIRECT ? (size_t)tile * TM + rr : (size_t)M.src[rr][0];
                        const float *src = srcb + row * pitch + kk;
                        if (vec) {
                            v[i] = __ldg((const float4 *)src);
                        } else {
                            float o[4];
#pragma unroll
                            for (int q = 0; q < 4; ++q) o[q] = (kk + q < width) ? __ldg(src + q) : 0.f;
                            v[i] = make_float4(o[0], o[1], o[2], o[3]);
                        }
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < STEPS; ++i) {
                const int rr = r0 + (t >> 3) + RS * i;
                *reinterpret_cast<float4 *>(A + swz(rr, j8)) =
                    make_float4(to_tf32(v[i].x), to_tf32(v[i].y), to_tf32(v[i].z), to_tf32(v[i].w));
            }
        }
    } else if (p.mode_in == IN_SA) {
        // relative xyz segment: [x - cx, y - cy, z - cz, (<= 5 feature channels,) 0 ...]; one K=8 step
        if (t < TM) {
            const int r = t;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f), v2 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (M.valid[r]) {
                const float *q = p.xyz + (size_t)M.src[r][0] * 3;
                v.x = to_tf32(__ldg(q + 0) - M.aux[r][0]);
                v.y = to_tf32(__ldg(q + 1) - M.aux[r][1]);
                v.z = to_tf32(__ldg(q + 2) - M.aux[r][2]);
                if (p.c_feat > 0 && p.c_feat <= 5) {
                    const float *f = p.feats_pm + (size_t)M.src[r][0] * p.c_feat;
                    v.w = to_tf32(__ldg(f));
                    if (p.c_feat > 1) v2.x = to_tf32(__ldg(f + 1));
                    if (p.c_feat > 2) v2.y = to_tf32(__ldg(f + 2));
                    if (p.c_feat > 3) v2.z = to_tf32(__ldg(f + 3));
                    if (p.c_feat > 4) v2.w = to_tf32(__ldg(f + 4));
                }
            }
            *reinterpret_cast<float4 *>(A + swz(r, 0)) = v;
            *reinterpret_cast<float4 *>(A + swz(r, 1)) = v2;
        }
    } else {
        // FP skip segment: channel-major (b, c_skip, n); 4 threads per row (8 channels each), the threads of a warp run
        // along consecutive points
        const int r = t & (TM - 1);
        const long R = (long)tile * TM + r;
#pragma unroll(STEPS > 2 ? 256 / NT : 1)
        for (int i = 0; i < 256 / NT; ++i) {
            const int q8 = (t >> 6) + i * (NT / 64);
            float o[8];
            if (M.valid[r]) {
                const int scene = (int)(R / p.n), u = (int)(R - (long)scene * p.n);
                const float *bsrc = p.skip + (size_t)scene * p.c_skip * p.n + u;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int ch = k0 + 8 * q8 + q;
                    o[q] = ch < width ? to_tf32(__ldg(bsrc + (size_t)ch * p.n)) : 0.f;
                }
            } else {
#pragma unroll
                for (int q = 0; q < 8; ++q) o[q] = 0.f;
            }
            *reinterpret_cast<float4 *>(A + swz(r, 2 * q8)) = make_float4(o[0], o[1], o[2], o[3]);
            *reinterpret_cast<float4 *>(A + swz(r, 2 * q8 + 1)) = make_float4(o[4], o[5], o[6], o[7]);
        }
    }
    return ksteps;
}

// The accumulator fragment of a warpgroup that covers columns col0 .. col0 + 32 nsub of the layer: thread (wq, g, t4)
// holds rows 16 wq + g (+8), columns 2 t4 (+1) of each 8.
// Inner layer: relu(acc * scale + shift) -> tf32 -> the resident activations in `work` (the next layer's K chunks).
template <int NS>
__device__ __forceinline__ void store_activations(const ChainParams &p, const float (&acc)[16 * NS], int nsub, int col0, int wq,
                                                  int g, int t4, const float *sc, const float *sh, uint8_t *work) {
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        if (j >= nsub) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = col0 + 32 * j + 8 * i + 2 * t4;
            uint8_t *chunk = work + (size_t)(c >> 5) * A_STAGE_BYTES;
            const int ju = (c & 31) >> 2, within = (c & 3) * 4;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = 16 * wq + g + 8 * h;
                float2 o;
                const float a0 = acc[16 * j + 4 * i + 2 * h], a1 = acc[16 * j + 4 * i + 2 * h + 1];
                if (p.unit_scale) {
                    o.x = relu_to_tf32(a0 + sh[c]);
                    o.y = relu_to_tf32(a1 + sh[c + 1]);
                } else {
                    o.x = relu_to_tf32(fmaf(a0, sc[c], sh[c]));
                    o.y = relu_to_tf32(fmaf(a1, sc[c + 1], sh[c + 1]));
                }
                *reinterpret_cast<float2 *>(chunk + swz(r, ju) + within) = o;
            }
        }
    }
}

// Last layer: SA max-pool, FP (channel-major + optional point-major copy) or rows.  The SA pool reduces the fragment in
// registers: a centre's nse = min(ns, 64) rows are nse consecutive rows of the tile, so a centre of 4 or 8 rows lies in
// the lanes of one warp that differ in g (and one row half h), one of 16 rows in both row halves of one warp, and one of
// 32 or 64 rows in 2 or 4 warps, whose per-warp maxima meet in `red` (4 x np floats of the warpgroup's free work region)
// behind one named barrier bar_id over the warpgroup's 128 threads (tw = thread inside the warpgroup).  A centre spanning
// several tiles keeps its partial maxima in s_carry (indexed by column).
template <int NS>
__device__ __forceinline__ void final_epilogue(const ChainParams &p, float (&acc)[16 * NS], int nsub, int col0, int wq,
                                               int g, int t4, int tw, int tile, const float *sc, const float *sh, float *red,
                                               float *s_carry, int bar_id) {
    const float lo = p.linear_last ? -CUDART_INF_F : 0.f;   // ReLU = max(., 0); a linear last layer keeps the sign
    const bool pool_raw = p.unit_scale && p.mode_out == OUT_SA_MAX;
    const int Cl = p.c_last;
    auto value = [&](float a, int c) -> float {
        if (pool_raw) return a;   // max_s relu(x_s + t) == relu(max_s x_s + t): shift / ReLU after the max
        return p.unit_scale ? fmaxf(a + sh[c], lo) : fmaxf(fmaf(a, sc[c], sh[c]), lo);
    };
    if (p.mode_out == OUT_SA_MAX) {
        const int nse = p.ns < TM ? p.ns : TM, per = p.ns > TM ? p.ns / TM : 1;
        const bool halves = nse >= 16;              // a centre covers both row halves of the thread
        const int gspan = nse < 8 ? nse : 8;        // lanes (4 g + t4) of a centre that differ in g
        // the maxima of subtile j over the centre's rows of this warp, in place in acc[16 j + 4 i + e] (and in
        // acc[16 j + 4 i + 2 + e] for the second row half when it is another centre): in the thread, then over the lanes
        // that differ in g (2 steps for a centre of 4 rows, 3 for 8 rows and more); every lane of the centre ends with them
        auto warp_max = [&](int j) {
            float *v = acc + 16 * j;
#pragma unroll
            for (int q = 0; q < 16; ++q) v[q] = value(v[q], col0 + 32 * j + 8 * (q >> 2) + 2 * t4 + (q & 1));
            if (halves) {
#pragma unroll
                for (int q = 0; q < 16; ++q)
                    if (!(q & 2)) v[q] = fmaxf(v[q], v[q + 2]);
            }
            for (int m = 4; m < 4 * gspan; m <<= 1) {
#pragma unroll
                for (int q = 0; q < 16; ++q)
                    if (!(halves && (q & 2))) v[q] = fmaxf(v[q], __shfl_xor_sync(0xffffffffu, v[q], m));
            }
        };
        // the first element of centre ci in `out` (channel stride npoint) and in out_pm (channel stride 1), or nullptr
        // for a centre past the last row (a partial last tile holds whole centres)
        auto centre_out = [&](int ci, float *&o, float *&o2) {
            const long Rg = (long)tile * TM + ci * nse;
            o = nullptr;
            o2 = nullptr;
            if (Rg >= p.total_rows) return;
            const int pr = (int)(Rg >> p.log_ns);   // rows < 2^31
            const int scene = pr / p.npoint, pp = pr - scene * p.npoint;
            o = p.out + ((size_t)scene * p.out_stride_c + p.out_c_off) * p.npoint + pp;
            if (p.out_pm) o2 = p.out_pm + (size_t)pr * p.out_stride_c + p.out_c_off;
        };
        auto store = [&](float x, int c, float *o, float *o2) {
            if (pool_raw) x = fmaxf(x + sh[c], lo);
            if (o && c < Cl) {
                o[(size_t)c * p.npoint] = x;
                if (o2) o2[c] = x;
            }
        };
        if (nse <= 16) {
            // a centre inside one warp: the lanes with g % gspan == 0 write it
#pragma unroll
            for (int j = 0; j < NS; ++j)
                if (j < nsub) warp_max(j);
            if ((g & (gspan - 1)) == 0) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (halves && h) continue;
                    float *o, *o2;
                    centre_out((16 * wq + g + 8 * h) / nse, o, o2);
#pragma unroll
                    for (int j = 0; j < NS; ++j) {
                        if (j >= nsub) continue;
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int e = 0; e < 2; ++e)
                                store(acc[16 * j + 4 * i + 2 * h + e], col0 + 32 * j + 8 * i + 2 * t4 + e, o, o2);
                    }
                }
            }
        } else {
            // a centre of 2 or 4 warps: each warp's maxima to red[wq][c], one barrier, then one thread per (centre,
            // column) takes the max over the centre's warps; a centre spanning several tiles carries it in s_carry
#pragma unroll
            for (int j = 0; j < NS; ++j) {
                if (j >= nsub) continue;
                warp_max(j);
                if (g == 0) {
#pragma unroll
                    for (int q = 0; q < 16; ++q)
                        if (!(q & 2)) red[wq * RED_STRIDE + col0 + 32 * j + 8 * (q >> 2) + 2 * t4 + (q & 1)] = acc[16 * j + q];
                }
            }
            bar_wg_id(bar_id);
            const int np_w = 32 * nsub, wpc = nse >> 4, ncent = TM / nse;   // columns, warps per centre, centres per tile
            const int sub = tile % per;
            for (int o = tw; o < ncent * np_w; o += 128) {
                const int ci = o / np_w, c = col0 + o - ci * np_w;
                float x = red[(ci * wpc) * RED_STRIDE + c];
                for (int w = 1; w < wpc; ++w) x = fmaxf(x, red[(ci * wpc + w) * RED_STRIDE + c]);
                if (per > 1) {
                    if (sub > 0) x = fmaxf(x, s_carry[c]);
                    if (sub < per - 1) { s_carry[c] = x; continue; }
                }
                float *op, *op2;
                centre_out(ci, op, op2);
                store(x, c, op, op2);
            }
        }
    } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const long R = (long)tile * TM + 16 * wq + g + 8 * h;
            if (R >= p.total_rows) continue;
            int scene = 0, u = 0;
            if (p.mode_out == OUT_FP) { scene = (int)(R / p.n); u = (int)(R - (long)scene * p.n); }
#pragma unroll
            for (int j = 0; j < NS; ++j) {
                if (j >= nsub) continue;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int c = col0 + 32 * j + 8 * i + 2 * t4;
                    float v0 = value(acc[16 * j + 4 * i + 2 * h], c), v1 = value(acc[16 * j + 4 * i + 2 * h + 1], c + 1);
                    if (p.mode_out == OUT_ROWS) {
                        if (p.round_out) { v0 = to_tf32(v0); v1 = to_tf32(v1); }   // the next launch's A operand
                        *reinterpret_cast<float2 *>(p.out + (size_t)R * p.out_pitch + c) = make_float2(v0, v1);
                    } else {
                        float *o = p.out + ((size_t)scene * p.out_stride_c + p.out_c_off + c) * p.n + u;
                        if (c < Cl) o[0] = v0;
                        if (c + 1 < Cl) o[p.n] = v1;
                        if (p.out_pm) {   // point-major copy for the next consumer (no transpose kernel)
                            float *o2 = p.out_pm + (size_t)R * p.out_stride_c + p.out_c_off + c;
                            if (c < Cl) o2[0] = v0;
                            if (c + 1 < Cl) o2[1] = v1;
                        }
                    }
                }
            }
        }
    }
}

// per-layer scale / shift into shared memory (the scale is 1 where it is folded into the weights)
__device__ __forceinline__ void load_scale_shift(const ChainParams &p, float *s_scale, float *s_shift, int t, int nt) {
    int off = 0;
#pragma unroll
    for (int l = 0; l < MAX_LAYERS; ++l) {
        if (l >= p.num_layers) break;
        for (int i = t; i < p.np[l]; i += nt) {
            s_scale[off + i] = p.unit_scale ? 1.f : p.scale[l][i];
            s_shift[off + i] = p.shift[l][i];
        }
        off += p.np[l];
    }
}

// ------------------------------------------------------------------------------------------------ streaming kernel
// NS: 32-column subtiles per warpgroup of the widest layer.  T: 64-row tiles a CTA runs together (2: tiles 2u and 2u + 1
// share every weight chunk, drain, barrier and epilogue pass).  Accumulator registers: 16 * NS * T per thread.
template <int NS, int MINB, int T>
__global__ void __launch_bounds__(chain_threads(NS, T), MINB) mlp_chain_kernel(const ChainParams p) {
    static_assert(T == 1 || T == 2, "mlp_chain_kernel: one or two tiles per CTA");
    constexpr int NTHR = chain_threads(NS, T);
    extern __shared__ uint8_t smem_raw[];
    __shared__ SmemFixed<T> S;
    uint8_t *base = smem_raw + ((1024u - (s2u(smem_raw) & 1023u)) & 1023u);
    const int L = p.num_layers;
    int np_total = 0;
#pragma unroll
    for (int l = 0; l < MAX_LAYERS; ++l) np_total += l < L ? p.np[l] : 0;
    // T work regions of work_bytes, tile s at sW + s * work_bytes; by phase of a tile: layer-0 A slots -> resident
    // activations (layers >= 1) -> per-warp pool maxima
    uint8_t *sW = base;
    uint8_t *sB = sW + (size_t)T * p.work_bytes;
    float *s_scale = reinterpret_cast<float *>(sB + (size_t)p.nb * p.b_stage_bytes);
    float *s_shift = s_scale + np_total;
    float *s_carry = s_shift + np_total;     // SA max over several tiles: partial maxima of the last layer
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NB = p.nb;

    if (tid == 0) {
        for (int i = 0; i < NB; ++i) { mbar_init(s2u(&S.b_full[i]), 1); mbar_init(s2u(&S.b_empty[i]), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    load_scale_shift(p, s_scale, s_shift, tid, NTHR);
    __syncthreads();

    // a unit is an item's tiles one after another (T = 1), or tiles 2u and 2u + 1 together (T = 2: two items of at most
    // one tile, or the two tiles of one item); CTAs take units in a strided order
    const int num_units = T == 1 ? p.num_items : (p.num_tiles + 1) >> 1;
    const int steps = T == 1 ? p.tiles_per_item : 1;

    // the broadcast tells the compiler that wg -- and with it every column range and MMA width -- is warp-uniform
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    if (wg == 2) {
        // ===================================================== weight producer: every chunk once per step of a unit
        if constexpr (NTHR == 3 * 128) setmaxnreg_dec<PRODUCER_REGS>();
        if (tid == 2 * 128) {
            RingPos rb = {0, 0};
            for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x)
                for (int st = 0; st < steps && (T == 1 ? unit * p.tiles_per_item + st : 2 * unit) < p.num_tiles; ++st)
                    for (int l = 0; l < L; ++l) {
                        const int np_l = per_layer(p.np, l), nch = per_layer(p.nchunks, l);
                        const float *w = per_layer(p.w, l);
                        for (int kc = 0; kc < nch; ++kc) {
                            const uint32_t bytes = (uint32_t)np_l * KC * 4;
                            mbar_wait(s2u(&S.b_empty[rb.stage]), rb.phase ^ 1);
                            mbar_expect_tx(s2u(&S.b_full[rb.stage]), bytes);
                            bulk_g2s(s2u(sB + (size_t)rb.stage * p.b_stage_bytes), w + (size_t)kc * np_l * KC, bytes,
                                     s2u(&S.b_full[rb.stage]));
                            rb.advance(NB);
                        }
                    }
        }
        return;
    }

    // ===================================================== MMA / epilogue warpgroups
    if constexpr (NTHR == 3 * 128) setmaxnreg_inc<MMA_REGS>();
    const int wq = warp & 3;
    const int g = lane >> 2, t4 = lane & 3;      // accumulator fragment: rows 16 wq + g (+8), columns 2 t4 (+1) of each 8
    const int tw = tid & 127;                    // thread inside the warpgroup
    RingPos rb = {0, 0};
    int aslot = 0;
    float acc[T][16 * NS];                       // tile s, subtile j (32 columns) = registers acc[s][16 j .. 16 j + 15]
    // the row table and layer-0 gather of a tile: T = 1, both warpgroups (NT = 256 threads); T = 2, warpgroup wg alone runs
    // tile wg of the unit (NT = 128) with twice the row steps in flight, so a pair's chunk costs one dependent batch of
    // loads per thread, as a single tile's does: the gathers are latency-bound.  Every warpgroup's MMAs read both tiles'
    // slots after the barrier that follows.
    constexpr int NT = 256 / T;
    const int my = T == 1 ? 0 : wg;              // this thread's tile of the unit for those stages
    const int ti = T == 1 ? tid : tw;            // ... and its index among their NT threads

    for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        for (int st = 0; st < steps; ++st) {
            const int tile0 = T == 1 ? unit * p.tiles_per_item + st : 2 * unit;   // tile 2u + 1 may lie past the last
            if (tile0 >= p.num_tiles) break;                                         // one: no valid rows, nothing written
            bar_mma();   // the previous unit's readers of S.rows and of the pool maxima are done
            load_tile_rows(p, tile0 + my, ti, S.rows[my]);
            bar_mma();

            int sc_base = 0;   // layer l's scale / shift in s_scale / s_shift
            for (int l = 0; l < L; ++l) {
                const int np_l = per_layer(p.np, l);
                const int nsub_all = np_l >> 5, nsub0 = (nsub_all + 1) >> 1;
                const int nsub = wg == 0 ? nsub0 : nsub_all - nsub0;
                const int col0 = wg == 0 ? 0 : nsub0 * 32;            // first output column of this warpgroup
                const int nch = per_layer(p.nchunks, l);
                int prev_stage = -1;
                for (int kc = 0; kc < nch; ++kc) {
                    uint64_t adesc[T];
                    int ksteps = KC / 8;
                    if (l == 0) {
                        uint8_t *A = sW + (size_t)my * p.work_bytes + (size_t)aslot * A_STAGE_BYTES;
                        ksteps = gather_chunk<NT, 2 * T>(p, tile0 + my, kc, ti, S.rows[my], A);
                        fence_async_smem();
                        // slot `aslot` of every tile is complete.  It was last read by the MMAs of chunk kc-3, which both
                        // warpgroups retired (wgmma_wait<1> of chunk kc-2) before the barrier of chunk kc-1.
                        bar_mma();
#pragma unroll
                        for (int s = 0; s < T; ++s)
                            adesc[s] = make_desc(s2u(sW + (size_t)s * p.work_bytes + (size_t)aslot * A_STAGE_BYTES));
                        aslot = aslot == A_SLOTS - 1 ? 0 : aslot + 1;
                    } else {
#pragma unroll
                        for (int s = 0; s < T; ++s)
                            adesc[s] = make_desc(s2u(sW + (size_t)s * p.work_bytes + (size_t)kc * A_STAGE_BYTES));
                    }
                    mbar_wait(s2u(&S.b_full[rb.stage]), rb.phase);
                    const uint32_t b_addr = s2u(sB + (size_t)rb.stage * p.b_stage_bytes) + (uint32_t)col0 * (KC * 4);
                    wgmma_fence();
                    mma_chunk<NS, T>(acc, nsub, ksteps, adesc, make_desc(b_addr), kc > 0 ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait<1>();     // the previous chunk's MMAs are done: release its weight stage
                    if (prev_stage >= 0 && lane == 0) mbar_arrive(s2u(&S.b_empty[prev_stage]));
                    prev_stage = (int)rb.stage;
                    rb.advance(NB);
                }
                wgmma_wait<0>();
#pragma unroll
                for (int s = 0; s < T; ++s) reg_fence(acc[s]);
                if (lane == 0) mbar_arrive(s2u(&S.b_empty[prev_stage]));
                bar_mma();   // both warpgroups' MMAs of layer l have read their A operands: the work regions are free
                const float *sc = s_scale + sc_base, *sh = s_shift + sc_base;
                sc_base += np_l;

                if (l + 1 < L) {
#pragma unroll
                    for (int s = 0; s < T; ++s)
                        store_activations<NS>(p, acc[s], nsub, col0, wq, g, t4, sc, sh, sW + (size_t)s * p.work_bytes);
                    fence_async_smem();
                    bar_mma();   // the next layer's A operands are complete
                    continue;
                }
                // an SA centre of two tiles (T = 2) carries its partial maxima from tile 0 to tile 1 in s_carry: the
                // same thread writes and reads column c
#pragma unroll
                for (int s = 0; s < T; ++s)
                    final_epilogue<NS>(p, acc[s], nsub, col0, wq, g, t4, tw, tile0 + s, sc, sh,
                                       reinterpret_cast<float *>(sW + (size_t)s * p.work_bytes), s_carry, 2 + wg);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ resident kernel
// NS: 32-column subtiles of the widest layer, all of them in one warpgroup (np <= RES_NP_MAX).  T: 64-row tiles a
// warpgroup runs together (2: tiles 2u and 2u + 1 share every B operand, drain, barrier and epilogue pass).
// blockDim.x = 128 * nwg.
template <int NS, int NWG, int MINB, int T>
__global__ void __launch_bounds__(NWG * 128, MINB) mlp_resident_kernel(const ChainParams p) {
    static_assert(NWG <= RES_WG_MAX, "mlp_resident_kernel: one named barrier per warpgroup");
    static_assert(NS * 32 <= RES_NP_MAX, "mlp_resident_kernel: one warpgroup covers the widest layer");
    static_assert(T == 1 || T == 2, "mlp_resident_kernel: one or two tiles per warpgroup");
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t w_full;
    uint8_t *base = smem_raw + ((1024u - (s2u(smem_raw) & 1023u)) & 1023u);
    const int L = p.num_layers, nwg = blockDim.x >> 7;
    int np_total = 0, w_bytes = 0;
#pragma unroll
    for (int l = 0; l < MAX_LAYERS; ++l) {
        np_total += l < L ? p.np[l] : 0;
        w_bytes += l < L ? p.nchunks[l] * p.np[l] * KC * 4 : 0;
    }
    const int np_last = per_layer(p.np, L - 1);
    // [weight image of every layer | nwg x T work regions | scale | shift | nwg pool carries | nwg x T tile-row tables]
    uint8_t *sWt = base;
    uint8_t *sWork = sWt + w_bytes;
    float *s_scale = reinterpret_cast<float *>(sWork + (size_t)nwg * T * p.work_bytes);
    float *s_shift = s_scale + np_total;
    float *s_carry_all = s_shift + np_total;
    TileRows *rows_all = reinterpret_cast<TileRows *>(s_carry_all + nwg * np_last);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        mbar_init(s2u(&w_full), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    load_scale_shift(p, s_scale, s_shift, tid, blockDim.x);
    __syncthreads();
    if (tid == 0) {
        // the whole packed image, chunk by chunk, on one mbarrier; it stays for every tile of the CTA
        mbar_expect_tx(s2u(&w_full), (uint32_t)w_bytes);
        uint32_t off = 0;
        for (int l = 0; l < L; ++l) {
            const int np_l = per_layer(p.np, l), nch = per_layer(p.nchunks, l);
            const float *w = per_layer(p.w, l);
            const uint32_t bytes = (uint32_t)np_l * KC * 4;
            for (int kc = 0; kc < nch; ++kc, off += bytes)
                bulk_g2s(s2u(sWt + off), w + (size_t)kc * np_l * KC, bytes, s2u(&w_full));
        }
    }

    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    const int wq = warp & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const int tw = tid & 127;
    const int bar_id = 1 + wg;
    // tile s of the warpgroup's unit: work region (A slots / activations / pool maxima) W + s * work_bytes, row table
    // M[s]; its stages run on thread index tw ^ 64 s, so the half-warpgroup stages (row table, xyz gather) of the two
    // tiles run on different warps
    uint8_t *W = sWork + (size_t)wg * T * p.work_bytes;
    float *s_carry = s_carry_all + wg * np_last;
    TileRows *M = rows_all + wg * T;
    const int nslots = p.nchunks[0] < A_SLOTS ? p.nchunks[0] : A_SLOTS;
    bool w_ready = false;
    float acc[T][16 * NS];

    // a unit is an item's tiles one after another (T = 1), or tiles 2u and 2u + 1 together (T = 2: two items of at most
    // one tile, or the two tiles of one item); warpgroups take units in a strided order over the whole grid
    const int num_units = T == 1 ? p.num_items : (p.num_tiles + 1) >> 1;
    const int steps = T == 1 ? p.tiles_per_item : 1;
    for (int unit = blockIdx.x * nwg + wg; unit < num_units; unit += gridDim.x * nwg) {
        for (int st = 0; st < steps; ++st) {
            const int tile0 = T == 1 ? unit * p.tiles_per_item + st : 2 * unit;   // tile 2u + 1 may lie past the last
            if (tile0 >= p.num_tiles) break;                                         // one: no valid rows, nothing written
            bar_wg_id(bar_id);   // the previous unit's readers of M and of the pool maxima are done
#pragma unroll
            for (int s = 0; s < T; ++s) load_tile_rows(p, tile0 + s, tw ^ (64 * s), M[s]);
            bar_wg_id(bar_id);

            int sc_base = 0;
            uint32_t w_off = 0;   // layer l's image in sWt
            for (int l = 0; l < L; ++l) {
                const int np_l = per_layer(p.np, l), nsub = np_l >> 5;
                const int nch = per_layer(p.nchunks, l);
                int aslot = 0;
                for (int kc = 0; kc < nch; ++kc) {
                    uint64_t adesc[T];
                    int ksteps = KC / 8;
                    if (l == 0) {
#pragma unroll
                        for (int s = 0; s < T; ++s) {
                            uint8_t *A = W + (size_t)s * p.work_bytes + (size_t)aslot * A_STAGE_BYTES;
                            ksteps = gather_chunk<128>(p, tile0 + s, kc, tw ^ (64 * s), M[s], A);
                            adesc[s] = make_desc(s2u(A));
                        }
                        fence_async_smem();
                        // slot `aslot` was last read by the MMAs of chunk kc-3, which every warp of the warpgroup
                        // retired (wgmma_wait<1> of chunk kc-2) before the barrier of chunk kc-1
                        bar_wg_id(bar_id);
                        aslot = aslot == nslots - 1 ? 0 : aslot + 1;
                    } else {
#pragma unroll
                        for (int s = 0; s < T; ++s)
                            adesc[s] = make_desc(s2u(W + (size_t)s * p.work_bytes + (size_t)kc * A_STAGE_BYTES));
                    }
                    if (!w_ready) { mbar_wait(s2u(&w_full), 0); w_ready = true; }
                    const uint32_t b_addr = s2u(sWt) + w_off + (uint32_t)kc * np_l * (KC * 4);
                    wgmma_fence();
                    mma_chunk<NS, T>(acc, nsub, ksteps, adesc, make_desc(b_addr), kc > 0 ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait<1>();
                }
                w_off += (uint32_t)nch * np_l * (KC * 4);
                wgmma_wait<0>();
#pragma unroll
                for (int s = 0; s < T; ++s) reg_fence(acc[s]);
                bar_wg_id(bar_id);   // the warpgroup's MMAs of layer l have read their A operands: the work regions are free
                const float *sc = s_scale + sc_base, *sh = s_shift + sc_base;
                sc_base += np_l;
                if (l + 1 < L) {
#pragma unroll
                    for (int s = 0; s < T; ++s)
                        store_activations<NS>(p, acc[s], nsub, 0, wq, g, t4, sc, sh, W + (size_t)s * p.work_bytes);
                    fence_async_smem();
                    bar_wg_id(bar_id);   // the next layer's A operands are complete
                    continue;
                }
#pragma unroll
                for (int s = 0; s < T; ++s)
                    final_epilogue<NS>(p, acc[s], nsub, 0, wq, g, t4, tw, tile0 + s, sc, sh,
                                       reinterpret_cast<float *>(W + (size_t)s * p.work_bytes), s_carry, bar_id);
            }
        }
    }
    if (tid == 0 && !w_ready) mbar_wait(s2u(&w_full), 0);   // no CTA exits with its weight copy in flight
}

// ------------------------------------------------------------------------------------------------ wide-layer kernel
// One layer wider than WN_WIDE over rows already in global memory (row-major, tf32, K padded to a multiple of KC): the
// layers of a chain wider than 256 run here, each as its own launch.  A CTA tile is WM_WIDE = 128 rows x 32 NS output
// columns, where the layer's np columns are cut into two blocks of equal width (32 NS <= WN_WIDE = 256; where np / 32 is
// odd, the second block's last 32 columns lie past the layer and are computed from whatever the B stage holds there and
// never stored).  The persistent CTAs walk (row block, column block) tiles, the column blocks of a row block one after
// another so its A rows are still in L2 for the second.  Warpgroup 2's one thread fills a ring of WIDE_NB stages, each one
// K chunk of A (a TMA tensor-map load of 128 rows x 32 floats, SWIZZLE_128B, rows past the end zero) and of B (the
// column block's slab of the packed image, at most 32 KB, one bulk copy); warpgroups 0 and 1 take rows 0-63 and 64-127
// of the tile, one m64n(32 NS)k8 per K=8 step into 16 NS accumulators, and run the final epilogue while the producer
// fills the ring with the next tile's chunks.  Per K chunk a 128 x 256 tile moves 48 KB for 2.1 MFLOP.
// The K order and the epilogues are the fused kernels'.  Every chunk runs all four K=8 steps, with the MMA width fixed
// at compile time: a runtime choice of either makes ptxas serialise the wgmma (C7520).  The fused kernels skip the K=8
// steps past the end of a layer-0 segment; here they multiply the zeros of the gathered rows by the zeros of the packed
// image, and adding those +0 products leaves every fp32 sum unchanged (only an all-zero sum of -0 products would become
// +0).
constexpr int WM_WIDE = 2 * TM, WN_WIDE = 256, WIDE_NB = 4;
constexpr int WIDE_A_BYTES = WM_WIDE * KC * 4, WIDE_B_BYTES = WN_WIDE * KC * 4;
constexpr int WIDE_STAGE_BYTES = WIDE_A_BYTES + WIDE_B_BYTES;
constexpr int WIDE_THREADS = 3 * 128;

// 2D TMA load of the box at (column c0, row r0) of the tensor map into shared memory, completing on the mbarrier
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int c0, int r0, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(r0), "r"(bar)
                 : "memory");
}

template <int NS>
__global__ void __launch_bounds__(WIDE_THREADS, 1) mlp_wide_kernel(const __grid_constant__ CUtensorMap amap, const ChainParams p) {
    static_assert(NS >= 1 && NS <= NSUB_MAX, "mlp_wide_kernel: one m64n(32 NS)k8 per warpgroup and K=8 step");
    constexpr int BW = 32 * NS;   // columns per block
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full[WIDE_NB], empty[WIDE_NB];
    uint8_t *ring = smem_raw + ((1024u - (s2u(smem_raw) & 1023u)) & 1023u);
    // [ring: WIDE_NB x (A | B) | per-warp pool maxima of both warpgroups | scale | shift | pool carry]
    const int np = p.np[0], nch = p.nchunks[0];
    float *red_all = reinterpret_cast<float *>(ring + (size_t)WIDE_NB * WIDE_STAGE_BYTES);
    float *s_scale = red_all + 2 * 4 * RED_STRIDE;
    float *s_shift = s_scale + np;
    float *s_carry = s_shift + np;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < WIDE_NB; ++i) { mbar_init(s2u(&full[i]), 1); mbar_init(s2u(&empty[i]), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    load_scale_shift(p, s_scale, s_shift, tid, WIDE_THREADS);
    __syncthreads();
    const int ncb = (np + BW - 1) / BW;
    const int num_tiles = (int)((p.total_rows + WM_WIDE - 1) / WM_WIDE) * ncb;

    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);
    if (wg == 2) {
        // ===================================================== producer: A and B of every K chunk of every tile
        setmaxnreg_dec<PRODUCER_REGS>();
        if (tid == 2 * 128) {
            RingPos rb = {0, 0};
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int rblk = tile / ncb, col0 = (tile - rblk * ncb) * BW;
                const uint32_t b_bytes = (uint32_t)min(BW, np - col0) * KC * 4;
                for (int kc = 0; kc < nch; ++kc) {
                    mbar_wait(s2u(&empty[rb.stage]), rb.phase ^ 1);
                    const uint32_t stage = s2u(ring + (size_t)rb.stage * WIDE_STAGE_BYTES), bar = s2u(&full[rb.stage]);
                    mbar_expect_tx(bar, WIDE_A_BYTES + b_bytes);
                    tma_load_2d(stage, &amap, kc * KC, rblk * WM_WIDE, bar);
                    bulk_g2s(stage + WIDE_A_BYTES, p.w[0] + ((size_t)kc * np + col0) * KC, b_bytes, bar);
                    rb.advance(WIDE_NB);
                }
            }
        }
        return;
    }

    // ===================================================== MMA / epilogue warpgroups: rows 64 wg .. 64 wg + 63 of a tile
    setmaxnreg_inc<MMA_REGS>();
    const int wq = warp & 3, g = lane >> 2, t4 = lane & 3, tw = tid & 127;
    float *red = red_all + wg * 4 * RED_STRIDE;
    // an SA centre of 128 rows spans both warpgroups: warpgroup 0's pass leaves its maxima in s_carry for warpgroup 1's
    const bool carry = p.mode_out == OUT_SA_MAX && p.ns > TM;
    RingPos rb = {0, 0};
    float acc[1][16 * NS];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int rblk = tile / ncb, col0 = (tile - rblk * ncb) * BW;
        const int nsub = min(BW, np - col0) >> 5;   // the block's columns inside the layer
        int prev_stage = -1;
        for (int kc = 0; kc < nch; ++kc) {
            mbar_wait(s2u(&full[rb.stage]), rb.phase);
            const uint32_t stage = s2u(ring + (size_t)rb.stage * WIDE_STAGE_BYTES);
            const uint64_t adesc[1] = {make_desc(stage + (uint32_t)wg * A_STAGE_BYTES)};
            wgmma_fence();
            mma_steps<NS, KC / 8, NS, 1>(acc, adesc, make_desc(stage + WIDE_A_BYTES), kc > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();     // the previous chunk's MMAs are done: release its stage
            if (prev_stage >= 0 && lane == 0) mbar_arrive(s2u(&empty[prev_stage]));
            prev_stage = (int)rb.stage;
            rb.advance(WIDE_NB);
        }
        wgmma_wait<0>();
        reg_fence(acc[0]);
        if (lane == 0) mbar_arrive(s2u(&empty[prev_stage]));
        if (p.mode_out == OUT_SA_MAX) {
            if (carry && wg == 1) bar_mma();   // warpgroup 0's partial maxima are in s_carry
            bar_wg_id(2 + wg);                 // every warp of the warpgroup is done with the previous tile's pool maxima
        }
        final_epilogue<NS>(p, acc[0], nsub, col0, wq, g, t4, tw, 2 * rblk + wg, s_scale, s_shift, red, s_carry, 2 + wg);
        if (carry) {
            if (wg == 0) bar_mma();
            bar_mma();   // warpgroup 1 has read s_carry before warpgroup 0 writes the next tile's
        }
    }
}

// Layer 0's A operand of a chain whose first layer runs on the wide kernel: K chunk blockIdx.y of 64-row tile blockIdx.x,
// gathered exactly as the fused kernels gather it into their A slots (tf32, padded segment order), written row-major
// with `pitch` floats per row.  The columns past a segment's last K=8 step are written as zeros: the wide kernel runs
// those steps, and their products must be +0.
__global__ void __launch_bounds__(128) mlp_gather_kernel(const ChainParams p, float *rows, int pitch) {
    __shared__ __align__(128) uint8_t A[A_STAGE_BYTES];
    __shared__ TileRows M;
    const int tile = blockIdx.x, kc = blockIdx.y, t = threadIdx.x;
    load_tile_rows(p, tile, t, M);
    __syncthreads();
    const int ksteps = gather_chunk<128>(p, tile, kc, t, M, A);
    __syncthreads();
    for (int i = t; i < TM * 8; i += 128) {
        const int r = i >> 3, j = i & 7;
        const long R = (long)tile * TM + r;
        if (R >= p.total_rows) continue;
        const float4 v = j < 2 * ksteps ? *reinterpret_cast<const float4 *>(A + swz(r, j)) : make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4 *>(rows + (size_t)R * pitch + kc * KC + 4 * j) = v;
    }
}

// ------------------------------------------------------------------------------------------------ host side
static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

struct LayerGeom {
    int k_chunks;  // K chunks
    int np;        // padded N
    size_t w_off;  // float offset of this layer's image in the packed buffer
};

// K layout of layer 0 = the given segments, each padded to KC; deeper layers: previous np
static void chain_geometry(int L, int nseg, const int *seg_width, const int *c_out, LayerGeom *g, size_t *total_floats) {
    size_t off = 0;
    for (int l = 0; l < L; ++l) {
        int chunks = 0;
        if (l == 0) for (int s = 0; s < nseg; ++s) chunks += round_up(seg_width[s], KC) / KC;
        else chunks = g[l - 1].np / KC;
        g[l].k_chunks = chunks;
        g[l].np = round_up(c_out[l], 32);
        g[l].w_off = off;
        off += (size_t)chunks * g[l].np * KC;
    }
    if (total_floats) *total_floats = off;
}

static inline float tf32_rna_host(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) != 0x7f800000u) u += 0x1000u;  // round to nearest, ties away (cvt.rna)
    u &= 0xffffe000u;
    float r;
    memcpy(&r, &u, 4);
    return r;
}

}  // namespace prb

using namespace prb;

// segment description used by the packer: our K order is seg 0 then seg 1; each segment names the first
// column it takes from the ORIGINAL (c_out0, c_in) weight and its width
struct PackSegs {
    int nseg;
    int src_off[2], width[2];
};

static void default_segs(int kind, int c_in, int a, PackSegs *ps) {
    // kind 0 (SA): original columns [xyz(3), feats(a)] -> ours [feats(a), xyz(3)];  a = c_feat
    // kind 1 (FP): original [interp(a), skip(c_in-a)] kept in order, split in two padded segments
    // kind 2 (DIRECT): one segment
    if (kind == 0) {
        // a handful of feature channels (e.g. the intensity of the first RPN level) ride in the xyz chunk: [xyz, feats]
        if (a > 0 && a <= 5) { ps->nseg = 1; ps->src_off[0] = 0; ps->width[0] = 3 + a; }
        else if (a > 0) { ps->nseg = 2; ps->src_off[0] = 3; ps->width[0] = a; ps->src_off[1] = 0; ps->width[1] = 3; }
        else { ps->nseg = 1; ps->src_off[0] = 0; ps->width[0] = 3; }
    } else if (kind == 1 && c_in - a > 0) {
        ps->nseg = 2; ps->src_off[0] = 0; ps->width[0] = a; ps->src_off[1] = a; ps->width[1] = c_in - a;
    } else {
        ps->nseg = 1; ps->src_off[0] = 0; ps->width[0] = c_in;
    }
}

extern "C" {

// extended packing entry points (kind / split) -- the header's prb_mlp_packed_bytes / prb_mlp_pack_weights
// are the DIRECT (kind 2) forms
PRB_API size_t prb_mlp_packed_bytes_ex(int kind, int split, int num_layers, int c_in, const int *c_out) {
    PackSegs ps;
    default_segs(kind, c_in, split, &ps);
    LayerGeom g[MAX_LAYERS];
    size_t total = 0;
    chain_geometry(num_layers, ps.nseg, ps.width, c_out, g, &total);
    return total * sizeof(float);
}

PRB_API int prb_mlp_pack_weights_ex(int kind, int split, int num_layers, int c_in, const int *c_out, const float *const *w, void *dst) {
    PRB_REQUIRE(num_layers >= 1 && num_layers <= MAX_LAYERS && w && dst && c_out, "mlp_pack: bad arguments");
    PackSegs ps;
    default_segs(kind, c_in, split, &ps);
    LayerGeom g[MAX_LAYERS];
    size_t total = 0;
    chain_geometry(num_layers, ps.nseg, ps.width, c_out, g, &total);
    float *out = (float *)dst;
    memset(out, 0, total * sizeof(float));
    for (int l = 0; l < num_layers; ++l) {
        const int np = g[l].np;
        const int kin = l == 0 ? c_in : c_out[l - 1];
        // map our K index -> original column (or -1 for padding)
        std::vector<int> kmap((size_t)g[l].k_chunks * KC, -1);
        if (l == 0) {
            int base = 0;
            for (int s = 0; s < ps.nseg; ++s) {
                for (int i = 0; i < ps.width[s]; ++i) kmap[base + i] = ps.src_off[s] + i;
                base += round_up(ps.width[s], KC);
            }
        } else {
            for (int i = 0; i < kin; ++i) kmap[i] = i;
        }
        for (int kc = 0; kc < g[l].k_chunks; ++kc)
            for (int n = 0; n < np; ++n)
                for (int kk = 0; kk < KC; ++kk) {
                    const int src = kmap[(size_t)kc * KC + kk];
                    float v = 0.f;
                    if (n < c_out[l] && src >= 0) v = tf32_rna_host(w[l][(size_t)n * kin + src]);
                    // K-major SWIZZLE_128B image of an (np x 32) tile: row n at n*128 B, 16-B unit j at j ^ (n & 7)
                    const int j = kk >> 2, q = kk & 3;
                    const size_t o = g[l].w_off + (size_t)kc * np * KC + (size_t)n * KC + (size_t)(((j ^ (n & 7)) << 2) + q);
                    out[o] = v;
                }
    }
    return 0;
}

size_t prb_mlp_packed_bytes(int num_layers, int c_in, const int *c_out) {
    return prb_mlp_packed_bytes_ex(2, 0, num_layers, c_in, c_out);
}
int prb_mlp_pack_weights(int num_layers, int c_in, const int *c_out, const float *const *w, void *dst) {
    return prb_mlp_pack_weights_ex(2, 0, num_layers, c_in, c_out, w, dst);
}

}  // extern "C"

namespace prb {

// shared memory of a fused segment [l0, l1) in the streaming kernel with t tiles per CTA and an nb-deep weight ring:
// dynamic (returned) and static (*fixed); *work_bytes is one tile's work region
static size_t segment_smem(const int *np, int n, int nb, int t, int *work_bytes, int *b_stage_bytes, size_t *fixed) {
    int np_total = 0, np_max = 0, mid_max = 0;
    for (int i = 0; i < n; ++i) {
        np_total += np[i];
        np_max = np[i] > np_max ? np[i] : np_max;
        if (i + 1 < n && np[i] > mid_max) mid_max = np[i];
    }
    int work = A_SLOTS * A_STAGE_BYTES;   // a multiple of 8 KB, so every tile's region stays 1024-byte aligned
    if (TM * mid_max * 4 > work) work = TM * mid_max * 4;
    if (work_bytes) *work_bytes = work;
    if (b_stage_bytes) *b_stage_bytes = np_max * KC * 4;
    if (fixed) *fixed = t == 2 ? sizeof(SmemFixed<2>) : sizeof(SmemFixed<1>);
    return chain_smem_bytes(t * work, nb, np_max * KC * 4, np_total, np[n - 1]);
}

// Resident variant of one launch, if it applies: every layer at most RES_NP_MAX wide, one of the three plain mode pairs,
// and the whole packed image plus one warpgroup's working set within the shared memory of a CTA.  Warpgroups per CTA
// and CTAs per SM are the pair that keeps the most warpgroups on an SM (registers, shared memory and threads as the
// occupancy calculator counts them); on a tie, the fewer CTAs, so fewer copies of the image.  Returns false if the
// launch is for the streaming kernel.
static bool launch_resident(ChainParams &p, int max_optin, cudaStream_t st, int *rc) {
    if (!opts().mlp_resident) return false;
    const bool modes = (p.mode_in == IN_SA && p.mode_out == OUT_SA_MAX) || (p.mode_in == IN_FP && p.mode_out == OUT_FP) ||
                       (p.mode_in == IN_DIRECT && p.mode_out == OUT_ROWS);
    if (!modes) return false;
    const int L = p.num_layers;
    int np_total = 0, np_max = 0, mid_max = 0;
    size_t w_bytes = 0;
    for (int l = 0; l < L; ++l) {
        np_total += p.np[l];
        np_max = p.np[l] > np_max ? p.np[l] : np_max;
        if (l + 1 < L && p.np[l] > mid_max) mid_max = p.np[l];
        w_bytes += (size_t)p.nchunks[l] * p.np[l] * KC * 4;
    }
    if (np_max > RES_NP_MAX) return false;
    // the image takes at most half of a CTA's shared memory, so at least three warpgroups' work regions fit beside it.
    // Measured on an H100 80GB HBM3 (600 W limit): the two larger images of the RPN backbone -- the FP0 chain, 144 KB
    // (2 warpgroups per SM), and its projection, 128 KB (3) -- ran 1.33x and 1.16x slower resident than streamed.
    if (2 * w_bytes > (size_t)max_optin) return false;
    // two 64-row tiles per warpgroup where every layer is at most 64 wide: a tile's serial steps (row table, gather, MMA,
    // drain, barrier, epilogue per layer, pool) are short there, and the pair halves their count per row
    const int T = np_max <= 64 ? 2 : 1;
    // a tile's work region: its layer-0 A slots, the activations of the widest inner layer (the pool maxima fit in either)
    const int slots = p.nchunks[0] < A_SLOTS ? p.nchunks[0] : A_SLOTS;
    int work = slots * A_STAGE_BYTES;
    if (TM * mid_max * 4 > work) work = TM * mid_max * 4;
    work = round_up(work, 1024);
    const int np_last = p.np[L - 1];
    auto smem_for = [&](int nwg) -> size_t {
        return 1024 /*alignment slack*/ + w_bytes + 2 * (size_t)np_total * sizeof(float) +
               (size_t)nwg * (T * (work + sizeof(TileRows)) + np_last * sizeof(float));
    };
    if (smem_for(1) + 64 /*static: the weight mbarrier*/ > (size_t)max_optin) return false;
    p.work_bytes = work;
    auto go = [&](auto kern, int nwg_max) -> int {
        cudaFuncAttributes fa;
        PRB_CUDA(cudaFuncGetAttributes(&fa, kern));
        const size_t dyn_max = (size_t)max_optin - fa.sharedSizeBytes;
        PRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_max));
        int best_nwg = 1, best_occ = 1, best_total = 0;
        for (int nwg = 1; nwg <= nwg_max; ++nwg) {
            if (smem_for(nwg) > dyn_max) break;
            int occ = 0;
            PRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, nwg * 128, smem_for(nwg)));
            if (const int o = opts().mlp_occ; o >= 1 && o < occ) occ = o;
            if (occ * nwg >= best_total && occ >= 1) { best_nwg = nwg; best_occ = occ; best_total = occ * nwg; }
        }
        int sms = num_sms();
        if (const int v = opts().mlp_sms; v >= 1 && v < sms) sms = v;
        const int units = T == 2 ? (p.num_tiles + 1) / 2 : p.num_items;
        const int ctas = (units + best_nwg - 1) / best_nwg;   // every CTA has a unit for its warpgroup 0
        const int grid = ctas < sms * best_occ ? ctas : sms * best_occ;
        kern<<<grid, best_nwg * 128, smem_for(best_nwg), st>>>(p);
        return check_launch("mlp_resident_kernel");
    };
    // register bounds without spills: <1, 4, 1, 2> and <4, 4, 1, 1> 128 (four warpgroups per SM), <2, 3, 1, 2> 168 (three);
    // the pairs spilled at 96 and 128
    if (np_max <= 32) *rc = go(mlp_resident_kernel<1, 4, 1, 2>, 4);
    else if (np_max <= 64) *rc = go(mlp_resident_kernel<2, 3, 1, 2>, 3);
    else *rc = go(mlp_resident_kernel<4, 4, 1, 1>, 4);
    return true;
}

// launch one fused segment of the chain: the resident kernel where it applies, else the streaming kernel with the
// weight ring sized to the segment and the CTAs per SM it allows
static int launch_chain(ChainParams &p, cudaStream_t st) {
    int max_optin = 0, dev = 0;
    PRB_CUDA(cudaGetDevice(&dev));
    PRB_CUDA(cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    p.num_tiles = (int)((p.total_rows + TM - 1) / TM);
    if (p.num_tiles == 0) return 0;
    p.tiles_per_item = (p.mode_out == OUT_SA_MAX && p.ns > TM) ? p.ns / TM : 1;
    p.num_items = (p.num_tiles + p.tiles_per_item - 1) / p.tiles_per_item;
    if (int rc = 0; launch_resident(p, max_optin, st, &rc)) return rc;
    const int L = p.num_layers;
    int np_total = 0, ns_max = 1;
    for (int l = 0; l < L; ++l) {
        np_total += p.np[l];
        const int nsub0 = ((p.np[l] >> 5) + 1) >> 1;
        ns_max = nsub0 > ns_max ? nsub0 : ns_max;
    }
    // A tile pair where the widest layer is 129-256 wide and the pair still has a weight ring of three stages: each
    // warpgroup holds its column half of both tiles in 128 accumulator registers, and every weight chunk leaves L2 once
    // per 128 rows instead of once per 64.  Single tile against pair, ms per launch of the RPN backbone at B = 16 (H100
    // 80GB HBM3, 700 W limit):
    //   SA3 [259]->128,196,256, ns 16 / 32 (pair ring 3)   0.156 / 0.299 -> 0.130 / 0.232
    //   FP1 [512+96]->256,256 (pair ring 2, single 4)       0.367 -> 0.368
    //   128 wide, FP0 chain / projection (pair 1 CTA per SM, single 2)   0.231 / 0.065 -> 0.316 / 0.079
    size_t smem = 0, fixed = 0;
    const int T = ns_max > 2 && ns_max <= 4 &&
                  segment_smem(p.np, L, 3, 2, nullptr, nullptr, &fixed) + fixed <= (size_t)max_optin ? 2 : 1;
    // deepest weight ring that fits (a stage is one K chunk of the widest layer)
    for (p.nb = NB_MAX; p.nb >= 2; --p.nb) {
        smem = segment_smem(p.np, L, p.nb, T, &p.work_bytes, &p.b_stage_bytes, &fixed);
        if (smem + fixed <= (size_t)max_optin) break;
    }
    PRB_REQUIRE(p.nb >= 2, "mlp: %zu bytes of shared memory needed, %d available", smem + fixed, max_optin);
    // the accumulators of the widest layer set the register budget, and with it how many CTAs share an SM: several
    // CTAs of a narrow chain overlap one another's latency-bound gathers
    auto go = [&](auto kern, int threads) -> int {
        PRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        PRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
        if (occ < 1) occ = 1;
        if (const int o = opts().mlp_occ; o >= 1 && o < occ) occ = o;
        int sms = num_sms();
        if (const int v = opts().mlp_sms; v >= 1 && v < sms) sms = v;
        const int units = T == 2 ? (p.num_tiles + 1) / 2 : p.num_items;
        const int grid = units < sms * occ ? units : sms * occ;
        kern<<<grid, threads, smem, st>>>(p);
        return check_launch("mlp_chain_kernel");
    };
    // registers without spills: <2,2,1> 96 (two CTAs per SM), <4,1,1> 152; <4,1,2> 168 at launch, the MMA warpgroups
    // raised to 232 by setmaxnreg
    PRB_REQUIRE(ns_max <= 4, "mlp: a fused launch of a layer %d wide (wider than %d runs on the wide kernel)", 64 * ns_max, WN_WIDE);
    if (T == 2) return go(mlp_chain_kernel<4, 1, 2>, chain_threads(4, 2));
    if (ns_max <= 2) return go(mlp_chain_kernel<2, 2, 1>, chain_threads(2, 1));
    return go(mlp_chain_kernel<4, 1, 1>, chain_threads(4, 1));
}

// cuTensorMapEncodeTiled from the driver the runtime uses (the library links only the runtime)
static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static const PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
        void *f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            f = nullptr;
        return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
    }();
    return fn;
}

// one layer wider than WN_WIDE (p.num_layers = 1) over a_rows: total_rows rows of a_pitch floats (a multiple of KC, the
// layer's padded K), 16-byte aligned
static int launch_wide(ChainParams &p, const float *a_rows, int a_pitch, cudaStream_t st) {
    if (p.total_rows == 0) return 0;
    PRB_REQUIRE(a_pitch % KC == 0 && a_pitch >= p.nchunks[0] * KC && (reinterpret_cast<uintptr_t>(a_rows) & 15) == 0,
                "mlp_wide: rows of %d floats at %p cannot feed a layer of %d K chunks", a_pitch, (const void *)a_rows, p.nchunks[0]);
    const PFN_cuTensorMapEncodeTiled_v12000 encode = tensor_map_encoder();
    PRB_REQUIRE(encode, "mlp_wide: cuTensorMapEncodeTiled is not available from the driver");
    CUtensorMap amap;
    const cuuint64_t dims[2] = {(cuuint64_t)a_pitch, (cuuint64_t)p.total_rows};
    const cuuint64_t strides[1] = {(cuuint64_t)a_pitch * sizeof(float)};
    const cuuint32_t box[2] = {KC, WM_WIDE}, estr[2] = {1, 1};
    const CUresult r = encode(&amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(a_rows), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PRB_REQUIRE(r == CUDA_SUCCESS, "mlp_wide: cuTensorMapEncodeTiled failed (%d)", (int)r);
    const int np = p.np[0];
    const size_t smem = 1024 /*alignment slack*/ + (size_t)WIDE_NB * WIDE_STAGE_BYTES + (size_t)(2 * 4 * RED_STRIDE + 3 * np) * sizeof(float);
    // two column blocks of equal width (np <= MAX_NP = 2 WN_WIDE): a 384-wide layer as 2 x 192, not 256 + 128
    const int ns = ((np >> 5) + 1) >> 1;
    const long tiles = (p.total_rows + WM_WIDE - 1) / WM_WIDE * ((np + 32 * ns - 1) / (32 * ns));
    int sms = num_sms();
    if (const int v = opts().mlp_sms; v >= 1 && v < sms) sms = v;
    auto go = [&](auto kern) -> int {
        PRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<(int)(tiles < sms ? tiles : sms), WIDE_THREADS, smem, st>>>(amap, p);
        return check_launch("mlp_wide_kernel");
    };
    static_assert(MAX_NP == 2 * WN_WIDE, "mlp_wide: two column blocks cover every layer");
    switch (ns) {   // np in (WN_WIDE, MAX_NP]: 5 .. 8 subtiles per block
        case 5: return go(mlp_wide_kernel<5>);
        case 6: return go(mlp_wide_kernel<6>);
        case 7: return go(mlp_wide_kernel<7>);
        default: return go(mlp_wide_kernel<8>);
    }
}

// layer 0's A operand as rows of `pitch` floats (the padded K of layer 0) for a wide first layer
static int launch_gather(const ChainParams &p, float *rows, int pitch, cudaStream_t st) {
    const long tiles = (p.total_rows + TM - 1) / TM;
    if (tiles == 0) return 0;
    mlp_gather_kernel<<<dim3((unsigned)tiles, (unsigned)p.nchunks[0]), 128, 0, st>>>(p, rows, pitch);
    return check_launch("mlp_gather_kernel");
}

// can layers [l0, l1) run as one launch: the activations of the widest inner layer and two weight stages in shared memory
static bool fits(const LayerGeom *g, int l0, int l1) {
    int np[MAX_LAYERS];
    for (int l = l0; l < l1; ++l) np[l - l0] = g[l].np;
    size_t fixed = 0;
    return segment_smem(np, l1 - l0, 2, 1, nullptr, nullptr, &fixed) + fixed <= 227 * 1024;
}

struct ChainIO {
    int kind, split;          // packing kind (0 SA, 1 FP, 2 DIRECT) and its split argument
    ChainParams base;         // mode_in / sources / output filled by the caller
    long rows;
};

// The launches of a chain: every layer wider than WN_WIDE alone on the wide kernel, the layers between them fused in as
// few launches as shared memory allows (each the longest run from its first layer that fits).  Returns the end of the
// launch that starts at layer l0.
static int segment_end(const LayerGeom *g, int L, int l0) {
    if (g[l0].np > WN_WIDE) return l0 + 1;
    int l1 = l0 + 1;
    while (l1 < L && g[l1].np <= WN_WIDE) ++l1;
    while (l1 > l0 + 1 && !fits(g, l0, l1)) --l1;
    return l1;
}

// Two ping-pong row buffers, each of the widest rows a launch of the chain reads from global memory: the output of
// every launch but the last, and layer 0's gathered operand where the first layer is wide.  0 when the chain is one
// fused launch.
static size_t chain_workspace_bytes(long rows, int L, int kind, int c_in, int split, const int *c_out) {
    PackSegs ps;
    default_segs(kind, c_in, split, &ps);
    LayerGeom g[MAX_LAYERS];
    chain_geometry(L, ps.nseg, ps.width, c_out, g, nullptr);
    int wmax = g[0].np > WN_WIDE ? g[0].k_chunks * KC : 0;
    for (int l0 = 0, l1; l0 < L; l0 = l1) {
        l1 = segment_end(g, L, l0);
        if (l1 < L && g[l1 - 1].np > wmax) wmax = g[l1 - 1].np;
    }
    const size_t rows_pad = (size_t)((rows + TM - 1) / TM * TM);
    return wmax ? 2 * (rows_pad * wmax * sizeof(float) + 256) : 256;
}

// run the whole chain as the launches segment_end picks, materialising rows between them
static int run_chain(const ChainIO &io, const prb_mlp_desc *mlp, void *workspace, size_t workspace_bytes, cudaStream_t st) {
    const int L = mlp->num_layers;
    PRB_REQUIRE(io.rows < 0x7fffff00L, "mlp: %ld rows exceed the 2^31 row limit", io.rows);
    PRB_REQUIRE(L >= 1 && L <= MAX_LAYERS, "mlp: num_layers %d unsupported", L);
    PackSegs ps;
    default_segs(io.kind, mlp->c_in, io.split, &ps);
    LayerGeom g[MAX_LAYERS];
    chain_geometry(L, ps.nseg, ps.width, mlp->c_out, g, nullptr);
    for (int l = 0; l < L; ++l) PRB_REQUIRE(g[l].np <= MAX_NP, "mlp: layer width %d > %d unsupported", mlp->c_out[l], MAX_NP);
    size_t soff[MAX_LAYERS];
    size_t so = 0;
    for (int l = 0; l < L; ++l) { soff[l] = so; so += (size_t)g[l].np; }

    const long rows_pad = (io.rows + TM - 1) / TM * TM;
    // the next ping-pong buffer for rows of `width` floats
    int pingpong = 0;
    auto row_buffer = [&](int width, float **dst) -> int {
        const size_t buf_bytes = (size_t)rows_pad * width * sizeof(float);
        PRB_REQUIRE(workspace && workspace_bytes >= 2 * buf_bytes, "mlp: workspace too small (%zu < %zu)", workspace_bytes, 2 * buf_bytes);
        *dst = (float *)((char *)workspace + (pingpong ? workspace_bytes / 2 / 256 * 256 : 0));
        pingpong ^= 1;
        return 0;
    };
    const float *cur_rows = nullptr;
    int cur_pitch = 0;
    for (int l0 = 0, l1; l0 < L; l0 = l1) {
        l1 = segment_end(g, L, l0);
        const bool wide = g[l0].np > WN_WIDE;
        ChainParams p = io.base;
        p.unit_scale = mlp->scale ? 0 : 1;
        p.linear_last = (l1 == L && (mlp->flags & 1)) ? 1 : 0;
        p.total_rows = io.rows;
        p.num_layers = l1 - l0;
        for (int l = l0; l < l1; ++l) {
            const int i = l - l0;
            p.nchunks[i] = g[l].k_chunks;
            p.np[i] = g[l].np;
            p.w[i] = mlp->packed_w + g[l].w_off;
            p.scale[i] = mlp->scale ? mlp->scale + soff[l] : nullptr;
            p.shift[i] = mlp->shift + soff[l];
        }
        if (l0 == 0) {
            p.nseg = ps.nseg;
            for (int s = 0; s < ps.nseg; ++s) { p.seg_chunks[s] = round_up(ps.width[s], KC) / KC; p.seg_width[s] = ps.width[s]; }
            if (wide) {   // gather layer 0's operand into rows first
                float *dst = nullptr;
                if (int rc = row_buffer(g[0].k_chunks * KC, &dst)) return rc;
                if (int rc = launch_gather(p, dst, g[0].k_chunks * KC, st)) return rc;
                cur_rows = dst;
                cur_pitch = g[0].k_chunks * KC;
            }
        } else {  // continue from materialised rows
            p.mode_in = IN_DIRECT;
            p.x_rows = cur_rows;
            p.x_pitch = cur_pitch;
            p.x2_rows = nullptr;
            p.nseg = 1; p.seg_chunks[0] = g[l0].k_chunks; p.seg_width[0] = cur_pitch;
        }
        float *dst = nullptr;
        if (l1 < L) {  // materialise this launch's activations as rows
            if (int rc = row_buffer(g[l1 - 1].np, &dst)) return rc;
            p.mode_out = OUT_ROWS;
            p.round_out = 1;
            p.out_pm = nullptr;
            p.out = dst;
            p.out_pitch = g[l1 - 1].np;
            p.c_last = g[l1 - 1].np;
        } else {
            // row-major output: write the padded width so the padding channels are defined (zero)
            p.c_last = p.mode_out == OUT_ROWS ? g[L - 1].np : mlp->c_out[L - 1];
        }
        const int rc = wide ? launch_wide(p, cur_rows, cur_pitch, st) : launch_chain(p, st);
        if (rc) return rc;
        cur_rows = dst;
        cur_pitch = g[l1 - 1].np;
    }
    return 0;
}

}  // namespace prb

extern "C" {

PRB_API size_t prb_sa_workspace_bytes(int b, int npoint, int nsample, int c_feat, int num_layers, const int *c_out) {
    return chain_workspace_bytes((long)b * npoint * nsample, num_layers, 0, 3 + c_feat, c_feat, c_out);
}
PRB_API size_t prb_fp_workspace_bytes(int b, int n, int c_known, int c_skip, int num_layers, const int *c_out) {
    return chain_workspace_bytes((long)b * n, num_layers, 1, c_known + c_skip, c_known, c_out);
}
PRB_API size_t prb_rows_workspace_bytes(long rows, int c_in, int num_layers, const int *c_out) {
    return chain_workspace_bytes(rows, num_layers, 2, c_in, 0, c_out);
}

PRB_API int prb_sa_group_mlp_max_ws(int b, int n, int npoint, int nsample, int c_feat, const float *xyz, const float *new_xyz,
                                    const float *feats_pm, const int *idx, const prb_mlp_desc *mlp, float *out, float *out_pm,
                                    int out_stride_c, int out_c_off, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && n > 0 && npoint > 0 && nsample > 0 && xyz && new_xyz && idx && mlp && out, "sa_group_mlp_max: bad arguments");
    PRB_REQUIRE(mlp->c_in == 3 + c_feat, "sa_group_mlp_max: c_in %d != 3 + c_feat %d", mlp->c_in, c_feat);
    PRB_REQUIRE(c_feat == 0 || feats_pm, "sa_group_mlp_max: features missing");
    PRB_REQUIRE(nsample >= 4 && nsample <= 128 && (nsample & (nsample - 1)) == 0, "sa_group_mlp_max: nsample %d must be a power of two in [4,128]", nsample);
    if (b == 0) return 0;
    ChainIO io;
    memset(&io, 0, sizeof(io));
    io.kind = 0; io.split = c_feat;
    io.rows = (long)b * npoint * nsample;
    io.base.mode_in = IN_SA; io.base.mode_out = OUT_SA_MAX;
    io.base.n = n; io.base.npoint = npoint; io.base.ns = nsample; io.base.c_feat = c_feat;
    io.base.log_ns = 0;
    while ((1 << io.base.log_ns) < nsample) ++io.base.log_ns;
    io.base.xyz = xyz; io.base.new_xyz = new_xyz; io.base.feats_pm = feats_pm; io.base.idx = idx;
    io.base.out = out; io.base.out_pm = out_pm; io.base.out_stride_c = out_stride_c; io.base.out_c_off = out_c_off;
    return run_chain(io, mlp, workspace, workspace_bytes, (cudaStream_t)stream);
}

PRB_API int prb_fp_interp_mlp_ws(int b, int n, int m, int c_known, int c_skip, const float *known_pm, const int *idx,
                                 const float *weight, const float *skip, const prb_mlp_desc *mlp, float *out, float *out_pm,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && n > 0 && m > 0 && c_known > 0 && known_pm && idx && weight && mlp && out, "fp_interp_mlp: bad arguments");
    PRB_REQUIRE(mlp->c_in == c_known + c_skip, "fp_interp_mlp: c_in %d != %d + %d", mlp->c_in, c_known, c_skip);
    PRB_REQUIRE(c_skip == 0 || skip, "fp_interp_mlp: skip features missing");
    if (b == 0) return 0;
    ChainIO io;
    memset(&io, 0, sizeof(io));
    io.kind = 1; io.split = c_known;
    io.rows = (long)b * n;
    io.base.mode_in = IN_FP; io.base.mode_out = OUT_FP;
    io.base.n = n; io.base.m = m; io.base.c_known = c_known; io.base.c_skip = c_skip;
    io.base.known_pm = known_pm; io.base.idx = idx; io.base.weight = weight; io.base.skip = skip;
    io.base.out = out; io.base.out_pm = out_pm; io.base.out_stride_c = mlp->c_out[mlp->num_layers - 1]; io.base.out_c_off = 0;
    return run_chain(io, mlp, workspace, workspace_bytes, (cudaStream_t)stream);
}

// plain rows -> MLP -> rows (also the unit-test doorway of the tensor-core chain)
PRB_API int prb_mlp_rows(long rows, int c_in, const float *x_rows, const prb_mlp_desc *mlp, float *out_rows, int out_pitch,
                         void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(rows >= 0 && c_in > 0 && x_rows && mlp && out_rows, "mlp_rows: bad arguments");
    PRB_REQUIRE(mlp->c_in == c_in, "mlp_rows: c_in mismatch");
    const int np_last = (mlp->c_out[mlp->num_layers - 1] + 31) / 32 * 32;
    PRB_REQUIRE(out_pitch >= np_last && (out_pitch & 3) == 0, "mlp_rows: out_pitch %d must be >= %d and a multiple of 4", out_pitch, np_last);
    if (rows == 0) return 0;
    ChainIO io;
    memset(&io, 0, sizeof(io));
    io.kind = 2; io.split = 0;
    io.rows = rows;
    io.base.mode_in = IN_DIRECT; io.base.mode_out = OUT_ROWS;
    io.base.x_rows = x_rows; io.base.x_pitch = c_in;
    io.base.out = out_rows; io.base.out_pitch = out_pitch;
    return run_chain(io, mlp, workspace, workspace_bytes, (cudaStream_t)stream);
}

PRB_API size_t prb_rows2_workspace_bytes(long rows, int c_a, int c_b, int num_layers, const int *c_out) {
    return chain_workspace_bytes(rows, num_layers, c_b > 0 ? 1 : 2, c_a + c_b, c_b > 0 ? c_a : 0, c_out);
}

PRB_API int prb_mlp_rows2(long rows, int c_a, const float *a_rows, int a_pitch, int c_b, const float *b_rows, int b_pitch,
                          const prb_mlp_desc *mlp, float *out_rows, int out_pitch, void *workspace, size_t workspace_bytes,
                          void *stream) {
    PRB_REQUIRE(rows >= 0 && c_a > 0 && a_rows && a_pitch >= c_a && mlp && out_rows, "mlp_rows2: bad arguments");
    PRB_REQUIRE(c_b >= 0 && (c_b == 0 || (b_rows && b_pitch >= c_b)), "mlp_rows2: bad second segment");
    PRB_REQUIRE(mlp->c_in == c_a + c_b, "mlp_rows2: c_in %d != %d + %d", mlp->c_in, c_a, c_b);
    const int np_last = (mlp->c_out[mlp->num_layers - 1] + 31) / 32 * 32;
    PRB_REQUIRE(out_pitch >= np_last && (out_pitch & 3) == 0, "mlp_rows2: out_pitch %d must be >= %d and a multiple of 4", out_pitch, np_last);
    if (rows == 0) return 0;
    ChainIO io;
    memset(&io, 0, sizeof(io));
    io.kind = c_b > 0 ? 1 : 2; io.split = c_b > 0 ? c_a : 0;      // weights packed with prb_mlp_pack_weights_ex(kind, split, ...)
    io.rows = rows;
    io.base.mode_in = IN_DIRECT; io.base.mode_out = OUT_ROWS;
    io.base.x_rows = a_rows; io.base.x_pitch = a_pitch;
    io.base.x2_rows = c_b > 0 ? b_rows : nullptr; io.base.x2_pitch = b_pitch;
    io.base.out = out_rows; io.base.out_pitch = out_pitch;
    return run_chain(io, mlp, workspace, workspace_bytes, (cudaStream_t)stream);
}

// header forms without an explicit workspace: valid only for chains that need no split
int prb_sa_group_mlp_max(int b, int n, int npoint, int nsample, int c_feat, const float *xyz, const float *new_xyz,
                         const float *feats_pm, const int *idx, const prb_mlp_desc *mlp, float *out, int out_stride_c,
                         int out_c_off, void *stream) {
    return prb_sa_group_mlp_max_ws(b, n, npoint, nsample, c_feat, xyz, new_xyz, feats_pm, idx, mlp, out, nullptr, out_stride_c,
                                   out_c_off, nullptr, 0, stream);
}
int prb_fp_interp_mlp(int b, int n, int m, int c_known, int c_skip, const float *known_pm, const int *idx, const float *weight,
                      const float *skip, const prb_mlp_desc *mlp, float *out, void *stream) {
    return prb_fp_interp_mlp_ws(b, n, m, c_known, c_skip, known_pm, idx, weight, skip, mlp, out, nullptr, nullptr, 0, stream);
}

}  // extern "C"
