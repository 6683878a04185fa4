// mlp_dev.cuh -- constants, launch parameters and PTX wrappers of the tensor-core chain kernels (mlp_tc.cu).
#pragma once
#include <math_constants.h>

#include "common.cuh"

namespace prb {

constexpr int TM = 64;               // rows per tile (= wgmma M)
constexpr int KC = 32;               // K columns per chunk (128 bytes of fp32/tf32: one SWIZZLE_128B row)
constexpr int A_STAGE_BYTES = TM * KC * 4;        // 8 KB: one K chunk of a tile's A operand
constexpr int A_SLOTS = 3;           // layer-0 A chunks in flight (gather of chunk k overlaps the MMAs of chunk k-1)
constexpr int NB_MAX = 4;            // weight ring depth upper bound (runtime depth in ChainParams)
constexpr int MAX_LAYERS = 3;
constexpr int MAX_NP = 512;
constexpr int NSUB_MAX = 8;          // 32-column subtiles per warpgroup (2 warpgroups x 8 x 32 = MAX_NP; wgmma N <= 256)
constexpr int RED_STRIDE = MAX_NP;   // SA pool: floats per warp of the per-warp maxima of a centre spanning several warps
static_assert(4 * RED_STRIDE * 4 <= A_STAGE_BYTES, "the per-warp pool maxima fit in the smallest work region");
constexpr int CHAIN_THREADS = 2 * 128 + 32;       // two MMA / epilogue warpgroups + one weight-producer warp
// Threads of the streaming kernel with NS column subtiles per warpgroup and T tiles per CTA.  9 warps put 3 on one SM
// sub-partition (16384 registers), so no thread gets more than 168 registers; a pair of 128-wide column halves needs 128
// accumulators and more.  There the producer is a whole warpgroup that gives its registers to the MMA warpgroups with
// setmaxnreg: 40 + 2 x 232 per sub-partition.
constexpr int chain_threads(int ns, int t) { return t == 2 && ns > 2 ? 3 * 128 : CHAIN_THREADS; }
constexpr int PRODUCER_REGS = 40, MMA_REGS = 232;
constexpr int RES_NP_MAX = 128;      // resident kernel: widest layer (one warpgroup covers it: <= 64 accumulator registers)
constexpr int RES_WG_MAX = 5;        // resident kernel: warpgroups per CTA, at most

enum { IN_SA = 0, IN_FP = 1, IN_DIRECT = 2 };
enum { OUT_ROWS = 0, OUT_SA_MAX = 1, OUT_FP = 2 };

struct ChainParams {
    int mode_in, mode_out, num_layers;
    int nchunks[MAX_LAYERS];   // K chunks per layer
    int np[MAX_LAYERS];        // padded N (multiple of 32)
    const float *w[MAX_LAYERS];      // packed weight images
    const float *scale[MAX_LAYERS];  // np floats (zero padded); unused when unit_scale
    const float *shift[MAX_LAYERS];
    int unit_scale;                  // 1: the per-channel scale is folded into the packed weights, epilogues only add shift
    int linear_last;                 // the last layer of the chain has no ReLU (heads: y = W x + shift)
    int round_out;                   // OUT_ROWS: round to tf32 (intermediate segment of a split chain)
    // resources (sized per launch)
    int nb;                          // weight ring depth
    int b_stage_bytes;               // weight stage = one K chunk of the widest layer: max np * 128 bytes
    int work_bytes;                  // layer-0 A ring / resident activations / pool maxima (aliased, see the kernel)
    // layer-0 K segments (each padded to a multiple of KC)
    int nseg, seg_chunks[2], seg_width[2];
    long total_rows;
    int num_tiles;
    int tiles_per_item;              // SA max-pool over more samples than a tile holds: consecutive tiles of one CTA
    int num_items;
    // SA
    int n, npoint, ns, log_ns, c_feat;
    const float *xyz, *new_xyz, *feats_pm;
    const int *idx;
    // FP
    int m, c_known, c_skip;
    const float *known_pm, *weight, *skip;
    // DIRECT
    const float *x_rows;
    int x_pitch;
    const float *x2_rows;   // IN_DIRECT, second K segment (nullptr: one segment)
    int x2_pitch;
    // output
    float *out;
    float *out_pm;       // optional second copy of the final output in point-major layout (rows x out_stride_c)
    int c_last;          // true channel count of the last layer
    int out_stride_c, out_c_off, out_pitch;
};

// ------------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t s2u(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D_%=;\n\t"
        "bra W_%=;\n\t"
        "D_%=:\n\t}" ::"r"(bar), "r"(parity)
        : "memory");
}
// bulk (TMA engine) global->shared copy that completes `bytes` of transaction count on the mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// generic-proxy shared-memory stores become visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// per-thread register budget of the executing warpgroup (every thread of it runs the instruction)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers are written asynchronously: keep the compiler from moving their uses across a wait
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D(64 x 32*NSUB, fp32 registers) (+)= A(64x8, smem desc) * B(32*NSUB x 8, smem desc)^T, tf32 operands, both K-major:
// one wgmma m64nNk8 (N = 32*NSUB) on the first 16*NSUB registers of the flat accumulator d.  Register 16j + q of
// thread T in warp w of the warpgroup: row 16w + T/4 + 8*((q>>1)&1), column 32j + 8*(q>>2) + 2*(T%4) + (q&1) -- the
// m64nN fragment is NSUB m64n32 fragments side by side.
#define PRB_REGS0 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
#define PRB_REGS1 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define PRB_REGS2 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
#define PRB_REGS3 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define PRB_REGS4 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79"
#define PRB_REGS5 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
#define PRB_REGS6 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111"
#define PRB_REGS7 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
#define PRB_ACC4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define PRB_ACC16(i) PRB_ACC4(i), PRB_ACC4(i + 4), PRB_ACC4(i + 8), PRB_ACC4(i + 12)
// N: instruction width; REGS: the accumulator operands; IA, IB, IS: operand numbers of a_desc, b_desc, accumulate
#define PRB_WGMMA_TF32(N, REGS, IA, IB, IS, ...)                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" IS ", 0;\n\t"                                           \
                 "wgmma.mma_async.sync.aligned.m64n" N "k8.f32.tf32.tf32 {" REGS "}, %" IA ", %" IB ", p, 1, 1;\n\t}" \
                 : __VA_ARGS__                                                                                     \
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate))
template <int NSUB, int NS>
__device__ __forceinline__ void wgmma_tf32(float (&d)[16 * NS], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    static_assert(NSUB >= 1 && NSUB <= NS && NS <= NSUB_MAX, "wgmma_tf32: 1 <= NSUB <= NS <= NSUB_MAX");
    if constexpr (NSUB == 1) {
        PRB_WGMMA_TF32("32", PRB_REGS0, "16", "17", "18", PRB_ACC16(0));
    } else if constexpr (NSUB == 2) {
        PRB_WGMMA_TF32("64", PRB_REGS0 "," PRB_REGS1, "32", "33", "34", PRB_ACC16(0), PRB_ACC16(16));
    } else if constexpr (NSUB == 3) {
        PRB_WGMMA_TF32("96", PRB_REGS0 "," PRB_REGS1 "," PRB_REGS2, "48", "49", "50", PRB_ACC16(0), PRB_ACC16(16),
                       PRB_ACC16(32));
    } else if constexpr (NSUB == 4) {
        PRB_WGMMA_TF32("128", PRB_REGS0 "," PRB_REGS1 "," PRB_REGS2 "," PRB_REGS3, "64", "65", "66", PRB_ACC16(0),
                       PRB_ACC16(16), PRB_ACC16(32), PRB_ACC16(48));
    } else if constexpr (NSUB == 5) {
        PRB_WGMMA_TF32("160", PRB_REGS0 "," PRB_REGS1 "," PRB_REGS2 "," PRB_REGS3 "," PRB_REGS4, "80", "81", "82",
                       PRB_ACC16(0), PRB_ACC16(16), PRB_ACC16(32), PRB_ACC16(48), PRB_ACC16(64));
    } else if constexpr (NSUB == 6) {
        PRB_WGMMA_TF32("192", PRB_REGS0 "," PRB_REGS1 "," PRB_REGS2 "," PRB_REGS3 "," PRB_REGS4 "," PRB_REGS5, "96", "97",
                       "98", PRB_ACC16(0), PRB_ACC16(16), PRB_ACC16(32), PRB_ACC16(48), PRB_ACC16(64), PRB_ACC16(80));
    } else if constexpr (NSUB == 7) {
        PRB_WGMMA_TF32("224", PRB_REGS0 "," PRB_REGS1 "," PRB_REGS2 "," PRB_REGS3 "," PRB_REGS4 "," PRB_REGS5 "," PRB_REGS6,
                       "112", "113", "114", PRB_ACC16(0), PRB_ACC16(16), PRB_ACC16(32), PRB_ACC16(48), PRB_ACC16(64),
                       PRB_ACC16(80), PRB_ACC16(96));
    } else {
        PRB_WGMMA_TF32("256",
                       PRB_REGS0 "," PRB_REGS1 "," PRB_REGS2 "," PRB_REGS3 "," PRB_REGS4 "," PRB_REGS5 "," PRB_REGS6
                                 "," PRB_REGS7,
                       "128", "129", "130", PRB_ACC16(0), PRB_ACC16(16), PRB_ACC16(32), PRB_ACC16(48), PRB_ACC16(64),
                       PRB_ACC16(80), PRB_ACC16(96), PRB_ACC16(112));
    }
}
#undef PRB_WGMMA_TF32
#undef PRB_ACC16
#undef PRB_ACC4
#undef PRB_REGS0
#undef PRB_REGS1
#undef PRB_REGS2
#undef PRB_REGS3
#undef PRB_REGS4
#undef PRB_REGS5
#undef PRB_REGS6
#undef PRB_REGS7

// relu + round-to-nearest-even to tf32 in ONE instruction
__device__ __forceinline__ float relu_to_tf32(float x) {
    uint32_t r;
    asm("cvt.rn.relu.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// round-to-nearest-even to tf32 (cvt.rna would expand to a 4-instruction sequence)
__device__ __forceinline__ float to_tf32(float x) {
    uint32_t r;
    asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// wgmma shared-memory descriptor: K-major, SWIZZLE_128B, 8-row atoms of 1024 bytes (stride byte offset); the
// operand tile starts 1024-byte aligned.  +2 in the address field = +32 bytes = the next K=8 step inside the row.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address
    d |= (uint64_t)1 << 16;                         // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset
    d |= (uint64_t)1 << 62;                         // SWIZZLE_128B
    return d;
}
// byte offset of (row r, 16-byte unit j) inside a K-major SWIZZLE_128B chunk
__device__ __forceinline__ uint32_t swz(int r, int j) { return (uint32_t)(r * 128 + ((j ^ (r & 7)) << 4)); }

// the source rows of one 64-row tile, filled before its layer-0 gather
struct TileRows {
    int src[TM][3];      // SA: global point row (slot 0); FP: 3 known rows
    float aux[TM][3];    // SA: centre xyz; FP: 3 weights
    int valid[TM];
};

// static shared memory of the streaming kernel: the row tables of its T tiles and the weight ring's mbarriers
template <int T>
struct SmemFixed {
    TileRows rows[T];
    uint64_t b_full[NB_MAX], b_empty[NB_MAX];
};

// dynamic shared memory of one launch: work region, weight ring, scale / shift of every layer, pool carry of the last layer
__host__ __device__ inline size_t chain_smem_bytes(int work_bytes, int nb, int b_stage_bytes, int np_total, int np_last) {
    return 1024 /*alignment slack*/ + (size_t)work_bytes + (size_t)nb * b_stage_bytes + (size_t)(2 * np_total + np_last) * sizeof(float);
}

struct RingPos {
    uint32_t stage, phase;
    __device__ void advance(int depth) {
        if (++stage == (uint32_t)depth) { stage = 0; phase ^= 1; }
    }
};

// barrier over the two MMA warpgroups of the streaming kernel
__device__ __forceinline__ void bar_mma() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// barrier over the 128 threads of one warpgroup: named barrier `id` (streaming kernel: 2 + wg; resident kernel: 1 + wg)
// (immediate ids: ptxas then reserves only the barriers a kernel uses)
__device__ __forceinline__ void bar_wg_id(int id) {
    static_assert(RES_WG_MAX <= 5, "bar_wg_id: ids 1..6");
    switch (id) {
        case 1: asm volatile("bar.sync 1, 128;" ::: "memory"); break;
        case 2: asm volatile("bar.sync 2, 128;" ::: "memory"); break;
        case 3: asm volatile("bar.sync 3, 128;" ::: "memory"); break;
        case 4: asm volatile("bar.sync 4, 128;" ::: "memory"); break;
        case 5: asm volatile("bar.sync 5, 128;" ::: "memory"); break;
        default: asm volatile("bar.sync 6, 128;" ::: "memory"); break;
    }
}

}  // namespace prb
