// rev_index.cuh -- reverse index of a reference list, and the fixed-order gather-sum over it (csrc/rev_index.cu).
//
// References: b scenes of L references each, flat index q = s * L + l; reference q names the source point idx[q] of its
// scene (0 <= idx[q] < n; a reference outside that range is ignored).  The index lists, for every source j = s * n +
// idx[q], its references in list[off[j] .. off[j + 1]) in increasing q.  It is a counting sort: counts and slots use
// integer atomics, and a per-source sort fixes the order, so the index is the same on every call.
//
// Users: the FP training backward (3 taps per unknown point), the ordered grouping / gather / interpolation gradients (fp32
// and bfloat16) and the SA training backward's feature gradient (nsample references per centre, 1 per gathered point).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace prb {

struct RevIndex {
    int b, L, n;
    int *cnt;     // (b n) scratch counts
    int *off;     // (b n + 1) list offsets
    int *tot;     // per-block totals of the offset scan
    int *list;    // (b L) references grouped by source
};

// scratch bytes of the index (each part 256-byte aligned), and the index laid out at `ws`.  b * L and b * n must be below
// 2^31 (rev_index_fits).
size_t rev_index_bytes(int b, int L, int n);
RevIndex rev_index_at(int b, int L, int n, void *ws);
bool rev_index_fits(long b, long L, long n);

// builds the index of idx (b * L int32) on stream s: one memset and six launches, no host synchronisation
int rev_index_build(const RevIndex &R, const int *idx, cudaStream_t s);

// The value of reference q = s * L + l in channel ch:
//   SEG_GROUP  g (b, c, L)                      g[(s c + ch) L + l]
//   SEG_TAPS   g (b, c, L / 3), w (b L)         g[(s c + ch) (L / 3) + l / 3] * w[q]     (one fp32 product, rounded)
//   SEG_ROWS   g (b L, c)                       g[q c + ch]
enum { SEG_GROUP, SEG_TAPS, SEG_ROWS };
constexpr int kSegCh = 8;   // channels per thread of the gather-sum

// out (b, c, n): for every source j of scene s and channel ch, acc = +0.0f, then acc = acc + v over the source's
// references in increasing q (each add rounded to nearest, no contraction), then out = out + acc (accumulate) or out = acc.
int seg_sum(const RevIndex &R, int kind, int c, const float *g, const float *w, bool accumulate, float *out, cudaStream_t s);

// the same sum over bfloat16 values (each converted exactly to fp32; SEG_TAPS: the fp32 product with w rounded as above),
// then out = acc rounded once to bfloat16 (to nearest even), written: out is not read
int seg_sum_bf16(const RevIndex &R, int kind, int c, const __nv_bfloat16 *g, const float *w, __nv_bfloat16 *out, cudaStream_t s);

// out[i] = in[i] rounded to bfloat16 (to nearest even) for i < count: the last pass of the atomic bfloat16 gradients, which
// sum into fp32 scratch first
int round_bf16(size_t count, const float *in, void *out, cudaStream_t s);

}  // namespace prb
