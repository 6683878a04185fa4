// proposal.cu -- RPN proposal path on the device, without a host round trip (SURVEY.md section 8(f) rank 1).
//
// Replaces decode_bbox_target (lib/utils/bbox_transform.py:24-121, as called from lib/rpn/proposal_layer.py:23-32)
// and ProposalLayer.forward's per-scene Python loop (lib/rpn/proposal_layer.py:34-142: boolean-mask compaction by
// distance range, two slices, boxes3d_to_bev, NMS through the C++ extension with a D2H of the keep list, two torch.cat).
//
// decode: one thread per point, every torch op of the reference reproduced as ONE fp32 rounding (__fmul_rn /
// __fadd_rn, so nvcc cannot contract them into FMAs) => bit-identical boxes.
//
// selection + NMS: one CTA per (scene, distance range).  The CTA walks torch.sort's score order once, compacting the
// points of its range (first 6300 / 2700 of them, lists in shared memory).  NMS then exploits that only the first
// post_top_n survivors are ever used (proposal_layer.py:111, :140): greedy NMS in score order is "keep box i iff no
// EARLIER KEPT box overlaps it by more than the threshold" -- identical to the reference's full N x N bitmask followed
// by its sequential scan -- so candidates are tested against the <= post_top_n kept boxes only, 32 at a time (8 warps
// split the kept list; warp 0 resolves the 32 x 32 interactions inside the chunk in order), and the walk stops as
// soon as post_top_n boxes are kept: ~1e5 IoU evaluations instead of the 2e7 of a 6300 x 6300 mask.  The IoU is the
// bitmask kernel's (iou3d_dev.cuh: the kept list and each chunk as BoxPre in shared memory, a polygon scratch column
// per thread), with its argument order: suppressor first.
#include "iou3d_dev.cuh"

namespace prb {

struct DecodeParams {
    long n;
    int c, nb, nh, xz_fine;
    float bin_size, half_bin, scope, apc, half_apc, two_pi, pi;
    float anchor[3];
    const float *xyz, *reg;
    float *out;
};

__global__ void __launch_bounds__(256) decode_proposals_kernel(const DecodeParams p) {
    const long i = (long)blockIdx.x * 256 + threadIdx.x;
    if (i >= p.n) return;
    const float *r = p.reg + i * p.c;
    const float *q = p.xyz + i * 3;
    const int nb = p.nb;
    auto argmax = [&](int lo, int cnt) {          // first maximum, as torch.argmax: a NaN is the maximum
        int best = 0;
        float bv = __ldg(r + lo);
        for (int k = 1; k < cnt; ++k) {
            const float v = __ldg(r + lo + k);
            if (v > bv || (v != v && bv == bv)) { bv = v; best = k; }
        }
        return best;
    };
    const int xb = argmax(0, nb), zb = argmax(nb, nb);
    float px = __fsub_rn(__fadd_rn(__fmul_rn((float)xb, p.bin_size), p.half_bin), p.scope);   // bbox_transform.py:52-53
    float pz = __fsub_rn(__fadd_rn(__fmul_rn((float)zb, p.bin_size), p.half_bin), p.scope);
    int start = 2 * nb;
    if (p.xz_fine) {                                                                          // :55-67
        px = __fadd_rn(px, __fmul_rn(__ldg(r + 2 * nb + xb), p.bin_size));
        pz = __fadd_rn(pz, __fmul_rn(__ldg(r + 3 * nb + zb), p.bin_size));
        start = 4 * nb;
    }
    const float py = __fadd_rn(q[1], __ldg(r + start));                                       // :84
    start += 1;
    const int rb = argmax(start, p.nh);                                                       // :90
    const float rres = __fmul_rn(__ldg(r + start + p.nh + rb), p.half_apc);                   // :99
    float ry = __fadd_rn(__fmul_rn((float)rb, p.apc), rres);                                  // :102
    float m = fmodf(ry, p.two_pi);                                                            // torch.remainder
    if (m != 0.f && m < 0.f) m = __fadd_rn(m, p.two_pi);
    if (m > p.pi) m = __fsub_rn(m, p.two_pi);                                                 // :103
    const int s = start + 2 * p.nh;
    const float h = __fadd_rn(__fmul_rn(__ldg(r + s), p.anchor[0]), p.anchor[0]);             // :110
    const float w = __fadd_rn(__fmul_rn(__ldg(r + s + 1), p.anchor[1]), p.anchor[1]);
    const float l = __fadd_rn(__fmul_rn(__ldg(r + s + 2), p.anchor[2]), p.anchor[2]);
    float *o = p.out + i * 7;
    o[0] = __fadd_rn(px, q[0]);                                                               // :119
    o[1] = __fadd_rn(py, __fdiv_rn(h, 2.0f));                                                 // proposal_layer.py:32
    o[2] = __fadd_rn(pz, q[2]);
    o[3] = h; o[4] = w; o[5] = l;
    o[6] = m;
}

// ------------------------------------------------------------------------------------------ selection + NMS
constexpr int PL_THREADS = 256;
constexpr int PL_WARPS = PL_THREADS / 32;

struct ProposalParams {
    int b, n;
    int areas;                 // 2: distance based (0,40] / (40,80]; 1: score based
    int pre[2], post[2];       // per area
    float thresh;
    int normal;                // axis-aligned IoU (nms_normal_gpu) instead of the rotated one
    const float *boxes;        // (b, n, 7) decoded, y = bottom centre
    const float *scores;       // (b, n)
    const long long *order;    // (b, n) torch.sort(descending) indices
    float *out_boxes;          // (b, post[0] + post[1], 7)
    float *out_scores;         // (b, post[0] + post[1])
    float *tmp;                // (b, post[1], 8) second-area survivors {box, score}
    int *counts;               // (b, 2)
};

// IoU of a suppressor (a kept box or an earlier candidate) with a candidate; the axis-aligned one (nms_normal_gpu)
// reads only the unrotated extent
__device__ __forceinline__ float nms_iou(bool normal, const BoxPre &s, const BoxPre &c, float *px, float *py, float *pa) {
    if (normal) {
        const float a[4] = {s.x1, s.y1, s.x2, s.y2}, b[4] = {c.x1, c.y1, c.x2, c.y2};
        return iou_normal(a, b);
    }
    return iou_bev(s, c, px, py, pa, PL_THREADS);
}

__global__ void __launch_bounds__(PL_THREADS) proposal_select_nms_kernel(const ProposalParams p) {
    extern __shared__ float s_dyn[];
    __shared__ BoxPre s_chunk[32];
    __shared__ int s_wsum[2][PL_WARPS];
    __shared__ unsigned s_sup[PL_WARPS];
    __shared__ int s_nk, s_cnt[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.y, area = blockIdx.x;
    const int cap = p.pre[area], post = p.post[area];
    // shared memory: polygon scratch (3 x POLY_SLOTS x PL_THREADS), kept boxes (post), candidate list (cap), fallback list
    // (area 1 of 2 only: cap), kept indices (post)
    float *px = s_dyn + tid, *py = px + POLY_SLOTS * PL_THREADS, *pa = py + POLY_SLOTS * PL_THREADS;
    BoxPre *kept_box = reinterpret_cast<BoxPre *>(s_dyn + 3 * POLY_SLOTS * PL_THREADS);
    int *cand = reinterpret_cast<int *>(kept_box + post);
    int *fall = cand + cap;
    int *kidx = fall + ((p.areas == 2 && area == 1) ? cap : 0);
    const float *boxes = p.boxes + (size_t)scene * p.n * 7;
    const long long *order = p.order + (size_t)scene * p.n;

    // ---- phase 1: my candidates in score order (proposal_layer.py:75-103 / :128-133)
    if (tid == 0) { s_cnt[0] = 0; s_cnt[1] = 0; s_nk = 0; }
    __syncthreads();
    const int skip_first = (p.areas == 2 && area == 1) ? p.pre[0] : 0;    // fallback = first-area entries [pre0, pre0 + pre1)
    for (int i0 = 0; i0 < p.n; i0 += PL_THREADS) {
        const int i = i0 + tid;
        bool f0 = false, f1 = false;
        int idx = 0;
        if (i < p.n) {
            idx = (int)order[i];
            if (p.areas == 1) {
                f0 = true;
            } else {
                const float z = boxes[(size_t)idx * 7 + 2];
                const bool near = z > 0.f && z <= 40.f, far = z > 40.f && z <= 80.f;
                f0 = area == 0 ? near : far;
                f1 = area == 1 && near;
            }
        }
        const unsigned b0 = __ballot_sync(0xffffffffu, f0), b1 = __ballot_sync(0xffffffffu, f1);
        if (lane == 0) { s_wsum[0][warp] = __popc(b0); s_wsum[1][warp] = __popc(b1); }
        __syncthreads();
        int base0 = s_cnt[0], base1 = s_cnt[1], tot0 = 0, tot1 = 0;
        for (int w = 0; w < PL_WARPS; ++w) {
            if (w < warp) { base0 += s_wsum[0][w]; base1 += s_wsum[1][w]; }
            tot0 += s_wsum[0][w]; tot1 += s_wsum[1][w];
        }
        const unsigned lt = (1u << lane) - 1u;
        if (f0) { const int pos = base0 + __popc(b0 & lt); if (pos < cap) cand[pos] = idx; }
        if (f1) { const int pos = base1 + __popc(b1 & lt) - skip_first; if (pos >= 0 && pos < cap) fall[pos] = idx; }
        __syncthreads();
        if (tid == 0) { s_cnt[0] += tot0; s_cnt[1] += tot1; }
        __syncthreads();
        if (s_cnt[0] >= cap) break;          // list full: later entries are never used
    }
    int ncand = min(s_cnt[0], cap);
    if (p.areas == 2 && area == 1 && s_cnt[0] == 0) {     // no point in the far range: the next slice of the near range (:97-103)
        cand = fall;
        ncand = max(0, min(s_cnt[1] - skip_first, cap));
    }

    // ---- phase 2: greedy NMS in score order until `post` boxes are kept
    int nk = 0;
    for (int c0 = 0; c0 < ncand && nk < post; c0 += 32) {
        const int c = c0 + lane;
        const bool valid = c < ncand;
        if (warp == 0 && valid) {
            float bev[5];
            box7_to_bev(boxes + (size_t)cand[c] * 7, bev);                       // kitti_utils.py:134-147
            BoxPre &b = s_chunk[lane];
            if (p.normal) { b.x1 = bev[0]; b.y1 = bev[1]; b.x2 = bev[2]; b.y2 = bev[3]; }     // nms_iou reads the extent only
            else box_pre(bev, b);
        }
        __syncthreads();
        const BoxPre &mine = s_chunk[lane];
        // suppressed by an already kept box?  the 8 warps split the kept list
        bool sup = false;
        if (valid)
            for (int k = warp; k < nk && !sup; k += PL_WARPS) sup = nms_iou(p.normal, kept_box[k], mine, px, py, pa) > p.thresh;
        const unsigned sw = __ballot_sync(0xffffffffu, sup);
        if (lane == 0) s_sup[warp] = sw;
        __syncthreads();
        if (warp == 0) {
            unsigned dead = 0;
            for (int w = 0; w < PL_WARPS; ++w) dead |= s_sup[w];
            const unsigned alive = __ballot_sync(0xffffffffu, valid) & ~dead;
            // interactions inside the chunk: bit j of `hit` = candidate j (earlier) overlaps me too much
            unsigned hit = 0;
            if ((alive >> lane) & 1u)
                for (int j = 0; j < lane; ++j)
                    if (((alive >> j) & 1u) && nms_iou(p.normal, s_chunk[j], mine, px, py, pa) > p.thresh) hit |= 1u << j;
            unsigned kept = 0, removed = 0;
            for (int j = 0; j < 32; ++j) {
                const unsigned col = __ballot_sync(0xffffffffu, (hit >> j) & 1u);    // whom does candidate j suppress
                if (((alive >> j) & 1u) && !((removed >> j) & 1u)) { kept |= 1u << j; removed |= col; }
            }
            if ((kept >> lane) & 1u) {
                const int pos = nk + __popc(kept & ((1u << lane) - 1u));
                if (pos < post) {
                    kidx[pos] = cand[c];
                    kept_box[pos] = mine;
                }
            }
            if (lane == 0) s_nk = min(post, nk + __popc(kept));
        }
        __syncthreads();
        nk = s_nk;
    }

    // ---- phase 3: survivors.  Area 0 owns rows [0, nk); area 1 parks its rows for proposal_pack_kernel
    for (int k = warp; k < nk; k += PL_WARPS) {
        const int idx = kidx[k];
        if (area == 0) {
            if (lane < 7) p.out_boxes[((size_t)scene * (p.post[0] + (p.areas == 2 ? p.post[1] : 0)) + k) * 7 + lane] = boxes[(size_t)idx * 7 + lane];
            if (lane == 7) p.out_scores[(size_t)scene * (p.post[0] + (p.areas == 2 ? p.post[1] : 0)) + k] = p.scores[(size_t)scene * p.n + idx];
        } else {
            if (lane < 7) p.tmp[((size_t)scene * p.post[1] + k) * 8 + lane] = boxes[(size_t)idx * 7 + lane];
            if (lane == 7) p.tmp[((size_t)scene * p.post[1] + k) * 8 + 7] = p.scores[(size_t)scene * p.n + idx];
        }
    }
    if (tid == 0) p.counts[scene * 2 + area] = nk;
}

// second-area rows behind the first-area rows (torch.cat, proposal_layer.py:116-117), zeros behind both (:39-40)
__global__ void __launch_bounds__(256) proposal_pack_kernel(const ProposalParams p) {
    const int scene = blockIdx.x, tid = threadIdx.x;
    const int total = p.post[0] + (p.areas == 2 ? p.post[1] : 0);
    const int n0 = p.counts[scene * 2], n1 = p.areas == 2 ? p.counts[scene * 2 + 1] : 0;
    float *ob = p.out_boxes + (size_t)scene * total * 7;
    float *os = p.out_scores + (size_t)scene * total;
    for (int e = tid; e < n1 * 8; e += 256) {
        const int k = e >> 3, t = e & 7;
        const float v = p.tmp[((size_t)scene * p.post[1] + k) * 8 + t];
        if (t < 7) ob[(size_t)(n0 + k) * 7 + t] = v; else os[n0 + k] = v;
    }
    for (int e = (n0 + n1) * 7 + tid; e < total * 7; e += 256) ob[e] = 0.f;
    for (int e = n0 + n1 + tid; e < total; e += 256) os[e] = 0.f;
}

}  // namespace prb

using namespace prb;

extern "C" {

PRB_API int prb_decode_rpn_proposals(long n, int c, const float *xyz, const float *reg, const float *anchor_hwl, float loc_scope,
                                     float loc_bin_size, int num_head_bin, int get_xz_fine, float *out, void *stream) {
    PRB_REQUIRE(n >= 0 && xyz && reg && anchor_hwl && out && loc_bin_size > 0.f && num_head_bin > 0, "decode_rpn_proposals: bad arguments");
    if (n == 0) return 0;
    DecodeParams p;
    p.n = n; p.c = c;
    p.nb = (int)(loc_scope / loc_bin_size) * 2;                    // bbox_transform.py:41 (python float division, int())
    p.nh = num_head_bin; p.xz_fine = get_xz_fine ? 1 : 0;
    PRB_REQUIRE(c == (get_xz_fine ? 4 : 2) * p.nb + 1 + 2 * num_head_bin + 3, "decode_rpn_proposals: %d regression channels do not match the bin layout", c);
    const double bs = (double)loc_bin_size, apc = (2.0 * 3.141592653589793) / (double)num_head_bin;
    p.bin_size = loc_bin_size; p.half_bin = (float)(bs / 2.0); p.scope = loc_scope;
    p.apc = (float)apc; p.half_apc = (float)(apc / 2.0);
    p.two_pi = (float)(2.0 * 3.141592653589793); p.pi = (float)3.141592653589793;
    for (int t = 0; t < 3; ++t) p.anchor[t] = anchor_hwl[t];
    p.xyz = xyz; p.reg = reg; p.out = out;
    decode_proposals_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    return check_launch("decode_proposals_kernel");
}

PRB_API size_t prb_rpn_proposals_workspace_bytes(int b, int post_nms_top_n) { return (size_t)b * ((size_t)post_nms_top_n * 8 * 4 + 8) + 256; }

// boxes (b,n,7) from prb_decode_rpn_proposals, scores (b,n), order (b,n) = indices of a descending sort of scores
// -> out_boxes (b, post_nms_top_n, 7), out_scores (b, post_nms_top_n); no host synchronisation
PRB_API int prb_rpn_proposals(int b, int n, const float *boxes, const float *scores, const long long *order, int distance_based,
                              int pre_nms_top_n, int post_nms_top_n, float nms_thresh, int normal_nms, float *out_boxes,
                              float *out_scores, void *workspace, size_t workspace_bytes, void *stream) {
    PRB_REQUIRE(b >= 0 && n > 0 && boxes && scores && order && out_boxes && out_scores && workspace && pre_nms_top_n > 0 && post_nms_top_n > 0,
                "rpn_proposals: bad arguments");
    if (b == 0) return 0;
    PRB_REQUIRE(workspace_bytes >= prb_rpn_proposals_workspace_bytes(b, post_nms_top_n), "rpn_proposals: workspace too small");
    ProposalParams p;
    p.b = b; p.n = n; p.thresh = nms_thresh; p.normal = normal_nms ? 1 : 0;
    p.boxes = boxes; p.scores = scores; p.order = order; p.out_boxes = out_boxes; p.out_scores = out_scores;
    if (distance_based) {   // proposal_layer.py:66-69
        p.areas = 2;
        p.pre[0] = (int)(pre_nms_top_n * 0.7); p.pre[1] = pre_nms_top_n - p.pre[0];
        p.post[0] = (int)(post_nms_top_n * 0.7); p.post[1] = post_nms_top_n - p.post[0];
    } else {
        p.areas = 1;
        p.pre[0] = pre_nms_top_n; p.pre[1] = 0; p.post[0] = post_nms_top_n; p.post[1] = 0;
    }
    char *w = (char *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    p.counts = (int *)w;
    p.tmp = (float *)(w + (((size_t)b * 8 + 255) & ~(size_t)255));
    PRB_REQUIRE(workspace_bytes >= (size_t)((char *)(p.tmp + (size_t)b * (p.post[1] > 0 ? p.post[1] : 1) * 8) - (char *)workspace), "rpn_proposals: workspace too small");
    // shared memory: 4 bytes per candidate (8 in area 1 of 2: the fallback list), 68 per kept box (index + BoxPre) and
    // 192 per thread (polygon scratch: 48 KB); pre / post top-n of 9000 / 512 in one area need 117 KB
    size_t smem = 0;
    for (int a = 0; a < p.areas; ++a) {
        const size_t s = (size_t)p.pre[a] * ((p.areas == 2 && a == 1) ? 2 : 1) * sizeof(int) + (size_t)p.post[a] * (sizeof(int) + sizeof(BoxPre)) +
                         (size_t)3 * POLY_SLOTS * PL_THREADS * sizeof(float);
        smem = s > smem ? s : smem;
    }
    PRB_REQUIRE(smem <= 200 * 1024, "rpn_proposals: pre/post top-n of %d/%d need %zu bytes of shared memory", pre_nms_top_n, post_nms_top_n, smem);
    PRB_CUDA(cudaFuncSetAttribute(proposal_select_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaStream_t st = (cudaStream_t)stream;
    proposal_select_nms_kernel<<<dim3(p.areas, b), PL_THREADS, smem, st>>>(p);
    if (int rc = check_launch("proposal_select_nms_kernel")) return rc;
    proposal_pack_kernel<<<b, 256, 0, st>>>(p);
    return check_launch("proposal_pack_kernel");
}

}  // extern "C"
