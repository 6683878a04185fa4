// adam.cu -- the optimizer step of recipe.TrueWDAdam (fastai OptimWrapper true_wd + Adam) with lr and beta1 read from
// device memory, so that a CUDA graph that captured the step follows OneCycle's per-iteration values on every replay.
// torch's fused Adam takes beta1 as a host double, which a capture would freeze.
//
// Per element it computes what the eager step computes, bit for bit: torch._foreach_mul_(p, 1 - wd * lr) with the
// factor formed in double and rounded once to float, then the arithmetic of torch's fused Adam kernel
// (ATen/native/cuda/fused_adam_utils.cuh, adam_math with weight_decay 0, no amsgrad, no grad scale) in fp32 with its
// operation order written out as _rn intrinsics so that contraction cannot change it.
#include "common.cuh"

namespace prb {

constexpr int kAdamThreads = 256;
constexpr int kAdamBlocksPerTensor = 16;

__global__ void __launch_bounds__(kAdamThreads) adam_true_wd_kernel(const prb_adam_tensor *__restrict__ tensors,
                                                                    const double *__restrict__ hyper, double wd, double eps) {
    const prb_adam_tensor t = tensors[blockIdx.y];
    const double lr_d = hyper[0];
    const float lr = (float)lr_d, b1 = (float)hyper[1], b2 = (float)hyper[2], ep = (float)eps;
    const float decay = (float)__dsub_rn(1.0, __dmul_rn(wd, lr_d));
    const float steps = *t.step;
    const float bc1 = __fsub_rn(1.0f, powf(b1, steps));
    const float bc2_sqrt = __fsqrt_rn(__fsub_rn(1.0f, powf(b2, steps)));
    const float step_size = __fdiv_rn(lr, bc1);
    for (long long i = (long long)blockIdx.x * kAdamThreads + threadIdx.x; i < t.numel; i += (long long)gridDim.x * kAdamThreads) {
        const float p = __fmul_rn(t.param[i], decay);
        const float g = t.grad[i];
        const float gg = __fmul_rn(g, g);
        const float m = __fmaf_rn(b1, t.exp_avg[i], __fmaf_rn(-b1, g, g));
        const float v = __fmaf_rn(b2, t.exp_avg_sq[i], __fmaf_rn(-b2, gg, gg));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), ep);
        t.param[i] = __fsub_rn(p, __fdiv_rn(__fmul_rn(step_size, m), denom));
        t.exp_avg[i] = m;
        t.exp_avg_sq[i] = v;
    }
}

}  // namespace prb

using namespace prb;

extern "C" int prb_adam_true_wd_step(int n, const prb_adam_tensor *tensors, const double *hyper, double weight_decay, double eps,
                                     void *stream) {
    PRB_REQUIRE(n >= 0 && n <= 65535 && (n == 0 || (tensors && hyper)), "adam_true_wd_step: bad arguments (n = %d)", n);
    if (n == 0) return 0;
    adam_true_wd_kernel<<<dim3(kAdamBlocksPerTensor, n), kAdamThreads, 0, (cudaStream_t)stream>>>(tensors, hyper, weight_decay, eps);
    return check_launch("adam_true_wd_kernel");
}
