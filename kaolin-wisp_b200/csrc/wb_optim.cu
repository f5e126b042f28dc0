// wb_optim.cu -- the optimiser step over the whole model in ONE launch (SURVEY.md 8(f) rank 2): Adam, AdamW, RMSprop.
// The reference builds torch.optim.Adam / AdamW / RMSprop with three parameter groups (decoder: weight decay; grid: lr * grid_lr_weight;
// rest) in BaseTrainer.init_optimizer (wisp/trainers/base_trainer.py:205-235) and steps it once per batch
// (multiview_trainer.py:168-174).  Here every tensor of every group is one segment of a single grid-stride launch:
//   g  = grad * grad_scale (+ weight_decay * p)                    grad_scale folds the 1/world of the gradient all-reduce
//   m  = b1 m + (1 - b1) g ;  v = b2 v + (1 - b2) g^2              torch.optim.Adam (amsgrad = False, maximize = False)
//   p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// and the gradient is zeroed as it is consumed, so the 42 MB gradient table needs no separate memset per step
// (optimizer.zero_grad(), multiview_trainer.py:123).  fp32 master weights and moments; 28 bytes moved per parameter.
#include "wb_common.cuh"

#define WB_ADAM_MAX_SEG 64
struct WbAdamSeg { float* p; float* g; float* m; float* v; int64_t n; float lr, wd; };
struct WbAdam { WbAdamSeg seg[WB_ADAM_MAX_SEG]; int nseg; float b1, b2, eps, bc1, bc2_sqrt, grad_scale; int zero_grad; };
// The step description travels as a kernel parameter: the launch copies it, so the host may build the next step's description
// while this one is still queued (a host staging buffer + cudaMemcpyAsync would be overwritten by a host running steps ahead).
static_assert(sizeof(WbAdam) <= 4096, "WbAdam must fit the 4 KB kernel parameter space");

__global__ void __launch_bounds__(256)
wb_adam_kernel(const __grid_constant__ WbAdam A)
{
    const float b1 = A.b1, b2 = A.b2, eps = A.eps, bc1 = A.bc1, bc2s = A.bc2_sqrt, gs = A.grad_scale;
    for (int k = 0; k < A.nseg; ++k) {
        const WbAdamSeg sg = A.seg[k];
        const float step_size = sg.lr / bc1;
        const int64_t n4 = ((reinterpret_cast<uintptr_t>(sg.p) | reinterpret_cast<uintptr_t>(sg.g) | reinterpret_cast<uintptr_t>(sg.m) |
                             reinterpret_cast<uintptr_t>(sg.v)) & 15u) == 0 ? sg.n / 4 : 0;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            float4 p = reinterpret_cast<float4*>(sg.p)[i], g = reinterpret_cast<float4*>(sg.g)[i];
            float4 m = reinterpret_cast<float4*>(sg.m)[i], v = reinterpret_cast<float4*>(sg.v)[i];
            float* pp = &p.x; float* gp = &g.x; float* mp = &m.x; float* vp = &v.x;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float gg = gp[c] * gs; if (sg.wd != 0.0f) gg = fmaf(sg.wd, pp[c], gg);
                mp[c] = fmaf(b1, mp[c], (1.0f - b1) * gg);
                vp[c] = fmaf(b2, vp[c], (1.0f - b2) * gg * gg);
                pp[c] -= step_size * (mp[c] / (sqrtf(vp[c]) / bc2s + eps));
            }
            reinterpret_cast<float4*>(sg.p)[i] = p; reinterpret_cast<float4*>(sg.m)[i] = m; reinterpret_cast<float4*>(sg.v)[i] = v;
            if (A.zero_grad) reinterpret_cast<float4*>(sg.g)[i] = make_float4(0, 0, 0, 0);
        }
        for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < sg.n; i += (int64_t)gridDim.x * blockDim.x) {
            float gg = sg.g[i] * gs; if (sg.wd != 0.0f) gg = fmaf(sg.wd, sg.p[i], gg);
            const float m = fmaf(b1, sg.m[i], (1.0f - b1) * gg), v = fmaf(b2, sg.v[i], (1.0f - b2) * gg * gg);
            sg.m[i] = m; sg.v[i] = v;
            sg.p[i] -= step_size * (m / (sqrtf(v) / bc2s + eps));
            if (A.zero_grad) sg.g[i] = 0.0f;
        }
    }
}

// segs: HOST array of nseg wb_adam_segment, read before this call returns
extern "C" int wb_adam_step(const wb_adam_segment* segs, int32_t nseg, float beta1, float beta2, float eps, int32_t step, float grad_scale,
                            int32_t zero_grad, wb_stream s)
{
    WB_CHECK_ARG(segs, "null pointer");
    WB_CHECK_ARG(nseg >= 1 && nseg <= WB_ADAM_MAX_SEG && step >= 1, "nseg must be 1..64 and step >= 1");
    WbAdam A{};
    int64_t total = 0;
    for (int k = 0; k < nseg; ++k) {
        WB_CHECK_ARG(segs[k].param && segs[k].grad && segs[k].exp_avg && segs[k].exp_avg_sq && segs[k].numel >= 0, "bad segment");
        A.seg[k] = WbAdamSeg{ segs[k].param, segs[k].grad, segs[k].exp_avg, segs[k].exp_avg_sq, segs[k].numel, segs[k].lr, segs[k].weight_decay };
        total += segs[k].numel;
    }
    A.nseg = nseg; A.b1 = beta1; A.b2 = beta2; A.eps = eps; A.grad_scale = grad_scale; A.zero_grad = zero_grad;
    A.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
    A.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
    int64_t ctas = (total / 4 + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 8; if (ctas > cap) ctas = cap; if (ctas < 1) ctas = 1;
    wb_adam_kernel<<<(unsigned)ctas, 256, 0, (cudaStream_t)s>>>(A);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---- AdamW and RMSprop (wisp/config/presets/torch.py:37-67: ConfigAdamW, ConfigRMSprop; apex FusedAdam's default is AdamW) ------
// The same launch shape and contract as wb_adam_kernel, one instance per rule.  Every fp32 operation is spelled out, so the chain
// below IS the contract (tests/optim_reference.py follows it bit for bit); torch's separate kernels round elsewhere where noted.
//   AdamW    p' = fl(p * decay)                          decay = fl32(1 - lr * wd), formed by the host in double (torch: the same)
//            g  = fl(grad * grad_scale)
//            m  = fma(b1, m, fl((1 - b1) g))             torch: lerp, m + (1 - b1)(g - m)
//            v  = fma(b2, v, fl(fl((1 - b2) g) g))       torch: mul_(b2) then addcmul_, two roundings more
//            p  = fma(-fl(lr / bc1), fl(m / fl(fl(sqrt(v) / bc2_sqrt) + eps)), p')
//   RMSprop  g  = fl(grad * grad_scale), wd != 0: g = fma(wd, p, g)
//            sq = fma(alpha, sq, fl(fl((1 - alpha) g) g))
//            q  = fl(g / fl(sqrt(sq) + eps))
//            momentum == 0: p = fma(-lr, q, p)           torch: addcdiv_, the same up to its own contraction
//            otherwise:     buf = fma(momentum, buf, q) ; p = fma(-lr, buf, p)
enum { WB_RULE_ADAMW = 0, WB_RULE_RMSPROP = 1, WB_RULE_RMSPROP_MOMENTUM = 2 };
// s0 / s1: exp_avg / exp_avg_sq (AdamW), square_avg / momentum_buffer (RMSprop; s1 unused without momentum).  wd: AdamW's decay factor.
struct WbRuleSeg { float* p; float* g; float* s0; float* s1; int64_t n; float lr, wd; };
// c0 / c1: beta1 / beta2 (AdamW), alpha / momentum (RMSprop)
struct WbRule { WbRuleSeg seg[WB_ADAM_MAX_SEG]; int nseg; float c0, c1, eps, bc1, bc2_sqrt, grad_scale; int zero_grad; };
static_assert(sizeof(WbRule) <= 4096, "WbRule must fit the 4 KB kernel parameter space");

template <int RULE>
__device__ __forceinline__ void wb_rule_update(const WbRule& A, const WbRuleSeg& sg, float step_size, float& p, float g, float& s0, float& s1)
{
    float gg = __fmul_rn(g, A.grad_scale);
    if (RULE == WB_RULE_ADAMW) {
        const float pd = __fmul_rn(p, sg.wd);
        s0 = fmaf(A.c0, s0, __fmul_rn(1.0f - A.c0, gg));
        s1 = fmaf(A.c1, s1, __fmul_rn(__fmul_rn(1.0f - A.c1, gg), gg));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(s1), A.bc2_sqrt), A.eps);
        p = fmaf(-step_size, __fdiv_rn(s0, denom), pd);
    } else {
        if (sg.wd != 0.0f) gg = fmaf(sg.wd, p, gg);
        s0 = fmaf(A.c0, s0, __fmul_rn(__fmul_rn(1.0f - A.c0, gg), gg));
        const float q = __fdiv_rn(gg, __fadd_rn(__fsqrt_rn(s0), A.eps));
        if (RULE == WB_RULE_RMSPROP_MOMENTUM) { s1 = fmaf(A.c1, s1, q); p = fmaf(-sg.lr, s1, p); }
        else p = fmaf(-sg.lr, q, p);
    }
}

template <int RULE>
__global__ void __launch_bounds__(256)
wb_rule_kernel(const __grid_constant__ WbRule A)
{
    constexpr bool S1 = RULE != WB_RULE_RMSPROP;            // the second state tensor exists
    for (int k = 0; k < A.nseg; ++k) {
        const WbRuleSeg sg = A.seg[k];
        const float step_size = RULE == WB_RULE_ADAMW ? __fdiv_rn(sg.lr, A.bc1) : 0.0f;
        const int64_t n4 = ((reinterpret_cast<uintptr_t>(sg.p) | reinterpret_cast<uintptr_t>(sg.g) | reinterpret_cast<uintptr_t>(sg.s0) |
                             (S1 ? reinterpret_cast<uintptr_t>(sg.s1) : 0)) & 15u) == 0 ? sg.n / 4 : 0;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            float4 p = reinterpret_cast<float4*>(sg.p)[i], g = reinterpret_cast<float4*>(sg.g)[i];
            float4 a = reinterpret_cast<float4*>(sg.s0)[i], b = S1 ? reinterpret_cast<float4*>(sg.s1)[i] : make_float4(0, 0, 0, 0);
            float* pp = &p.x; float* gp = &g.x; float* ap = &a.x; float* bp = &b.x;
#pragma unroll
            for (int c = 0; c < 4; ++c) wb_rule_update<RULE>(A, sg, step_size, pp[c], gp[c], ap[c], bp[c]);
            reinterpret_cast<float4*>(sg.p)[i] = p; reinterpret_cast<float4*>(sg.s0)[i] = a;
            if (S1) reinterpret_cast<float4*>(sg.s1)[i] = b;
            if (A.zero_grad) reinterpret_cast<float4*>(sg.g)[i] = make_float4(0, 0, 0, 0);
        }
        for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < sg.n; i += (int64_t)gridDim.x * blockDim.x) {
            float p = sg.p[i], a = sg.s0[i], b = S1 ? sg.s1[i] : 0.0f;
            wb_rule_update<RULE>(A, sg, step_size, p, sg.g[i], a, b);
            sg.p[i] = p; sg.s0[i] = a;
            if (S1) sg.s1[i] = b;
            if (A.zero_grad) sg.g[i] = 0.0f;
        }
    }
}

template <int RULE>
static int wb_rule_launch(WbRule& A, int64_t total, wb_stream s)
{
    int64_t ctas = (total / 4 + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 8; if (ctas > cap) ctas = cap; if (ctas < 1) ctas = 1;
    wb_rule_kernel<RULE><<<(unsigned)ctas, 256, 0, (cudaStream_t)s>>>(A);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// segs: HOST array of nseg wb_adam_segment, read before this call returns
extern "C" int wb_adamw_step(const wb_adam_segment* segs, int32_t nseg, float beta1, float beta2, float eps, int32_t step, float grad_scale,
                             int32_t zero_grad, wb_stream s)
{
    WB_CHECK_ARG(segs, "null pointer");
    WB_CHECK_ARG(nseg >= 1 && nseg <= WB_ADAM_MAX_SEG && step >= 1, "nseg must be 1..64 and step >= 1");
    WbRule A{};
    int64_t total = 0;
    for (int k = 0; k < nseg; ++k) {
        WB_CHECK_ARG(segs[k].param && segs[k].grad && segs[k].exp_avg && segs[k].exp_avg_sq && segs[k].numel >= 0, "bad segment");
        const float decay = (float)(1.0 - (double)segs[k].lr * (double)segs[k].weight_decay);      // torch: param.mul_(1 - lr * weight_decay)
        A.seg[k] = WbRuleSeg{ segs[k].param, segs[k].grad, segs[k].exp_avg, segs[k].exp_avg_sq, segs[k].numel, segs[k].lr, decay };
        total += segs[k].numel;
    }
    A.nseg = nseg; A.c0 = beta1; A.c1 = beta2; A.eps = eps; A.grad_scale = grad_scale; A.zero_grad = zero_grad;
    A.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
    A.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
    return wb_rule_launch<WB_RULE_ADAMW>(A, total, s);
}

// segs: HOST array of nseg wb_rmsprop_segment, read before this call returns
extern "C" int wb_rmsprop_step(const wb_rmsprop_segment* segs, int32_t nseg, float alpha, float eps, float momentum, float grad_scale,
                               int32_t zero_grad, wb_stream s)
{
    WB_CHECK_ARG(segs, "null pointer");
    WB_CHECK_ARG(nseg >= 1 && nseg <= WB_ADAM_MAX_SEG, "nseg must be 1..64");
    WB_CHECK_ARG(momentum >= 0.0f, "momentum must be >= 0");
    WbRule A{};
    int64_t total = 0;
    for (int k = 0; k < nseg; ++k) {
        WB_CHECK_ARG(segs[k].param && segs[k].grad && segs[k].square_avg && segs[k].numel >= 0, "bad segment");
        WB_CHECK_ARG(momentum == 0.0f || segs[k].momentum_buffer, "momentum > 0 needs a momentum_buffer");
        A.seg[k] = WbRuleSeg{ segs[k].param, segs[k].grad, segs[k].square_avg, segs[k].momentum_buffer, segs[k].numel, segs[k].lr, segs[k].weight_decay };
        total += segs[k].numel;
    }
    A.nseg = nseg; A.c0 = alpha; A.c1 = momentum; A.eps = eps; A.grad_scale = grad_scale; A.zero_grad = zero_grad;
    return momentum > 0.0f ? wb_rule_launch<WB_RULE_RMSPROP_MOMENTUM>(A, total, s) : wb_rule_launch<WB_RULE_RMSPROP>(A, total, s);
}
