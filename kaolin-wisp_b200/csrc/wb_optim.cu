// wb_optim.cu -- Adam over the whole model in ONE launch (SURVEY.md 8(f) rank 2).
// The reference builds torch.optim.Adam / RMSprop with three parameter groups (decoder: weight decay; grid: lr * grid_lr_weight;
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
