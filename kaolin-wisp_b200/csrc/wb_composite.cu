// wb_composite.cu -- packed front-to-back compositing, forward and backward, one warp per ray.
// Replaces kaolin.render.spc.exponential_integration / sum_reduce and the per-ray buffer scatter of
// PackedRFTracer.trace (wisp/tracers/packed_rf_tracer.py:136-165):
//   tau = sigma*delta ; T = exp(-cumsum_excl(tau)) ; w = T*(1-exp(-tau))
//   C = sum w*c ; D = sum w*depth ; A = sum w ; rgb = bg*(1-A) + C ; hit = A > 0
// The reference runs ~10 elementwise kernels + 3 CUB scans over S-sized arrays; here each sample is read once
// (32 B) and the scan is a warp shuffle with a running carry.
#include "wb_common.cuh"

constexpr int WB_COMP_THREADS = 256;
constexpr int WB_COMP_BATCH = 4;        // rays whose first chunk is in flight together (per warp)

// A warp owns 32 CONSECUTIVE rays: lane i reads the sample range of ray r0 + i (one coalesced load instead of a dependent broadcast load
// per ray), rays without samples are finished by their lane alone, the others are composited one after the other by the whole warp
// (lane = sample, warp-shuffle scan with a running carry); every lane then writes its own ray's outputs (coalesced).
__global__ void __launch_bounds__(WB_COMP_THREADS, 4)
wb_composite_fwd_kernel(const float4* __restrict__ shaded, const float* __restrict__ depth, const float* __restrict__ deltas,
                        const int64_t* __restrict__ offsets, int64_t R, float bgr, float bgg, float bgb,
                        float* __restrict__ rgb, float* __restrict__ depth_out, float* __restrict__ alpha, uint8_t* __restrict__ hit)
{
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r0 = warp0 * 32; r0 < R; r0 += nwarps * 32) {
        const int64_t rm = r0 + lane;
        const int64_t mb = rm < R ? __ldg(offsets + rm) : 0, me = rm < R ? __ldg(offsets + rm + 1) : 0;
        float o_r = bgr, o_g = bgg, o_b = bgb, o_d = 0.0f, o_a = 0.0f;           // rgb = zeros + bg for rays without samples (:143)
        uint32_t todo = __ballot_sync(0xffffffffu, me > mb);
        // Rays are taken in batches of WB_COMP_BATCH: the first 32-sample chunk of every ray of the batch is requested before any of them is
        // composited, so four DRAM-latency loads overlap instead of one ray's samples waiting after the other (the kernel is a chain of
        // dependent loads per warp: ncu r02u long_scoreboard 9.4 per issue).  The arithmetic of a ray is unchanged.
        while (todo) {
            int js[WB_COMP_BATCH]; float4 shs[WB_COMP_BATCH]; float dls[WB_COMP_BATCH], ts[WB_COMP_BATCH];
#pragma unroll
            for (int q = 0; q < WB_COMP_BATCH; ++q) {
                js[q] = -1; shs[q] = make_float4(0, 0, 0, 0); dls[q] = 0.0f; ts[q] = 0.0f;
                if (todo) {
                    js[q] = __ffs(todo) - 1; todo &= todo - 1;
                    const int64_t b = __shfl_sync(0xffffffffu, mb, js[q]), e = __shfl_sync(0xffffffffu, me, js[q]);
                    if (b + lane < e) { shs[q] = __ldg(shaded + b + lane); dls[q] = __ldg(deltas + b + lane); ts[q] = __ldg(depth + b + lane); }
                }
            }
#pragma unroll
            for (int q = 0; q < WB_COMP_BATCH; ++q) {
                if (js[q] < 0) continue;                             // warp-uniform
                const int j = js[q];
                const int64_t b = __shfl_sync(0xffffffffu, mb, j), e = __shfl_sync(0xffffffffu, me, j);
                float4 sh = shs[q]; float dl = dls[q], t = ts[q];
                float cr = 0, cg = 0, cb = 0, dd = 0, aa = 0, carry = 0;
                for (int64_t k0 = b; k0 < e; k0 += 32) {
                    const int64_t k = k0 + lane;
                    if (k0 != b) {
                        sh = make_float4(0, 0, 0, 0); dl = 0.0f; t = 0.0f;
                        if (k < e) { sh = __ldg(shaded + k); dl = __ldg(deltas + k); t = __ldg(depth + k); }
                    }
                    const float tau = (k < e) ? sh.w * dl : 0.0f;
                    const float incl = wb_warp_incl_scan(tau, lane);
                    const float T = expf(-(carry + (incl - tau)));
                    const float w = (k < e) ? T * (1.0f - expf(-tau)) : 0.0f;
                    cr = fmaf(w, sh.x, cr); cg = fmaf(w, sh.y, cg); cb = fmaf(w, sh.z, cb); dd = fmaf(w, t, dd); aa += w;
                    carry += __shfl_sync(0xffffffffu, incl, 31);
                }
                cr = wb_warp_sum(cr); cg = wb_warp_sum(cg); cb = wb_warp_sum(cb); dd = wb_warp_sum(dd); aa = wb_warp_sum(aa);
                if (lane == j) {     // rgb[ridx_hit] = bg*(1-alpha) + ray_colors (:165)
                    o_r = bgr * (1.0f - aa) + cr; o_g = bgg * (1.0f - aa) + cg; o_b = bgb * (1.0f - aa) + cb; o_d = dd; o_a = aa;
                }
            }
        }
        if (rm < R) {
            rgb[3 * rm] = o_r; rgb[3 * rm + 1] = o_g; rgb[3 * rm + 2] = o_b;
            if (depth_out) depth_out[rm] = o_d;
            alpha[rm] = o_a; hit[rm] = o_a > 0.0f ? 1 : 0;
        }
    }
}

extern "C" int wb_composite_fwd(const float* shaded, const float* depth, const float* deltas, const int64_t* offsets, int64_t R,
                                const float* bg, float* rgb, float* depth_out, float* alpha, uint8_t* hit, wb_stream s)
{
    if (R == 0) return WB_OK;
    WB_CHECK_ARG(offsets && bg && rgb && alpha && hit, "null pointer");
    const float b3[3] = { bg[0], bg[1], bg[2] };   // host pointer (launch parameter)
    int64_t ctas = (R + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 32; if (ctas > cap) ctas = cap;      // 8 warps x 32 rays per CTA pass
    wb_composite_fwd_kernel<<<(unsigned)ctas, WB_COMP_THREADS, 0, (cudaStream_t)s>>>(
        reinterpret_cast<const float4*>(shaded), depth, deltas, offsets, R, b3[0], b3[1], b3[2], rgb, depth_out, alpha, hit);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// backward:  g_k = dL/dw_k = g_rgb.c_k + g_depth*t_k + (g_alpha - g_rgb.bg)
//            dL/dtau_k = g_k*T_{k+1} - sum_{j>k} g_j w_j      dL/dc_k = g_rgb*w_k      dL/dsigma_k = dL/dtau_k*delta_k
// pass 1 accumulates G = sum_j g_j w_j, pass 2 uses G - prefix_incl.
// LOSS: the trainer's image loss (multiview_trainer.py:140-154) is evaluated here instead of by torch: g_rgb holds the PREDICTED rgb
// (wb_composite_fwd's output), `target` the ground truth, and dL/drgb = loss'(rgb - target) * inv_count is formed per ray in
// registers; the loss value (sum over rays and channels * inv_count) is accumulated into *loss_out.
struct WbLoss { const float* target; int type; float inv_count; float* loss_out; };      // type 0 l2 (mse), 1 l1, 2 huber (smooth_l1, beta 1)
__device__ __forceinline__ float wb_loss_term(int type, float d, float& grad)
{
    if (type == 0) { grad = 2.0f * d; return d * d; }
    if (type == 1) { grad = d > 0.0f ? 1.0f : d < 0.0f ? -1.0f : 0.0f; return fabsf(d); }
    const float ad = fabsf(d);
    if (ad < 1.0f) { grad = d; return 0.5f * d * d; }
    grad = d > 0.0f ? 1.0f : -1.0f; return ad - 0.5f;
}

template <bool LOSS>
__global__ void __launch_bounds__(WB_COMP_THREADS)
wb_composite_bwd_kernel(const float4* __restrict__ shaded, const float* __restrict__ depth, const float* __restrict__ deltas,
                        const int64_t* __restrict__ offsets, int64_t R, float bgr, float bgg, float bgb,
                        const float* __restrict__ g_rgb, const float* __restrict__ g_depth, const float* __restrict__ g_alpha,
                        float4* __restrict__ g_shaded, float* __restrict__ absmax, WbLoss LS)
{
    float amax = 0.0f, lsum = 0.0f;
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r0 = warp0 * 32; r0 < R; r0 += nwarps * 32) {         // 32 consecutive rays per warp, as in the forward kernel
        const int64_t rm = r0 + lane;
        const int64_t mb = rm < R ? __ldg(offsets + rm) : 0, me = rm < R ? __ldg(offsets + rm + 1) : 0;
        float mgr = 0.0f, mgg = 0.0f, mgb = 0.0f, mgd = 0.0f, mga = 0.0f;    // this lane's ray: dL/d(rgb, depth, alpha)
        if (rm < R) {
            if (LOSS) {
                float l0 = wb_loss_term(LS.type, __ldg(g_rgb + 3 * rm) - __ldg(LS.target + 3 * rm), mgr);
                l0 += wb_loss_term(LS.type, __ldg(g_rgb + 3 * rm + 1) - __ldg(LS.target + 3 * rm + 1), mgg);
                l0 += wb_loss_term(LS.type, __ldg(g_rgb + 3 * rm + 2) - __ldg(LS.target + 3 * rm + 2), mgb);
                mgr *= LS.inv_count; mgg *= LS.inv_count; mgb *= LS.inv_count;
                lsum += l0;
            } else if (me > mb) {
                mgr = __ldg(g_rgb + 3 * rm); mgg = __ldg(g_rgb + 3 * rm + 1); mgb = __ldg(g_rgb + 3 * rm + 2);
                mgd = g_depth ? __ldg(g_depth + rm) : 0.0f; mga = g_alpha ? __ldg(g_alpha + rm) : 0.0f;
            }
        }
        uint32_t todo = __ballot_sync(0xffffffffu, me > mb);
        while (todo) {                                                    // batches of WB_COMP_BATCH rays, first chunks requested together (see the forward)
            int js[WB_COMP_BATCH]; float4 shs[WB_COMP_BATCH]; float dls[WB_COMP_BATCH], ts[WB_COMP_BATCH];
#pragma unroll
            for (int q = 0; q < WB_COMP_BATCH; ++q) {
                js[q] = -1; shs[q] = make_float4(0, 0, 0, 0); dls[q] = 0.0f; ts[q] = 0.0f;
                if (todo) {
                    js[q] = __ffs(todo) - 1; todo &= todo - 1;
                    const int64_t b = __shfl_sync(0xffffffffu, mb, js[q]), e = __shfl_sync(0xffffffffu, me, js[q]);
                    if (b + lane < e) { shs[q] = __ldg(shaded + b + lane); dls[q] = __ldg(deltas + b + lane); ts[q] = __ldg(depth + b + lane); }
                }
            }
#pragma unroll
            for (int q = 0; q < WB_COMP_BATCH; ++q) {
                if (js[q] < 0) continue;                                  // warp-uniform
                const int j = js[q];
                const int64_t b = __shfl_sync(0xffffffffu, mb, j), e = __shfl_sync(0xffffffffu, me, j);
                const float4 sh0 = shs[q]; const float dl0 = dls[q], t0 = ts[q];
                const float gr = __shfl_sync(0xffffffffu, mgr, j), gg = __shfl_sync(0xffffffffu, mgg, j), gb = __shfl_sync(0xffffffffu, mgb, j);
                const float gd = __shfl_sync(0xffffffffu, mgd, j);
                const float ga = __shfl_sync(0xffffffffu, mga, j) - (gr * bgr + gg * bgg + gb * bgb);
                if (e - b <= 32) {
                    // the whole ray is in registers: both passes without a second read (same arithmetic as the two-pass form with carry = 0)
                    const int64_t k = b + lane;
                    const bool in = k < e;
                    const float tau = in ? sh0.w * dl0 : 0.0f;
                    const float gk = in ? gr * sh0.x + gg * sh0.y + gb * sh0.z + gd * t0 + ga : 0.0f;
                    const float incl = wb_warp_incl_scan(tau, lane);
                    const float T = expf(-(0.0f + (incl - tau)));
                    const float Tn = expf(-(0.0f + incl));
                    const float w = in ? T * (1.0f - expf(-tau)) : 0.0f;
                    const float G = wb_warp_sum(fmaf(gk, w, 0.0f));
                    const float gw = gk * w;
                    const float gw_incl = wb_warp_incl_scan(gw, lane);
                    const float suffix = G - (0.0f + gw_incl);
                    const float gtau = gk * Tn - suffix;
                    if (in) {
                        const float4 gs = make_float4(gr * w, gg * w, gb * w, gtau * dl0);
                        g_shaded[k] = gs;
                        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(gs.x), fabsf(gs.y)), fmaxf(fabsf(gs.z), fabsf(gs.w))));
                    }
                    continue;
                }
                float G = 0, carry = 0;
                for (int64_t k0 = b; k0 < e; k0 += 32) {
                    const int64_t k = k0 + lane;
                    float tau = 0, gk = 0; float4 sh = sh0; float dl = dl0, t = t0;
                    if (k0 != b && k < e) { sh = __ldg(shaded + k); dl = __ldg(deltas + k); t = __ldg(depth + k); }
                    if (k < e) { tau = sh.w * dl; gk = gr * sh.x + gg * sh.y + gb * sh.z + gd * t + ga; }
                    const float incl = wb_warp_incl_scan(tau, lane);
                    const float T = expf(-(carry + (incl - tau)));
                    const float w = (k < e) ? T * (1.0f - expf(-tau)) : 0.0f;
                    G = fmaf(gk, w, G);
                    carry += __shfl_sync(0xffffffffu, incl, 31);
                }
                G = wb_warp_sum(G);
                carry = 0; float gw_carry = 0;
                for (int64_t k0 = b; k0 < e; k0 += 32) {
                    const int64_t k = k0 + lane;
                    float tau = 0, gk = 0, dl = 0; float4 sh = make_float4(0, 0, 0, 0);
                    if (k < e) { sh = __ldg(shaded + k); dl = __ldg(deltas + k); tau = sh.w * dl; gk = gr * sh.x + gg * sh.y + gb * sh.z + gd * __ldg(depth + k) + ga; }
                    const float incl = wb_warp_incl_scan(tau, lane);
                    const float T = expf(-(carry + (incl - tau)));
                    const float Tn = expf(-(carry + incl));                 // T_{k+1}
                    const float w = (k < e) ? T * (1.0f - expf(-tau)) : 0.0f;
                    const float gw = gk * w;
                    const float gw_incl = wb_warp_incl_scan(gw, lane);
                    const float suffix = G - (gw_carry + gw_incl);          // sum_{j>k} g_j w_j
                    const float gtau = gk * Tn - suffix;
                    if (k < e) {
                        const float4 gs = make_float4(gr * w, gg * w, gb * w, gtau * dl);
                        g_shaded[k] = gs;
                        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(gs.x), fabsf(gs.y)), fmaxf(fabsf(gs.z), fabsf(gs.w))));
                    }
                    carry += __shfl_sync(0xffffffffu, incl, 31);
                    gw_carry += __shfl_sync(0xffffffffu, gw_incl, 31);
                }
            }
        }
    }
    if (absmax != nullptr) {      // non-negative floats order like their bit patterns: one atomicMax per warp (NaN/Inf sort above finite values)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (lane == 0 && amax > 0.0f) atomicMax(reinterpret_cast<unsigned int*>(absmax), __float_as_uint(amax));
    }
    if (LOSS) { lsum = wb_warp_sum(lsum); if (lane == 0 && lsum != 0.0f) atomicAdd(LS.loss_out, lsum * LS.inv_count); }
}

extern "C" int wb_composite_bwd(const float* shaded, const float* depth, const float* deltas, const int64_t* offsets, int64_t R,
                                const float* bg, const float* g_rgb, const float* g_depth, const float* g_alpha,
                                float* g_shaded, float* absmax, wb_stream s)
{
    if (R == 0) return WB_OK;
    WB_CHECK_ARG(offsets && bg && g_rgb, "null pointer");
    const float b3[3] = { bg[0], bg[1], bg[2] };   // host pointer (launch parameter)
    int64_t ctas = (R + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 32; if (ctas > cap) ctas = cap;
    wb_composite_bwd_kernel<false><<<(unsigned)ctas, WB_COMP_THREADS, 0, (cudaStream_t)s>>>(
        reinterpret_cast<const float4*>(shaded), depth, deltas, offsets, R, b3[0], b3[1], b3[2], g_rgb, g_depth, g_alpha,
        reinterpret_cast<float4*>(g_shaded), absmax, WbLoss{ nullptr, 0, 0.0f, nullptr });
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// Image loss + its gradient + the compositing backward in one launch (SURVEY.md 8(f) rank 2): replaces smooth_l1_loss / mse_loss /
// abs, .mean(), their autograd kernels and the [R,3] gradient tensor of MultiviewTrainer.step (multiview_trainer.py:140-176).
// loss_out (device float, zeroed by the caller) receives sum(loss(rgb - target)) * inv_count; inv_count = 1 / (3 * rays) for
// rgb_loss_denom 'rays' (global ray count under data parallelism), 1 / prev_num_samples for 'samples'.
extern "C" int wb_composite_bwd_loss(const float* shaded, const float* depth, const float* deltas, const int64_t* offsets, int64_t R,
                                     const float* bg, const float* rgb_pred, const float* target, int32_t loss_type, float inv_count,
                                     float* g_shaded, float* absmax, float* loss_out, wb_stream s)
{
    if (R == 0) return WB_OK;
    WB_CHECK_ARG(offsets && bg && rgb_pred && target && g_shaded && loss_out, "null pointer");
    WB_CHECK_ARG(loss_type >= 0 && loss_type <= 2, "loss_type must be 0 (l2), 1 (l1) or 2 (huber)");
    const float b3[3] = { bg[0], bg[1], bg[2] };
    int64_t ctas = (R + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 32; if (ctas > cap) ctas = cap;
    wb_composite_bwd_kernel<true><<<(unsigned)ctas, WB_COMP_THREADS, 0, (cudaStream_t)s>>>(
        reinterpret_cast<const float4*>(shaded), depth, deltas, offsets, R, b3[0], b3[1], b3[2], rgb_pred, nullptr, nullptr,
        reinterpret_cast<float4*>(g_shaded), absmax, WbLoss{ target, loss_type, inv_count, loss_out });
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// Power-of-two loss scale of the fp16 decoder backward from max |g_shaded| (wb_composite_bwd's absmax): the largest gradient lands
// near 64 in fp16.  One thread; replaces five elementwise torch launches of round 1 and still needs no host sync.
__global__ void wb_loss_scale_kernel(const float* __restrict__ absmax, float* __restrict__ scale)
{
    const float amax = fmaxf(*absmax, 1e-30f);
    // floor(log2(64 / amax)) = 6 - ceil(log2(amax)), from the exponent: amax = f * 2^e with f in [0.5, 1).  (log2f(64.0f / amax)
    // rounds to the next integer for amax just above a power of two and gives a scale twice too large.)
    int e;
    const float f = frexpf(amax, &e);
    int k = isinf(amax) ? -20 : 6 - (f == 0.5f ? e - 1 : e);
    k = min(max(k, -20), 60);
    *scale = __int_as_float((k + 127) << 23);
}
extern "C" int wb_rf_loss_scale(const float* absmax, float* scale, wb_stream s)
{
    WB_CHECK_ARG(absmax && scale, "null pointer");
    wb_loss_scale_kernel<<<1, 1, 0, (cudaStream_t)s>>>(absmax, scale);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
