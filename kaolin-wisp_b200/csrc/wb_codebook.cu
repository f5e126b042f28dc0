// wb_codebook.cu -- CodebookOctreeGrid (VQAD, wisp/models/grids/codebook_grid.py:103-172), restructured ROW-WISE.
//
// The reference evaluates, for every (sample, corner) pair, a 2^bitwidth-wide softmax over the corner's logits and a
// [2^bitwidth x feature_dim] product with the dictionary (`_index_features`, :103-131) -- 8 x LODs x samples softmaxes per batch,
// almost all of them repeats, because the result depends only on the corner ROW, not on the sample.  Here the selection runs
// once per row and LOD:
//     E_l[row] = sum_k keys[row, k] * dictionary_l[k]          training: keys = y_hard - y_soft + y_soft (straight-through, :117-123)
//                                                              eval:     keys = one_hot(argmax logits)    (:128-131)
// and the per-sample work is the ordinary OctreeGrid trilinear blend of E_l through the trinkets (wb_octree_interp_*), whose
// backward hands back dE_l.  wb_codebook_rows_bwd then applies the softmax / straight-through Jacobian per row:
//     d dictionary[k] += keys[row, k] * dE[row]            d logits[row, k] = y_k * (c_k - sum_j y_j c_j),  c_k = <dictionary[k], dE[row]>
// Mathematically identical to the reference's per-(sample, corner) graph (the gradients of all samples sharing a row add up in dE).
// One warp per row, K = 2^bitwidth <= 1024 logits spread over the lanes, feature_dim <= 32.
#include "wb_common.cuh"

constexpr int WB_CB_MAXK = 1024;
constexpr int WB_CB_MAXF = 32;

__device__ __forceinline__ float wb_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// softmax statistics + argmax (lowest index among equal maxima, as torch.max) of one row held as KPL values per lane.
// Seeded with -inf, so every finite logit, -FLT_MAX included, can be a lane's maximum; padding lanes (k >= K) hold -inf and
// never win, and a lane without logits keeps mi = K and mx = -inf != gmx.  For any finite row amax lies in [0, K) and the
// maximum's expf(0) = 1 keeps the sum >= 1.
template <int KPL>
__device__ __forceinline__ void cb_row_softmax(const float* __restrict__ row, int K, int lane, float y[KPL], int& amax)
{
    float mx = -INFINITY; int mi = K;
#pragma unroll
    for (int i = 0; i < KPL; ++i) {
        const int k = lane + 32 * i;
        y[i] = k < K ? __ldg(row + k) : -INFINITY;
        if (y[i] > mx) { mx = y[i]; mi = k; }
    }
    const float gmx = wb_warp_max(mx);
    int cand = (mx == gmx) ? mi : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
    amax = cand;
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i < KPL; ++i) { const int k = lane + 32 * i; y[i] = k < K ? expf(y[i] - gmx) : 0.0f; sum += y[i]; }
    sum = wb_warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < KPL; ++i) y[i] *= inv;
}

template <int KPL>
__global__ void __launch_bounds__(256)
wb_codebook_rows_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ dict, int64_t rows, int K, int F, int training,
                            float* __restrict__ E, int32_t* __restrict__ argmax_out)
{
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < rows; r += nwarps) {
        float y[KPL]; int am;
        cb_row_softmax<KPL>(logits + r * K, K, lane, y, am);
        if (argmax_out && lane == 0) argmax_out[r] = am;
        if (!training) {                                       // dictionary[argmax]  (codebook_grid.py:128-131)
            if (lane < F) E[r * F + lane] = __ldg(dict + (int64_t)am * F + lane);
            continue;
        }
        // keys_k = (y_hard_k - y_soft_k) + y_soft_k, op by op as the reference's tensors (:117-123); E = sum_k keys_k * dict[k]
        for (int f = 0; f < F; ++f) {
            float acc = 0.0f;
#pragma unroll
            for (int i = 0; i < KPL; ++i) {
                const int k = lane + 32 * i;
                if (k < K) { const float key = ((k == am ? 1.0f : 0.0f) - y[i]) + y[i]; acc = fmaf(key, __ldg(dict + (int64_t)k * F + f), acc); }
            }
            acc = wb_warp_sum(acc);
            if (lane == 0) E[r * F + f] = acc;
        }
    }
}

template <int KPL>
__global__ void __launch_bounds__(256)
wb_codebook_rows_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ dict, const float* __restrict__ dE, int64_t rows, int K, int F,
                            float* __restrict__ g_logits, float* __restrict__ g_dict)
{
    extern __shared__ float gd[];                              // [K][F] dictionary gradient of this CTA, then [8 warps][32] dE rows
    for (int e = threadIdx.x; e < K * F; e += blockDim.x) gd[e] = 0.0f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < rows; r += nwarps) {
        const float de = lane < F ? __ldg(dE + r * F + lane) : 0.0f;
        if (__ballot_sync(0xffffffffu, de != 0.0f) == 0u) continue;     // rows no sample touched: zero gradient (g_logits is pre-zeroed)
        float* drow = gd + K * F + (threadIdx.x >> 5) * 32;              // this warp's copy of dE[row] (broadcast reads below)
        __syncwarp();
        drow[lane] = de;
        __syncwarp();
        float y[KPL]; int am;
        cb_row_softmax<KPL>(logits + r * K, K, lane, y, am);
        float c[KPL], dot = 0.0f;
#pragma unroll
        for (int i = 0; i < KPL; ++i) {
            const int k = lane + 32 * i;
            c[i] = 0.0f;
            if (k < K) {
                for (int f = 0; f < F; ++f) c[i] = fmaf(__ldg(dict + (int64_t)k * F + f), drow[f], c[i]);
                const float key = ((k == am ? 1.0f : 0.0f) - y[i]) + y[i];
                if (key != 0.0f) for (int f = 0; f < F; ++f) atomicAdd(gd + k * F + f, key * drow[f]);
                dot = fmaf(y[i], c[i], dot);
            }
        }
        dot = wb_warp_sum(dot);
#pragma unroll
        for (int i = 0; i < KPL; ++i) { const int k = lane + 32 * i; if (k < K) g_logits[r * K + k] = y[i] * (c[i] - dot); }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < K * F; e += blockDim.x) if (gd[e] != 0.0f) atomicAdd(g_dict + e, gd[e]);
}

extern "C" int wb_codebook_rows_fwd(const float* logits, const float* dictionary, int64_t rows, int32_t K, int32_t F, int32_t training,
                                    float* E, int32_t* argmax_out, wb_stream s)
{
    if (rows == 0) return WB_OK;
    WB_CHECK_ARG(logits && dictionary && E, "null pointer");
    WB_CHECK_ARG(K >= 1 && K <= WB_CB_MAXK && F >= 1 && F <= WB_CB_MAXF, "codebook: 1 <= 2^bitwidth <= 1024, feature_dim <= 32");
    int64_t ctas = (rows + 7) / 8; const int64_t cap = (int64_t)wb_num_sms() * 16; if (ctas > cap) ctas = cap;
    cudaStream_t st = (cudaStream_t)s;
    if (K <= 256) wb_codebook_rows_fwd_kernel<8><<<(unsigned)ctas, 256, 0, st>>>(logits, dictionary, rows, K, F, training, E, argmax_out);
    else wb_codebook_rows_fwd_kernel<32><<<(unsigned)ctas, 256, 0, st>>>(logits, dictionary, rows, K, F, training, E, argmax_out);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
extern "C" int wb_codebook_rows_bwd(const float* logits, const float* dictionary, const float* dE, int64_t rows, int32_t K, int32_t F,
                                    float* g_logits, float* g_dictionary, wb_stream s)
{
    if (rows == 0) return WB_OK;
    WB_CHECK_ARG(logits && dictionary && dE && g_logits && g_dictionary, "null pointer");
    WB_CHECK_ARG(K >= 1 && K <= WB_CB_MAXK && F >= 1 && F <= WB_CB_MAXF, "codebook: 1 <= 2^bitwidth <= 1024, feature_dim <= 32");
    int64_t ctas = (rows + 7) / 8; const int64_t cap = (int64_t)wb_num_sms() * 2; if (ctas > cap) ctas = cap;
    const int smem = (K * F + 8 * 32) * 4;          // dictionary gradient + one dE row per warp
    cudaStream_t st = (cudaStream_t)s;
    auto kern = K <= 256 ? wb_codebook_rows_bwd_kernel<8> : wb_codebook_rows_bwd_kernel<32>;
    WB_CUDA(wb_allow_smem(kern, smem));
    kern<<<(unsigned)ctas, 256, smem, st>>>(logits, dictionary, dE, rows, K, F, g_logits, g_dictionary);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
