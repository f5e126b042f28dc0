// wb_shade.cu -- fused "shade" stage of the render path, fp32 SIMT variant (precision 0).
//
// One thread per hit sample does, without touching HBM in between, what the reference spreads over
// 16 hash-grid launches + 6 cuBLAS GEMMs + ~10 elementwise kernels (SURVEY.md 3.1):
//   sample position (fma of the ray with the record's depth)            octree_as.py:283
//   HashGrid.interpolate, all LODs, 'cat' zeroing / 'sum'               hash_grid.py:205-233, hashgrid_interpolate_cuda.cu:38-79
//   [positional embedding of coords]                                     nerf.py:240-242
//   decoder_density (Linear/relu stack)                                  nerf.py:245, basic_decoders.py:73-101
//   view embedding, decoder_color, sigmoid, relu(density)                nerf.py:248-263
// Per-sample activations live in shared memory columns (act[col*NTP + tid], NTP = NT+1: conflict free both for
// the per-thread layer loops and for the cross-thread weight-gradient reduction).  The decoder weights are
// staged once per CTA with a single bulk (TMA) copy: cp.async.bulk.shared::cluster.global + mbarrier.
//
// Backward (wb_rf_shade_bwd) recomputes the forward per tile, then per layer runs weight-grad (CTA-cooperative,
// register tiles), bias-grad and data-grad, and finally scatters dL/dfeat to the hash table with vector
// reductions (red.global.add.v2.f32).  No S-sized activation tensor ever exists in HBM.
#include "wb_common.cuh"
#include "wb_featx.cuh"
#include "wb_shade_tc.cuh"
#include <math.h>

#define WB_ML 16          // max linear layers over both decoders

extern "C" int64_t wb_rf_workspace_bytes(const wb_nef_desc* nef, int32_t precision, int64_t R, int64_t S, int32_t backward)
{
    if (precision != 1) return 0;
    return wb_tc_workspace_bytes(nef, R, S, backward);
}

// Set by wb_rf_workspace_holds_ray_rows() for the next backward call of this thread only: the backward entries take it (read and
// clear) before anything else, so a call that returns early cannot leave it behind for a later call with another workspace.
static thread_local bool g_ray_rows_ready = false;
extern "C" int wb_rf_workspace_holds_ray_rows(int32_t yes) { g_ray_rows_ready = yes != 0; return WB_OK; }
static bool wb_take_ray_rows_ready() { const bool v = g_ray_rows_ready; g_ray_rows_ready = false; return v; }

// precision-1 backward in its two stages (wb_rf_shade_bwd == decoder_bwd followed by table_scatter)
extern "C" int wb_rf_decoder_bwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                                 int64_t S, const float* g_shaded, const float* loss_scale, const void* feat_saved, void* workspace,
                                 float* grad_dens, float* grad_col, wb_stream s)
{
    const bool ray_rows_ready = wb_take_ray_rows_ready();
    if (S == 0) return WB_OK;
    WB_CHECK_ARG(nef && blob && rays && rays->origins && rays->dirs && rec_t && rec_ray && g_shaded && grad_dens && grad_col, "null pointer");
    return wb_tc_decoder_bwd_ex(nef, blob, rays, rec_t, rec_ray, S, 0, S, g_shaded, loss_scale, feat_saved, workspace, ray_rows_ready,
                                grad_dens, grad_col, nullptr, nullptr, (cudaStream_t)s);
}
extern "C" int wb_rf_table_scatter(const wb_nef_desc* nef, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray, int64_t S,
                                   const float* loss_scale, void* workspace, float* grad_table, wb_stream s)
{
    if (S == 0) return WB_OK;
    WB_CHECK_ARG(nef && rays && rays->origins && rays->dirs && rec_t && rec_ray, "null pointer");
    return wb_tc_table_scatter(nef, rays, rec_t, rec_ray, S, 0, S, loss_scale, workspace, grad_table, (cudaStream_t)s);
}
extern "C" int64_t wb_rf_feat_bytes(const wb_nef_desc* nef, int32_t precision, int64_t S)
{
    if (precision != 1) return 0;
    return wb_tc_feat_bytes(nef, S);
}
extern "C" int wb_rf_precision_supported(const wb_nef_desc* nef, int32_t precision, int32_t backward)
{
    if (precision == 0) return 1;
    if (precision != 1 || nef == nullptr) return 0;
    return wb_tc_supported(nef, backward);
}

struct WbMlp {
    int nl_d, nl_c;                      // linear layers: density, colour
    int I[WB_ML], O[WB_ML], Opad[WB_ML], Ipad[WB_ML];
    int w_off[WB_ML], b_off[WB_ML];      // section 1 (forward): Wt [I][Opad] k-major, bias [Opad]
    int wo_off[WB_ML];                   // section 2 (data-grad): W [O][Ipad] o-major
    int src_w[WB_ML], src_b[WB_ML];      // offsets into the packed nn.Linear parameter vectors (b = -1: no bias)
    int fwd_floats, total_floats;
    int act_in[WB_ML], act_out[WB_ML];   // activation column offsets
    int act_cols, maxw;
    int feat_dim, pos_dim, view_dim;
    int pos_mode, pos_freq, view_mode, view_freq;
};

static int wb_embed_dim(int mode, int freq) { return mode == 0 ? 0 : mode == 1 ? 3 : mode == 2 ? 6 * freq : 3 + 6 * freq; }
static int wb_round_up(int v, int m) { return (v + m - 1) / m * m; }

// retain = true: every layer keeps its own input/output columns (backward); false: ping-pong (forward only)
static int wb_make_mlp(const wb_nef_desc* d, bool retain, WbMlp* m)
{
    WB_CHECK_ARG(d->dens_layers >= 1 && d->col_layers >= 1 && d->dens_layers + d->col_layers <= WB_ML, "unsupported decoder depth");
    WB_CHECK_ARG(d->dens_params && d->col_params, "null decoder parameters");
    memset(m, 0, sizeof(*m));
    m->nl_d = d->dens_layers; m->nl_c = d->col_layers;
    m->feat_dim = d->multiscale == 0 ? d->num_lods * d->feature_dim : d->feature_dim;
    m->pos_mode = d->pos_mode; m->pos_freq = d->pos_freq; m->view_mode = d->view_mode; m->view_freq = d->view_freq;
    m->pos_dim = wb_embed_dim(d->pos_mode, d->pos_freq); m->view_dim = wb_embed_dim(d->view_mode, d->view_freq);
    WB_CHECK_ARG(d->dens_dims[0] == m->feat_dim + m->pos_dim, "decoder_density input width != grid features + position embedding");
    const int dout = d->dens_dims[d->dens_layers];
    WB_CHECK_ARG(dout >= 2, "decoder_density output must be >= 2 wide");
    WB_CHECK_ARG(d->col_dims[0] == dout - 1 + m->view_dim, "decoder_color input width != density feats - 1 + view embedding");
    WB_CHECK_ARG(d->col_dims[d->col_layers] == 3, "decoder_color output must be 3 wide");
    int off = 0, srcd = 0, srcc = 0, maxw = 0;
    const int nl = m->nl_d + m->nl_c;
    for (int l = 0; l < nl; ++l) {
        const bool dens = l < m->nl_d;
        const int I = dens ? d->dens_dims[l] : d->col_dims[l - m->nl_d];
        const int O = dens ? d->dens_dims[l + 1] : d->col_dims[l - m->nl_d + 1];
        WB_CHECK_ARG(I >= 1 && I <= 256 && O >= 1 && O <= 256, "layer width out of range (1..256)");
        m->I[l] = I; m->O[l] = O; m->Opad[l] = wb_round_up(O, 8); m->Ipad[l] = wb_round_up(I, 8);
        m->w_off[l] = off; off += I * m->Opad[l];
        m->b_off[l] = off; off += m->Opad[l];
        int& src = dens ? srcd : srcc;
        m->src_w[l] = src; src += I * O;
        if (d->has_bias) { m->src_b[l] = src; src += O; } else m->src_b[l] = -1;
        if (m->Ipad[l] > maxw) maxw = m->Ipad[l];
        if (m->Opad[l] > maxw) maxw = m->Opad[l];
    }
    m->fwd_floats = wb_round_up(off, 4);
    off = m->fwd_floats;
    for (int l = 0; l < nl; ++l) { m->wo_off[l] = off; off += m->O[l] * m->Ipad[l]; }
    m->total_floats = wb_round_up(off, 4);
    m->maxw = maxw;
    if (retain) {
        int c = 0;
        for (int l = 0; l < nl; ++l) {
            if (l == 0 || l == m->nl_d) { m->act_in[l] = c; c += m->Ipad[l]; }     // fresh input region per decoder
            else m->act_in[l] = m->act_out[l - 1];
            m->act_out[l] = c; c += m->Opad[l];
        }
        m->act_cols = c;
    } else {
        for (int l = 0; l < nl; ++l) {
            if (l == 0) m->act_in[l] = 0;
            else if (l == m->nl_d) m->act_in[l] = (m->act_out[l - 1] == 0) ? maxw : 0;   // colour input goes to the other buffer
            else m->act_in[l] = m->act_out[l - 1];
            m->act_out[l] = (m->act_in[l] == 0) ? maxw : 0;
        }
        m->act_cols = 2 * maxw;
    }
    return WB_OK;
}

extern "C" int64_t wb_rf_param_blob_floats(const wb_nef_desc* nef, int32_t precision)
{
    if (precision == 1) return wb_tc_blob_floats(nef);
    WbMlp m; if (wb_make_mlp(nef, false, &m)) return -1;
    return m.total_floats;
}

__global__ void wb_pack_params_kernel(WbMlp m, const float* __restrict__ dens, const float* __restrict__ col, float* __restrict__ blob)
{
    const int nl = m.nl_d + m.nl_c;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < m.total_floats; e += gridDim.x * blockDim.x) {
        float v = 0.0f;
        for (int l = 0; l < nl; ++l) {
            const float* src = l < m.nl_d ? dens : col;
            const int I = m.I[l], O = m.O[l];
            if (e >= m.w_off[l] && e < m.w_off[l] + I * m.Opad[l]) {
                const int k = (e - m.w_off[l]) / m.Opad[l], o = (e - m.w_off[l]) % m.Opad[l];
                if (o < O) v = src[m.src_w[l] + o * I + k];
            } else if (e >= m.b_off[l] && e < m.b_off[l] + m.Opad[l]) {
                const int o = e - m.b_off[l];
                if (o < O && m.src_b[l] >= 0) v = src[m.src_b[l] + o];
            } else if (e >= m.wo_off[l] && e < m.wo_off[l] + O * m.Ipad[l]) {
                const int o = (e - m.wo_off[l]) / m.Ipad[l], k = (e - m.wo_off[l]) % m.Ipad[l];
                if (k < I) v = src[m.src_w[l] + o * I + k];
            }
        }
        blob[e] = v;
    }
}

extern "C" int wb_rf_pack_params(const wb_nef_desc* nef, int32_t precision, float* blob, wb_stream s)
{
    WB_CHECK_ARG(blob != nullptr, "null blob");
    WB_CHECK_ARG(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (fp16 tensor cores)");
    if (precision == 1) return wb_tc_pack(nef, blob, (cudaStream_t)s);
    WbMlp m; int rc = wb_make_mlp(nef, false, &m); if (rc) return rc;
    wb_pack_params_kernel<<<(m.total_floats + 255) / 256, 256, 0, (cudaStream_t)s>>>(m, nef->dens_params, nef->col_params, blob);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// device pieces
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t wb_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// TMA bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP + SYNCS)
__device__ __forceinline__ void wb_bulk_stage(float* dst_smem, const float* src, uint32_t bytes, uint64_t* bar)
{
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(wb_smem_u32(bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(wb_smem_u32(bar)), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"(wb_smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(wb_smem_u32(bar)) : "memory");
    }
    __syncthreads();                                   // barrier init visible to all waiters
    uint32_t done = 0;
    while (!done) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(wb_smem_u32(bar)), "r"(0u) : "memory");
    }
}

// positional_embedder.py:51-66: winded[f*3+c] = x[c]*2^f ; out = [x?, sin(winded), cos(winded)]
__device__ __forceinline__ void wb_embed(int mode, int freq, float x, float y, float z, float* col, int NTP)
{
    if (mode == 0) return;
    int o = 0;
    if (mode == 1 || mode == 3) { col[0] = x; col[NTP] = y; col[2 * NTP] = z; o = 3; }
    if (mode == 1) return;
    float band = 1.0f;
    for (int f = 0; f < freq; ++f) {
        const float wx = x * band, wy = y * band, wz = z * band;
        col[(o + f * 3 + 0) * NTP] = sinf(wx); col[(o + f * 3 + 1) * NTP] = sinf(wy); col[(o + f * 3 + 2) * NTP] = sinf(wz);
        col[(o + 3 * freq + f * 3 + 0) * NTP] = cosf(wx); col[(o + 3 * freq + f * 3 + 1) * NTP] = cosf(wy); col[(o + 3 * freq + f * 3 + 2) * NTP] = cosf(wz);
        band *= 2.0f;
    }
}

// out[o] = act( b[o] + sum_k W[o][k]*in[k] ), k ascending (same order as the oracle).  Wt: [I][Opad] k-major.
__device__ __forceinline__ void wb_layer_fwd(const float* __restrict__ Wt, const float* __restrict__ bias,
                                             const float* in, float* out, int I, int Opad, bool relu, int NTP)
{
    for (int ob = 0; ob < Opad; ob += 8) {
        float acc[8];
        const float4 b0 = *reinterpret_cast<const float4*>(bias + ob), b1 = *reinterpret_cast<const float4*>(bias + ob + 4);
        acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w; acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
        const float* wp = Wt + ob;
#pragma unroll 4
        for (int k = 0; k < I; ++k) {
            const float x = in[k * NTP];
            const float4 w0 = *reinterpret_cast<const float4*>(wp + k * Opad), w1 = *reinterpret_cast<const float4*>(wp + k * Opad + 4);
            acc[0] = fmaf(w0.x, x, acc[0]); acc[1] = fmaf(w0.y, x, acc[1]); acc[2] = fmaf(w0.z, x, acc[2]); acc[3] = fmaf(w0.w, x, acc[3]);
            acc[4] = fmaf(w1.x, x, acc[4]); acc[5] = fmaf(w1.y, x, acc[5]); acc[6] = fmaf(w1.z, x, acc[6]); acc[7] = fmaf(w1.w, x, acc[7]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) out[(ob + j) * NTP] = relu ? fmaxf(acc[j], 0.0f) : acc[j];
    }
}

// gather all LODs of one sample into the density-decoder input columns
__device__ __forceinline__ void wb_gather(const WbGrid& g, float px, float py, float pz, float* col, int NTP)
{
    const int L = g.L, F = g.F;
    if (g.multiscale == 0) {
        for (int l = 0; l < L; ++l) {
            if (l >= g.lod_idx) { for (int f = 0; f < F; ++f) col[(l * F + f) * NTP] = 0.0f; continue; }   // hash_grid.py:226-229
            uint32_t idx[8]; float cf[8];
            wb_corner_setup(g, l, px, py, pz, idx, cf);
            const float* tb = g.table + g.begin[l] * F;
            if (F == 2) {
                float2 v[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = __ldg(reinterpret_cast<const float2*>(tb) + idx[j]);
                float a0 = v[0].x * cf[0], a1 = v[0].y * cf[0];
#pragma unroll
                for (int j = 1; j < 8; ++j) { a0 = fmaf(v[j].x, cf[j], a0); a1 = fmaf(v[j].y, cf[j], a1); }
                col[(l * 2) * NTP] = a0; col[(l * 2 + 1) * NTP] = a1;
            } else {
                for (int f = 0; f < F; ++f) {
                    float a = __ldg(tb + (int64_t)idx[0] * F + f) * cf[0];
#pragma unroll
                    for (int j = 1; j < 8; ++j) a = fmaf(__ldg(tb + (int64_t)idx[j] * F + f), cf[j], a);
                    col[(l * F + f) * NTP] = a;
                }
            }
        }
    } else {     // 'sum' over LODs (hash_grid.py:230-231), level order
        float s[8];
        for (int f = 0; f < F; ++f) s[f] = 0.0f;
        for (int l = 0; l < L; ++l) {
            uint32_t idx[8]; float cf[8];
            wb_corner_setup(g, l, px, py, pz, idx, cf);
            const float* tb = g.table + g.begin[l] * F;
            for (int f = 0; f < F; ++f) {
                float a = __ldg(tb + (int64_t)idx[0] * F + f) * cf[0];
#pragma unroll
                for (int j = 1; j < 8; ++j) a = fmaf(__ldg(tb + (int64_t)idx[j] * F + f), cf[j], a);
                s[f] += a;
            }
        }
        for (int f = 0; f < F; ++f) col[f * NTP] = s[f];
    }
}

struct WbShadeIn {
    const float* origins; const float* dirs;
    const float* rec_t; const int32_t* rec_ray;
    int64_t S;
};

// forward of one sample through both decoders; activations at act (already offset by tid).  Returns sigma, rgb.
__device__ __forceinline__ void wb_sample_forward(const WbGrid& g, const WbGridX& gx, const WbMlp& m, const float* __restrict__ W,
                                                  const WbShadeIn& in, int64_t s, float* act, int NTP,
                                                  float& sigma, float& r, float& gg, float& b)
{
    const int ray = __ldg(in.rec_ray + s);
    const float t = __ldg(in.rec_t + s);
    const float ox = __ldg(in.origins + 3 * (int64_t)ray), oy = __ldg(in.origins + 3 * (int64_t)ray + 1), oz = __ldg(in.origins + 3 * (int64_t)ray + 2);
    const float dx = __ldg(in.dirs + 3 * (int64_t)ray), dy = __ldg(in.dirs + 3 * (int64_t)ray + 1), dz = __ldg(in.dirs + 3 * (int64_t)ray + 2);
    const float px = wb_addcmul(ox, dx, t), py = wb_addcmul(oy, dy, t), pz = wb_addcmul(oz, dz, t);
    float* x0 = act + m.act_in[0] * NTP;
    if (gx.kind == 0) wb_gather(g, px, py, pz, x0, NTP);
    else wb_featx_gather(gx, px, py, pz, [&](int f, float v) { x0[f * NTP] = v; });     // triplanar / octree grid
    wb_embed(m.pos_mode, m.pos_freq, px, py, pz, x0 + m.feat_dim * NTP, NTP);
    for (int k = m.I[0]; k < m.Ipad[0]; ++k) x0[k * NTP] = 0.0f;
    for (int l = 0; l < m.nl_d; ++l)
        wb_layer_fwd(W + m.w_off[l], W + m.b_off[l], act + m.act_in[l] * NTP, act + m.act_out[l] * NTP, m.I[l], m.Opad[l], l < m.nl_d - 1, NTP);
    const float* df = act + m.act_out[m.nl_d - 1] * NTP;
    const int dout = m.O[m.nl_d - 1];
    const float df0 = df[0];
    float* y = act + m.act_in[m.nl_d] * NTP;
    for (int i = 1; i < dout; ++i) y[(i - 1) * NTP] = df[i * NTP];                          // fdir[..., 1:]  (nerf.py:259)
    wb_embed(m.view_mode, m.view_freq, dx, dy, dz, y + (dout - 1) * NTP, NTP);             // nerf.py:248-253
    const int lc0 = m.nl_d;
    for (int k = m.I[lc0]; k < m.Ipad[lc0]; ++k) y[k * NTP] = 0.0f;
    const int nl = m.nl_d + m.nl_c;
    for (int l = lc0; l < nl; ++l)
        wb_layer_fwd(W + m.w_off[l], W + m.b_off[l], act + m.act_in[l] * NTP, act + m.act_out[l] * NTP, m.I[l], m.Opad[l], l < nl - 1, NTP);
    const float* c = act + m.act_out[nl - 1] * NTP;
    r = 1.0f / (1.0f + expf(-c[0])); gg = 1.0f / (1.0f + expf(-c[NTP])); b = 1.0f / (1.0f + expf(-c[2 * NTP]));   // sigmoid (nerf.py:259)
    sigma = fmaxf(df0, 0.0f);                                                               // relu (nerf.py:263)
}

// ---------------------------------------------------------------------------------------------------------
// forward kernel
// ---------------------------------------------------------------------------------------------------------
template <int NT>
__global__ void __launch_bounds__(NT)
wb_shade_fwd_kernel(WbGrid g, WbGridX gx, WbMlp m, const float* __restrict__ blob, WbShadeIn in, float4* __restrict__ shaded)
{
    extern __shared__ __align__(16) float smem[];
    constexpr int NTP = NT + 1;
    __shared__ __align__(8) uint64_t bar;
    float* W = smem;                              // fwd_floats
    float* act = smem + m.fwd_floats + threadIdx.x;
    wb_bulk_stage(W, blob, (uint32_t)m.fwd_floats * 4u, &bar);
    const int64_t ntiles = (in.S + NT - 1) / NT;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t s = tile * NT + threadIdx.x;
        if (s < in.S) {
            float sigma, r, gg, b;
            wb_sample_forward(g, gx, m, W, in, s, act, NTP, sigma, r, gg, b);
            shaded[s] = make_float4(r, gg, b, sigma);
        }
    }
}

template <int NT>
static int wb_shade_fwd_launch(const WbGrid& g, const WbGridX& gx, const WbMlp& m, const float* blob, const WbShadeIn& in, float* shaded, cudaStream_t st)
{
    const size_t smem = (size_t)(m.fwd_floats + m.act_cols * (NT + 1)) * sizeof(float);
    if (smem > 227 * 1024) return 1;
    { static int64_t done_for = -1; if (done_for != WB_ATTR_KEY(smem)) { WB_CUDA(cudaFuncSetAttribute(wb_shade_fwd_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); done_for = WB_ATTR_KEY(smem); } }
    const int64_t ntiles = (in.S + NT - 1) / NT;
    int per_sm = (int)((227 * 1024) / (smem + 1024)); if (per_sm < 1) per_sm = 1; if (per_sm > 8) per_sm = 8;
    int64_t grid = (int64_t)wb_num_sms() * per_sm; if (grid > ntiles) grid = ntiles;
    wb_shade_fwd_kernel<NT><<<(unsigned)grid, NT, smem, st>>>(g, gx, m, blob, in, reinterpret_cast<float4*>(shaded));
    WB_LAUNCH_CHECK();
    return WB_OK;
}

extern "C" int wb_rf_shade_fwd(const wb_nef_desc* nef, const float* blob, int32_t precision, const wb_rays* rays,
                               const float* rec_t, const int32_t* rec_ray, int64_t S, float* shaded, void* feat_save, void* workspace, wb_stream s)
{
    WB_CHECK_ARG(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (fp16 tensor cores)");
    if (S == 0) return WB_OK;
    WB_CHECK_ARG(blob && rays && rays->origins && rays->dirs && rec_t && rec_ray && shaded, "null pointer");
    if (precision == 1) return wb_tc_shade_fwd(nef, blob, rays, rec_t, rec_ray, S, shaded, feat_save, workspace, (cudaStream_t)s);
    WbGrid g; int rc = wb_make_grid(nef, &g); if (rc) return rc;
    WbGridX gx; rc = wb_make_gridx(nef, false, &gx); if (rc) return rc;
    WbMlp m; rc = wb_make_mlp(nef, false, &m); if (rc) return rc;
    WbShadeIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S };
    rc = wb_shade_fwd_launch<128>(g, gx, m, blob, in, shaded, (cudaStream_t)s);
    if (rc == 1) rc = wb_shade_fwd_launch<64>(g, gx, m, blob, in, shaded, (cudaStream_t)s);
    if (rc == 1) rc = wb_shade_fwd_launch<32>(g, gx, m, blob, in, shaded, (cudaStream_t)s);
    if (rc == 1) { wb_set_error("wb_rf_shade_fwd: decoder too large for shared memory"); return WB_ERR_INVALID; }
    return rc;
}

// ---------------------------------------------------------------------------------------------------------
// backward kernel
// ---------------------------------------------------------------------------------------------------------
// dW[o][k] += sum_s gout[o][s]*in[k][s].  Warp w owns o-blocks {4*(w + nwarps*it)}; lane owns k = lane + 32*j:
// gout reads are warp broadcasts, activation reads are conflict free (bank = (k + s) mod 32).
template <int NT>
__device__ __forceinline__ void wb_wgrad(const float* __restrict__ gbuf /*[O][NTP]*/, const float* __restrict__ abuf /*[I][NTP]*/,
                                         int I, int O, float* __restrict__ gW /*global [O][I]*/, float* __restrict__ gB /*global [O] or null*/)
{
    constexpr int NTP = NT + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NWARP = NT / 32;
    const int KJ = (I + 31) >> 5;                     // <= 8 (I <= 256)
    for (int ob = 4 * warp; ob < O; ob += 4 * NWARP) {
        for (int j0 = 0; j0 < KJ; j0 += 4) {
            float acc[4][4];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][c] = 0.0f;
            int kk[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) { kk[c] = lane + 32 * (j0 + c); if (kk[c] >= I) kk[c] = -1; }
            for (int s = 0; s < NT; ++s) {
                float gv[4], av[4];
#pragma unroll
                for (int a = 0; a < 4; ++a) gv[a] = (ob + a < O) ? gbuf[(ob + a) * NTP + s] : 0.0f;
#pragma unroll
                for (int c = 0; c < 4; ++c) av[c] = kk[c] >= 0 ? abuf[kk[c] * NTP + s] : 0.0f;
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(gv[a], av[c], acc[a][c]);
            }
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (ob + a < O && kk[c] >= 0 && acc[a][c] != 0.0f) atomicAdd(gW + (ob + a) * I + kk[c], acc[a][c]);
        }
        if (gB) {      // bias grad: lanes split the samples
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                if (ob + a >= O) continue;
                float sacc = 0.0f;
                for (int s = lane; s < NT; s += 32) sacc += gbuf[(ob + a) * NTP + s];
                sacc = wb_warp_sum(sacc);
                if (lane == 0 && sacc != 0.0f) atomicAdd(gB + ob + a, sacc);
            }
        }
    }
}

// gin[k] = sum_o gout[o]*W[o][k]; Wo: [O][Ipad] o-major (global, L1-resident broadcast loads)
__device__ __forceinline__ void wb_dgrad(const float* __restrict__ Wo, const float* gout, float* gin, int Ipad, int O, int NTP)
{
    for (int kb = 0; kb < Ipad; kb += 8) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
        for (int o = 0; o < O; ++o) {
            const float gv = gout[o * NTP];
            const float4 w0 = __ldg(reinterpret_cast<const float4*>(Wo + o * Ipad + kb)), w1 = __ldg(reinterpret_cast<const float4*>(Wo + o * Ipad + kb + 4));
            acc[0] = fmaf(gv, w0.x, acc[0]); acc[1] = fmaf(gv, w0.y, acc[1]); acc[2] = fmaf(gv, w0.z, acc[2]); acc[3] = fmaf(gv, w0.w, acc[3]);
            acc[4] = fmaf(gv, w1.x, acc[4]); acc[5] = fmaf(gv, w1.y, acc[5]); acc[6] = fmaf(gv, w1.z, acc[6]); acc[7] = fmaf(gv, w1.w, acc[7]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) gin[(kb + j) * NTP] = acc[j];
    }
}

struct WbShadeGrads { float* gtable; float* gdens; float* gcol; };

template <int NT>
__global__ void __launch_bounds__(NT)
wb_shade_bwd_kernel(WbGrid g, WbGridX gx, WbMlp m, const float* __restrict__ blob, WbShadeIn in, const float4* __restrict__ g_shaded, WbShadeGrads G)
{
    extern __shared__ __align__(16) float smem[];
    constexpr int NTP = NT + 1;
    float* actbase = smem;                                   // act_cols * NTP
    float* gA = smem + m.act_cols * NTP;                     // maxw * NTP
    float* gB = gA + m.maxw * NTP;                           // maxw * NTP
    float* act = actbase + threadIdx.x;
    const float* W = blob;                                   // weights read through L1 (broadcast) in the backward
    const int nl = m.nl_d + m.nl_c;
    const int64_t ntiles = (in.S + NT - 1) / NT;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        int64_t s = tile * NT + threadIdx.x;
        const bool valid = s < in.S;
        if (!valid) s = in.S - 1;                            // keep shared columns finite; its gradient is zeroed below
        float sigma, r, gg, b;
        wb_sample_forward(g, gx, m, W, in, s, act, NTP, sigma, r, gg, b);
        float4 go = valid ? __ldg(g_shaded + s) : make_float4(0, 0, 0, 0);
        // ---- colour decoder ----
        float* gout = gA + threadIdx.x; float* gin = gB + threadIdx.x;
        {
            const int l = nl - 1;
            gout[0] = go.x * r * (1.0f - r); gout[NTP] = go.y * gg * (1.0f - gg); gout[2 * NTP] = go.z * b * (1.0f - b);
            for (int o = 3; o < m.Opad[l]; ++o) gout[o * NTP] = 0.0f;
        }
        for (int l = nl - 1; l >= m.nl_d; --l) {
            __syncthreads();
            wb_wgrad<NT>(gout - threadIdx.x, actbase + m.act_in[l] * NTP, m.I[l], m.O[l],
                         G.gcol + m.src_w[l], m.src_b[l] >= 0 ? G.gcol + m.src_b[l] : nullptr);
            wb_dgrad(blob + m.wo_off[l], gout, gin, m.Ipad[l], m.O[l], NTP);
            if (l > m.nl_d) {                                 // relu' of the layer input
                const float* a = act + m.act_in[l] * NTP;
                for (int k = 0; k < m.I[l]; ++k) if (!(a[k * NTP] > 0.0f)) gin[k * NTP] = 0.0f;
            }
            __syncthreads();                                  // all warps done reading gout before it becomes next gin
            float* t = gout; gout = gin; gin = t;
        }
        // gout now holds dL/d(colour input): first dout-1 entries -> density feats 1..
        {
            const int l = m.nl_d - 1; const int dout = m.O[l];
            const float* df = act + m.act_out[l] * NTP;
            gin[0] = (df[0] > 0.0f) ? go.w : 0.0f;            // relu' of density
            for (int i = 1; i < dout; ++i) gin[i * NTP] = gout[(i - 1) * NTP];
            for (int i = dout; i < m.Opad[l]; ++i) gin[i * NTP] = 0.0f;
            float* t = gout; gout = gin; gin = t;
        }
        // ---- density decoder ----
        for (int l = m.nl_d - 1; l >= 0; --l) {
            __syncthreads();
            wb_wgrad<NT>(gout - threadIdx.x, actbase + m.act_in[l] * NTP, m.I[l], m.O[l],
                         G.gdens + m.src_w[l], m.src_b[l] >= 0 ? G.gdens + m.src_b[l] : nullptr);
            wb_dgrad(blob + m.wo_off[l], gout, gin, m.Ipad[l], m.O[l], NTP);
            if (l > 0) {
                const float* a = act + m.act_in[l] * NTP;
                for (int k = 0; k < m.I[l]; ++k) if (!(a[k * NTP] > 0.0f)) gin[k * NTP] = 0.0f;
            }
            __syncthreads();
            float* t = gout; gout = gin; gin = t;
        }
        // ---- scatter dL/dfeat into the table (hashgrid_interpolate_cuda.cu:151-160) ----
        if (valid) {
            const float3 p = wb_sample_pos(in.origins, in.dirs, in.rec_ray, in.rec_t, s);
            const int L = g.L, F = g.F;
            const int lmax = gx.kind != 0 ? 0 : g.multiscale == 0 ? min(L, g.lod_idx) : L;
            if (gx.kind != 0) wb_featx_scatter(gx, p.x, p.y, p.z, [&](int f) { return gout[f * NTP]; });     // triplanar / octree grid
            for (int l = 0; l < lmax; ++l) {
                uint32_t idx[8]; float cf[8];
                wb_corner_setup(g, l, p.x, p.y, p.z, idx, cf);
                float* tb = G.gtable + g.begin[l] * F;
                if (F == 2) {
                    const float g0 = g.multiscale == 0 ? gout[(l * 2) * NTP] : gout[0];
                    const float g1 = g.multiscale == 0 ? gout[(l * 2 + 1) * NTP] : gout[NTP];
                    if (g0 == 0.0f && g1 == 0.0f) continue;
#pragma unroll
                    for (int j = 0; j < 8; ++j) atomicAdd(reinterpret_cast<float2*>(tb) + idx[j], make_float2(g0 * cf[j], g1 * cf[j]));
                } else {
                    for (int f = 0; f < F; ++f) {
                        const float gv = g.multiscale == 0 ? gout[(l * F + f) * NTP] : gout[f * NTP];
                        if (gv == 0.0f) continue;
#pragma unroll
                        for (int j = 0; j < 8; ++j) atomicAdd(tb + (int64_t)idx[j] * F + f, gv * cf[j]);
                    }
                }
            }
        }
        __syncthreads();
    }
}

template <int NT>
static int wb_shade_bwd_launch(const WbGrid& g, const WbGridX& gx, const WbMlp& m, const float* blob, const WbShadeIn& in, const float* g_shaded,
                               const WbShadeGrads& G, cudaStream_t st)
{
    const size_t smem = (size_t)(m.act_cols + 2 * m.maxw) * (NT + 1) * sizeof(float);
    if (smem > 227 * 1024) return 1;
    { static int64_t done_for = -1; if (done_for != WB_ATTR_KEY(smem)) { WB_CUDA(cudaFuncSetAttribute(wb_shade_bwd_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); done_for = WB_ATTR_KEY(smem); } }
    const int64_t ntiles = (in.S + NT - 1) / NT;
    int per_sm = (int)((227 * 1024) / (smem + 1024)); if (per_sm < 1) per_sm = 1; if (per_sm > 8) per_sm = 8;
    int64_t grid = (int64_t)wb_num_sms() * per_sm; if (grid > ntiles) grid = ntiles;
    wb_shade_bwd_kernel<NT><<<(unsigned)grid, NT, smem, st>>>(g, gx, m, blob, in, reinterpret_cast<const float4*>(g_shaded), G);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

extern "C" int wb_rf_shade_bwd(const wb_nef_desc* nef, const float* blob, int32_t precision, const wb_rays* rays,
                               const float* rec_t, const int32_t* rec_ray, int64_t S, const float* g_shaded,
                               const float* loss_scale, const void* feat_saved, void* workspace,
                               float* grad_table, float* grad_dens, float* grad_col, wb_stream s)
{
    const bool ray_rows_ready = wb_take_ray_rows_ready();
    WB_CHECK_ARG(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (fp16 tensor cores)");
    if (S == 0) return WB_OK;
    WB_CHECK_ARG(blob && rays && rays->origins && rays->dirs && rec_t && rec_ray && g_shaded, "null pointer");
    WB_CHECK_ARG((grad_table || nef->grid_kind != 0) && grad_dens && grad_col, "null gradient buffer");
    if (precision == 1)
        return wb_tc_shade_bwd(nef, blob, rays, rec_t, rec_ray, S, g_shaded, loss_scale, feat_saved, workspace, ray_rows_ready, grad_table,
                               grad_dens, grad_col, (cudaStream_t)s);
    WbGrid g; int rc = wb_make_grid(nef, &g); if (rc) return rc;
    WbGridX gx; rc = wb_make_gridx(nef, true, &gx); if (rc) return rc;
    WbMlp m; rc = wb_make_mlp(nef, true, &m); if (rc) return rc;
    WbShadeIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S };
    WbShadeGrads G = { grad_table, grad_dens, grad_col };
    rc = wb_shade_bwd_launch<128>(g, gx, m, blob, in, g_shaded, G, (cudaStream_t)s);
    if (rc == 1) rc = wb_shade_bwd_launch<64>(g, gx, m, blob, in, g_shaded, G, (cudaStream_t)s);
    if (rc == 1) rc = wb_shade_bwd_launch<32>(g, gx, m, blob, in, g_shaded, G, (cudaStream_t)s);
    if (rc == 1) { wb_set_error("wb_rf_shade_bwd: decoder too large for shared memory"); return WB_ERR_INVALID; }
    return rc;
}
