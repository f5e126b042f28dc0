// wb_shade_tc.cu -- fused "shade" stage with tensor-core decoders (precision 1): wgmma + TMA-staged weights (sm_90a).
//
// Numerics = the reference under torch.cuda.amp.autocast (nerf_hash.yaml:76 enable_amp: True): decoder operands in
// fp16, fp32 accumulation; unlike the reference the hash table is read as fp32 master (no per-call .half() copy,
// ops/grid.py:88-89), features are blended in fp32 and table gradients accumulate in fp32.
//
// Unit of work = a 64-sample sub-tile handled by a GROUP of 128 threads = one warpgroup: row r of the tile is shared by two
// threads (column halves) for the per-sample work, and the warpgroup issues the layer's wgmma chain (A = sample tile, B = the
// TMA-staged weight pack, D[64 x N] in registers, initialised with the fp16 bias).  Per layer: every thread writes its part of
// the fp16 operand tile (slab layout, wb_tc.cuh) -> proxy fence -> group barrier -> wgmma chain -> wait -> group barrier ->
// epilogue straight from the accumulator fragments (relu -> next tile, relu' mask -> next dY, dL/dfeat -> planes) or, where a
// row needs its whole output (density / colour heads), through a small fp32 scratch tile.  Groups are independent (own named
// barrier, own tiles): the forward runs TC_FWD_GROUPS groups per CTA and several CTAs per SM, the backward one CTA per SM.
//
// Forward  (wb_shade_fwd_tc_kernel): gather 15 LODs x 8 corners (fp32 blend) -> decoders -> (r,g,b,sigma).  It also saves
//   the gathered feature rows (fp16, chunk-major [Kp0/8][S] x 16 B: coalesced both ways) for the backward.
// Backward (wb_mlp_bwd_tc_kernel): reloads those rows -- it touches neither the hash table nor the octree -- recomputes the
//   decoders (all activation tiles stay in shared memory) and per layer issues
//     weight grad   acc_l^T[out, in | 1] += dY_l^T . [X_l | 1]  (both operands MN-major straight from the sample tiles; a
//                                                               constant-one slab behind every X_l tile gives the bias gradient;
//                                                               fp32 accumulators in shared memory, one private copy per group)
//     data grad     dX_l = dY_l . W_l                           (weight pack read MN-major: no transposed copy)
//   and writes dL/dfeat as fp16 level-major planes [L][S][F], or scatters it into the hash table in its last epilogue.
// Scatter  (wb_table_scatter_kernel, SIMT): lanes = consecutive samples; a thread builds its sample position once and walks all
//   LODs; per LOD, runs of lanes that fall into the same cell are summed with a segmented warp scan and only the last lane of a
//   run issues the reductions (x-neighbour entries that differ only in bit 0 as one 16-byte red.global.add.v4.f32).
//   Neighbouring samples of a ray share cells on all but the finest LODs.
// The per-ray view embedding (positional_embedder.py:51-66) is evaluated once per ray (wb_ray_embed_kernel), not per sample.
// Gradients are carried in fp16 under a power-of-two loss scale supplied on the device (no host sync) and unscaled in fp32
// at the two exits (table scatter, weight-gradient flush).
#include "wb_common.cuh"
#include "wb_featx.cuh"
#include "wb_tc.cuh"
#include <math.h>

#define TC_ML 16
constexpr int TC_ROWS = 64;                 // samples per sub-tile (wgmma M)
constexpr int TC_GROUP = 128;               // threads per sub-tile group: one warpgroup, 64 rows x 2 column halves
constexpr int TC_SLAB = TC_ROWS * 16;       // bytes of one slab (8 features of every sample of the tile)
constexpr int TC_FWD_GROUPS = 2;            // sub-tile groups per forward CTA (they share the staged weights)
constexpr int TC_SCR_LD = 33;               // fp32 scratch tile [64][33]: the <= 32 columns an epilogue needs row by row
constexpr int TC_SCR_BYTES = (TC_ROWS * TC_SCR_LD * 4 + 15) / 16 * 16;
constexpr int TC_SMEM_MAX = 227 * 1024 - 1024;      // dynamic shared memory per CTA (H100: 227 KB, minus the static barriers)

struct WbTc {
    int nl_d, nl_c;
    int I[TC_ML], O[TC_ML], Kp[TC_ML], Np[TC_ML];
    int w_off[TC_ML], b_off[TC_ML];            // byte offsets in the parameter blob: weight pack, bias pack [Np x 16] (bias at k = 0)
    int has_bias;
    int src_w[TC_ML], src_b[TC_ML];
    int blob_bytes;
    int maxw;
    int tile_off[TC_ML];                       // byte offset of layer l's INPUT tile inside a group region
    int dy_off, scr_off, acc_off;              // byte offsets inside a group region: dY tile, fp32 scratch, weight-grad accumulators
    int acc_l[TC_ML];                          // float offset of layer l's accumulator [O][I + 1] (column I = bias), -1: not in this pass
    int group_bytes;                           // stride of the group regions
    int groups;                                // sub-tile groups per CTA
    int w_smem_off;                            // byte offset of the staged parameter blob (behind the group regions)
    int smem_bytes;
    int feat_dim, pos_dim, view_dim, pos_mode, pos_freq, view_mode, view_freq;
};

static int tc_round_up(int v, int m) { return (v + m - 1) / m * m; }
static int tc_embed_dim(int mode, int freq) { return mode == 0 ? 0 : mode == 1 ? 3 : mode == 2 ? 6 * freq : 3 + 6 * freq; }

// backward shared-memory plan for `groups` groups that accumulate the weight gradients of the layers in `wmask`;
// returns false when it does not fit
static bool tc_bwd_layout(WbTc* m, unsigned wmask, int groups)
{
    const int nl = m->nl_d + m->nl_c;
    int off = 0;
    for (int l = 0; l < nl; ++l) { m->tile_off[l] = off; off += (m->Kp[l] / 8 + 1) * TC_SLAB; }     // + constant-one slab
    // the weight-grad A operand (dY^T, M = 64 output features) reads 8 slabs even when the layer is narrower
    m->dy_off = off; off += (max(m->maxw, 64) / 8) * TC_SLAB;
    m->scr_off = off; off += TC_SCR_BYTES;
    m->acc_off = off;
    int acc = 0;
    for (int l = 0; l < nl; ++l) {
        m->acc_l[l] = -1;
        if ((wmask >> l) & 1u) { m->acc_l[l] = acc; acc += m->O[l] * (m->I[l] + 1); }
    }
    off += tc_round_up(acc * 4, 16);
    m->group_bytes = off;
    m->groups = groups;
    m->w_smem_off = groups * off;
    m->smem_bytes = m->w_smem_off + m->blob_bytes;
    return m->smem_bytes <= TC_SMEM_MAX;
}

// returns WB_OK, or WB_ERR_INVALID with a message when the configuration does not fit the tensor-core path
int wb_tc_make(const wb_nef_desc* d, bool backward, WbTc* m)
{
    WB_CHECK_ARG(d->dens_layers >= 1 && d->col_layers >= 1 && d->dens_layers + d->col_layers <= TC_ML, "unsupported decoder depth");
    WB_CHECK_ARG(d->dens_params && d->col_params, "null decoder parameters");
    memset(m, 0, sizeof(*m));
    m->nl_d = d->dens_layers; m->nl_c = d->col_layers;
    m->feat_dim = d->multiscale == 0 ? d->num_lods * d->feature_dim : d->feature_dim;
    m->pos_mode = d->pos_mode; m->pos_freq = d->pos_freq; m->view_mode = d->view_mode; m->view_freq = d->view_freq;
    m->pos_dim = tc_embed_dim(d->pos_mode, d->pos_freq); m->view_dim = tc_embed_dim(d->view_mode, d->view_freq);
    WB_CHECK_ARG(d->dens_dims[0] == m->feat_dim + m->pos_dim, "decoder_density input width != grid features + position embedding");
    const int dout = d->dens_dims[d->dens_layers];
    WB_CHECK_ARG(dout >= 2 && dout <= 16, "tensor-core path: decoder_density output must be 2..16 wide");
    WB_CHECK_ARG(d->col_dims[0] == dout - 1 + m->view_dim, "decoder_color input width != density feats - 1 + view embedding");
    WB_CHECK_ARG(d->col_dims[d->col_layers] == 3, "decoder_color output must be 3 wide");
    const int nl = m->nl_d + m->nl_c;
    int off = 0, srcd = 0, srcc = 0, maxw = 0;
    for (int l = 0; l < nl; ++l) {
        const bool dens = l < m->nl_d;
        const int I = dens ? d->dens_dims[l] : d->col_dims[l - m->nl_d];
        const int O = dens ? d->dens_dims[l + 1] : d->col_dims[l - m->nl_d + 1];
        WB_CHECK_ARG(I >= 1 && I <= 128 && O >= 1 && O <= 128, "tensor-core path: layer widths must be <= 128");
        m->I[l] = I; m->O[l] = O; m->Kp[l] = tc_round_up(I, 16); m->Np[l] = tc_round_up(O, 16);
        m->w_off[l] = off; off += m->Kp[l] * m->Np[l] * 2;
        m->b_off[l] = off; off += m->Np[l] * 32;
        int& src = dens ? srcd : srcc;
        m->src_w[l] = src; src += I * O;
        if (d->has_bias) { m->src_b[l] = src; src += O; } else m->src_b[l] = -1;
        maxw = max(maxw, max(m->Kp[l], m->Np[l]));
    }
    m->blob_bytes = tc_round_up(off, 16);
    m->has_bias = d->has_bias ? 1 : 0;
    m->maxw = maxw;
    if (!backward) {
        // every layer's input tile is overwritten in place by its output (the layer's MMAs have completed before the epilogue writes)
        for (int l = 0; l < nl; ++l) m->tile_off[l] = 0;
        m->scr_off = (maxw / 8) * TC_SLAB;
        m->group_bytes = m->scr_off + TC_SCR_BYTES;
        m->groups = TC_FWD_GROUPS;
        m->w_smem_off = m->groups * m->group_bytes;
        m->smem_bytes = m->w_smem_off + m->blob_bytes;
        WB_CHECK_ARG(m->smem_bytes <= TC_SMEM_MAX, "tensor-core path: decoder does not fit in shared memory (use precision 0)");
        return WB_OK;
    }
    // backward: decoders whose whole backward fits two groups per CTA in one pass, and decoders of the app/nerf depth (one hidden
    // density layer, two hidden colour layers) up to width 128, whose weight gradients may take several passes (every layer's
    // accumulator must fit beside the tiles of one group); deeper, wider decoders train on the fp32 kernels
    const bool one_pass = tc_bwd_layout(m, (1u << nl) - 1u, 2);
    bool passes = m->nl_d <= 2 && m->nl_c <= 3;
    for (int l = 0; l < nl && passes; ++l) passes = tc_bwd_layout(m, 1u << l, 1);
    WB_CHECK_ARG(one_pass || passes, "tensor-core path: decoder backward does not fit in shared memory (use precision 0)");
    tc_bwd_layout(m, (1u << nl) - 1u, 1);       // the plan of the first pass is left in *m
    return WB_OK;
}

// number of dL/dfeat planes and halfs per (plane, sample): 'cat' -> one plane per live LOD, 'sum' -> a single plane
static void tc_dfeat_shape(const wb_nef_desc* d, int* planes, int* width)
{
    *width = d->feature_dim;
    *planes = d->multiscale == 0 ? (d->lod_idx < d->num_lods ? d->lod_idx : d->num_lods) : 1;
    if (*planes < 0) *planes = 0;
}
static int64_t tc_align256(int64_t b) { return (b + 255) / 256 * 256; }

// workspace layout (bytes): [ray_embed: R * Kc * 2][dfeat: planes * S * F * 2 (backward only)]
int64_t wb_tc_workspace_bytes(const wb_nef_desc* nef, int64_t R, int64_t S, int backward)
{
    WbTc m; if (wb_tc_make(nef, false, &m)) return -1;
    int planes, width; tc_dfeat_shape(nef, &planes, &width);
    int64_t b = tc_align256(R * m.Kp[m.nl_d] * 2);
    if (backward) b += tc_align256((int64_t)planes * S * width * 2);
    return b + 256;
}
int wb_tc_supported(const wb_nef_desc* nef, int backward)
{
    WbTc m; if (wb_tc_make(nef, false, &m)) return 0;
    if (backward && wb_tc_make(nef, true, &m)) return 0;
    return 1;
}
// the features are only saved for a backward pass: refuse here (at forward time) if that pass cannot run
int64_t wb_tc_feat_bytes(const wb_nef_desc* nef, int64_t S)
{
    WbTc m; if (wb_tc_make(nef, true, &m) || wb_tc_make(nef, false, &m)) return -1;
    return (int64_t)m.Kp[0] * 2 * S + 256;
}

// ---- parameter blob: fp16 weight packs (wb_tc.cuh layout) + fp32 biases -------------------------------------------
__global__ void wb_tc_pack_kernel(WbTc m, const float* __restrict__ dens, const float* __restrict__ col, uint8_t* __restrict__ blob)
{
    const int nl = m.nl_d + m.nl_c;
    for (int l = 0; l < nl; ++l) {
        const float* src = l < m.nl_d ? dens : col;
        const int I = m.I[l], O = m.O[l], Kp = m.Kp[l], Np = m.Np[l];
        __half* w = reinterpret_cast<__half*>(blob + m.w_off[l]);
        for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Kp * Np; e += gridDim.x * blockDim.x) {
            const int kc = e / (Np * 8), n = (e / 8) % Np, k = kc * 8 + (e & 7);      // element (n,k) at (k/8)*(Np*8) + n*8 + k%8 halves
            w[e] = __float2half_rn((n < O && k < I) ? src[m.src_w[l] + n * I + k] : 0.0f);
        }
        // bias pack B[Np x 16] (K-major, same layout as the weights): column k = 0 holds the bias.  The accumulator
        // fragments start from it and the layer's MMAs accumulate on top (fp16 bias: what F.linear under autocast does)
        __half* b = reinterpret_cast<__half*>(blob + m.b_off[l]);
        for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Np * 16; e += gridDim.x * blockDim.x) {
            const int kc = e / (Np * 8), n = (e / 8) % Np, k = kc * 8 + (e & 7);
            b[e] = __float2half_rn((k == 0 && n < O && m.src_b[l] >= 0) ? src[m.src_b[l] + n] : 0.0f);
        }
    }
}

int wb_tc_blob_floats(const wb_nef_desc* nef) { WbTc m; if (wb_tc_make(nef, false, &m)) return -1; return m.blob_bytes / 4; }

int wb_tc_pack(const wb_nef_desc* nef, float* blob, cudaStream_t st)
{
    WbTc m; int rc = wb_tc_make(nef, false, &m); if (rc) return rc;
    wb_tc_pack_kernel<<<16, 256, 0, st>>>(m, nef->dens_params, nef->col_params, reinterpret_cast<uint8_t*>(blob));
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---- per-ray colour-input rows: zeros with the view embedding at features [dout-1, dout-1+view_dim) -----------------
__global__ void __launch_bounds__(128)
wb_ray_embed_kernel(WbTc m, const float* __restrict__ dirs, int64_t R, uint4* __restrict__ out)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const int Kc = m.Kp[m.nl_d], f0 = m.O[m.nl_d - 1] - 1;
    __align__(16) __half row[128];
    for (int i = 0; i < Kc; ++i) row[i] = __float2half_rn(0.0f);
    const float x = dirs[3 * r], y = dirs[3 * r + 1], z = dirs[3 * r + 2];
    int o = f0;
    if (m.view_mode == 1 || m.view_mode == 3) { row[o] = __float2half_rn(x); row[o + 1] = __float2half_rn(y); row[o + 2] = __float2half_rn(z); o += 3; }
    if (m.view_mode >= 2) {
        float band = 1.0f;
        for (int f = 0; f < m.view_freq; ++f) {
            const float w3[3] = { x * band, y * band, z * band };
            for (int c = 0; c < 3; ++c) {
                row[o + f * 3 + c] = __float2half_rn(sinf(w3[c]));
                row[o + 3 * m.view_freq + f * 3 + c] = __float2half_rn(cosf(w3[c]));
            }
            band *= 2.0f;
        }
    }
    const uint4* rv = reinterpret_cast<const uint4*>(row);
    for (int c = 0; c < Kc / 8; ++c) out[r * (Kc / 8) + c] = rv[c];
}

// ---------------------------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------------------------
struct TcIn {
    const float* origins; const float* dirs; const float* rec_t; const int32_t* rec_ray; int64_t S;
    const uint4* ray_embed;      // [R][Kc/8] rows prepared by wb_ray_embed_kernel
    uint4* x0_save;              // forward: optional [Kp0/8][S] copy of the density-decoder input rows
    const uint4* x0_saved;       // backward: the same buffer
    int64_t s_begin, s_end;      // backward kernels that take a sample range (a multiple of 64 .. s_end; s_end == 0: the whole [0, S)); S stays the plane stride
};

// byte offset of (sample s, feature f) in a slab tile
__device__ __forceinline__ uint32_t tc_slab_off(int s, int f) { return (uint32_t)((f >> 3) * TC_SLAB + s * 16 + (f & 7) * 2); }

__device__ __forceinline__ void tile_store1(uint8_t* tile, int r, int f, float v)
{
    *reinterpret_cast<__half*>(tile + tc_slab_off(r, f)) = __float2half_rn(v);
}
__device__ __forceinline__ void tile_store8(uint8_t* tile, int r, int slab, const float v[8])
{
    uint4 q; q.x = tc_pack2(v[0], v[1]); q.y = tc_pack2(v[2], v[3]); q.z = tc_pack2(v[4], v[5]); q.w = tc_pack2(v[6], v[7]);
    *reinterpret_cast<uint4*>(tile + slab * TC_SLAB + r * 16) = q;
}
// embedding (positional_embedder.py:51-66) written into tile features [f0, f0+dim)
__device__ __forceinline__ void tile_embed(uint8_t* tile, int r, int f0, int mode, int freq, float x, float y, float z)
{
    if (mode == 0) return;
    int o = f0;
    if (mode == 1 || mode == 3) { tile_store1(tile, r, o, x); tile_store1(tile, r, o + 1, y); tile_store1(tile, r, o + 2, z); o += 3; }
    if (mode == 1) return;
    float band = 1.0f;
    for (int f = 0; f < freq; ++f) {
        const float wx = x * band, wy = y * band, wz = z * band;
        tile_store1(tile, r, o + f * 3 + 0, sinf(wx)); tile_store1(tile, r, o + f * 3 + 1, sinf(wy)); tile_store1(tile, r, o + f * 3 + 2, sinf(wz));
        tile_store1(tile, r, o + 3 * freq + f * 3 + 0, cosf(wx)); tile_store1(tile, r, o + 3 * freq + f * 3 + 1, cosf(wy)); tile_store1(tile, r, o + 3 * freq + f * 3 + 2, cosf(wz));
        band *= 2.0f;
    }
}
// hash-grid gather of one sample -> features [0, feat_dim) of the X0 tile (fp32 blend, fp16 store)
// `half` (0/1): the two threads of a row split the work -- slab (4 LODs) k goes to half k & 1 on the F == 2 'cat' path, the
// generic paths are done by half 0 alone
__device__ __forceinline__ void tile_gather(const WbGrid& g, uint8_t* tile, int r, int half, float px, float py, float pz)
{
    const int L = g.L, F = g.F;
    if (g.multiscale == 0 && F == 2) {
        for (int l0 = 4 * half; l0 < L; l0 += 8) {              // 4 levels = 8 features = one slab row (16 B store)
            float v[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int l = l0 + q;
                if (l >= L || l >= g.lod_idx) { v[2 * q] = 0.0f; v[2 * q + 1] = 0.0f; continue; }       // hash_grid.py:226-229
                uint32_t idx[8]; float cf[8];
                wb_corner_setup(g, l, px, py, pz, idx, cf);
                const float2* tb = reinterpret_cast<const float2*>(g.table + g.begin[l] * 2);
                float2 c[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) c[j] = __ldg(tb + idx[j]);
                float a0 = c[0].x * cf[0], a1 = c[0].y * cf[0];
#pragma unroll
                for (int j = 1; j < 8; ++j) { a0 = fmaf(c[j].x, cf[j], a0); a1 = fmaf(c[j].y, cf[j], a1); }
                v[2 * q] = a0; v[2 * q + 1] = a1;
            }
            tile_store8(tile, r, l0 >> 2, v);
        }
    } else if (half != 0) {
        return;
    } else if (g.multiscale == 0) {
        for (int l = 0; l < L; ++l) {
            if (l >= g.lod_idx) { for (int f = 0; f < F; ++f) tile_store1(tile, r, l * F + f, 0.0f); continue; }
            uint32_t idx[8]; float cf[8];
            wb_corner_setup(g, l, px, py, pz, idx, cf);
            const float* tb = g.table + g.begin[l] * F;
            for (int f = 0; f < F; ++f) {
                float a = __ldg(tb + (int64_t)idx[0] * F + f) * cf[0];
#pragma unroll
                for (int j = 1; j < 8; ++j) a = fmaf(__ldg(tb + (int64_t)idx[j] * F + f), cf[j], a);
                tile_store1(tile, r, l * F + f, a);
            }
        }
    } else {
        float s[8];
#pragma unroll
        for (int f = 0; f < 8; ++f) s[f] = 0.0f;
        for (int l = 0; l < L; ++l) {
            uint32_t idx[8]; float cf[8];
            wb_corner_setup(g, l, px, py, pz, idx, cf);
            const float* tb = g.table + g.begin[l] * F;
#pragma unroll
            for (int f = 0; f < 8; ++f) if (f < F) {
                float a = __ldg(tb + (int64_t)idx[0] * F + f) * cf[0];
#pragma unroll
                for (int j = 1; j < 8; ++j) a = fmaf(__ldg(tb + (int64_t)idx[j] * F + f), cf[j], a);
                s[f] += a;
            }
        }
#pragma unroll
        for (int f = 0; f < 8; ++f) if (f < F) tile_store1(tile, r, f, s[f]);
    }
}
// zero features [f0, f1) of this thread's row
__device__ __forceinline__ void tile_zero(uint8_t* tile, int r, int f0, int f1) { for (int f = f0; f < f1; ++f) tile_store1(tile, r, f, 0.0f); }

// ---------------------------------------------------------------------------------------------------------------
// wgmma chains of one group
// ---------------------------------------------------------------------------------------------------------------
struct TcCtx {
    uint8_t* sub;               // this group's region (tiles, scratch, accumulators)
    const uint8_t* blob;        // staged parameter blob (shared by the CTA's groups)
    float* scr;                 // fp32 scratch tile [TC_ROWS][TC_SCR_LD]
    int g;                      // sub-tile group of this thread inside the CTA; named barrier g + 1
    int r, h;                   // row of the sub-tile, column half
    int wl;                     // thread index inside the warpgroup (accumulator fragment owner)
};
__device__ __forceinline__ void tc_ctx_init(TcCtx& c, const WbTc& m, uint8_t* smem)
{
    const int tig = threadIdx.x & (TC_GROUP - 1);
    c.g = threadIdx.x / TC_GROUP;
    c.sub = smem + c.g * m.group_bytes; c.blob = smem + m.w_smem_off;
    c.scr = reinterpret_cast<float*>(c.sub + m.scr_off);
    c.r = tig & (TC_ROWS - 1); c.h = tig / TC_ROWS; c.wl = tig;
}
__device__ __forceinline__ void tc_sync(const TcCtx& c) { tc_group_sync(c.g + 1, TC_GROUP); }
// operand tiles written by the group's threads -> visible to the tensor cores of the whole group
__device__ __forceinline__ void tc_publish(const TcCtx& c) { tc_fence_smem_async(); tc_sync(c); }

// One MMA chain of the group: D[64 x N] = bias (fp16, bias pack: entry n at half index 8n) or 0, then += A . B over nk K-steps of
// 16; wait; group barrier (every MMA of the group has read its operands: the epilogue may overwrite them); epi(d) on the fragments.
template <int N, int TA, int TB, class Epi>
__device__ __forceinline__ void tc_chain(const TcCtx& c, uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv,
                                         const __half* bias, Epi&& epi)
{
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = bias ? __half2float(bias[tc_frag_col(c.wl, i) * 8]) : 0.0f;
    tc_wg_fence();
    for (int kb = 0; kb < nk; ++kb) { WgMma<N, TA, TB>::run(d, da, db, 1u); da += aadv; db += badv; }
    tc_wg_commit();
    tc_wg_wait0();
    tc_wg_hold(d);
    tc_sync(c);
    epi(d);
}
// the same with N chosen at run time (a multiple of 16, at most NMAX <= 128: the widest padded layer the kernel was built for; a
// 128-wide accumulator alone needs 64 registers per thread)
template <int TA, int TB, int NMAX = 128, class Epi>
__device__ __forceinline__ void tc_chain_n(const TcCtx& c, int N, uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv,
                                           const __half* bias, Epi&& epi)
{
    switch (N) {
        case 16: tc_chain<16, TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        case 32: tc_chain<32, TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        case 48: tc_chain<48, TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        case 64: tc_chain<64, TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        case 80: tc_chain<(80 <= NMAX ? 80 : NMAX), TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        case 96: tc_chain<(96 <= NMAX ? 96 : NMAX), TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        case 112: tc_chain<(112 <= NMAX ? 112 : NMAX), TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
        default: tc_chain<NMAX, TA, TB>(c, da, db, nk, aadv, badv, bias, epi); break;
    }
}
// fragments -> fp32 scratch tile, columns [0, ncols); the caller synchronises the group before reading rows
#define TC_FRAG_TO_SCRATCH(c, d, ncols)                                                                          \
    do {                                                                                                         \
        constexpr int NR_ = sizeof(d) / sizeof(float);                                                          \
        _Pragma("unroll") for (int i = 0; i < NR_; ++i) {                                                        \
            const int col = tc_frag_col((c).wl, i);                                                              \
            if (col < (ncols)) (c).scr[tc_frag_row((c).wl, i) * TC_SCR_LD + col] = d[i];                          \
        }                                                                                                        \
    } while (0)

// forward layer l: D = bias + X_l . W_l^T   (A: input tile K-major, B: weight pack K-major)
template <int NMAX, class Epi>
__device__ __forceinline__ void tc_fwd_layer(const WbTc& m, const TcCtx& c, int l, int N, Epi&& epi)
{
    const uint32_t sb = tc_smem_u32(c.sub + m.tile_off[l]), wb = tc_smem_u32(c.blob);
    const int Np = m.Np[l];
    tc_chain_n<0, 0, NMAX>(c, N, tc_desc(sb, TC_SLAB, 128), tc_desc(wb + m.w_off[l], Np * 16, 128), m.Kp[l] / 16, (2 * TC_SLAB) >> 4,
                     (2 * Np * 16) >> 4, m.has_bias ? reinterpret_cast<const __half*>(c.blob + m.b_off[l]) : nullptr, epi);
}

// Decoders of one 64-sample sub-tile, starting from an X0 tile that the group has already written.
// Returns (per row, both column halves) the density-decoder output df[16] and the colour pre-activations c3[3].
template <int NMAX>
__device__ __forceinline__ void tc_decoders(const WbTc& m, const TcCtx& c, const TcIn& in, int64_t ray, float df[16], float c3[3])
{
    const int nl = m.nl_d + m.nl_c;
    for (int l = 0; l < nl; ++l) {
        const bool last_d = (l == m.nl_d - 1), last_c = (l == nl - 1);
        tc_publish(c);
        if (!last_d && !last_c) {
            // hidden layer: relu(acc) -> next input tile (F2FP.RELU), straight from the fragments; Np[l] == Kp[l+1], padded outputs
            // are relu(0 + 0) = 0
            uint8_t* tn = c.sub + m.tile_off[l + 1];
            tc_fwd_layer<NMAX>(m, c, l, m.Np[l], [&](auto& d) {
                constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                for (int i = 0; i < NR; i += 2) {
                    const int row = tc_frag_row(c.wl, i), col = tc_frag_col(c.wl, i);
                    *reinterpret_cast<uint32_t*>(tn + (col >> 3) * TC_SLAB + row * 16 + (col & 7) * 2) = tc_pack2_relu(d[i], d[i + 1]);
                }
            });
            continue;
        }
        tc_fwd_layer<NMAX>(m, c, l, 16, [&](auto& d) { TC_FRAG_TO_SCRATCH(c, d, 16); });      // both heads are <= 16 wide
        tc_sync(c);
        const float* srow = c.scr + c.r * TC_SCR_LD;
        if (last_d) {
#pragma unroll
            for (int j = 0; j < 16; ++j) df[j] = srow[j];
            // colour input = [df[1:], embed(ray_d)], zero padded (nerf.py:248-259): the per-ray row already holds the
            // embedding and the zero padding, only the first dout-1 (<= 15) features are per-sample.  16-byte chunk ch of the
            // row is written by column half ch & 1.
            uint8_t* tcol = c.sub + m.tile_off[l + 1];
            const int nd = m.O[l] - 1, nch = m.Kp[l + 1] / 8;
            const uint4* re = in.ray_embed + ray * nch;
            uint4 q = __ldg(re + c.h);
            __half* hq = reinterpret_cast<__half*>(&q);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                // feature 8*h + j <- df[8*h + j + 1]; select without dynamic register indexing
                const float dv = c.h == 0 ? df[(j + 1) & 15] : df[(j + 9) & 15];
                if (8 * c.h + j < nd) hq[j] = __float2half_rn(dv);
            }
            *reinterpret_cast<uint4*>(tcol + c.h * TC_SLAB + c.r * 16) = q;
            for (int ch = 2 + c.h; ch < nch; ch += 2) *reinterpret_cast<uint4*>(tcol + ch * TC_SLAB + c.r * 16) = __ldg(re + ch);
        } else {
            c3[0] = srow[0]; c3[1] = srow[1]; c3[2] = srow[2];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// forward kernel: CTA = TC_FWD_GROUPS groups, each walking its own 64-sample sub-tiles; several CTAs per SM overlap gather,
// MMA chains and epilogues
// ---------------------------------------------------------------------------------------------------------------
template <int MINB, bool GX, int NMAX>   // MINB: resident CTAs per SM the register allocation is bounded for; GX: triplanar / octree
                                         // feature grid (wb_featx.cuh) instead of the hash grid; NMAX: widest padded layer (64 or 128)
__global__ void __launch_bounds__(TC_FWD_GROUPS * TC_GROUP, MINB)
wb_shade_fwd_tc_kernel(WbGrid g, WbGridX gx, WbTc m, const uint8_t* __restrict__ blob, TcIn in, float4* __restrict__ shaded)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;
    if (threadIdx.x == 0) {
        tc_mbar_init(&bar, 1); tc_mbar_init_fence();
        tc_mbar_expect_tx(&bar, (uint32_t)m.blob_bytes);
        tc_bulk_g2s(smem + m.w_smem_off, blob, (uint32_t)m.blob_bytes, &bar);      // TMA: parameters -> shared memory
    }
    __syncthreads();
    tc_mbar_wait(&bar, 0);
    TcCtx c; tc_ctx_init(c, m, smem);
    uint8_t* t0 = c.sub + m.tile_off[0];
    const int nch0 = m.Kp[0] / 8;
    const int64_t ntiles = (in.S + TC_ROWS - 1) / TC_ROWS;
    for (int64_t tile = (int64_t)blockIdx.x * TC_FWD_GROUPS + c.g; tile < ntiles; tile += (int64_t)gridDim.x * TC_FWD_GROUPS) {
        int64_t s = tile * TC_ROWS + c.r;
        const bool valid = s < in.S;
        if (!valid) s = in.S - 1;
        const int64_t ray = __ldg(in.rec_ray + s);
        const float t = __ldg(in.rec_t + s);
        const float px = wb_addcmul(__ldg(in.origins + 3 * ray), __ldg(in.dirs + 3 * ray), t);
        const float py = wb_addcmul(__ldg(in.origins + 3 * ray + 1), __ldg(in.dirs + 3 * ray + 1), t);
        const float pz = wb_addcmul(__ldg(in.origins + 3 * ray + 2), __ldg(in.dirs + 3 * ray + 2), t);
        // density-decoder input row: grid features (+ position embedding), zero padded to Kp; the two threads of a row split the LODs
        if (!GX) tile_gather(g, t0, c.r, c.h, px, py, pz);
        else if (c.h == 0) {
            // one thread of the row pair gathers all LODs: the gather is latency-bound, splitting it over the pair costs a group
            // barrier and scratch traffic for partial sums of 'sum' grids
            wb_featx_gather(gx, px, py, pz, [&](int f, float v) { tile_store1(t0, c.r, f, v); });
        }
        if (c.h == 0) {
            tile_embed(t0, c.r, m.feat_dim, m.pos_mode, m.pos_freq, px, py, pz);
            tile_zero(t0, c.r, m.I[0], m.Kp[0]);
        }
        if (in.x0_save) {
            tc_sync(c);
            if (valid)
                for (int ch = c.h; ch < nch0; ch += 2) in.x0_save[(int64_t)ch * in.S + s] = *reinterpret_cast<const uint4*>(t0 + ch * TC_SLAB + c.r * 16);
        }
        float df[16], c3[3];
        tc_decoders<NMAX>(m, c, in, ray, df, c3);
        if (valid && c.h == 0) {
            const float r = 1.0f / (1.0f + expf(-c3[0])), gg = 1.0f / (1.0f + expf(-c3[1])), b = 1.0f / (1.0f + expf(-c3[2]));
            shaded[s] = make_float4(r, gg, b, fmaxf(df[0], 0.0f));
        }
    }
}

// set by wb_rf_workspace_holds_ray_rows(): the next backward of this thread finds the per-ray colour-input rows in its workspace already
static thread_local int g_tc_skip_embed = 0;
static thread_local int64_t g_tc_s_begin = 0, g_tc_s_end = 0;      // sample range of the next backward launches (0, 0 = everything); set by wb_tc_shade_bwd's chunked schedule
extern "C" int wb_rf_workspace_holds_ray_rows(int32_t yes) { g_tc_skip_embed = yes ? 1 : 0; return WB_OK; }

static int tc_launch_ray_embed(const WbTc& m, const wb_rays* rays, void* workspace, cudaStream_t st)
{
    const int64_t R = rays->num_rays;
    if (R == 0) return WB_OK;
    wb_ray_embed_kernel<<<(unsigned)((R + 127) / 128), 128, 0, st>>>(m, rays->dirs, R, reinterpret_cast<uint4*>(workspace));
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// Tuning knobs; the environment overrides exist for sweeps and variant tests and are read once per process.
static int tc_env_int(const char* name, int dflt) { const char* v = getenv(name); return v && *v ? atoi(v) : dflt; }
static int tc_knob_fuse_scatter() { static const int v = tc_env_int("WB_TC_FUSE_SCATTER", 1); return v; }     // 0 separate kernel, 1 last epilogue
static int tc_knob_bwd_groups() { static const int v = tc_env_int("WB_TC_BWD_GROUPS", 2); return v; }          // upper bound: 1 or 2
static int tc_knob_fwd_ctas() { static const int v = tc_env_int("WB_TC_FWD_CTAS", 3); return v; }
static int tc_knob_fuse_scatter_wide() { static const int v = tc_env_int("WB_TC_FUSE_SCATTER_WIDE", 0); return v; }
static int64_t tc_knob_wide_min_s() { static const int v = tc_env_int("WB_TC_WIDE_MIN_S", 1 << 20); return v; }      // below this many samples the chunked schedule is not worth its launches
static int tc_knob_wide_chunks() { static const int v = tc_env_int("WB_TC_WIDE_CHUNKS", 4); return v; }       // 1: no overlap of decoder backward and table scatter
static int tc_knob_scatter_lpb() { static const int v = tc_env_int("WB_TC_SCATTER_LPB", 16); return v; }
static int tc_knob_scatter_idx2() { static const int v = tc_env_int("WB_TC_SCATTER_IDX2", 1); return v; }
static int tc_knob_scatter_ctas() { static const int v = tc_env_int("WB_TC_SCATTER_CTAS", 16); return v; }
static int tc_knob_scatter_h2() { static const int v = tc_env_int("WB_TC_SCATTER_H2", 1); return v; }
static int tc_knob_scatter_v4() { static const int v = tc_env_int("WB_TC_SCATTER_V4", 1); return v; }

int wb_tc_shade_fwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                    int64_t S, float* shaded, void* feat_save, void* workspace, cudaStream_t st)
{
    WbGrid g; int rc = wb_make_grid(nef, &g); if (rc) return rc;
    WbGridX gx; rc = wb_make_gridx(nef, false, &gx); if (rc) return rc;
    WbTc m; rc = wb_tc_make(nef, false, &m); if (rc) return rc;
    WB_CHECK_ARG(workspace != nullptr, "precision 1 needs the workspace (wb_rf_workspace_bytes)");
    rc = tc_launch_ray_embed(m, rays, workspace, st); if (rc) return rc;
    TcIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S, reinterpret_cast<const uint4*>(workspace), reinterpret_cast<uint4*>(feat_save), nullptr };
    // CTAs per SM: more groups in flight hide the gather and chain latencies.  The register bound of the instantiation must match,
    // or the hardware silently runs fewer.
    // Decoders up to 64 wide: 2 or 3 CTAs (85 registers per thread); wider ones: 1 or 2 (a 128-wide accumulator is 64 registers).
    const bool wide = m.maxw > 64;
    int per_sm = max(1, min(3, TC_SMEM_MAX / (m.smem_bytes + 1024)));
    per_sm = min(per_sm, max(1, tc_knob_fwd_ctas()));
    // the generic grids keep more state per thread (octree gather: up to 32 accumulators)
    if (gx.kind != 0) per_sm = min(per_sm, tc_env_int("WB_TC_GX_CTAS", gx.kind == 1 ? 3 : 2));
    per_sm = wide ? min(per_sm, 2) : max(per_sm, 2);
    auto kern = wide ? (gx.kind != 0 ? (per_sm == 2 ? wb_shade_fwd_tc_kernel<2, true, 128> : wb_shade_fwd_tc_kernel<1, true, 128>)
                                     : (per_sm == 2 ? wb_shade_fwd_tc_kernel<2, false, 128> : wb_shade_fwd_tc_kernel<1, false, 128>))
                     : (gx.kind != 0 ? (per_sm == 3 ? wb_shade_fwd_tc_kernel<3, true, 64> : wb_shade_fwd_tc_kernel<2, true, 64>)
                                     : (per_sm == 3 ? wb_shade_fwd_tc_kernel<3, false, 64> : wb_shade_fwd_tc_kernel<2, false, 64>));
    {   // function attributes are driver calls that can wait behind other driver work (e.g. an NVML poll): set them once, not per launch
        static int64_t done_for[2][2][4] = { { { -1, -1, -1, -1 }, { -1, -1, -1, -1 } }, { { -1, -1, -1, -1 }, { -1, -1, -1, -1 } } };
        int64_t& done = done_for[wide ? 1 : 0][gx.kind != 0 ? 1 : 0][per_sm];
        if (done != WB_ATTR_KEY(m.smem_bytes)) {
            WB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, m.smem_bytes));
            done = WB_ATTR_KEY(m.smem_bytes);
        }
    }
    const int64_t ntiles = (S + TC_ROWS - 1) / TC_ROWS, nctas = (ntiles + TC_FWD_GROUPS - 1) / TC_FWD_GROUPS;
    int64_t grid = (int64_t)wb_num_sms() * per_sm; if (grid > nctas) grid = nctas;
    if (grid == 0) return WB_OK;
    kern<<<(unsigned)grid, TC_FWD_GROUPS * TC_GROUP, m.smem_bytes, st>>>(g, gx, m, reinterpret_cast<const uint8_t*>(blob), in, reinterpret_cast<float4*>(shaded));
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// decoder backward kernel: CTA = m.groups groups (one CTA per SM: the retained tiles and the weight-grad accumulators fill shared
// memory), each group walks its own sequence of 64-sample sub-tiles with its own barrier, so the groups drift out of phase and overlap
// ---------------------------------------------------------------------------------------------------------------
struct TcGrads { float* gdens; float* gcol; const float* scale; __half* dfeat; int planes, width; };

// One LOD of the hash-table scatter for the 32 consecutive samples of a warp (F == 2): the arithmetic of wb_table_scatter_kernel
// <2, true, true> (hashgrid_interpolate_cuda.cu:151-160 + run merging + paired 16-byte reductions), callable from the decoder
// backward's last epilogue so that dL/dfeat never leaves the SM.  s0, s1: this sample's (still loss-scaled) gradient of the LOD's two
// features.  Warp-collective: every lane of the warp calls it with the same `l`.
__device__ __forceinline__ void tc_scatter_level_f2(const WbGrid& g, int l, float px, float py, float pz, bool valid, float s0, float s1,
                                                    float inv_scale, int lane, float* __restrict__ gtable)
{
    float* tb = gtable + g.begin[l] * 2;
    const bool pair_ok = (reinterpret_cast<uintptr_t>(tb) & 15u) == 0;
    uint32_t idx[8]; float cf[8]; uint64_t key = ~0ull - (uint64_t)lane;    // invalid lanes never merge
    if (valid) {
        int ix, iy, iz; float wx, wy, wz, jx, jy, jz;
        wb_cell(px, g.hres[l], g.hi[l], ix, wx, jx); wb_cell(py, g.hres[l], g.hi[l], iy, wy, jy); wb_cell(pz, g.hres[l], g.hi[l], iz, wz, jz);
        key = (uint64_t)ix | ((uint64_t)iy << 20) | ((uint64_t)iz << 40);
        const float xy00 = jx * jy, xy01 = jx * wy, xy10 = wx * jy, xy11 = wx * wy;
        cf[0] = xy00 * jz; cf[1] = xy00 * wz; cf[2] = xy01 * jz; cf[3] = xy01 * wz;
        cf[4] = xy10 * jz; cf[5] = xy10 * wz; cf[6] = xy11 * jz; cf[7] = xy11 * wz;
        wb_corner_indices(g, l, ix, iy, iz, idx);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { idx[j] = 0; cf[j] = 0.0f; }
    }
    const uint64_t kprev = __shfl_up_sync(0xffffffffu, key, 1);
    const bool head = (lane == 0) || (kprev != key);
    const uint32_t heads = __ballot_sync(0xffffffffu, head);
    const int run_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
    const int dist = lane - run_head;
    const bool tail = (lane == 31) || ((heads >> (lane + 1)) & 1u);
    const int maxd = __reduce_max_sync(0xffffffffu, dist);
    float v0[8], v1[8];
    if (maxd > 0) {     // run sums as loss-scaled fp16 pairs (one shuffle per corner and scan step), unscaled after the scan
        __half2 h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(s0 * cf[j], s1 * cf[j]);
        for (int o = 1; o <= maxd; o <<= 1) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const __half2 a = __shfl_up_sync(0xffffffffu, h[j], o);
                if (dist >= o) h[j] = __hadd2(h[j], a);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float2 f = __half22float2(h[j]); v0[j] = f.x * inv_scale; v1[j] = f.y * inv_scale; }
    } else {
        const float g0 = s0 * inv_scale, g1 = s1 * inv_scale;
#pragma unroll
        for (int j = 0; j < 8; ++j) { v0[j] = g0 * cf[j]; v1[j] = g1 * cf[j]; }
    }
    if (tail && valid) {
        float2* t2 = reinterpret_cast<float2*>(tb);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t i0 = idx[j], i1 = idx[j + 4];
            const bool nz0 = (v0[j] != 0.0f || v1[j] != 0.0f), nz1 = (v0[j + 4] != 0.0f || v1[j + 4] != 0.0f);
            if (pair_ok && ((i0 ^ i1) == 1u)) {
                if (nz0 || nz1) {
                    const float4 val = (i0 & 1u) ? make_float4(v0[j + 4], v1[j + 4], v0[j], v1[j]) : make_float4(v0[j], v1[j], v0[j + 4], v1[j + 4]);
                    atomicAdd(reinterpret_cast<float4*>(t2 + (i0 & ~1u)), val);
                }
            } else {
                if (nz0) atomicAdd(t2 + i0, make_float2(v0[j], v1[j]));
                if (nz1) atomicAdd(t2 + i1, make_float2(v0[j + 4], v1[j + 4]));
            }
        }
    }
}

// wmask: layers whose weight gradients this launch accumulates; emit: this launch produces dL/dfeat (planes, or FUSE: the hash-table
// scatter of an F == 2 'cat' grid in the last epilogue).  Wide decoders whose accumulators do not all fit run several launches.
template <int NG, bool FUSE>
__global__ void __launch_bounds__(NG * TC_GROUP, 1)
wb_mlp_bwd_tc_kernel(WbTc m, const uint8_t* __restrict__ blob, TcIn in, const float4* __restrict__ g_shaded, TcGrads G,
                     unsigned wmask, int emit, WbGrid g, float* __restrict__ gtable)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;
    const int nl = m.nl_d + m.nl_c;
    if (threadIdx.x == 0) {
        tc_mbar_init(&bar, 1); tc_mbar_init_fence();
        tc_mbar_expect_tx(&bar, (uint32_t)m.blob_bytes);
        tc_bulk_g2s(smem + m.w_smem_off, blob, (uint32_t)m.blob_bytes, &bar);
    }
    TcCtx c; tc_ctx_init(c, m, smem);
    float* acc = reinterpret_cast<float*>(c.sub + m.acc_off);
    const int nacc = (m.group_bytes - m.acc_off) / 4;
    for (int i = c.wl; i < nacc; i += TC_GROUP) acc[i] = 0.0f;
    // constant-one slab behind every input tile: feature 0 = 1, features 1..7 = 0  (bias gradient column of the weight grad)
    for (int l = c.h; l < nl; l += 2) {
        uint4 one; one.x = 0x00003C00u; one.y = 0; one.z = 0; one.w = 0;           // fp16 1.0 in the low half
        *reinterpret_cast<uint4*>(c.sub + m.tile_off[l] + (m.Kp[l] / 8) * TC_SLAB + c.r * 16) = one;
    }
    __syncthreads();
    tc_mbar_wait(&bar, 0);
    const float scale = __ldg(G.scale), inv_scale = 1.0f / scale;
    uint8_t* dyt = c.sub + m.dy_off;
    uint8_t* t0 = c.sub + m.tile_off[0];
    const uint32_t dyb = tc_smem_u32(dyt), wb = tc_smem_u32(c.blob);
    const int nch0 = m.Kp[0] / 8;
    const int64_t s_end = in.s_end ? in.s_end : in.S;             // this launch's sample range (in.S stays the stride of the saved rows / planes)
    const int64_t tile0 = in.s_begin / TC_ROWS, ntiles = (s_end + TC_ROWS - 1) / TC_ROWS;
    const float z8[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    const int lane = threadIdx.x & 31;
    for (int64_t tile = tile0 + (int64_t)blockIdx.x * NG + c.g; tile < ntiles; tile += (int64_t)gridDim.x * NG) {
        int64_t s = tile * TC_ROWS + c.r;
        const bool valid = s < s_end;
        if (!valid) s = s_end - 1;
        const int64_t ray = __ldg(in.rec_ray + s);
        for (int ch = c.h; ch < nch0; ch += 2)                     // saved density-decoder input row (coalesced 16 B per lane)
            *reinterpret_cast<uint4*>(t0 + ch * TC_SLAB + c.r * 16) = __ldg(in.x0_saved + (int64_t)ch * in.S + s);
        float df[16], c3[3];
        tc_decoders<128>(m, c, in, ray, df, c3);
        const float4 go = valid ? __ldg(g_shaded + s) : make_float4(0, 0, 0, 0);
        // ---- colour decoder, last layer: dY = dL/d(pre-sigmoid), zero padded ----
        if (c.h == 0) {
            const float r = 1.0f / (1.0f + expf(-c3[0])), gg = 1.0f / (1.0f + expf(-c3[1])), b = 1.0f / (1.0f + expf(-c3[2]));
            float v[8] = { go.x * r * (1.0f - r) * scale, go.y * gg * (1.0f - gg) * scale, go.z * b * (1.0f - b) * scale, 0, 0, 0, 0, 0 };
            tile_store8(dyt, c.r, 0, v);
        }
        for (int sl = 1 + c.h; sl < m.Np[nl - 1] / 8; sl += 2) tile_store8(dyt, c.r, sl, z8);
        for (int l = nl - 1; l >= 0; --l) {
            tc_publish(c);
            const int I = m.I[l], O = m.O[l], Kp = m.Kp[l], Np = m.Np[l];
            const uint32_t xb = tc_smem_u32(c.sub + m.tile_off[l]);
            if (m.acc_l[l] >= 0) {
                // acc_l^T[out, in] += dY_l^T . X_l and, from the constant-one slab, acc_l^T[out, I] += dY_l^T . 1  (K = the 64 samples)
                float* al = acc + m.acc_l[l];
                for (int mb = 0; mb < Np; mb += 64) {
                    const uint64_t da = tc_desc(dyb + (uint32_t)(mb / 8) * TC_SLAB, 128, TC_SLAB);
                    tc_chain_n<1, 1>(c, Kp, da, tc_desc(xb, 128, TC_SLAB), TC_ROWS / 16, 256 >> 4, 256 >> 4, nullptr, [&](auto& d) {
                        constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                        for (int i = 0; i < NR; ++i) {
                            const int o = mb + tc_frag_row(c.wl, i), k = tc_frag_col(c.wl, i);
                            if (o < O && k < I) al[o * (I + 1) + k] += d[i];
                        }
                    });
                    if (m.src_b[l] >= 0)
                        tc_chain<8, 1, 1>(c, da, tc_desc(xb + (uint32_t)(Kp / 8) * TC_SLAB, 128, TC_SLAB), TC_ROWS / 16, 256 >> 4, 256 >> 4, nullptr, [&](auto& d) {
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const int o = mb + tc_frag_row(c.wl, i);
                                if (o < O && tc_frag_col(c.wl, i) == 0) al[o * (I + 1) + I] += d[i];
                            }
                        });
                }
            }
            if (l == 0 && !emit) break;
            // dX_l = dY_l . W_l  (A: dY tile K-major over the Np outputs, B: weight pack read MN-major); the first colour layer only needs
            // the gradient of its dout - 1 <= 15 density features
            const int N = (l == m.nl_d) ? 16 : Kp;
            const uint64_t da = tc_desc(dyb, TC_SLAB, 128), db = tc_desc(wb + m.w_off[l], 128, Np * 16);
            if (l == m.nl_d) {
                // first colour layer: inputs [df[1:dout], embed(ray_d)]; only the first dout-1 carry gradient (nerf.py:259)
                tc_chain_n<0, 1>(c, N, da, db, Np / 16, (2 * TC_SLAB) >> 4, 256 >> 4, nullptr, [&](auto& d) { TC_FRAG_TO_SCRATCH(c, d, 16); });
                tc_sync(c);
                const float* v = c.scr + c.r * TC_SCR_LD;
                const int dout = m.O[m.nl_d - 1];
                float gdf[16];
                gdf[0] = (df[0] > 0.0f) ? go.w * scale : 0.0f;   // relu' of density (nerf.py:263)
#pragma unroll
                for (int j = 1; j < 16; ++j) gdf[j] = (j < dout) ? v[j - 1] : 0.0f;
                if (c.h == 0) tile_store8(dyt, c.r, 0, gdf); else tile_store8(dyt, c.r, 1, gdf + 8);
                for (int sl = 2 + c.h; sl < m.Np[l - 1] / 8; sl += 2) tile_store8(dyt, c.r, sl, z8);
            } else if (l == 0 && FUSE) {
                // dL/d(grid features) -> hash table: column half h holds features [16h, 16h+16) = LODs 8h .. 8h+7; a warp = 32
                // consecutive samples of one half
                tc_chain_n<0, 1>(c, N, da, db, Np / 16, (2 * TC_SLAB) >> 4, 256 >> 4, nullptr, [&](auto& d) { TC_FRAG_TO_SCRATCH(c, d, 32); });
                tc_sync(c);
                const float* v = c.scr + c.r * TC_SCR_LD + c.h * 16;
                const float t = __ldg(in.rec_t + s);
                const float px = wb_addcmul(__ldg(in.origins + 3 * ray), __ldg(in.dirs + 3 * ray), t);
                const float py = wb_addcmul(__ldg(in.origins + 3 * ray + 1), __ldg(in.dirs + 3 * ray + 1), t);
                const float pz = wb_addcmul(__ldg(in.origins + 3 * ray + 2), __ldg(in.dirs + 3 * ray + 2), t);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int lv = c.h * 8 + q;
                    if (lv < G.planes) tc_scatter_level_f2(g, lv, px, py, pz, valid, v[2 * q], v[2 * q + 1], inv_scale, lane, gtable);
                }
            } else if (l == 0) {
                // dL/d(grid features) -> fp16 planes [plane][S][width] (still loss-scaled), straight from the fragments
                const int W = G.width, nfe = G.planes * W;
                const int64_t srow0 = tile * TC_ROWS;
                tc_chain_n<0, 1>(c, N, da, db, Np / 16, (2 * TC_SLAB) >> 4, 256 >> 4, nullptr, [&](auto& d) {
                    constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                    for (int i = 0; i < NR; i += 2) {
                        const int64_t sr = srow0 + tc_frag_row(c.wl, i);
                        const int fe = tc_frag_col(c.wl, i);
                        if (sr >= s_end || fe >= nfe) continue;
                        if (W == 2) reinterpret_cast<__half2*>(G.dfeat)[(int64_t)(fe >> 1) * in.S + sr] = __floats2half2_rn(d[i], d[i + 1]);
                        else {
                            G.dfeat[((int64_t)(fe / W) * in.S + sr) * W + (fe % W)] = __float2half_rn(d[i]);
                            if (fe + 1 < nfe) G.dfeat[((int64_t)((fe + 1) / W) * in.S + sr) * W + ((fe + 1) % W)] = __float2half_rn(d[i + 1]);
                        }
                    }
                });
            } else {
                // hidden layer input: apply relu' from the retained activation tile, write the next dY (Np[l-1] == Kp[l])
                const uint8_t* xt = c.sub + m.tile_off[l];
                tc_chain_n<0, 1>(c, N, da, db, Np / 16, (2 * TC_SLAB) >> 4, 256 >> 4, nullptr, [&](auto& d) {
                    constexpr int NR = sizeof(d) / sizeof(float);
                    const __half2 z2 = __float2half2_rn(0.0f);
#pragma unroll
                    for (int i = 0; i < NR; i += 2) {
                        const int row = tc_frag_row(c.wl, i), col = tc_frag_col(c.wl, i);
                        const int off = (col >> 3) * TC_SLAB + row * 16 + (col & 7) * 2;
                        // relu'(x) as a 16-bit lane mask of the retained fp16 activation (>= 0 by construction)
                        const uint32_t a = *reinterpret_cast<const uint32_t*>(xt + off);
                        *reinterpret_cast<uint32_t*>(dyt + off) = tc_pack2(d[i], d[i + 1]) & __hgt2_mask(*reinterpret_cast<const __half2*>(&a), z2);
                    }
                });
            }
        }
    }
    // ---- flush the weight / bias gradient accumulators of every group ----
    __syncthreads();
    for (int l = 0; l < nl; ++l) {
        if (m.acc_l[l] < 0) continue;
        float* gbase = l < m.nl_d ? G.gdens : G.gcol;
        const int I = m.I[l], O = m.O[l];
        for (int e = threadIdx.x; e < O * (I + 1); e += blockDim.x) {
            float v = 0.0f;
            for (int gi = 0; gi < NG; ++gi) v += reinterpret_cast<const float*>(smem + gi * m.group_bytes + m.acc_off)[m.acc_l[l] + e];
            const int o = e / (I + 1), i = e % (I + 1);
            const float val = v * inv_scale;
            if (i < I) { if (val != 0.0f) atomicAdd(gbase + m.src_w[l] + o * I + i, val); }
            else if (m.src_b[l] >= 0) atomicAdd(gbase + m.src_b[l] + o, val);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// table scatter: dL/dfeat planes -> hash table (hashgrid_interpolate_cuda.cu:151-160), with warp-level run merging
// ---------------------------------------------------------------------------------------------------------------
template <int F, bool H2, bool IDX2>   // H2: the run sums travel through the warp scan as loss-scaled fp16 pairs (one shuffle per corner)
                                       // IDX2: corner entries through wb_corner_indices (one multiply per axis) instead of 8 x wb_hash_idx
__global__ void __launch_bounds__(256)
wb_table_scatter_kernel(WbGrid g, TcIn in, const __half* __restrict__ dfeat, int planes, int levels, int lpb,
                        const float* __restrict__ scale_p, float* __restrict__ gtable, int pair_v4)
{
    const int l_begin = blockIdx.y * lpb, l_end = min(levels, l_begin + lpb);     // this CTA's LODs; the sample position is built once for all of them
    const int lane = threadIdx.x & 31;
    const float scale = __ldg(scale_p), inv_scale = 1.0f / scale;
    const int Fr = F > 0 ? F : g.F;
    const int64_t s_end = in.s_end ? in.s_end : in.S;
    const int64_t nwork = in.s_begin + ((s_end - in.s_begin + 31) & ~(int64_t)31);            // whole warps
    for (int64_t s = in.s_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nwork; s += (int64_t)gridDim.x * blockDim.x) {
        const bool valid = s < s_end;
        float px = 0.0f, py = 0.0f, pz = 0.0f;
        if (valid) {
            const int64_t ray = __ldg(in.rec_ray + s);
            const float t = __ldg(in.rec_t + s);
            px = wb_addcmul(__ldg(in.origins + 3 * ray), __ldg(in.dirs + 3 * ray), t);
            py = wb_addcmul(__ldg(in.origins + 3 * ray + 1), __ldg(in.dirs + 3 * ray + 1), t);
            pz = wb_addcmul(__ldg(in.origins + 3 * ray + 2), __ldg(in.dirs + 3 * ray + 2), t);
        }
        __half2 gnext = __float2half2_rn(0.0f);                  // F == 2: the next LOD's gradient is fetched one LOD ahead
        if (F == 2 && valid && l_begin < l_end)
            gnext = reinterpret_cast<const __half2*>(dfeat)[(int64_t)(g.multiscale == 0 ? l_begin : 0) * in.S + s];
        for (int l = l_begin; l < l_end; ++l) {
            const int pl = g.multiscale == 0 ? l : 0;
            float* tb = gtable + g.begin[l] * Fr;
            const bool pair_ok = pair_v4 && ((reinterpret_cast<uintptr_t>(tb) & 15u) == 0);       // level base 16-byte aligned
            uint32_t idx[8]; float cf[8]; uint64_t key = ~0ull - (uint64_t)lane;    // invalid lanes never merge
            float gv[F > 0 ? F : 8];
#pragma unroll
            for (int f = 0; f < (F > 0 ? F : 8); ++f) gv[f] = 0.0f;
            if (valid) {
                int ix, iy, iz; float wx, wy, wz, jx, jy, jz;
                wb_cell(px, g.hres[l], g.hi[l], ix, wx, jx); wb_cell(py, g.hres[l], g.hi[l], iy, wy, jy); wb_cell(pz, g.hres[l], g.hi[l], iz, wz, jz);
                key = (uint64_t)ix | ((uint64_t)iy << 20) | ((uint64_t)iz << 40);
                const float xy00 = jx * jy, xy01 = jx * wy, xy10 = wx * jy, xy11 = wx * wy;
                cf[0] = xy00 * jz; cf[1] = xy00 * wz; cf[2] = xy01 * jz; cf[3] = xy01 * wz;
                cf[4] = xy10 * jz; cf[5] = xy10 * wz; cf[6] = xy11 * jz; cf[7] = xy11 * wz;
                if (IDX2) wb_corner_indices(g, l, ix, iy, iz, idx);
                else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) idx[j] = wb_hash_idx(ix + ((j & 4) >> 2), iy + ((j & 2) >> 1), iz + (j & 1), g.res[l], g.Tmask, g.dense[l]);
                }
                if (F == 2) {
                    const float2 gg = __half22float2(gnext);
                    gv[0] = gg.x * inv_scale; gv[1] = gg.y * inv_scale;
                    if (l + 1 < l_end) gnext = reinterpret_cast<const __half2*>(dfeat)[(int64_t)(g.multiscale == 0 ? l + 1 : 0) * in.S + s];
                } else {
                    for (int f = 0; f < Fr; ++f) gv[f] = __half2float(dfeat[((int64_t)pl * in.S + s) * Fr + f]) * inv_scale;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) { idx[j] = 0; cf[j] = 0.0f; }
            }
            // runs of consecutive lanes with the same cell
            const uint64_t kprev = __shfl_up_sync(0xffffffffu, key, 1);
            const bool head = (lane == 0) || (kprev != key);
            const uint32_t heads = __ballot_sync(0xffffffffu, head);
            const int run_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
            const int dist = lane - run_head;
            const bool tail = (lane == 31) || ((heads >> (lane + 1)) & 1u);
            int maxd = dist;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) maxd = max(maxd, __shfl_xor_sync(0xffffffffu, maxd, o));
            if (F == 2) {
                float v0[8], v1[8];
                if (H2 && maxd > 0) {
                    // gradients arrive as fp16 anyway: scan the (still loss-scaled) products as half2, unscale after the scan
                    const float s0 = gv[0] * scale, s1 = gv[1] * scale;
                    __half2 h[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(s0 * cf[j], s1 * cf[j]);
                    for (int o = 1; o <= maxd; o <<= 1) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const __half2 a = __shfl_up_sync(0xffffffffu, h[j], o);
                            if (dist >= o) h[j] = __hadd2(h[j], a);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) { const float2 f = __half22float2(h[j]); v0[j] = f.x * inv_scale; v1[j] = f.y * inv_scale; }
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) { v0[j] = gv[0] * cf[j]; v1[j] = gv[1] * cf[j]; }
                    for (int o = 1; o <= maxd; o <<= 1) {               // segmented inclusive scan (warp-uniform trip count)
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float a = __shfl_up_sync(0xffffffffu, v0[j], o), b = __shfl_up_sync(0xffffffffu, v1[j], o);
                            if (dist >= o) { v0[j] += a; v1[j] += b; }
                        }
                    }
                }
                if (tail && valid) {
                    // corners j and j + 4 are x-neighbours at the same (y, z).  When their entries differ only in bit 0 (dense level with
                    // an even index; hashed level with an even x, because (x | 1) ^ A == (x ^ A) ^ 1) the two 8-byte updates are one
                    // aligned 16-byte red.global.add.v4.f32 (measured: -6 % kernel time).
                    float2* t2 = reinterpret_cast<float2*>(tb);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t i0 = idx[j], i1 = idx[j + 4];
                        const bool nz0 = (v0[j] != 0.0f || v1[j] != 0.0f), nz1 = (v0[j + 4] != 0.0f || v1[j + 4] != 0.0f);
                        if (pair_ok && ((i0 ^ i1) == 1u)) {
                            if (nz0 || nz1) {
                                const float4 val = (i0 & 1u) ? make_float4(v0[j + 4], v1[j + 4], v0[j], v1[j]) : make_float4(v0[j], v1[j], v0[j + 4], v1[j + 4]);
                                atomicAdd(reinterpret_cast<float4*>(t2 + (i0 & ~1u)), val);
                            }
                        } else {
                            if (nz0) atomicAdd(t2 + i0, make_float2(v0[j], v1[j]));
                            if (nz1) atomicAdd(t2 + i1, make_float2(v0[j + 4], v1[j + 4]));
                        }
                    }
                }
            } else {
                for (int f = 0; f < Fr; ++f) {
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = gv[f] * cf[j];
                    for (int o = 1; o <= maxd; o <<= 1) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) { const float a = __shfl_up_sync(0xffffffffu, v[j], o); if (dist >= o) v[j] += a; }
                    }
                    if (tail && valid) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) if (v[j] != 0.0f) atomicAdd(tb + (int64_t)idx[j] * Fr + f, v[j]);
                    }
                }
            }
        }
    }
}

// dL/dfeat planes -> triplanar planes / octree feature levels (kinds 1, 2): one thread per sample, lanes = consecutive samples.
// Triplanar: consecutive samples of a ray stay in the same texel cell for several steps on the coarse planes (8 / 4 / 2 / 1 samples per
// cell on the four LODs of config 4), and the plane reductions are the wall of that configuration (6.3e10 per 800^2 frame at the L2
// reduction rate): runs of lanes with the same (LOD, plane, cell) are summed with a segmented warp scan -- 4 texel weights x C channels
// per lane -- and only the last lane of a run issues the reductions, as the hash-grid scatter does for its cells.
__global__ void __launch_bounds__(256)
wb_featx_scatter_kernel(WbGridX gx, TcIn in, const __half* __restrict__ dfeat, int width, const float* __restrict__ scale_p)
{
    const float inv_scale = 1.0f / __ldg(scale_p);
    const int lane = threadIdx.x & 31;
    const int64_t nwork = (in.S + 31) & ~(int64_t)31;            // whole warps
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nwork; s += (int64_t)gridDim.x * blockDim.x) {
        const bool valid = s < in.S;
        float px = 0.0f, py = 0.0f, pz = 0.0f;
        if (valid) {
            const int64_t ray = __ldg(in.rec_ray + s);
            const float t = __ldg(in.rec_t + s);
            px = wb_addcmul(__ldg(in.origins + 3 * ray), __ldg(in.dirs + 3 * ray), t);
            py = wb_addcmul(__ldg(in.origins + 3 * ray + 1), __ldg(in.dirs + 3 * ray + 1), t);
            pz = wb_addcmul(__ldg(in.origins + 3 * ray + 2), __ldg(in.dirs + 3 * ray + 2), t);
        }
        auto grad = [&](int f) {                                  // feature f lives in plane f / width at column f % width
            return __half2float(dfeat[((int64_t)(f / width) * in.S + s) * width + (f % width)]) * inv_scale;
        };
        if (gx.kind != 1 || gx.C > 4) {                           // octree grid (or wide triplanar channels): no merging
            if (valid) wb_featx_scatter(gx, px, py, pz, grad);
            continue;
        }
        const int C = gx.C;
        float gsum[3][4];                                         // 'sum' grids: every LOD receives the same dL/dfeat -> loaded once per sample
#pragma unroll
        for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int c = 0; c < 4; ++c) gsum[p][c] = (gx.sum && valid && c < C) ? grad(p * C + c) : 0.0f;
        for (int l = 0; l < gx.nl; ++l) {
            const int size = gx.res[l] + 1; const int64_t hw = (int64_t)size * size;
#pragma unroll
            for (int p = 0; p < 3; ++p) {
                WbBilinear b = wb_tp_setup(px, py, pz, p, size);
                float v[4][4];                                    // [texel nw, ne, sw, se][channel]
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float g = gx.sum ? gsum[p][c] : ((valid && c < C) ? grad((l * 3 + p) * C + c) : 0.0f);
                    v[0][c] = g * b.nw; v[1][c] = g * b.ne; v[2][c] = g * b.sw; v[3][c] = g * b.se;
                }
                const int key = valid ? b.o00 : -1 - lane;        // invalid lanes never merge
                const int kprev = __shfl_up_sync(0xffffffffu, key, 1);
                const bool head = (lane == 0) || (kprev != key);
                const uint32_t heads = __ballot_sync(0xffffffffu, head);
                const int run_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
                const int dist = lane - run_head;
                const bool tail = (lane == 31) || ((heads >> (lane + 1)) & 1u);
                const int maxd = __reduce_max_sync(0xffffffffu, dist);
                for (int o = 1; o <= maxd; o <<= 1) {             // segmented inclusive scan (warp-uniform trip count)
#pragma unroll
                    for (int t4 = 0; t4 < 4; ++t4)
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const float a = __shfl_up_sync(0xffffffffu, v[t4][c], o);
                            if (dist >= o) v[t4][c] += a;
                        }
                }
                if (tail && valid && gx.chlast) {                 // C == 4, channel-last gradients: one 16-byte reduction per texel
                    float4* t4 = reinterpret_cast<float4*>(gx.gptr[l * 3 + p]);
                    auto nz = [](const float* q) { return q[0] != 0.0f || q[1] != 0.0f || q[2] != 0.0f || q[3] != 0.0f; };
                    if (nz(v[0])) atomicAdd(t4 + b.o00, make_float4(v[0][0], v[0][1], v[0][2], v[0][3]));
                    if (b.bx1 && nz(v[1])) atomicAdd(t4 + b.o01, make_float4(v[1][0], v[1][1], v[1][2], v[1][3]));
                    if (b.by1 && nz(v[2])) atomicAdd(t4 + b.o10, make_float4(v[2][0], v[2][1], v[2][2], v[2][3]));
                    if (b.bx1 && b.by1 && nz(v[3])) atomicAdd(t4 + b.o11, make_float4(v[3][0], v[3][1], v[3][2], v[3][3]));
                } else if (tail && valid) {
                    float* pl = gx.gptr[l * 3 + p];
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        if (c >= C) break;
                        float* ch = pl + c * hw;
                        if (v[0][c] != 0.0f) atomicAdd(ch + b.o00, v[0][c]);
                        if (b.bx1 && v[1][c] != 0.0f) atomicAdd(ch + b.o01, v[1][c]);
                        if (b.by1 && v[2][c] != 0.0f) atomicAdd(ch + b.o10, v[2][c]);
                        if (b.bx1 && b.by1 && v[3][c] != 0.0f) atomicAdd(ch + b.o11, v[3][c]);
                    }
                }
            }
        }
    }
}

// decoder backward only: dL/d(shaded) -> weight gradients + dL/dfeat planes in the workspace
// grad_table != NULL asks for the table scatter to be fused into the decoder backward; *fused_out reports whether it was (it is for
// F == 2 'cat' hash grids) -- otherwise the caller runs wb_tc_table_scatter afterwards
int wb_tc_decoder_bwd_ex(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                         int64_t S, const float* g_shaded, const float* scale, const void* feat_saved, void* workspace,
                         float* grad_dens, float* grad_col, float* grad_table, int* fused_out, cudaStream_t st);
int wb_tc_decoder_bwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                      int64_t S, const float* g_shaded, const float* scale, const void* feat_saved, void* workspace,
                      float* grad_dens, float* grad_col, cudaStream_t st)
{
    return wb_tc_decoder_bwd_ex(nef, blob, rays, rec_t, rec_ray, S, g_shaded, scale, feat_saved, workspace, grad_dens, grad_col, nullptr, nullptr, st);
}

// the launches of one decoder backward: layer masks of the weight-grad accumulators that fit beside the tiles, and the group count
static int tc_bwd_passes(WbTc* m, unsigned masks[TC_ML])
{
    const int nl = m->nl_d + m->nl_c;
    int n = 0; unsigned cur = 0;
    for (int l = 0; l < nl; ++l) {
        if (cur && !tc_bwd_layout(m, cur | (1u << l), 1)) { masks[n++] = cur; cur = 0; }
        cur |= 1u << l;
    }
    masks[n++] = cur;
    return n;
}

int wb_tc_decoder_bwd_ex(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                         int64_t S, const float* g_shaded, const float* scale, const void* feat_saved, void* workspace,
                         float* grad_dens, float* grad_col, float* grad_table, int* fused_out, cudaStream_t st)
{
    if (fused_out) *fused_out = 0;
    WbTc m; int rc = wb_tc_make(nef, true, &m); if (rc) return rc;
    WB_CHECK_ARG(scale != nullptr, "precision 1 needs the device loss-scale pointer");
    WB_CHECK_ARG(feat_saved != nullptr && workspace != nullptr, "precision 1 backward needs the saved features and the workspace");
    if (g_tc_skip_embed) g_tc_skip_embed = 0;          // the forward's workspace (same rays) is being reused: the rows are there
    else { rc = tc_launch_ray_embed(m, rays, workspace, st); if (rc) return rc; }
    int planes, width; tc_dfeat_shape(nef, &planes, &width);
    const int64_t R = rays->num_rays;
    __half* dfeat = reinterpret_cast<__half*>(reinterpret_cast<uint8_t*>(workspace) + tc_align256(R * m.Kp[m.nl_d] * 2));
    TcIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S, reinterpret_cast<const uint4*>(workspace), nullptr, reinterpret_cast<const uint4*>(feat_saved),
                g_tc_s_begin, g_tc_s_end };
    const int64_t S_launch = (g_tc_s_end ? g_tc_s_end : S) - g_tc_s_begin;
    if (S_launch <= 0) return WB_OK;
    TcGrads G = { grad_dens, grad_col, scale, dfeat, planes, width };
    unsigned masks[TC_ML];
    const int npass = tc_bwd_passes(&m, masks);
    for (int p = 0; p < npass; ++p) {
        tc_bwd_layout(&m, masks[p], 1);
        // two groups per CTA where they fit (the groups overlap each other's barrier and MMA latencies)
        if (tc_knob_bwd_groups() >= 2) { WbTc m2 = m; if (tc_bwd_layout(&m2, masks[p], 2)) m = m2; }
        const bool emit = p == npass - 1;
        // fused table scatter: F == 2 'cat' hash grids with <= 16 live LODs (32 features: the scratch tile); with one group per SM
        // only on request (WB_TC_FUSE_SCATTER_WIDE=1): the stand-alone scatter kernel runs beside the decoder CTAs instead
        const bool fuse = emit && grad_table != nullptr && tc_knob_fuse_scatter() && nef->grid_kind == 0 && nef->feature_dim == 2 &&
                          nef->multiscale == 0 && planes <= 16 && (m.groups > 1 || tc_knob_fuse_scatter_wide());
        WbGrid g; memset(&g, 0, sizeof(g));
        if (fuse) { rc = wb_make_grid(nef, &g); if (rc) return rc; }
        auto kern = m.groups == 2 ? (fuse ? wb_mlp_bwd_tc_kernel<2, true> : wb_mlp_bwd_tc_kernel<2, false>)
                                  : (fuse ? wb_mlp_bwd_tc_kernel<1, true> : wb_mlp_bwd_tc_kernel<1, false>);
        {
            static int64_t done_for[2][2] = { { -1, -1 }, { -1, -1 } };
            int64_t& done = done_for[m.groups - 1][fuse ? 1 : 0];
            if (done != WB_ATTR_KEY(TC_SMEM_MAX)) {        // the passes of one call differ in size: allow the largest once
                WB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX));
                done = WB_ATTR_KEY(TC_SMEM_MAX);
            }
        }
        const int64_t nctas = ((S_launch + g_tc_s_begin % TC_ROWS + TC_ROWS - 1) / TC_ROWS + m.groups - 1) / m.groups;
        int64_t grid = (int64_t)wb_num_sms(); if (grid > nctas) grid = nctas;         // 1 CTA / SM: shared memory holds the tiles and accumulators
        kern<<<(unsigned)grid, m.groups * TC_GROUP, m.smem_bytes, st>>>(m, reinterpret_cast<const uint8_t*>(blob), in,
                                                                        reinterpret_cast<const float4*>(g_shaded), G, masks[p], emit ? 1 : 0, g, grad_table);
        WB_LAUNCH_CHECK();
        if (fuse && fused_out) *fused_out = 1;
    }
    return WB_OK;
}
// table scatter only: dL/dfeat planes (written by wb_tc_decoder_bwd into the same workspace) -> grad_table
int wb_tc_table_scatter(const wb_nef_desc* nef, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray, int64_t S,
                        const float* scale, void* workspace, float* grad_table, cudaStream_t st)
{
    WbGrid g; int rc = wb_make_grid(nef, &g); if (rc) return rc;
    WbGridX gx; rc = wb_make_gridx(nef, true, &gx); if (rc) return rc;
    WbTc m; rc = wb_tc_make(nef, true, &m); if (rc) return rc;
    WB_CHECK_ARG(scale != nullptr && workspace != nullptr && (grad_table != nullptr || gx.kind != 0), "null pointer");
    int planes, width; tc_dfeat_shape(nef, &planes, &width);
    const int64_t R = rays->num_rays;
    const __half* dfeat = reinterpret_cast<const __half*>(reinterpret_cast<const uint8_t*>(workspace) + tc_align256(R * m.Kp[m.nl_d] * 2));
    TcIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S, nullptr, nullptr, nullptr, gx.kind != 0 ? 0 : g_tc_s_begin, gx.kind != 0 ? 0 : g_tc_s_end };
    const int64_t S_launch = gx.kind != 0 ? S : (g_tc_s_end ? g_tc_s_end : S) - g_tc_s_begin;
    if (gx.kind != 0) {
        int64_t bx = (S + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 16; if (bx > cap) bx = cap;
        wb_featx_scatter_kernel<<<(unsigned)bx, 256, 0, st>>>(gx, in, dfeat, width, scale);
        WB_LAUNCH_CHECK();
        return WB_OK;
    }
    const int levels = g.multiscale == 0 ? planes : g.L;
    if (levels > 0) {
        // LODs per CTA row: the sample position / record loads are shared by `lpb` LODs (measured sweep in profiles/README.md)
        const int lpb = max(1, min(levels, tc_knob_scatter_lpb()));
        int64_t bx = (S_launch + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * tc_knob_scatter_ctas(); if (bx > cap) bx = cap;
        dim3 grid2((unsigned)bx, (unsigned)((levels + lpb - 1) / lpb));
        const int v4 = tc_knob_scatter_v4();
        if (g.F == 2 && tc_knob_scatter_h2() && tc_knob_scatter_idx2()) wb_table_scatter_kernel<2, true, true><<<grid2, 256, 0, st>>>(g, in, dfeat, planes, levels, lpb, scale, grad_table, v4);
        else if (g.F == 2 && tc_knob_scatter_h2()) wb_table_scatter_kernel<2, true, false><<<grid2, 256, 0, st>>>(g, in, dfeat, planes, levels, lpb, scale, grad_table, v4);
        else if (g.F == 2) wb_table_scatter_kernel<2, false, false><<<grid2, 256, 0, st>>>(g, in, dfeat, planes, levels, lpb, scale, grad_table, v4);
        else wb_table_scatter_kernel<0, false, false><<<grid2, 256, 0, st>>>(g, in, dfeat, planes, levels, lpb, scale, grad_table, 0);
        WB_LAUNCH_CHECK();
    }
    return WB_OK;
}

// Wide decoders (one 256-thread group per SM, half the register file and all the other warp slots idle): the sample range is cut
// into chunks; the decoder backward of chunk c+1 runs on the caller's stream while the table scatter of chunk c (an issue-bound SIMT
// kernel with 48 registers per thread and no shared memory: two of its CTAs fit beside a decoder CTA) runs on a side stream.
struct TcSide { cudaStream_t stream; cudaEvent_t ev[17]; bool ok; };
static TcSide* tc_side_stream()
{
    static TcSide side[64];
    int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    TcSide& s = side[dev];
    if (!s.ok) {
        if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
        for (int i = 0; i < 17; ++i) if (cudaEventCreateWithFlags(&s.ev[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
        s.ok = true;
    }
    return &s;
}

int wb_tc_shade_bwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                    int64_t S, const float* g_shaded, const float* scale, const void* feat_saved, void* workspace,
                    float* grad_table, float* grad_dens, float* grad_col, cudaStream_t st)
{
    {
        WbTc m; unsigned masks[TC_ML];
        int chunks = tc_knob_wide_chunks(); if (chunks > 16) chunks = 16;
        TcSide* side = nullptr;
        bool wide = false;         // one group per SM (wide decoders): the decoder backward leaves most warp slots idle
        if (chunks > 1 && S >= tc_knob_wide_min_s() && nef->grid_kind == 0 && grad_table && wb_tc_make(nef, true, &m) == WB_OK) {
            tc_bwd_passes(&m, masks);
            tc_bwd_layout(&m, masks[0], 1);
            wide = !(tc_knob_bwd_groups() >= 2 && tc_bwd_layout(&m, masks[0], 2));
        }
        if (wide && !tc_knob_fuse_scatter_wide() && (side = tc_side_stream()) != nullptr) {
            const int64_t per = ((S + chunks - 1) / chunks + TC_ROWS - 1) / TC_ROWS * TC_ROWS;
            int rc = WB_OK, c = 0;
            for (int64_t s0 = 0; s0 < S && rc == WB_OK; s0 += per, ++c) {
                g_tc_s_begin = s0; g_tc_s_end = s0 + per < S ? s0 + per : S;
                if (c > 0) g_tc_skip_embed = 1;                       // the per-ray rows were written by the first chunk's launch
                rc = wb_tc_decoder_bwd_ex(nef, blob, rays, rec_t, rec_ray, S, g_shaded, scale, feat_saved, workspace, grad_dens, grad_col, nullptr, nullptr, st);
                if (rc == WB_OK && (cudaEventRecord(side->ev[c], st) != cudaSuccess || cudaStreamWaitEvent(side->stream, side->ev[c], 0) != cudaSuccess)) rc = WB_ERR_CUDA;
                if (rc == WB_OK) rc = wb_tc_table_scatter(nef, rays, rec_t, rec_ray, S, scale, workspace, grad_table, side->stream);
            }
            g_tc_s_begin = 0; g_tc_s_end = 0;
            // the caller's stream continues after the last scatter (also on an error path: never leave the side stream unjoined)
            if (cudaEventRecord(side->ev[16], side->stream) != cudaSuccess || cudaStreamWaitEvent(st, side->ev[16], 0) != cudaSuccess) { if (rc == WB_OK) rc = WB_ERR_CUDA; }
            return rc;
        }
    }
    int fused = 0;
    int rc = wb_tc_decoder_bwd_ex(nef, blob, rays, rec_t, rec_ray, S, g_shaded, scale, feat_saved, workspace, grad_dens, grad_col, grad_table, &fused, st);
    if (rc || fused) return rc;
    return wb_tc_table_scatter(nef, rays, rec_t, rec_ray, S, scale, workspace, grad_table, st);
}
