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
//   as one commit group and one wait per layer (layers with inputs wider than 64: one round per chain, for the registers),
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
#include "wb_shade_tc.cuh"
#include "wb_tc.cuh"
#include <math.h>
#include <mutex>
#include <type_traits>
#include <utility>

#define TC_ML (2 * WB_MAX_LAYERS)
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
    off += wb_round_up(acc * 4, 16);
    m->group_bytes = off;
    m->groups = groups;
    m->w_smem_off = groups * off;
    m->smem_bytes = m->w_smem_off + m->blob_bytes;
    return m->smem_bytes <= TC_SMEM_MAX;
}

// The decoder backward (wb_tc_make): npass passes over the samples, pass p with groups[p] sub-tile groups per CTA accumulating the
// weight gradients of the layers in mask[p]; the last pass emits dL/dfeat, or where `fuses` may scatter it into the hash table.
struct TcBwdPlan { int npass; unsigned mask[TC_ML]; int groups[TC_ML]; bool fuses; };

// The passes of decoders m: the layers in order while their accumulators fit beside the tiles of one group, two groups per CTA where
// they fit (they overlap each other's barrier and MMA latencies).  0 when the backward does not fit: it takes decoders whose whole
// backward fits two groups per CTA in one pass, and those of the app/nerf depth (one hidden density layer, two hidden colour layers) up
// to width 128, as long as each layer's accumulator fits beside the tiles of one group; deeper, wider decoders train on the fp32 kernels.
static int tc_bwd_passes(WbTc m, unsigned masks[TC_ML], int groups[TC_ML])
{
    const int nl = m.nl_d + m.nl_c;
    const bool one_pass = tc_bwd_layout(&m, (1u << nl) - 1u, 2);
    bool passes = m.nl_d <= 2 && m.nl_c <= 3;
    for (int l = 0; l < nl && passes; ++l) passes = tc_bwd_layout(&m, 1u << l, 1);
    if (!one_pass && !passes) return 0;
    int n = 0; unsigned cur = 0;
    for (int l = 0; l < nl; ++l) {
        if (cur && !tc_bwd_layout(&m, cur | (1u << l), 1)) { masks[n++] = cur; cur = 0; }
        cur |= 1u << l;
    }
    masks[n++] = cur;
    for (int p = 0; p < n; ++p) groups[p] = tc_bwd_layout(&m, masks[p], 2) ? 2 : 1;
    return n;
}

// decoders m with the shared-memory plan of pass p
static WbTc tc_bwd_pass(WbTc m, const TcBwdPlan& b, int p) { tc_bwd_layout(&m, b.mask[p], b.groups[p]); return m; }

// workspace layout (bytes): [ray_embed: R * Kc * 2][dfeat: planes * S * F * 2 (backward only)].  dL/dfeat of R rays: its offset,
// planes ('cat' -> one per live LOD, 'sum' -> one) and halfs per (plane, sample)
struct TcDfeat { int64_t off; int planes, width; };
static TcDfeat tc_dfeat(const wb_nef_desc* d, const WbTc& m, int64_t R)
{
    const int planes = d->multiscale == 0 ? (d->lod_idx < d->num_lods ? d->lod_idx : d->num_lods) : 1;
    return { wb_align256(R * m.Kp[m.nl_d] * 2), planes < 0 ? 0 : planes, d->feature_dim };
}

// fused table scatter: F == 2 'cat' hash grids with <= 16 live LODs (32 features: the scratch tile), when the pass planned in m
// runs two groups per CTA; with one group per SM the stand-alone scatter kernel runs beside the decoder CTAs instead
static bool tc_bwd_fuses(const wb_nef_desc* nef, const WbTc& m, int planes)
{
    return nef->grid_kind == 0 && nef->feature_dim == 2 && nef->multiscale == 0 && planes <= 16 && m.groups > 1;
}

// The padded decoders and their parameter blob in *m, with the forward's shared-memory plan, or (bwd) with none and the backward's plan
// in *bwd.  Returns WB_OK, or WB_ERR_INVALID with a message when that direction does not fit the tensor-core path.
int wb_tc_make(const wb_nef_desc* d, WbTc* m, TcBwdPlan* bwd = nullptr)
{
    WbDecoders dec; const int rc = wb_make_decoders(d, 128, "tensor-core path: layer widths must be <= 128", &dec); if (rc) return rc;
    const int dout = dec.O[dec.nl_d - 1];
    WB_CHECK_ARG(dout >= 2 && dout <= 16, "tensor-core path: decoder_density output must be 2..16 wide");
    memset(m, 0, sizeof(*m));
    m->nl_d = dec.nl_d; m->nl_c = dec.nl_c;
    m->feat_dim = dec.feat_dim; m->pos_dim = dec.pos_dim; m->view_dim = dec.view_dim;
    m->pos_mode = d->pos_mode; m->pos_freq = d->pos_freq; m->view_mode = d->view_mode; m->view_freq = d->view_freq;
    const int nl = m->nl_d + m->nl_c;
    int off = 0, maxw = 0;
    for (int l = 0; l < nl; ++l) {
        const int I = dec.I[l], O = dec.O[l];
        m->I[l] = I; m->O[l] = O; m->Kp[l] = wb_round_up(I, 16); m->Np[l] = wb_round_up(O, 16);
        m->w_off[l] = off; off += m->Kp[l] * m->Np[l] * 2;
        m->b_off[l] = off; off += m->Np[l] * 32;
        m->src_w[l] = dec.src_w[l]; m->src_b[l] = dec.src_b[l];
        maxw = max(maxw, max(m->Kp[l], m->Np[l]));
    }
    m->blob_bytes = wb_round_up(off, 16);
    m->has_bias = d->has_bias ? 1 : 0;
    m->maxw = maxw;
    if (bwd) {
        bwd->npass = tc_bwd_passes(*m, bwd->mask, bwd->groups);
        WB_CHECK_ARG(bwd->npass > 0, "tensor-core path: decoder backward does not fit in shared memory (use precision 0)");
        bwd->fuses = tc_bwd_fuses(d, tc_bwd_pass(*m, *bwd, bwd->npass - 1), tc_dfeat(d, *m, 0).planes);
        return WB_OK;
    }
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

int64_t wb_tc_workspace_bytes(const wb_nef_desc* nef, int64_t R, int64_t S, int backward)
{
    WbTc m; if (wb_tc_make(nef, &m)) return -1;
    const TcDfeat df = tc_dfeat(nef, m, R);
    int64_t b = df.off;
    if (backward) b += wb_align256((int64_t)df.planes * S * df.width * 2);
    return b + 256;
}
int wb_tc_supported(const wb_nef_desc* nef, int backward)
{
    WbTc m; TcBwdPlan plan; if (wb_tc_make(nef, &m)) return 0;
    if (backward && wb_tc_make(nef, &m, &plan)) return 0;
    return 1;
}
// the features are only saved for a backward pass: refuse here (at forward time) if that pass cannot run
int64_t wb_tc_feat_bytes(const wb_nef_desc* nef, int64_t S)
{
    WbTc m; TcBwdPlan plan; if (wb_tc_make(nef, &m, &plan) || wb_tc_make(nef, &m)) return -1;
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

int wb_tc_blob_floats(const wb_nef_desc* nef) { WbTc m; if (wb_tc_make(nef, &m)) return -1; return m.blob_bytes / 4; }

int wb_tc_pack(const wb_nef_desc* nef, float* blob, cudaStream_t st)
{
    WbTc m; int rc = wb_tc_make(nef, &m); if (rc) return rc;
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
    int64_t s_begin, s_end;      // backward: this launch's samples [s_begin, s_end), s_begin a multiple of 64 (s_end == 0: up to S); S stays the plane stride
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
// `half` (0/1): the two threads of a row split the work -- slab (4 LODs) k goes to half k & 1 on the F == 2 'cat' path, except a
// partial last slab (L % 4 != 0), which goes to half 0: its zero-filled tail holds the first features of the position embedding,
// which half 0 writes after the gather, so the two halves store disjoint bytes.  The generic paths are done by half 0 alone.
__device__ __forceinline__ void tile_gather(const WbGrid& g, uint8_t* tile, int r, int half, float px, float py, float pz)
{
    const int L = g.L, F = g.F;
    if (g.multiscale == 0 && F == 2) {
        const int nslab = (L + 3) >> 2, partial = (L & 3) ? nslab - 1 : -1;
        for (int sl = 0; sl < nslab; ++sl) {                    // 4 levels = 8 features = one slab row (16 B store)
            if ((sl == partial ? 0 : (sl & 1)) != half) continue;
            const int l0 = 4 * sl;
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
// decoder geometry as a kernel template parameter: the layer counts and padded widths, read from WbTc at run time (TcShapeRt) or
// fixed at compile time (TcShape).  A TcShape walks the layers unrolled, with the layer index and the widths as integral
// constants, so every wgmma chain and backward round gets its width at compile time and the kernel holds only the code its layers
// run: the run-time kernels switch over the widths 16 .. NMAX in every layer and inline each case's chains and epilogues, hundreds
// of KB of SASS that a 64-sample tile walks through in every round.
// ---------------------------------------------------------------------------------------------------------------
template <int L> using TcInt = std::integral_constant<int, L>;
// layer l + D: an int, or for a compile-time layer index the TcInt of its neighbour
template <int D> __device__ __forceinline__ int tc_step(int l) { return l + D; }
template <int D, int L> __device__ __forceinline__ TcInt<L + D> tc_step(TcInt<L>) { return {}; }
struct TcShapeRt {
    static constexpr bool fixed = false;
    static constexpr int kp0 = 0;                  // padded width of the first layer, when known at compile time
    static __device__ __forceinline__ int nl_d(const WbTc& m) { return m.nl_d; }
    static __device__ __forceinline__ int nl_c(const WbTc& m) { return m.nl_c; }
    static __device__ __forceinline__ int Kp(const WbTc& m, int l) { return m.Kp[l]; }
    static __device__ __forceinline__ int Np(const WbTc& m, int l) { return m.Np[l]; }
};
template <int... V> struct TcList {
    // 0 outside the list: the neighbour of the first / last layer, named only in branches that are dead for that layer
    static __host__ __device__ __forceinline__ constexpr int at(int i) { const int v[] = { V... }; return i >= 0 && i < (int)sizeof...(V) ? v[i] : 0; }
};
template <int ND, int NC, class KP, class NP>
struct TcShape {
    static constexpr bool fixed = true;
    static constexpr int kp0 = KP::at(0);
    static __device__ __forceinline__ int nl_d(const WbTc&) { return ND; }
    static __device__ __forceinline__ int nl_c(const WbTc&) { return NC; }
    static __device__ __forceinline__ int Kp(const WbTc&, int l) { return KP::at(l); }
    static __device__ __forceinline__ int Np(const WbTc&, int l) { return NP::at(l); }
    template <int L> static __device__ __forceinline__ TcInt<KP::at(L)> Kp(const WbTc&, TcInt<L>) { return {}; }
    template <int L> static __device__ __forceinline__ TcInt<NP::at(L)> Np(const WbTc&, TcInt<L>) { return {}; }
    template <bool REV, class F, int... L> static __device__ __forceinline__ void layers_(F& f, std::integer_sequence<int, L...>)
    {
        (f(TcInt<REV ? ND + NC - 1 - L : L>()), ...);
    }
    // f(TcInt<l>()) for every layer, first to last (REV: last to first)
    template <bool REV, class F> static __device__ __forceinline__ void layers(const WbTc&, F&& f)
    {
        layers_<REV>(f, std::make_integer_sequence<int, ND + NC>());
    }
    // the kernels of this shape run a decoder exactly when its geometry is this one (every other WbTc field stays a run-time value)
    static bool matches(const WbTc& m)
    {
        if (m.nl_d != ND || m.nl_c != NC) return false;
        for (int l = 0; l < ND + NC; ++l) if (m.Kp[l] != KP::at(l) || m.Np[l] != NP::at(l)) return false;
        return true;
    }
};
// app/nerf with 64-wide decoders and the 16-LOD F = 2 hash grid (bench.py's config 2): density 32 -> 64 -> 16, colour
// 15 + 27 (view embedding, 4 frequencies) -> 64 -> 64 -> 3
using TcShapeNerf64 = TcShape<2, 3, TcList<32, 64, 48, 64, 64>, TcList<64, 16, 64, 64, 16>>;

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
    // group and column half are broadcast from lane 0: ptxas then knows they are warp-uniform, and so is every branch and loop
    // bound derived from them (the tile loop, the per-half warp-collective scatter).  Without that it treats the wgmmas as issued
    // on a possibly divergent path and serializes every one of them (C7520).
    c.g = __shfl_sync(0xffffffffu, threadIdx.x / TC_GROUP, 0);
    c.sub = smem + c.g * m.group_bytes; c.blob = smem + m.w_smem_off;
    c.scr = reinterpret_cast<float*>(c.sub + m.scr_off);
    c.r = tig & (TC_ROWS - 1); c.h = __shfl_sync(0xffffffffu, tig / TC_ROWS, 0); c.wl = tig;
}
__device__ __forceinline__ void tc_sync(const TcCtx& c) { tc_group_sync(c.g + 1, TC_GROUP); }
// operand tiles written by the group's threads -> visible to the tensor cores of the whole group
__device__ __forceinline__ void tc_publish(const TcCtx& c) { tc_fence_smem_async(); tc_sync(c); }

// A round of the group: accumulators initialised (tc_acc_init), one fence, one or more chains issued (tc_issue), then
// tc_round_wait: commit, wait, group barrier (every MMA of the group has read its operands: the epilogues may overwrite them).
// Accumulator fragments D[64 x 2 NR] start from the bias (fp16, bias pack: entry n at half index 8n) or from +0.
template <int NR>
__device__ __forceinline__ void tc_acc_init(const TcCtx& c, float (&d)[NR], const __half* bias)
{
#pragma unroll
    for (int i = 0; i < NR; ++i) {
        if (bias) d[i] = __half2float(bias[tc_frag_col(c.wl, i) * 8]);
        else d[i] = tc_opaque_zero();
    }
}
// D += A . B over nk K-steps of 16, the descriptors advancing by aadv / badv (16-byte units) per step
template <int TA, int TB, int NR>
__device__ __forceinline__ void tc_issue(float (&d)[NR], uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv)
{
    for (int kb = 0; kb < nk; ++kb) { WgMma<2 * NR, TA, TB>::run(d, da, db, 1u); da += aadv; db += badv; }
}
template <class... D>
__device__ __forceinline__ void tc_round_wait(const TcCtx& c, D&... d)
{
    tc_wg_commit();
    tc_wg_wait0();
    (tc_wg_hold(d), ...);
    tc_sync(c);
}
// One round of a single chain D[64 x N] = bias or 0, += A . B; then epi(d) on the fragments.
template <int N, int TA, int TB, class Epi>
__device__ __forceinline__ void tc_chain(const TcCtx& c, uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv,
                                         const __half* bias, Epi&& epi)
{
    float d[N / 2];
    tc_acc_init(c, d, bias);
    tc_wg_fence();
    tc_issue<TA, TB>(d, da, db, nk, aadv, badv);
    tc_round_wait(c, d);
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
// N known at compile time (TcShape)
template <int TA, int TB, int NMAX = 128, int N, class Epi>
__device__ __forceinline__ void tc_chain_n(const TcCtx& c, TcInt<N>, uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv,
                                           const __half* bias, Epi&& epi)
{
    tc_chain<N, TA, TB>(c, da, db, nk, aadv, badv, bias, epi);
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
template <int NMAX, class S, class LT, class NT, class Epi>
__device__ __forceinline__ void tc_fwd_layer(const WbTc& m, const TcCtx& c, LT l, NT N, Epi&& epi)
{
    const uint32_t sb = tc_smem_u32(c.sub + m.tile_off[l]), wb = tc_smem_u32(c.blob);
    const int Np = S::Np(m, l);
    tc_chain_n<0, 0, NMAX>(c, N, tc_desc(sb, TC_SLAB, 128), tc_desc(wb + m.w_off[l], Np * 16, 128), S::Kp(m, l) / 16, (2 * TC_SLAB) >> 4,
                     (2 * Np * 16) >> 4, m.has_bias ? reinterpret_cast<const __half*>(c.blob + m.b_off[l]) : nullptr, epi);
}

// Decoders of one 64-sample sub-tile, starting from an X0 tile that the group has already written.
// Returns (per row, both column halves) the density-decoder output df[16] and the colour pre-activations c3[3].
template <int NMAX, class S>
__device__ __forceinline__ void tc_decoders(const WbTc& m, const TcCtx& c, const TcIn& in, int64_t ray, float df[16], float c3[3])
{
    const int nl = S::nl_d(m) + S::nl_c(m);
    if constexpr (S::fixed) {
        S::template layers<false>(m, [&](auto l) {
#define TC_NEXT_LAYER return
#include "wb_shade_tc_fwd_layer.cuh"
#undef TC_NEXT_LAYER
        });
    } else {
        for (int l = 0; l < nl; ++l) {
#define TC_NEXT_LAYER continue
#include "wb_shade_tc_fwd_layer.cuh"
#undef TC_NEXT_LAYER
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// forward kernel: CTA = TC_FWD_GROUPS groups, each walking its own 64-sample sub-tiles; several CTAs per SM overlap gather,
// MMA chains and epilogues
// ---------------------------------------------------------------------------------------------------------------
template <int MINB, bool GX, int NMAX, class S = TcShapeRt>   // MINB: resident CTAs per SM the register allocation is bounded for;
                                         // GX: triplanar / octree feature grid (wb_featx.cuh) instead of the hash grid; NMAX: widest
                                         // padded layer (64 or 128); S: decoder geometry
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
    const int nch0 = S::Kp(m, 0) / 8;
    const int64_t ntiles = (in.S + TC_ROWS - 1) / TC_ROWS;
    for (int64_t tile = (int64_t)blockIdx.x * TC_FWD_GROUPS + c.g; tile < ntiles; tile += (int64_t)gridDim.x * TC_FWD_GROUPS) {
        int64_t s = tile * TC_ROWS + c.r;
        const bool valid = s < in.S;
        if (!valid) s = in.S - 1;
        const int64_t ray = __ldg(in.rec_ray + s);
        const float3 p = wb_ray_point(in.origins, in.dirs, ray, __ldg(in.rec_t + s));
        // density-decoder input row: grid features (+ position embedding), zero padded to Kp; the two threads of a row split the LODs
        if (!GX) tile_gather(g, t0, c.r, c.h, p.x, p.y, p.z);
        else if (c.h == 0) {
            // one thread of the row pair gathers all LODs: the gather is latency-bound, splitting it over the pair costs a group
            // barrier and scratch traffic for partial sums of 'sum' grids
            wb_featx_gather(gx, p.x, p.y, p.z, [&](int f, float v) { tile_store1(t0, c.r, f, v); });
        }
        if (c.h == 0) {
            tile_embed(t0, c.r, m.feat_dim, m.pos_mode, m.pos_freq, p.x, p.y, p.z);
            tile_zero(t0, c.r, m.I[0], m.Kp[0]);
        }
        if (in.x0_save) {
            tc_sync(c);
            if (valid)
                for (int ch = c.h; ch < nch0; ch += 2) in.x0_save[(int64_t)ch * in.S + s] = *reinterpret_cast<const uint4*>(t0 + ch * TC_SLAB + c.r * 16);
        }
        float df[16], c3[3];
        tc_decoders<NMAX, S>(m, c, in, ray, df, c3);
        if (valid && c.h == 0) {
            const float r = 1.0f / (1.0f + expf(-c3[0])), gg = 1.0f / (1.0f + expf(-c3[1])), b = 1.0f / (1.0f + expf(-c3[2]));
            shaded[s] = make_float4(r, gg, b, fmaxf(df[0], 0.0f));
        }
    }
}

static int tc_launch_ray_embed(const WbTc& m, const wb_rays* rays, void* workspace, cudaStream_t st)
{
    const int64_t R = rays->num_rays;
    if (R == 0) return WB_OK;
    wb_ray_embed_kernel<<<(unsigned)((R + 127) / 128), 128, 0, st>>>(m, rays->dirs, R, reinterpret_cast<uint4*>(workspace));
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// the app/nerf decoder on the hash grid: the forward instance compiled for its geometry
static bool tc_fwd_nerf64(const WbTc& m, int grid_kind, int per_sm)
{
    return m.maxw <= 64 && grid_kind == 0 && per_sm == 3 && TcShapeNerf64::matches(m);
}

using TcFwdKernel = decltype(&wb_shade_fwd_tc_kernel<2, false, 64>);
// The forward instance of decoders m on grid kind `grid_kind` (the descriptor's, which wb_make_gridx copies into WbGridX::kind), and
// its CTAs per SM: more groups in flight hide the gather and chain latencies, and the register bound of the instance must match them,
// or the hardware silently runs fewer.  Decoders up to 64 wide: 2 or 3 CTAs (85 registers per thread); wider ones: 1 or 2 (a 128-wide
// accumulator is 64 registers).
static TcFwdKernel tc_fwd_kernel(const WbTc& m, int grid_kind, int& per_sm)
{
    const bool wide = m.maxw > 64, gx = grid_kind != 0;
    per_sm = max(1, min(3, TC_SMEM_MAX / (m.smem_bytes + 1024)));
    if (grid_kind == 2) per_sm = min(per_sm, 2);        // the octree gather keeps more state per thread (up to 32 accumulators)
    per_sm = wide ? min(per_sm, 2) : max(per_sm, 2);
    return tc_fwd_nerf64(m, grid_kind, per_sm) ? wb_shade_fwd_tc_kernel<3, false, 64, TcShapeNerf64>
         : wide ? (gx ? (per_sm == 2 ? wb_shade_fwd_tc_kernel<2, true, 128> : wb_shade_fwd_tc_kernel<1, true, 128>)
                      : (per_sm == 2 ? wb_shade_fwd_tc_kernel<2, false, 128> : wb_shade_fwd_tc_kernel<1, false, 128>))
                : (gx ? (per_sm == 3 ? wb_shade_fwd_tc_kernel<3, true, 64> : wb_shade_fwd_tc_kernel<2, true, 64>)
                      : (per_sm == 3 ? wb_shade_fwd_tc_kernel<3, false, 64> : wb_shade_fwd_tc_kernel<2, false, 64>));
}

int wb_tc_shade_fwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                    int64_t S, float* shaded, void* feat_save, void* workspace, cudaStream_t st)
{
    WbGrid g; int rc = wb_make_grid(nef, &g); if (rc) return rc;
    WbGridX gx; rc = wb_make_gridx(nef, false, &gx); if (rc) return rc;
    WbTc m; rc = wb_tc_make(nef, &m); if (rc) return rc;
    WB_CHECK_ARG(workspace != nullptr, "precision 1 needs the workspace (wb_rf_workspace_bytes)");
    rc = tc_launch_ray_embed(m, rays, workspace, st); if (rc) return rc;
    TcIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S, reinterpret_cast<const uint4*>(workspace), reinterpret_cast<uint4*>(feat_save), nullptr };
    int per_sm;
    const TcFwdKernel kern = tc_fwd_kernel(m, nef->grid_kind, per_sm);
    WB_CUDA(wb_allow_smem(kern, m.smem_bytes));
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

// Runs of consecutive lanes with equal keys: dist = lanes since the first lane of this lane's run, tail = last lane of its run.
// Returns the largest dist of the warp, the trip count of a segmented scan over the runs.  Warp-collective.
template <class K>
__device__ __forceinline__ int tc_warp_runs(K key, int lane, int& dist, bool& tail)
{
    const K kprev = __shfl_up_sync(0xffffffffu, key, 1);
    const bool head = (lane == 0) || (kprev != key);
    const uint32_t heads = __ballot_sync(0xffffffffu, head);
    const int run_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
    dist = lane - run_head;
    tail = (lane == 31) || ((heads >> (lane + 1)) & 1u);
    return __reduce_max_sync(0xffffffffu, dist);
}

// wb_corner_setup of sample position p on LOD l, plus the key of its cell (runs of lanes with the same key share the cell);
// invalid lanes get zero coefficients and a key that no other lane has
__device__ __forceinline__ uint64_t tc_scatter_setup(const WbGrid& g, int l, float3 p, bool valid, int lane, uint32_t idx[8], float cf[8])
{
    uint64_t key = ~0ull - (uint64_t)lane;
    if (valid) {
        int ix, iy, iz; float wx, wy, wz, jx, jy, jz;
        wb_cell(p.x, g.hres[l], g.hi[l], ix, wx, jx); wb_cell(p.y, g.hres[l], g.hi[l], iy, wy, jy); wb_cell(p.z, g.hres[l], g.hi[l], iz, wz, jz);
        key = (uint64_t)ix | ((uint64_t)iy << 20) | ((uint64_t)iz << 40);
        const float xy00 = jx * jy, xy01 = jx * wy, xy10 = wx * jy, xy11 = wx * wy;
        cf[0] = xy00 * jz; cf[1] = xy00 * wz; cf[2] = xy01 * jz; cf[3] = xy01 * wz;
        cf[4] = xy10 * jz; cf[5] = xy10 * wz; cf[6] = xy11 * jz; cf[7] = xy11 * wz;
        wb_corner_indices(g, l, ix, iy, iz, idx);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { idx[j] = 0; cf[j] = 0.0f; }
    }
    return key;
}

// One LOD of the hash-table scatter for the 32 consecutive samples of a warp (F == 2, hashgrid_interpolate_cuda.cu:151-160): runs of
// lanes in the same cell are summed with a segmented warp scan and only the last lane of a run issues the reductions.  Called by the
// decoder backward's last epilogue (dL/dfeat never leaves the SM) and by wb_table_scatter_kernel<2>.  s0, s1: this sample's (still
// loss-scaled) gradient of the LOD's two features.  Warp-collective: every lane of the warp calls it with the same `l`.
__device__ __forceinline__ void tc_scatter_level_f2(const WbGrid& g, int l, float3 p, bool valid, float s0, float s1,
                                                    float inv_scale, int lane, float* __restrict__ gtable)
{
    float* tb = gtable + g.begin[l] * 2;
    const bool pair_ok = (reinterpret_cast<uintptr_t>(tb) & 15u) == 0;       // level base 16-byte aligned
    uint32_t idx[8]; float cf[8];
    const uint64_t key = tc_scatter_setup(g, l, p, valid, lane, idx, cf);
    int dist; bool tail;
    const int maxd = tc_warp_runs(key, lane, dist, tail);
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
        // corners j and j + 4 are x-neighbours at the same (y, z).  When their entries differ only in bit 0 (dense level with an even
        // index; hashed level with an even x, because (x | 1) ^ A == (x ^ A) ^ 1) the two 8-byte updates are one aligned 16-byte
        // red.global.add.v4.f32
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

// One backward round of a layer, for the 64 output rows of the weight gradient whose dY^T slabs `dyw` addresses: the weight-grad
// chain acc^T[64 x NK] += dY^T . X (wg), the bias-grad chain acc^T[64 x 8] += dY^T . [1 | 0] from the constant-one slab `xone`
// (wg && bg) and the data-grad chain dX[64 x ND] = dY . W over nkd K-steps (dg) go out as one commit group, so their MMAs overlap;
// then one wait, one group barrier and the epilogues in that order.  NK: the layer's padded input width; ND: NK, or 16 for the
// first colour layer.
template <int NK, int ND, class WEpi, class BEpi, class DEpi>
__device__ __forceinline__ void tc_bwd_round(const TcCtx& c, bool wg, bool bg, bool dg, uint64_t dyw, uint64_t xw, uint64_t xone,
                                             uint64_t dyd, uint64_t wd, int nkd, WEpi&& wepi, BEpi&& bepi, DEpi&& depi)
{
    float aw[NK / 2], ab[4], ad[ND / 2];
    tc_acc_init(c, aw, nullptr); tc_acc_init(c, ab, nullptr); tc_acc_init(c, ad, nullptr);
    tc_wg_fence();
    if (wg) {
        tc_issue<1, 1>(aw, dyw, xw, TC_ROWS / 16, 256 >> 4, 256 >> 4);           // K = the 64 samples, both operands MN-major
        if (bg) tc_issue<1, 1>(ab, dyw, xone, TC_ROWS / 16, 256 >> 4, 256 >> 4);
    }
    if (dg) tc_issue<0, 1>(ad, dyd, wd, nkd, (2 * TC_SLAB) >> 4, 256 >> 4);       // weight pack read MN-major: no transposed copy
    tc_round_wait(c, aw, ab, ad);
    if (wg) { wepi(aw); if (bg) bepi(ab); }
    if (dg) depi(ad);
}
// the same chains as one round each: inputs wider than 64, where the accumulators of a merged round (up to 132 per thread) no
// longer fit the registers beside the rest of the kernel
template <int NK, int ND, class WEpi, class BEpi, class DEpi>
__device__ __forceinline__ void tc_bwd_rounds_seq(const TcCtx& c, bool wg, bool bg, bool dg, uint64_t dyw, uint64_t xw, uint64_t xone,
                                                  uint64_t dyd, uint64_t wd, int nkd, WEpi&& wepi, BEpi&& bepi, DEpi&& depi)
{
    if (wg) {
        tc_chain<NK, 1, 1>(c, dyw, xw, TC_ROWS / 16, 256 >> 4, 256 >> 4, nullptr, wepi);
        if (bg) tc_chain<8, 1, 1>(c, dyw, xone, TC_ROWS / 16, 256 >> 4, 256 >> 4, nullptr, bepi);
    }
    if (dg) tc_chain<ND, 0, 1>(c, dyd, wd, nkd, (2 * TC_SLAB) >> 4, 256 >> 4, nullptr, depi);
}
// the round(s) with NK = Kp chosen at run time (a multiple of 16, at most 128); D16: the data grad is 16 wide
template <bool D16, class... A>
__device__ __forceinline__ void tc_bwd_round_n(int Kp, A&&... a)
{
    switch (Kp) {
        case 16: tc_bwd_round<16, 16>(a...); break;
        case 32: tc_bwd_round<32, D16 ? 16 : 32>(a...); break;
        case 48: tc_bwd_round<48, D16 ? 16 : 48>(a...); break;
        case 64: tc_bwd_round<64, D16 ? 16 : 64>(a...); break;
        case 80: tc_bwd_rounds_seq<80, D16 ? 16 : 80>(a...); break;
        case 96: tc_bwd_rounds_seq<96, D16 ? 16 : 96>(a...); break;
        case 112: tc_bwd_rounds_seq<112, D16 ? 16 : 112>(a...); break;
        default: tc_bwd_rounds_seq<128, D16 ? 16 : 128>(a...); break;
    }
}
// Kp known at compile time (TcShape): the case of the switch above
template <bool D16, int K, class... A>
__device__ __forceinline__ void tc_bwd_round_n(TcInt<K>, A&&... a)
{
    if constexpr (K <= 64) tc_bwd_round<K, D16 ? 16 : K>(a...);
    else tc_bwd_rounds_seq<K, D16 ? 16 : K>(a...);
}

// wmask: layers whose weight gradients this launch accumulates; emit: this launch produces dL/dfeat (planes, or FUSE: the hash-table
// scatter of an F == 2 'cat' grid in the last epilogue).  Wide decoders whose accumulators do not all fit run several launches.
// S: decoder geometry.
template <int NG, bool FUSE, class S = TcShapeRt>
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
    // TcShape instances load the next tile's saved rows, ray index and incoming gradient while this tile runs, so that their latency
    // is spent under this tile's rounds and table scatter instead of at the start of the next tile (app/nerf: shade_bwd 16.3 -> 15.7 ms
    // on H100, DESIGN.md section 4).  PF: saved-row chunks per thread (the two threads of a row split them); 0 for the run-time shape,
    // which loads at the start of each tile.
    constexpr int PF = S::kp0 / 16;
    uint4 xr_n[PF > 0 ? PF : 1];
    int64_t ray_n = 0;
    float4 go_n = make_float4(0, 0, 0, 0);
    auto fetch = [&](int64_t t) {
        int64_t sn = t * TC_ROWS + c.r;
        const bool vn = sn < s_end;
        if (!vn) sn = s_end - 1;
        ray_n = __ldg(in.rec_ray + sn);
#pragma unroll
        for (int i = 0; i < PF; ++i) xr_n[i] = __ldg(in.x0_saved + (int64_t)(c.h + 2 * i) * in.S + sn);
        go_n = vn ? __ldg(g_shaded + sn) : make_float4(0, 0, 0, 0);
    };
    const int64_t tile_first = tile0 + (int64_t)blockIdx.x * NG + c.g, tile_step = (int64_t)gridDim.x * NG;
    if constexpr (PF > 0) { if (tile_first < ntiles) fetch(tile_first); }
    for (int64_t tile = tile_first; tile < ntiles; tile += tile_step) {
        int64_t s = tile * TC_ROWS + c.r;
        const bool valid = s < s_end;
        if (!valid) s = s_end - 1;
        float df[16], c3[3];
        int64_t ray;
        float4 go;
        if constexpr (PF > 0) {
            ray = ray_n;
            go = go_n;
#pragma unroll
            for (int i = 0; i < PF; ++i) *reinterpret_cast<uint4*>(t0 + (c.h + 2 * i) * TC_SLAB + c.r * 16) = xr_n[i];
            if (tile + tile_step < ntiles) fetch(tile + tile_step);
            tc_decoders<128, S>(m, c, in, ray, df, c3);
        } else {
            ray = __ldg(in.rec_ray + s);
            for (int ch = c.h; ch < nch0; ch += 2)                 // saved density-decoder input row (coalesced 16 B per lane)
                *reinterpret_cast<uint4*>(t0 + ch * TC_SLAB + c.r * 16) = __ldg(in.x0_saved + (int64_t)ch * in.S + s);
            tc_decoders<128, S>(m, c, in, ray, df, c3);
            go = valid ? __ldg(g_shaded + s) : make_float4(0, 0, 0, 0);
        }
        // ---- colour decoder, last layer: dY = dL/d(pre-sigmoid), zero padded ----
        if (c.h == 0) {
            const float r = 1.0f / (1.0f + expf(-c3[0])), gg = 1.0f / (1.0f + expf(-c3[1])), b = 1.0f / (1.0f + expf(-c3[2]));
            float v[8] = { go.x * r * (1.0f - r) * scale, go.y * gg * (1.0f - gg) * scale, go.z * b * (1.0f - b) * scale, 0, 0, 0, 0, 0 };
            tile_store8(dyt, c.r, 0, v);
        }
        for (int sl = 1 + c.h; sl < m.Np[nl - 1] / 8; sl += 2) tile_store8(dyt, c.r, sl, z8);
        if constexpr (S::fixed) {
            S::template layers<true>(m, [&](auto l) {
#define TC_END_LAYERS return
#include "wb_shade_tc_bwd_layer.cuh"
#undef TC_END_LAYERS
            });
        } else {
            for (int l = nl - 1; l >= 0; --l) {
#define TC_END_LAYERS break
#include "wb_shade_tc_bwd_layer.cuh"
#undef TC_END_LAYERS
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
constexpr int TC_SCATTER_LODS = 16;           // LODs per CTA row: they share the sample position and the record loads
constexpr int TC_SCATTER_CTAS_PER_SM = 16;
template <int F>      // 2: the F == 2 'cat' / 'sum' grids through tc_scatter_level_f2; 0: any feature width
__global__ void __launch_bounds__(256)
wb_table_scatter_kernel(WbGrid g, TcIn in, const __half* __restrict__ dfeat, int levels, const float* __restrict__ scale_p,
                        float* __restrict__ gtable)
{
    const int l_begin = blockIdx.y * TC_SCATTER_LODS, l_end = min(levels, l_begin + TC_SCATTER_LODS);   // this CTA's LODs
    const int lane = threadIdx.x & 31;
    const float inv_scale = 1.0f / __ldg(scale_p);
    const int64_t s_end = in.s_end ? in.s_end : in.S;
    const int64_t nwork = in.s_begin + ((s_end - in.s_begin + 31) & ~(int64_t)31);            // whole warps
    for (int64_t s = in.s_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nwork; s += (int64_t)gridDim.x * blockDim.x) {
        const bool valid = s < s_end;
        const float3 p = valid ? wb_sample_pos(in.origins, in.dirs, in.rec_ray, in.rec_t, s) : make_float3(0.0f, 0.0f, 0.0f);
        if constexpr (F == 2) {
            const __half2* gs = reinterpret_cast<const __half2*>(dfeat) + s;
            __half2 gnext = __float2half2_rn(0.0f);              // the next LOD's gradient is fetched one LOD ahead
            if (valid && l_begin < l_end) gnext = gs[(int64_t)(g.multiscale == 0 ? l_begin : 0) * in.S];
            for (int l = l_begin; l < l_end; ++l) {
                const float2 gl = __half22float2(gnext);
                if (valid && l + 1 < l_end) gnext = gs[(int64_t)(g.multiscale == 0 ? l + 1 : 0) * in.S];
                tc_scatter_level_f2(g, l, p, valid, gl.x, gl.y, inv_scale, lane, gtable);
            }
        } else {
            for (int l = l_begin; l < l_end; ++l) {
                const int pl = g.multiscale == 0 ? l : 0;
                float* tb = gtable + g.begin[l] * g.F;
                uint32_t idx[8]; float cf[8];
                const uint64_t key = tc_scatter_setup(g, l, p, valid, lane, idx, cf);
                int dist; bool tail;
                const int maxd = tc_warp_runs(key, lane, dist, tail);
                for (int f = 0; f < g.F; ++f) {
                    const float gv = valid ? __half2float(dfeat[((int64_t)pl * in.S + s) * g.F + f]) * inv_scale : 0.0f;
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = gv * cf[j];
                    for (int o = 1; o <= maxd; o <<= 1) {               // segmented inclusive scan (warp-uniform trip count)
#pragma unroll
                        for (int j = 0; j < 8; ++j) { const float a = __shfl_up_sync(0xffffffffu, v[j], o); if (dist >= o) v[j] += a; }
                    }
                    if (tail && valid) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) if (v[j] != 0.0f) atomicAdd(tb + (int64_t)idx[j] * g.F + f, v[j]);
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
        const float3 pos = valid ? wb_sample_pos(in.origins, in.dirs, in.rec_ray, in.rec_t, s) : make_float3(0.0f, 0.0f, 0.0f);
        auto grad = [&](int f) {                                  // feature f lives in plane f / width at column f % width
            return __half2float(dfeat[((int64_t)(f / width) * in.S + s) * width + (f % width)]) * inv_scale;
        };
        if (gx.kind != 1 || gx.C > 4) {                           // octree grid (or wide triplanar channels): no merging
            if (valid) wb_featx_scatter(gx, pos.x, pos.y, pos.z, grad);
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
                WbBilinear b = wb_tp_setup(pos.x, pos.y, pos.z, p, size);
                float v[4][4];                                    // [texel nw, ne, sw, se][channel]
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float g = gx.sum ? gsum[p][c] : ((valid && c < C) ? grad((l * 3 + p) * C + c) : 0.0f);
                    v[0][c] = g * b.nw; v[1][c] = g * b.ne; v[2][c] = g * b.sw; v[3][c] = g * b.se;
                }
                int dist; bool tail;
                const int maxd = tc_warp_runs(valid ? b.o00 : -1 - lane, lane, dist, tail);     // invalid lanes never merge
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

using TcBwdKernel = decltype(&wb_mlp_bwd_tc_kernel<1, false>);
// pass p's instance, and `fuse`: it runs the table scatter (the last pass, where the plan fuses, given a table gradient)
static TcBwdKernel tc_bwd_kernel(const WbTc& m, const TcBwdPlan& b, int p, bool table, bool& fuse)
{
    fuse = table && p == b.npass - 1 && b.fuses;
    if (fuse && TcShapeNerf64::matches(m)) return wb_mlp_bwd_tc_kernel<2, true, TcShapeNerf64>;       // compiled for its geometry
    return b.groups[p] == 2 ? (fuse ? wb_mlp_bwd_tc_kernel<2, true> : wb_mlp_bwd_tc_kernel<2, false>) : wb_mlp_bwd_tc_kernel<1, false>;
}

// decoder backward: dL/d(shaded) -> weight gradients + dL/dfeat planes in the workspace (or, fused, the hash-table scatter)
int wb_tc_decoder_bwd_ex(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                         int64_t S, int64_t s_begin, int64_t s_end, const float* g_shaded, const float* scale, const void* feat_saved,
                         void* workspace, bool ray_rows_ready, float* grad_dens, float* grad_col, float* grad_table, int* fused_out,
                         cudaStream_t st)
{
    if (fused_out) *fused_out = 0;
    WbTc m; TcBwdPlan plan; int rc = wb_tc_make(nef, &m, &plan); if (rc) return rc;
    WB_CHECK_ARG(scale != nullptr, "precision 1 needs the device loss-scale pointer");
    WB_CHECK_ARG(feat_saved != nullptr && workspace != nullptr, "precision 1 backward needs the saved features and the workspace");
    if (!ray_rows_ready) { rc = tc_launch_ray_embed(m, rays, workspace, st); if (rc) return rc; }
    const TcDfeat df = tc_dfeat(nef, m, rays->num_rays);
    TcIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S, reinterpret_cast<const uint4*>(workspace), nullptr, reinterpret_cast<const uint4*>(feat_saved),
                s_begin, s_end };
    if (s_end <= s_begin) return WB_OK;
    TcGrads G = { grad_dens, grad_col, scale, reinterpret_cast<__half*>(static_cast<uint8_t*>(workspace) + df.off), df.planes, df.width };
    for (int p = 0; p < plan.npass; ++p) {
        const WbTc mp = tc_bwd_pass(m, plan, p);
        bool fuse;
        const TcBwdKernel kern = tc_bwd_kernel(m, plan, p, grad_table != nullptr, fuse);
        WbGrid g; memset(&g, 0, sizeof(g));
        if (fuse) { rc = wb_make_grid(nef, &g); if (rc) return rc; }
        WB_CUDA(wb_allow_smem(kern, TC_SMEM_MAX));         // the passes of one call differ in size: allow the largest once
        const int64_t nctas = ((s_end - s_begin + s_begin % TC_ROWS + TC_ROWS - 1) / TC_ROWS + mp.groups - 1) / mp.groups;
        int64_t grid = (int64_t)wb_num_sms(); if (grid > nctas) grid = nctas;         // 1 CTA / SM: shared memory holds the tiles and accumulators
        kern<<<(unsigned)grid, mp.groups * TC_GROUP, mp.smem_bytes, st>>>(mp, reinterpret_cast<const uint8_t*>(blob), in, reinterpret_cast<const float4*>(g_shaded),
                                                                          G, plan.mask[p], p == plan.npass - 1 ? 1 : 0, g, grad_table);
        WB_LAUNCH_CHECK();
        if (fuse && fused_out) *fused_out = 1;
    }
    return WB_OK;
}

// table scatter only: dL/dfeat planes (written by wb_tc_decoder_bwd_ex into the same workspace) -> grad_table.  The triplanar / octree
// scatter always takes the whole range.
int wb_tc_table_scatter(const wb_nef_desc* nef, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray, int64_t S,
                        int64_t s_begin, int64_t s_end, const float* scale, void* workspace, float* grad_table, cudaStream_t st)
{
    WbGrid g; int rc = wb_make_grid(nef, &g); if (rc) return rc;
    WbGridX gx; rc = wb_make_gridx(nef, true, &gx); if (rc) return rc;
    // refuse the decoders whose backward does not fit: no decoder backward wrote their planes
    WbTc m; TcBwdPlan plan; rc = wb_tc_make(nef, &m, &plan); if (rc) return rc;
    WB_CHECK_ARG(scale != nullptr && workspace != nullptr && (grad_table != nullptr || gx.kind != 0), "null pointer");
    const TcDfeat df = tc_dfeat(nef, m, rays->num_rays);
    const __half* dfeat = reinterpret_cast<const __half*>(static_cast<const uint8_t*>(workspace) + df.off);
    TcIn in = { rays->origins, rays->dirs, rec_t, rec_ray, S, nullptr, nullptr, nullptr, s_begin, s_end };
    if (gx.kind != 0) {
        int64_t bx = (S + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * 16; if (bx > cap) bx = cap;
        wb_featx_scatter_kernel<<<(unsigned)bx, 256, 0, st>>>(gx, in, dfeat, df.width, scale);
        WB_LAUNCH_CHECK();
        return WB_OK;
    }
    const int levels = g.multiscale == 0 ? df.planes : g.L;
    if (levels > 0 && s_end > s_begin) {
        int64_t bx = (s_end - s_begin + 255) / 256; const int64_t cap = (int64_t)wb_num_sms() * TC_SCATTER_CTAS_PER_SM; if (bx > cap) bx = cap;
        dim3 grid2((unsigned)bx, (unsigned)((levels + TC_SCATTER_LODS - 1) / TC_SCATTER_LODS));
        if (g.F == 2) wb_table_scatter_kernel<2><<<grid2, 256, 0, st>>>(g, in, dfeat, levels, scale, grad_table);
        else wb_table_scatter_kernel<0><<<grid2, 256, 0, st>>>(g, in, dfeat, levels, scale, grad_table);
        WB_LAUNCH_CHECK();
    }
    return WB_OK;
}

// *shaped = 1 when the forward (backward == 0) or the decoder backward with the fused table scatter (backward == 1) of this decoder
// runs an instance compiled for its geometry (the launches' own choice: tc_fwd_kernel, tc_bwd_kernel); 0 when it runs a run-time one
int wb_tc_shaped(const wb_nef_desc* nef, int backward, int* shaped)
{
    WB_CHECK_ARG(shaped != nullptr, "null pointer");
    *shaped = 0;
    WbTc m; TcBwdPlan plan; int rc = wb_tc_make(nef, &m, backward ? &plan : nullptr); if (rc) return rc;
    int per_sm; bool fuse;
    if (!backward) *shaped = tc_fwd_kernel(m, nef->grid_kind, per_sm) ==wb_shade_fwd_tc_kernel<3, false, 64, TcShapeNerf64>;
    else *shaped = tc_bwd_kernel(m, plan, plan.npass - 1, true, fuse) == wb_mlp_bwd_tc_kernel<2, true, TcShapeNerf64>;
    return WB_OK;
}

// Wide decoders (one 256-thread group per SM, half the register file and all the other warp slots idle): from TC_CHUNKED_MIN_S samples
// on (below, the schedule is not worth its launches) the sample range is cut into TC_CHUNKS chunks; the decoder backward of chunk c+1
// runs on the caller's stream while the table scatter of chunk c (an issue-bound SIMT kernel with 48 registers per thread and no shared
// memory: two of its CTAs fit beside a decoder CTA) runs on a side stream.
constexpr int64_t TC_CHUNKED_MIN_S = 1 << 20;
constexpr int TC_CHUNKS = 4;
// One side stream and one set of fork / join events per device, shared by every caller on that device.  `mu` is held from the creation
// check to the end of a call's enqueue loop: an event recorded by one thread must not be re-recorded by another before this thread's
// cudaStreamWaitEvent has captured it, or a scatter would wait for another caller's decoder chunk instead of its own.
struct TcSide { std::mutex mu; cudaStream_t stream; cudaEvent_t ev[TC_CHUNKS + 1]; bool ok; };      // one event per chunk + the join
static TcSide* tc_side_stream_locked(TcSide& s)
{
    if (!s.ok) {
        if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
        for (int i = 0; i <= TC_CHUNKS; ++i) if (cudaEventCreateWithFlags(&s.ev[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
        s.ok = true;
    }
    return &s;
}
static TcSide* tc_side_slot()
{
    static TcSide side[64];
    int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    return &side[dev];
}

int wb_tc_shade_bwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                    int64_t S, const float* g_shaded, const float* scale, const void* feat_saved, void* workspace, bool ray_rows_ready,
                    float* grad_table, float* grad_dens, float* grad_col, cudaStream_t st)
{
    // one group per SM in the first pass (wide decoders): the decoder backward leaves most warp slots idle
    WbTc m; TcBwdPlan plan;
    bool wide = S >= TC_CHUNKED_MIN_S && nef->grid_kind == 0 && grad_table && wb_tc_make(nef, &m, &plan) == WB_OK && plan.groups[0] == 1;
    // A call being captured into a graph runs the one-stream schedule (the same sums up to the order of the atomic additions): the
    // shared side stream would otherwise join the capture, and another thread's eager call on it would be mixed into the graph.
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (wide && cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap != cudaStreamCaptureStatusNone) wide = false;
    if (TcSide* slot = wide ? tc_side_slot() : nullptr) {
        std::lock_guard<std::mutex> lock(slot->mu);
        if (TcSide* side = tc_side_stream_locked(*slot)) {
            const int64_t per = ((S + TC_CHUNKS - 1) / TC_CHUNKS + TC_ROWS - 1) / TC_ROWS * TC_ROWS;
            int rc = WB_OK, c = 0;
            for (int64_t s0 = 0; s0 < S && rc == WB_OK; s0 += per, ++c) {
                const int64_t s1 = s0 + per < S ? s0 + per : S;
                // the per-ray rows are written by the first chunk's launch
                rc = wb_tc_decoder_bwd_ex(nef, blob, rays, rec_t, rec_ray, S, s0, s1, g_shaded, scale, feat_saved, workspace, ray_rows_ready || c > 0,
                                          grad_dens, grad_col, nullptr, nullptr, st);
                if (rc == WB_OK && (cudaEventRecord(side->ev[c], st) != cudaSuccess || cudaStreamWaitEvent(side->stream, side->ev[c], 0) != cudaSuccess)) rc = WB_ERR_CUDA;
                if (rc == WB_OK) rc = wb_tc_table_scatter(nef, rays, rec_t, rec_ray, S, s0, s1, scale, workspace, grad_table, side->stream);
            }
            // the caller's stream continues after the last scatter (also on an error path: never leave the side stream unjoined)
            if (cudaEventRecord(side->ev[TC_CHUNKS], side->stream) != cudaSuccess || cudaStreamWaitEvent(st, side->ev[TC_CHUNKS], 0) != cudaSuccess) { if (rc == WB_OK) rc = WB_ERR_CUDA; }
            return rc;
        }
    }
    int fused = 0;
    int rc = wb_tc_decoder_bwd_ex(nef, blob, rays, rec_t, rec_ray, S, 0, S, g_shaded, scale, feat_saved, workspace, ray_rows_ready, grad_dens, grad_col,
                                  grad_table, &fused, st);
    if (rc || fused) return rc;
    return wb_tc_table_scatter(nef, rays, rec_t, rec_ray, S, 0, S, scale, workspace, grad_table, st);
}
