// wb_sdf.cuh -- the NeuralSDF(OctreeGrid | HashGrid) field shared by wb_sdf.cu (evaluation, sphere tracing) and wb_sdf_train.cu
// (training step): host-side description, the decoder's shared-memory image, the position embedding and the octree and hash-grid
// feature gathers.
#pragma once
#include "wb_common.cuh"

constexpr int WB_SDF_MAX_IN = 132;        // 3 + 6*freq position embedding + features
constexpr int WB_SDF_MAX_H = 128;
constexpr int WB_SDF_THREADS = 256;

struct WbSdf {
    // octree grid
    const int16_t* points; const int32_t* trinkets;
    const float* feats[WB_MAX_LODS];
    int F, base_lod, num_lods, multiscale, half_round;
    // decoder
    int pos_mode, pos_freq, pos_dim, feat_dim, in_dim, in_pad, H, nh;      // nh hidden layers (>= 1), all H wide
    const float* params;                                                     // packed [W0, b0, W1, b1, ..., Wout, bout] (nn.Linear layout)
    int smem_floats;
};

static inline int sdf_embed_dim(int mode, int freq) { return mode == 0 ? 0 : mode == 1 ? 3 : mode == 2 ? 6 * freq : 3 + 6 * freq; }

// hg: the hash grid of a hash field (d->hash != NULL), validated by wb_make_grid; hg->table == nullptr for an octree field
static inline int wb_make_sdf(const wb_sdf_desc* d, WbSdf* m, WbGrid* hg)
{
    memset(hg, 0, sizeof(*hg));
    WB_CHECK_ARG(d != nullptr && d->params && (d->hash || (d->points && d->trinkets && d->feats)), "null pointer in wb_sdf_desc");
    if (d->hash) {
        const int rc = wb_make_grid(d->hash, hg); if (rc) return rc;
        WB_CHECK_ARG(d->hash->grid_kind == 0 && (hg->F == 4 || hg->F == 8), "hash field: a hash grid of 4 or 8 features per LOD");
        WB_CHECK_ARG((reinterpret_cast<uintptr_t>(hg->table) & 15u) == 0, "hash field: the table must be 16-byte aligned");
        WB_CHECK_ARG(d->feature_dim == hg->F && d->num_lods == hg->L && d->multiscale == hg->multiscale && d->base_lod == 0,
                     "hash field: feature_dim / num_lods / multiscale differ from the hash description");
    }
    WB_CHECK_ARG(d->num_lods >= 1 && d->num_lods <= WB_MAX_LODS && d->base_lod >= 0, "bad LOD range");
    WB_CHECK_ARG(d->feature_dim >= 1 && d->feature_dim <= 64, "feature_dim must be in [1,64]");
    WB_CHECK_ARG(d->multiscale == 0 || d->multiscale == 1, "multiscale must be 0 ('cat') or 1 ('sum')");
    WB_CHECK_ARG(d->num_layers >= 1 && d->num_layers <= 4 && d->hidden_dim >= 1 && d->hidden_dim <= WB_SDF_MAX_H, "decoder: 1..4 hidden layers, <= 128 wide");
    WB_CHECK_ARG(d->pos_mode >= 0 && d->pos_mode <= 3 && d->pos_freq >= 0 && d->pos_freq <= 10, "bad position embedding");
    memset(m, 0, sizeof(*m));
    if (!d->hash) {
        m->points = d->points; m->trinkets = d->trinkets;
        for (int k = 0; k < d->num_lods; ++k) { WB_CHECK_ARG(d->feats[k] != nullptr, "null feature level"); m->feats[k] = d->feats[k]; }
        m->half_round = d->half_round;
    }
    m->F = d->feature_dim; m->base_lod = d->base_lod; m->num_lods = d->num_lods; m->multiscale = d->multiscale;
    m->pos_mode = d->pos_mode; m->pos_freq = d->pos_freq; m->pos_dim = sdf_embed_dim(d->pos_mode, d->pos_freq);
    m->feat_dim = d->multiscale ? d->feature_dim : d->feature_dim * d->num_lods;
    m->in_dim = m->pos_dim + m->feat_dim; m->in_pad = (m->in_dim + 3) & ~3;
    WB_CHECK_ARG(m->in_dim <= WB_SDF_MAX_IN, "decoder input too wide");
    m->H = d->hidden_dim; m->nh = d->num_layers; m->params = d->params;
    WB_CHECK_ARG(m->nh == 1 || (m->H % 4) == 0, "hidden_dim must be a multiple of 4 for multi-layer decoders");
    m->smem_floats = m->H * m->in_pad + m->H + (m->nh - 1) * (m->H * m->H + m->H) + m->H + 4;
    WB_CHECK_ARG(m->smem_floats * 4 <= 200 * 1024, "decoder does not fit in shared memory");
    return WB_OK;
}

// shared-memory image: W0 rows padded to in_pad floats | b0 | (W_k [H x H] | b_k) ... | Wout [H] | bout
__device__ __forceinline__ void sdf_stage(const WbSdf& m, float* sw)
{
    const float* p = m.params;
    int o = 0, src = 0;
    for (int e = threadIdx.x; e < m.H * m.in_pad; e += blockDim.x) {
        const int j = e / m.in_pad, k = e - j * m.in_pad;
        sw[e] = k < m.in_dim ? __ldg(p + j * m.in_dim + k) : 0.0f;
    }
    o += m.H * m.in_pad; src += m.H * m.in_dim;
    for (int e = threadIdx.x; e < m.H; e += blockDim.x) sw[o + e] = __ldg(p + src + e);
    o += m.H; src += m.H;
    for (int l = 1; l < m.nh; ++l) {
        for (int e = threadIdx.x; e < m.H * m.H + m.H; e += blockDim.x) sw[o + e] = __ldg(p + src + e);
        o += m.H * m.H + m.H; src += m.H * m.H + m.H;
    }
    for (int e = threadIdx.x; e < m.H + 1; e += blockDim.x) sw[o + e] = __ldg(p + src + e);
    __syncthreads();
}

__device__ __forceinline__ float sdf_h(float v) { return __half2float(__float2half_rn(v)); }

// positional_embedder.py:51-66 / neural_sdf.py:86-99: [x (include_input), sin(winded), cos(winded)], winded freq-major coord-minor
__device__ __forceinline__ int sdf_embed(int mode, int freq, float x, float y, float z, float* out)
{
    if (mode == 0) return 0;
    int o = 0;
    if (mode == 1 || mode == 3) { out[0] = x; out[1] = y; out[2] = z; o = 3; }
    if (mode == 1) return 3;
    float band = 1.0f;
    for (int f = 0; f < freq; ++f) {
        out[o + f * 3 + 0] = sinf(x * band); out[o + f * 3 + 1] = sinf(y * band); out[o + f * 3 + 2] = sinf(z * band);
        out[o + 3 * freq + f * 3 + 0] = cosf(x * band); out[o + 3 * freq + f * 3 + 1] = cosf(y * band); out[o + 3 * freq + f * 3 + 2] = cosf(z * band);
        band *= 2.0f;
    }
    return o + 6 * freq;
}

// OctreeGrid.interpolate for LODs 0..nl-1 of one point -> feat[] (zeros where the point leaves the octree); FT > 0: compile-time
// feature width of a 'sum' grid (accumulators in registers)
template <int FT>
__device__ __forceinline__ void sdf_features(const WbOct& oc, const WbSdf& m, int nl, float cx, float cy, float cz, float* feat)
{
    const int F = FT > 0 ? FT : m.F;
    const bool sum = FT > 0 ? true : (m.multiscale != 0 && nl > 1);         // lod_idx == 0: a single LOD either way (octree_grid.py:190-198)
    const int width = sum ? F : nl * F;
#pragma unroll
    for (int f = 0; f < (FT > 0 ? FT : 1); ++f) feat[f] = 0.0f;
    if (FT == 0) for (int f = 0; f < width; ++f) feat[f] = 0.0f;
    const int L = m.base_lod + nl - 1;                                       // level of the finest LOD used
    const float h = ldexpf(1.0f, L - 1), inv_h = ldexpf(1.0f, -(L - 1)), maxq = (float)((1 << L) - 1);
    int qx, qy, qz;
    if (!(wb_quantize(cx, h, inv_h, maxq, qx) && wb_quantize(cy, h, inv_h, maxq, qy) && wb_quantize(cz, h, inv_h, maxq, qz))) return;
    int node = 0;
    for (int l = 0; l <= L; ++l) {
        if (l > 0) {
            const int d = L - l;
            const int ci = (((qx >> d) & 1) << 2) | (((qy >> d) & 1) << 1) | ((qz >> d) & 1);
            const uint32_t b = __ldg(oc.octree + node);
            if (!(b & (1u << ci))) return;
            node = __ldg(oc.prefix + node) + __popc(b & ((2u << ci) - 1u));
        }
        const int k = l - m.base_lod;
        if (k < 0) continue;
        const float hl = ldexpf(1.0f, l - 1);
        const float ux = __fmaf_rn(cx, hl, hl) - (float)__ldg(m.points + 3 * (int64_t)node);
        const float uy = __fmaf_rn(cy, hl, hl) - (float)__ldg(m.points + 3 * (int64_t)node + 1);
        const float uz = __fmaf_rn(cz, hl, hl) - (float)__ldg(m.points + 3 * (int64_t)node + 2);
        const float ix = 1.0f - ux, iy = 1.0f - uy, iz = 1.0f - uz;
        float cf[8];
        cf[0] = (ix * iy) * iz; cf[1] = (ix * iy) * uz; cf[2] = (ix * uy) * iz; cf[3] = (ix * uy) * uz;
        cf[4] = (ux * iy) * iz; cf[5] = (ux * iy) * uz; cf[6] = (ux * uy) * iz; cf[7] = (ux * uy) * uz;
        const int4 t0 = __ldg(reinterpret_cast<const int4*>(m.trinkets + 8 * (int64_t)node));
        const int4 t1 = __ldg(reinterpret_cast<const int4*>(m.trinkets + 8 * (int64_t)node) + 1);
        const int tk[8] = { t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w };
        const float* ft = m.feats[k];
        if (FT > 0 && (FT % 4) == 0) {
            float acc[FT > 0 ? FT : 1];
#pragma unroll
            for (int f = 0; f < FT; ++f) acc[f] = 0.0f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4* row = reinterpret_cast<const float4*>(ft + (int64_t)tk[j] * FT);
#pragma unroll
                for (int q = 0; q < FT / 4; ++q) {
                    float4 v = __ldg(row + q);
                    if (m.half_round) { v.x = sdf_h(v.x); v.y = sdf_h(v.y); v.z = sdf_h(v.z); v.w = sdf_h(v.w); }
                    acc[4 * q] = fmaf(v.x, cf[j], acc[4 * q]); acc[4 * q + 1] = fmaf(v.y, cf[j], acc[4 * q + 1]);
                    acc[4 * q + 2] = fmaf(v.z, cf[j], acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v.w, cf[j], acc[4 * q + 3]);
                }
            }
#pragma unroll
            for (int f = 0; f < FT; ++f) feat[f] += m.half_round ? sdf_h(acc[f]) : acc[f];
        } else {
            for (int f = 0; f < F; ++f) {
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float v = __ldg(ft + (int64_t)tk[j] * F + f);
                    if (m.half_round) v = sdf_h(v);
                    acc = fmaf(v, cf[j], acc);
                }
                if (m.half_round) acc = sdf_h(acc);
                if (sum) feat[f] += acc; else feat[k * F + f] = acc;
            }
        }
        if (k == nl - 1) return;
    }
}

// HashGrid.interpolate (hash_grid.py:205-233) for one point -> feat[0 .. F) ('sum') or feat[0 .. L*F) ('cat').  Per LOD the corners
// of wb_corner_setup and wb_hashgrid_fwd's blend (v0 c0, then an fma over corners 1..7), so each LOD's features are bit-identical to
// wb_hashgrid_fwd's; 'sum' adds all L LODs in LOD order whatever lod_idx, 'cat' writes zeros for the LODs >= lod_idx = nl - 1 (the
// reference's in-place feats[..., lod_idx*F:] = 0).  F = 4 or 8: a row is one or two float4.
__device__ __forceinline__ void sdf_hash_features(const WbGrid& g, int nl, float cx, float cy, float cz, float* feat)
{
    const int F = g.F, nq = F / 4;
    const bool sum = g.multiscale != 0;
    const int act = sum ? g.L : nl - 1;                 // LODs evaluated
    for (int f = sum ? 0 : act * F; f < (sum ? F : g.L * F); ++f) feat[f] = 0.0f;
    for (int l = 0; l < act; ++l) {
        uint32_t idx[8]; float cf[8];
        wb_corner_setup(g, l, cx, cy, cz, idx, cf);
        const float4* tb = reinterpret_cast<const float4*>(g.table + g.begin[l] * F);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            if (q >= nq) break;
            float4 v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = __ldg(tb + (int64_t)idx[j] * nq + q);
            float a0 = v[0].x * cf[0], a1 = v[0].y * cf[0], a2 = v[0].z * cf[0], a3 = v[0].w * cf[0];
#pragma unroll
            for (int j = 1; j < 8; ++j) {
                a0 = fmaf(v[j].x, cf[j], a0); a1 = fmaf(v[j].y, cf[j], a1); a2 = fmaf(v[j].z, cf[j], a2); a3 = fmaf(v[j].w, cf[j], a3);
            }
            float* o = feat + (sum ? 0 : l * F) + 4 * q;
            if (sum) { o[0] += a0; o[1] += a1; o[2] += a2; o[3] += a3; }
            else { o[0] = a0; o[1] = a1; o[2] = a2; o[3] = a3; }
        }
    }
}

// The scatter of a hash field (HashGrid.interpolate's backward, wb_hashgrid_bwd's products): per LOD and corner fl(g * c_j) added to
// the table gradient gt [rows, F] with one float4 reduction per corner and quad of features; quads of zero gradients are skipped, and
// the 'cat' LODs >= lod_idx = nl - 1, whose features the forward zeroed, get nothing.  grad(f): dL/dfeat of decoder-input feature f.
// Shared by the training kernels of wb_sdf_train.cu and wb_sdf_train_tc.cu.
template <class Grad>
__device__ __forceinline__ void sdf_hash_scatter(const WbGrid& g, float* gt, int nl, float cx, float cy, float cz, Grad grad)
{
    const int F = g.F, nq = F / 4;
    const bool sum = g.multiscale != 0;
    const int act = sum ? g.L : nl - 1;
    for (int l = 0; l < act; ++l) {
        float gv[8];
        bool any = false;
#pragma unroll
        for (int f = 0; f < 8; ++f) { gv[f] = f < F ? grad(sum ? f : l * F + f) : 0.0f; any |= gv[f] != 0.0f; }
        if (!any) continue;
        uint32_t idx[8]; float cf[8];
        wb_corner_setup(g, l, cx, cy, cz, idx, cf);
        float4* tb = reinterpret_cast<float4*>(gt + g.begin[l] * F);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            if (q >= nq) break;
            const float g0 = gv[4 * q], g1 = gv[4 * q + 1], g2 = gv[4 * q + 2], g3 = gv[4 * q + 3];
            if (g0 == 0.0f && g1 == 0.0f && g2 == 0.0f && g3 == 0.0f) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j) atomicAdd(tb + (int64_t)idx[j] * nq + q, make_float4(g0 * cf[j], g1 * cf[j], g2 * cf[j], g3 * cf[j]));
        }
    }
}

// the app/nglod shape (nglod_octree.yaml): 'sum' grid of 16 features, identity position input, one hidden layer
static inline bool sdf_fast_shape(const WbSdf& m) { return m.multiscale == 1 && m.F == 16 && m.pos_mode == 1 && m.nh == 1; }
