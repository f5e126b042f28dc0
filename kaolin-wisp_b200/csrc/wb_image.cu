// wb_image.cu -- app/image natively: the 2-D HashGrid.interpolate kernels and ImageNeuralField (wisp/models/nefs/image_nef.py:37-97)
// evaluated (wb_image_eval) and trained (wb_image_train, ImageTrainer.step: wisp/trainers/image_trainer.py:51-80) in one launch each.
//
// 2-D cell math (hashgrid_interpolate_cuda.cu:214-339, hash_index_2d in hash_utils.cuh:65-84): per axis wb_cell, corner j =
// (x + (j>>1 & 1), y + (j & 1)), coefficients c00 = (1-wx)(1-wy), c01 = (1-wx)wy, c10 = wx(1-wy), c11 = wx wy, each rounded to fp32.
// Rows: dense when res < T and res^2 < T, x + y res; otherwise (x ^ y * 2654435761) & (T - 1).  The table layout does not follow the
// coordinate width: a grid built with coord_dim = 3 (image_hash.yaml does not set it) has min(res^3, T) rows per level, one built with
// coord_dim = 2 has min(res^2, T); rows are always level-local from begin_idxes.  From res 258 on a dense level's clamp bound
// fl(res - 1 - 1e-5) is res - 1 itself, so a coordinate at +1 lands on the level's last cell with weight 0 on its +1 corner; that corner
// keeps the cell's own row (wb_corner_indices' rule for 3-D), so no row outside the level is ever read or written.
//
// ImageNeuralField.rgb = sigmoid(lout(relu(l0(cat([grid features, embed(x, y)]))))), embed = [x, y, sin(c_a 2^f), cos(c_a 2^f)]
// (positional_embedder.py forward: frequency-major, coordinate-minor; 14 wide).  One thread per pixel, fp32 SIMT; the decoder lives in
// shared memory with W0 transposed ([in][H]) so that one float4 broadcast feeds four hidden units.
#include "wb_common.cuh"

constexpr int WB_IMG_THREADS = 128;
constexpr int WB_IMG_EMBED = 14;

// ---------------------------------------------------------------------------------------------------------------------
// 2-D cell
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void img_corner_setup(const WbGrid& g, int l, float cx, float cy, uint32_t idx[4], float cf[4])
{
    int px, py; float wx, wy, ix, iy;
    wb_cell(cx, g.hres[l], g.hi[l], px, wx, ix);
    wb_cell(cy, g.hres[l], g.hi[l], py, wy, iy);
    cf[0] = ix * iy; cf[1] = ix * wy; cf[2] = wx * iy; cf[3] = wx * wy;
    if (g.dense[l]) {
        const uint32_t r1 = (uint32_t)g.res[l], top = r1 - 1u;
        const uint32_t b = (uint32_t)px + (uint32_t)py * r1;
        const uint32_t sx = (uint32_t)px < top ? 1u : 0u, sy = (uint32_t)py < top ? r1 : 0u;
#pragma unroll
        for (int j = 0; j < 4; ++j) idx[j] = b + ((j & 2) ? sx : 0u) + ((j & 1) ? sy : 0u);
    } else {
        const uint32_t x0 = (uint32_t)px, x1 = x0 + 1u;
        const uint32_t y0 = (uint32_t)py * 2654435761u, y1 = y0 + 2654435761u;
#pragma unroll
        for (int j = 0; j < 4; ++j) idx[j] = (((j & 2) ? x1 : x0) ^ ((j & 1) ? y1 : y0)) & g.Tmask;
    }
}

// one table row of F features: F = 2 one float2, F = 4 / 8 one / two float4
template <int F>
__device__ __forceinline__ void img_row(const float* tb, uint32_t r, float* v)
{
    if constexpr (F == 2) {
        const float2 a = __ldg(reinterpret_cast<const float2*>(tb) + r);
        v[0] = a.x; v[1] = a.y;
    } else {
#pragma unroll
        for (int q = 0; q < F / 4; ++q) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(tb) + (int64_t)r * (F / 4) + q);
            v[4 * q] = a.x; v[4 * q + 1] = a.y; v[4 * q + 2] = a.z; v[4 * q + 3] = a.w;
        }
    }
}

// features of LOD l: fl(v_0 c_0), then an fma over corners 1..3 (the contraction of the reference's sum of four products)
template <int F>
__device__ __forceinline__ void img_blend(const WbGrid& g, int l, float cx, float cy, float* acc)
{
    uint32_t idx[4]; float cf[4];
    img_corner_setup(g, l, cx, cy, idx, cf);
    const float* tb = g.table + g.begin[l] * F;
    float v[F];
    img_row<F>(tb, idx[0], v);
#pragma unroll
    for (int f = 0; f < F; ++f) acc[f] = v[f] * cf[0];
#pragma unroll
    for (int j = 1; j < 4; ++j) {
        img_row<F>(tb, idx[j], v);
#pragma unroll
        for (int f = 0; f < F; ++f) acc[f] = fmaf(v[f], cf[j], acc[f]);
    }
}

// grad_table rows += fl(g_f c_j) for the 4 corners of LOD l: one vector reduction per corner and pair / quad, all-zero vectors skipped
template <int F>
__device__ __forceinline__ void img_scatter(const WbGrid& g, float* gtable, int l, float cx, float cy, const float* gv)
{
    uint32_t idx[4]; float cf[4];
    img_corner_setup(g, l, cx, cy, idx, cf);
    float* tb = gtable + g.begin[l] * F;
    if constexpr (F == 2) {
        if (gv[0] == 0.0f && gv[1] == 0.0f) return;
#pragma unroll
        for (int j = 0; j < 4; ++j) atomicAdd(reinterpret_cast<float2*>(tb) + idx[j], make_float2(gv[0] * cf[j], gv[1] * cf[j]));
    } else {
#pragma unroll
        for (int q = 0; q < F / 4; ++q) {
            const float g0 = gv[4 * q], g1 = gv[4 * q + 1], g2 = gv[4 * q + 2], g3 = gv[4 * q + 3];
            if (g0 == 0.0f && g1 == 0.0f && g2 == 0.0f && g3 == 0.0f) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                atomicAdd(reinterpret_cast<float4*>(tb) + (int64_t)idx[j] * (F / 4) + q, make_float4(g0 * cf[j], g1 * cf[j], g2 * cf[j], g3 * cf[j]));
        }
    }
}

// wb_make_grid's validation with the 2-D dense rule; F = 2 rows need 8-byte, F = 4 / 8 rows 16-byte alignment of the table (and of
// the gradient table, checked by the callers)
static int img_make_grid(const wb_nef_desc* d, WbGrid* g)
{
    int rc = wb_make_grid(d, g); if (rc) return rc;
    WB_CHECK_ARG(d->grid_kind == 0, "2-D hash grid: grid_kind must be 0 (hash)");
    const int64_t T = d->codebook_size;
    for (int l = 0; l < g->L; ++l) {
        const int64_t r = g->res[l];
        g->dense[l] = (r < T && r * r < T) ? 1 : 0;               // hash_utils.cuh:76-77
    }
    return WB_OK;
}

static bool img_aligned(const void* p, int F) { return (reinterpret_cast<uintptr_t>(p) & (F == 2 ? 7u : 15u)) == 0; }

// ---------------------------------------------------------------------------------------------------------------------
// HashGrid.interpolate over [N, 2] coordinates: one thread per (coordinate, LOD), all LODs in one launch; feats [N, L*F] raw
// (the host applies the 'cat' zeroing / 'sum' reduction, as for 3-D)
// ---------------------------------------------------------------------------------------------------------------------
template <int F>
__global__ void __launch_bounds__(256)
wb_hashgrid2d_fwd_kernel(WbGrid g, const float* __restrict__ coords, int64_t N, float* __restrict__ feats)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t i = t / g.L; const int l = (int)(t - i * g.L);
    if (i >= N) return;
    const float cx = __ldg(coords + 2 * i), cy = __ldg(coords + 2 * i + 1);
    if constexpr (F > 0) {
        float acc[F];
        img_blend<F>(g, l, cx, cy, acc);
        float* o = feats + (i * g.L + l) * F;
        if constexpr (F == 2) *reinterpret_cast<float2*>(o) = make_float2(acc[0], acc[1]);
        else {
#pragma unroll
            for (int q = 0; q < F / 4; ++q) reinterpret_cast<float4*>(o)[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
        }
    } else {
        uint32_t idx[4]; float cf[4];
        img_corner_setup(g, l, cx, cy, idx, cf);
        const int Fr = g.F;
        const float* tb = g.table + g.begin[l] * Fr;
        for (int f = 0; f < Fr; ++f) {
            float a = __ldg(tb + (int64_t)idx[0] * Fr + f) * cf[0];
#pragma unroll
            for (int j = 1; j < 4; ++j) a = fmaf(__ldg(tb + (int64_t)idx[j] * Fr + f), cf[j], a);
            feats[(i * g.L + l) * Fr + f] = a;
        }
    }
}

template <int F>
__global__ void __launch_bounds__(256)
wb_hashgrid2d_bwd_kernel(WbGrid g, const float* __restrict__ coords, int64_t N, const float* __restrict__ gfeats, float* __restrict__ gtable)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t i = t / g.L; const int l = (int)(t - i * g.L);
    if (i >= N) return;
    const float cx = __ldg(coords + 2 * i), cy = __ldg(coords + 2 * i + 1);
    if constexpr (F > 0) {
        float gv[F];
        const float* go = gfeats + (i * g.L + l) * F;
#pragma unroll
        for (int f = 0; f < F; ++f) gv[f] = __ldg(go + f);
        img_scatter<F>(g, gtable, l, cx, cy, gv);
    } else {
        uint32_t idx[4]; float cf[4];
        img_corner_setup(g, l, cx, cy, idx, cf);
        const int Fr = g.F;
        float* tb = gtable + g.begin[l] * Fr;
        for (int f = 0; f < Fr; ++f) {
            const float go = __ldg(gfeats + (i * g.L + l) * Fr + f);
            if (go == 0.0f) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) atomicAdd(tb + (int64_t)idx[j] * Fr + f, go * cf[j]);
        }
    }
}

extern "C" int wb_hashgrid2d_fwd(const float* coords, int64_t N, const wb_nef_desc* grid, float* feats, wb_stream s)
{
    WbGrid g; int rc = img_make_grid(grid, &g); if (rc) return rc;
    if (N == 0) return WB_OK;
    WB_CHECK_ARG(coords && feats && N > 0, "null pointer or negative N");
    const unsigned blocks = (unsigned)((N * g.L + 255) / 256);
    const cudaStream_t st = (cudaStream_t)s;
    const bool vec = img_aligned(g.table, g.F) && img_aligned(feats, g.F);
    if (vec && g.F == 2) wb_hashgrid2d_fwd_kernel<2><<<blocks, 256, 0, st>>>(g, coords, N, feats);
    else if (vec && g.F == 4) wb_hashgrid2d_fwd_kernel<4><<<blocks, 256, 0, st>>>(g, coords, N, feats);
    else if (vec && g.F == 8) wb_hashgrid2d_fwd_kernel<8><<<blocks, 256, 0, st>>>(g, coords, N, feats);
    else wb_hashgrid2d_fwd_kernel<0><<<blocks, 256, 0, st>>>(g, coords, N, feats);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

extern "C" int wb_hashgrid2d_bwd(const float* coords, int64_t N, const wb_nef_desc* grid, const float* grad_feats, float* grad_table, wb_stream s)
{
    WbGrid g; int rc = img_make_grid(grid, &g); if (rc) return rc;
    if (N == 0) return WB_OK;
    WB_CHECK_ARG(coords && grad_feats && grad_table && N > 0, "null pointer or negative N");
    const unsigned blocks = (unsigned)((N * g.L + 255) / 256);
    const cudaStream_t st = (cudaStream_t)s;
    const bool vec = img_aligned(grad_table, g.F) && img_aligned(grad_feats, g.F);
    if (vec && g.F == 2) wb_hashgrid2d_bwd_kernel<2><<<blocks, 256, 0, st>>>(g, coords, N, grad_feats, grad_table);
    else if (vec && g.F == 4) wb_hashgrid2d_bwd_kernel<4><<<blocks, 256, 0, st>>>(g, coords, N, grad_feats, grad_table);
    else if (vec && g.F == 8) wb_hashgrid2d_bwd_kernel<8><<<blocks, 256, 0, st>>>(g, coords, N, grad_feats, grad_table);
    else wb_hashgrid2d_bwd_kernel<0><<<blocks, 256, 0, st>>>(g, coords, N, grad_feats, grad_table);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// ImageNeuralField: decoder image in shared memory (floats): W0^T [IN][H] | b0 [H] | Wout [3][H] | bout [3]
// Training tile (floats, after the image): x [TS][XS] | h [TS][HS] | da [TS][HS] | dy [TS][4] | dL/dW0 [H][XS] | reduction [4 warps][4]
// XS = IN | 1 and HS = H + 1 are odd: a thread per sample (or per hidden unit) walking its own row hits 32 distinct banks.
// ---------------------------------------------------------------------------------------------------------------------
struct WbImg {
    WbGrid g;
    int nl;                                  // LODs gathered: 'cat' 0 .. lod_idx-1 (the rest are zero), 'sum' all L
    int FW, IN, H, XS, HS, TS;               // feature width, decoder input width (FW + 14), hidden width, row strides, sample tile
    const float* w0; const float* b0; const float* wo; const float* bo;     // W0 [H][IN], b0 [H], Wout [3][H], bout [3] (nn.Linear layout)
    int img_floats;                          // decoder image, rounded up to a float4
    int x_off, h_off, da_off, dy_off, gw_off, red_off;
    const float* coords; const float* gt; int64_t N; float inv_count;
    float* rgb; float* gtable; float* gparams; float* loss;
};

__device__ __forceinline__ void img_stage(const WbImg& m, float* sw)
{
    const int H = m.H, IN = m.IN;
    for (int e = threadIdx.x; e < IN * H; e += blockDim.x) { const int k = e / H, j = e - k * H; sw[e] = __ldg(m.w0 + j * IN + k); }
    float* t = sw + IN * H;
    for (int e = threadIdx.x; e < H; e += blockDim.x) t[e] = __ldg(m.b0 + e);
    for (int e = threadIdx.x; e < 3 * H; e += blockDim.x) t[H + e] = __ldg(m.wo + e);
    if (threadIdx.x < 3) t[4 * H + threadIdx.x] = __ldg(m.bo + threadIdx.x);
    __syncthreads();
}

// decoder input of one pixel into xr[0 .. IN): grid features ('cat': LOD-major, zero from lod_idx on; 'sum': LODs added in order),
// then the 14 embedding values
template <int F>
__device__ __forceinline__ void img_input(const WbImg& m, float cx, float cy, float* xr)
{
    const bool sum = m.g.multiscale != 0;
    if (sum) for (int f = 0; f < F; ++f) xr[f] = 0.0f;
    else for (int f = m.nl * F; f < m.FW; ++f) xr[f] = 0.0f;
    for (int l = 0; l < m.nl; ++l) {
        float acc[F];
        img_blend<F>(m.g, l, cx, cy, acc);
#pragma unroll
        for (int f = 0; f < F; ++f) { if (sum) xr[f] += acc[f]; else xr[l * F + f] = acc[f]; }
    }
    float* e = xr + m.FW;
    e[0] = cx; e[1] = cy;
    float band = 1.0f;                       // bands 2^0, 2^1, 2^2 (get_positional_embedder(3): linspace(0, 2) exponents)
#pragma unroll
    for (int f = 0; f < 3; ++f) {
        const float ux = cx * band, uy = cy * band;
        e[2 + 2 * f] = sinf(ux); e[3 + 2 * f] = sinf(uy);
        e[8 + 2 * f] = cosf(ux); e[9 + 2 * f] = cosf(uy);
        band *= 2.0f;
    }
}

// z = lout(relu(l0(x))): per hidden unit the chain b0_j + sum_k W0[j,k] x_k over k in order, per output bout_c + sum_j Wout[c,j] h_j
// over j in order; hr (optional) receives relu(a)
__device__ __forceinline__ void img_mlp(const WbImg& m, const float* sw, const float* xr, float* hr, float z[3])
{
    const int H = m.H, IN = m.IN, H4 = H / 4;
    const float4* W4 = reinterpret_cast<const float4*>(sw);
    const float* b0 = sw + IN * H; const float* wo = b0 + H; const float* bo = wo + 3 * H;
    float z0 = bo[0], z1 = bo[1], z2 = bo[2];
    for (int j = 0; j < H; j += 4) {
        float4 a = *reinterpret_cast<const float4*>(b0 + j);
        const float4* wc = W4 + j / 4;
        for (int k = 0; k < IN; ++k) {
            const float xv = xr[k];
            const float4 w = wc[k * H4];
            a.x = fmaf(w.x, xv, a.x); a.y = fmaf(w.y, xv, a.y); a.z = fmaf(w.z, xv, a.z); a.w = fmaf(w.w, xv, a.w);
        }
        const float h0 = fmaxf(a.x, 0.0f), h1 = fmaxf(a.y, 0.0f), h2 = fmaxf(a.z, 0.0f), h3 = fmaxf(a.w, 0.0f);
        if (hr) { hr[j] = h0; hr[j + 1] = h1; hr[j + 2] = h2; hr[j + 3] = h3; }
        z0 = fmaf(wo[j], h0, z0); z0 = fmaf(wo[j + 1], h1, z0); z0 = fmaf(wo[j + 2], h2, z0); z0 = fmaf(wo[j + 3], h3, z0);
        z1 = fmaf(wo[H + j], h0, z1); z1 = fmaf(wo[H + j + 1], h1, z1); z1 = fmaf(wo[H + j + 2], h2, z1); z1 = fmaf(wo[H + j + 3], h3, z1);
        z2 = fmaf(wo[2 * H + j], h0, z2); z2 = fmaf(wo[2 * H + j + 1], h1, z2); z2 = fmaf(wo[2 * H + j + 2], h2, z2); z2 = fmaf(wo[2 * H + j + 3], h3, z2);
    }
    z[0] = z0; z[1] = z1; z[2] = z2;
}

__device__ __forceinline__ float img_sigmoid(float z) { return 1.0f / (1.0f + expf(-z)); }

template <int F>
__global__ void __launch_bounds__(WB_IMG_THREADS)
wb_image_eval_kernel(WbImg m)
{
    extern __shared__ __align__(16) float sw[];
    img_stage(m, sw);
    float* xr = sw + m.x_off + threadIdx.x * m.XS;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m.N; i += (int64_t)gridDim.x * blockDim.x) {
        const float cx = __ldg(m.coords + 2 * i), cy = __ldg(m.coords + 2 * i + 1);
        img_input<F>(m, cx, cy, xr);
        float z[3];
        img_mlp(m, sw, xr, nullptr, z);
        m.rgb[3 * i] = img_sigmoid(z[0]); m.rgb[3 * i + 1] = img_sigmoid(z[1]); m.rgb[3 * i + 2] = img_sigmoid(z[2]);
    }
}

// One training launch (wb_sdf_train_kernel<0,0>'s two passes).  Per tile of TS pixels:
//   pass 1, thread per pixel: input, forward (relu(a) kept in h), y = sigmoid(z), the loss, dy_c = inv_count * 2 (y_c - gt_c) * y_c (1 - y_c)
//     (F.mse_loss's mean over 3N and sigmoid's backward), da_j = [a_j > 0] sum_c dy_c Wout[c,j] (kept in da), and per LOD the feature
//     part of dL/dx = sum_j da_j W0[j,:] scattered into the table gradient at once ('cat' LODs >= lod_idx, zero in the forward, get
//     nothing; 'sum' LODs all get the same gradient).
//   pass 2, thread per hidden unit j: dL/dW0[j,:] += da_j x, dL/db0[j] += da_j, dL/dWout[:,j] += dy relu(a_j), over the tile's pixels in
//     order, accumulated over all tiles of the CTA and added to grad_params once at the end.
template <int F>
__global__ void __launch_bounds__(WB_IMG_THREADS)
wb_image_train_kernel(WbImg m)
{
    extern __shared__ __align__(16) float sw[];
    img_stage(m, sw);
    const int H = m.H, IN = m.IN, TS = m.TS, tid = threadIdx.x;
    const float* W0T = sw; const float* wo = sw + IN * H + H;
    float* xs = sw + m.x_off; float* hs = sw + m.h_off; float* das = sw + m.da_off; float* dys = sw + m.dy_off; float* gw = sw + m.gw_off;
    for (int e = tid; e < H * m.XS; e += blockDim.x) gw[e] = 0.0f;
    float gb = 0.0f, gwo0 = 0.0f, gwo1 = 0.0f, gwo2 = 0.0f;
    float lsum = 0.0f, db0 = 0.0f, db1 = 0.0f, db2 = 0.0f;
    const bool sum = m.g.multiscale != 0;
    for (int64_t base = (int64_t)blockIdx.x * TS; base < m.N; base += (int64_t)gridDim.x * TS) {
        const int cnt = (int)min((int64_t)TS, m.N - base);
        if (tid < cnt) {
            const int64_t i = base + tid;
            float* xr = xs + tid * m.XS; float* hr = hs + tid * m.HS; float* dr = das + tid * m.HS;
            const float cx = __ldg(m.coords + 2 * i), cy = __ldg(m.coords + 2 * i + 1);
            img_input<F>(m, cx, cy, xr);
            float z[3], dy[3];
            img_mlp(m, sw, xr, hr, z);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float y = img_sigmoid(z[c]);
                const float d = y - __ldg(m.gt + 3 * i + c);
                lsum = fmaf(d, d, lsum);
                dy[c] = (m.inv_count * (2.0f * d)) * (y * (1.0f - y));
            }
            db0 += dy[0]; db1 += dy[1]; db2 += dy[2];
            dys[4 * tid] = dy[0]; dys[4 * tid + 1] = dy[1]; dys[4 * tid + 2] = dy[2];
            for (int j = 0; j < H; ++j)
                dr[j] = hr[j] > 0.0f ? fmaf(dy[2], wo[2 * H + j], fmaf(dy[1], wo[H + j], dy[0] * wo[j])) : 0.0f;
            float gv[F];
            for (int l = 0; l < (sum ? m.g.L : m.nl); ++l) {
                if (!sum || l == 0) {
#pragma unroll
                    for (int f = 0; f < F; ++f) {
                        const float* wk = W0T + (sum ? f : l * F + f) * H;
                        float a = 0.0f;
                        for (int j = 0; j < H; ++j) a = fmaf(dr[j], wk[j], a);
                        gv[f] = a;
                    }
                }
                img_scatter<F>(m.g, m.gtable, l, cx, cy, gv);
            }
        }
        __syncthreads();
        if (tid < H) {
            const int j = tid;
            float* gj = gw + j * m.XS;
            for (int s = 0; s < cnt; ++s) {
                const float da = das[s * m.HS + j], h = hs[s * m.HS + j];
                gb += da;
                gwo0 = fmaf(dys[4 * s], h, gwo0); gwo1 = fmaf(dys[4 * s + 1], h, gwo1); gwo2 = fmaf(dys[4 * s + 2], h, gwo2);
                if (da != 0.0f) {
                    const float* xv = xs + s * m.XS;
                    for (int k = 0; k < IN; ++k) gj[k] = fmaf(da, xv[k], gj[k]);
                }
            }
        }
        __syncthreads();
    }
    // flush: the decoder gradients of this CTA, then the loss and dL/dbout reduced over the CTA
    float* gp = m.gparams;
    if (tid < H) {
        const int j = tid;
        for (int k = 0; k < IN; ++k) { const float v = gw[j * m.XS + k]; if (v != 0.0f) atomicAdd(gp + j * IN + k, v); }
        if (gb != 0.0f) atomicAdd(gp + H * IN + j, gb);
        if (gwo0 != 0.0f) atomicAdd(gp + H * IN + H + j, gwo0);
        if (gwo1 != 0.0f) atomicAdd(gp + H * IN + 2 * H + j, gwo1);
        if (gwo2 != 0.0f) atomicAdd(gp + H * IN + 3 * H + j, gwo2);
    }
    float* red = sw + m.red_off;
    lsum = wb_warp_sum(lsum); db0 = wb_warp_sum(db0); db1 = wb_warp_sum(db1); db2 = wb_warp_sum(db2);
    if ((tid & 31) == 0) { float* r = red + 4 * (tid >> 5); r[0] = lsum; r[1] = db0; r[2] = db1; r[3] = db2; }
    __syncthreads();
    if (tid < 4) {
        float v = 0.0f;
        for (int w = 0; w < WB_IMG_THREADS / 32; ++w) v += red[4 * w + tid];
        if (v != 0.0f) {
            if (tid == 0) atomicAdd(m.loss, v * m.inv_count);
            else atomicAdd(gp + H * IN + 4 * H + tid - 1, v);
        }
    }
}

// validation + shared-memory plan.  train: the largest tile of {128, 64, 32} pixels that still gives every SM a CTA for N pixels
// (N = 4096, the app's batch: 32-pixel tiles, 128 CTAs) and fits next to the image and the accumulators; eval: one pixel per thread
static int img_plan(const wb_nef_desc* grid, int32_t hidden_dim, int32_t lod_idx, bool train, int64_t N, WbImg* m, int* smem)
{
    memset(m, 0, sizeof(*m));
    int rc = img_make_grid(grid, &m->g); if (rc) return rc;
    const int F = m->g.F, L = m->g.L;
    WB_CHECK_ARG(F == 2 || F == 4 || F == 8, "image field: a hash grid of 2, 4 or 8 features per LOD");
    WB_CHECK_ARG(img_aligned(m->g.table, F), "image field: the table must be 8-byte (F = 2) or 16-byte (F = 4, 8) aligned");
    WB_CHECK_ARG(hidden_dim >= 4 && hidden_dim <= WB_IMG_THREADS && hidden_dim % 4 == 0, "image field: hidden_dim must be a multiple of 4 in [4, 128]");
    WB_CHECK_ARG(lod_idx >= 0 && lod_idx <= L, "lod_idx out of range");
    const bool sum = m->g.multiscale != 0;
    m->nl = sum ? L : lod_idx;
    m->FW = sum ? F : L * F; m->IN = m->FW + WB_IMG_EMBED; m->H = hidden_dim;
    m->XS = m->IN | 1; m->HS = m->H + 1;
    m->img_floats = (m->IN * m->H + 4 * m->H + 3 + 3) & ~3;
    const int limit = 227 * 1024;
    m->x_off = m->img_floats;
    if (!train) {
        m->TS = WB_IMG_THREADS;
        *smem = (m->x_off + WB_IMG_THREADS * m->XS) * 4;
        WB_CHECK_ARG(*smem <= limit, "image field: decoder image and pixel rows exceed shared memory");
        return WB_OK;
    }
    const int sms = wb_num_sms();
    *smem = -1;
    for (int ts = WB_IMG_THREADS; ts >= 32; ts /= 2) {
        const int h_off = m->x_off + ts * m->XS, da_off = h_off + ts * m->HS, dy_off = da_off + ts * m->HS;
        const int gw_off = dy_off + 4 * ts, red_off = gw_off + m->H * m->XS;
        const int bytes = (red_off + 4 * (WB_IMG_THREADS / 32)) * 4;
        if (bytes > limit) continue;
        m->TS = ts; m->h_off = h_off; m->da_off = da_off; m->dy_off = dy_off; m->gw_off = gw_off; m->red_off = red_off; *smem = bytes;
        if ((N + ts - 1) / ts >= sms) break;                  // enough CTAs at this tile; otherwise try a smaller one
    }
    WB_CHECK_ARG(*smem > 0, "image field: decoder image, accumulators and a 32-pixel tile exceed shared memory");
    return WB_OK;
}

extern "C" int64_t wb_image_smem_bytes(const wb_nef_desc* grid, int32_t hidden_dim, int32_t train)
{
    WbImg m; int smem = 0;
    if (img_plan(grid, hidden_dim, grid ? grid->num_lods - 1 : 0, train != 0, INT64_MAX / 2, &m, &smem)) return -1;
    return smem;
}

template <class K>
static int img_launch(K kern, const WbImg& m, int smem, int64_t work, wb_stream s)
{
    WB_CUDA(cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int per_sm = 0;
    WB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)kern, WB_IMG_THREADS, smem));
    WB_CHECK_ARG(per_sm >= 1, "image kernel does not fit on an SM");
    int64_t ctas = work; const int64_t cap = (int64_t)wb_num_sms() * per_sm; if (ctas > cap) ctas = cap;
    kern<<<(unsigned)ctas, WB_IMG_THREADS, (size_t)smem, (cudaStream_t)s>>>(m);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

static int img_params(const float* const* params, WbImg* m)
{
    WB_CHECK_ARG(params && params[0] && params[1] && params[2] && params[3], "null decoder parameter");
    m->w0 = params[0]; m->b0 = params[1]; m->wo = params[2]; m->bo = params[3];
    return WB_OK;
}

extern "C" int wb_image_eval(const wb_nef_desc* grid, int32_t hidden_dim, const float* const* params, int32_t lod_idx, const float* coords,
                             int64_t N, float* rgb, wb_stream s)
{
    WbImg m; int smem = 0;
    int rc = img_plan(grid, hidden_dim, lod_idx, false, N, &m, &smem); if (rc) return rc;
    rc = img_params(params, &m); if (rc) return rc;
    WB_CHECK_ARG(coords && rgb, "null pointer");
    WB_CHECK_ARG(N >= 1, "empty batch");
    m.coords = coords; m.N = N; m.rgb = rgb;
    const int64_t work = (N + WB_IMG_THREADS - 1) / WB_IMG_THREADS;
    if (m.g.F == 2) return img_launch(wb_image_eval_kernel<2>, m, smem, work, s);
    if (m.g.F == 4) return img_launch(wb_image_eval_kernel<4>, m, smem, work, s);
    return img_launch(wb_image_eval_kernel<8>, m, smem, work, s);
}

extern "C" int wb_image_train(const wb_nef_desc* grid, int32_t hidden_dim, const float* const* params, int32_t lod_idx, const float* coords,
                              const float* rgb_gt, int64_t N, float inv_count, float* grad_table, float* grad_params, float* loss_out, wb_stream s)
{
    WbImg m; int smem = 0;
    int rc = img_plan(grid, hidden_dim, lod_idx, true, N, &m, &smem); if (rc) return rc;
    rc = img_params(params, &m); if (rc) return rc;
    WB_CHECK_ARG(coords && rgb_gt && grad_table && grad_params && loss_out, "null pointer");
    WB_CHECK_ARG(img_aligned(grad_table, m.g.F), "the table gradient must be aligned like the table");
    WB_CHECK_ARG(N >= 1, "empty batch");
    m.coords = coords; m.gt = rgb_gt; m.N = N; m.inv_count = inv_count;
    m.gtable = grad_table; m.gparams = grad_params; m.loss = loss_out;
    const int64_t work = (N + m.TS - 1) / m.TS;
    if (m.g.F == 2) return img_launch(wb_image_train_kernel<2>, m, smem, work, s);
    if (m.g.F == 4) return img_launch(wb_image_train_kernel<4>, m, smem, work, s);
    return img_launch(wb_image_train_kernel<8>, m, smem, work, s);
}
