// wb_sdf_train.cu -- the training step of app/nglod, SDFTrainer.step (wisp/trainers/sdf_trainer.py:65-124), over NeuralSDF.sdf
// (wisp/models/nefs/neural_sdf.py:120-155) on an OctreeGrid: forward, L2 loss and backward of one loss LOD in ONE launch.
// The reference runs the grid kernel, a cat, two cuBLAS GEMMs, the loss ops and their autograd backward (cuBLAS + the grid
// scatter) per LOD.
//
// One hidden layer (wb_sdf_train_kernel; decoders with 2 to 4 hidden layers: wb_sdf_train_deep_kernel below).
// A CTA works on tiles of WB_SDF_TRAIN_TILE samples, grid-stride:
//   pass 1, thread per sample: the forward of wb_sdf_eval (wb_sdf.cuh: same features, same summation order, so the same y), the
//     loss, and dL/dx = dy * sum_{j: a_j > 0} wout_j W0[j,:], whose feature part is scattered into the grid gradients at once with
//     wb_octree_interp_bwd's arithmetic (fp32 gradient, zeros skipped, no gradient to the coordinates; the fp16 rounding of the
//     forward is passed straight through).  The decoder input x and dy stay in shared memory.
//   pass 2, thread per hidden unit j: a_j recomputed for every sample of the tile (same order, so the same relu mask) and
//     dL/dW0[j,:] += da x, dL/db0[j] += da, dL/dwout[j] += dy relu(a), accumulated over all tiles of the CTA and added to
//     grad_params once at the end (per-sample atomics into the decoder would serialise on a few thousand addresses).
// fp32 SIMT throughout: ~15 kFLOP per sample against ~3 KB of feature gather and ~6 KB of scatter read-modify-write.
// A hash field (NeuralSDF(HashGrid), the HASH instances) runs the same kernels with the hash-grid gather of wb_sdf.cuh and the
// scatter below in place of the octree's; everything else (tiles, summation orders, footprint) is unchanged.
#include "wb_sdf.cuh"

constexpr int WB_SDF_TRAIN_TILE = 128;

struct WbSdfTrain {
    const float* coords; const float* gt; int64_t N; float inv_count;
    float* gparams; float* loss;
    int xs_off, gw_off, red_off;          // shared-memory offsets (floats): x [TILE][in_pad] + dy [TILE] | dL/dW0 [H][in_pad+1] | reduction
};

// 'sum' grid of FT features (FT % 4 == 0): every LOD gets the same dL/dfeat g (registers); one float4 reduction per corner and quad
template <int FT>
__device__ __forceinline__ void sdf_scatter_sum(const WbGridX& x, float cx, float cy, float cz, const float* g)
{
    wb_oct_walk(x, cx, cy, cz, [&](int l, int node) {
        float cf[8]; int tk[8];
        wb_oct_cell(x, node, l, cx, cy, cz, cf, tk);
        float4* gt = reinterpret_cast<float4*>(x.gptr[l - x.base_lod]);
#pragma unroll
        for (int q = 0; q < FT / 4; ++q) {
            if (g[4 * q] == 0.0f && g[4 * q + 1] == 0.0f && g[4 * q + 2] == 0.0f && g[4 * q + 3] == 0.0f) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                atomicAdd(gt + (int64_t)tk[j] * (FT / 4) + q, make_float4(g[4 * q] * cf[j], g[4 * q + 1] * cf[j], g[4 * q + 2] * cf[j], g[4 * q + 3] * cf[j]));
        }
    });
}

// HASH: a hash field, gathered from hg and scattered into gx.gptr[0] (the codebook gradient); gx's octree part is unused
template <int FT, int PT, bool HASH = false>
__global__ void __launch_bounds__(WB_SDF_TRAIN_TILE)
wb_sdf_train_kernel(WbOct oc, WbSdf m, WbGridX gx, int nl, WbSdfTrain T, WbGrid hg)
{
    constexpr bool FAST = FT > 0 && PT == 1;             // dispatch guarantees nh == 1, 'sum', identity position input
    constexpr int INF = FAST ? ((3 + FT + 3) & ~3) : 1;  // compile-time in_pad of the fast shape
    extern __shared__ __align__(16) float sw[];
    sdf_stage(m, sw);
    const int H = m.H, INP = FAST ? INF : m.in_pad, IN = m.in_dim;
    const float* b0 = sw + H * INP; const float* wo = b0 + H;
    float* xs = sw + T.xs_off; float* dys = xs + WB_SDF_TRAIN_TILE * INP;
    float* gw = sw + T.gw_off;                             // generic shape: dL/dW0, row j owned by thread j (odd stride: no bank conflicts)
    const int tid = threadIdx.x, GS = INP + 1;
    float gwr[INF];                                       // fast shape: dL/dW0[tid, :] in registers
#pragma unroll
    for (int k = 0; k < INF; ++k) gwr[k] = 0.0f;
    if (!FAST) for (int e = tid; e < H * GS; e += blockDim.x) gw[e] = 0.0f;
    float gb = 0.0f, gwo = 0.0f, lsum = 0.0f, dsum = 0.0f;
    for (int64_t base = (int64_t)blockIdx.x * WB_SDF_TRAIN_TILE; base < T.N; base += (int64_t)gridDim.x * WB_SDF_TRAIN_TILE) {
        const int64_t i = base + tid;
        float* xr = xs + tid * INP;
        float dy = 0.0f;
        if (i < T.N) {
            const float x = __ldg(T.coords + 3 * i), y = __ldg(T.coords + 3 * i + 1), z = __ldg(T.coords + 3 * i + 2);
            if constexpr (FAST) {
                float in[INF], g[INF];
                in[0] = x; in[1] = y; in[2] = z;
                sdf_features<FT>(oc, m, nl, x, y, z, in + 3);
#pragma unroll
                for (int k = 3 + FT; k < INF; ++k) in[k] = 0.0f;
#pragma unroll
                for (int k = 0; k < INF; ++k) g[k] = 0.0f;
                float out = wo[H];
                int j = 0;
                for (; j + 4 <= H; j += 4) {                    // wb_sdf_eval's order: four chains, output layer in unit order
                    float a0 = b0[j], a1 = b0[j + 1], a2 = b0[j + 2], a3 = b0[j + 3];
                    const float4* w0 = reinterpret_cast<const float4*>(sw + j * INF);
                    const float4* w1 = reinterpret_cast<const float4*>(sw + (j + 1) * INF);
                    const float4* w2 = reinterpret_cast<const float4*>(sw + (j + 2) * INF);
                    const float4* w3 = reinterpret_cast<const float4*>(sw + (j + 3) * INF);
#pragma unroll
                    for (int q = 0; q < INF / 4; ++q) {
                        const float4 u0 = w0[q], u1 = w1[q], u2 = w2[q], u3 = w3[q];
                        const float x0 = in[4 * q], x1 = in[4 * q + 1], x2 = in[4 * q + 2], x3 = in[4 * q + 3];
                        a0 = fmaf(u0.x, x0, a0); a1 = fmaf(u1.x, x0, a1); a2 = fmaf(u2.x, x0, a2); a3 = fmaf(u3.x, x0, a3);
                        a0 = fmaf(u0.y, x1, a0); a1 = fmaf(u1.y, x1, a1); a2 = fmaf(u2.y, x1, a2); a3 = fmaf(u3.y, x1, a3);
                        a0 = fmaf(u0.z, x2, a0); a1 = fmaf(u1.z, x2, a1); a2 = fmaf(u2.z, x2, a2); a3 = fmaf(u3.z, x2, a3);
                        a0 = fmaf(u0.w, x3, a0); a1 = fmaf(u1.w, x3, a1); a2 = fmaf(u2.w, x3, a2); a3 = fmaf(u3.w, x3, a3);
                    }
                    out = fmaf(wo[j], fmaxf(a0, 0.0f), out); out = fmaf(wo[j + 1], fmaxf(a1, 0.0f), out);
                    out = fmaf(wo[j + 2], fmaxf(a2, 0.0f), out); out = fmaf(wo[j + 3], fmaxf(a3, 0.0f), out);
                    const float c0 = a0 > 0.0f ? wo[j] : 0.0f, c1 = a1 > 0.0f ? wo[j + 1] : 0.0f;
                    const float c2 = a2 > 0.0f ? wo[j + 2] : 0.0f, c3 = a3 > 0.0f ? wo[j + 3] : 0.0f;
#pragma unroll
                    for (int q = 0; q < INF / 4; ++q) {
                        const float4 u0 = w0[q], u1 = w1[q], u2 = w2[q], u3 = w3[q];
                        g[4 * q] = fmaf(c0, u0.x, fmaf(c1, u1.x, fmaf(c2, u2.x, fmaf(c3, u3.x, g[4 * q]))));
                        g[4 * q + 1] = fmaf(c0, u0.y, fmaf(c1, u1.y, fmaf(c2, u2.y, fmaf(c3, u3.y, g[4 * q + 1]))));
                        g[4 * q + 2] = fmaf(c0, u0.z, fmaf(c1, u1.z, fmaf(c2, u2.z, fmaf(c3, u3.z, g[4 * q + 2]))));
                        g[4 * q + 3] = fmaf(c0, u0.w, fmaf(c1, u1.w, fmaf(c2, u2.w, fmaf(c3, u3.w, g[4 * q + 3]))));
                    }
                }
                for (; j < H; ++j) {
                    const float4* wr = reinterpret_cast<const float4*>(sw + j * INF);
                    float a = b0[j];
#pragma unroll
                    for (int q = 0; q < INF / 4; ++q) {
                        const float4 w = wr[q];
                        a = fmaf(w.x, in[4 * q], a); a = fmaf(w.y, in[4 * q + 1], a); a = fmaf(w.z, in[4 * q + 2], a); a = fmaf(w.w, in[4 * q + 3], a);
                    }
                    out = fmaf(wo[j], fmaxf(a, 0.0f), out);
                    const float c = a > 0.0f ? wo[j] : 0.0f;
#pragma unroll
                    for (int q = 0; q < INF / 4; ++q) {
                        const float4 w = wr[q];
                        g[4 * q] = fmaf(c, w.x, g[4 * q]); g[4 * q + 1] = fmaf(c, w.y, g[4 * q + 1]);
                        g[4 * q + 2] = fmaf(c, w.z, g[4 * q + 2]); g[4 * q + 3] = fmaf(c, w.w, g[4 * q + 3]);
                    }
                }
                const float d = out - __ldg(T.gt + i);
                lsum = fmaf(d, d, lsum);
                dy = T.inv_count * (2.0f * d);
                float4* x4 = reinterpret_cast<float4*>(xr);
#pragma unroll
                for (int q = 0; q < INF / 4; ++q) x4[q] = make_float4(in[4 * q], in[4 * q + 1], in[4 * q + 2], in[4 * q + 3]);
                float gf[FAST ? FT : 1];
#pragma unroll
                for (int f = 0; f < FT; ++f) gf[f] = dy * g[3 + f];
                sdf_scatter_sum<FT>(gx, x, y, z, gf);
            } else {
                float g[WB_SDF_MAX_IN];
                const int pd = sdf_embed(m.pos_mode, m.pos_freq, x, y, z, xr);
                if constexpr (HASH) sdf_hash_features(hg, nl, x, y, z, xr + pd);
                else sdf_features<0>(oc, m, nl, x, y, z, xr + pd);
                for (int k = IN; k < INP; ++k) xr[k] = 0.0f;
                for (int k = pd; k < IN; ++k) g[k] = 0.0f;
                float out = wo[H];
                for (int j = 0; j < H; ++j) {                   // wb_sdf_eval's order
                    const float* wj = sw + j * INP;
                    float a = b0[j];
                    for (int k = 0; k < IN; ++k) a = fmaf(wj[k], xr[k], a);
                    out = fmaf(wo[j], fmaxf(a, 0.0f), out);
                    if (a > 0.0f) for (int k = pd; k < IN; ++k) g[k] = fmaf(wo[j], wj[k], g[k]);
                }
                const float d = out - __ldg(T.gt + i);
                lsum = fmaf(d, d, lsum);
                dy = T.inv_count * (2.0f * d);
                if constexpr (HASH) sdf_hash_scatter(hg, gx.gptr[0], nl, x, y, z, [&](int f) { return dy * g[pd + f]; });
                else wb_featx_scatter(gx, x, y, z, [&](int f) { return dy * g[pd + f]; });
            }
        }
        dys[tid] = dy; dsum += dy;
        __syncthreads();
        const int cnt = (int)min((int64_t)WB_SDF_TRAIN_TILE, T.N - base);
        if (tid < H) {
            const int j = tid;
            const float bj = b0[j], woj = wo[j];
            if constexpr (FAST) {
                float wr[INF];
                const float4* w4 = reinterpret_cast<const float4*>(sw + j * INF);
#pragma unroll
                for (int q = 0; q < INF / 4; ++q) { const float4 w = w4[q]; wr[4 * q] = w.x; wr[4 * q + 1] = w.y; wr[4 * q + 2] = w.z; wr[4 * q + 3] = w.w; }
                for (int s = 0; s < cnt; ++s) {
                    const float4* x4 = reinterpret_cast<const float4*>(xs + s * INF);
                    float xv[INF];
#pragma unroll
                    for (int q = 0; q < INF / 4; ++q) { const float4 v = x4[q]; xv[4 * q] = v.x; xv[4 * q + 1] = v.y; xv[4 * q + 2] = v.z; xv[4 * q + 3] = v.w; }
                    float a = bj;
#pragma unroll
                    for (int k = 0; k < INF; ++k) a = fmaf(wr[k], xv[k], a);
                    const float ds = dys[s];
                    const float da = a > 0.0f ? ds * woj : 0.0f;
                    gb += da; gwo = fmaf(ds, fmaxf(a, 0.0f), gwo);
#pragma unroll
                    for (int k = 0; k < INF; ++k) gwr[k] = fmaf(da, xv[k], gwr[k]);
                }
            } else {
                const float* wj = sw + j * INP;
                float* gj = gw + j * GS;
                for (int s = 0; s < cnt; ++s) {
                    const float* xv = xs + s * INP;
                    float a = bj;
                    for (int k = 0; k < IN; ++k) a = fmaf(wj[k], xv[k], a);
                    const float ds = dys[s];
                    const float da = a > 0.0f ? ds * woj : 0.0f;
                    gb += da; gwo = fmaf(ds, fmaxf(a, 0.0f), gwo);
                    if (da != 0.0f) for (int k = 0; k < IN; ++k) gj[k] = fmaf(da, xv[k], gj[k]);
                }
            }
        }
        __syncthreads();
    }
    // flush: the decoder gradients of this CTA, then the loss and dL/dbout reduced over the CTA
    float* gp = T.gparams;
    if (tid < H) {
        const int j = tid;
        if constexpr (FAST) {
#pragma unroll
            for (int k = 0; k < INF; ++k) if (k < IN && gwr[k] != 0.0f) atomicAdd(gp + j * IN + k, gwr[k]);
        } else {
            for (int k = 0; k < IN; ++k) { const float v = gw[j * GS + k]; if (v != 0.0f) atomicAdd(gp + j * IN + k, v); }
        }
        if (gb != 0.0f) atomicAdd(gp + H * IN + j, gb);
        if (gwo != 0.0f) atomicAdd(gp + H * IN + H + j, gwo);
    }
    float* red = sw + T.red_off;
    lsum = wb_warp_sum(lsum); dsum = wb_warp_sum(dsum);
    if ((tid & 31) == 0) { red[2 * (tid >> 5)] = lsum; red[2 * (tid >> 5) + 1] = dsum; }
    __syncthreads();
    if (tid == 0) {
        float l = 0.0f, d = 0.0f;
        for (int w = 0; w < WB_SDF_TRAIN_TILE / 32; ++w) { l += red[2 * w]; d += red[2 * w + 1]; }
        if (l != 0.0f) atomicAdd(T.loss, l * T.inv_count);
        if (d != 0.0f) atomicAdd(gp + H * IN + 2 * H, d);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// decoders with 2 to 4 hidden layers (H % 4 == 0): layer by layer over a tile of T samples, everything in shared memory
// ---------------------------------------------------------------------------------------------------------------------
// Shared memory: the decoder image (sdf_stage) | the CTA's decoder-gradient accumulators in the image's layout | the tile: x
// [T][SX] | h_0 .. h_{nh-1} [T][SH] | dy [T] | reduction.  Row strides SX, SH = 4 (mod 32) floats: the layer loops put one sample
// per lane and read a float4 of its row, eight lanes per wavefront hit 32 distinct banks.
//   forward   layer k, thread per (sample, 4 units): wb_sdf_eval's chains (per unit seeded with the bias, over the inputs in order;
//             the output over the units in order), so the same y; relu(a) kept per layer (a > 0 <=> relu(a) > 0: the mask)
//   backward  delta_{nh-1} = relu'(a) * fl(dy wout), then for k = nh-1 .. 0: dL/dW_k += delta_k^T h_{k-1} (4x4 register blocks,
//             a chain over the CTA's samples in order), dL/db_k += delta_k (thread per unit), and delta_{k-1} = relu'(a_{k-1}) *
//             W_k^T delta_k (a chain over the units in order) written over h_{k-1}; through W0 the feature columns of the input
//             gradient, scattered as the one-layer kernel does.
// T (a multiple of 32, at most 128) is the largest tile that fits next to the image and the accumulators (sdf_train_plan).
constexpr int WB_SDF_DEEP_THREADS = 256;

struct WbSdfTrainDeep {
    const float* coords; const float* gt; int64_t N; float inv_count;
    float* gparams; float* loss;
    int T, SX, SH;                        // tile, row strides of x and of the hidden rows (floats)
    int acc_off, tile_off, red_off;       // shared-memory offsets (floats)
};

static inline int sdf_deep_stride(int n) { return ((n + 31) & ~31) + 4; }

// out[s][j] = relu(b[j] + sum_{i < IN} W[j][i] in[s][i]) for s < cnt, four units per thread
__device__ __forceinline__ void sdf_deep_fwd(const float* W, int ldw, const float* b, int IN, int H, const float* in, int ldi, float* out, int ldo,
                                             int T, int cnt)
{
    const int items = T * (H / 4);
    for (int e = threadIdx.x; e < items; e += blockDim.x) {
        const int s = e % T, j = (e / T) * 4;
        if (s >= cnt) continue;
        const float* x = in + s * ldi;
        const float* w0 = W + j * ldw; const float* w1 = w0 + ldw; const float* w2 = w1 + ldw; const float* w3 = w2 + ldw;
        float a0 = b[j], a1 = b[j + 1], a2 = b[j + 2], a3 = b[j + 3];
        int i = 0;
        for (; i + 4 <= IN; i += 4) {
            const float4 v = *reinterpret_cast<const float4*>(x + i);
            const float4 u0 = *reinterpret_cast<const float4*>(w0 + i), u1 = *reinterpret_cast<const float4*>(w1 + i);
            const float4 u2 = *reinterpret_cast<const float4*>(w2 + i), u3 = *reinterpret_cast<const float4*>(w3 + i);
            a0 = fmaf(u0.x, v.x, a0); a1 = fmaf(u1.x, v.x, a1); a2 = fmaf(u2.x, v.x, a2); a3 = fmaf(u3.x, v.x, a3);
            a0 = fmaf(u0.y, v.y, a0); a1 = fmaf(u1.y, v.y, a1); a2 = fmaf(u2.y, v.y, a2); a3 = fmaf(u3.y, v.y, a3);
            a0 = fmaf(u0.z, v.z, a0); a1 = fmaf(u1.z, v.z, a1); a2 = fmaf(u2.z, v.z, a2); a3 = fmaf(u3.z, v.z, a3);
            a0 = fmaf(u0.w, v.w, a0); a1 = fmaf(u1.w, v.w, a1); a2 = fmaf(u2.w, v.w, a2); a3 = fmaf(u3.w, v.w, a3);
        }
        for (; i < IN; ++i) {
            const float v = x[i];
            a0 = fmaf(w0[i], v, a0); a1 = fmaf(w1[i], v, a1); a2 = fmaf(w2[i], v, a2); a3 = fmaf(w3[i], v, a3);
        }
        *reinterpret_cast<float4*>(out + s * ldo + j) = make_float4(fmaxf(a0, 0.0f), fmaxf(a1, 0.0f), fmaxf(a2, 0.0f), fmaxf(a3, 0.0f));
    }
}

// out[s][i] = sum_{j < H} W[j][i] d[s][j] (units in order) for s < cnt and i in [i0, i1) (multiples of 4), four inputs per thread;
// mask: zero where the old out[s][i] (the forward's relu(a)) is not positive
__device__ __forceinline__ void sdf_deep_bwd(const float* W, int ldw, int H, const float* d, int ldd, float* out, int ldo, int i0, int i1, bool mask,
                                             int T, int cnt)
{
    const int items = T * ((i1 - i0) / 4);
    for (int e = threadIdx.x; e < items; e += blockDim.x) {
        const int s = e % T, i = i0 + (e / T) * 4;
        if (s >= cnt) continue;
        const float* dr = d + s * ldd;
        float g0 = 0.0f, g1 = 0.0f, g2 = 0.0f, g3 = 0.0f;
        for (int j = 0; j < H; j += 4) {
            const float4 dv = *reinterpret_cast<const float4*>(dr + j);
            const float dd[4] = { dv.x, dv.y, dv.z, dv.w };
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float4 u = *reinterpret_cast<const float4*>(W + (j + r) * ldw + i);
                g0 = fmaf(u.x, dd[r], g0); g1 = fmaf(u.y, dd[r], g1); g2 = fmaf(u.z, dd[r], g2); g3 = fmaf(u.w, dd[r], g3);
            }
        }
        float4* o = reinterpret_cast<float4*>(out + s * ldo + i);
        if (mask) {
            const float4 h = *o;
            g0 = h.x > 0.0f ? g0 : 0.0f; g1 = h.y > 0.0f ? g1 : 0.0f; g2 = h.z > 0.0f ? g2 : 0.0f; g3 = h.w > 0.0f ? g3 : 0.0f;
        }
        *o = make_float4(g0, g1, g2, g3);
    }
}

// G[j][i] += sum_{s < cnt} d[s][j] in[s][i] (samples in order) for j < H, i < INP (multiples of 4), 4 x 4 per thread;
// gb[j] += sum_{s < cnt} d[s][j], thread per unit
__device__ __forceinline__ void sdf_deep_grad(float* G, int ldg, float* gb, int H, int INP, const float* d, int ldd, const float* in, int ldi, int cnt)
{
    const int nib = INP / 4, items = (H / 4) * nib;
    for (int e = threadIdx.x; e < items; e += blockDim.x) {
        const int i = (e % nib) * 4, j = (e / nib) * 4;
        float acc[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float4 v = *reinterpret_cast<const float4*>(G + (j + r) * ldg + i);
            acc[r][0] = v.x; acc[r][1] = v.y; acc[r][2] = v.z; acc[r][3] = v.w;
        }
        for (int s = 0; s < cnt; ++s) {
            const float4 dv = *reinterpret_cast<const float4*>(d + s * ldd + j);
            const float4 xv = *reinterpret_cast<const float4*>(in + s * ldi + i);
            const float dd[4] = { dv.x, dv.y, dv.z, dv.w };
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                acc[r][0] = fmaf(dd[r], xv.x, acc[r][0]); acc[r][1] = fmaf(dd[r], xv.y, acc[r][1]);
                acc[r][2] = fmaf(dd[r], xv.z, acc[r][2]); acc[r][3] = fmaf(dd[r], xv.w, acc[r][3]);
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) *reinterpret_cast<float4*>(G + (j + r) * ldg + i) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
    }
    if (threadIdx.x < H) {
        const int j = threadIdx.x;
        float a = gb[j];
        for (int s = 0; s < cnt; ++s) a += d[s * ldd + j];
        gb[j] = a;
    }
}

template <bool HASH = false>      // as wb_sdf_train_kernel
__global__ void __launch_bounds__(WB_SDF_DEEP_THREADS)
wb_sdf_train_deep_kernel(WbOct oc, WbSdf m, WbGridX gx, int nl, WbSdfTrainDeep T, WbGrid hg)
{
    extern __shared__ __align__(16) float sw[];
    const int H = m.H, INP = m.in_pad, IN = m.in_dim, nh = m.nh, tid = threadIdx.x;
    const int TS = T.T, SX = T.SX, SH = T.SH;
    float* acc = sw + T.acc_off;
    for (int e = tid; e < m.smem_floats; e += blockDim.x) acc[e] = 0.0f;
    sdf_stage(m, sw);
    float* xs = sw + T.tile_off;
    float* hs = xs + TS * SX;                              // h_k: hs + k * TS * SH
    float* dys = hs + nh * TS * SH;
    const int lw = H * INP + H + (nh - 1) * (H * H + H);   // offset of wout in the image and in acc
    const float* wo = sw + lw;
    float lsum = 0.0f, dsum = 0.0f;
    for (int64_t base = (int64_t)blockIdx.x * TS; base < T.N; base += (int64_t)gridDim.x * TS) {
        const int cnt = (int)min((int64_t)TS, T.N - base);
        if (tid < cnt) {                                   // decoder input of sample tid
            const int64_t i = base + tid;
            float* xr = xs + tid * SX;
            const float x = __ldg(T.coords + 3 * i), y = __ldg(T.coords + 3 * i + 1), z = __ldg(T.coords + 3 * i + 2);
            const int pd = sdf_embed(m.pos_mode, m.pos_freq, x, y, z, xr);
            if constexpr (HASH) sdf_hash_features(hg, nl, x, y, z, xr + pd);
            else sdf_features<0>(oc, m, nl, x, y, z, xr + pd);
            for (int k = IN; k < INP; ++k) xr[k] = 0.0f;
        }
        __syncthreads();
        for (int l = 0; l < nh; ++l) {
            const float* Wl = l == 0 ? sw : sw + H * INP + H + (l - 1) * (H * H + H);
            sdf_deep_fwd(Wl, l == 0 ? INP : H, Wl + (l == 0 ? H * INP : H * H), l == 0 ? IN : H, H,
                         l == 0 ? xs : hs + (l - 1) * TS * SH, l == 0 ? SX : SH, hs + l * TS * SH, SH, TS, cnt);
            __syncthreads();
        }
        float* top = hs + (nh - 1) * TS * SH;
        if (tid < cnt) {                                   // output, loss, dy
            const float* hr = top + tid * SH;
            float out = wo[H];
            for (int j = 0; j < H; j += 4) {
                const float4 v = *reinterpret_cast<const float4*>(hr + j);
                out = fmaf(wo[j], v.x, out); out = fmaf(wo[j + 1], v.y, out); out = fmaf(wo[j + 2], v.z, out); out = fmaf(wo[j + 3], v.w, out);
            }
            const float d = out - __ldg(T.gt + base + tid);
            lsum = fmaf(d, d, lsum);
            const float dy = T.inv_count * (2.0f * d);
            dys[tid] = dy; dsum += dy;
        }
        __syncthreads();
        if (tid < H) {                                     // dL/dwout, and delta of the last hidden layer over its activations
            const int j = tid;
            const float woj = wo[j];
            float g = acc[lw + j];
            for (int s = 0; s < cnt; ++s) {
                const float ds = dys[s], h = top[s * SH + j];
                g = fmaf(ds, h, g);
                top[s * SH + j] = h > 0.0f ? ds * woj : 0.0f;
            }
            acc[lw + j] = g;
        }
        __syncthreads();
        for (int l = nh - 1; l >= 0; --l) {
            const int wof = l == 0 ? 0 : H * INP + H + (l - 1) * (H * H + H), ldw = l == 0 ? INP : H;
            const float* dl = hs + l * TS * SH;
            float* in = l == 0 ? xs : hs + (l - 1) * TS * SH;
            const int ldi = l == 0 ? SX : SH;
            sdf_deep_grad(acc + wof, ldw, acc + wof + H * ldw, H, ldw, dl, SH, in, ldi, cnt);
            __syncthreads();
            // l > 0: delta_{l-1} over h_{l-1}; l == 0: the input gradient's feature columns over x (x is no longer needed)
            const int pd4 = l == 0 ? m.pos_dim & ~3 : 0;
            sdf_deep_bwd(sw + wof, ldw, H, dl, SH, in, ldi, pd4, ldw, l > 0, TS, cnt);
            __syncthreads();
        }
        if (tid < cnt) {
            const int64_t i = base + tid;
            const float* gr = xs + tid * SX + m.pos_dim;
            const float x = __ldg(T.coords + 3 * i), y = __ldg(T.coords + 3 * i + 1), z = __ldg(T.coords + 3 * i + 2);
            if constexpr (HASH) sdf_hash_scatter(hg, gx.gptr[0], nl, x, y, z, [&](int f) { return gr[f]; });
            else wb_featx_scatter(gx, x, y, z, [&](int f) { return gr[f]; });
        }
        __syncthreads();
    }
    // flush: the decoder gradients of this CTA (W0 rows from in_pad to in_dim wide, the rest as packed), then loss and dL/dbout
    float* gp = T.gparams;
    const int P0 = H * INP;
    for (int e = tid; e < P0; e += blockDim.x) {
        const int j = e / INP, k = e - j * INP;
        const float v = acc[e];
        if (k < IN && v != 0.0f) atomicAdd(gp + j * IN + k, v);
    }
    for (int e = P0 + tid; e < lw + H; e += blockDim.x) { const float v = acc[e]; if (v != 0.0f) atomicAdd(gp + H * IN + (e - P0), v); }
    float* red = sw + T.red_off;
    lsum = wb_warp_sum(lsum); dsum = wb_warp_sum(dsum);
    if ((tid & 31) == 0) { red[2 * (tid >> 5)] = lsum; red[2 * (tid >> 5) + 1] = dsum; }
    __syncthreads();
    if (tid == 0) {
        float l = 0.0f, d = 0.0f;
        for (int w = 0; w < WB_SDF_DEEP_THREADS / 32; ++w) { l += red[2 * w]; d += red[2 * w + 1]; }
        if (l != 0.0f) atomicAdd(T.loss, l * T.inv_count);
        if (d != 0.0f) atomicAdd(gp + H * IN + (lw + H - P0), d);
    }
}

// shared memory of a wb_sdf_train launch (bytes) and its sample tile, or -1 when the field's training footprint does not fit
static int sdf_train_plan(const WbSdf& m, int* tile)
{
    const int limit = 227 * 1024;
    if (m.nh == 1) {
        const int xs_off = (m.smem_floats + 3) & ~3;
        const int red_off = xs_off + WB_SDF_TRAIN_TILE * m.in_pad + WB_SDF_TRAIN_TILE + (sdf_fast_shape(m) ? 0 : m.H * (m.in_pad + 1));
        const int smem = (red_off + 2 * (WB_SDF_TRAIN_TILE / 32)) * 4;
        *tile = WB_SDF_TRAIN_TILE;
        return smem <= limit ? smem : -1;
    }
    const int img = (m.smem_floats + 3) & ~3, row = sdf_deep_stride(m.in_pad) + m.nh * sdf_deep_stride(m.H) + 1;
    for (int t = 128; t >= 32; t -= 32) {
        const int smem = (2 * img + t * row + 2 * (WB_SDF_DEEP_THREADS / 32)) * 4;
        if (smem <= limit) { *tile = t; return smem; }
    }
    return -1;
}

extern "C" int64_t wb_sdf_train_smem_bytes(const wb_sdf_desc* nef)
{
    WbSdf m; WbGrid hg; if (wb_make_sdf(nef, &m, &hg)) return -1;
    int tile = 0;
    return sdf_train_plan(m, &tile);
}

extern "C" int wb_sdf_train(const wb_octree* oct, const wb_sdf_desc* nef, int32_t lod_idx, const float* coords, const float* sdf_gt, int64_t N,
                            float inv_count, float* const* grad_feats, float* grad_params, float* loss_out, wb_stream s)
{
    WbSdf m; WbGrid hg; int rc = wb_make_sdf(nef, &m, &hg); if (rc) return rc;
    const bool hash = hg.table != nullptr;
    int tile = 0; const int smem = sdf_train_plan(m, &tile);
    WB_CHECK_ARG(smem > 0, "decoder weights, their gradient accumulators and a 32-sample tile exceed shared memory (wb_sdf_train_smem_bytes < 0)");
    rc = sdf_check_lod(m, hash, lod_idx); if (rc) return rc;
    WB_CHECK_ARG(coords && sdf_gt && grad_feats && grad_params && loss_out && N >= 0, "null pointer");
    if (N == 0) return WB_OK;
    const bool fast = !hash && sdf_fast_shape(m);
    WbOct oc; WbGridX gx; rc = sdf_grad_target(oct, m, hash, lod_idx, grad_feats, fast, &oc, &gx); if (rc) return rc;
    int nl = lod_idx + 1;
    if (m.nh > 1) {
        WbSdfTrainDeep D;
        D.coords = coords; D.gt = sdf_gt; D.N = N; D.inv_count = inv_count; D.gparams = grad_params; D.loss = loss_out;
        D.T = tile; D.SX = sdf_deep_stride(m.in_pad); D.SH = sdf_deep_stride(m.H);
        D.acc_off = (m.smem_floats + 3) & ~3; D.tile_off = 2 * D.acc_off; D.red_off = D.tile_off + tile * (D.SX + m.nh * D.SH + 1);
        const void* kern = hash ? (const void*)wb_sdf_train_deep_kernel<true> : (const void*)wb_sdf_train_deep_kernel<false>;
        void* args[] = { &oc, &m, &gx, &nl, &D, &hg };
        return sdf_train_launch(kern, args, WB_SDF_DEEP_THREADS, smem, N, tile, (cudaStream_t)s);
    }
    WbSdfTrain T;
    T.coords = coords; T.gt = sdf_gt; T.N = N; T.inv_count = inv_count; T.gparams = grad_params; T.loss = loss_out;
    T.xs_off = (m.smem_floats + 3) & ~3;
    T.gw_off = T.xs_off + WB_SDF_TRAIN_TILE * m.in_pad + WB_SDF_TRAIN_TILE;
    T.red_off = T.gw_off + (fast ? 0 : m.H * (m.in_pad + 1));
    const void* kern = hash ? (const void*)wb_sdf_train_kernel<0, 0, true> : fast ? (const void*)wb_sdf_train_kernel<16, 1> : (const void*)wb_sdf_train_kernel<0, 0>;
    void* args[] = { &oc, &m, &gx, &nl, &T, &hg };
    return sdf_train_launch(kern, args, WB_SDF_TRAIN_TILE, smem, N, WB_SDF_TRAIN_TILE, (cudaStream_t)s);
}
