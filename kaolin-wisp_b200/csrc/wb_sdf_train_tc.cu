// wb_sdf_train_tc.cu -- the training step of app/nglod under enable_amp (every app/nglod/configs/*.yaml: enable_amp: True;
// BaseTrainer runs SDFTrainer.step inside torch.cuda.amp.autocast, wisp/trainers/base_trainer.py:338, and the SDF step calls a plain
// loss.backward() without a GradScaler, sdf_trainer.py:122-124) on the tensor cores: forward, L2 loss and backward of one loss LOD
// of NeuralSDF.sdf (wisp/models/nefs/neural_sdf.py:120-155) in ONE launch, the hidden layers as wgmma chains (sm_90a).
//
// Numerics = the reference's autocast nn.Linear: fp16 inputs, weights and biases, fp32 accumulation, fp16 layer outputs (the
// prediction y included); the loss in fp32.  Features are computed as wb_sdf_train computes them (octree: half_round; hash: the
// fp32 table) and rounded to fp16 at the decoder input.  Deviations from the reference: the hash table is read in fp32, the output
// gradient dY = fp16(2 (y - gt) inv_count scale) carries a power-of-two loss scale chosen on the host from inv_count (the
// reference's unscaled fp16 dpred goes subnormal for small residuals), and weight gradients accumulate in fp32 (the reference
// rounds each whole-batch fp16 GEMM result once).  The scale is removed exactly in fp32 at both exits (weight-gradient flush,
// feature-gradient scatter).
//
// One warpgroup (128 threads) per CTA works on 64-sample tiles, grid-stride.  Row r of a tile belongs to threads 2r and 2r + 1.
//   gather     thread 2r + 1: the position embedding (sdf_embed), thread 2r: the grid features (sdf_features / sdf_hash_features),
//              both rounded to fp16 into the X0 slab tile (wb_tc.cuh layout), zero padded to K % 16 == 0
//   hidden l   D[64 x Hp] = fp16 bias + X_l . W_l^T (A: input tile K-major, B: weight pack K-major), relu -> fp16 tile X_{l+1}
//   output     SIMT per row: y = fp16(bout + sum_j fp16(wout_j) h_j) (fp32 sum of exact fp16 products), d = y - gt (fp32),
//              dY = fp16(2 d inv_count scale) and dY_{nh-1}[j] = relu'(h_j) fp16(dY wout_j); dL/dwout += dY h (thread per unit)
//   backward   for l = nh-1 .. 0: dW_l^T[out, in | 1] += dY_l^T . [X_l | 1] (both operands MN-major; the constant-one slab behind
//              every input tile gives the bias gradient) into fp32 accumulators in shared memory; dX = dY_l . W_l (pack read MN-major)
//              masked by relu' of the retained activation tile -> dY_{l-1} (fp16), or for l = 0 the feature columns in fp32 -> the
//              existing scatters (wb_featx_scatter / sdf_hash_scatter), one thread per row.
// The decoder's fp16 weight packs are built by every CTA from the flat fp32 parameter buffer (the weights change every Adam step: no
// separate pack launch), and the CTA's accumulators are added to grad_params once at the end.  wgmma.wait_group 0 after every chain.
#include "wb_sdf.cuh"
#include "wb_tc.cuh"
#include <cmath>

constexpr int STC_ROWS = 64;                  // samples per tile (wgmma M)
constexpr int STC_THREADS = 128;              // one warpgroup
constexpr int STC_SLAB = STC_ROWS * 16;       // bytes of one slab: 8 fp16 features of every sample of the tile

struct WbSdfTc {
    const float* coords; const float* gt; int64_t N;
    float inv_count, scale, inv_scale;        // scale: the power-of-two loss scale of dY; inv_scale = 1 / scale
    float* gparams; float* loss;
    int IN, pd, FD, H, Hp, K0p, nh;           // decoder input width, position dims, feature dims, hidden width (padded to 16)
    int w_off[4], b_off, wo_off;              // byte offsets: fp16 weight packs [Hp x Kp_l], fp16 biases [nh][Hp], fp32 wout [Hp] + bout
    int acc_off, acc_l[5];                    // byte offset of the fp32 accumulators; float offset of layer l's [H][I_l + 1] (l = nh: wout)
    int x_off[5];                             // byte offset of layer l's input tile (l = nh: the last hidden activation)
    int dy_off, gf_off, dys_off, red_off;     // dY tile (Hp rounded up to 64: 8 or 16 slabs), fp32 feature gradient [64][FD + 1], fp32 dY [64], reduction
    int smem;
};

// shared memory of the launch for the field m (bytes), or -1 when it exceeds an SM's 227 KB
static int sdf_tc_plan(const WbSdf& m, WbSdfTc* P)
{
    memset(P, 0, sizeof(*P));
    P->IN = m.in_dim; P->pd = m.pos_dim; P->FD = m.feat_dim; P->H = m.H; P->nh = m.nh;
    P->Hp = wb_round_up(m.H, 16); P->K0p = wb_round_up(m.in_dim, 16);
    int off = 0;
    for (int l = 0; l < m.nh; ++l) { P->w_off[l] = off; off += P->Hp * (l == 0 ? P->K0p : P->Hp) * 2; }
    P->b_off = off; off += wb_round_up(m.nh * P->Hp * 2, 16);
    P->wo_off = off; off += (P->Hp + 4) * 4;
    P->acc_off = off = wb_round_up(off, 128);
    int acc = 0;
    for (int l = 0; l < m.nh; ++l) { P->acc_l[l] = acc; acc += m.H * ((l == 0 ? m.in_dim : m.H) + 1); }
    P->acc_l[m.nh] = acc; acc += m.H;
    off = wb_round_up(off + acc * 4, 128);
    for (int l = 0; l <= m.nh; ++l) { P->x_off[l] = off; off += ((l == 0 ? P->K0p : P->Hp) / 8 + 1) * STC_SLAB; }
    P->dy_off = off; off += wb_round_up(P->Hp, 64) / 8 * STC_SLAB;      // the weight-gradient A operand reads 64 outputs (8 slabs) per pass
    P->gf_off = off; off += wb_round_up(STC_ROWS * (P->FD + 1) * 4, 16);
    P->dys_off = off; off += STC_ROWS * 4;
    P->red_off = off; off += 2 * (STC_THREADS / 32) * 4;
    P->smem = off;
    return off <= 227 * 1024 ? off : -1;
}

// One wgmma chain: D[64 x N] = fp16 bias (bias[n]) or 0, += A . B over nk K-steps of 16; wait; CTA barrier (every MMA has read its
// operands: the epilogue may overwrite them); epi(d) on the accumulator fragments (tc_frag_row / tc_frag_col).
template <int N, int TA, int TB, class Epi>
__device__ __forceinline__ void stc_chain(uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv, const __half* bias, Epi&& epi)
{
    const int wl = threadIdx.x;
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = bias ? __half2float(bias[tc_frag_col(wl, i)]) : 0.0f;
    tc_wg_fence();
    for (int kb = 0; kb < nk; ++kb) { WgMma<N, TA, TB>::run(d, da, db, 1u); da += aadv; db += badv; }
    tc_wg_commit();
    tc_wg_wait0();
    tc_wg_hold(d);
    __syncthreads();
    epi(d);
}
// N chosen at run time: a multiple of 16 up to 128
template <int TA, int TB, class Epi>
__device__ __forceinline__ void stc_chain_n(int N, uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv, const __half* bias, Epi&& epi)
{
    switch (N) {
        case 16: stc_chain<16, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        case 32: stc_chain<32, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        case 48: stc_chain<48, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        case 64: stc_chain<64, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        case 80: stc_chain<80, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        case 96: stc_chain<96, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        case 112: stc_chain<112, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
        default: stc_chain<128, TA, TB>(da, db, nk, aadv, badv, bias, epi); break;
    }
}

__device__ __forceinline__ void stc_store1(uint8_t* tile, int r, int f, float v)
{
    *reinterpret_cast<__half*>(tile + (f >> 3) * STC_SLAB + r * 16 + (f & 7) * 2) = __float2half_rn(v);
}

// FT = 16: a 'sum' octree grid of 16 features (sdf_features' register path); HASH: a hash field, gathered from hg and scattered
// into gx.gptr[0]
template <int FT, bool HASH>
__global__ void __launch_bounds__(STC_THREADS)
wb_sdf_train_tc_kernel(WbOct oc, WbSdf m, WbGridX gx, int nl, WbSdfTc P, WbGrid hg)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const int tid = threadIdx.x, r = tid >> 1, hh = tid & 1;
    const int H = P.H, Hp = P.Hp, IN = P.IN, nh = P.nh, pd = P.pd;
    // ---- decoder: fp16 weight packs (element (n, k) at (k/8)*(Hp*16) + n*16 + (k%8)*2, zero padded), fp16 biases, fp32 of fp16 wout
    {
        const float* p = m.params;
        int src = 0;
        for (int l = 0; l < nh; ++l) {
            const int I = l == 0 ? IN : H, Kp = l == 0 ? P.K0p : Hp;
            __half* pk = reinterpret_cast<__half*>(smem + P.w_off[l]);
            for (int e = tid; e < Hp * Kp; e += STC_THREADS) {
                const int n = e / Kp, k = e - n * Kp;
                pk[(k >> 3) * (Hp * 8) + n * 8 + (k & 7)] = __float2half_rn(n < H && k < I ? __ldg(p + src + n * I + k) : 0.0f);
            }
            src += H * I;
            __half* b = reinterpret_cast<__half*>(smem + P.b_off) + l * Hp;
            for (int e = tid; e < Hp; e += STC_THREADS) b[e] = __float2half_rn(e < H ? __ldg(p + src + e) : 0.0f);
            src += H;
        }
        float* wo = reinterpret_cast<float*>(smem + P.wo_off);
        for (int e = tid; e <= Hp; e += STC_THREADS) wo[e] = e < H ? sdf_h(__ldg(p + src + e)) : e == Hp ? sdf_h(__ldg(p + src + H)) : 0.0f;
        float* acc = reinterpret_cast<float*>(smem + P.acc_off);
        for (int e = tid; e < P.acc_l[nh] + H; e += STC_THREADS) acc[e] = 0.0f;
        // constant-one slab behind every input tile (feature 0 = 1: the bias column of the weight gradient); dY tile zeroed once
        // (slabs beyond Hp / 8 stay zero: each weight-gradient pass reads 8 slabs, the last one past Hp when Hp % 64 != 0)
        for (int l = 0; l < nh; ++l) {
            const int Kp = l == 0 ? P.K0p : Hp;
            if (tid < STC_ROWS) {
                uint4 one; one.x = 0x00003C00u; one.y = 0; one.z = 0; one.w = 0;
                *reinterpret_cast<uint4*>(smem + P.x_off[l] + (Kp / 8) * STC_SLAB + tid * 16) = one;
            }
        }
        uint4* dy4 = reinterpret_cast<uint4*>(smem + P.dy_off);
        for (int e = tid; e < (Hp + 63) / 64 * 8 * STC_SLAB / 16; e += STC_THREADS) dy4[e] = make_uint4(0, 0, 0, 0);
        __syncthreads();
    }
    const __half* bias = reinterpret_cast<const __half*>(smem + P.b_off);
    const float* wo = reinterpret_cast<const float*>(smem + P.wo_off);
    float* acc = reinterpret_cast<float*>(smem + P.acc_off);
    uint8_t* x0 = smem + P.x_off[0];
    uint8_t* dyt = smem + P.dy_off;
    float* gf = reinterpret_cast<float*>(smem + P.gf_off);
    float* dys = reinterpret_cast<float*>(smem + P.dys_off);
    const int GS = P.FD + 1;
    const uint32_t dyb = tc_smem_u32(dyt), wbase = tc_smem_u32(smem);
    float lsum = 0.0f, dsum = 0.0f;
    const int64_t ntiles = (P.N + STC_ROWS - 1) / STC_ROWS;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t i = tile * STC_ROWS + r;
        const bool valid = i < P.N;
        float cx = 0.0f, cy = 0.0f, cz = 0.0f;
        if (valid) { cx = __ldg(P.coords + 3 * i); cy = __ldg(P.coords + 3 * i + 1); cz = __ldg(P.coords + 3 * i + 2); }
        // ---- gather: decoder input row r in fp16 ----
        if (hh == 1) {
            float e[64];
            if (valid) sdf_embed(m.pos_mode, m.pos_freq, cx, cy, cz, e);
            for (int k = 0; k < pd; ++k) stc_store1(x0, r, k, valid ? e[k] : 0.0f);
        } else {
            float f[FT > 0 ? FT : WB_SDF_MAX_IN];
            if (valid) {
                if constexpr (HASH) sdf_hash_features(hg, nl, cx, cy, cz, f);
                else sdf_features<FT>(oc, m, nl, cx, cy, cz, f);
            }
            const int FDc = FT > 0 ? FT : P.FD;
#pragma unroll
            for (int k = 0; k < FDc; ++k) stc_store1(x0, r, pd + k, valid ? f[k] : 0.0f);
            for (int k = IN; k < P.K0p; ++k) stc_store1(x0, r, k, 0.0f);
        }
        // ---- hidden layers: relu(fp16(bias + X_l . W_l^T)) -> X_{l+1} ----
        for (int l = 0; l < nh; ++l) {
            tc_fence_smem_async();
            __syncthreads();
            const int Kp = l == 0 ? P.K0p : Hp;
            uint8_t* tn = smem + P.x_off[l + 1];
            stc_chain_n<0, 0>(Hp, tc_desc(wbase + P.x_off[l], STC_SLAB, 128), tc_desc(wbase + P.w_off[l], Hp * 16, 128), Kp / 16,
                              (2 * STC_SLAB) >> 4, (2 * Hp * 16) >> 4, bias + l * Hp, [&](auto& d) {
                constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                for (int q = 0; q < NR; q += 2) {
                    const int row = tc_frag_row(tid, q), col = tc_frag_col(tid, q);
                    *reinterpret_cast<uint32_t*>(tn + (col >> 3) * STC_SLAB + row * 16 + (col & 7) * 2) = tc_pack2_relu(d[q], d[q + 1]);
                }
            });
        }
        __syncthreads();
        // ---- output layer, loss, dY and dY_{nh-1} (row r: slabs hh, hh + 2, ...) ----
        const uint8_t* top = smem + P.x_off[nh];
        {
            float part = 0.0f;
            for (int sl = hh; sl < Hp / 8; sl += 2) {
                const uint4 q = *reinterpret_cast<const uint4*>(top + sl * STC_SLAB + r * 16);
                const __half* hv = reinterpret_cast<const __half*>(&q);
#pragma unroll
                for (int j = 0; j < 8; ++j) part = fmaf(wo[8 * sl + j], __half2float(hv[j]), part);
            }
            const float tot = part + __shfl_xor_sync(0xffffffffu, part, 1);
            const float y = sdf_h(wo[Hp] + tot);
            float dyv = 0.0f;
            if (valid) {
                const float dd = y - __ldg(P.gt + i);
                if (hh == 0) { lsum = fmaf(dd, dd, lsum); }
                dyv = sdf_h((P.inv_count * (2.0f * dd)) * P.scale);
            }
            if (hh == 0) { dys[r] = dyv; dsum += dyv; }
            for (int sl = hh; sl < Hp / 8; sl += 2) {
                const uint4 q = *reinterpret_cast<const uint4*>(top + sl * STC_SLAB + r * 16);
                const __half* hv = reinterpret_cast<const __half*>(&q);
                uint4 o; __half* ov = reinterpret_cast<__half*>(&o);
#pragma unroll
                for (int j = 0; j < 8; ++j) ov[j] = __float2half_rn(__half2float(hv[j]) > 0.0f ? dyv * wo[8 * sl + j] : 0.0f);
                *reinterpret_cast<uint4*>(dyt + sl * STC_SLAB + r * 16) = o;
            }
        }
        __syncthreads();
        if (tid < H) {                                     // dL/dwout[j] += sum_s dY_s h_s[j]
            const __half* hc = reinterpret_cast<const __half*>(top + (tid >> 3) * STC_SLAB) + (tid & 7);
            float a = acc[P.acc_l[nh] + tid];
            for (int s = 0; s < STC_ROWS; ++s) a = fmaf(dys[s], __half2float(hc[s * 8]), a);
            acc[P.acc_l[nh] + tid] = a;
        }
        // ---- backward through the hidden layers ----
        for (int l = nh - 1; l >= 0; --l) {
            tc_fence_smem_async();
            __syncthreads();
            const int I = l == 0 ? IN : H, Kp = l == 0 ? P.K0p : Hp;
            const uint32_t xb = wbase + P.x_off[l];
            float* al = acc + P.acc_l[l];
            for (int mb = 0; mb < Hp; mb += 64) {
                const uint64_t da = tc_desc(dyb + (uint32_t)(mb / 8) * STC_SLAB, 128, STC_SLAB);
                for (int nb = 0; nb < Kp; nb += 128) {
                    stc_chain_n<1, 1>(min(Kp - nb, 128), da, tc_desc(xb + (uint32_t)(nb / 8) * STC_SLAB, 128, STC_SLAB), STC_ROWS / 16, 256 >> 4,
                                      256 >> 4, nullptr, [&](auto& d) {
                        constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                        for (int q = 0; q < NR; ++q) {
                            const int o = mb + tc_frag_row(tid, q), k = nb + tc_frag_col(tid, q);
                            if (o < H && k < I) al[o * (I + 1) + k] += d[q];
                        }
                    });
                }
                stc_chain<8, 1, 1>(da, tc_desc(xb + (uint32_t)(Kp / 8) * STC_SLAB, 128, STC_SLAB), STC_ROWS / 16, 256 >> 4, 256 >> 4, nullptr, [&](auto& d) {
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int o = mb + tc_frag_row(tid, q);
                        if (o < H && tc_frag_col(tid, q) == 0) al[o * (I + 1) + I] += d[q];
                    }
                });
            }
            const uint64_t da = tc_desc(dyb, STC_SLAB, 128);
            const uint32_t wb = wbase + P.w_off[l];
            if (l > 0) {
                // dY_{l-1} = relu'(X_l) fp16(dY_l . W_l), written over dY_l (the chain has read it)
                const uint8_t* xt = smem + P.x_off[l];
                stc_chain_n<0, 1>(Hp, da, tc_desc(wb, 128, Hp * 16), Hp / 16, (2 * STC_SLAB) >> 4, 256 >> 4, nullptr, [&](auto& d) {
                    constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                    for (int q = 0; q < NR; q += 2) {
                        const int row = tc_frag_row(tid, q), col = tc_frag_col(tid, q);
                        const int off = (col >> 3) * STC_SLAB + row * 16 + (col & 7) * 2;
                        const __half2 h = *reinterpret_cast<const __half2*>(xt + off);
                        const float v0 = __low2float(h) > 0.0f ? d[q] : 0.0f, v1 = __high2float(h) > 0.0f ? d[q + 1] : 0.0f;
                        *reinterpret_cast<uint32_t*>(dyt + off) = tc_pack2(v0, v1);
                    }
                });
                continue;
            }
            // l == 0: the feature columns [pd, IN) of dX_0 = dY_0 . W0 in fp32, unscaled, -> gf [64][FD + 1]
            for (int nb = pd & ~15; nb < P.K0p; nb += 128) {
                stc_chain_n<0, 1>(min(P.K0p - nb, 128), da, tc_desc(wb + (uint32_t)(nb / 8) * (Hp * 16), 128, Hp * 16), Hp / 16, (2 * STC_SLAB) >> 4,
                                  256 >> 4, nullptr, [&](auto& d) {
                    constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                    for (int q = 0; q < NR; ++q) {
                        const int k = nb + tc_frag_col(tid, q);
                        if (k >= pd && k < IN) gf[tc_frag_row(tid, q) * GS + (k - pd)] = d[q] * P.inv_scale;
                    }
                });
            }
        }
        __syncthreads();
        if (hh == 0 && valid) {
            const float* g = gf + r * GS;
            if constexpr (HASH) sdf_hash_scatter(hg, gx.gptr[0], nl, cx, cy, cz, [&](int f) { return g[f]; });
            else wb_featx_scatter(gx, cx, cy, cz, [&](int f) { return g[f]; });
        }
        __syncthreads();
    }
    // ---- flush: the CTA's decoder gradients (unscaled), then the loss and dL/dbout reduced over the CTA ----
    float* gp = P.gparams;
    int src = 0;
    for (int l = 0; l <= nh; ++l) {
        const int I = l == nh ? 0 : l == 0 ? IN : H, n = l == nh ? H : H * (I + 1);
        const float* al = acc + P.acc_l[l];
        for (int e = tid; e < n; e += STC_THREADS) {
            const float v = al[e];
            if (v == 0.0f) continue;
            if (l == nh) atomicAdd(gp + src + e, v * P.inv_scale);
            else {
                const int o = e / (I + 1), k = e - o * (I + 1);
                atomicAdd(gp + (k < I ? src + o * I + k : src + H * I + o), v * P.inv_scale);
            }
        }
        src += l == nh ? H : H * I + H;
    }
    float* red = reinterpret_cast<float*>(smem + P.red_off);
    lsum = wb_warp_sum(lsum); dsum = wb_warp_sum(dsum);
    if ((tid & 31) == 0) { red[2 * (tid >> 5)] = lsum; red[2 * (tid >> 5) + 1] = dsum; }
    __syncthreads();
    if (tid == 0) {
        float l = 0.0f, d = 0.0f;
        for (int w = 0; w < STC_THREADS / 32; ++w) { l += red[2 * w]; d += red[2 * w + 1]; }
        if (l != 0.0f) atomicAdd(P.loss, l * P.inv_count);
        if (d != 0.0f) atomicAdd(gp + src, d * P.inv_scale);
    }
}

// replaces, for one loss LOD under enable_amp: neural_sdf.py:120-155 (grid interpolate, cat, BasicDecoder's fp16 nn.Linear chain),
// sdf_trainer.py:90-116 (the L2 loss) and :122-124 (loss.backward(): the fp16 GEMMs of the decoder backward and the grid scatter)
extern "C" int64_t wb_sdf_train_tc_smem_bytes(const wb_sdf_desc* nef)
{
    WbSdf m; WbGrid hg; if (wb_make_sdf(nef, &m, &hg)) return -1;
    WbSdfTc P;
    return sdf_tc_plan(m, &P);
}

// replaces, for one loss LOD of SDFTrainer.step under torch.cuda.amp.autocast (base_trainer.py:338, sdf_trainer.py:65-124): the
// fp16 forward of NeuralSDF.sdf (neural_sdf.py:120-155), the loss (sdf_trainer.py:90-116) and loss.backward() (:122-124)
extern "C" int wb_sdf_train_tc(const wb_octree* oct, const wb_sdf_desc* nef, int32_t lod_idx, const float* coords, const float* sdf_gt, int64_t N,
                               float inv_count, float* const* grad_feats, float* grad_params, float* loss_out, wb_stream s)
{
    WbSdf m; WbGrid hg; int rc = wb_make_sdf(nef, &m, &hg); if (rc) return rc;
    const bool hash = hg.table != nullptr;
    WbSdfTc P; const int smem = sdf_tc_plan(m, &P);
    WB_CHECK_ARG(smem > 0, "fp16 weights, fp32 gradient accumulators and one 64-sample tile exceed shared memory (wb_sdf_train_tc_smem_bytes < 0)");
    rc = sdf_check_lod(m, hash, lod_idx); if (rc) return rc;
    WB_CHECK_ARG((N == 0 || (coords && sdf_gt)) && grad_feats && grad_params && loss_out && N >= 0, "null pointer");
    WB_CHECK_ARG(std::isfinite(inv_count) && inv_count >= 0.0f, "inv_count must be finite and >= 0");
    if (N == 0) return WB_OK;
    WbOct oc; WbGridX gx; rc = sdf_grad_target(oct, m, hash, lod_idx, grad_feats, false, &oc, &gx); if (rc) return rc;
    // loss scale: a power of two with inv_count * scale in [0.5, 1), so dY ~ 2 (y - gt) whatever the batch size
    int e = 0;
    if (inv_count > 0.0f) frexpf(inv_count, &e);
    P.coords = coords; P.gt = sdf_gt; P.N = N; P.gparams = grad_params; P.loss = loss_out;
    P.inv_count = inv_count; P.scale = ldexpf(1.0f, -e); P.inv_scale = ldexpf(1.0f, e);
    int nl = lod_idx + 1;
    const void* kern = hash ? (const void*)wb_sdf_train_tc_kernel<0, true>
                     : (m.multiscale == 1 && m.F == 16) ? (const void*)wb_sdf_train_tc_kernel<16, false> : (const void*)wb_sdf_train_tc_kernel<0, false>;
    void* args[] = { &oc, &m, &gx, &nl, &P, &hg };
    return sdf_train_launch(kern, args, STC_THREADS, smem, N, STC_ROWS, (cudaStream_t)s);
}
