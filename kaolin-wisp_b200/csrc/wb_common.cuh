// wb_common.cuh -- shared device/host helpers of libwispb200 (sm_90a only).
//
// Numerical contracts (bit-exact parts) are stated once here and mirrored by the CPU oracle
// (oracle/wisp_oracle.c).  Reference citations are relative to the kaolin-wisp checkout.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/wispb200.h"

// ---------------------------------------------------------------------------------------------
// error handling / bookkeeping (host)
// ---------------------------------------------------------------------------------------------
void wb_set_error(const char* fmt, ...);
void wb_count_launch(int n = 1);

#define WB_CHECK_ARG(cond, msg)                                                     \
    do { if (!(cond)) { wb_set_error("%s: %s", __func__, msg); return WB_ERR_INVALID; } } while (0)
#define WB_CUDA(call)                                                               \
    do { cudaError_t e__ = (call); if (e__ != cudaSuccess) {                        \
        wb_set_error("%s: %s failed: %s", __func__, #call, cudaGetErrorString(e__)); return WB_ERR_CUDA; } } while (0)
#define WB_LAUNCH_CHECK()                                                           \
    do { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) {            \
        wb_set_error("%s: kernel launch failed: %s", __func__, cudaGetErrorString(e__)); return WB_ERR_CUDA; } \
        wb_count_launch(); } while (0)

inline int wb_round_up(int v, int m) { return (v + m - 1) / m * m; }
inline int64_t wb_align256(int64_t bytes) { return (bytes + 255) / 256 * 256; }       // workspace carve-outs
// width of a position / view embedding (positional_embedder.py:51-66): mode 0 none, 1 identity, 2 sin/cos bands, 3 both
inline int wb_embed_dim(int mode, int freq) { return mode == 0 ? 0 : mode == 1 ? 3 : mode == 2 ? 6 * freq : 3 + 6 * freq; }

int wb_num_sms();          // multiprocessor count of the CURRENT device (cached per device)
int wb_cur_device();       // cudaGetDevice
// Lets `kernel` launch with `bytes` of dynamic shared memory on the current device: raises its cudaFuncAttributeMaxDynamicSharedMemorySize
// when the limit set so far for this (kernel, device) is lower, never lowers it.  Thread-safe: a call that needs less than another
// thread's launch of the same kernel cannot undercut that launch between its attribute set and the launch itself.  The attribute is a
// driver call that can wait behind other driver work (e.g. an NVML poll): it runs once per (kernel, device, larger size), not per launch.
cudaError_t wb_allow_smem_fn(const void* kernel, int64_t bytes);
template <class K> cudaError_t wb_allow_smem(K* kernel, int64_t bytes) { return wb_allow_smem_fn((const void*)kernel, bytes); }
inline cudaError_t wb_allow_smem(const void* kernel, int64_t bytes) { return wb_allow_smem_fn(kernel, bytes); }

// ---------------------------------------------------------------------------------------------
// Jitter contract: counter-based stream keyed by (seed, ray, step).
// The reference draws torch.rand(R, n) unseeded (octree_as.py:273); see DESIGN.md.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t wb_mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x21f0aaadu;
    x ^= x >> 15; x *= 0x735a2d97u;
    x ^= x >> 15;
    return x;
}
__host__ __device__ __forceinline__ uint32_t wb_ray_key(uint32_t seed, uint32_t ray) {
    return wb_mix32(seed + ray * 0x9E3779B1u);
}
__device__ __forceinline__ float wb_jitter(uint32_t ray_key, uint32_t step) {
    uint32_t h = wb_mix32(ray_key ^ (step * 0x85EBCA77u + 0x165667B1u));
    return __uint2float_rn(h >> 8) * (1.0f / 16777216.0f);
}

// ---------------------------------------------------------------------------------------------
// Candidate depth of OctreeAS._raymarch_ray (octree_as.py:272-277), op by op as the reference's
// separate torch kernels evaluate it (no contraction across ops):
//   lin = torch.linspace(0,1,n)[i]   (ATen: start+step*i below n/2, end-step*(n-1-i) above, FMA-contracted)
//   d   = (lin + jit/n) * (far-near) + near
// ---------------------------------------------------------------------------------------------
struct WbMarch {
    const float* origins; const float* dirs;
    const float* near_v; const float* far_v;
    const float* jitter;
    float near_s, range_s;       // scalar near and (float)(double(far)-double(near))
    float step;                  // 1/(n-1) (float division), 0 for n == 1
    float inv_n; int n_pow2;     // jit/n == jit*inv_n exactly when n is a power of two
    int n; uint32_t seed;
    int64_t R;
};
__device__ __forceinline__ float wb_linspace01(int i, int n, float step) {
    if (n == 1) return 0.0f;
    return (i < n / 2) ? __fmaf_rn(step, (float)i, 0.0f) : __fmaf_rn(-step, (float)(n - 1 - i), 1.0f);
}
__device__ __forceinline__ float wb_depth(const WbMarch& m, int64_t r, uint32_t key, int i, float nearv, float range) {
    float jit = m.jitter ? __ldg(m.jitter + r * m.n + i) : wb_jitter(key, (uint32_t)i);
    float q = m.n_pow2 ? __fmul_rn(jit, m.inv_n) : __fdiv_rn(jit, (float)m.n);
    float d = __fadd_rn(wb_linspace01(i, m.n, m.step), q);
    d = __fmul_rn(d, range);
    d = __fadd_rn(d, nearv);
    return d;
}
__device__ __forceinline__ void wb_ray_range(const WbMarch& m, int64_t r, float& nearv, float& range) {
    if (m.near_v) { nearv = m.near_v[r]; range = __fsub_rn(m.far_v[r], nearv); }
    else { nearv = m.near_s; range = m.range_s; }
}
// torch.addcmul(origins, dirs, depth) (octree_as.py:283): a + alpha*b*c == fma(b, c, a)
__device__ __forceinline__ float wb_addcmul(float o, float d, float t) { return __fmaf_rn(d, t, o); }
// the point at depth t of ray `ray`, as above
__device__ __forceinline__ float3 wb_ray_point(const float* origins, const float* dirs, int64_t ray, float t) {
    return make_float3(wb_addcmul(__ldg(origins + 3 * ray), __ldg(dirs + 3 * ray), t),
                       wb_addcmul(__ldg(origins + 3 * ray + 1), __ldg(dirs + 3 * ray + 1), t),
                       wb_addcmul(__ldg(origins + 3 * ray + 2), __ldg(dirs + 3 * ray + 2), t));
}
// position of sample record s.  A kernel that holds the ray index already passes it to wb_ray_point: the compiler does not merge a
// second load of rec_ray[s] across barriers.
__device__ __forceinline__ float3 wb_sample_pos(const float* origins, const float* dirs, const int32_t* rec_ray, const float* rec_t, int64_t s) {
    const int64_t ray = __ldg(rec_ray + s);
    return wb_ray_point(origins, dirs, ray, __ldg(rec_t + s));
}

// ---------------------------------------------------------------------------------------------
// Octree occupancy  [KAOLIN-EXT unbatched_query, SURVEY.md Appendix A]
//   q = floor(2^L (x+1)/2) evaluated exactly; miss outside [0, 2^L-1].
// ---------------------------------------------------------------------------------------------
struct WbOct {
    const uint8_t* octree; const int32_t* prefix; const uint32_t* bits;
    int level; int use_bits;
    float h, inv_h, maxq;        // 2^(L-1), 2^-(L-1), 2^L - 1
    int has_bbox; float blo[3], bhi[3];   // occupied extent, already widened by the safety margin
    const uint32_t* coarse; int clevel;   // dilated coarse occupancy (wb_octree_build_coarse) or nullptr
    float ch, cmax;                       // 2^(clevel-1), 2^clevel - 1
};
__device__ __forceinline__ bool wb_quantize(float x, float h, float inv_h, float maxq, int& q) {
    float yf = __fmaf_rn(x, h, h);
    float kf = floorf(yf);
    if (yf == kf && x < (kf - h) * inv_h) kf -= 1.0f;
    if (!(kf >= 0.0f) || kf > maxq) return false;
    q = (int)kf; return true;
}
// point index of the level-L cell containing (qx,qy,qz), -1 if empty; optional parents[0..L]
__device__ __forceinline__ int wb_descend(const uint8_t* __restrict__ octree, const int32_t* __restrict__ prefix,
                                          int qx, int qy, int qz, int L, int32_t* parents, int stride) {
    int node = 0;
    if (parents) parents[0] = 0;
    for (int l = 0; l < L; ++l) {
        int d = L - 1 - l;
        int ci = (((qx >> d) & 1) << 2) | (((qy >> d) & 1) << 1) | ((qz >> d) & 1);
        uint32_t b = __ldg(octree + node);
        if (!(b & (1u << ci))) return -1;
        node = __ldg(prefix + node) + __popc(b & ((2u << ci) - 1u));
        if (parents) parents[(l + 1) * stride] = node;
    }
    return node;
}
__device__ __forceinline__ bool wb_occupied(const WbOct& o, float x, float y, float z) {
    int qx, qy, qz;
    if (!wb_quantize(x, o.h, o.inv_h, o.maxq, qx)) return false;
    if (!wb_quantize(y, o.h, o.inv_h, o.maxq, qy)) return false;
    if (!wb_quantize(z, o.h, o.inv_h, o.maxq, qz)) return false;
    if (o.use_bits) {
        uint32_t idx = ((uint32_t)qx << (2 * o.level)) | ((uint32_t)qy << o.level) | (uint32_t)qz;
        return (__ldg(o.bits + (idx >> 5)) >> (idx & 31)) & 1u;
    }
    return wb_descend(o.octree, o.prefix, qx, qy, qz, o.level, nullptr, 0) >= 0;
}

// ---------------------------------------------------------------------------------------------
// Hash grid  (wisp/csrc/ops/hashgrid_interpolate_cuda.cu:38-79, hash_utils.cuh:18-40)
// ---------------------------------------------------------------------------------------------
struct WbGrid {
    const float* table;
    int L, F; uint32_t Tmask;            // T is a power of two (2^codebook_bitwidth)
    int multiscale, lod_idx;
    int res[WB_MAX_LODS];
    float hres[WB_MAX_LODS];             // res/2
    float hi[WB_MAX_LODS];               // (float)(res-1-1e-5)
    int dense[WB_MAX_LODS];              // res^3 < T && res^2 < T && res < T
    int64_t begin[WB_MAX_LODS + 1];
};
__device__ __forceinline__ uint32_t wb_hash_idx(int x, int y, int z, int res, uint32_t Tmask, int dense) {
    if (dense) return (uint32_t)(x + y * res + z * res * res);
    uint32_t h = ((uint32_t)x) ^ ((uint32_t)y * 2654435761u) ^ ((uint32_t)z * 805459861u);
    return h & Tmask;
}
// The 8 corner entries of cell (px,py,pz), corner j = (x + (j>>2&1), y + (j>>1&1), z + (j&1)): the same values as 8 calls of
// wb_hash_idx, evaluated with one multiply per axis.  The level kind is warp-uniform, so this is a branch, not a select: the
// straightforward form made ptxas compute BOTH index kinds for all 8 corners with the products and the constant loads repeated
// (~100 instructions per level in the gather and the scatter).
// Dense levels: from res 258 on the clamp bound fl(res - 1 - 1e-5) is res - 1 itself, so a coordinate at +1 lands on cell res - 1
// with weight 0 on its +1 corner, which would be row res on that axis -- outside the level's res^3 rows (past the table's end on the
// last level).  That corner keeps the cell's own row instead: its coefficient is 0, so finite tables give the same features.
__device__ __forceinline__ void wb_corner_indices(const WbGrid& g, int l, int px, int py, int pz, uint32_t idx[8]) {
    if (g.dense[l]) {
        const uint32_t r1 = (uint32_t)g.res[l], r2 = r1 * r1, top = r1 - 1u;
        const uint32_t b = (uint32_t)px + (uint32_t)py * r1 + (uint32_t)pz * r2;
        const uint32_t sx = (uint32_t)px < top ? 1u : 0u, sy = (uint32_t)py < top ? r1 : 0u, sz = (uint32_t)pz < top ? r2 : 0u;
#pragma unroll
        for (int j = 0; j < 8; ++j) idx[j] = b + ((j & 4) ? sx : 0u) + ((j & 2) ? sy : 0u) + ((j & 1) ? sz : 0u);
    } else {
        const uint32_t m = g.Tmask;
        const uint32_t x0 = (uint32_t)px, x1 = x0 + 1u;
        const uint32_t y0 = (uint32_t)py * 2654435761u, y1 = y0 + 2654435761u;
        const uint32_t z0 = (uint32_t)pz * 805459861u, z1 = z0 + 805459861u;
#pragma unroll
        for (int j = 0; j < 8; ++j) idx[j] = (((j & 4) ? x1 : x0) ^ ((j & 2) ? y1 : y0) ^ ((j & 1) ? z1 : z0)) & m;
    }
}
// position math: the reference evaluates res*(c*0.5+0.5) in double and rounds to float
// (hashgrid_interpolate_cuda.cu:40-42); fmaf(c, res/2, res/2) rounds the same exact value once.
__device__ __forceinline__ void wb_cell(float c, float hres, float hi, int& pos, float& w, float& iw) {
    float x = __fmaf_rn(c, hres, hres);
    x = fmaxf(0.0f, fminf(hi, x));
    float p = floorf(x);
    pos = (int)p; w = x - p; iw = 1.0f - w;
}
__device__ __forceinline__ void wb_corner_setup(const WbGrid& g, int l, float cx, float cy, float cz,
                                                uint32_t idx[8], float coef[8]) {
    int px, py, pz; float wx, wy, wz, ix, iy, iz;
    wb_cell(cx, g.hres[l], g.hi[l], px, wx, ix);
    wb_cell(cy, g.hres[l], g.hi[l], py, wy, iy);
    wb_cell(cz, g.hres[l], g.hi[l], pz, wz, iz);
    // coefficient order c000, c001, ... z fastest (cu:49-56); products left to right
    float xy00 = ix * iy, xy01 = ix * wy, xy10 = wx * iy, xy11 = wx * wy;
    coef[0] = xy00 * iz; coef[1] = xy00 * wz; coef[2] = xy01 * iz; coef[3] = xy01 * wz;
    coef[4] = xy10 * iz; coef[5] = xy10 * wz; coef[6] = xy11 * iz; coef[7] = xy11 * wz;
    wb_corner_indices(g, l, px, py, pz, idx);
}

int wb_make_grid(const wb_nef_desc* d, WbGrid* g);     // host: validate + derive per-level constants
// host: the decoders of a wb_nef_desc as the fp32 (WbMlp) and tensor-core (WbTc) shade planners both read them, before each applies
// its own head-width limit and padding; a layer narrower than 1 or wider than max_width is refused with the message width_msg
struct WbDecoders {
    int nl_d, nl_c;                                                  // linear layers: density, colour
    int I[2 * WB_MAX_LAYERS], O[2 * WB_MAX_LAYERS];                  // layer l's widths, the density layers first
    int src_w[2 * WB_MAX_LAYERS], src_b[2 * WB_MAX_LAYERS];          // offsets into the packed nn.Linear parameter vectors (b = -1: no bias)
    int feat_dim, pos_dim, view_dim;                                 // grid features, position and view embedding widths
};
int wb_make_decoders(const wb_nef_desc* d, int max_width, const char* width_msg, WbDecoders* dec);
int wb_make_march(const wb_rays* rays, int n, const float* jitter, uint32_t seed, WbMarch* m);
int wb_make_oct(const wb_octree* o, int level, WbOct* out);

// ---------------------------------------------------------------------------------------------
// small device utilities
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float wb_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float wb_warp_incl_scan(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { float t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    return v;
}
