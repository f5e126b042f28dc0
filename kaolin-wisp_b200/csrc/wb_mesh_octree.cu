// wb_mesh_octree.cu -- the occupancy of wisp.ops.spc.mesh_to_octree (wisp/ops/spc/conversions.py:91-109, sampler
// wisp/ops/mesh/sample_surface.py, random_face.py, area_weighted_distribution.py) without materialising a sample.
//
// The reference draws num_samples faces from Categorical(area), a point on each with u = sqrt(rand), v = rand, appends a jittered copy
// of every point, quantizes all of them (spc.quantize_points) and builds the octree of the distinct cells.  Here one thread iteration
// does the same for one sample and sets the bits of its two cells in a dense occupancy bitmask; the octree bytes are built from the set
// bits by the caller (spc.points_to_octree).  The arithmetic is the reference's, op by op (explicit __f*_rn: no FMA contraction); the
// random stream is this package's counter-based one (DESIGN.md "Sampling contract"), so the distribution is the reference's, the
// draws are not torch's.
#include "wb_common.cuh"

namespace {

constexpr int kMotThreads = 256;

// Draw d of sample i: a counter-based stream keyed by (seed, 64-bit sample index, draw number).  For a fixed seed and high word the
// key is a bijection of the low word, so the 2^32 samples of one high word never share a key.
__device__ __forceinline__ uint32_t mot_key(uint32_t seed, uint64_t i)
{
    return wb_mix32(wb_mix32(seed + (uint32_t)i * 0x9E3779B1u) ^ ((uint32_t)(i >> 32) * 0xC2B2AE35u + 0x27D4EB2Fu));
}
__device__ __forceinline__ uint32_t mot_draw(uint32_t key, uint32_t d) { return wb_mix32(key ^ (d * 0x85EBCA77u + 0x165667B1u)); }
// torch.rand's float32: a multiple of 2^-24 in [0, 1)
__device__ __forceinline__ float mot_u24(uint32_t h) { return __uint2float_rn(h >> 8) * (1.0f / 16777216.0f); }

// spc.quantize_points of one coordinate: floor(clamp(res * (x + 1) / 2, 0, res - 1)) in fp32 (res * and / 2 are exact)
__device__ __forceinline__ uint32_t mot_quantize(float x, float res)
{
    const float q = __fmul_rn(__fmul_rn(res, __fadd_rn(x, 1.0f)), 0.5f);
    return (uint32_t)floorf(fminf(fmaxf(q, 0.0f), res - 1.0f));
}

__device__ __forceinline__ void mot_set(uint32_t* __restrict__ bits, uint32_t x, uint32_t y, uint32_t z, int level)
{
    const uint32_t idx = (x << (2 * level)) | (y << level) | z;
    const uint32_t bit = 1u << (idx & 31);
    // almost every sample lands on a set bit: read it from L2 first and skip the atomic
    if (!(__ldcg(bits + (idx >> 5)) & bit)) atomicOr(bits + (idx >> 5), bit);
}

__global__ void __launch_bounds__(kMotThreads) wb_mesh_octree_kernel(const float* __restrict__ tris, const double* __restrict__ cdf, int64_t T,
                                                                    uint64_t n, int level, uint32_t seed, uint32_t* __restrict__ bits)
{
    const double total = __ldg(cdf + T);
    const float res = (float)(1 << level);
    const float h = __uint_as_float((uint32_t)(126 - level) << 23);          // 1 / 2^(level + 1)
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t key = mot_key(seed, i);
        // face: inverse CDF of the fp32 areas, at a 53-bit uniform; the face f with cdf[f] <= target < cdf[f + 1] (so never one of zero area)
        const uint64_t u53 = ((uint64_t)mot_draw(key, 0) << 21) | (mot_draw(key, 1) >> 11);
        const double target = (double)u53 * 0x1p-53 * total;
        int64_t lo = 0, hi = T;                                                // first index j in [1, T] with cdf[j] > target, minus 1
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(cdf + mid + 1) > target) hi = mid; else lo = mid + 1;
        }
        int64_t f = lo;
        if (f == T) {                                                          // target rounded up to the total: the last face of nonzero area
            f = T - 1;
            while (f > 0 && !(__ldg(cdf + f + 1) > __ldg(cdf + f))) --f;
        }
        const float r1 = mot_u24(mot_draw(key, 2)), v = mot_u24(mot_draw(key, 3));
        const float u = __fsqrt_rn(r1);
        const float wa = __fsub_rn(1.0f, u), wb = __fmul_rn(u, __fsub_rn(1.0f, v)), wc = __fmul_rn(u, v);
        const float* t = tris + f * 9;
        uint32_t q[3], qj[3];
        #pragma unroll
        for (int k = 0; k < 3; ++k) {
            // (1 - u) * a + (u * (1 - v)) * b + u * v * c, left to right as torch evaluates it
            const float x = __fadd_rn(__fadd_rn(__fmul_rn(wa, __ldg(t + k)), __fmul_rn(wb, __ldg(t + 3 + k))), __fmul_rn(wc, __ldg(t + 6 + k)));
            // x + (rand * 2 - 1) * (1 / 2^(level + 1))  (conversions.py:105-106)
            const float j = __fmul_rn(__fsub_rn(__fmul_rn(mot_u24(mot_draw(key, 4 + k)), 2.0f), 1.0f), h);
            q[k] = mot_quantize(x, res);
            qj[k] = mot_quantize(__fadd_rn(x, j), res);
        }
        mot_set(bits, q[0], q[1], q[2], level);
        mot_set(bits, qj[0], qj[1], qj[2], level);
    }
}

}  // namespace

extern "C" int wb_mesh_octree_bits(const float* tris, const double* cdf, int64_t num_triangles, int64_t num_samples, int32_t level,
                                   uint32_t seed, uint32_t* bits, wb_stream s)
{
    WB_CHECK_ARG(level >= 1 && level <= 10, "level must be 1..10 (the dense bitmask's limit)");
    WB_CHECK_ARG(num_triangles >= 1, "no triangles");
    WB_CHECK_ARG(num_samples >= 0, "num_samples must be >= 0");
    if (num_samples == 0) return WB_OK;
    WB_CHECK_ARG(tris && cdf && bits, "null pointer");
    const int64_t blocks = std::min<int64_t>((num_samples + kMotThreads - 1) / kMotThreads, 8 * (int64_t)wb_num_sms());
    wb_mesh_octree_kernel<<<(unsigned)blocks, kMotThreads, 0, (cudaStream_t)s>>>(tris, cdf, num_triangles, (uint64_t)num_samples, level,
                                                                                 seed, bits);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
