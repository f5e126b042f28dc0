// wb_spc.cu -- SPC (octree) helpers: dense occupancy bitmasks, point-in-octree query.
// Replaces kaolin.ops.spc.unbatched_query at the call sites
// wisp/ops/spc/conversions.py:84-87 and wisp/accelstructs/octree_as.py:146-163.
#include "wb_common.cuh"

__global__ void wb_build_bits_kernel(const int16_t* __restrict__ pts, int64_t n, int level, uint32_t* __restrict__ bits)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint16_t)pts[i * 3], y = (uint16_t)pts[i * 3 + 1], z = (uint16_t)pts[i * 3 + 2];
    uint32_t idx = (x << (2 * level)) | (y << level) | z;
    atomicOr(bits + (idx >> 5), 1u << (idx & 31));
}

extern "C" int wb_octree_build_bits(const int16_t* level_points, int64_t num_points, int32_t level, uint32_t* bits, wb_stream s)
{
    WB_CHECK_ARG(level_points && bits, "null pointer");
    WB_CHECK_ARG(level >= 0 && level <= 10, "bitmask supported up to level 10");
    if (num_points == 0) return WB_OK;
    wb_build_bits_kernel<<<(unsigned)((num_points + 255) / 256), 256, 0, (cudaStream_t)s>>>(level_points, num_points, level, bits);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

__global__ void wb_build_coarse_kernel(const int16_t* __restrict__ pts, int64_t n, int shift, int cl, uint32_t* __restrict__ cbits)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int cx = (int)(uint16_t)pts[i * 3] >> shift, cy = (int)(uint16_t)pts[i * 3 + 1] >> shift, cz = (int)(uint16_t)pts[i * 3 + 2] >> shift;
    const int cres = 1 << cl;
    for (int ax = -1; ax <= 1; ++ax) for (int ay = -1; ay <= 1; ++ay) for (int az = -1; az <= 1; ++az) {
        const int x = cx + ax, y = cy + ay, z = cz + az;
        if (x < 0 || y < 0 || z < 0 || x >= cres || y >= cres || z >= cres) continue;
        const uint32_t idx = ((uint32_t)x << (2 * cl)) | ((uint32_t)y << cl) | (uint32_t)z;
        const uint32_t bit = 1u << (idx & 31);
        if (!(cbits[idx >> 5] & bit)) atomicOr(cbits + (idx >> 5), bit);
    }
}

extern "C" int wb_octree_build_coarse(const int16_t* level_points, int64_t num_points, int32_t level, int32_t coarse_level,
                                      uint32_t* coarse_bits, wb_stream s)
{
    WB_CHECK_ARG(level_points && coarse_bits, "null pointer");
    WB_CHECK_ARG(level >= 1 && level <= 10 && coarse_level >= 1 && coarse_level < level, "need 1 <= coarse_level < level <= 10");
    if (num_points == 0) return WB_OK;
    wb_build_coarse_kernel<<<(unsigned)((num_points + 255) / 256), 256, 0, (cudaStream_t)s>>>(level_points, num_points, level - coarse_level,
                                                                                            coarse_level, coarse_bits);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// OctreeAS.query -> unbatched_query(octree, prefix, coords, level, with_parents) (octree_as.py:146-163)
__global__ void wb_query_kernel(WbOct o, const float* __restrict__ coords, int64_t N, int with_parents, int32_t* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float x = coords[i * 3], y = coords[i * 3 + 1], z = coords[i * 3 + 2];
    int L = o.level; int qx, qy, qz;
    bool in = wb_quantize(x, o.h, o.inv_h, o.maxq, qx) && wb_quantize(y, o.h, o.inv_h, o.maxq, qy) && wb_quantize(z, o.h, o.inv_h, o.maxq, qz);
    if (with_parents) {
        int32_t* p = out + i * (L + 1);
        for (int l = 0; l <= L; ++l) p[l] = -1;
        if (in) wb_descend(o.octree, o.prefix, qx, qy, qz, L, p, 1);
    } else {
        out[i] = in ? wb_descend(o.octree, o.prefix, qx, qy, qz, L, nullptr, 0) : -1;
    }
}

extern "C" int wb_query(const wb_octree* oct, const float* coords, int64_t N, int32_t level, int32_t with_parents,
                        int32_t* out, wb_stream s)
{
    WbOct o; int rc = wb_make_oct(oct, level, &o); if (rc) return rc;
    if (N == 0) return WB_OK;
    WB_CHECK_ARG(coords && out, "null pointer");
    wb_query_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)s>>>(o, coords, N, with_parents, out);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// NeuralRadianceField.prune (wisp/models/nefs/nerf.py:175-212): the two elementwise halves around the density probe.
//   wb_prune_samples: one probe point per finest-level cell, samples = ((points + u) / res) * 2 - 1 (:189-192), op by op in
//     fp32 as the reference's torch kernels, and a uniform direction on the sphere (wisp/ops/geometric.py:25-39; the density
//     does not depend on it).  u: explicit [N,3] tensor (parity tests replay the reference's draw) or the counter-based stream
//     keyed by (seed, cell, axis) -- the same seed on every rank gives the same probe points, so pruned octrees agree across
//     GPUs without a broadcast.
//   wb_prune_update: occupancy = max(density, occupancy * decay) (:186,:196) with torch.max's NaN propagation, keep = occupancy >
//     min_density (:198).
// The probe itself is the fused shade kernel (wb_rf_shade_fwd with the probe points as zero-length rays).
// ---------------------------------------------------------------------------------------------------------------
__global__ void wb_prune_samples_kernel(const int16_t* __restrict__ points, int64_t N, float res, const float* __restrict__ u, uint32_t seed,
                                        float* __restrict__ samples, float* __restrict__ dirs, float* __restrict__ rec_t, int32_t* __restrict__ rec_ray)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const uint32_t key = wb_ray_key(seed, (uint32_t)i);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float ua = u ? __ldg(u + 3 * i + a) : wb_jitter(key, (uint32_t)a);
        float v = __fadd_rn((float)points[3 * i + a], ua);
        v = __fdiv_rn(v, res);
        samples[3 * i + a] = __fsub_rn(__fmul_rn(v, 2.0f), 1.0f);
    }
    const float u0 = wb_jitter(key, 3u), u1 = wb_jitter(key, 4u);
    const float z = 1.0f - 2.0f * u0, r = sqrtf(fmaxf(1.0f - z * z, 0.0f)), phi = 6.283185307179586f * u1;
    dirs[3 * i] = r * cosf(phi); dirs[3 * i + 1] = r * sinf(phi); dirs[3 * i + 2] = z;
    rec_t[i] = 0.0f; rec_ray[i] = (int32_t)i;                      // probe point i = ray i at depth 0: fma(dir, 0, origin) == origin
}
extern "C" int wb_prune_samples(const int16_t* points, int64_t N, int32_t level, const float* u, uint32_t seed,
                                float* samples, float* dirs, float* rec_t, int32_t* rec_ray, wb_stream s)
{
    if (N == 0) return WB_OK;
    WB_CHECK_ARG(points && samples && dirs && rec_t && rec_ray, "null pointer");
    WB_CHECK_ARG(level >= 0 && level <= 15 && N < ((int64_t)1 << 31), "level / N out of range");
    wb_prune_samples_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)s>>>(points, N, (float)(1 << level), u, seed, samples, dirs, rec_t, rec_ray);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
__global__ void wb_prune_update_kernel(const float4* __restrict__ shaded, int64_t N, float decay, float min_density,
                                       float* __restrict__ occupancy, uint8_t* __restrict__ keep)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    // torch.stack([density, occupancy * decay], -1).max(-1) propagates a NaN from either side (fmaxf would drop it): a cell whose
    // density or occupancy has diverged stores NaN and is not kept
    const float d = __ldg(shaded + i).w, od = __fmul_rn(occupancy[i], decay);
    const float occ = (isnan(d) || isnan(od)) ? __fadd_rn(d, od) : fmaxf(d, od);
    occupancy[i] = occ;
    keep[i] = occ > min_density ? 1 : 0;
}
extern "C" int wb_prune_update(const float* shaded, int64_t N, float decay, float min_density, float* occupancy, uint8_t* keep, wb_stream s)
{
    if (N == 0) return WB_OK;
    WB_CHECK_ARG(shaded && occupancy && keep, "null pointer");
    wb_prune_update_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)s>>>(reinterpret_cast<const float4*>(shaded), N, decay, min_density, occupancy, keep);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
