// wb_raytrace.cu -- OctreeAS.raytrace and the 'voxel' / 'uniform' samplers built on it.
//   OctreeAS.raytrace          -> kaolin.render.spc.unbatched_raytrace       (wisp/accelstructs/octree_as.py:165-186)
//   OctreeAS._raymarch_voxel   + sample_from_depth_intervals                 (octree_as.py:188-245, ops/spc/sampling.py:35-71)
//   OctreeAS._raymarch_uniform + wisp._C.ops.uniform_sample_cuda              (octree_as.py:311-374, csrc/ops/uniform_sample_cuda.cu:18-98)
//
// Kaolin expands all rays level by level with a CUB scan + reallocation per level.  Here one thread walks one ray depth
// first through the octree with the direction-sign child order (i ^ mask), which yields the nuggets already sorted front to
// back, so a count pass + scan + fill pass is all that is needed and nothing is sorted or reallocated.
// Kaolin's source is not in the reference checkout: the nugget definition (positive-length slab intersection in front of the
// origin, entry clamped to 0) is this repository's and is shared bit-for-bit with oracle/wisp_oracle.c (DESIGN.md).
#include "wb_common.cuh"

__device__ __forceinline__ bool wb_slab(const float o[3], const float d[3], int cx, int cy, int cz, int level, float& t0, float& t1)
{
    const float size = 2.0f / (float)(1u << level);
    const int c[3] = { cx, cy, cz };
    float te = -INFINITY, tx = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float lo = __fsub_rn(__fmul_rn((float)c[a], size), 1.0f), hi = __fadd_rn(lo, size);
        if (d[a] != 0.0f) {
            const float ta = __fdiv_rn(__fsub_rn(lo, o[a]), d[a]), tb = __fdiv_rn(__fsub_rn(hi, o[a]), d[a]);
            te = fmaxf(te, fminf(ta, tb)); tx = fminf(tx, fmaxf(ta, tb));
        } else if (o[a] < lo || o[a] >= hi) return false;     // parallel axis: the cell's points, [lo, hi) as in wb_quantize
    }
    const float en = fmaxf(te, 0.0f);
    if (!(tx > en)) return false;
    t0 = en; t1 = tx; return true;
}

// MODE 0: count.  1: fill (second traversal).  2: count AND keep the first K nuggets of every ray in a cache laid out [K][R] (nugget-major:
// the 32 rays of a warp write neighbouring words).  3: fill from that cache; only rays with more than K nuggets are traversed again.
// Modes 2 + 3 replace the two full depth-first traversals of 0 + 1 by one (the traversal is a chain of dependent byte loads per ray and
// dominates both passes: 0.29 ms each for the 512^2 rays of the SDF configuration).
struct WbNugCache { int32_t* pidx; float2* depth; int K; };

template <int MODE>
__global__ void __launch_bounds__(128)
wb_raytrace_kernel(WbOct oc, const float* __restrict__ origins, const float* __restrict__ dirs, int64_t R,
                   int32_t* __restrict__ counts, const int64_t* __restrict__ offsets,
                   int32_t* __restrict__ ridx, int32_t* __restrict__ pidx, float* __restrict__ depth, WbNugCache cache)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    constexpr bool FILL = (MODE == 1 || MODE == 3);
    int64_t pos = FILL ? offsets[r] : 0;
    if (MODE == 3) {
        const int n = (int)(offsets[r + 1] - pos);
        if (n <= cache.K) {                                   // the whole ray is in the cache: copy, no traversal
            for (int i = 0; i < n; ++i) {
                const float2 dd = cache.depth[(int64_t)i * R + r];
                ridx[pos + i] = (int32_t)r; pidx[pos + i] = cache.pidx[(int64_t)i * R + r];
                depth[2 * (pos + i)] = dd.x; depth[2 * (pos + i) + 1] = dd.y;
            }
            return;
        }
    }
    const float o[3] = { origins[3 * r], origins[3 * r + 1], origins[3 * r + 2] };
    const float d[3] = { dirs[3 * r], dirs[3 * r + 1], dirs[3 * r + 2] };
    const int mask = (d[0] < 0.0f ? 4 : 0) | (d[1] < 0.0f ? 2 : 0) | (d[2] < 0.0f ? 1 : 0);
    // stack entry: node index + packed (level:4 | x:16 | y:16 | z:16)
    int32_t st_node[7 * 15 + 2]; uint64_t st_cell[7 * 15 + 2];
    int sp = 1; st_node[0] = 0; st_cell[0] = 0;
    int cnt = 0;
    while (sp > 0) {
        --sp;
        const int32_t node = st_node[sp]; const uint64_t cell = st_cell[sp];
        const int l = (int)(cell >> 48), cx = (int)((cell >> 32) & 0xffff), cy = (int)((cell >> 16) & 0xffff), cz = (int)(cell & 0xffff);
        float t0, t1;
        if (!wb_slab(o, d, cx, cy, cz, l, t0, t1)) continue;
        if (l == oc.level) {
            if (FILL) { ridx[pos] = (int32_t)r; pidx[pos] = node; depth[2 * pos] = t0; depth[2 * pos + 1] = t1; ++pos; }
            if (MODE == 2 && cnt < cache.K) { cache.pidx[(int64_t)cnt * R + r] = node; cache.depth[(int64_t)cnt * R + r] = make_float2(t0, t1); }
            ++cnt; continue;
        }
        const uint32_t bits = __ldg(oc.octree + node);
        const int32_t base = __ldg(oc.prefix + node);
        for (int i = 7; i >= 0; --i) {                    // push in reverse: child (0 ^ mask) is visited first
            const int c = i ^ mask;
            if (!(bits & (1u << c))) continue;
            st_node[sp] = base + __popc(bits & ((2u << c) - 1u));
            st_cell[sp] = ((uint64_t)(l + 1) << 48) | ((uint64_t)(2 * cx + ((c >> 2) & 1)) << 32) | ((uint64_t)(2 * cy + ((c >> 1) & 1)) << 16) | (uint64_t)(2 * cz + (c & 1));
            ++sp;
        }
    }
    if (!FILL) counts[r] = cnt;
}

static int wb_raytrace_launch(int mode, const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t* counts, const int64_t* offsets,
                              int32_t* ridx, int32_t* pidx, float* depth, void* cache, int32_t cache_k, wb_stream s)
{
    WbOct o; int rc = wb_make_oct(oct, level, &o); if (rc) return rc;
    WB_CHECK_ARG(rays != nullptr, "null rays");
    const int64_t R = rays->num_rays;
    if (R == 0) return WB_OK;
    WB_CHECK_ARG(rays->origins && rays->dirs, "null pointer");
    WbNugCache nc = { nullptr, nullptr, 0 };
    if (mode >= 2) {
        WB_CHECK_ARG(cache != nullptr && cache_k >= 1, "null nugget cache");
        nc.K = cache_k; nc.depth = reinterpret_cast<float2*>(cache); nc.pidx = reinterpret_cast<int32_t*>(nc.depth + (int64_t)cache_k * R);
    }
    const unsigned grid = (unsigned)((R + 127) / 128);
    cudaStream_t st = (cudaStream_t)s;
    if (mode == 0) wb_raytrace_kernel<0><<<grid, 128, 0, st>>>(o, rays->origins, rays->dirs, R, counts, nullptr, nullptr, nullptr, nullptr, nc);
    else if (mode == 1) wb_raytrace_kernel<1><<<grid, 128, 0, st>>>(o, rays->origins, rays->dirs, R, nullptr, offsets, ridx, pidx, depth, nc);
    else if (mode == 2) wb_raytrace_kernel<2><<<grid, 128, 0, st>>>(o, rays->origins, rays->dirs, R, counts, nullptr, nullptr, nullptr, nullptr, nc);
    else wb_raytrace_kernel<3><<<grid, 128, 0, st>>>(o, rays->origins, rays->dirs, R, nullptr, offsets, ridx, pidx, depth, nc);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

extern "C" int wb_raytrace_count(const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t* counts, wb_stream s)
{
    WB_CHECK_ARG(counts != nullptr || (rays && rays->num_rays == 0), "null pointer");
    return wb_raytrace_launch(0, oct, level, rays, counts, nullptr, nullptr, nullptr, nullptr, nullptr, 0, s);
}
extern "C" int wb_raytrace_fill(const wb_octree* oct, int32_t level, const wb_rays* rays, const int64_t* offsets,
                                int32_t* ridx, int32_t* pidx, float* depth, wb_stream s)
{
    WB_CHECK_ARG((offsets && ridx && pidx && depth) || (rays && rays->num_rays == 0), "null pointer");
    return wb_raytrace_launch(1, oct, level, rays, nullptr, offsets, ridx, pidx, depth, nullptr, 0, s);
}
// One-traversal form: count + cache of the first cache_k nuggets per ray (cache: wb_raytrace_cache_bytes(R, cache_k) bytes), then the fill
// that copies from the cache and re-traverses only the rays that overflowed it.  Same outputs as wb_raytrace_count / wb_raytrace_fill.
extern "C" int64_t wb_raytrace_cache_bytes(int64_t R, int32_t cache_k) { return (R < 0 || cache_k < 1) ? -1 : R * (int64_t)cache_k * 12; }
extern "C" int wb_raytrace_count_cached(const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t* counts, void* cache, int32_t cache_k, wb_stream s)
{
    WB_CHECK_ARG(counts != nullptr || (rays && rays->num_rays == 0), "null pointer");
    return wb_raytrace_launch(2, oct, level, rays, counts, nullptr, nullptr, nullptr, nullptr, cache, cache_k, s);
}
extern "C" int wb_raytrace_fill_cached(const wb_octree* oct, int32_t level, const wb_rays* rays, const int64_t* offsets, const void* cache, int32_t cache_k,
                                       int32_t* ridx, int32_t* pidx, float* depth, wb_stream s)
{
    WB_CHECK_ARG((offsets && ridx && pidx && depth) || (rays && rays->num_rays == 0), "null pointer");
    return wb_raytrace_launch(3, oct, level, rays, nullptr, offsets, ridx, pidx, depth, const_cast<void*>(cache), cache_k, s);
}

// ---- 'voxel': n jittered samples per nugget ------------------------------------------------------------------------
__device__ __forceinline__ float wb_voxel_depth(float en, float len, int k, float jit, float inv_n)
{   // steps = (arange + rand) * (1/n); samples = entry + (exit - entry) * steps   (sampling.py:50-53), op by op
    float st = __fadd_rn((float)k, jit); st = __fmul_rn(st, inv_n);
    return __fadd_rn(en, __fmul_rn(len, st));
}
__global__ void __launch_bounds__(256)
wb_voxel_fill_kernel(const float* __restrict__ origins, const float* __restrict__ dirs, const int32_t* __restrict__ nug_ridx,
                     const float2* __restrict__ nug_depth, int64_t Ng, int n, float inv_n, const float* __restrict__ jitter, uint32_t seed,
                     int64_t* __restrict__ ridx, float* __restrict__ samples, float* __restrict__ depth, float* __restrict__ deltas,
                     uint8_t* __restrict__ boundary, int32_t* __restrict__ rec_ray)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Ng * n) return;
    const int64_t g = i / n; const int k = (int)(i - g * n);
    const int32_t r = __ldg(nug_ridx + g);
    const float2 dd = __ldg(nug_depth + g);
    const float len = __fsub_rn(dd.y, dd.x);
    const uint32_t key = wb_ray_key(seed, (uint32_t)g);
    const float jit = jitter ? __ldg(jitter + i) : wb_jitter(key, (uint32_t)k);
    const float sdep = wb_voxel_depth(dd.x, len, k, jit, inv_n);
    float prev = dd.x;
    if (k > 0) { const float jp = jitter ? __ldg(jitter + i - 1) : wb_jitter(key, (uint32_t)(k - 1)); prev = wb_voxel_depth(dd.x, len, k - 1, jp, inv_n); }
    if (depth) depth[i] = sdep;
    if (deltas) deltas[i] = __fsub_rn(sdep, prev);                               // diff(prepend = entry), octree_as.py:220
    if (ridx) ridx[i] = r;
    if (rec_ray) rec_ray[i] = r;
    if (samples) {
        samples[3 * i] = wb_addcmul(__ldg(origins + 3 * (int64_t)r), __ldg(dirs + 3 * (int64_t)r), sdep);
        samples[3 * i + 1] = wb_addcmul(__ldg(origins + 3 * (int64_t)r + 1), __ldg(dirs + 3 * (int64_t)r + 1), sdep);
        samples[3 * i + 2] = wb_addcmul(__ldg(origins + 3 * (int64_t)r + 2), __ldg(dirs + 3 * (int64_t)r + 2), sdep);
    }
    if (boundary) boundary[i] = (k == 0 && (g == 0 || __ldg(nug_ridx + g - 1) != r)) ? 1 : 0;     // mark_first_hit + expand_pack_boundary
}

extern "C" int wb_raymarch_voxel_fill(const wb_rays* rays, const int32_t* nug_ridx, const float* nug_depth, int64_t Ng, int32_t num_samples,
                                      const float* jitter, uint32_t seed, int64_t* ridx, float* samples, float* depth, float* deltas,
                                      uint8_t* boundary, int32_t* rec_ray, wb_stream s)
{
    WB_CHECK_ARG(num_samples >= 1, "num_samples must be >= 1");
    if (Ng == 0) return WB_OK;
    WB_CHECK_ARG(rays && rays->origins && rays->dirs && nug_ridx && nug_depth, "null pointer");
    const int64_t S = Ng * num_samples;
    const float inv_n = (float)(1.0 / (double)num_samples);
    wb_voxel_fill_kernel<<<(unsigned)((S + 255) / 256), 256, 0, (cudaStream_t)s>>>(rays->origins, rays->dirs, nug_ridx, reinterpret_cast<const float2*>(nug_depth),
                                                                                    Ng, num_samples, inv_n, jitter, seed, ridx, samples, depth, deltas, boundary, rec_ray);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---- 'uniform': samples on the global lattice depth = k/scale inside every nugget -----------------------------------------
__global__ void wb_uniform_count_kernel(const float2* __restrict__ nug_depth, int64_t Ng, float scale, int32_t* __restrict__ cnt)
{
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= Ng) return;
    const float2 d = __ldg(nug_depth + g);
    cnt[g] = (int)ceilf(__fmul_rn(scale, d.y)) - (int)ceilf(__fmul_rn(scale, d.x));      // octree_as.py:340-342
}
__global__ void wb_uniform_fill_kernel(const float* __restrict__ origins, const float* __restrict__ dirs, const int32_t* __restrict__ nug_ridx,
                                       const float2* __restrict__ nug_depth, int64_t Ng, float scale, float inv_scale, float step,
                                       const int64_t* __restrict__ soff, const int64_t* __restrict__ ray_nug_off,
                                       int64_t* __restrict__ ridx, float* __restrict__ samples, float* __restrict__ depth, float* __restrict__ deltas,
                                       uint8_t* __restrict__ boundary, int32_t* __restrict__ rec_ray)
{
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= Ng) return;
    const int64_t b = soff[g], e = soff[g + 1];
    if (e == b) return;                                   // nuggets without lattice points are dropped (octree_as.py:345-349)
    const int32_t r = __ldg(nug_ridx + g);
    const float first = ceilf(__fmul_rn(scale, __ldg(nug_depth + g).x));
    // boundary: first sample of the first KEPT nugget of the ray (uniform_sample_cuda.cu:42) == no sample of this ray before it
    const bool ray_first = (b == soff[ray_nug_off[r]]);
    const float ox = __ldg(origins + 3 * (int64_t)r), oy = __ldg(origins + 3 * (int64_t)r + 1), oz = __ldg(origins + 3 * (int64_t)r + 2);
    const float dx = __ldg(dirs + 3 * (int64_t)r), dy = __ldg(dirs + 3 * (int64_t)r + 1), dz = __ldg(dirs + 3 * (int64_t)r + 2);
    float f = 0.0f;
    for (int64_t i = b; i < e; ++i) {
        const float sdep = __fmul_rn(inv_scale, __fadd_rn(first, f)); f += 1.0f;      // uniform_sample_cuda.cu:47-48
        if (depth) depth[i] = sdep;
        if (deltas) deltas[i] = step;
        if (ridx) ridx[i] = r;
        if (rec_ray) rec_ray[i] = r;
        if (samples) { samples[3 * i] = wb_addcmul(ox, dx, sdep); samples[3 * i + 1] = wb_addcmul(oy, dy, sdep); samples[3 * i + 2] = wb_addcmul(oz, dz, sdep); }
        if (boundary) boundary[i] = (ray_first && i == b) ? 1 : 0;
    }
}

extern "C" int wb_raymarch_uniform_count(const float* nug_depth, int64_t Ng, int32_t scale, int32_t* cnt, wb_stream s)
{
    if (Ng == 0) return WB_OK;
    WB_CHECK_ARG(nug_depth && cnt && scale >= 1, "bad argument");
    wb_uniform_count_kernel<<<(unsigned)((Ng + 255) / 256), 256, 0, (cudaStream_t)s>>>(reinterpret_cast<const float2*>(nug_depth), Ng, (float)scale, cnt);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
extern "C" int wb_raymarch_uniform_fill(const wb_rays* rays, const int32_t* nug_ridx, const float* nug_depth, int64_t Ng, int32_t scale,
                                        const int64_t* sample_offsets, const int64_t* ray_nugget_offsets,
                                        int64_t* ridx, float* samples, float* depth, float* deltas, uint8_t* boundary, int32_t* rec_ray, wb_stream s)
{
    if (Ng == 0) return WB_OK;
    WB_CHECK_ARG(rays && rays->origins && rays->dirs && nug_ridx && nug_depth && sample_offsets && ray_nugget_offsets && scale >= 1, "bad argument");
    const float inv_scale = 1.0f / (float)scale, step = (float)(1.0 / (double)scale);
    wb_uniform_fill_kernel<<<(unsigned)((Ng + 255) / 256), 256, 0, (cudaStream_t)s>>>(rays->origins, rays->dirs, nug_ridx, reinterpret_cast<const float2*>(nug_depth), Ng,
                                                                                       (float)scale, inv_scale, step, sample_offsets, ray_nugget_offsets,
                                                                                       ridx, samples, depth, deltas, boundary, rec_ray);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---- PackedSPCTracer.trace: the first nugget of every ray (packed_spc_tracer.py:50-90) -----------------------------------
// wb_raytrace_kernel's walk (same stack, same i ^ mask child order, same wb_slab nugget) stopped at the first cell of `level`:
// the walk visits a ray's nuggets front to back, so that cell is the nugget the reference keeps after mark_pack_boundaries.
// One launch replaces count + scan + fill + the first-hit selection, and no nugget list is written.
__global__ void __launch_bounds__(128)
wb_spc_trace_kernel(WbOct oc, const float* __restrict__ origins, const float* __restrict__ dirs, int64_t R,
                    const float* __restrict__ colors, int64_t color_stride, int64_t point_offset,
                    float* __restrict__ depth, uint8_t* __restrict__ hit, float* __restrict__ rgb, float* __restrict__ alpha)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float o[3] = { origins[3 * r], origins[3 * r + 1], origins[3 * r + 2] };
    const float d[3] = { dirs[3 * r], dirs[3 * r + 1], dirs[3 * r + 2] };
    const int mask = (d[0] < 0.0f ? 4 : 0) | (d[1] < 0.0f ? 2 : 0) | (d[2] < 0.0f ? 1 : 0);
    int32_t st_node[7 * 15 + 2]; uint64_t st_cell[7 * 15 + 2];
    int sp = 1; st_node[0] = 0; st_cell[0] = 0;
    while (sp > 0) {
        --sp;
        const int32_t node = st_node[sp]; const uint64_t cell = st_cell[sp];
        const int l = (int)(cell >> 48), cx = (int)((cell >> 32) & 0xffff), cy = (int)((cell >> 16) & 0xffff), cz = (int)(cell & 0xffff);
        float t0, t1;
        if (!wb_slab(o, d, cx, cy, cz, l, t0, t1)) continue;
        if (l == oc.level) {
            const float* c = colors + ((int64_t)node - point_offset) * color_stride;
            depth[r] = t0; hit[r] = 1; alpha[r] = 1.0f;
            rgb[3 * r] = __ldg(c); rgb[3 * r + 1] = __ldg(c + 1); rgb[3 * r + 2] = __ldg(c + 2);
            return;
        }
        const uint32_t bits = __ldg(oc.octree + node);
        const int32_t base = __ldg(oc.prefix + node);
        for (int i = 7; i >= 0; --i) {
            const int c = i ^ mask;
            if (!(bits & (1u << c))) continue;
            st_node[sp] = base + __popc(bits & ((2u << c) - 1u));
            st_cell[sp] = ((uint64_t)(l + 1) << 48) | ((uint64_t)(2 * cx + ((c >> 2) & 1)) << 32) | ((uint64_t)(2 * cy + ((c >> 1) & 1)) << 16) | (uint64_t)(2 * cz + (c & 1));
            ++sp;
        }
    }
    depth[r] = 0.0f; hit[r] = 0; alpha[r] = 0.0f;                 // miss: the reference's zero-initialised buffers (:76-83)
    rgb[3 * r] = 0.0f; rgb[3 * r + 1] = 0.0f; rgb[3 * r + 2] = 0.0f;
}

extern "C" int wb_spc_trace(const wb_octree* oct, int32_t level, const wb_rays* rays, const float* colors, int64_t color_stride, int64_t point_offset,
                            float* depth, uint8_t* hit, float* rgb, float* alpha, wb_stream s)
{
    WbOct o; int rc = wb_make_oct(oct, level, &o); if (rc) return rc;
    WB_CHECK_ARG(rays != nullptr, "null rays");
    const int64_t R = rays->num_rays;
    WB_CHECK_ARG(R >= 0 && R < ((int64_t)1 << 31) * 128, "num_rays out of range");
    if (R == 0) return WB_OK;
    WB_CHECK_ARG(rays->origins && rays->dirs && colors && depth && hit && rgb && alpha, "null pointer");
    WB_CHECK_ARG(color_stride >= 3 && point_offset >= 0, "color_stride must be >= 3 and point_offset >= 0");
    wb_spc_trace_kernel<<<(unsigned)((R + 127) / 128), 128, 0, (cudaStream_t)s>>>(o, rays->origins, rays->dirs, R, colors, color_stride, point_offset,
                                                                                 depth, hit, rgb, alpha);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
