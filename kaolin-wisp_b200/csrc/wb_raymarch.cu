// wb_raymarch.cu -- OctreeAS._raymarch_ray (wisp/accelstructs/octree_as.py:247-309) on sm_90a.
//
// The reference materialises all R*n candidates ([R,n,3] fp32), queries the octree for each, runs
// torch.nonzero (host sync + compaction) and four fancy-index gathers.  Here one warp owns one ray:
//   count : 32 candidates per iteration (lane = candidate), occupancy test, ballot -> hit bitmask word;
//           the mask (n/8 bytes per ray) and the per-ray count are the only outputs (C*29 B never exist).
//   fill  : re-evaluates depth/delta ONLY for the set bits and writes either the reference's
//           ASRaymarchResults layout or the fused path's 12-byte records.
// Bit-exactness contract: wb_common.cuh (depth op order, exact quantisation).
#include "wb_common.cuh"

constexpr int WB_MARCH_THREADS = 256;

__global__ void __launch_bounds__(WB_MARCH_THREADS)
wb_march_count_kernel(WbOct o, WbMarch m, uint32_t* __restrict__ hitmask, int32_t* __restrict__ counts)
{
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nw = (m.n + 31) >> 5;
    for (int64_t r = warp0; r < m.R; r += nwarps) {
        float nearv, range; wb_ray_range(m, r, nearv, range);
        const uint32_t key = wb_ray_key(m.seed, (uint32_t)r);
        const float ox = __ldg(m.origins + 3 * r), oy = __ldg(m.origins + 3 * r + 1), oz = __ldg(m.origins + 3 * r + 2);
        const float dx = __ldg(m.dirs + 3 * r), dy = __ldg(m.dirs + 3 * r + 1), dz = __ldg(m.dirs + 3 * r + 2);
        // Candidates whose depth lies outside the ray's intersection with the (widened) box of occupied cells cannot be
        // occupied: restrict the exact per-candidate test to the iterations [w0, w1] that can overlap it.  The candidate
        // index bounds are conservative by one candidate on each side (jitter < one spacing, float slack << spacing).
        int w0 = 0, w1 = nw - 1;
        float tc0 = -3.0e38f, tc1 = 3.0e38f;                     // depth range of the ray inside the widened box
        if (o.has_bbox) {
            float t0 = -3.0e38f, t1 = 3.0e38f; bool miss = false;
            const float oo[3] = { ox, oy, oz }, dd[3] = { dx, dy, dz };
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                if (fabsf(dd[a]) > 1e-12f) {
                    const float inv = 1.0f / dd[a];
                    const float ta = (o.blo[a] - oo[a]) * inv, tb = (o.bhi[a] - oo[a]) * inv;
                    t0 = fmaxf(t0, fminf(ta, tb)); t1 = fminf(t1, fmaxf(ta, tb));
                } else if (oo[a] < o.blo[a] || oo[a] > o.bhi[a]) miss = true;
            }
            t0 -= 1e-4f * (1.0f + fabsf(t0)); t1 += 1e-4f * (1.0f + fabsf(t1));
            tc0 = t0; tc1 = t1;
            if (miss || t1 < t0 || !(range > 0.0f)) { if (miss || t1 < t0) { w0 = 1; w1 = 0; } }
            else {
                // depth(i) in [lin_i*range + near, (lin_i + 1/n)*range + near], lin_i ~ i/(n-1)
                const float nm1 = (float)max(m.n - 1, 1);
                const float f0 = ((t0 - nearv) / range - m.inv_n) * nm1 - 2.0f;
                const float f1 = ((t1 - nearv) / range) * nm1 + 2.0f;
                const int i0 = f0 <= 0.0f ? 0 : (f0 >= (float)m.n ? m.n : (int)f0);
                const int i1 = f1 < 0.0f ? -1 : (f1 >= (float)(m.n - 1) ? m.n - 1 : (int)f1 + 1);
                w0 = i0 >> 5; w1 = i1 < 0 ? -1 : (i1 >> 5);
                if (w1 > nw - 1) w1 = nw - 1;
            }
        }
        // Word-level rejection with the dilated coarse mask (wb_octree_build_coarse): test points every half coarse cell along the
        // clipped segment; a word is visited only if one of them falls into a marked coarse cell.  Conservative: an occupied
        // candidate X at depth d has a test point within a quarter coarse cell, whose (clamped) cell is c(X) or a neighbour, and
        // the candidate indices whose depth can lie within one spacing of that test point are all flagged (+-2 slack).
        uint64_t active = ~0ull;
        if (o.coarse != nullptr && nw <= 64 && w1 >= w0 && range > 0.0f) {
            const float dlen = sqrtf(dx * dx + dy * dy + dz * dz);
            const float delta = (0.5f / o.ch) / fmaxf(dlen, 1e-20f);           // half a coarse cell, in depth units
            const float ta = fmaxf(tc0, nearv), tb = fminf(tc1, nearv + range * (1.0f + m.inv_n));
            const float fn = (tb - ta) / delta;
            if (tb >= ta && fn < 1024.0f) {
                const int npts = (int)fn + 2;
                const float nm1 = (float)max(m.n - 1, 1);
                uint32_t lo = 0, hi = 0;
                for (int k = lane; k < npts; k += 32) {
                    const float tau = fminf(ta + (float)k * delta, tb);
                    const float px = __fmaf_rn(dx, tau, ox), py = __fmaf_rn(dy, tau, oy), pz = __fmaf_rn(dz, tau, oz);
                    const int qx = (int)fminf(fmaxf(floorf(__fmaf_rn(px, o.ch, o.ch)), 0.0f), o.cmax);
                    const int qy = (int)fminf(fmaxf(floorf(__fmaf_rn(py, o.ch, o.ch)), 0.0f), o.cmax);
                    const int qz = (int)fminf(fmaxf(floorf(__fmaf_rn(pz, o.ch, o.ch)), 0.0f), o.cmax);
                    const uint32_t idx = ((uint32_t)qx << (2 * o.clevel)) | ((uint32_t)qy << o.clevel) | (uint32_t)qz;
                    if ((__ldg(o.coarse + (idx >> 5)) >> (idx & 31)) & 1u) {
                        const float f0 = ((tau - delta - nearv) / range - m.inv_n) * nm1 - 2.0f;
                        const float f1 = ((tau + delta - nearv) / range) * nm1 + 2.0f;
                        const int i0 = f0 <= 0.0f ? 0 : (f0 >= (float)(m.n - 1) ? m.n - 1 : (int)f0);
                        const int i1 = f1 <= 0.0f ? 0 : (f1 >= (float)(m.n - 1) ? m.n - 1 : (int)f1 + 1);
                        const int a0 = i0 >> 5, a1 = min(i1 >> 5, 63);
                        const uint64_t span = (a1 >= 63 ? ~0ull : ((1ull << (a1 + 1)) - 1ull)) & ~((1ull << a0) - 1ull);
                        lo |= (uint32_t)span; hi |= (uint32_t)(span >> 32);
                    }
                }
                lo = __reduce_or_sync(0xffffffffu, lo); hi = __reduce_or_sync(0xffffffffu, hi);
                active = ((uint64_t)hi << 32) | lo;
            }
        }
        int cnt = 0;
        for (int wg = 0; wg < nw; wg += 32) {                    // groups of 32 words: lane j keeps word wg + j, one coalesced store
            uint32_t keep = 0;
            const int wa = max(wg, w0), wb = min(wg + 31, w1);
            for (int w = wa; w <= wb; ++w) {
                if (nw <= 64 && !((active >> w) & 1ull)) continue;
                const int i = (w << 5) + lane;
                bool hit = false;
                if (i < m.n) {
                    const float d = wb_depth(m, r, key, i, nearv, range);
                    hit = wb_occupied(o, wb_addcmul(ox, dx, d), wb_addcmul(oy, dy, d), wb_addcmul(oz, dz, d));
                }
                const uint32_t word = __ballot_sync(0xffffffffu, hit);
                cnt += __popc(word);
                if ((w & 31) == lane) keep = word;
            }
            if (wg + lane < nw) hitmask[r * nw + wg + lane] = keep;
        }
        if (lane == 0) counts[r] = cnt;
    }
}

extern "C" int wb_raymarch_ray_count(const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t num_samples,
                                     const float* jitter, uint32_t seed, uint32_t* hitmask, int32_t* counts, wb_stream s)
{
    WbOct o; int rc = wb_make_oct(oct, level, &o); if (rc) return rc;
    WbMarch m; rc = wb_make_march(rays, num_samples, jitter, seed, &m); if (rc) return rc;
    if (m.R == 0) return WB_OK;
    WB_CHECK_ARG(hitmask && counts, "null output");
    const int warps_per_cta = WB_MARCH_THREADS / 32;
    int64_t ctas = (m.R + warps_per_cta - 1) / warps_per_cta;
    const int64_t cap = (int64_t)wb_num_sms() * 8 * 4;          // persistent-ish: a few waves of 8 CTAs/SM
    if (ctas > cap) ctas = cap;
    wb_march_count_kernel<<<(unsigned)ctas, WB_MARCH_THREADS, 0, (cudaStream_t)s>>>(o, m, hitmask, counts);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

// ---- scan -------------------------------------------------------------------------------------------------
// offsets = exclusive scan of counts (int32 -> int64), offsets[R] = total.  Three small kernels:
// per-chunk sums, a single-CTA scan of the chunk sums, per-chunk scan + base.  workspace: int64 [nchunks].
constexpr int WB_SCAN_THREADS = 256;
constexpr int WB_SCAN_ITEMS = 16;
constexpr int WB_SCAN_CHUNK = WB_SCAN_THREADS * WB_SCAN_ITEMS;     // 4096 counts per CTA

__device__ __forceinline__ int64_t wb_block_excl_scan(int64_t v, int64_t* total)
{   // exclusive scan of one value per thread across the CTA (WB_SCAN_THREADS threads)
    __shared__ int64_t wsum[WB_SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int64_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int64_t w = lane < WB_SCAN_THREADS / 32 ? wsum[lane] : 0, wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int64_t t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
        if (lane < WB_SCAN_THREADS / 32) wsum[lane] = wi - w;
        if (lane == 31 && total) *total = wi;
    }
    __syncthreads();
    const int64_t r = incl - v + wsum[warp];
    __syncthreads();
    return r;
}
__global__ void __launch_bounds__(WB_SCAN_THREADS) wb_scan_sums_kernel(const int32_t* __restrict__ counts, int64_t R, int64_t* __restrict__ sums)
{
    const int64_t base = (int64_t)blockIdx.x * WB_SCAN_CHUNK;
    int64_t v = 0;
    for (int i = 0; i < WB_SCAN_ITEMS; ++i) { const int64_t k = base + i * WB_SCAN_THREADS + threadIdx.x; if (k < R) v += counts[k]; }
    __shared__ int64_t tot;
    wb_block_excl_scan(v, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(WB_SCAN_THREADS) wb_scan_top_kernel(int64_t* __restrict__ sums, int64_t n, int64_t* __restrict__ total_out)
{   // in-place exclusive scan of the chunk sums by one CTA
    __shared__ int64_t tot; int64_t carry = 0;
    for (int64_t b = 0; b < n; b += WB_SCAN_THREADS) {
        const int64_t k = b + threadIdx.x;
        const int64_t v = k < n ? sums[k] : 0;
        const int64_t ex = wb_block_excl_scan(v, &tot);
        if (k < n) sums[k] = carry + ex;
        carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total_out = carry;
}
__global__ void __launch_bounds__(WB_SCAN_THREADS) wb_scan_final_kernel(const int32_t* __restrict__ counts, int64_t R,
                                                                         const int64_t* __restrict__ sums, int64_t* __restrict__ offsets)
{
    const int64_t base = (int64_t)blockIdx.x * WB_SCAN_CHUNK + (int64_t)threadIdx.x * WB_SCAN_ITEMS;   // blocked arrangement
    int32_t c[WB_SCAN_ITEMS]; int64_t v = 0;
#pragma unroll
    for (int i = 0; i < WB_SCAN_ITEMS; ++i) { c[i] = (base + i < R) ? counts[base + i] : 0; v += c[i]; }
    int64_t run = wb_block_excl_scan(v, nullptr) + sums[blockIdx.x];
#pragma unroll
    for (int i = 0; i < WB_SCAN_ITEMS; ++i) { if (base + i < R) offsets[base + i] = run; run += c[i]; }
}

extern "C" int64_t wb_scan_workspace_bytes(int64_t R)
{
    const int64_t chunks = (R + WB_SCAN_CHUNK - 1) / WB_SCAN_CHUNK;
    return (chunks + 1) * (int64_t)sizeof(int64_t);
}
extern "C" int wb_scan_counts(const int32_t* counts, int64_t R, int64_t* offsets, void* workspace, int64_t workspace_bytes, wb_stream s)
{
    WB_CHECK_ARG(offsets && workspace && (counts || R == 0), "null pointer");
    WB_CHECK_ARG(R >= 0 && R < ((int64_t)1 << 31), "R out of range");
    WB_CHECK_ARG(workspace_bytes >= wb_scan_workspace_bytes(R), "workspace too small");
    cudaStream_t st = (cudaStream_t)s;
    const int64_t chunks = (R + WB_SCAN_CHUNK - 1) / WB_SCAN_CHUNK;
    int64_t* sums = reinterpret_cast<int64_t*>(workspace);
    if (chunks > 0) { wb_scan_sums_kernel<<<(unsigned)chunks, WB_SCAN_THREADS, 0, st>>>(counts, R, sums); WB_LAUNCH_CHECK(); }
    wb_scan_top_kernel<<<1, WB_SCAN_THREADS, 0, st>>>(sums, chunks, offsets + R); WB_LAUNCH_CHECK();
    if (chunks > 0) { wb_scan_final_kernel<<<(unsigned)chunks, WB_SCAN_THREADS, 0, st>>>(counts, R, sums, offsets); WB_LAUNCH_CHECK(); }
    return WB_OK;
}

// ---- fill -------------------------------------------------------------------------------------------------
// FUSED = false : ASRaymarchResults (base_as.py:57-84)    FUSED = true : (t, delta, ray) records
template <bool FUSED>
__global__ void __launch_bounds__(WB_MARCH_THREADS)
wb_march_fill_kernel(WbMarch m, const uint32_t* __restrict__ hitmask, const int64_t* __restrict__ offsets,
                     int64_t* __restrict__ ridx, float* __restrict__ samples, float* __restrict__ depth,
                     float* __restrict__ deltas, uint8_t* __restrict__ boundary, int32_t* __restrict__ rec_ray)
{
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nw = (m.n + 31) >> 5;
    for (int64_t r = warp0; r < m.R; r += nwarps) {
        const int64_t base = offsets[r];
        if (offsets[r + 1] == base) continue;                    // ray without samples
        float nearv, range; wb_ray_range(m, r, nearv, range);
        const uint32_t key = wb_ray_key(m.seed, (uint32_t)r);
        float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 0;
        if (!FUSED && samples) {
            ox = __ldg(m.origins + 3 * r); oy = __ldg(m.origins + 3 * r + 1); oz = __ldg(m.origins + 3 * r + 2);
            dx = __ldg(m.dirs + 3 * r); dy = __ldg(m.dirs + 3 * r + 1); dz = __ldg(m.dirs + 3 * r + 2);
        }
        int64_t run = base;
        for (int wb = 0; wb < nw; wb += 32) {
            const uint32_t mine = (wb + lane < nw) ? __ldg(hitmask + r * nw + wb + lane) : 0u;
            uint32_t nz = __ballot_sync(0xffffffffu, mine != 0u);     // visit only the words that hold samples
            while (nz) {
                const int j = __ffs(nz) - 1; nz &= nz - 1u;
                const uint32_t word = __shfl_sync(0xffffffffu, mine, j);
                if (word & (1u << lane)) {
                    const int i = ((wb + j) << 5) + lane;
                    const int64_t dst = run + __popc(word & ((1u << lane) - 1u));
                    const float d = wb_depth(m, r, key, i, nearv, range);
                    // deltas = depth.diff(prepend = zeros + dist_min): to the previous CANDIDATE (octree_as.py:290-291)
                    const float prev = (i == 0) ? __fadd_rn(0.0f, nearv) : wb_depth(m, r, key, i - 1, nearv, range);
                    const float dl = __fsub_rn(d, prev);
                    if (depth) depth[dst] = d;
                    if (deltas) deltas[dst] = dl;
                    if (FUSED) { rec_ray[dst] = (int32_t)r; }
                    else {
                        if (ridx) ridx[dst] = r;
                        if (samples) { samples[3 * dst] = wb_addcmul(ox, dx, d); samples[3 * dst + 1] = wb_addcmul(oy, dy, d); samples[3 * dst + 2] = wb_addcmul(oz, dz, d); }
                        if (boundary) boundary[dst] = (dst == base) ? 1 : 0;      // mark_pack_boundaries (octree_as.py:300)
                    }
                }
                run += __popc(word);
            }
        }
    }
}

static int wb_fill_launch(bool fused, const wb_rays* rays, int32_t n, const float* jitter, uint32_t seed,
                          const uint32_t* hitmask, const int64_t* offsets, int64_t* ridx, float* samples, float* depth,
                          float* deltas, uint8_t* boundary, int32_t* rec_ray, wb_stream s)
{
    WbMarch m; int rc = wb_make_march(rays, n, jitter, seed, &m); if (rc) return rc;
    if (m.R == 0) return WB_OK;
    WB_CHECK_ARG(hitmask && offsets, "null pointer");
    const int warps_per_cta = WB_MARCH_THREADS / 32;
    int64_t ctas = (m.R + warps_per_cta - 1) / warps_per_cta;
    const int64_t cap = (int64_t)wb_num_sms() * 8 * 4;
    if (ctas > cap) ctas = cap;
    if (fused) wb_march_fill_kernel<true><<<(unsigned)ctas, WB_MARCH_THREADS, 0, (cudaStream_t)s>>>(m, hitmask, offsets, ridx, samples, depth, deltas, boundary, rec_ray);
    else wb_march_fill_kernel<false><<<(unsigned)ctas, WB_MARCH_THREADS, 0, (cudaStream_t)s>>>(m, hitmask, offsets, ridx, samples, depth, deltas, boundary, rec_ray);
    WB_LAUNCH_CHECK();
    return WB_OK;
}

extern "C" int wb_raymarch_ray_fill(const wb_rays* rays, int32_t num_samples, const float* jitter, uint32_t seed,
                                    const uint32_t* hitmask, const int64_t* offsets,
                                    int64_t* ridx, float* samples, float* depth, float* deltas, uint8_t* boundary, wb_stream s)
{
    return wb_fill_launch(false, rays, num_samples, jitter, seed, hitmask, offsets, ridx, samples, depth, deltas, boundary, nullptr, s);
}

extern "C" int wb_rf_march_fill(const wb_rays* rays, int32_t num_samples, const float* jitter, uint32_t seed,
                                const uint32_t* hitmask, const int64_t* offsets,
                                float* rec_t, float* rec_delta, int32_t* rec_ray, wb_stream s)
{
    return wb_fill_launch(true, rays, num_samples, jitter, seed, hitmask, offsets, nullptr, nullptr, rec_t, rec_delta, nullptr, rec_ray, s);
}
