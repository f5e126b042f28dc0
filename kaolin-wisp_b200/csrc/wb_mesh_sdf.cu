// wb_mesh_sdf.cu -- wisp.ops.mesh.compute_sdf (wisp/ops/mesh/compute_sdf.py, kernel wisp/csrc/external/mesh2sdf_kernel.cu:334-584
// and :844-903) behind a bounding-volume hierarchy: the same per-pair arithmetic, evaluated only for the pairs that can set a point's
// fp32 minimum or one of its 26 stab flags.
//
// Per call, on the current stream, without host synchronisation or allocation:
//   wb_msdf_bounds_kernel   centroid bounds, the largest |vertex coordinate| and the longest edge (atomics on ordered keys)
//   wb_msdf_morton_kernel   30-bit Morton code of each centroid, with the triangle index in the low 32 bits (unique keys)
//   cub::DeviceRadixSort    the keys (counted as one launch)
//   wb_msdf_karras_kernel   the internal nodes of the LBVH (Karras 2012): children and parents
//   wb_msdf_refit_kernel    leaf triangles copied to leaf order in fp64, leaf boxes, then boxes bottom-up (second arrival merges)
//   wb_msdf_query_kernel    one thread per point: the distance traversal, then the 13 line traversals of the stab
// Node numbering: internal nodes 0 .. T-2, leaf j (the j-th sorted triangle) is node T-1+j; node 0 is the root for every T >= 1.
//
// Culling is conservative with respect to the reference's rounded arithmetic (the exact bounds are stated at wb_msdf_query_kernel).
#include "wb_common.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace {

constexpr int kMsdfThreads = 128;
constexpr int kMsdfStack = 64;          // the tree's depth is at most the 62 key bits

// The 13 stab directions as the reference writes them: fp32 literals, widened to double (mesh2sdf_kernel.cu:368-380).
__constant__ float kStabDir[13][3] = {
    {1.0f, 0.0f, 0.0f}, {0.0f, 1.0f, 0.0f}, {0.0f, 0.0f, 1.0f},
    {0.0f, 0.707106781f, 0.707106781f}, {0.707106781f, 0.0f, 0.707106781f}, {0.707106781f, 0.707106781f, 0.0f},
    {0.0f, 0.707106781f, -0.707106781f}, {0.707106781f, 0.0f, -0.707106781f}, {0.707106781f, -0.707106781f, 0.0f},
    {0.577350269f, 0.577350269f, 0.577350269f}, {-0.577350269f, 0.577350269f, 0.577350269f},
    {0.577350269f, -0.577350269f, 0.577350269f}, {0.577350269f, 0.577350269f, -0.577350269f}};

// Float <-> monotone uint32 key, so that atomicMin orders floats.  Slots: [0..2] min centroid, [3..5] ~key of max centroid,
// [6] ~key of max |vertex coordinate|, [7] ~key of the longest edge.  Every slot starts at 0xffffffff.
__device__ __forceinline__ uint32_t fkey(float f)
{
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

struct MsdfWs {
    size_t bounds, keys_in, keys_out, cub, cub_bytes, tris, box, child, parent, flag, total;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int msdf_layout(int64_t T, MsdfWs* w)
{
    size_t cub_bytes = 0;
    if (T > 0 && cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)T, 0, 62) != cudaSuccess)
        return -1;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align256(o + bytes); return at; };
    const size_t nodes = T > 0 ? (size_t)(2 * T - 1) : 0, inner = T > 1 ? (size_t)(T - 1) : 0;
    w->bounds = take(8 * sizeof(uint32_t));
    w->keys_in = take((size_t)T * sizeof(uint64_t));
    w->keys_out = take((size_t)T * sizeof(uint64_t));
    w->cub_bytes = cub_bytes;
    w->cub = take(cub_bytes);
    w->tris = take((size_t)T * 9 * sizeof(double));
    w->box = take(nodes * 2 * sizeof(float4));
    w->child = take(inner * sizeof(int2));
    w->parent = take(nodes * sizeof(int32_t));
    w->flag = take(inner * sizeof(int32_t));
    w->total = o;
    return 0;
}

__device__ __forceinline__ float warp_min(float v)
{
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__global__ void wb_msdf_bounds_kernel(const double* __restrict__ tris, int64_t T, uint32_t* __restrict__ bounds)
{
    float lo[3] = {INFINITY, INFINITY, INFINITY}, nhi[3] = {INFINITY, INFINITY, INFINITY}, nvmax = INFINITY, nemax = INFINITY;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < T; t += (int64_t)gridDim.x * blockDim.x) {
        const double* v = tris + t * 9;
        double e2 = 0.0;
        for (int k = 0; k < 3; ++k) {
            const int a = k, b = (k + 1) % 3;
            const double dx = v[3 * b] - v[3 * a], dy = v[3 * b + 1] - v[3 * a + 1], dz = v[3 * b + 2] - v[3 * a + 2];
            e2 = fmax(e2, dx * dx + dy * dy + dz * dz);
        }
        for (int a = 0; a < 3; ++a) {
            const float c = (float)((v[a] + v[3 + a] + v[6 + a]) * (1.0 / 3.0));
            if (isfinite(c)) { lo[a] = fminf(lo[a], c); nhi[a] = fminf(nhi[a], -c); }
            for (int k = 0; k < 3; ++k)
                nvmax = fminf(nvmax, -__double2float_ru(fabs(v[3 * k + a])));      // NaN is ignored; inf is kept
        }
        nemax = fminf(nemax, -__double2float_ru(sqrt(e2)));
    }
    for (int a = 0; a < 3; ++a) { lo[a] = warp_min(lo[a]); nhi[a] = warp_min(nhi[a]); }
    nvmax = warp_min(nvmax);
    nemax = warp_min(nemax);
    if ((threadIdx.x & 31) == 0) {
        for (int a = 0; a < 3; ++a) {
            atomicMin(bounds + a, fkey(lo[a]));
            atomicMin(bounds + 3 + a, ~fkey(-nhi[a]));
        }
        atomicMin(bounds + 6, ~fkey(-nvmax));
        atomicMin(bounds + 7, ~fkey(-nemax));
    }
}

__device__ __forceinline__ uint32_t spread10(uint32_t x)
{
    x &= 0x3ffu;
    x = (x | (x << 16)) & 0x030000ffu;
    x = (x | (x << 8)) & 0x0300f00fu;
    x = (x | (x << 4)) & 0x030c30c3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}

__global__ void wb_msdf_morton_kernel(const double* __restrict__ tris, int64_t T, const uint32_t* __restrict__ bounds, uint64_t* __restrict__ keys)
{
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= T) return;
    const double* v = tris + t * 9;
    uint32_t code = 0;
    for (int a = 0; a < 3; ++a) {
        const float lo = fkey_inv(bounds[a]), hi = fkey_inv(~bounds[3 + a]);
        const float c = (float)((v[a] + v[3 + a] + v[6 + a]) * (1.0 / 3.0));
        const float ext = hi - lo;
        float q = ext > 0.0f ? (c - lo) * (1023.0f / ext) : 0.0f;
        q = fminf(fmaxf(q, 0.0f), 1023.0f);                 // NaN centroids land on 0
        code |= spread10((uint32_t)q) << (2 - a);
    }
    keys[t] = ((uint64_t)code << 32) | (uint64_t)t;
}

__device__ __forceinline__ int msdf_delta(const uint64_t* __restrict__ k, int64_t n, int64_t i, int64_t j)
{
    return (j < 0 || j >= n) ? -1 : __clzll(k[i] ^ k[j]);
}

// Internal node i of the Karras tree over n unique sorted keys.
__global__ void wb_msdf_karras_kernel(const uint64_t* __restrict__ k, int64_t n, int2* __restrict__ child, int32_t* __restrict__ parent)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const int d = msdf_delta(k, n, i, i + 1) > msdf_delta(k, n, i, i - 1) ? 1 : -1;
    const int dmin = msdf_delta(k, n, i, i - d);
    int64_t lmax = 2;
    while (msdf_delta(k, n, i, i + lmax * d) > dmin) lmax *= 2;
    int64_t l = 0;
    for (int64_t t = lmax / 2; t >= 1; t /= 2)
        if (msdf_delta(k, n, i, i + (l + t) * d) > dmin) l += t;
    const int64_t j = i + l * d;
    const int dnode = msdf_delta(k, n, i, j);
    int64_t s = 0, step = l;
    do {
        step = (step + 1) >> 1;
        if (msdf_delta(k, n, i, i + (s + step) * d) > dnode) s += step;
    } while (step > 1);
    const int64_t gamma = i + s * d + (d < 0 ? -1 : 0);
    const int left = (int)((i < j ? i : j) == gamma ? (n - 1) + gamma : gamma);
    const int right = (int)((i > j ? i : j) == gamma + 1 ? (n - 1) + gamma + 1 : gamma + 1);
    child[i] = make_int2(left, right);
    parent[left] = (int32_t)i;
    parent[right] = (int32_t)i;
    if (i == 0) parent[0] = -1;
}

// Box of one triangle, rounded outward to fp32; a triangle with a NaN coordinate gets the whole space, since the reference's stab
// gives it a negative hit in every direction (its NaN t fails `t >= 0`).
__device__ __forceinline__ void tri_box(const double* v, float4& lo, float4& hi)
{
    double l[3], h[3];
    bool nan = false;
    for (int a = 0; a < 3; ++a) {
        l[a] = fmin(v[a], fmin(v[3 + a], v[6 + a]));
        h[a] = fmax(v[a], fmax(v[3 + a], v[6 + a]));
        nan |= isnan(v[a]) || isnan(v[3 + a]) || isnan(v[6 + a]);
    }
    if (nan) {
        lo = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
        hi = make_float4(INFINITY, INFINITY, INFINITY, 0.0f);
        return;
    }
    lo = make_float4(__double2float_rd(l[0]), __double2float_rd(l[1]), __double2float_rd(l[2]), 0.0f);
    hi = make_float4(__double2float_ru(h[0]), __double2float_ru(h[1]), __double2float_ru(h[2]), 0.0f);
}

__global__ void wb_msdf_refit_kernel(const double* __restrict__ tris_in, const uint64_t* __restrict__ keys, int64_t T,
                                     double* __restrict__ tris, float4* __restrict__ box, const int2* __restrict__ child,
                                     const int32_t* __restrict__ parent, int32_t* __restrict__ flag)
{
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= T) return;
    const double* src = tris_in + (int64_t)(uint32_t)keys[j] * 9;
    double v[9];
    for (int k = 0; k < 9; ++k) { v[k] = src[k]; tris[j * 9 + k] = v[k]; }
    float4 lo, hi;
    tri_box(v, lo, hi);
    int64_t node = T - 1 + j;
    box[2 * node] = lo;
    box[2 * node + 1] = hi;
    if (T == 1) return;
    node = parent[node];
    while (node >= 0) {
        __threadfence();
        if (atomicAdd(flag + node, 1) == 0) return;         // the sibling subtree is not finished: its last thread merges
        const int2 c = child[node];
        const float4 la = __ldcg(box + 2 * c.x), ha = __ldcg(box + 2 * c.x + 1), lb = __ldcg(box + 2 * c.y), hb = __ldcg(box + 2 * c.y + 1);
        box[2 * node] = make_float4(fminf(la.x, lb.x), fminf(la.y, lb.y), fminf(la.z, lb.z), 0.0f);
        box[2 * node + 1] = make_float4(fmaxf(ha.x, hb.x), fmaxf(ha.y, hb.y), fmaxf(ha.z, hb.z), 0.0f);
        node = parent[node];
    }
}

__device__ __forceinline__ double fdot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ void fcross(const double* a, const double* b, double* r)
{
    r[0] = a[1] * b[2] - a[2] * b[1];
    r[1] = a[2] * b[0] - a[0] * b[2];
    r[2] = a[0] * b[1] - a[1] * b[0];
}
// |a x - b|^2 for the edge parameter x
__device__ __forceinline__ double fdist2(const double* a, double x, const double* b)
{
    const double t0 = a[0] * x - b[0], t1 = a[1] * x - b[1], t2 = a[2] * x - b[2];
    return t0 * t0 + t1 * t1 + t2 * t2;
}
// fp32 reciprocal of the fp32-rounded squared length, widened (the reference's idot2: __frcp_rn)
__device__ __forceinline__ double finv2(const double* a) { return (double)__frcp_rn((float)(a[0] * a[0] + a[1] * a[1] + a[2] * a[2])); }
// the edge parameter clamped in fp32 (fmaxf(0, fminf(t, 1)))
__device__ __forceinline__ double fclamp01(double t) { return (double)fmaxf(0.0f, fminf((float)t, 1.0f)); }
__device__ __forceinline__ double fsign(double x) { return (double)copysignf(1.0f, (float)x); }

// One point against one triangle v[9] (fp64), in the reference's arithmetic.
//   dir < 0 : the squared distance, folded into the fp32 running minimum `best` (fminf: a NaN distance is ignored); a triangle with
//             an exactly zero normal adds nothing.
//   dir >= 0: the Moller-Trumbore test along stab direction `dir` only; a hit sets bit 0 of `flags` for t >= 0 and bit 1 otherwise.
__device__ __forceinline__ void wb_msdf_pair(const double* p, const double* v, int dir, float& best, uint32_t& flags)
{
    const double p0[3] = {p[0] - v[0], p[1] - v[1], p[2] - v[2]};
    const double e10[3] = {v[3] - v[0], v[4] - v[1], v[5] - v[2]};
    const double e02[3] = {v[0] - v[6], v[1] - v[7], v[2] - v[8]};
    if (dir < 0) {
        const double e21[3] = {v[6] - v[3], v[7] - v[4], v[8] - v[5]};
        double nor[3];
        fcross(e10, e02, nor);
        if (nor[0] == 0.0 && nor[1] == 0.0 && nor[2] == 0.0) return;
        const double p1[3] = {p[0] - v[3], p[1] - v[4], p[2] - v[5]};
        const double p2[3] = {p[0] - v[6], p[1] - v[7], p[2] - v[8]};
        double c10[3], c21[3], c02[3];
        fcross(e10, nor, c10);
        fcross(e21, nor, c21);
        fcross(e02, nor, c02);
        const double s = fsign(fdot(c10, p0)) + fsign(fdot(c21, p1)) + fsign(fdot(c02, p2));
        double d2;
        if (s < 2.0) {
            const double a = fdist2(e10, fclamp01(fdot(e10, p0) * finv2(e10)), p0);
            const double b = fdist2(e21, fclamp01(fdot(e21, p1) * finv2(e21)), p1);
            const double c = fdist2(e02, fclamp01(fdot(e02, p2) * finv2(e02)), p2);
            d2 = fminf(a, fminf(b, c));
        } else {
            const double dn = fdot(nor, p0);
            d2 = dn * dn * finv2(nor);
        }
        if (d2 < 0.0) d2 = 0.0;
        best = fminf(best, d2);
        return;
    }
    const double d[3] = {(double)kStabDir[dir][0], (double)kStabDir[dir][1], (double)kStabDir[dir][2]};
    const double e20[3] = {-e02[0], -e02[1], -e02[2]};
    double pv[3], qv[3];
    fcross(d, e20, pv);
    const double det = fdot(e10, pv);
    if (det > -1e-8 && det < 1e-8) return;                  // a NaN det is tested on, as in the reference
    const double inv_det = 1.0 / det;
    const double u = fdot(p0, pv) * inv_det;
    if (u < 0.0 || u > 1.0) return;
    fcross(p0, e10, qv);
    const double w = fdot(d, qv) * inv_det;
    if (w < 0.0 || u + w > 1.0) return;
    const double t = fdot(e20, qv) * inv_det;
    flags |= t >= 0.0 ? 1u : 2u;
}

// Lower bound of the squared distance from p to node's box (0 inside).
__device__ __forceinline__ double box_dist2(const float4* __restrict__ box, int node, const double* p)
{
    const float4 lo = __ldg(box + 2 * node), hi = __ldg(box + 2 * node + 1);
    const double gx = fmax(fmax((double)lo.x - p[0], p[0] - (double)hi.x), 0.0);
    const double gy = fmax(fmax((double)lo.y - p[1], p[1] - (double)hi.y), 0.0);
    const double gz = fmax(fmax((double)lo.z - p[2], p[2] - (double)hi.z), 0.0);
    return gx * gx + gy * gy + gz * gz;
}

// Does the infinite line p + t d meet node's box grown by m on every side?
__device__ __forceinline__ bool box_line(const float4* __restrict__ box, int node, const double* p, const double* d, const double* inv_d, double m)
{
    const float4 lo4 = __ldg(box + 2 * node), hi4 = __ldg(box + 2 * node + 1);
    const double lo[3] = {lo4.x, lo4.y, lo4.z}, hi[3] = {hi4.x, hi4.y, hi4.z};
    double tmin = -INFINITY, tmax = INFINITY;
    for (int a = 0; a < 3; ++a) {
        if (d[a] == 0.0) {
            if (p[a] < lo[a] - m || p[a] > hi[a] + m) return false;
        } else {
            const double t1 = (lo[a] - m - p[a]) * inv_d[a], t2 = (hi[a] + m - p[a]) * inv_d[a];
            tmin = fmax(tmin, fmin(t1, t2));
            tmax = fmin(tmax, fmax(t1, t2));
        }
    }
    return tmin <= tmax;
}

// One thread per point.  Culling bounds, with S = max|p_i| + max|vertex coordinate| and E the longest edge:
//  - distance: a subtree is skipped when its box's squared distance d2 satisfies d2 (1 - 2^-20) - 2^-40 S^2 > best.  Every distance
//    the pair test can return for a triangle in the box is at least d2 (1 - 2^-22) - (double rounding, < 2^-45 S^2): the fp32
//    reciprocal idot2 and the fp32 rounding of the result each lose at most 2^-24 relative, and a face distance taken when the
//    projection lies just outside the triangle (a sign flipped by rounding) is short by at most the rounding of that sign's dot
//    product.  So a skipped triangle can never lower the fp32 minimum.
//  - stab: a box is searched only when the line meets it grown by m = 2^-30 S + 2^-40 E^2 (S + E) / 1e-8.  The test rejects
//    |det| < 1e-8, and for |det| >= 1e-8 the barycentric u, v it accepts are off the exact ones by less than
//    10 2^-53 E (S + E) / |det|: the line then passes within 2^-40 E^2 (S + E) / 1e-8 of the triangle, inside the grown box.
//    The 2^-30 S term covers the rounding of the slab test itself.
// The search orders: distance nearest child first; stab one direction at a time, stopping a direction once both flags are set and
// the whole stab once a direction finishes without one of them (outside).
__global__ void __launch_bounds__(kMsdfThreads) wb_msdf_query_kernel(const double* __restrict__ points, int64_t N, const double* __restrict__ tris,
                                                                     const float4* __restrict__ box, const int2* __restrict__ child, int T,
                                                                     const uint32_t* __restrict__ bounds, double* __restrict__ out)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= N) return;
    const double p[3] = {points[3 * i], points[3 * i + 1], points[3 * i + 2]};
    if (isnan(p[0]) || isnan(p[1]) || isnan(p[2])) {        // every distance is NaN and no hit has t >= 0: the rule gives +inf
        out[i] = INFINITY;
        return;
    }
    float best = INFINITY;
    bool inside = false;
    if (T > 0) {
        const double R = (double)fkey_inv(~bounds[6]), E = (double)fkey_inv(~bounds[7]);      // max |vertex coordinate|, longest edge
        const double S = fmax(fabs(p[0]), fmax(fabs(p[1]), fabs(p[2]))) + R;
        const double slack = 0x1p-40 * S * S;
        const int leaf0 = T - 1;
        int stack[kMsdfStack];
        double lbs[kMsdfStack];
        uint32_t unused = 0;

        int sp = 0, node = 0;
        for (;;) {
            if (node >= leaf0) {
                wb_msdf_pair(p, tris + (int64_t)(node - leaf0) * 9, -1, best, unused);
            } else {
                const int2 c = __ldg(child + node);
                const double l0 = box_dist2(box, c.x, p), l1 = box_dist2(box, c.y, p);
                const bool v0 = !(l0 * (1.0 - 0x1p-20) - slack > (double)best), v1 = !(l1 * (1.0 - 0x1p-20) - slack > (double)best);
                if (v0 && v1) {
                    const bool first = l0 <= l1;
                    stack[sp] = first ? c.y : c.x;
                    lbs[sp++] = first ? l1 : l0;
                    node = first ? c.x : c.y;
                    continue;
                }
                if (v0 || v1) { node = v0 ? c.x : c.y; continue; }
            }
            bool found = false;
            while (sp > 0) {
                --sp;
                if (!(lbs[sp] * (1.0 - 0x1p-20) - slack > (double)best)) { node = stack[sp]; found = true; break; }
            }
            if (!found) break;
        }

        const double m = 0x1p-30 * S + 0x1p-40 * E * E * (S + E) * 1e8;
        inside = true;
        for (int dir = 0; dir < 13 && inside; ++dir) {
            const double d[3] = {(double)kStabDir[dir][0], (double)kStabDir[dir][1], (double)kStabDir[dir][2]};
            const double inv_d[3] = {1.0 / d[0], 1.0 / d[1], 1.0 / d[2]};
            uint32_t flags = 0;
            sp = 0;
            node = 0;
            bool go = node >= leaf0 || box_line(box, node, p, d, inv_d, m);
            while (go) {
                if (node >= leaf0) {
                    wb_msdf_pair(p, tris + (int64_t)(node - leaf0) * 9, dir, best, flags);
                    if (flags == 3u) break;
                } else {
                    const int2 c = __ldg(child + node);
                    const bool h0 = box_line(box, c.x, p, d, inv_d, m), h1 = box_line(box, c.y, p, d, inv_d, m);
                    if (h0 && h1) { stack[sp++] = c.y; node = c.x; continue; }
                    if (h0 || h1) { node = h0 ? c.x : c.y; continue; }
                }
                if (sp == 0) break;
                node = stack[--sp];
            }
            inside = flags == 3u;
        }
    }
    if (best < 0.0f) best = 0.0f;
    const double dist = (double)sqrtf(best);
    out[i] = inside ? -dist : dist;
}

}  // namespace

extern "C" int64_t wb_mesh_sdf_workspace_bytes(int64_t num_triangles)
{
    if (num_triangles < 0 || num_triangles >= ((int64_t)1 << 31)) {
        wb_set_error("%s: num_triangles out of range", __func__);
        return -1;
    }
    MsdfWs w;
    if (msdf_layout(num_triangles, &w)) {
        wb_set_error("%s: the sort's workspace query failed", __func__);
        return -1;
    }
    return (int64_t)w.total;
}

extern "C" int wb_mesh_sdf(const double* tris, int64_t num_triangles, const double* points, int64_t num_points, void* workspace,
                           int64_t workspace_bytes, double* out, wb_stream s)
{
    const int64_t T = num_triangles, N = num_points;
    WB_CHECK_ARG(T >= 0 && T < ((int64_t)1 << 31), "num_triangles out of range");
    WB_CHECK_ARG(N >= 0 && N < ((int64_t)1 << 31) * kMsdfThreads, "num_points out of range");
    if (N == 0) return WB_OK;
    WB_CHECK_ARG(points && out && (tris || T == 0), "null pointer");
    MsdfWs w;
    WB_CHECK_ARG(msdf_layout(T, &w) == 0, "the sort's workspace query failed");
    WB_CHECK_ARG(workspace && workspace_bytes >= (int64_t)w.total, "workspace too small (wb_mesh_sdf_workspace_bytes)");
    cudaStream_t st = (cudaStream_t)s;
    char* ws = static_cast<char*>(workspace);
    uint32_t* bounds = reinterpret_cast<uint32_t*>(ws + w.bounds);
    uint64_t* keys_in = reinterpret_cast<uint64_t*>(ws + w.keys_in);
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + w.keys_out);
    double* leaf_tris = reinterpret_cast<double*>(ws + w.tris);
    float4* box = reinterpret_cast<float4*>(ws + w.box);
    int2* child = reinterpret_cast<int2*>(ws + w.child);
    int32_t* parent = reinterpret_cast<int32_t*>(ws + w.parent);
    int32_t* flag = reinterpret_cast<int32_t*>(ws + w.flag);
    if (T > 0) {
        const unsigned tb = (unsigned)((T + kMsdfThreads - 1) / kMsdfThreads);
        WB_CUDA(cudaMemsetAsync(bounds, 0xff, 8 * sizeof(uint32_t), st));
        if (T > 1) WB_CUDA(cudaMemsetAsync(flag, 0, (size_t)(T - 1) * sizeof(int32_t), st));
        wb_msdf_bounds_kernel<<<(unsigned)std::min<int64_t>(tb, 4 * (int64_t)wb_num_sms()), kMsdfThreads, 0, st>>>(tris, T, bounds);
        WB_LAUNCH_CHECK();
        wb_msdf_morton_kernel<<<tb, kMsdfThreads, 0, st>>>(tris, T, bounds, keys_in);
        WB_LAUNCH_CHECK();
        size_t cub_bytes = w.cub_bytes;
        WB_CUDA(cub::DeviceRadixSort::SortKeys(ws + w.cub, cub_bytes, (const uint64_t*)keys_in, keys, (int)T, 0, 62, st));
        WB_LAUNCH_CHECK();
        if (T > 1) {
            wb_msdf_karras_kernel<<<(unsigned)((T - 1 + kMsdfThreads - 1) / kMsdfThreads), kMsdfThreads, 0, st>>>(keys, T, child, parent);
            WB_LAUNCH_CHECK();
        }
        wb_msdf_refit_kernel<<<tb, kMsdfThreads, 0, st>>>(tris, keys, T, leaf_tris, box, child, parent, flag);
        WB_LAUNCH_CHECK();
    }
    wb_msdf_query_kernel<<<(unsigned)((N + kMsdfThreads - 1) / kMsdfThreads), kMsdfThreads, 0, st>>>(points, N, leaf_tris, box, child, (int)T,
                                                                                                    bounds, out);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
