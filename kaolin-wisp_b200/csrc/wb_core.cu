// wb_core.cu -- error channel, launch accounting and descriptor validation of libwispb200.
#include "wb_common.cuh"
#include "wb_featx.cuh"
#include <stdarg.h>
#include <atomic>
#include <map>
#include <mutex>
#include <utility>
#include <math.h>

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void wb_set_error(const char* fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}
void wb_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int wb_cur_device() { int dev = 0; cudaGetDevice(&dev); return dev < 0 ? 0 : (dev & 63); }
cudaError_t wb_allow_smem_fn(const void* kernel, int64_t bytes) {
    if (bytes <= 48 * 1024) return cudaSuccess;                  // the default limit of every kernel
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, int64_t> allowed;
    const int dev = wb_cur_device();
    std::lock_guard<std::mutex> lock(mu);
    int64_t& cur = allowed[std::make_pair(kernel, dev)];
    if (cur >= bytes) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) cur = bytes;
    return e;
}
int wb_num_sms() {
    static std::atomic<int> sms[64];
    const int dev = wb_cur_device();
    int v = sms[dev].load(std::memory_order_relaxed);
    if (v == 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 148;
        sms[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}

extern "C" const char* wb_last_error(void) { return g_err; }
extern "C" int wb_version(void) { return 100; }
extern "C" int64_t wb_launch_count(void) { return g_launches.load(); }

extern "C" int wb_device_check(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { wb_set_error("wb_device_check: no CUDA device (there is no CPU fallback)"); return WB_ERR_NODEVICE; }
    WB_CHECK_ARG(device >= 0 && device < n, "device index out of range");
    int major = 0, minor = 0;
    WB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    WB_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    if (major != 9 || minor != 0) { wb_set_error("wb_device_check: device %d is sm_%d%d; libwispb200 is built for sm_90a only", device, major, minor); return WB_ERR_NODEVICE; }
    return WB_OK;
}

int wb_make_grid(const wb_nef_desc* d, WbGrid* g) {
    WB_CHECK_ARG(d != nullptr, "null descriptor");
    WB_CHECK_ARG(d->num_lods >= 1 && d->num_lods <= WB_MAX_LODS, "num_lods out of range");
    WB_CHECK_ARG(d->multiscale == 0 || d->multiscale == 1, "multiscale must be 0 ('cat') or 1 ('sum')");
    memset(g, 0, sizeof(*g));
    g->L = d->num_lods; g->F = d->feature_dim; g->multiscale = d->multiscale; g->lod_idx = d->lod_idx;
    if (d->grid_kind != 0) {                 // triplanar / octree: the features come from wb_featx_gather (WbGridX), not from a table
        WB_CHECK_ARG(d->grid_kind == 1 || d->grid_kind == 2, "grid_kind must be 0 (hash), 1 (triplanar) or 2 (octree)");
        WB_CHECK_ARG(d->feature_dim >= 1 && d->feature_dim <= 64, "feature width out of range");
        g->lod_idx = d->num_lods;
        return WB_OK;
    }
    WB_CHECK_ARG(d->feature_dim >= 1 && d->feature_dim <= 8, "feature_dim must be in [1,8]");
    WB_CHECK_ARG(d->codebook_size > 0 && (d->codebook_size & (d->codebook_size - 1)) == 0, "codebook_size must be a power of two");
    WB_CHECK_ARG(d->table != nullptr, "null table");
    g->table = d->table; g->Tmask = (uint32_t)d->codebook_size - 1u;
    const int64_t T = d->codebook_size;
    for (int l = 0; l < d->num_lods; ++l) {
        int res = d->resolutions[l];
        WB_CHECK_ARG(res >= 2 && res < (1 << 20), "resolution out of range");
        int64_t r2 = (int64_t)res * res, r3 = r2 * res;
        g->res[l] = res; g->hres[l] = 0.5f * (float)res;
        g->hi[l] = (float)((double)(res - 1) - 1e-5);          // clamp upper bound, cu:40
        g->dense[l] = (res < T && r2 < T && r3 < T) ? 1 : 0;   // hash_utils.cuh:27-29
        g->begin[l] = d->begin_idxes[l];
    }
    g->begin[d->num_lods] = d->begin_idxes[d->num_lods];
    return WB_OK;
}

int wb_make_decoders(const wb_nef_desc* d, int max_width, const char* width_msg, WbDecoders* dec) {
    WB_CHECK_ARG(d->dens_layers >= 1 && d->dens_layers <= WB_MAX_LAYERS && d->col_layers >= 1 && d->col_layers <= WB_MAX_LAYERS, "unsupported decoder depth");
    WB_CHECK_ARG(d->dens_params && d->col_params, "null decoder parameters");
    memset(dec, 0, sizeof(*dec));
    dec->nl_d = d->dens_layers; dec->nl_c = d->col_layers;
    dec->feat_dim = d->multiscale == 0 ? d->num_lods * d->feature_dim : d->feature_dim;
    dec->pos_dim = wb_embed_dim(d->pos_mode, d->pos_freq); dec->view_dim = wb_embed_dim(d->view_mode, d->view_freq);
    WB_CHECK_ARG(d->dens_dims[0] == dec->feat_dim + dec->pos_dim, "decoder_density input width != grid features + position embedding");
    WB_CHECK_ARG(d->col_dims[0] == d->dens_dims[d->dens_layers] - 1 + dec->view_dim, "decoder_color input width != density feats - 1 + view embedding");
    WB_CHECK_ARG(d->col_dims[d->col_layers] == 3, "decoder_color output must be 3 wide");
    int srcd = 0, srcc = 0;
    for (int l = 0; l < dec->nl_d + dec->nl_c; ++l) {
        const bool dens = l < dec->nl_d;
        const int I = dens ? d->dens_dims[l] : d->col_dims[l - dec->nl_d];
        const int O = dens ? d->dens_dims[l + 1] : d->col_dims[l - dec->nl_d + 1];
        WB_CHECK_ARG(I >= 1 && I <= max_width && O >= 1 && O <= max_width, width_msg);
        dec->I[l] = I; dec->O[l] = O;
        int& src = dens ? srcd : srcc;
        dec->src_w[l] = src; src += I * O;
        if (d->has_bias) { dec->src_b[l] = src; src += O; } else dec->src_b[l] = -1;
    }
    return WB_OK;
}

int wb_make_gridx(const wb_nef_desc* d, bool backward, WbGridX* x) {
    WB_CHECK_ARG(d != nullptr, "null descriptor");
    memset(x, 0, sizeof(*x));
    x->kind = d->grid_kind;
    if (d->grid_kind == 0) return WB_OK;
    WB_CHECK_ARG(d->grid_kind == 1 || d->grid_kind == 2, "grid_kind must be 0 (hash), 1 (triplanar) or 2 (octree)");
    WB_CHECK_ARG(d->num_lods >= 1 && d->num_lods <= WB_X_MAX_LODS, "triplanar / octree grids: at most 12 LODs on the fused path");
    WB_CHECK_ARG(d->grid_ptrs != nullptr && (!backward || d->grid_grads != nullptr), "null grid_ptrs / grid_grads");
    x->nl = d->num_lods; x->sum = d->multiscale;
    const int np = d->grid_kind == 1 ? 3 * d->num_lods : d->num_lods;
    for (int i = 0; i < np; ++i) {
        WB_CHECK_ARG(d->grid_ptrs[i] != nullptr && (!backward || d->grid_grads[i] != nullptr), "null grid tensor");
        x->ptr[i] = d->grid_ptrs[i]; x->gptr[i] = backward ? d->grid_grads[i] : nullptr;
    }
    if (d->grid_kind == 1) {
        WB_CHECK_ARG(d->feature_dim % 3 == 0 && d->feature_dim / 3 <= WB_X_MAX_C, "triplanar: feature_dim = 3 * fdim, fdim <= 8");
        x->C = d->feature_dim / 3;
        WB_CHECK_ARG(d->grid_layout == 0 || (d->grid_layout == 1 && x->C == 4), "triplanar: channel-last planes need fdim == 4");
        x->chlast = d->grid_layout;
        for (int l = 0; l < d->num_lods; ++l) { WB_CHECK_ARG(d->resolutions[l] >= 1, "plane resolution must be >= 1"); x->res[l] = d->resolutions[l]; }
    } else {
        WB_CHECK_ARG(d->feature_dim <= WB_X_MAX_F, "octree: feature_dim <= 32 on the fused path");
        WB_CHECK_ARG(d->oct && d->oct->octree && d->oct->prefix && d->points && d->trinkets, "octree grid: null octree / points / trinkets");
        WB_CHECK_ARG(d->base_lod >= 0 && d->base_lod + d->num_lods - 1 <= d->oct->max_level && d->base_lod + d->num_lods - 1 <= 15, "octree grid: LOD range outside the octree");
        x->C = d->feature_dim; x->octree = d->oct->octree; x->prefix = d->oct->prefix; x->points = d->points; x->trinkets = d->trinkets;
        x->base_lod = d->base_lod; x->half_round = d->half_round;
    }
    return WB_OK;
}

int wb_make_march(const wb_rays* rays, int n, const float* jitter, uint32_t seed, WbMarch* m) {
    WB_CHECK_ARG(rays != nullptr && (rays->num_rays == 0 || (rays->origins && rays->dirs)), "null rays");
    WB_CHECK_ARG(rays->num_rays >= 0 && rays->num_rays < ((int64_t)1 << 31), "num_rays out of range");
    WB_CHECK_ARG(n >= 1 && n <= (1 << 20), "num_samples out of range");
    WB_CHECK_ARG((rays->near_v == nullptr) == (rays->far_v == nullptr), "near_v and far_v must both be given or both be NULL");
    m->origins = rays->origins; m->dirs = rays->dirs; m->near_v = rays->near_v; m->far_v = rays->far_v;
    m->jitter = jitter; m->near_s = rays->dist_min;
    m->range_s = (float)((double)rays->dist_max - (double)rays->dist_min);
    m->step = n > 1 ? 1.0f / (float)(n - 1) : 0.0f;
    m->n_pow2 = (n & (n - 1)) == 0; m->inv_n = 1.0f / (float)n;
    m->n = n; m->seed = seed; m->R = rays->num_rays;
    return WB_OK;
}

int wb_make_oct(const wb_octree* o, int level, WbOct* out) {
    WB_CHECK_ARG(o != nullptr && o->octree && o->prefix, "null octree");
    WB_CHECK_ARG(level >= 0 && level <= o->max_level && level <= 15, "level out of range");
    out->octree = o->octree; out->prefix = o->prefix; out->bits = o->bits; out->level = level;
    out->use_bits = (o->bits != nullptr && o->bits_level == level && level <= 10) ? 1 : 0;
    out->h = ldexpf(1.0f, level - 1); out->inv_h = ldexpf(1.0f, -(level - 1)); out->maxq = (float)((1 << level) - 1);
    out->has_bbox = (o->has_bbox && o->bits_level == level) ? 1 : 0;
    for (int a = 0; a < 3; ++a) {   // widen by 1e-4: far above the fp32 error of p = fma(d,t,o) near the unit cube
        out->blo[a] = fmaxf(o->bbox_lo[a], -1.0f) - 1e-4f; out->bhi[a] = fminf(o->bbox_hi[a], 1.0f) + 1e-4f;
    }
    const bool coarse_ok = out->has_bbox && o->coarse_bits != nullptr && o->coarse_level >= 1 && o->coarse_level < level;
    out->coarse = coarse_ok ? o->coarse_bits : nullptr; out->clevel = coarse_ok ? o->coarse_level : 0;
    out->ch = ldexpf(1.0f, out->clevel - 1); out->cmax = (float)((1 << out->clevel) - 1);
    return WB_OK;
}
