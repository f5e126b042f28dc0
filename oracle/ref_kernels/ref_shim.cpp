// ref_shim.cpp -- TEST INFRASTRUCTURE.  C entry points around the REFERENCE's own CUDA operators (compiled from the sources under
// a kaolin-wisp checkout's wisp/csrc by oracle/ref_kernels/build_ref.py into oracle/_ref/libwisp_ref_kernels.so), so that
// oracle/make_ref_golden.py can store what the kernels this repository replaces compute, for the GPU tests:
//   wisp::hashgrid_interpolate_cuda / _backward_cuda   (wisp/csrc/ops/hashgrid_interpolate.cpp:46-105, hashgrid_interpolate_cuda.cu)
//   wisp::uniform_sample_cuda                          (wisp/csrc/ops/uniform_sample.cpp:28-42, uniform_sample_cuda.cu)
//   wisp::find_depth_bound_cuda                        (wisp/csrc/render/find_depth_bound.cpp:23-36, find_depth_bound_cuda.cu)
// Nothing here is product code: only tests/ load the library, and only when it exists.  Raw device pointers in, results copied into
// caller-provided device buffers; tensors are views (at::from_blob) on the caller's memory.
#include <ATen/ATen.h>
#include <cuda_runtime.h>
#include <vector>

namespace wisp {
at::Tensor hashgrid_interpolate_cuda(at::Tensor coords, at::Tensor codebook, at::Tensor codebook_first_idx, at::Tensor resolution, int32_t codebook_bitwidth);
std::vector<at::Tensor> hashgrid_interpolate_backward_cuda(at::Tensor coords, at::Tensor grad_output, at::Tensor codebook, at::Tensor codebook_first_idx,
                                                           at::Tensor resolution, int32_t codebook_bitwidth, int32_t feature_dim, bool require_grad_coords);
std::vector<at::Tensor> uniform_sample_cuda(int scale, at::Tensor ridx, at::Tensor depth, at::Tensor insum);
at::Tensor find_depth_bound_cuda(at::Tensor query, at::Tensor curr_idxes_in, at::Tensor depth);
}

static at::TensorOptions dev_opts(at::ScalarType t, int device) { return at::TensorOptions().dtype(t).device(at::kCUDA, device); }
static thread_local char g_err[512] = "";
#define REF_TRY(body) try { body; return 0; } catch (const std::exception& e) { snprintf(g_err, sizeof(g_err), "%s", e.what()); return -1; }

extern "C" const char* ref_last_error(void) { return g_err; }

// feats [N, L*F] fp32 (the raw kernel output, before HashGrid.interpolate's 'cat' zeroing / 'sum')
extern "C" int ref_hashgrid_fwd(int device, const float* coords, int64_t N, const float* table, int64_t rows, int F, const int64_t* first_idx_dev, int L,
                                const int64_t* resolutions_host, int bitwidth, float* feats)
{
    REF_TRY({
        auto c = at::from_blob((void*)coords, {N, 3}, dev_opts(at::kFloat, device));
        auto cb = at::from_blob((void*)table, {rows, F}, dev_opts(at::kFloat, device));
        auto fi = at::from_blob((void*)first_idx_dev, {L + 1}, dev_opts(at::kLong, device));
        auto res = at::from_blob((void*)resolutions_host, {L, 1}, at::TensorOptions().dtype(at::kLong));       // CPU tensor, as MultiTable.resolutions
        auto out = wisp::hashgrid_interpolate_cuda(c, cb, fi, res, bitwidth);
        auto dst = at::from_blob((void*)feats, {N, (int64_t)L * F}, dev_opts(at::kFloat, device));
        dst.copy_(out.reshape({N, (int64_t)L * F}));
        cudaDeviceSynchronize();
    })
}
extern "C" int ref_hashgrid_bwd(int device, const float* coords, int64_t N, const float* grad_feats, const float* table, int64_t rows, int F,
                                const int64_t* first_idx_dev, int L, const int64_t* resolutions_host, int bitwidth, float* grad_table)
{
    REF_TRY({
        auto c = at::from_blob((void*)coords, {N, 3}, dev_opts(at::kFloat, device));
        auto g = at::from_blob((void*)grad_feats, {N, (int64_t)L * F}, dev_opts(at::kFloat, device));
        auto cb = at::from_blob((void*)table, {rows, F}, dev_opts(at::kFloat, device));
        auto fi = at::from_blob((void*)first_idx_dev, {L + 1}, dev_opts(at::kLong, device));
        auto res = at::from_blob((void*)resolutions_host, {L, 1}, at::TensorOptions().dtype(at::kLong));
        auto out = wisp::hashgrid_interpolate_backward_cuda(c, g, cb, fi, res, bitwidth, F, false);
        auto dst = at::from_blob((void*)grad_table, {rows, F}, dev_opts(at::kFloat, device));
        dst.copy_(out[1].reshape({rows, F}));
        cudaDeviceSynchronize();
    })
}
// total = insum[V-1]; outputs sized by the caller: ridx i64 [total], depth f32 [total], boundary u8 [total]
extern "C" int ref_uniform_sample(int device, int scale, const int32_t* nug_ridx, const float* nug_depth, const int32_t* insum, int64_t V, int64_t total,
                                  int64_t* ridx, float* depth, uint8_t* boundary)
{
    REF_TRY({
        auto r = at::from_blob((void*)nug_ridx, {V}, dev_opts(at::kInt, device));
        auto d = at::from_blob((void*)nug_depth, {V, 2}, dev_opts(at::kFloat, device));
        auto s = at::from_blob((void*)insum, {V}, dev_opts(at::kInt, device));
        auto out = wisp::uniform_sample_cuda(scale, r, d, s);
        TORCH_CHECK(out[0].size(0) == total, "uniform_sample_cuda returned ", out[0].size(0), " samples, caller expected ", total);
        at::from_blob((void*)ridx, {total}, dev_opts(at::kLong, device)).copy_(out[0]);
        at::from_blob((void*)depth, {total}, dev_opts(at::kFloat, device)).copy_(out[1].reshape({total}));
        at::from_blob((void*)boundary, {total}, dev_opts(at::kBool, device)).copy_(out[2]);
        cudaDeviceSynchronize();
    })
}
extern "C" int ref_find_depth_bound(int device, const float* query, const int32_t* curr_idxes, const float* depth, int64_t P, int64_t Ng, int32_t* out)
{
    REF_TRY({
        auto q = at::from_blob((void*)query, {P, 1}, dev_opts(at::kFloat, device));
        auto ci = at::from_blob((void*)curr_idxes, {P}, dev_opts(at::kInt, device));
        auto dp = at::from_blob((void*)depth, {Ng, 2}, dev_opts(at::kFloat, device));
        auto o = wisp::find_depth_bound_cuda(q, ci, dp);
        at::from_blob((void*)out, {P}, dev_opts(at::kInt, device)).copy_(o);
        cudaDeviceSynchronize();
    })
}
