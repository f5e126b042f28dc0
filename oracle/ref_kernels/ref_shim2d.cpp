// ref_shim2d.cpp -- TEST INFRASTRUCTURE.  C entry points around the REFERENCE's own 2-D hash-grid kernels (app/image):
//   wisp::hashgrid_interpolate_cuda / _backward_cuda on [N, 2] coordinates, which pick hashgrid_interpolate_2d_cuda_kernel and its
//   backward from coords.size(1) (wisp/csrc/ops/hashgrid_interpolate_cuda.cu:214-339, dispatch at :374).
// Built by oracle/ref_kernels/build_ref2d.py into oracle/_ref/libwisp_ref_hashgrid2d.so against the operators that
// oracle/ref_kernels/build_ref.py compiled into oracle/_ref/libwisp_ref_kernels.so; oracle/make_ref_golden2d.py stores what they compute
// for tests/test_gpu_ref_hashgrid2d.py.  Nothing here is product code.  Raw device pointers in, results copied into caller-provided
// device buffers; tensors are views (at::from_blob) on the caller's memory.
#include <ATen/ATen.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <vector>

namespace wisp {
at::Tensor hashgrid_interpolate_cuda(at::Tensor coords, at::Tensor codebook, at::Tensor codebook_first_idx, at::Tensor resolution, int32_t codebook_bitwidth);
std::vector<at::Tensor> hashgrid_interpolate_backward_cuda(at::Tensor coords, at::Tensor grad_output, at::Tensor codebook, at::Tensor codebook_first_idx,
                                                           at::Tensor resolution, int32_t codebook_bitwidth, int32_t feature_dim, bool require_grad_coords);
}

static at::TensorOptions dev_opts(at::ScalarType t, int device) { return at::TensorOptions().dtype(t).device(at::kCUDA, device); }
static thread_local char g_err[512] = "";
#define REF_TRY(body) try { body; return 0; } catch (const std::exception& e) { snprintf(g_err, sizeof(g_err), "%s", e.what()); return -1; }

extern "C" const char* ref2d_last_error(void) { return g_err; }

// feats [N, L*F] fp32 (the raw kernel output, before HashGrid.interpolate's 'cat' zeroing / 'sum')
extern "C" int ref_hashgrid2d_fwd(int device, const float* coords, int64_t N, const float* table, int64_t rows, int F, const int64_t* first_idx_dev,
                                  int L, const int64_t* resolutions_host, int bitwidth, float* feats)
{
    REF_TRY({
        auto c = at::from_blob((void*)coords, {N, 2}, dev_opts(at::kFloat, device));
        auto cb = at::from_blob((void*)table, {rows, F}, dev_opts(at::kFloat, device));
        auto fi = at::from_blob((void*)first_idx_dev, {L + 1}, dev_opts(at::kLong, device));
        auto res = at::from_blob((void*)resolutions_host, {L, 1}, at::TensorOptions().dtype(at::kLong));       // CPU tensor, as MultiTable.resolutions
        auto out = wisp::hashgrid_interpolate_cuda(c, cb, fi, res, bitwidth);
        auto dst = at::from_blob((void*)feats, {N, (int64_t)L * F}, dev_opts(at::kFloat, device));
        dst.copy_(out.reshape({N, (int64_t)L * F}));
        cudaDeviceSynchronize();
    })
}
extern "C" int ref_hashgrid2d_bwd(int device, const float* coords, int64_t N, const float* grad_feats, const float* table, int64_t rows, int F,
                                  const int64_t* first_idx_dev, int L, const int64_t* resolutions_host, int bitwidth, float* grad_table)
{
    REF_TRY({
        auto c = at::from_blob((void*)coords, {N, 2}, dev_opts(at::kFloat, device));
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
