// ref_shim_mesh.cpp -- TEST INFRASTRUCTURE.  C entry points around the REFERENCE's own mesh-to-SDF kernel:
//   mesh2sdf_gpu_fast_nopre (wisp/csrc/external/mesh2sdf_kernel.cu:1251-1283), what wisp.ops.mesh.compute_sdf calls through
//   wisp._C.external.mesh_to_sdf_cuda for each split of the points.
// Built by oracle/ref_kernels/build_ref_mesh.py, together with that file compiled unchanged, into oracle/_ref/libwisp_ref_mesh2sdf.so;
// oracle/make_ref_golden_mesh.py stores what it computes for tests/test_gpu_mesh_sdf.py.  Nothing here is product code.
#include <ATen/ATen.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <vector>

std::vector<at::Tensor> mesh2sdf_gpu_fast_nopre(at::Tensor& points, at::Tensor& mesh);

static thread_local char g_err[1024] = "";
#define REF_TRY(body) try { body; return 0; } catch (const std::exception& e) { snprintf(g_err, sizeof(g_err), "%s", e.what()); return -1; }

extern "C" const char* ref_mesh_last_error(void) { return g_err; }

// points f64 [N, 3], mesh f64 [T, 3, 3] (V[F]) on `device` -> out f64 [N], the kernel's result for one split.
extern "C" int ref_mesh2sdf(int device, const double* points, int64_t N, const double* mesh, int64_t T, double* out)
{
    REF_TRY({
        auto o = at::TensorOptions().dtype(at::kDouble).device(at::kCUDA, device);
        auto p = at::from_blob((void*)points, {N, 3}, o);
        auto m = at::from_blob((void*)mesh, {T, 3, 3}, o);
        auto r = mesh2sdf_gpu_fast_nopre(p, m)[0];
        at::from_blob((void*)out, {N}, o).copy_(r);
        cudaDeviceSynchronize();
    })
}

// The same call on float32 inputs, as wisp's SDF datasets pass them (load_obj's FloatTensor vertices, the samplers' float32 points):
// returns -1 with the exception's message when the reference refuses them.
extern "C" int ref_mesh2sdf_f32(int device, const float* points, int64_t N, const float* mesh, int64_t T)
{
    REF_TRY({
        auto o = at::TensorOptions().dtype(at::kFloat).device(at::kCUDA, device);
        auto p = at::from_blob((void*)points, {N, 3}, o);
        auto m = at::from_blob((void*)mesh, {T, 3, 3}, o);
        mesh2sdf_gpu_fast_nopre(p, m);
        cudaDeviceSynchronize();
    })
}
