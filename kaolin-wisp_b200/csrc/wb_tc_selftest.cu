// wb_tc_selftest.cu -- one-tile wgmma GEMM used by the GPU tests to pin the operand layouts of wb_tc.cuh
// (K-major / MN-major shared-memory descriptors, the accumulator fragment mapping) against a reference matmul.
// The tiles are 128 samples high (slab = 2048 bytes; each of the two warpgroups computes 64 rows of D) or, with mode bit 4, 64
// samples high like the decoder kernels' tiles (slab = 1024 bytes; modes 0 / 1: one warpgroup).
#include "wb_common.cuh"
#include "wb_tc.cuh"

// R = 128 samples, or 64 with mode bit 4:
// mode 0 (forward)   : D[R x N] = A[R x K] . W[N x K]^T       A: sample tile K-major,  B: weight pack (N x K) K-major
// mode 1 (data grad) : D[R x N] = A[R x K] . W[K x N]         A: sample tile K-major,  B: weight pack (K x N) read MN-major
// mode 2 (weight grad): D[128 x N] = A^T . B                  A: sample tile [R samples x 128 features] MN-major,
//                                                               B: sample tile [R samples x N] MN-major, K = R samples
// N = 8 (mode 2) is the bias-gradient chain of the decoder backward (B = the constant-one slab).
template <int N, int TA, int TB>
__device__ __forceinline__ void tc_selftest_tile(uint64_t da, uint64_t db, int nk, uint32_t aadv, uint32_t badv, float* __restrict__ D, int row0)
{
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.0f;
    tc_wg_fence();
    for (int kb = 0; kb < nk; ++kb) { WgMma<N, TA, TB>::run(d, da, db, 1u); da += aadv; db += badv; }
    tc_wg_commit();
    tc_wg_wait0();
    tc_wg_hold(d);
    const int wl = threadIdx.x & 127;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) D[(row0 + tc_frag_row(wl, i)) * N + tc_frag_col(wl, i)] = d[i];
}

template <int N>
__device__ __forceinline__ void tc_selftest_mode(int mode, int rows, uint32_t a0, uint32_t b0, int K, float* D)
{
    const int wg = threadIdx.x >> 7;                                  // warpgroup: rows 64*wg .. +63 of D
    const int slab = rows * 16;
    if (mode != 2 && 64 * wg >= rows) return;
    if (mode == 0)        // A rows 64*wg.. at +1024*wg; per K step: 2 slabs of A, 2 K-chunks of the weight pack
        tc_selftest_tile<N, 0, 0>(tc_desc(a0 + wg * 1024, slab, 128), tc_desc(b0, N * 16, 128), K / 16, (2 * slab) >> 4, (2 * N * 16) >> 4, D, 64 * wg);
    else if (mode == 1)   // weight pack of W[K x N] (out = K, in = N): element (o=k, i=n) at (n/8)*(K*16) + k*16 + (n%8)*2
        tc_selftest_tile<N, 0, 1>(tc_desc(a0 + wg * 1024, slab, 128), tc_desc(b0, 128, K * 16), K / 16, (2 * slab) >> 4, 256 >> 4, D, 64 * wg);
    else                  // M = features 64*wg.. = 8 slabs further per warpgroup; K = the tile's samples
        tc_selftest_tile<N, 1, 1>(tc_desc(a0 + wg * 8 * slab, 128, slab), tc_desc(b0, 128, slab), rows / 16, 256 >> 4, 256 >> 4, D, 64 * wg);
}

__global__ void __launch_bounds__(256)
wb_tc_selftest_kernel(const uint4* __restrict__ a_img, int a_bytes, const uint4* __restrict__ b_img, int b_bytes,
                      float* __restrict__ D, int N, int K, int mode)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sa = smem; uint8_t* sb = smem + ((a_bytes + 1023) & ~1023);
    for (int i = threadIdx.x; i < a_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sa)[i] = a_img[i];
    for (int i = threadIdx.x; i < b_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sb)[i] = b_img[i];
    tc_fence_smem_async();
    __syncthreads();
    const uint32_t a0 = tc_smem_u32(sa), b0 = tc_smem_u32(sb);
    const int rows = (mode & 4) ? 64 : 128;
    mode &= 3;
    switch (N) {
        case 8: tc_selftest_mode<8>(mode, rows, a0, b0, K, D); break;
        case 16: tc_selftest_mode<16>(mode, rows, a0, b0, K, D); break;
        case 32: tc_selftest_mode<32>(mode, rows, a0, b0, K, D); break;
        case 48: tc_selftest_mode<48>(mode, rows, a0, b0, K, D); break;
        case 64: tc_selftest_mode<64>(mode, rows, a0, b0, K, D); break;
        case 80: tc_selftest_mode<80>(mode, rows, a0, b0, K, D); break;
        case 96: tc_selftest_mode<96>(mode, rows, a0, b0, K, D); break;
        case 112: tc_selftest_mode<112>(mode, rows, a0, b0, K, D); break;
        default: tc_selftest_mode<128>(mode, rows, a0, b0, K, D); break;
    }
}

extern "C" int wb_tc_selftest(const void* a_img, int a_bytes, const void* b_img, int b_bytes, float* D, int N, int K, int mode, wb_stream s)
{
    WB_CHECK_ARG(a_img && b_img && D, "null pointer");
    WB_CHECK_ARG((N == 8 || (N % 16 == 0 && N >= 16 && N <= 128)) && K % 16 == 0 && (mode & 3) <= 2 && a_bytes % 16 == 0 && b_bytes % 16 == 0, "bad shape");
    const size_t smem = ((a_bytes + 1023) & ~1023) + b_bytes + 1024;
    WB_CHECK_ARG(smem <= 200 * 1024, "tiles too large");
    WB_CUDA(cudaFuncSetAttribute(wb_tc_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    wb_tc_selftest_kernel<<<1, 256, smem, (cudaStream_t)s>>>(reinterpret_cast<const uint4*>(a_img), a_bytes, reinterpret_cast<const uint4*>(b_img), b_bytes, D, N, K, mode);
    WB_LAUNCH_CHECK();
    return WB_OK;
}
