// wb_tc.cuh -- wgmma / mbarrier / bulk-copy primitives for the tensor-core decoder kernels (sm_90a).
//
// Operand layouts (no swizzle, "interleaved" canonical form of the wgmma shared-memory descriptor):
//   core matrix = 8 rows x 16 bytes (8 fp16), stored contiguously (128 B).
//   SAMPLE TILE  [R samples x C features], C multiple of 8, "slab" layout (one slab = 8 features of all R samples, R * 16 bytes):
//        element (s, f) at byte (f/8)*(R*16) + s*16 + (f%8)*2
//     as K-major  A (M = sample,  K = feature): LBO = R*16 (next 8 features), SBO = 128 (next 8 samples)
//     as MN-major A/B (MN = feature, K = sample): SBO = R*16 (next 8 features), LBO = 128 (next 8 samples)
//   WEIGHT PACK  W[N x K] (nn.Linear weight, N = out, K = in), N multiple of 8, K multiple of 8:
//        element (n, k) at byte (k/8)*(N*16) + n*16 + (k%8)*2
//     as K-major  B (N = out, K = in):  LBO = N*16, SBO = 128
//     as MN-major B (N' = in, K' = out) for data-grad:  SBO = N*16, LBO = 128
// Accumulators: a warpgroup (128 threads) owns D[64 x N] fp32 in registers; register i of thread t (warp w = t/32, lane l) holds
//   row 16w + l/4 + 8*((i>>1)&1), column 8*(i>>2) + 2*(l%4) + (i&1)  (tc_frag_row / tc_frag_col).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

__device__ __forceinline__ uint32_t tc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- shared-memory matrix descriptor (wgmma, layout INTERLEAVE = no swizzle) ------------------------------------
__device__ __forceinline__ uint64_t tc_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);            // start address  [0,14)
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;       // leading byte offset [16,30)
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;       // stride byte offset  [32,46)
    return d;                                                // base_offset 0, layout type 0 (no swizzle)
}
// advance a descriptor's start address by `bytes` (multiple of 16; the 14-bit address field must not wrap: smem < 256 KB)
__device__ __forceinline__ uint64_t tc_desc_adv(uint64_t d, uint32_t bytes) { return d + (uint64_t)(bytes >> 4); }

// ---- warpgroup MMA: D[64 x N] (+)= A[64 x 16] . B[16 x N], fp16 x fp16 -> fp32, both operands from shared memory -----
// TA / TB: 0 = K-major, 1 = MN-major (transposed) operand.  Warpgroup-collective (.sync.aligned): all 128 threads issue it.
template <int N, int TA, int TB> struct WgMma;
template <int TA, int TB> struct WgMma<8, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[4], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<16, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<32, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<48, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[24], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, %28;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<64, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<80, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[40], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, %43, %44;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<96, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[48], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, %51, %52;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<112, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[56], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %58, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, %59, %60;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct WgMma<128, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc)
    {
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
    }
};

__device__ __forceinline__ void tc_wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keep the accumulator registers live across the asynchronous MMAs (the compiler must not move reads above the wait)
template <int NR> __device__ __forceinline__ void tc_wg_hold(float (&d)[NR])
{
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}
// fragment coordinates of accumulator register i (see the header comment); `wl` = threadIdx.x % 128
__device__ __forceinline__ int tc_frag_row(int wl, int i) { return ((wl >> 5) << 4) + ((wl & 31) >> 2) + ((i & 2) << 2); }
__device__ __forceinline__ int tc_frag_col(int wl, int i) { return ((i >> 2) << 3) + ((wl & 3) << 1) + (i & 1); }

// generic-proxy shared-memory writes -> visible to the async proxy (tensor core operand fetch)
__device__ __forceinline__ void tc_fence_smem_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// named barrier over `nthreads` threads (sub-tile groups of a CTA synchronise independently of each other)
__device__ __forceinline__ void tc_group_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

// ---- mbarrier ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tc_mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(tc_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void tc_mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void tc_mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(tc_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tc_mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t done = 0;
    while (!done) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(tc_smem_u32(bar)), "r"(parity) : "memory");
    }
}
// TMA bulk copy global -> shared (bytes multiple of 16, both addresses 16-byte aligned)
__device__ __forceinline__ void tc_bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(tc_smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(tc_smem_u32(bar)) : "memory");
}

// ---- fp16 packing ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t tc_pack2(float a, float b)
{
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// {relu(lo), relu(hi)} -> packed fp16x2 in ONE instruction (F2FP.RELU): the whole hidden-layer activation
__device__ __forceinline__ uint32_t tc_pack2_relu(float lo, float hi)
{
    uint32_t d;
    asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
