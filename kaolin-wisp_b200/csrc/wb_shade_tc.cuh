// wb_shade_tc.cuh -- the tensor-core (precision 1) shade stage of wb_shade_tc.cu, as the C-ABI entries of wb_shade.cu call it.
#pragma once
#include "wb_common.cuh"

int wb_tc_supported(const wb_nef_desc* nef, int backward);
int wb_tc_blob_floats(const wb_nef_desc* nef);
int wb_tc_pack(const wb_nef_desc* nef, float* blob, cudaStream_t st);
int64_t wb_tc_workspace_bytes(const wb_nef_desc* nef, int64_t R, int64_t S, int backward);
int64_t wb_tc_feat_bytes(const wb_nef_desc* nef, int64_t S);
int wb_tc_shade_fwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                    int64_t S, float* shaded, void* feat_save, void* workspace, cudaStream_t st);
// ray_rows_ready: the workspace already holds the per-ray colour-input rows (the forward's, same rays)
int wb_tc_shade_bwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                    int64_t S, const float* g_shaded, const float* scale, const void* feat_saved, void* workspace, bool ray_rows_ready,
                    float* grad_table, float* grad_dens, float* grad_col, cudaStream_t st);
// The two stages of wb_tc_shade_bwd on the samples [s_begin, s_end) of S (s_begin a multiple of 64).  grad_table != NULL asks for the
// table scatter to be fused into the decoder backward; *fused_out reports whether it was (F == 2 'cat' hash grids whose last pass runs
// two groups per CTA) -- otherwise the caller runs wb_tc_table_scatter afterwards.
int wb_tc_decoder_bwd_ex(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                         int64_t S, int64_t s_begin, int64_t s_end, const float* g_shaded, const float* scale, const void* feat_saved,
                         void* workspace, bool ray_rows_ready, float* grad_dens, float* grad_col, float* grad_table, int* fused_out,
                         cudaStream_t st);
int wb_tc_table_scatter(const wb_nef_desc* nef, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray, int64_t S,
                        int64_t s_begin, int64_t s_end, const float* scale, void* workspace, float* grad_table, cudaStream_t st);
