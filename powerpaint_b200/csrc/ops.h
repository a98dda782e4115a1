// Internal host-side op interface: each op is "prepared" once from its C-ABI descriptor
// (validation, tile selection, TMA tensor-map encoding) into a launch record, and the
// record is launched any number of times. pp_program stores launch records.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/powerpaint_b200.h"

namespace pp {

// ---------------------------------------------------------------- GEMM / conv
struct GemmKParams {
    CUtensorMap tmA[4];  // matrix/conv: [src0, src1]; stride-2 conv: 4 parity maps
    CUtensorMap tmB;
    CUtensorMap tmOut[2];  // output tile store (modes 0 / 2): 64-column boxes, and the 32-column remainder box
    CUtensorMap tmOutT[2];  // mode 5: transposed tile store, boxes of 128 rows (tokens) x 64 / 32 channels
    CUtensorMap tmRes[2];   // modes 0 / 3 with res1: tmOut's boxes over res1 (pitch ldr1), loaded into the staging tile
    int32_t trans_first_tile;  // mode 5: n-tiles from here on are stored transposed (into out_t)
    int32_t a_mode;
    int32_t M, N;            // GEMM extents (conv: M = nb*ho*wo)
    int32_t num_k_iters;     // total 64-wide K chunks
    int32_t chunks0, chunks1;  // per tap: chunks of src0 then src1
    // conv tiling
    int32_t nb, ho, wo;
    int32_t bw, bh, bn;      // conv pixel box (powers of two, bw * bh * bn == 128)
    int32_t bw_log2, bh_log2;
    int32_t tiles_x, tiles_y;
    int32_t m_tiles, n_tiles;  // persistent tile walk: tile = m_tile * n_tiles + n_tile
    uint32_t a_bytes;  // bytes one A stage receives (box volume * 128)
    // epilogue
    int32_t epilogue, act, out_fp32;
    const float* bias;
    const float* rowvec;
    int32_t rows_per_group;
    int64_t rowvec_ld;
    const __nv_bfloat16* res1;
    int64_t ldr1;
    const __nv_bfloat16* res2;
    int64_t ldr2;
    float alpha;
    const float* alpha_dev;     // optional device multiplier: alpha *= alpha_dev[*alpha_step * alpha_stride]
    const int32_t* alpha_step;  // (NULL: index 0) — per-step side-net scale without re-recording the program
    int32_t alpha_stride;
    void* out;
    int64_t ldc;
    int32_t t_rows;
    int64_t t_ld;
    int32_t t_fp16;
    // per-channel partial sums of the stored tile for the consumer's GroupNorm (mode 0 only):
    // chan_stats[(m_tile * stat_segs + seg)][N][2] = {sum, sum of squares} over the valid rows of the segment
    float* chan_stats;
    int32_t stat_segs;           // samples per m-tile (1, 2 or 4 ...)
    int32_t stat_seg_rows_log2;  // rows of one sample inside the tile
    // LayerNorm fold (see pp_gemm_desc): records emitted per row and half n-tile / consumed by the epilogue
    // split-K x2 (see pp_gemm_desc): 1 or 2
    int32_t ksplit;
    float* splitk_ws;
    int32_t* splitk_flags;
    float4* row_stats;
    int64_t row_stats_ld;
    float2* row_final;     // {rstd, -rstd * mean} per row, written by the CTA finishing a row block's last n-tile
    int32_t* row_ticket;   // per m-tile arrival counter (self-resetting)
    const float2* ln_stats;  // consumer: a producer's row_final
    const float* ln_u;
    float ln_eps;
};

struct GemmLaunch {
    GemmKParams p;
    int block_n;
    int mode;  // epilogue flavour: 0 fast bf16, 1 generic, 2 GEGLU, 3 fast bf16 + LayerNorm records out, 4 fast bf16 + LayerNorm of A,
               // 5 row-major then transposed columns through the staging tile (optional LayerNorm of A)
    dim3 grid;
    size_t smem;
};

int gemm_prepare(const pp_gemm_desc& d, GemmLaunch* out);
int gemm_launch(const GemmLaunch& l, cudaStream_t s);

// ---------------------------------------------------------------- attention
struct AttnKParams {
    CUtensorMap tmQ, tmK, tmV;
    int32_t batch, heads, d, nq, nk;
    int32_t dv;        // N of the PV product: d rounded up to an instantiated width (>= ceil16(d))
    float scale_log2;  // scale * log2(e)
    int32_t vt_fp16;   // V^T (and P) in fp16 instead of bf16
    __nv_bfloat16* out;
    int64_t o_ld;
};
struct AttnLaunch {
    AttnKParams p;
    dim3 grid;
    size_t smem;
    int variant;  // 2 * (index of dv among the instantiated widths) + vt_fp16
};
int attn_prepare(const pp_attn_desc& d, AttnLaunch* out);
int attn_launch(const AttnLaunch& l, cudaStream_t s);

// ---------------------------------------------------------------- simple ops
int gemm_stats_geometry(const pp_gemm_desc& d, pp_stats_geom* out);
int gemm_row_stats_records(const pp_gemm_desc& d);
int gemm_variant(const pp_gemm_desc& d, int* block_n, int* mode, int* ksplit);
int group_norm_launch(const pp_gn_desc& d, cudaStream_t s);
int group_norm_validate(const pp_gn_desc& d);
int64_t group_norm_scratch_bytes(int batch, int hw, int channels, int groups);
int layer_norm_launch(const void* x, void* y, const float* gamma, const float* beta, int rows,
                      int c, float eps, cudaStream_t s);
int upsample_nearest_launch(const void* x, void* y, int nb, int h, int w, int c, int ho, int wo, cudaStream_t s);
int add_launch(const void* a, const void* b, void* y, int64_t n, cudaStream_t s);
int time_embed_launch(const float* timesteps, const int32_t* step_idx, void* out, int batch,
                      int dim, cudaStream_t s);
int nchw_to_nhwc_launch(const float* x, void* y, int nb, int c, int hw, int c_pad, cudaStream_t s);
int nhwc_to_nchw_launch(const void* x, int x_is_fp32, float* y, int nb, int c, int hw, int c_ld,
                        cudaStream_t s);
int softmax_rows_launch(const float* s, void* p, int64_t rows, int cols, int64_t ld_s, int64_t ld_p, cudaStream_t st);
int image_preprocess_launch(const uint8_t* img, const void* mask, int mask_mode, void* out, int nb, int hw, int c_pad,
                            float divisor, float shift, cudaStream_t s);
int image_postprocess_launch(const void* x, int x_fp32, int c_ld, uint8_t* out_u8, float* out_f32, int nb, int hw,
                             cudaStream_t s);
int window_copy_validate(const void* src, void* dst, int elem_bytes, int channels, int64_t src_pix, int64_t dst_pix,
                         const pp_window* windows, int count, int max_pixels);
int window_copy_launch(const void* src, void* dst, int elem_bytes, int channels, int64_t src_pix, int64_t dst_pix,
                       const pp_window* windows, int count, int max_pixels, cudaStream_t s);
int tile_blend_validate(const pp_tile_blend_desc& d);
int tile_blend_launch(const pp_tile_blend_desc& d, cudaStream_t s);
int embed_gather_launch(const int32_t* idx, const float* base, const float* ext, const float* pos, void* out, int rows,
                        int vocab, int seq, int dim, cudaStream_t s);
int causal_attention_small_launch(const void* qkv, void* out, int batch, int seq, int heads, int d, float scale,
                                  cudaStream_t s);
int cfg_ddim_validate(const pp_cfg_ddim_desc& d);
int cfg_ddim_launch(const pp_cfg_ddim_desc& d, cudaStream_t s);
int unipc_validate(const pp_unipc_desc& d);
int unipc_launch(const pp_unipc_desc& d, cudaStream_t s);
int solver_validate(const pp_solver_desc& d);
int solver_launch(const pp_solver_desc& d, cudaStream_t s);
int plms_validate(const pp_plms_desc& d);
int plms_launch(const pp_plms_desc& d, cudaStream_t s);
int pool_broadcast_validate(const pp_pool_broadcast_desc& d);
int pool_broadcast_launch(const pp_pool_broadcast_desc& d, cudaStream_t s);

}  // namespace pp
