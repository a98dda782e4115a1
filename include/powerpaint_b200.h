/*
 * powerpaint_b200.h — C ABI of the H100-native (sm_90a) PowerPaint denoising hot path.
 *
 * The reference (open-mmlab/PowerPaint) is pure Python over diffusers; it has no FFI of
 * its own. The boundary a maintainer binds is therefore the set of *operators* its
 * per-step hot path executes, each entry point citing the reference call site it
 * replaces (paths relative to the reference checkout):
 *
 *   pp_gemm_conv      nn.Conv2d 3x3 / 1x1 and nn.Linear inside ResnetBlock2D,
 *                     Transformer2DModel, Downsample2D, Upsample2D, conv_in/conv_out,
 *                     BrushNet zero-convs  (powerpaint/models/unet_2d_blocks.py:789,807,
 *                     1274,1289,1319,1428,2499,2514,2542,2672,2689;
 *                     unet_2d_condition.py:256,477; BrushNet_CA.py:223-228,330-376,446-454)
 *                     with bias / time-embedding broadcast / skip add / BrushNet add /
 *                     output scale / GEGLU fused into the epilogue
 *                     (unet_2d_condition.py:1223,1300; unet_2d_blocks.py:1388-1398,2627-2638)
 *   pp_attention      Attention + AttnProcessor2_0 -> F.scaled_dot_product_attention
 *                     (processors referenced at unet_2d_condition.py:24-31)
 *   pp_group_norm     nn.GroupNorm(32)+SiLU in ResnetBlock2D / Transformer2DModel.norm /
 *                     conv_norm_out (unet_2d_condition.py:466,1351-1353), also performs the
 *                     up-path torch.cat (unet_2d_blocks.py:2589,2732) while normalising
 *   pp_layer_norm     nn.LayerNorm x3 per BasicTransformerBlock
 *   pp_upsample2x     Upsample2D's F.interpolate(scale_factor=2, mode="nearest")
 *   pp_time_embed     Timesteps(320, flip_sin_to_cos=True, shift=0)
 *                     (unet_2d_condition.py:914-938)
 *   pp_cfg_ddim_step  CFG combine + DDIMScheduler.step + next-step input build
 *                     (pipelines/pipeline_PowerPaint.py:990-996,1018-1023;
 *                      pipeline_PowerPaint_Brushnet_CA.py:1390,1444-1449)
 *   pp_unipc_step     CFG combine + UniPCMultistepScheduler.step (the v2 app's scheduler, app.py:197)
 *   pp_solver_step    CFG combine + DPMSolverMultistepScheduler / EulerDiscreteScheduler /
 *                     EulerAncestralDiscreteScheduler.step (the scheduler a user swaps in, as app.py:197 does)
 *   pp_plms_step      CFG combine + PNDMScheduler.step with skip_prk_steps (the scheduler stored by the v1
 *                     checkpoint, app.py:91-93) + 4-channel blend
 *   pp_pool_broadcast spatial mean of a side-net residual, broadcast to full size (global_pool_conditions,
 *                     BrushNet_CA.py:936-943), added onto an optional running Multi-ControlNet sum
 *   pp_upsample_nearest  Upsample2D with an explicit output size (unet_2d_condition.py:1120-1126,1311-1312)
 *                     Also carries: LayerNorm of BasicTransformerBlock folded into the producing / consuming
 *                     GEMMs (row_stats / ln_stats; diffusers LayerNorm norm1/2/3, SURVEY.md App. A.3), and
 *                     to_q | to_k | to_v^T of a self-attention as one launch (PP_EPI_ROWS_THEN_TRANSPOSED).
 *   pp_gemm_stats_geometry  host-only: layout of the GroupNorm partial sums a GEMM / conv emits from its
 *                     epilogue (pp_gemm_desc.chan_stats -> pp_gn_desc.part0 / part1)
 *   pp_gemm_row_stats_records, pp_gemm_splitk_bytes  host-only: scratch sizes of the LayerNorm-statistics
 *                     producer and of the optional split-K workspace
 *   pp_softmax_rows, pp_image_preprocess_u8, pp_image_postprocess   VAE attention softmax and the uint8
 *                     pre/post-processing either side of vae.encode / vae.decode
 *                     (pipeline_PowerPaint.py:39-153,657-669,1051,1062)
 *   pp_resample_u8, pp_box_blur_u8, pp_canny_u8, pp_outpaint_canvas_u8, pp_app_blend_u8   the app's request
 *                     pre / post-processing (Pillow resize and GaussianBlur, cv2.Canny, canvas and blends;
 *                     app.py:258-387,405-473); pp_gaussian_box_radius, pp_canny_workspace_bytes host-only
 *   pp_window_copy, pp_tile_blend   tiled VAE encode / decode (diffusers AutoencoderKL.enable_tiling,
 *                     pipeline_PowerPaint_ControlNet.py:341-356): tile gather / assembly and the seam blend
 *   pp_embed_gather, pp_causal_attention_small   CLIP text encoder: embeddings with the task-prompt splice
 *                     (utils/utils.py:256-483) and the causal 77-token attention (pipeline_PowerPaint.py:317-518)
 *   pp_program_*      a recorded list of the above, replayed per denoising step (pp_program_run_range: a slice
 *                     of it as plain launches, for bisecting a step op by op)
 *                     (the `for i, t in enumerate(timesteps)` loops,
 *                      pipeline_PowerPaint.py:988-1041, Brushnet_CA.py:1384-1466,
 *                      ControlNet.py:1663-1741)
 *
 * Conventions: all pointers are DEVICE pointers unless named host_*; activations are
 * bf16, channels-last (NHWC == [batch, tokens, channels]); every call enqueues on the
 * given cudaStream_t and never synchronises the host; no allocation happens inside a
 * call; a non-zero return code means nothing was enqueued and pp_last_error() holds the
 * reason. Handles are thread-compatible (one thread per handle at a time).
 */
#ifndef POWERPAINT_B200_H_
#define POWERPAINT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int pp_status; /* 0 = ok, 1 = invalid argument, 2 = CUDA error, 3 = unsupported */
typedef void* pp_stream; /* cudaStream_t */

const char* pp_last_error(void);
/* ABI version of this library (bumped on incompatible struct changes). */
int pp_abi_version(void);
/* 1 if the current device is sm_90 (H100) and the kernels can run on it. */
int pp_device_supported(void);

/* ------------------------------------------------------------------ GEMM / conv */
enum {
    PP_A_MATRIX = 0,    /* A is [M, K] row-major (a Linear or 1x1 conv over tokens) */
    PP_A_CONV3X3 = 1,   /* implicit GEMM, 3x3 stride 1 pad 1 over NHWC [nb, h, w, c] */
    PP_A_CONV3X3_S2 = 2,  /* implicit GEMM, 3x3 stride 2 pad 1 (Downsample2D); output ceil(h/2) x ceil(w/2) */
    PP_A_CONV3X3_S2P0 = 3 /* 3x3 stride 2 over F.pad(x, (0,1,0,1)) (the VAE encoder's Downsample2D(padding=0));
                             output floor(h/2) x floor(w/2) */
};
enum {
    PP_EPI_PLAIN = 0,
    PP_EPI_GEGLU = 1,      /* out[:, j] = (acc_a + bias_a) * gelu(acc_g + bias_g); weights tile-interleaved */
    PP_EPI_TRANSPOSED = 2, /* out[(m / t_rows) * N + n][m % t_rows], row pitch t_ld (V^T for attention) */
    PP_EPI_ROWS_THEN_TRANSPOSED = 3 /* columns [0, trans_from_col) row-major into `out` (pitch ldc), columns
                               [trans_from_col, N) transposed into `out_t` like PP_EPI_TRANSPOSED with
                               N - trans_from_col channels: to_q | to_k | to_v^T of one attention in ONE launch */
};
enum { PP_ACT_NONE = 0, PP_ACT_SILU = 1, PP_ACT_QUICK_GELU = 2 /* x * sigmoid(1.702 x): CLIP text encoder MLP */ };

/* Geometry of the per-channel GroupNorm partial sums a GEMM / conv can emit from its epilogue
   (pp_gemm_desc.chan_stats) and pp_group_norm consumes (pp_gn_desc.part0 / part1): one record
   {sum of (x - shift), sum of (x - shift)^2, shift, 0} per (m-tile, sample segment of the tile, output channel),
   fp32, laid out [m_tiles][segs][N][4]; shift = the segment's first row, so the variance does not cancel for a
   large mean over a small spread. Filled by pp_gemm_stats_geometry(). */
typedef struct pp_stats_geom {
    int32_t supported;   /* 0: this GEMM cannot emit statistics (the consumer runs its own statistics pass) */
    int32_t channels;    /* N */
    int32_t segs;        /* samples per m-tile */
    int32_t seg_rows;    /* rows of one sample inside an m-tile */
    int32_t tiles_per_group; /* m-tiles that cover one group of `segs` samples */
    int32_t tiles_x, tiles_y, bw, bh, wo, ho; /* pixel-tile geometry (matrix mode: a 1-D strip) */
    int64_t bytes;       /* size of the partials buffer */
} pp_stats_geom;

typedef struct pp_gemm_desc {
    int32_t a_mode;
    int32_t epilogue;
    /* A operand: up to two sources concatenated along K / channels (skip-concat without torch.cat) */
    const void* a0;
    const void* a1;      /* may be NULL */
    int32_t c0, c1;      /* channels (K per tap) of each source; c1 = 0 if a1 is NULL */
    int64_t lda0, lda1;  /* PP_A_MATRIX: row pitch in elements; conv modes: ignored (tight NHWC) */
    int32_t nb, h, w;    /* conv modes: INPUT batch / height / width */
    int32_t M;           /* PP_A_MATRIX: rows. conv modes: ignored (= nb*ho*wo) */
    int32_t N;           /* GEMM N (for GEGLU: 2x the output width) */
    /* B operand: weights [N, Kw] bf16 row-major, Kw = taps * (pad64(c0) + pad64(c1)) when
       taps == 9 or a1 != NULL, else row pitch ldb >= c0 */
    const void* b;
    int64_t ldb;
    /* epilogue: v = acc + bias[n] + rowvec[m / rows_per_group][n] + res1[m][n];
                 v = v * alpha + res2[m][n]; v = act(v) */
    const float* bias;
    const float* rowvec;
    int32_t rows_per_group;
    int64_t rowvec_ld; /* row pitch of rowvec in elements; 0 = N */
    const void* res1; /* bf16 */
    int64_t ldr1;
    const void* res2; /* bf16 */
    int64_t ldr2;
    float alpha;
    int32_t act;
    void* out;
    int64_t ldc;
    int32_t out_fp32; /* 0: bf16 output, 1: fp32 output */
    int32_t t_rows;   /* PP_EPI_TRANSPOSED */
    int64_t t_ld;
    int32_t block_n;  /* 0 = auto, else one of 64/128/160/256 */
    int32_t t_fp16;   /* PP_EPI_TRANSPOSED: store fp16 instead of bf16 (V^T for pp_attention) */
    /* alpha is multiplied by alpha_dev[(alpha_step ? *alpha_step : 0) * alpha_stride] when alpha_dev != NULL:
       the BrushNet / ControlNet conditioning scale x per-step keep flag lives in a device table, so one
       recorded program serves every scale (Brushnet_CA.py:1369-1376,1403-1409; ControlNet.py:1652-1658) */
    const float* alpha_dev;
    const int32_t* alpha_step;
    int32_t alpha_stride;
    /* optional GroupNorm partial sums of the stored output (bf16 row-major outputs only), see pp_stats_geom;
       rows_per_group must hold the rows per sample in PP_A_MATRIX mode */
    float* chan_stats;
    /* LayerNorm folded into the GEMMs either side of it (BasicTransformerBlock norm1/2/3, SURVEY.md App. A.3):
       PRODUCER (PP_A_MATRIX, bf16 row-major output): row_stats != NULL makes the epilogue emit, per output row and
       per half n-tile, one record {sum of (x - shift), sum of (x - shift)^2, shift, count} (fp32 x 4) of the values
       it computes, laid out [records][row_stats_ld] with records = pp_gemm_row_stats_records(desc) — scratch of this
       launch. The CTA that finishes the LAST n-tile of a 128-row block (row_ticket[m-tile], zero-initialised int32,
       left at zero again) folds the records of its rows (Chan's combination) into
         row_final[m] = {rstd, -rstd * mean}   (fp32 x 2, eps = ln_eps).
       CONSUMER: ln_stats != NULL (a producer's row_final) applies LayerNorm(A) algebraically in the epilogue. With
       W' = W * gamma (folded into b on the host), ln_u[n] = sum_k W'[n, k] and bias[n] = sum_k W[n, k] beta[k]
       (+ the layer's own bias):  acc' = rstd[m] * acc - rstd[m] mean[m] * ln_u[n];  everything after (bias, GEGLU
       gate, transposed store ...) is unchanged. */
    float* row_stats;
    int64_t row_stats_ld;
    float* row_final;
    int32_t* row_ticket;
    const float* ln_stats;
    const float* ln_u;
    float ln_eps;
    /* PP_EPI_ROWS_THEN_TRANSPOSED: transposed destination and the first transposed column (a multiple of the tile
       width: pass block_n explicitly). t_rows must be a multiple of 128 and divide M. */
    void* out_t;
    int32_t trans_from_col;
    /* optional split-K x2 for long-K launches whose tiles fill at most half of the GPU (8x8-resolution layers): fp32
       workspace of pp_gemm_splitk_bytes(desc) bytes and the same number of tiles of zero-initialised int32 flags (the
       kernel leaves them at zero). NULL: never split. Results are deterministic (owner + donor, fixed order). */
    float* splitk_ws;
    int32_t* splitk_flags;
} pp_gemm_desc;

pp_status pp_gemm_conv(const pp_gemm_desc* d, pp_stream stream);
/* host-only query: can this GEMM emit GroupNorm partial sums, and with which layout */
pp_status pp_gemm_stats_geometry(const pp_gemm_desc* d, pp_stats_geom* out);
/* host-only query: bytes of split-K workspace this launch could use (0: it would not split); flags: one int32 per
   (m-tile, n-tile), i.e. bytes / (128 * block_n * 4) of them — pass `*tiles_out` to size the flag array */
int64_t pp_gemm_splitk_bytes(const pp_gemm_desc* d, int32_t* tiles_out);
/* host-only query: number of per-row LayerNorm records this GEMM emits through row_stats (0: it cannot emit them) */
int32_t pp_gemm_row_stats_records(const pp_gemm_desc* d);
/* host-only query: the kernel variant pp_gemm_conv would launch for this descriptor: tile width (64/128/160/256),
   epilogue mode (0 plain bf16, 1 generic, 2 GEGLU, 3 LayerNorm-statistics producer, 4 LayerNorm-folded consumer,
   5 transposed columns through the staging tile) and split-K factor (1 or 2; 2 runs the mode-0 split-K kernel).
   It validates the shape and the tile width only: the answer is the launch's for a descriptor pp_gemm_conv accepts
   (e.g. row_stats together with ln_stats reports mode 3, while pp_gemm_conv refuses that descriptor) */
pp_status pp_gemm_variant(const pp_gemm_desc* d, int32_t* block_n, int32_t* mode, int32_t* ksplit);
/* host-only query: the epilogue terms this launch stages in shared memory during the main loop (modes 0 / 3): res1
   through the output staging tile (*stage_res; the split-K donor half has no epilogue and stages nothing), the row
   vector through the second staging row when every tile lies in one sample (*stage_rv). 1 = staged, 0 = not */
pp_status pp_gemm_staging(const pp_gemm_desc* d, int32_t* stage_res, int32_t* stage_rv);

/* ------------------------------------------------------------------ attention */
typedef struct pp_attn_desc {
    /* q: [batch, nq, heads, d] with token pitch q_ld (elements); k likewise with nk, k_ld.
       vt: V transposed, [batch, heads*d, vt_ld] (keys contiguous, vt_ld >= nk, vt_ld % 8 == 0), bf16 or fp16.
       out: [batch, nq, heads*d] row pitch o_ld. softmax(q k^T * scale) v, no mask. */
    const void* q;
    const void* k;
    const void* vt;
    void* out;
    int32_t batch, heads, d, nq, nk;
    int64_t q_ld, k_ld, vt_ld, o_ld;
    int64_t q_batch_stride, k_batch_stride; /* elements between batches */
    float scale;
    int32_t vt_fp16; /* != 0: vt holds fp16 (P is then computed in fp16 too); 0: bf16 */
} pp_attn_desc;

pp_status pp_attention(const pp_attn_desc* d, pp_stream stream);
/* host-only query: the kernel variant pp_attention would launch: PV width dv (d rounded up to one of
   32/48/64/80/96/128/160/192) and whether P is fp16 (vt_fp16) or bf16 */
pp_status pp_attention_variant(const pp_attn_desc* d, int32_t* dv, int32_t* p_fp16);

/* ------------------------------------------------------------------ norms */
typedef struct pp_gn_desc {
    /* GroupNorm over NHWC x = concat(x0[..., :c0], x1[..., :c1]) -> y [.., c0+c1] bf16 */
    const void* x0;
    const void* x1; /* may be NULL */
    int32_t c0, c1;
    int32_t batch, hw, groups;
    const float* gamma;
    const float* beta;
    float eps;
    int32_t silu;
    float* stats; /* scratch of pp_group_norm_scratch_bytes() bytes, 16-byte aligned: the per-(sample, group)
                     (mean, rstd) [batch, groups, 2] fp32 both statistics paths write, then (standalone path,
                     at the next 16-byte boundary) the ticket counters [batch] uint32 and, again 16-byte
                     aligned, the per-block partials of the deterministic reduction */
    void* y;
    int32_t stats_prezeroed; /* 1: the scratch was zeroed once when it was allocated (every call leaves its
                                ticket counters zero again) or by one memset per step over all scratch;
                                0: the call clears its ticket counters with a memset of its own */
    /* from_partials != 0: the statistics pass is replaced by a small finalize kernel that folds the
       per-tile channel sums the producing GEMMs emitted (part0 for x0, part1 for x1) into
       (mean, rstd) per (sample, group) — Chan's parallel combination in fp64, fixed order. `stats` then
       only needs batch * groups * 2 floats. */
    int32_t from_partials;
    const float* part0;
    const float* part1;
    pp_stats_geom geom0, geom1;
} pp_gn_desc;
pp_status pp_group_norm(const pp_gn_desc* d, pp_stream stream);
/* bytes of `stats` scratch a GroupNorm over [batch, hw, channels] with `groups` groups needs (0: invalid) */
int64_t pp_group_norm_scratch_bytes(int32_t batch, int32_t hw, int32_t channels, int32_t groups);

pp_status pp_layer_norm(const void* x, void* y, const float* gamma, const float* beta,
                        int32_t rows, int32_t c, float eps, pp_stream stream);

/* ------------------------------------------------------------------ small ops */
/* nearest 2x upsample of NHWC bf16 [nb,h,w,c] -> [nb,2h,2w,c] */
pp_status pp_upsample2x(const void* x, void* y, int32_t nb, int32_t h, int32_t w, int32_t c,
                        pp_stream stream);
/* F.interpolate(x, size=(ho, wo), mode="nearest") on NHWC bf16 — Upsample2D with an explicit output size
   (unet_2d_condition.py:1120-1126,1311-1312: latent sizes that are not multiples of 8) */
pp_status pp_upsample_nearest(const void* x, void* y, int32_t nb, int32_t h, int32_t w, int32_t c,
                              int32_t ho, int32_t wo, pp_stream stream);
/* y = a + b (bf16, n elements, n % 8 == 0) — ControlNet skip residuals */
pp_status pp_add(const void* a, const void* b, void* y, int64_t n, pp_stream stream);
/* sinusoidal timestep embedding [batch, dim] bf16: cat(cos, sin) (flip_sin_to_cos=True, shift 0).
   t comes from timesteps[*step_idx] when step_idx != NULL, else timesteps[0..batch). */
pp_status pp_time_embed(const float* timesteps, const int32_t* step_idx, void* out, int32_t batch,
                        int32_t dim, pp_stream stream);
/* NCHW fp32 <-> NHWC bf16 (c padded to c_pad with zeros on the way in) */
pp_status pp_nchw_to_nhwc(const float* x, void* y, int32_t nb, int32_t c, int32_t hw,
                          int32_t c_pad, pp_stream stream);
pp_status pp_nhwc_to_nchw(const void* x, int32_t x_is_fp32, float* y, int32_t nb, int32_t c,
                          int32_t hw, int32_t c_ld, pp_stream stream);

/* ------------------------------------------------------------------ VAE attention / image I/O */
/* p[r, :] = softmax(s[r, :]): fp32 scores in, bf16 probabilities out, cols <= 16384. The VAE mid-block
   attention (one head of 512 channels; pipeline_PowerPaint.py:657-669,:1051 through vae.encode / decode) runs as
   S = Q K^T (pp_gemm_conv, fp32 out, alpha = 1/sqrt(512)) -> pp_softmax_rows -> O = P V (pp_gemm_conv). */
pp_status pp_softmax_rows(const float* s, void* p, int64_t rows, int32_t cols, int64_t ld_s, int64_t ld_p,
                          pp_stream stream);
/* uint8 NCHW [nb,3,h,w] (+ mask [nb,1,h,w]: mask_mode 1 = uint8, 2 = fp32, 0 = none) -> bf16 NHWC
   [nb, hw, c_pad]: (px / divisor + shift) * (mask < 0.5), channels >= 3 zero — `prepare_mask_and_masked_image`
   (pipeline_PowerPaint.py:39-153) on the device */
pp_status pp_image_preprocess_u8(const uint8_t* image, const void* mask, int32_t mask_mode, void* out, int32_t nb,
                                 int32_t hw, int32_t c_pad, float divisor, float shift, pp_stream stream);
/* decoded image NHWC (channels 0..2 of c_ld) -> clamp(x/2 + 0.5, 0, 1) as uint8 NHWC [nb,hw,3] (x255, rounded)
   and / or fp32 NCHW [nb,3,hw] — `VaeImageProcessor.postprocess` (pipeline_PowerPaint.py:1062) */
pp_status pp_image_postprocess(const void* x, int32_t x_is_fp32, int32_t c_ld, uint8_t* out_u8, float* out_f32,
                               int32_t nb, int32_t hw, pp_stream stream);

/* ------------------------------------------------------------------ the app's request pre / post-processing */
/* All images are uint8 HWC with 1 or 3 channels; each result equals the library named, byte for byte
   (ref:app.py:258-387,405-473). */
/* Pillow Image.resize (modes L / RGB): a horizontal pass when out_w != in_w, then a vertical one when
   out_h != in_h (a copy when neither). The host builds each axis's tables as Pillow does: bounds [out * 2] =
   (first source pixel, tap count), k [out * taps] = weights in 22-bit fixed point. A two-pass resize writes its
   horizontal result to tmp [in_h, out_w, channels]. */
pp_status pp_resample_u8(const uint8_t* src, uint8_t* tmp, uint8_t* dst, int32_t in_h, int32_t in_w, int32_t out_h,
                         int32_t out_w, int32_t channels, const int32_t* bounds_x, const int32_t* k_x, int32_t taps_x,
                         const int32_t* bounds_y, const int32_t* k_y, int32_t taps_y, pp_stream stream);
/* host-only: the extended box radius Pillow's GaussianBlur(radius) runs `passes` passes of per axis */
float pp_gaussian_box_radius(float radius, int32_t passes);
/* Pillow's extended box blur: `passes` horizontal then `passes` vertical passes, edges replicated; tmp is an
   image-sized scratch buffer distinct from src and dst. GaussianBlur(r) = pp_box_blur_u8 with
   pp_gaussian_box_radius(r, 3) and 3 passes. */
pp_status pp_box_blur_u8(const uint8_t* src, uint8_t* tmp, uint8_t* dst, int32_t h, int32_t w, int32_t channels,
                         float box_radius, int32_t passes, pp_stream stream);
/* host-only: workspace bytes pp_canny_u8 needs for an h x w image (-1 for a zero size) */
int64_t pp_canny_workspace_bytes(int32_t h, int32_t w);
/* cv2.Canny(src, low, high) with aperture 3 and the L1 norm -> dst [h, w] in {0, 255}. Five launches: Sobel,
   suppression + tile-local union-find, tile merge, root marking, output; no host synchronisation. */
pp_status pp_canny_u8(const uint8_t* src, uint8_t* dst, void* workspace, int64_t workspace_bytes, int32_t h, int32_t w,
                      int32_t channels, double low, double high, pp_stream stream);
/* The outpainting canvas: img = 127 with src [o_h, o_w, 3] at (top, left); mask = 255 except 0 in rows
   [hole_y0, hole_y1) x columns [hole_x0, hole_x1) (an empty range leaves it all 255). Both RGB [c_h, c_w, 3]. */
pp_status pp_outpaint_canvas_u8(const uint8_t* src, int32_t o_h, int32_t o_w, uint8_t* img, uint8_t* mask,
                                int32_t c_h, int32_t c_w, int32_t top, int32_t left, int32_t hole_y0, int32_t hole_y1,
                                int32_t hole_x0, int32_t hole_x1, pp_stream stream);
/* Per-pixel steps over RGB a [h, w, 3] and a mask b [h, w, b_channels] (1 or 3), float64 in NumPy's operation order,
   truncated to uint8:
     PP_BLEND_LUMA         out [h, w, 1] = Pillow's RGB -> L of a (b, c unused)
     PP_BLEND_HOLE_FILL    out = a * (1 - b / 255.0)                                  (the v2 hole fill)
     PP_BLEND_RED_OVERLAY  out = a * (1 - b / 512.0) + b / 512.0 * (180, 0, 0)
     PP_BLEND_PASTE        out = (a / 255.0 * (b / 255.0) + (1 - b / 255.0) * (c / 255.0)) * 255, c RGB */
enum { PP_BLEND_LUMA = 0, PP_BLEND_HOLE_FILL = 1, PP_BLEND_RED_OVERLAY = 2, PP_BLEND_PASTE = 3 };
pp_status pp_app_blend_u8(int32_t op, const uint8_t* a, const uint8_t* b, const uint8_t* c, uint8_t* out, int32_t h,
                          int32_t w, int32_t b_channels, pp_stream stream);

/* ------------------------------------------------------------------ tiled VAE (diffusers enable_tiling) */
/* One rectangular window of pixels: `rows` x `cols` pixels starting at element offset src_off of the source and
   dst_off of the destination, consecutive rows src_row / dst_row elements apart. */
typedef struct pp_window {
    int64_t src_off, dst_off;
    int64_t src_row, dst_row;
    int32_t rows, cols;
} pp_window;
/* Copies `count` windows (a DEVICE array) of `channels` elements per pixel from src to dst, pixels src_pix / dst_pix
   elements apart; elem_bytes 2 (bf16) or 4 (fp32). max_pixels >= rows * cols of every window sizes the grid.
   Windows must not overlap in dst. The tiled VAE gathers its tiles out of the canvas with it and assembles the
   cropped tiles into the output. */
pp_status pp_window_copy(const void* src, void* dst, int32_t elem_bytes, int32_t channels, int64_t src_pix,
                         int64_t dst_pix, const pp_window* windows, int32_t count, int32_t max_pixels, pp_stream stream);
/* In-place blend of one tile b of an fp32 NHWC tile store (`channels` floats per pixel) with the tile above (av)
   and the tile to its left (ah), for `batch` samples; diffusers AutoencoderKL.blend_v then blend_h:
     for y < e_v: b[y, :] = av[av_h - e_v + y, :] * (1 - y/e_v) + b[y, :] * (y/e_v)
     for x < e_h: b[:, x] = ah[:, ah_w - e_h + x] * (1 - x/e_h) + b[:, x] * (x/e_h)
   Each weight is the double expression rounded to fp32, each product and the sum are rounded separately (no FMA):
   bit-identical to the torch loop. av has b_w columns and ah has b_h rows; e_v = 0 / e_h = 0 skips a direction
   (its pointer may then be NULL). Sample s of a tile starts s * *_stride floats after its pointer. */
typedef struct pp_tile_blend_desc {
    float* b;
    const float* av;
    const float* ah;
    int64_t b_stride, av_stride, ah_stride;
    int32_t batch, channels;
    int32_t b_h, b_w;
    int32_t av_h, ah_w;
    int32_t e_v, e_h;
} pp_tile_blend_desc;
pp_status pp_tile_blend(const pp_tile_blend_desc* d, pp_stream stream);

/* ------------------------------------------------------------------ text encoder */
/* out[r] = (idx[r] < vocab ? base[idx[r]] : ext[idx[r] - vocab]) + pos[r % seq]  (bf16 [rows, dim]; fp32 tables).
   CLIP token + position embedding with the EmbeddingLayerWithFixes task-prompt splice (utils.py:256-483) resolved
   by the host into one gather index per position. */
pp_status pp_embed_gather(const int32_t* idx, const float* base, const float* ext, const float* pos, void* out,
                          int32_t rows, int32_t vocab, int32_t seq, int32_t dim, pp_stream stream);
/* causal softmax(q k^T * scale) v over seq <= 128 tokens; qkv [batch*seq, 3*heads*d] bf16 (q | k | v),
   out [batch*seq, heads*d] — the CLIP text transformer's self-attention (pipeline_PowerPaint.py:317-518) */
pp_status pp_causal_attention_small(const void* qkv, void* out, int32_t batch, int32_t seq, int32_t heads, int32_t d,
                                    float scale, pp_stream stream);

/* ------------------------------------------------------------------ device-drawn step noise */
/* One draw of torch's CUDA randn: the noise a stochastic step adds is, element for element,
   `torch.randn(shape, generator=g, device="cuda", dtype=torch.float32)` of a draw of N = rows * 4 * hw elements
   (NCHW [rows, 4, h, w]), computed by the step kernel where it uses it. torch's launch policy fixes every element:
     threads = 256 * min(ceil(N / 256), SMs * (maxThreadsPerSM / 256)),   q = li / threads
     element li = lane q % 4 of the (q / 4)-th curand_normal4 of curand_init(seed, li % threads, offset)
   and each draw advances the generator by offset_per_step = ((N - 1) / (threads * 4) + 1) * 4.
   The draw of step s uses offset = offset0 + s * offset_per_step (s = *step_idx of the step descriptor), so a
   replayed CUDA graph needs nothing from the host. Latent row b in [first_row, first_row + rows), pixel p and
   channel c of the NHWC step tensors take element li = ((b - first_row) * 4 + c) * hw + p. The host reserves the
   generator's stream (advances its offset past the loop's draws) when it fills the table. */
typedef struct pp_randn_draw {
    uint64_t seed;
    uint64_t offset0;
    uint64_t offset_per_step;
    int64_t threads;      /* 256 * grid of torch's launch for this draw */
    int32_t first_row;    /* latent rows [first_row, first_row + rows) of the step take this draw */
    int32_t rows;         /* 0: the entry matches no row */
} pp_randn_draw;

/* ------------------------------------------------------------------ CFG + DDIM */
typedef struct pp_cfg_ddim_desc {
    /* eps: model output for the 2*batch CFG-duplicated samples (unconditional half first),
       NHWC [2*batch, hw, eps_ld] (fp32 or bf16), channels 0..3 used.
       latents: fp32 NHWC [batch, hw, 4], updated in place (x_t -> x_{t-1}).
       coef: [n_steps, 8] fp32 rows {sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-sigma^2),
             sigma, 0, 0, 0}; row *step_idx is used, then *step_idx is incremented when
             advance_step != 0 (so a captured CUDA graph can be replayed once per step).
       noise: optional fp32 NHWC [batch, hw, 4] variance noise (eta > 0).
       next_in: optional bf16 NHWC [n_copies*batch, hw, next_c]: channels 0..3 = x_{t-1},
             channels 4..4+extra_c = extra[b] (mask + masked-image latents, fp32 NHWC
             [batch, hw, extra_c]), rest zero; written for both CFG halves. */
    const void* eps;
    int32_t eps_fp32;
    int32_t eps_ld;
    float* latents;
    const float* coef;
    int32_t* step_idx;
    int32_t advance_step;
    const float* noise;
    float guidance_scale;
    int32_t do_cfg; /* 0: eps has `batch` samples and is used as is */
    int32_t batch, hw;
    void* next_in;
    int32_t next_c, n_copies;
    const float* extra;
    int32_t extra_c;
    int32_t guidance_from_coef; /* != 0: guidance scale = coef[row][5] (graph-replay friendly) */
    int32_t extra_per_copy;     /* != 0: extra is [n_copies*batch, hw, extra_c] (one set per CFG half) */
    /* 4-channel-UNet blend after the step (pipeline_PowerPaint.py:1025-1035):
         x = (1 - m) * (a * x0 + sqrt(1 - a^2) * noise_b) + m * x,  a = coef[row][7] (sqrt(alpha_bar) of the NEXT
       timestep, 1 for the last step); x0 / m are the FIRST image's latents [hw, 4] / latent mask [hw] (the
       reference indexes `[:1]` and broadcasts over the batch), noise_b [batch, hw, 4]. NULL = no blend. */
    const float* blend_x0;
    const float* blend_mask;
    const float* blend_noise;
    /* device-drawn variance noise (pp_randn_draw): n_draws entries, 8-byte aligned; a row no entry covers gets
       zero noise. Exclusive with `noise`. Nothing is drawn when sigma (coef[row][4]) is exactly 0, so a table whose
       rows all have sigma 0 gives the same bits as draws = NULL. NULL / 0 = none. */
    const pp_randn_draw* draws;
    int32_t n_draws;
} pp_cfg_ddim_desc;
pp_status pp_cfg_ddim_step(const pp_cfg_ddim_desc* d, pp_stream stream);

/* CFG combine + UniPCMultistepScheduler.step (solver_order 2, bh2, predict_x0, epsilon prediction; the v2 app's
   scheduler, app.py:197) + next-step input build. The multistep update is linear in the tensors it touches, so
   the host folds the schedule into per-step scalars (ucoef rows of 12 floats):
     m_t    = u[0] * x + u[1] * eps                                   (x0 prediction, `convert_model_output`)
     x_c    = u[2] != 0 ? u[3] * last + u[4] * m1 + u[5] * m2 + u[6] * m_t : x      (UniC corrector)
     x_next = u[7] * x_c + u[8] * m_t + u[9] * m1                                     (UniP predictor)
     last <- x_c, m2 <- m1, m1 <- m_t, latents <- x_next
   guidance scale = coef[row][5] of the shared 8-float table. State tensors are fp32 NHWC [batch, hw, 4]. */
typedef struct pp_unipc_desc {
    const void* eps;
    int32_t eps_fp32;
    int32_t eps_ld;
    float* latents;
    float* last_sample;
    float* m1;
    float* m2;
    const float* coef;   /* [n_steps, 8], column 5 = guidance scale */
    const float* ucoef;  /* [n_steps, 12] */
    int32_t* step_idx;
    int32_t advance_step;
    int32_t do_cfg;
    int32_t batch, hw;
    void* next_in;       /* bf16 NHWC [n_copies*batch, hw, next_c]: channels 0..3 refreshed */
    int32_t next_c, n_copies;
} pp_unipc_desc;
pp_status pp_unipc_step(const pp_unipc_desc* d, pp_stream stream);

/* CFG combine + one step of DPMSolverMultistepScheduler (dpmsolver++ / sde-dpmsolver++, solver_order 1 or 2),
   EulerDiscreteScheduler or EulerAncestralDiscreteScheduler + next-step input build. Each update is linear in the
   tensors it touches, so the host folds the step into one row of 8 floats (scoef, computed in float64):
     m_t     = r[0] * x + r[1] * eps                                  (x0 prediction)
     x_next  = r[2] * x + r[3] * m_t + r[4] * m1 + r[5] * noise       (m1: the previous step's x0 prediction)
     m1 <- m_t, latents <- x_next
     next_in = bf16(r[6] * x_next) into channels 0..3 of every copy   (the next step's scale_model_input)
   r[7] is the input scale of the row's own step (unused by the kernel). guidance scale = coef[row][5] of the shared
   8-float table. latents, m1 and noise (optional, NULL = none) are fp32 NHWC [batch, hw, 4], 16-byte aligned. */
typedef struct pp_solver_desc {
    const void* eps;     /* as pp_unipc_desc: [n_copies*batch, hw, eps_ld] fp32 or bf16, unconditional half first */
    int32_t eps_fp32;
    int32_t eps_ld;
    float* latents;
    float* m1;
    const float* noise;
    const float* coef;   /* [n_steps, 8], column 5 = guidance scale */
    const float* scoef;  /* [n_steps, 8] */
    int32_t* step_idx;
    int32_t advance_step;
    int32_t do_cfg;
    int32_t batch, hw;
    void* next_in;       /* bf16 NHWC [n_copies*batch, hw, next_c]: channels 0..3 refreshed */
    int32_t next_c, n_copies;
    /* device-drawn noise, as pp_cfg_ddim_desc.draws: exclusive with `noise`; nothing is drawn when r[5] is
       exactly 0. NULL / 0 = none. */
    const pp_randn_draw* draws;
    int32_t n_draws;
} pp_solver_desc;
pp_status pp_solver_step(const pp_solver_desc* d, pp_stream stream);

/* CFG combine + one step of PNDMScheduler with skip_prk_steps (PLMS: the Heun restart at counter 1, then
   Adams-Bashforth of order up to 4 on the eps history) + the optional 4-channel blend + next-step input build.
   Every step is linear in the tensors it touches, so the host folds it into one row of 8 floats (pcoef, computed in
   float64), with the history already mapped onto physical ring slots:
     x_next  = r[0] * x + r[1] * cur_sample + r[2] * eps + r[3] * ets[0] + r[4] * ets[1] + r[5] * ets[2]
     cur_sample <- x                  if r[7] != 0   (the sample a Heun restart starts again from)
     ets[(int)r[6]] <- eps            if r[6] >= 0   (written after the reads: it may replace the oldest entry)
     blend (blend_x0 != NULL), as pp_cfg_ddim_desc, with sqrt(alpha_bar) = coef[row][7]
     latents <- x_next; next_in = bf16(x_next) into channels 0..3 of every copy
   A term whose weight is exactly 0 is not read. guidance scale = coef[row][5] of the shared 8-float table.
   latents, cur_sample and every ring slot are fp32 NHWC [batch, hw, 4]; ets holds the 3 slots back to back
   ([3, batch, hw, 4]); all of them 16-byte aligned. */
typedef struct pp_plms_desc {
    const void* eps;     /* as pp_unipc_desc: [n_copies*batch, hw, eps_ld] fp32 or bf16, unconditional half first */
    int32_t eps_fp32;
    int32_t eps_ld;
    float* latents;
    float* cur_sample;
    float* ets;
    const float* coef;   /* [n_steps, 8], column 5 = guidance scale, column 7 = the blend's sqrt(alpha_bar) */
    const float* pcoef;  /* [n_steps, 8] */
    int32_t* step_idx;
    int32_t advance_step;
    int32_t do_cfg;
    int32_t batch, hw;
    void* next_in;       /* bf16 NHWC [n_copies*batch, hw, next_c]: channels 0..3 refreshed */
    int32_t next_c, n_copies;
    const float* blend_x0;     /* as pp_cfg_ddim_desc: [hw, 4] fp32, all three NULL or all set */
    const float* blend_mask;   /* [hw] fp32 */
    const float* blend_noise;  /* [batch, hw, 4] fp32 */
} pp_plms_desc;
pp_status pp_plms_step(const pp_plms_desc* d, pp_stream stream);

/* ------------------------------------------------------------------ side-net global pooling */
/* Global pooling of a side net's residual (`global_pool_conditions`: BrushNet_CA.py:936-943, diffusers
   ControlNetModel): for every sample s, pixel p and channel c of the bf16 NHWC [batch, hw, channels] buffers
     out[s, p, c] = bf16(prev[s, p, c] + mean_p x[s, p, c])          (prev == NULL: bf16(mean_p x[s, p, c]))
   The sum over p is fp32 in a fixed order, so the result is bit-identical from run to run. out is written at full
   size, so the UNet's consumers of the residual are unchanged; prev adds the residuals of earlier nets of a
   Multi-ControlNet. channels % 8 == 0; out must not alias x, prev may equal out. */
typedef struct pp_pool_broadcast_desc {
    const void* x;
    const void* prev; /* may be NULL */
    void* out;
    int32_t batch, hw, channels;
} pp_pool_broadcast_desc;
pp_status pp_pool_broadcast(const pp_pool_broadcast_desc* d, pp_stream stream);

/* ------------------------------------------------------------------ programs */
/* A program records op descriptors once (tensor maps are encoded at record time) and
   replays them with one call per denoising step; it can be instantiated as a CUDA graph. */
typedef struct pp_program pp_program;
pp_status pp_program_create(pp_program** out);
void pp_program_destroy(pp_program* p);
pp_status pp_program_add_gemm(pp_program* p, const pp_gemm_desc* d);
pp_status pp_program_add_attention(pp_program* p, const pp_attn_desc* d);
pp_status pp_program_add_group_norm(pp_program* p, const pp_gn_desc* d);
pp_status pp_program_add_layer_norm(pp_program* p, const void* x, void* y, const float* gamma,
                                    const float* beta, int32_t rows, int32_t c, float eps);
pp_status pp_program_add_upsample2x(pp_program* p, const void* x, void* y, int32_t nb, int32_t h,
                                    int32_t w, int32_t c);
pp_status pp_program_add_upsample_nearest(pp_program* p, const void* x, void* y, int32_t nb, int32_t h,
                                          int32_t w, int32_t c, int32_t ho, int32_t wo);
pp_status pp_program_add_add(pp_program* p, const void* a, const void* b, void* y, int64_t n);
pp_status pp_program_add_time_embed(pp_program* p, const float* timesteps,
                                    const int32_t* step_idx, void* out, int32_t batch, int32_t dim);
pp_status pp_program_add_cfg_ddim(pp_program* p, const pp_cfg_ddim_desc* d);
pp_status pp_program_add_unipc(pp_program* p, const pp_unipc_desc* d);
pp_status pp_program_add_solver_step(pp_program* p, const pp_solver_desc* d);
pp_status pp_program_add_plms_step(pp_program* p, const pp_plms_desc* d);
pp_status pp_program_add_memset(pp_program* p, void* ptr, int64_t bytes);
pp_status pp_program_add_embed_gather(pp_program* p, const int32_t* idx, const float* base, const float* ext,
                                      const float* pos, void* out, int32_t rows, int32_t vocab, int32_t seq, int32_t dim);
pp_status pp_program_add_causal_attention_small(pp_program* p, const void* qkv, void* out, int32_t batch, int32_t seq,
                                                int32_t heads, int32_t d, float scale);
pp_status pp_program_add_softmax_rows(pp_program* p, const float* s, void* out, int64_t rows, int32_t cols,
                                      int64_t ld_s, int64_t ld_p);
pp_status pp_program_add_window_copy(pp_program* p, const void* src, void* dst, int32_t elem_bytes, int32_t channels,
                                     int64_t src_pix, int64_t dst_pix, const pp_window* windows, int32_t count,
                                     int32_t max_pixels);
pp_status pp_program_add_tile_blend(pp_program* p, const pp_tile_blend_desc* d);
pp_status pp_program_add_pool_broadcast(pp_program* p, const pp_pool_broadcast_desc* d);
int32_t pp_program_num_ops(const pp_program* p);
/* number of kernel launches one run enqueues */
int32_t pp_program_num_launches(const pp_program* p);
/* enqueue every recorded op on `stream` (plain launches) */
pp_status pp_program_run(pp_program* p, pp_stream stream);
/* diagnostic: replay only ops [first, first + count) as plain launches */
pp_status pp_program_run_range(pp_program* p, int32_t first, int32_t count, pp_stream stream);
/* capture the program into a CUDA graph (once), then replay it with pp_program_graph_launch */
pp_status pp_program_graph_build(pp_program* p, pp_stream stream);
pp_status pp_program_graph_launch(pp_program* p, pp_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* POWERPAINT_B200_H_ */
