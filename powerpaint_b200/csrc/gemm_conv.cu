// wgmma GEMM / implicit-GEMM convolution for the PowerPaint UNet hot path (sm_90a).
//
//   D[M, N] = epilogue( A[M, K] * W[N, K]^T )        bf16 operands, fp32 accumulate in registers
//
// One kernel serves every dense contraction of the per-step UNet / BrushNet forward
// (reference call sites: nn.Linear / nn.Conv2d inside ResnetBlock2D, Transformer2DModel,
// Downsample2D, Upsample2D — powerpaint/models/unet_2d_blocks.py:789,807,1274,1289,1319,
// 1428,2499,2514,2542,2672,2689 — conv_in / conv_out unet_2d_condition.py:256,477, and the
// BrushNet zero-convs BrushNet_CA.py:330-376,446-454):
//
//  * A operand. PP_A_MATRIX: 2-D TMA tiles of a token-major matrix. PP_A_CONV3X3: the
//    activation stays NHWC in HBM and each of the 9 filter taps is one 4-D TMA box
//    (64 channels x bw x bh x bn pixels) shifted by the tap offset; the halo and every
//    ragged edge (channels, width, height, batch) are zero-filled by TMA's out-of-bounds
//    rule, so there is no im2col buffer and no padding copy. PP_A_CONV3X3_S2 (Downsample2D)
//    uses four parity-plane tensor maps so a stride-2 tap is again a dense box.
//    Up to two A sources are walked back to back along K: the up-path skip concat
//    (unet_2d_blocks.py:2589,2732) never materialises.
//  * B operand: weights [N, K] K-major, K ordered (tap, source, channel) to match.
//  * Pipeline: persistent kernel, one 288-thread CTA per SM. Warp 8 = TMA producer; warps 0..7 = two consumer
//    warpgroups, each issuing the wgmma.mma_async of 64 rows of the 128 x BLOCK_N tile and then running the epilogue
//    of those rows. STAGES-deep smem ring with full/empty mbarriers that keeps running across tile boundaries, so the
//    producer streams the next tile's operands while the consumers run this tile's epilogue. The accumulators go
//    through a shared-memory fp32 tile (row per epilogue thread) that shares its space with the output staging tile.
//  * Split-K x2 (few tiles, long K): two CTAs per tile each stream half of K; the second hands its fp32 partial tile
//    to the first through a global workspace (see the comment at the kernel).
//  * Epilogue (fused): + bias[n] + time-embedding row vector + residual (skip / shortcut)
//    → × alpha (1/output_scale_factor or BrushNet conditioning_scale) → + second residual
//    (BrushNet / ControlNet feature injection, unet_2d_condition.py:1223,1300) → SiLU /
//    GEGLU gate → bf16 or fp32 store, optionally transposed (V^T for the attention kernel; q | k | v^T of an attention
//    leave one launch, the V tiles through a transposed staging tile). The LayerNorms of BasicTransformerBlock live in
//    the epilogues either side of them: the producer leaves {rstd, -rstd * mean} per row, the consumer multiplies the
//    raw activations by W * gamma and finishes the normalisation with two FMAs per element.
#include <algorithm>
#include <type_traits>

#include <cuda_fp16.h>

#include "common.cuh"
#include "ops.h"
#include "wgmma.cuh"

// -DGEMM_TRACE: CTA 0 records clock64() at the role hand-overs of its first tiles (read with pp_debug_gemm_trace)
#ifdef GEMM_TRACE
__device__ long long g_gemm_trace[64 * 32];
#define GT(tile_local, slot)                                                                     \
    do {                                                                                         \
        if (blockIdx.x == 0 && (tile_local) < 64) g_gemm_trace[(tile_local) * 32 + (slot)] = clock64(); \
    } while (0)
extern "C" int pp_debug_gemm_trace(long long* host_out, int n) {
    return (int)cudaMemcpyFromSymbol(host_out, g_gemm_trace, sizeof(long long) * (size_t)n);
}
#else
#define GT(tile_local, slot) do {} while (0)
#endif

namespace pp {

static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;
static constexpr int WGMMA_K = 16;
static constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KiB
static constexpr int GEMM_EPI_WARPS = 8;                     // two consumer warpgroups
static constexpr int GEMM_THREADS = 32 + 32 * GEMM_EPI_WARPS;
static constexpr int GEMM_SMEM_LIMIT = 227 * 1024 - 256;     // H100 per-block opt-in maximum, minus static shared memory

__device__ __forceinline__ float apply_act(float v, int act) {
    return act == PP_ACT_SILU ? silu_f(v) : act == PP_ACT_QUICK_GELU ? quick_gelu_f(v) : v;
}

// effective alpha of a launch: the recorded constant times an optional device-side factor (the
// per-step side-net scale, read through the device step counter so a captured graph stays valid)
__device__ __forceinline__ float effective_alpha(const GemmKParams& p) {
    float a = p.alpha;
    if (p.alpha_dev) a *= __ldg(p.alpha_dev + (int64_t)(p.alpha_step ? *p.alpha_step : 0) * p.alpha_stride);
    return a;
}

// Column sums of the staged output tile for the consumer's GroupNorm. L threads (consecutive lanes of a
// warp) share one 8-channel piece and split the rows of a sample segment between them (row = l, l + L, ...:
// conflict-free shared-memory reads); v[] holds {sum, sum of squares} interleaved per channel, both of
// x - shift where shift is the segment's first row (so a large mean over a small spread does not cancel when
// the consumer forms the variance). A halving butterfly leaves every lane with 16 / L of the 16 totals, in
// memory order; per channel the record is {sum, sum of squares, shift, 0} (16 bytes).
template <int L>
__device__ __forceinline__ void stats_butterfly_store(const float (&v)[16], const float (&shift)[8], int l, float* dst,
                                                      bool write) {
    float a[8], b[4], c[2];
    {
        const bool hi = (l & (L / 2)) != 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float send = hi ? v[k] : v[k + 8], keep = hi ? v[k + 8] : v[k];
            a[k] = keep + __shfl_xor_sync(0xffffffffu, send, L / 2);
        }
    }
    {
        const bool hi = (l & (L / 4)) != 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float send = hi ? a[k] : a[k + 4], keep = hi ? a[k + 4] : a[k];
            b[k] = keep + __shfl_xor_sync(0xffffffffu, send, L / 4);
        }
    }
    {
        const bool hi = (l & (L / 8)) != 0;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float send = hi ? b[k] : b[k + 2], keep = hi ? b[k + 2] : b[k];
            c[k] = keep + __shfl_xor_sync(0xffffffffu, send, L / 8);
        }
    }
    // per channel: {sum of (x - shift), sum of (x - shift)^2, shift, 0}; lane -> channel via a static select
    auto shift_of = [&](int ch) {
        float r = shift[0];
#pragma unroll
        for (int j = 1; j < 8; ++j) r = ch == j ? shift[j] : r;
        return r;
    };
    if constexpr (L == 8) {
        if (write) *reinterpret_cast<float4*>(dst + 4 * l) = make_float4(c[0], c[1], shift_of(l), 0.f);
    } else {
        static_assert(L == 16, "row lanes");
        const bool hi = (l & 1) != 0;
        const float send = hi ? c[0] : c[1], keep = hi ? c[1] : c[0];
        const float d = keep + __shfl_xor_sync(0xffffffffu, send, 1);
        if (write) {
            dst[4 * (l >> 1) + (l & 1)] = d;
            if (!hi) *reinterpret_cast<float2*>(dst + 4 * (l >> 1) + 2) = make_float2(shift_of(l >> 1), 0.f);
        }
    }
}

// (m_tile, n_tile) of the tiles one persistent CTA walks: tile = blockIdx.x + i * gridDim.x, n fastest.
// Kept incrementally — a runtime integer division costs ~40 dependent instructions, and the producer
// and every consumer thread would otherwise pay two of them per tile.
struct TileWalk {
    int m, n, step_m, step_n, n_tiles;
    __device__ __forceinline__ TileWalk(int first, int stride, int n_tiles_) : n_tiles(n_tiles_) {
        m = first / n_tiles_;
        n = first - m * n_tiles_;
        step_m = stride / n_tiles_;
        step_n = stride - step_m * n_tiles_;
    }
    __device__ __forceinline__ void next() {
        m += step_m;
        n += step_n;
        if (n >= n_tiles) {
            n -= n_tiles;
            ++m;
        }
    }
};

// Epilogue for 8 consecutive output columns of one row. v[] holds the accumulators; `sbias` points
// at this tile's bias staged in shared memory (column n0 - n_base), r1/r2 hold the 8 bf16 residual
// values that were loaded ahead of time (vector path only).
template <bool kVec>
__device__ __forceinline__ void epilogue_store8(const GemmKParams& p, float alpha, float (&v)[8], int64_t row, int grp,
                                                int n0, const float* sbias, uint4 r1, uint4 r2) {
    if (p.bias) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += sbias[j];
    }
    if (p.rowvec) {
        const float* rv = p.rowvec + (int64_t)grp * p.rowvec_ld + n0;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (kVec || n0 + j < p.N) v[j] += __ldg(rv + j);
    }
    if (p.res1) {
        if (kVec) {
            v[0] += bf16_lo(r1.x); v[1] += bf16_hi(r1.x); v[2] += bf16_lo(r1.y); v[3] += bf16_hi(r1.y);
            v[4] += bf16_lo(r1.z); v[5] += bf16_hi(r1.z); v[6] += bf16_lo(r1.w); v[7] += bf16_hi(r1.w);
        } else {
            const __nv_bfloat16* r = p.res1 + row * p.ldr1 + n0;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (n0 + j < p.N) v[j] += __bfloat162float(r[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= alpha;
    if (p.res2) {
        if (kVec) {
            v[0] += bf16_lo(r2.x); v[1] += bf16_hi(r2.x); v[2] += bf16_lo(r2.y); v[3] += bf16_hi(r2.y);
            v[4] += bf16_lo(r2.z); v[5] += bf16_hi(r2.z); v[6] += bf16_lo(r2.w); v[7] += bf16_hi(r2.w);
        } else {
            const __nv_bfloat16* r = p.res2 + row * p.ldr2 + n0;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (n0 + j < p.N) v[j] += __bfloat162float(r[j]);
        }
    }
    if (p.act != PP_ACT_NONE) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = apply_act(v[j], p.act);
    }
    if (p.epilogue == PP_EPI_TRANSPOSED) {
        // out[(row / t_rows) * N + n][row % t_rows]; lanes of a warp hold consecutive rows,
        // so each per-column store is a 64-byte contiguous run across the warp.
        const int64_t b = (int)row / p.t_rows;  // 32-bit: a 64-bit division is a subroutine call, which would serialise the wgmma pipeline
        const int64_t t = row - b * p.t_rows;
        if (p.t_fp16) {
            __half* o = reinterpret_cast<__half*>(p.out) + (b * p.N + n0) * p.t_ld + t;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (kVec || n0 + j < p.N) o[(int64_t)j * p.t_ld] = __float2half_rn(v[j]);
            return;
        }
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + (b * p.N + n0) * p.t_ld + t;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (kVec || n0 + j < p.N) o[(int64_t)j * p.t_ld] = __float2bfloat16_rn(v[j]);
        return;
    }
    if (p.out_fp32) {
        float* o = reinterpret_cast<float*>(p.out) + row * p.ldc + n0;
        if (kVec) {
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (n0 + j < p.N) o[j] = v[j];
        }
    } else {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + row * p.ldc + n0;
        if (kVec) {
            uint4 q;
            q.x = pack_bf16x2(v[0], v[1]);
            q.y = pack_bf16x2(v[2], v[3]);
            q.z = pack_bf16x2(v[4], v[5]);
            q.w = pack_bf16x2(v[6], v[7]);
            *reinterpret_cast<uint4*>(o) = q;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (n0 + j < p.N) o[j] = __float2bfloat16_rn(v[j]);
        }
    }
}

// Accumulator tile in shared memory: fp32 rows of BLOCK_N + 4 floats (the pad spreads the row-per-thread reads over
// the banks). Up to 160 columns it holds all 128 rows; the 256-wide tile holds the 64 rows of one warpgroup at a
// time (the two warpgroups take turns), which leaves room for three ring stages.
__host__ __device__ constexpr int acc_rows_for(int block_n) { return block_n == 256 ? 64 : 128; }
__host__ __device__ constexpr int acc_ld_for(int block_n) { return block_n + 4; }
// Output staging tile: the epilogue writes its accumulator rows (bf16) into shared memory laid out as the boxes
// of a TMA store — 64-column sub-tiles [128 rows][128 B] with the 128-byte swizzle (the 160-wide tile ends in a
// 32-column sub-tile [128][64 B] with the 64-byte swizzle) — and one thread per sub-tile hands them to the TMA unit,
// which writes whole rows and clips whatever lies outside the tensor (ragged conv tiles, rows >= M, columns >= N).
__host__ __device__ constexpr int out_stage_bytes_for(int block_n) {
    return (block_n / 64) * 16384 + (block_n % 64) * 256;
}
// the staging tile and the accumulator tile share one 1024-byte aligned region
__host__ __device__ constexpr int acc_region_bytes_for(int block_n) {
    return ((acc_rows_for(block_n) * acc_ld_for(block_n) * 4 > out_stage_bytes_for(block_n)
                 ? acc_rows_for(block_n) * acc_ld_for(block_n) * 4
                 : out_stage_bytes_for(block_n)) + 1023) / 1024 * 1024;
}
// fixed part: 1 KB alignment slack, barriers, bias + LayerNorm-sum staging [4][BLOCK_N] floats, row table
__host__ __device__ constexpr int fixed_smem_for(int block_n) {
    return 1024 + 256 + 4 * block_n * 4 + 128 * 8 + 1024 + acc_region_bytes_for(block_n);
}
// as many ring stages as the per-block shared memory takes (at most 8)
__host__ __device__ constexpr int stages_for(int block_n) {
    return (GEMM_SMEM_LIMIT - fixed_smem_for(block_n)) / (A_STAGE_BYTES + block_n * BLOCK_K * 2) < 8
               ? (GEMM_SMEM_LIMIT - fixed_smem_for(block_n)) / (A_STAGE_BYTES + block_n * BLOCK_K * 2)
               : 8;
}
__host__ __device__ constexpr int smem_bytes_for(int block_n) {
    return stages_for(block_n) * (A_STAGE_BYTES + block_n * BLOCK_K * 2) + fixed_smem_for(block_n);
}
static_assert(stages_for(256) >= 2 && smem_bytes_for(256) <= GEMM_SMEM_LIMIT, "256-wide tile does not fit");
static_assert(stages_for(160) >= 3 && stages_for(128) >= 3 && stages_for(64) >= 3, "ring too shallow");

// Persistent, warp-specialised kernel: grid = min(#tiles, #SMs); each CTA walks tiles
// blockIdx.x, blockIdx.x + gridDim.x, ... (n fastest, so CTAs running concurrently share A tiles
// through L2 and the weights stay L2-resident).
//   warp 8      TMA producer  (smem ring continues across tile boundaries)
//   warps 0..7  two consumer warpgroups: warpgroup g issues the wgmma of tile rows [64 g, 64 g + 64) and then runs
//               the epilogue of the same rows — each of its four warps takes 32 rows and one half of the columns
//               (alternating 32-column chunks), reading its row of the accumulator tile in shared memory
// MODE selects the epilogue flavour at compile time (keeps the hot epilogue short and the
// instruction footprint small): 0 = bf16 row-major output, N % 8 == 0 (bias, rowvec, two residuals,
// alpha, SiLU), 1 = generic (fp32 / transposed / ragged N), 2 = GEGLU, 3 = mode 0 emitting the per-row records of the
// consumer's LayerNorm, 4 = mode 0 with LayerNorm of A applied algebraically (bias only), 5 = bias-only bf16 output
// whose n-tiles from trans_first_tile on are stored TRANSPOSED through the staging tile (to_q | to_k | to_v^T of an
// attention in one launch, or V^T alone), optionally with the LayerNorm fold.
// kSplitK (mode 0 only, p.ksplit == 2): the launch has one work item per CTA, item = 2 * tile + half; the CTA with
// half 1 ("donor") hands its fp32 partial accumulators to the CTA with half 0 ("owner") through a global workspace and
// a flag, the owner adds them (always owner + donor: deterministic) and runs the epilogue. For the layers whose tiles
// fill less than half of the GPU (8x8 resolution; 16x16 at small batch) every CTA then streams half of K. The grid
// (2 x tiles) never exceeds the SM count, so owner and donor are resident together.
template <int BLOCK_N, int MODE, bool kSplitK = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_conv_kernel(const __grid_constant__ GemmKParams p) {
    constexpr int STAGES = stages_for(BLOCK_N);
    constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;
    constexpr int ACC_ROWS = acc_rows_for(BLOCK_N), ACC_LD = acc_ld_for(BLOCK_N);
    constexpr bool kAccShared = ACC_ROWS < BLOCK_M;  // the two warpgroups take turns in the accumulator tile

    extern __shared__ uint8_t smem_raw[];
    // mode 3 (LayerNorm-statistics producer): mailbox between the epilogue and the ticket-server lane, and the verdict
    // ("this CTA finished the last n-tile of the row block") of the tile whose records are folded next
    __shared__ volatile int s_req_seq, s_req_mtile, s_resp_seq, s_resp_last;
    __shared__ int s_last_tile;
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem_base;
    const uint32_t sB = sA + STAGES * A_STAGE_BYTES;
    // accumulator tile / output staging tile (aliased), 1024-byte aligned
    const uint32_t s_out_addr = sB + STAGES * B_STAGE_BYTES;
    uint8_t* s_out = smem_raw + (s_out_addr - smem_u32(smem_raw));
    float* sacc = reinterpret_cast<float*>(s_out);
    const uint32_t bar_base = s_out_addr + acc_region_bytes_for(BLOCK_N);
    // barriers: full[STAGES], empty[STAGES]
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
    // bias of the current / next tile, staged by the epilogue warps: [2][BLOCK_N] floats
    float* sbias_all = reinterpret_cast<float*>(smem_raw + (bar_base + 256 - smem_u32(smem_raw)));
    // column sums of the gamma-folded weights (LayerNorm fold), staged like the bias: [2][BLOCK_N] floats
    float* su_all = sbias_all + 2 * BLOCK_N;
    // validity of each tile row (statistics pass)
    long long* s_row = reinterpret_cast<long long*>(reinterpret_cast<uint8_t*>(sbias_all) + 4 * BLOCK_N * 4);
    // 16-byte piece of row r holding columns [col, col + 8) of the staged tile
    auto stage_ptr = [&](int r, int col) -> uint8_t* {
        const int sub = col >> 6, c = (col & 63) >> 3;
        if ((BLOCK_N % 64) != 0 && sub == BLOCK_N / 64)  // 32-column remainder sub-tile, 64-byte swizzle
            return s_out + sub * 16384 + r * 64 + ((c ^ ((r >> 1) & 3)) << 4);
        return s_out + sub * 16384 + r * 128 + ((c ^ (r & 7)) << 4);
    };

    const int warp = threadIdx.x >> 5;
    const int n_tiles = p.n_tiles;
    const int num_tiles = p.m_tiles * n_tiles;
    constexpr bool split = kSplitK;
    const int khalf = split ? (int)(blockIdx.x & 1) : 0;
    const int walk_first = split ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
    const int walk_stride = split ? num_tiles : (int)gridDim.x;
    const int num_k_iters = p.num_k_iters;
    const int k_begin = split ? khalf * (num_k_iters / 2) : 0;
    const int k_end = split ? (khalf ? num_k_iters : num_k_iters / 2) : num_k_iters;

    constexpr int W_PROD = GEMM_EPI_WARPS;
    if (warp == W_PROD && elect_one()) {
        prefetch_tmap(&p.tmA[0]);
        prefetch_tmap(&p.tmB);
        if constexpr (MODE != 1) prefetch_tmap(&p.tmOut[0]);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), GEMM_EPI_WARPS);  // one arrival per consumer warp
        }
        fence_mbar_init();
        if constexpr (MODE == 3) { s_req_seq = 0; s_resp_seq = 0; s_req_mtile = 0; s_resp_last = 0; }
    }
    __syncthreads();
    // everything above touched only shared memory and kernel parameters; global memory
    // written by the preceding kernel is read (and this kernel's output written) from here on
    pdl_wait();
    pdl_launch_dependents();

    // conv tile origin of an m-tile index
    auto tile_origin = [&](int m_tile, int& x0, int& y0, int& nb0) {
        const int tx = m_tile % p.tiles_x;
        const int ty = (m_tile / p.tiles_x) % p.tiles_y;
        const int tn = m_tile / (p.tiles_x * p.tiles_y);
        x0 = tx * p.bw;
        y0 = ty * p.bh;
        nb0 = tn * p.bn;
    };

    if (warp == W_PROD) {
        // ===================== TMA producer =====================
        // mode 3: lane 0 produces and lane 31 serves the row-block tickets. The ticket of a tile (fence + atomic round
        // trip, ~1500 cycles) used to sit between the epilogue's two barriers; the server takes it while the epilogue
        // is already in the next tile, which collects the verdict at its first barrier.
        const bool is_producer = MODE == 3 ? lane_id() == 0 : elect_one();
        if (MODE == 3 && lane_id() == 31) {
            for (int seq = 1;; ++seq) {
                const uint64_t t0 = global_timer_ns();
                uint32_t spins = 0;
                while (s_req_seq < seq) {
                    __nanosleep(40);
                    if ((++spins & 0x3FFu) == 0 && global_timer_ns() - t0 > PP_WAIT_TIMEOUT_NS) __trap();
                }
                __threadfence_block();
                const int mt = s_req_mtile;
                if (mt < 0) break;  // the epilogue is done
                // the epilogue's barrier ordered every warp's record stores before the request; this fence is
                // cumulative, so they are visible device-wide before the ticket is
                __threadfence();
                const int t = atomicAdd(p.row_ticket + mt, 1);
                if (t == n_tiles - 1) p.row_ticket[mt] = 0;  // ready for the next launch
                s_resp_last = (t == n_tiles - 1) ? 1 : 0;
                __threadfence_block();
                s_resp_seq = seq;
            }
        }
        if (is_producer) {
            const int cpt = p.chunks0 + p.chunks1;  // chunks per tap
            int s = 0;                              // ring slot and its phase, carried across tiles
            uint32_t ph = 0;
            TileWalk tw(walk_first, walk_stride, n_tiles);
            for (int tile = walk_first; tile < num_tiles; tile += walk_stride, tw.next()) {
                const int n_tile = tw.n, m_tile = tw.m;
                int x0 = 0, y0 = 0, nb0 = 0;
                if (p.a_mode != PP_A_MATRIX) tile_origin(m_tile, x0, y0, nb0);
                int ky = 0, kx = 0, ch = 0;  // filter tap and 64-channel chunk of this k-iteration
                if (k_begin) {  // second half of a split contraction: tap / chunk of its first k-iteration
                    const int tap = k_begin / cpt;
                    ch = k_begin - tap * cpt;
                    ky = tap / 3;
                    kx = tap - ky * 3;
                }
                for (int it = k_begin; it < k_end; ++it) {
                    mbar_wait(empty_bar(s), ph ^ 1u);
                    if (it == k_begin) GT((tile - walk_first) / walk_stride, 0);
                    if (it == k_end - 1) GT((tile - walk_first) / walk_stride, 1);
#if defined(GEMM_EXP_NOLOAD)  // experiment: no TMA traffic at all (operands are whatever the smem holds)
                    mbar_arrive(full_bar(s));
                    if (++ch == cpt) {
                        ch = 0;
                        if (++kx == 3) { kx = 0; ++ky; }
                    }
                    if (++s == STAGES) { s = 0; ph ^= 1u; }
                    continue;
#elif defined(GEMM_EXP_NOLOADB)  // experiment: activations only
                    mbar_arrive_expect_tx(full_bar(s), p.a_bytes);
#elif defined(GEMM_EXP_NOLOADA)  // experiment: weights only
                    mbar_arrive_expect_tx(full_bar(s), B_STAGE_BYTES);
#else
                    mbar_arrive_expect_tx(full_bar(s), p.a_bytes + B_STAGE_BYTES);
#endif
                    const uint32_t dstA = sA + s * A_STAGE_BYTES;
                    const uint32_t dstB = sB + s * B_STAGE_BYTES;
                    const int src = ch >= p.chunks0 ? 1 : 0;
                    const int cc = (src ? ch - p.chunks0 : ch) * BLOCK_K;
#ifdef GEMM_EXP_NOLOADA
                    if (false) {
                    } else
#endif
                    if (p.a_mode == PP_A_MATRIX) {
                        tma_load_2d(dstA, &p.tmA[src], full_bar(s), cc, m_tile * BLOCK_M);
                    } else if (p.a_mode == PP_A_CONV3X3) {
                        tma_load_4d(dstA, &p.tmA[src], full_bar(s), cc, x0 + kx - 1, y0 + ky - 1, nb0);
                    } else if (p.a_mode == PP_A_CONV3X3_S2) {
                        // stride 2: input (2*oy + ky - 1, 2*ox + kx - 1) = parity plane (py, px) at
                        // (oy + dy, ox + dx) with d = -1 for k == 0 else 0, parity = (k != 1)
                        const int py = (ky != 1), px = (kx != 1);
                        const int dy = (ky == 0) ? -1 : 0, dx = (kx == 0) ? -1 : 0;
                        tma_load_4d(dstA, &p.tmA[py * 2 + px], full_bar(s), cc, x0 + dx, y0 + dy, nb0);
                    } else {
                        // stride 2 over the bottom/right zero-padded input: (2*oy + ky, 2*ox + kx) = parity
                        // plane (k & 1) at (o + (k >> 1)); the pad row / column is TMA's out-of-bounds zero
                        tma_load_4d(dstA, &p.tmA[(ky & 1) * 2 + (kx & 1)], full_bar(s), cc, x0 + (kx >> 1), y0 + (ky >> 1),
                                    nb0);
                    }
#ifndef GEMM_EXP_NOLOADB
                    tma_load_2d(dstB, &p.tmB, full_bar(s), it * BLOCK_K, n_tile * BLOCK_N);
#endif
                    if (++ch == cpt) {
                        ch = 0;
                        if (++kx == 3) { kx = 0; ++ky; }
                    }
                    if (++s == STAGES) { s = 0; ph ^= 1u; }
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: MMA + epilogue =====================
        const int wg = warp >> 2;                         // warpgroup: tile rows [64 wg, 64 wg + 64)
        const int quarter = (warp & 1) + 2 * wg;          // rows of this warp: [32*quarter, +32)
        const int half = (warp >> 1) & 1;                 // which of the two warps sharing those rows
        const int etid = threadIdx.x;        // 0..255 among the epilogue threads
        const int r = quarter * 32 + (int)lane_id();
        // this thread's row of the accumulator tile
        const float* arow = sacc + (r - (kAccShared ? 64 * wg : 0)) * ACC_LD;
        auto acc_ld = [](const float* src, auto& dst) {
            constexpr int NV = sizeof(dst) / sizeof(dst[0]);
#pragma unroll
            for (int i = 0; i < NV; i += 4) {
                const float4 v = *reinterpret_cast<const float4*>(src + i);
                dst[i] = __float_as_uint(v.x); dst[i + 1] = __float_as_uint(v.y);
                dst[i + 2] = __float_as_uint(v.z); dst[i + 3] = __float_as_uint(v.w);
            }
        };
        const bool vec_ok = (p.N % 8 == 0);
        auto epi_sync = [] { asm volatile("bar.sync 1, %0;" ::"n"(GEMM_EPI_WARPS * 32) : "memory"); };
        // ---- main loop of one tile: this warpgroup's 64 x BLOCK_N accumulators, then into the accumulator tile
        int ks = 0;  // ring slot and its phase, carried across tiles (the producer's sequence)
        uint32_t kph = 0;
        auto mainloop = [&](int m_tile, int n_tile) {
            // zeroed here (not by the first MMA's scale-d): the registers are then dead between tiles
            float facc[BLOCK_N / 2];
#pragma unroll
            for (int i = 0; i < BLOCK_N / 2; ++i) facc[i] = 0.f;
            int prev = 0;
            for (int it = k_begin; it < k_end; ++it) {
                mbar_wait(full_bar(ks), kph);
                const uint64_t da = wgmma_desc_kmajor_sw128(sA + ks * A_STAGE_BYTES + wg * (A_STAGE_BYTES / 2));
                const uint64_t db = wgmma_desc_kmajor_sw128(sB + ks * B_STAGE_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
                    Wgmma<BLOCK_N>::ss_bf16(facc, wgmma_desc_advance_k(da, k * WGMMA_K), wgmma_desc_advance_k(db, k * WGMMA_K), 1);
                wgmma_commit();
                // one group stays in flight: the previous stage's MMAs have retired, its slot goes back to the producer
                wgmma_wait<1>();
                if (it > k_begin && lane_id() == 0) mbar_arrive(empty_bar(prev));
                prev = ks;
                if (++ks == STAGES) { ks = 0; kph ^= 1u; }
            }
            wgmma_wait<0>();
            wgmma_fence_regs(facc);
            if (lane_id() == 0) mbar_arrive(empty_bar(prev));
            if constexpr (kSplitK) {
                if (!khalf && etid == 0) {  // owner: the donor's partial tile is complete (flag set after its fence)
                    volatile int32_t* fl = p.splitk_flags + (int64_t)m_tile * n_tiles + n_tile;
                    const uint64_t t0 = global_timer_ns();
                    uint32_t spins = 0;
                    while (*fl == 0) {
                        if ((++spins & 0xFFFu) == 0 && global_timer_ns() - t0 > PP_WAIT_TIMEOUT_NS) __trap();
                    }
                    __threadfence();
                    *fl = 0;  // ready for the next launch
                }
            }
            // the accumulator tile shares its space with the staging tile: the TMA unit has read the previous tile out
            // of it, and every epilogue thread is past its reads of it (statistics pass included)
            if constexpr (MODE != 1) {
                if ((etid & 31) == 0) bulk_wait_read_all();
            }
            epi_sync();
            if constexpr (kAccShared) {  // warpgroup 1 waits until warpgroup 0 has read its rows out
                if (wg == 1) asm volatile("bar.sync 2, %0;" ::"n"(GEMM_EPI_WARPS * 32) : "memory");
            }
            {
                const int w4 = warp & 3, l = (int)lane_id();
                float* dst = sacc + ((kAccShared ? 0 : 64 * wg) + 16 * w4 + (l >> 2)) * ACC_LD + 2 * (l & 3);
#pragma unroll
                for (int i = 0; i < BLOCK_N / 8; ++i) {
                    *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(facc[4 * i], facc[4 * i + 1]);
                    *reinterpret_cast<float2*>(dst + 8 * ACC_LD + 8 * i) = make_float2(facc[4 * i + 2], facc[4 * i + 3]);
                }
            }
            // the warpgroup's rows are complete (each warpgroup reads only the rows it wrote)
            if (wg == 0) asm volatile("bar.sync 3, 128;" ::: "memory");
            else asm volatile("bar.sync 4, 128;" ::: "memory");
        };
        auto load_bias = [&](int n_tile_of) -> float {
            const int n = n_tile_of * BLOCK_N + etid;
            // volatile asm: the load must be issued HERE (a tile ahead of its use); a plain __ldg gets
            // sunk by the compiler to just before the shared-memory store at the end of the tile, which
            // exposes a full global-memory latency per tile right in front of the epilogue barrier
            float v = 0.f;
            if (p.bias && etid < BLOCK_N && n < p.N)
                asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p.bias + n));
            return v;
        };
        // LayerNorm of A folded into this epilogue: modes 1 and 2 decide at run time; of the fast bf16 flavours only
        // mode 4 carries it (and only mode 3 emits the records), so the big convs in mode 0 keep their register budget
        const bool ln = (MODE == 1 || MODE == 2 || MODE == 4 || MODE == 5) && p.ln_stats != nullptr;
        auto load_u = [&](int n_tile_of) -> float {
            const int n = n_tile_of * BLOCK_N + etid;
            float v = 0.f;
            if (ln && etid < BLOCK_N && n < p.N)
                asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p.ln_u + n));
            return v;
        };
        // stage the first tile's bias
        TileWalk tw(walk_first, walk_stride, n_tiles);
        if (walk_first < num_tiles) {
            const float b0 = load_bias(tw.n);
            const float u0 = load_u(tw.n);
            if (etid < BLOCK_N) {
                sbias_all[etid] = b0;
                su_all[etid] = u0;
            }
        }
        epi_sync();
        float2 ln_cur = make_float2(1.f, 0.f);  // {rstd, -rstd * mean} of this thread's row in the current tile
        if (ln && walk_first < num_tiles) {
            const int64_t row0 = (int64_t)tw.m * BLOCK_M + r;
            if (row0 < p.M) ln_cur = __ldg(p.ln_stats + row0);
        }
        // ---- mode 3: verdict of the ticket server for request number `seq`, and the fold of a row's records
        int64_t prev_row = 0;
        bool prev_valid = false;
        auto ticket_verdict = [&](int seq) -> int {
            const uint64_t t0 = global_timer_ns();
            uint32_t spins = 0;
            while (s_resp_seq < seq) {
                if ((++spins & 0xFFFu) == 0 && global_timer_ns() - t0 > PP_WAIT_TIMEOUT_NS) __trap();
            }
            __threadfence_block();
            return s_resp_last;
        };
        auto fold_row_records = [&](const float4 (&first)[4], int64_t frow) {
            // Chan's combination of the (count, mean, M2) of the row's half-tile records -> {rstd, -rstd * mean}
            float cnt = 0.f, mean = 0.f, m2 = 0.f;
            auto fold = [&](const float4& rc) {
                if (rc.w > 0.f) {
                    const float inv = __fdividef(1.f, rc.w);
                    const float mi = fmaf(rc.x, inv, rc.z);
                    const float m2i = fmaxf(fmaf(-rc.x * inv, rc.x, rc.y), 0.f);
                    const float tot = cnt + rc.w;
                    const float wgt = __fdividef(rc.w, tot);
                    const float dl = mi - mean;
                    mean = fmaf(dl, wgt, mean);
                    m2 += m2i + dl * dl * cnt * wgt;
                    cnt = tot;
                }
            };
#pragma unroll
            for (int u = 0; u < 4; ++u) fold(first[u]);
            const int nrec = 2 * n_tiles;
            for (int i0 = 4; i0 < nrec; i0 += 4) {
                float4 rc[4];
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    rc[u] = i0 + u < nrec ? __ldcg(p.row_stats + (int64_t)(i0 + u) * p.row_stats_ld + frow)
                                          : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int u = 0; u < 4; ++u) fold(rc[u]);
            }
            const float var = cnt > 0.f ? __fdividef(m2, cnt) : 0.f;
            const float rs = rsqrtf(var + p.ln_eps);
            p.row_final[frow] = make_float2(rs, -rs * mean);
        };
        uint32_t lt = 0;
        for (int tile = walk_first; tile < num_tiles; tile += walk_stride, ++lt) {
            if (etid == 0) GT(lt, 15);  // top of the tile
            const int n_tile = tw.n, m_tile = tw.m;
            tw.next();  // now at the tile after this one
            const uint32_t acc = lt & 1u;  // bias staging buffer of this tile
            const float* sbias = sbias_all + acc * BLOCK_N;
            const float* su = su_all + acc * BLOCK_N;
            // bias (and LayerNorm weight row sums) of the NEXT tile: an asynchronous global -> shared copy straight into the
            // other staging buffer (its readers, tile lt - 1, are all past that tile's second barrier). A value loaded
            // into a register here had to live across the whole tile; with the kernel at its register cap it was spilled
            // at once, which made every thread wait ~700 cycles for the load right here, in front of each tile.
            const int next_tile = tile + walk_stride;
            if (etid < BLOCK_N) {
                const int nn = tw.n * BLOCK_N + etid;
                float* db = sbias_all + (acc ^ 1u) * BLOCK_N + etid;
                float* du = su_all + (acc ^ 1u) * BLOCK_N + etid;
                if (next_tile < num_tiles && p.bias && nn < p.N) cp_async_f32(db, p.bias + nn);
                else *db = 0.f;
                if (next_tile < num_tiles && ln && nn < p.N) cp_async_f32(du, p.ln_u + nn);
                else *du = 0.f;
            }
            if (etid == 0) GT(lt, 16);
            // output row of this thread
            bool valid;
            int64_t row;
            int grp;
            if (p.a_mode == PP_A_MATRIX) {
                row = (int64_t)m_tile * BLOCK_M + r;
                valid = row < p.M;
                grp = p.rowvec ? (int)row / p.rows_per_group : 0;
            } else {
                int x0, y0, nb0;
                tile_origin(m_tile, x0, y0, nb0);
                // bw, bh, bn are powers of two
                const int ix = r & (p.bw - 1);
                const int iy = (r >> p.bw_log2) & (p.bh - 1);
                const int in = r >> (p.bw_log2 + p.bh_log2);
                const int ox = x0 + ix, oy = y0 + iy, on = nb0 + in;
                valid = in < p.bn && ox < p.wo && oy < p.ho && on < p.nb;
                row = ((int64_t)on * p.ho + oy) * p.wo + ox;
                grp = on;
            }
            if (etid == 0) GT(lt, 17);
            const int n_base = n_tile * BLOCK_N;
            // mode 5: this tile's columns are stored transposed ([channel][token], V^T for the attention kernel)
            const bool ttile = MODE == 5 && n_tile >= p.trans_first_tile;
            // LayerNorm fold: acc' = ln_rs * acc + ln_nm * u[n] with {ln_rs, ln_nm} = {rstd, -rstd * mean} of this row, as
            // left by the producer (row_final). The pair of the NEXT tile's row is fetched now, so that its global-memory
            // latency is off the epilogue's serial path (a per-tile fold of the raw records cost ~2500 cycles a tile).
            const float ln_rs = ln_cur.x, ln_nm = ln_cur.y;
            if (ln) {
                const int64_t nrow = (int64_t)tw.m * BLOCK_M + r;  // tw is already at the next tile
                ln_cur = (next_tile < num_tiles && nrow < p.M) ? __ldg(p.ln_stats + nrow) : make_float2(1.f, 0.f);
            }
            // The tile's results stay in registers (packed bf16, 8 columns per uint4) until every thread has read its
            // row of the accumulator tile, whose space the staging tile reuses.
            constexpr int PK_N = MODE == 2 ? BLOCK_N / 32 : MODE == 1 ? 1 : BLOCK_N / 16;
            uint4 pk[PK_N];
            if constexpr (MODE == 2) {
                constexpr int HALF = BLOCK_N / 2;
                const int o_base = n_tile * HALF;  // output column of this tile
                const int n_out = p.N / 2;
                mainloop(m_tile, n_tile);
#pragma unroll
                for (int k = 0; k < BLOCK_N / 64; ++k) {
                    const int c0 = half * 16 + 32 * k;
                    uint32_t ra[16], rg[16];
                    acc_ld(arow + c0, ra);
                    acc_ld(arow + HALF + c0, rg);
                    pk[2 * k] = pk[2 * k + 1] = make_uint4(0u, 0u, 0u, 0u);
                    if (valid && o_base + c0 < n_out) {
#pragma unroll
                        for (int h8 = 0; h8 < 16; h8 += 8) {
                            // bias (and, with the LayerNorm fold, the weight row sums) of the 8 value / 8 gate columns
                            // as 16-byte shared-memory loads: scalar loads made this epilogue LSU-bound
                            float ba[8], bg[8], ua[8], ug[8];
                            *reinterpret_cast<float4*>(&ba[0]) = *reinterpret_cast<const float4*>(sbias + c0 + h8);
                            *reinterpret_cast<float4*>(&ba[4]) = *reinterpret_cast<const float4*>(sbias + c0 + h8 + 4);
                            *reinterpret_cast<float4*>(&bg[0]) = *reinterpret_cast<const float4*>(sbias + HALF + c0 + h8);
                            *reinterpret_cast<float4*>(&bg[4]) = *reinterpret_cast<const float4*>(sbias + HALF + c0 + h8 + 4);
                            if (ln) {
                                *reinterpret_cast<float4*>(&ua[0]) = *reinterpret_cast<const float4*>(su + c0 + h8);
                                *reinterpret_cast<float4*>(&ua[4]) = *reinterpret_cast<const float4*>(su + c0 + h8 + 4);
                                *reinterpret_cast<float4*>(&ug[0]) = *reinterpret_cast<const float4*>(su + HALF + c0 + h8);
                                *reinterpret_cast<float4*>(&ug[4]) = *reinterpret_cast<const float4*>(su + HALF + c0 + h8 + 4);
                            }
                            float v[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                float a = __uint_as_float(ra[h8 + j]), g = __uint_as_float(rg[h8 + j]);
                                if (ln) {
                                    a = fmaf(a, ln_rs, fmaf(ln_nm, ua[j], ba[j]));
                                    g = fmaf(g, ln_rs, fmaf(ln_nm, ug[j], bg[j]));
                                } else {
                                    a += ba[j];
                                    g += bg[j];
                                }
                                v[j] = a * gelu_tanh_f(g);
                            }
                            uint4 q;
                            q.x = pack_bf16x2(v[0], v[1]);
                            q.y = pack_bf16x2(v[2], v[3]);
                            q.z = pack_bf16x2(v[4], v[5]);
                            q.w = pack_bf16x2(v[6], v[7]);
                            pk[2 * k + h8 / 8] = q;
                        }
                    }
                }
            } else if constexpr (MODE == 0 || MODE == 3 || MODE == 4 || MODE == 5) {
                // lean path: per-row base pointers, 32-bit column offsets, uniform flags hoisted.
                // The epilogue runs with only two warps per scheduler, so it is latency-bound unless
                // the four 8-column groups of a chunk are independent straight-line code: the common
                // case (tile fully inside the matrix, all 32 rows of the warp valid) has no per-group
                // branches at all, and launches without residual / row-vector terms skip those adds.
                if (etid == 0) GT(lt, 18);
                const float alpha = effective_alpha(p);
                const bool has_r1 = p.res1 != nullptr, has_r2 = p.res2 != nullptr, has_rv = p.rowvec != nullptr;
                const int act = p.act;
                const __nv_bfloat16* r1row = p.res1 + row * p.ldr1 + n_base;
                const __nv_bfloat16* r2row = p.res2 + row * p.ldr2 + n_base;
                const float* rvrow = p.rowvec + (int64_t)grp * p.rowvec_ld + n_base;
                const int ncols = min(BLOCK_N, p.N - n_base);  // multiple of 8
                const bool full = ncols == BLOCK_N && __all_sync(0xffffffffu, valid);
                const bool plain = !has_r1 && !has_r2 && !has_rv;
                if (etid == 0) GT(lt, 14);  // tile set-up done, about to run the main loop
                mainloop(m_tile, n_tile);
                if (etid == 0) GT(lt, 5);  // accumulator tile ready (epilogue thread 0)
                // column split between the two warps sharing 32 rows: alternating 32-column chunks, except for the
                // 160-wide tile (5 chunks would split 3 / 2): there each warp takes one contiguous 80-column half
                // as 32 + 32 + 16, so both finish together
                constexpr bool kSplitHalves = BLOCK_N == 160;
                constexpr int NCH = kSplitHalves ? 3 : BLOCK_N / 64;  // chunks per thread (160: 32 + 32 + 16 columns)
                auto chunk_col = [&](int k) { return kSplitHalves ? half * 80 + 32 * k : half * 32 + 64 * k; };
                uint32_t accA[32], accB[32];
                acc_ld(arow + chunk_col(0), accA);
                // per-row partial sums for the consumer's LayerNorm (this warp's columns of the row): shifted by the
                // first value seen so a large common offset does not cancel in the variance
                constexpr bool want_rows = MODE == 3;  // mode 3 is only selected with row_stats set
                // (packed fp32x2 arithmetic: three instructions per column pair)
                uint64_t st_s1 = 0ull, st_s2 = 0ull;  // {even, odd} column lanes of sum and sum of squares
                float st_shift = 0.f, st_cnt = 0.f;
                // ---- store helper: 8 fp32 -> (silu) -> bf16 -> 16-byte store
                auto store8 = [&](float (&v)[8], uint4& dst) {
                    if (want_rows) {
                        if (st_cnt == 0.f) st_shift = v[0];
                        const uint64_t sh2 = pack_f32x2(st_shift, st_shift);
#pragma unroll
                        for (int j = 0; j < 8; j += 2) {
                            const uint64_t d = sub_f32x2(pack_f32x2(v[j], v[j + 1]), sh2);
                            st_s1 = add_f32x2(st_s1, d);
                            st_s2 = fma_f32x2(d, d, st_s2);
                        }
                        st_cnt += 8.f;
                    }
                    if (act == PP_ACT_SILU) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] = silu_f(v[j]);
                    } else if (act == PP_ACT_QUICK_GELU) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] = quick_gelu_f(v[j]);
                    }
                    uint4 q;
                    if (MODE == 5 && ttile && p.t_fp16) {  // V^T is fp16 (P is fp16 in the attention kernel)
                        q.x = pack_f16x2(v[0], v[1]);
                        q.y = pack_f16x2(v[2], v[3]);
                        q.z = pack_f16x2(v[4], v[5]);
                        q.w = pack_f16x2(v[6], v[7]);
                    } else {
                        q.x = pack_bf16x2(v[0], v[1]);
                        q.y = pack_bf16x2(v[2], v[3]);
                        q.z = pack_bf16x2(v[4], v[5]);
                        q.w = pack_bf16x2(v[6], v[7]);
                    }
                    dst = q;
                };
                // ---- one chunk of NG 8-column groups (32 or 16 columns); results go to pk[PKB + g]
                auto process = [&](const uint32_t* accv, auto ng_tag, int c0, auto pkb_tag) {
                    constexpr int NG = decltype(ng_tag)::value;
                    constexpr int PKB = decltype(pkb_tag)::value;
                    if (MODE == 4 || (MODE == 5 && ln)) {
                        // LayerNorm-folded consumer (q|k, cross-attention q): acc' = rstd * (acc - mean * u[n]) + bias
                        // fused as two FMAs; these launches carry no residual / row vector
#pragma unroll
                        for (int g = 0; g < NG; ++g) {
                            const int col = c0 + g * 8;
                            pk[PKB + g] = make_uint4(0u, 0u, 0u, 0u);
                            if (valid && col < ncols) {
                                const float4 b0 = *reinterpret_cast<const float4*>(sbias + col);
                                const float4 b1 = *reinterpret_cast<const float4*>(sbias + col + 4);
                                const float4 u0 = *reinterpret_cast<const float4*>(su + col);
                                const float4 u1 = *reinterpret_cast<const float4*>(su + col + 4);
                                float v[8];  // alpha == 1 for LayerNorm-folded launches (checked at prepare time)
                                v[0] = fmaf(__uint_as_float(accv[g * 8 + 0]), ln_rs, fmaf(ln_nm, u0.x, b0.x));
                                v[1] = fmaf(__uint_as_float(accv[g * 8 + 1]), ln_rs, fmaf(ln_nm, u0.y, b0.y));
                                v[2] = fmaf(__uint_as_float(accv[g * 8 + 2]), ln_rs, fmaf(ln_nm, u0.z, b0.z));
                                v[3] = fmaf(__uint_as_float(accv[g * 8 + 3]), ln_rs, fmaf(ln_nm, u0.w, b0.w));
                                v[4] = fmaf(__uint_as_float(accv[g * 8 + 4]), ln_rs, fmaf(ln_nm, u1.x, b1.x));
                                v[5] = fmaf(__uint_as_float(accv[g * 8 + 5]), ln_rs, fmaf(ln_nm, u1.y, b1.y));
                                v[6] = fmaf(__uint_as_float(accv[g * 8 + 6]), ln_rs, fmaf(ln_nm, u1.z, b1.z));
                                v[7] = fmaf(__uint_as_float(accv[g * 8 + 7]), ln_rs, fmaf(ln_nm, u1.w, b1.w));
                                store8(v, pk[PKB + g]);
                            }
                        }
                        return;
                    }
                    if constexpr (MODE != 4) {
                    if (full && plain) {
#pragma unroll
                        for (int g = 0; g < NG; ++g) {
                            const int col = c0 + g * 8;
                            const float4 b0 = *reinterpret_cast<const float4*>(sbias + col);
                            const float4 b1 = *reinterpret_cast<const float4*>(sbias + col + 4);
                            float v[8];
                            v[0] = (__uint_as_float(accv[g * 8 + 0]) + b0.x) * alpha; v[1] = (__uint_as_float(accv[g * 8 + 1]) + b0.y) * alpha;
                            v[2] = (__uint_as_float(accv[g * 8 + 2]) + b0.z) * alpha; v[3] = (__uint_as_float(accv[g * 8 + 3]) + b0.w) * alpha;
                            v[4] = (__uint_as_float(accv[g * 8 + 4]) + b1.x) * alpha; v[5] = (__uint_as_float(accv[g * 8 + 5]) + b1.y) * alpha;
                            v[6] = (__uint_as_float(accv[g * 8 + 6]) + b1.z) * alpha; v[7] = (__uint_as_float(accv[g * 8 + 7]) + b1.w) * alpha;
                            store8(v, pk[PKB + g]);
                        }
                        return;
                    }
                    // general: residuals / row vector / ragged tile. All loads of the chunk are issued
                    // before any arithmetic so their latencies overlap.
                    uint4 q1[NG], q2[NG];
                    float4 t0[NG], t1[NG];
                    bool ok[NG];
#pragma unroll
                    for (int g = 0; g < NG; ++g) {
                        const int col = c0 + g * 8;
                        ok[g] = valid && col < ncols;
                        q1[g] = (ok[g] && has_r1) ? __ldg(reinterpret_cast<const uint4*>(r1row + col)) : make_uint4(0, 0, 0, 0);
                        q2[g] = (ok[g] && has_r2) ? __ldg(reinterpret_cast<const uint4*>(r2row + col)) : make_uint4(0, 0, 0, 0);
                        t0[g] = (ok[g] && has_rv) ? __ldg(reinterpret_cast<const float4*>(rvrow + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
                        t1[g] = (ok[g] && has_rv) ? __ldg(reinterpret_cast<const float4*>(rvrow + col + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int g = 0; g < NG; ++g) {
                        const int col = c0 + g * 8;
                        pk[PKB + g] = make_uint4(0u, 0u, 0u, 0u);
                        if (ok[g]) {
                            const float4 b0 = *reinterpret_cast<const float4*>(sbias + col);
                            const float4 b1 = *reinterpret_cast<const float4*>(sbias + col + 4);
                            float v[8];
                            v[0] = __uint_as_float(accv[g * 8 + 0]) + b0.x + t0[g].x; v[1] = __uint_as_float(accv[g * 8 + 1]) + b0.y + t0[g].y;
                            v[2] = __uint_as_float(accv[g * 8 + 2]) + b0.z + t0[g].z; v[3] = __uint_as_float(accv[g * 8 + 3]) + b0.w + t0[g].w;
                            v[4] = __uint_as_float(accv[g * 8 + 4]) + b1.x + t1[g].x; v[5] = __uint_as_float(accv[g * 8 + 5]) + b1.y + t1[g].y;
                            v[6] = __uint_as_float(accv[g * 8 + 6]) + b1.z + t1[g].z; v[7] = __uint_as_float(accv[g * 8 + 7]) + b1.w + t1[g].w;
                            v[0] = (v[0] + bf16_lo(q1[g].x)) * alpha + bf16_lo(q2[g].x); v[1] = (v[1] + bf16_hi(q1[g].x)) * alpha + bf16_hi(q2[g].x);
                            v[2] = (v[2] + bf16_lo(q1[g].y)) * alpha + bf16_lo(q2[g].y); v[3] = (v[3] + bf16_hi(q1[g].y)) * alpha + bf16_hi(q2[g].y);
                            v[4] = (v[4] + bf16_lo(q1[g].z)) * alpha + bf16_lo(q2[g].z); v[5] = (v[5] + bf16_hi(q1[g].z)) * alpha + bf16_hi(q2[g].z);
                            v[6] = (v[6] + bf16_lo(q1[g].w)) * alpha + bf16_lo(q2[g].w); v[7] = (v[7] + bf16_hi(q1[g].w)) * alpha + bf16_hi(q2[g].w);
                            store8(v, pk[PKB + g]);
                        }
                    }
                    }
                };
                using G4 = std::integral_constant<int, 4>;
                using G2 = std::integral_constant<int, 2>;
                // software pipeline over the chunks: the shared-memory load of chunk k + 1 is issued before chunk k is
                // processed
                auto chunk = [&](auto k_tag, uint32_t (&cur)[32], uint32_t (&nxt)[32]) {
                    constexpr int K = decltype(k_tag)::value;
                    if constexpr (K < NCH) {
                        if constexpr (K + 1 < NCH) {
                            if constexpr (kSplitHalves && K + 1 == 2) acc_ld(arow + chunk_col(K + 1), reinterpret_cast<uint32_t(&)[16]>(nxt));
                            else acc_ld(arow + chunk_col(K + 1), nxt);
                        }
                        if constexpr (kSplitK) {
                            // split-K: the donor's raw fp32 accumulators go to the workspace ([tile][row][BLOCK_N]); the
                            // owner adds the donor's to its own (owner + donor, always in this order) before the epilogue
                            constexpr int NQ = (kSplitHalves && K == 2) ? 4 : 8;  // float4 pieces of this chunk
                            float4* wsp = reinterpret_cast<float4*>(
                                p.splitk_ws + (((int64_t)m_tile * n_tiles + n_tile) * BLOCK_M + r) * BLOCK_N + chunk_col(K));
                            if (khalf) {
#pragma unroll
                                for (int q = 0; q < NQ; ++q)
                                    wsp[q] = make_float4(__uint_as_float(cur[4 * q]), __uint_as_float(cur[4 * q + 1]),
                                                         __uint_as_float(cur[4 * q + 2]), __uint_as_float(cur[4 * q + 3]));
                                return;
                            }
#pragma unroll
                            for (int q = 0; q < NQ; ++q) {
                                const float4 pp = __ldcg(wsp + q);
                                cur[4 * q] = __float_as_uint(__uint_as_float(cur[4 * q]) + pp.x);
                                cur[4 * q + 1] = __float_as_uint(__uint_as_float(cur[4 * q + 1]) + pp.y);
                                cur[4 * q + 2] = __float_as_uint(__uint_as_float(cur[4 * q + 2]) + pp.z);
                                cur[4 * q + 3] = __float_as_uint(__uint_as_float(cur[4 * q + 3]) + pp.w);
                            }
                        }
#ifndef GEMM_EXP_NOEPI  // experiment: drain the accumulator only (what does the tile cost without the epilogue math?)
                        if constexpr (kSplitHalves && K == 2) process(cur, G2{}, chunk_col(K), std::integral_constant<int, 4 * K>{});
                        else process(cur, G4{}, chunk_col(K), std::integral_constant<int, 4 * K>{});
#endif
                    }
                };
                chunk(std::integral_constant<int, 0>{}, accA, accB);
                chunk(std::integral_constant<int, 1>{}, accB, accA);
                chunk(std::integral_constant<int, 2>{}, accA, accB);
                chunk(std::integral_constant<int, 3>{}, accB, accA);
                if constexpr (want_rows) {
                    if (valid)
                        p.row_stats[(int64_t)(n_tile * 2 + half) * p.row_stats_ld + row] =
                            make_float4(f32x2_lo(st_s1) + f32x2_hi(st_s1), f32x2_lo(st_s2) + f32x2_hi(st_s2), st_shift, st_cnt);
                }
            } else {
                // residuals of a 32-column chunk are fetched one chunk ahead (the first chunk's
                // before the main loop), so their latency hides behind the accumulator reads and
                // the previous chunk's stores
                const float alpha1 = effective_alpha(p);
                uint4 c1[4], c2[4], x1[4], x2[4];
                auto fetch = [&](int c0, uint4 (&a)[4], uint4 (&b)[4]) {
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const int n0 = n_base + c0 + g * 8;
                        const bool ok = valid && vec_ok && c0 < BLOCK_N && n0 + 8 <= p.N;
                        a[g] = (ok && p.res1) ? __ldg(reinterpret_cast<const uint4*>(p.res1 + row * p.ldr1 + n0))
                                              : make_uint4(0, 0, 0, 0);
                        b[g] = (ok && p.res2) ? __ldg(reinterpret_cast<const uint4*>(p.res2 + row * p.ldr2 + n0))
                                              : make_uint4(0, 0, 0, 0);
                    }
                };
                fetch(half * 32, c1, c2);
                mainloop(m_tile, n_tile);
#pragma unroll 1
                for (int c0 = half * 32; c0 < BLOCK_N; c0 += 64) {
                    fetch(c0 + 64, x1, x2);
                    uint32_t accv[32];
                    acc_ld(arow + c0, accv);
                    if (valid) {
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            const int n0 = n_base + c0 + g * 8;
                            if (n0 < p.N) {
                                float v[8];
#pragma unroll
                                for (int j = 0; j < 8; ++j) v[j] = __uint_as_float(accv[g * 8 + j]);
                                if (ln) {
#pragma unroll
                                    for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], ln_rs, ln_nm * su[c0 + g * 8 + j]);
                                }
                                if (vec_ok && n0 + 8 <= p.N)
                                    epilogue_store8<true>(p, alpha1, v, row, grp, n0, sbias + c0 + g * 8, c1[g], c2[g]);
                                else
                                    epilogue_store8<false>(p, alpha1, v, row, grp, n0, sbias + c0 + g * 8, c1[g], c2[g]);
                            }
                        }
                    }
#pragma unroll
                    for (int g = 0; g < 4; ++g) { c1[g] = x1[g]; c2[g] = x2[g]; }
                }
            }
            // this thread's reads of the accumulator tile are complete: warpgroup 1 may take it over
            if (etid == 0) GT(lt, 6);  // tile math done (results in registers)
            if constexpr (kAccShared) {
                if (wg == 0) asm volatile("bar.arrive 2, %0;" ::"n"(GEMM_EPI_WARPS * 32) : "memory");
            }
            // the next tile's bias has landed in the other staging buffer (asynchronous copies issued at the top of this
            // tile); the barrier below publishes it before tile lt + 1 reads it
            cp_async_wait_all();
            if constexpr (kSplitK) {
                if (khalf) {
                    // donor: the partial tile is in the workspace; publish it and leave (no output of its own)
                    __threadfence();
                    epi_sync();
                    if (etid == 0) {
                        __threadfence();
                        *(volatile int32_t*)(p.splitk_flags + (int64_t)m_tile * n_tiles + n_tile) = 1;
                    }
                    continue;
                }
            }
            if constexpr (MODE == 3) {
                if (etid == 0 && lt > 0) s_last_tile = ticket_verdict((int)lt);  // of tile lt - 1 (request number lt)
            }
            epi_sync();
            if (etid == 0) GT(lt, 11);  // first barrier passed
            // mode 3: the previous tile was the last n-tile of its row block -> fold the block's records (first four loads
            // now, the arithmetic after the hand-over to the TMA unit); then post this tile's ticket request
            float4 frc[4];
            bool fold_prev = false;
            if constexpr (MODE == 3) {
                fold_prev = lt > 0 && s_last_tile != 0 && half == 0 && prev_valid;
                if (fold_prev) {
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        frc[u] = u < 2 * n_tiles ? __ldcg(p.row_stats + (int64_t)u * p.row_stats_ld + prev_row)
                                                 : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                if (etid == 0) {
                    s_req_mtile = m_tile;
                    __threadfence_block();
                    s_req_seq = (int)lt + 1;
                }
            }
            if constexpr (MODE != 1) {
                // stage the tile (generic-proxy writes -> async proxy), one barrier, one thread issues the TMA stores
                // (one per sub-tile); the unit writes whole rows and clips out-of-range parts
#pragma unroll
                for (int i = 0; i < PK_N; ++i) {
                    int col;
                    if constexpr (MODE == 2) col = half * 16 + 32 * (i / 2) + 8 * (i % 2);
                    else if constexpr (BLOCK_N == 160) col = half * 80 + 8 * i;
                    else col = half * 32 + 64 * (i / 4) + 8 * (i % 4);
                    if (MODE == 5 && ttile) {
                        // transposed staging: [column][128 rows] 16-bit, 64-column sub-tiles of 16 KB — the boxes of the
                        // transposed TMA store; a warp's 32 lanes write 64 contiguous bytes per column (conflict-free)
                        uint8_t* tb = s_out + (col >> 6) * 16384 + (col & 63) * 256 + r * 2;
                        const uint32_t w[4] = {pk[i].x, pk[i].y, pk[i].z, pk[i].w};
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            *reinterpret_cast<uint16_t*>(tb + (2 * j) * 256) = (uint16_t)(w[j] & 0xFFFFu);
                            *reinterpret_cast<uint16_t*>(tb + (2 * j + 1) * 256) = (uint16_t)(w[j] >> 16);
                        }
                    } else {
                        *reinterpret_cast<uint4*>(stage_ptr(r, col)) = pk[i];
                    }
                }
                if (etid == 0) GT(lt, 12);  // staging stores issued
                fence_proxy_async_smem();
                if (etid == 0) GT(lt, 13);  // proxy fence done
                if (half == 0) s_row[r] = valid ? (long long)row : -1ll;
                epi_sync();
                if (etid == 0) GT(lt, 7);  // all epilogue warps staged
                constexpr int OUT_COLS = MODE == 2 ? BLOCK_N / 2 : BLOCK_N;
                constexpr int PIECES = OUT_COLS / 8;
                // one thread per 64-column sub-tile (lane 0 of the first warps) issues its store: a single thread issuing
                // three stores back to back took ~600 cycles of the epilogue's serial path
                if ((etid & 31) == 0 && (etid >> 5) * 64 < (MODE == 5 ? BLOCK_N : OUT_COLS)) {
                    const int sub = etid >> 5;
                    const int out_base = n_tile * OUT_COLS;
                    const int n_out = MODE == 2 ? p.N / 2 : MODE == 5 ? p.trans_first_tile * BLOCK_N : p.N;
                    if (MODE == 5 && ttile) {
                        // (token, channel, sample) coordinates of the transposed destination; tiles never straddle samples
                        const int row0 = m_tile * BLOCK_M;
                        const int sb = row0 / p.t_rows, t0 = row0 - sb * p.t_rows;
                        const int cbase = (n_tile - p.trans_first_tile) * BLOCK_N;
                        if (n_base + sub * 64 < p.N) {
                            const CUtensorMap* tm = (BLOCK_N - sub * 64) >= 64 ? &p.tmOutT[0] : &p.tmOutT[1];
#ifndef GEMM_EXP_NOSTORE
                            tma_store_3d(tm, s_out_addr + sub * 16384, t0, cbase + sub * 64, sb);
#endif
                        }
                    } else {
                        const int col = out_base + sub * 64;
                        if (col < n_out) {
                            const CUtensorMap* tm = (OUT_COLS - sub * 64) >= 64 ? &p.tmOut[0] : &p.tmOut[1];
#ifndef GEMM_EXP_NOSTORE  // experiment: no global write of the tile
                            if (p.a_mode == PP_A_MATRIX) {
                                tma_store_2d(tm, s_out_addr + sub * 16384, col, m_tile * BLOCK_M);
                            } else {
                                int x0, y0, nb0;
                                tile_origin(m_tile, x0, y0, nb0);
                                tma_store_4d(tm, s_out_addr + sub * 16384, col, x0, y0, nb0);
                            }
#endif
                        }
                    }
                    bulk_commit_group();
                    if (etid == 0) GT(lt, 8);  // TMA stores issued
                }
                if constexpr (MODE == 3) {
                    if (fold_prev) fold_row_records(frc, prev_row);
                    prev_row = row;
                    prev_valid = valid;
                }
                if constexpr (MODE == 0 || MODE == 3 || MODE == 4) {  // (never mode 5: transposed tiles hold no rows)
                    // GroupNorm partial sums of exactly the bf16 values the consumer will read
                    if (p.chan_stats) {
                        constexpr int L = (BLOCK_N <= 128) ? 16 : 8;
                        if (etid < PIECES * L) {  // warp-uniform: PIECES * L is a multiple of 32
                            const int piece = etid / L, l = etid % L;
                            const int col0 = n_base + piece * 8;
                            const int seg_rows = 1 << p.stat_seg_rows_log2;
                            for (int sg = 0; sg < p.stat_segs; ++sg) {
                                float v[16];
#pragma unroll
                                for (int j = 0; j < 16; ++j) v[j] = 0.f;
                                const int rb = sg << p.stat_seg_rows_log2;
                                // the segment's first row is its shift (valid whenever the segment holds any row:
                                // it is the pixel-box origin of the sample / the sample's first row of the tile)
                                float sh[8];
                                {
                                    const uint4 q = *reinterpret_cast<const uint4*>(stage_ptr(rb, piece * 8));
                                    const bool okr = s_row[rb] >= 0;
                                    sh[0] = okr ? bf16_lo(q.x) : 0.f; sh[1] = okr ? bf16_hi(q.x) : 0.f;
                                    sh[2] = okr ? bf16_lo(q.y) : 0.f; sh[3] = okr ? bf16_hi(q.y) : 0.f;
                                    sh[4] = okr ? bf16_lo(q.z) : 0.f; sh[5] = okr ? bf16_hi(q.z) : 0.f;
                                    sh[6] = okr ? bf16_lo(q.w) : 0.f; sh[7] = okr ? bf16_hi(q.w) : 0.f;
                                }
                                for (int rr = rb + l; rr < rb + seg_rows; rr += L) {
                                    if (s_row[rr] >= 0) {
                                        const uint4 q = *reinterpret_cast<const uint4*>(stage_ptr(rr, piece * 8));
                                        const float x[8] = {bf16_lo(q.x), bf16_hi(q.x), bf16_lo(q.y), bf16_hi(q.y),
                                                            bf16_lo(q.z), bf16_hi(q.z), bf16_lo(q.w), bf16_hi(q.w)};
#pragma unroll
                                        for (int j = 0; j < 8; ++j) {
                                            const float dlt = x[j] - sh[j];
                                            v[2 * j] += dlt;
                                            v[2 * j + 1] = fmaf(dlt, dlt, v[2 * j + 1]);
                                        }
                                    }
                                }
                                float* dst = p.chan_stats +
                                             (((int64_t)m_tile * p.stat_segs + sg) * p.N + col0) * 4;
                                stats_butterfly_store<L>(v, sh, l, dst, col0 < p.N);
                            }
                        }
                    }
                }
            }
            if (etid == 0) GT(lt, 10);
        }
        if constexpr (MODE == 3) {
            // the last tile's verdict and fold, then release the ticket server
            if (etid == 0 && lt > 0) s_last_tile = ticket_verdict((int)lt);
            epi_sync();
            if (lt > 0 && s_last_tile != 0 && half == 0 && prev_valid) {
                float4 frc[4];
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    frc[u] = u < 2 * n_tiles ? __ldcg(p.row_stats + (int64_t)u * p.row_stats_ld + prev_row)
                                             : make_float4(0.f, 0.f, 0.f, 0.f);
                fold_row_records(frc, prev_row);
            }
            if (etid == 0) {
                s_req_mtile = -1;
                __threadfence_block();
                s_req_seq = (int)lt + 1;
            }
        }
        if constexpr (MODE != 1) {
            if ((etid & 31) == 0) bulk_wait_all();  // global writes of the last tile performed before the CTA retires
        }
    }

}

// ---------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int pad64(int c) { return ceil_div(c, 64) * 64; }

static size_t smem_for_block_n(int bn) { return (size_t)smem_bytes_for(bn); }

static int num_sms() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;  // H100 SXM (host-only queries without a device)
    }
    return n;
}

template <int BLOCK_N, int MODE>
static int launch_variant(const GemmLaunch& l, cudaStream_t s) {
    PP_CUDA_CHECK(launch(gemm_conv_kernel<BLOCK_N, MODE>, l.grid, GEMM_THREADS, l.smem, s, l.p));
    return PP_OK;
}
// split-K flavour (mode 0 only)
template <int BLOCK_N>
static int launch_splitk(const GemmLaunch& l, cudaStream_t s) {
    PP_CUDA_CHECK(launch(gemm_conv_kernel<BLOCK_N, 0, true>, l.grid, GEMM_THREADS, l.smem, s, l.p));
    return PP_OK;
}
template <int BLOCK_N>
static int ensure_attr_splitk() {
    static bool done[PP_MAX_DEVICES] = {};
    int dev = 0;
    PP_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev < 0 || dev >= PP_MAX_DEVICES || !done[dev]) {
        PP_CUDA_CHECK(cudaFuncSetAttribute(gemm_conv_kernel<BLOCK_N, 0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem_for_block_n(BLOCK_N)));
        if (dev >= 0 && dev < PP_MAX_DEVICES) done[dev] = true;
    }
    return PP_OK;
}

// opt the kernel variant into its dynamic shared memory size (done at prepare time so that
// launches are pure and can be stream-captured)
template <int BLOCK_N, int MODE>
static int ensure_attr() {
    // the attribute is per device: one flag per device ordinal
    static bool done[PP_MAX_DEVICES] = {};
    int dev = 0;
    PP_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev < 0 || dev >= PP_MAX_DEVICES || !done[dev]) {
        PP_CUDA_CHECK(cudaFuncSetAttribute(gemm_conv_kernel<BLOCK_N, MODE>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem_for_block_n(BLOCK_N)));
        if (dev >= 0 && dev < PP_MAX_DEVICES) done[dev] = true;
    }
    return PP_OK;
}

#define PP_GEMM_DISPATCH(FN, bn, mode, ...)                                      \
    switch ((bn) * 8 + (mode)) {                                                 \
        case 64 * 8 + 0: return FN<64, 0>(__VA_ARGS__);                          \
        case 64 * 8 + 1: return FN<64, 1>(__VA_ARGS__);                          \
        case 64 * 8 + 3: return FN<64, 3>(__VA_ARGS__);                          \
        case 128 * 8 + 3: return FN<128, 3>(__VA_ARGS__);                        \
        case 160 * 8 + 3: return FN<160, 3>(__VA_ARGS__);                        \
        case 256 * 8 + 3: return FN<256, 3>(__VA_ARGS__);                        \
        case 64 * 8 + 4: return FN<64, 4>(__VA_ARGS__);                          \
        case 64 * 8 + 5: return FN<64, 5>(__VA_ARGS__);                          \
        case 128 * 8 + 5: return FN<128, 5>(__VA_ARGS__);                        \
        case 160 * 8 + 5: return FN<160, 5>(__VA_ARGS__);                        \
        case 256 * 8 + 5: return FN<256, 5>(__VA_ARGS__);                        \
        case 128 * 8 + 4: return FN<128, 4>(__VA_ARGS__);                        \
        case 160 * 8 + 4: return FN<160, 4>(__VA_ARGS__);                        \
        case 256 * 8 + 4: return FN<256, 4>(__VA_ARGS__);                        \
        case 128 * 8 + 0: return FN<128, 0>(__VA_ARGS__);                        \
        case 128 * 8 + 1: return FN<128, 1>(__VA_ARGS__);                        \
        case 128 * 8 + 2: return FN<128, 2>(__VA_ARGS__);                        \
        case 160 * 8 + 0: return FN<160, 0>(__VA_ARGS__);                        \
        case 160 * 8 + 1: return FN<160, 1>(__VA_ARGS__);                        \
        case 256 * 8 + 0: return FN<256, 0>(__VA_ARGS__);                        \
        case 256 * 8 + 1: return FN<256, 1>(__VA_ARGS__);                        \
        case 256 * 8 + 2: return FN<256, 2>(__VA_ARGS__);                        \
    }

static int ensure_attr_for(int block_n, int mode) {
    PP_GEMM_DISPATCH(ensure_attr, block_n, mode)
    return PP_ERR_INVALID;
}

int gemm_launch(const GemmLaunch& l, cudaStream_t s) {
    if (l.p.ksplit == 2) {
        switch (l.block_n) {
            case 128: return launch_splitk<128>(l, s);
            case 160: return launch_splitk<160>(l, s);
            case 256: return launch_splitk<256>(l, s);
        }
        set_last_error("gemm_launch: no split-K variant for block_n %d", l.block_n);
        return PP_ERR_INVALID;
    }
    PP_GEMM_DISPATCH(launch_variant, l.block_n, l.mode, l, s)
    set_last_error("gemm_launch: unsupported block_n %d / mode %d", l.block_n, l.mode);
    return PP_ERR_INVALID;
}

// Tile width: minimise (rounds over the SMs) x (per-tile cost ~ width + fixed overhead), where
// padding beyond N is paid as well; ties go to the wider tile (fewer A re-reads).
static int pick_block_n(int N, int m_tiles, bool geglu) {
    const int cands[4] = {256, 160, 128, 64};
    const int sms = num_sms();
    int best = 0;
    double best_cost = 1e30;
    for (int c : cands) {
        if (geglu && (c == 64 || c == 160 || N % c != 0)) continue;  // 160: 80 output columns are no TMA-store box
        const int nt = ceil_div(N, c);
        const long tiles = (long)m_tiles * nt;
        const long rounds = (tiles + sms - 1) / sms;
        const double cost = (double)rounds * (c + 24);
        if (cost < best_cost - 1e-9) {
            best_cost = cost;
            best = c;
        }
    }
    return best ? best : 128;
}

// Tile geometry of a launch (everything that needs no device or driver): validation of the shape
// fields, the conv pixel box, the tile width and the walk. Shared by gemm_prepare and the host-only
// statistics-geometry query.
static bool gemm_fast_mode(const pp_gemm_desc& d);
// transposed columns through the staging tile + TMA store (mode 5): whole 128-row tiles inside one sample, bias only
static bool gemm_trans_staged(const pp_gemm_desc& d) {
    const bool t = d.epilogue == PP_EPI_TRANSPOSED || d.epilogue == PP_EPI_ROWS_THEN_TRANSPOSED;
    return t && d.a_mode == PP_A_MATRIX && !d.out_fp32 && d.N % 8 == 0 && d.t_rows > 0 && d.t_rows % BLOCK_M == 0 &&
           d.M % d.t_rows == 0 && d.t_ld % 8 == 0 && !d.a1 && !d.rowvec && !d.res1 && !d.res2 && d.act == PP_ACT_NONE &&
           d.alpha == 1.0f && !d.alpha_dev && !d.chan_stats && !d.row_stats;
}

// split-K x2 is considered for contractions at least this long (36 k-iterations: a 3x3 conv over 256 channels)
static constexpr int SPLITK_MIN_K_ITERS = 36;

static int gemm_geometry(const pp_gemm_desc& d, GemmKParams& p, int* block_n_out, int* ksplit_out = nullptr) {
    PP_REQUIRE(d.a_mode >= PP_A_MATRIX && d.a_mode <= PP_A_CONV3X3_S2P0, "gemm: bad a_mode %d", d.a_mode);
    PP_REQUIRE(d.epilogue >= PP_EPI_PLAIN && d.epilogue <= PP_EPI_ROWS_THEN_TRANSPOSED, "gemm: bad epilogue %d", d.epilogue);
    PP_REQUIRE(d.a0 && d.b && d.out, "gemm: null operand pointer");
    PP_REQUIRE(d.c0 > 0 && d.c0 % 8 == 0, "gemm: c0=%d must be a positive multiple of 8", d.c0);
    PP_REQUIRE((d.a1 == nullptr) == (d.c1 == 0), "gemm: a1/c1 mismatch");
    PP_REQUIRE(d.c1 % 8 == 0, "gemm: c1=%d must be a multiple of 8", d.c1);
    PP_REQUIRE(d.N > 0, "gemm: N must be positive");
    PP_REQUIRE(d.act >= PP_ACT_NONE && d.act <= PP_ACT_QUICK_GELU, "gemm: bad act %d", d.act);
    const int taps = d.a_mode == PP_A_MATRIX ? 1 : 9;
    p.a_mode = d.a_mode;
    p.chunks0 = ceil_div(d.c0, 64);
    p.chunks1 = d.a1 ? ceil_div(d.c1, 64) : 0;
    p.num_k_iters = taps * (p.chunks0 + p.chunks1);
    int m_tiles;
    if (d.a_mode == PP_A_MATRIX) {
        PP_REQUIRE(d.M > 0, "gemm: M must be positive");
        p.M = d.M;
        m_tiles = ceil_div(d.M, BLOCK_M);
        p.a_bytes = A_STAGE_BYTES;
    } else {
        PP_REQUIRE(d.nb > 0 && d.h > 0 && d.w > 0, "gemm: conv dims must be positive");
        const bool s2 = d.a_mode != PP_A_CONV3X3;
        if (s2) {
            PP_REQUIRE(d.h >= 2 && d.w >= 2, "gemm: stride-2 conv needs h, w >= 2 (got %d x %d)", d.h, d.w);
            PP_REQUIRE(d.a1 == nullptr, "gemm: stride-2 conv takes a single source");
        }
        p.nb = d.nb;
        // pad 1: ceil(h / 2); bottom/right pad (S2P0): floor(h / 2)
        p.ho = d.a_mode == PP_A_CONV3X3_S2 ? (d.h + 1) / 2 : s2 ? d.h / 2 : d.h;
        p.wo = d.a_mode == PP_A_CONV3X3_S2 ? (d.w + 1) / 2 : s2 ? d.w / 2 : d.w;
        p.M = d.nb * p.ho * p.wo;
        // pick the pixel box (bw, bh, bn), bw*bh*bn <= 128, minimising padded volume
        int64_t best_cost = -1;
        for (int bw = 128; bw >= 1; bw >>= 1) {
            for (int bh = 128 / bw; bh >= 1; bh >>= 1) {
                int bn = 128 / (bw * bh);
                int64_t cost = (int64_t)ceil_div(p.wo, bw) * ceil_div(p.ho, bh) * ceil_div(p.nb, bn);
                if (best_cost < 0 || cost < best_cost) {
                    best_cost = cost;
                    p.bw = bw; p.bh = bh; p.bn = bn;
                }
            }
        }
        p.bw_log2 = 0;
        while ((1 << p.bw_log2) < p.bw) ++p.bw_log2;
        p.bh_log2 = 0;
        while ((1 << p.bh_log2) < p.bh) ++p.bh_log2;
        p.tiles_x = ceil_div(p.wo, p.bw);
        p.tiles_y = ceil_div(p.ho, p.bh);
        m_tiles = p.tiles_x * p.tiles_y * ceil_div(p.nb, p.bn);
        p.a_bytes = (uint32_t)(p.bw * p.bh * p.bn) * 128u;
    }
    p.N = d.N;
    const bool geglu = d.epilogue == PP_EPI_GEGLU;
    int bn = d.block_n ? d.block_n : pick_block_n(d.N, m_tiles, geglu);
    // split-K x2 (needs the caller's workspace): plain bf16 launches with a long K whose tiles, doubled, still fit the
    // SMs in one round, when that shortens the per-CTA work of pick_block_n's cost model (half of K per work item)
    int ksplit = 1;
    if (d.splitk_ws && d.splitk_flags && (d.a_mode == PP_A_MATRIX || d.a_mode == PP_A_CONV3X3) && !geglu &&
        gemm_fast_mode(d) && !d.row_stats && !d.ln_stats && p.num_k_iters >= SPLITK_MIN_K_ITERS &&
        p.num_k_iters % 2 == 0) {
        const int sms = num_sms();
        const long plain_tiles = (long)m_tiles * ceil_div(d.N, bn);
        const double plain_cost = (double)((plain_tiles + sms - 1) / sms) * (bn + 24);
        int best = 0;
        double best_cost = plain_cost;
        const int cands[3] = {128, 160, 256};
        for (int c : cands) {
            if (d.block_n && c != d.block_n) continue;
            const long items = 2L * m_tiles * ceil_div(d.N, c);
            const double cost = 0.5 * (c + 24);
            if (items <= sms && cost < best_cost - 1e-9) { best = c; best_cost = cost; }
        }
        if (best) {
            bn = best;
            ksplit = 2;
        }
    }
    PP_REQUIRE(bn == 64 || bn == 128 || bn == 160 || bn == 256, "gemm: block_n %d unsupported", bn);
    if (geglu) {
        PP_REQUIRE(d.N % bn == 0, "gemm: GEGLU needs N %% block_n == 0 (N=%d, block_n=%d)", d.N, bn);
        PP_REQUIRE(bn == 128 || bn == 256, "gemm: GEGLU block_n must be 128 or 256 (got %d)", bn);
    }
    p.m_tiles = m_tiles;
    p.n_tiles = ceil_div(d.N, bn);
    *block_n_out = bn;
    if (ksplit_out) *ksplit_out = ksplit;
    return PP_OK;
}

static bool gemm_fast_mode(const pp_gemm_desc& d) {
    const int64_t rv_ld = d.rowvec_ld ? d.rowvec_ld : d.N;
    return d.epilogue == PP_EPI_PLAIN && !d.out_fp32 && d.N % 8 == 0 &&
           (!d.rowvec || (rv_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d.rowvec) & 15) == 0));
}

int gemm_stats_geometry(const pp_gemm_desc& d, pp_stats_geom* g) {
    memset(g, 0, sizeof(*g));
    GemmKParams p;
    memset(&p, 0, sizeof(p));
    int bn = 0;
    int rc = gemm_geometry(d, p, &bn);
    if (rc) return rc;
    g->channels = d.N;
    if (!gemm_fast_mode(d)) return PP_OK;  // statistics come from the bf16 staging tile of the fast epilogue
    const int min_rows = 16;               // >= the row lanes of the statistics pass
    if (d.a_mode == PP_A_MATRIX) {
        const int hw = d.rows_per_group;
        if (hw <= 0 || d.M % hw != 0) return PP_OK;
        if (hw % BLOCK_M == 0) {
            g->segs = 1; g->seg_rows = BLOCK_M; g->tiles_per_group = hw / BLOCK_M;
        } else if (BLOCK_M % hw == 0 && hw >= min_rows) {
            g->segs = BLOCK_M / hw; g->seg_rows = hw; g->tiles_per_group = 1;
        } else {
            return PP_OK;
        }
        g->tiles_x = g->tiles_per_group; g->tiles_y = 1; g->bw = g->seg_rows; g->bh = 1; g->wo = hw; g->ho = 1;
    } else {
        if (p.bw * p.bh < min_rows) return PP_OK;
        g->segs = p.bn; g->seg_rows = p.bw * p.bh; g->tiles_per_group = p.tiles_x * p.tiles_y;
        g->tiles_x = p.tiles_x; g->tiles_y = p.tiles_y; g->bw = p.bw; g->bh = p.bh; g->wo = p.wo; g->ho = p.ho;
    }
    g->supported = 1;
    g->bytes = (int64_t)p.m_tiles * g->segs * d.N * 4 * (int64_t)sizeof(float);
    return PP_OK;
}

// records per row a GEMM emits for the consumer's LayerNorm: one per half n-tile (the two epilogue warps that share a
// row each own a set of columns); 0 = this launch cannot emit them
int gemm_row_stats_records(const pp_gemm_desc& d0) {
    // the query comes before the record buffer exists: answer for the launch WITH row_stats attached (that one never
    // runs split-K, which can pick a different tile width and hence a different record count)
    pp_gemm_desc d = d0;
    if (!d.row_stats) d.row_stats = reinterpret_cast<float*>(uintptr_t(16));
    GemmKParams p;
    memset(&p, 0, sizeof(p));
    int bn = 0;
    if (gemm_geometry(d, p, &bn)) return 0;
    if (d.a_mode != PP_A_MATRIX || !gemm_fast_mode(d) || d.act != PP_ACT_NONE) return 0;
    return 2 * p.n_tiles;
}

// Epilogue flavour (the MODE template argument) of a launch: 2 GEGLU, 5 transposed columns through the staging tile,
// 3 / 4 / 0 the fast bf16 epilogue (LayerNorm-statistics producer / LayerNorm-folded consumer / plain), 1 the generic
// one. Shared by gemm_prepare and the host-only pp_gemm_variant.
static int gemm_select_mode(const pp_gemm_desc& d) {
    if (d.epilogue == PP_EPI_GEGLU) return 2;
    if (gemm_trans_staged(d)) return 5;
    if (gemm_fast_mode(d)) return d.row_stats ? 3 : d.ln_stats ? 4 : 0;
    return 1;
}

int gemm_variant(const pp_gemm_desc& d, int* block_n, int* mode, int* ksplit) {
    GemmKParams p;
    memset(&p, 0, sizeof(p));
    int bn = 0, ks = 1;
    int rc = gemm_geometry(d, p, &bn, &ks);
    if (rc) return rc;
    *block_n = bn;
    *mode = gemm_select_mode(d);
    *ksplit = ks;
    return PP_OK;
}

int gemm_prepare(const pp_gemm_desc& d, GemmLaunch* out) {
    GemmLaunch l;
    memset(&l, 0, sizeof(l));
    GemmKParams& p = l.p;
    int bn = 0, ksplit = 1;
    {
        int rc = gemm_geometry(d, p, &bn, &ksplit);
        if (rc) return rc;
    }
    const int taps = d.a_mode == PP_A_MATRIX ? 1 : 9;
    const bool packed_k = taps == 9 || d.a1 != nullptr;
    const int64_t kw = packed_k ? (int64_t)taps * (pad64(d.c0) + pad64(d.c1)) : d.c0;
    const int64_t ldb = packed_k ? kw : d.ldb;
    PP_REQUIRE(ldb >= kw && ldb % 8 == 0, "gemm: ldb=%lld invalid for K=%lld", (long long)ldb, (long long)kw);

    if (d.a_mode == PP_A_MATRIX) {
        PP_REQUIRE(d.lda0 >= d.c0 && d.lda0 % 8 == 0, "gemm: lda0=%lld invalid", (long long)d.lda0);
        uint64_t dims[2] = {(uint64_t)d.c0, (uint64_t)d.M};
        uint64_t str[1] = {(uint64_t)d.lda0 * 2};
        uint32_t box[2] = {64, BLOCK_M};
        int rc = make_tmap_bf16(&p.tmA[0], d.a0, 2, dims, str, box, true);
        if (rc) return rc;
        if (d.a1) {
            PP_REQUIRE(d.lda1 >= d.c1 && d.lda1 % 8 == 0, "gemm: lda1=%lld invalid", (long long)d.lda1);
            uint64_t dims1[2] = {(uint64_t)d.c1, (uint64_t)d.M};
            uint64_t str1[1] = {(uint64_t)d.lda1 * 2};
            rc = make_tmap_bf16(&p.tmA[1], d.a1, 2, dims1, str1, box, true);
            if (rc) return rc;
        }
    } else {
        uint32_t box[4] = {64, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
        if (d.a_mode == PP_A_CONV3X3) {
            const void* srcs[2] = {d.a0, d.a1};
            const int cs[2] = {d.c0, d.c1};
            for (int i = 0; i < 2; ++i) {
                if (!srcs[i]) continue;
                uint64_t dims[4] = {(uint64_t)cs[i], (uint64_t)d.w, (uint64_t)d.h, (uint64_t)d.nb};
                uint64_t str[3] = {(uint64_t)cs[i] * 2, (uint64_t)cs[i] * 2 * d.w, (uint64_t)cs[i] * 2 * d.w * d.h};
                int rc = make_tmap_bf16(&p.tmA[i], srcs[i], 4, dims, str, box, true);
                if (rc) return rc;
            }
        } else {
            // parity planes: plane (py, px) holds input rows py, py + 2, ... (ceil((h - py) / 2) of them) and
            // columns px, px + 2, ...; for odd h / w the planes differ in size and the missing last row /
            // column reads as TMA's out-of-bounds zero, which is exactly the conv's padding
            for (int py = 0; py < 2; ++py)
                for (int px = 0; px < 2; ++px) {
                    const __nv_bfloat16* base =
                        reinterpret_cast<const __nv_bfloat16*>(d.a0) + ((int64_t)py * d.w + px) * d.c0;
                    uint64_t dims[4] = {(uint64_t)d.c0, (uint64_t)(d.w + 1 - px) / 2, (uint64_t)(d.h + 1 - py) / 2,
                                        (uint64_t)d.nb};
                    uint64_t str[3] = {(uint64_t)d.c0 * 2 * 2, (uint64_t)d.c0 * 2 * d.w * 2,
                                       (uint64_t)d.c0 * 2 * d.w * d.h};
                    int rc = make_tmap_bf16(&p.tmA[py * 2 + px], base, 4, dims, str, box, true);
                    if (rc) return rc;
                }
        }
    }
    const bool geglu = d.epilogue == PP_EPI_GEGLU;
    if (geglu) {
        PP_REQUIRE(!d.out_fp32 && !d.rowvec && !d.res1 && !d.res2, "gemm: GEGLU epilogue takes bias only");
        PP_REQUIRE(d.ldc % 8 == 0, "gemm: GEGLU ldc must be a multiple of 8");
    }
    l.block_n = bn;
    {
        uint64_t dims[2] = {(uint64_t)kw, (uint64_t)d.N};
        uint64_t str[1] = {(uint64_t)ldb * 2};
        uint32_t box[2] = {64, (uint32_t)bn};
        int rc = make_tmap_bf16(&p.tmB, d.b, 2, dims, str, box, true);
        if (rc) return rc;
    }
    // epilogue
    p.epilogue = d.epilogue;
    p.act = d.act;
    p.out_fp32 = d.out_fp32;
    p.bias = d.bias;
    p.rowvec = d.rowvec;
    p.rows_per_group = d.rows_per_group;
    p.rowvec_ld = d.rowvec_ld ? d.rowvec_ld : d.N;
    if (d.rowvec && d.a_mode == PP_A_MATRIX)
        PP_REQUIRE(d.rows_per_group > 0, "gemm: rowvec needs rows_per_group > 0");
    p.res1 = reinterpret_cast<const __nv_bfloat16*>(d.res1);
    p.ldr1 = d.ldr1;
    p.res2 = reinterpret_cast<const __nv_bfloat16*>(d.res2);
    p.ldr2 = d.ldr2;
    p.alpha = d.alpha;
    p.alpha_dev = d.alpha_dev;
    p.alpha_step = d.alpha_step;
    p.alpha_stride = d.alpha_stride;
    p.out = d.out;
    p.ldc = d.ldc;
    p.t_rows = d.t_rows;
    p.t_ld = d.t_ld;
    p.t_fp16 = d.t_fp16;
    if (d.epilogue == PP_EPI_TRANSPOSED || d.epilogue == PP_EPI_ROWS_THEN_TRANSPOSED) {
        PP_REQUIRE(d.t_rows > 0 && d.t_ld >= d.t_rows, "gemm: transposed store needs t_rows/t_ld");
        PP_REQUIRE(!d.out_fp32, "gemm: transposed store is bf16 only");
    }
    if (d.epilogue != PP_EPI_TRANSPOSED) {
        const int n_rows_part = geglu ? d.N / 2 : d.epilogue == PP_EPI_ROWS_THEN_TRANSPOSED ? d.trans_from_col : d.N;
        PP_REQUIRE(d.ldc >= n_rows_part, "gemm: ldc=%lld too small", (long long)d.ldc);
        if (d.N % 8 == 0) {
            PP_REQUIRE(d.ldc % (d.out_fp32 ? 4 : 8) == 0, "gemm: ldc=%lld breaks 16-byte store alignment", (long long)d.ldc);
            PP_REQUIRE((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "gemm: out pointer not 16-byte aligned");
        }
    }
    if (d.N % 8 == 0) {
        if (d.res1) PP_REQUIRE(d.ldr1 % 8 == 0 && (reinterpret_cast<uintptr_t>(d.res1) & 15) == 0, "gemm: res1 alignment");
        if (d.res2) PP_REQUIRE(d.ldr2 % 8 == 0 && (reinterpret_cast<uintptr_t>(d.res2) & 15) == 0, "gemm: res2 alignment");
        if (d.bias) PP_REQUIRE((reinterpret_cast<uintptr_t>(d.bias) & 15) == 0, "gemm: bias alignment");
    }
    {
        const long tiles = (long)p.m_tiles * p.n_tiles;
        l.grid = dim3((unsigned)std::min<long>(tiles, num_sms()), 1, 1);
        // split-K x2 (decided with the geometry): two CTAs per tile, one work item each
        p.ksplit = ksplit;
        if (ksplit == 2) {
            PP_REQUIRE((reinterpret_cast<uintptr_t>(d.splitk_ws) & 15) == 0, "gemm: splitk_ws not 16-byte aligned");
            p.splitk_ws = d.splitk_ws;
            p.splitk_flags = d.splitk_flags;
            l.grid = dim3((unsigned)(2 * tiles), 1, 1);
        }
    }
    l.smem = smem_for_block_n(bn);
    l.mode = gemm_select_mode(d);
    if (l.mode == 5) {
        const bool mixed = d.epilogue == PP_EPI_ROWS_THEN_TRANSPOSED;
        if (mixed)
            PP_REQUIRE(d.out_t && d.trans_from_col > 0 && d.trans_from_col < d.N && d.trans_from_col % bn == 0 &&
                           (d.N - d.trans_from_col) % 8 == 0,
                       "gemm: trans_from_col=%d must be a positive multiple of the tile width %d below N=%d",
                       d.trans_from_col, bn, d.N);
        p.trans_first_tile = mixed ? d.trans_from_col / bn : 0;
        void* out_t = mixed ? d.out_t : d.out;
        const uint64_t nt = (uint64_t)(d.N - (mixed ? d.trans_from_col : 0));
        PP_REQUIRE((reinterpret_cast<uintptr_t>(out_t) & 15) == 0, "gemm: transposed output not 16-byte aligned");
        for (int k = 0; k < 2; ++k) {
            if (k == 1 && bn % 64 == 0) break;
            uint64_t dims[3] = {(uint64_t)d.t_rows, nt, (uint64_t)(d.M / d.t_rows)};
            uint64_t str[2] = {(uint64_t)d.t_ld * 2, nt * (uint64_t)d.t_ld * 2};
            uint32_t box[3] = {(uint32_t)BLOCK_M, k == 0 ? 64u : 32u, 1u};
            int rc = make_tmap_bf16_sw(&p.tmOutT[k], out_t, 3, dims, str, box, 0);
            if (rc) return rc;
        }
    } else if (l.mode != 2) {
        PP_REQUIRE(d.epilogue != PP_EPI_ROWS_THEN_TRANSPOSED, "gemm: PP_EPI_ROWS_THEN_TRANSPOSED needs a plain bf16 GEMM "
                   "(bias only) whose t_rows is a multiple of 128 and divides M");
        PP_REQUIRE(!(d.row_stats && d.ln_stats), "gemm: a launch either emits LayerNorm statistics or consumes them");
    }
    if (l.mode != 1 && !(l.mode == 5 && p.trans_first_tile == 0)) {
        // TMA-store boxes of the staged output tile: 64 columns (128-byte swizzle), and a 32-column box (64-byte
        // swizzle) for the tail of the 160-wide tile; tensor extents clip ragged tiles and columns >= N
        const uint64_t n_out = geglu ? (uint64_t)d.N / 2 : l.mode == 5 ? (uint64_t)d.trans_from_col : (uint64_t)d.N;
        const int out_cols = geglu ? bn / 2 : bn;
        for (int k = 0; k < 2; ++k) {
            const uint32_t inner = k == 0 ? 64u : 32u;
            if (k == 1 && out_cols % 64 == 0) break;
            int rc;
            if (d.a_mode == PP_A_MATRIX) {
                uint64_t dims[2] = {n_out, (uint64_t)d.M};
                uint64_t str[1] = {(uint64_t)d.ldc * 2};
                uint32_t box[2] = {inner, BLOCK_M};
                rc = make_tmap_bf16_sw(&p.tmOut[k], d.out, 2, dims, str, box, k == 0 ? 128 : 64);
            } else {
                uint64_t dims[4] = {n_out, (uint64_t)p.wo, (uint64_t)p.ho, (uint64_t)p.nb};
                uint64_t str[3] = {(uint64_t)d.ldc * 2, (uint64_t)d.ldc * 2 * p.wo, (uint64_t)d.ldc * 2 * p.wo * p.ho};
                uint32_t box[4] = {inner, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
                rc = make_tmap_bf16_sw(&p.tmOut[k], d.out, 4, dims, str, box, k == 0 ? 128 : 64);
            }
            if (rc) return rc;
        }
    }
    if (d.chan_stats) {
        pp_stats_geom g;
        int rc = gemm_stats_geometry(d, &g);
        if (rc) return rc;
        PP_REQUIRE(g.supported && (l.mode == 0 || l.mode >= 3), "gemm: chan_stats requested but this launch cannot emit statistics "
                   "(query pp_gemm_stats_geometry first)");
        PP_REQUIRE((reinterpret_cast<uintptr_t>(d.chan_stats) & 15) == 0, "gemm: chan_stats not 16-byte aligned");
        p.chan_stats = d.chan_stats;
        p.stat_segs = g.segs;
        p.stat_seg_rows_log2 = 0;
        while ((1 << p.stat_seg_rows_log2) < g.seg_rows) ++p.stat_seg_rows_log2;
    }
    if (d.row_stats) {
        PP_REQUIRE(gemm_row_stats_records(d) > 0, "gemm: row_stats requested but this launch cannot emit them "
                   "(query pp_gemm_row_stats_records first)");
        PP_REQUIRE(d.row_stats_ld >= d.M && (reinterpret_cast<uintptr_t>(d.row_stats) & 15) == 0,
                   "gemm: row_stats_ld=%lld < M or row_stats not 16-byte aligned", (long long)d.row_stats_ld);
        PP_REQUIRE(d.row_final && d.row_ticket && d.ln_eps > 0.f && (reinterpret_cast<uintptr_t>(d.row_final) & 7) == 0,
                   "gemm: row_stats needs row_final (8-byte aligned), row_ticket and ln_eps > 0");
        p.row_stats = reinterpret_cast<float4*>(d.row_stats);
        p.row_stats_ld = d.row_stats_ld;
        p.row_final = reinterpret_cast<float2*>(d.row_final);
        p.row_ticket = d.row_ticket;
        p.ln_eps = d.ln_eps;
    }
    if (d.ln_stats) {
        PP_REQUIRE(d.a_mode == PP_A_MATRIX && d.ln_u, "gemm: LayerNorm fold needs PP_A_MATRIX and ln_u");
        PP_REQUIRE(!d.res1 && !d.res2 && !d.rowvec && !d.a1 && d.alpha == 1.0f && !d.alpha_dev,
                   "gemm: LayerNorm-folded launches take bias only (no residual / row vector / alpha)");
        PP_REQUIRE((reinterpret_cast<uintptr_t>(d.ln_stats) & 7) == 0, "gemm: ln_stats not 8-byte aligned");
        p.ln_stats = reinterpret_cast<const float2*>(d.ln_stats);
        p.ln_u = d.ln_u;
        p.ln_eps = d.ln_eps;
    }
    if (ksplit == 2) {
        PP_REQUIRE(l.mode == 0 && (bn == 128 || bn == 160 || bn == 256), "gemm: split-K needs the plain bf16 epilogue");
        int rc = bn == 128 ? ensure_attr_splitk<128>() : bn == 160 ? ensure_attr_splitk<160>() : ensure_attr_splitk<256>();
        if (rc) return rc;
    } else {
        int rc = ensure_attr_for(bn, l.mode);
        if (rc) return rc;
    }
    *out = l;
    return PP_OK;
}

}  // namespace pp

extern "C" pp_status pp_gemm_stats_geometry(const pp_gemm_desc* d, pp_stats_geom* out) {
    if (!d || !out) {
        pp::set_last_error("pp_gemm_stats_geometry: null argument");
        return pp::PP_ERR_INVALID;
    }
    return pp::gemm_stats_geometry(*d, out);
}

extern "C" int32_t pp_gemm_row_stats_records(const pp_gemm_desc* d) { return d ? pp::gemm_row_stats_records(*d) : 0; }

extern "C" int64_t pp_gemm_splitk_bytes(const pp_gemm_desc* d0, int32_t* tiles_out) {
    if (tiles_out) *tiles_out = 0;
    if (!d0) return 0;
    // the query comes before the workspace exists: answer for the launch WITH a workspace attached
    pp_gemm_desc d = *d0;
    if (!d.splitk_ws) d.splitk_ws = reinterpret_cast<float*>(uintptr_t(16));
    if (!d.splitk_flags) d.splitk_flags = reinterpret_cast<int32_t*>(uintptr_t(16));
    pp::GemmKParams p;
    memset(&p, 0, sizeof(p));
    int bn = 0, ksplit = 1;
    if (pp::gemm_geometry(d, p, &bn, &ksplit) || ksplit != 2) return 0;
    if (tiles_out) *tiles_out = p.m_tiles * p.n_tiles;
    return (int64_t)p.m_tiles * p.n_tiles * pp::BLOCK_M * bn * 4;
}

extern "C" pp_status pp_gemm_variant(const pp_gemm_desc* d, int32_t* block_n, int32_t* mode, int32_t* ksplit) {
    if (!d || !block_n || !mode || !ksplit) {
        pp::set_last_error("pp_gemm_variant: null argument");
        return pp::PP_ERR_INVALID;
    }
    int bn = 0, m = 0, ks = 0;
    int rc = pp::gemm_variant(*d, &bn, &m, &ks);
    if (rc) return rc;
    *block_n = bn;
    *mode = m;
    *ksplit = ks;
    return pp::PP_OK;
}

extern "C" pp_status pp_gemm_conv(const pp_gemm_desc* d, pp_stream stream) {
    if (!d) {
        pp::set_last_error("pp_gemm_conv: null descriptor");
        return pp::PP_ERR_INVALID;
    }
    pp::GemmLaunch l;
    int rc = pp::gemm_prepare(*d, &l);
    if (rc) return rc;
    return pp::gemm_launch(l, reinterpret_cast<cudaStream_t>(stream));
}
