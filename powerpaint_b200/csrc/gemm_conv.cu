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
//    producer streams the next tile's operands while the consumers run this tile's epilogue. Each thread finishes its
//    own accumulators in the wgmma fragment layout and writes the results to the output staging tile with stmatrix.
//    Modes 0 / 3: the producer loads the tile's residual (res1) into that staging tile by TMA during the main loop,
//    and the epilogue reads it back with ldmatrix where its stmatrix will write the result.
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

// Generic epilogue of one output element (mode 1: fp32 / transposed / ragged N; the caller checks the row and n < N).
// `bias` is the staged bias of column n.
__device__ __forceinline__ void epilogue_store1(const GemmKParams& p, float alpha, float v, int64_t row, int grp, int n,
                                                float bias) {
    if (p.bias) v += bias;
    if (p.rowvec) v += __ldg(p.rowvec + (int64_t)grp * p.rowvec_ld + n);
    if (p.res1) v += __bfloat162float(p.res1[row * p.ldr1 + n]);
    v *= alpha;
    if (p.res2) v += __bfloat162float(p.res2[row * p.ldr2 + n]);
    if (p.act != PP_ACT_NONE) v = apply_act(v, p.act);
    if (p.epilogue == PP_EPI_TRANSPOSED) {
        // out[(row / t_rows) * N + n][row % t_rows]
        const int64_t b = (int)row / p.t_rows;  // 32-bit: a 64-bit division is a subroutine call, which would serialise the wgmma pipeline
        const int64_t t = row - b * p.t_rows;
        if (p.t_fp16) reinterpret_cast<__half*>(p.out)[(b * p.N + n) * p.t_ld + t] = __float2half_rn(v);
        else reinterpret_cast<__nv_bfloat16*>(p.out)[(b * p.N + n) * p.t_ld + t] = __float2bfloat16_rn(v);
    } else if (p.out_fp32) {
        reinterpret_cast<float*>(p.out)[row * p.ldc + n] = v;
    } else {
        reinterpret_cast<__nv_bfloat16*>(p.out)[row * p.ldc + n] = __float2bfloat16_rn(v);
    }
}

// Four 8x8 16-bit matrices from the accumulator fragment into shared memory; lane l gives the address of row l % 8 of
// matrix l / 8. With .trans each matrix is stored transposed (a fragment column becomes a row).
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c),
                 "r"(d)
                 : "memory");
}
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b),
                 "r"(c), "r"(d)
                 : "memory");
}

// The inverse: lane l addresses row l % 8 of matrix l / 8, and gets back each matrix in the fragment layout.
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr)
                 : "memory");
}

// Output staging tile: the epilogue writes its results (bf16) straight from the accumulator fragments (stmatrix) into
// shared memory laid out as the boxes of a TMA store — 64-column sub-tiles [128 rows][128 B] with the 128-byte swizzle (the 160-wide tile ends in a
// 32-column sub-tile [128][64 B] with the 64-byte swizzle) — and one thread per sub-tile hands them to the TMA unit,
// which writes whole rows and clips whatever lies outside the tensor (ragged conv tiles, rows >= M, columns >= N).
__host__ __device__ constexpr int out_stage_bytes_for(int block_n) {
    return (block_n / 64) * 16384 + (block_n % 64) * 256;
}
// fixed part: 1 KB alignment slack, barriers, bias + LayerNorm-sum staging [4][BLOCK_N] floats, row table
__host__ __device__ constexpr int fixed_smem_for(int block_n) {
    return 1024 + 256 + 4 * block_n * 4 + 128 * 8 + 1024 + out_stage_bytes_for(block_n);
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
static_assert(stages_for(160) == 5 && stages_for(128) == 5 && stages_for(256) == 3 && stages_for(64) == 8,
              "ring stages per tile width");

// Persistent, warp-specialised kernel: grid = min(#tiles, #SMs); each CTA walks tiles
// blockIdx.x, blockIdx.x + gridDim.x, ... (n fastest, so CTAs running concurrently share A tiles
// through L2 and the weights stay L2-resident).
//   warp 8      TMA producer  (smem ring continues across tile boundaries)
//   warps 0..7  two consumer warpgroups: warpgroup g issues the wgmma of tile rows [64 g, 64 g + 64) and then runs
//               the epilogue of the same rows straight from the accumulator registers (a thread holds two rows, 8 apart,
//               and two columns of every 8-column group)
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

    extern __shared__ uint8_t smem_raw[];
    // mode 3 (LayerNorm-statistics producer): mailbox between the epilogue and the ticket-server lane, and the verdict
    // ("this CTA finished the last n-tile of the row block") of the tile whose records are folded next
    __shared__ volatile int s_req_seq, s_req_mtile, s_resp_seq, s_resp_last;
    __shared__ int s_last_tile;
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sA = smem_base;
    const uint32_t sB = sA + STAGES * A_STAGE_BYTES;
    // output staging tile, 1024-byte aligned
    const uint32_t s_out_addr = sB + STAGES * B_STAGE_BYTES;
    uint8_t* s_out = smem_raw + (s_out_addr - smem_u32(smem_raw));
    const uint32_t bar_base = s_out_addr + out_stage_bytes_for(BLOCK_N);
    // barriers: full[STAGES], empty[STAGES] (at most 8 each), then the residual staging pair: stage_free (every consumer
    // warp is in the tile's main loop and its stores of the previous tile have read the staging tile) and res_full
    // (the tile's residual boxes have landed in the staging tile)
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
    const uint32_t stage_free_bar = bar_base + 128u, res_full_bar = bar_base + 136u;
    // bias of the current / next tile, staged by the epilogue warps: [2][BLOCK_N] floats
    float* sbias_all = reinterpret_cast<float*>(smem_raw + (bar_base + 256 - smem_u32(smem_raw)));
    // column sums of the gamma-folded weights (LayerNorm fold) or, in modes 0 / 3, the tile's row-vector row (stage_rv),
    // staged like the bias: [2][BLOCK_N] floats
    float* su_all = sbias_all + 2 * BLOCK_N;
    // validity of each tile row (statistics pass)
    long long* s_row = reinterpret_cast<long long*>(reinterpret_cast<uint8_t*>(sbias_all) + 4 * BLOCK_N * 4);
    // offset in the staging tile of the 16-byte piece of row r holding columns [col, col + 8)
    auto stage_off = [&](int r, int col) -> uint32_t {
        const int sub = col >> 6, c = (col & 63) >> 3;
        if ((BLOCK_N % 64) != 0 && sub == BLOCK_N / 64)  // 32-column remainder sub-tile, 64-byte swizzle
            return sub * 16384 + r * 64 + ((c ^ ((r >> 1) & 3)) << 4);
        return sub * 16384 + r * 128 + ((c ^ (r & 7)) << 4);
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
    // modes 0 / 3: res1 reaches the epilogue through the staging tile (TMA during the main loop), and the time-embedding
    // row vector through the second staging row (su_all, unused without the LayerNorm fold) when every tile lies in one
    // sample; the split-K donor has no epilogue
    constexpr bool kRes = MODE == 0 || MODE == 3;
    const bool stage_res = kRes && p.res1 != nullptr && !(kSplitK && khalf);
    const bool stage_rv =
        kRes && p.rowvec != nullptr && (p.a_mode == PP_A_MATRIX ? p.rows_per_group % BLOCK_M == 0 : p.bn == 1);

    constexpr int W_PROD = GEMM_EPI_WARPS;
    if (warp == W_PROD && elect_one()) {
        prefetch_tmap(&p.tmA[0]);
        prefetch_tmap(&p.tmB);
        if constexpr (MODE != 1) prefetch_tmap(&p.tmOut[0]);
        if (stage_res) prefetch_tmap(&p.tmRes[0]);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), GEMM_EPI_WARPS);  // one arrival per consumer warp
        }
        mbar_init(stage_free_bar, GEMM_EPI_WARPS);
        mbar_init(res_full_bar, 1);
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
            // res1 of the producer's residual tile r_tile (local index r_lt) goes into the staging tile once stage_free
            // says it is free, i.e. while the consumers run that tile's main loop: the same boxes and swizzles as the
            // output store, so each value lands where the epilogue's stmatrix puts the result of its element.
            // Out-of-bounds rows and columns read as zero; sub-tiles wholly beyond N are not loaded. The producer
            // probes stage_free without blocking wherever it waits for a ring slot, so the operand stream never waits
            // for the staging tile.
            TileWalk rw(walk_first, walk_stride, n_tiles);
            int r_tile = walk_first;
            uint32_t r_lt = 0;
            auto issue_res = [&] {
                const int n_base = rw.n * BLOCK_N;
                uint32_t bytes = 0;
                for (int sub = 0; sub * 64 < BLOCK_N; ++sub)
                    if (n_base + sub * 64 < p.N) bytes += (BLOCK_N - sub * 64) >= 64 ? 16384u : 8192u;
                int x0 = 0, y0 = 0, nb0 = 0;
                if (p.a_mode != PP_A_MATRIX) tile_origin(rw.m, x0, y0, nb0);
                mbar_arrive_expect_tx(res_full_bar, bytes);
                for (int sub = 0; sub * 64 < BLOCK_N && n_base + sub * 64 < p.N; ++sub) {
                    const CUtensorMap* tm = (BLOCK_N - sub * 64) >= 64 ? &p.tmRes[0] : &p.tmRes[1];
                    if (p.a_mode == PP_A_MATRIX)
                        tma_load_2d(s_out_addr + sub * 16384, tm, res_full_bar, n_base + sub * 64, rw.m * BLOCK_M);
                    else
                        tma_load_4d(s_out_addr + sub * 16384, tm, res_full_bar, n_base + sub * 64, x0, y0, nb0);
                }
                rw.next();
                r_tile += walk_stride;
                ++r_lt;
            };
            auto poll_res = [&] {
                while (r_tile < num_tiles && mbar_test_wait(stage_free_bar, r_lt & 1u)) issue_res();
            };
            auto wait_slot = [&](uint32_t bar, uint32_t parity) {
                if (!stage_res) {
                    mbar_wait(bar, parity);
                    return;
                }
                poll_res();
                const uint64_t t0 = global_timer_ns();
                uint32_t spins = 0;
                while (!mbar_test_wait(bar, parity)) {
                    poll_res();
                    if ((++spins & 0xFFu) == 0 && global_timer_ns() - t0 > PP_WAIT_TIMEOUT_NS) __trap();
                }
            };
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
                    wait_slot(empty_bar(s), ph ^ 1u);
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
            // the operands are all on their way: the residuals of the last tiles
            if (stage_res) {
                while (r_tile < num_tiles) {
                    mbar_wait(stage_free_bar, r_lt & 1u);
                    issue_res();
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: MMA + epilogue =====================
        const int wg = warp >> 2;  // warpgroup: tile rows [64 wg, 64 wg + 64)
        const int etid = threadIdx.x;  // 0..255 among the epilogue threads
        const int lane = (int)lane_id(), quad = lane & 3;
        // this thread's accumulators (wgmma fragment): tile rows r0 (h = 0) and r0 + 8 (h = 1), and per 8-column group i
        // the columns 8 i + 2 quad + {0, 1}: facc[4 i + 2 h + {0, 1}]
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
        // stmatrix.x4 of the 8-column groups (i, i + 1): matrix lane / 8 is (rows + 8 ((lane / 8) & 1), group i + lane / 16);
        // this lane addresses its row lane % 8 (transposed: its column)
        const int st_row = 64 * wg + 16 * (warp & 3) + 8 * ((lane >> 3) & 1);
        const int st_grp = lane >> 4, st_j = lane & 7;
        auto epi_sync = [] { asm volatile("bar.sync 1, %0;" ::"n"(GEMM_EPI_WARPS * 32) : "memory"); };
        // ---- main loop of one tile: this warpgroup's 64 x BLOCK_N accumulators. `before_drain` runs ahead of the last
        // wait, so global loads it issues overlap the final MMAs.
        int ks = 0;  // ring slot and its phase, carried across tiles (the producer's sequence)
        uint32_t kph = 0;
        auto mainloop = [&](float (&facc)[BLOCK_N / 2], int m_tile, int n_tile, auto&& before_drain) {
            // zeroed here (not by the first MMA's scale-d): the registers are then dead between tiles
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
                if (stage_res && it == k_begin) {
                    // this warp is done with the staging tile of the previous tile (its stmatrix writes were fenced to
                    // the async proxy before the store): once its stores have read it, the residual may go in
                    __syncwarp();
                    if (lane_id() == 0) {
                        bulk_wait_read_all();
                        mbar_arrive(stage_free_bar);
                    }
                }
                prev = ks;
                if (++ks == STAGES) { ks = 0; kph ^= 1u; }
            }
            before_drain();
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
            // the epilogue writes the staging tile next: the TMA unit has read the previous tile out of it, and every
            // epilogue thread is past its reads of it (statistics pass included)
            if constexpr (MODE != 1) {
                if ((etid & 31) == 0) bulk_wait_read_all();
            }
            epi_sync();
            if constexpr (kSplitK) {
                // split-K: the donor's raw fp32 accumulators go to the workspace in fragment order ([tile][group][thread]
                // float4, coalesced); the owner adds the donor's to its own (owner + donor, always in this order)
                float4* ws = reinterpret_cast<float4*>(p.splitk_ws) +
                             ((int64_t)m_tile * n_tiles + n_tile) * (BLOCK_M * BLOCK_N / 4) + etid;
                if (khalf) {
#pragma unroll
                    for (int i = 0; i < BLOCK_N / 8; ++i)
                        ws[i * (GEMM_EPI_WARPS * 32)] = make_float4(facc[4 * i], facc[4 * i + 1], facc[4 * i + 2], facc[4 * i + 3]);
                } else {
#pragma unroll
                    for (int i = 0; i < BLOCK_N / 8; ++i) {
                        const float4 pp = __ldcg(ws + i * (GEMM_EPI_WARPS * 32));
                        facc[4 * i] = facc[4 * i] + pp.x;
                        facc[4 * i + 1] = facc[4 * i + 1] + pp.y;
                        facc[4 * i + 2] = facc[4 * i + 2] + pp.z;
                        facc[4 * i + 3] = facc[4 * i + 3] + pp.w;
                    }
                }
            }
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
        // row-vector row of an m-tile that lies in one sample (stage_rv)
        auto rv_row = [&](int m_tile_of) -> const float* {
            const int g = p.a_mode == PP_A_MATRIX ? m_tile_of * BLOCK_M / p.rows_per_group : m_tile_of / (p.tiles_x * p.tiles_y);
            return p.rowvec + (int64_t)g * p.rowvec_ld;
        };
        // stage the first tile's bias
        TileWalk tw(walk_first, walk_stride, n_tiles);
        if (walk_first < num_tiles) {
            const float b0 = load_bias(tw.n);
            float u0 = load_u(tw.n);
            if (stage_rv && etid < BLOCK_N && tw.n * BLOCK_N + etid < p.N) u0 = __ldg(rv_row(tw.m) + tw.n * BLOCK_N + etid);
            if (etid < BLOCK_N) {
                sbias_all[etid] = b0;
                su_all[etid] = u0;
            }
        }
        epi_sync();
        // {rstd, -rstd * mean} of this thread's two rows in the current tile
        float2 ln_cur[2] = {make_float2(1.f, 0.f), make_float2(1.f, 0.f)};
        if (ln && walk_first < num_tiles) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row0 = (int64_t)tw.m * BLOCK_M + r0 + 8 * h;
                if (row0 < p.M) ln_cur[h] = __ldg(p.ln_stats + row0);
            }
        }
        // ---- mode 3: verdict of the ticket server for request number `seq`, and the fold of a row's records
        // (one thread per row: quad lanes 0 / 1 fold rows r0 / r0 + 8)
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
                else if (next_tile < num_tiles && stage_rv && nn < p.N) cp_async_f32(du, rv_row(tw.m) + nn);
                else *du = 0.f;
            }
            if (etid == 0) GT(lt, 16);
            // output rows of this thread (tile rows r0 and r0 + 8)
            bool valid[2];
            int64_t row[2];
            int grp[2];
            if (p.a_mode == PP_A_MATRIX) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    row[h] = (int64_t)m_tile * BLOCK_M + r0 + 8 * h;
                    valid[h] = row[h] < p.M;
                    grp[h] = p.rowvec ? (int)row[h] / p.rows_per_group : 0;
                }
            } else {
                int x0, y0, nb0;
                tile_origin(m_tile, x0, y0, nb0);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    // bw, bh, bn are powers of two
                    const int r = r0 + 8 * h;
                    const int ix = r & (p.bw - 1);
                    const int iy = (r >> p.bw_log2) & (p.bh - 1);
                    const int in = r >> (p.bw_log2 + p.bh_log2);
                    const int ox = x0 + ix, oy = y0 + iy, on = nb0 + in;
                    valid[h] = in < p.bn && ox < p.wo && oy < p.ho && on < p.nb;
                    row[h] = ((int64_t)on * p.ho + oy) * p.wo + ox;
                    grp[h] = on;
                }
            }
            if (etid == 0) GT(lt, 17);
            const int n_base = n_tile * BLOCK_N;
            // mode 5: this tile's columns are stored transposed ([channel][token], V^T for the attention kernel)
            const bool ttile = MODE == 5 && n_tile >= p.trans_first_tile;
            // LayerNorm fold: acc' = ln_rs * acc + ln_nm * u[n] with {ln_rs, ln_nm} = {rstd, -rstd * mean} of the row, as
            // left by the producer (row_final). The pairs of the NEXT tile's rows are fetched now, so that their
            // global-memory latency is off the epilogue's serial path (a per-tile fold of the raw records cost ~2500
            // cycles a tile).
            const float ln_rs[2] = {ln_cur[0].x, ln_cur[1].x}, ln_nm[2] = {ln_cur[0].y, ln_cur[1].y};
            if (ln) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t nrow = (int64_t)tw.m * BLOCK_M + r0 + 8 * h;  // tw is already at the next tile
                    ln_cur[h] = (next_tile < num_tiles && nrow < p.M) ? __ldg(p.ln_stats + nrow) : make_float2(1.f, 0.f);
                }
            }
            float facc[BLOCK_N / 2];
            if constexpr (MODE == 2) {
                // GEGLU: value column c and gate column c + BLOCK_N / 2 sit in the same thread (BLOCK_N / 2 is a multiple
                // of 8); the HALF output columns are staged like a HALF-wide tile
                constexpr int HALF = BLOCK_N / 2;
                const int o_base = n_tile * HALF;  // output column of this tile
                const int n_out = p.N / 2;
                mainloop(facc, m_tile, n_tile, [] {});
                if (etid == 0) GT(lt, 5);
#pragma unroll
                for (int k = 0; k < HALF / 16; ++k) {
                    uint32_t q[4];  // stmatrix operands: (group 2k, row h = 0 / 1), (group 2k + 1, row h = 0 / 1)
#pragma unroll
                    for (int g = 0; g < 2; ++g) {
                        const int i = 2 * k + g, c = 8 * i + 2 * quad;
                        const float2 ba = *reinterpret_cast<const float2*>(sbias + c);
                        const float2 bg = *reinterpret_cast<const float2*>(sbias + HALF + c);
                        float2 ua = make_float2(0.f, 0.f), ug = make_float2(0.f, 0.f);
                        if (ln) {
                            ua = *reinterpret_cast<const float2*>(su + c);
                            ug = *reinterpret_cast<const float2*>(su + HALF + c);
                        }
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            float v[2];
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                float a = facc[4 * i + 2 * h + e], gt = facc[4 * (i + HALF / 8) + 2 * h + e];
                                const float bae = e ? ba.y : ba.x, bge = e ? bg.y : bg.x;
                                if (ln) {
                                    a = fmaf(a, ln_rs[h], fmaf(ln_nm[h], e ? ua.y : ua.x, bae));
                                    gt = fmaf(gt, ln_rs[h], fmaf(ln_nm[h], e ? ug.y : ug.x, bge));
                                } else {
                                    a += bae;
                                    gt += bge;
                                }
                                v[e] = (valid[h] && o_base + 8 * i < n_out) ? a * gelu_tanh_f(gt) : 0.f;
                            }
                            q[2 * g + h] = pack_bf16x2(v[0], v[1]);
                        }
                    }
                    stmatrix_x4(s_out_addr + stage_off(st_row + st_j, 16 * k + 8 * st_grp), q[0], q[1], q[2], q[3]);
                }
            } else if constexpr (MODE == 0 || MODE == 3 || MODE == 4 || MODE == 5) {
                // lean path: uniform flags hoisted. The epilogue runs with only two warps per scheduler, so it is
                // latency-bound unless the 8-column groups are independent straight-line code: the common case (tile
                // fully inside the matrix, all rows of the warp valid) has no per-group branches at all, and launches
                // without residual / row-vector terms skip those adds.
                if (etid == 0) GT(lt, 18);
                const float alpha = effective_alpha(p);
                const bool has_r1 = p.res1 != nullptr, has_r2 = p.res2 != nullptr, has_rv = p.rowvec != nullptr;
                const int act = p.act;
                const int ncols = min(BLOCK_N, p.N - n_base);  // multiple of 8
                const bool full = ncols == BLOCK_N && __all_sync(0xffffffffu, valid[0] && valid[1]);
                const bool plain = !has_r1 && !has_r2 && !has_rv;
                const bool ln_fold = MODE == 4 || (MODE == 5 && ln);  // these launches carry no residual / row vector
                // res1 comes from the staging tile and the row vector, where every tile lies in one sample, from su (both
                // staged during the main loop). The other terms (res2, the row vector of tiles spanning two samples) of
                // the column pair (8 i + 2 quad, + 1) of both rows are fetched D group pairs ahead of their use; the first
                // D before the main loop's last wait. The 256-wide statistics producer has no registers for that: it
                // fetches each pair's terms where it uses them (with D = 1 it spilled 614 bytes, more than the 506 of the
                // fp32-tile epilogue).
                constexpr int NP = BLOCK_N / 16;  // group pairs: one stmatrix.x4 each
                constexpr int D = (MODE == 3 && BLOCK_N == 256) ? 0 : 1;
                uint32_t q2[NP][2][2];  // [pair][group][row]
                float2 tv[NP][2][2];
                const bool fetch_rv = has_rv && !stage_rv;
                // uniform: a launch without register-path terms skips their address arithmetic altogether (predicated
                // off, it still took more than a third of each pair's instructions, in an issue-bound loop)
                const bool reg_terms = has_r2 || fetch_rv;
                auto fetch = [&](int k) {
                    if constexpr (kRes) {
                        if (k >= NP) return;
                        if (!reg_terms) {
#pragma unroll
                            for (int g = 0; g < 2; ++g) {
#pragma unroll
                                for (int h = 0; h < 2; ++h) {
                                    q2[k][g][h] = 0u;
                                    tv[k][g][h] = make_float2(0.f, 0.f);
                                }
                            }
                            return;
                        }
#pragma unroll
                        for (int g = 0; g < 2; ++g) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int col = 16 * k + 8 * g;
                                const bool ok = valid[h] && col < ncols;
                                const int64_t c = n_base + col + 2 * quad;
                                q2[k][g][h] = (ok && has_r2) ? __ldg(reinterpret_cast<const uint32_t*>(p.res2 + row[h] * p.ldr2 + c)) : 0u;
                                tv[k][g][h] = (ok && fetch_rv) ? __ldg(reinterpret_cast<const float2*>(p.rowvec + (int64_t)grp[h] * p.rowvec_ld + c))
                                                               : make_float2(0.f, 0.f);
                            }
                        }
                    }
                };
                if (etid == 0) GT(lt, 14);  // tile set-up done, about to run the main loop
                mainloop(facc, m_tile, n_tile, [&] {
#pragma unroll
                    for (int k = 0; k < D; ++k) fetch(k);
                });
                if (etid == 0) GT(lt, 5);  // accumulators ready
                if constexpr (kSplitK) {
                    if (khalf) {
                        // donor: the partial tile is in the workspace; publish it and leave (no output of its own)
                        cp_async_wait_all();
                        __threadfence();
                        epi_sync();
                        if (etid == 0) {
                            __threadfence();
                            *(volatile int32_t*)(p.splitk_flags + (int64_t)m_tile * n_tiles + n_tile) = 1;
                        }
                        continue;
                    }
                }
                // mode 3: per row and half n-tile ([0, BLOCK_N / 2), [BLOCK_N / 2, BLOCK_N)) the sums of x - shift and
                // (x - shift)^2, shift = the half's first value of the row (so a large common offset does not cancel in
                // the variance)
                float st_s1[2], st_s2[2], st_shift[2];
                constexpr int HALF_NP = NP / 2;
                // staged residual: ldmatrix.x4 at the address of the pair's stmatrix.x4 returns it in fragment order
                // (group g, row h in register 2 g + h), and the result goes back to the same place. A warp reads and
                // writes only its own 16 rows.
                auto st_addr = [&](int k) { return s_out_addr + stage_off(st_row + st_j, 16 * k + 8 * st_grp); };
                if (stage_res) mbar_wait(res_full_bar, lt & 1u);
#pragma unroll
                for (int k = 0; k < NP; ++k) {
                    fetch(k + D);
                    uint32_t r1q[4] = {0u, 0u, 0u, 0u};
                    if (stage_res) ldmatrix_x4(st_addr(k), r1q);
                    float v[2][2][2];  // [group][row][column of the pair]
#pragma unroll
                    for (int g = 0; g < 2; ++g) {
                        const int i = 2 * k + g, c = 8 * i + 2 * quad;
                        const float2 b = *reinterpret_cast<const float2*>(sbias + c);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float a0 = facc[4 * i + 2 * h], a1 = facc[4 * i + 2 * h + 1];
                            const bool ok = valid[h] && 8 * i < ncols;
                            if (ln_fold) {
                                const float2 u = *reinterpret_cast<const float2*>(su + c);
                                // alpha == 1 for LayerNorm-folded launches (checked at prepare time)
                                v[g][h][0] = ok ? fmaf(a0, ln_rs[h], fmaf(ln_nm[h], u.x, b.x)) : 0.f;
                                v[g][h][1] = ok ? fmaf(a1, ln_rs[h], fmaf(ln_nm[h], u.y, b.y)) : 0.f;
                            } else if (MODE == 4 || (full && plain)) {
                                v[g][h][0] = (a0 + b.x) * alpha;
                                v[g][h][1] = (a1 + b.y) * alpha;
                            } else {
                                const uint32_t r1 = kRes ? r1q[2 * g + h] : 0u, r2 = kRes ? q2[k][g][h] : 0u;
                                const float2 t = !kRes ? make_float2(0.f, 0.f)
                                                 : stage_rv ? *reinterpret_cast<const float2*>(su + c) : tv[k][g][h];
                                float x0 = a0 + b.x + t.x, x1 = a1 + b.y + t.y;
                                x0 = (x0 + bf16_lo(r1)) * alpha + bf16_lo(r2);
                                x1 = (x1 + bf16_hi(r1)) * alpha + bf16_hi(r2);
                                v[g][h][0] = ok ? x0 : 0.f;
                                v[g][h][1] = ok ? x1 : 0.f;
                            }
                        }
                    }
                    if constexpr (MODE == 3) {  // mode 3 is only selected with row_stats set, and without activation
                        if (k % HALF_NP == 0) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                st_shift[h] = __shfl_sync(0xffffffffu, v[0][h][0], lane & ~3);
                                st_s1[h] = st_s2[h] = 0.f;
                            }
                        }
#pragma unroll
                        for (int g = 0; g < 2; ++g) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                if (8 * (2 * k + g) < ncols) {
#pragma unroll
                                    for (int e = 0; e < 2; ++e) {
                                        const float d = v[g][h][e] - st_shift[h];
                                        st_s1[h] += d;
                                        st_s2[h] = fmaf(d, d, st_s2[h]);
                                    }
                                }
                            }
                        }
                        if (k % HALF_NP == HALF_NP - 1) {
                            const int hf = k / HALF_NP;  // half n-tile
                            const float cnt = (float)min(max(ncols - hf * (BLOCK_N / 2), 0), BLOCK_N / 2);
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                float s1 = st_s1[h], s2 = st_s2[h];
                                s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
                                s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
                                s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
                                s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
                                if (quad == h && valid[h])
                                    p.row_stats[(int64_t)(n_tile * 2 + hf) * p.row_stats_ld + row[h]] =
                                        make_float4(s1, s2, st_shift[h], cnt);
                            }
                        }
                    }
                    if (act == PP_ACT_SILU) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) (&v[0][0][0])[j] = silu_f((&v[0][0][0])[j]);
                    } else if (act == PP_ACT_QUICK_GELU) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) (&v[0][0][0])[j] = quick_gelu_f((&v[0][0][0])[j]);
                    }
                    if (MODE == 5 && ttile) {
                        // transposed staging: [column][128 rows] 16-bit, 64-column sub-tiles of 16 KB (the boxes of the
                        // transposed TMA store); V^T is fp16 (P is fp16 in the attention kernel). The layout is the TMA
                        // box's and cannot be swizzled: the 16-byte rows of one stmatrix.trans are 256 bytes apart, so
                        // its 512 bytes take 16 shared-memory wavefronts (a conflict-free store would take 4)
                        uint32_t q[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            q[j] = p.t_fp16 ? pack_f16x2(v[j >> 1][j & 1][0], v[j >> 1][j & 1][1])
                                            : pack_bf16x2(v[j >> 1][j & 1][0], v[j >> 1][j & 1][1]);
                        const int col = 16 * k + 8 * st_grp + st_j;
                        stmatrix_x4_trans(s_out_addr + (col >> 6) * 16384 + (col & 63) * 256 + st_row * 2, q[0], q[1], q[2],
                                          q[3]);
                    } else {
                        stmatrix_x4(st_addr(k), pack_bf16x2(v[0][0][0], v[0][0][1]), pack_bf16x2(v[0][1][0], v[0][1][1]),
                                    pack_bf16x2(v[1][0][0], v[1][0][1]), pack_bf16x2(v[1][1][0], v[1][1][1]));
                    }
                }
            } else {
                // generic (fp32 / transposed / ragged N): straight from the fragment to global memory
                const float alpha1 = effective_alpha(p);
                mainloop(facc, m_tile, n_tile, [] {});
#pragma unroll
                for (int i = 0; i < BLOCK_N / 8; ++i) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = 8 * i + 2 * quad + e;
                            if (valid[h] && n_base + c < p.N) {
                                float v = facc[4 * i + 2 * h + e];
                                if (ln) v = fmaf(v, ln_rs[h], ln_nm[h] * su[c]);
                                epilogue_store1(p, alpha1, v, row[h], grp[h], n_base + c, sbias[c]);
                            }
                        }
                    }
                }
            }
            if (etid == 0) GT(lt, 6);  // tile math done
            // the next tile's bias has landed in the other staging buffer (asynchronous copies issued at the top of this
            // tile); the barrier below publishes it before tile lt + 1 reads it
            cp_async_wait_all();
            if constexpr (MODE == 3) {
                if (etid == 0 && lt > 0) s_last_tile = ticket_verdict((int)lt);  // of tile lt - 1 (request number lt)
            }
            if constexpr (MODE != 1) {
                fence_proxy_async_smem();  // the staging stores (generic proxy) -> the TMA unit (async proxy)
                if (quad == 0) {
                    s_row[r0] = valid[0] ? (long long)row[0] : -1ll;
                    s_row[r0 + 8] = valid[1] ? (long long)row[1] : -1ll;
                }
            }
            epi_sync();
            if (etid == 0) GT(lt, 7);  // all epilogue warps staged
            // mode 3: the previous tile was the last n-tile of its row block -> fold the block's records (first four loads
            // now, the arithmetic after the hand-over to the TMA unit); then post this tile's ticket request
            float4 frc[4];
            bool fold_prev = false;
            if constexpr (MODE == 3) {
                fold_prev = lt > 0 && s_last_tile != 0 && prev_valid;
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
                    prev_row = quad == 0 ? row[0] : row[1];
                    prev_valid = quad < 2 && (quad == 0 ? valid[0] : valid[1]);
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
                                    const uint4 q = *reinterpret_cast<const uint4*>(s_out + stage_off(rb, piece * 8));
                                    const bool okr = s_row[rb] >= 0;
                                    sh[0] = okr ? bf16_lo(q.x) : 0.f; sh[1] = okr ? bf16_hi(q.x) : 0.f;
                                    sh[2] = okr ? bf16_lo(q.y) : 0.f; sh[3] = okr ? bf16_hi(q.y) : 0.f;
                                    sh[4] = okr ? bf16_lo(q.z) : 0.f; sh[5] = okr ? bf16_hi(q.z) : 0.f;
                                    sh[6] = okr ? bf16_lo(q.w) : 0.f; sh[7] = okr ? bf16_hi(q.w) : 0.f;
                                }
                                for (int rr = rb + l; rr < rb + seg_rows; rr += L) {
                                    if (s_row[rr] >= 0) {
                                        const uint4 q = *reinterpret_cast<const uint4*>(s_out + stage_off(rr, piece * 8));
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
            // the last tile's verdict and fold, then release the ticket server. The barrier first: every warp has read
            // the previous verdict (fold_prev, after the last tile's second barrier) before etid 0 overwrites it
            epi_sync();
            if (etid == 0 && lt > 0) s_last_tile = ticket_verdict((int)lt);
            epi_sync();
            if (lt > 0 && s_last_tile != 0 && prev_valid) {
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

// records per row a GEMM emits for the consumer's LayerNorm: one per half n-tile (columns [0, BLOCK_N / 2) and
// [BLOCK_N / 2, BLOCK_N)); 0 = this launch cannot emit them
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

static int gemm_staging(const pp_gemm_desc& d, int* stage_res, int* stage_rv) {
    GemmKParams p;
    memset(&p, 0, sizeof(p));
    int bn = 0;
    int rc = gemm_geometry(d, p, &bn);
    if (rc) return rc;
    // the kernel's stage_res / stage_rv of a launch (the split-K donor's half stages nothing: it has no epilogue)
    const int mode = gemm_select_mode(d);
    const bool kRes = mode == 0 || mode == 3;
    *stage_res = kRes && d.res1 != nullptr;
    *stage_rv = kRes && d.rowvec != nullptr && (d.a_mode == PP_A_MATRIX ? d.rows_per_group % BLOCK_M == 0 : p.bn == 1);
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
            if ((l.mode == 0 || l.mode == 3) && d.res1) {
                // the residual tile goes through the same boxes into the staging tile, so it lands where the
                // epilogue's stmatrix writes the results
                if (d.a_mode == PP_A_MATRIX) {
                    uint64_t dims[2] = {(uint64_t)d.N, (uint64_t)d.M};
                    uint64_t str[1] = {(uint64_t)d.ldr1 * 2};
                    uint32_t box[2] = {inner, BLOCK_M};
                    rc = make_tmap_bf16_sw(&p.tmRes[k], d.res1, 2, dims, str, box, k == 0 ? 128 : 64);
                } else {
                    uint64_t dims[4] = {(uint64_t)d.N, (uint64_t)p.wo, (uint64_t)p.ho, (uint64_t)p.nb};
                    uint64_t str[3] = {(uint64_t)d.ldr1 * 2, (uint64_t)d.ldr1 * 2 * p.wo,
                                       (uint64_t)d.ldr1 * 2 * p.wo * p.ho};
                    uint32_t box[4] = {inner, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
                    rc = make_tmap_bf16_sw(&p.tmRes[k], d.res1, 4, dims, str, box, k == 0 ? 128 : 64);
                }
                if (rc) return rc;
            }
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

extern "C" pp_status pp_gemm_staging(const pp_gemm_desc* d, int32_t* stage_res, int32_t* stage_rv) {
    if (!d || !stage_res || !stage_rv) {
        pp::set_last_error("pp_gemm_staging: null argument");
        return pp::PP_ERR_INVALID;
    }
    int r = 0, v = 0;
    int rc = pp::gemm_staging(*d, &r, &v);
    if (rc) return rc;
    *stage_res = r;
    *stage_rv = v;
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
