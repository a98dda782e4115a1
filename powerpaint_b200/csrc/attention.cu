// Fused scaled-dot-product attention on wgmma / TMA (sm_90a), no mask, non-causal.
//
// Reference: diffusers Attention + AttnProcessor2_0 -> F.scaled_dot_product_attention(q, k, v)
// with scale 1/sqrt(d) (processors referenced at powerpaint/models/unet_2d_condition.py:24-31;
// instantiated through Transformer2DModel at unet_2d_blocks.py:807,1289,2514). Self-attention
// over N = h*w latent tokens (4096/1024/256/64 at 512^2) and cross-attention over 77 text
// tokens; 8 heads of d = 40 / 80 / 160.
//
// One CTA = one (128-query tile, head, sample), 288 threads. Flash-style streaming over 128-key blocks:
//   warp 8      TMA producer: Q once, then K / V^T blocks through a ring of kv stages
//   warps 0..7  two consumer warpgroups of 64 query rows each. Per key block: S = Q K^T (wgmma, both operands
//               in shared memory) into registers; online softmax in fp32 registers (exp2 domain; a row lives in
//               the four lanes of a quad, so row max / sum need two shuffles); P rounded to fp16 / bf16 stays in
//               registers and is the A operand of O += P V (wgmma with A from registers, V^T from shared memory,
//               O in registers). DV <= 64: the warpgroups take turns on the tensor cores and each issues S of the
//               next key block with PV of this one, so the exponentials overlap MMAs; DV > 64: they run independently.
// The row sums add the 16-bit P the MMA actually sees (DV <= 64 with d < DV: the PV MMA adds them up itself, in
// column d, against a row of ones in V^T). Head dims that are not multiples of 64/16 need no
// padding in HBM: the Q/K tensor maps are (d, heads, tokens, batch) so TMA zero-fills channels >= d of each head,
// and V is consumed transposed ([batch, heads*d, keys], keys contiguous; produced by the projection GEMM's
// transposed epilogue) so both MMAs read K-major SWIZZLE_128B operands; V^T rows >= d read as zeros (DV > 64).
#include <math.h>

#include <algorithm>

#include <cuda_fp16.h>

#include "common.cuh"
#include "ops.h"
#include "wgmma.cuh"

namespace pp {

static constexpr int ATT_BM = 128;   // queries per CTA
static constexpr int ATT_BN = 128;   // keys per block
static constexpr int ATT_THREADS = 288;
static constexpr uint32_t ATT_CHUNK_BYTES = 128 * 128;  // [128 rows x 64 bf16]

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// named barriers of `nthreads` threads (multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// DV: width of the PV product (head dim rounded up to one of the instantiated widths)
__host__ __device__ constexpr int att_dch(int dv) { return (dv + 63) / 64; }  // 64-channel chunks of Q / K
__host__ __device__ constexpr int att_stages(int dv) { return att_dch(dv) == 1 ? 3 : att_dch(dv) == 2 ? 2 : 1; }
__host__ __device__ constexpr uint32_t att_smem_bytes(int dv) {
    return att_dch(dv) * ATT_CHUNK_BYTES                                            // Q
           + att_stages(dv) * (att_dch(dv) * ATT_CHUNK_BYTES + (uint32_t)dv * 256u)  // K + V^T ring
           + 256 + 1024;
}

template <bool F16>
__device__ __forceinline__ uint32_t pack_p(float lo, float hi) {
    return F16 ? pack_f16x2(lo, hi) : pack_bf16x2(lo, hi);
}
template <bool F16>
__device__ __forceinline__ float sum_p(uint32_t v) {
    if constexpr (F16) {
        const __half2 h = *reinterpret_cast<const __half2*>(&v);
        return __low2float(h) + __high2float(h);
    } else {
        return bf16_lo(v) + bf16_hi(v);
    }
}

template <int DV, bool F16>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_kernel(const __grid_constant__ AttnKParams p) {
    constexpr int DCH = att_dch(DV), S = att_stages(DV);
    constexpr uint32_t V_CHUNK = DV * 128u, V_STAGE = 2 * V_CHUNK;  // V^T tile: two 64-key chunks [DV rows][128 B]

    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const uint32_t sQ = base;
    const uint32_t sK0 = sQ + DCH * ATT_CHUNK_BYTES;
    const uint32_t sV0 = sK0 + S * DCH * ATT_CHUNK_BYTES;
    const uint32_t bars = sV0 + S * V_STAGE;
    const uint32_t bar_q = bars;
    auto bar_kv_full = [&](int s) { return bars + 8u * (1 + s); };
    auto bar_kv_empty = [&](int s) { return bars + 8u * (1 + S + s); };

    const int warp = threadIdx.x >> 5;
    const int q0 = blockIdx.x * ATT_BM;
    const int head = blockIdx.y;
    const int b = blockIdx.z;
    const int nkv = (p.nk + ATT_BN - 1) / ATT_BN;

    if (warp == 8 && elect_one()) {
        prefetch_tmap(&p.tmQ);
        prefetch_tmap(&p.tmK);
        prefetch_tmap(&p.tmV);
        mbar_init(bar_q, 1);
        for (int s = 0; s < S; ++s) {
            mbar_init(bar_kv_full(s), 1);
            mbar_init(bar_kv_empty(s), 8);  // one arrival per consumer warp
        }
        fence_mbar_init();
    }
    if constexpr (DCH == 1) {
        // d < DV: the V^T box has d rows, and rows d .. DV - 1 of both chunks of every stage are written here, once:
        // row d is 1.0 in the P type, the rest 0. Column d of O then accumulates the row sum of P. A row of equal
        // 16-byte units is the same under the 128-byte swizzle, and TMA never writes outside its box.
        if (p.d < DV) {
            const uint32_t one2 = F16 ? 0x3C003C00u : 0x3F803F80u;
            const int rows = DV - p.d;
            for (int i = threadIdx.x; i < 2 * S * rows * 8; i += ATT_THREADS) {  // 8 16-byte units per 128-byte row
                const int r = (i >> 3) % rows, chunk = (i >> 3) / rows;
                const uint32_t v = r == 0 ? one2 : 0u;
                *reinterpret_cast<uint4*>(smem_raw + (sV0 - raw) + chunk * V_CHUNK + (p.d + r) * 128 + (i & 7) * 16) =
                    make_uint4(v, v, v, v);
            }
            fence_proxy_async_smem();  // the tensor cores read these rows through the async proxy
        }
    }
    __syncthreads();
    pdl_wait();  // Q / K / V^T come from the preceding kernels
    pdl_launch_dependents();

    if (warp == 8) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            mbar_arrive_expect_tx(bar_q, DCH * ATT_CHUNK_BYTES);
#pragma unroll
            for (int dc = 0; dc < DCH; ++dc)
                tma_load_4d(sQ + dc * ATT_CHUNK_BYTES, &p.tmQ, bar_q, dc * 64, head, q0, b);
            for (int j = 0; j < nkv; ++j) {
                const int s = j % S;
                const uint32_t ph = (j / S) & 1;
                mbar_wait(bar_kv_empty(s), ph ^ 1u);
                if constexpr (DCH == 1) mbar_arrive_expect_tx(bar_kv_full(s), ATT_CHUNK_BYTES + 256u * p.d);  // V^T: d rows
                else mbar_arrive_expect_tx(bar_kv_full(s), DCH * ATT_CHUNK_BYTES + V_STAGE);
                const uint32_t dK = sK0 + s * DCH * ATT_CHUNK_BYTES;
                const uint32_t dV = sV0 + s * V_STAGE;
#pragma unroll
                for (int dc = 0; dc < DCH; ++dc)
                    tma_load_4d(dK + dc * ATT_CHUNK_BYTES, &p.tmK, bar_kv_full(s), dc * 64, head, j * ATT_BN, b);
                tma_load_3d(dV, &p.tmV, bar_kv_full(s), j * ATT_BN, 0, b * p.heads + head);
                tma_load_3d(dV + V_CHUNK, &p.tmV, bar_kv_full(s), j * ATT_BN + 64, 0, b * p.heads + head);
            }
        }
    } else if constexpr (DCH == 1) {
        // ============ consumer warpgroups, DV <= 64: tensor-core turns and look-ahead ============
        // At these widths the exponentials (MUFU) bound the block, not the MMAs, so the MMAs are hidden under them:
        //  - turns: a warpgroup issues its MMAs only in its turn (named barrier 1 + wg) and then hands the turn to the
        //    other warpgroup, so one warpgroup's softmax runs while the other's MMAs run;
        //  - look-ahead: S(j+1) = Q K(j+1)^T and O += P(j) V(j) are issued as two commit groups, and the max and the
        //    exponentials of S(j+1) run while PV(j) is still on the tensor cores. A warp therefore holds stage j + 1
        //    before it releases stage j, which needs a ring of two stages or more.
        // The arithmetic is the one of the DV > 64 loop below, operation for operation, except for the row sums when
        // d < DV: the tensor cores add them up in column d of O (V^T row d is all ones), which the rescale of O by
        // alpha rescales too. They add the same 16-bit P the MMA multiplies.
        static_assert(S >= 2, "the look-ahead holds two ring stages at once");
        const int wg = warp >> 2, w4 = warp & 3;
        const int lane = (int)lane_id();
        const int qc = 2 * (lane & 3);  // first of the two columns this thread holds in each 8-column group
        const float c = p.scale_log2;
        const bool sum_in_o = p.d < DV;
        // turn barriers: both warpgroups (256 threads) meet on each; warpgroup wg waits on 1 + wg, arrives on 2 - wg
        const int turn_mine = 1 + wg, turn_other = 2 - wg;
        float o[DV / 2];
#pragma unroll
        for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
        float m_run0 = -INFINITY, m_run1 = -INFINITY, l0 = 0.f, l1 = 0.f;
        float sc[64];    // S of the newest key block, then its exponentials
        uint32_t pa[32];  // P of the block whose PV product is next, in the A-operand layout of the k16 slices
        const uint32_t zero = (uint32_t)p.nk >> 31;  // nk > 0, so 0, but not a constant to the compiler
        const uint32_t qa = sQ + wg * (ATT_CHUNK_BYTES / 2);
        // S = Q K(j)^T into sc. Every wgmma count is a compile-time constant and no wgmma sits under a runtime
        // condition: that would make ptxas serialise all of them (C7519).
        auto issue_s = [&](int j) {
            const uint32_t kb = sK0 + (j % S) * ATT_CHUNK_BYTES;
#pragma unroll
            for (int ks = 0; ks < DV / 16; ++ks)
                Wgmma<ATT_BN>::ss_bf16(sc, wgmma_desc_advance_k(wgmma_desc_kmajor_sw128(qa), ks * 16),
                                       wgmma_desc_advance_k(wgmma_desc_kmajor_sw128(kb), ks * 16), 1);
            wgmma_commit();
        };
        // O += P(j) V(j), all 8 k-steps of 16 keys: keys past the end have P = 0
        auto issue_pv = [&](int j) {
            const uint32_t vb = sV0 + (j % S) * V_STAGE;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const uint64_t db = wgmma_desc_advance_k(wgmma_desc_kmajor_sw128(vb + (ks >> 2) * V_CHUNK), (ks & 3) * 16);
                const uint32_t(&a)[4] = *reinterpret_cast<const uint32_t(*)[4]>(&pa[4 * ks]);
                if constexpr (F16) Wgmma<DV>::rs_f16(o, a, db, 1);
                else Wgmma<DV>::rs_bf16(o, a, db, 1);
            }
            wgmma_commit();
        };
        // masks and exponentiates sc (key block j) in place; returns the factors O and l are rescaled by
        auto softmax = [&](int j, float& al0, float& al1) {
            const int nvalid = min(ATT_BN, p.nk - j * ATT_BN);
            if (nvalid < ATT_BN) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    if (8 * i + qc >= nvalid) sc[4 * i] = sc[4 * i + 2] = -INFINITY;
                    if (8 * i + qc + 1 >= nvalid) sc[4 * i + 1] = sc[4 * i + 3] = -INFINITY;
                }
            }
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                mx0 = fmaxf(mx0, fmaxf(sc[4 * i], sc[4 * i + 1]));
                mx1 = fmaxf(mx1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            const float mn0 = fmaxf(m_run0, mx0 * c), mn1 = fmaxf(m_run1, mx1 * c);
            al0 = fast_exp2(m_run0 - mn0);
            al1 = fast_exp2(m_run1 - mn1);
            m_run0 = mn0;
            m_run1 = mn1;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                sc[4 * i] = fast_exp2(fmaf(sc[4 * i], c, -mn0));
                sc[4 * i + 1] = fast_exp2(fmaf(sc[4 * i + 1], c, -mn0));
                sc[4 * i + 2] = fast_exp2(fmaf(sc[4 * i + 2], c, -mn1));
                sc[4 * i + 3] = fast_exp2(fmaf(sc[4 * i + 3], c, -mn1));
            }
        };
        // after PV(j) has retired: rescale O and l, round the exponentials to P(j + 1)
        auto rescale_and_pack = [&](float al0, float al1) {
            l0 *= al0;
            l1 *= al1;
#pragma unroll
            for (int i = 0; i < DV / 8; ++i) {
                o[4 * i] *= al0; o[4 * i + 1] *= al0;
                o[4 * i + 2] *= al1; o[4 * i + 3] *= al1;
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                pa[2 * i] = pack_p<F16>(sc[4 * i], sc[4 * i + 1]);
                pa[2 * i + 1] = pack_p<F16>(sc[4 * i + 2], sc[4 * i + 3]);
            }
            if (!sum_in_o) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    l0 += sum_p<F16>(pa[2 * i]);
                    l1 += sum_p<F16>(pa[2 * i + 1]);
                }
            }
        };
        float al0, al1;
        if (wg == 1) named_bar_arrive(turn_other, 256);  // warpgroup 0 takes the first turn
        mbar_wait(bar_q, 0);
        {
            const int j = 0, s = 0;
            mbar_wait(bar_kv_full(s), (j / S) & 1);
#pragma unroll
            for (int i = 0; i < 64; ++i) sc[i] = 0.f;
            named_bar_sync(turn_mine, 256);
            wgmma_fence();
            issue_s(j);
            named_bar_arrive(turn_other, 256);
            wgmma_wait<0>();
            wgmma_fence_regs(sc);
            softmax(j, al0, al1);
            rescale_and_pack(al0, al1);
        }
        for (int j = 0; j + 1 < nkv; ++j) {
            const int s = j % S, s1 = (j + 1) % S;
            mbar_wait(bar_kv_full(s1), ((j + 1) / S) & 1);  // hold stage j + 1 ...
#pragma unroll
            for (int i = 0; i < 64; ++i) sc[i] = 0.f;
            named_bar_sync(turn_mine, 256);
            wgmma_fence();
            issue_s(j + 1);
            issue_pv(j);
            named_bar_arrive(turn_other, 256);
            wgmma_wait<1>();  // S(j + 1) has landed; PV(j) may still run
            wgmma_fence_regs(sc);
            softmax(j + 1, al0, al1);
            // The exponentials are what overlaps PV(j), so they must stay ahead of the wait, but ptxas would start
            // their block with the wait, and sinks them past any branch whose other side does not read them. This
            // branch never runs (zero is 0); its use of every exponential pins them above the wait.
            if (zero) {
                float t = 0.f;
#pragma unroll
                for (int i = 0; i < 64; ++i) t += sc[i];
                p.out[0] = __float2bfloat16(t);
            }
            wgmma_wait<0>();
            wgmma_fence_regs(o);
            wgmma_fence_regs(pa);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_kv_empty(s));  // ... then release stage j
            rescale_and_pack(al0, al1);
        }
        {
            const int s = (nkv - 1) % S;
            named_bar_sync(turn_mine, 256);
            wgmma_fence();
            issue_pv(nkv - 1);
            if (wg == 0) named_bar_arrive(turn_other, 256);  // the last turn is warpgroup 1's: nothing left pending
            wgmma_wait<0>();
            wgmma_fence_regs(o);
            wgmma_fence_regs(pa);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_kv_empty(s));
        }
        // epilogue: O / l -> bf16
        if (sum_in_o) {
            // column d (a multiple of 8) is element 4 (d / 8) (+ 2 for the second row) of the quad's first lane;
            // selected with constant register indices, so O stays in registers
            const int di = p.d >> 3;
#pragma unroll
            for (int i = 0; i < DV / 8; ++i) {
                if (i == di) {
                    l0 = o[4 * i];
                    l1 = o[4 * i + 2];
                }
            }
            l0 = __shfl_sync(0xffffffffu, l0, lane & ~3);
            l1 = __shfl_sync(0xffffffffu, l1, lane & ~3);
        } else {
            l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
            l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
            l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        }
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
        const int qi0 = q0 + 64 * wg + 16 * w4 + (lane >> 2), qi1 = qi0 + 8;
        __nv_bfloat16* orow0 = p.out + ((int64_t)b * p.nq + qi0) * p.o_ld + head * p.d;
        __nv_bfloat16* orow1 = orow0 + 8 * p.o_ld;
#pragma unroll
        for (int i = 0; i < DV / 8; ++i) {
            const int col = 8 * i + qc;  // d % 8 == 0: col < d implies col + 1 < d
            if (col < p.d) {
                if (qi0 < p.nq) *reinterpret_cast<uint32_t*>(orow0 + col) = pack_bf16x2(o[4 * i] * inv0, o[4 * i + 1] * inv0);
                if (qi1 < p.nq) *reinterpret_cast<uint32_t*>(orow1 + col) = pack_bf16x2(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
            }
        }
    } else {
        // ===================== consumer warpgroups =====================
        const int wg = warp >> 2, w4 = warp & 3;
        const int lane = (int)lane_id();
        const int qc = 2 * (lane & 3);  // first of the two columns this thread holds in each 8-column group
        const float c = p.scale_log2;
        float o[DV / 2];
#pragma unroll
        for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
        // rows 16 w4 + lane / 4 (index 0) and that + 8 (index 1) of this warpgroup's 64
        float m_run0 = -INFINITY, m_run1 = -INFINITY, l0 = 0.f, l1 = 0.f;
        const uint32_t qa = sQ + wg * (ATT_CHUNK_BYTES / 2);  // rows [64 wg, 64 wg + 64) of each Q chunk
        mbar_wait(bar_q, 0);
        for (int j = 0; j < nkv; ++j) {
            const int s = j % S;
            mbar_wait(bar_kv_full(s), (j / S) & 1);
            const uint32_t kb = sK0 + s * DCH * ATT_CHUNK_BYTES;
            const uint32_t vb = sV0 + s * V_STAGE;
            float sc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) sc[i] = 0.f;
            // Every wgmma count in this loop is a compile-time constant: a wgmma under a runtime condition makes ptxas
            // serialise all of them (C7519). Channels d .. DV - 1 of Q and K are TMA zero fill and add exact zeros.
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < DV / 16; ++ks) {
                const int dc = ks >> 2, kk = (ks & 3) * 16;
                Wgmma<ATT_BN>::ss_bf16(sc, wgmma_desc_advance_k(wgmma_desc_kmajor_sw128(qa + dc * ATT_CHUNK_BYTES), kk),
                                       wgmma_desc_advance_k(wgmma_desc_kmajor_sw128(kb + dc * ATT_CHUNK_BYTES), kk), 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(sc);
            // keys past the end of the sequence (ragged last block) do not take part
            const int nvalid = min(ATT_BN, p.nk - j * ATT_BN);
            if (nvalid < ATT_BN) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    if (8 * i + qc >= nvalid) sc[4 * i] = sc[4 * i + 2] = -INFINITY;
                    if (8 * i + qc + 1 >= nvalid) sc[4 * i + 1] = sc[4 * i + 3] = -INFINITY;
                }
            }
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                mx0 = fmaxf(mx0, fmaxf(sc[4 * i], sc[4 * i + 1]));
                mx1 = fmaxf(mx1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            // running max in the exp2 domain (scale > 0), and the factor O and l are rescaled by (0 on the first block)
            const float mn0 = fmaxf(m_run0, mx0 * c), mn1 = fmaxf(m_run1, mx1 * c);
            const float al0 = fast_exp2(m_run0 - mn0), al1 = fast_exp2(m_run1 - mn1);
            m_run0 = mn0;
            m_run1 = mn1;
            l0 *= al0;
            l1 *= al1;
#pragma unroll
            for (int i = 0; i < DV / 8; ++i) {
                o[4 * i] *= al0; o[4 * i + 1] *= al0;
                o[4 * i + 2] *= al1; o[4 * i + 3] *= al1;
            }
            // P in the A-operand layout of the k16 slices: slice kk = {pa[4 kk], .., pa[4 kk + 3]}
            uint32_t pa[32];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint32_t p01 = pack_p<F16>(fast_exp2(fmaf(sc[4 * i], c, -mn0)), fast_exp2(fmaf(sc[4 * i + 1], c, -mn0)));
                const uint32_t p23 = pack_p<F16>(fast_exp2(fmaf(sc[4 * i + 2], c, -mn1)), fast_exp2(fmaf(sc[4 * i + 3], c, -mn1)));
                l0 += sum_p<F16>(p01);
                l1 += sum_p<F16>(p23);
                pa[2 * i] = p01;
                pa[2 * i + 1] = p23;
            }
            // all 8 k-steps of 16 keys, ragged block included: keys past the end have P = 0 and V^T = TMA zero fill
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const uint64_t db = wgmma_desc_advance_k(wgmma_desc_kmajor_sw128(vb + (ks >> 2) * V_CHUNK), (ks & 3) * 16);
                const uint32_t(&a)[4] = *reinterpret_cast<const uint32_t(*)[4]>(&pa[4 * ks]);
                if constexpr (F16) Wgmma<DV>::rs_f16(o, a, db, 1);
                else Wgmma<DV>::rs_bf16(o, a, db, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(o);
            wgmma_fence_regs(pa);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_kv_empty(s));  // this warp is done with the K / V^T stage
        }
        // epilogue: O / l -> bf16
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
        const int qi0 = q0 + 64 * wg + 16 * w4 + (lane >> 2), qi1 = qi0 + 8;
        __nv_bfloat16* orow0 = p.out + ((int64_t)b * p.nq + qi0) * p.o_ld + head * p.d;
        __nv_bfloat16* orow1 = orow0 + 8 * p.o_ld;
#pragma unroll
        for (int i = 0; i < DV / 8; ++i) {
            const int col = 8 * i + qc;  // d % 8 == 0: col < d implies col + 1 < d
            if (col < p.d) {
                if (qi0 < p.nq) *reinterpret_cast<uint32_t*>(orow0 + col) = pack_bf16x2(o[4 * i] * inv0, o[4 * i + 1] * inv0);
                if (qi1 < p.nq) *reinterpret_cast<uint32_t*>(orow1 + col) = pack_bf16x2(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
            }
        }
    }
}

// ---------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------
// instantiated PV widths: the head dim is rounded up to the next of these (SD-1.5: d = 40 / 80 / 160)
static constexpr int ATT_DVS[8] = {32, 48, 64, 80, 96, 128, 160, 192};

// index into ATT_DVS of the PV width a head dim d (8..192) runs at. Shared by attn_prepare and pp_attention_variant.
static int att_dv_index(int d) {
    int dvi = 0;
    while (dvi < 7 && ATT_DVS[dvi] < d) ++dvi;
    return dvi;
}

template <int DV, bool F16>
static int attn_ensure_attr() {
    static bool done[PP_MAX_DEVICES] = {};  // the attribute is per device
    int dev = 0;
    PP_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev < 0 || dev >= PP_MAX_DEVICES || !done[dev]) {
        PP_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<DV, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)att_smem_bytes(DV)));
        if (dev >= 0 && dev < PP_MAX_DEVICES) done[dev] = true;
    }
    return PP_OK;
}

// variant = 2 * (index into ATT_DVS) + vt_fp16
#define PP_ATTN_DISPATCH(FN, variant, ...)                                  \
    switch (variant) {                                                       \
        case 0: return FN<32, false>(__VA_ARGS__);                           \
        case 1: return FN<32, true>(__VA_ARGS__);                            \
        case 2: return FN<48, false>(__VA_ARGS__);                           \
        case 3: return FN<48, true>(__VA_ARGS__);                            \
        case 4: return FN<64, false>(__VA_ARGS__);                           \
        case 5: return FN<64, true>(__VA_ARGS__);                            \
        case 6: return FN<80, false>(__VA_ARGS__);                           \
        case 7: return FN<80, true>(__VA_ARGS__);                            \
        case 8: return FN<96, false>(__VA_ARGS__);                           \
        case 9: return FN<96, true>(__VA_ARGS__);                            \
        case 10: return FN<128, false>(__VA_ARGS__);                         \
        case 11: return FN<128, true>(__VA_ARGS__);                          \
        case 12: return FN<160, false>(__VA_ARGS__);                         \
        case 13: return FN<160, true>(__VA_ARGS__);                          \
        case 14: return FN<192, false>(__VA_ARGS__);                         \
        case 15: return FN<192, true>(__VA_ARGS__);                          \
    }

static int attn_ensure_attr_for(int variant) {
    PP_ATTN_DISPATCH(attn_ensure_attr, variant)
    set_last_error("attention: no kernel variant %d", variant);
    return PP_ERR_INVALID;
}

template <int DV, bool F16>
static int attn_launch_variant(const AttnLaunch& l, cudaStream_t s) {
    PP_CUDA_CHECK(launch(attn_fwd_kernel<DV, F16>, l.grid, ATT_THREADS, l.smem, s, l.p));
    return PP_OK;
}

int attn_prepare(const pp_attn_desc& d, AttnLaunch* out) {
    AttnLaunch l;
    memset(&l, 0, sizeof(l));
    AttnKParams& p = l.p;
    PP_REQUIRE(d.q && d.k && d.vt && d.out, "attention: null pointer");
    PP_REQUIRE(d.batch > 0 && d.heads > 0 && d.nq > 0 && d.nk > 0, "attention: empty problem");
    PP_REQUIRE(d.d >= 8 && d.d % 8 == 0 && d.d <= 192, "attention: head dim %d unsupported (multiple of 8, <= 192)", d.d);
    PP_REQUIRE(d.vt_ld >= d.nk && d.vt_ld % 8 == 0, "attention: vt_ld=%lld invalid", (long long)d.vt_ld);
    PP_REQUIRE(d.q_ld % 8 == 0 && d.k_ld % 8 == 0 && d.o_ld % 8 == 0, "attention: row pitches must be multiples of 8");
    PP_REQUIRE(d.q_batch_stride % 8 == 0 && d.k_batch_stride % 8 == 0, "attention: batch strides must be multiples of 8");
    PP_REQUIRE(d.o_ld >= (int64_t)d.heads * d.d, "attention: o_ld too small");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "attention: out not 16-byte aligned");
    p.batch = d.batch; p.heads = d.heads; p.d = d.d; p.nq = d.nq; p.nk = d.nk;
    const int dvi = att_dv_index(d.d);
    p.dv = ATT_DVS[dvi];
    p.scale_log2 = d.scale * 1.4426950408889634f;
    p.vt_fp16 = d.vt_fp16;
    p.out = reinterpret_cast<__nv_bfloat16*>(d.out);
    p.o_ld = d.o_ld;
    {
        uint64_t dims[4] = {(uint64_t)d.d, (uint64_t)d.heads, (uint64_t)d.nq, (uint64_t)d.batch};
        uint64_t str[3] = {(uint64_t)d.d * 2, (uint64_t)d.q_ld * 2, (uint64_t)d.q_batch_stride * 2};
        uint32_t box[4] = {64, 1, ATT_BM, 1};
        int rc = make_tmap_bf16(&p.tmQ, d.q, 4, dims, str, box, true);
        if (rc) return rc;
    }
    {
        uint64_t dims[4] = {(uint64_t)d.d, (uint64_t)d.heads, (uint64_t)d.nk, (uint64_t)d.batch};
        uint64_t str[3] = {(uint64_t)d.d * 2, (uint64_t)d.k_ld * 2, (uint64_t)d.k_batch_stride * 2};
        uint32_t box[4] = {64, 1, ATT_BN, 1};
        int rc = make_tmap_bf16(&p.tmK, d.k, 4, dims, str, box, true);
        if (rc) return rc;
    }
    {
        // dv > 64: rows d .. dv - 1 of the box lie outside the head, TMA zero-fills them. dv <= 64: the box has d rows,
        // the kernel writes the rows past it itself (the row-sum row)
        uint64_t dims[3] = {(uint64_t)d.nk, (uint64_t)d.d, (uint64_t)d.batch * d.heads};
        uint64_t str[2] = {(uint64_t)d.vt_ld * 2, (uint64_t)d.vt_ld * 2 * d.d};
        uint32_t box[3] = {64, (uint32_t)(p.dv <= 64 ? d.d : p.dv), 1};
        int rc = make_tmap_bf16(&p.tmV, d.vt, 3, dims, str, box, true);
        if (rc) return rc;
    }
    l.variant = 2 * dvi + (d.vt_fp16 ? 1 : 0);
    l.grid = dim3((unsigned)((d.nq + ATT_BM - 1) / ATT_BM), (unsigned)d.heads, (unsigned)d.batch);
    l.smem = att_smem_bytes(p.dv);
    int rc = attn_ensure_attr_for(l.variant);
    if (rc) return rc;
    *out = l;
    return PP_OK;
}

int attn_launch(const AttnLaunch& l, cudaStream_t s) {
    PP_ATTN_DISPATCH(attn_launch_variant, l.variant, l, s)
    set_last_error("attention: no kernel variant %d", l.variant);
    return PP_ERR_INVALID;
}

}  // namespace pp

extern "C" pp_status pp_attention_variant(const pp_attn_desc* d, int32_t* dv, int32_t* p_fp16) {
    if (!d || !dv || !p_fp16) {
        pp::set_last_error("pp_attention_variant: null argument");
        return pp::PP_ERR_INVALID;
    }
    if (d->d < 8 || d->d % 8 != 0 || d->d > 192) {
        pp::set_last_error("attention: head dim %d unsupported (multiple of 8, <= 192)", d->d);
        return pp::PP_ERR_INVALID;
    }
    *dv = pp::ATT_DVS[pp::att_dv_index(d->d)];
    *p_fp16 = d->vt_fp16 ? 1 : 0;
    return pp::PP_OK;
}

extern "C" pp_status pp_attention(const pp_attn_desc* d, pp_stream stream) {
    if (!d) {
        pp::set_last_error("pp_attention: null descriptor");
        return pp::PP_ERR_INVALID;
    }
    pp::AttnLaunch l;
    int rc = pp::attn_prepare(*d, &l);
    if (rc) return rc;
    return pp::attn_launch(l, reinterpret_cast<cudaStream_t>(stream));
}
