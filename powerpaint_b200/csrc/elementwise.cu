// HBM-bound glue kernels of the denoising step: fused CFG + DDIM update (+ next UNet input),
// sinusoidal timestep embedding, nearest 2x upsample, residual add, NCHW<->NHWC conversion.
#include <curand_kernel.h>  // header-only device API: Philox4x32-10 and the Box-Muller torch's CUDA randn compiles

#include "common.cuh"
#include "ops.h"

namespace pp {

// ------------------------------------------------------------------------------------
// Element li of torch's CUDA randn for one draw (pp_randn_draw, include/powerpaint_b200.h), at the draw's Philox
// offset `offset`. torch's grid-stride kernel (ATen/native/cuda/DistributionTemplates.h) gives thread t the elements
// t + threads * q, the q-th one as lane q % 4 of its (q / 4)-th curand_normal4; a state initialised (q / 4) * 4
// further along the counter makes that call its first.
// ------------------------------------------------------------------------------------
__device__ __forceinline__ float torch_randn_at(const pp_randn_draw& d, unsigned long long offset, int64_t li) {
    const int64_t q = li / d.threads;
    curandStatePhilox4_32_10_t st;
    curand_init(d.seed, (unsigned long long)(li - q * d.threads), offset + (unsigned long long)(q >> 2) * 4ull, &st);
    const float4 r = curand_normal4(&st);
    const int lane = (int)(q & 3);
    return lane == 0 ? r.x : lane == 1 ? r.y : lane == 2 ? r.z : r.w;
}

// The four channels of NHWC pixel i (row i / hw) of a step's noise, from the draw that covers the row (zero if none).
__device__ __forceinline__ void randn_nhwc(const pp_randn_draw* __restrict__ draws, int n_draws, int step, int64_t i,
                                           int hw, float nz[4]) {
    const int64_t b = i / hw, p = i - b * hw;
    for (int k = 0; k < n_draws; ++k) {
        const pp_randn_draw d = draws[k];
        if (b < d.first_row || b >= (int64_t)d.first_row + d.rows) continue;
        const unsigned long long off = d.offset0 + (unsigned long long)step * d.offset_per_step;
#pragma unroll
        for (int c = 0; c < 4; ++c) nz[c] = torch_randn_at(d, off, ((b - d.first_row) * 4 + c) * hw + p);
        return;
    }
}

static int draws_validate(const void* noise, const pp_randn_draw* draws, int32_t n_draws, const char* what) {
    PP_REQUIRE(n_draws >= 0 && (draws == nullptr) == (n_draws == 0), "%s: draws and n_draws go together", what);
    PP_REQUIRE(!(noise && draws), "%s: noise and draws are exclusive", what);
    PP_REQUIRE((reinterpret_cast<uintptr_t>(draws) & 7) == 0, "%s: draws need 8-byte alignment", what);
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Fused classifier-free guidance + DDIMScheduler.step + next-input build.
//
// Reference: `noise_pred_uncond, noise_pred_text = noise_pred.chunk(2);
//             noise_pred = uncond + guidance_scale * (text - uncond)`
//            (powerpaint/pipelines/pipeline_PowerPaint.py:1018-1020, Brushnet_CA.py:1444-1446),
//            `latents = scheduler.step(noise_pred, t, latents)` (:1023) with DDIM (eta):
//              x0 = (x - sqrt(1-a_t) eps) / sqrt(a_t)
//              x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev - sigma^2) eps + sigma * noise
//            and the next iteration's `torch.cat([latents]*2)` / `torch.cat([x, mask,
//            masked_image_latents], dim=1)` (:990,:996).
// The reference rounds to the model dtype after every elementwise op; here everything is
// fp32 in registers and rounded once when the bf16 UNet input is written.
// One thread per pixel, everything as 16-byte (eps halves, latents) / 8-byte (next input) accesses, so a
// warp touches contiguous 512 / 256-byte runs. Algorithmic bytes per pixel (CFG, fp32 eps): eps 2*16 +
// latents read 16 + write 16 + next input 2*8 = 80 B (C2: 8 x 4096 px -> 2.6 MB per step).
// ------------------------------------------------------------------------------------
__global__ void cfg_ddim_kernel(pp_cfg_ddim_desc d) {
    pdl_wait();  // inputs come from the preceding kernel
    pdl_launch_dependents();
    const int64_t total = (int64_t)d.batch * d.hw;
    const int step = d.step_idx ? *d.step_idx : 0;
    const float* cf = d.coef + (int64_t)step * 8;
    const float sa_t = cf[0], s1a_t = cf[1], sa_p = cf[2], dir_c = cf[3], sigma = cf[4];
    const float inv_sa_t = 1.0f / sa_t;
    const float gscale = d.guidance_from_coef ? cf[5] : d.guidance_scale;
    const bool eps_vec = d.eps_fp32 && d.eps_ld == 4;  // the UNet's fp32 conv_out: one 16-byte load per half
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        float eu[4], ec[4];
        if (eps_vec) {
            const float4* e = reinterpret_cast<const float4*>(d.eps);
            const float4 u = __ldg(e + i);
            const float4 c = __ldg(e + i + (d.do_cfg ? total : 0));
            eu[0] = u.x; eu[1] = u.y; eu[2] = u.z; eu[3] = u.w;
            ec[0] = c.x; ec[1] = c.y; ec[2] = c.z; ec[3] = c.w;
        } else if (d.eps_fp32) {
            const float* e = reinterpret_cast<const float*>(d.eps);
            const float* pu = e + i * d.eps_ld;
            const float* pc = e + (i + (d.do_cfg ? total : 0)) * d.eps_ld;
#pragma unroll
            for (int j = 0; j < 4; ++j) { eu[j] = pu[j]; ec[j] = pc[j]; }
        } else {
            const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(d.eps);
            const __nv_bfloat16* pu = e + i * d.eps_ld;
            const __nv_bfloat16* pc = e + (i + (d.do_cfg ? total : 0)) * d.eps_ld;
#pragma unroll
            for (int j = 0; j < 4; ++j) { eu[j] = __bfloat162float(pu[j]); ec[j] = __bfloat162float(pc[j]); }
        }
        float4 x4 = *reinterpret_cast<const float4*>(d.latents + i * 4);
        float x[4] = {x4.x, x4.y, x4.z, x4.w};
        float nz[4] = {0.f, 0.f, 0.f, 0.f};
        if (d.noise) {
            float4 n4 = *reinterpret_cast<const float4*>(d.noise + i * 4);
            nz[0] = n4.x; nz[1] = n4.y; nz[2] = n4.z; nz[3] = n4.w;
        } else if (d.draws && sigma != 0.f) {
            randn_nhwc(d.draws, d.n_draws, step, i, d.hw, nz);
        }
        float xp[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float eps = d.do_cfg ? eu[j] + gscale * (ec[j] - eu[j]) : eu[j];
            const float x0 = (x[j] - s1a_t * eps) * inv_sa_t;
            xp[j] = sa_p * x0 + dir_c * eps + sigma * nz[j];
        }
        if (d.blend_x0) {
            // 4-channel UNet: keep the known region on the noised original (pipeline_PowerPaint.py:1025-1035)
            const float a = cf[7], s1a = sqrtf(fmaxf(1.f - a * a, 0.f));
            const int64_t pix = i % d.hw;
            const float m = __ldg(d.blend_mask + pix);
            const float4 o4 = __ldg(reinterpret_cast<const float4*>(d.blend_x0) + pix);
            const float4 n4 = __ldg(reinterpret_cast<const float4*>(d.blend_noise) + i);
            const float o[4] = {o4.x, o4.y, o4.z, o4.w}, nn[4] = {n4.x, n4.y, n4.z, n4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) xp[j] = (1.f - m) * (a * o[j] + s1a * nn[j]) + m * xp[j];
        }
        *reinterpret_cast<float4*>(d.latents + i * 4) = make_float4(xp[0], xp[1], xp[2], xp[3]);
        if (d.next_in) {
            __nv_bfloat16* ni = reinterpret_cast<__nv_bfloat16*>(d.next_in);
            if (d.extra_c == 0) {
                // the constant channels (mask, masked-image latents, ...) were written once before the loop
                // and never change: only the 4 latent channels are refreshed, one 8-byte store per CFG half
                const uint2 v = make_uint2(pack_bf16x2(xp[0], xp[1]), pack_bf16x2(xp[2], xp[3]));
                for (int cpy = 0; cpy < d.n_copies; ++cpy)
                    *reinterpret_cast<uint2*>(ni + ((int64_t)cpy * total + i) * d.next_c) = v;
            } else {
                for (int cpy = 0; cpy < d.n_copies; ++cpy) {
                    __nv_bfloat16* o = ni + ((int64_t)cpy * total + i) * d.next_c;
                    for (int c = 0; c < d.next_c; ++c) {
                        float v = 0.f;
                        if (c < 4) v = xp[c];
                        else if (c - 4 < d.extra_c)
                            v = d.extra[((d.extra_per_copy ? (int64_t)cpy * total : 0) + i) * d.extra_c + (c - 4)];
                        o[c] = __float2bfloat16_rn(v);
                    }
                }
            }
        }
    }
    // the step counter is advanced by a dedicated single-thread launch (cfg_ddim_advance_kernel)
    // enqueued right after this kernel.
}

__global__ void cfg_ddim_advance_kernel(int32_t* step_idx) {
    pdl_wait();
    pdl_launch_dependents();
    *step_idx += 1;
}

int cfg_ddim_validate(const pp_cfg_ddim_desc& d) {
    PP_REQUIRE(d.eps && d.latents && d.coef, "cfg_ddim: null pointer");
    PP_REQUIRE(d.batch > 0 && d.hw > 0, "cfg_ddim: empty input");
    PP_REQUIRE(d.eps_ld >= 4, "cfg_ddim: eps_ld must be >= 4");
    PP_REQUIRE(!d.advance_step || d.step_idx, "cfg_ddim: advance_step needs step_idx");
    PP_REQUIRE((d.blend_x0 == nullptr) == (d.blend_mask == nullptr) && (d.blend_x0 == nullptr) == (d.blend_noise == nullptr),
               "cfg_ddim: blend_x0 / blend_mask / blend_noise go together");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.latents) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.noise) & 15) == 0,
               "cfg_ddim: latents / noise need 16-byte alignment");
    PP_REQUIRE(!(d.eps_fp32 && d.eps_ld == 4) || (reinterpret_cast<uintptr_t>(d.eps) & 15) == 0,
               "cfg_ddim: fp32 eps with eps_ld 4 needs 16-byte alignment");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.blend_x0) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.blend_noise) & 15) == 0,
               "cfg_ddim: blend_x0 / blend_noise need 16-byte alignment");
    if (int rc = draws_validate(d.noise, d.draws, d.n_draws, "cfg_ddim")) return rc;
    if (d.next_in) {
        PP_REQUIRE(d.next_c >= 4 && d.n_copies >= 1, "cfg_ddim: next_in needs next_c >= 4, n_copies >= 1");
        PP_REQUIRE(d.extra_c == 0 || d.extra, "cfg_ddim: extra_c without extra");
        PP_REQUIRE(4 + d.extra_c <= d.next_c, "cfg_ddim: next_c too small for 4 + extra_c");
        PP_REQUIRE(d.next_c % 4 == 0 && (reinterpret_cast<uintptr_t>(d.next_in) & 7) == 0,
                   "cfg_ddim: next_in needs next_c %% 4 == 0 and 8-byte alignment");
    }
    return PP_OK;
}

int cfg_ddim_launch(const pp_cfg_ddim_desc& d, cudaStream_t s) {
    int rc = cfg_ddim_validate(d);
    if (rc) return rc;
    const int64_t total = (int64_t)d.batch * d.hw;
    const int threads = 128;
    const int blocks = (int)std::min<int64_t>((total + threads - 1) / threads, 132 * 8);
    PP_CUDA_CHECK(launch(cfg_ddim_kernel, blocks, threads, 0, s, d));
    PP_CUDA_CHECK(cudaGetLastError());
    if (d.advance_step) {
        PP_CUDA_CHECK(launch(cfg_ddim_advance_kernel, 1, 1, 0, s, d.step_idx));
        PP_CUDA_CHECK(cudaGetLastError());
    }
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Fused CFG + UniPCMultistepScheduler.step (order-2 bh2 predictor-corrector in x0 space; see
// include/powerpaint_b200.h for the folded per-step scalars) + next-input refresh. One thread per pixel,
// 16-byte accesses; state (last corrected sample, the two previous x0 predictions) stays fp32 in HBM.
// Algorithmic bytes per pixel (CFG): eps 32 + 4 state reads x 16 + 4 state writes x 16 + next input 16 = 176 B.
// ------------------------------------------------------------------------------------
__global__ void unipc_step_kernel(pp_unipc_desc d) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)d.batch * d.hw;
    const int step = d.step_idx ? *d.step_idx : 0;
    const float gscale = d.coef[(int64_t)step * 8 + 5];
    const float* u = d.ucoef + (int64_t)step * 12;
    const float u0 = u[0], u1 = u[1], use_c = u[2], u3 = u[3], u4 = u[4], u5 = u[5], u6 = u[6], u7 = u[7], u8 = u[8], u9 = u[9];
    const bool eps_vec = d.eps_fp32 && d.eps_ld == 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        float eu[4], ec[4];
        if (eps_vec) {
            const float4* e = reinterpret_cast<const float4*>(d.eps);
            const float4 a = __ldg(e + i), c = __ldg(e + i + (d.do_cfg ? total : 0));
            eu[0] = a.x; eu[1] = a.y; eu[2] = a.z; eu[3] = a.w;
            ec[0] = c.x; ec[1] = c.y; ec[2] = c.z; ec[3] = c.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t iu = i * d.eps_ld + j, ic = (i + (d.do_cfg ? total : 0)) * d.eps_ld + j;
                eu[j] = d.eps_fp32 ? reinterpret_cast<const float*>(d.eps)[iu]
                                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(d.eps)[iu]);
                ec[j] = d.eps_fp32 ? reinterpret_cast<const float*>(d.eps)[ic]
                                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(d.eps)[ic]);
            }
        }
        const float4 x4 = *reinterpret_cast<const float4*>(d.latents + i * 4);
        const float4 l4 = *reinterpret_cast<const float4*>(d.last_sample + i * 4);
        const float4 a4 = *reinterpret_cast<const float4*>(d.m1 + i * 4);
        const float4 b4 = *reinterpret_cast<const float4*>(d.m2 + i * 4);
        const float x[4] = {x4.x, x4.y, x4.z, x4.w}, ls[4] = {l4.x, l4.y, l4.z, l4.w};
        const float m1[4] = {a4.x, a4.y, a4.z, a4.w}, m2[4] = {b4.x, b4.y, b4.z, b4.w};
        float mt[4], xc[4], xn[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float eps = d.do_cfg ? eu[j] + gscale * (ec[j] - eu[j]) : eu[j];
            mt[j] = u0 * x[j] + u1 * eps;
            xc[j] = use_c != 0.f ? u3 * ls[j] + u4 * m1[j] + u5 * m2[j] + u6 * mt[j] : x[j];
            xn[j] = u7 * xc[j] + u8 * mt[j] + u9 * m1[j];
        }
        *reinterpret_cast<float4*>(d.last_sample + i * 4) = make_float4(xc[0], xc[1], xc[2], xc[3]);
        *reinterpret_cast<float4*>(d.m2 + i * 4) = a4;
        *reinterpret_cast<float4*>(d.m1 + i * 4) = make_float4(mt[0], mt[1], mt[2], mt[3]);
        *reinterpret_cast<float4*>(d.latents + i * 4) = make_float4(xn[0], xn[1], xn[2], xn[3]);
        if (d.next_in) {
            __nv_bfloat16* ni = reinterpret_cast<__nv_bfloat16*>(d.next_in);
            const uint2 v = make_uint2(pack_bf16x2(xn[0], xn[1]), pack_bf16x2(xn[2], xn[3]));
            for (int cpy = 0; cpy < d.n_copies; ++cpy)
                *reinterpret_cast<uint2*>(ni + ((int64_t)cpy * total + i) * d.next_c) = v;
        }
    }
}

int unipc_validate(const pp_unipc_desc& d) {
    PP_REQUIRE(d.eps && d.latents && d.last_sample && d.m1 && d.m2 && d.coef && d.ucoef, "unipc: null pointer");
    PP_REQUIRE(d.batch > 0 && d.hw > 0 && d.eps_ld >= 4, "unipc: invalid shape");
    PP_REQUIRE(!d.advance_step || d.step_idx, "unipc: advance_step needs step_idx");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.latents) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.last_sample) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(d.m1) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.m2) & 15) == 0,
               "unipc: latents / last_sample / m1 / m2 need 16-byte alignment");
    PP_REQUIRE(!(d.eps_fp32 && d.eps_ld == 4) || (reinterpret_cast<uintptr_t>(d.eps) & 15) == 0,
               "unipc: fp32 eps with eps_ld 4 needs 16-byte alignment");
    if (d.next_in)
        PP_REQUIRE(d.next_c >= 4 && d.next_c % 4 == 0 && d.n_copies >= 1 && (reinterpret_cast<uintptr_t>(d.next_in) & 7) == 0,
                   "unipc: next_in needs next_c %% 4 == 0, n_copies >= 1 and 8-byte alignment");
    return PP_OK;
}

int unipc_launch(const pp_unipc_desc& d, cudaStream_t s) {
    int rc = unipc_validate(d);
    if (rc) return rc;
    const int64_t total = (int64_t)d.batch * d.hw;
    const int blocks = (int)std::min<int64_t>((total + 127) / 128, 132 * 8);
    PP_CUDA_CHECK(launch(unipc_step_kernel, blocks, 128, 0, s, d));
    PP_CUDA_CHECK(cudaGetLastError());
    if (d.advance_step) {
        PP_CUDA_CHECK(launch(cfg_ddim_advance_kernel, 1, 1, 0, s, d.step_idx));
        PP_CUDA_CHECK(cudaGetLastError());
    }
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Fused CFG + one step of DPMSolverMultistepScheduler (dpmsolver++ / sde-dpmsolver++, order 1 or 2) or
// Euler / Euler-ancestral + next-input refresh. All of them are linear in (x, eps, previous x0 prediction,
// noise), so the host folds each step into one 8-float row (include/powerpaint_b200.h, pp_solver_desc).
// One thread per pixel, 16-byte accesses. Algorithmic bytes per pixel (CFG, fp32 eps): eps 32 + latents 16 + 16 +
// m1 16 + 16 + next input 2 x 8 = 112 B; + 16 B of noise for the SDE / ancestral variants, or none when the
// noise is drawn in the kernel (pp_randn_draw: four Philox4x32-10 evaluations and Box-Muller pairs per pixel).
// ------------------------------------------------------------------------------------
__global__ void solver_step_kernel(pp_solver_desc d) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)d.batch * d.hw;
    const int step = d.step_idx ? *d.step_idx : 0;
    const float gscale = d.coef[(int64_t)step * 8 + 5];
    const float* r = d.scoef + (int64_t)step * 8;
    const float r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3], r4 = r[4], r5 = r[5], r6 = r[6];
    const bool eps_vec = d.eps_fp32 && d.eps_ld == 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        float eu[4], ec[4];
        if (eps_vec) {
            const float4* e = reinterpret_cast<const float4*>(d.eps);
            const float4 a = __ldg(e + i), c = __ldg(e + i + (d.do_cfg ? total : 0));
            eu[0] = a.x; eu[1] = a.y; eu[2] = a.z; eu[3] = a.w;
            ec[0] = c.x; ec[1] = c.y; ec[2] = c.z; ec[3] = c.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t iu = i * d.eps_ld + j, ic = (i + (d.do_cfg ? total : 0)) * d.eps_ld + j;
                eu[j] = d.eps_fp32 ? reinterpret_cast<const float*>(d.eps)[iu]
                                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(d.eps)[iu]);
                ec[j] = d.eps_fp32 ? reinterpret_cast<const float*>(d.eps)[ic]
                                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(d.eps)[ic]);
            }
        }
        const float4 x4 = *reinterpret_cast<const float4*>(d.latents + i * 4);
        const float4 a4 = *reinterpret_cast<const float4*>(d.m1 + i * 4);
        float4 n4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (d.noise) n4 = __ldg(reinterpret_cast<const float4*>(d.noise) + i);
        const float x[4] = {x4.x, x4.y, x4.z, x4.w}, m1[4] = {a4.x, a4.y, a4.z, a4.w};
        float nz[4] = {n4.x, n4.y, n4.z, n4.w};
        if (d.draws && r5 != 0.f) randn_nhwc(d.draws, d.n_draws, step, i, d.hw, nz);
        float mt[4], xn[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float eps = d.do_cfg ? eu[j] + gscale * (ec[j] - eu[j]) : eu[j];
            mt[j] = r0 * x[j] + r1 * eps;
            xn[j] = r2 * x[j] + r3 * mt[j] + r4 * m1[j] + r5 * nz[j];
        }
        *reinterpret_cast<float4*>(d.m1 + i * 4) = make_float4(mt[0], mt[1], mt[2], mt[3]);
        *reinterpret_cast<float4*>(d.latents + i * 4) = make_float4(xn[0], xn[1], xn[2], xn[3]);
        if (d.next_in) {
            __nv_bfloat16* ni = reinterpret_cast<__nv_bfloat16*>(d.next_in);
            const uint2 v = make_uint2(pack_bf16x2(r6 * xn[0], r6 * xn[1]), pack_bf16x2(r6 * xn[2], r6 * xn[3]));
            for (int cpy = 0; cpy < d.n_copies; ++cpy)
                *reinterpret_cast<uint2*>(ni + ((int64_t)cpy * total + i) * d.next_c) = v;
        }
    }
}

int solver_validate(const pp_solver_desc& d) {
    PP_REQUIRE(d.eps && d.latents && d.m1 && d.coef && d.scoef, "solver: null pointer");
    PP_REQUIRE(d.batch > 0 && d.hw > 0 && d.eps_ld >= 4, "solver: invalid shape");
    PP_REQUIRE(!d.advance_step || d.step_idx, "solver: advance_step needs step_idx");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.latents) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.m1) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(d.noise) & 15) == 0,
               "solver: latents / m1 / noise need 16-byte alignment");
    PP_REQUIRE(!(d.eps_fp32 && d.eps_ld == 4) || (reinterpret_cast<uintptr_t>(d.eps) & 15) == 0,
               "solver: fp32 eps with eps_ld 4 needs 16-byte alignment");
    if (int rc = draws_validate(d.noise, d.draws, d.n_draws, "solver")) return rc;
    if (d.next_in)
        PP_REQUIRE(d.next_c >= 4 && d.next_c % 4 == 0 && d.n_copies >= 1 && (reinterpret_cast<uintptr_t>(d.next_in) & 7) == 0,
                   "solver: next_in needs next_c %% 4 == 0, n_copies >= 1 and 8-byte alignment");
    return PP_OK;
}

int solver_launch(const pp_solver_desc& d, cudaStream_t s) {
    int rc = solver_validate(d);
    if (rc) return rc;
    const int64_t total = (int64_t)d.batch * d.hw;
    const int blocks = (int)std::min<int64_t>((total + 127) / 128, 132 * 8);
    PP_CUDA_CHECK(launch(solver_step_kernel, blocks, 128, 0, s, d));
    PP_CUDA_CHECK(cudaGetLastError());
    if (d.advance_step) {
        PP_CUDA_CHECK(launch(cfg_ddim_advance_kernel, 1, 1, 0, s, d.step_idx));
        PP_CUDA_CHECK(cudaGetLastError());
    }
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Fused CFG + one step of PNDMScheduler with skip_prk_steps (PLMS) + 4-channel blend + next-input refresh.
// Every PLMS step is linear in (x, cur_sample, eps, the earlier eps in the history ring), so the host folds it into
// one 8-float row (include/powerpaint_b200.h, pp_plms_desc) that already names the physical ring slots: the kernel
// never shifts history. A weight of exactly zero skips its load (uniform per launch), so a ring slot or cur_sample
// that has never been written is never read. One thread per pixel, 16-byte accesses. Algorithmic bytes per pixel
// (CFG, fp32 eps, 4-entry AB step): eps 32 + latents 16 + 16 + ring 3 x 16 + 16 + next input 2 x 8 = 144 B; the
// Heun restart (counter 1) reads cur_sample and one slot instead.
// ------------------------------------------------------------------------------------
__global__ void plms_step_kernel(pp_plms_desc d) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)d.batch * d.hw;
    const int step = d.step_idx ? *d.step_idx : 0;
    const float* cf = d.coef + (int64_t)step * 8;
    const float gscale = cf[5];
    const float* r = d.pcoef + (int64_t)step * 8;
    const float wx = r[0], wc = r[1], we = r[2];
    const float wh[3] = {r[3], r[4], r[5]};
    const int slot = (int)r[6];  // ring slot the new eps goes to, -1 = none
    const bool save_cur = r[7] != 0.f;
    const int64_t slot_stride = total * 4;
    const bool eps_vec = d.eps_fp32 && d.eps_ld == 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        float eu[4], ec[4];
        if (eps_vec) {
            const float4* e = reinterpret_cast<const float4*>(d.eps);
            const float4 a = __ldg(e + i), c = __ldg(e + i + (d.do_cfg ? total : 0));
            eu[0] = a.x; eu[1] = a.y; eu[2] = a.z; eu[3] = a.w;
            ec[0] = c.x; ec[1] = c.y; ec[2] = c.z; ec[3] = c.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t iu = i * d.eps_ld + j, ic = (i + (d.do_cfg ? total : 0)) * d.eps_ld + j;
                eu[j] = d.eps_fp32 ? reinterpret_cast<const float*>(d.eps)[iu]
                                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(d.eps)[iu]);
                ec[j] = d.eps_fp32 ? reinterpret_cast<const float*>(d.eps)[ic]
                                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(d.eps)[ic]);
            }
        }
        const float4 x4 = *reinterpret_cast<const float4*>(d.latents + i * 4);
        const float x[4] = {x4.x, x4.y, x4.z, x4.w};
        float eps[4], xn[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            eps[j] = d.do_cfg ? eu[j] + gscale * (ec[j] - eu[j]) : eu[j];
            xn[j] = we * eps[j];
        }
        if (wx != 0.f) {
#pragma unroll
            for (int j = 0; j < 4; ++j) xn[j] += wx * x[j];
        }
        if (wc != 0.f) {
            const float4 c4 = *reinterpret_cast<const float4*>(d.cur_sample + i * 4);
            xn[0] += wc * c4.x; xn[1] += wc * c4.y; xn[2] += wc * c4.z; xn[3] += wc * c4.w;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (wh[k] != 0.f) {
                const float4 h4 = *reinterpret_cast<const float4*>(d.ets + k * slot_stride + i * 4);
                xn[0] += wh[k] * h4.x; xn[1] += wh[k] * h4.y; xn[2] += wh[k] * h4.z; xn[3] += wh[k] * h4.w;
            }
        }
        // history writes after every read of this pixel: the new eps may replace the oldest entry this step read
        if (save_cur) *reinterpret_cast<float4*>(d.cur_sample + i * 4) = x4;
        if (slot >= 0)
            *reinterpret_cast<float4*>(d.ets + slot * slot_stride + i * 4) = make_float4(eps[0], eps[1], eps[2], eps[3]);
        if (d.blend_x0) {
            // 4-channel UNet: keep the known region on the noised original (pipeline_PowerPaint.py:1025-1035)
            const float a = cf[7], s1a = sqrtf(fmaxf(1.f - a * a, 0.f));
            const int64_t pix = i % d.hw;
            const float m = __ldg(d.blend_mask + pix);
            const float4 o4 = __ldg(reinterpret_cast<const float4*>(d.blend_x0) + pix);
            const float4 n4 = __ldg(reinterpret_cast<const float4*>(d.blend_noise) + i);
            const float o[4] = {o4.x, o4.y, o4.z, o4.w}, nn[4] = {n4.x, n4.y, n4.z, n4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) xn[j] = (1.f - m) * (a * o[j] + s1a * nn[j]) + m * xn[j];
        }
        *reinterpret_cast<float4*>(d.latents + i * 4) = make_float4(xn[0], xn[1], xn[2], xn[3]);
        if (d.next_in) {
            __nv_bfloat16* ni = reinterpret_cast<__nv_bfloat16*>(d.next_in);
            const uint2 v = make_uint2(pack_bf16x2(xn[0], xn[1]), pack_bf16x2(xn[2], xn[3]));
            for (int cpy = 0; cpy < d.n_copies; ++cpy)
                *reinterpret_cast<uint2*>(ni + ((int64_t)cpy * total + i) * d.next_c) = v;
        }
    }
}

int plms_validate(const pp_plms_desc& d) {
    PP_REQUIRE(d.eps && d.latents && d.cur_sample && d.ets && d.coef && d.pcoef, "plms: null pointer");
    PP_REQUIRE(d.batch > 0 && d.hw > 0 && d.eps_ld >= 4, "plms: invalid shape");
    PP_REQUIRE(!d.advance_step || d.step_idx, "plms: advance_step needs step_idx");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.latents) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.cur_sample) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(d.ets) & 15) == 0,
               "plms: latents / cur_sample / ets need 16-byte alignment");
    PP_REQUIRE(!(d.eps_fp32 && d.eps_ld == 4) || (reinterpret_cast<uintptr_t>(d.eps) & 15) == 0,
               "plms: fp32 eps with eps_ld 4 needs 16-byte alignment");
    PP_REQUIRE((d.blend_x0 == nullptr) == (d.blend_mask == nullptr) && (d.blend_x0 == nullptr) == (d.blend_noise == nullptr),
               "plms: blend_x0 / blend_mask / blend_noise go together");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.blend_x0) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.blend_noise) & 15) == 0,
               "plms: blend_x0 / blend_noise need 16-byte alignment");
    if (d.next_in)
        PP_REQUIRE(d.next_c >= 4 && d.next_c % 4 == 0 && d.n_copies >= 1 && (reinterpret_cast<uintptr_t>(d.next_in) & 7) == 0,
                   "plms: next_in needs next_c %% 4 == 0, n_copies >= 1 and 8-byte alignment");
    return PP_OK;
}

int plms_launch(const pp_plms_desc& d, cudaStream_t s) {
    int rc = plms_validate(d);
    if (rc) return rc;
    const int64_t total = (int64_t)d.batch * d.hw;
    const int blocks = (int)std::min<int64_t>((total + 127) / 128, 132 * 8);
    PP_CUDA_CHECK(launch(plms_step_kernel, blocks, 128, 0, s, d));
    PP_CUDA_CHECK(cudaGetLastError());
    if (d.advance_step) {
        PP_CUDA_CHECK(launch(cfg_ddim_advance_kernel, 1, 1, 0, s, d.step_idx));
        PP_CUDA_CHECK(cudaGetLastError());
    }
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0)
// (powerpaint/models/unet_2d_condition.py:914-938): emb = [cos(t f_i), sin(t f_i)],
// f_i = exp(-ln(10000) i / half).
// ------------------------------------------------------------------------------------
__global__ void time_embed_kernel(const float* __restrict__ timesteps, const int32_t* __restrict__ step_idx,
                                  __nv_bfloat16* __restrict__ out, int batch, int dim) {
    pdl_wait();  // inputs come from the preceding kernel
    pdl_launch_dependents();
    const int half = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= batch * half) return;
    const int b = i / half, k = i % half;
    const float t = step_idx ? timesteps[*step_idx] : timesteps[b];
    const float f = expf(-9.210340371976184f * (float)k / (float)half);
    const float a = t * f;
    out[(int64_t)b * dim + k] = __float2bfloat16_rn(cosf(a));
    out[(int64_t)b * dim + half + k] = __float2bfloat16_rn(sinf(a));
}

int time_embed_launch(const float* timesteps, const int32_t* step_idx, void* out, int batch, int dim,
                      cudaStream_t s) {
    PP_REQUIRE(timesteps && out, "time_embed: null pointer");
    PP_REQUIRE(batch > 0 && dim > 0 && dim % 2 == 0, "time_embed: batch=%d dim=%d invalid", batch, dim);
    const int n = batch * dim / 2;
    PP_CUDA_CHECK(launch(time_embed_kernel, (n + 127) / 128, 128, 0, s, timesteps, step_idx,
                                                       reinterpret_cast<__nv_bfloat16*>(out), batch, dim));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Upsample2D's F.interpolate(mode="nearest") on NHWC bf16: scale_factor=2.0, or an explicit output
// size when the latent is not a multiple of 8 (unet_2d_condition.py:1120-1126,1311-1312). Source index
// as in PyTorch's nearest kernel: min(floor(dst * (float)in / out), in - 1).
// ------------------------------------------------------------------------------------
__global__ void upsample_nearest_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int nb, int h, int w,
                                        int cv, int ho, int wo, float sy, float sx, int exact2x) {
    pdl_wait();  // inputs come from the preceding kernel
    pdl_launch_dependents();
    const int64_t total = (int64_t)nb * ho * wo * cv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cv);
        int64_t p = i / cv;
        const int ox = (int)(p % wo); p /= wo;
        const int oy = (int)(p % ho);
        const int n = (int)(p / ho);
        const int iy = exact2x ? (oy >> 1) : min((int)floorf((float)oy * sy), h - 1);
        const int ix = exact2x ? (ox >> 1) : min((int)floorf((float)ox * sx), w - 1);
        y[i] = __ldg(&x[(((int64_t)n * h + iy) * w + ix) * cv + c]);
    }
}

int upsample_nearest_launch(const void* x, void* y, int nb, int h, int w, int c, int ho, int wo, cudaStream_t s) {
    PP_REQUIRE(x && y, "upsample: null pointer");
    PP_REQUIRE(nb > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && ho > 0 && wo > 0, "upsample: bad shape");
    const int64_t total = (int64_t)nb * ho * wo * (c / 8);
    const int blocks = (int)std::min<int64_t>((total + 255) / 256, 132 * 16);
    const int exact = (ho == 2 * h && wo == 2 * w) ? 1 : 0;
    PP_CUDA_CHECK(launch(upsample_nearest_kernel, blocks, 256, 0, s, reinterpret_cast<const uint4*>(x),
                         reinterpret_cast<uint4*>(y), nb, h, w, c / 8, ho, wo, (float)h / (float)ho,
                         (float)w / (float)wo, exact));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

// y = a + b (bf16), ControlNet skip residuals (`down_block_res_samples += residuals`,
// powerpaint/models/unet_2d_condition.py:1263-1272).
__global__ void add_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ y,
                           int64_t nvec) {
    pdl_wait();  // inputs come from the preceding kernel
    pdl_launch_dependents();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
         i += (int64_t)gridDim.x * blockDim.x) {
        uint4 p = __ldg(&a[i]), q = __ldg(&b[i]);
        uint4 o;
        o.x = pack_bf16x2(bf16_lo(p.x) + bf16_lo(q.x), bf16_hi(p.x) + bf16_hi(q.x));
        o.y = pack_bf16x2(bf16_lo(p.y) + bf16_lo(q.y), bf16_hi(p.y) + bf16_hi(q.y));
        o.z = pack_bf16x2(bf16_lo(p.z) + bf16_lo(q.z), bf16_hi(p.z) + bf16_hi(q.z));
        o.w = pack_bf16x2(bf16_lo(p.w) + bf16_lo(q.w), bf16_hi(p.w) + bf16_hi(q.w));
        y[i] = o;
    }
}

int add_launch(const void* a, const void* b, void* y, int64_t n, cudaStream_t s) {
    PP_REQUIRE(a && b && y, "add: null pointer");
    PP_REQUIRE(n > 0 && n % 8 == 0, "add: n=%lld must be a positive multiple of 8", (long long)n);
    const int64_t nvec = n / 8;
    const int blocks = (int)std::min<int64_t>((nvec + 255) / 256, 132 * 16);
    PP_CUDA_CHECK(launch(add_kernel, blocks, 256, 0, s, reinterpret_cast<const uint4*>(a), reinterpret_cast<const uint4*>(b),
                                      reinterpret_cast<uint4*>(y), nvec));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// Layout conversion at the boundary (the reference API is NCHW; the engine is NHWC bf16).
// Tile-transposed through shared memory so both sides are coalesced.
// ------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int c, int hw,
                                    int c_pad) {
    pdl_wait();  // inputs come from the preceding kernel
    pdl_launch_dependents();
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int cc = c0 + j, p = p0 + threadIdx.x;
        tile[j][threadIdx.x] = (cc < c && p < hw) ? x[((int64_t)n * c + cc) * hw + p] : 0.f;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int p = p0 + j, cc = c0 + threadIdx.x;
        if (p < hw && cc < c_pad) y[((int64_t)n * hw + p) * c_pad + cc] = __float2bfloat16_rn(tile[threadIdx.x][j]);
    }
}

int nchw_to_nhwc_launch(const float* x, void* y, int nb, int c, int hw, int c_pad, cudaStream_t s) {
    PP_REQUIRE(x && y, "nchw_to_nhwc: null pointer");
    PP_REQUIRE(nb > 0 && c > 0 && hw > 0 && c_pad >= c, "nchw_to_nhwc: bad shape");
    dim3 grid((hw + 31) / 32, (c_pad + 31) / 32, nb);
    PP_CUDA_CHECK(launch(nchw_to_nhwc_kernel, grid, dim3(32, 8), 0, s, x, reinterpret_cast<__nv_bfloat16*>(y), c, hw, c_pad));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

__global__ void nhwc_to_nchw_kernel(const void* __restrict__ x, int x_is_fp32, float* __restrict__ y, int c,
                                    int hw, int c_ld) {
    pdl_wait();  // inputs come from the preceding kernel
    pdl_launch_dependents();
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int p = p0 + j, cc = c0 + threadIdx.x;
        float v = 0.f;
        if (p < hw && cc < c) {
            const int64_t idx = ((int64_t)n * hw + p) * c_ld + cc;
            v = x_is_fp32 ? reinterpret_cast<const float*>(x)[idx]
                          : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(x)[idx]);
        }
        tile[j][threadIdx.x] = v;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int cc = c0 + j, p = p0 + threadIdx.x;
        if (cc < c && p < hw) y[((int64_t)n * c + cc) * hw + p] = tile[threadIdx.x][j];
    }
}

int nhwc_to_nchw_launch(const void* x, int x_is_fp32, float* y, int nb, int c, int hw, int c_ld,
                        cudaStream_t s) {
    PP_REQUIRE(x && y, "nhwc_to_nchw: null pointer");
    PP_REQUIRE(nb > 0 && c > 0 && hw > 0 && c_ld >= c, "nhwc_to_nchw: bad shape");
    dim3 grid((hw + 31) / 32, (c + 31) / 32, nb);
    PP_CUDA_CHECK(launch(nhwc_to_nchw_kernel, grid, dim3(32, 8), 0, s, x, x_is_fp32, y, c, hw, c_ld));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

}  // namespace pp

extern "C" {
pp_status pp_upsample2x(const void* x, void* y, int32_t nb, int32_t h, int32_t w, int32_t c, pp_stream s) {
    return pp::upsample_nearest_launch(x, y, nb, h, w, c, 2 * h, 2 * w, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_upsample_nearest(const void* x, void* y, int32_t nb, int32_t h, int32_t w, int32_t c, int32_t ho,
                              int32_t wo, pp_stream s) {
    return pp::upsample_nearest_launch(x, y, nb, h, w, c, ho, wo, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_add(const void* a, const void* b, void* y, int64_t n, pp_stream s) {
    return pp::add_launch(a, b, y, n, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_time_embed(const float* timesteps, const int32_t* step_idx, void* out, int32_t batch, int32_t dim,
                        pp_stream s) {
    return pp::time_embed_launch(timesteps, step_idx, out, batch, dim, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_nchw_to_nhwc(const float* x, void* y, int32_t nb, int32_t c, int32_t hw, int32_t c_pad,
                          pp_stream s) {
    return pp::nchw_to_nhwc_launch(x, y, nb, c, hw, c_pad, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_nhwc_to_nchw(const void* x, int32_t x_is_fp32, float* y, int32_t nb, int32_t c, int32_t hw,
                          int32_t c_ld, pp_stream s) {
    return pp::nhwc_to_nchw_launch(x, x_is_fp32, y, nb, c, hw, c_ld, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_unipc_step(const pp_unipc_desc* d, pp_stream s) {
    if (!d) { pp::set_last_error("pp_unipc_step: null descriptor"); return pp::PP_ERR_INVALID; }
    return pp::unipc_launch(*d, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_solver_step(const pp_solver_desc* d, pp_stream s) {
    if (!d) { pp::set_last_error("pp_solver_step: null descriptor"); return pp::PP_ERR_INVALID; }
    return pp::solver_launch(*d, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_plms_step(const pp_plms_desc* d, pp_stream s) {
    if (!d) { pp::set_last_error("pp_plms_step: null descriptor"); return pp::PP_ERR_INVALID; }
    return pp::plms_launch(*d, reinterpret_cast<cudaStream_t>(s));
}
pp_status pp_cfg_ddim_step(const pp_cfg_ddim_desc* d, pp_stream s) {
    if (!d) { pp::set_last_error("pp_cfg_ddim_step: null descriptor"); return pp::PP_ERR_INVALID; }
    return pp::cfg_ddim_launch(*d, reinterpret_cast<cudaStream_t>(s));
}
}
