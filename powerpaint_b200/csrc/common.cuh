// Common device/host helpers for the PowerPaint hot path (sm_90a only).
//
// Everything here is a thin inline-PTX wrapper over the Hopper primitives the
// kernels use: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / commit / wait,
// the shared-memory matrix descriptor; the MMAs themselves are in wgmma.cuh).
// No CUTLASS/CuTe dependency: descriptors are built by hand; the bit layouts
// follow the PTX ISA "matrix descriptor" table of the wgmma section.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#ifndef PP_WAIT_TIMEOUT_NS
// mbarrier waits trap instead of hanging the GPU if a pipeline bug leaves a
// barrier un-arrived (wall-clock bound, checked every 256 polls).
#define PP_WAIT_TIMEOUT_NS 4000000000ull
#endif

namespace pp {

// Programmatic dependent launch (opt-in, PP_B200_PDL=1). Kernels are then launched with the programmatic-
// serialisation attribute (pp::launch below), so a kernel may become resident while its predecessor
// drains: pdl_launch_dependents() lets the successor's CTAs take freed SMs and run their prologue
// (barrier init, tensor-map prefetch); pdl_wait() blocks until the predecessor grid
// has completed and its writes are visible, and must precede the first access to global memory.
// Both are no-ops for a launch without the attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n"
        ".reg .b32 rx;\n"
        ".reg .pred px;\n"
        "elect.sync rx|px, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, px;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA / tensor core reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// non-blocking probe of the same condition
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// No report before the trap: a printf is a function call, and ptxas serialises every wgmma of a kernel that
// contains one (warning C7510), whichever warp role the call sits in. The trap surfaces as a launch error.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const uint64_t t0 = global_timer_ns();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0xFFu) == 0 && global_timer_ns() - t0 > PP_WAIT_TIMEOUT_NS) __trap();
    }
}

// ----------------------------------------------------------------------------
// TMA loads (tile mode), completing on an mbarrier in this CTA
// ----------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

// TMA stores (tile mode, bulk-group completion): shared::cta -> global, out-of-bounds parts of the box are clipped
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(src), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
// asynchronous 4-byte global -> shared copy (LDGSTS: no register, nothing to wait for until cp_async_wait_all)
__device__ __forceinline__ void cp_async_f32(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk groups have finished READING their shared-memory source (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... have completed entirely (global writes performed)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------
// wgmma: ordering of the asynchronous warpgroup MMAs, shared-memory matrix descriptor
// ----------------------------------------------------------------------------
// before the first wgmma that reads / accumulates into registers written by ordinary instructions
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed groups of this warpgroup still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(uint32_t (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// Shared-memory matrix descriptor for a K-major 16-bit operand tile whose rows are
// 128 bytes (64 elements) with the 128-byte swizzle, i.e. exactly what a TMA box with
// inner extent 64 elements + CU_TENSOR_MAP_SWIZZLE_128B writes to a 1024-byte aligned
// buffer. 8-row groups are 1024 bytes apart (SBO); LBO is unused for swizzled
// K-major layouts; layout type 1 = SWIZZLE_128B.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);  // start address  [0,14)
    d |= static_cast<uint64_t>(1024 >> 4) << 32;          // SBO = 1024 B   [32,46)
    d |= static_cast<uint64_t>(1) << 62;                  // SWIZZLE_128B   [62,64)
    return d;
}
// advance along K by `k_elems` 16-bit elements inside the 128-byte swizzle atom (k_elems*2 < 128)
__device__ __forceinline__ uint64_t wgmma_desc_advance_k(uint64_t desc, uint32_t k_elems) {
    return desc + static_cast<uint64_t>((k_elems * 2u) >> 4);
}

// ----------------------------------------------------------------------------
// small numeric helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %2, %1;" : "=r"(r) : "f"(lo), "f"(hi));
    return r;
}
// two exponentials per MUFU op: packed fp16 in, packed fp16 out
// volatile variants: the compiler keeps volatile asm statements in program order relative to each
// other, which lets a kernel fix the distance between a MUFU and the first consumer of its result
__device__ __forceinline__ float ex2_ordered(float x) {
    float y;
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_f16x2_ordered(float lo, float hi) {
    uint32_t y;
    asm volatile("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(y) : "f"(hi), "f"(lo));
    return y;
}
// 2^x on the FMA / integer pipes (no MUFU): x = n + f with n = round(x), f in [-0.5, 0.5];
// 2^f by a degree-3 minimax polynomial (max relative error 7.5e-5, below fp16 half-ulp), 2^n by
// adding n to the exponent field. Valid for x in [-120, 120]; smaller inputs are clamped (result ~ 0).
// Used to take a share of the softmax exponentials off the 16 / clk / SM MUFU pipe.
__device__ __forceinline__ float exp2_poly3(float x) {
    x = fmaxf(x, -120.f);
    const float xr = x + 12582912.f;  // 1.5 * 2^23: round(x) lands in the low mantissa bits
    const float f = x - (xr - 12582912.f);
    float p = fmaf(f, 0.0551716648f, 0.2426111251f);
    p = fmaf(p, f, 0.6932609677f);
    p = fmaf(p, f, 0.9999280572f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(xr) << 23));
}
// fp32 pairs held in one 64-bit register pair (two scalar instructions per operation on sm_90)
__device__ __forceinline__ uint64_t pack_f32x2(float lo, float hi) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ float f32x2_lo(uint64_t v) {
    float lo;
    [[maybe_unused]] float hi;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
    return lo;
}
__device__ __forceinline__ float f32x2_hi(uint64_t v) {
    [[maybe_unused]] float lo;
    float hi;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
    return hi;
}
__device__ __forceinline__ uint64_t add_f32x2(uint64_t a, uint64_t b) {
    return pack_f32x2(f32x2_lo(a) + f32x2_lo(b), f32x2_hi(a) + f32x2_hi(b));
}
__device__ __forceinline__ uint64_t sub_f32x2(uint64_t a, uint64_t b) {
    return pack_f32x2(f32x2_lo(a) - f32x2_lo(b), f32x2_hi(a) - f32x2_hi(b));
}
__device__ __forceinline__ uint64_t fma_f32x2(uint64_t a, uint64_t b, uint64_t c) {
    return pack_f32x2(fmaf(f32x2_lo(a), f32x2_lo(b), f32x2_lo(c)), fmaf(f32x2_hi(a), f32x2_hi(b), f32x2_hi(c)));
}
__device__ __forceinline__ uint32_t ex2_f16x2(uint32_t x) {
    uint32_t r;
    asm("ex2.approx.f16x2 %0, %1;" : "=r"(r) : "r"(x));
    return r;
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
// x * sigmoid(x) = h + h * tanh(h), h = x / 2: one MUFU.TANH and two FMA-pipe instructions instead of
// ex2 + an IEEE division (absolute error <= |h| * 2^-11, below bf16 output resolution)
__device__ __forceinline__ float silu_f(float x) {
    const float h = 0.5f * x;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}
// CLIP's quick_gelu: x * sigmoid(1.702 x) = h + h * tanh(0.851 x), h = x / 2
__device__ __forceinline__ float quick_gelu_f(float x) {
    const float h = 0.5f * x;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.851f * x));
    return fmaf(h, t, h);
}
// exact-erf GELU with erf from Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7, far below bf16
// output resolution): 1 rcp + 1 ex2 + a degree-5 polynomial instead of libdevice erff.
__device__ __forceinline__ float gelu_fast_f(float x) {
    const float z = x * 0.70710678118654752440f;
    const float az = fabsf(z);
    const float t = __fdividef(1.0f, fmaf(0.3275911f, az, 1.0f));
    float poly = fmaf(t, 1.061405429f, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    poly *= t;
    const float erf_abs = 1.0f - poly * __expf(-az * az);
    return 0.5f * x * (1.0f + copysignf(erf_abs, z));
}
// erf-GELU through one MUFU.TANH: 0.5 x (1 + tanh(x (c0 + c1 x^2 + c2 x^4))) with the odd inner
// polynomial refitted against the exact erf form (max abs deviation 3.0e-5 over the real line, two
// orders below bf16 output resolution; the textbook tanh form with 0.044715 is off by 4.7e-4).
// x^2 is clamped at 64, where tanh has long saturated and before the x^4 term can flip the sign.
__device__ __forceinline__ float gelu_tanh_f(float x) {
    const float x2 = fminf(x * x, 64.0f);
    const float u = x * fmaf(x2, fmaf(x2, -3.58732362e-4f, 3.70503451e-2f), 7.97458471e-1f);
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
    const float h = 0.5f * x;
    return fmaf(h, t, h);
}
__device__ __forceinline__ float gelu_erf_f(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

}  // namespace pp

// ----------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------
namespace pp {

static constexpr int PP_MAX_DEVICES = 64;  // per-device "kernel attribute set" flags

// status codes of the C ABI (see include/powerpaint_b200.h)
enum : int { PP_OK = 0, PP_ERR_INVALID = 1, PP_ERR_CUDA = 2, PP_ERR_UNSUPPORTED = 3 };

void set_last_error(const char* fmt, ...);
const char* last_error();

// Encodes a bf16 tiled tensor map (rank <= 5). dims/strides innermost first;
// strides_bytes has rank-1 entries (dimension 0 is contiguous). Returns PP_OK or sets
// the last error.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128);
// swizzle_bytes: 0 (none), 64 or 128
int make_tmap_bf16_sw(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

}  // namespace pp

#define PP_CUDA_CHECK(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            pp::set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),   \
                               __FILE__, __LINE__);                                      \
            return pp::PP_ERR_CUDA;                                                      \
        }                                                                                \
    } while (0)

namespace pp {
bool pdl_enabled();  // PP_B200_PDL=1 opts in to programmatic dependent launch (off by default, see runtime.cu)

// <<<>>> replacement that opts the launch into programmatic stream serialisation
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                          Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
}  // namespace pp

#define PP_REQUIRE(cond, ...)                   \
    do {                                        \
        if (!(cond)) {                          \
            pp::set_last_error(__VA_ARGS__);    \
            return pp::PP_ERR_INVALID;          \
        }                                       \
    } while (0)
