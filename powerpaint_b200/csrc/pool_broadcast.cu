// Global pooling of a side net's residual (`global_pool_conditions`, e.g. the SD-1.5 "shuffle" ControlNet;
// BrushNet_CA.py:936-943 and diffusers' ControlNetModel): every residual is replaced by its spatial mean, which the
// UNet then broadcast-adds. Writing the broadcast at full size keeps the UNet's consumers (the ControlNet skip adds,
// the BrushNet res2 epilogues) unchanged; `prev` lets a pooled net of a Multi-ControlNet add onto the running sum.
#include "common.cuh"
#include "ops.h"

namespace pp {

// ------------------------------------------------------------------------------------
// blockIdx.y = sample, blockIdx.x = a strip of 64 channels. 256 threads = 32 channel lanes (2 channels each, one
// bf16x2 load) x 8 pixel rows. Thread row r sums the pixels p = r, r + 8, ... in ascending order, then row 0 adds
// the 8 partial sums in row order: one fixed fp32 summation order, so the result is bit-identical run to run.
// ------------------------------------------------------------------------------------
constexpr int POOL_LANES = 32, POOL_ROWS = 8;

__global__ void __launch_bounds__(POOL_LANES * POOL_ROWS)
pool_broadcast_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* prev, __nv_bfloat16* out, int hw,
                      int C) {  // prev may equal out (each element is read, then written, by one thread): no __restrict__
    pdl_wait();
    pdl_launch_dependents();
    __shared__ float2 part[POOL_ROWS][POOL_LANES];
    __shared__ float2 mean[POOL_LANES];
    const int lane = threadIdx.x % POOL_LANES, row = threadIdx.x / POOL_LANES;
    const int c = blockIdx.x * (2 * POOL_LANES) + 2 * lane;
    const bool active = c < C;
    const int64_t base = (int64_t)blockIdx.y * hw * C + c;
    float2 s = make_float2(0.f, 0.f);
    if (active) {
        for (int p = row; p < hw; p += POOL_ROWS) {
            const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + base + (int64_t)p * C));
            s.x += v.x;
            s.y += v.y;
        }
    }
    part[row][lane] = s;
    __syncthreads();
    if (row == 0) {
        float2 t = part[0][lane];
        for (int r = 1; r < POOL_ROWS; ++r) {
            t.x += part[r][lane].x;
            t.y += part[r][lane].y;
        }
        mean[lane] = make_float2(t.x / (float)hw, t.y / (float)hw);
    }
    __syncthreads();
    if (!active) return;
    const float2 m = mean[lane];
    for (int p = row; p < hw; p += POOL_ROWS) {
        const int64_t off = base + (int64_t)p * C;
        float2 v = m;
        if (prev) {
            const float2 q = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(prev + off));
            v = make_float2(q.x + m.x, q.y + m.y);
        }
        *reinterpret_cast<__nv_bfloat162*>(out + off) = __floats2bfloat162_rn(v.x, v.y);
    }
}

int pool_broadcast_validate(const pp_pool_broadcast_desc& d) {
    PP_REQUIRE(d.x && d.out && d.batch > 0 && d.hw > 0 && d.channels > 0, "pool_broadcast: invalid arguments");
    PP_REQUIRE(d.channels % 8 == 0, "pool_broadcast: channels=%d must be a multiple of 8", d.channels);
    PP_REQUIRE(d.batch <= 65535, "pool_broadcast: at most 65535 samples (got %d)", d.batch);
    PP_REQUIRE(d.out != d.x, "pool_broadcast: out must not alias x (every block reads all pixels of its strip of x)");
    PP_REQUIRE((reinterpret_cast<uintptr_t>(d.x) | reinterpret_cast<uintptr_t>(d.out) |
                reinterpret_cast<uintptr_t>(d.prev)) % 4 == 0,
               "pool_broadcast: x, prev and out must be 4-byte aligned");
    return PP_OK;
}

int pool_broadcast_launch(const pp_pool_broadcast_desc& d, cudaStream_t s) {
    int rc = pool_broadcast_validate(d);
    if (rc) return rc;
    const dim3 grid((unsigned)((d.channels + 2 * POOL_LANES - 1) / (2 * POOL_LANES)), (unsigned)d.batch);
    PP_CUDA_CHECK(launch(pool_broadcast_kernel, grid, POOL_LANES * POOL_ROWS, 0, s,
                         reinterpret_cast<const __nv_bfloat16*>(d.x), reinterpret_cast<const __nv_bfloat16*>(d.prev),
                         reinterpret_cast<__nv_bfloat16*>(d.out), d.hw, d.channels));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

}  // namespace pp

extern "C" {
pp_status pp_pool_broadcast(const pp_pool_broadcast_desc* d, pp_stream stream) {
    if (!d) { pp::set_last_error("pp_pool_broadcast: null descriptor"); return pp::PP_ERR_INVALID; }
    return pp::pool_broadcast_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
}
