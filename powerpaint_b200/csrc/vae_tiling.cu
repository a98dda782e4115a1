// Tiled VAE encode / decode (diffusers AutoencoderKL.enable_tiling; the reference ControlNet pipeline's
// enable_vae_tiling, pipeline_PowerPaint_ControlNet.py:341-356): the window copy that gathers tiles out of the
// canvas and assembles the cropped tiles into the output, and the in-place seam blend of one tile with its upper
// and left neighbours. Both are memory-bound and touch a few MB per tile.
#include "common.cuh"
#include "ops.h"

namespace pp {

// ------------------------------------------------------------------------------------
// blockIdx.y = window; the x-blocks stride over its pixels, one pixel (all channels) per thread iteration.
// ------------------------------------------------------------------------------------
template <typename T>
__global__ void window_copy_kernel(const T* __restrict__ src, T* __restrict__ dst, int channels, int64_t src_pix,
                                   int64_t dst_pix, const pp_window* __restrict__ windows) {
    pdl_wait();
    pdl_launch_dependents();
    const pp_window wdw = windows[blockIdx.y];
    const int64_t n = (int64_t)wdw.rows * wdw.cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = i / wdw.cols, x = i - y * wdw.cols;
        const T* s = src + wdw.src_off + y * wdw.src_row + x * src_pix;
        T* d = dst + wdw.dst_off + y * wdw.dst_row + x * dst_pix;
        for (int c = 0; c < channels; ++c) d[c] = s[c];
    }
}

int window_copy_validate(const void* src, void* dst, int elem_bytes, int channels, int64_t src_pix, int64_t dst_pix,
                         const pp_window* windows, int count, int max_pixels) {
    PP_REQUIRE(src && dst && windows && count > 0 && max_pixels > 0, "window_copy: invalid arguments");
    PP_REQUIRE(elem_bytes == 2 || elem_bytes == 4, "window_copy: elem_bytes=%d must be 2 or 4", elem_bytes);
    PP_REQUIRE(channels > 0 && channels <= src_pix && channels <= dst_pix,
               "window_copy: %d channels do not fit pixel pitches %lld / %lld", channels, (long long)src_pix,
               (long long)dst_pix);
    PP_REQUIRE(count <= 65535, "window_copy: at most 65535 windows per launch (got %d)", count);
    return PP_OK;
}

int window_copy_launch(const void* src, void* dst, int elem_bytes, int channels, int64_t src_pix, int64_t dst_pix,
                       const pp_window* windows, int count, int max_pixels, cudaStream_t s) {
    int rc = window_copy_validate(src, dst, elem_bytes, channels, src_pix, dst_pix, windows, count, max_pixels);
    if (rc) return rc;
    const dim3 grid((unsigned)std::min((max_pixels + 255) / 256, 132 * 4), (unsigned)count);
    if (elem_bytes == 2)
        PP_CUDA_CHECK(launch(window_copy_kernel<uint16_t>, grid, 256, 0, s, reinterpret_cast<const uint16_t*>(src),
                             reinterpret_cast<uint16_t*>(dst), channels, src_pix, dst_pix, windows));
    else
        PP_CUDA_CHECK(launch(window_copy_kernel<uint32_t>, grid, 256, 0, s, reinterpret_cast<const uint32_t*>(src),
                             reinterpret_cast<uint32_t*>(dst), channels, src_pix, dst_pix, windows));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

// ------------------------------------------------------------------------------------
// blend_v then blend_h of one tile. Only the pixels of the two seam strips change: the top e_v rows (all columns)
// and the left e_h columns of the rows below them. A pixel's horizontal blend reads its own vertically blended
// value, so one thread does both in diffusers order. The weights are the double expressions 1 - y/e and y/e
// rounded to fp32 (what torch does with a Python-float scalar); __fmul_rn / __fadd_rn keep every product and the
// sum separately rounded, as the torch loop's separate kernels do.
// ------------------------------------------------------------------------------------
__device__ __forceinline__ float blend_pair(float a, float b, int k, int e) {
    const double t = (double)k / (double)e;
    return __fadd_rn(__fmul_rn(a, (float)(1.0 - t)), __fmul_rn(b, (float)t));
}

__global__ void tile_blend_kernel(pp_tile_blend_desc d) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t top = (int64_t)d.e_v * d.b_w;
    const int64_t n = top + (int64_t)(d.b_h - d.e_v) * d.e_h;
    const int64_t sample = blockIdx.y;
    float* b = d.b + sample * d.b_stride;
    const float* av = d.av + (d.e_v ? sample * d.av_stride : 0);
    const float* ah = d.ah + (d.e_h ? sample * d.ah_stride : 0);
    const int C = d.channels;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t y, x;
        if (i < top) {
            y = i / d.b_w;
            x = i - y * d.b_w;
        } else {
            const int64_t q = i - top;
            y = d.e_v + q / d.e_h;
            x = q - (y - d.e_v) * d.e_h;
        }
        float* pb = b + (y * d.b_w + x) * C;
        for (int c = 0; c < C; ++c) {
            float v = pb[c];
            if (y < d.e_v) v = blend_pair(av[((d.av_h - d.e_v + y) * d.b_w + x) * C + c], v, (int)y, d.e_v);
            if (x < d.e_h) v = blend_pair(ah[(y * d.ah_w + (d.ah_w - d.e_h + x)) * C + c], v, (int)x, d.e_h);
            pb[c] = v;
        }
    }
}

int tile_blend_validate(const pp_tile_blend_desc& d) {
    PP_REQUIRE(d.b && d.batch > 0 && d.channels > 0 && d.b_h > 0 && d.b_w > 0, "tile_blend: invalid arguments");
    PP_REQUIRE(d.e_v >= 0 && d.e_h >= 0 && d.e_v <= d.b_h && d.e_h <= d.b_w,
               "tile_blend: blend extents %d / %d exceed the %d x %d tile", d.e_v, d.e_h, d.b_h, d.b_w);
    PP_REQUIRE(d.e_v == 0 || (d.av && d.av_h >= d.e_v), "tile_blend: upper neighbour missing or shorter than e_v");
    PP_REQUIRE(d.e_h == 0 || (d.ah && d.ah_w >= d.e_h), "tile_blend: left neighbour missing or narrower than e_h");
    PP_REQUIRE(d.batch <= 65535, "tile_blend: at most 65535 samples");
    return PP_OK;
}

int tile_blend_launch(const pp_tile_blend_desc& d, cudaStream_t s) {
    int rc = tile_blend_validate(d);
    if (rc) return rc;
    const int64_t n = (int64_t)d.e_v * d.b_w + (int64_t)(d.b_h - d.e_v) * d.e_h;
    if (n == 0) return PP_OK;  // no seam: nothing to enqueue
    const dim3 grid((unsigned)std::min<int64_t>((n + 255) / 256, 132 * 4), (unsigned)d.batch);
    PP_CUDA_CHECK(launch(tile_blend_kernel, grid, 256, 0, s, d));
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
}

}  // namespace pp

extern "C" {
pp_status pp_window_copy(const void* src, void* dst, int32_t elem_bytes, int32_t channels, int64_t src_pix,
                         int64_t dst_pix, const pp_window* windows, int32_t count, int32_t max_pixels,
                         pp_stream stream) {
    return pp::window_copy_launch(src, dst, elem_bytes, channels, src_pix, dst_pix, windows, count, max_pixels,
                                  reinterpret_cast<cudaStream_t>(stream));
}
pp_status pp_tile_blend(const pp_tile_blend_desc* d, pp_stream stream) {
    if (!d) { pp::set_last_error("pp_tile_blend: null descriptor"); return pp::PP_ERR_INVALID; }
    return pp::tile_blend_launch(*d, reinterpret_cast<cudaStream_t>(stream));
}
}
