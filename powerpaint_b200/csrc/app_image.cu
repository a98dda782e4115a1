// The app's request pre- and post-processing on uint8 HWC images (SURVEY.md §(f) row 3, DESIGN.md §6b): Pillow's
// Image.resize (bilinear / bicubic / lanczos) and GaussianBlur, OpenCV's Canny (aperture 3, L1), and the app's
// elementwise steps (outpainting canvas, RGB -> L, v2 hole fill, red overlay, paste-back). Every result equals the
// library's byte for byte; tests/test_imageops_gpu.py checks that against the libraries themselves.
//
// Reference call sites: ref:app.py:258-387 (predict), :405-473 (predict_controlnet).
#include "common.cuh"
#include "ops.h"

#include <math.h>

namespace pp {

namespace {

constexpr int kResampleBits = 22;  // Pillow's PRECISION_BITS for 8-bit images

__device__ __forceinline__ uint8_t clip8(int32_t v) {
    v >>= kResampleBits;
    return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// ------------------------------------------------------------------------------------
// Resampling: out[y, x, c] = clip8(2^21 + sum_t in[.., xmin + t, ..] * k[x, t]). The host builds the tables
// (bounds = (xmin, taps) per output pixel, k = 22-bit fixed-point weights). One thread per output pixel.
// ------------------------------------------------------------------------------------
template <int CH>
__global__ void resample_h_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int rows, int in_w,
                                  int out_w, const int32_t* __restrict__ bounds, const int32_t* __restrict__ k,
                                  int ksize) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)rows * out_w;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = i / out_w;
        const int x = (int)(i - y * out_w);
        const int xmin = __ldg(bounds + 2 * x), n = __ldg(bounds + 2 * x + 1);
        const int32_t* kx = k + (int64_t)x * ksize;
        const uint8_t* s = src + (y * in_w + xmin) * CH;
        int32_t acc[CH];
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[c] = 1 << (kResampleBits - 1);
        for (int t = 0; t < n; ++t) {
            const int32_t w = __ldg(kx + t);
#pragma unroll
            for (int c = 0; c < CH; ++c) acc[c] += (int32_t)s[t * CH + c] * w;
        }
#pragma unroll
        for (int c = 0; c < CH; ++c) dst[i * CH + c] = clip8(acc[c]);
    }
}

__global__ void resample_v_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int out_h, int w, int ch,
                                  const int32_t* __restrict__ bounds, const int32_t* __restrict__ k, int ksize) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t row = (int64_t)w * ch;  // bytes per row; each thread owns one byte of the output row
    const int64_t total = (int64_t)out_h * row;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = i / row;
        const int64_t xc = i - y * row;
        const int ymin = __ldg(bounds + 2 * y), n = __ldg(bounds + 2 * y + 1);
        const int32_t* ky = k + y * ksize;
        const uint8_t* s = src + (int64_t)ymin * row + xc;
        int32_t acc = 1 << (kResampleBits - 1);
        for (int t = 0; t < n; ++t) acc += (int32_t)s[t * row] * __ldg(ky + t);
        dst[i] = clip8(acc);
    }
}

// ------------------------------------------------------------------------------------
// One pass of Pillow's extended box blur along x (vertical = 0) or y (vertical = 1), edges replicated:
// out = (acc * ww + (in[p - r - 1] + in[p + r + 1]) * fw + 2^23) >> 24, acc the sum over [p - r, p + r].
// ------------------------------------------------------------------------------------
__global__ void box_blur_pass_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int h, int w, int ch,
                                     int vertical, int r, uint32_t ww, uint32_t fw) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)h * w * ch;
    const int n = vertical ? h : w;
    const int64_t step = vertical ? (int64_t)w * ch : ch;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pix = i / ch;
        const int p = vertical ? (int)(pix / w) : (int)(pix % w);
        const uint8_t* line = src + i - (int64_t)p * step;  // element 0 of this pixel's line, same channel
        uint32_t acc = 0;
        for (int j = p - r; j <= p + r; ++j) acc += line[(int64_t)min(max(j, 0), n - 1) * step];
        const uint32_t far = (uint32_t)line[(int64_t)max(p - r - 1, 0) * step] +
                             (uint32_t)line[(int64_t)min(p + r + 1, n - 1) * step];
        dst[i] = (uint8_t)((acc * ww + far * fw + (1u << 23)) >> 24);
    }
}

// ------------------------------------------------------------------------------------
// Canny. 1) Sobel (replicated borders) -> L1 magnitude and (dx, dy) of the channel with the largest magnitude.
// ------------------------------------------------------------------------------------
constexpr int kTileW = 32, kTileH = 16;  // union-find tile = one block of 512 threads, one pixel each

__global__ void canny_sobel_kernel(const uint8_t* __restrict__ img, int h, int w, int ch, int32_t* __restrict__ mag,
                                   int32_t* __restrict__ dxdy) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)h * w;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / w), x = (int)(i - (int64_t)y * w);
        const int ys[3] = {max(y - 1, 0), y, min(y + 1, h - 1)};
        const int xs[3] = {max(x - 1, 0), x, min(x + 1, w - 1)};
        int best_m = -1, best_dx = 0, best_dy = 0;
        for (int c = 0; c < ch; ++c) {
            int v[3][3];
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int b = 0; b < 3; ++b) v[a][b] = img[((int64_t)ys[a] * w + xs[b]) * ch + c];
            const int dx = (v[0][2] + 2 * v[1][2] + v[2][2]) - (v[0][0] + 2 * v[1][0] + v[2][0]);
            const int dy = (v[2][0] + 2 * v[2][1] + v[2][2]) - (v[0][0] + 2 * v[0][1] + v[0][2]);
            const int m = abs(dx) + abs(dy);
            if (m > best_m) best_m = m, best_dx = dx, best_dy = dy;  // strict: the first channel wins ties
        }
        mag[i] = best_m;
        dxdy[i] = (int32_t)(((uint32_t)(uint16_t)(int16_t)best_dx << 16) | (uint16_t)(int16_t)best_dy);
    }
}

// Lock-free union-find over labels that only ever point to smaller indices (Playne & Hawick, IEEE TPDS 2018).
// L is shared memory in the block-local phase and global memory in the merge; stale reads only cost a retry.
__device__ __forceinline__ int uf_find(const volatile int32_t* L, int x) {
    int y = L[x];
    while (y != x) {
        x = y;
        y = L[x];
    }
    return x;
}

__device__ __forceinline__ void uf_union(int32_t* L, int a, int b) {
    for (;;) {
        a = uf_find(L, a);
        b = uf_find(L, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(L + b, a);
        if (old == b) return;
        b = old;  // b had been linked meanwhile: join a with what it was linked to
    }
}

// 2) Non-maximum suppression (OpenCV's 15-bit tan 22.5 sector test, its > / >= pattern, magnitude 0 outside the
// image) -> class 0 / 1 (> low) / 2 (> high); then union-find of the 8-connected candidates inside the tile.
// Labels are global pixel indices of each pixel's root, -1 for non-candidates; `strong` is cleared.
__global__ void __launch_bounds__(kTileW * kTileH) canny_nms_local_kernel(
    const int32_t* __restrict__ mag, const int32_t* __restrict__ dxdy, int h, int w, int low, int high,
    uint8_t* __restrict__ cls, int32_t* __restrict__ labels, uint8_t* __restrict__ strong) {
    pdl_wait();
    pdl_launch_dependents();
    __shared__ int32_t s_lab[kTileW * kTileH];
    const int lx = threadIdx.x, ly = threadIdx.y, li = ly * kTileW + lx;
    const int x = blockIdx.x * kTileW + lx, y = blockIdx.y * kTileH + ly;
    const bool inside = x < w && y < h;
    const int64_t gi = (int64_t)y * w + x;
    int c = 0;
    if (inside) {
        const int m = mag[gi];
        if (m > low) {
            auto M = [&](int yy, int xx) -> int {
                return (yy < 0 || yy >= h || xx < 0 || xx >= w) ? 0 : mag[(int64_t)yy * w + xx];
            };
            const int32_t packed = dxdy[gi];
            const int xs = (int16_t)(packed >> 16), ys = (int16_t)(packed & 0xffff);
            const int ax = abs(xs), ay = abs(ys) << 15;
            const int tg22x = ax * 13573;  // (int)(tan(22.5 deg) * 2^15 + 0.5)
            bool keep;
            if (ay < tg22x) {
                keep = m > M(y, x - 1) && m >= M(y, x + 1);
            } else {
                const int tg67x = tg22x + (ax << 16);
                if (ay > tg67x) {
                    keep = m > M(y - 1, x) && m >= M(y + 1, x);
                } else {
                    const int s = (xs ^ ys) < 0 ? -1 : 1;
                    keep = m > M(y - 1, x - s) && m > M(y + 1, x + s);
                }
            }
            if (keep) c = m > high ? 2 : 1;
        }
        cls[gi] = (uint8_t)c;
        strong[gi] = 0;
    }
    s_lab[li] = c ? li : -1;
    __syncthreads();
    if (c) {
        // backward neighbours W, NW, N, NE cover every 8-adjacent pair of the tile once
        if (lx > 0 && s_lab[li - 1] >= 0) uf_union(s_lab, li, li - 1);
        if (ly > 0) {
            if (lx > 0 && s_lab[li - kTileW - 1] >= 0) uf_union(s_lab, li, li - kTileW - 1);
            if (s_lab[li - kTileW] >= 0) uf_union(s_lab, li, li - kTileW);
            if (lx + 1 < kTileW && s_lab[li - kTileW + 1] >= 0) uf_union(s_lab, li, li - kTileW + 1);
        }
    }
    __syncthreads();
    if (inside) {
        int32_t g = -1;
        if (c) {
            const int r = uf_find(s_lab, li);
            g = (int32_t)((int64_t)(blockIdx.y * kTileH + r / kTileW) * w + blockIdx.x * kTileW + r % kTileW);
        }
        labels[gi] = g;
    }
}

// 3) Join the tiles: candidates unite with their backward neighbours that lie in another tile.
__global__ void canny_merge_kernel(const uint8_t* __restrict__ cls, int32_t* labels, int h, int w) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)h * w;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / w), x = (int)(i - (int64_t)y * w);
        const bool left = x % kTileW == 0, top = y % kTileH == 0, right = x % kTileW == kTileW - 1;
        if (!(left || top || right) || !cls[i]) continue;
        auto join = [&](int yy, int xx) {
            if (yy < 0 || xx < 0 || xx >= w) return;
            const int64_t j = (int64_t)yy * w + xx;
            if (cls[j]) uf_union(labels, (int)i, (int)j);
        };
        if (left) join(y, x - 1);
        if (left || top) join(y - 1, x - 1);
        if (top) join(y - 1, x);
        if (top || right) join(y - 1, x + 1);
    }
}

// 4) Point every candidate at its root; strong pixels mark their root.
__global__ void canny_mark_kernel(const uint8_t* __restrict__ cls, int32_t* labels, uint8_t* strong, int64_t total) {
    pdl_wait();
    pdl_launch_dependents();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = cls[i];
        if (!c) continue;
        const int r = uf_find(labels, (int)i);
        labels[i] = r;
        if (c == 2) strong[r] = 1;
    }
}

// 5) An edge is a candidate whose component holds a strong pixel.
__global__ void canny_output_kernel(const uint8_t* __restrict__ cls, const int32_t* labels,
                                    const uint8_t* __restrict__ strong, uint8_t* __restrict__ out, int64_t total) {
    pdl_wait();
    pdl_launch_dependents();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = cls[i] && strong[uf_find(labels, (int)i)] ? 255 : 0;
}

// ------------------------------------------------------------------------------------
// The app's elementwise steps. The blends are NumPy float64 expressions, evaluated here in NumPy's operation order
// with explicitly rounded operations (no FMA contraction) and truncated to uint8 like `astype(np.uint8)`.
// ------------------------------------------------------------------------------------
__global__ void outpaint_canvas_kernel(const uint8_t* __restrict__ src, int o_h, int o_w, uint8_t* __restrict__ img,
                                       uint8_t* __restrict__ mask, int c_h, int c_w, int top, int left, int y0, int y1,
                                       int x0, int x1) {
    pdl_wait();
    pdl_launch_dependents();
    const int64_t total = (int64_t)c_h * c_w;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / c_w), x = (int)(i - (int64_t)y * c_w);
        const int sy = y - top, sx = x - left;
        const bool in_src = sy >= 0 && sy < o_h && sx >= 0 && sx < o_w;
        const uint8_t m = (y >= y0 && y < y1 && x >= x0 && x < x1) ? 0 : 255;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            img[i * 3 + c] = in_src ? src[((int64_t)sy * o_w + sx) * 3 + c] : 127;
            mask[i * 3 + c] = m;
        }
    }
}

__global__ void app_blend_kernel(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                 const uint8_t* __restrict__ c, uint8_t* __restrict__ out, int b_ch, int64_t total) {
    pdl_wait();
    pdl_launch_dependents();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const uint8_t* pa = a + i * 3;
        if (op == PP_BLEND_LUMA) {
            // Pillow's RGB -> L (ImagingConvert rgb2l): ITU-R 601-2 luma in 16-bit fixed point
            out[i] = (uint8_t)((19595u * pa[0] + 38470u * pa[1] + 7471u * pa[2] + 0x8000u) >> 16);
            continue;
        }
        const uint8_t* pb = b + i * b_ch;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const double px = (double)pa[ch];
            const double m = (double)pb[b_ch == 3 ? ch : 0];
            double v;
            if (op == PP_BLEND_HOLE_FILL) {
                // img * (1 - mask / 255.0)
                v = __dmul_rn(px, __dsub_rn(1.0, __ddiv_rn(m, 255.0)));
            } else if (op == PP_BLEND_RED_OVERLAY) {
                // res * (1 - mask / 512.0) + mask / 512.0 * red, red = (180, 0, 0)
                const double t = __ddiv_rn(m, 512.0);
                v = __dadd_rn(__dmul_rn(px, __dsub_rn(1.0, t)), __dmul_rn(t, ch == 0 ? 180.0 : 0.0));
            } else {
                // (res / 255.0 * mb + (1 - mb) * img / 255.0) * 255, mb = blurred mask / 255.0
                const double mb = __ddiv_rn(m, 255.0);
                const double img = __ddiv_rn((double)c[i * 3 + ch], 255.0);
                v = __dmul_rn(__dadd_rn(__dmul_rn(__ddiv_rn(px, 255.0), mb), __dmul_rn(__dsub_rn(1.0, mb), img)),
                              255.0);
            }
            out[i * 3 + ch] = (uint8_t)(int)v;  // astype(np.uint8): truncation (v is in [0, 256))
        }
    }
}

int grid_for(int64_t total) { return (int)std::min<int64_t>((total + 255) / 256, 132 * 16); }

}  // namespace

// Pillow's _gaussian_blur_radius (float arithmetic around a double sqrt): the extended box radius with the same
// variance as a Gaussian of `radius` after `passes` passes
float gaussian_box_radius(float radius, int passes) {
    float sigma2, L, l, a;
    sigma2 = radius * radius / passes;
    L = (float)sqrt(12.0 * sigma2 + 1.0);
    l = (float)floor((L - 1.0) / 2.0);
    a = (2 * l + 1) * (l * (l + 1) - 3 * sigma2);
    a /= 6 * (sigma2 - (l + 1) * (l + 1));
    return l + a;
}

int64_t canny_workspace_bytes(int h, int w) {
    const int64_t n = (int64_t)h * w, a = (n * 4 + 255) / 256 * 256, b = (n + 255) / 256 * 256;
    return 3 * a + 2 * b;  // mag, dx|dy, labels (int32); class, strong (uint8)
}

}  // namespace pp

extern "C" {

pp_status pp_resample_u8(const uint8_t* src, uint8_t* tmp, uint8_t* dst, int32_t in_h, int32_t in_w, int32_t out_h,
                         int32_t out_w, int32_t channels, const int32_t* bounds_x, const int32_t* k_x, int32_t taps_x,
                         const int32_t* bounds_y, const int32_t* k_y, int32_t taps_y, pp_stream stream) {
    auto st = reinterpret_cast<cudaStream_t>(stream);
    PP_REQUIRE(src && dst, "pp_resample_u8: null image pointer");
    PP_REQUIRE(in_h > 0 && in_w > 0 && out_h > 0 && out_w > 0, "pp_resample_u8: zero size (%dx%d -> %dx%d)", in_w,
               in_h, out_w, out_h);
    PP_REQUIRE(channels == 1 || channels == 3, "pp_resample_u8: %d channels (1 or 3 supported)", channels);
    const bool hpass = out_w != in_w, vpass = out_h != in_h;
    PP_REQUIRE(!hpass || (bounds_x && k_x && taps_x > 0), "pp_resample_u8: horizontal pass needs its tables");
    PP_REQUIRE(!vpass || (bounds_y && k_y && taps_y > 0), "pp_resample_u8: vertical pass needs its tables");
    PP_REQUIRE(!(hpass && vpass) || tmp, "pp_resample_u8: a two-pass resize needs the [in_h, out_w] scratch image");
    if (!hpass && !vpass) {
        PP_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)in_h * in_w * channels, cudaMemcpyDeviceToDevice, st));
        return pp::PP_OK;
    }
    const uint8_t* v_src = src;
    if (hpass) {
        uint8_t* h_dst = vpass ? tmp : dst;
        PP_CUDA_CHECK(pp::launch(channels == 3 ? pp::resample_h_kernel<3> : pp::resample_h_kernel<1>,
                                 pp::grid_for((int64_t)in_h * out_w), 256, 0, st, src, h_dst, in_h, in_w, out_w,
                                 bounds_x, k_x, taps_x));
        v_src = h_dst;
    }
    if (vpass)
        PP_CUDA_CHECK(pp::launch(pp::resample_v_kernel, pp::grid_for((int64_t)out_h * out_w * channels), 256, 0, st,
                                 v_src, dst, out_h, out_w, channels, bounds_y, k_y, taps_y));
    PP_CUDA_CHECK(cudaGetLastError());
    return pp::PP_OK;
}

float pp_gaussian_box_radius(float radius, int32_t passes) { return pp::gaussian_box_radius(radius, passes); }

pp_status pp_box_blur_u8(const uint8_t* src, uint8_t* tmp, uint8_t* dst, int32_t h, int32_t w, int32_t channels,
                         float box_radius, int32_t passes, pp_stream stream) {
    auto st = reinterpret_cast<cudaStream_t>(stream);
    PP_REQUIRE(src && tmp && dst, "pp_box_blur_u8: null pointer");
    PP_REQUIRE(h > 0 && w > 0, "pp_box_blur_u8: zero size (%dx%d)", w, h);
    PP_REQUIRE(channels == 1 || channels == 3, "pp_box_blur_u8: %d channels (1 or 3 supported)", channels);
    PP_REQUIRE(box_radius > 0.f && box_radius < 1e6f, "pp_box_blur_u8: box radius %g out of range", box_radius);
    PP_REQUIRE(passes > 0 && passes <= 16, "pp_box_blur_u8: %d passes (1..16)", passes);
    PP_REQUIRE(tmp != src && tmp != dst && dst != src, "pp_box_blur_u8: src, tmp and dst must be distinct");
    // Pillow's ImagingHorizontalBoxBlur: the weight divides in float, its end taps take the remainder
    const int r = (int)box_radius;
    const uint32_t ww = (uint32_t)((float)(1 << 24) / (box_radius * 2 + 1));
    const uint32_t fw = ((1u << 24) - (uint32_t)(r * 2 + 1) * ww) / 2;
    const int64_t total = (int64_t)h * w * channels;
    const uint8_t* in = src;
    for (int p = 0; p < 2 * passes; ++p) {
        uint8_t* out = ((2 * passes - p) % 2 == 0) ? tmp : dst;  // ping-pong that ends in dst
        PP_CUDA_CHECK(pp::launch(pp::box_blur_pass_kernel, pp::grid_for(total), 256, 0, st, in, out, h, w, channels,
                                 p >= passes ? 1 : 0, r, ww, fw));
        in = out;
    }
    PP_CUDA_CHECK(cudaGetLastError());
    return pp::PP_OK;
}

int64_t pp_canny_workspace_bytes(int32_t h, int32_t w) {
    return h > 0 && w > 0 ? pp::canny_workspace_bytes(h, w) : -1;
}

pp_status pp_canny_u8(const uint8_t* src, uint8_t* dst, void* workspace, int64_t workspace_bytes, int32_t h, int32_t w,
                      int32_t channels, double low, double high, pp_stream stream) {
    auto st = reinterpret_cast<cudaStream_t>(stream);
    PP_REQUIRE(src && dst && workspace, "pp_canny_u8: null pointer");
    PP_REQUIRE(h > 0 && w > 0, "pp_canny_u8: zero size (%dx%d)", w, h);
    PP_REQUIRE((int64_t)h * w < (1ll << 31), "pp_canny_u8: %dx%d exceeds 2^31 pixels", w, h);
    PP_REQUIRE(channels == 1 || channels == 3, "pp_canny_u8: %d channels (1 or 3 supported)", channels);
    PP_REQUIRE(workspace_bytes >= pp::canny_workspace_bytes(h, w), "pp_canny_u8: workspace of %lld bytes, needs %lld",
               (long long)workspace_bytes, (long long)pp::canny_workspace_bytes(h, w));
    PP_REQUIRE(low == low && high == high && fabs(low) < 1e9 && fabs(high) < 1e9, "pp_canny_u8: bad thresholds");
    if (low > high) {
        const double t = low;
        low = high;
        high = t;
    }
    const int lo = (int)floor(low), hi = (int)floor(high);  // cvFloor
    const int64_t n = (int64_t)h * w, a = (n * 4 + 255) / 256 * 256, b = (n + 255) / 256 * 256;
    char* ws = static_cast<char*>(workspace);
    int32_t* mag = reinterpret_cast<int32_t*>(ws);
    int32_t* dxdy = reinterpret_cast<int32_t*>(ws + a);
    int32_t* labels = reinterpret_cast<int32_t*>(ws + 2 * a);
    uint8_t* cls = reinterpret_cast<uint8_t*>(ws + 3 * a);
    uint8_t* strong = reinterpret_cast<uint8_t*>(ws + 3 * a + b);
    PP_CUDA_CHECK(pp::launch(pp::canny_sobel_kernel, pp::grid_for(n), 256, 0, st, src, h, w, channels, mag, dxdy));
    const dim3 tiles((w + pp::kTileW - 1) / pp::kTileW, (h + pp::kTileH - 1) / pp::kTileH);
    PP_CUDA_CHECK(pp::launch(pp::canny_nms_local_kernel, tiles, dim3(pp::kTileW, pp::kTileH), 0, st,
                             (const int32_t*)mag, (const int32_t*)dxdy, h, w, lo, hi, cls, labels, strong));
    PP_CUDA_CHECK(pp::launch(pp::canny_merge_kernel, pp::grid_for(n), 256, 0, st, (const uint8_t*)cls, labels, h, w));
    PP_CUDA_CHECK(pp::launch(pp::canny_mark_kernel, pp::grid_for(n), 256, 0, st, (const uint8_t*)cls, labels, strong, n));
    PP_CUDA_CHECK(pp::launch(pp::canny_output_kernel, pp::grid_for(n), 256, 0, st, (const uint8_t*)cls,
                             (const int32_t*)labels, (const uint8_t*)strong, dst, n));
    PP_CUDA_CHECK(cudaGetLastError());
    return pp::PP_OK;
}

pp_status pp_outpaint_canvas_u8(const uint8_t* src, int32_t o_h, int32_t o_w, uint8_t* img, uint8_t* mask,
                                int32_t c_h, int32_t c_w, int32_t top, int32_t left, int32_t hole_y0, int32_t hole_y1,
                                int32_t hole_x0, int32_t hole_x1, pp_stream stream) {
    PP_REQUIRE(src && img && mask, "pp_outpaint_canvas_u8: null pointer");
    PP_REQUIRE(o_h > 0 && o_w > 0 && c_h > 0 && c_w > 0, "pp_outpaint_canvas_u8: zero size");
    PP_REQUIRE(top >= 0 && left >= 0 && top + o_h <= c_h && left + o_w <= c_w,
               "pp_outpaint_canvas_u8: a %dx%d image at (%d, %d) does not fit a %dx%d canvas", o_w, o_h, left, top,
               c_w, c_h);
    PP_CUDA_CHECK(pp::launch(pp::outpaint_canvas_kernel, pp::grid_for((int64_t)c_h * c_w), 256, 0,
                             reinterpret_cast<cudaStream_t>(stream), src, o_h, o_w, img, mask, c_h, c_w, top, left,
                             hole_y0, hole_y1, hole_x0, hole_x1));
    PP_CUDA_CHECK(cudaGetLastError());
    return pp::PP_OK;
}

pp_status pp_app_blend_u8(int32_t op, const uint8_t* a, const uint8_t* b, const uint8_t* c, uint8_t* out, int32_t h,
                          int32_t w, int32_t b_channels, pp_stream stream) {
    PP_REQUIRE(op >= PP_BLEND_LUMA && op <= PP_BLEND_PASTE, "pp_app_blend_u8: unknown op %d", op);
    PP_REQUIRE(a && out && (op == PP_BLEND_LUMA || b) && (op != PP_BLEND_PASTE || c), "pp_app_blend_u8: null pointer");
    PP_REQUIRE(h > 0 && w > 0, "pp_app_blend_u8: zero size (%dx%d)", w, h);
    PP_REQUIRE(op == PP_BLEND_LUMA || b_channels == 1 || b_channels == 3,
               "pp_app_blend_u8: mask with %d channels (1 or 3 supported)", b_channels);
    const int64_t total = (int64_t)h * w;
    PP_CUDA_CHECK(pp::launch(pp::app_blend_kernel, pp::grid_for(total), 256, 0, reinterpret_cast<cudaStream_t>(stream),
                             (int)op, a, b, c, out, (int)b_channels, total));
    PP_CUDA_CHECK(cudaGetLastError());
    return pp::PP_OK;
}
}
