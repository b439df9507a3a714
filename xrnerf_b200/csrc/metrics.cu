// xrnerf_b200 — image metrics: SSIM of image pairs (xrb_ssim). The definition, the arithmetic and the workspace are stated in include/xrnerf_b200.h.
//
//   ssim_tile_kernel   block = one 32 x 16 tile of one image, all channels: the tile and its 3-pixel reflected halo are read once into shared memory,
//                      then per channel the five horizontal 7-sums (x, y, x^2, y^2, xy) of every halo row, then the vertical 7-sums and S of every
//                      output entry. Each block stores the sum of its S (whole tile, and the part inside the crop) in the workspace.
//   ssim_mean_kernel   block = one image: sums its tiles' partials in a fixed order and divides.
// Every sum runs in a fixed order that depends on the image's size alone, so an image's results do not depend on the batch it is scored in.
#include <cmath>

#include "common.cuh"

namespace xrb {

constexpr int SSIM_WIN = 7, SSIM_R = 3;                    // skimage's default window and its half width (the crop of mean_crop)
constexpr int SSIM_TW = 32, SSIM_TH = 16, SSIM_THREADS = 256;
constexpr int SSIM_HW = SSIM_TW + 2 * SSIM_R, SSIM_HH = SSIM_TH + 2 * SSIM_R;
constexpr int SSIM_SEG = 4;                                // horizontal sums per thread in the row pass
constexpr int SSIM_MEAN_THREADS = 256;

inline int ssim_tiles(int h, int w) { return ((w + SSIM_TW - 1) / SSIM_TW) * ((h + SSIM_TH - 1) / SSIM_TH); }
inline size_t ssim_smem(int c) { return sizeof(double) * 5 * SSIM_HH * SSIM_TW + sizeof(float) * 2 * (size_t)c * SSIM_HH * SSIM_HW; }

// scipy.ndimage mode 'reflect' (d c b a | a b c d | d c b a); n >= 7 and |overshoot| <= 3 need one reflection. Halo entries past the reflected
// range belong to no output entry and are clamped only to stay inside the image.
__device__ __forceinline__ int reflect(int i, int n) {
    i = i < 0 ? -i - 1 : (i >= n ? 2 * n - i - 1 : i);
    return i < 0 ? 0 : (i >= n ? n - 1 : i);
}

// S of one entry from its five window sums, skimage's formula with every operation rounded once (no contraction), so that S(x, x) = 1 and
// S(x, y) = S(y, x) hold exactly
__device__ __forceinline__ double ssim_entry(double sx, double sy, double sxx, double syy, double sxy, double c1, double c2) {
    constexpr double NP = SSIM_WIN * SSIM_WIN, INV_NP = 1.0 / NP, CN = NP / (NP - 1.0);
    const double ux = __dmul_rn(sx, INV_NP), uy = __dmul_rn(sy, INV_NP);
    const double uxx = __dmul_rn(sxx, INV_NP), uyy = __dmul_rn(syy, INV_NP), uxy = __dmul_rn(sxy, INV_NP);
    const double vx = __dmul_rn(CN, __dsub_rn(uxx, __dmul_rn(ux, ux)));
    const double vy = __dmul_rn(CN, __dsub_rn(uyy, __dmul_rn(uy, uy)));
    const double vxy = __dmul_rn(CN, __dsub_rn(uxy, __dmul_rn(ux, uy)));
    const double a1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), c1), a2 = __dadd_rn(__dmul_rn(2.0, vxy), c2);
    const double b1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), c1), b2 = __dadd_rn(__dadd_rn(vx, vy), c2);
    return __ddiv_rn(__dmul_rn(a1, a2), __dmul_rn(b1, b2));
}

// (a, b) summed over the block in a fixed order; the result is valid in thread 0
template <int THREADS>
__device__ __forceinline__ void block_sum2(double &a, double &b) {
    __shared__ double red[2][THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, o)); b = __dadd_rn(b, __shfl_xor_sync(0xffffffffu, b, o)); }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = red[0][0]; b = red[1][0];
        for (int w = 1; w < THREADS / 32; ++w) { a = __dadd_rn(a, red[0][w]); b = __dadd_rn(b, red[1][w]); }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(SSIM_THREADS, 3) ssim_tile_kernel(const float *__restrict__ x, const float *__restrict__ y, int n, int h, int w, int c, double c1, double c2,
                                                                 float *__restrict__ s_map, double *__restrict__ partial) {
    extern __shared__ double smem[];
    double *hs = smem;                                              // [5][SSIM_HH][SSIM_TW]: horizontal sums of x, y, x^2, y^2, xy
    float *xs = (float *)(hs + 5 * SSIM_HH * SSIM_TW);              // [c][SSIM_HH][SSIM_HW]
    float *ys = xs + c * SSIM_HH * SSIM_HW;
    constexpr int PLANE = SSIM_HH * SSIM_TW;
    const int tiles_x = (w + SSIM_TW - 1) / SSIM_TW, tiles = gridDim.x;
    const int w0 = (blockIdx.x % tiles_x) * SSIM_TW, h0 = (blockIdx.x / tiles_x) * SSIM_TH;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int row_len = SSIM_HW * c;
    for (int img = blockIdx.y; img < n; img += gridDim.y) {
        const size_t base = (size_t)img * h * w * c;
        for (int i = threadIdx.x; i < SSIM_HH * row_len; i += SSIM_THREADS) {
            const int r = i / row_len, rem = i - r * row_len, q = rem / c, ch = rem - q * c;
            const size_t g = base + ((size_t)reflect(h0 - SSIM_R + r, h) * w + reflect(w0 - SSIM_R + q, w)) * c + ch;
            const int s = (ch * SSIM_HH + r) * SSIM_HW + q;
            xs[s] = __ldg(x + g);
            ys[s] = __ldg(y + g);
        }
        __syncthreads();
        double full = 0.0, crop = 0.0;
        for (int ch = 0; ch < c; ++ch) {
            // a thread forms SSIM_SEG consecutive horizontal sums of one row: each input is converted once, each product formed once per segment
            for (int e = threadIdx.x; e < SSIM_HH * (SSIM_TW / SSIM_SEG); e += SSIM_THREADS) {
                const int r = e / (SSIM_TW / SSIM_SEG), j0 = (e - r * (SSIM_TW / SSIM_SEG)) * SSIM_SEG;
                const float *xr = xs + (ch * SSIM_HH + r) * SSIM_HW + j0, *yr = ys + (ch * SSIM_HH + r) * SSIM_HW + j0;
                double a[SSIM_SEG + 2 * SSIM_R], b[SSIM_SEG + 2 * SSIM_R];
#pragma unroll
                for (int k = 0; k < SSIM_SEG + 2 * SSIM_R; ++k) { a[k] = xr[k]; b[k] = yr[k]; }
#pragma unroll
                for (int q = 0; q < 5; ++q) {
                    double v[SSIM_SEG + 2 * SSIM_R];
#pragma unroll
                    for (int k = 0; k < SSIM_SEG + 2 * SSIM_R; ++k)
                        v[k] = q == 0 ? a[k] : q == 1 ? b[k] : q == 2 ? __dmul_rn(a[k], a[k]) : q == 3 ? __dmul_rn(b[k], b[k]) : __dmul_rn(a[k], b[k]);
#pragma unroll
                    for (int o = 0; o < SSIM_SEG; ++o) {
                        double t = 0.0;
#pragma unroll
                        for (int k = 0; k < SSIM_WIN; ++k) t = __dadd_rn(t, v[o + k]);
                        hs[q * PLANE + r * SSIM_TW + j0 + o] = t;
                    }
                }
            }
            __syncthreads();
            const int col = w0 + tx;
#pragma unroll
            for (int rr = 0; rr < SSIM_TH; rr += SSIM_THREADS / 32) {
                const int r = ty + rr, row = h0 + r;
                if (row < h && col < w) {
                    double v[5];
#pragma unroll
                    for (int s = 0; s < 5; ++s) {
                        const double *p = hs + s * PLANE + r * SSIM_TW + tx;
                        double t = 0.0;
#pragma unroll
                        for (int k = 0; k < SSIM_WIN; ++k) t = __dadd_rn(t, p[k * SSIM_TW]);
                        v[s] = t;
                    }
                    const double sv = ssim_entry(v[0], v[1], v[2], v[3], v[4], c1, c2);
                    if (s_map) s_map[base + ((size_t)row * w + col) * c + ch] = (float)sv;
                    full = __dadd_rn(full, sv);
                    if (row >= SSIM_R && row < h - SSIM_R && col >= SSIM_R && col < w - SSIM_R) crop = __dadd_rn(crop, sv);
                }
            }
            __syncthreads();
        }
        block_sum2<SSIM_THREADS>(full, crop);
        if (threadIdx.x == 0) {
            double *p = partial + 2 * ((size_t)img * tiles + blockIdx.x);
            p[0] = full; p[1] = crop;
        }
    }
}

__global__ void __launch_bounds__(SSIM_MEAN_THREADS) ssim_mean_kernel(const double *__restrict__ partial, int n, int tiles, double n_full, double n_crop,
                                                                      double *__restrict__ mean_full, double *__restrict__ mean_crop) {
    for (int img = blockIdx.x; img < n; img += gridDim.x) {
        const double *p = partial + 2 * (size_t)img * tiles;
        double full = 0.0, crop = 0.0;
        for (int t = threadIdx.x; t < tiles; t += SSIM_MEAN_THREADS) { full = __dadd_rn(full, p[2 * t]); crop = __dadd_rn(crop, p[2 * t + 1]); }
        block_sum2<SSIM_MEAN_THREADS>(full, crop);
        if (threadIdx.x == 0) { mean_full[img] = __ddiv_rn(full, n_full); mean_crop[img] = __ddiv_rn(crop, n_crop); }
    }
}

inline bool ssim_sizes_ok(int n, int h, int w) { return n >= 0 && h >= SSIM_WIN && w >= SSIM_WIN; }

}  // namespace xrb

using namespace xrb;

extern "C" {

size_t xrb_ssim_workspace(int n, int height, int width) {
    if (!ssim_sizes_ok(n, height, width)) return 0;
    return sizeof(double) * 2 * (size_t)n * ssim_tiles(height, width);
}

int xrb_ssim(const float *x, const float *y, int n, int height, int width, int channels, double data_range, double *mean_full, double *mean_crop, float *s_map,
             void *workspace, size_t workspace_bytes, void *stream) {
    XRB_REQUIRE(n >= 0, "ssim: negative image count");
    XRB_REQUIRE(height >= SSIM_WIN && width >= SSIM_WIN, "ssim: the 7x7 window does not fit: height and width must be at least 7");
    XRB_REQUIRE(channels >= 1 && channels <= 4, "ssim: channels must be 1..4");
    XRB_REQUIRE(std::isfinite(data_range) && data_range > 0.0, "ssim: data_range must be finite and > 0");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(x && y && mean_full && mean_crop && workspace, "ssim: null pointer");
    XRB_REQUIRE(workspace_bytes >= xrb_ssim_workspace(n, height, width), "ssim: workspace smaller than xrb_ssim_workspace(n, height, width)");
    XRB_REQUIRE(((uintptr_t)x & 3) == 0 && ((uintptr_t)y & 3) == 0 && ((uintptr_t)s_map & 3) == 0 && ((uintptr_t)mean_full & 7) == 0 && ((uintptr_t)mean_crop & 7) == 0 &&
                    ((uintptr_t)workspace & 7) == 0,
                "ssim: misaligned pointer");
    const double k1r = 0.01 * data_range, k2r = 0.03 * data_range;
    const int tiles = ssim_tiles(height, width);
    const size_t smem = ssim_smem(channels);
    cudaFuncSetAttribute(ssim_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   // per call: the attribute is per device
    cudaStream_t s = (cudaStream_t)stream;
    double *partial = (double *)workspace;
    const dim3 grid((unsigned)tiles, (unsigned)(n < 65535 ? n : 65535));
    ssim_tile_kernel<<<grid, SSIM_THREADS, smem, s>>>(x, y, n, height, width, channels, k1r * k1r, k2r * k2r, s_map, partial);
    ssim_mean_kernel<<<(unsigned)(n < 65535 ? n : 65535), SSIM_MEAN_THREADS, 0, s>>>(partial, n, tiles, (double)height * width * channels,
                                                                                      (double)(height - 2 * SSIM_R) * (width - 2 * SSIM_R) * channels, mean_full, mean_crop);
    return check_launch("ssim");
}

}  // extern "C"
