// xrnerf_b200 — the band columns of BaseEmbedder's positional encoding (embedders/base.py:26-52), one definition for every writer that must produce
// the same fp16 tile-image values: the fast tile-image encoder (csrc/nerf.cu) and the NerfMLP density lattice (csrc/nerf_mlp_tc.cu). Likewise the
// integrated positional encoding of a Mip-NeRF point query (ipe_point_bands): the point encoder (csrc/nerf.cu) and the Mip-NeRF density lattice
// (csrc/nerf_mlp_tc.cu); and Mip-NeRF's view-direction bands (mip_dir_bands): the ray and point encoders (csrc/nerf.cu). Each point encoding's
// derivative (posenc_bands_grad, ipe_point_bands_grad) sits beside it, for the gradient kernel of csrc/nerf.cu.
#pragma once
#include <stdint.h>
#include <cmath>

namespace xrb {

constexpr float HALF_PI = 1.5707963267948966f;

__device__ __forceinline__ float pow2i(int e) { return __int_as_float((127 + e) << 23); }   // 2^e, exact, -126 <= e <= 127
__device__ __forceinline__ float sel3(const float *a, int i) { return i == 0 ? a[0] : i == 1 ? a[1] : a[2]; }   // keeps a register array out of local memory

// columns 3 + 6b + a = sin(2^b x_a) and 6 + 6b + a = cos(2^b x_a) of the encoding of x, for the NB bands b < NB (columns 0..2 are x itself):
// put(column, value) for each, columns compile-time constants
template <int NB, class Put>
__device__ __forceinline__ void posenc_bands(const float *x, Put put) {
#pragma unroll
    for (int bnd = 0; bnd < NB; ++bnd)
#pragma unroll
        for (int a = 0; a < 3; ++a) { float sn, cs; sincosf(x[a] * pow2i(bnd), &sn, &cs); put(3 + 6 * bnd + a, sn); put(6 + 6 * bnd + a, cs); }
}
// the same into a register row v
template <int NB>
__device__ __forceinline__ void posenc_bands(const float *x, float *v) { posenc_bands<NB>(x, [&](int c, float y) { v[c] = y; }); }
// the gradient with respect to x through columns 0 .. 2 + 6 nb of the encoding (x itself, then the bands b < nb <= NB), given e(c) = dL/d(column c):
//   g_a = e(a) + sum_b 2^b (cos(2^b x_a) e(3 + 6b + a) - sin(2^b x_a) e(6 + 6b + a))
template <int NB, class E>
__device__ __forceinline__ void posenc_bands_grad(const float *x, int nb, E e, float *g) {
#pragma unroll
    for (int a = 0; a < 3; ++a) g[a] = e(a);
#pragma unroll
    for (int bnd = 0; bnd < NB; ++bnd) {
        if (bnd >= nb) break;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float sn, cs; sincosf(x[a] * pow2i(bnd), &sn, &cs);
            g[a] += pow2i(bnd) * (cs * e(3 + 6 * bnd + a) - sn * e(6 + 6 * bnd + a));
        }
    }
}

// ---- Mip-NeRF point query at footprint sigma: MipNerfEmbedder.integrated_pos_enc (embedders/mipnerf_embedder.py:43-64) of the isotropic Gaussian
// with mean x and covariance sigma^2 I. Band k = 0 .. n_deg-1 (degree min_deg + k), axis a: y = x_a 2^(min_deg+k), a_k = exp(-0.5 sigma^2 4^(min_deg+k));
// column 3k + a = a_k sin(y), column 3 n_deg + 3k + a = a_k sin(y + pi/2) (the reference's expression, as the ray encoder mip_ipe_tiles_fast_kernel).
// a_k is the same for every point, so it is formed once per launch on the host. A band whose 0.5 (sigma^2 2^deg) 2^deg exceeds 20 in fp32 is zero
// (|value| < 2^-25 rounds to 0 in fp16: the ray encoder's rule); such bands are a suffix, k >= n_live, and are not evaluated.
constexpr int IPE_MAX_BANDS = 21;   // 6 * 21 <= 128 columns: the two point blocks of a tile image
struct IpeBands { float fac[IPE_MAX_BANDS]; int min_deg, n_deg, n_live; };

// the point degrees ipe_bands accepts: 1 <= max_deg - min_deg, 6 (max_deg - min_deg) <= 128, both in [-100, 100]
static inline bool ipe_point_degrees_ok(int min_deg, int max_deg) { return max_deg > min_deg && 6 * (max_deg - min_deg) <= 128 && min_deg >= -100 && max_deg <= 100; }

// host: the factors of a launch (sigma finite and >= 0, 1 <= max_deg - min_deg <= 21, degrees in [-100, 100]); a_k = exp(-hv) rounded once to fp32
static inline IpeBands ipe_bands(float sigma, int min_deg, int max_deg) {
    IpeBands B{};
    B.min_deg = min_deg; B.n_deg = max_deg - min_deg; B.n_live = 0;
    const float cov = sigma * sigma;
    for (int k = 0; k < B.n_deg; ++k) {
        const float sc = std::ldexp(1.f, min_deg + k);
        const float hv = 0.5f * (cov * sc * sc);   // the ray encoder's fp32 expression; nondecreasing in k
        if (!(hv <= 20.f)) break;
        B.fac[k] = (float)std::exp(-(double)hv);
        B.n_live = k + 1;
    }
    return B;
}

// the 6 n_deg IPE columns of point x: put(column, value) for every column, dead bands as 0 (columns are run-time values)
template <class Put>
__device__ __forceinline__ void ipe_point_bands(const float *x, const IpeBands &B, Put put) {
#pragma unroll 1
    for (int k = 0; k < B.n_deg; ++k) {
        const bool live = k < B.n_live;
        const float f = B.fac[k], sc = pow2i(B.min_deg + k);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float s = 0.f, c = 0.f;
            if (live) { const float y = x[a] * sc; s = f * sinf(y); c = f * sinf(y + HALF_PI); }
            put(3 * k + a, s); put(3 * B.n_deg + 3 * k + a, c);
        }
    }
}
// the gradient with respect to x through those columns, given e(c) = dL/d(column c) (dead bands are constant zero):
//   g_a = sum_{k < n_live} a_k 2^deg (cos(y) e(3k + a) + cos(y + pi/2) e(3 n_deg + 3k + a)),  y = x_a 2^deg, deg = min_deg + k
template <class E>
__device__ __forceinline__ void ipe_point_bands_grad(const float *x, const IpeBands &B, E e, float *g) {
#pragma unroll
    for (int a = 0; a < 3; ++a) g[a] = 0.f;
    for (int k = 0; k < B.n_live; ++k) {
        const float sc = pow2i(B.min_deg + k), f = B.fac[k];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float y = x[a] * sc;
            g[a] += f * sc * (cosf(y) * e(3 * k + a) + cosf(y + HALF_PI) * e(3 * B.n_deg + 3 * k + a));
        }
    }
}

// ---- MipNerfEmbedder's view-direction encoding (mipnerf_embedder.py:35-41, :55-60), n_deg_view bands from min_deg_view: column a = vd_a, and for
// q = 3 (deg - min_deg_view) + a column 3 + q = sin(2^deg vd_a), column 3 + 3 n_deg_view + q = sin(2^deg vd_a + pi/2) (the reference's expression,
// not cos). put(column, value) for every column; fully unrolled when n_deg_view is a compile-time constant.
template <class Put>
__device__ __forceinline__ void mip_dir_bands(const float *vd, int min_deg_view, int n_deg_view, Put put) {
#pragma unroll
    for (int a = 0; a < 3; ++a) put(a, vd[a]);
#pragma unroll
    for (int q = 0; q < 3 * n_deg_view; ++q) {
        const float x = sel3(vd, q % 3) * pow2i(q / 3 + min_deg_view);
        put(3 + q, sinf(x)); put(3 + 3 * n_deg_view + q, sinf(x + HALF_PI));
    }
}

}  // namespace xrb
