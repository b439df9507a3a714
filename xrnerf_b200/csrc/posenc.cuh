// xrnerf_b200 — the band columns of BaseEmbedder's positional encoding (embedders/base.py:26-52), one definition for every writer that must produce
// the same fp16 tile-image values: the fast tile-image encoder (csrc/nerf.cu) and the NerfMLP density lattice (csrc/nerf_mlp_tc.cu). Likewise the
// integrated positional encoding of a Mip-NeRF point query (ipe_point_bands): the point encoder (csrc/nerf.cu) and the Mip-NeRF density lattice
// (csrc/nerf_mlp_tc.cu); and Mip-NeRF's view-direction bands (mip_dir_bands): the ray and point encoders (csrc/nerf.cu). Each point encoding's
// derivative (posenc_bands_grad, ipe_point_bands_grad) sits beside it, for the gradient kernel of csrc/nerf.cu; the ray IPE's (ipe_ray_grad) serves the
// normal-map gradient kernel of csrc/nerf_grad_tc.cu. A ray sample's position (get_pts, sample_gaussian) is defined here once, for the ray encoders of
// csrc/nerf.cu and that gradient kernel.
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

// ---- a ray sample's position. NeRF: the point o + d z; Mip-NeRF: the Gaussian of the sample's conical frustum (its mean is the position)
// cast_rays (networks/utils/mip.py:117-129): the conical frustum -> Gaussian (:91-114), lift_gaussian (:66-88), diagonal covariance
__device__ __forceinline__ void frustum_gaussian(float t0, float t1, float radius, const float d[3], const float o[3], float dmag_sq, float mean[3], float cov[3]) {
    float mu = (t0 + t1) / 2.f, hw = (t1 - t0) / 2.f;
    float mu2 = mu * mu, hw2 = hw * hw, hw4 = hw2 * hw2, den = 3.f * mu2 + hw2;
    float t_mean = mu + (2.f * mu * hw2) / den;
    float t_var = hw2 / 3.f - (4.f / 15.f) * ((hw4 * (12.f * mu2 - hw2)) / (den * den));
    float r_var = radius * radius * (mu2 / 4.f + (5.f / 12.f) * hw2 - 4.f / 15.f * hw4 / den);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float dd = d[c] * d[c];
        mean[c] = d[c] * t_mean + o[c];
        cov[c] = t_var * dd + r_var * (1.f - dd / dmag_sq);
    }
}
// the Gaussian of sample k (interval z[k], z[k+1]) of ray `ray`
__device__ __forceinline__ void sample_gaussian(const float *z_vals, const float *rays_o, const float *rays_d, const float *radii, int S, int64_t ray, int k, float mean[3],
                                                float cov[3]) {
    const float d[3] = {rays_d[3 * ray], rays_d[3 * ray + 1], rays_d[3 * ray + 2]};
    const float o[3] = {rays_o[3 * ray], rays_o[3 * ray + 1], rays_o[3 * ray + 2]};
    const float dmag = fmaxf(1e-10f, d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    frustum_gaussian(z_vals[ray * (S + 1) + k], z_vals[ray * (S + 1) + k + 1], radii[ray], d, o, dmag, mean, cov);
}
// GetPts (create.py:588-597): o + d * z as a rounded product then a rounded sum (torch), never an FMA — the 2^9-scaled sin arguments amplify the difference
__device__ __forceinline__ void get_pts(const float *rays_o, const float *rays_d, int64_t ray, float z, float p[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(rays_o[3 * ray + a], __fmul_rn(rays_d[3 * ray + a], z));
}

// the gradient with respect to the mean of the ray IPE columns mip_ipe_tiles_fast_kernel writes (NDEG bands from min_deg, covariance cov held fixed),
// given e(c) = dL/d(column c):
//   g_a = sum_k exp(-0.5 cov_a 4^deg) 2^deg (cos(y) e(3k + a) + cos(y + pi/2) e(3 NDEG + 3k + a)),  y = mean_a 2^deg, deg = min_deg + k,
// with the encoder's dead-band rule: a band whose 0.5 cov_a 4^deg exceeds 20 is constant zero
template <int NDEG, class E>
__device__ __forceinline__ void ipe_ray_grad(const float *mean, const float *cov, int min_deg, E e, float *g) {
#pragma unroll
    for (int a = 0; a < 3; ++a) g[a] = 0.f;
#pragma unroll
    for (int k = 0; k < NDEG; ++k) {
        const float sc = pow2i(min_deg + k);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float y = mean[a] * sc, hv = 0.5f * (cov[a] * sc * sc);
            if (hv <= 20.f) g[a] += expf(-hv) * sc * (cosf(y) * e(3 * k + a) + cosf(y + HALF_PI) * e(3 * NDEG + 3 * k + a));
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
