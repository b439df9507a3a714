// xrnerf_b200 — the band columns of BaseEmbedder's positional encoding (embedders/base.py:26-52), one definition for every writer that must produce
// the same fp16 tile-image values: the fast tile-image encoder (csrc/nerf.cu) and the NerfMLP density lattice (csrc/nerf_mlp_tc.cu). Likewise the
// integrated positional encoding of a Mip-NeRF point query (ipe_point_bands): the point encoder and the gradient (csrc/nerf.cu) and the Mip-NeRF
// density lattice (csrc/nerf_mlp_tc.cu).
#pragma once
#include <stdint.h>
#include <cmath>

namespace xrb {

constexpr float HALF_PI = 1.5707963267948966f;

__device__ __forceinline__ float pow2i(int e) { return __int_as_float((127 + e) << 23); }   // 2^e, exact, -126 <= e <= 127

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

}  // namespace xrb
