// xrnerf_b200 — the band columns of BaseEmbedder's positional encoding (embedders/base.py:26-52), one definition for every writer that must produce
// the same fp16 tile-image values: the fast tile-image encoder (csrc/nerf.cu) and the NerfMLP density lattice (csrc/nerf_mlp_tc.cu).
#pragma once
#include <stdint.h>

namespace xrb {

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

}  // namespace xrb
