// xrnerf_b200 — the NerfMLP wgmma kernels' shared pieces: the compile-time layer schedule of the inference kernel (nm_layer, csrc/nerf_mlp_tc.cu) and of
// the density gradient's backward (ng_step, csrc/nerf_grad_tc.cu), and the consumer's slab loop over the weight ring (nm_slabs), which both kernels run.
#pragma once
#include "tc.cuh"

namespace xrb {

constexpr int NM_THREADS = 384;
constexpr int NM_LAYERS = 11;
constexpr int NM_MAX_SLABS = 12;

// ---- compile-time layer schedule (the consumer's loops over layers and slabs are fully unrolled: accumulator offsets must be constants)
struct NmSlab {
    int a_blk;     // A block the slab contracts with
    int kh;        // -1: all 64 columns of the block (128-byte swizzled [rows x 64] slab); 0 / 1: columns 32kh.. ([rows x 32], 64-byte swizzle)
    int rows;      // output columns the slab covers (slab rows)
    int first;     // first slab of the layer: overwrite the accumulator instead of accumulating
};
struct NmLayer {
    int N, relu, bias_off, alpha_dot, n_slabs;
    NmSlab s[NM_MAX_SLABS];
};
__host__ __device__ constexpr uint32_t nm_slab_bytes(const NmSlab &s) { return (uint32_t)s.rows * (s.kh >= 0 ? 64u : 128u); }

template <bool MIP>
__host__ __device__ constexpr NmLayer nm_layer(int l) {
    const int aux = MIP ? 2 : 1, P0 = 4, P1 = 5, DIR = 4 + aux;
    NmLayer L{};
    L.N = l == 9 ? 128 : (l == 10 ? 16 : 256);
    L.relu = (l == 8 || l == 10) ? 0 : 1;
    L.alpha_dot = l == 7;
    L.bias_off = l <= 9 ? 256 * l : 2432;
    int src[6] = {0, 1, 2, 3, 0, 0}, nk = 4;
    if (l == 0) { src[0] = P0; src[1] = P1; nk = aux; }
    else if (l == 5) { src[0] = P0; src[1] = 0; src[2] = 1; src[3] = 2; src[4] = 3; src[5] = P1; nk = 4 + aux; }
    else if (l == 9) { src[0] = DIR; src[1] = 0; src[2] = 1; src[3] = 2; src[4] = 3; nk = 5; }
    else if (l == 10) nk = 2;
    int n = 0;
    for (int k = 0; k < nk; ++k) {
        if (L.N == 256) { L.s[n++] = NmSlab{src[k], 0, 256, k == 0}; L.s[n++] = NmSlab{src[k], 1, 256, 0}; }
        else L.s[n++] = NmSlab{src[k], -1, L.N, k == 0};
    }
    L.n_slabs = n;
    return L;
}

struct NmCtx {
    uint8_t *A, *ring; uint64_t *full, *empty;
    uint32_t it, wg, t, r0, lane, n_slots, slot_bytes;
};

template <int N>
__device__ __forceinline__ void nm_mma(float *acc, uint64_t ad, uint64_t bd, uint32_t sc) { tc::wgmma<N>(acc, ad, bd, sc); }

// ---- the density gradient's backward schedule (xrb_nerf_density_grad_rays): step g of the gradient image contracts dZ (A blocks 0-3, K = the
// layer's 256 outputs) with W^T: 0, 1 = pts_linears.7, .6; 2 = the point columns of pts_linears.5 (the skip term of the encoding gradient); 3 = its
// hidden columns; 4..7 = pts_linears.4 .. .1; 8 = pts_linears.0. The 256-wide steps are [256 x 32] K-half slabs, the encoding steps [NP x 64] slabs
// (NP = 64 | 128: the point-encoding columns, zero padded).
constexpr int NG_STEPS = 9;
template <bool MIP>
__host__ __device__ constexpr NmLayer ng_step(int g) {
    NmLayer L{};
    const bool enc = g == 2 || g == 8;
    L.N = enc ? (MIP ? 128 : 64) : 256;
    L.n_slabs = enc ? 4 : 8;
    for (int k = 0; k < 4; ++k) {
        if (enc) L.s[k] = NmSlab{k, -1, L.N, k == 0};
        else { L.s[2 * k] = NmSlab{k, 0, 256, k == 0}; L.s[2 * k + 1] = NmSlab{k, 1, 256, 0}; }
    }
    return L;
}

// the MMAs of slabs [S, n_slabs) of layer L (GRAD: of gradient step L), one slab at a time through the ring
template <bool MIP, int L, int S, bool GRAD = false>
__device__ __forceinline__ void nm_slabs(NmCtx &x, float *acc) {
    constexpr NmLayer Ly = GRAD ? ng_step<MIP>(L) : nm_layer<MIP>(L);
    if constexpr (S < Ly.n_slabs) {
        constexpr NmSlab sl = Ly.s[S];
        const uint32_t slot = x.it % x.n_slots, ph = (x.it / x.n_slots) & 1u;
        tc::mbar_wait(x.full + slot, ph);
        const uint32_t a0 = tc::smem_u32(x.A + (size_t)sl.a_blk * TILE_BLOCK_BYTES) + x.wg * 8192u + (sl.kh > 0 ? 64u : 0u);
        const uint32_t b0 = tc::smem_u32(x.ring + (size_t)slot * x.slot_bytes);
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < (sl.kh >= 0 ? 2 : 4); ++k) {
            const uint32_t sc = (sl.first && k == 0) ? 0u : 1u;
            const uint64_t ad = tc::desc_k128(a0 + k * 32), bd = sl.kh >= 0 ? tc::desc_k64(b0 + k * 32) : tc::desc_k128(b0 + k * 32);
            nm_mma<sl.rows>(acc, ad, bd, sc);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        __syncwarp();
        if (x.lane == 0) tc::mbar_arrive(x.empty + slot);   // this warp's share of the MMAs reading the slot is complete
        ++x.it;
        nm_slabs<MIP, L, S + 1, GRAD>(x, acc);
    }
}

}  // namespace xrb
