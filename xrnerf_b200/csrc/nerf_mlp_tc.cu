// xrnerf_b200 — NerfMLP.run_mlp (/root/reference/xrnerf/models/mlps/nerf_mlp.py:70-94: 8x256 ReLU MLP, skip-concat after layer 4,
// alpha head, 256-wide feature layer, 128-wide view branch, rgb head) as ONE persistent wgmma kernel.
// The reference runs it as 11 cuBLAS fp32 GEMMs + 2 cat per 32 768-row chunk with every [chunk,256] activation round-tripping HBM.
//
// Per CTA (1 per SM, 384 threads), per 128-row tile:
//   warps 0-7  two consumer warpgroups: warpgroup h owns rows 64h..64h+63 of the tile. Per layer it issues wgmma.m64nNk16 (N = 256 | 128 | 16)
//              over the weight slabs as they arrive, keeps the [64 x N] fp32 accumulator in registers (up to 128 per thread), then adds the bias,
//              applies ReLU, rounds to fp16 and writes its rows of the next layer's A operand blocks straight from the accumulator fragment.
//              The two warpgroups never wait for each other: a row's next-layer input depends on that row only.
//   warp 8     TMA producer (its warpgroup gives its registers to the two consumer warpgroups: setmaxnreg 40 / 232): streams the pre-swizzled weight slabs of all 11 layers from the L2-resident weight image through a shared-memory
//              ring (cp.async.bulk + mbarrier expect_tx; a slot is released when all 8 consumer warps have finished the MMAs that read it), and
//              the tile's fp16 encoding blocks, re-armed once both warpgroups are past their last reader (views_linears.0).
// A operand: [128 x 64]-blocks, K-major, 128-byte swizzle: blocks 0-3 hidden state h (256 wide), 4..4+AUX-1 the point encoding
// (63 -> 64 for NeRF, 96 -> 128 for Mip-NeRF), last block the view-direction encoding (27 -> 64). The encoding blocks come from the fp16
// encoding tile image (tc.cuh layout), written by the encoders in nerf.cu (xrb_nerf_pack_embedded / posenc / IPE).
// Weights (packed by xrnerf_b200/nerf_mlp.py pack_nerf_mlp): [256 x 32] K-half slabs (64-byte swizzle) for the 256-wide layers, [N x 64] slabs
// (128-byte swizzle) otherwise.
// Numeric contract: fp16 operands (weights and activations), fp32 accumulate; each layer's accumulator is rounded to fp16, then the bias is added in
// fp16; alpha is an fp32 register dot product of the fp16 pts_linears.7 output with alpha_linear, formed in that layer's epilogue.
// Parity tolerance vs the fp32 reference in tests/test_gpu_nerf_mlp.py.
//
// The density lattice (xrb_nerf_density_lattice, mesh export) is the same kernel with LAT = true: the layer schedule stops after pts_linears.7, the
// producer streams only those layers' slabs (a prefix of the weight image) and no encoding blocks, each consumer warpgroup writes the point-encoding
// rows of its 64 lattice points into A block 4 before layer 0 (from the lattice index, in registers), and the pts_linears.7 epilogue stores alpha.
#include <string>

#include "tc.cuh"
#include "common.cuh"
#include "lattice.cuh"
#include "posenc.cuh"
#include "nerf_mlp_tc.cuh"

namespace xrb {

struct NmParams {
    const uint8_t *weight_image; const float *bias; const uint8_t *enc_image;
    int64_t n_rows; int input_ch, input_ch_dirs;
    float *raw;
    uint32_t slot_bytes; int n_slots;
    uint32_t n_slabs[NM_LAYERS]; uint32_t slab_bytes[NM_LAYERS][NM_MAX_SLABS];   // the producer's stream (from nm_layer on the host)
    Lattice lat;                                                                   // LAT: the lattice; raw is then out f32[n_rows]
    IpeBands lat_ipe;                                                              // LAT && MIP: the point query's IPE bands
};

// layers [L, 11) of one tile for my 64 rows (LAT: [L, 8))
template <bool MIP, bool LAT, int L>
__device__ __forceinline__ void nm_layers(NmCtx &x, const NmParams &P, int64_t tile, float *alpha) {
    if constexpr (L < (LAT ? 8 : NM_LAYERS)) {
        constexpr NmLayer Ly = nm_layer<MIP>(L);
        float acc[Ly.N / 2];
        if constexpr (LAT) asm volatile("" : "+l"(x.A), "+r"(x.t), "+r"(x.r0));   // the layer's addresses are formed here, not hoisted out of the tile loop
        tc::fence_proxy_async_smem();        // my epilogue writes -> visible to the tensor core
        tc::named_bar_sync(1 + x.wg, 128);   // ... and every row of my warpgroup written
        nm_slabs<MIP, L, 0>(x, acc);
        tc::acc_fence<Ly.N / 2>(acc);
        tc::named_bar_sync(1 + x.wg, 128);   // every warp's share of this layer's MMAs has completed before A blocks are rewritten
        const float *b = P.bias + Ly.bias_off;
        if constexpr (L == NM_LAYERS - 1) {
            // rgb_linear: columns 0,1 sit in lane q = 0 of a quad, columns 2,3 in lane q = 1
            const float c2a = __shfl_down_sync(0xffffffffu, acc[0], 1), c2b = __shfl_down_sync(0xffffffffu, acc[2], 1);
            if ((x.t & 3u) == 0) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int64_t i = tile * 128 + x.r0 + 8 * e;
                    if (i < P.n_rows) reinterpret_cast<float4 *>(P.raw)[i] = make_float4(acc[2 * e] + __ldg(b), acc[2 * e + 1] + __ldg(b + 1), (e ? c2b : c2a) + __ldg(b + 2), alpha[e]);
                }
            }
        } else {
            float adot[2] = {0.f, 0.f};
            const float *wa = P.bias + 2448;   // alpha_linear weights follow the per-layer biases, then its bias
#pragma unroll
            for (int j = 0; j < Ly.N / 8; ++j) {
                const uint32_t col = tc::frag_col(x.t, j);
                uint8_t *blk = x.A + (size_t)(col >> 6) * TILE_BLOCK_BYTES;
                const float b0 = __ldg(b + col), b1 = __ldg(b + col + 1);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    __half2 h = __hadd2(__floats2half2_rn(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]), __floats2half2_rn(b0, b1));
                    if (Ly.relu) h = __hmax2(h, __float2half2_rn(0.f));
                    if (Ly.alpha_dot) { const float2 f = __half22float2(h); adot[e] = fmaf(f.x, __ldg(wa + col), adot[e]); adot[e] = fmaf(f.y, __ldg(wa + col + 1), adot[e]); }
                    if (!(LAT && Ly.alpha_dot)) *reinterpret_cast<__half2 *>(sw128_elem(blk, x.r0 + 8u * (uint32_t)e, col & 63u)) = h;   // LAT: h7 has no reader
                }
            }
            if constexpr (Ly.alpha_dot) {   // the four lanes of a quad hold all 256 columns of its two rows
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    adot[e] += __shfl_xor_sync(0xffffffffu, adot[e], 1);
                    adot[e] += __shfl_xor_sync(0xffffffffu, adot[e], 2);
                    alpha[e] = adot[e] + __ldg(wa + 256);
                }
                if constexpr (LAT) {
                    if ((x.t & 3u) == 0) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int64_t i = tile * 128 + x.r0 + 8 * e;
                            if (i < P.n_rows) P.raw[i] = alpha[e];
                        }
                    }
                }
            }
        }
        nm_layers<MIP, LAT, L + 1>(x, P, tile, alpha);
    }
}

// LAT: the point encoding of lattice point p, zero past the last point, as row `row` of the point-encoding A blocks from `blk`: the positional encoding
// (multires 10, column 63 zero) or, when MIP, the IPE at the launch's footprint (ipe_point_bands, as xrb_mip_ipe_tiles_points; columns 6 n_deg .. 127
// zero, so the row is zeroed first). Each column goes to shared memory as soon as it is formed (fp16, the rounding of pack_h8), so no row of floats
// is live beside the trig reductions.
template <bool MIP>
__device__ __forceinline__ void nm_lattice_row(const NmParams &P, uint8_t *blk, uint32_t row, int64_t p) {
    auto put = [&](int c, float y) { *reinterpret_cast<__half *>(sw128_elem(blk + (c >> 6) * TILE_BLOCK_BYTES, row, (uint32_t)(c & 63))) = __float2half_rn(y); };
    if (MIP || p >= P.n_rows) {
#pragma unroll
        for (int b = 0; b < (MIP ? 2 : 1); ++b) {
            uint8_t *r = blk + b * TILE_BLOCK_BYTES + sw128_row(row);
#pragma unroll
            for (int ch = 0; ch < 8; ++ch) st_chunk(r + sw128_chunk(row, ch), make_uint4(0u, 0u, 0u, 0u));
        }
    }
    if (p < P.n_rows) {
        float x[3];
        P.lat.position(p, x);
        if constexpr (MIP) ipe_point_bands(x, P.lat_ipe, put);
        else {
#pragma unroll
            for (int a = 0; a < 3; ++a) put(a, x[a]);
            posenc_bands<10>(x, put);
            put(63, 0.f);
        }
    }
}

template <bool MIP, bool LAT>
__global__ void __launch_bounds__(NM_THREADS, 1) nerf_mlp_wg_kernel(const __grid_constant__ NmParams P) {
    extern __shared__ uint8_t dyn_smem[];
    constexpr int AUX = MIP ? 2 : 1;
    uint8_t *base = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    uint8_t *A = base, *ring = A + (size_t)(5 + AUX) * TILE_BLOCK_BYTES;
    uint64_t *bars = (uint64_t *)(ring + (size_t)P.n_slots * P.slot_bytes);
    uint64_t *full = bars, *empty = bars + P.n_slots, *enc_full = bars + 2 * P.n_slots, *enc_free = enc_full + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < P.n_slots; ++s) { tc::mbar_init(full + s, 1); tc::mbar_init(empty + s, 8); }
        tc::mbar_init(enc_full, 1); tc::mbar_init(enc_free, 8);
        tc::fence_mbar_init();
    }
    __syncthreads();
    const int64_t n_tiles = (P.n_rows + 127) / 128;
    const uint32_t enc_bytes = (uint32_t)(AUX + 1) * TILE_BLOCK_BYTES;

    if (warp >= 8) {
        // ===================================================== TMA producer (one lane)
        tc::setmaxnreg_dec<40>();
        if (warp == 8 && lane == 0) {
            uint32_t it = 0, n = 0;
            for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++n) {
                // the tile's encoding blocks land in A blocks 4.. (point blocks, then the direction block); LAT: the consumers write them
                if constexpr (!LAT) {
                    if (n > 0) tc::mbar_wait(enc_free, (n - 1) & 1);
                    tc::mbar_expect_tx(enc_full, enc_bytes);
                    tc::tma_bulk_g2s(A + 4 * TILE_BLOCK_BYTES, P.enc_image + (size_t)tile * enc_bytes, enc_bytes, enc_full);
                }
                size_t off = 0;
                for (int l = 0; l < NM_LAYERS; ++l)
                    for (uint32_t s = 0; s < P.n_slabs[l]; ++s, ++it) {
                        const uint32_t slot = it % P.n_slots, round = it / P.n_slots, bytes = P.slab_bytes[l][s];
                        if (round > 0) tc::mbar_wait(empty + slot, (round - 1) & 1);
                        tc::mbar_expect_tx(full + slot, bytes);
                        tc::tma_bulk_g2s(ring + (size_t)slot * P.slot_bytes, P.weight_image + off, bytes, full + slot);
                        off += bytes;
                    }
            }
        }
        return;
    }
    // ===================================================== consumer warpgroups
    tc::setmaxnreg_inc<232>();
    NmCtx x;
    x.A = A; x.ring = ring; x.full = full; x.empty = empty; x.it = 0; x.n_slots = (uint32_t)P.n_slots; x.slot_bytes = P.slot_bytes;
    x.wg = threadIdx.x >> 7; x.t = threadIdx.x & 127; x.lane = lane; x.r0 = 64u * x.wg + tc::frag_row(x.t);
    uint32_t n = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++n) {
        if constexpr (LAT) {   // my rows' MMAs of the previous tile are complete; layer 0's fence and barrier publish these writes
            if (x.t < 64) nm_lattice_row<MIP>(P, A + 4 * TILE_BLOCK_BYTES, 64u * x.wg + x.t, tile * 128 + 64 * x.wg + x.t);
        } else {
            tc::mbar_wait(enc_full, n & 1);
        }
        float alpha[2] = {0.f, 0.f};
        nm_layers<MIP, LAT, 0>(x, P, tile, alpha);
        if constexpr (!LAT) {
            // views_linears.0 was the last reader of the encoding blocks: the producer may load the next tile's
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(enc_free);
        }
    }
}

// P holds the pointers, n_rows and channels (and the lattice when `lattice`); the schedule and the launch shape are filled in here
static void nm_launch(NmParams &P, bool lattice, cudaStream_t s) {
    const int64_t n_rows = P.n_rows;
    const bool mip = P.input_ch > 64;
    uint32_t max_bytes = 0;
    for (int l = 0; l < NM_LAYERS; ++l) {
        const NmLayer L = mip ? nm_layer<true>(l) : nm_layer<false>(l);
        P.n_slabs[l] = lattice && l > 7 ? 0u : (uint32_t)L.n_slabs;   // the lattice stops after pts_linears.7: its stream is a prefix of the image
        for (int k = 0; k < L.n_slabs; ++k) { P.slab_bytes[l][k] = nm_slab_bytes(L.s[k]); if (P.slab_bytes[l][k] > max_bytes) max_bytes = P.slab_bytes[l][k]; }
    }
    P.slot_bytes = (max_bytes + 1023) & ~1023u;
    P.n_slots = 4;
    const size_t smem = 1024 + (size_t)(5 + (mip ? 2 : 1)) * TILE_BLOCK_BYTES + (size_t)P.n_slots * P.slot_bytes + 8 * (2 * P.n_slots + 2);
    const int grid = persistent_grid(1, (n_rows + 127) / 128);
    auto k = lattice ? (mip ? nerf_mlp_wg_kernel<true, true> : nerf_mlp_wg_kernel<false, true>) : mip ? nerf_mlp_wg_kernel<true, false> : nerf_mlp_wg_kernel<false, false>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<grid, NM_THREADS, smem, s>>>(P);
}

// the rest of a density-lattice entry after its size check (sz: lattice_sizes' result) and its encoding checks: the box, the pointers, the launch
static int nm_density_lattice(const char *who, int sz, int input_ch, const IpeBands &ipe, const void *weight_image, const float *bias, int nx, int ny, int nz,
                              const float *box_min_host, const float *box_max_host, float *out, void *stream) {
    const std::string w = who;
    Box b;
    const int e = read_box(box_min_host, box_max_host, false, &b, (w + ": the box must be finite with box_min < box_max on every axis").c_str());
    if (e) return e;
    if (sz == 0) return XRB_OK;
    XRB_REQUIRE(weight_image && bias && out, (w + ": null pointer").c_str());
    XRB_REQUIRE(((uintptr_t)weight_image & 15) == 0 && ((uintptr_t)bias & 15) == 0 && ((uintptr_t)out & 3) == 0,
                (w + ": weight image / bias must be 16-byte aligned, out 4-byte aligned").c_str());
    NmParams P{};
    P.weight_image = (const uint8_t *)weight_image; P.bias = bias;
    P.n_rows = (int64_t)nx * ny * nz; P.input_ch = input_ch; P.input_ch_dirs = 27; P.raw = out;
    P.lat = make_lattice(nx, ny, nz, b); P.lat_ipe = ipe;
    nm_launch(P, true, (cudaStream_t)stream);
    return check_launch(who);
}

}  // namespace xrb

using namespace xrb;

extern "C" {

// image/bias from xrnerf_b200.nerf_mlp.pack_nerf_mlp (in the order nm_layer streams the slabs); enc_image: the fp16 encoding tile image
int xrb_nerf_mlp_forward(const void *weight_image, const float *bias, const void *enc_image, int64_t n_rows, int input_ch, int input_ch_dirs, float *raw, void *stream) {
    XRB_REQUIRE(n_rows >= 0, "nerf_mlp_forward: negative size");
    if (!((input_ch == 63 && input_ch_dirs == 27) || (input_ch == 96 && input_ch_dirs == 27))) {
        set_error("nerf_mlp_forward: implemented for NerfMLP(netdepth=8, netwidth=256, skips=[4], use_viewdirs) with (63,27) or (96,27) input channels");
        return XRB_E_UNSUPPORTED;
    }
    if (n_rows == 0) return XRB_OK;
    XRB_REQUIRE(weight_image && bias && enc_image && raw, "nerf_mlp_forward: null pointer");
    XRB_REQUIRE(((uintptr_t)weight_image & 15) == 0 && ((uintptr_t)raw & 15) == 0 && ((uintptr_t)enc_image & 15) == 0 && ((uintptr_t)bias & 15) == 0,
                "nerf_mlp_forward: images / bias / raw must be 16-byte aligned");
    NmParams P{};
    P.weight_image = (const uint8_t *)weight_image; P.bias = bias; P.enc_image = (const uint8_t *)enc_image;
    P.n_rows = n_rows; P.input_ch = input_ch; P.input_ch_dirs = input_ch_dirs; P.raw = raw;
    nm_launch(P, false, (cudaStream_t)stream);
    return check_launch("nerf_mlp_forward");
}

// the raw alpha of xrb_nerf_mlp_forward at every point of a lattice, the point encoding formed inside the kernel. See include/xrnerf_b200.h.
int xrb_nerf_density_lattice(const void *weight_image, const float *bias, int input_ch, int multires, int nx, int ny, int nz, const float *box_min_host,
                             const float *box_max_host, float *out, void *stream) {
    const int sz = lattice_sizes(nx, ny, nz, "nerf_density_lattice: bad size: every lattice size must be 2..1024");
    if (sz < 0) return XRB_E_BADARG;
    if (!(input_ch == 63 && multires == 10)) {
        set_error("nerf_density_lattice: implemented for the NerfMLP point encoding of the reference configs, input_ch 63 (multires 10)");
        return XRB_E_UNSUPPORTED;
    }
    return nm_density_lattice("nerf_density_lattice", sz, 63, IpeBands{}, weight_image, bias, nx, ny, nz, box_min_host, box_max_host, out, stream);
}

// the raw alpha of xrb_nerf_mlp_forward (Mip-NeRF layout) at every point of a lattice, on the xrb_mip_ipe_tiles_points encoding at footprint sigma
// formed inside the kernel. See include/xrnerf_b200.h.
int xrb_mip_density_lattice(const void *weight_image, const float *bias, int min_deg_point, int max_deg_point, float sigma, int nx, int ny, int nz,
                            const float *box_min_host, const float *box_max_host, float *out, void *stream) {
    const int sz = lattice_sizes(nx, ny, nz, "mip_density_lattice: bad size: every lattice size must be 2..1024");
    if (sz < 0) return XRB_E_BADARG;
    XRB_REQUIRE(ipe_point_degrees_ok(min_deg_point, max_deg_point), "mip_density_lattice: bad degrees (6 (max - min) <= 128, both in [-100, 100])");
    XRB_REQUIRE(std::isfinite(sigma) && sigma >= 0.f, "mip_density_lattice: the footprint sigma must be finite and >= 0");
    return nm_density_lattice("mip_density_lattice", sz, 96, ipe_bands(sigma, min_deg_point, max_deg_point), weight_image, bias, nx, ny, nz, box_min_host,
                              box_max_host, out, stream);
}

}  // extern "C"
