// xrnerf_b200 — the NerfMLP's density gradient at every sample of a ray batch (normal maps of the NeRF / Mip-NeRF renderers, include/xrnerf_b200.h
// "NeRF / Mip-NeRF normal maps"): one wgmma kernel runs the trunk's forward and its input-gradient backward per 128-row tile, on the schedule and slab
// loop of the inference kernel (csrc/nerf_mlp_tc.cuh); the per-ray normal composite.
#include <string>

#include "tc.cuh"
#include "common.cuh"
#include "posenc.cuh"
#include "nerf_mlp_tc.cuh"

namespace xrb {

// ---- density gradient for normal maps (xrb_nerf_density_grad_rays, xrb_mip_density_grad_rays): per 128-row tile, the trunk's forward (pts_linears.0..7
// and the alpha dot, exactly as nerf_mlp_wg_kernel) and its input-gradient backward in one kernel, nothing in HBM between them. Warps 0-7 are the two
// consumer warpgroups (rows 64h..64h+63 each), warp 8 the TMA producer: it streams the forward's prefix of the weight image (layers 0..7), then the
// whole gradient image, and loads only the tile's point-encoding blocks. As in nerf_mlp_wg_kernel, the producer's warpgroup gives its registers to the
// consumers (setmaxnreg 40 / 232): a backward epilogue holds a [64 x 256] fp32 accumulator (128 registers) beside its mask word, row exponents and
// addresses, which does not fit the 168 registers a 384-thread (or 288-thread: three warps on one sub-partition) launch otherwise allows.
// Per layer l the forward keeps the ReLU mask (fp16(acc) + fp16(b) > 0, the value __hmax2 keeps) as 128 bits per thread in shared memory, in the
// accumulator fragment's order, so the backward reads back exactly its own fragment's bits. The backward starts from dZ_7 = w_alpha (.) mask_7; each
// dZ_l is staged as fp16 in A blocks 0-3 (h is dead by then), every row scaled by a power of two that puts its largest |entry| in [2^14, 2^15)
// (a quad reduction, as the alpha dot), the exponents summed per row and undone in fp32 at the end: exact, so g is finite whenever fp32 allows.
// The encoding gradient: e = e_5 + e_0 in fp32, in that order, e_5 = dZ_5 . W_5[:, :input_ch] (the skip term), e_0 = dZ_0 . W_0. From step 2 to
// step 8, e_5 waits in shared memory as each thread's fp32 fragment (ng_park): in the warpgroup's halves of the encoding blocks, dead after the
// forward, then in a region of its own; the producer loads the next tile's encoding blocks only once both warpgroups have read it back (it issues
// that tile's layer-0 slabs first, so the weight ring keeps streaming across the tile boundary). e goes to shared memory as fp32 rows, and one
// thread per row contracts it with the encoding's derivative at the fp32 position the encoder formed: posenc_bands_grad at get_pts (NeRF), ipe_ray_grad at sample_gaussian's mean, covariance held fixed (Mip-NeRF).
constexpr int NG_THREADS = 384;
constexpr int NG_LAYERS = 8 + NG_STEPS;   // the producer's stream: forward layers 0..7, then the gradient steps

struct NgParams {
    const uint8_t *weight_image, *grad_image, *enc_image; const float *bias;
    const float *rays_o, *rays_d, *z_vals, *radii;
    int64_t n_rows; int S, min_deg;
    float *density, *grad;
    uint32_t slot_bytes; int n_slots;
    uint32_t n_slabs[NG_LAYERS]; uint32_t slab_bytes[NG_LAYERS][NM_MAX_SLABS];
};

// forward layers [L, 8) of my 64 rows: the epilogue of nm_layers (same roundings, same alpha dot order), plus the layer's mask bits
template <bool MIP, int L>
__device__ __forceinline__ void ng_forward(NmCtx &x, const float *bias, uint4 *mask, float *alpha) {
    if constexpr (L < 8) {
        constexpr NmLayer Ly = nm_layer<MIP>(L);
        float acc[128];
        tc::fence_proxy_async_smem();
        tc::named_bar_sync(1 + x.wg, 128);
        nm_slabs<MIP, L, 0>(x, acc);
        tc::acc_fence<128>(acc);
        tc::named_bar_sync(1 + x.wg, 128);
        const float *b = bias + Ly.bias_off, *wa = bias + 2448;
        float adot[2] = {0.f, 0.f};
        uint32_t m[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const uint32_t col = tc::frag_col(x.t, j);
            uint8_t *blk = x.A + (size_t)(col >> 6) * TILE_BLOCK_BYTES;
            const float b0 = __ldg(b + col), b1 = __ldg(b + col + 1);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                __half2 h = __hadd2(__floats2half2_rn(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]), __floats2half2_rn(b0, b1));
                h = __hmax2(h, __float2half2_rn(0.f));
                const float2 f = __half22float2(h);
                const int i = 4 * j + 2 * e;
                m[i >> 5] |= (f.x > 0.f ? 1u : 0u) << (i & 31) | (f.y > 0.f ? 2u : 0u) << (i & 31);
                if constexpr (L == 7) { adot[e] = fmaf(f.x, __ldg(wa + col), adot[e]); adot[e] = fmaf(f.y, __ldg(wa + col + 1), adot[e]); }
                else *reinterpret_cast<__half2 *>(sw128_elem(blk, x.r0 + 8u * (uint32_t)e, col & 63u)) = h;
            }
        }
        mask[L * 128] = make_uint4(m[0], m[1], m[2], m[3]);
        if constexpr (L == 7) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                adot[e] += __shfl_xor_sync(0xffffffffu, adot[e], 1);
                adot[e] += __shfl_xor_sync(0xffffffffu, adot[e], 2);
                alpha[e] = adot[e] + __ldg(wa + 256);
            }
        }
        ng_forward<MIP, L + 1>(x, bias, mask, alpha);
    }
}

// dZ = v (.) mask (v: the fragment of a [64 x 256] accumulator, mask: its bits) into A blocks 0-3 as fp16, row e scaled by 2^k with its largest
// |entry| then in [2^14, 2^15) (k = 0 for a zero row); sh[e] += k
__device__ __forceinline__ void ng_stage(const NmCtx &x, float *v, uint4 mq, int *sh) {
    const uint32_t mw[4] = {mq.x, mq.y, mq.z, mq.w};
    float mx[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 128; ++i) {
        if (!((mw[i >> 5] >> (i & 31)) & 1u)) v[i] = 0.f;
        mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], fabsf(v[i]));
    }
    float sc[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
        mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
        const int k = mx[e] > 0.f ? min(14 - (((__float_as_int(mx[e]) >> 23) & 255) - 127), 127) : 0;
        sh[e] += k;
        sc[e] = pow2i(k);
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const uint32_t col = tc::frag_col(x.t, j);
        uint8_t *blk = x.A + (size_t)(col >> 6) * TILE_BLOCK_BYTES;
#pragma unroll
        for (int e = 0; e < 2; ++e)
            *reinterpret_cast<__half2 *>(sw128_elem(blk, x.r0 + 8u * (uint32_t)e, col & 63u)) = __floats2half2_rn(v[4 * j + 2 * e] * sc[e], v[4 * j + 2 * e + 1] * sc[e]);
    }
}

// word i (< NP / 2) of the parked skip term of thread t of warpgroup wg: 8 KB chunks of 128 threads x 16 words, chunk c < AUX in the warpgroup's half
// of encoding block c, the others in the region after the encoding blocks
template <int AUX>
__device__ __forceinline__ float *ng_park(uint8_t *A, uint32_t wg, uint32_t t, int i) {
    const int c = i >> 4;
    uint8_t *chunk = c < AUX ? A + (size_t)(4 + c) * TILE_BLOCK_BYTES + wg * 8192u : A + (size_t)(4 + AUX) * TILE_BLOCK_BYTES + (uint32_t)(2 * (c - AUX) + (int)wg) * 8192u;
    return reinterpret_cast<float *>(chunk) + (i & 15) * 128 + t;
}

// gradient steps [G, 9) of my 64 rows; sh: the rows' exponents, sh5: those of the parked skip term e_5
template <bool MIP, int G>
__device__ __forceinline__ void ng_backward(NmCtx &x, const uint4 *mask, int *sh, int *sh5) {
    constexpr int AUX = MIP ? 2 : 1;
    if constexpr (G < NG_STEPS) {
        constexpr NmLayer Ly = ng_step<MIP>(G);
        tc::fence_proxy_async_smem();        // my staging writes -> visible to the tensor core
        tc::named_bar_sync(1 + x.wg, 128);
        if constexpr (G == 2) {
            float acc[Ly.N / 2];
            nm_slabs<MIP, G, 0, true>(x, acc);
            tc::acc_fence<Ly.N / 2>(acc);
#pragma unroll
            for (int i = 0; i < Ly.N / 2; ++i) *ng_park<AUX>(x.A, x.wg, x.t, i) = acc[i];
            sh5[0] = sh[0]; sh5[1] = sh[1];
        } else if constexpr (G == NG_STEPS - 1) {
            float acc[Ly.N / 2];
            nm_slabs<MIP, G, 0, true>(x, acc);
            tc::acc_fence<Ly.N / 2>(acc);
            tc::named_bar_sync(1 + x.wg, 128);   // dZ_0 has no reader left: A blocks 0-3 take e
            // e(row, c) as fp32 in A block c / 32, my warpgroup's half: 128-byte rows, word (c % 32) ^ (row % 32)
#pragma unroll
            for (int j = 0; j < Ly.N / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
#pragma unroll
                    for (int q = 0; q < 2; ++q) {
                        const int i = 4 * j + 2 * e + q;
                        const uint32_t col = tc::frag_col(x.t, j) + q, row = tc::frag_row(x.t) + 8u * e;
                        float *dst = reinterpret_cast<float *>(x.A + (size_t)(col >> 5) * TILE_BLOCK_BYTES + x.wg * 8192u + row * 128u) + ((col & 31u) ^ (row & 31u));
                        *dst = ldexpf(*ng_park<AUX>(x.A, x.wg, x.t, i), -sh5[e]) + ldexpf(acc[i], -sh[e]);
                    }
        } else {
            float acc[128];
            nm_slabs<MIP, G, 0, true>(x, acc);
            tc::acc_fence<128>(acc);
            tc::named_bar_sync(1 + x.wg, 128);   // every warp's share of this step's MMAs has completed before A blocks are rewritten
            constexpr int layer = G < 2 ? 7 - G : (G == 3 ? 5 : 8 - G);   // the layer whose input gradient this is: mask of layer - 1
            ng_stage(x, acc, mask[(layer - 1) * 128], sh);
        }
        ng_backward<MIP, G + 1>(x, mask, sh, sh5);
    }
}

template <bool MIP>
__global__ void __launch_bounds__(NG_THREADS, 1) nerf_grad_wg_kernel(const __grid_constant__ NgParams P) {
    extern __shared__ uint8_t dyn_smem[];
    constexpr int AUX = MIP ? 2 : 1;
    uint8_t *base = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    uint8_t *A = base, *ring = A + (size_t)(4 + 2 * AUX) * TILE_BLOCK_BYTES;   // hidden blocks, encoding blocks, the rest of the skip term's park
    uint4 *masks = (uint4 *)(ring + (size_t)P.n_slots * P.slot_bytes);   // [warpgroup][layer 0..7][thread 0..127]
    uint64_t *bars = (uint64_t *)(masks + 2 * 8 * 128);
    uint64_t *full = bars, *empty = bars + P.n_slots, *enc_full = bars + 2 * P.n_slots, *enc_free = enc_full + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < P.n_slots; ++s) { tc::mbar_init(full + s, 1); tc::mbar_init(empty + s, 8); }
        tc::mbar_init(enc_full, 1); tc::mbar_init(enc_free, 8);
        tc::fence_mbar_init();
    }
    __syncthreads();
    const int64_t n_tiles = (P.n_rows + 127) / 128;

    if (warp >= 8) {
        // ===================================================== TMA producer (one lane)
        tc::setmaxnreg_dec<40>();
        if (warp == 8 && lane == 0) {
            uint32_t it = 0, n = 0;
            for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++n) {
                size_t off = 0;
                for (int l = 0; l < NG_LAYERS; ++l) {
                    if (l == 1) {   // layer 0's slabs are in flight: now wait for the encoding blocks to be free (the parked skip term read back)
                        if (n > 0) tc::mbar_wait(enc_free, (n - 1) & 1);
                        tc::mbar_expect_tx(enc_full, AUX * TILE_BLOCK_BYTES);   // the tile's point blocks (the direction block is not read)
                        tc::tma_bulk_g2s(A + 4 * TILE_BLOCK_BYTES, P.enc_image + (size_t)tile * (AUX + 1) * TILE_BLOCK_BYTES, AUX * TILE_BLOCK_BYTES, enc_full);
                    }
                    if (l == 8) off = 0;
                    const uint8_t *img = l < 8 ? P.weight_image : P.grad_image;
                    for (uint32_t s = 0; s < P.n_slabs[l]; ++s, ++it) {
                        const uint32_t slot = it % P.n_slots, round = it / P.n_slots, bytes = P.slab_bytes[l][s];
                        if (round > 0) tc::mbar_wait(empty + slot, (round - 1) & 1);
                        tc::mbar_expect_tx(full + slot, bytes);
                        tc::tma_bulk_g2s(ring + (size_t)slot * P.slot_bytes, img + off, bytes, full + slot);
                        off += bytes;
                    }
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
    uint4 *mask = masks + x.wg * 8 * 128 + x.t;
    const float *wa = P.bias + 2448;
    uint32_t n = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++n) {
        tc::mbar_wait(enc_full, n & 1);
        float alpha[2] = {0.f, 0.f};
        ng_forward<MIP, 0>(x, P.bias, mask, alpha);
        if (P.density && (x.t & 3u) == 0) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int64_t i = tile * 128 + x.r0 + 8 * e;
                if (i < P.n_rows) P.density[i] = alpha[e];
            }
        }
        // dZ_7 = w_alpha (.) mask_7
        int sh[2] = {0, 0}, sh5[2] = {0, 0};
        {
            float v[128];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const uint32_t col = tc::frag_col(x.t, j);
                const float w0 = __ldg(wa + col), w1 = __ldg(wa + col + 1);
                v[4 * j] = w0; v[4 * j + 1] = w1; v[4 * j + 2] = w0; v[4 * j + 3] = w1;
            }
            ng_stage(x, v, mask[7 * 128], sh);
        }
        ng_backward<MIP, 0>(x, mask, sh, sh5);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(enc_free);   // the parked skip term has been read back: the producer may load the next tile's encoding blocks
        tc::named_bar_sync(1 + x.wg, 128);   // e of every row of my warpgroup is in shared memory
        if (x.t < 64) {
            const int64_t i = tile * 128 + 64 * x.wg + x.t;
            if (i < P.n_rows) {
                const uint32_t row = x.t;
                auto e = [&](int c) {
                    return *(reinterpret_cast<const float *>(A + (size_t)(c >> 5) * TILE_BLOCK_BYTES + x.wg * 8192u + row * 128u) + (((uint32_t)c & 31u) ^ (row & 31u)));
                };
                const int64_t ray = i / P.S; const int k = (int)(i - ray * P.S);
                float g[3];
                if constexpr (MIP) {
                    float mean[3], cov[3];
                    sample_gaussian(P.z_vals, P.rays_o, P.rays_d, P.radii, P.S, ray, k, mean, cov);
                    ipe_ray_grad<16>(mean, cov, P.min_deg, e, g);
                } else {
                    float p[3];
                    get_pts(P.rays_o, P.rays_d, ray, P.z_vals[i], p);
                    posenc_bands_grad<10>(p, 10, e, g);
                }
#pragma unroll
                for (int a = 0; a < 3; ++a) P.grad[3 * i + a] = g[a];
            }
        }
        // the next tile's layer 0 barrier orders these reads before its epilogue rewrites A blocks 0-3
    }
}

// the per-ray normal: sum over k from 0 of w_k n_k, n_k = -g_k / norm3df(g_k), 0 where g_k = 0. One thread per ray.
__global__ void __launch_bounds__(256) composite_normals_kernel(const float *__restrict__ weights, const float *__restrict__ grad, int n_rays, int S, float *__restrict__ out) {
    const int ray = blockIdx.x * 256 + threadIdx.x;
    if (ray >= n_rays) return;
    float n0 = 0.f, n1 = 0.f, n2 = 0.f;
    for (int k = 0; k < S; ++k) {
        const int64_t i = (int64_t)ray * S + k;
        const float w = __ldg(weights + i), gx = __ldg(grad + 3 * i), gy = __ldg(grad + 3 * i + 1), gz = __ldg(grad + 3 * i + 2);
        const float nrm = norm3df(gx, gy, gz);
        if (nrm > 0.f) { n0 += w * (-gx / nrm); n1 += w * (-gy / nrm); n2 += w * (-gz / nrm); }
    }
    out[3 * (int64_t)ray] = n0; out[3 * (int64_t)ray + 1] = n1; out[3 * (int64_t)ray + 2] = n2;
}

// the shared part of the two gradient entries after their own checks: pointers, alignment, schedule, launch
static int ng_density_grad(const char *who, bool mip, const void *weight_image, const void *grad_image, const float *bias, const void *enc_image, const float *rays_o,
                           const float *rays_d, const float *z_vals, const float *radii, int n_rays, int S, int min_deg, float *density_out, float *grad_out, void *stream) {
    const std::string w = who;
    XRB_REQUIRE(weight_image && grad_image && bias && enc_image && rays_o && rays_d && z_vals && (radii || !mip) && grad_out, (w + ": null pointer").c_str());
    XRB_REQUIRE(((uintptr_t)weight_image & 15) == 0 && ((uintptr_t)grad_image & 15) == 0 && ((uintptr_t)bias & 15) == 0 && ((uintptr_t)enc_image & 15) == 0,
                (w + ": images / bias must be 16-byte aligned").c_str());
    NgParams P{};
    P.weight_image = (const uint8_t *)weight_image; P.grad_image = (const uint8_t *)grad_image; P.enc_image = (const uint8_t *)enc_image; P.bias = bias;
    P.rays_o = rays_o; P.rays_d = rays_d; P.z_vals = z_vals; P.radii = radii;
    P.n_rows = (int64_t)n_rays * S; P.S = S; P.min_deg = min_deg; P.density = density_out; P.grad = grad_out;
    uint32_t max_bytes = 0;
    for (int l = 0; l < NG_LAYERS; ++l) {
        const NmLayer L = l < 8 ? (mip ? nm_layer<true>(l) : nm_layer<false>(l)) : (mip ? ng_step<true>(l - 8) : ng_step<false>(l - 8));
        P.n_slabs[l] = (uint32_t)L.n_slabs;
        for (int k = 0; k < L.n_slabs; ++k) { P.slab_bytes[l][k] = nm_slab_bytes(L.s[k]); if (P.slab_bytes[l][k] > max_bytes) max_bytes = P.slab_bytes[l][k]; }
    }
    P.slot_bytes = (max_bytes + 1023) & ~1023u;
    P.n_slots = 4;
    const size_t smem = 1024 + (size_t)(4 + 2 * (mip ? 2 : 1)) * TILE_BLOCK_BYTES + (size_t)P.n_slots * P.slot_bytes + 2 * 8 * 128 * 16 + 8 * (2 * P.n_slots + 2);
    const int grid = persistent_grid(1, (P.n_rows + 127) / 128);
    auto k = mip ? nerf_grad_wg_kernel<true> : nerf_grad_wg_kernel<false>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<grid, NG_THREADS, smem, (cudaStream_t)stream>>>(P);
    return check_launch(who);
}

}  // namespace xrb

using namespace xrb;

extern "C" {

// the raw density and its gradient with respect to each sample's position, for the rows of a ray batch's encoding image. See include/xrnerf_b200.h.
int xrb_nerf_density_grad_rays(const void *weight_image, const void *grad_image, const float *bias, const void *enc_image, const float *rays_o, const float *rays_d,
                               const float *z_vals, int n_rays, int S, int input_ch, int input_ch_dirs, float *density_out, float *grad_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && S >= 1, "nerf_density_grad_rays: bad size (n_rays >= 0, S >= 1)");
    if (!(input_ch == 63 && input_ch_dirs == 27)) {
        set_error("nerf_density_grad_rays: implemented for the fused NerfMLP with BaseEmbedder(multires=10, multires_dirs=4), input channels (63, 27)");
        return XRB_E_UNSUPPORTED;
    }
    if (n_rays == 0) return XRB_OK;
    return ng_density_grad("nerf_density_grad_rays", false, weight_image, grad_image, bias, enc_image, rays_o, rays_d, z_vals, nullptr, n_rays, S, 0, density_out,
                           grad_out, stream);
}

// the Mip-NeRF form: positions are the means of the samples' frustum Gaussians (z_vals [n, S+1]). See include/xrnerf_b200.h.
int xrb_mip_density_grad_rays(const void *weight_image, const void *grad_image, const float *bias, const void *enc_image, const float *rays_o, const float *rays_d,
                              const float *z_vals, const float *radii, int n_rays, int S, int input_ch, int input_ch_dirs, int min_deg_point, int max_deg_point,
                              float *density_out, float *grad_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && S >= 1, "mip_density_grad_rays: bad size (n_rays >= 0, S >= 1)");
    if (!(input_ch == 96 && input_ch_dirs == 27 && max_deg_point - min_deg_point == 16 && min_deg_point >= -100 && max_deg_point <= 100)) {
        set_error("mip_density_grad_rays: implemented for the fused NerfMLP with the MipNerfEmbedder of 16 point and 4 view bands, input channels (96, 27)");
        return XRB_E_UNSUPPORTED;
    }
    if (n_rays == 0) return XRB_OK;
    return ng_density_grad("mip_density_grad_rays", true, weight_image, grad_image, bias, enc_image, rays_o, rays_d, z_vals, radii, n_rays, S, min_deg_point,
                           density_out, grad_out, stream);
}

// normal f32[n,3] <- sum_k w_k n_k of each ray. See include/xrnerf_b200.h.
int xrb_nerf_composite_normals(const float *weights, const float *grad, int n_rays, int S, float *normal_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && S >= 1, "nerf_composite_normals: bad size (n_rays >= 0, S >= 1)");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(weights && grad && normal_out, "nerf_composite_normals: null pointer");
    composite_normals_kernel<<<(n_rays + 255) / 256, 256, 0, (cudaStream_t)stream>>>(weights, grad, n_rays, S, normal_out);
    return check_launch("nerf_composite_normals");
}

}  // extern "C"
