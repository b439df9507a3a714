// xrnerf_b200 — the Instant-NGP field (hash encode -> density MLP -> SH concat -> colour MLP) evaluated by one
// 128-thread warpgroup on one 128-sample tile with wgmma tensor-core tiles. Used by ngp_mlp.cu (stand-alone
// HashNerfMLP.run_mlp) and ngp_fused.cu (fused render).
//
// Mapping (thread r of the warpgroup == sample r: it writes A row r and receives the field output of row r):
//   A tile   : [128 x 64] fp16, K-major, SWIZZLE_128B, 16 KB per warpgroup: the input of each net's FIRST layer (the encoding for density_net,
//              density outputs 1..15 ++ SH ++ 1 for color_net), one row per thread
//   weights  : packed once per optimiser step into the same swizzled layout (xrb_ngp_pack_weights), bulk-copied (TMA,
//              cp.async.bulk) into shared memory once per CTA and kept resident for the whole persistent kernel
//   per net  : the tile runs as two M=64 halves, one after the other. Per half the first layer (A from the shared-memory tile) is followed by a
//              register chain: the fp32 accumulator fragment of an m64n64 layer, ReLU'd and packed to fp16 pairs, IS the A fragment of the next layer's
//              K steps (tc.cuh wgmma_ra), so the hidden layers and the N=16 output layer need no st.shared, no proxy fence and no barrier, and each
//              warp's rows stay in that warp. A half holds 32 fp32 accumulators and 16 A registers per thread (the fused render kernel runs 768
//              threads per SM, i.e. at most 80 registers each).
//   outputs  : the N=16 output layer of each net goes through an 8 KB per-warpgroup staging tile, from which thread r reads row r.
#pragma once
#include "ngp_field.cuh"
#include "tc.cuh"

namespace xrb {

struct TcWarpgroup {
    uint8_t *A;        // this warpgroup's 16 KB A tile (1024-byte aligned shared memory)
    const uint8_t *W;  // weight image in shared memory (1024-byte aligned)
    float *stage;      // this warpgroup's [128 x 16] fp32 output staging tile (8 KB)
    uint32_t wg;       // warpgroup index inside the CTA (named barrier id = bar_base + wg)
    uint32_t row;      // 0..127
    uint32_t bar;      // named barrier id of this warpgroup
};
constexpr uint32_t TC_STAGE_BYTES = 128 * 16 * 4;

__device__ __forceinline__ void a_store_chunk(const TcWarpgroup &c, uint32_t chunk, uint4 v) { st_chunk(c.A + sw128_offset(c.row, chunk), v); }
__device__ __forceinline__ void tc_bar(const TcWarpgroup &c) { tc::named_bar_sync(c.bar, 128); }

// accumulator (fp32 pair) -> fp16 -> ReLU. Rounding to fp16 first and clamping the packed pair (one cvt.rn.f16x2 + one max.f16x2 per two values)
// gives the same bits as clamp-then-round: rounding is monotone and maps 0 to 0.
__device__ __forceinline__ uint32_t pack_relu_h2f(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    h = __hmax2(h, __float2half2_rn(0.f));
    return *reinterpret_cast<uint32_t *>(&h);
}
// m64n64 accumulator -> ReLU(fp16) A fragment of the next layer: K step s = accumulator registers 8s..8s+7 (tc.cuh wgmma_ra)
__device__ __forceinline__ void acc_relu_to_a(const float *acc, uint32_t *a) {
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = pack_relu_h2f(acc[2 * i], acc[2 * i + 1]);
}

// first layer of a net on half h of the tile: D[64 x 64] = A[rows 64h.., K] * W[64 x K]^T, issued (not waited for)
template <int K>
__device__ __forceinline__ void tc_first_issue(const TcWarpgroup &c, uint32_t w_off, int h, float *acc) {
    const uint32_t a0 = tc::smem_u32(c.A) + (uint32_t)h * 8192u, b0 = tc::smem_u32(c.W + w_off);
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < K / 16; ++k) tc::wgmma<64>(acc, tc::desc_k128(a0 + k * 32), tc::desc_k128(b0 + k * 32), k > 0 ? 1u : 0u);
    tc::wg_commit();
}
// chained layer: D[64 x N] = a[64 x 64] * W[N x 64]^T with a in registers, issued (not waited for)
template <int N>
__device__ __forceinline__ void tc_chain_issue(const TcWarpgroup &c, uint32_t w_off, const uint32_t *a, float *acc) {
    const uint32_t b0 = tc::smem_u32(c.W + w_off);
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) tc::wgmma_ra<N>(acc, a + 4 * k, tc::desc_k128(b0 + k * 32), k > 0 ? 1u : 0u);
    tc::wg_commit();
}
template <int N>
__device__ __forceinline__ void tc_wait_all(float *acc) {
    tc::wg_wait<0>();
    tc::acc_fence<N>(acc);
}
// my st.shared of the A rows -> visible to the tensor core (async proxy), and every row of the warpgroup written
__device__ __forceinline__ void tc_sync_a(const TcWarpgroup &c) {
    tc::fence_proxy_async_smem();
    tc_bar(c);
}

// output fragment of half h of an N=16 layer -> staging tile (its own rows: no barrier needed before the stores)
__device__ __forceinline__ void tc_stage_half(const TcWarpgroup &c, int h, const float *acc) {
    // staging word of (row, col): row * 16 + (col ^ 4 (row & 3)) — conflict-free float2 stores, float4 loads of a row
    const uint32_t r = 64u * (uint32_t)h + tc::frag_row(c.row);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const uint32_t col = tc::frag_col(c.row, j);
        *reinterpret_cast<float2 *>(c.stage + r * 16 + (col ^ ((r & 3u) << 2))) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2 *>(c.stage + (r + 8) * 16 + (col ^ (((r + 8) & 3u) << 2))) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
}
// One net (first layer from the A tile, n_hidden - 1 chained hidden layers, chained N=16 output layer) on the whole tile; thread r receives the 16 fp32
// outputs of row r. Hidden layer l's weights follow the first layer's at w_in + 8192 (l + 1) (weight_image_layout; computed, so that no layout array is
// indexed at run time, which would put it in local memory). The A tile must have been published (tc_sync_a). Half 1's first layer is issued while half 0's
// output layer is still in flight.
template <int K_IN>
__device__ __forceinline__ void tc_net(const TcWarpgroup &c, uint32_t w_in, int n_hidden, uint32_t w_out, float *out) {
    float acc[32], acc16[8];
    uint32_t a[16];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        tc_first_issue<K_IN>(c, w_in, h, acc);
        tc_wait_all<32>(acc);   // (h = 1: also half 0's output layer, the last reader of a)
        if (h == 1) { tc::acc_fence<8>(acc16); tc_stage_half(c, 0, acc16); }
        acc_relu_to_a(acc, a);
        for (int l = 0; l < n_hidden - 1; ++l) {
            tc_chain_issue<64>(c, w_in + 8192u * (uint32_t)(l + 1), a, acc);
            tc_wait_all<32>(acc);
            acc_relu_to_a(acc, a);
        }
        tc_chain_issue<16>(c, w_out, a, acc16);
    }
    tc_wait_all<8>(acc16);
    tc_stage_half(c, 1, acc16);
    tc_bar(c);   // every row staged; also every warp's wgmma of the net has completed, so the A tile may be rewritten after this
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float4 v = *reinterpret_cast<const float4 *>(c.stage + c.row * 16 + (((uint32_t)k ^ (c.row & 3u)) << 2));
        out[4 * k] = v.x; out[4 * k + 1] = v.y; out[4 * k + 2] = v.z; out[4 * k + 3] = v.w;
    }
    // the staging tile is rewritten only after the next net's tc_sync_a barrier: every row has been read by then
}
// density_net on the tile, the 32 encoded features already sitting in chunks 0..3 of my A row: its 16 fp16-rounded outputs for my row
__device__ __forceinline__ void tc_density_from_a(const TcWarpgroup &c, const WeightImageLayout &L, int density_hidden, float *dout) {
    tc_sync_a(c);
    tc_net<32>(c, L.d_in, density_hidden, L.d_out, dout);
#pragma unroll
    for (int k = 0; k < 16; ++k) dout[k] = round_h(dout[k]);
}

// colour-net input row of my sample (color_input_row) -> my A row
__device__ __forceinline__ void tc_store_color_input(const TcWarpgroup &c, const float *dout, float dx, float dy, float dz) {
    float cin[32];
    color_input_row(dout, dx, dy, dz, cin);
#pragma unroll
    for (int q = 0; q < 4; ++q) a_store_chunk(c, q, pack_h8(cin + 8 * q));
}
// Colour half (HashNerfMLP.run_mlp, hashnerf_mlp.py:66-79) given density_net's outputs: raw = (rgb[3], density[1]) for my sample
__device__ __forceinline__ float4 tc_color_from_density(const TcWarpgroup &c, const WeightImageLayout &L, int color_hidden, const float *dout, float dx, float dy, float dz) {
    tc_store_color_input(c, dout, dx, dy, dz);
    tc_sync_a(c);
    float cout[16];
    tc_net<32>(c, L.c_in, color_hidden, L.c_out, cout);
    return make_float4(round_h(cout[0]), round_h(cout[1]), round_h(cout[2]), dout[0]);
}

// levels [L0, L1) of the hash encoding of one sample as packed half2 words
template <int NP, int L0, int L1>
__device__ __forceinline__ void tc_gather_levels(const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const HashGridDev &g, float x, float y, float z, uint32_t *e) {
#pragma unroll
    for (int l = L0; l < L1; ++l) { const float2 f = hash_level(table, cells, g, l, x, y, z, plan_mode<NP>(l)); e[l] = pack_h2(f.x, f.y); }
}
// ---- CTA-level setup shared by the kernels that use the warpgroup evaluator
// dynamic shared memory layout: [weights image][A tile x WG][staging tile x WG][mbarrier]
template <int WG>
__host__ __device__ inline size_t tc_cta_smem_bytes(uint32_t image_bytes) { return 1024 /*align slack*/ + image_bytes + (size_t)WG * (TILE_BLOCK_BYTES + TC_STAGE_BYTES) + 16; }

// Called by every thread of the CTA: bulk-copies (TMA) the weight image to the first 1024-byte aligned address of the dynamic shared memory, waits for it
// and returns that address. tiles_bytes: what the kernel keeps between the image (a multiple of 1024 bytes) and the copy's mbarrier.
__device__ __forceinline__ uint8_t *tc_load_weight_image(uint8_t *dyn_smem, const void *weight_image, uint32_t image_bytes, size_t tiles_bytes) {
    uint8_t *W = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    uint64_t *wbar = (uint64_t *)(W + image_bytes + tiles_bytes);
    if (threadIdx.x == 0) {
        tc::mbar_init(wbar, 1);
        tc::fence_mbar_init();
        tc::mbar_expect_tx(wbar, image_bytes);
        tc::tma_bulk_g2s(W, weight_image, image_bytes, wbar);
    }
    __syncthreads();
    tc::mbar_wait(wbar, 0);  // weights have landed
    return W;
}

template <int WG>
__device__ __forceinline__ TcWarpgroup tc_cta_setup(uint8_t *dyn_smem, const void *weight_image, uint32_t image_bytes) {
    uint8_t *W = tc_load_weight_image(dyn_smem, weight_image, image_bytes, (size_t)WG * (TILE_BLOCK_BYTES + TC_STAGE_BYTES));
    uint8_t *A0 = W + image_bytes;
    float *stage0 = (float *)(A0 + (size_t)WG * TILE_BLOCK_BYTES);
    TcWarpgroup c;
    c.wg = threadIdx.x >> 7; c.row = threadIdx.x & 127; c.bar = 1 + c.wg;
    c.A = A0 + (size_t)c.wg * TILE_BLOCK_BYTES; c.W = W; c.stage = stage0 + (size_t)c.wg * (TC_STAGE_BYTES / 4);
    return c;
}

}  // namespace xrb
