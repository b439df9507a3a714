// xrnerf_b200 — the Instant-NGP field (hash encode -> density MLP -> SH concat -> colour MLP) evaluated by one
// 128-thread warpgroup on one 128-sample tile with wgmma tensor-core tiles. Used by ngp_mlp.cu (stand-alone
// HashNerfMLP.run_mlp) and ngp_fused.cu (fused render).
//
// Mapping (thread r of the warpgroup == sample r: it writes A row r and receives the field output of row r):
//   A tile   : [128 x 64] fp16, K-major, SWIZZLE_128B, 16 KB per warpgroup, rewritten in place layer after layer
//   weights  : packed once per optimiser step into the same swizzled layout (xrb_ngp_pack_weights), bulk-copied (TMA,
//              cp.async.bulk) into shared memory once per CTA and kept resident for the whole persistent kernel
//   per layer: all threads write their A row (st.shared) -> fence.proxy.async -> warpgroup named barrier -> the warpgroup issues
//              K/16 wgmma.m64nNk16 for rows 0-63, waits, writes ReLU(fp16) of that half straight from the accumulator fragment into
//              the next A tile, then the same for rows 64-127. Halves run one after the other so that a layer holds 32 fp32 accumulator
//              registers per thread (the fused render kernel runs 768 threads per SM, i.e. at most 80 registers each).
//   outputs  : the two N=16 output layers go through an 8 KB per-warpgroup staging tile, from which thread r reads row r.
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

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ void a_store_chunk(const TcWarpgroup &c, uint32_t chunk, uint4 v) { *reinterpret_cast<uint4 *>(c.A + sw128_offset(c.row, chunk)) = v; }
__device__ __forceinline__ void tc_bar(const TcWarpgroup &c) { tc::named_bar_sync(c.bar, 128); }

// accumulator (fp32 pair) -> fp16 -> ReLU. Rounding to fp16 first and clamping the packed pair (one cvt.rn.f16x2 + one max.f16x2 per two values)
// gives the same bits as clamp-then-round: rounding is monotone and maps 0 to 0.
__device__ __forceinline__ uint32_t pack_relu_h2f(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    h = __hmax2(h, __float2half2_rn(0.f));
    return *reinterpret_cast<uint32_t *>(&h);
}

// D[64 x N] = A[rows 64h.., K] * W[N x K]^T, issued (not waited for)
template <int K, int N>
__device__ __forceinline__ void tc_half_issue(const TcWarpgroup &c, uint32_t w_off, int h, float *acc) {
    const uint32_t a0 = tc::smem_u32(c.A) + (uint32_t)h * 8192u, b0 = tc::smem_u32(c.W + w_off);
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < K / 16; ++k) tc::wgmma<N>(acc, tc::desc_k128(a0 + k * 32), tc::desc_k128(b0 + k * 32), k > 0 ? 1u : 0u);
    tc::wg_commit();
}
template <int N>
__device__ __forceinline__ void tc_half_wait(float *acc) {
    tc::wg_wait<0>();
    tc::acc_fence<N / 2>(acc);
}
// my st.shared of the A rows -> visible to the tensor core (async proxy), and every row of the warpgroup written
__device__ __forceinline__ void tc_sync_a(const TcWarpgroup &c) {
    tc::fence_proxy_async_smem();
    tc_bar(c);
}
// half h of a 64-wide accumulator -> ReLU(fp16) -> A rows 64h.. (the rows this thread's fragment holds)
__device__ __forceinline__ void tc_epilogue_relu_half(const TcWarpgroup &c, int h, const float *acc) {
    const uint32_t r = 64u * (uint32_t)h + tc::frag_row(c.row), q4 = (c.row & 3u) * 4u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t *>(c.A + sw128_offset(r, j) + q4) = pack_relu_h2f(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<uint32_t *>(c.A + sw128_offset(r + 8, j) + q4) = pack_relu_h2f(acc[4 * j + 2], acc[4 * j + 3]);
    }
}
// hidden layer: A (K wide) -> ReLU(A W^T) (64 wide) in place, split in two so that a caller can put independent work (the next tile's hash gather)
// between the issue of the first half and its wait:  float acc[32]; tc_hidden_begin<K>(c, w, acc); ...; tc_hidden_end<K>(c, w, acc);
template <int K>
__device__ __forceinline__ void tc_hidden_begin(const TcWarpgroup &c, uint32_t w_off, float *acc) {
    tc_sync_a(c);
    tc_half_issue<K, 64>(c, w_off, 0, acc);
}
template <int K>
__device__ __forceinline__ void tc_hidden_end(const TcWarpgroup &c, uint32_t w_off, float *acc) {
    tc_half_wait<64>(acc);
    tc_bar(c);   // every warp's share of this half's MMA has completed before A rows are overwritten
    tc_epilogue_relu_half(c, 0, acc);
    tc_half_issue<K, 64>(c, w_off, 1, acc);   // reads rows 64-127, which the epilogue above did not touch
    tc_half_wait<64>(acc);
    tc_bar(c);
    tc_epilogue_relu_half(c, 1, acc);
}
template <int K>
__device__ __forceinline__ void tc_hidden_layer(const TcWarpgroup &c, uint32_t w_off) {
    float acc[32];
    tc_hidden_begin<K>(c, w_off, acc);
    tc_hidden_end<K>(c, w_off, acc);
}
// output layer (N = 16): thread r receives the 16 fp32 outputs of row r;  float acc[16]; tc_output_begin(c, w, acc); ...; tc_output_end(c, acc, out);
__device__ __forceinline__ void tc_output_begin(const TcWarpgroup &c, uint32_t w_off, float *acc) {
    tc_sync_a(c);
    tc_half_issue<64, 16>(c, w_off, 0, acc);
    tc_half_issue<64, 16>(c, w_off, 1, acc + 8);
}
__device__ __forceinline__ void tc_output_end(const TcWarpgroup &c, float *acc, float *out) {
    tc::wg_wait<0>();
    tc::acc_fence<16>(acc);
    // staging word of (row, col): row * 16 + (col ^ 4 (row & 3)) — conflict-free float2 stores, float4 loads of a row
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t r = 64u * (uint32_t)h + tc::frag_row(c.row);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const uint32_t col = tc::frag_col(c.row, j);
            *reinterpret_cast<float2 *>(c.stage + r * 16 + (col ^ ((r & 3u) << 2))) = make_float2(acc[8 * h + 4 * j], acc[8 * h + 4 * j + 1]);
            *reinterpret_cast<float2 *>(c.stage + (r + 8) * 16 + (col ^ (((r + 8) & 3u) << 2))) = make_float2(acc[8 * h + 4 * j + 2], acc[8 * h + 4 * j + 3]);
        }
    }
    tc_bar(c);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float4 v = *reinterpret_cast<const float4 *>(c.stage + c.row * 16 + (((uint32_t)k ^ (c.row & 3u)) << 2));
        out[4 * k] = v.x; out[4 * k + 1] = v.y; out[4 * k + 2] = v.z; out[4 * k + 3] = v.w;
    }
    // the staging tile is rewritten only after the next layer's tc_sync_a barrier: every row has been read by then
}
__device__ __forceinline__ void tc_output_layer(const TcWarpgroup &c, uint32_t w_off, float *out) {
    float acc[16];
    tc_output_begin(c, w_off, acc);
    tc_output_end(c, acc, out);
}

// Density half of the field, the 32 encoded features already sitting in chunks 0..3 of my A row: density_net's 16 fp16-rounded outputs.
__device__ __forceinline__ void tc_density_from_a(TcWarpgroup &c, const WeightImageLayout &L, int density_hidden, float *dout) {
    tc_hidden_layer<32>(c, L.d_in);
    for (int h = 0; h < density_hidden - 1; ++h) tc_hidden_layer<64>(c, L.d_hid[h]);
    tc_output_layer(c, L.d_out, dout);
#pragma unroll
    for (int k = 0; k < 16; ++k) dout[k] = round_h(dout[k]);
}
template <int NP>
__device__ __forceinline__ void tc_density(TcWarpgroup &c, const WeightImageLayout &L, int density_hidden, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells,
                                           const HashGridDev &g, float x, float y, float z, float *dout) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        uint32_t e[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { float2 f = hash_level(table, cells, g, 4 * q + k, x, y, z, plan_mode<NP>(4 * q + k)); e[k] = pack_h2(f.x, f.y); }
        a_store_chunk(c, q, make_uint4(e[0], e[1], e[2], e[3]));
    }
    tc_density_from_a(c, L, density_hidden, dout);
}

// colour-net input row of my sample: density_out[1:16] (15) ++ SH (16) ++ 1.0 pad (tcnn.Network pads 31 -> 32 with ones)
__device__ __forceinline__ void tc_store_color_input(TcWarpgroup &c, const float *dout, float dx, float dy, float dz) {
    float sh[16];
    sh4(dx, dy, dz, sh);
    float cin[32];
#pragma unroll
    for (int k = 0; k < 15; ++k) cin[k] = dout[k + 1];
#pragma unroll
    for (int k = 0; k < 16; ++k) cin[15 + k] = sh[k];
    cin[31] = 1.0f;
#pragma unroll
    for (int q = 0; q < 4; ++q)
        a_store_chunk(c, q, make_uint4(pack_h2(cin[8 * q], cin[8 * q + 1]), pack_h2(cin[8 * q + 2], cin[8 * q + 3]), pack_h2(cin[8 * q + 4], cin[8 * q + 5]), pack_h2(cin[8 * q + 6], cin[8 * q + 7])));
}
// Colour half (HashNerfMLP.run_mlp, hashnerf_mlp.py:66-79) given density_net's outputs: raw = (rgb[3], density[1]) for my sample
__device__ __forceinline__ float4 tc_color_from_density(TcWarpgroup &c, const WeightImageLayout &L, int color_hidden, const float *dout, float dx, float dy, float dz) {
    tc_store_color_input(c, dout, dx, dy, dz);
    tc_hidden_layer<32>(c, L.c_in);
    for (int h = 0; h < color_hidden - 1; ++h) tc_hidden_layer<64>(c, L.c_hid[h]);
    float cout[16];
    tc_output_layer(c, L.c_out, cout);
    return make_float4(round_h(cout[0]), round_h(cout[1]), round_h(cout[2]), dout[0]);
}
// Whole field: hash encode + both nets
template <int NP>
__device__ __forceinline__ float4 tc_field(TcWarpgroup &c, const WeightImageLayout &L, int density_hidden, int color_hidden, const __half2 *__restrict__ table,
                                           const uint8_t *__restrict__ cells, const HashGridDev &g, float x, float y, float z, float dx, float dy, float dz) {
    float dout[16];
    tc_density<NP>(c, L, density_hidden, table, cells, g, x, y, z, dout);
    return tc_color_from_density(c, L, color_hidden, dout, dx, dy, dz);
}

// levels [L0, L1) of the hash encoding of one sample as packed half2 words
template <int NP, int L0, int L1>
__device__ __forceinline__ void tc_gather_levels(const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const HashGridDev &g, float x, float y, float z, uint32_t *e) {
#pragma unroll
    for (int l = L0; l < L1; ++l) { const float2 f = hash_level(table, cells, g, l, x, y, z, plan_mode<NP>(l)); e[l] = pack_h2(f.x, f.y); }
}
// One tile of the field with the NEXT tile's gather folded into the waits of this tile's tensor-core layers (the layers of a tile are a chain of
// issue -> wait round trips during which this warpgroup would otherwise load nothing).
//   e  : encoding of THIS tile's sample (16 packed half2), already gathered
//   en : receives the encoding of the next tile's sample at (xn, yn, zn) when has_next
// Same arithmetic, same order per sample: bit-identical to tc_density / tc_color_from_density.
template <int NP, bool DENSITY_ONLY>
__device__ __forceinline__ float4 tc_field_gather_ahead(TcWarpgroup &c, const WeightImageLayout &L, int density_hidden, int color_hidden, const __half2 *__restrict__ table,
                                                        const uint8_t *__restrict__ cells, const HashGridDev &g, const uint32_t *e, float dx, float dy, float dz, bool has_next, float xn, float yn,
                                                        float zn, uint32_t *en) {
#pragma unroll
    for (int q = 0; q < 4; ++q) a_store_chunk(c, q, make_uint4(e[4 * q], e[4 * q + 1], e[4 * q + 2], e[4 * q + 3]));
    float acc[32], acc16[16];
    tc_hidden_begin<32>(c, L.d_in, acc);
    if (has_next) tc_gather_levels<NP, 0, 3>(table, cells, g, xn, yn, zn, en);
    tc_hidden_end<32>(c, L.d_in, acc);
    for (int h = 0; h < density_hidden - 1; ++h) tc_hidden_layer<64>(c, L.d_hid[h]);
    float dout[16];
    tc_output_begin(c, L.d_out, acc16);
    if (has_next) tc_gather_levels<NP, 3, 6>(table, cells, g, xn, yn, zn, en);
    tc_output_end(c, acc16, dout);
#pragma unroll
    for (int k = 0; k < 16; ++k) dout[k] = round_h(dout[k]);
    if (DENSITY_ONLY) {
        if (has_next) tc_gather_levels<NP, 6, 16>(table, cells, g, xn, yn, zn, en);
        return make_float4(dout[0], 0.f, 0.f, 0.f);
    }
    tc_store_color_input(c, dout, dx, dy, dz);
    tc_hidden_begin<32>(c, L.c_in, acc);
    if (has_next) tc_gather_levels<NP, 6, 9>(table, cells, g, xn, yn, zn, en);
    tc_hidden_end<32>(c, L.c_in, acc);
    for (int h = 0; h < color_hidden - 1; ++h) {
        tc_hidden_begin<64>(c, L.c_hid[h], acc);
        if (h == 0 && has_next) tc_gather_levels<NP, 9, 12>(table, cells, g, xn, yn, zn, en);
        tc_hidden_end<64>(c, L.c_hid[h], acc);
    }
    if (color_hidden < 2 && has_next) tc_gather_levels<NP, 9, 12>(table, cells, g, xn, yn, zn, en);
    float cout[16];
    tc_output_begin(c, L.c_out, acc16);
    if (has_next) tc_gather_levels<NP, 12, 16>(table, cells, g, xn, yn, zn, en);
    tc_output_end(c, acc16, cout);
    return make_float4(round_h(cout[0]), round_h(cout[1]), round_h(cout[2]), dout[0]);
}

// ---- CTA-level setup shared by the kernels that use the warpgroup evaluator
// dynamic shared memory layout: [weights image][A tile x WG][staging tile x WG][mbarrier]
template <int WG>
__host__ __device__ inline size_t tc_cta_smem_bytes(uint32_t image_bytes) { return 1024 /*align slack*/ + image_bytes + (size_t)WG * (16384 + TC_STAGE_BYTES) + 16; }

template <int WG>
__device__ __forceinline__ TcWarpgroup tc_cta_setup(uint8_t *dyn_smem, const void *weight_image, uint32_t image_bytes) {
    uint8_t *base = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    uint8_t *W = base, *A0 = base + image_bytes;  // image_bytes is a multiple of 1024
    float *stage0 = (float *)(A0 + (size_t)WG * 16384);
    uint64_t *wbar = (uint64_t *)((uint8_t *)stage0 + (size_t)WG * TC_STAGE_BYTES);
    if (threadIdx.x == 0) {
        tc::mbar_init(wbar, 1);
        tc::fence_mbar_init();
        tc::mbar_expect_tx(wbar, image_bytes);
        tc::tma_bulk_g2s(W, weight_image, image_bytes, wbar);
    }
    __syncthreads();
    tc::mbar_wait(wbar, 0);  // weights have landed
    TcWarpgroup c;
    c.wg = threadIdx.x >> 7; c.row = threadIdx.x & 127; c.bar = 1 + c.wg;
    c.A = A0 + (size_t)c.wg * 16384; c.W = W; c.stage = stage0 + (size_t)c.wg * (TC_STAGE_BYTES / 4);
    return c;
}

}  // namespace xrb
