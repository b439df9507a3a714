// xrnerf_b200 — backward of the Instant-NGP field (HashNerfMLP.run_mlp, /root/reference/xrnerf/models/mlps/hashnerf_mlp.py:55-79: what tcnn's
// backward computes behind it) on wgmma tensor-core tiles. Replaces the CUDA-core kernel of ngp_backward.cu on the training path (that kernel
// stays as impl 0: reference-grade arithmetic for every (density_hidden, color_hidden) and the comparator of the tests).
//
// One persistent kernel, two warpgroups per CTA, each working on its own 128-sample tile (thread r == sample r == row r of every
// shared-memory tile). Per tile:
//   forward recompute   hash gather -> ENC tile -> density net -> CIN tile (density features ++ SH ++ 1) -> colour hidden layers; every layer
//                       INPUT stays in shared memory as a [128 x 64] fp16 tile (K-major, 128-byte swizzle: the wgmma operand layout);
//   backward chain      per layer ONE round of tensor-core work issued by the warpgroup:
//                         dX  = dZ . W            M=64 (samples, two halves), N=in, K=out : A = dZ tile (K-major), B = the FORWARD weight image read
//                                                 MN-major (W[out][in] rows are `in`-contiguous: no transposed weight copy exists)
//                         dW += dZ^T . X          M=64 (out features), N=in, K=128 samples : both operands are the sample tiles read MN-major
//                                                 (contraction over ROWS); the accumulators stay in registers for the whole persistent loop
//                       then the epilogue masks dX with ReLU'(activation) and writes the next dZ tile (fp16, fixed 2^12 scale like the CUDA-core
//                       kernel; tcnn uses fp16 gradients with a loss scale);
//   scatter             dL/d(encoding) -> fp32 hash-table gradient with vector atomics (red.global.add.v4.f32 / v2).
// At the end each warpgroup adds its dW accumulators to the fp32 gradient with atomics.
// Shared memory: weight image + 2 x (ENC, H.., CIN, C.., dZ) tiles. Row-wise reads of accumulators (density outputs, dL/dcin, dL/dencoding) are
// staged through a tile that is dead at that point (fp32 [128 x 16|32]).
#include <cstdio>

#include "tc_field.cuh"

namespace xrb {

constexpr float BT_SCALE = 4096.f;        // dZ staging scale (fp16): |dL/draw| < 16 stays finite, 1e-8 stays normal

struct BtWg {
    uint8_t *tiles;      // this warpgroup's tiles, TILE_BLOCK_BYTES bytes each
    const uint8_t *W;    // forward weight image (shared by both warpgroups)
    uint32_t wg, row, bar;
    bool first;          // first tile of this warpgroup: dW accumulators are overwritten, not accumulated
};

__device__ __forceinline__ uint8_t *bt_tile(const BtWg &c, int t) { return c.tiles + (size_t)t * TILE_BLOCK_BYTES; }
__device__ __forceinline__ void bt_store_chunk(const BtWg &c, int t, uint32_t chunk, uint4 v) { st_chunk(bt_tile(c, t) + sw128_offset(c.row, chunk), v); }
__device__ __forceinline__ void bt_bar(const BtWg &c) { tc::named_bar_sync(c.bar, 128); }
// my smem writes -> visible to the tensor core; every row of the warpgroup written
__device__ __forceinline__ void bt_sync(const BtWg &c) { tc::fence_proxy_async_smem(); bt_bar(c); }

// D[64 x N] of rows 64h.. = X[rows 64h.., K] . W[N x K]^T (both K-major)
template <int K, int N>
__device__ __forceinline__ void bt_fwd_issue(const BtWg &c, int x_tile, uint32_t w_off, int h, float *acc) {
    const uint32_t a0 = tc::smem_u32(bt_tile(c, x_tile)) + (uint32_t)h * 8192u, b0 = tc::smem_u32(c.W + w_off);
#pragma unroll
    for (int k = 0; k < K / 16; ++k) tc::wgmma<N>(acc, tc::desc_k128(a0 + k * 32), tc::desc_k128(b0 + k * 32), k > 0 ? 1u : 0u);
}
// the fp16 pair at (row r, columns col, col+1) of tile t
__device__ __forceinline__ uint32_t *bt_word(const BtWg &c, int t, uint32_t r, uint32_t col) {
    return reinterpret_cast<uint32_t *>(bt_tile(c, t) + sw128_offset(r, col >> 3) + (col & 7u) * 2u);   // written out: through sw128_elem this kernel allocates registers differently
}
// forward hidden layer: out_tile = ReLU(fp16(X W^T)), 64 wide
template <int K>
__device__ __forceinline__ void bt_fwd_hidden(const BtWg &c, int x_tile, uint32_t w_off, int out_tile) {
    bt_sync(c);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float acc[32];
        tc::wg_fence();
        bt_fwd_issue<K, 64>(c, x_tile, w_off, h, acc);
        tc::wg_commit();
        tc::wg_wait<0>();
        tc::acc_fence<32>(acc);
        const uint32_t r = 64u * (uint32_t)h + tc::frag_row(c.row);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t col = tc::frag_col(c.row, j);
            *bt_word(c, out_tile, r, col) = pack_relu_h2f(acc[4 * j], acc[4 * j + 1]);
            *bt_word(c, out_tile, r + 8, col) = pack_relu_h2f(acc[4 * j + 2], acc[4 * j + 3]);
        }
    }
}
// accumulator fragments of both halves (N columns) -> fp32 [128 x N] staging in tile `st` (swizzled: word (r, c) at r*N + (c ^ 4 (r % (N/4))))
// -> thread r reads row r. Barriers: before (other warps' MMAs of this round may still read the tile), between, after (the tile is rewritten next).
template <int N>
__device__ __forceinline__ void bt_stage_rows(const BtWg &c, int st, const float *acc0, const float *acc1, float *out) {
    float *sp = reinterpret_cast<float *>(bt_tile(c, st));
    constexpr uint32_t SW = N / 4 - 1;
    bt_bar(c);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float *acc = h ? acc1 : acc0;
        const uint32_t r = 64u * (uint32_t)h + tc::frag_row(c.row);
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            const uint32_t col = tc::frag_col(c.row, j);
            *reinterpret_cast<float2 *>(sp + r * N + (col ^ ((r & SW) << 2))) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2 *>(sp + (r + 8) * N + (col ^ (((r + 8) & SW) << 2))) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
    }
    bt_bar(c);
#pragma unroll
    for (int k = 0; k < N / 4; ++k) {
        const float4 v = *reinterpret_cast<const float4 *>(sp + c.row * N + (((uint32_t)k ^ (c.row & SW)) << 2));
        out[4 * k] = v.x; out[4 * k + 1] = v.y; out[4 * k + 2] = v.z; out[4 * k + 3] = v.w;
    }
    bt_bar(c);
}
// forward output layer (N = 16): thread r receives the 16 fp32 outputs of row r (staged through tile `st`)
__device__ __forceinline__ void bt_fwd_out(const BtWg &c, int x_tile, uint32_t w_off, int st, float *out) {
    bt_sync(c);
    float acc[2][8];
    tc::wg_fence();
    bt_fwd_issue<64, 16>(c, x_tile, w_off, 0, acc[0]);
    bt_fwd_issue<64, 16>(c, x_tile, w_off, 1, acc[1]);
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::acc_fence<8>(acc[0]); tc::acc_fence<8>(acc[1]);
    bt_stage_rows<16>(c, st, acc[0], acc[1], out);
}

// input gradient of one layer with OUT outputs and IN inputs, issued (not committed): dX[128 x IN] = dZ[128 x OUT] . W[OUT x IN] as two M=64 halves,
// contraction over OUT; A = the dZ tile at z0 (K-major), B = the forward weight image W[OUT rows][IN cols] at w0 read MN-major (N = IN contiguous, K = OUT rows)
template <int IN, int OUT>
__device__ __forceinline__ void bt_dx_issue(uint32_t z0, uint32_t w0, float (*acc)[IN / 2]) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < OUT / 16; ++k) tc::wgmma<IN, 0, 1>(acc[h], tc::desc_k128(z0 + h * 8192 + k * 32), tc::desc_mn128(w0 + k * 2048, 1024), k > 0 ? 1u : 0u);
}
// what happens to a completed dX (accumulators fenced):
// EPI 0: dZ tile := fp16(dX) * [act > 0] (act_tile);  EPI 1: thread r receives dX row r in `out` (fp32, staged through tile `st`)
template <int IN, int EPI>
__device__ __forceinline__ void bt_dx_epilogue(const BtWg &c, float (*acc)[IN / 2], int dz_tile, int act_tile, int st, float *out) {
    if (EPI == 1) { bt_stage_rows<IN>(c, st, acc[0], acc[1], out); return; }
    bt_bar(c);   // every warp's share of the MMAs that read the dZ rows has completed before dZ is overwritten
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t r = 64u * (uint32_t)h + tc::frag_row(c.row);
#pragma unroll
        for (int j = 0; j < IN / 8; ++j) {
            const uint32_t col = tc::frag_col(c.row, j);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const uint32_t rr = r + 8u * (uint32_t)e;
                const __half2 g = __floats2half2_rn(acc[h][4 * j + 2 * e], acc[h][4 * j + 2 * e + 1]);
                const __half2 a = *reinterpret_cast<const __half2 *>(bt_word(c, act_tile, rr, col));
                const __half2 o = __hmul2(g, __hgt2(a, __float2half2_rn(0.f)));   // 1.0 / 0.0 per half
                *bt_word(c, dz_tile, rr, col) = *reinterpret_cast<const uint32_t *>(&o);
            }
        }
    }
}
// backward round of one layer with OUT outputs and IN inputs:
//   dX[128 x IN] = dZ[128 x OUT] . W[OUT x IN]          (bt_dx_issue, then bt_dx_epilogue<IN, EPI>)
//   dW accumulators (registers, M = 64):
//     OUT == 64:  D[m = out][n = in]  += dZ^T X   (A = dZ tile, B = X tile, N = IN)            IN/2 registers
//     OUT == 16:  D[m = in][n = out]  += X^T dZ   (A = X tile (IN == 64), B = dZ tile, N = 16)   8 registers, stored transposed at the flush
template <int IN, int OUT, int EPI>
__device__ __forceinline__ void bt_bwd(const BtWg &c, int dz_tile, int x_tile, uint32_t w_off, float *dw, int act_tile, int st, float *out) {
    constexpr int DWN = OUT == 64 ? IN : 16;
    bt_sync(c);
    const uint32_t z0 = tc::smem_u32(bt_tile(c, dz_tile)), x0 = tc::smem_u32(bt_tile(c, x_tile)), w0 = tc::smem_u32(c.W + w_off);
    float acc[2][IN / 2];
    tc::wg_fence();
    // weight gradient: contraction over the 128 sample rows, 16 rows (2 x 1024 bytes) per instruction
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t sc = (k > 0 || !c.first) ? 1u : 0u;
        if (OUT == 64) tc::wgmma<DWN, 1, 1>(dw, tc::desc_mn128(z0 + k * 2048, 1024), tc::desc_mn128(x0 + k * 2048, 1024), sc);
        else tc::wgmma<DWN, 1, 1>(dw, tc::desc_mn128(x0 + k * 2048, 1024), tc::desc_mn128(z0 + k * 2048, 1024), sc);
    }
    bt_dx_issue<IN, OUT>(z0, w0, acc);
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::acc_fence<DWN / 2>(dw); tc::acc_fence<IN / 2>(acc[0]); tc::acc_fence<IN / 2>(acc[1]);
    bt_dx_epilogue<IN, EPI>(c, acc, dz_tile, act_tile, st, out);
}
// the input-gradient half of bt_bwd alone (no weight gradient): a chain that differentiates with respect to the inputs only
template <int IN, int OUT, int EPI>
__device__ __forceinline__ void bt_bwd_dx(const BtWg &c, int dz_tile, uint32_t w_off, int act_tile, int st, float *out) {
    bt_sync(c);
    float acc[2][IN / 2];
    tc::wg_fence();
    bt_dx_issue<IN, OUT>(tc::smem_u32(bt_tile(c, dz_tile)), tc::smem_u32(c.W + w_off), acc);
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::acc_fence<IN / 2>(acc[0]); tc::acc_fence<IN / 2>(acc[1]);
    bt_dx_epilogue<IN, EPI>(c, acc, dz_tile, act_tile, st, out);
}
// 16 fp32 values -> chunks 0,1 of tile t (fp16)
__device__ __forceinline__ void bt_store16(const BtWg &c, int t, const float *v) {
    bt_store_chunk(c, t, 0, pack_h8(v));
    bt_store_chunk(c, t, 1, pack_h8(v + 8));
}

// flush one M=64 dW accumulator (fragment rows m = frag_row (+8), columns n) into the fp32 gradient
// TRANSPOSED == false: D[m = out][n = in] -> dW[out][in] (row length in_w);  true: D[m = in][n = out] -> dW[out][in]
template <int N, bool TRANSPOSED>
__device__ __forceinline__ void bt_flush(const BtWg &c, const float *acc, float *__restrict__ dW, int in_w) {
    const uint32_t m0 = tc::frag_row(c.row);
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t m = m0 + 8u * (uint32_t)(i >> 1), n = tc::frag_col(c.row, j) + (uint32_t)(i & 1);
            float *dst = TRANSPOSED ? dW + (size_t)n * in_w + m : dW + (size_t)m * in_w + n;
            atomicAdd(dst, acc[4 * j + i] * (1.f / BT_SCALE));
        }
}

struct BtLayout {   // tile indices for (DH, CH)
    int enc, h0, cin, c0, dz, n_tiles;
    };
__host__ __device__ constexpr BtLayout bt_layout(int DH, int CH) {
    BtLayout L{};
    L.enc = 0; L.h0 = 1; L.cin = 1 + DH; L.c0 = 2 + DH; L.dz = 2 + DH + CH; L.n_tiles = 3 + DH + CH;
    return L;
}
template <int DH, int CH>
__host__ __device__ constexpr size_t bt_smem_bytes(uint32_t image_bytes) { return 1024 + image_bytes + 2 * (size_t)bt_layout(DH, CH).n_tiles * TILE_BLOCK_BYTES + 16; }

// The body of both field backward kernels. INPUTS (ngp_field_bwd_tc_inputs_kernel, xrb_ngp_mlp_backward_tc_inputs): also d_rows f32[n,6] = (dL/dx, dL/dw)
// of each row: dL/dSH through sh4_grad right after the colour net's input round, dL/d(encoding) through position_grad_level inside the scatter loop. The
// parameter gradients are those of ngp_field_bwd_tc_kernel: same operands, same order.
template <int DH, int CH, int NP, bool INPUTS>
__device__ __forceinline__ void ngp_field_bwd_tc(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const void *__restrict__ weight_image,
                                                 uint32_t image_bytes, const float *__restrict__ pts, int pts_stride, const float *__restrict__ dirs, int dirs_stride,
                                                 const float4 *__restrict__ dl_draw, int n, const int32_t *__restrict__ n_dev, float *__restrict__ d_table,
                                                 float *__restrict__ d_dens, float *__restrict__ d_color, float *__restrict__ d_rows) {
    extern __shared__ uint8_t dyn_smem[];
    if (n_dev) n = min(n, max(*n_dev, 0));
    constexpr BtLayout T = bt_layout(DH, CH);
    uint8_t *W = tc_load_weight_image(dyn_smem, weight_image, image_bytes, 2 * (size_t)T.n_tiles * TILE_BLOCK_BYTES);
    uint8_t *tiles0 = W + image_bytes;
    BtWg c;
    c.wg = threadIdx.x >> 7; c.row = threadIdx.x & 127; c.bar = 1 + c.wg;
    c.tiles = tiles0 + (size_t)c.wg * T.n_tiles * TILE_BLOCK_BYTES; c.W = W; c.first = true;
    const WeightImageLayout L = weight_image_layout(DH, CH);
    // weight-gradient accumulators of this warpgroup, in registers for the whole persistent loop (M = 64 fragments)
    float dw_din[16], dw_dhid[DH > 1 ? DH - 1 : 1][32], dw_dout[8], dw_cin[16], dw_chid[CH > 1 ? CH - 1 : 1][32], dw_cout[8];

    const int n_tiles = (n + 127) / 128;
    for (int tile = blockIdx.x * 2 + c.wg; tile < n_tiles; tile += gridDim.x * 2) {
        const int i = tile * 128 + c.row;
        const bool valid = i < n;
        float px = 0.5f, py = 0.5f, pz = 0.5f, dx = 0.5f, dy = 0.5f, dz = 0.5f;
        float4 gr = make_float4(0.f, 0.f, 0.f, 0.f);       // padding rows: zero dL/draw -> every dZ row of theirs is zero -> no contribution to any gradient
        if (valid) {
            const float *pp = pts + (size_t)i * pts_stride; px = pp[0]; py = pp[1]; pz = pp[2];
            const float *dd = dirs + (size_t)i * dirs_stride; dx = dd[0]; dy = dd[1]; dz = dd[2];
            gr = __ldg(dl_draw + i);
        }
        // ------------------------------------------------ forward recompute: every layer input parked as a tile
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            uint32_t e[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float2 f = hash_level(table, cells, g, 4 * q + k, px, py, pz, plan_mode<NP>(4 * q + k));
                e[k] = pack_h2(f.x, f.y);
            }
            bt_store_chunk(c, T.enc, q, make_uint4(e[0], e[1], e[2], e[3]));
        }
        float genc[32];
        bt_fwd_hidden<32>(c, T.enc, L.d_in, T.h0);
#pragma unroll
        for (int h = 1; h < DH; ++h) bt_fwd_hidden<64>(c, T.h0 + h - 1, L.d_hid[h - 1], T.h0 + h);
        {
            float dout[16], cin[32];
            bt_fwd_out(c, T.h0 + DH - 1, L.d_out, T.dz, dout);    // dZ is free until the colour backward
            color_input_row(dout, dx, dy, dz, cin);                   // fp16 rounding happens in the pack below (round(round(x)) == round(x))
#pragma unroll
            for (int q = 0; q < 4; ++q)
                bt_store_chunk(c, T.cin, q, pack_h8(cin + 8 * q));
        }
        bt_fwd_hidden<32>(c, T.cin, L.c_in, T.c0);
#pragma unroll
        for (int h = 1; h < CH; ++h) bt_fwd_hidden<64>(c, T.c0 + h - 1, L.c_hid[h - 1], T.c0 + h);
        // (the colour output layer itself is not needed: dL/draw is given)
        // ------------------------------------------------ backward: colour net
        {
            float gy[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) gy[k] = 0.f;
            gy[0] = gr.x * BT_SCALE; gy[1] = gr.y * BT_SCALE; gy[2] = gr.z * BT_SCALE;
            bt_store16(c, T.dz, gy);
        }
        bt_bwd<64, 16, 0>(c, T.dz, T.c0 + CH - 1, L.c_out, dw_cout, T.c0 + CH - 1, 0, nullptr);
#pragma unroll
        for (int k = CH - 1; k >= 1; --k)       // hidden layer k: input C[k-1], output C[k]
            bt_bwd<64, 64, 0>(c, T.dz, T.c0 + k - 1, L.c_hid[k - 1], dw_chid[k - 1], T.c0 + k - 1, 0, nullptr);
        {
            float gcin[32], gy[16];
            bt_bwd<32, 64, 1>(c, T.dz, T.cin, L.c_in, dw_cin, 0, T.cin, gcin);   // dL/dcin (scaled); CIN is dead after this round
            if (INPUTS && valid) {   // dL/dw from dL/dSH = gcin[15..30]; written now, so it holds no registers through the density backward
                const float3 gw = sh4_grad(dx, dy, dz, gcin + 15);
                float *o = d_rows + 6 * (size_t)i;
                o[3] = gw.x * (1.f / BT_SCALE); o[4] = gw.y * (1.f / BT_SCALE); o[5] = gw.z * (1.f / BT_SCALE);
            }
            gy[0] = gr.w * BT_SCALE;                // dL/d density_out = (draw.w, dcin[0..14])   (hashnerf_mlp.py:69-78: raw[3] = density_out[0], colour input = density_out[1:])
#pragma unroll
            for (int k = 0; k < 15; ++k) gy[k + 1] = gcin[k];
            bt_store16(c, T.dz, gy);
        }
        // ------------------------------------------------ backward: density net
        bt_bwd<64, 16, 0>(c, T.dz, T.h0 + DH - 1, L.d_out, dw_dout, T.h0 + DH - 1, 0, nullptr);
#pragma unroll
        for (int k = DH - 1; k >= 1; --k)
            bt_bwd<64, 64, 0>(c, T.dz, T.h0 + k - 1, L.d_hid[k - 1], dw_dhid[k - 1], T.h0 + k - 1, 0, nullptr);
        bt_bwd<32, 64, 1>(c, T.dz, T.enc, L.d_in, dw_din, 0, T.enc, genc);      // dL/d encoding (scaled); ENC is dead after this round
        c.first = false;
        // ------------------------------------------------ hash-table gradient scatter
        if (valid) {
            // as xrb_ngp_density_grad_tc: a row outside [-0.5, 1.5]^3 (or not finite) gets a zero position gradient without reading the table again
            const bool inside = INPUTS && fabsf(px - 0.5f) <= 1.f && fabsf(py - 0.5f) <= 1.f && fabsf(pz - 0.5f) <= 1.f;
            float3 gx = make_float3(0.f, 0.f, 0.f);
#pragma unroll 1
            for (int l = 0; l < 16; ++l) {
                float g0 = 0.f, g1 = 0.f;
#pragma unroll
                for (int q = 0; q < 16; ++q) if (q == l) { g0 = genc[2 * q]; g1 = genc[2 * q + 1]; }   // register array indexed by the rolled loop counter: select, never spill
                scatter_level_paired(d_table, grid_cell(g, l, px, py, pz), (g.hashed_mask >> l) & 1u, g0 * (1.f / BT_SCALE), g1 * (1.f / BT_SCALE));
                if (inside) position_grad_level(table, g, l, px, py, pz, g0 * (1.f / BT_SCALE), g1 * (1.f / BT_SCALE), gx);
            }
            if (INPUTS) { float *o = d_rows + 6 * (size_t)i; o[0] = gx.x; o[1] = gx.y; o[2] = gx.z; }
        }
    }
    // ---------------------------------------------------- flush the weight-gradient accumulators (once per warpgroup)
    if (!c.first) {
        float *dd = d_dens, *dc = d_color;
        bt_flush<32, false>(c, dw_din, dd, 32);
#pragma unroll
        for (int k = 1; k < DH; ++k) bt_flush<64, false>(c, dw_dhid[k - 1], dd + 64 * 32 + (k - 1) * 64 * 64, 64);
        bt_flush<16, true>(c, dw_dout, dd + 64 * 32 + (DH - 1) * 64 * 64, 64);
        bt_flush<32, false>(c, dw_cin, dc, 32);
#pragma unroll
        for (int k = 1; k < CH; ++k) bt_flush<64, false>(c, dw_chid[k - 1], dc + 64 * 32 + (k - 1) * 64 * 64, 64);
        bt_flush<16, true>(c, dw_cout, dc + 64 * 32 + (CH - 1) * 64 * 64, 64);
    }
}

template <int DH, int CH, int NP>
__global__ void __launch_bounds__(256, 1) ngp_field_bwd_tc_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const void *__restrict__ weight_image,
                                                                  uint32_t image_bytes, const float *__restrict__ pts, int pts_stride, const float *__restrict__ dirs, int dirs_stride,
                                                                  const float4 *__restrict__ dl_draw, int n, const int32_t *__restrict__ n_dev, float *__restrict__ d_table,
                                                                  float *__restrict__ d_dens, float *__restrict__ d_color) {
    ngp_field_bwd_tc<DH, CH, NP, false>(g, table, cells, weight_image, image_bytes, pts, pts_stride, dirs, dirs_stride, dl_draw, n, n_dev, d_table, d_dens, d_color, nullptr);
}
template <int DH, int CH, int NP>
__global__ void __launch_bounds__(256, 1) ngp_field_bwd_tc_inputs_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells,
                                                                         const void *__restrict__ weight_image, uint32_t image_bytes, const float *__restrict__ pts, int pts_stride,
                                                                         const float *__restrict__ dirs, int dirs_stride, const float4 *__restrict__ dl_draw, int n,
                                                                         const int32_t *__restrict__ n_dev, float *__restrict__ d_table, float *__restrict__ d_dens,
                                                                         float *__restrict__ d_color, float *__restrict__ d_rows) {
    ngp_field_bwd_tc<DH, CH, NP, true>(g, table, cells, weight_image, image_bytes, pts, pts_stride, dirs, dirs_stride, dl_draw, n, n_dev, d_table, d_dens, d_color, d_rows);
}

template <int DH, int CH, int NP, bool INPUTS>
static int launch_bwd_tc(const HashGridDev &g, const xrb_ngp_table *tab, const void *image, uint32_t image_bytes, const float *pts, int pts_stride, const float *dirs, int dirs_stride,
                         const float *dl_draw, int n, const int32_t *n_dev, float *d_table, float *d_dens, float *d_color, float *d_rows, cudaStream_t s) {
    const size_t smem = bt_smem_bytes<DH, CH>(image_bytes);
    const int n_tiles = (n + 127) / 128, grid = persistent_grid(1, (n_tiles + 1) / 2);   // one CTA per SM, two tiles (warpgroups) per CTA
    const __half2 *table = (const __half2 *)tab->table_fp16;
    const uint8_t *cells = (const uint8_t *)tab->cell_image;
    if (INPUTS) {
        auto k = ngp_field_bwd_tc_inputs_kernel<DH, CH, NP>;
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        k<<<grid, 256, smem, s>>>(g, table, cells, image, image_bytes, pts, pts_stride, dirs, dirs_stride, (const float4 *)dl_draw, n, n_dev, d_table, d_dens, d_color, d_rows);
    } else {
        auto k = ngp_field_bwd_tc_kernel<DH, CH, NP>;
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        k<<<grid, 256, smem, s>>>(g, table, cells, image, image_bytes, pts, pts_stride, dirs, dirs_stride, (const float4 *)dl_draw, n, n_dev, d_table, d_dens, d_color);
    }
    return check_launch(INPUTS ? "ngp_mlp_backward_tc_inputs" : "ngp_mlp_backward_tc");
}

// ---------------------------------------------------------------------------- density and its position gradient on tensor cores (xrb_ngp_density_grad_tc)
// The gradient stage of the chain render's normal maps. One warpgroup per CTA and 128-row tile, persistent:
//   forward   hash gather -> ENC tile; density hidden layers through bt_fwd_hidden, each activation parked as a tile (its ReLU mask is "fp16 value > 0");
//             the N=16 output layer through bt_fwd_out. Same fp16 operands, K order and roundings as the production field (tc_net), so the density is
//             bit-identical to ngp_field_tc_kernel<true, *>'s.
//   backward  only output 0 is differentiated: dZ of the last hidden layer = fp16(DG_TC_SCALE * W_out[0,:]) * [H > 0], written row by row from the resident
//             weight image; then the masked W^T rounds of bt_bwd_dx (the weight-gradient half of the training backward is not issued) down to
//             dL/d(encoding) in fp32 (EPI 1), and position_grad_level per level.
// Tiles per warpgroup: ENC, H0..H(dh-1), dZ. Only the density part of the weight image is loaded. dh is a run-time loop: tile indices and weight offsets
// are computed, nothing is indexed in registers.
__device__ __forceinline__ uint32_t h2_as_u32(__half2 h) { return *reinterpret_cast<uint32_t *>(&h); }
constexpr float DG_TC_SCALE = 1024.f;    // dZ staging scale (fp16): |d density / d hidden unit| < 64 stays finite, entries down to 2^-24 / 1024 stay exact
__global__ void __launch_bounds__(128) ngp_density_grad_tc_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells,
                                                                   const void *__restrict__ weight_image, uint32_t image_bytes, int dh, const float *__restrict__ pts,
                                                                   int pts_stride, int n, const int32_t *__restrict__ n_dev, const uint32_t *__restrict__ order,
                                                                   float *__restrict__ density, float *__restrict__ grad) {
    extern __shared__ uint8_t dyn_smem[];
    if (n_dev) n = min(n, max(*n_dev, 0));
    if (n > (int)SAMPLE_ORDER_MAX_ROWS) order = nullptr;   // as the field: beyond this the chain evaluates rows in ray order
    const int T_ENC = 0, T_H0 = 1, T_DZ = 1 + dh;
    uint8_t *W = tc_load_weight_image(dyn_smem, weight_image, image_bytes, (size_t)(dh + 2) * TILE_BLOCK_BYTES);
    BtWg c;
    c.wg = 0; c.row = threadIdx.x; c.bar = 1;
    c.tiles = W + image_bytes; c.W = W; c.first = true;
    const WeightImageLayout L = weight_image_layout(dh, 1);
    const int n_tiles = (n + 127) / 128;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int j = tile * 128 + (int)c.row;
        const bool valid = j < n;
        const int i = valid && order ? (int)__ldg(order + j) : j;   // the row this tile slot evaluates: the rows of a tile are independent
        float x = 0.5f, y = 0.5f, z = 0.5f;
        if (valid) { const float *p = pts + (size_t)i * pts_stride; x = p[0]; y = p[1]; z = p[2]; }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            uint32_t e[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) { const float2 f = hash_level(table, cells, g, 4 * q + k, x, y, z); e[k] = pack_h2(f.x, f.y); }
            bt_store_chunk(c, T_ENC, q, make_uint4(e[0], e[1], e[2], e[3]));
        }
        bt_fwd_hidden<32>(c, T_ENC, L.d_in, T_H0);
        for (int h = 1; h < dh; ++h) bt_fwd_hidden<64>(c, T_H0 + h - 1, L.d_in + 8192u * (uint32_t)h, T_H0 + h);
        const int t_last = T_H0 + dh - 1;
        {
            float dout[16];
            bt_fwd_out(c, t_last, L.d_out, T_DZ, dout);   // dZ is free until it is written below (bt_stage_rows ends with a barrier)
            if (valid && density) density[i] = round_h(dout[0]);
        }
        // dZ row r = fp16(scale * W_out[0, :]) masked by the last hidden layer's activation of row r
        const __half2 s2 = __float2half2_rn(DG_TC_SCALE), zero2 = __float2half2_rn(0.f);
#pragma unroll
        for (int ch = 0; ch < 8; ++ch) {
            const uint4 w = *reinterpret_cast<const uint4 *>(W + L.d_out + sw128_offset(0, (uint32_t)ch));
            const uint4 a = *reinterpret_cast<const uint4 *>(bt_tile(c, t_last) + sw128_offset(c.row, (uint32_t)ch));
            auto masked = [&](uint32_t wk, uint32_t ak) { return h2_as_u32(__hmul2(__hmul2(as_h2(wk), s2), __hgt2(as_h2(ak), zero2))); };
            bt_store_chunk(c, T_DZ, (uint32_t)ch, make_uint4(masked(w.x, a.x), masked(w.y, a.y), masked(w.z, a.z), masked(w.w, a.w)));
        }
        for (int k = dh - 1; k >= 1; --k) bt_bwd_dx<64, 64, 0>(c, T_DZ, L.d_in + 8192u * (uint32_t)k, T_H0 + k - 1, 0, nullptr);
        float genc[32];
        bt_bwd_dx<32, 64, 1>(c, T_DZ, L.d_in, 0, T_ENC, genc);   // d density / d encoding (scaled); ENC is dead after this round
        if (valid) {
            float3 d = make_float3(0.f, 0.f, 0.f);
            // a row no march writes (outside [-0.5, 1.5]^3, or not finite: stale rows past an overflowed ray) gets 0 without touching the table
            if (fabsf(x - 0.5f) <= 1.f && fabsf(y - 0.5f) <= 1.f && fabsf(z - 0.5f) <= 1.f) {
#pragma unroll 1
                for (int l = 0; l < 16; ++l) {
                    float g0 = 0.f, g1 = 0.f;
#pragma unroll
                    for (int q = 0; q < 16; ++q) if (q == l) { g0 = genc[2 * q]; g1 = genc[2 * q + 1]; }   // select, as the training backward's scatter: never indexed in registers
                    position_grad_level(table, g, l, x, y, z, g0 * (1.f / DG_TC_SCALE), g1 * (1.f / DG_TC_SCALE), d);
                }
            }
            float *o = grad + 3 * (size_t)i;
            o[0] = d.x; o[1] = d.y; o[2] = d.z;
        }
    }
}

// launched by xrb_ngp_density_grad_tc and by the normal-map render (ngp_render.cu); arguments validated by the caller
int launch_density_grad_tc(const xrb_ngp_config *cfg, const xrb_ngp_table *tab, const void *weight_image, const float *pts, int pts_stride, int n, const int32_t *n_dev,
                           const uint32_t *order, float *density, float *grad, cudaStream_t s) {
    HashGridDev g; int e = table_setup(cfg, tab, &g); if (e) return e;
    const int dh = cfg->density_hidden;
    const uint32_t image_bytes = weight_image_layout(dh, 1).c_in;   // the density net's matrices lead the image
    const size_t smem = 1024 + image_bytes + (size_t)(dh + 2) * TILE_BLOCK_BYTES + 16;
    cudaFuncSetAttribute(ngp_density_grad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int grid = persistent_grid((const void *)ngp_density_grad_tc_kernel, 128, smem, (n + 127) / 128);
    ngp_density_grad_tc_kernel<<<grid, 128, smem, s>>>(g, (const __half2 *)tab->table_fp16, (const uint8_t *)tab->cell_image, weight_image, image_bytes, dh, pts, pts_stride, n, n_dev,
                                                       order, density, grad);
    return check_launch("ngp_density_grad_tc");
}

}  // namespace xrb

using namespace xrb;

// both entry points of the field backward: d_rows == NULL launches the parameter-gradient kernel, otherwise its INPUTS variant (what names the errors)
static int ngp_mlp_backward_tc(const char *what, const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const float *pts, int pts_stride,
                               const float *dirs, int dirs_stride, const float *dl_draw, int n, const int32_t *n_rows_dev, float *d_table, float *d_density, float *d_color,
                               float *d_rows, void *stream) {
    static char msg[256];
    auto fail = [&](const char *m) { snprintf(msg, sizeof msg, "%s: %s", what, m); set_error(msg); return XRB_E_BADARG; };
    int e = check_cfg(cfg); if (e) return e;
    if (!(n >= 0 && pts_stride >= 3 && dirs_stride >= 3)) return fail("bad size");
    if (n == 0) return XRB_OK;
    if (!(table && weight_image && pts && dirs && dl_draw && d_table && d_density && d_color)) return fail("null pointer");
    if (!(((uintptr_t)dl_draw & 15) == 0 && ((uintptr_t)d_table & 15) == 0 && ((uintptr_t)weight_image & 15) == 0))
        return fail("dl_draw, d_table and the weight image must be 16-byte aligned");
    if (!((cfg->density_hidden == 1 && cfg->color_hidden == 1) || (cfg->density_hidden == 1 && cfg->color_hidden == 2))) {
        snprintf(msg, sizeof msg, "%s: tensor-core backward is built for (density_hidden, color_hidden) = (1,1) or (1,2); use xrb_ngp_mlp_backward", what);
        set_error(msg);
        return XRB_E_UNSUPPORTED;
    }
    HashGridDev g; e = table_setup(cfg, table, &g); if (e) return e;
    const uint32_t image_bytes = weight_image_layout(cfg->density_hidden, cfg->color_hidden).total;
    cudaStream_t s = (cudaStream_t)stream;
    const bool plan6 = plan_valid(g, table->n_packed_levels) && table->n_packed_levels == 6;
#define XRB_BWT(DH, CH, IN)                                                                                                                                      \
    if (cfg->density_hidden == DH && cfg->color_hidden == CH)                                                                                                    \
        return plan6 ? launch_bwd_tc<DH, CH, 6, IN>(g, table, weight_image, image_bytes, pts, pts_stride, dirs, dirs_stride, dl_draw, n, n_rows_dev, d_table, d_density, d_color, d_rows, s) \
                     : launch_bwd_tc<DH, CH, 0, IN>(g, table, weight_image, image_bytes, pts, pts_stride, dirs, dirs_stride, dl_draw, n, n_rows_dev, d_table, d_density, d_color, d_rows, s);
    if (d_rows) { XRB_BWT(1, 1, true) XRB_BWT(1, 2, true) }
    else { XRB_BWT(1, 1, false) XRB_BWT(1, 2, false) }
#undef XRB_BWT
    return XRB_E_UNSUPPORTED;
}

extern "C" {

int xrb_ngp_mlp_backward_tc(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const float *pts, int pts_stride, const float *dirs, int dirs_stride,
                            const float *dl_draw, int n, const int32_t *n_rows_dev, float *d_table, float *d_density, float *d_color, void *stream) {
    return ngp_mlp_backward_tc("ngp_mlp_backward_tc", cfg, table, weight_image, pts, pts_stride, dirs, dirs_stride, dl_draw, n, n_rows_dev, d_table, d_density, d_color, nullptr,
                               stream);
}

int xrb_ngp_mlp_backward_tc_inputs(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const float *pts, int pts_stride, const float *dirs,
                                   int dirs_stride, const float *dl_draw, int n, const int32_t *n_rows_dev, float *d_table, float *d_density, float *d_color, float *d_rows,
                                   void *stream) {
    if (n > 0 && !d_rows) { set_error("ngp_mlp_backward_tc_inputs: null pointer (d_rows)"); return XRB_E_BADARG; }
    return ngp_mlp_backward_tc("ngp_mlp_backward_tc_inputs", cfg, table, weight_image, pts, pts_stride, dirs, dirs_stride, dl_draw, n, n_rows_dev, d_table, d_density, d_color,
                               d_rows, stream);
}

int xrb_ngp_density_grad_tc(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const float *pts, int pts_stride, int n, const int32_t *n_rows_dev,
                            const uint32_t *order, float *density, float *grad, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && pts_stride >= 3, "ngp_density_grad_tc: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(table && weight_image && pts && grad, "ngp_density_grad_tc: null pointer");
    XRB_REQUIRE(((uintptr_t)weight_image & 15) == 0, "ngp_density_grad_tc: the weight image must be 16-byte aligned");
    return launch_density_grad_tc(cfg, table, weight_image, pts, pts_stride, n, n_rows_dev, order, density, grad, (cudaStream_t)stream);
}

}  // extern "C"
