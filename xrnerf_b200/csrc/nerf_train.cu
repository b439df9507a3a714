// xrnerf_b200 — NerfMLP training (forward with saved activations + backward) on wgmma tensor cores.
//
// The reference trains NerfMLP (/root/reference/xrnerf/models/mlps/nerf_mlp.py:70-94: 8 x 256 ReLU trunk with the skip at layer 4, alpha / feature heads, a 128-wide view
// branch) with torch.autograd over 11 nn.Linear modules: cuBLAS fp32 GEMMs forward, two more per layer backward, every [rows, 256] activation through HBM in fp32
// (networks/nerf.py:71-92, networks/mipnerf.py:45-74). Here every dense contraction of the training step is a hand-written wgmma kernel over TILE IMAGES:
//
//   tile image   an activation matrix [rows x C] stored per 128-row tile as C/64 blocks of [128 x 64] fp16 in the wgmma shared-memory layout (K-major, 128-byte swizzle,
//                16 KB per block) — the layout the encoders already write (xrb_nerf_posenc_tiles*, xrb_mip_ipe_tiles_rays). A block moves between HBM and shared memory
//                with ONE 1-D bulk TMA copy and is an MMA operand as it lies; read K-major it contracts over its 64 columns, read MN-major over its 128 rows.
//   tg_kernel    Y = epilogue( sum_p A_p . op(W_p) ) per 128-row tile, accumulators in registers (warpgroup h: rows 64h..64h+63, up to 256 columns):
//                  forward   A = layer input blocks, W slabs [N x 64] K-major, epilogue +bias, ReLU, fp16 -> output blocks (saved: they are the backward's operands)
//                  input grad dX = dZ . W : A = dZ blocks, the SAME weight slabs read MN-major (no transposed copy), epilogue * [activation > 0] -> dZ of the layer below
//   tg_dw_kernel dW += dZ^T . X over all rows: both operands read MN-major (contraction over the 128 rows of a tile), M = 128 output features per CTA (one 64-row
//                half per warpgroup), accumulators stay in registers across the CTA's whole tile range; the bias gradient (column sums of dZ) is summed on the
//                CUDA cores from the same staged dZ block while the MMAs run. One flush per CTA (fp32 atomics).
// Warp roles: warps 0-7 two consumer warpgroups (issue the MMAs of their rows, run the epilogue), warp 8 TMA producer (one lane); in tg_kernel the producer's
// warpgroup (warps 8-11) hands its registers to the consumers (setmaxnreg 40 / 232).
// dZ is staged in fp16 with a per-batch power-of-two scale s, chosen on the device from max |dL/draw| so that the head's largest staged value is in [2^12, 2^13)
// (tg_draw_max_kernel + tg_pack_draw_kernel), and removed exactly at the dW flush: the NeRF loss gives dL/draw of 1e-8 .. 1e-5, and with a fixed scale most of the
// trunk's dZ fell below fp16's normal range. No host synchronisation; the head cannot overflow, and dZ shrinks on its way down the trunk.
#include "tc.cuh"
#include "common.cuh"
#include <cuda_fp16.h>
#include <stdio.h>

namespace xrb {

constexpr int TG_MAX_A = 6, TG_MAX_SLABS = 10, TG_THREADS = 384, TG_DW_THREADS = 288;   // 6 A blocks: Mip-NeRF's skip layer reads 2 IPE blocks + 4 hidden blocks
constexpr uint32_t TG_RING_SLOT = 32768;   // one [256 x 64] fp16 slab
constexpr float TG_SCALE = 16384.f;      // the scale when dL/draw is all zero or not finite
constexpr int TG_HEAD_EXP = 12;          // max |dL/draw| s is in [2^TG_HEAD_EXP, 2^(TG_HEAD_EXP + 1))

struct TgOp { const uint8_t *base; uint32_t tile_stride, blk_off; int n_blk; };   // blocks [blk_off/16K, +n_blk) of every tile of an image
struct TgSlab { uint32_t w_off, bytes; int n_sub, a_blk0, d_col, first, n_k; };    // one weight slab: loaded once per tile, used by n_sub MMA groups (A block a_blk0 + j) of n_k K-steps of 16
struct TgP {
    TgOp a[2]; int n_a;                    // A operand sources, concatenated block-wise into the shared-memory A buffer
    const uint8_t *w;                      // weight image base
    TgSlab slab[TG_MAX_SLABS]; int n_slabs;
    int b_mn;                              // 0: slabs are K-major B operands (forward), 1: MN-major (input gradient)
    int mma_n;                             // N of each MMA (forward: layer width 16/128/256; input gradient: 64)
    int out_cols;                          // accumulator columns the epilogue reads (multiple of 16, <= 256)
    int epi;                               // 0: +bias, relu?, fp16 -> y image; 1: +bias -> fp32 rows (yf); 2: * [x > 0] -> fp16 y image; 3: plain fp16 -> y image
    int relu; const float *bias;
    TgOp x;                                // epi 2: the activation whose sign masks the gradient (out_cols/64 blocks per tile)
    uint8_t *y; uint32_t y_tile_stride, y_blk_off;
    float *yf; int yf_stride, yf_col, yf_n; float yf_scale;
    long long n_rows;
};

enum { TB_AFULL = 0, TB_AEMPTY = 1, TB_SFULL = 2, TB_SEMPTY = 4, TB_XFULL = 6, TB_YEMPTY = 7, TB_N = 8 };

// acc[mma_n / 2 registers at column d_col] (+)= A . B for the run-time (mma_n, d_col) pairs the host produces: forward N = 16 | 128 | 256 at column 0,
// input gradient N = 64 at column 0 | 64 | 128 | 192 (register arrays need compile-time offsets)
template <int TB>
__device__ __forceinline__ void tg_mma(float *acc, int mma_n, int d_col, uint64_t ad, uint64_t bd, uint32_t sc) {
    if (mma_n == 256) tc::wgmma<256, 0, TB>(acc, ad, bd, sc);
    else if (mma_n == 128) tc::wgmma<128, 0, TB>(acc, ad, bd, sc);
    else if (mma_n == 16) tc::wgmma<16, 0, TB>(acc, ad, bd, sc);
    else if (d_col == 0) tc::wgmma<64, 0, TB>(acc, ad, bd, sc);
    else if (d_col == 64) tc::wgmma<64, 0, TB>(acc + 32, ad, bd, sc);
    else if (d_col == 128) tc::wgmma<64, 0, TB>(acc + 64, ad, bd, sc);
    else tc::wgmma<64, 0, TB>(acc + 96, ad, bd, sc);
}

__global__ void __launch_bounds__(TG_THREADS, 1) tg_kernel(const __grid_constant__ TgP P) {
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *base = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    uint8_t *A = base, *RING = A + TG_MAX_A * TILE_BLOCK_BYTES, *Y = RING + 2 * TG_RING_SLOT;
    uint64_t *bars = (uint64_t *)(Y + 4 * TILE_BLOCK_BYTES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int k = 0; k < TB_N; ++k) tc::mbar_init(bars + k, 1);
        tc::mbar_init(bars + TB_AEMPTY, 8); tc::mbar_init(bars + TB_SEMPTY, 8); tc::mbar_init(bars + TB_SEMPTY + 1, 8);   // one arrival per consumer warp
        tc::mbar_init(bars + TB_YEMPTY, 2);                                                                             // one per consumer warpgroup
        tc::fence_mbar_init();
    }
    __syncthreads();
    const long long n_tiles = (P.n_rows + 127) / 128;
    int n_ablk = 0;
    for (int s = 0; s < P.n_a; ++s) n_ablk += P.a[s].n_blk;
    const int n_xblk = P.epi == 2 ? P.out_cols / 64 : 0;

    if (warp >= 8) {
        // ===================================================== producer (one lane): A blocks of the tile, then its weight slabs through the 2-slot ring, then the mask blocks
        tc::setmaxnreg_dec<40>();   // registers go to the consumer warpgroups
        if (warp == 8 && lane == 0) {
            uint32_t it = 0, g = 0;
            for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
                if (it > 0) tc::mbar_wait(bars + TB_AEMPTY, (it - 1) & 1);
                tc::mbar_expect_tx(bars + TB_AFULL, (uint32_t)n_ablk * TILE_BLOCK_BYTES);
                int ab = 0;
                for (int s = 0; s < P.n_a; ++s)
                    for (int k = 0; k < P.a[s].n_blk; ++k, ++ab)
                        tc::tma_bulk_g2s(A + (size_t)ab * TILE_BLOCK_BYTES, P.a[s].base + (size_t)tile * P.a[s].tile_stride + P.a[s].blk_off + (size_t)k * TILE_BLOCK_BYTES, TILE_BLOCK_BYTES, bars + TB_AFULL);
                for (int s = 0; s < P.n_slabs; ++s, ++g) {
                    const uint32_t slot = g & 1u, round = g >> 1;
                    if (round > 0) tc::mbar_wait(bars + TB_SEMPTY + slot, (round - 1) & 1);
                    tc::mbar_expect_tx(bars + TB_SFULL + slot, P.slab[s].bytes);
                    tc::tma_bulk_g2s(RING + (size_t)slot * TG_RING_SLOT, P.w + P.slab[s].w_off, P.slab[s].bytes, bars + TB_SFULL + slot);
                }
                if (n_xblk) {
                    if (it > 0) tc::mbar_wait(bars + TB_YEMPTY, (it - 1) & 1);     // the previous tile's output has left the Y region
                    tc::mbar_expect_tx(bars + TB_XFULL, (uint32_t)n_xblk * TILE_BLOCK_BYTES);
                    for (int k = 0; k < n_xblk; ++k)
                        tc::tma_bulk_g2s(Y + (size_t)k * TILE_BLOCK_BYTES, P.x.base + (size_t)tile * P.x.tile_stride + P.x.blk_off + (size_t)k * TILE_BLOCK_BYTES, TILE_BLOCK_BYTES, bars + TB_XFULL);
                }
            }
        }
    } else {
        // ===================================================== two consumer warpgroups: warpgroup h issues the MMAs of rows 64h..64h+63 and runs their epilogue
        tc::setmaxnreg_inc<232>();
        const int wg = warp >> 2, t = threadIdx.x & 127;
        const uint32_t r0 = 64u * (uint32_t)wg + tc::frag_row((uint32_t)t);   // my fragment rows: r0, r0 + 8
        uint32_t it = 0, g = 0;
        float acc[128];
        for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
            tc::mbar_wait(bars + TB_AFULL, it & 1);
            for (int s = 0; s < P.n_slabs; ++s, ++g) {
                const uint32_t slot = g & 1u, round = g >> 1;
                tc::mbar_wait(bars + TB_SFULL + slot, round & 1);
                const TgSlab &S = P.slab[s];
                const uint32_t b_base = tc::smem_u32(RING + (size_t)slot * TG_RING_SLOT);
                tc::wg_fence();
                for (int j = 0; j < S.n_sub; ++j) {
                    const uint32_t a0 = tc::smem_u32(A + (size_t)(S.a_blk0 + j) * TILE_BLOCK_BYTES) + (uint32_t)wg * 8192u;
                    for (int k = 0; k < S.n_k; ++k) {
                        const uint64_t ad = tc::desc_k128(a0 + k * 32);
                        const uint32_t sc = (S.first && j == 0 && k == 0) ? 0u : 1u;
                        if (P.b_mn) tg_mma<1>(acc, P.mma_n, S.d_col, ad, tc::desc_mn128(b_base + j * 8192 + k * 2048, 1024), sc);
                        else tg_mma<0>(acc, P.mma_n, S.d_col, ad, tc::desc_k128(b_base + k * 32), sc);
                    }
                }
                tc::wg_commit();
                tc::wg_wait<0>();
                tc::acc_fence<128>(acc);
                __syncwarp();
                if (lane == 0) tc::mbar_arrive(bars + TB_SEMPTY + slot);   // this warp's share of the MMAs reading the slot is complete
            }
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(bars + TB_AEMPTY);
            // ---- epilogue straight from the accumulator fragments
            if (P.epi == 2) tc::mbar_wait(bars + TB_XFULL, it & 1);
            else tc::named_bar_sync(1 + wg, 128);                   // the previous tile's bulk store has finished reading my half of Y (its issuer waited)
            if (P.epi == 1) {
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int col = (int)tc::frag_col((uint32_t)t, j) + (i & 1);
                        const long long row = tile * 128 + r0 + 8 * (i >> 1);
                        if (col < P.yf_n && row < P.n_rows) P.yf[(size_t)row * P.yf_stride + P.yf_col + col] = (acc[4 * j + i] + (P.bias ? __ldg(P.bias + col) : 0.f)) * P.yf_scale;
                    }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const uint32_t col = tc::frag_col((uint32_t)t, j);
                    if ((int)col >= P.out_cols) break;
                    float v[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};
                    if (P.epi == 0) {
                        const float b0 = P.bias ? __ldg(P.bias + col) : 0.f, b1 = P.bias ? __ldg(P.bias + col + 1) : 0.f;
                        v[0] += b0; v[1] += b1; v[2] += b0; v[3] += b1;
                        if (P.relu) { v[0] = fmaxf(v[0], 0.f); v[1] = fmaxf(v[1], 0.f); v[2] = fmaxf(v[2], 0.f); v[3] = fmaxf(v[3], 0.f); }
                    }
                    uint8_t *yb = Y + (size_t)(col >> 6) * TILE_BLOCK_BYTES;
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        uint32_t *w = reinterpret_cast<uint32_t *>(sw128_elem(yb, r0 + 8u * (uint32_t)e, col & 63u));
                        __half2 h = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
                        if (P.epi == 2) h = __hmul2(h, __hgt2(*reinterpret_cast<const __half2 *>(w), __float2half2_rn(0.f)));   // * [x > 0]
                        *w = *reinterpret_cast<uint32_t *>(&h);
                    }
                }
                // my rows of Y are complete: one thread of the warpgroup stores them (rows 64h.. of every block are its second / first 8 KB)
                tc::fence_proxy_async_smem();
                tc::named_bar_sync(1 + wg, 128);
                if (t == 0) {
                    const int n_out_blk = (P.out_cols + 63) / 64;
                    for (int k = 0; k < n_out_blk; ++k)
                        tc::tma_bulk_s2g(P.y + (size_t)tile * P.y_tile_stride + P.y_blk_off + (size_t)k * TILE_BLOCK_BYTES + (size_t)wg * 8192, Y + (size_t)k * TILE_BLOCK_BYTES + (size_t)wg * 8192, 8192);
                    tc::tma_bulk_commit_wait_read();
                    if (P.epi == 2) tc::mbar_arrive(bars + TB_YEMPTY);
                }
            }
        }
        if (t == 0) tc::tma_bulk_wait_all();
    }
}

// ---------------------------------------------------------------------------------------------------- weight gradient
struct TgDwP {
    TgOp z;                 // dZ image of the layer: N/64 blocks per tile (one block for the 16-output layers)
    TgOp x;                 // one source of the layer input: 1..4 blocks per tile
    int n_chunks;           // normal: N / 128 chunks of output rows; transposed: chunks of 128 input columns
    int transposed;         // 0: D[m = out (128 per chunk), n = in]; 1 (N <= 16 layers): D[m = in (128 per chunk), n = out (16)]
    int N, K;               // true layer shape (dW[N][K], fp32 parameter)
    int k_off, k_cols;      // this source's columns [k_off, k_off + k_cols) of the layer input
    float *dW; float *db;   // fp32 gradients (accumulated); db == NULL: no bias gradient from this launch
    long long n_rows;
    const float *scale;     // the dZ staging scale (device, written by tg_pack_draw_kernel); NULL: TG_SCALE
};

// Warps 0-7: two consumer warpgroups, warpgroup h owns accumulator rows 64h..64h+63 of the CTA's 128-row chunk (registers, across the CTA's whole
// tile range); warp 8: producer (one lane). One flush per CTA (fp32 atomics).
__global__ void __launch_bounds__(TG_DW_THREADS, 1) tg_dw_kernel(const __grid_constant__ TgDwP P) {
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *base = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    // two stages of (dZ chunk: 2 blocks | X: 4 blocks)
    constexpr uint32_t STAGE = 6 * TILE_BLOCK_BYTES;
    uint64_t *bars = (uint64_t *)(base + 2 * STAGE);      // full[2], empty[2]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { tc::mbar_init(bars, 1); tc::mbar_init(bars + 1, 1); tc::mbar_init(bars + 2, 8); tc::mbar_init(bars + 3, 8); tc::fence_mbar_init(); }
    __syncthreads();
    const long long n_tiles = (P.n_rows + 127) / 128;
    const int chunk = blockIdx.x % P.n_chunks, cta = blockIdx.x / P.n_chunks, n_cta = gridDim.x / P.n_chunks;
    const int n_xblk = P.x.n_blk;
    const int z_blk = P.transposed ? 1 : 2;                                   // blocks of dZ per stage
    if (warp == 8) {
        if (lane == 0) {
            uint32_t it = 0;
            for (long long tile = cta; tile < n_tiles; tile += n_cta, ++it) {
                const uint32_t st = it & 1u;
                if (it >= 2) tc::mbar_wait(bars + 2 + st, ((it >> 1) - 1) & 1);
                uint8_t *S = base + (size_t)st * STAGE;
                tc::mbar_expect_tx(bars + st, (uint32_t)(z_blk + n_xblk) * TILE_BLOCK_BYTES);
                const uint32_t z_first = P.transposed ? 0u : (uint32_t)chunk * 2u;
                for (int k = 0; k < z_blk; ++k)
                    tc::tma_bulk_g2s(S + (size_t)k * TILE_BLOCK_BYTES, P.z.base + (size_t)tile * P.z.tile_stride + P.z.blk_off + (size_t)(z_first + k) * TILE_BLOCK_BYTES, TILE_BLOCK_BYTES, bars + st);
                for (int k = 0; k < n_xblk; ++k)
                    tc::tma_bulk_g2s(S + (size_t)(2 + k) * TILE_BLOCK_BYTES, P.x.base + (size_t)tile * P.x.tile_stride + P.x.blk_off + (size_t)k * TILE_BLOCK_BYTES, TILE_BLOCK_BYTES, bars + st);
            }
        }
        return;
    }
    if (cta >= n_tiles) return;
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const bool bias_here = P.db && (!P.transposed || (chunk == 0 && wg == 0));
    // bias gradient = column sums of dZ, on the CUDA cores from the staged dZ block: transposed (<= 16 outputs): column t % 16, rows 16 (t / 16) ..;
    // otherwise: column t % 64 of dZ block wg (output 64 wg + t % 64 of the chunk), rows 64 (t / 64) ..
    const uint32_t b_col = P.transposed ? (uint32_t)t & 15u : (uint32_t)t & 63u, b_rows = P.transposed ? 16u : 64u, b_row0 = ((uint32_t)t / (P.transposed ? 16u : 64u)) * b_rows;
    float acc[4][32], bsum = 0.f;
    uint32_t it = 0;
    for (long long tile = cta; tile < n_tiles; tile += n_cta, ++it) {
        const uint32_t st = it & 1u;
        tc::mbar_wait(bars + st, (it >> 1) & 1);
        const uint32_t S = tc::smem_u32(base + (size_t)st * STAGE);
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) {   // 16 sample rows (2 x 1024 bytes) per instruction
            const uint32_t sc = (it | (uint32_t)k) ? 1u : 0u;
            if (!P.transposed) {
                // D[64 out (dZ block 2 chunk + h) x 64 in per X block] += dZ^T . X
                const uint64_t ad = tc::desc_mn128(S + (uint32_t)wg * TILE_BLOCK_BYTES + k * 2048, 1024);
#pragma unroll
                for (int xb = 0; xb < 4; ++xb)
                    if (xb < n_xblk) tc::wgmma<64, 1, 1>(acc[xb], ad, tc::desc_mn128(S + (2 + xb) * TILE_BLOCK_BYTES + k * 2048, 1024), sc);
            } else {
                // D[64 in (X block 2 chunk + h) x 16 out] += X^T . dZ
                tc::wgmma<16, 1, 1>(acc[0], tc::desc_mn128(S + (2 + 2 * chunk + wg) * TILE_BLOCK_BYTES + k * 2048, 1024), tc::desc_mn128(S + k * 2048, 1024), sc);
            }
        }
        tc::wg_commit();
        if (bias_here) {
            const uint8_t *zb = base + (size_t)st * STAGE + (P.transposed ? 0 : (size_t)wg * TILE_BLOCK_BYTES);
            for (uint32_t r = b_row0; r < b_row0 + b_rows; ++r) bsum += __half2float(*reinterpret_cast<const __half *>(sw128_elem(zb, r, b_col)));
        }
        tc::wg_wait<0>();
        tc::acc_fence<32>(acc[0]); tc::acc_fence<32>(acc[1]); tc::acc_fence<32>(acc[2]); tc::acc_fence<32>(acc[3]);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(bars + 2 + st);
    }
    // ---- flush from the fragments: register 4j + i holds row m0 + 8 (i / 2), column 8j + 2 (t % 4) + i % 2
    const float inv = 1.f / (P.scale ? *P.scale : TG_SCALE);   // a power of two: exact
    const int m0 = 64 * wg + (int)tc::frag_row((uint32_t)t);
    if (!P.transposed) {
#pragma unroll
        for (int xb = 0; xb < 4; ++xb) {
            if (xb >= n_xblk) break;
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int out = chunk * 128 + m0 + 8 * (i >> 1), kc = xb * 64 + (int)tc::frag_col((uint32_t)t, j) + (i & 1);
                    if (out < P.N && kc < P.k_cols) atomicAdd(P.dW + (size_t)out * P.K + P.k_off + kc, acc[xb][4 * j + i] * inv);
                }
        }
        if (bias_here) { const int out = chunk * 128 + 64 * wg + (int)b_col; if (out < P.N) atomicAdd(P.db + out, bsum * inv); }
    } else {
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int kin = chunk * 128 + m0 + 8 * (i >> 1), n = (int)tc::frag_col((uint32_t)t, j) + (i & 1);
                if (kin < P.k_cols && n < P.N) atomicAdd(P.dW + (size_t)n * P.K + P.k_off + kin, acc[0][4 * j + i] * inv);
            }
        if (bias_here && (int)b_col < P.N) atomicAdd(P.db + b_col, bsum * inv);
    }
}

// ---------------------------------------------------------------------------------------------------- small helpers
// nn.Linear weight W[N][K_in] (fp32, row-major) -> slabs: for every 64-column input block kb (columns map[kb] .. +64 of the layer input, zero beyond `valid`): [n_pad x 64] fp16 SW128 K-major
struct TgPackP { const float *W; int N, K_in, n_pad; int n_kb; int col0[TG_MAX_A]; int valid[TG_MAX_A]; uint8_t *out; };
__global__ void tg_pack_weights_kernel(const __grid_constant__ TgPackP P) {
    const int kb = blockIdx.x;
    uint8_t *slab = P.out + (size_t)kb * P.n_pad * 128;
    for (int t = threadIdx.x; t < P.n_pad * 8; t += blockDim.x) pack_slab_chunk(slab, P.W, P.K_in, P.N, P.col0[kb], P.valid[kb], t >> 3, t & 7);
}
// max |dL/draw| over the batch -> scale[0] (its fp32 bits: for non-negative floats the unsigned order is the numeric order; NaN sorts above +inf)
__global__ void __launch_bounds__(256) tg_draw_max_kernel(const float *__restrict__ d_raw, long long n, float *scale) {
    uint32_t m = 0;
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) m = max(m, __float_as_uint(fabsf(d_raw[i])));
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int *>(scale), m);
}
// the power of two s with max |dL/draw| s in [2^12, 2^13) (TG_SCALE when the maximum is 0 or not finite), kept within fp32's normal range
__device__ __forceinline__ float tg_scale_of(uint32_t max_bits) {
    const float m = __uint_as_float(max_bits);
    if (!(m > 0.f) || !isfinite(m)) return TG_SCALE;
    return exp2f((float)min(max(TG_HEAD_EXP - ilogbf(m), -120), 120));
}
// dL/draw fp32 [rows,4] -> two one-block tile images (fp16 of dL/draw * s): d_rgb in columns 0..2, d_alpha in column 0, every other entry and the rows beyond
// n_rows zero; s (from the maximum in scale[0]) -> scale[1] for the dW flushes
__global__ void __launch_bounds__(128) tg_pack_draw_kernel(const float4 *__restrict__ d_raw, long long n_rows, uint8_t *__restrict__ z_rgb, uint8_t *__restrict__ z_alpha,
                                                           float *scale) {
    const long long tile = blockIdx.x, i = tile * 128 + threadIdx.x;
    const float s = tg_scale_of(__float_as_uint(scale[0]));
    if (tile == 0 && threadIdx.x == 0) scale[1] = s;
    const float4 g = i < n_rows ? d_raw[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const int row = threadIdx.x;
    uint8_t *br = z_rgb + (size_t)tile * TILE_BLOCK_BYTES, *ba = z_alpha + (size_t)tile * TILE_BLOCK_BYTES;
    const uint4 z = make_uint4(0, 0, 0, 0);
    st_chunk(br + sw128_offset(row, 0), make_uint4(pack_h2(g.x * s, g.y * s), pack_h2(g.z * s, 0.f), 0u, 0u));
    st_chunk(ba + sw128_offset(row, 0), make_uint4(pack_h2(g.w * s, 0.f), 0u, 0u, 0u));
#pragma unroll
    for (uint32_t c = 1; c < 8; ++c) { st_chunk(br + sw128_offset(row, c), z); st_chunk(ba + sw128_offset(row, c), z); }
}

static size_t tg_smem() { return 1024 + (size_t)TG_MAX_A * TILE_BLOCK_BYTES + 2 * TG_RING_SLOT + 4 * TILE_BLOCK_BYTES + 8 * TB_N + 64; }
static size_t tg_dw_smem() { return 1024 + 2 * 6 * (size_t)TILE_BLOCK_BYTES + 8 * 4 + 64; }

}  // namespace xrb

using namespace xrb;

extern "C" {

// One dense layer of the NerfMLP training forward / input-gradient pass over tile images. See include/xrnerf_b200.h.
int xrb_nerf_tg_layer(const xrb_tg_layer *L, void *stream) {
    XRB_REQUIRE(L, "tg_layer: null descriptor");
    XRB_REQUIRE(L->n_rows >= 0 && L->n_a >= 1 && L->n_a <= 2 && L->n_slabs >= 1 && L->n_slabs <= TG_MAX_SLABS, "tg_layer: bad sizes");
    if (L->n_rows == 0) return XRB_OK;
    XRB_REQUIRE(L->w && L->a_base[0], "tg_layer: null pointer");
    XRB_REQUIRE(L->epi >= 0 && L->epi <= 3 && L->out_cols >= 16 && L->out_cols <= 256 && (L->out_cols % 16) == 0, "tg_layer: bad epilogue");
    XRB_REQUIRE(L->mma_n == 16 || L->mma_n == 64 || L->mma_n == 128 || L->mma_n == 256, "tg_layer: MMA N must be 16, 64, 128 or 256");
    TgP P{};
    int n_ablk = 0;
    for (int s = 0; s < L->n_a; ++s) {
        P.a[s] = TgOp{(const uint8_t *)L->a_base[s], L->a_tile_stride[s], L->a_blk_off[s], L->a_n_blk[s]};
        XRB_REQUIRE(((uintptr_t)L->a_base[s] & 127) == 0 && L->a_n_blk[s] >= 1, "tg_layer: A image must be 128-byte aligned");
        n_ablk += L->a_n_blk[s];
    }
    XRB_REQUIRE(n_ablk <= TG_MAX_A, "tg_layer: at most 6 input blocks per tile");
    P.n_a = L->n_a; P.w = (const uint8_t *)L->w; P.n_slabs = L->n_slabs;
    for (int s = 0; s < L->n_slabs; ++s) {
        P.slab[s] = TgSlab{L->slab_w_off[s], L->slab_bytes[s], L->slab_n_sub[s], L->slab_a_blk0[s], L->slab_d_col[s], L->slab_first[s], L->slab_n_k[s]};
        XRB_REQUIRE(L->slab_n_k[s] >= 1 && L->slab_n_k[s] <= 4 && L->slab_n_sub[s] >= 1, "tg_layer: slab K-steps");
        XRB_REQUIRE(L->slab_bytes[s] <= TG_RING_SLOT && (L->slab_bytes[s] % 1024) == 0 && (L->slab_w_off[s] % 128) == 0, "tg_layer: slab size/offset");
        XRB_REQUIRE(L->slab_a_blk0[s] + L->slab_n_sub[s] <= n_ablk && L->slab_d_col[s] + L->mma_n <= 256, "tg_layer: slab refers outside the tile");
        // every MMA reads inside the slab's bytes: K-major, mma_n rows of 128 bytes; MN-major, group j K-step k reads the 2 KB at (4 j + k) * 2048
        XRB_REQUIRE(L->b_mn ? ((uint32_t)((L->slab_n_sub[s] - 1) * 4 + L->slab_n_k[s]) * 2048u <= L->slab_bytes[s]) : ((uint32_t)L->mma_n * 128u <= L->slab_bytes[s]),
                    "tg_layer: MMA reads past the slab");
        XRB_REQUIRE(L->mma_n == 64 ? (L->slab_d_col[s] >= 0 && L->slab_d_col[s] % 64 == 0) : L->slab_d_col[s] == 0,
                    "tg_layer: implemented MMA shapes are N = 16 / 128 / 256 at accumulator column 0 and N = 64 at columns 0 / 64 / 128 / 192");
    }
    P.b_mn = L->b_mn; P.mma_n = L->mma_n; P.out_cols = L->out_cols; P.epi = L->epi; P.relu = L->relu; P.bias = L->bias;
    P.x = TgOp{(const uint8_t *)L->x_base, L->x_tile_stride, L->x_blk_off, L->out_cols / 64};
    P.y = (uint8_t *)L->y; P.y_tile_stride = L->y_tile_stride; P.y_blk_off = L->y_blk_off;
    P.yf = L->yf; P.yf_stride = L->yf_stride; P.yf_col = L->yf_col; P.yf_n = L->yf_n; P.yf_scale = L->yf_scale; P.n_rows = L->n_rows;
    XRB_REQUIRE(L->epi == 1 ? (L->yf != nullptr && L->yf_n >= 1 && L->yf_n <= 16) : (L->y != nullptr && (L->out_cols % 64) == 0), "tg_layer: output");
    XRB_REQUIRE(L->epi != 2 || L->x_base != nullptr, "tg_layer: mask image missing");
    const size_t smem = tg_smem();
    cudaFuncSetAttribute(tg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int grid = persistent_grid(1, (L->n_rows + 127) / 128);
    tg_kernel<<<grid, TG_THREADS, smem, (cudaStream_t)stream>>>(P);
    return check_launch("nerf_tg_layer");
}

int xrb_nerf_tg_dw(const xrb_tg_dw *L, void *stream) {
    XRB_REQUIRE(L, "tg_dw: null descriptor");
    XRB_REQUIRE(L->n_rows >= 0 && L->N >= 1 && L->K >= 1 && L->x_n_blk >= 1 && L->x_n_blk <= 4 && L->k_off >= 0 && L->k_cols >= 1 && L->k_off + L->k_cols <= L->K, "tg_dw: bad sizes");
    XRB_REQUIRE(L->k_cols <= 64 * L->x_n_blk, "tg_dw: k_cols wider than the input blocks");
    if (L->n_rows == 0) return XRB_OK;
    XRB_REQUIRE(L->z_base && L->x_base && L->dW, "tg_dw: null pointer");
    TgDwP P{};
    P.z = TgOp{(const uint8_t *)L->z_base, L->z_tile_stride, L->z_blk_off, 0};
    P.x = TgOp{(const uint8_t *)L->x_base, L->x_tile_stride, L->x_blk_off, L->x_n_blk};
    P.N = L->N; P.K = L->K; P.k_off = L->k_off; P.k_cols = L->k_cols; P.dW = L->dW; P.db = L->db; P.n_rows = L->n_rows; P.scale = L->scale;
    P.transposed = L->N <= 16;
    if (P.transposed) { XRB_REQUIRE((L->x_n_blk % 2) == 0, "tg_dw: 16-output layers take an input image of 128 or 256 columns"); P.n_chunks = L->x_n_blk / 2; }
    else { XRB_REQUIRE(L->N == 128 || L->N == 256, "tg_dw: N must be 128 or 256 (or <= 16)"); P.n_chunks = L->N / 128; }
    const size_t smem = tg_dw_smem();
    cudaFuncSetAttribute(tg_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    long long n_tiles = (L->n_rows + 127) / 128;
    int per = sm_count() / P.n_chunks; if (per > n_tiles) per = (int)n_tiles; if (per < 1) per = 1;
    tg_dw_kernel<<<per * P.n_chunks, TG_DW_THREADS, smem, (cudaStream_t)stream>>>(P);
    return check_launch("nerf_tg_dw");
}

int xrb_nerf_tg_pack_weights(const float *W, int N, int K_in, int n_pad, int n_kb, const int *col0_host, const int *valid_host, void *slabs, void *stream) {
    XRB_REQUIRE(W && slabs && col0_host && valid_host && N >= 1 && n_pad >= N && (n_pad % 8) == 0 && n_kb >= 1 && n_kb <= TG_MAX_A, "tg_pack_weights: bad arguments");
    XRB_REQUIRE(((uintptr_t)slabs & 127) == 0, "tg_pack_weights: slabs must be 128-byte aligned");
    TgPackP P{}; P.W = W; P.N = N; P.K_in = K_in; P.n_pad = n_pad; P.n_kb = n_kb; P.out = (uint8_t *)slabs;
    for (int k = 0; k < n_kb; ++k) { P.col0[k] = col0_host[k]; P.valid[k] = valid_host[k]; XRB_REQUIRE(col0_host[k] >= 0 && valid_host[k] >= 0 && valid_host[k] <= 64 && col0_host[k] + valid_host[k] <= K_in, "tg_pack_weights: block outside the matrix"); }
    tg_pack_weights_kernel<<<n_kb, 256, 0, (cudaStream_t)stream>>>(P);
    return check_launch("nerf_tg_pack_weights");
}

int xrb_nerf_tg_pack_draw(const float *d_raw, int64_t n_rows, void *z_rgb_image, void *z_alpha_image, float *scale, void *stream) {
    XRB_REQUIRE(n_rows >= 0, "tg_pack_draw: negative size");
    if (n_rows == 0) return XRB_OK;
    XRB_REQUIRE(d_raw && z_rgb_image && z_alpha_image && scale && ((uintptr_t)d_raw & 15) == 0 && ((uintptr_t)scale & 3) == 0, "tg_pack_draw: null / misaligned pointer");
    cudaMemsetAsync(scale, 0, sizeof(float), (cudaStream_t)stream);
    tg_draw_max_kernel<<<stride_grid((4 * n_rows + 255) / 256, 4), 256, 0, (cudaStream_t)stream>>>(d_raw, 4 * n_rows, scale);
    tg_pack_draw_kernel<<<(unsigned)((n_rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>((const float4 *)d_raw, n_rows, (uint8_t *)z_rgb_image, (uint8_t *)z_alpha_image, scale);
    return check_launch("nerf_tg_pack_draw");
}

float xrb_nerf_tg_grad_scale(void) { return TG_SCALE; }

}  // extern "C"
