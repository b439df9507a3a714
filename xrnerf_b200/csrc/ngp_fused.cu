// xrnerf_b200 — the Instant-NGP inference render of a ray batch in ONE kernel launch:
//   occupancy-grid march -> multiresolution hash encoding -> density / colour MLPs (wgmma tiles) -> alpha compositing
// (replaces ngp_grid_sampler.py:205-228 + hashnerf_mlp.py:55-79 + hashnerf_render.py:42-46 + the 4096-ray chunk loop of
// hashnerf.py:54-93; no sample ever touches HBM: no coords[S,7], no raw[S,4]).
//
// One persistent CTA per SM, warp-specialised (768 threads):
//   warps 0..7   two "field" warpgroups: they own the tensor core. Thread r == row r of a 128-row tile. Per tile a
//                warpgroup copies the encoded rows out of a tile slot into its swizzled A tile, runs the 5 (=1+1 / 1+2+1 hidden) layers
//                with wgmma (weights resident in shared memory, accumulators in registers) and posts (rgb, sigma) of every row to the
//                mailbox of the producer warp that submitted it. Tiles alternate between the two warpgroups.
//   warps 8..23  "producer" warps, each autonomous over groups of 32 rays taken from a global counter:
//                  march   : lane i marches ray i (the march() of xrb_rm_rays_sampler, so bit-identical sample positions), in
//                            rounds of <= 64 samples per ray; the sample parameters t go to a per-warp scratch (L1/L2 resident)
//                  encode  : the round's samples are laid out in ray order (warp prefix sum); 32 at a time, lane = sample: a quarter
//                            of a tile slot is claimed (ticket from a shared counter) and the 16 hash levels are gathered (8 loads in
//                            flight per lane per level) straight into the slot row as fp16 pairs
//                  fold    : (rgb, sigma) of the PREVIOUS chunk come back through the mailbox (its MLP ran during this gather); a
//                            segmented warp scan composites them and lane i accumulates ray i's transmittance / colour in registers
//                            (DEPTH: alpha * t as a fourth scanned channel, so lane i also accumulates ray i's depth)
//                finally lane i writes rgb/alpha (and depth) of ray i.
// Tiles are ELASTIC: when a field warpgroup is idle it closes the current tile with however many 32-row chunks (1..4) have
// been ticketed (the missing quarters are skipped), so a chunk never waits for other producers. A producer never waits for a
// result while it owes an arrival, and arrivals never wait for results: nothing can deadlock.
// The level loop is ROLLED on purpose: 16 producer warps at 16 different places of a 16x unrolled body (~130 KB of SASS) thrash
// the instruction cache (ncu r01c: 55 % of the producers' stall samples were "no instruction").
#include "tc_field.cuh"
#include <stdio.h>
#include <stdlib.h>

namespace xrb {

constexpr uint32_t FR_ROW_BYTES = 80;                    // tile-slot row: 64 B = 32 fp16 features, 16 B = warped direction (3 floats) + pad
constexpr uint32_t FR_SLOT_BYTES = 128 * FR_ROW_BYTES;   // 80-byte row stride is bank-conflict-free for 16-byte accesses
constexpr uint32_t FR_TCAP = 64;                         // samples per ray per march round
constexpr int FR_N_WG = 2;                               // field warpgroups per CTA
constexpr int FR_N_PROD = 16;                            // producer warps per CTA (one 768-thread CTA per SM)
constexpr int FR_N_SLOTS = 5;                            // tile slots

struct FusedParams {
    HashGridDev g;
    const __half2 *table; const uint8_t *cells; int np; const void *weight_image; uint32_t image_bytes; int density_hidden, color_hidden;
    const uint8_t *bitfield; const float *rays_o; const float *rays_d; int n_rays;
    float lo, hi, near_distance, cone; Pcg32 rng;
    float bg[3]; int rgb_act, dens_act;
    float *rgb_out; float *alpha_out; int32_t *n_samples_out;
    float *tscratch;     // [gridDim.x * FR_N_PROD][32][FR_TCAP]
    uint32_t *sched;     // [0] next ray group, [1] CTAs finished (both zero between launches)
    unsigned long long *dbg_out;   // [gridDim.x][16]: start ns, end ns, smid, tiles, 5 field-phase (warpgroup 0) and 7 producer-phase cycle sums (only written when dbg & 8)
    int dbg;             // developer ablation bits (XRB_FUSED_DBG): 1 skip the hash gather, 2 skip the MLP layers, 4 fake march (11 samples/ray)
    float *depth_out;    // [n_rays], written by the DEPTH instantiation only (last member: the depth-free kernel reads every other one at its old offset)
};

struct FusedCtl {
    uint64_t full[FR_N_SLOTS];            // count 4: one arrival per chunk (producer lane 0, or the closing field thread for a skipped quarter)
    uint64_t mail[FR_N_PROD][2];          // count 32: the 32 field threads holding a producer's rows; a producer's chunk k uses mailbox k & 1
    uint64_t wbar;
    uint32_t rounds_done[FR_N_SLOTS];     // slot s may be written for round r once rounds_done[s] >= r (set when its rows have been copied out)
    uint32_t owner[FR_N_SLOTS][4];        // (producer index << 1 | mailbox parity) of each quarter
    uint32_t issued_bcast[FR_N_WG];
    uint32_t ticket, closed, done, prod_done;
    uint32_t morton[128];                 // expand_bits7 table for the occupancy test (common.cuh morton_lut_init)
};
__host__ __device__ inline size_t fused_smem_bytes(uint32_t image_bytes) {
    return 1024 + image_bytes + (size_t)FR_N_WG * (TILE_BLOCK_BYTES + TC_STAGE_BYTES) + (size_t)FR_N_SLOTS * FR_SLOT_BYTES + (size_t)FR_N_PROD * 1024 + sizeof(FusedCtl) + 64;
}

__device__ __forceinline__ void spin_until_ge(volatile uint32_t *p, uint32_t v) {
    while (*p < v) __nanosleep(20);
}

// DEPTH = false is the kernel without depth (no register or instruction of the depth channel exists in it).
template <bool DEPTH>
__global__ void __launch_bounds__((4 * FR_N_WG + FR_N_PROD) * 32, 1) ngp_render_fused_kernel(const __grid_constant__ FusedParams P) {
    extern __shared__ uint8_t dyn_smem[];
    uint8_t *base = (uint8_t *)(((uintptr_t)dyn_smem + 1023) & ~(uintptr_t)1023);
    uint8_t *W = base, *A = W + P.image_bytes, *stage = A + (size_t)FR_N_WG * TILE_BLOCK_BYTES, *slots = stage + (size_t)FR_N_WG * TC_STAGE_BYTES, *mailbox = slots + (size_t)FR_N_SLOTS * FR_SLOT_BYTES;
    FusedCtl *ctl = (FusedCtl *)(mailbox + (size_t)FR_N_PROD * 1024);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if ((P.dbg & 8) && threadIdx.x == 0) {
        unsigned long long t0; uint32_t smid;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0)); asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        P.dbg_out[16 * blockIdx.x] = t0; P.dbg_out[16 * blockIdx.x + 2] = smid; for (int k = 3; k < 16; ++k) P.dbg_out[16 * blockIdx.x + k] = 0;
    }

    if (threadIdx.x == 0) {
        for (int k = 0; k < FR_N_SLOTS; ++k) { tc::mbar_init(ctl->full + k, 4); ctl->rounds_done[k] = 0; }
        for (int k = 0; k < FR_N_PROD; ++k) { tc::mbar_init(&ctl->mail[k][0], 32); tc::mbar_init(&ctl->mail[k][1], 32); }
        for (int k = 0; k < FR_N_WG; ++k) ctl->issued_bcast[k] = 0;
        tc::mbar_init(&ctl->wbar, 1);
        ctl->ticket = 0; ctl->closed = 0; ctl->done = 0; ctl->prod_done = 0;
        tc::fence_mbar_init();
        tc::mbar_expect_tx(&ctl->wbar, P.image_bytes);
        tc::tma_bulk_g2s(W, P.weight_image, P.image_bytes, &ctl->wbar);
    }
    morton_lut_init(ctl->morton, threadIdx.x, blockDim.x);
    __syncthreads();

    if (warp < 4 * FR_N_WG) {
        // ===================================================================== field warpgroups
        TcWarpgroup c;
        c.wg = warp >> 2; c.row = threadIdx.x & 127;
        c.A = A + (size_t)c.wg * TILE_BLOCK_BYTES; c.W = W; c.stage = (float *)(stage + (size_t)c.wg * TC_STAGE_BYTES); c.bar = 1 + c.wg;
        const WeightImageLayout L = weight_image_layout(P.density_hidden, P.color_hidden);
        const bool timed = (P.dbg & 8) && c.wg == 0;
        tc::mbar_wait(&ctl->wbar, 0);
        long long fc[5] = {0, 0, 0, 0, 0}, ck = 0; (void)ck; (void)timed;
#ifdef XRB_FUSED_TIMERS
#define FTICK(k) do { if (timed) { long long n_ = clock64(); fc[k] += n_ - ck; ck = n_; } } while (0)
#else
#define FTICK(k) do { } while (0)
#endif
        for (uint32_t X = c.wg;; X += FR_N_WG) {
            const uint32_t s = X % FR_N_SLOTS, r = X / FR_N_SLOTS;
            FTICK(4);
            if (c.row == 0) {
                volatile uint32_t *tk = &ctl->ticket; volatile uint32_t *dn = &ctl->done; volatile uint32_t *cl = &ctl->closed;
                while (*cl != X) __nanosleep(20);   // tiles are closed in order, alternately by the warpgroups
                uint32_t issued = 0;
                while (true) {
                    if (*tk > 4 * X) { issued = 1; break; }
                    if (*dn) { if (*tk > 4 * X) issued = 1; break; }
                    __nanosleep(20);
                }
                if (issued) {   // close the tile: later tickets go to tile X+1
                    while (true) {
                        uint32_t cur = *tk;
                        if (cur >= 4 * (X + 1)) { issued = 4; break; }
                        if (atomicCAS(&ctl->ticket, cur, 4 * (X + 1)) == cur) { issued = cur - 4 * X; break; }
                    }
                    for (uint32_t k = issued; k < 4; ++k) tc::mbar_arrive(ctl->full + s);
                }
                ctl->issued_bcast[c.wg] = issued;
                __threadfence_block();
                *cl = X + 1;
            }
            tc::named_bar_sync(3 + c.wg, 128);
            const uint32_t issued = *(volatile uint32_t *)&ctl->issued_bcast[c.wg];
            FTICK(0);
            if (issued == 0) { if (timed && c.row == 0) { P.dbg_out[16 * blockIdx.x + 3] = X; for (int k = 0; k < 5; ++k) P.dbg_out[16 * blockIdx.x + 4 + k] = (unsigned long long)fc[k]; } break; }
            tc::mbar_wait(ctl->full + s, r & 1);
            FTICK(1);
            const uint8_t *rowp = slots + (size_t)s * FR_SLOT_BYTES + (size_t)c.row * FR_ROW_BYTES;
            const uint4 f0 = *reinterpret_cast<const uint4 *>(rowp), f1 = *reinterpret_cast<const uint4 *>(rowp + 16), f2 = *reinterpret_cast<const uint4 *>(rowp + 32),
                        f3 = *reinterpret_cast<const uint4 *>(rowp + 48);
            const float4 dir = *reinterpret_cast<const float4 *>(rowp + 64);
            const uint32_t sub = c.row >> 5;
            const uint32_t own = ctl->owner[s][sub];
            a_store_chunk(c, 0, f0); a_store_chunk(c, 1, f1); a_store_chunk(c, 2, f2); a_store_chunk(c, 3, f3);
            tc::named_bar_sync(3 + c.wg, 128);   // every row of the slot has been read
            if (c.row == 0) { __threadfence_block(); *(volatile uint32_t *)&ctl->rounds_done[s] = r + 1; }
            FTICK(2);
            float4 raw = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!(P.dbg & 2)) {
                float dout[16];
                tc_density_from_a(c, L, P.density_hidden, dout);
                raw = tc_color_from_density(c, L, P.color_hidden, dout, dir.x, dir.y, dir.z);
            }
            FTICK(3);
            if (sub < issued) {
                *reinterpret_cast<float4 *>(mailbox + (size_t)own * 512 + (c.row & 31) * 16) = raw;   // own = producer << 1 | parity: 512-byte mailboxes
                tc::mbar_arrive(&ctl->mail[own >> 1][own & 1]);
            }
        }
    } else {
        // ===================================================================== producer warps
        const uint32_t pw = warp - 4 * FR_N_WG;
        float *tb = P.tscratch + ((size_t)blockIdx.x * FR_N_PROD + pw) * 32 * FR_TCAP;
        const float diag = sub_(P.hi, P.lo);
        uint32_t n_submitted = 0;   // chunks this warp has submitted so far (chunk k: mailbox k & 1, phase (k >> 1) & 1)
        long long pc[7] = {0, 0, 0, 0, 0, 0, 0}, ck = 0; (void)ck;
#ifdef XRB_FUSED_TIMERS
#define PTICK(k) do { if (P.dbg & 8) { long long n_ = clock64(); pc[k] += n_ - ck; ck = n_; } } while (0)
#else
#define PTICK(k) do { } while (0)
#endif
        // claim a quarter of a tile slot, write my sample's warped direction and its 16 encoded levels into the slot row, arrive (one call per 32-sample chunk, all lanes)
        auto submit_chunk = [&](float x, float y, float z, float wd0, float wd1, float wd2) {
            uint32_t tk = 0;
            if (lane == 0) tk = atomicAdd(&ctl->ticket, 1u);
            tk = __shfl_sync(0xffffffffu, tk, 0);
            const uint32_t X = tk >> 2, sub = tk & 3, s = X % FR_N_SLOTS, r = X / FR_N_SLOTS;
            if (lane == 0) { spin_until_ge(&ctl->rounds_done[s], r); __threadfence_block(); ctl->owner[s][sub] = (pw << 1) | (n_submitted & 1); }
            __syncwarp();
            PTICK(5);
            uint8_t *rowp = slots + (size_t)s * FR_SLOT_BYTES + (size_t)(sub * 32 + lane) * FR_ROW_BYTES;
            *reinterpret_cast<float4 *>(rowp + 64) = make_float4(wd0, wd1, wd2, 0.f);
            // hash encoding of my sample, level by level into the slot row (invalid lanes gather the cell of (0.5,0.5,0.5): L1 hits)
            if (P.dbg & 1) {
                for (int l = 0; l < 16; ++l) *reinterpret_cast<uint32_t *>(rowp + 4 * l) = pack_h2(x, y);
            } else if (P.np > 0) {   // two ROLLED loops (see the file header), each with ONE gather form when the static plan holds
#pragma unroll 1
                for (int l = 0; l < P.np; ++l) {
                    const float2 f = hash_level(P.table, P.cells, P.g, l, x, y, z, GATHER_PACKED);
                    *reinterpret_cast<uint32_t *>(rowp + 4 * l) = pack_h2(f.x, f.y);
                }
#pragma unroll 1
                for (int l = P.np; l < 16; ++l) {
                    const float2 f = hash_level(P.table, P.cells, P.g, l, x, y, z, GATHER_HASHED);
                    *reinterpret_cast<uint32_t *>(rowp + 4 * l) = pack_h2(f.x, f.y);
                }
            } else {
#pragma unroll 1
                for (int l = 0; l < 16; ++l) {
                    const float2 f = hash_level(P.table, P.cells, P.g, l, x, y, z, GATHER_RUNTIME);
                    *reinterpret_cast<uint32_t *>(rowp + 4 * l) = pack_h2(f.x, f.y);
                }
            }
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(ctl->full + s);
        };
        for (;;) {
            PTICK(6);
            uint32_t grp = 0;
            if (lane == 0) grp = atomicAdd(P.sched, 1u);
            grp = __shfl_sync(0xffffffffu, grp, 0);
            if ((uint64_t)grp * 32 >= (uint64_t)P.n_rays) break;
            const uint32_t ray = grp * 32 + lane;
            bool alive = ray < (uint32_t)P.n_rays;
            float t = 0.f; uint32_t nsteps = 0;
            if (alive) {
                const float o[3] = {__ldg(P.rays_o + 3 * (size_t)ray), __ldg(P.rays_o + 3 * (size_t)ray + 1), __ldg(P.rays_o + 3 * (size_t)ray + 2)};
                const float d[3] = {__ldg(P.rays_d + 3 * (size_t)ray), __ldg(P.rays_d + 3 * (size_t)ray + 1), __ldg(P.rays_d + 3 * (size_t)ray + 2)};
                t = ray_start_t(P.rng, ray, P.lo, P.hi, o, d, P.near_distance, P.cone);
            }
            float T = 1.f, ax = 0.f, ay = 0.f, az = 0.f, ad = 0.f;
            bool any_alive;
            do {
                // ---- march round: up to FR_TCAP samples of my ray (ray_sampler.cu:58-72; pausing keeps the t sequence unchanged)
                uint32_t m = 0;
                if (alive && (P.dbg & 4)) {
                    float *tl = tb + (size_t)lane * FR_TCAP;
                    for (; m < 11; ++m) { tl[m] = t; t += 0.01f; }
                    nsteps = 11; alive = false;
                }
                if (alive) {
                    const float o[3] = {__ldg(P.rays_o + 3 * (size_t)ray), __ldg(P.rays_o + 3 * (size_t)ray + 1), __ldg(P.rays_o + 3 * (size_t)ray + 2)};
                    const float d[3] = {__ldg(P.rays_d + 3 * (size_t)ray), __ldg(P.rays_d + 3 * (size_t)ray + 1), __ldg(P.rays_d + 3 * (size_t)ray + 2)};
                    float *tl = tb + (size_t)lane * FR_TCAP;
                    alive = !march(t, nsteps, NERF_STEPS, o, d, P.lo, P.hi, P.cone, P.bitfield, ctl->morton, [&](uint32_t, float t, float) {
                        tl[m] = t;
                        return ++m != FR_TCAP;
                    });
                }
                __syncwarp();
                PTICK(0);
                any_alive = __any_sync(0xffffffffu, alive);
                const uint32_t incl = warp_incl_scan_u32(m, lane);
                const uint32_t rbase = incl - m, total = __shfl_sync(0xffffffffu, incl, 31);

                bool pending = false; uint32_t pend_key = 0; float pend_dt = 0.f, pend_t = 0.f;   // pend_key: ray-in-group of my sample of the previous chunk (>= 32: none)
                for (uint32_t q0 = 0; q0 < total || pending; q0 += 32) {
                    const bool have_chunk = q0 < total;
                    float dtc = 0.f, tc = 0.f; uint32_t key = 32u + lane;
                    PTICK(6);
                    if (have_chunk) {
                        // ---- lane = sample q of the round's ray-ordered stream: which ray, which t
                        const uint32_t q = q0 + lane;
                        const bool valid = q < total;
                        uint32_t j = 0;
#pragma unroll
                        for (uint32_t step = 16; step >= 1; step >>= 1) {
                            const uint32_t cand = j + step;
                            const uint32_t b = __shfl_sync(0xffffffffu, rbase, cand & 31);
                            if (cand < 32 && b <= q) j = cand;
                        }
                        const uint32_t bj = __shfl_sync(0xffffffffu, rbase, j);
                        float x[3] = {0.5f, 0.5f, 0.5f}, wd[3] = {0.5f, 0.5f, 0.5f};
                        if (valid) {
                            const float tt = *(volatile float *)(tb + (size_t)j * FR_TCAP + (q - bj));
                            const size_t rj = (size_t)grp * 32 + j;
                            const float oj[3] = {__ldg(P.rays_o + 3 * rj), __ldg(P.rays_o + 3 * rj + 1), __ldg(P.rays_o + 3 * rj + 2)};
                            const float dj[3] = {__ldg(P.rays_d + 3 * rj), __ldg(P.rays_d + 3 * rj + 1), __ldg(P.rays_d + 3 * rj + 2)};
                            sample_warped_pos(oj, dj, tt, P.lo, diag, x);
                            sample_warped_dir(dj, wd);
                            dtc = sample_row_dt(tt, P.cone);   // the value the unfused composite reads back from the row
                            if (DEPTH) tc = tt;
                            key = j;
                        }
#ifdef XRB_FUSED_TIMERS
                        if (P.dbg & 8) { if (__float_as_uint(x[0] + x[1] + x[2] + dtc) == 0x7fc12345u) pc[6] += 1; }   // force the loads to have landed
#endif
                        PTICK(1);
                        submit_chunk(x[0], x[1], x[2], wd[0], wd[1], wd[2]);
                        PTICK(2);
                    }
                    // ---- results of the previous chunk (its tile ran on the tensor core during this gather): composite
                    if (pending) {
                        const uint32_t kprev = n_submitted - 1;
                        if (lane == 0) tc::mbar_wait(&ctl->mail[pw][kprev & 1], (kprev >> 1) & 1);   // one lane polls: 32 lanes leaving a spin loop at different
                        __syncwarp();                                                               // iterations run the scan below diverged (shfl slow path)
                        PTICK(3);
                        const float4 raw = *reinterpret_cast<const float4 *>(mailbox + (size_t)((pw << 1) | (kprev & 1)) * 512 + lane * 16);
                        float alpha = 0.f, sx = 0.f, sy = 0.f, sz = 0.f, sd = 0.f;
                        if (pend_key < 32) {
                            const CompositeTerm s = composite_term(raw, pend_dt, P.rgb_act, P.dens_act);
                            alpha = s.alpha; sx = alpha * s.r; sy = alpha * s.g; sz = alpha * s.b;
                            if (DEPTH) sd = alpha * pend_t;
                        }
                        float pr = 1.f - alpha;
                        // segmented inclusive scan over the 32 samples; a segment = consecutive samples of one ray
                        const uint32_t prev_key = __shfl_up_sync(0xffffffffu, pend_key, 1);
                        const uint32_t heads = __ballot_sync(0xffffffffu, lane == 0 || pend_key != prev_key);
                        const int seg_start = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
#pragma unroll
                        for (int off = 1; off < 32; off <<= 1) {
                            const float np = __shfl_up_sync(0xffffffffu, pr, off), nx = __shfl_up_sync(0xffffffffu, sx, off), ny = __shfl_up_sync(0xffffffffu, sy, off),
                                        nz = __shfl_up_sync(0xffffffffu, sz, off);
                            const float nd = DEPTH ? __shfl_up_sync(0xffffffffu, sd, off) : 0.f;
                            if ((int)lane - off >= seg_start) { sx = nx + np * sx; sy = ny + np * sy; sz = nz + np * sz; if (DEPTH) sd = nd + np * sd; pr = np * pr; }
                        }
                        // lane i == ray i: take the aggregate of my segment (at its last sample inside the previous chunk [q0-32, q0))
                        const uint32_t pq0 = q0 - 32;
                        const uint32_t lo_q = max(rbase, pq0), hi_q = min(rbase + m, q0);
                        const uint32_t tail = (hi_q - 1 - pq0) & 31;
                        const float gp = __shfl_sync(0xffffffffu, pr, tail), gx = __shfl_sync(0xffffffffu, sx, tail), gy = __shfl_sync(0xffffffffu, sy, tail),
                                    gz = __shfl_sync(0xffffffffu, sz, tail);
                        const float gd = DEPTH ? __shfl_sync(0xffffffffu, sd, tail) : 0.f;
                        if (hi_q > lo_q) { ax += T * gx; ay += T * gy; az += T * gz; if (DEPTH) ad += T * gd; T *= gp; }
                        pending = false;
                        PTICK(4);
                    }
                    if (have_chunk) { ++n_submitted; pending = true; pend_key = key; pend_dt = dtc; if (DEPTH) pend_t = tc; }
                }
            } while (any_alive);
            if (ray < (uint32_t)P.n_rays) {
                P.rgb_out[3 * (size_t)ray] = ax + T * P.bg[0]; P.rgb_out[3 * (size_t)ray + 1] = ay + T * P.bg[1]; P.rgb_out[3 * (size_t)ray + 2] = az + T * P.bg[2];
                P.alpha_out[ray] = 1.f - T;
                if (DEPTH) P.depth_out[ray] = ad;
                if (P.n_samples_out) P.n_samples_out[ray] = (int32_t)nsteps;
            }
        }
        if ((P.dbg & 8) && lane == 0) { for (int k = 0; k < 7; ++k) atomicAdd(P.dbg_out + 16 * blockIdx.x + 9 + k, (unsigned long long)pc[k]); }
        if (lane == 0) {
            __threadfence_block();
            if (atomicAdd(&ctl->prod_done, 1u) == FR_N_PROD - 1) *(volatile uint32_t *)&ctl->done = 1u;
        }
    }
    __syncthreads();
    if ((P.dbg & 8) && threadIdx.x == 0) { unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); P.dbg_out[16 * blockIdx.x + 1] = t1; }
    if (threadIdx.x == 0) {   // leave the scheduler words zero for the next launch
        __threadfence();
        if (atomicAdd(P.sched + 1, 1u) == gridDim.x - 1) { P.sched[0] = 0; P.sched[1] = 0; __threadfence(); }
    }
}

constexpr int FUSED_MAX_PROD_PER_SM = 24;

// xrb_ngp_render_fused (DEPTH = false, depth_out unused) and xrb_ngp_render_fused_depth
template <bool DEPTH>
static int render_fused(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield, const float *rays_o, const float *rays_d, int n_rays,
                        float aabb0, float aabb1, float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act, int dens_act,
                        float *rgb_out, float *alpha_out, float *depth_out, int32_t *n_samples_out, void *workspace, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n_rays >= 0, "ngp_render_fused: bad size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(table && weight_image && bitfield && rays_o && rays_d && bg3_host && rgb_out && alpha_out && (depth_out || !DEPTH) && workspace, "ngp_render_fused: null pointer");
    XRB_REQUIRE(((uintptr_t)workspace & 255) == 0 && ((uintptr_t)weight_image & 15) == 0, "ngp_render_fused: workspace must be 256-byte aligned, weight image 16-byte aligned");
    FusedParams P;
    e = table_setup(cfg, table, &P.g); if (e) return e;
    P.table = (const __half2 *)table->table_fp16; P.cells = (const uint8_t *)table->cell_image; P.np = plan_valid(P.g, table->n_packed_levels) ? table->n_packed_levels : 0;
    P.weight_image = weight_image; P.image_bytes = weight_image_layout(cfg->density_hidden, cfg->color_hidden).total;
    P.density_hidden = cfg->density_hidden; P.color_hidden = cfg->color_hidden;
    P.bitfield = bitfield; P.rays_o = rays_o; P.rays_d = rays_d; P.n_rays = n_rays;
    P.lo = aabb0; P.hi = aabb1; P.near_distance = near_distance; P.cone = cone_angle; P.rng = host_rng(seed, n_prior_calls);
    P.bg[0] = bg3_host[0]; P.bg[1] = bg3_host[1]; P.bg[2] = bg3_host[2]; P.rgb_act = rgb_act; P.dens_act = dens_act;
    P.rgb_out = rgb_out; P.alpha_out = alpha_out; P.depth_out = depth_out; P.n_samples_out = n_samples_out;
    { static const int dbg = getenv("XRB_FUSED_DBG") ? atoi(getenv("XRB_FUSED_DBG")) : 0; P.dbg = dbg; }
    const int sms = sm_count();
    P.sched = (uint32_t *)workspace; P.tscratch = (float *)((uint8_t *)workspace + 256);
    P.dbg_out = (unsigned long long *)((uint8_t *)workspace + 256 + (size_t)sms * FUSED_MAX_PROD_PER_SM * 32 * FR_TCAP * sizeof(float));
    const int64_t n_groups = ((int64_t)n_rays + 31) / 32;
    const size_t smem = fused_smem_bytes(P.image_bytes);
    cudaFuncSetAttribute(ngp_render_fused_kernel<DEPTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   // per call: the attribute is per device and per image size
    int grid = sms; if (n_groups < grid) grid = (int)n_groups;
    ngp_render_fused_kernel<DEPTH><<<grid, (4 * FR_N_WG + FR_N_PROD) * 32, smem, (cudaStream_t)stream>>>(P);
    return check_launch("ngp_render_fused");
}

}  // namespace xrb

using namespace xrb;

extern "C" {

size_t xrb_ngp_render_fused_workspace(void) {
    const int sms = sm_count();
    return 256 + (size_t)sms * FUSED_MAX_PROD_PER_SM * 32 * FR_TCAP * sizeof(float) + (size_t)sms * 2 * 128;
}

int xrb_ngp_render_fused(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield, const float *rays_o, const float *rays_d, int n_rays,
                         float aabb0, float aabb1, float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act, int dens_act,
                         float *rgb_out, float *alpha_out, int32_t *n_samples_out, void *workspace, void *stream) {
    return render_fused<false>(cfg, table, weight_image, bitfield, rays_o, rays_d, n_rays, aabb0, aabb1, near_distance, cone_angle, seed, n_prior_calls, bg3_host, rgb_act, dens_act,
                               rgb_out, alpha_out, nullptr, n_samples_out, workspace, stream);
}

int xrb_ngp_render_fused_depth(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield, const float *rays_o, const float *rays_d,
                               int n_rays, float aabb0, float aabb1, float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act,
                               int dens_act, float *rgb_out, float *alpha_out, float *depth_out, int32_t *n_samples_out, void *workspace, void *stream) {
    return render_fused<true>(cfg, table, weight_image, bitfield, rays_o, rays_d, n_rays, aabb0, aabb1, near_distance, cone_angle, seed, n_prior_calls, bg3_host, rgb_act, dens_act,
                              rgb_out, alpha_out, depth_out, n_samples_out, workspace, stream);
}

}  // extern "C"
