// xrnerf_b200 — sm_90a replacements for the 10 `raymarch_cuda` ops (C ABI: xrb_rm_*, include/xrnerf_b200.h).
//
// What differs from the reference kernels (all <<<n/128,128>>> thread-per-element, extensions/ngp_raymarch/src/*.cu):
//   * ray march: count pass + 2-level exclusive scan + emit pass => deterministic ray-order layout, no global
//     atomics, no device sync, start-t (the only RNG use) computed once and cached in the workspace;
//   * compositing: one WARP per ray, lanes over samples (coalesced float4 reads of raw[S,4]), transmittance by a
//     warp product-scan instead of a serial loop per thread;
//   * grid kernels: 128-bit vector loads/stores, grid sized to a multiple of the SM count with grid-stride loops,
//     bitfield + 7 max-pool levels produced by ONE kernel launch sequence without atomics, fixed-order mean.
// HBM roofline per op (algorithmic bytes) is listed in DESIGN.md §4.
#include "common.cuh"
#include <stdio.h>
#include <string.h>

namespace xrb {

static thread_local char g_err[256] = "";
void set_error(const char *msg) { strncpy(g_err, msg, sizeof(g_err) - 1); g_err[sizeof(g_err) - 1] = 0; }
int check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e)); return (int)e; }
    return XRB_OK;
}

// ============================================================================ ray march
// Count pass: one thread per ray marches it (common.cuh march(), ray_sampler.cu:58-72). Emit pass: one warp per ray writes its rows (:99-115).
constexpr uint32_t TCAP = 64;                      // per-ray sample-t slots cached inline by the count pass
constexpr uint32_t OVF_CAP = NERF_STEPS - TCAP;    // a ray with more samples gets ONE overflow chunk of this many slots (bump-allocated), so the emit
                                                   // pass can rebuild all of its rows in parallel; only when the chunk pool is exhausted is it re-marched
struct OvfPool { uint32_t *counter; float *area; uint32_t n_chunks; int32_t *chunk_of; };

constexpr int MARCH_BLOCK = 128;
// grid for warp-per-ray kernels with persistent (ray-strided) warps
static inline int warp_grid(int n_rays) { return stride_grid(((int64_t)n_rays * 32 + 255) / 256, 8); }

struct MarchWs {  // device workspace layout for N rays
    uint32_t *local_excl;  // [N]
    float *startt;         // [N]
    uint32_t *block_sum;   // [n_blocks] -> exclusive block offsets after scan
    uint32_t *misc;        // [16]: base0, ray0, total, overflow-chunk counter
    float *tbuf;           // [N][TCAP] sample t values found by the count pass
    int32_t *chunk_of;     // [N] overflow chunk of a ray with more than TCAP samples (-1: pool exhausted); valid only for such rays
    float *ovf;            // [n_chunks][OVF_CAP]
    uint32_t n_chunks;
};
__host__ __device__ inline size_t march_n_blocks(int n) { return ((size_t)n + MARCH_BLOCK - 1) / MARCH_BLOCK; }   // count-pass blocks = block sums in the workspace
__host__ __device__ inline uint32_t march_n_chunks(int n) { uint32_t c = (uint32_t)n / 8u; return c < 64u ? 64u : c; }   // every 8th ray may be longer than TCAP samples
__host__ __device__ inline size_t march_ws_bytes(int n) {
    return sizeof(uint32_t) * ((size_t)n * 3 + march_n_blocks(n) + 16 + (size_t)n * TCAP + (size_t)march_n_chunks(n) * OVF_CAP);
}
inline MarchWs march_ws(void *ws, int n) {
    MarchWs w; w.local_excl = (uint32_t *)ws; w.startt = (float *)(w.local_excl + n); w.block_sum = (uint32_t *)(w.startt + n); w.misc = w.block_sum + march_n_blocks(n); w.tbuf = (float *)(w.misc + 16);
    w.chunk_of = (int32_t *)(w.tbuf + (size_t)n * TCAP); w.ovf = (float *)(w.chunk_of + n); w.n_chunks = march_n_chunks(n);
    return w;
}

// Count pass: thread i marches ray i, caching its sample t values, and the block scans the per-ray sample counts.
__global__ void __launch_bounds__(MARCH_BLOCK) march_count_kernel(int n_rays, const float *__restrict__ rays_o, const float *__restrict__ rays_d,
                                                                  const uint8_t *__restrict__ bitfield, float lo, float hi, float near_distance, float cone,
                                                                  Pcg32 rng, uint32_t *__restrict__ local_excl, float *__restrict__ startt_out,
                                                                  uint32_t *__restrict__ block_sum, int32_t *__restrict__ numsteps, float *__restrict__ tbuf, OvfPool pool) {
    __shared__ uint32_t lut[128];
    morton_lut_init(lut, threadIdx.x, MARCH_BLOCK);
    __syncthreads();
    uint32_t i = blockIdx.x * MARCH_BLOCK + threadIdx.x;
    uint32_t n = 0;
    if (i < (uint32_t)n_rays) {
        float o[3] = {rays_o[3 * (size_t)i], rays_o[3 * (size_t)i + 1], rays_o[3 * (size_t)i + 2]};
        float d[3] = {rays_d[3 * (size_t)i], rays_d[3 * (size_t)i + 1], rays_d[3 * (size_t)i + 2]};
        float t = ray_start_t(rng, i, lo, hi, o, d, near_distance, cone);
        startt_out[i] = t;
        float *tl = tbuf ? tbuf + (size_t)i * TCAP : nullptr, *ovf = nullptr;   // tbuf == nullptr: count only
        const OvfPool *pp = tbuf ? &pool : nullptr;   // through a pointer, as ever: the by-value form made the training step 0.4 % slower (H100 80GB HBM3, 700 W)
        march(t, n, NERF_STEPS, o, d, lo, hi, cone, bitfield, lut, [&](uint32_t j, float t, float) {
            if (!tl) return true;
            if (j < TCAP) { tl[j] = t; return true; }
            if (!pp) return true;
            if (j == TCAP) {   // claim the overflow chunk
                const uint32_t c = atomicAdd(pp->counter, 1u);
                const bool got = c < pp->n_chunks;
                pp->chunk_of[i] = got ? (int32_t)c : -1;
                ovf = got ? pp->area + (size_t)c * OVF_CAP : nullptr;
            }
            if (ovf) ovf[j - TCAP] = t;
            return true;
        });
        numsteps[2 * (size_t)i] = (int32_t)n;
    }
    uint32_t tot;
    uint32_t ex = block_excl_scan<MARCH_BLOCK>(n, &tot);
    if (i < (uint32_t)n_rays) local_excl[i] = ex;
    if (threadIdx.x == 0) block_sum[blockIdx.x] = tot;
}

// single block: exclusive scan of block sums, base/ray counters bookkeeping (counters[] accumulate like the reference's atomics)
__global__ void __launch_bounds__(1024) march_scan_kernel(int n_blocks, uint32_t *__restrict__ block_sum, uint32_t *__restrict__ misc, int32_t *__restrict__ counters) {
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int b0 = 0; b0 < n_blocks; b0 += 1024) {
        int b = b0 + threadIdx.x;
        uint32_t tot, ex = block_excl_scan<1024>(b < n_blocks ? block_sum[b] : 0u, &tot);
        uint32_t carry = carry_s;
        if (b < n_blocks) block_sum[b] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t base0 = counters ? (uint32_t)counters[1] : 0u, ray0 = counters ? (uint32_t)counters[0] : 0u;
        misc[0] = base0; misc[1] = ray0; misc[2] = carry_s;
        if (counters) counters[1] = (int32_t)(base0 + carry_s);
    }
}

// Emit pass, one WARP per ray: lanes rebuild rows from the cached t values (pos = o + t d and dt = calc_dt(t) are the very
// expressions of the march, so the rows are bit-identical to a second march) and write 32 consecutive 28-byte rows per step.
// Rays longer than TCAP are re-marched by lane 0 (ray_sampler.cu:99-115).
__global__ void __launch_bounds__(256) march_emit_kernel(int n_rays, const float *__restrict__ rays_o, const float *__restrict__ rays_d, const uint8_t *__restrict__ bitfield, float lo,
                                                         float hi, float cone, uint32_t max_samples, const uint32_t *__restrict__ local_excl, const float *__restrict__ startt,
                                                         const uint32_t *__restrict__ block_off, const uint32_t *__restrict__ misc, const float *__restrict__ tbuf,
                                                         const int32_t *__restrict__ chunk_of, const float *__restrict__ ovf, float *__restrict__ coords_out, int32_t *__restrict__ rays_index, int32_t *__restrict__ numsteps,
                                                         int32_t *__restrict__ counters) {
    const int lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * 256) >> 5;
    uint32_t ok_count = 0;
    for (uint32_t i = (blockIdx.x * 256 + threadIdx.x) >> 5; i < (uint32_t)n_rays; i += n_warps) {   // persistent warps: 8192 tiny blocks cost more to schedule than to run
        uint32_t n = (uint32_t)numsteps[2 * (size_t)i];
        uint32_t base = misc[0] + block_off[i / MARCH_BLOCK] + local_excl[i];
        __syncwarp();
        if (base + n > max_samples) {  // ray_sampler.cu:76-82
            if (lane == 0) { numsteps[2 * (size_t)i] = 0; numsteps[2 * (size_t)i + 1] = (int32_t)base; }
        } else {
            ok_count += 1;
            if (lane == 0) {
                numsteps[2 * (size_t)i + 1] = (int32_t)base;
                // serial-order equivalent of `ray_idx = atomicAdd(ray_counter,1)`: slots are a prefix of the rays (see DESIGN.md §3.1)
                rays_index[i] = n == 0 ? -1 : (int32_t)(misc[1] + i);
            }
            if (n > 0) {
                const float o[3] = {rays_o[3 * (size_t)i], rays_o[3 * (size_t)i + 1], rays_o[3 * (size_t)i + 2]};
                const float d[3] = {rays_d[3 * (size_t)i], rays_d[3 * (size_t)i + 1], rays_d[3 * (size_t)i + 2]};
                const float diag = sub_(hi, lo);
                // rows whose t is cached (inline slots, then the ray's overflow chunk) are rebuilt by all lanes
                const int32_t chunk = n > TCAP ? chunk_of[i] : -1;
                const float *tl = tbuf + (size_t)i * TCAP, *to = chunk >= 0 ? ovf + (size_t)chunk * OVF_CAP : nullptr;
                const uint32_t n_par = n <= TCAP ? n : (to ? n : TCAP - 1);
                for (uint32_t j = lane; j < n_par; j += 32) write_sample_row(coords_out + ROW_FLOATS * (size_t)(base + j), o, d, j < TCAP ? tl[j] : to[j - TCAP], cone, lo, diag);
                // chunk pool exhausted: lane 0 resumes the march AT cached sample TCAP-1 (the march state is just t) and emits the remaining rows (ray_sampler.cu:99-115)
                if (n_par < n && lane == 0) {
                    float *rows = coords_out + ROW_FLOATS * (size_t)(base + TCAP - 1);
                    float t = tl[TCAP - 1]; uint32_t j = 0;
                    march(t, j, n - (TCAP - 1), o, d, lo, hi, cone, bitfield, nullptr, [&](uint32_t j, float t, float) {
                        write_sample_row(rows + ROW_FLOATS * (size_t)j, o, d, t, cone, lo, diag);
                        return true;
                    });
                }
            }
        }
    }
    if (lane == 0 && ok_count && counters) atomicAdd((unsigned int *)counters, ok_count);
}

// ============================================================================ compaction (compacted_coord.cu:5-77)
__global__ void __launch_bounds__(MARCH_BLOCK) compact_count_kernel(int n_rays, const int32_t *__restrict__ numsteps, uint32_t *__restrict__ local_excl,
                                                                    uint32_t *__restrict__ block_sum) {
    uint32_t i = blockIdx.x * MARCH_BLOCK + threadIdx.x;
    uint32_t n = i < (uint32_t)n_rays ? (uint32_t)numsteps[2 * (size_t)i] : 0u;
    uint32_t tot, ex = block_excl_scan<MARCH_BLOCK>(n, &tot);
    if (i < (uint32_t)n_rays) local_excl[i] = ex;
    if (threadIdx.x == 0) block_sum[blockIdx.x] = tot;
}
// warp per ray: copies its rows as a flat stream of floats (coalesced)
__global__ void __launch_bounds__(256) compact_copy_kernel(int n_rays, uint32_t max_compacted, const float *__restrict__ coords_in, const int32_t *__restrict__ numsteps,
                                                           const uint32_t *__restrict__ local_excl, const uint32_t *__restrict__ block_off, const uint32_t *__restrict__ misc,
                                                           float *__restrict__ coords_out, int32_t *__restrict__ numsteps_c, int32_t *__restrict__ ray_counter) {
    int lane = threadIdx.x & 31;
    uint32_t ray = (blockIdx.x * 256 + threadIdx.x) >> 5;
    if (ray >= (uint32_t)n_rays) return;
    uint32_t n = (uint32_t)numsteps[2 * (size_t)ray], base = (uint32_t)numsteps[2 * (size_t)ray + 1];
    uint32_t cbase = misc[0] + block_off[ray / MARCH_BLOCK] + local_excl[ray];
    uint32_t nc = min(max_compacted - min(max_compacted, cbase), n);  // :64
    if (lane == 0) { numsteps_c[2 * (size_t)ray] = (int32_t)nc; numsteps_c[2 * (size_t)ray + 1] = (int32_t)cbase; if (nc) atomicAdd((unsigned int *)ray_counter, 1u); }
    const float *src = coords_in + ROW_FLOATS * (size_t)base; float *dst = coords_out + ROW_FLOATS * (size_t)cbase;
    for (uint32_t k = lane; k < nc * ROW_FLOATS; k += 32) dst[k] = src[k];
}

// rays of a compacted batch whose every marched sample survived the compaction (numsteps_c.count == numsteps.count): the rays a training step really trains
__global__ void __launch_bounds__(256) count_trained_kernel(int n_rays, const int32_t *__restrict__ numsteps, const int32_t *__restrict__ numsteps_c, unsigned long long *__restrict__ accum) {
    unsigned int local = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rays; i += gridDim.x * blockDim.x) local += numsteps_c[2 * (size_t)i] == numsteps[2 * (size_t)i] ? 1u : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(accum, (unsigned long long)local);
}

// ============================================================================ compositing (calc_rgb.cu)
// what the depth composite (MODE 2) needs to rebuild each sample's t from its warped position; MODE 3 also reads each row's density gradient
// (grad f32[rows,3]) and writes normal_out f32[n_rays,3]
struct CompositeDepth {
    const float *rays_o, *rays_d; float lo, diag; float *depth_out;
    const float *grad; float *normal_out;
};

// MODE 0: training forward (per-ray bg, background only if not truncated; calc_rgb.cu:5-67)
// MODE 1: inference (global bg, alpha out; calc_rgb.cu:143-206)
// MODE 2: inference as MODE 1, plus depth = sum of w * t (include/xrnerf_b200.h, xrb_ngp_render_depth)
// MODE 3: MODE 2, plus normal = sum of w * n, n = -g / |g| (0 where g = 0) of the row's gradient g (xrb_ngp_render_normals)
// MODE 4: training forward as MODE 0, plus alpha = 1 - T and depth = sum of w * t as in MODE 2 (xrb_rm_calc_rgb_forward_geom)
template <int MODE>
__global__ void __launch_bounds__(256) composite_fwd_kernel(int n_rays, const float4 *__restrict__ raw, const float *__restrict__ coords, const int32_t *__restrict__ numsteps,
                                                            const int32_t *__restrict__ numsteps_c, const float *__restrict__ bg, float3 bg_global, int rgb_act, int dens_act,
                                                            float *__restrict__ rgb_out, float *__restrict__ alpha_out, CompositeDepth dp) {
    int lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * 256) >> 5;
    for (uint32_t ray = (blockIdx.x * 256 + threadIdx.x) >> 5; ray < (uint32_t)n_rays; ray += n_warps) {
    const int32_t *ns = MODE == 0 || MODE == 4 ? numsteps_c : numsteps;
    uint32_t n = (uint32_t)ns[2 * (size_t)ray], base = (uint32_t)ns[2 * (size_t)ray + 1];
    float3 b = MODE == 0 || MODE == 4 ? make_float3(bg[3 * (size_t)ray], bg[3 * (size_t)ray + 1], bg[3 * (size_t)ray + 2]) : bg_global;
    if (n == 0) {
        if (lane == 0) {
            rgb_out[3 * (size_t)ray] = b.x; rgb_out[3 * (size_t)ray + 1] = b.y; rgb_out[3 * (size_t)ray + 2] = b.z;
            if (MODE >= 1) alpha_out[ray] = 0.f;
            if (MODE >= 2) dp.depth_out[ray] = 0.f;
            if (MODE == 3) { dp.normal_out[3 * (size_t)ray] = 0.f; dp.normal_out[3 * (size_t)ray + 1] = 0.f; dp.normal_out[3 * (size_t)ray + 2] = 0.f; }
        }
        continue;
    }
    float o[3] = {0.f, 0.f, 0.f}, d[3] = {0.f, 0.f, 0.f}, inv_dd = 1.f;   // one division per ray, not per sample
    if (MODE >= 2) {
        o[0] = __ldg(dp.rays_o + 3 * (size_t)ray); o[1] = __ldg(dp.rays_o + 3 * (size_t)ray + 1); o[2] = __ldg(dp.rays_o + 3 * (size_t)ray + 2);
        d[0] = __ldg(dp.rays_d + 3 * (size_t)ray); d[1] = __ldg(dp.rays_d + 3 * (size_t)ray + 1); d[2] = __ldg(dp.rays_d + 3 * (size_t)ray + 2);
        inv_dd = 1.f / (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    }
    float T = 1.f, ax = 0.f, ay = 0.f, az = 0.f, ad = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
    for (uint32_t k0 = 0; k0 < n; k0 += 32) {
        uint32_t k = k0 + lane; bool valid = k < n;
        CompositeTerm s{0.f, 0.f, 0.f, 0.f}; float t = 0.f, n3[3] = {0.f, 0.f, 0.f};
        if (valid) {
            s = composite_term(__ldg(raw + base + k), row_dt(coords + ROW_FLOATS * (size_t)(base + k)), rgb_act, dens_act);
            if (MODE >= 2) t = row_t(coords + ROW_FLOATS * (size_t)(base + k), o, d, inv_dd, dp.lo, dp.diag);
            if (MODE == 3) {   // the sample's outward unit normal: inside is the larger density
                const float *gp = dp.grad + 3 * (size_t)(base + k);
                const float g0 = __ldg(gp), g1 = __ldg(gp + 1), g2 = __ldg(gp + 2), len = norm3df(g0, g1, g2);
                if (len > 0.f) { n3[0] = -g0 / len; n3[1] = -g1 / len; n3[2] = -g2 / len; }
            }
        }
        float incl, ex = warp_excl_prod(1.f - s.alpha, lane, &incl);
        float w = s.alpha * (T * ex);
        ax += w * s.r; ay += w * s.g; az += w * s.b;
        if (MODE >= 2) ad += w * t;
        if (MODE == 3) { nx += w * n3[0]; ny += w * n3[1]; nz += w * n3[2]; }
        T *= __shfl_sync(0xffffffffu, incl, 31);
    }
    ax = warp_sum(ax); ay = warp_sum(ay); az = warp_sum(az);
    if (MODE >= 2) ad = warp_sum(ad);
    if (MODE == 3) { nx = warp_sum(nx); ny = warp_sum(ny); nz = warp_sum(nz); }
    if (lane == 0) {
        bool add_bg = MODE >= 1 && MODE <= 3 ? true : (n == (uint32_t)numsteps[2 * (size_t)ray]);  // :61-64 / :199-202
        if (add_bg) { ax += T * b.x; ay += T * b.y; az += T * b.z; }
        rgb_out[3 * (size_t)ray] = ax; rgb_out[3 * (size_t)ray + 1] = ay; rgb_out[3 * (size_t)ray + 2] = az;
        if (MODE >= 1) alpha_out[ray] = 1.f - T;
        if (MODE >= 2) dp.depth_out[ray] = ad;
        if (MODE == 3) { dp.normal_out[3 * (size_t)ray] = nx; dp.normal_out[3 * (size_t)ray + 1] = ny; dp.normal_out[3 * (size_t)ray + 2] = nz; }
    }
    }
}

// the chain render's composite with depth (xrb_ngp_render_depth; arguments validated there)
int launch_composite_depth(const float *raw, const float *coords, const int32_t *numsteps, const float *bg3_host, int n_rays, int rgb_act, int dens_act, const float *rays_o,
                           const float *rays_d, float aabb0, float aabb1, float *rgb_out, float *alpha_out, float *depth_out, cudaStream_t s, const float *grad,
                           float *normal_out) {
    const CompositeDepth dp{rays_o, rays_d, aabb0, aabb1 - aabb0, depth_out, grad, normal_out};
    const float3 bg = make_float3(bg3_host[0], bg3_host[1], bg3_host[2]);
    if (normal_out) {
        composite_fwd_kernel<3><<<warp_grid(n_rays), 256, 0, s>>>(n_rays, (const float4 *)raw, coords, numsteps, nullptr, nullptr, bg, rgb_act, dens_act, rgb_out, alpha_out, dp);
        return check_launch("ngp_render_normals composite");
    }
    composite_fwd_kernel<2><<<warp_grid(n_rays), 256, 0, s>>>(n_rays, (const float4 *)raw, coords, numsteps, nullptr, nullptr, bg, rgb_act, dens_act, rgb_out, alpha_out, dp);
    return check_launch("ngp_render_depth composite");
}

// what the geometry backward (GEOM) reads beyond the colour gradient: the rays (t of each row, as row_t in MODE 2 / 4), the forward's depth and alpha,
// and their gradients (either may be NULL: no such term)
struct CompositeGeom {
    const float *rays_o, *rays_d; float lo, diag;
    const float *depth, *alpha, *grad_depth, *grad_alpha;
};

// compute_rgbs_grad (calc_rgb.cu:70-140). GEOM: the density channel also carries the depth and opacity terms,
// d depth / d(sigma_k dt_k) = Ta t_k - (D - D_<=k) and d alpha / d(sigma_k dt_k) = Ta - (A - A_<=k), under the same loss_scale
template <bool GEOM = false>
__global__ void __launch_bounds__(256) composite_bwd_kernel(int n_rays, const float4 *__restrict__ raw, const float *__restrict__ coords, const int32_t *__restrict__ numsteps_c,
                                                            const float *__restrict__ grad_rgb, const float *__restrict__ rgb_final, const float *__restrict__ grid_mean,
                                                            int rgb_act, int dens_act, float4 *__restrict__ dl_draw, CompositeGeom gm) {
    int lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * 256) >> 5;
    for (uint32_t ray = (blockIdx.x * 256 + threadIdx.x) >> 5; ray < (uint32_t)n_rays; ray += n_warps) {
    uint32_t n = (uint32_t)numsteps_c[2 * (size_t)ray], base = (uint32_t)numsteps_c[2 * (size_t)ray + 1];
    if (n == 0) continue;
    float loss_scale = 128.f / (float)n_rays;                                         // :92-93
    const float l2 = rgb_act == XRB_ACT_EXPONENTIAL ? 1e-4f : 0.0f;                   // :103
    const float l1 = __ldg(grid_mean) < NERF_MIN_OPTICAL_THICKNESS ? 1e-4f : 0.0f;    // :104
    float gx = grad_rgb[3 * (size_t)ray], gy = grad_rgb[3 * (size_t)ray + 1], gz = grad_rgb[3 * (size_t)ray + 2];
    float fx = rgb_final[3 * (size_t)ray], fy = rgb_final[3 * (size_t)ray + 1], fz = rgb_final[3 * (size_t)ray + 2];
    float gd = 0.f, ga = 0.f, fd = 0.f, fa = 0.f, ro[3] = {0.f, 0.f, 0.f}, d[3] = {0.f, 0.f, 0.f}, inv_dd = 1.f;
    const bool geo = GEOM && (gm.grad_depth || gm.grad_alpha);   // without either gradient, the colour-only arithmetic exactly
    if (geo) {
        gd = gm.grad_depth ? gm.grad_depth[ray] : 0.f; ga = gm.grad_alpha ? gm.grad_alpha[ray] : 0.f;
        fd = gm.depth[ray]; fa = gm.alpha[ray];
        ro[0] = __ldg(gm.rays_o + 3 * (size_t)ray); ro[1] = __ldg(gm.rays_o + 3 * (size_t)ray + 1); ro[2] = __ldg(gm.rays_o + 3 * (size_t)ray + 2);
        d[0] = __ldg(gm.rays_d + 3 * (size_t)ray); d[1] = __ldg(gm.rays_d + 3 * (size_t)ray + 1); d[2] = __ldg(gm.rays_d + 3 * (size_t)ray + 2);
        inv_dd = 1.f / (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    }
    float T = 1.f, px = 0.f, py = 0.f, pz = 0.f, pd = 0.f, pa = 0.f;  // running transmittance / prefix colour (and depth, alpha) carried across 32-sample chunks
    for (uint32_t k0 = 0; k0 < n; k0 += 32) {
        uint32_t k = k0 + lane; bool valid = k < n;
        float4 r = make_float4(0, 0, 0, 0); float dt = 0.f, t = 0.f; CompositeTerm s{0.f, 0.f, 0.f, 0.f};
        if (valid) {
            r = __ldg(raw + base + k);
            dt = row_dt(coords + ROW_FLOATS * (size_t)(base + k));
            s = composite_term(r, dt, rgb_act, dens_act);
            if (geo) t = row_t(coords + ROW_FLOATS * (size_t)(base + k), ro, d, inv_dd, gm.lo, gm.diag);
        }
        float incl, ex = warp_excl_prod(1.f - s.alpha, lane, &incl);
        float Tb = T * ex, w = s.alpha * Tb, Ta = Tb * (1.f - s.alpha);
        float sx = px + warp_incl_sum(w * s.r, lane), sy = py + warp_incl_sum(w * s.g, lane), sz = pz + warp_incl_sum(w * s.b, lane);  // rgb_ray2 after this sample
        float sd = 0.f, sa = 0.f;
        if (geo) { sd = pd + warp_incl_sum(w * t, lane); sa = pa + warp_incl_sum(w, lane); }     // depth and alpha after this sample
        if (valid) {
            float4 o;
            o.x = loss_scale * (w * gx * net_to_rgb_deriv(r.x, rgb_act) + fmaxf(0.0f, l2 * r.x));
            o.y = loss_scale * (w * gy * net_to_rgb_deriv(r.y, rgb_act) + fmaxf(0.0f, l2 * r.y));
            o.z = loss_scale * (w * gz * net_to_rgb_deriv(r.z, rgb_act) + fmaxf(0.0f, l2 * r.z));
            float dot = gx * (Ta * s.r - (fx - sx)) + (gy * (Ta * s.g - (fy - sy)) + gz * (Ta * s.b - (fz - sz)));
            if (geo) dot += gd * (Ta * t - (fd - sd)) + ga * (Ta - (fa - sa));
            o.w = loss_scale * (net_to_density_deriv(r.w, dens_act) * (dt * dot)) + (r.w < 0.f ? -l1 : 0.0f);
            dl_draw[base + k] = o;
        }
        T *= __shfl_sync(0xffffffffu, incl, 31);
        px = __shfl_sync(0xffffffffu, sx, 31); py = __shfl_sync(0xffffffffu, sy, 31); pz = __shfl_sync(0xffffffffu, sz, 31);
        if (geo) { pd = __shfl_sync(0xffffffffu, sd, 31); pa = __shfl_sync(0xffffffffu, sa, 31); }
    }
    }
}

// NGP camera pose refinement (xrb_ngp_ray_grad): per-row (dL/dx, dL/dw) of the field's INPUTS backward -> dL/do and dL/dd of each ray, t_k held fixed:
//   dL/do = sum_k dL/dx_k / diag,  dL/dd = sum_k t_k dL/dx_k / diag + 1/2 sum_k dL/dw_k,  times `scale`; one warp per ray over its compacted rows
__global__ void __launch_bounds__(256) ray_grad_kernel(int n_rays, const float *__restrict__ d_rows, const float *__restrict__ coords, const int32_t *__restrict__ numsteps_c,
                                                       const float *__restrict__ rays_o, const float *__restrict__ rays_d, float lo, float diag, float scale,
                                                       float *__restrict__ grad_o, float *__restrict__ grad_d) {
    const int lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * 256) >> 5;
    for (uint32_t ray = (blockIdx.x * 256 + threadIdx.x) >> 5; ray < (uint32_t)n_rays; ray += n_warps) {
        const uint32_t n = (uint32_t)numsteps_c[2 * (size_t)ray], base = (uint32_t)numsteps_c[2 * (size_t)ray + 1];
        float o[3], d[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { o[c] = __ldg(rays_o + 3 * (size_t)ray + c); d[c] = __ldg(rays_d + 3 * (size_t)ray + c); }
        const float inv_dd = 1.f / (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        float sx[3] = {0.f, 0.f, 0.f}, stx[3] = {0.f, 0.f, 0.f}, sw[3] = {0.f, 0.f, 0.f};
        for (uint32_t k = lane; k < n; k += 32) {
            const float *r = d_rows + 6 * (size_t)(base + k);
            const float t = row_t(coords + ROW_FLOATS * (size_t)(base + k), o, d, inv_dd, lo, diag);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float gx = __ldg(r + c);
                sx[c] += gx; stx[c] = fmaf(t, gx, stx[c]); sw[c] += __ldg(r + 3 + c);
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { sx[c] = warp_sum(sx[c]); stx[c] = warp_sum(stx[c]); sw[c] = warp_sum(sw[c]); }
        if (lane == 0) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                grad_o[3 * (size_t)ray + c] = scale * (sx[c] / diag);
                grad_d[3 * (size_t)ray + c] = scale * (stx[c] / diag + 0.5f * sw[c]);
            }
        }
    }
}

// ============================================================================ occupancy grid kernels
constexpr int GRID_THREADS = 256;
static inline int stream_grid(size_t work_items) { return stride_grid((int64_t)((work_items + GRID_THREADS - 1) / GRID_THREADS), 8); }

// mark_untrained_density_grid.cu:5-51; always writes (Q1)
__global__ void __launch_bounds__(GRID_THREADS) mark_untrained_kernel(uint32_t n_elements, float *__restrict__ grid, uint32_t n_images, const float2 *__restrict__ focal,
                                                                      const float *__restrict__ xforms, int res0, int res1) {
    extern __shared__ float s_cam[];  // [n_images][14]: 12 xform + 2 focal (cameras are read by every thread)
    for (uint32_t k = threadIdx.x; k < n_images * 14; k += blockDim.x) {
        uint32_t j = k / 14, c = k % 14;
        s_cam[k] = c < 12 ? xforms[12 * (size_t)j + c] : (c == 12 ? focal[j].x : focal[j].y);
    }
    __syncthreads();
    const float half_resx = mul_((float)res0, 0.5f), half_resy = mul_((float)res1, 0.5f);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_elements; i += gridDim.x * blockDim.x) {
        uint32_t level = i / GRID_CELLS, pos_idx = i % GRID_CELLS;
        float x = (float)morton3D_invert(pos_idx >> 0), y = (float)morton3D_invert(pos_idx >> 1), z = (float)morton3D_invert(pos_idx >> 2);
        float s = __uint_as_float((127u + level) << 23);
        float px = add_(mul_(sub_(div_(add_(x, 0.5f), (float)NERF_GRIDSIZE), 0.5f), s), 0.5f);
        float py = add_(mul_(sub_(div_(add_(y, 0.5f), (float)NERF_GRIDSIZE), 0.5f), s), 0.5f);
        float pz = add_(mul_(sub_(div_(add_(z, 0.5f), (float)NERF_GRIDSIZE), 0.5f), s), 0.5f);
        float voxel_radius = div_(mul_(mul_(0.5f, SQRT3()), s), (float)NERF_GRIDSIZE);
        int count = 0;
        for (uint32_t j = 0; j < n_images; ++j) {
            const float *m = s_cam + 14 * j;
            float lx = sub_(px, m[9]), ly = sub_(py, m[10]), lz = sub_(pz, m[11]);
            // Eigen fixed-size-3 dot = p0 + (p1 + p2)
            float cx = add_(mul_(lx, m[0]), add_(mul_(ly, m[1]), mul_(lz, m[2])));
            float cy = add_(mul_(lx, m[3]), add_(mul_(ly, m[4]), mul_(lz, m[5])));
            float cz = add_(mul_(lx, m[6]), add_(mul_(ly, m[7]), mul_(lz, m[8])));
            if (cz > 0.f) {
                if (sub_(fabsf(cx), voxel_radius) < mul_(div_(cz, m[12]), half_resx) && sub_(fabsf(cy), voxel_radius) < mul_(div_(cz, m[13]), half_resy)) { count++; break; }
            }
        }
        grid[i] = count > 0 ? 0.f : -1.f;
    }
}

// generate_grid_samples_nerf_nonuniform.cu:6-42
__global__ void __launch_bounds__(GRID_THREADS) generate_grid_samples_kernel(uint32_t n_elements, Pcg32 rng0, uint32_t step, float lo, float hi, const float *__restrict__ grid,
                                                                             float *__restrict__ positions, int32_t *__restrict__ indices, uint32_t n_cascades, float thresh) {
    const float diag = sub_(hi, lo);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_elements; i += gridDim.x * blockDim.x) {
        Pcg32 rng = rng0; rng.advance((uint64_t)(i * 4u));
        uint32_t level = (uint32_t)mul_(rng.next_float(), (float)n_cascades) % n_cascades;
        uint32_t idx = 0;
        for (uint32_t j = 0; j < 10; ++j) {
            idx = ((i + step * n_elements) * 56924617u + j * 19349663u + 96925573u) % GRID_CELLS;
            idx += level * GRID_CELLS;
            if (__ldg(grid + idx) > thresh) break;
        }
        uint32_t pos_idx = idx % GRID_CELLS;
        float x = (float)morton3D_invert(pos_idx >> 0), y = (float)morton3D_invert(pos_idx >> 1), z = (float)morton3D_invert(pos_idx >> 2);
        float u0 = rng.next_float(), u1 = rng.next_float(), u2 = rng.next_float();
        float s = __uint_as_float((127u + level) << 23);
        float px = add_(mul_(sub_(div_(add_(x, u0), (float)NERF_GRIDSIZE), 0.5f), s), 0.5f);
        float py = add_(mul_(sub_(div_(add_(y, u1), (float)NERF_GRIDSIZE), 0.5f), s), 0.5f);
        float pz = add_(mul_(sub_(div_(add_(z, u2), (float)NERF_GRIDSIZE), 0.5f), s), 0.5f);
        positions[3 * (size_t)i] = div_(sub_(px, lo), diag); positions[3 * (size_t)i + 1] = div_(sub_(py, lo), diag); positions[3 * (size_t)i + 2] = div_(sub_(pz, lo), diag);
        indices[i] = (int32_t)idx;
    }
}

// splat_grid_samples_nerf_max_nearest_neighbor.cu:6-27
__global__ void __launch_bounds__(GRID_THREADS) splat_kernel(uint32_t n, const int32_t *__restrict__ indices, int padded_width, const float *__restrict__ mlp_out,
                                                             float *__restrict__ grid_tmp) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float thickness = mul_(__expf(__ldg(mlp_out + (size_t)i * padded_width)), MIN_CONE_STEPSIZE());
        atomicMax((unsigned int *)&grid_tmp[(uint32_t)indices[i]], __float_as_uint(thickness));
    }
}

// ema_grid_samples_nerf.cu:3-26, float4-vectorised stream
__global__ void __launch_bounds__(GRID_THREADS) ema_kernel(uint32_t n4, float decay, float4 *__restrict__ grid, const float4 *__restrict__ tmp) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
        float4 g = grid[i], t = __ldg(tmp + i);
        g.x = g.x < 0.f ? g.x : fmaxf(mul_(g.x, decay), t.x); g.y = g.y < 0.f ? g.y : fmaxf(mul_(g.y, decay), t.y);
        g.z = g.z < 0.f ? g.z : fmaxf(mul_(g.z, decay), t.z); g.w = g.w < 0.f ? g.w : fmaxf(mul_(g.w, decay), t.w);
        grid[i] = g;
    }
}
__global__ void ema_tail_kernel(uint32_t start, uint32_t n, float decay, float *__restrict__ grid, const float *__restrict__ tmp) {
    uint32_t i = start + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { float p = grid[i]; grid[i] = p < 0.f ? p : fmaxf(mul_(p, decay), tmp[i]); }
}

// update_bitfield.cu:74-116. Mean: the reference sums fmaxf(v,0)/N per element in 1024-thread float4 blocks combined by an
// xor-butterfly, then atomically across its 512 blocks (order undefined). Here: same per-block association, blocks combined in
// index order by a second single-warp kernel => deterministic and equal to the reference run serially.
constexpr int MEAN_BLOCKS = GRID_CELLS / 4096;  // 512
__global__ void __launch_bounds__(1024) grid_mean_partial_kernel(const float4 *__restrict__ grid, float *__restrict__ partial) {
    __shared__ float sdata[32];
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float4 v = __ldg(grid + (size_t)blockIdx.x * 1024 + threadIdx.x);
    const float N = (float)GRID_CELLS;
    float val = add_(add_(add_(div_(fmaxf(v.x, 0.f), N), div_(fmaxf(v.y, 0.f), N)), div_(fmaxf(v.z, 0.f), N)), div_(fmaxf(v.w, 0.f), N));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) val = add_(val, __shfl_xor_sync(0xffffffffu, val, o));
    if (lane == 0) sdata[w] = val;
    __syncthreads();
    if (w == 0) {
        val = sdata[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) val = add_(val, __shfl_xor_sync(0xffffffffu, val, o));
        if (lane == 0) partial[blockIdx.x] = val;
    }
}
__global__ void grid_mean_final_kernel(const float *__restrict__ partial, float *__restrict__ mean) {
    if (threadIdx.x == 0) { float t = 0.f; for (int b = 0; b < MEAN_BLOCKS; ++b) t = add_(t, partial[b]); mean[0] = t; }
}
// 8 cells -> 1 byte over all cascades; each thread builds 4 bytes (one 32-bit store) from 8 float4 loads
__global__ void __launch_bounds__(GRID_THREADS) grid_to_bitfield_kernel(uint32_t n_words, const float4 *__restrict__ grid, uint32_t *__restrict__ bitfield, const float *__restrict__ mean) {
    float m = __ldg(mean);
    float thresh = NERF_MIN_OPTICAL_THICKNESS < m ? NERF_MIN_OPTICAL_THICKNESS : m;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += gridDim.x * blockDim.x) {
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float4 v = __ldg(grid + (size_t)i * 8 + q);
            uint32_t nib = (v.x > thresh ? 1u : 0u) | (v.y > thresh ? 2u : 0u) | (v.z > thresh ? 4u : 0u) | (v.w > thresh ? 8u : 0u);
            word |= nib << (4 * q);
        }
        bitfield[i] = word;
    }
}
// update_bitfield.cu:47-71: one thread per output byte of the next level
__global__ void __launch_bounds__(GRID_THREADS) bitfield_max_pool_kernel(uint32_t n_elements, const uint2 *__restrict__ prev_level, uint8_t *__restrict__ next_level) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_elements) return;
    uint2 p = __ldg(prev_level + i);
    uint8_t bits = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) { bits |= ((p.x >> (8 * j)) & 0xffu) ? (uint8_t)(1u << j) : 0; bits |= ((p.y >> (8 * j)) & 0xffu) ? (uint8_t)(1u << (j + 4)) : 0; }
    uint32_t x = morton3D_invert(i >> 0) + NERF_GRIDSIZE / 8, y = morton3D_invert(i >> 1) + NERF_GRIDSIZE / 8, z = morton3D_invert(i >> 2) + NERF_GRIDSIZE / 8;
    next_level[morton3D(x, y, z)] |= bits;
}

}  // namespace xrb

using namespace xrb;

// ============================================================================ C ABI
extern "C" {

// 2: xrb_ngp_table (cell image), explicit profile events in xrb_ngp_render
// 3: xrb_nerf_mlp_forward takes the fp16 encoding tile image where it took fp32 `embedded` rows, and the K-half weight packing; the other NerfMLP
//    entry points are gone. The symbol name is unchanged but its arguments mean something else, so an old caller must not load this library silently.
int xrb_abi_version(void) { return 5; }
int xrb_built_for_sm(void) { return 90; }
const char *xrb_last_error(void) { return g_err; }

size_t xrb_rm_rays_sampler_workspace(int n_rays) { return march_ws_bytes(n_rays) + 2048 * sizeof(float); }

int xrb_rm_rays_sampler(const float *rays_o, const float *rays_d, const uint8_t *bitfield, const float *metadata, const int32_t *img_ids, const float *xforms,
                        int n_rays, int max_samples, float aabb0, float aabb1, float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls,
                        float *coords_out, int32_t *rays_index, int32_t *numsteps, int32_t *counters, void *workspace, void *stream) {
    (void)metadata; (void)img_ids; (void)xforms;
    XRB_REQUIRE(n_rays >= 0 && max_samples >= 0, "rays_sampler: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(rays_o && rays_d && bitfield && coords_out && rays_index && numsteps && counters && workspace, "rays_sampler: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    MarchWs w = march_ws(workspace, n_rays);
    const int nb = (int)march_n_blocks(n_rays);
    Pcg32 rng = host_rng(seed, n_prior_calls);
    cudaMemsetAsync(w.misc + 3, 0, sizeof(uint32_t), s);   // overflow-chunk counter
    OvfPool pool{w.misc + 3, w.ovf, w.n_chunks, w.chunk_of};
    march_count_kernel<<<nb, MARCH_BLOCK, 0, s>>>(n_rays, rays_o, rays_d, bitfield, aabb0, aabb1, near_distance, cone_angle, rng, w.local_excl, w.startt, w.block_sum, numsteps, w.tbuf, pool);
    march_scan_kernel<<<1, 1024, 0, s>>>(nb, w.block_sum, w.misc, counters);
    march_emit_kernel<<<warp_grid(n_rays), 256, 0, s>>>(n_rays, rays_o, rays_d, bitfield, aabb0, aabb1, cone_angle, (uint32_t)max_samples, w.local_excl, w.startt,
                                                                             w.block_sum, w.misc, w.tbuf, w.chunk_of, w.ovf, coords_out, rays_index, numsteps, counters);
    return check_launch("rays_sampler");
}

size_t xrb_rm_compacted_coord_workspace(int n_rays) {   // the compaction uses only the scan part of the march workspace layout (local_excl, startt, block_sum, misc)
    return sizeof(uint32_t) * ((size_t)n_rays * 2 + march_n_blocks(n_rays) + 16);
}

int xrb_rm_compacted_coord(const float *network_output, const float *coords_in, const int32_t *numsteps, int n_rays, int max_compacted, float *coords_out,
                           int32_t *numsteps_compacted, int32_t *ray_counter, int32_t *step_counter, void *workspace, void *stream) {
    (void)network_output;
    XRB_REQUIRE(n_rays >= 0 && max_compacted >= 0, "compacted_coord: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(coords_in && numsteps && coords_out && numsteps_compacted && ray_counter && step_counter && workspace, "compacted_coord: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    MarchWs w = march_ws(workspace, n_rays);
    const int nb = (int)march_n_blocks(n_rays);
    compact_count_kernel<<<nb, MARCH_BLOCK, 0, s>>>(n_rays, numsteps, w.local_excl, w.block_sum);
    // reuse the scan kernel: "counters" = {ray_counter, step_counter} must be adjacent for it; they are separate tensors in the
    // reference API, so run it on a 2-int staging area in the workspace instead.
    int32_t *stage = (int32_t *)(w.misc + 4);
    cudaMemcpyAsync(stage, ray_counter, sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
    cudaMemcpyAsync(stage + 1, step_counter, sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
    march_scan_kernel<<<1, 1024, 0, s>>>(nb, w.block_sum, w.misc, stage);
    cudaMemcpyAsync(step_counter, stage + 1, sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
    int blocks = (int)(((size_t)n_rays * 32 + 255) / 256);
    compact_copy_kernel<<<blocks, 256, 0, s>>>(n_rays, (uint32_t)max_compacted, coords_in, numsteps, w.local_excl, w.block_sum, w.misc, coords_out, numsteps_compacted, ray_counter);
    return check_launch("compacted_coord");
}

int xrb_ngp_count_trained_rays(const int32_t *numsteps, const int32_t *numsteps_compacted, int n_rays, int64_t *accum, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "count_trained_rays: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(numsteps && numsteps_compacted && accum && ((uintptr_t)accum & 7) == 0, "count_trained_rays: null / misaligned pointer");
    count_trained_kernel<<<stride_grid((n_rays + 255) / 256, 4), 256, 0, (cudaStream_t)stream>>>(n_rays, numsteps, numsteps_compacted, (unsigned long long *)accum);
    return check_launch("count_trained_rays");
}

int xrb_rm_calc_rgb_forward(const float *raw, const float *coords, const int32_t *numsteps, const int32_t *numsteps_compacted, const float *bg, int n_rays, int rgb_act,
                            int dens_act, float *rgb_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "calc_rgb_forward: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(raw && coords && numsteps && numsteps_compacted && bg && rgb_out, "calc_rgb_forward: null pointer");
    XRB_REQUIRE(((uintptr_t)raw & 15) == 0, "calc_rgb_forward: raw must be 16-byte aligned");
    int blocks = warp_grid(n_rays);
    composite_fwd_kernel<0><<<blocks, 256, 0, (cudaStream_t)stream>>>(n_rays, (const float4 *)raw, coords, numsteps, numsteps_compacted, bg, make_float3(0, 0, 0), rgb_act, dens_act,
                                                                      rgb_out, nullptr, CompositeDepth{});
    return check_launch("calc_rgb_forward");
}

int xrb_rm_calc_rgb_forward_geom(const float *raw, const float *coords, const int32_t *numsteps, const int32_t *numsteps_compacted, const float *bg, const float *rays_o,
                                 const float *rays_d, int n_rays, float aabb0, float aabb1, int rgb_act, int dens_act, float *rgb_out, float *alpha_out, float *depth_out,
                                 void *stream) {
    XRB_REQUIRE(n_rays >= 0, "calc_rgb_forward_geom: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(raw && coords && numsteps && numsteps_compacted && bg && rays_o && rays_d && rgb_out && alpha_out && depth_out, "calc_rgb_forward_geom: null pointer");
    XRB_REQUIRE(((uintptr_t)raw & 15) == 0, "calc_rgb_forward_geom: raw must be 16-byte aligned");
    const CompositeDepth dp{rays_o, rays_d, aabb0, aabb1 - aabb0, depth_out, nullptr, nullptr};
    composite_fwd_kernel<4><<<warp_grid(n_rays), 256, 0, (cudaStream_t)stream>>>(n_rays, (const float4 *)raw, coords, numsteps, numsteps_compacted, bg, make_float3(0, 0, 0), rgb_act,
                                                                                 dens_act, rgb_out, alpha_out, dp);
    return check_launch("calc_rgb_forward_geom");
}

int xrb_rm_calc_rgb_backward_geom(const float *raw, const int32_t *numsteps_compacted, const float *coords, const float *grad_rgb, const float *rgb, const float *grid_mean,
                                  const float *rays_o, const float *rays_d, float aabb0, float aabb1, const float *depth, const float *alpha, const float *grad_depth,
                                  const float *grad_alpha, int n_rays, int rgb_act, int dens_act, float *dl_draw, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "calc_rgb_backward_geom: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(raw && coords && numsteps_compacted && grad_rgb && rgb && grid_mean && rays_o && rays_d && depth && alpha && dl_draw, "calc_rgb_backward_geom: null pointer");
    XRB_REQUIRE(((uintptr_t)raw & 15) == 0 && ((uintptr_t)dl_draw & 15) == 0, "calc_rgb_backward_geom: raw/dl_draw must be 16-byte aligned");
    const CompositeGeom gm{rays_o, rays_d, aabb0, aabb1 - aabb0, depth, alpha, grad_depth, grad_alpha};
    composite_bwd_kernel<true><<<warp_grid(n_rays), 256, 0, (cudaStream_t)stream>>>(n_rays, (const float4 *)raw, coords, numsteps_compacted, grad_rgb, rgb, grid_mean, rgb_act,
                                                                                    dens_act, (float4 *)dl_draw, gm);
    return check_launch("calc_rgb_backward_geom");
}

int xrb_rm_calc_rgb_backward(const float *raw, const int32_t *numsteps_compacted, const float *coords, const float *grad_rgb, const float *rgb, const float *grid_mean,
                             int n_rays, int rgb_act, int dens_act, float *dl_draw, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "calc_rgb_backward: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(raw && coords && numsteps_compacted && grad_rgb && rgb && grid_mean && dl_draw, "calc_rgb_backward: null pointer");
    XRB_REQUIRE(((uintptr_t)raw & 15) == 0 && ((uintptr_t)dl_draw & 15) == 0, "calc_rgb_backward: raw/dl_draw must be 16-byte aligned");
    int blocks = warp_grid(n_rays);
    composite_bwd_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(n_rays, (const float4 *)raw, coords, numsteps_compacted, grad_rgb, rgb, grid_mean, rgb_act, dens_act,
                                                                   (float4 *)dl_draw, CompositeGeom{});
    return check_launch("calc_rgb_backward");
}

int xrb_ngp_ray_grad(const float *d_rows, const float *coords, const int32_t *numsteps_compacted, const float *rays_o, const float *rays_d, int n_rays, float aabb0, float aabb1,
                     float scale, float *grad_o, float *grad_d, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "ngp_ray_grad: negative size");
    XRB_REQUIRE(aabb1 > aabb0, "ngp_ray_grad: need aabb0 < aabb1");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(d_rows && coords && numsteps_compacted && rays_o && rays_d && grad_o && grad_d, "ngp_ray_grad: null pointer");
    ray_grad_kernel<<<warp_grid(n_rays), 256, 0, (cudaStream_t)stream>>>(n_rays, d_rows, coords, numsteps_compacted, rays_o, rays_d, aabb0, aabb1 - aabb0, scale, grad_o, grad_d);
    return check_launch("ngp_ray_grad");
}

int xrb_rm_calc_rgb_inference(const float *raw, const float *coords, const int32_t *numsteps, const float *bg3_host, int n_rays, int rgb_act, int dens_act, float *rgb_out,
                              float *alpha_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "calc_rgb_inference: negative size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(raw && coords && numsteps && bg3_host && rgb_out && alpha_out, "calc_rgb_inference: null pointer");
    XRB_REQUIRE(((uintptr_t)raw & 15) == 0, "calc_rgb_inference: raw must be 16-byte aligned");
    int blocks = warp_grid(n_rays);
    composite_fwd_kernel<1><<<blocks, 256, 0, (cudaStream_t)stream>>>(n_rays, (const float4 *)raw, coords, numsteps, nullptr, nullptr,
                                                                      make_float3(bg3_host[0], bg3_host[1], bg3_host[2]), rgb_act, dens_act, rgb_out, alpha_out,
                                                                      CompositeDepth{});
    return check_launch("calc_rgb_inference");
}

int xrb_rm_mark_untrained_density_grid(const float *focal, const float *xforms, int n_elements, int n_images, int res0, int res1, float *grid, void *stream) {
    XRB_REQUIRE(n_elements >= 0 && n_images >= 0, "mark_untrained: negative size");
    if (n_elements == 0) return XRB_OK;
    XRB_REQUIRE(focal && xforms && grid, "mark_untrained: null pointer");
    size_t smem = (size_t)n_images * 14 * sizeof(float);
    XRB_REQUIRE(smem <= 200 * 1024, "mark_untrained: too many images for one shared-memory camera table (max 3657)");
    if (smem > 48 * 1024) cudaFuncSetAttribute(mark_untrained_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    mark_untrained_kernel<<<stream_grid(n_elements), GRID_THREADS, smem, (cudaStream_t)stream>>>((uint32_t)n_elements, grid, (uint32_t)n_images, (const float2 *)focal, xforms, res0, res1);
    return check_launch("mark_untrained");
}

int xrb_rm_generate_grid_samples(const float *grid, int ema_step, int n_elements, int max_cascade, float thresh, float aabb0, float aabb1, uint64_t seed, int64_t n_prior_calls,
                                 float *positions, int32_t *indices, void *stream) {
    XRB_REQUIRE(n_elements >= 0 && max_cascade >= 0 && max_cascade < (int)NERF_CASCADES, "generate_grid_samples: bad size/cascade");
    if (n_elements == 0) return XRB_OK;
    XRB_REQUIRE(grid && positions && indices, "generate_grid_samples: null pointer");
    Pcg32 rng = host_rng(seed, n_prior_calls);
    generate_grid_samples_kernel<<<stream_grid(n_elements), GRID_THREADS, 0, (cudaStream_t)stream>>>((uint32_t)n_elements, rng, (uint32_t)ema_step, aabb0, aabb1, grid, positions, indices,
                                                                                                     (uint32_t)max_cascade + 1, thresh);
    return check_launch("generate_grid_samples");
}

int xrb_rm_splat_grid_samples(const float *mlp_out, const int32_t *indices, int padded_width, int n, float *grid_tmp, void *stream) {
    XRB_REQUIRE(n >= 0 && padded_width >= 1, "splat: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(mlp_out && indices && grid_tmp, "splat: null pointer");
    splat_kernel<<<stream_grid(n), GRID_THREADS, 0, (cudaStream_t)stream>>>((uint32_t)n, indices, padded_width, mlp_out, grid_tmp);
    return check_launch("splat");
}

int xrb_rm_ema_grid_samples(const float *grid_tmp, int n_elements, float decay, float *grid, void *stream) {
    XRB_REQUIRE(n_elements >= 0, "ema: negative size");
    if (n_elements == 0) return XRB_OK;
    XRB_REQUIRE(grid_tmp && grid, "ema: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    bool aligned = (((uintptr_t)grid | (uintptr_t)grid_tmp) & 15) == 0;
    uint32_t n4 = aligned ? (uint32_t)n_elements / 4 : 0;
    if (n4) ema_kernel<<<stream_grid(n4), GRID_THREADS, 0, s>>>(n4, decay, (float4 *)grid, (const float4 *)grid_tmp);
    uint32_t rest = (uint32_t)n_elements - n4 * 4;
    if (rest) ema_tail_kernel<<<(rest + 255) / 256, 256, 0, s>>>(n4 * 4, (uint32_t)n_elements, decay, grid, grid_tmp);
    return check_launch("ema");
}

size_t xrb_rm_update_bitfield_workspace(void) { return MEAN_BLOCKS * sizeof(float); }

int xrb_rm_update_bitfield(const float *grid, float *mean, uint8_t *bitfield, void *workspace, void *stream) {
    XRB_REQUIRE(grid && mean && bitfield && workspace, "update_bitfield: null pointer");
    XRB_REQUIRE(((uintptr_t)grid & 15) == 0 && ((uintptr_t)bitfield & 7) == 0 && ((uintptr_t)workspace & 3) == 0, "update_bitfield: grid must be 16-byte, bitfield 8-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    // the per-block partial sums of the fixed-order mean live in caller-owned scratch: no allocation inside the call (CUDA-graph capturable),
    // nothing shared between streams or host threads
    float *partial = (float *)workspace;
    grid_mean_partial_kernel<<<MEAN_BLOCKS, 1024, 0, s>>>((const float4 *)grid, partial);
    grid_mean_final_kernel<<<1, 32, 0, s>>>(partial, mean);
    uint32_t n_words = GRID_CELLS / 8 * NERF_CASCADES / 4;
    grid_to_bitfield_kernel<<<stream_grid(n_words), GRID_THREADS, 0, s>>>(n_words, (const float4 *)grid, (uint32_t *)bitfield, mean);
    for (uint32_t level = 1; level < NERF_CASCADES; ++level) {
        uint32_t n = GRID_CELLS / 64;
        bitfield_max_pool_kernel<<<(n + GRID_THREADS - 1) / GRID_THREADS, GRID_THREADS, 0, s>>>(n, (const uint2 *)(bitfield + (size_t)GRID_CELLS * (level - 1) / 8), bitfield + (size_t)GRID_CELLS * level / 8);
    }
    return check_launch("update_bitfield");
}

}  // extern "C"
