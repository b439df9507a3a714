// xrnerf_b200 — render of a ray batch through the Instant-NGP path (inference):
//   march (count -> scan -> emit)  ->  sample order (key + histogram -> scan -> scatter)  ->  field (hash encode + MLPs on wgmma tiles)  ->  composite (warp per ray)
// replacing ngp_grid_sampler.py:205-228 + hashnerf_mlp.py:55-79 + hashnerf_render.py:42-46 of the reference with ZERO host
// synchronisations: the sample count stays on the device (the ordering kernels and the field kernel read it from `counters[1]`).
// The stages are separate launches chained on one stream (CUDA-graph capturable); the single-launch variant is tracked in DESIGN.md §6.
#include "ngp_field.cuh"

namespace xrb {

// ---------------------------------------------------------------------------- sample order
// The march writes rows in ray order, so a 128-sample field tile holds ~12 unrelated rays and at the fine hash levels every lane reads its own
// L2 sectors. The field's output row depends on that row's inputs alone (independent wgmma rows, fixed K order), so the rows are evaluated
// bucketed by position instead: a counting sort on the Morton index of a 64^3 grid over the warped unit cube. Neighbouring lanes then share
// cells and sectors, and every output stays bit-identical. The order inside a bucket varies from run to run; the outputs do not depend on it.
constexpr int ORDER_BITS = 6;                                          // per axis (DESIGN.md §4.1 has the 6 vs 7 bit measurement)
constexpr uint32_t ORDER_BUCKETS = 1u << (3 * ORDER_BITS);             // 2^18: a 1 MB histogram
constexpr int ORDER_THREADS = 256;
constexpr uint32_t ORDER_CHUNK = ORDER_THREADS * 4;                    // buckets per scan block (one uint4 per thread)
constexpr int ORDER_SCAN_BLOCKS = (int)(ORDER_BUCKETS / ORDER_CHUNK);  // 256
constexpr uint32_t NO_KEY = ~0u;

// bucket of a sample: its warped position (the field's input) on the 64^3 grid; NaN-safe clamp, since rows past the first overflowed ray are
// never written by the march and hold stale memory
__device__ __forceinline__ uint32_t order_key(const float *__restrict__ c) {
    constexpr float S = (float)(1 << ORDER_BITS), HI = (float)((1 << ORDER_BITS) - 1);
    const uint32_t x = (uint32_t)fminf(fmaxf(c[0] * S, 0.f), HI), y = (uint32_t)fminf(fmaxf(c[1] * S, 0.f), HI), z = (uint32_t)fminf(fmaxf(c[2] * S, 0.f), HI);
    return morton3D(x, y, z);
}
// rows to order: none above SAMPLE_ORDER_MAX_ROWS, where the field ignores the order (ngp_field.cuh)
__device__ __forceinline__ uint32_t order_rows(uint32_t max_samples, const int32_t *__restrict__ n_dev) {
    const uint32_t n = min(max_samples, (uint32_t)max(__ldg(n_dev), 0));
    return n <= SAMPLE_ORDER_MAX_ROWS ? n : 0u;
}

// key of every row + bucket counts. Consecutive samples of a ray mostly share a bucket: one atomic per distinct key of a warp.
__global__ void __launch_bounds__(ORDER_THREADS) order_key_kernel(const float *__restrict__ coords, uint32_t max_samples, const int32_t *__restrict__ n_dev,
                                                                  uint32_t *__restrict__ key, uint32_t *__restrict__ count) {
    const uint32_t n = order_rows(max_samples, n_dev), lane = threadIdx.x & 31;
    for (uint32_t j0 = (blockIdx.x * ORDER_THREADS + threadIdx.x) & ~31u; j0 < n; j0 += gridDim.x * ORDER_THREADS) {   // warp-uniform trip count
        const uint32_t j = j0 + lane;
        const uint32_t k = j < n ? order_key(coords + 7 * (size_t)j) : NO_KEY;
        if (j < n) key[j] = k;
        const uint32_t peers = __match_any_sync(0xffffffffu, k);
        if (k != NO_KEY && lane == (uint32_t)__ffs(peers) - 1) atomicAdd(count + k, (uint32_t)__popc(peers));
    }
}

// exclusive scan of one value per thread over the block; *total = the block's sum
__device__ __forceinline__ uint32_t order_block_excl_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t warp_tot[ORDER_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t incl = warp_incl_scan_u32(v, lane);
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    uint32_t off = 0, tot = 0;
#pragma unroll
    for (int k = 0; k < ORDER_THREADS / 32; ++k) { const uint32_t s = warp_tot[k]; if (k < w) off += s; tot += s; }
    __syncthreads();   // warp_tot may be reused by the next call
    *total = tot;
    return off + incl - v;
}

// total of each chunk of ORDER_CHUNK buckets
__global__ void __launch_bounds__(ORDER_THREADS) order_chunk_sum_kernel(const uint4 *__restrict__ count, uint32_t *__restrict__ chunk_sum) {
    const uint4 v = count[blockIdx.x * ORDER_THREADS + threadIdx.x];
    uint32_t tot;
    order_block_excl_scan(v.x + v.y + v.z + v.w, &tot);
    if (threadIdx.x == 0) chunk_sum[blockIdx.x] = tot;
}

// counts -> exclusive bucket offsets, in place (block b: its chunk, offset by the totals of chunks [0, b))
__global__ void __launch_bounds__(ORDER_THREADS) order_scan_kernel(uint4 *__restrict__ count, const uint32_t *__restrict__ chunk_sum) {
    uint32_t base = 0, tot;
    for (uint32_t t = threadIdx.x; t < blockIdx.x; t += ORDER_THREADS) base += chunk_sum[t];
    order_block_excl_scan(base, &base);
    uint4 v = count[blockIdx.x * ORDER_THREADS + threadIdx.x];
    uint32_t o = base + order_block_excl_scan(v.x + v.y + v.z + v.w, &tot);
    uint4 r;
    r.x = o; o += v.x; r.y = o; o += v.y; r.z = o; o += v.z; r.w = o;
    count[blockIdx.x * ORDER_THREADS + threadIdx.x] = r;
}

// order[cursor[key]++] = row, one atomic per distinct key of a warp
__global__ void __launch_bounds__(ORDER_THREADS) order_scatter_kernel(const uint32_t *__restrict__ key, uint32_t max_samples, const int32_t *__restrict__ n_dev,
                                                                      uint32_t *__restrict__ cursor, uint32_t *__restrict__ order) {
    const uint32_t n = order_rows(max_samples, n_dev), lane = threadIdx.x & 31;
    for (uint32_t j0 = (blockIdx.x * ORDER_THREADS + threadIdx.x) & ~31u; j0 < n; j0 += gridDim.x * ORDER_THREADS) {
        const uint32_t j = j0 + lane;
        const uint32_t k = j < n ? key[j] : NO_KEY;
        const uint32_t peers = __match_any_sync(0xffffffffu, k), leader = (uint32_t)__ffs(peers) - 1;
        uint32_t base = 0;
        if (k != NO_KEY && lane == leader) base = atomicAdd(cursor + k, (uint32_t)__popc(peers));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (k != NO_KEY) order[base + __popc(peers & ((1u << lane) - 1u))] = j;
    }
}

struct RenderWs {   // xrb_ngp_render's workspace (layout documented in include/xrnerf_b200.h)
    void *march; float *coords, *raw; uint32_t *order; int32_t *rays_index; uint32_t *count, *chunk_sum;
};
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static RenderWs render_ws(void *ws, int n_rays, int max_samples, size_t *bytes) {
    RenderWs w;
    uint8_t *p = (uint8_t *)ws;
    size_t a = align256(xrb_rm_rays_sampler_workspace(n_rays));
    w.march = p;
    w.coords = (float *)(p + a);
    w.raw = w.coords + (size_t)max_samples * 7;
    w.order = (uint32_t *)(w.raw + (size_t)max_samples * 4);
    a += align256((size_t)max_samples * (7 + 4 + 1) * sizeof(float));
    w.count = (uint32_t *)(p + a); a += ORDER_BUCKETS * sizeof(uint32_t);
    w.chunk_sum = (uint32_t *)(p + a); a += ORDER_SCAN_BLOCKS * sizeof(uint32_t);
    w.rays_index = (int32_t *)(p + a); a += (size_t)n_rays * sizeof(int32_t);
    if (bytes) *bytes = a;
    return w;
}

// order[0, n) = a permutation of the rows [0, n), n = min(*n_dev, max_samples), bucketed by position (nothing is written when n > SAMPLE_ORDER_MAX_ROWS).
// `key` (max_samples words) is scratch.
static void launch_sample_order(const float *coords, int max_samples, const int32_t *n_dev, uint32_t *key, uint32_t *count, uint32_t *chunk_sum, uint32_t *order, cudaStream_t s) {
    size_t b = ((size_t)max_samples + ORDER_THREADS - 1) / ORDER_THREADS, cap = (size_t)NUM_SMS * 8;
    const int grid = (int)(b < cap ? b : cap);
    cudaMemsetAsync(count, 0, ORDER_BUCKETS * sizeof(uint32_t), s);
    order_key_kernel<<<grid, ORDER_THREADS, 0, s>>>(coords, (uint32_t)max_samples, n_dev, key, count);
    order_chunk_sum_kernel<<<ORDER_SCAN_BLOCKS, ORDER_THREADS, 0, s>>>((const uint4 *)count, chunk_sum);
    order_scan_kernel<<<ORDER_SCAN_BLOCKS, ORDER_THREADS, 0, s>>>((uint4 *)count, chunk_sum);
    order_scatter_kernel<<<grid, ORDER_THREADS, 0, s>>>(key, (uint32_t)max_samples, n_dev, count, order);
}

}  // namespace xrb

extern "C" {

size_t xrb_ngp_render_workspace(int n_rays, int max_samples) {
    size_t bytes = 0;
    xrb::render_ws(nullptr, n_rays, max_samples, &bytes);
    return bytes + 256;
}

int xrb_ngp_render(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield, const float *rays_o, const float *rays_d, int n_rays,
                   int max_samples, float aabb0, float aabb1, float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act,
                   int dens_act, float *rgb_out, float *alpha_out, int32_t *numsteps, int32_t *counters, void *workspace, void *ev_before_field, void *ev_after_field, void *stream) {
    int e = xrb::check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n_rays >= 0 && max_samples > 0, "ngp_render: bad size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(table && weight_image && bitfield && rays_o && rays_d && bg3_host && rgb_out && alpha_out && numsteps && counters && workspace, "ngp_render: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const xrb::RenderWs w = xrb::render_ws(workspace, n_rays, max_samples, nullptr);
    cudaMemsetAsync(counters, 0, 2 * sizeof(int32_t), s);
    e = xrb_rm_rays_sampler(rays_o, rays_d, bitfield, nullptr, nullptr, nullptr, n_rays, max_samples, aabb0, aabb1, near_distance, cone_angle, seed, n_prior_calls, w.coords, w.rays_index,
                            numsteps, counters, w.march, stream);
    if (e) return e;
    // counters[1] counts overflowed rays too; rows beyond max_samples do not exist, the ordering kernels and launch_field clamp to max_samples
    // measurement hook: events recorded right before the sample order / after the field kernel let a caller time them inside its own timed region
    if (ev_before_field) cudaEventRecord((cudaEvent_t)ev_before_field, s);
    // the keys live in `raw` until the field kernel overwrites it with its outputs
    xrb::launch_sample_order(w.coords, max_samples, counters + 1, (uint32_t *)w.raw, w.count, w.chunk_sum, w.order, s);
    e = xrb::launch_field(cfg, table, nullptr, nullptr, weight_image, w.coords, 7, w.coords + 4, 7, max_samples, counters + 1, w.order, w.raw, 1, false, s);
    if (ev_after_field) cudaEventRecord((cudaEvent_t)ev_after_field, s);
    if (e) return e;
    return xrb_rm_calc_rgb_inference(w.raw, w.coords, numsteps, bg3_host, n_rays, rgb_act, dens_act, rgb_out, alpha_out, stream);
}

}  // extern "C"
