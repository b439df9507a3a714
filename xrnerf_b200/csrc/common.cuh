// xrnerf_b200 — shared device helpers (sm_90a only).
//
// Index-path arithmetic is written with explicit round-to-nearest intrinsics (__fmul_rn/__fadd_rn/__fdiv_rn):
// nvcc never contracts those into FMAs, which makes the per-ray sample sets bit-reproducible against the
// un-contracted IEEE fp32 semantics of the reference's C++ source (SURVEY §8c). Reference citations are
// relative to /root/reference/extensions/ngp_raymarch/.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <float.h>
#include "../../include/xrnerf_b200.h"

namespace xrb {

constexpr uint32_t NERF_STEPS = 1024u;      // raymarch_shared.h:42
constexpr uint32_t NERF_CASCADES = 8u;      // :43
constexpr uint32_t NERF_GRIDSIZE = 128u;    // :48
constexpr uint32_t GRID_CELLS = 128u * 128u * 128u;
constexpr float NERF_MIN_OPTICAL_THICKNESS = 0.01f;  // :56
constexpr int NUM_SMS = 132;   // H100 SXM: the default of launches that query the device, and the cap of some grid-stride launches

// constants folded exactly as the reference's constexpr chain folds them (fp32, left to right)
__host__ __device__ constexpr float SQRT3() { return 1.73205080757f; }
__host__ __device__ constexpr float MIN_CONE_STEPSIZE() { return SQRT3() / NERF_STEPS; }
__host__ __device__ constexpr float MAX_CONE_STEPSIZE() { return (SQRT3() / NERF_STEPS) * (1 << (NERF_CASCADES - 1)) * NERF_STEPS / NERF_GRIDSIZE; }

void set_error(const char *msg);
int check_launch(const char *what);

#define XRB_REQUIRE(cond, msg)                                   \
    do {                                                         \
        if (!(cond)) { xrb::set_error(msg); return XRB_E_BADARG; } \
    } while (0)

// ---------------------------------------------------------------- persistent launches (host)
// SM count of the current device; a failed query clears the sticky error and falls back to NUM_SMS
inline int sm_count() {
    int dev = 0, sms = NUM_SMS;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) { cudaGetLastError(); sms = NUM_SMS; }
    return sms;
}
// grid of a persistent kernel that keeps per_sm CTAs resident on every SM: never more CTAs than there is work, never fewer than one
inline int persistent_grid(int per_sm, int64_t work_ctas) {
    const int64_t g = (int64_t)sm_count() * per_sm;
    return (int)(work_ctas < g ? (work_ctas > 0 ? work_ctas : 1) : g);
}
// the same with per_sm taken from the occupancy calculator, but at least min_per_sm
inline int persistent_grid(const void *kernel, int block, size_t smem, int64_t work_ctas, int min_per_sm = 1) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem) != cudaSuccess) cudaGetLastError();
    if (per_sm < min_per_sm) per_sm = min_per_sm;  // the calculator has been seen to under-report; extra CTAs simply queue
    return persistent_grid(per_sm, work_ctas);
}
// grid of a grid-stride launch: the blocks the work needs, at most per_sm blocks on each of NUM_SMS SMs, never fewer than one
inline int stride_grid(int64_t blocks, int per_sm) {
    const int64_t cap = (int64_t)NUM_SMS * per_sm;
    return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// ---------------------------------------------------------------- pcg32 (include/op_include/pcg32/pcg32.h:41-165)
struct Pcg32 {
    uint64_t state, inc;
    __host__ __device__ uint32_t next_uint() {
        uint64_t old = state;
        state = old * 0x5851f42d4c957f2dULL + inc;
        uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
        uint32_t rot = (uint32_t)(old >> 59u);
        return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
    }
    __host__ __device__ void seed(uint64_t initstate, uint64_t initseq) {
        state = 0; inc = (initseq << 1u) | 1u; next_uint(); state += initstate; next_uint();
    }
    __host__ __device__ float next_float() {
#ifdef __CUDA_ARCH__
        return __fadd_rn(__uint_as_float((next_uint() >> 9) | 0x3f800000u), -1.0f);
#else
        union { uint32_t u; float f; } x; x.u = (next_uint() >> 9) | 0x3f800000u; return x.f - 1.0f;
#endif
    }
    __host__ __device__ void advance(uint64_t delta) {
        uint64_t cur_mult = 0x5851f42d4c957f2dULL, cur_plus = inc, acc_mult = 1u, acc_plus = 0u;
        while (delta > 0) {
            if (delta & 1) { acc_mult *= cur_mult; acc_plus = acc_plus * cur_mult + cur_plus; }
            cur_plus = (cur_mult + 1) * cur_plus; cur_mult *= cur_mult; delta /= 2;
        }
        state = acc_mult * state + acc_plus;
    }
};
// host rng of one reference translation unit after n_prior_calls API calls (raymarch_shared.h:38, ray_sampler.cu:198)
inline Pcg32 host_rng(uint64_t seed, int64_t n_prior_calls) {
    Pcg32 r; r.seed(seed, 1u);
    r.advance((uint64_t)n_prior_calls << 32);   // k calls of advance(2^32) == one jump of k*2^32 (mod 2^64): O(64) on the host instead of O(64 k)
    return r;
}

// ---------------------------------------------------------------- Morton (raymarch_shared.h:122-131, :753-768)
__host__ __device__ __forceinline__ uint32_t expand_bits(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu; v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u; v = (v * 0x00000005u) & 0x49249249u; return v;
}
__host__ __device__ __forceinline__ uint32_t morton3D(uint32_t x, uint32_t y, uint32_t z) { return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2); }
__host__ __device__ __forceinline__ uint32_t morton3D_invert(uint32_t x) {
    x = x & 0x49249249; x = (x | (x >> 2)) & 0xc30c30c3; x = (x | (x >> 4)) & 0x0f00f00f;
    x = (x | (x >> 8)) & 0xff0000ff; x = (x | (x >> 16)) & 0x0000ffff; return x;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------- exact-rounding helpers
__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float clampf(float v, float lo, float hi) { return v < lo ? lo : (hi < v ? hi : v); }  // raymarch_shared.h:104-107
__device__ __forceinline__ float calc_dt(float t, float cone) { return clampf(mul_(t, cone), MIN_CONE_STEPSIZE(), MAX_CONE_STEPSIZE()); }  // ray_sampler_header.h:24-25

// floor() of |p| < 2^22 and its integer value on the FMA/ALU pipes (F2I / FRND / I2F run on the quarter-rate XU pipe):
// t = p + 1.5*2^23 rounds p to the nearest integer into the low mantissa bits; one compare turns round-to-nearest into floor. Exact.
__device__ __forceinline__ float floor_small(float p, int *ip) {
    float t = __fadd_rn(p, 12582912.0f);
    float r = __fadd_rn(t, -12582912.0f);
    int i = __float_as_int(t) - 0x4B400000;
    if (r > p) { r = __fadd_rn(r, -1.0f); i -= 1; }
    *ip = i;
    return r;
}
// expand_bits() of raymarch_shared.h:753-760 for 7-bit inputs via the identity spread3(v) = sum of bit b moved to 3b: same value, 2 steps
__device__ __forceinline__ uint32_t expand_bits7(uint32_t v) {
    v = (v | (v << 8)) & 0x0000F00Fu;   // bits 0-3 stay, bits 4-6 -> 12-14
    v = (v | (v << 4)) & 0x000C30C3u;   // pairs apart
    v = (v | (v << 2)) & 0x00249249u;   // every third bit
    return v;
}

// frexpf exponent for finite positive normal/zero inputs (the only ones the march produces); matches frexpf incl. 0 -> 0
__device__ __forceinline__ int frexp_exponent(float v) {
    // v >= 0 finite. Normal numbers: biased exponent - 126 (frexpf's convention 0.5 <= m < 1); zero -> 0; denormals take libm.
    uint32_t e = __float_as_uint(v) >> 23;
    if (e != 0) return (int)e - 126;
    if (v == 0.f) return 0;
    int r; frexpf(v, &r); return r;
}
// frexpf exponent e of m: m in [2^(e-1), 2^e). The march only needs clamp(e + 1, 0, 7):
//   m >= 0.25 (a normal number): e = biased exponent - 126 >= -1;   0 < m < 0.25 (incl. denormals): e <= -2 -> 0;   m == 0: frexpf yields e = 0 -> 1
__device__ __forceinline__ int mip_from_pos(float px, float py, float pz) {  // ray_sampler_header.h:37-43
    float m = fmaxf(fabsf(sub_(px, 0.5f)), fmaxf(fabsf(sub_(py, 0.5f)), fabsf(sub_(pz, 0.5f))));
    if (m >= 0.25f) return min((int)NERF_CASCADES - 1, (int)(__float_as_uint(m) >> 23) - 125);
    return m == 0.f ? 1 : 0;
}
__device__ __forceinline__ int mip_from_dt(float dt, float px, float py, float pz) {  // ray_sampler_header.h:45-54
    int mip = mip_from_pos(px, py, pz);
    dt = mul_(dt, (float)(2 * NERF_GRIDSIZE));
    if (dt < 1.f) return mip;
    int e = (int)(__float_as_uint(dt) >> 23) - 126;   // dt >= 1: a normal number, frexpf exponent = biased exponent - 126
    return min((int)NERF_CASCADES - 1, max(e, mip));
}
// expand_bits() of a 7-bit cell coordinate through a 128-entry shared-memory table (3 LDS + 2 LEA instead of ~27 ALU ops per tested position)
__device__ __forceinline__ void morton_lut_init(uint32_t *lut, int tid, int nthreads) {
    for (int v = tid; v < 128; v += nthreads) lut[v] = expand_bits7((uint32_t)v);
}
__device__ __forceinline__ uint32_t cascaded_grid_idx_at(float px, float py, float pz, uint32_t mip, const uint32_t *lut = nullptr) {  // ray_sampler_header.h:298-313
    float s = __uint_as_float((127u - mip) << 23);  // scalbnf(1, -mip), exact
    float q[3] = {px, py, pz}; uint32_t c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float v = add_(mul_(sub_(q[k], 0.5f), s), 0.5f);
        // the reference truncates toward zero (cast<int>) then clamps to [0,127]; floor differs from trunc only for negative values,
        // which both clamp to 0 -> identical cell. floor_small keeps this off the XU pipe.
        int i; floor_small(mul_(v, (float)NERF_GRIDSIZE), &i);
        c[k] = (uint32_t)min(max(i, 0), (int)NERF_GRIDSIZE - 1);
    }
    if (lut) return lut[c[0]] + (lut[c[1]] << 1) + (lut[c[2]] << 2);   // disjoint bit sets: + == |
    return expand_bits7(c[0]) | (expand_bits7(c[1]) << 1) | (expand_bits7(c[2]) << 2);
}
__device__ __forceinline__ bool occupied_at(float px, float py, float pz, const uint8_t *__restrict__ bitfield, uint32_t mip, const uint32_t *lut = nullptr) {  // :315-319
    uint32_t idx = cascaded_grid_idx_at(px, py, pz, mip, lut);
    return __ldg(bitfield + (idx >> 3) + ((GRID_CELLS * mip) >> 3)) & (1u << (idx & 7u));
}
__device__ __forceinline__ float signf_(float x) { return copysignf(1.0f, x); }
__device__ __forceinline__ float distance_to_next_voxel(const float p[3], const float d[3], const float idir[3], uint32_t res) {  // :271-280
    float t3[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float pr = mul_((float)res, p[k]);
        int unused; float fl = floor_small(add_(add_(pr, 0.5f), mul_(0.5f, signf_(d[k]))), &unused);   // == floorf, |arg| < 2^22
        t3[k] = mul_(sub_(fl, pr), idir[k]);
    }
    float t = fminf(fminf(t3[0], t3[1]), t3[2]);
    return fmaxf(mul_(t, __uint_as_float((254u - (__float_as_uint((float)res) >> 23)) << 23)), 0.0f);  // t / res, res = 2^k: exact reciprocal, same bits as the division
}
__device__ __forceinline__ float advance_to_next_voxel(float t, float cone, const float p[3], const float d[3], const float idir[3], uint32_t res) {  // :282-296
    float t_target = add_(t, distance_to_next_voxel(p, d, idir, res));
    do { t = add_(t, calc_dt(t, cone)); } while (t < t_target);
    return t;
}
// BoundingBox::ray_intersect (raymarch_shared.h:506-563): returns tmin (FLT_MAX on a miss)
__device__ __forceinline__ float aabb_ray_tmin(float lo, float hi, const float o[3], const float d[3]) {
    float tmin = div_(sub_(lo, o[0]), d[0]), tmax = div_(sub_(hi, o[0]), d[0]);
    if (tmin > tmax) { float c = tmin; tmin = tmax; tmax = c; }
    float tymin = div_(sub_(lo, o[1]), d[1]), tymax = div_(sub_(hi, o[1]), d[1]);
    if (tymin > tymax) { float c = tymin; tymin = tymax; tymax = c; }
    if (tmin > tymax || tymin > tmax) return FLT_MAX;
    if (tymin > tmin) tmin = tymin;
    if (tymax < tmax) tmax = tymax;
    float tzmin = div_(sub_(lo, o[2]), d[2]), tzmax = div_(sub_(hi, o[2]), d[2]);
    if (tzmin > tzmax) { float c = tzmin; tzmin = tzmax; tzmax = c; }
    if (tmin > tzmax || tzmin > tmax) return FLT_MAX;
    if (tzmin > tmin) tmin = tzmin;
    return tmin;
}
__device__ __forceinline__ bool aabb_contains(float lo, float hi, float x, float y, float z) {  // raymarch_shared.h:570-575
    return x >= lo && x <= hi && y >= lo && y <= hi && z >= lo && z <= hi;
}
__device__ __forceinline__ float warp_dt(float dt) {  // raymarch_shared.h:110-114
    const float max_stepsize = MIN_CONE_STEPSIZE() * (1 << (NERF_CASCADES - 1));
    return div_(sub_(dt, MIN_CONE_STEPSIZE()), max_stepsize - MIN_CONE_STEPSIZE());
}
__device__ __forceinline__ float unwarp_dt(float dt) {  // ray_sampler_header.h:388-392
    const float max_stepsize = MIN_CONE_STEPSIZE() * (1 << (NERF_CASCADES - 1));
    return add_(mul_(dt, max_stepsize - MIN_CONE_STEPSIZE()), MIN_CONE_STEPSIZE());
}

// ---------------------------------------------------------------- sample row coords[S, ROW_FLOATS] (ray_sampler.cu:99-115)
// warped position (0..2), warped dt (ROW_DT), warped direction (ROW_DIR..ROW_DIR+2) of the sample at t on ray (o, d); diag = hi - lo
constexpr int ROW_FLOATS = 7, ROW_DT = 3, ROW_DIR = 4;
__device__ __forceinline__ void sample_warped_pos(const float o[3], const float d[3], float t, float lo, float diag, float x[3]) {  // warp_position
#pragma unroll
    for (int k = 0; k < 3; ++k) x[k] = div_(sub_(add_(o[k], mul_(t, d[k])), lo), diag);
}
__device__ __forceinline__ void sample_warped_dir(const float d[3], float w[3]) {  // warp_direction
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = mul_(add_(d[k], 1.0f), 0.5f);
}
// one float at a time, in row order
__device__ __forceinline__ void write_sample_row(float *c, const float o[3], const float d[3], float t, float cone, float lo, float diag) {
    float x[3], w[3];
    sample_warped_pos(o, d, t, lo, diag, x);
    sample_warped_dir(d, w);
    c[0] = x[0]; c[1] = x[1]; c[2] = x[2];
    c[ROW_DT] = warp_dt(calc_dt(t, cone));
    c[ROW_DIR] = w[0]; c[ROW_DIR + 1] = w[1]; c[ROW_DIR + 2] = w[2];
}
// the dt the composite reads back from a row, and the same value for the sample at t without a row in memory
__device__ __forceinline__ float row_dt(const float *c) { return unwarp_dt(__ldg(c + ROW_DT)); }
__device__ __forceinline__ float sample_row_dt(float t, float cone) { return unwarp_dt(warp_dt(calc_dt(t, cone))); }
// t of a row rebuilt from its warped position: the projection of (position - o) onto d, inv_dd = 1 / |d|^2
__device__ __forceinline__ float row_t(const float *c, const float o[3], const float d[3], float inv_dd, float lo, float diag) {
    const float p0 = lo + __ldg(c) * diag - o[0], p1 = lo + __ldg(c + 1) * diag - o[1], p2 = lo + __ldg(c + 2) * diag - o[2];
    return (p0 * d[0] + p1 * d[1] + p2 * d[2]) * inv_dd;
}

// start of the march for ray i (ray_sampler.cu:31,:43-51)
__device__ __forceinline__ float ray_start_t(Pcg32 rng, uint32_t i, float lo, float hi, const float o[3], const float d[3], float near_distance, float cone) {
    rng.advance((uint64_t)(i * 8u));
    float tmin = fmaxf(aabb_ray_tmin(lo, hi, o, d), near_distance);
    return add_(tmin, mul_(calc_dt(tmin, cone), rng.next_float()));
}
// The march of ray (o, d) through the cascaded occupancy grid (ray_sampler.cu:58-72), from t with n samples taken so far. Every occupied
// sample calls on_sample(n, t, dt) and is counted; the march stops when the ray leaves the box, when n reaches limit (both: returns true,
// the ray has ended) or when on_sample returns false (returns false, a pause: marching on from the returned t and n continues the same sequence).
template <typename OnSample>
__device__ __forceinline__ bool march(float &t, uint32_t &n, uint32_t limit, const float o[3], const float d[3], float lo, float hi, float cone, const uint8_t *__restrict__ bitfield,
                                      const uint32_t *lut, OnSample &&on_sample) {
    const float idir[3] = {div_(1.0f, d[0]), div_(1.0f, d[1]), div_(1.0f, d[2])};
    while (true) {
        float p[3] = {add_(o[0], mul_(t, d[0])), add_(o[1], mul_(t, d[1])), add_(o[2], mul_(t, d[2]))};
        if (!(aabb_contains(lo, hi, p[0], p[1], p[2]) && n < limit)) return true;
        float dt = calc_dt(t, cone);
        uint32_t mip = (uint32_t)mip_from_dt(dt, p[0], p[1], p[2]);
        if (occupied_at(p[0], p[1], p[2], bitfield, mip, lut)) {
            const bool go_on = on_sample(n, t, dt);
            ++n; t = add_(t, dt);
            if (!go_on) return false;
        } else {
            t = advance_to_next_voxel(t, cone, p, d, idir, NERF_GRIDSIZE >> mip);
        }
    }
}

// activations (ray_sampler_header.h:440-456, :534-574; raymarch_shared.h:615-642). __expf as in the reference.
__device__ __forceinline__ float logistic(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float net_to_rgb(float v, int act) {
    switch (act) { case 0: return v; case 1: return v > 0.f ? v : 0.f; case 2: return logistic(v); case 3: return __expf(clampf(v, -10.f, 10.f)); }
    return 0.f;
}
__device__ __forceinline__ float net_to_density(float v, int act) {
    switch (act) { case 0: return v; case 1: return v > 0.f ? v : 0.f; case 2: return logistic(v); case 3: return __expf(v); }
    return 0.f;
}
__device__ __forceinline__ float net_to_rgb_deriv(float v, int act) {
    switch (act) { case 0: return 1.f; case 1: return v > 0.f ? 1.f : 0.f; case 2: { float s = logistic(v); return s * (1 - s); } case 3: return __expf(clampf(v, -10.f, 10.f)); }
    return 0.f;
}
__device__ __forceinline__ float net_to_density_deriv(float v, int act) {
    switch (act) { case 0: return 1.f; case 1: return v > 0.f ? 1.f : 0.f; case 2: { float s = logistic(v); return s * (1 - s); } case 3: return __expf(clampf(v, -15.f, 15.f)); }
    return 0.f;
}
// what one sample adds to the composite (calc_rgb.cu:31-39): its alpha over dt and its activated colour
struct CompositeTerm { float alpha, r, g, b; };
__device__ __forceinline__ CompositeTerm composite_term(float4 raw, float dt, int rgb_act, int dens_act) {
    return {1.f - __expf(-net_to_density(raw.w, dens_act) * dt), net_to_rgb(raw.x, rgb_act), net_to_rgb(raw.y, rgb_act), net_to_rgb(raw.z, rgb_act)};
}

// ---------------------------------------------------------------- warp and block scans
__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += n; }
    return v;
}
__device__ __forceinline__ float warp_incl_sum(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { float n = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += n; }
    return v;
}
__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { float n = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v *= n; }
    return v;
}
// exclusive product (1 on lane 0); *incl_out = the inclusive one
__device__ __forceinline__ float warp_excl_prod(float v, int lane, float *incl_out) {
    const float incl = warp_incl_prod(v, lane), ex = __shfl_up_sync(0xffffffffu, incl, 1);
    *incl_out = incl;
    return lane == 0 ? 1.f : ex;
}
// sum over the warp, on every lane (butterfly)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// exclusive scan of one uint32 per thread over a THREADS-thread block; *total = the block's sum. A kernel that calls it twice
// needs a __syncthreads() between the calls (both use the same shared words).
template <int THREADS>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t warp_tot[THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t incl = warp_incl_scan_u32(v, lane);
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    uint32_t off = 0, tot = 0;
#pragma unroll
    for (int k = 0; k < THREADS / 32; ++k) { const uint32_t s = warp_tot[k]; if (k < w) off += s; tot += s; }
    *total = tot;
    return off + incl - v;
}
#endif  // __CUDACC__

}  // namespace xrb
