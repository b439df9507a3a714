// xrnerf_b200 — device building blocks of the Instant-NGP field (hash-grid encoding, SH, tiny MLP) shared by the
// stand-alone tcnn-shaped kernels (ngp_mlp.cu), the backward kernels (ngp_backward.cu, ngp_backward_tc.cu) and the fused render kernel (ngp_fused.cu).
//
// Semantics restated from tiny-cuda-nn (see oracle/tcnn_oracle.c header: the reference delegates this arithmetic to an
// unpinned third-party package; call sites /root/reference/xrnerf/models/mlps/hashnerf_mlp.py:36-45,:55-79).
#pragma once
#include "common.cuh"

namespace xrb {

constexpr int MAX_LEVELS = 16;
struct HashGridDev {
    uint32_t offset[MAX_LEVELS + 1];  // in feature vectors
    float scale[MAX_LEVELS];
    uint32_t res[MAX_LEVELS];
    int n_levels;
    uint32_t hashed_mask;             // bit l: level l is hashed (its table is the 2^log2_hashmap_size cap), else dense
    uint32_t packed_mask;             // bit l: level l is gathered from the CELL IMAGE (one 32-byte record per grid cell), see cell_image_build()
    uint32_t cell_off[MAX_LEVELS];    // first record of level l inside the cell image (units: 32-byte records)
};

inline int64_t hashgrid_build(const xrb_ngp_config *cfg, HashGridDev *g) {
    g->n_levels = cfg->n_levels; g->hashed_mask = 0;
    const float log2_pls = log2f(cfg->per_level_scale);
    uint32_t off = 0;
    for (int l = 0; l < cfg->n_levels; ++l) {
        float scale = exp2f(l * log2_pls) * (float)cfg->base_resolution - 1.0f;
        uint32_t res = (uint32_t)ceilf(scale) + 1;
        uint64_t cube = (uint64_t)res * res * res; uint32_t maxp = 0xffffffffu / 2;
        uint32_t p = cube > maxp ? maxp : (uint32_t)cube;
        p = (p + 7u) / 8u * 8u;
        uint32_t cap = 1u << cfg->log2_hashmap_size; if (p > cap) p = cap;
        if (cube > p) g->hashed_mask |= 1u << l;   // then p == cap, a power of two: `% hashmap_size` is a mask
        g->offset[l] = off; g->scale[l] = scale; g->res[l] = res; off += p;
    }
    g->offset[cfg->n_levels] = off;
    g->packed_mask = 0;
    for (int l = 0; l < MAX_LEVELS; ++l) g->cell_off[l] = 0;
    return (int64_t)off * cfg->n_features;
}
// Cell image: a gather-friendly COPY of the first `n_packed` levels of the fp16 table. Level l stores, for every grid cell
// (gx,gy,gz) in [0,res)^3, its 8 corner feature pairs as ONE aligned 32-byte record (corner c = bit0 x, bit1 y, bit2 z; the entry
// tcnn's grid_index() addresses for that corner), cells in x-fastest order. A sample then reads one 32-byte record per level (one
// sector) instead of 8 scattered 4-byte entries (up to 8 wavefronts / sectors). The master parameters keep tcnn's
// layout (state_dict compatibility); the image is rebuilt from the fp16 table whenever that changes. Returns the image size in bytes
// and fills packed_mask / cell_off.
inline size_t cell_image_layout(HashGridDev *g, int n_packed) {
    size_t rec = 0; g->packed_mask = 0;
    for (int l = 0; l < g->n_levels && l < n_packed; ++l) {
        g->cell_off[l] = (uint32_t)rec; g->packed_mask |= 1u << l;
        rec += (size_t)g->res[l] * g->res[l] * g->res[l];
    }
    return rec * 32;
}
constexpr int MAX_PACKED_LEVELS = 13;  // image sizes for the reference grid: ..6 = 73 MB, ..7 = 190 MB, ..9 = 1.3 GB, ..12 = 25 GB;
                                       // levels past the L2 are served by HBM at ONE 32-byte sector per sample and level, where the hashed table costs ~4.5 sectors of L2
                                       // traffic (4 (y,z) rows, the x neighbour shares the sector in 7 of 8 cases). Level 13 alone would be 39 GB.
__host__ __device__ constexpr int64_t mlp_num_params(int in_w, int width, int n_hidden, int out_pad) { return (int64_t)width * in_w + (int64_t)(n_hidden - 1) * width * width + (int64_t)out_pad * width; }

inline int check_cfg(const xrb_ngp_config *cfg) {
    if (!cfg) { set_error("ngp config is null"); return XRB_E_BADARG; }
    if (cfg->n_levels != 16 || cfg->n_features != 2 || cfg->width != 64 || cfg->density_hidden < 1 || cfg->density_hidden > 4 || cfg->color_hidden < 1 || cfg->color_hidden > 4 ||
        cfg->log2_hashmap_size < 8 || cfg->log2_hashmap_size > 24 || cfg->base_resolution < 1) {
        set_error("ngp config unsupported: need n_levels=16, n_features=2, n_neurons=64, 1..4 hidden layers");
        return XRB_E_UNSUPPORTED;
    }
    return XRB_OK;
}

// Sample order of the chain render (ngp_render.cu): the field evaluates the rows bucketed by position only while there are at most this many.
// Beyond that the 28-byte sample rows no longer fit in L2, and reading and writing them in permuted order through HBM costs more than the
// coherent hash gather saves (measured: 0.7 M- and 1.8 M-sample batches faster, 6.5 M-sample whole 800x800 images slower; DESIGN.md §4.1).
constexpr uint32_t SAMPLE_ORDER_MAX_ROWS = 1u << 21;

// defined in ngp_mlp.cu: launches the field (impl 0 CUDA cores / 1 wgmma) on n rows; if n_dev != NULL the effective row
// count is min(n, *n_dev) read on the device. order (impl 1, full field only; NULL = row order): a permutation of the effective rows, evaluated
// in that order (tile slot j reads and writes row order[j]); ignored when there are more than SAMPLE_ORDER_MAX_ROWS effective rows.
// table_setup validates an xrb_ngp_table and describes it for the device.
int table_setup(const xrb_ngp_config *cfg, const xrb_ngp_table *t, HashGridDev *g);
int launch_field(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *dens, const void *color, const void *image, const float *pts, int pts_stride, const float *dirs,
                 int dirs_stride, int n, const int32_t *n_dev, const uint32_t *order, float *out, int impl, bool density_only, cudaStream_t s);
// defined in raymarch.cu: xrb_rm_calc_rgb_inference that also writes depth f32[n_rays] (t of each sample rebuilt from its coords row and the ray);
// with normal_out (and grad f32[rows,3], the per-row density gradient), also normal f32[n_rays,3] = sum of w * (-g / |g|)
int launch_composite_depth(const float *raw, const float *coords, const int32_t *numsteps, const float *bg3_host, int n_rays, int rgb_act, int dens_act, const float *rays_o,
                           const float *rays_d, float aabb0, float aabb1, float *rgb_out, float *alpha_out, float *depth_out, cudaStream_t s,
                           const float *grad = nullptr, float *normal_out = nullptr);
// defined in ngp_backward_tc.cu: xrb_ngp_density_grad_tc after its argument checks (n_dev, order as in launch_field)
int launch_density_grad_tc(const xrb_ngp_config *cfg, const xrb_ngp_table *tab, const void *weight_image, const float *pts, int pts_stride, int n, const int32_t *n_dev,
                           const uint32_t *order, float *density, float *grad, cudaStream_t s);

#ifdef __CUDACC__
__device__ __forceinline__ float round_h(float x) { return __half2float(__float2half_rn(x)); }

__device__ __forceinline__ uint32_t grid_index(uint32_t x, uint32_t y, uint32_t z, uint32_t hashmap_size, uint32_t res) {
    // tcnn grid.h grid_index(): dense strides while they fit, else the coherent prime hash; then `% hashmap_size`.
    // The modulo is strength-reduced without changing its value (an integer division is a multi-instruction sequence):
    //   hashed levels have hashmap_size == 2^log2_hashmap_size (the cap)          -> mask (never the generic `%`: it costs ~130 issue slots);
    //   dense levels have index <= res^3 + res^2 + res < 2 * hashmap_size          -> one conditional subtract.
    if ((uint64_t)res * res * res > hashmap_size) {   // uniform per level
        uint32_t h = x ^ (y * 2654435761u) ^ (z * 805459861u);
        return h & (hashmap_size - 1);   // a hashed level's table is always the 2^log2_hashmap_size cap (hashgrid_build)
    }
    uint32_t index = x + y * res + z * res * res;
    return index >= hashmap_size ? index - hashmap_size : index;
}

// one 32-byte cell record (one sector) as two 128-bit read-only loads (sm_90 has no 256-bit load)
struct __align__(32) Cell32 { uint32_t v[8]; };
__device__ __forceinline__ Cell32 ldg_cell(const void *p) {
    Cell32 r;
    const uint4 lo = __ldg(reinterpret_cast<const uint4 *>(p)), hi = __ldg(reinterpret_cast<const uint4 *>(p) + 1);
    r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w; r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
    return r;
}
__device__ __forceinline__ __half2 as_h2(uint32_t u) { return *reinterpret_cast<__half2 *>(&u); }

// The grid cell of a sample on level l: the level's slice of the table (first entry `off`, `hs` entries), its resolution, the integer cell and the
// position inside it. The ONLY place this arithmetic is written: the gather (hash_level) and every gradient scatter must agree on it bit for bit,
// or a sample on a cell boundary scatters into a different cell than it gathered from.
struct GridCell { uint32_t off, hs, res, gx, gy, gz; float fx, fy, fz; };
__device__ __forceinline__ GridCell grid_cell(const HashGridDev &g, int l, float x, float y, float z) {
    GridCell c;
    c.off = g.offset[l]; c.hs = g.offset[l + 1] - c.off; c.res = g.res[l];
    const float sc = g.scale[l];
    const float px = __fmaf_rn(sc, x, 0.5f), py = __fmaf_rn(sc, y, 0.5f), pz = __fmaf_rn(sc, z, 0.5f);
    int ix, iy, iz;
    const float flx = floor_small(px, &ix), fly = floor_small(py, &iy), flz = floor_small(pz, &iz);
    c.gx = (uint32_t)ix; c.gy = (uint32_t)iy; c.gz = (uint32_t)iz;
    c.fx = px - flx; c.fy = py - fly; c.fz = pz - flz;
    return c;
}

// one level of the multiresolution hash encoding: returns the two interpolated features (fp32, NOT yet rounded).
// Index arithmetic is tcnn's grid_index() strength-reduced without changing any value:
//   hashed level (res^3 > table size == 2^log2_hashmap_size): (x ^ y*P1 ^ z*P2) & (size-1); the two products are shared by the 8 corners
//   dense level: x + y*res + z*res^2 < 2*size -> one conditional subtract instead of `% size`
// (the generic `%` compiled to ~130 predicated-off but ISSUED instructions per level: ncu r01d source view)
// Three gather forms, all returning the same 8 entries (the L1 processes one 128-byte line per cycle per load instruction, and a warp's
// 32 scattered 4-byte reads touch up to 32 lines: the number of load instructions x lines is what the field kernel is bound by):
//   packed level   : the cell's 32-byte record from the cell image (cells: see cell_image_layout)
//   hashed level   : the x-prime of the hash is 1, so entries (gx, y, z) and (gx^1, y, z) are the two halves of one aligned 8-byte word:
//                    4 x 64-bit loads fetch both x-corners when gx is even and the gx corner when it is odd; odd lanes add 4 predicated
//                    32-bit loads for gx+1 (6 instead of 8 lines per lane on average)
//   dense, unpacked: 8 x 32-bit loads (only when the cell image is not given)
// MODE: the gather form of level l when the caller knows it at compile time (the field kernels are specialised on "the first NP levels
// are packed, every other level is hashed", which removes two of the three code paths per unrolled level), GATHER_RUNTIME otherwise.
enum { GATHER_RUNTIME = 0, GATHER_PACKED = 1, GATHER_HASHED = 2, GATHER_DENSE = 3 };
// gather form of level l under the static plan NP (NP == 0: decided at run time from the masks)
template <int NP> __host__ __device__ constexpr int plan_mode(int l) { return NP == 0 ? GATHER_RUNTIME : (l < NP ? GATHER_PACKED : GATHER_HASHED); }
// the static plan NP is valid for a grid iff exactly the first NP levels are packed and all others are hashed
inline bool plan_valid(const HashGridDev &g, int np) {
    if (np <= 0 || np > g.n_levels) return false;
    const uint32_t all = g.n_levels >= 32 ? 0xffffffffu : ((1u << g.n_levels) - 1u), packed = (1u << np) - 1u;
    return g.packed_mask == packed && ((g.hashed_mask | packed) & all) == all;
}

// (MODE is an ordinary argument of a force-inlined function: after unrolling it is a constant and the dead forms disappear)
__device__ __forceinline__ float2 hash_level(const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const HashGridDev &g, int l, float x, float y, float z,
                                             const int MODE = GATHER_RUNTIME) {
    const GridCell c = grid_cell(g, l, x, y, z);
    const uint32_t off = c.off, hs = c.hs, res = c.res, gx = c.gx, gy = c.gy, gz = c.gz;
    const float fx = c.fx, fy = c.fy, fz = c.fz;
    __half2 v[8];
    const bool is_packed = MODE == GATHER_PACKED || (MODE == GATHER_RUNTIME && ((g.packed_mask >> l) & 1u));
    const bool is_hashed = MODE == GATHER_HASHED || (MODE == GATHER_RUNTIME && ((g.hashed_mask >> l) & 1u));
    if (is_packed) {   // uniform per level
        // inputs are warped positions in [0,1] (cell coordinates in [0,res-1]); the clamp only keeps out-of-contract inputs inside the image
        const uint32_t rm1 = res - 1u, cx = min(gx, rm1), cy = min(gy, rm1), cz = min(gz, rm1);
        const Cell32 r = ldg_cell(cells + ((size_t)(g.cell_off[l] + cx + res * (cy + res * cz)) << 5));
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = as_h2(r.v[c]);
    } else if (is_hashed) {   // uniform per level
        const __half2 *tl = table + off;
        asm volatile("" : "+l"(tl));   // keep the level base in a register pair: each gather address is then ONE imad.wide (base + idx*4), not a 64-bit add chain
        const uint32_t mask = hs - 1u;
        const uint32_t hy0 = gy * 2654435761u, hy1 = hy0 + 2654435761u, hz0 = gz * 805459861u, hz1 = hz0 + 805459861u;
        const uint32_t a00 = hy0 ^ hz0, a10 = hy1 ^ hz0, a01 = hy0 ^ hz1, a11 = hy1 ^ hz1, gx1 = gx + 1u;
        const uint32_t i0 = (gx ^ a00) & mask, i1 = (gx ^ a10) & mask, i2 = (gx ^ a01) & mask, i3 = (gx ^ a11) & mask;
        // level offsets are multiples of 8 entries and the table is 16-byte aligned: (tl + (i & ~1)) is 8-byte aligned
        const uint2 w0 = __ldg(reinterpret_cast<const uint2 *>(tl + (i0 & ~1u))), w1 = __ldg(reinterpret_cast<const uint2 *>(tl + (i1 & ~1u))),
                    w2 = __ldg(reinterpret_cast<const uint2 *>(tl + (i2 & ~1u))), w3 = __ldg(reinterpret_cast<const uint2 *>(tl + (i3 & ~1u)));
        uint32_t n0 = 0, n1 = 0, n2 = 0, n3 = 0;
        const bool odd = gx & 1u;
        if (odd) {   // gx+1 carries out of the aligned pair: its entry is elsewhere
            n0 = __ldg(reinterpret_cast<const uint32_t *>(tl + ((gx1 ^ a00) & mask))); n1 = __ldg(reinterpret_cast<const uint32_t *>(tl + ((gx1 ^ a10) & mask)));
            n2 = __ldg(reinterpret_cast<const uint32_t *>(tl + ((gx1 ^ a01) & mask))); n3 = __ldg(reinterpret_cast<const uint32_t *>(tl + ((gx1 ^ a11) & mask)));
        }
        // entry of gx = half (i & 1) of the word; entry of gx^1 = the other half (== gx+1 when gx is even)
        const uint32_t e0 = (i0 & 1u) ? w0.y : w0.x, o0 = (i0 & 1u) ? w0.x : w0.y, e1 = (i1 & 1u) ? w1.y : w1.x, o1 = (i1 & 1u) ? w1.x : w1.y;
        const uint32_t e2 = (i2 & 1u) ? w2.y : w2.x, o2 = (i2 & 1u) ? w2.x : w2.y, e3 = (i3 & 1u) ? w3.y : w3.x, o3 = (i3 & 1u) ? w3.x : w3.y;
        v[0] = as_h2(e0); v[1] = as_h2(odd ? n0 : o0);
        v[2] = as_h2(e1); v[3] = as_h2(odd ? n1 : o1);
        v[4] = as_h2(e2); v[5] = as_h2(odd ? n2 : o2);
        v[6] = as_h2(e3); v[7] = as_h2(odd ? n3 : o3);
    } else {
        const __half2 *tl = table + off;
        asm volatile("" : "+l"(tl));
        const uint32_t sy = res, sz = res * res, b = gx + gy * sy + gz * sz;
#pragma unroll
        for (int c = 0; c < 8; ++c) {  // all 8 gathers are issued before any is consumed (8 independent loads in flight per level)
            uint32_t idx = b + (c & 1) + ((c >> 1) & 1) * sy + ((c >> 2) & 1) * sz;
            idx = idx >= hs ? idx - hs : idx;
            v[c] = __ldg(tl + idx);
        }
    }
    const float ux = 1.f - fx, uy = 1.f - fy, uz = 1.f - fz;
    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        float w = ((c & 1) ? fx : ux) * ((c & 2) ? fy : uy) * ((c & 4) ? fz : uz);
        float2 f = __half22float2(v[c]);
        acc.x += w * f.x; acc.y += w * f.y;
    }
    return acc;
}

// SH degree 4 on dir*2-1 (tcnn spherical_harmonics.h), fp32 values (caller rounds to fp16)
__device__ __forceinline__ void sh4(float dx01, float dy01, float dz01, float *out) {
    float x = dx01 * 2.f - 1.f, y = dy01 * 2.f - 1.f, z = dz01 * 2.f - 1.f;
    float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    out[0] = 0.28209479177387814f;
    out[1] = -0.48860251190291987f * y;
    out[2] = 0.48860251190291987f * z;
    out[3] = -0.48860251190291987f * x;
    out[4] = 1.0925484305920792f * xy;
    out[5] = -1.0925484305920792f * yz;
    out[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    out[7] = -1.0925484305920792f * xz;
    out[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    out[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    out[10] = 2.8906114426405538f * xy * z;
    out[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    out[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    out[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    out[14] = 1.4453057213202769f * z * (x2 - y2);
    out[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}
// Backward of sh4 with respect to its input: g[16] = dL/d(the 16 SH values) -> dL/d(dx01, dy01, dz01) = 2 sum_k g_k dSH_k/d(x, y, z), fp32
__device__ __forceinline__ float3 sh4_grad(float dx01, float dy01, float dz01, const float *g) {
    const float x = dx01 * 2.f - 1.f, y = dy01 * 2.f - 1.f, z = dz01 * 2.f - 1.f;
    const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    const float C1 = 0.48860251190291987f, C4 = 1.0925484305920792f, C6 = 0.94617469575755997f, C8 = 0.54627421529603959f, C9 = 0.59004358992664352f,
                C10 = 2.8906114426405538f, C11 = 0.45704579946446572f, C12 = 0.3731763325901154f, C14 = 1.4453057213202769f;
    float gx = -C1 * g[3] + C4 * y * g[4] - C4 * z * g[7] + 2.f * C8 * x * g[8] - 6.f * C9 * xy * g[9] + C10 * yz * g[10] + C11 * (1.f - 5.f * z2) * g[13]
               + 2.f * C14 * xz * g[14] + 3.f * C9 * (y2 - x2) * g[15];
    float gy = -C1 * g[1] + C4 * x * g[4] - C4 * z * g[5] - 2.f * C8 * y * g[8] + 3.f * C9 * (y2 - x2) * g[9] + C10 * xz * g[10] + C11 * (1.f - 5.f * z2) * g[11]
               - 2.f * C14 * yz * g[14] + 6.f * C9 * xy * g[15];
    float gz = C1 * g[2] - C4 * y * g[5] + 2.f * C6 * z * g[6] - C4 * x * g[7] + C10 * xy * g[10] - 10.f * C11 * yz * g[11] + C12 * (15.f * z2 - 3.f) * g[12]
               - 10.f * C11 * xz * g[13] + C14 * (x2 - y2) * g[14];
    return make_float3(2.f * gx, 2.f * gy, 2.f * gz);
}

// Backward of hash_level: adds the trilinear shares of (g0, g1) = dL/d(the level's two features) to the 8 corner entries of the fp32 table gradient.
// The plain form: one red.global.add.v2.f32 per corner. The CUDA-core backward kernels use it; they are what the tests compare the paired form against.
__device__ __forceinline__ void scatter_level(float *__restrict__ d_table, const GridCell &c, float g0, float g1) {
    float2 *tl = reinterpret_cast<float2 *>(d_table) + c.off;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        float w = ((k & 1) ? c.fx : 1.f - c.fx) * ((k & 2) ? c.fy : 1.f - c.fy) * ((k & 4) ? c.fz : 1.f - c.fz);
        uint32_t idx = grid_index(c.gx + (k & 1), c.gy + ((k >> 1) & 1), c.gz + ((k >> 2) & 1), c.hs, c.res);
        atomicAdd(tl + idx, make_float2(w * g0, w * g1));
    }
}
// Backward of hash_level with respect to the position: adds scale_l * sum_c (dw_c/df) * (v_c . (g0, g1)) to d, where v_c are the 8 corner feature pairs
// (re-read from the fp16 table at grid_index), w_c the trilinear weights and f the in-cell position grid_cell computes; (g0, g1) = dL/d(the level's two
// features). df/dx = scale_l. At a cell face the derivative is the one inside the cell grid_cell selects, the cell the gather read.
__device__ __forceinline__ void position_grad_level(const __half2 *__restrict__ table, const HashGridDev &g, int l, float x, float y, float z, float g0, float g1, float3 &d) {
    const GridCell c = grid_cell(g, l, x, y, z);
    const float ux = 1.f - c.fx, uy = 1.f - c.fy, uz = 1.f - c.fz;
    float dx = 0.f, dy = 0.f, dz = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t idx = grid_index(c.gx + (k & 1), c.gy + ((k >> 1) & 1), c.gz + ((k >> 2) & 1), c.hs, c.res);
        const float2 v = __half22float2(__ldg(table + c.off + idx));
        const float s = fmaf(v.y, g1, v.x * g0);   // dL/dw_c
        const float wx = (k & 1) ? c.fx : ux, wy = (k & 2) ? c.fy : uy, wz = (k & 4) ? c.fz : uz;
        const float ayz = wy * wz, axz = wx * wz, axy = wx * wy;
        dx = fmaf((k & 1) ? ayz : -ayz, s, dx);
        dy = fmaf((k & 2) ? axz : -axz, s, dy);
        dz = fmaf((k & 4) ? axy : -axy, s, dz);
    }
    const float sc = g.scale[l];
    d.x = fmaf(sc, dx, d.x); d.y = fmaf(sc, dy, d.y); d.z = fmaf(sc, dz, d.z);
}
// The paired form of the tensor-core backward (d_table 16-byte aligned). Its scatter is bound by the LSU's reduction issue rate (~1.3 cycles per lane
// and RED, measured: 450 of 880 us per 700 K samples with 128 two-float REDs per sample), so x-adjacent corners that are also adjacent in memory go out
// as ONE 16-byte red.global.add.v4.f32:
//   hashed level: entries of (gx, y, z) and (gx^1, y, z) are the two halves of an aligned 16-byte pair -> even gx: 4 v4 instead of 8 v2
//   dense level : idx and idx + 1 -> one v4 when idx is even (and the pair does not wrap at the table end)
__device__ __forceinline__ void scatter_level_paired(float *__restrict__ d_table, const GridCell &c, bool hashed, float g0, float g1) {
    float2 *tl = reinterpret_cast<float2 *>(d_table) + c.off;
#pragma unroll
    for (int yz = 0; yz < 4; ++yz) {
        const float wyz = ((yz & 1) ? c.fy : 1.f - c.fy) * ((yz & 2) ? c.fz : 1.f - c.fz);
        const float w0 = (1.f - c.fx) * wyz, w1 = c.fx * wyz;
        const uint32_t i0 = grid_index(c.gx, c.gy + (yz & 1), c.gz + (yz >> 1), c.hs, c.res), i1 = grid_index(c.gx + 1u, c.gy + (yz & 1), c.gz + (yz >> 1), c.hs, c.res);
        const bool pair = hashed ? ((c.gx & 1u) == 0u) : (((i0 & 1u) == 0u) && i1 == i0 + 1u);   // hashed, even gx: i1 == i0 ^ 1; both cases: i0 even, i1 = i0 + 1... or i0 odd (hashed)
        if (pair) {
            const uint32_t lo = i0 & ~1u;                      // hashed level with an odd i0: the pair is (i1, i0) in memory order
            const bool swap = (i0 & 1u) != 0u;
            const float a0 = swap ? w1 : w0, a1 = swap ? w0 : w1;
            atomicAdd(reinterpret_cast<float4 *>(tl + lo), make_float4(a0 * g0, a0 * g1, a1 * g0, a1 * g1));
        } else {
            atomicAdd(tl + i0, make_float2(w0 * g0, w0 * g1));
            atomicAdd(tl + i1, make_float2(w1 * g0, w1 * g1));
        }
    }
}

// colour-net input row of a sample: density_out[1:16] (15) ++ SH of the direction (16) ++ 1.0 pad (tcnn.Network pads 31 -> 32 with ones).
// fp32 values; the caller rounds to fp16
__device__ __forceinline__ void color_input_row(const float *dout, float dx, float dy, float dz, float *cin) {
#pragma unroll
    for (int k = 0; k < 15; ++k) cin[k] = dout[k + 1];
    sh4(dx, dy, dz, cin + 15);
    cin[31] = 1.0f;
}

// One layer on CUDA cores: y[o] = act(sum_k W[o][k] x[k]), W fp16 in shared memory (all lanes read the same address: broadcast), x/y fp32 registers.
// UNROLL: how many outputs are unrolled (all by default; the backward kernels, which are short of registers, take 4)
template <int IN, int OUT, bool RELU, int UNROLL = OUT>
__device__ __forceinline__ void simt_layer(const __half *__restrict__ W, const float *x, float *y) {
#pragma unroll UNROLL
    for (int o = 0; o < OUT; ++o) {
        float s = 0.f;
        const __half2 *w2 = reinterpret_cast<const __half2 *>(W + (size_t)o * IN);
#pragma unroll
        for (int k = 0; k < IN / 2; ++k) { float2 w = __half22float2(w2[k]); s = fmaf(w.x, x[2 * k], s); s = fmaf(w.y, x[2 * k + 1], s); }
        y[o] = round_h(RELU ? fmaxf(s, 0.f) : s);
    }
}

// ---------------------------------------------------------------------------- wgmma weight image
// Each matrix is a slab in the tile-image block layout (tc.cuh): row r (one output neuron) occupies 128 bytes = 64 halfs.
struct WeightImageLayout {  // byte offsets of each matrix inside the packed image
    uint32_t d_in, d_hid[3], d_out, c_in, c_hid[3], c_out, total;
};
__host__ __device__ inline WeightImageLayout weight_image_layout(int density_hidden, int color_hidden) {
    WeightImageLayout L{}; uint32_t o = 0;
    L.d_in = o; o += 64 * 128;
    for (int k = 0; k < density_hidden - 1; ++k) { L.d_hid[k] = o; o += 64 * 128; }
    L.d_out = o; o += 16 * 128;
    L.c_in = o; o += 64 * 128;
    for (int k = 0; k < color_hidden - 1; ++k) { L.c_hid[k] = o; o += 64 * 128; }
    L.c_out = o; o += 16 * 128;
    L.total = o;
    return L;
}
#endif  // __CUDACC__

}  // namespace xrb
