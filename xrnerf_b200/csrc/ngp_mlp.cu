// xrnerf_b200 — tcnn-shaped boundary (#2): hash-grid / SH encodings, fully-fused MLP, and the fused HashNerfMLP field.
// Two implementations of the field: impl 0 = CUDA cores (reference-grade, one thread per sample, weights broadcast from
// shared memory), impl 1 = wgmma tensor-core tiles (tc_field.cuh). Both follow the numeric contract in
// oracle/tcnn_oracle.c (fp16 operands, fp32 accumulate, fp16 activations).
#include "tc_field.cuh"

namespace xrb {

// ---------------------------------------------------------------------------- param casting / packing
__global__ void __launch_bounds__(256) cast_f32_to_f16_kernel(const float *__restrict__ src, __half *__restrict__ dst, int64_t n) {
    int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
    for (; i + 3 < n; i += stride) {
        float4 v = *reinterpret_cast<const float4 *>(src + i);
        __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
        uint2 o; o.x = *reinterpret_cast<uint32_t *>(&a); o.y = *reinterpret_cast<uint32_t *>(&b);
        *reinterpret_cast<uint2 *>(dst + i) = o;
    }
    if (blockIdx.x == 0 && threadIdx.x < 4) { int64_t t = (n & ~(int64_t)3) + threadIdx.x; if (t < n) dst[t] = __float2half_rn(src[t]); }
}

// one thread per (matrix row, 16-byte chunk): writes the swizzled K-major image, zero-filling k >= K
__global__ void pack_weights_kernel(const float *__restrict__ dens, const float *__restrict__ color, uint8_t *__restrict__ image, int density_hidden, int color_hidden) {
    const WeightImageLayout L = weight_image_layout(density_hidden, color_hidden);
    const int n_mats = density_hidden + 1 + color_hidden + 1;
    for (int m = blockIdx.x; m < n_mats; m += gridDim.x) {
        const bool is_color = m > density_hidden;
        const int li = is_color ? m - (density_hidden + 1) : m;            // layer index inside its net
        const int n_hidden = is_color ? color_hidden : density_hidden;
        const float *params = is_color ? color : dens;
        const int K = li == 0 ? 32 : 64, N = li == n_hidden ? 16 : 64;
        size_t poff = 0;
        for (int q = 0; q < li; ++q) poff += (size_t)64 * (q == 0 ? 32 : 64);
        const float *Wm = params + poff;                                   // W[N][K] row-major (tcnn layout)
        uint32_t ioff = is_color ? (li == 0 ? L.c_in : (li == n_hidden ? L.c_out : L.c_hid[li - 1])) : (li == 0 ? L.d_in : (li == n_hidden ? L.d_out : L.d_hid[li - 1]));
        for (int t = threadIdx.x; t < N * 8; t += blockDim.x) pack_slab_chunk(image + ioff, Wm, K, N, 0, K, t >> 3, t & 7);
    }
}

// ---------------------------------------------------------------------------- cell image (ngp_field.cuh: cell_image_layout)
// thread = (record, corner): copies the entry tcnn's grid_index() addresses for that corner; 32 consecutive threads write 128 consecutive bytes
__global__ void __launch_bounds__(256) cell_image_build_kernel(HashGridDev g, const __half2 *__restrict__ table, uint32_t *__restrict__ image, int n_packed, uint64_t n_words) {
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_words; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t rec = (uint32_t)(t >> 3), c = (uint32_t)t & 7u;
        int l = 0;
#pragma unroll
        for (int k = 1; k < MAX_PACKED_LEVELS; ++k) if (k < n_packed && rec >= g.cell_off[k]) l = k;   // cell_off is increasing
        const uint32_t res = g.res[l], cell = rec - g.cell_off[l];
        const uint32_t gx = cell % res, gy = (cell / res) % res, gz = cell / (res * res);
        const uint32_t hs = g.offset[l + 1] - g.offset[l];
        const uint32_t idx = grid_index(gx + (c & 1u), gy + ((c >> 1) & 1u), gz + ((c >> 2) & 1u), hs, res);
        image[t] = reinterpret_cast<const uint32_t *>(table)[g.offset[l] + idx];
    }
}

// ---------------------------------------------------------------------------- stand-alone encodings
__global__ void __launch_bounds__(256) hashgrid_forward_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const float *__restrict__ x,
                                                               int x_stride, int n, __half2 *__restrict__ enc) {
    // thread = (sample, level): consecutive lanes take consecutive levels of the same sample -> 64-byte coalesced row writes
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t i = t >> 4; int l = (int)(t & 15);
    if (i >= n) return;
    const float *p = x + (size_t)i * x_stride;
    float2 f = hash_level(table, cells, g, l, p[0], p[1], p[2]);
    enc[(size_t)i * 16 + l] = __floats2half2_rn(f.x, f.y);
}
__global__ void __launch_bounds__(256) sh4_forward_kernel(const float *__restrict__ dirs, int stride, int n, __half *__restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *d = dirs + (size_t)i * stride;
    float s[16]; sh4(d[0], d[1], d[2], s);
    __half h[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) h[k] = __float2half_rn(s[k]);
    uint4 *o = reinterpret_cast<uint4 *>(out + (size_t)i * 16);
    o[0] = reinterpret_cast<uint4 *>(h)[0]; o[1] = reinterpret_cast<uint4 *>(h)[1];
}

// ---------------------------------------------------------------------------- CUDA-core MLP (impl 0)
// generic net: in_w (32) -> [64]*n_hidden -> 16; params = contiguous fp16 in shared memory
__device__ __forceinline__ void simt_net(const __half *__restrict__ P, int n_hidden, const float *x32, float *out16) {
    float a[64], b[64];
    simt_layer<32, 64, true>(P, x32, a); P += 64 * 32;
    for (int h = 0; h < n_hidden - 1; ++h) {
        simt_layer<64, 64, true>(P, a, b); P += 64 * 64;
#pragma unroll
        for (int k = 0; k < 64; ++k) a[k] = b[k];
    }
    simt_layer<64, 16, false>(P, a, out16);
}

template <bool DENSITY_ONLY>
__global__ void __launch_bounds__(128) ngp_field_simt_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const __half *__restrict__ dens_p, const __half *__restrict__ color_p,
                                                             int density_hidden, int color_hidden, const float *__restrict__ pts, int pts_stride, const float *__restrict__ dirs,
                                                             int dirs_stride, int n, const int32_t *__restrict__ n_dev, float *__restrict__ out) {
    extern __shared__ __half s_w[];
    if (n_dev) n = min(n, max(*n_dev, 0));  // sample count produced on the device by the march (no host sync)
    const int nd = (int)mlp_num_params(32, 64, density_hidden, 16), nc = DENSITY_ONLY ? 0 : (int)mlp_num_params(32, 64, color_hidden, 16);
    for (int k = threadIdx.x; k < nd; k += blockDim.x) s_w[k] = dens_p[k];
    for (int k = threadIdx.x; k < nc; k += blockDim.x) s_w[nd + k] = color_p[k];
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float *p = pts + (size_t)i * pts_stride;
        float enc[32];
#pragma unroll
        for (int l = 0; l < 16; ++l) { float2 f = hash_level(table, cells, g, l, p[0], p[1], p[2]); enc[2 * l] = round_h(f.x); enc[2 * l + 1] = round_h(f.y); }
        float dout[16];
        simt_net(s_w, density_hidden, enc, dout);
        if (DENSITY_ONLY) { out[i] = dout[0]; continue; }
        const float *d = dirs + (size_t)i * dirs_stride;
        float cin[32];
        color_input_row(dout, d[0], d[1], d[2], cin);
#pragma unroll
        for (int k = 15; k < 31; ++k) cin[k] = round_h(cin[k]);   // the SH values; dout and 1.0 are fp16 values already
        float cout[16];
        simt_net(s_w + nd, color_hidden, cin, cout);
        reinterpret_cast<float4 *>(out)[i] = make_float4(cout[0], cout[1], cout[2], dout[0]);
    }
}

// stand-alone tcnn.Network forward (fp16 in, fp16 out[16])
__global__ void __launch_bounds__(128) mlp_forward_simt_kernel(const __half *__restrict__ params, const __half *__restrict__ x, int n, int n_hidden, __half *__restrict__ y) {
    extern __shared__ __half s_w[];
    const int np = (int)mlp_num_params(32, 64, n_hidden, 16);
    for (int k = threadIdx.x; k < np; k += blockDim.x) s_w[k] = params[k];
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float xin[32], out[16];
#pragma unroll
        for (int k = 0; k < 32; ++k) xin[k] = __half2float(x[(size_t)i * 32 + k]);
        simt_net(s_w, n_hidden, xin, out);
#pragma unroll
        for (int k = 0; k < 16; ++k) y[(size_t)i * 16 + k] = __float2half_rn(out[k]);
    }
}

// ---------------------------------------------------------------------------- tensor-core field (impl 1)
// FIELD_NWG warpgroups (= concurrent 128-sample tiles) per CTA share ONE resident weight image; accumulators live in registers (tc_field.cuh).
// The gather is latency-bound; two CTAs per SM (16 warps), which caps a thread at 128 registers, is the fastest shape measured and the only one
// without spills (DESIGN §4.1 has the sweep).
// NP: static gather plan (ngp_field.cuh plan_mode): 0 = per-level form decided at run time, >0 = levels [0,NP) from the cell image, the rest hashed.
// Per tile a warpgroup gathers the 16 levels, then runs both nets; the four warpgroups of an SM overlap one's gather with another's tensor-core layers.
constexpr int FIELD_NWG = 2;
template <bool DENSITY_ONLY, int NP>
__global__ void __launch_bounds__(128 * FIELD_NWG, 2)
ngp_field_tc_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const void *__restrict__ weight_image, uint32_t image_bytes, int density_hidden,
                    int color_hidden, const float *__restrict__ pts, int pts_stride, const float *__restrict__ dirs, int dirs_stride, int n, const int32_t *__restrict__ n_dev,
                    const uint32_t *__restrict__ order, float *__restrict__ out) {
    extern __shared__ uint8_t dyn_smem[];
    if (n_dev) n = min(n, max(*n_dev, 0));
    if (n > (int)SAMPLE_ORDER_MAX_ROWS) order = nullptr;
    TcWarpgroup c = tc_cta_setup<FIELD_NWG>(dyn_smem, weight_image, image_bytes);
    const WeightImageLayout L = weight_image_layout(density_hidden, color_hidden);
    const int n_tiles = (n + 127) / 128;
    for (int tile = blockIdx.x * FIELD_NWG + c.wg; tile < n_tiles; tile += gridDim.x * FIELD_NWG) {
        const int j = tile * 128 + c.row;
        const bool valid = j < n;
        const int i = !DENSITY_ONLY && valid && order ? (int)__ldg(order + j) : j;   // the row this tile slot evaluates: the rows of a tile are independent
        float x = 0.5f, y = 0.5f, z = 0.5f, dx = 0.5f, dy = 0.5f, dz = 0.5f;
        if (valid) {
            const float *p = pts + (size_t)i * pts_stride; x = p[0]; y = p[1]; z = p[2];
            if (!DENSITY_ONLY) { const float *d = dirs + (size_t)i * dirs_stride; dx = d[0]; dy = d[1]; dz = d[2]; }
        }
        uint32_t e[16];
        tc_gather_levels<NP, 0, 16>(table, cells, g, x, y, z, e);
#pragma unroll
        for (int q = 0; q < 4; ++q) a_store_chunk(c, q, make_uint4(e[4 * q], e[4 * q + 1], e[4 * q + 2], e[4 * q + 3]));
        float dout[16];
        tc_density_from_a(c, L, density_hidden, dout);
        if (DENSITY_ONLY) {
            if (valid) out[i] = dout[0];
        } else {
            const float4 raw = tc_color_from_density(c, L, color_hidden, dout, dx, dy, dz);
            if (valid) reinterpret_cast<float4 *>(out)[i] = raw;
        }
    }
}

// ---------------------------------------------------------------------------- host side: table description and the field launchers
// validates an xrb_ngp_table and fills the device-side grid description (incl. the cell-image layout)
int table_setup(const xrb_ngp_config *cfg, const xrb_ngp_table *t, HashGridDev *g) {
    if (!t || !t->table_fp16) { set_error("null hash table"); return XRB_E_BADARG; }
    if (((uintptr_t)t->table_fp16 & 15) != 0) { set_error("hash table must be 16-byte aligned"); return XRB_E_BADARG; }
    hashgrid_build(cfg, g);
    if (t->n_packed_levels < 0 || t->n_packed_levels > MAX_PACKED_LEVELS) { set_error("n_packed_levels must be 0..13"); return XRB_E_BADARG; }
    if (t->n_packed_levels > 0) {
        if (!t->cell_image || ((uintptr_t)t->cell_image & 31) != 0) { set_error("cell image missing or not 32-byte aligned"); return XRB_E_BADARG; }
        cell_image_layout(g, t->n_packed_levels);
    }
    return XRB_OK;
}

template <bool DENSITY_ONLY, int NP>
static void launch_field_tc(const xrb_ngp_config *cfg, const HashGridDev &g, const void *table, const uint8_t *cells, const void *image, uint32_t image_bytes, const float *pts,
                            int pts_stride, const float *dirs, int dirs_stride, int n, const int32_t *n_dev, const uint32_t *order, float *out, cudaStream_t s) {
    auto k = ngp_field_tc_kernel<DENSITY_ONLY, NP>;
    const size_t smem = tc_cta_smem_bytes<FIELD_NWG>(image_bytes);
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int n_tiles = (n + 127) / 128;
    const int grid = persistent_grid((const void *)k, 128 * FIELD_NWG, smem, (n_tiles + FIELD_NWG - 1) / FIELD_NWG, 2);
    k<<<grid, 128 * FIELD_NWG, smem, s>>>(g, (const __half2 *)table, cells, image, image_bytes, cfg->density_hidden, cfg->color_hidden, pts, pts_stride, dirs, dirs_stride, n, n_dev, order,
                                          out);
}

int launch_field(const xrb_ngp_config *cfg, const xrb_ngp_table *tab, const void *dens, const void *color, const void *image, const float *pts, int pts_stride, const float *dirs,
                 int dirs_stride, int n, const int32_t *n_dev, const uint32_t *order, float *out, int impl, bool density_only, cudaStream_t s) {
    HashGridDev g; int e = table_setup(cfg, tab, &g); if (e) return e;
    const void *table = tab->table_fp16; const uint8_t *cells = (const uint8_t *)tab->cell_image;
    XRB_REQUIRE(impl != 0 || order == nullptr, "field: an evaluation order needs the tensor-core field");
    if (impl == 0) {
        size_t smem = (mlp_num_params(32, 64, cfg->density_hidden, 16) + (density_only ? 0 : mlp_num_params(32, 64, cfg->color_hidden, 16))) * sizeof(__half);
        const void *k = density_only ? (const void *)ngp_field_simt_kernel<true> : (const void *)ngp_field_simt_kernel<false>;
        if (smem > 48 * 1024) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int grid = persistent_grid(k, 128, smem, (n + 127) / 128);
        if (density_only)
            ngp_field_simt_kernel<true><<<grid, 128, smem, s>>>(g, (const __half2 *)table, cells, (const __half *)dens, (const __half *)color, cfg->density_hidden, cfg->color_hidden, pts, pts_stride,
                                                                dirs, dirs_stride, n, n_dev, out);
        else
            ngp_field_simt_kernel<false><<<grid, 128, smem, s>>>(g, (const __half2 *)table, cells, (const __half *)dens, (const __half *)color, cfg->density_hidden, cfg->color_hidden, pts, pts_stride,
                                                                 dirs, dirs_stride, n, n_dev, out);
    } else {
        uint32_t image_bytes = weight_image_layout(cfg->density_hidden, cfg->color_hidden).total;
        // Measured with scripts/field_bench.py on one H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock), 699 K samples, 7-level cell image: 248 us
        // (ptxas: 128 registers, 0 spill bytes).
        // static gather plan: the kernel is specialised for "levels [0,NP) packed, all others hashed" (NP = 6, 7); anything else takes the run-time form
        const int npl = tab->n_packed_levels;
        const int np = (plan_valid(g, npl) && (npl == 6 || npl == 7)) ? npl : 0;
        auto launch = density_only ? (np == 6 ? launch_field_tc<true, 6> : np == 7 ? launch_field_tc<true, 7> : launch_field_tc<true, 0>)
                                   : (np == 6 ? launch_field_tc<false, 6> : np == 7 ? launch_field_tc<false, 7> : launch_field_tc<false, 0>);
        launch(cfg, g, table, cells, image, image_bytes, pts, pts_stride, dirs, dirs_stride, n, n_dev, order, out, s);
    }
    return check_launch(density_only ? "ngp_density_forward" : "ngp_mlp_forward");
}

}  // namespace xrb

using namespace xrb;

extern "C" {

int64_t xrb_tcnn_hashgrid_num_params(const xrb_ngp_config *cfg) { if (check_cfg(cfg)) return -1; HashGridDev g; return hashgrid_build(cfg, &g); }
int64_t xrb_tcnn_density_num_params(const xrb_ngp_config *cfg) { if (check_cfg(cfg)) return -1; return mlp_num_params(32, 64, cfg->density_hidden, 16); }
int64_t xrb_tcnn_color_num_params(const xrb_ngp_config *cfg) { if (check_cfg(cfg)) return -1; return mlp_num_params(32, 64, cfg->color_hidden, 16); }
int xrb_tcnn_hashgrid_layout(const xrb_ngp_config *cfg, uint32_t *offsets_host, float *scales_host, uint32_t *res_host) {
    int e = check_cfg(cfg); if (e) return e;
    HashGridDev g; hashgrid_build(cfg, &g);
    for (int l = 0; l <= cfg->n_levels; ++l) if (offsets_host) offsets_host[l] = g.offset[l];
    for (int l = 0; l < cfg->n_levels; ++l) { if (scales_host) scales_host[l] = g.scale[l]; if (res_host) res_host[l] = g.res[l]; }
    return XRB_OK;
}

int xrb_tcnn_cast_params(const float *src, void *dst_fp16, int64_t n, void *stream) {
    XRB_REQUIRE(n >= 0, "cast_params: negative size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(src && dst_fp16, "cast_params: null pointer");
    XRB_REQUIRE(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst_fp16 & 7) == 0, "cast_params: misaligned");
    const int blocks = stride_grid((n / 4 + 255) / 256, 16);
    cast_f32_to_f16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, (__half *)dst_fp16, n);
    return check_launch("cast_params");
}

size_t xrb_ngp_weight_image_bytes(const xrb_ngp_config *cfg) { if (check_cfg(cfg)) return 0; return weight_image_layout(cfg->density_hidden, cfg->color_hidden).total; }

int xrb_ngp_pack_weights(const xrb_ngp_config *cfg, const float *density_params, const float *color_params, void *image, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(density_params && color_params && image, "pack_weights: null pointer");
    XRB_REQUIRE(((uintptr_t)image & 15) == 0, "pack_weights: image must be 16-byte aligned");
    pack_weights_kernel<<<cfg->density_hidden + cfg->color_hidden + 2, 256, 0, (cudaStream_t)stream>>>(density_params, color_params, (uint8_t *)image, cfg->density_hidden, cfg->color_hidden);
    return check_launch("pack_weights");
}

size_t xrb_ngp_cell_image_bytes(const xrb_ngp_config *cfg, int n_packed_levels) {
    if (check_cfg(cfg) || n_packed_levels <= 0) return 0;
    if (n_packed_levels > MAX_PACKED_LEVELS) n_packed_levels = MAX_PACKED_LEVELS;
    HashGridDev g; hashgrid_build(cfg, &g);
    return cell_image_layout(&g, n_packed_levels);
}

int xrb_ngp_build_cell_image(const xrb_ngp_config *cfg, const void *table_fp16, int n_packed_levels, void *cell_image, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n_packed_levels >= 0 && n_packed_levels <= MAX_PACKED_LEVELS, "build_cell_image: n_packed_levels must be 0..13");
    if (n_packed_levels == 0) return XRB_OK;
    XRB_REQUIRE(table_fp16 && cell_image, "build_cell_image: null pointer");
    XRB_REQUIRE(((uintptr_t)cell_image & 31) == 0 && ((uintptr_t)table_fp16 & 15) == 0, "build_cell_image: cell image must be 32-byte, table 16-byte aligned");
    HashGridDev g; hashgrid_build(cfg, &g);
    const uint64_t n_words = cell_image_layout(&g, n_packed_levels) / 4;
    cell_image_build_kernel<<<stride_grid((int64_t)(n_words + 255) / 256, 32), 256, 0, (cudaStream_t)stream>>>(g, (const __half2 *)table_fp16, (uint32_t *)cell_image, n_packed_levels, n_words);
    return check_launch("build_cell_image");
}

int xrb_tcnn_hashgrid_forward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const float *x, int x_stride, int n, void *enc_fp16, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && x_stride >= 3, "hashgrid_forward: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(table && x && enc_fp16, "hashgrid_forward: null pointer");
    HashGridDev g; e = table_setup(cfg, table, &g); if (e) return e;
    int64_t threads = (int64_t)n * 16;
    hashgrid_forward_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, (const __half2 *)table->table_fp16, (const uint8_t *)table->cell_image, x, x_stride, n,
                                                                                                 (__half2 *)enc_fp16);
    return check_launch("hashgrid_forward");
}

int xrb_tcnn_sh4_forward(const float *dirs, int dir_stride, int n, void *out_fp16, void *stream) {
    XRB_REQUIRE(n >= 0 && dir_stride >= 3, "sh4_forward: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(dirs && out_fp16, "sh4_forward: null pointer");
    sh4_forward_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(dirs, dir_stride, n, (__half *)out_fp16);
    return check_launch("sh4_forward");
}

int xrb_tcnn_mlp_forward(const void *params_fp16, const void *x_fp16, int n, int in_w, int width, int n_hidden, void *y_fp16, void *stream) {
    XRB_REQUIRE(n >= 0, "mlp_forward: negative size");
    if (in_w != 32 || width != 64 || n_hidden < 1 || n_hidden > 4) { set_error("mlp_forward: only in=32 (padded), width=64, 1..4 hidden layers"); return XRB_E_UNSUPPORTED; }
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(params_fp16 && x_fp16 && y_fp16, "mlp_forward: null pointer");
    size_t smem = mlp_num_params(32, 64, n_hidden, 16) * sizeof(__half);
    if (smem > 48 * 1024) cudaFuncSetAttribute(mlp_forward_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int grid = persistent_grid((const void *)mlp_forward_simt_kernel, 128, smem, (n + 127) / 128);
    mlp_forward_simt_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>((const __half *)params_fp16, (const __half *)x_fp16, n, n_hidden, (__half *)y_fp16);
    return check_launch("mlp_forward");
}

int xrb_ngp_mlp_forward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *color_fp16, const void *weight_image, const float *pts, int pts_stride,
                        const float *dirs, int dirs_stride, int n, const int32_t *n_rows_dev, float *raw, int impl, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && pts_stride >= 3 && dirs_stride >= 3, "ngp_mlp_forward: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(table && pts && dirs && raw, "ngp_mlp_forward: null pointer");
    XRB_REQUIRE(((uintptr_t)raw & 15) == 0, "ngp_mlp_forward: raw must be 16-byte aligned");
    XRB_REQUIRE(impl == 0 ? (density_fp16 && color_fp16) : (weight_image != nullptr), "ngp_mlp_forward: missing weights for the requested impl");
    return launch_field(cfg, table, density_fp16, color_fp16, weight_image, pts, pts_stride, dirs, dirs_stride, n, n_rows_dev, nullptr, raw, impl, false, (cudaStream_t)stream);
}

int xrb_ngp_density_forward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *weight_image, const float *pts, int pts_stride, int n, float *density,
                            int impl, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && pts_stride >= 3, "ngp_density_forward: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(table && pts && density, "ngp_density_forward: null pointer");
    XRB_REQUIRE(impl == 0 ? (density_fp16 != nullptr) : (weight_image != nullptr), "ngp_density_forward: missing weights for the requested impl");
    return launch_field(cfg, table, density_fp16, nullptr, weight_image, pts, pts_stride, nullptr, 3, n, nullptr, nullptr, density, impl, true, (cudaStream_t)stream);
}

}  // extern "C"
