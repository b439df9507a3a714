// xrnerf_b200 — NeRF / Mip-NeRF kernels for what is pure PyTorch in the reference (≈25 tiny ATen kernels per render call, a full
// sort + expanded gathers per sample_pdf call; SURVEY §3a). Compositing, sample_pdf and Mip-NeRF resampling: one launch each, one WARP per
// ray, lanes over samples with shuffle scans. Every encoder: positional encoding and Mip-NeRF IPE, into fp32 `embedded` rows or straight
// into the fp16 tile images the NerfMLP kernels read. Ray generation and z values. References relative to /root/reference/xrnerf/models/.
#include "common.cuh"
#include "posenc.cuh"
#include "tc.cuh"

namespace xrb {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float softplusf_(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // F.softplus(beta=1, threshold=20)

struct CompositeParams { int n_rays, n_samples, mip, white_bkgd, density_act; float rgb_padding, density_bias; };

// per-sample quantities of renders/nerf_render.py:61-83 (and mipnerf_render.py:27-33 when mip)
__device__ __forceinline__ void sample_terms(const CompositeParams &p, const float *__restrict__ raw, const float *__restrict__ z, float dnorm, int k, float4 &r, float &sd,
                                             float &alpha) {
    r = __ldg(reinterpret_cast<const float4 *>(raw) + k);
    float dist = p.mip ? (z[k + 1] - z[k]) : (k + 1 < p.n_samples ? z[k + 1] - z[k] : 1e10f);
    dist *= dnorm;
    float a = r.w + p.density_bias;
    float dens = p.density_act == XRB_ACT_SOFTPLUS ? softplusf_(a) : fmaxf(a, 0.f);
    sd = dens * dist;
    alpha = 1.f - expf(-sd);
}
// transmittance before each lane's sample; carry = the running sum of sigma*delta (mip) or product of (1-alpha+1e-10) (nerf) of the earlier chunks
__device__ __forceinline__ float transmittance(bool mip, bool valid, float sd, float alpha, int lane, float &carry) {
    float T;
    if (mip) { const float inc = warp_incl_sum(sd, lane); T = expf(-(carry + inc - sd)); carry += __shfl_sync(0xffffffffu, inc, 31); }
    else { float incl, ex = warp_excl_prod(valid ? (1.f - alpha + 1e-10f) : 1.f, lane, &incl); T = carry * ex; carry *= __shfl_sync(0xffffffffu, incl, 31); }
    return T;
}

// BACKWARD == false: rgb/disp/acc/weights, plus depth_out = sum of w * z (interval mid-points when mip) when DEPTH.
// BACKWARD == true: d_raw given grad_rgb (loss on rgb only, nerf.py:79-84 / mipnerf.py:49-57); GEOM: also given grad_depth and grad_acc (either may be
// NULL), the gradients of the depth DEPTH writes and of acc, so that d L / d w_k = G_k = g . (c_k - wb) + g_d z_k + g_a
template <bool BACKWARD, bool DEPTH = false, bool GEOM = false>
__global__ void __launch_bounds__(256) nerf_composite_kernel(CompositeParams p, const float *__restrict__ raw, const float *__restrict__ z_vals, const float *__restrict__ rays_d,
                                                             const float *__restrict__ grad_rgb, float *__restrict__ rgb_out, float *__restrict__ disp_out, float *__restrict__ acc_out,
                                                             float *__restrict__ weights_out, float *__restrict__ d_raw, float *__restrict__ depth_out,
                                                             const float *__restrict__ grad_depth, const float *__restrict__ grad_acc) {
    static_assert(!(BACKWARD && DEPTH), "depth is a forward output");
    static_assert(!GEOM || BACKWARD, "the geometry gradients are a backward input");
    const int lane = threadIdx.x & 31;
    const int ray = (blockIdx.x * 256 + threadIdx.x) >> 5;
    if (ray >= p.n_rays) return;
    const int S = p.n_samples, zs = p.mip ? S + 1 : S;
    const float *rw = raw + (size_t)ray * S * 4, *z = z_vals + (size_t)ray * zs;
    const float dx = rays_d[3 * (size_t)ray], dy = rays_d[3 * (size_t)ray + 1], dz = rays_d[3 * (size_t)ray + 2];
    const float dnorm = sqrtf(dx * dx + dy * dy + dz * dz);
    const float pad_mul = 1.f + 2.f * p.rgb_padding;
    float gx = 0, gy = 0, gz = 0;
    if (BACKWARD) { gx = grad_rgb[3 * (size_t)ray]; gy = grad_rgb[3 * (size_t)ray + 1]; gz = grad_rgb[3 * (size_t)ray + 2]; }
    float gd = 0.f, ga = 0.f;
    const bool geo = GEOM && (grad_depth || grad_acc);   // without either gradient, the colour-only arithmetic exactly
    if (geo) { gd = grad_depth ? grad_depth[ray] : 0.f; ga = grad_acc ? grad_acc[ray] : 0.f; }
    // ---- pass 1: forward accumulation
    float carry = p.mip ? 0.f : 1.f;  // mip: running sum of sigma*delta; nerf: running product of (1-alpha+1e-10)
    float ax = 0, ay = 0, az = 0, acc = 0, depth = 0, total_wg = 0;
    for (int k0 = 0; k0 < S; k0 += 32) {
        int k = k0 + lane; bool valid = k < S;
        float4 r = make_float4(0, 0, 0, 0); float sd = 0, alpha = 0;
        if (valid) sample_terms(p, rw, z, dnorm, k, r, sd, alpha);
        const float T = transmittance(p.mip, valid, sd, alpha, lane, carry);
        float w = valid ? alpha * T : 0.f;
        float cx = sigmoidf_(r.x) * pad_mul - p.rgb_padding, cy = sigmoidf_(r.y) * pad_mul - p.rgb_padding, cz = sigmoidf_(r.z) * pad_mul - p.rgb_padding;
        if (!BACKWARD) {
            ax += w * cx; ay += w * cy; az += w * cz; acc += w;
            if (valid) { depth += w * (p.mip ? 0.5f * (z[k] + z[k + 1]) : z[k]); weights_out[(size_t)ray * S + k] = w; }
        } else {
            float wb = p.white_bkgd ? 1.f : 0.f;
            float G = gx * (cx - wb) + gy * (cy - wb) + gz * (cz - wb);
            if (geo && valid) G += gd * (p.mip ? 0.5f * (z[k] + z[k + 1]) : z[k]) + ga;
            total_wg += w * G;
        }
    }
    if (!BACKWARD) {
        ax = warp_sum(ax); ay = warp_sum(ay); az = warp_sum(az); acc = warp_sum(acc); depth = warp_sum(depth);
        if (lane == 0) {
            if (p.white_bkgd) { ax += 1.f - acc; ay += 1.f - acc; az += 1.f - acc; }
            rgb_out[3 * (size_t)ray] = ax; rgb_out[3 * (size_t)ray + 1] = ay; rgb_out[3 * (size_t)ray + 2] = az;
            acc_out[ray] = acc;
            if (DEPTH) depth_out[ray] = depth;
            float q = depth / acc, disp;
            if (p.mip) { if (isnan(q)) q = INFINITY; disp = fmaxf(fminf(q, z[S]), z[0]); }          // mipnerf_render.py:18-24
            else disp = 1.f / fmaxf(1e-10f, q);                                                       // nerf_render.py:32-36 (torch.max propagates NaN)
            if (!p.mip && isnan(q)) disp = q;
            disp_out[ray] = disp;
        }
        return;
    }
    // ---- pass 2 (backward): dL/d(sigma*delta_i) needs the suffix sum of w_k*G_k over k > i
    total_wg = warp_sum(total_wg);
    carry = p.mip ? 0.f : 1.f;
    float prefix_wg = 0.f;
    for (int k0 = 0; k0 < S; k0 += 32) {
        int k = k0 + lane; bool valid = k < S;
        float4 r = make_float4(0, 0, 0, 0); float sd = 0, alpha = 0;
        if (valid) sample_terms(p, rw, z, dnorm, k, r, sd, alpha);
        const float T = transmittance(p.mip, valid, sd, alpha, lane, carry);
        float w = valid ? alpha * T : 0.f;
        float sx = sigmoidf_(r.x), sy = sigmoidf_(r.y), sz = sigmoidf_(r.z);
        float cx = sx * pad_mul - p.rgb_padding, cy = sy * pad_mul - p.rgb_padding, cz = sz * pad_mul - p.rgb_padding;
        float wb = p.white_bkgd ? 1.f : 0.f;
        float G = gx * (cx - wb) + gy * (cy - wb) + gz * (cz - wb);
        if (geo && valid) G += gd * (p.mip ? 0.5f * (z[k] + z[k + 1]) : z[k]) + ga;
        float inc_wg = warp_incl_sum(w * G, lane);
        float suffix = total_wg - (prefix_wg + inc_wg);
        prefix_wg += __shfl_sync(0xffffffffu, inc_wg, 31);
        if (valid) {
            float one_m = 1.f - alpha;
            float dL_dsd = p.mip ? (one_m * T * G - suffix) : (one_m * (T * G - suffix / (one_m + 1e-10f)));
            float dist = p.mip ? (z[k + 1] - z[k]) : (k + 1 < S ? z[k + 1] - z[k] : 1e10f);
            dist *= dnorm;
            float a = r.w + p.density_bias;
            float dact = p.density_act == XRB_ACT_SOFTPLUS ? (a > 20.f ? 1.f : sigmoidf_(a)) : (a > 0.f ? 1.f : 0.f);
            float4 o;
            o.x = gx * w * sx * (1.f - sx) * pad_mul; o.y = gy * w * sy * (1.f - sy) * pad_mul; o.z = gz * w * sz * (1.f - sz) * pad_mul;
            o.w = dL_dsd * dist * dact;
            reinterpret_cast<float4 *>(d_raw)[(size_t)ray * S + k] = o;
        }
    }
}

// sample_pdf (networks/utils/hierarchical_sample.py:6-53): one warp per ray, everything in shared memory, bitonic merge sort
constexpr int PDF_WARPS = 4;
constexpr int PDF_MAX_S = 256;   // coarse samples
constexpr int PDF_MAX_OUT = 512; // coarse + importance
__global__ void __launch_bounds__(PDF_WARPS * 32) sample_pdf_kernel(int n_rays, int S, int n_imp, const float *__restrict__ z_vals, const float *__restrict__ weights,
                                                                    const float *__restrict__ rays_o, const float *__restrict__ rays_d, const float *__restrict__ u_in,
                                                                    float *__restrict__ z_out, float *__restrict__ pts_out) {
    __shared__ float s_cdf[PDF_WARPS][PDF_MAX_S];
    __shared__ float s_bins[PDF_WARPS][PDF_MAX_S];
    __shared__ float s_z[PDF_WARPS][PDF_MAX_OUT];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int ray = blockIdx.x * PDF_WARPS + wid;
    if (ray >= n_rays) return;
    const float *z = z_vals + (size_t)ray * S, *w = weights + (size_t)ray * S;
    float *cdf = s_cdf[wid], *bins = s_bins[wid], *zz = s_z[wid];
    const int nb = S - 1;   // bins (mid-points): S-1 ; pdf entries: S-2 ; cdf entries: S-1
    float part = 0.f;
    for (int k = lane; k < S - 2; k += 32) part += w[k + 1] + 1e-5f;
    const float wsum_all = warp_sum(part);
    for (int k = lane; k < nb; k += 32) bins[k] = 0.5f * (z[k + 1] + z[k]);
    __syncwarp();
    if (lane == 0) {  // sequential cumsum like torch.cumsum on the reference's CPU path
        float c = 0.f; cdf[0] = 0.f;
        for (int k = 0; k < S - 2; ++k) { c += (w[k + 1] + 1e-5f) / wsum_all; cdf[k + 1] = c; }
    }
    __syncwarp();
    const int ncdf = S - 1;
    for (int j = lane; j < n_imp; j += 32) {
        // torch.linspace(0,1,n): step = 1/(n-1); second half computed from the end (ATen's symmetric formulation)
        float u;
        if (u_in) u = u_in[(size_t)ray * n_imp + j];
        else { float step = 1.0f / (float)(n_imp - 1); u = j < n_imp / 2 ? step * (float)j : 1.0f - step * (float)(n_imp - 1 - j); }
        int lo = 0, hi = ncdf;   // searchsorted(right=True): first index with cdf[idx] > u
        while (lo < hi) { int mid = (lo + hi) >> 1; if (cdf[mid] <= u) lo = mid + 1; else hi = mid; }
        int below = max(0, lo - 1), above = min(ncdf - 1, lo);
        float c0 = cdf[below], c1 = cdf[above], b0 = bins[below], b1 = bins[above];
        float denom = c1 - c0; if (denom < 1e-5f) denom = 1.f;
        float t = (u - c0) / denom;
        zz[S + j] = b0 + t * (b1 - b0);
    }
    for (int k = lane; k < S; k += 32) zz[k] = z[k];
    const int total = S + n_imp;
    int np2 = 1; while (np2 < total) np2 <<= 1;
    for (int k = total + lane; k < np2; k += 32) zz[k] = INFINITY;
    __syncwarp();
    for (int size = 2; size <= np2; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = lane; t < np2 / 2; t += 32) {
                int i = 2 * t - (t & (stride - 1)), j = i + stride;
                bool up = ((i & size) == 0);
                float a = zz[i], b = zz[j];
                if ((a > b) == up) { zz[i] = b; zz[j] = a; }
            }
            __syncwarp();
        }
    const float ox = rays_o[3 * (size_t)ray], oy = rays_o[3 * (size_t)ray + 1], oz = rays_o[3 * (size_t)ray + 2];
    const float dx = rays_d[3 * (size_t)ray], dy = rays_d[3 * (size_t)ray + 1], dz = rays_d[3 * (size_t)ray + 2];
    for (int k = lane; k < total; k += 32) {
        float v = zz[k];
        z_out[(size_t)ray * total + k] = v;
        if (pts_out) { float *pp = pts_out + ((size_t)ray * total + k) * 3; pp[0] = ox + dx * v; pp[1] = oy + dy * v; pp[2] = oz + dz * v; }
    }
}

// ---- NeRF / Mip-NeRF encodings. Each encoding column is written once below and used both by the fp32 kernels (one thread per output element of
// `embedded`) and by the generic tile-image kernels, so a tile image holds the fp16 roundings of exactly the fp32 kernels' values. The tile images
// (tc.cuh layout) are what the NerfMLP kernels TMA-load: per 128-row tile the point-encoding block(s), zero padded to 64 columns each, then the
// direction block.
// BaseEmbedder (embedders/base.py:26-52), column c of the encoding of x: x_c for c < 3, then per band b: sin(2^b x_a), cos(2^b x_a) for a = 0, 1, 2
__device__ __forceinline__ float posenc_col(const float *x, int c) {
    if (c < 3) return x[c];
    const int q = c - 3, band = q / 6, r = q % 6;
    const float y = x[r % 3] * exp2f((float)band);
    return r < 3 ? sinf(y) : cosf(y);
}
// MipNerfEmbedder (mipnerf_embedder.py:35-41, :55-60), IPE column c < c_ipe = 6 n_deg of a sample's Gaussian: exp(-0.5 cov_a 4^deg) sin(mean_a 2^deg),
// in the second half of the columns sin(mean_a 2^deg + pi/2)
__device__ __forceinline__ float ipe_col(const float *mean, const float *cov, int c, int c_ipe, int min_deg) {
    const int q = c < c_ipe / 2 ? c : c - c_ipe / 2, ax = q % 3;
    const float sc = exp2f((float)(q / 3 + min_deg));
    float y = sel3(mean, ax) * sc;
    const float yv = sel3(cov, ax) * sc * sc;
    if (c >= c_ipe / 2) y += HALF_PI;
    return expf(-0.5f * yv) * sinf(y);
}
// MipNerfEmbedder view-direction column c < 3 + 6 n_deg_v: vd_c for c < 3, then sin(2^deg vd_a), then sin(2^deg vd_a + pi/2)
__device__ __forceinline__ float mip_dir_col(const float *vd, int c, int n_deg_v, int min_deg_view) {
    if (c < 3) return vd[c];
    const int q = c - 3, halfn = 3 * n_deg_v, qq = q < halfn ? q : q - halfn;
    float x = vd[qq % 3] * exp2f((float)(qq / 3 + min_deg_view));
    if (q >= halfn) x += HALF_PI;
    return sinf(x);
}

// BaseEmbedder.forward (embedders/base.py:57-74): one thread per output element (coalesced row writes)
__global__ void __launch_bounds__(256) posenc_kernel(int64_t n_pts, int samples_per_ray, int multires, int multires_dirs, const float *__restrict__ pts,
                                                     const float *__restrict__ viewdirs, float *__restrict__ out) {
    const int c_pts = 3 + 6 * multires, c_dir = 3 + 6 * multires_dirs, C = c_pts + c_dir;
    const int64_t total = n_pts * C;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t i = idx / C; int c = (int)(idx - i * C);
        const float *src; int cc;
        if (c < c_pts) { src = pts + 3 * i; cc = c; } else { src = viewdirs + 3 * (i / samples_per_ray); cc = c - c_pts; }
        out[idx] = posenc_col(src, cc);
    }
}

// Mip-NeRF: cast_rays fused with MipNerfEmbedder.forward (embedders/mipnerf_embedder.py:43-99): one thread per output element of
// embedded[N*S, 6*n_deg + C_dir]. The Gaussians (means/covs) are recomputed per element in registers and optionally also written out (API parity: data['samples']).
__global__ void __launch_bounds__(256) mip_embed_kernel(int n_rays, int S, int min_deg, int max_deg, int min_deg_view, int max_deg_view, const float *__restrict__ z_vals,
                                                        const float *__restrict__ rays_o, const float *__restrict__ rays_d, const float *__restrict__ radii,
                                                        const float *__restrict__ viewdirs, float *__restrict__ embedded, float *__restrict__ means_out, float *__restrict__ covs_out) {
    const int n_deg = max_deg - min_deg, n_deg_v = max_deg_view - min_deg_view;
    const int c_ipe = 6 * n_deg, c_dir = 3 + 6 * n_deg_v, C = c_ipe + c_dir;
    const int64_t total = (int64_t)n_rays * S * C;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t row = idx / C; int c = (int)(idx - row * C);
        int ray = (int)(row / S), k = (int)(row - (int64_t)ray * S);
        float v;
        if (c < c_ipe) {
            float mean[3], cov[3];
            sample_gaussian(z_vals, rays_o, rays_d, radii, S, ray, k, mean, cov);
            v = ipe_col(mean, cov, c, c_ipe, min_deg);
            if (means_out && c < 3) { means_out[row * 3 + c] = sel3(mean, c); covs_out[row * 3 + c] = sel3(cov, c); }
        } else v = mip_dir_col(viewdirs + 3 * (size_t)ray, c - c_ipe, n_deg_v, min_deg_view);
        embedded[idx] = v;
    }
}

// ---- generic tile-image encoders: one thread per (row, 16-byte chunk) of every tile, fully coalesced 16-byte stores. Blocks 0..n_blk-2 hold the
// c_pts point columns, block n_blk-1 the c_dir direction columns. For a row < n_rows and a chunk holding n > 0 of its section's columns,
// enc(row, is_dir, k0, n, v) sets v[q] = column k0 + q of the section for q < n; every other value is zero.
template <class Enc>
__device__ __forceinline__ void write_tiles(int64_t n_rows, int n_blk, int c_pts, int c_dir, uint8_t *image, Enc enc) {
    const int chunks_per_row = n_blk * 8;
    const int64_t total = (n_rows + 127) / 128 * 128 * chunks_per_row;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = idx / chunks_per_row; const int cc = (int)(idx - row * chunks_per_row);
        const int blk = cc >> 3, ch = cc & 7;
        const bool is_dir = blk == n_blk - 1;
        const int k0 = (is_dir ? 0 : blk * 64) + ch * 8, n = (is_dir ? c_dir : c_pts) - k0;
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = 0.f;
        if (row < n_rows && n > 0) enc(row, is_dir, k0, n, v);
        st_chunk(tile_block(image, row >> 7, n_blk, blk) + sw128_offset((uint32_t)(row & 127), ch), pack_h8(v));
    }
}
// an fp32 embedded[n_rows, ic + icd] (any encoder's output) -> tile image
__global__ void __launch_bounds__(256) pack_embedded_tiles_kernel(const float *__restrict__ embedded, int64_t n_rows, int ic, int icd, int aux, uint8_t *__restrict__ image) {
    write_tiles(n_rows, aux + 1, ic, icd, image, [&](int64_t row, bool is_dir, int k0, int n, float *v) {
        const float *src = embedded + (size_t)row * (ic + icd) + (is_dir ? ic : 0) + k0;
#pragma unroll
        for (int q = 0; q < 8; ++q) if (q < n) v[q] = __ldg(src + q);
    });
}
// BaseEmbedder: pts f32[n,3], viewdirs f32[n/S,3]. Ray mode (rays_o != NULL): `pts` is z_vals f32[n_rays, S] and the sample position o + d*z is formed
// in registers (never materialised: 491 MB per 800x800 image in the reference)
__global__ void __launch_bounds__(256) posenc_tiles_kernel(const float *__restrict__ pts, const float *__restrict__ viewdirs, int64_t n_rows, int samples_per_ray, int multires,
                                                           int multires_dirs, uint8_t *__restrict__ image, const float *__restrict__ rays_o, const float *__restrict__ rays_d) {
    const int ic = 3 + 6 * multires;
    write_tiles(n_rows, (ic + 63) / 64 + 1, ic, 3 + 6 * multires_dirs, image, [&](int64_t row, bool is_dir, int k0, int n, float *v) {
        const int64_t ray = row / samples_per_ray;
        float p[3];
        const float *x = pts + 3 * row;
        if (is_dir) x = viewdirs + 3 * ray;
        else if (rays_o) { get_pts(rays_o, rays_d, ray, pts[row], p); x = p; }
#pragma unroll
        for (int q = 0; q < 8; ++q) if (q < n) v[q] = posenc_col(x, k0 + q);
    });
}
// Mip-NeRF cast_rays + IPE + view-direction encoding: no fp32 `embedded` [N*S,123] round trip (63 GB per 800x800 image in the reference); the frustum
// Gaussian is formed once per thread in registers
__global__ void __launch_bounds__(256) mip_ipe_tiles_kernel(int64_t n_rays, int S, int min_deg, int max_deg, int min_deg_view, int max_deg_view, const float *__restrict__ z_vals,
                                                            const float *__restrict__ rays_o, const float *__restrict__ rays_d, const float *__restrict__ radii,
                                                            const float *__restrict__ viewdirs, uint8_t *__restrict__ image) {
    const int n_deg = max_deg - min_deg, n_deg_v = max_deg_view - min_deg_view, c_ipe = 6 * n_deg;
    write_tiles(n_rays * S, (c_ipe + 63) / 64 + 1, c_ipe, 3 + 6 * n_deg_v, image, [&](int64_t row, bool is_dir, int k0, int n, float *v) {
        const int64_t ray = row / S; const int k = (int)(row - ray * S);
        if (is_dir) {
#pragma unroll
            for (int q = 0; q < 8; ++q) if (q < n) v[q] = mip_dir_col(viewdirs + 3 * ray, k0 + q, n_deg_v, min_deg_view);
        } else {
            float mean[3], cov[3];
            sample_gaussian(z_vals, rays_o, rays_d, radii, S, ray, k, mean, cov);
#pragma unroll
            for (int q = 0; q < 8; ++q) if (q < n) v[q] = ipe_col(mean, cov, k0 + q, c_ipe, min_deg);
        }
    });
}

// ---- fast tile-image encoders for the reference configurations (thread == (tile, encoding block, row): a warp works on 32 rows of ONE block
// kind, so there is no intra-warp divergence; every trig evaluation is shared by the columns that use it and all column indices are compile-time).
// The generic kernels above serve every other degree. Before these kernels existed (32768 rays on an H100):
// mip_ipe_tiles_kernel 4.29 ms per 4.2 M rows and posenc_tiles_kernel 1.92 ms per 6.3 M rows next to 8.46 ms of MLP.
// Mip-NeRF, 6*NDEG <= 128 point columns (two blocks) + direction block. item 0 = both point blocks of the row, item 1 = direction block.
// IPE column q (< 3*NDEG): exp(-0.5 * cov_ax * 4^deg) * sin(mean_ax * 2^deg), column 3*NDEG + q: the same with sin(y + pi/2) — the reference's
// expression, NOT cos(y): fl(y + pi/2) differs from y + pi/2 by up to ulp(y)/2 and the reference's value includes that (mipnerf_embedder.py:35-41,:55-60).
// |value| <= exp(-0.5 y_var) < 2^-25 rounds to (+-)0 in fp16, so the trig evaluation is skipped when 0.5 * y_var > 20.
template <int NDEG, int NDEGV>
__global__ void __launch_bounds__(256) mip_ipe_tiles_fast_kernel(int64_t n_rays, int S, int min_deg, int min_deg_view, const float *__restrict__ z_vals, const float *__restrict__ rays_o,
                                                                 const float *__restrict__ rays_d, const float *__restrict__ radii, const float *__restrict__ viewdirs, uint8_t *__restrict__ image) {
    static_assert(3 * NDEG % 8 == 0 && 6 * NDEG > 64 && 6 * NDEG <= 128 && 3 + 6 * NDEGV <= 64, "tile-image geometry");
    constexpr int HALF = 3 * NDEG, NJ = HALF / 8;
    const int64_t n_rows = n_rays * S, n_tiles = (n_rows + 127) / 128, total = n_tiles * 256;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(idx & 127); const int item = (int)((idx >> 7) & 1); const int64_t tile = idx >> 8;
        const int64_t row = tile * 128 + r;
        const bool live = row < n_rows;
        const uint32_t r7 = r & 7u;
        uint8_t *trow = sw128_row_ptr(tile_block(image, tile, 3, 0), r);   // my row inside block 0 of the tile
        const int64_t ray = live ? row / S : 0; const int k = (int)(row - ray * S);
        if (item == 0) {
            float mean[3] = {0.f, 0.f, 0.f}, cov[3] = {0.f, 0.f, 0.f};
            if (live) sample_gaussian(z_vals, rays_o, rays_d, radii, S, ray, k, mean, cov);
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                float sv[8], cv[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const int q = 8 * j + e, deg = q / 3, ax = q % 3;
                    const float sc = pow2i(deg + min_deg);
                    const float y = mean[ax] * sc, hv = 0.5f * (cov[ax] * sc * sc);
                    float s = 0.f, c = 0.f;
                    if (live && hv <= 20.f) { const float ex = expf(-hv); s = ex * sinf(y); c = ex * sinf(y + HALF_PI); }
                    sv[e] = s; cv[e] = c;
                }
                st_row_chunk(trow, r7, j, sv);                                          // columns 8j .. 8j+7 of block 0
                const int cs = HALF + 8 * j;                                                                     // first "cos" column of this group
                st_row_chunk(trow + (cs >> 6) * TILE_BLOCK_BYTES, r7, (uint32_t)(cs & 63) >> 3, cv);
            }
            const float z8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ch = (6 * NDEG - 64) / 8; ch < 8; ++ch) st_row_chunk(trow + TILE_BLOCK_BYTES, r7, ch, z8);   // zero padding of block 1
        } else {
            float v[64];
#pragma unroll
            for (int e = 0; e < 64; ++e) v[e] = 0.f;
            if (live) {
                const float vd[3] = {viewdirs[3 * ray], viewdirs[3 * ray + 1], viewdirs[3 * ray + 2]};
                mip_dir_bands(vd, min_deg_view, NDEGV, [&](int c, float y) { v[c] = y; });
            }
#pragma unroll
            for (int ch = 0; ch < 8; ++ch) st_row_chunk(trow + 2 * TILE_BLOCK_BYTES, r7, ch, v + 8 * ch);
        }
    }
}

// BaseEmbedder (embedders/base.py:26-52), 3 + 6*LP <= 64 point columns (one block) + direction block; item 0 = point block, item 1 = direction block.
// column 3 + 6b + a = sin(2^b x_a), column 3 + 6b + 3 + a = cos(2^b x_a). ray mode as posenc_tiles_kernel (rays_o != NULL: `pts` is z_vals).
template <int LP, int LD>
__global__ void __launch_bounds__(256) posenc_tiles_fast_kernel(const float *__restrict__ pts, const float *__restrict__ viewdirs, int64_t n_rows, int samples_per_ray,
                                                                uint8_t *__restrict__ image, const float *__restrict__ rays_o, const float *__restrict__ rays_d) {
    static_assert(3 + 6 * LP <= 64 && 3 + 6 * LD <= 64, "one block each");
    const int64_t n_tiles = (n_rows + 127) / 128, total = n_tiles * 256;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(idx & 127); const int item = (int)((idx >> 7) & 1); const int64_t tile = idx >> 8;
        const int64_t row = tile * 128 + r;
        const bool live = row < n_rows;
        uint8_t *trow = tile_block(image, tile, 2, item) + sw128_row(r);
        float v[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) v[e] = 0.f;
        if (live) {
            float x[3];
            const int64_t ray = row / samples_per_ray;
            if (item == 1) { x[0] = viewdirs[3 * ray]; x[1] = viewdirs[3 * ray + 1]; x[2] = viewdirs[3 * ray + 2]; }
            else if (rays_o) get_pts(rays_o, rays_d, ray, pts[row], x);
            else { x[0] = pts[3 * row]; x[1] = pts[3 * row + 1]; x[2] = pts[3 * row + 2]; }
#pragma unroll
            for (int a = 0; a < 3; ++a) v[a] = x[a];
            if (item == 0) posenc_bands<LP>(x, v);
            else posenc_bands<LD>(x, v);
        }
#pragma unroll
        for (int ch = 0; ch < 8; ++ch) st_chunk(trow + sw128_chunk(r, ch), pack_h8(v + 8 * ch));
    }
}

// Mip-NeRF point query at a footprint (mesh export): ipe_point_bands of pts into point blocks 0 and 1, and MipNerfEmbedder.pos_enc of the view
// direction into block 2 with the expressions of mip_ipe_tiles_fast_kernel's direction block. thread == (tile, item, row) as in the fast encoders:
// item 0 = both point blocks of the row, item 1 = the direction block. The degrees are run-time values, so the row is zeroed with 16-byte stores and
// each column is then stored as fp16 (the rounding of pack_h8).
__global__ void __launch_bounds__(256) mip_ipe_tiles_points_kernel(const float *__restrict__ pts, const float *__restrict__ viewdirs, int64_t n_rows, int samples_per_ray,
                                                                   const __grid_constant__ IpeBands B, int min_deg_view, int n_deg_view, uint8_t *__restrict__ image) {
    const int64_t n_tiles = (n_rows + 127) / 128, total = n_tiles * 256;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(idx & 127); const int item = (int)((idx >> 7) & 1); const int64_t tile = idx >> 8;
        const int64_t row = tile * 128 + r;
        uint8_t *blk = tile_block(image, tile, 3, item == 0 ? 0 : 2);
        for (int b = 0; b < (item == 0 ? 2 : 1); ++b)
#pragma unroll
            for (int ch = 0; ch < 8; ++ch) st_chunk(blk + b * TILE_BLOCK_BYTES + sw128_offset(r, ch), make_uint4(0u, 0u, 0u, 0u));
        if (row >= n_rows) continue;
        auto put = [&](int c, float y) { *reinterpret_cast<__half *>(sw128_elem(blk + (c >> 6) * TILE_BLOCK_BYTES, r, (uint32_t)(c & 63))) = __float2half_rn(y); };
        if (item == 0) {
            const float x[3] = {pts[3 * row], pts[3 * row + 1], pts[3 * row + 2]};
            ipe_point_bands(x, B, put);
        } else {
            const int64_t ray = row / samples_per_ray;
            const float vd[3] = {viewdirs[3 * ray], viewdirs[3 * ray + 1], viewdirs[3 * ray + 2]};
            mip_dir_bands(vd, min_deg_view, n_deg_view, put);
        }
    }
}

// The gradient with respect to the position through a point encoding (mesh normals of a NerfMLP), one thread per point: BaseEmbedder's
// (posenc_bands_grad, multires <= 10, one point block) or, when MIP, the point query's IPE (ipe_point_bands_grad, two point blocks). The gradient with
// respect to the encoding, e, is the sum of the n_terms fp16 terms of d_enc (term t = point blocks P t .. P t + P - 1 of every tile: the input
// gradients of the layers that read the point encoding) divided by the staging scale. enc_grad_read forms entries of e; NeRF reads its whole row with
// 16-byte loads, Mip-NeRF reads each entry where it is needed (its columns are run-time values).
template <int P, int W>
__device__ __forceinline__ void enc_grad_read(const uint8_t *d_enc, int n_terms, int64_t i, int c0, float inv, float *e) {
    static_assert(W == 1 || W == 64, "one entry or a whole block row");
    const uint32_t r = (uint32_t)(i & 127);
#pragma unroll
    for (int c = 0; c < W; ++c) e[c] = 0.f;
    for (int t = 0; t < n_terms; ++t) {
        const uint8_t *blk = tile_block(const_cast<uint8_t *>(d_enc), i >> 7, P * n_terms, P * t + (c0 >> 6));
        if constexpr (W == 1) e[0] += __half2float(__ldg(reinterpret_cast<const __half *>(sw128_elem(blk, r, (uint32_t)(c0 & 63)))));
        else {
#pragma unroll
            for (int ch = 0; ch < 8; ++ch) {
                const uint4 q = __ldg(reinterpret_cast<const uint4 *>(blk + sw128_offset(r, ch)));
                const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[j]));
                    e[8 * ch + 2 * j] += f.x; e[8 * ch + 2 * j + 1] += f.y;
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < W; ++c) e[c] *= inv;
}
template <bool MIP>
__global__ void __launch_bounds__(256) point_enc_grad_kernel(const float *__restrict__ pts, int64_t n_pts, int multires, const __grid_constant__ IpeBands B,
                                                             const uint8_t *__restrict__ d_enc, int n_terms, const float *__restrict__ scale, float *__restrict__ grad) {
    const float inv = 1.f / *scale;   // a power of two: exact
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_pts; i += (int64_t)gridDim.x * blockDim.x) {
        const float x[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        float g[3];
        if constexpr (MIP) {
            ipe_point_bands_grad(x, B, [&](int c) { float v; enc_grad_read<2, 1>(d_enc, n_terms, i, c, inv, &v); return v; }, g);
        } else {
            float e[64];
            enc_grad_read<1, 64>(d_enc, n_terms, i, 0, inv, e);
            posenc_bands_grad<10>(x, multires, [&](int c) { return e[c]; }, g);
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) grad[3 * i + a] = g[a];
    }
}

// Mip-NeRF resample_along_rays + sorted_piecewise_constant_pdf (networks/utils/mip.py:146-176, :7-63), randomized=False or
// caller-supplied jitter: one warp per ray, O(S log S) interval search instead of the reference's [N,S+2,S+1] mask.
constexpr int MIP_MAX_S = 256;
__global__ void __launch_bounds__(PDF_WARPS * 32) mip_resample_kernel(int n_rays, int S, float resample_padding, const float *__restrict__ z_vals, const float *__restrict__ weights,
                                                                      const float *__restrict__ u_in, float *__restrict__ z_out) {
    __shared__ float s_w[PDF_WARPS][MIP_MAX_S + 2];
    __shared__ float s_cdf[PDF_WARPS][MIP_MAX_S + 2];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int ray = blockIdx.x * PDF_WARPS + wid;
    if (ray >= n_rays) return;
    const float *z = z_vals + (size_t)ray * (S + 1), *w_in = weights + (size_t)ray * S;
    float *w = s_w[wid], *cdf = s_cdf[wid];
    // blur: pad, pairwise max, pairwise mean, + padding constant (mip.py:154-163)
    float part = 0.f;
    for (int k = lane; k < S; k += 32) {
        float wm1 = w_in[max(k - 1, 0)], w0 = w_in[k], wp1 = w_in[min(k + 1, S - 1)];
        float v = 0.5f * (fmaxf(wm1, w0) + fmaxf(w0, wp1)) + resample_padding;
        w[k] = v; part += v;
    }
    float wsum_all = warp_sum(part);
    const float eps = 1e-5f;
    float padding = fmaxf(0.f, eps - wsum_all);
    const float add = padding / (float)S;
    wsum_all += padding;
    __syncwarp();
    if (lane == 0) {
        float c = 0.f; cdf[0] = 0.f;
        for (int k = 0; k < S - 1; ++k) { c += (w[k] + add) / wsum_all; cdf[k + 1] = fminf(1.f, c); }
        cdf[S] = 1.f;
    }
    __syncwarp();
    const int num = S + 1;   // samples drawn == len(z_vals)
    for (int j = lane; j < num; j += 32) {
        float u;
        if (u_in) u = u_in[(size_t)ray * num + j];
        else { const float end = 1.f - 1.1920929e-07f; float step = end / (float)(num - 1); u = j < num / 2 ? step * (float)j : end - step * (float)(num - 1 - j); }
        int lo = 0, hi = num;   // first index with cdf[idx] > u  (cdf has S+1 entries; cdf[0]=0 <= u always)
        while (lo < hi) { int mid = (lo + hi) >> 1; if (cdf[mid] <= u) lo = mid + 1; else hi = mid; }
        int i0 = lo - 1, i1 = lo < num ? lo : num - 1;
        float c0 = cdf[i0], c1 = cdf[i1], b0 = z[i0], b1 = z[i1];
        float t = (u - c0) / (c1 - c0);
        if (isnan(t)) t = 0.f;
        t = fminf(fmaxf(t, 0.f), 1.f);
        z_out[(size_t)ray * num + j] = b0 + t * (b1 - b0);
    }
}


// Ray generation (SURVEY §8 a1-a3): GetRays (+ Mip-NeRF radii) + GetViewdirs (datasets/pipelines/create.py:205-245, :437-448) and the
// NGP-convention get_rays_np_hash (datasets/load_data/get_rays.py:35-69), one thread per pixel, any pixel subset.
//   convention 0 (NeRF / Mip): dirs = ((i-cx)/fx, -(j-cy)/fy, -1), rays_d = c2w[:3,:3] dirs, viewdirs = rays_d/|rays_d|,
//                              radii = |rays_d(j,i) - rays_d(j+1,i)| * 2/sqrt(12) (last row reuses row H-3, create.py:237-243)
//   convention 1 (NGP):        pixel centres +0.5, dirs = ((i-cx)/fx, (j-cy)/fy, 1), rays_d normalised, pose given as [4,3] (ngp xforms)
struct RayGenParams { float c2w[12]; float fx, fy, cx, cy; int H, W, convention; };
__device__ __forceinline__ void raygen_dir(const RayGenParams &p, float i, float j, float d[3]) {
    float x, y, z;
    if (p.convention == 0) { x = (i - p.cx) / p.fx; y = -(j - p.cy) / p.fy; z = -1.f; }
    else { x = (i + 0.5f - p.cx) / p.fx; y = (j + 0.5f - p.cy) / p.fy; z = 1.f; }
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = (x * p.c2w[4 * c] + y * p.c2w[4 * c + 1]) + z * p.c2w[4 * c + 2];
}
// The NGP training-ray source on the device (SURVEY §8f-1): what HashNerfDataset + HashBatchSample + RandomBGColor produce on the host
//   load_rays_hash (datasets/load_data/get_rays.py:72-98): row r of the [I*H*W, 11] table = (rays_o3, rays_d3 by get_rays_np_hash, rgba4, image id) of pixel r % (H*W) of image r / (H*W)
//   the table shuffle (hashnerf_dataset.py:41-44) = the caller's row permutation; HashBatchSample (create.py:153-190) = a slice of it
//   RandomBGColor (augment.py:290-313): bg = U[0,1)^3, target = rgb * alpha + bg * (1 - alpha) (float64 on the host, rounded to fp32)
// without the 2.8 GB host table: one thread per ray regenerates its row from (pose, pixel) and blends the background.
// pixel `row` of the virtual [I*H*W] table of an NGP batch: its image and its pixel in the image
__device__ __forceinline__ void ngp_pixel(int64_t row, int64_t hw, int &img, int &pix) { img = (int)(row / hw); pix = (int)(row % hw); }
// the camera-frame direction (x, y, 1) through the centre of pixel `pix` of a W-wide image (get_rays.py:35-69)
__device__ __forceinline__ void ngp_pixel_dir(int pix, int W, float fx, float fy, float cx, float cy, float &x, float &y) {
    const int j = pix / W, i = pix % W;
    x = ((float)i + 0.5f - cx) / fx; y = ((float)j + 0.5f - cy) / fy;
}

__global__ void __launch_bounds__(256) ngp_batch_sample_kernel(const float *__restrict__ poses, const float *__restrict__ images, int n_img, int H, int W, float fx, float fy, float cx,
                                                               float cy, const int64_t *__restrict__ row_idx, int64_t n, const float *__restrict__ u_bg, Pcg32 rng,
                                                               float *__restrict__ rays_o, float *__restrict__ rays_d, float *__restrict__ target_s, float *__restrict__ alpha_out,
                                                               float *__restrict__ img_ids, float *__restrict__ bg_color) {
    const int64_t hw = (int64_t)H * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        int img, pix; float x, y;
        ngp_pixel(row_idx[t], hw, img, pix);
        const float *P = poses + (size_t)img * 12;                 // [4,3]: rows 0..2 = rotation columns (c2w = P^T), row 3 = camera origin
        ngp_pixel_dir(pix, W, fx, fy, cx, cy, x, y);
        float d[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = (x * P[c] + y * P[3 + c]) + P[6 + c];
        const float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        const float4 px = *reinterpret_cast<const float4 *>(images + ((size_t)img * hw + pix) * 4);
        float u[3];
        if (u_bg) { u[0] = u_bg[3 * t]; u[1] = u_bg[3 * t + 1]; u[2] = u_bg[3 * t + 2]; }
        else { Pcg32 r = rng; r.advance((uint64_t)t * 3u); u[0] = r.next_float(); u[1] = r.next_float(); u[2] = r.next_float(); }
        const float rgb[3] = {px.x, px.y, px.z};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            rays_o[3 * t + c] = P[9 + c];
            rays_d[3 * t + c] = d[c] / nrm;
            target_s[3 * t + c] = (float)((double)(rgb[c] * px.w) + (double)u[c] * (double)(1.f - px.w));
            bg_color[3 * t + c] = u[c];
        }
        alpha_out[t] = px.w;
        img_ids[t] = (float)img;
    }
}

// target depth of an NGP batch: the z-depth of the pixel (along the optical axis) as the ray parameter of the unit-direction NGP ray, t = scale z |(x, y, 1)|
__global__ void __launch_bounds__(256) ngp_batch_depth_kernel(const float *__restrict__ depths, int H, int W, float fx, float fy, float cx, float cy, float scale,
                                                              const int64_t *__restrict__ row_idx, int64_t n, float *__restrict__ target_depth) {
    const int64_t hw = (int64_t)H * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        int img, pix; float x, y;
        ngp_pixel(row_idx[t], hw, img, pix);
        ngp_pixel_dir(pix, W, fx, fy, cx, cy, x, y);
        target_depth[t] = scale * depths[(size_t)img * hw + pix] * sqrtf(x * x + y * y + 1.f);
    }
}

// NGP camera pose refinement (xrb_ngp_pose_grad): dL/d(rays_o, unit rays_d) of each batch ray -> dL/dP' [I,4,3] of the corrected poses it was generated
// from (ngp_batch_sample_kernel's ray generation, differentiated): d~ = R' (x, y, 1), dL/dd~ = (I - d^ d^T) grad_d / |d~|; row r < 3 of P' gets
// dL/dd~ (x, y, 1)[r], row 3 gets grad_o. SHARED: each block sums into shared memory [I x 12] and adds its non-zero entries to the output; otherwise each
// warp adds, per distinct image among its rays, one warp-reduced sum per entry with a global atomic.
constexpr int POSE_GRAD_SMEM_MAX = 48 * 1024;
template <bool SHARED>
__global__ void __launch_bounds__(256) ngp_pose_grad_kernel(const int64_t *__restrict__ row_idx, int64_t n, int n_img, int H, int W, float fx, float fy, float cx, float cy,
                                                            const float *__restrict__ poses, const float *__restrict__ grad_o, const float *__restrict__ grad_d,
                                                            float *__restrict__ d_poses) {
    extern __shared__ float s_acc[];
    if (SHARED) {
        for (int k = threadIdx.x; k < n_img * 12; k += blockDim.x) s_acc[k] = 0.f;
        __syncthreads();
    }
    const int64_t hw = (int64_t)H * W;
    const int lane = threadIdx.x & 31;
    for (int64_t t0 = (int64_t)blockIdx.x * blockDim.x; t0 < n; t0 += (int64_t)gridDim.x * blockDim.x) {   // uniform per block: every lane takes part in the warp sums
        const int64_t t = t0 + threadIdx.x;
        const bool valid = t < n;
        float v[12];
        int img = -1;
        if (valid) {
            int pix; float x, y;
            ngp_pixel(row_idx[t], hw, img, pix);
            ngp_pixel_dir(pix, W, fx, fy, cx, cy, x, y);
            const float *P = poses + (size_t)img * 12;
            float d[3], g[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) { d[c] = (x * P[c] + y * P[3 + c]) + P[6 + c]; g[c] = grad_d[3 * t + c]; }
            const float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), inv = 1.f / nrm;
            const float u[3] = {d[0] * inv, d[1] * inv, d[2] * inv}, ug = u[0] * g[0] + u[1] * g[1] + u[2] * g[2];
            const float in[3] = {x, y, 1.f};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float gd = (g[c] - u[c] * ug) * inv;   // dL/dd~
#pragma unroll
                for (int r = 0; r < 3; ++r) v[3 * r + c] = gd * in[r];
                v[9 + c] = grad_o[3 * t + c];
            }
        } else {
#pragma unroll
            for (int k = 0; k < 12; ++k) v[k] = 0.f;
        }
        if (SHARED) {
            if (valid) {
#pragma unroll
                for (int k = 0; k < 12; ++k) atomicAdd(s_acc + 12 * img + k, v[k]);
            }
        } else {
            unsigned pending = __ballot_sync(0xffffffffu, valid);
            while (pending) {   // one round per distinct image among the warp's rays
                const int leader = __ffs(pending) - 1, mine = __shfl_sync(0xffffffffu, img, leader);
                const bool in_group = valid && img == mine;
                pending &= ~__ballot_sync(0xffffffffu, in_group);
#pragma unroll
                for (int k = 0; k < 12; ++k) {
                    const float sum = warp_sum(in_group ? v[k] : 0.f);
                    if (lane == leader) atomicAdd(d_poses + 12 * (size_t)mine + k, sum);
                }
            }
        }
    }
    if (SHARED) {
        __syncthreads();
        for (int k = threadIdx.x; k < n_img * 12; k += blockDim.x)
            if (s_acc[k] != 0.f) atomicAdd(d_poses + k, s_acc[k]);
    }
}

__global__ void __launch_bounds__(256) get_rays_kernel(RayGenParams p, const int32_t *__restrict__ pixel_idx, int64_t n, float *__restrict__ rays_o, float *__restrict__ rays_d,
                                                       float *__restrict__ viewdirs, float *__restrict__ radii) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int pix = pixel_idx ? pixel_idx[t] : (int)t;
        const int j = pix / p.W, i = pix % p.W;
        float d[3]; raygen_dir(p, (float)i, (float)j, d);
        const float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        if (p.convention == 1) { d[0] /= nrm; d[1] /= nrm; d[2] /= nrm; }
#pragma unroll
        for (int c = 0; c < 3; ++c) { rays_o[3 * t + c] = p.c2w[4 * c + 3]; rays_d[3 * t + c] = d[c]; if (viewdirs) viewdirs[3 * t + c] = p.convention == 1 ? d[c] : d[c] / nrm; }
        if (radii) {
            const int ja = j < p.H - 1 ? j : p.H - 3;   // dx = cat([dx, dx[-2:-1]]): the last row takes dx of row H-3
            float a[3], b[3]; raygen_dir(p, (float)i, (float)ja, a); raygen_dir(p, (float)i, (float)(ja + 1), b);
            const float dx = sqrtf((a[0] - b[0]) * (a[0] - b[0]) + (a[1] - b[1]) * (a[1] - b[1]) + (a[2] - b[2]) * (a[2] - b[2]));
            radii[t] = dx * 2.f / sqrtf(12.f);
        }
    }
}
// GetZvals (create.py:502-531, randomized=False) + PerturbZvals (augment.py:269-283) when u != NULL: one thread per (ray, sample)
__global__ void __launch_bounds__(256) zvals_kernel(int64_t n_rays, int S, float near_, float far_, int lindisp, const float *__restrict__ u, float *__restrict__ z_out) {
    const float step = 1.0f / (float)(S - 1);
    auto zat = [&](int k) { float t = k < S / 2 ? step * (float)k : 1.0f - step * (float)(S - 1 - k);   // torch.linspace
                            return lindisp ? 1.f / (1.f / near_ * (1.f - t) + 1.f / far_ * t) : near_ * (1.f - t) + far_ * t; };
    const int64_t total = n_rays * S;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(idx % S);
        float z = zat(k);
        if (u) {
            float lower = k == 0 ? z : 0.5f * (z + zat(k - 1)), upper = k == S - 1 ? z : 0.5f * (zat(k + 1) + z);
            z = lower + (upper - lower) * u[idx];
        }
        z_out[idx] = z;
    }
}

}  // namespace xrb

using namespace xrb;

extern "C" {

static int composite_args_ok(const float *raw, const float *z, const float *d, int n_rays, int n_samples, int density_act) {
    if (n_rays < 0 || n_samples < 1) { set_error("nerf_composite: bad size"); return XRB_E_BADARG; }
    if (!(density_act == XRB_ACT_RELU || density_act == XRB_ACT_SOFTPLUS)) { set_error("nerf_composite: density activation must be relu(1) or softplus(4)"); return XRB_E_UNSUPPORTED; }
    if (n_rays && (!raw || !z || !d)) { set_error("nerf_composite: null pointer"); return XRB_E_BADARG; }
    if (((uintptr_t)raw & 15) != 0) { set_error("nerf_composite: raw must be 16-byte aligned"); return XRB_E_BADARG; }
    return XRB_OK;
}

int xrb_nerf_composite_forward(const float *raw, const float *z_vals, const float *rays_d, int n_rays, int n_samples, int mip, int white_bkgd, float rgb_padding, float density_bias,
                               int density_act, float *rgb, float *disp, float *acc, float *weights, void *stream) {
    int e = composite_args_ok(raw, z_vals, rays_d, n_rays, n_samples, density_act); if (e) return e;
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(rgb && disp && acc && weights, "nerf_composite_forward: null output");
    CompositeParams p{n_rays, n_samples, mip, white_bkgd, density_act, rgb_padding, density_bias};
    int blocks = (int)(((size_t)n_rays * 32 + 255) / 256);
    nerf_composite_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(p, raw, z_vals, rays_d, nullptr, rgb, disp, acc, weights, nullptr, nullptr, nullptr, nullptr);
    return check_launch("nerf_composite_forward");
}

int xrb_nerf_composite_forward_depth(const float *raw, const float *z_vals, const float *rays_d, int n_rays, int n_samples, int mip, int white_bkgd, float rgb_padding,
                                     float density_bias, int density_act, float *rgb, float *disp, float *acc, float *weights, float *depth, void *stream) {
    int e = composite_args_ok(raw, z_vals, rays_d, n_rays, n_samples, density_act); if (e) return e;
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(rgb && disp && acc && weights && depth, "nerf_composite_forward_depth: null output");
    CompositeParams p{n_rays, n_samples, mip, white_bkgd, density_act, rgb_padding, density_bias};
    int blocks = (int)(((size_t)n_rays * 32 + 255) / 256);
    nerf_composite_kernel<false, true><<<blocks, 256, 0, (cudaStream_t)stream>>>(p, raw, z_vals, rays_d, nullptr, rgb, disp, acc, weights, nullptr, depth, nullptr, nullptr);
    return check_launch("nerf_composite_forward_depth");
}

int xrb_nerf_composite_backward(const float *raw, const float *z_vals, const float *rays_d, const float *grad_rgb, int n_rays, int n_samples, int mip, int white_bkgd, float rgb_padding,
                                float density_bias, int density_act, float *d_raw, void *stream) {
    int e = composite_args_ok(raw, z_vals, rays_d, n_rays, n_samples, density_act); if (e) return e;
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(grad_rgb && d_raw && ((uintptr_t)d_raw & 15) == 0, "nerf_composite_backward: null/misaligned pointer");
    CompositeParams p{n_rays, n_samples, mip, white_bkgd, density_act, rgb_padding, density_bias};
    int blocks = (int)(((size_t)n_rays * 32 + 255) / 256);
    nerf_composite_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(p, raw, z_vals, rays_d, grad_rgb, nullptr, nullptr, nullptr, nullptr, d_raw, nullptr, nullptr, nullptr);
    return check_launch("nerf_composite_backward");
}

int xrb_nerf_composite_backward_geom(const float *raw, const float *z_vals, const float *rays_d, const float *grad_rgb, const float *grad_depth, const float *grad_acc,
                                     int n_rays, int n_samples, int mip, int white_bkgd, float rgb_padding, float density_bias, int density_act, float *d_raw, void *stream) {
    int e = composite_args_ok(raw, z_vals, rays_d, n_rays, n_samples, density_act); if (e) return e;
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(grad_rgb && d_raw && ((uintptr_t)d_raw & 15) == 0, "nerf_composite_backward_geom: null/misaligned pointer");
    CompositeParams p{n_rays, n_samples, mip, white_bkgd, density_act, rgb_padding, density_bias};
    int blocks = (int)(((size_t)n_rays * 32 + 255) / 256);
    nerf_composite_kernel<true, false, true><<<blocks, 256, 0, (cudaStream_t)stream>>>(p, raw, z_vals, rays_d, grad_rgb, nullptr, nullptr, nullptr, nullptr, d_raw, nullptr,
                                                                                       grad_depth, grad_acc);
    return check_launch("nerf_composite_backward_geom");
}

int xrb_nerf_sample_pdf(const float *z_vals, const float *weights, const float *rays_o, const float *rays_d, const float *u, int n_rays, int n_samples, int n_importance, float *z_out,
                        float *pts_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && n_samples >= 3 && n_importance >= 2, "sample_pdf: bad size");
    if (n_samples > PDF_MAX_S || n_samples + n_importance > PDF_MAX_OUT) { set_error("sample_pdf: n_samples<=256 and n_samples+n_importance<=512 supported"); return XRB_E_UNSUPPORTED; }
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(z_vals && weights && rays_o && rays_d && z_out, "sample_pdf: null pointer");
    sample_pdf_kernel<<<(n_rays + PDF_WARPS - 1) / PDF_WARPS, PDF_WARPS * 32, 0, (cudaStream_t)stream>>>(n_rays, n_samples, n_importance, z_vals, weights, rays_o, rays_d, u, z_out, pts_out);
    return check_launch("sample_pdf");
}

int xrb_nerf_posenc(const float *pts, const float *viewdirs, int64_t n_pts, int samples_per_ray, int multires, int multires_dirs, float *embedded, void *stream) {
    XRB_REQUIRE(n_pts >= 0 && samples_per_ray >= 1 && multires >= 0 && multires_dirs >= 0, "posenc: bad size");
    if (n_pts == 0) return XRB_OK;
    XRB_REQUIRE(pts && viewdirs && embedded, "posenc: null pointer");
    int64_t total = n_pts * (6 + 6 * (int64_t)(multires + multires_dirs));
    const int blocks = stride_grid((total + 255) / 256, 16);
    posenc_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n_pts, samples_per_ray, multires, multires_dirs, pts, viewdirs, embedded);
    return check_launch("posenc");
}

int xrb_mip_embed(const float *z_vals, const float *rays_o, const float *rays_d, const float *radii, const float *viewdirs, int n_rays, int n_samples, int min_deg_point,
                  int max_deg_point, int min_deg_view, int max_deg_view, float *embedded, float *means_out, float *covs_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && n_samples >= 1 && max_deg_point > min_deg_point && max_deg_view >= min_deg_view, "mip_embed: bad size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(z_vals && rays_o && rays_d && radii && viewdirs && embedded && ((means_out == nullptr) == (covs_out == nullptr)), "mip_embed: null pointer");
    int64_t total = (int64_t)n_rays * n_samples * (6 * (max_deg_point - min_deg_point) + 3 + 6 * (max_deg_view - min_deg_view));
    const int blocks = stride_grid((total + 255) / 256, 16);
    mip_embed_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n_rays, n_samples, min_deg_point, max_deg_point, min_deg_view, max_deg_view, z_vals, rays_o, rays_d, radii, viewdirs, embedded,
                                                                   means_out, covs_out);
    return check_launch("mip_embed");
}

// grid of a tile-image encoder launch with `per_tile` threads per 128-row tile (generic kernels: 128 x 8 per block, fast kernels: 256)
static int tile_grid(int64_t n_rows, int64_t per_tile) { return stride_grid(((n_rows + 127) / 128 * per_tile + 255) / 256, 16); }

int xrb_mip_ipe_tiles_rays(const float *z_vals, const float *rays_o, const float *rays_d, const float *radii, const float *viewdirs, int64_t n_rays, int n_samples, int min_deg_point,
                           int max_deg_point, int min_deg_view, int max_deg_view, void *enc_image, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && n_samples >= 1 && max_deg_point > min_deg_point && max_deg_view >= min_deg_view, "mip_ipe_tiles_rays: bad size");
    XRB_REQUIRE(6 * (max_deg_point - min_deg_point) <= 128 && 3 + 6 * (max_deg_view - min_deg_view) <= 64, "mip_ipe_tiles_rays: encoding wider than the tile image (128 + 64 columns)");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(z_vals && rays_o && rays_d && radii && viewdirs && enc_image && ((uintptr_t)enc_image & 15) == 0, "mip_ipe_tiles_rays: null/misaligned pointer");
    const int64_t n_rows = n_rays * n_samples;
    const cudaStream_t s = (cudaStream_t)stream;
    if (max_deg_point - min_deg_point == 16 && max_deg_view - min_deg_view == 4 && min_deg_point >= -100 && max_deg_point <= 100 && min_deg_view >= -100 && max_deg_view <= 100)
        // the reference configuration (configs/mipnerf/*.py): specialised kernel
        mip_ipe_tiles_fast_kernel<16, 4><<<tile_grid(n_rows, 256), 256, 0, s>>>(n_rays, n_samples, min_deg_point, min_deg_view, z_vals, rays_o, rays_d, radii, viewdirs, (uint8_t *)enc_image);
    else
        mip_ipe_tiles_kernel<<<tile_grid(n_rows, 128 * 8 * ((6 * (max_deg_point - min_deg_point) + 63) / 64 + 1)), 256, 0, s>>>(n_rays, n_samples, min_deg_point, max_deg_point, min_deg_view,
                                                                                                                          max_deg_view, z_vals, rays_o, rays_d, radii, viewdirs, (uint8_t *)enc_image);
    return check_launch("mip_ipe_tiles_rays");
}

size_t xrb_nerf_enc_image_bytes(int64_t n_rows, int input_ch) { return tile_image_bytes(n_rows, (input_ch + 63) / 64 + 1); }

int xrb_nerf_pack_embedded(const float *embedded, int64_t n_rows, int input_ch, int input_ch_dirs, void *enc_image, void *stream) {
    XRB_REQUIRE(n_rows >= 0 && input_ch >= 1 && input_ch <= 128 && input_ch_dirs >= 0 && input_ch_dirs <= 64, "nerf_pack_embedded: bad size");
    if (n_rows == 0) return XRB_OK;
    XRB_REQUIRE(embedded && enc_image && ((uintptr_t)enc_image & 15) == 0, "nerf_pack_embedded: null/misaligned pointer");
    const int aux = (input_ch + 63) / 64;
    pack_embedded_tiles_kernel<<<tile_grid(n_rows, 128 * 8 * (aux + 1)), 256, 0, (cudaStream_t)stream>>>(embedded, n_rows, input_ch, input_ch_dirs, aux, (uint8_t *)enc_image);
    return check_launch("nerf_pack_embedded");
}

// positional encoding into a tile image; ray mode when rays_o != NULL (`pts` is then z_vals). The reference configuration multires = 10,
// multires_dirs = 4 takes the specialised kernel.
static int posenc_tiles(const float *pts, const float *viewdirs, int64_t n_rows, int samples_per_ray, int multires, int multires_dirs, void *enc_image, const float *rays_o,
                        const float *rays_d, void *stream, const char *what) {
    const cudaStream_t s = (cudaStream_t)stream;
    if (multires == 10 && multires_dirs == 4)
        posenc_tiles_fast_kernel<10, 4><<<tile_grid(n_rows, 256), 256, 0, s>>>(pts, viewdirs, n_rows, samples_per_ray, (uint8_t *)enc_image, rays_o, rays_d);
    else
        posenc_tiles_kernel<<<tile_grid(n_rows, 128 * 8 * ((3 + 6 * multires + 63) / 64 + 1)), 256, 0, s>>>(pts, viewdirs, n_rows, samples_per_ray, multires, multires_dirs,
                                                                                                          (uint8_t *)enc_image, rays_o, rays_d);
    return check_launch(what);
}

int xrb_nerf_posenc_tiles(const float *pts, const float *viewdirs, int64_t n_pts, int samples_per_ray, int multires, int multires_dirs, void *enc_image, void *stream) {
    XRB_REQUIRE(n_pts >= 0 && samples_per_ray >= 1 && multires >= 0 && multires <= 20 && multires_dirs >= 0 && multires_dirs <= 10, "nerf_posenc_tiles: bad size");
    if (n_pts == 0) return XRB_OK;
    XRB_REQUIRE(pts && viewdirs && enc_image && ((uintptr_t)enc_image & 15) == 0, "nerf_posenc_tiles: null/misaligned pointer");
    return posenc_tiles(pts, viewdirs, n_pts, samples_per_ray, multires, multires_dirs, enc_image, nullptr, nullptr, stream, "nerf_posenc_tiles");
}

int xrb_nerf_posenc_tiles_rays(const float *rays_o, const float *rays_d, const float *z_vals, const float *viewdirs, int64_t n_rays, int samples_per_ray, int multires, int multires_dirs,
                               void *enc_image, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && samples_per_ray >= 1 && multires >= 0 && multires <= 20 && multires_dirs >= 0 && multires_dirs <= 10, "nerf_posenc_tiles_rays: bad size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(rays_o && rays_d && z_vals && viewdirs && enc_image && ((uintptr_t)enc_image & 15) == 0, "nerf_posenc_tiles_rays: null/misaligned pointer");
    return posenc_tiles(z_vals, viewdirs, n_rays * samples_per_ray, samples_per_ray, multires, multires_dirs, enc_image, rays_o, rays_d, stream, "nerf_posenc_tiles_rays");
}

int xrb_nerf_posenc_grad(const float *pts, int64_t n_pts, int multires, const void *d_enc_image, int n_terms, const float *scale, float *grad, void *stream) {
    XRB_REQUIRE(n_pts >= 0 && multires >= 0 && multires <= 10 && n_terms >= 1 && n_terms <= 4, "nerf_posenc_grad: bad size (multires 0..10, n_terms 1..4)");
    if (n_pts == 0) return XRB_OK;
    XRB_REQUIRE(pts && d_enc_image && scale && grad && ((uintptr_t)d_enc_image & 15) == 0, "nerf_posenc_grad: null/misaligned pointer");
    point_enc_grad_kernel<false><<<stride_grid((n_pts + 255) / 256, 16), 256, 0, (cudaStream_t)stream>>>(pts, n_pts, multires, IpeBands{}, (const uint8_t *)d_enc_image, n_terms,
                                                                                                       scale, grad);
    return check_launch("nerf_posenc_grad");
}

int xrb_mip_ipe_tiles_points(const float *pts, const float *viewdirs, int64_t n_pts, int samples_per_ray, float sigma, int min_deg_point, int max_deg_point, int min_deg_view,
                             int max_deg_view, void *enc_image, void *stream) {
    XRB_REQUIRE(n_pts >= 0 && samples_per_ray >= 1 && ipe_point_degrees_ok(min_deg_point, max_deg_point) && max_deg_view >= min_deg_view && min_deg_view >= -100
                && max_deg_view <= 100 && 3 + 6 * (max_deg_view - min_deg_view) <= 64,
                "mip_ipe_tiles_points: bad size (point degrees: 6 (max - min) <= 128, view degrees: 3 + 6 (max - min) <= 64, degrees in [-100, 100])");
    XRB_REQUIRE(std::isfinite(sigma) && sigma >= 0.f, "mip_ipe_tiles_points: the footprint sigma must be finite and >= 0");
    if (n_pts == 0) return XRB_OK;
    XRB_REQUIRE(pts && viewdirs && enc_image && ((uintptr_t)enc_image & 15) == 0, "mip_ipe_tiles_points: null/misaligned pointer");
    mip_ipe_tiles_points_kernel<<<tile_grid(n_pts, 256), 256, 0, (cudaStream_t)stream>>>(pts, viewdirs, n_pts, samples_per_ray, ipe_bands(sigma, min_deg_point, max_deg_point),
                                                                                          min_deg_view, max_deg_view - min_deg_view, (uint8_t *)enc_image);
    return check_launch("mip_ipe_tiles_points");
}

int xrb_mip_ipe_grad(const float *pts, int64_t n_pts, float sigma, int min_deg_point, int max_deg_point, const void *d_enc_image, int n_terms, const float *scale, float *grad,
                     void *stream) {
    XRB_REQUIRE(n_pts >= 0 && ipe_point_degrees_ok(min_deg_point, max_deg_point) && n_terms >= 1 && n_terms <= 4,
                "mip_ipe_grad: bad size (point degrees: 6 (max - min) <= 128 in [-100, 100], n_terms 1..4)");
    XRB_REQUIRE(std::isfinite(sigma) && sigma >= 0.f, "mip_ipe_grad: the footprint sigma must be finite and >= 0");
    if (n_pts == 0) return XRB_OK;
    XRB_REQUIRE(pts && d_enc_image && scale && grad && ((uintptr_t)d_enc_image & 15) == 0, "mip_ipe_grad: null/misaligned pointer");
    point_enc_grad_kernel<true><<<stride_grid((n_pts + 255) / 256, 16), 256, 0, (cudaStream_t)stream>>>(pts, n_pts, 0, ipe_bands(sigma, min_deg_point, max_deg_point),
                                                                                                      (const uint8_t *)d_enc_image, n_terms, scale, grad);
    return check_launch("mip_ipe_grad");
}

int xrb_mip_resample(const float *z_vals, const float *weights, const float *u, int n_rays, int n_samples, float resample_padding, float *z_out, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && n_samples >= 2, "mip_resample: bad size");
    if (n_samples > MIP_MAX_S) { set_error("mip_resample: n_samples <= 256 supported"); return XRB_E_UNSUPPORTED; }
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(z_vals && weights && z_out, "mip_resample: null pointer");
    mip_resample_kernel<<<(n_rays + PDF_WARPS - 1) / PDF_WARPS, PDF_WARPS * 32, 0, (cudaStream_t)stream>>>(n_rays, n_samples, resample_padding, z_vals, weights, u, z_out);
    return check_launch("mip_resample");
}

int xrb_ngp_batch_sample(const float *poses, const float *images_rgba, int n_images, int H, int W, float fx, float fy, float cx, float cy, const int64_t *row_idx, int64_t n,
                         const float *u_bg, uint64_t seed, int64_t n_prior_calls, float *rays_o, float *rays_d, float *target_s, float *alpha, float *img_ids, float *bg_color, void *stream) {
    XRB_REQUIRE(n_images >= 1 && H >= 1 && W >= 1 && n >= 0, "ngp_batch_sample: bad arguments");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(poses && images_rgba && row_idx && rays_o && rays_d && target_s && alpha && img_ids && bg_color, "ngp_batch_sample: null pointer");
    XRB_REQUIRE(((uintptr_t)images_rgba & 15) == 0, "ngp_batch_sample: images must be 16-byte aligned");
    const int blocks = stride_grid((n + 255) / 256, 16);
    ngp_batch_sample_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(poses, images_rgba, n_images, H, W, fx, fy, cx, cy, row_idx, n, u_bg, host_rng(seed, n_prior_calls), rays_o, rays_d,
                                                                          target_s, alpha, img_ids, bg_color);
    return check_launch("ngp_batch_sample");
}

int xrb_ngp_batch_depth(const float *depths, int n_images, int H, int W, float fx, float fy, float cx, float cy, float scale, const int64_t *row_idx, int64_t n,
                        float *target_depth, void *stream) {
    XRB_REQUIRE(n_images >= 1 && H >= 1 && W >= 1 && n >= 0, "ngp_batch_depth: bad arguments");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(depths && row_idx && target_depth, "ngp_batch_depth: null pointer");
    ngp_batch_depth_kernel<<<stride_grid((n + 255) / 256, 16), 256, 0, (cudaStream_t)stream>>>(depths, H, W, fx, fy, cx, cy, scale, row_idx, n, target_depth);
    return check_launch("ngp_batch_depth");
}

int xrb_ngp_pose_grad(const int64_t *row_idx, int64_t n, const float *poses, int n_images, int H, int W, float fx, float fy, float cx, float cy, const float *grad_o,
                      const float *grad_d, float *d_poses, void *stream) {
    XRB_REQUIRE(n_images >= 1 && H >= 1 && W >= 1 && n >= 0, "ngp_pose_grad: bad arguments");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(row_idx && poses && grad_o && grad_d && d_poses, "ngp_pose_grad: null pointer");
    const int blocks = stride_grid((n + 255) / 256, 4);
    const size_t smem = (size_t)n_images * 12 * sizeof(float);
    if (smem <= (size_t)POSE_GRAD_SMEM_MAX)
        ngp_pose_grad_kernel<true><<<blocks, 256, smem, (cudaStream_t)stream>>>(row_idx, n, n_images, H, W, fx, fy, cx, cy, poses, grad_o, grad_d, d_poses);
    else
        ngp_pose_grad_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(row_idx, n, n_images, H, W, fx, fy, cx, cy, poses, grad_o, grad_d, d_poses);
    return check_launch("ngp_pose_grad");
}

int xrb_nerf_get_rays(const float *c2w_host, int H, int W, float fx, float fy, float cx, float cy, int convention, const int32_t *pixel_idx, int64_t n, float *rays_o, float *rays_d,
                      float *viewdirs, float *radii, void *stream) {
    XRB_REQUIRE(H >= 1 && W >= 1 && n >= 0 && (convention == 0 || convention == 1), "get_rays: bad arguments");
    XRB_REQUIRE(!(radii && H < 3), "get_rays: radii need H >= 3");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(c2w_host && rays_o && rays_d, "get_rays: null pointer");
    RayGenParams p; for (int k = 0; k < 12; ++k) p.c2w[k] = c2w_host[k];
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.H = H; p.W = W; p.convention = convention;
    const int blocks = stride_grid((n + 255) / 256, 16);
    get_rays_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p, pixel_idx, n, rays_o, rays_d, viewdirs, radii);
    return check_launch("get_rays");
}

int xrb_nerf_zvals(int64_t n_rays, int n_samples, float near_, float far_, int lindisp, const float *u, float *z_vals, void *stream) {
    XRB_REQUIRE(n_rays >= 0 && n_samples >= 2, "zvals: bad size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(z_vals, "zvals: null pointer");
    const int blocks = stride_grid((n_rays * n_samples + 255) / 256, 16);
    zvals_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n_rays, n_samples, near_, far_, lindisp, u, z_vals);
    return check_launch("zvals");
}

}  // extern "C"
