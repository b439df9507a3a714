// xrnerf_b200 — depth and opacity supervision loss (xrb_geom_loss_grad, include/xrnerf_b200.h): one kernel for NGP, NeRF and Mip-NeRF.
//   loss = w_d * sum |D - D*| / c_d + w_a * sum (A - A*)^2 / c_a
// over the rays each term keeps; c = 1 ('sum', NGP) or the number of rays the term keeps ('mean', NeRF / Mip-NeRF).
#include "common.cuh"

namespace xrb {

constexpr int GEOM_THREADS = 1024;

// ONE block: a count pass (mean only), then the gradients and a fixed-order reduction of the loss, so the result does not depend on scheduling
__global__ void __launch_bounds__(GEOM_THREADS) geom_loss_kernel(int n, const float *__restrict__ depth, const float *__restrict__ alpha, const float *__restrict__ target_depth,
                                                                 const float *__restrict__ target_alpha, const int32_t *__restrict__ numsteps,
                                                                 const int32_t *__restrict__ numsteps_c, float wd, float wa, int mean, float *__restrict__ grad_depth,
                                                                 float *__restrict__ grad_alpha, float *__restrict__ loss_accum) {
    __shared__ float s_part[2][GEOM_THREADS / 32];
    __shared__ float s_inv[2];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const bool use_d = wd > 0.f, use_a = wa > 0.f;
    // a ray takes part when all of its samples were trained (NGP: the compaction did not truncate it); its depth term also needs a finite target > 0
    auto trained = [&](int i) { return !numsteps || numsteps_c[2 * (size_t)i] == numsteps[2 * (size_t)i]; };
    auto keep_d = [&](int i) { const float t = target_depth[i]; return trained(i) && isfinite(t) && t > 0.f; };
    if (threadIdx.x == 0) { s_inv[0] = 1.f; s_inv[1] = 1.f; }
    if (mean) {
        float cd = 0.f, ca = 0.f;
        for (int i = threadIdx.x; i < n; i += GEOM_THREADS) {
            if (use_d && keep_d(i)) cd += 1.f;
            if (use_a && trained(i)) ca += 1.f;
        }
        cd = warp_sum(cd); ca = warp_sum(ca);
        if (lane == 0) { s_part[0][w] = cd; s_part[1][w] = ca; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float td = 0.f, ta = 0.f;
            for (int k = 0; k < GEOM_THREADS / 32; ++k) { td += s_part[0][k]; ta += s_part[1][k]; }
            s_inv[0] = td > 0.f ? 1.f / td : 0.f; s_inv[1] = ta > 0.f ? 1.f / ta : 0.f;
        }
    }
    __syncthreads();
    const float sd = wd * s_inv[0], sa = wa * s_inv[1];
    float ld = 0.f, la = 0.f;
    for (int i = threadIdx.x; i < n; i += GEOM_THREADS) {
        if (grad_depth) {
            float g = 0.f;
            if (use_d && keep_d(i)) {
                const float r = depth[i] - target_depth[i];
                g = r > 0.f ? sd : (r < 0.f ? -sd : 0.f);
                ld += fabsf(r);
            }
            grad_depth[i] = g;
        }
        if (grad_alpha) {
            float g = 0.f;
            if (use_a && trained(i)) {
                const float r = alpha[i] - target_alpha[i];
                g = 2.f * sa * r;
                la += r * r;
            }
            grad_alpha[i] = g;
        }
    }
    ld = warp_sum(ld); la = warp_sum(la);
    __syncthreads();
    if (lane == 0) { s_part[0][w] = ld; s_part[1][w] = la; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float td = 0.f, ta = 0.f;
        for (int k = 0; k < GEOM_THREADS / 32; ++k) { td += s_part[0][k]; ta += s_part[1][k]; }
        loss_accum[0] += sd * td + sa * ta;
    }
}

}  // namespace xrb

using namespace xrb;

extern "C" {

int xrb_geom_loss_grad(const float *depth, const float *alpha, const float *target_depth, const float *target_alpha, const int32_t *numsteps,
                       const int32_t *numsteps_compacted, int n_rays, float depth_weight, float opacity_weight, int mean, float *grad_depth, float *grad_alpha,
                       float *loss_accum, void *stream) {
    XRB_REQUIRE(n_rays >= 0, "geom_loss_grad: negative size");
    XRB_REQUIRE(std::isfinite(depth_weight) && depth_weight >= 0.f && std::isfinite(opacity_weight) && opacity_weight >= 0.f,
                "geom_loss_grad: the weights must be finite and >= 0");
    XRB_REQUIRE(mean == 0 || mean == 1, "geom_loss_grad: mean must be 0 (sum) or 1 (mean over the kept rays)");
    XRB_REQUIRE((numsteps == nullptr) == (numsteps_compacted == nullptr), "geom_loss_grad: numsteps and numsteps_compacted go together");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(loss_accum, "geom_loss_grad: null loss_accum");
    XRB_REQUIRE(!(depth_weight > 0.f) || (depth && target_depth && grad_depth), "geom_loss_grad: depth_weight > 0 needs depth, target_depth and grad_depth");
    XRB_REQUIRE(!(opacity_weight > 0.f) || (alpha && target_alpha && grad_alpha), "geom_loss_grad: opacity_weight > 0 needs alpha, target_alpha and grad_alpha");
    geom_loss_kernel<<<1, GEOM_THREADS, 0, (cudaStream_t)stream>>>(n_rays, depth, alpha, target_depth, target_alpha, numsteps, numsteps_compacted, depth_weight, opacity_weight,
                                                                    mean, grad_depth, grad_alpha, loss_accum);
    return check_launch("geom_loss_grad");
}

}  // extern "C"
