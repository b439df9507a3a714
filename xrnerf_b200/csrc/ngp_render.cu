// xrnerf_b200 — render of a ray batch through the Instant-NGP path (inference):
//   march (count -> scan -> emit)  ->  field (hash encode + MLPs on wgmma tiles)  ->  composite (warp per ray)
// replacing ngp_grid_sampler.py:205-228 + hashnerf_mlp.py:55-79 + hashnerf_render.py:42-46 of the reference with ZERO host
// synchronisations: the sample count stays on the device (the field kernel reads it from `counters[1]`).
// v1: the three stages are separate launches chained on one stream (5 launches per batch, CUDA-graph capturable);
// the single-launch variant is tracked in DESIGN.md §6.
#include "ngp_field.cuh"

extern "C" {

size_t xrb_ngp_render_workspace(int n_rays, int max_samples) {
    size_t a = (xrb_rm_rays_sampler_workspace(n_rays) + 255) & ~(size_t)255;
    return a + (size_t)max_samples * (7 + 4) * sizeof(float) + (size_t)n_rays * sizeof(int32_t) + 256;
}

int xrb_ngp_render(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *weight_image, const uint8_t *bitfield, const float *rays_o, const float *rays_d, int n_rays,
                   int max_samples, float aabb0, float aabb1, float near_distance, float cone_angle, uint64_t seed, int64_t n_prior_calls, const float *bg3_host, int rgb_act,
                   int dens_act, float *rgb_out, float *alpha_out, int32_t *numsteps, int32_t *counters, void *workspace, void *ev_before_field, void *ev_after_field, void *stream) {
    int e = xrb::check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n_rays >= 0 && max_samples > 0, "ngp_render: bad size");
    if (n_rays == 0) return XRB_OK;
    XRB_REQUIRE(table && weight_image && bitfield && rays_o && rays_d && bg3_host && rgb_out && alpha_out && numsteps && counters && workspace, "ngp_render: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    uint8_t *ws = (uint8_t *)workspace;
    size_t a = (xrb_rm_rays_sampler_workspace(n_rays) + 255) & ~(size_t)255;
    float *coords = (float *)(ws + a);
    float *raw = coords + (size_t)max_samples * 7;
    int32_t *rays_index = (int32_t *)(raw + (size_t)max_samples * 4);
    cudaMemsetAsync(counters, 0, 2 * sizeof(int32_t), s);
    e = xrb_rm_rays_sampler(rays_o, rays_d, bitfield, nullptr, nullptr, nullptr, n_rays, max_samples, aabb0, aabb1, near_distance, cone_angle, seed, n_prior_calls, coords, rays_index,
                            numsteps, counters, ws, stream);
    if (e) return e;
    // counters[1] counts overflowed rays too; rows beyond max_samples do not exist, launch_field clamps to max_samples
    // measurement hook: events recorded right before / after the field kernel let a caller time the dominant kernel inside its own timed region
    if (ev_before_field) cudaEventRecord((cudaEvent_t)ev_before_field, s);
    e = xrb::launch_field(cfg, table, nullptr, nullptr, weight_image, coords, 7, coords + 4, 7, max_samples, counters + 1, raw, 1, false, s);
    if (ev_after_field) cudaEventRecord((cudaEvent_t)ev_after_field, s);
    if (e) return e;
    return xrb_rm_calc_rgb_inference(raw, coords, numsteps, bg3_host, n_rays, rgb_act, dens_act, rgb_out, alpha_out, stream);
}

}  // extern "C"
