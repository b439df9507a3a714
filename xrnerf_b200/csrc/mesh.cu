// xrnerf_b200 — NGP mesh export: the field's density on a lattice (xrb_ngp_density_lattice) and marching cubes (xrb_mc_count / xrb_mc_emit).
// The contracts (lattice positions, inside rule, vertex interpolation, output order, workspace) are stated in include/xrnerf_b200.h.
//
// Marching cubes has the march's count -> scan -> emit shape, so the output order is fixed without atomics:
//   mc_count_kernel   thread = lattice point p: the crossing edges p owns (+x, +y, +z) and the triangle count of the cell whose lowest corner
//                     is p; the block scans the vertex counts and stores, per point, its in-block vertex offset and crossing mask (4 bytes),
//                     per block, its vertex and triangle sums;
//   mc_scan_kernel    one block: exclusive scans of the block sums, the totals (V, F);
//   mc_emit_kernel    thread = p again: writes p's vertices at its base, recomputes the in-block triangle offsets with block_excl_scan and
//                     writes the cell's triangles; a triangle's vertex owned by a neighbouring point is that point's block base + in-block
//                     offset + the crossing edges it owns on lower axes.
#include <cmath>

#include "ngp_field.cuh"
#include "lattice.cuh"
#include "mc_table.cuh"

namespace xrb {

// ---------------------------------------------------------------------------------------------------------------- density on a lattice
// positions of `n` consecutive lattice points from `first` (x fastest) as the field's [n,3] rows
constexpr int LATTICE_CHUNK = 1 << 20;
__global__ void __launch_bounds__(256) lattice_points_kernel(int64_t first, int n, Lattice L, float *__restrict__ pts) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    L.position(first + i, pts + 3 * (size_t)i);
}

// ---------------------------------------------------------------------------------------------------------------- marching cubes
constexpr int MC_BLOCK = 256;
constexpr uint32_t MC_OFF_MASK = 0xfffu, MC_CROSS_SHIFT = 12;   // point word: in-block vertex offset (< 3 * MC_BLOCK) | crossing mask << 12
struct McWs {
    uint32_t *word;     // [points]
    uint32_t *vblock;   // [blocks] vertex sum of the block, then its first vertex
    uint32_t *fblock;   // [blocks] the same for triangles
    uint32_t *misc;     // [4] V, F, overflow flag
};
inline int64_t mc_points(int nx, int ny, int nz) { return (int64_t)nx * ny * nz; }
inline int64_t mc_blocks(int64_t points) { return (points + MC_BLOCK - 1) / MC_BLOCK; }
inline size_t mc_ws_bytes(int64_t points) { return sizeof(uint32_t) * ((size_t)points + 2 * (size_t)mc_blocks(points) + 4); }
inline McWs mc_ws(void *ws, int64_t points) {
    McWs w; w.word = (uint32_t *)ws; w.vblock = w.word + points; w.fblock = w.vblock + mc_blocks(points); w.misc = w.fblock + mc_blocks(points);
    return w;
}

// case index of the cell whose lowest corner is p (corner c at p + (c & 1, c >> 1 & 1, c >> 2 & 1))
__device__ __forceinline__ uint32_t cell_case(const float *__restrict__ vol, const Lattice &L, int64_t p, float thr) {
    uint32_t c = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) c |= (uint32_t)(__ldg(vol + p + (k & 1) + ((k >> 1) & 1) * (int64_t)L.n[0] + ((k >> 2) & 1) * L.nxy) > thr) << k;
    return c;
}

__global__ void __launch_bounds__(MC_BLOCK) mc_count_kernel(const float *__restrict__ vol, Lattice L, float thr, uint32_t *__restrict__ word, uint32_t *__restrict__ vblock,
                                                            uint32_t *__restrict__ fblock) {
    const int64_t p = (int64_t)blockIdx.x * MC_BLOCK + threadIdx.x;
    uint32_t mask = 0, nt = 0;
    if (p < L.points) {
        int idx[3]; L.coords(p, idx);
        const bool in0 = __ldg(vol + p) > thr;
        if (idx[0] + 1 < L.n[0]) mask |= (uint32_t)(in0 != (__ldg(vol + p + 1) > thr));
        if (idx[1] + 1 < L.n[1]) mask |= (uint32_t)(in0 != (__ldg(vol + p + L.n[0]) > thr)) << 1;
        if (idx[2] + 1 < L.n[2]) mask |= (uint32_t)(in0 != (__ldg(vol + p + L.nxy) > thr)) << 2;
        if (idx[0] + 1 < L.n[0] && idx[1] + 1 < L.n[1] && idx[2] + 1 < L.n[2]) nt = MC_TRI_COUNT[cell_case(vol, L, p, thr)];
    }
    uint32_t vtot, ftot;
    const uint32_t vex = block_excl_scan<MC_BLOCK>(__popc(mask), &vtot);
    __syncthreads();
    block_excl_scan<MC_BLOCK>(nt, &ftot);
    if (p < L.points) word[p] = vex | (mask << MC_CROSS_SHIFT);
    if (threadIdx.x == 0) { vblock[blockIdx.x] = vtot; fblock[blockIdx.x] = ftot; }
}

// one block: block sums -> first vertex / triangle of each block; totals to misc and counts. A total past INT32_MAX sets the overflow flag
// (the emit pass then writes nothing) and counts (-1, -1).
constexpr int MC_SCAN_ITEMS = 8;
__global__ void __launch_bounds__(1024) mc_scan_kernel(int64_t n_blocks, uint32_t *__restrict__ vblock, uint32_t *__restrict__ fblock, uint32_t *__restrict__ misc,
                                                       int32_t *__restrict__ counts) {
    __shared__ unsigned long long carry_s[2];
    if (threadIdx.x < 2) carry_s[threadIdx.x] = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < n_blocks; b0 += 1024 * MC_SCAN_ITEMS) {
        const int64_t b = b0 + (int64_t)threadIdx.x * MC_SCAN_ITEMS;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            uint32_t *s = q == 0 ? vblock : fblock;
            uint32_t v[MC_SCAN_ITEMS], sum = 0;
#pragma unroll
            for (int k = 0; k < MC_SCAN_ITEMS; ++k) { v[k] = b + k < n_blocks ? s[b + k] : 0u; sum += v[k]; }   // <= 8 * 5 * MC_BLOCK
            uint32_t tot, ex = block_excl_scan<1024>(sum, &tot);
            const unsigned long long carry = carry_s[q];
            unsigned long long run = carry + ex;
#pragma unroll
            for (int k = 0; k < MC_SCAN_ITEMS; ++k) { if (b + k < n_blocks) s[b + k] = (uint32_t)run; run += v[k]; }
            __syncthreads();
            if (threadIdx.x == 0) carry_s[q] = carry + tot;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        const bool overflow = carry_s[0] > 0x7fffffffull || carry_s[1] > 0x7fffffffull;
        misc[0] = (uint32_t)carry_s[0]; misc[1] = (uint32_t)carry_s[1]; misc[2] = overflow;
        counts[0] = overflow ? -1 : (int32_t)carry_s[0];
        counts[1] = overflow ? -1 : (int32_t)carry_s[1];
    }
}

// index of the vertex on the edge that point q owns along `axis`
__device__ __forceinline__ int32_t owned_vertex(const uint32_t *__restrict__ word, const uint32_t *__restrict__ vblock, int64_t q, int axis) {
    const uint32_t w = __ldg(word + q);
    return (int32_t)(__ldg(vblock + q / MC_BLOCK) + (w & MC_OFF_MASK) + __popc((w >> MC_CROSS_SHIFT) & ((1u << axis) - 1u)));
}

__global__ void __launch_bounds__(MC_BLOCK) mc_emit_kernel(const float *__restrict__ vol, Lattice L, float thr, const uint32_t *__restrict__ word,
                                                           const uint32_t *__restrict__ vblock, const uint32_t *__restrict__ fblock, const uint32_t *__restrict__ misc,
                                                           float *__restrict__ verts, int32_t *__restrict__ faces) {
    if (misc[2]) return;
    const int64_t p = (int64_t)blockIdx.x * MC_BLOCK + threadIdx.x;
    uint32_t nt = 0, cs = 0;
    if (p < L.points) {
        int idx[3]; L.coords(p, idx);
        const uint32_t w = word[p], mask = w >> MC_CROSS_SHIFT;
        if (mask) {
            float pos[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) pos[a] = L.coord(a, idx[a]);
            const float vp = __ldg(vol + p);
            float *out = verts + 3 * (size_t)(vblock[blockIdx.x] + (w & MC_OFF_MASK));
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                if (!((mask >> a) & 1u)) continue;
                // t = (thr - v_out) / (v_in - v_out) from the outside endpoint; the position moves along axis a only
                const float vq = __ldg(vol + p + L.stride(a));
                const bool p_in = vp > thr;
                const float v_in = p_in ? vp : vq, v_out = p_in ? vq : vp;
                const float t = div_(sub_(thr, v_out), sub_(v_in, v_out));
                const float P = pos[a], Q = L.coord(a, idx[a] + 1);
                const float P_in = p_in ? P : Q, P_out = p_in ? Q : P;
                float v[3] = {pos[0], pos[1], pos[2]};
                v[a] = add_(P_out, mul_(t, sub_(P_in, P_out)));
                out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
                out += 3;
            }
        }
        if (idx[0] + 1 < L.n[0] && idx[1] + 1 < L.n[1] && idx[2] + 1 < L.n[2]) { cs = cell_case(vol, L, p, thr); nt = MC_TRI_COUNT[cs]; }
    }
    uint32_t ftot;
    const uint32_t fex = block_excl_scan<MC_BLOCK>(nt, &ftot);
    if (nt == 0) return;
    int32_t *f = faces + 3 * (size_t)(fblock[blockIdx.x] + fex);
    for (uint32_t k = 0; k < 3 * nt; ++k) {
        // edge e runs along axis e / 4 from the corner with that axis' bit 0; the other two axes, in increasing order, take the bits of e % 4
        const int e = MC_TRI_EDGES[cs][k], a = e >> 2, lo = e & 1, hi = (e >> 1) & 1;
        const int dx = a == 0 ? 0 : lo, dy = a == 0 ? lo : (a == 1 ? 0 : hi), dz = a == 2 ? 0 : hi;
        f[k] = owned_vertex(word, vblock, p + dx + dy * (int64_t)L.n[0] + dz * L.nxy, a);
    }
}

}  // namespace xrb

using namespace xrb;

extern "C" {

size_t xrb_ngp_density_lattice_workspace(void) { return (size_t)LATTICE_CHUNK * 3 * sizeof(float); }

int xrb_ngp_density_lattice(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *weight_image, int nx, int ny, int nz,
                            const float *box_min_host, const float *box_max_host, float *out, int impl, void *workspace, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    const int sz = lattice_sizes(nx, ny, nz, "ngp_density_lattice: bad size: every lattice size must be 2..1024");
    if (sz < 0) return XRB_E_BADARG;
    Box b;
    e = read_box(box_min_host, box_max_host, true, &b, "ngp_density_lattice: the box must satisfy 0 <= box_min < box_max <= 1 on every axis (the field's warped domain)");
    if (e) return e;
    if (sz == 0) return XRB_OK;
    XRB_REQUIRE(table && out && workspace, "ngp_density_lattice: null pointer");
    XRB_REQUIRE(impl == 0 ? (density_fp16 != nullptr) : (weight_image != nullptr), "ngp_density_lattice: missing weights for the requested impl");
    XRB_REQUIRE(((uintptr_t)workspace & 15) == 0, "ngp_density_lattice: workspace must be 16-byte aligned");
    HashGridDev g; e = table_setup(cfg, table, &g); if (e) return e;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t points = mc_points(nx, ny, nz);
    float *pts = (float *)workspace;
    for (int64_t first = 0; first < points; first += LATTICE_CHUNK) {
        const int n = (int)(points - first < LATTICE_CHUNK ? points - first : LATTICE_CHUNK);
        lattice_points_kernel<<<(n + 255) / 256, 256, 0, s>>>(first, n, make_lattice(nx, ny, nz, b), pts);
        e = launch_field(cfg, table, density_fp16, nullptr, weight_image, pts, 3, nullptr, 3, n, nullptr, nullptr, out + first, impl, true, s);
        if (e) return e;
    }
    return XRB_OK;
}

size_t xrb_mc_workspace(int nx, int ny, int nz) {
    if (lattice_sizes(nx, ny, nz, "mc_workspace: bad size") < 0) return 0;
    return mc_ws_bytes(mc_points(nx, ny, nz));
}

int xrb_mc_count(const float *volume, int nx, int ny, int nz, float threshold, void *workspace, int32_t *counts, void *stream) {
    const int sz = lattice_sizes(nx, ny, nz, "mc_count: bad size: every lattice size must be 2..1024");
    if (sz < 0) return XRB_E_BADARG;
    XRB_REQUIRE(!std::isnan(threshold), "mc_count: threshold is NaN");
    if (sz == 0) return XRB_OK;
    XRB_REQUIRE(volume && workspace && counts, "mc_count: null pointer");
    XRB_REQUIRE(((uintptr_t)volume & 3) == 0 && ((uintptr_t)workspace & 7) == 0 && ((uintptr_t)counts & 7) == 0, "mc_count: misaligned pointer");
    const Lattice L = make_lattice(nx, ny, nz);
    const McWs w = mc_ws(workspace, L.points);
    const int64_t nb = mc_blocks(L.points);
    cudaStream_t s = (cudaStream_t)stream;
    mc_count_kernel<<<(unsigned)nb, MC_BLOCK, 0, s>>>(volume, L, threshold, w.word, w.vblock, w.fblock);
    mc_scan_kernel<<<1, 1024, 0, s>>>(nb, w.vblock, w.fblock, w.misc, counts);
    return check_launch("mc_count");
}

int xrb_mc_emit(const float *volume, int nx, int ny, int nz, float threshold, const float *box_min_host, const float *box_max_host, const void *workspace, float *verts,
                int32_t *faces, void *stream) {
    const int sz = lattice_sizes(nx, ny, nz, "mc_emit: bad size: every lattice size must be 2..1024");
    if (sz < 0) return XRB_E_BADARG;
    XRB_REQUIRE(!std::isnan(threshold), "mc_emit: threshold is NaN");
    Box b;
    int e = read_box(box_min_host, box_max_host, false, &b, "mc_emit: the box must be finite with box_min < box_max on every axis");
    if (e) return e;
    if (sz == 0) return XRB_OK;
    XRB_REQUIRE(volume && workspace && verts && faces, "mc_emit: null pointer");
    XRB_REQUIRE(((uintptr_t)volume & 3) == 0 && ((uintptr_t)workspace & 7) == 0 && ((uintptr_t)verts & 3) == 0 && ((uintptr_t)faces & 3) == 0, "mc_emit: misaligned pointer");
    const Lattice L = make_lattice(nx, ny, nz, b);
    const McWs w = mc_ws(const_cast<void *>(workspace), L.points);
    mc_emit_kernel<<<(unsigned)mc_blocks(L.points), MC_BLOCK, 0, (cudaStream_t)stream>>>(volume, L, threshold, w.word, w.vblock, w.fblock, w.misc, verts, faces);
    return check_launch("mc_emit");
}

}  // extern "C"
