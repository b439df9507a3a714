// xrnerf_b200 — the density lattice shared by the mesh-export entry points (xrb_ngp_density_lattice, xrb_nerf_density_lattice,
// xrb_mip_density_lattice, xrb_mc_count, xrb_mc_emit): a lattice point's coordinates and position, and the checks of the lattice sizes and box.
// The contract is in include/xrnerf_b200.h (mesh section).
#pragma once
#include <cmath>

#include "common.cuh"

namespace xrb {

// coordinate of lattice index i on an axis of n points from lo to hi: min(lo + i * ((hi - lo) / (n - 1)), hi), each operation rounded once.
// The min keeps the last point inside the box when the rounded step overshoots.
__device__ __forceinline__ float lattice_coord(float lo, float hi, int n, int i) { return fminf(add_(lo, mul_((float)i, div_(sub_(hi, lo), (float)(n - 1)))), hi); }

struct Box { float lo[3], hi[3]; };

// n[0] x n[1] x n[2] points over `box`, point index p = x + n[0] (y + n[1] z)
struct Lattice {
    int n[3];
    int64_t nxy, points;
    Box box;
    __device__ void coords(int64_t p, int idx[3]) const { idx[0] = (int)(p % n[0]); idx[1] = (int)((p / n[0]) % n[1]); idx[2] = (int)(p / nxy); }
    __device__ float coord(int a, int i) const { return lattice_coord(box.lo[a], box.hi[a], n[a], i); }
    __device__ void position(int64_t p, float x[3]) const {
        int idx[3]; coords(p, idx);
#pragma unroll
        for (int a = 0; a < 3; ++a) x[a] = coord(a, idx[a]);
    }
    __device__ int64_t stride(int axis) const { return axis == 0 ? 1 : axis == 1 ? (int64_t)n[0] : nxy; }
};
static inline Lattice make_lattice(int nx, int ny, int nz, const Box &b = Box{}) {
    Lattice L{{nx, ny, nz}, (int64_t)nx * ny, (int64_t)nx * ny * nz, b};
    return L;
}

// 0: an empty lattice (some size 0); 1: every size in [2, 1024]; -1: otherwise (the error is set)
static inline int lattice_sizes(int nx, int ny, int nz, const char *who) {
    const int n[3] = {nx, ny, nz};
    bool empty = false, ok = true;
    for (int a = 0; a < 3; ++a) { empty |= n[a] == 0; ok &= n[a] == 0 || (n[a] >= 2 && n[a] <= 1024); }
    if (!ok) { set_error(who); return -1; }
    return empty ? 0 : 1;
}
// a finite box with lo < hi on every axis (inside [0,1]^3 when `unit`)
static inline int read_box(const float *lo, const float *hi, bool unit, Box *b, const char *who) {
    XRB_REQUIRE(lo && hi, who);
    for (int a = 0; a < 3; ++a) {
        XRB_REQUIRE(lo[a] < hi[a] && std::isfinite(lo[a]) && std::isfinite(hi[a]), who);
        XRB_REQUIRE(!unit || (lo[a] >= 0.f && hi[a] <= 1.f), who);
        b->lo[a] = lo[a]; b->hi[a] = hi[a];
    }
    return XRB_OK;
}

}  // namespace xrb
