// xrnerf_b200 — backward of the Instant-NGP field (HashNerfMLP.run_mlp) and the training loss.
//
// One persistent kernel per training step replaces tcnn's backward (3 network/encoding backward launches + 2 `cat`
// backward kernels in the reference stack, hashnerf_mlp.py:55-79) :
//   per 128-sample tile (thread == sample):
//     1. recompute the forward (hash gather -> density net -> SH concat -> colour net), parking every layer INPUT as fp16 in
//        shared memory (needed both for the ReLU masks and as the X operand of the weight gradients);
//     2. walk the layers backwards: dX = W^T dY per thread (weights broadcast from shared memory), and after each layer a
//        block-level register-tiled GEMM  dW[o][i] += sum_s dY[s][o] * X[s][i]  over the tile (dY staged as scaled fp16);
//        the dW accumulators live in REGISTERS for the whole persistent loop and hit HBM once per CTA (atomicAdd);
//     3. scatter dL/d(encoding) into the fp32 hash-table gradient with vector atomics (red.global.add.v2.f32).
// Numeric contract: fp32 backward math on the fp16-rounded forward activations (oracle/tcnn_oracle.c
// oracle_ngp_mlp_backward); the dY staging uses fp16 with a fixed 2^12 scale (tcnn uses fp16 + loss scale 128).
// v1 runs the GEMM-shaped parts on CUDA cores; the tensor-core version is ngp_backward_tc.cu.
#include "ngp_field.cuh"

namespace xrb {

constexpr int BW_THREADS = 128;
constexpr float DY_SCALE = 4096.f;

// loads / stores my row of a shared-memory tile (fp16) as fp32 registers
__device__ __forceinline__ void load_row_h(const __half *row, float *v, int n) {
#pragma unroll
    for (int k = 0; k < n; k += 2) { float2 f = __half22float2(reinterpret_cast<const __half2 *>(row)[k >> 1]); v[k] = f.x; v[k + 1] = f.y; }
}
__device__ __forceinline__ void store_row_h(__half *row, const float *v, int n) {
    for (int k = 0; k < n; k += 2) reinterpret_cast<__half2 *>(row)[k >> 1] = __floats2half2_rn(v[k], v[k + 1]);
}
// gx[k] = sum_o W[o][k] * gy[o]. UNROLL: how many outputs are unrolled (the training kernels take 2; OUT keeps gy in registers)
template <int IN, int OUT, int UNROLL = 2>
__device__ __forceinline__ void bwd_layer_dx(const __half *__restrict__ W, const float *gy, float *gx) {
#pragma unroll
    for (int k = 0; k < IN; ++k) gx[k] = 0.f;
#pragma unroll UNROLL
    for (int o = 0; o < OUT; ++o) {
        const float g = gy[o];
        const __half2 *w2 = reinterpret_cast<const __half2 *>(W + (size_t)o * IN);
#pragma unroll
        for (int k = 0; k < IN / 2; ++k) { float2 w = __half22float2(w2[k]); gx[2 * k] = fmaf(w.x, g, gx[2 * k]); gx[2 * k + 1] = fmaf(w.y, g, gx[2 * k + 1]); }
    }
}
// block GEMM: acc[TO][TI] += sum_s DY[s][o0+a] * X[s][i0+b]; thread tile TOxTI, 128 threads cover OUT x IN exactly
template <int IN, int OUT, int TO, int TI>
__device__ __forceinline__ void dw_accumulate(const __half *__restrict__ DY /*[128][64]*/, const __half *__restrict__ X /*[128][IN]*/, float *acc, int n_valid) {
    static_assert((OUT / TO) * (IN / TI) == BW_THREADS, "thread tiling must cover the matrix");
    const int to = threadIdx.x / (IN / TI), ti = threadIdx.x % (IN / TI);
    for (int s = 0; s < n_valid; ++s) {
        float dy[TO], x[TI];
#pragma unroll
        for (int a = 0; a < TO; a += 2) { float2 v = __half22float2(*reinterpret_cast<const __half2 *>(DY + (size_t)s * 64 + to * TO + a)); dy[a] = v.x; dy[a + 1] = v.y; }
#pragma unroll
        for (int b = 0; b < TI; b += 2) { float2 v = __half22float2(*reinterpret_cast<const __half2 *>(X + (size_t)s * IN + ti * TI + b)); x[b] = v.x; x[b + 1] = v.y; }
#pragma unroll
        for (int a = 0; a < TO; ++a)
#pragma unroll
            for (int b = 0; b < TI; ++b) acc[a * TI + b] = fmaf(dy[a], x[b], acc[a * TI + b]);
    }
}
template <int IN, int OUT, int TO, int TI>
__device__ __forceinline__ void dw_flush(const float *acc, float *__restrict__ dW /* [OUT][IN] */) {
    const int to = threadIdx.x / (IN / TI), ti = threadIdx.x % (IN / TI);
#pragma unroll
    for (int a = 0; a < TO; ++a)
#pragma unroll
        for (int b = 0; b < TI; ++b) atomicAdd(dW + (size_t)(to * TO + a) * IN + ti * TI + b, acc[a * TI + b] * (1.f / DY_SCALE));
}
__device__ __forceinline__ void stage_dy(__half *DY, const float *g, int n) {  // my row; n <= 64, rest untouched
    __half *row = DY + (size_t)threadIdx.x * 64;
    for (int k = 0; k < n; k += 2) reinterpret_cast<__half2 *>(row)[k >> 1] = __floats2half2_rn(g[k] * DY_SCALE, g[k + 1] * DY_SCALE);
}

// ---------------------------------------------------------------------------- backward of one tcnn-shaped net (32 -> 64 x NH -> 16) on a 128-sample tile
// NH is a template parameter so that the register accumulators have static shapes. Parameters in tcnn's order: W_in [64][32], NH - 1 x W_hid [64][64], W_out [16][64].
constexpr int NET_IN = 64 * 32, NET_HID = 64 * 64;   // elements of the input matrix / of one hidden matrix
__host__ __device__ constexpr int net_params(int nh) { return (int)mlp_num_params(32, 64, nh, 16); }
__host__ __device__ constexpr int net_tile_halfs(int nh) { return 128 * 32 + nh * 128 * 64; }
// the net's layer inputs of the tile, fp16 in shared memory: needed both for the ReLU masks and as the X operand of the weight gradients
template <int NH> struct NetTiles {
    __half *X;       // [128][32] input rows
    __half *H[NH];   // [128][64] output of hidden layer k
    __device__ __forceinline__ explicit NetTiles(__half *&p) { X = p; p += 128 * 32; for (int k = 0; k < NH; ++k) { H[k] = p; p += 128 * 64; } }
};
// the net's weight-gradient accumulators (scaled by DY_SCALE): this thread's tile of each matrix (dw_accumulate), in registers for the whole persistent loop
template <int NH> struct NetGrad { float in[16] = {}, hid[NH > 1 ? (NH - 1) * 32 : 1] = {}, out[8] = {}; };

// forward recompute of my row from t.X (already written), parking every hidden layer's output in t.H; out16 != NULL: also the output layer
template <int NH>
__device__ __forceinline__ void net_forward_park(const __half *__restrict__ W, const NetTiles<NH> &t, float *out16) {
    float x[64], h[64];
    load_row_h(t.X + (size_t)threadIdx.x * 32, x, 32);
    simt_layer<32, 64, true, 4>(W, x, h);
    store_row_h(t.H[0] + (size_t)threadIdx.x * 64, h, 64);
#pragma unroll
    for (int k = 1; k < NH; ++k) {
        load_row_h(t.H[k - 1] + (size_t)threadIdx.x * 64, x, 64);
        simt_layer<64, 64, true, 4>(W + NET_IN + (k - 1) * NET_HID, x, h);
        store_row_h(t.H[k] + (size_t)threadIdx.x * 64, h, 64);
    }
    if (out16) { load_row_h(t.H[NH - 1] + (size_t)threadIdx.x * 64, x, 64); simt_layer<64, 16, false, 4>(W + NET_IN + (NH - 1) * NET_HID, x, out16); }
}
// one layer step: gy (my row of dL/d layer output, staged for the block) -> dW += gy^T X over the tile's n_valid rows, gx = W^T gy. Two barriers: the
// staged rows are complete before the GEMM reads them, and read before the next step overwrites them.
template <int IN, int OUT, int TO, int TI>
__device__ __forceinline__ void net_layer_backward(const __half *__restrict__ W, const __half *X, __half *DY, const float *gy, float *gx, float *acc, int n_valid) {
    stage_dy(DY, gy, OUT);
    __syncthreads();
    dw_accumulate<IN, OUT, TO, TI>(DY, X, acc, n_valid);
    bwd_layer_dx<IN, OUT>(W, gy, gx);
    __syncthreads();
}
// gx = gx masked by ReLU'(my row of the activation tile) -> gy
__device__ __forceinline__ void relu_mask(const __half *act_tile, const float *gx, float *gy) {
    const __half *act = act_tile + (size_t)threadIdx.x * 64;
#pragma unroll
    for (int q = 0; q < 64; ++q) gy[q] = __half2float(act[q]) > 0.f ? gx[q] : 0.f;
}
// backward of the net on the tile: gy[0..15] = dL/d(my output row) on entry; gx[0..31] = dL/d(my input row) on return (both are 64-wide work arrays)
template <int NH>
__device__ __forceinline__ void net_backward(const __half *__restrict__ W, const NetTiles<NH> &t, __half *DY, float *gy, float *gx, NetGrad<NH> &acc, int n_valid) {
    net_layer_backward<64, 16, 2, 4>(W + NET_IN + (NH - 1) * NET_HID, t.H[NH - 1], DY, gy, gx, acc.out, n_valid);
#pragma unroll
    for (int k = NH - 1; k >= 1; --k) {  // hidden layer k: input H[k-1], output H[k]
        relu_mask(t.H[k], gx, gy);
        net_layer_backward<64, 64, 4, 8>(W + NET_IN + (k - 1) * NET_HID, t.H[k - 1], DY, gy, gx, acc.hid + (k - 1) * 32, n_valid);
    }
    relu_mask(t.H[0], gx, gy);
    net_layer_backward<32, 64, 4, 4>(W, t.X, DY, gy, gx, acc.in, n_valid);
}
// adds the accumulators to the fp32 parameter gradient (once per CTA)
template <int NH>
__device__ __forceinline__ void net_flush(const NetGrad<NH> &acc, float *__restrict__ dW) {
    dw_flush<32, 64, 4, 4>(acc.in, dW);
#pragma unroll
    for (int k = 1; k < NH; ++k) dw_flush<64, 64, 4, 8>(acc.hid + (k - 1) * 32, dW + NET_IN + (k - 1) * NET_HID);
    dw_flush<64, 16, 2, 4>(acc.out, dW + NET_IN + (NH - 1) * NET_HID);
}
// opts a backward kernel in to `smem` bytes of dynamic shared memory and returns its persistent grid for n samples (one CTA works on 128-sample tiles)
template <typename K>
static int bwd_grid(K kernel, size_t smem, int n) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    return persistent_grid((const void *)kernel, BW_THREADS, smem, (n + 127) / 128);
}

template <int DH, int CH>
__global__ void __launch_bounds__(BW_THREADS) ngp_field_bwd_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const __half *__restrict__ dens_p, const __half *__restrict__ color_p,
                                                                   const float *__restrict__ pts, int pts_stride, const float *__restrict__ dirs, int dirs_stride,
                                                                   const float4 *__restrict__ dl_draw, int n, const int32_t *__restrict__ n_dev, float *__restrict__ d_table,
                                                                   float *__restrict__ d_dens, float *__restrict__ d_color) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    if (n_dev) n = min(n, max(*n_dev, 0));
    constexpr int ND = net_params(DH), NC = net_params(CH);
    __half *p = reinterpret_cast<__half *>(smem_raw);
    __half *W = p; p += ND + NC;      // fp16 weights: density net then colour net (tcnn layout)
    const NetTiles<DH> D(p);          // X = the encoding
    const NetTiles<CH> C(p);          // X = the colour-net input row
    __half *DY = p;                   // [128][64] staged, scaled dY of the layer being processed
    for (int k = threadIdx.x; k < ND; k += BW_THREADS) W[k] = dens_p[k];
    for (int k = threadIdx.x; k < NC; k += BW_THREADS) W[ND + k] = color_p[k];
    const __half *Wd = W, *Wc = W + ND;
    NetGrad<DH> a_d;
    NetGrad<CH> a_c;
    __syncthreads();

    const int n_tiles = (n + 127) / 128;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int i = tile * 128 + threadIdx.x;
        const bool valid = i < n;
        const int n_valid = min(128, n - tile * 128);
        float px = 0.5f, py = 0.5f, pz = 0.5f, dx = 0.5f, dy = 0.5f, dz = 0.5f;
        float4 gr = make_float4(0, 0, 0, 0);
        if (valid) {
            const float *pp = pts + (size_t)i * pts_stride; px = pp[0]; py = pp[1]; pz = pp[2];
            const float *dd = dirs + (size_t)i * dirs_stride; dx = dd[0]; dy = dd[1]; dz = dd[2];
            gr = __ldg(dl_draw + i);
        }
        // ------------------------------------------------ forward recompute, layer inputs parked in shared memory
        {
            float enc[32];
#pragma unroll
            for (int l = 0; l < 16; ++l) { float2 f = hash_level(table, cells, g, l, px, py, pz); enc[2 * l] = f.x; enc[2 * l + 1] = f.y; }
            store_row_h(D.X + (size_t)threadIdx.x * 32, enc, 32);
        }
        float dout[16];
        net_forward_park<DH>(Wd, D, dout);
        {
            float cin[32];
            color_input_row(dout, dx, dy, dz, cin);
            store_row_h(C.X + (size_t)threadIdx.x * 32, cin, 32);
        }
        net_forward_park<CH>(Wc, C, nullptr);   // (the colour output layer itself is not needed: dL/draw is given)
        // ------------------------------------------------ backward: colour net, then density net with dL/ddout = (draw.w, dcin[0..14])
        float gy[64], gx[64];
#pragma unroll
        for (int k = 0; k < 16; ++k) gy[k] = 0.f;
        gy[0] = gr.x; gy[1] = gr.y; gy[2] = gr.z;
        net_backward<CH>(Wc, C, DY, gy, gx, a_c, n_valid);   // gx[0..31] = dL/dcin
        gy[0] = gr.w;
#pragma unroll
        for (int k = 0; k < 15; ++k) gy[k + 1] = gx[k];
        net_backward<DH>(Wd, D, DY, gy, gx, a_d, n_valid);   // gx[0..31] = dL/denc
        // ------------------------------------------------ hash-table gradient scatter
        if (valid) {
#pragma unroll 1
            for (int l = 0; l < 16; ++l) scatter_level(d_table, grid_cell(g, l, px, py, pz), gx[2 * l], gx[2 * l + 1]);
        }
    }
    net_flush<DH>(a_d, d_dens);
    net_flush<CH>(a_c, d_color);
}

template <int DH, int CH>
static int launch_bwd(const HashGridDev &g, const void *table, const void *cells, const void *dens, const void *color, const float *pts, int pts_stride, const float *dirs, int dirs_stride,
                      const float *dl_draw, int n, const int32_t *n_dev, float *d_table, float *d_dens, float *d_color, cudaStream_t s) {
    const size_t smem = sizeof(__half) * ((size_t)net_params(DH) + net_params(CH) + net_tile_halfs(DH) + net_tile_halfs(CH) + 128 * 64);
    auto k = ngp_field_bwd_kernel<DH, CH>;
    k<<<bwd_grid(k, smem, n), BW_THREADS, smem, s>>>(g, (const __half2 *)table, (const uint8_t *)cells, (const __half *)dens, (const __half *)color, pts, pts_stride, dirs, dirs_stride,
                                                     (const float4 *)dl_draw, n, n_dev, d_table, d_dens, d_color);
    return check_launch("ngp_mlp_backward");
}

// ---------------------------------------------------------------------------- backward of the stand-alone tcnn-shaped modules (xrnerf_b200/tcnn.py autograd)
// tcnn.Encoding(HashGrid).backward: dL/d enc fp16[n,32] -> fp32 table gradient (+=). thread = (sample, level) like hashgrid_forward_kernel.
__global__ void __launch_bounds__(256) hashgrid_backward_kernel(HashGridDev g, const float *__restrict__ x, int x_stride, int n, const __half2 *__restrict__ d_enc, float scale,
                                                                float *__restrict__ d_table) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t i = t >> 4; int l = (int)(t & 15);
    if (i >= n) return;
    const float *p = x + (size_t)i * x_stride;
    const float2 gy = __half22float2(d_enc[(size_t)i * 16 + l]);
    const float g0 = gy.x * scale, g1 = gy.y * scale;
    if (g0 == 0.f && g1 == 0.f) return;
    scatter_level(d_table, grid_cell(g, l, p[0], p[1], p[2]), g0, g1);
}

// tcnn.Network(FullyFusedMLP).backward: x fp16[n,32], dy fp16[n,16] -> dx fp16[n,32] (optional), fp32 parameter gradient (+=): the net backward above on its own.
template <int NH>
__global__ void __launch_bounds__(BW_THREADS) tcnn_mlp_bwd_kernel(const __half *__restrict__ params, const __half *__restrict__ x, const __half *__restrict__ dy, int n,
                                                                  __half *__restrict__ dx, float *__restrict__ d_params) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    constexpr int NPAR = net_params(NH);
    __half *p = reinterpret_cast<__half *>(smem_raw);
    __half *W = p; p += NPAR;
    const NetTiles<NH> T(p);
    __half *DY = p;
    for (int k = threadIdx.x; k < NPAR; k += BW_THREADS) W[k] = params[k];
    NetGrad<NH> acc;
    __syncthreads();
    const int n_tiles = (n + 127) / 128;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int i = tile * 128 + threadIdx.x;
        const bool valid = i < n;
        const int n_valid = min(128, n - tile * 128);
        {
            uint4 *dst = reinterpret_cast<uint4 *>(T.X + (size_t)threadIdx.x * 32);
            const uint4 *src = reinterpret_cast<const uint4 *>(x + (size_t)i * 32);
#pragma unroll
            for (int q = 0; q < 4; ++q) dst[q] = valid ? src[q] : make_uint4(0, 0, 0, 0);
        }
        net_forward_park<NH>(W, T, nullptr);
        float gy[64], gx[64];
#pragma unroll
        for (int k = 0; k < 16; ++k) gy[k] = valid ? __half2float(dy[(size_t)i * 16 + k]) : 0.f;
        net_backward<NH>(W, T, DY, gy, gx, acc, n_valid);
        if (dx && valid) store_row_h(dx + (size_t)i * 32, gx, 32);
    }
    net_flush<NH>(acc, d_params);
}

template <int NH>
static int launch_tcnn_mlp_bwd(const void *params, const void *x, const void *dy, int n, void *dx, float *d_params, cudaStream_t s) {
    const size_t smem = sizeof(__half) * ((size_t)net_params(NH) + net_tile_halfs(NH) + 128 * 64);
    auto k = tcnn_mlp_bwd_kernel<NH>;
    k<<<bwd_grid(k, smem, n), BW_THREADS, smem, s>>>((const __half *)params, (const __half *)x, (const __half *)dy, n, (__half *)dx, d_params);
    return check_launch("tcnn_mlp_backward");
}

// ---------------------------------------------------------------------------- density and its position gradient (xrb_ngp_density_grad: mesh normals)
// thread = point. The forward is the CUDA-core density of ngp_field_simt_kernel<true> (same gather, rounding and FMA order, so the density is bit-identical),
// keeping each hidden layer's ReLU mask (relu_mask's convention: the fp16 activation is > 0). The backward differentiates output 0 only: its weight row,
// masked, then the W^T chain down to dL/d(encoding), fp32 throughout (fp16 roundings are taken as the identity), then position_grad_level per level.
// The hidden layers are a run-time loop (density_hidden 1..4, as simt_net); each thread parks its layers' 64-bit masks in its own shared-memory slots, so
// nothing is indexed dynamically in registers. The density net's fp16 weights follow the masks in shared memory, read as broadcasts.
constexpr int DG_THREADS = 128;
__host__ __device__ constexpr size_t density_grad_smem(int dh) { return sizeof(uint64_t) * dh * DG_THREADS + sizeof(__half) * (size_t)net_params(dh); }
__global__ void __launch_bounds__(DG_THREADS) ngp_density_grad_kernel(HashGridDev g, const __half2 *__restrict__ table, const uint8_t *__restrict__ cells, const __half *__restrict__ dens_p,
                                                                      int dh, const float *__restrict__ pts, int pts_stride, int n, float *__restrict__ density, float *__restrict__ grad) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    uint64_t *s_mask = reinterpret_cast<uint64_t *>(smem_raw);              // [dh][DG_THREADS]
    __half *s_w = reinterpret_cast<__half *>(s_mask + dh * DG_THREADS);
    const int nd = net_params(dh);
    for (int k = threadIdx.x; k < nd; k += DG_THREADS) s_w[k] = dens_p[k];
    __syncthreads();
    const __half *w_out = s_w + NET_IN + (dh - 1) * NET_HID;
    for (int base = blockIdx.x * DG_THREADS; base < n; base += gridDim.x * DG_THREADS) {   // (a block-uniform base keeps the point index out of the register file)
        const int i = base + threadIdx.x;
        if (i >= n) break;
        const float *p = pts + (size_t)i * pts_stride;
        const float x = p[0], y = p[1], z = p[2];
        float a[64], b[64];
        {
            float enc[32];
#pragma unroll
            for (int l = 0; l < 16; ++l) { float2 f = hash_level(table, cells, g, l, x, y, z); enc[2 * l] = round_h(f.x); enc[2 * l + 1] = round_h(f.y); }
            simt_layer<32, 64, true>(s_w, enc, a);
        }
        for (int k = 0;; ++k) {   // a = output of hidden layer k
            uint64_t m = 0;
#pragma unroll
            for (int q = 0; q < 64; ++q) m |= (uint64_t)(a[q] > 0.f) << q;
            s_mask[k * DG_THREADS + threadIdx.x] = m;
            if (k == dh - 1) break;
            simt_layer<64, 64, true>(s_w + NET_IN + k * NET_HID, a, b);
#pragma unroll
            for (int q = 0; q < 64; ++q) a[q] = b[q];
        }
        float d;
        simt_layer<64, 1, false>(w_out, a, &d);
        if (density) density[i] = d;
        // a <- d(out 0)/d(output of the last hidden layer), masked; then one masked W^T step per hidden matrix
        uint64_t m = s_mask[(dh - 1) * DG_THREADS + threadIdx.x];
#pragma unroll
        for (int q = 0; q < 64; ++q) a[q] = (m >> q) & 1u ? __half2float(w_out[q]) : 0.f;
        for (int k = dh - 1; k >= 1; --k) {
            bwd_layer_dx<64, 64, 64>(s_w + NET_IN + (k - 1) * NET_HID, a, b);
            m = s_mask[(k - 1) * DG_THREADS + threadIdx.x];
#pragma unroll
            for (int q = 0; q < 64; ++q) a[q] = (m >> q) & 1u ? b[q] : 0.f;
        }
        bwd_layer_dx<32, 64, 64>(s_w, a, b);   // b[0..31] = d(out 0)/d(encoding)
        float3 dp = make_float3(0.f, 0.f, 0.f);
#pragma unroll
        for (int l = 0; l < 16; ++l) position_grad_level(table, g, l, x, y, z, b[2 * l], b[2 * l + 1], dp);
        float *o = grad + 3 * (size_t)i;
        o[0] = dp.x; o[1] = dp.y; o[2] = dp.z;
    }
}

// 5 * HuberLoss(delta, 'sum') of HashNerfNetwork.train_step (networks/utils/metrics.py:8-16, hashnerf.py:39-44): gradient wrt rgb and the loss value in ONE pass
__global__ void __launch_bounds__(256) huber5_kernel(const float *__restrict__ rgb, const float *__restrict__ target, int64_t n, float delta, float *__restrict__ grad, float *__restrict__ loss_accum) {
    float local = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float diff = rgb[i] - target[i], rel = fabsf(diff);
        local += rel > delta ? rel - 0.5f * delta : (0.5f / delta) * rel * rel;
        grad[i] = 5.f * (rel > delta ? copysignf(1.f, diff) : diff / delta);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    __shared__ float part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int k = 0; k < 8; ++k) t += part[k]; atomicAdd(loss_accum, 5.f * t); }
}

}  // namespace xrb

using namespace xrb;

extern "C" {

int xrb_ngp_huber5_grad(const float *rgb, const float *target, int64_t n_elements, float delta, float *grad_out, float *loss_accum, void *stream) {
    XRB_REQUIRE(n_elements >= 0 && delta > 0.f, "huber5_grad: bad arguments");
    if (n_elements == 0) return XRB_OK;
    XRB_REQUIRE(rgb && target && grad_out && loss_accum, "huber5_grad: null pointer");
    const int blocks = stride_grid((n_elements + 255) / 256, 8);
    huber5_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rgb, target, n_elements, delta, grad_out, loss_accum);
    return check_launch("huber5_grad");
}

int xrb_tcnn_hashgrid_backward(const xrb_ngp_config *cfg, const float *x, int x_stride, int n, const void *d_enc_fp16, float grad_scale, float *d_table, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && x_stride >= 3, "hashgrid_backward: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(x && d_enc_fp16 && d_table, "hashgrid_backward: null pointer");
    XRB_REQUIRE(((uintptr_t)d_table & 7) == 0 && ((uintptr_t)d_enc_fp16 & 3) == 0, "hashgrid_backward: misaligned");
    HashGridDev g; hashgrid_build(cfg, &g);
    int64_t threads = (int64_t)n * 16;
    hashgrid_backward_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, x, x_stride, n, (const __half2 *)d_enc_fp16, grad_scale, d_table);
    return check_launch("hashgrid_backward");
}

int xrb_tcnn_mlp_backward(const void *params_fp16, const void *x_fp16, const void *dy_fp16, int n, int in_w, int width, int n_hidden, void *dx_fp16, float *d_params, void *stream) {
    XRB_REQUIRE(n >= 0, "mlp_backward: negative size");
    if (in_w != 32 || width != 64 || n_hidden < 1 || n_hidden > 4) { set_error("mlp_backward: only in=32 (padded), width=64, 1..4 hidden layers"); return XRB_E_UNSUPPORTED; }
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(params_fp16 && x_fp16 && dy_fp16 && d_params, "mlp_backward: null pointer");
    XRB_REQUIRE(((uintptr_t)x_fp16 & 15) == 0 && (!dx_fp16 || ((uintptr_t)dx_fp16 & 3) == 0), "mlp_backward: x must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    switch (n_hidden) {
        case 1: return launch_tcnn_mlp_bwd<1>(params_fp16, x_fp16, dy_fp16, n, dx_fp16, d_params, s);
        case 2: return launch_tcnn_mlp_bwd<2>(params_fp16, x_fp16, dy_fp16, n, dx_fp16, d_params, s);
        case 3: return launch_tcnn_mlp_bwd<3>(params_fp16, x_fp16, dy_fp16, n, dx_fp16, d_params, s);
        default: return launch_tcnn_mlp_bwd<4>(params_fp16, x_fp16, dy_fp16, n, dx_fp16, d_params, s);
    }
}

int xrb_ngp_mlp_backward(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const void *color_fp16, const float *pts, int pts_stride, const float *dirs,
                         int dirs_stride, const float *dl_draw, int n, float *d_table, float *d_density, float *d_color, void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && pts_stride >= 3 && dirs_stride >= 3, "ngp_mlp_backward: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(table && density_fp16 && color_fp16 && pts && dirs && dl_draw && d_table && d_density && d_color, "ngp_mlp_backward: null pointer");
    XRB_REQUIRE(((uintptr_t)dl_draw & 15) == 0 && ((uintptr_t)d_table & 7) == 0, "ngp_mlp_backward: dl_draw must be 16-byte, d_table 8-byte aligned");
    HashGridDev g; e = table_setup(cfg, table, &g); if (e) return e;
    cudaStream_t s = (cudaStream_t)stream;
#define XRB_BW(DH, CH) if (cfg->density_hidden == DH && cfg->color_hidden == CH) return launch_bwd<DH, CH>(g, table->table_fp16, table->cell_image, density_fp16, color_fp16, pts, pts_stride, dirs, dirs_stride, dl_draw, n, nullptr, d_table, d_density, d_color, s);
    XRB_BW(1, 1) XRB_BW(1, 2) XRB_BW(2, 2) XRB_BW(1, 3) XRB_BW(2, 3)
#undef XRB_BW
    set_error("ngp_mlp_backward: (density_hidden, color_hidden) must be one of (1,1) (1,2) (2,2) (1,3) (2,3)");
    return XRB_E_UNSUPPORTED;
}

int xrb_ngp_density_grad(const xrb_ngp_config *cfg, const xrb_ngp_table *table, const void *density_fp16, const float *pts, int pts_stride, int n, float *density, float *grad,
                         void *stream) {
    int e = check_cfg(cfg); if (e) return e;
    XRB_REQUIRE(n >= 0 && pts_stride >= 3, "ngp_density_grad: bad size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(table && density_fp16 && pts && grad, "ngp_density_grad: null pointer");
    HashGridDev g; e = table_setup(cfg, table, &g); if (e) return e;
    const size_t smem = density_grad_smem(cfg->density_hidden);   // <= 34 KB (density_hidden 4): no opt-in needed
    const int grid = persistent_grid((const void *)ngp_density_grad_kernel, DG_THREADS, smem, (n + DG_THREADS - 1) / DG_THREADS);
    ngp_density_grad_kernel<<<grid, DG_THREADS, smem, (cudaStream_t)stream>>>(g, (const __half2 *)table->table_fp16, (const uint8_t *)table->cell_image, (const __half *)density_fp16,
                                                                              cfg->density_hidden, pts, pts_stride, n, density, grad);
    return check_launch("ngp_density_grad");
}

}  // extern "C"
