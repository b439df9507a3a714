// xrnerf_b200 — the optimiser step of the Instant-NGP trainer in every gradient-exchange mode. One Adam + EMA element update (adam_update) and one host
// computation of its hyper-parameters (adam_hyper) serve both the local step (xrb_adam_ema_step*: one rank, or after a collective) and the peer step below.
//
// The peer step: the data-parallel optimiser step as ONE exchange over NVLink peer memory.
// The reference trains under MMDistributedDataParallel: torch DDP all-reduces the dense fp32 gradient (49 MB for the hash table) and every rank runs the same
// torch.optim.Adam over all 12.2 M parameters (core/apis/train.py:28-36, hashnerf.py:32-52). Round 2's first answer was reduce-scatter (bf16) -> Adam on this
// rank's 1/N -> all-gather (fp16) through NCCL: three collectives + five kernels per step, ~113 us of which ~90 are launch / rendezvous latency of the collectives.
// Here the exchange IS the optimiser kernel. Every rank owns one cudaMalloc'ed exchange block, mapped into every other process with CUDA IPC:
//     flags | g16[padded] bf16 packed gradient of the hash table | gmlp[n_mlp] fp32 gradient of the two MLPs | t16[padded] fp16 working copy of the table
//   publish   (1 kernel)  my fp32 gradients -> g16 / gmlp of MY block; the last CTA raises ready[me] = step in every rank's flags (release, system scope)
//   adam_peer (1 kernel)  waits for ready[*] == step, then for my 1/N of the table: g = sum over ranks of g16_p[i] (16-byte loads over NVLink), Adam on my fp32
//                         master / moments (local HBM), the new fp16 value stored into t16 of EVERY rank (16-byte stores over NVLink) = the all-gather;
//                         the small MLPs: every rank sums all ranks' gmlp in the same order and updates its own copy (identical on all ranks, nothing to send back);
//                         the last CTA raises done[me] = step everywhere
//   wait_done (1 kernel)  waits for done[*] == step: my t16 now holds every rank's slice, and nobody reads my g16 any more (it may be overwritten by the next step)
// NVLink bytes per rank and step: (N-1)/N x 12.2 M x (2 + 2) B - what reduce-scatter + all-gather move - with no collective launch. Waits poll LOCAL memory.
// A wait that lasts longer than ~10 s sets status != 0 in the block (read by xrb_peer_status) instead of hanging the GPU.
#include "common.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string.h>
#include <math.h>

namespace xrb {

// ---------------------------------------------------------------------------- the Adam + EMA element update
struct AdamHyper { float lr, b1, b2, eps, wd, bc1, bc2_sqrt_inv, grad_mul, ema_m; };

static AdamHyper adam_hyper(float lr, float beta1, float beta2, float eps, float weight_decay, int step, float grad_div, float ema_momentum) {
    const double bc1 = 1.0 - pow((double)beta1, step), bc2 = 1.0 - pow((double)beta2, step);
    return AdamHyper{lr, beta1, beta2, eps, weight_decay, (float)bc1, (float)(1.0 / sqrt(bc2)), 1.f / grad_div, ema_momentum};
}

// torch.optim.Adam on element i (weight_decay folded into the gradient), then mmcv's EMAHook.after_train_iter on it: ema[i] = (1 - m) ema[i] + m w
// (ema == NULL: no EMA). m, v: the element's moments, updated in place. Returns the new weight.
__device__ __forceinline__ float adam_update(float w, float g, float &m, float &v, float *ema, int64_t i, const AdamHyper &h) {
    const float gval = g * h.grad_mul + h.wd * w;
    m = h.b1 * m + (1.f - h.b1) * gval;
    v = h.b2 * v + (1.f - h.b2) * gval * gval;
    w -= (h.lr / h.bc1) * (m / (sqrtf(v) * h.bc2_sqrt_inv + h.eps));   // sqrt(v)/sqrt(bias_correction2) + eps
    if (ema) ema[i] = ema[i] * (1.f - h.ema_m) + h.ema_m * w;
    return w;
}

// ---------------------------------------------------------------------------- local step: Adam (+ fp16 shadow refresh) over one vector
template <typename G> __device__ __forceinline__ float grad_load(const G *g, int64_t i);
template <> __device__ __forceinline__ float grad_load<float>(const float *g, int64_t i) { return g[i]; }
template <> __device__ __forceinline__ float grad_load<__nv_bfloat16>(const __nv_bfloat16 *g, int64_t i) { return __bfloat162float(g[i]); }

template <typename G>
__global__ void __launch_bounds__(256) adam_kernel(float *__restrict__ p, __half *__restrict__ p16, const G *__restrict__ grad, float *__restrict__ m, float *__restrict__ v,
                                                   float *__restrict__ ema, int64_t n, AdamHyper h) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float w = adam_update(p[i], grad_load<G>(grad, i), m[i], v[i], ema, i, h);
        p[i] = w;
        if (p16) p16[i] = __float2half_rn(w);
    }
}

// fp32 gradient -> bf16 (the wire format of the sharded data-parallel step: reduce-scatter in bf16, see xrnerf_b200/train.py)
__global__ void __launch_bounds__(256) pack_bf16_kernel(const float *__restrict__ src, __nv_bfloat16 *__restrict__ dst, int64_t n) {
    int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
    for (; i + 3 < n; i += stride) {
        float4 v = *reinterpret_cast<const float4 *>(src + i);
        __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 o; o.x = *reinterpret_cast<uint32_t *>(&a); o.y = *reinterpret_cast<uint32_t *>(&b);
        *reinterpret_cast<uint2 *>(dst + i) = o;
    }
    if (blockIdx.x == 0 && threadIdx.x < 4) { int64_t t = (n & ~(int64_t)3) + threadIdx.x; if (t < n) dst[t] = __float2bfloat16_rn(src[t]); }
}

// ---------------------------------------------------------------------------- peer step
constexpr int PEER_MAX = 8;
constexpr long long PEER_SPIN_LIMIT = 20000000000ll;   // cycles (~10 s)
// flags (uint32) at the start of a block: ready[8], done[8], ticket[2], status
constexpr int F_READY = 0, F_DONE = 8, F_TICKET = 16, F_STATUS = 18;

struct PeerDev {
    int world, rank;
    uint8_t *base[PEER_MAX];
    size_t off_g16, off_gmlp, off_t16;
    int64_t n_table, per, n_mlp;
};

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) { uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

// every CTA calls this after its last store of the phase; the last one to arrive raises flag[slot + rank] = step in every rank's block
__device__ __forceinline__ void peer_signal_when_all_ctas_done(const PeerDev &P, int slot, uint32_t step, int ticket) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t *mine = reinterpret_cast<uint32_t *>(P.base[P.rank]);
        const uint32_t t = atomicAdd(mine + F_TICKET + ticket, 1u);
        if (t == gridDim.x - 1) {
            mine[F_TICKET + ticket] = 0;
            __threadfence_system();
            for (int p = 0; p < P.world; ++p) st_release_sys(reinterpret_cast<uint32_t *>(P.base[p]) + slot + P.rank, step);
        }
    }
}
// thread 0 polls MY flags until every rank's flag[slot + p] reached step; the CTA then proceeds. false (and status set) after ~10 s.
__device__ __forceinline__ bool peer_wait_all(const PeerDev &P, int slot, uint32_t step) {
    __shared__ int ok;
    if (threadIdx.x == 0) {
        const uint32_t *mine = reinterpret_cast<const uint32_t *>(P.base[P.rank]);
        const long long t0 = clock64();
        int good = 1;
        for (int p = 0; p < P.world && good; ++p)
            while ((int32_t)(ld_acquire_sys(mine + slot + p) - step) < 0) {
                if (clock64() - t0 > PEER_SPIN_LIMIT) { good = 0; atomicExch(reinterpret_cast<unsigned int *>(P.base[P.rank]) + F_STATUS, 1u + (unsigned)slot); break; }
                __nanosleep(200);
            }
        ok = good;
    }
    __syncthreads();
    __threadfence_system();
    return ok != 0;
}

__global__ void __launch_bounds__(256) peer_publish_kernel(PeerDev P, const float *__restrict__ g_table, const float *__restrict__ g_mlp, uint32_t step) {
    __nv_bfloat16 *g16 = reinterpret_cast<__nv_bfloat16 *>(P.base[P.rank] + P.off_g16);
    float *gm = reinterpret_cast<float *>(P.base[P.rank] + P.off_gmlp);
    const int64_t padded = P.per * P.world, n4 = padded / 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = 4 * i + k < P.n_table ? g_table[4 * i + k] : 0.f;
        __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
        uint2 w; w.x = *reinterpret_cast<uint32_t *>(&a); w.y = *reinterpret_cast<uint32_t *>(&b);
        reinterpret_cast<uint2 *>(g16)[i] = w;
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P.n_mlp; i += (int64_t)gridDim.x * blockDim.x) gm[i] = g_mlp[i];
    peer_signal_when_all_ctas_done(P, F_READY, step, 0);
}

struct MlpGroup { float *p; __half *p16; float *m, *v, *ema; int64_t n, g_off; };

__global__ void __launch_bounds__(256) peer_adam_kernel(PeerDev P, float *__restrict__ master /*my slice*/, float *__restrict__ m, float *__restrict__ v, float *__restrict__ ema, int64_t cnt /*live elements of my slice*/,
                                                        AdamHyper h, MlpGroup g0, MlpGroup g1, uint32_t step) {
    if (!peer_wait_all(P, F_READY, step)) { peer_signal_when_all_ctas_done(P, F_DONE, step, 1); return; }
    const int64_t begin = P.per * P.rank;
    // ---- my slice of the table, 8 elements (16 bytes of bf16 / fp16) per thread and iteration
    const int64_t n8 = (cnt + 7) / 8;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n8; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = 8 * q;
        float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int p = 0; p < P.world; ++p) {
            const uint4 w = __ldcv(reinterpret_cast<const uint4 *>(P.base[p] + P.off_g16 + 2 * (size_t)(begin + i)));   // never from a cache: the block is rewritten every step
            const __nv_bfloat162 *b = reinterpret_cast<const __nv_bfloat162 *>(&w);
#pragma unroll
            for (int k = 0; k < 4; ++k) { const float2 f = __bfloat1622float2(b[k]); g[2 * k] += f.x; g[2 * k + 1] += f.y; }
        }
        __half out[8];
        if (i + 8 <= cnt) {
            float4 w0 = *reinterpret_cast<float4 *>(master + i), w1 = *reinterpret_cast<float4 *>(master + i + 4);
            float4 m0 = *reinterpret_cast<float4 *>(m + i), m1 = *reinterpret_cast<float4 *>(m + i + 4), v0 = *reinterpret_cast<float4 *>(v + i), v1 = *reinterpret_cast<float4 *>(v + i + 4);
            float *wp = &w0.x, *wq = &w1.x, *mp = &m0.x, *mq = &m1.x, *vp = &v0.x, *vq = &v1.x;
#pragma unroll
            for (int k = 0; k < 4; ++k) wp[k] = adam_update(wp[k], g[k], mp[k], vp[k], ema, i + k, h);
#pragma unroll
            for (int k = 0; k < 4; ++k) wq[k] = adam_update(wq[k], g[4 + k], mq[k], vq[k], ema, i + 4 + k, h);
            *reinterpret_cast<float4 *>(master + i) = w0; *reinterpret_cast<float4 *>(master + i + 4) = w1;
            *reinterpret_cast<float4 *>(m + i) = m0; *reinterpret_cast<float4 *>(m + i + 4) = m1; *reinterpret_cast<float4 *>(v + i) = v0; *reinterpret_cast<float4 *>(v + i + 4) = v1;
#pragma unroll
            for (int k = 0; k < 4; ++k) { out[k] = __float2half_rn(wp[k]); out[4 + k] = __float2half_rn(wq[k]); }
        } else {
            for (int k = 0; k < 8; ++k) {
                float w = 0.f;
                if (i + k < cnt) {
                    w = adam_update(master[i + k], g[k], m[i + k], v[i + k], ema, i + k, h);
                    master[i + k] = w;
                }
                out[k] = __float2half_rn(w);
            }
        }
        const uint4 ov = *reinterpret_cast<const uint4 *>(out);
        for (int p = 0; p < P.world; ++p) *reinterpret_cast<uint4 *>(P.base[p] + P.off_t16 + 2 * (size_t)(begin + i)) = ov;   // the all-gather: my slice into every rank's working table
    }
    // ---- the two small MLPs: every rank reduces all ranks' gradients in rank order and updates its own copy
    for (int grp = 0; grp < 2; ++grp) {
        const MlpGroup G = grp ? g1 : g0;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < G.n; i += (int64_t)gridDim.x * blockDim.x) {
            float g = 0.f;
            for (int p = 0; p < P.world; ++p) g += __ldcv(reinterpret_cast<const float *>(P.base[p] + P.off_gmlp) + G.g_off + i);
            const float w = adam_update(G.p[i], g, G.m[i], G.v[i], G.ema, i, h);
            G.p[i] = w;
            if (G.p16) G.p16[i] = __float2half_rn(w);
        }
    }
    peer_signal_when_all_ctas_done(P, F_DONE, step, 1);
}

__global__ void peer_wait_done_kernel(PeerDev P, uint32_t step) { peer_wait_all(P, F_DONE, step); }

static int peer_dev(const xrb_peer_layout *L, PeerDev *P) {
    if (!L || L->world < 1 || L->world > PEER_MAX || L->rank < 0 || L->rank >= L->world) { set_error("peer: world must be 1..8 and 0 <= rank < world"); return XRB_E_BADARG; }
    if (L->per <= 0 || (L->per % 8) != 0 || L->n_table < 0 || L->n_table > L->per * L->world || L->n_mlp < 0) { set_error("peer: slice length must be a positive multiple of 8 covering the table"); return XRB_E_BADARG; }
    if ((L->off_g16 % 16) || (L->off_t16 % 16) || (L->off_gmlp % 16) || L->off_g16 < 128) { set_error("peer: offsets must be 16-byte aligned and leave 128 bytes of flags"); return XRB_E_BADARG; }
    P->world = L->world; P->rank = L->rank; P->off_g16 = L->off_g16; P->off_gmlp = L->off_gmlp; P->off_t16 = L->off_t16; P->n_table = L->n_table; P->per = L->per; P->n_mlp = L->n_mlp;
    for (int p = 0; p < L->world; ++p) { if (!L->base[p]) { set_error("peer: null block pointer"); return XRB_E_BADARG; } P->base[p] = (uint8_t *)L->base[p]; }
    return XRB_OK;
}

}  // namespace xrb

using namespace xrb;

extern "C" {

static int adam_launch(float *param, void *param_fp16, const void *grad, bool grad_bf16, float *exp_avg, float *exp_avg_sq, int64_t n, float lr, float beta1, float beta2, float eps,
                       float weight_decay, int step, float grad_div, float *ema, float ema_momentum, void *stream) {
    XRB_REQUIRE(n >= 0 && step >= 1 && grad_div != 0.f && ema_momentum >= 0.f && ema_momentum <= 1.f, "adam_step: bad arguments");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(param && grad && exp_avg && exp_avg_sq, "adam_step: null pointer");
    const AdamHyper h = adam_hyper(lr, beta1, beta2, eps, weight_decay, step, grad_div, ema_momentum);
    const int blocks = stride_grid((n + 255) / 256, 16);
    if (grad_bf16)
        adam_kernel<__nv_bfloat16><<<blocks, 256, 0, (cudaStream_t)stream>>>(param, (__half *)param_fp16, (const __nv_bfloat16 *)grad, exp_avg, exp_avg_sq, ema, n, h);
    else
        adam_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(param, (__half *)param_fp16, (const float *)grad, exp_avg, exp_avg_sq, ema, n, h);
    return check_launch("adam_step");
}

int xrb_adam_ema_step(float *param, void *param_fp16, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                      int step, float grad_div, float *ema, float ema_momentum, void *stream) {
    return adam_launch(param, param_fp16, grad, false, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, grad_div, ema, ema_momentum, stream);
}

int xrb_adam_ema_step_bf16grad(float *param, void *param_fp16, const void *grad_bf16, float *exp_avg, float *exp_avg_sq, int64_t n, float lr, float beta1, float beta2, float eps,
                               float weight_decay, int step, float grad_div, float *ema, float ema_momentum, void *stream) {
    return adam_launch(param, param_fp16, grad_bf16, true, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, grad_div, ema, ema_momentum, stream);
}

int xrb_pack_bf16(const float *src, void *dst_bf16, int64_t n, void *stream) {
    XRB_REQUIRE(n >= 0, "pack_bf16: negative size");
    if (n == 0) return XRB_OK;
    XRB_REQUIRE(src && dst_bf16, "pack_bf16: null pointer");
    XRB_REQUIRE(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst_bf16 & 7) == 0, "pack_bf16: misaligned");
    const int blocks = stride_grid((n / 4 + 255) / 256, 16);
    pack_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, (__nv_bfloat16 *)dst_bf16, n);
    return check_launch("pack_bf16");
}

int xrb_peer_alloc(size_t bytes, void **ptr, void *ipc_handle64) {
    XRB_REQUIRE(ptr && ipc_handle64 && bytes >= 128, "peer_alloc: null pointer / block smaller than its flags");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return (int)e; }
    cudaMemset(p, 0, bytes);
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); cudaFree(p); return (int)e; }
    memcpy(ipc_handle64, &h, 64);
    cudaDeviceSynchronize();
    *ptr = p;
    return XRB_OK;
}
int xrb_peer_open(const void *ipc_handle64, void **ptr) {
    XRB_REQUIRE(ptr && ipc_handle64, "peer_open: null pointer");
    cudaIpcMemHandle_t h; memcpy(&h, ipc_handle64, 64);
    cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); cudaGetLastError(); return (int)e; }
    return XRB_OK;
}
int xrb_peer_close(void *ptr) { if (!ptr) return XRB_OK; cudaError_t e = cudaIpcCloseMemHandle(ptr); if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return (int)e; } return XRB_OK; }
int xrb_peer_free(void *ptr) { if (!ptr) return XRB_OK; cudaError_t e = cudaFree(ptr); if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return (int)e; } return XRB_OK; }

int xrb_peer_publish_grads(const xrb_peer_layout *L, const float *grad_table, const float *grad_mlp, uint32_t step, void *stream) {
    PeerDev P; int e = peer_dev(L, &P); if (e) return e;
    XRB_REQUIRE(grad_table && (grad_mlp || L->n_mlp == 0) && step > 0, "peer_publish_grads: null pointer / step must start at 1");
    const int blocks = stride_grid((P.per * P.world / 4 + 255) / 256, 8);
    peer_publish_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(P, grad_table, grad_mlp, step);
    return check_launch("peer_publish_grads");
}

int xrb_peer_adam_step(const xrb_peer_layout *L, float *master_slice, float *exp_avg_slice, float *exp_avg_sq_slice, float *ema_slice, const xrb_peer_mlp_group *mlp0,
                       const xrb_peer_mlp_group *mlp1, float lr, float beta1, float beta2, float eps, float weight_decay, int opt_step, float ema_momentum, uint32_t step, void *stream) {
    PeerDev P; int e = peer_dev(L, &P); if (e) return e;
    const int64_t begin = P.per * P.rank, cnt = begin >= P.n_table ? 0 : (P.n_table - begin < P.per ? P.n_table - begin : P.per);
    XRB_REQUIRE(opt_step >= 1 && step > 0 && mlp0 && mlp1, "peer_adam_step: bad step / null group");
    XRB_REQUIRE(cnt == 0 || (master_slice && exp_avg_slice && exp_avg_sq_slice), "peer_adam_step: null slice pointer");
    XRB_REQUIRE((((uintptr_t)master_slice | (uintptr_t)exp_avg_slice | (uintptr_t)exp_avg_sq_slice) & 15) == 0, "peer_adam_step: slices must be 16-byte aligned");
    XRB_REQUIRE(!(ema_slice && !(ema_momentum > 0.f && ema_momentum < 1.f)), "peer_adam_step: EMA momentum must be in (0,1)");
    XRB_REQUIRE(mlp0->g_off >= 0 && mlp1->g_off >= 0 && mlp0->g_off + mlp0->n <= P.n_mlp && mlp1->g_off + mlp1->n <= P.n_mlp, "peer_adam_step: MLP group outside the gradient block");
    const AdamHyper h = adam_hyper(lr, beta1, beta2, eps, weight_decay, opt_step, (float)P.world, ema_momentum);
    MlpGroup g0{mlp0->param, (__half *)mlp0->param_fp16, mlp0->exp_avg, mlp0->exp_avg_sq, mlp0->ema, mlp0->n, mlp0->g_off};
    MlpGroup g1{mlp1->param, (__half *)mlp1->param_fp16, mlp1->exp_avg, mlp1->exp_avg_sq, mlp1->ema, mlp1->n, mlp1->g_off};
    const int blocks = stride_grid(((cnt + 7) / 8 + 255) / 256, 8);
    peer_adam_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(P, master_slice, exp_avg_slice, exp_avg_sq_slice, ema_slice, cnt, h, g0, g1, step);
    peer_wait_done_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(P, step);
    return check_launch("peer_adam_step");
}

int xrb_peer_status(const void *own_block, uint32_t *status_host, void *stream) {
    XRB_REQUIRE(own_block && status_host, "peer_status: null pointer");
    cudaError_t e = cudaMemcpyAsync(status_host, (const uint32_t *)own_block + F_STATUS, sizeof(uint32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return (int)e; }
    return XRB_OK;
}

}  // extern "C"
