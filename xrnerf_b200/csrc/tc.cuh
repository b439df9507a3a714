// xrnerf_b200 — thin inline-PTX wrappers for the Hopper (sm_90a) tensor-core path: wgmma (warpgroup MMA, shared-memory operands,
// register accumulators), mbarrier, 1-D TMA bulk copy, proxy fences. No CUTLASS dependency; descriptor encodings follow the PTX ISA
// ("Matrix Descriptor Format" of wgmma) and cute/arch/mma_sm90_desc.hpp. Also the one definition of the tile-image layout those
// descriptors read (end of file).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace xrb { namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) { while (!mbar_try_wait(bar, parity)) {} }

// ---- TMA: 1-D bulk copy global -> shared, completion on an mbarrier
__device__ __forceinline__ void tma_bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes),
                 "r"(smem_u32(bar)) : "memory");
}
// 1-D bulk copy shared -> global (bulk-group completion)
__device__ __forceinline__ void tma_bulk_s2g(void *gdst, const void *ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_commit_wait_read() { asm volatile("cp.async.bulk.commit_group;\n\tcp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- fences / barriers
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n_threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory"); }

// ---- register re-balancing between warpgroups (all 128 threads of a warpgroup execute it): a producer warpgroup that only issues TMA copies hands its
// registers to the MMA warpgroups, whose accumulators live in registers
template <uint32_t R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- wgmma shared-memory matrix descriptors (sm_90: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46), layout type [62,64): 1 = 128-byte swizzle, 2 = 64-byte)
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo, uint32_t sbo, uint32_t layout) {
    return (uint64_t)((addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}
// K-major, SWIZZLE_128B: one row = 64 fp16 (128 bytes), 8-row atoms 1024 B apart (SBO); LBO unused. A K step of 16 advances the start by 32 bytes.
__device__ __forceinline__ uint64_t desc_k128(uint32_t addr) { return smem_desc(addr, 16, 1024, 1); }
// K-major, SWIZZLE_64B: one row = 32 fp16 (64 bytes), 8-row atoms 512 B apart
__device__ __forceinline__ uint64_t desc_k64(uint32_t addr) { return smem_desc(addr, 16, 512, 2); }
// MN-major, SWIZZLE_128B: 64 MN elements contiguous per K row (128 bytes), 8-row K groups 1024 B apart (SBO), next 64-element MN atom `lbo` bytes away.
// A K step of 16 advances the start by 2048 bytes.
__device__ __forceinline__ uint64_t desc_mn128(uint32_t addr, uint32_t lbo) { return smem_desc(addr, lbo, 1024, 1); }

// ---- wgmma: D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands from shared memory, fp32 accumulators in registers; issued by all 128 threads of a
// warpgroup. TA / TB: 0 = K-major, 1 = MN-major. scale_d == 0 overwrites D.
// Accumulator fragment (PTX ISA, wgmma .m64nNk16 D fragment): thread t of the warpgroup, w = t / 32, l = t % 32, register i:
//   row = 16 w + l / 4 + 8 ((i % 4) / 2),   col = 8 (i / 4) + 2 (l % 4) + (i % 2)
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float *d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<32> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float *d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<64> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float *d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<128> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float *d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<256> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float *d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, %131, %132;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};

template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma(float *d, uint64_t ad, uint64_t bd, uint32_t scale_d) { Wgmma<N>::template mma<TA, TB>(d, ad, bd, scale_d); }

// ---- wgmma with A from registers: D[64 x N] (+)= A[64 x 16] * B[16 x N], B K-major from shared memory. A fragment (PTX ISA, wgmma .m64nNk16 A
// fragment, f16): thread t, w = t / 32, l = t % 32, register j holds the fp16 pair (row, col), (row, col + 1) with
//   row = 16 w + l / 4 + 8 (j % 2),   col = 2 (l % 4) + 8 (j / 2)
// i.e. the registers 8s..8s+7 of an m64nN accumulator (columns 16s..16s+15), packed pairwise, are the A fragment of K step s: each warp's rows stay in that warp.
// The A registers must not be written until the wgmma that reads them has been waited for.
template <int N> struct WgmmaRA;
template <> struct WgmmaRA<16> {
    static __device__ __forceinline__ void mma(float *d, const uint32_t *a, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd), "r"(scale_d));
    }
};
template <> struct WgmmaRA<64> {
    static __device__ __forceinline__ void mma(float *d, const uint32_t *a, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd), "r"(scale_d));
    }
};
template <int N>
__device__ __forceinline__ void wgmma_ra(float *d, const uint32_t *a, uint64_t bd, uint32_t scale_d) { WgmmaRA<N>::mma(d, a, bd, scale_d); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait points
template <int N>
__device__ __forceinline__ void acc_fence(float *d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// row (0..63) and first column of accumulator register pair j (registers 4j, 4j+1: row r; 4j+2, 4j+3: row r + 8)
__device__ __forceinline__ uint32_t frag_row(uint32_t t) { return ((t >> 5) << 4) + ((t & 31) >> 2); }
__device__ __forceinline__ uint32_t frag_col(uint32_t t, uint32_t j) { return 8u * j + 2u * (t & 3u); }

}  // namespace tc

// ---- tile images: a matrix [rows x C] stored per 128-row tile as C/64 blocks of [128 x 64] fp16, K-major with the 128-byte swizzle desc_k128
// reads. Row r of a block is 128 bytes (eight 16-byte chunks) in 8-row atoms of 1024 B; chunk c of row r sits at chunk position c ^ (r % 8).
// The NGP field's A tile and every weight slab [N x 64] use the same block layout.
constexpr uint32_t TILE_ROWS = 128, TILE_BLOCK_COLS = 64, TILE_BLOCK_BYTES = TILE_ROWS * TILE_BLOCK_COLS * 2;

// byte offset of 16-byte chunk `chunk16` (0..7) of `row` in a block = sw128_row(row) + sw128_chunk(row, chunk16)
__host__ __device__ __forceinline__ uint32_t sw128_row(uint32_t row) { return (row >> 3) * 1024u + (row & 7u) * 128u; }
// the address of `row` in the block at blk, its two terms added to the pointer one by one (the schedule of the fast IPE encoder depends on it)
__device__ __forceinline__ uint8_t *sw128_row_ptr(uint8_t *blk, uint32_t row) { return blk + (row >> 3) * 1024u + (row & 7u) * 128u; }
__host__ __device__ __forceinline__ uint32_t sw128_chunk(uint32_t row, uint32_t chunk16) { return (chunk16 ^ (row & 7u)) << 4; }
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk16) { return sw128_row(row) + sw128_chunk(row, chunk16); }
// address of the fp16 element (row, col) of the block at blk, col < 64
template <class B> __device__ __forceinline__ B *sw128_elem(B *blk, uint32_t row, uint32_t col) { return blk + sw128_offset(row, col >> 3) + (col & 7u) * 2u; }

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
// 8 floats -> one chunk of fp16
__device__ __forceinline__ uint4 pack_h8(const float *v) { return make_uint4(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]), pack_h2(v[4], v[5]), pack_h2(v[6], v[7])); }
__device__ __forceinline__ void st_chunk(uint8_t *p, uint4 v) { *reinterpret_cast<uint4 *>(p) = v; }
// 8 floats as fp16 into chunk `chunk16` of `row`, given the row's address (kernels that write a whole row compute it once)
__device__ __forceinline__ void st_row_chunk(uint8_t *row_ptr, uint32_t row, uint32_t chunk16, const float *v) { st_chunk(row_ptr + sw128_chunk(row, chunk16), pack_h8(v)); }

// block b of tile `tile` of an image with n_blk blocks per tile, and the bytes of an image of n_rows rows
__host__ __device__ __forceinline__ uint8_t *tile_block(uint8_t *image, int64_t tile, int n_blk, int b) { return image + ((size_t)tile * n_blk + b) * TILE_BLOCK_BYTES; }
__host__ __device__ __forceinline__ size_t tile_image_bytes(int64_t n_rows, int n_blk) { return (size_t)((n_rows + TILE_ROWS - 1) / TILE_ROWS) * n_blk * TILE_BLOCK_BYTES; }

// chunk `chunk` of row `row` of a weight slab <- fp16 of W[row][col0 + 8 chunk ..] (W fp32 row-major with row length ld); zero for rows >= n and
// for the columns from `valid` on
__device__ __forceinline__ void pack_slab_chunk(uint8_t *slab, const float *W, int ld, int n, int col0, int valid, int row, int chunk) {
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { const int c = 8 * chunk + e; v[e] = (row < n && c < valid) ? W[(size_t)row * ld + col0 + c] : 0.f; }
    st_chunk(slab + sw128_offset(row, chunk), pack_h8(v));
}

}  // namespace xrb
