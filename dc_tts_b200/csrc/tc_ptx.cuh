// tc_ptx.cuh -- thin inline-PTX wrappers for the sm_90a features the tensor-core kernels
// use: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory
// descriptors), thread-block clusters and distributed shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dctts { namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- mbarrier ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait (about 2 s of SM clock): a protocol bug must surface as a trapped launch -- an
// error the host sees -- never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > 4000000000ll) __trap();
}
// The same wait with acquire semantics at CLUSTER scope: for a phase completed by other CTAs' st.async, whose complete_tx
// releases their stores at cluster scope.
__device__ __forceinline__ bool mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait_cluster(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait_cluster(bar, parity))
        if (clock64() - t0 > 4000000000ll) __trap();
}
// st.async: registers -> shared memory of a CTA of the cluster (dst and bar are shared::cluster addresses, from mapa), the
// bytes completing as transaction count on that CTA's mbarrier `bar` (which must live in the same CTA as dst)
__device__ __forceinline__ void st_async_v4(uint32_t dst, float4 v, uint32_t bar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
                 :: "r"(dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(bar) : "memory");
}
__device__ __forceinline__ void st_async_v2(uint32_t dst, float a, float b, uint32_t bar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
                 :: "r"(dst), "f"(a), "f"(b), "r"(bar) : "memory");
}

// ---- TMA ----------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}

// multicast variant: the box lands at the same CTA-relative offset in every CTA of `mask`, and
// each destination CTA's barrier (same offset) receives the complete_tx
__device__ __forceinline__ void tma_load_3d_mc(const void* tmap, uint64_t* bar, void* dst, int c0, int c1, int c2, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
                 : "memory");
}

// TMA store: shared (swizzled tile) -> global, rows/columns outside the tensor are clipped
__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 :: "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_commit_and_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma (sm_90a warpgroup MMA) ---------------------------------------------------------
// D (registers of the 128 threads of a warpgroup) (+)= A[smem desc] * B[smem desc]^T, fp16 inputs, fp32 accumulate,
// M = 64.  Fragment of m64nNk16: register i of thread t (warp w = t/32 of the warpgroup, lane l) holds
// row 16w + l/4 + 8*((i>>1)&1), column 8*(i>>2) + 2*(l&3) + (i&1).
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

#define DCTTS_WG_D8(o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
// N = 16 * NQ columns (NQ = 1..4): the first 8 * NQ registers of d
template <int NQ, int R>
__device__ __forceinline__ void wgmma_f16(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(NQ >= 1 && NQ <= 4 && 8 * NQ <= R, "wgmma_f16: 16..64 columns");
    if constexpr (NQ == 1) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0) : "l"(da), "l"(db), "r"(accumulate));
    } else if constexpr (NQ == 2) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15},"
                     " %16, %17, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8) : "l"(da), "l"(db), "r"(accumulate));
    } else if constexpr (NQ == 3) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                     "%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8), DCTTS_WG_D8(16) : "l"(da), "l"(db), "r"(accumulate));
    } else {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                     "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8), DCTTS_WG_D8(16), DCTTS_WG_D8(24) : "l"(da), "l"(db), "r"(accumulate));
    }
}
// One m64nNk16 over the full accumulator width of a CTA: N = 64, 80, 144 or 256 (the widths the networks' blocks use),
// d holds the N / 2 fp32 registers of the fragment above
template <int N>
__device__ __forceinline__ void wgmma_full(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 64 || N == 80 || N == 144 || N == 256, "wgmma_full: unsupported width");
    if constexpr (N == 64) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31},"
                     " %32, %33, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8), DCTTS_WG_D8(16), DCTTS_WG_D8(24) : "l"(da), "l"(db), "r"(accumulate));
    } else if constexpr (N == 80) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39},"
                     " %40, %41, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8), DCTTS_WG_D8(16), DCTTS_WG_D8(24), DCTTS_WG_D8(32) : "l"(da), "l"(db), "r"(accumulate));
    } else if constexpr (N == 144) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n144k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71},"
                     " %72, %73, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8), DCTTS_WG_D8(16), DCTTS_WG_D8(24), DCTTS_WG_D8(32), DCTTS_WG_D8(40), DCTTS_WG_D8(48), DCTTS_WG_D8(56), DCTTS_WG_D8(64) : "l"(da), "l"(db), "r"(accumulate));
    } else if constexpr (N == 256) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127},"
                     " %128, %129, p, 1, 1, 0, 0;\n\t}"
                     : DCTTS_WG_D8(0), DCTTS_WG_D8(8), DCTTS_WG_D8(16), DCTTS_WG_D8(24), DCTTS_WG_D8(32), DCTTS_WG_D8(40), DCTTS_WG_D8(48), DCTTS_WG_D8(56), DCTTS_WG_D8(64), DCTTS_WG_D8(72), DCTTS_WG_D8(80), DCTTS_WG_D8(88), DCTTS_WG_D8(96), DCTTS_WG_D8(104), DCTTS_WG_D8(112), DCTTS_WG_D8(120) : "l"(da), "l"(db), "r"(accumulate));
    }

}
#undef DCTTS_WG_D8

// hi*Bhi + hi*Blo + lo*Bhi into one accumulator of `cols` (16, 32, 48 or 64) columns, chosen at run time
template <int R>
__device__ __forceinline__ void wgmma_split3(float (&d)[R], int cols, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                             uint32_t accumulate) {
    if (cols >= 64) { wgmma_f16<4>(d, a_hi, b_hi, accumulate); wgmma_f16<4>(d, a_hi, b_lo, 1u); wgmma_f16<4>(d, a_lo, b_hi, 1u); }
    else if (cols == 48) { wgmma_f16<3>(d, a_hi, b_hi, accumulate); wgmma_f16<3>(d, a_hi, b_lo, 1u); wgmma_f16<3>(d, a_lo, b_hi, 1u); }
    else if (cols == 32) { wgmma_f16<2>(d, a_hi, b_hi, accumulate); wgmma_f16<2>(d, a_hi, b_lo, 1u); wgmma_f16<2>(d, a_lo, b_hi, 1u); }
    else { wgmma_f16<1>(d, a_hi, b_hi, accumulate); wgmma_f16<1>(d, a_hi, b_lo, 1u); wgmma_f16<1>(d, a_lo, b_hi, 1u); }
}

// K-major swizzled operand tile, rows of SW bytes (SW = 128 or 64), 8-row atoms of 8*SW bytes: the layout TMA writes with
// CU_TENSOR_MAP_SWIZZLE_{128B,64B}.  sm_90 descriptor: start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled K-major),
// SBO>>4 [32,46) = 8*SW, layout [62,64): SWIZZLE_128B = 1, SWIZZLE_64B = 2.  Tiles start on a swizzle-atom boundary; a
// k step of 16 halfs inside the atom adds 32 bytes to the start address.
template <int SW>
__device__ __forceinline__ uint64_t gmma_desc_kmajor(uint32_t smem_addr) {
    static_assert(SW == 128 || SW == 64, "swizzle span");
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= 1ull << 16;
    d |= static_cast<uint64_t>((8 * SW) >> 4) << 32;
    d |= static_cast<uint64_t>(SW == 128 ? 1 : 2) << 62;
    return d;
}
// no-swizzle K-major core-matrix layout: LBO = bytes between the two 8-wide k groups, SBO = bytes between 8-row groups
__device__ __forceinline__ uint64_t gmma_desc_noswz(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
    d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;
    return d;
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t smem_addr, uint32_t rank);
// arrive on the barrier at the same offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" :: "r"(mapa(smem_u32(bar), rank)) : "memory");
}
// the same with release semantics at CTA scope only: the caller's MMAs, whose reads it announces, have completed
// (wgmma.wait_group), and cluster scope would make every arrive wait for the thread's earlier global stores
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" :: "r"(mapa(smem_u32(bar), rank)) : "memory");
}
// named barrier of `n` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(n) : "memory"); }

// per-thread register budget of the executing warpgroup (all of its warps execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(N)); }

// ---- clusters / DSMEM ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t mapa(uint32_t smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ float4 ld_cluster_f4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_cluster_f4(uint32_t addr, float a, float b, float c, float d) {
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" :: "r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

}}  // namespace dctts::ptx
