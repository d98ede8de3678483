// Inline-PTX wrappers for sm_90a: mbarrier, wgmma (warpgroup MMA), bulk async copies.
// Hand-written; field layouts follow the PTX ISA "wgmma" chapter (matrix descriptor format).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>

namespace mdk {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make mbarrier.init visible to the async proxy (bulk copies)
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
// plain arrive (release at CTA scope)
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (an error code on the host),
// never as a hung GPU.  ~4e9 SM cycles is > 2 s, far beyond any legitimate wait here.  No printf: a function call
// inside a loop that issues wgmma makes ptxas serialise the MMAs (warning C7510).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}

// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- thread-block clusters (distributed shared memory)
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// shared::cta address of this CTA -> shared::cluster address of the same variable in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_u32(uint32_t cluster_addr, uint32_t v) {
    asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(cluster_addr), "r"(v) : "memory");
}
// generic-proxy writes to shared memory anywhere in the cluster (st.shared::cluster) -> visible to the async proxy of
// the CTA that owns the memory, once a release / acquire at cluster scope orders them before its wgmma
__device__ __forceinline__ void fence_proxy_async_cluster() {
    asm volatile("fence.proxy.async.shared::cluster;" ::: "memory");
}
// arrive on an mbarrier of another CTA of the cluster (address from mapa_shared); release at cluster scope: the
// arriving thread's prior writes, and those ordered before it by a CTA barrier, are visible to an acquiring waiter
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_cluster(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded like mbar_wait; acquire at cluster scope pairs with mbar_arrive_cluster
__device__ __forceinline__ void mbar_wait_cluster(uint64_t *bar, uint32_t parity) {
    if (mbar_try_wait_cluster(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait_cluster(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}
// whole-cluster barrier (all threads of every CTA), release / acquire at cluster scope.  Used once, after the mbarrier
// initialisation: the CTAs of a cluster are co-scheduled, so it cannot wait on a CTA that has not started.
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// named barrier over `count` threads (a warpgroup: 128)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// L2 prefetch of a contiguous range (16-B aligned, size % 16 == 0); no destination, no completion tracking
__device__ __forceinline__ void bulk_prefetch_l2(const void *gmem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// ---------------------------------------------------------------- bulk async copy (TMA engine, 1-D)
// global -> shared, completion counted in bytes on an mbarrier.  16-B aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// L2 policy for data written once and not read again soon (the bulk-store counterpart of st.global.cs)
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// shared -> global, completion tracked per issuing thread in bulk groups (bulk_commit / bulk_wait_*).  16-B aligned,
// size % 16 == 0.  The source must be made visible to the async proxy first (fence_proxy_async_smem).
__device__ __forceinline__ void bulk_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes, uint64_t policy) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(gmem_dst),
                 "r"(smem_u32(smem_src)), "r"(bytes), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's bulk stores have finished reading their shared-memory source (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// this thread's bulk stores are complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- wgmma (warpgroup MMA, sm_90a)
// Shared-memory matrix descriptor, K-major operand, no swizzle ("interleaved" core matrices):
//   core matrix = 8 rows x 16 bytes, stored as 128 contiguous bytes (row r at +16*r);
//   LBO = byte distance between core matrices adjacent along K,
//   SBO = byte distance between core matrices adjacent along M/N (next 8 rows).
// bits [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4, [49,52) base offset 0, [62,64) layout type 0.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
// ordering of register / shared-memory writes before the warpgroup's next wgmma (whole warpgroup)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// every group but the most recently committed one is complete (for the executing warp)
__device__ __forceinline__ void wg_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// keeps the compiler from touching an accumulator between the asynchronous MMA and wg_wait_all
template <int R>
__device__ __forceinline__ void wg_hold(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, fp16 in, fp32 accumulate; issued by all 128 threads of a warpgroup.
// Accumulator fragment: warp w of the warpgroup, lane l holds rows 16w + l/4 (+8) and columns 8i + 2(l%4) (+1):
// d[4i] = (row, col), d[4i+1] = (row, col+1), d[4i+2] = (row+8, col), d[4i+3] = (row+8, col+1).
// SS: A from shared memory (descriptor).  RS: A from registers, the mma.m16n8k16 A fragment of the warp's 16 rows:
// a[0] = (row, k 2(l%4) +0/1), a[1] = (row+8, same k), a[2] = (row, k+8), a[3] = (row+8, k+8).
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
    __device__ __forceinline__ static void ss(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a), "l"(b), "r"(accumulate));
    }
    __device__ __forceinline__ static void rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
    }
    // the same SS MMA into columns 0-15 of an m64n32 accumulator: its d[0..7] (the fragment layout above is that of n16)
    __device__ __forceinline__ static void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<32> {
    __device__ __forceinline__ static void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(accumulate));
    }
    __device__ __forceinline__ static void rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<128> {
    __device__ __forceinline__ static void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b), "r"(accumulate));
    }
    __device__ __forceinline__ static void rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
    }
};

// ---------------------------------------------------------------- stmatrix (sm_90)
// Four 8x8 b16 matrices, each held in the mma fragment layout (lane l: row l/4, columns 2(l%4) and +1 in the low and
// high half of its register r[m]), stored TRANSPOSED: the 16 bytes at the address from lane 8m + c (16-B aligned)
// receive column c of matrix m, rows 0..7 in order.
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t smem_addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(smem_addr), "r"(r0),
                 "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}

// ---------------------------------------------------------------- fp16 hi/lo split
// v ~= hi + lo with hi = fp16(v), lo = fp16(v - hi): ~22 significant bits for |v| in [2^-14, 65504],
// absolute error <= 2^-25 below that (fp16 subnormals).  Three fp16 MMAs (hi*hi + hi*lo + lo*hi) with
// fp32 accumulation then reproduce an fp32 product to ~1e-7 relative.  The host weight packers use the same split.
__host__ __device__ __forceinline__ void split_f16(float v, __half &hi, __half &lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}
// the same split of two values, packed as f16x2 (v0 in the low half): bit for bit what split_f16 gives for each
__device__ __forceinline__ void split_f16x2(float v0, float v1, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(v0, v1);
    const __half2 l = __floats2half2_rn(v0 - __low2float(h), v1 - __high2float(h));
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}
// split_f16x2's hi with lo rounded toward zero: |lo| < half an fp16 unit of hi unless v lies exactly halfway, where
// round-to-nearest-even picks hi again, so fp16(hi + lo) == hi for every v.  The fp16 mode's h0 tiles: the products read
// hi only, and h0 read back as hi + lo (~22 bits) rounds to the very hi they used.
__device__ __forceinline__ void split_f16x2_rz(float v0, float v1, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(v0, v1);
    const __half2 l = __halves2half2(__float2half_rz(v0 - __low2float(h)), __float2half_rz(v1 - __high2float(h)));
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}

// ---------------------------------------------------------------- streaming global access
__device__ __forceinline__ float ldg_stream(const float *p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

__device__ __forceinline__ float4 ld_stream4(const float *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}

}  // namespace mdk
