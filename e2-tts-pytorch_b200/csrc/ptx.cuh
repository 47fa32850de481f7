// Raw sm_90a PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA), fences.
// No CUTLASS/CuTe — everything here is inline PTX assembled by nvcc for compute_90a.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

#ifndef B200_SPIN_LIMIT
#define B200_SPIN_LIMIT (1u << 28)  // bounded mbarrier spins: a protocol bug traps instead of hanging the box
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// try_wait with a suspend-time hint: the warp is parked by the hardware until the phase completes (or the hint, in ns, expires)
// instead of re-issuing the test, so waiting warps do not take issue slots from the working ones.
#ifndef B200_WAIT_HINT_NS
#define B200_WAIT_HINT_NS 0x989680u
#endif
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
#ifdef B200_WAIT_NO_HINT   // developer A/B: the plain form (hardware default suspend time)
    asm volatile(
        "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
#else
    asm volatile(
        "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(B200_WAIT_HINT_NS)
        : "memory");
#endif
    return ok != 0;
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// Bounded wait: a protocol bug traps after B200_WAIT_TIMEOUT_NS instead of hanging the box (each failed try_wait may already
// have been parked for up to the suspend hint, so the bound is on wall time, not on the iteration count).
#ifndef B200_WAIT_TIMEOUT_NS
#define B200_WAIT_TIMEOUT_NS 4000000000ull
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const unsigned long long t0 = global_ns();
    while (!mbar_try_wait(bar, parity)) {
        if (global_ns() - t0 > B200_WAIT_TIMEOUT_NS) __trap();
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
// 2-D tiled load, coordinates (c0 = innermost element index, c1 = row index); completes `bytes` on `bar`.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// TMA tile STORE (shared -> global, bulk async group): rows / columns of the box that fall outside the tensor are clipped by the hardware.
// The issuing thread must have ordered the generic-proxy smem writes of the whole warp before it (fence.proxy.async by every writer,
// then a warp barrier); the staging buffer may be rewritten once cp.async.bulk.wait_group.read has returned.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(m), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
// TMA tile REDUCTION (shared -> global, element-wise add into the tensor, bulk async group), 3-D coordinates; the same ordering rules
// as tma_store_2d, and the same hardware clipping of the box at the tensor's bounds.
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(m), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// named barriers (ids 1..15; __syncthreads owns id 0): bar.sync waits until `n` threads of the CTA have reached barrier `id`
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// counts the calling threads towards barrier `id` without waiting: the producer side of a producer / consumer hand-off
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// 1-D bulk copy global -> shared (TMA engine, no tensor map): `bytes` a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// A warpgroup (4 consecutive warps, first warp index a multiple of 4) issues the MMAs together; the accumulators live in the
// registers of its 128 threads. wgmma_fence() orders earlier register / shared-memory writes of the operands before the next MMA,
// wgmma_commit() closes a group of MMAs, wgmma_wait<N>() returns when at most N groups are still in flight.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of an accumulator array across the asynchronous MMAs that own it.
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Register budget of a warp-specialised CTA: the TMA warpgroup gives registers back, the MMA warpgroups take them.
template <int N>
__device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- generated wgmma wrappers: D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 inputs, fp32 accumulators in registers
// TA / TB: 0 = K-major, 1 = MN-major operand in shared memory (the transpose immediates of wgmma).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TB>
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate), "n"(TB));
}


// ---------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor of wgmma for 128B-swizzled tiles: start addr>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// base_offset [49,52) = 0 (tiles are 1024-byte aligned), layout type [62,64) = 1 (SWIZZLE_128B).
// K-major: 8-row groups SBO = 1024 B apart, one swizzle atom (64 bf16) along K, LBO unused. MN-major: 64-element MN atoms LBO apart,
// 8-k-row groups SBO = 1024 B apart.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// Paired fp32 arithmetic: two independent round-to-nearest operations (the kernels keep their math in fp32x2 pairs).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// Coalesced fp32 accumulation of a row-per-lane 32 x 32 block: lane l holds v[0..31] = 32 consecutive columns of row (row0 + l).
// The block is transposed through a padded smem tile so that every RED instruction adds 32 CONSECUTIVE floats of one row
// (one 128-byte L2 transaction instead of 32 scattered 4-byte ones).  stg: 32 x 33 floats, private to the warp.
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// stg: 32 x 32 fp32 staging tile (4 KB), 16-byte groups XOR-swizzled by the row so that both the row-per-lane writes and the
// 8-lanes-per-row reads are bank-conflict free without padding (the 4 KB tile doubles as the TMA-store staging buffer of the bf16 path)
__device__ __forceinline__ void warp_red_rows_f32(float* stg, const float (&v)[32], float* base, long long ld, int row0, int nrows_total,
                                                  int ncols_valid, int lane) {
    __syncwarp();
#pragma unroll
    for (int g = 0; g < 8; ++g)
        *reinterpret_cast<float4*>(stg + lane * 32 + ((g ^ (lane & 7)) << 2)) = make_float4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]);
    __syncwarp();
    if (((ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(base) & 15) == 0)) {
        // 16-byte vector reductions (REDG.F32x4): 8 lanes cover the 128 bytes of a row, 4 rows per instruction
        const int g = lane & 7, cg = g * 4, rsub = lane >> 3;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int r = it * 4 + rsub;
            if (row0 + r < nrows_total) {
                const float4 s4 = *reinterpret_cast<const float4*>(stg + r * 32 + ((g ^ (r & 7)) << 2));
                float* dst = base + (long long)(row0 + r) * ld + cg;
                if (cg + 4 <= ncols_valid) red_add_v4(dst, s4.x, s4.y, s4.z, s4.w);
                else {
                    const float sp[4] = {s4.x, s4.y, s4.z, s4.w};
                    for (int j = 0; j < 4; ++j)
                        if (cg + j < ncols_valid) atomicAdd(dst + j, sp[j]);
                }
            }
        }
    } else if (lane < ncols_valid) {
#pragma unroll 4
        for (int r = 0; r < 32; ++r)
            if (row0 + r < nrows_total) atomicAdd(base + (long long)(row0 + r) * ld + lane, stg[r * 32 + ((((lane >> 2) ^ (r & 7)) << 2) | (lane & 3))]);
    }
    __syncwarp();
}

// ---------------------------------------------------------------- misc
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

// counter-based RNG for dropout masks (recomputed in backward from the same (seed, index))
__device__ __forceinline__ uint32_t hash_u32(uint64_t seed, uint64_t idx) {
    uint64_t z = seed + idx * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return (uint32_t)((z ^ (z >> 31)) >> 32);
}
__device__ __forceinline__ bool dropout_keep(uint64_t seed, uint64_t idx, float p) {
    return (hash_u32(seed, idx) >> 8) * (1.0f / 16777216.0f) >= p;
}

// Dropout masks: counter-based, recomputed by the backward kernels from the same (seed, index). One mixing step decides TWO
// neighbouring elements: x = pair * golden + seed; x ^= x >> 15; then the HIGH bits of two different odd multiples of x are compared
// against the threshold as full 32-bit words — keep iff word >= thresh16 << 16, i.e. P(drop) = thresh16 / 65536. idx = row_id *
// stride + column with an even stride, so (idx >> 1) pairs columns (2k, 2k+1) of one row; only the low 32 bits of the pair index
// are hashed (the pattern repeats after 2^33 elements).
// Cost per pair: 3 IMAD (FMA pipe) + SHF + LOP3 + 2 ISETP (+ the two selects): the round-1 hash (two xorshift-multiply rounds, then
// 16-bit field extraction) put 10 instructions per pair on the half-rate ALU pipe, which the softmax threads of the attention kernels
// are bound by.
struct DropWords { uint32_t a, b; };
__device__ __forceinline__ DropWords drop_words(uint32_t seedmix, uint32_t pair) {
    uint32_t x = pair * 0x9E3779B1u + seedmix;
    x ^= x >> 15;
    DropWords w;
    w.a = x * 0x85EBCA6Bu;
    w.b = x * 0xC2B2AE35u;
    return w;
}
__device__ __forceinline__ uint32_t drop_thresh32(uint32_t thresh16) { return thresh16 << 16; }
// The 16-bit threshold of drop probability p, and the scale of the kept elements, 1 / P(keep) = 65536 / (65536 - thresh16).
__host__ __device__ __forceinline__ uint32_t drop_thresh16(float p) { return (uint32_t)(p * 65536.f); }
__host__ __device__ __forceinline__ float drop_keep_scale(uint32_t thresh16) { return 65536.f / (65536.f - (float)thresh16); }
// The 32-bit seed word drop_words hashes with: seed plus the optional device addend (CUDA-graph replays), folded to 32 bits.
__device__ __forceinline__ uint32_t drop_seed_word(uint64_t seed, const unsigned long long* seed_dev) {
    const uint64_t s = seed + (seed_dev ? __ldg(seed_dev) : 0ull);
    return (uint32_t)s ^ ((uint32_t)(s >> 32) * 0x85EBCA77u);
}
// Pair index of GLU hidden units (hcol, hcol + 1) of `row` in an [rows, inner] hidden tensor: the forward GEMM's GLU epilogue and
// the GLU backward must agree on it. inner is even, so hidden units (2k, 2k+1) of one row share a pair.
__device__ __forceinline__ uint32_t glu_drop_pair(long long row, int inner, int hcol) {
    return (uint32_t)(((unsigned long long)row * (unsigned long long)inner + hcol) >> 1);
}

}  // namespace b200
