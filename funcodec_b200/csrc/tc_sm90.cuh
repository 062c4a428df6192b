// sm_90a tensor-core primitives used by the implicit-GEMM conv and the RVQ distance kernels:
// mbarrier, wgmma (warpgroup MMA, fp16 / tf32 operands in shared memory, fp32 accumulators in registers), wgmma
// shared-memory descriptors, 1-D bulk async copies (cp.async.bulk, the TMA engine without a tensor map) and TMA tensor loads.
//
// Bit layouts follow the PTX ISA "matrix descriptor format" for warpgroup-level MMA (the fields CUTLASS exposes as
// cute::GMMA::DescriptorSM90).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fcb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ------------------------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
// arrival by the threads whose `pred` is set, as a predicated instruction (no branch: usable between wgmma of one warpgroup)
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\t.reg .b64 st;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(
                     smem_u32(bar)),
                 "r"((uint32_t)pred)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
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
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
// Same, with a back-off between polls: for waiters that are NOT on the critical path (a spinning warp still takes
// issue slots away from the producer warps of its SM sub-partition).
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, unsigned ns) {
    while (!mbar_try_wait(bar, parity)) { __nanosleep(ns); }
}

// Same, with cluster-scope acquire: for a barrier that the peer CTA of a cluster arrives on, so that the waiter's later writes
// into the peer's shared memory are ordered after the peer's reads that preceded its arrival.
__device__ __forceinline__ void mbar_wait_cluster_backoff(uint64_t* bar, uint32_t parity, unsigned ns) {
    for (;;) {
        uint32_t ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (ok) return;
        __nanosleep(ns);
    }
}

// generic-proxy writes (st.shared by threads) -> visible to the async proxy (wgmma / bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// CTAs in this CTA's cluster (1 for a launch without clusters)
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
    return r;
}
// arrival on an mbarrier of another CTA of the cluster (`remote_bar`: from mapa_shared), by the threads whose `pred` is set, as a
// predicated instruction (usable between wgmma of one warpgroup)
__device__ __forceinline__ void mbar_arrive_remote_if(uint32_t remote_bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];\n\t}" ::"r"(
                     remote_bar),
                 "r"((uint32_t)pred)
                 : "memory");
}
// this CTA's shared memory -> the same-sized region of another CTA of the cluster (`dst_remote`, `bar_remote`: from mapa_shared),
// completion signalled on that CTA's mbarrier (complete_tx::bytes).  16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_s2peer(uint32_t dst_remote, const void* src_smem, uint32_t bytes, uint32_t bar_remote) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_remote),
                 "r"(smem_u32(src_smem)), "r"(bytes), "r"(bar_remote)
                 : "memory");
}
// barrier over every thread of every CTA of the cluster (not .aligned: the roles reach it from divergent code)
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

// ------------------------------------------------------------------------------------------------ bulk copy (TMA engine, 1-D)
// global -> shared, completion signalled on an mbarrier (complete_tx::bytes).  16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// TMA tensor load (cp.async.bulk.tensor, SASS UTMALDG): a 4-D box of the tensor described by `tmap` (a CUtensorMap passed as a
// __grid_constant__ kernel parameter) -> dense shared-memory tile, completion on an mbarrier (complete_tx::bytes).
// Out-of-bounds coordinates are zero-filled by the hardware.
__device__ __forceinline__ void tma_load_4d(void* dst_smem, const void* tmap, int c0, int c1, int c2, int c3, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(dst_smem)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

__device__ __forceinline__ void tma_load_5d(void* dst_smem, const void* tmap, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
            smem_u32(dst_smem)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

// ------------------------------------------------------------------------------------------------ register budgets
// Executed by all 128 threads of a warpgroup: lower / raise its per-thread register count to R (multiple of 8, 24..256).  The
// raise waits until the CTA's pool (the launch allocation) has the registers that other warpgroups released.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ------------------------------------------------------------------------------------------------ wgmma
// Every wgmma below is issued by all 128 threads of a warpgroup; accumulator fragment of m64nN (per warp w of the group, lane l):
// d[4j + 0..1] = row 16w + l/4, columns 8j + 2(l%4) + 0..1;  d[4j + 2..3] = row 16w + l/4 + 8, same columns.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma_wait
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 16] (+)= A[64 x 16] * B[16 x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers.
__device__ __forceinline__ void wgmma_m64n16k16_f16(float (&d)[8], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 32] (+)= A[64 x 16] * B[32 x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers.
__device__ __forceinline__ void wgmma_m64n32k16_f16(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers.
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers.
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, tf32 operands from shared memory, fp32 accumulator in registers.
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

template <int N> struct WgmmaF16;
template <> struct WgmmaF16<16> { static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n16k16_f16(d, a, b, acc); } };
template <> struct WgmmaF16<32> { static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n32k16_f16(d, a, b, acc); } };
template <> struct WgmmaF16<64> { static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n64k16_f16(d, a, b, acc); } };
template <> struct WgmmaF16<128> { static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128k16_f16(d, a, b, acc); } };

// ------------------------------------------------------------------------------------------------ descriptors
// K-major operand tile in the canonical SWIZZLE_128B layout: rows of 128 bytes (64 fp16 / 32 tf32), 8-row groups
// 1024 bytes apart (SBO), 16-byte chunk index XOR (row & 7).  `addr` = shared address of row 0 (+ 32 bytes per K step of
// 16 fp16 / 8 tf32 inside the 128-byte row).  The row-0 address may be any multiple of 128 bytes inside a slab whose base
// is 1024-byte aligned and that was written with chunk ^= (absolute_row & 7): tap-shifted views.  The swizzle XOR is taken
// from the absolute shared-memory address bits [7,10), so such a view needs base offset 0.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t addr) {
    uint64_t d = 0;
    d |= (uint64_t)((addr & 0x3FFFFu) >> 4);            // [0,14)  start address >> 4
    d |= (uint64_t)1 << 16;                              // [16,30) leading byte offset (unused for swizzled K-major) = 1
    d |= (uint64_t)(1024 >> 4) << 32;                    // [32,46) stride byte offset = 1024 B between 8-row groups
    d |= (uint64_t)1 << 62;                              // [62,64) layout type: SWIZZLE_128B
    return d;
}
// byte offset of element (row, col) (col in tf32 elements, < 32) inside a SWIZZLE_128B K-major slab whose row 0
// sits at a 1024-byte aligned address
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t col) {
    return row * 128u + ((((col >> 2) ^ (row & 7u)) << 4) | ((col & 3u) << 2));
}

// FP16 split of two (pre-scaled) fp32 values: hi = fp16(x) round-to-nearest, lo = fp16(x - hi) (x - hi is exact in fp32);
// element 0 in the low half.  Saturating conversions: |x| beyond the fp16 range clamps instead of producing inf.
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    float f0, f1;
    asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}" : "=f"(f0), "=f"(f1) : "r"(hi));
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - f1), "f"(x0 - f0));
}
__device__ __forceinline__ float exp2f_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// 3xTF32 split: hi = x with the low 13 mantissa bits cleared after round-to-nearest on the tf32 grid,
// lo = x - hi (exact in fp32); the tensor core ignores lo's bits below tf32 precision.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    uint32_t u = __float_as_uint(x);
    u = (u + 0x1000u) & 0xFFFFE000u;       // round half up in magnitude on the 10-bit-mantissa grid
    hi = __uint_as_float(u);
    lo = x - hi;
}

}  // namespace tc
}  // namespace fcb
