// wg.cuh -- minimal hand-written Hopper warpgroup MMA (wgmma) / mbarrier primitives for sm_90a (inline PTX).
//
// Operand tiles live in shared memory in the no-swizzle ("interleave") canonical layout of the wgmma
// shared-memory descriptor: 8x8 fp16 core matrices of 128 contiguous bytes (8 rows x 16 B).
// All tiles in this library are stored CHUNK-MAJOR:
//      byte(r, c) = (c / 8) * chunk_bytes + (r / 8) * 128 + (r % 8) * 16 + (c % 8) * 2,
//      chunk_bytes = rows / 8 * 128
// so the same physical tile can be fed to the tensor core either
//   * K-major   (rows = M/N index, cols = K):  SBO = 128, LBO = chunk_bytes, or
//   * MN-major  (cols = M/N index, rows = K):  SBO = chunk_bytes, LBO = 128
// (interleave-mode strides of the canonical layouts in the PTX ISA, "Matrix Descriptor Format" of wgmma).
// That is what lets one activation tile serve forward/dgrad (K-major) and wgrad (MN-major), and
// one weight tile serve forward (K-major B) and dgrad (MN-major B), without any transposition.
//
// A wgmma of shape m64nNk16 is issued by all 128 threads of a warpgroup; its fp32 accumulator lives
// in registers, N/2 per thread.  Thread (warp w of the warpgroup, lane l) holds, for i = 0 .. N/2-1,
//      row = 16 w + l / 4 + 8 * ((i >> 1) & 1),   col = 8 * (i >> 2) + 2 * (l % 4) + (i & 1).
// A 128-row tile is two such m64 halves (rows 0..63, 64..127), each with its own accumulator.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// byte offset of element (r, c) in a chunk-major tile with `rows` rows (fp16)
__host__ __device__ __forceinline__ uint32_t tile_off(uint32_t r, uint32_t c, uint32_t rows) {
    return (c >> 3) * (rows << 4) + (r >> 3) * 128u + (r & 7u) * 16u + (c & 7u) * 2u;
}

// ---- descriptors --------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;                              // base_offset 0, layout type 0 (interleave, no swizzle)
}

// A tile: `rows` rows (chunk-major).  K-major operand: M/N = rows, K = cols.  MN-major operand: M/N = cols, K = rows.
struct Operand {
    uint32_t saddr;      // shared address of the tile element (0, first column used)
    uint32_t rows;       // rows of the physical tile (defines chunk_bytes)
    bool mn_major;
    __device__ __forceinline__ uint64_t desc(uint32_t k0) const {
        const uint32_t chunk = rows << 4;
        if (!mn_major)   // K along columns: 16 k = 2 chunks
            return smem_desc(saddr + (k0 >> 3) * chunk, /*lbo=*/chunk, /*sbo=*/128u);
        // K along rows: 16 k = 2 groups of 8 rows = 256 B
        return smem_desc(saddr + (k0 >> 3) * 128u, /*lbo=*/128u, /*sbo=*/chunk);
    }
    // the same operand moved by `mn` rows (K-major) or columns (MN-major) of the M/N index
    __device__ __forceinline__ Operand shifted(uint32_t mn) const {
        return Operand{saddr + (mn_major ? (mn >> 3) * (rows << 4) : (mn >> 3) * 128u), rows, mn_major};
    }
};

// ---- ordering -----------------------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (tensor core operand fetch, bulk copies)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int NR>
__device__ __forceinline__ void fence_regs(float (&d)[NR]) {
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

// ---- MMA ----------------------------------------------------------------------------------------
// D[64 x N] (+)= A[64 x 16] * B[16 x N] (fp16 operands from shared memory, fp32 accumulator in registers); executed by all
// 128 threads of the warpgroup between wgmma_fence() and commit() / wait().  TA / TB: operand A / B is MN-major.
template <int N, int TA, int TB> struct Mma;
template <int TA, int TB> struct Mma<16, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[8], uint64_t a, uint64_t b, bool acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a), "l"(b), "r"(acc ? 1u : 0u), "n"(TA), "n"(TB) : "memory");
    }
};
template <int TA, int TB> struct Mma<32, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[16], uint64_t a, uint64_t b, bool acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(acc ? 1u : 0u), "n"(TA), "n"(TB) : "memory");
    }
};
template <int TA, int TB> struct Mma<48, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[24], uint64_t a, uint64_t b, bool acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, %28;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(a), "l"(b), "r"(acc ? 1u : 0u), "n"(TA), "n"(TB) : "memory");
    }
};
template <int TA, int TB> struct Mma<64, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[32], uint64_t a, uint64_t b, bool acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(acc ? 1u : 0u), "n"(TA), "n"(TB) : "memory");
    }
};

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int NH, int NR>
__device__ __forceinline__ void fence_regs(float (&d)[NH][NR]) {
#pragma unroll
    for (int h = 0; h < NH; ++h) fence_regs(d[h]);
}
// wait for every committed wgmma; the accumulators named here are read only after it
template <typename... Acc>
__device__ __forceinline__ void wait(Acc&... acc) {
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    (fence_regs(acc), ...);
}

// D[64 x N] (+)= A[64 x K] * B[K x N] over KSTEPS k-steps of 16 (issue only: the caller fences, commits and waits)
template <int N, int KSTEPS, bool A_MN, bool B_MN>
__device__ __forceinline__ void gemm64(float (&d)[N / 2], const Operand& a, const Operand& b, bool accumulate_first) {
#pragma unroll
    for (int s = 0; s < KSTEPS; ++s)
        Mma<N, A_MN ? 1 : 0, B_MN ? 1 : 0>::run(d, a.desc(16 * s), b.desc(16 * s), accumulate_first || s > 0);
}
// the 128-row form: rows 0..63 into d[0], rows 64..127 into d[1]
template <int N, int KSTEPS, bool A_MN, bool B_MN>
__device__ __forceinline__ void gemm128(float (&d)[2][N / 2], const Operand& a, const Operand& b, bool accumulate_first) {
    gemm64<N, KSTEPS, A_MN, B_MN>(d[0], a, b, accumulate_first);
    gemm64<N, KSTEPS, A_MN, B_MN>(d[1], a.shifted(64), b, accumulate_first);
}

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug traps (launch error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > 4000000u) __trap();
    }
}

}  // namespace wg
