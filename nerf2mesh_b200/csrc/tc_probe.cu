// tc_probe.cu -- self-test of the wgmma primitives in wg.cuh: one 128 x N x K GEMM with the
// operands in K-major or MN-major form, used by tests/test_gpu_tc05.py to pin the descriptor
// conventions against torch.matmul before the MLP kernels rely on them.
#include "n2m_common.cuh"
#include "wg.cuh"

namespace n2m {
namespace {

// A_phys: [ra x ca] row-major fp16 in global, B_phys: [rb x cb]; D: [128 x N] fp32 row-major.
//   a_mn == 0: A_phys is [128(M) x K]         a_mn == 1: A_phys is [K x 128(M)]
//   b_mn == 0: B_phys is [N x K]              b_mn == 1: B_phys is [K x N]
template <int N, bool A_MN, bool B_MN>
__device__ __forceinline__ void probe_gemm(const wg::Operand& oa, const wg::Operand& ob, uint32_t K, float* __restrict__ D) {
    float d[2][N / 2];
    wg::wgmma_fence();
    for (uint32_t k = 0; k < K; k += 16) {
        wg::Mma<N, A_MN, B_MN>::run(d[0], oa.desc(k), ob.desc(k), k > 0);
        wg::Mma<N, A_MN, B_MN>::run(d[1], oa.shifted(64).desc(k), ob.desc(k), k > 0);
    }
    wg::commit(); wg::wait(d);
    const uint32_t tid = threadIdx.x;
    for (int h = 0; h < 2; ++h)
        for (int i = 0; i < N / 2; ++i) {
            const uint32_t row = 64u * h + 16u * (tid >> 5) + ((tid & 31u) >> 2) + 8u * ((i >> 1) & 1u);
            const uint32_t col = 8u * (i >> 2) + 2u * (tid & 3u) + (i & 1u);
            D[row * N + col] = d[h][i];
        }
}

template <int N>
__device__ __forceinline__ void probe_majors(const wg::Operand& oa, const wg::Operand& ob, uint32_t K, float* __restrict__ D) {
    if (!oa.mn_major && !ob.mn_major) probe_gemm<N, false, false>(oa, ob, K, D);
    else if (!oa.mn_major) probe_gemm<N, false, true>(oa, ob, K, D);
    else if (!ob.mn_major) probe_gemm<N, true, false>(oa, ob, K, D);
    else probe_gemm<N, true, true>(oa, ob, K, D);
}

__global__ void __launch_bounds__(128)
k_tc_probe(const __half* __restrict__ A, const __half* __restrict__ B, float* __restrict__ D,
           uint32_t N, uint32_t K, int a_mn, int b_mn) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t ra = a_mn ? K : 128u, ca = a_mn ? 128u : K;
    const uint32_t rb = b_mn ? K : N, cb = b_mn ? N : K;
    uint8_t* sa = smem;
    uint8_t* sb = smem + ra * ca * 2;
    const uint32_t tid = threadIdx.x;
    for (uint32_t i = tid; i < ra * ca; i += 128) {
        const uint32_t r = i / ca, c = i % ca;
        *reinterpret_cast<__half*>(sa + wg::tile_off(r, c, ra)) = A[i];
    }
    for (uint32_t i = tid; i < rb * cb; i += 128) {
        const uint32_t r = i / cb, c = i % cb;
        *reinterpret_cast<__half*>(sb + wg::tile_off(r, c, rb)) = B[i];
    }
    wg::fence_async_smem();
    __syncthreads();
    const wg::Operand oa{wg::smem_u32(sa), ra, a_mn != 0};
    const wg::Operand ob{wg::smem_u32(sb), rb, b_mn != 0};
    switch (N) {
        case 16: probe_majors<16>(oa, ob, K, D); break;
        case 32: probe_majors<32>(oa, ob, K, D); break;
        case 48: probe_majors<48>(oa, ob, K, D); break;
        case 64: probe_majors<64>(oa, ob, K, D); break;
    }
}

}  // namespace
}  // namespace n2m

using namespace n2m;

extern "C" int n2m_tc_probe(const void* A, const void* B, float* D, uint32_t N, uint32_t K, int a_mn, int b_mn,
                            n2m_stream_t stream) {
    N2M_REQUIRE(A && B && D, "tc_probe", "null pointer");
    N2M_REQUIRE(N % 16 == 0 && N >= 16 && N <= 64 && K % 16 == 0 && K >= 16 && K <= 128, "tc_probe", "bad N/K");
    const size_t smem = (size_t)128 * K * 2 + (size_t)N * K * 2;
    cudaFuncSetAttribute(k_tc_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_tc_probe<<<1, 128, smem, as_stream(stream)>>>(static_cast<const __half*>(A), static_cast<const __half*>(B), D, N, K, a_mn, b_mn);
    return check_launch("tc_probe");
}
