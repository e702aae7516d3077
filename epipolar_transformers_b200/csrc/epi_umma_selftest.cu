// epi_umma_selftest.cu — one-CTA GEMM that exercises exactly the wgmma operand forms the fusion
// kernels use, so descriptor / swizzle / fragment-mapping mistakes show up as a plain matrix mismatch:
//   mode 0:  D[128 x N] = A[128 x K] · B[N x K]ᵀ          (A, B K-major panels)          -> S = F·Qᵀ
//   mode 1:  D[128 x N] = Atᵀ[128 x Kd] · B[N x Kd]ᵀ      (A MN-major: At is [Kd x 128])  -> Oᵀ = Fᵀ·βᵀ
// split=1 stages every operand as a bf16 (hi, lo) pair and issues hi·hi + hi·lo + lo·hi.
// One warpgroup computes the product in m64n32 blocks (two 64-row halves, N/32 column blocks), like the fusion kernels.
#include "../../include/epipolar_b200.h"
#include "epi_umma.cuh"

namespace epi {
using namespace umma;

__global__ void __launch_bounds__(128) umma_selftest_kernel(int mode, const float *__restrict__ A, const float *__restrict__ B,
                                                            float *__restrict__ D, int N, int K, int split) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x;
    // A region: (hi, lo) x panels.  mode 0: K/64 panels of 128 rows.  mode 1: 2 panels of K rows.
    const uint32_t a_rows = mode == 0 ? 128 : K, a_cols = mode == 0 ? K : 128;
    const uint32_t a_panel = a_rows * 128, a_bytes = a_panel * (a_cols / 64);
    const uint32_t b_panel = (uint32_t)N * 128, b_bytes = b_panel * (K / 64);
    uint8_t *a_hi = smem, *a_lo = smem + a_bytes, *b_hi = smem + 2 * a_bytes, *b_lo = b_hi + b_bytes;

    for (uint32_t idx = tid; idx < a_rows * a_cols; idx += blockDim.x) {
        uint32_t r = idx / a_cols, c = idx % a_cols;
        __nv_bfloat16 hi, lo;
        split_bf16(A[idx], hi, lo);
        uint32_t off = panel_offset(r, c, a_panel);
        *reinterpret_cast<__nv_bfloat16 *>(a_hi + off) = hi;
        *reinterpret_cast<__nv_bfloat16 *>(a_lo + off) = lo;
    }
    for (uint32_t idx = tid; idx < (uint32_t)N * K; idx += blockDim.x) {
        uint32_t r = idx / K, c = idx % K;
        __nv_bfloat16 hi, lo;
        split_bf16(B[idx], hi, lo);
        uint32_t off = panel_offset(r, c, b_panel);
        *reinterpret_cast<__nv_bfloat16 *>(b_hi + off) = hi;
        *reinterpret_cast<__nv_bfloat16 *>(b_lo + off) = lo;
    }
    fence_proxy_async_smem();
    __syncthreads();

    for (int nb = 0; nb * 32 < N; nb++)
        for (int mh = 0; mh < 2; mh++) {
            float acc[16];
#pragma unroll
            for (int e = 0; e < 16; e++) acc[e] = 0.f;
            wg_fence();
            for (int ks = 0; ks < K / 16; ks++) {
                for (int term = 0; term < (split ? 3 : 1); term++) {
                    const uint8_t *ap = term == 2 ? a_lo : a_hi;
                    const uint8_t *bp = term == 1 ? b_lo : b_hi;
                    const uint64_t bd = make_smem_desc(smem_u32(bp) + (ks / 4) * b_panel + (ks % 4) * 32 + nb * 4096, 16, 1024);
                    if (mode == 0) wgmma_m64n32<0>(acc, make_smem_desc(smem_u32(ap) + (ks / 4) * a_panel + (ks % 4) * 32 + mh * 8192, 16, 1024), bd);
                    else           wgmma_m64n32<1>(acc, make_smem_desc(smem_u32(ap) + mh * a_panel + ks * 2048, a_panel, 1024), bd);
                }
            }
            wg_commit();
            wg_wait_all();
#pragma unroll
            for (int e = 0; e < 16; e++) {
                const int col = nb * 32 + acc_col(tid, e);
                if (col < N) D[(size_t)(mh * 64 + acc_row(tid, e)) * N + col] = acc[e];
            }
        }
}

}  // namespace epi

extern "C" int epi_umma_selftest(int mode, const float *A, const float *B, float *D, int N, int K, int split, void *stream) {
    if (!A || !B || !D || N < 16 || N > 256 || N % 16 || K < 64 || K > 256 || K % 64 || (mode != 0 && mode != 1)) return EPI_EINVAL;
    const size_t a_bytes = 128 * (size_t)K * 2, b_bytes = (size_t)N * K * 2;
    const size_t smem = 2 * a_bytes + 2 * b_bytes + 1024 + 4096;      // + slack: an n32 block may read past N = 16 rows
    cudaError_t e = cudaFuncSetAttribute(epi::umma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return EPI_ECUDA;
    epi::umma_selftest_kernel<<<1, 128, smem, reinterpret_cast<cudaStream_t>(stream)>>>(mode, A, B, D, N, K, split);
    return cudaGetLastError() == cudaSuccess ? EPI_OK : EPI_ECUDA;
}
