// epi_zgemm.cu — z-projection epilogue on the tensor cores (TMA + warpgroup MMA).
//
//   y[n,o,p] = Σ_c Wf[o,c]·x[n,c,p] + bf[o]  (+ x[n,o,p] if ZRESIDUAL)  (+ feat_ref[q,o,p] for the caller's residual, read in
//   the map's own element type; q = pair_items(n, n_ref, n_views[, vs]).q, the pair's query item)
// restates  finalout = bn(z(out)) [+ out]   /root/reference/modeling/layers/epipolar.py:249-253 (eval-mode BN folded
// into Wf, bf by epi_fold_z_bn_f32) and  ret + feat   /root/reference/modeling/backbones/resnet.py:388.
//
// One CTA per 128 pixels and block of 128 output channels (blockIdx.y); small CTAs (69 KB, one K panel in flight) so that several
// are resident per SM and their load / MMA / store phases overlap each other:
// D[128 px, C out] = X[128 px, C]·Wfᵀ with X supplied by the fusion kernel as bf16
// (hi, lo) planes [N·HW, C] (K-major rows) and Wf split to (hi, lo) while it is staged.  Three MMAs per
// product (hi·hi + hi·lo + lo·hi), fp32 accumulation in registers (two warpgroups of M=64, N=128), K streamed in 64-channel
// panels — the X and W panels arrive by TMA (cp.async.bulk.tensor.2d with the 128-byte swizzle the wgmma descriptors expect,
// completion on an mbarrier); the epilogue adds bias/residuals and writes NCHW in y's type, fp32 or the fp32 result rounded once
// to bf16 / fp16 (a warp's lanes are 32 consecutive pixels, so every store instruction is one 128-byte line per channel, 64
// bytes for a 16-bit y).
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstring>

#include <type_traits>

#include "epi_kernels.cuh"
#include "epi_umma.cuh"

namespace epi {
using namespace umma;

namespace zg {
constexpr int NT = 256;
constexpr uint32_t A_PLANE = 16384;                 // 128 rows x 128 B
constexpr int NB = 128;                             // output channels per CTA (MMA N)
constexpr uint32_t B_PLANE = 16384;                 // 128 rows x 128 B
constexpr uint32_t STAGE = 2 * A_PLANE + 2 * B_PLANE;   // 64 KB: one K panel of (A hi, A lo, W hi, W lo)
constexpr int OT = 132;                             // epilogue tile pitch (floats)
constexpr uint32_t TILE_BYTES = NB * OT * 4;        // 67 584 B: the epilogue tile re-uses the stage
constexpr uint32_t BUF_BYTES = TILE_BYTES > STAGE ? TILE_BYTES : STAGE;
constexpr uint32_t SMEM_ALLOC = BUF_BYTES + 1024 + 128;     // ~69 KB: up to three CTAs per SM by shared memory (two by registers)

// 2-D tiled TMA load of a [128 rows x 64 bf16] box into a swizzled panel, completion counted on `bar`
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *tmap, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     umma::smem_u32(smem_dst)),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(umma::smem_u32(bar))
                 : "memory");
}
}  // namespace zg

// TABLE: vs is the call's source table; else an empty struct (one byte, no table code): the z GEMM's parameters hold tensor
// maps, which a trailing parameter pack cannot follow here
struct NoTable {};
__device__ __forceinline__ PairItems pair_items(int p, int n_ref, int n_views, NoTable) { return pair_items(p, n_ref, n_views); }

// four consecutive fp32 results rounded once to TO, one streaming store (16 bytes for fp32, 8 for bf16 / fp16); p is aligned
// to 4 elements
__device__ __forceinline__ void st4_cs(float *p, float4 v) { __stcs(reinterpret_cast<float4 *>(p), v); }
__device__ __forceinline__ void st4_cs(__nv_bfloat16 *p, float4 v) {
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    __stcs(reinterpret_cast<uint2 *>(p), make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b)));
}
__device__ __forceinline__ void st4_cs(__half *p, float4 v) {
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    __stcs(reinterpret_cast<uint2 *>(p), make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b)));
}

// TO: element type of y (the fp32 result rounded once)
template <bool TABLE, typename TO>
__global__ void __launch_bounds__(zg::NT, 2) epi_zgemm_kernel(const ZGemmArgs z, const __grid_constant__ CUtensorMap tm_hi,
                                                              const __grid_constant__ CUtensorMap tm_lo,
                                                              const __grid_constant__ CUtensorMap tw_hi,
                                                              const __grid_constant__ CUtensorMap tw_lo,
                                                              const std::conditional_t<TABLE, ViewSources, NoTable> vs) {
    using namespace zg;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + BUF_BYTES);        // K panel landed (TMA)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int C = z.C, HW = z.HW, W = z.W;
    const int tiles = (HW + 127) / 128;
    const int n = blockIdx.x / tiles, p0 = (blockIdx.x % tiles) * 128;
    const int nq = (C + 63) / 64;                      // K panels of 64 channels
    const int oc0 = (int)blockIdx.y * NB;             // this CTA's block of output channels
    const int CO = min(NB, C - oc0);

    pdl_launch_dependents();
    // The bias and the caller's residual (inputs of the whole forward, not products of the previous launches) are fetched into
    // registers FIRST: their latency is paid under the previous kernel's tail and this kernel's main loop instead of once per
    // output row of the epilogue (16 dependent round trips per warp).
    const bool addr = z.ref && z.add_ref;
    const bool vec = (z.y_stride[3] == 1) && (z.y_stride[2] == W) && (HW % 4 == 0) && (z.y_stride[1] % 4 == 0) && (z.y_stride[0] % 4 == 0) &&
                     ((reinterpret_cast<uintptr_t>(z.y) & (4 * sizeof(TO) - 1)) == 0) &&
                     (!addr || ((z.ref_stride[3] == 1) && (z.ref_stride[2] == W) && (z.ref_stride[1] % 4 == 0) && (z.ref_stride[0] % 4 == 0) &&
                                ((reinterpret_cast<uintptr_t>(z.ref) & (4 * feat_esize(z.ref_dtype) - 1)) == 0)));
    constexpr int ROWS = NB / (NT / 32);              // output rows per warp
    float4 res[ROWS];
    float bias[ROWS];
    {
        const int p = p0 + lane * 4;
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int ol = warp + k * (NT / 32);
            res[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            bias[k] = ol < CO ? __ldg(z.bf + oc0 + ol) : 0.f;      // folded bias: written long before the staging launch
            if (addr && vec && p + 3 < HW && ol < CO) {
                const int64_t i = (int64_t)pair_items(n, z.n_ref, z.n_views, vs).q * z.ref_stride[0] + (int64_t)(oc0 + ol) * z.ref_stride[1] + p;     // the caller's map, in its type
                res[k] = z.ref_dtype == kBF16 ? ld4_cs(static_cast<const __nv_bfloat16 *>(z.ref) + i)
                       : z.ref_dtype == kF16  ? ld4_cs(static_cast<const __half *>(z.ref) + i)
                                              : ld4_cs(static_cast<const float *>(z.ref) + i);
            }
        }
    }
    if (tid == 32) { mbar_init(bar, 1); mbar_fence_init(); }
    if (tid == 64) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tw_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tw_lo) : "memory");
    }
    __syncthreads();
    pdl_wait();                                        // the fused kernel's feature planes

    // Main loop: thread 0 issues the TMA loads of a K panel (A: 128 pixel rows x 64 channels of the (hi, lo) planes of x; B: NB output
    // rows x 64 input channels of the (hi, lo) planes of Wf); warpgroup wg multiplies pixel rows 64 wg .. +63, three MMAs per
    // 16-channel step, and waits for them before the panel is reloaded.  Output columns >= CO are computed and discarded.
    const int wg = warp >> 2, t128 = tid & 127;
    float acc[64];
#pragma unroll
    for (int e = 0; e < 64; e++) acc[e] = 0.f;
    {
        const uint32_t wrows = (uint32_t)(C < NB ? C : NB);            // W box rows (the tensor map's box)
        for (int q = 0; q < nq; q++) {
            if (tid == 0) {
                mbar_arrive_expect_tx(bar, 2 * A_PLANE + 2 * wrows * 128u);
                tma_load_2d(smem, &tm_hi, q * 64, n * HW + p0, bar);
                tma_load_2d(smem + A_PLANE, &tm_lo, q * 64, n * HW + p0, bar);
                tma_load_2d(smem + 2 * A_PLANE, &tw_hi, q * 64, oc0, bar);
                tma_load_2d(smem + 2 * A_PLANE + B_PLANE, &tw_lo, q * 64, oc0, bar);
            }
            for (uint32_t it = 0; !mbar_try_wait(bar, q & 1); ++it) if (it > (1u << 24)) __trap();
            const uint32_t sa = smem_u32(smem) + (uint32_t)wg * 8192u, sb = smem_u32(smem) + 2 * A_PLANE;
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ks++) {
                const uint64_t a_hi = make_smem_desc(sa + ks * 32, 16, 1024), a_lo = desc_add(a_hi, A_PLANE);
                const uint64_t b_hi = make_smem_desc(sb + ks * 32, 16, 1024), b_lo = desc_add(b_hi, B_PLANE);
                wgmma_m64n128<0>(acc, a_hi, b_hi);
                wgmma_m64n128<0>(acc, a_hi, b_lo);
                wgmma_m64n128<0>(acc, a_lo, b_hi);
            }
            wg_commit();
            wg_wait_all();
            __syncthreads();                           // both warpgroups are done with the panel
        }
    }

    // ---- epilogue ------------------------------------------------------------------------------------------------
    // phase 1 (accumulator fragments): registers -> shared tile [channel][128 pixels] (the operand stage is free now).
    //   The ZRESIDUAL needs no pass: the staged weight is Wf + I;
    // phase 2 (warp <-> channel row, lane <-> 4 consecutive pixels): + bias + caller residual, 512-byte row segments of the NCHW output
    //   per warp instruction.  Falls back to per-element addressing for strides that are not pixel-contiguous.
    float *otile = reinterpret_cast<float *>(smem);            // [NB][132] fp32 over the (now idle) stage
#pragma unroll
    for (int e = 0; e < 64; e++) {
        const int col = acc_col(t128, e);
        if (col < CO) otile[col * OT + wg * 64 + acc_row(t128, e)] = acc[e];
    }
    __syncthreads();
    {
        const int pp = lane * 4, p = p0 + pp;
#pragma unroll
        for (int k = 0; k < ROWS; k++) {
            const int ol = warp + k * (NT / 32);
            if (ol >= CO) break;
            const int o = oc0 + ol;
            const float4 t = *reinterpret_cast<const float4 *>(otile + ol * OT + pp);
            const float b = bias[k];
            float y[4] = {t.x + b, t.y + b, t.z + b, t.w + b};
            if (vec && p + 3 < HW) {
                st4_cs(static_cast<TO *>(z.y) + (int64_t)n * z.y_stride[0] + (int64_t)o * z.y_stride[1] + p,     // written once, read by
                       make_float4(y[0] + res[k].x, y[1] + res[k].y, y[2] + res[k].z, y[3] + res[k].w));       // nobody here: streaming
            } else {
                for (int e = 0; e < 4 && p + e < HW; e++) {
                    const int py = (p + e) / W, px = (p + e) % W;
                    float val = y[e];
                    if (addr) val += ld_feat(z.ref, (int64_t)pair_items(n, z.n_ref, z.n_views, vs).q * z.ref_stride[0] + (int64_t)o * z.ref_stride[1] + (int64_t)py * z.ref_stride[2] + (int64_t)px * z.ref_stride[3], z.ref_dtype);
                    static_cast<TO *>(z.y)[(int64_t)n * z.y_stride[0] + (int64_t)o * z.y_stride[1] + (int64_t)py * z.y_stride[2] + (int64_t)px * z.y_stride[3]] = from_f32<TO>(val);
                }
            }
        }
    }
}


bool zgemm_supported(int C) { return C % 64 == 0 && C >= 64 && C <= 512; }   // whole 64-channel TMA panels

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) p = nullptr;
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}
// [rows, cols = C] bf16 plane, box = 64 columns x box_rows rows, 128-byte swizzle (what the wgmma K-major descriptor reads)
bool make_plane_map(CUtensorMap *m, const __nv_bfloat16 *base, int rows, int C, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn || C % 8 != 0) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)C * 2};
    const cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1u, 1u};
    return fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16 *>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
}  // namespace

template <bool TABLE, typename TO>
static cudaError_t launch_zgemm_t(const ZGemmArgs &z, cudaStream_t st, const std::conditional_t<TABLE, ViewSources, NoTable> &vs) {
    const int tiles = (z.HW + 127) / 128;
    const auto kern = epi_zgemm_kernel<TABLE, TO>;
    static thread_local bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)zg::SMEM_ALLOC);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    // tensor maps are a pure function of (pointers, shape): keep the last set per host thread
    struct MapCache { const void *xh, *wh; int rows, C; CUtensorMap m[4]; };
    static thread_local MapCache mc = {nullptr, nullptr, 0, 0, {}};
    if (mc.xh != z.x_hi || mc.wh != z.w_hi || mc.rows != z.N * z.HW || mc.C != z.C) {
        const int wrows = z.C < zg::NB ? z.C : zg::NB;
        if (!make_plane_map(&mc.m[0], z.x_hi, z.N * z.HW, z.C, 128) || !make_plane_map(&mc.m[1], z.x_lo, z.N * z.HW, z.C, 128) ||
            !make_plane_map(&mc.m[2], z.w_hi, z.C, z.C, wrows) || !make_plane_map(&mc.m[3], z.w_lo, z.C, z.C, wrows))
            return cudaErrorInvalidValue;
        mc.xh = z.x_hi; mc.wh = z.w_hi; mc.rows = z.N * z.HW; mc.C = z.C;
    }
    return launch_pdl(kern, dim3((unsigned)(z.N * tiles), (unsigned)((z.C + zg::NB - 1) / zg::NB)), dim3(zg::NT), (size_t)zg::SMEM_ALLOC, st, z, mc.m[0], mc.m[1], mc.m[2], mc.m[3], vs);
}

template <typename TO>
static cudaError_t launch_zgemm_out(const ZGemmArgs &z, const ViewSources &vs, cudaStream_t st) {
    return vs.S ? launch_zgemm_t<true, TO>(z, st, vs) : launch_zgemm_t<false, TO>(z, st, NoTable{});
}

cudaError_t launch_zgemm(const ZGemmArgs &z, const ViewSources &vs, int y_dtype, cudaStream_t st) {
    return y_dtype == kBF16 ? launch_zgemm_out<__nv_bfloat16>(z, vs, st)
         : y_dtype == kF16  ? launch_zgemm_out<__half>(z, vs, st) : launch_zgemm_out<float>(z, vs, st);
}

}  // namespace epi
