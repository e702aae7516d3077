// epi_zgemm.cu — z-projection epilogue on the tensor cores (TMA + warpgroup MMA).
//
//   y[n,o,p] = Σ_c Wf[o,c]·x[n,c,p] + bf[o]  (+ x[n,o,p] if ZRESIDUAL)  (+ feat_ref[q,o,p] for the caller's residual, read in
//   the map's own element type; q = pair_items(n, n_ref, n_views[, vs]).q, the pair's query item)
// restates  finalout = bn(z(out)) [+ out]   /root/reference/modeling/layers/epipolar.py:249-253 (eval-mode BN folded
// into Wf, bf by epi_fold_z_bn_f32) and  ret + feat   /root/reference/modeling/backbones/resnet.py:388.
//
// The product is computed transposed, Yᵀ[128 out-ch, 256 px] = (Wf + I)·Xᵀ per CTA (grid: pixel tiles of one item × blocks of
// 128 output channels), so that an accumulator row is one output channel and its columns are consecutive pixels of one NCHW
// row: each warp turns its fragments into whole row segments in a slice of the idle ring, with no CTA-wide tile or barrier
// beyond one named barrier between the two MMA warpgroups.  Both operands are K-major as they lie in memory: the staged weight's
// (hi, lo) planes [C out][C in] (MMA A, one warpgroup per 64 output channels) and the fused feature's (hi, lo) planes
// [N·HW, C] (MMA B, N = 256 pixels).  Three MMAs per product (hi·hi + lo·hi + hi·lo), fp32 accumulation in registers.
// K is streamed in 64-channel panels through a ring of STAGES shared-memory stages: one lane of a ninth warp issues the TMA
// loads (cp.async.bulk.tensor.2d, 128-byte swizzle, completion on the stage's `full` mbarrier), the warpgroups issue panel q's
// MMAs before they retire panel q-1's (wgmma.wait_group 1) and hand the stage back through its `empty` mbarrier, and the
// loader refills it with panel q+1 while panel q multiplies.  The loader has a warp of its own because a loader branch inside
// the MMA loop would make ptxas serialise the wgmmas (C7518).
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstring>

#include <type_traits>

#include "epi_kernels.cuh"
#include "epi_umma.cuh"

namespace epi {
using namespace umma;

namespace zg {
constexpr int NT = 288;                             // two MMA warpgroups and the loader warp
constexpr int MO = 128;                             // output channels per CTA (MMA M: 64 per warpgroup)
constexpr int NP = 256;                             // pixels per CTA (MMA N)
constexpr uint32_t W_PLANE = MO * 128;              // 16 KB: 128 channel rows x 128 B
constexpr uint32_t X_PLANE = NP * 128;              // 32 KB: 256 pixel rows x 128 B
constexpr uint32_t STAGE = 2 * W_PLANE + 2 * X_PLANE;   // 96 KB: one K panel of (W hi, W lo, X hi, X lo)
constexpr int STAGES = 2;
constexpr int OP = NP + 8;                         // epilogue slice pitch (floats): two-way bank conflicts at most
constexpr uint32_t SMEM_ALLOC = STAGES * STAGE + 1024 + 64;     // ~193 KB: one CTA per SM

// 2-D tiled TMA load of a [box rows x 64 bf16] box into a swizzled panel, completion counted on `bar`
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *tmap, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     umma::smem_u32(smem_dst)),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(umma::smem_u32(bar))
                 : "memory");
}
// a bounded wait: a phase that never completes (a lost TMA) traps instead of hanging the stream
__device__ __forceinline__ void wait_or_trap(uint64_t *bar, uint32_t parity) {
    for (uint32_t it = 0; !mbar_try_wait(bar, parity); ++it) if (it > (1u << 24)) __trap();
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
__global__ void __launch_bounds__(zg::NT, 1) epi_zgemm_kernel(const ZGemmArgs z, const __grid_constant__ CUtensorMap tm_hi,
                                                              const __grid_constant__ CUtensorMap tm_lo,
                                                              const __grid_constant__ CUtensorMap tw_hi,
                                                              const __grid_constant__ CUtensorMap tw_lo,
                                                              const std::conditional_t<TABLE, ViewSources, NoTable> vs) {
    using namespace zg;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + STAGES * STAGE);  // stage s holds its K panel (TMA)
    uint64_t *empty = full + STAGES;                                         // every MMA warpgroup is done with stage s
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, t128 = tid & 127;
    const int C = z.C, HW = z.HW, W = z.W;
    const int tiles = (HW + NP - 1) / NP;
    const int n = blockIdx.x / tiles, p0 = (blockIdx.x % tiles) * NP;
    const int nq = C / 64;                             // K panels of 64 channels
    const int oc0 = (int)blockIdx.y * MO;             // this CTA's block of output channels
    const int CO = min(MO, C - oc0);
    const int nwg = CO > 64 ? 2 : 1;                   // warpgroups with output channels (C = 64 and a last block of 64 use one)

    // No pdl_launch_dependents(): the next forward's staging launch then starts when this grid completes.  Triggered early,
    // its persistent CTAs were placed on the SMs this one-CTA-per-SM grid leaves partly free and made the bench.py step
    // 5-6 µs longer (DESIGN.md §3.3).  This launch itself still starts under the fused kernel's tail (pdl_wait below).
    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(full + s, 1); mbar_init(empty + s, (uint32_t)nwg); }
        mbar_fence_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tw_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tw_lo) : "memory");
    }
    __syncthreads();
    pdl_wait();                                        // the fused kernel's feature planes (and the staged weight)
    // The loader (lane 0 of warp 8) loads K panel q into stage q % STAGES once the MMAs of panel q - STAGES have released it:
    // W rows oc0 .. +127 (rows past C arrive zero-filled; a C of 64 is one 64-row box) and pixel rows n·HW + p0 .. +255 of the
    // (hi, lo) planes (rows past N·HW zero-filled, rows of the next item computed and discarded).
    const uint32_t wrows = (uint32_t)(C < MO ? C : MO);            // W box rows (the tensor map's box)
    auto load = [&](int q) {
        const int s = q % STAGES;
        uint8_t *st = smem + s * STAGE;
        mbar_arrive_expect_tx(full + s, 2 * wrows * 128u + 2 * X_PLANE);
        tma_load_2d(st, &tw_hi, q * 64, oc0, full + s);
        tma_load_2d(st + W_PLANE, &tw_lo, q * 64, oc0, full + s);
        tma_load_2d(st + 2 * W_PLANE, &tm_hi, q * 64, n * HW + p0, full + s);
        tma_load_2d(st + 2 * W_PLANE + X_PLANE, &tm_lo, q * 64, n * HW + p0, full + s);
    };
    if (warp == 8) {
        if (lane == 0)
            for (int q = 0; q < nq; q++) {
                if (q >= STAGES) wait_or_trap(empty + q % STAGES, (uint32_t)(q / STAGES - 1) & 1u);
                load(q);
            }
        return;
    }
    if (wg >= nwg) return;                             // no output channels for this warpgroup (and no barrier left to meet)

    // Main loop: warpgroup wg multiplies output channels oc0 + 64 wg .. +63 by the CTA's 256 pixels.  Every element's sum runs
    // over K in one fixed order (panel, 16-channel step, hi·hi, lo·hi, hi·lo), whatever the tile, grid or batch.
    float acc[128];
#pragma unroll
    for (int e = 0; e < 128; e++) acc[e] = 0.f;
    for (int q = 0; q < nq; q++) {
        const int s = q % STAGES;
        wait_or_trap(full + s, (uint32_t)(q / STAGES) & 1u);
        const uint32_t sa = smem_u32(smem + s * STAGE) + (uint32_t)wg * 8192u, sb = smem_u32(smem + s * STAGE) + 2 * W_PLANE;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
            const uint64_t a_hi = make_smem_desc(sa + ks * 32, 16, 1024), a_lo = desc_add(a_hi, W_PLANE);
            const uint64_t b_hi = make_smem_desc(sb + ks * 32, 16, 1024), b_lo = desc_add(b_hi, X_PLANE);
            wgmma_m64n256<0>(acc, a_hi, b_hi);
            wgmma_m64n256<0>(acc, a_lo, b_hi);
            wgmma_m64n256<0>(acc, a_hi, b_lo);
        }
        wg_commit();
        wg_wait_1();                                   // panel q-1's MMAs have retired; panel q's run on
        if (q > 0 && t128 == 0) mbar_arrive(empty + (q - 1) % STAGES);
    }
    wg_wait_all();

    // ---- epilogue -> NCHW --------------------------------------------------------------------------------------------
    // Thread t128 holds output channels r and r + 8 (r = acc_row(t128, 0)) at pixel pairs p0 + 8j + 2(t128 & 3), j = 0..31.
    // Vector path: each warp passes its 16 channel rows x 256 pixels through a private slice of the (now idle) ring, so that
    // every store instruction writes 512 contiguous bytes of one channel row (for fp32; 256 for a 16-bit y), as full 128-byte
    // lines: stored straight from the fragments, four lanes cover only 32 bytes of a row, and the partly written lines cost
    // step time (measured).  The ZRESIDUAL needs no term: the staged weight is Wf + I.  The bias and the caller's residual are
    // read here, not held across the main loop.  Strides that are not pixel-contiguous take per-element stores from the fragments.
    const bool addr = z.ref && z.add_ref;
    const bool vec = (z.y_stride[3] == 1) && (z.y_stride[2] == W) && (HW % 4 == 0) && (z.y_stride[1] % 4 == 0) && (z.y_stride[0] % 4 == 0) &&
                     ((reinterpret_cast<uintptr_t>(z.y) & (4 * sizeof(TO) - 1)) == 0) &&
                     (!addr || ((z.ref_stride[3] == 1) && (z.ref_stride[2] == W) && (z.ref_stride[1] % 4 == 0) && (z.ref_stride[0] % 4 == 0) &&
                                ((reinterpret_cast<uintptr_t>(z.ref) & (4 * feat_esize(z.ref_dtype) - 1)) == 0)));
    const int64_t qref = addr ? (int64_t)pair_items(n, z.n_ref, z.n_views, vs).q * z.ref_stride[0] : 0;
    if (vec) {
        asm volatile("bar.sync 1, %0;" ::"r"(nwg * 128) : "memory");     // every MMA warpgroup is done reading the ring
        float *buf = reinterpret_cast<float *>(smem) + (wg * 4 + (warp & 3)) * (16 * OP);   // this warp's [16][OP] slice
#pragma unroll
        for (int e = 0; e < 128; e += 2)
            *reinterpret_cast<float2 *>(buf + acc_row(lane, e) * OP + acc_col(lane, e)) = make_float2(acc[e], acc[e + 1]);
        __syncwarp();
        const int rw = wg * 64 + (warp & 3) * 16;      // the warp's first channel row in the CTA's block
        for (int lr = 0; lr < 16 && rw + lr < CO; lr++) {
            const int o = oc0 + rw + lr;
            const float b = __ldg(z.bf + o);           // folded bias: written long before the staging launch
            TO *yrow = static_cast<TO *>(z.y) + (int64_t)n * z.y_stride[0] + (int64_t)o * z.y_stride[1];
#pragma unroll
            for (int half = 0; half < 2; half++) {
                const int pp = half * 128 + lane * 4, p = p0 + pp;
                if (p >= HW) break;                    // HW % 4 == 0: p < HW covers p + 3
                const float4 t = *reinterpret_cast<const float4 *>(buf + lr * OP + pp);
                float4 v = make_float4(t.x + b, t.y + b, t.z + b, t.w + b);
                if (addr) {
                    const int64_t i = qref + (int64_t)o * z.ref_stride[1] + p;      // the caller's map, in its type
                    const float4 rv = z.ref_dtype == kBF16 ? ld4_cs(static_cast<const __nv_bfloat16 *>(z.ref) + i)
                                    : z.ref_dtype == kF16  ? ld4_cs(static_cast<const __half *>(z.ref) + i)
                                                           : ld4_cs(static_cast<const float *>(z.ref) + i);
                    v = make_float4(v.x + rv.x, v.y + rv.y, v.z + rv.z, v.w + rv.w);
                }
                st4_cs(yrow + p, v);
            }
        }
        return;
    }
    const int r = wg * 64 + acc_row(t128, 0), pc = p0 + ((t128 & 3) << 1);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int ol = r + 8 * h;
        if (ol >= CO) continue;
        const int o = oc0 + ol;
        const float b = __ldg(z.bf + o);
        TO *yrow = static_cast<TO *>(z.y) + (int64_t)n * z.y_stride[0] + (int64_t)o * z.y_stride[1];
        const int64_t rrow = qref + (int64_t)o * z.ref_stride[1];
#pragma unroll
        for (int j = 0; j < 32; j++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int p = pc + 8 * j + e;
                if (p >= HW) continue;
                const int py = p / W, px = p % W;
                float val = acc[4 * j + 2 * h + e] + b;
                if (addr) val += ld_feat(z.ref, rrow + (int64_t)py * z.ref_stride[2] + (int64_t)px * z.ref_stride[3], z.ref_dtype);
                yrow[(int64_t)py * z.y_stride[2] + (int64_t)px * z.y_stride[3]] = from_f32<TO>(val);
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
    const int tiles = (z.HW + zg::NP - 1) / zg::NP;
    const auto kern = epi_zgemm_kernel<TABLE, TO>;
    static thread_local DeviceFlags attr_set;
    const int dev = current_device();
    if (!attr_set.has(dev)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)zg::SMEM_ALLOC);
        if (e != cudaSuccess) return e;
        attr_set.set(dev);
    }
    // tensor maps are a pure function of (pointers, shape): keep the last set per host thread
    struct MapCache { const void *xh, *wh; int rows, C; CUtensorMap m[4]; };
    static thread_local MapCache mc = {nullptr, nullptr, 0, 0, {}};
    if (mc.xh != z.x_hi || mc.wh != z.w_hi || mc.rows != z.N * z.HW || mc.C != z.C) {
        const int wrows = z.C < zg::MO ? z.C : zg::MO;
        if (!make_plane_map(&mc.m[0], z.x_hi, z.N * z.HW, z.C, zg::NP) || !make_plane_map(&mc.m[1], z.x_lo, z.N * z.HW, z.C, zg::NP) ||
            !make_plane_map(&mc.m[2], z.w_hi, z.C, z.C, wrows) || !make_plane_map(&mc.m[3], z.w_lo, z.C, z.C, wrows))
            return cudaErrorInvalidValue;
        mc.xh = z.x_hi; mc.wh = z.w_hi; mc.rows = z.N * z.HW; mc.C = z.C;
    }
    return launch_pdl(kern, dim3((unsigned)(z.N * tiles), (unsigned)((z.C + zg::MO - 1) / zg::MO)), dim3(zg::NT), (size_t)zg::SMEM_ALLOC, st, z, mc.m[0], mc.m[1], mc.m[2], mc.m[3], vs);
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
