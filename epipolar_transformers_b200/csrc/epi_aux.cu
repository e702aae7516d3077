// epi_aux.cu — layout staging, parameter folding, the z/BN epilogue and the geometry-only kernel.
#include "epi_kernels.cuh"

namespace epi {

// ------------------------------------------------------------------------------------------
// [N,C,H,W] (any strides, element type T) -> [N,H,W,C] contiguous fp32.  32x32 shared-memory transpose per
// item: reads are coalesced along the pixel axis when stride[3]==1 (NCHW), writes along channels.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const T *__restrict__ src, int64_t sn, int64_t sc,
                                                           int64_t sh, int64_t sw, float *__restrict__ dst,
                                                           int C, int H, int W) {
    __shared__ float tile[32][33];
    const int HW = H * W;
    const int n = blockIdx.z, c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
    const T *s = src + (int64_t)n * sn;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int c = c0 + ty + i * 8, p = p0 + tx;
        tile[ty + i * 8][tx] = (c < C && p < HW) ? to_f32(__ldg(s + c * sc + (p / W) * sh + (p % W) * sw)) : 0.f;
    }
    __syncthreads();
    float *d = dst + (size_t)n * HW * C;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int p = p0 + ty + i * 8, c = c0 + tx;
        if (c < C && p < HW) d[(size_t)p * C + c] = tile[tx][ty + i * 8];
    }
}

cudaError_t launch_nchw_to_nhwc(const void *src, const int64_t stride[4], float *dst, int N, int C, int H, int W, int dtype,
                                cudaStream_t st) {
    dim3 grid((H * W + 31) / 32, (C + 31) / 32, N);
    if (dtype == kBF16)
        nchw_to_nhwc_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16 *>(src), stride[0], stride[1], stride[2], stride[3], dst, C, H, W);
    else if (dtype == kF16)
        nchw_to_nhwc_kernel<<<grid, 256, 0, st>>>(static_cast<const __half *>(src), stride[0], stride[1], stride[2], stride[3], dst, C, H, W);
    else
        nchw_to_nhwc_kernel<<<grid, 256, 0, st>>>(static_cast<const float *>(src), stride[0], stride[1], stride[2], stride[3], dst, C, H, W);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// [N,C,H,W] (any strides, element type T) -> two bf16 planes [N,H,W,C] with src ≈ hi + lo (operands of the
// tensor-core kernel).  Lo planes are written for bf16 maps too: the tile kernel reads them.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) split_planes_kernel(const T *__restrict__ src, int64_t sn, int64_t sc, int64_t sh,
                                                           int64_t sw, __nv_bfloat16 *__restrict__ hi,
                                                           __nv_bfloat16 *__restrict__ lo, int C, int H, int W, int *zero_me) {
    __shared__ float tile[64][65];
    if (zero_me && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0) *zero_me = 0;   // tile scheduler counter
    const int n = blockIdx.z;
    const T *s = src + (int64_t)n * sn;
    stage_planes_tile<T, true>(tile, s, sc, sh, sw, nchw_vec4(s, sc, sh, sw, W, H * W), hi, lo, n, blockIdx.y * 64, blockIdx.x * 64, C, H, W);
}

cudaError_t launch_split_planes(const void *src, const int64_t stride[4], __nv_bfloat16 *hi, __nv_bfloat16 *lo, int N, int C,
                                int H, int W, int *zero_me, int dtype, cudaStream_t st) {
    dim3 grid((H * W + 63) / 64, (C + 63) / 64, N);
    if (dtype == kBF16)
        split_planes_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16 *>(src), stride[0], stride[1], stride[2], stride[3], hi, lo, C, H, W, zero_me);
    else if (dtype == kF16)
        split_planes_kernel<<<grid, 256, 0, st>>>(static_cast<const __half *>(src), stride[0], stride[1], stride[2], stride[3], hi, lo, C, H, W, zero_me);
    else
        split_planes_kernel<<<grid, 256, 0, st>>>(static_cast<const float *>(src), stride[0], stride[1], stride[2], stride[3], hi, lo, C, H, W, zero_me);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Pixel-major fp32 plane [N,H*W,C] (what the fused kernel writes with full 128-byte lines) -> the caller's
// [N,C,H,W] tensor of element type TO (any strides; fp32 sums rounded once), optionally adding the caller's residual
// feat_ref of element type TR (resnet.py:388).  64 x 64
// tiles through shared memory: reads along channels (float4 when C % 4 == 0, so that every pixel row starts on a
// 16-byte boundary; scalar otherwise, as for the source gradient of a backward with C % 4 != 0), float4 writes
// along pixels.
// ------------------------------------------------------------------------------------------
template <typename TO, typename TR>
__global__ void __launch_bounds__(256) unstage_kernel(const float *__restrict__ pm, const TR *__restrict__ ref, int64_t rn,
                                                      int64_t rc, int64_t rh, int64_t rw, TO *__restrict__ out, int64_t on,
                                                      int64_t oc, int64_t oh, int64_t ow, int n_ref, int n_views, const ViewSources vs,
                                                      int C, int H, int W) {
    __shared__ float tile[64][65];                              // [channel][pixel]
    const int HW = H * W, t = threadIdx.x;
    const int n = blockIdx.z, c0 = blockIdx.y * 64, p0 = blockIdx.x * 64;
    const int64_t rofs = (int64_t)pair_items(n, n_ref, n_views, vs).q * rn;      // the item's reference (several pairs may share one)
    {
        const int q = t & 15, pl = t >> 4;                      // 16 float4 per pixel row (64 channels), 16 pixels per pass
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int p = p0 + pl + i * 16, c = c0 + q * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < HW && c < C) {
                const float *row = pm + ((size_t)n * HW + p) * C + c;
                if (C % 4 == 0) v = __ldg(reinterpret_cast<const float4 *>(row));
                else v = make_float4(__ldg(row), c + 1 < C ? __ldg(row + 1) : 0.f, c + 2 < C ? __ldg(row + 2) : 0.f,
                                     c + 3 < C ? __ldg(row + 3) : 0.f);
            }
            tile[q * 4 + 0][pl + i * 16] = v.x; tile[q * 4 + 1][pl + i * 16] = v.y;
            tile[q * 4 + 2][pl + i * 16] = v.z; tile[q * 4 + 3][pl + i * 16] = v.w;
        }
    }
    __syncthreads();
    const bool vec_o = (ow == 1) && (oh == W) && (HW % 4 == 0) && (oc % 4 == 0) && (on % 4 == 0) && ((reinterpret_cast<uintptr_t>(out) & (4 * sizeof(TO) - 1)) == 0);
    const bool vec_r = !ref || ((rw == 1) && (rh == W) && (rc % 4 == 0) && (rn % 4 == 0) && ((reinterpret_cast<uintptr_t>(ref) & (4 * sizeof(TR) - 1)) == 0));
    const int q = t & 15, cy = t >> 4;                          // 16 float4 per channel row, 16 channels per pass
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int c = c0 + cy + i * 16, p = p0 + q * 4;
        if (c >= C || p >= HW) continue;
        float v[4] = {tile[cy + i * 16][q * 4], tile[cy + i * 16][q * 4 + 1], tile[cy + i * 16][q * 4 + 2], tile[cy + i * 16][q * 4 + 3]};
        if (vec_o && vec_r && p + 3 < HW) {
            if (ref) {
                const float4 r4 = ld4_nc(ref + rofs + (int64_t)c * rc + p);
                v[0] += r4.x; v[1] += r4.y; v[2] += r4.z; v[3] += r4.w;
            }
            st4(out + (int64_t)n * on + (int64_t)c * oc + p, make_float4(v[0], v[1], v[2], v[3]));
        } else {
            for (int j = 0; j < 4 && p + j < HW; j++) {
                const int y = (p + j) / W, x = (p + j) % W;
                float o = v[j];
                if (ref) o += to_f32(__ldg(ref + rofs + (int64_t)c * rc + (int64_t)y * rh + (int64_t)x * rw));
                out[(int64_t)n * on + (int64_t)c * oc + (int64_t)y * oh + (int64_t)x * ow] = from_f32<TO>(o);
            }
        }
    }
}

template <typename TO, typename TR>
static void unstage_t(dim3 grid, cudaStream_t st, const float *pm, const void *ref, const int64_t ref_stride[4], void *out,
                      const int64_t out_stride[4], int n_ref, int n_views, const ViewSources &vs, int C, int H, int W) {
    unstage_kernel<TO, TR><<<grid, 256, 0, st>>>(pm, static_cast<const TR *>(ref), ref ? ref_stride[0] : 0, ref ? ref_stride[1] : 0,
                                                 ref ? ref_stride[2] : 0, ref ? ref_stride[3] : 0, static_cast<TO *>(out), out_stride[0],
                                                 out_stride[1], out_stride[2], out_stride[3], n_ref, n_views, vs, C, H, W);
}

// without a residual TR is float and never read
template <typename TO>
static void unstage_out(dim3 grid, cudaStream_t st, const float *pm, const void *ref, int ref_dtype, const int64_t ref_stride[4], void *out,
                        const int64_t out_stride[4], int n_ref, int n_views, const ViewSources &vs, int C, int H, int W) {
    if (ref && ref_dtype == kBF16) unstage_t<TO, __nv_bfloat16>(grid, st, pm, ref, ref_stride, out, out_stride, n_ref, n_views, vs, C, H, W);
    else if (ref && ref_dtype == kF16) unstage_t<TO, __half>(grid, st, pm, ref, ref_stride, out, out_stride, n_ref, n_views, vs, C, H, W);
    else unstage_t<TO, float>(grid, st, pm, ref, ref_stride, out, out_stride, n_ref, n_views, vs, C, H, W);
}

cudaError_t launch_unstage(const float *pm, const void *ref, int ref_dtype, const int64_t ref_stride[4], void *out, int out_dtype,
                           const int64_t out_stride[4], int N, int n_ref, int n_views, const ViewSources &vs, int C, int H, int W,
                           cudaStream_t st) {
    dim3 grid((H * W + 63) / 64, (C + 63) / 64, N);
    if (out_dtype == kBF16) unstage_out<__nv_bfloat16>(grid, st, pm, ref, ref_dtype, ref_stride, out, out_stride, n_ref, n_views, vs, C, H, W);
    else if (out_dtype == kF16) unstage_out<__half>(grid, st, pm, ref, ref_dtype, ref_stride, out, out_stride, n_ref, n_views, vs, C, H, W);
    else unstage_out<float>(grid, st, pm, ref, ref_dtype, ref_stride, out, out_stride, n_ref, n_views, vs, C, H, W);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Deterministic backward: fixed-point sums [N,HW,C] (int64, scale 2^s of pair n, det_scale) -> the pixel-major fp32 gradient
// buffer the transposition pass reads, each value rounded once: fp32(acc·2^-s).  A pair whose bound is not finite was not
// scattered and comes out all NaN; a pair with a zero bound comes out zero.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) acc_to_f32_kernel(const long long *__restrict__ acc, const unsigned *__restrict__ pair_max,
                                                         float *__restrict__ dsrc, int HW, int C) {
    const int n = blockIdx.y;
    const size_t len = (size_t)HW * C, base = (size_t)n * len;
    const unsigned word = __ldg(pair_max + n);
    int s = 0;
    const bool scaled = det_scale(word, HW, s);
    const float fill = __uint_as_float(word) == 0.f ? 0.f : __int_as_float(0x7fffffff);     // zero bound: zeros; else NaN
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (size_t)gridDim.x * blockDim.x)
        dsrc[base + i] = scaled ? (float)ldexp((double)__ldg(acc + base + i), -s) : fill;
}

cudaError_t launch_acc_to_f32(const long long *acc, const unsigned *pair_max, float *dsrc, int N, int HW, int C, cudaStream_t st) {
    const size_t len = (size_t)HW * C;
    const int blocks = (int)((len + 255) / 256 < 1024 ? (len + 255) / 256 : 1024);
    acc_to_f32_kernel<<<dim3(blocks, N), 256, 0, st>>>(acc, pair_max, dsrc, HW, C);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Views form of the backward: one pass per view item sums its query terms (one pixel-major fp32 plane per pair, order-fixed) in
// the order of its pairs and adds its source term, float sums or fixed-point sums converted with the item's scale (NaN for an
// item one of whose pairs has a non-finite bound, zero for a zero bound).  Each element is read and written by one thread, so
// `g` may be `dsrc`.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) views_grad_sum_kernel(const float *__restrict__ gq, const float *dsrc, const long long *__restrict__ acc,
                                                             const unsigned *__restrict__ item_max, float *g, const BwdViews vw,
                                                             int HW, int C) {
    const int i = blockIdx.y, v = i / vw.n_ref, n = i - v * vw.n_ref;
    const int S = vw.vs.S ? vw.vs.S : vw.n_views - 1;
    const size_t len = (size_t)HW * C, base = (size_t)i * len;
    int s = 0;
    bool scaled = false;
    float fill = 0.f;
    if (acc) {
        const unsigned word = __ldg(item_max + i);
        scaled = det_item_scale(word, HW, view_source_count(v, vw.n_views, vw.vs), s);
        fill = __uint_as_float(word) == 0.f ? 0.f : __int_as_float(0x7fffffff);
    }
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < len; e += (size_t)gridDim.x * blockDim.x) {
        float sum = __ldg(gq + (size_t)(v * S * vw.n_ref + n) * len + e);
        for (int j = 1; j < S; j++) sum += __ldg(gq + (size_t)((v * S + j) * vw.n_ref + n) * len + e);
        if (dsrc) sum += dsrc[base + e];
        else if (acc) sum += scaled ? (float)ldexp((double)__ldg(acc + base + e), -s) : fill;
        g[base + e] = sum;
    }
}

cudaError_t launch_views_grad_sum(const float *gq, const float *dsrc, const long long *acc, const unsigned *item_max, float *g,
                                  const BwdViews &vw, int HW, int C, cudaStream_t st) {
    const size_t len = (size_t)HW * C;
    const int blocks = (int)((len + 255) / 256 < 1024 ? (len + 255) / 256 : 1024);
    views_grad_sum_kernel<<<dim3(blocks, vw.n_views * vw.n_ref), 256, 0, st>>>(gq, dsrc, acc, item_max, g, vw, HW, C);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Fold conv1x1 z + eval BN (epipolar.py:250-251, BN.py:79 with training=False) into Wf, bf.
// ------------------------------------------------------------------------------------------
__global__ void fold_z_bn_kernel(const float *__restrict__ zw, const float *__restrict__ zb,
                                 const float *__restrict__ g, const float *__restrict__ b,
                                 const float *__restrict__ mean, const float *__restrict__ var, float eps, int C,
                                 float *__restrict__ wf, float *__restrict__ bf) {
    const int o = blockIdx.x;
    const float s = g[o] / sqrtf(var[o] + eps);
    for (int c = threadIdx.x; c < C; c += blockDim.x) wf[(size_t)o * C + c] = s * zw[(size_t)o * C + c];
    if (threadIdx.x == 0) bf[o] = s * ((zb ? zb[o] : 0.f) - mean[o]) + b[o];
}

cudaError_t launch_fold_z_bn(const float *zw, const float *zb, const float *g, const float *b, const float *mean,
                             const float *var, float eps, int C, float *wf, float *bf, cudaStream_t st) {
    fold_z_bn_kernel<<<C, 128, 0, st>>>(zw, zb, g, b, mean, var, eps, C, wf, bf);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// z epilogue: per item Y[C x HW] = Wf[C x C] · X[C x HW] + bf (+X) (+ref).  fp32 CUDA-core
// SGEMM, 64x64 tile, 4x4 per thread.  X is the library's own contiguous pre-z buffer.
// ------------------------------------------------------------------------------------------
constexpr int ZT = 64, ZK = 16;

// (min 5 blocks per SM: 48 registers.  Unbounded, ptxas spends 64 on the source-table branch of pair_items and a block fewer fits.)
// TO: element type of y, the fp32 result rounded once
template <typename TO>
__global__ void __launch_bounds__(256, 5) z_epilogue_kernel(const ZArgs z) {
    __shared__ float Ws[ZK][ZT + 1];     // [k][o]
    __shared__ float Xs[ZK][ZT + 1];     // [k][p]
    const int n = blockIdx.z, o0 = blockIdx.y * ZT, p0 = blockIdx.x * ZT;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;       // tx -> p, ty -> o
    const int C = z.C, HW = z.HW, W = z.W;
    const float *X = z.x + (int64_t)n * z.x_stride[0];
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < C; k0 += ZK) {
        for (int idx = tid; idx < ZK * ZT; idx += 256) {
            int kk = idx & (ZK - 1), oo = idx / ZK;                   // W rows are contiguous in c
            int o = o0 + oo, c = k0 + kk;
            Ws[kk][oo] = (o < C && c < C) ? __ldg(z.Wf + (size_t)o * C + c) : 0.f;
            int pp = idx & (ZT - 1), kx = idx / ZT;
            int p = p0 + pp, cx = k0 + kx;
            Xs[kx][pp] = (p < HW && cx < C) ? __ldg(X + cx * z.x_stride[1] + (p / W) * z.x_stride[2] + (p % W) * z.x_stride[3]) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < ZK; kk++) {
            float wv[4], xv[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { wv[i] = Ws[kk][ty * 4 + i]; xv[i] = Xs[kk][tx + 16 * i]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(wv[i], xv[j], acc[i][j]);
        }
        __syncthreads();
    }
    TO *Y = static_cast<TO *>(z.y) + (int64_t)n * z.y_stride[0];
    const float *R = z.ref ? z.ref + (int64_t)pair_items(n, z.n_ref, z.n_views, z.vsrc).q * z.ref_stride[0] : nullptr;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int o = o0 + ty * 4 + i;
        if (o >= C) continue;
        float b = __ldg(z.bf + o);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int p = p0 + tx + 16 * j;
            if (p >= HW) continue;
            int yy = p / W, xx = p % W;
            float v = acc[i][j] + b;
            if (z.z_residual) v += __ldg(X + o * z.x_stride[1] + yy * z.x_stride[2] + xx * z.x_stride[3]);
            if (z.add_ref && R) v += __ldg(R + o * z.ref_stride[1] + yy * z.ref_stride[2] + xx * z.ref_stride[3]);
            Y[o * z.y_stride[1] + yy * z.y_stride[2] + xx * z.y_stride[3]] = from_f32<TO>(v);
        }
    }
}

cudaError_t launch_z_epilogue(const ZArgs &z, int y_dtype, cudaStream_t st) {
    dim3 grid((z.HW + ZT - 1) / ZT, (z.C + ZT - 1) / ZT, z.N);
    if (y_dtype == kBF16) z_epilogue_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(z);
    else if (y_dtype == kF16) z_epilogue_kernel<__half><<<grid, 256, 0, st>>>(z);
    else z_epilogue_kernel<float><<<grid, 256, 0, st>>>(z);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// geometry only: sample locations [K,N,H,W,2] (grid2sample_locs, epipolar.py:323-418)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sample_locs_kernel(const float *__restrict__ P_ref, const float *__restrict__ P_src,
                                                          float *__restrict__ locs, int N, const GeomCfg gc) {
    __shared__ PairGeom sg;
    const int n = blockIdx.y, HW = gc.H * gc.W;
    if (threadIdx.x == 0) pair_geom_from_krt(P_ref + 12 * n, P_src + 12 * n, sg);
    __syncthreads();
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    float sx, sy, ex, ey;
    line_endpoints(sg, gc, pix2coord(p % gc.W, gc.ds, gc.r), pix2coord(p / gc.W, gc.ds, gc.r), sx, sy, ex, ey);
    for (int k = 0; k < gc.K; k++) {
        float t = (float)k / (float)(gc.K - 1);
        reinterpret_cast<float2 *>(locs)[((size_t)k * N + n) * HW + p] =
            make_float2(img2grid_x(sx + (ex - sx) * t, gc), img2grid_y(sy + (ey - sy) * t, gc));
    }
}

cudaError_t launch_sample_locs(const float *P_ref, const float *P_src, float *locs, int N, const GeomCfg &gc,
                               cudaStream_t st) {
    dim3 grid((gc.H * gc.W + 255) / 256, N);
    sample_locs_kernel<<<grid, 256, 0, st>>>(P_ref, P_src, locs, N, gc);
    return cudaGetLastError();
}

}  // namespace epi
