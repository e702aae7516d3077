// epi_common.cuh — shared device code of the epipolar fusion kernels (sm_90a).
//
// Geometry restates grid2sample_locs (/root/reference/modeling/layers/epipolar.py:323-418) and
// the helpers of /root/reference/vision/multiview.py (:16-21 camera_center, :25-37 normalize,
// :39-57 de_normalize, :154-163 pix2coord/coord2pix) per pixel, with the better-conditioned
// infinite-homography point x2' = (A2 A1^-1) p on the same epipolar line (SURVEY.md app. B).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace epi {

constexpr float kFar = 10000.0f;      // epipolar.py:51-53
constexpr float kMasked = -1e10f;     // epipolar.py:298

// Element types of the feature maps (EPI_DTYPE_* of the C ABI).  bf16 and fp16 values are exact in fp32, so every kernel
// computes on the fp32 value of the input; only the loads (and the backward's gradient stores) see the storage type.
enum FeatDtype { kF32 = 0, kBF16 = 1, kF16 = 2 };

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// four consecutive elements as fp32; p is aligned to 4 elements.  Streaming (read-once) load.
__device__ __forceinline__ float4 ld4_cs(const float *p) { return __ldcs(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 ld4_cs(const __nv_bfloat16 *p) {
    const uint2 r = __ldcs(reinterpret_cast<const uint2 *>(p));
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.x)), b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 ld4_cs(const __half *p) {
    const uint2 r = __ldcs(reinterpret_cast<const uint2 *>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&r.x)), b = __half22float2(*reinterpret_cast<const __half2 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
// the same through the read-only cache
__device__ __forceinline__ float4 ld4_nc(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 ld4_nc(const __nv_bfloat16 *p) {
    const uint2 r = __ldg(reinterpret_cast<const uint2 *>(p));
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.x)), b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 ld4_nc(const __half *p) {
    const uint2 r = __ldg(reinterpret_cast<const uint2 *>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&r.x)), b = __half22float2(*reinterpret_cast<const __half2 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
// four consecutive elements from fp32, rounded once to T; p is aligned to 4 elements
__device__ __forceinline__ void st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
__device__ __forceinline__ void st4(__nv_bfloat16 *p, float4 v) {
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b));
}
__device__ __forceinline__ void st4(__half *p, float4 v) {
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b));
}
// element i of a feature map whose type is only known at run time (residual reads off the hot loops)
__device__ __forceinline__ float ld_feat(const void *p, int64_t i, int dtype) {
    if (dtype == kBF16) return __bfloat162float(__ldg(static_cast<const __nv_bfloat16 *>(p) + i));
    if (dtype == kF16) return __half2float(__ldg(static_cast<const __half *>(p) + i));
    return __ldg(static_cast<const float *>(p) + i);
}
__host__ __device__ __forceinline__ int feat_esize(int dtype) { return dtype == kF32 ? 4 : 2; }

// The bf16 (hi, lo) operand format of the tensor-core kernels: x ≈ hi + lo with hi = bf16(x), lo = bf16(x - hi)
// (|x - hi - lo| <~ 2^-17 |x|, exact for bf16 and fp16 values).  Every operand plane is split here, so all of them round alike.
// Two floats -> one bf16x2 word of hi parts and one of lo parts (a in the low 16 bits).
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t &hi, uint32_t &lo) {
    const __nv_bfloat162 hv = __floats2bfloat162_rn(a, b);
    const float2 hf = __bfloat1622float2(hv);
    const __nv_bfloat162 lv = __floats2bfloat162_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t *>(&hv);
    lo = *reinterpret_cast<const uint32_t *>(&lv);
}
// 8 floats -> one 16-byte chunk of hi parts and one of lo parts
__device__ __forceinline__ void split8(const float *f, uint4 &hi, uint4 &lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int u = 0; u < 4; u++) split_bf16x2(f[2 * u], f[2 * u + 1], h[u], l[u]);
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// an [N,C,H,W] item at s can be read as 4-element vectors along pixels (pixel-contiguous rows, 4-element aligned)
template <typename T>
__device__ __forceinline__ bool nchw_vec4(const T *s, int64_t sc, int64_t sh, int64_t sw, int W, int HW) {
    return (sw == 1) && (sh == W) && (HW % 4 == 0) && (sc % 4 == 0) && ((reinterpret_cast<uintptr_t>(s) & (4 * sizeof(T) - 1)) == 0);
}

// One tile of 64 channels x 64 pixels (from c0, p0) of item n of an [N,C,H,W] map -> pixel-major bf16 (hi, lo) planes
// [N,H*W,C]; LO = false writes the hi plane only (bf16 maps, whose lo part is zero).  s: the item (any strides, element type
// T); vec: nchw_vec4 of it; tile: [64][65] fp32 in shared memory; 256 threads; C % 8 == 0.  NCHW items are read as 4-pixel
// vectors where vec allows (a warp covers two 256-byte runs, which also keeps NVLink requests large when the map is a
// peer-mapped tensor of another GPU), channels-last ones along channels; the planes are written as 16-byte chunks of 8 channels.
template <typename T, bool LO>
__device__ __forceinline__ void stage_planes_tile(float (*tile)[65], const T *s, int64_t sc, int64_t sh, int64_t sw, bool vec,
                                                  __nv_bfloat16 *hi, __nv_bfloat16 *lo, int n, int c0, int p0, int C, int H, int W) {
    const int HW = H * W, t = threadIdx.x;
    if (sc != 1) {
        const int q = t % 16, cy = t / 16;                      // 16 float4 per channel row, 16 channels per pass
        float4 v[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int c = c0 + cy + i * 16, p = p0 + q * 4;
            v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c < C) {
                if (vec && p + 3 < HW) v[i] = ld4_nc(s + c * sc + p);
                else {
                    float e[4] = {0.f, 0.f, 0.f, 0.f};
                    for (int j = 0; j < 4; j++) if (p + j < HW) e[j] = to_f32(__ldg(s + c * sc + ((p + j) / W) * sh + ((p + j) % W) * sw));
                    v[i] = make_float4(e[0], e[1], e[2], e[3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            float *row = &tile[cy + i * 16][q * 4];
            row[0] = v[i].x; row[1] = v[i].y; row[2] = v[i].z; row[3] = v[i].w;
        }
    } else {
        const int cx = t % 64, py = t / 64;                     // channels-last: a warp reads 32 consecutive channels of one pixel
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const int p = p0 + py + i * 4, c = c0 + cx;
            tile[cx][py + i * 4] = (c < C && p < HW) ? to_f32(__ldg(s + c + (p / W) * sh + (p % W) * sw)) : 0.f;
        }
    }
    __syncthreads();
    const int cg = t % 8, pl = t / 8;                           // 8 channel groups x 32 pixels per pass
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int pp = pl + i * 32, p = p0 + pp, c = c0 + cg * 8;
        if (p < HW && c < C) {
            uint32_t h[4], l[4];
#pragma unroll
            for (int u = 0; u < 4; u++) split_bf16x2(tile[cg * 8 + 2 * u][pp], tile[cg * 8 + 2 * u + 1][pp], h[u], l[u]);
            const size_t o = ((size_t)n * HW + p) * C + c;
            *reinterpret_cast<uint4 *>(hi + o) = make_uint4(h[0], h[1], h[2], h[3]);
            if (LO) *reinterpret_cast<uint4 *>(lo + o) = make_uint4(l[0], l[1], l[2], l[3]);
        }
    }
}

// The source table of the views form (EPI_VIEW_SOURCES_MAX in the header): view v is fused with views src[v·S + j], j < S.
// S = 0 is the all-others form (u = j + (j >= v), no table).  Kernels take it by value in their arguments, so a table reaches
// them in the launch's parameter block: no copy to the device, no synchronisation.  Indexed reads compile to constant-bank loads.
constexpr int kMaxViewSources = 256;
struct ViewSources { int S; uint8_t src[kMaxViewSources]; };

// The two map items a (query, source) pair reads: every kernel maps pair p through this one function.
//   n_views == 0: p fuses reference item p % n_ref with source item p (n_src sources per reference item: p = s·n_ref + n).
//   n_views == V >= 2: one map holds the V·n_ref view items and is both the query and the source map; with S sources per view
//   (vs.S, or V−1 for the all-others form), p = (v·S + j)·n_ref + n fuses item v·n_ref + n with item u·n_ref + n, where
//   u = vs.src[v·S + j], or u = j + (j >= v) (the other views in increasing order) when vs.S == 0.
// Without `vs`: the forms that have no table.  The staging, pipelined and z GEMM kernels take the table as a trailing parameter
// pack (`const Tab... vs`) that is empty unless the call has a table, so the one-source, several-source and all-others forms
// launch them with no table bytes and no table code; the other kernels take a ViewSources and test vs.S at run time.
struct PairItems { int q, s; };
__host__ __device__ __forceinline__ PairItems pair_items(int p, int n_ref, int n_views) {
    if (n_views == 0) return {p % n_ref, p};
    const int vj = p / n_ref, n = p - vj * n_ref, v = vj / (n_views - 1), j = vj - v * (n_views - 1);
    return {v * n_ref + n, (j + (j >= v)) * n_ref + n};
}
__host__ __device__ __forceinline__ PairItems pair_items(int p, int n_ref, int n_views, const ViewSources &vs) {
    if (n_views == 0 || vs.S == 0) return pair_items(p, n_ref, n_views);
    const int vj = p / n_ref, n = p - vj * n_ref;
    return {vj / vs.S * n_ref + n, (int)vs.src[vj] * n_ref + n};
}

// Number of pairs whose source is view u: V−1 in the all-others form, else the table entries that name u.
__host__ __device__ __forceinline__ int view_source_count(int u, int n_views, const ViewSources &vs) {
    if (vs.S == 0) return n_views - 1;
    int c = 0;
    for (int i = 0; i < n_views * vs.S; i++) c += vs.src[i] == u;
    return c;
}

// Per-(ref,src)-pair constants: M = A2·A1^-1 (row-major 3x3) and the epipole e2/e2.z.
struct PairGeom {
    float M[9];
    float ex, ey;
};

// Launch-invariant geometry configuration.
struct GeomCfg {
    float ds, r, eps;
    float inv_rds, off_ds;          // image coord -> feature px:  pix = v*inv_rds + off_ds
    float gsx, gox, gsy, goy;       // feature px -> grid coord:   g = pix*gs + go   (per axis)
    float xmin, xmax, ymin, ymax;   // image coords of first/last pixel centres (epipolar.py:46-49)
    int correct;                    // USE_CORRECT_NORMALIZE
    int align;                      // grid_sample align_corners
    int H, W, K;
};

__host__ __device__ __forceinline__ float pix2coord(int i, float ds, float r) {
    return ((float)i * ds + ds * 0.5f - 0.5f) * r;           // multiview.py:154-157, epipolar.py:35-38
}

// fp64 pieces of a camera P = [A | t] (row-major 3x4): one thread each, so the per-pixel fp32 math starts from correctly
// rounded constants (SURVEY fact 10: the reference's fp32 pinv path is noisy).  Every pair constant and every epipole of a
// pixel order is computed by these, with one operation order.
// A and t in fp64
__device__ __forceinline__ void cam_load(const float *P, double A[9], double t[3]) {
    for (int r = 0; r < 3; r++) {
        for (int q = 0; q < 3; q++) A[r * 3 + q] = (double)P[r * 4 + q];
        t[r] = (double)P[r * 4 + 3];
    }
}
// A^-1 (row-major) by cofactors
__device__ __forceinline__ void cam_inverse(const double a[9], double ai[9]) {
    const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
    const double id = 1.0 / (a[0] * c00 + a[1] * c01 + a[2] * c02);
    ai[0] = c00 * id; ai[1] = (a[2] * a[7] - a[1] * a[8]) * id; ai[2] = (a[1] * a[5] - a[2] * a[4]) * id;
    ai[3] = c01 * id; ai[4] = (a[0] * a[8] - a[2] * a[6]) * id; ai[5] = (a[2] * a[3] - a[0] * a[5]) * id;
    ai[6] = c02 * id; ai[7] = (a[1] * a[6] - a[0] * a[7]) * id; ai[8] = (a[0] * a[4] - a[1] * a[3]) * id;
}
// camera centre -A^-1 t (multiview.py:16-21), ai = A^-1
__device__ __forceinline__ void cam_centre(const double ai[9], const double t[3], double c[3]) {
    for (int r = 0; r < 3; r++) c[r] = -(ai[r * 3] * t[0] + ai[r * 3 + 1] * t[1] + ai[r * 3 + 2] * t[2]);
}
// row r of the homogeneous projection [A | t]·[x; 1]
__device__ __forceinline__ double cam_project(const double A[9], const double t[3], const double x[3], int r) {
    return A[r * 3] * x[0] + A[r * 3 + 1] * x[1] + A[r * 3 + 2] * x[2] + t[r];
}

// pair constants: M = A2·A1^-1 and the epipole P2·[C1; 1] of the reference camera in the source view
__device__ inline void pair_geom_from_krt(const float *__restrict__ P1, const float *__restrict__ P2, PairGeom &g) {
    double a[9], b[9], ai[9], t1[3], t2[3], c[3], e[3];
    // both cameras in one loop, not two cam_load calls: the same values, but loading one camera after the other
    // reschedules (and re-spills) every kernel that inlines this, the staging kernel's hot streaming path included
    for (int r = 0; r < 3; r++) {
        for (int q = 0; q < 3; q++) { a[r * 3 + q] = (double)P1[r * 4 + q]; b[r * 3 + q] = (double)P2[r * 4 + q]; }
        t1[r] = (double)P1[r * 4 + 3]; t2[r] = (double)P2[r * 4 + 3];
    }
    cam_inverse(a, ai);
    cam_centre(ai, t1, c);
    for (int r = 0; r < 3; r++) {
        e[r] = cam_project(b, t2, c, r);
        for (int q = 0; q < 3; q++)
            g.M[r * 3 + q] = (float)(b[r * 3] * ai[q] + b[r * 3 + 1] * ai[3 + q] + b[r * 3 + 2] * ai[6 + q]);
    }
    g.ex = (float)(e[0] / e[2]);
    g.ey = (float)(e[1] / e[2]);
}

__device__ __forceinline__ float sdiv(float v, float eps) {       // sign(v)*max(|v|,eps), epipolar.py:370-373
    float a = fmaxf(fabsf(v), eps);
    return v > 0.f ? a : (v < 0.f ? -a : 0.f);
}

// Endpoints (image coords) of the epipolar line of reference pixel (px,py) clipped to the
// pixel-centre rectangle; far sentinel when fewer than two valid intersections (:369-405).
// A pixel whose ray is parallel to the source image plane has zz == 0 (exactly, when the fp32 constants cancel): x2 is
// then a point at infinity and l2 is not finite (also when a quotient overflows).  Its line is e2 × (zx, zy, zz), the
// zz → 0 limit of e2 × x2 up to the factor 1/zz; that factor grows without bound, so in the limit the eps clamp of the
// denominators never acts on a non-zero component, and the homogeneous line is clipped without it.  Every pixel with a
// finite l2 takes the quotient form unchanged.
__device__ __forceinline__ void line_endpoints(const PairGeom &g, const GeomCfg &c, float px, float py,
                                               float &sx, float &sy, float &ex, float &ey) {
    float zx = g.M[0] * px + g.M[1] * py + g.M[2];
    float zy = g.M[3] * px + g.M[4] * py + g.M[5];
    float zz = g.M[6] * px + g.M[7] * py + g.M[8];
    float x2 = zx / zz, y2 = zy / zz;
    float l0 = g.ey - y2, l1 = x2 - g.ex, l2 = g.ex * y2 - g.ey * x2;    // e2 × x2, both with z = 1
    float clamp = c.eps;
    if (!(fabsf(l2) <= 3.402823466e38f)) {                               // x2 not finite: e2 × (zx, zy, zz)
        l0 = g.ey * zz - zy; l1 = zx - g.ex * zz; l2 = g.ex * zy - g.ey * zx;
        clamp = 0.f;
    }
    float d1 = sdiv(l1, clamp), d0 = sdiv(l0, clamp);
    float by1 = -(c.xmin * l0 + l2) / d1;
    float by2 = -(c.xmax * l0 + l2) / d1;
    float bx0 = -(c.ymin * l1 + l2) / d0;
    float bx3 = -(c.ymax * l1 + l2) / d0;
    bool ok0 = (bx0 >= c.xmin + c.eps) && (bx0 < c.xmax - c.eps);
    bool ok1 = (by1 > c.ymin + c.eps) && (by1 <= c.ymax - c.eps);
    bool ok2 = (by2 >= c.ymin + c.eps) && (by2 < c.ymax - c.eps);
    bool ok3 = (bx3 > c.xmin + c.eps) && (bx3 <= c.xmax - c.eps);
    int n = (int)ok0 + (int)ok1 + (int)ok2 + (int)ok3;
    if (n < 2) { sx = ex = c.xmin - kFar; sy = ey = c.ymin - kFar; return; }
    // first two valid candidates in the order (y=ymin, x=xmin, x=xmax, y=ymax)
    bool have = false;
    sx = sy = ex = ey = 0.f;
    if (ok0) { sx = bx0; sy = c.ymin; have = true; }
    if (ok1) { if (!have) { sx = c.xmin; sy = by1; have = true; } else { ex = c.xmin; ey = by1; return; } }
    if (ok2) { if (!have) { sx = c.xmax; sy = by2; have = true; } else { ex = c.xmax; ey = by2; return; } }
    ex = bx3; ey = c.ymax;
}

// image coordinate of sample k -> normalised grid_sample coordinate (:405-415, multiview.py:25-37,159-163)
// Evaluated with host-precomputed reciprocals (a couple of ulp from the reference's division chain,
// i.e. ~1e-6 feature px; the emitted sample_locs are exactly what the kernels sample).
__device__ __forceinline__ float img2grid_x(float v, const GeomCfg &c) { return fmaf(fmaf(v, c.inv_rds, c.off_ds), c.gsx, c.gox); }
__device__ __forceinline__ float img2grid_y(float v, const GeomCfg &c) { return fmaf(fmaf(v, c.inv_rds, c.off_ds), c.gsy, c.goy); }

// normalised grid coordinate -> source feature-pixel coordinate (ATen grid_sampler unnormalize)
// (explicit intrinsics: the union-marking code and the sampling code must produce bit-identical pixel coordinates, so
// no step may be left to the compiler's FMA contraction)
__device__ __forceinline__ float grid2pix(float g, int size, int align) {
    const float g1 = __fadd_rn(g, 1.f);
    return align ? __fmul_rn(__fmul_rn(g1, 0.5f), (float)(size - 1)) : __fmul_rn(__fmaf_rn(g1, (float)size, -1.f), 0.5f);
}
// sample at parameter t in [0,1] on the segment (sx,sy)-(ex,ey) (image coordinates) -> normalised grid coordinates
__device__ __forceinline__ float lerp_exact(float a, float b, float t) { return __fmaf_rn(__fsub_rn(b, a), t, a); }

// de_normalize (multiview.py:39-57): grid coordinate -> feature px as the reference reports corr_pos
__device__ __forceinline__ float grid2corr(float g, int size, int correct) {
    return correct ? (g + 1.f) * (float)(size - 1) * 0.5f : (g + 1.f) * (float)size * 0.5f - 0.5f;
}

struct Taps {            // bilinear footprint of one sample in the source map
    int x0, y0;          // north-west tap (may be out of bounds)
    float w[4];          // nw, ne, sw, se — already zero for out-of-bounds taps
    bool any;            // at least one tap in bounds
};

__device__ __forceinline__ Taps make_taps(float gx, float gy, int H, int W, int align) {
    Taps t;
    float ix = grid2pix(gx, W, align), iy = grid2pix(gy, H, align);
    float fx = floorf(ix), fy = floorf(iy);
    // clamp before the int conversion so far sentinels / NaN cannot overflow
    fx = fminf(fmaxf(fx, -2.f), (float)W);  fy = fminf(fmaxf(fy, -2.f), (float)H);
    float ax = ix - floorf(ix), ay = iy - floorf(iy);
    if (!(ix == ix) || !(iy == iy)) { ax = ay = 0.f; fx = fy = -2.f; }     // NaN location: all taps out
    t.x0 = (int)fx; t.y0 = (int)fy;
    bool xin0 = t.x0 >= 0 && t.x0 < W, xin1 = t.x0 + 1 >= 0 && t.x0 + 1 < W;
    bool yin0 = t.y0 >= 0 && t.y0 < H, yin1 = t.y0 + 1 >= 0 && t.y0 + 1 < H;
    t.w[0] = (xin0 && yin0) ? (1.f - ax) * (1.f - ay) : 0.f;
    t.w[1] = (xin1 && yin0) ? ax * (1.f - ay) : 0.f;
    t.w[2] = (xin0 && yin1) ? (1.f - ax) * ay : 0.f;
    t.w[3] = (xin1 && yin1) ? ax * ay : 0.f;
    t.any = (xin0 || xin1) && (yin0 || yin1);
    return t;
}

// Fixed-point scale of the deterministic backward's source-gradient sums for one pair: `word` holds the bits of M_max, the
// pair's bound on Σ_pixels |contribution| to any one element.  With M_max in [2^(e-1), 2^e) and HW <= 2^L, s = 61 - L - e keeps
// every sum below HW·M_max·2^s < 2^61, inside int64 with headroom for the fp32 rounding of the contributions.  Returns false
// (no scatter) for M_max = 0 and for a non-finite bound.
__device__ __forceinline__ bool det_scale(unsigned word, int HW, int &s) {
    const float m = __uint_as_float(word);
    if (!(m > 0.f && m <= 3.402823466e38f)) return false;
    int e;
    frexpf(m, &e);
    s = 61 - (32 - __clz(HW - 1)) - e;
    return true;
}

// The same for one view item of the views form's backward, into which `pairs` pairs of its frame scatter: `word` holds the largest
// of their bounds, so their sums stay below pairs·HW·M_max·2^s, and s is lowered by ceil(log2(pairs)) to keep that under 2^61.
// Only the frame's own pairs enter the scale, and one non-finite bound among them makes the item's sums NaN.
__device__ __forceinline__ bool det_item_scale(unsigned word, int HW, int pairs, int &s) {
    if (!det_scale(word, HW, s)) return false;
    s -= 32 - __clz(pairs - 1);
    return true;
}

// arg-max over the samples (DESIGN a6): the first maximum wins, like torch.argmax, so a candidate (v, k) replaces the best
// (bv, bk) so far when it is larger, or equal at a lower sample index.  Every merge of partial arg-maxes uses this rule.
// (A macro: as a function returning bool it leaves the kernels' branch structure, and so their machine code, different.)
#define EPI_FIRST_MAX_BEATS(v, k, bv, bk) ((v) > (bv) || ((v) == (bv) && (k) < (bk)))


// Programmatic dependent launch (the three launches of a forward are chained with
// cudaLaunchAttributeProgrammaticStreamSerialization): a kernel's CTAs may become resident and run their prologue
// (barrier init, tensor-map prefetch) while the previous kernel of the stream drains;
// pdl_wait() returns once that kernel has completed and its writes are visible.  Nothing the previous kernels
// wrote may be read, and nothing they read may be written, before pdl_wait().
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#endif

}  // namespace epi
