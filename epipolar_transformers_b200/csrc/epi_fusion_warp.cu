// epi_fusion_warp.cu — baseline fused kernel: one warp per reference pixel.
//
// Fuses, for ATTENTION='avg' / SIMILARITY='dot' / SOFTMAX_ENABLED:
//   grid2sample_locs   /root/reference/modeling/layers/epipolar.py:323-418  (per-pixel, registers)
//   F.grid_sample x2   :199,:210   (4 bilinear taps per sample from a channels-last source map)
//   epipolar_similarity :295-307   (dot, ==0 mask, scale, softmax — online over K)
//   argmax + de_normalize :237-242 ; weighted sum :243
// Each lane owns C/32 channels of the query, the running weighted sum stays in registers,
// the C-wide dot is a warp-shuffle butterfly, K is consumed with an online softmax.
// The CTA (8 warps) owns 32 consecutive reference pixels so that the query tile, the output
// tile and the attention tile move through shared memory with coalesced 128-byte rows.
#include "epi_kernels.cuh"

namespace epi {

constexpr int kWarpTilePix = 32;                 // reference pixels per CTA
constexpr int kWarpTileWarps = 8;
constexpr int kMaxKChunks = 8;                   // K <= 256

template <int VEC> struct VecT;
template <> struct VecT<1> { using T = float; };
template <> struct VecT<2> { using T = float2; };
template <> struct VecT<4> { using T = float4; };

template <int VEC>
__device__ __forceinline__ void ld_vec(const float *p, float *dst) {
    using T = typename VecT<VEC>::T;
    T v = __ldg(reinterpret_cast<const T *>(p));
    const float *f = reinterpret_cast<const float *>(&v);
#pragma unroll
    for (int i = 0; i < VEC; i++) dst[i] = f[i];
}

// VEC floats per lane per chunk, NV chunks: lane owns channels (j*32+lane)*VEC+v, C <= 32*VEC*NV.
template <int VEC, int NV>
__global__ void __launch_bounds__(kWarpTileWarps * 32)
epi_fusion_warp_kernel(const FusionArgs a, const ViewSources vs) {
    extern __shared__ float smem[];
    const int C = a.C, K = a.geom.K, H = a.geom.H, W = a.geom.W, HW = H * W;
    const int tiles_per_item = (HW + kWarpTilePix - 1) / kWarpTilePix;
    const int n = blockIdx.x / tiles_per_item;
    const int p0 = (blockIdx.x % tiles_per_item) * kWarpTilePix;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int npix = min(kWarpTilePix, HW - p0);

    float *q_tile = smem;                                    // [C][33]  query in, fused feature out
    float *a_tile = smem + (size_t)C * 33;                   // [K][33]  attention weights
    __shared__ PairGeom s_geom;

    const PairItems it = pair_items(n, a.n_ref, a.n_views, vs);  // the pair's query and source items
    const int nr = it.q;
    if (tid == 0 && a.locs_in == nullptr) pair_geom_from_krt(a.P_ref + 12 * nr, a.P_src + 12 * it.s, s_geom);

    // ---- stage the query tile: coalesced along whichever of (pixel, channel) is contiguous ----
    {
        const float *base = a.feat_ref + (int64_t)nr * a.ref_stride[0];
        const int64_t sc = a.ref_stride[1], sh = a.ref_stride[2], sw = a.ref_stride[3];
        if (sc != 1) {
            for (int idx = tid; idx < C * kWarpTilePix; idx += blockDim.x) {
                int pp = idx & 31, c = idx >> 5, p = p0 + pp;
                float v = 0.f;
                if (pp < npix) v = __ldg(base + c * sc + (p / W) * sh + (p % W) * sw);
                q_tile[c * 33 + pp] = v;
            }
        } else {
            for (int idx = tid; idx < C * kWarpTilePix; idx += blockDim.x) {
                int c = idx % C, pp = idx / C, p = p0 + pp;
                float v = 0.f;
                if (pp < npix) v = __ldg(base + c + (p / W) * sh + (p % W) * sw);
                q_tile[c * 33 + pp] = v;
            }
        }
    }
    __syncthreads();

    const PairGeom g = s_geom;
    const GeomCfg gc = a.geom;
    const float *src = a.src_nhwc + (size_t)it.s * HW * C;
    // exp(x*scale - m) as exp2(x*scale*log2e - m*log2e)
    const float sl2 = a.softmax_scale * 1.4426950408889634f;

    for (int pi = 0; pi < kWarpTilePix / kWarpTileWarps; pi++) {
        const int pp = warp * (kWarpTilePix / kWarpTileWarps) + pi;
        if (pp >= npix) break;                       // warp-uniform
        const int p = p0 + pp, py_i = p / W, px_i = p % W;

        float q[NV * VEC], acc[NV * VEC];
#pragma unroll
        for (int j = 0; j < NV; j++)
#pragma unroll
            for (int v = 0; v < VEC; v++) {
                int c = (j * 32 + lane) * VEC + v;
                q[j * VEC + v] = c < C ? q_tile[c * 33 + pp] : 0.f;
                acc[j * VEC + v] = 0.f;
            }

        float sx = 0.f, sy = 0.f, ex = 0.f, ey = 0.f;
        if (a.locs_in == nullptr)
            line_endpoints(g, gc, pix2coord(px_i, gc.ds, gc.r), pix2coord(py_i, gc.ds, gc.r), sx, sy, ex, ey);

        float m_run = -INFINITY, l_run = 0.f;       // running max (log2 domain) and sum
        float my_sim[kMaxKChunks];                  // lane holds the logit of sample k = j*32+lane
        float my_gx[kMaxKChunks], my_gy[kMaxKChunks];
#pragma unroll
        for (int j = 0; j < kMaxKChunks; j++) { my_sim[j] = -INFINITY; my_gx[j] = 0.f; my_gy[j] = 0.f; }

#pragma unroll
        for (int j = 0; j < kMaxKChunks; j++) {
            if (j * 32 >= K) break;
            // each lane computes the location of "its" sample of this chunk, then broadcasts
            {
                int k = j * 32 + lane;
                float gx = 0.f, gy = 0.f;
                if (k < K) {
                    if (a.locs_in) {
                        const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)k * a.N + n) * HW + p);
                        gx = l.x; gy = l.y;
                    } else {
                        float t = (float)k / (float)(K - 1);
                        gx = img2grid_x(sx + (ex - sx) * t, gc);
                        gy = img2grid_y(sy + (ey - sy) * t, gc);
                    }
                    if (a.locs_out) reinterpret_cast<float2 *>(a.locs_out)[((size_t)k * a.N + n) * HW + p] = make_float2(gx, gy);
                }
                my_gx[j] = gx; my_gy[j] = gy;
            }
            const int kend = min(32, K - j * 32);
            for (int kk = 0; kk < kend; kk++) {
                const float gx = __shfl_sync(0xffffffffu, my_gx[j], kk);
                const float gy = __shfl_sync(0xffffffffu, my_gy[j], kk);
                const Taps t = make_taps(gx, gy, H, W, gc.align);
                float s[NV * VEC];
#pragma unroll
                for (int i = 0; i < NV * VEC; i++) s[i] = 0.f;
                float part = 0.f;
                if (t.any) {
#pragma unroll
                    for (int tap = 0; tap < 4; tap++) {
                        const float w = t.w[tap];
                        if (w != 0.f) {                                     // warp-uniform
                            const int xx = t.x0 + (tap & 1), yy = t.y0 + (tap >> 1);
                            const float *row = src + ((size_t)yy * W + xx) * C;
#pragma unroll
                            for (int jj = 0; jj < NV; jj++) {
                                const int c0 = (jj * 32 + lane) * VEC;
                                if (c0 < C) {
                                    float f[VEC];
                                    ld_vec<VEC>(row + c0, f);
#pragma unroll
                                    for (int v = 0; v < VEC; v++) s[jj * VEC + v] = fmaf(w, f[v], s[jj * VEC + v]);
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int i = 0; i < NV * VEC; i++) part = fmaf(s[i], q[i], part);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
                float sim = part;
                if (sim == 0.f) sim = kMasked;                              // epipolar.py:298
                const float x = sim * sl2;                                  // :306 (log2 domain)
                if (lane == kk) my_sim[j] = x;
                const float m_new = fmaxf(m_run, x);
                const float corr = exp2f(m_run - m_new);                    // 0 on the first sample
                const float pk = exp2f(x - m_new);
                l_run = l_run * corr + pk;
                m_run = m_new;
#pragma unroll
                for (int i = 0; i < NV * VEC; i++) acc[i] = fmaf(acc[i], corr, pk * s[i]);
            }
        }

        // ---- finalise: softmax weights, arg-max, normalised weighted sum ----
        const float inv_l = 1.f / l_run;
        float best_v = -1.f, best_gx = 0.f, best_gy = 0.f;
        int best_k = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < kMaxKChunks; j++) {
            if (j * 32 >= K) break;
            const int k = j * 32 + lane;
            if (k < K) {
                const float w = exp2f(my_sim[j] - m_run) * inv_l;
                if (a.attn) a_tile[k * 33 + pp] = w;
                if (w > best_v) { best_v = w; best_k = k; best_gx = my_gx[j]; best_gy = my_gy[j]; }
            }
        }
        if (a.corr_pos) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                float ov = __shfl_xor_sync(0xffffffffu, best_v, o);
                int ok = __shfl_xor_sync(0xffffffffu, best_k, o);
                float ogx = __shfl_xor_sync(0xffffffffu, best_gx, o), ogy = __shfl_xor_sync(0xffffffffu, best_gy, o);
                if (EPI_FIRST_MAX_BEATS(ov, ok, best_v, best_k)) { best_v = ov; best_k = ok; best_gx = ogx; best_gy = ogy; }
            }
            if (lane == 0)
                reinterpret_cast<float2 *>(a.corr_pos)[(size_t)n * HW + p] =
                    make_float2(grid2corr(best_gx, W, gc.correct), grid2corr(best_gy, H, gc.correct));
        }
#pragma unroll
        for (int j = 0; j < NV; j++)
#pragma unroll
            for (int v = 0; v < VEC; v++) {
                int c = (j * 32 + lane) * VEC + v;
                if (c < C) q_tile[c * 33 + pp] = acc[j * VEC + v] * inv_l;   // same column this warp read q from
            }
    }
    __syncthreads();

    // ---- write the fused tile (+ optional reference residual) and the attention tile ----
    {
        float *obase = a.out + (int64_t)n * a.out_stride[0];
        const int64_t sc = a.out_stride[1], sh = a.out_stride[2], sw = a.out_stride[3];
        const float *rbase = a.feat_ref + (int64_t)nr * a.ref_stride[0];
        if (sc != 1) {
            for (int idx = tid; idx < C * kWarpTilePix; idx += blockDim.x) {
                int pp = idx & 31, c = idx >> 5, p = p0 + pp;
                if (pp < npix) {
                    float v = q_tile[c * 33 + pp];
                    if (a.add_ref) v += __ldg(rbase + c * a.ref_stride[1] + (p / W) * a.ref_stride[2] + (p % W) * a.ref_stride[3]);
                    obase[c * sc + (p / W) * sh + (p % W) * sw] = v;
                }
            }
        } else {
            for (int idx = tid; idx < C * kWarpTilePix; idx += blockDim.x) {
                int c = idx % C, pp = idx / C, p = p0 + pp;
                if (pp < npix) {
                    float v = q_tile[c * 33 + pp];
                    if (a.add_ref) v += __ldg(rbase + c * a.ref_stride[1] + (p / W) * a.ref_stride[2] + (p % W) * a.ref_stride[3]);
                    obase[c + (p / W) * sh + (p % W) * sw] = v;
                }
            }
        }
        if (a.attn) {
            float *ab = a.attn + (size_t)n * K * HW;
            for (int idx = tid; idx < K * kWarpTilePix; idx += blockDim.x) {
                int pp = idx & 31, k = idx >> 5;
                if (pp < npix) ab[(size_t)k * HW + p0 + pp] = a_tile[k * 33 + pp];
            }
        }
    }
}

template <int VEC, int NV>
static cudaError_t launch_warp_t(const FusionArgs &a, const ViewSources &vs, cudaStream_t st) {
    const int HW = a.geom.H * a.geom.W;
    const int tiles = (HW + kWarpTilePix - 1) / kWarpTilePix;
    const size_t smem = ((size_t)a.C * 33 + (size_t)a.geom.K * 33) * sizeof(float);
    auto kern = epi_fusion_warp_kernel<VEC, NV>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<a.N * tiles, kWarpTileWarps * 32, smem, st>>>(a, vs);
    return cudaGetLastError();
}

cudaError_t launch_fusion_warp(const FusionArgs &a, const ViewSources &vs, cudaStream_t st) {
    const int C = a.C;
    if (C % 4 == 0 && C <= 128) return launch_warp_t<4, 1>(a, vs, st);
    if (C % 4 == 0 && C <= 256) return launch_warp_t<4, 2>(a, vs, st);
    if (C % 4 == 0 && C <= 512) return launch_warp_t<4, 4>(a, vs, st);
    if (C % 4 == 0 && C <= 1024) return launch_warp_t<4, 8>(a, vs, st);
    if (C <= 32) return launch_warp_t<1, 1>(a, vs, st);
    if (C <= 128) return launch_warp_t<1, 4>(a, vs, st);
    if (C <= 512) return launch_warp_t<1, 16>(a, vs, st);
    return cudaErrorInvalidValue;
}

}  // namespace epi
