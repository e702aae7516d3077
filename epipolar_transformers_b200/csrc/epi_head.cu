// epi_head.cu — the heat-map epilogue: the pose head's 1×1 conv applied to the fused feature (epi_fusion_heatmaps_f32), and
// the fold of z / BN and the head into its weights (epi_fold_head_f32).
//   heat = A·X + B·R + b    per pixel, X the pre-z fused feature, R the caller's residual (feat_ref of the pair's query item)
//   A = Wh·(Wf + z_res·I),  B = Wh,  b = Wh·bf + bh                        (/root/reference/modeling/backbones/resnet.py:388,421)
#include "epi_kernels.cuh"

namespace epi {

// ------------------------------------------------------------------------------------------
// Fold: one thread per (j, c) of A and one warp per j of b, sums in fp64, each rounded once to fp32.  Wf null: A = Wh, b = bh.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) fold_head_kernel(const float *__restrict__ Wh, const float *__restrict__ bh,
                                                        const float *__restrict__ Wf, const float *__restrict__ bf, int z_res, int C,
                                                        float *__restrict__ A, float *__restrict__ b) {
    const int j = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    const float *wh = Wh + (size_t)j * C;
    if (c < C) {
        double s = 0.0;
        if (Wf) {
            for (int o = 0; o < C; o++) s = fma((double)__ldg(wh + o), (double)__ldg(Wf + (size_t)o * C + c), s);
            if (z_res) s += (double)__ldg(wh + c);
        } else {
            s = __ldg(wh + c);
        }
        A[(size_t)j * C + c] = (float)s;
    }
    if (blockIdx.x == 0 && threadIdx.x < 32) {
        double s = 0.0;
        if (Wf && bf)
            for (int o = threadIdx.x; o < C; o += 32) s = fma((double)__ldg(wh + o), (double)__ldg(bf + o), s);
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);      // fixed tree: the same bits every run
        if (threadIdx.x == 0) b[j] = (float)(s + (bh ? (double)__ldg(bh + j) : 0.0));
    }
}

cudaError_t launch_fold_head(const float *Wh, const float *bh, const float *Wf, const float *bf, int z_res, int J, int C, float *A,
                             float *b, cudaStream_t st) {
    fold_head_kernel<<<dim3((C + 127) / 128, J), 128, 0, st>>>(Wh, bh, Wf, bf, z_res, C, A, b);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// Head kernel: per CTA (256 threads) one pair and kHeadPx pixels; warp w computes joints 4·jc .. 4·jc + 3 for jc = w, w + 8
// (< ceil(J/4)) on two adjacent pixels per lane.  Channels arrive in chunks of kHeadKc through shared memory: X from the fused
// kernel's pixel-major plane [N,HW,C] (a warp reads one pixel's channels), R from the caller's map in its layout and type (along
// pixels for NCHW items, along channels otherwise), A and B transposed to [c][joint].  Each thread loads its share of the next
// chunk into registers while the CTA multiplies the current one, so the loads of one chunk overlap the products of the other.
// Every heat element is the fp32 chain
//   b[j], + A[j,0]·X[0], + B[j,0]·R[0], + A[j,1]·X[1], ...        (fmaf, c increasing)
// whatever the tile, the pair's position in the batch and the form of the call; TO rounds it once.
// ------------------------------------------------------------------------------------------
constexpr int kHeadPx = 64, kHeadKc = 32, kHeadJ = 64, kHeadXs = kHeadPx + 2;     // Xs / Rs rows: even (float2 reads), 2-way writes
constexpr int kHeadThreads = 256, kHeadLd = kHeadKc * kHeadPx / kHeadThreads;      // elements per thread and array per chunk
static_assert(kHeadKc * kHeadJ / kHeadThreads == kHeadLd, "A / B chunks load like X / R");

template <typename TO, typename TR, bool RES>
__global__ void __launch_bounds__(kHeadThreads) head_kernel(const HeadArgs h, const ViewSources vs) {
    __shared__ __align__(16) float Xs[kHeadKc][kHeadXs];
    __shared__ __align__(16) float Rs[RES ? kHeadKc : 1][kHeadXs];
    __shared__ __align__(16) float As[kHeadKc][kHeadJ];
    __shared__ __align__(16) float Bs[RES ? kHeadKc : 1][kHeadJ];
    const int n = blockIdx.z, p0 = blockIdx.x * kHeadPx, HW = h.HW, C = h.C, J = h.J;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int JC = (J + 3) / 4;                                // joint chunks (joints padded to them with zero weights)
    const float *X = h.x + (size_t)n * HW * C;
    const TR *R = RES ? static_cast<const TR *>(h.ref) + (int64_t)pair_items(n, h.n_ref, h.n_views, vs).q * h.ref_stride[0] : nullptr;
    const bool r_px = h.ref_stride[3] == 1 && h.ref_stride[2] == h.W;     // R's pixels contiguous (NCHW item)
    // load k of a chunk: X (and R along channels) element (pixel t/32 + 8k, channel t%32); R along pixels and A / B element
    // (pixel or joint t%64, channel t/64 + 4k)
    const int px_r = p0 + t % 64;
    const int64_t roff = (int64_t)(px_r / h.W) * h.ref_stride[2] + (int64_t)(px_r % h.W) * h.ref_stride[3];
    float xr[kHeadLd], rr[kHeadLd], ar[kHeadLd], br[kHeadLd];
    auto load = [&](int c0) {
#pragma unroll
        for (int k = 0; k < kHeadLd; k++) {
            const int p = p0 + t / 32 + 8 * k, c = c0 + t % 32;
            xr[k] = p < HW && c < C ? __ldg(X + (size_t)p * C + c) : 0.f;
            const int cr = c0 + t / 64 + 4 * k, j = t % 64;
            ar[k] = j < J && cr < C ? __ldg(h.A + (size_t)j * C + cr) : 0.f;
            if (RES) {
                br[k] = j < J && cr < C ? __ldg(h.B + (size_t)j * C + cr) : 0.f;
                if (r_px) rr[k] = px_r < HW && cr < C ? to_f32(__ldg(R + (int64_t)cr * h.ref_stride[1] + roff)) : 0.f;
                else rr[k] = p < HW && c < C ? to_f32(__ldg(R + (int64_t)c * h.ref_stride[1] + (int64_t)(p / h.W) * h.ref_stride[2] +
                                                            (int64_t)(p % h.W) * h.ref_stride[3])) : 0.f;
            }
        }
    };

    float acc[2][4][2];
#pragma unroll
    for (int s = 0; s < 2; s++)
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int j = 4 * (warp + 8 * s) + u;
            const float bj = j < J ? __ldg(h.b + j) : 0.f;
            acc[s][u][0] = acc[s][u][1] = bj;
        }

    load(0);
    for (int c0 = 0; c0 < C; c0 += kHeadKc) {
        __syncthreads();                                           // the previous chunk's products are done
#pragma unroll
        for (int k = 0; k < kHeadLd; k++) {
            Xs[t % 32][t / 32 + 8 * k] = xr[k];
            As[t / 64 + 4 * k][t % 64] = ar[k];
            if (RES) {
                Bs[t / 64 + 4 * k][t % 64] = br[k];
                if (r_px) Rs[t / 64 + 4 * k][t % 64] = rr[k];
                else Rs[t % 32][t / 32 + 8 * k] = rr[k];
            }
        }
        __syncthreads();
        if (c0 + kHeadKc < C) load(c0 + kHeadKc);                  // in flight during the products below
        const int kc = C - c0 < kHeadKc ? C - c0 : kHeadKc;
        for (int cl = 0; cl < kc; cl++) {
            const float2 x = *reinterpret_cast<const float2 *>(&Xs[cl][2 * lane]);
            float2 r = make_float2(0.f, 0.f);
            if (RES) r = *reinterpret_cast<const float2 *>(&Rs[cl][2 * lane]);
#pragma unroll
            for (int s = 0; s < 2; s++) {
                const int jc = warp + 8 * s;
                if (jc >= JC) break;                               // warp-uniform
                const float4 a = *reinterpret_cast<const float4 *>(&As[cl][4 * jc]);
                const float av[4] = {a.x, a.y, a.z, a.w};
                float bv[4] = {0.f, 0.f, 0.f, 0.f};
                if (RES) {
                    const float4 bb = *reinterpret_cast<const float4 *>(&Bs[cl][4 * jc]);
                    bv[0] = bb.x; bv[1] = bb.y; bv[2] = bb.z; bv[3] = bb.w;
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    acc[s][u][0] = fmaf(av[u], x.x, acc[s][u][0]);
                    acc[s][u][1] = fmaf(av[u], x.y, acc[s][u][1]);
                    if (RES) {
                        acc[s][u][0] = fmaf(bv[u], r.x, acc[s][u][0]);
                        acc[s][u][1] = fmaf(bv[u], r.y, acc[s][u][1]);
                    }
                }
            }
        }
    }

    TO *heat = static_cast<TO *>(h.heat) + (int64_t)n * h.heat_stride[0];
#pragma unroll
    for (int s = 0; s < 2; s++)
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int j = 4 * (warp + 8 * s) + u;
            if (j >= J) continue;
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int p = p0 + 2 * lane + e;
                if (p < HW)
                    heat[(int64_t)j * h.heat_stride[1] + (int64_t)(p / h.W) * h.heat_stride[2] + (int64_t)(p % h.W) * h.heat_stride[3]] =
                        from_f32<TO>(acc[s][u][e]);
            }
        }
}

template <typename TO, typename TR, bool RES>
static void head_t(const HeadArgs &h, const ViewSources &vs, dim3 grid, cudaStream_t st) {
    head_kernel<TO, TR, RES><<<grid, kHeadThreads, 0, st>>>(h, vs);
}

// without a residual TR is float and never read
template <typename TO>
static void head_out(const HeadArgs &h, const ViewSources &vs, dim3 grid, cudaStream_t st) {
    if (!h.ref) head_t<TO, float, false>(h, vs, grid, st);
    else if (h.ref_dtype == kBF16) head_t<TO, __nv_bfloat16, true>(h, vs, grid, st);
    else if (h.ref_dtype == kF16) head_t<TO, __half, true>(h, vs, grid, st);
    else head_t<TO, float, true>(h, vs, grid, st);
}

cudaError_t launch_head(const HeadArgs &h, const ViewSources &vs, int heat_dtype, cudaStream_t st) {
    const dim3 grid((h.HW + kHeadPx - 1) / kHeadPx, 1, h.N);
    if (heat_dtype == kBF16) head_out<__nv_bfloat16>(h, vs, grid, st);
    else if (heat_dtype == kF16) head_out<__half>(h, vs, grid, st);
    else head_out<float>(h, vs, grid, st);
    return cudaGetLastError();
}

}  // namespace epi
