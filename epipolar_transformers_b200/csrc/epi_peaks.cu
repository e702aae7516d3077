// epi_peaks.cu — find_tensor_peak_batch on the GPU (SURVEY.md 8f rank 3): the step right after the fusion layer's 1x1 head.
//
// Restates /root/reference/modeling/backbones/basic_batch.py:17-63, which the caller runs once per batch item in a Python
// loop (modeling/backbones/resnet.py:423-428), for a whole [B, J, H, W] stack of heat-maps in ONE launch, one warp per
// (item, joint):
//   score, index = max over the flattened map: the first NaN if there is one (torch.max), else the first maximum (:24)
//   index_w = index % W ; index_h = index / W   — TRUE division under torch >= 1.5 (the semantics of the torch
//       installed here, which is what the golden vectors freeze), integer division under the torch < 1.4 the repo
//       names in its README: `int_div` selects it                                                     (:25-26)
//   (2R+1)^2 bilinear samples (zero padding, align_corners=False) of the window [index -+ radius] laid out by
//   F.affine_grid(align_corners=False), R = int(radius + 0.5); values <= threshold -> 0, NaN kept          (:30-50)
//   x = Σ sub·X / (Σ sub + eps) + index_w, y likewise with Y ; X, Y = arange(-radius, radius + 1e-4, radius / R)  (:52-57)
//   pix2coord: v·downsample + downsample/2 − 0.5                                                         (:59-61)
#include "epi_kernels.cuh"

namespace epi {

// One warp: the peak of heat-map m [H,W] -> image coordinates (x, y) and score, identical on every lane.  Both kernels below
// call this one function, so a best-source result is bit for bit the single-source result of the winning source.
__device__ __forceinline__ void peak_of(const float *__restrict__ m, int H, int W, float radius, float downsample, float threshold,
                                        int int_div, float &out_x, float &out_y, float &out_score) {
    const int lane = threadIdx.x & 31;
    const int HW = H * W;
    // ---- arg-max as torch.max computes it: NaN beats any number and the lowest index wins among NaNs; otherwise the
    // first maximum.  A map of -inf alone records nothing and takes index 0, torch.max's first maximum. ----
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = lane; i < HW; i += 32) {                                // increasing i: the first NaN / maximum stays
        const float v = __ldg(m + i);
        if (v > best || (v != v && best == best)) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        const bool onan = ov != ov, bnan = best != best;
        if (onan ? (!bnan || oi < bi) : (!bnan && (ov > best || (ov == best && oi < bi)))) { best = ov; bi = oi; }
    }
    if (bi == 0x7fffffff) bi = 0;
    const float index_w = (float)(bi % W);
    const float index_h = int_div ? (float)(bi / W) : (float)bi / (float)W;
    // ---- window in normalised coordinates (normalize(x, L) = -1 + 2x/(L-1)) and its affine grid ----
    const float b0 = -1.f + 2.f * (index_w - radius) / (float)(W - 1), b2 = -1.f + 2.f * (index_w + radius) / (float)(W - 1);
    const float b1 = -1.f + 2.f * (index_h - radius) / (float)(H - 1), b3 = -1.f + 2.f * (index_h + radius) / (float)(H - 1);
    const float ax = (b2 - b0) * 0.5f, cx = (b2 + b0) * 0.5f, ay = (b3 - b1) * 0.5f, cy = (b3 + b1) * 0.5f;
    const int R = (int)(radius + 0.5f), S = 2 * R + 1;
    const float step = radius * 1.0f / (float)R;
    float sum = 0.f, sx = 0.f, sy = 0.f;
    for (int e = lane; e < S * S; e += 32) {
        const int iy = e / S, ix = e % S;
        // affine_grid base coordinates, align_corners=False: (2i + 1)/S - 1
        const float gx = ax * ((2.f * ix + 1.f) / (float)S - 1.f) + cx, gy = ay * ((2.f * iy + 1.f) / (float)S - 1.f) + cy;
        // grid_sample, bilinear, zeros, align_corners=False
        const float px = ((gx + 1.f) * (float)W - 1.f) * 0.5f, py = ((gy + 1.f) * (float)H - 1.f) * 0.5f;
        const float fx = floorf(px), fy = floorf(py);
        const float wx = px - fx, wy = py - fy;
        float v = 0.f;
        if (fx >= -1.f && fx < (float)W && fy >= -1.f && fy < (float)H) {
            const int x0 = (int)fx, y0 = (int)fy;
            const bool xa = x0 >= 0, xb = x0 + 1 < W, ya = y0 >= 0, yb = y0 + 1 < H;
            if (xa && ya) v += (1.f - wx) * (1.f - wy) * __ldg(m + y0 * W + x0);
            if (xb && ya) v += wx * (1.f - wy) * __ldg(m + y0 * W + x0 + 1);
            if (xa && yb) v += (1.f - wx) * wy * __ldg(m + (y0 + 1) * W + x0);
            if (xb && yb) v += wx * wy * __ldg(m + (y0 + 1) * W + x0 + 1);
        }
        if (v <= threshold) v = 0.f;                                     // F.threshold(sub, threshold, 0): NaN is kept
        sum += v;
        sx = fmaf(v, -radius + step * (float)ix, sx);
        sy = fmaf(v, -radius + step * (float)iy, sy);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sx += __shfl_xor_sync(0xffffffffu, sx, o);
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
    }
    const float den = sum + 2.220446049250313e-16f;                      // np.finfo(float).eps
    const float x = sx / den + index_w, y = sy / den + index_h;
    out_x = x * downsample + downsample * 0.5f - 0.5f;
    out_y = y * downsample + downsample * 0.5f - 0.5f;
    out_score = best;
}

__global__ void __launch_bounds__(128) epi_peaks_kernel(const float *__restrict__ heat, float *__restrict__ locs,
                                                        float *__restrict__ scores, int BJ, int H, int W, float radius,
                                                        float downsample, float threshold, int int_div) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= BJ) return;
    float x, y, score;
    peak_of(heat + (size_t)warp * H * W, H, W, radius, downsample, threshold, int_div, x, y, score);
    if (lane == 0) {
        locs[2 * warp] = x;
        locs[2 * warp + 1] = y;
        scores[warp] = score;
    }
}

// Multi-view test (modeling/model.py:229-234): heat [S,B,J,H,W]; warp (b, j) runs the single-source peak of every source and
// keeps the one torch.max over the sources picks: the first NaN score if there is one, else the first highest score (strict
// `>`, so a tie keeps the earlier source).
__global__ void __launch_bounds__(128) epi_peaks_best_kernel(const float *__restrict__ heat, float *__restrict__ locs,
                                                             float *__restrict__ scores, int *__restrict__ src_index, int S, int BJ,
                                                             int H, int W, float radius, float downsample, float threshold,
                                                             int int_div) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= BJ) return;
    float bx = 0.f, by = 0.f, bs = 0.f;
    int bsrc = 0;
    for (int s = 0; s < S; s++) {
        float x, y, score;
        peak_of(heat + ((size_t)s * BJ + warp) * H * W, H, W, radius, downsample, threshold, int_div, x, y, score);
        if (s == 0 || (score != score ? bs == bs : score > bs)) { bx = x; by = y; bs = score; bsrc = s; }
    }
    if (lane == 0) {
        locs[2 * warp] = bx;
        locs[2 * warp + 1] = by;
        scores[warp] = bs;
        if (src_index) src_index[warp] = bsrc;
    }
}

cudaError_t launch_peaks_best(const float *heat, float *locs, float *scores, int *src_index, int S, int B, int J, int H, int W,
                              float radius, float downsample, float threshold, int int_div, cudaStream_t st) {
    const int BJ = B * J;
    epi_peaks_best_kernel<<<(BJ + 3) / 4, 128, 0, st>>>(heat, locs, scores, src_index, S, BJ, H, W, radius, downsample, threshold, int_div);
    return cudaGetLastError();
}

cudaError_t launch_peaks(const float *heat, float *locs, float *scores, int B, int J, int H, int W, float radius, float downsample,
                         float threshold, int int_div, cudaStream_t st) {
    const int BJ = B * J;
    epi_peaks_kernel<<<(BJ + 3) / 4, 128, 0, st>>>(heat, locs, scores, BJ, H, W, radius, downsample, threshold, int_div);
    return cudaGetLastError();
}

}  // namespace epi
