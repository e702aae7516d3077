// epi_fusion_pipe.cu — the fused epipolar attention kernel (default): warp-specialised, mbarrier-pipelined,
// warpgroup MMA (wgmma).  One persistent CTA per SM, 24 warps:
//
//   warps  0-15  workers   four warpgroups: GEMM1 (wgmma, registers -> score table), 4-tap interpolation, ==0 mask,
//                          softmax over K, attn / corr_pos / sample_locs, β scatter, β -> bf16 (hi, lo) panels,
//                          GEMM2 (wgmma, registers -> table) and the epilogue table -> global
//   warps 16-19  setup     next work item: pixel list (sector order), epipolar line end points, union bitmap of the
//                          bilinear taps of the item's pixels, prefix ranks, row list for the gathers
//   warps 20-23  gather    16-byte cp.async (LDGSTS) of query rows and source-feature rows (bf16 hi/lo planes, pixel-major)
//                          into 128-byte-swizzled shared-memory panels; completion through cp.async.mbarrier.arrive
//
// Maths (identical to epi_fusion_tile.cu, restating /root/reference/modeling/layers/epipolar.py:199,210 grid_sample taps,
// :295-307 similarity / ==0 mask / scale / softmax, :237-243 arg-max + weighted sum, :323-418 geometry):
//   sim_k = Σ_t w_kt · (q · f[p_t])        out = Σ_p β_p · f[p],   β_p = Σ_{k,t→p} a_k w_kt
// over the UNION of source pixels touched by the item's ≤32 (or ≤64) epipolar lines (D ≤ 256 rows; items whose union is larger
// are split by the setup warps).  Operands are bf16 (hi, lo) pairs: hi·hi + hi·lo + lo·hi, fp32 accumulation in registers.
//
// Pipeline: the setup warps build item j+1 and the gather warps fill the feature ring (3 stages of 32 KB; 2 with 64-pixel items) for item j's GEMM2
// and item j+1's GEMM1 while the workers are in item j's softmax phase.  The workers' warpgroups issue the MMAs of a stage
// together (warpgroup wg owns 64 rows of the accumulator), wait for them and hand the stage back; the accumulators go from
// registers straight into the shared-memory table.  Everything between the roles is mbarrier producer/consumer hand-off.
#include <cstddef>

#include <cuda_bf16.h>

#include "epi_kernels.cuh"
#include "epi_umma.cuh"

namespace epi {
using namespace umma;

namespace pipe {
constexpr int PREC = 32;           // pixels per plan-cache record slot (the 32-pixel item's descriptor)
constexpr int CHUNK = 128;         // union rows per GEMM1 accumulator (MMA M)
constexpr int DMAX = 256;          // max union rows per item (two chunks)
constexpr int NWORK = 16;          // worker warps
constexpr int NT_WORK = NWORK * 32;
constexpr int W_SETUP = 16, W_GATHER = 20;
constexpr int NSETUP = 128;        // setup threads
constexpr int NGATHER = 128;       // gather threads
constexpr int NT_ALL = 768;
constexpr int MAXWORDS = 512;      // bitmap words: H*W <= 16384
constexpr int MAXKPL = 4;          // samples per lane: K <= 128
constexpr int NSTAGE_MAX = 3;
constexpr int NDESC = 4;
constexpr float FIX = 1073741824.0f;           // 2^30 fixed point for the β scatter (bit-reproducible)

constexpr uint32_t STAGE_BYTES = 32768;        // GEMM1: [plane][128 rows x 128 B]; GEMM2: [plane][2 panels][64 rows x 128 B]
constexpr uint32_t PLANE_BYTES = 16384;
constexpr uint32_t PANEL_B2 = 8192;            // stacked B panel: 64 rows x 128 B (rows 0-31 hi, 32-63 lo)
constexpr uint32_t TABLE_HALF = DMAX * 32 * 4; // one 32-pixel half of the table: [DMAX][32] fp32 / int32
// d-major score table T[rank][pixel]: 32 floats per row, the float4 column XOR-ed with rank % 8.  Lane <-> pixel accesses hit
// bank (pixel-derived) regardless of each lane's rank pattern; lane <-> rank accesses are conflict free too.
__device__ __forceinline__ int tix(int r, int i) { return r * 32 + ((((i >> 2) ^ r) & 7) << 2) + (i & 3); }

template <int P>                   // P = 32 or 64 reference pixels
struct ItemDesc;
template <>
struct ItemDesc<32> {              // one work item, written by the setup warps
    uint32_t bitmap[MAXWORDS];
    uint16_t prefix[MAXWORDS];
    uint16_t idx[DMAX];            // union rank -> source pixel (padded to a multiple of 16 with a valid row)
    float4 ends[32];               // line end points in image coordinates (fused geometry)
    uint32_t pix[32];              // y << 16 | x, 0xFFFFFFFF = no pixel
    int tile;                      // < 0: no more work
    int n, g0, gn, D;
    uint32_t epoch, claim_tag;     // plan cache: valid for the pair's epoch `epoch`, built for claim `claim_tag - 1` (+ bit 31: 64 pixels)
    int pad[1];
};
// A 64-pixel record spans the cache slots of two 32-pixel records.  It carries its tag where either slot keeps a 32-pixel
// record's tag: in its own bytes (tag32) for the first slot, and in one word written behind it for the second.  A 32-pixel
// record written over either slot replaces one of the two, and a 32-pixel reader of either slot finds a 64-pixel tag.
template <>
struct ItemDesc<64> {
    uint32_t bitmap[MAXWORDS];
    uint16_t prefix[MAXWORDS];
    uint16_t idx[DMAX];
    uint32_t pix[64];
    uint32_t gap[96];              // up to where a 32-pixel record keeps its header
    uint32_t tag32[8];             // [6]: the tag, at the first slot's 32-pixel tag
    float4 ends[64];
    int tile;
    int n, g0, gn, D;
    uint32_t epoch, claim_tag;
    int pad[1];
};
constexpr uint32_t REC_BYTES = (sizeof(ItemDesc<PREC>) + 127) / 128 * 128;     // one plan-cache record slot

// Shared memory of the kernel with P-pixel items.  32 pixels: 3 ring stages, 4 query panels, 4 β panels, a [DMAX][32] table.
// 64 pixels: 2 ring stages, two halves of 4 query panels, and a table of two [DMAX][32] halves that holds each half's scores,
// then its int32 β, then (in place) its β panels; the epilogue transposes [64][256] fp32 through all of it.
template <int P>
struct Layout {
    static constexpr int NSTAGE = P == 32 ? 3 : 2;
    static constexpr uint32_t DESC_BYTES = (sizeof(ItemDesc<P>) + 127) / 128 * 128;
    static constexpr uint32_t OFF_STAGE = 0;
    static constexpr uint32_t OFF_Q = NSTAGE * STAGE_BYTES;                         // P/32 halves of 4 stacked panels
    static constexpr uint32_t OFF_BETA = OFF_Q + P / 32 * 4 * PANEL_B2;             // 32 pixels: 4 stacked panels (256 d)
    static constexpr uint32_t OFF_TABLE = OFF_BETA + (P == 32 ? 4 * PANEL_B2 : 0);   // P/32 halves [DMAX][32]
    static constexpr uint32_t OFF_RED = OFF_TABLE + P / 32 * TABLE_HALF;            // softmax / arg-max split-reduction scratch [4][16][32]
    static constexpr uint32_t OFF_DESC = OFF_RED + 4 * NWORK * 32 * 4;
    static constexpr uint32_t OFF_CTRL = OFF_DESC + NDESC * DESC_BYTES;
};
static_assert(REC_BYTES == 4352, "the plan cache's size per record slot");
static_assert(Layout<64>::DESC_BYTES <= 2 * REC_BYTES, "a 64-pixel descriptor fits the record slots of its two 32-pixel tiles");
static_assert(offsetof(ItemDesc<64>, tag32) + 6 * 4 == offsetof(ItemDesc<32>, claim_tag), "the first slot's 32-pixel tag");
static_assert(sizeof(ItemDesc<64>) <= REC_BYTES + offsetof(ItemDesc<32>, claim_tag), "the second slot's 32-pixel tag lies behind the record");
// a cached 64-pixel record is whole when both of its slots still carry its tag where a 32-pixel record keeps one
__device__ __forceinline__ bool tags64_intact(const uint8_t *rec, uint32_t tag) {
    return reinterpret_cast<const ItemDesc<64> *>(rec)->tag32[6] == tag &&
           *reinterpret_cast<const uint32_t *>(rec + REC_BYTES + offsetof(ItemDesc<32>, claim_tag)) == tag;
}

// Maps above 16384 pixels (up to 256 rows x 1024 columns) do not fit a one-bit-per-pixel bitmap in the descriptor.  Their items
// re-use the same 3 KB (bitmap + prefix) as a ROW-WINDOWED bitmap: per source row a mask of the 32-pixel words the union touches,
// and only those words are stored, in (row, word) order — at most one word per union pixel, so WIN_WORDS = DMAX always suffices.
//   rank(x, y) = prefix[w] + popc(bitmap[w] & below(x % 32)),   w = wbase[y] + popc(rowmask[y] & below(x / 32))
constexpr int WIN_WORDS = 256, WIN_ROWS = 256, WIN_MAXW = 1024;
struct WinView { uint32_t *bitmap, *rowmask; uint16_t *prefix, *wbase; };
template <int P>
__device__ __forceinline__ WinView win_view(ItemDesc<P> &d) {
    uint8_t *b = reinterpret_cast<uint8_t *>(d.bitmap);
    return {reinterpret_cast<uint32_t *>(b), reinterpret_cast<uint32_t *>(b + 1024), reinterpret_cast<uint16_t *>(b + 2048), reinterpret_cast<uint16_t *>(b + 2560)};
}
static_assert(sizeof(uint32_t) * MAXWORDS + sizeof(uint16_t) * MAXWORDS >= 4 * WIN_WORDS + 4 * WIN_ROWS + 2 * WIN_WORDS + 2 * WIN_ROWS, "windowed view fits");

struct Ctrl {
    uint64_t desc_full[NDESC], desc_free[NDESC];
    uint64_t q_full, q_empty;
    uint64_t f_full[NSTAGE_MAX], f_empty[NSTAGE_MAX];
    int stack[16];
    int sp;
    int cur;                       // item being built: g0 | gn << 8
    int cur_tile;
    int cur_claim;                 // claim index of the item being built, -1 for a piece of a split tile
    int total;
    int done;
};
template <int P>
constexpr uint32_t smem_alloc() { return Layout<P>::OFF_CTRL + ((sizeof(Ctrl) + 127) / 128 * 128) + 1024; }   // + 1024-byte alignment slack
static_assert(smem_alloc<32>() <= 232448 - 2048 && smem_alloc<64>() <= 232448 - 2048, "keep head-room below the 227 KB opt-in limit");

__device__ __forceinline__ void named_bar(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// Bounded mbarrier wait: a protocol bug must never hang the GPU.  On timeout the error word is set and the whole CTA
// is torn down by __trap() (the launch fails with a sticky error instead of a hung box).
__device__ __forceinline__ void wait_n(uint64_t *bar, uint32_t n) {
    const uint32_t parity = n & 1u;
    for (uint32_t it = 0; !mbar_try_wait(bar, parity); ++it)
        if (it > (1u << 24)) __trap();
}

}  // namespace pipe

using namespace pipe;

#ifdef EPI_PIPE_TIMERS
__device__ unsigned long long g_pipe_timers[32];
__device__ long long g_pipe_trace[64 * 16];
__device__ unsigned long long g_pipe_cta[256 * 4];     // per CTA: globaltimer at entry, after the dependency wait, at exit; items processed
#define TR(item, ev) do { if (blockIdx.x == 0 && (item) < 64) g_pipe_trace[(item) * 16 + (ev)] = clock64(); } while (0)
#define PT_DECL long long pt_prev = clock64()
#define PT(slot) do { if (pt_on) { const long long t_ = clock64(); atomicAdd(&g_pipe_timers[slot], (unsigned long long)(t_ - pt_prev)); pt_prev = t_; } } while (0)
#else
#define PT_DECL do { } while (0)
#define TR(item, ev) do { } while (0)
#define PT(slot) do { } while (0)
#endif

// LO: the operands have a lo part (fp32 / fp16 maps).  bf16 maps are their own hi part: no lo planes are gathered, GEMM1 is
// the single product hi·hi and GEMM2 (whose β is fp32-derived) hi·β_hi + hi·β_lo.  The products that remain are issued in the
// same order as with LO, and the ones left out are exact zeros, so both forms accumulate the same sums.
//
// P: reference pixels per work item.  A 64-pixel item is two 32-pixel halves that share one tap union: every warpgroup multiplies
// on every ring stage (GEMM1: row half wg & 1 of the chunk against query half wg >> 1; GEMM2: channel block wg & 1 of the stage
// for pixel half wg >> 1), and the softmax phase runs once per half with the 32-pixel code.  The host picks 64 for maps of at
// most 64 pixels a side with C <= 256, whose 64-pixel unions stay within DMAX rows.
// vs: the source table of a table call, else empty (pair_items)
template <int KPL, bool LO, int P, typename... Tab>
__global__ void __launch_bounds__(NT_ALL, 1) epi_fusion_pipe_kernel(const FusionArgs a, const Tab... vs) {
    using Desc = ItemDesc<P>;
    using L = Layout<P>;
    constexpr int NSTAGE = L::NSTAGE;
    constexpr uint32_t DESC_BYTES = L::DESC_BYTES, OFF_STAGE = L::OFF_STAGE, OFF_Q = L::OFF_Q, OFF_BETA = L::OFF_BETA,
                       OFF_TABLE = L::OFF_TABLE, OFF_RED = L::OFF_RED, OFF_DESC = L::OFF_DESC, OFF_CTRL = L::OFF_CTRL;
    constexpr int NPH = P / 32;                     // pixel halves of an item
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    float *table = reinterpret_cast<float *>(smem + OFF_TABLE);
    Ctrl &ct = *reinterpret_cast<Ctrl *>(smem + OFF_CTRL);
    auto desc_at = [&](int j) -> Desc & { return *reinterpret_cast<Desc *>(smem + OFF_DESC + (uint32_t)(j % NDESC) * DESC_BYTES); };

    const int C = a.C, K = a.geom.K, H = a.geom.H, W = a.geom.W, HW = H * W;
    const int tiles_per_item = (HW + P - 1) / P;
    const int total_tiles = a.N * tiles_per_item;
    // tail balancing: the tiles of the last, partial round over the grid are handed out as half items (P/2 pixels).  How a tile
    // is split changes the union rows its pixels share, hence the order of the GEMM sums, so with several sources per reference
    // item (n_ref < N), or several view pairs (n_views), the split is the one a call with the n_ref pairs of a single source makes
    // on its own grid: every source gets, bit for bit, what a separate call gives it.  A 64-pixel half costs well over half an item (the union barely shrinks),
    // so 64-pixel items split the last round only when it is at most half full: the halves then still fit one round.
    const int grid1 = min(a.n_ref * tiles_per_item, (int)gridDim.x);
    const int tail_tiles = a.tile_counter ? (a.n_ref * tiles_per_item) % grid1 : 0;
    const int r_half = (P == 64 && 2 * tail_tiles > grid1) ? 0 : min(tiles_per_item, (tail_tiles + a.n_ref - 1) / a.n_ref);  // per pair
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nwords = (HW + 31) >> 5;
    const bool big = nwords > MAXWORDS;             // row-windowed union bitmap (see WinView)
    const int NH = (C + 127) >> 7;                  // channel halves of 128 (GEMM2 M)
    const int NP = (C + 63) >> 6;                   // 64-channel panels
    // C > 256 ("wide"): the query panels are loaded in two halves of four (GEMM1 accumulates over both), the fused-feature
    // accumulator takes all 256 columns of the O region (four channel halves, single-buffered) and the epilogue runs twice.
    const bool wide = P == 32 && C > 256;           // 64-pixel items run only at C <= 256
    const int NQH = wide ? 2 : 1;
    const GeomCfg gc = a.geom;
    constexpr int KW = 2 * KPL;                     // samples per worker warp (k = warp + 16 jj)

    // ---------------- one-time setup (overlaps the staging launch's tail: programmatic dependent launch) ----------------
    pdl_launch_dependents();
#ifdef EPI_PIPE_TIMERS
    if (tid == 0 && blockIdx.x < 256) { unsigned long long g; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g)); g_pipe_cta[blockIdx.x * 4] = g; }
#endif
    if (tid == 32) {
        for (int i = 0; i < NDESC; i++) { mbar_init(&ct.desc_full[i], 1); mbar_init(&ct.desc_free[i], 2); }
        mbar_init(&ct.q_full, NGATHER); mbar_init(&ct.q_empty, 1);
        for (int i = 0; i < NSTAGE; i++) { mbar_init(&ct.f_full[i], NGATHER); mbar_init(&ct.f_empty[i], 1); }
        ct.sp = 0; ct.done = 0;
        mbar_fence_init();
    }
    __syncthreads();
    pdl_wait();                                     // operand planes, pixel order, pair constants, counters: the staging launch
#ifdef EPI_PIPE_TIMERS
    if (tid == 0 && blockIdx.x < 256) { unsigned long long g; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g)); g_pipe_cta[blockIdx.x * 4 + 1] = g; }
#endif

    if (warp < NWORK) {
        // =====================================================================================================
        // WORKERS (16 warps).  lane <-> pixel of the item, warp <-> samples k = warp, warp+16, ...  The score table is
        // d-major, T[rank][pixel] with a 33-float row pitch: every access of a warp (32 pixels, nearly equal ranks) is
        // bank-conflict free, the K-wide softmax is a 16-way split reduction through shared memory.
        // =====================================================================================================
        const float sl2 = a.softmax_scale * 1.4426950408889634f;
        const int wg = warp >> 2, t128 = tid & 127;                      // warpgroup, thread within it
        const uint32_t sq = smem_u32(smem + OFF_Q), sb = smem_u32(smem + OFF_BETA);
        uint32_t qcount = 0, fcount = 0;
        float *red_max = reinterpret_cast<float *>(smem + OFF_RED);     // [16][32]
        float *red_sum = red_max + NWORK * 32;
        float *red_bv = red_sum + NWORK * 32;
        int *red_bk = reinterpret_cast<int *>(red_bv + NWORK * 32);
        float tkw[KW];                                                   // sample parameters of this warp
#pragma unroll
        for (int jj = 0; jj < KW; jj++) tkw[jj] = (float)(warp + NWORK * jj) / (float)(K - 1);

        // One feature stage of the ring: every worker waits for it, the warpgroups that own part of it issue their MMAs and wait
        // for them, then the stage goes back to the gather warps.
        auto consume_stage = [&]() -> uint32_t {
            const uint32_t s = fcount % NSTAGE;
            if (warp == 0) wait_n(&ct.f_full[s], fcount / NSTAGE);
            named_bar(1, NT_WORK);
            fence_proxy_async_smem();           // cp.async (generic proxy) writes -> wgmma (async proxy) reads
            return s;
        };
        auto release_stage = [&](uint32_t s) {
            named_bar(1, NT_WORK);              // the MMAs of every warpgroup on this stage have completed
            if (tid == 0) mbar_arrive(&ct.f_empty[s]);
            fcount++;
        };

        // GEMM2 Oᵀ = Fᵀ·βᵀ of item j, then its epilogue: fused feature -> table (as [pixel][channel]) -> global.
        // 32 pixels: warpgroup wg accumulates channels (wg >> 1) * 128 + (wg & 1) * 64 .. +63 of each 256-channel part (two parts
        // when C > 256).  64 pixels: warpgroup wg accumulates channels h * 128 + (wg & 1) * 64 .. +63 (o0: h = 0, o1: h = 1) of pixel
        // half wg >> 1, whose β panels are in its half of the table.
        auto epilogue = [&](int j) {
            const Desc &d = desc_at(j);
            float o0[16], o1[16];
#pragma unroll
            for (int e = 0; e < 16; e++) { o0[e] = 0.f; o1[e] = 0.f; }      // D == 0: all masked, zero vectors
            if (d.D > 0) {
                const int D16 = (d.D + 15) & ~15, nblk = (D16 + 63) >> 6;
                for (int blk = 0; blk < nblk; blk++)
                    for (int h = 0; h < NH; h++) {
                        const uint32_t s = consume_stage();
                        if (P == 64 || (h & 1) == (wg >> 1)) {
                            const uint32_t sa = smem_u32(smem + OFF_STAGE + s * STAGE_BYTES) + (uint32_t)(wg & 1) * 8192u;
                            const uint32_t sbw = P == 64 ? smem_u32(table) + (uint32_t)(wg >> 1) * TABLE_HALF : sb;
                            const int nk = min(4, (D16 - blk * 64) >> 4);
                            wg_fence();
                            for (int kk = 0; kk < nk; kk++) {
                                const uint64_t a_hi = make_smem_desc(sa + kk * 2048, 8192, 1024), a_lo = desc_add(a_hi, PLANE_BYTES);
                                const uint64_t b = make_smem_desc(sbw + blk * PANEL_B2 + kk * 32, 16, 1024), b_lo = desc_add(b, 4096);
                                if (P == 64 ? h != 0 : (h >> 1) != 0) { wgmma_m64n32<1>(o1, a_hi, b); wgmma_m64n32<1>(o1, a_hi, b_lo); if (LO) wgmma_m64n32<1>(o1, a_lo, b); }
                                else        { wgmma_m64n32<1>(o0, a_hi, b); wgmma_m64n32<1>(o0, a_hi, b_lo); if (LO) wgmma_m64n32<1>(o0, a_lo, b); }
                            }
                            wg_commit();
                            wg_wait_all();
                        }
                        release_stage(s);
                    }
            }
            const int nparts = wide ? 2 : 1;
            for (int part = 0; part < nparts; part++) {
                if (part) named_bar(1, NT_WORK);            // the first 256 channels have left the table
                if (P == 64) {                              // GEMM2 has completed: its β panels are no longer read
                    const int pb = (wg >> 1) * 32, cb = (wg & 1) * 64;
#pragma unroll
                    for (int e = 0; e < 16; e++) table[(pb + acc_col(t128, e)) * 256 + cb + acc_row(t128, e)] = o0[e];
                    if (NH > 1) {
#pragma unroll
                        for (int e = 0; e < 16; e++) table[(pb + acc_col(t128, e)) * 256 + 128 + cb + acc_row(t128, e)] = o1[e];
                    }
                } else if (part * 2 + (wg >> 1) < NH) {
                    const int cb = (wg >> 1) * 128 + (wg & 1) * 64;
#pragma unroll
                    for (int e = 0; e < 16; e++) table[acc_col(t128, e) * 256 + cb + acc_row(t128, e)] = part ? o1[e] : o0[e];
                }
                named_bar(1, NT_WORK);
#pragma unroll
                for (int u = 0; u < P / 16; u++) {
                    const int i = warp * (P / 16) + u;
                    const uint32_t p = d.pix[i];
                    if (i < d.g0 || i >= d.g0 + d.gn || p == 0xFFFFFFFFu) continue;          // warp-uniform
                    const int y = (int)(p >> 16), x = (int)(p & 0xffffu);
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) {
                        const int ct0 = hh * 128 + lane * 4, c0 = part * 256 + ct0;
                        if (c0 >= C) continue;
                        const float4 o = *reinterpret_cast<const float4 *>(table + i * 256 + ct0);
                        if (a.out_hi) {
                            uint2 h2, l2;
                            split_bf16x2(o.x, o.y, h2.x, l2.x);
                            split_bf16x2(o.z, o.w, h2.y, l2.y);
                            const size_t off = ((size_t)d.n * HW + y * W + x) * C + c0;
                            *reinterpret_cast<uint2 *>(a.out_hi + off) = h2;
                            *reinterpret_cast<uint2 *>(a.out_lo + off) = l2;
                        } else if (a.out_stride[1] == 1 && !a.add_ref) {
                            // channel-contiguous output (channels_last, or the library's pixel-major plane): one 16-byte store per lane
                            *reinterpret_cast<float4 *>(a.out + (int64_t)d.n * a.out_stride[0] + (int64_t)y * a.out_stride[2] + (int64_t)x * a.out_stride[3] + c0) = o;
                        } else {
                            const float ov[4] = {o.x, o.y, o.z, o.w};
                            float *ob = a.out + (int64_t)d.n * a.out_stride[0] + (int64_t)y * a.out_stride[2] + (int64_t)x * a.out_stride[3];
                            const int64_t rb = (int64_t)pair_items(d.n, a.n_ref, a.n_views, vs...).q * a.ref_stride[0] + (int64_t)y * a.ref_stride[2] + (int64_t)x * a.ref_stride[3];
#pragma unroll
                            for (int e = 0; e < 4; e++) {
                                float val = ov[e];
                                if (a.add_ref) val += ld_feat(a.feat_ref, rb + (int64_t)(c0 + e) * a.ref_stride[1], a.ref_dtype);
                                ob[(int64_t)(c0 + e) * a.out_stride[1]] = val;
                            }
                        }
                    }
                }
            }
        };

        const bool pt_on = tid == 0; (void)pt_on;
        PT_DECL;
        int j = 0;
        for (;; j++) {
            // Only warp 0 polls the mbarriers; the other 15 warps sleep in the hardware barrier instead of spinning through
            // issue slots.  The barrier also separates item j-1's use of the table.
            if (warp == 0) wait_n(&ct.desc_full[j % NDESC], (uint32_t)(j / NDESC));
            named_bar(1, NT_WORK);
            PT(0);
            if (tid == 0) TR(j, 4);
            if (tid == 0 && j >= 2) mbar_arrive(&ct.desc_free[(j - 2) % NDESC]);
            const Desc &d = desc_at(j);
            PT(1);
#ifdef EPI_PIPE_TIMERS
            if (d.tile < 0 && tid == 0 && blockIdx.x < 256) g_pipe_cta[blockIdx.x * 4 + 3] = (unsigned long long)j;
#endif
            if (d.tile < 0) break;
            const int D = d.D, n = d.n;
            const int nch = (D + CHUNK - 1) / CHUNK;

            // ---------------- B1: S = F·Qᵀ on the tensor cores -> T[rank][pixel] ----------------
            // Warpgroup wg accumulates union rows (wg >> 1) * 128 + (wg & 1) * 64 .. +63, i.e. half of chunk wg >> 1.
            PT(2);
            if (P == 64 && D > 0) {
                // Warpgroup wg accumulates union rows c * 128 + (wg & 1) * 64 .. +63 of chunk c against query half wg >> 1; the
                // accumulators go to that half's table after each chunk.
                float sacc[16];
#pragma unroll
                for (int e = 0; e < 16; e++) sacc[e] = 0.f;
                const uint32_t sqw = sq + (uint32_t)(wg >> 1) * 4u * PANEL_B2;
                float *th = table + (wg >> 1) * (DMAX * 32);
                if (warp == 0) wait_n(&ct.q_full, qcount);               // ordered before the MMAs by the first stage's barrier
                for (int c = 0; c < nch; c++) {
                    const int r0 = c * CHUNK + (wg & 1) * 64;
                    const bool mine = r0 < D;
                    for (int kp = 0; kp < NP; kp++) {
                        const uint32_t s = consume_stage();
                        if (mine) {
                            const uint32_t sa = smem_u32(smem + OFF_STAGE + s * STAGE_BYTES) + (uint32_t)(wg & 1) * 8192u;
                            wg_fence();
#pragma unroll
                            for (int ks = 0; ks < 4; ks++) {
                                const uint64_t a_hi = make_smem_desc(sa + ks * 32, 16, 1024), a_lo = desc_add(a_hi, PLANE_BYTES);
                                const uint64_t b = make_smem_desc(sqw + kp * PANEL_B2 + ks * 32, 16, 1024), b_lo = desc_add(b, 4096);
                                wgmma_m64n32<0>(sacc, a_hi, b);
                                if (LO) { wgmma_m64n32<0>(sacc, a_hi, b_lo); wgmma_m64n32<0>(sacc, a_lo, b); }
                            }
                            wg_commit();
                            wg_wait_all();
                        }
                        release_stage(s);
                    }
                    if (mine) {
#pragma unroll
                        for (int e = 0; e < 16; e++) {
                            const int r = r0 + acc_row(t128, e);
                            if (r < D) th[tix(r, acc_col(t128, e))] = sacc[e];
                            sacc[e] = 0.f;
                        }
                    }
                }
                if (tid == 0) mbar_arrive(&ct.q_empty);
                qcount++;
            } else if (D > 0) {
                float sacc[16];
#pragma unroll
                for (int e = 0; e < 16; e++) sacc[e] = 0.f;
                const int r0 = (wg >> 1) * CHUNK + (wg & 1) * 64;
                const bool mine = r0 < D;
                for (int qh = 0; qh < NQH; qh++) {
                    const int npq = min(4, NP - qh * 4);
                    if (warp == 0) wait_n(&ct.q_full, qcount);           // ordered before the MMAs by the first stage's barrier
                    for (int c = 0; c < nch; c++)
                        for (int kp = 0; kp < npq; kp++) {
                            const uint32_t s = consume_stage();
                            if (c == (wg >> 1) && mine) {
                                const uint32_t sa = smem_u32(smem + OFF_STAGE + s * STAGE_BYTES) + (uint32_t)(wg & 1) * 8192u;
                                wg_fence();
#pragma unroll
                                for (int ks = 0; ks < 4; ks++) {
                                    const uint64_t a_hi = make_smem_desc(sa + ks * 32, 16, 1024), a_lo = desc_add(a_hi, PLANE_BYTES);
                                    const uint64_t b = make_smem_desc(sq + kp * PANEL_B2 + ks * 32, 16, 1024), b_lo = desc_add(b, 4096);
                                    wgmma_m64n32<0>(sacc, a_hi, b);
                                    if (LO) { wgmma_m64n32<0>(sacc, a_hi, b_lo); wgmma_m64n32<0>(sacc, a_lo, b); }
                                }
                                wg_commit();
                                wg_wait_all();
                            }
                            release_stage(s);
                        }
                    if (tid == 0) mbar_arrive(&ct.q_empty);
                    qcount++;
                }
                if (mine) {
#pragma unroll
                    for (int e = 0; e < 16; e++) {
                        const int r = r0 + acc_row(t128, e);
                        if (r < D) table[tix(r, acc_col(t128, e))] = sacc[e];
                    }
                }
            }
            named_bar(1, NT_WORK);
            if (tid == 0) TR(j, 5);
            PT(3);

            // ---------------- softmax phase, once per 32-pixel half: lane <-> pixel ph * 32 + lane, T[rank][lane] in the half's table ----------------
            auto softmax_half = [&](int ph) {
                float *th = table + ph * (DMAX * 32);
                int *Ti = reinterpret_cast<int *>(th);
                // ---------------- B2a: bilinear interpolation of the scores, ==0 mask, scale ----------------
                const int i = ph * 32 + lane;                       // pixel of the item
                const uint32_t p = d.pix[i];
                const bool act = i >= d.g0 && i < d.g0 + d.gn && p != 0xFFFFFFFFu;
                const int py = (int)(p >> 16), px = (int)(p & 0xffffu);
                const int pofs = act ? py * W + px : 0;
                const float4 en = d.ends[i];
                float x[KW], tw[KW][4];
                uint32_t rk[KW][2];
                float mloc = -INFINITY;
                // Branch-free stages over the warp's KW samples so that their dependency chains (location -> footprint -> two bitmap
                // rank lookups -> four table reads) interleave instead of running one sample after the other.
                {
                    float gxs[KW], gys[KW];
                    bool live[KW], firstx0[KW];
                    // stage 1: locations, footprints, weights (zero for every tap that is out of bounds or not sampled)
#pragma unroll
                    for (int jj = 0; jj < KW; jj++) {
                        const int k = warp + NWORK * jj;
                        live[jj] = act && k < K;
                        float gx = 0.f, gy = 0.f;
                        if (a.locs_in) {
                            if (live[jj]) {
                                const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)k * a.N + n) * HW + pofs);
                                gx = l.x; gy = l.y;
                            }
                        } else {
                            gx = img2grid_x(lerp_exact(en.x, en.z, tkw[jj]), gc);
                            gy = img2grid_y(lerp_exact(en.y, en.w, tkw[jj]), gc);
                        }
                        gxs[jj] = gx; gys[jj] = gy;
                        const float ix = grid2pix(gx, W, gc.align), iy = grid2pix(gy, H, gc.align);
                        const bool in = live[jj] && ix > -1.f && ix < (float)W && iy > -1.f && iy < (float)H;   // else no tap in bounds (or NaN)
                        const float fx = in ? floorf(ix) : 0.f, fy = in ? floorf(iy) : 0.f;
                        const int x0 = (int)fx, y0 = (int)fy;                // -1 .. size-1
                        const float ax = ix - fx, ay = iy - fy;
                        const bool xin0 = in && x0 >= 0, xin1 = in && x0 + 1 < W, yin0 = y0 >= 0, yin1 = y0 + 1 < H;
                        tw[jj][0] = (xin0 && yin0) ? (1.f - ax) * (1.f - ay) : 0.f; tw[jj][1] = (xin1 && yin0) ? ax * (1.f - ay) : 0.f;
                        tw[jj][2] = (xin0 && yin1) ? (1.f - ax) * ay : 0.f;         tw[jj][3] = (xin1 && yin1) ? ax * ay : 0.f;
                        // each footprint row is looked up at its first in-bounds pixel: (x0, y) or, for x0 == -1, (0, y); pixel 0 when unused
                        const int first0 = y0 * W + x0 + (xin0 ? 0 : 1);
                        if (!big) {
                            rk[jj][0] = (uint32_t)((in && yin0) ? first0 : 0);
                            rk[jj][1] = (uint32_t)((in && yin1) ? first0 + W : 0);
                        } else {                                    // windowed bitmap: row << 16 | column
                            const uint32_t xf = (uint32_t)(x0 + (xin0 ? 0 : 1));
                            rk[jj][0] = (in && yin0) ? ((uint32_t)y0 << 16 | xf) : 0u;
                            rk[jj][1] = (in && yin1) ? ((uint32_t)(y0 + 1) << 16 | xf) : 0u;
                        }
                        firstx0[jj] = xin0;
                    }
                    if (a.locs_out) {
#pragma unroll
                        for (int jj = 0; jj < KW; jj++)
                            if (live[jj]) reinterpret_cast<float2 *>(a.locs_out)[((size_t)(warp + NWORK * jj) * a.N + n) * HW + pofs] = make_float2(gxs[jj], gys[jj]);
                    }
                    if (D > 0) {
                        const WinView wv = win_view(const_cast<Desc &>(d));
                        // stage 2: ranks — one bitmap lookup per footprint row; the row's second pixel is marked too, so it is rank + 1
                        const int rmax = D - 1;                               // defensive: a rank can never leave the table
#pragma unroll
                        for (int jj = 0; jj < KW; jj++)
#pragma unroll
                            for (int rw = 0; rw < 2; rw++) {
                                const int pix = (int)rk[jj][rw];
                                int ra;
                                if (!big) ra = (int)d.prefix[pix >> 5] + __popc(d.bitmap[pix >> 5] & ((1u << (pix & 31)) - 1u));
                                else {
                                    const int yy = pix >> 16, xx = pix & 0xffff;
                                    const int wi = min((int)wv.wbase[yy] + __popc(wv.rowmask[yy] & ((1u << (xx >> 5)) - 1u)), WIN_WORDS - 1);
                                    ra = (int)wv.prefix[wi] + __popc(wv.bitmap[wi] & ((1u << (xx & 31)) - 1u));
                                }
                                // first pixel = x0: taps (x0, x0+1) -> ranks (ra, ra+1);  first pixel = x0+1 (x0 == -1): tap x0+1 -> rank ra
                                rk[jj][rw] = (uint32_t)min(ra, rmax) | ((uint32_t)min(firstx0[jj] ? ra + 1 : ra, rmax) << 16);
                            }
                        // stage 3: interpolate the scores
#pragma unroll
                        for (int jj = 0; jj < KW; jj++) {
                            float sim = tw[jj][0] * th[tix((int)(rk[jj][0] & 0xffffu), lane)];
                            sim = fmaf(tw[jj][1], th[tix((int)(rk[jj][0] >> 16), lane)], sim);
                            sim = fmaf(tw[jj][2], th[tix((int)(rk[jj][1] & 0xffffu), lane)], sim);
                            sim = fmaf(tw[jj][3], th[tix((int)(rk[jj][1] >> 16), lane)], sim);
                            x[jj] = sim;
                        }
                    } else {
#pragma unroll
                        for (int jj = 0; jj < KW; jj++) { x[jj] = 0.f; rk[jj][0] = rk[jj][1] = 0u; }
                    }
                    // ==0 mask (epipolar.py:298), scale
#pragma unroll
                    for (int jj = 0; jj < KW; jj++) {
                        const float sim = x[jj] == 0.f ? kMasked : x[jj];
                        x[jj] = live[jj] ? sim * sl2 : -INFINITY;
                        mloc = fmaxf(mloc, x[jj]);
                    }
                }
                red_max[warp * 32 + lane] = mloc;
                named_bar(1, NT_WORK);
                PT(4);

                // ---------------- B2b: softmax over K (16-way split), zero the table for the β scatter ----------------
                float M = -INFINITY;
#pragma unroll
                for (int w = 0; w < NWORK; w++) M = fmaxf(M, red_max[w * 32 + lane]);
                float sloc = 0.f;
#pragma unroll
                for (int jj = 0; jj < KW; jj++) { x[jj] = (act && warp + NWORK * jj < K) ? exp2f(x[jj] - M) : 0.f; sloc += x[jj]; }
                red_sum[warp * 32 + lane] = sloc;
                for (int q = tid; q < D * 8; q += NT_WORK) reinterpret_cast<int4 *>(Ti)[q] = make_int4(0, 0, 0, 0);
                named_bar(1, NT_WORK);
                float S = 0.f;
#pragma unroll
                for (int w = 0; w < NWORK; w++) S += red_sum[w * 32 + lane];
                const float inv = 1.f / S;
                float best_v = -1.f;
                int best_k = 0x7fffffff;
                float *ab = a.attn ? a.attn + (size_t)n * K * HW + pofs : nullptr;
#pragma unroll
                for (int jj = 0; jj < KW; jj++) {
                    const int k = warp + NWORK * jj;
                    if (act && k < K) {
                        const float av = x[jj] * inv;
                        if (ab) __stcs(ab + (size_t)k * HW, av);          // outputs are written once and not re-read here: streaming stores keep L2 for the planes
                        if (av > best_v) { best_v = av; best_k = k; }
                        // deterministic fixed-point scatter of a_k·w_kt into β[rank][pixel]
#pragma unroll
                        for (int tp = 0; tp < 4; tp++)
                            if (tw[jj][tp] != 0.f) {
                                const uint32_t r = (rk[jj][tp >> 1] >> ((tp & 1) * 16)) & 0xffffu;
                                atomicAdd(&Ti[tix((int)r, lane)], __float2int_rn(av * tw[jj][tp] * FIX));
                            }
                    }
                }
                if (a.corr_pos) { red_bv[warp * 32 + lane] = best_v; red_bk[warp * 32 + lane] = best_k; }
                named_bar(1, NT_WORK);
                PT(5);
                // ---------------- arg-max -> corr_pos (first maximum, like torch.argmax) ----------------
                if (a.corr_pos && warp == 0 && act) {
                    float bv = -1.f; int bk = 0x7fffffff;
#pragma unroll
                    for (int w = 0; w < NWORK; w++) {
                        const float v = red_bv[w * 32 + lane]; const int kk = red_bk[w * 32 + lane];
                        if (EPI_FIRST_MAX_BEATS(v, kk, bv, bk)) { bv = v; bk = kk; }
                    }
                    float gx, gy;
                    if (a.locs_in) {
                        const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)bk * a.N + n) * HW + pofs);
                        gx = l.x; gy = l.y;
                    } else {
                        const float t = (float)bk / (float)(K - 1);
                        gx = img2grid_x(lerp_exact(en.x, en.z, t), gc); gy = img2grid_y(lerp_exact(en.y, en.w, t), gc);
                    }
                    __stcs(reinterpret_cast<float2 *>(a.corr_pos) + (size_t)n * HW + pofs, make_float2(grid2corr(gx, W, gc.correct), grid2corr(gy, H, gc.correct)));
                }
                // ---------------- β[rank][pixel] -> bf16 (hi, lo) stacked K-major panels; warp <-> 16 ranks, lane <-> pixel ----------------
                PT(6);
                // 64 pixels: the panels take the place of the half's int32 β (4 bytes per (rank, pixel) either way), so every β value
                // is read into registers before any panel is written
                auto panels = [&](uint8_t *bb, int hh, const float (&f)[8]) {
                    const int d0 = warp * 16 + hh * 8;
                    uint4 hi, lo;
                    split8(f, hi, lo);
                    const uint32_t off = (uint32_t)(d0 >> 6) * PANEL_B2 + (uint32_t)lane * 128u + (uint32_t)((((d0 & 63) >> 3) ^ (lane & 7)) << 4);
                    *reinterpret_cast<uint4 *>(bb + off) = hi;
                    *reinterpret_cast<uint4 *>(bb + 4096 + off) = lo;
                };
                auto beta = [&](int hh, float (&f)[8]) {
                    const int d0 = warp * 16 + hh * 8;
#pragma unroll
                    for (int e = 0; e < 8; e++) f[e] = (act && d0 + e < D) ? (float)Ti[tix(d0 + e, lane)] * (1.0f / FIX) : 0.f;
                };
                if constexpr (P == 64) {
                    float f[2][8];
                    beta(0, f[0]); beta(1, f[1]);
                    named_bar(1, NT_WORK);
                    panels(reinterpret_cast<uint8_t *>(Ti), 0, f[0]); panels(reinterpret_cast<uint8_t *>(Ti), 1, f[1]);
                } else {
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) { float f[8]; beta(hh, f); panels(smem + OFF_BETA, hh, f); }
                }
                fence_proxy_async_smem();
            };
            if constexpr (NPH == 1) softmax_half(0);
            else {
#pragma unroll 1
                for (int ph = 0; ph < NPH; ph++) softmax_half(ph);
            }
            if (tid == 0) TR(j, 6);
            named_bar(1, NT_WORK);                          // the table is free: the epilogue transposes through it
            PT(7);
            // ---------------- GEMM2 and epilogue ----------------
            epilogue(j);
            if (tid == 0) TR(j, 7);
            PT(9);
#ifdef EPI_PIPE_TIMERS
            if (pt_on) atomicAdd(&g_pipe_timers[8], 1ull);
#endif
        }
    } else if (warp < W_GATHER) {
        // =====================================================================================================
        // SETUP (4 warps): build work items
        // =====================================================================================================
        const int st = tid - W_SETUP * 32;                 // 0..127
        const int sw = warp - W_SETUP;
        int claimed = 0;
        const bool pt_on = st == 0; (void)pt_on;
        PT_DECL;
        float tk[KPL];                                      // this lane's sample parameters k/(K-1), k = lane + 32 jj
#pragma unroll
        for (int jj = 0; jj < KPL; jj++) tk[jj] = (float)(lane + 32 * jj) / (float)(K - 1);
        // every in-bounds pixel of the 2x2 bilinear footprint (a superset of the taps with non-zero weight): one atomicOr per
        // footprint row (two only when the row's pixels straddle a 32-bit word)
        auto footprint = [&](float gx, float gy, int &x0, int &y0) -> bool {
            const float ix = grid2pix(gx, W, gc.align), iy = grid2pix(gy, H, gc.align);
            if (!(ix > -1.f && ix < (float)W && iy > -1.f && iy < (float)H)) return false;    // also rejects NaN / far sentinels
            x0 = (int)floorf(ix); y0 = (int)floorf(iy);                                       // -1 .. size-1
            return true;
        };
        auto mark = [&](Desc &d, float gx, float gy) {
            int x0, y0;
            if (!footprint(gx, gy, x0, y0)) return;
            const uint32_t mbits = x0 < 0 ? 1u : (x0 + 1 < W ? 3u : 1u);                   // pixels max(x0,0) [, x0+1]
            const int pos = y0 * W + max(x0, 0);
            auto row = [&](int ps) {
                const uint32_t sh = (uint32_t)ps & 31u;
                atomicOr(&d.bitmap[ps >> 5], mbits << sh);
                if (sh == 31u && mbits == 3u) atomicOr(&d.bitmap[(ps >> 5) + 1], 1u);
            };
            if (y0 >= 0) row(pos);
            if (y0 + 1 < H) row(pos + W);
        };
        // row-windowed variant, pass A: which 32-pixel words of each source row the union touches
        auto mark_rows = [&](const WinView &wv, float gx, float gy) {
            int x0, y0;
            if (!footprint(gx, gy, x0, y0)) return;
            const int xa = max(x0, 0), xb = min(x0 + 1, W - 1);
            const uint32_t m = (1u << (xa >> 5)) | (1u << (xb >> 5));
            if (y0 >= 0) atomicOr(&wv.rowmask[y0], m);
            if (y0 + 1 < H) atomicOr(&wv.rowmask[y0 + 1], m);
        };
        // pass B: the pixels, into the compacted words
        auto mark_bits = [&](const WinView &wv, float gx, float gy) {
            int x0, y0;
            if (!footprint(gx, gy, x0, y0)) return;
            const int xa = max(x0, 0), xb = min(x0 + 1, W - 1);
            auto row = [&](int y) {
                const uint32_t rm = wv.rowmask[y];
                const int wa = min((int)wv.wbase[y] + __popc(rm & ((1u << (xa >> 5)) - 1u)), WIN_WORDS - 1);
                if ((xa >> 5) == (xb >> 5)) atomicOr(&wv.bitmap[wa], (1u << (xa & 31)) | (1u << (xb & 31)));
                else { atomicOr(&wv.bitmap[wa], 1u << 31); atomicOr(&wv.bitmap[min(wa + 1, WIN_WORDS - 1)], 1u); }
            };
            if (y0 >= 0) row(y0);
            if (y0 + 1 < H) row(y0 + 1);
        };
        // every (pixel, sample) location of the group [g0, g0 + gn): lane <-> sample
        auto for_each_loc = [&](Desc &d, int n, int g0, int gn, auto &&fn) {
            for (int i = g0 + sw; i < g0 + gn; i += NSETUP / 32) {
                const uint32_t p = d.pix[i];
                if (p == 0xFFFFFFFFu) continue;
                if (a.locs_in) {
#pragma unroll
                    for (int jj = 0; jj < KPL; jj++) {
                        const int k = lane + 32 * jj;
                        if (k < K) {
                            const float2 l = __ldg(reinterpret_cast<const float2 *>(a.locs_in) + ((size_t)k * a.N + n) * HW + (p >> 16) * W + (p & 0xffffu));
                            fn(l.x, l.y);
                        }
                    }
                } else {
                    const float4 e = d.ends[i];
#pragma unroll
                    for (int jj = 0; jj < KPL; jj++)
                        if (lane + 32 * jj < K) fn(img2grid_x(lerp_exact(e.x, e.z, tk[jj]), gc), img2grid_y(lerp_exact(e.y, e.w, tk[jj]), gc));
                }
            }
        };
        // exclusive prefix of the popcounts of `nw` words by the first setup warp; leaves the total in ct.total
        auto prefix_words = [&](const uint32_t *bm, uint16_t *pf, int nw) {
            const int per = (nw + 31) >> 5;
            int cnt = 0;
            for (int q = 0; q < per; q++) { const int w = lane * per + q; if (w < nw) cnt += __popc(bm[w]); }
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
            int run = incl - cnt;
            for (int q = 0; q < per; q++) {
                const int w = lane * per + q;
                if (w < nw) { pf[w] = (uint16_t)run; run += __popc(bm[w]); }
            }
            if (lane == 31) ct.total = incl;
        };
        for (int j = 0;; j++) {
            Desc &d = desc_at(j);
            if (st == 0 && j >= NDESC) wait_n(&ct.desc_free[j % NDESC], (uint32_t)(j / NDESC - 1));   // the claim barrier below releases the rest
            if (st == 0) TR(j, 0);
            PT(10);
            bool done = false;
            while (true) {
                // ---- next group: pop the split stack or claim a new tile ----
                if (st == 0) {
                    if (ct.sp == 0) {
                        int c;
                        if (claimed == 0) c = (int)blockIdx.x;
                        else c = a.tile_counter ? (int)gridDim.x + atomicAdd(a.tile_counter, 1) : (int)blockIdx.x + claimed * (int)gridDim.x;
                        claimed++;
                        ct.cur_claim = c;
                        // per pair: tiles [0, tpi - r_half) are claimed whole, the last r_half tiles as two halves each (the same
                        // tiles of every pair, so results do not depend on a pair's position in the batch)
                        const int whole = tiles_per_item - r_half;
                        if (c < a.N * whole) { ct.cur_tile = (c / whole) * tiles_per_item + c % whole; ct.stack[0] = 0 | (P << 8); ct.sp = 1; }
                        else if (c < a.N * whole + 2 * a.N * r_half) {
                            const int h = c - a.N * whole, hh = h >> 1;
                            ct.cur_tile = (hh / r_half) * tiles_per_item + whole + hh % r_half;
                            ct.stack[0] = ((h & 1) * (P / 2)) | ((P / 2) << 8); ct.sp = 1;
                        } else ct.done = 1;
                    }
                    else ct.cur_claim = -1;                               // a piece of a split tile: never cached
                    if (!ct.done) ct.cur = ct.stack[--ct.sp];
                }
                named_bar(2, NSETUP);
                PT(28);
                if (ct.done) { done = true; break; }
                const int tile = ct.cur_tile, g0 = ct.cur & 0xff, gn = ct.cur >> 8;
                const int n = tile / tiles_per_item, trem = tile % tiles_per_item;
                // ---- plan cache: a work item depends on the cameras only (pixel list, line end points, tap union, ranks, row list), so a
                // claim whose record carries the pair's current epoch is copied instead of rebuilt (records live in the caller's cache) ----
                // A 64-pixel item's record takes the two slots of its two 32-pixel tiles: claim c -> slots 2c, 2c + 1 (a claim whose
                // slots are not all in the region is rebuilt every call); bit 31 of its tag keeps the two record kinds apart.
                const int claim = ct.cur_claim;                            // >= 0 only for a freshly claimed (unsplit) item
                constexpr int SLOTS = P / PREC;
                constexpr uint32_t KIND = P == 64 ? 0x80000000u : 0u;
                uint8_t *rec = (a.plan_cache && !a.locs_in && claim >= 0 && claim < a.plan_records / SLOTS) ? a.plan_cache + (size_t)claim * SLOTS * REC_BYTES : nullptr;
                const uint32_t ep = rec ? __ldg(a.pair_epoch + 32 * n) : 0u;
                if (rec) {
                    const Desc *g = reinterpret_cast<const Desc *>(rec);
                    if (g->epoch == ep && g->claim_tag == ((uint32_t)claim + 1u | KIND) && g->tile == tile && (P == 32 || tags64_intact(rec, g->claim_tag))) {      // uniform: every thread reads the same words
                        const uint4 *src4 = reinterpret_cast<const uint4 *>(rec);
                        uint4 *dst4 = reinterpret_cast<uint4 *>(&d);
                        for (int q = st; q < (int)(sizeof(Desc) / 16); q += NSETUP) dst4[q] = src4[q];
                        named_bar(2, NSETUP);
                        break;
                    }
                }
                if (st < P) {                               // pixel + its epipolar line end points
                    const int e = trem * P + st;
                    unsigned p = 0u;
                    if (e < HW) p = a.order ? (unsigned)a.order[(size_t)n * HW + e] : (unsigned)e;
                    const int py = (int)(p / W), px = (int)(p % W);
                    d.pix[st] = (e < HW) ? ((uint32_t)py << 16 | (uint32_t)px) : 0xFFFFFFFFu;
                    float4 en = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (e < HW && !a.locs_in) {
                        PairGeom g;
                        const float *gp = reinterpret_cast<const float *>(a.pair_geom + n);
#pragma unroll
                        for (int q = 0; q < 9; q++) g.M[q] = __ldg(gp + q);
                        g.ex = __ldg(gp + 9); g.ey = __ldg(gp + 10);
                        line_endpoints(g, gc, pix2coord(px, gc.ds, gc.r), pix2coord(py, gc.ds, gc.r), en.x, en.y, en.z, en.w);
                    }
                    d.ends[st] = en;
                } else if (st == P) { d.tile = tile; d.n = n; d.g0 = g0; d.gn = gn; }
                for (int w = st - 64; w >= 0 && w < (big ? 2 * WIN_WORDS : nwords); w += 64) d.bitmap[w] = 0u;     // warps 2,3 clear the bitmap (+ row masks)
                named_bar(2, NSETUP);
                PT(29);
                // ---- union of the in-bounds taps: lane <-> sample (consecutive samples fall into different words) ----
                const WinView wv = win_view(d);
                bool too_wide = false;
                if (!big) {
                    for_each_loc(d, n, g0, gn, [&](float gx, float gy) { mark(d, gx, gy); });
                    named_bar(2, NSETUP);
                    PT(30);
                    if (sw == 0) prefix_words(d.bitmap, d.prefix, nwords);
                } else {
                    for_each_loc(d, n, g0, gn, [&](float gx, float gy) { mark_rows(wv, gx, gy); });
                    named_bar(2, NSETUP);
                    if (sw == 0) prefix_words(wv.rowmask, wv.wbase, H);             // wbase[y] = words before row y
                    named_bar(2, NSETUP);
                    const int TW = ct.total;
                    named_bar(2, NSETUP);                                            // ct.total is rewritten below
                    too_wide = TW > WIN_WORDS;                                        // more touched words than union rows allowed: split
                    if (!too_wide) {
                        for_each_loc(d, n, g0, gn, [&](float gx, float gy) { mark_bits(wv, gx, gy); });
                        named_bar(2, NSETUP);
                        PT(30);
                        if (sw == 0) prefix_words(wv.bitmap, wv.prefix, TW);
                    } else if (st == 0) ct.total = DMAX + 1;
                }
                named_bar(2, NSETUP);
                PT(31);
                const int D = ct.total;
                if (D > DMAX && gn > 1) {                 // split the group
                    if (st == 0) {
                        const int h1 = gn >> 1;
                        ct.stack[ct.sp++] = (g0 + h1) | ((gn - h1) << 8);
                        ct.stack[ct.sp++] = g0 | (h1 << 8);
                    }
                    named_bar(2, NSETUP);
                    continue;
                }
                const int Dc = D > DMAX ? 0 : D;          // a single pixel over DMAX cannot happen for supported shapes (host check)
                if (D > DMAX && st == 0 && a.err_flag) atomicOr(a.err_flag, 1);
                // ---- union list: idx[rank] = source pixel; pad to a multiple of 16 with a valid row ----
                if (Dc > 0 && !big)
                    for (int w = st; w < nwords; w += NSETUP) {
                        uint32_t bits = d.bitmap[w];
                        int r = d.prefix[w];
                        while (bits) { const int b = __ffs(bits) - 1; bits &= bits - 1; d.idx[r++] = (uint16_t)(w * 32 + b); }
                    }
                if (Dc > 0 && big)
                    for (int y = st; y < H; y += NSETUP) {
                        uint32_t rm = wv.rowmask[y];
                        int wi = wv.wbase[y];
                        while (rm) {
                            const int xw = __ffs(rm) - 1; rm &= rm - 1;
                            uint32_t bits = wv.bitmap[wi];
                            int r = wv.prefix[wi];
                            while (bits) { const int b = __ffs(bits) - 1; bits &= bits - 1; d.idx[r++] = (uint16_t)(y * W + xw * 32 + b); }
                            wi++;
                        }
                    }
                named_bar(2, NSETUP);
                PT(17);
                if (st < 16 && Dc > 0) { const int r = Dc + st; if (r < ((Dc + 15) & ~15)) d.idx[r] = d.idx[0]; }
                if (st == 16) { d.D = Dc; d.epoch = ep; d.claim_tag = (uint32_t)claim + 1u | KIND; if constexpr (P == 64) d.tag32[6] = d.claim_tag; }
                named_bar(2, NSETUP);
                if (rec && D <= DMAX) {                                   // publish the record (read by later launches only)
                    const uint4 *src4 = reinterpret_cast<const uint4 *>(&d);
                    uint4 *dst4 = reinterpret_cast<uint4 *>(rec);
                    for (int q = st; q < (int)(sizeof(Desc) / 16); q += NSETUP) dst4[q] = src4[q];
                    if constexpr (P == 64) if (st == 0) *reinterpret_cast<uint32_t *>(rec + REC_BYTES + offsetof(ItemDesc<32>, claim_tag)) = d.claim_tag;
                }
                PT(18);
                break;
            }
            if (done) {
                if (st == 0) { d.tile = -1; mbar_arrive(&ct.desc_full[j % NDESC]); }
                break;
            }
            if (st == 0) mbar_arrive(&ct.desc_full[j % NDESC]);
            if (st == 0) TR(j, 1);
            PT(11);
        }
    } else {
        // =====================================================================================================
        // GATHER WARPS (128 threads): query rows and feature stages, 16-byte cp.async into swizzled panels.
        // Thread t copies chunk j = t & 7 (8 channels) of rows (t >> 3) + 16·it; a row's 128-byte segment is read by 8
        // consecutive lanes.  Completion: cp.async.mbarrier.arrive.noinc on the stage's mbarrier (count = 128 threads).
        // =====================================================================================================
        const int gt = tid - W_GATHER * 32, gj = gt & 7, gr = gt >> 3;
        // [ref_hi | ref_lo | src_hi | src_lo] (LO) or [ref_hi | src_hi]; a lo plane follows its hi plane.  Reference planes are
        // [n_ref*HW][C], source planes [N*HW][C]; the views form has one pair of planes [n_views*n_ref*HW][C] (pair_items)
        const size_t plane_elems = LO ? (size_t)(a.src_lo - a.src_hi) : 0, ref_plane_elems = LO ? (size_t)(a.ref_lo - a.ref_hi) : 0;
        uint32_t qcount = 0, fcount = 0;
        const bool pt_on = gt == 0; (void)pt_on;
        PT_DECL;
        auto stage_acquire = [&]() -> uint8_t * {
            const uint32_t s = fcount % NSTAGE;
            PT(13);
            if (fcount >= NSTAGE) {
                if (gt < 32) wait_n(&ct.f_empty[s], fcount / NSTAGE - 1);
                named_bar(3, NGATHER);
            }
            PT(14);
            return smem + OFF_STAGE + s * STAGE_BYTES;
        };
        auto arrive_async = [&](uint64_t *bar) {
            asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
        };
        // shared-memory offset of this thread's 16-byte chunk inside a 128-byte-row panel: rows gr + 16·it keep (row & 7) = gr & 7
        const uint32_t so0 = (uint32_t)gr * 128u + (uint32_t)((gj ^ (gr & 7)) << 4);
        const uint32_t smem_base = smem_u32(smem);
        auto cp16 = [&](uint32_t dst, const __nv_bfloat16 *srcp, bool valid) {
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(srcp), "r"(valid ? 16 : 0) : "memory");
        };
        auto gemm2_stages = [&](int jj, const __nv_bfloat16 *src) {      // src: the hi plane of the item's source map
            const Desc &d = desc_at(jj);
            const int D16 = (d.D + 15) & ~15, nblk = (D16 + 63) >> 6;
            for (int blk = 0; blk < nblk; blk++) {               // (block of 64 union rows) outer, channel half inner: row addresses are
                const int rows = min(64, D16 - blk * 64);        // computed once per block
                uint32_t roff[4];
#pragma unroll
                for (int it = 0; it < 4; it++) roff[it] = (gr + 16 * it < rows) ? (uint32_t)d.idx[blk * 64 + gr + 16 * it] * (uint32_t)C : 0u;
                for (int h = 0; h < NH; h++) {
                    const uint32_t stg = smem_base + (uint32_t)(stage_acquire() - smem);
#pragma unroll
                    for (int it = 0; it < 4; it++) {
                        if (gr + 16 * it < rows) {
                            const __nv_bfloat16 *row = src + roff[it];
                            const uint32_t so = so0 + (uint32_t)it * 2048u;
#pragma unroll
                            for (int pn = 0; pn < 2; pn++) {
                                const int ch = (h * 2 + pn) * 64 + gj * 8;
                                if (ch < C) {
                                    cp16(stg + pn * 8192 + so, row + ch, true);
                                    if (LO) cp16(stg + PLANE_BYTES + pn * 8192 + so, row + plane_elems + ch, true);
                                }
                            }
                        }
                    }
                    arrive_async(&ct.f_full[fcount % NSTAGE]);
                    fcount++;
                }
            }
        };
        for (int j = 0;; j++) {
            PT(13);
            if (gt < 32) wait_n(&ct.desc_full[j % NDESC], (uint32_t)(j / NDESC));
            named_bar(3, NGATHER);
            PT(15);
            const Desc &d = desc_at(j);
            const bool last = d.tile < 0;
            const PairItems items = pair_items(d.n, a.n_ref, a.n_views, vs...);
            const __nv_bfloat16 *src = a.src_hi + (size_t)items.s * HW * C;
            if (!last && d.D > 0) {
                // ---- per half of the query panels (one half unless C > 256): the item's query rows as stacked panels
                //      [hi 32 rows | lo 32 rows], then the GEMM1 stages (chunk, 64-channel panel) that multiply with them ----
                const int D16 = (d.D + 15) & ~15, nch = (d.D + CHUNK - 1) / CHUNK;
                for (int qh = 0; qh < NQH; qh++) {
                    const int npq = min(4, NP - qh * 4);
                    if (qcount >= 1) {
                        if (gt < 32) wait_n(&ct.q_empty, qcount - 1);
                        named_bar(3, NGATHER);
                    }
                    PT(16);
                    {
                        const __nv_bfloat16 *ref = a.ref_hi + (size_t)items.q * HW * C;
#pragma unroll
                        for (int it = 0; it < P / 16; it++) {           // pixel r goes to row r % 32 of query half r / 32
                            const int r = gr + 16 * it;
                            const uint32_t p = d.pix[r];
                            const __nv_bfloat16 *row = ref + (size_t)(p == 0xFFFFFFFFu ? 0 : (int)(p >> 16) * W + (int)(p & 0xffffu)) * C;
                            const uint32_t so = smem_base + OFF_Q + (uint32_t)(it >> 1) * 4u * PANEL_B2 + so0 + (uint32_t)(it & 1) * 2048u;
#pragma unroll
                            for (int kp = 0; kp < 4; kp++) {
                                const int ch = (qh * 4 + kp) * 64 + gj * 8;
                                if (kp < npq) {                 // channels beyond C are zero-filled: they are part of the MMA K range
                                    const bool ok = ch < C;
                                    cp16(so + kp * PANEL_B2, ok ? row + ch : row, ok);
                                    if (LO) cp16(so + kp * PANEL_B2 + 4096, ok ? row + ref_plane_elems + ch : row, ok);
                                }
                            }
                        }
                    }
                    arrive_async(&ct.q_full);
                    qcount++;
                    for (int c = 0; c < nch; c++) {             // the row addresses of a chunk are computed once for its panels
                        const int rows = min(CHUNK, D16 - c * CHUNK);
                        uint32_t roff[8];
#pragma unroll
                        for (int it = 0; it < 8; it++) roff[it] = (gr + 16 * it < rows) ? (uint32_t)d.idx[c * CHUNK + gr + 16 * it] * (uint32_t)C : 0u;
                        for (int kp = 0; kp < npq; kp++) {
                            const uint32_t stg = smem_base + (uint32_t)(stage_acquire() - smem);
                            const int ch = (qh * 4 + kp) * 64 + gj * 8;
                            const bool ok = ch < C;
                            const __nv_bfloat16 *colp = src + (ok ? ch : 0);
#pragma unroll
                            for (int it = 0; it < 8; it++) {
                                if (gr + 16 * it < rows) {
                                    const __nv_bfloat16 *row = colp + roff[it];
                                    const uint32_t so = stg + so0 + (uint32_t)it * 2048u;
                                    cp16(so, row, ok);
                                    if (LO) cp16(so + PLANE_BYTES, row + plane_elems, ok);
                                }
                            }
                            arrive_async(&ct.f_full[fcount % NSTAGE]);
                            fcount++;
                        }
                    }
                }
            }
            if (gt == 0) TR(j, 2);
            if (last) break;
            if (d.D > 0) gemm2_stages(j, src);                   // the workers run GEMM2(j) before GEMM1(j+1)
            if (gt == 0) TR(j, 8);
            named_bar(3, NGATHER);                          // every gather thread has read item j's row list
            if (gt == 0) mbar_arrive(&ct.desc_free[j % NDESC]);
        }
    }

    // ---------------- teardown ----------------
    __syncthreads();
#ifdef EPI_PIPE_TIMERS
    if (tid == 0 && blockIdx.x < 256) { unsigned long long g; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g)); g_pipe_cta[blockIdx.x * 4 + 2] = g; }
#endif
}


#ifdef EPI_PIPE_TIMERS
extern "C" void epi_pipe_cta_read(unsigned long long *out1024) { cudaMemcpyFromSymbol(out1024, g_pipe_cta, sizeof(unsigned long long) * 1024); }
extern "C" void epi_pipe_trace_read(long long *out1024) { cudaMemcpyFromSymbol(out1024, g_pipe_trace, sizeof(long long) * 64 * 16); }
extern "C" void epi_pipe_timers_read(unsigned long long *out32, int reset) {
    cudaMemcpyFromSymbol(out32, g_pipe_timers, sizeof(unsigned long long) * 32);
    if (reset) { unsigned long long z[32] = {0}; cudaMemcpyToSymbol(g_pipe_timers, z, sizeof(z)); }
}
#endif

size_t fusion_pipe_plan_record_bytes() { return REC_BYTES; }
// claims = whole tiles + the half items of the last partial round over the grid of n_ref pairs (< number of SMs, rounded up per
// pair), for each of the N / n_ref sources; counted in 32-pixel record slots
int fusion_pipe_plan_records(int N, int n_ref, int H, int W) { return N * ((H * W + PREC - 1) / PREC) + (N / n_ref) * (256 + n_ref); }

bool fusion_pipe_shape_ok(int C, int H, int W, int K, bool has_locs_in) {
    if (C % 8 != 0 || C > 512 || C < 8) return false;
    if (H * W > MAXWORDS * 32 && (H > WIN_ROWS || W > WIN_MAXW || H * W > 65536)) return false;   // row-windowed bitmap above 16384 pixels
    if (K > 32 * MAXKPL) return false;
    // A single pixel's union must fit DMAX (items are split down to one pixel).  4 taps per sample; and for the fused geometry the
    // samples lie on a straight segment: along its dominant axis it crosses at most max(W, H) columns, and a column u belongs to the
    // footprint of samples with ix in [u-1, u+1) — over that interval iy moves by at most 2, so floor(iy) takes at most 3 values and
    // the 2-row footprints cover at most 4 rows: the union has at most 4 * max(W, H) pixels.
    const int mx = H > W ? H : W;
    const int single = has_locs_in ? 4 * K : (4 * K < 4 * mx ? 4 * K : 4 * mx);
    return single <= DMAX;
}

// 64-pixel items on maps of at most 64 pixels a side with C <= 256: there the union of 64 pixels' taps stays well inside DMAX rows
// (at most 232 at K = 128 on the benchmark's cameras; a larger one splits into its 32-pixel halves).
int fusion_pipe_item_pixels(int C, int H, int W) { return (H > W ? H : W) <= 64 && C <= 256 ? 64 : 32; }

template <int P, typename... Tab>
static cudaError_t launch_items(const FusionArgs &a, cudaStream_t st, const Tab &... vs) {
    const int HW = a.geom.H * a.geom.W;
    const int tiles = a.N * ((HW + P - 1) / P);
    const int kpl = (a.geom.K + 31) / 32;
    const bool lo = a.src_lo != nullptr;
    void (*kern)(const FusionArgs, const Tab...) =
        lo ? (kpl <= 1 ? epi_fusion_pipe_kernel<1, true, P, Tab...> : (kpl <= 2 ? epi_fusion_pipe_kernel<2, true, P, Tab...> : epi_fusion_pipe_kernel<4, true, P, Tab...>))
           : (kpl <= 1 ? epi_fusion_pipe_kernel<1, false, P, Tab...> : (kpl <= 2 ? epi_fusion_pipe_kernel<2, false, P, Tab...> : epi_fusion_pipe_kernel<4, false, P, Tab...>));
    static thread_local DeviceFlags attr_set[6];
    const int ki = (kpl <= 1 ? 0 : (kpl <= 2 ? 1 : 2)) + (lo ? 0 : 3);
    const int dev = current_device();
    if (!attr_set[ki].has(dev)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_alloc<P>());
        if (e != cudaSuccess) return e;
        attr_set[ki].set(dev);
    }
    const int sms = sm_count();
    const int grid = tiles < sms ? tiles : sms;                    // one persistent CTA per SM
    cudaError_t le = launch_pdl(kern, dim3((unsigned)grid), dim3(NT_ALL), (size_t)smem_alloc<P>(), st, a, vs...);
    if (le != cudaSuccess) return le;
    return cudaGetLastError();
}

cudaError_t launch_fusion_pipe(const FusionArgs &a, const ViewSources &vs, cudaStream_t st) {
    if (vs.S) return a.item_px == 64 ? launch_items<64>(a, st, vs) : launch_items<32>(a, st, vs);
    return a.item_px == 64 ? launch_items<64>(a, st) : launch_items<32>(a, st);
}

}  // namespace epi
