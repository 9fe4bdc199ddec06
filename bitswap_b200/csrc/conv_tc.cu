// wgmma implicit-GEMM convolution for the dense W->W layers, the in-convs and the mu/sigma heads (sm_90a).
//
// Replaces F.conv2d inside WnConv2d._forward for the 3x3 / 5x5 W->W convolutions of the ResNet blocks
// (utils/torch/modules.py:98-106 called from ResNetLayer.forward :229-241), which are 98 % of the
// model's FLOPs (SURVEY.md 6.3).
//
// GEMM view (per image):  D[p, o] = sum_{tap, c} A_tap[p, c] * W[tap][o, c]
//     one tile = 128 pixels (8 image rows of a 16x16 image) x N output channels (N = 128 for the W->W convs and the
//     in-convs, 64 for those of a model of padded width 64 or 192, 32 for the heads), K = taps x input channels, walked as
//     (tap, 32-channel chunk) k-blocks.
//   * A_tap is never materialised (no im2col): the activation tensor is NHWC bf16 and one 4-D TMA box
//     {32 ch, 16 w, 8 h, 1 img} at coordinates (c0, dx-r, dy-r+8*half, img) IS the shifted tile; TMA's
//     out-of-bounds zero fill supplies the "same" padding.
//   * float32 accuracy on bf16 tensor cores: every operand is split x = hi + lo (two bf16 planes) and
//     each k-block issues three MMAs: hi*hi into a MAIN float32 accumulator, hi*lo and lo*hi into a
//     separate CROSS accumulator.  The tensor core truncates on every accumulate; keeping the 2^-8 smaller
//     cross terms out of the main accumulator cuts its truncating adds 3x.
//   * warp roles (384 threads): warps 0..7 = two consumer warpgroups, each owning 64 of the tile's 128 pixels and
//     issuing wgmma.m64nNk16 from shared memory into register accumulators ({main, cross} x N/2 floats per thread);
//     after the last k-block they write main + cross into an fp32 hand-off tile in shared memory and go on with the
//     next tile.  Warp 8 = TMA producer (one elected lane) feeding an NSTAGE ring of mbarrier-guarded stages; warps
//     9..11 = epilogue (bias / residual / ELU / bf16 split -> HBM) from the hand-off tile.  setmaxnreg gives the
//     consumers 160 registers and the producer / epilogue warpgroup 64.
//   * a CTA walks tiles t = blockIdx.x, + gridDim.x, ...: with one CTA per tile (per-tile grid) or one per SM
//     (persistent grid: the producer prefetches the next tile's k-blocks and the consumers run its MMAs while the
//     epilogue warps store the previous tile).
//   * the dense convs and in-convs run as four-CTA clusters, one image per cluster, CTA rank r = tile t & 3 =
//     (pixel half r & 1, channel block r >> 1): the two channel blocks of a pixel half read the same A boxes, the two
//     pixel halves of a channel block the same W boxes.  Each CTA issues two of a stage's four boxes with TMA multicast
//     to itself and the peer that shares them, so every CTA pulls 16 of its 32 KB per k-block from L2 (the launches are
//     bound by L2 -> SM bytes, not by their MMAs).  A stage is refilled only after all three CTAs writing into it
//     released it.
//     A model of padded width 64 (reswidth 1..64, the MNIST models) has one 64-channel block per pixel half: its dense
//     convs and in-convs run the narrow tile (DenseArgs<64>) as single CTAs, one per tile.  Padded width 128 runs the
//     N = 128 tile with one channel block (DenseArgs<128>), padded width 192 the N = 64 tile with three
//     (DenseArgs<192>), both as single CTAs.  Padded widths 320, 384, 448 and 512 (reswidth 257..512) run the N = 64
//     tile with Wp / 64 channel blocks (DenseArgs<Wp>), single CTAs too.  Their dense convs and heads (HeadArgs<true>)
//     fold the main accumulator into a float32 register accumulator after every tap: K reaches 49 x 512 there, and the
//     tensor core's truncating accumulate would otherwise lose accuracy in proportion to K.
//   * the kernel size (1, 3, 5 or 7) is a run-time argument: taps = ks^2 k-blocks per input chunk, TMA's zero fill pads
//     every shift; a 1x1 in-conv tile is a single k-block.
//   * fixed k order, no split-K, no atomics: results are bit-identical for any batch size, position in the batch
//     or grid (the decoder must regenerate the encoder's tables exactly, SURVEY.md H3).
//   * single-pass bf16 arithmetic (BSW_TC_BF16, Bf16<Args>): one hi*hi MMA per k16 step into the main accumulator, no
//     cross accumulator, only the hi boxes loaded (the stage layout stays the split tile's, its lo halves unused), and only
//     the hi plane of the next conv's input written.  The hi planes are RNE(x) in both arithmetics, so the two share the
//     weights, planes and tensor maps.  Four-CTA clusters issue one box per CTA: A_hi of pixel half h by the CTA of
//     channel block h, W_hi of channel block b by the CTA of pixel half 1 - b.  Folding tiles still fold per tap.
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>
#include <type_traits>
#include <vector>
#include "bsw_common.cuh"
#include "nets.cuh"

extern "C" int bsw_has_tensor_cores(void) { return 1; }

namespace {

constexpr int BK = 32;                      // channels per k-block (64-byte rows, SWIZZLE_64B)
constexpr int MT = 128;                     // pixels per tile: two warpgroups x 64
constexpr int BN = 128;                     // output channels per tile of the W->W convs and in-convs
constexpr int NW = 64;                      // output channels per tile of a padded-width-64 model's W->W convs and in-convs
constexpr int HD_N = 32;                    // output channels of the heads (n_mu + n_sc <= 32, zero padded)
constexpr int A_BYTES = MT * BK * 2;        // one 128-row x 32-col bf16 activation tile = 8 KB
constexpr int WG_THREADS = 384;             // two consumer warpgroups + the producer / epilogue warpgroup
constexpr int PRODUCER_WARP = 8;
constexpr int EPI_WARP0 = 9, EPI_WARPS = 3; // warps 9..11: epilogue
// Registers per thread: 128 at launch (384 x 128 = 48 K of the SM's 64 K, so a coder CTA fits beside a conv CTA), then
// setmaxnreg moves them from the producer / epilogue warpgroup to the consumers: 256 x 160 + 128 x 64 = 48 K.  Both
// sides compile without spills at these counts (ptxas -v).
constexpr int REGS_CONSUMER = 160, REGS_EPILOGUE = 64;
constexpr int HD_LD = MT + 4;               // heads' hand-off row stride (floats): bank-conflict free both ways

template <int N> struct TileCfg {
    static constexpr int W_BYTES = N * BK * 2;                       // one N-row weight tile
    static constexpr int STAGE = 2 * A_BYTES + 2 * W_BYTES;          // A_hi, A_lo, B_hi, B_lo
    // 128 KB (N = 128) / 144 KB (N = 64: six 24 KB stages, 2.7 of a dense 3x3's 18 k-blocks in flight) / 100 KB
    // (N = 32) of stages
    static constexpr int NSTAGE = N == BN ? 4 : N == NW ? 6 : 5;
    // fp32 hand-off tile (main + cross) from the consumers to the epilogue warps: 64 KB (N = 128) / 32 KB (N = 64) /
    // 16.5 KB (N = 32)
    static constexpr int HAND = N == HD_N ? N * HD_LD * 4 : MT * N * 4;
    static constexpr int SMEM = NSTAGE * STAGE + HAND + 1024 /*align*/ + 256 /*barriers*/;
};
static_assert(TileCfg<BN>::SMEM <= 227 * 1024, "stages and hand-off must fit one H100 SM's shared memory");
static_assert(TileCfg<NW>::SMEM <= TileCfg<BN>::SMEM, "the narrow tile takes no more shared memory than the wide one");

struct TcState {
    // bf16 hi/lo activation planes, ping-pong: [max_batch, 256 px, 256 ch]
    __nv_bfloat16 *act[2][2];
    CUtensorMap act_map[2][2];     // box = 8 image rows (one tile's 128 pixels)
    // in-conv input: the flat `given` re-laid as NHWC bf16 hi/lo planes with the (1..12) input channels padded to 32
    __nv_bfloat16 *inp[2];
    CUtensorMap inp_map[2];
    std::vector<void *> wbufs;
};

// ---- PTX wrappers -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Arrive on the barrier at the same shared-memory offset in cluster CTA `rank` (this CTA included).  Used to release a
// stage after wgmma.wait_group has retired the MMAs that read it: no read is left in flight for a fence to order.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t *bar, uint32_t rank) {
    asm volatile(
        "{\n"
        ".reg .b32 ra;\n"
        "mapa.shared::cluster.u32 ra, %0, %1;\n"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(rank) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a mis-programmed TMA/MMA must not hang the GPU -- trap instead (surfaces as a CUDA error).
// The bound is wall time (2 s on %globaltimer, sampled every 2^14 failed polls), not a spin count: a time-sliced or
// preempted context makes honest waits arbitrarily long in spins but not in device time spent inside this kernel.
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t spins = 0;
    uint64_t t0 = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3fffu) == 0) {
            uint64_t now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 2000000000ull) __trap();
        }
    }
}
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// Multicast: the box lands at the same shared-memory offset in every cluster CTA of `mask` and completes its bytes on
// the barrier at `bar`'s offset in each of them.
__device__ __forceinline__ void tma_load_4d_mc(void *dst, const CUtensorMap *map, uint64_t *bar, uint16_t mask, int c0, int c1, int c2,
                                               int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
                 " [%0], [%1, {%4, %5, %6, %7}], [%2], %3;"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d_mc(void *dst, const CUtensorMap *map, uint64_t *bar, uint16_t mask, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
                 " [%0], [%1, {%4, %5, %6}], [%2], %3;"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t n;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
    return n;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// K-major, SWIZZLE_64B wgmma shared-memory matrix descriptor:
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (unused for swizzled K-major, 1) | [32,46) SBO >> 4 = 512 B
//   (8 rows x 64 B) | [62,64) layout type 2 = SWIZZLE_64B.  The k16 slices of a 64-byte row start 32 B apart.
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fff);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;
    return d;
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, bf16 operands from shared memory, float32 accumulators in registers.
// Accumulator layout (per warpgroup thread, warp w, lane l): d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e].
template <int N> struct Wgmma;
template <> struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "setp.ne.b32 p, %66, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
            "%64, %65, p, 1, 1, 0, 0;\n"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(1));
    }
};
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "setp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "%32, %33, p, 1, 1, 0, 0;\n"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(1));
    }
};
template <> struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "setp.ne.b32 p, %18, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
            "%16, %17, p, 1, 1, 0, 0;\n"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(1));
    }
};

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int K> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(K) : "memory"); }
// The accumulators are written asynchronously: pin every read of them after the wait that retires the writes.
template <int R> __device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ELU(x) = x > 0 ? x : exp(x) - 1 (utils/torch/modules.py:229-241 F.elu).  exp by the hardware ex2 (2 ulp of the result,
// |error| <= 2.4e-7 absolute after the subtraction): far inside the 1e-4 bar on mu/sigma (measured in the P3 tests) and
// a third of expm1f's instructions.
__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : __expf(x) - 1.0f; }

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// Dense W->W convs and in-convs of a model of padded width WP = 64, 128, ..., 512 (reswidth 1..512): the N = kN tile
// with kCoBlocks channel blocks per pixel half (tile t -> image t / (2 kCoBlocks), channel block (t >> 1) % kCoBlocks,
// pixel half t & 1).  Padded widths 128 and 256 take the N = 128 tile, every other width the N = 64 tile.  Trunk,
// residual, planes and bias are WP channels wide.  Above 256 the dense convs fold the main accumulator once per tap (see
// k_conv_wg), so it never sums more than WP terms; widths <= 256 do not fold.
template <int WP> struct DenseArgs {
    static constexpr int kN = (WP == 128 || WP == 256) ? BN : NW, kCoBlocks = WP / kN;
    static constexpr bool kFold = WP > 256;
    static constexpr bool kBf16 = false;
    int taps, ks;
    int cchunks;             // 32-channel chunks per tap: WP / 32 for the dense W->W convs, 1 for the in-convs
    const float *bias;       // [WP]
    const float *resid;      // [n,256,WP] fp32 or null
    float *T;                // trunk out or null
    int T_elu;
    __nv_bfloat16 *A_hi, *A_lo;   // next conv's input planes [n,256,WP] or null
    int A_elu;
};

// Hand-off tile of the dense convs and in-convs: s = main + cross as fp32 [128 px][N ch] (N = kN, 128 or 64), the
// 32-byte column chunks of row r XOR-swizzled by r & 3.  A row is a whole number of 128-byte bank lines, so without
// the swizzle chunk j of rows r..r+3 would sit on the same 8 banks.  The consumers' float2 writes (a half warp covers
// chunk j of 4 consecutive rows) go to chunks j ^ 0..3, and the epilogue's float4 reads (a quarter warp covers 4
// consecutive chunks of one row) to 4 chunks; either way the low two chunk bits differ -> 32 distinct banks.
template <int N> __device__ __forceinline__ int hand_idx(int r, int c) { return r * N + (((c >> 3) ^ (r & 3)) << 3) + (c & 7); }

// Folding tiles: s = (outer + main) + cross, in that order for every element, so the result does not depend on the grid.
// The other tiles pass a one-element `outer` that is never read.  BF16: s = outer + main or main (`dc` is never read).
template <bool BF16, int WP, int O>
__device__ __forceinline__ void hand_store(const DenseArgs<WP> &, float *hand, const float (&outer)[O],
                                           const float (&dm)[DenseArgs<WP>::kN / 2], const float (&dc)[DenseArgs<WP>::kN / 2],
                                           int row, int lane) {
    constexpr int N = DenseArgs<WP>::kN;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = 4 * j + 2 * h;
            float2 s;
            if constexpr (BF16 && DenseArgs<WP>::kFold) s = make_float2(outer[i] + dm[i], outer[i + 1] + dm[i + 1]);
            else if constexpr (BF16) s = make_float2(dm[i], dm[i + 1]);
            else if constexpr (DenseArgs<WP>::kFold) s = make_float2((outer[i] + dm[i]) + dc[i], (outer[i + 1] + dm[i + 1]) + dc[i + 1]);
            else s = make_float2(dm[i] + dc[i], dm[i + 1] + dc[i + 1]);
            *reinterpret_cast<float2 *>(hand + hand_idx<N>(row + 8 * h, 8 * j + 2 * (lane & 3))) = s;
        }
}

// Dense / in-conv epilogue, run by the epilogue warps from the hand-off tile: s + bias (+ residual) (-> ELU) -> trunk;
// (-> ELU) -> bf16 hi/lo planes of the next conv.  Tensors are NHWC with WP channels per pixel and the hand-off tile has
// N channels per row; ROWS = 128 / N tile rows are stored per warp step, 32 / ROWS lanes per row, 4 channels per lane
// (N = 128: 128 channels of one row per step; N = 64: two 64-channel rows), at channel block co0.  Warp ew takes row
// steps ew, ew + 3, ..., so a warp stores 512 contiguous bytes of the trunk and 256 of each plane per step.  The
// residual is the trunk itself (updated in place: resid == T): each element is read and then written by the same
// thread, and the loads of the next RD steps are issued before the current step's stores.  BF16: the hi plane only.
template <bool BF16, int WP>
__device__ __forceinline__ void epilogue(const DenseArgs<WP> &a, const float *hand, int img, int mh, int co0, int ew, int lane) {
    constexpr int N = DenseArgs<WP>::kN, ROWS = 128 / N;
    constexpr int RD = 3, LPR = 32 / ROWS;
    const int hl = lane % LPR, sub = lane / LPR;
    const float4 bq = __ldg(reinterpret_cast<const float4 *>(a.bias + co0) + hl);
    const int64_t base = ((int64_t)img * 256 + mh * 128 + sub) * WP + co0 + 4 * hl;     // + ROWS * step * WP
    const int nr = (MT / ROWS - ew + EPI_WARPS - 1) / EPI_WARPS;
    auto resid = [&](int k) {
        return (a.resid && k < nr) ? *reinterpret_cast<const float4 *>(a.resid + base + ROWS * (ew + EPI_WARPS * k) * WP)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    float4 q[RD];
#pragma unroll
    for (int d = 0; d < RD; ++d) q[d] = resid(d);
    for (int k0 = 0; k0 < nr; k0 += RD) {
#pragma unroll
        for (int d = 0; d < RD; ++d) {
            const int k = k0 + d, rs = ew + EPI_WARPS * k, r = ROWS * rs + sub;
            if (k >= nr) break;
            const float4 rq = q[d];
            q[d] = resid(k + RD);
            const float4 s = *reinterpret_cast<const float4 *>(hand + hand_idx<N>(r, 4 * hl));
            float x[4] = {s.x + bq.x, s.y + bq.y, s.z + bq.z, s.w + bq.w};
            if (a.resid) { x[0] += rq.x; x[1] += rq.y; x[2] += rq.z; x[3] += rq.w; }
            if (a.T_elu)
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = elu1(x[e]);
            const int64_t off = base + ROWS * rs * WP;
            if (a.T) *reinterpret_cast<float4 *>(a.T + off) = make_float4(x[0], x[1], x[2], x[3]);
            if constexpr (BF16) {
                if (a.A_hi) {
                    __nv_bfloat16 hi[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) hi[e] = __float2bfloat16_rn(a.A_elu ? elu1(x[e]) : x[e]);
                    *reinterpret_cast<uint2 *>(a.A_hi + off) = make_uint2(pack_bf16x2(hi[0], hi[1]), pack_bf16x2(hi[2], hi[3]));
                }
            } else if (a.A_hi) {
                __nv_bfloat16 hi[4], lo[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float y = a.A_elu ? elu1(x[e]) : x[e];
                    hi[e] = __float2bfloat16_rn(y);
                    lo[e] = __float2bfloat16_rn(y - __bfloat162float(hi[e]));
                }
                *reinterpret_cast<uint2 *>(a.A_hi + off) = make_uint2(pack_bf16x2(hi[0], hi[1]), pack_bf16x2(hi[2], hi[3]));
                *reinterpret_cast<uint2 *>(a.A_lo + off) = make_uint2(pack_bf16x2(lo[0], lo[1]), pack_bf16x2(lo[2], lo[3]));
            }
        }
    }
}

// mu/sigma heads: the 3x3 W -> (n_mu + n_sc <= 32) convolution that ends every net (cifar_train.py:349,368,411,426),
// with the scale transforms and the UnSqueeze2d index map of the x head in the epilogue.  FOLD: the heads of a model of
// padded width 320..512, where K = taps x Wp (up to 49 x 512), fold once per tap like the dense convs of that width.
template <bool FOLD> struct HeadArgs {
    static constexpr int kN = HD_N, kCoBlocks = 1;
    static constexpr bool kFold = FOLD;
    static constexpr bool kBf16 = false;
    int taps, ks;
    int cchunks;             // Wp / 32: K = taps x Wp
    const float *bias;       // [>= n_mu + n_sc]
    float *mu, *scale;
    int n_mu, n_sc, scale_kind, out_mode, out_dim;
};

__device__ __forceinline__ float hd_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float hd_softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }   // modules.py:112-114
__device__ __forceinline__ float hd_scale(float r, int kind) {      // same expressions as nets.cu scale_transform
    switch (kind) {
        case SCALE_INFER:   return 0.1f + 0.9f * hd_sigmoid(r + 2.f);                               // cifar_train.py:349,368
        case SCALE_DEEPGEN: return 0.1f + 0.9f * hd_softplus(r + 0.54132485461291810f);             // :426
        case SCALE_X:       return ((2.f / 255.f) / 8.f) + hd_softplus(r);                          // :411 / imagenetcrop :417
    }
    return r;
}

// Heads' hand-off tile: channel-major [32 ch][HD_LD], so the epilogue's lanes read consecutive pixels of one channel; the
// row stride of 132 floats also spreads the consumers' writes (8 rows x 4 channels per register) over 32 banks.  The sum
// is the dense tiles': (outer + main) + cross when folding, main + cross otherwise (BF16: without the cross term).
template <bool BF16, bool FOLD, int O>
__device__ __forceinline__ void hand_store(const HeadArgs<FOLD> &, float *hand, const float (&outer)[O], const float (&dm)[HD_N / 2],
                                           const float (&dc)[HD_N / 2], int row, int lane) {
#pragma unroll
    for (int j = 0; j < HD_N / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = 4 * j + 2 * h + e;
                float s;
                if constexpr (BF16 && FOLD) s = outer[i] + dm[i];
                else if constexpr (BF16) s = dm[i];
                else if constexpr (FOLD) s = (outer[i] + dm[i]) + dc[i];
                else s = dm[i] + dc[i];
                hand[(8 * j + 2 * (lane & 3) + e) * HD_LD + row + 8 * h] = s;
            }
}

// Heads' epilogue: lane = pixel, so the flat CHW stores dst[o * 256 + p] of a warp are coalesced.  Both arithmetics.
template <bool BF16, bool FOLD>
__device__ __forceinline__ void epilogue(const HeadArgs<FOLD> &a, const float *hand, int img, int mh, int co0, int ew, int lane) {
    float *mu_row = a.mu + (int64_t)img * a.out_dim;
    float *sc_row = a.scale ? a.scale + (int64_t)img * a.out_dim : nullptr;
    for (int r = ew * 32 + lane; r < MT; r += EPI_WARPS * 32) {
        const int p = mh * 128 + r, y = p >> 4, x = p & 15;
        for (int c = 0; c < a.n_mu + a.n_sc; ++c) {
            const bool is_mu = c < a.n_mu;
            const int o = is_mu ? c : c - a.n_mu;
            float v = hand[c * HD_LD + r] + __ldg(a.bias + co0 + c);
            if (!is_mu) v = hd_scale(v, a.scale_kind);
            float *dst = is_mu ? mu_row : sc_row;
            if (a.out_mode == OUT_HEAD_Z) dst[o * 256 + p] = v;
            else dst[(o >> 2) * 1024 + (2 * y + ((o >> 1) & 1)) * 32 + 2 * x + (o & 1)] = v;      // UnSqueeze2d, modules.py:205-207
        }
    }
}

// The tile of Args in single-pass bf16 arithmetic (BSW_TC_BF16): same arguments, shared memory and launch shape.
template <class Args> struct Bf16 : Args {
    static constexpr bool kBf16 = true;
};

// Tile t -> image t / (2 * kCoBlocks), output-channel block, pixel half (t & 1): the tiles of one image run on
// neighbouring SMs at about the same time, so the activation planes they share come out of L2.
// Launched as four-CTA clusters (DenseArgs<256> only, see the file comment), gridDim.x is a multiple of 4: t & 3 is the
// CTA's cluster rank and the four CTAs of a cluster walk the same images in step.
// Each tile's accumulators go through the shared-memory hand-off tile to the epilogue warps, so the consumers start the
// next tile's MMAs while its epilogue runs: acc_full (256 consumer threads arrive) publishes the tile, acc_empty (96
// epilogue threads arrive after their last read of it) frees it.
template <class Args>
__global__ void __maxnreg__(128)
k_conv_wg(const __grid_constant__ CUtensorMap amap_hi, const __grid_constant__ CUtensorMap amap_lo,
          const __grid_constant__ CUtensorMap wmap_hi, const __grid_constant__ CUtensorMap wmap_lo, const Args a, int ntiles) {
#include "conv_wg_body.cuh"
}
// The same tile in single-pass bf16 arithmetic (Args = Bf16<DenseArgs<WP>> or Bf16<HeadArgs<FOLD>>), a kernel of its own name.
template <class Args>
__global__ void __maxnreg__(128)
k_conv_bf16(const __grid_constant__ CUtensorMap amap_hi, const __grid_constant__ CUtensorMap amap_lo,
            const __grid_constant__ CUtensorMap wmap_hi, const __grid_constant__ CUtensorMap wmap_lo, const Args a, int ntiles) {
#include "conv_wg_body.cuh"
}
// The kernel of tile type Args.
template <class Args> auto conv_kernel() {
    if constexpr (Args::kBf16) return k_conv_bf16<Args>;
    else return k_conv_wg<Args>;
}

// float32 NHWC -> bf16 hi/lo planes (used once per net, after the SIMT in-conv)
__global__ void k_split_planes(const float *__restrict__ in, __nv_bfloat16 *__restrict__ hi, __nv_bfloat16 *__restrict__ lo, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = in[i];
    __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(x - __bfloat162float(h));
}

// cuTensorMapEncodeTiled through the runtime's driver entry point: the library must load (and export its
// symbols) on machines without libcuda.so.1, e.g. the CPU-only build container.
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// flat CHW `given` (float32) -> NHWC bf16 hi/lo planes with 32 channels (zero padded).  mode IN_CHW_Z: channel c at
// given[c*256 + p]; IN_CHW_X: Squeeze2d(2) on the fly, channel c*4+fh*2+fw <- pixel (2h+fh, 2w+fw) of image channel c
// (utils/torch/modules.py:183-185).
__global__ void k_given_to_planes(const float *__restrict__ given, int in_dim, int cin, int mode, __nv_bfloat16 *__restrict__ hi,
                                  __nv_bfloat16 *__restrict__ lo, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one thread per (image, pixel, channel)
    if (i >= n * 256 * 32) return;
    int ch = (int)(i & 31);
    int p = (int)((i >> 5) & 255);
    int64_t img = i >> 13;
    float x = 0.f;
    if (ch < cin) {
        const float *src = given + img * in_dim;
        int y = p >> 4, xx = p & 15;
        x = (mode == IN_CHW_Z) ? src[ch * 256 + p] : src[(ch >> 2) * 1024 + (2 * y + ((ch >> 1) & 1)) * 32 + 2 * xx + (ch & 1)];
    }
    __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(x - __bfloat162float(h));
}

int encode_map(CUtensorMap *m, void *base, int rank, const cuuint64_t *dims, const cuuint64_t *strides_bytes,
               const cuuint32_t *box) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        BSW_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
        if (!p || qres != cudaDriverEntryPointSuccess) {
            bsw_set_error("cuTensorMapEncodeTiled not available from this driver");
            return BSW_E_CUDA;
        }
        fn = (EncodeTiledFn)p;
    }
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, base, dims, strides_bytes, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        bsw_set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
        return BSW_E_CUDA;
    }
    return BSW_OK;
}

// Calls f(DenseArgs<Wp>{}) for the run-time padded width Wp: the one list of the widths the tensor-core convs run.
template <class F> int with_width(int Wp, F &&f) {
    switch (Wp) {
        case 64:  return f(DenseArgs<64>{});
        case 128: return f(DenseArgs<128>{});
        case 192: return f(DenseArgs<192>{});
        case 256: return f(DenseArgs<256>{});
        case 320: return f(DenseArgs<320>{});
        case 384: return f(DenseArgs<384>{});
        case 448: return f(DenseArgs<448>{});
        case 512: return f(DenseArgs<512>{});
    }
    BSW_REQUIRE(false, "tensor-core conv path needs a padded width of 64, 128, ..., 512 (reswidth 1..512)");
}

// Calls f(Args{}) with the dense tile of the model's padded width in the model's arithmetic: DenseArgs<Wp>, or
// Bf16<DenseArgs<Wp>> when bsw_model_set_tc_precision chose BSW_TC_BF16.  The heads take HeadT<Args>.
template <class F> int with_tile(const bsw_model *m, F &&f) {
    return with_width(m->Wp, [&](auto t) { return m->tc_precision == BSW_TC_BF16 ? f(Bf16<decltype(t)>{}) : f(t); });
}
template <class Args> using HeadT = std::conditional_t<Args::kBf16, Bf16<HeadArgs<Args::kFold>>, HeadArgs<Args::kFold>>;

}  // namespace

struct TcSlot { CUtensorMap map_hi, map_lo; };

int bsw_model_tc_prepare(bsw_model *m) {
    const int Wp = m->Wp;
    // The dense / in-conv and head kernels of the model's width, with one SM-wide L1/shared split for every kernel of
    // the path (see bsw_prefer_max_shared).  dense_n: output channels per tile of the dense convs and in-convs.
    int dense_n = 0;
    if (int rc = with_width(Wp, [&](auto t) {
            using Args = decltype(t);
            using Head = HeadArgs<Args::kFold>;
            dense_n = Args::kN;
            BSW_CUDA(cudaFuncSetAttribute(k_conv_wg<Args>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileCfg<Args::kN>::SMEM));
            BSW_CUDA(cudaFuncSetAttribute(k_conv_wg<Head>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileCfg<HD_N>::SMEM));
            bsw_prefer_max_shared(k_conv_wg<Args>);
            bsw_prefer_max_shared(k_conv_wg<Head>);
            // the bf16 tiles: same shared memory (bsw_model_set_tc_precision may switch at any net call)
            BSW_CUDA(cudaFuncSetAttribute(k_conv_bf16<Bf16<Args>>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileCfg<Args::kN>::SMEM));
            BSW_CUDA(cudaFuncSetAttribute(k_conv_bf16<Bf16<Head>>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileCfg<HD_N>::SMEM));
            bsw_prefer_max_shared(k_conv_bf16<Bf16<Args>>);
            bsw_prefer_max_shared(k_conv_bf16<Bf16<Head>>);
            return BSW_OK;
        }))
        return rc;
    bsw_prefer_max_shared(k_given_to_planes);
    TcState *ts = new TcState();
    m->tc_state = ts;
    const size_t act_elems = (size_t)m->d.max_batch * 256 * Wp;
    for (int b = 0; b < 2; ++b)
        for (int pl = 0; pl < 2; ++pl) {
            BSW_CUDA(cudaMalloc(&ts->act[b][pl], act_elems * sizeof(__nv_bfloat16)));
            BSW_CUDA(cudaMemset(ts->act[b][pl], 0, act_elems * sizeof(__nv_bfloat16)));
            cuuint64_t dims[4] = {(cuuint64_t)Wp, 16, 16, (cuuint64_t)m->d.max_batch};
            cuuint64_t str[3] = {(cuuint64_t)Wp * 2, (cuuint64_t)16 * Wp * 2, (cuuint64_t)256 * Wp * 2};
            cuuint32_t box[4] = {BK, 16, 8, 1};
            if (int rc = encode_map(&ts->act_map[b][pl], ts->act[b][pl], 4, dims, str, box)) return rc;
        }
    for (int pl = 0; pl < 2; ++pl) {
        size_t elems = (size_t)m->d.max_batch * 256 * 32;
        BSW_CUDA(cudaMalloc(&ts->inp[pl], elems * sizeof(__nv_bfloat16)));
        cuuint64_t dims[4] = {32, 16, 16, (cuuint64_t)m->d.max_batch};
        cuuint64_t str[3] = {32 * 2, 16 * 32 * 2, 256 * 32 * 2};
        cuuint32_t box[4] = {BK, 16, 8, 1};
        if (int rc = encode_map(&ts->inp_map[pl], ts->inp[pl], 4, dims, str, box)) return rc;
    }
    // weights: [tap][o=rows][c=Kc] bf16 hi/lo planes, K (=c) innermost; Kc = Wp for the dense convs and heads, 32 for the
    // in-convs; rows = Wp for the dense convs and in-convs, 32 for the heads
    std::vector<TcSlot> *slots = new std::vector<TcSlot>();
    std::vector<char> is_in(m->convs.size(), 0), is_head(m->convs.size(), 0);
    for (auto &np : m->infer) { is_in[np.in_conv] = 1; is_head[np.head] = 1; }
    for (auto &np : m->gen) { is_in[np.in_conv] = 1; is_head[np.head] = 1; }
    for (size_t ci_ = 0; ci_ < m->convs.size(); ++ci_) {
        ConvSlot &c = m->convs[ci_];
        // by role, not by shape alone: on a narrow model an in-conv (zchannels = reswidth) or a head (2 zchannels =
        // reswidth) can have the dense convs' W -> W shape
        bool dense = !is_in[ci_] && !is_head[ci_] && c.Cin == m->d.reswidth && c.Cout == m->d.reswidth;
        bool inconv = is_in[ci_] && c.Cin <= 32 && c.Cout == m->d.reswidth;
        bool head = is_head[ci_] && !dense && c.Cin == m->d.reswidth && c.Cout <= HD_N;
        if (!dense && !inconv && !head) continue;
        BSW_REQUIRE(!c.host_w.empty(), "tc_prepare: host weights already released");
        const int taps = c.ks * c.ks;
        const int Kc = inconv ? 32 : Wp;
        const int rows = head ? HD_N : Wp;               // output-channel rows per tap (heads: zero padded to 32)
        std::vector<__nv_bfloat16> hi((size_t)taps * rows * Kc), lo(hi.size());
        for (int tp = 0; tp < taps; ++tp)
            for (int ci = 0; ci < Kc; ++ci)
                for (int o = 0; o < rows; ++o) {
                    float w = (ci < c.CinP && o < c.CoutP) ? c.host_w[((size_t)tp * c.CinP + ci) * c.CoutP + o] : 0.f;
                    __nv_bfloat16 h = __float2bfloat16_rn(w);
                    size_t idx = ((size_t)tp * rows + o) * Kc + ci;
                    hi[idx] = h;
                    lo[idx] = __float2bfloat16_rn(w - __bfloat162float(h));
                }
        BSW_CUDA(cudaMalloc(&c.w_hi, hi.size() * 2));
        BSW_CUDA(cudaMalloc(&c.w_lo, lo.size() * 2));
        BSW_CUDA(cudaMemcpy(c.w_hi, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
        BSW_CUDA(cudaMemcpy(c.w_lo, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
        ts->wbufs.push_back(c.w_hi);
        ts->wbufs.push_back(c.w_lo);
        TcSlot s;
        cuuint64_t dims[3] = {(cuuint64_t)Kc, (cuuint64_t)rows, (cuuint64_t)taps};
        cuuint64_t str[2] = {(cuuint64_t)Kc * 2, (cuuint64_t)rows * Kc * 2};
        cuuint32_t box[3] = {BK, (cuuint32_t)(head ? HD_N : dense_n), 1};
        if (int rc = encode_map(&s.map_hi, c.w_hi, 3, dims, str, box)) return rc;
        if (int rc = encode_map(&s.map_lo, c.w_lo, 3, dims, str, box)) return rc;
        c.tc_index = (int)slots->size();
        slots->push_back(s);
    }
    m->tc_slots = slots;
    m->tc_ready = true;
    return BSW_OK;
}

void bsw_model_tc_release(bsw_model *m) {
    TcState *ts = (TcState *)m->tc_state;
    if (!ts) return;
    for (int b = 0; b < 2; ++b)
        for (int pl = 0; pl < 2; ++pl) cudaFree(ts->act[b][pl]);
    for (int pl = 0; pl < 2; ++pl) cudaFree(ts->inp[pl]);
    for (void *p : ts->wbufs) cudaFree(p);
    delete ts;
    delete (std::vector<TcSlot> *)m->tc_slots;
    m->tc_state = nullptr;
    m->tc_slots = nullptr;
}

// Plane buffer addressing for nets.cu: which == 0 -> the "A" ping-pong buffer, 1 -> "B".
void bsw_tc_planes(bsw_model *m, int which, void **hi, void **lo) {
    TcState *ts = (TcState *)m->tc_state;
    *hi = ts->act[which][0];
    *lo = ts->act[which][1];
}

int bsw_tc_split(bsw_model *m, const float *in, int which, int64_t n, cudaStream_t st) {
    TcState *ts = (TcState *)m->tc_state;
    int64_t cnt = n * 256 * m->Wp;
    k_split_planes<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(in, ts->act[which][0], ts->act[which][1], cnt);
    BSW_LAUNCH_CHECK();
    return BSW_OK;
}

// Launch shape of the convolutions, a bit mask -- 1 / 2 = dense convs of kernel size <= 3 / >= 5 (1x1 and 3x3 go with
// 3x3, 7x7 with 5x5), 4 = in-convs and heads on a persistent grid (one CTA or cluster per SM / cluster slot walking the
// tiles, the TMA ring prefetching across tile boundaries); a clear bit means one CTA per tile.  8 = the dense convs and
// in-convs without TMA multicast: single CTAs, each loading its whole stage; it has no effect on a model of padded width
// other than 256, whose tiles always run as single CTAs.  Default 7
// (BSW_TC_PERSIST overrides).  Same tiles, same k order per tile: results are bit-identical in every mode.
static int g_tc_mode = -1;
static int tc_mode() {
    static const int env = getenv("BSW_TC_PERSIST") ? atoi(getenv("BSW_TC_PERSIST")) : 7;
    return (g_tc_mode < 0) ? env : g_tc_mode;
}
static bool tc_persistent(int which) { return (tc_mode() & which) != 0; }
extern "C" int bsw_set_conv_mode(int mode) {
    BSW_REQUIRE(mode >= -1 && mode <= 15, "bsw_set_conv_mode: -1 (default) or a mask of 1 | 2 | 4 (persistent grid: dense 3x3, 5x5, "
                                          "in-convs and heads) | 8 (no TMA multicast)");
    g_tc_mode = mode;
    return BSW_OK;
}
static int cur_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev < 0 || dev >= 64) ? 0 : dev;
}
static unsigned tc_grid(int ntiles, bool persistent) {   // one CTA per tile, or one per SM of the current device
    static int sms[64] = {0};
    if (!persistent) return (unsigned)ntiles;
    const int dev = cur_device();
    if (!sms[dev]) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        sms[dev] = v > 0 ? v : 132;
    }
    return (unsigned)(ntiles < sms[dev] ? ntiles : sms[dev]);
}

// One dense conv or in-conv on the tile of the model's padded width and arithmetic, reading the planes behind amap_hi /
// amap_lo (bf16: amap_hi only);
// cchunks = 32-channel chunks per tap of those planes.  The tile with two channel blocks (padded width 256) runs one
// four-CTA cluster per image (TMA multicast, see k_conv_wg), or single CTAs with mode bit 8; its persistent grid is as
// many clusters as the device holds at once (GPCs of 16-18 SMs leave some SMs out), cluster c walking images c, c + C,
// ...  Every other tile runs single CTAs, one per tile or a persistent grid of one per SM.
static int launch_dense(bsw_model *m, const CUtensorMap &amap_hi, const CUtensorMap &amap_lo, const TcSlot &s,
                        const ConvSlot &c, const ConvArgs &a, const float *resid, int cchunks, int64_t n, bool persistent,
                        cudaStream_t st) {
    TcState *ts = (TcState *)m->tc_state;
    return with_tile(m, [&](auto t) {
        using Args = decltype(t);
        t.taps = c.ks * c.ks; t.ks = c.ks; t.cchunks = cchunks;
        t.bias = c.bias; t.resid = resid; t.T = a.T; t.T_elu = a.T_elu;
        t.A_hi = a.A_planes >= 0 ? ts->act[a.A_planes][0] : nullptr;
        t.A_lo = a.A_planes >= 0 && !Args::kBf16 ? ts->act[a.A_planes][1] : nullptr;
        t.A_elu = a.A_elu;
        const int ntiles = (int)n * 2 * Args::kCoBlocks;
        if constexpr (Args::kCoBlocks == 2) {
            static int clusters[64] = {0};
            const bool mc = (tc_mode() & 8) == 0;
            cudaLaunchAttribute attr;
            attr.id = cudaLaunchAttributeClusterDimension;
            attr.val.clusterDim.x = 4; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)ntiles);
            cfg.blockDim = dim3(WG_THREADS);
            cfg.dynamicSmemBytes = TileCfg<Args::kN>::SMEM;
            cfg.stream = st;
            cfg.attrs = &attr;
            cfg.numAttrs = mc ? 1 : 0;
            if (persistent && !mc) cfg.gridDim = dim3(tc_grid(ntiles, true));
            if (persistent && mc) {
                const int dev = cur_device();
                if (!clusters[dev]) {
                    int v = 0;
                    BSW_CUDA(cudaOccupancyMaxActiveClusters(&v, conv_kernel<Args>(), &cfg));
                    BSW_REQUIRE(v > 0, "launch_dense: a cluster of four conv CTAs does not fit this device");
                    clusters[dev] = v;
                }
                cfg.gridDim = dim3(4u * (unsigned)(n < clusters[dev] ? n : clusters[dev]));
            }
            BSW_CUDA(cudaLaunchKernelEx(&cfg, conv_kernel<Args>(), amap_hi, amap_lo, s.map_hi, s.map_lo, t, ntiles));
        } else {
            conv_kernel<Args>()<<<tc_grid(ntiles, persistent), WG_THREADS, TileCfg<Args::kN>::SMEM, st>>>(amap_hi, amap_lo, s.map_hi,
                                                                                                          s.map_lo, t, ntiles);
            BSW_LAUNCH_CHECK();
        }
        return BSW_OK;
    });
}

// a.in must be one of the plane buffers: a.in_planes = 0/1 selects it; outputs a.A_planes = 0/1/-1.
int bsw_conv_tc(bsw_model *m, const ConvSlot &c, const ConvArgs &a, int64_t n, cudaStream_t st) {
    TcState *ts = (TcState *)m->tc_state;
    BSW_REQUIRE(ts && c.tc_index >= 0, "bsw_conv_tc: conv has no tensor-core weights");
    const TcSlot &s = (*(std::vector<TcSlot> *)m->tc_slots)[c.tc_index];
    return launch_dense(m, ts->act_map[a.in_planes][0], ts->act_map[a.in_planes][1], s, c, a, a.resid, m->Wp / BK, n,
                        tc_persistent(c.ks <= 3 ? 1 : 2), st);
}

// Heads: reads the planes the last ResNet conv wrote (in_planes), writes mu / sigma.  BSW_TC_HEADS=0 keeps the float32 SIMT
// kernel (A/B runs).
bool bsw_conv_tc_head_available(bsw_model *m, const ConvSlot &c) {
    static const bool off = getenv("BSW_TC_HEADS") && getenv("BSW_TC_HEADS")[0] == '0';
    return !off && m->tc_ready && c.tc_index >= 0 && c.Cout <= HD_N && c.Cin == m->d.reswidth;
}
int bsw_conv_tc_head(bsw_model *m, const ConvSlot &c, const ConvArgs &a, int64_t n, cudaStream_t st) {
    TcState *ts = (TcState *)m->tc_state;
    BSW_REQUIRE(ts && c.tc_index >= 0 && a.n_mu + a.n_sc <= HD_N, "bsw_conv_tc_head: conv has no tensor-core head weights");
    const TcSlot &s = (*(std::vector<TcSlot> *)m->tc_slots)[c.tc_index];
    const int ntiles = (int)n * 2;
    const unsigned grid = tc_grid(ntiles, tc_persistent(4));
    return with_tile(m, [&](auto t) {
        using Head = HeadT<decltype(t)>;                 // the heads fold where the model's dense convs do
        Head h;
        h.taps = c.ks * c.ks; h.ks = c.ks; h.cchunks = m->Wp / BK; h.bias = c.bias; h.mu = a.mu; h.scale = a.scale; h.n_mu = a.n_mu; h.n_sc = a.n_sc;
        h.scale_kind = a.scale_kind; h.out_mode = a.out_mode; h.out_dim = a.out_dim;
        conv_kernel<Head>()<<<grid, WG_THREADS, TileCfg<HD_N>::SMEM, st>>>(ts->act_map[a.in_planes][0], ts->act_map[a.in_planes][1],
                                                                        s.map_hi, s.map_lo, h, ntiles);
        BSW_LAUNCH_CHECK();
        return BSW_OK;
    });
}

// In-conv on the tensor cores: `given` (flat CHW float32) -> 32-channel bf16 planes -> k_conv_wg with one channel chunk
// per tap.  Epilogue as for every conv: T = ELU(raw) (the trunk), A planes = ELU(T) for the first ResNet layer.
int bsw_conv_tc_in(bsw_model *m, const ConvSlot &c, const ConvArgs &a, int64_t n, cudaStream_t st, int *launches) {
    TcState *ts = (TcState *)m->tc_state;
    BSW_REQUIRE(ts && c.tc_index >= 0, "bsw_conv_tc_in: conv has no tensor-core weights");
    const TcSlot &s = (*(std::vector<TcSlot> *)m->tc_slots)[c.tc_index];
    int64_t cnt = n * 256 * 32;
    k_given_to_planes<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(a.in, a.in_dim, c.Cin, a.in_mode, ts->inp[0], ts->inp[1], n);
    BSW_LAUNCH_CHECK();
    if (int rc = launch_dense(m, ts->inp_map[0], ts->inp_map[1], s, c, a, nullptr, 1, n, tc_persistent(4), st)) return rc;
    *launches += 2;
    return BSW_OK;
}
