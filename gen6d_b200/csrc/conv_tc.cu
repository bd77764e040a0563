// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, sm_90a), fp32-faithful through a
// three-term operand split:  A*B ~= A_hi*B_hi + A_hi*B_lo + A_lo*B_hi, x_hi = round(x) to an 11-bit
// significand, x_lo = x - x_hi (exact in fp32).  The dropped A_lo*B_lo term is O(2^-22) relative, so
// index selections (detection cell, viewpoint) stay bit-exact against the fp32 reference while the
// contraction runs on the tensor pipe instead of the FFMA pipe.  Two operand kinds share every kernel:
//
//   G6D_TC_TF32  hi/lo are tf32 (fp32 containers, 8-bit exponent): any fp32 range, tf32 wgmmas
//                (K = 8 per instruction, 32 K-elements per 128-byte swizzle row);
//   G6D_TC_F16   hi = fp16(x), lo = fp16((x - hi) * 2^11): the same 11 + 11 significand bits, but
//                f16 wgmmas issue K = 16 per instruction at twice the tf32 rate and every operand
//                byte (shared-memory tile, TMA weight stream, operand re-read) carries twice the K:
//                2x the tensor ceiling and half the shared-memory traffic per flop.  The lo halves are
//                pre-scaled by 2^11 so that they live in the same exponent range as the hi halves (no
//                fp16 subnormals); both cross terms accumulate in their own accumulator, which the
//                epilogue folds in with an exact 2^-11.  Range contract: |x| <= 65504 for activations
//                and weights (saturating conversion beyond that), full relative accuracy for |x| >=
//                6.1e-5, absolute error <= ~2^-36 below.  Inside this network every tensor-core operand
//                is a BN-folded weight, a post-ReLU / InstanceNorm-ed / L2-normalised activation or a
//                VGG feature, all O(1e-3 .. 1e3).  G6D_CONV_KIND=tf32 selects the wide-range kind.
//
// GEMM view (same as conv_ffma.cu): M = B*Do*Ho*Wo, N = Cout, K = taps*Cin, channels-last.
// One CTA computes 128 x BLOCK_N output tiles, 64 rows per consumer warpgroup (wgmma M = 64,
// accumulators in registers).  16 warps:
//   warps 0-7   A producers: gather the im2col rows of the K-block from global memory (coalesced
//               128-bit loads, register prefetch ring; 16 rows per warp), apply the folded
//               InstanceNorm(+ReLU) / selector q(.)ref prologue to in-bounds elements, split into hi/lo
//               and st.shared both tiles in the canonical K-major SWIZZLE_128B layout the wgmma
//               descriptor expects (conv_tc2_kernel with a split input: one thread loads the same tiles
//               by TMA im2col instead, see split_input_ok);
//   warps 8-15  two consumer warpgroups, rows 0-63 and 64-127 of the tile, both reading the same
//               weight tiles of a stage: 12 wgmmas per K-block each (4 K-steps x 3 split terms),
//               one group in flight while the next stage is awaited, then the
//               epilogue (bias / activation -> global, or split-K partials) straight from the
//               accumulator registers.  The first consumer thread also streams the pre-split weight
//               tiles W_hi / W_lo [Cout, K] (K-major) by TMA (cp.async.bulk.tensor.2d, 128B swizzle)
//               into the stages the consumers free (with a split input, the thread that loads A does).
// A consumer's accumulators alone take 128 registers, the launch bound of 512 threads allows 128 per
// thread: the producer warpgroups give registers up (setmaxnreg.dec to TC_PRODUCER_REGS) and the
// consumer warpgroups take them (setmaxnreg.inc to TC_CONSUMER_REGS); ptxas allocates the code after
// each setmaxnreg within its new count.
// conv_tc2_kernel handles general strides / shapes (persistent); conv_tcflat_kernel (stride-1
// multi-tap convolutions whose halo fits in shared memory) reuses the A operand across taps, see below.
#include <cuda_fp16.h>
#include <string.h>

#include "tc_common.cuh"

namespace g6d {

constexpr int TC_BM = 128;                                 // rows per tile: 64 (wgmma M) per consumer warpgroup
constexpr int TC_PRODUCER_WARPS = 8;
constexpr int TC_CONSUMER_WARPS = 8;                       // two warpgroups
constexpr int TC_THREADS = (TC_PRODUCER_WARPS + TC_CONSUMER_WARPS) * 32;
constexpr int TC_ISSUER = TC_PRODUCER_WARPS * 32;          // consumer thread that also issues the weight TMA
constexpr int TC_PRODUCER_REGS = 96, TC_CONSUMER_REGS = 160;
static_assert(TC_PRODUCER_WARPS * TC_PRODUCER_REGS + TC_CONSUMER_WARPS * TC_CONSUMER_REGS <= 65536 / 32, "register file of one SM");
// Folded K splits (G6D_TC_FOLD_SPLITS, split input only): one producer thread issues every load, so the producer warps
// give up most of their registers and each consumer thread keeps the tile's running sum (BN / 2 more) in registers.
constexpr int TC_FOLD_PRODUCER_REGS = 40, TC_FOLD_CONSUMER_REGS = 216;
static_assert(TC_PRODUCER_WARPS * TC_FOLD_PRODUCER_REGS + TC_CONSUMER_WARPS * TC_FOLD_CONSUMER_REGS <= 65536 / 32, "register file of one SM");
static_assert(TC_BM == 64 * (TC_CONSUMER_WARPS / 4), "one 64-row wgmma tile per consumer warpgroup");
constexpr int TC_MAX_K_PER_CHAIN = 2048;                   // longest accumulate chain per CTA (see fill_tc_params)

template <int KIND> struct KindCfg;
template <> struct KindCfg<G6D_TC_TF32> {
    static constexpr int BK = 32;          // K elements per 128-byte swizzle row
    static constexpr int NV = 1;           // float4 loads per (thread, row) chunk of 16 smem bytes
    static constexpr float CROSS = 1.f;    // scale of the cross-term accumulator
};
template <> struct KindCfg<G6D_TC_F16> {
    static constexpr int BK = 64;
    static constexpr int NV = 2;
    static constexpr float CROSS = 1.f / 2048.f;
};
constexpr float F16_LO_SCALE = 2048.f;
// The producers' register prefetch ring holds one float4 column (ROWS rows x 16 bytes of fp32 input) per
// slot, i.e. a K-block of fp32 or half a K-block of fp16 operands; RING - 1 slots are in flight while one
// is transformed and stored.  The persistent kernel's producers also keep per-row coordinates, so within
// TC_PRODUCER_REGS they hold two slots (16 KB in flight per SM) and the A-reuse kernel's three (32 KB).
constexpr int TC2_RING = 2, FLAT_RING = 3;
// K order inside a 64-element fp16 K-block.  A producer thread fills one 16-byte shared-memory chunk
// (8 halves) of a tile row from two 128-bit global loads; to keep BOTH loads of a warp fully coalesced
// (8 lanes x 16 B = one 128-byte line per row) lane c reads channels [4c, 4c+4) and [32+4c, 32+4c+4), so
// chunk c holds those eight channels.  The contraction does not care about the order of K as long as the
// weight operand uses the same one: the pack / split kernels write K position p from source channel
// f16_k_source(p).  (ncu, round 2: with adjacent channels per lane every gather touched 8 lines per
// instruction instead of 4 -- twice the L1 tag requests and L2 sectors of the ideal.)
__host__ __device__ __forceinline__ int f16_k_source(int p) {      // p in [0, 64)
    const int c = p >> 3, i = p & 7;
    return i < 4 ? 4 * c + i : 32 + 4 * c + (i - 4);
}

struct ConvTcP {
    const float* x; const float* bias; const float* ps; const float* pb;
    float* y; float* ws;
    int B, D, H, W, Cin, ics, ico, Cout, kd, kh, kw, stride, pd, ph, pw, Do, Ho, Wo, ocs, oco, pro, act;
    long long group_rows;
    int M, K, kblocks, splits, kb_per_split;
    double* stats; long long stats_rows;      // fused InstanceNorm statistics of the OUTPUT (see epilogue_stats)
    int split_in;                             // A tiles by TMA im2col from the pre-split input (see split_input_ok)
    int reuse_order;                          // K-blocks in the A-reuse kernel's order (G6D_TC_REUSE_IM2COL, see kblock_src)
    int fold;                                 // a work item is a tile whose K splits one CTA sums (G6D_TC_FOLD_SPLITS)
    int xr, Wp, Mp, xr_rows;                  // one A box per row of taps (see xr_ok): padded width, rows, box pixels
};

// Filter tap (kz, ky, kx flattened) and 64-channel block of K-block `it` of split `sp` when the input is split
// (K = tap * Cin + c).  Default: tap-major over the whole K.  reuse_order: the A-reuse kernel's order -- splits
// over channel blocks, then per channel block kz, then the (ky, kx) tap -- so that every output element sums the
// same products into the same accumulators in the same order as conv_tcflat_kernel.
__device__ __forceinline__ void kblock_src(const ConvTcP& p, int sp, int it, int& tap, int& cb) {
    if (p.reuse_order) {
        const int taps2 = p.kh * p.kw;
        const int u = it / taps2, t = it - u * taps2;            // unit (channel block, kz), tap (ky, kx)
        cb = sp * (p.kb_per_split / (taps2 * p.kd)) + u / p.kd;
        tap = (u % p.kd) * taps2 + t;
    } else {
        const int cblocks = p.Cin / 64, kb = sp * p.kb_per_split + it;
        tap = kb / cblocks;
        cb = kb - tap * cblocks;
    }
}

// The (tap, channel block) sequence of one chain, stepped K-block by K-block in kblock_src's order without its divides:
// the split-input TMA thread issues every load of the CTA alone, so its per-K-block integer work is on the critical path
// of the whole pipeline.  The tap is kept as (kx, ky, kz); start() pays the divides once per chain.
struct KbIter {
    int kx, ky, kz, cb;
    __device__ __forceinline__ void start(const ConvTcP& p, int sp, int it) {
        int tap;
        kblock_src(p, sp, it, tap, cb);
        kx = tap % p.kw;
        const int tq = tap / p.kw;
        ky = tq % p.kh;
        kz = tq / p.kh;
    }
    __device__ __forceinline__ void next(const ConvTcP& p) {
        if (p.reuse_order) {                                 // channel block, then kz, then (ky, kx)
            if (++kx < p.kw) return;
            kx = 0;
            if (++ky < p.kh) return;
            ky = 0;
            if (++kz < p.kd) return;
            kz = 0; ++cb;
        } else {                                             // tap-major, channel blocks innermost
            if (++cb < p.Cin / 64) return;
            cb = 0;
            if (++kx < p.kw) return;
            kx = 0;
            if (++ky < p.kh) return;
            ky = 0; ++kz;
        }
    }
    __device__ __forceinline__ int tap(const ConvTcP& p) const { return (kz * p.kh + ky) * p.kw + kx; }
};

// ------------------------------------------------------------------------------------------ operand split
// fp16 pair (element 0 in the low half, as laid out in memory), saturating instead of overflowing to inf
__device__ __forceinline__ uint32_t cvt_f16x2_sat(float e0, float e1) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(e1), "f"(e0));
    return r;
}
__device__ __forceinline__ void split_f16x2(float e0, float e1, uint32_t& hi, uint32_t& lo) {
    hi = cvt_f16x2_sat(e0, e1);
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    // (x - hi) is exact in fp32 and so is the power-of-two scaling
    lo = cvt_f16x2_sat((e0 - hf.x) * F16_LO_SCALE, (e1 - hf.y) * F16_LO_SCALE);
}
// tf32: hi = round-to-nearest (ties away) of the fp32 significand to 10 bits with integer ops (same
// as cvt.rna.tf32.f32 for finite values), lo = v - hi (exact; the tensor core ignores its low 13 bits)
__device__ __forceinline__ void split_tf32x4(const float4 v, float4& hi, float4& lo) {
    hi.x = __uint_as_float((__float_as_uint(v.x) + 0x1000u) & 0xFFFFE000u);
    hi.y = __uint_as_float((__float_as_uint(v.y) + 0x1000u) & 0xFFFFE000u);
    hi.z = __uint_as_float((__float_as_uint(v.z) + 0x1000u) & 0xFFFFE000u);
    hi.w = __uint_as_float((__float_as_uint(v.w) + 0x1000u) & 0xFFFFE000u);
    lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_v2(uint32_t addr, uint32_t a, uint32_t b) {
    asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
// float4 e (< NV) of the 16-byte chunk of a tile row: fp32 input -> hi and lo tiles (all 16 bytes for tf32,
// bytes [8e, 8e + 8) for fp16)
template <int KIND>
__device__ __forceinline__ void split_store(uint32_t hi_addr, uint32_t lo_addr, const float4 v, int e) {
    if constexpr (KIND == G6D_TC_TF32) {
        float4 hi, lo;
        split_tf32x4(v, hi, lo);
        st_shared_v4(hi_addr, __float_as_uint(hi.x), __float_as_uint(hi.y), __float_as_uint(hi.z), __float_as_uint(hi.w));
        st_shared_v4(lo_addr, __float_as_uint(lo.x), __float_as_uint(lo.y), __float_as_uint(lo.z), __float_as_uint(lo.w));
    } else {
        uint32_t h[2], l[2];
        split_f16x2(v.x, v.y, h[0], l[0]);
        split_f16x2(v.z, v.w, h[1], l[1]);
        st_shared_v2(hi_addr + 8 * e, h[0], h[1]);
        st_shared_v2(lo_addr + 8 * e, l[0], l[1]);
    }
}
// 128 pixels x 64 fp16 channels of a 4-D NHWC tensor by TMA im2col: the pixels the traversal of the map's
// bounding box reaches from (w, h, n), each shifted by the filter tap (ox, oy), one 128-byte swizzled row each;
// pixels outside the tensor arrive as zeros
__device__ __forceinline__ void tma_im2col_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c, int w, int h, int n,
                                              uint16_t ox, uint16_t oy) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(ox), "h"(oy) : "memory");
}
// the same over a 5-D NDHWC tensor: the traversal runs over (w, h, d, n), the tap is (ox, oy, oz)
__device__ __forceinline__ void tma_im2col_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c, int w, int h, int d,
                                              int n, uint16_t ox, uint16_t oy, uint16_t oz) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2], {%8, %9, %10};"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "h"(ox), "h"(oy), "h"(oz) : "memory");
}

__device__ __forceinline__ float4 affine4(float4 x, const float4 sc, const float4 sh, bool relu) {
    x.x = fmaf(x.x, sc.x, sh.x); x.y = fmaf(x.y, sc.y, sh.y); x.z = fmaf(x.z, sc.z, sh.z); x.w = fmaf(x.w, sc.w, sh.w);
    if (relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
    return x;
}
// The prologue (pro != G6D_PRO_NONE) of input channels [c, c + 4) of an in-bounds element of image b at spatial
// offset sp (within its plane): G6D_PRO_CORR scales by ps[sp, c] and shifts by pb[c], G6D_PRO_AFFINE(_RELU) by
// ps / pb[b / group_rows, c].  The persistent kernel's producers and split_input_f16_kernel both transform
// their elements here, so a pre-normalised split input holds the bytes the producers would store.
__device__ __forceinline__ float4 prologue4(float4 x, int pro, const float* __restrict__ ps, const float* __restrict__ pb,
                                            int Cin, long long group_rows, long long b, long long sp, int c) {
    const float4* scp; const float4* shp;
    if (pro == G6D_PRO_CORR) {
        scp = reinterpret_cast<const float4*>(ps + sp * Cin + c);
        shp = reinterpret_cast<const float4*>(pb + c);
    } else {
        const long long g = (int)b / (int)group_rows;               // 32-bit divide (the host checks the range)
        scp = reinterpret_cast<const float4*>(ps + g * Cin + c);
        shp = reinterpret_cast<const float4*>(pb + g * Cin + c);
    }
    return affine4(x, __ldg(scp), __ldg(shp), pro == G6D_PRO_AFFINE_RELU);
}

// ------------------------------------------------------------------------------------------ MMA
// Each consumer warpgroup owns 64 rows x BN columns of the tile with every accumulator in registers:
// NMAIN round-robin chains for the main (hi*hi) term and one for the two cross terms, BN / 2 registers
// each (128 per thread for every BN).  Each tensor-core accumulate truncates to fp32; spreading the
// K-blocks over several shorter, smaller-magnitude chains (summed in fp32 round-to-nearest by the
// epilogue) divides the resulting bias on same-sign data by ~NMAIN at no cost.  The accumulators are
// zeroed in registers at the start of a tile and every wgmma accumulates.
template <int BN> struct AccCfg {
    static constexpr int NMAIN = BN == 32 ? 7 : (BN == 64 ? 3 : 1);
    static constexpr int R = BN / 2;
};

template <int BN, int NMAIN>
__device__ __forceinline__ void zero_acc(float (&acc)[NMAIN][BN / 2], float (&cross)[BN / 2]) {
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) {
        cross[j] = 0.f;
#pragma unroll
        for (int a = 0; a < NMAIN; ++a) acc[a][j] = 0.f;
    }
}

// The 4 K steps x 3 split terms of one stage of a warpgroup's 64 rows into the main accumulator `main`
// and the cross accumulator, committed as one wgmma group.  The callers unroll their K-block loop by
// NMAIN so that `main` is a compile-time register array (a runtime choice makes ptxas serialize the
// wgmmas).  A_hi*B_hi and A_hi*B_lo are not merged into one wgmma of width 2 BN over the adjacent B
// tiles: its accumulator registers would have to be `main` followed by `cross`, which ptxas cannot
// arrange for NMAIN > 1 main chains, and for BN = 128 ptxas rejects the n256 instruction under the
// 128-register launch budget (it checks the instruction against that count, not the setmaxnreg one).
template <int BN, int KIND>
__device__ __forceinline__ void mma_stage(float (&main)[BN / 2], float (&cross)[BN / 2], uint32_t a_hi, uint32_t a_lo,
                                          uint32_t b_hi, uint32_t b_lo) {
    const uint64_t dah = gmma_desc_sw128(a_hi), dal = gmma_desc_sw128(a_lo);
    const uint64_t dbh = gmma_desc_sw128(b_hi), dbl = gmma_desc_sw128(b_lo);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {             // 4 x 32 bytes of K per 128-byte row
        const uint64_t adv = (uint64_t)((ks * 32) >> 4);
        wgmma<BN, KIND>(cross, dal + adv, dbh + adv, 1u);
        wgmma<BN, KIND>(cross, dah + adv, dbl + adv, 1u);
        wgmma<BN, KIND>(main, dah + adv, dbh + adv, 1u);
    }
    wgmma_commit();
}

// (sum y, sum y^2) of one column over a warp's 16-row slice, rows r and r + 8 (y0, y1) per lane, r = lane / 4, in every
// lane of the column.  epilogue_tile and flat_moments_kernel share it, so the same slice gives the same fp32 partials.
__device__ __forceinline__ float2 slice_moments(float y0, float y1) {
    float s1 = y0 + y1, s2 = y0 * y0 + y1 * y1;
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {                // the 8 lanes that share this column
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    return make_float2(s1, s2);
}

// Folds the cross terms (smallest magnitude first, scaled back by the lo pre-scale) and the main chains of a consumer
// thread's accumulators into `cross`: the sum of the tile's K-blocks (of one K split).
template <int BN, int KIND>
__device__ __forceinline__ void sum_chains(float (&acc)[AccCfg<BN>::NMAIN][BN / 2], float (&cross)[BN / 2], int n_acc) {
    constexpr int NMAIN = AccCfg<BN>::NMAIN;
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) {
        float v = cross[j] * KindCfg<KIND>::CROSS;
#pragma unroll
        for (int a = 0; a < NMAIN; ++a)
            if (a < n_acc) v += acc[a][j];
        cross[j] = v;
    }
}

// Epilogue of one consumer thread: rows r and r + 8 of the tile (dst0 / dst1 point at column n_base of
// their output row, nullptr for rows outside the output), columns 8 i + 2 (lane & 3) + {0, 1}.  Takes the
// summed tile (sum_chains), adds bias + activation unless the output is a split-K partial, stores, and -- when
// stats is given -- adds the InstanceNorm moments of the stored values to the per (group, channel) fp64 accumulators
// (the reference normalises the raw conv result and the next layer's loader applies it).  All 16 rows
// of a warp belong to one group (the host only enables this for groups of whole 32-row slices / planes).
template <int BN>
__device__ __forceinline__ void store_tile(float (&cross)[BN / 2], float* dst0, float* dst1, int n_base, int Cout,
                                           const float* __restrict__ bias, int act, bool partial, bool vec2,
                                           double* __restrict__ stats, long long group, int lane) {
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
        const int c = 8 * i + cq, n = n_base + c;
        float b0 = 0.f, b1 = 0.f;
        if (!partial && bias) {
            if (n < Cout) b0 = __ldg(bias + n);
            if (n + 1 < Cout) b1 = __ldg(bias + n + 1);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float& x0 = cross[4 * i + 2 * h];
            float& x1 = cross[4 * i + 2 * h + 1];
            if (!partial) { x0 = tc_act(x0 + b0, act); x1 = tc_act(x1 + b1, act); }
            float* dst = h ? dst1 : dst0;
            if (dst) {
                if (vec2 && n + 2 <= Cout) {
                    *reinterpret_cast<float2*>(dst + c) = make_float2(x0, x1);
                } else {
                    if (n < Cout) dst[c] = x0;
                    if (n + 1 < Cout) dst[c + 1] = x1;
                }
            }
        }
    }
    if (!stats || partial) return;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float y0 = dst0 ? cross[4 * i + e] : 0.f, y1 = dst1 ? cross[4 * i + 2 + e] : 0.f;
            const float2 s = slice_moments(y0, y1);
            const int n = n_base + 8 * i + cq + e;
            if (lane < 4 && n < Cout) {
                atomicAdd(stats + (group * Cout + n) * 2, (double)s.x);
                atomicAdd(stats + (group * Cout + n) * 2 + 1, (double)s.y);
            }
        }
    }
}

template <int BN, int KIND>
__device__ __forceinline__ void epilogue_tile(float (&acc)[AccCfg<BN>::NMAIN][BN / 2], float (&cross)[BN / 2], int n_acc,
                                              float* dst0, float* dst1, int n_base, int Cout, const float* __restrict__ bias,
                                              int act, bool partial, bool vec2, double* __restrict__ stats, long long group,
                                              int lane) {
    sum_chains<BN, KIND>(acc, cross, n_acc);
    store_tile<BN>(cross, dst0, dst1, n_base, Cout, bias, act, partial, vec2, stats, group, lane);
}

// ==========================================================================================
// conv_tc2_kernel: persistent implicit-GEMM convolution.
//   * one CTA per SM loops over (M tile, N tile, K split) work items, so there is no wave tail and
//     the per-CTA set-up (barrier init, descriptor prefetch) is paid once;
//   * the eight producer warps keep a register prefetch ring (global loads of the next K-block(s) in
//     flight while K-block it is transformed and stored) and never drain the smem ring between tiles
//     (one global K-block counter), so they fill the next tile's stages during the epilogue;
//   * each of the two consumer warpgroups issues the wgmmas of its 64 rows of a stage, keeps one
//     stage's group in flight while it waits for the next (BN 128 with the split input: none, see
//     `early`), releases each stage once its group has completed (a stage is free when all 8 consumer
//     warps have released it) and runs the epilogue;
//   * one consumer thread streams the weight tiles by TMA, STAGES K-blocks ahead of the MMAs.
constexpr int TC2_PF_BYTES = 12 * 128;      // weight-tile L2 prefetch distance, in bytes of K per row

template <int BN> struct Tc2Cfg {
    static constexpr int A_BYTES = TC_BM * 128;
    static constexpr int B_BYTES = BN * 128;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
    static constexpr int STAGES = (208 * 1024) / STAGE_BYTES > 6 ? 6 : (208 * 1024) / STAGE_BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

// One A box per row of taps (XR, see xr_ok): BOXES slots of hi / lo boxes of up to BOX_ROWS pixels (roundup8(128 + kw - 1)
// for kw <= 17, a whole number of 1024-byte swizzle atoms), released after the last kx tap of their (cb, kz, ky) group,
// and a ring of B_STAGES weight stages with their own barriers.
template <int BN> struct Tc2XrCfg {
    static constexpr int BOX_ROWS = 144;
    static constexpr int BOX_BYTES = BOX_ROWS * 128;
    static constexpr int BOXES = 3;
    static constexpr int B_BYTES = BN * 128;
    static constexpr int B_STAGES = 6;
    static constexpr int SMEM_BYTES = BOXES * 2 * BOX_BYTES + B_STAGES * 2 * B_BYTES + 1024 + 256;
};
static_assert(Tc2XrCfg<64>::SMEM_BYTES <= 227 * 1024, "x-reuse rings of BN 64");

struct Tc2Work { int m_tiles, n_tiles, total; };

template <int BN, int KIND, bool FOLD, bool XR>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc2_kernel(const ConvTcP p, const Tc2Work wk, const __grid_constant__ CUtensorMap map_hi,
                const __grid_constant__ CUtensorMap map_lo, const __grid_constant__ CUtensorMap map_a) {
    using Cfg = Tc2Cfg<BN>;
    using XC = Tc2XrCfg<BN>;
    using KC = KindCfg<KIND>;
    constexpr int NPW = TC_PRODUCER_WARPS;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int NMAIN = AccCfg<BN>::NMAIN;
    constexpr int BK = KC::BK, NV = KC::NV;
    constexpr int RSTEP = NPW * 4;                       // rows r0 + RSTEP*j
    constexpr int ROWS = TC_BM / RSTEP;                  // tile rows per producer thread
    constexpr int RING = TC2_RING;                       // register prefetch ring (float4 columns); RING-1 in flight
    constexpr int PF = TC2_PF_BYTES / 128;               // K-blocks
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = base + STAGES * Cfg::STAGE_BYTES;
    auto a_hi = [&](int s) { return base + s * Cfg::STAGE_BYTES; };
    auto a_lo = [&](int s) { return base + s * Cfg::STAGE_BYTES + Cfg::A_BYTES; };
    auto b_hi = [&](int s) { return base + s * Cfg::STAGE_BYTES + 2 * Cfg::A_BYTES; };
    auto b_lo = [&](int s) { return base + s * Cfg::STAGE_BYTES + 2 * Cfg::A_BYTES + Cfg::B_BYTES; };
    auto full_a = [&](int s) { return bar_base + 8 * s; };
    auto full_b = [&](int s) { return bar_base + 8 * (STAGES + s); };
    auto empty = [&](int s) { return bar_base + 8 * (2 * STAGES + s); };
    // XR layout: the box slots, then the weight stages, then their barriers
    auto box_hi = [&](int s) { return base + s * 2 * XC::BOX_BYTES; };
    auto box_lo = [&](int s) { return base + s * 2 * XC::BOX_BYTES + XC::BOX_BYTES; };
    const uint32_t xb_base = base + XC::BOXES * 2 * XC::BOX_BYTES;
    auto xb_hi = [&](int s) { return xb_base + s * 2 * XC::B_BYTES; };
    auto xb_lo = [&](int s) { return xb_base + s * 2 * XC::B_BYTES + XC::B_BYTES; };
    const uint32_t xbar = xb_base + XC::B_STAGES * 2 * XC::B_BYTES;
    auto box_full = [&](int s) { return xbar + 8 * s; };
    auto box_empty = [&](int s) { return xbar + 8 * (XC::BOXES + s); };
    auto xb_full = [&](int s) { return xbar + 8 * (2 * XC::BOXES + s); };
    auto xb_empty = [&](int s) { return xbar + 8 * (2 * XC::BOXES + XC::B_STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (XR && threadIdx.x == TC_ISSUER) {
        for (int s = 0; s < XC::BOXES; ++s) {
            mbar_init(box_full(s), 1);
            mbar_init(box_empty(s), TC_CONSUMER_WARPS);
        }
        for (int s = 0; s < XC::B_STAGES; ++s) {
            mbar_init(xb_full(s), 1);
            mbar_init(xb_empty(s), TC_CONSUMER_WARPS);
        }
        fence_barrier_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    } else if (threadIdx.x == TC_ISSUER) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_a(s), p.split_in ? 1 : NPW);   // the A TMA transaction, or the producer warps
            mbar_init(full_b(s), 1);          // the TMA transaction
            mbar_init(empty(s), TC_CONSUMER_WARPS);
        }
        fence_barrier_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_lo) : "memory");
        if (p.split_in) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    }
    __syncthreads();

    // work item -> (m tile, n tile, split); n fastest so neighbouring CTAs share the gathered A rows in L2
    auto decode = [&](int w, int& mt, int& nt, int& sp) {
        nt = w % wk.n_tiles; w /= wk.n_tiles;
        mt = w % wk.m_tiles;
        sp = w / wk.m_tiles;
    };
    auto kblocks_of = [&](int sp) { return min(p.kblocks, sp * p.kb_per_split + p.kb_per_split) - sp * p.kb_per_split; };
    // The CTA's j-th chain: work item blockIdx.x + (j / chains) gridDim.x.  Folded (FOLD), an item is a tile and its K
    // splits are consecutive chains; otherwise an item is one (tile, split) chain.  The A/B TMA thread and the consumers
    // walk the same sequence.  Folding is only planned with the split input, so the producer warps and the consumers'
    // weight stream (gathered A) keep their per-item loops.  False past the last item.
    const int chains = FOLD ? p.splits : 1;
    auto chain_of = [&](int j, int& mt, int& nt, int& sp) {
        const int w = blockIdx.x + (j / chains) * gridDim.x;
        if (w >= wk.total) return false;
        decode(w, mt, nt, sp);
        sp += j % chains;
        return true;
    };

    if (warp < NPW) {
        setmaxnreg_dec<FOLD ? TC_FOLD_PRODUCER_REGS : TC_PRODUCER_REGS>();
        if (XR && threadIdx.x == 0) {
            // One box pair per (cb, kz, ky) group of kw consecutive K-blocks (the A-reuse K order starts every chain at
            // kx = 0), over the padded enumeration of Wp columns: tile row j + kx of the box is tap kx of row j.  The
            // weight tiles go to their own ring, one stage per K-block.
            const bool vol = p.D > 1 || p.kd > 1;
            const uint32_t box_tx = 2u * p.xr_rows * 128u;
            int g = 0, gb = 0;                               // K-blocks, boxes
            int mt, nt, sp;
            for (int j = 0; chain_of(j, mt, nt, sp); ++j) {
                const int nkb = kblocks_of(sp);
                int m = mt * TC_BM;
                const int xo = m % p.Wp; m /= p.Wp;
                const int yo = m % p.Ho; m /= p.Ho;
                const int zo = m % p.Do;
                const int b = m / p.Do;
                KbIter k;                                    // no weight L2 prefetch, see below
                k.start(p, sp, 0);
                for (int it = 0; it < nkb; ++it, ++g, k.next(p)) {
                    if (k.kx == 0) {
                        const int s = gb % XC::BOXES;
                        const uint16_t oy = (uint16_t)k.ky, oz = (uint16_t)k.kz;
                        mbar_wait(box_empty(s), ((gb / XC::BOXES) & 1) ^ 1, 6, gb);
                        mbar_expect_tx(box_full(s), box_tx);
                        if (vol) {
                            tma_im2col_5d(box_hi(s), &map_a, box_full(s), 2 * BK * k.cb, xo - p.pw, yo - p.ph, zo - p.pd, b, 0, oy, oz);
                            tma_im2col_5d(box_lo(s), &map_a, box_full(s), 2 * BK * k.cb + BK, xo - p.pw, yo - p.ph, zo - p.pd, b, 0, oy, oz);
                        } else {
                            tma_im2col_4d(box_hi(s), &map_a, box_full(s), 2 * BK * k.cb, xo - p.pw, yo - p.ph, b, 0, oy);
                            tma_im2col_4d(box_lo(s), &map_a, box_full(s), 2 * BK * k.cb + BK, xo - p.pw, yo - p.ph, b, 0, oy);
                        }
                        ++gb;
                    }
                    const int s = g % XC::B_STAGES;
                    mbar_wait(xb_empty(s), ((g / XC::B_STAGES) & 1) ^ 1, 1, g);
                    mbar_expect_tx(xb_full(s), 2 * XC::B_BYTES);
                    tma_load_2d(xb_hi(s), &map_hi, xb_full(s), k.tap(p) * p.Cin + k.cb * BK, nt * BN);
                    tma_load_2d(xb_lo(s), &map_lo, xb_full(s), k.tap(p) * p.Cin + k.cb * BK, nt * BN);
                }
            }
            return;
        }
        if (XR || FOLD || p.split_in) {
            // =========================== A by TMA im2col ===========================
            // The input is already split (hi / lo of channel block cb at channels [128 cb, 128 cb + 64) /
            // [128 cb + 64, 128 cb + 128) of each pixel, in f16_k_source order), so a K-block of tap (kx, ky)
            // is two im2col boxes of the 128 output pixels of the tile: byte for byte what the producers
            // below would store.  One thread issues them, and the stage's weight tiles with them (the consumers
            // then issue no loads); the other producer warps have nothing to do.  Volumes (D > 1 or kd > 1) use
            // the rank-5 map, see make_split_input_map.
            if (!XR && threadIdx.x == 0) {
                const bool vol = p.D > 1 || p.kd > 1;
                int g = 0;
                int mt, nt, sp;
                for (int j = 0; chain_of(j, mt, nt, sp); ++j) {
                    const int nkb = kblocks_of(sp);
                    int m = mt * TC_BM;
                    const int xo = m % p.Wo; m /= p.Wo;
                    const int yo = m % p.Ho; m /= p.Ho;
                    const int zo = m % p.Do;
                    const int b = m / p.Do;
                    // No L2 prefetch of the weight tiles ahead of their loads (the consumers' weight stream below keeps
                    // one): the TMA unit walks a prefetch box row by row like a load, so the two prefetches per K-block
                    // were a third of the box rows it processed, and every bench shape ran faster without them
                    // (DESIGN.md section 5).  The x-reuse thread above does without it for the same reason.
                    KbIter k;
                    k.start(p, sp, 0);
                    for (int it = 0; it < nkb; ++it, ++g, k.next(p)) {
                        const int tap = k.tap(p), cb = k.cb;
                        const uint16_t ox = (uint16_t)k.kx, oy = (uint16_t)k.ky, oz = (uint16_t)k.kz;
                        const int s = g % STAGES;
                        mbar_wait(empty(s), ((g / STAGES) & 1) ^ 1, 1, g);
                        mbar_expect_tx(full_b(s), 2 * Cfg::B_BYTES);
                        tma_load_2d(b_hi(s), &map_hi, full_b(s), tap * p.Cin + cb * BK, nt * BN);
                        tma_load_2d(b_lo(s), &map_lo, full_b(s), tap * p.Cin + cb * BK, nt * BN);
                        mbar_expect_tx(full_a(s), 2 * Cfg::A_BYTES);
                        if (vol) {
                            tma_im2col_5d(a_hi(s), &map_a, full_a(s), 2 * BK * cb, xo - p.pw, yo - p.ph, zo - p.pd, b, ox, oy, oz);
                            tma_im2col_5d(a_lo(s), &map_a, full_a(s), 2 * BK * cb + BK, xo - p.pw, yo - p.ph, zo - p.pd, b, ox, oy, oz);
                        } else {
                            tma_im2col_4d(a_hi(s), &map_a, full_a(s), 2 * BK * cb, xo - p.pw, yo - p.ph, b, ox, oy);
                            tma_im2col_4d(a_lo(s), &map_a, full_a(s), 2 * BK * cb + BK, xo - p.pw, yo - p.ph, b, ox, oy);
                        }
                    }
                }
            }
            return;
        }
        // =============================== A producers ===============================
        // All producer warps fill every K-block: ROWS rows x one 16-byte smem chunk (4 or 8 channels) per thread.
        const int chunk = threadIdx.x & 7;
        const int cofs = chunk * 4;                        // this thread's channels inside the K-block: [cofs, cofs+4) (+32 for the 2nd load)
        const int r0 = threadIdx.x >> 3;                   // rows r0 + RSTEP*j, j < ROWS
        int git = 0;                                       // global K-block counter of this CTA
        for (int w = blockIdx.x; w < wk.total; w += gridDim.x) {
            int mt, nt, sp;
            decode(w, mt, nt, sp);
            const int m_base = mt * TC_BM;
            const int kb_begin = sp * p.kb_per_split;
            const int nkb = kblocks_of(sp);
            int rb[ROWS], rsp[ROWS], rc[ROWS];
            unsigned rvmask = 0;
            const long long plane_sz = (long long)p.D * p.H * p.W;
#pragma unroll
            for (int j = 0; j < ROWS; ++j) {
                int m = m_base + r0 + RSTEP * j;
                const bool v = m < p.M;
                if (!v) m = 0;
                const int xo = m % p.Wo; m /= p.Wo;
                const int yo = m % p.Ho; m /= p.Ho;
                const int zo = m % p.Do; m /= p.Do;
                rb[j] = m;
                const int z = zo * p.stride - p.pd, y = yo * p.stride - p.ph, x = xo * p.stride - p.pw;
                rsp[j] = (z * p.H + y) * p.W + x;
                rc[j] = ((z + 8) << 24) | ((y + 8) << 12) | (x + 8);
                if (v) rvmask |= 1u << j;
            }
            int c0, kx, ky, kz;
            {
                const int k = kb_begin * BK;
                int tap = 0; c0 = k;
                if (p.K != p.Cin) { tap = k / p.Cin; c0 = k - tap * p.Cin; }
                kx = tap % p.kw; const int tq = tap / p.kw; ky = tq % p.kh; kz = tq / p.kh;
            }
            // prefetch ring: slot q holds float4 column e = u % NV of K-block u / NV, u % RING == q
            float4 v[RING][ROWS];
            unsigned okm[RING]; int kc[RING]; int ksp[RING];
            auto issue_loads = [&](int q, int e) {
                const int tap_sp = (kz * p.H + ky) * p.W + kx;
                okm[q] = 0; kc[q] = c0 + cofs + 32 * e; ksp[q] = tap_sp;
                const float* xb = p.x + p.ico + kc[q];
#pragma unroll
                for (int j = 0; j < ROWS; ++j) {
                    const int z = ((rc[j] >> 24) & 0xff) - 8 + kz, y = ((rc[j] >> 12) & 0xfff) - 8 + ky, x = (rc[j] & 0xfff) - 8 + kx;
                    const bool inb = ((rvmask >> j) & 1u) && (unsigned)z < (unsigned)p.D && (unsigned)y < (unsigned)p.H &&
                                     (unsigned)x < (unsigned)p.W;
                    v[q][j] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (inb) {
                        v[q][j] = __ldg(reinterpret_cast<const float4*>(xb + ((long long)rb[j] * plane_sz + rsp[j] + tap_sp) * p.ics));
                        okm[q] |= 1u << j;
                    }
                }
                if (e == NV - 1) {
                    c0 += BK;
                    if (c0 == p.Cin) { c0 = 0; if (++kx == p.kw) { kx = 0; if (++ky == p.kh) { ky = 0; ++kz; } } }
                }
            };
            auto process = [&](int q, int e, int it) {
                const int g_it = git + it;
                const int s = g_it % STAGES;
                const uint32_t n_use = g_it / STAGES;
                if (p.pro != G6D_PRO_NONE) {
#pragma unroll
                    for (int j = 0; j < ROWS; ++j)
                        if (okm[q] & (1u << j))
                            v[q][j] = prologue4(v[q][j], p.pro, p.ps, p.pb, p.Cin, p.group_rows, rb[j], rsp[j] + ksp[q], kc[q]);
                }
                if (e == 0) mbar_wait(empty(s), (n_use & 1) ^ 1, 1, g_it);
#pragma unroll
                for (int j = 0; j < ROWS; ++j) {
                    const int r = r0 + RSTEP * j;
                    const uint32_t so = r * 128 + ((chunk ^ (r & 7)) << 4);        // Swizzle<3,4,3>
                    split_store<KIND>(a_hi(s) + so, a_lo(s) + so, v[q][j], e);
                }
                if (e == NV - 1) {
                    fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
                    __syncwarp();
                    if (lane == 0) mbar_arrive(full_a(s));
                }
            };
            // software pipeline over the nkb * NV columns, unrolled by RING so that the ring slots are
            // compile-time register names
            const int ncol = nkb * NV;
#pragma unroll
            for (int q = 0; q < RING - 1; ++q)
                if (q < ncol) issue_loads(q, q % NV);
            for (int u = 0; u < ncol; u += RING) {
#pragma unroll
                for (int q = 0; q < RING; ++q) {
                    if (u + q < ncol) {
                        if (u + q + RING - 1 < ncol) issue_loads((q + RING - 1) % RING, (u + q + RING - 1) % NV);
                        process(q, (u + q) % NV, (u + q) / NV);
                    }
                }
            }
            git += nkb;
        }
    } else {
        // =============================== consumer warpgroups ===============================
        setmaxnreg_inc<FOLD ? TC_FOLD_CONSUMER_REGS : TC_CONSUMER_REGS>();
        const int cw = warp - NPW;                     // consumer warp: rows 16 cw .. 16 cw + 15 of the tile
        const uint32_t a_row = (cw >> 2) * 64 * 128;   // this warpgroup's 64 rows of the A tiles
        const bool issuer = !FOLD && !XR && threadIdx.x == TC_ISSUER && !p.split_in;   // with the split input, the A issuer loads B
        // weight-tile stream of the issuer: the next global K-block lg = K-block lit of work item lw
        int lw = blockIdx.x, lit = 0, lg = 0;
        auto load_next = [&]() {
            int mt, nt, sp, nkb = 0;
            for (; lw < wk.total; lw += gridDim.x, lit = 0) {
                decode(lw, mt, nt, sp);
                nkb = kblocks_of(sp);
                if (lit < nkb) break;
            }
            if (lw >= wk.total) return;
            const int kb_begin = sp * p.kb_per_split;
            // The weight tiles of a small-M layer are touched once and come from HBM: with only STAGES
            // tiles in flight the ring is latency-bound.  An L2 prefetch running PF K-blocks ahead costs
            // no shared memory.
            if (lit == 0) {
                for (int i = 0; i < min(nkb, PF); ++i) {
                    tma_prefetch_2d(&map_hi, (kb_begin + i) * BK, nt * BN);
                    tma_prefetch_2d(&map_lo, (kb_begin + i) * BK, nt * BN);
                }
            } else if (lit + PF - 1 < nkb) {
                tma_prefetch_2d(&map_hi, (kb_begin + lit + PF - 1) * BK, nt * BN);
                tma_prefetch_2d(&map_lo, (kb_begin + lit + PF - 1) * BK, nt * BN);
            }
            const int s = lg % STAGES;
            mbar_wait(empty(s), ((lg / STAGES) & 1) ^ 1, 3, lg);
            mbar_expect_tx(full_b(s), 2 * Cfg::B_BYTES);
            tma_load_2d(b_hi(s), &map_hi, full_b(s), (kb_begin + lit) * BK, nt * BN);
            tma_load_2d(b_lo(s), &map_lo, full_b(s), (kb_begin + lit) * BK, nt * BN);
            ++lit; ++lg;
        };
        // the wgmma group of global K-block g has completed: hand its stage back to the producers
        auto release = [&](int g) {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty(g % STAGES));
            if (issuer) load_next();
        };
        if (issuer)
            for (int i = 0; i < STAGES; ++i) load_next();

        // Early release (BN 128 with the split input): only three 64 KB stages fit, and a consumer that keeps one
        // group in flight holds two of them, which leaves the TMA thread one stage ahead.  These consumers instead
        // wait for each stage's group and release the stage at once: two stages ahead, while the other warpgroup's
        // wgmmas keep the tensor cores busy across the wait.  The wgmmas and their order are unchanged.
        const bool early = BN == 128 && p.split_in;
        float acc[NMAIN][BN / 2];
        float cross[BN / 2];
        float run[FOLD ? BN / 2 : 1];                  // FOLD: the tile's sum of its splits so far
        int g = 0;
        int gb = 0, rb = 0;                            // XR: boxes awaited, boxes released
        // XR: the weight stage of K-block g is free, and with it the box of a group whose last tap it was
        auto xr_release = [&](int g, bool box_done) {
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(xb_empty(g % XC::B_STAGES));
                if (box_done) mbar_arrive(box_empty(rb % XC::BOXES));
            }
            if (box_done) ++rb;
        };
        int mt, nt, sp;
        for (int j = 0; chain_of(j, mt, nt, sp); ++j) {
            const int nkb = kblocks_of(sp);
            zero_acc<BN, NMAIN>(acc, cross);
            if constexpr (XR) {
                // tap kx of a (cb, kz, ky) group reads the group's box shifted by kx rows
                int kx = 0;
                bool box_done = false;
                for (int it0 = 0; it0 < nkb; it0 += NMAIN) {
#pragma unroll
                    for (int a = 0; a < NMAIN; ++a) {
                        const int it = it0 + a;
                        if (it < nkb) {
                            if (kx == 0) {
                                mbar_wait(box_full(gb % XC::BOXES), (gb / XC::BOXES) & 1, 7, gb);
                                ++gb;
                            }
                            const int s = g % XC::B_STAGES, sb = (gb - 1) % XC::BOXES;
                            mbar_wait(xb_full(s), (g / XC::B_STAGES) & 1, 5, g);
                            const uint32_t sh = a_row + kx * 128;
                            mma_stage<BN, KIND>(acc[a], cross, box_hi(sb) + sh, box_lo(sb) + sh, xb_hi(s), xb_lo(s));
                            wgmma_wait<1>();
                            if (it > 0) xr_release(g - 1, box_done);
                            box_done = kx == p.kw - 1;
                            ++g;
                            if (++kx == p.kw) kx = 0;
                        }
                    }
                }
                wgmma_wait<0>();
                if (nkb > 0) xr_release(g - 1, true);
            } else {
            for (int it0 = 0; it0 < nkb; it0 += NMAIN) {
#pragma unroll
                for (int a = 0; a < NMAIN; ++a) {              // K-block it uses main accumulator it % NMAIN
                    const int it = it0 + a;
                    if (it < nkb) {
                        const int s = g % STAGES;
                        mbar_wait(full_a(s), (g / STAGES) & 1, 4, g);
                        mbar_wait(full_b(s), (g / STAGES) & 1, 5, g);
                        mma_stage<BN, KIND>(acc[a], cross, a_hi(s) + a_row, a_lo(s) + a_row, b_hi(s), b_lo(s));
                        if (early) {
                            wgmma_wait<0>();
                            release(g);
                        } else {
                            wgmma_wait<1>();
                            if (it > 0) release(g - 1);
                        }
                        ++g;
                    }
                }
            }
            wgmma_wait<0>();
            if (nkb > 0 && !early) release(g - 1);
            }

            sum_chains<BN, KIND>(acc, cross, nkb < NMAIN ? nkb : NMAIN);
            if constexpr (FOLD) {
                // the running sum in conv_tc_reduce4_kernel's order: 0.f + split 0, then each further split; the last
                // split stores it with bias + activation
#pragma unroll
                for (int jj = 0; jj < BN / 2; ++jj) run[jj] = (sp == 0 ? 0.f : run[jj]) + cross[jj];
                if (sp < p.splits - 1) continue;
#pragma unroll
                for (int jj = 0; jj < BN / 2; ++jj) cross[jj] = run[jj];
            }
            const bool partial = p.splits > 1 && !FOLD;
            const int n_base = nt * BN;
            const int m0 = mt * TC_BM + 16 * cw + (lane >> 2), m1 = m0 + 8;
            float* out = partial ? p.ws + (long long)sp * p.M * p.Cout + n_base : p.y + p.oco + n_base;
            const long long ld = partial ? p.Cout : p.ocs;
            // 64-bit stores need 8-byte aligned column pairs
            const bool vec2 = partial ? (p.Cout & 1) == 0
                                      : ((p.ocs & 1) == 0 && (p.oco & 1) == 0 && (reinterpret_cast<uintptr_t>(p.y) & 7) == 0);
            // XR: m0 / m1 count the padded enumeration; its columns xp >= Wo are never written (no fused moments either:
            // XR plans take them from y, see g6d_conv_tc_ex)
            auto dst = [&](int m) -> float* {
                if constexpr (XR) {
                    if (m >= p.Mp) return nullptr;
                    const int q = m / p.Wp, xp = m - q * p.Wp;
                    return xp < p.Wo ? out + ((long long)q * p.Wo + xp) * ld : nullptr;
                } else {
                    return m < p.M ? out + m * ld : nullptr;
                }
            };
            store_tile<BN>(cross, dst(m0), dst(m1), n_base, p.Cout, p.bias,
                           p.act, partial, vec2, p.stats, (long long)(mt * TC_BM + 16 * cw) / p.stats_rows, lane);
        }
    }
}


// Split-K epilogue: y = act(sum_s ws[s] + bias); one thread per output element.
__global__ void conv_tc_reduce_kernel(const float* __restrict__ ws, const float* __restrict__ bias,
                                      float* __restrict__ y, int M, int Cout, int splits, int ocs, int oco, int act) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)M * Cout) return;
    const int n = (int)(i % Cout);
    const long long m = i / Cout;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += ws[(long long)s * M * Cout + i];
    if (bias) v += bias[n];
    y[m * ocs + oco + n] = tc_act(v, act);
}

// The same for Cout % 4 == 0, four columns of one output row per thread: 128-bit partial loads, all `splits` of them
// issued before the first add, and one divide per four elements.  Each element is summed in the same order (split 0
// first, then bias), so the output equals conv_tc_reduce_kernel's bit for bit.  vec_out: y + oco and ocs keep 16-byte
// alignment, so the row is stored as one float4.
template <int SPLITS>
__device__ __forceinline__ float4 sum_splits4(const float4* __restrict__ ws4, long long slab4, long long i4, int splits) {
    float4 p[SPLITS > 0 ? SPLITS : 1];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (SPLITS > 0) {
#pragma unroll
        for (int s = 0; s < SPLITS; ++s) p[s] = __ldg(ws4 + s * slab4 + i4);
#pragma unroll
        for (int s = 0; s < SPLITS; ++s) { v.x += p[s].x; v.y += p[s].y; v.z += p[s].z; v.w += p[s].w; }
    } else {
        for (int s = 0; s < splits; ++s) {
            const float4 q = __ldg(ws4 + s * slab4 + i4);
            v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
        }
    }
    return v;
}

template <int SPLITS>
__global__ void conv_tc_reduce4_kernel(const float* __restrict__ ws, const float* __restrict__ bias, float* __restrict__ y,
                                       int M, int Cout, int splits, int ocs, int oco, int act, bool vec_out) {
    const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int c4 = Cout >> 2;
    if (i4 >= (long long)M * c4) return;
    const long long m = i4 / c4;
    const int n = (int)(i4 - m * c4) * 4;
    float4 v = sum_splits4<SPLITS>(reinterpret_cast<const float4*>(ws), (long long)M * c4, i4, splits);
    if (bias) { v.x += bias[n]; v.y += bias[n + 1]; v.z += bias[n + 2]; v.w += bias[n + 3]; }
    v = make_float4(tc_act(v.x, act), tc_act(v.y, act), tc_act(v.z, act), tc_act(v.w, act));
    float* dst = y + m * ocs + oco + n;
    if (vec_out) {
        *reinterpret_cast<float4*>(dst) = v;
    } else {
        dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
    }
}

// The same with the fused InstanceNorm statistics of y: a 256-thread block owns 32 consecutive output
// rows (one group: stats_rows % 32 == 0) x 64 channels; thread = (channel, 8-row slice); the four slices
// are combined in shared memory and one (sum, sum^2) pair per (block, channel) goes to the fp64 accumulators.
// value(m, n) is output element (m, n) (n < Cout, m < M).  conv_tc_reduce_stats_kernel and fold_moments_kernel
// share this, so a folded layer's moments have the same fp32 partials as the split-K reduce's.
template <class Value>
__device__ __forceinline__ void block_moments_32x64(Value value, int M, int Cout, double* __restrict__ stats,
                                                    long long stats_rows) {
    __shared__ float red[2][4][64];
    const int c = threadIdx.x & 63, rg = threadIdx.x >> 6;
    const int n = blockIdx.y * 64 + c;
    const int m0 = blockIdx.x * 32 + rg * 8;
    float s1 = 0.f, s2 = 0.f;
    if (n < Cout) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int m = m0 + r;
            if (m < M) {
                const float v = value(m, n);
                s1 += v; s2 = fmaf(v, v, s2);
            }
        }
    }
    red[0][rg][c] = s1; red[1][rg][c] = s2;
    __syncthreads();
    if (threadIdx.x < 128) {
        const int q = threadIdx.x >> 6;                       // 0: sum, 1: sum of squares
        const float t = red[q][0][c] + red[q][1][c] + red[q][2][c] + red[q][3][c];
        if (n < Cout) atomicAdd(stats + ((long long)((blockIdx.x * 32) / stats_rows) * Cout + n) * 2 + q, (double)t);
    }
}

__global__ void __launch_bounds__(256) conv_tc_reduce_stats_kernel(const float* __restrict__ ws, const float* __restrict__ bias,
                                                                   float* __restrict__ y, int M, int Cout, int splits, int ocs,
                                                                   int oco, int act, double* __restrict__ stats, long long stats_rows) {
    const long long slab = (long long)M * Cout;
    block_moments_32x64([&](int m, int n) {
        const long long i = (long long)m * Cout + n;
        float v = 0.f;
        for (int s = 0; s < splits; ++s) v += ws[(long long)s * slab + i];
        v = tc_act(v + (bias ? bias[n] : 0.f), act);
        y[(long long)m * ocs + oco + n] = v;
        return v;
    }, M, Cout, stats, stats_rows);
}

// The moments of a folded layer (G6D_TC_FOLD_SPLITS with stats): the conv wrote the final y, which is what
// conv_tc_reduce_stats_kernel would have written, and this pass takes that kernel's moments of it.
__global__ void __launch_bounds__(256) fold_moments_kernel(const float* __restrict__ y, int M, int Cout, int ocs, int oco,
                                                           double* __restrict__ stats, long long stats_rows) {
    block_moments_32x64([&](int m, int n) { return y[(long long)m * ocs + oco + n]; }, M, Cout, stats, stats_rows);
}

static void launch_reduce(const float* ws, const float* bias, float* y, int M, int Cout, int splits, int ocs, int oco, int act,
                          double* stats, long long stats_rows, cudaStream_t st) {
    if (stats) {
        dim3 grid(ceil_div(M, 32), ceil_div(Cout, 64));
        conv_tc_reduce_stats_kernel<<<grid, 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act, stats, stats_rows);
    } else if ((Cout & 3) == 0) {
        const long long n4 = (long long)M * (Cout / 4);
        const bool vec_out = (ocs & 3) == 0 && (oco & 3) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0;
        const unsigned grid = (unsigned)ceil_div(n4, 256);
        switch (splits) {       // the split counts of the network's layers get their loads unrolled
            case 2: conv_tc_reduce4_kernel<2><<<grid, 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act, vec_out); break;
            case 3: conv_tc_reduce4_kernel<3><<<grid, 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act, vec_out); break;
            case 4: conv_tc_reduce4_kernel<4><<<grid, 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act, vec_out); break;
            case 8: conv_tc_reduce4_kernel<8><<<grid, 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act, vec_out); break;
            default: conv_tc_reduce4_kernel<0><<<grid, 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act, vec_out);
        }
    } else {
        const long long n = (long long)M * Cout;
        conv_tc_reduce_kernel<<<ceil_div(n, 256), 256, 0, st>>>(ws, bias, y, M, Cout, splits, ocs, oco, act);
    }
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

static int kind_bk(int kind) { return kind == G6D_TC_F16 ? 64 : 32; }
static int kind_esize(int kind) { return kind == G6D_TC_F16 ? 2 : 4; }

// 2-D tensor map over W [rows = Cout_pad, cols = K] (K-major), box = [one 128-byte swizzle row of K, bn rows]
static int make_weight_map(CUtensorMap* map, const void* w, int rows, int K, int bn, int kind) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_error("g6d_conv_tc: cuTensorMapEncodeTiled unavailable"); return G6D_ECUDA; }
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)K * kind_esize(kind)};
    cuuint32_t box[2] = {(cuuint32_t)kind_bk(kind), (cuuint32_t)bn};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, kind == G6D_TC_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                     const_cast<void*>(w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("g6d_conv_tc: cuTensorMapEncodeTiled failed (%d)", (int)r); return G6D_ECUDA; }
    return G6D_OK;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeIm2colFn get_encode_im2col_fn() {
    static EncodeIm2colFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeIm2colFn>(sym);
    }
    return fn;
}

// im2col map over the split input [B, H, W, 2 Cin] fp16: 64 channels x 128 pixels per box (one 128-byte swizzle
// row per pixel); the bounding box of filter origins runs from -pad to dim - 1 + pad - (k - 1), i.e. the output
// plane of a stride-1 convolution, and taps outside the tensor are filled with zeros (the padding).  Volumes
// (D > 1 or kd > 1, the same test as the kernel's) get the rank-5 map over [B, D, H, W, 2 Cin].
static bool split_input_rank5(const g6d_conv_desc* d) { return d->D > 1 || d->kd > 1; }

static int make_split_input_map(CUtensorMap* map, const void* xs, const g6d_conv_desc* d, int xr_rows) {
    EncodeIm2colFn enc = get_encode_im2col_fn();
    if (!enc) { set_error("g6d_conv_tc: cuTensorMapEncodeIm2col unavailable"); return G6D_ECUDA; }
    const cuuint64_t C2 = 2ull * d->Cin;
    const cuuint32_t rank = split_input_rank5(d) ? 5 : 4;
    cuuint64_t dims[5] = {C2, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->D, (cuuint64_t)d->B};
    cuuint64_t strides[4] = {C2 * 2, C2 * 2 * d->W, C2 * 2 * d->W * d->H, C2 * 2 * d->W * d->H * d->D};
    if (rank == 4) dims[3] = d->B;
    int lower[3] = {-d->pw, -d->ph, -d->pd};
    int upper[3] = {d->pw - (xr_rows ? 0 : d->kw - 1), d->ph - (d->kh - 1), d->pd - (d->kd - 1)};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(xs), dims, strides, lower, upper, 64,
                     xr_rows ? xr_rows : TC_BM, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("g6d_conv_tc: cuTensorMapEncodeIm2col failed (%d)", (int)r); return G6D_ECUDA; }
    return G6D_OK;
}

static int tc_block_n(int Cout) { return Cout > 64 ? 128 : (Cout > 32 ? 64 : 32); }
static int tc_nmain(int bn) { return bn == 32 ? AccCfg<32>::NMAIN : (bn == 64 ? AccCfg<64>::NMAIN : AccCfg<128>::NMAIN); }

// the persistent kernel packs (z, y, x) + 8 into 8/12/12 bits and uses 32-bit spatial offsets and group indices
static bool tc2_dims_ok(const g6d_conv_desc* d) {
    return d->D + d->pd + 8 < 256 && d->H + d->ph + 8 < 4096 && d->W + d->pw + 8 < 4096 &&
           (long long)d->D * d->H * d->W < (1ll << 30) && d->group_rows < (1ll << 31);
}

static int fill_tc_params(const g6d_conv_desc* d, int kind, ConvTcP& p) {
    G6D_REQUIRE(d != nullptr, "g6d_conv_tc: null desc");
    G6D_REQUIRE(kind == G6D_TC_TF32 || kind == G6D_TC_F16, "g6d_conv_tc: bad operand kind %d", kind);
    G6D_REQUIRE(d->B > 0 && d->D > 0 && d->H > 0 && d->W > 0 && d->Cin > 0, "g6d_conv_tc: bad dims");
    G6D_REQUIRE(d->Cout >= 16, "g6d_conv_tc: Cout (%d) must be at least 16", d->Cout);
    G6D_REQUIRE(d->kd > 0 && d->kh > 0 && d->kw > 0 && d->stride > 0, "g6d_conv_tc: bad kernel/stride");
    const int bk = kind_bk(kind);
    G6D_REQUIRE((d->Cin % bk) == 0, "g6d_conv_tc: Cin (%d) must be a multiple of %d", d->Cin, bk);
    G6D_REQUIRE((d->in_cstride & 3) == 0 && (d->in_coff & 3) == 0, "g6d_conv_tc: in_cstride/in_coff must be multiples of 4");
    G6D_REQUIRE(d->in_coff + d->Cin <= d->in_cstride, "g6d_conv_tc: input channel slice out of row");
    G6D_REQUIRE(d->out_coff + d->Cout <= d->out_cstride, "g6d_conv_tc: output channel slice out of row");
    G6D_REQUIRE(tc2_dims_ok(d), "g6d_conv_tc: spatial extent too large for the tensor-core kernel");
    const int Do = (d->D + 2 * d->pd - d->kd) / d->stride + 1;
    const int Ho = (d->H + 2 * d->ph - d->kh) / d->stride + 1;
    const int Wo = (d->W + 2 * d->pw - d->kw) / d->stride + 1;
    G6D_REQUIRE(Do > 0 && Ho > 0 && Wo > 0 && Do == d->Do && Ho == d->Ho && Wo == d->Wo, "g6d_conv_tc: output dims mismatch");
    G6D_REQUIRE(d->prologue >= 0 && d->prologue <= 3 && d->act >= 0 && d->act <= 2, "g6d_conv_tc: bad prologue/act");
    const long long M = (long long)d->B * Do * Ho * Wo;
    const long long K = (long long)d->kd * d->kh * d->kw * d->Cin;
    G6D_REQUIRE(M < (1ll << 31) && K < (1ll << 31), "g6d_conv_tc: problem too large");
    G6D_REQUIRE(d->plan_rows >= 0 && d->plan_rows % ((long long)Do * Ho * Wo) == 0,
                "g6d_conv_tc: plan_rows (%d) must be a multiple of the %d output rows of one image", d->plan_rows, Do * Ho * Wo);
    p.B = d->B; p.D = d->D; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.ics = d->in_cstride; p.ico = d->in_coff;
    p.Cout = d->Cout; p.kd = d->kd; p.kh = d->kh; p.kw = d->kw; p.stride = d->stride; p.pd = d->pd; p.ph = d->ph;
    p.pw = d->pw; p.Do = Do; p.Ho = Ho; p.Wo = Wo; p.ocs = d->out_cstride; p.oco = d->out_coff; p.pro = d->prologue;
    p.act = d->act; p.group_rows = d->group_rows > 0 ? d->group_rows : 1;
    p.M = (int)M; p.K = (int)K; p.kblocks = (int)(K / bk);
    const int bn = tc_block_n(d->Cout);
    const long long plan_m = d->plan_rows > 0 ? d->plan_rows : M;     // the rows the K splits are planned for
    const long long ctas = (long long)ceil_div(plan_m, TC_BM) * ceil_div(d->Cout, bn);
    const int min_kb = 256 / bk;                     // never split below 256 K-elements per item
    int splits = 1;
    if (ctas < kNumSMs && p.kblocks >= 2 * min_kb) {
        // as many K splits as still fit in ONE wave of the persistent CTAs (a second, partial wave
        // of long items costs more than the parallelism it adds)
        splits = (int)(kNumSMs / ctas);
        splits = splits > p.kblocks / min_kb ? p.kblocks / min_kb : splits;
        splits = splits < 1 ? 1 : splits;
    }
    // The tensor core adds each K-step into the fp32 accumulator with truncation; over long K chains
    // of same-sign products that is a systematic bias (detector correlation, K = 115200 of post-ReLU
    // features: ~4e-5 relative; on Hopper it already shows in the 3x3x512 VGG layers and compounds
    // through the pyramid: 3.4e-5 on the detector's raw correlation, 2.2e-5 with the split, at +0.9 %
    // detection time, see DESIGN.md section 3).  For K > 2048 the chain per accumulator is bounded to
    // 2048 terms and the partials are summed in fp32 round-to-nearest.
    // d->max_chain_k bounds the K-elements per ACCUMULATOR; a split rotates over NMAIN of them
    const int nmain = tc_nmain(bn);
    const int chain = d->max_chain_k > 0 ? d->max_chain_k * nmain : (K > TC_MAX_K_PER_CHAIN ? TC_MAX_K_PER_CHAIN * nmain : 0);
    const int max_kb = chain > bk ? chain / bk : 1;
    const int min_splits = chain > 0 ? (p.kblocks + max_kb - 1) / max_kb : 1;
    splits = splits < min_splits ? min_splits : splits;
    splits = splits > 64 ? 64 : splits;
    p.kb_per_split = (p.kblocks + splits - 1) / splits;
    p.splits = (p.kblocks + p.kb_per_split - 1) / p.kb_per_split;
    return G6D_OK;
}

template <int BN, int KIND, bool FOLD, bool XR>
static int launch_tc2(const ConvTcP& p, const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& ma, cudaStream_t st) {
    constexpr int SMEM = XR ? Tc2XrCfg<BN>::SMEM_BYTES : Tc2Cfg<BN>::SMEM_BYTES;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc2_kernel<BN, KIND, FOLD, XR>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
        if (e != cudaSuccess) { set_error("g6d_conv_tc: cannot opt in to %d B of shared memory: %s", SMEM, cudaGetErrorString(e)); return G6D_ECUDA; }
        configured = true;
    }
    Tc2Work wk;
    wk.m_tiles = ceil_div(XR ? p.Mp : p.M, TC_BM); wk.n_tiles = ceil_div(p.Cout, BN);
    const long long total = (long long)wk.m_tiles * wk.n_tiles * (FOLD ? 1 : p.splits);
    wk.total = (int)total;
    const int grid = total < kNumSMs ? (int)total : kNumSMs;
    conv_tc2_kernel<BN, KIND, FOLD, XR><<<grid, TC_THREADS, SMEM, st>>>(p, wk, mh, ml, ma);
    G6D_CHECK_LAUNCH("g6d_conv_tc");
    return G6D_OK;
}

// elementwise operand split of an fp32 array (detector reference features used as kernels)
__global__ void split_tf32_kernel(const float* __restrict__ in, float* __restrict__ hi, float* __restrict__ lo, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = in[i];
    const float h = to_tf32(v);
    hi[i] = h;
    lo[i] = to_tf32(v - h);
}
__device__ __forceinline__ void split_f16_scalar(float v, __half& h, __half& l) {
    uint32_t hh, ll;
    split_f16x2(v, 0.f, hh, ll);
    h = __ushort_as_half((unsigned short)(hh & 0xffffu));
    l = __ushort_as_half((unsigned short)(ll & 0xffffu));
}
// rows of K-major operands, K a multiple of 64: position p of every 64-block comes from source f16_k_source(p)
__global__ void split_f16_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    split_f16_scalar(in[(i & ~63ll) + f16_k_source((int)(i & 63))], hi[i], lo[i]);
}

// Activation [rows, ics] (channels [ico, ico + Cin)) -> split form [rows, 2 Cin] fp16 for the im2col A loads: channel
// block cb of a row holds hi at [128 cb, 128 cb + 64) and lo at [128 cb + 64, 128 cb + 128), position p from channel
// 64 cb + f16_k_source(p).  A thread makes one 16-byte chunk of each from the same two float4 loads and the same
// split_f16x2 calls as a producer thread of conv_tc2_kernel, so the tiles are bit-identical.  With a prologue
// (G6D_TC_PRENORM) every element is transformed by prologue4 first, as the producers transform every in-bounds
// element; the padding stays zero, as the im2col map fills it after this pass.  plane = D * H * W pixels per image.
__global__ void split_input_f16_kernel(const float* __restrict__ x, int ics, int ico, int Cin, long long rows,
                                       long long plane, int pro, const float* __restrict__ ps, const float* __restrict__ pb,
                                       long long group_rows, __half* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int chunks = Cin / 8;
    if (i >= rows * chunks) return;
    const long long r = i / chunks;
    const int q = (int)(i - r * chunks), cb = q >> 3, c = q & 7;
    const float* src = x + r * ics + ico + cb * 64 + 4 * c;
    float4 a = __ldg(reinterpret_cast<const float4*>(src));
    float4 b = __ldg(reinterpret_cast<const float4*>(src + 32));
    if (pro != G6D_PRO_NONE) {
        const long long img = r / plane, sp = r - img * plane;
        a = prologue4(a, pro, ps, pb, Cin, group_rows, img, sp, cb * 64 + 4 * c);
        b = prologue4(b, pro, ps, pb, Cin, group_rows, img, sp, cb * 64 + 32 + 4 * c);
    }
    uint4 h, l;
    split_f16x2(a.x, a.y, h.x, l.x);
    split_f16x2(a.z, a.w, h.y, l.y);
    split_f16x2(b.x, b.y, h.z, l.z);
    split_f16x2(b.z, b.w, h.w, l.w);
    __half* row = out + r * 2 * Cin + cb * 128;
    *reinterpret_cast<uint4*>(row + 8 * c) = h;
    *reinterpret_cast<uint4*>(row + 64 + 8 * c) = l;
}

// [Cout, Cin, taps] (reference layout) -> hi/lo [rows_pad, taps*Cin_pad], K index = tap*Cin_pad + c
template <int KIND>
__global__ void pack_conv_weight_tc_kernel(const float* __restrict__ w, void* __restrict__ hi, void* __restrict__ lo,
                                           int Cout, int Cin, int Cin_pad, int taps, int rows_pad,
                                           const float* __restrict__ scale) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long K = (long long)taps * Cin_pad;
    if (i >= K * rows_pad) return;
    const int o = (int)(i / K);
    const long long k = i % K;
    const int tap = (int)(k / Cin_pad);
    int c = (int)(k % Cin_pad);
    if constexpr (KIND == G6D_TC_F16) c = (c & ~63) + f16_k_source(c & 63);       // K order of the fp16 K-block
    float v = 0.f;
    if (o < Cout && c < Cin) {
        v = w[((long long)o * Cin + c) * taps + tap];
        if (scale) v *= scale[o];
    }
    if constexpr (KIND == G6D_TC_TF32) {
        const float h = to_tf32(v);
        static_cast<float*>(hi)[i] = h;
        static_cast<float*>(lo)[i] = to_tf32(v - h);
    } else {
        split_f16_scalar(v, static_cast<__half*>(hi)[i], static_cast<__half*>(lo)[i]);
    }
}

// ==========================================================================================
// conv_tcflat_kernel: stride-1 convolutions with A-operand reuse across taps.
//
// The output positions of one image plane are enumerated over the PADDED width Wp = W + 2*pw:
// f = y*Wp + x.  Tap (ky,kx) of output f reads padded-input position f + ky*Wp + kx, so for a
// tile of 128 consecutive f the A operand of EVERY tap is a window of 128 consecutive rows of
// one shared-memory buffer holding padded-input positions [f0, f0 + 127 + (kh-1)*Wp + kw-1]:
// the tap is selected by the wgmma descriptor's start address (+shift*128 B; the 128B swizzle is a
// function of the absolute smem address, checked by g6d_debug_desc_shift).  The producers
// therefore gather (and prologue-transform, and hi/lo split) each input element ONCE per channel
// block instead of once per tap: 9x less producer work / L2 traffic for 3x3.  Columns x >= Wo of the
// padded enumeration are computed and dropped.  A unit is one (channel block, kz) pair; B tiles stream
// by TMA per (unit, tap), issued by one consumer thread b_stages blocks ahead of the MMAs.
struct ConvFlatP {
    const float* x; const float* bias; const float* ps; const float* pb; float* y; float* ws;
    int B, D, H, W, Cin, ics, ico, Cout, kd, kh, kw, pd, ph, pw, Do, Ho, Wo, ocs, oco, pro, act;
    long long group_rows;
    int Wp, tiles_per_plane, seg_rows, rows_pad, cblocks;
    int a_stages, b_stages, splits, cb_per_split, M;
    double* stats; long long stats_rows;
};

template <int BN, int KIND>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tcflat_kernel(const ConvFlatP p, const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo) {
    using KC = KindCfg<KIND>;
    constexpr int NMAIN = AccCfg<BN>::NMAIN;
    constexpr int B_BYTES = BN * 128;
    constexpr int BK = KC::BK, NV = KC::NV;
    constexpr int RSTEP = TC_PRODUCER_WARPS * 4;         // rows r0 + RSTEP*j of a trip
    constexpr int ROWS = TC_BM / RSTEP;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const int A_TILE = p.rows_pad * 128;                 // one of hi / lo
    const uint32_t a_base = base;
    const uint32_t b_base = base + p.a_stages * 2 * A_TILE;
    const uint32_t bar_base = b_base + p.b_stages * 2 * B_BYTES;
    auto a_hi = [&](int s) { return a_base + s * 2 * A_TILE; };
    auto a_lo = [&](int s) { return a_base + s * 2 * A_TILE + A_TILE; };
    auto b_hi = [&](int s) { return b_base + s * 2 * B_BYTES; };
    auto b_lo = [&](int s) { return b_base + s * 2 * B_BYTES + B_BYTES; };
    auto a_full = [&](int s) { return bar_base + 8 * s; };
    auto a_empty = [&](int s) { return bar_base + 8 * (4 + s); };
    auto b_full = [&](int s) { return bar_base + 8 * (8 + s); };
    auto b_empty = [&](int s) { return bar_base + 8 * (12 + s); };
    const uint32_t bar_off = (bar_base - base);
    int* rowtab = reinterpret_cast<int*>(base_ptr + bar_off + 256);   // [seg_rows]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int tile = blockIdx.x;
    const int t_in_plane = tile % p.tiles_per_plane; tile /= p.tiles_per_plane;
    const int zo = tile % p.Do;
    const int b = tile / p.Do;
    const int f0 = t_in_plane * TC_BM;
    const int n_base = blockIdx.y * BN;
    const int split = blockIdx.z;
    const int cb_begin = split * p.cb_per_split;
    const int cb_end = min(p.cblocks, cb_begin + p.cb_per_split);
    const int nunits = (cb_end - cb_begin) * p.kd;

    // ---- setup: row table (element offset of each gathered row inside its image plane, -1 = zero)
    for (int i = threadIdx.x; i < p.seg_rows; i += blockDim.x) {
        const int g = f0 + i;                                     // padded-input flat position
        const int yy = g / p.Wp - p.ph, xx = g % p.Wp - p.pw;
        rowtab[i] = ((unsigned)yy < (unsigned)p.H && (unsigned)xx < (unsigned)p.W) ? yy * p.W + xx : -1;
    }
    if (threadIdx.x == TC_ISSUER) {
        for (int s = 0; s < 4; ++s) {
            mbar_init(a_full(s), TC_PRODUCER_WARPS);
            mbar_init(a_empty(s), TC_CONSUMER_WARPS);
            mbar_init(b_full(s), 1);
            mbar_init(b_empty(s), TC_CONSUMER_WARPS);
        }
        fence_barrier_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_lo) : "memory");
    }
    __syncthreads();

    if (warp < TC_PRODUCER_WARPS) {
        setmaxnreg_dec<TC_PRODUCER_REGS>();
        // =============================== A producers ===============================
        const int chunk = threadIdx.x & 7;
        const int cofs = chunk * 4;                             // channels [cofs, cofs+4) (+32 for the 2nd load), see f16_k_source
        const int r0 = threadIdx.x >> 3;                        // rows r0 + RSTEP*j
        const long long plane = (long long)p.H * p.W;
        const long long gi = (long long)b / p.group_rows;
        const bool relu = p.pro == G6D_PRO_AFFINE_RELU;
        // Software pipeline over (unit, TC_BM-row trip) with a ring of NB register slots: the global loads of
        // the next NB-1 trips (possibly of the next unit: they only touch registers, so they do not wait for
        // the stage to be free) are in flight while a trip is transformed and stored.  Without it every trip
        // paid a full L2 round trip before its first st.shared.
        // A slot holds one float4 column (e = tt % NV) of a trip, see FLAT_RING.
        constexpr int NB = FLAT_RING;
        const int trips = (p.seg_rows + TC_BM - 1) / TC_BM;
        const int total = nunits * trips * NV;
        float4 v[NB][ROWS]; int off[NB][ROWS];
        auto unit_of = [&](int tt, int& u, int& rbase, int& cb, int& kz) {
            tt /= NV;
            u = tt / trips; rbase = (tt - u * trips) * TC_BM;
            cb = cb_begin + u / p.kd;
            kz = u % p.kd;
        };
        auto issue = [&](int tt, int q, int e) {
            int u, rbase, cb, kz;
            unit_of(tt, u, rbase, cb, kz);
            const int zz = zo + kz - p.pd;
            const bool zok = (unsigned)zz < (unsigned)p.D;
            const float* xplane = p.x + ((long long)b * p.D + (zok ? zz : 0)) * plane * p.ics + p.ico + cb * BK + cofs + 32 * e;
#pragma unroll
            for (int j = 0; j < ROWS; ++j) {
                const int r = rbase + r0 + RSTEP * j;
                off[q][j] = (r < p.seg_rows && zok) ? rowtab[r] : -1;
                v[q][j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (off[q][j] >= 0) v[q][j] = __ldg(reinterpret_cast<const float4*>(xplane + (long long)off[q][j] * p.ics));
            }
        };
        auto store = [&](int tt, int q, int e) {
            int u, rbase, cb, kz;
            unit_of(tt, u, rbase, cb, kz);
            const int s = u % p.a_stages;
            const int zz = zo + kz - p.pd;
            const int c = cb * BK + cofs + 32 * e;
            if (rbase == 0 && e == 0) mbar_wait(a_empty(s), ((u / p.a_stages) & 1) ^ 1, 1, u);
#pragma unroll
            for (int j = 0; j < ROWS; ++j) {
                const int r = rbase + r0 + RSTEP * j;
                if (r >= p.rows_pad) continue;
                if (p.pro != G6D_PRO_NONE && off[q][j] >= 0) {
                    const float4* scp; const float4* shp;
                    if (p.pro == G6D_PRO_CORR) {
                        const long long sp = (long long)zz * plane + off[q][j];
                        scp = reinterpret_cast<const float4*>(p.ps + sp * p.Cin + c);
                        shp = reinterpret_cast<const float4*>(p.pb + c);
                    } else {
                        scp = reinterpret_cast<const float4*>(p.ps + gi * p.Cin + c);
                        shp = reinterpret_cast<const float4*>(p.pb + gi * p.Cin + c);
                    }
                    v[q][j] = affine4(v[q][j], __ldg(scp), __ldg(shp), relu);
                }
                const uint32_t so = r * 128 + ((chunk ^ (r & 7)) << 4);
                split_store<KIND>(a_hi(s) + so, a_lo(s) + so, v[q][j], e);
            }
            if (rbase + TC_BM >= p.seg_rows && e == NV - 1) {     // last column of the unit: publish the stage
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) mbar_arrive(a_full(s));
            }
        };
#pragma unroll
        for (int q = 0; q < NB - 1; ++q)
            if (q < total) issue(q, q, q % NV);
        for (int tt = 0; tt < total; tt += NB) {
#pragma unroll
            for (int q = 0; q < NB; ++q) {
                if (tt + q < total) {
                    if (tt + q + NB - 1 < total) issue(tt + q + NB - 1, (q + NB - 1) % NB, (tt + q + NB - 1) % NV);
                    store(tt + q, q, (tt + q) % NV);
                }
            }
        }
    } else {
        // =============================== consumer warpgroups ===============================
        setmaxnreg_inc<TC_CONSUMER_REGS>();
        const int cw = warp - TC_PRODUCER_WARPS;
        const uint32_t a_row = (cw >> 2) * 64 * 128;   // this warpgroup's 64 rows of the A window
        const bool issuer = threadIdx.x == TC_ISSUER;
        const int taps = p.kh * p.kw;
        const int nb_total = nunits * taps;
        int lb = 0;                                    // next B block the issuer loads
        auto load_b = [&]() {
            if (lb >= nb_total) return;
            const int u = lb / taps, t = lb % taps;
            const int cb = cb_begin + u / p.kd, kz = u % p.kd;
            const int s = lb % p.b_stages;
            mbar_wait(b_empty(s), ((lb / p.b_stages) & 1) ^ 1, 3, lb);
            mbar_expect_tx(b_full(s), 2 * B_BYTES);
            const int k = (kz * taps + t) * p.Cin + cb * BK;
            tma_load_2d(b_hi(s), &map_hi, b_full(s), k, n_base);
            tma_load_2d(b_lo(s), &map_lo, b_full(s), k, n_base);
            ++lb;
        };
        // the wgmma group of B block q has completed: free its B stage and, after a unit's last tap, its A stage
        auto release = [&](int q) {
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(b_empty(q % p.b_stages));
                if (q % taps == taps - 1) mbar_arrive(a_empty((q / taps) % p.a_stages));
            }
            if (issuer) load_b();
        };
        if (issuer)
            for (int i = 0; i < p.b_stages; ++i) load_b();

        float acc[NMAIN][BN / 2];
        float cross[BN / 2];
        zero_acc<BN, NMAIN>(acc, cross);
        // B block bi = (unit u, tap t) = (bi / taps, bi % taps) uses main accumulator bi % NMAIN
        for (int b0 = 0; b0 < nb_total; b0 += NMAIN) {
#pragma unroll
            for (int a = 0; a < NMAIN; ++a) {
                const int bi = b0 + a;
                if (bi < nb_total) {
                    const int u = bi / taps, t = bi - u * taps;
                    const int sa = u % p.a_stages, sb = bi % p.b_stages;
                    if (t == 0) mbar_wait(a_full(sa), (u / p.a_stages) & 1, 4, u);
                    mbar_wait(b_full(sb), (bi / p.b_stages) & 1, 5, bi);
                    const int shift = (t / p.kw) * p.Wp + (t % p.kw);     // rows
                    mma_stage<BN, KIND>(acc[a], cross, a_hi(sa) + shift * 128 + a_row, a_lo(sa) + shift * 128 + a_row, b_hi(sb),
                                        b_lo(sb));
                    wgmma_wait<1>();
                    if (bi > 0) release(bi - 1);
                }
            }
        }
        wgmma_wait<0>();
        if (nb_total > 0) release(nb_total - 1);

        // =============================== epilogue ===============================
        const bool partial = p.splits > 1;
        const long long m_plane = ((long long)b * p.Do + zo) * p.Ho * p.Wo;
        float* dst[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int f = f0 + 16 * cw + (lane >> 2) + 8 * h;
            const int yo = f / p.Wp, xo = f % p.Wp;
            const long long m = m_plane + (long long)yo * p.Wo + xo;
            dst[h] = (yo < p.Ho && xo < p.Wo) ? (partial ? p.ws + ((long long)split * p.M + m) * p.Cout + n_base
                                                         : p.y + m * p.ocs + p.oco + n_base)
                                              : nullptr;
        }
        const bool vec2 = partial ? (p.Cout & 1) == 0
                                  : ((p.ocs & 1) == 0 && (p.oco & 1) == 0 && (reinterpret_cast<uintptr_t>(p.y) & 7) == 0);
        // tiles never span planes and a group is made of whole planes
        epilogue_tile<BN, KIND>(acc, cross, nb_total < NMAIN ? nb_total : NMAIN, dst[0], dst[1], n_base, p.Cout, p.bias,
                                p.act, partial, vec2, p.stats, m_plane / p.stats_rows, lane);
    }
}


// The A-reuse kernel's parameters for a descriptor that fill_tc_params has accepted, or false when the
// shape does not suit that kernel: it needs stride 1, more than one tap, image planes that fill most of
// their 128-row tiles, and room for two A stages of the full halo and three B stages.
static bool fill_flat_params(const g6d_conv_desc* d, int kind, ConvFlatP& p, int* smem_bytes) {
    if (d->stride != 1 || d->kd * d->kh * d->kw == 1) return false;       // 1x1: nothing to reuse
    const int Do = d->Do, Ho = d->Ho, Wo = d->Wo;
    const int bn = tc_block_n(d->Cout);
    const int Wp = d->W + 2 * d->pw;
    const int rows = TC_BM + (d->kh - 1) * Wp + d->kw - 1;
    const int budget = 220 * 1024;
    const int b_stage = 2 * bn * 128;
    // tiles never span image planes: small planes (selector 4x4 / 8x8 maps) would leave most of a
    // 128-row tile empty -> keep those on the batch-flattened kernel
    {
        const long long tiles = ((long long)Ho * Wp + TC_BM - 1) / TC_BM;
        if ((long long)Ho * Wo * 100 < tiles * TC_BM * 60) return false;
    }
    const long long a_stage = 2ll * ((rows + 7) / 8 * 8) * 128;
    const int tab_bytes = 4 * rows;
    int a_st = 2, b_st = 3;
    long long used = a_st * a_stage + b_st * b_stage + tab_bytes + 2048;
    if (used > budget) return false;
    while (b_st < 4 && used + b_stage <= budget) { ++b_st; used += b_stage; }
    while (a_st < 4 && used + a_stage <= budget) { ++a_st; used += a_stage; }
    p.B = d->B; p.D = d->D; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.ics = d->in_cstride; p.ico = d->in_coff;
    p.Cout = d->Cout; p.kd = d->kd; p.kh = d->kh; p.kw = d->kw; p.pd = d->pd; p.ph = d->ph; p.pw = d->pw;
    p.Do = Do; p.Ho = Ho; p.Wo = Wo; p.ocs = d->out_cstride; p.oco = d->out_coff; p.pro = d->prologue; p.act = d->act;
    p.group_rows = d->group_rows > 0 ? d->group_rows : 1;
    p.Wp = Wp; p.tiles_per_plane = (Ho * Wp + TC_BM - 1) / TC_BM;
    p.seg_rows = rows; p.rows_pad = (rows + 7) / 8 * 8; p.cblocks = d->Cin / kind_bk(kind);
    p.M = d->B * Do * Ho * Wo;
    p.a_stages = a_st; p.b_stages = b_st;
    *smem_bytes = (int)(a_st * a_stage) + b_st * b_stage + 256 + tab_bytes + 1024 + 64;
    // split over channel blocks when the tile grid cannot fill the machine, or to bound accumulate chains
    const long long plan_b = d->plan_rows > 0 ? d->plan_rows / ((long long)Do * Ho * Wo) : d->B;  // see g6d_conv_desc
    const long long ctas = plan_b * Do * p.tiles_per_plane * ((d->Cout + bn - 1) / bn);
    const long long K = (long long)d->Cin * d->kd * d->kh * d->kw;
    int splits = 1;
    if (ctas < kNumSMs && p.cblocks >= 2) splits = (int)((kNumSMs + ctas - 1) / ctas);
    const int nmain = tc_nmain(bn);
    const long long chain = d->max_chain_k > 0 ? (long long)d->max_chain_k * nmain : (K > TC_MAX_K_PER_CHAIN ? TC_MAX_K_PER_CHAIN * nmain : 0);
    if (chain > 0) { const int ms = (int)((K + chain - 1) / chain); splits = splits < ms ? ms : splits; }
    splits = splits > p.cblocks ? p.cblocks : splits;
    splits = splits < 1 ? 1 : splits;
    p.cb_per_split = (p.cblocks + splits - 1) / splits;
    p.splits = (p.cblocks + p.cb_per_split - 1) / p.cb_per_split;
    return true;
}

// The fused moments conv_tcflat_kernel's epilogue adds, from the output of a layer that ran on the persistent kernel
// in that kernel's K order instead (G6D_TC_REUSE_IM2COL, one K split): the same 16-row slices of each plane's padded
// enumeration f = yo * Wp + xo (columns xo >= Wo count as zeros) through slice_moments.  So the fp32 partials are the
// same; the fp64 sums of a plane's slices are added in another order (the A-reuse kernel's atomics have no fixed order
// either).  The persistent kernel's own slices (16 output rows) would round differently.  A block sums one plane for
// 8 channels: its 8 warps take every 8th slice, then one atomic pair per channel.
__global__ void __launch_bounds__(256) flat_moments_kernel(const float* __restrict__ y, int ocs, int oco, int Cout, int Ho, int Wo,
                                                           int Wp, int slices_per_plane, double* __restrict__ stats,
                                                           long long stats_rows) {
    __shared__ double red[8][4][4];                              // [warp][lane < 4][(sum, sum^2) of column e = 0, 1]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long m_plane = (long long)blockIdx.x * Ho * Wo;
    const int n0 = 8 * blockIdx.y + 2 * (lane & 3);
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int sl = warp; sl < slices_per_plane; sl += 8) {
        const int f = sl * 16 + (lane >> 2);
        const float* row[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int yo = (f + 8 * h) / Wp, xo = (f + 8 * h) % Wp;
            row[h] = yo < Ho && xo < Wo ? y + (m_plane + (long long)yo * Wo + xo) * ocs + oco : nullptr;
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int n = n0 + e;
            const float2 s = slice_moments(row[0] && n < Cout ? row[0][n] : 0.f, row[1] && n < Cout ? row[1][n] : 0.f);
            acc[2 * e] += (double)s.x;
            acc[2 * e + 1] += (double)s.y;
        }
    }
    if (lane < 4)
        for (int q = 0; q < 4; ++q) red[warp][lane][q] = acc[q];
    __syncthreads();
    if (threadIdx.x < 16) {
        const int l = threadIdx.x >> 2, q = threadIdx.x & 3, n = 8 * blockIdx.y + 2 * l + (q >> 1);
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w][l][q];
        if (n < Cout) atomicAdd(stats + ((m_plane / stats_rows) * Cout + n) * 2 + (q & 1), t);
    }
}

template <int BN, int KIND>
static int launch_flat(const ConvFlatP& p, int smem, const CUtensorMap& mh, const CUtensorMap& ml, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv_tcflat_kernel<BN, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) { set_error("g6d_conv_tc(flat): cannot opt in to shared memory: %s", cudaGetErrorString(e)); return G6D_ECUDA; }
        configured = true;
    }
    dim3 grid((unsigned)((long long)p.B * p.Do * p.tiles_per_plane), ceil_div(p.Cout, BN), p.splits);
    conv_tcflat_kernel<BN, KIND><<<grid, TC_THREADS, smem, st>>>(p, mh, ml);
    G6D_CHECK_LAUNCH("g6d_conv_tc(flat)");
    return G6D_OK;
}

// What runs for one descriptor.  fill_tc_params validates it; the A-reuse kernel then takes the shapes it
// suits and the persistent kernel the rest.  Every entry point below is built on make_plan, so they all
// accept the same descriptors and agree on the kernel and its splits.
struct ConvPlan {
    ConvTcP tc;                // the validated descriptor; the persistent kernel's parameters
    ConvFlatP flat;            // the A-reuse kernel's parameters when use_flat
    bool use_flat;
    int bn, splits, flat_smem;
    long long split_in_off;    // byte offset of the split input in the workspace (tc.split_in)
    long long ws_bytes;        // workspace: split-K partials (none when folded), then the split input
};

// G6D_TC_FOLD_SPLITS: the K splits of a persistent split-input plan run back to back in the CTA of their tile, which
// keeps their running sum in registers and stores the total in the split-K reduce's order (no partials, no reduce pass,
// same bits).  A tile's splits then take one CTA, so the grid loses the splits' parallelism: fold only when the waves of
// S-chain tiles, ceil(T / P) S, are within TC_FOLD_SLACK of the waves of single chains, ceil(T S / P).  The slack is what
// the saved partial traffic and reduce pass pay for, measured per layer on an H100 (DESIGN.md section 5): folding was
// faster at every ratio up to 1.143 and 0-4 % slower from 1.154.
constexpr double TC_FOLD_SLACK = 0.15;

static bool fold_ok(const ConvPlan& pl) {
    if (pl.use_flat || !pl.tc.split_in || pl.splits < 2) return false;
    const long long T = (long long)ceil_div(pl.tc.M, TC_BM) * ceil_div(pl.tc.Cout, pl.bn), S = pl.splits;
    return (double)(ceil_div(T, kNumSMs) * S) <= (1.0 + TC_FOLD_SLACK) * (double)ceil_div(T * S, kNumSMs);
}

// The persistent kernel loads A by TMA im2col from a pre-split copy of the input for fp16 multi-tap 2-D
// convolutions with stride 1 and no prologue: the gather, split and swizzle of 8 producer warps (each input
// element once per tap, 16 KB in flight per SM) become two bulk copies per K-block.  The split pass reads and
// writes the input once.  The bounding box of the im2col map is the output plane shifted by the padding.
// G6D_TC_PRENORM extends this to layers with a prologue: the split pass applies it (see split_input_f16_kernel).
// G6D_TC_REUSE_IM2COL extends it to volumes through the rank-5 map, whose box corners the driver only takes in
// [-16, 15]; a volume outside that range keeps the producer warps.
static bool split_input_ok(const g6d_conv_desc* d, int kind, int flags, bool use_flat) {
    if (use_flat || kind != G6D_TC_F16 || (d->prologue != G6D_PRO_NONE && !(flags & G6D_TC_PRENORM)) || d->stride != 1 ||
        d->kd * d->kh * d->kw == 1)
        return false;
    if (!split_input_rank5(d)) return d->kw <= 64 && d->kh <= 64 && d->pw < 64 && d->ph < 64;
    auto corners_ok = [](int k, int pad) { return k <= 16 && pad <= 16 && pad - (k - 1) >= -16 && pad - (k - 1) <= 15; };
    return (flags & G6D_TC_REUSE_IM2COL) && corners_ok(d->kw, d->pw) && corners_ok(d->kh, d->ph) && corners_ok(d->kd, d->pd);
}

// One A box per row of taps: in the A-reuse kernel's K order the kw taps of a (channel block, kz, ky) group are kw
// consecutive K-blocks, and over an enumeration of Wp = Wo + kw - 1 columns per output row, row j + kx of ONE im2col box
// of roundup8(128 + kw - 1) pixels at kx = 0 is tap kx of row j (a real column xp < Wo never wraps past Wp).  So the
// TMA thread loads one box pair per group instead of one per K-block (kw times fewer A bytes, with (kw - 1) / Wp more
// rows), the consumers read tap kx through a descriptor shifted by kx rows, and the epilogue drops the padded columns.
// Every real output element sums the same products in the same order.  Measured on an H100 (DESIGN.md section 5), the
// saved A traffic pays for the padding at BN 64, where the weight tile is small and A is two thirds of the operand
// bytes; at BN 128 it did not.
static bool xr_ok(const g6d_conv_desc* d, const ConvPlan& pl) {
    if (!pl.tc.split_in || !pl.tc.reuse_order || pl.bn != 64 || d->kw < 2 || d->kw > 17) return false;
    if (split_input_rank5(d) && d->pw > 15) return false;     // the rank-5 map's upper W corner becomes pw
    return (long long)pl.tc.M / pl.tc.Wo * (pl.tc.Wo + d->kw - 1) < (1ll << 31);
}

static int make_plan(const g6d_conv_desc* d, int kind, int flags, ConvPlan& pl) {
    G6D_REQUIRE((flags & ~(G6D_TC_PRENORM | G6D_TC_REUSE_IM2COL | G6D_TC_FOLD_SPLITS)) == 0, "g6d_conv_tc: bad flags %d", flags);
    const int rc = fill_tc_params(d, kind, pl.tc);
    if (rc != G6D_OK) return rc;
    pl.use_flat = fill_flat_params(d, kind, pl.flat, &pl.flat_smem);
    pl.tc.reuse_order = 0;
    if (pl.use_flat && (flags & G6D_TC_REUSE_IM2COL) && split_input_ok(d, kind, flags, false)) {
        // the persistent kernel with im2col A, in the A-reuse kernel's K order and K splits (bit-identical)
        pl.use_flat = false;
        pl.tc.reuse_order = 1;
        pl.tc.kb_per_split = pl.flat.cb_per_split * d->kd * d->kh * d->kw;
        pl.tc.splits = pl.flat.splits;
    }
    pl.bn = tc_block_n(d->Cout);
    pl.splits = pl.use_flat ? pl.flat.splits : pl.tc.splits;
    pl.tc.split_in = split_input_ok(d, kind, flags, pl.use_flat) ? 1 : 0;
    pl.tc.fold = (flags & G6D_TC_FOLD_SPLITS) && fold_ok(pl) ? 1 : 0;
    pl.tc.xr = xr_ok(d, pl) ? 1 : 0;
    if (pl.tc.xr) {
        pl.tc.Wp = pl.tc.Wo + d->kw - 1;
        pl.tc.Mp = (int)((long long)pl.tc.M / pl.tc.Wo * pl.tc.Wp);
        pl.tc.xr_rows = (TC_BM + d->kw - 1 + 7) / 8 * 8;
    }
    const long long partials =
        pl.splits > 1 && !pl.tc.fold ? (long long)pl.splits * pl.tc.M * pl.tc.Cout * (long long)sizeof(float) : 0;
    pl.split_in_off = (partials + 255) / 256 * 256;
    pl.ws_bytes = pl.tc.split_in
                      ? pl.split_in_off + (long long)d->B * d->D * d->H * d->W * d->Cin * 2 * (long long)sizeof(__half)
                      : partials;
    return G6D_OK;
}

// fused output statistics are possible when every 32-row epilogue slice lies in one group; the A-reuse
// kernel's tiles never span image planes, so its groups (and those of flat_moments_kernel) must also be made of
// whole planes
static bool stats_ok(const ConvPlan& pl, long long stats_rows) {
    if (stats_rows <= 0 || stats_rows % 32 != 0 || pl.tc.M % stats_rows != 0) return false;
    return !(pl.use_flat || pl.tc.reuse_order) || stats_rows % ((long long)pl.flat.Ho * pl.flat.Wo) == 0;
}

template <class P>
static void bind_tensors(P& p, const float* x, const float* bias, const float* ps, const float* pb, float* y, void* ws,
                         double* stats, long long stats_rows) {
    p.x = x; p.bias = bias; p.ps = ps; p.pb = pb; p.y = y; p.ws = static_cast<float*>(ws);
    p.stats = stats; p.stats_rows = stats ? stats_rows : 1;
}

template <int BN, int KIND>
static int launch_plan(const ConvPlan& pl, const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& ma, cudaStream_t st) {
    if (pl.use_flat) return launch_flat<BN, KIND>(pl.flat, pl.flat_smem, mh, ml, st);
    if constexpr (KIND == G6D_TC_F16) {                    // the split input, hence folding and x reuse, is fp16 only
        if constexpr (BN == 64)
            if (pl.tc.xr) return pl.tc.fold ? launch_tc2<BN, KIND, true, true>(pl.tc, mh, ml, ma, st)
                                            : launch_tc2<BN, KIND, false, true>(pl.tc, mh, ml, ma, st);
        if (pl.tc.fold) return launch_tc2<BN, KIND, true, false>(pl.tc, mh, ml, ma, st);
    }
    return launch_tc2<BN, KIND, false, false>(pl.tc, mh, ml, ma, st);
}
template <int KIND>
static int dispatch(const ConvPlan& pl, const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& ma, cudaStream_t st) {
    if (pl.bn == 128) return launch_plan<128, KIND>(pl, mh, ml, ma, st);
    if (pl.bn == 64) return launch_plan<64, KIND>(pl, mh, ml, ma, st);
    return launch_plan<32, KIND>(pl, mh, ml, ma, st);
}

}  // namespace g6d

using namespace g6d;

// Debug aid: copies the 8-int timeout record (0 = no timeout; else [1]=waiter role 1 A-producer/empty,
// 3 weight-TMA issuer/empty, 4 MMA/full_a, 5 MMA/full_b, 6 x-reuse box TMA/box empty, 7 x-reuse MMA/box full; [2]=iteration;
// [3]=parity; [4..6]=block; [7]=thread) and clears it.  Synchronises the device.
extern "C" int g6d_conv_tc_debug(int* host_out8) {
    G6D_REQUIRE(host_out8 != nullptr, "g6d_conv_tc_debug: null");
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("g6d_conv_tc_debug: sync: %s", cudaGetErrorString(e)); return G6D_ECUDA; }
    e = cudaMemcpyFromSymbol(host_out8, g_tc_timeout, sizeof(int) * 8);
    if (e != cudaSuccess) { set_error("g6d_conv_tc_debug: %s", cudaGetErrorString(e)); return G6D_ECUDA; }
    int zeros[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    cudaMemcpyToSymbol(g_tc_timeout, zeros, sizeof(zeros));
    return G6D_OK;
}

extern "C" int g6d_conv_tc_supported(const g6d_conv_desc* d, int kind) {
    ConvPlan pl{};
    return make_plan(d, kind, 0, pl) == G6D_OK ? 1 : 0;
}

extern "C" long long g6d_conv_tc_workspace_bytes_ex(const g6d_conv_desc* desc, int kind, int flags) {
    ConvPlan pl{};
    if (make_plan(desc, kind, flags, pl) != G6D_OK) return -1;
    return pl.ws_bytes;
}

extern "C" long long g6d_conv_tc_workspace_bytes(const g6d_conv_desc* desc, int kind) {
    return g6d_conv_tc_workspace_bytes_ex(desc, kind, 0);
}

extern "C" int g6d_conv_tc_stats_supported(const g6d_conv_desc* desc, int kind, long long stats_rows) {
    ConvPlan pl{};
    return make_plan(desc, kind, 0, pl) == G6D_OK && stats_ok(pl, stats_rows) ? 1 : 0;
}

extern "C" int g6d_conv_tc_plan_ex(const g6d_conv_desc* desc, int kind, int flags, int* out4) {
    G6D_REQUIRE(out4 != nullptr, "g6d_conv_tc_plan: null output");
    ConvPlan pl{};
    const int rc = make_plan(desc, kind, flags, pl);
    if (rc != G6D_OK) return rc;
    out4[0] = pl.use_flat ? 1 : 0;
    out4[1] = pl.bn;
    out4[2] = pl.splits;
    out4[3] = pl.tc.split_in;
    return G6D_OK;
}

extern "C" int g6d_conv_tc_plan_v2(const g6d_conv_desc* desc, int kind, int flags, int* out, int n) {
    G6D_REQUIRE(out != nullptr && n > 0, "g6d_conv_tc_plan_v2: null output");
    ConvPlan pl{};
    const int rc = make_plan(desc, kind, flags, pl);
    if (rc != G6D_OK) return rc;
    const int v[6] = {pl.use_flat ? 1 : 0, pl.bn, pl.splits, pl.tc.split_in, pl.tc.fold, pl.tc.xr};
    for (int i = 0; i < n && i < 6; ++i) out[i] = v[i];
    return G6D_OK;
}

extern "C" int g6d_conv_tc_plan(const g6d_conv_desc* desc, int kind, int* out4) {
    return g6d_conv_tc_plan_ex(desc, kind, 0, out4);
}

extern "C" int g6d_conv_tc_ex(const g6d_conv_desc* desc, const float* x, const void* w_hi, const void* w_lo, int w_rows,
                              int kind, const float* bias, const float* pro_scale, const float* pro_shift, float* y,
                              void* ws, double* stats, long long stats_rows, int flags, g6d_stream_t stream) {
    ConvPlan pl{};
    int rc = make_plan(desc, kind, flags, pl);
    if (rc != G6D_OK) return rc;
    const ConvTcP& p = pl.tc;
    if (stats) G6D_REQUIRE(stats_ok(pl, stats_rows), "g6d_conv_tc: fused statistics need groups of whole 32-row slices / planes (stats_rows %lld)", stats_rows);
    G6D_REQUIRE(x && w_hi && w_lo && y, "g6d_conv_tc: null tensor pointer");
    G6D_REQUIRE(w_rows >= p.Cout, "g6d_conv_tc: weight rows (%d) < Cout (%d)", w_rows, p.Cout);
    if (p.pro != G6D_PRO_NONE) G6D_REQUIRE(pro_scale && pro_shift, "g6d_conv_tc: prologue operands missing");
    if (pl.ws_bytes > 0) G6D_REQUIRE(ws != nullptr, "g6d_conv_tc: workspace required (%lld bytes)", pl.ws_bytes);
    cudaStream_t st = as_stream(stream);
    if (stats) {
        cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * (p.M / stats_rows) * p.Cout, st);
        if (e != cudaSuccess) { set_error("g6d_conv_tc: memset: %s", cudaGetErrorString(e)); return G6D_ECUDA; }
    }
    // in the A-reuse kernel's K order without K splits, the moments are those of its epilogue (flat_moments_kernel)
    const bool flat_moments = stats && p.reuse_order && pl.splits == 1;
    // folded, the split-K reduce's moments, taken from the final y by fold_moments_kernel
    const bool fold_moments = stats && p.fold;
    if (pl.use_flat) bind_tensors(pl.flat, x, bias, pro_scale, pro_shift, y, ws, stats, stats_rows);
    else bind_tensors(pl.tc, x, bias, pro_scale, pro_shift, y, ws, flat_moments || fold_moments ? nullptr : stats, stats_rows);
    CUtensorMap mh, ml, ma;
    if ((rc = make_weight_map(&mh, w_hi, w_rows, p.K, pl.bn, kind)) != G6D_OK) return rc;
    if ((rc = make_weight_map(&ml, w_lo, w_rows, p.K, pl.bn, kind)) != G6D_OK) return rc;
    memset(&ma, 0, sizeof(ma));
    if (p.split_in) {
        __half* xs = reinterpret_cast<__half*>(static_cast<char*>(ws) + pl.split_in_off);
        if ((rc = make_split_input_map(&ma, xs, desc, p.xr ? p.xr_rows : 0)) != G6D_OK) return rc;
        const long long plane = (long long)p.D * p.H * p.W, rows = p.B * plane, n = rows * (p.Cin / 8);
        split_input_f16_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, p.ics, p.ico, p.Cin, rows, plane, p.pro, pro_scale,
                                                                  pro_shift, p.group_rows, xs);
        G6D_CHECK_LAUNCH("g6d_conv_tc(split input)");
    }
    rc = kind == G6D_TC_F16 ? dispatch<G6D_TC_F16>(pl, mh, ml, ma, st) : dispatch<G6D_TC_TF32>(pl, mh, ml, ma, st);
    if (rc != G6D_OK) return rc;
    if (flat_moments) {
        const ConvFlatP& f = pl.flat;
        dim3 grid((unsigned)((long long)f.B * f.Do), ceil_div(f.Cout, 8));
        flat_moments_kernel<<<grid, 256, 0, st>>>(y, f.ocs, f.oco, f.Cout, f.Ho, f.Wo, f.Wp, f.tiles_per_plane * TC_CONSUMER_WARPS,
                                                  stats, stats_rows);
        G6D_CHECK_LAUNCH("g6d_conv_tc(moments)");
    }
    if (fold_moments) {
        fold_moments_kernel<<<dim3(ceil_div(p.M, 32), ceil_div(p.Cout, 64)), 256, 0, st>>>(y, p.M, p.Cout, p.ocs, p.oco, stats,
                                                                                          stats_rows);
        G6D_CHECK_LAUNCH("g6d_conv_tc(fold moments)");
    }
    if (pl.splits > 1 && !p.fold) {
        launch_reduce(static_cast<float*>(ws), bias, y, p.M, p.Cout, pl.splits, p.ocs, p.oco, p.act, stats, stats_rows, st);
        G6D_CHECK_LAUNCH("g6d_conv_tc(split reduce)");
    }
    return G6D_OK;
}

extern "C" int g6d_conv_tc(const g6d_conv_desc* desc, const float* x, const void* w_hi, const void* w_lo, int w_rows,
                           int kind, const float* bias, const float* pro_scale, const float* pro_shift, float* y,
                           void* ws, double* stats, long long stats_rows, g6d_stream_t stream) {
    return g6d_conv_tc_ex(desc, x, w_hi, w_lo, w_rows, kind, bias, pro_scale, pro_shift, y, ws, stats, stats_rows, 0, stream);
}

extern "C" int g6d_split_operand(const float* in, void* hi, void* lo, long long n, int kind, g6d_stream_t stream) {
    G6D_REQUIRE(in && hi && lo && n > 0, "g6d_split_operand: bad args");
    G6D_REQUIRE(kind == G6D_TC_TF32 || kind == G6D_TC_F16, "g6d_split_operand: bad operand kind %d", kind);
    G6D_REQUIRE(kind != G6D_TC_F16 || (n & 63) == 0, "g6d_split_operand: fp16 operands are laid out in 64-element K-blocks (n = %lld)", n);
    if (kind == G6D_TC_F16)
        split_f16_kernel<<<ceil_div(n, 256), 256, 0, as_stream(stream)>>>(in, static_cast<__half*>(hi), static_cast<__half*>(lo), n);
    else
        split_tf32_kernel<<<ceil_div(n, 256), 256, 0, as_stream(stream)>>>(in, static_cast<float*>(hi), static_cast<float*>(lo), n);
    G6D_CHECK_LAUNCH("g6d_split_operand");
    return G6D_OK;
}

extern "C" int g6d_pack_conv_weight_tc(const float* w, void* out_hi, void* out_lo, int Cout, int Cin, int Cin_pad,
                                       int taps, int rows_pad, const float* cout_scale, int kind, g6d_stream_t stream) {
    G6D_REQUIRE(w && out_hi && out_lo && Cout > 0 && Cin > 0 && Cin_pad >= Cin && taps > 0 && rows_pad >= Cout,
                "g6d_pack_conv_weight_tc: bad args");
    G6D_REQUIRE(kind == G6D_TC_TF32 || kind == G6D_TC_F16, "g6d_pack_conv_weight_tc: bad operand kind %d", kind);
    const long long total = (long long)taps * Cin_pad * rows_pad;
    if (kind == G6D_TC_F16)
        pack_conv_weight_tc_kernel<G6D_TC_F16><<<ceil_div(total, 256), 256, 0, as_stream(stream)>>>(w, out_hi, out_lo, Cout, Cin,
                                                                                                    Cin_pad, taps, rows_pad, cout_scale);
    else
        pack_conv_weight_tc_kernel<G6D_TC_TF32><<<ceil_div(total, 256), 256, 0, as_stream(stream)>>>(w, out_hi, out_lo, Cout, Cin,
                                                                                                     Cin_pad, taps, rows_pad, cout_scale);
    G6D_CHECK_LAUNCH("g6d_pack_conv_weight_tc");
    return G6D_OK;
}

// ------------------------------------------------------------------------------------------
// Probe (debug/test only): does a K-major SWIZZLE_128B A operand tolerate a start address that is
// shifted by `shift` rows (shift*128 B, not 1024-aligned) when the data was written with the
// swizzle phase of its ABSOLUTE shared-memory row?  D[64 x 32] = A[shift .. shift+64) x B^T with
// K = 32, A[r][k] = r + k/64 (exact in fp32), B = 32x32 identity, so D[i][n] = shift + i + n/64.
// `mode` selects the descriptor's base_offset field: 0 -> 0, 1 -> (start_address >> 7) & 7.
namespace g6d {
__global__ void __launch_bounds__(128) desc_shift_probe_kernel(float* out, int shift, int mode) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* bp = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t a_base = base;                 // 96 rows x 128 B
    const uint32_t b_base = base + 96 * 128;      // 32 rows x 128 B (12288 is 1024-aligned)
    const int t = threadIdx.x;
    for (int r = t; r < 96; r += 128)
        for (int c = 0; c < 8; ++c) {
            float4 v = make_float4(r + (c * 4 + 0) / 64.f, r + (c * 4 + 1) / 64.f, r + (c * 4 + 2) / 64.f, r + (c * 4 + 3) / 64.f);
            *reinterpret_cast<float4*>(bp + r * 128 + ((c ^ (r & 7)) << 4)) = v;
        }
    for (int r = t; r < 32; r += 128)
        for (int c = 0; c < 8; ++c) {
            float4 v = make_float4(r == c * 4 ? 1.f : 0.f, r == c * 4 + 1 ? 1.f : 0.f, r == c * 4 + 2 ? 1.f : 0.f, r == c * 4 + 3 ? 1.f : 0.f);
            *reinterpret_cast<float4*>(bp + 96 * 128 + r * 128 + ((c ^ (r & 7)) << 4)) = v;
        }
    fence_proxy_async();
    __syncthreads();
    const uint32_t start = a_base + shift * 128;
    uint64_t da = gmma_desc_sw128(start);
    if (mode == 1) da |= (uint64_t)((start >> 7) & 7) << 49;
    const uint64_t db = gmma_desc_sw128(b_base);
    float d[16];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma<32, G6D_TC_TF32>(d, da + (uint64_t)(ks * 2), db + (uint64_t)(ks * 2), ks > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    const int warp = t >> 5, lane = t & 31;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int row = 16 * warp + (lane >> 2) + 8 * ((j >> 1) & 1), col = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
        out[row * 32 + col] = d[j];
    }
}
}  // namespace g6d

extern "C" int g6d_debug_desc_shift(float* out, int shift, int mode, g6d_stream_t stream) {
    G6D_REQUIRE(out && shift >= 0 && shift <= 31, "g6d_debug_desc_shift: bad args");
    g6d::desc_shift_probe_kernel<<<1, 128, 96 * 128 + 32 * 128 + 1024, g6d::as_stream(stream)>>>(out, shift, mode);
    G6D_CHECK_LAUNCH("g6d_debug_desc_shift");
    return G6D_OK;
}
