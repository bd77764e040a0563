// Detector-specific kernels: fused normalise/clip/upsample/resize/stack/score_conv/max-over-refs
// (D2 epilogue + D3 head) and the argmax decode (D4).
#include <cmath>

#include "common.cuh"

namespace g6d {

constexpr int kDetFuseMaxScales = 6;   // det_score_fuse_kernel is instantiated for 1..6 scales (NIN = 3..18)

struct DetFuseParams {
    g6d_det_maps maps;
    const float* w1; const float* b1; const float* w2; const float* b2;
    float* out;
    int qn;
};

__device__ __forceinline__ void bil_src(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
    float s = scale * ((float)dst + 0.5f) - 0.5f;   // align_corners=False, clamped at 0 (ATen)
    s = s < 0.f ? 0.f : s;
    i0 = (int)s;
    i0 = i0 > in_size - 1 ? in_size - 1 : i0;
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    l1 = s - (float)i0;
}

// One warp per output pixel; lanes stride over the reference views.  For each (pixel, ref) the 3S
// inputs are gathered straight from the raw per-level correlation maps: level l of a scale is
// nearest-upsampled by 2^l (detector.py:225-226: index >> l), normalised and clipped
// (detector.py:207-216) at the 4 bilinear taps of the (Hc,Wc)->(hs,ws) resize (detector.py:243),
// then blended.  score_conv (12->64 ReLU ->64, detector.py:159-163,246) runs in registers with
// the weights in shared memory, and the max over references (detector.py:247) is a warp max.
template <int NIN>
__global__ void __launch_bounds__(128) det_score_fuse_kernel(const DetFuseParams p) {
    constexpr int D = 64;
    __shared__ float w1s[D * NIN], b1s[D], b2s[D];
    __shared__ __align__(16) float w2s[D * D];
    for (int i = threadIdx.x; i < D * NIN; i += blockDim.x) w1s[i] = p.w1[i];
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) w2s[i] = p.w2[i];
    for (int i = threadIdx.x; i < D; i += blockDim.x) { b1s[i] = p.b1[i]; b2s[i] = p.b2[i]; }
    __syncthreads();
    const g6d_det_maps& M = p.maps;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
    const long long npix = (long long)p.qn * M.hs * M.ws;
    if (pix >= npix) return;
    const int x = (int)(pix % M.ws), y = (int)((pix / M.ws) % M.hs), qi = (int)(pix / ((long long)M.ws * M.hs));

    auto gather = [&](int r, float* in) {
        const bool valid = r < M.rfn;
#pragma unroll
        for (int s = 0; s < NIN / 3; ++s) {
            const int Hc = M.H[s][0], Wc = M.W[s][0];
            int y0, y1, x0, x1; float ly, lx;
            bil_src(y, (float)Hc / (float)M.hs, Hc, y0, y1, ly);
            bil_src(x, (float)Wc / (float)M.ws, Wc, x0, x1, lx);
            const float hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
            for (int l = 0; l < 3; ++l) {
                float v = 0.f;
                if (valid) {
                    const int Hl = M.H[s][l], Wl = M.W[s][l];
                    const float* mp = M.map[s][l] + (long long)qi * Hl * Wl * M.rfn + r;
                    auto tap = [&](int yy, int xx) {
                        const float raw = __ldg(mp + ((long long)(yy >> l) * Wl + (xx >> l)) * M.rfn);
                        const float n = (raw - M.mu[l]) * M.inv_sigma[l];
                        return fminf(fmaxf(n, -M.clip), M.clip);
                    };
                    v = hy * (hx * tap(y0, x0) + lx * tap(y0, x1)) + ly * (hx * tap(y1, x0) + lx * tap(y1, x1));
                }
                in[s * 3 + l] = v;
            }
        }
    };
    auto hidden = [&](const float* in, float* hid) {
#pragma unroll
        for (int h = 0; h < D; ++h) {
            float a = b1s[h];
#pragma unroll
            for (int i = 0; i < NIN; ++i) a = fmaf(w1s[h * NIN + i], in[i], a);
            hid[h] = fmaxf(a, 0.f);
        }
    };

    // references are processed 64 at a time (two per lane) so the hidden vectors stay in registers
    for (int r0 = 0; r0 < M.rfn; r0 += 64) {
        float in[NIN], hidA[D], hidB[D];
        const int ra = r0 + lane, rb = r0 + 32 + lane;
        gather(ra, in); hidden(in, hidA);
        gather(rb, in); hidden(in, hidB);
        const bool va = ra < M.rfn, vb = rb < M.rfn;
#pragma unroll 2
        for (int o = 0; o < D; ++o) {
            float a = b2s[o], b = a;
            const float4* wr = reinterpret_cast<const float4*>(&w2s[o * D]);
#pragma unroll
            for (int h4 = 0; h4 < D / 4; ++h4) {
                const float4 w = wr[h4];
                a = fmaf(w.x, hidA[h4 * 4 + 0], fmaf(w.y, hidA[h4 * 4 + 1], fmaf(w.z, hidA[h4 * 4 + 2], fmaf(w.w, hidA[h4 * 4 + 3], a))));
                b = fmaf(w.x, hidB[h4 * 4 + 0], fmaf(w.y, hidB[h4 * 4 + 1], fmaf(w.z, hidB[h4 * 4 + 2], fmaf(w.w, hidB[h4 * 4 + 3], b))));
            }
            float m = fmaxf(va ? a : -INFINITY, vb ? b : -INFINITY);
            m = warp_max(m);
            if (lane == 0) {
                float* dst = p.out + pix * D + o;
                *dst = r0 == 0 ? m : fmaxf(*dst, m);
            }
        }
    }
}

__global__ void det_parse_kernel(const float* __restrict__ scores, const float* __restrict__ scales,
                                 const float* __restrict__ offsets, int hs, int ws, int pool, float* __restrict__ out,
                                 long long* __restrict__ out_idx) {
    const int qi = blockIdx.x;
    const int n = hs * ws;
    const float* sc = scores + (long long)qi * n;
    // first-max argmax (torch.argmax returns the lowest index among ties and treats NaN as the
    // maximum, detector.py:91): candidate (v, i) beats (bv, bi) under that order
    auto beats = [](float v, int i, float bv, int bi) {
        const bool vn = v != v, bn = bv != bv;
        if (vn || bn) return vn && (!bn || i < bi);
        return v > bv || (v == bv && i < bi);
    };
    float bv = -INFINITY; int bi = 0x7fffffff;      // sentinel: loses to every real element (even -inf) on the index
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = sc[i];
        if (beats(v, i, bv, bi)) { bv = v; bi = i; }
    }
    __shared__ float sv[256]; __shared__ int si[256];
    sv[threadIdx.x] = bv; si[threadIdx.x] = bi;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            const float v = sv[threadIdx.x + o]; const int i = si[threadIdx.x + o];
            if (beats(v, i, sv[threadIdx.x], si[threadIdx.x])) { sv[threadIdx.x] = v; si[threadIdx.x] = i; }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int idx = min(max(si[0], 0), n - 1);
        const int y = idx / ws, x = idx % ws;
        const float ox = offsets[((long long)qi * n + idx) * 2 + 0], oy = offsets[((long long)qi * n + idx) * 2 + 1];
        out[qi * 4 + 0] = ((float)x + ox + 0.5f) * (float)pool - 0.5f;
        out[qi * 4 + 1] = ((float)y + oy + 0.5f) * (float)pool - 0.5f;
        out[qi * 4 + 2] = exp2f(scales[(long long)qi * n + idx]);
        out[qi * 4 + 3] = sv[0];
        out_idx[qi] = idx;
    }
}

// ---- multi-peak detection with greedy non-maximum suppression (g6d_det_parse_peaks) ----------------------------------
// The selection code is shared by the kernel and the host twin; only the decode differs (see det_peak_decode).
// first-max order of det_parse_kernel: NaN counts as the maximum, ties go to the lower flat index
__host__ __device__ __forceinline__ bool peak_beats(float v, int i, float bv, int bi) {
    const bool vn = v != v, bn = bv != bv;
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

// fp32 arithmetic that is never contracted into an FMA (the IoU's operation order is part of the contract)
__host__ __device__ __forceinline__ float pk_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ float pk_sub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ __forceinline__ float pk_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float pk_div(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}

struct PeakBox { float x0, y0, x1, y1, area; };

// the square of side box_size * scale centred at (x, y)
__host__ __device__ __forceinline__ PeakBox peak_box(float x, float y, float scale, float box_size) {
    const float side = pk_mul(box_size, scale), half = pk_mul(side, 0.5f);
    return {pk_sub(x, half), pk_sub(y, half), pk_add(x, half), pk_add(y, half), pk_mul(side, side)};
}

__host__ __device__ __forceinline__ float peak_iou(const PeakBox& a, const PeakBox& b) {
    const float iw = fmaxf(pk_sub(fminf(a.x1, b.x1), fmaxf(a.x0, b.x0)), 0.f);
    const float ih = fmaxf(pk_sub(fminf(a.y1, b.y1), fmaxf(a.y0, b.y0)), 0.f);
    const float inter = pk_mul(iw, ih);
    return pk_div(inter, pk_sub(pk_add(a.area, b.area), inter));
}

// det_parse_kernel's decode of cell idx: out = (x, y, scale, score).  On the device its compiled form is an fma.rn for the
// position and ex2.approx for the scale; the host twin uses std::fma and libm's exp2f (a few ulp apart in the scale).
__host__ __device__ __forceinline__ void det_peak_decode(const float* sc, const float* scl, const float* off, int idx, int ws,
                                                         int pool, float* out) {
    const int y = idx / ws, x = idx % ws;
    const float ox = off[(long long)idx * 2 + 0], oy = off[(long long)idx * 2 + 1];
#ifdef __CUDA_ARCH__
    out[0] = fmaf((float)x + ox + 0.5f, (float)pool, -0.5f);
    out[1] = fmaf((float)y + oy + 0.5f, (float)pool, -0.5f);
#else
    out[0] = std::fma((float)x + ox + 0.5f, (float)pool, -0.5f);
    out[1] = std::fma((float)y + oy + 0.5f, (float)pool, -0.5f);
#endif
    out[2] = exp2f(scl[idx]);
    out[3] = sc[idx];
}

// no cell within Chebyshev distance `radius` (window clipped at the border) beats cell i
__host__ __device__ __forceinline__ bool det_is_peak(const float* sc, int i, float v, int hs, int ws, int radius) {
    const int y = i / ws, x = i % ws;
    const int y0 = max(y - radius, 0), y1 = min(y + radius, hs - 1), x0 = max(x - radius, 0), x1 = min(x + radius, ws - 1);
    for (int yy = y0; yy <= y1; ++yy)
        for (int xx = x0; xx <= x1; ++xx) {
            const int j = yy * ws + xx;
            if (j != i && peak_beats(sc[j], j, v, i)) return false;
        }
    return true;
}

struct PeakArgs {
    int n_maps, hs, ws, pool, max_inst, radius;
    float nms_iou, box_size, min_score;
};

// Cell i can be the next instance after the last kept cell (last_v, last_i): it comes after it in the order (the greedy
// picks are strictly decreasing, so this also excludes every kept cell), clears min_score, is a peak and no kept box
// suppresses it.  `best` prunes: a cell that cannot beat the caller's running best skips the peak and IoU tests.
__host__ __device__ __forceinline__ bool peak_candidate(const float* sc, const float* scl, const float* off, int i, float v,
                                                        float last_v, int last_i, float bv, int bi, const PeakBox* kept, int n_kept,
                                                        const PeakArgs& a) {
    if (!(v >= a.min_score) || !peak_beats(last_v, last_i, v, i) || !peak_beats(v, i, bv, bi)) return false;
    if (!det_is_peak(sc, i, v, a.hs, a.ws, a.radius)) return false;
    float d[4];
    det_peak_decode(sc, scl, off, i, a.ws, a.pool, d);
    const PeakBox b = peak_box(d[0], d[1], d[2], a.box_size);
    for (int k = 0; k < n_kept; ++k)
        if (peak_iou(kept[k], b) > a.nms_iou) return false;
    return true;
}

// the outputs of map j: rows m*n_maps + j; rows after the kept ones repeat instance 0 with valid = 0
__host__ __device__ __forceinline__ void peak_write(const PeakArgs& a, int j, int m, const float* d, int idx, int valid, float* det_out,
                                                   long long* idx_out, int* valid_out) {
    const long long r = (long long)m * a.n_maps + j;
    for (int c = 0; c < 4; ++c) det_out[r * 4 + c] = d[c];
    idx_out[r] = idx;
    valid_out[r] = valid;
}

constexpr int kPeakThreads = 512;

// One CTA per map: the instance-0 argmax, then max_inst - 1 rounds of a block-wide argmax over the remaining candidates.
__global__ void __launch_bounds__(kPeakThreads) det_parse_peaks_kernel(const float* __restrict__ scores, const float* __restrict__ scales,
                                                                       const float* __restrict__ offsets, const PeakArgs a,
                                                                       float* __restrict__ det_out, long long* __restrict__ idx_out,
                                                                       int* __restrict__ valid_out, int* __restrict__ count_out) {
    const int j = blockIdx.x;
    const int n = a.hs * a.ws;
    const float* sc = scores + (long long)j * n;
    const float* scl = scales + (long long)j * n;
    const float* off = offsets + (long long)j * n * 2;
    __shared__ float sv[kPeakThreads / 32];
    __shared__ int si[kPeakThreads / 32];
    __shared__ PeakBox kept[G6D_DET_MAX_INSTANCES];
    __shared__ float first[4], last_v;
    __shared__ int first_i, last_i, n_kept, done;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    // block argmax of (bv, bi) under peak_beats; the result lands in sv[0], si[0]
    auto block_best = [&](float bv, int bi) {
        for (int o = 16; o > 0; o >>= 1) {
            const float v = __shfl_down_sync(0xffffffffu, bv, o);
            const int i = __shfl_down_sync(0xffffffffu, bi, o);
            if (peak_beats(v, i, bv, bi)) { bv = v; bi = i; }
        }
        if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            bv = lane < kPeakThreads / 32 ? sv[lane] : -INFINITY;
            bi = lane < kPeakThreads / 32 ? si[lane] : 0x7fffffff;
            for (int o = 16; o > 0; o >>= 1) {
                const float v = __shfl_down_sync(0xffffffffu, bv, o);
                const int i = __shfl_down_sync(0xffffffffu, bi, o);
                if (peak_beats(v, i, bv, bi)) { bv = v; bi = i; }
            }
            if (lane == 0) { sv[0] = bv; si[0] = bi; }
        }
        __syncthreads();
    };

    float bv = -INFINITY; int bi = 0x7fffffff;       // sentinel: loses to every real element (even -inf) on the index
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = sc[i];
        if (peak_beats(v, i, bv, bi)) { bv = v; bi = i; }
    }
    block_best(bv, bi);
    if (threadIdx.x == 0) {
        const int idx = min(max(si[0], 0), n - 1);
        det_peak_decode(sc, scl, off, idx, a.ws, a.pool, first);
        const int valid = first[3] >= a.min_score;
        peak_write(a, j, 0, first, idx, valid, det_out, idx_out, valid_out);
        kept[0] = peak_box(first[0], first[1], first[2], a.box_size);
        first_i = idx; last_v = first[3]; last_i = idx;
        n_kept = 1;
        done = !valid;                               // an invalid instance 0 ends the map: valid instances form a prefix
    }
    __syncthreads();
    for (int m = 1; m < a.max_inst; ++m) {
        if (!done) {
            const float lv = last_v; const int li = last_i, nk = n_kept;
            bv = -INFINITY; bi = 0x7fffffff;
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const float v = sc[i];
                if (peak_candidate(sc, scl, off, i, v, lv, li, bv, bi, kept, nk, a)) { bv = v; bi = i; }
            }
            block_best(bv, bi);
        }
        if (threadIdx.x == 0) {
            if (!done && si[0] != 0x7fffffff) {
                float d[4];
                det_peak_decode(sc, scl, off, si[0], a.ws, a.pool, d);
                peak_write(a, j, m, d, si[0], 1, det_out, idx_out, valid_out);
                kept[n_kept++] = peak_box(d[0], d[1], d[2], a.box_size);
                last_v = d[3]; last_i = si[0];
            } else {
                done = 1;
                peak_write(a, j, m, first, first_i, 0, det_out, idx_out, valid_out);
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) count_out[j] = first[3] >= a.min_score ? n_kept : 0;
}

// the kernel's selection for map j, serially on host memory
static void det_parse_peaks_map_host(const float* scores, const float* scales, const float* offsets, const PeakArgs& a, int j,
                                     float* det_out, long long* idx_out, int* valid_out, int* count_out) {
    const int n = a.hs * a.ws;
    const float* sc = scores + (long long)j * n;
    const float* scl = scales + (long long)j * n;
    const float* off = offsets + (long long)j * n * 2;
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int i = 0; i < n; ++i)
        if (peak_beats(sc[i], i, bv, bi)) { bv = sc[i]; bi = i; }
    float first[4];
    det_peak_decode(sc, scl, off, bi, a.ws, a.pool, first);
    const int valid0 = first[3] >= a.min_score;
    peak_write(a, j, 0, first, bi, valid0, det_out, idx_out, valid_out);
    PeakBox kept[G6D_DET_MAX_INSTANCES];
    kept[0] = peak_box(first[0], first[1], first[2], a.box_size);
    int n_kept = 1, last_i = bi;
    float last_v = first[3];
    bool done = !valid0;
    for (int m = 1; m < a.max_inst; ++m) {
        bv = -INFINITY; bi = 0x7fffffff;
        if (!done)
            for (int i = 0; i < n; ++i)
                if (peak_candidate(sc, scl, off, i, sc[i], last_v, last_i, bv, bi, kept, n_kept, a)) { bv = sc[i]; bi = i; }
        if (!done && bi != 0x7fffffff) {
            float d[4];
            det_peak_decode(sc, scl, off, bi, a.ws, a.pool, d);
            peak_write(a, j, m, d, bi, 1, det_out, idx_out, valid_out);
            kept[n_kept++] = peak_box(d[0], d[1], d[2], a.box_size);
            last_v = d[3]; last_i = bi;
        } else {
            done = true;
            peak_write(a, j, m, first, (int)idx_out[j], 0, det_out, idx_out, valid_out);
        }
    }
    count_out[j] = valid0 ? n_kept : 0;
}

static int det_parse_peaks_args(const char* name, const void* scores, const void* scales, const void* offsets, int n_maps, int hs, int ws,
                                int pool_ratio, int max_inst, int radius, float nms_iou, float box_size, float min_score,
                                const void* det_out, const void* idx_out, const void* valid_out, const void* count_out, PeakArgs* a) {
    G6D_REQUIRE(scores && scales && offsets && det_out && idx_out && valid_out && count_out, "%s: null pointer", name);
    G6D_REQUIRE(n_maps > 0 && hs > 0 && ws > 0 && (long long)hs * ws <= 0x7fffffffLL && pool_ratio > 0,
                "%s: bad map shape (n_maps=%d hs=%d ws=%d pool_ratio=%d)", name, n_maps, hs, ws, pool_ratio);
    G6D_REQUIRE(max_inst >= 1 && max_inst <= G6D_DET_MAX_INSTANCES, "%s: max_inst=%d outside [1, %d]", name, max_inst,
                G6D_DET_MAX_INSTANCES);
    G6D_REQUIRE(radius >= 0 && radius <= G6D_DET_MAX_PEAK_RADIUS, "%s: radius=%d outside [0, %d]", name, radius, G6D_DET_MAX_PEAK_RADIUS);
    G6D_REQUIRE(nms_iou >= 0.f && nms_iou <= 1.f, "%s: nms_iou=%g outside [0, 1]", name, (double)nms_iou);
    G6D_REQUIRE(box_size > 0.f && box_size <= 3.0e38f, "%s: box_size=%g must be positive and finite", name, (double)box_size);
    G6D_REQUIRE(min_score == min_score, "%s: min_score is NaN (use -inf for no threshold)", name);
    *a = PeakArgs{n_maps, hs, ws, pool_ratio, max_inst, radius, nms_iou, box_size, min_score};
    return G6D_OK;
}

// Second half of the row-decomposed sliding inner product (detector.py:222-224 F.conv2d(que, ref) with
// the reference features as k x k kernels):  out[y,x,r] = sum_ky partial[y + ky, x, ky*rfn + r], where
// partial = (1 x k convolution with k*rfn output channels (ky-major), zero padding k/2 in BOTH axes) holds,
// for every input row y' = y + ky - k/2, the contribution of kernel row ky.  The 1 x k form turns the
// N = rfn (32) GEMM of the direct formulation into an N = k*rfn (480) one: full-width tensor-core tiles.
__global__ void det_corr_rowsum_kernel(const float4* __restrict__ partial, float4* __restrict__ out, long long total,
                                       int H, int W, int k, int rfn4) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int r = (int)(i % rfn4);
    long long t = i / rfn4;
    const int x = (int)(t % W); t /= W;
    const int y = (int)(t % H);
    const long long q = t / H;
    const long long row_stride = (long long)W * k * rfn4;            // float4 per partial row y'
    const float4* p = partial + (q * (H + k - 1) + y) * row_stride + (long long)x * k * rfn4 + r;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int ky = 0; ky < k; ++ky) {
        const float4 v = __ldg(p + ky * row_stride + ky * rfn4);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    out[i] = acc;
}

// Several objects' correlations from ONE 1 x k convolution whose output channels are the objects' kernel rows
// concatenated: channel = (obj*k + ky)*rfn + r.  out is object-major [n_obj, qn, H, W, rfn]; each output element adds
// its k rows in det_corr_rowsum_kernel's order, so n_obj = 1 gives that kernel's bits.  k = 1 only regroups
// [qn, H, W, n_obj*rfn] into [n_obj, qn, H, W, rfn] (the direct, not row-decomposed, correlation).
__global__ void det_corr_rowsum_objects_kernel(const float4* __restrict__ partial, float4* __restrict__ out, long long total,
                                               int qn, int H, int W, int k, int rfn4, int n_obj) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int r = (int)(i % rfn4);
    long long t = i / rfn4;
    const int x = (int)(t % W); t /= W;
    const int y = (int)(t % H); t /= H;
    const long long q = t % qn;
    const int obj = (int)(t / qn);
    const long long pix_stride = (long long)n_obj * k * rfn4;         // float4 per partial pixel (all objects)
    const long long row_stride = (long long)W * pix_stride;           // float4 per partial row y'
    const float4* p = partial + (q * (H + k - 1) + y) * row_stride + (long long)x * pix_stride + (long long)obj * k * rfn4 + r;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int ky = 0; ky < k; ++ky) {
        const float4 v = __ldg(p + ky * row_stride + ky * rfn4);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    out[i] = acc;
}


// ------------------------------------------------------------------------------------------ detections from boxes
// A caller-supplied box (x0, y0, x1, y1, score) -> a detection record as g6d_det_parse_peaks writes one.  The box is
// usable when all five values are finite and it has positive width and height.  The record is the square on the box's
// longer side: (x0 + x1) * 0.5, (y0 + y1) * 0.5, max(w, h) * inv_box_size, score.  An add followed by a multiply has
// no fused form, so host and device round every operation the same way.
__host__ __device__ __forceinline__ bool box_usable(const float* b) {
    return isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]) && isfinite(b[4]) && b[2] > b[0] && b[3] > b[1];
}

__host__ __device__ __forceinline__ void box_record(const float* b, float inv_box_size, float* r) {
    const float w = b[2] - b[0], h = b[3] - b[1];
    r[0] = (b[0] + b[2]) * 0.5f;
    r[1] = (b[1] + b[3]) * 0.5f;
    r[2] = (w > h ? w : h) * inv_box_size;
    r[3] = b[4];
}

// box a (score sa, index ia) comes before box b: score descending, ties to the lower index
__host__ __device__ __forceinline__ bool box_before(float sa, int ia, float sb, int ib) {
    return sa > sb || (sa == sb && ia < ib);
}

struct BoxArgs { int n_maps, N, max_inst; float inv_box_size; };

__host__ __device__ __forceinline__ void box_write(const BoxArgs& a, int j, int m, const float* r, int valid, float* det_out,
                                                   int* valid_out) {
    const long long row = (long long)m * a.n_maps + j;
    for (int k = 0; k < 4; ++k) det_out[row * 4 + k] = r[k];
    valid_out[row] = valid;
}

// One block per map, one thread per box: a usable box's rank is the number of usable boxes before it; the boxes of rank
// < max_inst are the valid rows.  Rows past the count repeat row 0 (the empty-map record when no box is usable).
__global__ void __launch_bounds__(G6D_DET_MAX_BOXES) det_from_boxes_kernel(const float* __restrict__ boxes,
                                                                           const int* __restrict__ counts, const BoxArgs a,
                                                                           float* det_out, int* valid_out, int* count_out) {
    __shared__ float sc[G6D_DET_MAX_BOXES];
    __shared__ int use[G6D_DET_MAX_BOXES];
    __shared__ float row0[4];
    const int j = blockIdx.x, b = threadIdx.x;
    const int n = min(max(counts[j], 0), a.N);
    float box[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    bool u = false;
    if (b < n) {
        const float* p = boxes + ((long long)j * a.N + b) * 5;
        for (int k = 0; k < 5; ++k) box[k] = p[k];
        u = box_usable(box);
    }
    sc[b] = box[4];
    use[b] = u;
    if (b == 0) { row0[0] = 0.f; row0[1] = 0.f; row0[2] = 1.f; row0[3] = -INFINITY; }
    const int n_use = __syncthreads_count(u);
    const int count = min(n_use, a.max_inst);
    if (u) {
        int rank = 0;
        for (int i = 0; i < n; ++i) rank += use[i] && box_before(sc[i], i, box[4], b);
        if (rank < a.max_inst) {
            float r[4];
            box_record(box, a.inv_box_size, r);
            box_write(a, j, rank, r, 1, det_out, valid_out);
            if (rank == 0)
                for (int k = 0; k < 4; ++k) row0[k] = r[k];
        }
    }
    __syncthreads();
    if (b >= count && b < a.max_inst) box_write(a, j, b, row0, 0, det_out, valid_out);
    if (b == 0) count_out[j] = count;
}

// the kernel's records for map j, serially on host memory
static void det_from_boxes_map_host(const float* boxes, const int* counts, const BoxArgs& a, int j, float* det_out, int* valid_out,
                                    int* count_out) {
    const int n = counts[j] < 0 ? 0 : counts[j] > a.N ? a.N : counts[j];
    const float* bj = boxes + (long long)j * a.N * 5;
    float row0[4] = {0.f, 0.f, 1.f, -INFINITY};
    int count = 0;
    for (int b = 0; b < n; ++b) {
        if (!box_usable(bj + b * 5)) continue;
        int rank = 0;
        for (int i = 0; i < n; ++i) rank += box_usable(bj + i * 5) && box_before(bj[i * 5 + 4], i, bj[b * 5 + 4], b);
        if (rank >= a.max_inst) continue;
        float r[4];
        box_record(bj + b * 5, a.inv_box_size, r);
        box_write(a, j, rank, r, 1, det_out, valid_out);
        if (rank == 0)
            for (int k = 0; k < 4; ++k) row0[k] = r[k];
        ++count;
    }
    for (int m = count; m < a.max_inst; ++m) box_write(a, j, m, row0, 0, det_out, valid_out);
    count_out[j] = count;
}

static int det_from_boxes_args(const char* name, const void* boxes, const void* counts, int n_maps, int N, int max_inst,
                               float inv_box_size, const void* det_out, const void* valid_out, const void* count_out, BoxArgs* a) {
    G6D_REQUIRE(boxes && counts && det_out && valid_out && count_out, "%s: null pointer", name);
    G6D_REQUIRE(n_maps > 0, "%s: n_maps=%d must be positive", name, n_maps);
    G6D_REQUIRE(N >= 1 && N <= G6D_DET_MAX_BOXES, "%s: N=%d outside [1, %d]", name, N, G6D_DET_MAX_BOXES);
    G6D_REQUIRE(max_inst >= 1 && max_inst <= G6D_DET_MAX_INSTANCES, "%s: max_inst=%d outside [1, %d]", name, max_inst,
                G6D_DET_MAX_INSTANCES);
    G6D_REQUIRE(inv_box_size > 0.f && inv_box_size <= 3.0e38f, "%s: inv_box_size=%g must be positive and finite", name,
                (double)inv_box_size);
    *a = BoxArgs{n_maps, N, max_inst, inv_box_size};
    return G6D_OK;
}

}  // namespace g6d

using namespace g6d;

extern "C" int g6d_det_corr_rowsum(const float* partial, float* out, int qn, int H, int W, int k, int rfn,
                                   g6d_stream_t stream) {
    G6D_REQUIRE(partial && out && qn > 0 && H > 0 && W > 0 && k > 0 && rfn > 0 && (rfn & 3) == 0,
                "g6d_det_corr_rowsum: bad args (rfn must be a multiple of 4)");
    const long long total = (long long)qn * H * W * (rfn / 4);
    det_corr_rowsum_kernel<<<ceil_div(total, 256), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(partial), reinterpret_cast<float4*>(out), total, H, W, k, rfn / 4);
    G6D_CHECK_LAUNCH("g6d_det_corr_rowsum");
    return G6D_OK;
}

extern "C" int g6d_det_corr_rowsum_objects(const float* partial, float* out, int n_obj, int qn, int H, int W, int k, int rfn,
                                           g6d_stream_t stream) {
    G6D_REQUIRE(partial && out && n_obj > 0 && qn > 0 && H > 0 && W > 0 && k > 0 && rfn > 0 && (rfn & 3) == 0,
                "g6d_det_corr_rowsum_objects: bad args (n_obj, qn, H, W, k must be positive, rfn a positive multiple of 4)");
    const long long total = (long long)n_obj * qn * H * W * (rfn / 4);
    det_corr_rowsum_objects_kernel<<<ceil_div(total, 256), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4*>(partial), reinterpret_cast<float4*>(out), total, qn, H, W, k, rfn / 4, n_obj);
    G6D_CHECK_LAUNCH("g6d_det_corr_rowsum_objects");
    return G6D_OK;
}

extern "C" int g6d_det_score_fuse(const g6d_det_maps* host_maps, int qn, const float* w1, const float* b1,
                                  const float* w2, const float* b2, float* out, g6d_stream_t stream) {
    G6D_REQUIRE(host_maps && w1 && b1 && w2 && b2 && out && qn > 0, "g6d_det_score_fuse: bad args");
    const g6d_det_maps& M = *host_maps;
    G6D_REQUIRE(M.n_scales >= 1 && M.n_scales <= kDetFuseMaxScales, "g6d_det_score_fuse: n_scales=%d outside [1, %d]",
                M.n_scales, kDetFuseMaxScales);
    G6D_REQUIRE(M.rfn > 0 && M.hs > 0 && M.ws > 0, "g6d_det_score_fuse: bad map table (rfn=%d hs=%d ws=%d must be positive)",
                M.rfn, M.hs, M.ws);
    // the kernel reads level l at (y >> l, x >> l) for y < H[s][0], x < W[s][0]: exact sizes keep it in bounds
    for (int s = 0; s < M.n_scales; ++s) {
        G6D_REQUIRE(M.H[s][0] > 0 && M.W[s][0] > 0, "g6d_det_score_fuse: scale %d has level-0 size %dx%d", s, M.H[s][0],
                    M.W[s][0]);
        for (int l = 0; l < 3; ++l) {
            G6D_REQUIRE(M.map[s][l], "g6d_det_score_fuse: map[%d][%d] is null", s, l);
            G6D_REQUIRE(M.H[s][l] > 0 && M.W[s][l] > 0 && ((long long)M.H[s][l] << l) == M.H[s][0] &&
                            ((long long)M.W[s][l] << l) == M.W[s][0],
                        "g6d_det_score_fuse: scale %d level %d is %dx%d; it must be the level-0 size %dx%d divided by %d exactly",
                        s, l, M.H[s][l], M.W[s][l], M.H[s][0], M.W[s][0], 1 << l);
        }
    }
    DetFuseParams p;
    p.maps = *host_maps; p.w1 = w1; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.out = out; p.qn = qn;
    const long long npix = (long long)qn * host_maps->hs * host_maps->ws;
    const int grid = ceil_div(npix, 4);
    cudaStream_t st = as_stream(stream);
    switch (host_maps->n_scales) {
        case 1: det_score_fuse_kernel<3><<<grid, 128, 0, st>>>(p); break;
        case 2: det_score_fuse_kernel<6><<<grid, 128, 0, st>>>(p); break;
        case 3: det_score_fuse_kernel<9><<<grid, 128, 0, st>>>(p); break;
        case 4: det_score_fuse_kernel<12><<<grid, 128, 0, st>>>(p); break;
        case 5: det_score_fuse_kernel<15><<<grid, 128, 0, st>>>(p); break;
        case 6: det_score_fuse_kernel<18><<<grid, 128, 0, st>>>(p); break;
        default:
            set_error("g6d_det_score_fuse: %d scales not instantiated (max 6)", host_maps->n_scales);
            return G6D_EINVAL;
    }
    G6D_CHECK_LAUNCH("g6d_det_score_fuse");
    return G6D_OK;
}

extern "C" int g6d_det_parse(const float* scores, const float* scales, const float* offsets, int qn, int hs, int ws,
                             int pool_ratio, float* out, long long* out_idx, g6d_stream_t stream) {
    G6D_REQUIRE(scores && scales && offsets && out && out_idx && qn > 0 && hs > 0 && ws > 0, "g6d_det_parse: bad args");
    det_parse_kernel<<<qn, 256, 0, as_stream(stream)>>>(scores, scales, offsets, hs, ws, pool_ratio, out, out_idx);
    G6D_CHECK_LAUNCH("g6d_det_parse");
    return G6D_OK;
}

extern "C" int g6d_det_parse_peaks(const float* scores, const float* scales, const float* offsets, int n_maps, int hs, int ws,
                                   int pool_ratio, int max_inst, int radius, float nms_iou, float box_size, float min_score,
                                   float* det_out, long long* idx_out, int* valid_out, int* count_out, g6d_stream_t stream) {
    PeakArgs a;
    const int rc = det_parse_peaks_args("g6d_det_parse_peaks", scores, scales, offsets, n_maps, hs, ws, pool_ratio, max_inst, radius,
                                        nms_iou, box_size, min_score, det_out, idx_out, valid_out, count_out, &a);
    if (rc != G6D_OK) return rc;
    det_parse_peaks_kernel<<<n_maps, kPeakThreads, 0, as_stream(stream)>>>(scores, scales, offsets, a, det_out, idx_out, valid_out,
                                                                            count_out);
    G6D_CHECK_LAUNCH("g6d_det_parse_peaks");
    return G6D_OK;
}

extern "C" int g6d_det_parse_peaks_host(const float* scores, const float* scales, const float* offsets, int n_maps, int hs, int ws,
                                        int pool_ratio, int max_inst, int radius, float nms_iou, float box_size, float min_score,
                                        float* det_out, long long* idx_out, int* valid_out, int* count_out) {
    PeakArgs a;
    const int rc = det_parse_peaks_args("g6d_det_parse_peaks_host", scores, scales, offsets, n_maps, hs, ws, pool_ratio, max_inst, radius,
                                        nms_iou, box_size, min_score, det_out, idx_out, valid_out, count_out, &a);
    if (rc != G6D_OK) return rc;
    for (int j = 0; j < n_maps; ++j) det_parse_peaks_map_host(scores, scales, offsets, a, j, det_out, idx_out, valid_out, count_out);
    return G6D_OK;
}

extern "C" int g6d_det_from_boxes(const float* boxes, const int* counts, int n_maps, int N, int max_inst, float inv_box_size,
                                  float* det_out, int* valid_out, int* count_out, g6d_stream_t stream) {
    BoxArgs a;
    const int rc = det_from_boxes_args("g6d_det_from_boxes", boxes, counts, n_maps, N, max_inst, inv_box_size, det_out, valid_out,
                                       count_out, &a);
    if (rc != G6D_OK) return rc;
    const int threads = (max(N, max_inst) + 31) / 32 * 32;
    det_from_boxes_kernel<<<n_maps, threads, 0, as_stream(stream)>>>(boxes, counts, a, det_out, valid_out, count_out);
    G6D_CHECK_LAUNCH("g6d_det_from_boxes");
    return G6D_OK;
}

extern "C" int g6d_det_from_boxes_host(const float* boxes, const int* counts, int n_maps, int N, int max_inst, float inv_box_size,
                                       float* det_out, int* valid_out, int* count_out) {
    BoxArgs a;
    const int rc = det_from_boxes_args("g6d_det_from_boxes_host", boxes, counts, n_maps, N, max_inst, inv_box_size, det_out,
                                       valid_out, count_out, &a);
    if (rc != G6D_OK) return rc;
    for (int j = 0; j < n_maps; ++j) det_from_boxes_map_host(boxes, counts, a, j, det_out, valid_out, count_out);
    return G6D_OK;
}
