// Refiner-specific kernels: the unproject-and-aggregate volume fill (R2) and the pose heads.
#include "common.cuh"

namespace g6d {

constexpr int kMaxRefViews = 8;

struct VolParams {
    const float* ref_feats; const float* que_feats;
    const float* ref_Ks; const float* ref_poses; const float* que_Ks; const float* que_poses;
    float* mean_in; float* stdv;
    int Q, R, fh, fw, C, sn, img_h, img_w;
};

// ---- volume fill, v2 -------------------------------------------------------------------------
// A CTA (8 warps) owns a 2x4x8 brick of voxels so that the bilinear footprints of its voxels
// overlap in L1; a warp processes 4 consecutive voxels (along k) at a time:
//   phase A  lane = (view, voxel-in-quad): ONE projection + tap set per (voxel, view) pair,
//            28 of 32 lanes busy (6 refs + query), instead of every lane recomputing all views;
//   phase B  per voxel: the 4 taps of each view are broadcast with warp shuffles and every lane
//            gathers its 4 channels (128-bit, one 512 B feature row per tap per warp), then
//            mean / unbiased two-pass std / query sample are written as full 512 B rows with
//            streaming stores.
// Feature maps (3.7 MB / pose) are L2/L1 resident; algorithmic HBM traffic is the 50 MB of output.
// The floor of this formulation is the L1 gather: 28 taps x 512 B per voxel = 14 KB through the
// 128 B/clk L1 of each SM.
constexpr int kViewsMax = kMaxRefViews;   // views = R references + the query (view index R) <= 8

template <int RT>   // RT > 0: number of reference views known at compile time (6 on the estimator path); 0: runtime
__global__ void __launch_bounds__(256, 3) ref_volume_fill_kernel(const VolParams p) {
    __shared__ float sP[kViewsMax][12];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sn = p.sn;
    const int nbk = (sn + 7) / 8, nbj = (sn + 3) / 4, nbi = (sn + 1) / 2;
    const int bricks = nbi * nbj * nbk;
    const int qi = blockIdx.x / bricks;
    int b = blockIdx.x % bricks;
    const int bk = b % nbk; b /= nbk;
    const int bj = b % nbj;
    const int bi = b / nbj;
    const int R = RT > 0 ? RT : p.R;
    const int nviews = R + 1;

    // P_v = K_v @ [R|t]_v for the R references and the query of this pose (refiner.py:227,243)
    if (threadIdx.x < nviews * 12) {
        const int v = threadIdx.x / 12, e = threadIdx.x % 12, r = e / 4, c = e % 4;
        const float* K = v < R ? p.ref_Ks + ((long long)qi * R + v) * 9 : p.que_Ks + (long long)qi * 9;
        const float* T = v < R ? p.ref_poses + ((long long)qi * R + v) * 12 : p.que_poses + (long long)qi * 12;
        sP[v][e] = fmaf(K[r * 3 + 0], T[c], fmaf(K[r * 3 + 1], T[4 + c], K[r * 3 + 2] * T[8 + c]));
    }
    __syncthreads();

    const int my_view = lane >> 2, my_vox = lane & 3;
    const bool proj_lane = my_view < nviews;
    const float* P = sP[proj_lane ? my_view : 0];     // read from shared memory in phase A (keeps registers low)
    const float* qp = p.que_poses + (long long)qi * 12;
    const float r00 = qp[0], r01 = qp[1], r02 = qp[2], r10 = qp[4], r11 = qp[5], r12 = qp[6], r20 = qp[8], r21 = qp[9],
                r22 = qp[10];
    const float step = 2.f / (float)(sn - 1);
    auto lin = [&](int a) { return a < sn / 2 ? -1.f + step * (float)a : 1.f - step * (float)(sn - 1 - a); };
    const long long fsz = (long long)p.fh * p.fw * p.C;
    const float* ref_base = p.ref_feats + (long long)qi * R * fsz;
    const float* que_base = p.que_feats + (long long)qi * fsz;
    const long long nvox = (long long)sn * sn * sn;

    for (int qd = warp; qd < 16; qd += 8) {
        const int i = bi * 2 + (qd >> 3), j = bj * 4 + ((qd >> 1) & 3), k0 = bk * 8 + (qd & 1) * 4;
        if (i >= sn || j >= sn || k0 >= sn) continue;          // warp-uniform
        // ---- phase A: this lane's (voxel, view) projection and bilinear tap set
        int tidx[4]; float tw[4];
        {
            const int k = min(k0 + my_vox, sn - 1);
            const float ci = lin(i), cj = lin(j), ck = lin(k);
            // row vector @ R_in (refiner.py:216-220)
            const float vx = fmaf(ci, r00, fmaf(cj, r10, ck * r20));
            const float vy = fmaf(ci, r01, fmaf(cj, r11, ck * r21));
            const float vz = fmaf(ci, r02, fmaf(cj, r12, ck * r22));
            const float px = fmaf(vx, P[0], fmaf(vy, P[1], fmaf(vz, P[2], P[3])));
            const float py = fmaf(vx, P[4], fmaf(vy, P[5], fmaf(vz, P[6], P[7])));
            float pz = fmaf(vx, P[8], fmaf(vy, P[9], fmaf(vz, P[10], P[11])));
            if (pz < 1e-4f) pz = 1e-4f;                               // refiner.py:199-200
            const float u = px / pz, v = py / pz;
            const float gx = ((u + 0.5f) / (float)p.img_w - 0.5f) * 2.f;   // operator.py:4-17
            const float gy = ((v + 0.5f) / (float)p.img_h - 0.5f) * 2.f;
            const float ix = ((gx + 1.f) * (float)p.fw - 1.f) * 0.5f;      // grid_sample, align_corners=False
            const float iy = ((gy + 1.f) * (float)p.fh - 1.f) * 0.5f;
            const float fx0 = floorf(ix), fy0 = floorf(iy);
            const float lx = ix - fx0, ly = iy - fy0;
            const bool close_by = (fx0 > -2.f) && (fx0 < (float)p.fw + 1.f) && (fy0 > -2.f) && (fy0 < (float)p.fh + 1.f);
            const int x0 = close_by ? (int)fx0 : -10, y0 = close_by ? (int)fy0 : -10;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int xx = x0 + (t & 1), yy = y0 + (t >> 1);
                const bool inb = proj_lane && (unsigned)xx < (unsigned)p.fw && (unsigned)yy < (unsigned)p.fh;
                // out-of-bounds taps (zeros padding) keep a valid address and get weight 0, so the
                // gather below is branch-free and all loads of a view can be in flight together
                tidx[t] = inb ? (yy * p.fw + xx) * p.C : 0;
                tw[t] = inb ? ((t & 1) ? lx : 1.f - lx) * ((t >> 1) ? ly : 1.f - ly) : 0.f;
            }
        }
        // ---- phase B: gather + aggregate, one voxel at a time, all lanes on channels
        for (int vq = 0; vq < 4; ++vq) {
            const int k = k0 + vq;
            if (k >= sn) break;                                        // warp-uniform
            const long long orow = (long long)qi * nvox + ((long long)i * sn + j) * sn + k;
            // every lane runs ceil(C/128) trips so the full-warp shuffles below see all 32 lanes;
            // when C % 128 != 0 the lanes past the last channel skip their loads and stores
            for (int c0 = 0; c0 < p.C; c0 += 128) {
                const int c = c0 + lane * 4;
                const bool on = c < p.C;
                float4 s[kViewsMax];
                float4 mean = make_float4(0.f, 0.f, 0.f, 0.f), qs = mean;
#pragma unroll
                for (int v = 0; v < kViewsMax; ++v) {
                    if (v < nviews) {
                        // 32-bit element offsets from one base per tensor; the tap offset arrives by shuffle
                        const float* fmap = v < R ? ref_base + v * (int)fsz + c : que_base + c;
                        float4 f[4]; float w[4];
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const int idx = __shfl_sync(0xffffffffu, tidx[t], v * 4 + vq);
                            w[t] = __shfl_sync(0xffffffffu, tw[t], v * 4 + vq);
                            f[t] = on ? __ldg(reinterpret_cast<const float4*>(fmap + idx)) : make_float4(0.f, 0.f, 0.f, 0.f);
                        }
                        float4 acc;
                        acc.x = f[0].x * w[0]; acc.y = f[0].y * w[0]; acc.z = f[0].z * w[0]; acc.w = f[0].w * w[0];
#pragma unroll
                        for (int t = 1; t < 4; ++t) {
                            acc.x = fmaf(f[t].x, w[t], acc.x); acc.y = fmaf(f[t].y, w[t], acc.y);
                            acc.z = fmaf(f[t].z, w[t], acc.z); acc.w = fmaf(f[t].w, w[t], acc.w);
                        }
                        if (v < R) {
                            s[v] = acc;
                            mean.x += acc.x; mean.y += acc.y; mean.z += acc.z; mean.w += acc.w;
                        } else {
                            qs = acc;
                        }
                    }
                }
                const float inv_r = 1.f / (float)R;            // mean = sum * (1/R): within 1 ulp of sum / R
                mean.x *= inv_r; mean.y *= inv_r; mean.z *= inv_r; mean.w *= inv_r;
                float4 var = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int v = 0; v < kViewsMax; ++v) {
                    if (v < R) {
                        float d;
                        d = s[v].x - mean.x; var.x = fmaf(d, d, var.x);
                        d = s[v].y - mean.y; var.y = fmaf(d, d, var.y);
                        d = s[v].z - mean.z; var.z = fmaf(d, d, var.z);
                        d = s[v].w - mean.w; var.w = fmaf(d, d, var.w);
                    }
                }
                const float inv_u = 1.f / (float)(R - 1);      // unbiased (torch.std default, refiner.py:237)
                float4 sd;
                sd.x = sqrtf(var.x * inv_u); sd.y = sqrtf(var.y * inv_u); sd.z = sqrtf(var.z * inv_u); sd.w = sqrtf(var.w * inv_u);
                if (!on) continue;
                float* mrow = p.mean_in + orow * (2 * p.C);
                __stcs(reinterpret_cast<float4*>(mrow + c), mean);
                __stcs(reinterpret_cast<float4*>(mrow + p.C + c), qs);
                __stcs(reinterpret_cast<float4*>(p.stdv + orow * p.C + c), sd);
            }
        }
    }
}

// ---- volume fill, v3 (C = 128, the refiner's feature width) -----------------------------------
// Same arithmetic as v2, restructured around what ncu showed v2 to be bound by (issue slots: 964
// warp-instructions per voxel, of which 112 SHFL + 112 WARPSYNC/ENDCOLLECTIVE from shuffles under a
// divergent-looking channel loop, ~430 integer address instructions):
//   phase A  thread = one (voxel, view) pair of the CTA's 64-voxel brick: projection + bilinear tap set,
//            written ONCE to shared memory as (4 element offsets, 4 weights) -- 16 KB per CTA;
//   phase B  warp = 8 voxels of the brick, lane = 4 channels: per view two broadcast LDS.128 bring the
//            taps, 4 x (IMAD.WIDE + LDG.128 + 4 FFMA) gather and blend them; mean / unbiased two-pass
//            std / query sample leave as three 512-byte streaming row stores.
// ~300 instructions per voxel; the remaining bound is the L1 gather itself (28 taps x 512 B per voxel
// through the 128 B/clk data pipe = 13 us per pose), above the 8.2 us of the 54 MB algorithmic HBM
// traffic -- see DESIGN.md.
constexpr int kBrickVox = 64;
// base + idx (elements) in ONE integer instruction (IMAD.WIDE) instead of the LEA / LEA.HI.X pair
__device__ __forceinline__ float4 ldg_at(const float* base, int idx) {
    unsigned long long a;
    asm("mad.wide.s32 %0, %1, 4, %2;" : "=l"(a) : "r"(idx), "l"(base));
    return __ldg(reinterpret_cast<const float4*>(a));
}
template <int RT>
__global__ void __launch_bounds__(256, 2) ref_volume_fill_c128_kernel(const VolParams p) {
    constexpr int C = 128;
    constexpr int NV = RT + 1;                    // views: RT references + the query
    __shared__ float sP[NV][12];
    __shared__ int4 s_idx[kBrickVox][NV];
    __shared__ float4 s_w[kBrickVox][NV];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sn = p.sn;
    const int nbk = (sn + 7) / 8, nbj = (sn + 3) / 4, nbi = (sn + 1) / 2;
    const int bricks = nbi * nbj * nbk;
    const int qi = blockIdx.x / bricks;
    int b = blockIdx.x % bricks;
    const int bk = b % nbk; b /= nbk;
    const int bj = b % nbj;
    const int bi = b / nbj;

    if (threadIdx.x < NV * 12) {                  // P_v = K_v @ [R|t]_v (refiner.py:227,243)
        const int v = threadIdx.x / 12, e = threadIdx.x % 12, r = e / 4, c = e % 4;
        const float* K = v < RT ? p.ref_Ks + ((long long)qi * RT + v) * 9 : p.que_Ks + (long long)qi * 9;
        const float* T = v < RT ? p.ref_poses + ((long long)qi * RT + v) * 12 : p.que_poses + (long long)qi * 12;
        sP[v][e] = fmaf(K[r * 3 + 0], T[c], fmaf(K[r * 3 + 1], T[4 + c], K[r * 3 + 2] * T[8 + c]));
    }
    __syncthreads();

    // ---- phase A: one (voxel, view) pair per thread; brick voxel n = (di, dj, dk) = (n >> 5, (n >> 3) & 3, n & 7)
    {
        const float* qp = p.que_poses + (long long)qi * 12;
        const float r00 = qp[0], r01 = qp[1], r02 = qp[2], r10 = qp[4], r11 = qp[5], r12 = qp[6], r20 = qp[8], r21 = qp[9],
                    r22 = qp[10];
        const float step = 2.f / (float)(sn - 1);
        auto lin = [&](int a) { return a < sn / 2 ? -1.f + step * (float)a : 1.f - step * (float)(sn - 1 - a); };   // torch.linspace
        for (int e = threadIdx.x; e < kBrickVox * NV; e += 256) {
            const int n = e / NV, v = e - n * NV;
            const int i = min(bi * 2 + (n >> 5), sn - 1), j = min(bj * 4 + ((n >> 3) & 3), sn - 1), k = min(bk * 8 + (n & 7), sn - 1);
            const float* P = sP[v];
            const float ci = lin(i), cj = lin(j), ck = lin(k);
            const float vx = fmaf(ci, r00, fmaf(cj, r10, ck * r20));          // row vector @ R_in (refiner.py:216-220)
            const float vy = fmaf(ci, r01, fmaf(cj, r11, ck * r21));
            const float vz = fmaf(ci, r02, fmaf(cj, r12, ck * r22));
            const float px = fmaf(vx, P[0], fmaf(vy, P[1], fmaf(vz, P[2], P[3])));
            const float py = fmaf(vx, P[4], fmaf(vy, P[5], fmaf(vz, P[6], P[7])));
            float pz = fmaf(vx, P[8], fmaf(vy, P[9], fmaf(vz, P[10], P[11])));
            if (pz < 1e-4f) pz = 1e-4f;                                       // refiner.py:199-200
            const float u = px / pz, vv = py / pz;
            const float gx = ((u + 0.5f) / (float)p.img_w - 0.5f) * 2.f;      // operator.py:4-17
            const float gy = ((vv + 0.5f) / (float)p.img_h - 0.5f) * 2.f;
            const float ix = ((gx + 1.f) * (float)p.fw - 1.f) * 0.5f;         // grid_sample, align_corners=False
            const float iy = ((gy + 1.f) * (float)p.fh - 1.f) * 0.5f;
            const float fx0 = floorf(ix), fy0 = floorf(iy);
            const float lx = ix - fx0, ly = iy - fy0;
            const bool close_by = (fx0 > -2.f) && (fx0 < (float)p.fw + 1.f) && (fy0 > -2.f) && (fy0 < (float)p.fh + 1.f);
            const int x0 = close_by ? (int)fx0 : -10, y0 = close_by ? (int)fy0 : -10;
            int ti[4]; float tw[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int xx = x0 + (t & 1), yy = y0 + (t >> 1);
                const bool inb = (unsigned)xx < (unsigned)p.fw && (unsigned)yy < (unsigned)p.fh;
                // out-of-bounds taps (zeros padding) keep a valid address and get weight 0: branch-free gather
                ti[t] = inb ? (yy * p.fw + xx) * C : 0;
                tw[t] = inb ? ((t & 1) ? lx : 1.f - lx) * ((t >> 1) ? ly : 1.f - ly) : 0.f;
            }
            s_idx[n][v] = make_int4(ti[0], ti[1], ti[2], ti[3]);
            s_w[n][v] = make_float4(tw[0], tw[1], tw[2], tw[3]);
        }
    }
    __syncthreads();

    // ---- phase B: warp = 8 voxels (one k-run), lane = channels [4 lane, 4 lane + 4)
    const long long fsz = (long long)p.fh * p.fw * C;
    const float* vbase[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v)
        vbase[v] = (v < RT ? p.ref_feats + ((long long)qi * RT + v) * fsz : p.que_feats + (long long)qi * fsz) + lane * 4;
    const long long nvox = (long long)sn * sn * sn;
    const int i = bi * 2 + (warp >> 2), j = bj * 4 + (warp & 3);
    if (i >= sn || j >= sn) return;                                           // warp-uniform
    constexpr float inv_r = 1.f / (float)RT;                                  // mean = sum * (1/R): within 1 ulp of sum / R
    constexpr float inv_u = 1.f / (float)(RT - 1);                            // unbiased (torch.std default, refiner.py:237)
#pragma unroll 2
    for (int dk = 0; dk < 8; ++dk) {
        const int k = bk * 8 + dk;
        if (k >= sn) break;                                                   // warp-uniform
        const int n = warp * 8 + dk;
        float4 s[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
            const int4 ti = s_idx[n][v];
            const float4 tw = s_w[n][v];
            const float4 f0 = ldg_at(vbase[v], ti.x), f1 = ldg_at(vbase[v], ti.y), f2 = ldg_at(vbase[v], ti.z), f3 = ldg_at(vbase[v], ti.w);
            float4 a;
            a.x = f0.x * tw.x; a.y = f0.y * tw.x; a.z = f0.z * tw.x; a.w = f0.w * tw.x;
            a.x = fmaf(f1.x, tw.y, a.x); a.y = fmaf(f1.y, tw.y, a.y); a.z = fmaf(f1.z, tw.y, a.z); a.w = fmaf(f1.w, tw.y, a.w);
            a.x = fmaf(f2.x, tw.z, a.x); a.y = fmaf(f2.y, tw.z, a.y); a.z = fmaf(f2.z, tw.z, a.z); a.w = fmaf(f2.w, tw.z, a.w);
            a.x = fmaf(f3.x, tw.w, a.x); a.y = fmaf(f3.y, tw.w, a.y); a.z = fmaf(f3.z, tw.w, a.z); a.w = fmaf(f3.w, tw.w, a.w);
            s[v] = a;
        }
        float4 mean = s[0];
#pragma unroll
        for (int v = 1; v < RT; ++v) { mean.x += s[v].x; mean.y += s[v].y; mean.z += s[v].z; mean.w += s[v].w; }
        mean.x *= inv_r; mean.y *= inv_r; mean.z *= inv_r; mean.w *= inv_r;
        float4 var = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int v = 0; v < RT; ++v) {
            float d;
            d = s[v].x - mean.x; var.x = fmaf(d, d, var.x);
            d = s[v].y - mean.y; var.y = fmaf(d, d, var.y);
            d = s[v].z - mean.z; var.z = fmaf(d, d, var.z);
            d = s[v].w - mean.w; var.w = fmaf(d, d, var.w);
        }
        float4 sd;
        sd.x = sqrtf(var.x * inv_u); sd.y = sqrtf(var.y * inv_u); sd.z = sqrtf(var.z * inv_u); sd.w = sqrtf(var.w * inv_u);
        const long long orow = (long long)qi * nvox + ((long long)i * sn + j) * sn + k;
        float* mrow = p.mean_in + orow * (2 * C) + lane * 4;
        __stcs(reinterpret_cast<float4*>(mrow), mean);
        __stcs(reinterpret_cast<float4*>(mrow + C), s[RT]);
        __stcs(reinterpret_cast<float4*>(p.stdv + orow * C + lane * 4), sd);
    }
}

// x [M,K] -> out [M,7]: quaternion (normalised, F.normalize eps 1e-12), 2-D offset, log2 scale
__global__ void ref_pose_heads_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                      const float* __restrict__ b, float* __restrict__ out, int K) {
    const int m = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __shared__ float res[7];
    if (warp < 7) {
        float acc = 0.f;
        for (int k = lane; k < K; k += 32) acc = fmaf(x[(long long)m * K + k], w[(long long)warp * K + k], acc);
        acc = warp_sum(acc);
        if (lane == 0) res[warp] = acc + b[warp];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float n = fmaxf(sqrtf(res[0] * res[0] + res[1] * res[1] + res[2] * res[2] + res[3] * res[3]), 1e-12f);
        for (int i = 0; i < 4; ++i) out[m * 7 + i] = res[i] / n;
        for (int i = 4; i < 7; ++i) out[m * 7 + i] = res[i];
    }
}

}  // namespace g6d

using namespace g6d;

extern "C" int g6d_ref_volume_fill(const float* ref_feats, const float* que_feats, const float* ref_Ks,
                                   const float* ref_poses, const float* que_Ks, const float* que_poses, int Q, int R,
                                   int fh, int fw, int C, int sn, int img_h, int img_w, float* mean_in, float* stdv,
                                   g6d_stream_t stream) {
    G6D_REQUIRE(ref_feats && que_feats && ref_Ks && ref_poses && que_Ks && que_poses && mean_in && stdv,
                "g6d_ref_volume_fill: null pointer");
    // at most 7 references: they and the query fill the 8 projection lanes x 4 voxels of a warp
    G6D_REQUIRE(Q > 0 && R >= 2 && R <= kMaxRefViews - 1 && fh > 0 && fw > 0 && C > 0 && (C & 3) == 0 && sn >= 2 &&
                    img_h > 0 && img_w > 0,
                "g6d_ref_volume_fill: bad dims (Q=%d R=%d fh=%d fw=%d C=%d sn=%d img %dx%d; need 2 <= R <= %d, C > 0, "
                "C%%4 == 0, sn >= 2)", Q, R, fh, fw, C, sn, img_h, img_w, kMaxRefViews - 1);
    VolParams p{ref_feats, que_feats, ref_Ks, ref_poses, que_Ks, que_poses, mean_in, stdv,
                Q, R, fh, fw, C, sn, img_h, img_w};
    const long long bricks = (long long)((sn + 1) / 2) * ((sn + 3) / 4) * ((sn + 7) / 8);
    if (R == 6 && C == 128) ref_volume_fill_c128_kernel<6><<<(unsigned)(Q * bricks), 256, 0, as_stream(stream)>>>(p);
    else if (R == 6) ref_volume_fill_kernel<6><<<(unsigned)(Q * bricks), 256, 0, as_stream(stream)>>>(p);
    else ref_volume_fill_kernel<0><<<(unsigned)(Q * bricks), 256, 0, as_stream(stream)>>>(p);
    G6D_CHECK_LAUNCH("g6d_ref_volume_fill");
    return G6D_OK;
}

extern "C" int g6d_ref_pose_heads(const float* x, const float* w, const float* b, float* out, int M, int K,
                                  g6d_stream_t stream) {
    G6D_REQUIRE(x && w && b && out && M > 0 && K > 0, "g6d_ref_pose_heads: bad args");
    ref_pose_heads_kernel<<<M, 256, 0, as_stream(stream)>>>(x, w, b, out, K);
    G6D_CHECK_LAUNCH("g6d_ref_pose_heads");
    return G6D_OK;
}
