// predict.py's drawn frames (DESIGN.md row f16) as __host__ __device__ code: utils/draw_utils.py draw_bbox_3d, i.e.
// draw_keypoints' 8 red corner dots (cv2.circle, radius 2, filled) and 12 box edges (cv2.line, thickness 2), at the
// corners np.round(project_points(bbox, pose, K)).astype(np.int32), then cv2.cvtColor(COLOR_RGB2YUV_I420) for NV12
// destinations.  Restated from OpenCV's 8-bit drawing code (imgproc/drawing.cpp) for LINE_8 and shift 0:
//   - a filled circle is Circle(): the integer midpoint walk, each step filling rows cy +- dy and cy +- dx;
//   - a thick line is ThickLine(): a 4-point FillConvexPoly at XY_SHIFT = 16 around the segment (its outline drawn by
//     Line2, its interior by the scanline walk with int64 edges) and a radius-1 Circle() fill at each end.
// Every walk is integer, so the pixels a primitive puts on one row are computed directly for that row: the kernel
// (draw.cu) evaluates each output row on its own, the host twin runs the same functions row by row.
// This translation unit is compiled with -fmad=false: the float32 projection rounds as numpy's does.
#pragma once
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include "track_math.cuh"

namespace g6d {
namespace draw {

constexpr int kShift = 16;
constexpr long long kOne = 1LL << kShift;
constexpr int kLines = 12;
constexpr int kPrims = track::kCorners + kLines;   // per box: the 8 corner dots, then the 12 edges
constexpr int kSpansPerPrim = 11;                  // a thick line: fill + 4 outline runs and end points + 2 end dots
// the reference's edge order (draw_bbox_3d)
G6D_HD int edge_end(int e, int which) {
    const int a[kLines] = {0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3};
    const int b[kLines] = {1, 2, 3, 0, 5, 6, 7, 4, 4, 5, 6, 7};
    return which ? b[e] : a[e];
}

struct Span {
    int lo, hi;     // inclusive pixel columns on one row, empty when lo > hi
};

// x86 cvttsd2si: a value outside int32 (or NaN) converts to INT_MIN, the "integer indefinite"
G6D_HD int trunc_i32(double v) {
    return (v >= -2147483648.0 && v < 2147483648.0) ? (int)v : INT_MIN;
}
// np.round(v).astype(np.int32): round half to even, then the x86 conversion
G6D_HD int round_i32(double v) { return trunc_i32(rint(v)); }
// cvRound(double): the SSE2 conversion under round-to-nearest-even, INT_MIN outside int32
G6D_HD int cv_round(double v) { return round_i32(v); }
// OpenCV's int arithmetic on corners near INT_MIN / INT_MAX wraps
G6D_HD int wsub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }
G6D_HD int wadd(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
G6D_HD long long wmul(long long a, long long b) { return (long long)((unsigned long long)a * (unsigned long long)b); }
G6D_HD long long floor_div(long long a, long long b) {   // b > 0
    long long q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

// ------------------------------------------------------------------------------------------ corners
// project_points(bbox, pose, K) then np.round(...).astype(np.int32).  in_f32: the float32 pose of the refiner, projected
// in float32 exactly as the smoothing's history holds it (track::project_box); else the float64 smoothed pose with the
// float32 bbox and K values in float64, the pts__ of predict.py.
G6D_HD void box_corners(const float* bbox, const double* pose, int in_f32, const double* K, int* pts) {
    if (in_f32) {
        float p[16];
        track::project_box(bbox, pose, 1, K, p);
        for (int e = 0; e < 16; ++e) pts[e] = round_i32((double)p[e]);
        return;
    }
    for (int c = 0; c < track::kCorners; ++c) {
        const float* X = bbox + c * 3;
        double p[3], q[3];
        for (int i = 0; i < 3; ++i)
            p[i] = (((double)X[0] * pose[i * 4] + (double)X[1] * pose[i * 4 + 1]) + (double)X[2] * pose[i * 4 + 2]) + pose[i * 4 + 3];
        for (int j = 0; j < 3; ++j) q[j] = (p[0] * K[j * 3] + p[1] * K[j * 3 + 1]) + p[2] * K[j * 3 + 2];
        double d = q[2];
        if (fabs(d) < 1e-4 && fabs(d) > 0.) d = 1e-4;
        pts[c * 2] = round_i32(q[0] / d);
        pts[c * 2 + 1] = round_i32(q[1] / d);
    }
}

// ------------------------------------------------------------------------------------------ Circle() fill
// The pixels of row y covered by the filled circle: the union of the walk's spans on that row (every span holds cx, so
// the union is one span), clipped as OpenCV clips them.
G6D_HD Span circle_row(int cx, int cy, int radius, int y, int width, int height) {
    Span s{1, 0};
    int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
    const bool inside = cx >= radius && cx < width - radius && cy >= radius && cy < height - radius;
    auto put = [&](int row, int a, int b) {
        if (row != y) return;
        if (s.lo > s.hi) {
            s.lo = a;
            s.hi = b;
        } else {
            s.lo = a < s.lo ? a : s.lo;
            s.hi = b > s.hi ? b : s.hi;
        }
    };
    while (dx >= dy) {
        const int y11 = wsub(cy, dy), y12 = wadd(cy, dy), y21 = wsub(cy, dx), y22 = wadd(cy, dx);
        int x11 = wsub(cx, dx), x12 = wadd(cx, dx), x21 = wsub(cx, dy), x22 = wadd(cx, dy);
        if (inside) {
            put(y11, x11, x12);
            put(y12, x11, x12);
            put(y21, x21, x22);
            put(y22, x21, x22);
        } else if (x11 < width && x12 >= 0 && y21 < height && y22 >= 0) {
            x11 = x11 > 0 ? x11 : 0;
            x12 = x12 < width - 1 ? x12 : width - 1;
            if ((unsigned)y11 < (unsigned)height) put(y11, x11, x12);
            if ((unsigned)y12 < (unsigned)height) put(y12, x11, x12);
            if (x21 < width && x22 >= 0) {
                x21 = x21 > 0 ? x21 : 0;
                x22 = x22 < width - 1 ? x22 : width - 1;
                if ((unsigned)y21 < (unsigned)height) put(y21, x21, x22);
                if ((unsigned)y22 < (unsigned)height) put(y22, x21, x22);
            }
        }
        dy++;
        err += plus;
        plus += 2;
        const int mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
    return s;
}

// ------------------------------------------------------------------------------------------ Line2 (polygon outline)
// clipLine on the XY_SHIFT-scaled frame, then the fixed-point DDA.  Prepared once per segment; line2_row gives a row's
// run of the DDA and the end point Line2 puts first.
struct Line2 {
    int ok;                    // not clipped away
    int xmajor;
    long long p1x, p1y;        // DDA start (p1 after the swap, + XY_ONE/2; the major coordinate already shifted down)
    long long step;            // minor-axis step
    int ecount;
    int ex, ey;                // the end point
};

G6D_HD bool clip_line(long long width, long long height, long long& x1, long long& y1, long long& x2, long long& y2) {
    const long long right = width - 1, bottom = height - 1;
    if (width <= 0 || height <= 0) return false;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (long long)((double)(a - y1) * (double)(x2 - x1) / (double)(y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (long long)((double)(a - y2) * (double)(x2 - x1) / (double)(y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (long long)((double)(a - x1) * (double)(y2 - y1) / (double)(x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (long long)((double)(a - x2) * (double)(y2 - y1) / (double)(x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

G6D_HD Line2 line2_setup(long long x1, long long y1, long long x2, long long y2, int width, int height) {
    Line2 L{};
    L.ok = clip_line((long long)width << kShift, (long long)height << kShift, x1, y1, x2, y2);
    if (!L.ok) return L;
    long long dx = x2 - x1, dy = y2 - y1;
    const long long j = dx < 0 ? -1 : 0, ax = (dx ^ j) - j;
    const long long i = dy < 0 ? -1 : 0, ay = (dy ^ i) - i;
    if (ax > ay) {
        dy = (dy ^ j) - j;
        x1 ^= x2 & j; x2 ^= x1 & j; x1 ^= x2 & j;
        y1 ^= y2 & j; y2 ^= y1 & j; y1 ^= y2 & j;
        L.xmajor = 1;
        L.step = (long long)((unsigned long long)dy << kShift) / (ax | 1);
        L.ecount = (int)((x2 - x1) >> kShift);
    } else {
        dx = (dx ^ i) - i;
        x1 ^= x2 & i; x2 ^= x1 & i; x1 ^= x2 & i;
        y1 ^= y2 & i; y2 ^= y1 & i; y1 ^= y2 & i;
        L.xmajor = 0;
        L.step = (long long)((unsigned long long)dx << kShift) / (ay | 1);
        L.ecount = (int)((y2 - y1) >> kShift);
    }
    x1 += kOne >> 1;
    y1 += kOne >> 1;
    L.ex = (int)((x2 + (kOne >> 1)) >> kShift);
    L.ey = (int)((y2 + (kOne >> 1)) >> kShift);
    if (L.xmajor) x1 >>= kShift; else y1 >>= kShift;
    L.p1x = x1;
    L.p1y = y1;
    return L;
}

// row y of the DDA (one run) and of the end point, each clipped to the frame as ICV_PUT_POINT clips
G6D_HD void line2_row(const Line2& L, int y, int width, int height, Span* run, Span* end) {
    run->lo = 1; run->hi = 0;
    end->lo = 1; end->hi = 0;
    if (!L.ok || y < 0 || y >= height) return;
    if (L.ey == y && L.ex >= 0 && L.ex < width) end->lo = end->hi = L.ex;
    long long k0, k1;
    if (L.xmajor) {       // pixel k at (p1x + k, (p1y + k*step) >> 16)
        const long long lo = (long long)y << kShift, hi = lo + kOne - 1;
        if (L.step == 0) {
            if ((L.p1y >> kShift) != y) return;
            k0 = 0; k1 = L.ecount;
        } else if (L.step > 0) {
            k0 = -floor_div(-(lo - L.p1y), L.step);
            k1 = floor_div(hi - L.p1y, L.step);
        } else {
            k0 = -floor_div(-(L.p1y - hi), -L.step);
            k1 = floor_div(L.p1y - lo, -L.step);
        }
        k0 = k0 > 0 ? k0 : 0;
        k1 = k1 < L.ecount ? k1 : L.ecount;
        if (k0 > k1) return;
        long long a = L.p1x + k0, b = L.p1x + k1;
        a = a > 0 ? a : 0;
        b = b < width - 1 ? b : width - 1;
        if (a <= b) { run->lo = (int)a; run->hi = (int)b; }
    } else {              // pixel k at ((p1x + k*step) >> 16, p1y + k)
        const long long k = (long long)y - L.p1y;
        if (k < 0 || k > L.ecount) return;
        const int x = (int)((L.p1x + k * L.step) >> kShift);
        if (x >= 0 && x < width) run->lo = run->hi = x;
    }
}

// ------------------------------------------------------------------------------------------ FillConvexPoly scanline
// The scanline walk of a 4-point polygon at XY_SHIFT, as bands of rows over which both edges advance by a fixed dx: the
// walk's state only changes at an edge's end row, so a row's span is the band's start x + (row - band start) * dx.
constexpr int kMaxBands = 8;
struct Poly {
    long long v[8];                 // 4 points (x, y), XY_SHIFT fixed point
    Line2 outline[4];               // Line2(v[3], v[0]), Line2(v[0], v[1]), ...
    int nb;                         // bands
    int y0[kMaxBands], y1[kMaxBands];   // rows [y0, y1)
    long long xa[kMaxBands], dxa[kMaxBands], xb[kMaxBands], dxb[kMaxBands];
};

G6D_HD void poly_setup(const long long* v, int width, int height, Poly& P) {
    constexpr int npts = 4;
    const long long delta = kOne >> 1;
    for (int i = 0; i < 2 * npts; ++i) P.v[i] = v[i];
    P.nb = 0;
    long long xmin = v[0], xmax = v[0], ymin = v[1], ymax = v[1];
    int imin = 0;
    for (int i = 0; i < npts; ++i) {
        const long long px = v[2 * i], py = v[2 * i + 1];
        if (py < ymin) { ymin = py; imin = i; }
        ymax = py > ymax ? py : ymax;
        xmax = px > xmax ? px : xmax;
        xmin = px < xmin ? px : xmin;
        const int p = (i + npts - 1) % npts;
        P.outline[i] = line2_setup(v[2 * p], v[2 * p + 1], px, py, width, height);
    }
    xmin = (xmin + delta) >> kShift;
    xmax = (xmax + delta) >> kShift;
    ymin = (ymin + delta) >> kShift;
    ymax = (ymax + delta) >> kShift;
    if ((int)xmax < 0 || (int)ymax < 0 || (int)xmin >= width || (int)ymin >= height) return;
    ymax = ymax < height - 1 ? ymax : height - 1;
    struct { int idx, di; long long x, dx; int ye; } edge[2];
    int edges = npts;
    edge[0].idx = edge[1].idx = imin;
    int y = (int)ymin;
    edge[0].ye = edge[1].ye = y;
    edge[0].di = 1;
    edge[1].di = npts - 1;
    edge[0].x = edge[1].x = -kOne;
    edge[0].dx = edge[1].dx = 0;
    for (;;) {
        for (int i = 0; i < 2; ++i) {
            if (y >= edge[i].ye) {
                int idx0 = edge[i].idx, di = edge[i].di;
                int idx = idx0 + di;
                if (idx >= npts) idx -= npts;
                for (; edges-- > 0;) {
                    const int ty = (int)((v[2 * idx + 1] + delta) >> kShift);
                    if (ty > y) {
                        const long long xs = v[2 * idx0], xe = v[2 * idx];
                        edge[i].ye = ty;
                        edge[i].dx = ((xe - xs) * 2 + ((long long)ty - y)) / (2 * ((long long)ty - y));
                        edge[i].x = xs;
                        edge[i].idx = idx;
                        break;
                    }
                    idx0 = idx;
                    idx += di;
                    if (idx >= npts) idx -= npts;
                }
            }
        }
        if (edges < 0) break;
        // rows y .. end-1 run with these edges: the next refresh is at the smaller end row (the next row when an edge
        // ran out, which then stops the walk)
        long long next = edge[0].ye < edge[1].ye ? edge[0].ye : edge[1].ye;
        next = next > (long long)y + 1 ? next : (long long)y + 1;
        const long long end = next < ymax + 1 ? next : ymax + 1;
        if (P.nb < kMaxBands) {
            const int b = P.nb++;
            P.y0[b] = y;
            P.y1[b] = (int)end;
            P.xa[b] = edge[0].x; P.dxa[b] = edge[0].dx;
            P.xb[b] = edge[1].x; P.dxb[b] = edge[1].dx;
        }
        edge[0].x += wmul(edge[0].dx, end - y);
        edge[1].x += wmul(edge[1].dx, end - y);
        if (end > ymax) break;
        y = (int)end;
    }
}

G6D_HD Span poly_row(const Poly& P, int y, int width) {
    Span s{1, 0};
    if (y < 0) return s;
    for (int b = 0; b < P.nb; ++b) {
        if (y < P.y0[b] || y >= P.y1[b]) continue;
        const long long k = (long long)y - P.y0[b];
        const long long xa = P.xa[b] + wmul(P.dxa[b], k), xb = P.xb[b] + wmul(P.dxb[b], k);
        const long long xl = xa > xb ? xb : xa, xr = xa > xb ? xa : xb;
        int x1 = (int)((xl + (kOne >> 1)) >> kShift), x2 = (int)((xr + (kOne >> 1)) >> kShift);
        if (x2 >= 0 && x1 < width) {
            s.lo = x1 < 0 ? 0 : x1;
            s.hi = x2 >= width ? width - 1 : x2;
        }
        return s;
    }
    return s;
}

// ------------------------------------------------------------------------------------------ ThickLine, thickness 2
struct Thick {
    int drawn;                      // not clipped away
    int has_poly;
    Poly poly;
    int p0x, p0y, p1x, p1y;         // the radius-1 end dots
};

G6D_HD void thick_setup(int ax, int ay, int bx, int by, int width, int height, Thick& T) {
    // cv::line first clips the segment to the frame grown by the thickness on every side (and draws nothing when
    // nothing is left), in int as clipLine(Rect) does
    constexpr int m = 2;
    long long x1 = wadd(ax, m), y1 = wadd(ay, m), x2 = wadd(bx, m), y2 = wadd(by, m);
    T.drawn = clip_line((long long)width + 2 * m, (long long)height + 2 * m, x1, y1, x2, y2);
    T.has_poly = 0;
    if (!T.drawn) return;
    ax = wsub((int)x1, m); ay = wsub((int)y1, m); bx = wsub((int)x2, m); by = wsub((int)y2, m);
    const long long p0x = (long long)ax << kShift, p0y = (long long)ay << kShift;
    const long long p1x = (long long)bx << kShift, p1y = (long long)by << kShift;
    const double inv = 1. / (double)kOne;
    const double dx = (double)(p0x - p1x) * inv, dy = (double)(p1y - p0y) * inv;
    double r = dx * dx + dy * dy;
    const int thickness = 2 << (kShift - 1);
    T.has_poly = fabs(r) > 2.220446049250313e-16;
    if (T.has_poly) {
        r = (thickness + 0 * kOne * 0.5) / sqrt(r);
        const long long dpx = cv_round(dy * r), dpy = cv_round(dx * r);
        const long long v[8] = {p0x + dpx, p0y + dpy, p0x - dpx, p0y - dpy, p1x - dpx, p1y - dpy, p1x + dpx, p1y + dpy};
        poly_setup(v, width, height, T.poly);
    }
    T.p0x = ax; T.p0y = ay; T.p1x = bx; T.p1y = by;
}

// the spans of one thick line on row y: [0] fill, [1..8] the 4 outline runs and end points, [9], [10] the end dots
G6D_HD void thick_row(const Thick& T, int y, int width, int height, Span* out) {
    for (int k = 0; k < kSpansPerPrim; ++k) { out[k].lo = 1; out[k].hi = 0; }
    if (!T.drawn) return;
    if (T.has_poly && y >= 0 && y < height) {
        for (int k = 0; k < 4; ++k) line2_row(T.poly.outline[k], y, width, height, &out[1 + 2 * k], &out[2 + 2 * k]);
        out[0] = poly_row(T.poly, y, width);
    }
    const int r = ((2 << (kShift - 1)) + (int)(kOne >> 1)) >> kShift;
    out[9] = circle_row(T.p0x, T.p0y, r, y, width, height);
    out[10] = circle_row(T.p1x, T.p1y, r, y, width, height);
}

// ------------------------------------------------------------------------------------------ RGB -> NV12
// cv2.cvtColor(COLOR_RGB2YUV_I420)'s fixed point (BT.601 limited range, 20 fractional bits); the chroma of a 2x2 block
// from its top-left pixel.
constexpr int kYuvShift = 20;
G6D_HD uint8_t rgb_to_y(int r, int g, int b) {
    return (uint8_t)((269484 * r + 528482 * g + 102760 * b + (1 << (kYuvShift - 1)) + (16 << kYuvShift)) >> kYuvShift);
}
G6D_HD uint8_t rgb_to_u(int r, int g, int b) {
    return (uint8_t)((-155188 * r - 305135 * g + 460324 * b + (1 << (kYuvShift - 1)) + (128 << kYuvShift)) >> kYuvShift);
}
G6D_HD uint8_t rgb_to_v(int r, int g, int b) {
    return (uint8_t)((460324 * r - 385875 * g - 74448 * b + (1 << (kYuvShift - 1)) + (128 << kYuvShift)) >> kYuvShift);
}

}  // namespace draw
}  // namespace g6d
