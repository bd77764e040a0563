// Device frames into the packed layout (DESIGN.md row f14), as __host__ __device__ functions: g6d_frames_gather runs
// them over a device table of frames that already live on the GPU, and g6d_frames_gather_host runs the very same code
// on host memory, so the CPU tests pin the NV12 conversion against cv2.cvtColor without a GPU.
//
// The unit of work is one 2x2 pixel block of one frame: an RGB frame copies its (up to) 2x2 pixels from the pitched
// rows, an NV12 frame converts 4 Y samples and the block's one interleaved (U, V) pair into 12 RGB bytes.
//
// NV12 -> RGB is OpenCV's COLOR_YUV2RGB_NV12 (modules/imgproc/src/color_yuv.simd.hpp, BT.601 limited range) in its
// 20-bit fixed point: Y' = max(0, Y - 16) * 1220542, and with u = U - 128, v = V - 128 and the rounding term 2^19
//   R = sat((Y' + 2^19 + 1673527 v) >> 20)
//   G = sat((Y' + 2^19 - 852492 v - 409993 u) >> 20)
//   B = sat((Y' + 2^19 + 2116026 u) >> 20)
// Every term fits in int32 (|Y'| <= 239 * 1220542, |chroma| <= 2^19 + 2116026 * 128), and >> of a negative int is an
// arithmetic shift on every compiler this builds with, as in OpenCV; sat clamps to [0, 255].
//
// Frames resized and rotated to a working size on the way in (row f15) use the same conversion per source tap; the
// resize arithmetic is described above resized_pixel below.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/gen6d_b200.h"

#if defined(__CUDACC__)
#define G6D_FRAMES_HD __host__ __device__ inline
#else
#define G6D_FRAMES_HD inline
#endif

namespace g6d {
namespace frames {

constexpr int kCY = 1220542, kCUB = 2116026, kCUG = -409993, kCVG = -852492, kCVR = 1673527, kShift = 20;

G6D_FRAMES_HD uint8_t sat_u8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// one pixel from its Y sample and the block's chroma terms -> RGB at out[0..2]
G6D_FRAMES_HD void yuv_pixel(int Y, int ruv, int guv, int buv, uint8_t* out) {
    const int y = (Y > 16 ? Y - 16 : 0) * kCY;
    out[0] = sat_u8((y + ruv) >> kShift);
    out[1] = sat_u8((y + guv) >> kShift);
    out[2] = sat_u8((y + buv) >> kShift);
}

// block (bx, by) of frame fe: pixels (2*by + dy, 2*bx + dx) for dy, dx in {0, 1} inside rows x cols, written into its
// tightly packed [rows, cols, 3] image at packed + fe.offset
G6D_FRAMES_HD void gather_block(const g6d_device_frame& fe, int bx, int by, uint8_t* packed) {
    const int x0 = 2 * bx, y0 = 2 * by;
    uint8_t* dst = packed + fe.offset;
    const long long row_bytes = (long long)fe.cols * 3;
    if (fe.format == G6D_FRAME_NV12) {           // rows and cols are even: the block is whole
        const uint8_t* uv = fe.plane1 + (long long)by * fe.pitch1 + x0;
        const int u = (int)uv[0] - 128, v = (int)uv[1] - 128;
        const int half = 1 << (kShift - 1);
        const int ruv = half + kCVR * v, guv = half + kCVG * v + kCUG * u, buv = half + kCUB * u;
        for (int dy = 0; dy < 2; ++dy) {
            const uint8_t* ys = fe.plane0 + (long long)(y0 + dy) * fe.pitch0 + x0;
            uint8_t* d = dst + (long long)(y0 + dy) * row_bytes + (long long)x0 * 3;
            yuv_pixel(ys[0], ruv, guv, buv, d);
            yuv_pixel(ys[1], ruv, guv, buv, d + 3);
        }
        return;
    }
    const int nx = fe.cols - x0 < 2 ? fe.cols - x0 : 2, ny = fe.rows - y0 < 2 ? fe.rows - y0 : 2;
    for (int dy = 0; dy < ny; ++dy) {
        const uint8_t* s = fe.plane0 + (long long)(y0 + dy) * fe.pitch0 + (long long)x0 * 3;
        uint8_t* d = dst + (long long)(y0 + dy) * row_bytes + (long long)x0 * 3;
        for (int k = 0; k < nx * 3; ++k) d[k] = s[k];
    }
}

G6D_FRAMES_HD long long frame_end(const g6d_device_frame& fe) { return fe.offset + (long long)fe.rows * fe.cols * 3; }
G6D_FRAMES_HD long long frame_end(const g6d_resized_frame& fe) { return fe.offset + (long long)fe.rows * fe.cols * 3; }

// The bytes of packed that frame i zeroes: [end of frame i, start of the next frame or packed_bytes), and for the frame
// at the lowest offset also [0, its offset).  Over a table of non-overlapping frames (g6d_frames_table_check) these
// runs cover exactly the bytes no frame covers, each once.  -> (lo0, hi0) and (lo1, hi1), empty when lo >= hi.
template <class Frame>
G6D_FRAMES_HD void gap_runs(const Frame* table, int n, int i, long long packed_bytes, long long* lo0, long long* hi0,
                            long long* lo1, long long* hi1) {
    const long long start = table[i].offset, end = frame_end(table[i]);
    long long next = packed_bytes;
    bool lowest = true;
    for (int j = 0; j < n; ++j) {
        if (j == i) continue;
        if (table[j].offset >= end && table[j].offset < next) next = table[j].offset;
        if (table[j].offset < start) lowest = false;
    }
    *lo0 = end, *hi0 = next;
    *lo1 = 0, *hi1 = lowest ? start : 0;
}

// ------------------------------------------------------------------------------------------ resize + rotation (row f15)
// cv2.rotate(cv2.resize(frame, (cols, rows), interpolation=INTER_LINEAR), code) for a uint8 3-channel frame, as OpenCV
// computes it on x86 (modules/imgproc/src/resize.cpp, downscales and identity only):
//   - same size: a copy;
//   - exactly 2x in both axes (|scale - 2| < DBL_EPSILON): cv::resize takes INTER_AREA's fast path, (a+b+c+d+2) >> 2;
//   - otherwise fixed-point INTER_LINEAR with 11-bit coefficients.  Per destination column
//       scale = 1 / ((double)cols / src_cols),  fx = (float)((dx + 0.5) * scale - 0.5),  sx = floor(fx),  fx -= sx,
//     sx < 0 -> (sx, fx) = (0, 0) and sx >= src_cols - 1 -> (src_cols - 1, 0); weights sat_short(rint((1 - fx) * 2048))
//     and sat_short(rint(fx * 2048)); S = src[sx] * a0 + src[sx + 1] * a1 per channel.  Rows take the same fy, sy and
//     weights without the clamp of fy: only the row indices sy, sy + 1 are clamped to the frame.  The vertical pass rounds
//     as OpenCV's SIMD kernel (VResizeLinearVec_32s8u) does, which is what x86 builds return for every byte:
//       v = sat_u8((((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2).
// The double and float expressions are written as OpenCV writes them and must not be contracted into FMAs (frames.cu is
// built with -fmad=false; x86-64 host code has no FMA without -mfma).  The resize runs in source orientation and the
// rotation only maps output pixels to resized pixels, video2image's order.  NV12 taps are converted pixel by pixel with
// yuv_pixel first, as cv2.cvtColor then cv2.resize would see them.
constexpr int kCoefBits = 11, kCoefScale = 1 << kCoefBits;

G6D_FRAMES_HD int round_coef(float v) {             // saturate_cast<short>(v * INTER_RESIZE_COEF_SCALE): round half even
    const float r = rintf(v * (float)kCoefScale);
    return r < -32768.f ? -32768 : (r > 32767.f ? 32767 : (int)r);
}

// OpenCV's scale of an axis: 1 / inv_scale with inv_scale = dst / src, both in double
G6D_FRAMES_HD double axis_scale(int dst, int src) { return 1.0 / ((double)dst / (double)src); }

// is_area_fast && iscale == 2 for one axis
G6D_FRAMES_HD bool axis_halves(int dst, int src) {
    const double s = axis_scale(dst, src);
    return (s - 2.0 < 0 ? 2.0 - s : s - 2.0) < 2.220446049250313e-16;
}

// destination index d of an axis of dst samples over src -> source index s (not clamped) and its two weights
G6D_FRAMES_HD void linear_coefs(int d, int dst, int src, int* s, int* w0, int* w1, bool clamp) {
    float f = (float)(((double)d + 0.5) * axis_scale(dst, src) - 0.5);
    int i = (int)floorf(f);
    f -= (float)i;
    if (clamp) {
        if (i < 0) f = 0.f, i = 0;
        if (i >= src - 1) f = 0.f, i = src - 1;
    }
    *s = i;
    *w0 = round_coef(1.f - f);
    *w1 = round_coef(f);
}

// source pixel (y, x) of a resized-table frame as RGB
G6D_FRAMES_HD void source_pixel(const g6d_resized_frame& fe, int y, int x, uint8_t* out) {
    if (fe.format == G6D_FRAME_NV12) {
        const uint8_t* uv = fe.plane1 + (long long)(y >> 1) * fe.pitch1 + (x & ~1);
        const int u = (int)uv[0] - 128, v = (int)uv[1] - 128;
        const int half = 1 << (kShift - 1);
        yuv_pixel(fe.plane0[(long long)y * fe.pitch0 + x], half + kCVR * v, half + kCVG * v + kCUG * u, half + kCUB * u, out);
        return;
    }
    const uint8_t* s = fe.plane0 + (long long)y * fe.pitch0 + (long long)x * 3;
    out[0] = s[0], out[1] = s[1], out[2] = s[2];
}

// the working size (after the rotation) of a resized-table frame
G6D_FRAMES_HD int working_rows(const g6d_resized_frame& fe) { return fe.rotate == 90 || fe.rotate == 270 ? fe.cols : fe.rows; }
G6D_FRAMES_HD int working_cols(const g6d_resized_frame& fe) { return fe.rotate == 90 || fe.rotate == 270 ? fe.rows : fe.cols; }

// working pixel (r, c) of frame fe (inside working_rows x working_cols) into its packed image at packed + fe.offset
G6D_FRAMES_HD void resized_pixel(const g6d_resized_frame& fe, int r, int c, uint8_t* packed) {
    int ry = r, rx = c;                          // the pixel of the resized, not yet rotated image it shows
    if (fe.rotate == 90) ry = fe.rows - 1 - c, rx = r;
    else if (fe.rotate == 180) ry = fe.rows - 1 - r, rx = fe.cols - 1 - c;
    else if (fe.rotate == 270) ry = c, rx = fe.cols - 1 - r;
    uint8_t* dst = packed + fe.offset + ((long long)r * working_cols(fe) + c) * 3;
    if (fe.rows == fe.src_rows && fe.cols == fe.src_cols) {
        source_pixel(fe, ry, rx, dst);
        return;
    }
    uint8_t p[4][3];
    if (axis_halves(fe.rows, fe.src_rows) && axis_halves(fe.cols, fe.src_cols)) {
        source_pixel(fe, 2 * ry, 2 * rx, p[0]);
        source_pixel(fe, 2 * ry, 2 * rx + 1, p[1]);
        source_pixel(fe, 2 * ry + 1, 2 * rx, p[2]);
        source_pixel(fe, 2 * ry + 1, 2 * rx + 1, p[3]);
        for (int k = 0; k < 3; ++k) dst[k] = (uint8_t)(((int)p[0][k] + p[1][k] + p[2][k] + p[3][k] + 2) >> 2);
        return;
    }
    int sx, a0, a1, sy, b0, b1;
    linear_coefs(rx, fe.cols, fe.src_cols, &sx, &a0, &a1, true);
    linear_coefs(ry, fe.rows, fe.src_rows, &sy, &b0, &b1, false);
    const int x1 = sx + 1 < fe.src_cols ? sx + 1 : fe.src_cols - 1;
    const int y0 = sy < 0 ? 0 : (sy >= fe.src_rows ? fe.src_rows - 1 : sy);
    const int y1 = sy + 1 < 0 ? 0 : (sy + 1 >= fe.src_rows ? fe.src_rows - 1 : sy + 1);
    source_pixel(fe, y0, sx, p[0]);
    source_pixel(fe, y0, x1, p[1]);
    source_pixel(fe, y1, sx, p[2]);
    source_pixel(fe, y1, x1, p[3]);
    for (int k = 0; k < 3; ++k) {
        // S >> 4 <= 255 * 2049 >> 4 fits int16, so the SIMD kernel's saturating pack to int16 never clamps
        const int s0 = (p[0][k] * a0 + p[1][k] * a1) >> 4, s1 = (p[2][k] * a0 + p[3][k] * a1) >> 4;
        dst[k] = sat_u8((((b0 * s0) >> 16) + ((b1 * s1) >> 16) + 2) >> 2);
    }
}

}  // namespace frames
}  // namespace g6d
