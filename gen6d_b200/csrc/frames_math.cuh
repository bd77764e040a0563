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
#pragma once
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

// The bytes of packed that frame i zeroes: [end of frame i, start of the next frame or packed_bytes), and for the frame
// at the lowest offset also [0, its offset).  Over a table of non-overlapping frames (g6d_frames_table_check) these
// runs cover exactly the bytes no frame covers, each once.  -> (lo0, hi0) and (lo1, hi1), empty when lo >= hi.
G6D_FRAMES_HD void gap_runs(const g6d_device_frame* table, int n, int i, long long packed_bytes, long long* lo0, long long* hi0,
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

}  // namespace frames
}  // namespace g6d
