// Frames of different sizes on one zero-padded canvas (DESIGN.md row f13).
//
// The crops between the stages are cut by g6d_warp_affine_u8 / g6d_warp_perspective_u8 from g6d_warp_job records whose
// `src` the glue kernels compute as frames + i*rows*cols*3.  A batch of frames of different sizes is therefore handed to
// them as one canvas [n, H, W, 3] (H, W the largest frame size) with every frame in its top-left corner and zeros
// elsewhere: a warp tap outside rows x cols contributes 0 (BORDER_CONSTANT 0) and a tap in the padding reads a 0 byte,
// so every crop is bit-identical to the crop of the true-size frame.
//
// The canvas is written in one launch from the frames packed back to back.  Every byte is written, padding included,
// so a graph replay never depends on what the canvas held before.  The table is a kernel parameter: it is fixed by the
// frame sizes, which every captured graph of the canvas keys on.
#include "common.cuh"

namespace g6d {

template <int CAP>
struct FrameTable {
    g6d_frame_entry e[CAP];
};

constexpr int kCanvasThreads = 256, kCanvasBytesPerThread = 4;

// grid (ceil(W*3 / 1024), H, n): one canvas row segment of 1024 bytes per CTA, consecutive threads on consecutive bytes
template <int CAP>
__global__ void __launch_bounds__(kCanvasThreads)
frames_canvas_kernel(const uint8_t* __restrict__ packed, const __grid_constant__ FrameTable<CAP> table,
                     uint8_t* __restrict__ canvas, int H, int W) {
    const int y = blockIdx.y, i = blockIdx.z;
    const g6d_frame_entry fe = table.e[i];
    const long long row_bytes = (long long)W * 3;
    uint8_t* dst = canvas + ((long long)i * H + y) * row_bytes;
    const long long valid = y < fe.rows ? (long long)fe.cols * 3 : 0;        // bytes of this row that come from the frame
    const uint8_t* src = packed + fe.offset + (long long)y * fe.cols * 3;
    const long long x0 = (long long)blockIdx.x * kCanvasThreads * kCanvasBytesPerThread + threadIdx.x;
#pragma unroll
    for (int k = 0; k < kCanvasBytesPerThread; ++k) {
        const long long x = x0 + (long long)k * kCanvasThreads;
        if (x < row_bytes) dst[x] = x < valid ? src[x] : (uint8_t)0;
    }
}

template <int CAP>
int launch_canvas(const uint8_t* packed, const g6d_frame_entry* host_table, int n, uint8_t* canvas, int H, int W,
                  cudaStream_t stream) {
    FrameTable<CAP> t;
    for (int i = 0; i < n; ++i) t.e[i] = host_table[i];
    for (int i = n; i < CAP; ++i) t.e[i] = g6d_frame_entry{0, 0, 0};
    dim3 grid(ceil_div((long long)W * 3, kCanvasThreads * kCanvasBytesPerThread), H, n);
    frames_canvas_kernel<CAP><<<grid, kCanvasThreads, 0, stream>>>(packed, t, canvas, H, W);
    G6D_CHECK_LAUNCH("g6d_frames_canvas");
    return G6D_OK;
}

}  // namespace g6d

extern "C" int g6d_frames_canvas(const uint8_t* packed, long long packed_bytes, const g6d_frame_entry* host_table, int n,
                                 uint8_t* canvas, int H, int W, g6d_stream_t stream) {
    G6D_REQUIRE(packed && host_table && canvas && packed_bytes > 0, "g6d_frames_canvas: null buffer or empty packed input");
    G6D_REQUIRE(n > 0 && n <= G6D_FRAMES_MAX, "g6d_frames_canvas: n = %d frames, need 1..%d", n, G6D_FRAMES_MAX);
    G6D_REQUIRE(H > 0 && W > 0 && H <= 65535 && (long long)W * 3 <= 0x7fffffffLL,
                "g6d_frames_canvas: bad canvas size %d x %d", H, W);
    for (int i = 0; i < n; ++i) {
        const g6d_frame_entry& e = host_table[i];
        G6D_REQUIRE(e.rows > 0 && e.cols > 0 && e.rows <= H && e.cols <= W,
                    "g6d_frames_canvas: frame %d is %d x %d, the canvas %d x %d", i, e.rows, e.cols, H, W);
        G6D_REQUIRE(e.offset >= 0 && e.offset + (long long)e.rows * e.cols * 3 <= packed_bytes,
                    "g6d_frames_canvas: frame %d (offset %lld, %d x %d) lies outside the %lld-byte packed buffer", i, e.offset,
                    e.rows, e.cols, packed_bytes);
    }
    cudaStream_t s = g6d::as_stream(stream);
    return n <= 32 ? g6d::launch_canvas<32>(packed, host_table, n, canvas, H, W, s)
                   : g6d::launch_canvas<G6D_FRAMES_MAX>(packed, host_table, n, canvas, H, W, s);
}
