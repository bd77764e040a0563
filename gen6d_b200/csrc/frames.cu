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
//
// Frames already on the device (row f14) reach the packed layout through g6d_frames_gather below: a pitched copy for
// RGB, OpenCV's NV12 conversion for decoder surfaces (frames_math.cuh).  g6d_frames_gather_resized (row f15) also
// resizes and rotates them to a working size as cv2.resize + cv2.rotate do; its float coefficients need this file built
// without FMA contraction (build.NO_FMA).
#include "common.cuh"
#include "frames_math.cuh"

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

// ------------------------------------------------------------------------------------------ device frames (row f14)
// The first node of a captured graph over frames that are already on the device: the table (a graph input, uploaded per
// call) holds their pointers and pitches, so the same graph serves every allocation and pitch of the same size pattern.

constexpr int kGatherThreads = 128;

// the conditions g6d_frames_table_check enforces on one entry; the kernel skips an entry that breaks them rather than
// write outside `packed`
__device__ __forceinline__ bool frame_ok(const g6d_device_frame& fe, long long packed_bytes) {
    if (fe.rows <= 0 || fe.cols <= 0 || fe.offset < 0 || frames::frame_end(fe) > packed_bytes) return false;
    if (fe.format == G6D_FRAME_NV12) return (fe.rows & 1) == 0 && (fe.cols & 1) == 0;
    return fe.format == G6D_FRAME_RGB;
}

// grid (ceil(ceil(max_cols/2) / 128), ceil(max_rows/2), n): one 2x2 pixel block per thread, consecutive threads on
// consecutive blocks of a row pair.  CTA (0, 0, i) also zeroes the bytes after frame i that no frame covers.
__global__ void __launch_bounds__(kGatherThreads)
frames_gather_kernel(const g6d_device_frame* __restrict__ table, int n, uint8_t* __restrict__ packed, long long packed_bytes) {
    const int i = blockIdx.z;
    const g6d_device_frame fe = table[i];
    if (!frame_ok(fe, packed_bytes)) return;
    if (blockIdx.x == 0 && blockIdx.y == 0) {
        __shared__ long long runs[4];
        if (threadIdx.x == 0) frames::gap_runs(table, n, i, packed_bytes, &runs[0], &runs[1], &runs[2], &runs[3]);
        __syncthreads();
        for (int r = 0; r < 2; ++r)
            for (long long x = runs[2 * r] + threadIdx.x; x < runs[2 * r + 1]; x += kGatherThreads) packed[x] = 0;
    }
    const int bx = blockIdx.x * kGatherThreads + threadIdx.x, by = blockIdx.y;
    if (2 * bx >= fe.cols || 2 * by >= fe.rows) return;
    frames::gather_block(fe, bx, by, packed);
}

// ------------------------------------------------------------------------------------------ resized frames (row f15)
// The same first node for frames resized and rotated to their working size on the way in: one working pixel per thread,
// each computing its own column and row coefficients and converting its (up to) four source taps.
constexpr int kResizedThreads = 128;

__device__ __forceinline__ bool resized_ok(const g6d_resized_frame& fe, long long packed_bytes) {
    if (fe.rows <= 0 || fe.cols <= 0 || fe.rows > fe.src_rows || fe.cols > fe.src_cols || fe.offset < 0 ||
        frames::frame_end(fe) > packed_bytes)
        return false;
    if (fe.rotate != 0 && fe.rotate != 90 && fe.rotate != 180 && fe.rotate != 270) return false;
    if (fe.format == G6D_FRAME_NV12) return (fe.src_rows & 1) == 0 && (fe.src_cols & 1) == 0;
    return fe.format == G6D_FRAME_RGB;
}

// grid (ceil(max working cols / 128), max working rows, n); CTA (0, 0, i) also zeroes the bytes after frame i that no
// frame covers
__global__ void __launch_bounds__(kResizedThreads)
frames_gather_resized_kernel(const g6d_resized_frame* __restrict__ table, int n, uint8_t* __restrict__ packed,
                             long long packed_bytes) {
    const int i = blockIdx.z;
    const g6d_resized_frame fe = table[i];
    if (!resized_ok(fe, packed_bytes)) return;
    if (blockIdx.x == 0 && blockIdx.y == 0) {
        __shared__ long long runs[4];
        if (threadIdx.x == 0) frames::gap_runs(table, n, i, packed_bytes, &runs[0], &runs[1], &runs[2], &runs[3]);
        __syncthreads();
        for (int r = 0; r < 2; ++r)
            for (long long x = runs[2 * r] + threadIdx.x; x < runs[2 * r + 1]; x += kResizedThreads) packed[x] = 0;
    }
    const int c = blockIdx.x * kResizedThreads + threadIdx.x, r = blockIdx.y;
    if (c >= frames::working_cols(fe) || r >= frames::working_rows(fe)) return;
    frames::resized_pixel(fe, r, c, packed);
}

}  // namespace g6d

static int check_table(const char* name, const g6d_device_frame* t, int n, long long packed_bytes) {
    G6D_REQUIRE(t, "%s: null table", name);
    G6D_REQUIRE(n > 0 && n <= G6D_FRAMES_MAX, "%s: n = %d frames, need 1..%d", name, n, G6D_FRAMES_MAX);
    G6D_REQUIRE(packed_bytes > 0, "%s: packed_bytes = %lld", name, packed_bytes);
    for (int i = 0; i < n; ++i) {
        const g6d_device_frame& e = t[i];
        G6D_REQUIRE(e.format == G6D_FRAME_RGB || e.format == G6D_FRAME_NV12, "%s: frame %d has unknown format %d (RGB %d, NV12 %d)",
                    name, i, e.format, G6D_FRAME_RGB, G6D_FRAME_NV12);
        G6D_REQUIRE(e.rows > 0 && e.cols > 0 && e.rows <= 131070, "%s: frame %d is %d x %d", name, i, e.rows, e.cols);
        G6D_REQUIRE(e.plane0 && (e.format == G6D_FRAME_RGB || e.plane1), "%s: frame %d has a null plane", name, i);
        if (e.format == G6D_FRAME_NV12) {
            G6D_REQUIRE(e.rows % 2 == 0 && e.cols % 2 == 0, "%s: NV12 frame %d is %d x %d; NV12 needs an even height and width",
                        name, i, e.rows, e.cols);
            G6D_REQUIRE(e.pitch0 >= e.cols && e.pitch1 >= e.cols,
                        "%s: NV12 frame %d has row pitches %lld (Y) and %lld (UV) below its width %d", name, i, e.pitch0, e.pitch1,
                        e.cols);
        } else {
            G6D_REQUIRE(e.pitch0 >= 3LL * e.cols, "%s: RGB frame %d has row pitch %lld below 3 x its width %d", name, i, e.pitch0,
                        e.cols);
        }
        G6D_REQUIRE(e.offset >= 0 && g6d::frames::frame_end(e) <= packed_bytes,
                    "%s: frame %d (offset %lld, %d x %d) lies outside the %lld-byte packed buffer", name, i, e.offset, e.rows,
                    e.cols, packed_bytes);
    }
    for (int i = 0; i < n; ++i)                 // no two packed images overlap (n <= G6D_FRAMES_MAX: at most 2^19 pairs)
        for (int j = i + 1; j < n; ++j)
            G6D_REQUIRE(t[i].offset >= g6d::frames::frame_end(t[j]) || t[j].offset >= g6d::frames::frame_end(t[i]),
                        "%s: the packed images of frames %d and %d overlap", name, i, j);
    return G6D_OK;
}

extern "C" int g6d_frames_table_check(const g6d_device_frame* host_table, int n, long long packed_bytes) {
    return check_table("g6d_frames_table_check", host_table, n, packed_bytes);
}

extern "C" int g6d_frames_gather(const g6d_device_frame* table, int n, int max_rows, int max_cols, uint8_t* packed,
                                 long long packed_bytes, g6d_stream_t stream) {
    G6D_REQUIRE(table && packed && packed_bytes > 0, "g6d_frames_gather: null table or buffer, or empty packed buffer");
    G6D_REQUIRE(n > 0 && n <= G6D_FRAMES_MAX, "g6d_frames_gather: n = %d frames, need 1..%d", n, G6D_FRAMES_MAX);
    G6D_REQUIRE(max_rows > 0 && max_cols > 0 && max_rows <= 131070, "g6d_frames_gather: bad frame bound %d x %d", max_rows,
                max_cols);
    const long long blocks_x = ((long long)(max_cols + 1) / 2 + g6d::kGatherThreads - 1) / g6d::kGatherThreads;
    dim3 grid((unsigned)blocks_x, (max_rows + 1) / 2, n);
    g6d::frames_gather_kernel<<<grid, g6d::kGatherThreads, 0, g6d::as_stream(stream)>>>(table, n, packed, packed_bytes);
    G6D_CHECK_LAUNCH("g6d_frames_gather");
    return G6D_OK;
}

extern "C" int g6d_frames_gather_host(const g6d_device_frame* host_table, int n, uint8_t* packed, long long packed_bytes) {
    const int rc = check_table("g6d_frames_gather_host", host_table, n, packed_bytes);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(packed, "g6d_frames_gather_host: null packed buffer");
    for (int i = 0; i < n; ++i) {
        const g6d_device_frame& fe = host_table[i];
        long long run[4];
        g6d::frames::gap_runs(host_table, n, i, packed_bytes, &run[0], &run[1], &run[2], &run[3]);
        for (int r = 0; r < 2; ++r)
            for (long long x = run[2 * r]; x < run[2 * r + 1]; ++x) packed[x] = 0;
        for (int by = 0; 2 * by < fe.rows; ++by)
            for (int bx = 0; 2 * bx < fe.cols; ++bx) g6d::frames::gather_block(fe, bx, by, packed);
    }
    return G6D_OK;
}

static int check_resized_table(const char* name, const g6d_resized_frame* t, int n, long long packed_bytes) {
    G6D_REQUIRE(t, "%s: null table", name);
    G6D_REQUIRE(n > 0 && n <= G6D_FRAMES_MAX, "%s: n = %d frames, need 1..%d", name, n, G6D_FRAMES_MAX);
    G6D_REQUIRE(packed_bytes > 0, "%s: packed_bytes = %lld", name, packed_bytes);
    for (int i = 0; i < n; ++i) {
        const g6d_resized_frame& e = t[i];
        G6D_REQUIRE(e.format == G6D_FRAME_RGB || e.format == G6D_FRAME_NV12, "%s: frame %d has unknown format %d (RGB %d, NV12 %d)",
                    name, i, e.format, G6D_FRAME_RGB, G6D_FRAME_NV12);
        G6D_REQUIRE(e.rotate == 0 || e.rotate == 90 || e.rotate == 180 || e.rotate == 270,
                    "%s: frame %d has rotation %d; need 0, 90, 180 or 270 degrees clockwise", name, i, e.rotate);
        G6D_REQUIRE(e.src_rows > 0 && e.src_cols > 0 && e.src_rows <= 131070, "%s: frame %d has a %d x %d source", name, i,
                    e.src_rows, e.src_cols);
        G6D_REQUIRE(e.plane0 && (e.format == G6D_FRAME_RGB || e.plane1), "%s: frame %d has a null plane", name, i);
        if (e.format == G6D_FRAME_NV12) {
            G6D_REQUIRE(e.src_rows % 2 == 0 && e.src_cols % 2 == 0,
                        "%s: NV12 frame %d is %d x %d; NV12 needs an even height and width", name, i, e.src_rows, e.src_cols);
            G6D_REQUIRE(e.pitch0 >= e.src_cols && e.pitch1 >= e.src_cols,
                        "%s: NV12 frame %d has row pitches %lld (Y) and %lld (UV) below its width %d", name, i, e.pitch0,
                        e.pitch1, e.src_cols);
        } else {
            G6D_REQUIRE(e.pitch0 >= 3LL * e.src_cols, "%s: RGB frame %d has row pitch %lld below 3 x its width %d", name, i,
                        e.pitch0, e.src_cols);
        }
        G6D_REQUIRE(e.rows >= 1 && e.cols >= 1 && e.rows <= e.src_rows && e.cols <= e.src_cols && e.rows <= 65535 &&
                        e.cols <= 65535,
                    "%s: frame %d resizes %d x %d to %d x %d; need a working size of at least 1 x 1 and at most the source "
                    "size (no upscaling) and 65535 on each axis", name, i, e.src_rows, e.src_cols, e.rows, e.cols);
        G6D_REQUIRE(e.offset >= 0 && g6d::frames::frame_end(e) <= packed_bytes,
                    "%s: frame %d (offset %lld, %d x %d) lies outside the %lld-byte packed buffer", name, i, e.offset, e.rows,
                    e.cols, packed_bytes);
    }
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j)
            G6D_REQUIRE(t[i].offset >= g6d::frames::frame_end(t[j]) || t[j].offset >= g6d::frames::frame_end(t[i]),
                        "%s: the packed images of frames %d and %d overlap", name, i, j);
    return G6D_OK;
}

extern "C" int g6d_frames_resized_table_check(const g6d_resized_frame* host_table, int n, long long packed_bytes) {
    return check_resized_table("g6d_frames_resized_table_check", host_table, n, packed_bytes);
}

extern "C" int g6d_frames_gather_resized(const g6d_resized_frame* table, int n, int max_rows, int max_cols, uint8_t* packed,
                                         long long packed_bytes, g6d_stream_t stream) {
    G6D_REQUIRE(table && packed && packed_bytes > 0, "g6d_frames_gather_resized: null table or buffer, or empty packed buffer");
    G6D_REQUIRE(n > 0 && n <= G6D_FRAMES_MAX, "g6d_frames_gather_resized: n = %d frames, need 1..%d", n, G6D_FRAMES_MAX);
    G6D_REQUIRE(max_rows > 0 && max_cols > 0 && max_rows <= 65535 && max_cols <= 65535,
                "g6d_frames_gather_resized: bad frame bound %d x %d", max_rows, max_cols);
    dim3 grid((unsigned)((max_cols + g6d::kResizedThreads - 1) / g6d::kResizedThreads), max_rows, n);
    g6d::frames_gather_resized_kernel<<<grid, g6d::kResizedThreads, 0, g6d::as_stream(stream)>>>(table, n, packed, packed_bytes);
    G6D_CHECK_LAUNCH("g6d_frames_gather_resized");
    return G6D_OK;
}

extern "C" int g6d_frames_gather_resized_host(const g6d_resized_frame* host_table, int n, uint8_t* packed, long long packed_bytes) {
    const int rc = check_resized_table("g6d_frames_gather_resized_host", host_table, n, packed_bytes);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(packed, "g6d_frames_gather_resized_host: null packed buffer");
    for (int i = 0; i < n; ++i) {
        const g6d_resized_frame& fe = host_table[i];
        long long run[4];
        g6d::frames::gap_runs(host_table, n, i, packed_bytes, &run[0], &run[1], &run[2], &run[3]);
        for (int r = 0; r < 2; ++r)
            for (long long x = run[2 * r]; x < run[2 * r + 1]; ++x) packed[x] = 0;
        for (int r = 0; r < g6d::frames::working_rows(fe); ++r)
            for (int c = 0; c < g6d::frames::working_cols(fe); ++c) g6d::frames::resized_pixel(fe, r, c, packed);
    }
    return G6D_OK;
}

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
