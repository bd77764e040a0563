// Drawn frames (DESIGN.md row f16): predict.py's draw_bbox_3d into every destination frame, one launch per frame set.
//
// One CTA per (row pair, destination).  It projects and rounds the corners of the destination's boxes, lets one thread
// per primitive (a corner dot or a thick edge) compute the spans that primitive puts on the CTA's two rows
// (draw_math.cuh), then writes the rows pixel by pixel: the colour of the last primitive covering the pixel, else the
// source pixel.  An NV12 destination converts the pair's 2x2 blocks in the same pass.  Every destination byte is
// written once and every source byte read once.
#include "common.cuh"
#include "draw_math.cuh"

namespace g6d {

constexpr int kDrawThreads = 256;
constexpr int kDrawPrims = G6D_DRAW_MAX_BOXES * draw::kPrims;

namespace draw {

struct RowSpans {           // one row's spans: per primitive its bound and its kSpansPerPrim spans (lo > hi: empty)
    uint16_t blo[kDrawPrims], bhi[kDrawPrims];
    uint16_t lo[kDrawPrims][kSpansPerPrim], hi[kDrawPrims][kSpansPerPrim];
};

G6D_HD void prim_row_spans(const int* pts, int k, int y, int width, int height, Span* s) {
    if (k < track::kCorners) {
        s[0] = circle_row(pts[2 * k], pts[2 * k + 1], 2, y, width, height);
        for (int j = 1; j < kSpansPerPrim; ++j) { s[j].lo = 1; s[j].hi = 0; }
        return;
    }
    const int e = k - track::kCorners, a = edge_end(e, 0), b = edge_end(e, 1);
    Thick T;
    thick_setup(pts[2 * a], pts[2 * a + 1], pts[2 * b], pts[2 * b + 1], width, height, T);
    thick_row(T, y, width, height, s);
}

// the colour of pixel x from the spans of row `row`, primitives last to first; false: no primitive covers it
G6D_HD bool pixel_color(const RowSpans& R, int np, const uint8_t (*colors)[4], int x, uint8_t* rgb) {
    for (int p = np - 1; p >= 0; --p) {
        if (x < R.blo[p] || x > R.bhi[p]) continue;
        for (int j = 0; j < kSpansPerPrim; ++j)
            if (x >= R.lo[p][j] && x <= R.hi[p][j]) {
                const uint8_t* c = colors[p];
                rgb[0] = c[0]; rgb[1] = c[1]; rgb[2] = c[2];
                return true;
            }
    }
    return false;
}

G6D_HD void store_spans(RowSpans& R, int p, const Span* s) {
    int blo = 65535, bhi = -1;
    for (int j = 0; j < kSpansPerPrim; ++j) {
        const bool e = s[j].lo > s[j].hi;
        R.lo[p][j] = e ? 1 : (uint16_t)s[j].lo;
        R.hi[p][j] = e ? 0 : (uint16_t)s[j].hi;
        if (!e) {
            blo = s[j].lo < blo ? s[j].lo : blo;
            bhi = s[j].hi > bhi ? s[j].hi : bhi;
        }
    }
    R.blo[p] = bhi < 0 ? 1 : (uint16_t)blo;
    R.bhi[p] = bhi < 0 ? 0 : (uint16_t)bhi;
}

G6D_HD void box_colors(const g6d_draw_box& b, uint8_t (*colors)[4]) {
    for (int k = 0; k < kPrims; ++k) {
        const bool dot = k < track::kCorners;
        colors[k][0] = dot ? 255 : b.color[0];
        colors[k][1] = dot ? 0 : b.color[1];
        colors[k][2] = dot ? 0 : b.color[2];
        colors[k][3] = 0;
    }
}

G6D_HD void write_pixel_pair(const g6d_device_frame& d, int y, int bx, const uint8_t* px) {   // px: 2 rows x 2 cols RGB
    uint8_t* Y = (uint8_t*)d.plane0;
    for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 2; ++c) {
            const uint8_t* p = px + (r * 2 + c) * 3;
            Y[(long long)(y + r) * d.pitch0 + 2 * bx + c] = rgb_to_y(p[0], p[1], p[2]);
        }
    uint8_t* uv = (uint8_t*)d.plane1 + (long long)(y / 2) * d.pitch1 + 2 * bx;
    uv[0] = rgb_to_u(px[0], px[1], px[2]);
    uv[1] = rgb_to_v(px[0], px[1], px[2]);
}

}  // namespace draw

__device__ __forceinline__ bool draw_dst_ok(const g6d_device_frame& d, const g6d_draw_src& s) {
    if (d.rows != s.rows || d.cols != s.cols || d.rows <= 0 || d.cols <= 0) return false;
    if (d.format == G6D_FRAME_NV12) return (d.rows & 1) == 0 && (d.cols & 1) == 0;
    return d.format == G6D_FRAME_RGB;
}

__global__ void __launch_bounds__(kDrawThreads)
draw_boxes_kernel(const uint8_t* __restrict__ src, const g6d_draw_src* __restrict__ srcs, int n_src, const double* __restrict__ poses,
                  const double* __restrict__ Ks, const float* __restrict__ bboxes, const long long* __restrict__ ids,
                  const g6d_draw_box* __restrict__ boxes, int n_boxes, const g6d_device_frame* __restrict__ dsts) {
    __shared__ draw::RowSpans rows[2];
    __shared__ uint8_t colors[kDrawPrims][4];
    __shared__ int pts[G6D_DRAW_MAX_BOXES][16];
    __shared__ int box_idx[G6D_DRAW_MAX_BOXES];
    __shared__ int nb;
    const int d = blockIdx.y, y0 = 2 * blockIdx.x, tid = threadIdx.x;
    const g6d_device_frame dst = dsts[d];
    const g6d_draw_src sf = srcs[d % n_src];
    if (!draw_dst_ok(dst, sf) || y0 >= dst.rows) return;
    if (tid == 0) {
        int n = 0;
        for (int b = 0; b < n_boxes && n < G6D_DRAW_MAX_BOXES; ++b)
            if (boxes[b].dst == d && (boxes[b].valid < 0 || ids[boxes[b].valid] >= 0)) box_idx[n++] = b;
        nb = n;
    }
    __syncthreads();
    if (tid < nb) {
        const g6d_draw_box b = boxes[box_idx[tid]];
        draw::box_corners(bboxes + (long long)b.bbox * 24, poses + (long long)b.pose * 12, b.pose_f32, Ks + (long long)b.K * 9, pts[tid]);
        draw::box_colors(b, colors + tid * draw::kPrims);
    }
    __syncthreads();
    const int np = nb * draw::kPrims;
    for (int t = tid; t < 2 * np; t += kDrawThreads) {
        const int r = t / np, p = t % np;
        draw::Span s[draw::kSpansPerPrim];
        draw::prim_row_spans(pts[p / draw::kPrims], p % draw::kPrims, y0 + r, dst.cols, dst.rows, s);
        draw::store_spans(rows[r], p, s);
    }
    __syncthreads();
    const uint8_t* srow = src + sf.offset + (long long)y0 * sf.pitch;
    const int nrows = y0 + 1 < dst.rows ? 2 : 1;
    if (dst.format == G6D_FRAME_RGB) {
        for (int i = tid; i < nrows * dst.cols; i += kDrawThreads) {
            const int r = i / dst.cols, x = i % dst.cols;
            const uint8_t* sp = srow + (long long)r * sf.pitch + 3 * x;
            uint8_t px[3] = {sp[0], sp[1], sp[2]};
            draw::pixel_color(rows[r], np, colors, x, px);
            uint8_t* dp = (uint8_t*)dst.plane0 + (long long)(y0 + r) * dst.pitch0 + 3 * x;
            dp[0] = px[0]; dp[1] = px[1]; dp[2] = px[2];
        }
    } else {
        for (int bx = tid; 2 * bx < dst.cols; bx += kDrawThreads) {
            uint8_t px[12];
            for (int r = 0; r < 2; ++r)
                for (int c = 0; c < 2; ++c) {
                    const uint8_t* sp = srow + (long long)r * sf.pitch + 3 * (2 * bx + c);
                    uint8_t* q = px + (r * 2 + c) * 3;
                    q[0] = sp[0]; q[1] = sp[1]; q[2] = sp[2];
                    draw::pixel_color(rows[r], np, colors, 2 * bx + c, q);
                }
            draw::write_pixel_pair(dst, y0, bx, px);
        }
    }
}

__global__ void __launch_bounds__(kDrawThreads)
rgb_to_nv12_kernel(const uint8_t* __restrict__ rgb, long long pitch, int rows, int cols, uint8_t* y, long long pitch_y, uint8_t* uv,
                   long long pitch_uv) {
    const int bx = blockIdx.x * kDrawThreads + threadIdx.x, by = blockIdx.y;
    if (2 * bx >= cols) return;
    const g6d_device_frame d{y, uv, pitch_y, pitch_uv, rows, cols, G6D_FRAME_NV12, 0};
    uint8_t px[12];
    for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 2; ++c)
            for (int k = 0; k < 3; ++k) px[(r * 2 + c) * 3 + k] = rgb[(long long)(2 * by + r) * pitch + 3 * (2 * bx + c) + k];
    draw::write_pixel_pair(d, 2 * by, bx, px);
}

}  // namespace g6d

extern "C" int g6d_draw_check(const g6d_draw_src* srcs, int n_src, const g6d_draw_box* boxes, int n_boxes, const g6d_device_frame* dsts,
                              int n_dst, int n_poses, int n_Ks, int n_bboxes, int n_ids) {
    G6D_REQUIRE(srcs && dsts && (boxes || n_boxes == 0), "g6d_draw_check: null table");
    G6D_REQUIRE(n_src > 0 && n_src <= G6D_FRAMES_MAX, "g6d_draw_check: n_src = %d, need 1..%d", n_src, G6D_FRAMES_MAX);
    G6D_REQUIRE(n_dst > 0 && n_dst <= 65535, "g6d_draw_check: n_dst = %d, need 1..65535", n_dst);
    G6D_REQUIRE(n_boxes >= 0, "g6d_draw_check: n_boxes = %d", n_boxes);
    for (int i = 0; i < n_src; ++i)
        G6D_REQUIRE(srcs[i].rows > 0 && srcs[i].cols > 0 && srcs[i].rows <= 65535 && srcs[i].cols <= 65535 &&
                        srcs[i].offset >= 0 && srcs[i].pitch >= 3LL * srcs[i].cols,
                    "g6d_draw_check: source %d is %d x %d (offset %lld, pitch %lld); need 1..65535 on each axis and a pitch >= "
                    "3 x its width", i, srcs[i].rows, srcs[i].cols, srcs[i].offset, srcs[i].pitch);
    for (int d = 0; d < n_dst; ++d) {
        const g6d_device_frame& e = dsts[d];
        const g6d_draw_src& s = srcs[d % n_src];
        G6D_REQUIRE(e.rows == s.rows && e.cols == s.cols, "g6d_draw_check: destination %d is %d x %d, its source %d is %d x %d", d,
                    e.rows, e.cols, d % n_src, s.rows, s.cols);
        G6D_REQUIRE(e.plane0 && (e.format == G6D_FRAME_RGB || e.plane1), "g6d_draw_check: destination %d has a null plane", d);
        if (e.format == G6D_FRAME_NV12) {
            G6D_REQUIRE(e.rows % 2 == 0 && e.cols % 2 == 0, "g6d_draw_check: NV12 destination %d is %d x %d; NV12 needs an even "
                        "height and width", d, e.rows, e.cols);
            G6D_REQUIRE(e.pitch0 >= e.cols && e.pitch1 >= e.cols, "g6d_draw_check: NV12 destination %d has row pitches %lld, %lld "
                        "below its width %d", d, e.pitch0, e.pitch1, e.cols);
        } else {
            G6D_REQUIRE(e.format == G6D_FRAME_RGB, "g6d_draw_check: destination %d has unknown format %d", d, e.format);
            G6D_REQUIRE(e.pitch0 >= 3LL * e.cols, "g6d_draw_check: RGB destination %d has row pitch %lld below 3 x its width %d", d,
                        e.pitch0, e.cols);
        }
        int n = 0;
        for (int b = 0; b < n_boxes; ++b) n += boxes[b].dst == d;
        G6D_REQUIRE(n <= G6D_DRAW_MAX_BOXES, "g6d_draw_check: destination %d has %d boxes, at most %d", d, n, G6D_DRAW_MAX_BOXES);
    }
    for (int b = 0; b < n_boxes; ++b) {
        const g6d_draw_box& e = boxes[b];
        G6D_REQUIRE(e.dst >= 0 && e.dst < n_dst && e.pose >= 0 && e.pose < n_poses && e.K >= 0 && e.K < n_Ks && e.bbox >= 0 &&
                        e.bbox < n_bboxes && e.valid >= -1 && e.valid < n_ids,
                    "g6d_draw_check: box %d (dst %d, pose %d, K %d, bbox %d, valid %d) indexes outside %d destinations, %d poses, "
                    "%d Ks, %d boxes, %d ids", b, e.dst, e.pose, e.K, e.bbox, e.valid, n_dst, n_poses, n_Ks, n_bboxes, n_ids);
    }
    return G6D_OK;
}

extern "C" int g6d_draw_boxes(const uint8_t* src, const g6d_draw_src* srcs, int n_src, const double* poses, const double* Ks,
                              const float* bboxes, const long long* ids, const g6d_draw_box* boxes, int n_boxes,
                              const g6d_device_frame* dsts, int n_dst, int max_rows, int max_cols, g6d_stream_t stream) {
    G6D_REQUIRE(src && srcs && dsts && (n_boxes == 0 || (boxes && poses && Ks && bboxes)), "g6d_draw_boxes: null pointer");
    G6D_REQUIRE(n_src > 0 && n_src <= G6D_FRAMES_MAX && n_dst > 0 && n_dst <= 65535 && n_boxes >= 0,
                "g6d_draw_boxes: %d sources, %d destinations, %d boxes", n_src, n_dst, n_boxes);
    G6D_REQUIRE(max_rows > 0 && max_cols > 0 && max_rows <= 65535 && max_cols <= 65535, "g6d_draw_boxes: bad frame bound %d x %d",
                max_rows, max_cols);
    dim3 grid((unsigned)((max_rows + 1) / 2), (unsigned)n_dst);
    g6d::draw_boxes_kernel<<<grid, g6d::kDrawThreads, 0, g6d::as_stream(stream)>>>(src, srcs, n_src, poses, Ks, bboxes, ids, boxes,
                                                                                  n_boxes, dsts);
    G6D_CHECK_LAUNCH("g6d_draw_boxes");
    return G6D_OK;
}

extern "C" int g6d_draw_boxes_host(const uint8_t* src, const g6d_draw_src* srcs, int n_src, const double* poses, int n_poses,
                                   const double* Ks, int n_Ks, const float* bboxes, int n_bboxes, const long long* ids, int n_ids,
                                   const g6d_draw_box* boxes, int n_boxes, const g6d_device_frame* dsts, int n_dst) {
    using namespace g6d;
    const int rc = g6d_draw_check(srcs, n_src, boxes, n_boxes, dsts, n_dst, n_poses, n_Ks, n_bboxes, n_ids);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(src && (n_boxes == 0 || (poses && Ks && bboxes)) && (n_ids == 0 || ids), "g6d_draw_boxes_host: null buffer");
    static thread_local draw::RowSpans rows[2];
    uint8_t colors[kDrawPrims][4];
    int pts[G6D_DRAW_MAX_BOXES][16];
    for (int d = 0; d < n_dst; ++d) {
        const g6d_device_frame& dst = dsts[d];
        const g6d_draw_src& sf = srcs[d % n_src];
        int nb = 0;
        for (int b = 0; b < n_boxes; ++b) {
            if (boxes[b].dst != d || (boxes[b].valid >= 0 && ids[boxes[b].valid] < 0)) continue;
            const g6d_draw_box& e = boxes[b];
            draw::box_corners(bboxes + (long long)e.bbox * 24, poses + (long long)e.pose * 12, e.pose_f32, Ks + (long long)e.K * 9, pts[nb]);
            draw::box_colors(e, colors + nb * draw::kPrims);
            ++nb;
        }
        const int np = nb * draw::kPrims;
        for (int y0 = 0; y0 < dst.rows; y0 += 2) {
            const int nrows = y0 + 1 < dst.rows ? 2 : 1;
            for (int r = 0; r < nrows; ++r)
                for (int p = 0; p < np; ++p) {
                    draw::Span s[draw::kSpansPerPrim];
                    draw::prim_row_spans(pts[p / draw::kPrims], p % draw::kPrims, y0 + r, dst.cols, dst.rows, s);
                    draw::store_spans(rows[r], p, s);
                }
            const uint8_t* srow = src + sf.offset + (long long)y0 * sf.pitch;
            if (dst.format == G6D_FRAME_RGB) {
                for (int r = 0; r < nrows; ++r)
                    for (int x = 0; x < dst.cols; ++x) {
                        const uint8_t* sp = srow + (long long)r * sf.pitch + 3 * x;
                        uint8_t px[3] = {sp[0], sp[1], sp[2]};
                        draw::pixel_color(rows[r], np, colors, x, px);
                        uint8_t* dp = (uint8_t*)dst.plane0 + (long long)(y0 + r) * dst.pitch0 + 3 * x;
                        dp[0] = px[0]; dp[1] = px[1]; dp[2] = px[2];
                    }
            } else {
                for (int bx = 0; 2 * bx < dst.cols; ++bx) {
                    uint8_t px[12];
                    for (int r = 0; r < 2; ++r)
                        for (int c = 0; c < 2; ++c) {
                            const uint8_t* sp = srow + (long long)r * sf.pitch + 3 * (2 * bx + c);
                            uint8_t* q = px + (r * 2 + c) * 3;
                            q[0] = sp[0]; q[1] = sp[1]; q[2] = sp[2];
                            draw::pixel_color(rows[r], np, colors, 2 * bx + c, q);
                        }
                    draw::write_pixel_pair(dst, y0, bx, px);
                }
            }
        }
    }
    return G6D_OK;
}

static int check_nv12(const char* name, const uint8_t* rgb, long long pitch, int rows, int cols, const uint8_t* y, long long pitch_y,
                      const uint8_t* uv, long long pitch_uv) {
    G6D_REQUIRE(rgb && y && uv, "%s: null buffer", name);
    G6D_REQUIRE(rows >= 2 && cols >= 2 && rows % 2 == 0 && cols % 2 == 0 && rows <= 131070,
                "%s: %d x %d; NV12 needs an even height and width", name, rows, cols);
    G6D_REQUIRE(pitch >= 3LL * cols && pitch_y >= cols && pitch_uv >= cols, "%s: row pitches %lld, %lld, %lld below the width %d",
                name, pitch, pitch_y, pitch_uv, cols);
    return G6D_OK;
}

extern "C" int g6d_rgb_to_nv12(const uint8_t* rgb, long long pitch, int rows, int cols, uint8_t* y, long long pitch_y, uint8_t* uv,
                               long long pitch_uv, g6d_stream_t stream) {
    const int rc = check_nv12("g6d_rgb_to_nv12", rgb, pitch, rows, cols, y, pitch_y, uv, pitch_uv);
    if (rc != G6D_OK) return rc;
    dim3 grid((unsigned)((cols / 2 + g6d::kDrawThreads - 1) / g6d::kDrawThreads), (unsigned)(rows / 2));
    g6d::rgb_to_nv12_kernel<<<grid, g6d::kDrawThreads, 0, g6d::as_stream(stream)>>>(rgb, pitch, rows, cols, y, pitch_y, uv, pitch_uv);
    G6D_CHECK_LAUNCH("g6d_rgb_to_nv12");
    return G6D_OK;
}

extern "C" int g6d_rgb_to_nv12_host(const uint8_t* rgb, long long pitch, int rows, int cols, uint8_t* y, long long pitch_y, uint8_t* uv,
                                    long long pitch_uv) {
    const int rc = check_nv12("g6d_rgb_to_nv12_host", rgb, pitch, rows, cols, y, pitch_y, uv, pitch_uv);
    if (rc != G6D_OK) return rc;
    const g6d_device_frame d{y, uv, pitch_y, pitch_uv, rows, cols, G6D_FRAME_NV12, 0};
    for (int by = 0; by < rows / 2; ++by)
        for (int bx = 0; bx < cols / 2; ++bx) {
            uint8_t px[12];
            for (int r = 0; r < 2; ++r)
                for (int c = 0; c < 2; ++c)
                    for (int k = 0; k < 3; ++k) px[(r * 2 + c) * 3 + k] = rgb[(long long)(2 * by + r) * pitch + 3 * (2 * bx + c) + k];
            g6d::draw::write_pixel_pair(d, 2 * by, bx, px);
        }
    return G6D_OK;
}
