// Temporal smoothing of tracked poses on the device (see track_math.cuh): one thread per sequence projects the box
// with the new raw pose, updates the sequence's corner history, averages it and solves the PnP, so a tracking step's
// graph runs from the uploaded frames to the smoothed poses without the host.  The *_host entry point runs the same
// code on host memory (CPU tests against numpy and cv2.solvePnP, no GPU needed).
#include "common.cuh"
#include "track_math.cuh"

namespace g6d {

__global__ void __launch_bounds__(32) track_smooth_kernel(const double* poses, int in_f32, const float* bbox, const double* Ks,
                                                           float* ring, int* count, int num, const double* weights, int S,
                                                           double* smoothed, double* avg_pts) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < S) track::smooth_one(s, poses, in_f32, bbox, Ks, ring, count, num, weights, smoothed, avg_pts);
}

// Several objects, rows object-major: row i = o * rows_per_obj + s is object o on sequence s, smoothed with box o and Ks[s].
// The row is sequence 0 of pointers shifted to it, so it runs smooth_one exactly as the single-object kernel does.
G6D_HD void smooth_row_objects(int i, int rows_per_obj, const double* poses, int in_f32, const float* bboxes, const double* Ks, float* ring,
                               int* count, int num, const double* w, double* smoothed, double* avg_pts) {
    const long long r = i;
    track::smooth_one(0, poses + r * 12, in_f32, bboxes + (long long)(i / rows_per_obj) * track::kCorners * 3,
                      Ks + (long long)(i % rows_per_obj) * 9, ring + r * num * 2 * track::kCorners, count + r, num, w, smoothed + r * 12,
                      avg_pts + r * 2 * track::kCorners);
}
__global__ void __launch_bounds__(32) track_smooth_objects_kernel(const double* poses, int in_f32, const float* bboxes, int n_rows,
                                                                   int rows_per_obj, const double* Ks, float* ring, int* count, int num,
                                                                   const double* weights, double* smoothed, double* avg_pts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_rows) smooth_row_objects(i, rows_per_obj, poses, in_f32, bboxes, Ks, ring, count, num, weights, smoothed, avg_pts);
}

}  // namespace g6d

using namespace g6d;

extern "C" int g6d_track_smooth(const double* poses, int poses_are_f32, const float* bbox, const double* Ks, float* ring, int* count,
                                int num, const double* weights, int S, double* smoothed, double* avg_pts, g6d_stream_t stream) {
    G6D_REQUIRE(poses && bbox && Ks && ring && count && weights && smoothed && avg_pts, "g6d_track_smooth: null pointer");
    G6D_REQUIRE(num >= 1 && S >= 1, "g6d_track_smooth: need num >= 1 and S >= 1 (got num=%d, S=%d)", num, S);
    track_smooth_kernel<<<ceil_div(S, 32), 32, 0, as_stream(stream)>>>(poses, poses_are_f32, bbox, Ks, ring, count, num, weights, S,
                                                                         smoothed, avg_pts);
    G6D_CHECK_LAUNCH("g6d_track_smooth");
    return G6D_OK;
}

extern "C" int g6d_track_smooth_host(const double* poses, int poses_are_f32, const float* bbox, const double* Ks, float* ring,
                                     int* count, int num, const double* weights, int S, double* smoothed, double* avg_pts) {
    G6D_REQUIRE(poses && bbox && Ks && ring && count && weights && smoothed && avg_pts, "g6d_track_smooth_host: null pointer");
    G6D_REQUIRE(num >= 1 && S >= 1, "g6d_track_smooth_host: need num >= 1 and S >= 1 (got num=%d, S=%d)", num, S);
    for (int s = 0; s < S; ++s)
        G6D_REQUIRE(count[s] >= 0 && count[s] <= num, "g6d_track_smooth_host: count[%d] = %d is beyond the ring of %d frames", s,
                    count[s], num);
    for (int s = 0; s < S; ++s) track::smooth_one(s, poses, poses_are_f32, bbox, Ks, ring, count, num, weights, smoothed, avg_pts);
    return G6D_OK;
}

extern "C" int g6d_track_smooth_objects(const double* poses, int poses_are_f32, const float* bboxes, int n_obj, int rows_per_obj,
                                        const double* Ks, float* ring, int* count, int num, const double* weights, double* smoothed,
                                        double* avg_pts, g6d_stream_t stream) {
    G6D_REQUIRE(poses && bboxes && Ks && ring && count && weights && smoothed && avg_pts, "g6d_track_smooth_objects: null pointer");
    G6D_REQUIRE(n_obj >= 1 && rows_per_obj >= 1 && num >= 1,
                "g6d_track_smooth_objects: need n_obj >= 1, rows_per_obj >= 1 and num >= 1 (got n_obj=%d, rows_per_obj=%d, num=%d)", n_obj,
                rows_per_obj, num);
    const int n_rows = n_obj * rows_per_obj;
    track_smooth_objects_kernel<<<ceil_div(n_rows, 32), 32, 0, as_stream(stream)>>>(poses, poses_are_f32, bboxes, n_rows, rows_per_obj, Ks,
                                                                                    ring, count, num, weights, smoothed, avg_pts);
    G6D_CHECK_LAUNCH("g6d_track_smooth_objects");
    return G6D_OK;
}

extern "C" int g6d_track_smooth_objects_host(const double* poses, int poses_are_f32, const float* bboxes, int n_obj, int rows_per_obj,
                                             const double* Ks, float* ring, int* count, int num, const double* weights, double* smoothed,
                                             double* avg_pts) {
    G6D_REQUIRE(poses && bboxes && Ks && ring && count && weights && smoothed && avg_pts, "g6d_track_smooth_objects_host: null pointer");
    G6D_REQUIRE(n_obj >= 1 && rows_per_obj >= 1 && num >= 1,
                "g6d_track_smooth_objects_host: need n_obj >= 1, rows_per_obj >= 1 and num >= 1 (got n_obj=%d, rows_per_obj=%d, num=%d)",
                n_obj, rows_per_obj, num);
    const int n_rows = n_obj * rows_per_obj;
    for (int i = 0; i < n_rows; ++i)
        G6D_REQUIRE(count[i] >= 0 && count[i] <= num, "g6d_track_smooth_objects_host: count[%d] = %d is beyond the ring of %d frames", i,
                    count[i], num);
    for (int i = 0; i < n_rows; ++i) smooth_row_objects(i, rows_per_obj, poses, poses_are_f32, bboxes, Ks, ring, count, num, weights, smoothed, avg_pts);
    return G6D_OK;
}
