// Temporal smoothing of tracked poses on the device (see track_math.cuh): one thread per sequence projects the box
// with the new raw pose, updates the sequence's corner history, averages it and solves the PnP, so a tracking step's
// graph runs from the uploaded frames to the smoothed poses without the host.  The *_host entry point runs the same
// code on host memory (CPU tests against numpy and cv2.solvePnP, no GPU needed).  The multi-instance tracker's
// association (instance_track_math.cuh) lives here too: it needs the same no-contraction fp64.
#include "common.cuh"
#include "track_math.cuh"
#include "instance_track_math.cuh"

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

// Association of the multi-instance trackers (instance_track_math.cuh): ONE CTA.  Phase 1 runs one thread per
// (sequence, object) pair, pairs object-major (pair p = o*S + s); phase 2 numbers the spawned tracks in ascending
// (object, sequence, slot) order -- which is (object, sequence, detection) order, since a pair's unmatched detections take
// its empty slots in ascending order -- by an exclusive block scan of the pairs' spawn counts, chunk by chunk; thread 0
// then advances the counter.  Pair p's slot t is row p + t*K*S.  With a det_index (a step in which only some sequences
// detect) non-detecting pairs spawn nothing, and the threads also fill the list entries of the detection batch's padding
// rows.
constexpr int kAssocThreads = 256;

__global__ void __launch_bounds__(kAssocThreads) instances_associate_kernel(assoc::Args a, long long* next_id) {
    __shared__ int s_warp[kAssocThreads / 32];
    __shared__ long long s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int P = a.K * a.S;
    const long long stride = (long long)a.K * a.S;
    for (int p = tid; p < P; p += kAssocThreads) assoc::associate_sequence(p % a.S, p / a.S, a);
    if (a.det_index)
        for (int j = tid; j < a.D; j += kAssocThreads) assoc::pad_lists(j, a);
    if (tid == 0) s_base = *next_id;
    __syncthreads();
    for (int p0 = 0; p0 < P; p0 += kAssocThreads) {
        const int p = p0 + tid;
        int n = 0;
        if (p < P)
            for (int m = 0; m < a.M; ++m) n += a.spawned[p + m * stride];
        int incl = n;
        for (int o = 1; o < 32; o <<= 1) {
            const int x = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += x;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < kAssocThreads / 32; ++w) {
            before += w < warp ? s_warp[w] : 0;
            total += s_warp[w];
        }
        long long id = s_base + before + incl - n;
        if (p < P)
            for (int m = 0; m < a.M; ++m) {
                const long long i = p + m * stride;
                if (a.spawned[i]) a.ids[i] = id++;
            }
        __syncthreads();
        if (tid == 0) s_base += total;
        __syncthreads();
    }
    if (tid == 0) *next_id = s_base;
}

static int associate_ok(const char* name, const assoc::Args& a, const long long* next_id) {
    G6D_REQUIRE(a.S >= 1 && a.M >= 1 && a.M <= assoc::kMaxSlots, "%s: need S >= 1 and 1 <= M <= %d (got S=%d, M=%d)", name,
                assoc::kMaxSlots, a.S, a.M);
    G6D_REQUIRE(a.K >= 1 && (long long)a.K * a.S * a.M * 2 <= 0x7fffffffLL, "%s: need K >= 1 and 2*M*K*S rows within int (got K=%d)",
                name, a.K);
    G6D_REQUIRE(a.F >= 0 && a.r >= 0 && (a.F > 0 || a.r > 0) && a.num >= 1 && a.max_misses >= 0,
                "%s: need F, r >= 0 with max(F, r) >= 1, num >= 1 and max_misses >= 0 (got F=%d, r=%d, num=%d, max_misses=%d)", name,
                a.F, a.r, a.num, a.max_misses);
    G6D_REQUIRE(a.gate > 0. && a.gate < INFINITY && a.ref_resolution > 0., "%s: need a finite gate > 0 and ref_resolution > 0", name);
    const bool detects = !a.det_index || a.D > 0;
    G6D_REQUIRE(!a.det_index || (a.D >= 0 && a.D <= a.S), "%s: need 0 <= D <= S (got D=%d, S=%d)", name, a.D, a.S);
    G6D_REQUIRE(((a.det && a.valid && a.init) || !detects) && a.cams && a.prev && a.live && a.ids && a.misses && a.park && a.ring && a.count && a.work &&
                a.flags0 && a.lists && a.det_slot && a.spawned && a.dropped && next_id, "%s: null pointer", name);
    return G6D_OK;
}

static void associate_host(const assoc::Args& a, long long* next_id) {
    const long long stride = (long long)a.K * a.S;
    for (int p = 0; p < a.K * a.S; ++p) assoc::associate_sequence(p % a.S, p / a.S, a);
    if (a.det_index)
        for (int j = 0; j < a.D; ++j) assoc::pad_lists(j, a);
    for (int p = 0; p < a.K * a.S; ++p)
        for (int m = 0; m < a.M; ++m)
            if (a.spawned[p + m * stride]) a.ids[p + m * stride] = (*next_id)++;
}

static int associate_launch(const char* name, const assoc::Args& a, long long* next_id, g6d_stream_t stream) {
    const int rc = associate_ok(name, a, next_id);
    if (rc != G6D_OK) return rc;
    instances_associate_kernel<<<1, kAssocThreads, 0, as_stream(stream)>>>(a, next_id);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}

// Verification's slot update: one thread per row.
__global__ void __launch_bounds__(128) instances_verify_update_kernel(int n, const int* lost, const int* verified, int max_misses, int* live,
                                                                      long long* ids, int* misses, long long* dropped) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) assoc::verify_update(i, lost, verified, max_misses, live, ids, misses, dropped);
}

static int verify_update_ok(const char* name, int n, const int* lost, const int* verified, int max_misses, const int* live,
                            const long long* ids, const int* misses, const long long* dropped) {
    G6D_REQUIRE(n >= 1 && max_misses >= 0, "%s: need n >= 1 and max_misses >= 0 (got n=%d, max_misses=%d)", name, n, max_misses);
    G6D_REQUIRE(lost && verified && live && ids && misses && dropped, "%s: null pointer", name);
    return G6D_OK;
}

}  // namespace g6d

using namespace g6d;

extern "C" int g6d_instances_associate(int S, int M, int F, int r, const float* det, const int* valid, const double* init,
                                       const g6d_glue_camera* cams, double cx, double cy, double cz, double ref_resolution, double gate,
                                       int max_misses, const double* prev, int* live, long long* ids, int* misses, long long* next_id,
                                       double* park, float* ring, int* count, int num, double* work, uint8_t* flags0, int* lists,
                                       int* det_slot, int* spawned, long long* dropped, g6d_stream_t stream) {
    const assoc::Args a{S, 1, M, F, r, num, max_misses, det, valid, init, reinterpret_cast<const double*>(cams), nullptr, {cx, cy, cz},
                        ref_resolution, gate, prev, live, ids, misses, park, ring, count, work, flags0, lists, det_slot, spawned, dropped};
    return associate_launch("g6d_instances_associate", a, next_id, stream);
}

extern "C" int g6d_instances_associate_host(int S, int M, int F, int r, const float* det, const int* valid, const double* init,
                                            const g6d_glue_camera* cams, double cx, double cy, double cz, double ref_resolution,
                                            double gate, int max_misses, const double* prev, int* live, long long* ids, int* misses,
                                            long long* next_id, double* park, float* ring, int* count, int num, double* work,
                                            uint8_t* flags0, int* lists, int* det_slot, int* spawned, long long* dropped) {
    const assoc::Args a{S, 1, M, F, r, num, max_misses, det, valid, init, reinterpret_cast<const double*>(cams), nullptr, {cx, cy, cz},
                        ref_resolution, gate, prev, live, ids, misses, park, ring, count, work, flags0, lists, det_slot, spawned, dropped};
    const int rc = associate_ok("g6d_instances_associate_host", a, next_id);
    if (rc != G6D_OK) return rc;
    associate_host(a, next_id);
    return G6D_OK;
}

extern "C" int g6d_instances_associate_objects(int S, int K, int M, int F, int r, const float* det, const int* valid, const double* init,
                                               const g6d_glue_camera* cams, const double* centers, double ref_resolution, double gate,
                                               int max_misses, const double* prev, int* live, long long* ids, int* misses,
                                               long long* next_id, double* park, float* ring, int* count, int num, double* work,
                                               uint8_t* flags0, int* lists, int* det_slot, int* spawned, long long* dropped,
                                               g6d_stream_t stream) {
    G6D_REQUIRE(centers, "g6d_instances_associate_objects: null pointer (centers)");
    const assoc::Args a{S, K, M, F, r, num, max_misses, det, valid, init, reinterpret_cast<const double*>(cams), centers, {0., 0., 0.},
                        ref_resolution, gate, prev, live, ids, misses, park, ring, count, work, flags0, lists, det_slot, spawned, dropped};
    return associate_launch("g6d_instances_associate_objects", a, next_id, stream);
}

extern "C" int g6d_instances_associate_objects_host(int S, int K, int M, int F, int r, const float* det, const int* valid,
                                                    const double* init, const g6d_glue_camera* cams, const double* centers,
                                                    double ref_resolution, double gate, int max_misses, const double* prev, int* live,
                                                    long long* ids, int* misses, long long* next_id, double* park, float* ring, int* count,
                                                    int num, double* work, uint8_t* flags0, int* lists, int* det_slot, int* spawned,
                                                    long long* dropped) {
    G6D_REQUIRE(centers, "g6d_instances_associate_objects_host: null pointer (centers)");
    const assoc::Args a{S, K, M, F, r, num, max_misses, det, valid, init, reinterpret_cast<const double*>(cams), centers, {0., 0., 0.},
                        ref_resolution, gate, prev, live, ids, misses, park, ring, count, work, flags0, lists, det_slot, spawned, dropped};
    const int rc = associate_ok("g6d_instances_associate_objects_host", a, next_id);
    if (rc != G6D_OK) return rc;
    associate_host(a, next_id);
    return G6D_OK;
}

// det_index [S] on the host: every entry -1 or a row j < D, no row twice.
static int det_index_ok(const char* name, const int* det_index, int S, int D) {
    G6D_REQUIRE(det_index, "%s: null pointer (det_index)", name);
    G6D_REQUIRE(D >= 0 && D <= S, "%s: need 0 <= D <= S (got D=%d, S=%d)", name, D, S);
    for (int s = 0; s < S; ++s) {
        G6D_REQUIRE(det_index[s] >= -1 && det_index[s] < D, "%s: det_index[%d] = %d is outside [-1, %d)", name, s, det_index[s], D);
        for (int q = 0; q < s; ++q)
            G6D_REQUIRE(det_index[s] < 0 || det_index[q] != det_index[s], "%s: det_index[%d] and det_index[%d] are both %d", name, q, s,
                        det_index[s]);
    }
    return G6D_OK;
}

extern "C" int g6d_instances_associate_sequences(int S, int K, int M, int F, int r, int D, const int* det_index, const float* det,
                                                 const int* valid, const double* init, const g6d_glue_camera* cams, const double* centers,
                                                 double ref_resolution, double gate, int max_misses, const double* prev, int* live,
                                                 long long* ids, int* misses, long long* next_id, double* park, float* ring, int* count,
                                                 int num, double* work, uint8_t* flags0, int* lists, int* det_slot, int* spawned,
                                                 long long* dropped, g6d_stream_t stream) {
    G6D_REQUIRE(centers && det_index, "g6d_instances_associate_sequences: null pointer (centers, det_index)");
    const assoc::Args a{S, K, M, F, r, num, max_misses, det, valid, init, reinterpret_cast<const double*>(cams), centers, {0., 0., 0.},
                        ref_resolution, gate, prev, live, ids, misses, park, ring, count, work, flags0, lists, det_slot, spawned, dropped,
                        det_index, D};
    return associate_launch("g6d_instances_associate_sequences", a, next_id, stream);
}

extern "C" int g6d_instances_associate_sequences_host(int S, int K, int M, int F, int r, int D, const int* det_index, const float* det,
                                                      const int* valid, const double* init, const g6d_glue_camera* cams,
                                                      const double* centers, double ref_resolution, double gate, int max_misses,
                                                      const double* prev, int* live, long long* ids, int* misses, long long* next_id,
                                                      double* park, float* ring, int* count, int num, double* work, uint8_t* flags0,
                                                      int* lists, int* det_slot, int* spawned, long long* dropped) {
    const char* name = "g6d_instances_associate_sequences_host";
    G6D_REQUIRE(centers, "%s: null pointer (centers)", name);
    int rc = det_index_ok(name, det_index, S, D);
    if (rc != G6D_OK) return rc;
    const assoc::Args a{S, K, M, F, r, num, max_misses, det, valid, init, reinterpret_cast<const double*>(cams), centers, {0., 0., 0.},
                        ref_resolution, gate, prev, live, ids, misses, park, ring, count, work, flags0, lists, det_slot, spawned, dropped,
                        det_index, D};
    rc = associate_ok(name, a, next_id);
    if (rc != G6D_OK) return rc;
    associate_host(a, next_id);
    return G6D_OK;
}

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

extern "C" int g6d_instances_verify_update(int n, const int* lost, const int* verified, int max_misses, int* live, long long* ids,
                                           int* misses, long long* dropped, g6d_stream_t stream) {
    const char* name = "g6d_instances_verify_update";
    const int rc = verify_update_ok(name, n, lost, verified, max_misses, live, ids, misses, dropped);
    if (rc != G6D_OK) return rc;
    instances_verify_update_kernel<<<ceil_div(n, 128), 128, 0, as_stream(stream)>>>(n, lost, verified, max_misses, live, ids, misses,
                                                                                     dropped);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}

extern "C" int g6d_instances_verify_update_host(int n, const int* lost, const int* verified, int max_misses, int* live, long long* ids,
                                                int* misses, long long* dropped) {
    const int rc = verify_update_ok("g6d_instances_verify_update_host", n, lost, verified, max_misses, live, ids, misses, dropped);
    if (rc != G6D_OK) return rc;
    for (int i = 0; i < n; ++i) assoc::verify_update(i, lost, verified, max_misses, live, ids, misses, dropped);
    return G6D_OK;
}
