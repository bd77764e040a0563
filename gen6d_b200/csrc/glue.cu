// Device-resident camera algebra between the stages of a batched prediction (see glue_math.cuh): four tiny
// kernels turn detector output into the selector's crop jobs, detector + selector output into the initial poses,
// poses into the refiner's crop jobs + camera tensors, and the refiner's output into the next poses -- so that
// detect -> select -> refine x N is ONE stream-ordered sequence (one CUDA graph) with no host in the loop.
// The *_host entry points run the same functions on host memory (unit tests against geometry.py, no GPU needed).
#include "common.cuh"
#include "glue_math.cuh"

#include <vector>

namespace g6d {
using namespace glue;

G6D_HD void do_detection_job(int i, const float* det_out, const uint8_t* frames, int rows, int cols, int size, g6d_warp_job* jobs) {
    g6d_warp_job j;
    j.src = frames + (long long)i * rows * cols * 3;
    j.rows = rows; j.cols = cols;
    detection_crop_matrix(det_out[i * 4], det_out[i * 4 + 1], det_out[i * 4 + 2], size, j.M);
    jobs[i] = j;
}

G6D_HD void do_initial_pose(int i, const float* det_out, const long long* sel_idx, const float* sel_out, const g6d_glue_refs& r,
                            const g6d_glue_camera* cams, double* poses) {
    const long long k = sel_idx[i];
    pose_from_similarity(det_out[i * 4], det_out[i * 4 + 1], det_out[i * 4 + 2], sel_out[i * 2], r.poses + k * 12, r.cen + k * 2,
                         r.f[k], r.dist[k], cams[i].Kinv, cams[i].f, cams[i].f_sq, r.center, poses + (long long)i * 12);
}

G6D_HD NormParams norm_of(const g6d_glue_views& v) {
    NormParams n;
    n.scale = v.norm_scale;
    n.offset[0] = v.norm_offset[0]; n.offset[1] = v.norm_offset[1]; n.offset[2] = v.norm_offset[2];
    return n;
}

// frame part of one refinement problem: normalise, look at the object, choose the ref_num nearest views
G6D_HD void do_refine_frame(int i, const g6d_glue_views& v, const g6d_glue_camera* cams, const double* poses, int in_f32,
                            FrameProblem& fp, int* chosen /* [ref_num] table rows */) {
    float pose_n[12];
    normalize_pose(poses + (long long)i * 12, in_f32, norm_of(v), pose_n);
    refine_frame(pose_n, cams[i].K, cams[i].Kinv, cams[i].f, v.size, v.size_scale, fp);
    // database_utils.py:125-139: the ref_num views of the FPS subset with the largest cosine to the viewing direction
    for (int r = 0; r < v.ref_num; ++r) {
        int best = -1; float bv = 0.f;
        for (int e = 0; e < v.n_even; ++e) {
            bool used = false;
            for (int q = 0; q < r; ++q) used |= chosen[q] == v.even_idx[e];
            if (used) continue;
            const float* d = v.even_dirs + e * 3;
            const float dot = (d[0] * fp.qdir[0] + d[1] * fp.qdir[1]) + d[2] * fp.qdir[2];
            if (best < 0 || dot > bv) { best = e; bv = dot; }
        }
        chosen[r] = v.even_idx[best];
    }
}

G6D_HD void store_frame(int i, const g6d_glue_views& v, const FrameProblem& fp, const uint8_t* frames, int rows, int cols,
                        g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect) {
    for (int e = 0; e < 9; ++e) que_K[i * 9 + e] = fp.K_warp[e];
    for (int e = 0; e < 12; ++e) { que_pose[i * 12 + e] = fp.pose_warp[e]; rect[i * 12 + e] = fp.rect[e]; }
    g6d_warp_job j;
    j.src = frames + (long long)i * rows * cols * 3;
    j.rows = rows; j.cols = cols;
    inv3_cv(fp.que_H, j.M);
    jobs[(long long)i * (v.ref_num + 1)] = j;
}

G6D_HD void do_refine_view(int i, int r, int row, const g6d_glue_views& v, const double* Rq, g6d_warp_job* jobs, float* ref_Ks,
                           float* ref_poses, int* ref_rows) {
    ViewProblem vp;
    refine_view(Rq, v.poses + (long long)row * 12, v.R_look + (long long)row * 9, v.RlookR + (long long)row * 9, v.f[row],
                v.Kinv + (long long)row * 9, v.size, vp);
    const long long o = (long long)i * v.ref_num + r;
    for (int e = 0; e < 9; ++e) ref_Ks[o * 9 + e] = vp.K[e];
    for (int e = 0; e < 12; ++e) ref_poses[o * 12 + e] = vp.pose[e];
    ref_rows[o] = row;
    g6d_warp_job j;
    j.src = reinterpret_cast<const uint8_t*>(v.src[row]);
    j.rows = v.rows[row]; j.cols = v.cols[row];
    inv3_cv(vp.H, j.M);
    jobs[(long long)i * (v.ref_num + 1) + 1 + r] = j;
}

G6D_HD void do_apply(int i, const g6d_glue_views& v, const float* que_pose, const float* que_K, const float* rect, const float* net_out,
                     double* poses) {
    float p[12];
    apply_refinement(que_pose + i * 12, que_K + i * 9, rect + i * 12, net_out + i * 7, norm_of(v), p);
    for (int e = 0; e < 12; ++e) poses[(long long)i * 12 + e] = (double)p[e];
}

// ------------------------------------------------------------------------------------------ kernels
__global__ void glue_detection_jobs_kernel(const float* det_out, const uint8_t* frames, int rows, int cols, int qn, int size,
                                           g6d_warp_job* jobs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < qn) do_detection_job(i, det_out, frames, rows, cols, size, jobs);
}
__global__ void glue_initial_poses_kernel(const float* det_out, const long long* sel_idx, const float* sel_out, const g6d_glue_refs r,
                                          const g6d_glue_camera* cams, int qn, double* poses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < qn) do_initial_pose(i, det_out, sel_idx, sel_out, r, cams, poses);
}
// one block per frame: thread 0 does the frame part, then one thread per selected view
constexpr int kGlueMaxViews = 8;
__global__ void __launch_bounds__(32) glue_refine_problems_kernel(const g6d_glue_views v, const g6d_glue_camera* cams,
                                                                  const uint8_t* frames, int rows, int cols, const double* poses,
                                                                  int in_f32, g6d_warp_job* jobs, float* que_K, float* que_pose,
                                                                  float* rect, float* ref_Ks, float* ref_poses, int* ref_rows) {
    __shared__ double s_Rq[9];
    __shared__ int s_rows[kGlueMaxViews];
    const int i = blockIdx.x;
    if (threadIdx.x == 0) {
        FrameProblem fp;
        do_refine_frame(i, v, cams, poses, in_f32, fp, s_rows);
        store_frame(i, v, fp, frames, rows, cols, jobs, que_K, que_pose, rect);
        for (int e = 0; e < 9; ++e) s_Rq[e] = fp.Rq[e];
    }
    __syncthreads();
    if ((int)threadIdx.x < v.ref_num) do_refine_view(i, threadIdx.x, s_rows[threadIdx.x], v, s_Rq, jobs, ref_Ks, ref_poses, ref_rows);
}
__global__ void glue_apply_kernel(const g6d_glue_views v, const float* que_pose, const float* que_K, const float* rect,
                                  const float* net_out, int qn, double* poses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < qn) do_apply(i, v, que_pose, que_K, rect, net_out, poses);
}

static bool views_ok(const g6d_glue_views* v) {
    return v && v->poses && v->R_look && v->RlookR && v->f && v->Kinv && v->src && v->rows && v->cols && v->even_idx && v->even_dirs &&
           v->n_views > 0 && v->n_even > 0 && v->ref_num >= 2 && v->ref_num < kGlueMaxViews && v->ref_num <= v->n_even && v->size > 0 &&
           v->norm_scale > 0;
}

// ------------------------------------------------------------------------------------------ several objects
// Rows are object-major: row i = o * rows_per_obj + s is object o on frame s, so it reads views[o], cams[s] and frame s, and
// writes row i of every output (the layout of the per-object calls concatenated).  The per-row functions above get the
// frame's camera and image as row 0 of shifted pointers and the row's outputs at index i, so every row runs the very code
// of the single-object kernels.
struct GlueViewsPack {                 // by value: one kernel parameter block for all objects of a launch
    g6d_glue_views v[G6D_GLUE_MAX_OBJECTS];
};
static_assert(sizeof(GlueViewsPack) + 256 <= 4096, "the objects' view structs must fit the 4 KB kernel parameter space");

// the frame part of input row `row` (frame s), written to output row j
G6D_HD void do_refine_frame_row(int j, int row, int s, const g6d_glue_views& v, const g6d_glue_camera* cams, const uint8_t* frames,
                                int rows, int cols, const double* poses, int in_f32, g6d_warp_job* jobs, float* que_K,
                                float* que_pose, float* rect, FrameProblem& fp, int* chosen) {
    do_refine_frame(0, v, cams + s, poses + (long long)row * 12, in_f32, fp, chosen);
    store_frame(0, v, fp, frames + (long long)s * rows * cols * 3, rows, cols, jobs + (long long)j * (v.ref_num + 1), que_K + (long long)j * 9,
                que_pose + (long long)j * 12, rect + (long long)j * 12);
}
G6D_HD void do_refine_frame_objects(int i, int s, const g6d_glue_views& v, const g6d_glue_camera* cams, const uint8_t* frames,
                                    int rows, int cols, const double* poses, int in_f32, g6d_warp_job* jobs, float* que_K,
                                    float* que_pose, float* rect, FrameProblem& fp, int* chosen) {
    do_refine_frame_row(i, i, s, v, cams, frames, rows, cols, poses, in_f32, jobs, que_K, que_pose, rect, fp, chosen);
}

__global__ void __launch_bounds__(32) glue_refine_problems_objects_kernel(const GlueViewsPack pk, int rows_per_obj,
                                                                          const g6d_glue_camera* cams, const uint8_t* frames, int rows,
                                                                          int cols, const double* poses, int in_f32, g6d_warp_job* jobs,
                                                                          float* que_K, float* que_pose, float* rect, float* ref_Ks,
                                                                          float* ref_poses, int* ref_rows) {
    __shared__ double s_Rq[9];
    __shared__ int s_rows[kGlueMaxViews];
    const int i = blockIdx.x;
    const g6d_glue_views v = pk.v[i / rows_per_obj];
    if (threadIdx.x == 0) {
        FrameProblem fp;
        do_refine_frame_objects(i, i % rows_per_obj, v, cams, frames, rows, cols, poses, in_f32, jobs, que_K, que_pose, rect, fp, s_rows);
        for (int e = 0; e < 9; ++e) s_Rq[e] = fp.Rq[e];
    }
    __syncthreads();
    if ((int)threadIdx.x < v.ref_num) do_refine_view(i, threadIdx.x, s_rows[threadIdx.x], v, s_Rq, jobs, ref_Ks, ref_poses, ref_rows);
}
__global__ void glue_apply_objects_kernel(const GlueViewsPack pk, int rows_per_obj, const float* que_pose, const float* que_K,
                                          const float* rect, const float* net_out, int qn, double* poses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < qn) do_apply(i, pk.v[i / rows_per_obj], que_pose, que_K, rect, net_out, poses);
}

// ------------------------------------------------------------------------------------------ a subset of the rows
// Output row j is input row row_idx[j] (object-major numbering as above): the problem is built from poses[row_idx[j]] with
// that row's own dtype flag row_f32[row_idx[j]], and the update of output row j goes back to poses[row_idx[j]].  Rows that
// are not listed are neither read nor written, so a tracker refines exactly the rows whose chain is still running.
G6D_HD void do_refine_frame_rows(int j, const GlueViewsPack& pk, int rows_per_obj, const int* row_idx, const uint8_t* row_f32,
                                 const g6d_glue_camera* cams, const uint8_t* frames, int rows, int cols, const double* poses,
                                 g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect, FrameProblem& fp, int* chosen) {
    const int row = row_idx[j];
    do_refine_frame_row(j, row, row % rows_per_obj, pk.v[row / rows_per_obj], cams, frames, rows, cols, poses, row_f32[row], jobs, que_K,
                        que_pose, rect, fp, chosen);
}
G6D_HD void do_apply_rows(int j, const GlueViewsPack& pk, int rows_per_obj, const int* row_idx, const float* que_pose, const float* que_K,
                          const float* rect, const float* net_out, double* poses) {
    const int row = row_idx[j];
    do_apply(0, pk.v[row / rows_per_obj], que_pose + (long long)j * 12, que_K + (long long)j * 9, rect + (long long)j * 12,
             net_out + (long long)j * 7, poses + (long long)row * 12);
}

__global__ void __launch_bounds__(32) glue_refine_problems_rows_kernel(const GlueViewsPack pk, int rows_per_obj, const g6d_glue_camera* cams,
                                                                       const uint8_t* frames, int rows, int cols, const double* poses,
                                                                       const int* row_idx, const uint8_t* row_f32, g6d_warp_job* jobs,
                                                                       float* que_K, float* que_pose, float* rect, float* ref_Ks,
                                                                       float* ref_poses, int* ref_rows) {
    __shared__ double s_Rq[9];
    __shared__ int s_rows[kGlueMaxViews];
    const int j = blockIdx.x;
    const g6d_glue_views& v = pk.v[row_idx[j] / rows_per_obj];
    if (threadIdx.x == 0) {
        FrameProblem fp;
        do_refine_frame_rows(j, pk, rows_per_obj, row_idx, row_f32, cams, frames, rows, cols, poses, jobs, que_K, que_pose, rect, fp, s_rows);
        for (int e = 0; e < 9; ++e) s_Rq[e] = fp.Rq[e];
    }
    __syncthreads();
    if ((int)threadIdx.x < v.ref_num) do_refine_view(j, threadIdx.x, s_rows[threadIdx.x], v, s_Rq, jobs, ref_Ks, ref_poses, ref_rows);
}
__global__ void glue_apply_rows_kernel(const GlueViewsPack pk, int rows_per_obj, const float* que_pose, const float* que_K,
                                       const float* rect, const float* net_out, const int* row_idx, int n_sel, double* poses) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_sel) do_apply_rows(j, pk, rows_per_obj, row_idx, que_pose, que_K, rect, net_out, poses);
}

// host checks shared by the device and host entry points; also fills the parameter block
static int objects_ok(const char* name, const g6d_glue_views* views, int n_obj, int rows_per_obj, bool full, GlueViewsPack* pk) {
    G6D_REQUIRE(views, "%s: null views", name);
    G6D_REQUIRE(n_obj >= 1 && n_obj <= G6D_GLUE_MAX_OBJECTS, "%s: need 1 <= n_obj <= %d (got n_obj=%d)", name, G6D_GLUE_MAX_OBJECTS, n_obj);
    G6D_REQUIRE(rows_per_obj >= 1, "%s: need rows_per_obj >= 1 (got %d)", name, rows_per_obj);
    for (int o = 0; o < n_obj; ++o) {
        if (full) {
            G6D_REQUIRE(views_ok(views + o), "%s: incomplete view tables of object %d (2 <= ref_num < %d)", name, o, kGlueMaxViews);
            G6D_REQUIRE(views[o].ref_num == views[0].ref_num, "%s: object %d has ref_num %d, object 0 has %d; all objects need the same",
                        name, o, views[o].ref_num, views[0].ref_num);
        } else {
            G6D_REQUIRE(views[o].norm_scale > 0, "%s: object %d has no normalisation (norm_scale <= 0)", name, o);
        }
        pk->v[o] = views[o];
    }
    return G6D_OK;
}

}  // namespace g6d

using namespace g6d;

extern "C" int g6d_glue_detection_jobs(const float* det_out, const uint8_t* frames, int rows, int cols, int qn, int size,
                                       g6d_warp_job* jobs, g6d_stream_t stream) {
    G6D_REQUIRE(det_out && frames && jobs && qn > 0 && rows > 0 && cols > 0 && size > 0, "g6d_glue_detection_jobs: bad args");
    glue_detection_jobs_kernel<<<ceil_div(qn, 32), 32, 0, as_stream(stream)>>>(det_out, frames, rows, cols, qn, size, jobs);
    G6D_CHECK_LAUNCH("g6d_glue_detection_jobs");
    return G6D_OK;
}
extern "C" int g6d_glue_detection_jobs_host(const float* det_out, const uint8_t* frames, int rows, int cols, int qn, int size,
                                            g6d_warp_job* jobs) {
    G6D_REQUIRE(det_out && jobs && qn > 0, "g6d_glue_detection_jobs_host: bad args");
    for (int i = 0; i < qn; ++i) do_detection_job(i, det_out, frames, rows, cols, size, jobs);
    return G6D_OK;
}

extern "C" int g6d_glue_initial_poses(const float* det_out, const long long* sel_idx, const float* sel_out, const g6d_glue_refs* refs,
                                      const g6d_glue_camera* cams, int qn, double* poses, g6d_stream_t stream) {
    G6D_REQUIRE(det_out && sel_idx && sel_out && refs && refs->poses && refs->cen && refs->f && refs->dist && cams && poses && qn > 0,
                "g6d_glue_initial_poses: bad args");
    glue_initial_poses_kernel<<<ceil_div(qn, 32), 32, 0, as_stream(stream)>>>(det_out, sel_idx, sel_out, *refs, cams, qn, poses);
    G6D_CHECK_LAUNCH("g6d_glue_initial_poses");
    return G6D_OK;
}
extern "C" int g6d_glue_initial_poses_host(const float* det_out, const long long* sel_idx, const float* sel_out, const g6d_glue_refs* refs,
                                           const g6d_glue_camera* cams, int qn, double* poses) {
    G6D_REQUIRE(det_out && sel_idx && sel_out && refs && cams && poses && qn > 0, "g6d_glue_initial_poses_host: bad args");
    for (int i = 0; i < qn; ++i) do_initial_pose(i, det_out, sel_idx, sel_out, *refs, cams, poses);
    return G6D_OK;
}

extern "C" int g6d_glue_refine_problems(const g6d_glue_views* views, const g6d_glue_camera* cams, const uint8_t* frames, int rows,
                                        int cols, const double* poses, int poses_are_f32, int qn, g6d_warp_job* jobs, float* que_K,
                                        float* que_pose, float* rect, float* ref_Ks, float* ref_poses, int* ref_rows,
                                        g6d_stream_t stream) {
    G6D_REQUIRE(views_ok(views), "g6d_glue_refine_problems: incomplete view tables (2 <= ref_num < %d)", kGlueMaxViews);
    G6D_REQUIRE(cams && frames && poses && jobs && que_K && que_pose && rect && ref_Ks && ref_poses && ref_rows && qn > 0 && rows > 0 &&
                    cols > 0, "g6d_glue_refine_problems: bad args");
    glue_refine_problems_kernel<<<qn, 32, 0, as_stream(stream)>>>(*views, cams, frames, rows, cols, poses, poses_are_f32, jobs, que_K,
                                                                  que_pose, rect, ref_Ks, ref_poses, ref_rows);
    G6D_CHECK_LAUNCH("g6d_glue_refine_problems");
    return G6D_OK;
}
extern "C" int g6d_glue_refine_problems_host(const g6d_glue_views* views, const g6d_glue_camera* cams, const uint8_t* frames, int rows,
                                             int cols, const double* poses, int poses_are_f32, int qn, g6d_warp_job* jobs, float* que_K,
                                             float* que_pose, float* rect, float* ref_Ks, float* ref_poses, int* ref_rows) {
    G6D_REQUIRE(views_ok(views), "g6d_glue_refine_problems_host: incomplete view tables");
    G6D_REQUIRE(cams && poses && jobs && que_K && que_pose && rect && ref_Ks && ref_poses && ref_rows && qn > 0, "g6d_glue_refine_problems_host: bad args");
    for (int i = 0; i < qn; ++i) {
        FrameProblem fp;
        int chosen[kGlueMaxViews];
        do_refine_frame(i, *views, cams, poses, poses_are_f32, fp, chosen);
        store_frame(i, *views, fp, frames, rows, cols, jobs, que_K, que_pose, rect);
        for (int r = 0; r < views->ref_num; ++r) do_refine_view(i, r, chosen[r], *views, fp.Rq, jobs, ref_Ks, ref_poses, ref_rows);
    }
    return G6D_OK;
}

extern "C" int g6d_glue_apply_refinements(const g6d_glue_views* views, const float* que_pose, const float* que_K, const float* rect,
                                          const float* net_out, int qn, double* poses, g6d_stream_t stream) {
    G6D_REQUIRE(views && views->norm_scale > 0 && que_pose && que_K && rect && net_out && poses && qn > 0, "g6d_glue_apply_refinements: bad args");
    glue_apply_kernel<<<ceil_div(qn, 32), 32, 0, as_stream(stream)>>>(*views, que_pose, que_K, rect, net_out, qn, poses);
    G6D_CHECK_LAUNCH("g6d_glue_apply_refinements");
    return G6D_OK;
}
extern "C" int g6d_glue_apply_refinements_host(const g6d_glue_views* views, const float* que_pose, const float* que_K, const float* rect,
                                               const float* net_out, int qn, double* poses) {
    G6D_REQUIRE(views && views->norm_scale > 0 && que_pose && que_K && rect && net_out && poses && qn > 0, "g6d_glue_apply_refinements_host: bad args");
    for (int i = 0; i < qn; ++i) do_apply(i, *views, que_pose, que_K, rect, net_out, poses);
    return G6D_OK;
}

extern "C" int g6d_glue_refine_problems_objects(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                                const uint8_t* frames, int rows, int cols, const double* poses, int poses_are_f32,
                                                g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect, float* ref_Ks,
                                                float* ref_poses, int* ref_rows, g6d_stream_t stream) {
    const char* name = "g6d_glue_refine_problems_objects";
    GlueViewsPack pk;
    const int rc = objects_ok(name, views, n_obj, rows_per_obj, true, &pk);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(cams && frames && poses && jobs && que_K && que_pose && rect && ref_Ks && ref_poses && ref_rows && rows > 0 && cols > 0,
                "%s: bad args", name);
    glue_refine_problems_objects_kernel<<<n_obj * rows_per_obj, 32, 0, as_stream(stream)>>>(
        pk, rows_per_obj, cams, frames, rows, cols, poses, poses_are_f32, jobs, que_K, que_pose, rect, ref_Ks, ref_poses, ref_rows);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}
extern "C" int g6d_glue_refine_problems_objects_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                                     const uint8_t* frames, int rows, int cols, const double* poses, int poses_are_f32,
                                                     g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect, float* ref_Ks,
                                                     float* ref_poses, int* ref_rows) {
    const char* name = "g6d_glue_refine_problems_objects_host";
    GlueViewsPack pk;
    const int rc = objects_ok(name, views, n_obj, rows_per_obj, true, &pk);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(cams && poses && jobs && que_K && que_pose && rect && ref_Ks && ref_poses && ref_rows, "%s: bad args", name);
    for (int i = 0; i < n_obj * rows_per_obj; ++i) {
        const g6d_glue_views& v = pk.v[i / rows_per_obj];
        FrameProblem fp;
        int chosen[kGlueMaxViews];
        do_refine_frame_objects(i, i % rows_per_obj, v, cams, frames, rows, cols, poses, poses_are_f32, jobs, que_K, que_pose, rect, fp,
                                chosen);
        for (int r = 0; r < v.ref_num; ++r) do_refine_view(i, r, chosen[r], v, fp.Rq, jobs, ref_Ks, ref_poses, ref_rows);
    }
    return G6D_OK;
}

extern "C" int g6d_glue_apply_refinements_objects(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                                  const float* que_K, const float* rect, const float* net_out, double* poses,
                                                  g6d_stream_t stream) {
    const char* name = "g6d_glue_apply_refinements_objects";
    GlueViewsPack pk;
    const int rc = objects_ok(name, views, n_obj, rows_per_obj, false, &pk);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(que_pose && que_K && rect && net_out && poses, "%s: bad args", name);
    const int qn = n_obj * rows_per_obj;
    glue_apply_objects_kernel<<<ceil_div(qn, 32), 32, 0, as_stream(stream)>>>(pk, rows_per_obj, que_pose, que_K, rect, net_out, qn, poses);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}
extern "C" int g6d_glue_apply_refinements_objects_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                                       const float* que_K, const float* rect, const float* net_out, double* poses) {
    const char* name = "g6d_glue_apply_refinements_objects_host";
    GlueViewsPack pk;
    const int rc = objects_ok(name, views, n_obj, rows_per_obj, false, &pk);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(que_pose && que_K && rect && net_out && poses, "%s: bad args", name);
    for (int i = 0; i < n_obj * rows_per_obj; ++i) do_apply(i, pk.v[i / rows_per_obj], que_pose, que_K, rect, net_out, poses);
    return G6D_OK;
}

// check_idx (host twins): every index in range and, for the updates (unique), no row listed twice
static int rows_ok(const char* name, int n_obj, int rows_per_obj, const int* row_idx, int n_sel, bool check_idx, bool unique) {
    G6D_REQUIRE(row_idx && n_sel >= 1, "%s: need a row list and n_sel >= 1 (got n_sel=%d)", name, n_sel);
    if (check_idx) {
        const long long n = (long long)n_obj * rows_per_obj;
        std::vector<unsigned char> seen(unique ? n : 0, 0);
        for (int j = 0; j < n_sel; ++j) {
            G6D_REQUIRE(row_idx[j] >= 0 && row_idx[j] < n, "%s: row_idx[%d] = %d is outside [0, %lld)", name, j, row_idx[j], n);
            if (unique) {
                G6D_REQUIRE(!seen[row_idx[j]], "%s: row %d is listed twice (each row takes one update)", name, row_idx[j]);
                seen[row_idx[j]] = 1;
            }
        }
    }
    return G6D_OK;
}

extern "C" int g6d_glue_refine_problems_rows(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                             const uint8_t* frames, int rows, int cols, const double* poses, const int* row_idx, int n_sel,
                                             const uint8_t* row_f32, g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect,
                                             float* ref_Ks, float* ref_poses, int* ref_rows, g6d_stream_t stream) {
    const char* name = "g6d_glue_refine_problems_rows";
    GlueViewsPack pk;
    int rc = objects_ok(name, views, n_obj, rows_per_obj, true, &pk);
    if (rc == G6D_OK) rc = rows_ok(name, n_obj, rows_per_obj, row_idx, n_sel, false, false);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(cams && frames && poses && row_f32 && jobs && que_K && que_pose && rect && ref_Ks && ref_poses && ref_rows && rows > 0 &&
                    cols > 0, "%s: bad args", name);
    glue_refine_problems_rows_kernel<<<n_sel, 32, 0, as_stream(stream)>>>(pk, rows_per_obj, cams, frames, rows, cols, poses, row_idx, row_f32,
                                                                          jobs, que_K, que_pose, rect, ref_Ks, ref_poses, ref_rows);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}
extern "C" int g6d_glue_refine_problems_rows_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                                  const uint8_t* frames, int rows, int cols, const double* poses, const int* row_idx,
                                                  int n_sel, const uint8_t* row_f32, g6d_warp_job* jobs, float* que_K, float* que_pose,
                                                  float* rect, float* ref_Ks, float* ref_poses, int* ref_rows) {
    const char* name = "g6d_glue_refine_problems_rows_host";
    GlueViewsPack pk;
    int rc = objects_ok(name, views, n_obj, rows_per_obj, true, &pk);
    if (rc == G6D_OK) rc = rows_ok(name, n_obj, rows_per_obj, row_idx, n_sel, true, false);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(cams && poses && row_f32 && jobs && que_K && que_pose && rect && ref_Ks && ref_poses && ref_rows, "%s: bad args", name);
    for (int j = 0; j < n_sel; ++j) {
        const g6d_glue_views& v = pk.v[row_idx[j] / rows_per_obj];
        FrameProblem fp;
        int chosen[kGlueMaxViews];
        do_refine_frame_rows(j, pk, rows_per_obj, row_idx, row_f32, cams, frames, rows, cols, poses, jobs, que_K, que_pose, rect, fp, chosen);
        for (int r = 0; r < v.ref_num; ++r) do_refine_view(j, r, chosen[r], v, fp.Rq, jobs, ref_Ks, ref_poses, ref_rows);
    }
    return G6D_OK;
}

extern "C" int g6d_glue_apply_refinements_rows(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                               const float* que_K, const float* rect, const float* net_out, const int* row_idx, int n_sel,
                                               double* poses, g6d_stream_t stream) {
    const char* name = "g6d_glue_apply_refinements_rows";
    GlueViewsPack pk;
    int rc = objects_ok(name, views, n_obj, rows_per_obj, false, &pk);
    if (rc == G6D_OK) rc = rows_ok(name, n_obj, rows_per_obj, row_idx, n_sel, false, false);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(que_pose && que_K && rect && net_out && poses, "%s: bad args", name);
    glue_apply_rows_kernel<<<ceil_div(n_sel, 32), 32, 0, as_stream(stream)>>>(pk, rows_per_obj, que_pose, que_K, rect, net_out, row_idx,
                                                                              n_sel, poses);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}
extern "C" int g6d_glue_apply_refinements_rows_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                                    const float* que_K, const float* rect, const float* net_out, const int* row_idx,
                                                    int n_sel, double* poses) {
    const char* name = "g6d_glue_apply_refinements_rows_host";
    GlueViewsPack pk;
    int rc = objects_ok(name, views, n_obj, rows_per_obj, false, &pk);
    if (rc == G6D_OK) rc = rows_ok(name, n_obj, rows_per_obj, row_idx, n_sel, true, true);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(que_pose && que_K && rect && net_out && poses, "%s: bad args", name);
    for (int j = 0; j < n_sel; ++j) do_apply_rows(j, pk, rows_per_obj, row_idx, que_pose, que_K, rect, net_out, poses);
    return G6D_OK;
}

// ------------------------------------------------------------------------------------------ verification windows
namespace g6d {
struct GlueRefsPack {                  // by value: the objects' selector references of one launch
    g6d_glue_refs r[G6D_GLUE_MAX_OBJECTS];
};

// row i = o * rows_per_obj + s: object o's pose on frame s
G6D_HD void do_verify_window(int i, const GlueRefsPack& pk, int rows_per_obj, const g6d_glue_camera* cams, const double* poses,
                             int in_f32, float* rec) {
    const g6d_glue_refs& r = pk.r[i / rows_per_obj];
    const g6d_glue_camera& c = cams[i % rows_per_obj];
    window_from_pose(poses + (long long)i * 12, in_f32, r.center, c.K, c.Kinv, c.f, c.f_sq, r.dist[0], r.f[0], rec + (long long)i * 4);
}

__global__ void verify_windows_kernel(const GlueRefsPack pk, int rows_per_obj, const g6d_glue_camera* cams, const double* poses,
                                      int in_f32, int n, float* rec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) do_verify_window(i, pk, rows_per_obj, cams, poses, in_f32, rec);
}

__global__ void verify_judge_kernel(const float* rec, const float* det, int n, int window, double ref_resolution, int use_score,
                                    double lost_score, int use_gate, double lost_gate, float* out, int* lost) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        lost[i] = verify_judge(rec + i * 4, det + i * 4, window, ref_resolution, use_score, lost_score, use_gate, lost_gate, out + i * 5);
}

static int verify_refs_ok(const char* name, const g6d_glue_refs* refs, int n_obj, int rows_per_obj, GlueRefsPack* pk) {
    G6D_REQUIRE(refs, "%s: null refs", name);
    G6D_REQUIRE(n_obj >= 1 && n_obj <= G6D_GLUE_MAX_OBJECTS, "%s: need 1 <= n_obj <= %d (got n_obj=%d)", name, G6D_GLUE_MAX_OBJECTS, n_obj);
    G6D_REQUIRE(rows_per_obj >= 1, "%s: need rows_per_obj >= 1 (got %d)", name, rows_per_obj);
    for (int o = 0; o < n_obj; ++o) {
        G6D_REQUIRE(refs[o].f && refs[o].dist, "%s: object %d has no reference distances (f, dist)", name, o);
        pk->r[o] = refs[o];
    }
    return G6D_OK;
}

static int judge_ok(const char* name, const float* rec, const float* det, int n, int window, double ref_resolution, int use_score,
                    double lost_score, int use_gate, double lost_gate, const float* out, const int* lost) {
    G6D_REQUIRE(rec && det && out && lost && n >= 1, "%s: bad args", name);
    G6D_REQUIRE(window > 0 && ref_resolution > 0, "%s: need window > 0 and ref_resolution > 0 (got %d, %g)", name, window, ref_resolution);
    G6D_REQUIRE(!use_score || lost_score == lost_score, "%s: lost_score is NaN", name);
    G6D_REQUIRE(!use_gate || lost_gate == lost_gate, "%s: lost_gate is NaN", name);
    return G6D_OK;
}
}  // namespace g6d

extern "C" int g6d_verify_windows(const double* poses, int poses_are_f32, const g6d_glue_refs* refs, int n_obj, int rows_per_obj,
                                  const g6d_glue_camera* cams, float* rec, g6d_stream_t stream) {
    const char* name = "g6d_verify_windows";
    GlueRefsPack pk;
    const int rc = verify_refs_ok(name, refs, n_obj, rows_per_obj, &pk);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(poses && cams && rec, "%s: bad args", name);
    const int n = n_obj * rows_per_obj;
    verify_windows_kernel<<<ceil_div(n, 32), 32, 0, as_stream(stream)>>>(pk, rows_per_obj, cams, poses, poses_are_f32, n, rec);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}
extern "C" int g6d_verify_windows_host(const double* poses, int poses_are_f32, const g6d_glue_refs* refs, int n_obj, int rows_per_obj,
                                       const g6d_glue_camera* cams, float* rec) {
    const char* name = "g6d_verify_windows_host";
    GlueRefsPack pk;
    const int rc = verify_refs_ok(name, refs, n_obj, rows_per_obj, &pk);
    if (rc != G6D_OK) return rc;
    G6D_REQUIRE(poses && cams && rec, "%s: bad args", name);
    for (int i = 0; i < n_obj * rows_per_obj; ++i) do_verify_window(i, pk, rows_per_obj, cams, poses, poses_are_f32, rec);
    return G6D_OK;
}

extern "C" int g6d_verify_judge(const float* rec, const float* det, int n, int window, double ref_resolution, int use_score,
                                double lost_score, int use_gate, double lost_gate, float* out, int* lost, g6d_stream_t stream) {
    const char* name = "g6d_verify_judge";
    const int rc = judge_ok(name, rec, det, n, window, ref_resolution, use_score, lost_score, use_gate, lost_gate, out, lost);
    if (rc != G6D_OK) return rc;
    verify_judge_kernel<<<ceil_div(n, 32), 32, 0, as_stream(stream)>>>(rec, det, n, window, ref_resolution, use_score, lost_score,
                                                                         use_gate, lost_gate, out, lost);
    G6D_CHECK_LAUNCH(name);
    return G6D_OK;
}
extern "C" int g6d_verify_judge_host(const float* rec, const float* det, int n, int window, double ref_resolution, int use_score,
                                     double lost_score, int use_gate, double lost_gate, float* out, int* lost) {
    const char* name = "g6d_verify_judge_host";
    const int rc = judge_ok(name, rec, det, n, window, ref_resolution, use_score, lost_score, use_gate, lost_gate, out, lost);
    if (rc != G6D_OK) return rc;
    for (int i = 0; i < n; ++i)
        lost[i] = verify_judge(rec + i * 4, det + i * 4, window, ref_resolution, use_score, lost_score, use_gate, lost_gate, out + i * 5);
    return G6D_OK;
}
