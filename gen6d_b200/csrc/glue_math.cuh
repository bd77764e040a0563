// Camera algebra between the stages of a prediction (estimator.py:176-214 of the reference; the numpy
// restatement is gen6d_b200/geometry.py: crop_similarity / poses_from_similarity / refine_problems /
// apply_refinements), as __host__ __device__ functions: the device kernels of glue.cu keep a whole batch
// prediction on the GPU (no device -> host -> device round trip between detect, select and the refinement
// iterations), and the *_host entry points run the very same code on the CPU so that the unit tests can pin it
// against geometry.py without a GPU.  Every step mirrors the dtype of the numpy expression it replaces
// (float32 where numpy computes in float32, rounding to float32 where numpy stores into a float32 array).
// This translation unit is compiled with -fmad=false: products and sums round separately, like numpy's.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/gen6d_b200.h"

#if defined(__CUDACC__)
#define G6D_HD __host__ __device__ inline
#else
#define G6D_HD inline
#endif

namespace g6d {
namespace glue {

// ------------------------------------------------------------------------------------------ 3x3 helpers (row-major)
G6D_HD void mat3_mul(const double* a, const double* b, double* c) {          // c = a @ b
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
}
G6D_HD void mat3_mul_bt(const double* a, const double* b, double* c) {       // c = a @ b^T
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i * 3 + j] = a[i * 3] * b[j * 3] + a[i * 3 + 1] * b[j * 3 + 1] + a[i * 3 + 2] * b[j * 3 + 2];
}
G6D_HD void mat3_at_mul(const double* a, const double* b, double* c) {       // c = a^T @ b
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i * 3 + j] = a[i] * b[j] + a[3 + i] * b[3 + j] + a[6 + i] * b[6 + j];
}
G6D_HD void mat3_vec(const double* a, const double* v, double* o) {
    for (int i = 0; i < 3; ++i) o[i] = a[i * 3] * v[0] + a[i * 3 + 1] * v[1] + a[i * 3 + 2] * v[2];
}
// cv::invert of a 3x3 in double (DECOMP_LU takes the closed form for n <= 3; modules/core/src/lapack.cpp)
G6D_HD void inv3_cv(const double* s, double* t) {
    double d = s[0] * (s[4] * s[8] - s[5] * s[7]) - s[1] * (s[3] * s[8] - s[5] * s[6]) + s[2] * (s[3] * s[7] - s[4] * s[6]);
    if (d == 0.) { for (int i = 0; i < 9; ++i) t[i] = 0.; return; }
    d = 1. / d;
    t[0] = (s[4] * s[8] - s[5] * s[7]) * d; t[1] = (s[2] * s[7] - s[1] * s[8]) * d; t[2] = (s[1] * s[5] - s[2] * s[4]) * d;
    t[3] = (s[5] * s[6] - s[3] * s[8]) * d; t[4] = (s[0] * s[8] - s[2] * s[6]) * d; t[5] = (s[2] * s[3] - s[0] * s[5]) * d;
    t[6] = (s[3] * s[7] - s[4] * s[6]) * d; t[7] = (s[1] * s[6] - s[0] * s[7]) * d; t[8] = (s[0] * s[4] - s[1] * s[3]) * d;
}
// geometry._look_at_batch for one view: rotation that centres pixel (px, py); f = (K00 + K11) / 2 evaluated by the
// caller in K's own dtype; (cx, cy) = K[:2, 2]
G6D_HD void look_at(double px, double py, double f, double cx, double cy, double* R, double* f_ray) {
    const double c0 = px - cx, c1 = py - cy;
    const double a = -atan2(c0 / f, 1.0), b = atan2(c1 / f, 1.0);
    const double ca = cos(a), sa = sin(a), cb = cos(b), sb = sin(b);
    R[0] = ca; R[1] = 0.; R[2] = sa;
    R[3] = sb * sa; R[4] = cb; R[5] = -(sb * ca);
    R[6] = -(cb * sa); R[7] = sb; R[8] = cb * ca;
    if (f_ray) *f_ray = sqrt((c0 * c0 + c1 * c1) + f * f);
}
// geometry._project_center_batch for one camera: pixel of `center` under pose [3,4] (row-major) and K
G6D_HD void project_center(const double* center, const double* pose, const double* K, double* px, double* py) {
    double p[3], q[3];
    for (int i = 0; i < 3; ++i) p[i] = (pose[i * 4] * center[0] + pose[i * 4 + 1] * center[1] + pose[i * 4 + 2] * center[2]) + pose[i * 4 + 3];
    mat3_vec(K, p, q);
    double d = q[2];
    if (fabs(d) < 1e-4 && fabs(d) > 0) d = 1e-4;
    *px = q[0] / d; *py = q[1] / d;
}

// ------------------------------------------------------------------------------------------ A: detection -> crop job
// geometry.crop_similarity (float32 2x3, angle 0) followed by geometry.affine_dst_to_src (OpenCV's closed form in
// double): the dst -> src matrix of the selector's detection crop.  M9[6..8] = 0, 0, 1.
G6D_HD void detection_crop_matrix(float px, float py, float scale_r2q, int size, double* M9) {
    const float s = 1.0f / scale_r2q;
    const float half = (float)size / 2;
    float m[6] = {s, 0.f, s * -px + half, 0.f, s, s * -py + half};
    double d[6];
    for (int i = 0; i < 6; ++i) d[i] = (double)m[i];
    double D = d[0] * d[4] - d[1] * d[3];
    D = D != 0. ? 1.0 / D : 0.;
    const double a11 = d[4] * D, a22 = d[0] * D;
    d[0] = a11; d[1] = d[1] * -D; d[3] = d[3] * -D; d[4] = a22;
    const double b1 = -d[0] * d[2] - d[1] * d[5];
    const double b2 = -d[3] * d[2] - d[4] * d[5];
    d[2] = b1; d[5] = b2;
    for (int i = 0; i < 6; ++i) M9[i] = d[i];
    M9[6] = 0.; M9[7] = 0.; M9[8] = 1.;
}

// ------------------------------------------------------------------------------------------ B: pose from similarity
// geometry.poses_from_similarity for one detection.  Per-reference constants come from a table computed with numpy
// at build time (ref_cen = projected object centre, ref_f = (K00 + K11) / 2, ref_dist = |camera - centre|), per-frame
// camera constants from the caller (Kinv = np.linalg.inv(que_K) as float64 values, que_f).
G6D_HD void pose_from_similarity(float pos_x, float pos_y, float scale_r2q, float angle_r2q, const double* ref_pose,
                                 const double* ref_cen, double ref_f, double ref_dist, const double* que_Kinv, double que_f,
                                 double que_f_sq, const double* center, double* pose_out /* [12] */) {
    const float sc = 1.0f / scale_r2q, ang = -angle_r2q;
    // numpy evaluates cos / sin of a float32 angle in float32 (correctly rounded here)
    const float c = (float)cos((double)ang), s = (float)sin((double)ang);
    double M[9] = {(double)(sc * c), (double)(sc * -s), 0., (double)(sc * s), (double)(sc * c), 0., 0., 0., 1.};
    M[2] = ref_cen[0] - (M[0] * (double)pos_x + M[1] * (double)pos_y);
    M[5] = ref_cen[1] - (M[3] * (double)pos_x + M[4] * (double)pos_y);
    double Mi[9];
    inv3_cv(M, Mi);                                                    // np.linalg.inv (LAPACK) to ~1e-16
    const double qx = (Mi[0] * ref_cen[0] + Mi[1] * ref_cen[1]) + Mi[2], qy = (Mi[3] * ref_cen[0] + Mi[4] * ref_cen[1]) + Mi[5];
    const double v[3] = {qx, qy, 1.0};
    double bearing[3];
    mat3_vec(que_Kinv, v, bearing);
    const double bx = bearing[0] / bearing[2], by = bearing[1] / bearing[2];
    const double scale = sqrt(Mi[0] * Mi[4] - Mi[1] * Mi[3]);
    const double rotation = atan2(Mi[3], Mi[0]);
    const double n2 = sqrt((bx * que_f) * (bx * que_f) + (by * que_f) * (by * que_f));
    const double que_f_ray = sqrt(que_f_sq + n2 * n2);
    const double que_dist = ref_dist * que_f_ray / ref_f / scale;
    const double rn = sqrt((bx * bx + by * by) + 1.0);
    const double cen3d[3] = {bx / rn * que_dist, by / rn * que_dist, 1.0 / rn * que_dist};
    double R_look[9];
    look_at(bx, by, 1.0, 0.0, 0.0, R_look, nullptr);
    const double cr = cos(rotation), sr = sin(rotation);
    const double Rz[9] = {cr, -sr, 0., sr, cr, 0., 0., 0., 1.};
    double Rref[9], T[9], R[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rref[i * 3 + j] = ref_pose[i * 4 + j];
    mat3_mul(Rz, Rref, T);
    mat3_at_mul(R_look, T, R);
    double Rc[3];
    mat3_vec(R, center, Rc);
    for (int i = 0; i < 3; ++i) {
        pose_out[i * 4] = R[i * 3]; pose_out[i * 4 + 1] = R[i * 3 + 1]; pose_out[i * 4 + 2] = R[i * 3 + 2];
        pose_out[i * 4 + 3] = cen3d[i] - Rc[i];
    }
}

// ------------------------------------------------------------------------------------------ C: refinement problem
struct NormParams {              // geometry.NormalizedView: scale (double) and offset (float32 values)
    double scale;
    float offset[3];
};
// NormalizedView.normalize_poses for one pose.  in_f32: the pose is a float32 array (every pose after the first
// refinement) and numpy computes R @ -offset + scale * t in float32; else in float64, rounded once.
G6D_HD void normalize_pose(const double* pose, int in_f32, const NormParams& np_, float* out /* [12] */) {
    for (int i = 0; i < 3; ++i) {
        if (in_f32) {
            const float r0 = (float)pose[i * 4], r1 = (float)pose[i * 4 + 1], r2 = (float)pose[i * 4 + 2], t = (float)pose[i * 4 + 3];
            out[i * 4] = r0; out[i * 4 + 1] = r1; out[i * 4 + 2] = r2;
            out[i * 4 + 3] = ((r0 * -np_.offset[0] + r1 * -np_.offset[1]) + r2 * -np_.offset[2]) + (float)np_.scale * t;
        } else {
            const double* r = pose + i * 4;
            out[i * 4] = (float)r[0]; out[i * 4 + 1] = (float)r[1]; out[i * 4 + 2] = (float)r[2];
            out[i * 4 + 3] = (float)(((r[0] * -(double)np_.offset[0] + r[1] * -(double)np_.offset[1]) + r[2] * -(double)np_.offset[2]) +
                                     np_.scale * r[3]);
        }
    }
}

struct FrameProblem {            // the per-frame half of geometry.refine_problems
    float K_warp[9];             // float32 intrinsics of the look-at crop
    float pose_warp[12];         // float32 pose of the look-at crop (network input)
    float rect[12];              // float32 look-at rectification [R_look | 0]
    double que_H[9];             // frame -> crop homography
    float qdir[3];               // unit viewing direction (view selection)
    double Rq[9];                // look-at-rectified rotation of the crop camera (in-plane alignment of the views)
};
// camK: the frame's intrinsics as float64 values; camKinv = np.linalg.inv(K) as float64 values; camf = (K00 + K11) / 2
// evaluated in K's dtype.  size_scale = float32(size * (1 - margin) / diameter).
G6D_HD void refine_frame(const float* pose_n, const double* camK, const double* camKinv, double camf, int size,
                         float size_scale, FrameProblem& o) {
    const double zero3[3] = {0., 0., 0.};
    double P[12];
    for (int i = 0; i < 12; ++i) P[i] = (double)pose_n[i];
    double px, py;
    project_center(zero3, P, camK, &px, &py);
    double R_look[9], f_look;
    look_at(px, py, camf, camK[2], camK[5], R_look, &f_look);
    // |camera centre| in float32: -R^T t, then sqrt(x . x)
    float cam[3];
    for (int i = 0; i < 3; ++i) cam[i] = -((pose_n[i] * pose_n[3] + pose_n[4 + i] * pose_n[7]) + pose_n[8 + i] * pose_n[11]);
    const float dist = sqrtf((cam[0] * cam[0] + cam[1] * cam[1]) + cam[2] * cam[2]);
    const double scale = (double)(size_scale * dist) / f_look;
    const float fw = (float)(f_look * scale);
    const float half = (float)size / 2;
    const float Kw[9] = {fw, 0.f, half, 0.f, fw, half, 0.f, 0.f, 1.f};
    double Kd[9], T[9];
    for (int i = 0; i < 9; ++i) { o.K_warp[i] = Kw[i]; Kd[i] = (double)Kw[i]; }
    mat3_mul(Kd, R_look, T);
    mat3_mul(T, camKinv, o.que_H);
    float r[9];
    for (int i = 0; i < 9; ++i) r[i] = (float)R_look[i];
    for (int i = 0; i < 3; ++i) {
        o.rect[i * 4] = r[i * 3]; o.rect[i * 4 + 1] = r[i * 3 + 1]; o.rect[i * 4 + 2] = r[i * 3 + 2]; o.rect[i * 4 + 3] = 0.f;
        for (int j = 0; j < 4; ++j)
            o.pose_warp[i * 4 + j] = (r[i * 3] * pose_n[j] + r[i * 3 + 1] * pose_n[4 + j]) + r[i * 3 + 2] * pose_n[8 + j];
    }
    // viewing direction of the crop camera (float32)
    float cw[3];
    for (int i = 0; i < 3; ++i) cw[i] = -((o.pose_warp[i] * o.pose_warp[3] + o.pose_warp[4 + i] * o.pose_warp[7]) + o.pose_warp[8 + i] * o.pose_warp[11]);
    const float nn = sqrtf((cw[0] * cw[0] + cw[1] * cw[1]) + cw[2] * cw[2]);
    for (int i = 0; i < 3; ++i) o.qdir[i] = cw[i] / nn;
    // Rq = look_at(projected centre under the crop camera) @ R_warp, all float64
    double ap[12];
    for (int i = 0; i < 12; ++i) ap[i] = (double)o.pose_warp[i];
    double qx, qy, R2[9], Rw[9];
    project_center(zero3, ap, Kd, &qx, &qy);
    look_at(qx, qy, (Kd[0] + Kd[4]) / 2, Kd[2], Kd[5], R2, nullptr);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rw[i * 3 + j] = ap[i * 4 + j];
    mat3_mul(R2, Rw, o.Rq);
}

struct ViewProblem {
    float K[9];
    float pose[12];
    double H[9];
};
// geometry._views_at_angle for one table row aligned to Rq
G6D_HD void refine_view(const double* Rq, const double* tab_pose /* [12] */, const double* tab_R_look, const double* tab_RlookR,
                        double tab_f, const double* tab_Kinv, int size, ViewProblem& o) {
    double rel[9];
    mat3_mul_bt(Rq, tab_RlookR, rel);
    const double angle = atan2(-rel[1], rel[0]);
    const float ca = (float)cos(angle), sa = (float)sin(angle);
    const double Rz[9] = {(double)ca, (double)-sa, 0., (double)sa, (double)ca, 0., 0., 0., 1.};
    double R[9], T[9], Kd[9];
    mat3_mul(Rz, tab_R_look, R);
    const float f = (float)tab_f, half = (float)size / 2;
    const float Kn[9] = {f, 0.f, half, 0.f, f, half, 0.f, 0.f, 1.f};
    for (int i = 0; i < 9; ++i) { o.K[i] = Kn[i]; Kd[i] = (double)Kn[i]; }
    mat3_mul(Kd, R, T);
    mat3_mul(T, tab_Kinv, o.H);
    for (int i = 0; i < 3; ++i) {
        const double r0 = (double)(float)R[i * 3], r1 = (double)(float)R[i * 3 + 1], r2 = (double)(float)R[i * 3 + 2];
        for (int j = 0; j < 4; ++j) o.pose[i * 4 + j] = (float)((r0 * tab_pose[j] + r1 * tab_pose[4 + j]) + r2 * tab_pose[8 + j]);
    }
}

// ------------------------------------------------------------------------------------------ D: apply the update
// geometry.apply_refinements for one frame: out7 = (quaternion w x y z, offset x y, log2 scale) of the network
G6D_HD void apply_refinement(const float* que_pose, const float* que_K, const float* rect, const float* out7, const NormParams& np_,
                             float* pose_out /* [12] float32, denormalised */) {
    double Pin[12];
    for (int i = 0; i < 12; ++i) Pin[i] = (double)que_pose[i];
    const double cen_in[3] = {Pin[3], Pin[7], Pin[11]};                   // R @ 0 + t
    // 2.0 ** float32 stays float32 in numpy: the correctly rounded float32 power
    const double s = (double)(float)exp2((double)out7[6]);
    const double w = (double)out7[0], x = (double)out7[1], y = (double)out7[2], z = (double)out7[3];
    const double n = w * w + x * x + y * y + z * z;
    double Q[9] = {1., 0., 0., 0., 1., 0., 0., 0., 1.};
    if (n >= 2.220446049250313e-16) {
        const double sc = 2.0 / n;
        Q[0] = 1 - sc * (y * y + z * z); Q[1] = sc * (x * y - w * z); Q[2] = sc * (x * z + w * y);
        Q[3] = sc * (x * y + w * z); Q[4] = 1 - sc * (x * x + z * z); Q[5] = sc * (y * z - w * x);
        Q[6] = sc * (x * z - w * y); Q[7] = sc * (y * z + w * x); Q[8] = 1 - sc * (x * x + y * y);
    }
    double A[9];
    for (int i = 0; i < 9; ++i) A[i] = s * Q[i];
    const double cen_que[3] = {cen_in[0] + (double)out7[4], cen_in[1] + (double)out7[5], cen_in[2] + 0.0};
    double A_cen[3];
    mat3_vec(A, cen_in, A_cen);
    const double sim_t[3] = {cen_que[0] - A_cen[0], cen_que[1] - A_cen[1], cen_que[2] - A_cen[2]};
    // A = s * Q with Q orthogonal to rounding: the SVD's U V^T is the polar factor (Q after one Newton step
    // 0.5 (Q + Q^-T)) and all singular values equal |A|_F / sqrt(3)
    double Qi[9], Rd[9];
    inv3_cv(Q, Qi);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rd[i * 3 + j] = 0.5 * (Q[i * 3 + j] + Qi[j * 3 + i]);
    double fro = 0.;
    for (int i = 0; i < 9; ++i) fro += A[i] * A[i];
    const double meanS = sqrt(fro / 3.0);
    const double f = ((double)que_K[0] + (double)que_K[4]) / 2;
    const double depth = cen_in[2] / meanS * f / f;
    const double cen_sim[3] = {A_cen[0] + sim_t[0], A_cen[1] + sim_t[1], A_cen[2] + sim_t[2]};
    const double cen_new[3] = {cen_sim[0] / cen_sim[2] * depth, cen_sim[1] / cen_sim[2] * depth, cen_sim[2] / cen_sim[2] * depth};
    double Rin[9], Rn[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rin[i * 3 + j] = Pin[i * 4 + j];
    mat3_mul(Rd, Rin, Rn);
    // centre = 0: pose = [Rn | cen_new]; undo the look-at rectification (inverse of [R_rect | 0] = [R_rect^T | 0])
    double Rr[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rr[i * 3 + j] = (double)rect[i * 4 + j];
    double Rf[9], tf[3];
    mat3_at_mul(Rr, Rn, Rf);
    for (int i = 0; i < 3; ++i) tf[i] = (Rr[i] * cen_new[0] + Rr[3 + i] * cen_new[1]) + Rr[6 + i] * cen_new[2];
    // NormalizedView.denormalize_poses
    for (int i = 0; i < 3; ++i) {
        const double ro = (Rf[i * 3] * (double)np_.offset[0] + Rf[i * 3 + 1] * (double)np_.offset[1]) + Rf[i * 3 + 2] * (double)np_.offset[2];
        pose_out[i * 4] = (float)Rf[i * 3]; pose_out[i * 4 + 1] = (float)Rf[i * 3 + 1]; pose_out[i * 4 + 2] = (float)Rf[i * 3 + 2];
        pose_out[i * 4 + 3] = (float)(ro / np_.scale + tf[i] / np_.scale);
    }
}

// ------------------------------------------------------------------------------------------ E: pose -> detection window
// The inverse of pose_from_similarity for one pose: the detection record (cx, cy, s, 1) that B would have turned into
// this pose's centre and distance.  c = project_center(center, pose, K); s = ref_dist * que_f_ray / ref_f / que_dist
// with que_dist = |camera centre - object centre| and que_f_ray computed at c as B computes it.  ref_dist / ref_f is the
// same for every normalised reference view, so the caller passes row 0's.  in_f32: the pose holds float32 values (as
// after a refinement) and is read rounded to float32; everything else is float64.  A pose whose centre is not in front
// of the camera, or whose c or s is not finite in float32, gives the invalid record (0, 0, 1, 0).
G6D_HD void window_from_pose(const double* pose_in, int in_f32, const double* center, const double* K, const double* Kinv,
                             double f, double f_sq, double ref_dist, double ref_f, float* rec /* [4] */) {
    double P[12];
    for (int i = 0; i < 12; ++i) P[i] = in_f32 ? (double)(float)pose_in[i] : pose_in[i];
    const double depth = (P[8] * center[0] + P[9] * center[1] + P[10] * center[2]) + P[11];
    double px, py;
    project_center(center, P, K, &px, &py);
    double d[3];
    for (int i = 0; i < 3; ++i) d[i] = -((P[i] * P[3] + P[4 + i] * P[7]) + P[8 + i] * P[11]) - center[i];
    const double que_dist = sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
    const double v[3] = {px, py, 1.0};
    double bearing[3];
    mat3_vec(Kinv, v, bearing);
    const double bx = bearing[0] / bearing[2], by = bearing[1] / bearing[2];
    const double n2 = sqrt((bx * f) * (bx * f) + (by * f) * (by * f));
    const double que_f_ray = sqrt(f_sq + n2 * n2);
    const double s = ref_dist * que_f_ray / ref_f / que_dist;
    const float cx = (float)px, cy = (float)py, fs = (float)s;
    if (depth > 0 && isfinite(cx) && isfinite(cy) && isfinite(fs) && fs > 0.f) {
        rec[0] = cx; rec[1] = cy; rec[2] = fs; rec[3] = 1.f;
    } else {
        rec[0] = 0.f; rec[1] = 0.f; rec[2] = 1.f; rec[3] = 0.f;
    }
}

// A detection (x, y, scale, score) in the window of record `rec` (size `window`) mapped back to the frame:
// out = (cx + (x - window/2) s, cy + (y - window/2) s, scale s, score, offset), offset = |(x, y) - window/2| s /
// (ref_resolution s), the distance of the detection from the pose's centre in reference sizes.  lost: the record is
// invalid, or use_score and not score >= lost_score (NaN is lost), or use_gate and not offset <= lost_gate (NaN is
// lost); both comparisons take the float32 values returned, so a tie with the threshold is kept.
G6D_HD int verify_judge(const float* rec, const float* det, int window, double ref_resolution, int use_score, double lost_score,
                        int use_gate, double lost_gate, float* out /* [5] */) {
    const double cx = rec[0], cy = rec[1], s = rec[2], half = window / 2;
    const double dx = ((double)det[0] - half) * s, dy = ((double)det[1] - half) * s;
    out[0] = (float)(cx + dx);
    out[1] = (float)(cy + dy);
    out[2] = (float)((double)det[2] * s);
    out[3] = det[3];
    out[4] = (float)(sqrt(dx * dx + dy * dy) / (ref_resolution * s));
    int lost = rec[3] == 0.f;
    if (use_score && !((double)out[3] >= lost_score)) lost = 1;
    if (use_gate && !((double)out[4] <= lost_gate)) lost = 1;
    return lost;
}

}  // namespace glue
}  // namespace g6d
