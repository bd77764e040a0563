// Temporal smoothing of a tracked pose (predict.py:18-26,61-70 of the reference) as __host__ __device__ code: project
// the object's 3-D bounding box with the new raw pose (utils/base_utils.py:256-265 project_points), push the corners
// into a per-sequence history, take predict.py's exponentially weighted average of the last `num` frames' corners
// (weighted_pts), and turn the average back into a pose with OpenCV's SOLVEPNP_ITERATIVE for non-planar points
// (utils/pose_utils.py:246-279 pnp; calib3d cvFindExtrinsicCameraParams2: DLT initialisation, then Levenberg-Marquardt
// on the pixel reprojection error).  track.cu runs it inside the tracking step's graph, one thread per sequence; its
// *_host entry point runs the very same code on host memory, so the CPU tests pin it against numpy and cv2.solvePnP.
// This translation unit is compiled with -fmad=false: products and sums round separately, like numpy's.
#pragma once
#include <float.h>
#include <math.h>

#include "glue_math.cuh"

namespace g6d {
namespace track {

constexpr int kCorners = 8;

// the larger steps stay out of line on the device: their arrays live in the stack frame instead of being unrolled
// into registers (one thread per sequence; this is not a throughput kernel)
#if defined(__CUDACC__)
#define G6D_HD_NOINLINE static __host__ __device__ __noinline__
#else
#define G6D_HD_NOINLINE static
#endif

// ------------------------------------------------------------------------------------------ projection
// project_points(bbox, pose, K) for the 8 corners: (pts @ R^T + t) @ K^T, then the depth clamp 0 < |d| < 1e-4 -> 1e-4
// (the reference's second mask, -1e-4 < |d| < 0, is never true).  in_f32: the pose is float32 (refiner output) and
// numpy computes in float32 with the float32 bbox and K of predict.py; else in float64.  pts [16] = (u, v) per corner.
G6D_HD_NOINLINE void project_box(const float* bbox, const double* pose, int in_f32, const double* K, float* pts) {
    for (int c = 0; c < kCorners; ++c) {
        const float* X = bbox + c * 3;
        if (in_f32) {
            float p[3], q[3];
            // numpy's float32 matmul goes to BLAS sgemm, which evaluates each 3-term dot as a fused multiply-add chain
            for (int i = 0; i < 3; ++i)
                p[i] = fmaf(X[2], (float)pose[i * 4 + 2], fmaf(X[1], (float)pose[i * 4 + 1], X[0] * (float)pose[i * 4])) + (float)pose[i * 4 + 3];
            for (int j = 0; j < 3; ++j) q[j] = fmaf(p[2], (float)K[j * 3 + 2], fmaf(p[1], (float)K[j * 3 + 1], p[0] * (float)K[j * 3]));
            float d = q[2];
            if (fabsf(d) < 1e-4f && fabsf(d) > 0.f) d = 1e-4f;
            pts[c * 2] = q[0] / d;
            pts[c * 2 + 1] = q[1] / d;
        } else {
            double p[3], q[3];
            for (int i = 0; i < 3; ++i)
                p[i] = (((double)X[0] * pose[i * 4] + (double)X[1] * pose[i * 4 + 1]) + (double)X[2] * pose[i * 4 + 2]) + pose[i * 4 + 3];
            for (int j = 0; j < 3; ++j) q[j] = (p[0] * K[j * 3] + p[1] * K[j * 3 + 1]) + p[2] * K[j * 3 + 2];
            double d = q[2];
            if (fabs(d) < 1e-4 && fabs(d) > 0.) d = 1e-4;
            pts[c * 2] = (float)(q[0] / d);
            pts[c * 2 + 1] = (float)(q[1] / d);
        }
    }
}

// ------------------------------------------------------------------------------------------ weighted average
// numpy's np.sum of a 1-D float64 array (pairwise_sum): a plain loop below 8 elements, else 8 accumulators combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) and the remainder added in order (n <= 128 here).
G6D_HD double numpy_sum(const double* a, int n) {
    if (n < 8) {
        double res = 0.;
        for (int i = 0; i < n; ++i) res += a[i];
        return res;
    }
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
}

// Push the newest corners into the history ring [num][16] (oldest first; count = frames held, <= num) and return
// weighted_pts(history, num, std) in float64: weights w[num] = np.exp(-(np.arange(num) / std) ** 2)[::-1] (oldest first,
// computed by the caller with numpy), the newest min(count, num) of them; the frames summed oldest first as numpy's
// axis-0 reduction does, divided by np.sum of the weights used.
G6D_HD_NOINLINE void push_and_average(float* ring, int* count, int num, const float* pts, const double* w, double* avg) {
    int c = *count;
    c = c < 0 ? 0 : (c > num ? num : c);
    if (c == num) {
        for (int k = 0; k + 1 < num; ++k)
            for (int e = 0; e < 2 * kCorners; ++e) ring[k * 2 * kCorners + e] = ring[(k + 1) * 2 * kCorners + e];
        c = num - 1;
    }
    for (int e = 0; e < 2 * kCorners; ++e) ring[c * 2 * kCorners + e] = pts[e];
    const int n = c + 1;
    *count = n;
    const double* wn = w + (num - n);
    for (int e = 0; e < 2 * kCorners; ++e) {
        double acc = (double)ring[e] * wn[0];
        for (int k = 1; k < n; ++k) acc = acc + (double)ring[k * 2 * kCorners + e] * wn[k];
        avg[e] = acc;
    }
    const double ws = numpy_sum(wn, n);
    for (int e = 0; e < 2 * kCorners; ++e) avg[e] = avg[e] / ws;
}

// ------------------------------------------------------------------------------------------ small dense algebra
G6D_HD double det3(const double* a) {
    return a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) + a[2] * (a[3] * a[7] - a[4] * a[6]);
}
G6D_HD double fro(const double* a, int n) {
    double s = 0.;
    for (int i = 0; i < n; ++i) s += a[i] * a[i];
    return sqrt(s);
}

// Eigenvector of the smallest eigenvalue of a symmetric 12x12 matrix (cyclic Jacobi; A is destroyed).  For the
// symmetric positive semi-definite L^T L this is the right singular vector OpenCV's cvSVD returns last.
G6D_HD_NOINLINE void sym12_min_eigvec(double* A, double* v_out) {
    constexpr int n = 12;
    double V[n * n];
    for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1. : 0.;
#pragma unroll 1
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0., diag = 0.;
        for (int p = 0; p < n; ++p) {
            diag += A[p * n + p] * A[p * n + p];
            for (int q = p + 1; q < n; ++q) off += A[p * n + q] * A[p * n + q];
        }
        if (off <= 1e-34 * diag || off == 0.) break;
#pragma unroll 1
        for (int p = 0; p < n - 1; ++p)
#pragma unroll 1
            for (int q = p + 1; q < n; ++q) {
                const double apq = A[p * n + q];
                if (apq == 0.) continue;
                const double app = A[p * n + p], aqq = A[q * n + q];
                const double theta = (aqq - app) / (2. * apq);
                const double t = (theta >= 0. ? 1. : -1.) / (fabs(theta) + sqrt(theta * theta + 1.));
                const double c = 1. / sqrt(t * t + 1.), s = t * c;
                for (int k = 0; k < n; ++k) {         // A <- A J (columns p, q)
                    const double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq;
                    A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; ++k) {         // A <- J^T A (rows p, q)
                    const double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk;
                    A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; ++k) {         // V <- V J
                    const double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s * vkq;
                    V[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    int best = 0;
    for (int i = 1; i < n; ++i)
        if (A[i * n + i] < A[best * n + best]) best = i;
    for (int i = 0; i < n; ++i) v_out[i] = V[i * n + best];
}

// Orthogonal polar factor U V^T of a 3x3 with det > 0 (Newton: X <- (X + X^-T) / 2, scaled while far from converged).
G6D_HD_NOINLINE void polar3(const double* A, double* R) {
    double X[9];
    for (int i = 0; i < 9; ++i) X[i] = A[i];
    for (int it = 0; it < 100; ++it) {
        double Xi[9];
        g6d::glue::inv3_cv(X, Xi);
        const double g = it < 6 ? sqrt(fro(Xi, 9) / fro(X, 9)) : 1.;
        double Y[9], dif = 0.;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                Y[i * 3 + j] = 0.5 * (g * X[i * 3 + j] + Xi[j * 3 + i] / g);
                dif += (Y[i * 3 + j] - X[i * 3 + j]) * (Y[i * 3 + j] - X[i * 3 + j]);
            }
        for (int i = 0; i < 9; ++i) X[i] = Y[i];
        if (it >= 6 && dif < 1e-30) break;
    }
    for (int i = 0; i < 9; ++i) R[i] = X[i];
}

// cv::Rodrigues, rotation vector -> matrix, with OpenCV's Jacobian J[i*9 + k] = dR_k / dr_i (J may be null)
G6D_HD_NOINLINE void rodrigues_vec(const double* r, double* R, double* J) {
    const double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    if (theta < DBL_EPSILON) {
        for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1. : 0.;
        if (J) {
            for (int i = 0; i < 27; ++i) J[i] = 0.;
            J[5] = J[15] = J[19] = -1.;
            J[7] = J[11] = J[21] = 1.;
        }
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1. - c, itheta = 1. / theta;
    const double x = r[0] * itheta, y = r[1] * itheta, z = r[2] * itheta;
    const double rrt[9] = {x * x, x * y, x * z, x * y, y * y, y * z, x * z, y * z, z * z};
    const double rx[9] = {0., -z, y, z, 0., -x, -y, x, 0.};
    for (int k = 0; k < 9; ++k) R[k] = ((k % 4 == 0) ? c : 0.) + c1 * rrt[k] + s * rx[k];
    if (J) {
        const double I[9] = {1., 0., 0., 0., 1., 0., 0., 0., 1.};
        const double drrt[27] = {x + x, y, z, y, 0., 0., z, 0., 0.,
                                 0., x, 0., x, y + y, z, 0., z, 0.,
                                 0., 0., x, 0., 0., y, x, y, z + z};
        const double drx[27] = {0., 0., 0., 0., 0., -1., 0., 1., 0.,
                                0., 0., 1., 0., 0., 0., -1., 0., 0.,
                                0., -1., 0., 1., 0., 0., 0., 0., 0.};
        for (int i = 0; i < 3; ++i) {
            const double ri = i == 0 ? x : (i == 1 ? y : z);
            const double a0 = -s * ri, a1 = (s - 2. * c1 * itheta) * ri, a2 = c1 * itheta;
            const double a3 = (c - s * itheta) * ri, a4 = s * itheta;
            for (int k = 0; k < 9; ++k)
                J[i * 9 + k] = a0 * I[k] + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * rx[k] + a4 * drx[i * 9 + k];
        }
    }
}

// cv::Rodrigues, matrix -> rotation vector (R orthonormal to rounding)
G6D_HD_NOINLINE void rodrigues_mat(const double* R, double* r) {
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1.) * 0.5;
    c = c > 1. ? 1. : (c < -1. ? -1. : c);
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0.) {
            rx = ry = rz = 0.;
        } else {
            double t = (R[0] + 1.) * 0.5;
            rx = sqrt(t > 0. ? t : 0.);
            t = (R[4] + 1.) * 0.5;
            ry = sqrt(t > 0. ? t : 0.) * (R[1] < 0. ? -1. : 1.);
            t = (R[8] + 1.) * 0.5;
            rz = sqrt(t > 0. ? t : 0.) * (R[2] < 0. ? -1. : 1.);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0.) != (ry * rz > 0.)) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            rx *= theta; ry *= theta; rz *= theta;
        }
    } else {
        const double vth = 1. / (2. * s) * theta;
        rx *= vth; ry *= vth; rz *= vth;
    }
    r[0] = rx; r[1] = ry; r[2] = rz;
}

// Solve the symmetric positive definite 6x6 system A x = b (Cholesky; A is destroyed).  Returns false if not SPD.
G6D_HD_NOINLINE bool spd6_solve(double* A, const double* b, double* x) {
    constexpr int n = 6;
    for (int j = 0; j < n; ++j) {
        double d = A[j * n + j];
        for (int k = 0; k < j; ++k) d -= A[j * n + k] * A[j * n + k];
        if (!(d > 0.)) return false;
        d = sqrt(d);
        A[j * n + j] = d;
        for (int i = j + 1; i < n; ++i) {
            double s = A[i * n + j];
            for (int k = 0; k < j; ++k) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / d;
        }
    }
    double y[n];
    for (int i = 0; i < n; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= A[i * n + k] * y[k];
        y[i] = s / A[i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < n; ++k) s -= A[k * n + i] * x[k];
        x[i] = s / A[i * n + i];
    }
    return true;
}

// ------------------------------------------------------------------------------------------ PnP
struct PnPInput {
    double M[kCorners * 3];      // object points (the float32 bbox as float64)
    double m[kCorners * 2];      // image points (pixels)
    double fx, fy, cx, cy;
};

// reprojection residuals (projected - observed) of param = (rvec, t) and, if J != null, their Jacobian [16][6]
G6D_HD_NOINLINE void pnp_residuals(const PnPInput& in, const double* param, double* err, double* J) {
    double R[9], dRdr[27];
    rodrigues_vec(param, R, J ? dRdr : nullptr);
    const double* t = param + 3;
    for (int i = 0; i < kCorners; ++i) {
        const double* X = in.M + i * 3;
        const double Y[3] = {R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0], R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1],
                             R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2]};
        const double z = Y[2] != 0. ? 1. / Y[2] : 1.;
        const double x = Y[0] * z, y = Y[1] * z;
        err[i * 2] = (x * in.fx + in.cx) - in.m[i * 2];
        err[i * 2 + 1] = (y * in.fy + in.cy) - in.m[i * 2 + 1];
        if (J) {
            double* ju = J + (i * 2) * 6;
            double* jv = J + (i * 2 + 1) * 6;
            for (int j = 0; j < 3; ++j) {
                const double* d = dRdr + j * 9;
                const double dY0 = d[0] * X[0] + d[1] * X[1] + d[2] * X[2];
                const double dY1 = d[3] * X[0] + d[4] * X[1] + d[5] * X[2];
                const double dY2 = d[6] * X[0] + d[7] * X[1] + d[8] * X[2];
                ju[j] = in.fx * (z * (dY0 - x * dY2));
                jv[j] = in.fy * (z * (dY1 - y * dY2));
            }
            ju[3] = in.fx * z; ju[4] = 0.; ju[5] = -in.fx * x * z;
            jv[3] = 0.; jv[4] = in.fy * z; jv[5] = -in.fy * y * z;
        }
    }
}

// OpenCV's CvLevMarq::step: param = prev - solve(JtJ with its diagonal scaled by 1 + 10^lambdaLg10, JtErr)
G6D_HD_NOINLINE void lm_step(const double* JtJ, const double* JtErr, const double* prev, int lambda_lg10, double* param) {
    double A[36], d[6];
    const double lambda = exp(lambda_lg10 * log(10.));
    for (int i = 0; i < 36; ++i) A[i] = JtJ[i];
    for (int i = 0; i < 6; ++i) A[i * 7] *= 1. + lambda;
    if (!spd6_solve(A, JtErr, d))
        for (int i = 0; i < 6; ++i) d[i] = 0.;
    for (int i = 0; i < 6; ++i) param[i] = prev[i] - d[i];
}

// DLT initialisation of cvFindExtrinsicCameraParams2 for non-planar points: the 12-vector of the smallest singular value
// of the 2n x 12 system on the normalised image points, its sign fixed so that det(R) > 0, R orthonormalised (U V^T of
// its SVD) and t scaled by |R_orth| / |R_dlt|; param = (Rodrigues vector, t)
G6D_HD_NOINLINE void pnp_dlt(const PnPInput& in, double* param) {
    const double ifx = 1. / in.fx, ify = 1. / in.fy;
    double LL[144];
    for (int i = 0; i < 144; ++i) LL[i] = 0.;
#pragma unroll 1
    for (int i = 0; i < kCorners; ++i) {
        const double* X = in.M + i * 3;
        const double x = -((in.m[i * 2] - in.cx) * ifx), y = -((in.m[i * 2 + 1] - in.cy) * ify);   // cvUndistortPoints
        const double r0[12] = {X[0], X[1], X[2], 1., 0., 0., 0., 0., x * X[0], x * X[1], x * X[2], x};
        const double r1[12] = {0., 0., 0., 0., X[0], X[1], X[2], 1., y * X[0], y * X[1], y * X[2], y};
#pragma unroll 1
        for (int a = 0; a < 12; ++a)
#pragma unroll 1
            for (int b = 0; b < 12; ++b) LL[a * 12 + b] += r0[a] * r0[b] + r1[a] * r1[b];
    }
    double v[12];
    sym12_min_eigvec(LL, v);
    double RR[9] = {v[0], v[1], v[2], v[4], v[5], v[6], v[8], v[9], v[10]};
    double tt[3] = {v[3], v[7], v[11]};
    if (det3(RR) < 0.) {
        for (int i = 0; i < 9; ++i) RR[i] = -RR[i];
        for (int i = 0; i < 3; ++i) tt[i] = -tt[i];
    }
    const double sc = fro(RR, 9);
    double R[9];
    polar3(RR, R);
    const double ts = fro(R, 9) / sc;
    rodrigues_mat(R, param);
    for (int i = 0; i < 3; ++i) param[3 + i] = tt[i] * ts;
}

// CvLevMarq as cvFindExtrinsicCameraParams2 drives it: lambda 1e-3, at most 20 iterations, stop at a relative parameter
// change below FLT_EPSILON; a step that raises the error norm is retried with ten times the damping
G6D_HD_NOINLINE void pnp_lm(const PnPInput& in, double* param) {
    double err[kCorners * 2], J[kCorners * 2 * 6], JtJ[36], JtErr[6], prev[6];
    int lambda_lg10 = -3, iters = 0;
    double prev_err = 0.;
#pragma unroll 1
    for (;;) {
        pnp_residuals(in, param, err, J);
#pragma unroll 1
        for (int a = 0; a < 6; ++a) {
#pragma unroll 1
            for (int b = 0; b < 6; ++b) {
                double s = 0.;
                for (int k = 0; k < kCorners * 2; ++k) s += J[k * 6 + a] * J[k * 6 + b];
                JtJ[a * 6 + b] = s;
            }
            double s = 0.;
            for (int k = 0; k < kCorners * 2; ++k) s += J[k * 6 + a] * err[k];
            JtErr[a] = s;
        }
        for (int i = 0; i < 6; ++i) prev[i] = param[i];
        lm_step(JtJ, JtErr, prev, lambda_lg10, param);
        if (iters == 0) prev_err = fro(err, kCorners * 2);
        double err_norm;
#pragma unroll 1
        for (;;) {
            pnp_residuals(in, param, err, nullptr);
            err_norm = fro(err, kCorners * 2);
            if (err_norm > prev_err && ++lambda_lg10 <= 16) {
                lm_step(JtJ, JtErr, prev, lambda_lg10, param);
                continue;
            }
            break;
        }
        lambda_lg10 = lambda_lg10 - 1 > -16 ? lambda_lg10 - 1 : -16;
        double dn = 0., pn = 0.;
        for (int i = 0; i < 6; ++i) {
            dn += (param[i] - prev[i]) * (param[i] - prev[i]);
            pn += prev[i] * prev[i];
        }
        if (++iters >= 20 || sqrt(dn) / (sqrt(pn) + DBL_EPSILON) < FLT_EPSILON) break;
        prev_err = err_norm;
    }
}

// cv2.solvePnP(bbox, pts, K, zeros, flags=SOLVEPNP_ITERATIVE) for 8 non-coplanar corners, then [cv2.Rodrigues(r) | t].
// K: float64 values [9]; pose_out [12] row-major [R | t].
G6D_HD_NOINLINE void pnp_iterative(const float* bbox, const double* pts, const double* K, double* pose_out) {
    PnPInput in;
    for (int i = 0; i < kCorners * 3; ++i) in.M[i] = (double)bbox[i];
    for (int i = 0; i < kCorners * 2; ++i) in.m[i] = pts[i];
    in.fx = K[0]; in.fy = K[4]; in.cx = K[2]; in.cy = K[5];
    double param[6], R[9];
    pnp_dlt(in, param);
    pnp_lm(in, param);
    rodrigues_vec(param, R, nullptr);
    for (int i = 0; i < 3; ++i) {
        pose_out[i * 4] = R[i * 3]; pose_out[i * 4 + 1] = R[i * 3 + 1]; pose_out[i * 4 + 2] = R[i * 3 + 2];
        pose_out[i * 4 + 3] = param[3 + i];
    }
}

// ------------------------------------------------------------------------------------------ one sequence, one step
G6D_HD_NOINLINE void smooth_one(int s, const double* poses, int in_f32, const float* bbox, const double* Ks, float* ring, int* count, int num,
                       const double* w, double* smoothed, double* avg_pts) {
    float pts[2 * kCorners];
    const double* K = Ks + (long long)s * 9;
    project_box(bbox, poses + (long long)s * 12, in_f32, K, pts);
    double* avg = avg_pts + (long long)s * 2 * kCorners;
    push_and_average(ring + (long long)s * num * 2 * kCorners, count + s, num, pts, w, avg);
    pnp_iterative(bbox, avg, K, smoothed + (long long)s * 12);
}

}  // namespace track
}  // namespace g6d
