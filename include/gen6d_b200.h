/*
 * gen6d_b200.h -- C ABI of libgen6d_b200.so: the sm_90a (H100) kernels behind the Gen6D inference
 * hot path (detector correlation head, selector similarity scoring, refiner feature volume +
 * conv stacks).
 *
 * The reference (liuyuan-pal/Gen6D) is pure PyTorch and has no FFI of its own (SURVEY.md 8b);
 * this header is the "lower face" of the drop-in boundary: the entry points that the Python
 * classes mirroring network/{detector,selector,refiner}.py bind with ctypes.  Each entry cites
 * the reference call site whose arithmetic it replaces.
 *
 * Conventions
 *  - every function returns 0 on success, a negative G6D_E* code otherwise;
 *    g6d_last_error() gives a thread-local message for the last failure on this thread;
 *  - all pointers are DEVICE pointers unless the parameter is named host_*; the caller owns
 *    every buffer (inputs, outputs, workspaces); the library never allocates device memory,
 *    never synchronises, and only enqueues work on the `stream` it is given (so calls can be
 *    captured into CUDA graphs);
 *  - activations are fp32, channels-last: [B, (D,) H, W, C] with C contiguous.  The NCHW
 *    tensors of the reference API are converted at the Python boundary with
 *    g6d_nchw_to_nhwc / g6d_nhwc_to_nchw;
 *  - convolution weights are packed [K, ldw] (ldw = Cout rounded up to 4) with
 *    K = ((kz*kh + ky)*kw + kx)*Cin + c
 *    (g6d_pack_conv_weight does this from the reference's [Cout, Cin, kd, kh, kw]).
 */
#ifndef GEN6D_B200_H
#define GEN6D_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define G6D_OK 0
#define G6D_EINVAL (-1)   /* bad argument / unsupported shape */
#define G6D_ECUDA (-2)    /* CUDA runtime error at launch */

typedef void* g6d_stream_t; /* cudaStream_t */

const char* g6d_last_error(void);
int g6d_version(void);
/* number of kernel launches issued through this library since load (all threads) */
long long g6d_launch_count(void);

/* ------------------------------------------------------------------ layout / image ops ---- */
/* utils/base_utils.py:117-118 color_map_forward (+ torchvision Normalize of
 * network/detector.py:156,189 when imagenet_norm != 0).  u8 [n_pixels,3] -> f32 [n_pixels,out_c],
 * out_c = 3 or 4 (channel 3 = 0: padding so the first VGG conv can use 128-bit loads). */
int g6d_preprocess_u8(const uint8_t* img, float* out, long long n_pixels, int out_c, int imagenet_norm,
                      g6d_stream_t stream);
/* One image warp: `src` is a device uint8 [rows, cols, 3] image; M is the row-major DST -> SRC map
 * (what OpenCV holds after its internal inversion: cv::invert of the 3x3 for warpPerspective; the
 * closed-form 2x3 inverse, rows M[0..2] and M[3..5], for warpAffine - M[6..8] unused there). */
typedef struct g6d_warp_job {
    const uint8_t* src;
    int rows, cols;
    double M[9];
} g6d_warp_job;
/* cv2.warpPerspective(src, H, (w, h), flags=INTER_LINEAR) with a zero constant border, bit-exact with
 * OpenCV's 8-bit fixed-point path, for n_jobs (image, matrix) pairs at once: the look-at crops of
 * network/refiner.py:285-325 (utils/database_utils.py:8-25 look_at_crop, :54-110
 * normalize_reference_views).  jobs: DEVICE array [n_jobs]; out u8 [n_jobs, h, w, 3]. */
int g6d_warp_perspective_u8(const g6d_warp_job* jobs, int n_jobs, uint8_t* out, int h, int w, g6d_stream_t stream);
/* cv2.warpAffine(src, M, (w, h), flags=INTER_LINEAR), same conventions: the detection crop of
 * estimator.py:184 (utils/base_utils.py:646-655 transformation_crop). */
int g6d_warp_affine_u8(const g6d_warp_job* jobs, int n_jobs, uint8_t* out, int h, int w, g6d_stream_t stream);
/* Frames of different sizes as one zero-padded canvas (the `frames` argument of the g6d_glue_* kernels): frame i is
 * the uint8 [rows, cols, 3] image at packed + offset, and canvas [n, H, W, 3] gets it in its top-left corner and 0 in
 * every other byte (every byte is written).  A crop cut from the canvas with rows = H, cols = W equals the crop cut from
 * the frame itself, bit for bit (taps outside a frame read the zero border either way).  host_table: HOST array [n],
 * validated (rows <= H, cols <= W, each frame inside packed_bytes) and passed by value, n <= G6D_FRAMES_MAX. */
#define G6D_FRAMES_MAX 1024
typedef struct g6d_frame_entry {
    long long offset;              /* byte offset of the frame in the packed buffer */
    int rows, cols;
} g6d_frame_entry;
int g6d_frames_canvas(const uint8_t* packed, long long packed_bytes, const g6d_frame_entry* host_table, int n, uint8_t* canvas,
                      int H, int W, g6d_stream_t stream);
/* Frames already on the device (a decoder surface, a CUDA RGB tensor) into the packed layout of g6d_frames_canvas:
 * frame i of the table becomes the tightly packed uint8 [rows, cols, 3] RGB image at packed + offset.
 *   G6D_FRAME_RGB:  plane0 is the RGB image, pixel (y, x) at plane0 + y*pitch0 + 3*x (pitch0 >= 3*cols); a pitched copy.
 *   G6D_FRAME_NV12: plane0 the Y plane [rows, cols] (row pitch pitch0 >= cols), plane1 the interleaved U,V plane
 *                   [rows/2, cols] (pitch1 >= cols); rows and cols even.  Converted as cv2.cvtColor(COLOR_YUV2RGB_NV12)
 *                   does, bit for bit: BT.601 limited range in OpenCV's 20-bit fixed point (csrc/frames_math.cuh).
 * Planes need no alignment.  Every byte of packed is written: bytes no frame covers get 0, so a graph replay never
 * depends on what packed held before.  g6d_frames_table_check validates a HOST copy of a table: formats, positive and
 * (NV12) even sizes, non-null planes, pitches, every frame inside packed_bytes, no two frames overlapping, and
 * 1 <= n <= G6D_FRAMES_MAX; G6D_EINVAL with a message otherwise.  g6d_frames_gather reads `table` from DEVICE memory
 * (like g6d_warp_job arrays), so the pointers and pitches of a captured launch change with the table's contents; the
 * caller checks the table before uploading it, and max_rows / max_cols bound every frame's size.  The frames must be
 * ready on `stream`.  g6d_frames_gather_host runs the same code on a HOST table of host planes (checked first). */
#define G6D_FRAME_RGB 0
#define G6D_FRAME_NV12 1
typedef struct g6d_device_frame {
    const uint8_t* plane0;         /* RGB: the [rows, cols, 3] image; NV12: the Y plane */
    const uint8_t* plane1;         /* NV12: the interleaved U,V plane; RGB: unused */
    long long pitch0, pitch1;      /* row pitches in bytes */
    int rows, cols, format;
    long long offset;              /* byte offset of the frame's packed [rows, cols, 3] image */
} g6d_device_frame;
int g6d_frames_table_check(const g6d_device_frame* host_table, int n, long long packed_bytes);
int g6d_frames_gather(const g6d_device_frame* table, int n, int max_rows, int max_cols, uint8_t* packed, long long packed_bytes,
                      g6d_stream_t stream);
int g6d_frames_gather_host(const g6d_device_frame* host_table, int n, uint8_t* packed, long long packed_bytes);
/* Device frames resized and rotated to a working size on the way into the packed layout: frame i becomes
 *   cv2.rotate(cv2.resize(rgb, (cols, rows), interpolation=cv2.INTER_LINEAR), code)
 * bit for bit, as x86 OpenCV computes it, with rgb the RGB image of its source planes (src_rows x src_cols, planes,
 * pitches and format as in g6d_device_frame, NV12 converted as g6d_frames_gather converts it) and code the rotation
 * (0 none, 90 ROTATE_90_CLOCKWISE, 180 ROTATE_180, 270 ROTATE_90_COUNTERCLOCKWISE).  Downscales and identity only:
 * 1 <= rows <= src_rows and 1 <= cols <= src_cols.  The same size is a copy, exactly half the size in both axes
 * OpenCV's INTER_AREA switch, anything else its 11-bit fixed-point INTER_LINEAR (csrc/frames_math.cuh).  The packed
 * image at offset is the working [rows, cols, 3] image, [cols, rows, 3] for 90 and 270.  Every byte of packed is
 * written, as by g6d_frames_gather.  g6d_frames_resized_table_check validates a HOST table like g6d_frames_table_check
 * (plus the rotation and the working size, <= 65535 on each axis); g6d_frames_gather_resized reads the table from DEVICE
 * memory, max_rows / max_cols bounding every frame's working size (<= 65535); g6d_frames_gather_resized_host runs the
 * same code on a HOST table of host planes (checked first). */
typedef struct g6d_resized_frame {
    const uint8_t* plane0;         /* as g6d_device_frame */
    const uint8_t* plane1;
    long long pitch0, pitch1;
    int src_rows, src_cols, format;
    int rows, cols;                /* the resized size, before the rotation */
    int rotate;                    /* degrees clockwise: 0, 90, 180 or 270 */
    long long offset;              /* byte offset of the frame's packed working image */
} g6d_resized_frame;
int g6d_frames_resized_table_check(const g6d_resized_frame* host_table, int n, long long packed_bytes);
int g6d_frames_gather_resized(const g6d_resized_frame* table, int n, int max_rows, int max_cols, uint8_t* packed,
                              long long packed_bytes, g6d_stream_t stream);
int g6d_frames_gather_resized_host(const g6d_resized_frame* host_table, int n, uint8_t* packed, long long packed_bytes);

/* ---- camera algebra between the stages, on the device (estimator.py:176-214; utils/pose_utils.py:12-58,104-111,
 * 217-244; utils/database_utils.py:8-25,54-139; dataset/database.py:400-404,667-694).  With these four launches a
 * batched prediction detect -> select -> refine x N is one stream-ordered sequence with no host round trip.  The
 * *_host variants run the identical code on host memory (unit tests against the numpy restatement). */
typedef struct g6d_glue_camera {   /* one query frame; filled by the caller (numpy), float64 VALUES of:           */
    double K[9];                   /*   the intrinsics,                                                           */
    double Kinv[9];                /*   np.linalg.inv(K) evaluated in K's own dtype,                              */
    double f;                      /*   (K[0,0] + K[1,1]) / 2 evaluated in K's own dtype,                         */
    double f_sq;                   /*   f ** 2 evaluated in K's own dtype (a float32 K squares in float32)        */
} g6d_glue_camera;
typedef struct g6d_glue_refs {     /* the selector's reference views (device arrays, built once per object)       */
    const double* poses;           /* [rfn,12] normalised reference poses (estimator.py:167 ref_info['poses'])    */
    const double* cen;             /* [rfn,2]  projected object centre                                            */
    const double* f;               /* [rfn]    (K00 + K11) / 2                                                    */
    const double* dist;            /* [rfn]    |camera centre - object centre|                                    */
    double center[3];
} g6d_glue_refs;
typedef struct g6d_glue_views {    /* the refiner's database views in unit-sphere coordinates (device arrays)     */
    const double* poses;           /* [n,12] */
    const double* R_look;          /* [n,9]  look-at rotation of every view                                        */
    const double* RlookR;          /* [n,9]  R_look @ R                                                            */
    const double* f;               /* [n]    focal length of the normalised crop                                   */
    const double* Kinv;            /* [n,9]  */
    const unsigned long long* src; /* [n]    device address of the view's uint8 [rows, cols, 3] image              */
    const int* rows; const int* cols;
    const int* even_idx;           /* [n_even] table rows of the FPS re-spread subset (database_utils.py:129-134)  */
    const float* even_dirs;        /* [n_even,3] their unit viewing directions                                     */
    int n_views, n_even, ref_num, size;
    double norm_scale;             /* 2 / object diameter                                                          */
    float norm_offset[3];          /* -norm_scale * object centre (float32, as numpy holds it)                     */
    float size_scale;              /* float32(size * (1 - margin) / 2)                                             */
} g6d_glue_views;
/* det_out [qn,4] (x, y, scale, score; g6d_det_parse) -> the selector's crop jobs [qn] (g6d_warp_affine_u8), frame i at
 * frames + i*rows*cols*3 */
int g6d_glue_detection_jobs(const float* det_out, const uint8_t* frames, int rows, int cols, int qn, int size,
                            g6d_warp_job* jobs, g6d_stream_t stream);
int g6d_glue_detection_jobs_host(const float* det_out, const uint8_t* frames, int rows, int cols, int qn, int size,
                                 g6d_warp_job* jobs);
/* detection + selection (sel_idx [qn] int64, sel_out [qn,2] = angle, logit; g6d_sel_parse) -> poses float64 [qn,12] */
int g6d_glue_initial_poses(const float* det_out, const long long* sel_idx, const float* sel_out, const g6d_glue_refs* refs,
                           const g6d_glue_camera* cams, int qn, double* poses, g6d_stream_t stream);
int g6d_glue_initial_poses_host(const float* det_out, const long long* sel_idx, const float* sel_out, const g6d_glue_refs* refs,
                                const g6d_glue_camera* cams, int qn, double* poses);
/* poses [qn,12] (float64 storage; poses_are_f32: the values are float32 poses, as after a refinement) -> everything one
 * refinement stage reads: jobs [qn*(ref_num+1)] (query crop, then its views; g6d_warp_perspective_u8), que_K [qn,9],
 * que_pose [qn,12], rect [qn,12], ref_Ks [qn,ref_num,9], ref_poses [qn,ref_num,12] (float32), ref_rows [qn,ref_num] */
int g6d_glue_refine_problems(const g6d_glue_views* views, const g6d_glue_camera* cams, const uint8_t* frames, int rows, int cols,
                             const double* poses, int poses_are_f32, int qn, g6d_warp_job* jobs, float* que_K, float* que_pose,
                             float* rect, float* ref_Ks, float* ref_poses, int* ref_rows, g6d_stream_t stream);
int g6d_glue_refine_problems_host(const g6d_glue_views* views, const g6d_glue_camera* cams, const uint8_t* frames, int rows,
                                  int cols, const double* poses, int poses_are_f32, int qn, g6d_warp_job* jobs, float* que_K,
                                  float* que_pose, float* rect, float* ref_Ks, float* ref_poses, int* ref_rows);
/* network output [qn,7] (quaternion, offset, log2 scale) -> refined poses (float32 values in float64 storage) */
int g6d_glue_apply_refinements(const g6d_glue_views* views, const float* que_pose, const float* que_K, const float* rect,
                               const float* net_out, int qn, double* poses, g6d_stream_t stream);
int g6d_glue_apply_refinements_host(const g6d_glue_views* views, const float* que_pose, const float* que_K, const float* rect,
                                    const float* net_out, int qn, double* poses);
/* ---- the same two refinement steps for several objects in one launch each (an object set; gen6d_b200/objects.py).
 * views [n_obj] (host array, passed to the kernel by value: 1 <= n_obj <= G6D_GLUE_MAX_OBJECTS, every object with the
 * same ref_num).  Rows are object-major: row i = o*rows_per_obj + s is object o on frame s, reading views[o], cams[s]
 * and frame s at frames + s*rows*cols*3, and writing row i of every output, i.e. the per-object calls' outputs
 * concatenated: jobs [n_obj*rows_per_obj*(ref_num+1)], then [n_obj*rows_per_obj, ...].  Every row runs the code of
 * g6d_glue_refine_problems / g6d_glue_apply_refinements and is bit-identical to that call on the object's slice. */
#define G6D_GLUE_MAX_OBJECTS 16
int g6d_glue_refine_problems_objects(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                     const uint8_t* frames, int rows, int cols, const double* poses, int poses_are_f32,
                                     g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect, float* ref_Ks, float* ref_poses,
                                     int* ref_rows, g6d_stream_t stream);
int g6d_glue_refine_problems_objects_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                          const uint8_t* frames, int rows, int cols, const double* poses, int poses_are_f32,
                                          g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect, float* ref_Ks,
                                          float* ref_poses, int* ref_rows);
int g6d_glue_apply_refinements_objects(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                       const float* que_K, const float* rect, const float* net_out, double* poses, g6d_stream_t stream);
int g6d_glue_apply_refinements_objects_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                            const float* que_K, const float* rect, const float* net_out, double* poses);
/* ---- the same two steps on a subset of those rows (a tracker whose sequences are at different points of their chains).
 * views, n_obj, rows_per_obj, cams, frames and the object-major row numbering are those of the *_objects calls; row_idx
 * [n_sel] (int32, device memory for the device calls) lists the rows, in any order, n_sel >= 1.
 * refine_problems_rows: output row j is the problem of poses[row_idx[j]], read with that row's own dtype flag
 * row_f32[row_idx[j]] (uint8 [n_obj*rows_per_obj]; 1: float32 values), into row j of jobs [n_sel*(ref_num+1)], que_K
 * [n_sel,9], ... ref_rows [n_sel,ref_num]; bit-identical to that row of g6d_glue_refine_problems_objects with that flag.
 * apply_refinements_rows: network output row j [7] updates poses[row_idx[j]] in place; unlisted rows are untouched.  Its
 * list must name each row at most once (on the device a row listed twice is a race: undefined result).  The *_host
 * variants reject an index outside [0, n_obj*rows_per_obj), and apply_refinements_rows_host a row listed twice. */
int g6d_glue_refine_problems_rows(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                  const uint8_t* frames, int rows, int cols, const double* poses, const int* row_idx, int n_sel,
                                  const uint8_t* row_f32, g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect, float* ref_Ks,
                                  float* ref_poses, int* ref_rows, g6d_stream_t stream);
int g6d_glue_refine_problems_rows_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const g6d_glue_camera* cams,
                                       const uint8_t* frames, int rows, int cols, const double* poses, const int* row_idx, int n_sel,
                                       const uint8_t* row_f32, g6d_warp_job* jobs, float* que_K, float* que_pose, float* rect,
                                       float* ref_Ks, float* ref_poses, int* ref_rows);
int g6d_glue_apply_refinements_rows(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose, const float* que_K,
                                    const float* rect, const float* net_out, const int* row_idx, int n_sel, double* poses,
                                    g6d_stream_t stream);
int g6d_glue_apply_refinements_rows_host(const g6d_glue_views* views, int n_obj, int rows_per_obj, const float* que_pose,
                                         const float* que_K, const float* rect, const float* net_out, const int* row_idx, int n_sel,
                                         double* poses);
/* ---- checking a pose with the detector on a window around the object (gen6d_b200/verify.py).
 * verify_windows: poses [n_obj*rows_per_obj,12] (float64 storage; poses_are_f32: float32 values), object-major as the
 * *_objects calls take them (row o*rows_per_obj + s with refs[o] and cams[s]; refs is a host array of n_obj <=
 * G6D_GLUE_MAX_OBJECTS) -> rec [n,4] float32 in g6d_det_parse's layout: (cx, cy, s, 1), cx, cy the projected object centre
 * and s the scale_r2q a detection there would need to give this pose (the inverse of g6d_glue_initial_poses, with
 * refs[o].dist[0] / refs[o].f[0]); (0, 0, 1, 0) for a pose whose centre is not in front of the camera or whose values are
 * not finite.  g6d_glue_detection_jobs(rec, frames, window) cuts the windows.
 * verify_judge: rec [n,4] and the detector's records det [n,4] on those windows (x, y, scale, score) -> out [n,5] float32
 * (x, y, scale in the frame, score, offset = |detection - window centre| / (ref_resolution * s)) and lost [n] int32: the
 * record is invalid, use_score and not score >= lost_score, or use_gate and not offset <= lost_gate (NaN is lost). */
int g6d_verify_windows(const double* poses, int poses_are_f32, const g6d_glue_refs* refs, int n_obj, int rows_per_obj,
                       const g6d_glue_camera* cams, float* rec, g6d_stream_t stream);
int g6d_verify_windows_host(const double* poses, int poses_are_f32, const g6d_glue_refs* refs, int n_obj, int rows_per_obj,
                            const g6d_glue_camera* cams, float* rec);
int g6d_verify_judge(const float* rec, const float* det, int n, int window, double ref_resolution, int use_score, double lost_score,
                     int use_gate, double lost_gate, float* out, int* lost, g6d_stream_t stream);
int g6d_verify_judge_host(const float* rec, const float* det, int n, int window, double ref_resolution, int use_score,
                          double lost_score, int use_gate, double lost_gate, float* out, int* lost);
/* ---- temporal smoothing of tracked poses (predict.py:18-26,61-70; utils/base_utils.py:256-265 project_points;
 * utils/pose_utils.py:246-279 pnp).  Per sequence s: project the object's bounding box bbox [8,3] (float32) with the raw
 * pose poses[s] [12] (float64 storage; poses_are_f32: float32 values, projected in float32 like numpy does with
 * predict.py's float32 K) and Ks[s] [9] (float64 values), append the corners to the history ring[s] [num,8,2]
 * (oldest first; count[s] frames held, 0..num, advanced by the call), average the newest count[s] frames with
 * weights [num] (np.exp(-(np.arange(num)/std)**2)[::-1]: oldest first, the newest count[s] of them used) -> avg_pts[s]
 * [8,2] float64, and solve cv2.solvePnP(SOLVEPNP_ITERATIVE) for non-coplanar corners -> smoothed[s] [12] = [R | t]
 * float64.  One thread per sequence.  The *_host variant runs the identical code on host memory and also rejects a
 * count beyond the ring. */
int g6d_track_smooth(const double* poses, int poses_are_f32, const float* bbox, const double* Ks, float* ring, int* count, int num,
                     const double* weights, int S, double* smoothed, double* avg_pts, g6d_stream_t stream);
int g6d_track_smooth_host(const double* poses, int poses_are_f32, const float* bbox, const double* Ks, float* ring, int* count,
                          int num, const double* weights, int S, double* smoothed, double* avg_pts);
/* The same smoothing for n_obj objects tracked through rows_per_obj sequences, rows object-major: row i = o*rows_per_obj
 * + s smooths poses[i] with box bboxes[o] ([n_obj,8,3]) and Ks[s] ([rows_per_obj,9]), into ring[i] ([n_obj*rows_per_obj,
 * num,8,2]), count[i], smoothed[i] and avg_pts[i].  Each row runs g6d_track_smooth's per-sequence code.  One thread per
 * row; the *_host variant also rejects a count beyond the ring. */
int g6d_track_smooth_objects(const double* poses, int poses_are_f32, const float* bboxes, int n_obj, int rows_per_obj, const double* Ks,
                             float* ring, int* count, int num, const double* weights, double* smoothed, double* avg_pts,
                             g6d_stream_t stream);
int g6d_track_smooth_objects_host(const double* poses, int poses_are_f32, const float* bboxes, int n_obj, int rows_per_obj,
                                  const double* Ks, float* ring, int* count, int num, const double* weights, double* smoothed,
                                  double* avg_pts);
/* ---- drawn frames (predict.py:61-72 with utils/draw_utils.py:94-103,274-294 draw_bbox_3d): each destination frame is
 * its source frame with the 3-D boxes of its g6d_draw_box entries drawn one after the other, bit for bit as
 *   img = draw_bbox_3d(img, np.round(project_points(bbox, pose, K)) ..., color)
 * with OpenCV's 8-bit drawing (8 filled red dots of radius 2, then 12 edges of thickness 2; csrc/draw_math.cuh).
 * Source frame i is the uint8 RGB image [rows, cols, 3] at src + offset with row pitch `pitch` (>= 3*cols).  Destination
 * d (a g6d_device_frame row: RGB with any pitch, or NV12 planes with an even size, converted as
 * cv2.cvtColor(COLOR_RGB2YUV_I420) with U and V interleaved; its `offset` is unused) shows source d % n_src and has its
 * size.  Box b projects bboxes[bbox] (float32 [8,3]) with poses[pose] (float64 values [12]; pose_f32: float32 values,
 * projected in float32 as the smoothing projects them, else in float64) and Ks[K] (float64 values [9]); valid >= 0
 * draws it only when ids[valid] >= 0 (a live track of an instance tracker), valid = -1 always; at most
 * G6D_DRAW_MAX_BOXES boxes per destination, drawn in table order.  g6d_draw_check validates HOST copies of the tables
 * (n_poses, n_Ks, n_bboxes, n_ids: the rows each array holds); g6d_draw_boxes reads srcs, boxes and dsts from DEVICE memory
 * (checked by the caller before the upload; max_rows / max_cols bound every destination) and writes every byte of every
 * destination's image; g6d_draw_boxes_host runs the same code on HOST tables and buffers (checked first).
 * g6d_rgb_to_nv12 / _host convert without drawing: the RGB image [rows, cols, 3] (row pitch `pitch`) to the NV12 planes
 * y [rows, cols] (pitch_y) and uv [rows/2, cols] (pitch_uv), rows and cols even. */
#define G6D_DRAW_MAX_BOXES 16
typedef struct g6d_draw_src {
    long long offset, pitch;       /* byte offset from src, row pitch in bytes */
    int rows, cols;
} g6d_draw_src;
typedef struct g6d_draw_box {
    int dst, pose, K, bbox, pose_f32, valid;
    uint8_t color[4];              /* the edges' (R, G, B); [3] unused */
} g6d_draw_box;
int g6d_draw_check(const g6d_draw_src* host_srcs, int n_src, const g6d_draw_box* host_boxes, int n_boxes,
                   const g6d_device_frame* host_dsts, int n_dst, int n_poses, int n_Ks, int n_bboxes, int n_ids);
int g6d_draw_boxes(const uint8_t* src, const g6d_draw_src* srcs, int n_src, const double* poses, const double* Ks,
                   const float* bboxes, const long long* ids, const g6d_draw_box* boxes, int n_boxes,
                   const g6d_device_frame* dsts, int n_dst, int max_rows, int max_cols, g6d_stream_t stream);
int g6d_draw_boxes_host(const uint8_t* src, const g6d_draw_src* host_srcs, int n_src, const double* poses, int n_poses,
                        const double* Ks, int n_Ks, const float* bboxes, int n_bboxes, const long long* ids, int n_ids,
                        const g6d_draw_box* host_boxes, int n_boxes, const g6d_device_frame* host_dsts, int n_dst);
int g6d_rgb_to_nv12(const uint8_t* rgb, long long pitch, int rows, int cols, uint8_t* y, long long pitch_y, uint8_t* uv,
                    long long pitch_uv, g6d_stream_t stream);
int g6d_rgb_to_nv12_host(const uint8_t* rgb, long long pitch, int rows, int cols, uint8_t* y, long long pitch_y, uint8_t* uv,
                         long long pitch_uv);
/* ---- the re-detection step of the multi-instance tracker (gen6d_b200/instance_track.py): M slots per sequence, rows
 * instance-major (row m*S + s is slot m of sequence s; 1 <= M <= G6D_DET_MAX_INSTANCES).  Per sequence s:
 *  1. the track point of each live slot: the object centre (cx, cy, cz) projected with prev[row] [12] and cams[s].K in
 *     fp64, p_i = ((P[i,0]*cx + P[i,1]*cy) + P[i,2]*cz) + P[i,3], q_j = (K[j,0]*p_0 + K[j,1]*p_1) + K[j,2]*p_2,
 *     u = (q_0/q_2, q_1/q_2); cost(t, d) = sqrt(dx*dx + dy*dy) / (ref_resolution * scale_d), (dx, dy) = u - (x_d, y_d)
 *     from det [M*S,4] (x, y, scale, score), for valid detections (valid [M*S]) only; a track with q_2 <= 0 has no pair.
 *  2. greedy matching: repeatedly the pair with cost < gate of smallest cost, ties to the lower slot, then the lower
 *     detection; both leave the pool.
 *  3. a matched track keeps its id and pose, misses = 0; an unmatched one takes a miss and is dropped (live 0, id -1,
 *     dropped[row] = its id) when misses > max_misses.  Unmatched valid detections, in index order, take the lowest
 *     empty slots (det_slot [M*S]: the slot detection d went to, -1 if matched to none and discarded, or invalid);
 *     spawned [M*S] marks them, their ring rows ([M*S,num,8,2]) and count are zeroed, and they get the ids *next_id,
 *     *next_id + 1, ... in ascending (sequence, detection) order (the counter [1] is advanced).
 *  4. every empty slot parks on detection row m of its frame: park[row] = init[row] ([M*S,12], the detections' initial
 *     poses).
 *  5. the chain: work [M*2S,12] holds per slot m the S real rows m*2S + s, then S scratch copies m*2S + S + s; a
 *     continuing track starts from prev (flags0 = 1: float32 values), a spawned one from its detection's initial pose
 *     and an empty slot from its parking pose (flags0 = 0).  Continuing tracks run r refinements, the others F; lists
 *     [max(F,r)*M*S] int32 hold each iteration's M*S rows (entry it*M*S + m*S + s), a row whose chain is complete
 *     replaced by its scratch row.
 * live, ids, misses and park are updated in place.  The device call is one CTA (one thread per sequence, a block scan for
 * the ids): no workspace, no synchronisation, deterministic.  The *_host variant runs the same per-sequence code. */
int g6d_instances_associate(int S, int M, int F, int r, const float* det, const int* valid, const double* init,
                            const g6d_glue_camera* cams, double cx, double cy, double cz, double ref_resolution, double gate,
                            int max_misses, const double* prev, int* live, long long* ids, int* misses, long long* next_id,
                            double* park, float* ring, int* count, int num, double* work, uint8_t* flags0, int* lists,
                            int* det_slot, int* spawned, long long* dropped, g6d_stream_t stream);
int g6d_instances_associate_host(int S, int M, int F, int r, const float* det, const int* valid, const double* init,
                                 const g6d_glue_camera* cams, double cx, double cy, double cz, double ref_resolution, double gate,
                                 int max_misses, const double* prev, int* live, long long* ids, int* misses, long long* next_id,
                                 double* park, float* ring, int* count, int num, double* work, uint8_t* flags0, int* lists,
                                 int* det_slot, int* spawned, long long* dropped);
/* The same association for K objects of an object set with M instance slots each (gen6d_b200/instance_track.py,
 * ObjectSet.instance_tracker()).  Slot group g = m*K + o is instance slot m of object o; det, valid, init, prev, live,
 * ids, misses, park, ring, count, det_slot, spawned and dropped have M*K*S rows, row g*S + s (the layout of
 * ObjectSet.predict_instances' slots on S frames).  work [M*K*2S,12] holds group g's S real rows g*2S + s, then its S
 * scratch copies g*2S + S + s; flags0 has one entry per work row; lists [max(F,r)*M*K*S] has entry (it*M*K + g)*S + s.
 * centers [K,3] float64 are the objects' centres (device memory for the device call, host memory for the *_host one).
 * Each (sequence s, object o) pair is associated as above over object o's M slots, with cams[s] and centers[o], against
 * object o's detections only.  The id counter is shared: the spawned tracks are numbered in ascending (object, sequence,
 * detection) order, so the call equals K calls of g6d_instances_associate on the objects' slices in object order, each
 * continuing the counter.  K = 1 is g6d_instances_associate itself, bit for bit.  One CTA, one thread per (sequence,
 * object) pair; no workspace, no synchronisation.  Needs K >= 1, 1 <= M <= G6D_DET_MAX_INSTANCES and centers. */
int g6d_instances_associate_objects(int S, int K, int M, int F, int r, const float* det, const int* valid, const double* init,
                                    const g6d_glue_camera* cams, const double* centers, double ref_resolution, double gate,
                                    int max_misses, const double* prev, int* live, long long* ids, int* misses, long long* next_id,
                                    double* park, float* ring, int* count, int num, double* work, uint8_t* flags0, int* lists,
                                    int* det_slot, int* spawned, long long* dropped, g6d_stream_t stream);
int g6d_instances_associate_objects_host(int S, int K, int M, int F, int r, const float* det, const int* valid, const double* init,
                                         const g6d_glue_camera* cams, const double* centers, double ref_resolution, double gate,
                                         int max_misses, const double* prev, int* live, long long* ids, int* misses,
                                         long long* next_id, double* park, float* ring, int* count, int num, double* work,
                                         uint8_t* flags0, int* lists, int* det_slot, int* spawned, long long* dropped);
/* The association of g6d_instances_associate_objects for a step in which only some sequences re-detect
 * (gen6d_b200/instance_track.py, the per-sequence schedules).  det_index [S] int32 gives each sequence its row j in a
 * detection batch of D rows per slot group (0 <= j < D, no row twice), or -1 when the sequence does not detect this
 * step; det, valid and init are [M*K*D,...], row g*D + j.  A detecting (sequence, object) pair is associated exactly as
 * g6d_instances_associate_objects does it.  A non-detecting pair only sets up its refinement, as a refine-only step
 * does: its real work row is prev when the slot is live, else park, with its scratch copy; flags0 = live; its chain is r;
 * spawned 0, dropped and det_slot -1; live, ids, misses, park, ring and count are untouched.  det_slot, spawned and
 * dropped have M*K*S rows (det_slot row g*S + s: detection m of sequence s).  The spawned tracks are numbered in
 * ascending (object, sequence, detection) order over the detecting pairs, continuing the shared counter.  In lists,
 * iterations it < r list all M*K*S rows (entry (it*M*K + g)*S + s), then iterations r <= it < F
 * list the M*K*D rows of the detecting sequences only (entry r*M*K*S + ((it - r)*M*K + g)*D + j), a finished chain
 * replaced by its scratch row; a padding row j (used by no sequence) lists the scratch rows of the rank-th
 * non-detecting sequence, rank its rank among the unused rows, so it never touches a row another entry lists.  lists
 * thus has r*M*K*S + max(F - r, 0)*M*K*D entries.  det_index the identity with D = S is g6d_instances_associate_objects
 * bit for bit; every entry -1 (D = 0; det, valid and init may be null) is a refine-only step's set-up.  det_index is
 * device memory for the device call (the caller validates it) and host memory for the *_host one, which rejects
 * out-of-range and repeated rows.  Needs 0 <= D <= S and centers [K,3]. */
int g6d_instances_associate_sequences(int S, int K, int M, int F, int r, int D, const int* det_index, const float* det,
                                      const int* valid, const double* init, const g6d_glue_camera* cams, const double* centers,
                                      double ref_resolution, double gate, int max_misses, const double* prev, int* live,
                                      long long* ids, int* misses, long long* next_id, double* park, float* ring, int* count,
                                      int num, double* work, uint8_t* flags0, int* lists, int* det_slot, int* spawned,
                                      long long* dropped, g6d_stream_t stream);
int g6d_instances_associate_sequences_host(int S, int K, int M, int F, int r, int D, const int* det_index, const float* det,
                                           const int* valid, const double* init, const g6d_glue_camera* cams, const double* centers,
                                           double ref_resolution, double gate, int max_misses, const double* prev, int* live,
                                           long long* ids, int* misses, long long* next_id, double* park, float* ring, int* count,
                                           int num, double* work, uint8_t* flags0, int* lists, int* det_slot, int* spawned,
                                           long long* dropped);
/* A verifying instance-tracking step's slot update (row f21), per row i of n = M*K*S (the association's layout):
 * dropped[i] = -1; then, when verified[i] and live[i], a row judged lost (lost[i] != 0, g6d_verify_judge) takes a miss
 * and is dropped past max_misses exactly as the association drops an unmatched track (live 0, ids -1, misses 0, its id
 * in dropped[i]), and a row judged found restarts its misses.  Empty slots and unverified rows (verified[i] == 0: a
 * sequence that re-detected this step, or a padding row) are untouched.  live, ids and misses are updated in place. */
int g6d_instances_verify_update(int n, const int* lost, const int* verified, int max_misses, int* live, long long* ids, int* misses,
                                long long* dropped, g6d_stream_t stream);
int g6d_instances_verify_update_host(int n, const int* lost, const int* verified, int max_misses, int* live, long long* ids,
                                     int* misses, long long* dropped);
/* (x - mean) / std on f32 [n_pixels, in_c] -> [n_pixels, out_c] (in_c, out_c in {3,4})
 * (network/detector.py:189, selector.py:115, refiner.py:65) */
int g6d_imagenet_norm(const float* in, float* out, long long n_pixels, int in_c, int out_c, g6d_stream_t stream);
/* NCHW [N,C,H,W] -> channels-last [N,H,W,out_c] (channels >= C zero) and back */
int g6d_nchw_to_nhwc(const float* in, float* out, int N, int C, int H, int W, int out_c, g6d_stream_t stream);
int g6d_nhwc_to_nchw(const float* in, float* out, int N, int C, int H, int W, int in_c, g6d_stream_t stream);
/* F.interpolate(mode='bilinear', align_corners=False) on channels-last data
 * (network/detector.py:240,243; network/refiner.py:75-76).  Output rows have `out_cstride`
 * channels and the C results land at channel offset `out_coff` (writes into concat buffers). */
int g6d_resize_bilinear(const float* in, float* out, int N, int Hi, int Wi, int Ho, int Wo, int C,
                        int out_cstride, int out_coff, g6d_stream_t stream);
/* F.interpolate default (nearest): src = floor(dst * in / out) (network/detector.py:201) */
int g6d_resize_nearest(const float* in, float* out, int N, int Hi, int Wi, int Ho, int Wo, int C, g6d_stream_t stream);
/* MaxPool 2x2 stride 2 over (H, W), output floor(H/2) x floor(W/2) like torch (VGG M layers;
 * selector MaxPool3d((1,2,2))) */
int g6d_maxpool2x2(const float* in, float* out, int N, int H, int W, int C, g6d_stream_t stream);
/* F.normalize(dim=1) == x / max(||x||_2, eps) over the channel axis of each row
 * (network/selector.py:118, network/refiner.py:69-71) */
int g6d_l2norm_channels(const float* in, float* out, long long rows, int C, float eps, g6d_stream_t stream);
/* y = act(x * scale[g,c] + shift[g,c]); rows_per_group consecutive rows share a group.
 * act: 0 none, 1 ReLU.  Materialises an InstanceNorm (+ReLU) where a consumer needs it.
 * Input rows have `in_cstride` channels (C taken from offset in_coff); same for output. */
int g6d_affine_act(const float* in, float* out, long long rows, int C, long long rows_per_group,
                   const float* scale, const float* shift, int act,
                   int in_cstride, int in_coff, int out_cstride, int out_coff, g6d_stream_t stream);
/* mean over `spatial` consecutive rows of act(x*scale+shift) -> [groups_of_rows, C]
 * (AvgPool3d((1,4,4)) of network/selector.py:76 applied after the fused IN+ReLU). */
int g6d_avgpool_affine(const float* in, float* out, long long n_out, int spatial, int C, long long rows_per_group,
                       const float* scale, const float* shift, int act, g6d_stream_t stream);
int g6d_add(const float* a, const float* b, float* out, long long n, g6d_stream_t stream);

/* ------------------------------------------------------------------ instance-norm stats ---- */
/* InstanceNorm{1,2,3}d(affine=False, eps) statistics (biased variance) of a channels-last
 * tensor: `rows` rows of C channels (taken at channel offset `coff` of rows `cstride` wide),
 * `rows_per_group` consecutive rows form one (sample, *) group.  Writes scale = rstd and
 * shift = -mean*rstd, each [groups, C], for consumption by prologues / g6d_affine_act.
 * ws: 2*groups*C doubles of workspace.  (network/selector.py:27-87, refiner.py:18-22,82-86) */
int g6d_instnorm_stats(const float* x, long long rows, int C, int cstride, int coff, long long rows_per_group,
                       float eps, float* scale, float* shift, double* ws, g6d_stream_t stream);

/* The two halves of g6d_instnorm_stats, for statistics that span GPUs (reference-sharded selector):
 * partial writes ws[g,c] = (sum, sum of squares) as doubles; the caller all-reduces ws across ranks;
 * finalize turns it into scale/shift with `count` = total rows per group over all ranks. */
int g6d_instnorm_partial(const float* x, long long rows, int C, int cstride, int coff, long long rows_per_group,
                         double* ws, g6d_stream_t stream);
int g6d_instnorm_finalize(const double* ws, long long groups, int C, long long count, float eps, float* scale,
                          float* shift, g6d_stream_t stream);

/* ------------------------------------------------------------------ convolution ------------ */
typedef struct g6d_conv_desc {
    int B, D, H, W, Cin;      /* input [B,D,H,W,*]; channels [in_coff, in_coff+Cin) of rows in_cstride wide */
    int in_cstride, in_coff;
    int Cout, kd, kh, kw;
    int stride;               /* same in all spatial dims that have k>1 */
    int pd, ph, pw;           /* zero padding */
    int Do, Ho, Wo;           /* output dims (validated) */
    int out_cstride, out_coff;
    int prologue;             /* G6D_PRO_* applied to in-bounds input elements before the MAC */
    long long group_rows;     /* G6D_PRO_AFFINE*: input batch items per norm group */
    int act;                  /* G6D_ACT_* epilogue after bias */
    int max_chain_k;          /* tensor-core path: 0 = default; > 0 bounds the K-elements accumulated into one
                                 accumulator (longer problems are split and summed in fp32 round-to-nearest).  The tensor
                                 core truncates on every accumulate, which biases long chains of SAME-SIGN products
                                 (detector correlation: post-ReLU features x post-ReLU features) by ~5e-8 per step. */
    int plan_rows;            /* 0 = M.  > 0: every K-split count that depends on the number of output rows (the tensor-core
                                 kernels' fill-the-GPU splits, the FFMA split-K heuristic) is chosen as for a call of
                                 plan_rows rows, a multiple of Do*Ho*Wo.  A call over Q groups of rows then sums every
                                 output element in the same chains as the call over one group (bit-identical). */
} g6d_conv_desc;

#define G6D_PRO_NONE 0
#define G6D_PRO_AFFINE 1        /* x*scale[g,c] + shift[g,c]          (folded InstanceNorm)        */
#define G6D_PRO_AFFINE_RELU 2   /* relu(x*scale[g,c] + shift[g,c])    (folded InstanceNorm + ReLU) */
#define G6D_PRO_CORR 3          /* x*scale[pos,c] + shift[c]: selector correlation volume
                                   q (.) ref with the first InstanceNorm3d folded in            */
#define G6D_ACT_NONE 0
#define G6D_ACT_RELU 1
#define G6D_ACT_LEAKY01 2

/* Implicit-GEMM convolution (1x1 ... 3x3x3, stride 1/2) with fused prologue/bias/activation.
 * Replaces F.conv2d / Conv3d call sites: VGG (pretrain_models.py:17-31), detector correlation
 * (detector.py:222-224, reference features as kernels) and heads (:159-184), selector towers
 * (selector.py:27-77) and 1x1 convs (:79-111), refiner feature/volume nets (refiner.py:24-52,
 * 88-134).  w: packed [K, Cout]; bias may be NULL.  ws: split-K workspace of
 * g6d_conv_workspace_bytes(desc) bytes (may be NULL when that returns 0). */
int g6d_conv(const g6d_conv_desc* desc, const float* x, const float* w, const float* bias,
             const float* pro_scale, const float* pro_shift, float* y, void* ws, g6d_stream_t stream);
long long g6d_conv_workspace_bytes(const g6d_conv_desc* desc);
/* First VGG block in one kernel: 3x3 conv 4 -> 64 (RGB + zero channel, BN folded) + ReLU + 2x2 max-pool
 * (network/pretrain_models.py:17-31 features[0:4]); x [B,H,W,4], w packed [36,64] (g6d_pack_conv_weight),
 * y [B,H/2,W/2,64]; H, W even.  Bit-identical to g6d_conv -> ReLU -> g6d_maxpool2x2. */
int g6d_vgg_first_block(const float* x, const float* w, const float* bias, float* y, int B, int H, int W,
                        g6d_stream_t stream);
/* [Cout, Cin, kd, kh, kw] (reference layout) -> [taps*Cin_pad, ldw] with ldw = Cout rounded up
 * to 4; channels [Cin, Cin_pad) and columns [Cout, ldw) are zero; optional per-Cout scale
 * (eval-mode BatchNorm fold). */
int g6d_pack_conv_weight(const float* w, float* out, int Cout, int Cin, int Cin_pad, int taps,
                         const float* cout_scale, g6d_stream_t stream);
/* ---- tensor-core path (wgmma, three-term operand split: fp32-faithful on the tensor pipe) --------
 * Same contract as g6d_conv, for problems g6d_conv_tc_supported accepts (Cin a multiple of the
 * kind's K-block, Cout >= 16, and every other descriptor check g6d_conv_tc makes).
 * A*B ~= A_hi*B_hi + A_hi*B_lo + A_lo*B_hi with 11-bit-significand halves; `kind` selects their container:
 *   G6D_TC_TF32: hi = tf32(x), lo = tf32(x - hi), fp32 arrays, K-block 32, tf32 wgmma;
 *   G6D_TC_F16 : hi = fp16(x), lo = fp16((x - hi) * 2^11), __half arrays, K-block 64, f16 wgmma (twice
 *                the K per instruction and per operand byte; the kernels undo the 2^11 in the epilogue).
 *                Range contract: |x| <= 65504 (saturating), full accuracy for |x| >= 6.1e-5.
 * Weights are pre-split [w_rows >= Cout, K] K-major arrays (K = tap*Cin + c), see
 * g6d_pack_conv_weight_tc / g6d_split_operand.  A tiles are gathered + transformed + split by
 * producer warps, B tiles arrive by TMA, accumulators live in the consumer warpgroup's registers. */
#define G6D_TC_TF32 0
#define G6D_TC_F16 1
int g6d_conv_tc_supported(const g6d_conv_desc* desc, int kind);
/* debug probe: D[64x32] = A[shift..shift+64) x I for a row-shifted SWIZZLE_128B descriptor (mode: base_offset rule) */
int g6d_debug_desc_shift(float* out, int shift, int mode, g6d_stream_t stream);
/* debug: host_out8[0] != 0 if a pipeline wait inside g6d_conv_tc timed out (kernel bailed out); syncs */
int g6d_conv_tc_debug(int* host_out8);
long long g6d_conv_tc_workspace_bytes(const g6d_conv_desc* desc, int kind);
/* stats (optional, may be NULL): fused InstanceNorm statistics of the OUTPUT.  [M / stats_rows, Cout, 2] doubles
 * receive, per group of stats_rows consecutive output rows and channel, (sum y, sum y^2) -- what
 * g6d_instnorm_partial computes in a separate pass over y; feed them to g6d_instnorm_finalize.  Zeroed by
 * the call.  Allowed when g6d_conv_tc_stats_supported (groups made of whole 32-row slices / image planes). */
int g6d_conv_tc_stats_supported(const g6d_conv_desc* desc, int kind, long long stats_rows);
/* What g6d_conv_tc would launch for desc (no launch): out4 = {kernel (0 persistent, 1 A-reuse), BN, K splits,
 * split input (1: the persistent kernel loads A by TMA im2col from an fp16 hi/lo copy of x that the call writes
 * into the workspace -- fp16 kind, stride 1, no prologue (see G6D_TC_PRENORM), 2-D multi-tap (3-D: G6D_TC_REUSE_IM2COL))}.  G6D_EINVAL with g6d_conv_tc's
 * message when the descriptor is rejected. */
int g6d_conv_tc_plan(const g6d_conv_desc* desc, int kind, int* out4);
int g6d_conv_tc(const g6d_conv_desc* desc, const float* x, const void* w_hi, const void* w_lo, int w_rows, int kind,
                const float* bias, const float* pro_scale, const float* pro_shift, float* y, void* ws,
                double* stats, long long stats_rows, g6d_stream_t stream);
/* The same three entry points with option flags; flags = 0 is exactly g6d_conv_tc_plan / _workspace_bytes / g6d_conv_tc.
 * G6D_TC_PRENORM: where the split input would apply if the layer had no prologue (fp16 kind, persistent kernel, 2-D,
 * stride 1, multi-tap), it applies with the prologue too: the call's split pass writes prologue(x) split into hi/lo,
 * and the kernel loads A from it by TMA im2col.  Bit-identical to the producer warps (selector towers: their 8x8
 * and 4x4 InstanceNorm-ed layers).  Elsewhere the flag changes nothing.
 * G6D_TC_REUSE_IM2COL: a layer the A-reuse kernel would take that could have the split input (as above, with
 * G6D_TC_PRENORM where it has a prologue) runs on the persistent kernel with TMA im2col A instead, in the A-reuse
 * kernel's K order and K splits: bit-identical outputs.  It also lets 3-D layers (and 2-D planes stacked in D)
 * have the split input on the persistent kernel, through a rank-5 im2col map; a volume whose box corners leave
 * [-16, 15] (pad > 16 or kernel > 16) keeps the gathering kernels.  Elsewhere (1x1, stride 2, tf32) it changes nothing.
 * G6D_TC_FOLD_SPLITS: a persistent-kernel plan with the split input and K splits whose tiles keep the GPU about as busy
 * without the splits' parallelism (the wave count grows by at most 15 %) runs each tile's splits back to back in one CTA,
 * which keeps their running sum in registers and stores it in the split-K reduce's order: bit-identical outputs, no fp32
 * partials in the workspace and no reduce pass.  The splits and their
 * K-blocks are unchanged.  With stats the moments are taken from y afterwards in the reduce's grouping (only the order
 * of the fp64 additions differs).  Elsewhere the flag changes nothing.
 * Other bits: G6D_EINVAL. */
#define G6D_TC_PRENORM 1
#define G6D_TC_REUSE_IM2COL 4
#define G6D_TC_FOLD_SPLITS 32
int g6d_conv_tc_plan_ex(const g6d_conv_desc* desc, int kind, int flags, int* out4);
/* g6d_conv_tc_plan_ex's four values, then folded (1: G6D_TC_FOLD_SPLITS applies), then x reuse (1: one im2col A box per
 * row of kw taps, read through row-shifted descriptors; planned for the A-reuse K order at BN 64); the first min(n, 6)
 * are written. */
int g6d_conv_tc_plan_v2(const g6d_conv_desc* desc, int kind, int flags, int* out, int n);
long long g6d_conv_tc_workspace_bytes_ex(const g6d_conv_desc* desc, int kind, int flags);
int g6d_conv_tc_ex(const g6d_conv_desc* desc, const float* x, const void* w_hi, const void* w_lo, int w_rows, int kind,
                   const float* bias, const float* pro_scale, const float* pro_shift, float* y, void* ws,
                   double* stats, long long stats_rows, int flags, g6d_stream_t stream);
/* [Cout, Cin, taps] (reference layout) -> hi/lo [rows_pad, taps*Cin_pad] of the given kind; optional BN-fold scale */
int g6d_pack_conv_weight_tc(const float* w, void* out_hi, void* out_lo, int Cout, int Cin, int Cin_pad, int taps,
                            int rows_pad, const float* cout_scale, int kind, g6d_stream_t stream);
/* hi/lo split of a K-major fp32 operand [rows, K] into the given kind (detector reference features as
 * kernels).  G6D_TC_F16 operands use the kernels' K order inside every 64-element block (position p holds
 * source element 4*(p/8) + p%8 for p%8 < 4, else 32 + 4*(p/8) + p%8 - 4: it keeps the activation gathers
 * coalesced); K % 64 == 0.  g6d_pack_conv_weight_tc applies the same order. */
int g6d_split_operand(const float* in, void* hi, void* lo, long long n, int kind, g6d_stream_t stream);
/* [rows, K] row-major -> [K, rows] (detector reference features [rfn,k,k,512] -> correlation kernels) */
int g6d_transpose2d(const float* in, float* out, int rows, int cols, g6d_stream_t stream);
/* y[m, n] = act(sum_k x[m,k] w[n,k] + b[n]) for small m (<= 8): weight-bandwidth bound
 * (refiner regressor fc 32768->512, refiner.py:156-159).  w is [N, K] row-major. */
int g6d_linear_smallm(const float* x, const float* w, const float* bias, float* y, int M, int N, int K, int act,
                      g6d_stream_t stream);

/* ------------------------------------------------------------------ detector ---------------- */
#define G6D_DET_MAX_SCALES 8
typedef struct g6d_det_maps {
    int n_scales;
    int rfn, hs, ws;                 /* output resolution (h/8, w/8) */
    const float* map[G6D_DET_MAX_SCALES][3]; /* raw correlation [qn, Hl, Wl, rfn], level l = 0,1,2 */
    int H[G6D_DET_MAX_SCALES][3];
    int W[G6D_DET_MAX_SCALES][3];
    float mu[3], inv_sigma[3], clip; /* vgg_score_stats / vgg_score_max */
} g6d_det_maps;
/* Fuses detector.py:225-226 (nearest x2/x4), :207-216 (normalise + clip), :243 (bilinear resize
 * to (hs,ws)), :245 (stack), :246 score_conv (1x1x1 Conv3d 3S->64, ReLU, 64->64) and :247 (max
 * over references).  w1 [64, 3S] (channel = scale*3 + level), w2 [64, 64].  out [qn, hs, ws, 64].
 * 1 <= n_scales <= 6; rfn, hs, ws > 0; every map non-null.  Level l of scale s must have exactly
 * H[s][0] >> l rows and W[s][0] >> l columns, i.e. H[s][l] << l == H[s][0] and W[s][l] << l == W[s][0]
 * (the nearest x2^l upsampling of detector.py:225-226 must land on the level-0 grid); otherwise
 * G6D_EINVAL. */
int g6d_det_score_fuse(const g6d_det_maps* host_maps, int qn, const float* w1, const float* b1,
                       const float* w2, const float* b2, float* out, g6d_stream_t stream);
/* Row-decomposed form of the sliding inner product of detector.py:222-224: with the reference features
 * [rfn, k, k, C] packed as a 1 x k convolution of k*rfn output channels (channel = ky*rfn + r, zero
 * padding k/2 in both axes, so the result has H + k - 1 rows), partial [qn, H+k-1, W, k*rfn] holds the
 * contribution of kernel row ky to input row y'; out[q,y,x,r] = sum_ky partial[q, y+ky, x, ky*rfn + r]
 * is the k x k correlation map [qn, H, W, rfn].  rfn % 4 == 0. */
int g6d_det_corr_rowsum(const float* partial, float* out, int qn, int H, int W, int k, int rfn, g6d_stream_t stream);
/* g6d_det_corr_rowsum for n_obj objects at once: partial [qn, H+k-1, W, n_obj*k*rfn] is ONE 1 x k convolution with
 * the objects' kernels concatenated along its output channels (channel = (obj*k + ky)*rfn + r);
 * out[obj,q,y,x,r] = sum_ky partial[q, y+ky, x, (obj*k + ky)*rfn + r] is object-major [n_obj, qn, H, W, rfn], the k
 * rows added in g6d_det_corr_rowsum's order.  k = 1 regroups a direct correlation [qn, H, W, n_obj*rfn].
 * n_obj > 0, rfn % 4 == 0. */
int g6d_det_corr_rowsum_objects(const float* partial, float* out, int n_obj, int qn, int H, int W, int k, int rfn,
                                g6d_stream_t stream);
/* detector.py:85-121: first-max flat argmax of scores [qn,hs,ws,1], then
 * position = ((x,y) + offset[y,x] + 0.5)*pool - 0.5, scale = 2**scale[y,x].
 * out [qn, 4] = (x, y, scale, score); out_idx [qn] (int64 flat index y*ws + x). */
int g6d_det_parse(const float* scores, const float* scales, const float* offsets, int qn, int hs, int ws,
                  int pool_ratio, float* out, long long* out_idx, g6d_stream_t stream);
/* Every instance of the object in a frame: up to max_inst peaks of each of n_maps score maps (the maps of g6d_det_parse,
 * qn -> n_maps), chosen by greedy non-maximum suppression.  Order: g6d_det_parse's (NaN is the maximum, ties go to the
 * lower flat index).  Cell i is a peak when no other cell within Chebyshev distance `radius` (window clipped at the
 * border) beats it; radius 0 makes every cell a peak.  A cell decodes as g6d_det_parse decodes its argmax (x, y, scale,
 * score), and its box is the square of side box_size*scale centred at (x, y).  IoU is fp32 in a fixed order
 *   iw = max(min(x1a,x1b) - max(x0a,x0b), 0), ih likewise, inter = iw*ih, iou = inter / ((area_a + area_b) - inter),
 * never contracted; a box is suppressed when its IoU with a kept box is strictly greater than nms_iou.
 * Instance 0 is the argmax, always kept, bit-identical to g6d_det_parse's row.  Instance m > 0 is the best remaining peak
 * with score >= min_score that no kept box suppresses; the rounds stop after max_inst kept peaks or when none is left.
 * valid = kept and score >= min_score.  An invalid instance 0 (below min_score, or NaN) ends its map, so the valid
 * instances always form a prefix and count[j] is their number.  Rows past the kept ones repeat instance 0 with valid 0.
 * Outputs are instance-major: row m*n_maps + j is instance m of map j: det_out [max_inst, n_maps, 4] (x, y, scale,
 * score), idx_out [max_inst, n_maps] (flat index y*ws + x), valid_out [max_inst, n_maps], count_out [n_maps].
 * 1 <= max_inst <= G6D_DET_MAX_INSTANCES, 0 <= radius <= G6D_DET_MAX_PEAK_RADIUS, 0 <= nms_iou <= 1, box_size > 0, finite,
 * min_score not NaN (-inf: no threshold), pool_ratio > 0.  No workspace, no synchronisation.
 * The *_host variant runs the same selection on host memory; its decode uses std::fma and libm exp2f, so its scale can
 * differ by a few ulp from the device's ex2.approx (and with it an IoU, near the threshold). */
#define G6D_DET_MAX_INSTANCES 16
#define G6D_DET_MAX_PEAK_RADIUS 3
int g6d_det_parse_peaks(const float* scores, const float* scales, const float* offsets, int n_maps, int hs, int ws,
                        int pool_ratio, int max_inst, int radius, float nms_iou, float box_size, float min_score,
                        float* det_out, long long* idx_out, int* valid_out, int* count_out, g6d_stream_t stream);
int g6d_det_parse_peaks_host(const float* scores, const float* scales, const float* offsets, int n_maps, int hs, int ws,
                             int pool_ratio, int max_inst, int radius, float nms_iou, float box_size, float min_score,
                             float* det_out, long long* idx_out, int* valid_out, int* count_out);
/* Detections from caller-supplied boxes, in g6d_det_parse_peaks' layout, so another detector's boxes replace the score
 * maps and peaks.  Map j (one (frame, object) pair, j = o*qn + f) has its own list boxes[j] of N rows (x0, y0, x1, y1,
 * score), of which the first counts[j] (clamped to [0, N]) are read.  A box is usable when its five values are finite,
 * x1 > x0 and y1 > y0; others are skipped.  The usable boxes are ordered by score descending, ties to the lower index,
 * and the first max_inst become instances 0.. of map j, each the record (fp32, round to nearest, never contracted)
 *   x = (x0 + x1) * 0.5, y = (y0 + y1) * 0.5, scale = max(x1 - x0, y1 - y0) * inv_box_size, score
 * i.e. the square on the box's longer side, whose side is box_size * scale (inv_box_size = 1 / ref_resolution).  As in
 * g6d_det_parse_peaks, the valid rows form a prefix, count_out[j] is their number and rows past it repeat row 0 with
 * valid 0.  A map with no usable box gets row 0 = (0, 0, 1, -inf), valid 0, count 0.  Outputs are instance-major:
 * det_out [max_inst, n_maps, 4], valid_out [max_inst, n_maps], count_out [n_maps].  1 <= N <= G6D_DET_MAX_BOXES,
 * 1 <= max_inst <= G6D_DET_MAX_INSTANCES, inv_box_size > 0 and finite.  No workspace, no synchronisation.  The *_host
 * variant writes the same bytes from host memory. */
#define G6D_DET_MAX_BOXES 256
int g6d_det_from_boxes(const float* boxes, const int* counts, int n_maps, int N, int max_inst, float inv_box_size,
                       float* det_out, int* valid_out, int* count_out, g6d_stream_t stream);
int g6d_det_from_boxes_host(const float* boxes, const int* counts, int n_maps, int N, int max_inst, float inv_box_size,
                            float* det_out, int* valid_out, int* count_out);

/* ------------------------------------------------------------------ selector ---------------- */
/* Load-time sums over the reference stack ref [S, P, C]: sum_s ref and sum_s ref^2, as doubles
 * [P, C] each.  They give the first InstanceNorm3d's statistics of the correlation volume in
 * closed form at query time (SURVEY.md 8a S2 note). */
int g6d_sel_ref_sums(const float* ref, int S, int P, int C, double* sum1, double* sum2, g6d_stream_t stream);
/* From q [P, C] and the sums: scale[p,c] = q[p,c]*rstd_c, shift[c] = -mean_c*rstd_c, the
 * G6D_PRO_CORR prologue operands of the first tower conv (selector.py:28,49,63 InstanceNorm3d
 * over (S,h,w) of que*ref). */
int g6d_sel_corr_prologue(const float* q, const double* sum1, const double* sum2, int S, int P, int C, float eps,
                          float* scale, float* shift, g6d_stream_t stream);
/* The rotated-similarity score, selector.py:183-186,192-194: s[p] = sum_c q[p,c]*ref[s,p,c];
 * score[s] = sum_p s[p]^2 / max_p s[p].  ref [S, P, C] is streamed once from HBM. */
int g6d_sel_corr_score(const float* ref, const float* q, int S, int P, int C, float* score, g6d_stream_t stream);
/* The same score for the three pyramid levels in one streaming pass (what select_que_imgs uses):
 * score [3, S]; ws: g6d_sel_corr_score3_workspace_bytes(S, P0, P1, P2) bytes (per-location inner
 * products, L2-resident).  counters: 3*S ints, one per (level, slice), ZERO on entry and left zero on
 * exit (allocate + clear once, reuse for every call on the same stream): the CTA that completes the last
 * location of a slice reduces it, so the whole op is one launch.  counters == NULL: two launches. */
long long g6d_sel_corr_score3_workspace_bytes(int S, int P0, int P1, int P2);
int g6d_sel_corr_score3(const float* ref0, const float* ref1, const float* ref2, const float* q0, const float* q1,
                        const float* q2, int S, int P0, int P1, int P2, int C, float* score, float* ws, int* counters,
                        g6d_stream_t stream);
/* vp_norm (InstanceNorm2d(3), selector.py:78,201): normalise each of the L score rows [L, n]
 * (biased var, eps) and scatter into feats[n, cstride] at channel coff + l. */
/* (channels [coff + L, cstride) of every feats row -- padding that the consumer multiplies by zero weights -- are set to 0) */
int g6d_sel_vp_norm(const float* score, int L, int n, float eps, float* feats, int cstride, int coff,
                    g6d_stream_t stream);
/* selector.py:203-204: out[r,c] = max_a x[r,a,c] + embed[r,c] */
int g6d_sel_max_angle_add(const float* x, const float* embed, float* out, int rfn, int an, int C, g6d_stream_t stream);
/* attention.py:4-17 with the reference's channel->(d, head) mapping c = d*heads + head:
 * q,k,v [n, C] -> out [n, C]; softmax(q_h^T k_h / sqrt(C/heads)) over keys.  n <= 8192, and a block keeps
 * its n probabilities and its C/heads query values in shared memory next to a 32-float reduction buffer, all
 * within the 48 KB a kernel gets without opting in: n + C/heads <= G6D_ATTENTION_MAX_SMEM_FLOATS. */
#define G6D_ATTENTION_MAX_SMEM_FLOATS (12288 - 32)
int g6d_attention(const float* q, const float* k, const float* v, float* out, int n, int C, int heads,
                  g6d_stream_t stream);
/* The same attention over HEAD-MAJOR channels (c = head*64 + d): the layout a caller gets for free by
 * permuting the output rows of conv_query / conv_key / conv_feats (and the input columns of conv_merge)
 * once at pack time.  Tiled (8 queries x 1 head per block, K / V tiles staged in shared memory by coalesced
 * loads): what the selector uses, and what keeps the replicated tail of a reference-sharded selector
 * (n = all references over all GPUs) cheap.  n <= 2048, C = heads * 64. */
int g6d_attention_headmajor(const float* q, const float* k, const float* v, float* out, int n, int C, int heads,
                            g6d_stream_t stream);
/* nn.LayerNorm(C) over the channel axis of each row (attention.py:19-26) */
int g6d_layernorm(const float* x, const float* gamma, const float* beta, float* out, int rows, int C, float eps,
                  g6d_stream_t stream);
/* selector.py:172-175: idx = first argmax of logits [qn, rfn]; out [qn,2] = (angle[idx], logit[idx]) */
int g6d_sel_parse(const float* logits, const float* angles, int qn, int rfn, long long* out_idx, float* out,
                  g6d_stream_t stream);

/* ------------------------------------------------------------------ refiner ----------------- */
/* refiner.py:183-247 + operator.py:4-17: for every voxel of the sn^3 unit-cube grid rotated by
 * the input pose (row vector @ R_in, R_in = que_poses[:, :3, :3]), project into each of the R
 * reference views and the query view (P = K @ pose), bilinear-sample (zeros padding,
 * align_corners=False) the C-channel feature maps, and write mean / unbiased std over the
 * references and the query sample.
 *   ref_feats [Q, R, fh, fw, C], que_feats [Q, fh, fw, C]
 *   ref_Ks [Q, R, 3, 3], ref_poses [Q, R, 3, 4], que_Ks [Q, 3, 3], que_poses [Q, 3, 4]
 *   mean_in [Q, sn^3, 2C]: channels [0,C) mean, [C,2C) query sample;  stdv [Q, sn^3, C]
 * img_h/img_w: the image size the projections refer to (128), NOT the feature size. */
int g6d_ref_volume_fill(const float* ref_feats, const float* que_feats, const float* ref_Ks,
                        const float* ref_poses, const float* que_Ks, const float* que_poses, int Q, int R,
                        int fh, int fw, int C, int sn, int img_h, int img_w, float* mean_in, float* stdv,
                        g6d_stream_t stream);
/* refiner.py:161-166 tail: r = normalize(x Wr^T + br) (4), t (2), s (1) from x [M,512];
 * w [7, K] rows = fcr(4), fct(2), fcs(1).  out [M, 7] = (qw,qx,qy,qz, tx,ty, log2 scale). */
int g6d_ref_pose_heads(const float* x, const float* w, const float* b, float* out, int M, int K, g6d_stream_t stream);

/* ------------------------------------------------------------------ evaluation (row f4) ---- */
/* utils/pose_utils.py:149-158,192-196 (compute_pose_errors / the symmetric branch of
 * compute_metrics_impl) with utils/base_utils.py:256-265 project_points and :390-394: for each of
 * n_poses (predicted, ground-truth) pairs, out[p] = (mean reprojection error in pixels, mean 3-D
 * point error = ADD, mean closest-point error = ADD-S or NaN when symmetric == 0) over the n_pts
 * object points.  pts [n_pts,3], poses [n_poses,3,4], Ks [n_poses,3,3], out [n_poses,3], all f32 on
 * the device; ws: g6d_pose_errors_workspace_bytes(n_pts, n_poses) bytes. */
long long g6d_pose_errors_workspace_bytes(int n_pts, int n_poses);
int g6d_pose_errors(const float* pts, int n_pts, const float* poses_pr, const float* poses_gt, const float* Ks,
                    int n_poses, int symmetric, float* out, void* ws, g6d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GEN6D_B200_H */
