/*
 * viwb.h -- C ABI of the H100-native sliding-window backend ("viwb") for VIW-Fusion's vins_estimator.
 *
 * This is the drop-in boundary of SURVEY.md section 8(b).  The reference has no FFI layer: its boundary
 * is source level (estimator.cpp includes <ceres/ceres.h>; feature_tracker.cpp calls
 * cv::calcOpticalFlowPyrLK).  A replacement therefore has two faces:
 *   (1) a C++ header shim that reproduces the ceres:: subset used by Estimator::optimization()
 *       (viw-fusion_b200/host/ceres_shim.hpp) and lowers a ceres::Problem to the tables below;
 *   (2) this C ABI, which is what the shim, the Python ctypes binding, the tests and bench.py call.
 *
 * Every entry point cites the reference interface it replaces (paths relative to
 * VIW-Fusion's vins_estimator/src).  Plain C structs, caller-owned host buffers, int return codes
 * (0 ok, <0 error), no exceptions, a context is single-threaded (one per calling thread).
 *
 * The same POD problem description is consumed by the CPU oracle (oracle/viw_oracle.h) so that the
 * parity tests feed identical bytes to both sides.  The oracle is test infrastructure only.
 */
#ifndef VIWB_H
#define VIWB_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * State layout (estimator/estimator.h:191-204: para_Pose, para_SpeedBias, para_Ex_Pose, para_Ex_Pose_wheel,
 * para_plane_R, para_plane_Z, para_Ix_s{x,y,w}_wheel, para_Td, para_Td_wheel, para_Feature).
 *
 * One window's parameter blocks live in ONE flat double array:
 *   state[0 .. VIWB_STATE_FIXED)            the 32 "fixed" blocks below (always laid out, present or not)
 *   state[VIWB_STATE_FIXED + k]             inverse depth of landmark k  (para_Feature[k][0])
 * Pose blocks are [px,py,pz,qx,qy,qz,qw] (estimator.cpp:1159-1166), speed-bias blocks [v,ba,bg]
 * (:1170-1180), plane_R is [qx,qy,qz,qw] (:1209-1213).
 * ---------------------------------------------------------------------------------------------- */
#define VIWB_WINDOW_SIZE 10                 /* parameters.h:25 WINDOW_SIZE */
#define VIWB_NUM_FRAMES 11                  /* WINDOW_SIZE + 1 */
#define VIWB_MAX_LANDMARKS 1000             /* parameters.h:26 NUM_OF_F */
#define VIWB_NUM_FIXED_BLOCKS 32
#define VIWB_STATE_FIXED 207                /* doubles in the fixed part of the state */
#define VIWB_TANGENT_FIXED 192              /* tangent (local) dimension of the fixed part */
#define VIWB_MAX_PRIOR_DIM 200              /* n of the marginalization prior (marg. local size rule) */

enum viwb_block_id {
    VIWB_BLK_POSE0 = 0,        /* 0..10  para_Pose[i]            size 7, tangent 6 */
    VIWB_BLK_SPEEDBIAS0 = 11,  /* 11..21 para_SpeedBias[i]       size 9 */
    VIWB_BLK_EX_POSE0 = 22,    /* 22,23  para_Ex_Pose[c]         size 7, tangent 6 */
    VIWB_BLK_EX_POSE1 = 23,
    VIWB_BLK_EX_WHEEL = 24,    /* para_Ex_Pose_wheel[0]          size 7, tangent 6 */
    VIWB_BLK_PLANE_R = 25,     /* para_plane_R[0]                size 4, tangent 3 */
    VIWB_BLK_PLANE_Z = 26,     /* para_plane_Z[0]                size 1 */
    VIWB_BLK_SX = 27,          /* para_Ix_sx_wheel[0]            size 1 */
    VIWB_BLK_SY = 28,
    VIWB_BLK_SW = 29,
    VIWB_BLK_TD = 30,          /* para_Td[0]                     size 1 */
    VIWB_BLK_TD_WHEEL = 31,    /* para_Td_wheel[0]               size 1 */
    VIWB_BLK_LANDMARK0 = 32    /* 32+k   para_Feature[k]         size 1 */
};

/* global size, state offset, tangent size, tangent offset of a fixed block */
static inline int viwb_block_size(int b) {
    return b < 11 ? 7 : b < 22 ? 9 : b < 25 ? 7 : b == 25 ? 4 : 1;
}
static inline int viwb_block_offset(int b) {
    return b < 11 ? 7 * b : b < 22 ? 77 + 9 * (b - 11) : b < 25 ? 176 + 7 * (b - 22) : b == 25 ? 197 : 201 + (b - 26);
}
static inline int viwb_block_tsize(int b) {
    return b < 11 ? 6 : b < 22 ? 9 : b < 25 ? 6 : b == 25 ? 3 : 1;
}
static inline int viwb_block_toffset(int b) {
    return b < 11 ? 6 * b : b < 22 ? 66 + 9 * (b - 11) : b < 25 ? 165 + 6 * (b - 22) : b == 25 ? 183 : 186 + (b - 26);
}
/* local size under the marginalization rule "7 -> 6, else unchanged"
 * (factor/marginalization_factor.cpp:140-143): plane_R counts 4 there. */
static inline int viwb_block_marg_size(int b) { int s = viwb_block_size(b); return s == 7 ? 6 : s; }

/* block flag bits (problem.block_flags[b]) */
#define VIWB_BLOCK_PRESENT 1u   /* problem.AddParameterBlock was called for it (estimator.cpp:1394-1515) */
#define VIWB_BLOCK_CONSTANT 2u  /* problem.SetParameterBlockConstant (estimator.cpp:1403,1439,1468,...) */

/* visual factor types */
enum viwb_factor_type {
    VIWB_F_PROJ_2F1C = 0,  /* ProjectionTwoFrameOneCamFactor  <2,7,7,7,1,1>   factor/projectionTwoFrameOneCamFactor.h:21 */
    VIWB_F_PROJ_2F2C = 1,  /* ProjectionTwoFrameTwoCamFactor  <2,7,7,7,7,1,1> factor/projectionTwoFrameTwoCamFactor.h:21 */
    VIWB_F_PROJ_1F2C = 2,  /* ProjectionOneFrameTwoCamFactor  <2,7,7,1,1>     factor/projectionOneFrameTwoCamFactor.h:21 */
    VIWB_F_IMU = 3,        /* IMUFactor                       <15,7,9,7,9>    factor/imu_factor.h:23 */
    VIWB_F_WHEEL = 4,      /* WheelFactor                     <6,7,7,7,1,1,1,1> factor/wheel_factor.h:20 */
    VIWB_F_PLANE = 5       /* PlaneFactor                     <3,7,7,4,1>     factor/plane_factor.h:21 */
};

/* per-factor constant records (doubles) */
#define VIWB_VIS_OBS_DOUBLES 12   /* pts_i(3) pts_j(3) vel_i(2) vel_j(2) td_i td_j  (projectionTwoFrameOneCamFactor.h:29-31) */
/* IMU: IntegrationBase members used by IMUFactor::Evaluate (factor/integration_base.h:197-214, imu_factor.h:71-189)
 *  [0] sum_dt  [1..3] delta_p  [4..7] delta_q (x,y,z,w)  [8..10] delta_v  [11..13] linearized_ba  [14..16] linearized_bg
 *  [17..25] dp_dba  [26..34] dp_dbg  [35..43] dq_dbg  [44..52] dv_dba  [53..61] dv_dbg   (3x3 row-major blocks of `jacobian`)
 *  [62..286] covariance 15x15 row-major */
#define VIWB_IMU_DOUBLES 287
/* Wheel: WheelIntegrationBase members used by WheelFactor::Evaluate (factor/wheel_integration_base.h:220-243)
 *  [0..2] delta_p  [3..6] delta_q (x,y,z,w)  [7..24] jacobian 6x3 row-major  [25..60] covariance 6x6 row-major
 *  [61..63] linearized_sx,sy,sw  [64] linearized_td  [65..67] linearized_vel  [68..70] linearized_gyr
 *  [71..73] vel_1  [74..76] gyr_1  [77] sum_dt */
#define VIWB_WHEEL_DOUBLES 78

/* Marginalization prior = MarginalizationInfo after marginalize()+getParameterBlocks()
 * (factor/marginalization_factor.cpp:183-334): linearized_jacobians (n x n, row-major here),
 * linearized_residuals (n), and for each kept block its id, its column offset idx-m in [0,n) and
 * its linearisation point x0 (keep_block_data). x0 is stored in the fixed-state layout (207 doubles). */
typedef struct viwb_prior {
    int32_t valid;                 /* MarginalizationInfo::valid (marginalization_factor.cpp:205-210) */
    int32_t n;                     /* residual dimension / column count */
    int32_t num_blocks;            /* number of kept parameter blocks (<= 32; landmarks are never kept) */
    int32_t block_id[VIWB_NUM_FIXED_BLOCKS];   /* kept block ids (after the addr_shift remap) */
    int32_t block_idx[VIWB_NUM_FIXED_BLOCKS];  /* column offset of the block inside [0,n) */
    double *x0;                    /* [VIWB_STATE_FIXED]  keep_block_data, fixed-state layout */
    double *J;                     /* [n*n] row-major linearized_jacobians */
    double *r;                     /* [n]   linearized_residuals */
} viwb_prior;

/* Globals that the reference keeps in static/global variables. */
typedef struct viwb_globals {
    double G[3];                   /* estimator/parameters.cpp:32,149  G = (0,0,g_norm) */
    double vis_sqrt_info[4];       /* 2x2 row-major; estimator.cpp:157-159: FOCAL_LENGTH/1.5 * I */
    double plane_sqrt_info[3];     /* PITCH_N_INV, ROLL_N_INV, ZPW_N_INV (factor/plane_factor.h:52) */
    double huber_delta;            /* ceres::HuberLoss(1.0) (estimator.cpp:1391) */
} viwb_globals;

/* One Estimator::optimization() problem (estimator.cpp:1388-1638) lowered to tables. */
typedef struct viwb_problem {
    int32_t frame_count;           /* poses 0..frame_count exist (estimator.cpp:1394) */
    int32_t num_landmarks;         /* feature_index+1 (estimator.cpp:1587-1593) */
    uint8_t block_flags[VIWB_NUM_FIXED_BLOCKS];   /* VIWB_BLOCK_* bits */
    /* bit i set -> delta[i] is zeroed in Plus (PoseSubsetParameterization / OrientationSubsetParameterization,
     * factor/pose_subset_parameterization.cpp:27-33, orientation_subset_parameterization.cpp:27-35);
     * ComputeJacobian stays [I;0] so the linear solver still sees the direction (SURVEY quirk 2). */
    uint8_t subset_mask[VIWB_NUM_FIXED_BLOCKS];

    /* visual factors (estimator.cpp:1585-1638); loss = HuberLoss for all of them */
    int32_t num_vis;
    const int32_t *vis_type;       /* [num_vis] VIWB_F_PROJ_* */
    const int32_t *vis_landmark;   /* [num_vis] feature_index */
    const int32_t *vis_frame_i;    /* [num_vis] imu_i (host frame) */
    const int32_t *vis_frame_j;    /* [num_vis] imu_j */
    const double *vis_obs;         /* [num_vis*12] */

    int32_t num_imu;               /* IMUFactor(pre_integrations[j]) between frames i=j-1 and j (estimator.cpp:1528-1545) */
    const int32_t *imu_frame_i;
    const int32_t *imu_frame_j;
    const double *imu_data;        /* [num_imu*287] */

    int32_t num_wheel;             /* WheelFactor (estimator.cpp:1546-1567) */
    const int32_t *wheel_frame_i;
    const int32_t *wheel_frame_j;
    const double *wheel_data;      /* [num_wheel*78] */

    int32_t num_plane;             /* PlaneFactor on pose[plane_frame] (estimator.cpp:1569-1583) */
    const int32_t *plane_frame;

    const viwb_prior *prior;       /* NULL or !valid -> no MarginalizationFactor (estimator.cpp:1521-1527) */
    viwb_globals globals;
} viwb_problem;

/* ceres::Solver::Options subset (estimator.cpp:1643-1655) + the Ceres defaults it leaves untouched
 * (SURVEY Appendix B). viwb_default_options() fills the reference configuration. */
typedef struct viwb_options {
    int32_t max_num_iterations;            /* NUM_ITERATIONS (8 in every shipped config) */
    double max_solver_time_in_seconds;     /* SOLVER_TIME; 0 = disabled (parity runs disable it, SURVEY quirk 13) */
    double function_tolerance;             /* 1e-6 */
    double gradient_tolerance;             /* 1e-10 */
    double parameter_tolerance;            /* 1e-8 */
    double initial_trust_region_radius;    /* 1e4 */
    double max_trust_region_radius;        /* 1e16 */
    double min_trust_region_radius;        /* 1e-32 */
    double min_relative_decrease;          /* 1e-3 */
    double min_lm_diagonal;                /* 1e-6 */
    double max_lm_diagonal;                /* 1e32 */
    int32_t max_num_consecutive_invalid_steps; /* 5 */
    int32_t jacobi_scaling;                /* 1 */
} viwb_options;

enum viwb_termination { VIWB_CONVERGENCE = 0, VIWB_NO_CONVERGENCE = 1, VIWB_FAILURE = 2 };

/* ceres::Solver::Summary subset (estimator.cpp:1657-1660) */
typedef struct viwb_summary {
    int32_t termination_type;      /* viwb_termination */
    int32_t num_iterations;        /* summary.iterations.size() (includes iteration 0) */
    int32_t num_successful_steps;
    int32_t num_linear_solves;     /* Cholesky factorisations performed (mu retries included) */
    double initial_cost;
    double final_cost;
    double final_radius;
    double final_mu;
} viwb_summary;

enum viwb_margin_flag { VIWB_MARGIN_OLD = 0, VIWB_MARGIN_SECOND_NEW = 1 };  /* estimator.h:39-43 */

/* error codes */
#define VIWB_OK 0
#define VIWB_ERR_INVALID (-1)      /* bad argument / inconsistent tables */
#define VIWB_ERR_CUDA (-2)         /* CUDA runtime error (message via viwb_last_error) */
#define VIWB_ERR_UNSUPPORTED (-3)
#define VIWB_ERR_NUMERIC (-4)      /* e.g. marginalization block not positive definite on the fast path */

typedef struct viwb_context viwb_context;

/* ---- lifecycle -------------------------------------------------------------------------------- */
int viwb_create(int device, viwb_context **out);
void viwb_destroy(viwb_context *ctx);
const char *viwb_last_error(const viwb_context *ctx);
/* run all work of this context on an externally owned cudaStream_t (e.g. torch's current stream; NULL = CUDA's default stream).  The caller
 * keeps ownership: viwb_destroy only destroys the stream viwb_create made.  Waits for the work queued so far. */
int viwb_set_stream(viwb_context *ctx, void *cuda_stream);
/* number of kernels this context launched since creation (bench.py's gpu_launches) */
long long viwb_launch_count(const viwb_context *ctx);
/* Bytes of window tables this context has uploaded so far (host -> device, the library's packed wire format; images of the LK entry points are
 * not included: their size is the caller's).  Like viwb_launch_count it has no reference counterpart: measurement only. */
long long viwb_h2d_bytes(const viwb_context *ctx);
/* optional CUDA-event timing around every kernel launch (used by bench.py for the live roofline numbers) */
int viwb_set_profiling(viwb_context *ctx, int enable);
int viwb_profile_count(viwb_context *ctx);
int viwb_profile_get(viwb_context *ctx, int idx, char *name, int name_cap, double *total_ms, long long *launches);
void viwb_default_options(viwb_options *opt);
void viwb_default_globals(viwb_globals *g);

/* ---- factor level: ceres::CostFunction::Evaluate for the six analytic factor classes ------------
 * Same contract as the reference's Evaluate (e.g. factor/projectionTwoFrameOneCamFactor.cpp:45-152):
 * `parameters[i]` are the parameter blocks in the factor's own order, `jacobians` may be NULL,
 * `jacobians[i]` may be NULL, Jacobians are row-major num_residuals x global_size with the last
 * pose column zero.  `consts` is the per-factor record (VIWB_VIS_OBS_DOUBLES / VIWB_IMU_DOUBLES /
 * VIWB_WHEEL_DOUBLES doubles; NULL for the plane factor).  Runs on the GPU (no host arithmetic). */
int viwb_factor_evaluate(viwb_context *ctx, int factor_type, const viwb_globals *globals,
                         const double *consts, const double *const *parameters,
                         double *residuals, double **jacobians);
/* MarginalizationFactor::Evaluate (factor/marginalization_factor.cpp:349-397). `state` is a full
 * fixed-layout state; residuals[n]; jacobian (may be NULL) is n x VIWB_STATE_FIXED row-major holding,
 * for each kept block, the n x global_size block at the block's state offset. */
int viwb_prior_evaluate(viwb_context *ctx, const viwb_prior *prior, const double *state,
                        double *residuals, double *jacobian);

/* ---- window level ------------------------------------------------------------------------------
 * viwb_window_solve     = ceres::Solve(options,&problem,&summary) with DENSE_SCHUR + DOGLEG
 *                         (estimator.cpp:1643-1658); `state` is updated in place like para_*.
 * viwb_gauge_reanchor   = double2vector()+vector2double() on the pose/velocity part
 *                         (estimator.cpp:1224-1276): rotate the window so that frame-0 yaw and position
 *                         equal `state_before`'s.
 * viwb_marginalize      = the MarginalizationInfo block of optimization() (estimator.cpp:1669-1893,
 *                         marginalization_factor.cpp:98-334); writes the next prior (caller-owned buffers
 *                         x0[207], J[VIWB_MAX_PRIOR_DIM^2], r[VIWB_MAX_PRIOR_DIM]).
 * viwb_optimization     = all three in sequence = one Estimator::optimization() call.
 */
int viwb_window_solve(viwb_context *ctx, const viwb_problem *problem, double *state,
                      const viwb_options *options, viwb_summary *summary);
int viwb_gauge_reanchor(viwb_context *ctx, const viwb_problem *problem, const double *state_before, double *state);
int viwb_marginalize(viwb_context *ctx, const viwb_problem *problem, const double *state, int margin_flag,
                     viwb_prior *prior_out);
int viwb_optimization(viwb_context *ctx, const viwb_problem *problem, double *state, const viwb_options *options,
                      int margin_flag, viwb_summary *summary, viwb_prior *prior_out);

/* Estimator::outliersRejection (estimator.cpp:2127-2185, SURVEY 8 f-3) on a solved window: outliers[k] = 1 when the mean
 * reprojectionError (:2115-2125) of landmark k over its observations, times focal_length (FOCAL_LENGTH = 460), exceeds
 * threshold_px (3).  outliers: [num_landmarks]. */
int viwb_outlier_rejection(viwb_context *ctx, const viwb_problem *problem, const double *state, double focal_length,
                           double threshold_px, uint8_t *outliers);

/* FeatureManager::triangulate for features without a depth (feature_manager.cpp:309-385; triangulatePoint :198-213): two-view
 * linear triangulation, stereo[k] = 1: left / right camera of frame[k] (pt0 = point, pt1 = pointRight of the first observation),
 * stereo[k] = 0: left camera of frame[k] and frame[k]+1 (pt0, pt1 = the first two observations).  pt*: [n][2] normalised
 * coordinates.  depth[k] = z in the first camera if positive, else init_depth (INIT_DEPTH = 5.0, parameters.cpp:387). */
int viwb_triangulate(viwb_context *ctx, const double *state, int n, const int32_t *stereo, const int32_t *frame,
                     const double *pt0, const double *pt1, double init_depth, double *depth);
/* FeatureManager::removeBackShiftDepth (feature_manager.cpp:457-493) for the features that started in the marginalised frame:
 * re-express depth in the new frame 0.  uv: [n][3] first-observation points; R row-major 3x3 (camera-to-world), P [3]. */
int viwb_shift_depth(viwb_context *ctx, int n, const double *uv, const double *depth_in, const double *marg_R, const double *marg_P,
                     const double *new_R, const double *new_P, double init_depth, double *depth_out);
/* Estimator::predictPtsInNextFrame (estimator.cpp:2080-2113): constant-velocity next pose nextT = curT * (prevT^-1 * curT) from frames
 * frame_count-1 and frame_count of `state` (getPoseInWorldFrame, :2066-2078); for every feature with depth > 0, num_obs >= 2 and
 * start_frame + num_obs - 1 == frame_count: pts_cam in the predicted left camera.  The feature list is the caller's
 * FeatureManager::feature (every feature with a depth, also those optimization() leaves out), not the window's landmark table.
 * pt0: [n][3] first observation (feature_per_frame[0].point), extrinsics of camera 0 from `state`.  pts_cam: [n][3]; valid[n] = 1
 * where the reference inserts the id into predictPts (other rows of pts_cam are 0).  frame_count < 2: every valid[k] = 0 (:2083).
 * prevT^-1 is formed as the rigid inverse [R^T | -R^T p]. */
int viwb_predict_pts(viwb_context *ctx, const double *state, int frame_count, int n, const int32_t *start_frame,
                     const int32_t *num_obs, const double *pt0, const double *depth, double *pts_cam, uint8_t *valid);

/* Batch of B independent windows (one per sequence), host buffers in, host buffers out. */
int viwb_optimization_batch(viwb_context *ctx, int batch, const viwb_problem *problems, double *const *states,
                            const viwb_options *options, const int32_t *margin_flags, viwb_summary *summaries,
                            viwb_prior *priors_out /* [batch] or NULL to skip marginalization */);

/* Device-resident batch: upload once, run many times (bench.py `value`: inputs already in HBM). */
typedef struct viwb_batch viwb_batch;
int viwb_batch_create(viwb_context *ctx, int batch, const viwb_problem *problems, const double *const *states,
                      const viwb_options *options, const int32_t *margin_flags, viwb_batch **out);
int viwb_batch_reset_states(viwb_context *ctx, viwb_batch *b);  /* restore the uploaded initial states */
int viwb_batch_run(viwb_context *ctx, viwb_batch *b);           /* solve + reanchor + marginalize, async on the stream */
int viwb_batch_download(viwb_context *ctx, viwb_batch *b, double *const *states, viwb_summary *summaries,
                        viwb_prior *priors_out);
/* outliersRejection on the windows as the batch currently holds them (after viwb_batch_run: solved and re-anchored);
 * outliers[w]: [num_landmarks of window w] or NULL */
int viwb_batch_outliers(viwb_context *ctx, viwb_batch *b, double focal_length, double threshold_px, uint8_t *const *outliers);
/* algorithmic bytes of one viwb_batch_run (SURVEY 8(d) B_solve model, summed over the batch) */
double viwb_batch_algorithmic_bytes(const viwb_batch *b);
/* The solve kernel's launch for this batch: threads per block, dynamic shared memory per block (bytes; sized by the batch's widest window) and
 * how many such blocks one SM of the context's device holds (cudaOccupancyMaxActiveBlocksPerMultiprocessor).  Measurement only, like
 * viwb_launch_count.  Any output pointer may be NULL. */
int viwb_batch_solve_launch(viwb_context *ctx, const viwb_batch *b, int *threads, int *smem_bytes, int *blocks_per_sm);
void viwb_batch_destroy(viwb_context *ctx, viwb_batch *b);

/* Normal equations at `state` exactly as the solver assembles them (debug/parity hook):
 * H [192*192] row-major over the fixed tangent layout, g [192], per landmark lm[k*82 + {0:a_k, 1:g_k, 2..81:w_k}],
 * where w_k is indexed like the "visual subspace": 11 poses x 6, ex0 6, ex1 6, td 1 (79, padded to 80). */
int viwb_debug_normal_equations(viwb_context *ctx, const viwb_problem *problem, const double *state,
                                double *H, double *g, double *lm, double *cost);

/* ---- pre-integration (SURVEY 8 f-2): the producers of the IMU / wheel records above --------------------
 * IntegrationBase::propagate over a buffer of samples (factor/integration_base.h:63-167) and
 * WheelIntegrationBase::propagate (factor/wheel_integration_base.h:67-177), `n` independent intervals per call.
 * Interval i has counts[i] steps: dt holds the steps of all intervals back to back, the sample arrays hold
 * counts[i]+1 rows of 3 per interval back to back (row 0 = acc_0 / gyr_0 resp. vel_0 / gyr_0).
 * ba, bg: [n][3] linearisation biases; noise = {ACC_N, GYR_N, ACC_W, GYR_W} (parameters.cpp) resp.
 * {VEL_N_wheel, GYR_N_wheel}; s: [n][3] = sx, sy, sw; td: [n] linearized_td.  records: [n][287] / [n][78]. */
int viwb_imu_preintegrate(viwb_context *ctx, int n, const int32_t *counts, const double *dt, const double *acc,
                          const double *gyr, const double *ba, const double *bg, const double *noise, double *records);
int viwb_wheel_preintegrate(viwb_context *ctx, int n, const int32_t *counts, const double *dt, const double *vel,
                            const double *gyr, const double *s, const double *td, const double *noise, double *records);

/* ---- initialisation: visual-inertial(-wheel) alignment (SURVEY 8 f-4 ii) -------------------------------
 * initial/initial_aligment.cpp, the three steps of VisualIMUAlignment (:336-344) as the caller sequences them:
 *   viwb_solve_gyroscope_bias  = solveGyroscopeBias (:14-48) up to delta_bg; the repropagation that follows it there is
 *                                viwb_imu_preintegrate with ba = 0, bg = Bgs[0] + delta_bg on the same sample buffers;
 *   viwb_linear_alignment      = LinearAlignment + RefineGravity (:66-203) when wheel_data is NULL, else
 *                                LinearAlignmentWithWheel + RefineGravityWithWheel (:204-334).
 * Frames = all_image_frame in time order: R [num_frames][9] row-major ImageFrame::R, T [num_frames][3]; imu_data / wheel_data
 * [num_frames-1] records (VIWB_IMU_DOUBLES / VIWB_WHEEL_DOUBLES) of frame j's pre-integration; tic = TIC[0], rio / tio = RIO (row-major) /
 * TIO, g_norm = G.norm().  Outputs: g, x (capacity 3*num_frames+4; *x_size = 3*num_frames+4 when the first stage already fails its
 * |g| / scale test, else 3*num_frames+3 with x.tail = s as the reference leaves it), *aligned = the reference's bool. */
#define VIWB_MAX_INIT_FRAMES 64
int viwb_solve_gyroscope_bias(viwb_context *ctx, int num_frames, const double *R, const double *imu_data, double *delta_bg);
int viwb_linear_alignment(viwb_context *ctx, int num_frames, const double *R, const double *T, const double *imu_data,
                          const double *wheel_data, const double *tic, const double *rio, const double *tio, double g_norm,
                          double *g, double *x, int32_t *x_size, int32_t *aligned);

/* ---- feature tracker: cv::calcOpticalFlowPyrLK replacement ---------------------------------------
 * Call sites featureTracker/feature_tracker.cpp:125-127,136,139,145-146,240,244.  Images are 8-bit
 * single channel, `stride` in bytes.  next_pts is in/out (read when flags & VIWB_LK_USE_INITIAL_FLOW).
 * status/err follow OpenCV semantics (SURVEY Appendix C). */
#define VIWB_LK_USE_INITIAL_FLOW 4   /* cv::OPTFLOW_USE_INITIAL_FLOW */
int viwb_lk_track(viwb_context *ctx, const uint8_t *prev_img, const uint8_t *next_img, int width, int height,
                  int stride, const float *prev_pts, float *next_pts, int n, int win_size, int max_level,
                  int max_iter, float eps, int flags, float min_eig_threshold, uint8_t *status, float *err);

/* Temporal / stereo tracking step of FeatureTracker::trackImage with the reference's status
 * post-processing (feature_tracker.cpp:139-162 and :240-251): forward LK (maxLevel 3), optional
 * reverse check (temporal: maxLevel 1 + initial flow seeded with prev_pts; stereo: maxLevel 3, no
 * initial flow), round trip <= 0.5 px, inBorder with a 1 px border after rounding.
 * mode 0 = temporal (prev -> cur), 1 = stereo (left -> right). */
int viwb_track_checked(viwb_context *ctx, const uint8_t *img_a, const uint8_t *img_b, int width, int height,
                       int stride, const float *pts_a, float *pts_b, int n, int mode, int flow_back,
                       uint8_t *status);

/* FeatureTracker::undistortedPts (feature_tracker.cpp:606-617; PinholeCamera::liftProjective, recursive distortion model with
 * 8 iterations, camera_models/src/camera_models/PinholeCamera.cc:450-517) and FeatureTracker::ptsVelocity (:619-657) for points
 * paired index-wise with the previous tick (SURVEY 8 f-1).  pts: pixel coordinates [n][2]; un_pts: normalised, narrowed to float
 * like cv::Point2f; velocity (optional): (un - prev_un) / dt where has_prev[i] (NULL = all) and prev_un_pts are given, else 0. */
typedef struct viwb_pinhole { double fx, fy, cx, cy, k1, k2, p1, p2; } viwb_pinhole;
int viwb_undistort_velocity(viwb_context *ctx, const viwb_pinhole *cam, int n, const float *pts, const float *prev_un_pts,
                            const uint8_t *has_prev, double dt, float *un_pts, float *velocity);

/* A camera of either model camodocal builds for the reference's tracker (FeatureTracker::readIntrinsicParameter, feature_tracker.cpp):
 *   VIWB_CAMERA_PINHOLE: p = fx fy cx cy k1 k2 p1 p2 (viwb_pinhole's order; p[8] unused), PinholeCamera.
 *   VIWB_CAMERA_MEI:     p = xi k1 k2 p1 p2 gamma1 gamma2 u0 v0 (CataCamera's constructor and its yaml order, CataCamera.cc:300-303), the
 *                        unified omnidirectional model with mirror parameter xi: the lift is CataCamera::liftProjective (:556-626, recursive
 *                        distortion n = 8, distortion :766-782, m_inv_K* :319-323) and the projection CataCamera::spaceToPlane (:636-659).
 *   VIWB_CAMERA_KANNALA_BRANDT: p = k2 k3 k4 k5 mu mv u0 v0 (EquidistantCamera::Parameters' and its yaml order; p[8] unused), the
 *                        generic fisheye model r(theta) = theta + k2 theta^3 + k3 theta^5 + k4 theta^7 + k5 theta^9 (Kalibr's `equidistant`,
 *                        OpenCV's cv::fisheye): the lift is EquidistantCamera::liftProjective (:428-442, m_inv_K* :271-274) over
 *                        backprojectSymmetric (:716-818: theta = the smallest non-negative real root of r(theta) = |p_u|, from the eigenvalues
 *                        of the polynomial's companion matrix, restated from Eigen 3.3's EigenSolver), the projection
 *                        EquidistantCamera::spaceToPlane (:451-461, r() of EquidistantCamera.h:158-168).
 * The MEI arithmetic is rounded operation by operation (no fused multiply-add), so its floats are the reference's bit for bit.  So is the
 * Kannala-Brandt arithmetic, except for sin / cos / acos / atan2, which the GPU evaluates within 2 ulp: a float may then differ from the
 * reference's by one ulp where the double lies next to a float rounding boundary.  Parameter values are not checked, as the reference does
 * not check them: a ray with 1 + (1 - xi^2) rho^2 < 0 lifts to NaN as it does there, a Kannala-Brandt ray past 90 degrees lifts to the
 * mirrored point.  The one refusal: a Kannala-Brandt camera whose companion matrix would divide by zero is VIWB_ERR_INVALID.  That is the
 * case where the polynomial degree npow (9, less 2 for every k_i == 0, wherever it sits) is above 1 and its coefficient at npow is 0 --
 * k4 == 0 with k5 != 0, or k2 == k4 == k5 == 0 with k3 != 0, for example; the reference then feeds inf / NaN to its eigen-solver. */
typedef enum { VIWB_CAMERA_PINHOLE = 0, VIWB_CAMERA_MEI = 1, VIWB_CAMERA_KANNALA_BRANDT = 2 } viwb_camera_model;
typedef struct viwb_camera {
    int32_t model;      /* viwb_camera_model */
    double p[9];
} viwb_camera;
/* viwb_undistort_velocity with the lift of `cam`'s model.  An unknown model, a NULL cam or a refused Kannala-Brandt camera is
 * VIWB_ERR_INVALID (viwb_last_error says why).
 * With a PINHOLE camera this is viwb_undistort_velocity, to the bit. */
int viwb_undistort_velocity_camera(viwb_context *ctx, const viwb_camera *cam, int n, const float *pts, const float *prev_un_pts,
                                   const uint8_t *has_prev, double dt, float *un_pts, float *velocity);

/* ---- batched tracker: one camera tick of `streams` independent VIO sessions per submission --------
 * Replaces, per stream, the four calcOpticalFlowPyrLK calls of one FeatureTracker::trackImage()
 * (feature_tracker.cpp:139 temporal forward, :145-146 temporal reverse, :240 stereo forward, :244 stereo
 * reverse) and the status rules of :147-162 / :245-251.  The object keeps three device image slots per
 * stream; uploading a new `cur` image turns the previous one (and its pyramid) into `prev`, as
 * trackImage's prev_img = cur_img (:296) does.  Point arrays are flat [streams][max_points][2] floats,
 * status arrays [streams][max_points]; n_* give the valid count per stream. */
typedef struct viwb_lk_batch viwb_lk_batch;
int viwb_lk_batch_create(viwb_context *ctx, int streams, int width, int height, int max_points, int stereo,
                         int flow_back /* FLOW_BACK */, viwb_lk_batch **out);
void viwb_lk_batch_destroy(viwb_lk_batch *b);
/* Host -> device.  prev/cur/right: `streams` image pointers each (8-bit, `stride` bytes per row) or NULL to
 * keep what the device holds (prev is only needed on the first tick).  prev_pts: points of the previous
 * image to follow into cur; stereo_pts: points of cur to follow into right (trackImage runs the stereo
 * match on cur_pts after goodFeaturesToTrack topped them up, :200-240).  Asynchronous on the context stream;
 * the host buffers must stay valid until the next synchronising call. */
int viwb_lk_batch_upload(viwb_lk_batch *b, const uint8_t *const *prev, const uint8_t *const *cur,
                         const uint8_t *const *right, int stride, const float *prev_pts, const int32_t *n_prev,
                         const float *stereo_pts, const int32_t *n_stereo);
/* pyramids of the freshly uploaded images + forward / reverse flows + status rules; device only, asynchronous */
int viwb_lk_batch_run(viwb_lk_batch *b);
/* Device -> host (synchronises). Any pointer may be NULL. */
int viwb_lk_batch_download(viwb_lk_batch *b, float *cur_pts, uint8_t *status, float *right_pts, uint8_t *status_right);
/* compulsory HBM bytes of one viwb_lk_batch_run (new images read once, coarser levels written once, points) */
double viwb_lk_batch_algorithmic_bytes(const viwb_lk_batch *b);

/* ---- feature detection: the rest of FeatureTracker::trackImage() between the LK calls (SURVEY 8 f-1) ----------------
 * viwb_set_mask = FeatureTracker::setMask() (feature_tracker.cpp:59-89): visit the tracked points by descending track count,
 * keep a point iff the mask is still 255 under its rounded position, blank a filled circle of radius MIN_DIST around every
 * kept point.  keep[] receives the surviving indices in visiting order (the order cur_pts / ids / track_cnt are rebuilt in);
 * base_mask (NULL = white) is the FISHEYE mask the reference clones at :62; mask_out (may be NULL) is the [height][width] result.
 * Points with equal track counts are visited in their original order (std::sort leaves that order unspecified). */
int viwb_set_mask(viwb_context *ctx, int width, int height, const float *pts, const int32_t *track_cnt, int n, int min_dist,
                  const uint8_t *base_mask, uint8_t *mask_out, int32_t *keep, int32_t *n_keep);
/* cv::goodFeaturesToTrack(image, corners, maxCorners, qualityLevel, minDistance, mask) with blockSize 3, gradientSize 3 and
 * the minimum-eigenvalue measure, the call of feature_tracker.cpp:192.  corners: [capacity][2] floats (capacity <= 1024);
 * max_corners <= 0 means "all" (still bounded by capacity). */
int viwb_good_features_to_track(viwb_context *ctx, const uint8_t *image, int width, int height, int stride, int max_corners,
                                double quality_level, double min_distance, const uint8_t *mask, int mask_stride,
                                float *corners, int capacity, int32_t *n_corners);
/* Batched detector: one camera tick of `streams` independent sessions per submission -- setMask over each stream's tracked
 * points, then goodFeaturesToTrack for the max_cnt - n_keep corners that are missing (feature_tracker.cpp:175-200).
 * images: `streams` host image pointers, or NULL to detect on the current left images that `resident` (a viwb_lk_batch of the
 * same geometry) already holds in HBM.  pts [streams][max_pts][2], track_cnt [streams][max_pts], n_pts [streams];
 * keep [streams][max_pts] / n_keep [streams]; new_pts [streams][max_pts][2] / n_new [streams]; mask_out NULL or
 * [streams][height][width]; base_masks NULL or `streams` pointers to [height][width] fisheye masks. */
typedef struct viwb_detector viwb_detector;
int viwb_detector_create(viwb_context *ctx, int streams, int width, int height, int max_pts, int min_dist /* MIN_DIST */,
                         viwb_detector **out);
void viwb_detector_destroy(viwb_detector *d);
int viwb_detector_detect(viwb_detector *d, const uint8_t *const *images, int stride, const viwb_lk_batch *resident,
                         const uint8_t *const *base_masks, const float *pts, const int32_t *track_cnt, const int32_t *n_pts,
                         int max_cnt /* MAX_CNT */, double quality_level, int32_t *keep, int32_t *n_keep, float *new_pts,
                         int32_t *n_new, uint8_t *mask_out);
/* compulsory HBM bytes of one viwb_detector_detect: every stream's image read once, the points in, the corners out */
double viwb_detector_algorithmic_bytes(const viwb_detector *d);

/* ---- session tracker: FeatureTracker::trackImage() as one call (featureTracker/feature_tracker.cpp:99-331, SURVEY 8 f-1) ----------
 * `streams` independent FeatureTracker sessions (feature_tracker.h:50-95: prev_img, prev_pts, ids, track_cnt, n_id, the id -> point
 * maps) live in HBM.  One viwb_tracker_track() per camera tick does, per stream and without a host round trip: the temporal flow
 * (with the hasPrediction branch of :122-137 when predict_pts is given), the reverse check and status rules, reduceVector, track_cnt++,
 * setMask, goodFeaturesToTrack(MAX_CNT - n, 0.01, MIN_DIST, mask), id assignment (n_id++), undistortedPts + ptsVelocity, the stereo
 * flow cur -> right with its reverse check, the right camera's undistortedPts + ptsVelocity, and prev_* = cur_*.  Only the images go
 * up and the featureFrame rows come down.  cam[0] / cam[1]: pinhole + radtan intrinsics of the left / right camera (m_camera[0/1]). */
typedef struct viwb_tracker_config {
    int max_cnt;        /* MAX_CNT  (parameters.cpp: "max_cnt"), also the per-stream row capacity of every output array, <= 1024 */
    int min_dist;       /* MIN_DIST ("min_dist") */
    int flow_back;      /* FLOW_BACK ("flow_back") */
    int stereo;         /* stereo_cam && a right image every tick */
    viwb_pinhole cam[2];
} viwb_tracker_config;
typedef struct viwb_tracker viwb_tracker;
int viwb_tracker_create(viwb_context *ctx, int streams, int width, int height, const viwb_tracker_config *config, viwb_tracker **out);
/* viwb_tracker_create with cam[0] / cam[1] = m_camera[0] / m_camera[1] of any viwb_camera model, each camera its own (an MEI left camera
 * beside a pinhole right camera is legal); config->cam is not read.  Both entries must name a known model, cam[1] also in a mono session,
 * where it is not used.  The lift of undistortedPts (feature_tracker.cpp:606-617, both cameras) and setPrediction's spaceToPlane
 * (:729, camera 0, viwb_tracker_feedback) follow each camera's model.  An unknown model, a NULL cam or a refused Kannala-Brandt camera
 * is VIWB_ERR_INVALID, and no session is made. */
int viwb_tracker_create_camera(viwb_context *ctx, int streams, int width, int height, const viwb_tracker_config *config,
                               const viwb_camera cam[2], viwb_tracker **out);
void viwb_tracker_destroy(viwb_tracker *t);
/* trackImage(cur_time, left[s], right[s]) for every stream s.  left / right: `streams` host image pointers (8-bit, `stride` bytes per
 * row; right may be NULL for a mono session).  predict_pts (optional): [streams][max_cnt][2] = FeatureTracker::setPrediction()'s
 * predict_pts, aligned with the rows returned by the previous tick; has_prediction: [streams] flags (hasPrediction).  Asynchronous on
 * the context stream: the host buffers must stay valid until viwb_tracker_download returns. */
int viwb_tracker_track(viwb_tracker *t, double cur_time, const uint8_t *const *left, const uint8_t *const *right, int stride,
                       const float *predict_pts, const uint8_t *has_prediction);
/* The featureFrame of the tick (:307-350), as rows: camera 0 rows in cur_pts order -- ids / track_cnt [streams][max_cnt], feat
 * [streams][max_cnt][6] = {x, y, p_u, p_v, velocity_x, velocity_y} (z = 1) -- and camera 1 rows in ids_right order.  n_left / n_right:
 * [streams] row counts.  Any pointer may be NULL.  Synchronises. */
int viwb_tracker_download(viwb_tracker *t, int32_t *n_left, int32_t *ids, int32_t *track_cnt, float *feat, int32_t *n_right,
                          int32_t *ids_right, float *feat_right);
/* The estimator's way back into the sessions, once per estimator tick (estimator.cpp:841-843, MULTIPLE_THREAD == 0), for every stream:
 * FeatureTracker::removeOutliers(remove_ids) (feature_tracker.cpp:739-755: stable reduceVector of prev_pts, ids, track_cnt; the id ->
 * undistorted point maps stay as they are) and then, for the streams with has_prediction[s] != 0, FeatureTracker::setPrediction
 * (:715-736): for each remaining row, the prediction with the row's id projected by m_camera[0]->spaceToPlane (pinhole + radtan,
 * PinholeCamera.cc:520-542, MEI, CataCamera.cc:636-659, or Kannala-Brandt, EquidistantCamera.cc:451-461) and rounded to float as cv::Point2f does, else the row's prev_pts.  The prediction stays in HBM and is
 * consumed by the next viwb_tracker_track, which must then be called with predict_pts == NULL (VIWB_ERR_INVALID otherwise, and the
 * session stays as it was); hasPrediction is cleared by that tick (:279).
 * n_remove / n_pred: [streams] list lengths; remove_ids, pred_ids: the streams' lists back to back; pred_pts_cam: [sum n_pred][3]
 * camera-frame points (viwb_predict_pts' output, compacted to its valid rows).  An id listed twice behaves as in the reference's
 * std::set / std::map: removed once; of several predictions for one id the last one counts (predictPts[id] = pts_cam).  Either half
 * may be absent (n_remove == NULL / n_pred == NULL); n_pred needs has_prediction.  A call without the prediction half while an
 * earlier call's prediction is still pending is VIWB_ERR_INVALID (its rows would no longer line up), as are a call before the
 * first tick, a negative length, and a non-zero length with a NULL list.  viwb_tracker_download still returns the last tick's
 * rows afterwards.  Asynchronous on the context stream. */
int viwb_tracker_feedback(viwb_tracker *t, const int32_t *n_remove, const int32_t *remove_ids, const int32_t *n_pred,
                          const int32_t *pred_ids, const double *pred_pts_cam, const uint8_t *has_prediction);
/* compulsory HBM bytes of one tick: the new images read once by the pyramid and once by the detector, pyramid levels written, rows out */
double viwb_tracker_algorithmic_bytes(const viwb_tracker *t);

/* ---- resident FeatureManager: estimator/feature_manager.{h,cpp} for `streams` independent sessions ----------------------------------------
 * The NON_LINEAR branch of Estimator::processImage (estimator.cpp:690-878) around the solve, per stream and without a host round trip:
 *   add (+ decisions)   f_manager.addFeatureCheckParallax (:694-703; feature_manager.cpp:52-119, compensatedParallax2 :538-571)
 *   triangulate         f_manager.triangulate (:832; feature_manager.cpp:309-389, the two live branches)
 *   window              the visual-factor loop of optimization() (:1585-1638) and getDepthVector (feature_manager.cpp:179-195)
 *   set_depth           double2vector's f_manager.setDepth (:1324-1327; feature_manager.cpp:142-160)
 *   remove_outliers     f_manager.removeOutlier(removeIndex) (:835-837; feature_manager.cpp:440-455)
 *   predict             predictPtsInNextFrame (:2080-2113)
 *   slide               slideWindowOld / slideWindowNew's FeatureManager part (:1898-2063; feature_manager.cpp:457-536)
 *   remove_failures     f_manager.removeFailures (:859; feature_manager.cpp:162-171)
 * Each stream's list keeps the reference's order: insertion order (new ids appended in ascending id order, as the image map iterates),
 * stable erasures; an id erased and then seen again is appended as a new feature.  The landmark numbering of a window export is that order
 * filtered by num_obs >= 4.  Observations are stored as the six floats {x, y, p_u, p_v, v_x, v_y} per camera (z = 1) and the double cur_td:
 * every featureFrame producer of the reference takes its numbers from floats, so these reproduce FeaturePerFrame exactly.
 * Per-stream host arrays lie back to back with fixed strides.  Every call launches the same number of kernels whatever `streams` is; calls
 * that return data synchronise, the others are asynchronous on the context stream. */
typedef struct viwb_features_config {
    int max_rows;          /* featureFrame rows per stream and tick (MAX_CNT), <= 1024; a tracker fed to add_tracked needs max_cnt <= max_rows */
    int max_features;      /* list capacity per stream; 0 = (VIWB_WINDOW_SIZE + 1) * max_rows, which valid input cannot exceed */
    int stereo;            /* STEREO */
    double min_parallax;   /* MIN_PARALLAX = keyframe_parallax / FOCAL_LENGTH (parameters.cpp:267-268) */
    double focal_length;   /* FOCAL_LENGTH (460); only last_average_parallax uses it */
    double init_depth;     /* INIT_DEPTH (5.0) */
} viwb_features_config;
typedef struct viwb_features viwb_features;
int viwb_features_create(viwb_context *ctx, int streams, const viwb_features_config *config, viwb_features **out);
void viwb_features_destroy(viwb_features *fs);
/* addFeatureCheckParallax(frame_count[s], image, td[s]) per stream, the image map built from host rows in viwb_tracker_download's layout
 * with max_rows as the stride: n_left [streams], ids [streams][max_rows], feat [streams][max_rows][6], and the right camera's rows (n_right
 * NULL or a mono configuration: none).  A duplicate left or right id, a right id without a left row (the reference asserts, :65-70), a row
 * count outside [0, max_rows] or a frame_count outside [0, VIWB_WINDOW_SIZE] returns VIWB_ERR_INVALID at once and nothing is queued.  A list
 * that would exceed max_features or a feature that would get a twelfth observation is found on the device: then no list changes and the
 * next synchronising call (decisions, window, remove_outliers, predict, download) returns VIWB_ERR_INVALID naming the stream, and does
 * nothing else.  Such an error stays set on the device until that call reads it: an add queued behind a failed one changes no list either,
 * so no failure is ever overwritten and no frame is skipped silently.  The decisions stay those of the last add that was applied. */
int viwb_features_add(viwb_features *fs, const int32_t *frame_count, const double *td, const int32_t *n_left, const int32_t *ids, const float *feat,
                      const int32_t *n_right, const int32_t *ids_right, const float *feat_right);
/* The same with the rows of the last tick of `t` read in HBM: no row crosses the bus.  t must belong to the same context and have the same
 * stream count (else VIWB_ERR_INVALID at once).  The row rules above are checked on the device.  A stream whose tick overflowed
 * goodFeaturesToTrack's candidate list is not consumed (its list stays as it was, the other streams are added) and the next synchronising
 * call reports it; until then later adds leave that stream's list alone too. */
int viwb_features_add_tracked(viwb_features *fs, const viwb_tracker *t, const int32_t *frame_count, const double *td);
/* The verdicts of the last add, [streams] each (any pointer may be NULL): margin_flag = VIWB_MARGIN_OLD (keyframe) or VIWB_MARGIN_SECOND_NEW,
 * last_track_num, long_track_num (a feature counts when it has >= 4 observations after the push), new_feature_num, last_average_parallax
 * (0 unless the parallax branch ran).  Synchronises. */
int viwb_features_decisions(viwb_features *fs, int32_t *margin_flag, int32_t *last_track_num, int32_t *long_track_num, int32_t *new_feature_num,
                            double *last_average_parallax);
/* f_manager.triangulate(frame_count, Ps, Rs, tic, ric) on every stream: states [streams][VIWB_STATE_FIXED] (poses and extrinsics as in
 * viwb_problem's state).  Per feature the function of viwb_triangulate, so a depth is the one viwb_triangulate gives on the downloaded list. */
int viwb_features_triangulate(viwb_features *fs, const double *states);
/* The visual table of every stream in viwb_problem's layout (estimator.cpp:1585-1638): rows [streams][vis_cap] of vis_type / vis_landmark /
 * vis_frame_i / vis_frame_j (imu_j; == vis_frame_i for 1F2C) / vis_obs [12], num_vis [streams]; landmark k's inverse depth (getDepthVector,
 * 1 / estimated_depth) and feature id in [streams][VIWB_MAX_LANDMARKS], num_landmarks [streams].  The doubles are the stored floats and
 * cur_td, so the table is exact.  More than VIWB_MAX_LANDMARKS landmarks or more than vis_cap rows in a stream is VIWB_ERR_INVALID naming
 * it.  The export's numbering is what set_depth and remove_outliers take.  Synchronises. */
int viwb_features_window(viwb_features *fs, int vis_cap, int32_t *num_landmarks, int32_t *num_vis, int32_t *vis_type, int32_t *vis_landmark,
                         int32_t *vis_frame_i, int32_t *vis_frame_j, double *vis_obs, double *inv_depth, int32_t *landmark_ids);
/* setDepth: landmark k's estimated_depth = 1.0 / inv_depth[s][k] and solve_flag = 2 if negative else 1.  VIWB_ERR_INVALID if a list changed
 * (add, remove_outliers, slide, remove_failures) since the last export. */
int viwb_features_set_depth(viwb_features *fs, const double *inv_depth /* [streams][VIWB_MAX_LANDMARKS] */);
/* removeOutlier with per-landmark verdicts in the numbering of the last export (what viwb_batch_outliers / viwb_outlier_rejection produce);
 * the removed ids of each stream in ascending order (std::set order), ready for viwb_tracker_feedback.  VIWB_ERR_INVALID if a list changed
 * since the last export.  Synchronises. */
int viwb_features_remove_outliers(viwb_features *fs, const uint8_t *outliers /* [streams][VIWB_MAX_LANDMARKS] */, int32_t *n_removed,
                                  int32_t *removed_ids /* [streams][max_features] */);
/* predictPtsInNextFrame over the resident lists (the function of viwb_predict_pts), compacted to the features it inserts, in list order and
 * the streams back to back: n_pred [streams], pred_ids / pred_pts_cam [sum n_pred] / [sum n_pred][3] (capacity streams * max_features),
 * has_prediction [streams] = frame_count >= 2 (:2083 returns before setPrediction) -- viwb_tracker_feedback's arguments.  Synchronises. */
int viwb_features_predict(viwb_features *fs, const double *states, const int32_t *frame_count, int32_t *n_pred, int32_t *pred_ids,
                          double *pred_pts_cam, uint8_t *has_prediction);
/* slideWindow's FeatureManager part with the margin flag of the last add; a stream with frame_count != VIWB_WINDOW_SIZE is left alone.
 * MARGIN_OLD: shift_depth[s] (solver_flag == NON_LINEAR) -> removeBackShiftDepth(marg_R, marg_P, new_R, new_P) with the camera poses of
 * slideWindowOld (:2053-2059; R row-major [streams][9], P [streams][3]; may be NULL when no shift_depth[s] is set), else removeBack.
 * MARGIN_SECOND_NEW: removeFront(frame_count), including its missing depth shift (feature_manager.cpp:533). */
int viwb_features_slide(viwb_features *fs, const int32_t *frame_count, const uint8_t *shift_depth, const double *marg_R, const double *marg_P,
                        const double *new_R, const double *new_P);
/* removeFailures: erase every feature with solve_flag == 2 */
int viwb_features_remove_failures(viwb_features *fs);
/* The lists as they stand (tests, PnP initialisation on the host, debugging): n [streams]; [streams][max_features] ids, start_frame, num_obs,
 * depth, solve_flag; obs [streams][max_features][11][12] floats (left x y p_u p_v v_x v_y, then the right camera's, 0 without one), cur_td
 * [..][11], is_stereo [..][11].  Entries past n[s] or num_obs are undefined.  Any pointer may be NULL.  Synchronises. */
int viwb_features_download(viwb_features *fs, int32_t *n, int32_t *ids, int32_t *start_frame, int32_t *num_obs, double *depth, int32_t *solve_flag,
                           float *obs, double *cur_td, uint8_t *is_stereo);
/* optimization()'s visual loop + getDepthVector + viwb_batch_create in one call: one window per stream, in stream order, its visual factors
 * and landmark inverse depths taken from the lists in HBM.  problems[s] carries everything else (frame_count, block flags / masks, IMU /
 * wheel / plane tables, prior, globals) with num_vis == 0, num_landmarks == 0 and NULL visual tables; states [streams][VIWB_STATE_FIXED].
 * margin_flags as in viwb_batch_create (NULL: no marginalisation).  num_landmarks [streams] (may be NULL): each window's landmark count.
 * The result is an ordinary viwb_batch (run / reset_states / download / outliers / destroy unchanged) and counts as an export for
 * set_depth / remove_outliers.  Only a digest of a few bytes per landmark crosses the bus, and the batch's upload leaves out the observations
 * and the landmark states, so the windows are bit for bit those of viwb_features_window + viwb_batch_create.  VIWB_ERR_INVALID with no batch
 * made: an add error still unread, a stream with more than VIWB_MAX_LANDMARKS landmarks, a problem with visual rows or landmarks, a list
 * observation beyond the problem's frame_count, or any refusal of viwb_batch_create.  Synchronises. */
int viwb_features_batch_create(viwb_features *fs, const viwb_problem *problems, const double *states, const viwb_options *options,
                               const int32_t *margin_flags, int32_t *num_landmarks, viwb_batch **out);
/* The feedback calls below take a batch of viwb_features_batch_create on these lists (VIWB_ERR_INVALID for a batch of other lists or of
 * viwb_batch_create) and read it in HBM. */
/* setDepth from the batch's current landmark states (after viwb_batch_run: the solution), device to device: the function of
 * viwb_features_set_depth fed them.  VIWB_ERR_INVALID if a list changed since the batch's create. */
int viwb_features_set_depth_batch(viwb_features *fs, const viwb_batch *b);
/* outliersRejection on the batch (the verdicts viwb_batch_outliers gives) + removeOutlier, without the verdicts crossing the bus; outputs as
 * viwb_features_remove_outliers.  VIWB_ERR_INVALID if a list changed since the batch's create.  Synchronises. */
int viwb_features_remove_outliers_batch(viwb_features *fs, viwb_batch *b, double focal_length, double threshold_px,
                                        int32_t *n_removed, int32_t *removed_ids);
/* predictPtsInNextFrame with each stream's fixed state read from the batch; outputs as viwb_features_predict.  Only the fixed states are
 * read, so it follows remove_outliers_batch as predictPtsInNextFrame follows removeOutlier in processImage.  Synchronises. */
int viwb_features_predict_batch(viwb_features *fs, const viwb_batch *b, const int32_t *frame_count, int32_t *n_pred, int32_t *pred_ids,
                                double *pred_pts_cam, uint8_t *has_prediction);

/* Page-lock / unlock caller-owned host memory (camera frame buffers) for asynchronous full-rate uploads. */
int viwb_host_register(viwb_context *ctx, void *ptr, size_t bytes);
int viwb_host_unregister(viwb_context *ctx, void *ptr);

#ifdef __cplusplus
}
#endif
#endif /* VIWB_H */
