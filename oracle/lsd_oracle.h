/*
 * lsd_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C, Eigen-free restatement of the two LSD-SLAM hot paths
 *   SE3Tracker::trackFrame            lsd_slam_core/src/Tracking/SE3Tracker.cpp:280-486
 *   DepthMap::updateKeyframe          lsd_slam_core/src/DepthEstimation/DepthMap.cpp:1072-1213
 *   DepthMap::createKeyFrame          lsd_slam_core/src/DepthEstimation/DepthMap.cpp:1222-1327
 * and of everything below them (Frame builders, TrackingReference point cloud,
 * Sophus SE3 exp / product / inverse, 6x6 LDLT).  Each function cites the
 * reference file:line it follows.
 *
 * PARITY PINNED TO THE REFERENCE'S OWN CODE (round 2): oracle/ref_build.py compiles DepthMap.cpp, SE3Tracker.cpp,
 * Sim3Tracker.cpp, Frame.cpp, TrackingReference.cpp ... unmodified from /root/reference against stand-in headers
 * (oracle/ref_shim/: an Eigen 3.2 subset, Boost -> std, OpenCV debug stubs) into oracle/_ref/liblsd_ref.so, exported under the
 * same lsdo_* API by oracle/ref_driver.cpp; tests/test_ref_pin.py holds this restatement to it BIT FOR BIT on every function of
 * the path, and tests/golden/reference_320x240.npz are outputs of that library.  UndistorterPTAM is pinned the same way:
 * util/Undistorter.cpp is part of the _ref build, and tests/test_ref_pin_undistort.py holds lsd_oracle_undistort.inc and the
 * library's table builder to it over a calibration sweep (tests/golden/ref_pin_undistort.npz).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library.  The product (lsd_slam_b200/) never does.
 *
 * Third-party arithmetic restated here because its source is not vendored:
 *   Eigen 3.x (find_package(Eigen3 REQUIRED), lsd_slam_core/CMakeLists.txt:19; conventions of Eigen 3.2, the release the
 *   reference was written against: the vendored Sophus test programs pass on the same conventions, tests/test_ref_pin.py)
 *   - 3x3 inverse by cofactors (Eigen/src/LU/Inverse.h compute_inverse_size3)
 *   - Quaternion product / toRotationMatrix / _transformVector (Eigen/src/Geometry/Quaternion.h)
 *   - LDLT with diagonal pivoting (Eigen/src/Cholesky/LDLT.h, unblocked)
 *   - fixed-size 3x3*3x1 products evaluated coefficient-wise, left to right.
 */
#ifndef LSD_ORACLE_H
#define LSD_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LSDO_LEVELS 5           /* PYRAMID_LEVELS, util/settings.h:106 */

/* DepthMapPixelHypothesis, DepthEstimation/DepthMapPixelHypothesis.h:37-61 (sizeof == 32) */
typedef struct {
    uint8_t isValid;
    uint8_t _pad[3];
    int32_t blacklisted;
    float   nextStereoFrameMinID;
    int32_t validity_counter;
    float   idepth;
    float   idepth_var;
    float   idepth_smoothed;
    float   idepth_var_smoothed;
} lsdo_hyp;

/* global runtime flags, util/settings.cpp:77-88 */
typedef struct {
    float minUseGrad;                 /* 5   */
    float cameraPixelNoise2;          /* 16  */
    float depthSmoothingFactor;       /* 1   */
    int   allowNegativeIdepths;       /* 1   */
    int   useSubpixelStereo;          /* 1   */
    int   useAffineLightningEstimation; /* 1 (settings.cpp:88); cfg/LSDParams.cfg:28 sets 0 under ROS */
    int   multiThreading;             /* 1: DepthMap row ranges on MAPPING_THREADS=4 workers */
    int   useSSE;                     /* 0: scalar parity path; 1: the reference's SSE loops (timing flavour) */
    int   exactAffineSums;            /* DIAGNOSTIC, default 0 = the reference: 1 accumulates the five affine-lighting sums of
                                       * calcSim3Buffers in double, to separate the float-accumulation noise of the reference
                                       * (sums ~1e9 in fp32) from real differences when a parity test looks at residuals */
    int   exactTrackingSums;          /* DIAGNOSTIC, default 0 = the reference: 1 accumulates every sum of the SE3 tracker (affine-lighting
                                       * sums, residual sums, LGS6 A / b / error) in double from the same fp32 terms -- the result the
                                       * reference's sequential fp32 accumulation approximates.  Used to measure the reference's OWN
                                       * summation noise in the tracked pose (tests/test_gpu_fullsize.py, DESIGN.md section 5) */
    int   exactSim3Sums;              /* DIAGNOSTIC, default 0 = the reference: 1 accumulates every sum of the scalar Sim3 tracker
                                       * (the five affine-lighting sums, the depth and photometric residual sums, LGS4 / LGS6 A / b /
                                       * error) in double from the same fp32 terms -- what the device's tree sums approach */
} lsdo_globals;

/* DenseDepthTrackerSettings, util/settings.h:355-402 */
typedef struct {
    float lambdaSuccessFac, lambdaFailFac;
    float lambdaInitial[LSDO_LEVELS];
    float stepSizeMin[LSDO_LEVELS];
    float convergenceEps[LSDO_LEVELS];
    int   maxItsPerLvl[LSDO_LEVELS];
    float huber_d, var_weight;
} lsdo_track_settings;

/* everything SlamSystem reads back from the tracker, Tracking/SE3Tracker.h:82-93 */
typedef struct {
    double frameToRef_qt[7];          /* (qx,qy,qz,qw, tx,ty,tz) */
    float  pointUsage, lastGoodCount, lastBadCount, lastMeanRes, lastResidual;
    float  affineEstimation_a, affineEstimation_b;
    int    diverged, trackingWasGood;
    int    numCalcResidualCalls[LSDO_LEVELS];
    int    numCalcWarpUpdateCalls[LSDO_LEVELS];
    float  initialTrackedResidual;    /* frame->initialTrackedResidual, SE3Tracker.cpp:482 */
} lsdo_track_result;

/* one fused evaluation: calcResidualAndBuffers + calcWeightsAndResidual + calculateWarpUpdate */
typedef struct {
    float A[36];                      /* row-major 6x6, divided by num_constraints (LGSX.h:319-325) */
    float b[6];
    float lsError;                    /* LGS6::error after finish */
    float meanWeightedRes;            /* return value of calcWeightsAndResidual */
    float meanUnweightedRes;          /* return value of calcResidualAndBuffers */
    int   warpedSize;                 /* buf_warped_size */
    float pointUsage, goodCount, badCount, meanRes;
    float affine_a_lastIt, affine_b_lastIt;
    float sxx, syy, sx, sy, sw;
} lsdo_eval_result;

/* Sim3Tracker (SURVEY 8f row 1): everything SlamSystem::tryTrackSim3 reads back, Tracking/Sim3Tracker.h:66,127-138 */
typedef struct {
    double frameToRef_qts[8];         /* unit (qx,qy,qz,qw), (tx,ty,tz), scale; Sim3() = identity on the early returns */
    float  lastSim3Hessian[49];       /* ls7.A, NOT divided by num_constraints (Sim3Tracker.cpp:360) */
    float  lastResidual, lastDepthResidual, lastPhotometricResidual;
    float  pointUsage;
    float  affineEstimation_a, affineEstimation_b;
    int    diverged;
    int    numCalcResidualCalls[LSDO_LEVELS];
    int    numCalcWarpUpdateCalls[LSDO_LEVELS];
} lsdo_sim3_result;

/* one fused evaluation: calcSim3Buffers + calcSim3WeightsAndResidual + calcSim3LGS */
typedef struct {
    float A[49], b[7];                /* LGS7, undivided */
    int   num_constraints;            /* 2 * warpedSize */
    float sumResD, sumResP; int numTermsD, numTermsP;
    float mean, meanD, meanP;
    int   warpedSize;
    float pointUsage, affine_a_lastIt, affine_b_lastIt;
} lsdo_sim3_eval_result;

typedef struct lsdo_frame lsdo_frame;
typedef struct lsdo_depthmap lsdo_depthmap;

void lsdo_default_globals(lsdo_globals* g);
void lsdo_set_globals(const lsdo_globals* g);
void lsdo_get_globals(lsdo_globals* g);
void lsdo_default_track_settings(lsdo_track_settings* s);

/* ---- SE3 / Sim3 host math (thirdparty/Sophus/sophus/se3.hpp, so3.hpp) ---- */
void lsdo_se3d_exp(const double a[6], double qt[7]);
void lsdo_se3d_mul(const double a[7], const double b[7], double out[7]);
void lsdo_se3d_inverse(const double a[7], double out[7]);
void lsdo_se3d_matrix(const double a[7], double R[9], double t[3]);
void lsdo_se3f_exp(const float a[6], float qt[7]);
void lsdo_se3f_mul(const float a[7], const float b[7], float out[7]);
void lsdo_se3f_inverse(const float a[7], float out[7]);
void lsdo_se3f_matrix(const float a[7], float R[9], float t[3]);
void lsdo_se3d_log(const double a[7], double out[6]);
int  lsdo_ldlt6_solve(const float A[36], const float b[6], float x[6]);
int  lsdo_ldlt7_solve(const float A[49], const float b[7], float x[7]);
/* Sim3 as qts[8] = unit quaternion (x,y,z,w), translation, scale  (thirdparty/Sophus/sophus/sim3.hpp, rxso3.hpp) */
void lsdo_sim3d_exp(const double a[7], double out_qts[8]);
void lsdo_sim3d_mul(const double a[8], const double b[8], double out[8]);
void lsdo_sim3d_inverse(const double a[8], double out[8]);
/* the per-pose constants of calcSim3Buffers (Sim3Tracker.cpp:447-460): rxso3 matrix, translation, xRoll0/1 yRoll0/1 */
void lsdo_sim3_pose_constants(const double refToFrame_qts[8], float rotMat[9], float transVec[3], float roll[4]);
void lsdo_mat3_inverse(const float K[9], float Kinv[9]);

/* ---- Frame (DataStructures/Frame.{h,cpp}) ---- */
lsdo_frame* lsdo_frame_create_u8(int id, int w, int h, const float K[9], const uint8_t* image);
void  lsdo_frame_destroy(lsdo_frame* f);
int   lsdo_frame_id(const lsdo_frame* f);
int   lsdo_frame_width(const lsdo_frame* f, int level);
int   lsdo_frame_height(const lsdo_frame* f, int level);
const float* lsdo_frame_image(lsdo_frame* f, int level);
const float* lsdo_frame_gradients(lsdo_frame* f, int level);      /* 4 floats / px */
const float* lsdo_frame_maxGradients(lsdo_frame* f, int level);
const float* lsdo_frame_idepth(lsdo_frame* f, int level);
const float* lsdo_frame_idepthVar(lsdo_frame* f, int level);
void  lsdo_frame_K(const lsdo_frame* f, int level, float K[9], float Kinv[9]);
uint8_t* lsdo_frame_refPixelWasGood(lsdo_frame* f);                /* creates (all true) */
uint8_t* lsdo_frame_refPixelWasGoodNoCreate(lsdo_frame* f);
void  lsdo_frame_clear_refPixelWasGood(lsdo_frame* f);
void  lsdo_frame_setDepthFromGroundTruth(lsdo_frame* f, const float* depth, float cov_scale);
void  lsdo_frame_setDepth(lsdo_frame* f, const lsdo_hyp* newDepth);
int   lsdo_frame_numMappablePixels(lsdo_frame* f);
float lsdo_frame_meanIdepth(const lsdo_frame* f);
int   lsdo_frame_numPoints(const lsdo_frame* f);
int   lsdo_frame_depthHasBeenUpdatedFlag(const lsdo_frame* f);
void  lsdo_frame_set_depthHasBeenUpdatedFlag(lsdo_frame* f, int v);
float lsdo_frame_initialTrackedResidual(const lsdo_frame* f);
void  lsdo_frame_set_initialTrackedResidual(lsdo_frame* f, float v);   /* test hook: a frame tracked elsewhere */
void  lsdo_frame_get_thisToParent(const lsdo_frame* f, double qts[8]);  /* Sim3: q(4) t(3) s */
void  lsdo_frame_set_thisToParent(lsdo_frame* f, const double qts[8], lsdo_frame* parent);
int   lsdo_frame_numFramesTrackedOnThis(const lsdo_frame* f);
int   lsdo_frame_numMappedOnThis(const lsdo_frame* f);
void  lsdo_frame_set_counters(lsdo_frame* f, int tracked, int mapped);

/* ---- TrackingReference point cloud (Tracking/TrackingReference.cpp:96-147) ---- */
/* Frame::takeReActivationData (Frame.cpp:107-145) and the keyframeMsg packing loop (ROSOutput3DWrapper.cpp:91-110), SURVEY 8f row 4 */
void  lsdo_frame_takeReActivationData(lsdo_frame* f, const lsdo_hyp* depthMap);
const float* lsdo_frame_idepth_reAct(const lsdo_frame* f);
const float* lsdo_frame_idepthVar_reAct(const lsdo_frame* f);
const uint8_t* lsdo_frame_validity_reAct(const lsdo_frame* f);
void  lsdo_pack_pointcloud(lsdo_frame* f, int publishLvl, void* out /* w_l*h_l records of 12 bytes */);
/* returns numData[level]; out arrays sized w_l*h_l by the caller (NULL = skip) */
int lsdo_make_point_cloud(lsdo_frame* kf, int level, float* posData /*3/pt*/, float* gradData /*2/pt*/,
                          float* colorAndVarData /*2/pt*/, int* pointPosInXYGrid);

/* ---- SE3Tracker (Tracking/SE3Tracker.cpp) ---- */
int lsdo_se3_eval(lsdo_frame* kf, lsdo_frame* frame, int level, const float refToFrame_qt[7],
                  float affine_a, float affine_b, const lsdo_track_settings* s,
                  int writeGoodMask, lsdo_eval_result* out);
int lsdo_se3_track(lsdo_frame* kf, lsdo_frame* frame, const double frameToRef_init_qt[7],
                   const lsdo_track_settings* s, lsdo_track_result* out);

/* ---- Sim3Tracker (Tracking/Sim3Tracker.cpp), SURVEY 8f row 1; `frame` must carry depth (a keyframe) ---- */
int lsdo_sim3_eval(lsdo_frame* ref_kf, lsdo_frame* frame, int level, const double refToFrame_qts[8],
                   float affine_a, float affine_b, const lsdo_track_settings* s, lsdo_sim3_eval_result* out);
int lsdo_sim3_track(lsdo_frame* ref_kf, lsdo_frame* frame, const double frameToRef_init_qts[8],
                    int startLevel, int finalLevel, const lsdo_track_settings* s, lsdo_sim3_result* out);

/* ---- UndistorterPTAM (util/Undistorter.cpp:171-317, 355-411), SURVEY 8f row 3.  outputCalibration[0] = -1 "crop", -2 "full";
 * returns 0 tables valid, 1 undistort() is the identity (:370-375), -1 invalid ---- */
int  lsdo_undistorter_ptam_prepare(const float inputCalibration[5], int in_width, int in_height, const float outputCalibration[5],
                                   int out_width, int out_height, float* remapX, float* remapY, float K_out[9]);
void lsdo_undistort(const float* remapX, const float* remapY, int in_width, int out_width, int out_height,
                    const uint8_t* image, uint8_t* out);

/* ---- permaRef tracking, SURVEY 8f row 2 (Frame.cpp:149-174, SE3Tracker.cpp:121-272) ---- */
int   lsdo_frame_setPermaRef(lsdo_frame* kf, float* posData, float* colorAndVarData);      /* returns permaRefNumPts */
float lsdo_checkPermaRefOverlap(int w0, int h0, const float K4[9], const float* permaPos, int numPts, const double refToFrame_qt[7]);
int   lsdo_trackFrameOnPermaref(int w0, int h0, const float* permaPos, const float* permaColVar, int numPts,
                                lsdo_frame* frame, const double refToFrame_qt[7], lsdo_track_result* out /* frameToRef_qt holds referenceToFrame */);
/* the reference-compiled library only: SE3Tracker's own two calls on a keyframe whose setPermaRef ran (the reference reads the
 * snapshot from the Frame); the LM call counters are locals there and come back as -1 */
float lsdo_ref_checkPermaRefOverlap(lsdo_frame* kf, const double refToFrame_qt[7]);
int   lsdo_ref_trackFrameOnPermaref(lsdo_frame* kf, lsdo_frame* frame, const double refToFrame_qt[7], lsdo_track_result* out);

/* ---- DepthMap (DepthEstimation/DepthMap.cpp) ---- */
lsdo_depthmap* lsdo_depthmap_create(int w, int h, const float K[9]);
void lsdo_depthmap_destroy(lsdo_depthmap* d);
void lsdo_depthmap_reset(lsdo_depthmap* d);
void lsdo_depthmap_initializeFromGTDepth(lsdo_depthmap* d, lsdo_frame* f);
void lsdo_depthmap_initializeRandomly(lsdo_depthmap* d, lsdo_frame* f);
void lsdo_depthmap_setFromExistingKF(lsdo_depthmap* d, lsdo_frame* kf, const float* idepth_reAct, const float* idepthVar_reAct, const unsigned char* validity_reAct);
void lsdo_depthmap_updateKeyframe(lsdo_depthmap* d, lsdo_frame** refs, int n_refs);
void lsdo_depthmap_createKeyFrame(lsdo_depthmap* d, lsdo_frame* new_kf);
void lsdo_depthmap_finalizeKeyFrame(lsdo_depthmap* d);
const lsdo_hyp* lsdo_depthmap_current(const lsdo_depthmap* d);
void lsdo_depthmap_set_current(lsdo_depthmap* d, const lsdo_hyp* h);
const int* lsdo_depthmap_integral(const lsdo_depthmap* d);
lsdo_frame* lsdo_depthmap_activeKeyFrame(lsdo_depthmap* d);
/* individual passes, for per-kernel parity tests */
void lsdo_depthmap_observeDepth(lsdo_depthmap* d, lsdo_frame** refs, int n_refs);
void lsdo_depthmap_regularizeFillHoles(lsdo_depthmap* d);
void lsdo_depthmap_regularize(lsdo_depthmap* d, int removeOcclusions, int validityTH);
void lsdo_depthmap_propagateDepth(lsdo_depthmap* d, lsdo_frame* new_kf);
/* the stereo constants Frame::prepareForStereoWith leaves in `frame` (Frame.cpp:295-317): K_otherToThis_R[9], K_otherToThis_t,
 * otherToThis_t, thisToOther_t, otherToThis_R_row0..2, distSquared, referenceID, referenceLevel */
void lsdo_ref_prepareForStereoWith(lsdo_frame* frame, lsdo_frame* kf, const double thisToOther_qts[8], const float K[9], float out[30]);
/* per-stage EMA timers of the reference (DepthMap.cpp:1126-1162), ms of the last call */
void lsdo_depthmap_last_timings(const lsdo_depthmap* d, float out_ms[8]);
/* diagnostic branch counters of doLineStereo, observeDepth and propagateDepth, summed over every depth map of the process (C restatement only:
 * they show which branches a test reaches; no float is read or written by them) */
enum {
    LSDO_BR_DEPTH_X,          /* x-dominant depth formula, DepthMap.cpp:1876-1886 */
    LSDO_BR_DEPTH_Y,          /* y-dominant depth formula, :1887-1898 */
    LSDO_BR_FIRSTX_GATE,      /* first/last sample point outside the image, :1463-1469 */
    LSDO_BR_RESCALE_GATE,     /* rescaleFactor outside (0.7, 1.4), :1470 */
    LSDO_BR_NEAR_CLAMP,       /* pClose behind the near plane, max_idepth clamped, :1491-1495 */
    LSDO_BR_EPL_CROP,         /* eplLength > MAX_EPL_LENGTH_CROP, :1520-1524 */
    LSDO_BR_CLIP_LEFT, LSDO_BR_CLIP_RIGHT, LSDO_BR_CLIP_TOP, LSDO_BR_CLIP_BOTTOM,     /* pClose clipped at a border, :1567-1592 */
    LSDO_BR_SUBPIXEL_PRE, LSDO_BR_SUBPIXEL_POST, LSDO_BR_SUBPIXEL_NONE,             /* subpixel refinement outcome, :1768-1845 */
    LSDO_BR_PROP_SKIP,        /* propagateDepth: occluded source skipped, :592-593 */
    LSDO_BR_PROP_INVALIDATE,  /* propagateDepth: target replaced by a nearer source, :600 */
    LSDO_BR_PROP_MERGE,       /* propagateDepth: source merged into a consistent target, :619-631 */
    LSDO_BR_PROP_MERGE_CAP,   /* propagateDepth: merged validity capped, :626-627 */
    LSDO_BR_STEREO_ERR_SEARCH,  /* doLineStereo -3: best match error of the search above 4 MAX_ERROR_STEREO, :1750-1754 */
    LSDO_BR_STEREO_ERR_INTERP,  /* doLineStereo -3: interpolated error above the gradient-dependent bound, :1861-1865 */
    LSDO_BR_STEREO_UNCLEAR,     /* doLineStereo -2: no clear winner, :1758-1762 */
    LSDO_BR_STEREO_NEGATIVE,    /* doLineStereo -2: negative idepth with allowNegativeIdepths off, :1903-1908 */
    LSDO_BR_UPDATE_FAIL_INVALIDATE,  /* observeDepthUpdate on -2: variance inflated above MAX_VAR, invalidated, :381-385 */
    LSDO_BR_UPDATE_INCONSISTENT,     /* observeDepthUpdate: inconsistent observation, variance inflated, :410-417 */
    LSDO_BR_CREATE_BLACKLIST,   /* observeDepthCreate: blacklisted-- on -3 or -2, :269-273 */
    LSDO_BR_PROP_MASK,          /* propagateDepth: source dropped by the tracking mask, :550-555 */
    LSDO_BR_PROP_COLOR,         /* propagateDepth without a mask: source dropped by the colour difference, :559-569 */
    LSDO_BR_REG_OCCLUSION,      /* regularizeDepthMapRow<true>: invalidated by numOccluding > numNotOccluding, :826-834 */
    LSDO_BR_REG_VALIDITY,       /* regularizeDepthMapRow: dropped by val_sum < validityTH, :815-823 */
    LSDO_BR_FILL_CREATE,        /* regularizeDepthMapFillHolesRow: hypothesis created, :690-700 */
    LSDO_BR_EPL_REJECT_GRAD,    /* makeAndCheckEPL: gradient along the epipolar line below MIN_EPL_GRAD_SQUARED, :213-217 */
    LSDO_BR_EPL_REJECT_ANGLE,   /* makeAndCheckEPL: angle to the epipolar line above MIN_EPL_ANGLE_SQUARED, :221-225 */
    LSDO_BR_COUNT
};
void lsdo_depth_branch_counts(int64_t out[LSDO_BR_COUNT]);
void lsdo_depth_branch_counts_reset(void);
/* the same for the Sim3 tracker's scalar path, the permaRef overlap and the 7x7 solve (C restatement only) */
enum {
    LSDO_S3_OUTSIDE,          /* calcSim3Buffers: point warped outside the image, Sim3Tracker.cpp:486 */
    LSDO_S3_NO_DEPTH,         /* calcSim3Buffers: warped onto a frame pixel without depth (var_frameDepth <= 0), :531-541 */
    LSDO_S3_USAGE_CLAMP,      /* calcSim3Buffers: depthChange >= 1, usage clamped to 1, :579-580 */
    LSDO_S3_AFFINE_CLAMP,     /* calcSim3Buffers: |residual_p| >= 2, affine weight 2/|r|, :514 */
    LSDO_S3_HUBER,            /* calcSim3WeightsAndResidual: weighted residual >= huber_d, :795 */
    LSDO_S3_LDLT7_SOLVE,      /* trackFrameSim3's 7x7 LDLT solves, Sim3Tracker.cpp:224 */
    LSDO_S3_LDLT7_PIVOT,      /* ... of which the pivoting permuted a row (Eigen LDLT) */
    LSDO_PERMA_OUTSIDE,       /* checkPermaRefOverlap: point outside, SE3Tracker.cpp:148 */
    LSDO_PERMA_USAGE_CLAMP,   /* checkPermaRefOverlap: depthChange >= 1, :150-151 */
    LSDO_S3_COUNT
};
void lsdo_sim3_branch_counts(int64_t out[LSDO_S3_COUNT]);
void lsdo_sim3_branch_counts_reset(void);

#ifdef __cplusplus
}
#endif
#endif
