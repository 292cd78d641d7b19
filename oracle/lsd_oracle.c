/*
 * lsd_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).  See lsd_oracle.h.
 *
 * Build: gcc -O2 -std=gnu11 -ffp-contract=off -fno-fast-math -msse2 (parity flavour, strict
 * IEEE fp32, no FMA contraction).  All citations are relative to /root/reference/lsd_slam_core/src/.
 *
 * Conventions restated from the reference build: Release => NDEBUG => enablePrintDebugInfo == false
 * (util/settings.h:44-48), i.e. every `if(enablePrintDebugInfo && ...)` is constant-false and
 * `else` branches hanging off such an `if` ARE evaluated (SURVEY.md App. A-17).
 * Pool buffers are defined as zero-filled (SURVEY.md App. A-12).
 */
#define _GNU_SOURCE
#include "lsd_oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <time.h>
#include <xmmintrin.h>

/* ------------------------------------------------------------------------------------------
 * constants, util/settings.h:50-174
 * ---------------------------------------------------------------------------------------- */
#define DIVISION_EPS 1e-10f
/* UNZERO mixes float and double literals; the value is converted back to float at every use site */
static inline float unzero_f(float val)
{
    double r = (val < 0 ? (val > -1e-10 ? -1e-10 : (double)val) : (val < 1e-10 ? 1e-10 : (double)val));
    return (float)r;
}
#define VALIDITY_COUNTER_MAX (5.0f)
#define VALIDITY_COUNTER_MAX_VARIABLE (250.0f)
#define VALIDITY_COUNTER_INC 5
#define VALIDITY_COUNTER_DEC 5
#define VALIDITY_COUNTER_INITIAL_OBSERVE 5
#define VAL_SUM_MIN_FOR_CREATE (30)
#define VAL_SUM_MIN_FOR_KEEP (24)
#define VAL_SUM_MIN_FOR_UNBLACKLIST (100)
#define MIN_BLACKLIST -1
#define SUCC_VAR_INC_FAC (1.01f)
#define FAIL_VAR_INC_FAC 1.1f
#define MAX_VAR (0.5f*0.5f)
#define VAR_GT_INIT_INITIAL 0.01f*0.01f
#define VAR_RANDOM_INIT_INITIAL (0.5f*MAX_VAR)
#define MAPPING_THREADS 4
#define SE3TRACKING_MIN_LEVEL 1
#define SE3TRACKING_MAX_LEVEL 5
#define MIN_DEPTH 0.05f
#define MAX_EPL_LENGTH_CROP 30.0f
#define MIN_EPL_LENGTH_CROP (3.0f)
#define GRADIENT_SAMPLE_DIST 1.0f
#define SAMPLE_POINT_TO_BORDER 7
#define MAX_ERROR_STEREO (1300.0f)
#define MIN_DISTANCE_ERROR_STEREO (1.5f)
#define STEREO_EPL_VAR_FAC 2.0f
#define REG_DIST_VAR (0.075f*0.075f*G.depthSmoothingFactor*G.depthSmoothingFactor)
#define DIFF_FAC_SMOOTHING (1.0f*1.0f)
#define DIFF_FAC_OBSERVE (1.0f*1.0f)
#define DIFF_FAC_PROP_MERGE (1.0f*1.0f)
#define MIN_EPL_GRAD_SQUARED (2.0f*2.0f)
#define MIN_EPL_LENGTH_SQUARED (1.0f*1.0f)
#define MIN_EPL_ANGLE_SQUARED (0.3f*0.3f)
#define MIN_ABS_GRAD_CREATE (G.minUseGrad)
#define MIN_ABS_GRAD_DECREASE (G.minUseGrad)
#define MAX_DIFF_CONSTANT (40.0f*40.0f)
#define MAX_DIFF_GRAD_MULT (0.5f*0.5f)
#define MIN_GOODPERGOODBAD_PIXEL (0.5f)
#define MIN_GOODPERALL_PIXEL (0.04f)
#define MIN_GOODPERALL_PIXEL_ABSMIN (0.01f)

static lsdo_globals G = { 5.0f, 16.0f, 1.0f, 1, 1, 1, 1, 0, 0 };

void lsdo_default_globals(lsdo_globals* g)
{   /* util/settings.cpp:77-88 */
    g->minUseGrad = 5; g->cameraPixelNoise2 = 4*4; g->depthSmoothingFactor = 1;
    g->allowNegativeIdepths = 1; g->useSubpixelStereo = 1; g->useAffineLightningEstimation = 1;
    g->multiThreading = 1; g->useSSE = 0; g->exactAffineSums = 0; g->exactTrackingSums = 0; g->exactSim3Sums = 0;
}
void lsdo_set_globals(const lsdo_globals* g) { G = *g; }
void lsdo_get_globals(lsdo_globals* g) { *g = G; }

void lsdo_default_track_settings(lsdo_track_settings* s)
{   /* util/settings.h:358-386 */
    static const int maxIterations[6] = {5, 20, 50, 100, 100, 100};
    s->lambdaSuccessFac = 0.5f; s->lambdaFailFac = 2.0f;
    for (int l = 0; l < LSDO_LEVELS; l++) {
        s->lambdaInitial[l] = 0; s->stepSizeMin[l] = 1e-8; s->convergenceEps[l] = 0.999f;
        s->maxItsPerLvl[l] = maxIterations[l];
    }
    s->var_weight = 1.0; s->huber_d = 3;
}

/* ------------------------------------------------------------------------------------------
 * Eigen-free linear algebra
 * ---------------------------------------------------------------------------------------- */
/* Eigen/src/LU/Inverse.h compute_inverse_size3 (cofactor / determinant form), row-major in/out */
void lsdo_mat3_inverse(const float m[9], float r[9])
{
#define M(i,j) m[(i)*3+(j)]
#define COF(i,j) (M(((i)+1)%3,((j)+1)%3)*M(((i)+2)%3,((j)+2)%3) - M(((i)+1)%3,((j)+2)%3)*M(((i)+2)%3,((j)+1)%3))
    float c00 = COF(0,0), c10 = COF(1,0), c20 = COF(2,0);
    float det = (c00*M(0,0) + c10*M(1,0)) + c20*M(2,0);
    float invdet = 1.0f/det;
    r[0*3+0] = c00*invdet; r[0*3+1] = c10*invdet; r[0*3+2] = c20*invdet;
    r[1*3+0] = COF(0,1)*invdet; r[1*3+1] = COF(1,1)*invdet; r[1*3+2] = COF(2,1)*invdet;
    r[2*3+0] = COF(0,2)*invdet; r[2*3+1] = COF(1,2)*invdet; r[2*3+2] = COF(2,2)*invdet;
#undef COF
#undef M
}

/* redux_novec_unroller<Func, Derived, Start, Length> (Eigen/src/Core/Redux.h): sum(first Length/2) + sum(rest) */
static float tree_sum_f(const float* v, int n)
{
    if (n == 1) return v[0];
    int h = n/2;
    return tree_sum_f(v, h) + tree_sum_f(v+h, n-h);
}

/* diagnostic counters of the Sim3 tracker and the permaRef overlap (lsd_oracle.h, LSDO_S3_*): relaxed atomic adds that read
 * and write no float, as the depth map's in lsd_oracle_depth.inc */
static int64_t sim3Counts[LSDO_S3_COUNT];
#define COUNT_S3(b) __atomic_fetch_add(&sim3Counts[b], 1, __ATOMIC_RELAXED)
void lsdo_sim3_branch_counts(int64_t out[LSDO_S3_COUNT])
{
    for (int i = 0; i < LSDO_S3_COUNT; i++) out[i] = __atomic_load_n(&sim3Counts[i], __ATOMIC_RELAXED);
}
void lsdo_sim3_branch_counts_reset(void)
{
    for (int i = 0; i < LSDO_S3_COUNT; i++) __atomic_store_n(&sim3Counts[i], 0, __ATOMIC_RELAXED);
}

/* Eigen LDLT (Cholesky/LDLT.h, unblocked lower, largest-|diagonal| pivoting) + solve, float; N <= 8.
 * *permuted (if given) is set when the pivoting swapped a row. */
static int ldlt_solve_n(int N, const float* Ain, const float* bin, float* x, int* permuted)
{
    float A[8][8]; int tr[8]; float cutoff = 0;
    for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) A[i][j] = Ain[i*N+j];
    for (int k = 0; k < N; k++) {
        int p = k; float big = fabsf(A[k][k]);
        for (int i = k+1; i < N; i++) if (fabsf(A[i][i]) > big) { big = fabsf(A[i][i]); p = i; }
        if (k == 0) cutoff = fabsf(1.1920929e-07f * big);
        tr[k] = p;
        if (big < cutoff) { for (int i = k; i < N; i++) tr[i] = i; break; }     /* not full rank: LDLT.h stops here */
        if (p != k) {   /* symmetric swap of rows/cols k,p in the lower triangle */
            for (int j = 0; j < k; j++) { float t = A[k][j]; A[k][j] = A[p][j]; A[p][j] = t; }
            for (int i = p+1; i < N; i++) { float t = A[i][k]; A[i][k] = A[i][p]; A[i][p] = t; }
            for (int i = k+1; i < p; i++) { float t = A[i][k]; A[i][k] = A[p][i]; A[p][i] = t; }
            { float t = A[k][k]; A[k][k] = A[p][p]; A[p][p] = t; }
        }
        /* A[k][k] -= sum_j L[k][j]^2 D[j] ; column below */
        if (k > 0) {
            float temp[8];
            for (int j = 0; j < k; j++) temp[j] = A[j][j]*A[k][j];
            float s = 0; for (int j = 0; j < k; j++) s += A[k][j]*temp[j];
            A[k][k] -= s;
            for (int i = k+1; i < N; i++) {
                float t = 0; for (int j = 0; j < k; j++) t += A[i][j]*temp[j];
                A[i][k] -= t;
            }
        }
        float d = A[k][k];
        if (fabsf(d) > cutoff) for (int i = k+1; i < N; i++) A[i][k] /= d;
    }
    /* LDLT::solve (LDLT.h): dst = P b; L^-1; D^+ (pseudo-inverse, tolerance max|D| eps); L^-T; P^T.  The right-hand side is a
     * fixed-size vector of <= 8 coefficients, so both triangular solves are Eigen's completely unrolled
     * triangular_solver_unroller: rhs(I) -= (lhs.row(I).segment(S, n) .* rhs.segment(S, n)).sum(), the sum being the binary
     * tree of redux_novec_unroller (split n/2 | n - n/2).  oracle/ref_shim/Eigen/Core implements the same statement. */
    float y[8];
    for (int i = 0; i < N; i++) y[i] = bin[i];
    for (int k = 0; k < N; k++) if (tr[k] != k) { float t = y[k]; y[k] = y[tr[k]]; y[tr[k]] = t; }
    for (int i = 1; i < N; i++) { float pr[8]; for (int j = 0; j < i; j++) pr[j] = A[i][j]*y[j]; y[i] -= tree_sum_f(pr, i); }
    float dmax = 0; for (int i = 0; i < N; i++) if (fabsf(A[i][i]) > dmax) dmax = fabsf(A[i][i]);
    float tol = dmax * 1.1920929e-07f; if (tol < 1.0f/3.40282347e+38f) tol = 1.0f/3.40282347e+38f;
    for (int i = 0; i < N; i++) { float d = A[i][i]; y[i] = (fabsf(d) > tol) ? y[i]/d : 0.0f; }
    for (int i = N-2; i >= 0; i--) { float pr[8]; int n = N-1-i; for (int j = 0; j < n; j++) pr[j] = A[i+1+j][i]*y[i+1+j]; y[i] -= tree_sum_f(pr, n); }
    for (int k = N-1; k >= 0; k--) if (tr[k] != k) { float t = y[k]; y[k] = y[tr[k]]; y[tr[k]] = t; }
    for (int i = 0; i < N; i++) x[i] = y[i];
    if (permuted) { *permuted = 0; for (int k = 0; k < N; k++) *permuted |= tr[k] != k; }
    return 0;
}
int lsdo_ldlt6_solve(const float Ain[36], const float bin[6], float x[6]) { return ldlt_solve_n(6, Ain, bin, x, 0); }
int lsdo_ldlt7_solve(const float Ain[49], const float bin[7], float x[7]) { return ldlt_solve_n(7, Ain, bin, x, 0); }

/* ---- Sophus SE3 in float and double; qt = (qx,qy,qz,qw, tx,ty,tz) ----
 * generated twice through a macro so that the float flavour really computes in float
 * (the tracker runs Sophus::SE3f, SE3Tracker.cpp:306). */
#define DEFINE_SE3(T, SUF, SQRT, SIN, COS, EPS)                                                     \
static void quat_mul_##SUF(const T a[4], const T b[4], T o[4])                                      \
{   /* Eigen Quaternion.h quat_product (scalar path); coeffs (x,y,z,w) */                           \
    T w = a[3]*b[3] - a[0]*b[0] - a[1]*b[1] - a[2]*b[2];                                            \
    T x = a[3]*b[0] + a[0]*b[3] + a[1]*b[2] - a[2]*b[1];                                            \
    T y = a[3]*b[1] + a[1]*b[3] + a[2]*b[0] - a[0]*b[2];                                            \
    T z = a[3]*b[2] + a[2]*b[3] + a[0]*b[1] - a[1]*b[0];                                            \
    o[0] = x; o[1] = y; o[2] = z; o[3] = w;                                                         \
}                                                                                                   \
static void quat_normalize_##SUF(T q[4])                                                            \
{   /* so3.hpp:196-202 */                                                                           \
    /* coeffs().norm(): redux tree over 4 coefficients (Redux.h): (x^2 + y^2) + (z^2 + w^2) */      \
    T len = SQRT((q[0]*q[0] + q[1]*q[1]) + (q[2]*q[2] + q[3]*q[3]));                                 \
    q[0] /= len; q[1] /= len; q[2] /= len; q[3] /= len;                                             \
}                                                                                                   \
static void quat_rot_##SUF(const T q[4], const T v[3], T o[3])                                      \
{   /* Eigen QuaternionBase::_transformVector: uv = q.vec x v; uv += uv; v + w*uv + q.vec x uv */   \
    T uv0 = q[1]*v[2] - q[2]*v[1], uv1 = q[2]*v[0] - q[0]*v[2], uv2 = q[0]*v[1] - q[1]*v[0];        \
    uv0 += uv0; uv1 += uv1; uv2 += uv2;                                                             \
    T c0 = q[1]*uv2 - q[2]*uv1, c1 = q[2]*uv0 - q[0]*uv2, c2 = q[0]*uv1 - q[1]*uv0;                 \
    o[0] = v[0] + q[3]*uv0 + c0; o[1] = v[1] + q[3]*uv1 + c1; o[2] = v[2] + q[3]*uv2 + c2;          \
}                                                                                                   \
static void quat_to_R_##SUF(const T q[4], T R[9])                                                   \
{   /* Eigen QuaternionBase::toRotationMatrix */                                                    \
    T tx = 2*q[0], ty = 2*q[1], tz = 2*q[2];                                                        \
    T twx = tx*q[3], twy = ty*q[3], twz = tz*q[3];                                                  \
    T txx = tx*q[0], txy = ty*q[0], txz = tz*q[0];                                                  \
    T tyy = ty*q[1], tyz = tz*q[1], tzz = tz*q[2];                                                  \
    R[0] = 1-(tyy+tzz); R[1] = txy-twz; R[2] = txz+twy;                                             \
    R[3] = txy+twz; R[4] = 1-(txx+tzz); R[5] = tyz-twx;                                             \
    R[6] = txz-twy; R[7] = tyz+twx; R[8] = 1-(txx+tyy);                                             \
}                                                                                                   \
void lsdo_se3##SUF##_matrix(const T a[7], T R[9], T t[3])                                           \
{ quat_to_R_##SUF(a, R); t[0] = a[4]; t[1] = a[5]; t[2] = a[6]; }                                   \
void lsdo_se3##SUF##_mul(const T a[7], const T b[7], T out[7])                                      \
{   /* se3.hpp:159-162 fastMultiply + normalize (operator*=, :256-259) */                           \
    T rt[3], q[4];                                                                                  \
    quat_rot_##SUF(a, b+4, rt);                                                                     \
    quat_mul_##SUF(a, b, q);                                                                        \
    quat_normalize_##SUF(q);                                                                        \
    out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];                                     \
    out[4] = a[4] + rt[0]; out[5] = a[5] + rt[1]; out[6] = a[6] + rt[2];                            \
}                                                                                                   \
void lsdo_se3##SUF##_inverse(const T a[7], T out[7])                                                \
{   /* se3.hpp:167-172; SO3 inverse = conjugate + normalising ctor (so3.hpp:173-175,631-633) */     \
    T q[4] = { -a[0], -a[1], -a[2], a[3] };                                                         \
    quat_normalize_##SUF(q);                                                                        \
    T nt[3] = { a[4]*(T)-1, a[5]*(T)-1, a[6]*(T)-1 }, r[3];                                         \
    quat_rot_##SUF(q, nt, r);                                                                       \
    out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];                                     \
    out[4] = r[0]; out[5] = r[1]; out[6] = r[2];                                                    \
}                                                                                                   \
void lsdo_se3##SUF##_exp(const T a[6], T out[7])                                                    \
{   /* se3.hpp:406-428 with so3.hpp:342-369 (expAndTheta); tangent = [upsilon, omega] */            \
    const T* om = a + 3;                                                                            \
    T theta_sq = om[0]*om[0] + (om[1]*om[1] + om[2]*om[2]);     /* omega.squaredNorm(): 1 + 2 tree */  \
    T theta = SQRT(theta_sq);                                                                       \
    T half_theta = (T)0.5*theta;                                                                    \
    T imag_factor, real_factor;                                                                     \
    if (theta < (T)EPS) {                                                                           \
        T theta_po4 = theta_sq*theta_sq;                                                            \
        imag_factor = (T)0.5 - (T)(1.0/48.0)*theta_sq + (T)(1.0/3840.0)*theta_po4;                  \
        real_factor = (T)1 - (T)0.5*theta_sq + (T)(1.0/384.0)*theta_po4;                            \
    } else {                                                                                        \
        T sin_half_theta = SIN(half_theta);                                                         \
        imag_factor = sin_half_theta/theta;                                                         \
        real_factor = COS(half_theta);                                                              \
    }                                                                                               \
    T q[4] = { imag_factor*om[0], imag_factor*om[1], imag_factor*om[2], real_factor };              \
    quat_normalize_##SUF(q);                                                                        \
    /* Omega = hat(omega), so3.hpp hat(): [0 -z y; z 0 -x; -y x 0] */                               \
    T Om[9] = { 0, -om[2], om[1],  om[2], 0, -om[0],  -om[1], om[0], 0 };                           \
    T Om2[9];                                                                                       \
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)                                         \
        Om2[i*3+j] = (Om[i*3+0]*Om[0*3+j] + Om[i*3+1]*Om[1*3+j]) + Om[i*3+2]*Om[2*3+j];             \
    T V[9];                                                                                         \
    if (theta < (T)EPS) {                                                                           \
        quat_to_R_##SUF(q, V);                                                                      \
    } else {                                                                                        \
        T tsq = theta*theta;            /* se3.hpp:419 recomputes theta_sq from theta */             \
        T c1 = ((T)1 - COS(theta))/tsq;                                                             \
        T c2 = (theta - SIN(theta))/(tsq*theta);                                                    \
        for (int i = 0; i < 9; i++) V[i] = (((i%4)==0 ? (T)1 : (T)0) + c1*Om[i]) + c2*Om2[i];       \
    }                                                                                               \
    out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];                                     \
    for (int i = 0; i < 3; i++) out[4+i] = (V[i*3+0]*a[0] + V[i*3+1]*a[1]) + V[i*3+2]*a[2];         \
}

DEFINE_SE3(double, d, sqrt, sin, cos, 1e-10)
DEFINE_SE3(float,  f, sqrtf, sinf, cosf, 1e-5)

/* SE3 log (se3.hpp:340-380 / so3.hpp logAndTheta) -- double only, used by tests and the generator */
void lsdo_se3d_log(const double a[7], double out[6])
{
    double n2 = a[0]*a[0] + a[1]*a[1] + a[2]*a[2];
    double n = sqrt(n2), w = a[3];
    double two_atan_nbyw_by_n;
    if (n < 1e-10) {
        double sw = w*w;
        two_atan_nbyw_by_n = 2.0/w - 2.0*n2/(w*sw);
    } else if (fabs(w) < 1e-10) {
        two_atan_nbyw_by_n = (w > 0 ? M_PI : -M_PI)/n;
    } else {
        two_atan_nbyw_by_n = 2.0*atan(n/w)/n;
    }
    double om[3] = { two_atan_nbyw_by_n*a[0], two_atan_nbyw_by_n*a[1], two_atan_nbyw_by_n*a[2] };
    double theta = sqrt(om[0]*om[0] + om[1]*om[1] + om[2]*om[2]);
    double Om[9] = { 0, -om[2], om[1],  om[2], 0, -om[0],  -om[1], om[0], 0 };
    double Om2[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
        Om2[i*3+j] = Om[i*3+0]*Om[0*3+j] + Om[i*3+1]*Om[1*3+j] + Om[i*3+2]*Om[2*3+j];
    double Vinv[9];
    if (theta < 1e-10) {
        for (int i = 0; i < 9; i++) Vinv[i] = ((i%4)==0 ? 1.0 : 0.0) - 0.5*Om[i] + (1.0/12.0)*Om2[i];
    } else {
        double c = (1.0 - theta*cos(0.5*theta)/(2.0*sin(0.5*theta)))/(theta*theta);
        for (int i = 0; i < 9; i++) Vinv[i] = ((i%4)==0 ? 1.0 : 0.0) - 0.5*Om[i] + c*Om2[i];
    }
    for (int i = 0; i < 3; i++) out[i] = Vinv[i*3+0]*a[4] + Vinv[i*3+1]*a[5] + Vinv[i*3+2]*a[6];
    out[3] = om[0]; out[4] = om[1]; out[5] = om[2];
}

/* SE3d -> SE3f cast (se3.hpp cast<>: quaternion and translation cast, normalising ctor) */
static void se3_d2f(const double a[7], float o[7])
{
    float q[4] = { (float)a[0], (float)a[1], (float)a[2], (float)a[3] };
    quat_normalize_f(q);
    o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3];
    o[4] = (float)a[4]; o[5] = (float)a[5]; o[6] = (float)a[6];
}
static void se3_f2d(const float a[7], double o[7])
{
    double q[4] = { a[0], a[1], a[2], a[3] };
    quat_normalize_d(q);
    o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3];
    o[4] = a[4]; o[5] = a[5]; o[6] = a[6];
}

/* ------------------------------------------------------------------------------------------
 * Frame, DataStructures/Frame.{h,cpp}
 * ---------------------------------------------------------------------------------------- */
struct lsdo_frame {
    int id;
    int width[LSDO_LEVELS], height[LSDO_LEVELS];
    float K[LSDO_LEVELS][9], KInv[LSDO_LEVELS][9];
    float fx[LSDO_LEVELS], fy[LSDO_LEVELS], cx[LSDO_LEVELS], cy[LSDO_LEVELS];
    float fxInv[LSDO_LEVELS], fyInv[LSDO_LEVELS], cxInv[LSDO_LEVELS], cyInv[LSDO_LEVELS];
    float* image[LSDO_LEVELS];       int imageValid[LSDO_LEVELS];
    float* gradients[LSDO_LEVELS];   int gradientsValid[LSDO_LEVELS];   /* Vector4f per px */
    float* maxGradients[LSDO_LEVELS];int maxGradientsValid[LSDO_LEVELS];
    float* idepth[LSDO_LEVELS];      int idepthValid[LSDO_LEVELS];
    float* idepthVar[LSDO_LEVELS];   int idepthVarValid[LSDO_LEVELS];
    int hasIDepthBeenSet, depthHasBeenUpdatedFlag;
    uint8_t* refPixelWasGood;
    float* idepth_reAct; float* idepthVar_reAct; uint8_t* validity_reAct; int reActivationDataValid;   /* Frame.h data.*_reAct */
    int numMappablePixels;
    float meanIdepth; int numPoints;
    int numFramesTrackedOnThis, numMappedOnThis, numMappedOnThisTotal;
    float initialTrackedResidual;
    /* FramePoseStruct: thisToParent_raw (Sim3 as unit q, t, s) + trackingParent */
    double thisToParent_q[4], thisToParent_t[3], thisToParent_s;
    lsdo_frame* trackingParent;
    /* prepareForStereoWith results, Frame.h:160-175 */
    float K_otherToThis_R[9], K_otherToThis_t[3], otherToThis_t[3];
    float thisToOther_t[3], K_thisToOther_t[3], thisToOther_R[9];
    float otherToThis_R_row0[3], otherToThis_R_row1[3], otherToThis_R_row2[3];
    float distSquared; int referenceID, referenceLevel;
};

static void frame_initialize(lsdo_frame* f, int id, int width, int height, const float K[9])
{   /* Frame.cpp:397-484 */
    memset(f, 0, sizeof(*f));
    f->id = id;
    memcpy(f->K[0], K, 9*sizeof(float));
    f->fx[0] = K[0]; f->fy[0] = K[4]; f->cx[0] = K[2]; f->cy[0] = K[5];
    lsdo_mat3_inverse(f->K[0], f->KInv[0]);
    f->fxInv[0] = f->KInv[0][0]; f->fyInv[0] = f->KInv[0][4]; f->cxInv[0] = f->KInv[0][2]; f->cyInv[0] = f->KInv[0][5];
    f->referenceID = -1; f->referenceLevel = -1; f->numMappablePixels = -1;
    for (int level = 0; level < LSDO_LEVELS; ++level) {
        f->width[level] = width >> level;
        f->height[level] = height >> level;
        if (level > 0) {
            f->fx[level] = f->fx[level-1] * 0.5;
            f->fy[level] = f->fy[level-1] * 0.5;
            f->cx[level] = (f->cx[0] + 0.5) / ((int)1<<level) - 0.5;
            f->cy[level] = (f->cy[0] + 0.5) / ((int)1<<level) - 0.5;
            float* Kl = f->K[level];
            Kl[0] = f->fx[level]; Kl[1] = 0.0; Kl[2] = f->cx[level];
            Kl[3] = 0.0; Kl[4] = f->fy[level]; Kl[5] = f->cy[level];
            Kl[6] = 0.0; Kl[7] = 0.0; Kl[8] = 1.0;
            lsdo_mat3_inverse(Kl, f->KInv[level]);
            f->fxInv[level] = f->KInv[level][0]; f->fyInv[level] = f->KInv[level][4];
            f->cxInv[level] = f->KInv[level][2]; f->cyInv[level] = f->KInv[level][5];
        }
    }
    f->meanIdepth = 1; f->numPoints = 0;
    f->thisToParent_q[3] = 1; f->thisToParent_s = 1;
}

lsdo_frame* lsdo_frame_create_u8(int id, int w, int h, const float K[9], const uint8_t* image)
{   /* Frame.cpp:35-54 */
    lsdo_frame* f = (lsdo_frame*)malloc(sizeof(lsdo_frame));
    frame_initialize(f, id, w, h, K);
    f->image[0] = (float*)calloc((size_t)w*h, sizeof(float));
    for (int i = 0; i < w*h; i++) f->image[0][i] = image[i];
    f->imageValid[0] = 1;
    return f;
}

void lsdo_frame_destroy(lsdo_frame* f)
{
    if (!f) return;
    for (int l = 0; l < LSDO_LEVELS; l++) {
        free(f->image[l]); free(f->gradients[l]); free(f->maxGradients[l]); free(f->idepth[l]); free(f->idepthVar[l]);
    }
    free(f->refPixelWasGood);
    free(f->idepth_reAct); free(f->idepthVar_reAct); free(f->validity_reAct);
    free(f);
}

static void frame_buildImage(lsdo_frame* f, int level);
static void frame_requireImage(lsdo_frame* f, int level) { if (!f->imageValid[level]) frame_buildImage(f, level); }

static void frame_buildImage(lsdo_frame* f, int level)
{   /* Frame.cpp:491-630, scalar loop :614-627 (exact for u8-origin data, SURVEY App. A-11) */
    if (level == 0) return;
    frame_requireImage(f, level-1);
    int width = f->width[level-1], height = f->height[level-1];
    const float* source = f->image[level-1];
    if (!f->image[level]) f->image[level] = (float*)calloc((size_t)f->width[level]*f->height[level], sizeof(float));
    float* dest = f->image[level];
    int wh = width*height;
    for (int y = 0; y < wh; y += width*2)
        for (int x = 0; x < width; x += 2) {
            const float* s = source + x + y;
            *dest = (s[0] + s[1] + s[width] + s[1+width]) * 0.25f;
            dest++;
        }
    f->imageValid[level] = 1;
}

static void frame_buildGradients(lsdo_frame* f, int level)
{   /* Frame.cpp:643-680.  Linear sweep from row 1 to row h-2 inclusive: x=0 / x=w-1 wrap across rows. */
    frame_requireImage(f, level);
    if (f->gradientsValid[level]) return;
    int width = f->width[level], height = f->height[level];
    if (!f->gradients[level]) f->gradients[level] = (float*)calloc((size_t)4*width*height, sizeof(float));
    const float* img_pt = f->image[level] + width;
    const float* img_pt_max = f->image[level] + width*(height-1);
    float* g = f->gradients[level] + 4*width;
    float val_m1 = *(img_pt-1), val_00 = *img_pt, val_p1;
    for (; img_pt < img_pt_max; img_pt++, g += 4) {
        val_p1 = *(img_pt+1);
        g[0] = 0.5f*(val_p1 - val_m1);
        g[1] = 0.5f*(*(img_pt+width) - *(img_pt-width));
        g[2] = val_00;
        val_m1 = val_00; val_00 = val_p1;
    }
    f->gradientsValid[level] = 1;
}

static void frame_buildMaxGradients(lsdo_frame* f, int level)
{   /* Frame.cpp:690-767; temp + destination zero-filled (App. A-12) */
    if (!f->gradientsValid[level]) frame_buildGradients(f, level);
    if (f->maxGradientsValid[level]) return;
    int width = f->width[level], height = f->height[level];
    if (!f->maxGradients[level]) f->maxGradients[level] = (float*)calloc((size_t)width*height, sizeof(float));
    float* maxGradTemp = (float*)calloc((size_t)width*height, sizeof(float));
    const float* g = f->gradients[level] + 4*width;
    float* maxgrad_pt = f->maxGradients[level] + width;
    float* maxgrad_pt_max = f->maxGradients[level] + width*(height-1);
    for (; maxgrad_pt < maxgrad_pt_max; maxgrad_pt++, g += 4) {
        float dx = g[0], dy = g[1];
        *maxgrad_pt = sqrtf(dx*dx + dy*dy);
    }
    maxgrad_pt = f->maxGradients[level] + width+1;
    maxgrad_pt_max = f->maxGradients[level] + width*(height-1)-1;
    float* maxgrad_t_pt = maxGradTemp + width+1;
    for (; maxgrad_pt < maxgrad_pt_max; maxgrad_pt++, maxgrad_t_pt++) {
        float g1 = maxgrad_pt[-width], g2 = maxgrad_pt[0];
        if (g1 < g2) g1 = g2;
        float g3 = maxgrad_pt[width];
        *maxgrad_t_pt = (g1 < g3) ? g3 : g1;
    }
    float numMappablePixels = 0;
    maxgrad_pt = f->maxGradients[level] + width+1;
    maxgrad_pt_max = f->maxGradients[level] + width*(height-1)-1;
    maxgrad_t_pt = maxGradTemp + width+1;
    for (; maxgrad_pt < maxgrad_pt_max; maxgrad_pt++, maxgrad_t_pt++) {
        float g1 = maxgrad_t_pt[-1], g2 = maxgrad_t_pt[0];
        if (g1 < g2) g1 = g2;
        float g3 = maxgrad_t_pt[1];
        if (g1 < g3) { *maxgrad_pt = g3; if (g3 >= MIN_ABS_GRAD_CREATE) numMappablePixels++; }
        else         { *maxgrad_pt = g1; if (g1 >= MIN_ABS_GRAD_CREATE) numMappablePixels++; }
    }
    if (level == 0) f->numMappablePixels = numMappablePixels;
    free(maxGradTemp);
    f->maxGradientsValid[level] = 1;
}

static void frame_buildIDepthAndIDepthVar(lsdo_frame* f, int level)
{   /* Frame.cpp:775-877 */
    if (!f->hasIDepthBeenSet || level == 0) return;
    if (!f->idepthValid[level-1]) frame_buildIDepthAndIDepthVar(f, level-1);
    if (f->idepthValid[level] && f->idepthVarValid[level]) return;
    int width = f->width[level], height = f->height[level];
    if (!f->idepth[level]) f->idepth[level] = (float*)calloc((size_t)width*height, sizeof(float));
    if (!f->idepthVar[level]) f->idepthVar[level] = (float*)calloc((size_t)width*height, sizeof(float));
    int sw = f->width[level-1];
    const float* idepthSource = f->idepth[level-1];
    const float* idepthVarSource = f->idepthVar[level-1];
    float* idepthDest = f->idepth[level];
    float* idepthVarDest = f->idepthVar[level];
    for (int y = 0; y < height; y++)
        for (int x = 0; x < width; x++) {
            int idx = 2*(x+y*sw);
            int idxDest = (x+y*width);
            float idepthSumsSum = 0, ivarSumsSum = 0;
            int num = 0;
            float ivar, var;
            static const int dofs[4][2] = {{0,0},{1,0},{0,1},{1,1}};
            for (int k = 0; k < 4; k++) {
                int o = idx + dofs[k][0] + dofs[k][1]*sw;
                var = idepthVarSource[o];
                if (var > 0) {
                    ivar = 1.0f / var;
                    ivarSumsSum += ivar;
                    idepthSumsSum += ivar * idepthSource[o];
                    num++;
                }
            }
            if (num > 0) {
                float depth = ivarSumsSum / idepthSumsSum;
                idepthDest[idxDest] = 1.0f / depth;
                idepthVarDest[idxDest] = num / ivarSumsSum;
            } else {
                idepthDest[idxDest] = -1;
                idepthVarDest[idxDest] = -1;
            }
        }
    f->idepthValid[level] = 1;
    f->idepthVarValid[level] = 1;
}

static void frame_releaseIDepthPyr(lsdo_frame* f)
{   /* Frame::release(IDEPTH|IDEPTH_VAR, pyramidsOnly=true) -- levels >= 1 become invalid */
    for (int l = 1; l < LSDO_LEVELS; l++) { f->idepthValid[l] = 0; f->idepthVarValid[l] = 0; }
}

int lsdo_frame_id(const lsdo_frame* f) { return f->id; }
int lsdo_frame_width(const lsdo_frame* f, int l) { return f->width[l]; }
int lsdo_frame_height(const lsdo_frame* f, int l) { return f->height[l]; }
const float* lsdo_frame_image(lsdo_frame* f, int l) { frame_requireImage(f, l); return f->image[l]; }
const float* lsdo_frame_gradients(lsdo_frame* f, int l) { if (!f->gradientsValid[l]) frame_buildGradients(f, l); return f->gradients[l]; }
const float* lsdo_frame_maxGradients(lsdo_frame* f, int l) { if (!f->maxGradientsValid[l]) frame_buildMaxGradients(f, l); return f->maxGradients[l]; }
const float* lsdo_frame_idepth(lsdo_frame* f, int l) { if (!f->hasIDepthBeenSet) return 0; if (!f->idepthValid[l]) frame_buildIDepthAndIDepthVar(f, l); return f->idepth[l]; }
const float* lsdo_frame_idepthVar(lsdo_frame* f, int l) { if (!f->hasIDepthBeenSet) return 0; if (!f->idepthVarValid[l]) frame_buildIDepthAndIDepthVar(f, l); return f->idepthVar[l]; }
void lsdo_frame_K(const lsdo_frame* f, int l, float K[9], float Kinv[9]) { memcpy(K, f->K[l], 36); memcpy(Kinv, f->KInv[l], 36); }

uint8_t* lsdo_frame_refPixelWasGood(lsdo_frame* f)
{   /* Frame.h:421-437 */
    if (!f->refPixelWasGood) {
        int n = f->width[SE3TRACKING_MIN_LEVEL]*f->height[SE3TRACKING_MIN_LEVEL];
        f->refPixelWasGood = (uint8_t*)malloc(n);
        memset(f->refPixelWasGood, 1, n);
    }
    return f->refPixelWasGood;
}
uint8_t* lsdo_frame_refPixelWasGoodNoCreate(lsdo_frame* f) { return f->refPixelWasGood; }
void lsdo_frame_clear_refPixelWasGood(lsdo_frame* f) { free(f->refPixelWasGood); f->refPixelWasGood = 0; }

void lsdo_frame_setDepth(lsdo_frame* f, const lsdo_hyp* newDepth)
{   /* Frame.cpp:199-243 */
    int n = f->width[0]*f->height[0];
    if (!f->idepth[0]) f->idepth[0] = (float*)calloc(n, sizeof(float));
    if (!f->idepthVar[0]) f->idepthVar[0] = (float*)calloc(n, sizeof(float));
    float sumIdepth = 0; int numIdepth = 0;
    for (int i = 0; i < n; i++, newDepth++) {
        if (newDepth->isValid && newDepth->idepth_smoothed >= -0.05) {
            f->idepth[0][i] = newDepth->idepth_smoothed;
            f->idepthVar[0][i] = newDepth->idepth_var_smoothed;
            numIdepth++;
            sumIdepth += newDepth->idepth_smoothed;
        } else {
            f->idepth[0][i] = -1;
            f->idepthVar[0][i] = -1;
        }
    }
    f->meanIdepth = sumIdepth / numIdepth;
    f->numPoints = numIdepth;
    f->idepthValid[0] = 1; f->idepthVarValid[0] = 1;
    frame_releaseIDepthPyr(f);
    f->hasIDepthBeenSet = 1;
    f->depthHasBeenUpdatedFlag = 1;
}

void lsdo_frame_setDepthFromGroundTruth(lsdo_frame* f, const float* depth, float cov_scale)
{   /* Frame.cpp:245-293 */
    const float* pyrMaxGradient = lsdo_frame_maxGradients(f, 0);
    int width0 = f->width[0], height0 = f->height[0];
    if (!f->idepth[0]) f->idepth[0] = (float*)calloc((size_t)width0*height0, sizeof(float));
    if (!f->idepthVar[0]) f->idepthVar[0] = (float*)calloc((size_t)width0*height0, sizeof(float));
    float* pyrIDepth = f->idepth[0];
    float* pyrIDepthVar = f->idepthVar[0];
    for (int y = 0; y < height0; y++)
        for (int x = 0; x < width0; x++) {
            if (x > 0 && x < width0-1 && y > 0 && y < height0-1 &&
                pyrMaxGradient[x+y*width0] >= MIN_ABS_GRAD_CREATE &&
                !isnan(*depth) && *depth > 0) {
                *pyrIDepth = 1.0f / *depth;
                *pyrIDepthVar = VAR_GT_INIT_INITIAL * cov_scale;
            } else {
                *pyrIDepth = -1;
                *pyrIDepthVar = -1;
            }
            ++depth; ++pyrIDepth; ++pyrIDepthVar;
        }
    f->idepthValid[0] = 1; f->idepthVarValid[0] = 1;
    frame_releaseIDepthPyr(f);
    f->hasIDepthBeenSet = 1;
}

/* Frame::takeReActivationData, DataStructures/Frame.cpp:107-145.  Pool buffers are defined zero-filled (SURVEY appendix A.12);
 * entries of invalid pixels keep their previous content, as in the reference. */
void lsdo_frame_takeReActivationData(lsdo_frame* f, const lsdo_hyp* depthMap)
{
    size_t n = (size_t)f->width[0]*f->height[0];
    if (f->validity_reAct == 0) f->validity_reAct = (uint8_t*)calloc(n, 1);
    if (f->idepth_reAct == 0) f->idepth_reAct = (float*)calloc(n, sizeof(float));
    if (f->idepthVar_reAct == 0) f->idepthVar_reAct = (float*)calloc(n, sizeof(float));
    float* id_pt = f->idepth_reAct; float* id_pt_max = f->idepth_reAct + n;
    float* idv_pt = f->idepthVar_reAct; uint8_t* val_pt = f->validity_reAct;
    for (; id_pt < id_pt_max; ++id_pt, ++idv_pt, ++val_pt, ++depthMap) {
        if (depthMap->isValid) {
            *id_pt = depthMap->idepth;
            *idv_pt = depthMap->idepth_var;
            *val_pt = depthMap->validity_counter;
        } else if (depthMap->blacklisted < MIN_BLACKLIST) {
            *idv_pt = -2;
        } else {
            *idv_pt = -1;
        }
    }
    f->reActivationDataValid = 1;
}
const float* lsdo_frame_idepth_reAct(const lsdo_frame* f) { return f->idepth_reAct; }
const float* lsdo_frame_idepthVar_reAct(const lsdo_frame* f) { return f->idepthVar_reAct; }
const uint8_t* lsdo_frame_validity_reAct(const lsdo_frame* f) { return f->validity_reAct; }

/* ROSOutput3DWrapper::publishKeyframe packing loop, IOWrapper/ROS/ROSOutput3DWrapper.cpp:91-110; InputPointDense
 * {float idepth; float idepth_var; uchar color[4];} ROSOutput3DWrapper.h:34-39 (= keyframeMsg.pointcloud, 12 B per pixel) */
void lsdo_pack_pointcloud(lsdo_frame* f, int publishLvl, void* out)
{
    int w = f->width[publishLvl], h = f->height[publishLvl];
    struct { float idepth; float idepth_var; unsigned char color[4]; }* pc = out;
    const float* idepth = lsdo_frame_idepth(f, publishLvl);
    const float* idepthVar = lsdo_frame_idepthVar(f, publishLvl);
    const float* color = lsdo_frame_image(f, publishLvl);
    for (int idx = 0; idx < w*h; idx++) {
        pc[idx].idepth = idepth[idx];
        pc[idx].idepth_var = idepthVar[idx];
        pc[idx].color[0] = color[idx];
        pc[idx].color[1] = color[idx];
        pc[idx].color[2] = color[idx];
        pc[idx].color[3] = color[idx];
    }
}

int   lsdo_frame_numMappablePixels(lsdo_frame* f) { lsdo_frame_maxGradients(f, 0); return f->numMappablePixels; }
float lsdo_frame_meanIdepth(const lsdo_frame* f) { return f->meanIdepth; }
int   lsdo_frame_numPoints(const lsdo_frame* f) { return f->numPoints; }
int   lsdo_frame_depthHasBeenUpdatedFlag(const lsdo_frame* f) { return f->depthHasBeenUpdatedFlag; }
void  lsdo_frame_set_depthHasBeenUpdatedFlag(lsdo_frame* f, int v) { f->depthHasBeenUpdatedFlag = v; }
float lsdo_frame_initialTrackedResidual(const lsdo_frame* f) { return f->initialTrackedResidual; }
void  lsdo_frame_get_thisToParent(const lsdo_frame* f, double o[8])
{ memcpy(o, f->thisToParent_q, 32); memcpy(o+4, f->thisToParent_t, 24); o[7] = f->thisToParent_s; }
void  lsdo_frame_set_thisToParent(lsdo_frame* f, const double o[8], lsdo_frame* parent)
{ memcpy(f->thisToParent_q, o, 32); memcpy(f->thisToParent_t, o+4, 24); f->thisToParent_s = o[7]; f->trackingParent = parent; }
int   lsdo_frame_numFramesTrackedOnThis(const lsdo_frame* f) { return f->numFramesTrackedOnThis; }
int   lsdo_frame_numMappedOnThis(const lsdo_frame* f) { return f->numMappedOnThis; }
void  lsdo_frame_set_counters(lsdo_frame* f, int tracked, int mapped) { f->numFramesTrackedOnThis = tracked; f->numMappedOnThis = mapped; }

/* Frame::prepareForStereoWith, Frame.cpp:295-317.  thisToOther = (q,t,s) double; K = level-0 K. */
static void frame_prepareForStereoWith(lsdo_frame* f, lsdo_frame* other, const double q[4], const double t[3], double s, const float K[9])
{
    /* Sim3 inverse (sim3.hpp:169-173, rxso3.hpp:195-200,263-269) */
    double qi[4] = { -q[0], -q[1], -q[2], q[3] };
    double si = 1.0/s;
    double nt[3] = { t[0]*-1.0, t[1]*-1.0, t[2]*-1.0 }, rt[3];
    quat_rot_d(qi, nt, rt);
    double oTt_t[3] = { si*rt[0], si*rt[1], si*rt[2] };
    double Ri[9]; quat_to_R_d(qi, Ri);
    double R[9];  quat_to_R_d(q, R);
    /* K_otherToThis_R = K * otherToThis.rotationMatrix().cast<float>() * otherToThis.scale(); */
    float Rif[9]; for (int i = 0; i < 9; i++) Rif[i] = (float)Ri[i];
    float KR[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
        KR[i*3+j] = (K[i*3+0]*Rif[0*3+j] + K[i*3+1]*Rif[1*3+j]) + K[i*3+2]*Rif[2*3+j];
    /* Matrix3f * double: Eigen converts the scalar to float first (operator*(const Scalar&)) */
    for (int i = 0; i < 9; i++) f->K_otherToThis_R[i] = KR[i] * (float)si;
    for (int i = 0; i < 3; i++) f->otherToThis_t[i] = (float)oTt_t[i];
    for (int i = 0; i < 3; i++)
        f->K_otherToThis_t[i] = (K[i*3+0]*f->otherToThis_t[0] + K[i*3+1]*f->otherToThis_t[1]) + K[i*3+2]*f->otherToThis_t[2];
    for (int i = 0; i < 3; i++) f->thisToOther_t[i] = (float)t[i];
    for (int i = 0; i < 3; i++)
        f->K_thisToOther_t[i] = (K[i*3+0]*f->thisToOther_t[0] + K[i*3+1]*f->thisToOther_t[1]) + K[i*3+2]*f->thisToOther_t[2];
    for (int i = 0; i < 9; i++) f->thisToOther_R[i] = (float)R[i] * (float)s;
    for (int i = 0; i < 3; i++) {   /* rows of otherToThis_R == columns of thisToOther_R */
        f->otherToThis_R_row0[i] = f->thisToOther_R[i*3+0];
        f->otherToThis_R_row1[i] = f->thisToOther_R[i*3+1];
        f->otherToThis_R_row2[i] = f->thisToOther_R[i*3+2];
    }
    f->distSquared = (float)(oTt_t[0]*oTt_t[0] + oTt_t[1]*oTt_t[1] + oTt_t[2]*oTt_t[2]);
    f->referenceID = other->id;
    f->referenceLevel = 0;
}

/* test hooks shared with oracle/ref_driver.cpp (the reference-compiled twin exports the same names) */
void lsdo_frame_set_initialTrackedResidual(lsdo_frame* f, float v) { f->initialTrackedResidual = v; }
void lsdo_ref_prepareForStereoWith(lsdo_frame* frame, lsdo_frame* kf, const double thisToOther_qts[8], const float K[9], float out[30])
{
    frame_prepareForStereoWith(frame, kf, thisToOther_qts, thisToOther_qts + 4, thisToOther_qts[7], K);
    int k = 0;
    for (int i = 0; i < 9; i++) out[k++] = frame->K_otherToThis_R[i];
    for (int i = 0; i < 3; i++) out[k++] = frame->K_otherToThis_t[i];
    for (int i = 0; i < 3; i++) out[k++] = frame->otherToThis_t[i];
    for (int i = 0; i < 3; i++) out[k++] = frame->thisToOther_t[i];
    for (int i = 0; i < 3; i++) out[k++] = frame->otherToThis_R_row0[i];
    for (int i = 0; i < 3; i++) out[k++] = frame->otherToThis_R_row1[i];
    for (int i = 0; i < 3; i++) out[k++] = frame->otherToThis_R_row2[i];
    out[k++] = frame->distSquared;
    out[k++] = (float)frame->referenceID;
    out[k++] = (float)frame->referenceLevel;
}

/* ------------------------------------------------------------------------------------------
 * interpolation, util/globalFuncs.h:43-109
 * ---------------------------------------------------------------------------------------- */
static inline float getInterpolatedElement(const float* mat, float x, float y, int width)
{
    int ix = (int)x, iy = (int)y;
    float dx = x - ix, dy = y - iy;
    float dxdy = dx*dy;
    const float* bp = mat + ix + iy*width;
    float res = dxdy * bp[1+width] + (dy-dxdy) * bp[width] + (dx-dxdy) * bp[1] + (1-dx-dy+dxdy) * bp[0];
    return res;
}
/* getInterpolatedElement43 / 42: n = 3 or 2 lanes of a Vector4f image */
static inline void getInterpolatedElement4n(const float* mat4, float x, float y, int width, int n, float* out)
{
    int ix = (int)x, iy = (int)y;
    float dx = x - ix, dy = y - iy;
    float dxdy = dx*dy;
    const float* bp = mat4 + 4*(ix + iy*width);
    float w0 = dxdy, w1 = (dy-dxdy), w2 = (dx-dxdy), w3 = (1-dx-dy+dxdy);
    for (int k = 0; k < n; k++)
        out[k] = w0 * bp[4*(1+width)+k] + w1 * bp[4*width+k] + w2 * bp[4+k] + w3 * bp[k];
}

/* ------------------------------------------------------------------------------------------
 * TrackingReference::makePointCloud, Tracking/TrackingReference.cpp:96-147
 * ---------------------------------------------------------------------------------------- */
int lsdo_make_point_cloud(lsdo_frame* kf, int level, float* posData, float* gradData, float* colorAndVarData, int* pointPosInXYGrid)
{
    int w = kf->width[level], h = kf->height[level];
    float fxInvLevel = kf->fxInv[level], fyInvLevel = kf->fyInv[level];
    float cxInvLevel = kf->cxInv[level], cyInvLevel = kf->cyInv[level];
    const float* pyrIdepthSource = lsdo_frame_idepth(kf, level);
    const float* pyrIdepthVarSource = lsdo_frame_idepthVar(kf, level);
    const float* pyrColorSource = lsdo_frame_image(kf, level);
    const float* pyrGradSource = lsdo_frame_gradients(kf, level);
    int n = 0;
    for (int x = 1; x < w-1; x++)
        for (int y = 1; y < h-1; y++) {
            int idx = x + y*w;
            if (pyrIdepthVarSource[idx] <= 0 || pyrIdepthSource[idx] == 0) continue;
            float s = (1.0f / pyrIdepthSource[idx]);
            if (posData) {
                posData[3*n+0] = s * (fxInvLevel*x+cxInvLevel);
                posData[3*n+1] = s * (fyInvLevel*y+cyInvLevel);
                posData[3*n+2] = s * 1;
            }
            if (gradData) { gradData[2*n] = pyrGradSource[4*idx]; gradData[2*n+1] = pyrGradSource[4*idx+1]; }
            if (colorAndVarData) { colorAndVarData[2*n] = pyrColorSource[idx]; colorAndVarData[2*n+1] = pyrIdepthVarSource[idx]; }
            if (pointPosInXYGrid) pointPosInXYGrid[n] = idx;
            n++;
        }
    return n;
}

/* ------------------------------------------------------------------------------------------
 * SE3Tracker, Tracking/SE3Tracker.cpp + LGS6, Tracking/LGSX.h:184-402
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    float A[36], b[6], error; size_t num_constraints;
    float SSEData[4*28] __attribute__((aligned(16)));
    double dA[36], db[6], derror;     /* diagnostic twin (lsdo_globals.exactTrackingSums): the same terms accumulated in double */
} LGS6;

static void lgs6_initialize(LGS6* ls) { memset(ls, 0, sizeof(*ls)); }
static inline void lgs6_update(LGS6* ls, const float J[6], float res, float weight)
{   /* LGSX.h:390-396 */
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) ls->A[i*6+j] += J[i]*J[j]*weight;
    float rw = res*weight;
    for (int i = 0; i < 6; i++) ls->b[i] -= J[i]*rw;
    ls->error += res*res*weight;
    ls->num_constraints += 1;
    if (G.exactTrackingSums) {        /* the same fp32 terms, summed without accumulation error */
        for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) ls->dA[i*6+j] += (double)(J[i]*J[j]*weight);
        for (int i = 0; i < 6; i++) ls->db[i] -= (double)(J[i]*rw);
        ls->derror += (double)(res*res*weight);
    }
}
static inline void lgs6_updateSSE(LGS6* ls, __m128 J1, __m128 J2, __m128 J3, __m128 J4, __m128 J5, __m128 J6, __m128 res, __m128 weight)
{   /* LGSX.h:328-386 */
    float* S = ls->SSEData;
#define ACC(k, v) _mm_store_ps(S+4*(k), _mm_add_ps(_mm_load_ps(S+4*(k)), (v)))
    __m128 J1w = _mm_mul_ps(J1, weight);
    ACC(0, _mm_mul_ps(J1w,J1)); ACC(1, _mm_mul_ps(J1w,J2)); ACC(2, _mm_mul_ps(J1w,J3));
    ACC(3, _mm_mul_ps(J1w,J4)); ACC(4, _mm_mul_ps(J1w,J5)); ACC(5, _mm_mul_ps(J1w,J6));
    __m128 J2w = _mm_mul_ps(J2, weight);
    ACC(6, _mm_mul_ps(J2w,J2)); ACC(7, _mm_mul_ps(J2w,J3)); ACC(8, _mm_mul_ps(J2w,J4));
    ACC(9, _mm_mul_ps(J2w,J5)); ACC(10, _mm_mul_ps(J2w,J6));
    __m128 J3w = _mm_mul_ps(J3, weight);
    ACC(11, _mm_mul_ps(J3w,J3)); ACC(12, _mm_mul_ps(J3w,J4)); ACC(13, _mm_mul_ps(J3w,J5)); ACC(14, _mm_mul_ps(J3w,J6));
    __m128 J4w = _mm_mul_ps(J4, weight);
    ACC(15, _mm_mul_ps(J4w,J4)); ACC(16, _mm_mul_ps(J4w,J5)); ACC(17, _mm_mul_ps(J4w,J6));
    __m128 J5w = _mm_mul_ps(J5, weight);
    ACC(18, _mm_mul_ps(J5w,J5)); ACC(19, _mm_mul_ps(J5w,J6));
    __m128 J6w = _mm_mul_ps(J6, weight);
    ACC(20, _mm_mul_ps(J6w,J6));
    __m128 resw = _mm_mul_ps(res, weight);
    ACC(21, _mm_mul_ps(resw,J1)); ACC(22, _mm_mul_ps(resw,J2)); ACC(23, _mm_mul_ps(resw,J3));
    ACC(24, _mm_mul_ps(resw,J4)); ACC(25, _mm_mul_ps(resw,J5)); ACC(26, _mm_mul_ps(resw,J6));
    ACC(27, _mm_mul_ps(resw,res));
#undef ACC
    ls->num_constraints += 6;
}
static void lgs6_finish(LGS6* ls)
{   /* LGSX.h:205-325 */
    static const int ij[21][2] = {{0,0},{0,1},{0,2},{0,3},{0,4},{0,5},{1,1},{1,2},{1,3},{1,4},{1,5},
                                  {2,2},{2,3},{2,4},{2,5},{3,3},{3,4},{3,5},{4,4},{4,5},{5,5}};
    const float* S = ls->SSEData;
    for (int k = 0; k < 21; k++) {
        int i = ij[k][0], j = ij[k][1];
        float v = S[4*k+0] + S[4*k+1] + S[4*k+2] + S[4*k+3];
        /* note LGSX.h:215-281: the mirrored entry is overwritten with the (upper/lower) accumulated one */
        if (i == j) ls->A[i*6+i] += v;
        else if (i == 0) { ls->A[0*6+j] += v; ls->A[j*6+0] = ls->A[0*6+j]; }
        else { ls->A[j*6+i] += v; ls->A[i*6+j] = ls->A[j*6+i]; }
    }
    for (int k = 0; k < 6; k++) ls->b[k] -= S[4*(21+k)+0] + S[4*(21+k)+1] + S[4*(21+k)+2] + S[4*(21+k)+3];
    ls->error += S[4*27+0] + S[4*27+1] + S[4*27+2] + S[4*27+3];
    if (G.exactTrackingSums && !G.useSSE) {
        for (int i = 0; i < 36; i++) ls->A[i] = (float)ls->dA[i];
        for (int i = 0; i < 6; i++) ls->b[i] = (float)ls->db[i];
        ls->error = (float)ls->derror;
    }
    float n = (float)ls->num_constraints;
    for (int i = 0; i < 36; i++) ls->A[i] /= n;
    for (int i = 0; i < 6; i++) ls->b[i] /= n;
    ls->error /= n;
}

typedef struct {
    int width, height;
    float* buf_warped_residual; float* buf_warped_dx; float* buf_warped_dy;
    float* buf_warped_x; float* buf_warped_y; float* buf_warped_z;
    float* buf_d; float* buf_idepthVar; float* buf_weight_p;
    int buf_warped_size;
    float pointUsage, lastGoodCount, lastBadCount, lastMeanRes, lastResidual;
    float affineEstimation_a, affineEstimation_b, affineEstimation_a_lastIt, affineEstimation_b_lastIt;
    float sxx, syy, sx, sy, sw;
    int diverged, trackingWasGood;
    lsdo_track_settings settings;
} Tracker;

static float* amalloc(size_t n) { void* p = 0; if (posix_memalign(&p, 64, n*sizeof(float))) return 0; memset(p, 0, n*sizeof(float)); return (float*)p; }
static void tracker_init(Tracker* t, int w, int h, const lsdo_track_settings* s)
{   /* SE3Tracker.cpp:46-94 */
    memset(t, 0, sizeof(*t));
    t->width = w; t->height = h;
    size_t n = (size_t)w*h;
    t->buf_warped_residual = amalloc(n); t->buf_warped_dx = amalloc(n); t->buf_warped_dy = amalloc(n);
    t->buf_warped_x = amalloc(n); t->buf_warped_y = amalloc(n); t->buf_warped_z = amalloc(n);
    t->buf_d = amalloc(n); t->buf_idepthVar = amalloc(n); t->buf_weight_p = amalloc(n);
    t->settings = *s;
}
static void tracker_free(Tracker* t)
{
    free(t->buf_warped_residual); free(t->buf_warped_dx); free(t->buf_warped_dy);
    free(t->buf_warped_x); free(t->buf_warped_y); free(t->buf_warped_z);
    free(t->buf_d); free(t->buf_idepthVar); free(t->buf_weight_p);
}

/* SE3Tracker::calcResidualAndBuffers, SE3Tracker.cpp:885-1029 */
static float calcResidualAndBuffers(Tracker* t, const float* refPoint, const float* refColVar, const int* idxBuf, int refNum,
                                    lsdo_frame* frame, const float refToFrame[7], int level)
{
    int w = frame->width[level], h = frame->height[level];
    float fx_l = frame->K[level][0], fy_l = frame->K[level][4], cx_l = frame->K[level][2], cy_l = frame->K[level][5];
    float rotMat[9], transVec[3];
    lsdo_se3f_matrix(refToFrame, rotMat, transVec);
    const float* refPoint_max = refPoint + 3*refNum;
    const float* frame_gradients = lsdo_frame_gradients(frame, level);
    int idx = 0;
    float sumResUnweighted = 0;
    uint8_t* isGoodOutBuffer = idxBuf != 0 ? lsdo_frame_refPixelWasGood(frame) : 0;
    int goodCount = 0, badCount = 0;
    float sumSignedRes = 0;
    float sxx = 0, syy = 0, sx = 0, sy = 0, sw = 0;
    float usageCount = 0;
    double dxx = 0, dyy = 0, dx = 0, dy = 0, dw = 0, dUsage = 0, dResU = 0, dSigned = 0;   /* exactTrackingSums twin */
    for (; refPoint < refPoint_max; refPoint += 3, refColVar += 2, idxBuf++) {
        float Wxp[3];
        for (int i = 0; i < 3; i++)
            Wxp[i] = ((rotMat[i*3+0]*refPoint[0] + rotMat[i*3+1]*refPoint[1]) + rotMat[i*3+2]*refPoint[2]) + transVec[i];
        float u_new = (Wxp[0]/Wxp[2])*fx_l + cx_l;
        float v_new = (Wxp[1]/Wxp[2])*fy_l + cy_l;
        if (!(u_new > 1 && v_new > 1 && u_new < w-2 && v_new < h-2)) {
            if (isGoodOutBuffer != 0) isGoodOutBuffer[*idxBuf] = 0;
            continue;
        }
        float resInterp[3];
        getInterpolatedElement4n(frame_gradients, u_new, v_new, w, 3, resInterp);
        float c1 = t->affineEstimation_a * refColVar[0] + t->affineEstimation_b;
        float c2 = resInterp[2];
        float residual = c1 - c2;
        float weight = fabsf(residual) < 5.0f ? 1 : 5.0f / fabsf(residual);
        sxx += c1*c1*weight; syy += c2*c2*weight; sx += c1*weight; sy += c2*weight; sw += weight;
        dxx += (double)(c1*c1*weight); dyy += (double)(c2*c2*weight); dx += (double)(c1*weight); dy += (double)(c2*weight); dw += (double)weight;
        int isGood = residual*residual / (MAX_DIFF_CONSTANT + MAX_DIFF_GRAD_MULT*(resInterp[0]*resInterp[0] + resInterp[1]*resInterp[1])) < 1;
        if (isGoodOutBuffer != 0) isGoodOutBuffer[*idxBuf] = isGood;
        t->buf_warped_x[idx] = Wxp[0]; t->buf_warped_y[idx] = Wxp[1]; t->buf_warped_z[idx] = Wxp[2];
        t->buf_warped_dx[idx] = fx_l * resInterp[0];
        t->buf_warped_dy[idx] = fy_l * resInterp[1];
        t->buf_warped_residual[idx] = residual;
        t->buf_d[idx] = 1.0f / refPoint[2];
        t->buf_idepthVar[idx] = refColVar[1];
        idx++;
        if (isGood) { sumResUnweighted += residual*residual; sumSignedRes += residual; goodCount++; dResU += (double)(residual*residual); dSigned += (double)residual; }
        else badCount++;
        float depthChange = refPoint[2] / Wxp[2];
        usageCount += depthChange < 1 ? depthChange : 1;
        dUsage += (double)(depthChange < 1 ? depthChange : 1);
    }
    if (G.exactTrackingSums) {
        sxx = (float)dxx; syy = (float)dyy; sx = (float)dx; sy = (float)dy; sw = (float)dw;
        usageCount = (float)dUsage; sumResUnweighted = (float)dResU; sumSignedRes = (float)dSigned;
    }
    t->buf_warped_size = idx;
    t->pointUsage = usageCount / (float)refNum;
    t->lastGoodCount = goodCount;
    t->lastBadCount = badCount;
    t->lastMeanRes = sumSignedRes / goodCount;
    t->affineEstimation_a_lastIt = sqrtf((syy - sy*sy/sw) / (sxx - sx*sx/sw));
    t->affineEstimation_b_lastIt = (sy - t->affineEstimation_a_lastIt*sx)/sw;
    t->sxx = sxx; t->syy = syy; t->sx = sx; t->sy = sy; t->sw = sw;
    return sumResUnweighted / goodCount;
}

/* SE3Tracker::calcWeightsAndResidual (scalar), SE3Tracker.cpp:749-790 */
static float calcWeightsAndResidual(Tracker* t, const float refToFrame[7])
{
    float tx = refToFrame[4], ty = refToFrame[5], tz = refToFrame[6];
    float sumRes = 0;
    double dSumRes = 0;               /* exactTrackingSums twin */
    for (int i = 0; i < t->buf_warped_size; i++) {
        float px = t->buf_warped_x[i], py = t->buf_warped_y[i], pz = t->buf_warped_z[i];
        float d = t->buf_d[i];
        float rp = t->buf_warped_residual[i];
        float gx = t->buf_warped_dx[i], gy = t->buf_warped_dy[i];
        float s = t->settings.var_weight * t->buf_idepthVar[i];
        float g0 = (tx * pz - tz * px) / (pz*pz*d);
        float g1 = (ty * pz - tz * py) / (pz*pz*d);
        float drpdd = gx * g0 + gy * g1;
        float w_p = 1.0f / ((G.cameraPixelNoise2) + s * drpdd * drpdd);
        float weighted_rp = fabsf(rp*sqrtf(w_p));
        float wh = fabsf(weighted_rp < (t->settings.huber_d/2) ? 1 : (t->settings.huber_d/2) / weighted_rp);
        sumRes += wh * w_p * rp*rp;
        dSumRes += (double)(wh * w_p * rp*rp);
        t->buf_weight_p[i] = wh * w_p;
    }
    if (G.exactTrackingSums) sumRes = (float)dSumRes;
    return sumRes / t->buf_warped_size;
}

/* SE3Tracker::calcWeightsAndResidualSSE, SE3Tracker.cpp:492-575 (timing flavour; uses rcp_ps) */
static float calcWeightsAndResidualSSE(Tracker* t, const float refToFrame[7])
{
    const __m128 txs = _mm_set1_ps(refToFrame[4]), tys = _mm_set1_ps(refToFrame[5]), tzs = _mm_set1_ps(refToFrame[6]);
    const __m128 zeros = _mm_set1_ps(0.0f), ones = _mm_set1_ps(1.0f);
    const __m128 depthVarFacs = _mm_set1_ps(t->settings.var_weight);
    const __m128 sigma_i2s = _mm_set1_ps(G.cameraPixelNoise2);
    const __m128 huber_res_ponlys = _mm_set1_ps(t->settings.huber_d/2);
    __m128 sumResP = zeros;
    for (int i = 0; i < t->buf_warped_size-3; i += 4) {
        __m128 pzs = _mm_load_ps(t->buf_warped_z+i);
        __m128 pz2ds = _mm_rcp_ps(_mm_mul_ps(_mm_mul_ps(pzs, pzs), _mm_load_ps(t->buf_d+i)));
        __m128 g0s = _mm_sub_ps(_mm_mul_ps(pzs, txs), _mm_mul_ps(_mm_load_ps(t->buf_warped_x+i), tzs));
        g0s = _mm_mul_ps(g0s, pz2ds);
        __m128 g1s = _mm_sub_ps(_mm_mul_ps(pzs, tys), _mm_mul_ps(_mm_load_ps(t->buf_warped_y+i), tzs));
        g1s = _mm_mul_ps(g1s, pz2ds);
        __m128 drpdds = _mm_add_ps(_mm_mul_ps(g0s, _mm_load_ps(t->buf_warped_dx+i)), _mm_mul_ps(g1s, _mm_load_ps(t->buf_warped_dy+i)));
        __m128 w_ps = _mm_rcp_ps(_mm_add_ps(sigma_i2s, _mm_mul_ps(drpdds, _mm_mul_ps(drpdds, _mm_mul_ps(depthVarFacs, _mm_load_ps(t->buf_idepthVar+i))))));
        __m128 weighted_rps = _mm_mul_ps(_mm_load_ps(t->buf_warped_residual+i), _mm_sqrt_ps(w_ps));
        weighted_rps = _mm_max_ps(weighted_rps, _mm_sub_ps(zeros, weighted_rps));
        __m128 whs = _mm_cmplt_ps(weighted_rps, huber_res_ponlys);
        whs = _mm_or_ps(_mm_and_ps(whs, ones), _mm_andnot_ps(whs, _mm_mul_ps(huber_res_ponlys, _mm_rcp_ps(weighted_rps))));
        if (i+3 < t->buf_warped_size)
            sumResP = _mm_add_ps(sumResP, _mm_mul_ps(whs, _mm_mul_ps(weighted_rps, weighted_rps)));
        _mm_store_ps(t->buf_weight_p+i, _mm_mul_ps(whs, w_ps));
    }
    float sr[4] __attribute__((aligned(16))); _mm_store_ps(sr, sumResP);
    float sumRes = sr[0] + sr[1] + sr[2] + sr[3];
    return sumRes / ((t->buf_warped_size >> 2)<<2);
}

/* SE3Tracker::calculateWarpUpdate (scalar), SE3Tracker.cpp:1258-1299 */
static void calculateWarpUpdate(Tracker* t, LGS6* ls)
{
    lgs6_initialize(ls);
    for (int i = 0; i < t->buf_warped_size; i++) {
        float px = t->buf_warped_x[i], py = t->buf_warped_y[i], pz = t->buf_warped_z[i];
        float r = t->buf_warped_residual[i];
        float gx = t->buf_warped_dx[i], gy = t->buf_warped_dy[i];
        float z = 1.0f / pz;
        float z_sqr = 1.0f / (pz*pz);
        float v[6];
        v[0] = z*gx + 0;
        v[1] = 0 + z*gy;
        v[2] = (-px * z_sqr) * gx + (-py * z_sqr) * gy;
        /* the literals 1.0 are double in the reference: these two rows are evaluated in double */
        v[3] = (float)((-px * py * z_sqr) * gx + (-(1.0 + py * py * z_sqr)) * gy);
        v[4] = (float)((1.0 + px * px * z_sqr) * gx + (px * py * z_sqr) * gy);
        v[5] = (-py * z) * gx + (px * z) * gy;
        lgs6_update(ls, v, r, t->buf_weight_p[i]);
    }
    lgs6_finish(ls);
}

/* SE3Tracker::calculateWarpUpdateSSE, SE3Tracker.cpp:1033-1130 (timing flavour) */
static void calculateWarpUpdateSSE(Tracker* t, LGS6* ls)
{
    lgs6_initialize(ls);
    for (int i = 0; i < t->buf_warped_size-3; i += 4) {
        __m128 val1, val2, val3, val4, J61, J62, J63, J64, J65, J66;
        __m128 pz = _mm_rcp_ps(_mm_load_ps(t->buf_warped_z+i));
        __m128 gx = _mm_load_ps(t->buf_warped_dx+i);
        J61 = _mm_mul_ps(pz, gx);
        __m128 gy = _mm_load_ps(t->buf_warped_dy+i);
        J62 = _mm_mul_ps(pz, gy);
        __m128 px = _mm_load_ps(t->buf_warped_x+i);
        val1 = _mm_mul_ps(_mm_mul_ps(px, gy), pz);
        __m128 py = _mm_load_ps(t->buf_warped_y+i);
        val2 = _mm_mul_ps(_mm_mul_ps(py, gx), pz);
        J66 = _mm_sub_ps(val1, val2);
        pz = _mm_mul_ps(pz, pz);
        val1 = _mm_mul_ps(_mm_mul_ps(px, gx), pz);
        val2 = _mm_mul_ps(_mm_mul_ps(py, gy), pz);
        val3 = _mm_add_ps(val1, val2);
        J63 = _mm_sub_ps(_mm_setr_ps(0,0,0,0), val3);
        val3 = _mm_mul_ps(val1, py);
        val4 = _mm_add_ps(gy, val3);
        val3 = _mm_mul_ps(val2, py);
        val4 = _mm_add_ps(val3, val4);
        J64 = _mm_sub_ps(_mm_setr_ps(0,0,0,0), val4);
        val3 = _mm_mul_ps(val1, px);
        val4 = _mm_add_ps(gx, val3);
        val3 = _mm_mul_ps(val2, px);
        J65 = _mm_add_ps(val4, val3);
        /* i+3 < size always holds inside this loop (SE3Tracker.cpp:1110-1122: the tail branch is dead) */
        lgs6_updateSSE(ls, J61, J62, J63, J64, J65, J66, _mm_load_ps(t->buf_warped_residual+i), _mm_load_ps(t->buf_weight_p+i));
    }
    lgs6_finish(ls);
}

typedef struct { float* pos; float* colvar; int* idx; int n; } PointCloud;
static void pc_make(PointCloud* pc, lsdo_frame* kf, int level)
{
    size_t n = (size_t)kf->width[level]*kf->height[level];
    pc->pos = (float*)malloc(n*3*sizeof(float)); pc->colvar = (float*)malloc(n*2*sizeof(float)); pc->idx = (int*)malloc(n*sizeof(int));
    pc->n = lsdo_make_point_cloud(kf, level, pc->pos, 0, pc->colvar, pc->idx);
}
static void pc_free(PointCloud* pc) { free(pc->pos); free(pc->colvar); free(pc->idx); }

/* one fused evaluation at a given pose (the GPU kernel's per-call parity hook) */
int lsdo_se3_eval(lsdo_frame* kf, lsdo_frame* frame, int level, const float refToFrame_qt[7],
                  float affine_a, float affine_b, const lsdo_track_settings* s, int writeGoodMask, lsdo_eval_result* out)
{
    Tracker t; tracker_init(&t, kf->width[0], kf->height[0], s);
    PointCloud pc; pc_make(&pc, kf, level);
    t.affineEstimation_a = affine_a; t.affineEstimation_b = affine_b;
    out->meanUnweightedRes = calcResidualAndBuffers(&t, pc.pos, pc.colvar, writeGoodMask ? pc.idx : 0, pc.n, frame, refToFrame_qt, level);
    out->meanWeightedRes = G.useSSE ? calcWeightsAndResidualSSE(&t, refToFrame_qt) : calcWeightsAndResidual(&t, refToFrame_qt);
    LGS6 ls;
    if (G.useSSE) calculateWarpUpdateSSE(&t, &ls); else calculateWarpUpdate(&t, &ls);
    memcpy(out->A, ls.A, sizeof(ls.A)); memcpy(out->b, ls.b, sizeof(ls.b));
    out->lsError = ls.error;
    out->warpedSize = t.buf_warped_size;
    out->pointUsage = t.pointUsage; out->goodCount = t.lastGoodCount; out->badCount = t.lastBadCount; out->meanRes = t.lastMeanRes;
    out->affine_a_lastIt = t.affineEstimation_a_lastIt; out->affine_b_lastIt = t.affineEstimation_b_lastIt;
    out->sxx = t.sxx; out->syy = t.syy; out->sx = t.sx; out->sy = t.sy; out->sw = t.sw;
    pc_free(&pc); tracker_free(&t);
    return 0;
}

/* SE3Tracker::trackFrame, SE3Tracker.cpp:280-486 */
int lsdo_se3_track(lsdo_frame* kf, lsdo_frame* frame, const double frameToRef_init_qt[7],
                   const lsdo_track_settings* s, lsdo_track_result* out)
{
    Tracker T; Tracker* t = &T; tracker_init(t, kf->width[0], kf->height[0], s);
    memset(out, 0, sizeof(*out));
    t->diverged = 0; t->trackingWasGood = 1;
    t->affineEstimation_a = 1; t->affineEstimation_b = 0;

    double initInv[7]; lsdo_se3d_inverse(frameToRef_init_qt, initInv);
    float referenceToFrame[7]; se3_d2f(initInv, referenceToFrame);
    LGS6 ls;
    float last_residual = 0;
    int ret_diverged = 0;

    for (int lvl = SE3TRACKING_MAX_LEVEL-1; lvl >= SE3TRACKING_MIN_LEVEL; lvl--) {
        PointCloud pc; pc_make(&pc, kf, lvl);    /* reference->makePointCloud(lvl), :321 */
        const int* idxb = (SE3TRACKING_MIN_LEVEL == lvl) ? pc.idx : 0;
        calcResidualAndBuffers(t, pc.pos, pc.colvar, idxb, pc.n, frame, referenceToFrame, lvl);
        if (t->buf_warped_size < MIN_GOODPERALL_PIXEL_ABSMIN * (t->width>>lvl)*(t->height>>lvl)) {
            t->diverged = 1; t->trackingWasGood = 0; ret_diverged = 1; pc_free(&pc); break;
        }
        if (G.useAffineLightningEstimation) {
            t->affineEstimation_a = t->affineEstimation_a_lastIt;
            t->affineEstimation_b = t->affineEstimation_b_lastIt;
        }
        float lastErr = G.useSSE ? calcWeightsAndResidualSSE(t, referenceToFrame) : calcWeightsAndResidual(t, referenceToFrame);
        out->numCalcResidualCalls[lvl]++;
        float LM_lambda = t->settings.lambdaInitial[lvl];

        for (int iteration = 0; iteration < t->settings.maxItsPerLvl[lvl]; iteration++) {
            if (G.useSSE) calculateWarpUpdateSSE(t, &ls); else calculateWarpUpdate(t, &ls);
            out->numCalcWarpUpdateCalls[lvl]++;
            int incTry = 0;
            while (1) {
                float b[6], A[36], inc[6];
                for (int i = 0; i < 6; i++) b[i] = -ls.b[i];
                memcpy(A, ls.A, sizeof(A));
                for (int i = 0; i < 6; i++) A[i*6+i] *= 1+LM_lambda;
                lsdo_ldlt6_solve(A, b, inc);
                incTry++;
                float expInc[7], new_referenceToFrame[7];
                lsdo_se3f_exp(inc, expInc);
                lsdo_se3f_mul(expInc, referenceToFrame, new_referenceToFrame);
                calcResidualAndBuffers(t, pc.pos, pc.colvar, idxb, pc.n, frame, new_referenceToFrame, lvl);
                if (t->buf_warped_size < MIN_GOODPERALL_PIXEL_ABSMIN * (t->width>>lvl)*(t->height>>lvl)) {
                    t->diverged = 1; t->trackingWasGood = 0; ret_diverged = 1; break;
                }
                float error = G.useSSE ? calcWeightsAndResidualSSE(t, new_referenceToFrame) : calcWeightsAndResidual(t, new_referenceToFrame);
                out->numCalcResidualCalls[lvl]++;
                if (error < lastErr) {
                    memcpy(referenceToFrame, new_referenceToFrame, sizeof(referenceToFrame));
                    if (G.useAffineLightningEstimation) {
                        t->affineEstimation_a = t->affineEstimation_a_lastIt;
                        t->affineEstimation_b = t->affineEstimation_b_lastIt;
                    }
                    if (error / lastErr > t->settings.convergenceEps[lvl])
                        iteration = t->settings.maxItsPerLvl[lvl];
                    last_residual = lastErr = error;
                    if (LM_lambda <= 0.2) LM_lambda = 0;
                    else LM_lambda *= t->settings.lambdaSuccessFac;
                    break;
                } else {
                    float dot = 0; for (int i = 0; i < 6; i++) dot += inc[i]*inc[i];
                    if (!(dot > t->settings.stepSizeMin[lvl])) {
                        iteration = t->settings.maxItsPerLvl[lvl];
                        break;
                    }
                    if (LM_lambda == 0) LM_lambda = 0.2;
                    else LM_lambda *= pow(t->settings.lambdaFailFac, incTry);
                }
            }
            if (ret_diverged) break;
        }
        pc_free(&pc);
        if (ret_diverged) break;
    }

    if (ret_diverged) {
        /* return SE3(): identity (SE3Tracker.cpp:324-329, 369-374) */
        out->frameToRef_qt[3] = 1;
        out->diverged = 1; out->trackingWasGood = 0;
        out->pointUsage = t->pointUsage; out->lastGoodCount = t->lastGoodCount; out->lastBadCount = t->lastBadCount;
        out->lastMeanRes = t->lastMeanRes; out->lastResidual = t->lastResidual;
        out->affineEstimation_a = t->affineEstimation_a; out->affineEstimation_b = t->affineEstimation_b;
        tracker_free(t);
        return 0;
    }

    t->lastResidual = last_residual;
    t->trackingWasGood = !t->diverged
        && t->lastGoodCount / (frame->width[SE3TRACKING_MIN_LEVEL]*frame->height[SE3TRACKING_MIN_LEVEL]) > MIN_GOODPERALL_PIXEL
        && t->lastGoodCount / (t->lastGoodCount + t->lastBadCount) > MIN_GOODPERGOODBAD_PIXEL;
    if (t->trackingWasGood) kf->numFramesTrackedOnThis++;
    frame->initialTrackedResidual = t->lastResidual / t->pointUsage;
    float inv[7]; lsdo_se3f_inverse(referenceToFrame, inv);
    double invd[7]; se3_f2d(inv, invd);
    memcpy(frame->thisToParent_q, invd, 32); memcpy(frame->thisToParent_t, invd+4, 24); frame->thisToParent_s = 1;
    frame->trackingParent = kf;
    memcpy(out->frameToRef_qt, invd, sizeof(invd));
    out->pointUsage = t->pointUsage; out->lastGoodCount = t->lastGoodCount; out->lastBadCount = t->lastBadCount;
    out->lastMeanRes = t->lastMeanRes; out->lastResidual = t->lastResidual;
    out->affineEstimation_a = t->affineEstimation_a; out->affineEstimation_b = t->affineEstimation_b;
    out->diverged = t->diverged; out->trackingWasGood = t->trackingWasGood;
    out->initialTrackedResidual = frame->initialTrackedResidual;
    tracker_free(t);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * permaRef tracking (SURVEY 8f row 2): Frame::setPermaRef DataStructures/Frame.cpp:149-174,
 * SE3Tracker::checkPermaRefOverlap Tracking/SE3Tracker.cpp:121-157,
 * SE3Tracker::trackFrameOnPermaref Tracking/SE3Tracker.cpp:162-272  (QUICK_KF_CHECK_LVL = 4, util/settings.h:104)
 * ---------------------------------------------------------------------------------------- */
#define QUICK_KF_CHECK_LVL 4
int lsdo_frame_setPermaRef(lsdo_frame* kf, float* posData /*3/pt, >= w4*h4*/, float* colorAndVarData /*2/pt*/)
{
    return lsdo_make_point_cloud(kf, QUICK_KF_CHECK_LVL, posData, 0, colorAndVarData, 0);
}

float lsdo_checkPermaRefOverlap(int w0, int h0, const float K4[9], const float* permaPos, int numPts, const double refToFrame_qt[7])
{
    float q[7]; se3_d2f(refToFrame_qt, q);
    int w2 = (w0 >> QUICK_KF_CHECK_LVL)-1, h2 = (h0 >> QUICK_KF_CHECK_LVL)-1;
    float fx_l = K4[0], fy_l = K4[4], cx_l = K4[2], cy_l = K4[5];
    float rotMat[9], transVec[3];
    lsdo_se3f_matrix(q, rotMat, transVec);
    float usageCount = 0;
    for (int k = 0; k < numPts; k++) {
        const float* p = permaPos + 3*k;
        float Wxp[3];
        for (int i = 0; i < 3; i++) Wxp[i] = ((rotMat[i*3+0]*p[0] + rotMat[i*3+1]*p[1]) + rotMat[i*3+2]*p[2]) + transVec[i];
        float u_new = (Wxp[0]/Wxp[2])*fx_l + cx_l;
        float v_new = (Wxp[1]/Wxp[2])*fy_l + cy_l;
        if ((u_new > 0 && v_new > 0 && u_new < w2 && v_new < h2)) {
            float depthChange = p[2] / Wxp[2];
            if (!(depthChange < 1)) COUNT_S3(LSDO_PERMA_USAGE_CLAMP);
            usageCount += depthChange < 1 ? depthChange : 1;
        } else COUNT_S3(LSDO_PERMA_OUTSIDE);
    }
    return usageCount / (float)numPts;
}

/* returns referenceToFrame (NOT inverted, SE3Tracker.cpp:271) in out->frameToRef_qt */
int lsdo_trackFrameOnPermaref(int w0, int h0, const float* permaPos, const float* permaColVar, int numPts,
                              lsdo_frame* frame, const double refToFrame_qt[7], lsdo_track_result* out)
{
    lsdo_track_settings s; lsdo_default_track_settings(&s);
    Tracker T; Tracker* t = &T; tracker_init(t, w0, h0, &s);
    memset(out, 0, sizeof(*out));
    const float lambdaInitialTestTrack = 0, stepSizeMinTestTrack = 1e-3, convergenceEpsTestTrack = 0.98, maxItsTestTrack = 5;   /* settings.h:379-382 */
    float referenceToFrame[7]; se3_d2f(refToFrame_qt, referenceToFrame);
    t->affineEstimation_a = 1; t->affineEstimation_b = 0;
    LGS6 ls;
    t->diverged = 0; t->trackingWasGood = 1;
    const float divTh = MIN_GOODPERALL_PIXEL_ABSMIN * (w0>>QUICK_KF_CHECK_LVL)*(h0>>QUICK_KF_CHECK_LVL);
    int diverged = 0;
    calcResidualAndBuffers(t, permaPos, permaColVar, 0, numPts, frame, referenceToFrame, QUICK_KF_CHECK_LVL);
    float lastErr = 0;
    if (t->buf_warped_size < divTh) diverged = 1;
    else {
        if (G.useAffineLightningEstimation) { t->affineEstimation_a = t->affineEstimation_a_lastIt; t->affineEstimation_b = t->affineEstimation_b_lastIt; }
        lastErr = calcWeightsAndResidual(t, referenceToFrame);
        out->numCalcResidualCalls[QUICK_KF_CHECK_LVL]++;
        float LM_lambda = lambdaInitialTestTrack;
        for (int iteration = 0; iteration < maxItsTestTrack && !diverged; iteration++) {
            calculateWarpUpdate(t, &ls);
            out->numCalcWarpUpdateCalls[QUICK_KF_CHECK_LVL]++;
            int incTry = 0;
            while (1) {
                float b[6], A[36], inc[6];
                for (int i = 0; i < 6; i++) b[i] = -ls.b[i];
                memcpy(A, ls.A, sizeof(A));
                for (int i = 0; i < 6; i++) A[i*6+i] *= 1+LM_lambda;
                lsdo_ldlt6_solve(A, b, inc);
                incTry++;
                float expInc[7], newT[7];
                lsdo_se3f_exp(inc, expInc);
                lsdo_se3f_mul(expInc, referenceToFrame, newT);
                calcResidualAndBuffers(t, permaPos, permaColVar, 0, numPts, frame, newT, QUICK_KF_CHECK_LVL);
                if (t->buf_warped_size < divTh) { diverged = 1; break; }
                float error = calcWeightsAndResidual(t, newT);
                out->numCalcResidualCalls[QUICK_KF_CHECK_LVL]++;
                if (error < lastErr) {
                    memcpy(referenceToFrame, newT, sizeof(newT));
                    if (G.useAffineLightningEstimation) { t->affineEstimation_a = t->affineEstimation_a_lastIt; t->affineEstimation_b = t->affineEstimation_b_lastIt; }
                    if (error / lastErr > convergenceEpsTestTrack) iteration = maxItsTestTrack;
                    lastErr = error;
                    if (LM_lambda <= 0.2) LM_lambda = 0; else LM_lambda *= s.lambdaSuccessFac;
                    break;
                } else {
                    float dot = 0; for (int i = 0; i < 6; i++) dot += inc[i]*inc[i];
                    if (!(dot > stepSizeMinTestTrack)) { iteration = maxItsTestTrack; break; }
                    if (LM_lambda == 0) LM_lambda = 0.2; else LM_lambda *= pow(s.lambdaFailFac, incTry);
                }
            }
        }
    }
    out->pointUsage = t->pointUsage; out->lastGoodCount = t->lastGoodCount; out->lastBadCount = t->lastBadCount; out->lastMeanRes = t->lastMeanRes;
    out->affineEstimation_a = t->affineEstimation_a; out->affineEstimation_b = t->affineEstimation_b;
    if (diverged) { out->frameToRef_qt[3] = 1; out->diverged = 1; out->trackingWasGood = 0; tracker_free(t); return 0; }
    out->lastResidual = lastErr;
    out->trackingWasGood = t->lastGoodCount / (frame->width[QUICK_KF_CHECK_LVL]*frame->height[QUICK_KF_CHECK_LVL]) > MIN_GOODPERALL_PIXEL
        && t->lastGoodCount / (t->lastGoodCount + t->lastBadCount) > MIN_GOODPERGOODBAD_PIXEL;
    double d[7]; se3_f2d(referenceToFrame, d);
    memcpy(out->frameToRef_qt, d, sizeof(d));
    tracker_free(t);
    return 0;
}

#include "lsd_oracle_sim3.inc"
#include "lsd_oracle_undistort.inc"
#include "lsd_oracle_depth.inc"
