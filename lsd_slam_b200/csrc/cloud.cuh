// cloud.cuh -- the resident map as one filtered world-frame point cloud, many keyframes per launch (lsdgpu_map_export_pointcloud).
//
// Replaces (paths relative to lsd_slam_viewer/):
//   KeyFrameDisplay::setFrom     src/KeyFrameDisplay.cpp:65-104    fxi = 1/fx, cxi = -cx/fx from the message's float fx, cx
//   KeyFrameDisplay::refreshPC   src/KeyFrameDisplay.cpp:106-222   filter + camera-frame vertex buffer, totalPoints / displayedPoints
//   KeyFrameDisplay::flushPC     src/KeyFrameDisplay.cpp:269-339   the same filter with refreshPC's my_* values + Sim3f * point
//   Sophus::Sim3f * p            thirdparty/Sophus/sophus/sim3.hpp:247-249, rxso3.hpp:263-269 (scale * (q/scale)._transformVector(p))
//
// One CTA takes a run of full rows of one keyframe (tiles are numbered in (keyframe, y) order), stages the idepth rows y-1 .. y+rows
// it needs for the 3x3 support test in shared memory, evaluates the filter, and compacts the kept points into the batch's output in
// global (keyframe, y, x) order.  The CTA's offset comes from a single-pass decoupled look-back over the tiles before it: the input
// (12 B per pixel) is read once, where a count pass + scan + emit pass would read idepth and idepthVar twice (20 B per pixel).
// Tiles are taken in ticket order (an atomic counter), so a CTA only waits for tiles already taken by running CTAs.  The offsets are
// integer sums, so the output is independent of scheduling and identical run to run.
#pragma once
#include "internal.cuh"

#define CLOUD_THREADS 256
#define CLOUD_TILE_PX 2048              // interior pixels per CTA (about): rows = max(1, CLOUD_TILE_PX / w)
#define CLOUD_MAX_ITERS 32              // kept flags of one thread live in one 32-bit word: rows * (w-2) <= 32 * CLOUD_THREADS

// Sophus::Sim3f constants of one keyframe, formed once on the host from the 7 floats of keyframeMsg.camToWorld, plus the level's
// camera constants of KeyFrameDisplay::setFrom
struct CloudKf {
    const float* idepth;
    const float* idepthVar;
    const float* image;
    float nq[4];                        // norm_quad = q / scale (rxso3.hpp:265-267)
    float scale;                        // q.norm() = camToWorld.scale() = my_scale (KeyFrameDisplay.cpp:143)
    float t[3];
    float fxi, fyi, cxi, cyi;
};

struct CloudParams {
    const CloudKf* kfs;
    int w, h, rows, tilesPerKf;
    float scaledTH, absTH;
    int minNearSupport;
    int layout, emit;
    const float* intensity;             // (float)(c / 255.0) for c = 0..255 (KeyFrameDisplay.cpp:331)
    unsigned long long* tileState;      // per tile: flag (bits 62-63: 1 = aggregate, 2 = inclusive prefix) | value
    unsigned int* ticket;
    int* counts;                        // 2 per keyframe of the batch: totalPoints, displayedPoints
    float4* out;
};

#define CLOUD_FLAG_AGG 1ull
#define CLOUD_FLAG_INC 2ull
#define CLOUD_VALUE_MASK ((1ull << 62) - 1)

// KeyFrameDisplay.cpp:153-186 (refreshPC) = :277-307 (flushPC) for one pixel whose idepth is not <= 0; c = the idepth plane at
// the pixel (staged rows, row stride w).  Operand order as the viewer's (compiled with --fmad=false, so nothing is contracted).
__device__ __forceinline__ bool cloudKeep(const float* c, int w, float idepth, float var, float scale, const CloudParams& P)
{
    const float depth = 1 / idepth;
    float depth4 = depth * depth;
    depth4 *= depth4;
    if (var * depth4 > P.scaledTH) return false;
    if (var * depth4 * scale * scale > P.absTH) return false;
    if (P.minNearSupport > 1) {
        int nearSupport = 0;
        for (int dx = -1; dx < 2; dx++)
            for (int dy = -1; dy < 2; dy++) {
                const float n = c[dx + dy * w];
                if (n > 0) {
                    const float diff = n - 1.0f / depth;
                    if (diff * diff < 2 * var) nearSupport++;
                }
            }
        if (nearSupport < P.minNearSupport) return false;
    }
    return true;
}

__device__ __forceinline__ unsigned long long cloudLoadState(const unsigned long long* p)
{
    return *(const volatile unsigned long long*)p;
}

__global__ void __launch_bounds__(CLOUD_THREADS) k_cloud_export(const __grid_constant__ CloudParams P)
{
    extern __shared__ float sId[];                      // (rows + 2) * w idepth values
    __shared__ unsigned int sTile;
    __shared__ int sWarp[CLOUD_MAX_ITERS][CLOUD_THREADS / 32];   // kept per (iteration, warp), then their exclusive prefix
    __shared__ unsigned long long sBase;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) sTile = atomicAdd(P.ticket, 1u);
    __syncthreads();
    const unsigned int tile = sTile;
    const int kf = tile / P.tilesPerKf, ty = tile - kf * P.tilesPerKf;
    const int w = P.w, iw = w - 2;
    const int y0 = 1 + ty * P.rows, ny = min(P.rows, P.h - 1 - y0);
    const CloudKf& K = P.kfs[kf];
    const float* idepth = K.idepth;
    const float* gsrc = idepth + (size_t)(y0 - 1) * w;
    for (int i = tid; i < (ny + 2) * w; i += CLOUD_THREADS) sId[i] = __ldg(gsrc + i);
    __syncthreads();

    const int npx = ny * iw, nIt = (npx + CLOUD_THREADS - 1) / CLOUD_THREADS;
    const float scale = K.scale;
    uint32_t keptBits = 0;
    int total = 0;
    for (int it = 0; it < nIt; it++) {
        const int p = it * CLOUD_THREADS + tid;
        bool valid = false, keep = false;
        if (p < npx) {
            const int ry = p / iw, x = 1 + p - ry * iw;
            const float* c = sId + (ry + 1) * w + x;
            const float id = c[0];
            if (!(id <= 0)) {                           // KeyFrameDisplay.cpp:153: NaN passes
                valid = true;
                keep = cloudKeep(c, w, id, __ldg(K.idepthVar + (size_t)(y0 + ry) * w + x), scale, P);
            }
        }
        total += __syncthreads_count(valid);
        const unsigned int b = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) sWarp[it][warp] = __popc(b);
        keptBits |= (uint32_t)keep << it;
    }
    __syncthreads();
    if (tid == 0) {
        int acc = 0;
        for (int it = 0; it < nIt; it++)
            for (int k = 0; k < CLOUD_THREADS / 32; k++) { const int v = sWarp[it][k]; sWarp[it][k] = acc; acc += v; }
        const unsigned long long agg = (unsigned long long)acc;
        unsigned long long* st = P.tileState;
        unsigned long long excl = 0;
        if (tile == 0) {
            *(volatile unsigned long long*)&st[0] = (CLOUD_FLAG_INC << 62) | agg;
        } else {
            *(volatile unsigned long long*)&st[tile] = (CLOUD_FLAG_AGG << 62) | agg;
            for (int j = (int)tile - 1; j >= 0;) {
                const unsigned long long v = cloudLoadState(st + j);
                const unsigned long long flag = v >> 62;
                if (flag == 0) continue;                // tile j is taken by a running CTA: its aggregate follows
                excl += v & CLOUD_VALUE_MASK;
                if (flag == CLOUD_FLAG_INC) break;
                j--;
            }
            *(volatile unsigned long long*)&st[tile] = (CLOUD_FLAG_INC << 62) | (excl + agg);
        }
        sBase = excl;
        atomicAdd(P.counts + 2 * kf, total);
        atomicAdd(P.counts + 2 * kf + 1, acc);
    }
    if (!P.emit) return;
    __syncthreads();
    const unsigned long long base = sBase;
    const float fxi = K.fxi, fyi = K.fyi, cxi = K.cxi, cyi = K.cyi;
    for (int it = 0; it < nIt; it++) {
        const bool keep = (keptBits >> it) & 1u;
        const unsigned int b = __ballot_sync(0xffffffffu, keep);
        if (!keep) continue;
        const int p = it * CLOUD_THREADS + tid;
        const int ry = p / iw, x = 1 + p - ry * iw, y = y0 + ry;
        const size_t px = (size_t)y * w + x;
        const float depth = 1 / sId[(ry + 1) * w + x];
        // KeyFrameDisplay.cpp:188-190 / :310: ((x*fxi + cxi)*depth, (y*fyi + cyi)*depth, 1*depth)
        const float p0 = (x * fxi + cxi) * depth, p1 = (y * fyi + cyi) * depth, p2 = depth;
        const uint32_t col = (uint32_t)(unsigned char)__ldg(K.image + px);   // (uchar) of the level image, as k_pack_pointcloud
        float4 o;
        if (P.layout == LSDGPU_CLOUD_VERTEX) {
            // MyVertex: color[2] = in.color[0], color[1] = in.color[1], color[0] = in.color[2], color[3] = 100 (:192-195)
            o = make_float4(p0, p1, p2, __uint_as_float(col | (col << 8) | (col << 16) | (100u << 24)));
        } else {
            // Sim3f * p = scale * norm_quad._transformVector(p) + t; Eigen 3.2 generic _transformVector:
            // uv = q.vec x p; uv += uv; p + w*uv + q.vec x uv
            const float qx = K.nq[0], qy = K.nq[1], qz = K.nq[2], qw = K.nq[3];
            float u0 = qy * p2 - qz * p1, u1 = qz * p0 - qx * p2, u2 = qx * p1 - qy * p0;
            u0 += u0; u1 += u1; u2 += u2;
            const float c0 = qy * u2 - qz * u1, c1 = qz * u0 - qx * u2, c2 = qx * u1 - qy * u0;
            const float r0 = p0 + qw * u0 + c0, r1 = p1 + qw * u1 + c1, r2 = p2 + qw * u2 + c2;
            o = make_float4(scale * r0 + K.t[0], scale * r1 + K.t[1], scale * r2 + K.t[2], __ldg(P.intensity + col));
        }
        const unsigned long long idx = base + (unsigned long long)sWarp[it][warp] + __popc(b & ((1u << lane) - 1u));
        P.out[idx] = o;
    }
}
