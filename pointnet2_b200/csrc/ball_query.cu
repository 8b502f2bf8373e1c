// ball_query.cu — query_ball_point for sm_90a.
//
// Replaces query_ball_point_gpu / queryBallPointLauncher
// (reference tf_ops/grouping/tf_grouping_g.cu:3-36, :125-128).
//
// Semantics (bit-exact): for each query j, the first `nsample` data indices k in ASCENDING order
// with max(sqrtf(d2),1e-20f) < radius, d2 in the reference's contraction pattern
// (pn2::d2_fma_pattern, operands query - point); the row is padded with the first hit; pts_cnt is
// the number of real hits.  Rows with no hit are undefined in the reference; here they are zeros.
//
// The sqrtf is removed exactly: correctly-rounded sqrtf is monotone, so the hit test equals
// !(d2 > thr) for the float threshold thr = max{t : sqrtf(t) < radius}, found once on the host by
// bisection over float bit patterns (pn2_ball_threshold).  The negated form keeps the reference's
// NaN behaviour (fmaxf(NaN,1e-20f) = 1e-20f < radius is a hit).
//
// Design: a group of G lanes (G = 1..32, chosen from the amount of parallelism B*M offers) owns one
// query and tests G consecutive data points per step; data points are staged through shared memory
// in float4-padded tiles (one LDS.128 per test, broadcast across the groups of a warp); hits are
// rare, so the ordered compaction (ballot + popc prefix within the group) sits behind one
// warp-uniform branch; a CTA stops scanning as soon as all of its queries are full.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kBqThreads = 256;
constexpr int kBqTile = 2048;             // data points per shared-memory tile
constexpr int kBqPairs = kBqTile / 2;     // stored as pairs: (x0,x1,y0,y1) + (z0,z1)
constexpr int kBqUnroll = 2;              // pairs per lane per step (4 points)

template <int G>
__global__ void __launch_bounds__(kBqThreads)
ball_query_kernel(int n, int m, float thr, int nsample, const float* __restrict__ xyz1,
                  const float* __restrict__ xyz2, int* __restrict__ idx, int* __restrict__ pts_cnt,
                  const int* __restrict__ grid_params, int grid_stride, const int* __restrict__ lengths) {
    // clouds the uniform-grid path serves (flag written by bq_grid_build_kernel) are skipped here
    if (grid_params && grid_params[(size_t)blockIdx.y * grid_stride] != 0 &&
        batch_uses_grid(grid_params, (size_t)grid_stride, (int)gridDim.y))
        return;
    constexpr int QPB = kBqThreads / G;      // queries per CTA
    constexpr int STEP = G * kBqUnroll;      // pairs consumed per unrolled step by one group
    // pair layout: s_xy[i] = (x0, x1, y0, y1) of points 2i, 2i+1; s_z[i] = (z0, z1)
    __shared__ ulonglong2 s_xy[kBqPairs + 32 * kBqUnroll];
    __shared__ unsigned long long s_z[kBqPairs + 32 * kBqUnroll];

    const int tid = threadIdx.x, lane = tid & 31;
    const int g = tid % G;                     // lane within the group
    const int gbase = lane - g;                // first lane of this group within the warp
    const unsigned gmask_all = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << gbase);
    const unsigned lt_mask = (1u << lane) - 1u;
    const int cloud = blockIdx.y;
    const int q = blockIdx.x * QPB + tid / G;
    const bool valid = q < m;

    const float* __restrict__ data = xyz1 + (size_t)cloud * n * 3;
    n = cloud_length(lengths, cloud, n);  // the row stride is used up: from here on n is this cloud's length
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (valid) {
        const float* qp = xyz2 + ((size_t)cloud * m + q) * 3;
        qx = qp[0];
        qy = qp[1];
        qz = qp[2];
    }
    const unsigned long long QX = f2_pack(qx, qx), QY = f2_pack(qy, qy), QZ = f2_pack(qz, qz);
    int* __restrict__ row = idx + ((size_t)cloud * m + (valid ? q : 0)) * nsample;

    int cnt = valid ? 0 : nsample;  // out-of-range groups count as already full

    for (int base = 0; base < n; base += kBqTile) {
        const int tn = min(kBqTile, n - base);
        const int tp = (tn + 1) >> 1;                              // pairs holding real points
        const int tp_pad = ((tp + STEP - 1) / STEP) * STEP;
        // (the __syncthreads_and at the bottom of the previous iteration guarantees the previous
        //  tile is fully consumed before it is overwritten)
        float* sxy = reinterpret_cast<float*>(s_xy);
        float* sz = reinterpret_cast<float*>(s_z);
        for (int p = tid; p < 2 * tp_pad; p += kBqThreads) {
            float x = 1e30f, y = 1e30f, z = 1e30f;  // padding: far away, never a hit
            if (p < tn) {
                const float* src = data + (size_t)(base + p) * 3;
                x = src[0];
                y = src[1];
                z = src[2];
            }
            const int pi = p >> 1, par = p & 1;
            sxy[4 * pi + par] = x;
            sxy[4 * pi + 2 + par] = y;
            sz[2 * pi + par] = z;
        }
        __syncthreads();

        bool warp_done = __all_sync(kFullMask, cnt >= nsample);
        for (int p = 0; p < tp_pad && !warp_done; p += STEP) {
            bool h[kBqUnroll][2];
            bool any = false;
#pragma unroll
            for (int u = 0; u < kBqUnroll; ++u) {
                const ulonglong2 xy = s_xy[p + u * G + g];
                const unsigned long long zz = s_z[p + u * G + g];
                const unsigned long long dx = f2_sub(QX, xy.x), dy = f2_sub(QY, xy.y), dz = f2_sub(QZ, zz);
                const unsigned long long d = f2_fma(dz, dz, f2_fma(dx, dx, f2_mul(dy, dy)));
                float d0, d1;
                f2_unpack(d, d0, d1);
                h[u][0] = !(d0 > thr);
                h[u][1] = !(d1 > thr);
                any |= h[u][0] | h[u][1];
            }
            if (__any_sync(kFullMask, any && (cnt < nsample))) {
#pragma unroll
                for (int u = 0; u < kBqUnroll; ++u) {
                    const int k0 = base + 2 * (p + u * G + g);
                    const bool a0 = h[u][0] && (k0 < n) && (cnt < nsample);
                    const bool a1 = h[u][1] && (k0 + 1 < n) && (cnt < nsample);
                    const unsigned b0 = __ballot_sync(kFullMask, a0), b1 = __ballot_sync(kFullMask, a1);
                    const unsigned g0 = b0 & gmask_all, g1 = b1 & gmask_all;
                    if (g0 | g1) {  // hits in this group: emit them in index order (lane, then parity)
                        const int r0 = cnt + __popc(g0 & lt_mask) + __popc(g1 & lt_mask);
                        if (a0 && r0 < nsample) row[r0] = k0;
                        const int r1 = r0 + (a0 ? 1 : 0);
                        if (a1 && r1 < nsample) row[r1] = k0 + 1;
                        cnt = min(cnt + __popc(g0) + __popc(g1), nsample);
                    }
                }
                warp_done = __all_sync(kFullMask, cnt >= nsample);
            }
        }
        if (__syncthreads_and(cnt >= nsample)) break;
    }

    if (valid) {
        // pad the tail of the row with the first hit (zeros if there was none); the first hit was
        // written by a lane of this warp: make it visible, then read it back through L2
        __syncwarp(gmask_all);
        const int first = (cnt > 0) ? __ldcg(row) : 0;
        for (int l = cnt + g; l < nsample; l += G) row[l] = first;
        if (g == 0) pts_cnt[(size_t)cloud * m + q] = cnt;
    }
}

template <int G>
static int launch_bq(int b, int n, int m, float thr, int nsample, const float* xyz1, const int* lengths, const float* xyz2,
                     int* idx, int* pts_cnt, const int* grid_params, int grid_stride, cudaStream_t st) {
    constexpr int QPB = kBqThreads / G;
    dim3 grid((m + QPB - 1) / QPB, b, 1);
    ball_query_kernel<G><<<grid, kBqThreads, 0, st>>>(n, m, thr, nsample, xyz1, xyz2, idx, pts_cnt, grid_params, grid_stride, lengths);
    return finish_launch();
}

// experiment override of the lanes per query (0: automatic): pn2_set_bq_group, or PN2_BQ_GROUP, applied at the first query
static std::atomic<int> g_bq_group{0};

static int pick_group(int b, int m) {
    static const bool env_applied = [] {  // thread-safe: runs once
        if (const char* e = getenv("PN2_BQ_GROUP")) g_bq_group.store(atoi(e), std::memory_order_relaxed);
        return true;
    }();
    (void)env_applied;
    const int forced = g_bq_group.load(std::memory_order_relaxed);
    if (forced > 0) return forced;
    // enough lanes to fill every SM's 2048 thread slots (more, smaller groups win until the machine
    // is full)
    const long long queries = (long long)b * m;
    int G = 1;
    while (G < 32 && queries * G < (long long)num_sms() * 2048) G *= 2;
    return G;
}

int launch_ball_query_brute(int b, int n, int m, float thr, int nsample, const float* xyz1, const int* lengths,
                            const float* xyz2, int* idx, int* pts_cnt, const int* grid_params, int grid_stride,
                            cudaStream_t st) {
    switch (pick_group(b, m)) {
        case 1: return launch_bq<1>(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, grid_params, grid_stride, st);
        case 2: return launch_bq<2>(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, grid_params, grid_stride, st);
        case 4: return launch_bq<4>(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, grid_params, grid_stride, st);
        case 8: return launch_bq<8>(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, grid_params, grid_stride, st);
        case 16: return launch_bq<16>(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, grid_params, grid_stride, st);
        default: return launch_bq<32>(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, grid_params, grid_stride, st);
    }
}

// pn2_query_ball_point on the clouds' first lengths[b] points (lengths == NULL: all n)
int query_ball_point_brute(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths,
                           const float* xyz2, int* idx, int* pts_cnt, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || nsample <= 0 || !(radius > 0.0f)) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz1 || !xyz2 || !idx || !pts_cnt) return (int)cudaErrorInvalidValue;
    if (b > 65535) return (int)cudaErrorInvalidValue;
    const float thr = pn2_ball_threshold(radius);
    if (thr < 0.0f) {  // radius <= 1e-20f: the reference's test can never pass
        cudaError_t e = cudaMemsetAsync(idx, 0, sizeof(int) * (size_t)b * m * nsample, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(pts_cnt, 0, sizeof(int) * (size_t)b * m, st);
        return (int)e;
    }
    return launch_ball_query_brute(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, nullptr, 0, st);
}

}  // namespace pn2

extern "C" {

float pn2_ball_threshold(float radius) {
    // Largest float t >= 0 with max(sqrtf(t), 1e-20f) < radius; -1 if there is none.
    if (!(radius > 1e-20f)) return -1.0f;
    uint32_t lo = 0u, hi = 0x7f7fffffu;  // +0 .. FLT_MAX: the predicate is monotone in the bit pattern
    float f;
    memcpy(&f, &hi, 4);
    if (sqrtf(f) < radius) return f;
    while (hi - lo > 1u) {  // invariant: pred(lo) holds, pred(hi) does not
        const uint32_t mid = lo + (hi - lo) / 2u;
        memcpy(&f, &mid, 4);
        if (sqrtf(f) < radius) lo = mid;
        else hi = mid;
    }
    memcpy(&f, &lo, 4);
    return f;
}

void pn2_set_bq_group(int lanes_per_query) { pn2::g_bq_group.store(lanes_per_query, std::memory_order_relaxed); }

int pn2_query_ball_point(int b, int n, int m, float radius, int nsample, const float* xyz1, const float* xyz2,
                         int* idx, int* pts_cnt, void* stream) {
    return pn2::query_ball_point_brute(b, n, m, radius, nsample, xyz1, nullptr, xyz2, idx, pts_cnt, pn2::as_stream(stream));
}

}  // extern "C"
