// ball_query_grid.cu — query_ball_point through a uniform grid, for sparse balls.
//
// Same contract and bit-exact results as ball_query.cu (reference tf_grouping_g.cu:3-36): the first
// `nsample` data indices in ascending order whose distance test passes, row padded with the first
// hit.  The brute-force kernel must scan the whole cloud whenever a ball holds fewer than nsample
// points (the common case in set abstraction: cfg2 averages 15 hits of 32 among 4096 points).
// Here each cloud is binned once into cells of edge h >= 1.01*radius (one CTA per cloud: counting
// sort with shared-memory atomics; the order inside a cell is irrelevant); a query then tests only
// the points of its 3x3x3 cell neighbourhood (~27 h^3/V of the cloud), gathers the hits and orders
// them by index with a rank sort.  The distance test is the very same
// expression on the very same operands, so the hit set — hence the output — is identical.
// Balls that overflow the hit buffer (dense spots, duplicate-heavy clouds) fall back, inside the
// kernel, to the index-ordered scan with early exit, which is cheap exactly when balls are dense.
// Clouds where the neighbourhood is not much smaller than the cloud (large radius) are flagged by
// the build kernel and served by the brute-force kernel instead.
#include <math.h>

#include <atomic>

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kGbThreads = 1024;   // build: one CTA per cloud
constexpr int kGqThreads = 256;    // query: 8 warps, one query per warp
constexpr int kGridMaxN = 1 << 20;   // workspace sizing only: larger clouds take the brute-force path
constexpr int kGridMinN = 2048;      // below this the brute-force kernel is already latency-bound
constexpr float kGridDenseFrac = 0.9f;  // local-density estimate of points per ball above this fraction of nsample: early-exit scan wins
constexpr int kHitCap = 128;       // hits buffered per query before falling back to the ordered scan
// per-cloud parameter block (ints): [0] use_grid flag, [1..3] dims, [4] origin.x bits, [5] origin.y, [6] origin.z, [7] inv_h bits
constexpr int kGridParamInts = 8;

__host__ __device__ inline size_t grid_ws_ints_per_cloud(int n) {
    return (size_t)kGridParamInts + (size_t)n + (size_t)kGridMaxDim * kGridMaxDim * kGridMaxDim + 1;
}

__global__ void __launch_bounds__(kGbThreads, 1)
bq_grid_build_kernel(int n, float radius, int nsample, const float* __restrict__ xyz1, int* __restrict__ ws, size_t ws_stride,
                     const int* __restrict__ lengths) {
    constexpr int T = kGbThreads;
    constexpr int MAXC = kGridMaxDim * kGridMaxDim * kGridMaxDim;
    __shared__ float s_red[6][32];
    __shared__ int s_cnt[MAXC];     // per-cell count, then the scatter cursor
    __shared__ int s_wsum[32];
    __shared__ int s_heavy;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const float* __restrict__ pts = xyz1 + (size_t)cloud * n * 3;
    int* __restrict__ params = ws + (size_t)cloud * ws_stride;
    int* __restrict__ sorted_idx = params + kGridParamInts;
    int* __restrict__ cell_start = sorted_idx + n;
    n = cloud_length(lengths, cloud, n);  // the layout above is sized for the stride; from here on n is the cloud's length

    const GridGeometry geo = grid_geometry(pts, n, radius, s_red, [&] {
        for (int c = tid; c < MAXC; c += T) s_cnt[c] = 0;
        if (tid == 0) s_heavy = 0;
    });
    // expected points per ball if the cloud were uniform in its box: when that reaches nsample the
    // ordered scan of the brute-force kernel exits early and beats the neighbourhood search
    const float vol = fmaxf(geo.ext[0], geo.h) * fmaxf(geo.ext[1], geo.h) * fmaxf(geo.ext[2], geo.h);
    const float expect = (float)n * 4.18879f * radius * radius * radius / vol;
    // neighbourhood / grid volume: use the grid only when it prunes at least ~70 % of the cloud
    bool use_grid = geo.finite_box && n >= kGridMinN && 10 * geo.nb <= 3 * geo.ncell && expect < 0.75f * (float)nsample;
    if (use_grid) {  // CTA-uniform
        // pass 1: histogram
        for (int k = tid; k < n; k += T) {
            int cc[3];
#pragma unroll
            for (int c = 0; c < 3; ++c)
                cc[c] = min(max(grid_cell(__ldg(pts + 3 * (size_t)k + c), geo.mn[c], geo.inv_h, geo.dims[c]), 0), geo.dims[c] - 1);
            atomicAdd(&s_cnt[(cc[2] * geo.dims[1] + cc[1]) * geo.dims[0] + cc[0]], 1);
        }
        __syncthreads();
        // exclusive scan over the cells: each thread owns a contiguous run of cells
        const int per = (geo.ncell + T - 1) / T;
        const int c0 = min(tid * per, geo.ncell), c1 = min(c0 + per, geo.ncell);
        int local = 0, heavy = 0;
        float sq = 0.f;
        for (int c = c0; c < c1; ++c) {
            const int cntc = s_cnt[c];
            local += cntc;
            sq += (float)cntc * (float)cntc;
            heavy |= (cntc > 256) ? 1 : 0;  // a crowded cell (duplicate-heavy data): its neighbourhoods degenerate to scans
        }
        // density-aware estimate of the points per ball: a point of cell i sees about
        // c_i * (ball volume / cell volume) neighbours, so the mean over points is
        // sum(c_i^2)/n * 4.19 (r/h)^3.  Surface-like clouds fill few cells densely: their balls
        // fill up and the early-exit scan wins even though the box-uniform estimate says sparse.
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(kFullMask, sq, o);
        if (lane == 0) s_red[0][warp] = sq;
        if (heavy) s_heavy = 1;
        int run = cta_exclusive_sum_1024(local, s_wsum);
        for (int c = c0; c < c1; ++c) {
            const int cntc = s_cnt[c];
            cell_start[c] = run;
            s_cnt[c] = run;  // becomes the scatter cursor
            run += cntc;
        }
        if (tid == 0) cell_start[geo.ncell] = n;
        __syncthreads();
        float sqsum = s_red[0][lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sqsum += __shfl_xor_sync(kFullMask, sqsum, o);
        const float rh = radius * geo.inv_h;
        const float expect_local = 4.18879f * rh * rh * rh * sqsum / (float)n;
        use_grid = (s_heavy == 0) && (expect_local < kGridDenseFrac * (float)nsample);
        if (use_grid) {
            // pass 2: scatter (order inside a cell does not matter: hits are rank-sorted by index later)
            for (int k = tid; k < n; k += T) {
                int cc[3];
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    cc[c] = min(max(grid_cell(__ldg(pts + 3 * (size_t)k + c), geo.mn[c], geo.inv_h, geo.dims[c]), 0), geo.dims[c] - 1);
                const int pos = atomicAdd(&s_cnt[(cc[2] * geo.dims[1] + cc[1]) * geo.dims[0] + cc[0]], 1);
                sorted_idx[pos] = k;
            }
        }
    }
    if (tid == 0) {
        params[0] = use_grid ? 1 : 0;
        params[1] = geo.dims[0]; params[2] = geo.dims[1]; params[3] = geo.dims[2];
        params[4] = __float_as_int(geo.mn[0]); params[5] = __float_as_int(geo.mn[1]); params[6] = __float_as_int(geo.mn[2]);
        params[7] = __float_as_int(geo.inv_h);
    }
}

__global__ void __launch_bounds__(kGqThreads)
bq_grid_query_kernel(int n, int m, float thr, int nsample, const float* __restrict__ xyz1,
                     const float* __restrict__ xyz2, int* __restrict__ idx, int* __restrict__ pts_cnt,
                     const int* __restrict__ ws, size_t ws_stride, const int* __restrict__ lengths) {
    __shared__ int s_hits[kGqThreads / 32][kHitCap];
    __shared__ int s_first[kGqThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cloud = blockIdx.y;
    const int* __restrict__ params = ws + (size_t)cloud * ws_stride;
    // this cloud is served by the brute-force kernel (its own flag, or the batch-level rule)
    if (params[0] == 0 || !batch_uses_grid(ws, ws_stride, (int)gridDim.y)) return;
    const int q = blockIdx.x * (kGqThreads / 32) + warp;
    if (q >= m) return;  // warp-uniform; no CTA-wide barriers below
    const int dx = params[1], dy = params[2], dz = params[3];
    const float ox = __int_as_float(params[4]), oy = __int_as_float(params[5]), oz = __int_as_float(params[6]);
    const float inv_h = __int_as_float(params[7]);
    const int* __restrict__ sorted_idx = params + kGridParamInts;
    const int* __restrict__ cell_start = sorted_idx + n;
    const float* __restrict__ data = xyz1 + (size_t)cloud * n * 3;
    n = cloud_length(lengths, cloud, n);  // the grid holds only these points; the ordered scan below stops here too
    const float* qp = xyz2 + ((size_t)cloud * m + q) * 3;
    const float qx = qp[0], qy = qp[1], qz = qp[2];
    int* __restrict__ row = idx + ((size_t)cloud * m + q) * nsample;
    const unsigned lt_mask = (1u << lane) - 1u;

    const int cx = grid_cell(qx, ox, inv_h, dx), cy = grid_cell(qy, oy, inv_h, dy), cz = grid_cell(qz, oz, inv_h, dz);
    const int x0 = max(cx - 1, 0), x1 = min(cx + 1, dx - 1);
    // the neighbourhood is 9 rows (dy, dz in {-1,0,1}) of up to 3 x-adjacent cells, i.e. 9 contiguous
    // candidate ranges; lanes 3r..3r+2 walk range r with stride 3
    int p = 0, p1 = 0;
    {
        const int r = lane / 3, sub = lane - 3 * r;
        const int y = cy + (r % 3) - 1, z = cz + (r / 3) - 1;
        if (lane < 27 && x0 <= x1 && y >= 0 && y < dy && z >= 0 && z < dz) {
            const int rowbase = (z * dy + y) * dx;
            p = __ldg(cell_start + rowbase + x0) + sub;
            p1 = __ldg(cell_start + rowbase + x1 + 1);
        }
    }
    int hcount = 0;
    // a non-finite query (NaN: a hit against EVERY point in the reference, fmaxf(NaN,1e-20f) < radius) cannot be
    // served from its cell neighbourhood: warp-uniformly take the ordered scan below
    const bool qfinite = (fabsf(qx) <= 3.0e38f) && (fabsf(qy) <= 3.0e38f) && (fabsf(qz) <= 3.0e38f);
    if (!qfinite) {
        p = p1 = 0;
        hcount = kHitCap + 1;
    }
    while (__any_sync(kFullMask, p < p1)) {
        bool hit = false;
        int k = 0;
        if (p < p1) {
            k = __ldg(sorted_idx + p);
            const float* s = data + (size_t)k * 3;
            const float d2 = d2_fma_pattern(qx, qy, qz, __ldg(s), __ldg(s + 1), __ldg(s + 2));
            hit = !(d2 > thr);
        }
        p += 3;
        const unsigned bal = __ballot_sync(kFullMask, hit);
        if (bal) {
            const int r = hcount + __popc(bal & lt_mask);
            if (hit && r < kHitCap) s_hits[warp][r] = k;
            hcount += __popc(bal);
            if (hcount > kHitCap) break;  // warp-uniform: dense ball, switch to the ordered scan
        }
    }
    const bool overflow = hcount > kHitCap;
    int cnt;
    if (overflow) {
        // dense ball: ordered scan with early exit (stops after ~nsample/density points)
        cnt = 0;
        for (int base = 0; base < n && cnt < nsample; base += 32) {
            const int k = base + lane;
            bool hit = false;
            if (k < n) {
                const float* s = data + (size_t)k * 3;
                const float d2 = d2_fma_pattern(qx, qy, qz, __ldg(s), __ldg(s + 1), __ldg(s + 2));
                hit = !(d2 > thr);
            }
            const unsigned bal = __ballot_sync(kFullMask, hit);
            if (bal) {
                const int r = cnt + __popc(bal & lt_mask);
                if (hit && r < nsample) row[r] = k;
                if (hit && r == 0) s_first[warp] = k;
                cnt = min(cnt + __popc(bal), nsample);
            }
        }
    } else {
        // order the (distinct) hit indices: rank = number of smaller hits
        __syncwarp();
        cnt = min(hcount, nsample);
        for (int e = lane; e < hcount; e += 32) {
            const int v = s_hits[warp][e];
            int r = 0;
            for (int f = 0; f < hcount; ++f) r += (s_hits[warp][f] < v) ? 1 : 0;
            if (r < nsample) row[r] = v;
            if (r == 0) s_first[warp] = v;
        }
    }
    __syncwarp();
    const int first = (cnt > 0) ? s_first[warp] : 0;
    for (int l = cnt + lane; l < nsample; l += 32) row[l] = first;
    if (lane == 0) pts_cnt[(size_t)cloud * m + q] = cnt;
}

static std::atomic<int> g_bq_mode{0};  // 0 auto (shared-memory grid kernel when the cloud fits it), 1 brute force only, 2 the global-memory grid path

// The grid build / query / whole-path entries below, on the clouds' first lengths[b] points (lengths == NULL: all n).
static int ball_grid_build(int b, int n, float radius, int nsample, const float* xyz1, const int* lengths, void* workspace,
                           size_t workspace_bytes, cudaStream_t st) {
    if (b <= 0 || n <= 0 || nsample <= 0 || !(radius > 0.0f) || !xyz1 || !workspace) return (int)cudaErrorInvalidValue;
    const size_t need = pn2_query_ball_point_workspace_bytes(b, n);
    // radius <= 1e-20: no distance passes the reference's max(d, 1e-20) < radius test, and the query half refuses it
    if (need == 0 || workspace_bytes < need || b > 65535 || pn2_ball_threshold(radius) < 0.0f) return (int)cudaErrorInvalidValue;
    bq_grid_build_kernel<<<b, kGbThreads, 0, st>>>(n, radius, nsample, xyz1, static_cast<int*>(workspace),
                                                   grid_ws_ints_per_cloud(n), lengths);
    return finish_launch();
}

static int query_ball_point_prebuilt(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths,
                                     const float* xyz2, int* idx, int* pts_cnt, const void* workspace, size_t workspace_bytes,
                                     cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || nsample <= 0 || !(radius > 0.0f)) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz1 || !xyz2 || !idx || !pts_cnt || !workspace) return (int)cudaErrorInvalidValue;
    const size_t need = pn2_query_ball_point_workspace_bytes(b, n);
    const float thr = pn2_ball_threshold(radius);
    if (need == 0 || workspace_bytes < need || b > 65535 || thr < 0.0f) return (int)cudaErrorInvalidValue;
    const int* ws = static_cast<const int*>(workspace);
    const size_t stride = grid_ws_ints_per_cloud(n);
    dim3 grid((m + kGqThreads / 32 - 1) / (kGqThreads / 32), b, 1);
    bq_grid_query_kernel<<<grid, kGqThreads, 0, st>>>(n, m, thr, nsample, xyz1, xyz2, idx, pts_cnt, ws, stride, lengths);
    int rc = finish_launch();
    if (rc) return rc;
    // clouds the build kernel did not flag for the grid are done by the brute-force kernel
    return launch_ball_query_brute(b, n, m, thr, nsample, xyz1, lengths, xyz2, idx, pts_cnt, ws, (int)stride, st);
}

int query_ball_point_ws(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths,
                        const float* xyz2, int* idx, int* pts_cnt, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || nsample <= 0 || !(radius > 0.0f)) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz1 || !xyz2 || !idx || !pts_cnt) return (int)cudaErrorInvalidValue;
    const size_t need = pn2_query_ball_point_workspace_bytes(b, n);
    const float thr = pn2_ball_threshold(radius);
    // clouds that fit the shared-memory grid of sa_fused.cu (n <= 9700): one launch that builds the grid in shared
    // memory and serves the queries from it — one launch instead of build + query + brute-force back to back from
    // n = 2048 up; no workspace needed
    const int mode = g_bq_mode.load(std::memory_order_relaxed);
    if (mode == 0 && n >= kGridMinN && pn2_ball_group_fits(n) && thr >= 0.0f) {
        // ... when there are queries enough to pay for the grids (every CTA builds its own): below ~4096 queries the
        // packed brute-force kernel is ahead (r2_report.json, cfg4 SA1024 at B = 2: 2048 queries x 8192 points,
        // 0.0246 ms against 0.0287)
        if ((long long)b * m >= 4096) return ball_group(b, n, m, radius, nsample, xyz1, lengths, xyz2, idx, pts_cnt, nullptr, 0, st);
        return query_ball_point_brute(b, n, m, radius, nsample, xyz1, lengths, xyz2, idx, pts_cnt, st);
    }
    if (mode == 1 || !workspace || need == 0 || workspace_bytes < need || thr < 0.0f || b > 65535)
        return query_ball_point_brute(b, n, m, radius, nsample, xyz1, lengths, xyz2, idx, pts_cnt, st);
    int rc = ball_grid_build(b, n, radius, nsample, xyz1, lengths, workspace, workspace_bytes, st);
    if (rc) return rc;
    return query_ball_point_prebuilt(b, n, m, radius, nsample, xyz1, lengths, xyz2, idx, pts_cnt, workspace, workspace_bytes, st);
}

// the largest pn2_query_ball_point_workspace_bytes(b, k) over k <= n (0 outside [kGridMinN, kGridMaxN], growing inside)
size_t query_ball_point_workspace_bound(int b, int n) { return pn2_query_ball_point_workspace_bytes(b, n < kGridMaxN ? n : kGridMaxN); }

}  // namespace pn2

extern "C" {

void pn2_set_bq_mode(int mode) { pn2::g_bq_mode.store(mode, std::memory_order_relaxed); }

size_t pn2_query_ball_point_workspace_bytes(int b, int n) {
    if (b <= 0 || n < pn2::kGridMinN || n > pn2::kGridMaxN) return 0;
    return sizeof(int) * (size_t)b * pn2::grid_ws_ints_per_cloud(n);
}

// Split form of pn2_query_ball_point_ws: the grid build only needs the data points, so a caller can
// run it on a second stream while farthest point sampling is still producing the queries.
int pn2_ball_grid_build(int b, int n, float radius, int nsample, const float* xyz1, void* workspace,
                        size_t workspace_bytes, void* stream) {
    return pn2::ball_grid_build(b, n, radius, nsample, xyz1, nullptr, workspace, workspace_bytes, pn2::as_stream(stream));
}

int pn2_query_ball_point_prebuilt(int b, int n, int m, float radius, int nsample, const float* xyz1, const float* xyz2,
                                  int* idx, int* pts_cnt, const void* workspace, size_t workspace_bytes, void* stream) {
    return pn2::query_ball_point_prebuilt(b, n, m, radius, nsample, xyz1, nullptr, xyz2, idx, pts_cnt, workspace, workspace_bytes,
                                          pn2::as_stream(stream));
}

int pn2_query_ball_point_ws(int b, int n, int m, float radius, int nsample, const float* xyz1, const float* xyz2,
                            int* idx, int* pts_cnt, void* workspace, size_t workspace_bytes, void* stream) {
    return pn2::query_ball_point_ws(b, n, m, radius, nsample, xyz1, nullptr, xyz2, idx, pts_cnt, workspace, workspace_bytes,
                                    pn2::as_stream(stream));
}

int pn2_query_ball_point_ragged(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths1,
                                const float* xyz2, int* idx, int* pts_cnt, void* workspace, size_t workspace_bytes,
                                void* stream) {
    return pn2::query_ball_point_ws(b, n, m, radius, nsample, xyz1, lengths1, xyz2, idx, pts_cnt, workspace, workspace_bytes,
                                    pn2::as_stream(stream));
}

}  // extern "C"
