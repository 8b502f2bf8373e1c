// sa_fused.cu — the sampling+grouping half of a set-abstraction layer as ONE overlapped pair of
// kernels, for sm_90a.
//
// Replaces the op sequence sample_and_group issues (reference utils/pointnet_util.py:40-46):
//   farthest_point_sample -> gather_point -> query_ball_point -> group_point(xyz) [-> tile/sub]
// i.e. tf_sampling_g.cu:105-181 + tf_grouping_g.cu:3-57, with results bit-identical to running
// pn2_fps_gather, pn2_query_ball_point and pn2_group_point one after the other.
//
// Why: farthest point sampling is a serial chain that keeps ONE SM per cloud busy (32 of 132 at
// B=32) for most of the layer, and run on their own the ball query + grouping start strictly after
// it.  Here a second grid — `ball_group_kernel`, one 1024-thread CTA per cloud —
// starts on the idle SMs as soon as every sampling CTA is resident (programmatic dependent launch:
// the sampling kernel pre-fills its index output with -1 and executes
// griddepcontrol.launch_dependents; SASS PREEXIT) and serves centroid j the moment index j turns
// non-negative.  The consumer needs no flag and the producer no fence: the 4-byte index IS the
// message (a centroid is a data point, so its coordinates are read from the immutable input cloud).
// When the chain ends, all that is left is the last few queries: the layer costs little more than
// the sampling time.
//
// The consumer builds, in shared memory, the same uniform grid as ball_query_grid.cu (cell edge >=
// 1.01 radius, points stored cell-sorted as float4 (x,y,z,index)) when the cloud's balls are sparse,
// or keeps the cloud in index order when they are dense; a warp per query then either walks the 9
// contiguous candidate ranges of the 3x3x3 cell neighbourhood and rank-sorts the hits by index, or
// scans in index order with early exit.  The hit test is the very same expression on the very same
// operands as ball_query.cu (pn2::d2_fma_pattern(query, point), !(d2 > thr)), so idx / pts_cnt are
// bit-identical; grouped_xyz is emitted in the same pass (raw gather, or centred on the query with
// one __fsub_rn per coordinate — utils/pointnet_util.py:46), so group_point(xyz) disappears.
//
// kNN grouping (sample_and_group(..., knn=True)) gets the same overlap from knn_group_kernel below: the
// consumer keeps the whole cloud in shared memory and runs knn_point's per-query warp routine
// (knn_warp.cuh) on each centroid as it appears.
//
// The same kernel also serves query_ball_point + group_point(xyz) on their own (all queries known up
// front: several CTAs per cloud, no polling) — one launch instead of grid build + grid query +
// brute-force + group.
#include <math.h>
#include <stdlib.h>

#include <atomic>

#include "knn_warp.cuh"
#include "pn2_common.cuh"

namespace pn2 {

constexpr int kBgThreads = 1024;
constexpr int kBgWarps = kBgThreads / 32;
constexpr int kBgMaxCells = kGridMaxDim * kGridMaxDim * kGridMaxDim;  // 4096
constexpr int kBgHitCap = 256;                                  // hit buffer per query (compacted to the nsample smallest indices when it fills up)
constexpr int kBgCompactMax = 128;                              // compaction needs nsample <= this (else a full buffer falls back to the ordered scan)
constexpr int kBgMinGridN = 512;                                // below this the in-smem ordered scan is already short
constexpr size_t kBgSmemMax = 200 * 1024;
constexpr int kBgPosBits = 14;  // positions and indices < 2^14 (n <= 9700 by the shared-memory budget): one int holds both

__host__ __device__ inline size_t bg_smem_bytes(int n) {
    // float4 points + cell_start[kBgMaxCells + 1] (padded to 16 B) + cursors / hit buffers (aliased)
    return (size_t)n * 16 + (size_t)(kBgMaxCells + 4) * 4 + (size_t)kBgWarps * kBgHitCap * 4;
}
// Small clouds keep BOTH layouts in shared memory — cell-sorted for the grid walk and index-ordered for the scan — so
// each query can take whichever is cheaper for its own ball (a ball that covers a quarter of the cloud is served by
// an index-ordered scan of a few dozen iterations; a small one by its 27 cells).
__host__ __device__ inline bool bg_dual_layout(int n) { return bg_smem_bytes(n) + (size_t)n * 16 <= kBgSmemMax; }

__device__ __forceinline__ int ld_volatile_s32(const int* p) {
    int v;
    asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// xyz1 (b,n,3) data.  Queries: xyz2 (b,m,3), or — when q_idx != NULL — the data points
// xyz1[b, q_idx[b,j]], where q_idx (b,m) is being filled by a concurrently running sampling kernel
// (-1 = not produced yet).  idx (b,m,nsample), pts_cnt (b,m), grouped (b,m,nsample,3) or NULL.
// L (ragged batch): cloud i is its first cloud_length(lengths, i, n) points.  A template flag, so that the instance
// without lengths compiles to the code it always did.
template <bool L>
__global__ void __launch_bounds__(kBgThreads, 1)
ball_group_kernel(int n, int m, float radius, float thr, int nsample, const float* __restrict__ xyz1,
                  const float* __restrict__ xyz2, const int* q_idx, int* __restrict__ idx,
                  int* __restrict__ pts_cnt, float* __restrict__ grouped, int center, int ctas_per_cloud,
                  int wait_primary, int trigger_next, const int* __restrict__ lengths) {
    constexpr int T = kBgThreads, NW = kBgWarps;
    extern __shared__ __align__(16) unsigned char s_raw[];
    float4* __restrict__ s_pts = reinterpret_cast<float4*>(s_raw);                     // [n]
    int* __restrict__ s_cell = reinterpret_cast<int*>(s_raw + (size_t)n * 16);          // [kBgMaxCells + 1]: cell_start
    int* __restrict__ s_cur = s_cell + (kBgMaxCells + 4);                               // build: histogram / cursors
    int(*s_hits)[kBgHitCap] = reinterpret_cast<int(*)[kBgHitCap]>(s_cur);               // query: per-warp hit positions
    const bool dual = bg_dual_layout(n);                                                // index-ordered copy behind the hit buffers
    float4* __restrict__ s_orig = reinterpret_cast<float4*>(s_raw + bg_smem_bytes(n));  // [n], valid when dual && use_grid
    __shared__ float s_red[6][32];
    __shared__ int s_wsum[32];
    __shared__ float4 s_first[NW];

    // multi-scale grouping chains several of these grids behind one sampling kernel: let the next one start
    // as soon as this one is resident (it polls the same index buffer)
    if (trigger_next) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x / ctas_per_cloud, part = blockIdx.x - cloud * ctas_per_cloud;
    const float* __restrict__ pts = xyz1 + (size_t)cloud * n * 3;
    // The shared-memory layout above is sized for the row stride; from here on n is this cloud's length: only its
    // points are boxed, binned and scanned (the layout choice below may then differ from a dense call; the results
    // cannot)
    if (L) n = cloud_length(lengths, cloud, n);

    // ---- bounding box and grid (a NaN coordinate makes the box infinite: such clouds take the ordered scan)
    const GridGeometry geo = grid_geometry(pts, n, radius, s_red, [&] {
        for (int c = tid; c < kBgMaxCells; c += T) s_cur[c] = 0;
    });
    // The grid is used whenever the 3x3x3 neighbourhood prunes >= 70 % of the cells — whatever the density:
    // a ball with just over nsample points makes the index-ordered scan read most of the cloud before it
    // has its nsample hits (surface-like clouds),
    // while the grid tests ~27 cells and keeps the nsample smallest indices in a bounded buffer.
    const bool use_grid = geo.finite_box && n >= kBgMinGridN && 10 * geo.nb <= 3 * geo.ncell;
    if (use_grid) {  // CTA-uniform
        for (int k = tid; k < n; k += T) {
            int cc[3];
#pragma unroll
            for (int c = 0; c < 3; ++c)
                cc[c] = min(max(grid_cell(__ldg(pts + 3 * (size_t)k + c), geo.mn[c], geo.inv_h, geo.dims[c]), 0), geo.dims[c] - 1);
            atomicAdd(&s_cur[(cc[2] * geo.dims[1] + cc[1]) * geo.dims[0] + cc[0]], 1);
        }
        __syncthreads();
        const int per = (geo.ncell + T - 1) / T;
        const int c0 = min(tid * per, geo.ncell), c1 = min(c0 + per, geo.ncell);
        int local = 0;
        for (int c = c0; c < c1; ++c) local += s_cur[c];
        int run = cta_exclusive_sum_1024(local, s_wsum);
        for (int c = c0; c < c1; ++c) {
            const int cntc = s_cur[c];
            s_cell[c] = run;
            s_cur[c] = run;
            run += cntc;
        }
        if (tid == 0) s_cell[geo.ncell] = n;
        __syncthreads();
        if (use_grid) {
            for (int k = tid; k < n; k += T) {
                const float x = __ldg(pts + 3 * (size_t)k), y = __ldg(pts + 3 * (size_t)k + 1), z = __ldg(pts + 3 * (size_t)k + 2);
                const int cx = min(max(grid_cell(x, geo.mn[0], geo.inv_h, geo.dims[0]), 0), geo.dims[0] - 1);
                const int cy = min(max(grid_cell(y, geo.mn[1], geo.inv_h, geo.dims[1]), 0), geo.dims[1] - 1);
                const int cz = min(max(grid_cell(z, geo.mn[2], geo.inv_h, geo.dims[2]), 0), geo.dims[2] - 1);
                const int pos = atomicAdd(&s_cur[(cz * geo.dims[1] + cy) * geo.dims[0] + cx], 1);
                s_pts[pos] = make_float4(x, y, z, __int_as_float(k));
                if (dual) s_orig[k] = make_float4(x, y, z, __int_as_float(k));
            }
        }
    }
    if (!use_grid) {  // index order: the ordered scan reads it straight from shared memory
        for (int k = tid; k < n; k += T)
            s_pts[k] = make_float4(__ldg(pts + 3 * (size_t)k), __ldg(pts + 3 * (size_t)k + 1), __ldg(pts + 3 * (size_t)k + 2),
                                   __int_as_float(k));
    }
    __syncthreads();  // grid / cloud complete; s_cur is dead from here on (s_hits aliases it)

    // ---- queries: warp `gw` of the cloud's ctas_per_cloud*32 warps serves queries gw, gw + stride, ... ----
    const unsigned lt_mask = (1u << lane) - 1u;
    const int qstride = ctas_per_cloud * NW;
    const int dxs = geo.dims[0], dys = geo.dims[1], dzs = geo.dims[2];
    const long long t_start = clock64();
    for (int q = part * NW + warp; q < m; q += qstride) {
        float qx, qy, qz;
        if (q_idx) {
            // wait for the sampling kernel to publish centroid q (its index turns non-negative)
            int qi = 0;
            if (lane == 0) {
                const int* src = q_idx + (size_t)cloud * m + q;
                qi = ld_volatile_s32(src);
                unsigned backoff = 32;
                while (qi < 0) {
                    __nanosleep(backoff);
                    if (backoff < 256) backoff <<= 1;
                    qi = ld_volatile_s32(src);
                    if (clock64() - t_start > 4000000000ll) break;  // ~2 s: never hang the device on a lost producer
                }
            }
            qi = __shfl_sync(kFullMask, qi, 0);
            if (qi < 0 || qi >= n) {  // producer lost / corrupt index: flag the row instead of faulting
                if (lane == 0) pts_cnt[(size_t)cloud * m + q] = -1;
                continue;
            }
            if (!use_grid || dual) {  // an index-ordered copy of the cloud is in shared memory: no L2 round trip
                const float4 c = use_grid ? s_orig[qi] : s_pts[qi];
                qx = c.x;
                qy = c.y;
                qz = c.z;
            } else {
                qx = __ldg(pts + 3 * (size_t)qi);
                qy = __ldg(pts + 3 * (size_t)qi + 1);
                qz = __ldg(pts + 3 * (size_t)qi + 2);
            }
        } else {
            const float* qp = xyz2 + ((size_t)cloud * m + q) * 3;
            qx = __ldg(qp);
            qy = __ldg(qp + 1);
            qz = __ldg(qp + 2);
        }
        const float ox = center ? qx : 0.f, oy = center ? qy : 0.f, oz = center ? qz : 0.f;
        int* __restrict__ row = idx + ((size_t)cloud * m + q) * nsample;
        float* __restrict__ grow = grouped ? grouped + ((size_t)cloud * m + q) * nsample * 3 : nullptr;
        auto emit = [&](int r, int k, float x, float y, float z) {
            row[r] = k;
            if (grow) {
                // centred: xyz[idx] - new_xyz, one rounding per coordinate (utils/pointnet_util.py:46); a raw copy
                // otherwise (x - 0 would canonicalise a NaN payload, which a gather never does)
                grow[3 * r + 0] = center ? __fsub_rn(x, ox) : x;
                grow[3 * r + 1] = center ? __fsub_rn(y, oy) : y;
                grow[3 * r + 2] = center ? __fsub_rn(z, oz) : z;
            }
        };

        int cnt = 0;
        bool scanned = false;
        const bool qfinite = (fabsf(qx) <= 3.0e38f) && (fabsf(qy) <= 3.0e38f) && (fabsf(qz) <= 3.0e38f);  // false for NaN / inf
        if (use_grid && qfinite) {
            const int cx = grid_cell(qx, geo.mn[0], geo.inv_h, dxs), cy = grid_cell(qy, geo.mn[1], geo.inv_h, dys), cz = grid_cell(qz, geo.mn[2], geo.inv_h, dzs);
            const int x0 = max(cx - 1, 0), x1 = min(cx + 1, dxs - 1);
            // 9 rows (dy, dz in {-1,0,1}) of up to 3 x-adjacent cells = 9 contiguous candidate ranges;
            // lanes 3r..3r+2 own range r
            int p = 0, p1 = 0;
            const int rr = lane / 3, sub = lane - 3 * rr;
            {
                const int y = cy + (rr % 3) - 1, z = cz + (rr / 3) - 1;
                if (lane < 27 && x0 <= x1 && y >= 0 && y < dys && z >= 0 && z < dzs) {
                    const int rowbase = (z * dys + y) * dxs;
                    p = s_cell[rowbase + x0];
                    p1 = s_cell[rowbase + x1 + 1];
                }
            }
            const int len = (sub == 0) ? p1 - p : 0;
            const int total = __reduce_add_sync(kFullMask, len), longest = __reduce_max_sync(kFullMask, len);
            // Hits go into a per-warp buffer as (data index << 14 | position) keys (indices are distinct, so keys
            // order by index).  When the buffer is nearly full it is sorted and cut back to its nsample smallest
            // keys; from then on only hits below the largest kept key are accepted — so a dense ball costs a few
            // sorts of 256 keys, never a scan of the cloud.
            // a neighbourhood that holds more than a quarter of the cloud (large radius, or a cell of coincident
            // points next door): the index-ordered scan from shared memory is at most n/32 cheap iterations and stops
            // early when the ball is dense — skip the grid walk for this query
            const bool scan_instead = dual && 4 * total > n;
            int hcount = 0, tau = 0x7fffffff, tested = 0;
            bool dense = false;  // at least nsample hits were seen (then pts_cnt = nsample)
            bool overflow = scan_instead;
            auto compact = [&]() {
                __syncwarp();
                int key[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) key[j] = (32 * j + lane < hcount) ? s_hits[warp][32 * j + lane] : 0x7fffffff;
                bitonic_sort_keys<8, 8>(key, lane);
#pragma unroll
                for (int j = 0; j < 8; ++j) s_hits[warp][32 * j + lane] = key[j];
                __syncwarp();
                if (hcount >= nsample) {
                    hcount = nsample;
                    tau = s_hits[warp][nsample - 1];
                    dense = true;
                }
            };
            auto test = [&](bool active, int pos) {  // one candidate per active lane
                if (hcount > kBgHitCap - 32) {       // warp-uniform: make room before the buffer can overflow
                    // The first time the buffer fills, hits/tested estimates the ball's population.  A VERY dense ball
                    // (a cell of coincident points: thousands of candidates, nearly all hits) is served faster by the
                    // index-ordered scan, which stops after ~n*nsample/population points (x3: it reads global memory),
                    // than by testing the rest of the neighbourhood; a moderately dense one by carrying on.
                    const float scan_cost = (dual ? 1.0f : 3.0f) * (float)n * (float)nsample * (float)tested / ((float)hcount * (float)total);
                    const float grid_cost = (float)(total - tested) + 2240.0f;  // + a few sorts of the buffer
                    if (nsample > kBgCompactMax || (!dense && scan_cost < grid_cost)) {
                        overflow = true;
                        return;
                    }
                    compact();
                }
                bool hit = false;
                int key = 0;
                if (active) {
                    const float4 c = s_pts[pos];
                    key = (__float_as_int(c.w) << kBgPosBits) | pos;
                    hit = !(d2_fma_pattern(qx, qy, qz, c.x, c.y, c.z) > thr) && key < tau;
                }
                tested += __popc(__ballot_sync(kFullMask, active));
                const unsigned bal = __ballot_sync(kFullMask, hit);
                if (bal) {
                    const int r = hcount + __popc(bal & lt_mask);
                    if (hit) s_hits[warp][r] = key;
                    hcount += __popc(bal);
                }
            };
            if (overflow) {
                // (scan_instead)
            } else if (longest <= 48) {
                // balanced ranges: lanes 3r..3r+2 walk range r with stride 3
                p += sub;
                while (!overflow && __any_sync(kFullMask, p < p1)) {
                    test(p < p1, p);
                    p += 3;
                }
            } else {
                // a crowded cell in the neighbourhood: all 32 lanes walk one range after the other
                for (int r = 0; r < 9 && !overflow; ++r) {
                    const int a = __shfl_sync(kFullMask, p, 3 * r), e = __shfl_sync(kFullMask, p1, 3 * r);
                    for (int pos = a + lane; pos - lane < e && !overflow; pos += 32) test(pos < e, pos);
                }
            }
            if (!overflow) {
                // order the hits by data index: bitonic sort of the keys in registers (element i lives in
                // register i/32 of lane i%32)
                __syncwarp();
                cnt = dense ? nsample : min(hcount, nsample);
                int key[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) key[j] = (32 * j + lane < hcount) ? s_hits[warp][32 * j + lane] : 0x7fffffff;
                const int nreg = (hcount + 31) >> 5;  // registers that hold real keys (warp-uniform)
                if (nreg <= 1) bitonic_sort_keys<1, 8>(key, lane);
                else if (nreg == 2) bitonic_sort_keys<2, 8>(key, lane);
                else if (nreg <= 4) bitonic_sort_keys<4, 8>(key, lane);
                else bitonic_sort_keys<8, 8>(key, lane);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int r = 32 * j + lane;
                    if (r < cnt) {
                        const float4 c = s_pts[key[j] & ((1 << kBgPosBits) - 1)];
                        emit(r, key[j] >> kBgPosBits, c.x, c.y, c.z);
                        if (r == 0) s_first[warp] = c;
                    }
                }
                scanned = true;
            }
        }
        if (!scanned) {
            // ordered scan with early exit: from shared memory when an index-ordered copy of the cloud is there (scan
            // mode, or the dual layout of small clouds), from global memory (L1/L2) when only the cell-sorted one is.
            // Hit indices are buffered (they arrive in order) and the row is written afterwards, 32 consecutive
            // entries per store instruction — storing hit by hit costs 4 sparsely populated store instructions per
            // 32 points scanned, which made dense balls slower here than in the grid walk.
            const bool buffered = nsample <= kBgHitCap;
            __syncwarp();  // an overflowed grid walk left entries in s_hits that other lanes overwrite below
            auto load_point = [&](int k, float& x, float& y, float& z) {
                if (use_grid && !dual) {
                    x = __ldg(pts + 3 * (size_t)k);
                    y = __ldg(pts + 3 * (size_t)k + 1);
                    z = __ldg(pts + 3 * (size_t)k + 2);
                } else {
                    const float4 c = use_grid ? s_orig[k] : s_pts[k];
                    x = c.x;
                    y = c.y;
                    z = c.z;
                }
            };
            if (buffered) {
                // two points per lane and trip, indices only (ncu, cfg3 layer 1 at r = 0.4: the loop is issue-bound —
                // 80 % issue-active — so what counts is instructions per point tested)
                for (int base = 0; base < n && cnt < nsample; base += 64) {
                    const int k0 = base + lane, k1 = k0 + 32;
                    float x0, y0, z0, x1, y1, z1;
                    load_point(min(k0, n - 1), x0, y0, z0);
                    load_point(min(k1, n - 1), x1, y1, z1);
                    const bool h0 = k0 < n && !(d2_fma_pattern(qx, qy, qz, x0, y0, z0) > thr);
                    const bool h1 = k1 < n && !(d2_fma_pattern(qx, qy, qz, x1, y1, z1) > thr);
                    const unsigned b0 = __ballot_sync(kFullMask, h0), b1 = __ballot_sync(kFullMask, h1);
                    if (b0 | b1) {
                        const int r0 = cnt + __popc(b0 & lt_mask);
                        const int c1 = cnt + __popc(b0);
                        const int r1 = c1 + __popc(b1 & lt_mask);
                        if (h0 && r0 < nsample) s_hits[warp][r0] = k0;
                        if (h1 && r1 < nsample) s_hits[warp][r1] = k1;
                        cnt = min(c1 + __popc(b1), nsample);
                    }
                }
            } else {
                for (int base = 0; base < n && cnt < nsample; base += 32) {
                    const int k = base + lane;
                    bool hit = false;
                    float x = 0.f, y = 0.f, z = 0.f;
                    if (k < n) {
                        load_point(k, x, y, z);
                        hit = !(d2_fma_pattern(qx, qy, qz, x, y, z) > thr);
                    }
                    const unsigned bal = __ballot_sync(kFullMask, hit);
                    if (bal) {
                        const int r = cnt + __popc(bal & lt_mask);
                        if (hit && r < nsample) emit(r, k, x, y, z);
                        if (hit && r == 0) s_first[warp] = make_float4(x, y, z, __int_as_float(k));
                        cnt = min(cnt + __popc(bal), nsample);
                    }
                }
            }
            if (buffered) {
                __syncwarp();
                for (int r = lane; r < cnt; r += 32) {
                    const int k = s_hits[warp][r];
                    float x, y, z;
                    load_point(k, x, y, z);
                    emit(r, k, x, y, z);
                    if (r == 0) s_first[warp] = make_float4(x, y, z, __int_as_float(k));
                }
            }
        }
        __syncwarp();
        // pad the row with the first hit (tf_grouping_g.cu:26-29); rows with no hit are zeros (undefined in the reference)
        const float4 f = (cnt > 0) ? s_first[warp] : make_float4(ox, oy, oz, __int_as_float(0));
        const int fk = (cnt > 0) ? __float_as_int(f.w) : 0;
        for (int l = cnt + lane; l < nsample; l += 32) {
            row[l] = fk;
            if (grow) {
                // rows with no hit: index 0 is what an unfused group_point would gather for an all-zero row
                const float px = (cnt > 0) ? f.x : __ldg(pts + 0), py = (cnt > 0) ? f.y : __ldg(pts + 1), pz = (cnt > 0) ? f.z : __ldg(pts + 2);
                grow[3 * l + 0] = center ? __fsub_rn(px, ox) : px;
                grow[3 * l + 1] = center ? __fsub_rn(py, oy) : py;
                grow[3 * l + 2] = center ? __fsub_rn(pz, oz) : pz;
            }
        }
        if (lane == 0) pts_cnt[(size_t)cloud * m + q] = cnt;
        __syncwarp();  // s_first / s_hits are reused by this warp's next query
    }
    // Completion of this grid must imply completion of the sampling grid it overlaps (stream order and
    // graph edges only see this grid): wait for the primary to finish and flush (SASS ACQBULK).
    if (wait_primary) asm volatile("griddepcontrol.wait;" ::: "memory");
}

struct BgOnce {
    std::atomic<long long> max_dyn[2][64];  // [ragged][device]: largest dynamic shared memory the kernel may request (0 = not asked yet)
};

static int launch_ball_group(int b, int n, int m, float radius, float thr, int nsample, const float* xyz1, const int* lengths,
                             const float* xyz2, const int* q_idx, int* idx, int* pts_cnt, float* grouped, int center,
                             int ctas_per_cloud, bool dependent, bool trigger_next, cudaStream_t st) {
    static BgOnce once;
    size_t dyn = bg_smem_bytes(n);
    if (dyn > kBgSmemMax) return (int)cudaErrorInvalidValue;
    if (bg_dual_layout(n)) dyn += (size_t)n * 16;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev < 0 || dev >= 64) return (int)cudaErrorInvalidDevice;
    const int ragged = lengths ? 1 : 0;
    auto kern = ragged ? ball_group_kernel<true> : ball_group_kernel<false>;
    long long max_dyn = once.max_dyn[ragged][dev].load(std::memory_order_acquire);
    if (max_dyn == 0) {
        int optin = 0;
        cudaFuncAttributes fa;
        e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, kern);
        if (e != cudaSuccess) return (int)e;
        max_dyn = (long long)optin - (long long)fa.sharedSizeBytes;
        if (max_dyn < (long long)kBgSmemMax) return (int)cudaErrorInvalidValue;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_dyn);
        if (e != cudaSuccess) return (int)e;
        once.max_dyn[ragged][dev].store(max_dyn, std::memory_order_release);
    }
    // Overlapped with the sampling kernel, the consumer must have an SM to ITSELF: a 1024-thread CTA next
    // to a sampling CTA would take issue slots from the serial chain the whole layer waits for (measured:
    // cfg3 layer 1, N=1024, +50 us).  Asking for every byte of shared memory the SM has makes co-residency
    // with any other CTA impossible.
    static const bool exclusive = [] { const char* e = getenv("PN2_SA_EXCLUSIVE"); return !e || e[0] != '0'; }();  // experiment switch
    if (dependent && exclusive) dyn = (size_t)max_dyn;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)b * (unsigned)ctas_per_cloud, 1, 1);
    cfg.blockDim = dim3(kBgThreads, 1, 1);
    cfg.dynamicSmemBytes = dyn;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = dependent ? 1 : 0;
    e = cudaLaunchKernelEx(&cfg, kern, n, m, radius, thr, nsample, xyz1, xyz2, q_idx, idx, pts_cnt, grouped, center,
                           ctas_per_cloud, dependent ? 1 : 0, trigger_next ? 1 : 0, lengths);
    count_launch();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

static size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// Consumer CTAs per cloud and scale in the overlapped layer.  One is enough to keep up with the sampling chain
// when balls are sparse (cfg2: the layer ends 4 us after the sampling kernel); it leaves the other SMs to
// further batches on other streams.  pn2_set_sa_consumer_ctas overrides (0 = automatic).
static std::atomic<int> g_sa_consumer_ctas{0};
static int sa_consumer_ctas(int b, int nscales) {
    int r = g_sa_consumer_ctas.load(std::memory_order_relaxed);
    const int sms = num_sms(), bb = b < sms ? b : sms;
    const int room = (sms - bb) / (bb * nscales);  // SMs left per cloud and scale
    if (r <= 0) r = 1;
    if (r > room) r = room;
    return r < 1 ? 1 : r;
}

// pn2_ball_group on the clouds' first lengths[b] points (lengths == NULL: all n)
int ball_group(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths, const float* xyz2, int* idx,
               int* pts_cnt, float* grouped_xyz, int center, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || nsample <= 0 || !(radius > 0.0f)) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz1 || !xyz2 || !idx || !pts_cnt) return (int)cudaErrorInvalidValue;
    const float thr = pn2_ball_threshold(radius);
    if (!pn2_ball_group_fits(n) || thr < 0.0f || (long long)b * num_sms() > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    // several CTAs per cloud until the machine is full (each builds its own copy of the grid: the
    // build is ~n/1024 shared-memory atomics per thread) — but never more than the queries can feed
    const int sms = num_sms();
    int r = sms / (b < sms ? b : sms);
    const int rmax = (m + kBgWarps - 1) / kBgWarps;
    if (r > rmax) r = rmax;
    if (r < 1) r = 1;
    return launch_ball_group(b, n, m, radius, thr, nsample, xyz1, lengths, xyz2, nullptr, idx, pts_cnt, grouped_xyz, center, r, false,
                             false, st);
}

// pn2_sa_layer_msg_device on the clouds' first lengths[b] points (lengths == NULL: all n)
static int sa_layer_msg(int b, int n, int m, int nscales, const float* radii, const int* nsamples, const float* xyz,
                        const int* lengths, int* fps_idx, float* new_xyz, int* const* idx, int* const* pts_cnt,
                        float* const* grouped_xyz, int center, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || nscales <= 0 || nscales > kSaMaxScales || !radii || !nsamples || !idx || !pts_cnt)
        return (int)cudaErrorInvalidValue;
    for (int k = 0; k < nscales; ++k)
        if (nsamples[k] <= 0 || !(radii[k] > 0.0f) || !idx[k] || !pts_cnt[k]) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz || !fps_idx || !new_xyz) return (int)cudaErrorInvalidValue;
    bool overlapped = fps_single_cta(b, n) && pn2_ball_group_fits(n);
    for (int k = 0; k < nscales; ++k) overlapped = overlapped && pn2_ball_threshold(radii[k]) >= 0.0f;
    if (overlapped) {
        // sampling (one CTA per cloud) + one dependent ball_group grid per scale, chained so that all of them
        // are resident while the sampling chain runs
        int rc = fps_dispatch(b, n, m, xyz, lengths, nullptr, fps_idx, new_xyz, /*sentinel=*/1, st);
        const int r = sa_consumer_ctas(b, nscales);
        for (int k = 0; k < nscales && rc == 0; ++k)
            rc = launch_ball_group(b, n, m, radii[k], pn2_ball_threshold(radii[k]), nsamples[k], xyz, lengths, nullptr, fps_idx, idx[k],
                                   pts_cnt[k], grouped_xyz ? grouped_xyz[k] : nullptr, center, r, true, k + 1 < nscales, st);
        return rc;
    }
    // sequential path (clustered / global-scratch sampling, or clouds too large for the in-smem grid); every index the
    // sampling and the ball query return is below the cloud's length, so the grouping needs no lengths
    const size_t fps_b = align256(pn2_fps_scratch_bytes(b, n)), bq_b = pn2_query_ball_point_workspace_bytes(b, n);
    char* ws = static_cast<char*>(workspace);
    float* temp = nullptr;
    void* bq_ws = nullptr;
    if (fps_b) {
        if (!ws || workspace_bytes < fps_b) return (int)cudaErrorInvalidValue;
        temp = reinterpret_cast<float*>(ws);
    }
    if (bq_b && ws && workspace_bytes >= fps_b + bq_b) bq_ws = ws + fps_b;
    void* stream = static_cast<void*>(st);
    int rc = fps_dispatch(b, n, m, xyz, lengths, temp, fps_idx, new_xyz, 0, st);
    for (int k = 0; k < nscales && rc == 0; ++k) {
        rc = query_ball_point_ws(b, n, m, radii[k], nsamples[k], xyz, lengths, new_xyz, idx[k], pts_cnt[k], bq_ws, bq_ws ? bq_b : 0, st);
        float* g = grouped_xyz ? grouped_xyz[k] : nullptr;
        if (rc || !g) continue;
        rc = center ? pn2_group_concat(b, n, 0, m, nsamples[k], xyz, new_xyz, nullptr, idx[k], 1, g, nullptr, stream)
                    : pn2_group_point(b, n, 3, m, nsamples[k], xyz, idx[k], g, stream);
    }
    return rc;
}


// ================================================================================================
// kNN grouping overlapped with the sampling chain: pn2_sa_knn_layer_device.
//
// knn_group_kernel<KC> (k <= 32 * KC) has ctas_per_cloud CTAs per cloud.  Each copies its cloud (n points, SoA) into
// shared memory once; warp gw of the cloud's CTAs then serves centroids gw, gw + stride, ...: it polls fps_idx as
// ball_group_kernel does, reads the centroid's coordinates from the copy (the floats gather_point writes into
// new_xyz), and runs knn_point's per-query routine (knn_warp.cuh) over the whole cloud in one offer.  The results are
// knn_point's bit for bit; grouped_xyz is the gather of the result row, raw or centred with one __fsub_rn per
// coordinate as group_point(xyz, idx) - new_xyz computes it.
//
// Shared memory: 12 n bytes of cloud + 24 k bytes of W buffers per warp (2k entries of value, original index and
// current position).  The warp count per CTA follows from what the cloud leaves, up to 32: 32 warps up to k = 64 at
// n = 8192, fewer for larger clouds; below kKgMinWarps the layer takes the sequential path.
//
// Ragged batches (L): cloud i is its first len_i = cloud_length(lengths, i, n) points.  Only those are copied into
// shared memory (the SoA stride stays n), a centroid index >= len_i is flagged like a lost one, and a cloud shorter than
// k runs KnnWarp with k_i = min(k, len_i) and repeats column 0 in columns [k_i, k), as knn_kernel<KC, true> does.
// ================================================================================================
constexpr int kKgMinWarps = 4;
constexpr int kKgMaxWarps = 32;
// Largest k the overlapped layer takes.  Measured on the H100 (DESIGN.md §6.2.1): at k = 128 the consumer's per-query
// cost is 3.5x the sampling step's and the layer trailed the sequential ops (0.63 against 0.54 ms at 16 x 1024 -> 512),
// so k > 64 takes the sequential path.
constexpr int kKgMaxK = 64;
constexpr size_t kKgSmemMax = 200 * 1024;

__host__ __device__ inline size_t kg_cloud_bytes(int n) { return ((size_t)n * 12 + 15) / 16 * 16; }

// warps per consumer CTA for (n, k); 0 = the overlapped layer does not hold this shape
static int kg_warps(int n, int k) {
    if (n <= 0 || k <= 0 || k > kKgMaxK || k > n) return 0;
    const size_t cloud = kg_cloud_bytes(n);
    if (cloud >= kKgSmemMax) return 0;
    const size_t w = (kKgSmemMax - cloud) / ((size_t)24 * k);
    const int nw = w < (size_t)kKgMaxWarps ? (int)w : kKgMaxWarps;
    return nw >= kKgMinWarps ? nw : 0;
}

__device__ __forceinline__ void kg_load(const float* __restrict__ s_x, int n, int pos, float& x, float& y, float& z) {
    x = s_x[pos];
    y = s_x[n + pos];
    z = s_x[2 * n + pos];
}

template <int KC, bool L>  // L: per-cloud lengths (a template flag: the instances without them keep their code)
__global__ void __launch_bounds__(kKgMaxWarps * 32, 1)
knn_group_kernel(int n, int m, int k, const float* __restrict__ xyz, const int* q_idx, int* __restrict__ idx,
                 float* __restrict__ dist, float* __restrict__ grouped, int center, int ctas_per_cloud,
                 const int* __restrict__ lengths) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    float* __restrict__ s_x = reinterpret_cast<float*>(s_raw);  // [3][n]: x, then y, then z
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    float* __restrict__ wv = reinterpret_cast<float*>(s_raw + kg_cloud_bytes(n)) + (size_t)warp * 6 * k;
    int* __restrict__ wo = reinterpret_cast<int*>(wv + 2 * k);
    int* __restrict__ wp = wo + 2 * k;
    const int cloud = blockIdx.x / ctas_per_cloud, part = blockIdx.x - cloud * ctas_per_cloud;
    const float* __restrict__ pts = xyz + (size_t)cloud * n * 3;
    const int len = L ? cloud_length(lengths, cloud, n) : n;
    for (int p = tid; p < 3 * len; p += blockDim.x) {  // coalesced reads, transposed into SoA
        const int pt = p / 3, c = p - 3 * pt;
        s_x[c * n + pt] = __ldg(pts + p);
    }
    __syncthreads();

    const int qstride = ctas_per_cloud * nwarps;
    const long long t_start = clock64();
    for (int q = part * nwarps + warp; q < m; q += qstride) {
        // wait for the sampling kernel to publish centroid q (its index turns non-negative)
        int qi = 0;
        if (lane == 0) {
            const int* src = q_idx + (size_t)cloud * m + q;
            qi = ld_volatile_s32(src);
            unsigned backoff = 32;
            while (qi < 0) {
                __nanosleep(backoff);
                if (backoff < 256) backoff <<= 1;
                qi = ld_volatile_s32(src);
                if (clock64() - t_start > 4000000000ll) break;  // ~2 s: never hang the device on a lost producer
            }
        }
        qi = __shfl_sync(kFullMask, qi, 0);
        const size_t row = ((size_t)cloud * m + q) * k;
        int* __restrict__ orow = idx + row;
        if (qi < 0 || qi >= len) {  // producer lost / corrupt index: flag the row instead of faulting
            for (int e = lane; e < k; e += 32) orow[e] = -1;
            continue;
        }
        float qx, qy, qz;
        kg_load(s_x, n, qi, qx, qy, qz);
        const int kq = L ? min(k, len) : k;  // columns the selection produces for this cloud
        KnnWarp<KC> w(kq, lane, qx, qy, qz);
        for (int pos = lane; pos < kq; pos += 32) {
            float x, y, z;
            kg_load(s_x, n, pos, x, y, z);
            w.put_a(wv, wo, pos, x, y, z);
        }
        w.offer(s_x, s_x + n, s_x + 2 * n, len, 0);
        float* __restrict__ drow = dist ? dist + row : nullptr;
        w.finish(wv, wo, wp, kq, [&](int e, float v, int i) {
            orow[e] = i;
            if (drow) drow[e] = v;
        });
        if (L && kq < k) {  // a cloud shorter than k: columns [kq, k) repeat column 0
            __syncwarp();   // the replay's column 0 was written by lane 0
            const int i0 = orow[0];
            const float v0 = drow ? drow[0] : 0.f;
            for (int e = kq + lane; e < k; e += 32) {
                orow[e] = i0;
                if (drow) drow[e] = v0;
            }
        }
        if (grouped) {
            __syncwarp();  // the replay's columns (and the filler) were written by other lanes
            float* __restrict__ grow = grouped + row * 3;
            for (int e = lane; e < k; e += 32) {
                float x, y, z;
                kg_load(s_x, n, orow[e], x, y, z);
                // centred: xyz[idx] - new_xyz, one rounding per coordinate; a raw copy otherwise (x - 0 would
                // canonicalise a NaN payload, which a gather never does)
                grow[3 * e + 0] = center ? __fsub_rn(x, qx) : x;
                grow[3 * e + 1] = center ? __fsub_rn(y, qy) : y;
                grow[3 * e + 2] = center ? __fsub_rn(z, qz) : z;
            }
        }
        __syncwarp();  // W is reused by this warp's next query
    }
    // completion of this grid must imply completion of the sampling grid it overlaps (see ball_group_kernel)
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

static int launch_knn_group(int b, int n, int m, int k, const float* xyz, const int* lengths, const int* q_idx, int* idx,
                            float* dist, float* grouped, int center, int ctas_per_cloud, cudaStream_t st) {
    static std::atomic<long long> max_dyn_once[4][64];  // [ragged * 2 + KC instance][device]: 0 = not asked yet
    const int nw = kg_warps(n, k);
    if (nw == 0) return (int)cudaErrorInvalidValue;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev < 0 || dev >= 64) return (int)cudaErrorInvalidDevice;
    const int kc = (lengths ? 2 : 0) + (k <= 32 ? 0 : 1);
    auto kern = kc == 0 ? knn_group_kernel<1, false> : kc == 1 ? knn_group_kernel<2, false> : kc == 2 ? knn_group_kernel<1, true>
                                                                                                   : knn_group_kernel<2, true>;
    long long max_dyn = max_dyn_once[kc][dev].load(std::memory_order_acquire);
    if (max_dyn == 0) {
        int optin = 0;
        cudaFuncAttributes fa;
        e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, kern);
        if (e != cudaSuccess) return (int)e;
        max_dyn = (long long)optin - (long long)fa.sharedSizeBytes;
        if (max_dyn < (long long)kKgSmemMax) return (int)cudaErrorInvalidValue;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_dyn);
        if (e != cudaSuccess) return (int)e;
        max_dyn_once[kc][dev].store(max_dyn, std::memory_order_release);
    }
    // an SM to itself, as for the ball query: every byte of shared memory rules out co-residency with a sampling CTA
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)b * (unsigned)ctas_per_cloud, 1, 1);
    cfg.blockDim = dim3((unsigned)nw * 32, 1, 1);
    cfg.dynamicSmemBytes = (size_t)max_dyn;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    e = cudaLaunchKernelEx(&cfg, kern, n, m, k, xyz, q_idx, idx, dist, grouped, center, ctas_per_cloud, lengths);
    count_launch();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

// SMs the sampling chain leaves per cloud (b sampling CTAs, one SM each)
static int knn_room(int b) {
    const int sms = num_sms();
    return b < sms ? (sms - b) / b : 0;
}

// Consumer CTAs per cloud: every SM the sampling chain leaves, but no more CTAs than give each warp one centroid.
// pn2_set_sa_consumer_ctas overrides (0 = automatic), within the same bounds.
static int knn_consumer_ctas(int b, int m, int k, int n) {
    const int room = knn_room(b), nw = kg_warps(n, k);
    int r = g_sa_consumer_ctas.load(std::memory_order_relaxed);
    if (r <= 0) r = room;
    if (r > room) r = room;
    const int rmax = (m + nw - 1) / nw;
    if (r > rmax) r = rmax;
    return r < 1 ? 1 : r;
}

// pn2_set_sa_knn_path: 0 = the rule below, 1 = overlapped wherever it can run, 2 = sequential (measurement)
static std::atomic<int> g_sa_knn_path{0};

// Overlapped or sequential.  The overlapped layer can run when the sampling is one CTA per cloud, k <= 64, the cloud
// and the W buffers fit in shared memory (kg_warps) and at least one idle SM is left per cloud.  Whether it WINS is a
// cost comparison, in units of one sampling step t (the sampling takes m t either way).  Let C = c / t, c the SM time
// of one kNN query, r the consumer CTAs per cloud, nw their warps, S the SMs.  Each consumer warp serves
// ceil(m / (r nw)) centroids and nw warps share an SM, so the consumers need about ceil(m / (r nw)) nw C; the
// sequential ops need m for the sampling plus b m C / S for knn_point on every SM:
//     overlapped  <=>  ceil(m / (r nw)) nw C <= m + b m C / S.
// C was measured on the H100 (DESIGN.md §6.2.1: knn_point against the sampling kernel, uniform and duplicate-heavy
// clouds): up to 4.0 at k = 8, 8.2 at k = 32 and 16.6 at k = 64 for N 4096, 20.9 at k = 64 for N 1024.
// max(4, k (0.26 + 80 / n)) bounds those.  At N 4096 -> 1024 on 132 SMs it overlaps k = 32 for b <= 33 (3 or more
// consumer CTAs per cloud) and k = 64 for b <= 26.
static bool knn_overlapped(int b, int n, int m, int k) {
    const int mode = g_sa_knn_path.load(std::memory_order_relaxed);
    if (mode == 2 || kg_warps(n, k) == 0 || knn_room(b) < 1 || !fps_single_cta(b, n)) return false;
    if (mode == 1) return true;
    const double S = num_sms(), r = knn_consumer_ctas(b, m, k, n), nw = kg_warps(n, k);
    const double C = fmax(4.0, k * (0.26 + 80.0 / n));
    const double per_warp = ceil((double)m / (r * nw));
    return per_warp * nw * C <= (double)m + (double)b * m * C / S;
}

static size_t knn_val_bytes(int b, int m, int k) { return (size_t)b * (size_t)m * (size_t)k * sizeof(float); }

// pn2_sa_knn_layer_device on the clouds' first lengths[b] points (lengths == NULL: all n); the path and the workspace are
// chosen from (b, n, m, k) either way
static int sa_knn_layer(int b, int n, int m, int k, const float* xyz, const int* lengths, int* fps_idx, float* new_xyz, int* idx,
                        float* dist, float* grouped_xyz, int center, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || k <= 0 || k > kKnnMaxK || k > n) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz || !fps_idx || !new_xyz || !idx || b > 65535) return (int)cudaErrorInvalidValue;
    if (knn_overlapped(b, n, m, k)) {
        int rc = fps_dispatch(b, n, m, xyz, lengths, nullptr, fps_idx, new_xyz, /*sentinel=*/1, st);
        if (rc == 0)
            rc = launch_knn_group(b, n, m, k, xyz, lengths, fps_idx, idx, dist, grouped_xyz, center, knn_consumer_ctas(b, m, k, n), st);
        return rc;
    }
    // sequential path: the sampling, knn_point and the xyz grouping one after the other; every index the sampling and
    // knn_point return is below the cloud's length, so the grouping needs no lengths
    const size_t fps_b = align256(pn2_fps_scratch_bytes(b, n));
    char* ws = static_cast<char*>(workspace);
    float* temp = nullptr;
    float* val = dist;
    if (fps_b) {
        if (!ws || workspace_bytes < fps_b) return (int)cudaErrorInvalidValue;
        temp = reinterpret_cast<float*>(ws);
    }
    if (!val) {  // knn_point writes the distances somewhere
        if (!ws || workspace_bytes < fps_b + knn_val_bytes(b, m, k)) return (int)cudaErrorInvalidValue;
        val = reinterpret_cast<float*>(ws + fps_b);
    }
    void* stream = static_cast<void*>(st);
    int rc = fps_dispatch(b, n, m, xyz, lengths, temp, fps_idx, new_xyz, 0, st);
    if (rc == 0) rc = pn2_knn_point_ragged(b, n, m, k, xyz, lengths, new_xyz, nullptr, val, idx, stream);
    if (rc == 0 && grouped_xyz)
        rc = center ? pn2_group_concat(b, n, 0, m, k, xyz, new_xyz, nullptr, idx, 1, grouped_xyz, nullptr, stream)
                    : pn2_group_point(b, n, 3, m, k, xyz, idx, grouped_xyz, stream);
    return rc;
}

}  // namespace pn2

extern "C" {

int pn2_ball_group_fits(int n) {
    return (n > 0 && n < (1 << pn2::kBgPosBits) && pn2::bg_smem_bytes(n) <= pn2::kBgSmemMax) ? 1 : 0;
}

int pn2_ball_group(int b, int n, int m, float radius, int nsample, const float* xyz1, const float* xyz2, int* idx,
                   int* pts_cnt, float* grouped_xyz, int center, void* stream) {
    return pn2::ball_group(b, n, m, radius, nsample, xyz1, nullptr, xyz2, idx, pts_cnt, grouped_xyz, center, pn2::as_stream(stream));
}

size_t pn2_sa_layer_device_workspace_bytes(int b, int n, int m, int nsample) {
    if (b <= 0 || n <= 0 || m <= 0 || nsample <= 0) return 0;
    (void)m;
    (void)nsample;
    // sequential fallback only: FPS scratch for clouds beyond the cluster capacity + the uniform-grid scratch
    return pn2::align256(pn2_fps_scratch_bytes(b, n)) + pn2::align256(pn2_query_ball_point_workspace_bytes(b, n));
}

int pn2_sa_layer_msg_device(int b, int n, int m, int nscales, const float* radii, const int* nsamples, const float* xyz,
                            int* fps_idx, float* new_xyz, int* const* idx, int* const* pts_cnt, float* const* grouped_xyz,
                            int center, void* workspace, size_t workspace_bytes, void* stream) {
    return pn2::sa_layer_msg(b, n, m, nscales, radii, nsamples, xyz, nullptr, fps_idx, new_xyz, idx, pts_cnt, grouped_xyz, center,
                             workspace, workspace_bytes, pn2::as_stream(stream));
}

int pn2_sa_layer_msg_device_ragged(int b, int n, int m, int nscales, const float* radii, const int* nsamples, const float* xyz,
                                   const int* lengths, int* fps_idx, float* new_xyz, int* const* idx, int* const* pts_cnt,
                                   float* const* grouped_xyz, int center, void* workspace, size_t workspace_bytes, void* stream) {
    return pn2::sa_layer_msg(b, n, m, nscales, radii, nsamples, xyz, lengths, fps_idx, new_xyz, idx, pts_cnt, grouped_xyz, center,
                             workspace, workspace_bytes, pn2::as_stream(stream));
}

int pn2_sa_layer_device_ragged(int b, int n, int m, float radius, int nsample, const float* xyz, const int* lengths, int* fps_idx,
                               float* new_xyz, int* idx, int* pts_cnt, float* grouped_xyz, int center, void* workspace,
                               size_t workspace_bytes, void* stream) {
    if (!idx || !pts_cnt) return (int)cudaErrorInvalidValue;
    int* idxs[1] = {idx};
    int* cnts[1] = {pts_cnt};
    float* grps[1] = {grouped_xyz};
    return pn2_sa_layer_msg_device_ragged(b, n, m, 1, &radius, &nsample, xyz, lengths, fps_idx, new_xyz, idxs, cnts,
                                          grouped_xyz ? grps : nullptr, center, workspace, workspace_bytes, stream);
}

int pn2_sa_layer_device(int b, int n, int m, float radius, int nsample, const float* xyz, int* fps_idx, float* new_xyz,
                        int* idx, int* pts_cnt, float* grouped_xyz, int center, void* workspace, size_t workspace_bytes,
                        void* stream) {
    return pn2_sa_layer_device_ragged(b, n, m, radius, nsample, xyz, nullptr, fps_idx, new_xyz, idx, pts_cnt, grouped_xyz, center,
                                      workspace, workspace_bytes, stream);
}

int pn2_sa_knn_layer_fits(int n, int k) { return pn2::kg_warps(n, k) > 0 ? 1 : 0; }

size_t pn2_sa_knn_layer_workspace_bytes(int b, int n, int m, int k) {
    if (b <= 0 || n <= 0 || m <= 0 || k <= 0 || k > pn2::kKnnMaxK || k > n) return 0;
    // the overlapped path needs none; the sequential one FPS scratch for clouds beyond the cluster capacity +
    // knn_point's distances when the caller does not want them
    if (pn2::knn_overlapped(b, n, m, k)) return 0;
    return pn2::align256(pn2_fps_scratch_bytes(b, n)) + pn2::align256(pn2::knn_val_bytes(b, m, k));
}

int pn2_sa_knn_layer_device(int b, int n, int m, int k, const float* xyz, int* fps_idx, float* new_xyz, int* idx, float* dist,
                            float* grouped_xyz, int center, void* workspace, size_t workspace_bytes, void* stream) {
    return pn2::sa_knn_layer(b, n, m, k, xyz, nullptr, fps_idx, new_xyz, idx, dist, grouped_xyz, center, workspace, workspace_bytes,
                             pn2::as_stream(stream));
}

int pn2_sa_knn_layer_device_ragged(int b, int n, int m, int k, const float* xyz, const int* lengths, int* fps_idx, float* new_xyz,
                                   int* idx, float* dist, float* grouped_xyz, int center, void* workspace, size_t workspace_bytes,
                                   void* stream) {
    return pn2::sa_knn_layer(b, n, m, k, xyz, lengths, fps_idx, new_xyz, idx, dist, grouped_xyz, center, workspace, workspace_bytes,
                             pn2::as_stream(stream));
}

void pn2_set_sa_knn_path(int mode) { pn2::g_sa_knn_path.store(mode >= 0 && mode <= 2 ? mode : 0, std::memory_order_relaxed); }

void pn2_set_sa_consumer_ctas(int ctas_per_cloud) { pn2::g_sa_consumer_ctas.store(ctas_per_cloud, std::memory_order_relaxed); }

}  // extern "C"
