// knn.cu — knn_point for sm_90a: tiled brute-force top-k without the (b,m,n) distance matrix.
//
// Replaces the reference's composite (tf_ops/grouping/tf_grouping.py:48-73):
//   dist = reduce_sum((tile(xyz1) - tile(xyz2))**2, -1)          # (b,m,n) matrix in HBM
//   outi, out = select_top_k(k, dist)                            # selection_sort_gpu, tf_grouping_g.cu:83-123
//   idx, val = slice(outi, k), slice(out, k)
// which at (32, 1024, 4096) materialises 1.6 GB of differences, a 537 MB matrix and two more
// (b,m,n) outputs, and runs k rounds of selection sort over whole rows.
//
// Semantics kept bit for bit — including ties, which duplicate-heavy clouds produce all the time:
//   * distance = ((dx*dx + dy*dy) + dz*dz), every product and sum rounded on its own (element-wise
//     square, then a 3-term sum, as the graph computes it);
//   * selection sort does k rounds of "first minimum of v[s..n) by strict '<', SWAP it into place s".
//     The swap moves the element that sat at s to the winner's old position, so ties are NOT simply
//     broken by original index.  Only two kinds of elements can ever move or be selected: the k
//     elements that start at positions < k (set A) and the k smallest of the rest under
//     (value, position) (set B) — every other element keeps its position and always loses to an
//     unselected member of B.  So the kernel (1) scans the row once, keeping A in shared memory and
//     a top-k list B in registers (one entry per lane and register, unsorted: an insertion is a few
//     ballots and shuffles), then (2) replays the k rounds on those <= 2k elements with their
//     current positions.  The result equals the first k columns of selection_sort_gpu exactly.
//
// One warp per query; the data points of the query's cloud are staged through shared-memory tiles
// shared by the CTA's 8 warps (coordinates as SoA: consecutive lanes read consecutive words).
//
// knn_warp.cuh holds the same per-query algorithm as a KnnWarp routine for the overlapped kNN set-abstraction layer
// (sa_fused.cu), and the distance and the sort this kernel uses.  This kernel keeps its own inline copy of the
// scan and the replay: built on KnnWarp it returned the same bits but ran 4-18 % slower on the H100
// (32 x 1024 queries x 4096 points, k = 8..128: ptxas needed up to 16 more registers), so a change to
// either copy must be made to both (test_parity_gpu.py and test_knn_layer_gpu.py pin both to the oracle).
#include "knn_warp.cuh"

namespace pn2 {

constexpr int kKnnThreads = 256;
constexpr int kKnnWarps = kKnnThreads / 32;
constexpr int kKnnTile = 1024;  // data points per shared-memory tile

template <int KC>  // registers per lane that hold the list B: k <= 32 * KC
__global__ void __launch_bounds__(kKnnThreads)
knn_kernel(int n, int m, int k, const float* __restrict__ xyz1, const float* __restrict__ xyz2, float* __restrict__ val,
           int* __restrict__ idx) {
    __shared__ float s_x[kKnnTile], s_y[kKnnTile], s_z[kKnnTile];
    // per warp: W[0..k) = set A (positions 0..k-1), W[k..2k) = set B (in no particular order)
    __shared__ float s_wv[kKnnWarps][2 * kKnnMaxK];
    __shared__ int s_wo[kKnnWarps][2 * kKnnMaxK];  // original index
    __shared__ int s_wp[kKnnWarps][2 * kKnnMaxK];  // current position (phase 2)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.y;
    const int q = blockIdx.x * kKnnWarps + warp;
    const bool valid = q < m;
    const float* __restrict__ data = xyz1 + (size_t)cloud * n * 3;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (valid) {
        const float* qp = xyz2 + ((size_t)cloud * m + q) * 3;
        qx = __ldg(qp);
        qy = __ldg(qp + 1);
        qz = __ldg(qp + 2);
    }
    float* __restrict__ wv = s_wv[warp];
    int* __restrict__ wo = s_wo[warp];
    int* __restrict__ wp = s_wp[warp];
    // the list B lives in REGISTERS while the row is scanned: entry e = register e/32 of lane e%32 (no shared memory,
    // no __syncwarp): round 2's first version kept a sorted B in shared memory and spent most of its time in the
    // read-sync-write shifts (1.02 ms at 32 x 1024 x 4096, k = 32).
    float bv[KC];
    int bo[KC];
#pragma unroll
    for (int c = 0; c < KC; ++c) {
        bv[c] = INFINITY;
        bo[c] = 0;
    }
    const int ka = min(k, n);       // |A|
    int nb = 0;                     // |B| so far (<= k)
    float tau = INFINITY;           // B full: its largest value; a later position must be strictly smaller to enter

    // set A: positions 0..k-1 keep their own slot (straight from global memory: at most 128 points)
    if (valid)
        for (int pos = lane; pos < ka; pos += 32) {
            const float* s = data + (size_t)pos * 3;
            wv[pos] = knn_dist(__ldg(s), __ldg(s + 1), __ldg(s + 2), qx, qy, qz);
            wo[pos] = pos;
        }

    // B's current maximum under (value, position) — the entry a better candidate evicts — and tau, its value
    int ev_pos = -1;
    auto find_max = [&]() {
        unsigned loc = 0u;  // distances are non-negative and never NaN here: unsigned order of the bits == float order
#pragma unroll
        for (int c = 0; c < KC; ++c)
            if (32 * c + lane < k) loc = max(loc, __float_as_uint(bv[c]));
        const unsigned mx = __reduce_max_sync(kFullMask, loc);
        int lp = -1;
#pragma unroll
        for (int c = 0; c < KC; ++c)
            if (32 * c + lane < k && __float_as_uint(bv[c]) == mx) lp = max(lp, bo[c]);
        ev_pos = __reduce_max_sync(kFullMask, lp);  // among equal values the latest position goes first
        tau = __uint_as_float(mx);
    };
    // one candidate group (32 consecutive positions, ascending): offer every lane of `cand` to the list.  B is kept
    // UNSORTED (phase 2 sorts W anyway): while it is open a candidate is appended, afterwards it replaces the current
    // maximum, and two redux.sync find the next one — ~20 instructions whatever k is (the sorted list this replaces
    // shifted KC registers per insertion: 35 instructions at k <= 32, ~70 at k = 128, 35 % of the kernel at k = 32).
    auto insert_group = [&](unsigned cand, float d, int pos0) {
        while (cand) {  // ascending position
            const int src = __ffs(cand) - 1;
            cand &= cand - 1;
            const float dv = __shfl_sync(kFullMask, d, src);
            const int dpos = pos0 + src;
            if (nb < k) {
#pragma unroll
                for (int c = 0; c < KC; ++c)
                    if (32 * c + lane == nb) {
                        bv[c] = dv;
                        bo[c] = dpos;
                    }
                if (++nb == k) find_max();
            } else if (dv < tau) {  // tau may have dropped since the ballot (warp-uniform)
#pragma unroll
                for (int c = 0; c < KC; ++c)
                    if (bo[c] == ev_pos && 32 * c + lane < k) {
                        bv[c] = dv;
                        bo[c] = dpos;
                    }
                find_max();
            }
        }
    };

    // candidates for B: positions >= k that beat the current k-th best (strictly, once B is full).  ncu (k = 32,
    // n = 4096): the kernel is issue-bound (91 % issue-active) and this loop was 27 % of its instructions at 44 per
    // 32 points — now two groups per trip and nothing about set A inside.
    for (int base = 0; base < n; base += kKnnTile) {
        const int tn = min(kKnnTile, n - base);
        __syncthreads();  // previous tile consumed
        for (int p = tid; p < tn; p += kKnnThreads) {
            const float* s = data + (size_t)(base + p) * 3;
            s_x[p] = __ldg(s);
            s_y[p] = __ldg(s + 1);
            s_z[p] = __ldg(s + 2);
        }
        __syncthreads();
        if (!valid) continue;
        for (int p0 = max(0, k - base); p0 < tn; p0 += 64) {
            const int pa = p0 + lane, pb = pa + 32;
            float d0 = INFINITY, d1 = INFINITY;
            if (pa < tn) d0 = knn_dist(s_x[pa], s_y[pa], s_z[pa], qx, qy, qz);
            if (pb < tn) d1 = knn_dist(s_x[pb], s_y[pb], s_z[pb], qx, qy, qz);
            const bool open = nb < k;
            // a NaN distance beyond position k-1 is never "less than" anything: the selection sort cannot pick it
            const unsigned c0 = __ballot_sync(kFullMask, pa < tn && (open ? d0 == d0 : d0 < tau));
            const unsigned c1 = __ballot_sync(kFullMask, pb < tn && (open ? d1 == d1 : d1 < tau));
            if (c0) insert_group(c0, d0, base + p0);
            if (c1) insert_group(c1, d1, base + p0 + 32);  // insert_group re-checks every candidate against the current tau
        }
    }
    if (!valid) return;
#pragma unroll
    for (int c = 0; c < KC; ++c) {
        if (32 * c + lane < nb) {
            wv[k + 32 * c + lane] = bv[c];
            wo[k + 32 * c + lane] = bo[c];
        }
    }
    __syncwarp();

    // ---- phase 2: replay the selection sort on W = A ∪ B -------------------------------------------
    const int nw = k + nb;  // slots [ka, k) are empty when n < k (then nb == 0)
    float* __restrict__ oval = val + ((size_t)cloud * m + q) * k;
    int* __restrict__ oidx = idx + ((size_t)cloud * m + q) * k;
    // Fast path (ncu: the k-round replay below was 28 % of the kernel's instructions).  Sort W by value once.  If the
    // k + 1 smallest values of W are finite and pairwise different, every round of the selection sort has a unique
    // minimum — the next value in sorted order, wherever the swaps have moved it — so the sorted prefix IS the
    // result.  Any tie (or inf / NaN distance) among them takes the exact replay.
    if (ka == k) {
        constexpr int E = 2 * KC;
        unsigned long long key[E];
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const int e = 32 * j + lane;
            key[j] = e < nw ? (((unsigned long long)__float_as_uint(wv[e]) << 32) | (unsigned)wo[e]) : ~0ull;
        }
        bitonic_sort_u64<E>(key, lane);
        bool bad = false;
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const int e = 32 * j + lane;
            const unsigned hi = (unsigned)(key[j] >> 32);
            unsigned nxt = __shfl_down_sync(kFullMask, hi, 1);
            if (j + 1 < E) {
                const unsigned first_of_next = __shfl_sync(kFullMask, (unsigned)(key[(j + 1 < E) ? j + 1 : j] >> 32), 0);
                if (lane == 31) nxt = first_of_next;
            } else if (lane == 31) {
                nxt = 0xffffffffu;
            }
            if (e < k && (hi >= 0x7f800000u || (e + 1 < nw && hi == nxt))) bad = true;
            if (e < nw && (hi & 0x7fffffffu) > 0x7f800000u) bad = true;  // a NaN anywhere in W is selected by POSITION (v[s] starts as the minimum)
        }
        if (!__any_sync(kFullMask, bad)) {
#pragma unroll
            for (int j = 0; j < E; ++j) {
                const int e = 32 * j + lane;
                if (e < k) {
                    oval[e] = __uint_as_float((unsigned)(key[j] >> 32));
                    oidx[e] = (int)(unsigned)key[j];
                }
            }
            return;
        }
    }
    for (int e = lane; e < nw; e += 32) wp[e] = (e < ka || e >= k) ? wo[e] : 0x7fffffff;
    if (ka < k)
        for (int e = ka + lane; e < k; e += 32) wv[e] = INFINITY;
    __syncwarp();
    for (int s = 0; s < ka; ++s) {
        // first minimum over the elements at positions >= s, by (value, current position).  The reference starts
        // from min = v[s] and replaces it by strict '<' (tf_grouping_g.cu:98-108): a NaN sitting AT position s is
        // never replaced, a NaN anywhere else is never taken.
        float bestv = INFINITY;
        int bestp = 0x7fffffff, beste = -1;
        for (int e = lane; e < nw; e += 32) {
            const int pe = wp[e];
            const float ve = wv[e];
            const bool nan_at_s = (pe == s) && (ve != ve);
            const bool usable = (ve == ve) || nan_at_s;
            if (pe >= s && pe != 0x7fffffff && usable && (beste < 0 || nan_at_s || ve < bestv || (ve == bestv && pe < bestp))) {
                bestv = ve;
                bestp = pe;
                beste = e;
            }
        }
        {   // a NaN at position s wins outright
            const unsigned nan_lanes = __ballot_sync(kFullMask, beste >= 0 && bestp == s && bestv != bestv);
            if (nan_lanes) {
                const int src = __ffs(nan_lanes) - 1;
                bestv = __shfl_sync(kFullMask, bestv, src);
                bestp = s;
                beste = __shfl_sync(kFullMask, beste, src);
                if (lane == 0) {
                    wp[beste] = s;
                    oval[s] = bestv;
                    oidx[s] = wo[beste];
                }
                __syncwarp();
                continue;
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float ov = __shfl_xor_sync(kFullMask, bestv, off);
            const int op = __shfl_xor_sync(kFullMask, bestp, off);
            const int oe = __shfl_xor_sync(kFullMask, beste, off);
            const bool take = (oe >= 0) && (beste < 0 || ov < bestv || (ov == bestv && op < bestp));
            if (take) {
                bestv = ov;
                bestp = op;
                beste = oe;
            }
        }
        // swap: the element sitting at position s moves to the winner's old position
        if (bestp != s) {
            for (int e = lane; e < nw; e += 32)
                if (wp[e] == s) wp[e] = bestp;
            __syncwarp();
        }
        if (lane == 0) {
            wp[beste] = s;
            oval[s] = bestv;
            oidx[s] = wo[beste];
        }
        __syncwarp();
    }
}

}  // namespace pn2

extern "C" {

int pn2_knn_point(int b, int n, int m, int k, const float* xyz1, const float* xyz2, float* val, int* idx, void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || m < 0 || k <= 0 || k > kKnnMaxK || k > n) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz1 || !xyz2 || !val || !idx || b > 65535) return (int)cudaErrorInvalidValue;
    dim3 grid((m + kKnnWarps - 1) / kKnnWarps, b, 1);
    if (k <= 32) knn_kernel<1><<<grid, kKnnThreads, 0, as_stream(stream)>>>(n, m, k, xyz1, xyz2, val, idx);
    else if (k <= 64) knn_kernel<2><<<grid, kKnnThreads, 0, as_stream(stream)>>>(n, m, k, xyz1, xyz2, val, idx);
    else knn_kernel<4><<<grid, kKnnThreads, 0, as_stream(stream)>>>(n, m, k, xyz1, xyz2, val, idx);
    return finish_launch();
}

}  // extern "C"
