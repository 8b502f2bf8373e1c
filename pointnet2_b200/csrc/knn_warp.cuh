// knn_warp.cuh — the per-query work of knn_point, one warp per query, as the KnnWarp routine that both kNN kernels
// run: knn_kernel (knn.cu: the cloud staged through shared-memory tiles) and knn_group_kernel (sa_fused.cu: the whole
// cloud in shared memory, queries taken from a concurrently running sampling kernel).
//
// Semantics (see knn.cu for the derivation): the first k columns of the reference's selection sort over the row of
// squared distances, ties included.  Only set A (positions < k) and set B (the k smallest of the rest under
// (value, position)) can ever be selected or moved, so a query
//   1. fills A into its W buffer          (put_a for each position < min(k, n), from wherever the caller keeps the cloud),
//   2. offers the positions >= k to B     (offer: points [0, tn) of SoA arrays in shared memory at global position
//                                          base, once per tile or once for a cloud held whole),
//   3. replays the k rounds on A and B    (finish: sorted fast path, or the exact replay with current positions),
//      handing each result column to the caller's emit(column, value, index).
// W is per warp: W[0..k) = A, W[k..2k) = B; wv = value, wo = original index, wp = current position (replay only).
#pragma once
#include <math.h>

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kKnnMaxK = 128;

// Ascending bitonic sort of 32*E 64-bit keys held E per lane (element i = register i/32 of lane i%32; E a power of 2).
template <int E>
__device__ __forceinline__ void bitonic_sort_u64(unsigned long long (&key)[E], int lane) {
#pragma unroll
    for (int size = 2; size <= 32 * E; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            if (stride >= 32) {  // partner in the same lane, another register
                const int js = stride >> 5;
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    if ((j & js) == 0) {
                        const bool up = (((32 * j) & size) == 0);
                        const unsigned long long x = key[j], y = key[j | js];
                        const bool sw = up ? (x > y) : (x < y);
                        key[j] = sw ? y : x;
                        key[j | js] = sw ? x : y;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    const int i = 32 * j + lane;
                    const unsigned long long other = __shfl_xor_sync(kFullMask, key[j], stride);
                    const bool up = ((i & size) == 0), lower = ((lane & stride) == 0);
                    const bool keep_min = (up == lower);  // the lower element of an ascending pair keeps the minimum
                    key[j] = (keep_min == (other < key[j])) ? other : key[j];
                }
            }
        }
    }
}

__device__ __forceinline__ float knn_dist(float x, float y, float z, float qx, float qy, float qz) {
    const float dx = __fsub_rn(x, qx), dy = __fsub_rn(y, qy), dz = __fsub_rn(z, qz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

template <int KC>  // registers per lane that hold the list B: k <= 32 * KC
struct KnnWarp {
    const int k, lane;
    const float qx, qy, qz;
    // the list B lives in REGISTERS while the row is scanned: entry e = register e/32 of lane e%32 (no shared memory,
    // no __syncwarp): round 2's first version kept a sorted B in shared memory and spent most of its time in the
    // read-sync-write shifts (1.02 ms at 32 x 1024 x 4096, k = 32).
    float bv[KC];
    int bo[KC];
    int nb = 0;            // |B| so far (<= k)
    float tau = INFINITY;  // B full: its largest value; a later position must be strictly smaller to enter
    int ev_pos = -1;       // B's current maximum under (value, position) — the entry a better candidate evicts

    __device__ __forceinline__ KnnWarp(int k_, int lane_, float qx_, float qy_, float qz_)
        : k(k_), lane(lane_), qx(qx_), qy(qy_), qz(qz_) {
#pragma unroll
        for (int c = 0; c < KC; ++c) {
            bv[c] = INFINITY;
            bo[c] = 0;
        }
    }

    // set A: position pos < min(k, n) keeps its own slot; (x, y, z) is data point pos.  The caller loops over the
    // positions: handed a loader callable instead, the front end re-associated knn_kernel's 64-bit address arithmetic
    // (a separate base per coordinate in the tile loads too) and ptxas took 48 / 40 + 8 bytes of spill / 64 registers.
    __device__ __forceinline__ void put_a(float* __restrict__ wv, int* __restrict__ wo, int pos, float x, float y, float z) const {
        wv[pos] = knn_dist(x, y, z, qx, qy, qz);
        wo[pos] = pos;
    }

    // candidates for B among the points [0, tn) of s_x / s_y / s_z, which sit at global positions base + p: those at
    // positions >= k that beat the current k-th best (strictly, once B is full).  Positions must be offered in
    // ascending order across calls.  ncu (k = 32, n = 4096): the kernel is issue-bound (91 % issue-active) and this
    // loop was 27 % of its instructions at 44 per 32 points — now two groups per trip and nothing about set A inside.
    //
    // nb, tau and ev_pos are copied into locals for the call.  Updated through `this` inside the loop, tau became an
    // integer and the eviction below a different chain of selects, and knn_kernel<2> took 43 registers instead of 40.
    __device__ __forceinline__ void offer(const float* __restrict__ s_x, const float* __restrict__ s_y,
                                          const float* __restrict__ s_z, int tn, int base) {
        int nb = this->nb;
        float tau = this->tau;
        int ev_pos = this->ev_pos;
        // B's maximum: ev_pos and tau
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
        this->nb = nb;
        this->tau = tau;
        this->ev_pos = ev_pos;
    }

    // ---- phase 2: replay the selection sort on W = A ∪ B; emit(column, value, index) for columns 0..ka-1 ----------
    template <class Emit>
    __device__ __forceinline__ void finish(float* __restrict__ wv, int* __restrict__ wo, int* __restrict__ wp, int ka, Emit emit) {
#pragma unroll
        for (int c = 0; c < KC; ++c) {
            if (32 * c + lane < nb) {
                wv[k + 32 * c + lane] = bv[c];
                wo[k + 32 * c + lane] = bo[c];
            }
        }
        __syncwarp();

        const int nw = k + nb;  // slots [ka, k) are empty when n < k (then nb == 0)
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
                    if (e < k) emit(e, __uint_as_float((unsigned)(key[j] >> 32)), (int)(unsigned)key[j]);
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
                        emit(s, bestv, wo[beste]);
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
                emit(s, bestv, wo[beste]);
            }
            __syncwarp();
        }
    }
};

}  // namespace pn2
