// pn2_common.cuh — shared device/host helpers for libpn2_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <atomic>

#include "pn2_api.h"

namespace pn2 {

constexpr unsigned kFullMask = 0xffffffffu;

// SMs of the current device (cudaDevAttrMultiProcessorCount, asked once per device): grid sizes and the
// split of SMs between concurrent kernels are planned for it.  Without a device (host-only planning
// queries) the H100 SXM's 132 is assumed.
inline int num_sms() {
    static std::atomic<int> cache[64];  // 0 = not asked yet
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        (void)cudaGetLastError();
        return 132;
    }
    int v = cache[dev].load(std::memory_order_relaxed);
    if (v > 0) return v;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) {
        (void)cudaGetLastError();
        return 132;
    }
    cache[dev].store(v, std::memory_order_relaxed);
    return v;
}

// ---- launch accounting (pn2_launch_count) --------------------------------------------------
extern unsigned long long g_launch_count;
inline void count_launch(int k = 1) { __atomic_fetch_add(&g_launch_count, (unsigned long long)k, __ATOMIC_RELAXED); }

inline int finish_launch() {
    count_launch();
    return (int)cudaGetLastError();
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

inline unsigned ceil_div_u(unsigned long long a, unsigned long long b) { return (unsigned)((a + b - 1) / b); }

// CTAs for a grid-stride kernel over work_items items, per_block per CTA: one item per thread up to 64 CTAs per SM,
// then grid-stride.
inline unsigned grid_for(unsigned long long work_items, unsigned per_block) {
    unsigned long long blocks = (work_items + per_block - 1) / per_block;
    const unsigned long long cap = (unsigned long long)num_sms() * 64;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

// cudaFuncSetAttribute once per (kernel instantiation, device), not on every launch
struct AttrOnce {
    std::atomic<unsigned long long> done{0ull};  // bit d: attributes set on device d (< 64)
};
template <typename K>
cudaError_t ensure_attrs(AttrOnce& once, K kern, size_t dyn, bool nonportable_cluster) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const unsigned long long bit = 1ull << (dev & 63);
    if (dev < 64 && (once.done.load(std::memory_order_acquire) & bit)) return cudaSuccess;
    if (dyn > 40 * 1024) {  // static + dynamic beyond the 48 KB default needs the opt-in
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
        if (e != cudaSuccess) return e;
    }
    if (nonportable_cluster) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        if (e != cudaSuccess) return e;
    }
    if (dev < 64) once.done.fetch_or(bit, std::memory_order_release);
    return cudaSuccess;
}

// ---- arithmetic contracts --------------------------------------------------------------------
// Squared distance exactly as nvcc contracts the reference's FPS and ball-query source
// (tf_sampling_g.cu:142, tf_grouping_g.cu:24; SASS: FMUL dy*dy, FFMA dx, FFMA dz).  Written with
// explicit round-to-nearest intrinsics so no compiler version or surrounding code can change it.
__device__ __forceinline__ float d2_fma_pattern(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// Squared distance exactly as x86-64 g++ -O2 (no FMA) evaluates threenn_cpu's expression
// (tf_interpolate.cpp:73): ((dx*dx + dy*dy) + dz*dz), each operation rounded on its own.
__device__ __forceinline__ float d2_nofma(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// ---- FP32 pairs: two points per helper call, each half rounded to nearest on its own, so bit-identical to the scalar
// expressions on either half.  sm_90 has no packed FP32x2 instructions: every helper issues two scalar FADD / FMUL /
// FFMA (the explicit .rn operations are never contracted) ---------------------------------------------------------
__device__ __forceinline__ unsigned long long f2_pack(float a, float b) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ void f2_unpack(unsigned long long v, float& a, float& b) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
__device__ __forceinline__ unsigned long long f2_sub(unsigned long long a, unsigned long long b) {
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    return f2_pack(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ unsigned long long f2_mul(unsigned long long a, unsigned long long b) {
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    return f2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ unsigned long long f2_fma(unsigned long long a, unsigned long long b, unsigned long long c) {
    float a0, a1, b0, b1, c0, c1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    f2_unpack(c, c0, c1);
    return f2_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

// ---- inverse-distance interpolation of three neighbours (three_interpolate, the FP front ends) --------------------
// ((p1*w1 + p2*w2) + p3*w3), every operation rounded on its own: the reference's x86 arithmetic
__device__ __forceinline__ float interp3(float p1, float p2, float p3, float w1, float w2, float w3) {
    return __fadd_rn(__fadd_rn(__fmul_rn(p1, w1), __fmul_rn(p2, w2)), __fmul_rn(p3, w3));
}

// ---- per-cloud lengths -----------------------------------------------------------------------
// Points of cloud `cloud` in a padded (b, n, 3) batch: lengths[cloud] clamped to [1, n] (a value out of range can
// never make a kernel read outside its row), or n when the batch has no lengths (lengths == NULL).  n stays the
// row stride; rows k >= the length are padding that no kernel reads.
__device__ __forceinline__ int cloud_length(const int* __restrict__ lengths, int cloud, int n) {
    return lengths ? min(max(__ldg(lengths + cloud), 1), n) : n;
}

// ---- warp helpers ----------------------------------------------------------------------------
// Batch-level rule of the uniform-grid ball query, evaluated identically by the grid kernel and by
// the brute-force kernel (each warp on its own, no barrier): the two kernels run back to back on one
// stream, so splitting a batch between them only pays when the grid serves a fair share of it
// (measured: 10 of 32 clouds pays, 2 of 32 costs 20 us).  `flags` is
// the per-cloud flag word written by bq_grid_build_kernel, one every `stride` ints; batches larger
// than 1024 clouds are judged on their first 1024.
__device__ __forceinline__ bool batch_uses_grid(const int* __restrict__ flags, size_t stride, int b) {
    const int lane = threadIdx.x & 31;
    const int bb = b < 1024 ? b : 1024;
    int cnt = 0;
    for (int c = lane; c < bb; c += 32) cnt += (__ldg(flags + (size_t)c * stride) != 0) ? 1 : 0;
    cnt = __reduce_add_sync(kFullMask, cnt);
    return 4 * cnt >= bb;
}

__device__ __forceinline__ unsigned warp_max_u32(unsigned v) { return __reduce_max_sync(kFullMask, v); }

// Lexicographic max of (hi, lo) pairs over the warp; every lane gets the result.
__device__ __forceinline__ void warp_max_pair(unsigned& hi, unsigned& lo) {
    const unsigned mh = warp_max_u32(hi);
    const unsigned ml = warp_max_u32(hi == mh ? lo : 0u);
    hi = mh;
    lo = ml;
}

// float min / max over the warp; every lane gets the result
__device__ __forceinline__ float warp_min_f32(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(kFullMask, v, o));
    return v;
}
__device__ __forceinline__ float warp_max_f32(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFullMask, v, o));
    return v;
}

// Exclusive prefix sum over a 1024-thread CTA: thread t gets the sum of v over threads 0..t-1.  Every thread must
// call it; s_w is 32 ints of shared scratch, written before the one __syncthreads inside and read after it, so a
// second call needs a barrier in between.
__device__ __forceinline__ int cta_exclusive_sum_1024(int v, int* s_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(kFullMask, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    // exclusive prefix over the warp totals (every warp scans the 32 totals with shuffles)
    const int wv = s_w[lane];
    int winc = wv;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(kFullMask, winc, o);
        if (lane >= o) winc += t;
    }
    return __shfl_sync(kFullMask, winc - wv, warp) + incl - v;
}

// ---- counter-based random draws (DESIGN.md §6.10; crops.cu, shapes.cu, vscan.cu) ----------------------------------
// rng_draw(seed, stream, e, i) = mix(mix(mix(seed + stream*G) + e*G) + i*G) with mix = SplitMix64's finaliser, in
// uint64 wrap-around arithmetic; rng_unit maps a draw to a double in [0, 1).  tests/crop_oracle.py restates both.
constexpr unsigned long long kRngGolden = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ unsigned long long rng_mix64(unsigned long long x) {
    x ^= x >> 30;
    x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27;
    x *= 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x;
}

__device__ __forceinline__ unsigned long long rng_draw(unsigned long long seed, unsigned long long stream,
                                                       unsigned long long e, unsigned long long i) {
    return rng_mix64(rng_mix64(rng_mix64(seed + stream * kRngGolden) + e * kRngGolden) + i * kRngGolden);
}

__device__ __forceinline__ double rng_unit(unsigned long long d) { return (double)(d >> 11) * 0x1.0p-53; }

// A sampler call's seed: read on the device when seed_dev is non-null (a (1,) tensor rewritten between replays of a
// captured graph), else the launch argument.
__device__ __forceinline__ unsigned long long rng_seed(const long long* seed_dev, unsigned long long seed) {
    return seed_dev ? (unsigned long long)__ldg(seed_dev) : seed;
}

// (key, local row) of row j of entry e as one 64-bit value: the high half of its draw, then j.  Distinct for distinct
// j < 2^32, so sorting them is the entry's seeded row order.
__device__ __forceinline__ unsigned long long rng_row_key(unsigned long long seed, unsigned long long stream,
                                                          unsigned long long e, long long j) {
    return (rng_draw(seed, stream, e, (unsigned long long)j) >> 32 << 32) | (unsigned long long)j;
}

// ---- seeded row selection (crops.cu, shapes.cu, vscan.cu) ----------------------------------------------------------
// Entry b of a packed set: k = index[b] and its rows off .. off + ps - 1 (offsets[k] .. offsets[k + 1] - 1).  False for
// an index outside [0, s) or an empty member; the kernels turn that into an empty entry.
__device__ __forceinline__ bool set_entry(const long long* __restrict__ index, int b, int s,
                                          const long long* __restrict__ offsets, int& k, long long& off, long long& ps) {
    const long long v = __ldg(index + b);
    if (v < 0 || v >= s) return false;
    k = (int)v;
    off = __ldg(offsets + k);
    ps = __ldg(offsets + k + 1) - off;
    return ps > 0;
}

constexpr __host__ __device__ int pow2_at_least(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

constexpr int kSelectRadixBins = 2048;
constexpr int kSelectMaxRows = 16384;  // m of cta_select_sorted: its sort buffer is pow2 >= m x 8 B of shared memory

struct SelectScratch {  // shared memory of cta_select_sorted
    int hist[kSelectRadixBins];
    int w[32];
    int digit, before, cnt, n;
};

// The m smallest orders among the members of [0, n), sorted ascending into s_keys[0 .. m), by a 1024-thread CTA.
// member(j) says whether j is a member and order(j) gives its distinct 64-bit order; c is the number of members and
// c >= m.  s_keys holds pow2 >= m values.  When c > m a radix select first finds the m smallest: they are those whose
// top `bits` bits are <= prefix, found with digits of 11, 11, 10 bits over the high half of the orders, then over the
// low half, stopping as soon as the whole boundary bucket is taken.  Every order is recomputed on each pass, so
// nothing per member is stored.  Every thread must call it; it ends with a barrier.
template <typename Member, typename Order>
__device__ __forceinline__ void cta_select_sorted(long long n, int c, int m, Member&& member, Order&& order,
                                                  unsigned long long* s_keys, SelectScratch& s) {
    const int tid = threadIdx.x;
    unsigned long long prefix = ~0ull;
    int bits = 0;
    if (c > m) {
        prefix = 0;
        int need = m;
        for (int pass = 0; pass < 6; ++pass) {
            const int wd = pass % 3 == 2 ? 10 : 11, shift = 64 - bits - wd;
            for (int k = tid; k < kSelectRadixBins; k += blockDim.x) s.hist[k] = 0;
            __syncthreads();
            for (long long j = tid; j < n; j += blockDim.x) {
                if (!member(j)) continue;
                const unsigned long long v = order(j);
                if (bits && (v >> (64 - bits)) != prefix) continue;
                atomicAdd(&s.hist[(int)((v >> shift) & ((1ull << wd) - 1))], 1);
            }
            __syncthreads();
            const int h0 = s.hist[2 * tid], h1 = s.hist[2 * tid + 1];
            const int ex = cta_exclusive_sum_1024(h0 + h1, s.w);
            if (ex < need && need <= ex + h0) {
                s.digit = 2 * tid;
                s.before = ex;
                s.cnt = h0;
            } else if (ex + h0 < need && need <= ex + h0 + h1) {
                s.digit = 2 * tid + 1;
                s.before = ex + h0;
                s.cnt = h1;
            }
            __syncthreads();
            need -= s.before;
            prefix = (prefix << wd) | (unsigned long long)s.digit;
            bits += wd;
            const bool done = s.cnt == need;
            __syncthreads();  // digit / before / cnt and hist are rewritten by the next pass
            if (done) break;
        }
    }
    // gather the m selected orders (in any order: the sort below fixes it) and sort them ascending
    if (tid == 0) s.n = 0;
    __syncthreads();
    for (long long j = tid; j < n; j += blockDim.x) {
        if (!member(j)) continue;
        const unsigned long long v = order(j);
        if (bits && (v >> (64 - bits)) > prefix) continue;
        s_keys[atomicAdd(&s.n, 1)] = v;
    }
    __syncthreads();
    const int sort_n = pow2_at_least(m);
    for (int k = m + tid; k < sort_n; k += blockDim.x) s_keys[k] = ~0ull;
    __syncthreads();
    for (int k = 2; k <= sort_n; k <<= 1) {
        for (int h = k >> 1; h > 0; h >>= 1) {
            for (int i = tid; i < sort_n; i += blockDim.x) {
                const int p = i ^ h;
                if (p > i) {
                    const unsigned long long x = s_keys[i], y = s_keys[p];
                    if ((x > y) == ((i & k) == 0)) {
                        s_keys[i] = y;
                        s_keys[p] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// Ordered compaction of rows 0 .. m-1 by a 1024-thread CTA: write(r, q) for every row r with keep(r), q being the
// number of kept rows before r.  Returns the number kept, to every thread.  Every thread must call it with the same
// m; s_w is 32 ints of shared scratch (SelectScratch::w), free again on return.
template <typename Keep, typename Write>
__device__ __forceinline__ int cta_compact(int m, Keep&& keep, Write&& write, int* s_w) {
    int kept = 0;
    for (int base = 0; base < m; base += blockDim.x) {
        const int r = base + threadIdx.x;
        const int k = r < m && keep(r);
        const int ex = cta_exclusive_sum_1024(k, s_w);
        if (k) write(r, kept + ex);
        kept += __reduce_add_sync(kFullMask, s_w[threadIdx.x & 31]);  // the 32 warp totals: this pass's count
        __syncthreads();  // s_w is rewritten by the next pass
    }
    return kept;
}

// ---- uniform grid over one cloud, for the ball query (ball_query_grid.cu, sa_fused.cu) ---------------------------
constexpr int kGridMaxDim = 16;  // cells per axis

// Cell of coordinate x: monotone in x; clamped so that out-of-box (and NaN) queries map to the border cells -1, dim.
__device__ __forceinline__ int grid_cell(float x, float origin, float inv_h, int dim) {
    float f = floorf(__fmul_rn(__fsub_rn(x, origin), inv_h));
    f = fminf(fmaxf(f, -1.0f), (float)dim);
    return (int)f;
}

struct GridGeometry {
    float mn[3];    // origin: the box's minimum corner
    float ext[3];   // box extent per axis
    float h, inv_h; // cell edge
    bool finite_box;
    int dims[3], ncell;
    int nb;  // cells of the 3x3x3 neighbourhood that fit in the grid
};

// Bounding box of the n points pts[0 .. 3n) and the grid over it, computed by a 1024-thread CTA; every thread gets
// the result.  Every thread must call it; it contains one __syncthreads, and s_red (6 x 32 floats of shared scratch)
// must not be written again before another barrier.  before_barrier() runs just before that barrier (the caller zeroes
// its cell counters there, behind the latency of the box loads).
template <typename F>
__device__ __forceinline__ GridGeometry grid_geometry(const float* __restrict__ pts, int n, float radius, float (&s_red)[6][32],
                                                      F&& before_barrier) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    GridGeometry g;
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int k = tid; k < n; k += 1024) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = __ldg(pts + 3 * (size_t)k + c);
            mn[c] = fminf(mn[c], v);
            // a NaN coordinate (fminf/fmaxf would ignore it) must disable the grid: the reference counts a NaN point
            // as a hit in EVERY ball (fmaxf(NaN,1e-20f) < radius, tf_grouping_g.cu:24-25), which only an index-ordered
            // scan reproduces; an infinite box does that (finite_box below)
            mx[c] = (v == v) ? fmaxf(mx[c], v) : INFINITY;
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float a = warp_min_f32(mn[c]), b = warp_max_f32(mx[c]);
        if (lane == 0) {
            s_red[c][warp] = a;
            s_red[3 + c][warp] = b;
        }
    }
    before_barrier();
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        g.mn[c] = warp_min_f32(s_red[c][lane]);
        g.ext[c] = warp_max_f32(s_red[3 + c][lane]) - g.mn[c];
    }
    const float emax = fmaxf(fmaxf(g.ext[0], g.ext[1]), g.ext[2]);
    // cell edge: at least 1.01 * radius (any point within the radius of a query is then at most one cell away on
    // every axis, with margin for the rounding of the cell function), and large enough for kGridMaxDim cells to span
    // the box
    g.h = fmaxf(1.01f * radius, emax / (float)(kGridMaxDim - 1));
    g.finite_box = (emax >= 0.f) && (emax < 1e30f) && (g.h > 0.f) && (g.h < 1e30f);
    if (!g.finite_box) g.h = 1.0f;
    g.inv_h = 1.0f / g.h;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int d = g.finite_box ? (int)floorf(g.ext[c] * g.inv_h) + 1 : 1;
        g.dims[c] = min(max(d, 1), kGridMaxDim);
    }
    g.ncell = g.dims[0] * g.dims[1] * g.dims[2];
    g.nb = min(g.dims[0], 3) * min(g.dims[1], 3) * min(g.dims[2], 3);
    return g;
}

// Ascending bitonic sort of 32*K ints held K per lane (element i = register i/32 of lane i%32; K <= KMAX, a power of 2).
template <int K, int KMAX>
__device__ __forceinline__ void bitonic_sort_keys(int (&key)[KMAX], int lane) {
#pragma unroll
    for (int size = 2; size <= 32 * K; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            if (stride >= 32) {  // partner in the same lane, another register
                const int js = stride >> 5;
#pragma unroll
                for (int j = 0; j < K; ++j) {
                    if ((j & js) == 0) {
                        const bool up = (((32 * j) & size) == 0);  // lane bits are below 32 <= stride < size: direction depends on j only
                        const int a = key[j], b = key[j | js];
                        const bool sw = up ? (a > b) : (a < b);
                        key[j] = sw ? b : a;
                        key[j | js] = sw ? a : b;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < K; ++j) {
                    const int i = 32 * j + lane;
                    const int other = __shfl_xor_sync(kFullMask, key[j], stride);
                    const bool up = ((i & size) == 0), lower = ((lane & stride) == 0);
                    // the lower element of an ascending pair keeps the minimum
                    key[j] = (up == lower) ? min(key[j], other) : max(key[j], other);
                }
            }
        }
    }
}

// brute-force ball query launcher (ball_query.cu); clouds whose grid_params[cloud*grid_stride] != 0
// are skipped (they are served by the uniform-grid kernels of ball_query_grid.cu).  lengths (b,) of xyz1 or NULL.
int launch_ball_query_brute(int b, int n, int m, float thr, int nsample, const float* xyz1, const int* lengths,
                            const float* xyz2, int* idx, int* pts_cnt, const int* grid_params, int grid_stride,
                            cudaStream_t st);
// pn2_query_ball_point (ball_query.cu), pn2_query_ball_point_ws (ball_query_grid.cu) and pn2_ball_group (sa_fused.cu) with
// the lengths of xyz1 (NULL: every cloud has n points)
int query_ball_point_brute(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths,
                           const float* xyz2, int* idx, int* pts_cnt, cudaStream_t st);
int query_ball_point_ws(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths,
                        const float* xyz2, int* idx, int* pts_cnt, void* workspace, size_t workspace_bytes, cudaStream_t st);
int ball_group(int b, int n, int m, float radius, int nsample, const float* xyz1, const int* lengths, const float* xyz2, int* idx,
               int* pts_cnt, float* grouped_xyz, int center, cudaStream_t st);

// farthest point sampling dispatch (fps.cu), shared with the fused set-abstraction layer (sa_fused.cu).
// sentinel != 0: single-CTA plans only (ask fps_single_cta first) — the kernel pre-fills `out` with -1 and
// signals programmatic launch completion so that a dependent grid can consume the picks as they appear.
// lengths (b,) device int32 or NULL (see cloud_length); the plan is chosen from n either way.
int fps_dispatch(int b, int n, int m, const float* inp, const int* lengths, float* temp, int* out, float* new_xyz,
                 int sentinel, cudaStream_t st);
bool fps_single_cta(int b, int n);
size_t fps_scratch_bytes(int b, int n);

// ordered-sum scatter through an inverse index (scatter_det.cu), shared by three_interpolate's gradient and the
// group_point / gather_point gradients: dst[b, i, :] = sum over the entries e with idx[b, e] == i, e ascending, of
//   WEIGHTED:  src[b, e / 3, :] * weight[b, e]   (ne = 3n: three_interpolate, n source rows)
//   otherwise: src[b, e, :]                      (ne = n)
// in float32, rounded once to T (float; unsigned short: f16 != 0 float16, else bfloat16).  Every dst row is written (0
// if no entry points at it).  b clouds of ne entries over nt targets; workspace of inv_workspace_bytes(b, ne, nt)
// bytes; lengths (WEIGHTED only): (b,) device int32 of the n source rows, or NULL.  The arguments are checked by the
// caller.
size_t inv_workspace_bytes(int b, long long ne, int nt);
template <bool WEIGHTED, typename T>
int inv_scatter_det(int b, int n, int ne, int c, int nt, const T* src, const int* idx, const float* weight, const int* lengths,
                    T* dst, void* workspace, int f16, cudaStream_t st);

// ---- streaming memory ops ---------------------------------------------------------------------
__device__ __forceinline__ void st_stream_f4(float4* p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream_i4(int4* p, int4 v) { __stcs(p, v); }

// ---- feature element types (PN2_F32 / PN2_BF16 / PN2_F16) -------------------------------------
// Features may be float, bfloat16 or half; arithmetic is always float32.  Loads upcast exactly,
// stores round once to nearest even (the rounding torch's .to(dtype) uses).
__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }
template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ float from_f32<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }

// ---- maxima that keep NaN (torch's max does; fmaxf would drop it) ------------------------------
// float -> key with  a < b  <=>  key(a) < key(b)  as unsigned, every NaN the largest key; 0 is below every key.  The
// maximum of exact keys is exact, so it does not depend on the order or the grouping of the comparisons.
__device__ __forceinline__ unsigned max_key(float v) {
    if (v != v) return 0xffffffffu;
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Four consecutive elements as one vector: float4 (16 bytes) for float, uint2 (8 bytes) for 2-byte types.
template <typename T> struct Pack4 { using type = uint2; };
template <> struct Pack4<float> { using type = float4; };

__device__ __forceinline__ float lo16_f32(unsigned w, __nv_bfloat16) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float lo16_f32(unsigned w, __half) { return __half2float(__ushort_as_half((unsigned short)(w & 0xffffu))); }
// (the second argument only selects the element type)
__device__ __forceinline__ float4 unpack4(float4 v, float) { return v; }
template <typename T> __device__ __forceinline__ float4 unpack4(uint2 v, T t) {
    return make_float4(lo16_f32(v.x, t), lo16_f32(v.x >> 16, t), lo16_f32(v.y, t), lo16_f32(v.y >> 16, t));
}
template <typename T> __device__ __forceinline__ unsigned short bits16(float a) {
    const T x = from_f32<T>(a);
    return *reinterpret_cast<const unsigned short*>(&x);
}
__device__ __forceinline__ float4 pack4(float4 v, float) { return v; }
template <typename T> __device__ __forceinline__ uint2 pack4(float4 v, T) {
    return make_uint2((unsigned)bits16<T>(v.x) | ((unsigned)bits16<T>(v.y) << 16),
                      (unsigned)bits16<T>(v.z) | ((unsigned)bits16<T>(v.w) << 16));
}

// 4 elements at p (4 * sizeof(T)-byte aligned) upcast to float: read-only path / streaming read
template <typename T> __device__ __forceinline__ float4 ldg4(const T* p) {
    return unpack4(__ldg(reinterpret_cast<const typename Pack4<T>::type*>(p)), T());
}
template <typename T> __device__ __forceinline__ float4 ldcs4(const T* p) {
    return unpack4(__ldcs(reinterpret_cast<const typename Pack4<T>::type*>(p)), T());
}
template <typename T> __device__ __forceinline__ void st4(T* p, float4 v) {
    *reinterpret_cast<typename Pack4<T>::type*>(p) = pack4(v, T());
}

// 2-byte features whose format is a runtime flag (f16 != 0: float16, else bfloat16), held as their raw unsigned short bits:
// one instantiation serves both where the code around the conversions is large (the FP front end's 3-NN phase).
// The float overloads ignore the flag.
__device__ __forceinline__ float f32_of(float x, int) { return x; }
__device__ __forceinline__ float f32_of(unsigned short x, int f16) {
    return f16 ? __half2float(__ushort_as_half(x)) : __uint_as_float((unsigned)x << 16);
}
template <typename T> __device__ __forceinline__ T of_f32(float x, int f16);
template <> __device__ __forceinline__ float of_f32<float>(float x, int) { return x; }
template <> __device__ __forceinline__ unsigned short of_f32<unsigned short>(float x, int f16) {
    return f16 ? __half_as_ushort(__float2half_rn(x)) : __bfloat16_as_ushort(__float2bfloat16_rn(x));
}
__device__ __forceinline__ float4 unpack4_of(float4 v, int) { return v; }
__device__ __forceinline__ float4 unpack4_of(uint2 v, int f16) { return f16 ? unpack4(v, __half()) : unpack4(v, __nv_bfloat16()); }
__device__ __forceinline__ float4 pack4_of(float4 v, float, int) { return v; }
__device__ __forceinline__ uint2 pack4_of(float4 v, unsigned short, int f16) {
    return f16 ? pack4(v, __half()) : pack4(v, __nv_bfloat16());
}

inline bool aligned_to(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1u)) == 0; }
inline bool valid_dtype(int dtype) { return dtype == PN2_F32 || dtype == PN2_BF16 || dtype == PN2_F16; }

}  // namespace pn2
