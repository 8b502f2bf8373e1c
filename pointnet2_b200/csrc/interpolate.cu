// interpolate.cu — three_nn, three_interpolate (+grad) and the fused feature-propagation front
// end, for sm_90a.
//
// Replaces the CPU-only functions of the reference (tf_ops/3d_interpolation/tf_interpolate.cpp):
//   threenn_cpu :60-103, threeinterpolate_cpu :107-127, threeinterpolate_grad_cpu :131-153
// — which TensorFlow runs on the host with D2H/H2D copies around them — with device kernels.
//
// three_nn is bit-exact with the reference's x86 arithmetic: squared distance without
// contraction (pn2::d2_nofma), strict '<' three-way insertion in ascending known index (earlier
// index wins ties), +inf / index 0 for missing neighbours.  three_interpolate evaluates
// ((p1*w1 + p2*w2) + p3*w3) with every operation rounded on its own, i.e. also bit-exact (the
// contract only asks for 1e-5 abs).
#include <math.h>

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kNnThreads = 128;
constexpr int kNnTile = 2048;  // known points per shared-memory tile (24 KB as pairs)

struct Top3 {
    float d1, d2, d3;
    int i1, i2, i3;
};

__device__ __forceinline__ void top3_init(Top3& t) {
    t.d1 = t.d2 = t.d3 = INFINITY;
    t.i1 = t.i2 = t.i3 = 0;
}

// Branch-free insertion (selects only): the reference's strict '<' cascade (tf_interpolate.cpp:74-89).
// A candidate that is not < d3 leaves the state untouched.
__device__ __forceinline__ void top3_insert(Top3& t, float d, int k) {
    const bool c3 = d < t.d3, c2 = d < t.d2, c1 = d < t.d1;  // c1 => c2 => c3 (d1 <= d2 <= d3)
    const float nd3 = c2 ? t.d2 : d;
    const int ni3 = c2 ? t.i2 : k;
    const float nd2 = c1 ? t.d1 : d;
    const int ni2 = c1 ? t.i1 : k;
    t.d3 = c3 ? nd3 : t.d3;
    t.i3 = c3 ? ni3 : t.i3;
    t.d2 = c2 ? nd2 : t.d2;
    t.i2 = c2 ? ni2 : t.i2;
    t.d1 = c1 ? d : t.d1;
    t.i1 = c1 ? k : t.i1;
}

constexpr int kNnPairs = kNnTile / 2;

// Shared-memory tile of known points stored as PAIRS: s_xy[i] = (x0, x1, y0, y1) of points 2i, 2i+1,
// s_z[i] = (z0, z1).  The tail up to a multiple of 2 pairs is +inf (distance +inf never passes '<').
struct KnownTile {
    ulonglong2 xy[kNnPairs];
    unsigned long long z[kNnPairs];
};

__device__ __forceinline__ int stage_known(KnownTile& tile, const float* __restrict__ known, int base, int m, int tid,
                                           int nthreads) {
    const int tn = min(kNnTile, m - base);
    const int tp_pad = (((tn + 1) >> 1) + 1) & ~1;  // pairs, rounded up to an even count
    float* sxy = reinterpret_cast<float*>(tile.xy);
    float* sz = reinterpret_cast<float*>(tile.z);
    for (int p = tid; p < 2 * tp_pad; p += nthreads) {
        float x = INFINITY, y = INFINITY, z = INFINITY;
        if (p < tn) {
            const float* s = known + (size_t)(base + p) * 3;
            x = s[0];
            y = s[1];
            z = s[2];
        }
        const int pi = p >> 1, par = p & 1;
        sxy[4 * pi + par] = x;
        sxy[4 * pi + 2 + par] = y;
        sz[2 * pi + par] = z;
    }
    return tp_pad;
}

// Scan one tile.  Candidates are offered in ascending known index; the (rare, per-lane) insertion
// sits behind a warp-uniform vote so the common path is distance math + one compare per point.
__device__ __forceinline__ void scan_tile(Top3& t, const KnownTile& tile, int tp_pad, int base, float ux, float uy,
                                          float uz) {
    const unsigned long long UX = f2_pack(ux, ux), UY = f2_pack(uy, uy), UZ = f2_pack(uz, uz);
    for (int p = 0; p < tp_pad; p += 2) {
        float d[4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const ulonglong2 xy = tile.xy[p + u];
            const unsigned long long zz = tile.z[p + u];
            const unsigned long long dx = f2_sub(xy.x, UX), dy = f2_sub(xy.y, UY), dz = f2_sub(zz, UZ);
            // the sums use the __fadd_rn intrinsic, which is never contracted with the products: the
            // reference's x86 code rounds every product before it is added
            float xx0, xx1, yy0, yy1, zz0, zz1;
            f2_unpack(f2_mul(dx, dx), xx0, xx1);
            f2_unpack(f2_mul(dy, dy), yy0, yy1);
            f2_unpack(f2_mul(dz, dz), zz0, zz1);
            d[2 * u] = __fadd_rn(__fadd_rn(xx0, yy0), zz0);
            d[2 * u + 1] = __fadd_rn(__fadd_rn(xx1, yy1), zz1);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (__any_sync(kFullMask, d[u] < t.d3)) top3_insert(t, d[u], base + 2 * p + u);
        }
    }
}

// One thread per unknown point; known points broadcast from shared memory.
// L (ragged unknown side): cloud i's unknown points are its first cloud_length(lengths, i, n) rows.  A template flag, so
// that the instance without lengths compiles to the code it always did.  Padding rows get the (+inf, 0) filler; a CTA
// made only of padding writes it and leaves before the known-point loop (CTA-uniform: the cloud is blockIdx.y).
template <bool L>
__global__ void __launch_bounds__(kNnThreads)
three_nn_kernel(int n, int m, const float* __restrict__ xyz1, const float* __restrict__ xyz2,
                float* __restrict__ dist, int* __restrict__ idx, const int* __restrict__ lengths) {
    __shared__ KnownTile s_tile;
    const int tid = threadIdx.x;
    const int cloud = blockIdx.y;
    const int j = blockIdx.x * kNnThreads + tid;
    const int len = L ? cloud_length(lengths, cloud, n) : n;
    const bool valid = j < len;
    if (L && (int)(blockIdx.x * kNnThreads) >= len) {
        if (j < n) {
            float* dd = dist + ((size_t)cloud * n + j) * 3;
            int* ii = idx + ((size_t)cloud * n + j) * 3;
            dd[0] = dd[1] = dd[2] = INFINITY;
            ii[0] = ii[1] = ii[2] = 0;
        }
        return;
    }
    const float* __restrict__ known = xyz2 + (size_t)cloud * m * 3;
    float ux = 0.f, uy = 0.f, uz = 0.f;
    if (valid) {
        const float* u = xyz1 + ((size_t)cloud * n + j) * 3;
        ux = u[0];
        uy = u[1];
        uz = u[2];
    }
    Top3 t;
    top3_init(t);
    for (int base = 0; base < m; base += kNnTile) {
        if (base) __syncthreads();
        const int tp_pad = stage_known(s_tile, known, base, m, tid, kNnThreads);
        __syncthreads();
        scan_tile(t, s_tile, tp_pad, base, ux, uy, uz);
    }
    if (L && !valid) top3_init(t);  // a padding row of a partly filled CTA: the filler
    if (L ? j < n : valid) {
        float* dd = dist + ((size_t)cloud * n + j) * 3;
        int* ii = idx + ((size_t)cloud * n + j) * 3;
        dd[0] = t.d1; dd[1] = t.d2; dd[2] = t.d3;
        ii[0] = t.i1; ii[1] = t.i2; ii[2] = t.i3;
    }
}

// ---- three_interpolate (interp3: pn2_common.cuh) ------------------------------------------------

constexpr int kItThreads = 256;

// One thread per output float4: 4 outputs in flight per thread cost 96 registers and quarter occupancy; staging
// channel slices of the known features in shared memory is worse still (one 160 KB CTA per SM cannot hide its own
// slice load).
// T = float, __nv_bfloat16 or __half: P = Pack4<T>::type holds 4 channels; they are upcast, interpolated in float32
// and rounded once on the way out.
// L (ragged unknown side, lengths (b,) of the n rows per cloud): padding rows j >= the cloud's length write zeros and read
// neither idx nor weight.  A template flag, as in three_nn_kernel.
template <typename IndexT, typename T, bool L = false, typename P = typename Pack4<T>::type>
__global__ void __launch_bounds__(kItThreads)
three_interp_vec4_kernel(int m, int c4, IndexT rows_per_cloud, IndexT total_vec, const P* __restrict__ points,
                         const int* __restrict__ idx, const float* __restrict__ weight, P* __restrict__ out,
                         const int* __restrict__ lengths) {
    const IndexT stride = (IndexT)gridDim.x * kItThreads;
    for (IndexT v = (IndexT)blockIdx.x * kItThreads + threadIdx.x; v < total_vec; v += stride) {
        const IndexT row = v / (IndexT)c4;
        const int l = (int)(v - row * (IndexT)c4);
        const IndexT cloud = row / rows_per_cloud;
        if (L && row - cloud * rows_per_cloud >= (IndexT)cloud_length(lengths, (int)cloud, (int)rows_per_cloud)) {
            __stcs(out + v, pack4(make_float4(0.f, 0.f, 0.f, 0.f), T()));
            continue;
        }
        const int i1 = __ldg(idx + (size_t)row * 3 + 0);
        const int i2 = __ldg(idx + (size_t)row * 3 + 1);
        const int i3 = __ldg(idx + (size_t)row * 3 + 2);
        const float w1 = __ldg(weight + (size_t)row * 3 + 0);
        const float w2 = __ldg(weight + (size_t)row * 3 + 1);
        const float w3 = __ldg(weight + (size_t)row * 3 + 2);
        const P* pb = points + (size_t)cloud * m * c4 + l;
        const float4 a = unpack4(__ldg(pb + (size_t)i1 * c4), T());
        const float4 b = unpack4(__ldg(pb + (size_t)i2 * c4), T());
        const float4 c = unpack4(__ldg(pb + (size_t)i3 * c4), T());
        float4 o;
        o.x = interp3(a.x, b.x, c.x, w1, w2, w3);
        o.y = interp3(a.y, b.y, c.y, w1, w2, w3);
        o.z = interp3(a.z, b.z, c.z, w1, w2, w3);
        o.w = interp3(a.w, b.w, c.w, w1, w2, w3);
        __stcs(out + v, pack4(o, T()));
    }
}

template <typename IndexT, typename T, bool L = false>
__global__ void __launch_bounds__(kItThreads)
three_interp_scalar_kernel(int m, int c, IndexT rows_per_cloud, IndexT total, const T* __restrict__ points,
                           const int* __restrict__ idx, const float* __restrict__ weight, T* __restrict__ out,
                           const int* __restrict__ lengths) {
    const IndexT stride = (IndexT)gridDim.x * kItThreads;
    for (IndexT e = (IndexT)blockIdx.x * kItThreads + threadIdx.x; e < total; e += stride) {
        const IndexT row = e / (IndexT)c;
        const int l = (int)(e - row * (IndexT)c);
        const IndexT cloud = row / rows_per_cloud;
        if (L && row - cloud * rows_per_cloud >= (IndexT)cloud_length(lengths, (int)cloud, (int)rows_per_cloud)) {
            out[e] = from_f32<T>(0.f);
            continue;
        }
        const int* ii = idx + (size_t)row * 3;
        const float* w = weight + (size_t)row * 3;
        const T* pb = points + (size_t)cloud * m * c + l;
        out[e] = from_f32<T>(interp3(to_f32(__ldg(pb + (size_t)__ldg(ii + 0) * c)), to_f32(__ldg(pb + (size_t)__ldg(ii + 1) * c)),
                                     to_f32(__ldg(pb + (size_t)__ldg(ii + 2) * c)), __ldg(w + 0), __ldg(w + 1), __ldg(w + 2)));
    }
}

// grad_points[b, idx[b,j,t], l] += grad_out[b,j,l] * weight[b,j,t]
// L: rows j >= the cloud's length (lengths, as in three_interp_vec4_kernel) are skipped.
template <typename IndexT, bool L = false>
__global__ void __launch_bounds__(kItThreads)
three_interp_grad_vec4_kernel(int m, int c4, IndexT rows_per_cloud, IndexT total_vec,
                              const float4* __restrict__ grad_out, const int* __restrict__ idx,
                              const float* __restrict__ weight, float4* __restrict__ grad_points,
                              const int* __restrict__ lengths) {
    const IndexT stride = (IndexT)gridDim.x * kItThreads;
    for (IndexT v = (IndexT)blockIdx.x * kItThreads + threadIdx.x; v < total_vec; v += stride) {
        const IndexT row = v / (IndexT)c4;
        const int l = (int)(v - row * (IndexT)c4);
        const IndexT cloud = row / rows_per_cloud;
        if (L && row - cloud * rows_per_cloud >= (IndexT)cloud_length(lengths, (int)cloud, (int)rows_per_cloud)) continue;
        const float4 g = __ldcs(grad_out + v);
        float4* gb = grad_points + (size_t)cloud * m * c4 + l;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            const int i = __ldg(idx + (size_t)row * 3 + t);
            const float w = __ldg(weight + (size_t)row * 3 + t);
            atomicAdd(gb + (size_t)i * c4,
                      make_float4(__fmul_rn(g.x, w), __fmul_rn(g.y, w), __fmul_rn(g.z, w), __fmul_rn(g.w, w)));
        }
    }
}

template <typename IndexT, bool L = false>
__global__ void __launch_bounds__(kItThreads)
three_interp_grad_scalar_kernel(int m, int c, IndexT rows_per_cloud, IndexT total, const float* __restrict__ grad_out,
                                const int* __restrict__ idx, const float* __restrict__ weight,
                                float* __restrict__ grad_points, const int* __restrict__ lengths) {
    const IndexT stride = (IndexT)gridDim.x * kItThreads;
    for (IndexT e = (IndexT)blockIdx.x * kItThreads + threadIdx.x; e < total; e += stride) {
        const IndexT row = e / (IndexT)c;
        const int l = (int)(e - row * (IndexT)c);
        const IndexT cloud = row / rows_per_cloud;
        if (L && row - cloud * rows_per_cloud >= (IndexT)cloud_length(lengths, (int)cloud, (int)rows_per_cloud)) continue;
        const float g = __ldcs(grad_out + e);
        float* gb = grad_points + (size_t)cloud * m * c + l;
#pragma unroll
        for (int t = 0; t < 3; ++t)
            atomicAdd(gb + (size_t)__ldg(idx + (size_t)row * 3 + t) * c, __fmul_rn(g, __ldg(weight + (size_t)row * 3 + t)));
    }
}

// ---- fused FP front end: three_nn -> inverse-distance weights -> three_interpolate -> concat -----
// utils/pointnet_util.py:211-219.  G lanes share one unknown point: lane g scans the known points of
// pairs p = g, g+G, ... (ascending index inside the lane), the G partial top-3 lists are merged by a
// shuffle butterfly under (distance, index) — exactly the order the reference's strict '<' scan over
// ascending indices produces — so small layers (64 or 256 unknown points per cloud) still fill the
// machine: a CTA covers 128/G points.  Phase 2 writes the CTA's rows of the output
// [interpolated (c2) | points1 (c1)] with consecutive lanes on consecutive channels; dist / idx /
// weight never touch HBM unless the caller asks for them, and the concat of :219 is not a separate pass.
__device__ __forceinline__ void top3_insert_lex(Top3& t, float d, int k) {
    // like top3_insert, with ties broken by the smaller index (candidates arrive out of index order)
    const bool c3 = d < t.d3 || (d == t.d3 && k < t.i3), c2 = d < t.d2 || (d == t.d2 && k < t.i2),
               c1 = d < t.d1 || (d == t.d1 && k < t.i1);
    const float nd3 = c2 ? t.d2 : d;
    const int ni3 = c2 ? t.i2 : k;
    const float nd2 = c1 ? t.d1 : d;
    const int ni2 = c1 ? t.i1 : k;
    t.d3 = c3 ? nd3 : t.d3;
    t.i3 = c3 ? ni3 : t.i3;
    t.d2 = c2 ? nd2 : t.d2;
    t.i2 = c2 ? ni2 : t.i2;
    t.d1 = c1 ? d : t.d1;
    t.i1 = c1 ? k : t.i1;
}

// lane g of G scans pairs g, g+G, ... of the tile (2 points per pair)
template <int G>
__device__ __forceinline__ void scan_tile_strided(Top3& t, const KnownTile& tile, int tp_pad, int base, int g, float ux, float uy,
                                                  float uz) {
    const unsigned long long UX = f2_pack(ux, ux), UY = f2_pack(uy, uy), UZ = f2_pack(uz, uz);
    for (int p = g; p < tp_pad; p += G) {
        const ulonglong2 xy = tile.xy[p];
        const unsigned long long zz = tile.z[p];
        const unsigned long long dx = f2_sub(xy.x, UX), dy = f2_sub(xy.y, UY), dz = f2_sub(zz, UZ);
        float xx0, xx1, yy0, yy1, zz0, zz1;
        f2_unpack(f2_mul(dx, dx), xx0, xx1);
        f2_unpack(f2_mul(dy, dy), yy0, yy1);
        f2_unpack(f2_mul(dz, dz), zz0, zz1);
        const float d0 = __fadd_rn(__fadd_rn(xx0, yy0), zz0), d1 = __fadd_rn(__fadd_rn(xx1, yy1), zz1);
        if (d0 < t.d3) top3_insert(t, d0, base + 2 * p);
        if (d1 < t.d3) top3_insert(t, d1, base + 2 * p + 1);
    }
}

// T: element type of points1 / points2 / out: float, or unsigned short for both 2-byte formats, f16 choosing float16 or
// bfloat16 at run time (the 3-NN phase is most of the code: one 2-byte instance per G instead of two).  Phase 2 upcasts,
// interpolates in float32 and rounds once; points1 is copied.
// L (ragged unknown side, as in three_nn_kernel): padding rows get dist +inf, idx 0, weight 0 and an all-zero output row
// (points1 is not read there).  A CTA made only of padding writes that and leaves before the known-point loop; in a
// partly filled one every lane still takes part in the merge, and `valid` gates only loads and stores.
template <int G, typename T, bool L>
__global__ void __launch_bounds__(kNnThreads)
fp_front_kernel(int n, int m, int c2, int c1, const float* __restrict__ xyz1, const float* __restrict__ xyz2,
                const T* __restrict__ points1, const T* __restrict__ points2, T* __restrict__ out,
                float* __restrict__ dist_o, int* __restrict__ idx_o, float* __restrict__ weight_o, int f16,
                const int* __restrict__ lengths) {
    constexpr int PPB = kNnThreads / G;  // unknown points per CTA
    __shared__ KnownTile s_tile;
    __shared__ int s_i[PPB][3];
    __shared__ float s_w[PPB][3];
    const int tid = threadIdx.x;
    const int g = tid % G, slot = tid / G;
    const int cloud = blockIdx.y;
    const int j0 = blockIdx.x * PPB;
    const int j = j0 + slot;
    const int len = L ? cloud_length(lengths, cloud, n) : n;
    const bool valid = j < len;
    if (L && j0 >= len) {
        if (g == 0 && j < n) {
            const size_t o = ((size_t)cloud * n + j) * 3;
            if (dist_o) { dist_o[o] = INFINITY; dist_o[o + 1] = INFINITY; dist_o[o + 2] = INFINITY; }
            if (idx_o) { idx_o[o] = 0; idx_o[o + 1] = 0; idx_o[o + 2] = 0; }
            if (weight_o) { weight_o[o] = 0.f; weight_o[o + 1] = 0.f; weight_o[o + 2] = 0.f; }
        }
        if (out) {
            const int cw = c2 + c1;
            T* __restrict__ ob = out + ((size_t)cloud * n + j0) * cw;
            for (int e = tid; e < min(PPB, n - j0) * cw; e += kNnThreads) ob[e] = of_f32<T>(0.f, f16);
        }
        return;
    }
    const float* __restrict__ known = xyz2 + (size_t)cloud * m * 3;
    float ux = 0.f, uy = 0.f, uz = 0.f;
    if (valid) {
        const float* u = xyz1 + ((size_t)cloud * n + j) * 3;
        ux = __ldg(u);
        uy = __ldg(u + 1);
        uz = __ldg(u + 2);
    }
    Top3 t;
    top3_init(t);
    for (int base = 0; base < m; base += kNnTile) {
        if (base) __syncthreads();
        const int tp_pad = stage_known(s_tile, known, base, m, tid, kNnThreads);
        __syncthreads();
        if (G == 1) scan_tile(t, s_tile, tp_pad, base, ux, uy, uz);
        else scan_tile_strided<G>(t, s_tile, tp_pad, base, g, ux, uy, uz);
    }
    if (G > 1) {  // merge the G partial lists of this point (all lanes end with the merged list)
#pragma unroll
        for (int o = 1; o < G; o <<= 1) {
            const float e1 = __shfl_xor_sync(kFullMask, t.d1, o), e2 = __shfl_xor_sync(kFullMask, t.d2, o),
                        e3 = __shfl_xor_sync(kFullMask, t.d3, o);
            const int f1 = __shfl_xor_sync(kFullMask, t.i1, o), f2 = __shfl_xor_sync(kFullMask, t.i2, o),
                      f3 = __shfl_xor_sync(kFullMask, t.i3, o);
            // +inf entries are the (inf, 0) filler of an unfilled slot: never insert them (index 0 would win ties)
            if (e1 < INFINITY) top3_insert_lex(t, e1, f1);
            if (e2 < INFINITY) top3_insert_lex(t, e2, f2);
            if (e3 < INFINITY) top3_insert_lex(t, e3, f3);
        }
    }
    // dist = max(dist, 1e-10); norm = sum(1/dist); weight = (1/dist)/norm   (pointnet_util.py:212-215)
    const float r1 = __fdiv_rn(1.0f, fmaxf(t.d1, 1e-10f));
    const float r2 = __fdiv_rn(1.0f, fmaxf(t.d2, 1e-10f));
    const float r3 = __fdiv_rn(1.0f, fmaxf(t.d3, 1e-10f));
    const float norm = __fadd_rn(__fadd_rn(r1, r2), r3);
    const float w1 = __fdiv_rn(r1, norm), w2 = __fdiv_rn(r2, norm), w3 = __fdiv_rn(r3, norm);
    if (g == 0) {
        s_i[slot][0] = t.i1; s_i[slot][1] = t.i2; s_i[slot][2] = t.i3;
        s_w[slot][0] = w1;   s_w[slot][1] = w2;   s_w[slot][2] = w3;
        if (valid) {
            const size_t o = ((size_t)cloud * n + j) * 3;
            if (dist_o) { dist_o[o] = t.d1; dist_o[o + 1] = t.d2; dist_o[o + 2] = t.d3; }
            if (idx_o) { idx_o[o] = t.i1; idx_o[o + 1] = t.i2; idx_o[o + 2] = t.i3; }
            if (weight_o) { weight_o[o] = w1; weight_o[o + 1] = w2; weight_o[o + 2] = w3; }
        } else if (L && j < n) {  // a padding row of a partly filled CTA
            const size_t o = ((size_t)cloud * n + j) * 3;
            if (dist_o) { dist_o[o] = INFINITY; dist_o[o + 1] = INFINITY; dist_o[o + 2] = INFINITY; }
            if (idx_o) { idx_o[o] = 0; idx_o[o + 1] = 0; idx_o[o + 2] = 0; }
            if (weight_o) { weight_o[o] = 0.f; weight_o[o + 1] = 0.f; weight_o[o + 2] = 0.f; }
        }
    }
    __syncthreads();
    if (!out) return;
    const int rows = min(PPB, n - j0);
    const int real_rows = L ? min(PPB, len - j0) : rows;  // rows from real_rows on are padding: zeros
    const int cw = c2 + c1;  // output row width
    const T* __restrict__ pb = points2 + (size_t)cloud * m * c2;
    const T* __restrict__ p1 = points1 ? points1 + ((size_t)cloud * n + j0) * c1 : nullptr;
    T* __restrict__ ob = out + ((size_t)cloud * n + j0) * cw;
    const bool vec = ((c2 | c1) & 3) == 0 &&
                     ((reinterpret_cast<uintptr_t>(pb) | reinterpret_cast<uintptr_t>(ob) | reinterpret_cast<uintptr_t>(p1)) & (4 * sizeof(T) - 1)) == 0;
    if (vec) {  // 4 channels per vector
        using P = typename Pack4<T>::type;
        const int c24 = c2 >> 2, cw4 = cw >> 2, c14 = c1 >> 2;
        const P* pb4 = reinterpret_cast<const P*>(pb);
        const P* p14 = reinterpret_cast<const P*>(p1);
        P* ob4 = reinterpret_cast<P*>(ob);
        for (int e = tid; e < rows * cw4; e += kNnThreads) {
            const int r = e / cw4, l = e - r * cw4;
            P o;
            if (L && r >= real_rows) {
                o = pack4_of(make_float4(0.f, 0.f, 0.f, 0.f), T(), f16);
            } else if (l < c24) {
                const float4 a = unpack4_of(__ldg(pb4 + (size_t)s_i[r][0] * c24 + l), f16),
                             b = unpack4_of(__ldg(pb4 + (size_t)s_i[r][1] * c24 + l), f16),
                             cc = unpack4_of(__ldg(pb4 + (size_t)s_i[r][2] * c24 + l), f16);
                const float x1 = s_w[r][0], x2 = s_w[r][1], x3 = s_w[r][2];
                float4 f;
                f.x = interp3(a.x, b.x, cc.x, x1, x2, x3);
                f.y = interp3(a.y, b.y, cc.y, x1, x2, x3);
                f.z = interp3(a.z, b.z, cc.z, x1, x2, x3);
                f.w = interp3(a.w, b.w, cc.w, x1, x2, x3);
                o = pack4_of(f, T(), f16);
            } else {
                o = __ldcs(p14 + (size_t)r * c14 + (l - c24));  // points1, read once, copied as it is
            }
            __stcs(ob4 + e, o);
        }
    } else {
        for (int e = tid; e < rows * cw; e += kNnThreads) {
            const int r = e / cw, l = e - r * cw;
            T o;
            if (L && r >= real_rows)
                o = of_f32<T>(0.f, f16);
            else if (l < c2)
                o = of_f32<T>(interp3(f32_of(__ldg(pb + (size_t)s_i[r][0] * c2 + l), f16), f32_of(__ldg(pb + (size_t)s_i[r][1] * c2 + l), f16),
                                      f32_of(__ldg(pb + (size_t)s_i[r][2] * c2 + l), f16), s_w[r][0], s_w[r][1], s_w[r][2]), f16);
            else
                o = __ldcs(p1 + (size_t)r * c1 + (l - c2));
            ob[e] = o;
        }
    }
}

template <int G, typename T>
static int launch_fp_front(int b, int n, int m, int c2, int c1, const float* xyz1, const int* lengths, const float* xyz2,
                           const T* points1, const T* points2, T* out, float* dist, int* idx, float* weight, int f16,
                           cudaStream_t st) {
    constexpr int PPB = kNnThreads / G;
    dim3 grid((n + PPB - 1) / PPB, b, 1);
    if (lengths)
        fp_front_kernel<G, T, true><<<grid, kNnThreads, 0, st>>>(n, m, c2, c1, xyz1, xyz2, points1, points2, out, dist, idx, weight, f16,
                                                                 lengths);
    else
        fp_front_kernel<G, T, false><<<grid, kNnThreads, 0, st>>>(n, m, c2, c1, xyz1, xyz2, points1, points2, out, dist, idx, weight,
                                                                  f16, nullptr);
    return finish_launch();
}

// lengths (b,) device int32 of xyz1 / points1 / out, or NULL
template <typename T>
static int fp_front_dispatch(int b, int n, int m, int c2, int c1, const float* xyz1, const int* lengths, const float* xyz2,
                             const T* points1, const T* points2, T* out, float* dist, int* idx, float* weight, int f16,
                             cudaStream_t st) {
    // lanes per unknown point: as many as it takes to put ~2 CTAs on every SM (a CTA covers 128/G points),
    // but never more lanes than there are pairs of known points to share.  Chosen from b*n with or without lengths.
    const long long pts = (long long)b * n;
    int G = 1;
    while (G < 32 && pts * G < 2LL * num_sms() * kNnThreads && 2 * G <= (m + 1) / 2) G *= 2;
#define PN2_FP_FRONT(GG) \
    launch_fp_front<GG, T>(b, n, m, c2, c1, xyz1, lengths, xyz2, points1, points2, out, dist, idx, weight, f16, st)
    switch (G) {
        case 1: return PN2_FP_FRONT(1);
        case 2: return PN2_FP_FRONT(2);
        case 4: return PN2_FP_FRONT(4);
        case 8: return PN2_FP_FRONT(8);
        case 16: return PN2_FP_FRONT(16);
        default: return PN2_FP_FRONT(32);
    }
#undef PN2_FP_FRONT
}

template <typename T, bool L>
static void three_interpolate_launch(int b, int m, int c, int n, const T* points, const int* idx, const float* weight,
                                     const int* lengths, T* out, cudaStream_t st) {
    using P = typename Pack4<T>::type;
    const unsigned long long total = (unsigned long long)b * n * c;
    if (c % 4 == 0 && aligned_to(points, sizeof(P)) && aligned_to(out, sizeof(P))) {
        const unsigned long long tv = total / 4;
        const unsigned grid = grid_for(tv, kItThreads);
        if (tv < (1ull << 31))
            three_interp_vec4_kernel<unsigned, T, L><<<grid, kItThreads, 0, st>>>(m, c / 4, (unsigned)n, (unsigned)tv, (const P*)points, idx, weight, (P*)out, lengths);
        else
            three_interp_vec4_kernel<unsigned long long, T, L><<<grid, kItThreads, 0, st>>>(m, c / 4, (unsigned long long)n, tv, (const P*)points, idx, weight, (P*)out, lengths);
    } else {
        const unsigned grid = grid_for(total, kItThreads);
        if (total < (1ull << 31))
            three_interp_scalar_kernel<unsigned, T, L><<<grid, kItThreads, 0, st>>>(m, c, (unsigned)n, (unsigned)total, points, idx, weight, out, lengths);
        else
            three_interp_scalar_kernel<unsigned long long, T, L><<<grid, kItThreads, 0, st>>>(m, c, (unsigned long long)n, total, points, idx, weight, out, lengths);
    }
}

// lengths (b,) device int32 of the n unknown rows, or NULL
template <typename T>
static int three_interpolate_impl(int b, int m, int c, int n, const T* points, const int* idx, const float* weight,
                                  const int* lengths, T* out, cudaStream_t st) {
    if (lengths) three_interpolate_launch<T, true>(b, m, c, n, points, idx, weight, lengths, out, st);
    else three_interpolate_launch<T, false>(b, m, c, n, points, idx, weight, nullptr, out, st);
    return finish_launch();
}

template <typename T>
static int three_interpolate_grad_det_impl(int b, int n, int c, int m, const T* grad_out, const int* idx, const float* weight,
                                           const int* lengths, T* grad_points, void* workspace, size_t workspace_bytes, int f16,
                                           void* stream) {
    if (b < 0 || m <= 0 || c < 0 || n < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * m * c == 0) return 0;
    if (!grad_points) return (int)cudaErrorInvalidValue;
    cudaStream_t st = as_stream(stream);
    if (n == 0) return (int)cudaMemsetAsync(grad_points, 0, sizeof(T) * (size_t)b * m * c, st);
    if (!grad_out || !idx || !weight || !workspace) return (int)cudaErrorInvalidValue;
    if (workspace_bytes < ::pn2_three_interpolate_grad_det_workspace_bytes(b, n, m) || (long long)n * 3 > 0x7fffffffLL)
        return (int)cudaErrorInvalidValue;
    return inv_scatter_det<true, T>(b, n, 3 * n, c, m, grad_out, idx, weight, lengths, grad_points, workspace, f16, st);
}

}  // namespace pn2

extern "C" {

// Every entry without lengths forwards to its *_ragged twin with lengths1 = NULL.

int pn2_three_nn_ragged(int b, int n, int m, const float* xyz1, const int* lengths1, const float* xyz2, float* dist, int* idx,
                        void* stream) {
    using namespace pn2;
    if (b < 0 || n < 0 || m < 0) return (int)cudaErrorInvalidValue;
    if (b == 0 || n == 0) return 0;
    if (!xyz1 || (m > 0 && !xyz2) || !dist || !idx) return (int)cudaErrorInvalidValue;
    if (b > 65535) return (int)cudaErrorInvalidValue;
    dim3 grid((n + kNnThreads - 1) / kNnThreads, b, 1);
    if (lengths1)
        three_nn_kernel<true><<<grid, kNnThreads, 0, as_stream(stream)>>>(n, m, xyz1, xyz2, dist, idx, lengths1);
    else
        three_nn_kernel<false><<<grid, kNnThreads, 0, as_stream(stream)>>>(n, m, xyz1, xyz2, dist, idx, nullptr);
    return finish_launch();
}

int pn2_three_nn(int b, int n, int m, const float* xyz1, const float* xyz2, float* dist, int* idx, void* stream) {
    return pn2_three_nn_ragged(b, n, m, xyz1, nullptr, xyz2, dist, idx, stream);
}

int pn2_three_interpolate_ragged_typed(int dtype, int b, int m, int c, int n, const void* points, const int* idx,
                                       const float* weight, const int* lengths1, void* out, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (b < 0 || m <= 0 || c < 0 || n < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * n * c == 0) return 0;
    if (!points || !idx || !weight || !out) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32)
        return three_interpolate_impl<float>(b, m, c, n, static_cast<const float*>(points), idx, weight, lengths1,
                                             static_cast<float*>(out), as_stream(stream));
    if (dtype == PN2_BF16)
        return three_interpolate_impl<__nv_bfloat16>(b, m, c, n, static_cast<const __nv_bfloat16*>(points), idx, weight, lengths1,
                                                     static_cast<__nv_bfloat16*>(out), as_stream(stream));
    return three_interpolate_impl<__half>(b, m, c, n, static_cast<const __half*>(points), idx, weight, lengths1,
                                          static_cast<__half*>(out), as_stream(stream));
}

int pn2_three_interpolate(int b, int m, int c, int n, const float* points, const int* idx, const float* weight,
                          float* out, void* stream) {
    return pn2_three_interpolate_ragged_typed(PN2_F32, b, m, c, n, points, idx, weight, nullptr, out, stream);
}

int pn2_three_interpolate_typed(int dtype, int b, int m, int c, int n, const void* points, const int* idx,
                                const float* weight, void* out, void* stream) {
    return pn2_three_interpolate_ragged_typed(dtype, b, m, c, n, points, idx, weight, nullptr, out, stream);
}

int pn2_three_interpolate_grad_ragged(int b, int n, int c, int m, const float* grad_out, const int* idx, const float* weight,
                                      const int* lengths1, float* grad_points, void* stream) {
    using namespace pn2;
    if (b < 0 || m <= 0 || c < 0 || n < 0) return (int)cudaErrorInvalidValue;
    const unsigned long long total = (unsigned long long)b * n * c;
    if (total == 0) return 0;
    if (!grad_out || !idx || !weight || !grad_points) return (int)cudaErrorInvalidValue;
    cudaStream_t st = as_stream(stream);
#define PN2_GRAD_ATOMIC(L, LEN)                                                                                                \
    if (c % 4 == 0 && aligned_to(grad_out, 16) && aligned_to(grad_points, 16)) {                                                                   \
        const unsigned long long tv = total / 4;                                                                               \
        const unsigned grid = grid_for(tv, kItThreads);                                                                         \
        if (tv < (1ull << 31))                                                                                                 \
            three_interp_grad_vec4_kernel<unsigned, L><<<grid, kItThreads, 0, st>>>(m, c / 4, (unsigned)n, (unsigned)tv,         \
                                                                                    (const float4*)grad_out, idx, weight,        \
                                                                                    (float4*)grad_points, LEN);                  \
        else                                                                                                                   \
            three_interp_grad_vec4_kernel<unsigned long long, L><<<grid, kItThreads, 0, st>>>(                                  \
                m, c / 4, (unsigned long long)n, tv, (const float4*)grad_out, idx, weight, (float4*)grad_points, LEN);          \
    } else {                                                                                                                   \
        const unsigned grid = grid_for(total, kItThreads);                                                                      \
        if (total < (1ull << 31))                                                                                              \
            three_interp_grad_scalar_kernel<unsigned, L><<<grid, kItThreads, 0, st>>>(m, c, (unsigned)n, (unsigned)total,        \
                                                                                      grad_out, idx, weight, grad_points, LEN);  \
        else                                                                                                                   \
            three_interp_grad_scalar_kernel<unsigned long long, L><<<grid, kItThreads, 0, st>>>(                                \
                m, c, (unsigned long long)n, total, grad_out, idx, weight, grad_points, LEN);                                   \
    }
    if (lengths1) {
        PN2_GRAD_ATOMIC(true, lengths1)
    } else {
        PN2_GRAD_ATOMIC(false, nullptr)
    }
#undef PN2_GRAD_ATOMIC
    return finish_launch();
}

int pn2_three_interpolate_grad(int b, int n, int c, int m, const float* grad_out, const int* idx, const float* weight,
                               float* grad_points, void* stream) {
    return pn2_three_interpolate_grad_ragged(b, n, c, m, grad_out, idx, weight, nullptr, grad_points, stream);
}

int pn2_three_nn_interpolate_ragged_typed(int dtype, int b, int n, int m, int c, const float* xyz1, const int* lengths1,
                                          const float* xyz2, const void* points2, void* out, float* dist, int* idx,
                                          float* weight, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (b < 0 || n < 0 || m <= 0 || c < 0) return (int)cudaErrorInvalidValue;
    if (b == 0 || n == 0) return 0;
    if (!xyz1 || !xyz2 || (c > 0 && (!points2 || !out))) return (int)cudaErrorInvalidValue;
    if (b > 65535) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32)
        return fp_front_dispatch<float>(b, n, m, c, 0, xyz1, lengths1, xyz2, nullptr, static_cast<const float*>(points2),
                                        c > 0 ? static_cast<float*>(out) : nullptr, dist, idx, weight, 0, as_stream(stream));
    using U16 = unsigned short;  // bfloat16 and float16 share one instance: dtype == PN2_F16 selects the format
    return fp_front_dispatch<U16>(b, n, m, c, 0, xyz1, lengths1, xyz2, nullptr, static_cast<const U16*>(points2),
                                  c > 0 ? static_cast<U16*>(out) : nullptr, dist, idx, weight, dtype == PN2_F16, as_stream(stream));
}

int pn2_three_nn_interpolate(int b, int n, int m, int c, const float* xyz1, const float* xyz2, const float* points2,
                             float* out, float* dist, int* idx, float* weight, void* stream) {
    return pn2_three_nn_interpolate_ragged_typed(PN2_F32, b, n, m, c, xyz1, nullptr, xyz2, points2, out, dist, idx, weight, stream);
}

int pn2_three_nn_interpolate_typed(int dtype, int b, int n, int m, int c, const float* xyz1, const float* xyz2,
                                   const void* points2, void* out, float* dist, int* idx, float* weight,
                                   void* stream) {
    return pn2_three_nn_interpolate_ragged_typed(dtype, b, n, m, c, xyz1, nullptr, xyz2, points2, out, dist, idx, weight, stream);
}

int pn2_fp_interpolate_concat_ragged_typed(int dtype, int b, int n, int m, int c2, int c1, const float* xyz1,
                                           const int* lengths1, const float* xyz2, const void* points1, const void* points2,
                                           void* out, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (b < 0 || n < 0 || m <= 0 || c2 <= 0 || c1 < 0) return (int)cudaErrorInvalidValue;
    if (b == 0 || n == 0) return 0;
    if (!xyz1 || !xyz2 || !points2 || !out || (c1 > 0 && !points1)) return (int)cudaErrorInvalidValue;
    if (b > 65535) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32)
        return fp_front_dispatch<float>(b, n, m, c2, c1, xyz1, lengths1, xyz2, c1 > 0 ? static_cast<const float*>(points1) : nullptr,
                                        static_cast<const float*>(points2), static_cast<float*>(out), nullptr, nullptr, nullptr, 0,
                                        as_stream(stream));
    using U16 = unsigned short;  // bfloat16 and float16 share one instance: dtype == PN2_F16 selects the format
    return fp_front_dispatch<U16>(b, n, m, c2, c1, xyz1, lengths1, xyz2, c1 > 0 ? static_cast<const U16*>(points1) : nullptr,
                                  static_cast<const U16*>(points2), static_cast<U16*>(out), nullptr, nullptr, nullptr, dtype == PN2_F16,
                                  as_stream(stream));
}

int pn2_fp_interpolate_concat(int b, int n, int m, int c2, int c1, const float* xyz1, const float* xyz2, const float* points1,
                              const float* points2, float* out, void* stream) {
    return pn2_fp_interpolate_concat_ragged_typed(PN2_F32, b, n, m, c2, c1, xyz1, nullptr, xyz2, points1, points2, out, stream);
}

int pn2_fp_interpolate_concat_typed(int dtype, int b, int n, int m, int c2, int c1, const float* xyz1,
                                    const float* xyz2, const void* points1, const void* points2, void* out,
                                    void* stream) {
    return pn2_fp_interpolate_concat_ragged_typed(dtype, b, n, m, c2, c1, xyz1, nullptr, xyz2, points1, points2, out, stream);
}

size_t pn2_three_interpolate_grad_det_workspace_bytes(int b, int n, int m) {
    if (b <= 0 || n <= 0 || m <= 0) return 0;
    return pn2::inv_workspace_bytes(b, 3 * (long long)n, m);
}

int pn2_three_interpolate_grad_det_ragged_typed(int dtype, int b, int n, int c, int m, const void* grad_out, const int* idx,
                                                const float* weight, const int* lengths1, void* grad_points, void* workspace,
                                                size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32)
        return three_interpolate_grad_det_impl<float>(b, n, c, m, static_cast<const float*>(grad_out), idx, weight, lengths1,
                                                      static_cast<float*>(grad_points), workspace, workspace_bytes, 0, stream);
    using U16 = unsigned short;  // bfloat16 and float16 share one instance: dtype == PN2_F16 selects the format
    return three_interpolate_grad_det_impl<U16>(b, n, c, m, static_cast<const U16*>(grad_out), idx, weight, lengths1,
                                                static_cast<U16*>(grad_points), workspace, workspace_bytes, dtype == PN2_F16, stream);
}

int pn2_three_interpolate_grad_det(int b, int n, int c, int m, const float* grad_out, const int* idx, const float* weight,
                                   float* grad_points, void* workspace, size_t workspace_bytes, void* stream) {
    return pn2_three_interpolate_grad_det_ragged_typed(PN2_F32, b, n, c, m, grad_out, idx, weight, nullptr, grad_points, workspace,
                                                       workspace_bytes, stream);
}

int pn2_three_interpolate_grad_det_typed(int dtype, int b, int n, int c, int m, const void* grad_out,
                                         const int* idx, const float* weight, void* grad_points, void* workspace,
                                         size_t workspace_bytes, void* stream) {
    return pn2_three_interpolate_grad_det_ragged_typed(dtype, b, n, c, m, grad_out, idx, weight, nullptr, grad_points, workspace,
                                                       workspace_bytes, stream);
}

}  // extern "C"
