// group.cu — gather_point, group_point, their gradients, the fused sample_and_group tail and
// selection_sort, for sm_90a.
//
// Replaces (reference, tf_ops/):
//   gatherpointKernel / scatteraddpointKernel   sampling/tf_sampling_g.cu:172-192
//   group_point_gpu / group_point_grad_gpu      grouping/tf_grouping_g.cu:40-78
//   selection_sort_gpu                          grouping/tf_grouping_g.cu:83-123
// and fuses the glue of utils/pointnet_util.py:45-54 / :179-186 (pn2_group_concat).
//
// These are the HBM-bound kernels of the path.  The reference gives one thread a whole
// (nsample x c) row block, so neighbouring lanes write nsample*c*4 bytes apart.  Here the output
// is treated as one flat array: consecutive lanes write consecutive 16-byte vectors (streaming
// stores, the output is write-once), and read the matching 16 bytes of the source row (rows are
// served from L2: the source tensor is at most tens of MB).
#include <stdlib.h>

#include <type_traits>

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kCopyThreads = 256;

// ---- gather_point: out[b,j,:] = inp[b,idx[b,j],:] (3 floats) -----------------------------------
__global__ void __launch_bounds__(kCopyThreads)
gather_point_kernel(int n, int m, long long total, const float* __restrict__ inp, const int* __restrict__ idx,
                    float* __restrict__ out) {
    for (long long r = (long long)blockIdx.x * kCopyThreads + threadIdx.x; r < total;
         r += (long long)gridDim.x * kCopyThreads) {
        const long long cloud = r / m;
        const float* s = inp + (cloud * n + idx[r]) * 3;
        float* d = out + r * 3;
        d[0] = s[0];
        d[1] = s[1];
        d[2] = s[2];
    }
}

__global__ void __launch_bounds__(kCopyThreads)
gather_point_grad_kernel(int n, int m, long long total, const float* __restrict__ out_g,
                         const int* __restrict__ idx, float* __restrict__ inp_g) {
    for (long long r = (long long)blockIdx.x * kCopyThreads + threadIdx.x; r < total;
         r += (long long)gridDim.x * kCopyThreads) {
        const long long cloud = r / m;
        float* d = inp_g + (cloud * n + idx[r]) * 3;
        const float* s = out_g + r * 3;
        atomicAdd(d + 0, s[0]);
        atomicAdd(d + 1, s[1]);
        atomicAdd(d + 2, s[2]);
    }
}

// ---- group_point, vector path: c % 4 == 0, 16-byte aligned bases -------------------------------
// One thread per output float4.  rows = b*m*nsample flat rows, rows_per_cloud = m*nsample.
template <typename IndexT>
__global__ void __launch_bounds__(kCopyThreads)
group_point_vec4_kernel(int n, int c4, IndexT rows_per_cloud, IndexT total_vec, const float4* __restrict__ points,
                        const int* __restrict__ idx, float4* __restrict__ out) {
    const IndexT stride = (IndexT)gridDim.x * kCopyThreads;
    for (IndexT v = (IndexT)blockIdx.x * kCopyThreads + threadIdx.x; v < total_vec; v += stride) {
        const IndexT row = v / (IndexT)c4;
        const int l = (int)(v - row * (IndexT)c4);
        const IndexT cloud = row / rows_per_cloud;
        const int a = __ldg(idx + row);
        st_stream_f4(out + v, __ldg(points + ((size_t)cloud * n + a) * c4 + l));
    }
}

// ---- group_point, vector path, row-batched: LPR lanes per row, R rows in flight per lane-group ----
// No per-vector integer division and no load->load dependency per vector: the R row indices of a
// batch are fetched first (one broadcast load each), then every lane issues R independent 16-byte
// gathers per channel step and streams them out (cfg3 layer 2, C=320).
template <int LPR, int R>
__global__ void __launch_bounds__(kCopyThreads)
group_rows_vec4_kernel(int n, int c4, unsigned rows_per_cloud, const float4* __restrict__ points,
                       const int* __restrict__ idx, float4* __restrict__ out) {
    constexpr int RPW = 32 / LPR;  // row slots per warp
    const int lane = threadIdx.x & 31, g = lane % LPR, sub = lane / LPR;
    const unsigned cloud = blockIdx.y;
    const unsigned warps = (gridDim.x * kCopyThreads) >> 5;
    const unsigned warp = (blockIdx.x * kCopyThreads + threadIdx.x) >> 5;
    const size_t cloud_row0 = (size_t)cloud * rows_per_cloud;
    const int* __restrict__ cidx = idx + cloud_row0;
    const float4* __restrict__ cpts = points + (size_t)cloud * n * c4;
    // this lane-group walks rows r = (warp*RPW + sub)*R + rr, stride warps*RPW*R
    for (unsigned r0 = (warp * RPW + sub) * R; r0 < rows_per_cloud; r0 += warps * RPW * R) {
        const float4* __restrict__ src[R];
        float4* __restrict__ dst[R];
        bool ok[R];
#pragma unroll
        for (int rr = 0; rr < R; ++rr) {
            const unsigned r = r0 + rr;
            ok[rr] = r < rows_per_cloud;
            const int a = ok[rr] ? __ldg(cidx + r) : 0;
            src[rr] = cpts + (size_t)a * c4;
            dst[rr] = out + (cloud_row0 + r) * c4;
        }
        for (int l = g; l < c4; l += LPR) {
            float4 v[R];
#pragma unroll
            for (int rr = 0; rr < R; ++rr)
                if (ok[rr]) v[rr] = __ldg(src[rr] + l);
#pragma unroll
            for (int rr = 0; rr < R; ++rr)
                if (ok[rr]) st_stream_f4(dst[rr] + l, v[rr]);
        }
    }
}

// ---- group_point general path and the fused sample_and_group tail: LPR lanes per output row ----
// Row r of cloud `blockIdx.y` is the (3+c)- or c-wide output row of one (centroid, sample) pair:
//   HAS_XYZ: out[r, xyz_lo..xyz_lo+3) = xyz[a] - new_xyz[r / nsample]   (also to grouped_xyz if given)
//            out[r, feat_lo..feat_lo+c) = points[a]                      a = idx[r]
//   else   : out[r, 0..c) = points[a]
// LPR consecutive lanes own one row and walk its channels with stride LPR, so a warp's loads and
// stores are runs of consecutive 4-byte words (full sectors) whatever the row width; the per-row
// index/centroid loads are broadcasts.  No per-element division or branching.
// T = float, or unsigned short for both 2-byte formats: features are copied as T, the xyz channels are the float32
// differences rounded once (f16 != 0: to float16, else bfloat16; grouped_xyz stays float32).
// The 2-byte instantiations hold twice the loaded values per lane (16 bytes of 2-byte words in 8 registers); they
// are held to the CTAs per SM of the float ones (48 / 40 registers: 5 / 6 CTAs of 256 threads), without spilling.
// (0 = no bound for float: even a bound of 1 CTA changes its register allocation.)
template <int LPR, bool HAS_XYZ, typename T>
__global__ void __launch_bounds__(kCopyThreads, sizeof(T) == 4 ? 0 : (HAS_XYZ ? 5 : 6))
group_rows_kernel(int n, int c, int nsample, unsigned rows_per_cloud, const float* __restrict__ xyz,
                  const float* __restrict__ new_xyz, const T* __restrict__ points,
                  const int* __restrict__ idx, int xyz_lo, int feat_lo, T* __restrict__ out,
                  float* __restrict__ grouped_xyz, int f16) {
    constexpr int RPW = 32 / LPR;  // rows per warp per pass
    const int lane = threadIdx.x & 31, g = lane % LPR, sub = lane / LPR;
    const unsigned cloud = blockIdx.y;
    const int w = c + (HAS_XYZ ? 3 : 0);
    const unsigned warps = (gridDim.x * kCopyThreads) >> 5;
    const unsigned warp = (blockIdx.x * kCopyThreads + threadIdx.x) >> 5;
    const size_t cloud_row0 = (size_t)cloud * rows_per_cloud;
    const int* __restrict__ cidx = idx + cloud_row0;
    const T* __restrict__ cpts = points ? points + (size_t)cloud * n * c : nullptr;
    const float* __restrict__ cxyz = HAS_XYZ ? xyz + (size_t)cloud * n * 3 : nullptr;
    // R rows per lane group and trip, U words per row and lane in flight: what limits these copies is bytes in
    // flight per SM (measured: 32 KB/SM -> 3.5 TB/s, 64 KB/SM -> 5.5 TB/s for the same gather), so all R*U loads of a
    // trip are issued before the first store.  U * sizeof(T) = 16 bytes per row and lane whatever the element size.
    // measured (float) at C = 320 + 3: R = 2: 58 / 94 / 172 us (38 registers); R = 4: 66 / 103 / 180 us (58 registers)
    constexpr int R = 2, U = 16 / (int)sizeof(T);
    for (unsigned r0 = (warp * RPW + sub) * R; r0 < rows_per_cloud; r0 += warps * RPW * R) {
        const T* __restrict__ src[R];
        T* __restrict__ d[R];
        bool ok[R];
#pragma unroll
        for (int rr = 0; rr < R; ++rr) {
            const unsigned r = r0 + rr;
            ok[rr] = r < rows_per_cloud;
            const int a = ok[rr] ? __ldg(cidx + r) : 0;
            T* __restrict__ dst = out + (cloud_row0 + r) * w;
            src[rr] = cpts ? cpts + (size_t)a * c : nullptr;
            d[rr] = dst + feat_lo;
            if (HAS_XYZ && ok[rr] && g < 3) {
                const size_t ctr = (size_t)cloud * (rows_per_cloud / (unsigned)nsample) + r / (unsigned)nsample;  // global centroid index
                const float v = __fsub_rn(__ldg(cxyz + (size_t)a * 3 + g), __ldg(new_xyz + ctr * 3 + g));
                __stcs(dst + xyz_lo + g, of_f32<T>(v, f16));
                if (grouped_xyz) __stcs(grouped_xyz + (cloud_row0 + r) * 3 + g, v);
            }
        }
        for (int l0 = g; l0 < c; l0 += LPR * U) {
            T v[R][U];
#pragma unroll
            for (int rr = 0; rr < R; ++rr)
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (ok[rr] && l0 + u * LPR < c) v[rr][u] = __ldg(src[rr] + l0 + u * LPR);
#pragma unroll
            for (int rr = 0; rr < R; ++rr)
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (ok[rr] && l0 + u * LPR < c) __stcs(d[rr] + l0 + u * LPR, v[rr][u]);
        }
    }
}

// ---- the fused sample_and_group tail with features, c % 4 == 0: 16-byte gathers AND 16-byte stores ----
// Output rows are w = 3 + c floats wide (67, 131, 259, 323 in the reference's networks), so a row's feature
// segment starts 0..3 floats past a 16-byte boundary — differently for every row.  The source rows ARE
// aligned (c % 4 == 0): lane k of the row's lane group loads source vector k (LDG.128); the output vector
// that starts `head` floats into the segment is the last 4-head floats of source vector k followed by the
// first head floats of vector k+1, which the lane gets from its neighbour by shuffle (the last lane of a
// pass loads it).  So the body of every row goes out as aligned STG.128 with the data re-aligned in
// registers; only the <= 3 head floats, <= 3 tail floats and the 3 xyz floats of a row are scalar stores.
// Round 1's kernel moved every float with a 4-byte load and a 4-byte store: 4x the LSU instructions, 42-54 %
// of the HBM peak at C = 320 where the aligned C % 4 == 0 gather (same bytes) reaches 84 %.
// R rows are in flight per lane group (all their gathers are issued before the first store).
template <int LPR, int R>
__global__ void __launch_bounds__(kCopyThreads, 4)  // <= 64 registers: at 114 (R = 4, unbounded) occupancy fell to 25 % and the kernel with it
group_concat_vec_kernel(int n, int c4, int nsample, unsigned rows_per_cloud, const float* __restrict__ xyz,
                        const float* __restrict__ new_xyz, const float4* __restrict__ points, const int* __restrict__ idx,
                        int xyz_lo, int feat_lo, float* __restrict__ out, float* __restrict__ grouped_xyz) {
    constexpr int RPW = 32 / LPR;
    const int lane = threadIdx.x & 31, g = lane % LPR, sub = lane / LPR;
    const unsigned cloud = blockIdx.y;
    const unsigned warps = (gridDim.x * kCopyThreads) >> 5;
    const unsigned warp = (blockIdx.x * kCopyThreads + threadIdx.x) >> 5;
    const size_t cloud_row0 = (size_t)cloud * rows_per_cloud;
    const unsigned m = rows_per_cloud / (unsigned)nsample;
    const int c = 4 * c4;
    const size_t w = (size_t)c + 3;
    const int* __restrict__ cidx = idx + cloud_row0;
    const float4* __restrict__ cpts = points + (size_t)cloud * n * c4;
    const float* __restrict__ cxyz = xyz + (size_t)cloud * n * 3;
    const float* __restrict__ cctr = new_xyz + (size_t)cloud * m * 3;
    for (unsigned r0 = (warp * RPW + sub) * R; r0 < rows_per_cloud; r0 += warps * RPW * R) {
        const float4* __restrict__ src[R];
        float* __restrict__ fdst[R];  // start of the row's feature segment
        int head[R];
        bool ok[R];
#pragma unroll
        for (int rr = 0; rr < R; ++rr) {
            const unsigned r = r0 + rr;
            ok[rr] = r < rows_per_cloud;
            const int a = ok[rr] ? __ldg(cidx + r) : 0;
            src[rr] = cpts + (size_t)a * c4;
            const size_t obase = (cloud_row0 + r) * w;
            fdst[rr] = out + obase + feat_lo;
            head[rr] = (int)((4u - (unsigned)((obase + (size_t)feat_lo) & 3u)) & 3u);
            // The row's scalar words — 3 centred xyz, `head` floats in front of the first aligned vector and 4-head
            // behind the last one — go out as ONE predicated store instruction: lane t < 3 takes xyz[t], the next
            // `head` lanes the head floats, the next 4-head lanes the tail floats (7 lanes at most).  (One store
            // instruction per word, as a first version did, is 9 store instructions per row against the 2.5 that
            // move the row's 80 vectors: the LSU queue, not the bytes, set the pace.)
            if (ok[rr] && g < 7) {
                const int h = head[rr];
                float* dst = nullptr;
                float val = 0.f;
                if (g < 3) {
                    val = __fsub_rn(__ldg(cxyz + (size_t)a * 3 + g), __ldg(cctr + (size_t)(r / (unsigned)nsample) * 3 + g));
                    dst = out + obase + xyz_lo + g;
                    if (grouped_xyz) __stcs(grouped_xyz + (cloud_row0 + r) * 3 + g, val);
                } else if (h != 0) {
                    const int t = g - 3;                  // 0..3
                    const int e = t < h ? t : c - 4 + t;  // head float t, or the tail float (c - 4) + t for t >= h
                    val = __ldg(reinterpret_cast<const float*>(src[rr]) + e);
                    dst = fdst[rr] + e;
                }
                if (dst) __stcs(dst, val);
            }
        }
        for (int k0 = 0; k0 < c4; k0 += LPR) {
            const int k = k0 + g;
            float4 v[R];
            float3 nx[R];
#pragma unroll
            for (int rr = 0; rr < R; ++rr) {
                v[rr] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ok[rr] && k < c4) v[rr] = __ldg(src[rr] + k);
            }
#pragma unroll
            for (int rr = 0; rr < R; ++rr) {
                nx[rr].x = __shfl_down_sync(kFullMask, v[rr].x, 1, LPR);
                nx[rr].y = __shfl_down_sync(kFullMask, v[rr].y, 1, LPR);
                nx[rr].z = __shfl_down_sync(kFullMask, v[rr].z, 1, LPR);
                if (g == LPR - 1 && ok[rr] && k + 1 < c4 && head[rr] != 0) {  // next pass's first vector
                    const float4 t = __ldg(src[rr] + k + 1);
                    nx[rr] = make_float3(t.x, t.y, t.z);
                }
            }
#pragma unroll
            for (int rr = 0; rr < R; ++rr) {
                if (!ok[rr] || k >= c4) continue;
                const int h = head[rr];
                float* __restrict__ d = fdst[rr];
                if (h == 0) {
                    st_stream_f4(reinterpret_cast<float4*>(d) + k, v[rr]);
                    continue;
                }
                if (k + 1 < c4) {  // aligned body vector: floats [h + 4k, h + 4k + 4) of the segment
                    float4 o;
                    o.x = h == 1 ? v[rr].y : (h == 2 ? v[rr].z : v[rr].w);
                    o.y = h == 1 ? v[rr].z : (h == 2 ? v[rr].w : nx[rr].x);
                    o.z = h == 1 ? v[rr].w : (h == 2 ? nx[rr].x : nx[rr].y);
                    o.w = h == 1 ? nx[rr].x : (h == 2 ? nx[rr].y : nx[rr].z);
                    st_stream_f4(reinterpret_cast<float4*>(d + h + 4 * k), o);
                }  // (the head floats [0, h) and the tail floats behind the last aligned vector were written above)
            }
        }
    }
}

// Narrow rows (w <= 4 floats, e.g. group_point(xyz) and the C=0 sample_and_group tail): one thread
// per output row — the per-row index/centroid work is the cost, not the copy.
template <bool HAS_XYZ, typename T>
__global__ void __launch_bounds__(kCopyThreads)
group_narrow_kernel(int n, int c, int nsample, unsigned rows_per_cloud, const float* __restrict__ xyz,
                    const float* __restrict__ new_xyz, const T* __restrict__ points,
                    const int* __restrict__ idx, T* __restrict__ out, float* __restrict__ grouped_xyz, int f16) {
    const unsigned cloud = blockIdx.y;
    const size_t cloud_row0 = (size_t)cloud * rows_per_cloud;
    const int* __restrict__ cidx = idx + cloud_row0;
    const unsigned m = rows_per_cloud / (unsigned)nsample;
    for (unsigned r = blockIdx.x * kCopyThreads + threadIdx.x; r < rows_per_cloud; r += gridDim.x * kCopyThreads) {
        const int a = __ldg(cidx + r);
        if (HAS_XYZ) {  // c == 0: the row is the centred xyz
            const float* __restrict__ s = xyz + ((size_t)cloud * n + a) * 3;
            const float* __restrict__ ctr = new_xyz + ((size_t)cloud * m + r / (unsigned)nsample) * 3;
            const float v0 = __fsub_rn(__ldg(s), __ldg(ctr)), v1 = __fsub_rn(__ldg(s + 1), __ldg(ctr + 1)),
                        v2 = __fsub_rn(__ldg(s + 2), __ldg(ctr + 2));
            T* __restrict__ d = out + (cloud_row0 + r) * 3;
            __stcs(d, of_f32<T>(v0, f16)); __stcs(d + 1, of_f32<T>(v1, f16)); __stcs(d + 2, of_f32<T>(v2, f16));
            if (grouped_xyz) {
                float* __restrict__ gq = grouped_xyz + (cloud_row0 + r) * 3;
                __stcs(gq, v0); __stcs(gq + 1, v1); __stcs(gq + 2, v2);
            }
        } else {
            const T* __restrict__ s = points + ((size_t)cloud * n + a) * c;
            T* __restrict__ d = out + (cloud_row0 + r) * c;
            for (int l = 0; l < c; ++l) __stcs(d + l, __ldg(s + l));
        }
    }
}

template <bool HAS_XYZ, typename T>
static int launch_group_rows(int b, int n, int c, int m, int nsample, const float* xyz, const float* new_xyz,
                             const T* points, const int* idx, int xyz_lo, int feat_lo, T* out,
                             float* grouped_xyz, int f16, cudaStream_t st) {
    const unsigned rpc = (unsigned)m * (unsigned)nsample;
    const int w = c + (HAS_XYZ ? 3 : 0);
    if (w <= 4 && (!HAS_XYZ || c == 0)) {
        unsigned gx = (rpc + kCopyThreads - 1) / kCopyThreads;
        const unsigned cap = ((unsigned)num_sms() * 16u + b - 1) / b;
        if (gx > cap) gx = cap;
        group_narrow_kernel<HAS_XYZ, T><<<dim3(gx, b, 1), kCopyThreads, 0, st>>>(n, c, nsample, rpc, xyz, new_xyz, points, idx, out,
                                                                                grouped_xyz, f16);
        return finish_launch();
    }
    if (std::is_same<T, float>::value && HAS_XYZ && c >= 8 && c <= 64 && c % 4 == 0 && aligned_to(points, 16) && aligned_to(out, 16)) {
        // vectorised tail (see group_concat_vec_kernel).  Measured: it wins at C = 64 (30.7 against 35.6 us, cfg4 SA256) and
        // loses to the row kernel below from C = 128 up (C = 320 + 3, S = 64: 125 against 94 us), so only narrow rows take it
        // c4 <= 16 <= LPR: one pass over the row's vectors, so the last lane never loads a next pass's first vector
        const int c4 = c / 4;
        const int lpr = c4 <= 8 ? 8 : 16;
        constexpr int R = 2;
        const unsigned rows_per_block = (kCopyThreads / 32) * (32 / lpr) * R;
        unsigned gx = (rpc + rows_per_block - 1) / rows_per_block;
        const unsigned cap = ((unsigned)num_sms() * 32u + b - 1) / b;
        if (gx > cap) gx = cap;
        if (gx < 1) gx = 1;
        dim3 grid(gx, b, 1);
        const float4* p4 = reinterpret_cast<const float4*>(points);
        float* o = reinterpret_cast<float*>(out);  // (float here: the condition above)
        if (lpr == 8) group_concat_vec_kernel<8, R><<<grid, kCopyThreads, 0, st>>>(n, c4, nsample, rpc, xyz, new_xyz, p4, idx, xyz_lo, feat_lo, o, grouped_xyz);
        else group_concat_vec_kernel<16, R><<<grid, kCopyThreads, 0, st>>>(n, c4, nsample, rpc, xyz, new_xyz, p4, idx, xyz_lo, feat_lo, o, grouped_xyz);
        return finish_launch();
    }
    const int lpr = w <= 4 ? 4 : (w <= 8 ? 8 : (w <= 16 ? 16 : 32));
    const unsigned rows_per_block = (kCopyThreads / 32) * (32 / lpr) * 2;  // R = 2 rows per lane group and trip
    unsigned gx = (rpc + rows_per_block - 1) / rows_per_block;
    const unsigned cap = ((unsigned)num_sms() * 32u + b - 1) / b;  // enough CTAs to fill the machine, then grid-stride
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    dim3 grid(gx, b, 1);
#define PN2_GROUP_ROWS(L) \
    group_rows_kernel<L, HAS_XYZ, T><<<grid, kCopyThreads, 0, st>>>(n, c, nsample, rpc, xyz, new_xyz, points, idx, xyz_lo, feat_lo, out, grouped_xyz, f16)
    if (lpr == 4) PN2_GROUP_ROWS(4);
    else if (lpr == 8) PN2_GROUP_ROWS(8);
    else if (lpr == 16) PN2_GROUP_ROWS(16);
    else PN2_GROUP_ROWS(32);
#undef PN2_GROUP_ROWS
    return finish_launch();
}

// ---- group_point_grad: atomic scatter-add (vector red.global.add.v4.f32 when c % 4 == 0) -------
// T: element type of grad_out (read and upcast 4 at a time); the accumulator is always float32
template <typename IndexT, typename T>
__global__ void __launch_bounds__(kCopyThreads)
group_point_grad_vec4_kernel(int n, int c4, IndexT rows_per_cloud, IndexT total_vec,
                             const T* __restrict__ grad_out, const int* __restrict__ idx,
                             float4* __restrict__ grad_points) {
    const IndexT stride = (IndexT)gridDim.x * kCopyThreads;
    for (IndexT v = (IndexT)blockIdx.x * kCopyThreads + threadIdx.x; v < total_vec; v += stride) {
        const IndexT row = v / (IndexT)c4;
        const int l = (int)(v - row * (IndexT)c4);
        const IndexT cloud = row / rows_per_cloud;
        const int a = __ldg(idx + row);
        const float4 g = ldcs4(grad_out + (size_t)v * 4);
        atomicAdd(grad_points + ((size_t)cloud * n + a) * c4 + l, g);  // red.global.add.v4.f32 (sm_90+)
    }
}

template <typename IndexT, typename T>
__global__ void __launch_bounds__(kCopyThreads)
group_point_grad_scalar_kernel(int n, int c, IndexT rows_per_cloud, IndexT total,
                               const T* __restrict__ grad_out, const int* __restrict__ idx,
                               float* __restrict__ grad_points) {
    const IndexT stride = (IndexT)gridDim.x * kCopyThreads;
    for (IndexT e = (IndexT)blockIdx.x * kCopyThreads + threadIdx.x; e < total; e += stride) {
        const IndexT row = e / (IndexT)c;
        const int l = (int)(e - row * (IndexT)c);
        const IndexT cloud = row / rows_per_cloud;
        const int a = __ldg(idx + row);
        atomicAdd(grad_points + ((size_t)cloud * n + a) * c + l, to_f32(__ldcs(grad_out + e)));
    }
}

// the float32 gradient accumulator rounded once to the feature type
template <typename T>
__global__ void __launch_bounds__(kCopyThreads)
round_to_kernel(unsigned long long total, const float* __restrict__ src, T* __restrict__ dst) {
    for (unsigned long long e = (unsigned long long)blockIdx.x * kCopyThreads + threadIdx.x; e < total;
         e += (unsigned long long)gridDim.x * kCopyThreads)
        dst[e] = from_f32<T>(__ldcs(src + e));
}

// ---- selection_sort: one warp per (b,m) row ------------------------------------------------------
// k rounds of "find the first minimum of v[s..n) (strict '<'), swap it into position s", indices
// carried along — the same permutation the reference's thread-per-row loop produces, with the
// argmin parallelised across the warp on the key (value, position).
// NaN, as the reference's scan `if (v[t] < v[min]) min = t` from min = s treats it: a NaN at v[s]
// is never replaced (nothing is '<' NaN), so the round keeps s; otherwise NaN candidates are
// never taken, and the round picks the first minimum of the non-NaN values.
__global__ void __launch_bounds__(kCopyThreads)
selection_sort_kernel(int n, int k, long long rows, const float* __restrict__ dist, int* __restrict__ outi,
                      float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * kCopyThreads + threadIdx.x) >> 5;
    if (warp >= rows) return;
    const float* src = dist + warp * n;
    float* v = out + warp * n;
    int* ix = outi + warp * n;
    for (int s = lane; s < n; s += 32) {
        v[s] = src[s];
        ix[s] = s;
    }
    __syncwarp();
    const int rounds = k < n ? k : n;
    for (int s = 0; s < rounds; ++s) {
        const float vs = v[s];
        if (vs != vs) continue;  // warp-uniform: v[s] is NaN, the round keeps s
        float bv = 0.f;
        int bt = -1;
        for (int t = s + lane; t < n; t += 32) {
            const float x = v[t];
            if (bt < 0 ? x == x : x < bv) {  // ascending t within a lane: strict '<' keeps the earliest; NaN never
                bv = x;
                bt = t;
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float ov = __shfl_xor_sync(kFullMask, bv, off);
            const int ot = __shfl_xor_sync(kFullMask, bt, off);
            // total order on non-NaN (value, position); lanes without candidates carry bt = -1
            const bool take = (ot >= 0) && (bt < 0 || ov < bv || (ov == bv && ot < bt));
            if (take) {
                bv = ov;
                bt = ot;
            }
        }
        if (lane == 0 && bt != s && bt >= 0) {
            const float tv = v[bt];
            v[bt] = v[s];
            v[s] = tv;
            const int ti = ix[bt];
            ix[bt] = ix[s];
            ix[s] = ti;
        }
        __syncwarp();
    }
}

// Tuning hooks of group_point's 16-byte path, read from the environment once: PN2_GROUP_MODE 0 = row-batched (default),
// 1 = flat one-vector-per-thread; PN2_GROUP_CTAS = CTAs per SM (default 16).
struct GroupTuning {
    int mode, ctas_per_sm;
};
static const GroupTuning& group_tuning() {
    static const GroupTuning t = [] {  // thread-safe: runs once
        const char* e = getenv("PN2_GROUP_MODE");
        const char* gq = getenv("PN2_GROUP_CTAS");
        return GroupTuning{e ? atoi(e) : 0, gq ? atoi(gq) : 16};
    }();
    return t;
}

// ---- entry bodies, one per element type T (float, __nv_bfloat16, __half) ----------------------------
// The 16-byte vector kernels copy bytes, so they serve every T: a row of c elements is c * sizeof(T) / 16 vectors
// (c % 4 == 0 for float, c % 8 == 0 for the 2-byte types); other widths and misaligned bases take the row kernels.
template <typename T>
static int group_point_impl(int b, int n, int c, int m, int nsample, const T* points, const int* idx, T* out,
                            cudaStream_t st) {
    const unsigned long long rows = (unsigned long long)b * m * nsample;
    const unsigned long long rpc = (unsigned long long)m * nsample;
    if (((size_t)c * sizeof(T)) % 16 == 0 && aligned_to(points, 16) && aligned_to(out, 16)) {
        const int c4 = (int)((size_t)c * sizeof(T) / 16);  // 16-byte vectors per row
        const unsigned long long tv = rows * c4;
        const GroupTuning& tune = group_tuning();
        const float4* p4 = reinterpret_cast<const float4*>(points);
        float4* o4 = reinterpret_cast<float4*>(out);
        if (tune.mode == 0 && rpc < (1ull << 32) && b <= 65535) {
            const int lpr = c4 <= 4 ? 4 : (c4 <= 8 ? 8 : (c4 <= 16 ? 16 : 32));
            constexpr int R = 4;
            const unsigned rows_per_block = (kCopyThreads / 32) * (32 / lpr) * R;
            unsigned gx = (unsigned)((rpc + rows_per_block - 1) / rows_per_block);
            const unsigned cap = ((unsigned)num_sms() * (unsigned)tune.ctas_per_sm + b - 1) / b;
            if (gx > cap) gx = cap;
            if (gx < 1) gx = 1;
            dim3 grid(gx, b, 1);
            if (lpr == 4) group_rows_vec4_kernel<4, R><<<grid, kCopyThreads, 0, st>>>(n, c4, (unsigned)rpc, p4, idx, o4);
            else if (lpr == 8) group_rows_vec4_kernel<8, R><<<grid, kCopyThreads, 0, st>>>(n, c4, (unsigned)rpc, p4, idx, o4);
            else if (lpr == 16) group_rows_vec4_kernel<16, R><<<grid, kCopyThreads, 0, st>>>(n, c4, (unsigned)rpc, p4, idx, o4);
            else group_rows_vec4_kernel<32, R><<<grid, kCopyThreads, 0, st>>>(n, c4, (unsigned)rpc, p4, idx, o4);
            return finish_launch();
        }
        unsigned long long blocks = (tv + kCopyThreads - 1) / kCopyThreads;
        const unsigned long long cap = (unsigned long long)num_sms() * (unsigned long long)tune.ctas_per_sm;
        const unsigned grid = (unsigned)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
        if (tv < (1ull << 31))
            group_point_vec4_kernel<unsigned><<<grid, kCopyThreads, 0, st>>>(n, c4, (unsigned)rpc, (unsigned)tv, p4, idx, o4);
        else
            group_point_vec4_kernel<unsigned long long><<<grid, kCopyThreads, 0, st>>>(n, c4, rpc, tv, p4, idx, o4);
    } else {
        if (rpc >= (1ull << 32) || b > 65535) return (int)cudaErrorInvalidValue;
        return launch_group_rows<false, T>(b, n, c, m, nsample, nullptr, nullptr, points, idx, 0, 0, out, nullptr, 0, st);
    }
    return finish_launch();
}

// scatter-add of grad_out (T) into the float32 accumulator (b,n,c)
template <typename T>
static int group_point_grad_impl(int b, int n, int c, int m, int nsample, const T* grad_out, const int* idx,
                                 float* accum, cudaStream_t st) {
    const unsigned long long total = (unsigned long long)b * m * nsample * c;
    const unsigned long long rpc = (unsigned long long)m * nsample;
    if (c % 4 == 0 && aligned_to(grad_out, 4 * sizeof(T)) && aligned_to(accum, 16)) {
        const unsigned long long tv = total / 4;
        const unsigned grid = grid_for(tv, kCopyThreads);
        if (tv < (1ull << 31))
            group_point_grad_vec4_kernel<unsigned, T><<<grid, kCopyThreads, 0, st>>>(
                n, c / 4, (unsigned)rpc, (unsigned)tv, grad_out, idx, (float4*)accum);
        else
            group_point_grad_vec4_kernel<unsigned long long, T><<<grid, kCopyThreads, 0, st>>>(
                n, c / 4, rpc, tv, grad_out, idx, (float4*)accum);
    } else {
        const unsigned grid = grid_for(total, kCopyThreads);
        if (total < (1ull << 31))
            group_point_grad_scalar_kernel<unsigned, T><<<grid, kCopyThreads, 0, st>>>(n, c, (unsigned)rpc, (unsigned)total, grad_out, idx, accum);
        else
            group_point_grad_scalar_kernel<unsigned long long, T><<<grid, kCopyThreads, 0, st>>>(n, c, rpc, total, grad_out, idx, accum);
    }
    return finish_launch();
}

template <typename T>
static int group_point_grad_round_impl(int b, int n, int c, int m, int nsample, const void* grad_out, const int* idx,
                                       void* grad_points, float* accum, cudaStream_t st) {
    int rc = group_point_grad_impl<T>(b, n, c, m, nsample, static_cast<const T*>(grad_out), idx, accum, st);
    if (rc != 0) return rc;
    const unsigned long long total = (unsigned long long)b * n * c;
    round_to_kernel<T><<<grid_for(total, kCopyThreads), kCopyThreads, 0, st>>>(total, accum, static_cast<T*>(grad_points));
    return finish_launch();
}

// the ordered-sum gradient (no atomics): T = float, or unsigned short for both 2-byte formats (f16 selects float16)
template <typename T>
static int group_point_grad_det_impl(int b, int n, int c, int m, int nsample, const T* grad_out, const int* idx,
                                     T* grad_points, void* workspace, size_t workspace_bytes, int f16, cudaStream_t st) {
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * n * c == 0) return 0;
    if (!grad_points) return (int)cudaErrorInvalidValue;
    const long long ne = (long long)m * nsample;  // entries per cloud
    if (ne == 0) return (int)cudaMemsetAsync(grad_points, 0, sizeof(T) * (size_t)b * n * c, st);
    if (!grad_out || !idx || !workspace) return (int)cudaErrorInvalidValue;
    if (ne > 0x7fffffffLL || workspace_bytes < inv_workspace_bytes(b, ne, n)) return (int)cudaErrorInvalidValue;
    return inv_scatter_det<false, T>(b, (int)ne, (int)ne, c, n, grad_out, idx, nullptr, nullptr, grad_points, workspace, f16, st);
}

template <typename T>
static int group_concat_impl(int b, int n, int c, int m, int nsample, const float* xyz, const float* new_xyz,
                             const void* points, const int* idx, int xyz_first, void* out, float* grouped_xyz, int f16,
                             cudaStream_t st) {
    const unsigned long long rpc = (unsigned long long)m * nsample;
    if (rpc >= (1ull << 32) || b > 65535) return (int)cudaErrorInvalidValue;
    const int xyz_lo = xyz_first ? 0 : c, feat_lo = xyz_first ? 3 : 0;
    return launch_group_rows<true, T>(b, n, c, m, nsample, xyz, new_xyz, static_cast<const T*>(points), idx, xyz_lo,
                                      feat_lo, static_cast<T*>(out), grouped_xyz, f16, st);
}

}  // namespace pn2

extern "C" {

int pn2_gather_point(int b, int n, int m, const float* inp, const int* idx, float* out, void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || m < 0) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!inp || !idx || !out) return (int)cudaErrorInvalidValue;
    const long long total = (long long)b * m;
    gather_point_kernel<<<grid_for(total, kCopyThreads), kCopyThreads, 0, as_stream(stream)>>>(n, m, total, inp, idx, out);
    return finish_launch();
}

int pn2_gather_point_grad(int b, int n, int m, const float* out_g, const int* idx, float* inp_g, void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || m < 0) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!out_g || !idx || !inp_g) return (int)cudaErrorInvalidValue;
    const long long total = (long long)b * m;
    gather_point_grad_kernel<<<grid_for(total, kCopyThreads), kCopyThreads, 0, as_stream(stream)>>>(n, m, total, out_g, idx, inp_g);
    return finish_launch();
}

int pn2_gather_point_grad_det(int b, int n, int m, const float* out_g, const int* idx, float* inp_g, void* workspace,
                              size_t workspace_bytes, void* stream) {
    return pn2::group_point_grad_det_impl<float>(b, n, 3, m, 1, out_g, idx, inp_g, workspace, workspace_bytes, 0,
                                                 pn2::as_stream(stream));
}

int pn2_group_point(int b, int n, int c, int m, int nsample, const float* points, const int* idx, float* out,
                    void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * m * nsample * c == 0) return 0;
    if (!points || !idx || !out) return (int)cudaErrorInvalidValue;
    return group_point_impl<float>(b, n, c, m, nsample, points, idx, out, as_stream(stream));
}

int pn2_group_point_typed(int dtype, int b, int n, int c, int m, int nsample, const void* points, const int* idx,
                          void* out, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32) return pn2_group_point(b, n, c, m, nsample, static_cast<const float*>(points), idx, static_cast<float*>(out), stream);
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * m * nsample * c == 0) return 0;
    if (!points || !idx || !out) return (int)cudaErrorInvalidValue;
    // a bit copy: bfloat16 and float16 are both moved as unsigned short
    return group_point_impl<unsigned short>(b, n, c, m, nsample, static_cast<const unsigned short*>(points), idx,
                                            static_cast<unsigned short*>(out), as_stream(stream));
}

int pn2_group_point_grad(int b, int n, int c, int m, int nsample, const float* grad_out, const int* idx,
                         float* grad_points, void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * m * nsample * c == 0) return 0;
    if (!grad_out || !idx || !grad_points) return (int)cudaErrorInvalidValue;
    return group_point_grad_impl<float>(b, n, c, m, nsample, grad_out, idx, grad_points, as_stream(stream));
}

int pn2_group_point_grad_typed(int dtype, int b, int n, int c, int m, int nsample, const void* grad_out,
                               const int* idx, void* grad_points, float* accum, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32)
        return pn2_group_point_grad(b, n, c, m, nsample, static_cast<const float*>(grad_out), idx, static_cast<float*>(grad_points), stream);
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    if ((unsigned long long)b * m * nsample * c == 0) return 0;
    if (!grad_out || !idx || !grad_points || !accum) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_BF16)
        return group_point_grad_round_impl<__nv_bfloat16>(b, n, c, m, nsample, grad_out, idx, grad_points, accum, as_stream(stream));
    return group_point_grad_round_impl<__half>(b, n, c, m, nsample, grad_out, idx, grad_points, accum, as_stream(stream));
}

size_t pn2_group_point_grad_det_workspace_bytes(int b, int n, int m, int nsample) {
    if (b <= 0 || n <= 0 || m <= 0 || nsample <= 0) return 0;
    return pn2::inv_workspace_bytes(b, (long long)m * nsample, n);
}

int pn2_group_point_grad_det(int b, int n, int c, int m, int nsample, const float* grad_out, const int* idx,
                             float* grad_points, void* workspace, size_t workspace_bytes, void* stream) {
    return pn2::group_point_grad_det_impl<float>(b, n, c, m, nsample, grad_out, idx, grad_points, workspace, workspace_bytes, 0,
                                                 pn2::as_stream(stream));
}

int pn2_group_point_grad_det_typed(int dtype, int b, int n, int c, int m, int nsample, const void* grad_out,
                                   const int* idx, void* grad_points, void* workspace, size_t workspace_bytes,
                                   void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    using U16 = unsigned short;  // bfloat16 and float16 share one instance: dtype == PN2_F16 selects the format
    if (dtype == PN2_F32)
        return group_point_grad_det_impl<float>(b, n, c, m, nsample, static_cast<const float*>(grad_out), idx,
                                                static_cast<float*>(grad_points), workspace, workspace_bytes, 0, as_stream(stream));
    return group_point_grad_det_impl<U16>(b, n, c, m, nsample, static_cast<const U16*>(grad_out), idx, static_cast<U16*>(grad_points),
                                          workspace, workspace_bytes, dtype == PN2_F16, as_stream(stream));
}

int pn2_group_concat(int b, int n, int c, int m, int nsample, const float* xyz, const float* new_xyz,
                     const float* points, const int* idx, int xyz_first, float* out, float* grouped_xyz,
                     void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    const unsigned long long rpc = (unsigned long long)m * nsample;
    if (b == 0 || rpc == 0) return 0;
    if (!xyz || !new_xyz || !idx || !out || (c > 0 && !points)) return (int)cudaErrorInvalidValue;
    return group_concat_impl<float>(b, n, c, m, nsample, xyz, new_xyz, points, idx, xyz_first, out, grouped_xyz, 0, as_stream(stream));
}

int pn2_group_concat_typed(int dtype, int b, int n, int c, int m, int nsample, const float* xyz,
                           const float* new_xyz, const void* points, const int* idx, int xyz_first, void* out,
                           float* grouped_xyz, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    if (dtype == PN2_F32)
        return pn2_group_concat(b, n, c, m, nsample, xyz, new_xyz, static_cast<const float*>(points), idx, xyz_first,
                                static_cast<float*>(out), grouped_xyz, stream);
    if (b < 0 || n <= 0 || c < 0 || m < 0 || nsample < 0) return (int)cudaErrorInvalidValue;
    const unsigned long long rpc = (unsigned long long)m * nsample;
    if (b == 0 || rpc == 0) return 0;
    if (!xyz || !new_xyz || !idx || !out || (c > 0 && !points)) return (int)cudaErrorInvalidValue;
    // bfloat16 and float16 share one instance: dtype == PN2_F16 selects the format of the xyz channels
    return group_concat_impl<unsigned short>(b, n, c, m, nsample, xyz, new_xyz, points, idx, xyz_first, out, grouped_xyz,
                                             dtype == PN2_F16, as_stream(stream));
}

int pn2_selection_sort(int b, int n, int m, int k, const float* dist, int* outi, float* out, void* stream) {
    using namespace pn2;
    if (b < 0 || n <= 0 || m < 0 || k <= 0) return (int)cudaErrorInvalidValue;
    const long long rows = (long long)b * m;
    if (rows == 0) return 0;
    if (!dist || !outi || !out) return (int)cudaErrorInvalidValue;
    const unsigned long long blocks = ((unsigned long long)rows * 32 + kCopyThreads - 1) / kCopyThreads;
    if (blocks > 0x7fffffffull) return (int)cudaErrorInvalidValue;
    selection_sort_kernel<<<(unsigned)blocks, kCopyThreads, 0, as_stream(stream)>>>(n, k, rows, dist, outi, out);
    return finish_launch();
}

}  // extern "C"
