// pn2_common.cuh — shared device/host helpers for libpn2_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
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
// are skipped (they are served by the uniform-grid kernels of ball_query_grid.cu)
int launch_ball_query_brute(int b, int n, int m, float thr, int nsample, const float* xyz1, const float* xyz2,
                            int* idx, int* pts_cnt, const int* grid_params, int grid_stride, cudaStream_t st);

// farthest point sampling dispatch (fps.cu), shared with the fused set-abstraction layer (sa_fused.cu).
// sentinel != 0: single-CTA plans only (ask fps_single_cta first) — the kernel pre-fills `out` with -1 and
// signals programmatic launch completion so that a dependent grid can consume the picks as they appear.
int fps_dispatch(int b, int n, int m, const float* inp, float* temp, int* out, float* new_xyz, int sentinel, cudaStream_t st);
bool fps_single_cta(int b, int n);
size_t fps_scratch_bytes(int b, int n);

// ordered-sum scatter through an inverse index (interpolate.cu), shared by three_interpolate's gradient and the
// group_point / gather_point gradients: dst[b, i, :] = sum of the rows src[b, e, :] with idx[b, e] == i, e ascending, in
// float32, rounded once to T (unsigned short: f16 != 0 float16, else bfloat16).  Every dst row is written (0 if no entry
// points at it).  b clouds of ne entries over nt targets; workspace of inv_workspace_bytes(b, ne, nt) bytes.
size_t inv_workspace_bytes(int b, long long ne, int nt);
template <typename T>
int inv_sum_rows_det(int b, int ne, int c, int nt, const T* src, const int* idx, T* dst, void* workspace, int f16, cudaStream_t st);

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
