// render.cu — the reference's point-cloud viewer on the GPU: z-buffered ball splats (utils/render_balls_so.cpp
// render_ball) over a ragged batch of clouds, and showpoints' view transform (utils/show3d_balls.py:27-29, 52-74).
// DESIGN.md §6.16.
//
// pn2_render_balls: one memset and three launches per call, nothing read back:
//   zrange:  grid (point chunks, B): each image's min and max z over its real points, as integer atomicMax on biased
//            keys in the workspace tail;
//   splat:   grid (point chunks, B): every (point, pattern entry) pair that lands on the canvas forms the 64-bit key
//            (z2 biased | ~i) and atomicMax-es it into its pixel, unless a plain read shows a key it cannot beat;
//   resolve: grid (pixel chunks, B): the key names the winning point; its pattern entry, shade and intensity are
//            recomputed in the reference's arithmetic order, or the background is written where no key was set.
// A point reaches a pixel through at most one pattern entry, so the reference's sequential z-buffer (strict depth test,
// points in index order) leaves each pixel to the contribution of largest z2 and, among equal z2, of lowest index: the
// largest key.  Every atomic is an integer one, so the images do not depend on the order of the threads.
//
// pn2_project_points: one CTA per cloud computes the float64 mean and scale in a fixed order, then a grid over
// (point chunks, B) applies the caller's rotations.
#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kRenderThreads = 256;
constexpr int kZrangeChunk = 4096;        // points per CTA of the zrange pass
constexpr int kSplatPairs = 4096;         // (point, pattern entry) pairs per CTA of the splat pass (at least one point)
constexpr int kMaxRadius = 4096;          // r^2 < 2^24: the pattern's integer square roots are exact in float
constexpr int kMaxImages = 65535;         // grid.y
constexpr int kDepthInit = -2100000000;   // render_balls_so.cpp: the z-buffer's initial depth; the test is strict
constexpr int kStatsThreads = 1024;
constexpr int kProjectThreads = 256;
constexpr int kMaxViewsPerLaunch = 32;    // rotations passed by value: 32 x 9 doubles of kernel parameters
constexpr double kMaxCoord = 1073741824.0;  // 2^30: projected coordinates are clamped to the renderer's contract

__device__ __forceinline__ unsigned bias(int v) { return (unsigned)v ^ 0x80000000u; }
__device__ __forceinline__ int unbias(unsigned u) { return (int)(u ^ 0x80000000u); }

// floor(sqrt(k)) for 0 < k < 2^24 (k and the square root are exact in float up to one step, fixed by the test).  It
// equals the reference's int(sqrt(double(k))): below 2^24 no sqrt(m^2 - 1) rounds up to m in double.
__device__ __forceinline__ int isqrt(int k) {
    int s = (int)__fsqrt_rn((float)k);
    if (s * s > k) --s;
    else if ((s + 1) * (s + 1) <= k) ++s;
    return s;
}

// double -> unsigned char as x86-64 g++ converts it: cvttsd2si to int32 (0x80000000 outside its range or on NaN),
// then the low byte.  Equal to truncation for values in [0, 256).
__device__ __forceinline__ unsigned char x86_u8(double v) {
    const int i = (v > -2147483649.0 && v < 2147483648.0) ? __double2int_rz(v) : (int)0x80000000;
    return (unsigned char)i;
}

struct RenderArgs {
    const int* xyz;        // (b, n, 3)
    const float* colors;   // (b, n, 3) = c0, c1, c2; NULL: 255
    const int* lengths;    // (b,) or NULL
    unsigned long long* keys;  // (b, h, w)
    unsigned* zrange;          // (b, 2): ~bias(min z), bias(max z), by atomicMax from 0
    int n, h, w, r;
};

__global__ void __launch_bounds__(kRenderThreads) render_zrange_kernel(RenderArgs a) {
    const int img = blockIdx.y;
    const int len = cloud_length0(a.lengths, img, a.n);
    const int p0 = blockIdx.x * kZrangeChunk;
    if (p0 >= len) return;
    const int p1 = min(len, p0 + kZrangeChunk);
    const int* xyz = a.xyz + (size_t)img * a.n * 3;
    unsigned lo = 0xffffffffu, hi = 0;
    for (int i = p0 + (int)threadIdx.x; i < p1; i += blockDim.x) {
        const unsigned k = bias(__ldg(xyz + (size_t)i * 3 + 2));
        lo = min(lo, k);
        hi = max(hi, k);
    }
    lo = __reduce_min_sync(kFullMask, lo);
    hi = __reduce_max_sync(kFullMask, hi);
    if ((threadIdx.x & 31) == 0 && lo <= hi) {
        atomicMax(a.zrange + 2 * img, ~lo);
        atomicMax(a.zrange + 2 * img + 1, hi);
    }
}

// kCount: also count the atomics issued and the ones a read of the pixel's key made unnecessary (counters[0], [1]).
template <bool kCount>
__global__ void __launch_bounds__(kRenderThreads) render_splat_kernel(RenderArgs a, int per_cta,
                                                                      unsigned long long* counters) {
    const int img = blockIdx.y;
    const int len = cloud_length0(a.lengths, img, a.n);
    const int p0 = blockIdx.x * per_cta;
    if (p0 >= len) return;
    const int r = a.r, side = 2 * r + 1, r2 = r * r;
    const unsigned s = (unsigned)side * (unsigned)side;
    const unsigned total = (unsigned)min(per_cta, len - p0) * s;
    const int* xyz = a.xyz + ((size_t)img * a.n + p0) * 3;
    unsigned long long* keys = a.keys + (size_t)img * a.h * a.w;
    unsigned issued = 0, skipped = 0;
    for (unsigned t = threadIdx.x; t < total; t += blockDim.x) {
        const unsigned p = t / s, e = t - p * s;
        const int row = (int)(e / (unsigned)side);
        const int dx = row - r, dy = (int)e - row * side - r;
        const int k = r2 - dx * dx - dy * dy;
        if (k <= 0) continue;  // dx^2 + dy^2 < r^2 only
        const int x2 = __ldg(xyz + p * 3) + dx, y2 = __ldg(xyz + p * 3 + 1) + dy;
        if ((unsigned)x2 >= (unsigned)a.h || (unsigned)y2 >= (unsigned)a.w) continue;
        const int z2 = __ldg(xyz + p * 3 + 2) + isqrt(k);
        if (z2 <= kDepthInit) continue;
        const unsigned long long key = ((unsigned long long)bias(z2) << 32) | (unsigned)~(p0 + (int)p);
        unsigned long long* slot = keys + (size_t)x2 * a.w + y2;
        // keys only grow: a value read here, however stale, that is not below ours means ours cannot win
        if (__ldcg(slot) >= key) {
            if (kCount) ++skipped;
            continue;
        }
        atomicMax(slot, key);
        if (kCount) ++issued;
    }
    if (kCount) {
        issued = __reduce_add_sync(kFullMask, issued);
        skipped = __reduce_add_sync(kFullMask, skipped);
        if ((threadIdx.x & 31) == 0) {
            atomicAdd(counters, (unsigned long long)issued);
            atomicAdd(counters + 1, (unsigned long long)skipped);
        }
    }
}

__global__ void __launch_bounds__(kRenderThreads) render_resolve_kernel(RenderArgs a, uchar3 bg, unsigned char* out) {
    const int img = blockIdx.y;
    const unsigned hw = (unsigned)a.h * (unsigned)a.w;
    const unsigned pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= hw) return;
    const unsigned long long key = __ldcs(a.keys + (size_t)img * hw + pix);
    unsigned char* o = out + ((size_t)img * hw + pix) * 3;
    if (key == 0) {
        o[0] = bg.x;
        o[1] = bg.y;
        o[2] = bg.z;
        return;
    }
    const int r = a.r;
    const int z2 = unbias((unsigned)(key >> 32));
    const int i = (int)~(unsigned)key;
    const int* p = a.xyz + ((size_t)img * a.n + i) * 3;
    const int x2 = (int)(pix / (unsigned)a.w), y2 = (int)(pix - (unsigned)x2 * (unsigned)a.w);
    const int dx = x2 - __ldg(p), dy = y2 - __ldg(p + 1);
    // the pattern entry's shade: (float)(sqrt(double(r^2 - dx^2 - dy^2)) / r)
    const double dz = __dsqrt_rn((double)(r * r - dx * dx - dy * dy));
    const float shade = __double2float_rn(__ddiv_rn(dz, (double)r));
    // zmin / zmax over all the cloud's points: min(z) - r, max(z) + r, in int, then double
    const double zmin = (double)(unbias(~a.zrange[2 * img]) - r);
    const double zmax = (double)(unbias(a.zrange[2 * img + 1]) + r);
    const double t = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn((double)z2, zmin), __dsub_rn(zmax, zmin)), 0.7), 0.3);
    const double intensity = t < 1.0 ? t : 1.0;
    float c0 = 255.f, c1 = 255.f, c2 = 255.f;
    if (a.colors) {
        const float* c = a.colors + ((size_t)img * a.n + i) * 3;
        c0 = __ldg(c);
        c1 = __ldg(c + 1);
        c2 = __ldg(c + 2);
    }
    // shade x colour rounded to float, then times the double intensity, then truncated: show[0] takes c2, [1] c0, [2] c1
    o[0] = x86_u8(__dmul_rn((double)__fmul_rn(shade, c2), intensity));
    o[1] = x86_u8(__dmul_rn((double)__fmul_rn(shade, c0), intensity));
    o[2] = x86_u8(__dmul_rn((double)__fmul_rn(shade, c1), intensity));
}

// One CTA per cloud: the float64 mean over its real points (thread t sums rows t, t + T, ... in order; a fixed tree
// adds the T partial sums), then radius = max |p - mean| and scale = (radius * 2.2) / size.  stats (b, 4): mean, scale.
__global__ void __launch_bounds__(kStatsThreads) project_stats_kernel(const double* xyz, const int* lengths, int n,
                                                                      int size, double* stats) {
    __shared__ double part[3][kStatsThreads];
    __shared__ double mean[3];
    __shared__ double wmax[kStatsThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int len = cloud_length0(lengths, b, n);
    const double* x = xyz + (size_t)b * n * 3;
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int i = tid; i < len; i += kStatsThreads) {
        sx = __dadd_rn(sx, x[(size_t)i * 3]);
        sy = __dadd_rn(sy, x[(size_t)i * 3 + 1]);
        sz = __dadd_rn(sz, x[(size_t)i * 3 + 2]);
    }
    part[0][tid] = sx;
    part[1][tid] = sy;
    part[2][tid] = sz;
    __syncthreads();
    for (int half = kStatsThreads / 2; half > 0; half >>= 1) {
        if (tid < half)
            for (int j = 0; j < 3; ++j) part[j][tid] = __dadd_rn(part[j][tid], part[j][tid + half]);
        __syncthreads();
    }
    if (tid < 3) mean[tid] = len > 0 ? __ddiv_rn(part[tid][0], (double)len) : 0.0;
    __syncthreads();
    double m = 0.0;  // squared norms are >= 0, so 0 is the identity of the max
    for (int i = tid; i < len; i += kStatsThreads) {
        const double dx = __dsub_rn(x[(size_t)i * 3], mean[0]), dy = __dsub_rn(x[(size_t)i * 3 + 1], mean[1]);
        const double dz = __dsub_rn(x[(size_t)i * 3 + 2], mean[2]);
        m = fmax(m, __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
    }
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(kFullMask, m, o));
    if ((tid & 31) == 0) wmax[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        for (int j = 1; j < kStatsThreads / 32; ++j) m = fmax(m, wmax[j]);
        double* s = stats + (size_t)b * 4;
        s[0] = mean[0];
        s[1] = mean[1];
        s[2] = mean[2];
        s[3] = __ddiv_rn(__dmul_rn(__dsqrt_rn(m), 2.2), (double)size);  // sqrt is monotone: max of the norms
    }
}

struct ViewRotations {
    double m[kMaxViewsPerLaunch][9];  // row-major 3 x 3: out_j = sum_k p_k m[k][j]
};

// (p - mean) / scale (0 for a cloud whose points all coincide), times each rotation, plus (size/2, size/2, 0), truncated
// toward zero to int32 after a clamp to +-2^30.  Padding rows are written as 0.
__global__ void __launch_bounds__(kProjectThreads) project_points_kernel(const double* xyz, const int* lengths, int n,
                                                                         int v, int v0, int nv, double center,
                                                                         const double* stats,
                                                                         const __grid_constant__ ViewRotations rot,
                                                                         int* out) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * kProjectThreads + threadIdx.x;
    if (i >= n) return;
    const int len = cloud_length0(lengths, b, n);
    double c[3] = {0.0, 0.0, 0.0};
    if (i < len) {
        const double* s = stats + (size_t)b * 4;
        const double* p = xyz + ((size_t)b * n + i) * 3;
        if (s[3] != 0.0)
            for (int k = 0; k < 3; ++k) c[k] = __ddiv_rn(__dsub_rn(p[k], s[k]), s[3]);
    }
    for (int q = 0; q < nv; ++q) {
        int* o = out + (((size_t)b * v + v0 + q) * n + i) * 3;
        if (i >= len) {
            o[0] = o[1] = o[2] = 0;
            continue;
        }
        const double* m = rot.m[q];
        for (int j = 0; j < 3; ++j) {
            double t = __dadd_rn(__dadd_rn(__dmul_rn(c[0], m[j]), __dmul_rn(c[1], m[3 + j])), __dmul_rn(c[2], m[6 + j]));
            if (j < 2) t = __dadd_rn(t, center);
            t = fmin(fmax(t, -kMaxCoord), kMaxCoord);
            o[j] = __double2int_rz(t);
        }
    }
}

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

bool render_shape_ok(int b, int h, int w) {
    return b >= 1 && b <= kMaxImages && h >= 1 && w >= 1 && (long long)h * w < (1ll << 31);
}

size_t render_keys_bytes(int b, int h, int w) { return align256(sizeof(unsigned long long) * (size_t)b * h * w); }

size_t render_ws_bytes(int b, int h, int w) { return render_keys_bytes(b, h, w) + align256(2 * sizeof(unsigned) * (size_t)b); }

int render_balls(int b, int n, int h, int w, const int* xyz, const float* colors, const int* lengths, int r,
                 const unsigned char* background, void* workspace, size_t workspace_bytes, unsigned char* out,
                 unsigned long long* counters, void* stream) {
    if (b == 0) return 0;
    if (n < 0 || n >= (1 << 30) / 3 || r > kMaxRadius || !render_shape_ok(b, h, w)) return (int)cudaErrorInvalidValue;
    if ((n > 0 && !xyz) || !background || !out || !workspace) return (int)cudaErrorInvalidValue;
    if (workspace_bytes < render_ws_bytes(b, h, w) || !aligned_to(workspace, 256)) return (int)cudaErrorInvalidValue;
    r = r < 1 ? 1 : r;
    cudaStream_t st = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(workspace, 0, render_ws_bytes(b, h, w), st);
    if (e != cudaSuccess) return (int)e;
    const RenderArgs a{xyz, colors, lengths, static_cast<unsigned long long*>(workspace),
                       reinterpret_cast<unsigned*>(static_cast<char*>(workspace) + render_keys_bytes(b, h, w)), n, h, w, r};
    int rc;
    if (n > 0) {
        render_zrange_kernel<<<dim3((unsigned)((n + kZrangeChunk - 1) / kZrangeChunk), (unsigned)b), kRenderThreads, 0,
                               st>>>(a);
        if ((rc = finish_launch())) return rc;
        const int side = 2 * r + 1;
        const int per_cta = side * side >= kSplatPairs ? 1 : kSplatPairs / (side * side);
        const dim3 grid((unsigned)((n + per_cta - 1) / per_cta), (unsigned)b);
        if (counters)
            render_splat_kernel<true><<<grid, kRenderThreads, 0, st>>>(a, per_cta, counters);
        else
            render_splat_kernel<false><<<grid, kRenderThreads, 0, st>>>(a, per_cta, nullptr);
        if ((rc = finish_launch())) return rc;
    }
    const uchar3 bg = make_uchar3(background[0], background[1], background[2]);
    render_resolve_kernel<<<dim3(ceil_div_u((unsigned long long)h * w, kRenderThreads), (unsigned)b), kRenderThreads, 0,
                            st>>>(a, bg, out);
    return finish_launch();
}

}  // namespace
}  // namespace pn2

extern "C" {

size_t pn2_render_balls_workspace_bytes(int b, int h, int w) {
    if (!pn2::render_shape_ok(b, h, w)) return 0;
    return pn2::render_ws_bytes(b, h, w);
}

int pn2_render_balls(int b, int n, int h, int w, const int* xyz, const float* colors, const int* lengths, int r,
                     const unsigned char* background, void* workspace, size_t workspace_bytes, unsigned char* out,
                     void* stream) {
    return pn2::render_balls(b, n, h, w, xyz, colors, lengths, r, background, workspace, workspace_bytes, out, nullptr,
                             stream);
}

int pn2_render_balls_counted(int b, int n, int h, int w, const int* xyz, const float* colors, const int* lengths, int r,
                             const unsigned char* background, void* workspace, size_t workspace_bytes,
                             unsigned char* out, unsigned long long* counters, void* stream) {
    if (!counters) return (int)cudaErrorInvalidValue;
    return pn2::render_balls(b, n, h, w, xyz, colors, lengths, r, background, workspace, workspace_bytes, out, counters,
                             stream);
}

int pn2_project_points(int b, int n, int v, const double* xyz, const int* lengths, const double* rotations, int size,
                       void* workspace, size_t workspace_bytes, int* out, void* stream) {
    using namespace pn2;
    if (b == 0 || n == 0) return 0;
    if (b < 0 || b > kMaxImages || n < 0 || n >= (1 << 30) / 3 || v < 1 || size < 1) return (int)cudaErrorInvalidValue;
    if (!xyz || !rotations || !workspace || !out || workspace_bytes < sizeof(double) * 4 * (size_t)b ||
        !aligned_to(workspace, 8))
        return (int)cudaErrorInvalidValue;
    cudaStream_t st = as_stream(stream);
    double* stats = static_cast<double*>(workspace);
    project_stats_kernel<<<(unsigned)b, kStatsThreads, 0, st>>>(xyz, lengths, n, size, stats);
    int rc = finish_launch();
    if (rc) return rc;
    const dim3 grid((unsigned)((n + kProjectThreads - 1) / kProjectThreads), (unsigned)b);
    for (int v0 = 0; v0 < v; v0 += kMaxViewsPerLaunch) {
        const int nv = v - v0 < kMaxViewsPerLaunch ? v - v0 : kMaxViewsPerLaunch;
        ViewRotations rot{};
        for (int q = 0; q < nv; ++q)
            for (int j = 0; j < 9; ++j) rot.m[q][j] = rotations[(size_t)(v0 + q) * 9 + j];
        project_points_kernel<<<grid, kProjectThreads, 0, st>>>(xyz, lengths, n, v, v0, nv, size / 2.0, stats, rot, out);
        if ((rc = finish_launch())) return rc;
    }
    return 0;
}

}  // extern "C"
