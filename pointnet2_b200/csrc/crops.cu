// crops.cu — ScanNet training crops: B seeded, validity-checked xy columns drawn from a set of scenes, as a padded
// ragged batch with point dropout and a rotation about z (scannet/scannet_dataset.py:27-60, scannet/train.py:181-197,
// utils/provider.py:52-70, without the resampling; DESIGN.md §6.10).
//
// Two kernels per call, nothing read back:
//   attempt: CTA (chunk, crop) reads a chunk of the crop's scene once and tests the boxes of all ten attempts: integer
//            context / labelled counts and the core voxel-key bitmap in shared memory, merged into the crop's workspace
//            with integer atomicAdd / atomicOr (order-free);
//   select:  one CTA per crop takes the first valid attempt (else attempt 9), takes the m smallest (key, scene index)
//            pairs of its members in order (cta_select_sorted) and writes the rows (dropout compaction, rotation,
//            labels, weights, padding).
// Every membership test is the double test of the definition, done exactly in float32: for a float p and a double t,
// (double)p >= t <=> p >= (t rounded up to float), and (double)p <= t <=> p <= (t rounded down to float).
#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kAttempts = 10;            // scannet_dataset.py:37
constexpr int kKeyWords = 1986;          // keys 0 .. 32*31*62 + 32*62 + 62 = 63550 -> 63551 bits
constexpr int kCropWsWords = kAttempts * 2 + kAttempts * kKeyWords;  // per crop: (context, labelled) x 10, 10 bitmaps
constexpr int kAttemptThreads = 512;
constexpr int kAttemptChunk = 8192;      // scene points per CTA of the attempt pass
constexpr int kSelectThreads = 1024;

struct CropArgs {
    const float* xyz;
    const int* label;
    const long long* offsets;
    const float* lo;
    const float* hi;
    const long long* crop_scene;
    const long long* seed_dev;  // non-null: the seed is read here, on the device
    unsigned long long seed;
    int s;
};

// One attempt's box: context and core bounds as exact float thresholds, and curmin / curmax - curmin for the keys.
struct CropBox {
    float c0[3], c1[3];  // context: c0 <= p <= c1
    float k0[3], k1[3];  // core
    double mn[3], ext[3];
};

__device__ __forceinline__ void crop_box(const CropArgs& a, unsigned long long seed, int b, int att, long long off, long long ps,
                                         int sc, CropBox& B) {
    const long long ci = off + (long long)(rng_draw(seed, 1, (unsigned long long)b, (unsigned long long)att) % (unsigned long long)ps);
    double mn[3], mx[3];
    for (int d = 0; d < 2; ++d) {
        const double c = (double)__ldg(a.xyz + 3 * ci + d);
        mn[d] = __dsub_rn(c, 0.75);
        mx[d] = __dadd_rn(c, 0.75);
    }
    mn[2] = (double)__ldg(a.lo + 3 * sc + 2);
    mx[2] = (double)__ldg(a.hi + 3 * sc + 2);
    for (int d = 0; d < 3; ++d) {
        B.c0[d] = __double2float_ru(__dsub_rn(mn[d], 0.2));
        B.c1[d] = __double2float_rd(__dadd_rn(mx[d], 0.2));
        B.k0[d] = __double2float_ru(__dsub_rn(mn[d], 0.01));
        B.k1[d] = __double2float_rd(__dadd_rn(mx[d], 0.01));
        B.mn[d] = mn[d];
        B.ext[d] = __dsub_rn(mx[d], mn[d]);
    }
}

__device__ __forceinline__ bool in_ctx(const CropBox& B, float x, float y, float z) {
    return x >= B.c0[0] && x <= B.c1[0] && y >= B.c0[1] && y <= B.c1[1] && z >= B.c0[2] && z <= B.c1[2];
}
__device__ __forceinline__ bool in_core(const CropBox& B, float x, float y, float z) {
    return x >= B.k0[0] && x <= B.k1[0] && y >= B.k0[1] && y <= B.k1[1] && z >= B.k0[2] && z <= B.k1[2];
}

// ceil((p - curmin) / (curmax - curmin) * (31, 31, 62)), then vx*31*62 + vy*62 + vz (scannet_dataset.py:49-50).  The
// clamp only guards the bitmap: for a core member the key is always in [0, 63550].
__device__ __forceinline__ int voxel_key(const CropBox& B, float x, float y, float z) {
    const double vx = ceil(__dmul_rn(__ddiv_rn(__dsub_rn((double)x, B.mn[0]), B.ext[0]), 31.0));
    const double vy = ceil(__dmul_rn(__ddiv_rn(__dsub_rn((double)y, B.mn[1]), B.ext[1]), 31.0));
    const double vz = ceil(__dmul_rn(__ddiv_rn(__dsub_rn((double)z, B.mn[2]), B.ext[2]), 62.0));
    const int k = (int)vx * (31 * 62) + (int)vy * 62 + (int)vz;
    return min(max(k, 0), kKeyWords * 32 - 1);
}

// grid (chunks, B).  ws: per crop, counts[10][2] then bitmap[10][kKeyWords], zeroed by the caller.
__global__ void __launch_bounds__(kAttemptThreads) crop_attempt_kernel(CropArgs a, unsigned* __restrict__ ws) {
    extern __shared__ unsigned s_bits[];  // [kAttempts][kKeyWords]
    __shared__ CropBox s_box[kAttempts];
    __shared__ int s_cnt[kAttempts][2];
    __shared__ int s_any[kAttempts];
    const int b = blockIdx.y;
    int sc;
    long long off, ps;
    if (!set_entry(a.crop_scene, b, a.s, a.offsets, sc, off, ps)) return;
    const long long q0 = (long long)blockIdx.x * kAttemptChunk;
    if (q0 >= ps) return;
    const long long q1 = min(ps, q0 + kAttemptChunk);
    if (threadIdx.x < kAttempts) {
        crop_box(a, rng_seed(a.seed_dev, a.seed), b, threadIdx.x, off, ps, sc, s_box[threadIdx.x]);
        s_cnt[threadIdx.x][0] = s_cnt[threadIdx.x][1] = 0;
        s_any[threadIdx.x] = 0;
    }
    for (int k = threadIdx.x; k < kAttempts * kKeyWords; k += blockDim.x) s_bits[k] = 0u;
    __syncthreads();
    int ctx[kAttempts], lab[kAttempts];
#pragma unroll
    for (int t = 0; t < kAttempts; ++t) ctx[t] = lab[t] = 0;
    for (long long q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
        const long long g = off + q;
        const float x = __ldg(a.xyz + 3 * g), y = __ldg(a.xyz + 3 * g + 1), z = __ldg(a.xyz + 3 * g + 2);
        const int labelled = __ldg(a.label + g) > 0;
#pragma unroll
        for (int t = 0; t < kAttempts; ++t) {
            const CropBox& B = s_box[t];
            if (!in_ctx(B, x, y, z)) continue;
            ++ctx[t];
            lab[t] += labelled;
            if (in_core(B, x, y, z)) {
                const int key = voxel_key(B, x, y, z);
                atomicOr(&s_bits[t * kKeyWords + (key >> 5)], 1u << (key & 31));
                s_any[t] = 1;
            }
        }
    }
#pragma unroll
    for (int t = 0; t < kAttempts; ++t) {
        const int c = __reduce_add_sync(kFullMask, ctx[t]), l = __reduce_add_sync(kFullMask, lab[t]);
        if ((threadIdx.x & 31) == 0 && c) {
            atomicAdd(&s_cnt[t][0], c);
            atomicAdd(&s_cnt[t][1], l);
        }
    }
    __syncthreads();
    unsigned* w = ws + (size_t)b * kCropWsWords;
    if (threadIdx.x < kAttempts && s_cnt[threadIdx.x][0]) {
        atomicAdd(reinterpret_cast<int*>(w) + 2 * threadIdx.x, s_cnt[threadIdx.x][0]);
        atomicAdd(reinterpret_cast<int*>(w) + 2 * threadIdx.x + 1, s_cnt[threadIdx.x][1]);
    }
    for (int k = threadIdx.x; k < kAttempts * kKeyWords; k += blockDim.x) {
        if (!s_any[k / kKeyWords]) continue;
        const unsigned v = s_bits[k];
        if (v) atomicOr(w + 2 * kAttempts + k, v);
    }
}

struct CropOut {
    float* xyz;
    long long* label;
    float* weight;
    int* lengths;
    int* point_idx;
    unsigned char* core;
    int* attempt;
    unsigned char* valid;
};

// One CTA per crop.  Dynamic shared memory: the sort buffer, pow2 >= npoints 64-bit values.
__global__ void __launch_bounds__(kSelectThreads) crop_select_kernel(CropArgs a, const unsigned* __restrict__ ws, int num_class,
                                                                     const float* __restrict__ label_weights, int npoints,
                                                                     double max_dropout, int rotate, CropOut o) {
    extern __shared__ unsigned long long s_keys[];
    __shared__ SelectScratch s_sel;
    __shared__ int s_vox[kAttempts];
    __shared__ CropBox s_box;
    __shared__ int s_c;
    __shared__ double s_cos, s_sin;
    const int b = blockIdx.x, tid = threadIdx.x;
    const size_t row0 = (size_t)b * npoints;
    int sc, kept = 0;
    long long off, ps;
    if (set_entry(a.crop_scene, b, a.s, a.offsets, sc, off, ps)) {
        const unsigned long long seed = rng_seed(a.seed_dev, a.seed);
        const unsigned* w = ws + (size_t)b * kCropWsWords;
        // distinct voxel keys of every attempt
        if (tid < kAttempts) s_vox[tid] = 0;
        __syncthreads();
        for (int t = 0; t < kAttempts; ++t) {
            int v = 0;
            for (int k = tid; k < kKeyWords; k += blockDim.x) v += __popc(__ldg(w + 2 * kAttempts + t * kKeyWords + k));
            v = __reduce_add_sync(kFullMask, v);
            if ((tid & 31) == 0 && v) atomicAdd(&s_vox[t], v);
        }
        __syncthreads();
        if (tid == 0) {
            int att = kAttempts - 1, ok = 0;
            for (int t = 0; t < kAttempts; ++t) {
                const int c = (int)__ldg(w + 2 * t), l = (int)__ldg(w + 2 * t + 1);
                const bool lab_ok = __ddiv_rn((double)l, (double)c) >= 0.7;
                const bool vox_ok = __ddiv_rn(__ddiv_rn(__ddiv_rn((double)s_vox[t], 31.0), 31.0), 62.0) >= 0.02;
                if (lab_ok && vox_ok) {
                    att = t;
                    ok = 1;
                    break;
                }
            }
            s_c = (int)__ldg(w + 2 * att);
            crop_box(a, seed, b, att, off, ps, sc, s_box);
            o.attempt[b] = att;
            o.valid[b] = (unsigned char)ok;
            if (rotate) {
                // theta = u * 2 pi: sincospi(2u) needs no argument reduction (2u is exact) and agrees with cos / sin
                // of the rounded theta to within a double ulp, far below the float32 result's rounding
                double sn, cs;
                sincospi(__dmul_rn(rng_unit(rng_draw(seed, 5, (unsigned long long)b, 0)), 2.0), &sn, &cs);
                s_cos = cs;
                s_sin = sn;
            }
        }
        __syncthreads();
        const CropBox B = s_box;
        const int c = s_c, m = min(c, npoints);
        // the m smallest member orders, sorted
        cta_select_sorted(
            ps, c, m,
            [&](long long j) {
                const long long g = off + j;
                return in_ctx(B, __ldg(a.xyz + 3 * g), __ldg(a.xyz + 3 * g + 1), __ldg(a.xyz + 3 * g + 2));
            },
            [&](long long j) { return rng_row_key(seed, 2, (unsigned long long)b, j); }, s_keys, s_sel);
        // rows: dropout compaction (row 0 always stays), then each survivor written in row order
        const double ratio = __dmul_rn(rng_unit(rng_draw(seed, 3, (unsigned long long)b, 0)), max_dropout);
        const auto dropped = [&](int r) {
            return rng_unit(rng_draw(seed, 4, (unsigned long long)b, (unsigned long long)r)) <= ratio;
        };
        kept = cta_compact(
            m, [&](int r) { return r == 0 || !dropped(r); },
            [&](int r, int at) {
                const size_t row = row0 + at;
                const long long j = (long long)(s_keys[r] & 0xffffffffull), g = off + j;
                const float x = __ldg(a.xyz + 3 * g), y = __ldg(a.xyz + 3 * g + 1), z = __ldg(a.xyz + 3 * g + 2);
                const int l = __ldg(a.label + g);
                const bool is_core = in_core(B, x, y, z);
                float wt = (is_core && l >= 0 && l < num_class) ? __ldg(label_weights + l) : 0.f;
                if (r == 0 && dropped(0)) wt = 0.f;  // row 0 whose own draw drops it: its point stays, unweighted
                float ox = x, oy = y;
                if (rotate) {
                    ox = __double2float_rn(__dsub_rn(__dmul_rn((double)x, s_cos), __dmul_rn((double)y, s_sin)));
                    oy = __double2float_rn(__dadd_rn(__dmul_rn((double)x, s_sin), __dmul_rn((double)y, s_cos)));
                }
                o.xyz[3 * row] = ox;
                o.xyz[3 * row + 1] = oy;
                o.xyz[3 * row + 2] = z;
                o.label[row] = l;
                o.weight[row] = wt;
                o.point_idx[row] = (int)g;
                o.core[row] = is_core ? 1 : 0;
            },
            s_sel.w);
    } else if (tid == 0) {  // a scene index outside [0, S): an empty crop, attempt -1
        o.attempt[b] = -1;
        o.valid[b] = 0;
    }
    for (int r = kept + tid; r < npoints; r += blockDim.x) {
        const size_t row = row0 + r;
        o.xyz[3 * row] = o.xyz[3 * row + 1] = o.xyz[3 * row + 2] = 0.f;
        o.label[row] = 0;
        o.weight[row] = 0.f;
        o.point_idx[row] = -1;
        o.core[row] = 0;
    }
    if (tid == 0) o.lengths[b] = kept;
}

size_t crop_ws_bytes(int b) { return ((size_t)b * kCropWsWords * sizeof(unsigned) + 255) / 256 * 256; }
bool crop_shape_ok(int b, int npoints) {
    return b >= 1 && b <= 65535 && npoints >= 1 && npoints <= kSelectMaxRows && (long long)b * npoints * 3 < (1ll << 31);
}

AttrOnce g_attempt_attr, g_select_attr;

}  // namespace
}  // namespace pn2

extern "C" {

size_t pn2_scene_crops_workspace_bytes(int b, int npoints) {
    if (!pn2::crop_shape_ok(b, npoints)) return 0;
    return pn2::crop_ws_bytes(b);
}

int pn2_scene_crops(int s, int p, int max_scene, const float* xyz, const int* label, const long long* offsets, const float* lo,
                    const float* hi, int num_class, const float* label_weights, int b, const long long* crop_scene,
                    long long seed, const long long* seed_dev, int npoints, double max_dropout, int rotate, float* out_xyz,
                    long long* out_label, float* out_weight, int* lengths, int* point_idx, unsigned char* core, int* attempt,
                    unsigned char* valid, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (s < 1 || p < 1 || p >= 0x7fffffff || max_scene < 1 || max_scene > p || num_class < 1 || !crop_shape_ok(b, npoints))
        return (int)cudaErrorInvalidValue;
    if (!(max_dropout >= 0.0 && max_dropout <= 1.0)) return (int)cudaErrorInvalidValue;
    if (!xyz || !label || !offsets || !lo || !hi || !label_weights || !crop_scene || !out_xyz || !out_label || !out_weight ||
        !lengths || !point_idx || !core || !attempt || !valid || !workspace)
        return (int)cudaErrorInvalidValue;
    if (workspace_bytes < crop_ws_bytes(b) || !aligned_to(workspace, 256)) return (int)cudaErrorInvalidValue;
    cudaStream_t st = as_stream(stream);
    const size_t attempt_smem = sizeof(unsigned) * kAttempts * kKeyWords;
    cudaError_t e = ensure_attrs(g_attempt_attr, crop_attempt_kernel, attempt_smem, false);
    if (e != cudaSuccess) return (int)e;
    e = ensure_attrs(g_select_attr, crop_select_kernel, sizeof(unsigned long long) * kSelectMaxRows, false);
    if (e != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(workspace, 0, crop_ws_bytes(b), st)) != cudaSuccess) return (int)e;
    const CropArgs a{xyz, label, offsets, lo, hi, crop_scene, seed_dev, (unsigned long long)seed, s};
    const dim3 grid((unsigned)((max_scene + kAttemptChunk - 1) / kAttemptChunk), (unsigned)b);
    unsigned* ws = static_cast<unsigned*>(workspace);
    crop_attempt_kernel<<<grid, kAttemptThreads, attempt_smem, st>>>(a, ws);
    int rc = finish_launch();
    if (rc) return rc;
    const CropOut o{out_xyz, out_label, out_weight, lengths, point_idx, core, attempt, valid};
    crop_select_kernel<<<b, kSelectThreads, sizeof(unsigned long long) * pow2_at_least(npoints), st>>>(
        a, ws, num_class, label_weights, npoints, max_dropout, rotate, o);
    return finish_launch();
}

}  // extern "C"
