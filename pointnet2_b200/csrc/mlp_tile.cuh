// mlp_tile.cuh — the tile machinery of the fused inference MLPs (sa_mlp.cu, fp_mlp.cu), for sm_90a.
//
// A CTA of kMlpThreads threads holds TM rows in shared memory and runs up to kMlpMaxLayers layers
//   row = act(row . W^T * scale + shift),  scale / shift from the Linear's bias and the batch norm's running statistics,
// the activations ping-ponging between two shared buffers from layer to layer.  One tile structure, two arithmetic
// instantiations:
//   float:            register-tiled FP32, explicit fmaf in ascending k (the library builds with -fmad=false), weights
//                     streamed through shared memory in 64 x 32 slabs with cp.async, double-buffered;
//   bfloat16 / half:  mma.sync.m16n8k16 with float32 accumulators, A fragments by ldmatrix from a padded layout, weights
//                     converted to the 16-bit type while they are staged; activations are rounded to the 16-bit type once
//                     per layer, after the batch-norm affine and the ReLU, both applied in float32.
// Every output row depends on its own input row only (the weights are the same for every row) and every sum has a fixed
// order, so a row's result has the same bits whatever else is in the tile.
#pragma once

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kMlpThreads = 256;
constexpr int kMlpTN = 64;         // output channels per pass
constexpr int kMlpKS = 32;         // input channels per weight slab
constexpr int kMlpMaxLayers = 4;
constexpr int kMlpMaxWidth = 1024;
constexpr size_t kMlpSmemLimit = 227 * 1024;

struct MlpLayer {
    const float *w, *bias, *gamma, *beta, *mean, *var;  // mean == nullptr: no batch norm; gamma == nullptr: not affine
    float eps;
    int cin, cout, relu;
};

// Row strides that keep the shared-memory reads free of bank conflicts: float rows 4 words past a multiple of 32 (the
// 16-byte reads of 8 consecutive rows then cover all 32 banks), 16-bit rows 16 bytes past a multiple of 128 (ldmatrix).
template <typename T> constexpr __host__ __device__ int act_stride(int c) {
    return sizeof(T) == 4 ? (c + 31) / 32 * 32 + 4 : (c + 63) / 64 * 64 + 8;
}
template <typename T> constexpr __host__ __device__ int slab_stride() { return sizeof(T) == 4 ? kMlpKS + 4 : kMlpKS + 8; }

// Elements of the two weight slabs, of type T
template <typename T> constexpr __host__ __device__ int slab_elems() { return 2 * kMlpTN * slab_stride<T>(); }

// Input channels rounded up to whole slabs: a tile's rows are zero from cin to here
__host__ __device__ __forceinline__ int slab_pad(int c) { return (c + kMlpKS - 1) / kMlpKS * kMlpKS; }

__device__ __forceinline__ void cp_async_f32(float* dst, const float* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    const int bytes = valid ? 4 : 0;  // 0 source bytes: the word is zero-filled
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(bytes));
}
__device__ __forceinline__ void cp_async_commit_wait() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ void mma_16816(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1, __nv_bfloat16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1, __half) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ReLU that keeps NaN, as torch's does
__device__ __forceinline__ float relu_nan(float y) { return y < 0.f ? 0.f : y; }

// The accumulator tile of one thread and where its elements sit in the CTA's TM x 64 pass.
//   float:  16 x 16 threads; thread (tx, ty) holds rows ty*RM .. ty*RM+RM-1 and columns tx + 16 j (j < 4).
//   16-bit: warps WM x WN; a warp holds 16 rows x NT n-tiles of 8 columns in the m16n8 accumulator layout.
template <typename T, int TM> struct Tile {
    static constexpr bool kMma = sizeof(T) == 2;
    static constexpr int RM = TM / 16;                 // float: rows per thread
    static constexpr int WM = TM / 16, WN = 8 / WM;    // 16-bit: warps along rows / columns
    static constexpr int NT = kMlpTN / (8 * WN);       // 16-bit: n-tiles per warp
    static constexpr int kAcc = kMma ? NT * 4 : RM * 4;
    // a warp's rows lie in [row_lo(), row_lo() + kRowSpan)
    static constexpr int kRowSpan = kMma ? 16 : 2 * RM;

    // element i of a thread's accumulators is (row_of(i), col_of(i, pass))
    __device__ static __forceinline__ int row_of(int i) {
        const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
        if constexpr (kMma) return (warp % WM) * 16 + (lane >> 2) + ((i & 2) ? 8 : 0);
        else return (tid >> 4) * RM + i / 4;
    }
    __device__ static __forceinline__ int col_of(int i, int pass) {
        const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
        if constexpr (kMma) return pass * kMlpTN + (warp / WM) * 8 * NT + (i / 4) * 8 + (lane & 3) * 2 + (i & 1);
        else return pass * kMlpTN + (tid & 15) + 16 * (i & 3);
    }
    __device__ static __forceinline__ int row_lo() {
        const int warp = threadIdx.x >> 5;
        if constexpr (kMma) return (warp % WM) * 16;
        else return (warp * 2) * RM;  // the warp's two ty
    }
};

// The layers of one tile.  act0 holds the TM input rows of layer 0, zero from layer[0].cin up to slab_pad of it; layer
// l reads buffer l & 1 and writes the other one (row strides stride0 / stride1).  Each layer's result is rounded to T
// and stored there, zero from cout up to slab_pad(cout), except the last layer's when kStoreLast is false: its float32
// results go to last(y, pass) at the end of every pass instead (y holds the thread's Tile::kAcc elements, see
// Tile::row_of / col_of; columns >= cout hold 0).  wbuf holds slab_elems<T>() elements, s_scale / s_shift one float per
// output channel of the widest layer.  The caller synchronises the CTA between filling act0 and this call; the call
// ends with a barrier.
template <typename T, int TM, bool kStoreLast, typename Last>
__device__ __forceinline__ void mlp_tile_layers(const MlpLayer* layers, int nlayers, T* act0, T* act1, int stride0,
                                                int stride1, T* wbuf, float* s_scale, float* s_shift, Last&& last) {
    using TL = Tile<T, TM>;
    constexpr int WS = slab_stride<T>();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int l = 0; l < nlayers; ++l) {
        const MlpLayer& L = layers[l];
        const bool store = kStoreLast || l + 1 < nlayers;
        const T* ain = (l & 1) ? act1 : act0;
        T* aout = (l & 1) ? act0 : act1;
        const int sa = (l & 1) ? stride1 : stride0, so = (l & 1) ? stride0 : stride1;
        const int cout_pad = slab_pad(L.cout);

        // y = acc * scale + shift: the Linear's bias and the batch norm's running statistics and affine, per channel
        for (int ch = tid; ch < L.cout; ch += kMlpThreads) {
            float scale = 1.f, shift = L.bias ? __ldg(L.bias + ch) : 0.f;
            if (L.mean) {
                scale = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__ldg(L.var + ch), L.eps)));
                if (L.gamma) scale = __fmul_rn(scale, __ldg(L.gamma + ch));
                shift = __fmaf_rn(__fsub_rn(shift, __ldg(L.mean + ch)), scale, L.beta ? __ldg(L.beta + ch) : 0.f);
            }
            s_scale[ch] = scale;
            s_shift[ch] = shift;
        }

        const int nslabs = (L.cin + kMlpKS - 1) / kMlpKS, npass = (L.cout + kMlpTN - 1) / kMlpTN;
        const int total = nslabs * npass;
        float staged[8];  // 16-bit: a slab's 8 words per thread on their way from global to shared memory

        // slab t = (pass, k-slab): W[pass*64 + nn][s*32 + kk] for nn < 64, kk < 32, zero outside the matrix
        auto issue = [&](int t) {
            const int pass = t / nslabs, s = t - pass * nslabs;
            T* dst = wbuf + (t & 1) * kMlpTN * WS;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int e = tid + kMlpThreads * i, kk = e & 31, nn = e >> 5;
                const int nrow = pass * kMlpTN + nn, kcol = s * kMlpKS + kk;
                const bool ok = nrow < L.cout && kcol < L.cin;
                const float* src = ok ? L.w + (size_t)nrow * L.cin + kcol : L.w;
                if constexpr (TL::kMma) staged[i] = ok ? __ldg(src) : 0.f;
                else cp_async_f32(reinterpret_cast<float*>(dst) + nn * WS + kk, src, ok);
            }
        };
        auto land = [&](int t) {
            if constexpr (TL::kMma) {
                T* dst = wbuf + (t & 1) * kMlpTN * WS;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int e = tid + kMlpThreads * i;
                    dst[(e >> 5) * WS + (e & 31)] = from_f32<T>(staged[i]);
                }
            } else {
                cp_async_commit_wait();
            }
        };

        float acc[TL::kAcc];
        issue(0);
        land(0);
        __syncthreads();
        for (int t = 0; t < total; ++t) {
            const int pass = t / nslabs, s = t - pass * nslabs;
            if (t + 1 < total) issue(t + 1);
            if (s == 0) {
#pragma unroll
                for (int i = 0; i < TL::kAcc; ++i) acc[i] = 0.f;
            }
            const T* wb = wbuf + (t & 1) * kMlpTN * WS;
            if constexpr (!TL::kMma) {
                const int tx = tid & 15, ty = tid >> 4;
                const float* arow = reinterpret_cast<const float*>(ain) + (size_t)(ty * TL::RM) * sa + s * kMlpKS;
                const float* wrow = reinterpret_cast<const float*>(wb) + tx * WS;
#pragma unroll
                for (int k4 = 0; k4 < kMlpKS; k4 += 4) {
                    float4 av[TL::RM], wv[4];
#pragma unroll
                    for (int i = 0; i < TL::RM; ++i) av[i] = *reinterpret_cast<const float4*>(arow + (size_t)i * sa + k4);
#pragma unroll
                    for (int j = 0; j < 4; ++j) wv[j] = *reinterpret_cast<const float4*>(wrow + 16 * j * WS + k4);
#pragma unroll
                    for (int i = 0; i < TL::RM; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            float v = acc[i * 4 + j];
                            v = __fmaf_rn(av[i].x, wv[j].x, v);
                            v = __fmaf_rn(av[i].y, wv[j].y, v);
                            v = __fmaf_rn(av[i].z, wv[j].z, v);
                            v = __fmaf_rn(av[i].w, wv[j].w, v);
                            acc[i * 4 + j] = v;
                        }
                }
            } else {
                const int wm = warp % TL::WM, wn = warp / TL::WM;
                const T* abase = ain + (size_t)(wm * 16 + (lane & 15)) * sa + s * kMlpKS + (lane >> 4) * 8;
                const T* bbase = wb + (wn * 8 * TL::NT + (lane >> 2)) * WS + (lane & 3) * 2;
#pragma unroll
                for (int kk = 0; kk < kMlpKS; kk += 16) {
                    unsigned a[4];
                    const unsigned addr = (unsigned)__cvta_generic_to_shared(abase + kk);
                    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                                 : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(addr));
#pragma unroll
                    for (int nt = 0; nt < TL::NT; ++nt) {
                        const T* bp = bbase + nt * 8 * WS + kk;
                        const unsigned b0 = *reinterpret_cast<const unsigned*>(bp);
                        const unsigned b1 = *reinterpret_cast<const unsigned*>(bp + 8);
                        float(&c)[4] = *reinterpret_cast<float(*)[4]>(acc + nt * 4);
                        mma_16816(c, a, b0, b1, T());
                    }
                }
            }

            if (s == nslabs - 1) {
                // ---- epilogue of this pass: affine + ReLU, then to the other buffer or to the caller ----
                float y[TL::kAcc];
#pragma unroll
                for (int i = 0; i < TL::kAcc; ++i) {
                    const int col = TL::col_of(i, pass);
                    float v = 0.f;
                    if (col < L.cout) {
                        v = __fmaf_rn(acc[i], s_scale[col], s_shift[col]);
                        if (L.relu) v = relu_nan(v);
                    }
                    y[i] = v;
                }
                if (store) {
#pragma unroll
                    for (int i = 0; i < TL::kAcc; ++i) {
                        const int col = TL::col_of(i, pass);
                        if (col < cout_pad) aout[(size_t)TL::row_of(i) * so + col] = from_f32<T>(y[i]);  // 0 beyond cout
                    }
                } else {
                    last(y, pass);
                }
            }
            if (t + 1 < total) land(t + 1);
            __syncthreads();
        }
    }
}

// The layers of a C entry's per-layer HOST arrays (see pn2_sa_mlp_max_typed) as MlpLayer entries, layer 0 taking cin
// inputs; max_cout receives the widest layer.  false: an invalid argument (nothing may be launched).
inline bool mlp_layers_from_args(MlpLayer* layer, int& max_cout, int cin, int nlayers, const int* widths,
                                 const float* const* weight, const float* const* bias, const float* const* bn_weight,
                                 const float* const* bn_bias, const float* const* bn_mean, const float* const* bn_var,
                                 const float* bn_eps, const int* relu) {
    if (nlayers < 1 || nlayers > kMlpMaxLayers || !widths || !weight || !bias || !relu) return false;
    int prev = cin;
    max_cout = 0;
    for (int l = 0; l < nlayers; ++l) {
        if (widths[l] < 1 || widths[l] > kMlpMaxWidth || !weight[l]) return false;
        const bool has_bn = bn_mean && bn_mean[l];
        if (has_bn && (!bn_var || !bn_var[l] || !bn_eps)) return false;
        layer[l] = MlpLayer{weight[l], bias[l], has_bn && bn_weight ? bn_weight[l] : nullptr,
                            has_bn && bn_bias ? bn_bias[l] : nullptr, has_bn ? bn_mean[l] : nullptr,
                            has_bn ? bn_var[l] : nullptr, has_bn ? bn_eps[l] : 0.f, prev, widths[l], relu[l] != 0};
        if (widths[l] > max_cout) max_cout = widths[l];
        prev = widths[l];
    }
    return true;
}

}  // namespace pn2
