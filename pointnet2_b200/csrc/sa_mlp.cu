// sa_mlp.cu — the inference tail of a set-abstraction level in one launch, for sm_90a:
//   gather (utils/pointnet_util.py:45-54 / :179-186)  ->  shared MLP, each layer 1x1 conv + eval-mode batch norm + ReLU
//   (:115-121 / :187-190)  ->  max over the group's rows (:124 / :191).
// Nothing of shape (b*m*nsample, .) reaches global memory: a CTA holds a tile of TM rows (whole groups, or one piece of
// a group larger than the tile) in shared memory, the activations ping-pong between two shared buffers from layer to
// layer, and the last layer's accumulators go from registers into a per-group running maximum.
//
// One tile structure, two arithmetic instantiations:
//   float:            register-tiled FP32, explicit fmaf in ascending k (the library builds with -fmad=false), weights
//                     streamed through shared memory in 64 x 32 slabs with cp.async, double-buffered;
//   bfloat16 / half:  mma.sync.m16n8k16 with float32 accumulators, A fragments by ldmatrix from a padded layout, weights
//                     converted to the 16-bit type while they are staged; activations are rounded to the 16-bit type once
//                     per layer, after the batch-norm affine and the ReLU, both applied in float32.
// Every output depends on its own group only and every sum has a fixed order, so results are bit-identical from run to
// run and whatever else is in the batch.  The maximum keeps NaN (torch's max does; fmaxf would drop it): values are
// compared as order-preserving integer keys in which NaN is the largest.
#include <type_traits>

#include "pn2_common.cuh"

namespace pn2 {

constexpr int kMlpThreads = 256;
constexpr int kMlpTN = 64;         // output channels per pass
constexpr int kMlpKS = 32;         // input channels per weight slab
constexpr int kMlpMaxLayers = 4;
constexpr int kMlpMaxWidth = 1024;
constexpr int kMlpMaxIn = kMlpMaxWidth + 3;
constexpr size_t kMlpSmemLimit = 227 * 1024;

struct SaMlpLayer {
    const float *w, *bias, *gamma, *beta, *mean, *var;  // mean == nullptr: no batch norm; gamma == nullptr: not affine
    float eps;
    int cin, cout, relu;
};

struct SaMlpParams {
    const float* xyz;
    const float* new_xyz;  // nullptr: zeros
    const void* points;    // nullptr: no features
    const int* idx;        // nullptr: row k of every group is point k (nsample == n)
    void* out;
    long long out_stride;  // elements between consecutive groups of out
    long long groups;      // b * m
    int n, c, m, nsample;
    int xyz_lo, feat_lo;   // first column of the centred xyz (-1: none) and of the features in a row
    int nlayers;
    int groups_per_tile;   // whole groups in a tile (nsample <= TM), or 1 with the group walked in pieces of TM rows
    int stride0, stride1;  // row strides of the two activation buffers, in elements
    int max_cout;
    SaMlpLayer layer[kMlpMaxLayers];
};

// Row strides that keep the shared-memory reads free of bank conflicts: float rows 4 words past a multiple of 32 (the
// 16-byte reads of 8 consecutive rows then cover all 32 banks), 16-bit rows 16 bytes past a multiple of 128 (ldmatrix).
template <typename T> constexpr __host__ __device__ int act_stride(int c) {
    return sizeof(T) == 4 ? (c + 31) / 32 * 32 + 4 : (c + 63) / 64 * 64 + 8;
}
template <typename T> constexpr __host__ __device__ int slab_stride() { return sizeof(T) == 4 ? kMlpKS + 4 : kMlpKS + 8; }

// float -> key with  a < b  <=>  key(a) < key(b)  as unsigned, every NaN the largest key; 0 is below every key
__device__ __forceinline__ unsigned max_key(float v) {
    if (v != v) return 0xffffffffu;
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

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
};

template <typename T, int TM>
__global__ void __launch_bounds__(kMlpThreads, sizeof(T) == 4 && TM == 64 ? 1 : 2)
sa_mlp_max_kernel(const __grid_constant__ SaMlpParams p) {
    using TL = Tile<T, TM>;
    constexpr int WS = slab_stride<T>();
    extern __shared__ __align__(16) unsigned char smem[];
    T* act0 = reinterpret_cast<T*>(smem);
    T* act1 = act0 + (size_t)TM * p.stride0;
    T* wbuf = act1 + (size_t)TM * p.stride1;  // two slabs of 64 x WS
    float* s_scale = reinterpret_cast<float*>(wbuf + 2 * kMlpTN * WS);
    float* s_shift = s_scale + p.max_cout;
    int* s_slot = reinterpret_cast<int*>(s_shift + p.max_cout);  // per tile row: its group's slot in s_max, -1 = no row
    unsigned* s_max = reinterpret_cast<unsigned*>(s_slot + TM);   // (groups_per_tile, last cout) keys

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = p.nsample;
    const int cout_last = p.layer[p.nlayers - 1].cout;
    const long long group0 = (long long)blockIdx.x * p.groups_per_tile;
    const int pieces = K > TM ? (K + TM - 1) / TM : 1;
    const int cin0 = p.layer[0].cin;
    const int cin0_pad = (cin0 + kMlpKS - 1) / kMlpKS * kMlpKS;

    for (int e = tid; e < p.groups_per_tile * cout_last; e += kMlpThreads) s_max[e] = 0u;

    for (int piece = 0; piece < pieces; ++piece) {
        // ---- gather: one warp per row, lanes over the row's channels; unused rows and the padding columns are 0 ----
        for (int r = warp; r < TM; r += kMlpThreads / 32) {
            int slot, k;
            if (K > TM) {
                slot = 0;
                k = piece * TM + r;
            } else {
                slot = r / K;
                k = r - slot * K;
            }
            const long long g = group0 + slot;
            const bool live = k < K && slot < p.groups_per_tile && g < p.groups;
            if (lane == 0) s_slot[r] = live ? slot : -1;
            T* row = act0 + (size_t)r * p.stride0;
            if (!live) {
                for (int ch = lane; ch < cin0_pad; ch += 32) row[ch] = from_f32<T>(0.f);
                continue;
            }
            const long long cloud = g / p.m;
            const int a = p.idx ? __ldg(p.idx + g * K + k) : k;
            if (p.xyz_lo >= 0 && lane < 3) {
                const float ctr = p.new_xyz ? __ldg(p.new_xyz + g * 3 + lane) : 0.f;
                row[p.xyz_lo + lane] = from_f32<T>(__fsub_rn(__ldg(p.xyz + (cloud * p.n + a) * 3 + lane), ctr));
            }
            if (p.points) {
                const T* src = static_cast<const T*>(p.points) + (cloud * p.n + a) * p.c;
                for (int ch = lane; ch < p.c; ch += 32) row[p.feat_lo + ch] = src[ch];
            }
            for (int ch = cin0 + lane; ch < cin0_pad; ch += 32) row[ch] = from_f32<T>(0.f);
        }
        __syncthreads();

        // ---- the layers ----
        for (int l = 0; l < p.nlayers; ++l) {
            const SaMlpLayer& L = p.layer[l];
            const bool last = l + 1 == p.nlayers;
            const T* ain = (l & 1) ? act1 : act0;
            T* aout = (l & 1) ? act0 : act1;
            const int sa = (l & 1) ? p.stride1 : p.stride0, so = (l & 1) ? p.stride0 : p.stride1;
            const int cout_pad = (L.cout + kMlpKS - 1) / kMlpKS * kMlpKS;

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
                    // ---- epilogue of this pass: affine + ReLU, then to the other buffer or into the running maximum ----
                    // element i of acc is (row_of(i), col_of(i)); a thread's rows lie in [row_lo, row_lo + row_span)
                    int row_lo, row_span;
                    if constexpr (TL::kMma) {
                        row_lo = (warp % TL::WM) * 16;
                        row_span = 16;
                    } else {
                        row_lo = (warp * 2) * TL::RM;  // the warp's two ty
                        row_span = 2 * TL::RM;
                    }
                    auto row_of = [&](int i) {
                        if constexpr (TL::kMma) return (warp % TL::WM) * 16 + (lane >> 2) + ((i & 2) ? 8 : 0);
                        else return (tid >> 4) * TL::RM + i / 4;
                    };
                    auto col_of = [&](int i) {
                        if constexpr (TL::kMma) return pass * kMlpTN + (warp / TL::WM) * 8 * TL::NT + (i / 4) * 8 + (lane & 3) * 2 + (i & 1);
                        else return pass * kMlpTN + (tid & 15) + 16 * (i & 3);
                    };
                    float y[TL::kAcc];
#pragma unroll
                    for (int i = 0; i < TL::kAcc; ++i) {
                        const int col = col_of(i);
                        float v = 0.f;
                        if (col < L.cout) {
                            v = __fmaf_rn(acc[i], s_scale[col], s_shift[col]);
                            if (L.relu) v = relu_nan(v);
                        }
                        y[i] = v;
                    }
                    if (!last) {
#pragma unroll
                        for (int i = 0; i < TL::kAcc; ++i) {
                            const int col = col_of(i);
                            if (col < cout_pad) aout[(size_t)row_of(i) * so + col] = from_f32<T>(y[i]);  // 0 beyond cout
                        }
                    } else {
                        const int s_lo = s_slot[row_lo], s_hi = s_slot[row_lo + row_span - 1];
                        if (s_lo >= 0 && s_lo == s_hi) {
                            // every row of the warp belongs to one group: reduce in registers and across the lanes that
                            // hold the same column, then one update per column
                            if constexpr (TL::kMma) {
#pragma unroll
                                for (int nt = 0; nt < TL::NT; ++nt)
#pragma unroll
                                    for (int h = 0; h < 2; ++h) {
                                        unsigned key = max(max_key(y[nt * 4 + h]), max_key(y[nt * 4 + 2 + h]));
                                        key = max(key, __shfl_xor_sync(kFullMask, key, 4));
                                        key = max(key, __shfl_xor_sync(kFullMask, key, 8));
                                        key = max(key, __shfl_xor_sync(kFullMask, key, 16));
                                        const int col = col_of(nt * 4 + h);
                                        if (lane < 4 && col < L.cout) atomicMax(s_max + s_lo * cout_last + col, key);
                                    }
                            } else {
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    unsigned key = max_key(y[j]);
#pragma unroll
                                    for (int i = 1; i < TL::RM; ++i) key = max(key, max_key(y[i * 4 + j]));
                                    key = max(key, __shfl_xor_sync(kFullMask, key, 16));
                                    const int col = col_of(j);
                                    if (lane < 16 && col < L.cout) atomicMax(s_max + s_lo * cout_last + col, key);
                                }
                            }
                        } else {
#pragma unroll
                            for (int i = 0; i < TL::kAcc; ++i) {
                                const int col = col_of(i), slot = s_slot[row_of(i)];
                                if (slot >= 0 && col < L.cout) atomicMax(s_max + slot * cout_last + col, max_key(y[i]));
                            }
                        }
                    }
                }
                if (t + 1 < total) land(t + 1);
                __syncthreads();
            }
        }
    }

    // ---- the groups' maxima, rounded once to the output type ----
    T* out = static_cast<T*>(p.out);
    for (int e = tid; e < p.groups_per_tile * cout_last; e += kMlpThreads) {
        const int slot = e / cout_last, col = e - slot * cout_last;
        const long long g = group0 + slot;
        if (g < p.groups) out[g * p.out_stride + col] = from_f32<T>(key_value(s_max[e]));
    }
}

// Shared memory of a tile of TM rows with `slots` group slots, in bytes
template <typename T>
static size_t sa_mlp_smem(const SaMlpParams& p, int tm, int slots) {
    const int cout_last = p.layer[p.nlayers - 1].cout;
    return sizeof(T) * ((size_t)tm * (p.stride0 + p.stride1) + 2 * kMlpTN * slab_stride<T>()) +
           sizeof(float) * 2 * (size_t)p.max_cout + sizeof(int) * (size_t)tm + sizeof(unsigned) * (size_t)slots * cout_last;
}

template <typename T, int TM>
static int sa_mlp_launch(const SaMlpParams& p, size_t smem, cudaStream_t st) {
    static AttrOnce once;
    // the opt-in is raised to the limit once, so that one setting serves every shape
    cudaError_t e = ensure_attrs(once, sa_mlp_max_kernel<T, TM>, kMlpSmemLimit, false);
    if (e != cudaSuccess) return (int)e;
    const long long tiles = (p.groups + p.groups_per_tile - 1) / p.groups_per_tile;
    if (tiles > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    sa_mlp_max_kernel<T, TM><<<(unsigned)tiles, kMlpThreads, smem, st>>>(p);
    return finish_launch();
}

// The row tile is the largest of 64 / 32 / 16 whose buffers fit (the widths decide: [256, 512, 1024] on 643 inputs
// takes 32 rows in float32 and 64 in 16 bits); groups of at most TM rows share a tile, as many as fit.
template <typename T>
static int sa_mlp_plan_launch(SaMlpParams& p, cudaStream_t st) {
    int w0 = p.layer[0].cin, w1 = 1;  // widest rows of buffer 0 (input, outputs of layers 1, 3) and 1 (layers 0, 2)
    for (int l = 0; l + 1 < p.nlayers; ++l) {
        int& w = (l & 1) ? w0 : w1;
        if (p.layer[l].cout > w) w = p.layer[l].cout;
    }
    p.stride0 = act_stride<T>(w0);
    p.stride1 = act_stride<T>(w1);
    for (int tm = 64; tm >= 16; tm >>= 1) {
        if (sa_mlp_smem<T>(p, tm, 1) > kMlpSmemLimit) continue;
        int slots = p.nsample <= tm ? tm / p.nsample : 1;
        while (slots > 1 && sa_mlp_smem<T>(p, tm, slots) > kMlpSmemLimit) --slots;
        p.groups_per_tile = slots;
        const size_t smem = sa_mlp_smem<T>(p, tm, slots);
        if (tm == 64) return sa_mlp_launch<T, 64>(p, smem, st);
        if (tm == 32) return sa_mlp_launch<T, 32>(p, smem, st);
        return sa_mlp_launch<T, 16>(p, smem, st);
    }
    return (int)cudaErrorInvalidValue;
}

}  // namespace pn2

extern "C" int pn2_sa_mlp_max_typed(int dtype, int b, int n, int c, int m, int nsample, const float* xyz,
                                    const float* new_xyz, const void* points, const int* idx, int xyz_first, int use_xyz,
                                    int nlayers, const int* widths, const float* const* weight, const float* const* bias,
                                    const float* const* bn_weight, const float* const* bn_bias,
                                    const float* const* bn_mean, const float* const* bn_var, const float* bn_eps,
                                    const int* relu, void* out, long long out_row_stride, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype) || b < 0 || n <= 0 || c < 0 || m < 0 || nsample <= 0) return (int)cudaErrorInvalidValue;
    if (nlayers < 1 || nlayers > kMlpMaxLayers || !widths || !weight || !bias || !relu) return (int)cudaErrorInvalidValue;
    if (!points) c = 0;
    const bool with_xyz = use_xyz || c == 0;
    const int cin = c + (with_xyz ? 3 : 0);
    if (cin > kMlpMaxIn || (!idx && nsample != n)) return (int)cudaErrorInvalidValue;
    SaMlpParams p{};
    int prev = cin;
    for (int l = 0; l < nlayers; ++l) {
        if (widths[l] < 1 || widths[l] > kMlpMaxWidth || !weight[l]) return (int)cudaErrorInvalidValue;
        const bool has_bn = bn_mean && bn_mean[l];
        if (has_bn && (!bn_var || !bn_var[l] || !bn_eps)) return (int)cudaErrorInvalidValue;
        p.layer[l] = SaMlpLayer{weight[l], bias[l], has_bn && bn_weight ? bn_weight[l] : nullptr,
                                has_bn && bn_bias ? bn_bias[l] : nullptr, has_bn ? bn_mean[l] : nullptr,
                                has_bn ? bn_var[l] : nullptr, has_bn ? bn_eps[l] : 0.f, prev, widths[l], relu[l] != 0};
        if (widths[l] > p.max_cout) p.max_cout = widths[l];
        prev = widths[l];
    }
    if (out_row_stride < prev) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz || !out) return (int)cudaErrorInvalidValue;
    p.xyz = xyz;
    p.new_xyz = new_xyz;
    p.points = points;
    p.idx = idx;
    p.out = out;
    p.out_stride = out_row_stride;
    p.groups = (long long)b * m;
    p.n = n;
    p.c = c;
    p.m = m;
    p.nsample = nsample;
    p.xyz_lo = with_xyz ? (xyz_first ? 0 : c) : -1;
    p.feat_lo = with_xyz && xyz_first ? 3 : 0;
    p.nlayers = nlayers;
    if (dtype == PN2_F32) return sa_mlp_plan_launch<float>(p, as_stream(stream));
    if (dtype == PN2_BF16) return sa_mlp_plan_launch<__nv_bfloat16>(p, as_stream(stream));
    return sa_mlp_plan_launch<__half>(p, as_stream(stream));
}
