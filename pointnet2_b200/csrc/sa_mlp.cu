// sa_mlp.cu — the inference tail of a set-abstraction level in one launch, for sm_90a:
//   gather (utils/pointnet_util.py:45-54 / :179-186)  ->  shared MLP, each layer 1x1 conv + eval-mode batch norm + ReLU
//   (:115-121 / :187-190)  ->  max over the group's rows (:124 / :191).
// Nothing of shape (b*m*nsample, .) reaches global memory: a CTA holds a tile of TM rows (whole groups, or one piece of
// a group larger than the tile) in shared memory, the activations ping-pong between two shared buffers from layer to
// layer, and the last layer's accumulators go from registers into a per-group running maximum.
//
// The tile, the weight slabs and the per-layer loop are mlp_tile.cuh's (shared with fp_mlp.cu).
// Every output depends on its own group only and every sum has a fixed order, so results are bit-identical from run to
// run and whatever else is in the batch.  The maximum keeps NaN (torch's max does; fmaxf would drop it): values are
// compared as order-preserving integer keys in which NaN is the largest.
#include <type_traits>

#include "mlp_tile.cuh"

namespace pn2 {

constexpr int kMlpMaxIn = kMlpMaxWidth + 3;

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
    MlpLayer layer[kMlpMaxLayers];
};

// float -> key with  a < b  <=>  key(a) < key(b)  as unsigned, every NaN the largest key; 0 is below every key
__device__ __forceinline__ unsigned max_key(float v) {
    if (v != v) return 0xffffffffu;
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <typename T, int TM>
__global__ void __launch_bounds__(kMlpThreads, sizeof(T) == 4 && TM == 64 ? 1 : 2)
sa_mlp_max_kernel(const __grid_constant__ SaMlpParams p) {
    using TL = Tile<T, TM>;
    extern __shared__ __align__(16) unsigned char smem[];
    T* act0 = reinterpret_cast<T*>(smem);
    T* act1 = act0 + (size_t)TM * p.stride0;
    T* wbuf = act1 + (size_t)TM * p.stride1;  // two slabs of 64 x slab_stride
    float* s_scale = reinterpret_cast<float*>(wbuf + slab_elems<T>());
    float* s_shift = s_scale + p.max_cout;
    int* s_slot = reinterpret_cast<int*>(s_shift + p.max_cout);  // per tile row: its group's slot in s_max, -1 = no row
    unsigned* s_max = reinterpret_cast<unsigned*>(s_slot + TM);   // (groups_per_tile, last cout) keys

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = p.nsample;
    const int cout_last = p.layer[p.nlayers - 1].cout;
    const long long group0 = (long long)blockIdx.x * p.groups_per_tile;
    const int pieces = K > TM ? (K + TM - 1) / TM : 1;
    const int cin0 = p.layer[0].cin;
    const int cin0_pad = slab_pad(cin0);

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

        // ---- the layers; the last one's results go into the running maximum of their group ----
        mlp_tile_layers<T, TM, false>(p.layer, p.nlayers, act0, act1, p.stride0, p.stride1, wbuf, s_scale, s_shift,
                                      [&](const float (&y)[TL::kAcc], int pass) {
            const int row_lo = TL::row_lo();
            const int s_lo = s_slot[row_lo], s_hi = s_slot[row_lo + TL::kRowSpan - 1];
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
                            const int col = TL::col_of(nt * 4 + h, pass);
                            if (lane < 4 && col < cout_last) atomicMax(s_max + s_lo * cout_last + col, key);
                        }
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        unsigned key = max_key(y[j]);
#pragma unroll
                        for (int i = 1; i < TL::RM; ++i) key = max(key, max_key(y[i * 4 + j]));
                        key = max(key, __shfl_xor_sync(kFullMask, key, 16));
                        const int col = TL::col_of(j, pass);
                        if (lane < 16 && col < cout_last) atomicMax(s_max + s_lo * cout_last + col, key);
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < TL::kAcc; ++i) {
                    const int col = TL::col_of(i, pass), slot = s_slot[TL::row_of(i)];
                    if (slot >= 0 && col < cout_last) atomicMax(s_max + slot * cout_last + col, max_key(y[i]));
                }
            }
        });
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
    return sizeof(T) * ((size_t)tm * (p.stride0 + p.stride1) + slab_elems<T>()) +
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
    if (!points) c = 0;
    const bool with_xyz = use_xyz || c == 0;
    const int cin = c + (with_xyz ? 3 : 0);
    if (cin > kMlpMaxIn || (!idx && nsample != n)) return (int)cudaErrorInvalidValue;
    SaMlpParams p{};
    if (!mlp_layers_from_args(p.layer, p.max_cout, cin, nlayers, widths, weight, bias, bn_weight, bn_bias, bn_mean, bn_var,
                              bn_eps, relu))
        return (int)cudaErrorInvalidValue;
    const int prev = widths[nlayers - 1];
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
