// fp_mlp.cu — row-wise fused inference MLPs for sm_90a: up to four Linear [+ eval-mode batch norm] [+ ReLU] layers
// applied to every row of a tensor, one output row per input row, on the tile machinery of sa_mlp.cu (mlp_tile.cuh).
// Two front ends fill a tile's rows:
//   feature propagation (utils/pointnet_util.py:199-229): row j of cloud i is
//       concat(interpolate(points2[i] at the 3-NN of xyz1[i, j] in xyz2[i]), points1[i, j]),
//   with the 3-NN indices and weights from fp_front_kernel (interpolate.cu) in a small workspace and the interpolation
//   done here with the same interp3, so the first layer reads exactly what pn2_fp_interpolate_concat_typed would write,
//   and no (b, n, c2 + c1) tensor reaches HBM;
//   plain rows: row r is x[r] (the segmentation and classifier heads).
// Padding rows (j >= the cloud's length, or a zero mask byte) are never read and are written as 0.  The last layer
// writes its rounded results to the free activation buffer, from which the tile's rows go out through a row stride.
// Every output row depends on its own input row alone and every sum has a fixed order, so results are the same bits at
// every batch size and next to any other row.
#include "mlp_tile.cuh"

namespace pn2 {

constexpr int kRowMlpMaxIn = 1536;  // first-layer inputs: PointNet2PartSegMSG.fp1 takes 512 + 1024

struct RowMlpParams {
    const void* x;              // (rows, c) in T: the rows (plain front end) or points1 (feature propagation); nullptr: c = 0
    const unsigned char* mask;  // plain front end: (rows,) nonzero on the real rows, or nullptr (every row is real)
    const int* nn_idx;          // feature propagation: (rows, 3) neighbour indices into xyz2; nullptr: the plain front end
    const float* nn_w;          // feature propagation: (rows, 3) their weights
    const void* points2;        // feature propagation: (b, m, c2) in T
    const int* lengths;         // feature propagation: (b,) real rows per cloud, or nullptr
    void* out;
    long long out_stride;       // elements between consecutive rows of out
    long long rows;             // b * n
    int n, m, c, c2;
    int nlayers;
    int stride0, stride1;       // row strides of the two activation buffers, in elements
    int max_cout;
    MlpLayer layer[kMlpMaxLayers];
};

template <typename T, int TM>
__global__ void __launch_bounds__(kMlpThreads, sizeof(T) == 4 && TM == 64 ? 1 : 2)
row_mlp_kernel(const __grid_constant__ RowMlpParams p) {
    extern __shared__ __align__(16) unsigned char smem[];
    T* act0 = reinterpret_cast<T*>(smem);
    T* act1 = act0 + (size_t)TM * p.stride0;
    T* wbuf = act1 + (size_t)TM * p.stride1;
    float* s_scale = reinterpret_cast<float*>(wbuf + slab_elems<T>());
    float* s_shift = s_scale + p.max_cout;
    int* s_live = reinterpret_cast<int*>(s_shift + p.max_cout);  // per tile row: 1 = a real row, 0 = padding or none

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long row0 = (long long)blockIdx.x * TM;
    const int cin0 = p.layer[0].cin, cin0_pad = slab_pad(cin0);

    // ---- gather: one warp per row, lanes over the row's channels; padding rows and the padding columns are 0 ----
    for (int r = warp; r < TM; r += kMlpThreads / 32) {
        const long long g = row0 + r;
        bool live = g < p.rows;
        long long cloud = 0;
        if (live) {
            if (p.nn_idx) {
                cloud = g / p.n;
                live = g - cloud * p.n < cloud_length(p.lengths, (int)cloud, p.n);
            } else if (p.mask) {
                live = __ldg(p.mask + g) != 0;
            }
        }
        if (lane == 0) s_live[r] = live ? 1 : 0;
        T* row = act0 + (size_t)r * p.stride0;
        if (!live) {
            for (int ch = lane; ch < cin0_pad; ch += 32) row[ch] = from_f32<T>(0.f);
            continue;
        }
        int lo = 0;
        if (p.nn_idx) {
            const int i1 = __ldg(p.nn_idx + g * 3), i2 = __ldg(p.nn_idx + g * 3 + 1), i3 = __ldg(p.nn_idx + g * 3 + 2);
            const float w1 = __ldg(p.nn_w + g * 3), w2 = __ldg(p.nn_w + g * 3 + 1), w3 = __ldg(p.nn_w + g * 3 + 2);
            const T* pb = static_cast<const T*>(p.points2) + cloud * p.m * p.c2;
            const T *a = pb + (size_t)i1 * p.c2, *b = pb + (size_t)i2 * p.c2, *c = pb + (size_t)i3 * p.c2;
            for (int ch = lane; ch < p.c2; ch += 32)
                row[ch] = from_f32<T>(interp3(to_f32(a[ch]), to_f32(b[ch]), to_f32(c[ch]), w1, w2, w3));
            lo = p.c2;
        }
        if (p.x) {
            const T* src = static_cast<const T*>(p.x) + g * p.c;
            for (int ch = lane; ch < p.c; ch += 32) row[lo + ch] = src[ch];
        }
        for (int ch = cin0 + lane; ch < cin0_pad; ch += 32) row[ch] = from_f32<T>(0.f);
    }
    __syncthreads();

    // ---- the layers, every one of them stored to the other activation buffer ----
    mlp_tile_layers<T, TM, true>(p.layer, p.nlayers, act0, act1, p.stride0, p.stride1, wbuf, s_scale, s_shift,
                                 [](const float (&)[Tile<T, TM>::kAcc], int) {});

    // ---- the tile's rows, consecutive threads on consecutive channels ----
    const T* res = (p.nlayers & 1) ? act1 : act0;
    const int rs = (p.nlayers & 1) ? p.stride1 : p.stride0;
    const int cout = p.layer[p.nlayers - 1].cout;
    T* out = static_cast<T*>(p.out);
    for (int e = tid; e < TM * cout; e += kMlpThreads) {
        const int r = e / cout, col = e - r * cout;
        const long long g = row0 + r;
        if (g < p.rows) out[g * p.out_stride + col] = s_live[r] ? res[(size_t)r * rs + col] : from_f32<T>(0.f);
    }
}

// Shared memory of a tile of TM rows, in bytes
template <typename T>
static size_t row_mlp_smem(const RowMlpParams& p, int tm) {
    return sizeof(T) * ((size_t)tm * (p.stride0 + p.stride1) + slab_elems<T>()) + sizeof(float) * 2 * (size_t)p.max_cout +
           sizeof(int) * (size_t)tm;
}

template <typename T, int TM>
static int row_mlp_launch(const RowMlpParams& p, size_t smem, cudaStream_t st) {
    static AttrOnce once;
    cudaError_t e = ensure_attrs(once, row_mlp_kernel<T, TM>, kMlpSmemLimit, false);
    if (e != cudaSuccess) return (int)e;
    const long long tiles = (p.rows + TM - 1) / TM;
    if (tiles > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    row_mlp_kernel<T, TM><<<(unsigned)tiles, kMlpThreads, smem, st>>>(p);
    return finish_launch();
}

// The row tile is the largest of 64 / 32 / 16 whose buffers fit, as in sa_mlp_plan_launch; here the last layer's
// output takes a buffer too.  A function of the widths alone, never of the row count.
template <typename T>
static int row_mlp_plan_launch(RowMlpParams& p, cudaStream_t st) {
    int w0 = p.layer[0].cin, w1 = 1;  // widest rows of buffer 0 (input, outputs of layers 1, 3) and 1 (layers 0, 2)
    for (int l = 0; l < p.nlayers; ++l) {
        int& w = (l & 1) ? w0 : w1;
        if (p.layer[l].cout > w) w = p.layer[l].cout;
    }
    p.stride0 = act_stride<T>(w0);
    p.stride1 = act_stride<T>(w1);
    for (int tm = 64; tm >= 16; tm >>= 1) {
        const size_t smem = row_mlp_smem<T>(p, tm);
        if (smem > kMlpSmemLimit) continue;
        if (tm == 64) return row_mlp_launch<T, 64>(p, smem, st);
        if (tm == 32) return row_mlp_launch<T, 32>(p, smem, st);
        return row_mlp_launch<T, 16>(p, smem, st);
    }
    return (int)cudaErrorInvalidValue;
}

static int row_mlp_dispatch(int dtype, RowMlpParams& p, cudaStream_t st) {
    if (dtype == PN2_F32) return row_mlp_plan_launch<float>(p, st);
    if (dtype == PN2_BF16) return row_mlp_plan_launch<__nv_bfloat16>(p, st);
    return row_mlp_plan_launch<__half>(p, st);
}

constexpr size_t kFpMlpAlign = 256;
inline size_t fp_mlp_part_bytes(long long rows) { return ((size_t)rows * 3 * 4 + kFpMlpAlign - 1) / kFpMlpAlign * kFpMlpAlign; }

}  // namespace pn2

extern "C" {

size_t pn2_fp_mlp_workspace_bytes(int b, int n) {
    if (b <= 0 || n <= 0) return 0;
    return 2 * pn2::fp_mlp_part_bytes((long long)b * n);
}

int pn2_fp_mlp_typed(int dtype, int b, int n, int m, int c2, int c1, const float* xyz1, const int* lengths1,
                     const float* xyz2, const void* points1, const void* points2, int nlayers, const int* widths,
                     const float* const* weight, const float* const* bias, const float* const* bn_weight,
                     const float* const* bn_bias, const float* const* bn_mean, const float* const* bn_var,
                     const float* bn_eps, const int* relu, void* out, long long out_row_stride, void* workspace,
                     size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype) || b < 0 || n < 0 || m <= 0 || c2 <= 0 || c1 < 0) return (int)cudaErrorInvalidValue;
    if (!points1) c1 = 0;
    if (c2 + c1 > kRowMlpMaxIn || b > 65535) return (int)cudaErrorInvalidValue;
    RowMlpParams p{};
    if (!mlp_layers_from_args(p.layer, p.max_cout, c2 + c1, nlayers, widths, weight, bias, bn_weight, bn_bias, bn_mean,
                              bn_var, bn_eps, relu))
        return (int)cudaErrorInvalidValue;
    if (out_row_stride < widths[nlayers - 1]) return (int)cudaErrorInvalidValue;
    if (b == 0 || n == 0) return 0;
    if (!xyz1 || !xyz2 || !points2 || !out || !workspace || workspace_bytes < pn2_fp_mlp_workspace_bytes(b, n))
        return (int)cudaErrorInvalidValue;
    const long long rows = (long long)b * n;
    int* nn_idx = static_cast<int*>(workspace);
    float* nn_w = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + fp_mlp_part_bytes(rows));
    // the 3-NN and their weights from the FP front end, without its output (c = 0 writes no features)
    const int rc = pn2_three_nn_interpolate_ragged_typed(dtype, b, n, m, 0, xyz1, lengths1, xyz2, nullptr, nullptr, nullptr,
                                                         nn_idx, nn_w, stream);
    if (rc != 0) return rc;
    p.x = points1;
    p.nn_idx = nn_idx;
    p.nn_w = nn_w;
    p.points2 = points2;
    p.lengths = lengths1;
    p.out = out;
    p.out_stride = out_row_stride;
    p.rows = rows;
    p.n = n;
    p.m = m;
    p.c = c1;
    p.c2 = c2;
    p.nlayers = nlayers;
    return row_mlp_dispatch(dtype, p, as_stream(stream));
}

int pn2_mlp_rows_typed(int dtype, long long rows, int c, const void* x, const unsigned char* mask, int nlayers,
                       const int* widths, const float* const* weight, const float* const* bias,
                       const float* const* bn_weight, const float* const* bn_bias, const float* const* bn_mean,
                       const float* const* bn_var, const float* bn_eps, const int* relu, void* out,
                       long long out_row_stride, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype) || rows < 0 || c <= 0 || c > kRowMlpMaxIn) return (int)cudaErrorInvalidValue;
    RowMlpParams p{};
    if (!mlp_layers_from_args(p.layer, p.max_cout, c, nlayers, widths, weight, bias, bn_weight, bn_bias, bn_mean, bn_var,
                              bn_eps, relu))
        return (int)cudaErrorInvalidValue;
    if (out_row_stride < widths[nlayers - 1]) return (int)cudaErrorInvalidValue;
    if (rows == 0) return 0;
    if (!x || !out) return (int)cudaErrorInvalidValue;
    p.x = x;
    p.mask = mask;
    p.out = out;
    p.out_stride = out_row_stride;
    p.rows = rows;
    p.n = 1;
    p.c = c;
    p.nlayers = nlayers;
    return row_mlp_dispatch(dtype, p, as_stream(stream));
}

}  // extern "C"
