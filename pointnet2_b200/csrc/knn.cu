// knn.cu — knn_point for sm_90a: tiled brute-force top-k without the (b,m,n) distance matrix.
//
// Replaces the reference's composite (tf_ops/grouping/tf_grouping.py:48-73):
//   dist = reduce_sum((tile(xyz1) - tile(xyz2))**2, -1)          # (b,m,n) matrix in HBM
//   outi, out = select_top_k(k, dist)                            # selection_sort_gpu, tf_grouping_g.cu:83-123
//   idx, val = slice(outi, k), slice(out, k)
// which at (32, 1024, 4096) materialises 1.6 GB of differences, a 537 MB matrix and two more
// (b,m,n) outputs, and runs k rounds of selection sort over whole rows.
//
// Semantics kept bit for bit — including ties, which duplicate-heavy clouds produce all the time:
//   * distance = ((dx*dx + dy*dy) + dz*dz), every product and sum rounded on its own (element-wise
//     square, then a 3-term sum, as the graph computes it);
//   * selection sort does k rounds of "first minimum of v[s..n) by strict '<', SWAP it into place s".
//     The swap moves the element that sat at s to the winner's old position, so ties are NOT simply
//     broken by original index.  Only two kinds of elements can ever move or be selected: the k
//     elements that start at positions < k (set A) and the k smallest of the rest under
//     (value, position) (set B) — every other element keeps its position and always loses to an
//     unselected member of B.  So the kernel (1) scans the row once, keeping A in shared memory and
//     a top-k list B in registers (one entry per lane and register, unsorted: an insertion is a few
//     ballots and shuffles), then (2) replays the k rounds on those <= 2k elements with their
//     current positions.  The result equals the first k columns of selection_sort_gpu exactly.
//
// One warp per query; the data points of the query's cloud are staged through shared-memory tiles
// shared by the CTA's 8 warps (coordinates as SoA: consecutive lanes read consecutive words).
//
// The per-query work (set A, the register list B, the replay) is KnnWarp in knn_warp.cuh, which the overlapped kNN
// set-abstraction layer (sa_fused.cu) runs as well; this kernel stages the tiles and feeds it.
#include "knn_warp.cuh"

namespace pn2 {

constexpr int kKnnThreads = 256;
constexpr int kKnnWarps = kKnnThreads / 32;
constexpr int kKnnTile = 1024;  // data points per shared-memory tile

// L (ragged batch): data cloud i is its first cloud_length(lengths1, i, n) points, query cloud i its first
// cloud_length(lengths2, i, m) queries (lengths2 == NULL: all m).  A template flag, so that the instances without lengths
// compile to the code they always did.  A cloud shorter than k runs KnnWarp with k_i = min(k, len) (KC still chosen
// from k): its columns [0, k_i) are knn_point(k_i) on the truncated cloud, and finish takes its usual ka == k entry;
// columns [k_i, k) repeat column 0.  Query rows past their length get idx 0 / val +inf.
template <int KC, bool L>  // KC: registers per lane that hold the list B: k <= 32 * KC
__global__ void __launch_bounds__(kKnnThreads)
knn_kernel(int n, int m, int k, const float* __restrict__ xyz1, const float* __restrict__ xyz2, float* __restrict__ val,
           int* __restrict__ idx, const int* __restrict__ lengths1, const int* __restrict__ lengths2) {
    __shared__ float s_x[kKnnTile], s_y[kKnnTile], s_z[kKnnTile];
    // per warp: W[0..k) = set A (positions 0..k-1), W[k..2k) = set B (in no particular order)
    __shared__ float s_wv[kKnnWarps][2 * kKnnMaxK];
    __shared__ int s_wo[kKnnWarps][2 * kKnnMaxK];  // original index
    __shared__ int s_wp[kKnnWarps][2 * kKnnMaxK];  // current position (phase 2)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.y;
    const int q = blockIdx.x * kKnnWarps + warp;
    const int len = L ? cloud_length(lengths1, cloud, n) : n;  // data points of this cloud: padding is never loaded
    const bool valid = q < (L ? cloud_length(lengths2, cloud, m) : m);
    const float* __restrict__ data = xyz1 + (size_t)cloud * n * 3;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (valid) {
        const float* qp = xyz2 + ((size_t)cloud * m + q) * 3;
        qx = __ldg(qp);
        qy = __ldg(qp + 1);
        qz = __ldg(qp + 2);
    }
    float* __restrict__ wv = s_wv[warp];
    int* __restrict__ wo = s_wo[warp];
    const int kq = L ? min(k, len) : k;  // columns the selection produces for this cloud
    KnnWarp<KC> w(kq, lane, qx, qy, qz);
    const int ka = min(kq, len);  // |A|
    // set A straight from global memory: at most 128 points
    if (valid)
        for (int pos = lane; pos < ka; pos += 32) {
            const float* s = data + (size_t)pos * 3;
            w.put_a(wv, wo, pos, __ldg(s), __ldg(s + 1), __ldg(s + 2));
        }
    for (int base = 0; base < len; base += kKnnTile) {
        const int tn = min(kKnnTile, len - base);
        __syncthreads();  // previous tile consumed
        for (int p = tid; p < tn; p += kKnnThreads) {
            const float* s = data + (size_t)(base + p) * 3;
            s_x[p] = __ldg(s);
            s_y[p] = __ldg(s + 1);
            s_z[p] = __ldg(s + 2);
        }
        __syncthreads();
        if (valid) w.offer(s_x, s_y, s_z, tn, base);
    }
    if (!valid) {
        if (L && q < m)  // a query row past its cloud's length: the missing-neighbour filler
            for (int e = lane; e < k; e += 32) {
                val[((size_t)cloud * m + q) * k + e] = INFINITY;
                idx[((size_t)cloud * m + q) * k + e] = 0;
            }
        return;
    }
    float* __restrict__ oval = val + ((size_t)cloud * m + q) * k;
    int* __restrict__ oidx = idx + ((size_t)cloud * m + q) * k;
    w.finish(wv, wo, s_wp[warp], ka, [&](int e, float v, int i) {
        oval[e] = v;
        oidx[e] = i;
    });
    if (L && kq < k) {  // a cloud shorter than k: columns [kq, k) repeat column 0, as the ball query pads a short row
        __syncwarp();   // the replay's column 0 was written by lane 0
        const float v0 = oval[0];
        const int i0 = oidx[0];
        for (int e = kq + lane; e < k; e += 32) {
            oval[e] = v0;
            oidx[e] = i0;
        }
    }
}

// pn2_knn_point on the clouds' first lengths1[b] points and the first lengths2[b] queries (NULL: all n / all m)
static int knn_point(int b, int n, int m, int k, const float* xyz1, const int* lengths1, const float* xyz2, const int* lengths2,
                     float* val, int* idx, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0 || k <= 0 || k > kKnnMaxK || k > n) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!xyz1 || !xyz2 || !val || !idx || b > 65535) return (int)cudaErrorInvalidValue;
    dim3 grid((m + kKnnWarps - 1) / kKnnWarps, b, 1);
    auto kern = k <= 32 ? knn_kernel<1, false> : k <= 64 ? knn_kernel<2, false> : knn_kernel<4, false>;
    if (lengths1 || lengths2) kern = k <= 32 ? knn_kernel<1, true> : k <= 64 ? knn_kernel<2, true> : knn_kernel<4, true>;
    kern<<<grid, kKnnThreads, 0, st>>>(n, m, k, xyz1, xyz2, val, idx, lengths1, lengths2);
    return finish_launch();
}

}  // namespace pn2

extern "C" {

int pn2_knn_point(int b, int n, int m, int k, const float* xyz1, const float* xyz2, float* val, int* idx, void* stream) {
    return pn2::knn_point(b, n, m, k, xyz1, nullptr, xyz2, nullptr, val, idx, pn2::as_stream(stream));
}

int pn2_knn_point_ragged(int b, int n, int m, int k, const float* xyz1, const int* lengths1, const float* xyz2, const int* lengths2,
                         float* val, int* idx, void* stream) {
    return pn2::knn_point(b, n, m, k, xyz1, lengths1, xyz2, lengths2, val, idx, pn2::as_stream(stream));
}

}  // extern "C"
