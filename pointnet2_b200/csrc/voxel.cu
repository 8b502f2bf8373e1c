// voxel.cu — voxel and pillar grouping: the cells of a V^3 grid (or of an I^2 grid of xy pillars) over [-radius,
// radius] as centroids, each holding up to nsample of its member rows, and those rows normalised to the cell
// (utils/pc_util.py point_cloud_to_volume, point_cloud_to_volume_v2, point_cloud_to_image; DESIGN.md §6.19).
//
// A counting sort of the batch's rows by cell, then one selection per cell, five launches and nothing read back:
//   count: one thread per row: the row's cell in float32, as numpy computes it; integer atomicAdd per cell (order-free);
//   scan:  one CTA per cloud: exclusive scan of the cloud's cell counts (cta_exclusive_scan_1024, as scene.cu's blocks);
//   fill:  one thread per row: the row goes to its cell's next slot (atomic cursor).  The order inside a cell is not
//          kept: every cell's rows are sorted by their order key below, so the fill needs no stable ranking;
//   warp:  one warp per cell of at most 128 rows: the rows' 64-bit order keys sorted in registers, the cell's nsample
//          slots written (c <= nsample: the rows ascending, the last repeated; c > nsample: the nsample smallest keys);
//          a larger cell is appended to a list;
//   cta:   1024-thread CTAs over that list: cta_select_sorted over the cell's rows (any count, the whole cloud
//          included), then the same writes.
// Order key of row j of cell e = b * cells + cell: j when c <= nsample, rng_row_key(seed, kStreamCell, e, j) otherwise.
#include <algorithm>

#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr unsigned long long kStreamCell = 9;  // the draws of over-full cells: a stream no other sampler uses
constexpr int kWarpKeys = 4;                   // order keys per lane in the warp kernel
constexpr int kWarpCell = 32 * kWarpKeys;      // cells of up to this many rows are served by one warp
constexpr int kRowThreads = 256;
constexpr int kWarpThreads = 256;
constexpr int kCtaThreads = 1024;

struct VoxelGrid {
    float radius_f, voxel_f, dim_f;  // radius and 2 * radius / dim rounded to float32; dim as a float
    double radius, voxel;            // the same in double, for the normalisation
    int dim, dims, cells;            // cells per axis, 2 or 3 axes, dim^dims
};

// Cell index along one axis, or -1: (p + radius) / voxel in float32, truncated toward zero, kept when the quotient
// lies in (-1, dim).  NaN and every quotient <= -1 or >= dim are in no cell.
__device__ __forceinline__ int voxel_axis(float p, const VoxelGrid& g) {
    const float q = __fdiv_rn(__fadd_rn(p, g.radius_f), g.voxel_f);
    return (q > -1.0f && q < g.dim_f) ? (int)q : -1;
}

// Cell of point p (3 floats), i-major ((i * dim + j) * dim + k, or i * dim + j for pillars), or -1.
__device__ __forceinline__ int voxel_cell(const float* __restrict__ p, const VoxelGrid& g) {
    const int i = voxel_axis(__ldg(p), g), j = voxel_axis(__ldg(p + 1), g);
    if (i < 0 || j < 0) return -1;
    if (g.dims == 2) return i * g.dim + j;
    const int k = voxel_axis(__ldg(p + 2), g);
    return k < 0 ? -1 : (i * g.dim + j) * g.dim + k;
}

// Coordinate d of cell `cell` along its axis.
__device__ __forceinline__ int cell_coord(int cell, int d, const VoxelGrid& g) {
    if (g.dims == 2) return d == 0 ? cell / g.dim : cell % g.dim;
    return d == 0 ? cell / (g.dim * g.dim) : (d == 1 ? (cell / g.dim) % g.dim : cell % g.dim);
}

// Coordinate d of a member normalised to its cell: (p - ((c + 0.5) * voxel - radius)) / voxel in double, each
// operation rounded; for pillars x and y are then rounded to float32 and z is the raw coordinate.
__device__ __forceinline__ double voxel_norm(float p, int cell, int d, const VoxelGrid& g) {
    if (g.dims == 2 && d == 2) return (double)p;
    const double centre = __dsub_rn(__dmul_rn((double)cell_coord(cell, d, g) + 0.5, g.voxel), g.radius);
    const double v = __ddiv_rn(__dsub_rn((double)p, centre), g.voxel);
    return g.dims == 2 ? (double)__double2float_rn(v) : v;
}

struct VoxelArgs {
    const float* xyz;
    const int* lengths;
    const long long* seed_dev;
    unsigned long long seed;
    int b, n, nsample;
};

__global__ void __launch_bounds__(kRowThreads) voxel_count_kernel(VoxelArgs a, VoxelGrid g, int* __restrict__ count) {
    const long long rows = (long long)a.b * a.n;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(r / a.n), j = (int)(r % a.n);
        if (j >= cloud_length0(a.lengths, b, a.n)) continue;
        const int cell = voxel_cell(a.xyz + 3 * r, g);
        if (cell >= 0) atomicAdd(count + (long long)b * g.cells + cell, 1);
    }
}

// CTA b: cursor[b, :] = exclusive scan of count[b, :] (the cloud's member list starts at cell 0's rows).
__global__ void __launch_bounds__(kCtaThreads) voxel_scan_kernel(int cells, const int* __restrict__ count, int* __restrict__ cursor) {
    __shared__ int s_w[32];
    __shared__ int s_carry;
    const long long off = (long long)blockIdx.x * cells;
    cta_exclusive_scan_1024(count + off, cursor + off, cells, s_w, &s_carry);
}

// member[b * n + cursor[b, cell]++] = j for every in-range row j of cloud b; afterwards cursor = start + count.
__global__ void __launch_bounds__(kRowThreads) voxel_fill_kernel(VoxelArgs a, VoxelGrid g, int* __restrict__ cursor,
                                                                 int* __restrict__ member) {
    const long long rows = (long long)a.b * a.n;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(r / a.n), j = (int)(r % a.n);
        if (j >= cloud_length0(a.lengths, b, a.n)) continue;
        const int cell = voxel_cell(a.xyz + 3 * r, g);
        if (cell >= 0) member[(long long)b * a.n + atomicAdd(cursor + (long long)b * g.cells + cell, 1)] = j;
    }
}

struct VoxelOut {
    const int* count;
    const int* cursor;
    const int* member;
    int* idx;
    double* grouped;
    int* big;   // cells of more than kWarpCell rows, appended by the warp kernel
    int* nbig;
};

__device__ __forceinline__ unsigned long long order_key(unsigned long long seed, int c, int s, long long e, int j) {
    return c <= s ? (unsigned long long)j : rng_row_key(seed, kStreamCell, (unsigned long long)e, j);
}

// One warp per cell e of the batch.  Slot s of a cell of c rows holds its sorted row min(s, m - 1), m = min(c, S);
// an empty cell is all zeros.
__global__ void __launch_bounds__(kWarpThreads) voxel_warp_kernel(VoxelArgs a, VoxelGrid g, VoxelOut o) {
    __shared__ double s_val[kWarpThreads / 32][kWarpCell][3];
    __shared__ int s_row[kWarpThreads / 32][kWarpCell];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int S = a.nsample;
    const long long total = (long long)a.b * g.cells, warps = (long long)gridDim.x * (blockDim.x >> 5);
    const unsigned long long seed = rng_seed(a.seed_dev, a.seed);
    for (long long e = (long long)blockIdx.x * (blockDim.x >> 5) + w; e < total; e += warps) {
        const int c = __ldg(o.count + e);
        if (c > kWarpCell) {
            if (lane == 0) o.big[atomicAdd(o.nbig, 1)] = (int)e;
            continue;
        }
        const int b = (int)(e / g.cells), cell = (int)(e % g.cells);
        const int* rows = o.member + (long long)b * a.n + (__ldg(o.cursor + e) - c);
        unsigned long long key[kWarpKeys];  // element k of the cell: key[k / 32] of lane k % 32
#pragma unroll
        for (int r = 0; r < kWarpKeys; ++r) {
            const int k = 32 * r + lane;
            key[r] = k < c ? order_key(seed, c, S, e, __ldg(rows + k)) : ~0ull;
        }
        if (c <= 32) bitonic_sort_keys<1, kWarpKeys>(key, lane);
        else if (c <= 64) bitonic_sort_keys<2, kWarpKeys>(key, lane);
        else bitonic_sort_keys<4, kWarpKeys>(key, lane);
        const int m = min(c, S);
#pragma unroll
        for (int r = 0; r < kWarpKeys; ++r) {
            const int k = 32 * r + lane;
            if (k >= m) break;
            const int j = (int)(key[r] & 0xffffffffull);
            const float* p = a.xyz + 3 * ((long long)b * a.n + j);
            s_row[w][k] = j;
#pragma unroll
            for (int d = 0; d < 3; ++d) s_val[w][k][d] = voxel_norm(__ldg(p + d), cell, d, g);
        }
        __syncwarp();
        int* idx = o.idx + e * S;
        for (int s = lane; s < S; s += 32) __stcs(idx + s, m ? s_row[w][min(s, m - 1)] : 0);
        double* out = o.grouped + e * 3 * S;
        for (int k = lane; k < 3 * S; k += 32) __stcs(out + k, m ? s_val[w][min(k / 3, m - 1)][k % 3] : 0.0);
        __syncwarp();  // s_row / s_val are rewritten for the next cell
    }
}

// 1024-thread CTAs over the listed cells.  Dynamic shared memory: the sort buffer, pow2 >= nsample 64-bit keys.
__global__ void __launch_bounds__(kCtaThreads, 1) voxel_cta_kernel(VoxelArgs a, VoxelGrid g, VoxelOut o) {
    extern __shared__ unsigned long long s_keys[];
    __shared__ SelectScratch s_sel;
    const int S = a.nsample, tid = threadIdx.x;
    const int nbig = *o.nbig;  // written by voxel_warp_kernel
    const unsigned long long seed = rng_seed(a.seed_dev, a.seed);
    for (int t = blockIdx.x; t < nbig; t += gridDim.x) {
        const long long e = o.big[t];
        const int c = __ldg(o.count + e), m = min(c, S);
        const int b = (int)(e / g.cells), cell = (int)(e % g.cells);
        const int* rows = o.member + (long long)b * a.n + (__ldg(o.cursor + e) - c);
        cta_select_sorted(
            c, c, m, [](long long) { return true; }, [&](long long q) { return order_key(seed, c, S, e, __ldg(rows + q)); },
            s_keys, s_sel);
        int* idx = o.idx + e * S;
        for (int s = tid; s < S; s += blockDim.x) __stcs(idx + s, (int)(s_keys[min(s, m - 1)] & 0xffffffffull));
        double* out = o.grouped + e * 3 * S;
        for (int k = tid; k < 3 * S; k += blockDim.x) {
            const int d = k % 3;
            const long long j = (long long)(s_keys[min(k / 3, m - 1)] & 0xffffffffull);
            __stcs(out + k, voxel_norm(__ldg(a.xyz + 3 * ((long long)b * a.n + j) + d), cell, d, g));
        }
        __syncthreads();  // s_keys is rewritten by the next cell
    }
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

struct VoxelLayout {
    size_t cursor, member, big, nbig, total;
    long long big_cap;
};

// The cells of a valid shape, else 0.
long long voxel_cells(int b, int n, int dim, int dims) {
    if (b < 1 || n < 1 || dim < 1 || (dims != 2 && dims != 3) || (long long)b * n >= (1ll << 31)) return 0;
    if (dim > (dims == 2 ? 46340 : 1290)) return 0;  // dim^dims < 2^31
    const long long cells = dims == 2 ? (long long)dim * dim : (long long)dim * dim * dim;
    return cells * b < (1ll << 31) ? cells : 0;
}

VoxelLayout voxel_layout(int b, int n, long long cells) {
    VoxelLayout L;
    L.big_cap = (long long)b * std::min<long long>(cells, n / (kWarpCell + 1));  // a cloud has at most n / 129 such cells
    size_t off = 0;
    L.cursor = off; off = align256(off + sizeof(int) * (size_t)b * cells);
    L.member = off; off = align256(off + sizeof(int) * (size_t)b * n);
    L.big = off;    off = align256(off + sizeof(int) * (size_t)L.big_cap);
    L.nbig = off;   off = align256(off + sizeof(int));
    L.total = off;
    return L;
}

AttrOnce g_cta_attr;

}  // namespace
}  // namespace pn2

extern "C" {

size_t pn2_voxel_group_workspace_bytes(int b, int n, int dim, int dims) {
    const long long cells = pn2::voxel_cells(b, n, dim, dims);
    return cells ? pn2::voxel_layout(b, n, cells).total : 0;
}

int pn2_voxel_group(int b, int n, const float* xyz, const int* lengths, int dim, int dims, double radius, int nsample,
                    long long seed, const long long* seed_dev, int* count, int* idx, double* grouped, void* workspace,
                    size_t workspace_bytes, void* stream) {
    using namespace pn2;
    const long long cells = voxel_cells(b, n, dim, dims);
    if (!cells || nsample < 1 || nsample > kSelectMaxRows) return (int)cudaErrorInvalidValue;
    VoxelGrid g;
    g.radius = radius;
    g.voxel = 2.0 * radius / (double)dim;
    g.radius_f = (float)radius;
    g.voxel_f = (float)g.voxel;
    g.dim_f = (float)dim;
    g.dim = dim;
    g.dims = dims;
    g.cells = (int)cells;
    if (!(radius > 0.0) || !(g.radius_f > 0.f) || !(g.voxel_f > 0.f) || !(g.radius_f < INFINITY) || !(g.voxel < INFINITY))
        return (int)cudaErrorInvalidValue;
    if (!xyz || !count || !idx || !grouped || !workspace) return (int)cudaErrorInvalidValue;
    const VoxelLayout L = voxel_layout(b, n, cells);
    if (workspace_bytes < L.total || !aligned_to(workspace, 256)) return (int)cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    int* cursor = reinterpret_cast<int*>(ws + L.cursor);
    int* member = reinterpret_cast<int*>(ws + L.member);
    int* big = reinterpret_cast<int*>(ws + L.big);
    int* nbig = reinterpret_cast<int*>(ws + L.nbig);
    cudaStream_t st = as_stream(stream);
    const size_t sort_bytes = sizeof(unsigned long long) * pow2_at_least(nsample);
    cudaError_t e = ensure_attrs(g_cta_attr, voxel_cta_kernel, sizeof(unsigned long long) * kSelectMaxRows, false);
    if (e != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(count, 0, sizeof(int) * (size_t)b * cells, st)) != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(nbig, 0, sizeof(int), st)) != cudaSuccess) return (int)e;
    const VoxelArgs a{xyz, lengths, seed_dev, (unsigned long long)seed, b, n, nsample};
    const unsigned row_grid = grid_for((unsigned long long)b * n, kRowThreads);
    voxel_count_kernel<<<row_grid, kRowThreads, 0, st>>>(a, g, count);
    int rc = finish_launch();
    if (rc) return rc;
    voxel_scan_kernel<<<b, kCtaThreads, 0, st>>>(g.cells, count, cursor);
    if ((rc = finish_launch())) return rc;
    voxel_fill_kernel<<<row_grid, kRowThreads, 0, st>>>(a, g, cursor, member);
    if ((rc = finish_launch())) return rc;
    const VoxelOut o{count, cursor, member, idx, grouped, big, nbig};
    voxel_warp_kernel<<<grid_for((unsigned long long)b * cells * 32, kWarpThreads), kWarpThreads, 0, st>>>(a, g, o);
    if ((rc = finish_launch())) return rc;
    if (L.big_cap == 0) return 0;  // no cloud has room for a cell of more than kWarpCell rows
    const unsigned cta_grid = (unsigned)std::min<long long>(L.big_cap, 2ll * num_sms());
    voxel_cta_kernel<<<cta_grid, kCtaThreads, sort_bytes, st>>>(a, g, o);
    return finish_launch();
}

}  // extern "C"
