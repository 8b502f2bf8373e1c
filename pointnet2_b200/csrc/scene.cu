// scene.cu — whole-scene segmentation: partition of a scene into xy blocks as a padded ragged batch, and the ordered
// merge of block logits back onto the scene's points (scannet/scannet_dataset.py:83-118 and scannet/train.py:326-427
// without the resampling; DESIGN.md §6.9).
//
// Partition = a stable counting sort of the (block, point) membership pairs by block, in two calls:
//   count: one CTA per tile of consecutive points histograms its context / core memberships per block in shared
//          memory (integer counts: the order of the shared atomics never reaches a result), then one CTA per block
//          scans that block's row of tile counts in tile order (cta_exclusive_sum_1024);
//   fill:  one warp per tile walks its points in ascending order, expands each 32-point group's memberships point by
//          point, ranks equal blocks with __match_any_sync and a per-block cursor in shared memory, and writes each
//          member to its sub-block row.  The same pass writes the point-major CSR of core occurrences.
// A point's memberships are a rectangle of blocks (the block tests are monotone in i and j), so nothing is stored
// per pair: both passes enumerate the rectangle.
#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kSceneMaxBlocks = 16384;    // shared memory: 2 x 64 KB histogram in the count pass
constexpr int kSceneMaxTiles = 2048;      // tiles x blocks histogram: at most 128 MB
constexpr double kCoreMargin = 0.001;     // scannet_dataset.py:103

struct SceneGrid {
    double lo_x, lo_y, size, stride, pad;
    int nx, ny;
};

struct Rect {
    int i0, i1, j0, j1;  // inclusive; empty when i0 > i1 or j0 > j1
};

// First and last block index along one axis whose [lo + i*t - m, lo + i*t + s + m] holds v (double arithmetic on the
// float32 coordinate, each operation rounded, as numpy evaluates coordmin + [i*1.5, ...] - 0.2).  Both tests are
// monotone in i, so the members form one interval; the estimate is corrected by exact tests.
__device__ __forceinline__ void axis_range(double v, double lo, double s, double t, double m, int nb, int& a, int& b) {
    // first i with v <= (lo + i*t + s) + m
    int e = (int)fmin(fmax(floor((v - lo - s - m) / t), 0.0), (double)(nb - 1));
    while (e > 0 && v <= __dadd_rn(__dadd_rn(__dadd_rn(lo, __dmul_rn((double)(e - 1), t)), s), m)) --e;
    while (e < nb && !(v <= __dadd_rn(__dadd_rn(__dadd_rn(lo, __dmul_rn((double)e, t)), s), m))) ++e;
    a = e;
    // last i with (lo + i*t) - m <= v
    e = (int)fmin(fmax(floor((v - lo + m) / t), 0.0), (double)(nb - 1));
    while (e < nb - 1 && __dsub_rn(__dadd_rn(lo, __dmul_rn((double)(e + 1), t)), m) <= v) ++e;
    while (e >= 0 && !(__dsub_rn(__dadd_rn(lo, __dmul_rn((double)e, t)), m) <= v)) --e;
    b = e;
}

// Context rectangle (padding g) and core rectangle (margin 0.001, within the context rectangle) of a point.
__device__ __forceinline__ void point_rects(float x, float y, const SceneGrid& g, Rect& ctx, Rect& core) {
    axis_range((double)x, g.lo_x, g.size, g.stride, g.pad, g.nx, ctx.i0, ctx.i1);
    axis_range((double)y, g.lo_y, g.size, g.stride, g.pad, g.ny, ctx.j0, ctx.j1);
    axis_range((double)x, g.lo_x, g.size, g.stride, kCoreMargin, g.nx, core.i0, core.i1);
    axis_range((double)y, g.lo_y, g.size, g.stride, kCoreMargin, g.ny, core.j0, core.j1);
    core.i0 = max(core.i0, ctx.i0);
    core.i1 = min(core.i1, ctx.i1);
    core.j0 = max(core.j0, ctx.j0);
    core.j1 = min(core.j1, ctx.j1);
}

__device__ __forceinline__ int rect_area(const Rect& r) {
    return (r.i1 >= r.i0 && r.j1 >= r.j0) ? (r.i1 - r.i0 + 1) * (r.j1 - r.j0 + 1) : 0;
}

// Points per tile: tiles of at least 256 points, at most kSceneMaxTiles tiles, a multiple of 32.
inline int scene_tile(int p) {
    const long long t = ((long long)p + kSceneMaxTiles - 1) / kSceneMaxTiles;
    return (int)(t <= 256 ? 256 : (t + 31) / 32 * 32);
}
inline int scene_tiles(int p) { return (int)(((long long)p + scene_tile(p) - 1) / scene_tile(p)); }

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

struct SceneLayout {
    size_t hist, tile_core, tile_core_off, total;
};
SceneLayout scene_layout(int p, int nblk) {
    const size_t tiles = (size_t)scene_tiles(p);
    SceneLayout L;
    size_t off = 0;
    L.hist = off;          off = align256(off + sizeof(int) * tiles * (size_t)nblk);
    L.tile_core = off;     off = align256(off + sizeof(int) * tiles);
    L.tile_core_off = off; off = align256(off + sizeof(int) * tiles);
    L.total = off;
    return L;
}

// hist[blk * tiles + tile] = context members of block blk among the tile's points; counts[nblk + blk] += its core
// members; tile_core[tile] = core occurrences of the tile's points.
__global__ void __launch_bounds__(256) scene_count_kernel(SceneGrid g, int p, int tile_pts, int tiles, const float* __restrict__ xyz,
                                                          int* __restrict__ hist, int* __restrict__ counts, int* __restrict__ tile_core) {
    extern __shared__ int s_hist[];  // [0, nblk): context, [nblk, 2 nblk): core
    __shared__ int s_occ;
    const int nblk = g.nx * g.ny;
    for (int k = threadIdx.x; k < 2 * nblk; k += blockDim.x) s_hist[k] = 0;
    if (threadIdx.x == 0) s_occ = 0;
    __syncthreads();
    const int tile = blockIdx.x;
    const int p0 = tile * tile_pts, p1 = min(p, p0 + tile_pts);
    int occ = 0;
    for (int q = p0 + threadIdx.x; q < p1; q += blockDim.x) {
        Rect ctx, core;
        point_rects(__ldg(xyz + 3 * (size_t)q), __ldg(xyz + 3 * (size_t)q + 1), g, ctx, core);
        for (int i = ctx.i0; i <= ctx.i1; ++i)
            for (int j = ctx.j0; j <= ctx.j1; ++j) atomicAdd(&s_hist[i * g.ny + j], 1);
        for (int i = core.i0; i <= core.i1; ++i)
            for (int j = core.j0; j <= core.j1; ++j) atomicAdd(&s_hist[nblk + i * g.ny + j], 1);
        occ += rect_area(core);
    }
    occ = __reduce_add_sync(kFullMask, occ);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s_occ, occ);
    __syncthreads();
    for (int k = threadIdx.x; k < nblk; k += blockDim.x) {
        hist[(size_t)k * tiles + tile] = s_hist[k];
        const int c = s_hist[nblk + k];
        if (c) atomicAdd(&counts[nblk + k], c);
    }
    if (threadIdx.x == 0) tile_core[tile] = s_occ;
}

// CTA blk < nblk: exclusive scan of block blk's tile counts in tile order (in place), counts[blk] = its members.
// CTA nblk: exclusive scan of the tiles' core occurrences.
__global__ void __launch_bounds__(1024) scene_scan_kernel(int nblk, int tiles, int* __restrict__ hist, int* __restrict__ counts,
                                                          const int* __restrict__ tile_core, int* __restrict__ tile_core_off) {
    __shared__ int s_w[32];
    __shared__ int s_carry;
    const int blk = blockIdx.x;
    const int* src = blk < nblk ? hist + (size_t)blk * tiles : tile_core;
    int* dst = blk < nblk ? hist + (size_t)blk * tiles : tile_core_off;
    const int total = cta_exclusive_scan_1024(src, dst, tiles, s_w, &s_carry);
    if (blk < nblk && threadIdx.x == 0) counts[blk] = total;
}

// One warp per tile.  Its points are taken 32 at a time in ascending order; the group's (point, block) pairs are
// enumerated point-major (for each point its rectangle i-major, then j), 32 pairs per round, so pairs of one block
// reach the cursor in ascending point order.  Member r of a block with k sub-blocks goes to sub-block r mod k, row
// r div k.
__global__ void __launch_bounds__(32) scene_fill_kernel(SceneGrid g, int p, int tile_pts, int tiles, const float* __restrict__ xyz,
                                                        const int* __restrict__ hist, const int* __restrict__ tile_core_off,
                                                        const int* __restrict__ sub_begin, const int* __restrict__ sub_count, int n,
                                                        float* __restrict__ out_xyz, int* __restrict__ out_idx,
                                                        unsigned char* __restrict__ out_core, int* __restrict__ occ_off,
                                                        int* __restrict__ occ_row) {
    extern __shared__ int s_cur[];  // nblk per-block cursors: the next member rank of each block
    __shared__ int s_excl[32], s_occ[32];
    __shared__ Rect s_ctx[32], s_core[32];
    __shared__ float s_pt[32][3];
    const int nblk = g.nx * g.ny;
    const int lane = threadIdx.x, tile = blockIdx.x;
    for (int k = lane; k < nblk; k += 32) s_cur[k] = hist[(size_t)k * tiles + tile];
    int occ_carry = tile_core_off[tile];
    const int p0 = tile * tile_pts, p1 = min(p, p0 + tile_pts);
    const unsigned lt = (1u << lane) - 1u;
    for (int base = p0; base < p1; base += 32) {
        const int q = base + lane;
        Rect ctx = {0, -1, 0, -1}, core = {0, -1, 0, -1};
        float x = 0.f, y = 0.f, z = 0.f;
        if (q < p1) {
            x = __ldg(xyz + 3 * (size_t)q);
            y = __ldg(xyz + 3 * (size_t)q + 1);
            z = __ldg(xyz + 3 * (size_t)q + 2);
            point_rects(x, y, g, ctx, core);
        }
        const int nctx = rect_area(ctx), ncore = rect_area(core);
        int ic = nctx, io = ncore;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int a = __shfl_up_sync(kFullMask, ic, o), b = __shfl_up_sync(kFullMask, io, o);
            if (lane >= o) {
                ic += a;
                io += b;
            }
        }
        const int total = __shfl_sync(kFullMask, ic, 31), total_core = __shfl_sync(kFullMask, io, 31);
        if (q < p1) occ_off[q] = occ_carry + io - ncore;
        __syncwarp();  // the previous group's readers are done with the shared arrays
        s_excl[lane] = ic - nctx;
        s_occ[lane] = occ_carry + io - ncore;
        s_ctx[lane] = ctx;
        s_core[lane] = core;
        s_pt[lane][0] = x;
        s_pt[lane][1] = y;
        s_pt[lane][2] = z;
        __syncwarp();
        for (int u0 = 0; u0 < total; u0 += 32) {
            const int u = u0 + lane;
            const bool act = u < total;
            int blk = -1, owner = 0, i = 0, j = 0;
            if (act) {
                // owner: the last lane whose exclusive pair offset is <= u (lanes without pairs share the offset of the
                // next lane, so the last of a run of equal offsets is the one that has pairs)
#pragma unroll
                for (int step = 16; step > 0; step >>= 1)
                    if (s_excl[owner + step] <= u) owner += step;
                const Rect r = s_ctx[owner];
                const int w = r.j1 - r.j0 + 1, local = u - s_excl[owner];
                i = r.i0 + local / w;
                j = r.j0 + local % w;
                blk = i * g.ny + j;
            }
            const unsigned peers = __match_any_sync(kFullMask, blk);
            const int rank = __popc(peers & lt);
            const int r0 = act ? s_cur[blk] : 0;
            __syncwarp();
            if (act && rank == 0) s_cur[blk] = r0 + __popc(peers);
            __syncwarp();
            if (!act) continue;
            const int k = __ldg(sub_count + blk);
            if (k <= 0) continue;  // a block without core points is dropped
            const int r = r0 + rank;
            const long long flat = (long long)(__ldg(sub_begin + blk) + r % k) * n + r / k;
            const Rect c = s_core[owner];
            const bool is_core = i >= c.i0 && i <= c.i1 && j >= c.j0 && j <= c.j1;
            out_xyz[3 * flat] = s_pt[owner][0];
            out_xyz[3 * flat + 1] = s_pt[owner][1];
            out_xyz[3 * flat + 2] = s_pt[owner][2];
            out_idx[flat] = base + owner;
            out_core[flat] = is_core ? 1 : 0;
            if (is_core) occ_row[s_occ[owner] + (i - c.i0) * (c.j1 - c.j0 + 1) + (j - c.j0)] = (int)flat;
        }
        occ_carry += total_core;
    }
    if (tile == tiles - 1 && lane == 0) occ_off[p] = occ_carry;
}

// One warp per logits row: the row that holds a point's first core occurrence inside [row_begin, row_end) adds all of
// that point's occurrences there, in ascending row order, onto accum (lanes over classes); other rows do nothing.
template <typename T>
__global__ void __launch_bounds__(256) scene_merge_kernel(int c, int row_begin, int row_end, const T* __restrict__ logits,
                                                          const int* __restrict__ point_idx, const unsigned char* __restrict__ core,
                                                          const int* __restrict__ occ_off, const int* __restrict__ occ_row,
                                                          float* __restrict__ accum) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long row = row_begin + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < row_end; row += warps) {
        if (!__ldg(core + row)) continue;
        const int pt = __ldg(point_idx + row);
        int o = __ldg(occ_off + pt);
        const int o1 = __ldg(occ_off + pt + 1);
        while (o < o1 && __ldg(occ_row + o) < row_begin) ++o;
        if (o >= o1 || __ldg(occ_row + o) != row) continue;  // not the point's first occurrence in this range
        float* dst = accum + (size_t)pt * c;
        for (int k = lane; k < c; k += 32) {
            float a = dst[k];
            for (int e = o; e < o1; ++e) {
                const int rr = __ldg(occ_row + e);
                if (rr >= row_end) break;
                a = __fadd_rn(a, to_f32(__ldg(logits + (size_t)(rr - row_begin) * c + k)));
            }
            dst[k] = a;
        }
    }
}

AttrOnce g_count_attr, g_fill_attr;

bool grid_ok(int p, double size, double stride, double pad, int nx, int ny) {
    return p > 0 && nx > 0 && ny > 0 && (long long)nx * ny <= kSceneMaxBlocks && size > 0.0 && stride > 0.0 &&
           stride <= size && pad >= 0.0 && size < 1e30 && pad < 1e30;
}

template <typename T>
int launch_merge(int c, int row_begin, int row_end, const void* logits, const int* point_idx, const unsigned char* core,
                 const int* occ_off, const int* occ_row, float* accum, cudaStream_t st) {
    scene_merge_kernel<T><<<grid_for((unsigned long long)(row_end - row_begin) * 32, 256), 256, 0, st>>>(
        c, row_begin, row_end, static_cast<const T*>(logits), point_idx, core, occ_off, occ_row, accum);
    return finish_launch();
}

}  // namespace
}  // namespace pn2

extern "C" {

size_t pn2_scene_blocks_workspace_bytes(int p, int nx, int ny) {
    if (p <= 0 || nx <= 0 || ny <= 0 || (long long)nx * ny > pn2::kSceneMaxBlocks) return 0;
    return pn2::scene_layout(p, nx * ny).total;
}

int pn2_scene_blocks_count(int p, const float* xyz, double lo_x, double lo_y, double block_size, double stride, double padding,
                           int nx, int ny, int* counts, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!grid_ok(p, block_size, stride, padding, nx, ny) || !xyz || !counts || !workspace) return (int)cudaErrorInvalidValue;
    const int nblk = nx * ny;
    const SceneLayout L = scene_layout(p, nblk);
    if (workspace_bytes < L.total || !aligned_to(workspace, 256)) return (int)cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    int* hist = reinterpret_cast<int*>(ws + L.hist);
    int* tile_core = reinterpret_cast<int*>(ws + L.tile_core);
    int* tile_core_off = reinterpret_cast<int*>(ws + L.tile_core_off);
    const SceneGrid g{lo_x, lo_y, block_size, stride, padding, nx, ny};
    const int tile_pts = scene_tile(p), tiles = scene_tiles(p);
    cudaStream_t st = as_stream(stream);
    cudaError_t e = ensure_attrs(g_count_attr, scene_count_kernel, 2 * sizeof(int) * kSceneMaxBlocks, false);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemsetAsync(counts + nblk, 0, sizeof(int) * nblk, st);
    if (e != cudaSuccess) return (int)e;
    scene_count_kernel<<<tiles, 256, 2 * sizeof(int) * nblk, st>>>(g, p, tile_pts, tiles, xyz, hist, counts, tile_core);
    int rc = finish_launch();
    if (rc) return rc;
    scene_scan_kernel<<<nblk + 1, 1024, 0, st>>>(nblk, tiles, hist, counts, tile_core, tile_core_off);
    return finish_launch();
}

int pn2_scene_blocks_fill(int p, const float* xyz, double lo_x, double lo_y, double block_size, double stride, double padding,
                          int nx, int ny, const int* sub_begin, const int* sub_count, int b, int n, float* out_xyz,
                          int* point_idx, unsigned char* core, int* occ_off, int* occ_row, void* workspace,
                          size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!grid_ok(p, block_size, stride, padding, nx, ny) || b <= 0 || n <= 0 || (long long)b * n * 3 >= (1ll << 31))
        return (int)cudaErrorInvalidValue;
    if (!xyz || !sub_begin || !sub_count || !out_xyz || !point_idx || !core || !occ_off || !occ_row || !workspace)
        return (int)cudaErrorInvalidValue;
    const int nblk = nx * ny;
    const SceneLayout L = scene_layout(p, nblk);
    if (workspace_bytes < L.total || !aligned_to(workspace, 256)) return (int)cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    const int* hist = reinterpret_cast<const int*>(ws + L.hist);
    const int* tile_core_off = reinterpret_cast<const int*>(ws + L.tile_core_off);
    const SceneGrid g{lo_x, lo_y, block_size, stride, padding, nx, ny};
    const int tile_pts = scene_tile(p), tiles = scene_tiles(p);
    cudaStream_t st = as_stream(stream);
    cudaError_t e = ensure_attrs(g_fill_attr, scene_fill_kernel, sizeof(int) * kSceneMaxBlocks, false);
    if (e != cudaSuccess) return (int)e;
    const size_t rows = (size_t)b * n;
    // padding rows: xyz 0, point index -1, not core
    if ((e = cudaMemsetAsync(out_xyz, 0, sizeof(float) * 3 * rows, st)) != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(point_idx, 0xff, sizeof(int) * rows, st)) != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(core, 0, rows, st)) != cudaSuccess) return (int)e;
    scene_fill_kernel<<<tiles, 32, sizeof(int) * nblk, st>>>(g, p, tile_pts, tiles, xyz, hist, tile_core_off, sub_begin, sub_count,
                                                             n, out_xyz, point_idx, core, occ_off, occ_row);
    return finish_launch();
}

int pn2_scene_merge_typed(int dtype, int p, int c, int b, int n, int row_begin, int row_end, const void* logits,
                          const int* point_idx, const unsigned char* core, const int* occ_off, const int* occ_row,
                          float* accum, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype) || p <= 0 || c <= 0 || b <= 0 || n <= 0 || (long long)b * n >= (1ll << 31)) return (int)cudaErrorInvalidValue;
    if (row_begin < 0 || row_end < row_begin || (long long)row_end > (long long)b * n) return (int)cudaErrorInvalidValue;
    if (!logits || !point_idx || !core || !occ_off || !occ_row || !accum) return (int)cudaErrorInvalidValue;
    if (row_end == row_begin) return 0;
    cudaStream_t st = as_stream(stream);
    switch (dtype) {
        case PN2_BF16: return launch_merge<__nv_bfloat16>(c, row_begin, row_end, logits, point_idx, core, occ_off, occ_row, accum, st);
        case PN2_F16: return launch_merge<__half>(c, row_begin, row_end, logits, point_idx, core, occ_off, occ_row, accum, st);
        default: return launch_merge<float>(c, row_begin, row_end, logits, point_idx, core, occ_off, occ_row, accum, st);
    }
}

}  // extern "C"
