// vscan.cu — virtual scans of ScanNet-style scenes: the points a depth camera at one viewpoint would see, as a padded
// ragged batch (scannet/scene_util.py virtual_scan, scannet/scannet_dataset.py:122-166, without the resampling;
// DESIGN.md §6.12).
//
// Five launches and one memset per call, nothing read back:
//   ray:    grid (ray chunks, B): the entry's 200 x 150 rays as (azimuth, elevation), counted into a uniform cell grid
//           over (az, el) with integer atomicAdd; the entry's z-buffer set to +inf (all bits set);
//   cell:   one CTA per entry scans the cell counts and scatters every ray into its cell, so that cell_end[c] becomes
//           the end of cell c in the cell-sorted ray table;
//   point:  grid (point chunks, B), twice.  A point's nearest ray lies in the 3 x 3 cells around the point's own cell
//           whenever it is nearer than 0.01 (the cell side is 0.0101).  Pass 0: every near point lowers its ray's
//           z-buffer entry with atomicMin on the bits of its range r (r >= 0, so the bit order is the numeric order),
//           sets its bit of the entry's bitmap and counts as near.  Pass 1: a near point keeps its bit when r equals
//           its ray's minimum, and counts as visible;
//   select: one CTA per entry takes the m = min(visible, npoints) smallest (key, scene index) pairs of the visible
//           points in order (cta_select_sorted) and writes the rows.
// Every atomic is an integer one, so the results do not depend on the order of the threads.  The arithmetic is double,
// each +, -, x, /, sqrt rounded on its own; sin / cos are sincospi of the half-turn count (no large-argument
// reduction) and atan2 is CUDA's, so decisions equal the float64 definition wherever their margin exceeds ~1e-12.
#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kRaysX = 200, kRaysY = 150, kRays = kRaysX * kRaysY;  // scene_util.py:34-35
constexpr double kNear = 0.01;                                     // scene_util.py:48
constexpr int kMinNear = 100;                                      // scene_util.py:49
// The (az, el) cell grid: side 0.0101, so that a ray within 0.01 of a point is at most one cell away on each axis with
// a 1 % margin for the rounding of the cell function.  It spans az in [-3.2, 3.2034) (atan2's range is [-pi, pi]) and
// el in [-0.8, 0.8059): every ray's |el| is at most |theta| + atan(0.45) < 0.66.
constexpr double kCellH = 0.0101, kAz0 = -3.2, kEl0 = -0.8;
constexpr int kCellsAz = 634, kCellsEl = 159, kCells = kCellsAz * kCellsEl;
constexpr int kScanMaxBatch = 4096;    // entries per call: the workspace is ~1.7 MB per entry
constexpr int kRayThreads = 256;
constexpr int kPointThreads = 256;
constexpr int kPointChunk = 4096;      // scene points per CTA of a point pass (a multiple of 32: warps own bitmap words)
constexpr int kCellThreads = 1024;
constexpr int kSelectThreads = 1024;
// random streams of DESIGN.md §6.12
constexpr unsigned long long kStreamAzimuth = 1, kStreamTilt = 2, kStreamDistance = 3, kStreamKey = 4;

struct ScanArgs {
    const float* xyz;
    const int* label;
    const long long* offsets;
    const double* mean;          // (s, 3): each scene's float64 mean
    const long long* scan_scene;
    const long long* scan_mode;  // -1: a random view; m: the fixed view at azimuth pi/4 m
    const long long* seed_dev;   // non-null: the seed is read here, on the device
    unsigned long long seed;
    int s;
};

// Per-entry workspace arrays (entry b's part of each starts at b times its per-entry size).  cnt, cell_end and bits are
// zeroed by the call's one memset; the others are written before they are read.
struct ScanWs {
    int* cnt;                   // (b, 4): near, visible
    int* cell_end;              // (b, kCells): ray counts, then cell ends
    unsigned* bits;             // (b, words): near, then visible points by scene-local index
    double* ray_az;             // (b, kRays), ray order
    double* ray_el;
    double* srt_az;             // (b, kRays), cell order
    double* srt_el;
    int* srt_k;
    unsigned long long* zbuf;   // (b, kRays): bits of each ray's minimum r
    long long words;
};

size_t align256(size_t x) { return (x + 255) / 256 * 256; }

size_t scan_zero_bytes(int b, int max_scene) {
    const long long words = ((long long)max_scene + 31) / 32;
    return align256(sizeof(int) * ((size_t)b * 4 + (size_t)b * kCells + (size_t)b * words));
}

size_t scan_ws_bytes(int b, int max_scene) {
    return scan_zero_bytes(b, max_scene) + 4 * align256(sizeof(double) * (size_t)b * kRays) +
           align256(sizeof(int) * (size_t)b * kRays) + align256(sizeof(unsigned long long) * (size_t)b * kRays);
}

ScanWs scan_ws(void* base, int b, int max_scene) {
    char* p = static_cast<char*>(base);
    ScanWs w;
    w.words = ((long long)max_scene + 31) / 32;
    w.cnt = reinterpret_cast<int*>(p);
    w.cell_end = w.cnt + (size_t)b * 4;
    w.bits = reinterpret_cast<unsigned*>(w.cell_end + (size_t)b * kCells);
    p += scan_zero_bytes(b, max_scene);
    double** d[4] = {&w.ray_az, &w.ray_el, &w.srt_az, &w.srt_el};
    for (double** q : d) {
        *q = reinterpret_cast<double*>(p);
        p += align256(sizeof(double) * (size_t)b * kRays);
    }
    w.srt_k = reinterpret_cast<int*>(p);
    p += align256(sizeof(int) * (size_t)b * kRays);
    w.zbuf = reinterpret_cast<unsigned long long*>(p);
    return w;
}

struct ScanView {
    double ct[3], hr[3], vt[3];  // view direction and the image plane's unit axes
    double cam[3];               // camera location
};

// np.cross(a, b) as numpy evaluates it: a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0
__device__ __forceinline__ void cross3(const double (&u)[3], const double (&v)[3], double (&c)[3]) {
    c[0] = __dsub_rn(__dmul_rn(u[1], v[2]), __dmul_rn(u[2], v[1]));
    c[1] = __dsub_rn(__dmul_rn(u[2], v[0]), __dmul_rn(u[0], v[2]));
    c[2] = __dsub_rn(__dmul_rn(u[0], v[1]), __dmul_rn(u[1], v[0]));
}

__device__ __forceinline__ void normalise3(double (&v)[3]) {
    const double n = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2])));
    for (int d = 0; d < 3; ++d) v[d] = __ddiv_rn(v[d], n);
}

// scene_util.py:21-33.  Random view: phi = 2 pi u1, theta = pi/10 (u2 - 0.75), the camera (0.8 + 0.7 u3) behind the
// centre; fixed view m: phi = pi/4 m, theta = 0, the camera 1 behind.  sin / cos as sincospi of phi / pi and theta / pi.
__device__ void scan_view(const ScanArgs& a, int b, int sc, ScanView& v) {
    const unsigned long long seed = rng_seed(a.seed_dev, a.seed), e = (unsigned long long)b;
    const long long mode = __ldg(a.scan_mode + b);
    double sp, cp, st = 0.0, cth = 1.0, dist = 1.0;
    if (mode == -1) {
        const double u1 = rng_unit(rng_draw(seed, kStreamAzimuth, e, 0)), u2 = rng_unit(rng_draw(seed, kStreamTilt, e, 0)),
                     u3 = rng_unit(rng_draw(seed, kStreamDistance, e, 0));
        sincospi(__dmul_rn(u1, 2.0), &sp, &cp);
        sincospi(__ddiv_rn(__dsub_rn(u2, 0.75), 10.0), &st, &cth);
        dist = __dadd_rn(0.8, __dmul_rn(0.7, u3));
    } else {
        sincospi(__dmul_rn((double)mode, 0.25), &sp, &cp);
    }
    v.ct[0] = __dmul_rn(cth, cp);
    v.ct[1] = __dmul_rn(cth, sp);
    v.ct[2] = st;
    const double z[3] = {0.0, 0.0, 1.0};
    cross3(v.ct, z, v.hr);
    normalise3(v.hr);
    cross3(v.hr, v.ct, v.vt);
    normalise3(v.vt);
    v.cam[0] = __dsub_rn(__ldg(a.mean + 3 * sc), __dmul_rn(dist, cp));
    v.cam[1] = __dsub_rn(__ldg(a.mean + 3 * sc + 1), __dmul_rn(dist, sp));
    v.cam[2] = 1.5;
}

// cart2sph's (azimuth, elevation) of (x, y, z), and r = sqrt((x^2 + y^2) + z^2)
__device__ __forceinline__ void sph(double x, double y, double z, double& az, double& el, double& r) {
    const double xy = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
    r = __dsqrt_rn(__dadd_rn(xy, __dmul_rn(z, z)));
    el = atan2(z, __dsqrt_rn(xy));
    az = atan2(y, x);
}

// element i of np.linspace(lo, -lo, n): i * ((-lo - lo) / (n - 1)) + lo, the last one -lo exactly
__device__ __forceinline__ double linspace_at(double lo, int n, int i) {
    if (i == n - 1) return -lo;
    return __dadd_rn(__dmul_rn((double)i, __ddiv_rn(__dsub_rn(-lo, lo), (double)(n - 1))), lo);
}

// cell coordinate of an angle, clamped to [-2, n + 1]: -2 and n + 1 have no cell within reach
__device__ __forceinline__ int cell_coord(double x, double x0, int n) {
    const double f = floor(__ddiv_rn(__dsub_rn(x, x0), kCellH));
    return (int)fmin(fmax(f, -2.0), (double)(n + 1));
}

__device__ __forceinline__ int ray_cell(double az, double el) {
    const int ca = min(max(cell_coord(az, kAz0, kCellsAz), 0), kCellsAz - 1);
    const int ce = min(max(cell_coord(el, kEl0, kCellsEl), 0), kCellsEl - 1);
    return ce * kCellsAz + ca;
}

// grid (ray chunks, B)
__global__ void __launch_bounds__(kRayThreads) vscan_ray_kernel(ScanArgs a, ScanWs w) {
    __shared__ ScanView s_v;
    const int b = blockIdx.y;
    int sc;
    long long off, ps;
    if (!set_entry(a.scan_scene, b, a.s, a.offsets, sc, off, ps)) return;
    if (threadIdx.x == 0) scan_view(a, b, sc, s_v);
    __syncthreads();
    const int k = blockIdx.x * kRayThreads + threadIdx.x;
    if (k >= kRays) return;
    // ray k = xx_i hr + yy_j vt + ct, k = j * 200 + i (meshgrid, then reshape)
    const double xx = linspace_at(-0.6, kRaysX, k % kRaysX), yy = linspace_at(-0.45, kRaysY, k / kRaysX);
    double r[3];
    for (int d = 0; d < 3; ++d) r[d] = __dadd_rn(__dadd_rn(__dmul_rn(xx, s_v.hr[d]), __dmul_rn(yy, s_v.vt[d])), s_v.ct[d]);
    double az, el, rr;
    sph(r[0], r[1], r[2], az, el, rr);
    const size_t e = (size_t)b * kRays + k;
    w.ray_az[e] = az;
    w.ray_el[e] = el;
    w.zbuf[e] = ~0ull;
    atomicAdd(w.cell_end + (size_t)b * kCells + ray_cell(az, el), 1);
}

// one CTA per entry: cell counts -> starts (exclusive scan), then the scatter turns them into ends
__global__ void __launch_bounds__(kCellThreads) vscan_cell_kernel(ScanArgs a, ScanWs w) {
    __shared__ int s_w[32];
    const int b = blockIdx.x;
    int sc;
    long long off, ps;
    if (!set_entry(a.scan_scene, b, a.s, a.offsets, sc, off, ps)) return;
    int* ce = w.cell_end + (size_t)b * kCells;
    constexpr int kPer = (kCells + kCellThreads - 1) / kCellThreads;
    const int c0 = min((int)threadIdx.x * kPer, kCells), c1 = min(c0 + kPer, kCells);
    int sum = 0;
    for (int c = c0; c < c1; ++c) sum += ce[c];
    int run = cta_exclusive_sum_1024(sum, s_w);
    for (int c = c0; c < c1; ++c) {
        const int v = ce[c];
        ce[c] = run;
        run += v;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < kRays; k += kCellThreads) {
        const size_t e = (size_t)b * kRays + k;
        const double az = w.ray_az[e], el = w.ray_el[e];
        const size_t q = (size_t)b * kRays + atomicAdd(ce + ray_cell(az, el), 1);
        w.srt_az[q] = az;
        w.srt_el[q] = el;
        w.srt_k[q] = k;
    }
}

// The nearest ray to (az, el) by sqrt(daz^2 + del^2), the lower ray index on ties, searched in the 3 x 3 cells around
// the point's cell (each row of three cells is one contiguous range of the cell-sorted table).  Exact whenever the
// nearest ray is nearer than 0.01; returns whether it is.
__device__ __forceinline__ bool nearest_ray(const ScanWs& w, int b, double az, double el, int& best_k) {
    const int ca = cell_coord(az, kAz0, kCellsAz), ce = cell_coord(el, kEl0, kCellsEl);
    const int a0 = max(ca - 1, 0), a1 = min(ca + 1, kCellsAz - 1);
    const int* cend = w.cell_end + (size_t)b * kCells;
    const size_t rb = (size_t)b * kRays;
    double best = INFINITY;
    int bk = 0x7fffffff;
    if (a0 <= a1) {
        for (int e = max(ce - 1, 0); e <= min(ce + 1, kCellsEl - 1); ++e) {
            const int c0 = e * kCellsAz + a0, c1 = e * kCellsAz + a1;
            const int q1 = __ldg(cend + c1);
            for (int q = c0 ? __ldg(cend + c0 - 1) : 0; q < q1; ++q) {
                const double da = __dsub_rn(az, __ldg(w.srt_az + rb + q)), de = __dsub_rn(el, __ldg(w.srt_el + rb + q));
                const double d = __dsqrt_rn(__dadd_rn(__dmul_rn(da, da), __dmul_rn(de, de)));
                const int k = __ldg(w.srt_k + rb + q);
                if (d < best || (d == best && k < bk)) {
                    best = d;
                    bk = k;
                }
            }
        }
    }
    best_k = bk;
    return best < kNear;
}

// grid (point chunks, B); pass 0: near points and the z-buffer, pass 1: visible points (after pass 0 completed)
__global__ void __launch_bounds__(kPointThreads) vscan_point_kernel(ScanArgs a, ScanWs w, int pass) {
    __shared__ ScanView s_v;
    const int b = blockIdx.y;
    int sc;
    long long off, ps;
    if (!set_entry(a.scan_scene, b, a.s, a.offsets, sc, off, ps)) return;
    const long long q0 = (long long)blockIdx.x * kPointChunk;
    if (q0 >= ps) return;
    if (pass && __ldg(w.cnt + 4 * b) < kMinNear) return;  // fewer than 100 near points: no scan
    const long long q1 = min(ps, q0 + kPointChunk);
    if (threadIdx.x == 0) scan_view(a, b, sc, s_v);
    __syncthreads();
    const double cam[3] = {s_v.cam[0], s_v.cam[1], s_v.cam[2]};
    const int lane = threadIdx.x & 31;
    unsigned* bits = w.bits + (size_t)b * w.words;
    unsigned long long* zbuf = w.zbuf + (size_t)b * kRays;
    int cnt = 0;
    for (long long base = q0 + (threadIdx.x & ~31); base < q1; base += kPointThreads) {
        const long long j = base + lane;
        const unsigned in = pass ? bits[base >> 5] : kFullMask;
        if (!in) continue;  // warp-uniform: no near point among these 32
        bool hit = false;
        if (j < q1 && ((in >> lane) & 1u)) {
            const long long g = off + j;
            double az, el, r;
            sph(__dsub_rn((double)__ldg(a.xyz + 3 * g), cam[0]), __dsub_rn((double)__ldg(a.xyz + 3 * g + 1), cam[1]),
                __dsub_rn((double)__ldg(a.xyz + 3 * g + 2), cam[2]), az, el, r);
            int k;
            if (nearest_ray(w, b, az, el, k)) {
                const unsigned long long rb = (unsigned long long)__double_as_longlong(r);
                if (pass) {
                    hit = rb == zbuf[k];
                } else {
                    atomicMin(zbuf + k, rb);
                    hit = true;
                }
            }
        }
        const unsigned word = __ballot_sync(kFullMask, hit);
        if (lane == 0) {
            if (word != (pass ? in : 0u)) bits[base >> 5] = word;  // the warp owns this word
            cnt += __popc(word);
        }
    }
    if (lane == 0 && cnt) atomicAdd(w.cnt + 4 * b + pass, cnt);
}

struct ScanOut {
    float* xyz;
    long long* label;
    float* weight;
    int* lengths;
    int* point_idx;
    int* visible;
    unsigned char* valid;
};

// One CTA per entry.  Dynamic shared memory: the sort buffer, pow2 >= npoints 64-bit values.
__global__ void __launch_bounds__(kSelectThreads) vscan_select_kernel(ScanArgs a, ScanWs w, int num_class,
                                                                      const float* __restrict__ label_weights, int npoints,
                                                                      int min_points, ScanOut o) {
    extern __shared__ unsigned long long s_keys[];
    __shared__ SelectScratch s_sel;
    const int b = blockIdx.x, tid = threadIdx.x;
    const size_t row0 = (size_t)b * npoints;
    int sc;
    long long off = 0, ps = 0;
    const bool in_range = set_entry(a.scan_scene, b, a.s, a.offsets, sc, off, ps);
    int vis = -1, m = 0;
    bool valid = false;
    if (in_range) {  // a scene index outside [0, S): an empty entry, visible -1
        const int near = __ldg(w.cnt + 4 * b);
        vis = near < kMinNear ? 0 : __ldg(w.cnt + 4 * b + 1);
        m = min(vis, npoints);
        valid = vis >= min_points;
        const unsigned long long seed = rng_seed(a.seed_dev, a.seed);
        const unsigned* bits = w.bits + (size_t)b * w.words;
        cta_select_sorted(
            vis > 0 ? ps : 0, vis, m, [&](long long j) { return ((__ldg(bits + (j >> 5)) >> (j & 31)) & 1u) != 0u; },
            [&](long long j) { return rng_row_key(seed, kStreamKey, (unsigned long long)b, j); }, s_keys, s_sel);
    }
    for (int r = tid; r < npoints; r += blockDim.x) {
        const size_t row = row0 + r;
        if (r < m) {
            const long long g = off + (long long)(s_keys[r] & 0xffffffffull);
            const int l = __ldg(a.label + g);
            o.xyz[3 * row] = __ldg(a.xyz + 3 * g);
            o.xyz[3 * row + 1] = __ldg(a.xyz + 3 * g + 1);
            o.xyz[3 * row + 2] = __ldg(a.xyz + 3 * g + 2);
            o.label[row] = l;
            o.weight[row] = (valid && l >= 0 && l < num_class) ? __ldg(label_weights + l) : 0.f;
            o.point_idx[row] = (int)g;
        } else {
            o.xyz[3 * row] = o.xyz[3 * row + 1] = o.xyz[3 * row + 2] = 0.f;
            o.label[row] = 0;
            o.weight[row] = 0.f;
            o.point_idx[row] = -1;
        }
    }
    if (tid == 0) {
        o.lengths[b] = m;
        o.visible[b] = vis;
        o.valid[b] = valid ? 1 : 0;
    }
}

bool scan_shape_ok(int b, int max_scene, int npoints) {
    return b >= 1 && b <= kScanMaxBatch && max_scene >= 1 && max_scene < 0x7fffffff && npoints >= 1 &&
           npoints <= kSelectMaxRows && (long long)b * npoints * 3 < (1ll << 31);
}

AttrOnce g_scan_select_attr;

}  // namespace
}  // namespace pn2

extern "C" {

size_t pn2_virtual_scans_workspace_bytes(int b, int max_scene, int npoints) {
    if (!pn2::scan_shape_ok(b, max_scene, npoints)) return 0;
    return pn2::scan_ws_bytes(b, max_scene);
}

int pn2_virtual_scans(int s, int p, int max_scene, const float* xyz, const int* label, const long long* offsets,
                      const double* mean, int num_class, const float* label_weights, int b, const long long* scan_scene,
                      const long long* scan_mode, long long seed, const long long* seed_dev, int npoints, int min_points,
                      float* out_xyz, long long* out_label, float* out_weight, int* lengths, int* point_idx, int* visible,
                      unsigned char* valid, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (s < 1 || p < 1 || p >= 0x7fffffff || max_scene > p || num_class < 1 || min_points < 0 ||
        !scan_shape_ok(b, max_scene, npoints))
        return (int)cudaErrorInvalidValue;
    if (!xyz || !label || !offsets || !mean || !label_weights || !scan_scene || !scan_mode || !out_xyz || !out_label ||
        !out_weight || !lengths || !point_idx || !visible || !valid || !workspace)
        return (int)cudaErrorInvalidValue;
    if (workspace_bytes < scan_ws_bytes(b, max_scene) || !aligned_to(workspace, 256)) return (int)cudaErrorInvalidValue;
    cudaStream_t st = as_stream(stream);
    cudaError_t e = ensure_attrs(g_scan_select_attr, vscan_select_kernel, sizeof(unsigned long long) * kSelectMaxRows, false);
    if (e != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(workspace, 0, scan_zero_bytes(b, max_scene), st)) != cudaSuccess) return (int)e;
    const ScanArgs a{xyz, label, offsets, mean, scan_scene, scan_mode, seed_dev, (unsigned long long)seed, s};
    const ScanWs w = scan_ws(workspace, b, max_scene);
    vscan_ray_kernel<<<dim3((kRays + kRayThreads - 1) / kRayThreads, (unsigned)b), kRayThreads, 0, st>>>(a, w);
    int rc = finish_launch();
    if (rc) return rc;
    vscan_cell_kernel<<<(unsigned)b, kCellThreads, 0, st>>>(a, w);
    if ((rc = finish_launch())) return rc;
    const dim3 pgrid((unsigned)((max_scene + kPointChunk - 1) / kPointChunk), (unsigned)b);
    for (int pass = 0; pass < 2; ++pass) {
        vscan_point_kernel<<<pgrid, kPointThreads, 0, st>>>(a, w, pass);
        if ((rc = finish_launch())) return rc;
    }
    const ScanOut o{out_xyz, out_label, out_weight, lengths, point_idx, visible, valid};
    vscan_select_kernel<<<(unsigned)b, kSelectThreads, sizeof(unsigned long long) * pow2_at_least(npoints), st>>>(
        a, w, num_class, label_weights, npoints, min_points, o);
    return finish_launch();
}

}  // extern "C"
