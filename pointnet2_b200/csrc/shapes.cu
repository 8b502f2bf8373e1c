// shapes.cu — ModelNet / ShapeNet-part batches drawn from a packed shape set: seeded rows, point dropout and the five
// augmentation steps of utils/provider.py (modelnet_dataset.py:60-72, part_seg/part_dataset_all_normal.py:83-112), and
// the rotated votes of evaluate.py:117-158, as a padded ragged batch (DESIGN.md §6.11).
//
// One kernel, one 1024-thread CTA per entry, nothing read back: the CTA draws the entry's transform, takes the m
// smallest (key, row) pairs of its pool in order (cta_select_sorted), and writes the rows with the dropout compaction.
#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kShapeThreads = 1024;
constexpr double kPi = 3.141592653589793;
// random streams of DESIGN.md §6.11
constexpr unsigned long long kStreamKey = 1, kStreamRatio = 2, kStreamDrop = 3, kStreamAngle = 4, kStreamPerturb = 5,
                             kStreamScale = 6, kStreamShift = 7, kStreamJitter = 8;

struct ShapeArgs {
    const float* xyz;            // (p, 3)
    const float* nrm;            // (p, 3), or NULL
    const int* label;            // (s,)
    const int* part;             // (p,), or NULL
    const long long* offsets;    // (s + 1,)
    const long long* shape_idx;  // (b,)
    const long long* seed_dev;   // non-null: the seed is read here, on the device
    unsigned long long seed;
    int s, b, votes, npoints, subset_random, with_normals;
    int rotate, perturb, scale_on, jitter_on;
    double scale_lo, scale_hi, shift, jitter_sigma, jitter_clip, max_dropout;
};

struct ShapeOut {
    float* points;       // (E, npoints, 3 or 6)
    long long* label;    // (E,)
    long long* part;     // (E, npoints), or NULL
    int* lengths;        // (E,)
    int* point_idx;      // (E, npoints)
};

// normal(s, e, i) = sqrt(-2 ln(1 - u(draw(seed,s,e,2i)))) * cospi(2 u(draw(seed,s,e,2i+1))): Box-Muller
__device__ __forceinline__ double rng_normal(unsigned long long seed, unsigned long long s, unsigned long long e,
                                             unsigned long long i) {
    const double u1 = rng_unit(rng_draw(seed, s, e, 2 * i)), u2 = rng_unit(rng_draw(seed, s, e, 2 * i + 1));
    return __dmul_rn(sqrt(__dmul_rn(-2.0, log(__dsub_rn(1.0, u1)))), cospi(__dmul_rn(2.0, u2)));
}

__device__ __forceinline__ double clip(double x, double c) { return fmin(fmax(x, -c), c); }

// C = A B for 3x3 row-major matrices, each entry (a0 b0 + a1 b1) + a2 b2, every operation rounded
__device__ __forceinline__ void mat3_mul(const double (&a)[9], const double (&b)[9], double (&c)[9]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            c[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(a[3 * i], b[j]), __dmul_rn(a[3 * i + 1], b[3 + j])),
                                     __dmul_rn(a[3 * i + 2], b[6 + j]));
}

// rotation about y as provider.py:45-47 writes it: [[c, 0, s], [0, 1, 0], [-s, 0, c]]
__device__ __forceinline__ void rot_y(double c, double s, double (&r)[9]) {
    r[0] = c; r[1] = 0.0; r[2] = s;
    r[3] = 0.0; r[4] = 1.0; r[5] = 0.0;
    r[6] = -s; r[7] = 0.0; r[8] = c;
}

struct EntryXform {
    double m[9];       // p' = p M (row vectors)
    double scale;
    double shift[3];
    double ratio;      // dropout threshold
    int has_m;
};

// One CTA per entry.  Dynamic shared memory: the sort buffer, pow2 >= m 64-bit values.
__global__ void __launch_bounds__(kShapeThreads) shape_batch_kernel(ShapeArgs a, ShapeOut o) {
    extern __shared__ unsigned long long s_keys[];
    __shared__ SelectScratch s_sel;
    __shared__ EntryXform s_x;
    const int tid = threadIdx.x;
    const unsigned long long e = blockIdx.x;
    const int npoints = a.npoints, ch = a.with_normals ? 6 : 3;
    const size_t row0 = (size_t)e * npoints;
    const int v = a.votes ? (int)(e / a.b) : 0, bi = a.votes ? (int)(e % a.b) : (int)e;
    int sv = 0;
    long long off = 0, ps = 0;
    // a shape index outside [0, S): an empty entry, zero rows and label 0
    const bool in_range = set_entry(a.shape_idx, bi, a.s, a.offsets, sv, off, ps);
    const unsigned long long seed = rng_seed(a.seed_dev, a.seed);
    if (tid == 0) {
        EntryXform x;
        double r[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
        x.has_m = a.votes || a.rotate || a.perturb;
        if (a.votes || a.rotate) {
            // theta = v / V * 2 pi or u * 2 pi: sincospi of the exact-or-rounded half turn count needs no argument
            // reduction and agrees with cos / sin of the rounded theta to within a double ulp
            const double turns = a.votes ? __ddiv_rn((double)(2 * v), (double)a.votes)
                                         : __dmul_rn(rng_unit(rng_draw(seed, kStreamAngle, e, 0)), 2.0);
            double sn, cs;
            sincospi(turns, &sn, &cs);
            rot_y(cs, sn, r);
        }
        if (a.perturb) {  // Rz Ry Rx of provider.py:171-181, angles clip(0.06 normal, +-0.18)
            double ang[3];
            for (int i = 0; i < 3; ++i) ang[i] = clip(__dmul_rn(0.06, rng_normal(seed, kStreamPerturb, e, i)), 0.18);
            // sin / cos of |angle| <= 0.18 as sincospi(angle / pi): within a double ulp or two of sin / cos, and without
            // the large-argument reduction of sincos (its local-memory frame)
            double sx, cx, sy, cy, sz, cz;
            sincospi(__ddiv_rn(ang[0], kPi), &sx, &cx);
            sincospi(__ddiv_rn(ang[1], kPi), &sy, &cy);
            sincospi(__ddiv_rn(ang[2], kPi), &sz, &cz);
            const double rx[9] = {1.0, 0.0, 0.0, 0.0, cx, -sx, 0.0, sx, cx};
            const double rz[9] = {cz, -sz, 0.0, sz, cz, 0.0, 0.0, 0.0, 1.0};
            double ry[9], ryx[9], rp[9];
            rot_y(cy, sy, ry);
            mat3_mul(ry, rx, ryx);
            mat3_mul(rz, ryx, rp);
            mat3_mul(r, rp, x.m);
        } else {
            for (int i = 0; i < 9; ++i) x.m[i] = r[i];
        }
        x.scale = a.scale_on ? __dadd_rn(a.scale_lo, __dmul_rn(__dsub_rn(a.scale_hi, a.scale_lo),
                                                               rng_unit(rng_draw(seed, kStreamScale, e, 0))))
                             : 1.0;
        for (int d = 0; d < 3; ++d)
            x.shift[d] = __dadd_rn(-a.shift, __dmul_rn(2.0 * a.shift, rng_unit(rng_draw(seed, kStreamShift, e, d))));
        x.ratio = __dmul_rn(rng_unit(rng_draw(seed, kStreamRatio, e, 0)), a.max_dropout);
        s_x = x;
        o.label[e] = in_range ? __ldg(a.label + sv) : 0;
    }
    // the pool: rows 0 .. q-1 of the shape; its m smallest row orders are the entry's rows
    const int q = !in_range ? 0 : (a.subset_random && !a.votes) ? (int)ps : (int)min(ps, (long long)npoints);
    const int m = min(q, npoints);
    cta_select_sorted(
        q, q, m, [](long long) { return true; }, [&](long long j) { return rng_row_key(seed, kStreamKey, e, j); },
        s_keys, s_sel);
    // rows: dropout compaction (row 0 always stays), then each survivor transformed and written in row order
    const EntryXform& X = s_x;
    const bool drop_on = !a.votes && a.max_dropout > 0.0, shift_on = !a.votes && a.shift > 0.0;
    const bool scale_on = !a.votes && a.scale_on, jitter_on = !a.votes && a.jitter_on;
    const int kept = cta_compact(
        m,
        [&](int r) {
            return !(drop_on && r >= 1 && rng_unit(rng_draw(seed, kStreamDrop, e, (unsigned long long)r)) <= X.ratio);
        },
        [&](int r, int at) {
            const size_t row = row0 + at;
            const int j = (int)(s_keys[r] & 0xffffffffull);
            const long long g = off + j;
            double p[3], out[3];
            for (int d = 0; d < 3; ++d) p[d] = (double)__ldg(a.xyz + 3 * g + d);
            for (int d = 0; d < 3; ++d) {
                double y = p[d];
                if (X.has_m)
                    y = __dadd_rn(__dadd_rn(__dmul_rn(p[0], X.m[d]), __dmul_rn(p[1], X.m[3 + d])), __dmul_rn(p[2], X.m[6 + d]));
                if (scale_on) y = __dmul_rn(y, X.scale);
                if (shift_on) y = __dadd_rn(y, X.shift[d]);
                if (jitter_on)
                    y = __dadd_rn(y, clip(__dmul_rn(a.jitter_sigma, rng_normal(seed, kStreamJitter, e, 3ull * r + d)),
                                          a.jitter_clip));
                out[d] = y;
            }
            float* dst = o.points + ch * row;
            for (int d = 0; d < 3; ++d) dst[d] = __double2float_rn(out[d]);
            if (a.with_normals) {
                double n[3];
                for (int d = 0; d < 3; ++d) n[d] = (double)__ldg(a.nrm + 3 * g + d);
                for (int d = 0; d < 3; ++d) {
                    double y = n[d];
                    if (X.has_m)
                        y = __dadd_rn(__dadd_rn(__dmul_rn(n[0], X.m[d]), __dmul_rn(n[1], X.m[3 + d])), __dmul_rn(n[2], X.m[6 + d]));
                    dst[3 + d] = __double2float_rn(y);
                }
            }
            if (o.part) o.part[row] = __ldg(a.part + g);
            o.point_idx[row] = (int)g;
        },
        s_sel.w);
    for (int r = kept + tid; r < npoints; r += blockDim.x) {
        const size_t row = row0 + r;
        for (int c = 0; c < ch; ++c) o.points[ch * row + c] = 0.f;
        if (o.part) o.part[row] = 0;
        o.point_idx[row] = -1;
    }
    if (tid == 0) o.lengths[e] = kept;
}

bool finite_d(double x) { return x == x && x - x == 0.0; }

AttrOnce g_shape_attr;

}  // namespace
}  // namespace pn2

extern "C" {

int pn2_shape_batch(int s, int p, int max_shape, const float* xyz, const float* normals, const int* label, const int* part,
                    const long long* offsets, int b, const long long* shape_idx, long long seed, const long long* seed_dev,
                    int votes, int npoints, int subset_random, int rotate, int perturb, int scale_on, double scale_lo,
                    double scale_hi, double shift, int jitter_on, double jitter_sigma, double jitter_clip,
                    double max_dropout, int with_normals, float* out_points, long long* out_label, long long* out_part,
                    int* lengths, int* point_idx, void* stream) {
    using namespace pn2;
    if (s < 1 || p < 1 || p >= 0x7fffffff || max_shape < 1 || max_shape > p || max_shape > kSelectMaxRows || b < 1 ||
        votes < 0 || npoints < 1 || npoints > kSelectMaxRows)
        return (int)cudaErrorInvalidValue;
    const long long ent = votes ? (long long)votes * b : (long long)b;
    const int ch = with_normals ? 6 : 3;
    if (ent > 0x7fffffffll || ent * npoints * ch >= (1ll << 31)) return (int)cudaErrorInvalidValue;
    if ((subset_random != 0 && subset_random != 1) || (rotate != 0 && rotate != 1) || (perturb != 0 && perturb != 1) ||
        (scale_on != 0 && scale_on != 1) || (jitter_on != 0 && jitter_on != 1) || (with_normals != 0 && with_normals != 1))
        return (int)cudaErrorInvalidValue;
    if (scale_on && !(finite_d(scale_lo) && finite_d(scale_hi) && scale_lo <= scale_hi)) return (int)cudaErrorInvalidValue;
    if (!(finite_d(shift) && shift >= 0.0)) return (int)cudaErrorInvalidValue;
    if (jitter_on && !(finite_d(jitter_sigma) && jitter_sigma >= 0.0 && finite_d(jitter_clip) && jitter_clip > 0.0))
        return (int)cudaErrorInvalidValue;
    if (!(max_dropout >= 0.0 && max_dropout <= 1.0)) return (int)cudaErrorInvalidValue;
    // a vote is a rotation by v / V of a turn and a row permutation of the first npoints rows, nothing else
    if (votes && (subset_random || rotate || perturb || scale_on || shift != 0.0 || jitter_on || max_dropout != 0.0))
        return (int)cudaErrorInvalidValue;
    if (!xyz || !label || !offsets || !shape_idx || !out_points || !out_label || !lengths || !point_idx)
        return (int)cudaErrorInvalidValue;
    if ((with_normals && !normals) || (out_part && !part)) return (int)cudaErrorInvalidValue;
    const int pool = subset_random ? max_shape : (max_shape < npoints ? max_shape : npoints);
    const size_t smem = sizeof(unsigned long long) * pow2_at_least(pool < npoints ? pool : npoints);
    cudaError_t e = ensure_attrs(g_shape_attr, shape_batch_kernel, sizeof(unsigned long long) * kSelectMaxRows, false);
    if (e != cudaSuccess) return (int)e;
    const ShapeArgs a{xyz, with_normals ? normals : nullptr, label, out_part ? part : nullptr, offsets, shape_idx, seed_dev,
                      (unsigned long long)seed, s, b, votes, npoints, subset_random, with_normals, rotate, perturb,
                      scale_on, jitter_on, scale_lo, scale_hi, shift, jitter_sigma, jitter_clip, max_dropout};
    const ShapeOut o{out_points, out_label, out_part, lengths, point_idx};
    shape_batch_kernel<<<(unsigned)ent, kShapeThreads, smem, as_stream(stream)>>>(a, o);
    return finish_launch();
}

}  // extern "C"
