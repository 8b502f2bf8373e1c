// masked_bn.cu — batch norm + ReLU on a padded (rows, c) tensor, with the statistics taken over the real rows only
// (keep[r] != 0).  The learned layers of the segmentation nets run it on every BatchNorm1d + ReLU pair of a ragged batch.
//
// Forward:  stats kernel (per CTA: exact two-pass over register-held row groups, Chan-merged) -> finalize kernel
//           (fixed-order Chan merge of the per-CTA partials, saved statistics, running statistics) -> normalise kernel.
// Backward: sums kernel (per CTA: column sums of g and g*xhat) -> finalize kernel (fixed-order sums, dgamma / dbeta, the
//           per-column dx coefficients) -> dx kernel.
// Determinism: the row partition (rows per CTA) depends on c only, every sum has a fixed order, and no float atomics are
// used, so results are bit-identical across runs and devices.  Padding rows are never read.
#include <type_traits>

#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kMbnThreads = 256;   // threads per CTA of the row kernels
constexpr int kMbnRows = 8;        // rows a thread holds in registers at once (one row group)
constexpr int kMbnGroups = 4;      // row groups per thread in one CTA's chunk
constexpr int kMbnMergeWarps = 32; // warps of a finalize CTA (one 32-column slice)

// Thread geometry of the row kernels, a function of c alone: each thread owns `vec` consecutive columns (4 when c is a
// multiple of 4, else 1), tx threads span a column tile, ty = 256 / tx rows are in flight per step.  A CTA of the
// statistics / sums kernels covers chunk_rows = ty * 8 * 4 rows of one column tile.
struct MbnGeom {
    int vec, tx, ty, col_tiles, chunk_rows;
    long long chunks;
};

MbnGeom mbn_geom(int rows, int c) {
    MbnGeom g;
    g.vec = (c % 4 == 0) ? 4 : 1;
    const int lanes = (c + g.vec - 1) / g.vec;
    int tx = 1;
    while (tx < lanes && tx < 32) tx <<= 1;
    g.tx = tx;
    g.ty = kMbnThreads / tx;
    g.col_tiles = (lanes + tx - 1) / tx;
    g.chunk_rows = g.ty * kMbnRows * kMbnGroups;
    g.chunks = rows > 0 ? ((long long)rows + g.chunk_rows - 1) / g.chunk_rows : 0;
    return g;
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// Workspace: two float partials per (chunk, column), one int count per chunk, three floats per column (backward).
struct MbnLayout {
    size_t pa, pb, cnt, coef, total;
};

MbnLayout mbn_layout(const MbnGeom& g, int c) {
    MbnLayout L;
    const size_t part = align256(sizeof(float) * (size_t)g.chunks * c);
    L.pa = 0;
    L.pb = part;
    L.cnt = 2 * part;
    L.coef = L.cnt + align256(sizeof(int) * (size_t)g.chunks);
    L.total = L.coef + align256(sizeof(float) * 3 * (size_t)c);
    return L;
}

// V consecutive elements at p, upcast to float: one vector load when VEC (p aligned to V elements), else V scalar loads
template <typename T, int V, bool VEC>
__device__ __forceinline__ void load_cols(const T* p, float (&v)[V]) {
    if constexpr (VEC) {
        const float4 f = ldg4(p);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) v[i] = to_f32(__ldg(p + i));
    }
}
template <typename T, int V, bool VEC>
__device__ __forceinline__ void store_cols(T* p, const float (&v)[V]) {
    if constexpr (VEC) {
        st4(p, make_float4(v[0], v[1], v[2], v[3]));
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) p[i] = from_f32<T>(v[i]);
    }
}

// Chan's merge of (nb, mb, m2b) into (na, ma, m2a), V columns sharing one count
template <int V>
__device__ __forceinline__ void chan_merge(int& na, float (&ma)[V], float (&m2a)[V], int nb, const float* mb, const float* m2b) {
    if (nb == 0) return;
    if (na == 0) {
        na = nb;
#pragma unroll
        for (int i = 0; i < V; ++i) { ma[i] = mb[i]; m2a[i] = m2b[i]; }
        return;
    }
    const int n = na + nb;
    const float wb = __fdiv_rn((float)nb, (float)n);  // nb / n
    const float wab = __fmul_rn((float)na, wb);       // na * nb / n
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const float d = __fsub_rn(mb[i], ma[i]);
        ma[i] = __fmaf_rn(d, wb, ma[i]);
        m2a[i] = __fadd_rn(__fadd_rn(m2a[i], m2b[i]), __fmul_rn(__fmul_rn(d, d), wab));
    }
    na = n;
}

// ---- forward ---------------------------------------------------------------------------------------------------------

// Per CTA (chunk blockIdx.x, column tile blockIdx.y): count, mean and M2 over the real rows of the chunk.  Each thread
// takes its rows in groups of kMbnRows held in registers, does an exact two-pass over each group and Chan-merges the
// groups in order; the ty threads of a column are then merged in a fixed tree.  Writes pmean / pm2 [chunk][c], pcnt[chunk].
template <typename T, int V, bool VEC>
__global__ void __launch_bounds__(kMbnThreads) mbn_stats_kernel(const T* __restrict__ x, const unsigned char* __restrict__ keep,
                                                                int rows, int c, float* __restrict__ pmean,
                                                                float* __restrict__ pm2, int* __restrict__ pcnt) {
    __shared__ float s_mean[kMbnThreads * V], s_m2[kMbnThreads * V];
    __shared__ int s_n[kMbnThreads];
    const int tx = blockDim.x, ty = blockDim.y, tid = threadIdx.y * tx + threadIdx.x;
    const int col = (blockIdx.y * tx + threadIdx.x) * V;
    const bool active = col < c;
    const long long row0 = (long long)blockIdx.x * ty * (kMbnRows * kMbnGroups) + threadIdx.y;
    int n = 0;
    float mean[V], m2[V];
#pragma unroll
    for (int i = 0; i < V; ++i) { mean[i] = 0.f; m2[i] = 0.f; }
#pragma unroll 1
    for (int grp = 0; grp < kMbnGroups; ++grp) {
        const long long rbase = row0 + (long long)grp * ty * kMbnRows;
        bool kf[kMbnRows];
#pragma unroll
        for (int k = 0; k < kMbnRows; ++k) {
            const long long r = rbase + (long long)k * ty;
            kf[k] = r < rows && __ldg(keep + r) != 0;
        }
        float v[kMbnRows][V];
#pragma unroll
        for (int k = 0; k < kMbnRows; ++k) {
            if (active && kf[k]) {
                load_cols<T, V, VEC>(x + (size_t)(rbase + (long long)k * ty) * c + col, v[k]);
            } else {
#pragma unroll
                for (int i = 0; i < V; ++i) v[k][i] = 0.f;
            }
        }
        int ng = 0;
#pragma unroll
        for (int k = 0; k < kMbnRows; ++k) ng += kf[k] ? 1 : 0;
        if (ng == 0) continue;
        float gmean[V], gm2[V];
        const float inv_ng = __fdiv_rn(1.0f, (float)ng);
#pragma unroll
        for (int i = 0; i < V; ++i) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < kMbnRows; ++k) s = __fadd_rn(s, v[k][i]);  // padding rows hold 0
            gmean[i] = __fmul_rn(s, inv_ng);
            float q = 0.f;
#pragma unroll
            for (int k = 0; k < kMbnRows; ++k) {
                const float d = kf[k] ? __fsub_rn(v[k][i], gmean[i]) : 0.f;
                q = __fmaf_rn(d, d, q);
            }
            gm2[i] = q;
        }
        chan_merge<V>(n, mean, m2, ng, gmean, gm2);
    }
    // fixed tree over the ty threads of each column: row slot y absorbs slot y + s
#pragma unroll
    for (int i = 0; i < V; ++i) {
        s_mean[tid * V + i] = mean[i];
        s_m2[tid * V + i] = m2[i];
    }
    s_n[tid] = n;
    __syncthreads();
    for (int s = ty >> 1; s > 0; s >>= 1) {
        if ((int)threadIdx.y < s) {
            const int o = tid + s * tx;
            chan_merge<V>(n, mean, m2, s_n[o], s_mean + o * V, s_m2 + o * V);
#pragma unroll
            for (int i = 0; i < V; ++i) {
                s_mean[tid * V + i] = mean[i];
                s_m2[tid * V + i] = m2[i];
            }
            s_n[tid] = n;
        }
        __syncthreads();
    }
    if (threadIdx.y == 0) {
        if (active) {
            const size_t o = (size_t)blockIdx.x * c + col;
#pragma unroll
            for (int i = 0; i < V; ++i) {
                pmean[o + i] = mean[i];
                pm2[o + i] = m2[i];
            }
        }
        if (threadIdx.x == 0 && blockIdx.y == 0) pcnt[blockIdx.x] = n;
    }
}

// One CTA per 32 columns: warp w Chan-merges its contiguous range of chunks in ascending order, then the 32 warps are
// merged in a fixed tree.  Writes the saved statistics and updates the running ones.
__global__ void __launch_bounds__(32 * kMbnMergeWarps) mbn_finalize_kernel(
    const float* __restrict__ pmean, const float* __restrict__ pm2, const int* __restrict__ pcnt, long long chunks, int c,
    float eps, float momentum, const long long* __restrict__ num_batches_tracked, float* __restrict__ running_mean,
    float* __restrict__ running_var, float* __restrict__ save_mean, float* __restrict__ save_invstd) {
    __shared__ float s_mean[kMbnMergeWarps][32], s_m2[kMbnMergeWarps][32];
    __shared__ int s_n[kMbnMergeWarps];
    const int lane = threadIdx.x, w = threadIdx.y;
    const int col = blockIdx.x * 32 + lane;
    const bool active = col < c;
    const long long per = (chunks + kMbnMergeWarps - 1) / kMbnMergeWarps;
    const long long k0 = min(chunks, (long long)w * per), k1 = min(chunks, k0 + per);
    int n = 0;
    float mean[1] = {0.f}, m2[1] = {0.f};
    for (long long k = k0; k < k1; ++k) {
        const int nb = __ldg(pcnt + k);
        float mb = 0.f, m2b = 0.f;
        if (active) {
            mb = __ldg(pmean + (size_t)k * c + col);
            m2b = __ldg(pm2 + (size_t)k * c + col);
        }
        chan_merge<1>(n, mean, m2, nb, &mb, &m2b);
    }
    s_mean[w][lane] = mean[0];
    s_m2[w][lane] = m2[0];
    if (lane == 0) s_n[w] = n;
    __syncthreads();
    for (int s = kMbnMergeWarps >> 1; s > 0; s >>= 1) {
        if (w < s) {
            chan_merge<1>(n, mean, m2, s_n[w + s], &s_mean[w + s][lane], &s_m2[w + s][lane]);
            s_mean[w][lane] = mean[0];
            s_m2[w][lane] = m2[0];
            __syncwarp();
            if (lane == 0) s_n[w] = n;
        }
        __syncthreads();
    }
    if (w != 0 || !active) return;
    const float cnt = (float)n;
    // without a real row the mean is 0 / 0 (NaN) as layers.masked_batch_norm computes it, and so are the variance and
    // both running statistics
    const float mu = n > 0 ? mean[0] : __fdiv_rn(0.f, cnt);
    const float var = __fdiv_rn(m2[0], cnt);  // biased
    save_mean[col] = mu;
    save_invstd[col] = rsqrtf(__fadd_rn(var, eps));
    if (running_mean) {
        // as layers.masked_batch_norm: momentum, or the cumulative average 1 / num_batches_tracked (already incremented)
        const float f = momentum < 0.f ? __fdiv_rn(1.0f, (float)__ldg(num_batches_tracked)) : momentum;
        const float keepf = __fsub_rn(1.0f, f);
        const float unbiased = __fdiv_rn(__fmul_rn(var, cnt), fmaxf(__fsub_rn(cnt, 1.0f), 1.0f));
        running_mean[col] = __fadd_rn(__fmul_rn(running_mean[col], keepf), __fmul_rn(mu, f));
        running_var[col] = __fadd_rn(__fmul_rn(running_var[col], keepf), __fmul_rn(unbiased, f));
    }
}

constexpr int kMbnUnroll = 4;  // rows per thread per step of the elementwise kernels

// y = keep ? max(0, (x - mean) * (invstd * gamma) + beta) : 0, one fused multiply-add per element
template <typename T, int V, bool VEC>
__global__ void __launch_bounds__(kMbnThreads) mbn_norm_relu_kernel(const T* __restrict__ x, const unsigned char* __restrict__ keep,
                                                                    int rows, int c, const float* __restrict__ mean,
                                                                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta, T* __restrict__ y) {
    const int tx = blockDim.x, ty = blockDim.y;
    const int col = (blockIdx.y * tx + threadIdx.x) * V;
    if (col >= c) return;  // no barrier in this kernel
    float mu[V], sc[V], sh[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        mu[i] = __ldg(mean + col + i);
        const float is = __ldg(invstd + col + i);
        sc[i] = gamma ? __fmul_rn(is, __ldg(gamma + col + i)) : is;
        sh[i] = beta ? __ldg(beta + col + i) : 0.f;
    }
    const long long step = (long long)gridDim.x * ty * kMbnUnroll;
    for (long long rb = (long long)blockIdx.x * ty * kMbnUnroll + threadIdx.y; rb < rows; rb += step) {
        bool kf[kMbnUnroll];
        float v[kMbnUnroll][V];
#pragma unroll
        for (int u = 0; u < kMbnUnroll; ++u) {
            const long long r = rb + (long long)u * ty;
            kf[u] = r < rows && __ldg(keep + r) != 0;
            if (kf[u]) {
                load_cols<T, V, VEC>(x + (size_t)r * c + col, v[u]);
            } else {
#pragma unroll
                for (int i = 0; i < V; ++i) v[u][i] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < kMbnUnroll; ++u) {
            const long long r = rb + (long long)u * ty;
            if (r >= rows) break;
            float o[V];
#pragma unroll
            for (int i = 0; i < V; ++i) {
                const float t = __fmaf_rn(__fsub_rn(v[u][i], mu[i]), sc[i], sh[i]);
                o[i] = kf[u] ? (t < 0.f ? 0.f : t) : 0.f;
            }
            store_cols<T, V, VEC>(y + (size_t)r * c + col, o);
        }
    }
}

// One CTA per (cloud, column tile) of a (b, n, c) x: y as mbn_norm_relu_kernel computes and rounds it, and per column
// its maximum over the cloud's real rows with the FIRST row that reaches it (where TF's MaxPoolGrad sends the gradient).
// Values are compared as max_key keys, so NaN wins.  Each thread walks rows threadIdx.y, + ty, ... and keeps the first
// of equal keys; the ty threads of a column are merged in a fixed tree that prefers the lower row on equal keys.
// A cloud without a real row gets out 0 and argmax -1.  Only out (b, c) and argmax (b, c) are written.
template <typename T, int V, bool VEC>
__global__ void __launch_bounds__(kMbnThreads) mbn_norm_relu_max_kernel(const T* __restrict__ x,
                                                                        const unsigned char* __restrict__ keep, int n, int c,
                                                                        const float* __restrict__ mean,
                                                                        const float* __restrict__ invstd,
                                                                        const float* __restrict__ gamma,
                                                                        const float* __restrict__ beta, T* __restrict__ out,
                                                                        int* __restrict__ argmax) {
    __shared__ unsigned s_key[kMbnThreads * V];
    __shared__ int s_row[kMbnThreads * V];
    const int tx = blockDim.x, ty = blockDim.y, tid = threadIdx.y * tx + threadIdx.x;
    const int col = (blockIdx.y * tx + threadIdx.x) * V;
    const bool active = col < c;
    const long long cloud = blockIdx.x;
    float mu[V], sc[V], sh[V];
    unsigned key[V];
    int arg[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        mu[i] = active ? __ldg(mean + col + i) : 0.f;
        const float is = active ? __ldg(invstd + col + i) : 0.f;
        sc[i] = gamma && active ? __fmul_rn(is, __ldg(gamma + col + i)) : is;
        sh[i] = beta && active ? __ldg(beta + col + i) : 0.f;
        key[i] = 0u;
        arg[i] = -1;
    }
    if (active) {
        const T* xc = x + (size_t)cloud * n * c + col;
        const unsigned char* kc = keep + (size_t)cloud * n;
        for (int jb = threadIdx.y; jb < n; jb += ty * kMbnUnroll) {
            bool kf[kMbnUnroll];
            float v[kMbnUnroll][V];
#pragma unroll
            for (int u = 0; u < kMbnUnroll; ++u) {
                const int j = jb + u * ty;
                kf[u] = j < n && __ldg(kc + j) != 0;
                if (kf[u]) {
                    load_cols<T, V, VEC>(xc + (size_t)j * c, v[u]);
                } else {
#pragma unroll
                    for (int i = 0; i < V; ++i) v[u][i] = 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < kMbnUnroll; ++u) {
#pragma unroll
                for (int i = 0; i < V; ++i) {
                    const float t = __fmaf_rn(__fsub_rn(v[u][i], mu[i]), sc[i], sh[i]);
                    // the value y holds in T, compared as a key: the maximum and its first row are those of the
                    // rounded tensor masked_batch_norm_relu would write
                    const unsigned k = max_key(to_f32(from_f32<T>(t < 0.f ? 0.f : t)));
                    if (kf[u] && k > key[i]) {
                        key[i] = k;
                        arg[i] = jb + u * ty;
                    }
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
        s_key[tid * V + i] = key[i];
        s_row[tid * V + i] = arg[i];
    }
    __syncthreads();
    for (int s = ty >> 1; s > 0; s >>= 1) {
        if ((int)threadIdx.y < s) {
            const int o = tid + s * tx;
#pragma unroll
            for (int i = 0; i < V; ++i) {
                const unsigned kb = s_key[o * V + i];
                const int rb = s_row[o * V + i];
                if (kb > key[i] || (kb == key[i] && kb != 0u && rb < arg[i])) {
                    key[i] = kb;
                    arg[i] = rb;
                }
                s_key[tid * V + i] = key[i];
                s_row[tid * V + i] = arg[i];
            }
        }
        __syncthreads();
    }
    if (threadIdx.y == 0 && active) {
#pragma unroll
        for (int i = 0; i < V; ++i) {
            out[(size_t)cloud * c + col + i] = from_f32<T>(key[i] ? key_value(key[i]) : 0.f);
            argmax[(size_t)cloud * c + col + i] = key[i] ? arg[i] : -1;
        }
    }
}

// ---- backward --------------------------------------------------------------------------------------------------------

// Backward of the max-pooled form, step 1.  One CTA per 32 columns: the CTA counts the real rows (an integer sum), then
// for each column g[i] = out[i] > 0 ? dout[i] : 0 (the gradient of the ReLU at the argmax row; the other rows get none),
// dbeta = sum_i g[i] and dgamma = sum_i g[i] * xhat(argmax row), both over the clouds i in ascending order: the warps
// take 32 clouds at a time and warp 0 adds their terms in order.  Writes dgamma / dbeta (either may be NULL), gsel (b, c)
// and the dx coefficients coef[3][c] of mbn_bwd_dx_kernel.
template <typename T>
__global__ void __launch_bounds__(32 * kMbnMergeWarps) mbn_max_bwd_finalize_kernel(
    const T* __restrict__ dout, const T* __restrict__ x, const T* __restrict__ out, const int* __restrict__ argmax,
    const unsigned char* __restrict__ keep, int b, int n, int c, const float* __restrict__ gamma,
    const float* __restrict__ mean, const float* __restrict__ invstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
    float* __restrict__ gsel, float* __restrict__ coef) {
    __shared__ float s_g[kMbnMergeWarps][32], s_xh[kMbnMergeWarps][32];
    __shared__ int s_cnt;
    const int lane = threadIdx.x, w = threadIdx.y, tid = w * 32 + lane;
    const int col = blockIdx.x * 32 + lane;
    const bool active = col < c;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    const long long rows = (long long)b * n;
    int cnt = 0;
    for (long long r = tid; r < rows; r += 32 * kMbnMergeWarps) cnt += __ldg(keep + r) != 0;
    cnt += __shfl_xor_sync(kFullMask, cnt, 16);
    cnt += __shfl_xor_sync(kFullMask, cnt, 8);
    cnt += __shfl_xor_sync(kFullMask, cnt, 4);
    cnt += __shfl_xor_sync(kFullMask, cnt, 2);
    cnt += __shfl_xor_sync(kFullMask, cnt, 1);
    if (lane == 0) atomicAdd(&s_cnt, cnt);  // an integer sum: exact in any order
    const float mu = active ? __ldg(mean + col) : 0.f, is = active ? __ldg(invstd + col) : 0.f;
    float sg = 0.f, sgx = 0.f;
    for (int i0 = 0; i0 < b; i0 += kMbnMergeWarps) {
        const int i = i0 + w;
        float g = 0.f, xh = 0.f;
        if (active && i < b) {
            const size_t o = (size_t)i * c + col;
            const int r = __ldg(argmax + o);
            if (r >= 0 && to_f32(out[o]) > 0.f) {
                g = to_f32(dout[o]);
                xh = __fmul_rn(__fsub_rn(to_f32(x[((size_t)i * n + r) * c + col]), mu), is);
            }
            gsel[o] = g;
        }
        s_g[w][lane] = g;
        s_xh[w][lane] = xh;
        __syncthreads();
        if (w == 0) {
            const int m = min(kMbnMergeWarps, b - i0);
            for (int k = 0; k < m; ++k) {
                sg = __fadd_rn(sg, s_g[k][lane]);
                sgx = __fmaf_rn(s_g[k][lane], s_xh[k][lane], sgx);
            }
        }
        __syncthreads();
    }
    if (w != 0 || !active) return;
    if (dbeta) dbeta[col] = sg;
    if (dgamma) dgamma[col] = sgx;
    const float fc = (float)s_cnt;
    coef[col] = gamma ? __fmul_rn(__ldg(gamma + col), is) : is;
    coef[c + col] = __fdiv_rn(sg, fc);
    coef[2 * c + col] = __fdiv_rn(sgx, fc);
}

// Step 2: dx = keep ? gamma * invstd * (g - sum g / cnt - xhat * sum g * xhat / cnt) : 0 with g = gsel[i] at the argmax
// row of cloud i and 0 elsewhere (the arithmetic of mbn_bwd_dx_kernel)
template <typename T, int V, bool VEC>
__global__ void __launch_bounds__(kMbnThreads) mbn_max_bwd_dx_kernel(const T* __restrict__ x, const unsigned char* __restrict__ keep,
                                                                     int rows, int n, int c, const int* __restrict__ argmax,
                                                                     const float* __restrict__ gsel,
                                                                     const float* __restrict__ mean,
                                                                     const float* __restrict__ invstd,
                                                                     const float* __restrict__ coef, T* __restrict__ dx) {
    const int tx = blockDim.x, ty = blockDim.y;
    const int col = (blockIdx.y * tx + threadIdx.x) * V;
    if (col >= c) return;  // no barrier in this kernel
    float mu[V], is[V], a[V], mg[V], mgx[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        mu[i] = __ldg(mean + col + i);
        is[i] = __ldg(invstd + col + i);
        a[i] = __ldg(coef + col + i);
        mg[i] = __ldg(coef + c + col + i);
        mgx[i] = __ldg(coef + 2 * c + col + i);
    }
    const long long step = (long long)gridDim.x * ty * kMbnUnroll;
    for (long long rb = (long long)blockIdx.x * ty * kMbnUnroll + threadIdx.y; rb < rows; rb += step) {
        bool kf[kMbnUnroll];
        float xv[kMbnUnroll][V];
#pragma unroll
        for (int u = 0; u < kMbnUnroll; ++u) {
            const long long r = rb + (long long)u * ty;
            kf[u] = r < rows && __ldg(keep + r) != 0;
            if (kf[u]) {
                load_cols<T, V, VEC>(x + (size_t)r * c + col, xv[u]);
            } else {
#pragma unroll
                for (int i = 0; i < V; ++i) xv[u][i] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < kMbnUnroll; ++u) {
            const long long r = rb + (long long)u * ty;
            if (r >= rows) break;
            const long long cloud = r / n;
            const int j = (int)(r - cloud * n);
            float o[V];
#pragma unroll
            for (int i = 0; i < V; ++i) {
                const size_t bc = (size_t)cloud * c + col + i;
                const float g = __ldg(argmax + bc) == j ? __ldg(gsel + bc) : 0.f;
                const float xh = __fmul_rn(__fsub_rn(xv[u][i], mu[i]), is[i]);
                const float t = __fmaf_rn(-xh, mgx[i], __fsub_rn(g, mg[i]));
                o[i] = kf[u] ? __fmul_rn(a[i], t) : 0.f;
            }
            store_cols<T, V, VEC>(dx + (size_t)r * c + col, o);
        }
    }
}

// Per CTA (same chunks as the forward): count and column sums of g = dy * [y > 0] and g * xhat over the real rows, each
// thread adding its rows in ascending order, then a fixed tree over the ty threads of each column.
template <typename T, int V, bool VEC>
__global__ void __launch_bounds__(kMbnThreads) mbn_bwd_sums_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                   const T* __restrict__ y, const unsigned char* __restrict__ keep,
                                                                   int rows, int c, const float* __restrict__ mean,
                                                                   const float* __restrict__ invstd, float* __restrict__ psg,
                                                                   float* __restrict__ psgx, int* __restrict__ pcnt) {
    __shared__ float s_a[kMbnThreads * V], s_b[kMbnThreads * V];
    __shared__ int s_n[kMbnThreads];
    const int tx = blockDim.x, ty = blockDim.y, tid = threadIdx.y * tx + threadIdx.x;
    const int col = (blockIdx.y * tx + threadIdx.x) * V;
    const bool active = col < c;
    float mu[V], is[V], sg[V], sgx[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        mu[i] = active ? __ldg(mean + col + i) : 0.f;
        is[i] = active ? __ldg(invstd + col + i) : 0.f;
        sg[i] = 0.f;
        sgx[i] = 0.f;
    }
    const long long row0 = (long long)blockIdx.x * ty * (kMbnRows * kMbnGroups) + threadIdx.y;
    int n = 0;
#pragma unroll 1
    for (int grp = 0; grp < kMbnGroups; ++grp) {
        const long long rbase = row0 + (long long)grp * ty * kMbnRows;
        bool kf[kMbnRows];
#pragma unroll
        for (int k = 0; k < kMbnRows; ++k) {
            const long long r = rbase + (long long)k * ty;
            kf[k] = r < rows && __ldg(keep + r) != 0;
            n += kf[k] ? 1 : 0;
        }
        if (!active) continue;
#pragma unroll
        for (int k = 0; k < kMbnRows; ++k) {
            if (!kf[k]) continue;
            const size_t o = (size_t)(rbase + (long long)k * ty) * c + col;
            float gv[V], xv[V], yv[V];
            load_cols<T, V, VEC>(dy + o, gv);
            load_cols<T, V, VEC>(y + o, yv);
            load_cols<T, V, VEC>(x + o, xv);
#pragma unroll
            for (int i = 0; i < V; ++i) {
                const float g = yv[i] > 0.f ? gv[i] : 0.f;
                const float xh = __fmul_rn(__fsub_rn(xv[i], mu[i]), is[i]);
                sg[i] = __fadd_rn(sg[i], g);
                sgx[i] = __fmaf_rn(g, xh, sgx[i]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
        s_a[tid * V + i] = sg[i];
        s_b[tid * V + i] = sgx[i];
    }
    s_n[tid] = n;
    __syncthreads();
    for (int s = ty >> 1; s > 0; s >>= 1) {
        if ((int)threadIdx.y < s) {
            const int o = tid + s * tx;
            n += s_n[o];
#pragma unroll
            for (int i = 0; i < V; ++i) {
                sg[i] = __fadd_rn(sg[i], s_a[o * V + i]);
                sgx[i] = __fadd_rn(sgx[i], s_b[o * V + i]);
                s_a[tid * V + i] = sg[i];
                s_b[tid * V + i] = sgx[i];
            }
            s_n[tid] = n;
        }
        __syncthreads();
    }
    if (threadIdx.y == 0) {
        if (active) {
            const size_t o = (size_t)blockIdx.x * c + col;
#pragma unroll
            for (int i = 0; i < V; ++i) {
                psg[o + i] = sg[i];
                psgx[o + i] = sgx[i];
            }
        }
        if (threadIdx.x == 0 && blockIdx.y == 0) pcnt[blockIdx.x] = n;
    }
}

// One CTA per 32 columns: warp w adds its contiguous range of chunks in ascending order, then a fixed tree over the 32
// warps.  Writes dbeta = sum g, dgamma = sum g * xhat (either may be NULL) and coef[3][c] = (gamma * invstd,
// sum g / cnt, sum g * xhat / cnt) for the dx kernel.
__global__ void __launch_bounds__(32 * kMbnMergeWarps) mbn_bwd_finalize_kernel(
    const float* __restrict__ psg, const float* __restrict__ psgx, const int* __restrict__ pcnt, long long chunks, int c,
    const float* __restrict__ gamma, const float* __restrict__ invstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
    float* __restrict__ coef) {
    __shared__ float s_a[kMbnMergeWarps][32], s_b[kMbnMergeWarps][32];
    __shared__ int s_n[kMbnMergeWarps];
    const int lane = threadIdx.x, w = threadIdx.y;
    const int col = blockIdx.x * 32 + lane;
    const bool active = col < c;
    const long long per = (chunks + kMbnMergeWarps - 1) / kMbnMergeWarps;
    const long long k0 = min(chunks, (long long)w * per), k1 = min(chunks, k0 + per);
    int n = 0;
    float sg = 0.f, sgx = 0.f;
    for (long long k = k0; k < k1; ++k) {
        n += __ldg(pcnt + k);
        if (active) {
            sg = __fadd_rn(sg, __ldg(psg + (size_t)k * c + col));
            sgx = __fadd_rn(sgx, __ldg(psgx + (size_t)k * c + col));
        }
    }
    s_a[w][lane] = sg;
    s_b[w][lane] = sgx;
    if (lane == 0) s_n[w] = n;
    __syncthreads();
    for (int s = kMbnMergeWarps >> 1; s > 0; s >>= 1) {
        if (w < s) {
            sg = __fadd_rn(sg, s_a[w + s][lane]);
            sgx = __fadd_rn(sgx, s_b[w + s][lane]);
            n += s_n[w + s];
            s_a[w][lane] = sg;
            s_b[w][lane] = sgx;
            __syncwarp();
            if (lane == 0) s_n[w] = n;
        }
        __syncthreads();
    }
    if (w != 0 || !active) return;
    if (dbeta) dbeta[col] = sg;
    if (dgamma) dgamma[col] = sgx;
    const float cnt = (float)n;
    const float is = __ldg(invstd + col);
    coef[col] = gamma ? __fmul_rn(__ldg(gamma + col), is) : is;
    coef[c + col] = __fdiv_rn(sg, cnt);
    coef[2 * c + col] = __fdiv_rn(sgx, cnt);
}

// dx = keep ? gamma * invstd * (g - sum g / cnt - xhat * sum g * xhat / cnt) : 0
template <typename T, int V, bool VEC>
__global__ void __launch_bounds__(kMbnThreads) mbn_bwd_dx_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                 const T* __restrict__ y, const unsigned char* __restrict__ keep,
                                                                 int rows, int c, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd, const float* __restrict__ coef,
                                                                 T* __restrict__ dx) {
    const int tx = blockDim.x, ty = blockDim.y;
    const int col = (blockIdx.y * tx + threadIdx.x) * V;
    if (col >= c) return;  // no barrier in this kernel
    float mu[V], is[V], a[V], mg[V], mgx[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        mu[i] = __ldg(mean + col + i);
        is[i] = __ldg(invstd + col + i);
        a[i] = __ldg(coef + col + i);
        mg[i] = __ldg(coef + c + col + i);
        mgx[i] = __ldg(coef + 2 * c + col + i);
    }
    const long long step = (long long)gridDim.x * ty * kMbnUnroll;
    for (long long rb = (long long)blockIdx.x * ty * kMbnUnroll + threadIdx.y; rb < rows; rb += step) {
        bool kf[kMbnUnroll];
        float gv[kMbnUnroll][V], xv[kMbnUnroll][V], yv[kMbnUnroll][V];
#pragma unroll
        for (int u = 0; u < kMbnUnroll; ++u) {
            const long long r = rb + (long long)u * ty;
            kf[u] = r < rows && __ldg(keep + r) != 0;
            if (kf[u]) {
                const size_t o = (size_t)r * c + col;
                load_cols<T, V, VEC>(dy + o, gv[u]);
                load_cols<T, V, VEC>(y + o, yv[u]);
                load_cols<T, V, VEC>(x + o, xv[u]);
            } else {
#pragma unroll
                for (int i = 0; i < V; ++i) gv[u][i] = xv[u][i] = yv[u][i] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < kMbnUnroll; ++u) {
            const long long r = rb + (long long)u * ty;
            if (r >= rows) break;
            float o[V];
#pragma unroll
            for (int i = 0; i < V; ++i) {
                const float g = yv[u][i] > 0.f ? gv[u][i] : 0.f;
                const float xh = __fmul_rn(__fsub_rn(xv[u][i], mu[i]), is[i]);
                const float t = __fmaf_rn(-xh, mgx[i], __fsub_rn(g, mg[i]));
                o[i] = kf[u] ? __fmul_rn(a[i], t) : 0.f;
            }
            store_cols<T, V, VEC>(dx + (size_t)r * c + col, o);
        }
    }
}

// CTAs along the rows of an elementwise kernel: enough for ~8 resident CTAs per SM over all column tiles (the result
// does not depend on it)
unsigned elementwise_row_blocks(const MbnGeom& g, int rows) {
    const unsigned long long need = ((unsigned long long)rows + (unsigned long long)g.ty * kMbnUnroll - 1) / ((unsigned long long)g.ty * kMbnUnroll);
    const unsigned long long cap = (unsigned long long)num_sms() * 8 / g.col_tiles + 1;
    return (unsigned)(need < cap ? need : cap);
}

template <typename T, int V, bool VEC>
int forward_launch(const MbnGeom& g, int rows, int c, const T* x, const unsigned char* keep, const float* gamma,
                   const float* beta, float eps, float momentum, const long long* nbt, float* running_mean,
                   float* running_var, T* y, float* save_mean, float* save_invstd, char* ws, const MbnLayout& L,
                   cudaStream_t st) {
    float* pa = reinterpret_cast<float*>(ws + L.pa);
    float* pb = reinterpret_cast<float*>(ws + L.pb);
    int* pc = reinterpret_cast<int*>(ws + L.cnt);
    const dim3 block(g.tx, g.ty);
    mbn_stats_kernel<T, V, VEC><<<dim3((unsigned)g.chunks, g.col_tiles), block, 0, st>>>(x, keep, rows, c, pa, pb, pc);
    int rc = finish_launch();
    if (rc) return rc;
    mbn_finalize_kernel<<<ceil_div_u(c, 32), dim3(32, kMbnMergeWarps), 0, st>>>(pa, pb, pc, g.chunks, c, eps, momentum, nbt,
                                                                                 running_mean, running_var, save_mean, save_invstd);
    rc = finish_launch();
    if (rc) return rc;
    mbn_norm_relu_kernel<T, V, VEC><<<dim3(elementwise_row_blocks(g, rows), g.col_tiles), block, 0, st>>>(
        x, keep, rows, c, save_mean, save_invstd, gamma, beta, y);
    return finish_launch();
}

template <typename T, int V, bool VEC>
int backward_launch(const MbnGeom& g, int rows, int c, const T* dy, const T* x, const T* y, const unsigned char* keep,
                    const float* gamma, const float* save_mean, const float* save_invstd, T* dx, float* dgamma,
                    float* dbeta, char* ws, const MbnLayout& L, cudaStream_t st) {
    float* pa = reinterpret_cast<float*>(ws + L.pa);
    float* pb = reinterpret_cast<float*>(ws + L.pb);
    int* pc = reinterpret_cast<int*>(ws + L.cnt);
    float* coef = reinterpret_cast<float*>(ws + L.coef);
    const dim3 block(g.tx, g.ty);
    mbn_bwd_sums_kernel<T, V, VEC><<<dim3((unsigned)g.chunks, g.col_tiles), block, 0, st>>>(dy, x, y, keep, rows, c, save_mean,
                                                                                           save_invstd, pa, pb, pc);
    int rc = finish_launch();
    if (rc) return rc;
    mbn_bwd_finalize_kernel<<<ceil_div_u(c, 32), dim3(32, kMbnMergeWarps), 0, st>>>(pa, pb, pc, g.chunks, c, gamma, save_invstd,
                                                                                     dgamma, dbeta, coef);
    rc = finish_launch();
    if (rc) return rc;
    mbn_bwd_dx_kernel<T, V, VEC><<<dim3(elementwise_row_blocks(g, rows), g.col_tiles), block, 0, st>>>(
        dy, x, y, keep, rows, c, save_mean, save_invstd, coef, dx);
    return finish_launch();
}

// the (vec, aligned) variant: 4-wide vector loads when c % 4 == 0 and every row tensor is aligned to 4 elements; the
// same geometry (and so the same sums) with scalar loads otherwise
template <typename T, typename F>
int dispatch_vec(const MbnGeom& g, bool aligned, F&& f) {
    if (g.vec == 4) {
        if (aligned) return f(std::integral_constant<int, 4>(), std::true_type());
        return f(std::integral_constant<int, 4>(), std::false_type());
    }
    return f(std::integral_constant<int, 1>(), std::false_type());
}

bool mbn_args_ok(int rows, int c, const MbnGeom& g) {
    return rows >= 0 && c > 0 && g.col_tiles <= 65535;
}

// ---- the max-pooled form: statistics as the plain form, then one pass that keeps each cloud's column maxima ----------

// Workspace of the backward: coef[3][c], then gsel (b, c)
struct MaxBwdLayout {
    size_t coef, gsel, total;
};
MaxBwdLayout max_bwd_layout(int b, int c) {
    MaxBwdLayout L;
    L.coef = 0;
    L.gsel = align256(sizeof(float) * 3 * (size_t)c);
    L.total = L.gsel + align256(sizeof(float) * (size_t)b * c);
    return L;
}

template <typename T, int V, bool VEC>
int max_forward_launch(const MbnGeom& g, int b, int n, int c, const T* x, const unsigned char* keep, const float* gamma,
                       const float* beta, float eps, float momentum, const long long* nbt, float* running_mean,
                       float* running_var, T* out, int* argmax, float* save_mean, float* save_invstd, char* ws,
                       const MbnLayout& L, cudaStream_t st) {
    float* pa = reinterpret_cast<float*>(ws + L.pa);
    float* pb = reinterpret_cast<float*>(ws + L.pb);
    int* pc = reinterpret_cast<int*>(ws + L.cnt);
    const dim3 block(g.tx, g.ty);
    const int rows = b * n;
    mbn_stats_kernel<T, V, VEC><<<dim3((unsigned)g.chunks, g.col_tiles), block, 0, st>>>(x, keep, rows, c, pa, pb, pc);
    int rc = finish_launch();
    if (rc) return rc;
    mbn_finalize_kernel<<<ceil_div_u(c, 32), dim3(32, kMbnMergeWarps), 0, st>>>(pa, pb, pc, g.chunks, c, eps, momentum, nbt,
                                                                                 running_mean, running_var, save_mean, save_invstd);
    rc = finish_launch();
    if (rc) return rc;
    mbn_norm_relu_max_kernel<T, V, VEC><<<dim3((unsigned)b, g.col_tiles), block, 0, st>>>(
        x, keep, n, c, save_mean, save_invstd, gamma, beta, out, argmax);
    return finish_launch();
}

template <typename T, int V, bool VEC>
int max_backward_launch(const MbnGeom& g, int b, int n, int c, const T* dout, const T* x, const T* out, const int* argmax,
                        const unsigned char* keep, const float* gamma, const float* save_mean, const float* save_invstd,
                        T* dx, float* dgamma, float* dbeta, char* ws, const MaxBwdLayout& L, cudaStream_t st) {
    float* coef = reinterpret_cast<float*>(ws + L.coef);
    float* gsel = reinterpret_cast<float*>(ws + L.gsel);
    const int rows = b * n;
    mbn_max_bwd_finalize_kernel<T><<<ceil_div_u(c, 32), dim3(32, kMbnMergeWarps), 0, st>>>(
        dout, x, out, argmax, keep, b, n, c, gamma, save_mean, save_invstd, dgamma, dbeta, gsel, coef);
    int rc = finish_launch();
    if (rc) return rc;
    mbn_max_bwd_dx_kernel<T, V, VEC><<<dim3(elementwise_row_blocks(g, rows), g.col_tiles), dim3(g.tx, g.ty), 0, st>>>(
        x, keep, rows, n, c, argmax, gsel, save_mean, save_invstd, coef, dx);
    return finish_launch();
}

bool max_args_ok(int b, int n, int c) {
    return b >= 0 && n > 0 && c > 0 && (long long)b * n <= 0x7fffffffLL && b <= 0x7fffffff &&
           mbn_geom(b * n, c).col_tiles <= 65535;
}

template <typename T>
int forward_typed(int rows, int c, const void* x, const unsigned char* keep, const float* gamma, const float* beta, float eps,
                  float momentum, const long long* nbt, float* running_mean, float* running_var, void* y, float* save_mean,
                  float* save_invstd, char* ws, const MbnGeom& g, const MbnLayout& L, cudaStream_t st) {
    const bool aligned = aligned_to(x, 4 * sizeof(T)) && aligned_to(y, 4 * sizeof(T));
    return dispatch_vec<T>(g, aligned, [&](auto v, auto vec) {
        return forward_launch<T, decltype(v)::value, decltype(vec)::value>(
            g, rows, c, static_cast<const T*>(x), keep, gamma, beta, eps, momentum, nbt, running_mean, running_var,
            static_cast<T*>(y), save_mean, save_invstd, ws, L, st);
    });
}

template <typename T>
int backward_typed(int rows, int c, const void* dy, const void* x, const void* y, const unsigned char* keep, const float* gamma,
                   const float* save_mean, const float* save_invstd, void* dx, float* dgamma, float* dbeta, char* ws,
                   const MbnGeom& g, const MbnLayout& L, cudaStream_t st) {
    const bool aligned = aligned_to(dy, 4 * sizeof(T)) && aligned_to(x, 4 * sizeof(T)) && aligned_to(y, 4 * sizeof(T)) &&
                         aligned_to(dx, 4 * sizeof(T));
    return dispatch_vec<T>(g, aligned, [&](auto v, auto vec) {
        return backward_launch<T, decltype(v)::value, decltype(vec)::value>(
            g, rows, c, static_cast<const T*>(dy), static_cast<const T*>(x), static_cast<const T*>(y), keep, gamma, save_mean,
            save_invstd, static_cast<T*>(dx), dgamma, dbeta, ws, L, st);
    });
}

}  // namespace
}  // namespace pn2

extern "C" {

size_t pn2_masked_bn_workspace_bytes(int rows, int c) {
    using namespace pn2;
    if (rows <= 0 || c <= 0) return 0;
    const MbnGeom g = mbn_geom(rows, c);
    return mbn_layout(g, c).total;
}

int pn2_masked_bn_relu_forward_typed(int dtype, int rows, int c, const void* x, const unsigned char* keep, const float* gamma,
                                     const float* beta, float eps, float momentum, const long long* num_batches_tracked,
                                     float* running_mean, float* running_var, void* y, float* save_mean, float* save_invstd,
                                     void* workspace, size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    const MbnGeom g = mbn_geom(rows, c);
    if (!mbn_args_ok(rows, c, g)) return (int)cudaErrorInvalidValue;
    if (!x || !keep || !y || !save_mean || !save_invstd) return (int)cudaErrorInvalidValue;
    if (!running_mean != !running_var) return (int)cudaErrorInvalidValue;
    if (running_mean && momentum < 0.f && !num_batches_tracked) return (int)cudaErrorInvalidValue;
    if (rows == 0) return 0;
    const MbnLayout L = mbn_layout(g, c);
    if (!workspace || workspace_bytes < L.total || !aligned_to(workspace, 16)) return (int)cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    const cudaStream_t st = as_stream(stream);
    if (dtype == PN2_F32)
        return forward_typed<float>(rows, c, x, keep, gamma, beta, eps, momentum, num_batches_tracked, running_mean, running_var, y,
                                    save_mean, save_invstd, ws, g, L, st);
    if (dtype == PN2_BF16)
        return forward_typed<__nv_bfloat16>(rows, c, x, keep, gamma, beta, eps, momentum, num_batches_tracked, running_mean,
                                            running_var, y, save_mean, save_invstd, ws, g, L, st);
    return forward_typed<__half>(rows, c, x, keep, gamma, beta, eps, momentum, num_batches_tracked, running_mean, running_var, y,
                                 save_mean, save_invstd, ws, g, L, st);
}

int pn2_masked_bn_relu_backward_typed(int dtype, int rows, int c, const void* dy, const void* x, const void* y,
                                      const unsigned char* keep, const float* gamma, const float* save_mean,
                                      const float* save_invstd, void* dx, float* dgamma, float* dbeta, void* workspace,
                                      size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype)) return (int)cudaErrorInvalidValue;
    const MbnGeom g = mbn_geom(rows, c);
    if (!mbn_args_ok(rows, c, g)) return (int)cudaErrorInvalidValue;
    if (!dy || !x || !y || !keep || !save_mean || !save_invstd || !dx) return (int)cudaErrorInvalidValue;
    if (rows == 0) return 0;
    const MbnLayout L = mbn_layout(g, c);
    if (!workspace || workspace_bytes < L.total || !aligned_to(workspace, 16)) return (int)cudaErrorInvalidValue;
    char* ws = static_cast<char*>(workspace);
    const cudaStream_t st = as_stream(stream);
    if (dtype == PN2_F32)
        return backward_typed<float>(rows, c, dy, x, y, keep, gamma, save_mean, save_invstd, dx, dgamma, dbeta, ws, g, L, st);
    if (dtype == PN2_BF16)
        return backward_typed<__nv_bfloat16>(rows, c, dy, x, y, keep, gamma, save_mean, save_invstd, dx, dgamma, dbeta, ws, g, L,
                                             st);
    return backward_typed<__half>(rows, c, dy, x, y, keep, gamma, save_mean, save_invstd, dx, dgamma, dbeta, ws, g, L, st);
}

size_t pn2_masked_bn_relu_max_workspace_bytes(int b, int n, int c) {
    using namespace pn2;
    if (b <= 0 || n <= 0 || c <= 0 || (long long)b * n > 0x7fffffffLL) return 0;
    const size_t fwd = mbn_layout(mbn_geom(b * n, c), c).total, bwd = max_bwd_layout(b, c).total;
    return fwd > bwd ? fwd : bwd;
}

int pn2_masked_bn_relu_max_forward_typed(int dtype, int b, int n, int c, const void* x, const unsigned char* keep,
                                         const float* gamma, const float* beta, float eps, float momentum,
                                         const long long* num_batches_tracked, float* running_mean, float* running_var,
                                         void* out, int* argmax, float* save_mean, float* save_invstd, void* workspace,
                                         size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype) || !max_args_ok(b, n, c)) return (int)cudaErrorInvalidValue;
    if (!x || !keep || !out || !argmax || !save_mean || !save_invstd) return (int)cudaErrorInvalidValue;
    if (!running_mean != !running_var) return (int)cudaErrorInvalidValue;
    if (running_mean && momentum < 0.f && !num_batches_tracked) return (int)cudaErrorInvalidValue;
    if (b == 0) return 0;
    if (!workspace || workspace_bytes < pn2_masked_bn_relu_max_workspace_bytes(b, n, c) || !aligned_to(workspace, 16))
        return (int)cudaErrorInvalidValue;
    const MbnGeom g = mbn_geom(b * n, c);
    const MbnLayout L = mbn_layout(g, c);
    char* ws = static_cast<char*>(workspace);
    const cudaStream_t st = as_stream(stream);
    auto run = [&](auto t) {
        using T = decltype(t);
        // the statistics read x in the plain form's geometry; the vector loads need x aligned to 4 elements
        return dispatch_vec<T>(g, aligned_to(x, 4 * sizeof(T)), [&](auto v, auto vec) {
            return max_forward_launch<T, decltype(v)::value, decltype(vec)::value>(
                g, b, n, c, static_cast<const T*>(x), keep, gamma, beta, eps, momentum, num_batches_tracked, running_mean,
                running_var, static_cast<T*>(out), argmax, save_mean, save_invstd, ws, L, st);
        });
    };
    if (dtype == PN2_F32) return run(float());
    if (dtype == PN2_BF16) return run(__nv_bfloat16());
    return run(__half());
}

int pn2_masked_bn_relu_max_backward_typed(int dtype, int b, int n, int c, const void* dout, const void* x, const void* out,
                                          const int* argmax, const unsigned char* keep, const float* gamma,
                                          const float* save_mean, const float* save_invstd, void* dx, float* dgamma,
                                          float* dbeta, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace pn2;
    if (!valid_dtype(dtype) || !max_args_ok(b, n, c)) return (int)cudaErrorInvalidValue;
    if (!dout || !x || !out || !argmax || !keep || !save_mean || !save_invstd || !dx) return (int)cudaErrorInvalidValue;
    if (b == 0) return 0;
    if (!workspace || workspace_bytes < pn2_masked_bn_relu_max_workspace_bytes(b, n, c) || !aligned_to(workspace, 16))
        return (int)cudaErrorInvalidValue;
    const MbnGeom g = mbn_geom(b * n, c);
    const MaxBwdLayout L = max_bwd_layout(b, c);
    char* ws = static_cast<char*>(workspace);
    const cudaStream_t st = as_stream(stream);
    auto run = [&](auto t) {
        using T = decltype(t);
        const bool aligned = aligned_to(x, 4 * sizeof(T)) && aligned_to(dx, 4 * sizeof(T));
        return dispatch_vec<T>(g, aligned, [&](auto v, auto vec) {
            return max_backward_launch<T, decltype(v)::value, decltype(vec)::value>(
                g, b, n, c, static_cast<const T*>(dout), static_cast<const T*>(x), static_cast<const T*>(out), argmax, keep,
                gamma, save_mean, save_invstd, static_cast<T*>(dx), dgamma, dbeta, ws, L, st);
        });
    };
    if (dtype == PN2_F32) return run(float());
    if (dtype == PN2_BF16) return run(__nv_bfloat16());
    return run(__half());
}

}  // extern "C"
