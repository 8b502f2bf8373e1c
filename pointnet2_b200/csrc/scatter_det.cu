// scatter_det.cu — scatter-add without atomics, for sm_90a: an inverse index, then one warp per target row.  The
// deterministic gradients of three_interpolate (interpolate.cu) and of group_point / gather_point (group.cu); the
// entry point is inv_scatter_det (pn2_common.cuh).
#include "pn2_common.cuh"

namespace pn2 {

// The weighted sum serves three_interpolate's gradient, the unweighted one the group_point / gather_point gradients.
// A cloud has `ne` entries, each pointing at one of `nt` target rows:
//   weighted:   grad_points[b,i,:] = sum over e = 3j+t with idx[b,j,t] == i of grad_out[b,j,:] * weight[b,j,t]
//   unweighted: dst[b,i,:]         = sum over e         with idx[b,e]   == i of src[b,e,:]
// accumulated in ASCENDING e — the very order threeinterpolate_grad_cpu (tf_interpolate.cpp:131-153: j outer,
// t = 1,2,3 inner) and group_point_grad_cpu (query_ball_point.cpp:70-84: j, k ascending) add them, each product and
// sum rounded on its own — so the result is not only deterministic but bit-identical to the reference's CPU
// functions, and the output needs no zero-fill.
// Build: count entries per target (int atomics), exclusive scan per cloud, fill the CSR lists (order inside a list
// is arbitrary), then every warp sorts its own list (<= 256 entries: bitonic sort in registers).  Longer lists are
// queued: inv_long_kernel (weighted) and inv_long_seq_kernel (unweighted) serve them with an index-ordered scan of
// the cloud's entries.
// L (three_interpolate's gradient on a ragged unknown side): a cloud of length len has the real entries e < 3*len (the
// prefix, since e = 3j+t); the build and the long-list kernels stop there, so off[nt] = 3*len and the padding's idx is
// never counted.  lengths (b,) holds the lengths of the ne / 3 rows per cloud.  A template flag, so that the instances
// without lengths, which also serve the unweighted sums, compile to the code they always did.
constexpr int kInvThreads = 256;
constexpr int kInvSortCap = 256;

__device__ __forceinline__ int real_entries(const int* __restrict__ lengths, int cloud, int ne) {
    return 3 * cloud_length(lengths, cloud, ne / 3);
}

template <bool L>
__global__ void __launch_bounds__(kInvThreads)
inv_count_kernel(int ne, int nt, long long total, const int* __restrict__ idx, int* __restrict__ cnt,
                 const int* __restrict__ lengths) {
    for (long long e = (long long)blockIdx.x * kInvThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kInvThreads) {
        const long long cloud = e / ne;
        if (L && e - cloud * ne >= real_entries(lengths, (int)cloud, ne)) continue;
        atomicAdd(cnt + cloud * (nt + 1) + __ldg(idx + e), 1);
    }
}

// one CTA per cloud: off[i] = exclusive prefix of cnt[i], i = 0..nt (off[nt] = ne); cur[i] = off[i]
__global__ void __launch_bounds__(1024)
inv_scan_kernel(int nt, int* __restrict__ cnt_off, int* __restrict__ cur) {
    __shared__ int s_w[32];
    __shared__ int s_carry;
    int* __restrict__ c = cnt_off + (size_t)blockIdx.x * (nt + 1);
    int* __restrict__ cu = cur + (size_t)blockIdx.x * nt;
    const int tid = threadIdx.x;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base <= nt; base += 1024) {
        const int i = base + tid;
        const int v = (i < nt) ? c[i] : 0;
        const int excl = s_carry + cta_exclusive_sum_1024(v, s_w);
        if (i <= nt) c[i] = excl;
        if (i < nt) cu[i] = excl;
        __syncthreads();
        if (tid == 1023) s_carry = excl + v;
        __syncthreads();
    }
}

template <bool L>
__global__ void __launch_bounds__(kInvThreads)
inv_fill_kernel(int ne, int nt, long long total, const int* __restrict__ idx, int* __restrict__ cur, int* __restrict__ entries,
                const int* __restrict__ lengths) {
    for (long long e = (long long)blockIdx.x * kInvThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kInvThreads) {
        const long long cloud = e / ne;
        if (L && e - cloud * ne >= real_entries(lengths, (int)cloud, ne)) continue;
        const int pos = atomicAdd(cur + cloud * nt + __ldg(idx + e), 1);
        entries[cloud * ne + pos] = (int)(e - cloud * ne);
    }
}

// count + scan + fill of one cloud in ONE CTA, with the counters and cursors in shared memory (nt <= 16000): the
// inverse index of a layer costs one launch instead of two memsets and three kernels.
constexpr int kInvBuildMaxM = 16000;
template <bool L>
__global__ void __launch_bounds__(1024)
inv_build_kernel(int ne, int nt, const int* __restrict__ idx, int* __restrict__ off, int* __restrict__ entries,
                 int* __restrict__ long_queue, const int* __restrict__ lengths) {
    extern __shared__ int s_c[];  // [nt + 1]: counts -> exclusive offsets (kept as the fill cursors)
    __shared__ int s_w[32];
    __shared__ int s_carry;
    const int tid = threadIdx.x;
    const long long cloud = blockIdx.x;
    const int* __restrict__ cidx = idx + cloud * ne;
    const int ne_c = L ? real_entries(lengths, (int)cloud, ne) : ne;  // entries of this cloud; ne stays the stride
    for (int i = tid; i <= nt; i += 1024) s_c[i] = 0;
    if (tid == 0) {
        s_carry = 0;
        if (cloud == 0) long_queue[0] = 0;
    }
    __syncthreads();
    for (int e = tid; e < ne_c; e += 1024) atomicAdd(&s_c[__ldg(cidx + e)], 1);
    __syncthreads();
    int* __restrict__ o = off + cloud * (nt + 1);
    for (int base = 0; base <= nt; base += 1024) {
        const int i = base + tid;
        const int v = (i < nt) ? s_c[i] : 0;
        const int excl = s_carry + cta_exclusive_sum_1024(v, s_w);
        if (i <= nt) {
            o[i] = excl;
            s_c[i] = excl;
        }
        __syncthreads();
        if (tid == 1023) s_carry = excl + v;
        __syncthreads();
    }
    int* __restrict__ ent = entries + cloud * ne;
    for (int e = tid; e < ne_c; e += 1024) ent[atomicAdd(&s_c[__ldg(cidx + e)], 1)] = e;
}

// one warp per target row (b, i); lanes over channels (float4 when VEC).  Lists longer than kInvSortCap are
// queued for the long-list kernel.
// WEIGHTED: entry e = 3j+t adds grad_out row j times weight[e] (three_interpolate, n = unknown points, ne = 3n);
// otherwise entry e adds grad_out row e as it is (n = ne = entries).  m = targets.
// T: element type of grad_out and grad_points (upcast on load, float32 sums, rounded once on the store): float, or
// unsigned short for both 2-byte formats with f16 choosing float16 / bfloat16 at run time (one instance for the two)
template <bool VEC, bool WEIGHTED, typename T>
__global__ void __launch_bounds__(kInvThreads)
inv_gather_kernel(int n, int c, int m, long long warps_total, const T* __restrict__ grad_out,
                  const float* __restrict__ weight, const int* __restrict__ off, const int* __restrict__ entries,
                  T* __restrict__ grad_points, int* __restrict__ long_queue, int f16) {
    __shared__ int s_e[kInvThreads / 32][kInvSortCap];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const long long gw = ((long long)blockIdx.x * kInvThreads + threadIdx.x) >> 5;
    if (gw >= warps_total) return;
    const long long cloud = gw / m;
    const int i = (int)(gw - cloud * m);
    const int ne = WEIGHTED ? 3 * n : n;
    const int* __restrict__ o = off + cloud * (m + 1);
    const int beg = o[i], len = o[i + 1] - beg;
    if (len > kInvSortCap) {  // warp-uniform
        if (lane == 0) long_queue[1 + atomicAdd(long_queue, 1)] = (int)gw;  // the order of the queue does not matter
        return;
    }
    {
        int key[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) key[q] = (32 * q + lane < len) ? __ldg(entries + cloud * ne + beg + 32 * q + lane) : 0x7fffffff;
        const int nreg = (len + 31) >> 5;
        if (nreg <= 1) bitonic_sort_keys<1, 8>(key, lane);
        else if (nreg == 2) bitonic_sort_keys<2, 8>(key, lane);
        else if (nreg <= 4) bitonic_sort_keys<4, 8>(key, lane);
        else bitonic_sort_keys<8, 8>(key, lane);
#pragma unroll
        for (int q = 0; q < 8; ++q)
            if (32 * q + lane < len) s_e[wib][32 * q + lane] = key[q];
        __syncwarp();
    }
    const T* __restrict__ go = grad_out + (size_t)cloud * n * c;
    const float* __restrict__ wt = WEIGHTED ? weight + (size_t)cloud * ne : nullptr;
    T* __restrict__ gp = grad_points + ((size_t)cloud * m + i) * c;
    constexpr int W = VEC ? 4 : 1;
    for (int l0 = 0; l0 < c; l0 += 32 * W) {  // 128 (VEC) or 32 channels per pass
        const int l = l0 + lane * W;
        if (l >= c) continue;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        // H entries at a time: their raw rows are all loaded before the first is upcast and added (in ascending order);
        // an upcast next to each load made the warp wait for the loads one by one
        constexpr int H = 4;
        for (int s0 = 0; s0 < len; s0 += H) {
            typename Pack4<T>::type gv[H];
            T gs[H];
            float w[H];
#pragma unroll
            for (int u = 0; u < H; ++u) {
                w[u] = 0.f;
                if (s0 + u < len) {
                    const int e = s_e[wib][s0 + u];
                    if (WEIGHTED) w[u] = __ldg(wt + e);
                    const T* __restrict__ src = go + (size_t)(WEIGHTED ? e / 3 : e) * c + l;
                    if (VEC) gv[u] = __ldg(reinterpret_cast<const typename Pack4<T>::type*>(src));
                    else gs[u] = __ldg(src);
                }
            }
#pragma unroll
            for (int u = 0; u < H; ++u) {
                if (s0 + u < len) {
                    if (VEC) {
                        const float4 g = unpack4_of(gv[u], f16);
                        a0 = __fadd_rn(a0, WEIGHTED ? __fmul_rn(g.x, w[u]) : g.x);
                        a1 = __fadd_rn(a1, WEIGHTED ? __fmul_rn(g.y, w[u]) : g.y);
                        a2 = __fadd_rn(a2, WEIGHTED ? __fmul_rn(g.z, w[u]) : g.z);
                        a3 = __fadd_rn(a3, WEIGHTED ? __fmul_rn(g.w, w[u]) : g.w);
                    } else {
                        const float g = f32_of(gs[u], f16);
                        a0 = __fadd_rn(a0, WEIGHTED ? __fmul_rn(g, w[u]) : g);
                    }
                }
            }
        }
        if (VEC) *reinterpret_cast<typename Pack4<T>::type*>(gp + l) = pack4_of(make_float4(a0, a1, a2, a3), T(), f16);
        else gp[l] = of_f32<T>(a0, f16);
    }
}

// Long lists of the unweighted sum, in plain ascending entry order like the short ones (the group_point and
// gather_point gradients are bit-identical to the reference's loop at any list length; at cls_msg layer 2 up to 5 %
// of the entries sit in lists longer than 256).  One CTA per list: it scans the cloud's entries in order, kSeqScan per
// thread and step, compacts the ones that point at i into shared memory in that order (ballot, then a popc prefix
// over the (step, warp) slots), and when the buffer is full every thread adds the buffered rows to its own channels
// in one chain.
constexpr int kSeqScan = 8;
constexpr int kSeqBuf = 2 * kSeqScan * kInvThreads;  // room for one more step whenever a step starts
// (the bound of 1 CTA per SM lifts the register budget: without it ptxas kept the VEC instances at 64 and spilled)
template <bool VEC, typename T>
__global__ void __launch_bounds__(kInvThreads, 1)
inv_long_seq_kernel(int ne, int c, int m, const T* __restrict__ grad_out, const int* __restrict__ idx,
                    const int* __restrict__ long_queue, T* __restrict__ grad_points, int f16) {
    constexpr int NW = kInvThreads / 32;
    constexpr int W = VEC ? 4 : 1;
    constexpr int H = sizeof(T) == 4 ? 4 : 8;  // rows in flight per thread, as in inv_long_kernel
    __shared__ int s_list[kSeqBuf];
    __shared__ int s_cnt[kSeqScan * NW];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned below = (1u << lane) - 1u;
    const int nq = long_queue[0];
    for (int q = blockIdx.x; q < nq; q += gridDim.x) {
        const long long gw = long_queue[1 + q];
        const long long cloud = gw / m;
        const int i = (int)(gw - cloud * m);
        const T* __restrict__ go = grad_out + (size_t)cloud * ne * c;
        const int* __restrict__ cidx = idx + cloud * ne;
        T* __restrict__ gp = grad_points + ((size_t)cloud * m + i) * c;
        for (int l0 = 0; l0 < c; l0 += kInvThreads * W) {
            const int l = l0 + tid * W;
            const bool act = l < c;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            long long e0 = 0;
            while (e0 < ne) {
                int cnt = 0;  // CTA-uniform
                while (e0 < ne && cnt <= kSeqBuf - kSeqScan * kInvThreads) {
                    int v[kSeqScan];
#pragma unroll
                    for (int u = 0; u < kSeqScan; ++u) {
                        const long long e = e0 + u * kInvThreads + tid;
                        v[u] = e < ne ? __ldg(cidx + e) : -1;
                    }
                    unsigned hits = 0, rank[kSeqScan];  // rank: matches of this step's slot u in the lanes below
#pragma unroll
                    for (int u = 0; u < kSeqScan; ++u) {
                        const unsigned bal = __ballot_sync(kFullMask, v[u] == i);
                        hits |= (v[u] == i ? 1u : 0u) << u;
                        rank[u] = __popc(bal & below);
                        if (lane == 0) s_cnt[u * NW + warp] = __popc(bal);
                    }
                    __syncthreads();
#pragma unroll
                    for (int u = 0; u < kSeqScan; ++u) {
                        int pos = cnt;
#pragma unroll
                        for (int w = 0; w < NW; ++w) {
                            const int k = s_cnt[u * NW + w];
                            pos += w < warp ? k : 0;
                            cnt += k;
                        }
                        if (hits >> u & 1u) s_list[pos + rank[u]] = (int)(e0 + u * kInvThreads + tid);
                    }
                    e0 += kSeqScan * kInvThreads;
                    __syncthreads();
                }
                if (act) {
                    for (int s0 = 0; s0 < cnt; s0 += H) {
                        typename Pack4<T>::type gv[H];
                        T gs[H];
#pragma unroll
                        for (int u = 0; u < H; ++u) {
                            if (s0 + u < cnt) {
                                const T* __restrict__ src = go + (size_t)s_list[s0 + u] * c + l;
                                if (VEC) gv[u] = __ldg(reinterpret_cast<const typename Pack4<T>::type*>(src));
                                else gs[u] = __ldg(src);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < H; ++u) {
                            if (s0 + u < cnt) {
                                if (VEC) {
                                    const float4 g = unpack4_of(gv[u], f16);
                                    a0 = __fadd_rn(a0, g.x);
                                    a1 = __fadd_rn(a1, g.y);
                                    a2 = __fadd_rn(a2, g.z);
                                    a3 = __fadd_rn(a3, g.w);
                                } else {
                                    a0 = __fadd_rn(a0, f32_of(gs[u], f16));
                                }
                            }
                        }
                    }
                }
                __syncthreads();  // s_list is refilled
            }
            if (act) {
                if (VEC) *reinterpret_cast<typename Pack4<T>::type*>(gp + l) = pack4_of(make_float4(a0, a1, a2, a3), T(), f16);
                else gp[l] = of_f32<T>(a0, f16);
            }
        }
    }
}

// Long lists (most unknown points share a neighbour: coincident points, m < 3, ...): one CTA per list.  The
// cloud's 3n entries are cut into 8 consecutive pieces, one per warp; each warp walks its piece in index order
// (coalesced index loads + ballot), adds the entries that point at i in that order, and the 8 partial sums are
// combined in piece order — a fixed association, hence deterministic (it differs from one long sequential sum
// only in rounding; short lists, the normal case, are bit-identical to the reference's loop).
// L: the cloud's 3*len real entries are cut into the 8 pieces, as the call on the truncated cloud cuts them.
template <bool VEC, typename T, bool L = false>
__global__ void __launch_bounds__(kInvThreads)
inv_long_kernel(int n, int c, int m, const T* __restrict__ grad_out, const int* __restrict__ idx,
                const float* __restrict__ weight, const int* __restrict__ long_queue, T* __restrict__ grad_points, int f16,
                const int* __restrict__ lengths) {
    constexpr int NW = kInvThreads / 32;
    constexpr int W = VEC ? 4 : 1;
    __shared__ float s_part[NW][32 * W];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nq = long_queue[0];
    const int n3 = 3 * n;
    const int piece = (n3 + NW - 1) / NW;
    for (int q = blockIdx.x; q < nq; q += gridDim.x) {
        const long long gw = long_queue[1 + q];
        const long long cloud = gw / m;
        const int i = (int)(gw - cloud * m);
        const T* __restrict__ go = grad_out + (size_t)cloud * n * c;
        const float* __restrict__ wt = weight + (size_t)cloud * n3;
        const int* __restrict__ cidx = idx + cloud * n3;
        T* __restrict__ gp = grad_points + ((size_t)cloud * m + i) * c;
        const int n3_c = L ? real_entries(lengths, (int)cloud, n3) : n3;
        const int piece_c = L ? (n3_c + NW - 1) / NW : piece;
        const int e_lo = warp * piece_c, e_hi = min(n3_c, e_lo + piece_c);
        for (int l0 = 0; l0 < c; l0 += 32 * W) {
            const int l = l0 + lane * W;
            const bool act = l < c;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            for (int base = e_lo; base < e_hi; base += 32) {
                const int e = base + lane;
                unsigned hit = __ballot_sync(kFullMask, e < e_hi && __ldg(cidx + e) == i);
                // up to H matching entries at a time: their rows are loaded together, then added in order.  Raw vectors: the
                // 2-byte types are upcast only when added, so all H loads are in flight first (an upcast next to each load
                // made the 16-bit kernel wait for every load in turn: 2x the float time); their smaller vectors leave the
                // registers for 8 rows in flight (4: still 6 % behind float at cfg4 FP8192 <- 1024)
                constexpr int H = sizeof(T) == 4 ? 4 : 8;
                while (hit) {
                    int ee[H];
                    float w[H];
                    typename Pack4<T>::type gv[H];
                    T gs[H];
#pragma unroll
                    for (int u = 0; u < H; ++u) {
                        ee[u] = -1;
                        if (hit) {
                            ee[u] = base + __ffs(hit) - 1;
                            hit &= hit - 1;
                        }
                    }
#pragma unroll
                    for (int u = 0; u < H; ++u) {
                        w[u] = 0.f;
                        if (ee[u] >= 0 && act) {
                            w[u] = __ldg(wt + ee[u]);
                            const T* __restrict__ src = go + (size_t)(ee[u] / 3) * c + l;
                            if (VEC) gv[u] = __ldg(reinterpret_cast<const typename Pack4<T>::type*>(src));
                            else gs[u] = __ldg(src);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < H; ++u) {
                        if (ee[u] >= 0 && act) {
                            const float4 g = VEC ? unpack4_of(gv[u], f16) : make_float4(f32_of(gs[u], f16), 0.f, 0.f, 0.f);
                            a0 = __fadd_rn(a0, __fmul_rn(g.x, w[u]));
                            if (VEC) {
                                a1 = __fadd_rn(a1, __fmul_rn(g.y, w[u]));
                                a2 = __fadd_rn(a2, __fmul_rn(g.z, w[u]));
                                a3 = __fadd_rn(a3, __fmul_rn(g.w, w[u]));
                            }
                        }
                    }
                }
            }
            s_part[warp][lane * W] = a0;
            if (VEC) {
                s_part[warp][lane * W + 1] = a1;
                s_part[warp][lane * W + 2] = a2;
                s_part[warp][lane * W + 3] = a3;
            }
            __syncthreads();
            if (warp == 0 && act) {
#pragma unroll
                for (int u = 0; u < W; ++u) {
                    float t = s_part[0][lane * W + u];
#pragma unroll
                    for (int p = 1; p < NW; ++p) t = __fadd_rn(t, s_part[p][lane * W + u]);
                    gp[l + u] = of_f32<T>(t, f16);
                }
            }
            __syncthreads();
        }
    }
}

size_t inv_workspace_bytes(int b, long long ne, int nt) {
    // offsets (b, nt+1) + cursors (b, nt) + entries (b, ne) + queue of long lists (1 + b * (ne / (cap+1) + 1)), ints
    const size_t longs = (size_t)b * ((size_t)ne / (kInvSortCap + 1) + 1);
    return sizeof(int) * ((size_t)b * (nt + 1) + (size_t)b * nt + (size_t)b * (size_t)ne + 1 + longs);
}

// The inverse index of the b clouds' entries over nt targets is built in `workspace`, then the sums are taken.
template <bool WEIGHTED, typename T>
int inv_scatter_det(int b, int n, int ne, int c, int nt, const T* grad_out, const int* idx, const float* weight,
                           const int* lengths, T* grad_points, void* workspace, int f16, cudaStream_t st) {
    const long long warps = (long long)b * nt;
    const unsigned long long blocks = ((unsigned long long)warps * 32 + kInvThreads - 1) / kInvThreads;
    if (blocks > 0x7fffffffull) return (int)cudaErrorInvalidValue;
    int* off = static_cast<int*>(workspace);
    int* cur = off + (size_t)b * (nt + 1);
    int* entries = cur + (size_t)b * nt;
    int* long_queue = entries + (size_t)b * (size_t)ne;  // [0] = count, then (cloud * nt + i) of every list > kInvSortCap
    int launches = 2;
    if (nt <= kInvBuildMaxM) {
        static AttrOnce once[2];  // [ragged]
        auto kern = lengths ? inv_build_kernel<true> : inv_build_kernel<false>;
        const cudaError_t e = ensure_attrs(once[lengths ? 1 : 0], kern, sizeof(int) * (kInvBuildMaxM + 1), false);
        if (e != cudaSuccess) return (int)e;
        kern<<<b, 1024, sizeof(int) * (size_t)(nt + 1), st>>>(ne, nt, idx, off, entries, long_queue, lengths);
        launches += 1;
    } else {
        cudaError_t e = cudaMemsetAsync(off, 0, sizeof(int) * (size_t)b * (nt + 1), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(long_queue, 0, sizeof(int), st);
        if (e != cudaSuccess) return (int)e;
        const long long total = (long long)b * ne;
        const unsigned g1 = grid_for((unsigned long long)total, kInvThreads);
        if (lengths) inv_count_kernel<true><<<g1, kInvThreads, 0, st>>>(ne, nt, total, idx, off, lengths);
        else inv_count_kernel<false><<<g1, kInvThreads, 0, st>>>(ne, nt, total, idx, off, nullptr);
        inv_scan_kernel<<<b, 1024, 0, st>>>(nt, off, cur);
        if (lengths) inv_fill_kernel<true><<<g1, kInvThreads, 0, st>>>(ne, nt, total, idx, cur, entries, lengths);
        else inv_fill_kernel<false><<<g1, kInvThreads, 0, st>>>(ne, nt, total, idx, cur, entries, nullptr);
        launches += 3;
    }
    // long lists: a fixed grid walks the queue (usually empty: the CTAs read one word and leave)
    const unsigned long_grid = (unsigned)num_sms() * 2u;
    const bool vec = c % 4 == 0 && aligned_to(grad_out, 4 * sizeof(T)) && aligned_to(grad_points, 4 * sizeof(T));
#define PN2_INV_SUMS(VEC)                                                                                                     \
    inv_gather_kernel<VEC, WEIGHTED, T><<<(unsigned)blocks, kInvThreads, 0, st>>>(n, c, nt, warps, grad_out, weight, off, entries, \
                                                                                  grad_points, long_queue, f16);            \
    if constexpr (WEIGHTED) {                                                                                                 \
        if (lengths)                                                                                                          \
            inv_long_kernel<VEC, T, true><<<long_grid, kInvThreads, 0, st>>>(n, c, nt, grad_out, idx, weight, long_queue,       \
                                                                             grad_points, f16, lengths);                      \
        else                                                                                                                  \
            inv_long_kernel<VEC, T, false><<<long_grid, kInvThreads, 0, st>>>(n, c, nt, grad_out, idx, weight, long_queue,      \
                                                                              grad_points, f16, nullptr);                     \
    } else                                                                                                                    \
        inv_long_seq_kernel<VEC, T><<<long_grid, kInvThreads, 0, st>>>(ne, c, nt, grad_out, idx, long_queue, grad_points, f16)
    if (vec) {
        PN2_INV_SUMS(true);
    } else {
        PN2_INV_SUMS(false);
    }
#undef PN2_INV_SUMS
    count_launch(launches - 1);
    return finish_launch();
}

template int inv_scatter_det<true, float>(int, int, int, int, int, const float*, const int*, const float*, const int*, float*, void*,
                                          int, cudaStream_t);
template int inv_scatter_det<true, unsigned short>(int, int, int, int, int, const unsigned short*, const int*, const float*,
                                                   const int*, unsigned short*, void*, int, cudaStream_t);
template int inv_scatter_det<false, float>(int, int, int, int, int, const float*, const int*, const float*, const int*, float*, void*,
                                           int, cudaStream_t);
template int inv_scatter_det<false, unsigned short>(int, int, int, int, int, const unsigned short*, const int*, const float*,
                                                    const int*, unsigned short*, void*, int, cudaStream_t);

}  // namespace pn2
