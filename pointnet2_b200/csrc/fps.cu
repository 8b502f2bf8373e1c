// fps.cu — farthest point sampling for sm_90a.
//
// Replaces farthestpointsamplingKernel / farthestpointsamplingLauncher
// (reference tf_ops/sampling/tf_sampling_g.cu:105-170, :203-205).
//
// Selection rule (bit-exact with the reference): start at index 0; every step the point whose
// running minimum squared distance to the picked set is largest wins, ties resolved by
// (k mod 512 ascending, then k ascending) — the order the reference's 512-thread strided scan
// and lower-slot-wins tree produce.  Distances use the reference's contraction pattern
// (pn2::d2_fma_pattern).
//
// Design (not a translation):
//   * the cloud's coordinates AND the running-minimum array live in REGISTERS (P points per
//     thread); nothing is re-read from or written to global memory inside the M-step chain
//     (the reference keeps the running minimum in global memory and re-reads points >= 3072
//     from global every step, and burns 10 __syncthreads per step);
//   * one step = P fused distance/min/compare updates per thread, two redux.sync warp
//     reductions on a 64-bit (value, tie-break) key, one shared-memory hop and ONE barrier;
//   * clouds too large for one CTA's register file are spread over a thread-block cluster
//     (up to 16 CTAs); the per-step cross-CTA argmax is exchanged through distributed shared
//     memory with st.async + mbarrier transaction counts (no cluster-wide barrier per step);
//   * anything larger still falls back to a global-scratch kernel (the reference's layout).
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <mutex>

#include "pn2_common.cuh"

namespace pn2 {

// ---- 64-bit selection key --------------------------------------------------------------------
// hi = float bits of the running minimum (non-negative, so unsigned order == float order)
// lo = ~tb(k), tb(k) = (k mod 512) << 23 | (k / 512): larger lo == earlier in the tie-break order.
__device__ __forceinline__ unsigned tb_encode(unsigned k) { return ((k & 511u) << 23) | (k >> 9); }
__device__ __forceinline__ unsigned tb_decode(unsigned tb) { return ((tb & 0x7fffffu) << 9) | (tb >> 23); }

// ---- PTX wrappers for the cluster exchange -----------------------------------------------------
__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned cluster_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned cluster_nctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned mapa_shared(unsigned addr, unsigned rank) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void mbar_init(unsigned addr, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(addr), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init_cluster() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned addr, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_parity_cluster(unsigned addr, unsigned parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "PN2_WAIT:\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra PN2_DONE;\n\t"
        "bra PN2_WAIT;\n\t"
        "PN2_DONE:\n\t"
        "}" ::"r"(addr),
        "r"(parity)
        : "memory");
}
// Stores into a peer CTA's shared memory that also complete their byte count on the peer's mbarrier
// (SASS: STAS.128 / STAS).
__device__ __forceinline__ void st_async_v4(unsigned remote_addr, unsigned a, unsigned b, unsigned c, unsigned d,
                                            unsigned remote_mbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(remote_addr),
                 "r"(a), "r"(b), "r"(c), "r"(d), "r"(remote_mbar)
                 : "memory");
}
__device__ __forceinline__ void st_async_u32(unsigned remote_addr, unsigned v, unsigned remote_mbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(remote_addr), "r"(v),
                 "r"(remote_mbar)
                 : "memory");
}

// ---- per-thread step: update P register-resident points against the last pick ------------------
// DD = number of distinct reference slots (k mod 512) one thread's points fall into (ScanOrder::DD).  The
// scan visits the points in tie-break order (slot ascending, then k ascending): for each slot residue
// r = j mod DD in turn, j ascending — so the strict '>' keeps the reference's winner.
template <int P, int DD = 1, int PT = P>
__device__ __forceinline__ void fps_step(const float (&px)[P], const float (&py)[P], const float (&pz)[P],
                                         float (&td)[PT], float x1, float y1, float z1, float& best, int& bj) {
    best = -1.0f;
    bj = 0;
#pragma unroll
    for (int r = 0; r < DD; ++r) {
#pragma unroll
        for (int j = r; j < P; j += DD) {
            const float d = d2_fma_pattern(px[j], py[j], pz[j], x1, y1, z1);
            const float d2 = fminf(d, td[j]);  // padding slots carry td = -1 and can never win
            td[j] = d2;
            if (d2 > best) {
                best = d2;
                bj = j;
            }
        }
    }
}

// PDL hook used by the fused set-abstraction layer (sa_fused.cu): lets the dependent grid launch
// as soon as every CTA of this grid has got here (SASS: PREEXIT).  A no-op for ordinary launches.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Packed pair update: the running minima of the H register-resident pairs (X, Y, Z)[h] = points 2h, 2h + 1 against
// the last pick (x1, y1, z1), d2_fma_pattern on both halves.
template <int H, int P>
__device__ __forceinline__ void pair_update(const unsigned long long (&X)[H], const unsigned long long (&Y)[H],
                                            const unsigned long long (&Z)[H], float (&td)[P], float x1, float y1, float z1) {
    const unsigned long long X1 = f2_pack(x1, x1), Y1 = f2_pack(y1, y1), Z1 = f2_pack(z1, z1);
#pragma unroll
    for (int h = 0; h < H; ++h) {
        const unsigned long long dx = f2_sub(X[h], X1), dy = f2_sub(Y[h], Y1), dz = f2_sub(Z[h], Z1);
        const unsigned long long d = f2_fma(dz, dz, f2_fma(dx, dx, f2_mul(dy, dy)));  // d2_fma_pattern on both halves
        float d0, d1;
        f2_unpack(d, d0, d1);
        td[2 * h] = fminf(d0, td[2 * h]);
        td[2 * h + 1] = fminf(d1, td[2 * h + 1]);
    }
}

// ---- streamed points of the cluster kernels: shared-memory float4 groups [(g*3 + c)*T + t], .x..w = four consecutive
// points of thread t.  Groups [G0, G1) hold the thread's points J0 + 4*(g - G0) + u, whose running minima are in td.
template <int G0, int G1, int J0, int T, int P>
__device__ __forceinline__ void stream_update_packed(const float4* __restrict__ s4, int tid, float (&td)[P], float x1,
                                                     float y1, float z1) {
    const unsigned long long X1 = f2_pack(x1, x1), Y1 = f2_pack(y1, y1), Z1 = f2_pack(z1, z1);
#pragma unroll
    for (int g = G0; g < G1; ++g) {
        const float4 X = s4[(g * 3 + 0) * T + tid], Y = s4[(g * 3 + 1) * T + tid], Z = s4[(g * 3 + 2) * T + tid];
        const unsigned long long xa = f2_pack(X.x, X.y), xb = f2_pack(X.z, X.w), ya = f2_pack(Y.x, Y.y),
                                 yb = f2_pack(Y.z, Y.w), za = f2_pack(Z.x, Z.y), zb = f2_pack(Z.z, Z.w);
        const unsigned long long dxa = f2_sub(xa, X1), dya = f2_sub(ya, Y1), dza = f2_sub(za, Z1);
        const unsigned long long dxb = f2_sub(xb, X1), dyb = f2_sub(yb, Y1), dzb = f2_sub(zb, Z1);
        const unsigned long long da = f2_fma(dza, dza, f2_fma(dxa, dxa, f2_mul(dya, dya)));
        const unsigned long long db = f2_fma(dzb, dzb, f2_fma(dxb, dxb, f2_mul(dyb, dyb)));
        float d0, d1, d2, d3;
        f2_unpack(da, d0, d1);
        f2_unpack(db, d2, d3);
        const int j = J0 + 4 * (g - G0);
        td[j + 0] = fminf(d0, td[j + 0]);
        td[j + 1] = fminf(d1, td[j + 1]);
        td[j + 2] = fminf(d2, td[j + 2]);
        td[j + 3] = fminf(d3, td[j + 3]);
    }
}
// The plain form continues fps_step's scan (best, bj) over the streamed points, which follow the register-resident ones
// in tie-break order.
template <int G0, int G1, int J0, int T, int P>
__device__ __forceinline__ void stream_update(const float4* __restrict__ s4, int tid, float (&td)[P], float x1, float y1,
                                              float z1, float& best, int& bj) {
#pragma unroll
    for (int g = G0; g < G1; ++g) {
        const float4 X = s4[(g * 3 + 0) * T + tid], Y = s4[(g * 3 + 1) * T + tid], Z = s4[(g * 3 + 2) * T + tid];
        const float xs[4] = {X.x, X.y, X.z, X.w}, ys[4] = {Y.x, Y.y, Y.z, Y.w}, zs[4] = {Z.x, Z.y, Z.z, Z.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int j = J0 + 4 * (g - G0) + u;
            const float d = d2_fma_pattern(xs[u], ys[u], zs[u], x1, y1, z1);
            const float d2 = fminf(d, td[j]);
            td[j] = d2;
            if (d2 > best) {
                best = d2;
                bj = j;
            }
        }
    }
}

// Pick `it` of a single-CTA chain: its index, and its coordinates when the caller asked for them.  The cluster kernels
// and the global fallback store the index first and keep their own stores: the other order compiles to other code.
__device__ __forceinline__ void write_pick(int* __restrict__ out, float* __restrict__ oxyz, int it, int idx, float x,
                                          float y, float z) {
    if (oxyz) {
        oxyz[3 * it + 0] = x;
        oxyz[3 * it + 1] = y;
        oxyz[3 * it + 2] = z;
    }
    out[it] = idx;
}

// Lexicographic (max hi, then min lo) over the warp; every lane gets the result.
__device__ __forceinline__ void warp_max_min_pair(unsigned& hi, unsigned& lo) {
    const unsigned mh = __reduce_max_sync(kFullMask, hi);
    const unsigned ml = __reduce_min_sync(kFullMask, hi == mh ? lo : 0xffffffffu);
    hi = mh;
    lo = ml;
}

// ---- a thread's points in SCAN order --------------------------------------------------------------
// Register slot e of thread t holds point k = t + j(e)*T, with j(e) running through the thread's points in the
// reference's tie-break order (slot k mod 512 ascending, then k ascending; see fps_step).  The tie-break word of
// that point splits into the thread's own part tb_encode(t) and a compile-time constant tbj(e) with disjoint bits.
// D = number of distinct reference slots (k mod 512) of thread t's points k = t + j*T: for T < 512 they cycle with
// period D = 512/T, and a thread with P < D points sees DD = P of them.
template <int P, int T>
struct ScanOrder {
    static constexpr int D = (T >= 512) ? 1 : 512 / T;
    static constexpr int DD = (D < P) ? D : P;
    static constexpr int Q = P / DD;                 // points per slot residue
    static constexpr int GS = (Q >= 4) ? 4 : Q;      // scan-order neighbours per search group
    __host__ __device__ static constexpr int j_of(int e) { return (e % Q) * DD + e / Q; }
    __host__ __device__ static constexpr unsigned tbj(int e) {
        return ((((unsigned)(j_of(e) * T)) & 511u) << 23) | (((unsigned)(j_of(e) * T)) >> 9);
    }
    // tbj(GS*a + u) == tbj(GS*a) | tbj(u) for every group a and in-group position u (checked at compile time)
    __host__ __device__ static constexpr bool separable() {
        for (int a = 0; a < P / GS; ++a)
            for (int u = 0; u < GS; ++u)
                if (tbj(GS * a + u) != (tbj(GS * a) | tbj(u)) || (u && (tbj(GS * a) & tbj(u)))) return false;
        return true;
    }
};

// Value-only maximum (floored at 0) of P running minima held in ascending tie-break order, and the position of the
// FIRST leaf that attains it: first group of four whose maximum equals the maximum, then the first equal leaf inside
// it — what a strict '>' scan from -1 over the same order selects whenever the maximum is >= 0.  Padding leaves
// carry -1 and never equal it; if no leaf does (a thread without points) the position is P-1 and the caller's
// tie-break part masks the key.
template <int P>
__device__ __forceinline__ void value_argmax_first(const float (&td)[P], float& mx, int& pos) {
    static_assert(P % 4 == 0, "groups of four");
    constexpr int G = P / 4;
    float g[G];
#pragma unroll
    for (int a = 0; a < G; ++a) g[a] = fmaxf(fmaxf(fmaxf(td[4 * a], td[4 * a + 1]), td[4 * a + 2]), td[4 * a + 3]);
    float m = 0.0f;
#pragma unroll
    for (int a = 0; a < G; ++a) m = fmaxf(m, g[a]);
    float s0 = td[4 * (G - 1)], s1 = td[4 * (G - 1) + 1], s2 = td[4 * (G - 1) + 2];
    int pg = 4 * (G - 1);
#pragma unroll
    for (int a = G - 2; a >= 0; --a) {
        const bool q = (g[a] == m);
        s0 = q ? td[4 * a] : s0;
        s1 = q ? td[4 * a + 1] : s1;
        s2 = q ? td[4 * a + 2] : s2;
        pg = q ? 4 * a : pg;
    }
    int pu = 3;
    pu = (s2 == m) ? 2 : pu;
    pu = (s1 == m) ? 1 : pu;
    pu = (s0 == m) ? 0 : pu;
    mx = m;
    pos = pg | pu;
}

// ---- the M-step chain of fps_cta_kernel, restructured around what binds it ---------------------------
// The plain chain (fps_step) spends 10 instructions per point and step: 6 on the FMA pipe (3 FADD, FMUL, 2 FFMA)
// and 4 on the half-rate ALU pipe (FMNMX, FSETP, FSEL, SEL: the running (value, position) maximum).  With two
// warps per scheduler the ALU pipe and the issue slot are both ~full during the update (SASS: 213 instructions per
// warp and step, 83 of them ALU).  This form keeps the arithmetic bit-identical and cuts both:
//   * the 6 distance operations run as packed FP32x2 (two scan-order neighbours per instruction);
//   * the update tracks VALUES only — groups of GS scan-order neighbours are reduced with 3-input maxima
//     (FMNMX3) — and the position of the first maximum is recovered afterwards: first group whose maximum equals
//     the thread's maximum, then first equal leaf inside it.  "First in scan order among equals" is exactly
//     what the strict '>' scan of fps_step selects, so the key is the same word for word;
//   * a thread without points (t >= n) contributes the all-zero key through its precomputed tie-break part
//     instead of a test per step; the floor 0 of the maximum replaces the `best >= 0` guard.
// SASS (P = 16, T = 256): 143 instructions per warp and step, 53 on the ALU pipe.
template <int P, int T>
__device__ __forceinline__ void fps_chain_packed(int n, int m, const float* __restrict__ src, int* __restrict__ out,
                                                 float* __restrict__ oxyz, uint2 (&s_keys)[2][32]) {
    using SO = ScanOrder<P, T>;
    constexpr int GS = SO::GS, G = P / GS, H = P / 2;
    static_assert(P % 2 == 0 && P % GS == 0 && SO::Q % GS == 0, "packed pairs and whole search groups");
    static_assert(SO::separable(), "group and in-group tie-break constants must OR together");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    unsigned long long X[H], Y[H], Z[H];
    float td[P];
#pragma unroll
    for (int h = 0; h < H; ++h) {
        float c[2][3];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int e = 2 * h + u;
            const int k = tid + SO::j_of(e) * T;
            c[u][0] = c[u][1] = c[u][2] = 0.0f;
            td[e] = -1.0f;  // padding: below the floor of the maximum, never equal to it
            if (k < n) {
                c[u][0] = src[3 * k + 0];
                c[u][1] = src[3 * k + 1];
                c[u][2] = src[3 * k + 2];
                td[e] = 1e38f;
            }
        }
        X[h] = f2_pack(c[0][0], c[1][0]);
        Y[h] = f2_pack(c[0][1], c[1][1]);
        Z[h] = f2_pack(c[0][2], c[1][2]);
    }
    // Keys of this chain are (value bits, tie-break word) reduced as max-then-MIN, i.e. the plain chain's
    // (value, ~word) max-then-max without the two complements per step.  Tie-break part of this thread: all ones
    // for a thread without points, so that its key (0, ~0) loses to every real point.
    const unsigned tp = (tid < n) ? tb_encode((unsigned)tid) : 0xffffffffu;

    float x1 = src[0], y1 = src[1], z1 = src[2];
    if (tid == 0) write_pick(out, oxyz, 0, 0, x1, y1, z1);
    // key slots of warps that do not exist stay (value 0, word ~0): the cross-warp reduction reads all 32 without a test
    if (tid < 64) (&s_keys[0][0])[tid] = make_uint2(0xffffffffu, 0u);
    __syncthreads();

#pragma unroll 2
    for (int it = 1; it < m; ++it) {
        pair_update(X, Y, Z, td, x1, y1, z1);
        // running minima are never NaN (fminf drops a NaN distance) and never -0, so == and the unsigned order of
        // the float bits are exact
        float g[G];
#pragma unroll
        for (int a = 0; a < G; ++a) {
            float v = td[GS * a];
#pragma unroll
            for (int u = 1; u < GS; ++u) v = fmaxf(v, td[GS * a + u]);
            g[a] = v;
        }
        float mx = 0.0f;
#pragma unroll
        for (int a = 0; a < G; ++a) mx = fmaxf(mx, g[a]);
        // first group in scan order that attains mx (a thread with points always has one), then the first leaf in it
        float s[GS];
#pragma unroll
        for (int u = 0; u < GS; ++u) s[u] = td[GS * (G - 1) + u];
        unsigned cg = SO::tbj(GS * (G - 1));
#pragma unroll
        for (int a = G - 2; a >= 0; --a) {
            const bool q = (g[a] == mx);
#pragma unroll
            for (int u = 0; u + 1 < GS; ++u) s[u] = q ? td[GS * a + u] : s[u];
            cg = q ? SO::tbj(GS * a) : cg;
        }
        unsigned cu = SO::tbj(GS - 1);
#pragma unroll
        for (int u = GS - 2; u >= 0; --u) cu = (s[u] == mx) ? SO::tbj(u) : cu;
        unsigned hi = __float_as_uint(mx), lo = tp | cg | cu;
        warp_max_min_pair(hi, lo);
        const int buf = it & 1;
        s_keys[buf][warp] = make_uint2(lo, hi);  // every lane holds the warp's key: one same-address store, no test
        __syncthreads();
        const uint2 e = s_keys[buf][lane];
        unsigned gh = e.y, gl = e.x;
        warp_max_min_pair(gh, gl);
        const int old = (int)tb_decode(gl);
        x1 = src[3 * old + 0];
        y1 = src[3 * old + 1];
        z1 = src[3 * old + 2];
        if (tid == 0) write_pick(out, oxyz, it, old, x1, y1, z1);
    }
}

// =================================================================================================
// One CTA per cloud.  Thread t owns points k = t + j*T (j < P).  When T is a multiple of 512 all of
// a thread's points share the reference slot k mod 512 and the in-thread strict '>' scan in
// ascending j reproduces the reference's in-slot order; for T < 512 the scan order is permuted
// (fps_step) so it is still the reference's (slot, k) order.
// Dynamic shared memory: 3*n floats — a copy of the cloud, so the picked point's coordinates are a
// 3-word broadcast LDS instead of a global/L2 round trip on the critical path.
// `sentinel` != 0 (fused SA layer only): the CTA first fills its row of idx_out with -1 and signals
// programmatic launch completion, so a dependent grid that polls idx_out for non-negative entries
// (sa_fused.cu) can consume the picks while this chain is still running — no fence in the loop.
// =================================================================================================
// V = 0: the plain chain (fps_step); V = 1: fps_chain_packed.  Same prologue, same outputs bit for bit.
// L (ragged batch): the cloud is its first cloud_length(lengths, ...) rows and n is only the row stride.  Every kernel
// below reads the length once, in its prologue, and from there on treats the rows beyond it as the padding slots of a
// short cloud.  L is a template flag so that the instances without lengths compile to the code they always did (a
// runtime test perturbs the register allocation of the chains).
template <int P, int T, int V = 0, bool L = false>
__global__ void __launch_bounds__(T, 1)
fps_cta_kernel(int n, int m, const float* __restrict__ xyz, int* __restrict__ idx_out,
               float* __restrict__ new_xyz, int sentinel, const int* __restrict__ lengths) {
    static_assert(T % 512 == 0 || 512 % T == 0, "T must divide or be a multiple of the reference's 512 slots");
    __shared__ uint2 s_keys[2][32];
    extern __shared__ __align__(16) float s_xyz[];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const float* __restrict__ pts = xyz + (size_t)cloud * n * 3;
    int* __restrict__ out = idx_out + (size_t)cloud * m;
    float* __restrict__ oxyz = new_xyz ? new_xyz + (size_t)cloud * m * 3 : nullptr;
    const int nb = L ? cloud_length(lengths, cloud, n) : n;

    // The cloud comes in as 16-byte loads, up to 12 per thread in flight before the first one is consumed, and the
    // sentinel fill with its fence runs under them.  (Measured against the 4-byte copy loop this replaces: 0.3 us of
    // the 332 us kernel at cfg2 — the prologue is not where the time goes; kept because it is the shorter chain.)
    const int total = 3 * nb;
    const bool vec = (reinterpret_cast<size_t>(pts) & 15) == 0;  // always when n % 4 == 0
    const int nv = vec ? (total >> 2) : 0;
    const float4* __restrict__ p4 = reinterpret_cast<const float4*>(pts);
    float4* __restrict__ s4 = reinterpret_cast<float4*>(s_xyz);
    constexpr int LB = 12;
    float4 v[LB];
#pragma unroll
    for (int u = 0; u < LB; ++u) {
        const int e = u * T + tid;
        if (e < nv) v[u] = __ldg(p4 + e);
    }
    if (sentinel) {  // CTA-uniform
        for (int e = tid; e < m; e += T) out[e] = -1;
        __threadfence();  // the fill is performed device-wide before the dependent grid may start
    }
#pragma unroll
    for (int u = 0; u < LB; ++u) {
        const int e = u * T + tid;
        if (e < nv) s4[e] = v[u];
    }
    for (int base = LB * T; base < nv; base += LB * T) {
#pragma unroll
        for (int u = 0; u < LB; ++u) {
            const int e = base + u * T + tid;
            if (e < nv) v[u] = __ldg(p4 + e);
        }
#pragma unroll
        for (int u = 0; u < LB; ++u) {
            const int e = base + u * T + tid;
            if (e < nv) s4[e] = v[u];
        }
    }
#pragma unroll 8
    for (int e = (nv << 2) + tid; e < total; e += T) s_xyz[e] = pts[e];
    __syncthreads();
    if (sentinel) pdl_launch_dependents();
    const float* __restrict__ src = s_xyz;

    if constexpr (V == 1) {
        fps_chain_packed<P, T>(nb, m, src, out, oxyz, s_keys);
    } else {
        // the plain chain stays in the kernel body: moved into a function of its own, it compiles to differently
        // scheduled code
        constexpr int NW = T / 32;
        float px[P], py[P], pz[P], td[P];
#pragma unroll
        for (int j = 0; j < P; ++j) {
            const int k = tid + j * T;
            if (k < nb) {
                px[j] = src[3 * k + 0];
                py[j] = src[3 * k + 1];
                pz[j] = src[3 * k + 2];
                td[j] = 1e38f;
            } else {
                px[j] = py[j] = pz[j] = 0.0f;
                td[j] = -1.0f;
            }
        }

        float x1 = src[0], y1 = src[1], z1 = src[2];
        if (tid == 0) write_pick(out, oxyz, 0, 0, x1, y1, z1);

        for (int it = 1; it < m; ++it) {
            float best;
            int bj;
            fps_step<P, ScanOrder<P, T>::DD>(px, py, pz, td, x1, y1, z1, best, bj);
            unsigned hi = 0u, lo = 0u;
            if (best >= 0.0f) {
                hi = __float_as_uint(best);
                lo = ~tb_encode((unsigned)(tid + bj * T));
            }
            warp_max_pair(hi, lo);
            const int buf = it & 1;
            if (lane == 0) s_keys[buf][warp] = make_uint2(lo, hi);
            __syncthreads();
            uint2 e = (lane < NW) ? s_keys[buf][lane] : make_uint2(0u, 0u);
            unsigned gh = e.y, gl = e.x;
            warp_max_pair(gh, gl);
            const int old = (int)tb_decode(~gl);
            x1 = src[3 * old + 0];
            y1 = src[3 * old + 1];
            z1 = src[3 * old + 2];
            if (tid == 0) write_pick(out, oxyz, it, old, x1, y1, z1);
        }
    }
}

// ---- pieces of the two cluster kernels ---------------------------------------------------------------------------
// Two step mbarriers, alternating by step parity; each step thread 0 arrives once, expecting the C messages' bytes.
__device__ __forceinline__ void init_step_mbars(unsigned long long (&s_mbar)[2]) {
    mbar_init(smem_addr(&s_mbar[0]), 1);
    mbar_init(smem_addr(&s_mbar[1]), 1);
    fence_mbar_init_cluster();
}

// This thread's points k = t + T*(rank + C*j), j < P: running minimum 1e38 (padding: coordinates 0, minimum -1), the
// coordinates of j < PR into registers, and every point to keep(j, x, y, z) for the CTA's shared-memory copy.
template <int P, int PR, int T, class Keep>
__device__ __forceinline__ void load_points(const float* __restrict__ pts, int n, long long C, unsigned rank, int tid,
                                            float (&px)[PR], float (&py)[PR], float (&pz)[PR], float (&td)[P], Keep keep) {
#pragma unroll
    for (int j = 0; j < P; ++j) {
        const long long k = (long long)tid + (long long)T * (rank + C * j);
        float x = 0.f, y = 0.f, z = 0.f, t = -1.0f;
        if (k < n) {
            x = pts[3 * k + 0];
            y = pts[3 * k + 1];
            z = pts[3 * k + 2];
            t = 1e38f;
        }
        td[j] = t;
        keep(j, x, y, z);
        if (j < PR) {
            px[j] = x;
            py[j] = y;
            pz[j] = z;
        }
    }
}

// The register-resident coordinates as packed pairs for the packed update (the scalar copies are then dead).
template <int H, int PR>
__device__ __forceinline__ void pack_pairs(const float (&px)[PR], const float (&py)[PR], const float (&pz)[PR],
                                           unsigned long long (&X)[H], unsigned long long (&Y)[H], unsigned long long (&Z)[H]) {
#pragma unroll
    for (int h = 0; h < H; ++h) {
        X[h] = f2_pack(px[2 * h], px[2 * h + 1]);
        Y[h] = f2_pack(py[2 * h], py[2 * h + 1]);
        Z[h] = f2_pack(pz[2 * h], pz[2 * h + 1]);
    }
}

// =================================================================================================
// One thread-block CLUSTER per cloud (C = 2..16 CTAs).  Thread t of CTA r owns points
// k = t + T*(r + C*j): all in one reference slot (k mod 512) whenever C*T % 512 == 0.
// Per step: CTA-local argmax as above; warp 0 then looks the CTA's candidate up in the CTA's
// shared-memory copy of its own points and pushes a 20-byte message — the 8-byte key AND the
// candidate's coordinates — into slot r of EVERY CTA's exchange buffer with st.async (one 16-byte
// and one 4-byte store per peer, each completing tx-bytes on that peer's mbarrier); all threads wait
// on their own CTA's mbarrier (expecting 20*C bytes), reduce the C keys and take the winner's
// coordinates from the same local buffer.  Nothing on the per-step critical path leaves the cluster
// (round 1 re-read the winner's coordinates from global memory/L2 every step: ~300 cycles).
// Two buffers/mbarriers alternate by step parity; there is no cluster-wide barrier per step.
// PR = points per thread whose coordinates are REGISTER-resident (the first PR of P).  PR == P: all
// of them.  PR < P (clouds too large for the register file): the remaining P-PR points are streamed
// from the shared-memory copy as 128-bit loads of 4 points per coordinate; the running minimum of
// every point stays in registers.
// =================================================================================================
// V = 1 (P % 4 == 0): the per-thread update of fps_chain_packed — packed FP32x2 distances, value-only maximum,
// position by value_argmax_first; a thread's points are already in tie-break order here (one slot per thread), and
// the tie-break word of point j is tb_encode(t + T*rank) | j << (log2(C*T) - 9).  The exchange is unchanged.
template <int P, int T, int PR, int V = 0, bool L = false>
__global__ void __launch_bounds__(T, 1)
fps_cluster_kernel(int n, int m, int log2c, const float* __restrict__ xyz, int* __restrict__ idx_out,
                   float* __restrict__ new_xyz, const int* __restrict__ lengths) {
    static_assert(T % 512 == 0 || 512 % T == 0, "T must divide or be a multiple of 512");
    static_assert(PR == P || (PR % 4 == 0 && P % 4 == 0 && PR < P), "streamed points come in groups of four");
    static_assert(V == 0 || (P % 4 == 0 && PR % 2 == 0), "the packed update works on pairs and groups of four");
    constexpr int NW = T / 32;
    constexpr bool STREAM = PR < P;
    __shared__ uint2 s_keys[2][32];
    __shared__ __align__(16) uint4 s_xa[2][16];   // per peer: (key lo, key hi, x bits, y bits)
    __shared__ __align__(4) unsigned s_xz[2][16];  // per peer: z bits
    __shared__ __align__(8) unsigned long long s_mbar[2];
    // this CTA's points.  !STREAM: SoA [c][j*T + t].  STREAM: float4 groups [(j/4)*3 + c][t] (.x..w = j%4)
    extern __shared__ __align__(16) float s_pts[];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned C = 1u << log2c, rank = cluster_ctarank();
    const int cloud = blockIdx.x >> log2c;
    const float* __restrict__ pts = xyz + (size_t)cloud * n * 3;
    int* __restrict__ out = idx_out + (size_t)cloud * m;
    float* __restrict__ oxyz = new_xyz ? new_xyz + (size_t)cloud * m * 3 : nullptr;
    const int nb = L ? cloud_length(lengths, cloud, n) : n;

    if (tid == 0) init_step_mbars(s_mbar);

    auto slot_addr = [&](int j, int t, int c) -> int {  // float index of coordinate c of local point (j, t)
        if constexpr (STREAM) return ((((j >> 2) * 3 + c) * T + t) << 2) + (j & 3);
        else return c * P * T + j * T + t;
    };

    float px[PR], py[PR], pz[PR], td[P];
    load_points<P, PR, T>(pts, nb, C, rank, tid, px, py, pz, td, [&](int j, float x, float y, float z) {
        s_pts[slot_addr(j, tid, 0)] = x;
        s_pts[slot_addr(j, tid, 1)] = y;
        s_pts[slot_addr(j, tid, 2)] = z;
    });
    constexpr int HR = (V == 1) ? PR / 2 : 1;
    unsigned long long X2[HR], Y2[HR], Z2[HR];
    unsigned tpc = 0u, jshift = 0u;
    if constexpr (V == 1) {
        pack_pairs(px, py, pz, X2, Y2, Z2);
        const unsigned base = (unsigned)tid + (unsigned)T * rank;  // this thread's point j = 0
        tpc = (base < (unsigned)nb) ? tb_encode(base) : 0xffffffffu;  // all ones: a thread without points sends key (0, 0)
        unsigned log2t = 0;
        while ((1u << log2t) < (unsigned)T) ++log2t;
        jshift = (unsigned)log2c + log2t - 9u;  // C*T is a multiple of 512 (checked by the dispatcher)
    }

    float x1 = pts[0], y1 = pts[1], z1 = pts[2];
    if (rank == 0 && tid == 0) {
        out[0] = 0;
        if (oxyz) {
            oxyz[0] = x1;
            oxyz[1] = y1;
            oxyz[2] = z1;
        }
    }
    // every CTA's mbarriers must be initialised (and its point copy complete) before any peer targets them
    cluster_sync_all();

    const unsigned mbar0 = smem_addr(&s_mbar[0]), mbar1 = smem_addr(&s_mbar[1]);
    const float4* __restrict__ s4 = reinterpret_cast<const float4*>(s_pts);

    for (int it = 1; it < m; ++it) {
        const int q = it - 1, buf = q & 1;
        const unsigned parity = (unsigned)(q >> 1) & 1u;
        const unsigned mbar = buf ? mbar1 : mbar0;
        if (tid == 0) mbar_arrive_expect_tx(mbar, 20u * C);

        unsigned hi = 0u, lo = 0u;
        if constexpr (V == 1) {
            pair_update(X2, Y2, Z2, td, x1, y1, z1);
            if constexpr (STREAM) stream_update_packed<PR / 4, P / 4, PR, T>(s4, tid, td, x1, y1, z1);
            float mx;
            int pos;
            value_argmax_first<P>(td, mx, pos);
            hi = __float_as_uint(mx);
            lo = ~(tpc | ((unsigned)pos << jshift));
        } else {
            float best;
            int bj;
            fps_step<PR, 1, P>(px, py, pz, td, x1, y1, z1, best, bj);  // the PR register-resident points
            if constexpr (STREAM) stream_update<PR / 4, P / 4, PR, T>(s4, tid, td, x1, y1, z1, best, bj);
            if (best >= 0.0f) {
                hi = __float_as_uint(best);
                lo = ~tb_encode((unsigned)(tid + T * (rank + C * bj)));
            }
        }
        warp_max_pair(hi, lo);
        if (lane == 0) s_keys[buf][warp] = make_uint2(lo, hi);
        __syncthreads();
        if (warp == 0) {
            uint2 e = (lane < NW) ? s_keys[buf][lane] : make_uint2(0u, 0u);
            unsigned ch = e.y, cl = e.x;
            warp_max_pair(ch, cl);
            // the CTA's candidate: local point (j, t) of k = t + T*(rank + C*j)
            float cx = 0.f, cy = 0.f, cz = 0.f;
            if (cl != 0u) {
                const unsigned k = tb_decode(~cl);
                const int t = (int)(k % (unsigned)T), j = (int)((k / (unsigned)T) >> log2c);
                if (j < P) {
                    cx = s_pts[slot_addr(j, t, 0)];
                    cy = s_pts[slot_addr(j, t, 1)];
                    cz = s_pts[slot_addr(j, t, 2)];
                }
            }
            const unsigned peer = lane & (C - 1u);
            if (lane < C) {
                st_async_v4(mapa_shared(smem_addr(&s_xa[buf][rank]), peer), cl, ch, __float_as_uint(cx), __float_as_uint(cy),
                            mapa_shared(mbar, peer));
            } else if (lane < 2u * C) {
                st_async_u32(mapa_shared(smem_addr(&s_xz[buf][rank]), peer), __float_as_uint(cz), mapa_shared(mbar, peer));
            }
        }
        mbar_wait_parity_cluster(mbar, parity);
        unsigned gh = 0u, gl = 0u;
        if (lane < C) {
            const uint2 kk = *reinterpret_cast<const uint2*>(&s_xa[buf][lane]);
            gl = kk.x;
            gh = kk.y;
        }
        warp_max_pair(gh, gl);
        const int old = (int)tb_decode(~gl);
        const unsigned wr = ((unsigned)old / (unsigned)T) & (C - 1u);  // the CTA that owns the winner
        const uint4 wa = s_xa[buf][wr];
        x1 = __uint_as_float(wa.z);
        y1 = __uint_as_float(wa.w);
        z1 = __uint_as_float(s_xz[buf][wr]);
        if (rank == 0 && tid == 0) {
            out[it] = old;
            if (oxyz) {
                oxyz[3 * it + 0] = x1;
                oxyz[3 * it + 1] = y1;
                oxyz[3 * it + 2] = z1;
            }
        }
    }
    // no CTA may exit while a peer can still write into its shared memory
    cluster_sync_all();
}

// =================================================================================================
// Clusters for the largest clouds (8 x 262 144 points on one GPU).  A GPU keeps only a few 16-CTA
// clusters resident when each CTA needs an SM of its own (cudaOccupancyMaxActiveClusters: seven on an
// H100), so eight such clouds run as two waves.  Smaller clusters are
// co-resident but then a CTA has to hold more points than fit when every point also sits in shared
// memory.  Here the PR register-resident points per thread are NOT copied to shared memory — the
// shared memory holds only the P-PR streamed points per thread — which makes the capacity of an SM
// registers + shared memory (T = 512: 16 + 36 points per thread = 26 624 points) and lets clusters of
// any size 2..16 (C*T is a multiple of 512 for every C) take 262 144 points with 10-12 CTAs.
// The price: the CTA's candidate coordinates can no longer be looked up by warp 0.  Instead every
// warp reduces the CTA's per-warp keys (as the single-CTA kernel does), the warp that owns the
// winning thread is the sender, and the winning lane takes the coordinates from its own registers
// (a select chain over PR entries, issued by that one warp) or from its own shared-memory column.
// =================================================================================================
// V = 1: packed update + value_argmax_first, as in fps_cluster_kernel; the tie-break word of point j is
// tb_encode(t + T*rank) + j*(C*T/512) (C*T is a multiple of 512 for every C because T is).
template <int P, int T, int PR, int V = 0, bool L = false>
__global__ void __launch_bounds__(T, 1)
fps_cluster_big_kernel(int n, int m, int C, const float* __restrict__ xyz, int* __restrict__ idx_out,
                       float* __restrict__ new_xyz, const int* __restrict__ lengths) {
    static_assert(T % 512 == 0, "every thread's points must share one reference slot for any cluster size");
    static_assert(PR < P && (P - PR) % 4 == 0, "streamed points come in groups of four");
    static_assert(V == 0 || (P % 4 == 0 && PR % 4 == 0), "the packed update works on pairs and groups of four");
    constexpr int NW = T / 32;
    constexpr int NG = (P - PR) / 4;
    __shared__ uint2 s_keys[2][32];
    __shared__ __align__(16) uint4 s_xa[2][16];   // per peer: (key lo, key hi, x bits, y bits)
    __shared__ __align__(4) unsigned s_xz[2][16];  // per peer: z bits
    __shared__ __align__(8) unsigned long long s_mbar[2];
    // streamed points only: float4 groups [(g*3 + c)*T + t], .x..w = point PR + 4g + u of thread t
    extern __shared__ __align__(16) float s_pts[];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned rank = cluster_ctarank();
    const int cloud = blockIdx.x / C;
    const float* __restrict__ pts = xyz + (size_t)cloud * n * 3;
    int* __restrict__ out = idx_out + (size_t)cloud * m;
    float* __restrict__ oxyz = new_xyz ? new_xyz + (size_t)cloud * m * 3 : nullptr;
    const int nb = L ? cloud_length(lengths, cloud, n) : n;

    if (tid == 0) init_step_mbars(s_mbar);

    float px[PR], py[PR], pz[PR], td[P];
    load_points<P, PR, T>(pts, nb, C, rank, tid, px, py, pz, td, [&](int j, float x, float y, float z) {
        if (j >= PR) {
            const int g = (j - PR) >> 2, u = (j - PR) & 3;
            s_pts[(((g * 3 + 0) * T + tid) << 2) + u] = x;
            s_pts[(((g * 3 + 1) * T + tid) << 2) + u] = y;
            s_pts[(((g * 3 + 2) * T + tid) << 2) + u] = z;
        }
    });
    constexpr int HR = (V == 1) ? PR / 2 : 1;
    unsigned long long X2[HR], Y2[HR], Z2[HR];
    unsigned tpc = 0u, jstep = 0u;
    if constexpr (V == 1) {
        pack_pairs(px, py, pz, X2, Y2, Z2);
        const unsigned base = (unsigned)tid + (unsigned)T * rank;  // this thread's point j = 0
        tpc = (base < (unsigned)nb) ? tb_encode(base) : 0xffffffffu;  // all ones: a thread without points sends key (0, 0)
        jstep = (unsigned)C * (unsigned)(T / 512);                   // k >> 9 grows by this per j; base >> 9 < jstep
    }

    float x1 = pts[0], y1 = pts[1], z1 = pts[2];
    if (rank == 0 && tid == 0) {
        out[0] = 0;
        if (oxyz) {
            oxyz[0] = x1;
            oxyz[1] = y1;
            oxyz[2] = z1;
        }
    }
    cluster_sync_all();  // every peer's mbarriers are initialised before anyone targets them

    const unsigned mbar0 = smem_addr(&s_mbar[0]), mbar1 = smem_addr(&s_mbar[1]);
    const float4* __restrict__ s4 = reinterpret_cast<const float4*>(s_pts);
    const unsigned uc = (unsigned)C;

    for (int it = 1; it < m; ++it) {
        const int q = it - 1, buf = q & 1;
        const unsigned parity = (unsigned)(q >> 1) & 1u;
        const unsigned mbar = buf ? mbar1 : mbar0;
        if (tid == 0) mbar_arrive_expect_tx(mbar, 20u * uc);

        int bj = 0;
        unsigned myhi = 0u, mylo = 0u;
        if constexpr (V == 1) {
            pair_update(X2, Y2, Z2, td, x1, y1, z1);
            stream_update_packed<0, NG, PR, T>(s4, tid, td, x1, y1, z1);
            float mx;
            value_argmax_first<P>(td, mx, bj);
            myhi = __float_as_uint(mx);
            mylo = ~(tpc + (unsigned)bj * jstep);  // tpc all ones (no points): the sum wraps to bj*jstep - 1, masked below
            if (tpc == 0xffffffffu) mylo = 0u;
        } else {
            float best;
            fps_step<PR, 1, P>(px, py, pz, td, x1, y1, z1, best, bj);
            stream_update<0, NG, PR, T>(s4, tid, td, x1, y1, z1, best, bj);
            if (best >= 0.0f) {
                myhi = __float_as_uint(best);
                mylo = ~tb_encode((unsigned)(tid + T * (rank + uc * bj)));
            }
        }
        unsigned hi = myhi, lo = mylo;
        warp_max_pair(hi, lo);
        if (lane == 0) s_keys[buf][warp] = make_uint2(lo, hi);
        __syncthreads();
        // every warp reduces the CTA's keys; the warp whose entry is the maximum sends (all-zero keys: warp 0)
        const uint2 e = (lane < NW) ? s_keys[buf][lane] : make_uint2(0u, 0u);
        unsigned ch = e.y, cl = e.x;
        warp_max_pair(ch, cl);
        const unsigned wmask = __ballot_sync(0xffffffffu, lane < NW && e.x == cl && e.y == ch);
        if (warp == __ffs((int)wmask) - 1) {
            const unsigned lmask = __ballot_sync(0xffffffffu, mylo == cl && myhi == ch);
            const int wl = __ffs((int)lmask) - 1;  // the winning thread's lane (keys are unique unless all are zero)
            float cx = 0.f, cy = 0.f, cz = 0.f;
            if constexpr (V == 1) {
#pragma unroll
                for (int h = 0; h < PR / 2; ++h) {
                    float a0, a1, b0, b1, c0, c1;
                    f2_unpack(X2[h], a0, a1);
                    f2_unpack(Y2[h], b0, b1);
                    f2_unpack(Z2[h], c0, c1);
                    if (bj == 2 * h) {
                        cx = a0;
                        cy = b0;
                        cz = c0;
                    }
                    if (bj == 2 * h + 1) {
                        cx = a1;
                        cy = b1;
                        cz = c1;
                    }
                }
            } else {
#pragma unroll
            for (int j = 0; j < PR; ++j)
                if (bj == j) {
                    cx = px[j];
                    cy = py[j];
                    cz = pz[j];
                }
            }
            if (bj >= PR) {
                const int g = (bj - PR) >> 2, u = (bj - PR) & 3;
                cx = s_pts[(((g * 3 + 0) * T + tid) << 2) + u];
                cy = s_pts[(((g * 3 + 1) * T + tid) << 2) + u];
                cz = s_pts[(((g * 3 + 2) * T + tid) << 2) + u];
            }
            cx = __shfl_sync(0xffffffffu, cx, wl);
            cy = __shfl_sync(0xffffffffu, cy, wl);
            cz = __shfl_sync(0xffffffffu, cz, wl);
            const unsigned ul = (unsigned)lane;
            if (ul < uc) {
                st_async_v4(mapa_shared(smem_addr(&s_xa[buf][rank]), ul), cl, ch, __float_as_uint(cx), __float_as_uint(cy),
                            mapa_shared(mbar, ul));
            } else if (ul < 2u * uc) {
                st_async_u32(mapa_shared(smem_addr(&s_xz[buf][rank]), ul - uc), __float_as_uint(cz), mapa_shared(mbar, ul - uc));
            }
        }
        mbar_wait_parity_cluster(mbar, parity);
        unsigned kh = 0u, kl = 0u;
        if ((unsigned)lane < uc) {
            const uint2 kk = *reinterpret_cast<const uint2*>(&s_xa[buf][lane]);
            kl = kk.x;
            kh = kk.y;
        }
        unsigned gh = kh, gl = kl;
        warp_max_pair(gh, gl);
        const int old = (int)tb_decode(~gl);
        const unsigned omask = __ballot_sync(0xffffffffu, (unsigned)lane < uc && kl == gl && kh == gh);
        const int wr = __ffs((int)omask) - 1;  // the CTA that owns the winner
        const uint4 wa = s_xa[buf][wr];
        x1 = __uint_as_float(wa.z);
        y1 = __uint_as_float(wa.w);
        z1 = __uint_as_float(s_xz[buf][wr]);
        if (rank == 0 && tid == 0) {
            out[it] = old;
            if (oxyz) {
                oxyz[3 * it + 0] = x1;
                oxyz[3 * it + 1] = y1;
                oxyz[3 * it + 2] = z1;
            }
        }
    }
    cluster_sync_all();  // no CTA may exit while a peer can still write into its shared memory
}

// =================================================================================================
// Any-size fallback: running minimum in caller-provided global scratch (32*n floats, the
// reference's own requirement, tf_sampling_g.cu:202), grid of <= 32 CTAs looping over clouds.
// =================================================================================================
template <int T>
__global__ void __launch_bounds__(T, 1)
fps_global_kernel(int b, int n, int m, const float* __restrict__ xyz, float* __restrict__ temp,
                  int* __restrict__ idx_out, float* __restrict__ new_xyz, const int* __restrict__ lengths) {
    constexpr int NW = T / 32;
    __shared__ uint2 s_keys[2][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float* __restrict__ td = temp + (size_t)blockIdx.x * n;
    for (int cloud = blockIdx.x; cloud < b; cloud += gridDim.x) {
        const float* __restrict__ pts = xyz + (size_t)cloud * n * 3;
        int* __restrict__ out = idx_out + (size_t)cloud * m;
        float* __restrict__ oxyz = new_xyz ? new_xyz + (size_t)cloud * m * 3 : nullptr;
        const int nb = cloud_length(lengths, cloud, n);
        for (int k = tid; k < nb; k += T) td[k] = 1e38f;
        float x1 = pts[0], y1 = pts[1], z1 = pts[2];
        if (tid == 0) {
            out[0] = 0;
            if (oxyz) {
                oxyz[0] = x1;
                oxyz[1] = y1;
                oxyz[2] = z1;
            }
        }
        __syncthreads();
        for (int it = 1; it < m; ++it) {
            float best = -1.0f;
            int bk = 0;
            for (int k = tid; k < nb; k += T) {  // T % 512 == 0: one slot per thread, ascending k
                const float d = d2_fma_pattern(pts[3 * (size_t)k], pts[3 * (size_t)k + 1], pts[3 * (size_t)k + 2], x1, y1, z1);
                const float d2 = fminf(d, td[k]);
                td[k] = d2;
                if (d2 > best) {
                    best = d2;
                    bk = k;
                }
            }
            unsigned hi = 0u, lo = 0u;
            if (best >= 0.0f) {
                hi = __float_as_uint(best);
                lo = ~tb_encode((unsigned)bk);
            }
            warp_max_pair(hi, lo);
            const int buf = it & 1;
            if (lane == 0) s_keys[buf][warp] = make_uint2(lo, hi);
            __syncthreads();
            uint2 e = (lane < NW) ? s_keys[buf][lane] : make_uint2(0u, 0u);
            unsigned gh = e.y, gl = e.x;
            warp_max_pair(gh, gl);
            const int old = (int)tb_decode(~gl);
            x1 = pts[3 * (size_t)old + 0];
            y1 = pts[3 * (size_t)old + 1];
            z1 = pts[3 * (size_t)old + 2];
            if (tid == 0) {
                out[it] = old;
                if (oxyz) {
                    oxyz[3 * it + 0] = x1;
                    oxyz[3 * it + 1] = y1;
                    oxyz[3 * it + 2] = z1;
                }
            }
        }
        __syncthreads();  // td reused by the next cloud
    }
}

// ---- host-side dispatch ------------------------------------------------------------------------
// Tuning override (pn2_set_fps_config / PN2_FPS_CFG): one atomic word, so concurrent launches from
// several host threads always see a consistent (threads, points/thread, cluster) triple.
static std::atomic<unsigned long long> g_fps_cfg{0ull};  // threads << 40 | ppt << 20 | (cluster + 64); 0 = built-in plan
static std::once_flag g_fps_env_once;
// Which chain the single-CTA kernel runs where both exist (points per thread >= 8): 1 = fps_chain_packed,
// 0 = the plain fps_step chain.  PN2_FPS_PACKED=0/1 overrides the built-in choice; an override plan with
// cluster = -1 / -2 (pn2_set_fps_config, PN2_FPS_CFG) forces the plain / packed chain for that plan.
constexpr int kFpsPackedDefault = 1;
static std::atomic<int> g_fps_packed{kFpsPackedDefault};
// The same choice for the cluster kernels (points per thread a multiple of 4): PN2_FPS_PACKED_CLUSTER=0/1; an override
// plan names the chain in the two low bits of `threads` (T is a multiple of 128): +1 = packed, +2 = plain.
constexpr int kFpsPackedClusterDefault = 1;
static std::atomic<int> g_fps_packed_cluster{kFpsPackedClusterDefault};

// The chain an override names in the two low bits of `threads` (T is a multiple of 128): +1 packed, +2 plain, +0 the
// built-in choice `builtin`.
static int override_chain(int threads, int builtin) {
    const int chain = threads & 3;
    return chain == 1 ? 1 : (chain == 2 ? 0 : builtin);
}

static unsigned long long pack_cfg(int threads, int ppt, int cluster) {
    if (threads <= 0) return 0ull;
    return ((unsigned long long)threads << 40) | ((unsigned long long)(ppt & 0xfffff) << 20) | (unsigned long long)(cluster + 64);
}

template <int P, int T, int V>
static int launch_cta(int b, int n, int m, const float* inp, const int* lengths, int* out, float* new_xyz, int sentinel,
                      cudaStream_t st) {
    static AttrOnce once[2];  // [ragged]
    auto kern = lengths ? fps_cta_kernel<P, T, V, true> : fps_cta_kernel<P, T, V, false>;
    // the opt-in is set for the largest cloud this instantiation can serve, so one call per device is enough
    size_t dyn = (size_t)n * 3 * sizeof(float);
    if (dyn > 200 * 1024) return (int)cudaErrorInvalidValue;
    // One sampling CTA per SM whenever the SMs are there (2b <= the SM count): the chain is bound by instruction issue on
    // its SM, so a second sampling CTA of ANOTHER batch (another stream) placed on the same SM slows both down —
    // which is what the block scheduler does when resources allow (measured: the host-buffer pipeline swung
    // between 0.34 and 0.51 ms/step with the in-flight depth).  Asking for more than half of the SM's shared
    // memory makes that placement impossible; the other SMs are there for the other batches.
    constexpr size_t kExclusive = 116 * 1024;
    if (2 * b <= num_sms() && dyn < kExclusive) dyn = kExclusive;
    cudaError_t e = ensure_attrs(once[lengths ? 1 : 0], kern, 200 * 1024, false);
    if (e != cudaSuccess) return (int)e;
    kern<<<b, T, dyn, st>>>(n, m, inp, out, new_xyz, sentinel, lengths);
    return finish_launch();
}

// `clusters` thread-block clusters of C CTAs of T threads
static cudaLaunchConfig_t cluster_config(int clusters, int C, int T, size_t dyn, cudaStream_t st, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)clusters * (unsigned)C, 1, 1);
    cfg.blockDim = dim3(T, 1, 1);
    cfg.dynamicSmemBytes = dyn;
    cfg.stream = st;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

// The two cluster kernels: fps_cluster_kernel keeps a shared-memory copy of every point (at most 200 KB),
// fps_cluster_big_kernel of the streamed points only (at most 226 KB).
template <int P, int T, int PR, int V>
struct ClusterKernel {
    static constexpr size_t dyn = (size_t)3 * P * T * sizeof(float), max_dyn = 200 * 1024;
    static constexpr int threads = T;
    static auto kernel(bool ragged = false) { return ragged ? fps_cluster_kernel<P, T, PR, V, true> : fps_cluster_kernel<P, T, PR, V, false>; }
};
template <int P, int T, int PR, int V>
struct ClusterBigKernel {
    static constexpr size_t dyn = (size_t)3 * (P - PR) * T * sizeof(float), max_dyn = 226 * 1024;
    static constexpr int threads = T;
    static auto kernel(bool ragged = false) {
        return ragged ? fps_cluster_big_kernel<P, T, PR, V, true> : fps_cluster_big_kernel<P, T, PR, V, false>;
    }
};

// cluster_arg: log2 C for fps_cluster_kernel, C for fps_cluster_big_kernel
template <class K>
static int launch_cluster(int C, int cluster_arg, int b, int n, int m, const float* inp, const int* lengths, int* out,
                          float* new_xyz, cudaStream_t st) {
    static AttrOnce once[2];  // [ragged]
    if (K::dyn > K::max_dyn) return (int)cudaErrorInvalidValue;
    const bool ragged = lengths != nullptr;
    cudaError_t e = ensure_attrs(once[ragged ? 1 : 0], K::kernel(ragged), K::dyn, true);
    if (e != cudaSuccess) return (int)e;
    cudaLaunchAttribute attr[1];
    const cudaLaunchConfig_t cfg = cluster_config(b, C, K::threads, K::dyn, st, attr);
    e = cudaLaunchKernelEx(&cfg, K::kernel(ragged), n, m, cluster_arg, inp, out, new_xyz, lengths);
    count_launch();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

// How many clusters of C CTAs of this kernel the device can hold at once (cudaOccupancyMaxActiveClusters): the
// planner must keep every cloud's cluster co-resident — a cluster that has to wait for a second wave doubles the time
// of the whole call.
template <class K>
static int cluster_capacity(int C) {
    static std::atomic<int> cache[17][64];  // [C][device]; 0 = not asked yet
    int dev = 0;
    if (C < 2 || C > 16 || cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
    const int hit = cache[C][dev].load(std::memory_order_relaxed);
    if (hit) return hit > 0 ? hit : 0;
    static AttrOnce once;
    if (K::dyn > K::max_dyn || ensure_attrs(once, K::kernel(), K::dyn, true) != cudaSuccess) return 0;
    cudaLaunchAttribute attr[1];
    const cudaLaunchConfig_t cfg = cluster_config(num_sms(), C, K::threads, K::dyn, nullptr, attr);
    int num = 0;
    if (cudaOccupancyMaxActiveClusters(&num, K::kernel(), &cfg) != cudaSuccess) {
        (void)cudaGetLastError();
        num = 0;
    }
    cache[C][dev].store(num > 0 ? num : -1, std::memory_order_relaxed);
    return num;
}

// ---- every kernel instantiation, listed once ------------------------------------------------------------------------
// X(P, T, packed): fps_cta_kernel<P, T, 0>, and <P, T, 1> where `packed` (the packed chain needs P >= 8)
#define PN2_FPS_CTA_KERNELS(X)                                                                       \
    X(1, 128, 0) X(2, 128, 0) X(4, 128, 0) X(8, 128, 1) X(16, 128, 1) X(32, 128, 1)                  \
    X(1, 256, 0) X(2, 256, 0) X(4, 256, 0) X(8, 256, 1) X(16, 256, 1) X(32, 256, 1)                  \
    X(1, 512, 0) X(2, 512, 0) X(4, 512, 0) X(8, 512, 1) X(16, 512, 1)                                \
    X(1, 1024, 0) X(2, 1024, 0) X(4, 1024, 0) X(8, 1024, 1)
// X(P, T, PR, packed): fps_cluster_kernel<P, T, PR, 0>, and <P, T, PR, 1> where `packed` (needs P % 4 == 0)
#define PN2_FPS_CLUSTER_KERNELS(X)                                                                   \
    X(4, 128, 4, 1) X(8, 128, 8, 1) X(16, 128, 16, 1) X(32, 128, 32, 1)                              \
    X(2, 256, 2, 0) X(4, 256, 4, 1) X(8, 256, 8, 1) X(16, 256, 16, 1) X(32, 256, 32, 1)              \
    X(1, 512, 1, 0) X(2, 512, 2, 0) X(4, 512, 4, 1) X(8, 512, 8, 1) X(16, 512, 16, 1) X(32, 512, 16, 1) \
    X(2, 1024, 2, 0) X(4, 1024, 4, 1) X(8, 1024, 8, 1)
// X(P, PR): fps_cluster_big_kernel<P, 512, PR, 0> and <P, 512, PR, 1>
#define PN2_FPS_BIG_KERNELS(X) X(44, 16) X(48, 12) X(52, 16)

struct FpsPlan {
    int threads, ppt, cluster;  // cluster == 0: global-scratch fallback; 1: single CTA; >= 2: thread-block cluster
    int pr;                     // cluster kernels: points per thread with register-resident coordinates (== ppt: all)
    int packed = 0;             // single CTA: 1 = fps_chain_packed where it is instantiated (ppt >= 8)
};

static int pow2_floor(int v) {
    int p = 1;
    while (p * 2 <= v) p *= 2;
    return p;
}

int fps_cluster_capacity(int threads, int ppt, int cluster, int packed);

static FpsPlan plan_fps(int b, int n) {
    std::call_once(g_fps_env_once, [] {  // PN2_FPS_CFG="threads,points_per_thread,cluster": profiling/tuning override
        const char* e = getenv("PN2_FPS_CFG");
        int t = 0, pp = 0, c = 0;
        if (e && sscanf(e, "%d,%d,%d", &t, &pp, &c) == 3) g_fps_cfg.store(pack_cfg(t, pp, c), std::memory_order_relaxed);
        const char* pk = getenv("PN2_FPS_PACKED");
        if (pk && (pk[0] == '0' || pk[0] == '1') && pk[1] == 0) g_fps_packed.store(pk[0] - '0', std::memory_order_relaxed);
        const char* pc = getenv("PN2_FPS_PACKED_CLUSTER");
        if (pc && (pc[0] == '0' || pc[0] == '1') && pc[1] == 0) g_fps_packed_cluster.store(pc[0] - '0', std::memory_order_relaxed);
    });
    const int packed = g_fps_packed.load(std::memory_order_relaxed);
    const int packed_cluster = g_fps_packed_cluster.load(std::memory_order_relaxed);
    const unsigned long long ov = g_fps_cfg.load(std::memory_order_relaxed);
    if (ov) {
        FpsPlan p;
        p.threads = (int)(ov >> 40);
        p.ppt = (int)((ov >> 20) & 0xfffff);
        p.cluster = (int)(ov & 0xfffff) - 64;
        p.packed = override_chain(p.threads, (p.cluster >= 2) ? packed_cluster : packed);
        p.threads &= ~3;
        p.pr = (p.ppt >= 32 && p.threads >= 512) ? 16 : p.ppt;  // ppt > 32: the register + shared-memory kernel
        if (p.cluster == -1 || p.cluster == -2) {  // single CTA with the chain named explicitly
            p.packed = (p.cluster == -2) ? 1 : 0;
            p.cluster = 1;
        }
        return p;
    }
    // single CTA, register-resident (cluster = 1): few warps with many points each (4-8 warps) — the
    // step is bound by the ALU pipe, the per-warp replicated reduction code and barrier latency, all of
    // which shrink with fewer warps.
    if (n <= 128) return {128, 1, 1, 1, packed};
    if (n <= 256) return {128, 2, 1, 2, packed};
    if (n <= 512) return {256, 2, 1, 2, packed};
    if (n <= 1024) return {128, 8, 1, 8, packed};
    if (n <= 2048) return {128, 16, 1, 16, packed};
    if (n <= 4096) return {256, 16, 1, 16, packed};
    if (n <= 8192) return {256, 32, 1, 32, packed};
    // cluster: as many CTAs per cloud as keeps all clouds co-resident on the SMs; inside each CTA
    // again few fat warps
    const int sms = num_sms();
    int cmax = pow2_floor(sms / (b > sms ? sms : b));
    if (cmax > 16) cmax = 16;
    if (cmax < 2) cmax = 2;
    auto pick = [packed_cluster](long long per, int C, FpsPlan& out) -> bool {
        const int t = (C >= 4) ? 128 : 256;  // C*T must be a multiple of 512
        const int pmin = (t == 128) ? 4 : 2;
        for (int pp = pmin; pp <= 32; pp *= 2) {
            if (per <= (long long)t * pp) {
                out = {t, pp, C, pp, packed_cluster};
                return true;
            }
        }
        if (per <= 256LL * 32) {
            out = {256, 32, C, 32, packed_cluster};
            return true;
        }
        if (per <= 512LL * 32) {
            out = {512, 32, C, 16, packed_cluster};  // half of the coordinates in registers, half streamed from shared memory
            return true;
        }
        return false;
    };
    FpsPlan first{0, 0, 0, 0};
    for (int C = cmax; C >= 2; C /= 2) {
        const long long per = ((long long)n + C - 1) / C;  // points per CTA
        if (per <= 1024 && C > 2) continue;                // too thin: fewer, fatter CTAs
        FpsPlan p;
        if (!pick(per, C, p)) break;                       // smaller clusters cannot hold the cloud either
        if (first.cluster == 0) first = p;
        // every cloud's cluster must be resident at once: a cluster left for a second wave doubles the call
        // (0 = capacity unknown, e.g. no device yet: take the plan)
        const int cap = fps_cluster_capacity(p.threads, p.ppt, p.cluster, p.packed);
        if (cap == 0 || cap >= b) return p;
    }
    // No power-of-two cluster keeps all b clouds resident, or none holds the cloud at all (n > 262 144).
    // Candidates: the widest power-of-two clusters in several waves, and the register + shared-memory kernel
    // (up to 512*52 points per CTA, any cluster size).  Cost model: a step costs 0.3 + 0.07 per 1000 point
    // slots of a CTA (relative units); waves run back to back.  Its constants were fitted on an earlier GPU
    // generation and have not been re-fitted on the H100; they only rank plans that hold the same cloud.
    FpsPlan best{0, 0, 0, 0};
    double best_cost = 1e30;
    auto consider = [&](const FpsPlan& p) {
        const int cap = fps_cluster_capacity(p.threads, p.ppt, p.cluster, p.packed);
        const int waves = cap > 0 ? (b + cap - 1) / cap : 1;
        double cost = waves * (0.3 + 0.07e-3 * (double)p.threads * p.ppt);
        if (cap > 0 && (long long)cap * p.cluster > sms) cost *= 1.3;  // CTAs of a wave share SMs
        if (cost < best_cost) {
            best_cost = cost;
            best = p;
        }
    };
    if (first.cluster) consider(first);
    FpsPlan widest;
    if (pick(((long long)n + 15) / 16, 16, widest)) consider(widest);
    for (int C = 16; C >= 2; --C) {
        const long long per = ((long long)n + C - 1) / C;
        if (per > 512LL * 52) break;
        consider({512, per <= 512LL * 44 ? 44 : (per <= 512LL * 48 ? 48 : 52), C, 16, packed_cluster});
    }
    if (best.cluster) return best;
    return {1024, 0, 0, 0};
}

bool fps_single_cta(int b, int n) { return plan_fps(b, n).cluster == 1; }

size_t fps_scratch_bytes(int b, int n) {
    if (b <= 0 || n <= 0) return 0;
    return plan_fps(b, n).cluster == 0 ? sizeof(float) * (size_t)(b < 32 ? b : 32) * (size_t)n : 0;
}

size_t fps_scratch_bound(int b, int n) {
    if (b <= 0 || n <= 0) return 0;
    return sizeof(float) * (size_t)(b < 32 ? b : 32) * (size_t)n;  // fps_scratch_bytes(b, k) for every k <= n is at most this
}

int fps_dispatch(int b, int n, int m, const float* inp, const int* lengths, float* temp, int* out, float* new_xyz,
                 int sentinel, cudaStream_t st) {
    if (b < 0 || n <= 0 || m < 0) return (int)cudaErrorInvalidValue;
    if (b == 0 || m == 0) return 0;
    if (!inp || !out) return (int)cudaErrorInvalidValue;
    const FpsPlan plan = plan_fps(b, n);
    if (sentinel && plan.cluster != 1) return (int)cudaErrorInvalidValue;  // the fused layer asks fps_single_cta() first
    if (plan.cluster >= 1) {
        const long long cap = (long long)plan.threads * plan.ppt * plan.cluster;
        if (cap < n) return (int)cudaErrorInvalidValue;
    }
    if (plan.cluster == 1) {
#define PN2_TRY(P, T, PK)                                                                           \
    if (plan.ppt == P && plan.threads == T)                                                                 \
        return (PK && plan.packed) ? launch_cta<P, T, PK>(b, n, m, inp, lengths, out, new_xyz, sentinel, st)         \
                                   : launch_cta<P, T, 0>(b, n, m, inp, lengths, out, new_xyz, sentinel, st);
        PN2_FPS_CTA_KERNELS(PN2_TRY)
#undef PN2_TRY
        return (int)cudaErrorInvalidValue;
    }
    const int C = plan.cluster;
    if (C >= 2 && plan.ppt > 32) {  // register + shared-memory kernel, any cluster size
        if (C > 16 || plan.threads != 512) return (int)cudaErrorInvalidValue;
#define PN2_TRY(P, PR)                                                                                       \
    if (plan.ppt == P)                                                                                               \
        return plan.packed ? launch_cluster<ClusterBigKernel<P, 512, PR, 1>>(C, C, b, n, m, inp, lengths, out, new_xyz, st)  \
                           : launch_cluster<ClusterBigKernel<P, 512, PR, 0>>(C, C, b, n, m, inp, lengths, out, new_xyz, st);
        PN2_FPS_BIG_KERNELS(PN2_TRY)
#undef PN2_TRY
        return (int)cudaErrorInvalidValue;
    }
    if (C >= 2) {
        if (C > 16 || (C & (C - 1))) return (int)cudaErrorInvalidValue;
        if (((long long)C * plan.threads) % 512 != 0) return (int)cudaErrorInvalidValue;
        int log2c = 0;
        while ((1 << log2c) < C) ++log2c;
#define PN2_TRY(P, T, PR, PK)                                                                                 \
    if (plan.ppt == P && plan.threads == T && plan.pr == PR)                                                  \
        return (PK && plan.packed)                                                                            \
                   ? launch_cluster<ClusterKernel<P, T, PR, PK>>(C, log2c, b, n, m, inp, lengths, out, new_xyz, st)    \
                   : launch_cluster<ClusterKernel<P, T, PR, 0>>(C, log2c, b, n, m, inp, lengths, out, new_xyz, st);
        PN2_FPS_CLUSTER_KERNELS(PN2_TRY)
#undef PN2_TRY
        return (int)cudaErrorInvalidValue;
    }
    // global-scratch fallback: needs the reference's (32, n) float scratch (tf_sampling_g.cu:202)
    if (!temp) return (int)cudaErrorInvalidValue;
    int grid = b < 32 ? b : 32;
    fps_global_kernel<1024><<<grid, 1024, 0, st>>>(b, n, m, inp, temp, out, new_xyz, lengths);
    return finish_launch();
}

int fps_cluster_capacity(int threads, int ppt, int cluster, int packed) {
#define PN2_CAP(P, PR)                                                                                      \
    if (threads == 512 && ppt == P)                                                                         \
        return packed ? cluster_capacity<ClusterBigKernel<P, 512, PR, 1>>(cluster)                          \
                      : cluster_capacity<ClusterBigKernel<P, 512, PR, 0>>(cluster);
    PN2_FPS_BIG_KERNELS(PN2_CAP)
#undef PN2_CAP
    if (cluster < 2 || cluster > 16 || (cluster & (cluster - 1))) return 0;
#define PN2_CAP(P, T, PR, PK)                                                                               \
    if (ppt == P && threads == T)                                                                           \
        return (PK && packed) ? cluster_capacity<ClusterKernel<P, T, PR, PK>>(cluster)                      \
                              : cluster_capacity<ClusterKernel<P, T, PR, 0>>(cluster);
    PN2_FPS_CLUSTER_KERNELS(PN2_CAP)
#undef PN2_CAP
    return 0;
}

}  // namespace pn2

extern "C" {

int pn2_fps_cluster_capacity(int threads, int points_per_thread, int cluster) {
    const int packed = pn2::override_chain(threads, pn2::g_fps_packed_cluster.load(std::memory_order_relaxed));
    return pn2::fps_cluster_capacity(threads & ~3, points_per_thread, cluster, packed);
}

int pn2_fps(int b, int n, int m, const float* inp, float* temp, int* out, void* stream) {
    return pn2::fps_dispatch(b, n, m, inp, nullptr, temp, out, nullptr, 0, pn2::as_stream(stream));
}

int pn2_fps_gather(int b, int n, int m, const float* inp, float* temp, int* out, float* new_xyz, void* stream) {
    return pn2::fps_dispatch(b, n, m, inp, nullptr, temp, out, new_xyz, 0, pn2::as_stream(stream));
}

int pn2_fps_gather_ragged(int b, int n, int m, const float* inp, const int* lengths, float* temp, int* out, float* new_xyz,
                          void* stream) {
    return pn2::fps_dispatch(b, n, m, inp, lengths, temp, out, new_xyz, 0, pn2::as_stream(stream));
}

size_t pn2_fps_scratch_bytes(int b, int n) { return pn2::fps_scratch_bytes(b, n); }

int pn2_fps_plan(int b, int n, int* threads, int* points_per_thread, int* cluster) {
    if (b <= 0 || n <= 0) return (int)cudaErrorInvalidValue;
    const pn2::FpsPlan p = pn2::plan_fps(b, n);
    if (threads) *threads = p.threads;
    if (points_per_thread) *points_per_thread = p.ppt;
    if (cluster) *cluster = p.cluster;
    return 0;
}

void pn2_set_fps_config(int threads, int points_per_thread, int cluster) {
    pn2::g_fps_cfg.store(pn2::pack_cfg(threads, points_per_thread, cluster), std::memory_order_relaxed);
}

}  // extern "C"
