/*
 * pn2_oracle.c — CPU restatement of the PointNet++ set-abstraction / feature-propagation
 * geometry ops.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this
 * library, and only as the checker (or the timed CPU baseline), never as a fallback for the
 * CUDA path.
 *
 * Parity status: PINNED.  Every function here is checked (tests/test_oracle_golden.py) against
 * golden vectors produced by the reference's own code (oracle/gen_golden.py -> tests/golden/;
 * reproduced bit for bit on an H100): the reference CUDA kernels of
 * tf_ops/sampling/tf_sampling_g.cu and tf_ops/grouping/tf_grouping_g.cu rebuilt unmodified for
 * sm_90a, and the reference CPU functions of tf_ops/3d_interpolation/tf_interpolate.cpp and
 * tf_ops/grouping/test/query_ball_point.cpp (oracle/_ref/, built by oracle/build.py).
 *
 * Each function cites the reference file:line whose behaviour it restates (paths relative to
 * the reference root).  The code is written against the behavioural spec (SURVEY.md section 8a /
 * Appendix A), not transcribed.
 *
 * Arithmetic contract (SURVEY.md section 8c):
 *   - FPS and ball query squared distance:  fmaf(dz,dz, fmaf(dx,dx, dy*dy)) — the contraction
 *     nvcc 12.9 -O2 emits for the reference sources on sm_90a (SASS: FMUL, FFMA, FFMA).
 *   - three_nn squared distance: ((dx*dx + dy*dy) + dz*dz), every op rounded on its own (the
 *     reference is x86-64 g++ -O2 without FMA).
 *   - three_interpolate: ((p1*w1 + p2*w2) + p3*w3), every op rounded on its own.
 * Build with -ffp-contract=off so the compiler adds no contraction of its own.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PN2_FPS_SLOTS 512 /* blockDim of the reference FPS launch, tf_sampling_g.cu:204 */

static inline float d2_gpu_pattern(float ax, float ay, float az, float bx, float by, float bz) {
    /* (a - b) per axis; y squared first, then x, then z folded in with fused multiply-adds */
    float dx = ax - bx, dy = ay - by, dz = az - bz;
    float t = dy * dy;
    t = fmaf(dx, dx, t);
    t = fmaf(dz, dz, t);
    return t;
}

/* ------------------------------------------------------------------------------------------
 * Farthest point sampling.
 * Restates farthestpointsamplingKernel, tf_ops/sampling/tf_sampling_g.cu:105-170, as launched by
 * farthestpointsamplingLauncher (:203-205, <<<32,512>>>): 512 slots each scanning k = slot,
 * slot+512, ... with a strict '>' against a running best that starts at -1 (:130-149), then a
 * pairwise tree over the 512 slots in which the lower slot survives a tie (:151-165).  The first
 * pick is index 0 (:114-116), the running min-distance starts at 1e38 (:118).
 * idx: (b, m) int32.
 * ------------------------------------------------------------------------------------------ */
void oracle_fps(int b, int n, int m, const float *xyz, int *idx) {
    if (m <= 0 || n <= 0) return;
    float *mind = (float *)malloc(sizeof(float) * (size_t)n);
    float slot_val[PN2_FPS_SLOTS];
    int slot_idx[PN2_FPS_SLOTS];
    for (int c = 0; c < b; ++c) {
        const float *p = xyz + (size_t)c * n * 3;
        int *o = idx + (size_t)c * m;
        for (int k = 0; k < n; ++k) mind[k] = 1e38f;
        int last = 0;
        o[0] = 0;
        for (int j = 1; j < m; ++j) {
            const float lx = p[last * 3 + 0], ly = p[last * 3 + 1], lz = p[last * 3 + 2];
            for (int s = 0; s < PN2_FPS_SLOTS; ++s) {
                float best = -1.0f;
                int besti = 0;
                for (int k = s; k < n; k += PN2_FPS_SLOTS) {
                    float d = d2_gpu_pattern(p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2], lx, ly, lz);
                    float d2 = fminf(d, mind[k]);
                    mind[k] = d2;
                    if (d2 > best) {
                        best = d2;
                        besti = k;
                    }
                }
                slot_val[s] = best;
                slot_idx[s] = besti;
            }
            /* pairwise tree: stride doubles, the right partner replaces the left only if larger */
            for (int stride = 1; stride < PN2_FPS_SLOTS; stride <<= 1) {
                for (int lo = 0; lo + stride < PN2_FPS_SLOTS; lo += 2 * stride) {
                    int hi = lo + stride;
                    if (slot_val[lo] < slot_val[hi]) {
                        slot_val[lo] = slot_val[hi];
                        slot_idx[lo] = slot_idx[hi];
                    }
                }
            }
            last = slot_idx[0];
            o[j] = last;
        }
    }
    free(mind);
}

/* Closed form of the same selection rule: argmax under the order
 * (min-dist desc, k mod 512 asc, k asc).  This is the form the CUDA kernels implement; the test
 * suite checks it equals oracle_fps (the literal restatement) on tie-heavy inputs. */
void oracle_fps_keyorder(int b, int n, int m, const float *xyz, int *idx) {
    if (m <= 0 || n <= 0) return;
    float *mind = (float *)malloc(sizeof(float) * (size_t)n);
    for (int c = 0; c < b; ++c) {
        const float *p = xyz + (size_t)c * n * 3;
        int *o = idx + (size_t)c * m;
        for (int k = 0; k < n; ++k) mind[k] = 1e38f;
        int last = 0;
        o[0] = 0;
        for (int j = 1; j < m; ++j) {
            const float lx = p[last * 3 + 0], ly = p[last * 3 + 1], lz = p[last * 3 + 2];
            float best = -1.0f;
            int besti = 0;
            for (int k = 0; k < n; ++k) {
                float d = d2_gpu_pattern(p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2], lx, ly, lz);
                float d2 = fminf(d, mind[k]);
                mind[k] = d2;
                int better = 0;
                if (d2 > best) better = 1;
                else if (d2 == best) {
                    int sk = k % PN2_FPS_SLOTS, sb = besti % PN2_FPS_SLOTS;
                    if (sk < sb || (sk == sb && k < besti)) better = 1;
                }
                if (better) {
                    best = d2;
                    besti = k;
                }
            }
            last = besti;
            o[j] = last;
        }
    }
    free(mind);
}

/* oracle_fps with a record of every step j >= 1: top[j] = the largest running minimum, count[j] = how many points
 * attain it, tied[j*64 ..] = the first 64 of them in tie-break order (slot k mod 512 ascending, then k ascending),
 * padded with -1.  The pick of step j is tied[j*64].  Same arithmetic as oracle_fps (d2_gpu_pattern, fminf, the 1e38
 * start); step 0 is recorded as top -1, count 0 and no points.  idx (b, m), top (b, m), count (b, m), tied (b, m, 64). */
#define PN2_TRACE_TIED 64
void oracle_fps_trace(int b, int n, int m, const float *xyz, int *idx, float *top, int *count, int *tied) {
    if (m <= 0 || n <= 0) return;
    float *mind = (float *)malloc(sizeof(float) * (size_t)n);
    for (int c = 0; c < b; ++c) {
        const float *p = xyz + (size_t)c * n * 3;
        int *o = idx + (size_t)c * m;
        float *tp = top + (size_t)c * m;
        int *cn = count + (size_t)c * m;
        int *td = tied + (size_t)c * m * PN2_TRACE_TIED;
        for (int k = 0; k < n; ++k) mind[k] = 1e38f;
        for (int e = 0; e < PN2_TRACE_TIED; ++e) td[e] = -1;
        int last = 0;
        o[0] = 0;
        tp[0] = -1.0f;
        cn[0] = 0;
        for (int j = 1; j < m; ++j) {
            const float lx = p[last * 3 + 0], ly = p[last * 3 + 1], lz = p[last * 3 + 2];
            float best = -1.0f;
            for (int k = 0; k < n; ++k) {
                float d = d2_gpu_pattern(p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2], lx, ly, lz);
                float d2 = fminf(d, mind[k]);
                mind[k] = d2;
                if (d2 > best) best = d2;
            }
            int *row = td + (size_t)j * PN2_TRACE_TIED;
            int cnt = 0;
            for (int e = 0; e < PN2_TRACE_TIED; ++e) row[e] = -1;
            for (int s = 0; s < PN2_FPS_SLOTS && s < n; ++s)
                for (int k = s; k < n; k += PN2_FPS_SLOTS)
                    if (mind[k] == best) {
                        if (cnt < PN2_TRACE_TIED) row[cnt] = k;
                        ++cnt;
                    }
            tp[j] = best;
            cn[j] = cnt;
            last = row[0];
            o[j] = last;
        }
    }
    free(mind);
}

/* gatherpointKernel, tf_ops/sampling/tf_sampling_g.cu:172-181 : out[b,j,:] = inp[b,idx[b,j],:] */
void oracle_gather_point(int b, int n, int m, const float *inp, const int *idx, float *out) {
    for (int c = 0; c < b; ++c)
        for (int j = 0; j < m; ++j) {
            int a = idx[(size_t)c * m + j];
            const float *s = inp + ((size_t)c * n + a) * 3;
            float *d = out + ((size_t)c * m + j) * 3;
            d[0] = s[0];
            d[1] = s[1];
            d[2] = s[2];
        }
}

/* scatteraddpointKernel, tf_sampling_g.cu:183-192 (caller zero-fills, tf_sampling.cpp:174).
 * Sequential summation order j ascending; the reference uses float atomics (order undefined). */
void oracle_gather_point_grad(int b, int n, int m, const float *out_g, const int *idx, float *inp_g) {
    for (int c = 0; c < b; ++c)
        for (int j = 0; j < m; ++j) {
            int a = idx[(size_t)c * m + j];
            float *d = inp_g + ((size_t)c * n + a) * 3;
            const float *s = out_g + ((size_t)c * m + j) * 3;
            d[0] += s[0];
            d[1] += s[1];
            d[2] += s[2];
        }
}

/* ------------------------------------------------------------------------------------------
 * Ball query.  Restates query_ball_point_gpu, tf_ops/grouping/tf_grouping_g.cu:3-36 (CPU twin:
 * tf_ops/grouping/test/query_ball_point.cpp:19-47): for each query, the first nsample indices k
 * (ascending) with max(sqrtf(d2), 1e-20f) < radius; the first hit pre-fills the whole row; the
 * count of real hits goes to pts_cnt.  Rows without a hit are left untouched by the reference
 * (undefined); here, as in the product, they are zero with pts_cnt = 0.
 * use_fma != 0: GPU contraction pattern (the parity target).  use_fma == 0: plain mul/add in
 * source order, what g++ -O2 makes of the CPU twin on x86-64.
 * ------------------------------------------------------------------------------------------ */
void oracle_query_ball_point(int b, int n, int m, float radius, int nsample, const float *xyz1,
                             const float *xyz2, int *idx, int *pts_cnt, int use_fma) {
    for (int c = 0; c < b; ++c) {
        const float *p = xyz1 + (size_t)c * n * 3;
        const float *q = xyz2 + (size_t)c * m * 3;
        for (int j = 0; j < m; ++j) {
            int *row = idx + ((size_t)c * m + j) * nsample;
            for (int l = 0; l < nsample; ++l) row[l] = 0;
            const float qx = q[j * 3 + 0], qy = q[j * 3 + 1], qz = q[j * 3 + 2];
            int cnt = 0;
            for (int k = 0; k < n && cnt < nsample; ++k) {
                float d2;
                if (use_fma) {
                    d2 = d2_gpu_pattern(qx, qy, qz, p[k * 3 + 0], p[k * 3 + 1], p[k * 3 + 2]);
                } else {
                    float dx = qx - p[k * 3 + 0], dy = qy - p[k * 3 + 1], dz = qz - p[k * 3 + 2];
                    d2 = dx * dx + dy * dy + dz * dz;
                }
                float d = fmaxf(sqrtf(d2), 1e-20f);
                if (d < radius) {
                    if (cnt == 0)
                        for (int l = 0; l < nsample; ++l) row[l] = k;
                    row[cnt++] = k;
                }
            }
            if (pts_cnt) pts_cnt[(size_t)c * m + j] = cnt;
        }
    }
}

/* Largest float t >= 0 with max(sqrtf(t),1e-20f) < radius, or -1 if none: the exact d2-domain
 * threshold the CUDA ball query compares against (sqrtf is correctly rounded, hence monotone).
 * Exposed so tests can check the product's host-side bisection against a brute-force scan. */
float oracle_ball_threshold(float radius) {
    if (!(radius > 1e-20f)) return -1.0f;
    uint32_t lo = 0, hi = 0x7f7fffffu; /* +0 .. FLT_MAX; predicate is monotone in the bit pattern */
    float f;
    memcpy(&f, &hi, 4);
    if (sqrtf(f) < radius) return f;
    /* invariant: pred(lo) true, pred(hi) false */
    while (hi - lo > 1) {
        uint32_t mid = lo + (hi - lo) / 2;
        memcpy(&f, &mid, 4);
        if (sqrtf(f) < radius) lo = mid;
        else hi = mid;
    }
    memcpy(&f, &lo, 4);
    return f;
}

/* group_point_gpu, tf_grouping_g.cu:40-57 (CPU twin test/query_ball_point.cpp:52-66):
 * out[b,j,k,:] = points[b, idx[b,j,k], :] */
void oracle_group_point(int b, int n, int c, int m, int nsample, const float *points, const int *idx,
                        float *out) {
    for (int i = 0; i < b; ++i)
        for (size_t r = 0; r < (size_t)m * nsample; ++r) {
            int a = idx[(size_t)i * m * nsample + r];
            memcpy(out + ((size_t)i * m * nsample + r) * c, points + ((size_t)i * n + a) * c,
                   sizeof(float) * (size_t)c);
        }
}

/* group_point_grad_gpu, tf_grouping_g.cu:61-78 (CPU twin test/query_ball_point.cpp:70-84);
 * caller zero-fills (tf_grouping.cpp:204). Sequential order (j, k, l) ascending. */
void oracle_group_point_grad(int b, int n, int c, int m, int nsample, const float *grad_out,
                             const int *idx, float *grad_points) {
    for (int i = 0; i < b; ++i)
        for (size_t r = 0; r < (size_t)m * nsample; ++r) {
            int a = idx[(size_t)i * m * nsample + r];
            const float *s = grad_out + ((size_t)i * m * nsample + r) * c;
            float *d = grad_points + ((size_t)i * n + a) * c;
            for (int l = 0; l < c; ++l) d[l] += s[l];
        }
}

/* ------------------------------------------------------------------------------------------
 * three_nn.  Restates threenn_cpu, tf_ops/3d_interpolation/tf_interpolate.cpp:60-103: for each
 * unknown point the three smallest squared distances to the known set, ascending, earlier index
 * first on ties (strict '<' cascade, :74-89); distance evaluated in float with no contraction
 * and compared in double against 1e40 sentinels (:66,73) — a float +inf sentinel with the same
 * strict '<' is equivalent, which is what is used here; missing neighbours (m < 3) give
 * (+inf, 0).
 * ------------------------------------------------------------------------------------------ */
void oracle_three_nn(int b, int n, int m, const float *xyz1, const float *xyz2, float *dist, int *idx) {
    for (int c = 0; c < b; ++c) {
        const float *u = xyz1 + (size_t)c * n * 3;
        const float *kn = xyz2 + (size_t)c * m * 3;
        for (int j = 0; j < n; ++j) {
            const float ux = u[j * 3 + 0], uy = u[j * 3 + 1], uz = u[j * 3 + 2];
            float b1 = INFINITY, b2 = INFINITY, b3 = INFINITY;
            int i1 = 0, i2 = 0, i3 = 0;
            for (int k = 0; k < m; ++k) {
                float dx = kn[k * 3 + 0] - ux, dy = kn[k * 3 + 1] - uy, dz = kn[k * 3 + 2] - uz;
                float d = (dx * dx + dy * dy) + dz * dz;
                if (d < b1) {
                    b3 = b2; i3 = i2;
                    b2 = b1; i2 = i1;
                    b1 = d;  i1 = k;
                } else if (d < b2) {
                    b3 = b2; i3 = i2;
                    b2 = d;  i2 = k;
                } else if (d < b3) {
                    b3 = d;  i3 = k;
                }
            }
            float *dd = dist + ((size_t)c * n + j) * 3;
            int *ii = idx + ((size_t)c * n + j) * 3;
            dd[0] = b1; dd[1] = b2; dd[2] = b3;
            ii[0] = i1; ii[1] = i2; ii[2] = i3;
        }
    }
}

/* threeinterpolate_cpu, tf_interpolate.cpp:107-127:
 * out[b,j,l] = points[b,i1,l]*w1 + points[b,i2,l]*w2 + points[b,i3,l]*w3 (left to right) */
void oracle_three_interpolate(int b, int m, int c, int n, const float *points, const int *idx,
                              const float *weight, float *out) {
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < n; ++j) {
            const int *ii = idx + ((size_t)i * n + j) * 3;
            const float *w = weight + ((size_t)i * n + j) * 3;
            const float *p1 = points + ((size_t)i * m + ii[0]) * c;
            const float *p2 = points + ((size_t)i * m + ii[1]) * c;
            const float *p3 = points + ((size_t)i * m + ii[2]) * c;
            float *o = out + ((size_t)i * n + j) * c;
            for (int l = 0; l < c; ++l) o[l] = (p1[l] * w[0] + p2[l] * w[1]) + p3[l] * w[2];
        }
}

/* threeinterpolate_grad_cpu, tf_interpolate.cpp:131-153; caller zero-fills (:258). */
void oracle_three_interpolate_grad(int b, int n, int c, int m, const float *grad_out, const int *idx,
                                   const float *weight, float *grad_points) {
    for (int i = 0; i < b; ++i)
        for (int j = 0; j < n; ++j) {
            const int *ii = idx + ((size_t)i * n + j) * 3;
            const float *w = weight + ((size_t)i * n + j) * 3;
            const float *g = grad_out + ((size_t)i * n + j) * c;
            for (int t = 0; t < 3; ++t) {
                float *d = grad_points + ((size_t)i * m + ii[t]) * c;
                for (int l = 0; l < c; ++l) d[l] += g[l] * w[t];
            }
        }
}

/* ------------------------------------------------------------------------------------------
 * selection_sort (select_top_k).  Restates selection_sort_gpu, tf_grouping_g.cu:83-123 (CPU twin
 * test/selection_sort.cpp:20-50): copy each row of the (b,m,n) distance matrix, then run the first
 * k rounds of selection sort (strict '<' when searching the minimum, swap into place), carrying
 * the indices along.  Outputs are full (b,m,n); only the first k columns are meaningful.
 * ------------------------------------------------------------------------------------------ */
void oracle_selection_sort(int b, int n, int m, int k, const float *dist, int *outi, float *out) {
    for (size_t r = 0; r < (size_t)b * m; ++r) {
        const float *src = dist + r * n;
        float *v = out + r * n;
        int *ix = outi + r * n;
        for (int s = 0; s < n; ++s) {
            v[s] = src[s];
            ix[s] = s;
        }
        for (int s = 0; s < k && s < n; ++s) {
            int mn = s;
            for (int t = s + 1; t < n; ++t)
                if (v[t] < v[mn]) mn = t;
            if (mn != s) {
                float tv = v[mn]; v[mn] = v[s]; v[s] = tv;
                int ti = ix[mn]; ix[mn] = ix[s]; ix[s] = ti;
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * prob_sample: inverse-CDF sampling.  Restates probsampleLauncher, tf_sampling_g.cu:198-201 =
 * cumsumKernel (:7-89) followed by binarysearchKernel (:91-104).
 *
 * The cumulative sum is a float32 sum whose ASSOCIATION matters for bit-exact indices, so the
 * restatement keeps the reference's addition tree:
 *   - the row is cut into chunks of 8192 values, each chunk into groups of four;
 *   - inside a complete group the inclusive prefixes are a, a+b, (a+b)+c, (c+d)+(a+b);
 *     an incomplete last group is summed left to right starting from 0 and its last prefix is
 *     its total;
 *   - the group totals go through a Brent-Kung scan (up-sweep pairing at strides 1,2,4,..,
 *     then the fill-in sweep back down), giving each group the inclusive total of the groups
 *     before it, which is added to the in-group prefixes (nothing is added to group 0);
 *   - the carry from earlier chunks is added last; the carry itself is kept as a compensated
 *     (two-float) running sum across chunks.
 * The search is the reference's descending power-of-two walk from r = n-1 over q = u * cum[n-1]:
 * step back by k whenever cum[r-k] >= q.
 * ------------------------------------------------------------------------------------------ */
void oracle_prob_cumsum(int b, int n, const float *inp, float *out) {
    enum { CHUNK = 8192 };
    float *pre = (float *)malloc(sizeof(float) * CHUNK);
    float *tot = (float *)malloc(sizeof(float) * (CHUNK / 4));
    for (int i = 0; i < b; ++i) {
        const float *src = inp + (size_t)i * n;
        float *dst = out + (size_t)i * n;
        float carry = 0.f, carry_lo = 0.f;
        for (int j = 0; j < n; j += CHUNK) {
            const int len = n - j < CHUNK ? n - j : CHUNK;
            const int groups = (len + 3) / 4;
            for (int g = 0; g < groups; ++g) {
                const float *v = src + j + 4 * g;
                float *p = pre + 4 * g;
                if (4 * g + 3 < len) {
                    const float ab = v[1] + v[0];
                    float cd = v[3] + v[2];
                    const float abc = v[2] + ab;
                    cd = cd + ab;
                    p[0] = v[0]; p[1] = ab; p[2] = abc; p[3] = cd;
                    tot[g] = cd;
                } else {
                    float acc = 0.f;
                    int t = 4 * g;
                    for (; t < len; ++t) { acc += src[j + t]; pre[t] = acc; }
                    for (; t < 4 * groups; ++t) pre[t] = acc;
                    tot[g] = acc;
                }
            }
            int lvl = 0;
            for (; (2 << lvl) <= groups; ++lvl)
                for (int k = 0; k < (groups >> (lvl + 1)); ++k)
                    tot[((2 * k + 2) << lvl) - 1] += tot[((2 * k + 1) << lvl) - 1];
            for (--lvl; lvl >= 0; --lvl) {
                const int cnt = (groups - (1 << lvl)) >> (lvl + 1);
                for (int k = 0; k < cnt; ++k)
                    tot[((2 * k + 3) << lvl) - 1] += tot[((2 * k + 2) << lvl) - 1];
            }
            for (int t = 0; t < len; ++t) {
                float p = pre[t];
                if (t >= 4) p += tot[t / 4 - 1];
                dst[j + t] = p + carry;
            }
            const float t = tot[groups - 1] + carry_lo;
            const float next = carry + t;
            carry_lo = t - (next - carry);
            carry = next;
        }
    }
    free(pre);
    free(tot);
}

void oracle_prob_search(int b, int n, int m, const float *cum, const float *query, int *result) {
    int top = 1;
    while (top < n) top <<= 1;
    for (int i = 0; i < b; ++i) {
        const float *c = cum + (size_t)i * n;
        for (int j = 0; j < m; ++j) {
            const float q = query[(size_t)i * m + j] * c[n - 1];
            int r = n - 1;
            for (int k = top; k >= 1; k >>= 1)
                if (r >= k && c[r - k] >= q) r -= k;
            result[(size_t)i * m + j] = r;
        }
    }
}

void oracle_prob_sample(int b, int n, int m, const float *inp_p, const float *inp_r, float *temp, int *out) {
    oracle_prob_cumsum(b, n, inp_p, temp);
    oracle_prob_search(b, n, m, temp, inp_r, out);
}

/* ------------------------------------------------------------------------------------------
 * The fused inference MLPs (pointnet2_b200/csrc/mlp_tile.cuh, mlp_tile_layers), float32 path:
 * up to 4 layers of Linear [+ eval-mode batch norm] [+ ReLU] on every row.  Not a reference op:
 * the restatement of the arithmetic the kernels document, so that their float32 outputs can be
 * checked bit for bit.  Per output channel, at the start of each layer,
 *     scale = 1 / sqrt(var + eps)  [* gamma when affine],  shift = fmaf(bias - mean, scale, beta)
 * (every operation rounded on its own; without a batch norm scale = 1, shift = bias); then per
 * row and channel
 *     acc = +0;  acc = fmaf(a[k], w[j][k], acc) for ascending k;  y = fmaf(acc, scale, shift)
 * and, with ReLU, y < 0 ? 0 : y (NaN and -0 pass).  A NULL bias is 0, a NULL gamma / beta means
 * a batch norm without affine, a NULL mean no batch norm.
 * ------------------------------------------------------------------------------------------ */
void oracle_mlp_affine_f32(int n, const float *bias, const float *gamma, const float *beta, const float *mean,
                           const float *var, float eps, float *scale, float *shift) {
    for (int j = 0; j < n; ++j) {
        float sc = 1.f, sh = bias ? bias[j] : 0.f;
        if (mean) {
            sc = 1.f / sqrtf(var[j] + eps);
            if (gamma) sc = sc * gamma[j];
            sh = fmaf(sh - mean[j], sc, beta ? beta[j] : 0.f);
        }
        scale[j] = sc;
        shift[j] = sh;
    }
}

/* x: (rows, cin); layer l maps widths[l-1] (cin for l = 0) to widths[l] channels, w[l] is
 * (widths[l], in) row-major; out: (rows, widths[nlayers-1]).  Returns 0, or -1 for bad arguments. */
int oracle_mlp_rows_f32(long long rows, int cin, int nlayers, const int *widths, const float *const *w,
                        const float *const *bias, const float *const *gamma, const float *const *beta,
                        const float *const *mean, const float *const *var, const float *eps, const int *relu,
                        const float *x, float *out) {
    if (rows < 0 || cin < 1 || nlayers < 1 || nlayers > 4) return -1;
    int widest = cin;
    for (int l = 0; l < nlayers; ++l) {
        if (widths[l] < 1) return -1;
        if (widths[l] > widest) widest = widths[l];
    }
    float *a = (float *)malloc(sizeof(float) * (size_t)widest);
    float *y = (float *)malloc(sizeof(float) * (size_t)widest);
    float *scale = (float *)malloc(sizeof(float) * (size_t)widest * nlayers);
    float *shift = (float *)malloc(sizeof(float) * (size_t)widest * nlayers);
    for (int l = 0; l < nlayers; ++l)
        oracle_mlp_affine_f32(widths[l], bias[l], gamma ? gamma[l] : NULL, beta ? beta[l] : NULL,
                              mean ? mean[l] : NULL, var ? var[l] : NULL, eps ? eps[l] : 0.f,
                              scale + (size_t)l * widest, shift + (size_t)l * widest);
    for (long long r = 0; r < rows; ++r) {
        int c = cin;
        memcpy(a, x + (size_t)r * cin, sizeof(float) * (size_t)cin);
        for (int l = 0; l < nlayers; ++l) {
            const float *sc = scale + (size_t)l * widest, *sh = shift + (size_t)l * widest;
            for (int j = 0; j < widths[l]; ++j) {
                const float *wj = w[l] + (size_t)j * c;
                float acc = 0.f;
                for (int k = 0; k < c; ++k) acc = fmaf(a[k], wj[k], acc);
                float v = fmaf(acc, sc[j], sh[j]);
                if (relu[l]) v = v < 0.f ? 0.f : v;
                y[j] = v;
            }
            c = widths[l];
            memcpy(a, y, sizeof(float) * (size_t)c);
        }
        memcpy(out + (size_t)r * c, a, sizeof(float) * (size_t)c);
    }
    free(a);
    free(y);
    free(scale);
    free(shift);
    return 0;
}

/* ---- masked batch norm + ReLU (csrc/masked_bn.cu), float32 -----------------------------------
 * A restatement of the documented order, not of the kernels' code: every result but invstd is
 * pinned bit for bit.  rsqrtf on the device is not correctly rounded, so the statistics return
 * the float32 var + eps it is applied to, and the later stages take the device's invstd.
 *
 * Geometry (a function of c): vec = 4 when c % 4 == 0 else 1; tx = the power of two >= the
 * lanes ceil(c / vec), capped at 32; ty = 256 / tx; chunk_rows = 32 * ty.  Row o of a chunk
 * belongs to thread y = o % ty, which holds it in group (o / ty) / 8; a thread's rows ascend.
 * Statistics per column: per group, s = the sum from +0 of its 8 rows (padding adds 0),
 * gmean = s * (1 / ng), q = fmaf(d, d, q) over the real rows; the groups Chan-merged in order;
 * the ty threads in a tree (slot y absorbs slot y + s, s = ty/2 .. 1); the chunks split into 32
 * contiguous ranges of ceil(chunks / 32), each merged in order, then a tree over the 32 ranges.
 * Chan's merge of (nb, mb, m2b) into (na, ma, m2a): wb = nb / n, d = mb - ma,
 * ma = fmaf(d, wb, ma), m2a = (m2a + m2b) + (d * d) * (na * wb).
 * With no real row at all the mean is 0 / 0 (NaN), as layers.masked_batch_norm computes it.
 * Backward sums: g = y > 0 ? dy : 0, xhat = (x - mean) * invstd, each thread adds its real rows
 * in order (sg += g, sgx = fmaf(g, xhat, sgx)), then the same two trees with plain adds.
 * ------------------------------------------------------------------------------------------ */
#define MBN_THREADS 256
#define MBN_ROWS 8
#define MBN_GROUPS 4
#define MBN_MERGE_WARPS 32

static int mbn_ty(int c) {
    const int vec = (c % 4 == 0) ? 4 : 1;
    const int lanes = (c + vec - 1) / vec;
    int tx = 1;
    while (tx < lanes && tx < 32) tx <<= 1;
    return MBN_THREADS / tx;
}

static void mbn_chan(int *na, float *ma, float *m2a, int nb, float mb, float m2b) {
    if (nb == 0) return;
    if (*na == 0) {
        *na = nb;
        *ma = mb;
        *m2a = m2b;
        return;
    }
    const int n = *na + nb;
    const float wb = (float)nb / (float)n;
    const float wab = (float)*na * wb;
    const float d = mb - *ma;
    *ma = fmaf(d, wb, *ma);
    *m2a = (*m2a + m2b) + (d * d) * wab;
    *na = n;
}

/* chunks of one column: the per-thread merge of its groups, then the tree over ty */
static void mbn_chunk_stats(long long rows, int c, int ty, long long chunk, int col, const float *x,
                            const unsigned char *keep, int *sn, float *smean, float *sm2) {
    const long long base = chunk * (long long)ty * MBN_ROWS * MBN_GROUPS;
    for (int y = 0; y < ty; ++y) {
        int n = 0;
        float mean = 0.f, m2 = 0.f;
        for (int grp = 0; grp < MBN_GROUPS; ++grp) {
            float v[MBN_ROWS];
            int kf[MBN_ROWS], ng = 0;
            for (int k = 0; k < MBN_ROWS; ++k) {
                const long long r = base + y + (long long)(grp * MBN_ROWS + k) * ty;
                kf[k] = r < rows && keep[r] != 0;
                v[k] = kf[k] ? x[(size_t)r * c + col] : 0.f;
                ng += kf[k];
            }
            if (ng == 0) continue;
            const float inv = 1.0f / (float)ng;
            float s = 0.f;
            for (int k = 0; k < MBN_ROWS; ++k) s = s + v[k];
            const float gm = s * inv;
            float q = 0.f;
            for (int k = 0; k < MBN_ROWS; ++k) {
                const float d = kf[k] ? v[k] - gm : 0.f;
                q = fmaf(d, d, q);
            }
            mbn_chan(&n, &mean, &m2, ng, gm, q);
        }
        sn[y] = n;
        smean[y] = mean;
        sm2[y] = m2;
    }
    for (int s = ty >> 1; s > 0; s >>= 1)
        for (int y = 0; y < s; ++y) mbn_chan(&sn[y], &smean[y], &sm2[y], sn[y + s], smean[y + s], sm2[y + s]);
}

/* x (rows, c) float32 values, keep (rows,).  Writes mean (c), var_eps (c) = var + eps with var
 * = M2 / cnt (biased) and *count = cnt.  When running_mean is given, updates running_mean /
 * running_var as the kernel does: f = momentum, or 1 / (float)nbt when momentum < 0;
 * unbiased = var * cnt / max(cnt - 1, 1); r = r * (1 - f) + stat * f. */
void oracle_mbn_stats(int rows, int c, const float *x, const unsigned char *keep, float eps, float momentum,
                      long long nbt, float *running_mean, float *running_var, float *mean, float *var_eps,
                      int *count) {
    const int ty = mbn_ty(c);
    const long long chunk_rows = (long long)ty * MBN_ROWS * MBN_GROUPS;
    const long long chunks = rows > 0 ? (rows + chunk_rows - 1) / chunk_rows : 0;
    int *pcnt = (int *)malloc(sizeof(int) * (size_t)(chunks + 1));
    float *pmean = (float *)malloc(sizeof(float) * (size_t)(chunks + 1));
    float *pm2 = (float *)malloc(sizeof(float) * (size_t)(chunks + 1));
    int *sn = (int *)malloc(sizeof(int) * MBN_THREADS);
    float *smean = (float *)malloc(sizeof(float) * MBN_THREADS);
    float *sm2 = (float *)malloc(sizeof(float) * MBN_THREADS);
    const long long per = (chunks + MBN_MERGE_WARPS - 1) / MBN_MERGE_WARPS;
    for (int col = 0; col < c; ++col) {
        for (long long k = 0; k < chunks; ++k) {
            mbn_chunk_stats(rows, c, ty, k, col, x, keep, sn, smean, sm2);
            pcnt[k] = sn[0];
            pmean[k] = smean[0];
            pm2[k] = sm2[0];
        }
        int wn[MBN_MERGE_WARPS];
        float wmean[MBN_MERGE_WARPS], wm2[MBN_MERGE_WARPS];
        for (int w = 0; w < MBN_MERGE_WARPS; ++w) {
            const long long k0 = (long long)w * per < chunks ? (long long)w * per : chunks;
            const long long k1 = k0 + per < chunks ? k0 + per : chunks;
            wn[w] = 0;
            wmean[w] = 0.f;
            wm2[w] = 0.f;
            for (long long k = k0; k < k1; ++k) mbn_chan(&wn[w], &wmean[w], &wm2[w], pcnt[k], pmean[k], pm2[k]);
        }
        for (int s = MBN_MERGE_WARPS >> 1; s > 0; s >>= 1)
            for (int w = 0; w < s; ++w) mbn_chan(&wn[w], &wmean[w], &wm2[w], wn[w + s], wmean[w + s], wm2[w + s]);
        const float cnt = (float)wn[0];
        const float mu = wn[0] > 0 ? wmean[0] : 0.f / cnt;
        const float var = wm2[0] / cnt;
        mean[col] = mu;
        var_eps[col] = var + eps;
        *count = wn[0];
        if (running_mean) {
            const float f = momentum < 0.f ? 1.0f / (float)nbt : momentum;
            const float keepf = 1.0f - f;
            const float unbiased = (var * cnt) / fmaxf(cnt - 1.0f, 1.0f);
            running_mean[col] = running_mean[col] * keepf + mu * f;
            running_var[col] = running_var[col] * keepf + unbiased * f;
        }
    }
    free(pcnt);
    free(pmean);
    free(pm2);
    free(sn);
    free(smean);
    free(sm2);
}

/* y = keep ? (t < 0 ? 0 : t) : 0 with t = fmaf(x - mean, invstd * gamma, beta) (gamma NULL: 1,
 * beta NULL: 0).  float32, before the rounding to the tensor's dtype. */
void oracle_mbn_norm_relu(int rows, int c, const float *x, const unsigned char *keep, const float *mean,
                          const float *invstd, const float *gamma, const float *beta, float *y) {
    for (long long r = 0; r < rows; ++r)
        for (int col = 0; col < c; ++col) {
            const size_t o = (size_t)r * c + col;
            const float sc = gamma ? invstd[col] * gamma[col] : invstd[col];
            const float t = fmaf(x[o] - mean[col], sc, beta ? beta[col] : 0.f);
            y[o] = keep[r] ? (t < 0.f ? 0.f : t) : 0.f;
        }
}

static float mbn_dx(float g, float xh, float a, float mg, float mgx) { return a * fmaf(-xh, mgx, g - mg); }

/* backward of the plain form from dy, x and y (the values of the tensors, y as the forward
 * rounded it): dx (float32, before rounding), dgamma = sum g * xhat, dbeta = sum g. */
void oracle_mbn_backward(int rows, int c, const float *dy, const float *x, const float *y, const unsigned char *keep,
                         const float *gamma, const float *mean, const float *invstd, float *dx, float *dgamma,
                         float *dbeta) {
    const int ty = mbn_ty(c);
    const long long chunk_rows = (long long)ty * MBN_ROWS * MBN_GROUPS;
    const long long chunks = rows > 0 ? (rows + chunk_rows - 1) / chunk_rows : 0;
    const long long per = (chunks + MBN_MERGE_WARPS - 1) / MBN_MERGE_WARPS;
    float *psg = (float *)malloc(sizeof(float) * (size_t)(chunks + 1));
    float *psgx = (float *)malloc(sizeof(float) * (size_t)(chunks + 1));
    float sg[MBN_THREADS], sgx[MBN_THREADS];
    int cnt = 0;
    for (long long r = 0; r < rows; ++r) cnt += keep[r] != 0;
    for (int col = 0; col < c; ++col) {
        const float mu = mean[col], is = invstd[col];
        for (long long k = 0; k < chunks; ++k) {
            for (int t = 0; t < ty; ++t) {
                sg[t] = 0.f;
                sgx[t] = 0.f;
                for (int i = 0; i < MBN_ROWS * MBN_GROUPS; ++i) {
                    const long long r = k * chunk_rows + t + (long long)i * ty;
                    if (r >= rows || !keep[r]) continue;
                    const size_t o = (size_t)r * c + col;
                    const float g = y[o] > 0.f ? dy[o] : 0.f;
                    sg[t] = sg[t] + g;
                    sgx[t] = fmaf(g, (x[o] - mu) * is, sgx[t]);
                }
            }
            for (int s = ty >> 1; s > 0; s >>= 1)
                for (int t = 0; t < s; ++t) {
                    sg[t] = sg[t] + sg[t + s];
                    sgx[t] = sgx[t] + sgx[t + s];
                }
            psg[k] = sg[0];
            psgx[k] = sgx[0];
        }
        float wg[MBN_MERGE_WARPS], wgx[MBN_MERGE_WARPS];
        for (int w = 0; w < MBN_MERGE_WARPS; ++w) {
            const long long k0 = (long long)w * per < chunks ? (long long)w * per : chunks;
            const long long k1 = k0 + per < chunks ? k0 + per : chunks;
            wg[w] = 0.f;
            wgx[w] = 0.f;
            for (long long k = k0; k < k1; ++k) {
                wg[w] = wg[w] + psg[k];
                wgx[w] = wgx[w] + psgx[k];
            }
        }
        for (int s = MBN_MERGE_WARPS >> 1; s > 0; s >>= 1)
            for (int w = 0; w < s; ++w) {
                wg[w] = wg[w] + wg[w + s];
                wgx[w] = wgx[w] + wgx[w + s];
            }
        if (dbeta) dbeta[col] = wg[0];
        if (dgamma) dgamma[col] = wgx[0];
        const float a = gamma ? gamma[col] * is : is;
        const float mg = wg[0] / (float)cnt, mgx = wgx[0] / (float)cnt;
        for (long long r = 0; r < rows; ++r) {
            const size_t o = (size_t)r * c + col;
            const float g = y[o] > 0.f ? dy[o] : 0.f;
            dx[o] = keep[r] ? mbn_dx(g, (x[o] - mu) * is, a, mg, mgx) : 0.f;
        }
    }
    free(psg);
    free(psgx);
}

static uint32_t mbn_key(float v) {
    if (v != v) return 0xffffffffu;
    uint32_t u;
    memcpy(&u, &v, sizeof u);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

/* max-pool of y (b, n, c), the values as rounded to the tensor's dtype: per (cloud, column) the
 * FIRST real row with the largest key (NaN largest, -0 < +0): out = y there, argmax = the row;
 * a cloud without a real row gets out 0, argmax -1. */
void oracle_mbn_max_pool(int b, int n, int c, const float *y, const unsigned char *keep, float *out, int *argmax) {
    for (long long i = 0; i < b; ++i)
        for (int col = 0; col < c; ++col) {
            uint32_t best = 0;
            int arg = -1;
            for (int j = 0; j < n; ++j) {
                if (!keep[i * n + j]) continue;
                const uint32_t k = mbn_key(y[((size_t)i * n + j) * c + col]);
                if (k > best) {
                    best = k;
                    arg = j;
                }
            }
            out[i * c + col] = arg >= 0 ? y[((size_t)i * n + arg) * c + col] : 0.f;
            argmax[i * c + col] = arg;
        }
}

/* backward of the max-pooled form: g_i = argmax >= 0 && out_i > 0 ? dout_i : 0 and xhat at the
 * argmax row, dbeta = sum_i g_i and dgamma = fmaf(g_i, xhat_i, .) over ascending clouds i;
 * dx = keep ? a * fmaf(-xhat, dgamma / cnt, g - dbeta / cnt) : 0 (g = g_i on the argmax row). */
void oracle_mbn_max_backward(int b, int n, int c, const float *dout, const float *x, const float *out,
                             const int *argmax, const unsigned char *keep, const float *gamma, const float *mean,
                             const float *invstd, float *dx, float *dgamma, float *dbeta) {
    int cnt = 0;
    for (long long r = 0; r < (long long)b * n; ++r) cnt += keep[r] != 0;
    for (int col = 0; col < c; ++col) {
        const float mu = mean[col], is = invstd[col];
        float sg = 0.f, sgx = 0.f;
        for (long long i = 0; i < b; ++i) {
            const int r = argmax[i * c + col];
            float g = 0.f, xh = 0.f;
            if (r >= 0 && out[i * c + col] > 0.f) {
                g = dout[i * c + col];
                xh = (x[((size_t)i * n + r) * c + col] - mu) * is;
            }
            sg = sg + g;
            sgx = fmaf(g, xh, sgx);
        }
        if (dbeta) dbeta[col] = sg;
        if (dgamma) dgamma[col] = sgx;
        const float a = gamma ? gamma[col] * is : is;
        const float mg = sg / (float)cnt, mgx = sgx / (float)cnt;
        for (long long i = 0; i < b; ++i)
            for (int j = 0; j < n; ++j) {
                const size_t o = ((size_t)i * n + j) * c + col;
                const int r = argmax[i * c + col];
                const float g = r == j && out[i * c + col] > 0.f ? dout[i * c + col] : 0.f;
                dx[o] = keep[i * n + j] ? mbn_dx(g, (x[o] - mu) * is, a, mg, mgx) : 0.f;
            }
    }
}
