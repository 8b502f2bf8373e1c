/*
 * render_oracle.c — CPU restatement of the reference's point-viewer splatter.
 *
 * TEST INFRASTRUCTURE ONLY, like pn2_oracle.c: only tests/ and tools/render_bench.py load this library, as the checker,
 * never as a fallback for the CUDA path.  Built by oracle/render_ref.py with -ffp-contract=off, so the compiler adds no
 * contraction of its own.  Pinned by tests/test_render_cpu.py against the reference's own render_ball
 * (oracle/_ref/libref_render.so) and the tests/golden/render_*.npz fixtures recorded from it.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* ------------------------------------------------------------------------------------------
 * Ball splats of the reference's point viewer.
 * Restates render_ball, utils/render_balls_so.cpp:14-56 (called by utils/show3d_balls.py:76-86), from its
 * contract (DESIGN.md §6.16) rather than its loop: r is raised to 1; the ball is every (dx, dy) in [-r, r]^2 with
 * dx^2 + dy^2 < r^2, of height int(sqrt(double(r^2 - dx^2 - dy^2))) and shade (float)(that sqrt / r); zmin / zmax are
 * min(z) - r and max(z) + r over all n points.  A pixel (x + dx, y + dy) on the canvas (x the row) goes to the
 * contribution of largest z2 = z + height above -2100000000, the lowest point index among equal z2 (a point reaches a
 * pixel once, and the sequential z-buffer's test is strict).  Its colour: intensity = min(1, (z2 - zmin) / (zmax - zmin)
 * * 0.7 + 0.3) in double; channel 0 = (shade * c2) * intensity, 1 from c0, 2 from c1, the product shade * colour
 * rounded to float, converted as x86-64 does (to int32, then the low byte).  Pixels nobody reaches keep `show`.
 */
static unsigned char x86_u8(double v) {
    int i = (v > -2147483649.0 && v < 2147483648.0) ? (int)v : (int)0x80000000u;
    return (unsigned char)i;
}

void oracle_render_ball(int h, int w, unsigned char *show, int n, const int *xyzs, const float *c0, const float *c1,
                        const float *c2, int r) {
    if (r < 1) r = 1;
    if (n <= 0 || h <= 0 || w <= 0) return;
    uint64_t *best = (uint64_t *)calloc((size_t)h * w, sizeof(uint64_t)); /* 0: no contribution */
    int zlo = xyzs[2], zhi = xyzs[2];
    for (int i = 1; i < n; ++i) {
        if (xyzs[3 * i + 2] < zlo) zlo = xyzs[3 * i + 2];
        if (xyzs[3 * i + 2] > zhi) zhi = xyzs[3 * i + 2];
    }
    const double zmin = (double)(zlo - r), zmax = (double)(zhi + r);
    for (int i = 0; i < n; ++i) {
        for (int dx = -r; dx <= r; ++dx) {
            for (int dy = -r; dy <= r; ++dy) {
                const int k = r * r - dx * dx - dy * dy;
                if (k <= 0) continue;
                const int px = xyzs[3 * i] + dx, py = xyzs[3 * i + 1] + dy;
                if (px < 0 || px >= h || py < 0 || py >= w) continue;
                const long long z2 = (long long)xyzs[3 * i + 2] + (int)sqrt((double)k);
                if (z2 <= -2100000000LL) continue;
                const uint64_t key = ((uint64_t)(uint32_t)(z2 + 2147483648LL) << 32) | (uint32_t)~(uint32_t)i;
                uint64_t *slot = best + (size_t)px * w + py;
                if (key > *slot) *slot = key;
            }
        }
    }
    for (size_t p = 0; p < (size_t)h * w; ++p) {
        if (!best[p]) continue;
        const int i = (int)~(uint32_t)best[p];
        const long long z2 = (long long)(best[p] >> 32) - 2147483648LL;
        const int dx = (int)(p / (size_t)w) - xyzs[3 * i], dy = (int)(p % (size_t)w) - xyzs[3 * i + 1];
        const double dz = sqrt((double)(r * r - dx * dx - dy * dy));
        const float shade = (float)(dz / r);
        double t = ((double)z2 - zmin) / (zmax - zmin);
        t = t * 0.7;
        t = t + 0.3;
        const double intensity = t < 1.0 ? t : 1.0;
        const float s2 = shade * c2[i], s0 = shade * c0[i], s1 = shade * c1[i];
        show[p * 3 + 0] = x86_u8((double)s2 * intensity);
        show[p * 3 + 1] = x86_u8((double)s0 * intensity);
        show[p * 3 + 2] = x86_u8((double)s1 * intensity);
    }
    free(best);
}
