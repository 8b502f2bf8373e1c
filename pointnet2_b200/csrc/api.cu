// api.cu — introspection entry points and the host-buffer set-abstraction calls of libpn2_b200.
#include "pn2_common.cuh"

namespace pn2 {
unsigned long long g_launch_count = 0;

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct SaLayout {
    size_t lengths, packed, xyz, new_xyz, fps_idx, dev_ws, dev_ws_bytes, total;
    size_t idx[kSaMaxScales], cnt[kSaMaxScales], grouped[kSaMaxScales];
};

// The workspace of the host-buffer layer with nscales ball-query scales (1 <= nscales <= kSaMaxScales, every
// nsamples[k] > 0): the input batch, new_xyz, fps_idx, then each scale's idx, pts_cnt and grouped_xyz in turn, then
// the device layer's scratch, which does not depend on nsample.  With one scale this is the single-scale layout.
// ragged: the lengths and the packed staging area come first, and the device layer's workspace is sized for every
// row stride up to n, since the ragged entries run the layer at the stride of each batch's longest cloud
static SaLayout sa_layout(int b, int n, int m, int nscales, const int* nsamples, bool ragged) {
    SaLayout L;
    size_t off = 0;
    L.lengths = off;
    if (ragged) off = align_up(off + sizeof(int) * (size_t)b, 256);
    L.packed = off;
    if (ragged) off = align_up(off + sizeof(float) * (size_t)b * n * 3, 256);
    L.xyz = off;     off = align_up(off + sizeof(float) * (size_t)b * n * 3, 256);
    L.new_xyz = off; off = align_up(off + sizeof(float) * (size_t)b * m * 3, 256);
    L.fps_idx = off; off = align_up(off + sizeof(int) * (size_t)b * m, 256);  // also the channel between the two overlapped kernels
    for (int k = 0; k < nscales; ++k) {
        const size_t s = (size_t)nsamples[k];
        L.idx[k] = off;     off = align_up(off + sizeof(int) * (size_t)b * m * s, 256);
        L.cnt[k] = off;     off = align_up(off + sizeof(int) * (size_t)b * m, 256);
        L.grouped[k] = off; off = align_up(off + sizeof(float) * (size_t)b * m * s * 3, 256);
    }
    L.dev_ws_bytes = ragged ? align_up(fps_scratch_bound(b, n), 256) + align_up(query_ball_point_workspace_bound(b, n), 256)
                            : pn2_sa_layer_device_workspace_bytes(b, n, m, nsamples[0]);  // 0 on the overlapped path
    L.dev_ws = off;  off = align_up(off + L.dev_ws_bytes, 256);
    L.total = off;
    return L;
}

// the scale list of a multi-scale call: 1 <= nscales <= kSaMaxScales, every nsample positive and, with check_radii,
// every radius too (the workspace size takes no radii)
static bool valid_scales(int nscales, const float* radii, const int* nsamples, bool check_radii) {
    if (nscales < 1 || nscales > kSaMaxScales || !nsamples || (check_radii && !radii)) return false;
    for (int k = 0; k < nscales; ++k)
        if (nsamples[k] <= 0 || (check_radii && !(radii[k] > 0.f))) return false;
    return true;
}

// The D2H copies of the host-buffer layer: new_xyz, then each scale's idx, pts_cnt and grouped_xyz, each whose host
// pointer is not NULL (h_grouped_xyz itself may be NULL).
static int copy_out(int b, int m, int nscales, const int* nsamples, const char* ws, const SaLayout& L, float* h_new_xyz,
                    int* const* h_idx, int* const* h_pts_cnt, float* const* h_grouped_xyz, cudaStream_t st) {
    if (h_new_xyz) {
        const cudaError_t e = cudaMemcpyAsync(h_new_xyz, ws + L.new_xyz, sizeof(float) * (size_t)b * m * 3, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) return (int)e;
    }
    for (int k = 0; k < nscales; ++k) {
        const size_t s = (size_t)nsamples[k];
        const struct { void* dst; size_t off, bytes; } outs[3] = {
            {h_idx[k], L.idx[k], sizeof(int) * (size_t)b * m * s},
            {h_pts_cnt[k], L.cnt[k], sizeof(int) * (size_t)b * m},
            {h_grouped_xyz ? h_grouped_xyz[k] : nullptr, L.grouped[k], sizeof(float) * (size_t)b * m * s * 3},
        };
        for (const auto& o : outs) {
            if (!o.dst) continue;
            const cudaError_t e = cudaMemcpyAsync(o.dst, ws + o.off, o.bytes, cudaMemcpyDeviceToHost, st);
            if (e != cudaSuccess) return (int)e;
        }
    }
    return 0;
}

// ---- packed clouds -> padded batch ---------------------------------------------------------------------------------
// CTA (cloud, chunk) copies its share of cloud `cloud`'s 3 len floats from the packed staging area (clouds back to
// back, offset = the sum of the lengths before it) to rows [0, len) of its row block of the padded (b, stride, 3)
// batch.  Padding rows are never written.  Lengths are clamped as every ragged kernel clamps them, so offset + len
// <= b * stride whatever the lengths array holds, and no read leaves the staging area.  Stores are 16-byte vectors
// once the destination is aligned; loads are too when the source is congruent to it (a quarter of the clouds),
// four scalar loads otherwise.  A bit copy: NaN payloads survive.
constexpr int kUnpackThreads = 256;
constexpr int kUnpackVecPerThread = 4;

__global__ void __launch_bounds__(kUnpackThreads)
ragged_unpack_kernel(const float* __restrict__ packed, const int* __restrict__ lengths, int stride, float* __restrict__ xyz) {
    __shared__ long long s_part[kUnpackThreads / 32];
    const int cloud = blockIdx.x;
    long long off = 0;
    for (int j = threadIdx.x; j < cloud; j += kUnpackThreads) off += cloud_length(lengths, j, stride);
    for (int o = 16; o > 0; o >>= 1) off += __shfl_xor_sync(kFullMask, off, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = off;
    __syncthreads();
    off = 0;
#pragma unroll
    for (int w = 0; w < kUnpackThreads / 32; ++w) off += s_part[w];

    const long long len3 = 3LL * cloud_length(lengths, cloud, stride);
    const long long d0 = 3LL * cloud * stride;
    const float* __restrict__ src = packed + 3 * off;
    float* __restrict__ dst = xyz + d0;
    const long long head = min((long long)((4 - (d0 & 3)) & 3), len3);  // scalars until dst is 16-byte aligned
    const long long nvec = (len3 - head) >> 2;
    const long long tail = head + 4 * nvec;
    const long long t = (long long)blockIdx.y * kUnpackThreads + threadIdx.x;
    const long long step = (long long)gridDim.y * kUnpackThreads;
    if (t < head) dst[t] = __ldg(src + t);
    if (t < len3 - tail) dst[tail + t] = __ldg(src + tail + t);
    const float* __restrict__ sv = src + head;
    float4* __restrict__ dv = reinterpret_cast<float4*>(dst + head);
    if (((3 * off + head) & 3) == 0) {
        const float4* __restrict__ sv4 = reinterpret_cast<const float4*>(sv);
        for (long long v = t; v < nvec; v += step) dv[v] = __ldg(sv4 + v);
    } else {
        for (long long v = t; v < nvec; v += step)
            dv[v] = make_float4(__ldg(sv + 4 * v), __ldg(sv + 4 * v + 1), __ldg(sv + 4 * v + 2), __ldg(sv + 4 * v + 3));
    }
}

static int launch_ragged_unpack(int b, int stride, const float* packed, const int* lengths, float* xyz, cudaStream_t st) {
    const long long vec = (3LL * stride + 3) / 4;
    long long chunks = (vec + (long long)kUnpackThreads * kUnpackVecPerThread - 1) / ((long long)kUnpackThreads * kUnpackVecPerThread);
    if (chunks > 65535) chunks = 65535;  // the kernel strides over whatever the grid does not cover
    ragged_unpack_kernel<<<dim3((unsigned)b, (unsigned)chunks, 1), kUnpackThreads, 0, st>>>(packed, lengths, stride, xyz);
    return finish_launch();
}

// The host-buffer layer behind the four entries.  Dense (ragged false): h_xyz is (b, n, 3).  Ragged: h_xyz is packed
// with the host lengths h_lengths, which are checked here, and the device layer runs at the stride of the longest
// cloud.  Everything is checked before the first enqueue.  The outputs follow copy_out; a scale whose grouped_xyz is
// not wanted is not computed either.
static int sa_layer_host(int b, int n, int m, int nscales, const float* radii, const int* nsamples, const float* h_xyz,
                         const int* h_lengths, bool ragged, float* h_new_xyz, int* const* h_idx, int* const* h_pts_cnt,
                         float* const* h_grouped_xyz, void* workspace, size_t workspace_bytes, void* stream) {
    if (b <= 0 || n <= 0 || m <= 0 || !valid_scales(nscales, radii, nsamples, true)) return (int)cudaErrorInvalidValue;
    if (!h_xyz || (ragged && !h_lengths) || !workspace) return (int)cudaErrorInvalidValue;
    // the lengths are host memory: checked here, and the row stride is this batch's longest cloud
    size_t rows = (size_t)b * n;
    int n_run = n;
    if (ragged) {
        rows = 0;
        n_run = 0;
        for (int i = 0; i < b; ++i) {
            const int l = h_lengths[i];
            if (l < 1 || l > n) return (int)cudaErrorInvalidValue;
            rows += (size_t)l;
            n_run = l > n_run ? l : n_run;
        }
    }
    const SaLayout L = sa_layout(b, n, m, nscales, nsamples, ragged);
    if (workspace_bytes < L.total) return (int)cudaErrorInvalidValue;
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return (int)cudaErrorMisalignedAddress;
    const size_t dev_ws_bytes = ragged ? pn2_sa_layer_device_workspace_bytes(b, n_run, m, nsamples[0]) : L.dev_ws_bytes;
    if (dev_ws_bytes > L.dev_ws_bytes) return (int)cudaErrorInvalidValue;  // the bounds in sa_layout cover every stride <= n
    cudaStream_t st = as_stream(stream);
    char* ws = static_cast<char*>(workspace);
    int* d_len = ragged ? reinterpret_cast<int*>(ws + L.lengths) : nullptr;
    float* d_xyz = reinterpret_cast<float*>(ws + L.xyz);
    int* d_idx[kSaMaxScales];
    int* d_cnt[kSaMaxScales];
    float* d_grp[kSaMaxScales];
    bool grouped = false;
    for (int k = 0; k < nscales; ++k) {
        d_idx[k] = reinterpret_cast<int*>(ws + L.idx[k]);
        d_cnt[k] = reinterpret_cast<int*>(ws + L.cnt[k]);
        // not wanted: not computed
        d_grp[k] = h_grouped_xyz && h_grouped_xyz[k] ? reinterpret_cast<float*>(ws + L.grouped[k]) : nullptr;
        grouped = grouped || d_grp[k];
    }

    cudaError_t e;
    if (ragged) {
        float* d_packed = reinterpret_cast<float*>(ws + L.packed);
        e = cudaMemcpyAsync(d_len, h_lengths, sizeof(int) * (size_t)b, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return (int)e;
        e = cudaMemcpyAsync(d_packed, h_xyz, sizeof(float) * 3 * rows, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return (int)e;
        const int rc = launch_ragged_unpack(b, n_run, d_packed, d_len, d_xyz, st);
        if (rc) return rc;
    } else {
        e = cudaMemcpyAsync(d_xyz, h_xyz, sizeof(float) * 3 * rows, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return (int)e;
    }
    const int rc = pn2_sa_layer_msg_device_ragged(b, n_run, m, nscales, radii, nsamples, d_xyz, d_len,
                                                  reinterpret_cast<int*>(ws + L.fps_idx), reinterpret_cast<float*>(ws + L.new_xyz),
                                                  d_idx, d_cnt, grouped ? d_grp : nullptr, /*center=*/0,
                                                  dev_ws_bytes ? ws + L.dev_ws : nullptr, dev_ws_bytes, stream);
    if (rc) return rc;
    return copy_out(b, m, nscales, nsamples, ws, L, h_new_xyz, h_idx, h_pts_cnt, h_grouped_xyz, st);
}

// the multi-scale entries' required outputs: new_xyz, and every scale's idx and pts_cnt
static bool msg_outputs_given(int nscales, const float* h_new_xyz, int* const* h_idx, int* const* h_pts_cnt) {
    if (nscales < 1 || nscales > kSaMaxScales || !h_new_xyz || !h_idx || !h_pts_cnt) return false;
    for (int k = 0; k < nscales; ++k)
        if (!h_idx[k] || !h_pts_cnt[k]) return false;
    return true;
}
}  // namespace pn2

extern "C" {

int pn2_api_version(void) { return PN2_API_VERSION; }

const char* pn2_error_string(int code) { return cudaGetErrorString((cudaError_t)code); }

unsigned long long pn2_launch_count(void) { return __atomic_load_n(&pn2::g_launch_count, __ATOMIC_RELAXED); }

size_t pn2_sa_layer_workspace_bytes(int b, int n, int m, int nsample) {
    if (b <= 0 || n <= 0 || m <= 0 || nsample <= 0) return 0;
    return pn2::sa_layout(b, n, m, 1, &nsample, /*ragged=*/false).total;
}

int pn2_sa_layer_host(int b, int n, int m, float radius, int nsample, const float* h_xyz, float* h_new_xyz,
                      int* h_idx, int* h_pts_cnt, float* h_grouped_xyz, void* workspace, size_t workspace_bytes,
                      void* stream) {
    return pn2::sa_layer_host(b, n, m, 1, &radius, &nsample, h_xyz, nullptr, /*ragged=*/false, h_new_xyz, &h_idx, &h_pts_cnt,
                              &h_grouped_xyz, workspace, workspace_bytes, stream);
}

size_t pn2_sa_layer_host_ragged_workspace_bytes(int b, int n, int m, int nsample) {
    if (b <= 0 || n <= 0 || m <= 0 || nsample <= 0) return 0;
    return pn2::sa_layout(b, n, m, 1, &nsample, /*ragged=*/true).total;
}

int pn2_sa_layer_host_ragged(int b, int n, int m, float radius, int nsample, const float* h_xyz, const int* h_lengths,
                             float* h_new_xyz, int* h_idx, int* h_pts_cnt, float* h_grouped_xyz, void* workspace,
                             size_t workspace_bytes, void* stream) {
    return pn2::sa_layer_host(b, n, m, 1, &radius, &nsample, h_xyz, h_lengths, /*ragged=*/true, h_new_xyz, &h_idx, &h_pts_cnt,
                              &h_grouped_xyz, workspace, workspace_bytes, stream);
}

size_t pn2_sa_layer_msg_host_workspace_bytes(int b, int n, int m, int nscales, const int* nsamples) {
    if (b <= 0 || n <= 0 || m <= 0 || !pn2::valid_scales(nscales, nullptr, nsamples, false)) return 0;
    return pn2::sa_layout(b, n, m, nscales, nsamples, /*ragged=*/false).total;
}

int pn2_sa_layer_msg_host(int b, int n, int m, int nscales, const float* radii, const int* nsamples, const float* h_xyz,
                          float* h_new_xyz, int* const* h_idx, int* const* h_pts_cnt, float* const* h_grouped_xyz,
                          void* workspace, size_t workspace_bytes, void* stream) {
    if (!pn2::msg_outputs_given(nscales, h_new_xyz, h_idx, h_pts_cnt)) return (int)cudaErrorInvalidValue;
    return pn2::sa_layer_host(b, n, m, nscales, radii, nsamples, h_xyz, nullptr, /*ragged=*/false, h_new_xyz, h_idx, h_pts_cnt,
                              h_grouped_xyz, workspace, workspace_bytes, stream);
}

size_t pn2_sa_layer_msg_host_ragged_workspace_bytes(int b, int n, int m, int nscales, const int* nsamples) {
    if (b <= 0 || n <= 0 || m <= 0 || !pn2::valid_scales(nscales, nullptr, nsamples, false)) return 0;
    return pn2::sa_layout(b, n, m, nscales, nsamples, /*ragged=*/true).total;
}

int pn2_sa_layer_msg_host_ragged(int b, int n, int m, int nscales, const float* radii, const int* nsamples, const float* h_xyz,
                                 const int* h_lengths, float* h_new_xyz, int* const* h_idx, int* const* h_pts_cnt,
                                 float* const* h_grouped_xyz, void* workspace, size_t workspace_bytes, void* stream) {
    if (!pn2::msg_outputs_given(nscales, h_new_xyz, h_idx, h_pts_cnt)) return (int)cudaErrorInvalidValue;
    return pn2::sa_layer_host(b, n, m, nscales, radii, nsamples, h_xyz, h_lengths, /*ragged=*/true, h_new_xyz, h_idx, h_pts_cnt,
                              h_grouped_xyz, workspace, workspace_bytes, stream);
}

}  // extern "C"
