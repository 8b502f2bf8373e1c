// textparse.cu — the point text of the reference's dataset files (modelnet_dataset.py:84, one shape per
// `np.loadtxt(fn, delimiter=',')`; part_seg/part_dataset_all_normal.py:88, `np.loadtxt(fn)`) parsed on the device into
// float32 rows, bit for bit what np.loadtxt(...).astype(np.float32) gives (DESIGN.md §6.18).
//
// One 1024-thread CTA per file walks it in tiles of kTile bytes: each thread finds the '\n' bytes of its 8 bytes, a
// CTA scan (cta_exclusive_sum_1024) lists them in order, and each thread then takes whole lines, reading them from
// global memory.  The line that crosses a tile boundary starts at the carried position and ends in the tile that
// holds its '\n', so no line is split.  A line is checked against a conservative grammar; a file with any line
// outside it gets the reason code of its first such line and is left to the host, which parses it with np.loadtxt.
#include "pn2_common.cuh"

namespace pn2 {
namespace {

constexpr int kTextThreads = 1024;
constexpr int kTextBytesPerThread = 8;
constexpr int kTile = kTextThreads * kTextBytesPerThread;  // < 2^16: tile offsets fit in 16 bits
constexpr int kMaxCols = 64;
constexpr int kExpCap = 1 << 20;  // exponent and fraction-digit counts saturate here; |E| > 22 goes to the host anyway
constexpr unsigned long long kNoFail = ~0ull;

// 10^0 .. 10^22: every one is exact in binary64 (5^22 < 2^53)
__constant__ double kPow10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                  1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

__device__ __forceinline__ bool is_digit(unsigned char c) { return c >= '0' && c <= '9'; }
__device__ __forceinline__ bool is_blank(unsigned char c) { return c == ' ' || c == '\t'; }

// the reason a byte that cannot continue a line sends the file to the host
__device__ __forceinline__ int byte_reason(unsigned char c) {
    return c == '\r' ? PN2_TEXT_CR : c == '#' ? PN2_TEXT_COMMENT : PN2_TEXT_SYNTAX;
}

// One field at text[p..le): [+-]? (digits [. digits]? | . digits) ([eE] [+-]? digits)?.  On success p is past it and
// *v (kWrite) holds the value: M * 10^E or M / 10^-E in one correctly rounded double operation, the sign applied
// after, rounded to float32 (Clinger's fast path: M <= 2^53 and |E| <= 22 make both operands exact).
template <bool kWrite>
__device__ int parse_field(const unsigned char* __restrict__ text, long long& p, long long le, float* v) {
    bool neg = false;
    unsigned char c = p < le ? text[p] : 0;
    if (c == '+' || c == '-') {
        neg = c == '-';
        c = ++p < le ? text[p] : 0;
    }
    unsigned long long m = 0;
    int nd = 0, frac = 0, digits = 0;  // significant digits (leading zeros stripped), fraction digits, all digits
    for (; is_digit(c); c = ++p < le ? text[p] : 0, ++digits) {
        if (m == 0 && c == '0') continue;
        if (nd < 17) m = m * 10 + (c - '0');
        ++nd;
    }
    if (c == '.') {
        c = ++p < le ? text[p] : 0;
        if (!is_digit(c)) return byte_reason(c);  // "1." and "." are outside the grammar
        for (; is_digit(c); c = ++p < le ? text[p] : 0, ++digits) {
            if (frac < kExpCap) ++frac;
            if (m == 0 && c == '0') continue;
            if (nd < 17) m = m * 10 + (c - '0');
            ++nd;
        }
    }
    if (!digits) return byte_reason(c);
    int e = 0;
    if (c == 'e' || c == 'E') {
        c = ++p < le ? text[p] : 0;
        bool eneg = false;
        if (c == '+' || c == '-') {
            eneg = c == '-';
            c = ++p < le ? text[p] : 0;
        }
        if (!is_digit(c)) return byte_reason(c);
        for (; is_digit(c); c = ++p < le ? text[p] : 0) e = min(e * 10 + (c - '0'), kExpCap);
        if (eneg) e = -e;
    }
    e -= frac;
    if (nd > 16 || m > (1ull << 53) || e > 22 || e < -22) return PN2_TEXT_INEXACT;
    if (kWrite) {
        double d = (double)m;
        if (e > 0) d = __dmul_rn(d, kPow10[e]);
        if (e < 0) d = __ddiv_rn(d, kPow10[-e]);
        *v = __double2float_rn(neg ? -d : d);
    }
    return PN2_TEXT_OK;
}

// Line text[ls..le), le at its '\n' (terminated) or at the end of the file.  kWrite: its ncol values go to out.  A
// failure at byte c reports byte_reason(c), with c = 0 past the end of the line.
template <bool kWrite>
__device__ int parse_line(const unsigned char* __restrict__ text, long long ls, long long le, bool terminated, int ncol,
                          int delim, float* __restrict__ out) {
    if (terminated && le > ls && text[le - 1] == '\r') --le;  // "\r\n"
    long long p = ls;
    if (delim == PN2_DELIM_WHITESPACE)
        while (p < le && is_blank(text[p])) ++p;
    if (p == le) return PN2_TEXT_BLANK;
    for (int f = 0;; ++f) {
        if (f == ncol) return PN2_TEXT_FIELDS;
        float v = 0.f;
        const int r = parse_field<kWrite>(text, p, le, &v);
        if (r != PN2_TEXT_OK) return r;
        if (kWrite) out[f] = v;
        if (p == le) return f + 1 == ncol ? PN2_TEXT_OK : PN2_TEXT_FIELDS;
        const unsigned char c = text[p];
        if (delim == PN2_DELIM_COMMA) {
            if (c != ',') return byte_reason(c);
            ++p;  // an empty field after it fails in parse_field
        } else {
            if (!is_blank(c)) return byte_reason(c);
            while (p < le && is_blank(text[p])) ++p;
            if (p == le) return f + 1 == ncol ? PN2_TEXT_OK : PN2_TEXT_FIELDS;
        }
    }
}

struct TextArgs {
    const unsigned char* text;
    const long long* file_off;  // (F + 1,)
    long long nbytes;           // text holds file_off[F] bytes; every offset is clamped to [0, nbytes]
    int ncol, delim;
};

// kParse = false: count every line of file blockIdx.x and check it; rows[f], status[f].
// kParse = true: for a file whose checked[f] (the scan's status) is 0, convert its first `keep` lines into
// out + ncol * row_off[f].
template <bool kParse>
__global__ void __launch_bounds__(kTextThreads)
    text_rows_kernel(TextArgs a, long long* __restrict__ rows, int* __restrict__ status, const int* __restrict__ checked,
                     long long keep, const long long* __restrict__ row_off, float* __restrict__ out, long long out_rows) {
    __shared__ unsigned short s_nl[kTile];
    __shared__ int s_w[32];
    __shared__ int s_count;
    __shared__ unsigned long long s_fail;  // (line << 8 | reason) of the first line outside the grammar
    const int f = blockIdx.x, tid = threadIdx.x;
    const long long begin = min(max(a.file_off[f], 0ll), a.nbytes);
    const long long end = min(max(a.file_off[f + 1], begin), a.nbytes);
    long long base = 0, cap = 0;
    if (kParse) {
        if (checked[f] != PN2_TEXT_OK) return;
        base = row_off[f];
        cap = base < 0 ? 0 : min(keep, out_rows - base);  // never write outside out
        if (cap <= 0) return;
    }
    if (tid == 0) s_fail = kNoFail;
    long long carry = begin, line0 = 0;  // the line that starts at `carry` is line number line0
    for (long long t0 = begin; t0 < end; t0 += kTile) {
        const long long lo = t0 + (long long)tid * kTextBytesPerThread;
        const int nb = (int)max(0ll, min((long long)kTextBytesPerThread, end - lo));
        unsigned char b[kTextBytesPerThread];
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < kTextBytesPerThread; ++j) {
            b[j] = j < nb ? a.text[lo + j] : 0;
            cnt += b[j] == '\n';
        }
        int at = cta_exclusive_sum_1024(cnt, s_w);
        if (tid == kTextThreads - 1) s_count = at + cnt;
#pragma unroll
        for (int j = 0; j < kTextBytesPerThread; ++j)
            if (b[j] == '\n') s_nl[at++] = (unsigned short)(tid * kTextBytesPerThread + j);
        __syncthreads();
        const int n = s_count;
        for (int i = tid; i < n; i += kTextThreads) {
            const long long ls = i == 0 ? carry : t0 + s_nl[i - 1] + 1, le = t0 + s_nl[i], line = line0 + i;
            if (kParse) {
                if (line < cap) parse_line<true>(a.text, ls, le, true, a.ncol, a.delim, out + a.ncol * (base + line));
            } else {
                const int r = parse_line<false>(a.text, ls, le, true, a.ncol, a.delim, nullptr);
                if (r != PN2_TEXT_OK) atomicMin(&s_fail, (unsigned long long)line << 8 | (unsigned)r);
            }
        }
        if (n) carry = t0 + s_nl[n - 1] + 1;
        line0 += n;
        __syncthreads();  // s_nl, s_count and s_w are rewritten by the next tile; s_fail is final for this one
        if (kParse ? line0 >= cap : s_fail != kNoFail) break;
    }
    if (carry < end && (kParse ? line0 < cap : s_fail == kNoFail)) {  // a last line without a terminator
        if (tid == 0) {
            if (kParse) {
                parse_line<true>(a.text, carry, end, false, a.ncol, a.delim, out + a.ncol * (base + line0));
            } else {
                const int r = parse_line<false>(a.text, carry, end, false, a.ncol, a.delim, nullptr);
                if (r != PN2_TEXT_OK) s_fail = (unsigned long long)line0 << 8 | (unsigned)r;
            }
        }
        ++line0;
    }
    if (!kParse) {
        __syncthreads();
        if (tid == 0) {
            rows[f] = line0;
            status[f] = s_fail == kNoFail ? PN2_TEXT_OK : (int)(s_fail & 0xff);
        }
    }
}

bool text_args_ok(int num_files, const unsigned char* text, const long long* file_off, long long nbytes, int ncol,
                  int delim) {
    return num_files >= 1 && text && file_off && nbytes >= 0 && ncol >= 1 && ncol <= kMaxCols &&
           (delim == PN2_DELIM_WHITESPACE || delim == PN2_DELIM_COMMA);
}

}  // namespace
}  // namespace pn2

extern "C" {

int pn2_text_rows_scan(int num_files, const unsigned char* text, const long long* file_off, long long nbytes, int ncol,
                       int delim, long long* rows, int* status, void* stream) {
    using namespace pn2;
    if (!text_args_ok(num_files, text, file_off, nbytes, ncol, delim) || !rows || !status)
        return (int)cudaErrorInvalidValue;
    const TextArgs a{text, file_off, nbytes, ncol, delim};
    text_rows_kernel<false><<<(unsigned)num_files, kTextThreads, 0, as_stream(stream)>>>(a, rows, status, nullptr, 0,
                                                                                         nullptr, nullptr, 0);
    return finish_launch();
}

int pn2_text_rows_parse(int num_files, const unsigned char* text, const long long* file_off, long long nbytes, int ncol,
                        int delim, const int* status, long long keep, const long long* row_off, float* out,
                        long long out_rows, void* stream) {
    using namespace pn2;
    if (!text_args_ok(num_files, text, file_off, nbytes, ncol, delim) || !status || keep < 0 || !row_off || !out ||
        out_rows < 0)
        return (int)cudaErrorInvalidValue;
    const TextArgs a{text, file_off, nbytes, ncol, delim};
    text_rows_kernel<true><<<(unsigned)num_files, kTextThreads, 0, as_stream(stream)>>>(
        a, nullptr, nullptr, status, keep, row_off, out, out_rows);
    return finish_launch();
}

}  // extern "C"
