// letor.cu -- LETOR text files read on the device: line index, line parse, grouping by qid, per-query scaling, label
// clipping, presort and the final gather (DESIGN.md "Reading LETOR files on the device").
//
// Reference functions replaced (wildltr/ptranking @ f1d366c), ptranking/data/data_utils.py:
//   iter_lines / parse_letor  :276-387   one line -> (label, qid, fid:val features); width = the file's largest fid
//   iter_queries              :420-549   documents collected per qid in order of first appearance, MSLETOR_LIST labels
//                                        n - r, per-query StandardScaler / MinMaxScaler (Istella clip first)
//   clip_query_data           :389-418   binary_rele / unknown_as_zero label clipping, min_docs / min_rele, presort
//
// Stages and their read-backs (each sizes the next stage's buffers):
//   ptrb200_letor_count_lines   newline count per 4 KiB chunk + scan            -> n_lines
//   ptrb200_letor_index_lines   line_start[n_lines + 1]
//   ptrb200_letor_parse         scan mode (X == NULL): labels, qid spans, width  -> width, first error, undecided count
//                               fill mode: the float64 rows [n_lines, W]         -> first error, undecided count
//   ptrb200_letor_group         hash of qid bytes, byte-exact equality          -> queries, longest query
//                               offsets[B + 1], lines grouped per query in file order
//   ptrb200_letor_select        labels, clipping, kept queries, presort order   -> kept queries, kept documents
//   ptrb200_letor_gather        per-query float64 scaling, fp32 / bf16 rows
#include <cuda_bf16.h>

#include "letor_float.cuh"
#include "losses_common.cuh"

namespace ptrb200 {

static constexpr int kChunk = 4096;             // bytes per line-index CTA (256 threads x 16 bytes)
static constexpr int kScanThreads = 512, kScanPer = 8, kScanTile = kScanThreads * kScanPer;

// parse error codes, reported with the 1-based line number of the first malformed line
enum { E_NONE = 0, E_EMPTY = 1, E_LABEL = 2, E_QID = 3, E_TOKEN = 4, E_FID_LOW = 5, E_FID_HIGH = 6, E_NO_FEATURES = 7 };
static const char* parse_error_text(int code) {
    switch (code) {
        case E_EMPTY: return "empty line";
        case E_LABEL: return "the label is not a decimal number";
        case E_QID: return "the second token is not qid:<id>";
        case E_TOKEN: return "a feature token is not <fid>:<decimal>";
        case E_FID_LOW: return "feature id below the first index (0 one-indexed, -1 zero-indexed)";
        case E_FID_HIGH: return "feature id above PTRB200_LETOR_MAX_FEATURES";
        case E_NO_FEATURES: return "no features";
        default: return "malformed line";
    }
}

// ---- device-wide exclusive scan of int32 (tiles of 4096, one CTA scans the tile sums) -------------------------------
static __device__ __forceinline__ int block_exclusive_scan(int v, int* red, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    __syncthreads();
    if (lane == 31) red[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int s = lane < nw ? red[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
        red[32 + lane] = s;
    }
    __syncthreads();
    *total = red[32 + nw - 1];
    return inc - v + (warp ? red[32 + warp - 1] : 0);
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_sums_kernel(const int32_t* __restrict__ in, int64_t n, int32_t* __restrict__ sums) {
    __shared__ int red[64];
    const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanPer;
    int s = 0;
    for (int k = 0; k < kScanPer; ++k) if (base + k < n) s += in[base + k];
    int total;
    block_exclusive_scan(s, red, &total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// one CTA: exclusive scan of the tile sums in place, grand total to *total
__global__ void __launch_bounds__(kScanThreads) scan_sums_kernel(int32_t* __restrict__ sums, int64_t m, int32_t* __restrict__ total) {
    __shared__ int red[64];
    int carry = 0;
    for (int64_t t0 = 0; t0 < m; t0 += kScanTile) {
        const int64_t base = t0 + (int64_t)threadIdx.x * kScanPer;
        int v[kScanPer], s = 0;
        for (int k = 0; k < kScanPer; ++k) { v[k] = base + k < m ? sums[base + k] : 0; s += v[k]; }
        int tot;
        int run = carry + block_exclusive_scan(s, red, &tot);
        for (int k = 0; k < kScanPer; ++k) { if (base + k < m) sums[base + k] = run; run += v[k]; }
        carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const int32_t* __restrict__ in, int64_t n, const int32_t* __restrict__ sums,
                                                                  int32_t* __restrict__ out) {
    __shared__ int red[64];
    const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanPer;
    int v[kScanPer], s = 0;
    for (int k = 0; k < kScanPer; ++k) { v[k] = base + k < n ? in[base + k] : 0; s += v[k]; }
    int tot;
    int run = sums[blockIdx.x] + block_exclusive_scan(s, red, &tot);
    for (int k = 0; k < kScanPer; ++k) if (base + k < n) { out[base + k] = run; run += v[k]; }
}

static int64_t scan_sums_len(int64_t n) { return (n + kScanTile - 1) / kScanTile; }

// out[i] = sum in[0..i), *total = sum in; `sums` holds scan_sums_len(n) ints.  in may equal out.
static int exclusive_scan(const int32_t* in, int64_t n, int32_t* out, int32_t* sums, int32_t* total, cudaStream_t st) {
    const int64_t m = scan_sums_len(n);
    if (m > 0x7fffffff) { set_error("letor: scan of %lld elements is too long", (long long)n); return PTRB200_ERR_UNSUPPORTED; }
    PTRB200_LAUNCH(scan_tile_sums_kernel, (unsigned)m, kScanThreads, 0, st, in, n, sums);
    PTRB200_LAUNCH(scan_sums_kernel, 1, kScanThreads, 0, st, sums, m, total);
    PTRB200_LAUNCH(scan_apply_kernel, (unsigned)m, kScanThreads, 0, st, in, n, sums, out);
    return check_launch("letor scan");
}

// ---- line index ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) count_newlines_kernel(const uint8_t* __restrict__ text, int64_t nbytes, int32_t* __restrict__ counts) {
    __shared__ int red[64];
    const int64_t base = (int64_t)blockIdx.x * kChunk + threadIdx.x * 16;
    int c = 0;
    for (int k = 0; k < 16; ++k) c += (base + k < nbytes && text[base + k] == '\n');
    int total;
    block_exclusive_scan(c, red, &total);
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// line_start[0] = 0; line_start[j + 1] = 1 + position of the j-th newline; a last line without a newline ends at nbytes
__global__ void __launch_bounds__(256) line_starts_kernel(const uint8_t* __restrict__ text, int64_t nbytes, const int32_t* __restrict__ chunk_base,
                                                          int64_t* __restrict__ line_start, int64_t n_lines) {
    __shared__ int red[64];
    const int64_t base = (int64_t)blockIdx.x * kChunk + threadIdx.x * 16;
    int c = 0;
    for (int k = 0; k < 16; ++k) c += (base + k < nbytes && text[base + k] == '\n');
    int total;
    int j = chunk_base[blockIdx.x] + block_exclusive_scan(c, red, &total);
    for (int k = 0; k < 16; ++k)
        if (base + k < nbytes && text[base + k] == '\n') line_start[++j] = base + k + 1;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        line_start[0] = 0;
        if (text[nbytes - 1] != '\n') line_start[n_lines] = nbytes + 1;
    }
}

// ---- line parse ----------------------------------------------------------------------------------------------------
// Python's str.split() whitespace for text decoded as ISO-8859-1 (data_utils.py:446)
static __device__ __forceinline__ bool is_space(uint8_t c) {
    return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f) || c == 0x85 || c == 0xa0;
}

struct ParseOut {
    double* labels; int64_t* qid_span; double* X; int W; unsigned long long* info; int64_t* undecided; int cap;
};
// info[0] = width (largest fid + 1), info[1] = first error as (line << 8) | code, info[2] = undecided tokens

static __device__ __forceinline__ void note_undecided(const ParseOut& o, int64_t tok, int len, int64_t dest) {
    const unsigned long long k = atomicAdd(&o.info[2], 1ull);
    if (k < (unsigned long long)o.cap) {
        o.undecided[3 * k] = tok; o.undecided[3 * k + 1] = len; o.undecided[3 * k + 2] = dest;
    }
}

// One thread per line.  Scan mode (o.X == NULL) validates every token and writes label, qid span and width; fill mode
// writes the feature row (the last value of a repeated fid wins, as in data_utils.py:326).  Every read stays inside
// [line_start[i], line_start[i+1] - 1), every write inside row i of [n_lines, W].
__global__ void parse_lines_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ line_start,
                                   int64_t n_lines, int one_indexed, int has_comment, ParseOut o) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_lines) return;
    const bool fill = o.X != nullptr;
    const uint8_t* const t0 = text;
    const uint8_t* p = text + line_start[i];
    const uint8_t* e = text + line_start[i + 1] - 1;
    if (has_comment) for (const uint8_t* c = p; c < e; ++c) if (*c == '#') { e = c; break; }
    int err = E_NONE, width = 0, tok_index = 0;
    double label = 0.0;
    while (err == E_NONE) {
        while (p < e && is_space(*p)) ++p;
        if (p >= e) break;
        const uint8_t* s = p;
        while (p < e && !is_space(*p)) ++p;
        const int len = (int)(p - s);
        if (tok_index == 0) {
            if (!fill) {
                const DecResult d = parse_decimal((const char*)s, (const char*)p);
                if (d.status == LETOR_DEC_BAD) err = E_LABEL;
                label = d.value;
                if (d.status == LETOR_DEC_HOST) note_undecided(o, s - t0, len, -1 - i);
            }
        } else if (tok_index == 1) {
            if (len < 4 || s[0] != 'q' || s[1] != 'i' || s[2] != 'd' || s[3] != ':') err = E_QID;
            else if (!fill) { o.qid_span[2 * i] = (s + 4) - t0; o.qid_span[2 * i + 1] = len - 4; }
        } else {
            const uint8_t* c = s;
            bool negf = false;
            if (c < p && (*c == '+' || *c == '-')) { negf = *c == '-'; ++c; }
            int fid = 0, nd = 0;
            for (; c < p && *c >= '0' && *c <= '9'; ++c, ++nd) if (fid <= PTRB200_LETOR_MAX_FEATURES) fid = fid * 10 + (*c - '0');
            if (nd == 0 || c >= p || *c != ':') { err = E_TOKEN; break; }
            if (negf) fid = -fid;
            if (one_indexed) fid -= 1;
            if (fid < 0) { err = E_FID_LOW; break; }
            if (fid >= PTRB200_LETOR_MAX_FEATURES) { err = E_FID_HIGH; break; }
            width = max(width, fid + 1);
            const DecResult d = parse_decimal((const char*)c + 1, (const char*)p);
            if (d.status == LETOR_DEC_BAD) { err = E_TOKEN; break; }
            if (fill) {
                if (fid >= o.W) { err = E_FID_HIGH; break; }                     // W is the scan's width: cannot happen
                o.X[(size_t)i * o.W + fid] = d.value;
                if (d.status == LETOR_DEC_HOST) note_undecided(o, (c + 1) - t0, (int)(p - c - 1), (int64_t)i * o.W + fid);
            }
        }
        ++tok_index;
    }
    if (err == E_NONE) {
        if (tok_index == 0) err = E_EMPTY;
        else if (tok_index == 1) err = E_QID;
        else if (tok_index == 2) err = E_NO_FEATURES;
    }
    if (err != E_NONE) atomicMin(&o.info[1], ((unsigned long long)i << 8) | (unsigned long long)err);
    else if (!fill) { o.labels[i] = label; atomicMax(&o.info[0], (unsigned long long)width); }
}

// ---- grouping by qid -----------------------------------------------------------------------------------------------
static __device__ __forceinline__ uint64_t fnv1a(const uint8_t* s, int64_t len) {
    uint64_t h = 0xcbf29ce484222325ull;
    for (int64_t k = 0; k < len; ++k) { h ^= s[k]; h *= 0x100000001b3ull; }
    return h;
}
static __device__ __forceinline__ bool same_qid(const uint8_t* text, const int64_t* span, int64_t a, int64_t b) {
    const int64_t la = span[2 * a + 1];
    if (la != span[2 * b + 1]) return false;
    const uint8_t* x = text + span[2 * a];
    const uint8_t* y = text + span[2 * b];
    for (int64_t k = 0; k < la; ++k) if (x[k] != y[k]) return false;
    return true;
}

// open addressing, linear probing; rep[s] = some line holding the slot's qid, first[s] = its first line
__global__ void __launch_bounds__(256) qid_insert_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ span, int n_lines,
                                                         int32_t* __restrict__ rep, int32_t* __restrict__ first, uint32_t mask,
                                                         int32_t* __restrict__ line_slot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_lines) return;
    uint32_t s = (uint32_t)fnv1a(text + span[2 * i], span[2 * i + 1]) & mask;
    while (true) {
        const int r = atomicCAS(&rep[s], -1, i);
        if (r == -1 || same_qid(text, span, r, i)) break;
        s = (s + 1) & mask;                                  // the table holds >= 2 slots per line: never full
    }
    atomicMin(&first[s], i);
    line_slot[i] = (int32_t)s;
}

__global__ void __launch_bounds__(256) first_flag_kernel(const int32_t* __restrict__ line_slot, const int32_t* __restrict__ first, int n_lines,
                                                         int32_t* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_lines) flag[i] = first[line_slot[i]] == i;
}

// query index of every line (scan of the first-appearance flags), documents per query, and the longest query
__global__ void __launch_bounds__(256) line_query_kernel(const int32_t* __restrict__ line_slot, const int32_t* __restrict__ first,
                                                         const int32_t* __restrict__ first_rank, int n_lines, int32_t* __restrict__ line_query,
                                                         int32_t* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_lines) return;
    const int q = first_rank[first[line_slot[i]]];
    line_query[i] = q;
    atomicAdd(&counts[q], 1);
}

__global__ void __launch_bounds__(256) max_kernel(const int32_t* __restrict__ v, int n, int32_t* __restrict__ out) {
    int m = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = max(m, v[i]);
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void __launch_bounds__(256) scatter_lines_kernel(const int32_t* __restrict__ line_query, const int32_t* __restrict__ offsets,
                                                            int n_lines, int32_t* __restrict__ fill, int32_t* __restrict__ lines) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_lines) return;
    const int q = line_query[i];
    lines[offsets[q] + atomicAdd(&fill[q], 1)] = i;
}

// each query's lines back into file order (the scatter above is unordered): one CTA per query, bitonic sort
__global__ void sort_query_lines_kernel(const int32_t* __restrict__ offsets, int32_t* __restrict__ lines) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    const int base = offsets[blockIdx.x], n = offsets[blockIdx.x + 1] - base;
    if (n <= 1) return;
    const int npow2 = next_pow2(n);
    for (int k = threadIdx.x; k < npow2; k += blockDim.x)
        keys[k] = k < n ? (u64)(0xffffffffu - (uint32_t)lines[base + k]) : 0ull;      // descending keys = ascending lines
    block_sort_desc(keys, npow2);
    for (int k = threadIdx.x; k < n; k += blockDim.x) lines[base + k] = (int32_t)(0xffffffffu - (uint32_t)keys[k]);
}

// ---- labels, clipping, kept queries --------------------------------------------------------------------------------
// One CTA per query: labels in grouped order as fp32 (for the tie shuffle), documents kept per query (0 if dropped)
__global__ void __launch_bounds__(256) query_labels_kernel(const double* __restrict__ labels, const int32_t* __restrict__ lines,
                                                           const int32_t* __restrict__ offsets, ptrb200_letor_cfg cfg,
                                                           float* __restrict__ y, int32_t* __restrict__ kept_docs,
                                                           int32_t* __restrict__ kept) {
    __shared__ float red[33];
    const int base = offsets[blockIdx.x], n = offsets[blockIdx.x + 1] - base;
    float pos = 0.0f;
    for (int r = threadIdx.x; r < n; r += blockDim.x) {
        double v = labels[lines[base + r]];
        if (cfg.rank_labels) v = (double)n - v;                          // MSLETOR_LIST: rank position -> grade
        if (cfg.binary_rele) v = fmin(fmax(v, -10.0), 1.0);              // np.clip(a_min=-10, a_max=1)
        if (cfg.unknown_as_zero) v = fmin(fmax(v, 0.0), 10.0);           // np.clip(a_min=0, a_max=10)
        pos += v > 0.0 ? 1.0f : 0.0f;
        y[base + r] = (float)v;
    }
    pos = block_sum(pos, red);
    if (threadIdx.x == 0) {
        const bool keep = !(n < cfg.min_docs || (int)pos < cfg.min_rele);
        kept_docs[blockIdx.x] = keep ? n : 0;
        kept[blockIdx.x] = keep ? 1 : 0;
    }
}

// ---- scaling and the final gather ----------------------------------------------------------------------------------
static __device__ __forceinline__ void store_feat(float* X, size_t k, float v) { X[k] = v; }
static __device__ __forceinline__ void store_feat(uint16_t* X, size_t k, float v) { X[k] = __bfloat16_as_ushort(__float2bfloat16_rn(v)); }

// One CTA per kept query, thread per column.  Scaling in float64 with a fixed per-column order (rows ascending):
//   StandardScaler: mean = sum/n, var = (sum d^2 - (sum d)^2 / n) / n with d = x - mean (sklearn's
//                   _incremental_mean_and_var from zero), scale 1 where var <= n eps var + (n mean eps)^2, (x - mean) / scale;
//   MinMaxScaler:   s = 1 / range (range < 10 eps counts as 1), m = 0 - min * s, x * s + m -- sklearn's two roundings;
// Istella clip min(x, 1e6) first.  Rows come out in presort order when `order` is given.
template <typename OutT>
__global__ void __launch_bounds__(256) gather_kernel(const double* __restrict__ X64, int W, const int32_t* __restrict__ lines,
                                                     const int32_t* __restrict__ offsets, const int32_t* __restrict__ kept_docs,
                                                     const int32_t* __restrict__ kept_rank, const int32_t* __restrict__ out_base,
                                                     const int32_t* __restrict__ order, const float* __restrict__ y, ptrb200_letor_cfg cfg,
                                                     OutT* __restrict__ Xout, float* __restrict__ yout, int32_t* __restrict__ out_offsets) {
    const int b = blockIdx.x;
    if (kept_docs[b] == 0) return;
    const int base = offsets[b], n = offsets[b + 1] - base, ob = out_base[b];
    if (threadIdx.x == 0) { out_offsets[kept_rank[b]] = ob; out_offsets[kept_rank[b] + 1] = ob + n; }
    for (int r = threadIdx.x; r < n; r += blockDim.x) yout[ob + r] = y[base + (order ? order[base + r] : r)];
    const double eps = 2.220446049250313e-16;
    const bool clip = cfg.clip_istella && cfg.scaler != PTRB200_LETOR_NONE;
    for (int f = threadIdx.x; f < W; f += blockDim.x) {
        double a = 0.0, c = 1.0;             // standard: (x - a) / c;  min-max: x * c + a
        if (cfg.scaler == PTRB200_LETOR_STANDARD) {
            double s = 0.0;
            for (int r = 0; r < n; ++r) { double v = X64[(size_t)lines[base + r] * W + f]; if (clip) v = fmin(v, 1e6); s += v; }
            const double mean = s / n;
            double corr = 0.0, q = 0.0;
            for (int r = 0; r < n; ++r) {
                double v = X64[(size_t)lines[base + r] * W + f];
                if (clip) v = fmin(v, 1e6);
                const double d = v - mean;
                corr += d;
                q = __dadd_rn(q, __dmul_rn(d, d));
            }
            const double var = (q - corr * corr / n) / n;
            const double nm = n * mean * eps;
            a = mean;
            c = var <= n * eps * var + nm * nm ? 1.0 : sqrt(var);
        } else if (cfg.scaler == PTRB200_LETOR_MINMAX) {
            double lo = INFINITY, hi = -INFINITY;
            for (int r = 0; r < n; ++r) {
                double v = X64[(size_t)lines[base + r] * W + f];
                if (clip) v = fmin(v, 1e6);
                lo = fmin(lo, v); hi = fmax(hi, v);
            }
            double range = hi - lo;
            if (range < 10.0 * eps) range = 1.0;
            c = 1.0 / range;
            a = 0.0 - __dmul_rn(lo, c);
        }
        for (int r = 0; r < n; ++r) {
            double v = X64[(size_t)lines[base + (order ? order[base + r] : r)] * W + f];
            if (clip) v = fmin(v, 1e6);
            if (cfg.scaler == PTRB200_LETOR_STANDARD) v = (v - a) / c;
            else if (cfg.scaler == PTRB200_LETOR_MINMAX) v = __dadd_rn(__dmul_rn(v, c), a);
            store_feat(Xout, (size_t)(ob + r) * W + f, (float)v);
        }
    }
}

static int parse_error(const char* who, unsigned long long key) {
    const long long line = (long long)(key >> 8) + 1;
    set_error("%s: line %lld: %s", who, line, parse_error_text((int)(key & 0xff)));
    return PTRB200_ERR_INVALID;
}

static int grid_of(int64_t n, int t) { return (int)((n + t - 1) / t); }

}  // namespace ptrb200

using namespace ptrb200;

extern "C" int64_t ptrb200_letor_index_workspace_bytes(int64_t nbytes) {
    const int64_t chunks = (nbytes + kChunk - 1) / kChunk;
    return 4 * (chunks + scan_sums_len(chunks) + 2);
}

extern "C" int ptrb200_letor_count_lines(const uint8_t* text, int64_t nbytes, void* workspace, int64_t* n_lines_host,
                                         ptrb200_stream_t stream) {
    if (!text || !workspace || !n_lines_host || nbytes <= 0) { set_error("letor_count_lines: empty input or null pointer"); return PTRB200_ERR_INVALID; }
    const cudaStream_t st = (cudaStream_t)stream;
    const int64_t chunks = (nbytes + kChunk - 1) / kChunk;
    if (chunks > 0x7fffffff) { set_error("letor_count_lines: file too large"); return PTRB200_ERR_UNSUPPORTED; }
    int32_t* counts = (int32_t*)workspace;
    int32_t* sums = counts + chunks;
    int32_t* total = sums + scan_sums_len(chunks);
    PTRB200_LAUNCH(count_newlines_kernel, (unsigned)chunks, 256, 0, st, text, nbytes, counts);
    int rc = exclusive_scan(counts, chunks, counts, sums, total, st);
    if (rc) return rc;
    int32_t nl = 0;
    uint8_t last = 0;
    if (cudaMemcpyAsync(&nl, total, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(&last, text + nbytes - 1, 1, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) return check_launch("letor_count_lines");
    *n_lines_host = (int64_t)nl + (last != '\n');
    if (*n_lines_host >= 0x7fffffff) { set_error("letor_count_lines: more than 2^31 - 2 lines"); return PTRB200_ERR_UNSUPPORTED; }
    return PTRB200_OK;
}

extern "C" int ptrb200_letor_index_lines(const uint8_t* text, int64_t nbytes, const void* workspace, int64_t n_lines,
                                         int64_t* line_start, ptrb200_stream_t stream) {
    if (!text || !workspace || !line_start || nbytes <= 0 || n_lines <= 0) { set_error("letor_index_lines: bad arguments"); return PTRB200_ERR_INVALID; }
    const int64_t chunks = (nbytes + kChunk - 1) / kChunk;
    PTRB200_LAUNCH(line_starts_kernel, (unsigned)chunks, 256, 0, stream, text, nbytes, (const int32_t*)workspace, line_start, n_lines);
    return check_launch("letor_index_lines");
}

extern "C" int ptrb200_letor_parse(const uint8_t* text, const int64_t* line_start, int64_t n_lines, int one_indexed, int has_comment,
                                   double* labels, int64_t* qid_span, double* X, int W, int64_t* undecided, int undecided_cap,
                                   unsigned long long* info, unsigned long long* info_host, ptrb200_stream_t stream) {
    if (!text || !line_start || !info || !info_host || n_lines <= 0 || undecided_cap < 0 || (undecided_cap && !undecided) ||
        (!X && (!labels || !qid_span)) || (X && (W <= 0 || W > PTRB200_LETOR_MAX_FEATURES))) {
        set_error("letor_parse: bad arguments"); return PTRB200_ERR_INVALID;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const unsigned long long init[3] = {0ull, ~0ull, 0ull};
    if (cudaMemcpyAsync(info, init, sizeof(init), cudaMemcpyHostToDevice, st) != cudaSuccess) return check_launch("letor_parse");
    if (X && cudaMemsetAsync(X, 0, (size_t)n_lines * W * sizeof(double), st) != cudaSuccess) return check_launch("letor_parse");
    ParseOut o{labels, qid_span, X, W, info, undecided, undecided_cap};
    PTRB200_LAUNCH(parse_lines_kernel, grid_of(n_lines, 128), 128, 0, st, text, line_start, n_lines, one_indexed, has_comment, o);
    int rc = check_launch("letor_parse");
    if (rc) return rc;
    if (cudaMemcpyAsync(info_host, info, sizeof(init), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return check_launch("letor_parse");
    if (info_host[1] != ~0ull) return parse_error("letor_parse", info_host[1]);
    return PTRB200_OK;
}

extern "C" int64_t ptrb200_letor_group_workspace_bytes(int64_t n_lines) {
    const int64_t slots = next_pow2((int)(2 * n_lines));
    return 4 * (2 * slots + 3 * n_lines + 2 * scan_sums_len(n_lines) + 8);
}

extern "C" int ptrb200_letor_group(const uint8_t* text, const int64_t* qid_span, int64_t n_lines, void* workspace,
                                   int32_t* lines, int32_t* offsets, int32_t* counts, int max_queries, int* stats_host,
                                   ptrb200_stream_t stream) {
    if (!text || !qid_span || !workspace || !lines || !stats_host || n_lines <= 0 || n_lines > (1 << 29)) {
        set_error("letor_group: bad arguments (n_lines=%lld)", (long long)n_lines); return PTRB200_ERR_INVALID;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const int n = (int)n_lines;
    const int64_t slots = next_pow2(2 * n);
    int32_t* rep = (int32_t*)workspace;
    int32_t* first = rep + slots;
    int32_t* line_slot = first + slots;
    int32_t* flag = line_slot + n;
    int32_t* line_query = flag + n;
    int32_t* sums = line_query + n;
    int32_t* scalars = sums + 2 * scan_sums_len(n);           // [0] queries, [1] longest query, [2] total
    if (cudaMemsetAsync(rep, 0xff, slots * 4, st) != cudaSuccess || cudaMemsetAsync(first, 0x7f, slots * 4, st) != cudaSuccess ||
        cudaMemsetAsync(scalars, 0, 32, st) != cudaSuccess) return check_launch("letor_group");
    PTRB200_LAUNCH(qid_insert_kernel, grid_of(n, 256), 256, 0, st, text, qid_span, n, rep, first, (uint32_t)(slots - 1), line_slot);
    PTRB200_LAUNCH(first_flag_kernel, grid_of(n, 256), 256, 0, st, line_slot, first, n, flag);
    int rc = exclusive_scan(flag, n, flag, sums, scalars, st);
    if (rc) return rc;
    if (!offsets || !counts) {                                  // sizing call: queries and the longest query
        if (cudaMemcpyAsync(stats_host, scalars, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return check_launch("letor_group");
        return PTRB200_OK;
    }
    const int B = max_queries;
    if (cudaMemsetAsync(counts, 0, (size_t)B * 4, st) != cudaSuccess) return check_launch("letor_group");
    PTRB200_LAUNCH(line_query_kernel, grid_of(n, 256), 256, 0, st, line_slot, first, flag, n, line_query, counts);
    PTRB200_LAUNCH(max_kernel, min(grid_of(B, 256), 1024), 256, 0, st, counts, B, scalars + 1);
    rc = exclusive_scan(counts, B, offsets, sums, scalars + 2, st);
    if (rc) return rc;
    if (cudaMemcpyAsync(offsets + B, scalars + 2, 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(counts, 0, (size_t)B * 4, st) != cudaSuccess) return check_launch("letor_group");
    PTRB200_LAUNCH(scatter_lines_kernel, grid_of(n, 256), 256, 0, st, line_query, offsets, n, counts, lines);
    if (cudaMemcpyAsync(stats_host + 1, scalars + 1, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return check_launch("letor_group");
    if (stats_host[1] > PTRB200_MAX_LIST_LEN) {
        set_error("letor_group: a query has %d documents, above PTRB200_MAX_LIST_LEN=%d", stats_host[1], PTRB200_MAX_LIST_LEN);
        return PTRB200_ERR_UNSUPPORTED;
    }
    const int npow2 = next_pow2(stats_host[1]);
    PTRB200_LAUNCH(sort_query_lines_kernel, B, block_threads(npow2 / 2), (size_t)npow2 * 8, st, offsets, lines);
    return check_launch("letor_group");
}

extern "C" int ptrb200_letor_select(const double* labels, const int32_t* lines, const int32_t* offsets, int B, int max_len,
                                    const ptrb200_letor_cfg* cfg, float* y, int32_t* kept_docs, int32_t* kept, int32_t* out_base,
                                    int32_t* order, int32_t* scan_tmp, int* stats_host, ptrb200_stream_t stream) {
    if (!labels || !lines || !offsets || !cfg || !y || !kept_docs || !kept || !out_base || !scan_tmp || !stats_host || B <= 0 ||
        max_len <= 0 || max_len > PTRB200_MAX_LIST_LEN) {
        set_error("letor_select: bad arguments"); return PTRB200_ERR_INVALID;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    PTRB200_LAUNCH(query_labels_kernel, B, 256, 0, st, labels, lines, offsets, *cfg, y, kept_docs, kept);
    int32_t* sums = scan_tmp;
    int32_t* totals = sums + scan_sums_len(B);                 // [0] kept documents, [1] kept queries
    int rc = exclusive_scan(kept_docs, B, out_base, sums, totals, st);
    if (rc) return rc;
    rc = exclusive_scan(kept, B, kept, sums, totals + 1, st);   // kept[b] -> rank of query b among the kept ones
    if (rc) return rc;
    if (order) {
        rc = ptrb200_shuffle_ties_perm(y, offsets, order, B, max_len, cfg->seed, 0ull, stream);
        if (rc) return rc;
    }
    if (cudaMemcpyAsync(stats_host, totals, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return check_launch("letor_select");
    return PTRB200_OK;
}

extern "C" int ptrb200_letor_gather(const double* X64, int W, const int32_t* lines, const int32_t* offsets, int B,
                                    const int32_t* kept_docs, const int32_t* kept_rank, const int32_t* out_base, const int32_t* order,
                                    const float* y, const ptrb200_letor_cfg* cfg, void* X, int dtype, float* y_out,
                                    int32_t* out_offsets, ptrb200_stream_t stream) {
    if (!X64 || !lines || !offsets || !kept_docs || !kept_rank || !out_base || !y || !cfg || !X || !y_out || !out_offsets ||
        B <= 0 || W <= 0 || W > PTRB200_LETOR_MAX_FEATURES || (dtype != PTRB200_DTYPE_F32 && dtype != PTRB200_DTYPE_BF16) ||
        cfg->scaler < PTRB200_LETOR_NONE || cfg->scaler > PTRB200_LETOR_MINMAX) {
        set_error("letor_gather: bad arguments"); return PTRB200_ERR_INVALID;
    }
    const int threads = W >= 256 ? 256 : ((W + 31) / 32) * 32;
    if (dtype == PTRB200_DTYPE_F32)
        PTRB200_LAUNCH_TAG("letor_gather_kernel", gather_kernel<float>, B, threads, 0, stream, X64, W, lines, offsets, kept_docs, kept_rank,
                           out_base, order, y, *cfg, (float*)X, y_out, out_offsets);
    else
        PTRB200_LAUNCH_TAG("letor_gather_bf16_kernel", gather_kernel<uint16_t>, B, threads, 0, stream, X64, W, lines, offsets, kept_docs,
                           kept_rank, out_base, order, y, *cfg, (uint16_t*)X, y_out, out_offsets);
    return check_launch("letor_gather");
}
