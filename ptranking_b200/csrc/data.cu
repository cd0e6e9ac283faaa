// data.cu -- the input side of the hot path on the device (SURVEY 8f-2).
//
// Reference functions replaced (wildltr/ptranking @ f1d366c):
//   per-query feature scaling  ptranking/data/data_utils.py:482-487 (sklearn StandardScaler().fit_transform per query,
//                              ISTELLA clip at :484-485; which datasets are scaled: :205-218)
#include <cuda_bf16.h>

#include "losses_common.cuh"

namespace ptrb200 {

// One CTA per query; thread t owns feature columns t, t+blockDim, ... so every row read is coalesced.
// sklearn semantics: mean over the query's documents, POPULATION variance (ddof = 0), both accumulated in float64
// (two passes: the variance is the mean squared deviation from the computed mean); a constant column -- variance not
// above sklearn's _is_constant_feature bound n*eps*var + (n*mean*eps)^2 -- is divided by 1 instead of 0.
// OutT = uint16_t: bf16 output, the fp32 result rounded to nearest even at the store.
static __device__ __forceinline__ float to_out(float v, float*) { return v; }
static __device__ __forceinline__ uint16_t to_out(float v, uint16_t*) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }

template <typename OutT>
__global__ void standard_scale_kernel(const float* __restrict__ X, const int32_t* __restrict__ offsets, OutT* __restrict__ out,
                                      int n_uniform, int F, float clip_max, int clip) {
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, n_uniform);
    const int n = sp.n;
    if (n == 0) return;
    const float* x = X + sp.base * (size_t)F;
    OutT* o = out + sp.base * (size_t)F;
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        double s = 0.0;
        for (int r = 0; r < n; ++r) { float v = x[(size_t)r * F + f]; if (clip) v = fminf(v, clip_max); s += (double)v; }
        const double mean = s / n;
        double q = 0.0;
        for (int r = 0; r < n; ++r) { float v = x[(size_t)r * F + f]; if (clip) v = fminf(v, clip_max); const double d = (double)v - mean; q += d * d; }
        const double var = q / n;
        const double eps = 2.220446049250313e-16;
        const double bound = n * eps * var + (n * mean * eps) * (n * mean * eps);
        const double scale = (var <= bound) ? 1.0 : sqrt(var);
        for (int r = 0; r < n; ++r) {
            float v = x[(size_t)r * F + f];
            if (clip) v = fminf(v, clip_max);
            o[(size_t)r * F + f] = to_out((float)(((double)v - mean) / scale), o);
        }
    }
}

// Ragged <-> padded: the list scorer's attention works on dense [B, n_max, .] tensors; a ragged batch (flat rows + prefix
// offsets) is padded on the way in (zeros behind each list) and the scores are gathered back on the way out.  One CTA
// per (query, row block).  Padded query b is query qidx[b] (b when qidx is NULL) of the prefix offsets; its rows are a
// column block of the flat rows, ld_src floats apart:
//   padded[b, r, 0:W] = src[(offsets[q] + r) * ld_src + 0:W] for r < len_q, 0 for len_q <= r < n_max
__global__ void pad_lists_kernel(const float* __restrict__ src, long long ld_src, const int32_t* __restrict__ offsets,
                                 const int32_t* __restrict__ qidx, float* __restrict__ dst, int n_max, int W) {
    const int b = blockIdx.x;
    const int q = qidx ? qidx[b] : b;
    const int base = offsets[q], n = min(offsets[q + 1] - base, n_max);
    for (int r = blockIdx.y; r < n_max; r += gridDim.y) {
        const float* s = src + (size_t)(base + r) * ld_src;
        float* d = dst + ((size_t)b * n_max + r) * W;
        const bool live = r < n;
        for (int f = threadIdx.x; f < W; f += blockDim.x) d[f] = live ? s[f] : 0.0f;
    }
}

// The inverse gather: flat[offsets[b] + r, 0:F] = padded[b, r, 0:F] for r < len_b; a list longer than n_max gives only
// the n_max rows its padded block holds.
__global__ void unpad_lists_kernel(const float* __restrict__ src, const int32_t* __restrict__ offsets, float* __restrict__ dst,
                                   int n_max, int F) {
    const int b = blockIdx.x;
    const int base = offsets[b], n = min(offsets[b + 1] - base, n_max);
    const size_t row_elems = (size_t)F;
    for (int r = blockIdx.y; r < n; r += gridDim.y) {
        const float* s = src + ((size_t)b * n_max + r) * row_elems;
        float* d = dst + (size_t)(base + r) * row_elems;
        for (int f = threadIdx.x; f < F; f += blockDim.x) d[f] = s[f];
    }
}

static inline int pad_lists_threads(int W) { return W >= 128 ? 128 : ((W + 31) / 32) * 32; }

}  // namespace ptrb200

using namespace ptrb200;

extern "C" int ptrb200_pad_lists(const float* src, long long ld_src, const int32_t* offsets, const int32_t* qidx, float* padded,
                                 int B, int n_max, int W, ptrb200_stream_t stream) {
    if (!src || !offsets || !padded || B <= 0 || n_max <= 0 || W <= 0 || ld_src < W) {
        set_error("pad_lists: bad arguments (B=%d n_max=%d W=%d ld_src=%lld)", B, n_max, W, ld_src);
        return PTRB200_ERR_INVALID;
    }
    PTRB200_LAUNCH(pad_lists_kernel, dim3(B, n_max < 64 ? n_max : 64), pad_lists_threads(W), 0, stream, src, ld_src, offsets,
                   qidx, padded, n_max, W);
    return check_launch("pad_lists");
}

extern "C" int ptrb200_unpad_lists(const float* padded, const int32_t* offsets, float* flat, int B, int n_max, int F,
                                   ptrb200_stream_t stream) {
    if (!flat || !offsets || !padded || B <= 0 || n_max <= 0 || F <= 0) { set_error("unpad_lists: bad arguments"); return PTRB200_ERR_INVALID; }
    PTRB200_LAUNCH(unpad_lists_kernel, dim3(B, n_max < 64 ? n_max : 64), pad_lists_threads(F), 0, stream, padded, offsets, flat, n_max, F);
    return check_launch("unpad_lists");
}

extern "C" int ptrb200_standard_scale(const float* X, const int32_t* offsets, void* out, int out_dtype, int B, int n, int F,
                                      int clip, float clip_max, ptrb200_stream_t stream) {
    if (!X || !out || B <= 0 || n <= 0 || F <= 0) { set_error("standard_scale: bad arguments (B=%d n=%d F=%d)", B, n, F); return PTRB200_ERR_INVALID; }
    int threads = ((F + 31) / 32) * 32; if (threads > 256) threads = 256;
    if (out_dtype == PTRB200_DTYPE_F32) {
        PTRB200_LAUNCH_TAG("standard_scale_kernel", standard_scale_kernel<float>, B, threads, 0, stream, X, offsets, static_cast<float*>(out), n, F, clip_max, clip);
    } else if (out_dtype == PTRB200_DTYPE_BF16) {
        if ((const void*)X == out) { set_error("standard_scale: a bf16 out must not alias X"); return PTRB200_ERR_INVALID; }
        PTRB200_LAUNCH_TAG("standard_scale_bf16_kernel", standard_scale_kernel<uint16_t>, B, threads, 0, stream, X, offsets, static_cast<uint16_t*>(out), n, F, clip_max, clip);
    } else {
        set_error("standard_scale: unknown out_dtype code %d", out_dtype);
        return PTRB200_ERR_INVALID;
    }
    return check_launch("standard_scale");
}
