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
static __device__ __forceinline__ void standard_scale_query(const float* __restrict__ X, const int32_t* __restrict__ offsets,
                                                            OutT* __restrict__ out, int n_uniform, int F, float clip_max, int clip) {
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
__global__ void standard_scale_kernel(const float* __restrict__ X, const int32_t* __restrict__ offsets, float* __restrict__ out,
                                      int n_uniform, int F, float clip_max, int clip) {
    standard_scale_query(X, offsets, out, n_uniform, F, clip_max, clip);
}
__global__ void standard_scale_bf16_kernel(const float* __restrict__ X, const int32_t* __restrict__ offsets, uint16_t* __restrict__ out,
                                           int n_uniform, int F, float clip_max, int clip) {
    standard_scale_query(X, offsets, out, n_uniform, F, clip_max, clip);
}

// Ragged <-> padded: the list scorer's attention works on dense [B, n_max, .] tensors; a ragged batch (flat rows + prefix
// offsets) is padded on the way in (zeros behind each list) and the scores are gathered back on the way out.  One CTA
// per (query, row block); rows are copied 16 bytes per thread when the width allows.
template <bool PAD>
__global__ void pad_lists_kernel(const float* __restrict__ src, const int32_t* __restrict__ offsets, float* __restrict__ dst,
                                 int n_max, int F) {
    const int b = blockIdx.x;
    const int base = offsets[b], n = offsets[b + 1] - base;
    const size_t row_elems = (size_t)F;
    for (int r = blockIdx.y; r < (PAD ? n_max : n); r += gridDim.y) {
        const float* s = PAD ? src + (size_t)(base + r) * row_elems : src + ((size_t)b * n_max + r) * row_elems;
        float* d = PAD ? dst + ((size_t)b * n_max + r) * row_elems : dst + (size_t)(base + r) * row_elems;
        const bool live = !PAD || r < n;
        for (int f = threadIdx.x; f < F; f += blockDim.x) d[f] = live ? s[f] : 0.0f;
    }
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" int ptrb200_pad_lists(const float* flat, const int32_t* offsets, float* padded, int B, int n_max, int F,
                                 ptrb200_stream_t stream) {
    if (!flat || !offsets || !padded || B <= 0 || n_max <= 0 || F <= 0) { set_error("pad_lists: bad arguments"); return PTRB200_ERR_INVALID; }
    const int threads = F >= 128 ? 128 : ((F + 31) / 32) * 32;
    PTRB200_LAUNCH_TAG("pad_lists_kernel", pad_lists_kernel<true>, dim3(B, n_max < 64 ? n_max : 64), threads, 0, stream, flat, offsets, padded, n_max, F);
    return check_launch("pad_lists");
}

extern "C" int ptrb200_unpad_lists(const float* padded, const int32_t* offsets, float* flat, int B, int n_max, int F,
                                   ptrb200_stream_t stream) {
    if (!flat || !offsets || !padded || B <= 0 || n_max <= 0 || F <= 0) { set_error("unpad_lists: bad arguments"); return PTRB200_ERR_INVALID; }
    const int threads = F >= 128 ? 128 : ((F + 31) / 32) * 32;
    PTRB200_LAUNCH_TAG("unpad_lists_kernel", pad_lists_kernel<false>, dim3(B, n_max < 64 ? n_max : 64), threads, 0, stream, padded, offsets, flat, n_max, F);
    return check_launch("unpad_lists");
}

extern "C" int ptrb200_standard_scale(const float* X, const int32_t* offsets, float* out, int B, int n, int F,
                                      int clip, float clip_max, ptrb200_stream_t stream) {
    if (!X || !out || B <= 0 || n <= 0 || F <= 0) { set_error("standard_scale: bad arguments (B=%d n=%d F=%d)", B, n, F); return PTRB200_ERR_INVALID; }
    int threads = ((F + 31) / 32) * 32; if (threads > 256) threads = 256;
    PTRB200_LAUNCH(standard_scale_kernel, B, threads, 0, stream, X, offsets, out, n, F, clip_max, clip);
    return check_launch("standard_scale");
}

extern "C" int ptrb200_standard_scale_bf16(const float* X, const int32_t* offsets, uint16_t* out, int B, int n, int F,
                                           int clip, float clip_max, ptrb200_stream_t stream) {
    if (!X || !out || B <= 0 || n <= 0 || F <= 0) { set_error("standard_scale_bf16: bad arguments (B=%d n=%d F=%d)", B, n, F); return PTRB200_ERR_INVALID; }
    if ((const void*)X == (const void*)out) { set_error("standard_scale_bf16: out must not alias X"); return PTRB200_ERR_INVALID; }
    int threads = ((F + 31) / 32) * 32; if (threads > 256) threads = 256;
    PTRB200_LAUNCH(standard_scale_bf16_kernel, B, threads, 0, stream, X, offsets, out, n, F, clip_max, clip);
    return check_launch("standard_scale_bf16");
}
