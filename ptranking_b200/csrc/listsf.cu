// listsf.cu -- LayerNorm and elementwise glue of the multi-head self-attention list scorer (fp32 SIMT).
//
// Reference functions replaced (wildltr/ptranking @ f1d366c):
//   LayerNorm.forward           ptranking/base/list_ranker.py:152-174  (unbiased std, eps added to the std)
//   DASALC latent cross / AttnDIN / AllRank residual glue  list_ranker.py:138-149, 357-373
// and the autograd graph PyTorch builds for them.  reduce_rows_kernel sums LayerNorm's per-CTA parameter-gradient
// partials.  The attention core runs on tensor cores (attention_tc.cu); the Linear projections (the fused Q|K|V
// projection, fc) run through the stacked-FF kernels (ffnet.cu / ffnet_tc.cuh).
#include "common.cuh"
#include "ffnet_act.cuh"

namespace ptrb200 {

// ---------------------------------------------------------------- reference LayerNorm (warp per row)
// y = a (x - mean) / (std_unbiased + eps) + b
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ a2, const float* __restrict__ b2,
                                     float* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ std_out,
                                     int rows, int F, float eps) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* xr = x + (size_t)row * F;
    float s = 0.0f;
    for (int c = lane; c < F; c += 32) s += xr[c];
    const float mu = warp_sum(s) / F;
    float v = 0.0f;
    for (int c = lane; c < F; c += 32) { const float d = xr[c] - mu; v = fmaf(d, d, v); }
    const float sd = sqrtf(warp_sum(v) / (float)(F - 1));
    const float inv = 1.0f / (sd + eps);
    for (int c = lane; c < F; c += 32) y[(size_t)row * F + c] = a2[c] * (xr[c] - mu) * inv + b2[c];
    if (lane == 0) { mean_out[row] = mu; std_out[row] = sd; }
}

// dx, and per-CTA partials of da2 / db2 (summed by reduce afterwards).  Lane `l` of every warp owns columns
// l, l+32, ...; warps are combined in fixed order through shared memory (deterministic).  F <= 32*LN_MAX_COLS.
constexpr int LN_MAX_COLS = 16;
__global__ void layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ a2, const float* __restrict__ dy,
                                     const float* __restrict__ mean, const float* __restrict__ stdv,
                                     float* __restrict__ dx, float* __restrict__ partials /* [gridDim.x, 2, F] */,
                                     int rows, int F, float eps) {
    extern __shared__ float acc[];           // [warps][2][F]
    const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float ga[LN_MAX_COLS], gb[LN_MAX_COLS];
#pragma unroll
    for (int t = 0; t < LN_MAX_COLS; ++t) { ga[t] = 0.0f; gb[t] = 0.0f; }
    for (int row = blockIdx.x * wpb + warp; row < rows; row += gridDim.x * wpb) {
        const float mu = mean[row], sd = stdv[row], s = sd + eps;
        const float* xr = x + (size_t)row * F;
        const float* gr = dy + (size_t)row * F;
        float s0 = 0.0f, s1 = 0.0f;
        for (int c = lane; c < F; c += 32) { const float d0 = gr[c] * a2[c]; s0 += d0; s1 = fmaf(d0, xr[c] - mu, s1); }
        s0 = warp_sum(s0); s1 = warp_sum(s1);
        const float m0 = s0 / F;
        const float k = sd > 0.0f ? s1 / (s * s * sd * (float)(F - 1)) : 0.0f;
#pragma unroll
        for (int t = 0; t < LN_MAX_COLS; ++t) {
            const int c = lane + 32 * t;
            if (c < F) {
                const float cen = xr[c] - mu, d0 = gr[c] * a2[c];
                dx[(size_t)row * F + c] = (d0 - m0) / s - cen * k;
                ga[t] += gr[c] * cen / s;
                gb[t] += gr[c];
            }
        }
    }
#pragma unroll
    for (int t = 0; t < LN_MAX_COLS; ++t) {
        const int c = lane + 32 * t;
        if (c < F) { acc[((size_t)warp * 2) * F + c] = ga[t]; acc[((size_t)warp * 2 + 1) * F + c] = gb[t]; }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < 2 * F; c += blockDim.x) {
        float v = 0.0f;
        for (int w = 0; w < wpb; ++w) v += acc[(size_t)w * 2 * F + c];
        partials[(size_t)blockIdx.x * 2 * F + c] = v;
    }
}

__global__ void reduce_rows_kernel(const float* __restrict__ partials, float* __restrict__ out, int splits, int count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    float s = 0.0f;
    for (int p = 0; p < splits; ++p) s += partials[(size_t)p * count + i];
    out[i] = s;
}

// ---------------------------------------------------------------- elementwise glue
enum { EW_ADD = 0, EW_LATENT_CROSS = 1, EW_MUL = 2, EW_RELU = 3, EW_RELU_BWD = 4, EW_DROPOUT = 5, EW_SCALE_ADD1 = 6, EW_MUL_SCALAR = 7, EW_ACT = 8, EW_ACT_GRAD = 9 };
// out = a + b | (a + 1) * b | a * b | relu(a) | (b > 0) ? a : 0 | dropout(a) | a*(b+1) | a * b[0]
__global__ void elementwise_kernel(int op, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                                   size_t n, DropCfg drop) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float v;
        switch (op) {
            case EW_ADD: v = a[i] + b[i]; break;
            case EW_LATENT_CROSS: v = (a[i] + 1.0f) * b[i]; break;
            case EW_MUL: v = a[i] * b[i]; break;
            case EW_RELU: v = fmaxf(a[i], 0.0f); break;
            case EW_RELU_BWD: v = b[i] > 0.0f ? a[i] : 0.0f; break;
            case EW_DROPOUT: v = (!drop.thr || dropout_keep(drop.key, i, drop.thr)) ? a[i] * drop.scale : 0.0f; break;
            case EW_MUL_SCALAR: v = a[i] * b[0]; break;
            case EW_ACT: v = activate((int)drop.thr, a[i]).y; break;          // activation code travels in drop.thr
            case EW_ACT_GRAD: v = activate((int)drop.thr, a[i]).dy; break;
            default: v = a[i] * (b[i] + 1.0f); break;
        }
        out[i] = v;
    }
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_layernorm_fwd(const float* x, const float* a2, const float* b2, float* y, float* mean, float* stdv,
                          int rows, int F, float eps, ptrb200_stream_t stream) {
    if (!x || !a2 || !b2 || !y || !mean || !stdv || rows <= 0 || F <= 1) { set_error("layernorm_fwd: bad arguments"); return PTRB200_ERR_INVALID; }
    PTRB200_LAUNCH(layernorm_fwd_kernel, (rows + 7) / 8, 256, 0, stream, x, a2, b2, y, mean, stdv, rows, F, eps);
    return check_launch("layernorm_fwd");
}

int ptrb200_layernorm_bwd(const float* x, const float* a2, const float* dy, const float* mean, const float* stdv,
                          float* dx, float* da2, float* db2, float* scratch /* 296*2*F floats */,
                          int rows, int F, float eps, ptrb200_stream_t stream) {
    if (!x || !a2 || !dy || !mean || !stdv || !dx || !da2 || !db2 || !scratch || rows <= 0 || F <= 1) { set_error("layernorm_bwd: bad arguments"); return PTRB200_ERR_INVALID; }
    int grid = (rows + 7) / 8; if (grid > 296) grid = 296;
    if (F > 32 * LN_MAX_COLS) { set_error("layernorm_bwd: F=%d > %d", F, 32 * LN_MAX_COLS); return PTRB200_ERR_UNSUPPORTED; }
    PTRB200_LAUNCH(layernorm_bwd_kernel, grid, 256, (size_t)8 * 2 * F * 4, stream, x, a2, dy, mean, stdv, dx, scratch, rows, F, eps);
    // partial layout [grid][2][F]: da2 = sum over grid of [0][:], db2 = of [1][:]; reduce both with one strided pass each
    PTRB200_LAUNCH(reduce_rows_kernel, (2 * F + 255) / 256, 256, 0, stream, (const float*)scratch, scratch + (size_t)296 * 2 * F, grid, 2 * F);
    cudaMemcpyAsync(da2, scratch + (size_t)296 * 2 * F, (size_t)F * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    cudaMemcpyAsync(db2, scratch + (size_t)296 * 2 * F + F, (size_t)F * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    return check_launch("layernorm_bwd");
}

int ptrb200_elementwise(int op, const float* a, const float* b, float* out, int64_t count,
                        float dropout_p, uint64_t seed, uint64_t offset, ptrb200_stream_t stream) {
    if (!a || !out || count <= 0 || op < EW_ADD || op > EW_ACT_GRAD) { set_error("elementwise: bad arguments"); return PTRB200_ERR_INVALID; }
    if (!b && op != EW_RELU && op != EW_DROPOUT && op != EW_ACT && op != EW_ACT_GRAD) { set_error("elementwise: op %d needs two inputs", op); return PTRB200_ERR_INVALID; }
    size_t blocks = ((size_t)count + 255) / 256; if (blocks > (size_t)num_sms() * 16) blocks = (size_t)num_sms() * 16;
    DropCfg dc = make_drop_call(dropout_p, seed, offset);
    if (op == EW_ACT || op == EW_ACT_GRAD) dc.thr = (uint32_t)seed;           // seed = PTRB200_AF_* code
    PTRB200_LAUNCH(elementwise_kernel, (unsigned)blocks, 256, 0, stream, op, a, b, out, (size_t)count, dc);
    return check_launch("elementwise");
}

}  // extern "C"
