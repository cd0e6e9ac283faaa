// listsf.cu -- kernels of the multi-head self-attention list scorer (fp32 SIMT path).
//
// Reference functions replaced (wildltr/ptranking @ f1d366c):
//   MultiheadAttention.forward  ptranking/base/list_ranker.py:208-254  (softmax(QK^T/sqrt(d)) -> dropout -> .V)
//   LayerNorm.forward           ptranking/base/list_ranker.py:152-174  (unbiased std, eps added to the std)
//   DASALC latent cross / AttnDIN / AllRank residual glue  list_ranker.py:138-149, 357-373
// and the autograd graph PyTorch builds for them.  The Linear projections (w_q, w_k, w_v, fc) run through
// the stacked-FF kernels (ffnet.cu / ffnet_tc.cuh).
//
// Attention is evaluated flash-style: one thread owns one query row (q, running max / sum and the
// output accumulator live in registers), keys/values stream through shared memory in tiles, and the
// [n,n] probability matrix is never written to HBM; the backward pass rebuilds probabilities from the
// saved per-row log-sum-exp.  Q, K, V, O are the [B, n, H*D] projection outputs, head h = columns
// [h*D, (h+1)*D) -- the reference's view/permute (list_ranker.py:222-224) is pure indexing here.
#include "common.cuh"
#include "ffnet_act.cuh"

namespace ptrb200 {

constexpr int ATT_ROWS = 128;      // query rows (threads) per CTA
constexpr int ATT_KT = 32;         // keys per shared-memory tile

struct AttArgs {
    const float *Q, *K, *V;        // [B, n, H*D]
    float* O;                      // [B, n, H*D]
    float* LSE;                    // [B, H, n]  log-sum-exp of the scaled scores per query row
    int B, n, H, D;
    float inv_scale;               // 1 / sqrt(D)
    DropCfg drop;                  // dropout on the attention probabilities, element id ((b*H+h)*n + i)*n + j
};

template <int D>
__global__ void __launch_bounds__(ATT_ROWS) attention_fwd_kernel(AttArgs a) {
    __shared__ float ks[ATT_KT][D + 1];
    __shared__ float vs[ATT_KT][D + 1];
    const int bh = blockIdx.x, b = bh / a.H, h = bh % a.H;
    const int i = blockIdx.y * ATT_ROWS + threadIdx.x;
    const int ld = a.H * D;
    const bool live = i < a.n;
    float q[D], o[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { q[d] = live ? a.Q[((size_t)b * a.n + i) * ld + h * D + d] * a.inv_scale : 0.0f; o[d] = 0.0f; }
    float m = -INFINITY, l = 0.0f;
    for (int j0 = 0; j0 < a.n; j0 += ATT_KT) {
        __syncthreads();
        for (int e = threadIdx.x; e < ATT_KT * D; e += ATT_ROWS) {
            const int jj = e / D, d = e % D, j = j0 + jj;
            ks[jj][d] = j < a.n ? a.K[((size_t)b * a.n + j) * ld + h * D + d] : 0.0f;
            vs[jj][d] = j < a.n ? a.V[((size_t)b * a.n + j) * ld + h * D + d] : 0.0f;
        }
        __syncthreads();
        const int jn = min(ATT_KT, a.n - j0);
        for (int jj = 0; jj < jn; ++jj) {
            float s = 0.0f;
#pragma unroll
            for (int d = 0; d < D; ++d) s = fmaf(q[d], ks[jj][d], s);
            const float mn = fmaxf(m, s);
            const float corr = expf(m - mn), p = expf(s - mn);
            l = l * corr + p;
            float pd = p;
            if (a.drop.thr) {
                const uint64_t e = ((uint64_t)bh * a.n + i) * a.n + (j0 + jj);
                pd = dropout_keep(a.drop.key, e, a.drop.thr) ? p * a.drop.scale : 0.0f;
            }
#pragma unroll
            for (int d = 0; d < D; ++d) o[d] = fmaf(pd, vs[jj][d], o[d] * corr);
            m = mn;
        }
    }
    if (live) {
        const float inv = 1.0f / l;
#pragma unroll
        for (int d = 0; d < D; ++d) a.O[((size_t)b * a.n + i) * ld + h * D + d] = o[d] * inv;
        a.LSE[(size_t)bh * a.n + i] = m + logf(l);
    }
}

struct AttBwdArgs {
    const float *Q, *K, *V, *O, *dO, *LSE;
    float *dQ, *dK, *dV;
    float* Dsum;                   // [B, H, n]  D_i = dO_i . O_i
    int B, n, H, D;
    float inv_scale;
    DropCfg drop;
};

// D_i = dO_i . O_i  (one thread per (b,h,i))
__global__ void attention_dsum_kernel(AttBwdArgs a) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)a.B * a.H * a.n) return;
    const int i = (int)(t % a.n), bh = (int)(t / a.n), b = bh / a.H, h = bh % a.H;
    const size_t off = ((size_t)b * a.n + i) * (a.H * a.D) + h * a.D;
    float s = 0.0f;
    for (int d = 0; d < a.D; ++d) s = fmaf(a.dO[off + d], a.O[off + d], s);
    a.Dsum[t] = s;
}

// dQ: thread per query row, stream keys/values
template <int D>
__global__ void __launch_bounds__(ATT_ROWS) attention_bwd_dq_kernel(AttBwdArgs a) {
    __shared__ float ks[ATT_KT][D + 1];
    __shared__ float vs[ATT_KT][D + 1];
    const int bh = blockIdx.x, b = bh / a.H, h = bh % a.H;
    const int i = blockIdx.y * ATT_ROWS + threadIdx.x;
    const int ld = a.H * D;
    const bool live = i < a.n;
    float q[D], g[D], dq[D];
    const size_t roff = ((size_t)b * a.n + (live ? i : 0)) * ld + h * D;
#pragma unroll
    for (int d = 0; d < D; ++d) { q[d] = live ? a.Q[roff + d] * a.inv_scale : 0.0f; g[d] = live ? a.dO[roff + d] : 0.0f; dq[d] = 0.0f; }
    const float lse = live ? a.LSE[(size_t)bh * a.n + i] : 0.0f;
    const float Di = live ? a.Dsum[(size_t)bh * a.n + i] : 0.0f;
    for (int j0 = 0; j0 < a.n; j0 += ATT_KT) {
        __syncthreads();
        for (int e = threadIdx.x; e < ATT_KT * D; e += ATT_ROWS) {
            const int jj = e / D, d = e % D, j = j0 + jj;
            ks[jj][d] = j < a.n ? a.K[((size_t)b * a.n + j) * ld + h * D + d] : 0.0f;
            vs[jj][d] = j < a.n ? a.V[((size_t)b * a.n + j) * ld + h * D + d] : 0.0f;
        }
        __syncthreads();
        const int jn = min(ATT_KT, a.n - j0);
        for (int jj = 0; jj < jn; ++jj) {
            float s = 0.0f, dp = 0.0f;
#pragma unroll
            for (int d = 0; d < D; ++d) { s = fmaf(q[d], ks[jj][d], s); dp = fmaf(g[d], vs[jj][d], dp); }
            const float p = expf(s - lse);
            if (a.drop.thr) {
                const uint64_t e = ((uint64_t)bh * a.n + i) * a.n + (j0 + jj);
                dp = dropout_keep(a.drop.key, e, a.drop.thr) ? dp * a.drop.scale : 0.0f;
            }
            const float ds = p * (dp - Di);
#pragma unroll
            for (int d = 0; d < D; ++d) dq[d] = fmaf(ds, ks[jj][d], dq[d]);
        }
    }
    if (live) {
#pragma unroll
        for (int d = 0; d < D; ++d) a.dQ[roff + d] = dq[d] * a.inv_scale;
    }
}

// dK, dV: thread per key row, stream queries
template <int D>
__global__ void __launch_bounds__(ATT_ROWS) attention_bwd_dkv_kernel(AttBwdArgs a) {
    __shared__ float qs[ATT_KT][D + 1];
    __shared__ float gs[ATT_KT][D + 1];
    __shared__ float ls[ATT_KT], dsm[ATT_KT];
    const int bh = blockIdx.x, b = bh / a.H, h = bh % a.H;
    const int j = blockIdx.y * ATT_ROWS + threadIdx.x;
    const int ld = a.H * D;
    const bool live = j < a.n;
    float k[D], v[D], dk[D], dv[D];
    const size_t roff = ((size_t)b * a.n + (live ? j : 0)) * ld + h * D;
#pragma unroll
    for (int d = 0; d < D; ++d) { k[d] = live ? a.K[roff + d] : 0.0f; v[d] = live ? a.V[roff + d] : 0.0f; dk[d] = 0.0f; dv[d] = 0.0f; }
    for (int i0 = 0; i0 < a.n; i0 += ATT_KT) {
        __syncthreads();
        for (int e = threadIdx.x; e < ATT_KT * D; e += ATT_ROWS) {
            const int ii = e / D, d = e % D, i = i0 + ii;
            qs[ii][d] = i < a.n ? a.Q[((size_t)b * a.n + i) * ld + h * D + d] * a.inv_scale : 0.0f;
            gs[ii][d] = i < a.n ? a.dO[((size_t)b * a.n + i) * ld + h * D + d] : 0.0f;
        }
        if (threadIdx.x < ATT_KT) {
            const int i = i0 + threadIdx.x;
            ls[threadIdx.x] = i < a.n ? a.LSE[(size_t)bh * a.n + i] : 0.0f;
            dsm[threadIdx.x] = i < a.n ? a.Dsum[(size_t)bh * a.n + i] : 0.0f;
        }
        __syncthreads();
        const int in = min(ATT_KT, a.n - i0);
        for (int ii = 0; ii < in; ++ii) {
            float s = 0.0f, dp = 0.0f;
#pragma unroll
            for (int d = 0; d < D; ++d) { s = fmaf(qs[ii][d], k[d], s); dp = fmaf(gs[ii][d], v[d], dp); }
            const float p = expf(s - ls[ii]);
            float pd = p;
            if (a.drop.thr) {
                const uint64_t e = ((uint64_t)bh * a.n + (i0 + ii)) * a.n + j;
                const bool keep = dropout_keep(a.drop.key, e, a.drop.thr);
                pd = keep ? p * a.drop.scale : 0.0f;
                dp = keep ? dp * a.drop.scale : 0.0f;
            }
            const float ds = p * (dp - dsm[ii]);
#pragma unroll
            for (int d = 0; d < D; ++d) { dv[d] = fmaf(pd, gs[ii][d], dv[d]); dk[d] = fmaf(ds, qs[ii][d], dk[d]); }
        }
    }
    if (live) {
#pragma unroll
        for (int d = 0; d < D; ++d) { a.dK[roff + d] = dk[d]; a.dV[roff + d] = dv[d]; }   // qs already carries 1/scale
    }
}

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

template <int D>
static void launch_att_fwd(const AttArgs& a, cudaStream_t st) {
    dim3 grid(a.B * a.H, (a.n + ATT_ROWS - 1) / ATT_ROWS);
    PTRB200_LAUNCH_TAG("attention_fwd", attention_fwd_kernel<D>, grid, ATT_ROWS, 0, st, a);
}
template <int D>
static void launch_att_bwd(const AttBwdArgs& a, cudaStream_t st) {
    dim3 grid(a.B * a.H, (a.n + ATT_ROWS - 1) / ATT_ROWS);
    PTRB200_LAUNCH_TAG("attention_bwd_dq", attention_bwd_dq_kernel<D>, grid, ATT_ROWS, 0, st, a);
    PTRB200_LAUNCH_TAG("attention_bwd_dkv", attention_bwd_dkv_kernel<D>, grid, ATT_ROWS, 0, st, a);
}
// One instantiation per supported head dimension (the accumulators are register arrays).
#define ATT_CASE(D_) case D_: CALL(D_); break;
#define ATT_DISPATCH(Dv)                                                                                  \
    switch (Dv) {                                                                                         \
        ATT_CASE(2) ATT_CASE(4) ATT_CASE(5) ATT_CASE(6) ATT_CASE(8) ATT_CASE(10) ATT_CASE(12) ATT_CASE(16) \
        ATT_CASE(17) ATT_CASE(20) ATT_CASE(23) ATT_CASE(24) ATT_CASE(32) ATT_CASE(34) ATT_CASE(40)        \
        ATT_CASE(46) ATT_CASE(48) ATT_CASE(50) ATT_CASE(64) ATT_CASE(68) ATT_CASE(72) ATT_CASE(96) ATT_CASE(100) \
        default: set_error("attention: head dimension %d is not instantiated", Dv); return PTRB200_ERR_UNSUPPORTED; \
    }

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_attention_fwd(const float* Q, const float* K, const float* V, float* O, float* LSE,
                          int B, int n, int H, int D, float dropout_p, uint64_t seed, uint64_t offset,
                          ptrb200_stream_t stream) {
    if (!Q || !K || !V || !O || !LSE || B <= 0 || n <= 0 || H <= 0 || D <= 0) { set_error("attention_fwd: bad arguments"); return PTRB200_ERR_INVALID; }
    AttArgs a{Q, K, V, O, LSE, B, n, H, D, 1.0f / sqrtf((float)D), make_drop(dropout_p, seed, offset)};
    cudaStream_t st = (cudaStream_t)stream;
#define CALL(DD) launch_att_fwd<DD>(a, st)
    ATT_DISPATCH(D)
#undef CALL
    return check_launch("attention_fwd");
}

int ptrb200_attention_bwd(const float* Q, const float* K, const float* V, const float* O, const float* dO, const float* LSE,
                          float* dQ, float* dK, float* dV, float* scratch /* B*H*n floats */,
                          int B, int n, int H, int D, float dropout_p, uint64_t seed, uint64_t offset,
                          ptrb200_stream_t stream) {
    if (!Q || !K || !V || !O || !dO || !LSE || !dQ || !dK || !dV || !scratch || B <= 0 || n <= 0 || H <= 0 || D <= 0) { set_error("attention_bwd: bad arguments"); return PTRB200_ERR_INVALID; }
    AttBwdArgs a{Q, K, V, O, dO, LSE, dQ, dK, dV, scratch, B, n, H, D, 1.0f / sqrtf((float)D), make_drop(dropout_p, seed, offset)};
    cudaStream_t st = (cudaStream_t)stream;
    const size_t cnt = (size_t)B * H * n;
    PTRB200_LAUNCH(attention_dsum_kernel, (unsigned)((cnt + 255) / 256), 256, 0, st, a);
#define CALL(DD) launch_att_bwd<DD>(a, st)
    ATT_DISPATCH(D)
#undef CALL
    return check_launch("attention_bwd");
}

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
    DropCfg dc = make_drop(dropout_p, seed, offset);
    if (op == EW_ACT || op == EW_ACT_GRAD) dc.thr = (uint32_t)seed;           // seed = PTRB200_AF_* code
    PTRB200_LAUNCH(elementwise_kernel, (unsigned)blocks, 256, 0, stream, op, a, b, out, (size_t)count, dc);
    return check_launch("elementwise");
}

}  // extern "C"
