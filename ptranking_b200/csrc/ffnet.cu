// ffnet.cu -- stacked feed-forward scorer: Dropout -> Linear -> (BN | BN2) -> activation, repeated,
// forward and backward, fp32 SIMT path (the tensor-core kernels live in ffnet_tc.cuh).
//
// Reference functions replaced (wildltr/ptranking @ f1d366c):
//   get_stacked_FFNet            ptranking/base/utils.py:288-356
//   LTRBatchNorm                 ptranking/base/utils.py:201-223 (batch statistics in train AND eval)
//   LTRBatchNorm2/ltr_batch_norm ptranking/base/utils.py:227-282 (per-query statistics)
//   get_AF                       ptranking/base/utils.py:101-143
//   PointNeuralRanker.forward    ptranking/base/point_ranker.py:45-55
// and the autograd graph PyTorch builds for them.
//
// Layout in HBM: activations are dense row-major [rows = B*n, width] fp32.  Per layer the
// workspace keeps Z (pre-normalisation Linear output), A (post-activation) and, when a norm
// is present, mean/rstd per (group, channel); group = whole batch (BN) or one query (BN2).
#include "common.cuh"
#include "ffnet_act.cuh"
#include "ffnet_tc.cuh"

namespace ptrb200 {

// ------------------------------------------------------------------ SIMT GEMM
// C[M,N] = Aop[M,K] * Bop[K,N] with operand accessors chosen by MODE.
enum { GEMM_FWD = 0, GEMM_BWD_DATA = 1, GEMM_BWD_WEIGHT = 2 };

struct GemmArgs {
    const float* A;      // FWD: layer input [rows,d_in]   BWD_DATA: dZ [rows,d_out]   BWD_WEIGHT: dZ [rows,d_out]
    const float* Bm;     // FWD: W [d_out,d_in]            BWD_DATA: W [d_out,d_in]    BWD_WEIGHT: layer input [rows,d_in]
    const float* bias;   // FWD only
    float* C;            // FWD: Z [rows,d_out]            BWD_DATA: dA [rows,d_in]    BWD_WEIGHT: partials [splits,d_out,d_in]
    int rows, d_in, d_out;
    int M, N, K;         // GEMM extents
    int k_chunk;         // BWD_WEIGHT: rows per split
    DropCfg drop;        // dropout on the layer input (thr == 0: none)
};

template <int MODE>
static __device__ __forceinline__ float load_a(const GemmArgs& g, int m, int k) {
    if (MODE == GEMM_FWD) {
        float v = g.A[(size_t)m * g.d_in + k];
        if (g.drop.thr) v = dropout_keep(g.drop.key, (uint64_t)m * g.d_in + k, g.drop.thr) ? v * g.drop.scale : 0.0f;
        return v;
    } else if (MODE == GEMM_BWD_DATA) {
        return g.A[(size_t)m * g.d_out + k];                 // dZ[m, k]
    } else {
        return g.A[(size_t)k * g.d_out + m];                 // dZ[row k, out m]
    }
}
template <int MODE>
static __device__ __forceinline__ float load_b(const GemmArgs& g, int k, int n) {
    if (MODE == GEMM_FWD) {
        return g.Bm[(size_t)n * g.d_in + k];                 // W[n, k]
    } else if (MODE == GEMM_BWD_DATA) {
        return g.Bm[(size_t)k * g.d_in + n];                 // W[k, n]
    } else {
        float v = g.Bm[(size_t)k * g.d_in + n];              // input[row k, n]
        if (g.drop.thr) v = dropout_keep(g.drop.key, (uint64_t)k * g.d_in + n, g.drop.thr) ? v * g.drop.scale : 0.0f;
        return v;
    }
}

template <int MODE, int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmArgs g) {
    constexpr int BK = 16;
    constexpr int TX = BN / TN, TY = BM / TM;
    static_assert(TX * TY == 256, "256 threads");
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int t = threadIdx.x;
    const int tx = t % TX, ty = t / TX;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    int k_begin = 0, k_end = g.K;
    if (MODE == GEMM_BWD_WEIGHT) { k_begin = blockIdx.z * g.k_chunk; k_end = min(g.K, k_begin + g.k_chunk); }
    // A is contiguous along K for FWD / BWD_DATA and along M for BWD_WEIGHT; B along K for FWD, along N otherwise
    constexpr bool A_K_CONTIG = (MODE != GEMM_BWD_WEIGHT);
    constexpr bool B_K_CONTIG = (MODE == GEMM_FWD);

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

    for (int k0 = k_begin; k0 < k_end; k0 += BK) {
        for (int e = t; e < BM * BK; e += 256) {
            const int kk = A_K_CONTIG ? e % BK : e / BM;
            const int mm = A_K_CONTIG ? e / BK : e % BM;
            const int m = m0 + mm, k = k0 + kk;
            As[kk][mm] = (m < g.M && k < k_end) ? load_a<MODE>(g, m, k) : 0.0f;
        }
        for (int e = t; e < BN * BK; e += 256) {
            const int kk = B_K_CONTIG ? e % BK : e / BN;
            const int nn = B_K_CONTIG ? e / BK : e % BN;
            const int n = n0 + nn, k = k0 + kk;
            Bs[kk][nn] = (n < g.N && k < k_end) ? load_b<MODE>(g, k, n) : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + ty * TM + i;
        if (m >= g.M) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            if (n >= g.N) continue;
            float v = acc[i][j];
            if (MODE == GEMM_FWD) {
                g.C[(size_t)m * g.d_out + n] = v + g.bias[n];
            } else if (MODE == GEMM_BWD_DATA) {
                if (g.drop.thr) v = dropout_keep(g.drop.key, (uint64_t)m * g.d_in + n, g.drop.thr) ? v * g.drop.scale : 0.0f;
                g.C[(size_t)m * g.d_in + n] = v;
            } else {
                g.C[((size_t)blockIdx.z * g.d_out + m) * g.d_in + n] = v;
            }
        }
    }
}

// sum partials[splits, count] over splits in fixed order -> out[count]
// out[i] = sum_p partials[p][i].  Block = 64 outputs x 4 split groups: group q adds splits q, q+4, ... (independent
// loads, unrolled), then the four group sums are combined in a fixed order -- deterministic, and 4x the loads in flight
// of a one-thread-per-output loop over one split per SM.
__global__ void __launch_bounds__(256) reduce_splits_kernel(const float* __restrict__ partials, float* __restrict__ out, int splits, int count) {
    __shared__ float sh[4][64];
    const int e = threadIdx.x & 63, q = threadIdx.x >> 6;
    const int i = blockIdx.x * 64 + e;
    float s = 0.0f;
    if (i < count) {
#pragma unroll 8
        for (int p = q; p < splits; p += 4) s += __ldg(partials + (size_t)p * count + i);
    }
    sh[q][e] = s;
    __syncthreads();
    if (q == 0 && i < count) out[i] = (sh[0][e] + sh[1][e]) + (sh[2][e] + sh[3][e]);
}

// ------------------------------------------------------------------ column statistics
// For rows split into G groups of `gr` rows and `S` slices per group, accumulate per channel
//   sum1 = sum_r u[r,c]          sum2 = sum_r u[r,c] * v[r,c]
// in double, one CTA per (group, slice).  WHAT selects u, v:
//   STAT_MOMENTS : u = z, v = z                         (forward mean / variance)
//   STAT_DY      : u = dY, v = xhat, dY = dA*act'(Y) written to dY_out  (backward sums)
//   STAT_COLSUM  : u = z, v unused                      (bias gradient)
enum { STAT_MOMENTS = 0, STAT_DY = 1, STAT_COLSUM = 2 };

struct NormRef {           // everything needed to rebuild Y = a*xhat + c for one layer
    const float* mean;     // [G,C] or NULL when the layer has no norm
    const float* rstd;     // [G,C]
    const float* gamma;    // [C] or NULL (=1)
    const float* beta;     // [C] or NULL (=0)
    const float* aff_w;    // [C] or NULL (=1)
    const float* aff_b;    // [C] or NULL (=0)
    int act;
};
static __device__ __forceinline__ void norm_coeffs(const NormRef& nr, int c, float& a, float& cc) {
    const float ga = nr.gamma ? nr.gamma[c] : 1.0f, be = nr.beta ? nr.beta[c] : 0.0f;
    const float w = nr.aff_w ? nr.aff_w[c] : 1.0f, bw = nr.aff_b ? nr.aff_b[c] : 0.0f;
    a = ga * w;
    cc = be * w + bw;
}

template <int WHAT>
__global__ void colstat_kernel(const float* __restrict__ Z, const float* __restrict__ dA, float* __restrict__ dY_out,
                               NormRef nr, double* __restrict__ partials, int gr, int C, int S, int slice_rows) {
    // block (32, 8): x = channel lane, y = row lane
    __shared__ double sh1[8][33], sh2[8][33];
    const int g = blockIdx.x, sl = blockIdx.y;
    const int r0 = sl * slice_rows, r1 = min(gr, r0 + slice_rows);
    for (int cb = 0; cb < C; cb += 32) {
        const int c = cb + threadIdx.x;
        double s1 = 0.0, s2 = 0.0;
        if (c < C) {
            float a = 1.0f, cc = 0.0f, mu = 0.0f, rs = 1.0f;
            if (WHAT == STAT_DY) {
                norm_coeffs(nr, c, a, cc);
                if (nr.mean) { mu = nr.mean[(size_t)g * C + c]; rs = nr.rstd[(size_t)g * C + c]; }
            }
            for (int r = r0 + threadIdx.y; r < r1; r += 8) {
                const size_t off = ((size_t)g * gr + r) * C + c;
                const float z = Z[off];
                if (WHAT == STAT_MOMENTS) { s1 += (double)z; s2 += (double)z * (double)z; }
                else if (WHAT == STAT_COLSUM) { s1 += (double)z; }
                else {
                    const float xh = nr.mean ? (z - mu) * rs : z;
                    const ActOut ao = activate(nr.act, a * xh + cc);
                    const float dy = dA[off] * ao.dy;
                    dY_out[off] = dy;
                    s1 += (double)dy; s2 += (double)dy * (double)xh;
                }
            }
        }
        sh1[threadIdx.y][threadIdx.x] = s1; sh2[threadIdx.y][threadIdx.x] = s2;
        __syncthreads();
        if (threadIdx.y == 0 && c < C) {
            for (int y = 1; y < 8; ++y) { s1 += sh1[y][threadIdx.x]; s2 += sh2[y][threadIdx.x]; }
            double* p = partials + (((size_t)g * S + sl) * C + c) * 2;
            p[0] = s1; p[1] = s2;
        }
        __syncthreads();
    }
}

// Vectorised column statistics for widths that are multiples of 4: thread (q, ry) owns channels 4q..4q+3 and
// walks rows ry, ry+RY, ... of its slice, so a warp reads 512 contiguous bytes per step.  Same partial layout
// as colstat_kernel.  blockDim = (Q = C/4, RY); dynamic smem = RY*Q*8 doubles.
// STAT_DY can take dA in factored form: the scorer's last Linear has one output, so its data gradient is the outer
// product dA[r,c] = dropmask(dz[r] * w[c]) -- built on the fly here instead of being written and re-read.
struct Rank1Src { const float* w; DropCfg drop; int round_bf16; };     // w == NULL: dA is a dense [rows, C] tensor

// (4 resident CTAs per SM = 64 registers: this sweep is latency-bound, so occupancy matters more than registers)
// ACT >= 0 fixes the activation at compile time (the default scorer's GELU and ReLU): no per-element switch, and only the
// derivative is evaluated.  ACT = -1 reads it from the NormRef.
// PF: the loads of the NEXT row are issued before the current row is processed (the ncu capture of the dY sweep has 53 % of
// its stall samples on the first use of the freshly loaded Z: with one row in flight per thread the sweep is latency-bound
// at 37 % of HBM bandwidth); the extra live registers cost the fourth resident CTA.
template <int WHAT, int ACT = -1, bool PF = false>
__global__ void __launch_bounds__(256, PF ? 3 : 4) colstat4_kernel(const float* __restrict__ Z, const float* __restrict__ dA, float* __restrict__ dY_out,
                                NormRef nr, double* __restrict__ partials, int gr, int C, int S, int slice_rows, Rank1Src rk) {
    extern __shared__ double sh4[];
    const int Q = blockDim.x, RY = blockDim.y, q = threadIdx.x, ry = threadIdx.y, c = q * 4;
    const int g = blockIdx.x, sl = blockIdx.y;
    const int r0 = sl * slice_rows, r1 = min(gr, r0 + slice_rows);
    float a[4] = {1.f, 1.f, 1.f, 1.f}, cc[4] = {0.f, 0.f, 0.f, 0.f}, mu[4] = {0.f, 0.f, 0.f, 0.f}, rs[4] = {1.f, 1.f, 1.f, 1.f};
    if (WHAT == STAT_DY) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            norm_coeffs(nr, c + e, a[e], cc[e]);
            if (nr.mean) { mu[e] = nr.mean[(size_t)g * C + c + e]; rs[e] = nr.rstd[(size_t)g * C + c + e]; }
        }
    }
    // per-thread partial sums run in fp32 over <= 32 rows at a time and are flushed into float64 accumulators,
    // which keeps FP64 work and register pressure out of the streaming loop at no loss of accuracy that matters
    double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
    float f1[4] = {0.f, 0.f, 0.f, 0.f}, f2[4] = {0.f, 0.f, 0.f, 0.f};
    int since_flush = 0;
    const bool dense_da = WHAT == STAT_DY && !rk.w;
    float4 zn = make_float4(0.f, 0.f, 0.f, 0.f), dn = zn;
    if (PF && r0 + ry < r1) {
        const size_t o0 = ((size_t)g * gr + r0 + ry) * C + c;
        zn = __ldg(reinterpret_cast<const float4*>(Z + o0));
        if (dense_da) dn = __ldg(reinterpret_cast<const float4*>(dA + o0));
    }
    for (int r = r0 + ry; r < r1; r += RY) {
        const size_t off = ((size_t)g * gr + r) * C + c;
        float4 z4, dpre = make_float4(0.f, 0.f, 0.f, 0.f);
        if (PF) {
            z4 = zn; dpre = dn;
            if (r + RY < r1) {
                const size_t o1 = off + (size_t)RY * C;
                zn = __ldg(reinterpret_cast<const float4*>(Z + o1));
                if (dense_da) dn = __ldg(reinterpret_cast<const float4*>(dA + o1));
            }
        } else z4 = __ldg(reinterpret_cast<const float4*>(Z + off));
        const float z[4] = {z4.x, z4.y, z4.z, z4.w};
        if (WHAT == STAT_MOMENTS) {
#pragma unroll
            for (int e = 0; e < 4; ++e) { s1[e] += (double)z[e]; s2[e] += (double)z[e] * (double)z[e]; }
        } else if (WHAT == STAT_COLSUM) {
#pragma unroll
            for (int e = 0; e < 4; ++e) f1[e] += z[e];
        } else {
            float4 d4;
            if (rk.w) {
                float dz = __ldg(dA + (size_t)g * gr + r);
                float4 w4 = __ldg(reinterpret_cast<const float4*>(rk.w + c));
                if (rk.round_bf16) { dz = bf16_rn(dz); w4 = make_float4(bf16_rn(w4.x), bf16_rn(w4.y), bf16_rn(w4.z), bf16_rn(w4.w)); }
                d4 = make_float4(dz * w4.x, dz * w4.y, dz * w4.z, dz * w4.w);
                if (rk.drop.thr) {
                    const uint64_t dd = dropout_draw4(rk.drop.key, off >> 2);
                    d4.x = ((uint32_t)(dd) & 0xffffu) >= rk.drop.thr ? d4.x * rk.drop.scale : 0.0f;
                    d4.y = ((uint32_t)(dd >> 16) & 0xffffu) >= rk.drop.thr ? d4.y * rk.drop.scale : 0.0f;
                    d4.z = ((uint32_t)(dd >> 32) & 0xffffu) >= rk.drop.thr ? d4.z * rk.drop.scale : 0.0f;
                    d4.w = ((uint32_t)(dd >> 48)) >= rk.drop.thr ? d4.w * rk.drop.scale : 0.0f;
                }
            } else d4 = PF ? dpre : __ldg(reinterpret_cast<const float4*>(dA + off));
            const float d[4] = {d4.x, d4.y, d4.z, d4.w};
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float xh = nr.mean ? (z[e] - mu[e]) * rs[e] : z[e];
                const float dy = d[e] * activate(ACT >= 0 ? ACT : nr.act, a[e] * xh + cc[e]).dy;
                o[e] = dy;
                f1[e] += dy; f2[e] = fmaf(dy, xh, f2[e]);
            }
            *reinterpret_cast<float4*>(dY_out + off) = make_float4(o[0], o[1], o[2], o[3]);
        }
        if (WHAT != STAT_MOMENTS && ++since_flush == 32) {
#pragma unroll
            for (int e = 0; e < 4; ++e) { s1[e] += (double)f1[e]; s2[e] += (double)f2[e]; f1[e] = 0.f; f2[e] = 0.f; }
            since_flush = 0;
        }
    }
    if (WHAT != STAT_MOMENTS) {
#pragma unroll
        for (int e = 0; e < 4; ++e) { s1[e] += (double)f1[e]; s2[e] += (double)f2[e]; }
    }
    double* mine = sh4 + ((size_t)ry * Q + q) * 8;
#pragma unroll
    for (int e = 0; e < 4; ++e) { mine[e] = s1[e]; mine[4 + e] = s2[e]; }
    __syncthreads();
    if (ry == 0) {
        for (int y = 1; y < RY; ++y) {
            const double* o = sh4 + ((size_t)y * Q + q) * 8;
#pragma unroll
            for (int e = 0; e < 4; ++e) { s1[e] += o[e]; s2[e] += o[4 + e]; }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            double* p = partials + (((size_t)g * S + sl) * C + c + e) * 2;
            p[0] = s1[e]; p[1] = s2[e];
        }
    }
}

static __device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// single-channel case (the scorer's output layer): a plain strided reduction, one row per thread per step
template <int WHAT>
__global__ void __launch_bounds__(128) colstat_c1_kernel(const float* __restrict__ Z, const float* __restrict__ dA, float* __restrict__ dY_out,
                                                          NormRef nr, double* __restrict__ partials, int gr, int S, int slice_rows) {
    __shared__ double sh[2][4];
    const int g = blockIdx.x, sl = blockIdx.y;
    const int r0 = sl * slice_rows, r1 = min(gr, r0 + slice_rows);
    float a = 1.0f, cc = 0.0f, mu = 0.0f, rs = 1.0f;
    if (WHAT == STAT_DY) {
        norm_coeffs(nr, 0, a, cc);
        if (nr.mean) { mu = nr.mean[g]; rs = nr.rstd[g]; }
    }
    double s1 = 0.0, s2 = 0.0;
    for (int r = r0 + threadIdx.x; r < r1; r += 128) {
        const size_t off = (size_t)g * gr + r;
        const float z = Z[off];
        if (WHAT == STAT_MOMENTS) { s1 += (double)z; s2 += (double)z * (double)z; }
        else if (WHAT == STAT_COLSUM) { s1 += (double)z; }
        else {
            const float xh = nr.mean ? (z - mu) * rs : z;
            const float dy = dA[off] * activate(nr.act, a * xh + cc).dy;
            dY_out[off] = dy;
            s1 += (double)dy; s2 += (double)dy * (double)xh;
        }
    }
    s1 = warp_sum_d(s1); s2 = warp_sum_d(s2);
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s1; sh[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double* p = partials + ((size_t)g * S + sl) * 2;
        p[0] = (sh[0][0] + sh[0][1]) + (sh[0][2] + sh[0][3]);
        p[1] = (sh[1][0] + sh[1][1]) + (sh[1][2] + sh[1][3]);
    }
}

static bool colstat_vectorised(int C) { return C % 4 == 0 && C / 4 <= 256; }
template <int WHAT>
static void launch_colstat(cudaStream_t st, const char* tag, const float* Z, const float* dA, float* dY, const NormRef& nr,
                           double* part, int G, int S, int gr, int C, int slice_rows, Rank1Src r1 = Rank1Src{nullptr, DropCfg{0, 1.0f, 0}, 0}) {
    dim3 grid(G, S);
    if (C == 1 && !r1.w) {
        PTRB200_LAUNCH_TAG(tag, colstat_c1_kernel<WHAT>, grid, 128, 0, st, Z, dA, dY, nr, part, gr, S, slice_rows);
    } else if (colstat_vectorised(C)) {
        const int Q = C / 4;
        int RY = 256 / Q; if (RY < 1) RY = 1; if (RY > 16) RY = 16;
        const size_t sm = (size_t)RY * Q * 8 * sizeof(double);
        if (WHAT == STAT_DY && nr.act == PTRB200_AF_GELU)
            PTRB200_LAUNCH_TAG(tag, (colstat4_kernel<WHAT, PTRB200_AF_GELU, true>), grid, dim3(Q, RY), sm, st, Z, dA, dY, nr, part, gr, C, S, slice_rows, r1);
        else if (WHAT == STAT_DY && nr.act == PTRB200_AF_RELU)
            PTRB200_LAUNCH_TAG(tag, (colstat4_kernel<WHAT, PTRB200_AF_RELU, true>), grid, dim3(Q, RY), sm, st, Z, dA, dY, nr, part, gr, C, S, slice_rows, r1);
        else
            PTRB200_LAUNCH_TAG(tag, (colstat4_kernel<WHAT, -1>), grid, dim3(Q, RY), sm, st, Z, dA, dY, nr, part, gr, C, S, slice_rows, r1);
    } else {
        PTRB200_LAUNCH_TAG(tag, colstat_kernel<WHAT>, grid, dim3(32, 8), 0, st, Z, dA, dY, nr, part, gr, C, S, slice_rows);
    }
}

// Finalize kernels: one CTA of FIN_THREADS per (group, channel) [moments] or per channel [dY sums]; threads
// stride over the partial slots and a fixed-shape tree combines them (deterministic).
constexpr int FIN_THREADS = 128;
static __device__ __forceinline__ void block_sum2_d(double& a, double& b) {
    __shared__ double sh[2][FIN_THREADS / 32];
    a = warp_sum_d(a); b = warp_sum_d(b);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) { sh[0][warp] = a; sh[1][warp] = b; }
    __syncthreads();
    a = 0.0; b = 0.0;
#pragma unroll
    for (int w = 0; w < FIN_THREADS / 32; ++w) { a += sh[0][w]; b += sh[1][w]; }
}

// forward finalize: partials [G,S,C,2] -> mean, rstd (biased variance, eps = 1e-5) and the fused prologue
// coefficients  y = a*(z-mean)*rstd + c  ==  z*scale + shift.   grid = G*C
__global__ void __launch_bounds__(FIN_THREADS) moments_finalize_kernel(
        const double* __restrict__ partials, float* __restrict__ mean, float* __restrict__ rstd,
        float* __restrict__ scale, float* __restrict__ shift, NormRef nr, int G, int C, int S, int gr,
        const double* __restrict__ gcount = nullptr) {
    // gcount (sync-BN): the statistics group spans every rank's rows; its size arrives all-reduced on the device
    const double grd = gcount ? *gcount : (double)gr;
    const int i = blockIdx.x, g = i / C, c = i % C;
    double s1 = 0.0, s2 = 0.0;
    for (int s = threadIdx.x; s < S; s += FIN_THREADS) { const double* p = partials + (((size_t)g * S + s) * C + c) * 2; s1 += p[0]; s2 += p[1]; }
    block_sum2_d(s1, s2);
    if (threadIdx.x == 0) {
        const double m = s1 / grd;
        double var = s2 / grd - m * m;
        if (var < 0.0) var = 0.0;
        const float mf = (float)m, rf = (float)(1.0 / sqrt(var + 1e-5));
        mean[i] = mf;
        rstd[i] = rf;
        if (scale) {
            float a, cc;
            norm_coeffs(nr, c, a, cc);
            scale[i] = a * rf;
            shift[i] = cc - a * rf * mf;
        }
    }
}

// backward finalize: per-(group,channel) sums S1,S2 (float, optional) + totals over groups T1,T2 per channel.  grid = C
// Everything that depends only on those sums rides along (DyTail): the norm-parameter gradients, the Linear bias gradient
// and the coefficients of the folded normalisation backward  dZ = k1*dY + k3*z + k0  with
//   k1 = a*rstd,  k3 = -a*rstd^2*S2/N,  k0 = -a*rstd*S1/N + a*rstd^2*S2/N*mean      (a = gamma*aff_w)
struct DyTail {
    NormRef nr;
    float *dgamma, *dbeta, *daff_w, *daff_b;    // norm parameter gradients from T1 = sum dY, T2 = sum dY*xhat (NULL: skip)
    float *k1, *k3, *k0;                        // [G,C] or NULL
    int gr;
    float* bias_grad;                           // [C] or NULL
    int bias_mode;                              // 1: exact zero (the bias feeds a normalisation), 2: T1
    // sync-BN: counts[0] = rows of the statistics group over all ranks, counts[1] = this rank's rows.  The sums are
    // global then; parameter gradients are scaled by counts[1]/counts[0] so that the gradient all-reduce (SUM over
    // ranks) restores them exactly once.
    const double* counts;
};
static __device__ __forceinline__ void dz_coeff_one(const DyTail& t, size_t i, int c, float s1, float s2) {
    float a, cc;
    norm_coeffs(t.nr, c, a, cc);
    const float rs = t.nr.rstd[i], mu = t.nr.mean[i], invN = t.counts ? (float)(1.0 / t.counts[0]) : 1.0f / (float)t.gr;
    const float ar = a * rs, q = ar * rs * (s2 * invN);
    t.k1[i] = ar;
    t.k3[i] = -q;
    t.k0[i] = q * mu - ar * (s1 * invN);
}

__global__ void __launch_bounds__(FIN_THREADS) dy_finalize_kernel(
        const double* __restrict__ partials, float* __restrict__ S1, float* __restrict__ S2,
        float* __restrict__ T1, float* __restrict__ T2, int G, int C, int S, DyTail tail) {
    const int c = blockIdx.x;
    double t1 = 0.0, t2 = 0.0;
    if (S == 1) {
        for (int g = threadIdx.x; g < G; g += FIN_THREADS) {
            const double* p = partials + ((size_t)g * C + c) * 2;
            if (S1) { S1[(size_t)g * C + c] = (float)p[0]; S2[(size_t)g * C + c] = (float)p[1]; }
            if (tail.k1) dz_coeff_one(tail, (size_t)g * C + c, c, (float)p[0], (float)p[1]);
            t1 += p[0]; t2 += p[1];
        }
        block_sum2_d(t1, t2);
    } else {
        for (int g = 0; g < G; ++g) {
            double s1 = 0.0, s2 = 0.0;
            for (int s = threadIdx.x; s < S; s += FIN_THREADS) { const double* p = partials + (((size_t)g * S + s) * C + c) * 2; s1 += p[0]; s2 += p[1]; }
            block_sum2_d(s1, s2);
            if (threadIdx.x == 0) {
                if (S1) { S1[(size_t)g * C + c] = (float)s1; S2[(size_t)g * C + c] = (float)s2; }
                if (tail.k1) dz_coeff_one(tail, (size_t)g * C + c, c, (float)s1, (float)s2);
            }
            t1 += s1; t2 += s2;
        }
    }
    if (threadIdx.x == 0) {
        if (tail.counts) { const double w = tail.counts[1] / tail.counts[0]; t1 *= w; t2 *= w; }
        const float f1 = (float)t1, f2 = (float)t2;
        if (T1) T1[c] = f1;
        if (T2) T2[c] = f2;
        const NormRef& nr = tail.nr;
        const float ga = nr.gamma ? nr.gamma[c] : 1.0f, be = nr.beta ? nr.beta[c] : 0.0f;
        const float w = nr.aff_w ? nr.aff_w[c] : 1.0f;
        if (tail.dgamma) tail.dgamma[c] = w * f2;
        if (tail.dbeta) tail.dbeta[c] = w * f1;
        if (tail.daff_w) tail.daff_w[c] = ga * f2 + be * f1;
        if (tail.daff_b) tail.daff_b[c] = f1;
        if (tail.bias_grad) tail.bias_grad[c] = tail.bias_mode == 1 ? 0.0f : f1;
    }
}

// sync-BN: fold the per-slot partials [S][C][2] of the single statistics group into buf[c][2]; buf[2C] and buf[2C+1]
// both receive this rank's row count.  The caller all-reduces buf[0 .. 2C] (sums and the first count) across ranks, so
// afterwards buf[2C] is the global group size while buf[2C+1] stays local.   grid = C
__global__ void __launch_bounds__(FIN_THREADS) partials_fold_kernel(const double* __restrict__ partials, double* __restrict__ buf,
                                                                     int S, int C, double local_rows) {
    const int c = blockIdx.x;
    double s1 = 0.0, s2 = 0.0;
    for (int s = threadIdx.x; s < S; s += FIN_THREADS) { const double* p = partials + ((size_t)s * C + c) * 2; s1 += p[0]; s2 += p[1]; }
    block_sum2_d(s1, s2);
    if (threadIdx.x == 0) {
        buf[c * 2] = s1; buf[c * 2 + 1] = s2;
        if (c == 0) { buf[2 * C] = local_rows; buf[2 * C + 1] = local_rows; }
    }
}

// host hook (ptrb200_set_hook): collectives and gradient-ready notifications are the caller's business (the library
// holds no communicator); the hook runs on the launching host thread between kernel launches of the same stream.
static ptrb200_hook_fn g_hook = nullptr;
static void* g_hook_user = nullptr;
static int call_hook(int what, int layer, void* ptr, int64_t count, cudaStream_t st) {
    if (!g_hook) return PTRB200_OK;
    const int rc = g_hook(what, layer, ptr, count, (void*)st, g_hook_user);
    if (rc) { set_error("hook(%d, layer %d) returned %d", what, layer, rc); return PTRB200_ERR_INVALID; }
    return PTRB200_OK;
}

// ------------------------------------------------------------------ elementwise passes
// A = act(a * (z - mean) * rstd + c)
__global__ void norm_act_fwd_kernel(const float* __restrict__ Z, float* __restrict__ A, NormRef nr,
                                    size_t total, int C, int gr) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t row = i / C;
        float a, cc;
        norm_coeffs(nr, c, a, cc);
        float xh = Z[i];
        if (nr.mean) { const size_t g = row / gr; xh = (xh - nr.mean[g * C + c]) * nr.rstd[g * C + c]; }
        A[i] = activate(nr.act, a * xh + cc).y;
    }
}

// float4 variants of the two elementwise passes (C % 4 == 0)
__global__ void norm_act_fwd4_kernel(const float* __restrict__ Z, float* __restrict__ A, NormRef nr, size_t units, int C, int gr) {
    const int Q = C >> 2;
    for (size_t u = (size_t)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(u % Q) * 4;
        const size_t row = u / Q, g = row / gr;
        const float4 z4 = __ldg(reinterpret_cast<const float4*>(Z) + u);
        const float z[4] = {z4.x, z4.y, z4.z, z4.w};
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float a, cc;
            norm_coeffs(nr, c + e, a, cc);
            float xh = z[e];
            if (nr.mean) xh = (xh - nr.mean[g * C + c + e]) * nr.rstd[g * C + c + e];
            o[e] = activate(nr.act, a * xh + cc).y;
        }
        reinterpret_cast<float4*>(A)[u] = make_float4(o[0], o[1], o[2], o[3]);
    }
}
__global__ void norm_bwd_apply4_kernel(const float* __restrict__ Z, float* __restrict__ dY, NormRef nr,
                                       const float* __restrict__ S1, const float* __restrict__ S2, size_t units, int C, int gr,
                                       const double* __restrict__ gcount = nullptr) {
    const int Q = C >> 2;
    const float invN = gcount ? (float)(1.0 / *gcount) : 1.0f / (float)gr;
    for (size_t u = (size_t)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(u % Q) * 4;
        const size_t g = (u / Q) / gr;
        const float4 z4 = __ldg(reinterpret_cast<const float4*>(Z) + u);
        const float4 d4 = reinterpret_cast<const float4*>(dY)[u];
        const float z[4] = {z4.x, z4.y, z4.z, z4.w}, d[4] = {d4.x, d4.y, d4.z, d4.w};
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float a, cc;
            norm_coeffs(nr, c + e, a, cc);
            const float mu = nr.mean[g * C + c + e], rs = nr.rstd[g * C + c + e];
            const float xh = (z[e] - mu) * rs;
            o[e] = a * rs * (d[e] - S1[g * C + c + e] * invN - xh * (S2[g * C + c + e] * invN));
        }
        reinterpret_cast<float4*>(dY)[u] = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// dZ = a * rstd * (dY - S1/N - xhat * S2/N)     (in place over dY)
__global__ void norm_bwd_apply_kernel(const float* __restrict__ Z, float* __restrict__ dY, NormRef nr,
                                      const float* __restrict__ S1, const float* __restrict__ S2,
                                      size_t total, int C, int gr, const double* __restrict__ gcount = nullptr) {
    const float invN = gcount ? (float)(1.0 / *gcount) : 1.0f / (float)gr;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t g = (i / C) / gr;
        float a, cc;
        norm_coeffs(nr, c, a, cc);
        const float mu = nr.mean[g * C + c], rs = nr.rstd[g * C + c];
        const float xh = (Z[i] - mu) * rs;
        dY[i] = a * rs * (dY[i] - S1[g * C + c] * invN - xh * (S2[g * C + c] * invN));
    }
}

// ------------------------------------------------------------------ host side
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct LayerPlan {
    bool has_act, has_norm;
    int d_in, d_out, act;
    size_t z_off, a_off, mean_off, rstd_off;     // byte offsets into the workspace (a_off unused for the last layer)
    size_t scale_off, shift_off;                 // tensor-core mode: fused prologue coefficients [G,d_out]
    size_t img_f_hi, img_f_lo, img_d_hi, img_d_lo;   // tensor-core mode: pre-swizzled B images of W (fwd) and W^T (dgrad)
    size_t ain_off;                              // tensor-core mode, l >= 1: the layer's rebuilt input dropout(act(norm(Z_{l-1}))) [rows,d_in]
};
struct Plan {
    bool use_tc;                                 // every layer fits the tensor-core kernels (else the SIMT path runs)
    int passes;                                  // 3 = 3xTF32 (fp32-equivalent), 1 = TF32
    bool bf16;                                   // single pass with every operand rounded to bf16 first
    int tile_rows, seg_len, group_rows, tiles_per_group, ntiles;
    int L, G, gr, S_stat, slice_rows, S_w, k_chunk;
    size_t rows;
    LayerPlan layer[PTRB200_MAX_FF_LAYERS];
    size_t partials_off, s1_off, s2_off, dbuf0_off, dbuf1_off, wpart_off, k1_off, k3_off, k0_off, sync_off, total;
    bool sync_bn;                                // batch-level BN statistics all-reduced across data-parallel ranks
    bool ragged;                                 // per-query BN2 over a ragged batch (query boundaries from prefix offsets)
    int pad_k;                                   // > 0: input width zero-padded to this multiple of 4 for the tensor-core path
    size_t xpad_off, w0pad_off, dw0pad_off, dxpad_off;
    // bf16 features (PTRB200_DTYPE_BF16): read natively by the layer-0 tensor-core kernels; the padded and SIMT paths
    // widen them once into an fp32 workspace copy (xpad_off resp. xwide_off) and run unchanged
    bool x_bf16;
    size_t xwide_off;
};

// column blocking of the weight gradient: dZ columns in blocks of 128 (two m64 MMA tiles), input columns in blocks of <= 256
struct WgBlocks { int mblocks, kb, kblocks, gx; };
static WgBlocks wgrad_blocks(int N, int K) {
    WgBlocks b;
    b.mblocks = (N + 127) / 128;
    b.kb = K <= 256 ? K : 256;
    b.kblocks = (K + b.kb - 1) / b.kb;
    const int pairs = b.mblocks * b.kblocks, sms = num_sms();
    b.gx = pairs == 1 ? sms : (sms / pairs < 8 ? 8 : sms / pairs);
    return b;
}

static int make_plan(const ptrb200_ffnet* net, int B, int n, Plan& p, int total_rows = 0, int x_dtype = PTRB200_DTYPE_F32) {
    if (!net || B <= 0 || n <= 0 || total_rows < 0) { set_error("ffnet: null net or non-positive B/n"); return PTRB200_ERR_INVALID; }
    if (x_dtype != PTRB200_DTYPE_F32 && x_dtype != PTRB200_DTYPE_BF16) { set_error("ffnet: unknown feature dtype code %d", x_dtype); return PTRB200_ERR_INVALID; }
    p.x_bf16 = x_dtype == PTRB200_DTYPE_BF16;
    if (net->num_linear < 1 || net->num_linear > PTRB200_MAX_FF_LAYERS) { set_error("ffnet: num_linear=%d outside 1..%d", net->num_linear, PTRB200_MAX_FF_LAYERS); return PTRB200_ERR_INVALID; }
    if (net->norm < PTRB200_NORM_NONE || net->norm > PTRB200_NORM_BN2) { set_error("ffnet: bad norm %d", net->norm); return PTRB200_ERR_INVALID; }
    if (!(net->dropout_p >= 0.0f && net->dropout_p < 1.0f)) { set_error("ffnet: dropout_p must be in [0,1)"); return PTRB200_ERR_INVALID; }
    p.L = net->num_linear;
    // total_rows > 0: a ragged batch -- B queries cut out of total_rows documents by prefix offsets, n = longest list.
    // Batch-level BN and norm-free nets see one long list of total_rows documents (the dense code path as is); per-query
    // BN2 needs the query boundaries and normalises with the per-query bn2_ragged_* kernels below.
    p.ragged = total_rows > 0 && net->norm == PTRB200_NORM_BN2;
    p.rows = total_rows > 0 ? (size_t)total_rows : (size_t)B * n;
    p.G = net->norm == PTRB200_NORM_BN2 ? B : 1;
    p.gr = net->norm == PTRB200_NORM_BN2 ? n : (int)p.rows;
    if (net->math_mode < PTRB200_MATH_SIMT || net->math_mode > PTRB200_MATH_BF16) { set_error("ffnet: bad math_mode %d", net->math_mode); return PTRB200_ERR_INVALID; }
    p.use_tc = net->math_mode != PTRB200_MATH_SIMT;
    p.sync_bn = net->sync_bn != 0 && net->norm == PTRB200_NORM_BN;
    p.passes = net->math_mode == PTRB200_MATH_3XTF32 ? 3 : 1;
    p.bf16 = net->math_mode == PTRB200_MATH_BF16;
    // A feature width that is not a multiple of 4 (MQ2007/2008: 46 features) would push the whole net onto the fp32 SIMT
    // kernels.  Instead the input and the first weight matrix are zero-padded to the next multiple of 4 (two small copy
    // kernels per call) and every layer runs on the tensor cores; the padded columns contribute exact zeros.
    p.pad_k = (p.use_tc && net->dims[0] % 4 != 0) ? ((net->dims[0] + 3) / 4) * 4 : 0;
    for (int l = 0; l < net->num_linear && p.use_tc; ++l) {
        const int di = (l == 0 && p.pad_k) ? p.pad_k : net->dims[l], dn = net->dims[l + 1];
        // float4 row access needs widths % 4; wider layers are tiled over output columns / weight-gradient blocks
        if (di % 4 != 0 || di > 1024 || dn > 1024 || (dn % 4 != 0 && dn > 4)) p.use_tc = false;
    }
    if (!p.use_tc) p.pad_k = 0;
    for (int l = 0; l < net->num_linear && p.bf16; ++l)
        if (net->dims[l + 1] != 1 && net->dims[l + 1] % 4 != 0) p.use_tc = false;       // such a layer's data gradient would run unrounded on SIMT
    if (p.bf16 && !p.use_tc) { set_error("ffnet: math_mode bf16 needs layer widths the tensor-core kernels take (multiples of 4, <= 1024)"); return PTRB200_ERR_UNSUPPORTED; }
    // statistics slices: one CTA per (group, slice); aim for ~4 CTAs per SM when there is a single group
    if (p.G == 1) { p.slice_rows = 512; p.S_stat = (int)((p.rows + 511) / 512); if (p.S_stat > 1024) { p.S_stat = 1024; p.slice_rows = (int)((p.rows + 1023) / 1024); p.S_stat = (int)((p.rows + p.slice_rows - 1) / p.slice_rows); } }
    else { p.slice_rows = p.gr; p.S_stat = 1; }
    p.tile_rows = 128; p.seg_len = 128; p.group_rows = 0; p.tiles_per_group = 0;
    if (p.use_tc) {
        // row tiles of the tensor-core kernels never straddle a statistics group in a way that splits a segment
        if (net->norm == PTRB200_NORM_BN2) {
            if (n <= 128) { p.tile_rows = (128 / n) * n; p.seg_len = n; p.S_stat = 1; p.slice_rows = n; }
            else { p.group_rows = n; p.tiles_per_group = (n + 127) / 128; p.S_stat = p.tiles_per_group; p.slice_rows = 128; }
        } else { p.slice_rows = 128; p.S_stat = (int)((p.rows + 127) / 128); }
        p.ntiles = p.group_rows > 0 ? B * p.tiles_per_group : (int)((p.rows + p.tile_rows - 1) / p.tile_rows);
    }
    if (p.ragged && !p.use_tc) { set_error("ffnet: ragged BN2 batches need the tensor-core path (layer widths multiples of 4)"); return PTRB200_ERR_UNSUPPORTED; }
    if (p.ragged) { p.tile_rows = 128; p.seg_len = 128; p.group_rows = 0; p.tiles_per_group = 0; p.ntiles = (int)((p.rows + 127) / 128); p.S_stat = 1; p.slice_rows = (int)p.rows; }
    if (p.sync_bn && !p.use_tc) { set_error("ffnet: sync_bn needs the tensor-core path (layer widths multiples of 4)"); return PTRB200_ERR_UNSUPPORTED; }
    if (p.sync_bn && !g_hook) { set_error("ffnet: sync_bn needs an all-reduce hook (ptrb200_set_hook)"); return PTRB200_ERR_INVALID; }
    p.k_chunk = 2048; p.S_w = (int)((p.rows + 2047) / 2048);
    if (p.S_w > 592) { p.S_w = 592; p.k_chunk = (int)((p.rows + 591) / 592); p.S_w = (int)((p.rows + p.k_chunk - 1) / p.k_chunk); }
    size_t off = 0;
    int maxd = 0; size_t maxw = 0;
    for (int l = 0; l < p.L; ++l) {
        LayerPlan& lp = p.layer[l];
        lp.d_in = (l == 0 && p.pad_k) ? p.pad_k : net->dims[l]; lp.d_out = net->dims[l + 1];
        if (lp.d_in <= 0 || lp.d_out <= 0) { set_error("ffnet: non-positive layer width"); return PTRB200_ERR_INVALID; }
        if (!net->weight[l] || !net->bias[l]) { set_error("ffnet: layer %d weight/bias is NULL", l); return PTRB200_ERR_INVALID; }
        lp.act = l < p.L - 1 ? net->act_hidden : net->act_tail;
        lp.has_act = l < p.L - 1 ? true : net->act_tail != PTRB200_AF_NONE;
        lp.has_norm = lp.has_act && net->norm != PTRB200_NORM_NONE;
        if (lp.has_norm && net->norm == PTRB200_NORM_BN2 && (!net->gamma[l] || !net->beta[l])) { set_error("ffnet: BN2 layer %d needs gamma/beta", l); return PTRB200_ERR_INVALID; }
        lp.z_off = off; off = align_up(off + p.rows * lp.d_out * 4, 256);
        lp.a_off = off; if (l < p.L - 1 && (!p.use_tc || p.ragged)) off = align_up(off + p.rows * lp.d_out * 4, 256);
        lp.mean_off = off; lp.rstd_off = off; lp.scale_off = off; lp.shift_off = off;
        lp.img_f_hi = lp.img_f_lo = lp.img_d_hi = lp.img_d_lo = lp.ain_off = off;
        if (lp.has_norm) {
            lp.mean_off = off; off = align_up(off + (size_t)p.G * lp.d_out * 4, 256); lp.rstd_off = off; off = align_up(off + (size_t)p.G * lp.d_out * 4, 256);
            lp.scale_off = off; off = align_up(off + (size_t)p.G * lp.d_out * 4, 256); lp.shift_off = off; off = align_up(off + (size_t)p.G * lp.d_out * 4, 256);
        }
        if (p.use_tc) {
            const size_t fbytes = (size_t)((lp.d_in + 31) / 32) * (((lp.d_out + 15) / 16) * 16) * 128;
            const size_t dbytes = (size_t)((lp.d_out + 31) / 32) * (((lp.d_in + 15) / 16) * 16) * 128;
            lp.img_f_hi = off; off = align_up(off + fbytes, 1024); lp.img_f_lo = off; off = align_up(off + fbytes, 1024);
            lp.img_d_hi = off; off = align_up(off + dbytes, 1024); lp.img_d_lo = off; off = align_up(off + dbytes, 1024);
            if (l > 0) { lp.ain_off = off; off = align_up(off + p.rows * lp.d_in * 4, 256); }
        }
        maxd = lp.d_in > maxd ? lp.d_in : maxd; maxd = lp.d_out > maxd ? lp.d_out : maxd;
        const size_t w = (size_t)lp.d_in * lp.d_out; maxw = w > maxw ? w : maxw;
    }
    p.partials_off = off; off = align_up(off + (size_t)p.G * p.S_stat * maxd * 2 * 8, 256);
    p.s1_off = off; off = align_up(off + (size_t)p.G * maxd * 4, 256);
    p.s2_off = off; off = align_up(off + (size_t)p.G * maxd * 4, 256);
    p.k1_off = off; off = align_up(off + (size_t)p.G * maxd * 4, 256);
    p.k3_off = off; off = align_up(off + (size_t)p.G * maxd * 4, 256);
    p.k0_off = off; off = align_up(off + (size_t)p.G * maxd * 4, 256);
    p.sync_off = off; off = align_up(off + ((size_t)2 * maxd + 2) * 8, 256);
    p.dbuf0_off = off; off = align_up(off + p.rows * maxd * 4, 256);
    p.dbuf1_off = off; off = align_up(off + p.rows * maxd * 4, 256);
    {
        size_t wbytes = (size_t)p.S_w * maxw * 4;
        if (p.use_tc) for (int l = 0; l < p.L; ++l) {
            const WgBlocks wb = wgrad_blocks(p.layer[l].d_out, p.layer[l].d_in);
            const size_t need = (size_t)wb.gx * p.layer[l].d_in * p.layer[l].d_out * 4;
            wbytes = need > wbytes ? need : wbytes;
        }
        p.wpart_off = off; off = align_up(off + wbytes, 256);
    }
    p.xpad_off = p.w0pad_off = p.dw0pad_off = p.dxpad_off = off;
    if (p.pad_k) {
        p.xpad_off = off; off = align_up(off + p.rows * p.pad_k * 4, 256);
        p.w0pad_off = off; off = align_up(off + (size_t)net->dims[1] * p.pad_k * 4, 256);
        p.dw0pad_off = off; off = align_up(off + (size_t)net->dims[1] * p.pad_k * 4, 256);
        p.dxpad_off = off; off = align_up(off + p.rows * p.pad_k * 4, 256);
    }
    p.xwide_off = off;
    if (p.x_bf16 && !p.use_tc) { p.xwide_off = off; off = align_up(off + p.rows * (size_t)net->dims[0] * 4, 256); }
    p.total = off;
    return PTRB200_OK;
}

static NormRef norm_ref(const ptrb200_ffnet* net, const Plan& p, int l, char* ws) {
    NormRef nr;
    const LayerPlan& lp = p.layer[l];
    nr.act = lp.has_act ? lp.act : PTRB200_AF_NONE;
    nr.mean = lp.has_norm ? reinterpret_cast<const float*>(ws + lp.mean_off) : nullptr;
    nr.rstd = lp.has_norm ? reinterpret_cast<const float*>(ws + lp.rstd_off) : nullptr;
    nr.gamma = nr.beta = nr.aff_w = nr.aff_b = nullptr;
    if (lp.has_norm) {
        if (net->norm == PTRB200_NORM_BN) { if (net->norm_affine) { nr.gamma = net->gamma[l]; nr.beta = net->beta[l]; } }
        else { nr.gamma = net->gamma[l]; nr.beta = net->beta[l]; if (net->norm_affine) { nr.aff_w = net->aff_w[l]; nr.aff_b = net->aff_b[l]; } }
    }
    return nr;
}

template <int MODE>
static void launch_gemm(const GemmArgs& g, int splits, cudaStream_t st) {
    const char* tag = MODE == GEMM_FWD ? "gemm_simt_fwd" : MODE == GEMM_BWD_DATA ? "gemm_simt_bwd_data" : "gemm_simt_bwd_weight";
    // tile shape by output extents: tall-skinny, short-wide or square
    if (g.N <= 4) {
        dim3 grid((g.N + 3) / 4, (g.M + 255) / 256, splits);
        PTRB200_LAUNCH_TAG(tag, (gemm_simt_kernel<MODE, 256, 4, 4, 1>), grid, 256, 0, st, g);
    } else if (g.M <= 4) {
        dim3 grid((g.N + 255) / 256, (g.M + 3) / 4, splits);
        PTRB200_LAUNCH_TAG(tag, (gemm_simt_kernel<MODE, 4, 256, 1, 4>), grid, 256, 0, st, g);
    } else {
        dim3 grid((g.N + 63) / 64, (g.M + 63) / 64, splits);
        PTRB200_LAUNCH_TAG(tag, (gemm_simt_kernel<MODE, 64, 64, 4, 4>), grid, 256, 0, st, g);
    }
}

static int elementwise_blocks(size_t total) {
    size_t b = (total + 255) / 256;
    const size_t cap = (size_t)num_sms() * 16;
    return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}


// data gradient of a Linear with a single output: dIn[r,k] = dropmask(dz[r] * W[0,k])  (the scorer's last layer)
__global__ void dgrad_rank1_kernel(const float* __restrict__ dz, const float* __restrict__ W, float* __restrict__ dIn,
                                   size_t units, int K, DropCfg drop, int round_bf16) {
    const int Q = K >> 2;
    for (size_t u = (size_t)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (size_t)gridDim.x * blockDim.x) {
        const size_t row = u / Q;
        const int k = (int)(u % Q) * 4;
        float d = __ldg(dz + row);
        float4 w = __ldg(reinterpret_cast<const float4*>(W + k));
        if (round_bf16) { d = bf16_rn(d); w = make_float4(bf16_rn(w.x), bf16_rn(w.y), bf16_rn(w.z), bf16_rn(w.w)); }
        float4 v = make_float4(d * w.x, d * w.y, d * w.z, d * w.w);
        if (drop.thr) {
            const uint64_t dd = dropout_draw4(drop.key, (row * K + k) >> 2);
            v.x = ((uint32_t)(dd) & 0xffffu) >= drop.thr ? v.x * drop.scale : 0.0f;
            v.y = ((uint32_t)(dd >> 16) & 0xffffu) >= drop.thr ? v.y * drop.scale : 0.0f;
            v.z = ((uint32_t)(dd >> 32) & 0xffffu) >= drop.thr ? v.z * drop.scale : 0.0f;
            v.w = ((uint32_t)(dd >> 48)) >= drop.thr ? v.w * drop.scale : 0.0f;
        }
        reinterpret_cast<float4*>(dIn)[u] = v;
    }
}

// dst[r, 0..kd) = src[r, 0..ks) (zero beyond ks when widening; truncated when narrowing): the zero-padding of the feature
// matrix / first weight matrix to a multiple of 4 columns, and the way back for their gradients.
// drop.thr != 0: layer 0's dropout mask is applied on the way, keyed by the element's index r * min(ks, kd) + k in the
// unpadded matrix -- the index every other kernel variant uses -- so the padded features carry the same mask.
static __device__ __forceinline__ float copy_drop(float v, const DropCfg& drop, size_t r, int k, int kl) {
    return (!drop.thr || k >= kl || dropout_keep(drop.key, (uint64_t)r * kl + k, drop.thr)) ? v * drop.scale : 0.0f;
}
__global__ void copy_cols_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t rows, int ks, int kd, DropCfg drop) {
    const size_t total = rows * (size_t)kd;
    const int kl = ks < kd ? ks : kd;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / kd;
        const int k = (int)(i - r * kd);
        const float v = k < ks ? src[r * ks + k] : 0.0f;
        dst[i] = drop.thr ? copy_drop(v, drop, r, k, kl) : v;
    }
}
// the same from bf16 features (exact widening): the padded fp32 copy of a bf16 feature matrix (ks % 4 != 0), and with
// kd == ks the fp32 copy the SIMT kernels read
__global__ void copy_cols_bf16_kernel(const uint16_t* __restrict__ src, float* __restrict__ dst, size_t rows, int ks, int kd, DropCfg drop) {
    const size_t total = rows * (size_t)kd;
    const int kl = ks < kd ? ks : kd;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / kd;
        const int k = (int)(i - r * kd);
        const float v = k < ks ? __uint_as_float((uint32_t)src[r * ks + k] << 16) : 0.0f;
        dst[i] = drop.thr ? copy_drop(v, drop, r, k, kl) : v;
    }
}

// ------------------------------------------------------------------ tensor-core host paths

template <typename K>
static int opt_in_smem(K kernel, size_t bytes) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu B): %s", bytes, cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
    return PTRB200_OK;
}


// picks the row-tile height R (32/16/8) and ring depth so the kernel's buffers fit the 227 KB of one SM
static size_t wgrad_smem(int N, int K, int KP, int& R, int passes, int& stages, bool fused_dz = false, int min_R = 8) {
    // Largest tile height whose operand buffers and a >= 2-deep raw ring fit; as many ring stages as then fit.
    const size_t limit = 227 * 1024;
    static const int heights[] = {32, 24, 16, 8};
    auto fit = [&](int rows, int& st) -> size_t {
        const size_t op = (size_t)(128 + KP) * 128 * (passes == 3 ? 2 : 1);      // transposed operands: one 128-byte chunk per row
        const size_t rawz = (((size_t)rows * N * 4 + 127) / 128 * 128) * (fused_dz ? 2 : 1), rawp = ((size_t)rows * K * 4 + 127) / 128 * 128;
        const size_t fixed = 1024 + 2 * op + 128 + 3 * 128 * 4;      // + barriers + the coefficient rows of the folded normalisation backward
        for (st = WG_MAX_STAGES; st >= 2; --st)
            if (fixed + st * (rawz + rawp) <= limit) return fixed + st * (rawz + rawp);
        return 0;
    };
    // (a 24-row tile leaves a quarter of the staging threads idle, so the tallest tile that fits with 2 stages wins over depth)
    for (int h : heights) {
        if (h < min_R) continue;
        int st = 0;
        const size_t bytes = fit(h, st);
        if (bytes) { R = h; stages = st; return bytes; }
    }
    R = 8; stages = 2;
    return limit + 1;        // does not fit
}

static bool rows_ws_fits(int K, int N, int passes) {
    const int NP = ((N + 15) / 16) * 16, nchunks = (K + 31) / 32;
    const size_t ws_smem = 1024 + (size_t)nchunks * NP * 128 * (passes == 3 ? 2 : 1) + 65536 + (size_t)RW_EPI_WARPS * NP * 8 + 128;
    return ws_smem <= 227 * 1024 && N <= RW_MAX_N;
}

// stats_kind: 0 none, 1 one statistics group over the whole batch (BN), 2 per-query groups (BN2).
// *S_out receives the number of partial slots per group the kernel wrote.
// xb: g.P holds bf16 features -- layer 0's forward (no scale/shift, no activation), the kernels' XB variants.
static int launch_rows_gemm(int mode, int passes, RowsGemmArgs& g, int ntiles, cudaStream_t st,
                            int stats_kind = 0, int* S_out = nullptr, int S_default = 1, bool xb = false) {
    g.NP = ((g.N + 15) / 16) * 16;
    int rc;
    if (xb && (mode != RG_FWD || g.scale || g.act != PTRB200_AF_NONE)) { set_error("rows_gemm: bf16 input only feeds layer 0's forward"); return PTRB200_ERR_INVALID; }
    const int nchunks = (g.K + 31) / 32;
    // ---- persistent warp-specialised kernel when the whole weight image fits beside the A ring ----
    const size_t ws_smem = 1024 + (size_t)nchunks * g.NP * 128 * (passes == 3 ? 2 : 1) + 65536 + (size_t)RW_EPI_WARPS * g.NP * 8 + 128;
    const bool seg_ok = !g.partials || g.seg_len == g.tile_rows || g.group_rows > 0;     // no sub-tile statistics segments
    if (ws_smem <= 227 * 1024 && seg_ok && g.N <= RW_MAX_N) {
        RowsWsExtra x{};
        x.ntiles = ntiles; x.nchunks = nchunks;
        x.stats_mode = (!g.partials || stats_kind == 0) ? 0 : (stats_kind == 1 ? 1 : 2);
        const int grid = ntiles < num_sms() ? ntiles : num_sms();
        if (S_out) *S_out = x.stats_mode == 1 ? grid : S_default;
#define RW_CASE_K(M, P, A, KT, TAG)                                                                 \
        if (mode == M && passes == P && act_t == A && g.K == KT) {                                  \
            if ((rc = opt_in_smem(rows_gemm_ws_kernel<M, P, A, KT>, ws_smem))) return rc;           \
            PTRB200_LAUNCH_TAG(TAG, (rows_gemm_ws_kernel<M, P, A, KT>), grid, RW_THREADS, ws_smem, st, g, x); \
            return PTRB200_OK;                                                                      \
        }
#define RW_CASE(M, P, A, TAG)                                                                       \
        if (mode == M && passes == P && act_t == A) {                                               \
            if ((rc = opt_in_smem(rows_gemm_ws_kernel<M, P, A>, ws_smem))) return rc;               \
            PTRB200_LAUNCH_TAG(TAG, (rows_gemm_ws_kernel<M, P, A>), grid, RW_THREADS, ws_smem, st, g, x); \
            return PTRB200_OK;                                                                      \
        }
        // the prologue activation is a template parameter for the common codes, -1 = generic run-time switch
        const int act_t = (g.act == PTRB200_AF_NONE || g.act == PTRB200_AF_RELU || g.act == PTRB200_AF_GELU || g.act == PTRB200_AF_SIGM) ? g.act : -1;
        if (xb) {
#define RWX_CASE(P, KT)                                                                                           \
            if (passes == P && (KT == 0 || g.K == KT)) {                                                          \
                if ((rc = opt_in_smem(rows_gemm_ws_kernel<RG_FWD, P, PTRB200_AF_NONE, KT, true>, ws_smem))) return rc; \
                PTRB200_LAUNCH_TAG("rows_gemm_ws_fwd_xbf16", (rows_gemm_ws_kernel<RG_FWD, P, PTRB200_AF_NONE, KT, true>), grid, RW_THREADS, ws_smem, st, g, x); \
                return PTRB200_OK;                                                                                \
            }
            RWX_CASE(3, 136) RWX_CASE(1, 136) RWX_CASE(3, 0) RWX_CASE(1, 0)
#undef RWX_CASE
            set_error("rows_gemm: no bf16-input variant for %d passes", passes);
            return PTRB200_ERR_INVALID;
        }
        // width-specialised instantiations for the default scorer (136 features, 100-wide hidden layers)
        RW_CASE_K(RG_FWD, 3, PTRB200_AF_NONE, 136, "rows_gemm_ws_fwd") RW_CASE_K(RG_FWD, 3, PTRB200_AF_GELU, 100, "rows_gemm_ws_fwd")
        RW_CASE_K(RG_DGRAD, 3, PTRB200_AF_NONE, 100, "rows_gemm_ws_dgrad")
        RW_CASE_K(RG_FWD, 1, PTRB200_AF_NONE, 136, "rows_gemm_ws_fwd") RW_CASE_K(RG_FWD, 1, PTRB200_AF_GELU, 100, "rows_gemm_ws_fwd")
        RW_CASE_K(RG_DGRAD, 1, PTRB200_AF_NONE, 100, "rows_gemm_ws_dgrad")
        RW_CASE(RG_FWD, 3, PTRB200_AF_NONE, "rows_gemm_ws_fwd") RW_CASE(RG_FWD, 3, PTRB200_AF_RELU, "rows_gemm_ws_fwd")
        RW_CASE(RG_FWD, 3, PTRB200_AF_GELU, "rows_gemm_ws_fwd") RW_CASE(RG_FWD, 3, PTRB200_AF_SIGM, "rows_gemm_ws_fwd")
        RW_CASE(RG_FWD, 3, -1, "rows_gemm_ws_fwd")
        RW_CASE(RG_FWD, 1, PTRB200_AF_NONE, "rows_gemm_ws_fwd") RW_CASE(RG_FWD, 1, PTRB200_AF_RELU, "rows_gemm_ws_fwd")
        RW_CASE(RG_FWD, 1, PTRB200_AF_GELU, "rows_gemm_ws_fwd") RW_CASE(RG_FWD, 1, PTRB200_AF_SIGM, "rows_gemm_ws_fwd")
        RW_CASE(RG_FWD, 1, -1, "rows_gemm_ws_fwd")
        RW_CASE(RG_DGRAD, 3, PTRB200_AF_NONE, "rows_gemm_ws_dgrad")
        RW_CASE(RG_DGRAD, 1, PTRB200_AF_NONE, "rows_gemm_ws_dgrad")
#undef RW_CASE
#undef RW_CASE_K
        return PTRB200_ERR_INVALID;
    }
    if (S_out) *S_out = S_default;
    // one-tile-per-CTA kernel; output columns are tiled (RG_MAX_N per CTA) when the layer is wider: the accumulators of
    // a tile live in registers
    g.n_tile = g.N <= RG_MAX_N ? g.N : RG_MAX_N;
    const int n_tiles = (g.N + g.n_tile - 1) / g.n_tile;
    const int NPt = ((g.n_tile + 15) / 16) * 16;
    const size_t operands = 32768 + (size_t)2 * NPt * 256, otile = (size_t)128 * g.n_tile * 4;      // A hi|lo + two weight-chunk stages
    g.tail_off = (int)(((operands > otile ? operands : otile) + 15) / 16 * 16);
    const size_t smem = 1024 + (size_t)g.tail_off + 64;
    const dim3 rg_grid(ntiles, n_tiles);
    if (xb) {
        if (passes == 3) {
            if ((rc = opt_in_smem(rows_gemm_tc_kernel<RG_FWD, 3, PTRB200_AF_NONE, true>, smem))) return rc;
            PTRB200_LAUNCH_TAG("rows_gemm_tc_fwd_xbf16", (rows_gemm_tc_kernel<RG_FWD, 3, PTRB200_AF_NONE, true>), rg_grid, RG_THREADS, smem, st, g);
        } else {
            if ((rc = opt_in_smem(rows_gemm_tc_kernel<RG_FWD, 1, -1, true>, smem))) return rc;
            PTRB200_LAUNCH_TAG("rows_gemm_tc_fwd_xbf16", (rows_gemm_tc_kernel<RG_FWD, 1, -1, true>), rg_grid, RG_THREADS, smem, st, g);
        }
        return PTRB200_OK;
    }
    // the prologue's activation as a compile-time constant for the common cases (a runtime switch per element is what the
    // ncu capture of the 256 -> 512 head layer showed: 65 thread instructions per staged element)
#define RG_CASE(M, P, A, TAG)                                                                      \
    if (mode == M && passes == P && (A < 0 || g.act == A)) {                                       \
        if ((rc = opt_in_smem(rows_gemm_tc_kernel<M, P, A>, smem))) return rc;                     \
        PTRB200_LAUNCH_TAG(TAG, (rows_gemm_tc_kernel<M, P, A>), rg_grid, RG_THREADS, smem, st, g); \
        return PTRB200_OK;                                                                         \
    }
    RG_CASE(RG_FWD, 3, PTRB200_AF_NONE, "rows_gemm_tc_fwd")
    RG_CASE(RG_FWD, 3, PTRB200_AF_RELU, "rows_gemm_tc_fwd")
    RG_CASE(RG_FWD, 3, PTRB200_AF_GELU, "rows_gemm_tc_fwd")
    RG_CASE(RG_FWD, 3, -1, "rows_gemm_tc_fwd")
    RG_CASE(RG_FWD, 1, -1, "rows_gemm_tc_fwd")
    RG_CASE(RG_DGRAD, 3, PTRB200_AF_NONE, "rows_gemm_tc_dgrad")
    RG_CASE(RG_DGRAD, 3, -1, "rows_gemm_tc_dgrad")
    RG_CASE(RG_DGRAD, 1, -1, "rows_gemm_tc_dgrad")
#undef RG_CASE
    return PTRB200_ERR_INVALID;
}

static void set_tiling(RowsGemmArgs& g, const Plan& p) {
    g.tile_rows = p.tile_rows; g.seg_len = p.seg_len; g.group_rows = p.group_rows; g.tiles_per_group = p.tiles_per_group;
}

// prologue that rebuilds the post-activation input of layer l from what layer l-1 stored (a ragged plan stores it whole)
static void set_prologue(const ptrb200_ffnet* net, const Plan& p, int l, char* ws, const float* X,
                         const float*& P, const float*& scale, const float*& shift, int& act) {
    if (l == 0) { P = X; scale = shift = nullptr; act = PTRB200_AF_NONE; return; }
    const LayerPlan& prev = p.layer[l - 1];
    if (p.ragged) { P = reinterpret_cast<const float*>(ws + prev.a_off); scale = shift = nullptr; act = PTRB200_AF_NONE; return; }
    P = reinterpret_cast<const float*>(ws + prev.z_off);
    scale = prev.has_norm ? reinterpret_cast<const float*>(ws + prev.scale_off) : nullptr;
    shift = prev.has_norm ? reinterpret_cast<const float*>(ws + prev.shift_off) : nullptr;
    act = prev.has_act ? prev.act : PTRB200_AF_NONE;
}

// ------------------------------------------------------------------ per-query BN2 over a ragged batch (SURVEY 8f-2)
// LTRBatchNorm2 (base/utils.py:227-282) normalises every query over its own documents.  With per-query offsets one CTA
// owns one query (32 channel lanes x 8 row lanes), so moments, dY sums and the normalisation backward need no cross-CTA
// reduction; the Linear contractions run on the same tensor-core kernels in their plain (no fused prologue) form.
__global__ void __launch_bounds__(256) bn2_ragged_moments_kernel(const float* __restrict__ Z, const int32_t* __restrict__ offsets,
                                                                  float* __restrict__ mean, float* __restrict__ rstd, int C) {
    __shared__ double sh1[8][33], sh2[8][33];
    const int g = blockIdx.x, r0 = offsets[g], n = offsets[g + 1] - r0;
    for (int cb = 0; cb < C; cb += 32) {
        const int c = cb + threadIdx.x;
        double s1 = 0.0, s2 = 0.0;
        if (c < C)
            for (int r = threadIdx.y; r < n; r += 8) { const double z = (double)Z[(size_t)(r0 + r) * C + c]; s1 += z; s2 += z * z; }
        sh1[threadIdx.y][threadIdx.x] = s1; sh2[threadIdx.y][threadIdx.x] = s2;
        __syncthreads();
        if (threadIdx.y == 0 && c < C) {
            for (int y = 1; y < 8; ++y) { s1 += sh1[y][threadIdx.x]; s2 += sh2[y][threadIdx.x]; }
            const double cnt = n > 0 ? (double)n : 1.0, m = s1 / cnt;
            double var = s2 / cnt - m * m;
            if (var < 0.0) var = 0.0;
            mean[(size_t)g * C + c] = (float)m;
            rstd[(size_t)g * C + c] = (float)(1.0 / sqrt(var + 1e-5));
        }
        __syncthreads();
    }
}

// A = act(a * (z - mean_g) * rstd_g + c) for the documents of query g
__global__ void __launch_bounds__(256) bn2_ragged_act_kernel(const float* __restrict__ Z, float* __restrict__ A, NormRef nr,
                                                              const int32_t* __restrict__ offsets, int C) {
    const int g = blockIdx.x, r0 = offsets[g], n = offsets[g + 1] - r0;
    for (int c = threadIdx.x; c < C; c += 32) {
        float a, cc;
        norm_coeffs(nr, c, a, cc);
        const float mu = nr.mean[(size_t)g * C + c], rs = nr.rstd[(size_t)g * C + c];
        for (int r = threadIdx.y; r < n; r += 8) {
            const size_t off = (size_t)(r0 + r) * C + c;
            A[off] = activate(nr.act, a * ((Z[off] - mu) * rs) + cc).y;
        }
    }
}

// dY = dA * act'(Y) (written) and, per (query, channel), S1 = sum dY, S2 = sum dY * xhat -> partials[g][c][2]
__global__ void __launch_bounds__(256) bn2_ragged_dy_kernel(const float* __restrict__ Z, const float* __restrict__ dA, float* __restrict__ dY,
                                                             NormRef nr, const int32_t* __restrict__ offsets, double* __restrict__ partials, int C) {
    __shared__ double sh1[8][33], sh2[8][33];
    const int g = blockIdx.x, r0 = offsets[g], n = offsets[g + 1] - r0;
    for (int cb = 0; cb < C; cb += 32) {
        const int c = cb + threadIdx.x;
        double s1 = 0.0, s2 = 0.0;
        if (c < C) {
            float a, cc;
            norm_coeffs(nr, c, a, cc);
            const float mu = nr.mean[(size_t)g * C + c], rs = nr.rstd[(size_t)g * C + c];
            for (int r = threadIdx.y; r < n; r += 8) {
                const size_t off = (size_t)(r0 + r) * C + c;
                const float xh = (Z[off] - mu) * rs;
                const float dy = dA[off] * activate(nr.act, a * xh + cc).dy;
                dY[off] = dy;
                s1 += (double)dy; s2 += (double)dy * (double)xh;
            }
        }
        sh1[threadIdx.y][threadIdx.x] = s1; sh2[threadIdx.y][threadIdx.x] = s2;
        __syncthreads();
        if (threadIdx.y == 0 && c < C) {
            for (int y = 1; y < 8; ++y) { s1 += sh1[y][threadIdx.x]; s2 += sh2[y][threadIdx.x]; }
            double* p = partials + ((size_t)g * C + c) * 2;
            p[0] = s1; p[1] = s2;
        }
        __syncthreads();
    }
}

// dZ = a * rstd_g * (dY - S1_g / n_g - xhat * S2_g / n_g), in place over dY
__global__ void __launch_bounds__(256) bn2_ragged_apply_kernel(const float* __restrict__ Z, float* __restrict__ dY, NormRef nr,
                                                                const float* __restrict__ S1, const float* __restrict__ S2,
                                                                const int32_t* __restrict__ offsets, int C) {
    const int g = blockIdx.x, r0 = offsets[g], n = offsets[g + 1] - r0;
    const float invN = n > 0 ? 1.0f / (float)n : 0.0f;
    for (int c = threadIdx.x; c < C; c += 32) {
        float a, cc;
        norm_coeffs(nr, c, a, cc);
        const float mu = nr.mean[(size_t)g * C + c], rs = nr.rstd[(size_t)g * C + c];
        const float s1 = S1[(size_t)g * C + c] * invN, s2 = S2[(size_t)g * C + c] * invN;
        for (int r = threadIdx.y; r < n; r += 8) {
            const size_t off = (size_t)(r0 + r) * C + c;
            const float xh = (Z[off] - mu) * rs;
            dY[off] = a * rs * (dY[off] - s1 - xh * s2);
        }
    }
}

// operand images of every weight matrix (and, for the backward pass, of its transpose) in one launch
static void pack_weight_images(const ptrb200_ffnet* net, const Plan& p, char* ws, bool fwd_only, cudaStream_t st) {
    PackJobs jobs{};
    int nj = 0, max_units = 0;
    for (int l = 0; l < p.L; ++l) {
        const LayerPlan& lp = p.layer[l];
        for (int tr = 0; tr < (fwd_only ? 1 : 2); ++tr) {
            if (tr == 1 && (l == 0 || lp.d_out % 4 != 0)) continue;     // dgrad images: only where launch_dgrad runs the tensor-core dgrad
            PackJob& j = jobs.job[nj++];
            j.round_bf16 = p.bf16;
            j.src = net->weight[l]; j.src_cols = lp.d_in; j.transpose = tr;
            j.N = tr ? lp.d_in : lp.d_out; j.K = tr ? lp.d_out : lp.d_in;
            j.NP = ((j.N + 15) / 16) * 16; j.nchunks = (j.K + 31) / 32;
            j.img_hi = reinterpret_cast<unsigned char*>(ws + (tr ? lp.img_d_hi : lp.img_f_hi));
            j.img_lo = p.passes == 3 ? reinterpret_cast<unsigned char*>(ws + (tr ? lp.img_d_lo : lp.img_f_lo)) : nullptr;
            const int units = j.nchunks * j.NP * 8;
            max_units = units > max_units ? units : max_units;
        }
    }
    PTRB200_LAUNCH(pack_b_images_kernel, dim3((max_units + 255) / 256, nj), 256, 0, st, jobs);
}

// dW[N,K] = sum_rows dZ^T (x) P on tensor cores.  The caller fills the operands of w (dZ, P, dropout, partials, rows and,
// for the folded normalisation backward, Z2 and the coefficients); grid.x persistent CTAs per (dZ block, input block)
// each write one partial, which reduce_splits_kernel sums in a fixed order.
// xb: w.P holds bf16 features (layer 0).  The tile height -- and with it the rows every CTA sums and the order of the
// partials -- is the one the fp32 layer input gets, so both give the same dW bit for bit; only the raw ring shrinks.
static int launch_wgrad(WgradArgs& w, int N, int K, int kb, dim3 grid, int passes, float* dW, cudaStream_t st, bool xb = false) {
    int rc;
    const bool fused_dz = w.Z2 != nullptr;
    w.N_full = N; w.K_full = K; w.kb = kb;
    w.N = N < 128 ? N : 128; w.K = kb;       // block maxima (buffer geometry)
    w.KP = ((w.K + 15) / 16) * 16;
    size_t smem = wgrad_smem(w.N, w.K, w.KP, w.tile_rows, passes, w.stages, fused_dz, fused_dz ? 24 : 8);
    if (xb) {
        // the kernel's layout at the same tile height and ring depth, with the layer-input slots at 2 bytes per element
        const size_t op = (size_t)(128 + w.KP) * 128 * (passes == 3 ? 2 : 1);
        const size_t rawz = (((size_t)w.tile_rows * w.N * 4 + 127) / 128 * 128) * (fused_dz ? 2 : 1);
        const size_t rawp = ((size_t)w.tile_rows * w.K * 2 + 127) / 128 * 128;
        smem = 1024 + 2 * op + 128 + 3 * 128 * 4 + (size_t)w.stages * (rawz + rawp);
        if (passes == 3) { if ((rc = opt_in_smem(wgrad_tc_kernel<3, true>, smem))) return rc; PTRB200_LAUNCH_TAG("wgrad_tc_xbf16", (wgrad_tc_kernel<3, true>), grid, WG_THREADS, smem, st, w); }
        else { if ((rc = opt_in_smem(wgrad_tc_kernel<1, true>, smem))) return rc; PTRB200_LAUNCH_TAG("wgrad_tc_xbf16", (wgrad_tc_kernel<1, true>), grid, WG_THREADS, smem, st, w); }
    }
    else if (passes == 3) { if ((rc = opt_in_smem(wgrad_tc_kernel<3>, smem))) return rc; PTRB200_LAUNCH_TAG("wgrad_tc", wgrad_tc_kernel<3>, grid, WG_THREADS, smem, st, w); }
    else { if ((rc = opt_in_smem(wgrad_tc_kernel<1>, smem))) return rc; PTRB200_LAUNCH_TAG("wgrad_tc", wgrad_tc_kernel<1>, grid, WG_THREADS, smem, st, w); }
    PTRB200_LAUNCH(reduce_splits_kernel, (N * K + 63) / 64, 256, 0, st, (const float*)w.partials, dW, (int)grid.x, N * K);
    return PTRB200_OK;
}

// dIn = dropmask(dZ W) of layer l: the tensor-core dgrad when d_out % 4 == 0, the outer product when the layer has a single
// output, else the SIMT GEMM.  Z non-NULL (tensor-core dgrad only): dZ holds dY and the normalisation backward
// k1*dY + k3*Z + k0 is folded into the operand staging, with the coefficients dy_finalize_kernel left in the workspace.
static int launch_dgrad(const ptrb200_ffnet* net, const Plan& p, int l, char* ws, const float* dZ, const float* Z, float* dIn,
                        DropCfg drop, cudaStream_t st) {
    const LayerPlan& lp = p.layer[l];
    if (lp.d_out % 4 == 0) {
        const int NPl = ((lp.d_in + 15) / 16) * 16, nch = (lp.d_out + 31) / 32;
        unsigned char* ih = reinterpret_cast<unsigned char*>(ws + lp.img_d_hi);
        unsigned char* il = p.passes == 3 ? reinterpret_cast<unsigned char*>(ws + lp.img_d_lo) : nullptr;
        if (l == 0)     // (layer 0's transpose image is only needed when dX is requested; deeper layers were packed by the forward call)
            PTRB200_LAUNCH(pack_b_image_kernel<true>, (nch * NPl * 8 + 255) / 256, 256, 0, st, net->weight[l], lp.d_out, lp.d_in, ih, il, lp.d_in, NPl, lp.d_out, nch, (int)p.bf16);
        RowsGemmArgs g{};
        g.round_bf16 = p.bf16;
        g.P = dZ; g.scale = g.shift = nullptr; g.act = PTRB200_AF_NONE; g.gr_prev = (int)p.rows;
        if (Z) {
            g.P2 = Z; g.gr_cur = p.gr;
            g.kc1 = reinterpret_cast<const float*>(ws + p.k1_off); g.kc3 = reinterpret_cast<const float*>(ws + p.k3_off); g.kc0 = reinterpret_cast<const float*>(ws + p.k0_off);
        }
        g.drop = drop;
        g.b_img_hi = ih; g.b_img_lo = il; g.bias = nullptr; g.Out = dIn; g.partials = nullptr;
        g.rows = (int)p.rows; g.K = lp.d_out; g.N = lp.d_in;
        g.tile_rows = 128; g.seg_len = 128; g.group_rows = 0; g.tiles_per_group = 0;
        return launch_rows_gemm(RG_DGRAD, p.passes, g, (int)((p.rows + 127) / 128), st);
    }
    if (lp.d_out == 1 && lp.d_in % 4 == 0) {
        const size_t units = p.rows * (lp.d_in / 4);
        PTRB200_LAUNCH(dgrad_rank1_kernel, elementwise_blocks(units), 256, 0, st, dZ, net->weight[l], dIn, units, lp.d_in, drop, (int)p.bf16);
        return PTRB200_OK;
    }
    GemmArgs g{};
    g.A = dZ; g.Bm = net->weight[l]; g.C = dIn;
    g.rows = (int)p.rows; g.d_in = lp.d_in; g.d_out = lp.d_out;
    g.M = (int)p.rows; g.N = lp.d_in; g.K = lp.d_out;
    g.drop = drop;
    launch_gemm<GEMM_BWD_DATA>(g, 1, st);
    return PTRB200_OK;
}

// norm-parameter gradient buffers of layer l (BN: gamma/beta only when affine; BN2: gamma/beta, and aff_w/aff_b when affine)
static void set_norm_grads(DyTail& t, const ptrb200_ffnet* net, const ptrb200_ffnet_grads* grads, int l) {
    if (net->norm == PTRB200_NORM_BN) { if (net->norm_affine) { t.dgamma = grads->gamma[l]; t.dbeta = grads->beta[l]; } }
    else { t.dgamma = grads->gamma[l]; t.dbeta = grads->beta[l]; if (net->norm_affine) { t.daff_w = grads->aff_w[l]; t.daff_b = grads->aff_b[l]; } }
}

// Dense and ragged plans share the contractions; p.ragged (per-query BN2 over a ragged batch) only changes the
// normalisation step: per-query bn2_ragged_* kernels on a materialised layer input instead of the epilogue statistics
// partials and the normalisation folded into the next layer's prologue.
// xb: X holds bf16 features, read natively by layer 0's forward and weight-gradient kernels.
// x_masked: X already carries layer 0's dropout (the zero-padded copy of a feature matrix whose width is not a multiple
// of 4), so layer 0 draws no mask of its own.
static int forward_tc(const ptrb200_ffnet* net, const Plan& p, const float* X, bool xb, bool x_masked, const int32_t* offsets, float* out,
                      char* ws, float drop, uint64_t seed, uint64_t offset, cudaStream_t st, bool fwd_only) {
    int rc;
    pack_weight_images(net, p, ws, fwd_only, st);
    for (int l = 0; l < p.L; ++l) {
        const LayerPlan& lp = p.layer[l];
        const bool last = l == p.L - 1;
        float* Z = (last && !lp.has_act && !lp.has_norm) ? out : reinterpret_cast<float*>(ws + lp.z_off);
        RowsGemmArgs g{};
        g.round_bf16 = p.bf16;
        set_prologue(net, p, l, ws, X, g.P, g.scale, g.shift, g.act);
        g.gr_prev = p.gr;
        g.drop = make_drop((last || (l == 0 && x_masked)) ? 0.0f : drop, seed, offset * 64 + (uint64_t)l);
        g.bias = net->bias[l]; g.Out = Z;
        g.a_out = (l > 0 && !fwd_only) ? reinterpret_cast<float*>(ws + lp.ain_off) : nullptr;     // a by-product for the backward pass
        g.partials = (lp.has_norm && !p.ragged) ? reinterpret_cast<double*>(ws + p.partials_off) : nullptr;
        g.rows = (int)p.rows; g.K = lp.d_in; g.N = lp.d_out;
        g.b_img_hi = reinterpret_cast<unsigned char*>(ws + lp.img_f_hi);
        g.b_img_lo = p.passes == 3 ? reinterpret_cast<unsigned char*>(ws + lp.img_f_lo) : nullptr;
        set_tiling(g, p);
        int S_fwd = p.S_stat;
        const int stats_kind = !g.partials ? 0 : (net->norm == PTRB200_NORM_BN ? 1 : 2);
        if ((rc = launch_rows_gemm(RG_FWD, p.passes, g, p.ntiles, st, stats_kind, &S_fwd, p.S_stat, xb && l == 0))) return rc;
        NormRef nr = norm_ref(net, p, l, ws);
        if (p.ragged) {
            if (lp.has_norm) {      // (under BN2 every layer with an activation has a norm)
                float* A = last ? out : reinterpret_cast<float*>(ws + lp.a_off);
                PTRB200_LAUNCH(bn2_ragged_moments_kernel, p.G, dim3(32, 8), 0, st, (const float*)Z, offsets,
                               reinterpret_cast<float*>(ws + lp.mean_off), reinterpret_cast<float*>(ws + lp.rstd_off), lp.d_out);
                PTRB200_LAUNCH(bn2_ragged_act_kernel, p.G, dim3(32, 8), 0, st, (const float*)Z, A, nr, offsets, lp.d_out);
            }
            continue;
        }
        if (lp.has_norm) {
            const int cnt = p.G * lp.d_out;
            const double* part = g.partials;
            const double* gcount = nullptr;
            if (p.sync_bn) {       // LTRBatchNorm over the GLOBAL batch: per-channel (sum, sum of squares, rows) summed over ranks
                double* buf = reinterpret_cast<double*>(ws + p.sync_off);
                PTRB200_LAUNCH(partials_fold_kernel, lp.d_out, FIN_THREADS, 0, st, (const double*)g.partials, buf, S_fwd, lp.d_out, (double)p.rows);
                if ((rc = call_hook(PTRB200_HOOK_ALLREDUCE_F64, l, buf, 2 * lp.d_out + 1, st))) return rc;
                part = buf; gcount = buf + 2 * lp.d_out; S_fwd = 1;
            }
            PTRB200_LAUNCH(moments_finalize_kernel, cnt, FIN_THREADS, 0, st, part,
                           reinterpret_cast<float*>(ws + lp.mean_off), reinterpret_cast<float*>(ws + lp.rstd_off),
                           reinterpret_cast<float*>(ws + lp.scale_off), reinterpret_cast<float*>(ws + lp.shift_off),
                           nr, p.G, lp.d_out, S_fwd, p.gr, gcount);
        }
        if (last && (lp.has_act || lp.has_norm)) {
            const size_t total = p.rows * lp.d_out;
            PTRB200_LAUNCH(norm_act_fwd_kernel, elementwise_blocks(total), 256, 0, st, (const float*)Z, out, nr, total, lp.d_out, p.gr);
        }
    }
    return check_launch("ffnet_forward(tc)");
}

static int backward_tc(const ptrb200_ffnet* net, const ptrb200_ffnet_grads* grads, const Plan& p, const float* X, bool xb, bool x_masked,
                       const int32_t* offsets, const float* dOut, float* dX, char* ws, float drop, uint64_t seed, uint64_t offset,
                       cudaStream_t st) {
    int rc;
    double* part = reinterpret_cast<double*>(ws + p.partials_off);
    float* S1 = reinterpret_cast<float*>(ws + p.s1_off);
    float* S2 = reinterpret_cast<float*>(ws + p.s2_off);
    float* dbuf[2] = {reinterpret_cast<float*>(ws + p.dbuf0_off), reinterpret_cast<float*>(ws + p.dbuf1_off)};
    float* wpart = reinterpret_cast<float*>(ws + p.wpart_off);
    const float* dA = dOut;
    int flip = 0;
    Rank1Src r1{nullptr, DropCfg{0, 1.0f, 0}, 0};   // pending outer-product data gradient of the single-output last layer
    for (int l = p.L - 1; l >= 0; --l) {
        const LayerPlan& lp = p.layer[l];
        const bool last = l == p.L - 1;
        if (!grads->weight[l] || !grads->bias[l]) { set_error("ffnet_backward: layer %d grad buffers NULL", l); return PTRB200_ERR_INVALID; }
        const float* Z = reinterpret_cast<const float*>(ws + lp.z_off);
        const float* dZ = dA;
        bool fuse_dz = false;
        NormRef nr = norm_ref(net, p, l, ws);
        const size_t total = p.rows * lp.d_out;
        if (lp.has_act || lp.has_norm) {
            float* dY = dbuf[flip]; flip ^= 1;
            if (p.ragged) PTRB200_LAUNCH(bn2_ragged_dy_kernel, p.G, dim3(32, 8), 0, st, Z, dA, dY, nr, offsets, part, lp.d_out);
            else launch_colstat<STAT_DY>(st, "colstat_dy", Z, dA, dY, nr, part, p.G, p.S_stat, p.gr, lp.d_out, p.slice_rows, r1);
            r1.w = nullptr;
            // one finalize launch: channel sums -> norm-parameter gradients, bias gradient, folded-dZ coefficients
            DyTail tail{};
            tail.nr = nr; tail.gr = p.gr;
            tail.bias_grad = grads->bias[l];
            // A Linear bias feeding a normalisation has an exactly-zero gradient (the norm removes every
            // per-channel shift); the reference's autograd produces rounding noise there.
            tail.bias_mode = lp.has_norm ? 1 : 2;
            if (lp.has_norm) {
                set_norm_grads(tail, net, grads, l);
                // fold dZ = a*rstd*(dY - S1/N - xhat*S2/N) into the operand staging of dgrad and wgrad when both can take it
                // (saves one 12-bytes-per-element pass); otherwise materialise dZ in place
                int Rf = 32, stf = 0;
                const int KPl = ((lp.d_in + 15) / 16) * 16;
                fuse_dz = !p.ragged && lp.d_out % 4 == 0 && lp.d_out <= 128 && lp.d_in <= 256 && (l == 0 || rows_ws_fits(lp.d_out, lp.d_in, p.passes)) &&
                          wgrad_smem(lp.d_out, lp.d_in, KPl, Rf, p.passes, stf, true, 24) <= (size_t)227 * 1024;
                if (fuse_dz) { tail.k1 = reinterpret_cast<float*>(ws + p.k1_off); tail.k3 = reinterpret_cast<float*>(ws + p.k3_off); tail.k0 = reinterpret_cast<float*>(ws + p.k0_off); }
            }
            int bS = p.S_stat;
            const double* fin_part = part;
            const double* gcount = nullptr;
            if (lp.has_norm && p.sync_bn) {   // S1 = sum dY, S2 = sum dY*xhat over the GLOBAL batch (same exchange as the forward moments)
                double* buf = reinterpret_cast<double*>(ws + p.sync_off);
                PTRB200_LAUNCH(partials_fold_kernel, lp.d_out, FIN_THREADS, 0, st, (const double*)part, buf, bS, lp.d_out, (double)p.rows);
                if ((rc = call_hook(PTRB200_HOOK_ALLREDUCE_F64, l, buf, 2 * lp.d_out + 1, st))) return rc;
                fin_part = buf; bS = 1; gcount = buf + 2 * lp.d_out;
                tail.counts = gcount;
            }
            PTRB200_LAUNCH(dy_finalize_kernel, lp.d_out, FIN_THREADS, 0, st, fin_part,
                           (lp.has_norm && !fuse_dz) ? S1 : (float*)nullptr, (lp.has_norm && !fuse_dz) ? S2 : (float*)nullptr,
                           (float*)nullptr, (float*)nullptr, p.G, lp.d_out, bS, tail);
            if (lp.has_norm && !fuse_dz) {
                if (p.ragged) PTRB200_LAUNCH(bn2_ragged_apply_kernel, p.G, dim3(32, 8), 0, st, Z, dY, nr, (const float*)S1, (const float*)S2, offsets, lp.d_out);
                else if (lp.d_out % 4 == 0) PTRB200_LAUNCH(norm_bwd_apply4_kernel, elementwise_blocks(total / 4), 256, 0, st, Z, dY, nr, (const float*)S1, (const float*)S2, total / 4, lp.d_out, p.gr, gcount);
                else PTRB200_LAUNCH(norm_bwd_apply_kernel, elementwise_blocks(total), 256, 0, st, Z, dY, nr, (const float*)S1, (const float*)S2, total, lp.d_out, p.gr, gcount);
            }
            dZ = dY;
        } else {        // bare Linear: the bias gradient is the column sum of the incoming gradient (a ragged batch: one group)
            const int G = p.ragged ? 1 : p.G, gr = p.ragged ? (int)p.rows : p.gr;
            launch_colstat<STAT_COLSUM>(st, "colstat_colsum", dA, nullptr, nullptr, nr, part, G, p.S_stat, gr, lp.d_out, p.slice_rows);
            PTRB200_LAUNCH(dy_finalize_kernel, lp.d_out, FIN_THREADS, 0, st, (const double*)part, (float*)nullptr, (float*)nullptr, grads->bias[l], (float*)nullptr, G, lp.d_out, p.S_stat, DyTail{});
        }
        // (x_masked: layer 0's input already carries its mask, and the caller applies it to dX)
        const DropCfg layer_drop = make_drop((last || (l == 0 && x_masked)) ? 0.0f : drop, seed, offset * 64 + (uint64_t)l);
        {   // dW = sum_rows dZ^T (x) layer input: dropout(X) rebuilt on the fly for layer 0, the operand the forward kernel built for deeper layers
            WgradArgs w{};
            w.round_bf16 = p.bf16;
            w.dZ = dZ;
            if (l == 0) { w.P = X; w.drop = layer_drop; }
            else { w.P = reinterpret_cast<const float*>(ws + lp.ain_off); w.drop = make_drop(0.0f, 0, 0); }
            w.partials = wpart;
            w.rows = (int)p.rows;
            if (fuse_dz) {
                w.Z2 = Z; w.gr_cur = p.gr;
                w.kc1 = reinterpret_cast<const float*>(ws + p.k1_off); w.kc3 = reinterpret_cast<const float*>(ws + p.k3_off); w.kc0 = reinterpret_cast<const float*>(ws + p.k0_off);
            }
            const WgBlocks wb = wgrad_blocks(lp.d_out, lp.d_in);
            if ((rc = launch_wgrad(w, lp.d_out, lp.d_in, wb.kb, dim3(wb.gx, wb.mblocks, wb.kblocks), p.passes, grads->weight[l], st, xb && l == 0))) return rc;
            // every parameter gradient of layer l is now enqueued: a data-parallel caller can start reducing it while the
            // layers below are still running (dist.GradBucket's overlapped all-reduce)
            if ((rc = call_hook(PTRB200_HOOK_LAYER_GRADS_READY, l, nullptr, 0, st))) return rc;
        }
        if (l > 0 || dX) {
            float* dIn = l == 0 ? dX : dbuf[flip];
            if (l > 0) flip ^= 1;
            // the next iteration's statistics pass rebuilds dIn = dropmask(dz (x) w) on the fly (dense plans only: the
            // per-query dY pass of a ragged batch reads a materialised dA)
            if (!p.ragged && lp.d_out == 1 && l > 0 && colstat_vectorised(lp.d_in) && (p.layer[l - 1].has_act || p.layer[l - 1].has_norm)) {
                r1.w = net->weight[l];
                r1.drop = layer_drop;
                r1.round_bf16 = p.bf16;
                flip ^= 1;                         // dIn's buffer stays unused; dZ (in the other one) must survive the next pass
                dA = dZ;
                continue;
            }
            if ((rc = launch_dgrad(net, p, l, ws, dZ, fuse_dz ? Z : nullptr, dIn, layer_drop, st))) return rc;
            dA = dIn;
        }
    }
    return check_launch("ffnet_backward(tc)");
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_set_hook(ptrb200_hook_fn fn, void* user) {
    g_hook = fn;
    g_hook_user = user;
    return PTRB200_OK;
}

int ptrb200_tc_wgrad(const float* dZ, const float* P, float* dW, float* partials, int rows, int N, int K, int passes,
                     ptrb200_stream_t stream) {
    if (!dZ || !P || !dW || !partials || rows <= 0 || N <= 0 || K <= 0) { set_error("tc_wgrad: bad arguments"); return PTRB200_ERR_INVALID; }
    if (N > 128 || K > 256 || K % 4 != 0) { set_error("tc_wgrad: needs N <= 128, K <= 256, K %% 4 == 0"); return PTRB200_ERR_UNSUPPORTED; }
    WgradArgs w{};
    w.dZ = dZ; w.P = P;
    w.drop = make_drop(0.0f, 0, 0); w.partials = partials;
    w.rows = rows;
    const int rc = launch_wgrad(w, N, K, K, dim3(296), passes, dW, (cudaStream_t)stream);     // 296 partial slots (header)
    return rc ? rc : check_launch("tc_wgrad");
}

int64_t ptrb200_ffnet_workspace_bytes(const ptrb200_ffnet* net, int x_dtype, int B, int n, int total_rows) {
    Plan p;
    const int rc = make_plan(net, B, n, p, total_rows, x_dtype);
    return rc ? (int64_t)rc : (int64_t)p.total;
}

// a bf16 feature matrix is read 4 elements (8 bytes) at a time
static int check_x(const void* X, int x_dtype, const char* who) {
    if (x_dtype == PTRB200_DTYPE_BF16 && (reinterpret_cast<uintptr_t>(X) & 7) != 0) {
        set_error("%s: bf16 features must be 8-byte aligned (X = %p)", who, X);
        return PTRB200_ERR_INVALID;
    }
    return PTRB200_OK;
}

int ptrb200_ffnet_forward(const ptrb200_ffnet* net, const void* Xv, int x_dtype, float* out, void* workspace,
                          int64_t workspace_bytes, int B, int n, const int32_t* offsets, int total_rows, int training,
                          uint64_t seed, uint64_t offset, ptrb200_stream_t stream) {
    Plan p;
    if ((offsets != nullptr) != (total_rows > 0)) { set_error("ffnet_forward: offsets and total_rows go together (ragged batch) or are both absent"); return PTRB200_ERR_INVALID; }
    int rc = make_plan(net, B, n, p, total_rows, x_dtype);
    if (rc) return rc;
    if (!Xv || !out || !workspace) { set_error("ffnet_forward: null buffer"); return PTRB200_ERR_INVALID; }
    if ((rc = check_x(Xv, x_dtype, "ffnet_forward"))) return rc;
    if ((size_t)workspace_bytes < p.total) { set_error("ffnet_forward: workspace %lld < %zu bytes", (long long)workspace_bytes, p.total); return PTRB200_ERR_WORKSPACE; }
    char* ws = static_cast<char*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    const float drop = (training & 1) ? net->dropout_p : 0.0f;
    const float* X = static_cast<const float*>(Xv);       // bf16: reinterpreted by the kernels that read it (xb)
    bool xb = p.x_bf16;
    ptrb200_ffnet padded;
    const DropCfg no_drop = make_drop(0.0f, 0, 0);
    if (p.pad_k) {          // zero-pad the features and the first weight matrix to a multiple of 4 columns (make_plan)
        // layer 0's dropout is applied in the copy, keyed by the unpadded index row * dims[0] + k (a padded index would
        // draw other masks than the SIMT path and the same features at their own width)
        const DropCfg d0 = make_drop(p.L > 1 ? drop : 0.0f, seed, offset * 64);
        float* Xp = reinterpret_cast<float*>(ws + p.xpad_off);
        float* Wp = reinterpret_cast<float*>(ws + p.w0pad_off);
        if (xb) PTRB200_LAUNCH(copy_cols_bf16_kernel, elementwise_blocks(p.rows * p.pad_k), 256, 0, st, static_cast<const uint16_t*>(Xv), Xp, p.rows, net->dims[0], p.pad_k, d0);
        else PTRB200_LAUNCH(copy_cols_kernel, elementwise_blocks(p.rows * p.pad_k), 256, 0, st, X, Xp, p.rows, net->dims[0], p.pad_k, d0);
        PTRB200_LAUNCH(copy_cols_kernel, elementwise_blocks((size_t)net->dims[1] * p.pad_k), 256, 0, st, net->weight[0], Wp, (size_t)net->dims[1], net->dims[0], p.pad_k, no_drop);
        padded = *net; padded.dims[0] = p.pad_k; padded.weight[0] = Wp;
        net = &padded; X = Xp; xb = false;
    } else if (xb && !p.use_tc) {       // the SIMT kernels read fp32: widen once into the workspace (backward reads it too)
        float* Xw = reinterpret_cast<float*>(ws + p.xwide_off);
        PTRB200_LAUNCH(copy_cols_bf16_kernel, elementwise_blocks(p.rows * net->dims[0]), 256, 0, st, static_cast<const uint16_t*>(Xv), Xw, p.rows, net->dims[0], net->dims[0], no_drop);
        X = Xw; xb = false;
    }
    if (p.use_tc) return forward_tc(net, p, X, xb, p.pad_k != 0, offsets, out, ws, drop, seed, offset, st, (training & PTRB200_FFNET_FORWARD_ONLY) != 0);
    const float* in = X;
    for (int l = 0; l < p.L; ++l) {
        const LayerPlan& lp = p.layer[l];
        const bool last = l == p.L - 1;
        float* Z = reinterpret_cast<float*>(ws + lp.z_off);
        float* A = last ? out : reinterpret_cast<float*>(ws + lp.a_off);
        float* lin_out = (lp.has_act || lp.has_norm) ? Z : A;     // a bare last Linear writes `out` directly
        GemmArgs g{};
        g.A = in; g.Bm = net->weight[l]; g.bias = net->bias[l]; g.C = lin_out;
        g.rows = (int)p.rows; g.d_in = lp.d_in; g.d_out = lp.d_out;
        g.M = (int)p.rows; g.N = lp.d_out; g.K = lp.d_in;
        g.drop = make_drop(last ? 0.0f : drop, seed, offset * 64 + (uint64_t)l);
        launch_gemm<GEMM_FWD>(g, 1, st);
        if (lp.has_act || lp.has_norm) {
            NormRef nr = norm_ref(net, p, l, ws);
            if (lp.has_norm) {
                double* part = reinterpret_cast<double*>(ws + p.partials_off);
                dim3 grid(p.G, p.S_stat);
                PTRB200_LAUNCH(colstat_kernel<STAT_MOMENTS>, grid, dim3(32, 8), 0, st, (const float*)Z, (const float*)nullptr,
                               (float*)nullptr, nr, part, p.gr, lp.d_out, p.S_stat, p.slice_rows);
                const int cnt = p.G * lp.d_out;
                PTRB200_LAUNCH(moments_finalize_kernel, cnt, FIN_THREADS, 0, st, (const double*)part,
                               reinterpret_cast<float*>(ws + lp.mean_off), reinterpret_cast<float*>(ws + lp.rstd_off),
                               (float*)nullptr, (float*)nullptr, nr, p.G, lp.d_out, p.S_stat, p.gr);
            }
            const size_t total = p.rows * lp.d_out;
            PTRB200_LAUNCH(norm_act_fwd_kernel, elementwise_blocks(total), 256, 0, st, (const float*)Z, A, nr, total, lp.d_out, p.gr);
        }
        in = A;
    }
    return check_launch("ffnet_forward");
}

int ptrb200_ffnet_backward(const ptrb200_ffnet* net, const ptrb200_ffnet_grads* grads, const void* Xv, int x_dtype,
                           const float* dOut, float* dX, void* workspace, int64_t workspace_bytes,
                           int B, int n, const int32_t* offsets, int total_rows, int training, uint64_t seed, uint64_t offset,
                           ptrb200_stream_t stream) {
    Plan p;
    if ((offsets != nullptr) != (total_rows > 0)) { set_error("ffnet_backward: offsets and total_rows go together (ragged batch) or are both absent"); return PTRB200_ERR_INVALID; }
    int rc = make_plan(net, B, n, p, total_rows, x_dtype);
    if (rc) return rc;
    if (!grads || !Xv || !dOut || !workspace) { set_error("ffnet_backward: null buffer"); return PTRB200_ERR_INVALID; }
    if ((rc = check_x(Xv, x_dtype, "ffnet_backward"))) return rc;
    if ((size_t)workspace_bytes < p.total) { set_error("ffnet_backward: workspace %lld < %zu bytes", (long long)workspace_bytes, p.total); return PTRB200_ERR_WORKSPACE; }
    // bf16 features: layer 0's weight-gradient kernel reads them natively on the tensor-core path; the padded and the
    // SIMT path read the fp32 copy the forward call left in the workspace
    const float* X = p.x_bf16 && !p.use_tc ? reinterpret_cast<const float*>(static_cast<char*>(workspace) + p.xwide_off)
                                           : static_cast<const float*>(Xv);
    const bool xb = p.x_bf16 && p.use_tc && !p.pad_k;
    char* ws = static_cast<char*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    const float drop = (training & 1) ? net->dropout_p : 0.0f;
    if (p.pad_k) {          // the forward call left the padded features and first weight matrix in the workspace
        ptrb200_ffnet padded = *net;
        ptrb200_ffnet_grads pg = *grads;
        padded.dims[0] = p.pad_k; padded.weight[0] = reinterpret_cast<const float*>(ws + p.w0pad_off);
        pg.weight[0] = reinterpret_cast<float*>(ws + p.dw0pad_off);
        float* dXp = dX ? reinterpret_cast<float*>(ws + p.dxpad_off) : nullptr;
        const float* Xp = reinterpret_cast<const float*>(ws + p.xpad_off);
        // Xp carries layer 0's dropout (forward call): layer 0 runs unmasked and its mask is applied to dX in the un-pad copy
        if ((rc = backward_tc(&padded, &pg, p, Xp, false, true, offsets, dOut, dXp, ws, drop, seed, offset, st))) return rc;
        if (!grads->weight[0]) { set_error("ffnet_backward: layer 0 grad buffer NULL"); return PTRB200_ERR_INVALID; }
        PTRB200_LAUNCH(copy_cols_kernel, elementwise_blocks((size_t)net->dims[1] * net->dims[0]), 256, 0, st, (const float*)pg.weight[0], grads->weight[0],
                       (size_t)net->dims[1], p.pad_k, net->dims[0], make_drop(0.0f, 0, 0));
        if (dX) PTRB200_LAUNCH(copy_cols_kernel, elementwise_blocks(p.rows * net->dims[0]), 256, 0, st, (const float*)dXp, dX, p.rows, p.pad_k, net->dims[0],
                               make_drop(p.L > 1 ? drop : 0.0f, seed, offset * 64));
        return check_launch("ffnet_backward(padded)");
    }
    if (p.use_tc) return backward_tc(net, grads, p, X, xb, false, offsets, dOut, dX, ws, drop, seed, offset, st);
    double* part = reinterpret_cast<double*>(ws + p.partials_off);
    float* S1 = reinterpret_cast<float*>(ws + p.s1_off);
    float* S2 = reinterpret_cast<float*>(ws + p.s2_off);
    float* dbuf[2] = {reinterpret_cast<float*>(ws + p.dbuf0_off), reinterpret_cast<float*>(ws + p.dbuf1_off)};
    float* wpart = reinterpret_cast<float*>(ws + p.wpart_off);
    const float* dA = dOut;                 // gradient w.r.t. the layer's post-activation output
    int flip = 0;
    for (int l = p.L - 1; l >= 0; --l) {
        const LayerPlan& lp = p.layer[l];
        const float* Z = reinterpret_cast<const float*>(ws + lp.z_off);
        const float* layer_in = l == 0 ? X : reinterpret_cast<const float*>(ws + p.layer[l - 1].a_off);
        if (!grads->weight[l] || !grads->bias[l]) { set_error("ffnet_backward: layer %d grad buffers NULL", l); return PTRB200_ERR_INVALID; }
        const float* dZ = dA;
        NormRef nr = norm_ref(net, p, l, ws);
        const size_t total = p.rows * lp.d_out;
        if (lp.has_act || lp.has_norm) {
            float* dY = dbuf[flip]; flip ^= 1;
            dim3 grid(p.G, p.S_stat);
            PTRB200_LAUNCH(colstat_kernel<STAT_DY>, grid, dim3(32, 8), 0, st, Z, dA, dY, nr, part, p.gr, lp.d_out, p.S_stat, p.slice_rows);
            // channel sums -> norm-parameter gradients, or without a norm the bias gradient (= sum dY)
            DyTail tail{};
            tail.nr = nr;
            if (lp.has_norm) set_norm_grads(tail, net, grads, l);
            else { tail.bias_grad = grads->bias[l]; tail.bias_mode = 2; }
            PTRB200_LAUNCH(dy_finalize_kernel, lp.d_out, FIN_THREADS, 0, st, (const double*)part,
                           lp.has_norm ? S1 : (float*)nullptr, lp.has_norm ? S2 : (float*)nullptr, (float*)nullptr, (float*)nullptr, p.G, lp.d_out, p.S_stat, tail);
            if (lp.has_norm) {
                PTRB200_LAUNCH(norm_bwd_apply_kernel, elementwise_blocks(total), 256, 0, st, Z, dY, nr, (const float*)S1, (const float*)S2, total, lp.d_out, p.gr);
                // bias gradient = column sums of dZ (zero up to rounding under a norm, as in the reference)
                PTRB200_LAUNCH(colstat_kernel<STAT_COLSUM>, grid, dim3(32, 8), 0, st, (const float*)dY, (const float*)nullptr, (float*)nullptr, nr, part, p.gr, lp.d_out, p.S_stat, p.slice_rows);
                PTRB200_LAUNCH(dy_finalize_kernel, lp.d_out, FIN_THREADS, 0, st, (const double*)part, (float*)nullptr, (float*)nullptr, grads->bias[l], (float*)nullptr, p.G, lp.d_out, p.S_stat, DyTail{});
            }
            dZ = dY;
        } else {
            dim3 grid(p.G, p.S_stat);
            PTRB200_LAUNCH(colstat_kernel<STAT_COLSUM>, grid, dim3(32, 8), 0, st, dA, (const float*)nullptr, (float*)nullptr, nr, part, p.gr, lp.d_out, p.S_stat, p.slice_rows);
            PTRB200_LAUNCH(dy_finalize_kernel, lp.d_out, FIN_THREADS, 0, st, (const double*)part, (float*)nullptr, (float*)nullptr, grads->bias[l], (float*)nullptr, p.G, lp.d_out, p.S_stat, DyTail{});
        }
        const bool last = l == p.L - 1;
        const float layer_drop = last ? 0.0f : drop;
        // dW = dZ^T * dropout(layer_in)
        {
            GemmArgs g{};
            g.A = dZ; g.Bm = layer_in; g.C = wpart;
            g.rows = (int)p.rows; g.d_in = lp.d_in; g.d_out = lp.d_out;
            g.M = lp.d_out; g.N = lp.d_in; g.K = (int)p.rows; g.k_chunk = p.k_chunk;
            g.drop = make_drop(layer_drop, seed, offset * 64 + (uint64_t)l);
            launch_gemm<GEMM_BWD_WEIGHT>(g, p.S_w, st);
            const int cnt = lp.d_in * lp.d_out;
            PTRB200_LAUNCH(reduce_splits_kernel, (cnt + 63) / 64, 256, 0, st, (const float*)wpart, grads->weight[l], p.S_w, cnt);
        }
        // dIn = dropout'(dZ * W)
        if (l > 0 || dX) {
            float* dIn = l == 0 ? dX : dbuf[flip];
            if (l > 0) flip ^= 1;
            GemmArgs g{};
            g.A = dZ; g.Bm = net->weight[l]; g.C = dIn;
            g.rows = (int)p.rows; g.d_in = lp.d_in; g.d_out = lp.d_out;
            g.M = (int)p.rows; g.N = lp.d_in; g.K = lp.d_out;
            g.drop = make_drop(layer_drop, seed, offset * 64 + (uint64_t)l);
            launch_gemm<GEMM_BWD_DATA>(g, 1, st);
            dA = dIn;
        }
    }
    return check_launch("ffnet_backward");
}

}  // extern "C"
