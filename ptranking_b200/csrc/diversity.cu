// diversity.cu -- the search-result-diversification path (ptranking/ltr_diversification/): DALETOR's alpha-DCG loss and
// its gradient, alpha-nDCG / ERR-IA / nERR-IA at several cutoffs, and the [q, q*d, d] input rows of the pointwise scorer.
//
// Subtopic relevance R of query q is a dense row-major [sub_counts[q], n_q] block starting at element rele_offsets[q]
// (documents in the query's presorted order, as DIVDataset stores q_doc_rele_mat).
#include "losses_common.cuh"

namespace ptrb200 {

// ---------------------------------------------------------------------------
// DALETOR: alphaDCG_as_a_loss, ltr_diversification/score_and_sort/daletor.py:8-40
// ---------------------------------------------------------------------------
// Forward, sigma = robust_sigmoid with scale rt:
//   sig_ij = sigma(rt (s_j - s_i)),  pi_i = 1/2 + sum_j sig_ij,  C_si = sum_j sig_ij R_sj - R_si / 2
//   g_si = R_si (1 - alpha)^C_si / log2(1 + pi_i),  L = -sum_{s < rows} sum_i g_si    (rows = min(top_k, m), or m)
// Backward, d_ij = rt sig_ij (1 - sig_ij):
//   a_i = sum_s g_si / ((1 + pi_i) ln(1 + pi_i)),  b_si = -ln(1 - alpha) g_si,  c_ij = a_i + sum_s b_si R_sj
//   dL/ds_k = sum_p d_pk (c_pk - c_kp) = sum_p d_pk [(a_p - a_k) + sum_s (b_sp R_sk - b_sk R_sp)]
// Subtopic rows beyond `rows` carry no weight (the reference slices rows, not documents, with top_k), so they are never
// read.  The rows go through shared memory DAL_SUB at a time: each chunk is one sweep over all pairs for C (the first
// one also sums pi) and one for the gradient (the last one also adds the a-terms).  Every per-document sum runs over its
// partners in index order with a fixed chunking, and the loss is summed from per-document values by one warp in a fixed
// pattern, so a query's results depend on neither the CTA width (256 threads, 1024 for launches with lists above 512
// documents) nor the launch it is in.
constexpr int DAL_SUB = 4;

static inline int daletor_threads(int n) { return n > 512 ? 1024 : 256; }
static inline size_t daletor_smem(int n) { return (size_t)n * 4 * (5 + 2 * DAL_SUB); }

__global__ void __launch_bounds__(1024)
daletor_kernel(const float* __restrict__ scores, const int32_t* __restrict__ offsets, const float* __restrict__ rele,
               const int64_t* __restrict__ rele_offsets, const int32_t* __restrict__ sub_counts, float* __restrict__ grad,
               float* __restrict__ loss_q, int nmax, int mmax, float rt, float log_q, float neg_ln_q, int top_k) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* ss = reinterpret_cast<float*>(smem_raw);   // scores
    float* pis = ss + nmax;                           // pi_i
    float* as = pis + nmax;                           // sum_s g_si, then a_i
    float* gacc = as + nmax;                          // gradient
    float* Rt = gacc + nmax;                          // [DAL_SUB][nmax] rows of R
    float* bt = Rt + DAL_SUB * nmax;                  // [DAL_SUB][nmax] b_si of those rows
    float* ls = bt + DAL_SUB * nmax;                  // document i's share of the loss, sum_s g_si
    const int b = blockIdx.x, tid = threadIdx.x, T = blockDim.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n;
    const int m = clampi(sub_counts[b], 0, mmax);
    const int rows = top_k > 0 ? min(top_k, m) : m;
    const float* R = rele + rele_offsets[b];
    for (int i = tid; i < n; i += T) { ss[i] = scores[sp.base + i]; as[i] = 0.0f; gacc[i] = 0.0f; }
    __syncthreads();
    for (int c0 = 0; c0 < rows; c0 += DAL_SUB) {
        const int cs = min(DAL_SUB, rows - c0);
        const bool first = c0 == 0, last = c0 + DAL_SUB >= rows;
        for (int idx = tid; idx < DAL_SUB * n; idx += T) {
            const int t = idx / n, j = idx - t * n;
            Rt[t * nmax + j] = t < cs ? R[(size_t)(c0 + t) * n + j] : 0.0f;
        }
        __syncthreads();
        for (int i = tid; i < n; i += T) {
            const float si = ss[i];
            float acc[DAL_SUB], pi = 0.0f;
#pragma unroll
            for (int t = 0; t < DAL_SUB; ++t) acc[t] = 0.0f;
            for (int j = 0; j < n; ++j) {
                const float sg = robust_sigmoid(ss[j] - si, rt);
                if (first) pi += sg;
#pragma unroll
                for (int t = 0; t < DAL_SUB; ++t) acc[t] += sg * Rt[t * nmax + j];
            }
            if (first) { pi += 0.5f; pis[i] = pi; } else pi = pis[i];
            const float lg = log2f(1.0f + pi);
            float gs = 0.0f;
#pragma unroll
            for (int t = 0; t < DAL_SUB; ++t) {
                const float r = Rt[t * nmax + i];
                const float g = t < cs ? r * exp2f(log_q * (acc[t] - 0.5f * r)) / lg : 0.0f;
                gs += g;
                bt[t * nmax + i] = neg_ln_q * g;
            }
            float a = as[i] + gs;
            if (last) { ls[i] = a; a /= (1.0f + pi) * logf(1.0f + pi); }
            as[i] = a;
        }
        __syncthreads();
        for (int k = tid; k < n; k += T) {
            const float sk = ss[k], ak = last ? as[k] : 0.0f;
            float rk[DAL_SUB], bk[DAL_SUB];
#pragma unroll
            for (int t = 0; t < DAL_SUB; ++t) { rk[t] = Rt[t * nmax + k]; bk[t] = bt[t * nmax + k]; }
            float acc = 0.0f;
            for (int p = 0; p < n; ++p) {
                const float sg = robust_sigmoid(sk - ss[p], rt);
                float v = last ? as[p] - ak : 0.0f;
#pragma unroll
                for (int t = 0; t < DAL_SUB; ++t) v += bt[t * nmax + p] * rk[t] - bk[t] * Rt[t * nmax + p];
                acc += (rt * sg * (1.0f - sg)) * v;
            }
            gacc[k] += acc;
        }
        __syncthreads();
    }
    for (int k = tid; k < n; k += T) grad[sp.base + k] = gacc[k];
    if (tid < 32) {
        float v = 0.0f;
        if (rows > 0)
            for (int i = tid; i < n; i += 32) v += ls[i];
        v = warp_sum(v);
        if (tid == 0) loss_q[b] = -v;
    }
}

// ---------------------------------------------------------------------------
// alpha-nDCG@ks, ERR-IA@ks, nERR-IA@ks: metric/srd/diversity_metric.py:12-103, 190-290
// ---------------------------------------------------------------------------
// One CTA per query: the scores are sorted once (descending, ties by ascending index), then four warps walk the ranked
// positions with one lane per subtopic -- alpha-DCG of the system and of the ideal (input) order, ERR-IA of both --
// and record the running sums at the cutoffs.
constexpr int SRD_THREADS = 256;

__global__ void __launch_bounds__(SRD_THREADS)
srd_metrics_kernel(const float* __restrict__ scores, const int32_t* __restrict__ offsets, const float* __restrict__ rele,
                   const int64_t* __restrict__ rele_offsets, const int32_t* __restrict__ sub_counts, Cutoffs ks,
                   float* __restrict__ out, int32_t* __restrict__ flags, int32_t* __restrict__ order, int nmax, int npow2max,
                   int mmax, float one_minus_alpha, float inv_2_max_label) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    int* ord = reinterpret_cast<int*>(keys + npow2max);
    __shared__ float cum[4][PTRB200_MAX_CUTOFFS];
    __shared__ float red[33];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    const int m = clampi(sub_counts[b], 0, mmax);
    const float* R = rele + rele_offsets[b];
    float* o = out + (size_t)b * 3 * ks.n;
    float tot = 0.0f;
    for (int e = tid; e < m * n; e += SRD_THREADS) tot += R[e];
    tot = block_sum(tot, red);
    if (tid == 0) flags[b] = (tot >= 1.0f ? PTRB200_SRD_RELE_GE1 : 0) | (tot > 0.0f ? PTRB200_SRD_RELE_GT0 : 0);
    if (n == 0) {
        for (int c = tid; c < 3 * ks.n; c += SRD_THREADS) o[c] = 0.0f;
        return;
    }
    for (int i = tid; i < npow2; i += SRD_THREADS) keys[i] = i < n ? desc_key(scores[sp.base + i], i) : 0ull;
    block_sort_desc(keys, npow2);
    for (int r = tid; r < n; r += SRD_THREADS) {
        ord[r] = key_index(keys[r]);
        if (order) order[sp.base + r] = ord[r];
    }
    __syncthreads();
    int kmax = 0;
    for (int c = 0; c < ks.n; ++c) if (ks.k[c] <= n) kmax = ks.k[c];
    if (warp < 4) {
        const bool sys = (warp & 1) == 0, err = warp >= 2;
        const bool on = lane < m;
        float cnt = 0.0f, casc = 1.0f, run = 0.0f;   // lane's cover count / unsatisfied probability; running sum
        int c = 0;
        for (int p = 0; p < kmax; ++p) {
            const int doc = sys ? ord[p] : p;
            const float r = on ? R[(size_t)lane * n + doc] : 0.0f;
            float v;
            if (!err) {
                v = r * powf(one_minus_alpha, cnt);
                cnt += r;
            } else {
                const float sat = (exp2f(r) - 1.0f) * inv_2_max_label;
                v = sat * casc;
                casc *= 1.0f - sat;
            }
            v = warp_sum(v);
            run += err ? v / (float)(p + 1) : v / log2f((float)p + 2.0f);
            while (c < ks.n && ks.k[c] == p + 1) { if (lane == 0) cum[warp][c] = run; ++c; }
        }
    }
    __syncthreads();
    for (int c = tid; c < ks.n; c += SRD_THREADS) {
        float andcg = 0.0f, err_ia = 0.0f, nerr_ia = 0.0f;
        if (ks.k[c] <= n) {
            const float dsys = cum[0][c], dide = cum[1][c];
            andcg = dide > 0.0f ? dsys / dide : 0.0f;
            const float esys = m > 0 ? cum[2][c] / (float)m : 0.0f, eide = m > 0 ? cum[3][c] / (float)m : 0.0f;
            err_ia = esys;
            nerr_ia = eide > 0.0f ? esys / eide : 0.0f;
        }
        o[c] = andcg;
        o[ks.n + c] = err_ia;
        o[2 * ks.n + c] = nerr_ia;
    }
}

// ---------------------------------------------------------------------------
// [q, q*d, d] rows: DivPointNeuralRanker.div_forward, ltr_diversification/base/div_point_ranker.py:14-19
// ---------------------------------------------------------------------------
__global__ void div_features_kernel(const float* __restrict__ q_repr, const float* __restrict__ docs,
                                    const int32_t* __restrict__ offsets, float* __restrict__ out, int nmax, int F) {
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const float* q = q_repr + (size_t)b * F;
    for (size_t e = threadIdx.x; e < (size_t)sp.n * F; e += blockDim.x) {
        const size_t row = sp.base + e / F;
        const int f = (int)(e % F);
        const float qv = q[f], dv = docs[row * F + f];
        float* orow = out + row * 3 * F;
        orow[f] = qv;
        orow[F + f] = qv * dv;
        orow[2 * F + f] = dv;
    }
}

// ---------------------------------------------------------------------------
// The diversification list scorer, ltr_diversification/base/div_list_ranker.py:61-85
// ---------------------------------------------------------------------------
// Encoder input [q, d, q*d] (note: d before q*d, unlike the pointwise [q, q*d, d]).
__global__ void div_list_features_kernel(const float* __restrict__ q_repr, const float* __restrict__ docs,
                                         const int32_t* __restrict__ offsets, float* __restrict__ out, int nmax, int F) {
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const float* q = q_repr + (size_t)b * F;
    for (size_t e = threadIdx.x; e < (size_t)sp.n * F; e += blockDim.x) {
        const size_t row = sp.base + e / F;
        const int f = (int)(e % F);
        const float qv = q[f], dv = docs[row * F + f];
        float* orow = out + row * 3 * F;
        orow[f] = qv;
        orow[F + f] = dv;
        orow[2 * F + f] = qv * dv;
    }
}

// A length class of a ragged batch: query b of the class is query qidx[b] (b when qidx is NULL) of the prefix offsets,
// padded to n_max rows.  One CTA per (class query, row block), as pad_lists_kernel.
//   PAD:  padded[b, r, 0:W] = src[(offsets[q] + r) * ld_src + 0:W] for r < len_q, 0 for len_q <= r < n_max
//   !PAD: the scorer input of the class's rows: out[row, 0:W] = feats[row, 0:W], out[row, W:2W] = enc[b, r, 0:W]
template <bool PAD>
__global__ void div_list_rows_kernel(const float* __restrict__ src, long long ld_src, const float* __restrict__ enc,
                                     const int32_t* __restrict__ offsets, const int32_t* __restrict__ qidx,
                                     float* __restrict__ dst, int n_max, int W) {
    const int b = blockIdx.x;
    const int q = qidx ? qidx[b] : b;
    const int base = offsets[q], n = min(offsets[q + 1] - base, n_max);
    for (int r = blockIdx.y; r < (PAD ? n_max : n); r += gridDim.y) {
        if (PAD) {
            const float* s = src + (size_t)(base + r) * ld_src;
            float* d = dst + ((size_t)b * n_max + r) * W;
            const bool live = r < n;
            for (int f = threadIdx.x; f < W; f += blockDim.x) d[f] = live ? s[f] : 0.0f;
        } else {
            const size_t row = (size_t)(base + r);
            const float* s = src + row * W;
            const float* e = enc + ((size_t)b * n_max + r) * W;
            float* d = dst + row * 2 * W;
            for (int f = threadIdx.x; f < W; f += blockDim.x) { d[f] = s[f]; d[W + f] = e[f]; }
        }
    }
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_daletor_fwd_bwd(const float* scores, const int32_t* offsets, const float* rele, const int64_t* rele_offsets,
                            const int32_t* sub_counts, float* grad, float* loss_per_query, int B, int n, int m, float rt,
                            float alpha, int top_k, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, rele, grad, loss_per_query, B, n);
    if (rc) return rc;
    if ((rc = check_rele_args("daletor", rele, rele_offsets, sub_counts, m))) return rc;
    if (!(alpha >= 0.0f && alpha < 1.0f)) { set_error("daletor: alpha=%g outside [0, 1)", alpha); return PTRB200_ERR_INVALID; }
    if (!(rt > 0.0f)) { set_error("daletor: rt must be positive"); return PTRB200_ERR_INVALID; }
    const float ln_q = logf(1.0f - alpha), log2_q = log2f(1.0f - alpha);
    const size_t smem = daletor_smem(n);
    if ((rc = allow_smem(daletor_kernel, smem))) return rc;
    PTRB200_LAUNCH(daletor_kernel, B, daletor_threads(n), smem, stream, scores, offsets, rele, rele_offsets, sub_counts, grad,
                   loss_per_query, n, m, rt, log2_q, -ln_q, top_k);
    return check_launch("daletor");
}

int ptrb200_srd_metrics_at_ks(const float* scores, const int32_t* offsets, const float* rele, const int64_t* rele_offsets,
                              const int32_t* sub_counts, const int32_t* ks_host, int nks, float* out, int32_t* flags,
                              int32_t* order, int B, int n, int m, float alpha, float max_label, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, rele, out, flags, B, n);
    if (rc) return rc;
    if ((rc = check_rele_args("srd_metrics", rele, rele_offsets, sub_counts, m))) return rc;
    if (!ks_host || nks <= 0 || nks > PTRB200_MAX_CUTOFFS) {
        set_error("srd_metrics: nks=%d outside 1..%d", nks, PTRB200_MAX_CUTOFFS);
        return PTRB200_ERR_INVALID;
    }
    Cutoffs ks;
    ks.n = nks;
    for (int c = 0; c < nks; ++c) {
        ks.k[c] = ks_host[c];
        if (ks.k[c] <= 0 || (c > 0 && ks.k[c] < ks.k[c - 1])) { set_error("srd_metrics: cutoffs must be positive and non-decreasing"); return PTRB200_ERR_INVALID; }
    }
    const int npow2 = next_pow2(n);
    const size_t smem = (size_t)npow2 * 8 + (size_t)n * 4;
    // the kernel also has static shared memory (cum, red): opt in once dynamic + static passes 48 KB
    if ((rc = allow_smem(srd_metrics_kernel, smem + 1024))) return rc;
    PTRB200_LAUNCH(srd_metrics_kernel, B, SRD_THREADS, smem, stream, scores, offsets, rele, rele_offsets, sub_counts, ks, out,
                   flags, order, n, npow2, m, 1.0f - alpha, exp2f(-max_label));
    return check_launch("srd_metrics");
}

int ptrb200_div_features(const float* q_repr, const float* docs, const int32_t* offsets, float* out, int B, int n, int F,
                         ptrb200_stream_t stream) {
    if (!q_repr || !docs || !out || B <= 0 || n <= 0 || F <= 0) {
        set_error("div_features: null pointer or non-positive size (B=%d n=%d F=%d)", B, n, F);
        return PTRB200_ERR_INVALID;
    }
    PTRB200_LAUNCH(div_features_kernel, B, 256, 0, stream, q_repr, docs, offsets, out, n, F);
    return check_launch("div_features");
}

int ptrb200_div_list_features(const float* q_repr, const float* docs, const int32_t* offsets, float* out, int B, int n,
                              int F, ptrb200_stream_t stream) {
    if (!q_repr || !docs || !out || B <= 0 || n <= 0 || F <= 0) {
        set_error("div_list_features: null pointer or non-positive size (B=%d n=%d F=%d)", B, n, F);
        return PTRB200_ERR_INVALID;
    }
    PTRB200_LAUNCH(div_list_features_kernel, B, 256, 0, stream, q_repr, docs, offsets, out, n, F);
    return check_launch("div_list_features");
}

static inline int div_list_threads(int W) { return W >= 128 ? 128 : ((W + 31) / 32) * 32; }

int ptrb200_pad_lists_pitched(const float* src, long long ld_src, const int32_t* offsets, const int32_t* qidx,
                              float* padded, int B, int n_max, int W, ptrb200_stream_t stream) {
    if (!src || !offsets || !padded || B <= 0 || n_max <= 0 || W <= 0 || ld_src < W) {
        set_error("pad_lists_pitched: bad arguments (B=%d n_max=%d W=%d ld_src=%lld)", B, n_max, W, ld_src);
        return PTRB200_ERR_INVALID;
    }
    PTRB200_LAUNCH_TAG("pad_lists_pitched_kernel", div_list_rows_kernel<true>, dim3(B, n_max < 64 ? n_max : 64), div_list_threads(W), 0, stream, src,
                   ld_src, nullptr, offsets, qidx, padded, n_max, W);
    return check_launch("pad_lists_pitched");
}

int ptrb200_div_list_concat(const float* feats, const float* enc, const int32_t* offsets, const int32_t* qidx, float* out,
                            int B, int n_max, int W, ptrb200_stream_t stream) {
    if (!feats || !enc || !offsets || !out || B <= 0 || n_max <= 0 || W <= 0) {
        set_error("div_list_concat: bad arguments (B=%d n_max=%d W=%d)", B, n_max, W);
        return PTRB200_ERR_INVALID;
    }
    PTRB200_LAUNCH_TAG("div_list_concat_kernel", div_list_rows_kernel<false>, dim3(B, n_max < 64 ? n_max : 64), div_list_threads(W), 0, stream, feats,
                   (long long)W, enc, offsets, qidx, out, n_max, W);
    return check_launch("div_list_concat");
}

}  // extern "C"
