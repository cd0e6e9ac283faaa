// divprob.cu -- DivProbRanker (ltr_diversification/score_and_sort/div_prob_ranker.py, base/div_mdn_ranker.py): the
// Gaussian head over the scorer's raw output, the expected-rank losses SuperSoft-aNDCG / SuperSoft-nERR-IA, the
// pairwise classification losses PairCLS / LambdaPairCLS, their gradients w.r.t. the raw output, and the sort keys.
//
// Head (div_mdn_ranker.py:276-299), per document u = raw[row, 0:D]:
//   K = 1 (D = 2):  mu = u0, v = T(u1);   K > 1 (D = 3K):  w = softmax(u[0:K]), mu = sum_k w_k u[K+k], v = sum_k w_k T(u[2K+k])
//   T(x) = exp(x), or limit_delta * sigmoid(x) with limit_delta set.
// Pairs (prob_utils.py:62-80), never stored:  x_ij = (mu_i - mu_j) / sqrt(2 (v_i + v_j)),  P_ij = erfc(x_ij) / 2 (the
// probability that j ranks above i), P_ii = 0,  E_i = 1 + sum_j P_ij (expected rank).
// With c_ij = dL/dP_ij and A_kj = c_kj - c_jk, w_kj = exp(-x_kj^2) / (sqrt(pi) sqrt(2 (v_k + v_j))):
//   dL/dmu_k = -sum_j w_kj A_kj,   dL/dv_k = sum_j w_kj x_kj / sqrt(2 (v_k + v_j)) A_kj
// and the head's chain rule gives d loss / d raw.  Per loss (DESIGN §4):
//   aNDCG:   L = -sum_{s<rows} sum_i g_si, g_si = R_si (1-beta)^C_si / log2(1+E_i), C_si = sum_j P_ij R_sj;
//            c_ij = a_i + sum_s b_si R_sj, a_i = sum_s g_si / ((1+E_i) ln(1+E_i)), b_si = -ln(1-beta) g_si
//   nERR-IA: L = -sum_s sum_{i<K} sat_si casc_si / E_i;  c_ij = sum_s sat_si casc_si / E_i^2 (i < K)
//   PairCLS / LambdaPairCLS: L = sum_{i<j} W_ij BCE(1 - P_ij, t_ij);  c_ij = -W_ij dBCE/dp for i < j, 0 otherwise
//
// One CTA of DP_THREADS per query.  mu, v, E, a and the per-document loss shares live in shared memory (5 n floats,
// 80 KB at n = 4096).  A thread owns documents k = tid, tid + DP_THREADS, ...; for each owned document it keeps its
// subtopic column (and b_k / G_k, h_k) in registers and walks every partner j in index order, the partners' columns
// passing through shared memory DP_TJ documents at a time.  Per-document subtopic values that partners need (b for
// aNDCG, h = D_j (1-beta)^cover for LambdaPairCLS) go to a workspace laid out like the relevance blocks.  Every
// per-document sum runs over its partners in index order and the loss is summed by one warp in a fixed pattern, so a
// query's results do not depend on the launch it is in.
#include "losses_common.cuh"

namespace ptrb200 {

constexpr int DP_THREADS = 256;
constexpr int DP_TJ = 32;
constexpr int DP_MS = PTRB200_MAX_SUBTOPICS;
constexpr int DP_KEY = 4;   // forward-only mode: the sort key

static __device__ __forceinline__ float dp_var(float u, float limit) {
    return limit > 0.0f ? (1.0f / (1.0f + expf(-u))) * limit : expf(u);
}
static __device__ __forceinline__ float dp_dvar(float u, float limit) {
    if (limit > 0.0f) { const float s = 1.0f / (1.0f + expf(-u)); return limit * s * (1.0f - s); }
    return expf(u);
}

static __device__ void dp_head(const float* __restrict__ u, int K, float limit, float& mu, float& var) {
    if (K == 1) { mu = u[0]; var = dp_var(u[1], limit); return; }
    float mx = u[0];
    for (int k = 1; k < K; ++k) mx = fmaxf(mx, u[k]);
    float se = 0.0f;
    for (int k = 0; k < K; ++k) se += expf(u[k] - mx);
    mu = 0.0f; var = 0.0f;
    for (int k = 0; k < K; ++k) {
        const float w = expf(u[k] - mx) / se;
        mu += w * u[K + k];
        var += w * dp_var(u[2 * K + k], limit);
    }
}

static __device__ void dp_head_bwd(const float* __restrict__ u, int K, float limit, float gmu, float gv, float* __restrict__ du) {
    if (K == 1) { du[0] = gmu; du[1] = gv * dp_dvar(u[1], limit); return; }
    float mx = u[0];
    for (int k = 1; k < K; ++k) mx = fmaxf(mx, u[k]);
    float se = 0.0f;
    for (int k = 0; k < K; ++k) se += expf(u[k] - mx);
    float dot = 0.0f;
    for (int k = 0; k < K; ++k) {
        const float w = expf(u[k] - mx) / se;
        dot += w * (gmu * u[K + k] + gv * dp_var(u[2 * K + k], limit));
    }
    for (int k = 0; k < K; ++k) {
        const float w = expf(u[k] - mx) / se;
        const float dw = gmu * u[K + k] + gv * dp_var(u[2 * K + k], limit);
        du[k] = w * (dw - dot);
        du[K + k] = gmu * w;
        du[2 * K + k] = gv * w * dp_dvar(u[2 * K + k], limit);
    }
}

// Partners [j0, j0 + DP_TJ): rows 0..ms of R (and of X, and G = 2^R - 1 when asked) into tile[s][t].
static __device__ __forceinline__ void dp_load_tile(int j0, int n, int ms, const float* __restrict__ R,
                                                    const float* __restrict__ X, bool gains, float* tR, float* tX, float* tG) {
    __syncthreads();
    for (int e = threadIdx.x; e < ms * DP_TJ; e += DP_THREADS) {
        const int s = e / DP_TJ, j = j0 + e - s * DP_TJ;
        const float r = j < n ? R[(size_t)s * n + j] : 0.0f;
        tR[e] = r;
        if (X) tX[e] = j < n ? X[(size_t)s * n + j] : 0.0f;
        if (gains) tG[e] = exp2f(r) - 1.0f;
    }
    __syncthreads();
}

template <int MODE>
__global__ void __launch_bounds__(DP_THREADS, 1)
divprob_kernel(const float* __restrict__ raw, int D, const int32_t* __restrict__ offsets, const float* __restrict__ rele,
               const int64_t* __restrict__ rele_offsets, const int32_t* __restrict__ sub_counts, float* __restrict__ ws,
               float* __restrict__ out, float* __restrict__ loss_q, int nmax, int mmax, int K, float limit, int top_k,
               int flag, float log2_q, float neg_ln_q) {
    // MODE: PTRB200_DIVPROB_* loss, or DP_KEY (out = sort key [rows], flag = sort id).  Otherwise out = d loss / d raw
    // and flag = LambdaPairCLS's norm.
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* mus = reinterpret_cast<float*>(smem_raw);
    float* vs = mus + nmax;
    float* Es = vs + nmax;
    float* as = Es + nmax;
    float* ls = as + nmax;
    float* tR = ls + nmax;                 // [ms][DP_TJ]
    float* tX = tR + mmax * DP_TJ;
    float* tG = tX + mmax * DP_TJ;
    __shared__ float idcg_s;
    const int b = blockIdx.x, tid = threadIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n;
    const int rounds = (n + DP_THREADS - 1) / DP_THREADS;
    const int m = (MODE == DP_KEY) ? 0 : clampi(sub_counts[b], 0, mmax);
    const float* R = (MODE == DP_KEY) ? nullptr : rele + rele_offsets[b];
    float* W = (MODE == PTRB200_DIVPROB_ANDCG || MODE == PTRB200_DIVPROB_LAMBDA_PAIRCLS) ? ws + rele_offsets[b] : nullptr;
    const float* U = raw + sp.base * (size_t)D;

    for (int i = tid; i < n; i += DP_THREADS) {
        float mu, v;
        dp_head(U + (size_t)i * D, K, limit, mu, v);
        mus[i] = mu; vs[i] = v; ls[i] = 0.0f; as[i] = 0.0f;
    }
    __syncthreads();

    // ---- expected ranks E_i = 1 + sum_{j != i} P_ij ----
    const bool need_E = MODE == PTRB200_DIVPROB_ANDCG || MODE == PTRB200_DIVPROB_NERRIA || (MODE == DP_KEY && flag == PTRB200_DIVPROB_KEY_RERAR);
    if (need_E) {
        for (int k = tid; k < n; k += DP_THREADS) {
            const float mk = mus[k], vk = vs[k];
            float acc = 0.0f;
            for (int j = 0; j < n; ++j)
                if (j != k) acc += 0.5f * erfcf((mk - mus[j]) / sqrtf(2.0f * (vk + vs[j])));
            Es[k] = acc + 1.0f;
        }
        __syncthreads();
    }
    if (MODE == DP_KEY) {
        for (int k = tid; k < n; k += DP_THREADS)
            out[sp.base + k] = flag == PTRB200_DIVPROB_KEY_RERAR ? 1.0f / Es[k]
                             : flag == PTRB200_DIVPROB_KEY_RISKAWARE ? mus[k] - 0.1f * vs[k] : mus[k];
        return;
    }

    // ---- per-document coefficients ----
    const int rows = (MODE == PTRB200_DIVPROB_ANDCG) ? (top_k > 0 ? min(top_k, m) : m) : m;
    if (MODE == PTRB200_DIVPROB_ANDCG) {
        // C_si = sum_j P_ij R_sj over s < rows, then g, a, b (b to the workspace: the partners read it)
        for (int r = 0; r < rounds; ++r) {
            const int k = tid + r * DP_THREADS;
            const bool own = k < n;
            const float mk = own ? mus[k] : 0.0f, vk = own ? vs[k] : 0.0f;
            float acc[DP_MS];
#pragma unroll
            for (int s = 0; s < DP_MS; ++s) acc[s] = 0.0f;
            for (int j0 = 0; j0 < n; j0 += DP_TJ) {
                dp_load_tile(j0, n, rows, R, nullptr, false, tR, tX, tG);
                if (!own) continue;
                const int jt = min(DP_TJ, n - j0);
                for (int t = 0; t < jt; ++t) {
                    const int j = j0 + t;
                    const float P = j == k ? 0.0f : 0.5f * erfcf((mk - mus[j]) / sqrtf(2.0f * (vk + vs[j])));
#pragma unroll
                    for (int s = 0; s < DP_MS; ++s) {
                        if (s >= rows) break;
                        acc[s] += P * tR[s * DP_TJ + t];
                    }
                }
            }
            if (own) {
                const float E = Es[k], lg = log2f(1.0f + E);
                float gs = 0.0f;
#pragma unroll
                for (int s = 0; s < DP_MS; ++s) {
                    if (s >= rows) break;
                    const float g = R[(size_t)s * n + k] * exp2f(log2_q * acc[s]) / lg;
                    gs += g;
                    W[(size_t)s * n + k] = neg_ln_q * g;
                }
                ls[k] = gs;
                as[k] = gs / ((1.0f + E) * logf(1.0f + E));
            }
        }
        __syncthreads();
    } else if (MODE == PTRB200_DIVPROB_NERRIA) {
        // one warp walks the documents in order, one lane per subtopic: casc_si = prod_{j<i} (1 - sat_sj)
        if (tid < 32) {
            const int kd = top_k > 0 ? min(top_k, n) : n;
            const bool on = tid < m;
            float casc = 1.0f;
            for (int i = 0; i < kd; ++i) {
                const float sat = on ? (exp2f(R[(size_t)tid * n + i]) - 1.0f) / 2.0f : 0.0f;
                const float E = Es[i];
                const float w = warp_sum(sat * casc);
                const float l = warp_sum((1.0f / E) * sat * casc);
                casc *= 1.0f - sat;
                if (tid == 0) { ls[i] = l; as[i] = w / (E * E); }
            }
        }
        __syncthreads();
    } else if (MODE == PTRB200_DIVPROB_LAMBDA_PAIRCLS) {
        // h_sj = (1-beta)^{sum_{i<j} R_si} / log2(j+2) to the workspace; the ideal alpha-DCG (gains R) for the norm
        if (tid < 32) {
            const bool on = tid < m;
            float cnt = 0.0f, dcg = 0.0f;
            for (int j = 0; j < n; ++j) {
                const float r = on ? R[(size_t)tid * n + j] : 0.0f;
                const float f = exp2f(log2_q * cnt), lj = log2f((float)j + 2.0f);
                if (on) W[(size_t)tid * n + j] = (1.0f / lj) * f;
                dcg += f * r / lj;
                cnt += r;
            }
            dcg = warp_sum(dcg);
            if (tid == 0) idcg_s = dcg;
        }
        __syncthreads();
    }

    // ---- gradient: one sweep over the partners per owned document ----
    constexpr bool PAIR = MODE == PTRB200_DIVPROB_PAIRCLS || MODE == PTRB200_DIVPROB_LAMBDA_PAIRCLS;
    constexpr bool LAMBDA = MODE == PTRB200_DIVPROB_LAMBDA_PAIRCLS;
    const int ms = (MODE == PTRB200_DIVPROB_NERRIA) ? 0 : rows;
    const float inv_m = 1.0f / (float)m;
    const bool norm = flag != 0;
    const float idcg = LAMBDA ? idcg_s : 1.0f;
    const float inv_sqrt_pi = 0.56418958354775628f;
    for (int r = 0; r < rounds; ++r) {
        const int k = tid + r * DP_THREADS;
        const bool own = k < n;
        const float mk = own ? mus[k] : 0.0f, vk = own ? vs[k] : 0.0f, ak = own ? as[k] : 0.0f;
        float rk[DP_MS], xk[DP_MS], gk[DP_MS];
#pragma unroll
        for (int s = 0; s < DP_MS; ++s) {
            const bool on = own && s < ms;
            rk[s] = on ? R[(size_t)s * n + k] : 0.0f;
            xk[s] = on && W ? W[(size_t)s * n + k] : 0.0f;
            gk[s] = LAMBDA ? exp2f(rk[s]) - 1.0f : 0.0f;
        }
        float gm = 0.0f, gv = 0.0f, lsum = 0.0f;
        for (int j0 = 0; j0 < n; j0 += DP_TJ) {
            dp_load_tile(j0, n, ms, R, W, LAMBDA, tR, tX, tG);
            if (!own) continue;
            const int jt = min(DP_TJ, n - j0);
            for (int t = 0; t < jt; ++t) {
                const int j = j0 + t;
                if (j == k) continue;
                const float sq = sqrtf(2.0f * (vk + vs[j]));
                const float x = (mk - mus[j]) / sq;                  // x_kj
                float A;
                if (PAIR) {
                    // the upper-triangle pair (lo, hi) = (min, max)(k, j): target, weight, p = 1 - P_lohi
                    const bool lo = k < j;
                    float tsum = 0.0f, s1 = 0.0f, s2 = 0.0f;
#pragma unroll
                    for (int s = 0; s < DP_MS; ++s) {
                        if (s >= ms) break;
                        const float rj = tR[s * DP_TJ + t];
                        const float d = lo ? rk[s] - rj : rj - rk[s];
                        tsum += 0.5f * (1.0f + fminf(fmaxf(d, -1.0f), 1.0f));
                        if (LAMBDA) {
                            const float dg = lo ? gk[s] - tG[s * DP_TJ + t] : tG[s * DP_TJ + t] - gk[s];
                            s1 += dg * (lo ? xk[s] : tX[s * DP_TJ + t]);
                            s2 += dg * (lo ? tX[s * DP_TJ + t] : xk[s]);
                        }
                    }
                    const float tt = tsum * inv_m;
                    float wt = 1.0f;
                    if (LAMBDA) { wt = fabsf(s1 - s2); if (norm) wt = wt / idcg; }
                    const float p = 1.0f - 0.5f * erfcf(lo ? x : -x);
                    if (lo)
                        lsum += ((tt - 1.0f) * fmaxf(log1pf(-p), -100.0f) - tt * fmaxf(logf(p), -100.0f)) * wt;
                    const float c = -(wt * (p - tt) / fmaxf((1.0f - p) * p, 1e-12f));   // dL/dP_lohi
                    A = lo ? c : -c;
                } else {
                    A = ak - as[j];
                    if (MODE == PTRB200_DIVPROB_ANDCG) {
#pragma unroll
                        for (int s = 0; s < DP_MS; ++s) {
                            if (s >= ms) break;
                            A += xk[s] * tR[s * DP_TJ + t] - tX[s * DP_TJ + t] * rk[s];
                        }
                    }
                }
                const float w = expf(-x * x) * inv_sqrt_pi / sq;
                gm -= w * A;
                gv += (w * x / sq) * A;
            }
        }
        if (own) {
            if (PAIR) ls[k] = lsum;
            const float* u = U + (size_t)k * D;
            float* du = out + (sp.base + k) * (size_t)D;
            dp_head_bwd(u, K, limit, gm, gv, du);
        }
    }
    __syncthreads();
    if (tid < 32) {
        float v = 0.0f;
        for (int i = tid; i < n; i += 32) v += ls[i];
        v = warp_sum(v);
        if (tid == 0) loss_q[b] = PAIR ? v : -v;
    }
}

// The head alone, one thread per row: mu[row], var[row] (DivMDNRanker.div_forward's output).
__global__ void divprob_head_kernel(const float* __restrict__ raw, int D, long long rows, int K, float limit,
                                    float* __restrict__ mu, float* __restrict__ var) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    float m, v;
    dp_head(raw + (size_t)r * D, K, limit, m, v);
    mu[r] = m;
    var[r] = v;
}

static inline size_t divprob_smem(int n, int m) { return ((size_t)5 * n + (size_t)3 * m * DP_TJ) * sizeof(float); }

template <int MODE>
static int divprob_launch(const float* raw, int D, const int32_t* offsets, const float* rele, const int64_t* rele_offsets,
                          const int32_t* sub_counts, float* ws, float* out, float* loss_q, int B, int n, int m, int K,
                          float limit, int top_k, int flag, float log2_q, float neg_ln_q, ptrb200_stream_t stream,
                          const char* tag) {
    const size_t smem = divprob_smem(n, m);
    int rc = allow_smem(divprob_kernel<MODE>, smem + 64);
    if (rc) return rc;
    PTRB200_LAUNCH_TAG(tag, divprob_kernel<MODE>, B, DP_THREADS, smem, stream, raw, D, offsets, rele, rele_offsets,
                       sub_counts, ws, out, loss_q, n, m, K, limit, top_k, flag, log2_q, neg_ln_q);
    return check_launch(tag);
}

static int check_head_args(const char* who, int out_dim, int K, float limit) {
    if (K < 1 || out_dim != (K == 1 ? 2 : 3 * K)) {
        set_error("%s: out_dim=%d does not match K=%d (2 for K = 1, 3K otherwise)", who, out_dim, K);
        return PTRB200_ERR_INVALID;
    }
    if (!(limit >= 0.0f)) { set_error("%s: limit_delta=%g must be >= 0 (0: exp variances)", who, limit); return PTRB200_ERR_INVALID; }
    return PTRB200_OK;
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_divprob_fwd_bwd(const float* raw, int out_dim, const int32_t* offsets, const float* rele,
                            const int64_t* rele_offsets, const int32_t* sub_counts, float* workspace, float* grad_raw,
                            float* loss_per_query, int B, int n, int m, int K, float limit_delta, int loss, int top_k,
                            int norm, ptrb200_stream_t stream) {
    int rc = check_list_args(raw, rele, grad_raw, loss_per_query, B, n);
    if (rc) return rc;
    if ((rc = check_rele_args("divprob", rele, rele_offsets, sub_counts, m))) return rc;
    if ((rc = check_head_args("divprob", out_dim, K, limit_delta))) return rc;
    if (loss < PTRB200_DIVPROB_ANDCG || loss > PTRB200_DIVPROB_LAMBDA_PAIRCLS) {
        set_error("divprob: unknown loss %d", loss);
        return PTRB200_ERR_INVALID;
    }
    if ((loss == PTRB200_DIVPROB_ANDCG || loss == PTRB200_DIVPROB_LAMBDA_PAIRCLS) && !workspace) {
        set_error("divprob: this loss needs a workspace of the relevance blocks' size");
        return PTRB200_ERR_INVALID;
    }
    const float beta = 0.5f, lq = log2f(1.0f - beta), nlq = -logf(1.0f - beta);
#define DP_CASE(L, TAG) \
    case L: return divprob_launch<L>(raw, out_dim, offsets, rele, rele_offsets, sub_counts, workspace, grad_raw, \
                                     loss_per_query, B, n, m, K, limit_delta, top_k, norm, lq, nlq, stream, TAG)
    switch (loss) {
        DP_CASE(PTRB200_DIVPROB_ANDCG, "divprob_andcg");
        DP_CASE(PTRB200_DIVPROB_NERRIA, "divprob_nerr_ia");
        DP_CASE(PTRB200_DIVPROB_PAIRCLS, "divprob_paircls");
        DP_CASE(PTRB200_DIVPROB_LAMBDA_PAIRCLS, "divprob_lambda_paircls");
    }
#undef DP_CASE
    return PTRB200_ERR_INVALID;
}

int ptrb200_divprob_sort_key(const float* raw, int out_dim, const int32_t* offsets, float* key, int B, int n, int K,
                             float limit_delta, int sort_id, ptrb200_stream_t stream) {
    int rc = check_list_args(raw, key, key, key, B, n);
    if (rc) return rc;
    if ((rc = check_head_args("divprob_sort_key", out_dim, K, limit_delta))) return rc;
    if (sort_id < PTRB200_DIVPROB_KEY_EXPRELE || sort_id > PTRB200_DIVPROB_KEY_RISKAWARE) {
        set_error("divprob_sort_key: unknown sort id %d", sort_id);
        return PTRB200_ERR_INVALID;
    }
    return divprob_launch<DP_KEY>(raw, out_dim, offsets, nullptr, nullptr, nullptr, nullptr, key, nullptr, B, n, 0, K,
                                  limit_delta, 0, sort_id, 0.0f, 0.0f, stream, "divprob_sort_key");
}

int ptrb200_divprob_head(const float* raw, int out_dim, long long rows, int K, float limit_delta, float* mu, float* var,
                         ptrb200_stream_t stream) {
    if (!raw || !mu || !var || rows <= 0) { set_error("divprob_head: null pointer or rows=%lld", rows); return PTRB200_ERR_INVALID; }
    int rc = check_head_args("divprob_head", out_dim, K, limit_delta);
    if (rc) return rc;
    PTRB200_LAUNCH(divprob_head_kernel, (unsigned)((rows + 255) / 256), 256, 0, stream, raw, out_dim, rows, K, limit_delta,
                   mu, var);
    return check_launch("divprob_head");
}

}  // extern "C"
