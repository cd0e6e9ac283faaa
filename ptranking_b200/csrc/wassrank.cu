// wassrank.cu -- WassRank's Sinkhorn optimal-transport loss, fused: cost, histograms, Sinkhorn iterations, loss and the
// gradient the reference hands to autograd, one CTA per query, everything in the log domain.
//
// Reference replaced (wildltr/ptranking @ f1d366c):
//   WassRank.custom_loss_function, mode 'SinkhornOT'   ptranking/ltr_adhoc/listwise/wassrank/wassRank.py:43-86
//   OldSinkhornOT (forward + backward)                 ptranking/ltr_adhoc/listwise/wassrank/pytorch_wasserstein.py:323-394
//   get_explicit_cost_mat (p1, p2, eg, dg, ddg)        ptranking/ltr_adhoc/listwise/wassrank/wasserstein_cost_mat.py:47-139
//   get_normalized_histograms ('ST', 'BothST')         ptranking/ltr_adhoc/listwise/wassrank/wasserstein_cost_mat.py:142-203
//
// Per query (scores s[n], labels y[n]):  log a = log_softmax(s), log b = log_softmax(y), log_u = log_v = -log n, then
// sh_itr times  log_v_j = log b_j - LSE_i(log_u_i - C_ij/lam),  log_u_i = log a_i - LSE_j(log_v_j - C_ij/lam).
// loss_q = sum_i exp(log_u_i + LSE_{j: C_ij > 0}(log C_ij - C_ij/lam + log_v_j)) / batch_queries.
// The gradient is the reference's dual potential, not the derivative of the loss: g = lam log_u, its row mean subtracted
// twice, divided by batch_queries, then through the softmax: grad_i = a_i (g_i - sum_k a_k g_k).
//
// No [n,n] array exists: C_ij is formed from (label, position) where it is used.  Two schedules, chosen per query:
//  - grouped (eg, dg with at most WASS_MAX_GROUPS distinct labels): off the diagonal C_ij depends only on the labels'
//    groups, so a half-step is one log-sum per group of the current potential and an R-term LSE per document, O(n R);
//  - general (p1, p2, ddg, and eg/dg lists with more distinct labels): an O(n^2) walk per half-step.
// The CTA size is fixed (WASS_THREADS), so a query's summation order does not depend on the launch it is part of: a
// length-bucketed batch and a single launch give bit-identical results.  No atomics.
#include "losses_common.cuh"

#include <limits.h>

namespace ptrb200 {

constexpr int WASS_THREADS = 256;
constexpr int WASS_WARPS = WASS_THREADS / 32;
constexpr int WASS_MAX_GROUPS = 16;

// Log-sum of the members of one label group: exp(m) * s is the sum, exp(m) * x the sum without the member `a` that
// attains the maximum (lowest index among ties).  A document's "sum of the others in my group" is then s - e_self for
// every member but `a` (e_self <= s/2: no cancellation) and x for `a` -- exact where s - e_self would cancel.
struct GStat { float m, s, x; int a; };

static __device__ __forceinline__ GStat gstat_empty() { GStat g; g.m = -INFINITY; g.s = 0.0f; g.x = 0.0f; g.a = INT_MAX; return g; }

static __device__ __forceinline__ GStat gstat_merge(const GStat& p, const GStat& q) {
    const bool p_hi = (p.m > q.m) || (p.m == q.m && p.a < q.a);
    GStat hi = p_hi ? p : q;
    const GStat lo = p_hi ? q : p;
    if (lo.a == INT_MAX) return hi;                  // empty side
    const float w = expf(lo.m - hi.m);
    hi.s = fmaf(lo.s, w, hi.s);
    hi.x = fmaf(lo.s, w, hi.x);                      // the excluded member is hi's; all of lo counts
    return hi;
}

static __device__ __forceinline__ GStat gstat_shfl_down(const GStat& g, int o) {
    GStat r;
    r.m = __shfl_down_sync(0xffffffffu, g.m, o);
    r.s = __shfl_down_sync(0xffffffffu, g.s, o);
    r.x = __shfl_down_sync(0xffffffffu, g.x, o);
    r.a = __shfl_down_sync(0xffffffffu, g.a, o);
    return r;
}

// online log-sum-exp: (m, s) with sum = exp(m) s; v may be -inf, m starts at -inf (never both -inf)
static __device__ __forceinline__ void lse_push(float& m, float& s, float v) {
    const float e = expf(-fabsf(v - m));
    s = v > m ? fmaf(s, e, 1.0f) : s + e;
    m = fmaxf(m, v);
}

// C_ij (i != j) of the general schedule.  f0: per-document gain term (eg: gain with the non-relevance gap, dg/ddg:
// 2^y - 1); f1: ddg's discount 1 / log2(i + 2).  Positions of p1/p2 are 1..n; their difference is exact in fp32.
template <int COST>
static __device__ __forceinline__ float wass_cost(int i, int j, const float* f0, const float* f1, float var_penalty) {
    if (COST == PTRB200_WASS_COST_P1) return fabsf((float)(i - j));
    if (COST == PTRB200_WASS_COST_P2) { const float d = fabsf((float)(i - j)); return d * d; }
    if (COST == PTRB200_WASS_COST_EG) { const float d = fabsf(f0[i] - f0[j]); return d < 1.0f ? var_penalty : d; }
    if (COST == PTRB200_WASS_COST_DG) return fabsf(f0[i] - f0[j]);
    return fabsf(f0[i] - f0[j]) * fabsf(f1[i] - f1[j]);
}

// dst_j = logm_j - LSE_i(src_i - C_ij / lam) for every document j: one thread per j walks i in index order
template <int COST>
static __device__ void wass_half_general(const float* src, const float* logm, float* dst, int n,
                                         const float* f0, const float* f1, float inv_lam, float var_penalty) {
    for (int j = threadIdx.x; j < n; j += WASS_THREADS) {
        float m = -INFINITY, s = 0.0f;
        for (int i = 0; i < n; ++i) {
            const float c = i == j ? 0.0f : wass_cost<COST>(i, j, f0, f1, var_penalty);
            lse_push(m, s, src[i] - c * inv_lam);
        }
        dst[j] = logm[j] - (m + logf(s));
    }
}

// sum_i exp(log_u_i + LSE_{j: C_ij > 0}(log C_ij - C_ij/lam + log_v_j)) over this thread's rows i
template <int COST>
static __device__ float wass_loss_general(const float* lu, const float* lv, int n, const float* f0, const float* f1,
                                          float inv_lam, float var_penalty) {
    float acc = 0.0f;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
        float m = -INFINITY, s = 0.0f;
        for (int j = 0; j < n; ++j) {
            if (j == i) continue;
            const float c = wass_cost<COST>(i, j, f0, f1, var_penalty);
            if (c > 0.0f) lse_push(m, s, logf(c) - c * inv_lam + lv[j]);
        }
        acc += expf(lu[i] + (m + logf(s)));            // no positive cost in the row: exp(-inf) = 0
    }
    return acc;
}

template <int COST>
static __device__ float wass_run_general(float* la, float* lb, float* lu, float* lv, int n, const float* f0, const float* f1,
                                         float inv_lam, float var_penalty, int sh_itr) {
    for (int it = 0; it < sh_itr; ++it) {
        wass_half_general<COST>(lu, lb, lv, n, f0, f1, inv_lam, var_penalty);
        __syncthreads();
        wass_half_general<COST>(lv, la, lu, n, f0, f1, inv_lam, var_penalty);
        __syncthreads();
    }
    return wass_loss_general<COST>(lu, lv, n, f0, f1, inv_lam, var_penalty);
}

// Shared state of the grouped schedule.  ctab[l][r] = C(l, r) / lam between documents of groups l and r (for l == r:
// two different documents of the same group), lctab = log C (-inf where C = 0).
struct WassGroups {
    float lab[WASS_MAX_GROUPS];
    float ctab[WASS_MAX_GROUPS][WASS_MAX_GROUPS];
    float lctab[WASS_MAX_GROUPS][WASS_MAX_GROUPS];
    float kself[WASS_MAX_GROUPS];                    // exp(-ctab[l][l])
    float lsum[WASS_MAX_GROUPS];                     // log of the group's sum of exp(potential)
    GStat st[WASS_MAX_GROUPS];
    GStat part[WASS_MAX_GROUPS][WASS_WARPS];
};

// per-group statistics of the potential x -> g.st / g.lsum (fixed order: thread stride, warp tree, warps in order)
static __device__ void wass_group_stats(const float* x, const int* gid, int n, int R, WassGroups& g) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = 0; r < R; ++r) {
        GStat acc = gstat_empty();
        for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
            if (gid[i] != r) continue;
            GStat one; one.m = x[i]; one.s = 1.0f; one.x = 0.0f; one.a = i;
            acc = gstat_merge(acc, one);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc = gstat_merge(acc, gstat_shfl_down(acc, o));
        if (lane == 0) g.part[r][warp] = acc;
    }
    __syncthreads();
    if (threadIdx.x < R) {
        const int r = threadIdx.x;
        GStat acc = g.part[r][0];
        for (int w = 1; w < WASS_WARPS; ++w) acc = gstat_merge(acc, g.part[r][w]);
        g.st[r] = acc;
        g.lsum[r] = acc.m + logf(acc.s);
    }
    __syncthreads();
}

// exp(-m) * (sum of exp(x) over the other members of document i's group); e = exp(x_i - m)
static __device__ __forceinline__ float wass_others(const GStat& st, float e, int i) {
    return i == st.a ? st.x : fmaxf(st.s - e, 0.0f);
}

// dst_j = logm_j - LSE_i(src_i - C_ij/lam), grouped: own group K_ll (V_l - v_j) + v_j, other groups K_lr V_r
static __device__ void wass_half_grouped(const float* src, const float* logm, float* dst, const int* gid, int n, int R, WassGroups& g) {
    wass_group_stats(src, gid, n, R, g);
    for (int j = threadIdx.x; j < n; j += WASS_THREADS) {
        const int l = gid[j];
        const GStat st = g.st[l];
        const float e = expf(src[j] - st.m);
        const float own = st.m + logf(fmaf(g.kself[l], wass_others(st, e, j), e));
        float mx = own;
        for (int r = 0; r < R; ++r) if (r != l) mx = fmaxf(mx, g.lsum[r] - g.ctab[l][r]);
        float sum = 0.0f;
        for (int r = 0; r < R; ++r) sum += expf((r == l ? own : g.lsum[r] - g.ctab[l][r]) - mx);
        dst[j] = logm[j] - (mx + logf(sum));
    }
    __syncthreads();
}

static __device__ float wass_run_grouped(float* la, float* lb, float* lu, float* lv, const int* gid, int n, int R, int sh_itr, WassGroups& g) {
    for (int it = 0; it < sh_itr; ++it) {
        wass_half_grouped(lu, lb, lv, gid, n, R, g);
        wass_half_grouped(lv, la, lu, gid, n, R, g);
    }
    wass_group_stats(lv, gid, n, R, g);
    float acc = 0.0f;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
        const int l = gid[i];
        const GStat st = g.st[l];
        // log of this document's mass on its own group (-inf for a group of one)
        const float own = st.m + logf(wass_others(st, expf(lv[i] - st.m), i));
        float mx = -INFINITY;
        for (int r = 0; r < R; ++r) mx = fmaxf(mx, g.lctab[l][r] - g.ctab[l][r] + (r == l ? own : g.lsum[r]));
        float L = -INFINITY;                             // no positive cost in the row
        if (mx > -INFINITY) {
            float sum = 0.0f;
            for (int r = 0; r < R; ++r) sum += expf(g.lctab[l][r] - g.ctab[l][r] + (r == l ? own : g.lsum[r]) - mx);
            L = mx + logf(sum);
        }
        acc += expf(lu[i] + L);
    }
    return acc;
}

// C between two different documents with labels ya, yb under the label-defined costs (wasserstein_cost_mat.py:63-111)
static __device__ float wass_label_cost(int cost, float ya, float yb, float var_penalty, float non_rele_gap, float gain_base) {
    if (cost == PTRB200_WASS_COST_DG) return fabsf(gain_of(ya) - gain_of(yb));
    float ga = powf(gain_base, ya) - 1.0f, gb = powf(gain_base, yb) - 1.0f;
    ga = ga < 1.0f ? -non_rele_gap : ga;
    gb = gb < 1.0f ? -non_rele_gap : gb;
    const float d = fabsf(ga - gb);
    return d < 1.0f ? var_penalty : d;
}

struct WassArgs {
    int cost, sh_itr;
    float lam, inv_lam, non_rele_gap, var_penalty, gain_base, inv_batch;
};

__global__ void __launch_bounds__(WASS_THREADS) wassrank_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                                                const int32_t* __restrict__ offsets, float* __restrict__ grad,
                                                                float* __restrict__ loss_q, int n_uniform, WassArgs p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* la = reinterpret_cast<float*>(smem_raw);      // log a = log_softmax(s)
    float* lb = la + n_uniform;                          // log b = log_softmax(y); later the gradient's g
    float* lu = lb + n_uniform;
    float* lv = lu + n_uniform;
    float* f0 = lv + n_uniform;                          // labels, then the general schedule's gain term
    float* f1 = f0 + n_uniform;                          // ddg discount
    int* gid = reinterpret_cast<int*>(f1 + n_uniform);   // group of each document (grouped schedule)
    __shared__ float red[33];
    __shared__ WassGroups g;
    __shared__ int s_groups;

    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, n_uniform);
    const int n = sp.n;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }

    // histograms: log-softmax of scores and of labels (wasserstein_cost_mat.py:166, :201)
    float ms = -INFINITY, my = -INFINITY;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
        const float s = scores[sp.base + i], y = labels[sp.base + i];
        la[i] = s; f0[i] = y;
        ms = fmaxf(ms, s); my = fmaxf(my, y);
    }
    ms = block_max(ms, red);
    my = block_max(my, red);
    float es = 0.0f, ey = 0.0f;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) { es += expf(la[i] - ms); ey += expf(f0[i] - my); }
    const float lse_s = ms + logf(block_sum(es, red));
    const float lse_y = my + logf(block_sum(ey, red));
    const float init = (float)(-log((double)n));        // pytorch_wasserstein.py:340-341: fill_(-np.log(n))
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
        la[i] -= lse_s;
        lb[i] = f0[i] - lse_y;
        lu[i] = init; lv[i] = init;
    }

    // label groups (ascending distinct values) for eg / dg; -1 = more than WASS_MAX_GROUPS distinct labels
    int R = -1;
    if (p.cost == PTRB200_WASS_COST_EG || p.cost == PTRB200_WASS_COST_DG) {
        float prev = -INFINITY;
        R = 0;
        for (int k = 0; k <= WASS_MAX_GROUPS; ++k) {
            float mn = INFINITY;
            for (int i = threadIdx.x; i < n; i += WASS_THREADS) { const float y = f0[i]; if (y > prev) mn = fminf(mn, y); }
            mn = -block_max(-mn, red);
            if (mn == INFINITY) break;
            if (k == WASS_MAX_GROUPS) { R = -1; break; }
            if (threadIdx.x == 0) g.lab[k] = mn;
            prev = mn;
            R = k + 1;
        }
        if (threadIdx.x == 0) s_groups = R;
        __syncthreads();
        R = s_groups;
    }

    float part;
    if (R > 0) {
        for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
            const float y = f0[i];
            int k = 0;
            while (k + 1 < R && g.lab[k] != y) ++k;
            gid[i] = k;
        }
        for (int e = threadIdx.x; e < R * R; e += WASS_THREADS) {
            const int l = e / R, r = e % R;
            const float c = wass_label_cost(p.cost, g.lab[l], g.lab[r], p.var_penalty, p.non_rele_gap, p.gain_base);
            g.ctab[l][r] = c * p.inv_lam;
            g.lctab[l][r] = c > 0.0f ? logf(c) : -INFINITY;
            if (l == r) g.kself[l] = expf(-(c * p.inv_lam));
        }
        __syncthreads();
        part = wass_run_grouped(la, lb, lu, lv, gid, n, R, p.sh_itr, g);
    } else {
        for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
            const float y = f0[i];
            if (p.cost == PTRB200_WASS_COST_EG) {
                const float gi = powf(p.gain_base, y) - 1.0f;
                f0[i] = gi < 1.0f ? -p.non_rele_gap : gi;
            } else {
                f0[i] = gain_of(y);
            }
            f1[i] = 1.0f / log2_rank(i);                 // wasserstein_cost_mat.py:73-74, 0-based positions
        }
        __syncthreads();
        switch (p.cost) {
            case PTRB200_WASS_COST_P1: part = wass_run_general<PTRB200_WASS_COST_P1>(la, lb, lu, lv, n, f0, f1, p.inv_lam, p.var_penalty, p.sh_itr); break;
            case PTRB200_WASS_COST_P2: part = wass_run_general<PTRB200_WASS_COST_P2>(la, lb, lu, lv, n, f0, f1, p.inv_lam, p.var_penalty, p.sh_itr); break;
            case PTRB200_WASS_COST_EG: part = wass_run_general<PTRB200_WASS_COST_EG>(la, lb, lu, lv, n, f0, f1, p.inv_lam, p.var_penalty, p.sh_itr); break;
            case PTRB200_WASS_COST_DG: part = wass_run_general<PTRB200_WASS_COST_DG>(la, lb, lu, lv, n, f0, f1, p.inv_lam, p.var_penalty, p.sh_itr); break;
            default: part = wass_run_general<PTRB200_WASS_COST_DDG>(la, lb, lu, lv, n, f0, f1, p.inv_lam, p.var_penalty, p.sh_itr); break;
        }
    }
    const float loss = block_sum(part, red);            // also orders the last half-step before the reads below

    // gradient (pytorch_wasserstein.py:371-380): g = lam log_u, row mean subtracted twice, / batch size; then softmax's
    // backward: grad_i = a_i (g_i - sum_k a_k g_k)
    float* gv = lb;
    const float inv_n = 1.0f / (float)n;
    float t = 0.0f;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) { gv[i] = lu[i] * p.lam; t += gv[i]; }
    const float mean1 = block_sum(t, red) * inv_n;
    t = 0.0f;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) { gv[i] -= mean1; t += gv[i]; }
    const float mean2 = block_sum(t, red) * inv_n;
    t = 0.0f;
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) {
        gv[i] = (gv[i] - mean2) * p.inv_batch;
        t = fmaf(expf(la[i]), gv[i], t);
    }
    const float ag = block_sum(t, red);
    for (int i = threadIdx.x; i < n; i += WASS_THREADS) grad[sp.base + i] = expf(la[i]) * (gv[i] - ag);
    if (threadIdx.x == 0) loss_q[b] = loss * p.inv_batch;
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_wassrank_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad,
                             float* loss_per_query, int B, int n, int batch_queries, int cost_type, float lam,
                             int sh_itr, float non_rele_gap, float var_penalty, float gain_base, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    if (batch_queries < B) { set_error("wassrank: batch_queries=%d is below the launch's B=%d", batch_queries, B); return PTRB200_ERR_INVALID; }
    if (cost_type < PTRB200_WASS_COST_P1 || cost_type > PTRB200_WASS_COST_DDG) {
        set_error("wassrank: unknown cost type %d", cost_type);
        return PTRB200_ERR_INVALID;
    }
    if (!(lam > 0.0f) || !isfinite(lam)) { set_error("wassrank: lam must be positive and finite"); return PTRB200_ERR_INVALID; }
    if (sh_itr < 0) { set_error("wassrank: sh_itr must be >= 0"); return PTRB200_ERR_INVALID; }
    WassArgs p;
    p.cost = cost_type; p.sh_itr = sh_itr;
    p.lam = lam; p.inv_lam = 1.0f / lam;
    p.non_rele_gap = non_rele_gap; p.var_penalty = var_penalty; p.gain_base = gain_base;
    p.inv_batch = 1.0f / (float)batch_queries;
    const size_t smem = (size_t)n * 4 * 7;
    // the static WassGroups block (~5 KB) counts against the same 48 KB default, so opt in early
    if (smem > 32 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(wassrank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu): %s", smem, cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
    }
    PTRB200_LAUNCH(wassrank_kernel, B, WASS_THREADS, smem, stream, scores, labels, offsets, grad, loss_per_query, n, p);
    return check_launch("wassrank");
}

}  // extern "C"
