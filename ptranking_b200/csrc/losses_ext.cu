// losses_ext.cu -- the sibling ranking losses of SURVEY 8f-4 on the same one-CTA-per-query skeleton, plus the Sinkhorn
// half-step (the reference's only CUDA kernel).
//
// Reference functions replaced (wildltr/ptranking @ f1d366c):
//   RankMSE     ptranking/ltr_adhoc/pointwise/rank_mse.py:13-22
//   RankCosine  ptranking/ltr_adhoc/listwise/rank_cosine.py:33 (nn.CosineSimilarity(dim=1), eps 1e-8)
//   STListNet   ptranking/ltr_adhoc/listwise/st_listnet.py:41-49
//   SoftRank    ptranking/ltr_adhoc/listwise/softrank.py:46-72
//   MDPRank     ptranking/ltr_adhoc/listwise/mdprank.py:24-79 (+ sample_ranking_PL / _gumbel_softmax, util/sampling_utils.py:31-79)
//   sinkstep    ptranking/ltr_adhoc/listwise/wassrank/pytorch_wasserstein.py:132-224 (CUDA string) / :277-291 (CPU form)
#include "losses_common.cuh"

namespace ptrb200 {

// ---------------------------------------------------------------------------
// RankMSE: mean over the batch of the per-query sum of squared errors.  loss_q[b] = sum_i (s-y)^2 / B so that the sum
// over queries is the reference's torch.mean(torch.sum(., dim=1)); grad = 2 (s - y) / B.
// ---------------------------------------------------------------------------
__global__ void rankmse_kernel(const float* __restrict__ scores, const float* __restrict__ labels, const int32_t* __restrict__ offsets,
                               float* __restrict__ grad, float* __restrict__ loss_q, int n_uniform, float inv_B) {
    __shared__ float red[33];
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, n_uniform);
    float acc = 0.0f;
    for (int i = threadIdx.x; i < sp.n; i += blockDim.x) {
        const float d = scores[sp.base + i] - labels[sp.base + i];
        acc = fmaf(d, d, acc);
        grad[sp.base + i] = (2.0f * d) * inv_B;
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) loss_q[b] = acc * inv_B;
}

// ---------------------------------------------------------------------------
// RankCosine: (1 - cos(s, y)) / 0.5 per query with ATen's cosine_similarity: cos = sum_i (s_i / max(|s|, eps)) (y_i / max(|y|, eps)).
// d cos / d s_i = y_i / (S Y) - [|s| > eps] (s . y) s_i / (S^2 |s| Y),  S = max(|s|, eps), Y = max(|y|, eps).
// ---------------------------------------------------------------------------
__global__ void rankcosine_kernel(const float* __restrict__ scores, const float* __restrict__ labels, const int32_t* __restrict__ offsets,
                                  float* __restrict__ grad, float* __restrict__ loss_q, int n_uniform, float eps) {
    __shared__ float red[33];
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, n_uniform);
    float ss = 0.0f, yy = 0.0f, sy = 0.0f;
    for (int i = threadIdx.x; i < sp.n; i += blockDim.x) {
        const float s = scores[sp.base + i], y = labels[sp.base + i];
        ss = fmaf(s, s, ss); yy = fmaf(y, y, yy); sy = fmaf(s, y, sy);
    }
    ss = block_sum(ss, red); yy = block_sum(yy, red); sy = block_sum(sy, red);
    const float ns = sqrtf(ss), ny = sqrtf(yy);
    const float S = fmaxf(ns, eps), Y = fmaxf(ny, eps);
    const float cosv = sy / (S * Y);
    const float a = 1.0f / (S * Y);
    const float c = ns > eps ? sy / (S * S * ns * Y) : 0.0f;
    for (int i = threadIdx.x; i < sp.n; i += blockDim.x) {
        const float s = scores[sp.base + i], y = labels[sp.base + i];
        grad[sp.base + i] = -2.0f * (y * a - c * s);
    }
    if (threadIdx.x == 0) loss_q[b] = sp.n > 0 ? (1.0f - cosv) * 2.0f : 0.0f;
}

// ---------------------------------------------------------------------------
// STListNet: ListNet on Gumbel-perturbed scores z = (s + g) / T, g = -log(-log(u + 1e-20) + 1e-20), u ~ U[0,1).
// `unif` (optional) injects the uniforms (parity tests replay the reference's torch.rand draw); otherwise u comes from
// Philox4x32-10 keyed by (seed, offset, flat doc index) as 24-bit fractions, the granularity of torch.rand(float32).
// grad = (softmax(z) - softmax(y)) / T.
// ---------------------------------------------------------------------------
__global__ void stlistnet_kernel(const float* __restrict__ scores, const float* __restrict__ labels, const int32_t* __restrict__ offsets,
                                 const float* __restrict__ unif, float* __restrict__ grad, float* __restrict__ loss_q,
                                 int n_uniform, float inv_T, uint64_t seed, uint64_t offset) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* zs = reinterpret_cast<float*>(smem_raw);
    float* ys = zs + n_uniform;
    float* red = ys + n_uniform;
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, n_uniform);
    const int n = sp.n;
    float mz = -INFINITY, my = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float u;
        if (unif) u = unif[sp.base + i];
        else u = (float)(dropout_bits(seed, offset, (uint64_t)(sp.base + i)) >> 8) * (1.0f / 16777216.0f);
        const float g = -logf(-logf(u + 1e-20f) + 1e-20f);
        const float z = (scores[sp.base + i] + g) * inv_T;
        const float y = labels[sp.base + i];
        zs[i] = z; ys[i] = y;
        mz = fmaxf(mz, z); my = fmaxf(my, y);
    }
    mz = block_max(mz, red);
    my = block_max(my, red);
    float sz = 0.0f, sy = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { sz += expf(zs[i] - mz); sy += expf(ys[i] - my); }
    sz = block_sum(sz, red);
    sy = block_sum(sy, red);
    const float log_sz = logf(sz);
    float loss = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float py = expf(ys[i] - my) / sy;
        const float lsm = (zs[i] - mz) - log_sz;
        loss -= py * lsm;
        grad[sp.base + i] = (expf(lsm) - py) * inv_T;
    }
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = n > 0 ? loss : 0.0f;
}

// ---------------------------------------------------------------------------
// SoftRank (metric nDCG): expected rank r_i = 1 + sum_{j != i} 0.5 erfc((s_i - s_j) / den), den = sqrt(2 * 2 delta^2);
// loss_q = - sum_{i < k} G(y_i) / (log2(r_i + 1) iDCG), iDCG over the labels as given (presort contract, softrank.py:40).
// c_i = d loss / d r_i = [i < k] G_i / (iDCG log2(r_i+1)^2 (r_i+1) ln 2); with e_ij = -exp(-x_ij^2) / (sqrt(pi) den)
// (= d r_i / d s_i contribution of j, symmetric in i,j):  grad_m = sum_{j != m} e_mj (c_m - c_j).
// ---------------------------------------------------------------------------
__global__ void softrank_kernel(const float* __restrict__ scores, const float* __restrict__ labels, const int32_t* __restrict__ offsets,
                                float* __restrict__ grad, float* __restrict__ loss_q, int n_uniform, float inv_den, int top_k) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* ss = reinterpret_cast<float*>(smem_raw);
    float* cc = ss + n_uniform;
    float* red = cc + n_uniform;
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, n_uniform);
    const int n = sp.n;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const float* y = labels + sp.base;
    float part = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { ss[i] = scores[sp.base + i]; part += gain_of(y[i]) / log2_rank(i); }
    const float idcg = block_sum(part, red);        // ends with a barrier: ss is visible
    const int K = (top_k > 0 && top_k < n) ? top_k : n;
    float dcg = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float si = ss[i];
        float r = 0.0f;
        for (int j = 0; j < n; ++j) r += (j != i) ? 0.5f * erfcf((si - ss[j]) * inv_den) : 0.0f;
        r += 1.0f;
        float c = 0.0f;
        if (i < K) {
            const float G = gain_of(y[i]);
            const float lg = log2f(r + 1.0f);
            dcg += (G / lg) / idcg;                  // (dist * gain) / idcg, the reference's association
            c = G / (idcg * lg * lg * (r + 1.0f) * 0.6931471805599453f);
        }
        cc[i] = c;
    }
    __syncthreads();
    const float ecoef = -0.5641895835477563f * inv_den;      // -1 / (sqrt(pi) den)
    for (int m = threadIdx.x; m < n; m += blockDim.x) {
        const float sm = ss[m], cm = cc[m];
        float acc = 0.0f;
        for (int j = 0; j < n; ++j) {
            const float x = (sm - ss[j]) * inv_den;
            acc = fmaf(expf(-x * x), cm - cc[j], acc);        // j == m contributes exactly 0
        }
        grad[sp.base + m] = ecoef * acc;
    }
    dcg = block_sum(dcg, red);
    if (threadIdx.x == 0) loss_q[b] = -dcg;
}

// ---------------------------------------------------------------------------
// MDPRank: REINFORCE on one sampled Plackett-Luce ranking sigma per query (mdprank.py:24-79).
// Sampling is Gumbel-top-k: sort keys s/T + g (PL) or (s + g)/T (STPL), g from the uniforms as in stlistnet_kernel;
// an injected PL ordering `perm` replaces the sort.  Action values a_t = s_sigma(t) (PL) or the perturbed key (STPL).
// Returns G_t = gamma^{t+1} sum_{t<=t'<k} (2^y_sigma(t') - 1) / log2(t'+2), C_t = sum_{j>=t} exp(a_j) over the whole
// list; loss = sum_{t<k} (log C_t - a_t) G_t, d loss / d a_j = sum_{t<=min(j,k-1)} G_t exp(a_j - log C_t) - [j<k] G_j,
// scattered to s_sigma(j) (times 1/T under STPL, where a depends on s through the division).
// Both sums over t are scans of (shift, sum) pairs, so nothing overflows or underflows where the action values spread
// over more than fp32's exponent range (STPL at small T): log C_t is exact to rounding at every position, and for STPL,
// whose a_t descend, log C_t - a_t is the log of a sum of terms <= 1 with no cancellation.
// ---------------------------------------------------------------------------
// (m, s) <- (m, s) + (m2, s2) for the value s e^m; m = -inf with s = 0 is the empty sum.
static __device__ __forceinline__ void lse_add(float& m, float& s, float m2, float s2) {
    if (m2 > m) { s = s * expf(m - m2) + s2; m = m2; }
    else if (m2 > -INFINITY) s += s2 * expf(m2 - m);
}

// Inclusive scan of pairs (mx[i], sm[i]) under lse_add, forward or reverse; the schedule of block_scan_inclusive.
template <bool REVERSE>
static __device__ void block_scan_lse(float* mx, float* sm, int n, float* red /* >= 128 floats */) {
    const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = (T + 31) >> 5;
    const int C = (n + T - 1) / T;
    const int c0 = min(tid * C, n), c1 = min(c0 + C, n);
    float rm = -INFINITY, rs = 0.0f;
    for (int i = c0; i < c1; ++i) {
        const int p = REVERSE ? n - 1 - i : i;
        lse_add(rm, rs, mx[p], sm[p]);
        mx[p] = rm; sm[p] = rs;
    }
    float im = rm, is = rs;                              // inclusive over the lanes of the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float tm = __shfl_up_sync(0xffffffffu, im, o), ts = __shfl_up_sync(0xffffffffu, is, o);
        if (lane >= o) lse_add(im, is, tm, ts);
    }
    float em = __shfl_up_sync(0xffffffffu, im, 1), es = __shfl_up_sync(0xffffffffu, is, 1);
    if (lane == 0) { em = -INFINITY; es = 0.0f; }
    __syncthreads();
    if (lane == 31) { red[warp] = im; red[32 + warp] = is; }
    __syncthreads();
    if (warp == 0) {
        float wm = lane < nw ? red[lane] : -INFINITY, ws = lane < nw ? red[32 + lane] : 0.0f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float tm = __shfl_up_sync(0xffffffffu, wm, o), ts = __shfl_up_sync(0xffffffffu, ws, o);
            if (lane >= o) lse_add(wm, ws, tm, ts);
        }
        float xm = __shfl_up_sync(0xffffffffu, wm, 1), xs = __shfl_up_sync(0xffffffffu, ws, 1);
        if (lane == 0) { xm = -INFINITY; xs = 0.0f; }
        red[64 + lane] = xm; red[96 + lane] = xs;       // exclusive over warps
    }
    __syncthreads();
    lse_add(em, es, red[64 + warp], red[96 + warp]);
    if (em > -INFINITY) {
        for (int i = c0; i < c1; ++i) {
            const int p = REVERSE ? n - 1 - i : i;
            float m = mx[p], s = sm[p];
            lse_add(m, s, em, es);
            mx[p] = m; sm[p] = s;
        }
    }
    __syncthreads();
}

__global__ void mdprank_kernel(const float* __restrict__ scores, const float* __restrict__ labels, const int32_t* __restrict__ offsets,
                               const int32_t* __restrict__ perm, const float* __restrict__ unif, int32_t* __restrict__ sample_out,
                               float* __restrict__ grad, float* __restrict__ loss_q, int nmax, int npow2max, int top_k,
                               float gamma, float temperature, int stpl, uint64_t seed, uint64_t offset) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* v = reinterpret_cast<float*>(keys + npow2max);     // by document: the value a takes when the document is drawn
    int* pid = reinterpret_cast<int*>(v + nmax);              // by position: sigma
    float* lm = reinterpret_cast<float*>(pid + nmax);         // by position: (shift, sum) pairs of C_t, then of
    float* ls = lm + nmax;                                    //   sum_{t'<=t} G_t' / C_t'
    float* G = ls + nmax;                                     // rewards, then returns (first k positions)
    float* red = G + nmax;
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const int k = (top_k > 0 && top_k < n) ? top_k : n;
    if (perm) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            pid[i] = clampi(perm[sp.base + i], 0, n - 1);      // positions within the query's own list
            v[i] = scores[sp.base + i];
        }
    } else {
        for (int i = threadIdx.x; i < npow2; i += blockDim.x) {
            u64 key = 0ull;
            if (i < n) {
                float u;
                if (unif) u = unif[sp.base + i];
                else u = (float)(dropout_bits(seed, offset, (uint64_t)(sp.base + i)) >> 8) * (1.0f / 16777216.0f);
                const float g = -logf(-logf(u + 1e-20f) + 1e-20f);
                const float s = scores[sp.base + i];
                const float z = stpl ? __fdiv_rn(s + g, temperature) : __fdiv_rn(s, temperature) + g;
                v[i] = stpl ? z : s;
                key = desc_key(z, i);
            }
            keys[i] = key;
        }
        block_sort_desc(keys, npow2);
        for (int t = threadIdx.x; t < n; t += blockDim.x) pid[t] = key_index(keys[t]);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
        const int id = pid[t];
        lm[t] = v[id]; ls[t] = 1.0f;
        if (t < k) G[t] = gain_of(labels[sp.base + id]) / log2_rank(t);
        if (sample_out) sample_out[sp.base + t] = id;
    }
    __syncthreads();
    block_scan_lse<true>(lm, ls, n, red);                // C_t = ls e^lm
    block_scan_inclusive<true>(G, k, red);               // returns within the top-k window
    float loss = 0.0f;
    for (int t = threadIdx.x; t < k; t += blockDim.x) {
        float Gt = G[t];
        if (gamma != 1.0f) { Gt *= powf(gamma, (float)(t + 1)); G[t] = Gt; }   // mdprank.py:59-61, applied after the sum
        const float lc = lm[t] + logf(ls[t]);
        loss += ((lm[t] - v[pid[t]]) + logf(ls[t])) * Gt;
        lm[t] = Gt != 0.0f ? logf(fabsf(Gt)) - lc : -INFINITY;                    // G_t / C_t = ls e^lm
        ls[t] = Gt > 0.0f ? 1.0f : (Gt < 0.0f ? -1.0f : 0.0f);
    }
    __syncthreads();
    block_scan_lse<false>(lm, ls, k, red);               // Q_t = sum_{t'<=t} G_t' / C_t'
    const float qm = lm[k - 1], qs = ls[k - 1];
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const float a = v[pid[j]];
        float gj = j < k ? ls[j] * expf(a + lm[j]) - G[j] : qs * expf(a + qm);
        if (stpl) gj = __fdiv_rn(gj, temperature);
        grad[sp.base + pid[j]] = gj;
    }
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// ---------------------------------------------------------------------------
// Sinkhorn half-step:  log_v[b][j] = log_nu[b][j] - logsumexp_i( -dist[i][j] / lambda + log_u[b][i] ).
// One CTA per (tile of 32 columns j, b): lane = column (coalesced reads of dist rows), the 8 warps split the reduction
// rows i, each lane keeps an online (max, sum-exp) pair, the eight partials of a column are merged through shared
// memory.  Infinite entries follow the reference's CPU form (the one that runs): plain IEEE arithmetic.
// ---------------------------------------------------------------------------
constexpr int SINK_WARPS = 8;
__global__ void sinkstep_kernel(const float* __restrict__ dist, const float* __restrict__ log_nu, const float* __restrict__ log_u,
                                float* __restrict__ log_v, int d1, int d2, float lambda) {
    __shared__ float smax[SINK_WARPS][33], ssum[SINK_WARPS][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * 32 + lane, b = blockIdx.y;
    float mx = -INFINITY, se = 0.0f;
    if (j < d2) {
        for (int i = warp; i < d1; i += SINK_WARPS) {
            const float v = __fdiv_rn(-dist[(size_t)i * d2 + j], lambda) + log_u[(size_t)b * d1 + i];   // -dist/lambda + log_u, the reference's order
            if (v > mx) { se = se * expf(mx - v) + 1.0f; mx = v; }      // exp(-inf) = 0 on the first finite value
            else if (v > -INFINITY) se += expf(v - mx);
        }
    }
    smax[warp][lane] = mx; ssum[warp][lane] = se;
    __syncthreads();
    if (warp == 0 && j < d2) {
        float M = smax[0][lane];
#pragma unroll
        for (int w = 1; w < SINK_WARPS; ++w) M = fmaxf(M, smax[w][lane]);
        float S = 0.0f;
#pragma unroll
        for (int w = 0; w < SINK_WARPS; ++w) S += smax[w][lane] > -INFINITY ? ssum[w][lane] * expf(smax[w][lane] - M) : 0.0f;
        // pytorch_wasserstein.py:289 (the path that runs): log_nu - logsumexp(...), IEEE arithmetic on the infinities --
        // an all -inf column gives +inf (NaN when log_nu is -inf too); the never-compiled CUDA string would give -inf
        const float lse = M > -INFINITY ? logf(S) + M : -INFINITY;
        log_v[(size_t)b * d2 + j] = log_nu[(size_t)b * d2 + j] - lse;
    }
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_rankmse_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                            int B, int n, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    PTRB200_LAUNCH(rankmse_kernel, B, block_threads(n), 0, stream, scores, labels, offsets, grad, loss_per_query, n, 1.0f / (float)B);
    return check_launch("rankmse");
}

int ptrb200_rankcosine_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                               int B, int n, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    PTRB200_LAUNCH(rankcosine_kernel, B, block_threads(n), 0, stream, scores, labels, offsets, grad, loss_per_query, n, 1e-8f);
    return check_launch("rankcosine");
}

int ptrb200_stlistnet_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, const float* unif,
                              float* grad, float* loss_per_query, int B, int n, float temperature,
                              uint64_t seed, uint64_t offset, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    if (!(temperature > 0.0f)) { set_error("stlistnet: temperature must be positive"); return PTRB200_ERR_INVALID; }
    const size_t smem = (size_t)n * 4 * 2 + 33 * 4;
    if ((rc = allow_smem(stlistnet_kernel, smem))) return rc;
    PTRB200_LAUNCH(stlistnet_kernel, B, block_threads(n), smem, stream, scores, labels, offsets, unif, grad, loss_per_query,
                   n, 1.0f / temperature, seed, offset);
    return check_launch("stlistnet");
}

int ptrb200_softrank_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                             int B, int n, float delta, int top_k, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    if (!(delta > 0.0f)) { set_error("softrank: delta must be positive"); return PTRB200_ERR_INVALID; }
    // softrank.py:50-52: pairsub_vars = 2 delta^2 (fp32 tensor arithmetic), denominator sqrt(2 * pairsub_vars)
    const float var2 = 2.0f * (delta * delta);
    const float den = sqrtf(2.0f * var2);
    const size_t smem = (size_t)n * 4 * 2 + 33 * 4;
    if ((rc = allow_smem(softrank_kernel, smem))) return rc;
    PTRB200_LAUNCH(softrank_kernel, B, block_threads(n), smem, stream, scores, labels, offsets, grad, loss_per_query, n, 1.0f / den, top_k);
    return check_launch("softrank");
}

int ptrb200_mdprank_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, const int32_t* perm,
                            const float* unif, int32_t* sample_out, float* grad, float* loss_per_query, int B, int n,
                            int top_k, float gamma, float temperature, int distribution, uint64_t seed, uint64_t offset,
                            ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    if (distribution != PTRB200_MDP_PL && distribution != PTRB200_MDP_STPL) {
        set_error("mdprank: unknown distribution %d", distribution);
        return PTRB200_ERR_INVALID;
    }
    if (!(temperature > 0.0f)) { set_error("mdprank: temperature must be positive"); return PTRB200_ERR_INVALID; }
    if (perm && distribution == PTRB200_MDP_STPL) {
        set_error("mdprank: an injected ordering is PL only (STPL's action values come from the uniforms)");
        return PTRB200_ERR_INVALID;
    }
    const int npow2 = next_pow2(n);
    const size_t smem = (size_t)npow2 * 8 + (size_t)n * 4 * 5 + 128 * 4;
    if ((rc = allow_smem(mdprank_kernel, smem))) return rc;
    PTRB200_LAUNCH(mdprank_kernel, B, block_threads(n), smem, stream, scores, labels, offsets, perm, unif, sample_out, grad,
                   loss_per_query, n, npow2, top_k, gamma, temperature, distribution == PTRB200_MDP_STPL ? 1 : 0, seed, offset);
    return check_launch("mdprank");
}

int ptrb200_sinkstep(const float* dist, const float* log_nu, const float* log_u, float* log_v,
                     int B, int d1, int d2, float lambda, ptrb200_stream_t stream) {
    if (!dist || !log_nu || !log_u || !log_v || B <= 0 || d1 <= 0 || d2 <= 0 || !(lambda != 0.0f)) {
        set_error("sinkstep: bad arguments (B=%d d1=%d d2=%d)", B, d1, d2);
        return PTRB200_ERR_INVALID;
    }
    if (B > 65535) { set_error("sinkstep: B=%d exceeds the grid's y extent", B); return PTRB200_ERR_UNSUPPORTED; }
    dim3 grid((d2 + 31) / 32, B);
    PTRB200_LAUNCH(sinkstep_kernel, grid, 32 * SINK_WARPS, 0, stream, dist, log_nu, log_u, log_v, d1, d2, lambda);
    return check_launch("sinkstep");
}

}  // extern "C"
