// losses.cu -- fused ranking-loss forward + gradient kernels (one CTA per query).
//
// Every kernel stages one query's scores/labels in shared memory, ranks the list
// in-CTA (bitonic sort on packed keys), and walks the pair / scan structure
// without ever materialising the reference's [B,n,n] temporaries.  Algorithmic
// HBM traffic: 12n bytes per query (scores + labels in, grad out).
//
// Reference functions replaced (wildltr/ptranking @ f1d366c):
//   RankNet     ptranking/ltr_adhoc/pairwise/ranknet.py:25-36
//   LambdaRank  ptranking/ltr_adhoc/listwise/lambdarank.py:27-56
//   LambdaLoss  ptranking/ltr_adhoc/listwise/lambdaloss.py:73-132
//   ListNet     ptranking/ltr_adhoc/listwise/listnet.py:39
//   ListMLE     ptranking/ltr_adhoc/listwise/listmle.py:83-97
//   ApproxNDCG  ptranking/ltr_adhoc/listwise/approxNDCG.py:19-28,45-62
//   nDCG@ks     ptranking/base/ranker.py:67-95, metric/adhoc/adhoc_metric.py:219-260
#include "losses_common.cuh"

namespace ptrb200 {

// ---------------------------------------------------------------------------
// RankNet / LambdaRank: weighted BCE over all pairs a<b (ATen clamps kept).
// Thread-per-row: the thread owning sorted position i visits every j != i and
// evaluates the ordered pair (min(i,j), max(i,j)) exactly as the reference's
// upper-triangular tensors do, so no scatter / atomics are needed.
// LambdaRank skips equal-label pairs, as lambdarank_runs_kernel does: their
// weight |G_i - G_j| |1/D_i - 1/D_j| is exactly 0 and they add exactly +-0,
// except in a list without a relevant document (iDCG = 0), where every
// normalised gain is 0/0.  Skipping them there too gives such a list loss 0
// and gradient 0 whichever kernel its launch picks.
// ---------------------------------------------------------------------------
template <bool LAMBDA>
__global__ void pairwise_bce_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                    float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets,
                                    int nmax, int npow2max, float sigma) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* ss = reinterpret_cast<float*>(keys + (LAMBDA ? npow2max : 0));
    float* ys = ss + nmax;
    float* ng = ys + nmax;
    float* dinv = ng + nmax;
    float* gout = dinv + nmax;
    int* idx = reinterpret_cast<int*>(gout + nmax);
    float* red = reinterpret_cast<float*>(idx + nmax);

    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const float* s = scores + sp.base;
    const float* y = labels + sp.base;

    if (LAMBDA) {
        const float idcg = block_idcg(y, n, npow2, /*presort=*/true, keys, red);
        for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(s[i], i) : 0ull;
        block_sort_desc(keys, npow2);
        for (int r = threadIdx.x; r < n; r += blockDim.x) {
            const int id = key_index(keys[r]);
            idx[r] = id;
            ss[r] = s[id];
            const float yr = y[id];
            ys[r] = yr;
            ng[r] = gain_of(yr) / idcg;
            dinv[r] = 1.0f / log2_rank(r);
        }
    } else {
        for (int r = threadIdx.x; r < n; r += blockDim.x) { ss[r] = s[r]; ys[r] = y[r]; idx[r] = r; }
    }
    __syncthreads();

    float loss = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float si = ss[i], yi = ys[i];
        const float gi = LAMBDA ? ng[i] : 0.0f, di = LAMBDA ? dinv[i] : 0.0f;
        float acc = 0.0f;
        for (int j = 0; j < n; ++j) {
            if (j == i || (LAMBDA && yi == ys[j])) continue;
            const bool upper = j > i;
            float x = sigma * (si - ss[j]);
            float S = fminf(fmaxf(yi - ys[j], -1.0f), 1.0f);
            if (!upper) { x = -x; S = -S; }
            const float w = LAMBDA ? fabsf(gi - ng[j]) * fabsf(di - dinv[j]) : 1.0f;
            const float p = sigmoid_aten(x);
            const float q = 1.0f - p;
            const float pq = p * q;
            const float pbar = 0.5f * (1.0f + S);
            // BCE backward (p-pbar)/max(pq,1e-12), sigmoid backward * pq, then * sigma
            const float g = sigma * (w * ((p - pbar) / fmaxf(pq, 1e-12f))) * pq;
            acc += upper ? g : -g;
            if (upper) {
                const float lp = fmaxf(logf(p), -100.0f);
                const float lq = fmaxf(logf(q), -100.0f);
                loss -= w * (pbar * lp + (1.0f - pbar) * lq);
            }
        }
        gout[idx[i]] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) grad[sp.base + i] = gout[i];
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// Same loss, every unordered pair {a<b} evaluated ONCE (lists of up to 1024 documents, one thread per position).
// In step k thread i takes the pair (i, (i+k) mod n), k = 1..floor((n-1)/2) [+ the n/2 diameter for even n]: a circulant
// schedule that touches each pair exactly once and keeps all lanes busy.  The pair's gradient goes to the thread's own
// accumulator and, negated, to its partner through a double-buffered shared-memory mailbox (one writer per slot per
// step, so no atomics and a fixed summation order); KB steps share one barrier.
constexpr int PAIR_KB = 4;

template <bool LAMBDA>
static __device__ __forceinline__ float pair_term(float sa, float sb, float ya, float yb, float ga, float gb, float da, float db,
                                                  float sigma, float& loss) {
    const float x = sigma * (sa - sb);
    const float S = fminf(fmaxf(ya - yb, -1.0f), 1.0f);
    const float w = LAMBDA ? fabsf(ga - gb) * fabsf(da - db) : 1.0f;
    const float p = sigmoid_aten(x);
    const float q = 1.0f - p;
    const float pq = p * q;
    const float pbar = 0.5f * (1.0f + S);
    // BCE backward (p-pbar)/max(pq,1e-12), sigmoid backward *pq, then *sigma (the quotient to 2 ulp: a reciprocal and a multiply)
    const float g = sigma * (w * __fdividef(p - pbar, fmaxf(pq, 1e-12f))) * pq;
    // A log whose coefficient is zero contributes exactly +-0 (the -100 clamp keeps it finite), so for pbar in {0, 1}
    // -- always the case when w != 0 under integer relevance grades -- ONE logarithm is evaluated.
    float acc;
    if (pbar == 1.0f || pbar == 0.0f) acc = fmaxf(logf(pbar == 1.0f ? p : q), -100.0f);
    else acc = pbar * fmaxf(logf(p), -100.0f) + (1.0f - pbar) * fmaxf(logf(q), -100.0f);
    loss -= w * acc;
    return g;
}

template <bool LAMBDA>
__global__ void pairwise_bce_circ_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                         float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets,
                                         int nmax, int npow2max, float sigma) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* ss = reinterpret_cast<float*>(keys + (LAMBDA ? npow2max : 0));
    float* ys = ss + nmax;
    float* ng = ys + nmax;
    float* dinv = ng + nmax;
    float* gout = dinv + nmax;
    int* idx = reinterpret_cast<int*>(gout + nmax);
    float* red = reinterpret_cast<float*>(idx + nmax);
    float* xch = red + 33;                              // [2][PAIR_KB][nmax] partner mailbox

    const int b = blockIdx.x, i = threadIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const float* s = scores + sp.base;
    const float* y = labels + sp.base;
    if (LAMBDA) {
        const float idcg = block_idcg(y, n, npow2, /*presort=*/true, keys, red);
        for (int t = threadIdx.x; t < npow2; t += blockDim.x) keys[t] = t < n ? desc_key(s[t], t) : 0ull;
        block_sort_desc(keys, npow2);
        for (int r = threadIdx.x; r < n; r += blockDim.x) {
            const int id = key_index(keys[r]);
            idx[r] = id;
            ss[r] = s[id];
            const float yr = y[id];
            ys[r] = yr;
            ng[r] = gain_of(yr) / idcg;
            dinv[r] = 1.0f / log2_rank(r);
        }
    } else {
        for (int r = threadIdx.x; r < n; r += blockDim.x) { ss[r] = s[r]; ys[r] = y[r]; idx[r] = r; }
    }
    __syncthreads();

    const bool mine = i < n;
    const float si = mine ? ss[i] : 0.0f, yi = mine ? ys[i] : 0.0f;
    const float gi = (LAMBDA && mine) ? ng[i] : 0.0f, di = (LAMBDA && mine) ? dinv[i] : 0.0f;
    float own = 0.0f, loss = 0.0f;
    auto visit = [&](int j, float* slot) {              // pair {i, j}: ordered as (min, max) like the reference's triu
        const float sj = ss[j], yj = ys[j];
        const float gj = LAMBDA ? ng[j] : 0.0f, dj = LAMBDA ? dinv[j] : 0.0f;
        const bool first = i < j;
        // (operand selects, then ONE evaluation: a conditional between two calls compiles to both)
        const float g = pair_term<LAMBDA>(first ? si : sj, first ? sj : si, first ? yi : yj, first ? yj : yi,
                                          first ? gi : gj, first ? gj : gi, first ? di : dj, first ? dj : di, sigma, loss);
        own += first ? g : -g;
        slot[j] = first ? -g : g;
    };
    const int half = (n - 1) / 2;
    int buf = 0;
    for (int k0 = 1; k0 <= half; k0 += PAIR_KB) {
        float* xb = xch + (size_t)buf * PAIR_KB * nmax;
#pragma unroll
        for (int kk = 0; kk < PAIR_KB; ++kk) {
            const int k = k0 + kk;
            if (mine && k <= half) {
                int j = i + k;
                if (j >= n) j -= n;
                visit(j, xb + kk * nmax);
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < PAIR_KB; ++kk)
            if (mine && k0 + kk <= half) own += xb[kk * nmax + i];
        buf ^= 1;
    }
    if ((n & 1) == 0 && n >= 2) {                       // the diameter pairs (i, i + n/2)
        float* xb = xch + (size_t)buf * PAIR_KB * nmax;
        if (i < n / 2) visit(i + n / 2, xb);
        __syncthreads();
        if (mine && i >= n / 2) own += xb[i];
    }
    if (mine) gout[idx[i]] = own;
    __syncthreads();
    for (int t = threadIdx.x; t < n; t += blockDim.x) grad[sp.base + t] = gout[t];
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// LambdaRank with the tie pairs left out.  The pair weight |G_a - G_b| |1/D_a - 1/D_b| is exactly zero whenever the two
// labels are equal (39 % of all pairs under the MSLR-WEB30K label marginals), and such a pair then adds exactly +-0 to the
// loss and to both gradients.  Labels arrive presorted descending (lambdarank.py:36), so equal labels form contiguous runs of
// the ORIGINAL document order: thread i (= document i) visits precisely the documents [0, run_start(i)) -- all strictly
// better labelled -- which enumerates every non-tie pair once, with trip counts that are uniform inside a warp (a warp lies
// in one run except at run boundaries).  All lanes of a warp visit the same partner in the same step, so the partner's
// share of the gradient is one fixed-order warp sum per step, accumulated in a per-warp row of shared memory (no atomics:
// bit-for-bit deterministic).  Each pair is oriented by predicted rank exactly like the reference's upper triangle.
__global__ void lambdarank_runs_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                       float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets,
                                       int nmax, int npow2max, float sigma) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* ss = reinterpret_cast<float*>(keys + npow2max);     // by ORIGINAL index
    float* ys = ss + nmax;
    float* ng = ys + nmax;
    float* dinv = ng + nmax;
    int* rk = reinterpret_cast<int*>(dinv + nmax);              // predicted rank of document i
    float* gown = reinterpret_cast<float*>(rk + nmax);          // each document's own share of its gradient
    float* red = gown + nmax;
    float* part = red + 33;                                     // [warps][nmax] partner contributions
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const float* s = scores + sp.base;
    const float* y = labels + sp.base;
    const float idcg = block_idcg(y, n, npow2, /*presort=*/true, keys, red);
    for (int t = threadIdx.x; t < npow2; t += blockDim.x) keys[t] = t < n ? desc_key(s[t], t) : 0ull;
    block_sort_desc(keys, npow2);
    for (int r = threadIdx.x; r < n; r += blockDim.x) rk[key_index(keys[r])] = r;
    for (int t = threadIdx.x; t < n; t += blockDim.x) { ss[t] = s[t]; const float yt = y[t]; ys[t] = yt; ng[t] = gain_of(yt) / idcg; }
    for (int t = threadIdx.x; t < nwarps * nmax; t += blockDim.x) part[t] = 0.0f;
    __syncthreads();
    for (int t = threadIdx.x; t < n; t += blockDim.x) dinv[t] = 1.0f / log2_rank(rk[t]);
    __syncthreads();
    float loss = 0.0f;
    float* prow = part + (size_t)warp * nmax;
    // lists longer than the CTA are walked in passes of blockDim documents (warps stay aligned with label runs)
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const bool mine = i < n;
        const float si = mine ? ss[i] : 0.0f, yi = mine ? ys[i] : 0.0f, gi = mine ? ng[i] : 0.0f, di = mine ? dinv[i] : 0.0f;
        const int ri = mine ? rk[i] : 0;
        int start = 0;                                          // first index carrying label yi (labels sorted descending)
        if (mine) {
            int lo = 0, hi = i;                                 // ys[lo..hi] is non-increasing and ys[i] == yi
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (ys[mid] > yi) lo = mid + 1; else hi = mid; }
            start = lo;
        }
        int trips = start;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) trips = max(trips, __shfl_xor_sync(0xffffffffu, trips, o));
        float own = 0.0f;
        for (int p = 0; p < trips; ++p) {
            float gp = 0.0f;                                    // this lane's contribution to document p's gradient
            if (p < start) {
                const float sj = ss[p], yj = ys[p], gj = ng[p], dj = dinv[p];
                const bool first = ri < rk[p];                  // the better-ranked document is the pair's first element
                const float g = pair_term<true>(first ? si : sj, first ? sj : si, first ? yi : yj, first ? yj : yi,
                                                first ? gi : gj, first ? gj : gi, first ? di : dj, first ? dj : di, sigma, loss);
                own += first ? g : -g;
                gp = first ? -g : g;
            }
            gp = warp_sum(gp);
            if (lane == 0) prow[p] += gp;
        }
        if (mine) gown[i] = own;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float tot = gown[i];
        for (int w = 0; w < nwarps; ++w) tot += part[(size_t)w * nmax + i];
        grad[sp.base + i] = tot;
    }
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// ---------------------------------------------------------------------------
// LambdaLoss (NDCG_Loss1 / NDCG_Loss2 / NDCG_Loss2++), truncated at the top-k
// predicted positions.
// ---------------------------------------------------------------------------
#define LOG2_EPS (-26.575424759098897f)   /* log2(1e-8) */
#define INV_LN2 1.4426950408889634f

struct LLTerm { float cell, g; };

// term of the ordered pair (a,b): loss cell and d cell / d (s_a - s_b)
static __device__ __forceinline__ LLTerm lambdaloss_term(float sa, float sb, float w, float sigma) {
    float dx = fminf(fmaxf(sa - sb, -1e8f), 1e8f);
    if (dx != dx) dx = 0.0f;                               // lambdaloss.py:116
    const float p = sigmoid_aten(sigma * dx);
    const float pc = fmaxf(p, 1e-8f);
    const float t = w * log2f(pc);                         // log2(pc^w)
    LLTerm r;
    r.cell = -fmaxf(t, LOG2_EPS);
    const bool live = (p >= 1e-8f) && (t >= LOG2_EPS);
    r.g = live ? -(w * sigma) * (1.0f - p) * INV_LN2 : 0.0f;
    return r;
}

__global__ void lambdaloss_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                  float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets,
                                  int nmax, int npow2max, int k, float sigma, float mu, int loss_type, int presort) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* ss = reinterpret_cast<float*>(keys + npow2max);
    float* ys = ss + nmax;
    float* ng = ys + nmax;
    float* gout = ng + nmax;
    int* idx = reinterpret_cast<int*>(gout + nmax);
    float* red = reinterpret_cast<float*>(idx + nmax);

    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const int K = k < n ? k : n;                          // truncation at the top-k predicted positions (lambdaloss.py:122-123)
    const float* s = scores + sp.base;
    const float* y = labels + sp.base;

    const float idcg = block_idcg(y, n, npow2, presort != 0, keys, red);
    __syncthreads();
    for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(s[i], i) : 0ull;
    block_sort_desc(keys, npow2);
    for (int r = threadIdx.x; r < n; r += blockDim.x) {
        const int id = key_index(keys[r]);
        idx[r] = id;
        ss[r] = s[id];
        const float yr = y[id];
        ys[r] = yr;
        ng[r] = gain_of(yr) / idcg;
        gout[r] = 0.0f;
    }
    __syncthreads();

    float loss = 0.0f;
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        const float si = ss[i], yi = ys[i], gi = ng[i];
        const float Di = log2_rank(i);
        float acc = 0.0f;
        for (int j = 0; j < K; ++j) {
            const float sj = ss[j], yj = ys[j], gj = ng[j];
            if (loss_type == PTRB200_NDCG_LOSS1) {
                // weight of cell (a,b) is w_b = ng_b * log2(b+2); every cell of the k x k window counts
                const LLTerm tij = lambdaloss_term(si, sj, gj * log2_rank(j), sigma);
                loss += tij.cell;
                if (j != i) {
                    const LLTerm tji = lambdaloss_term(sj, si, gi * Di, sigma);
                    acc += tij.g - tji.g;
                }
            } else {
                if (j == i || yi == yj) continue;
                const int d = i > j ? i - j : j - i;
                const float dgap = fabsf(log2f((float)d + 1.0f) - log2f((float)d + 2.0f));
                float w = dgap;
                if (loss_type == PTRB200_NDCG_LOSS2PP) w = fabsf(Di - log2_rank(j)) + mu * dgap;
                w *= fabsf(gi - gj);
                if (yi > yj) {
                    const LLTerm t = lambdaloss_term(si, sj, w, sigma);
                    loss += t.cell;
                    acc += t.g;
                } else {
                    const LLTerm t = lambdaloss_term(sj, si, w, sigma);
                    acc -= t.g;
                }
            }
        }
        gout[i] = acc;
    }
    __syncthreads();
    // scatter back to document order
    for (int r = threadIdx.x; r < n; r += blockDim.x) grad[sp.base + idx[r]] = gout[r];
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// ---------------------------------------------------------------------------
// ListNet: cross entropy between softmax(labels) and softmax(scores)
// ---------------------------------------------------------------------------
__global__ void listnet_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                               float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets, int nmax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* ss = reinterpret_cast<float*>(smem_raw);
    float* ys = ss + nmax;
    float* red = ys + nmax;
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    float ms = -INFINITY, my = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float a = scores[sp.base + i], c = labels[sp.base + i];
        ss[i] = a; ys[i] = c;
        ms = fmaxf(ms, a); my = fmaxf(my, c);
    }
    ms = block_max(ms, red);
    my = block_max(my, red);
    float zs = 0.0f, zy = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { zs += expf(ss[i] - ms); zy += expf(ys[i] - my); }
    zs = block_sum(zs, red);
    zy = block_sum(zy, red);
    const float log_zs = logf(zs);
    float loss = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float py = expf(ys[i] - my) / zy;
        const float lsm = (ss[i] - ms) - log_zs;
        loss -= py * lsm;
        grad[sp.base + i] = expf(lsm) - py;
    }
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// ---------------------------------------------------------------------------
// ListMLE: Plackett-Luce likelihood of the (tie-shuffled) ideal ordering
// ---------------------------------------------------------------------------
__global__ void listmle_kernel(const float* __restrict__ scores, const int32_t* __restrict__ perm,
                               float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets, int nmax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* z = reinterpret_cast<float*>(smem_raw);
    float* e = z + nmax;
    float* c = e + nmax;
    int* pid = reinterpret_cast<int*>(c + nmax);
    float* red = reinterpret_cast<float*>(pid + nmax);
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    float m = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int id = clampi(perm[sp.base + i], 0, n - 1);      // perm holds positions within the query's own list
        pid[i] = id;
        const float v = scores[sp.base + id];
        z[i] = v;
        m = fmaxf(m, v);
    }
    m = block_max(m, red);
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float v = expf(z[i] - m); e[i] = v; c[i] = v; }
    __syncthreads();
    block_scan_inclusive<true>(c, n, red);               // c_i = sum_{j>=i} e_j
    float loss = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float ci = c[i];
        loss += (logf(ci) + m) - z[i];
        c[i] = 1.0f / ci;
    }
    __syncthreads();
    block_scan_inclusive<false>(c, n, red);              // c_k = sum_{i<=k} 1/C_i
    for (int i = threadIdx.x; i < n; i += blockDim.x) grad[sp.base + pid[i]] = e[i] * c[i] - 1.0f;
    loss = block_sum(loss, red);
    if (threadIdx.x == 0) loss_q[b] = loss;
}

// perm for ListMLE: labels descending, ties broken by Philox noise (sampling_utils.py:13-28)
__global__ void shuffle_ties_kernel(const float* __restrict__ labels, int32_t* __restrict__ perm, const int32_t* __restrict__ offsets,
                                    int nmax, int npow2max, uint64_t seed, uint64_t offset) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) return;
    for (int i = threadIdx.x; i < npow2; i += blockDim.x) {
        u64 k = 0ull;
        if (i < n) {
            const u64 hi = desc_key(labels[sp.base + i], 0) >> 32;
            const uint32_t rnd = dropout_bits(seed, offset, (uint64_t)sp.base + (uint64_t)i);
            // [label order : 32][random : 19][1][doc index : 12]  (n <= 4096); low field never 0
            k = (hi << 32) | ((u64)(rnd >> 13) << 13) | (1ull << 12) | (u64)i;
        }
        keys[i] = k;
    }
    block_sort_desc(keys, npow2);
    for (int r = threadIdx.x; r < n; r += blockDim.x) perm[sp.base + r] = (int32_t)(keys[r] & 0xfffull);
}

// ---------------------------------------------------------------------------
// ApproxNDCG
// ---------------------------------------------------------------------------
// Robust_Sigmoid forward, base/utils.py:62-78 (branch on the sign of the unscaled input)
static __device__ __forceinline__ float robust_sigmoid(float in, float alpha) {
    const float x = alpha * in;
    if (in > 0.0f) return __fdividef(1.0f, 1.0f + expf(-x));
    if (in < 0.0f) { const float ex = expf(x); return __fdividef(ex, 1.0f + ex); }
    return 0.5f;
}

__global__ void inv_idcg_kernel(const float* __restrict__ labels, float* __restrict__ inv_idcg, const int32_t* __restrict__ offsets,
                                int nmax, int npow2max, int presort) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* red = reinterpret_cast<float*>(keys + npow2max);
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x == 0) inv_idcg[b] = 0.0f; return; }      // an empty list adds nothing to sum_a 1/iDCG_a
    const float idcg = block_idcg(labels + sp.base, n, npow2, presort != 0, keys, red);
    if (threadIdx.x == 0) inv_idcg[b] = 1.0f / idcg;
}

__global__ void approxndcg_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                  float* __restrict__ grad, float* __restrict__ loss_q, const int32_t* __restrict__ offsets,
                                  const float* __restrict__ scratch, int B, int nmax, float alpha, int batch_coupled) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* ss = reinterpret_cast<float*>(smem_raw);
    float* cc = ss + nmax;
    float* red = cc + nmax;
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n;
    if (n == 0) { if (threadIdx.x == 0) loss_q[b] = 0.0f; return; }
    const float scale = batch_coupled ? scratch[B] : scratch[b];
    for (int i = threadIdx.x; i < n; i += blockDim.x) ss[i] = scores[sp.base + i];
    __syncthreads();
    float dcg = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float si = ss[i];
        float pi = 0.0f;
        for (int j = 0; j < n; ++j) pi += robust_sigmoid(ss[j] - si, alpha);
        pi += 0.5f;
        const float G = gain_of(labels[sp.base + i]);
        const float lg = log2f(pi + 1.0f);
        dcg += G / lg;
        cc[i] = scale * G / (lg * lg * (pi + 1.0f) * 0.6931471805599453f);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const float sj = ss[j], cj = cc[j];
        float acc = 0.0f;
        for (int i = 0; i < n; ++i) {
            const float sg = robust_sigmoid(sj - ss[i], alpha);
            acc += (alpha * sg * (1.0f - sg)) * (cc[i] - cj);
        }
        grad[sp.base + j] = acc;
    }
    dcg = block_sum(dcg, red);
    if (threadIdx.x == 0) loss_q[b] = -scale * dcg;
}

// ---------------------------------------------------------------------------
// deterministic sum, nDCG@ks
// ---------------------------------------------------------------------------
__global__ void sum_kernel(const float* __restrict__ x, float* __restrict__ out, int n) {
    __shared__ float red[33];
    float v = 0.0f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) v += x[i];
    v = block_sum(v, red);
    if (threadIdx.x == 0) out[0] = v;
}

struct Cutoffs { int k[PTRB200_MAX_CUTOFFS]; int n; };

__global__ void ndcg_at_ks_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                  Cutoffs ks, float* __restrict__ out, int32_t* __restrict__ order, const int32_t* __restrict__ offsets,
                                  int nmax, int npow2max, int presort) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* tsys = reinterpret_cast<float*>(keys + npow2max);   // gain/discount in predicted order
    float* tide = tsys + nmax;                                 // gain/discount in ideal order
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x < ks.n) out[(size_t)b * ks.n + threadIdx.x] = 0.0f; return; }
    const float* s = scores + sp.base;
    const float* y = labels + sp.base;
    if (presort) {
        for (int r = threadIdx.x; r < n; r += blockDim.x) tide[r] = gain_of(y[r]) / log2_rank(r);
    } else {
        for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(y[i], i) : 0ull;
        block_sort_desc(keys, npow2);
        for (int r = threadIdx.x; r < n; r += blockDim.x) tide[r] = gain_of(y[key_index(keys[r])]) / log2_rank(r);
        __syncthreads();
    }
    for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(s[i], i) : 0ull;
    block_sort_desc(keys, npow2);
    for (int r = threadIdx.x; r < n; r += blockDim.x) {
        const int id = key_index(keys[r]);
        if (order) order[sp.base + r] = id;
        tsys[r] = gain_of(y[id]) / log2_rank(r);
    }
    __syncthreads();
    // sequential cumulative sums (the order torch.cumsum uses), one thread per series
    if (threadIdx.x == 0) {
        float cs = 0.0f, ci = 0.0f;
        int c = 0, r = 0;
        for (; c < ks.n; ++c) {
            const int k = ks.k[c];
            if (k > n) { out[(size_t)b * ks.n + c] = 0.0f; continue; }
            for (; r < k; ++r) { cs += tsys[r]; ci += tide[r]; }
            out[(size_t)b * ks.n + c] = cs / ci;
        }
    }
}


// nDCG, nERR, AP and P at every cutoff from ONE sort per query (SURVEY 8f row 1: adhoc_performance_at_ks,
// base/ranker.py:202-263 + metric/adhoc/adhoc_metric.py:18-260).  out[B][4][nks], metric order nDCG,nERR,AP,P.
__global__ void adhoc_metrics_kernel(const float* __restrict__ scores, const float* __restrict__ labels,
                                     Cutoffs ks, float* __restrict__ out, const int32_t* __restrict__ offsets,
                                     int nmax, int npow2max, int presort, float max_label) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* ysys = reinterpret_cast<float*>(keys + npow2max);   // labels in predicted order
    float* yide = ysys + nmax;                                 // labels in ideal order
    const int b = blockIdx.x;
    const ListSpan sp = list_span(offsets, b, nmax);
    const int n = sp.n, npow2 = offsets ? next_pow2(n) : npow2max;
    if (n == 0) { if (threadIdx.x < 4 * ks.n) out[(size_t)b * 4 * ks.n + threadIdx.x] = 0.0f; return; }
    const float* s = scores + sp.base;
    const float* y = labels + sp.base;
    if (presort) {
        for (int r = threadIdx.x; r < n; r += blockDim.x) yide[r] = y[r];
    } else {
        for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(y[i], i) : 0ull;
        block_sort_desc(keys, npow2);
        for (int r = threadIdx.x; r < n; r += blockDim.x) yide[r] = y[key_index(keys[r])];
        __syncthreads();
    }
    for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(s[i], i) : 0ull;
    block_sort_desc(keys, npow2);
    for (int r = threadIdx.x; r < n; r += blockDim.x) ysys[r] = y[key_index(keys[r])];
    __syncthreads();
    // four independent sequential scans (the order torch.cumsum / cumprod use), one warp each
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane != 0 || warp >= 4) return;
    float* o = out + ((size_t)b * 4 + warp) * ks.n;
    int c = 0, r = 0;
    if (warp == 0) {                    // nDCG
        float cs = 0.0f, ci = 0.0f;
        for (; c < ks.n; ++c) {
            const int k = ks.k[c];
            if (k > n) { o[c] = 0.0f; continue; }
            for (; r < k; ++r) { const float d = log2_rank(r); cs += gain_of(ysys[r]) / d; ci += gain_of(yide[r]) / d; }
            o[c] = cs / ci;
        }
    } else if (warp == 1) {             // nERR: sum_r (1/rank * satis_r) * prod_{q<r}(1 - satis_q)
        const float denom = exp2f(max_label);
        float es = 0.0f, ei = 0.0f, us = 1.0f, ui = 1.0f;
        for (; c < ks.n; ++c) {
            const int k = ks.k[c];
            if (k > n) { o[c] = 0.0f; continue; }
            for (; r < k; ++r) {
                const float inv = 1.0f / ((float)r + 1.0f);
                const float ps = gain_of(ysys[r]) / denom, pi = gain_of(yide[r]) / denom;
                es += (inv * ps) * us; ei += (inv * pi) * ui;
                us *= (1.0f - ps); ui *= (1.0f - pi);
            }
            o[c] = es / ei;
        }
    } else if (warp == 2) {             // AP (ideal labels are NOT binarised in the denominator, as in the reference)
        float cum_rel = 0.0f, cum_prec = 0.0f, cum_ideal = 0.0f;
        for (; c < ks.n; ++c) {
            const int k = ks.k[c];
            if (k > n) { o[c] = 0.0f; continue; }
            for (; r < k; ++r) {
                const float bi = fminf(fmaxf(ysys[r], 0.0f), 1.0f);
                cum_rel += bi;
                cum_prec += (cum_rel / ((float)r + 1.0f)) * bi;
                cum_ideal += yide[r];
            }
            o[c] = cum_prec / cum_ideal;
        }
    } else {                            // P
        float cum_rel = 0.0f;
        for (; c < ks.n; ++c) {
            const int k = ks.k[c];
            if (k > n) { o[c] = 0.0f; continue; }
            for (; r < k; ++r) cum_rel += fminf(fmaxf(ysys[r], 0.0f), 1.0f);
            o[c] = cum_rel / (float)k;
        }
    }
}

// ---------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------
template <bool LAMBDA>
static int launch_pairwise(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_q,
                           int B, int n, float sigma, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_q, B, n);
    if (rc) return rc;
    const int npow2 = next_pow2(n);
    const size_t smem = (LAMBDA ? (size_t)npow2 * 8 : 0) + (size_t)n * 4 * 6 + 33 * 4;
    // tie pairs skipped: partners = the better-labelled prefix.  One thread per document up to 512; longer lists (up to 2048)
    // are walked in passes by 1024 threads (512 when the per-warp partner rows would not fit in shared memory otherwise)
    int threads = n <= 512 ? block_threads(n) : 1024;
    size_t smem_r = (size_t)npow2 * 8 + (size_t)n * 4 * 6 + 33 * 4 + (size_t)(threads / 32) * n * 4;
    if (smem_r > 227 * 1024 && n > 512) { threads = 512; smem_r = (size_t)npow2 * 8 + (size_t)n * 4 * 6 + 33 * 4 + (size_t)(threads / 32) * n * 4; }
    if (LAMBDA && n <= 2048 && smem_r <= 227 * 1024) {
        if ((rc = allow_smem(lambdarank_runs_kernel, smem_r))) return rc;
        PTRB200_LAUNCH_TAG("pairwise_bce_kernel<LAMBDA>", lambdarank_runs_kernel, B, threads, smem_r, stream,
                           scores, labels, grad, loss_q, offsets, n, npow2, sigma);
        return check_launch("lambdarank");
    }
    if (n <= 1024) {        // one thread per position: each unordered pair once
        const size_t smem_c = smem + (size_t)2 * PAIR_KB * n * 4;
        if ((rc = allow_smem(pairwise_bce_circ_kernel<LAMBDA>, smem_c))) return rc;
        PTRB200_LAUNCH_TAG(LAMBDA ? "pairwise_bce_kernel<LAMBDA>" : "pairwise_bce_kernel<RANKNET>", pairwise_bce_circ_kernel<LAMBDA>, B, block_threads(n), smem_c, stream,
                           scores, labels, grad, loss_q, offsets, n, npow2, sigma);
        return check_launch(LAMBDA ? "lambdarank" : "ranknet");
    }
    if ((rc = allow_smem(pairwise_bce_kernel<LAMBDA>, smem))) return rc;
    PTRB200_LAUNCH(pairwise_bce_kernel<LAMBDA>, B, block_threads(n), smem, stream, scores, labels, grad, loss_q, offsets, n, npow2, sigma);
    return check_launch(LAMBDA ? "lambdarank" : "ranknet");
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_ranknet_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                            int B, int n, float sigma, ptrb200_stream_t stream) {
    return launch_pairwise<false>(scores, labels, offsets, grad, loss_per_query, B, n, sigma, stream);
}

int ptrb200_lambdarank_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                               int B, int n, float sigma, ptrb200_stream_t stream) {
    return launch_pairwise<true>(scores, labels, offsets, grad, loss_per_query, B, n, sigma, stream);
}

int ptrb200_lambdaloss_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                               int B, int n, int k, float sigma, float mu, int loss_type, int presort,
                               ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    if (loss_type < PTRB200_NDCG_LOSS1 || loss_type > PTRB200_NDCG_LOSS2PP || k <= 0) {
        set_error("lambdaloss: bad loss_type=%d or k=%d", loss_type, k);
        return PTRB200_ERR_INVALID;
    }
    const int npow2 = next_pow2(n);
    const size_t smem = (size_t)npow2 * 8 + (size_t)n * 4 * 5 + 33 * 4;
    if ((rc = allow_smem(lambdaloss_kernel, smem))) return rc;
    PTRB200_LAUNCH(lambdaloss_kernel, B, block_threads(n), smem, stream, scores, labels, grad, loss_per_query,
                   offsets, n, npow2, k, sigma, mu, loss_type, presort);
    return check_launch("lambdaloss");
}

int ptrb200_listnet_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                            int B, int n, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    const size_t smem = (size_t)n * 4 * 2 + 33 * 4;
    if ((rc = allow_smem(listnet_kernel, smem))) return rc;
    PTRB200_LAUNCH(listnet_kernel, B, block_threads(n), smem, stream, scores, labels, grad, loss_per_query, offsets, n);
    return check_launch("listnet");
}

int ptrb200_listmle_fwd_bwd(const float* scores, const int32_t* perm, const int32_t* offsets, float* grad, float* loss_per_query,
                            int B, int n, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, perm, grad, loss_per_query, B, n);
    if (rc) return rc;
    const size_t smem = (size_t)n * 4 * 4 + 72 * 4;
    if ((rc = allow_smem(listmle_kernel, smem))) return rc;
    PTRB200_LAUNCH(listmle_kernel, B, block_threads(n), smem, stream, scores, perm, grad, loss_per_query, offsets, n);
    return check_launch("listmle");
}

int ptrb200_shuffle_ties_perm(const float* labels, const int32_t* offsets, int32_t* perm, int B, int n,
                              uint64_t seed, uint64_t offset, ptrb200_stream_t stream) {
    int rc = check_list_args(labels, perm, labels, perm, B, n);
    if (rc) return rc;
    const int npow2 = next_pow2(n);
    PTRB200_LAUNCH(shuffle_ties_kernel, B, block_threads(n), (size_t)npow2 * 8, stream, labels, perm, offsets, n, npow2, seed, offset);
    return check_launch("shuffle_ties");
}

int ptrb200_approxndcg_fwd_bwd(const float* scores, const float* labels, const int32_t* offsets, float* grad, float* loss_per_query,
                               float* scratch, int B, int n, float alpha, int presort, int batch_coupled,
                               ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, grad, loss_per_query, B, n);
    if (rc) return rc;
    if (!scratch) { set_error("approxndcg: scratch (B+1 floats) is NULL"); return PTRB200_ERR_INVALID; }
    const int npow2 = next_pow2(n);
    PTRB200_LAUNCH(inv_idcg_kernel, B, block_threads(n), (size_t)npow2 * 8 + 33 * 4, stream, labels, scratch, offsets, n, npow2, presort);
    PTRB200_LAUNCH(sum_kernel, 1, 256, 0, stream, (const float*)scratch, scratch + B, B);
    const size_t smem = (size_t)n * 4 * 2 + 33 * 4;
    if ((rc = allow_smem(approxndcg_kernel, smem))) return rc;
    PTRB200_LAUNCH(approxndcg_kernel, B, block_threads(n), smem, stream, scores, labels, grad, loss_per_query, offsets,
                   (const float*)scratch, B, n, alpha, batch_coupled);
    return check_launch("approxndcg");
}

int ptrb200_sum_f32(const float* x, float* out, int n, ptrb200_stream_t stream) {
    if (!x || !out || n <= 0) { set_error("sum_f32: bad arguments"); return PTRB200_ERR_INVALID; }
    PTRB200_LAUNCH(sum_kernel, 1, 256, 0, stream, x, out, n);
    return check_launch("sum_f32");
}

int ptrb200_ndcg_at_ks(const float* scores, const float* labels, const int32_t* offsets, const int32_t* ks_host, int nks,
                       float* out, int32_t* order, int B, int n, int presort, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, out, ks_host, B, n);
    if (rc) return rc;
    if (nks <= 0 || nks > PTRB200_MAX_CUTOFFS) { set_error("ndcg_at_ks: nks=%d outside 1..%d", nks, PTRB200_MAX_CUTOFFS); return PTRB200_ERR_INVALID; }
    Cutoffs ks;
    ks.n = nks;
    for (int c = 0; c < nks; ++c) {
        ks.k[c] = ks_host[c];
        if (ks.k[c] <= 0 || (c > 0 && ks.k[c] < ks.k[c - 1])) { set_error("ndcg_at_ks: cutoffs must be positive and non-decreasing"); return PTRB200_ERR_INVALID; }
    }
    const int npow2 = next_pow2(n);
    const size_t smem = (size_t)npow2 * 8 + (size_t)n * 4 * 2;
    if ((rc = allow_smem(ndcg_at_ks_kernel, smem))) return rc;
    PTRB200_LAUNCH(ndcg_at_ks_kernel, B, block_threads(n), smem, stream, scores, labels, ks, out, order, offsets, n, npow2, presort);
    return check_launch("ndcg_at_ks");
}

int ptrb200_adhoc_metrics_at_ks(const float* scores, const float* labels, const int32_t* offsets, const int32_t* ks_host, int nks,
                                float* out, int B, int n, int presort, float max_label, ptrb200_stream_t stream) {
    int rc = check_list_args(scores, labels, out, ks_host, B, n);
    if (rc) return rc;
    if (nks <= 0 || nks > PTRB200_MAX_CUTOFFS) { set_error("adhoc_metrics: nks=%d outside 1..%d", nks, PTRB200_MAX_CUTOFFS); return PTRB200_ERR_INVALID; }
    Cutoffs ks;
    ks.n = nks;
    for (int c = 0; c < nks; ++c) {
        ks.k[c] = ks_host[c];
        if (ks.k[c] <= 0 || (c > 0 && ks.k[c] < ks.k[c - 1])) { set_error("adhoc_metrics: cutoffs must be positive and non-decreasing"); return PTRB200_ERR_INVALID; }
    }
    const int npow2 = next_pow2(n);
    const size_t smem = (size_t)npow2 * 8 + (size_t)n * 4 * 2;
    if ((rc = allow_smem(adhoc_metrics_kernel, smem))) return rc;
    int threads = block_threads(n); if (threads < 128) threads = 128;
    PTRB200_LAUNCH(adhoc_metrics_kernel, B, threads, smem, stream, scores, labels, ks, out, offsets, n, npow2, presort, max_label);
    return check_launch("adhoc_metrics_at_ks");
}

}  // extern "C"
