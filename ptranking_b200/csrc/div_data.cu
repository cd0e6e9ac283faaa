// div_data.cu -- the plain splits of the diversification driver (DIVDataset, ltr_diversification/util/div_data.py:53-127)
// built on the device: every query's greedy ideal alpha-DCG order (get_div_ideal_ranking,
// metric/srd/diversity_metric.py:113-141) and the split's packed rows and subtopic relevance blocks (to_matrix, :30-50).
//
//   div_ideal_order_kernel  one CTA per query: per-candidate gains (float64) and the 20 cover counts in shared memory,
//                           one block argmax per placed document; once no unplaced gain is positive the rest follow in
//                           pool order (a block scan compacts them)
//   div_pack_kernel         one CTA row per query: q rows, doc rows in ideal order (optionally + Gaussian noise) and the
//                           [m_q, n_q] relevance block, every element computed independently (no zero pass)
#include "losses_common.cuh"

namespace ptrb200 {

constexpr int DIV_ORDER_THREADS = 256;
constexpr int DIV_PACK_THREADS = 256, DIV_PACK_Y = 4;
constexpr int DIV_SUBTOPICS = 20;          // the reference's np.zeros(20) cover counts and rele_mat rows

// (gain, position) of the better candidate: larger gain, then lower pool position.
static __device__ __forceinline__ void better_of(double& g, int& i, double og, int oi) {
    if (og > g || (og == g && oi < i)) { g = og; i = oi; }
}

// Gain of pool position d: sum over its subtopic entries s, in their given order, of pw[cnt[s-1]].  The sum order and
// the power table make it the reference's float64 value bit for bit.
static __device__ __forceinline__ double doc_gain(const int32_t* __restrict__ sub_ids, int e0, int e1,
                                                  const int* cnt, const double* __restrict__ pw) {
    double g = 0.0;
    for (int e = e0; e < e1; ++e) {
        const int s = sub_ids[e];
        if (s >= 1 && s <= DIV_SUBTOPICS) g += pw[cnt[s - 1]];
    }
    return g;
}

// Shared memory: double gain[max_len] (placed: -1) + uint32 subtopic bit mask[max_len].
__global__ void __launch_bounds__(DIV_ORDER_THREADS)
div_ideal_order_kernel(const int32_t* __restrict__ offsets, const int32_t* __restrict__ sub_offsets,
                       const int32_t* __restrict__ sub_ids, const double* __restrict__ pw, int32_t* __restrict__ order,
                       int max_len) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ int cnt[DIV_SUBTOPICS];
    __shared__ double red_g[32];
    __shared__ int red_i[32];
    __shared__ int32_t scan_red[64];
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int base = offsets[b];
    const int n = min(offsets[b + 1] - base, max_len);
    double* gain = reinterpret_cast<double*>(smem_raw);
    uint32_t* mask = reinterpret_cast<uint32_t*>(gain + max_len);
    const int32_t* so = sub_offsets + base;
    int32_t* out = order + base;
    if (tid < DIV_SUBTOPICS) cnt[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += nt) {
        uint32_t m = 0;
        for (int e = so[i]; e < so[i + 1]; ++e) {
            const int s = sub_ids[e];
            if (s >= 1 && s <= DIV_SUBTOPICS) m |= 1u << (s - 1);
        }
        mask[i] = m;
        gain[i] = doc_gain(sub_ids, so[i], so[i + 1], cnt, pw);
    }
    __syncthreads();
    int j = 0;
    for (; j < n; ++j) {
        double g = -1.0;
        int best = n;
        for (int i = tid; i < n; i += nt) better_of(g, best, gain[i], i);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            better_of(g, best, __shfl_xor_sync(0xffffffffu, g, o), __shfl_xor_sync(0xffffffffu, best, o));
        if (lane == 0) { red_g[warp] = g; red_i[warp] = best; }
        __syncthreads();
        g = red_g[0]; best = red_i[0];
        for (int w = 1; w < nw; ++w) better_of(g, best, red_g[w], red_i[w]);
        if (!(g > 0.0)) break;                            // block-uniform: every thread reduced the same values
        const uint32_t hit = mask[best];
        if (tid == 0) {
            out[j] = best;
            gain[best] = -1.0;
            for (int e = so[best]; e < so[best + 1]; ++e) {
                const int s = sub_ids[e];
                if (s >= 1 && s <= DIV_SUBTOPICS) ++cnt[s - 1];
            }
        }
        __syncthreads();
        for (int i = tid; i < n; i += nt)
            if ((mask[i] & hit) && gain[i] >= 0.0) gain[i] = doc_gain(sub_ids, so[i], so[i + 1], cnt, pw);
        __syncthreads();
    }
    if (j == n) return;
    // every unplaced gain is 0: the rest in pool order
    const int per = (n + nt - 1) / nt;
    const int r0 = min(tid * per, n), r1 = min(r0 + per, n);
    int32_t c = 0;
    for (int r = r0; r < r1; ++r) c += gain[r] >= 0.0;
    int32_t tot;
    int32_t pos = j + block_exclusive_scan(c, scan_red, &tot);
    for (int r = r0; r < r1; ++r)
        if (gain[r] >= 0.0) out[pos++] = r;
}

// Standard normal draw for element `elem` of noise stream `stream`: Box-Muller on one Philox4x32-10 output.
static __device__ __forceinline__ float div_normal(uint64_t seed, uint64_t stream, uint64_t elem) {
    const uint4 r = Philox(seed)(elem, stream);
    const float u1 = (float)((r.x >> 8) + 1u) * 0x1.0p-24f;      // (0, 1]
    const float u2 = (float)(r.y >> 8) * 0x1.0p-24f;             // [0, 1)
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

__global__ void __launch_bounds__(DIV_PACK_THREADS)
div_pack_kernel(const float* __restrict__ table, int F, const float* __restrict__ q_src,
                const int32_t* __restrict__ offsets, const int32_t* __restrict__ rows,
                const int32_t* __restrict__ order, const int32_t* __restrict__ sub_offsets,
                const int32_t* __restrict__ sub_ids, const int64_t* __restrict__ rele_offsets,
                const int32_t* __restrict__ sub_counts, float std_delta, uint64_t seed, float* __restrict__ q_out,
                float* __restrict__ docs_out, float* __restrict__ rele_out) {
    const int b = blockIdx.x;
    const int base = offsets[b], n = offsets[b + 1] - base;
    const int32_t* ord = order + base;
    const size_t step = (size_t)gridDim.y * blockDim.x, first = (size_t)blockIdx.y * blockDim.x + threadIdx.x;
    const bool noise = std_delta > 0.0f;
    for (size_t f = first; f < (size_t)F; f += step) {
        const size_t e = (size_t)b * F + f;
        q_out[e] = noise ? q_src[e] + std_delta * div_normal(seed, 0, e) : q_src[e];
    }
    for (size_t e = first; e < (size_t)n * F; e += step) {
        const size_t j = e / F, f = e % F;
        const size_t o = (size_t)base * F + e;
        const float v = table[(size_t)rows[base + ord[j]] * F + f];
        docs_out[o] = noise ? v + std_delta * div_normal(seed, 1, o) : v;
    }
    const int m = sub_counts[b];
    float* R = rele_out + rele_offsets[b];
    for (size_t e = first; e < (size_t)m * n; e += step) {
        const int s = (int)(e / n) + 1, d = base + ord[e % n];
        float v = 0.0f;
        for (int k = sub_offsets[d]; k < sub_offsets[d + 1]; ++k) v = sub_ids[k] == s ? 1.0f : v;
        R[e] = v;
    }
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_div_ideal_order(const int32_t* offsets, const int32_t* sub_offsets, const int32_t* sub_ids,
                            const double* pw, int B, int max_len, int32_t* order, ptrb200_stream_t stream) {
    if (!offsets || !sub_offsets || !sub_ids || !pw || !order || B <= 0 || max_len <= 0) {
        set_error("div_ideal_order: null pointer or non-positive size (B=%d max_len=%d)", B, max_len);
        return PTRB200_ERR_INVALID;
    }
    if (max_len > PTRB200_MAX_LIST_LEN) {
        set_error("div_ideal_order: list length %d exceeds PTRB200_MAX_LIST_LEN=%d", max_len, PTRB200_MAX_LIST_LEN);
        return PTRB200_ERR_UNSUPPORTED;
    }
    const size_t smem = (size_t)max_len * (sizeof(double) + sizeof(uint32_t));
    // the opt-in covers dynamic plus static shared memory (about 0.7 KB): 4096 documents need 48 KB + static
    int rc = allow_smem(div_ideal_order_kernel, smem + 1024);
    if (rc) return rc;
    PTRB200_LAUNCH(div_ideal_order_kernel, B, DIV_ORDER_THREADS, smem, (cudaStream_t)stream, offsets, sub_offsets,
                   sub_ids, pw, order, max_len);
    return check_launch("div_ideal_order");
}

int ptrb200_div_pack_split(const float* table, int F, const float* q_src, const int32_t* offsets, const int32_t* rows,
                           const int32_t* order, const int32_t* sub_offsets, const int32_t* sub_ids,
                           const int64_t* rele_offsets, const int32_t* sub_counts, int B, float std_delta,
                           uint64_t seed, float* q_out, float* docs_out, float* rele_out, ptrb200_stream_t stream) {
    if (!table || !q_src || !offsets || !rows || !order || !sub_offsets || !sub_ids || !rele_offsets || !sub_counts ||
        !q_out || !docs_out || !rele_out || B <= 0 || F <= 0) {
        set_error("div_pack_split: null pointer or non-positive size (B=%d F=%d)", B, F);
        return PTRB200_ERR_INVALID;
    }
    if (!(std_delta >= 0.0f) || isinf(std_delta)) {
        set_error("div_pack_split: std_delta=%g must be finite and >= 0", (double)std_delta);
        return PTRB200_ERR_INVALID;
    }
    PTRB200_LAUNCH(div_pack_kernel, dim3(B, DIV_PACK_Y), DIV_PACK_THREADS, 0, (cudaStream_t)stream, table, F, q_src,
                   offsets, rows, order, sub_offsets, sub_ids, rele_offsets, sub_counts, std_delta, seed, q_out,
                   docs_out, rele_out);
    return check_launch("div_pack_split");
}

}  // extern "C"
