// div_rerank.cu -- rerank mode of the diversification driver: the first stage's top-k selection of every query of a
// split and the gather of the selected pools (RerankDIVDataset, ltr_diversification/util/div_data.py:130-192).
//
// The reference selects per query on the host: div_predict, a device-to-host copy, torch.sort(descending=True), the
// first rerank_k indices, re-sorted ascending.  Here one launch sequence selects for the whole split:
//   rerank_count_scan_kernel  one CTA: sel_counts[q] = min(n_q, rerank_k) and their exclusive scan sel_offsets
//   rerank_select_kernel      one CTA per query: (key, index) pairs sorted in shared memory, the first rerank_k marked,
//                             then compacted in index order by a block scan (a query with n_q <= rerank_k keeps all)
//   rerank_rele_scan_kernel   one CTA: offsets of the gathered [m_q, c_q] relevance blocks
//   rerank_gather_kernel      one CTA row per query: the selected document rows and relevance columns, plain copies
#include "losses_common.cuh"

namespace ptrb200 {

constexpr int RR_SELECT_THREADS = 256;
constexpr int RR_SCAN_THREADS = 1024;
constexpr int RR_GATHER_THREADS = 256, RR_GATHER_Y = 4;

__global__ void __launch_bounds__(RR_SCAN_THREADS)
rerank_count_scan_kernel(const int32_t* __restrict__ offsets, int B, int k, int32_t* __restrict__ counts,
                         int32_t* __restrict__ sel_offsets) {
    __shared__ int32_t red[64];
    int32_t carry = 0;
    for (int q0 = 0; q0 < B; q0 += blockDim.x) {
        const int q = q0 + threadIdx.x;
        const int32_t c = q < B ? max(0, min(offsets[q + 1] - offsets[q], k)) : 0;
        int32_t tot;
        const int32_t ex = block_exclusive_scan(c, red, &tot);
        if (q < B) { counts[q] = c; sel_offsets[q] = carry + ex; }
        carry += tot;
    }
    if (threadIdx.x == 0) sel_offsets[B] = carry;
}

__global__ void __launch_bounds__(RR_SCAN_THREADS)
rerank_rele_scan_kernel(const int32_t* __restrict__ sel_offsets, const int32_t* __restrict__ sub_counts, int B,
                        int64_t* __restrict__ out) {
    __shared__ int64_t red[64];
    int64_t carry = 0;
    for (int q0 = 0; q0 < B; q0 += blockDim.x) {
        const int q = q0 + threadIdx.x;
        const int64_t c = q < B ? (int64_t)sub_counts[q] * (int64_t)(sel_offsets[q + 1] - sel_offsets[q]) : 0;
        int64_t tot;
        const int64_t ex = block_exclusive_scan(c, red, &tot);
        if (q < B) out[q] = carry + ex;
        carry += tot;
    }
}

// Query b's winners: the first k entries of its rows sorted by desc_key (key descending, NaN first, index ascending),
// marked in win[] and written out in index order.  Shared memory: next_pow2(max_len) sort keys + one byte per row.
__global__ void __launch_bounds__(RR_SELECT_THREADS)
rerank_select_kernel(const float* __restrict__ keys, const int32_t* __restrict__ offsets,
                     const int32_t* __restrict__ sel_offsets, int32_t* __restrict__ sel_idx, int max_len, int k) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ int32_t red[64];
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int base = offsets[b];
    const int n = min(offsets[b + 1] - base, max_len);
    int32_t* out = sel_idx + sel_offsets[b];
    if (n <= k) {
        for (int i = tid; i < n; i += nt) out[i] = i;
        return;
    }
    const int npow2 = next_pow2(n);
    u64* sk = reinterpret_cast<u64*>(smem_raw);
    unsigned char* win = smem_raw + (size_t)npow2 * 8;
    for (int i = tid; i < npow2; i += nt) sk[i] = i < n ? desc_key(keys[base + i], i) : 0ull;   // real keys are > 0
    for (int i = tid; i < n; i += nt) win[i] = 0;
    block_sort_desc(sk, npow2);
    for (int i = tid; i < k; i += nt) win[key_index(sk[i])] = 1;
    __syncthreads();
    const int per = (n + nt - 1) / nt;
    const int r0 = min(tid * per, n), r1 = min(r0 + per, n);
    int32_t c = 0;
    for (int r = r0; r < r1; ++r) c += win[r];
    int32_t tot;
    int32_t pos = block_exclusive_scan(c, red, &tot);
    for (int r = r0; r < r1; ++r)
        if (win[r]) out[pos++] = r;
}

__global__ void __launch_bounds__(RR_GATHER_THREADS)
rerank_gather_kernel(const float* __restrict__ docs, int F, const int32_t* __restrict__ offsets,
                     const int32_t* __restrict__ sel_offsets, const int32_t* __restrict__ sel_idx,
                     const float* __restrict__ rele, const int64_t* __restrict__ rele_offsets,
                     const int32_t* __restrict__ sub_counts, float* __restrict__ docs_out, float* __restrict__ rele_out,
                     const int64_t* __restrict__ rele_offsets_out) {
    const int b = blockIdx.x;
    const int s0 = sel_offsets[b], c = sel_offsets[b + 1] - s0;
    const int base = offsets[b], n = offsets[b + 1] - base;
    const int32_t* idx = sel_idx + s0;
    const size_t step = (size_t)gridDim.y * blockDim.x, first = (size_t)blockIdx.y * blockDim.x + threadIdx.x;
    for (size_t e = first; e < (size_t)c * F; e += step) {
        const size_t j = e / F, f = e % F;
        docs_out[(s0 + j) * F + f] = docs[((size_t)base + idx[j]) * F + f];
    }
    const float* src = rele + rele_offsets[b];
    float* dst = rele_out + rele_offsets_out[b];
    for (size_t e = first; e < (size_t)sub_counts[b] * c; e += step) {
        const size_t r = e / c, j = e % c;
        dst[e] = src[r * n + idx[j]];
    }
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

int ptrb200_div_rerank_select(const float* keys, const int32_t* offsets, int B, int max_len, int rerank_k,
                              int32_t* sel_counts, int32_t* sel_offsets, int32_t* sel_idx, int32_t* total_host,
                              ptrb200_stream_t stream) {
    if (!keys || !offsets || !sel_counts || !sel_offsets || !sel_idx || B <= 0 || max_len <= 0) {
        set_error("div_rerank_select: null pointer or non-positive size (B=%d max_len=%d)", B, max_len);
        return PTRB200_ERR_INVALID;
    }
    if (rerank_k < 1) { set_error("div_rerank_select: rerank_k=%d must be >= 1", rerank_k); return PTRB200_ERR_INVALID; }
    if (max_len > PTRB200_MAX_LIST_LEN) {
        set_error("div_rerank_select: list length %d exceeds PTRB200_MAX_LIST_LEN=%d", max_len, PTRB200_MAX_LIST_LEN);
        return PTRB200_ERR_UNSUPPORTED;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    PTRB200_LAUNCH(rerank_count_scan_kernel, 1, RR_SCAN_THREADS, 0, st, offsets, B, rerank_k, sel_counts, sel_offsets);
    const size_t smem = (size_t)next_pow2(max_len) * 9;
    int rc = allow_smem(rerank_select_kernel, smem);
    if (rc) return rc;
    PTRB200_LAUNCH(rerank_select_kernel, B, RR_SELECT_THREADS, smem, st, keys, offsets, sel_offsets, sel_idx, max_len,
                   rerank_k);
    if ((rc = check_launch("div_rerank_select"))) return rc;
    if (total_host) {
        if (cudaMemcpyAsync(total_host, sel_offsets + B, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            return check_launch("div_rerank_select");
    }
    return PTRB200_OK;
}

int ptrb200_div_rerank_gather(const float* docs, int F, const int32_t* offsets, const int32_t* sel_offsets,
                              const int32_t* sel_idx, int B, const float* rele, const int64_t* rele_offsets,
                              const int32_t* sub_counts, float* docs_out, float* rele_out, int64_t* rele_offsets_out,
                              ptrb200_stream_t stream) {
    if (!docs || !offsets || !sel_offsets || !sel_idx || !rele || !rele_offsets || !sub_counts || !docs_out ||
        !rele_out || !rele_offsets_out || B <= 0 || F <= 0) {
        set_error("div_rerank_gather: null pointer or non-positive size (B=%d F=%d)", B, F);
        return PTRB200_ERR_INVALID;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    PTRB200_LAUNCH(rerank_rele_scan_kernel, 1, RR_SCAN_THREADS, 0, st, sel_offsets, sub_counts, B, rele_offsets_out);
    PTRB200_LAUNCH(rerank_gather_kernel, dim3(B, RR_GATHER_Y), RR_GATHER_THREADS, 0, st, docs, F, offsets, sel_offsets,
                   sel_idx, rele, rele_offsets, sub_counts, docs_out, rele_out, rele_offsets_out);
    return check_launch("div_rerank_gather");
}

}  // extern "C"
