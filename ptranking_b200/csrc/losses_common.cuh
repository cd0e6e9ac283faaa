// losses_common.cuh -- helpers shared by the per-list kernels (losses.cu, losses_ext.cu, wassrank.cu, diversity.cu): list
// addressing for uniform and ragged batches, iDCG, the robust sigmoid, metric cutoffs, block scans, host-side launch checks.
#pragma once
#include "common.cuh"

namespace ptrb200 {

typedef unsigned long long u64;

static __device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// One query's slice of the flat [total_docs] score / label / gradient arrays.  Uniform batches ([B,n] dense, the
// reference's contract: data_utils.py:683-718) pass offsets == NULL; ragged batches pass the B+1 prefix offsets
// (SURVEY 8f-2: variable-length lists inside one launch) and `n_uniform` then only bounds the shared-memory carve-up.
struct ListSpan { size_t base; int n; };
static __device__ __forceinline__ ListSpan list_span(const int32_t* __restrict__ offsets, int b, int n_uniform) {
    ListSpan s;
    if (offsets) { const int o = offsets[b]; s.base = (size_t)o; s.n = offsets[b + 1] - o; }
    else { s.base = (size_t)b * (size_t)n_uniform; s.n = n_uniform; }
    return s;
}

// iDCG of one query: labels as given when presorted, else labels sorted descending
// (torch_dcg_at_k over the whole list, metric/adhoc/adhoc_metric.py:197-217).
// `keys` is scratch for npow2 sort keys.  Every thread returns the value.
static __device__ float block_idcg(const float* __restrict__ y, int n, int npow2, bool presort,
                                   u64* keys, float* red) {
    float part = 0.0f;
    if (presort) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) part += gain_of(y[i]) / log2_rank(i);
    } else {
        for (int i = threadIdx.x; i < npow2; i += blockDim.x) keys[i] = i < n ? desc_key(y[i], i) : 0ull;
        block_sort_desc(keys, npow2);
        for (int r = threadIdx.x; r < n; r += blockDim.x) part += gain_of(y[key_index(keys[r])]) / log2_rank(r);
    }
    return block_sum(part, red);
}

// Robust_Sigmoid forward, base/utils.py:62-78 (branch on the sign of the unscaled input)
static __device__ __forceinline__ float robust_sigmoid(float in, float alpha) {
    const float x = alpha * in;
    if (in > 0.0f) return __fdividef(1.0f, 1.0f + expf(-x));
    if (in < 0.0f) { const float ex = expf(x); return __fdividef(ex, 1.0f + ex); }
    return 0.5f;
}

// metric cutoffs, ascending, passed by value to the metric kernels
struct Cutoffs { int k[PTRB200_MAX_CUTOFFS]; int n; };

// ---------------------------------------------------------------------------
// block-wide inclusive scan over a shared-memory array (forward or reverse)
// ---------------------------------------------------------------------------
template <bool REVERSE>
static __device__ void block_scan_inclusive(float* a, int n, float* red /* >= 66 floats */) {
    const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = (T + 31) >> 5;
    const int C = (n + T - 1) / T;
    const int c0 = min(tid * C, n), c1 = min(c0 + C, n);
    float run = 0.0f;
    for (int i = c0; i < c1; ++i) {
        const int p = REVERSE ? n - 1 - i : i;
        run += a[p];
        a[p] = run;
    }
    float inc = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) red[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        float v = lane < nw ? red[lane] : 0.0f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += t;
        }
        red[33 + lane] = v;   // inclusive over warps
    }
    __syncthreads();
    const float offset = (inc - run) + (warp > 0 ? red[33 + warp - 1] : 0.0f);
    for (int i = c0; i < c1; ++i) {
        const int p = REVERSE ? n - 1 - i : i;
        a[p] += offset;
    }
    __syncthreads();
}

// Block-wide exclusive scan; every thread gets its prefix and *total.  `red` = 64 elements of shared memory.
template <typename T>
static __device__ __forceinline__ T block_exclusive_scan(T v, T* red, T* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    __syncthreads();
    if (lane == 31) red[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        T s = lane < nw ? red[lane] : T(0);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
        red[32 + lane] = s;
    }
    __syncthreads();
    *total = red[32 + nw - 1];
    return inc - v + (warp ? red[32 + warp - 1] : T(0));
}

// ---------------------------------------------------------------------------
// host-side launch helpers
// ---------------------------------------------------------------------------
static inline int block_threads(int n) {
    int t = ((n + 31) / 32) * 32;
    return t < 32 ? 32 : (t > 1024 ? 1024 : t);
}
static inline int check_list_args(const void* a, const void* b, const void* c, const void* d, int B, int n) {
    if (!a || !b || !c || !d || B <= 0 || n <= 0) { set_error("null pointer or non-positive size (B=%d n=%d)", B, n); return PTRB200_ERR_INVALID; }
    if (n > PTRB200_MAX_LIST_LEN) { set_error("list length %d exceeds PTRB200_MAX_LIST_LEN=%d", n, PTRB200_MAX_LIST_LEN); return PTRB200_ERR_UNSUPPORTED; }
    return PTRB200_OK;
}
template <typename K>
static inline int allow_smem(K kernel, size_t bytes) {
    if (bytes > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu): %s", bytes, cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
    }
    return PTRB200_OK;
}


static inline int check_rele_args(const char* who, const void* rele, const void* rele_offsets, const void* sub_counts, int m) {
    if (!rele || !rele_offsets || !sub_counts || m <= 0) {
        set_error("%s: null subtopic relevance arguments or non-positive m=%d", who, m);
        return PTRB200_ERR_INVALID;
    }
    if (m > PTRB200_MAX_SUBTOPICS) {
        set_error("%s: %d subtopics exceed PTRB200_MAX_SUBTOPICS=%d", who, m, PTRB200_MAX_SUBTOPICS);
        return PTRB200_ERR_UNSUPPORTED;
    }
    return PTRB200_OK;
}

}  // namespace ptrb200
