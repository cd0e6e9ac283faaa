// common.cuh -- shared device helpers for the sm_90a kernels of libptranking_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <string.h>

#include "../../include/ptranking_b200.h"

namespace ptrb200 {

// ---- host-side bookkeeping (capi.cu owns the storage) ----------------------
void set_error(const char* fmt, ...);
void count_launch();
int check_launch(const char* what);   // cudaGetLastError -> PTRB200_* code

// per-launch CUDA-event timing (off by default; bench.py's roofline pass switches it on)
bool timing_enabled();
void timing_before(const char* tag, cudaStream_t st);
void timing_after(cudaStream_t st);

// streaming multiprocessors of the current device (persistent grids launch one CTA per SM, grid-stride loops cap at a
// multiple of it)
static inline int num_sms() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    }
    return sms;
}

#define PTRB200_LAUNCH(kernel, grid, block, smem, stream, ...) \
    PTRB200_LAUNCH_TAG(#kernel, kernel, grid, block, smem, stream, __VA_ARGS__)

#define PTRB200_LAUNCH_TAG(tag, kernel, grid, block, smem, stream, ...)               \
    do {                                                                              \
        const bool _tm = ::ptrb200::timing_enabled();                                 \
        if (_tm) ::ptrb200::timing_before(tag, (cudaStream_t)(stream));               \
        kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);     \
        if (_tm) ::ptrb200::timing_after((cudaStream_t)(stream));                     \
        ::ptrb200::count_launch();                                                    \
    } while (0)

// ---- math ------------------------------------------------------------------
__device__ __forceinline__ float gain_of(float label) { return exp2f(label) - 1.0f; }       // 2^l - 1
__device__ __forceinline__ float log2_rank(int r) { return log2f((float)r + 2.0f); }        // D(r)

// sigmoid exactly as ATen evaluates it in fp32: 1 / (1 + exp(-x))
__device__ __forceinline__ float sigmoid_aten(float x) { return __fdividef(1.0f, 1.0f + expf(-x)); }

// ---- reductions --------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// Block-wide sum; every thread gets the result.  `red` = 33 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = lane < nw ? red[lane] : 0.0f;
        t = warp_sum(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}
__device__ __forceinline__ float block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = lane < nw ? red[lane] : -INFINITY;
        t = warp_max(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}

// ---- per-list sort -----------------------------------------------------------
// 64-bit key whose DESCENDING order is (score descending, NaN first, doc index ascending):
// the total order torch.sort(descending=True) produces with a stable sort.
__device__ __forceinline__ unsigned long long desc_key(float s, int idx) {
    unsigned u = __float_as_uint(s + 0.0f);               // -0 -> +0
    if (s != s) u = 0x7fffffffu;                          // NaN sorts above +inf
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)idx);
}
__device__ __forceinline__ int key_index(unsigned long long k) { return (int)(0xffffffffu - (unsigned)(k & 0xffffffffull)); }

// In-place bitonic sort of keys[0..npow2) in shared memory, descending.  Pad with 0.
__device__ __forceinline__ void block_sort_desc(unsigned long long* keys, int npow2) {
    for (int k = 2; k <= npow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (npow2 >> 1); t += blockDim.x) {
                const int lo = ((t / j) * (j << 1)) + (t % j);
                const int hi = lo + j;
                const bool desc = ((lo & k) == 0);
                const unsigned long long a = keys[lo], b = keys[hi];
                if (desc ? (a < b) : (a > b)) { keys[lo] = b; keys[hi] = a; }
            }
        }
    }
    __syncthreads();
}

__host__ __device__ __forceinline__ int next_pow2(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

// ---- Philox4x32-10 (counter-based RNG for dropout masks and tie shuffles) -----
struct Philox {
    uint32_t k0, k1;
    __host__ __device__ Philox(uint64_t seed) : k0((uint32_t)seed), k1((uint32_t)(seed >> 32)) {}
    __host__ __device__ static inline void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#ifdef __CUDA_ARCH__
        hi = __umulhi(a, b);
        lo = a * b;
#else
        uint64_t p = (uint64_t)a * b;
        hi = (uint32_t)(p >> 32);
        lo = (uint32_t)p;
#endif
    }
    __host__ __device__ inline uint4 operator()(uint64_t ctr_lo, uint64_t ctr_hi) const {
        uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
        uint32_t a = k0, b = k1;
#pragma unroll
        for (int r = 0; r < 10; ++r) {
            uint32_t h0, l0, h1, l1;
            mulhilo(0xD2511F53u, c0, h0, l0);
            mulhilo(0xCD9E8D57u, c2, h1, l1);
            c0 = h1 ^ c1 ^ a; c1 = l1; c2 = h0 ^ c3 ^ b; c3 = l0;
            a += 0x9E3779B9u; b += 0xBB67AE85u;
        }
        return make_uint4(c0, c1, c2, c3);
    }
};
// keep-mask of Dropout(p) for element `elem` of stream `offset`: true = kept.
__host__ __device__ __forceinline__ uint32_t dropout_bits(uint64_t seed, uint64_t offset, uint64_t elem) {
    Philox ph(seed);
    uint4 r = ph(elem >> 2, offset);
    const uint32_t lane = (uint32_t)(elem & 3);
    return lane == 0 ? r.x : lane == 1 ? r.y : lane == 2 ? r.z : r.w;
}

// ---- dropout masks: splitmix64 counter stream, 16 random bits per element ---------------------------
// One 64-bit draw covers 4 consecutive elements (element e uses bits [16*(e&3), 16*(e&3)+16) of draw e>>2);
// an element is KEPT when its 16-bit value >= thr = round(p * 65536) and then scaled by 65536 / (65536 - thr).
// The mask of an element depends only on (key, element index), so forward, backward and every kernel variant
// regenerate identical masks.  Keys: dropout_key(seed, index) with
//   index = o*64 + l   the input of Linear layer l of a stacked-FF call at offset o (make_drop), element
//                      row * d_in(l) + col of the unpadded layer input;
//   index = o*64 + 63  a call at offset o that draws a single mask: elementwise dropout, attention (make_drop_call).
// Both kinds take o from the same counter (ops.next_dropout_offset); the FF net's layer slots stay below 63, so
// no two calls share a stream.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}
__host__ __device__ __forceinline__ uint64_t dropout_key(uint64_t seed, uint64_t offset) {
    return mix64(seed + 0x9e3779b97f4a7c15ull * (offset + 1));
}
__host__ __device__ __forceinline__ uint64_t dropout_draw4(uint64_t key, uint64_t quad) {
    return mix64(key + 0x9e3779b97f4a7c15ull * quad);
}
__host__ __device__ __forceinline__ bool dropout_keep(uint64_t key, uint64_t elem, uint32_t thr) {
    return (uint32_t)((dropout_draw4(key, elem >> 2) >> (16 * (elem & 3))) & 0xffffu) >= thr;
}
struct DropCfg { uint32_t thr; float scale; uint64_t key; };      // thr == 0: dropout off
static inline DropCfg make_drop(float p, uint64_t seed, uint64_t offset) {
    DropCfg d;
    d.thr = p > 0.0f ? (uint32_t)(p * 65536.0f + 0.5f) : 0u;
    d.scale = d.thr ? 65536.0f / (float)(65536u - d.thr) : 1.0f;
    d.key = dropout_key(seed, offset);
    return d;
}
static_assert(PTRB200_MAX_FF_LAYERS < 63, "the FF net's per-layer key slots must stay below the one-mask slot 63");
static inline DropCfg make_drop_call(float p, uint64_t seed, uint64_t offset) {
    return make_drop(p, seed, offset * 64 + 63);
}

}  // namespace ptrb200
