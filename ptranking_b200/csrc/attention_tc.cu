// attention_tc.cu -- multi-head self-attention with every contraction on wgmma tensor cores.
//
// MultiheadAttention.forward, ptranking/base/list_ranker.py:226-248:
//     S = Q K^T / sqrt(d)   ->   A = softmax(S)   ->   A_d = dropout(A)   ->   O = A_d V
// and its autograd.  "Materialised S" design: the six contractions of forward + backward
//     S = Q K^T,   O = A_d V,   dA_d = dO V^T,   dQ = dS K,   dK = dS^T Q,   dV = A_d^T dO
// all run through a batched, strided  C[z] = alpha * op(A[z]) * B[z]^T  kernel (tf32 wgmma, 3xTF32 split, fp32
// accumulation in registers); row softmax / softmax-backward are streaming SIMT kernels over the [n,n] score tensor.  A factor
// that enters a contraction transposed (V, K, Q, dO as [key|query, d]; dS and A_d as [query, key] for dK / dV) is read in
// place with coalesced loads and transposed on its way into shared memory (wgmma takes 32-bit operands K-major only), never
// transposed in HBM.  The [n,n] tensors live in HBM (n <= 1024 per list: 134 MB per layer at B=64, n=512, 2 heads).
// Two kernels implement the batched GEMM: bgemm_nt_tc_kernel takes any shape; bgemm_fast_kernel (every extent, pitch and
// base address a multiple of four floats -- the attention core's own shapes) has the operand layouts and the dropout view
// as template parameters, loads one K-chunk ahead and writes full-width tiles through shared memory; both produce the
// same bits.  The entry points take row pitches, so they read Q|K|V side by side from one projection output, and per-query
// key counts for padded ragged batches.
#include "common.cuh"
#include "tc.cuh"

namespace ptrb200 {

struct BGemmArgs {
    const float *A, *B;
    float* C;
    int M, N, K;                 // C[M,N] = alpha * A[M,K] * B[N,K]^T
    int lda, ldb, ldc;           // row pitches (floats)
    long long sAb, sAh, sBb, sBh, sCb, sCh;   // batch strides (floats) for z = b*H + h
    int H;
    float alpha;
    // optional dropout on A's elements: mode 1: element id = (z*M + row)*K + col ; mode 2 (A is a transposed view of
    // the attention matrix): id = (z*K + col)*M + row
    int drop_mode;
    DropCfg drop;
    // operand storage: 0 = K-major as written above (A[M,K], B[N,K] row-major); 1 = MN-major, the operand is stored
    // transposed ([K,M] resp. [K,N] row-major, pitch lda/ldb between k-rows) and transposed while it is staged, so a
    // transposed factor never has to be materialised in HBM.  drop_mode 2 goes with a_mn.
    int a_mn, b_mn;
};

constexpr int BG_THREADS = 256, BG_NT = 128;      // two warpgroups, 64 rows of the 128 x 128 tile each

// store 4 consecutive M (or N) elements of one k-row of an MN-major source into the K-major operand image
static __device__ __forceinline__ void store_mn4(unsigned char* buf, int r, int k, float4 v) {
    *reinterpret_cast<float*>(buf + tc::swz_elem(r, k)) = v.x;
    *reinterpret_cast<float*>(buf + tc::swz_elem(r + 1, k)) = v.y;
    *reinterpret_cast<float*>(buf + tc::swz_elem(r + 2, k)) = v.z;
    *reinterpret_cast<float*>(buf + tc::swz_elem(r + 3, k)) = v.w;
}
static __device__ __forceinline__ void store_op(unsigned char* buf, bool mn, uint32_t off_k, int r_mn, int k_mn, float4 v) {
    if (mn) store_mn4(buf, r_mn, k_mn, v);
    else *reinterpret_cast<float4*>(buf + off_k) = v;
}

// the four K-steps of one 32-column chunk (columns beyond K are staged as zeros): warpgroup wg multiplies A rows
// [64 wg, +64) by all NPc columns of B.  3xTF32: the small a_lo*b_hi + a_hi*b_lo terms accumulate apart from the main
// products (the epilogue adds them), so two thirds of the accumulate steps leave the main chain.
template <int NPc>
static __device__ __forceinline__ void bg_mma_chunk(float (&acc)[NPc / 2], float (&cor)[NPc / 2], const unsigned char* a_hi,
                                                    const unsigned char* b_hi, int wg) {
    const uint32_t a_s = tc::smem_u32(a_hi) + wg * 8192, b_s = tc::smem_u32(b_hi);
    const uint64_t ah = tc::smem_desc_sw128(a_s, 1024), al = tc::smem_desc_sw128(a_s + 16384, 1024);
    const uint64_t bh = tc::smem_desc_sw128(b_s, 1024), bl = tc::smem_desc_sw128(b_s + 16384, 1024);
    tc::wg_fence();
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        tc::mma_tf32<NPc>(cor, al + 2 * s, bh + 2 * s, 1u);
        tc::mma_tf32<NPc>(cor, ah + 2 * s, bl + 2 * s, 1u);
        tc::mma_tf32<NPc>(acc, ah + 2 * s, bh + 2 * s, 1u);
    }
    tc::wg_commit();
    tc::wg_wait<0>();                 // the same threads stage the next chunk
}

__global__ void __launch_bounds__(BG_THREADS) bgemm_nt_tc_kernel(BGemmArgs g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* a_hi = base;
    unsigned char* a_lo = a_hi + 16384;
    unsigned char* b_hi = a_lo + 16384;
    unsigned char* b_lo = b_hi + 16384;

    const int tid = threadIdx.x, wg = tid >> 7;
    const int z = blockIdx.z, zb = z / g.H, zh = z % g.H;
    const float* A = g.A + zb * g.sAb + zh * g.sAh;
    const float* B = g.B + zb * g.sBb + zh * g.sBh;
    float* C = g.C + zb * g.sCb + zh * g.sCh;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BG_NT;
    const int N = min(BG_NT, g.N - n0), NP = ((N + 15) / 16) * 16;
    const int K = g.K;
    const int nchunks = (K + 31) / 32;
    const bool vecA = (g.lda & 3) == 0 && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
    const bool vecB = (g.ldb & 3) == 0 && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);

    auto load4 = [&](const float* p, int k, bool vec) -> float4 {      // guarded 4-wide load at column k of a row
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k + 3 < K && vec) return __ldg(reinterpret_cast<const float4*>(p + k));
        if (k < K) v.x = p[k];
        if (k + 1 < K) v.y = p[k + 1];
        if (k + 2 < K) v.z = p[k + 2];
        if (k + 3 < K) v.w = p[k + 3];
        return v;
    };
    auto load4m = [&](const float* p, int c0, int lim, bool vec) -> float4 {   // guarded 4-wide load at column c0 (< lim) of a row
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 + 3 < lim && vec) return __ldg(reinterpret_cast<const float4*>(p + c0));
        if (c0 < lim) v.x = p[c0];
        if (c0 + 1 < lim) v.y = p[c0 + 1];
        if (c0 + 2 < lim) v.z = p[c0 + 2];
        if (c0 + 3 < lim) v.w = p[c0 + 3];
        return v;
    };
    tc::with_width(NP, [&](auto W) {
    constexpr int NPc = decltype(W)::value;
    float acc[NPc / 2], cor[NPc / 2];
#pragma unroll
    for (int e = 0; e < NPc / 2; ++e) { acc[e] = 0.0f; cor[e] = 0.0f; }
    for (int c = 0; c < nchunks; ++c) {
        const int k0 = c * 32;
        float4 av[4], bv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int u = tid + i * BG_THREADS, r = u >> 3, j = u & 7, k = k0 + j * 4;      // K-major: row r, 16-byte unit j
            const int kr = u >> 5, mu = (u & 31) * 4;                                       // MN-major: k-row kr, columns mu..mu+3
            if (g.a_mn) av[i] = (k0 + kr < K) ? load4m(A + (size_t)(k0 + kr) * g.lda, m0 + mu, g.M, vecA) : make_float4(0.f, 0.f, 0.f, 0.f);
            else av[i] = (m0 + r < g.M) ? load4(A + (size_t)(m0 + r) * g.lda, k, vecA) : make_float4(0.f, 0.f, 0.f, 0.f);
            if (g.b_mn) bv[i] = (k0 + kr < K) ? load4m(B + (size_t)(k0 + kr) * g.ldb, n0 + mu, n0 + N, vecB) : make_float4(0.f, 0.f, 0.f, 0.f);
            else bv[i] = (r < N) ? load4(B + (size_t)(n0 + r) * g.ldb, k, vecB) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (c > 0) __syncthreads();                           // both warpgroups' MMAs of chunk c-1 are done with the operand buffers
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int u = tid + i * BG_THREADS, r = u >> 3, j = u & 7, k = k0 + j * 4;
            const int kr = u >> 5, mu = (u & 31) * 4;
            const uint32_t off_k = tc::swz_offset(r, j);                                             // K-major slot
            float4 v = av[i];
            if (g.drop_mode && g.drop.thr) {
                float* e = &v.x;
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    // element ids follow the row-major order of the stored attention matrix in both views
                    const uint64_t id = g.a_mn ? ((uint64_t)z * K + (k0 + kr)) * g.M + (m0 + mu + t)
                                               : ((uint64_t)z * g.M + (m0 + r)) * K + (k + t);
                    e[t] = dropout_keep(g.drop.key, id, g.drop.thr) ? e[t] * g.drop.scale : 0.0f;      // (out-of-range elements are already 0)
                }
            }
            float4 h, l;
            tc::split_tf32_rn(v.x, h.x, l.x); tc::split_tf32_rn(v.y, h.y, l.y); tc::split_tf32_rn(v.z, h.z, l.z); tc::split_tf32_rn(v.w, h.w, l.w);
            store_op(a_hi, g.a_mn, off_k, mu, kr, h);
            store_op(a_lo, g.a_mn, off_k, mu, kr, l);
            const float4 w = bv[i];
            tc::split_tf32_rn(w.x, h.x, l.x); tc::split_tf32_rn(w.y, h.y, l.y); tc::split_tf32_rn(w.z, h.z, l.z); tc::split_tf32_rn(w.w, h.w, l.w);
            store_op(b_hi, g.b_mn, off_k, mu, kr, h);
            store_op(b_lo, g.b_mn, off_k, mu, kr, l);
        }
        tc::fence_proxy_async();
        __syncthreads();
        bg_mma_chunk<NPc>(acc, cor, a_hi, b_hi, wg);
    }
    {   // epilogue: registers -> C
        const bool vecC = (g.ldc & 3) == 0 && ((reinterpret_cast<uintptr_t>(C + n0) & 15) == 0);
#pragma unroll
        for (int e = 0; e < NPc / 2; e += 2) {
            const int row = m0 + wg * 64 + tc::acc_row(e), col = tc::acc_col(e);
            if (row >= g.M || col >= N) continue;
            const float v0 = (acc[e] + cor[e]) * g.alpha, v1 = (acc[e + 1] + cor[e + 1]) * g.alpha;
            float* p = C + (size_t)row * g.ldc + n0 + col;
            if (col + 1 < N && vecC) *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
            else { p[0] = v0; if (col + 1 < N) p[1] = v1; }
        }
    }
    });
}

// Alignment-specialised variant of the kernel above: same tiling, same accumulators, same results bit for bit (identical
// operand images and MMA order), but the operand layouts and the dropout view are template parameters and every pitch,
// extent and base address is a multiple of four floats (host-checked).  Row/column validity, global pointers, swizzled
// shared-memory offsets and the dropout counter of a thread's four 16-byte units are then chunk-invariant and leave the
// chunk loop; one 64-bit draw serves the four elements of a unit (the general kernel hashes per element because it
// cannot assume quad alignment); B units beyond the padded tile width are never touched.  The attention core's six
// contractions all qualify; odd shapes keep the general kernel.
template <int A_MN, int B_MN, int DROP>
__global__ void __launch_bounds__(BG_THREADS, 1) bgemm_fast_kernel(BGemmArgs g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* a_hi = base;
    unsigned char* a_lo = a_hi + 16384;
    unsigned char* b_hi = a_lo + 16384;
    unsigned char* b_lo = b_hi + 16384;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int z = blockIdx.z, zb = z / g.H, zh = z % g.H;
    const float* A = g.A + zb * g.sAb + zh * g.sAh;
    const float* B = g.B + zb * g.sBb + zh * g.sBh;
    float* C = g.C + zb * g.sCb + zh * g.sCh;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BG_NT;
    const int N = min(BG_NT, g.N - n0), NP = ((N + 15) / 16) * 16;
    const int K = g.K;
    const int nchunks = (K + 31) / 32;

    // ---- chunk-invariant geometry of this thread's units (unit index i = 0..3) ----
    const int jk = tid & 7, rk = tid >> 3;            // K-major: 16-byte unit jk of row rk + 32 i
    const int cm = (tid & 31) * 4, km = tid >> 5;     // MN-major: columns cm..cm+3 of k-row km + 8 i
    const float* pa; const float* pb;
    size_t sa, sb;                                    // pointer step per unit index
    uint32_t oa = 0, ob = 0;                          // K-major: swizzled offset of unit 0 (+4096 per unit index)
    uint32_t am = 0, bm = 0;                          // bit i: unit i lies inside the tile along M / N (bit 4+i: and is staged at all)
    if (A_MN) {
        pa = A + (size_t)km * g.lda + m0 + cm; sa = (size_t)8 * g.lda;
        am = (m0 + cm < g.M) ? 0xfu : 0u;
    } else {
        pa = A + (size_t)(m0 + rk) * g.lda + jk * 4; sa = (size_t)32 * g.lda;
        oa = tc::swz_offset(rk, jk);
#pragma unroll
        for (int i = 0; i < 4; ++i) am |= (m0 + rk + 32 * i < g.M) ? (1u << i) : 0u;
    }
    if (B_MN) {
        pb = B + (size_t)km * g.ldb + n0 + cm; sb = (size_t)8 * g.ldb;
        bm = (cm < N ? 0xfu : 0u) | (cm < NP ? 0xf0u : 0u);
    } else {
        pb = B + (size_t)(n0 + rk) * g.ldb + jk * 4; sb = (size_t)32 * g.ldb;
        ob = tc::swz_offset(rk, jk);
#pragma unroll
        for (int i = 0; i < 4; ++i) bm |= (rk + 32 * i < N ? (1u << i) : 0u) | (rk + 32 * i < NP ? (16u << i) : 0u);
    }
    // MN-major units are transposed into the K-major image: 4 elements (rows cm..cm+3) of k-row km + 8 i
    auto put = [&](unsigned char* buf, bool mn, uint32_t off, int i, float4 v) {
        if (mn) store_mn4(buf, cm, km + 8 * i, v);
        else *reinterpret_cast<float4*>(buf + off + i * 4096u) = v;
    };
    // dropout counter: key + GOLD * quad, quad = element id / 4 of the unit's first element (ids as in the general kernel)
    constexpr uint64_t GOLD = 0x9e3779b97f4a7c15ull;
    uint64_t dctr = 0, dstep_i = 0, dstep_c = 0;
    if (DROP == 1) {            // id = (z*M + row)*K + col ; unit step: 32 rows ; chunk step: 32 columns
        dctr = g.drop.key + GOLD * ((((uint64_t)z * g.M + (m0 + rk)) * K + jk * 4) >> 2);
        dstep_i = GOLD * (uint64_t)(8 * K); dstep_c = GOLD * 8ull;
    } else if (DROP == 2) {     // id = (z*K + krow)*M + col ; unit step: 8 k-rows ; chunk step: 32 k-rows
        dctr = g.drop.key + GOLD * ((((uint64_t)z * K + km) * g.M + (m0 + cm)) >> 2);
        dstep_i = GOLD * (uint64_t)(2 * g.M); dstep_c = GOLD * (uint64_t)(8 * g.M);
    }
    const bool drop_on = DROP != 0 && g.drop.thr != 0;
    const uint32_t thr = g.drop.thr; const float dscale = g.drop.scale;

    // global -> registers one chunk AHEAD: the loads of chunk c+1 are in flight while chunk c is split, stored, synchronised
    // and multiplied (a CTA has no other way to hide HBM latency: its chunks are strictly sequential)
    float4 nav[4], nbv[4];
    auto load_chunk = [&](int c) {
        const int k0 = c * 32;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const bool ka = A_MN ? (k0 + km + 8 * i < K) : (k0 + jk * 4 < K);
            const bool kb = B_MN ? (k0 + km + 8 * i < K) : (k0 + jk * 4 < K);
            nav[i] = (ka && ((am >> i) & 1u)) ? __ldg(reinterpret_cast<const float4*>(pa + i * sa)) : make_float4(0.f, 0.f, 0.f, 0.f);
            nbv[i] = (kb && ((bm >> i) & 1u)) ? __ldg(reinterpret_cast<const float4*>(pb + i * sb)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        pa += A_MN ? (size_t)32 * g.lda : 32; pb += B_MN ? (size_t)32 * g.ldb : 32;
    };
    load_chunk(0);
    tc::with_width(NP, [&](auto W) {
    constexpr int NPc = decltype(W)::value;
    float acc[NPc / 2], cor[NPc / 2];
#pragma unroll
    for (int e = 0; e < NPc / 2; ++e) { acc[e] = 0.0f; cor[e] = 0.0f; }
    for (int c = 0; c < nchunks; ++c) {
        const int k0 = c * 32;
        float4 av[4], bv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { av[i] = nav[i]; bv[i] = nbv[i]; }
        if (c + 1 < nchunks) load_chunk(c + 1);
        if (c > 0) __syncthreads();                           // both warpgroups' MMAs of chunk c-1 are done with the operand buffers
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float4 v = av[i];
            if (DROP != 0 && drop_on) {
                const uint64_t d = mix64(dctr + i * dstep_i);
                v.x = ((uint32_t)d & 0xffffu) >= thr ? v.x * dscale : 0.0f;
                v.y = ((uint32_t)(d >> 16) & 0xffffu) >= thr ? v.y * dscale : 0.0f;
                v.z = ((uint32_t)(d >> 32) & 0xffffu) >= thr ? v.z * dscale : 0.0f;
                v.w = (uint32_t)(d >> 48) >= thr ? v.w * dscale : 0.0f;
            }
            float4 h, l;
            tc::split_tf32_rn(v.x, h.x, l.x); tc::split_tf32_rn(v.y, h.y, l.y); tc::split_tf32_rn(v.z, h.z, l.z); tc::split_tf32_rn(v.w, h.w, l.w);
            put(a_hi, A_MN, oa, i, h);
            put(a_lo, A_MN, oa, i, l);
            if ((bm >> (4 + i)) & 1u) {
                const float4 w = bv[i];
                tc::split_tf32_rn(w.x, h.x, l.x); tc::split_tf32_rn(w.y, h.y, l.y); tc::split_tf32_rn(w.z, h.z, l.z); tc::split_tf32_rn(w.w, h.w, l.w);
                put(b_hi, B_MN, ob, i, h);
                put(b_lo, B_MN, ob, i, l);
            }
        }
        dctr += dstep_c;
        tc::fence_proxy_async();
        __syncthreads();
        bg_mma_chunk<NPc>(acc, cor, a_hi, b_hi, wg);
    }
    const float alpha = g.alpha;
    if (N == BG_NT) {
        // full 128-column tile (the [n,n] score / dP tensors: the 134 MB outputs of the attention core).  A thread's
        // accumulators are 2-column pieces of 2 rows, so the tile goes through shared memory (the operand buffers are free:
        // every MMA has completed) and leaves as whole 512-byte row segments, one row per warp instruction.
        constexpr int PITCH = BG_NT + 4;                  // floats
        float* tile = reinterpret_cast<float*>(base);     // [128][PITCH] = 67,584 B (operands 65,536 B + the slack the host adds)
        __syncthreads();                                  // every warpgroup's MMAs have completed
#pragma unroll
        for (int e = 0; e < NPc / 2; e += 2) {
            const int r = wg * 64 + tc::acc_row(e), col = tc::acc_col(e);
            *reinterpret_cast<float2*>(tile + r * PITCH + col) = make_float2((acc[e] + cor[e]) * alpha, (acc[e + 1] + cor[e + 1]) * alpha);
        }
        __syncthreads();
        const int rows_here = min(128, g.M - m0);
        for (int r = warp; r < rows_here; r += BG_THREADS / 32)
            *reinterpret_cast<float4*>(C + (size_t)(m0 + r) * g.ldc + n0 + lane * 4) = *reinterpret_cast<const float4*>(tile + r * PITCH + lane * 4);
    } else {   // narrow tile: direct stores; every extent is a multiple of 4
#pragma unroll
        for (int e = 0; e < NPc / 2; e += 2) {
            const int row = m0 + wg * 64 + tc::acc_row(e), col = tc::acc_col(e);
            if (row < g.M && col < N)
                *reinterpret_cast<float2*>(C + (size_t)row * g.ldc + n0 + col) =
                    make_float2((acc[e] + cor[e]) * alpha, (acc[e + 1] + cor[e + 1]) * alpha);
        }
    }
    });
}

// in-place row softmax over S[z][i][:] (one warp per row).
// key_lens (optional, [B]): only the first key_lens[b] keys of query b exist (a ragged batch padded to n); the others get
// probability exactly 0, so padded documents influence nothing (their own rows are never read back).
__global__ void softmax_rows_kernel(float* __restrict__ S, size_t rows, int n, const int32_t* __restrict__ key_lens,
                                    int rows_per_query) {
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float* s = S + row * n;
    const int nk = key_lens ? max(1, min(n, key_lens[row / (size_t)rows_per_query])) : n;
    float m = -INFINITY;
    for (int j = lane; j < nk; j += 32) m = fmaxf(m, s[j]);
    m = warp_max(m);
    float l = 0.0f;
    for (int j = lane; j < nk; j += 32) { const float e = expf(s[j] - m); s[j] = e; l += e; }
    l = warp_sum(l);
    const float inv = 1.0f / l;
    for (int j = lane; j < nk; j += 32) s[j] *= inv;
    for (int j = nk + lane; j < n; j += 32) s[j] = 0.0f;
}

// dS = A * (dA - sum_j A dA) * inv_scale in place over dAd, where dA = dropmask(dAd)  (one warp per row)
__global__ void softmax_bwd_rows_kernel(const float* __restrict__ P, float* __restrict__ dP, size_t rows, int n,
                                        float inv_scale, DropCfg drop) {
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* p = P + row * n;
    float* d = dP + row * n;
    float acc = 0.0f;
    for (int j = lane; j < n; j += 32) {
        float da = d[j];
        if (drop.thr) da = dropout_keep(drop.key, row * (uint64_t)n + j, drop.thr) ? da * drop.scale : 0.0f;
        d[j] = da;
        acc = fmaf(p[j], da, acc);
    }
    acc = warp_sum(acc);
    for (int j = lane; j < n; j += 32) d[j] = p[j] * (d[j] - acc) * inv_scale;
}

template <int A_MN, int B_MN, int DROP>
static int launch_bgemm_fast(const BGemmArgs& g, dim3 grid, size_t smem, cudaStream_t st, const char* tag) {
    const cudaError_t e = cudaFuncSetAttribute(bgemm_fast_kernel<A_MN, B_MN, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("bgemm smem attr: %s", cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
    PTRB200_LAUNCH_TAG(tag, (bgemm_fast_kernel<A_MN, B_MN, DROP>), grid, BG_THREADS, smem, st, g);
    return PTRB200_OK;
}

static bool bgemm_general_forced() {
    const char* e = getenv("PTRB200_BGEMM_GENERAL");      // read per launch: the parity test flips it inside one process
    return e && e[0] == '1';
}

static int launch_bgemm(BGemmArgs& g, int Z, cudaStream_t st, const char* tag) {
    const size_t smem = 1024 + 4 * 16384;
    dim3 grid((g.M + 127) / 128, (g.N + BG_NT - 1) / BG_NT, Z);
    // the alignment-specialised kernel: every pitch, stride, extent and base address a multiple of four floats
    const auto q4 = [](long long v) { return (v & 3) == 0; };
    const auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    const bool fast = !bgemm_general_forced() && q4(g.lda) && q4(g.ldb) && q4(g.ldc) && q4(g.M) && q4(g.N) && q4(g.K) &&
                      q4(g.sAb) && q4(g.sAh) && q4(g.sBb) && q4(g.sBh) && q4(g.sCb) && q4(g.sCh) && a16(g.A) && a16(g.B) && a16(g.C) &&
                      (g.drop_mode == 0 || (g.drop_mode == 1 && !g.a_mn) || (g.drop_mode == 2 && g.a_mn));
    if (fast) {
        const int drop = g.drop.thr ? g.drop_mode : 0;
        const size_t smem = 1024 + (size_t)128 * (BG_NT + 4) * 4;      // operands (64 KB) overlaid by the [128][132] output staging tile
#define PTRB200_BG_CASE(AM, BM, D) if (g.a_mn == AM && g.b_mn == BM && drop == D) return launch_bgemm_fast<AM, BM, D>(g, grid, smem, st, tag);
        // the attention core's shapes (list_ranker.py:226-248 forward + autograd)
        PTRB200_BG_CASE(0, 0, 0) PTRB200_BG_CASE(0, 1, 0) PTRB200_BG_CASE(0, 1, 1) PTRB200_BG_CASE(1, 1, 0) PTRB200_BG_CASE(1, 1, 2)
#undef PTRB200_BG_CASE
    }
    const cudaError_t e = cudaFuncSetAttribute(bgemm_nt_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("bgemm smem attr: %s", cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
    PTRB200_LAUNCH_TAG(tag, bgemm_nt_tc_kernel, grid, BG_THREADS, smem, st, g);
    return PTRB200_OK;
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" {

// the backward pass's scratch: dS[Z,n,n]
int64_t ptrb200_attention_tc_workspace_floats(int B, int n, int H) { return (int64_t)B * H * n * n; }

// P_out[B*H, n, n] receives the (un-dropped) attention probabilities and must be kept for the backward pass.
int ptrb200_attention_tc_fwd(const float* Q, const float* K, const float* V, float* O, float* P_out,
                             int B, int n, int H, int D, int ld_qkv, int ld_o, const int32_t* key_lens, float dropout_p,
                             uint64_t seed, uint64_t offset, ptrb200_stream_t stream) {
    if (!Q || !K || !V || !O || !P_out || B <= 0 || n <= 0 || H <= 0 || D <= 0) { set_error("attention_tc_fwd: bad arguments"); return PTRB200_ERR_INVALID; }
    cudaStream_t st = (cudaStream_t)stream;
    const int Z = B * H, HD = H * D;
    const int lq = ld_qkv > 0 ? ld_qkv : HD, lo = ld_o > 0 ? ld_o : HD;
    if (lq < HD || lo < HD) { set_error("attention_tc_fwd: row pitch below H*D"); return PTRB200_ERR_INVALID; }
    const long long sb = (long long)n * lq, sbo = (long long)n * lo, sh = D, nn = (long long)n * n;
    int rc;
    BGemmArgs g{};
    // S = Q K^T / sqrt(D)
    g.A = Q; g.B = K; g.C = P_out; g.M = n; g.N = n; g.K = D; g.lda = lq; g.ldb = lq; g.ldc = n;
    g.sAb = sb; g.sAh = sh; g.sBb = sb; g.sBh = sh; g.sCb = nn * H; g.sCh = nn; g.H = H; g.alpha = 1.0f / sqrtf((float)D);
    if ((rc = launch_bgemm(g, Z, st, "attn_tc_qk"))) return rc;
    const size_t rows = (size_t)Z * n;
    PTRB200_LAUNCH(softmax_rows_kernel, (unsigned)((rows + 7) / 8), 256, 0, st, P_out, rows, n, key_lens, H * n);
    // O = dropout(P) V : V is the [K = key, N = d] row-major factor, consumed MN-major
    BGemmArgs o{};
    o.A = P_out; o.B = V; o.C = O; o.M = n; o.N = D; o.K = n; o.lda = n; o.ldb = lq; o.ldc = lo; o.b_mn = 1;
    o.sAb = nn * H; o.sAh = nn; o.sBb = sb; o.sBh = sh; o.sCb = sbo; o.sCh = sh; o.H = H; o.alpha = 1.0f;
    o.drop_mode = 1; o.drop = make_drop_call(dropout_p, seed, offset);
    if ((rc = launch_bgemm(o, Z, st, "attn_tc_pv"))) return rc;
    return check_launch("attention_tc_fwd");
}

int ptrb200_attention_tc_bwd(const float* Q, const float* K, const float* V, const float* P, const float* dO,
                             float* dQ, float* dK, float* dV, float* scratch,
                             int B, int n, int H, int D, int ld_qkv, int ld_o, float dropout_p, uint64_t seed,
                             uint64_t offset, ptrb200_stream_t stream) {
    if (!Q || !K || !V || !P || !dO || !dQ || !dK || !dV || !scratch || B <= 0 || n <= 0 || H <= 0 || D <= 0) { set_error("attention_tc_bwd: bad arguments"); return PTRB200_ERR_INVALID; }
    cudaStream_t st = (cudaStream_t)stream;
    const int Z = B * H, HD = H * D;
    const int lq = ld_qkv > 0 ? ld_qkv : HD, lo = ld_o > 0 ? ld_o : HD;
    if (lq < HD || lo < HD) { set_error("attention_tc_bwd: row pitch below H*D"); return PTRB200_ERR_INVALID; }
    const long long sb = (long long)n * lq, sbo = (long long)n * lo, sh = D, nn = (long long)n * n;
    float* dS = scratch;                    // [Z,n,n]
    const DropCfg drop = make_drop_call(dropout_p, seed, offset);
    const float inv_scale = 1.0f / sqrtf((float)D);
    int rc;
    // dA_d = dO V^T
    BGemmArgs a{};
    a.A = dO; a.B = V; a.C = dS; a.M = n; a.N = n; a.K = D; a.lda = lo; a.ldb = lq; a.ldc = n;
    a.sAb = sbo; a.sAh = sh; a.sBb = sb; a.sBh = sh; a.sCb = nn * H; a.sCh = nn; a.H = H; a.alpha = 1.0f;
    if ((rc = launch_bgemm(a, Z, st, "attn_tc_dp"))) return rc;
    const size_t rows = (size_t)Z * n;
    PTRB200_LAUNCH(softmax_bwd_rows_kernel, (unsigned)((rows + 7) / 8), 256, 0, st, P, dS, rows, n, inv_scale, drop);
    // dQ = dS K : K is the [K = key, N = d] factor (MN-major B)
    BGemmArgs q{};
    q.A = dS; q.B = K; q.C = dQ; q.M = n; q.N = D; q.K = n; q.lda = n; q.ldb = lq; q.ldc = lq; q.b_mn = 1;
    q.sAb = nn * H; q.sAh = nn; q.sBb = sb; q.sBh = sh; q.sCb = sb; q.sCh = sh; q.H = H; q.alpha = 1.0f;
    if ((rc = launch_bgemm(q, Z, st, "attn_tc_dq"))) return rc;
    // dK = dS^T Q : dS itself is the [K = query, M = key] factor (MN-major A), Q the [K = query, N = d] factor (MN-major B)
    BGemmArgs k{};
    k.A = dS; k.B = Q; k.C = dK; k.M = n; k.N = D; k.K = n; k.lda = n; k.ldb = lq; k.ldc = lq; k.a_mn = 1; k.b_mn = 1;
    k.sAb = nn * H; k.sAh = nn; k.sBb = sb; k.sBh = sh; k.sCb = sb; k.sCh = sh; k.H = H; k.alpha = 1.0f;
    if ((rc = launch_bgemm(k, Z, st, "attn_tc_dk"))) return rc;
    // dV = dropout(P)^T dO : same shapes, the dropout mask regenerated through the transposed view
    BGemmArgs v{};
    v.A = P; v.B = dO; v.C = dV; v.M = n; v.N = D; v.K = n; v.lda = n; v.ldb = lo; v.ldc = lq; v.a_mn = 1; v.b_mn = 1;
    v.sAb = nn * H; v.sAh = nn; v.sBb = sbo; v.sBh = sh; v.sCb = sb; v.sCh = sh; v.H = H; v.alpha = 1.0f;
    v.drop_mode = 2; v.drop = drop;
    if ((rc = launch_bgemm(v, Z, st, "attn_tc_dv"))) return rc;
    return check_launch("attention_tc_bwd");
}

}  // extern "C"
