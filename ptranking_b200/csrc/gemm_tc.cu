// gemm_tc.cu -- wgmma (Hopper warpgroup tensor core) GEMM building block, fp32 in / fp32 out.
//
//   C[M,N] = A[M,K] * B[N,K]^T          (both operands K-major, i.e. nn.Linear's x @ W^T)
//
// fp32 operands are fed to tf32 wgmma MMAs either once (PASSES=1: TF32 accuracy) or as the
// error-compensated 3xTF32 split  a = a_hi + a_lo :  a_lo*b_hi + a_hi*b_lo + a_hi*b_hi  with
// fp32 accumulation in registers, which restores ~fp32 accuracy (|err| ~ 2^-21 per product) so the
// scorer keeps the reference's fp32 semantics (north_star: outputs within 1e-5 of the fp32 path).
// This file holds the plain (un-fused) kernel used by tests and odd shapes; the fused layer
// kernels in ffnet_tc.cuh reuse the same staging/issue code.
#include "common.cuh"
#include "tc.cuh"

namespace ptrb200 {

// stage one K-chunk (32 fp32 per row) of a row-major fp32 matrix into the swizzled hi/lo buffers.
// rows_valid/ k_valid guard the edges; everything outside is zero.
template <int ROWS, int THREADS, bool SPLIT>
static __device__ __forceinline__ void stage_chunk(const float* __restrict__ src, int ld, int row0, int rows_total,
                                                  int k0, int K, unsigned char* hi, unsigned char* lo) {
    constexpr int UNITS = ROWS * 8;
    for (int u = threadIdx.x; u < UNITS; u += THREADS) {
        const int r = u >> 3, j = u & 7;
        const int gr = row0 + r, gk = k0 + j * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gr < rows_total && gk < K) {
            const float* p = src + (size_t)gr * ld + gk;
            if (gk + 3 < K && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
                v = *reinterpret_cast<const float4*>(p);
            } else {
                v.x = p[0];
                if (gk + 1 < K) v.y = p[1];
                if (gk + 2 < K) v.z = p[2];
                if (gk + 3 < K) v.w = p[3];
            }
        }
        const uint32_t off = tc::swz_offset(r, j);
        if (SPLIT) {
            float4 h, l;
            tc::split_tf32(v.x, h.x, l.x); tc::split_tf32(v.y, h.y, l.y);
            tc::split_tf32(v.z, h.z, l.z); tc::split_tf32(v.w, h.w, l.w);
            *reinterpret_cast<float4*>(hi + off) = h;
            *reinterpret_cast<float4*>(lo + off) = l;
        } else {
            *reinterpret_cast<float4*>(hi + off) = v;
        }
    }
}

constexpr int TG_THREADS = 256;          // two warpgroups, 64 rows of the 128-row tile each
constexpr int TG_NT = 128;               // output columns per CTA (gridDim.y tiles)

template <int PASSES>
__global__ void __launch_bounds__(TG_THREADS) tc_gemm_nt_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                                float* __restrict__ C, int M, int N_full, int K) {
    extern __shared__ __align__(1024) unsigned char smem[];
    // [A_hi 16K][A_lo 16K][B_hi NP*128][B_lo NP*128]
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem) + 1023) & ~(uintptr_t)1023);
    const int n0 = blockIdx.y * TG_NT, N = min(TG_NT, N_full - n0), NP = ((N + 15) / 16) * 16;
    unsigned char* a_hi = base;
    unsigned char* a_lo = a_hi + 128 * 128;
    unsigned char* b_hi = a_lo + 128 * 128;
    unsigned char* b_lo = b_hi + NP * 128;
    const float* Bt = B + (size_t)n0 * K;

    const int wg = threadIdx.x >> 7;
    const int m0 = blockIdx.x * 128;
    const int nchunks = (K + 31) / 32;
    tc::with_width(NP, [&](auto W) {
        constexpr int NPc = decltype(W)::value;
        float acc[NPc / 2];
#pragma unroll
        for (int e = 0; e < NPc / 2; ++e) acc[e] = 0.0f;
        for (int c = 0; c < nchunks; ++c) {
            if (c > 0) __syncthreads();                               // both warpgroups' MMAs of the previous chunk are done
            stage_chunk<128, TG_THREADS, PASSES == 3>(A, K, m0, M, c * 32, K, a_hi, a_lo);
            // B rows beyond N are zero (guard inside stage_chunk via rows_total = N)
            if (NPc == 128) stage_chunk<128, TG_THREADS, PASSES == 3>(Bt, K, 0, N, c * 32, K, b_hi, b_lo);
            else {
                for (int u = threadIdx.x; u < NPc * 8; u += TG_THREADS) {
                    const int r = u >> 3, j = u & 7, gk = c * 32 + j * 4;
                    float v[4] = {0.f, 0.f, 0.f, 0.f};
                    if (r < N) for (int e = 0; e < 4; ++e) if (gk + e < K) v[e] = Bt[(size_t)r * K + gk + e];
                    float4 h, l;
                    if (PASSES == 3) { tc::split_tf32(v[0], h.x, l.x); tc::split_tf32(v[1], h.y, l.y); tc::split_tf32(v[2], h.z, l.z); tc::split_tf32(v[3], h.w, l.w); }
                    else { h = make_float4(v[0], v[1], v[2], v[3]); l = h; }
                    const uint32_t off = tc::swz_offset(r, j);
                    *reinterpret_cast<float4*>(b_hi + off) = h;
                    if (PASSES == 3) *reinterpret_cast<float4*>(b_lo + off) = l;
                }
            }
            tc::fence_proxy_async();
            __syncthreads();
            tc::wg_fence();
#pragma unroll
            for (int s = 0; s < 4; ++s) {                         // columns beyond K are staged as zeros
                const uint64_t ah = tc::smem_desc_sw128(tc::smem_u32(a_hi) + wg * 8192 + s * 32, 1024);
                const uint64_t bh = tc::smem_desc_sw128(tc::smem_u32(b_hi) + s * 32, 1024);
                if (PASSES == 3) {
                    const uint64_t al = tc::smem_desc_sw128(tc::smem_u32(a_lo) + wg * 8192 + s * 32, 1024);
                    const uint64_t bl = tc::smem_desc_sw128(tc::smem_u32(b_lo) + s * 32, 1024);
                    tc::mma_tf32<NPc>(acc, al, bh, 1u);
                    tc::mma_tf32<NPc>(acc, ah, bl, 1u);
                    tc::mma_tf32<NPc>(acc, ah, bh, 1u);
                } else {
                    tc::mma_tf32<NPc>(acc, ah, bh, 1u);
                }
            }
            tc::wg_commit();
            tc::wg_wait<0>();
        }
#pragma unroll
        for (int e = 0; e < NPc / 2; ++e) {
            const int row = m0 + wg * 64 + tc::acc_row(e & 7), col = (e >> 3) * 16 + tc::acc_col(e & 7);
            if (row < M && col < N) C[(size_t)row * N_full + n0 + col] = acc[e];
        }
    });
}

}  // namespace ptrb200

using namespace ptrb200;

extern "C" int ptrb200_tc_gemm_nt(const float* A, const float* B, float* C, int M, int N, int K, int passes,
                                  ptrb200_stream_t stream) {
    if (!A || !B || !C || M <= 0 || N <= 0 || K <= 0) { set_error("tc_gemm_nt: bad arguments"); return PTRB200_ERR_INVALID; }
    if (N > 256) { set_error("tc_gemm_nt: N=%d > 256", N); return PTRB200_ERR_UNSUPPORTED; }
    if (passes != 1 && passes != 3) { set_error("tc_gemm_nt: passes must be 1 or 3"); return PTRB200_ERR_INVALID; }
    const size_t smem = 1024 + 2 * 128 * 128 + 2 * (size_t)TG_NT * 128;
    const dim3 grid((M + 127) / 128, (N + TG_NT - 1) / TG_NT);
    cudaError_t e;
    if (passes == 3) {
        e = cudaFuncSetAttribute(tc_gemm_nt_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("tc_gemm_nt smem attr: %s", cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
        PTRB200_LAUNCH(tc_gemm_nt_kernel<3>, grid, TG_THREADS, smem, stream, A, B, C, M, N, K);
    } else {
        e = cudaFuncSetAttribute(tc_gemm_nt_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("tc_gemm_nt smem attr: %s", cudaGetErrorString(e)); return PTRB200_ERR_CUDA; }
        PTRB200_LAUNCH(tc_gemm_nt_kernel<1>, grid, TG_THREADS, smem, stream, A, B, C, M, N, K);
    }
    return check_launch("tc_gemm_nt");
}
