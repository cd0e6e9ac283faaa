// ffnet_tc.cuh -- wgmma layer kernels of the stacked feed-forward scorer.
//
// Three kernels cover one Linear layer in both directions; post-activation tensors are never
// written to HBM -- they are rebuilt from the previous layer's pre-activation Z in the operand
// staging prologue (one FMA + activation per element, free next to the HBM stream):
//
//   rows_gemm<FWD>    Z_l[rows,N]  = drop(act(Z_{l-1}*scale+shift)) * W^T + b     (+ BN partial sums)
//   rows_gemm<DGRAD>  dA[rows,K]   = dropmask( dZ_l * W )                           (Wt = W^T staged)
//   wgrad             dW[N,K]      = sum_rows dZ_l[r,:]^T (x) drop(act(Z_{l-1}*scale+shift))[r,:]
//
// All contractions run as tf32 wgmma with fp32 accumulation in registers; PASSES = 3 is the
// error-compensated 3xTF32 split (fp32-equivalent, the default), PASSES = 1 plain TF32.
#pragma once
#include "common.cuh"
#include "tc.cuh"
#include "ffnet_act.cuh"

namespace ptrb200 {

struct RowsGemmArgs {
    // A-side source and its prologue
    const float* P;        // [rows, K]
    const float* scale;    // [Gp, K] or NULL (identity)
    const float* shift;    // [Gp, K]
    int act;               // PTRB200_AF_* applied after scale/shift (AF_NONE = identity)
    int gr_prev;           // rows per statistics group of P's normalisation
    DropCfg drop;          // dropout stream: FWD masks A elements (row*K+k), DGRAD masks outputs (row*N+n)
    // DGRAD with the normalisation backward folded in: A = k1*P + k3*P2 + k0 (P = dY, P2 = Z of this layer,
    // coefficients per (statistics group, column) from dy_finalize_kernel).  P2 == NULL: A = P.
    const float* P2;
    const float *kc1, *kc3, *kc0;
    int gr_cur;            // rows per statistics group of kc*
    // B side: pre-split, pre-swizzled operand images written by pack_b_image_kernel:
    // chunk c of the image = [NP rows x 128 B] in the exact shared-memory layout (one bulk copy each)
    const unsigned char* b_img_hi;
    const unsigned char* b_img_lo;
    const float* bias;     // [N] (FWD) or NULL
    float* a_out;          // FWD: when non-NULL the rebuilt (post-activation, post-dropout) A operand is also written
                           // here [rows, K] so the weight-gradient kernel can read it back instead of recomputing it
    float* Out;            // [rows, N]
    double* partials;      // [slots, N, 2] column sum / sum of squares per statistics slot, or NULL
    int rows, K, N, NP;
    int n_tile;            // one-tile-per-CTA kernel: output columns per CTA (gridDim.y tiles, <= RG_MAX_N); N when untiled
    int tail_off;          // byte offset of the mbarriers behind max(operand buffers, output tile)
    // tile -> rows mapping
    int tile_rows;         // rows advanced per tile (<= 128)
    int seg_len;           // rows per statistics segment inside a tile
    int group_rows;        // BN2 with n > 128: rows per group (tiles restart at every group), else 0
    int tiles_per_group;
    int round_bf16;        // PTRB200_MATH_BF16: the A operand is rounded to bf16 on its way into shared memory
};

enum { RG_FWD = 0, RG_DGRAD = 1 };

// prologue transform of 4 consecutive elements (row r, columns k..k+3) of P
// ACT >= 0: the activation is a compile-time constant (no per-element switch); ACT = -1 reads g.act
template <int ACT = -1>
static __device__ __forceinline__ float4 prologue4(const RowsGemmArgs& g, float4 v, int row, int k, bool with_dropout, size_t coef_row_off) {
    if (g.scale) {
        const size_t o = coef_row_off + k;
        const float4 sc = *reinterpret_cast<const float4*>(g.scale + o);
        const float4 sh = *reinterpret_cast<const float4*>(g.shift + o);
        v.x = fmaf(v.x, sc.x, sh.x); v.y = fmaf(v.y, sc.y, sh.y); v.z = fmaf(v.z, sc.z, sh.z); v.w = fmaf(v.w, sc.w, sh.w);
    }
    const int af = ACT >= 0 ? ACT : g.act;
    if (af != PTRB200_AF_NONE) {
        v.x = activate(af, v.x).y; v.y = activate(af, v.y).y; v.z = activate(af, v.z).y; v.w = activate(af, v.w).y;
    }
    if (with_dropout && g.drop.thr) {
        const uint64_t e = (uint64_t)row * g.K + k;          // K % 4 == 0: the 4 elements share one draw
        const uint64_t d = dropout_draw4(g.drop.key, e >> 2);
        v.x = ((uint32_t)(d) & 0xffffu) >= g.drop.thr ? v.x * g.drop.scale : 0.0f;
        v.y = ((uint32_t)(d >> 16) & 0xffffu) >= g.drop.thr ? v.y * g.drop.scale : 0.0f;
        v.z = ((uint32_t)(d >> 32) & 0xffffu) >= g.drop.thr ? v.z * g.drop.scale : 0.0f;
        v.w = ((uint32_t)(d >> 48)) >= g.drop.thr ? v.w * g.drop.scale : 0.0f;
    }
    return v;
}

// round-to-nearest-even onto the bf16 grid (the result is still an fp32 / tf32 value)
static __device__ __forceinline__ float bf16_rn(float x) {
    const uint32_t u = __float_as_uint(x);
    return __uint_as_float((u + 0x7fffu + ((u >> 16) & 1u)) & 0xffff0000u);
}
// rn: round-to-nearest hi/lo split (unbiased, per-product error 2^-22) instead of the truncating one (2^-20, biased towards
// zero, 3 instructions per element cheaper) -- used where the contraction is long enough for the bias to show (K > 160)
static __device__ __forceinline__ void store_split(unsigned char* hi, unsigned char* lo, uint32_t off, float4 v, bool split, bool to_bf16 = false, bool rn = false) {
    if (to_bf16) v = make_float4(bf16_rn(v.x), bf16_rn(v.y), bf16_rn(v.z), bf16_rn(v.w));
    if (split) {
        float4 h, l;
        if (rn) {
            tc::split_tf32_rn(v.x, h.x, l.x); tc::split_tf32_rn(v.y, h.y, l.y);
            tc::split_tf32_rn(v.z, h.z, l.z); tc::split_tf32_rn(v.w, h.w, l.w);
        } else {
            tc::split_tf32(v.x, h.x, l.x); tc::split_tf32(v.y, h.y, l.y);
            tc::split_tf32(v.z, h.z, l.z); tc::split_tf32(v.w, h.w, l.w);
        }
        *reinterpret_cast<float4*>(hi + off) = h;
        *reinterpret_cast<float4*>(lo + off) = l;
    } else {
        *reinterpret_cast<float4*>(hi + off) = v;
    }
}

static __device__ __forceinline__ float4 ldg4_guard(const float* p, int k, int K) {
    // K % 4 == 0 and 16-byte aligned rows are guaranteed by the host launcher
    return (k < K) ? __ldg(reinterpret_cast<const float4*>(p)) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// bf16 features (the layer-0 "XB" kernel variants): `base` holds bf16 values behind a float pointer.  Elements
// elem .. elem+3 arrive in one 8-byte load (elem % 4 == 0, 8-byte aligned base: host guarantees) and widen exactly to fp32
// -- a bf16 value is its fp32 value with the low 16 bits zero -- so everything downstream sees the same numbers an fp32
// copy of the features would give.
static __device__ __forceinline__ float4 ldg_bf16x4(const float* base, size_t elem) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(base) + elem));
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u),
                       __uint_as_float(u.y << 16), __uint_as_float(u.y & 0xffff0000u));
}
template <bool XB>
static __device__ __forceinline__ float4 ldg_a4(const float* base, size_t elem) {
    if constexpr (XB) return ldg_bf16x4(base, elem);
    else return __ldg(reinterpret_cast<const float4*>(base + elem));
}

// Builds the B-operand image of a [N,K] row-major matrix (TRANSPOSE=false) or of its transpose
// (TRANSPOSE=true: image rows = columns of the source, used for dgrad's W^T): hi/lo tf32 split,
// rows padded to NP, K cut into 128-byte chunks, each chunk [NP][128 B] in SWIZZLE_128B order.
// One launch packs every image of a net: blockIdx.y picks the job (layer x {forward W, dgrad W^T}).
struct PackJob {
    const float* src;
    unsigned char *img_hi, *img_lo;
    int src_cols, N, NP, K, nchunks, transpose, round_bf16;
};
constexpr int PACK_MAX_JOBS = 2 * PTRB200_MAX_FF_LAYERS;
struct PackJobs { PackJob job[PACK_MAX_JOBS]; };

__global__ void pack_b_images_kernel(const __grid_constant__ PackJobs jobs) {
    const PackJob& jb = jobs.job[blockIdx.y];
    const float* __restrict__ src = jb.src;
    unsigned char* __restrict__ img_hi = jb.img_hi;
    unsigned char* __restrict__ img_lo = jb.img_lo;
    const int src_cols = jb.src_cols, N = jb.N, NP = jb.NP, K = jb.K, nchunks = jb.nchunks;
    const bool TRANSPOSE = jb.transpose != 0;
    const int total = nchunks * NP * 8;                        // 16-byte units
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
        const int c = u / (NP * 8), rem = u % (NP * 8), r = rem >> 3, j = rem & 7, k = c * 32 + j * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (r < N) {
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (k + e < K) v[e] = TRANSPOSE ? src[(size_t)(k + e) * src_cols + r] : src[(size_t)r * src_cols + k + e];
        }
        const size_t off = (size_t)c * NP * 128 + tc::swz_offset(r, j);
        if (jb.round_bf16) {
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = bf16_rn(v[e]);
        }
        float4 h, l;          // round-to-nearest split: the images are built once per step, the unbiased split is free here
        tc::split_tf32_rn(v[0], h.x, l.x); tc::split_tf32_rn(v[1], h.y, l.y); tc::split_tf32_rn(v[2], h.z, l.z); tc::split_tf32_rn(v[3], h.w, l.w);
        if (img_lo) {
            *reinterpret_cast<float4*>(img_hi + off) = h;
            *reinterpret_cast<float4*>(img_lo + off) = l;
        } else {
            *reinterpret_cast<float4*>(img_hi + off) = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

template <bool TRANSPOSE>
__global__ void pack_b_image_kernel(const float* __restrict__ src, int src_rows, int src_cols,
                                    unsigned char* __restrict__ img_hi, unsigned char* __restrict__ img_lo,
                                    int N, int NP, int K, int nchunks, int round_bf16 = 0) {
    const int total = nchunks * NP * 8;                        // 16-byte units
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
        const int c = u / (NP * 8), rem = u % (NP * 8), r = rem >> 3, j = rem & 7, k = c * 32 + j * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (r < N) {
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (k + e < K) v[e] = TRANSPOSE ? src[(size_t)(k + e) * src_cols + r] : src[(size_t)r * src_cols + k + e];
        }
        if (round_bf16) {
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = bf16_rn(v[e]);
        }
        const size_t off = (size_t)c * NP * 128 + tc::swz_offset(r, j);
        float4 h, l;          // round-to-nearest split: the images are built once per step, the unbiased split is free here
        tc::split_tf32_rn(v[0], h.x, l.x); tc::split_tf32_rn(v[1], h.y, l.y); tc::split_tf32_rn(v[2], h.z, l.z); tc::split_tf32_rn(v[3], h.w, l.w);
        if (img_lo) {
            *reinterpret_cast<float4*>(img_hi + off) = h;
            *reinterpret_cast<float4*>(img_lo + off) = l;
        } else {
            *reinterpret_cast<float4*>(img_hi + off) = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

constexpr int RG_THREADS = 256;         // two warpgroups, 64 rows of the 128-row tile each
constexpr int RG_MAX_N = 128;           // output columns per CTA: the accumulators of a 64 x 128 warpgroup tile fill 64 registers

// XB: g.P holds bf16 features (layer 0 only: FWD, no scale/shift, no activation)
template <int MODE, int PASSES, int ACT = -1, bool XB = false>
__global__ void __launch_bounds__(RG_THREADS) rows_gemm_tc_kernel(RowsGemmArgs g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    // output-column tile of this CTA (gridDim.y tiles of n_tile columns; the weight image is [NP_full rows] per chunk)
    const int N_full = g.N, NP_full = g.NP;
    const int n0 = blockIdx.y * g.n_tile;
    const int N = min(g.n_tile, N_full - n0);
    const int NP = ((N + 15) / 16) * 16;
    unsigned char* a_hi = base;                       // 128 rows x 128 B
    unsigned char* a_lo = a_hi + 16384;
    // weight chunk, double buffered: [2][hi | lo], NP rows x 128 B each (the copy of chunk c+1 is issued as soon as the MMAs
    // of chunk c-1 have released its buffer, a whole chunk ahead of its use)
    unsigned char* b_buf = a_lo + 16384;
    const uint32_t b_stage = (uint32_t)NP * 128u * (PASSES == 3 ? 2u : 1u);
    unsigned char* tail = base + g.tail_off;
    uint64_t* bbar = reinterpret_cast<uint64_t*>(tail);   // [2] weight chunk landed
    float* otile = reinterpret_cast<float*>(base);    // epilogue staging [128][N], aliases the operand buffers

    const int tid = threadIdx.x, wg = tid >> 7;
    // ---- tile -> rows ------------------------------------------------------------
    int row0, nrows, slot0;
    {
        const int t = blockIdx.x;
        if (g.group_rows > 0) {
            const int grp = t / g.tiles_per_group, tt = t % g.tiles_per_group;
            row0 = grp * g.group_rows + tt * 128;
            nrows = min(128, g.group_rows - tt * 128);
            slot0 = t;
        } else {
            row0 = t * g.tile_rows;
            nrows = min(g.tile_rows, g.rows - row0);
            slot0 = (row0 / g.seg_len);
        }
    }
    // The error of a 3xTF32 contraction grows with the number of accumulate steps (DESIGN.md 4): the small
    // a_lo*b_hi + a_hi*b_lo corrections accumulate apart from the main products (two thirds of the accumulate steps
    // leave the main chain; the epilogue adds the two), and contractions longer than 5 chunks (K > 160: the 256- and
    // 512-wide layers of the list scorer's head / tail nets) also stage A with the round-to-nearest split.
    const int K = g.K;
    const int nchunks = (K + 31) / 32;
    const bool long_k = PASSES == 3 && nchunks > 5;
    if (tid == 0) { tc::mbar_init(bbar, 1); tc::mbar_init(bbar + 1, 1); tc::mbar_fence_init(); }
    __syncthreads();
    constexpr int A_UNITS = 128 * 8 / RG_THREADS;      // 4 units of 16 B per thread per chunk
    size_t coef_off[A_UNITS];                           // (statistics group of the thread's rows) * K
#pragma unroll
    for (int i = 0; i < A_UNITS; ++i) {
        const int r = (tid + i * RG_THREADS) >> 3;
        coef_off[i] = (g.scale && g.gr_prev < g.rows) ? (size_t)((row0 + min(r, nrows - 1)) / g.gr_prev) * K : 0;
    }

    // ---- global -> registers one chunk AHEAD: the loads of chunk c+1 fly while chunk c is staged, synchronised and
    // multiplied (a tile's chunks are strictly sequential and few CTAs share an SM at list-scorer row counts, so nothing
    // else hides the HBM latency) ----
    float4 nav[A_UNITS];
    auto load_chunk = [&](int c) {
#pragma unroll
        for (int i = 0; i < A_UNITS; ++i) {
            const int u = tid + i * RG_THREADS, r = u >> 3, j = u & 7, k = c * 32 + j * 4;
            if constexpr (XB) nav[i] = (r < nrows && k < K) ? ldg_bf16x4(g.P, (size_t)(row0 + r) * K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
            else nav[i] = (r < nrows) ? ldg4_guard(g.P + (size_t)(row0 + r) * K + k, k, K) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    load_chunk(0);
    tc::with_width(NP, [&](auto W) {
    constexpr int NPc = decltype(W)::value;
    float acc[NPc / 2], acc2[NPc / 2];
#pragma unroll
    for (int e = 0; e < NPc / 2; ++e) { acc[e] = 0.0f; acc2[e] = 0.0f; }
    for (int c = 0; c < nchunks; ++c) {
        const int k0 = c * 32;
        float4 av[A_UNITS];
#pragma unroll
        for (int i = 0; i < A_UNITS; ++i) av[i] = nav[i];
        if (c + 1 < nchunks) load_chunk(c + 1);
        if (c > 0) __syncthreads();                        // both warpgroups' MMAs of chunk c-1 are done with the A buffer and B stage
        // ---- B: one TMA bulk copy per operand image chunk (no SM instructions beyond the issue), one chunk ahead ----
        if (tid == 0) {
            auto fetch_b = [&](int cc) {
                const uint32_t bytes = (uint32_t)NP * 128u;
                const size_t src = ((size_t)cc * NP_full + n0) * 128u;       // rows [n0, n0+NP) of chunk cc
                unsigned char* dst = b_buf + (size_t)(cc & 1) * b_stage;
                tc::mbar_expect_tx(bbar + (cc & 1), PASSES == 3 ? 2 * bytes : bytes);
                tc::bulk_g2s(dst, g.b_img_hi + src, bytes, bbar + (cc & 1));
                if (PASSES == 3) tc::bulk_g2s(dst + bytes, g.b_img_lo + src, bytes, bbar + (cc & 1));
            };
            if (c == 0) fetch_b(0);
            if (c + 1 < nchunks) fetch_b(c + 1);      // its buffer was last read by chunk c-1, whose MMAs have completed
        }
        // ---- A: prologue + split + swizzled store ----
#pragma unroll
        for (int i = 0; i < A_UNITS; ++i) {
            const int u = tid + i * RG_THREADS, r = u >> 3, j = u & 7, k = k0 + j * 4;
            float4 v = av[i];
            if (r < nrows && k < K) {
                if (MODE == RG_DGRAD && g.P2) {                   // dZ = k1*dY + k3*Z + k0 (normalisation backward folded in)
                    const size_t kc = (g.gr_cur < g.rows ? (size_t)((row0 + r) / g.gr_cur) * K : (size_t)0) + k;
                    const float4 z = __ldg(reinterpret_cast<const float4*>(g.P2 + (size_t)(row0 + r) * K + k));
                    const float4 a1 = __ldg(reinterpret_cast<const float4*>(g.kc1 + kc));
                    const float4 a3 = __ldg(reinterpret_cast<const float4*>(g.kc3 + kc));
                    const float4 a0 = __ldg(reinterpret_cast<const float4*>(g.kc0 + kc));
                    v.x = fmaf(a1.x, v.x, fmaf(a3.x, z.x, a0.x)); v.y = fmaf(a1.y, v.y, fmaf(a3.y, z.y, a0.y));
                    v.z = fmaf(a1.z, v.z, fmaf(a3.z, z.z, a0.z)); v.w = fmaf(a1.w, v.w, fmaf(a3.w, z.w, a0.w));
                }
                v = prologue4<ACT>(g, v, row0 + r, k, MODE == RG_FWD, coef_off[i]);
                if (MODE == RG_FWD && g.a_out && blockIdx.y == 0) *reinterpret_cast<float4*>(g.a_out + (size_t)(row0 + r) * K + k) = v;
            } else v = make_float4(0.f, 0.f, 0.f, 0.f);
            store_split(a_hi, a_lo, tc::swz_offset(r, j), v, PASSES == 3, PASSES == 1 && g.round_bf16 != 0, long_k);
        }
        tc::fence_proxy_async();
        __syncthreads();
        tc::mbar_wait(bbar + (c & 1), (c >> 1) & 1);          // weights chunk has landed
        const uint32_t a_s = tc::smem_u32(a_hi) + wg * 8192;
        const uint32_t b_hi_s = tc::smem_u32(b_buf) + (uint32_t)(c & 1) * b_stage, b_lo_s = b_hi_s + (uint32_t)NP * 128u;
        // four K-steps per chunk: the columns beyond K are staged as zeros, so a fixed chain keeps the wgmmas back to back
        tc::wg_fence();
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const uint64_t ah = tc::smem_desc_sw128(a_s + s * 32, 1024);
            const uint64_t bh = tc::smem_desc_sw128(b_hi_s + s * 32, 1024);
            if (PASSES == 3) {
                const uint64_t al = tc::smem_desc_sw128(a_s + 16384 + s * 32, 1024);
                const uint64_t bl = tc::smem_desc_sw128(b_lo_s + s * 32, 1024);
                tc::mma_tf32<NPc>(acc2, al, bh, 1u);
                tc::mma_tf32<NPc>(acc2, ah, bl, 1u);
            }
            tc::mma_tf32<NPc>(acc, ah, bh, 1u);
        }
        tc::wg_commit();
        tc::wg_wait<0>();                                 // the same threads stage the next chunk: its registers are needed there
    }
    __syncthreads();                                      // every MMA is done: the output tile may overwrite the operands

    // ---- epilogue: registers -> (+bias | dropout mask) -> smem tile [128][N] ----
#pragma unroll
    for (int e = 0; e < NPc / 2; ++e) {
        const int r = wg * 64 + tc::acc_row(e), col = tc::acc_col(e);
        if (col >= N) continue;
        float v = PASSES == 3 ? acc[e] + acc2[e] : acc[e];
        if (MODE == RG_FWD) v += __ldg(g.bias + n0 + col);
        else if (g.drop.thr)
            v = dropout_keep(g.drop.key, (uint64_t)(row0 + r) * N_full + n0 + col, g.drop.thr) ? v * g.drop.scale : 0.0f;
        otile[(size_t)r * N + col] = v;
    }
    });
    __syncthreads();
    // ---- tile -> global: contiguous when untiled, row segments of pitch N_full otherwise ----
    if (N == N_full) {
        const size_t total = (size_t)nrows * N;
        float* dst = g.Out + (size_t)row0 * N;
        if ((N & 3) == 0) {
            const float4* s4 = reinterpret_cast<const float4*>(otile);
            float4* d4 = reinterpret_cast<float4*>(dst);
            for (size_t i = tid; i < total / 4; i += RG_THREADS) d4[i] = s4[i];
        } else {
            for (size_t i = tid; i < total; i += RG_THREADS) dst[i] = otile[i];
        }
    } else {                                           // n0, N and N_full are multiples of 4 here (host guarantees)
        const int q4 = N >> 2;
        for (int i = tid; i < nrows * q4; i += RG_THREADS) {
            const int r = i / q4, qq = i - r * q4;
            *reinterpret_cast<float4*>(g.Out + (size_t)(row0 + r) * N_full + n0 + qq * 4) = *reinterpret_cast<const float4*>(otile + (size_t)r * N + qq * 4);
        }
    }
    // ---- per-segment column sums for the layer's normalisation (fixed order: deterministic) ----
    if (MODE == RG_FWD && g.partials) {
        for (int cidx = tid; cidx < N; cidx += RG_THREADS) {
            int seg = 0;
            for (int rbeg = 0; rbeg < nrows; rbeg += g.seg_len, ++seg) {
                const int rend = min(nrows, rbeg + g.seg_len);
                double s1 = 0.0, s2 = 0.0;
                for (int r = rbeg; r < rend; ++r) {
                    const float z = otile[(size_t)r * N + cidx];
                    s1 += (double)z; s2 += (double)z * (double)z;
                }
                double* p = g.partials + ((size_t)(slot0 + seg) * N_full + n0 + cidx) * 2;
                p[0] = s1; p[1] = s2;
            }
        }
    }
}

// --------------------------------------------------------------------------------------------
// rows_gemm, persistent warp-specialised variant (used whenever the whole weight image fits next to the
// A ring in shared memory, i.e. for every layer of the pointwise scorer).
//
//   warps 0-7   consumers: two warpgroups, 64 rows of the tile each; one-time TMA bulk load of the resident
//                          W image, per K-chunk wgmma issue, epilogue registers -> (+bias | dropout mask) ->
//                          global rows, BN column sums
//   warps 8-15  producers: global -> registers (prefetched one chunk ahead) -> prologue -> hi/lo split ->
//                          swizzled A stage (ring of 2)
// Producers and consumers only meet through mbarriers (aready/afree per A stage): the producers stage tile t+1
// while the consumers multiply and write out tile t.  512 threads start with 128 registers each; after the role
// branch the consumers give theirs down to RW_CONS_REGS (a 64 x 128 accumulator, descriptors, epilogue) and the
// producers take RW_PROD_REGS (the staged and the prefetched chunk, per-tile pointers, dropout keys): at 128 each
// the producers spill.
// --------------------------------------------------------------------------------------------
constexpr int RW_EPI_WARPS = 8, RW_PROD_WARPS = 8;
constexpr int RW_THREADS = (RW_EPI_WARPS + RW_PROD_WARPS) * 32;
constexpr int RW_PRODUCERS = RW_PROD_WARPS * 32;
constexpr int RW_PU = 128 * 8 / RW_PRODUCERS;            // 16-byte A units per producer thread per chunk
constexpr int RW_MAX_N = 128;
constexpr int RW_CONS_REGS = 120, RW_PROD_REGS = 136;
static_assert((RW_CONS_REGS * RW_EPI_WARPS + RW_PROD_REGS * RW_PROD_WARPS) * 32 <= 65536, "register split exceeds the register file");

struct RowsWsExtra {
    int ntiles;
    int stats_mode;        // 0 none, 1 one partial per CTA (BN over the whole batch), 2 one partial per tile (BN2)
    int nchunks;
};

static __device__ __forceinline__ void rw_tile(const RowsGemmArgs& g, int t, int& row0, int& nrows) {
    if (g.group_rows > 0) {
        const int grp = t / g.tiles_per_group, tt = t - grp * g.tiles_per_group;
        row0 = grp * g.group_rows + tt * 128;
        nrows = min(128, g.group_rows - tt * 128);
    } else {
        row0 = t * g.tile_rows;
        nrows = min(g.tile_rows, g.rows - row0);
    }
}

// ACT: the prologue activation as a compile-time constant (PTRB200_AF_*), or -1 to read g.act at run time
// KT:  the contraction width as a compile-time constant (0 = read g.K at run time).  The producers spend more instructions
//      on row / chunk address arithmetic, bounds predicates and the prefetch bookkeeping than on the prologue itself; with
//      K known the chunk loops unroll completely and that arithmetic folds into immediates (instantiated for the widths
//      of the default scorer, 136 and 100).
// XB:  g.P holds bf16 features (layer 0 only: FWD, no scale/shift, no activation); the producers load 4 of them as one
//      8-byte unit and widen it before the unchanged prologue and split.
template <int MODE, int PASSES, int ACT, int KT = 0, bool XB = false>
__global__ void __launch_bounds__(RW_THREADS, 1) rows_gemm_ws_kernel(RowsGemmArgs g, RowsWsExtra x) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int NP = g.NP, K = KT ? KT : g.K, N = g.N, nchunks = KT ? (KT + 31) / 32 : x.nchunks;
    const int wchunk = NP * 128;
    unsigned char* w_hi = base;                                   // [nchunks][NP][128 B]
    unsigned char* w_lo = w_hi + (size_t)nchunks * wchunk;
    unsigned char* a_ring = w_lo + (PASSES == 3 ? (size_t)nchunks * wchunk : 0);   // [2][hi 16 KB | lo 16 KB]
    float* stat_sm = reinterpret_cast<float*>(a_ring + 2 * 32768);                 // [8 consumer warps][NP][2]
    uint64_t* bars = reinterpret_cast<uint64_t*>(stat_sm + RW_EPI_WARPS * NP * 2);
    uint64_t* wfull = bars;            // W image landed
    uint64_t* aready = bars + 1;       // [2] A stage staged            (one arrive per producer warp)
    uint64_t* afree = bars + 3;        // [2] MMAs done with the stage  (one arrive per consumer warp)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        tc::mbar_init(wfull, 1);
        for (int i = 0; i < 2; ++i) { tc::mbar_init(aready + i, RW_PROD_WARPS); tc::mbar_init(afree + i, RW_EPI_WARPS); }
        tc::mbar_fence_init();
    }
    __syncthreads();
    const int my_tiles = blockIdx.x < x.ntiles ? (x.ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (warp >= RW_EPI_WARPS) {
        tc::setmaxnreg_inc<RW_PROD_REGS>();
        if constexpr (MODE == RG_DGRAD) {
        // (the data-gradient instantiation keeps the simpler producer loop: its fused dZ = k1*dY + k3*Z + k0 staging carries
        //  more live state, and the restructured loop below would add to it)
            // ================================ producer warps ================================
            const int ptid = tid - RW_EPI_WARPS * 32;
            const int j4 = (ptid & 7) * 4;                              // first column of this thread's 16-byte unit inside a chunk
            int r_[RW_PU];
            uint32_t sw_[RW_PU];
    #pragma unroll
            for (int i = 0; i < RW_PU; ++i) { r_[i] = (ptid >> 3) + i * (RW_PRODUCERS / 8); sw_[i] = tc::swz_offset(r_[i], ptid & 7); }
            const int total_q = my_tiles * nchunks;
            const bool has_coef = g.scale != nullptr;
            const bool per_group = has_coef && g.gr_prev < g.rows;
            const bool fused_dz = MODE == RG_DGRAD && g.P2 != nullptr;
            float4 pre[RW_PU], pre2[RW_PU];
            size_t soff[RW_PU];                                         // row * K + j4 for the tile being fetched
            bool ok[RW_PU];
            auto point = [&](int it) {                                  // set soff/ok for tile `it`
                int r0, nr;
                rw_tile(g, blockIdx.x + it * gridDim.x, r0, nr);
    #pragma unroll
                for (int i = 0; i < RW_PU; ++i) { ok[i] = r_[i] < nr; soff[i] = (size_t)(r0 + min(r_[i], nr - 1)) * K + j4; }
            };
            auto fetch = [&](int c) {
                const bool kv = c * 32 + j4 < K;
    #pragma unroll
                for (int i = 0; i < RW_PU; ++i) {
                    pre[i] = (ok[i] && kv) ? __ldg(reinterpret_cast<const float4*>(g.P + soff[i] + c * 32)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (MODE == RG_DGRAD) pre2[i] = (fused_dz && ok[i] && kv) ? __ldg(reinterpret_cast<const float4*>(g.P2 + soff[i] + c * 32)) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            };
            if (total_q > 0) { point(0); fetch(0); }
            int q = 0;
            for (int it = 0; it < my_tiles; ++it) {
                int row0, nrows;
                rw_tile(g, blockIdx.x + it * gridDim.x, row0, nrows);
                // per-tile invariants of this thread's two rows
                bool live[RW_PU];
                float* aout[RW_PU];
                const float* sc[RW_PU];
                const float* sh[RW_PU];
                size_t kco[RW_PU];
                uint64_t dq[RW_PU];
    #pragma unroll
                for (int i = 0; i < RW_PU; ++i) {
                    live[i] = r_[i] < nrows;
                    const size_t e0 = (size_t)(row0 + min(r_[i], nrows - 1)) * K + j4;
                    aout[i] = (MODE == RG_FWD && g.a_out) ? g.a_out + e0 : nullptr;
                    const size_t co = per_group ? (size_t)((row0 + min(r_[i], nrows - 1)) / g.gr_prev) * K + j4 : (size_t)j4;
                    sc[i] = has_coef ? g.scale + co : nullptr;
                    sh[i] = has_coef ? g.shift + co : nullptr;
                    kco[i] = (fused_dz && g.gr_cur < g.rows) ? (size_t)((row0 + min(r_[i], nrows - 1)) / g.gr_cur) * K + j4 : (size_t)j4;
                    dq[i] = (uint64_t)e0 >> 2;
                }
    #pragma unroll 1
            for (int c = 0; c < nchunks; ++c, ++q) {
                    const int s = q & 1;
                    float4 cur[RW_PU], cur2[RW_PU];
    #pragma unroll
                    for (int i = 0; i < RW_PU; ++i) { cur[i] = pre[i]; cur2[i] = pre2[i]; }
                    if (q + 1 < total_q) {                              // prefetch the next chunk (possibly of the next tile)
                        if (c + 1 < nchunks) fetch(c + 1); else { point(it + 1); fetch(0); }
                    }
                    if (q >= 2) tc::mbar_wait(afree + s, ((q - 2) >> 1) & 1);
                    unsigned char* a_hi = a_ring + s * 32768;
                    const bool kv = c * 32 + j4 < K;
    #pragma unroll
                    for (int i = 0; i < RW_PU; ++i) {
                        float4 v = cur[i];
                        if (live[i] && kv) {
                            if (MODE == RG_DGRAD && fused_dz) {           // dZ = k1*dY + k3*Z + k0
                                const float4 a1 = __ldg(reinterpret_cast<const float4*>(g.kc1 + kco[i] + c * 32));
                                const float4 a3 = __ldg(reinterpret_cast<const float4*>(g.kc3 + kco[i] + c * 32));
                                const float4 a0 = __ldg(reinterpret_cast<const float4*>(g.kc0 + kco[i] + c * 32));
                                const float4 z = cur2[i];
                                v.x = fmaf(a1.x, v.x, fmaf(a3.x, z.x, a0.x)); v.y = fmaf(a1.y, v.y, fmaf(a3.y, z.y, a0.y));
                                v.z = fmaf(a1.z, v.z, fmaf(a3.z, z.z, a0.z)); v.w = fmaf(a1.w, v.w, fmaf(a3.w, z.w, a0.w));
                            }
                            if (has_coef) {
                                const float4 a = __ldg(reinterpret_cast<const float4*>(sc[i] + c * 32));
                                const float4 b = __ldg(reinterpret_cast<const float4*>(sh[i] + c * 32));
                                v.x = fmaf(v.x, a.x, b.x); v.y = fmaf(v.y, a.y, b.y); v.z = fmaf(v.z, a.z, b.z); v.w = fmaf(v.w, a.w, b.w);
                            }
                            if (ACT != PTRB200_AF_NONE) {
                                const int af = ACT < 0 ? g.act : ACT;
                                v.x = activate(af, v.x).y; v.y = activate(af, v.y).y; v.z = activate(af, v.z).y; v.w = activate(af, v.w).y;
                            }
                            if (MODE == RG_FWD && g.drop.thr) {
                                const uint64_t d = dropout_draw4(g.drop.key, dq[i] + c * 8);
                                v.x = ((uint32_t)(d) & 0xffffu) >= g.drop.thr ? v.x * g.drop.scale : 0.0f;
                                v.y = ((uint32_t)(d >> 16) & 0xffffu) >= g.drop.thr ? v.y * g.drop.scale : 0.0f;
                                v.z = ((uint32_t)(d >> 32) & 0xffffu) >= g.drop.thr ? v.z * g.drop.scale : 0.0f;
                                v.w = ((uint32_t)(d >> 48)) >= g.drop.thr ? v.w * g.drop.scale : 0.0f;
                            }
                            if (MODE == RG_FWD && aout[i]) *reinterpret_cast<float4*>(aout[i] + c * 32) = v;
                        } else v = make_float4(0.f, 0.f, 0.f, 0.f);
                        store_split(a_hi, a_hi + 16384, sw_[i], v, PASSES == 3, PASSES == 1 && g.round_bf16 != 0);
                    }
                    tc::fence_proxy_async();
                    __syncwarp();
                    if (lane == 0) tc::mbar_arrive(aready + s);
                }
            }
        } else {
            // ================================ producer warps ================================
            const int ptid = tid - RW_EPI_WARPS * 32;
            const int j4 = (ptid & 7) * 4;                              // first column of this thread's 16-byte unit inside a chunk
            int r_[RW_PU];
            uint32_t sw_[RW_PU];
    #pragma unroll
            for (int i = 0; i < RW_PU; ++i) { r_[i] = (ptid >> 3) + i * (RW_PRODUCERS / 8); sw_[i] = tc::swz_offset(r_[i], ptid & 7); }
            const int total_q = my_tiles * nchunks;
            const bool has_coef = g.scale != nullptr;
            const bool per_group = has_coef && g.gr_prev < g.rows;
            const bool fused_dz = MODE == RG_DGRAD && g.P2 != nullptr;
            // A width that is not a multiple of 32 leaves the LAST K-chunk mostly empty (K = 100: 4 of its 32 columns).  With
            // the regular mapping (8 units per row) 7 of every 8 lanes would run the whole prologue on nothing, so that chunk
            // uses a unit-major mapping instead: unit jB = (ptid >> 7) + 4 i of row rB = ptid & 127 -- whole warps share jB
            // and only those below `vlast` run the prologue; units in [vlast, 8) are written as zeros (the MMAs read all four
            // K-steps of every chunk).
            const int lastc = nchunks - 1;
            const int vlast = (K - lastc * 32 + 3) >> 2;                // 16-byte units of the last chunk that hold data (1..8)
            // (forward only: the dgrad instantiation keeps the regular mapping, its fused staging already carries more live state)
            const bool partial = MODE == RG_FWD && vlast < 8;
            const int zfill = 8;                                        // units the last chunk's MMAs read
            const int rB = ptid & 127;
            int jB_[RW_PU];
    #pragma unroll
            for (int i = 0; i < RW_PU; ++i) jB_[i] = (ptid >> 7) + i * (RW_PRODUCERS / 128);
            float4 pre[RW_PU], pre2[RW_PU];
            size_t soff[RW_PU], soffB[RW_PU];                           // element offset of the thread's units in the tile being fetched
            bool ok[RW_PU], okB[RW_PU];
            auto point = [&](int it) {                                  // set soff/ok for tile `it`
                int r0, nr;
                rw_tile(g, blockIdx.x + it * gridDim.x, r0, nr);
    #pragma unroll
                for (int i = 0; i < RW_PU; ++i) {
                    ok[i] = r_[i] < nr; soff[i] = (size_t)(r0 + min(r_[i], nr - 1)) * K + j4;
                    okB[i] = rB < nr && jB_[i] < vlast; soffB[i] = (size_t)(r0 + min(rB, nr - 1)) * K + lastc * 32 + min(jB_[i], vlast - 1) * 4;
                }
            };
            auto fetch = [&](int c) {
                if (partial && c == lastc) {
    #pragma unroll
                    for (int i = 0; i < RW_PU; ++i) {
                        pre[i] = okB[i] ? ldg_a4<XB>(g.P, soffB[i]) : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (MODE == RG_DGRAD) pre2[i] = (fused_dz && okB[i]) ? __ldg(reinterpret_cast<const float4*>(g.P2 + soffB[i])) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                    return;
                }
                const bool kv = c * 32 + j4 < K;
    #pragma unroll
                for (int i = 0; i < RW_PU; ++i) {
                    pre[i] = (ok[i] && kv) ? ldg_a4<XB>(g.P, soff[i] + c * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (MODE == RG_DGRAD) pre2[i] = (fused_dz && ok[i] && kv) ? __ldg(reinterpret_cast<const float4*>(g.P2 + soff[i] + c * 32)) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            };
            // prologue of one 16-byte unit: [dZ = k1*dY + k3*Z + k0] -> scale/shift -> activation -> dropout -> by-product store
            auto xform = [&](float4 v, const float4 z, const float* scp, const float* shp, size_t kcoff, uint64_t dquad, float* aoutp) -> float4 {
                if (MODE == RG_DGRAD && fused_dz) {           // dZ = k1*dY + k3*Z + k0
                    const float4 a1 = __ldg(reinterpret_cast<const float4*>(g.kc1 + kcoff));
                    const float4 a3 = __ldg(reinterpret_cast<const float4*>(g.kc3 + kcoff));
                    const float4 a0 = __ldg(reinterpret_cast<const float4*>(g.kc0 + kcoff));
                    v.x = fmaf(a1.x, v.x, fmaf(a3.x, z.x, a0.x)); v.y = fmaf(a1.y, v.y, fmaf(a3.y, z.y, a0.y));
                    v.z = fmaf(a1.z, v.z, fmaf(a3.z, z.z, a0.z)); v.w = fmaf(a1.w, v.w, fmaf(a3.w, z.w, a0.w));
                }
                if (has_coef) {
                    const float4 a = __ldg(reinterpret_cast<const float4*>(scp));
                    const float4 b = __ldg(reinterpret_cast<const float4*>(shp));
                    v.x = fmaf(v.x, a.x, b.x); v.y = fmaf(v.y, a.y, b.y); v.z = fmaf(v.z, a.z, b.z); v.w = fmaf(v.w, a.w, b.w);
                }
                if (ACT != PTRB200_AF_NONE) {
                    const int af = ACT < 0 ? g.act : ACT;
                    v.x = activate(af, v.x).y; v.y = activate(af, v.y).y; v.z = activate(af, v.z).y; v.w = activate(af, v.w).y;
                }
                if (MODE == RG_FWD && g.drop.thr) {
                    const uint64_t d = dropout_draw4(g.drop.key, dquad);
                    v.x = ((uint32_t)(d) & 0xffffu) >= g.drop.thr ? v.x * g.drop.scale : 0.0f;
                    v.y = ((uint32_t)(d >> 16) & 0xffffu) >= g.drop.thr ? v.y * g.drop.scale : 0.0f;
                    v.z = ((uint32_t)(d >> 32) & 0xffffu) >= g.drop.thr ? v.z * g.drop.scale : 0.0f;
                    v.w = ((uint32_t)(d >> 48)) >= g.drop.thr ? v.w * g.drop.scale : 0.0f;
                }
                if (MODE == RG_FWD && aoutp) *reinterpret_cast<float4*>(aoutp) = v;
                return v;
            };
            if (total_q > 0) { point(0); fetch(0); }
            int q = 0;
            for (int it = 0; it < my_tiles; ++it) {
                int row0, nrows;
                rw_tile(g, blockIdx.x + it * gridDim.x, row0, nrows);
                // per-tile invariants of this thread's two rows
                bool live[RW_PU];
                float* aout[RW_PU];
                const float* sc[RW_PU];
                const float* sh[RW_PU];
                size_t kco[RW_PU];
                uint64_t dq[RW_PU];
    #pragma unroll
                for (int i = 0; i < RW_PU; ++i) {
                    live[i] = r_[i] < nrows;
                    const size_t e0 = (size_t)(row0 + min(r_[i], nrows - 1)) * K + j4;
                    aout[i] = (MODE == RG_FWD && g.a_out) ? g.a_out + e0 : nullptr;
                    const size_t co = per_group ? (size_t)((row0 + min(r_[i], nrows - 1)) / g.gr_prev) * K + j4 : (size_t)j4;
                    sc[i] = has_coef ? g.scale + co : nullptr;
                    sh[i] = has_coef ? g.shift + co : nullptr;
                    kco[i] = (fused_dz && g.gr_cur < g.rows) ? (size_t)((row0 + min(r_[i], nrows - 1)) / g.gr_cur) * K + j4 : (size_t)j4;
                    dq[i] = (uint64_t)e0 >> 2;
                }
    #pragma unroll (KT ? 8 : 1)
            for (int c = 0; c < nchunks; ++c, ++q) {
                    const int s = q & 1;
                    float4 cur[RW_PU], cur2[RW_PU];
    #pragma unroll
                    for (int i = 0; i < RW_PU; ++i) { cur[i] = pre[i]; cur2[i] = pre2[i]; }
                    if (q + 1 < total_q) {                              // prefetch the next chunk (possibly of the next tile)
                        if (c + 1 < nchunks) fetch(c + 1); else { point(it + 1); fetch(0); }
                    }
                    if (q >= 2) tc::mbar_wait(afree + s, ((q - 2) >> 1) & 1);
                    unsigned char* a_hi = a_ring + s * 32768;
                    if (partial && c == lastc) {
                        // unit-major mapping of the short last chunk: warps whose unit lies beyond `zfill` have nothing to do
    #pragma unroll
                        for (int i = 0; i < RW_PU; ++i) {
                            const int jB = jB_[i];
                            if (jB < zfill) {
                                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                                if (jB < vlast && rB < nrows) {
                                    const int col = lastc * 32 + jB * 4;
                                    const size_t e0 = (size_t)(row0 + rB) * K + col;
                                    const size_t co = (per_group ? (size_t)((row0 + rB) / g.gr_prev) * K : (size_t)0) + col;
                                    const size_t kc = ((fused_dz && g.gr_cur < g.rows) ? (size_t)((row0 + rB) / g.gr_cur) * K : (size_t)0) + col;
                                    v = xform(cur[i], cur2[i], has_coef ? g.scale + co : nullptr, has_coef ? g.shift + co : nullptr, kc,
                                              (uint64_t)e0 >> 2, (MODE == RG_FWD && g.a_out) ? g.a_out + e0 : nullptr);
                                }
                                store_split(a_hi, a_hi + 16384, tc::swz_offset(rB, jB), v, PASSES == 3, PASSES == 1 && g.round_bf16 != 0);
                            }
                        }
                    } else {
                        const bool kv = c * 32 + j4 < K;
    #pragma unroll
                        for (int i = 0; i < RW_PU; ++i) {
                            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (live[i] && kv)
                                v = xform(cur[i], cur2[i], has_coef ? sc[i] + c * 32 : nullptr, has_coef ? sh[i] + c * 32 : nullptr,
                                          kco[i] + c * 32, dq[i] + c * 8, aout[i] ? aout[i] + c * 32 : nullptr);
                            store_split(a_hi, a_hi + 16384, sw_[i], v, PASSES == 3, PASSES == 1 && g.round_bf16 != 0);
                        }
                    }
                    tc::fence_proxy_async();
                    __syncwarp();
                    if (lane == 0) tc::mbar_arrive(aready + s);
                }
            }
        }
    } else {
        tc::setmaxnreg_dec<RW_CONS_REGS>();
        if (my_tiles > 0) {
        // ================================ consumer warps (0..7) ================================
        // warpgroup wg multiplies rows [64 wg, +64) of every tile; the accumulator of the tile stays in registers
        const int wg = warp >> 2;
        if (tid == 0) {
            tc::mbar_expect_tx(wfull, (uint32_t)(nchunks * wchunk * (PASSES == 3 ? 2 : 1)));
            for (int c = 0; c < nchunks; ++c) {
                tc::bulk_g2s(w_hi + (size_t)c * wchunk, g.b_img_hi + (size_t)c * wchunk, wchunk, wfull);
                if (PASSES == 3) tc::bulk_g2s(w_lo + (size_t)c * wchunk, g.b_img_lo + (size_t)c * wchunk, wchunk, wfull);
            }
        }
        tc::mbar_wait(wfull, 0);
        const uint32_t a_base = tc::smem_u32(a_ring) + wg * 8192, wh_base = tc::smem_u32(w_hi), wl_base = tc::smem_u32(w_lo);
        double acc1 = 0.0, acc2 = 0.0;                        // per-CTA column sums for column `tid` (tid < 256)
        tc::with_width(NP, [&](auto W) {
        constexpr int NPc = decltype(W)::value;
        int q = 0;
        for (int it = 0; it < my_tiles; ++it) {
            const int t = blockIdx.x + it * gridDim.x;
            int row0, nrows;
            rw_tile(g, t, row0, nrows);
            float acc[NPc / 2];
#pragma unroll
            for (int e = 0; e < NPc / 2; ++e) acc[e] = 0.0f;
    #pragma unroll (KT ? 8 : 1)
            for (int c = 0; c < nchunks; ++c, ++q) {
                const int s = q & 1;
                tc::mbar_wait(aready + s, (q >> 1) & 1);
                uint32_t a_addr = a_base + s * 32768, b_off = c * wchunk;
                // opaque to the optimiser: the descriptors are rebuilt at every chunk (a few integer ops) instead of being
                // hoisted out of the tile loop, where the unrolled chunks' descriptors outgrow the consumers' registers
                asm volatile("" : "+r"(a_addr), "+r"(b_off));
                const uint64_t ah = tc::smem_desc_sw128(a_addr, 1024), al = tc::smem_desc_sw128(a_addr + 16384, 1024);
                const uint64_t bh = tc::smem_desc_sw128(wh_base + b_off, 1024), bl = tc::smem_desc_sw128(wl_base + b_off, 1024);
                // four K-steps per chunk (+32 B along K inside the swizzle atom each; columns beyond K are staged as zeros)
                tc::wg_fence();
#pragma unroll
                for (int st = 0; st < 4; ++st) {
                    if (PASSES == 3) {
                        tc::mma_tf32<NPc>(acc, al + 2 * st, bh + 2 * st, 1u);
                        tc::mma_tf32<NPc>(acc, ah + 2 * st, bl + 2 * st, 1u);
                    }
                    tc::mma_tf32<NPc>(acc, ah + 2 * st, bh + 2 * st, 1u);
                }
                tc::wg_commit();
                // the MMAs of the previous chunk have completed: release its A stage
                tc::wg_wait<1>();
                if (c > 0) { __syncwarp(); if (lane == 0) tc::mbar_arrive(afree + (s ^ 1)); }
            }
            tc::wg_wait<0>();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(afree + ((q - 1) & 1));
            // ---- epilogue: registers -> (+bias | dropout mask) -> global rows, per-warp column sums ----
            const float* bias = g.bias;
            asm volatile("" : "+l"(bias));          // loaded per tile: hoisted over the tile loop the bias would hold NPc / 2 registers
            bool live[2];
            float* orow[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = wg * 64 + tc::acc_row(2 * h);
                live[h] = r < nrows;
                orow[h] = g.Out + (size_t)(row0 + min(r, nrows - 1)) * N;
            }
            if (MODE == RG_FWD) {
#pragma unroll
                for (int e = 0; e < NPc / 2; ++e) {
                    const int col = tc::acc_col(e);
                    if (col >= N) { acc[e] = 0.0f; continue; }
                    acc[e] += __ldg(bias + col);
                }
            } else if (g.drop.thr && (N & 3) == 0) {
                // Accumulators e..e+3 (e % 4 == 0) are columns col, col + 1 of rows r and r + 8; lanes l and l ^ 1 together
                // hold the four columns of one quad of the dropout stream, whose mask is one 64-bit draw.  Each lane draws
                // one of the two rows' quads (even lane: row r, odd lane: row r + 8) and passes its partner the 32 bits
                // of that draw the partner's columns use: one draw per four elements instead of one per element.
                const bool odd = lane & 1;
#pragma unroll
                for (int e = 0; e < NPc / 2; e += 4) {
                    const int col = tc::acc_col(e);
                    const uint64_t el = (uint64_t)(row0 + wg * 64 + tc::acc_row(e) + (odd ? 8 : 0)) * N + (col & ~3);
                    const uint64_t d = dropout_draw4(g.drop.key, el >> 2);
                    const uint32_t other = __shfl_xor_sync(0xffffffffu, odd ? (uint32_t)d : (uint32_t)(d >> 32), 1);
                    const uint32_t ur = odd ? other : (uint32_t)d;               // row r: 16 bits per column
                    const uint32_t ur8 = odd ? (uint32_t)(d >> 32) : other;      // row r + 8
                    if (col >= N) { acc[e] = acc[e + 1] = acc[e + 2] = acc[e + 3] = 0.0f; continue; }   // (N % 4 == 0: col + 1 < N)
                    acc[e] = (ur & 0xffffu) >= g.drop.thr ? acc[e] * g.drop.scale : 0.0f;
                    acc[e + 1] = (ur >> 16) >= g.drop.thr ? acc[e + 1] * g.drop.scale : 0.0f;
                    acc[e + 2] = (ur8 & 0xffffu) >= g.drop.thr ? acc[e + 2] * g.drop.scale : 0.0f;
                    acc[e + 3] = (ur8 >> 16) >= g.drop.thr ? acc[e + 3] * g.drop.scale : 0.0f;
                }
            } else {
#pragma unroll
                for (int e = 0; e < NPc / 2; ++e) {
                    const int col = tc::acc_col(e);
                    if (col >= N) { acc[e] = 0.0f; continue; }
                    if (g.drop.thr) {
                        const int r = wg * 64 + tc::acc_row(e);
                        acc[e] = dropout_keep(g.drop.key, (uint64_t)(row0 + r) * N + col, g.drop.thr) ? acc[e] * g.drop.scale : 0.0f;
                    }
                }
            }
            // a thread holds two adjacent columns of two rows per 8-column group: 8-byte stores when N is even
#pragma unroll
            for (int e = 0; e < NPc / 2; e += 2) {
                const int col = tc::acc_col(e), h = (e >> 1) & 1;
                if (!live[h] || col >= N) continue;
                if ((N & 1) == 0) *reinterpret_cast<float2*>(orow[h] + col) = make_float2(acc[e], acc[e + 1]);
                else { orow[h][col] = acc[e]; if (col + 1 < N) orow[h][col + 1] = acc[e + 1]; }
            }
            if (MODE == RG_FWD && x.stats_mode) {
                int sl = lane, sw = warp;
                asm volatile("" : "+r"(sl), "+r"(sw));  // per tile, like the bias: the NPc / 4 stat_sm offsets are not kept live
#pragma unroll
                for (int j = 0; j < NPc / 16; ++j) {
                    const float* w = acc + 8 * j;
                    // column sums over the warp's 16 rows: lanes with equal lane % 4 hold the same columns.
                    // s[p] = sum, s[4 + p] = sum of squares of the lane's column p over its two rows
                    float s[8];
#pragma unroll
                    for (int p = 0; p < 4; ++p) {              // p = 2 * (e >> 2) + (e & 1): the four columns of this lane
                        const int e0 = (p >> 1) * 4 + (p & 1), e1 = e0 + 2;
                        const float v0 = live[0] ? w[e0] : 0.0f, v1 = live[1] ? w[e1] : 0.0f;
                        s[p] = v0 + v1; s[4 + p] = v0 * v0 + v1 * v1;
                    }
                    // reduce-scatter over the 8 lanes of equal lane % 4, partners lane ^ 4, ^ 8, ^ 16: each step adds the
                    // same pairs a butterfly all-reduce adds (so the sums are the same bits) but keeps only half of the
                    // values, 7 shuffles instead of 24.  Lane sl ends with the full sum of value 4 b2 + 2 b3 + b4 (bits of sl).
#pragma unroll
                    for (int st = 0; st < 3; ++st) {
                        const int h = 4 >> st, o = 4 << st;
                        const bool up = sl & o;
#pragma unroll
                        for (int i = 0; i < h; ++i) {
                            float keep = s[i], send = s[i + h];
                            if (up) { const float t = keep; keep = send; send = t; }
                            s[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                        }
                    }
                    const int v = ((sl >> 2) & 1) * 4 + ((sl >> 3) & 1) * 2 + ((sl >> 4) & 1), p = v & 3;
                    const int col = j * 16 + (p >> 1) * 8 + 2 * (sl & 3) + (p & 1);
                    stat_sm[(sw * NP + col) * 2 + (v >> 2)] = s[0];
                }
                asm volatile("bar.sync 2, 256;" ::: "memory");               // the 8 warps' column sums are in smem
                if (tid < N) {
                    double s1 = 0.0, s2 = 0.0;
#pragma unroll
                    for (int w = 0; w < RW_EPI_WARPS; ++w) { s1 += (double)stat_sm[(w * NP + tid) * 2]; s2 += (double)stat_sm[(w * NP + tid) * 2 + 1]; }
                    if (x.stats_mode == 2) {
                        double* p = g.partials + ((size_t)t * N + tid) * 2;
                        p[0] = s1; p[1] = s2;
                    } else { acc1 += s1; acc2 += s2; }
                }
                asm volatile("bar.sync 2, 256;" ::: "memory");               // smem free for the next tile
            }
        }
        });
        if (MODE == RG_FWD && x.stats_mode == 1 && tid < N) {
            double* p = g.partials + ((size_t)blockIdx.x * N + tid) * 2;
            p[0] = acc1; p[1] = acc2;
        }
        } else if (MODE == RG_FWD && x.stats_mode == 1 && tid < N) {      // a CTA without tiles contributes zero sums
            double* p = g.partials + ((size_t)blockIdx.x * N + tid) * 2;
            p[0] = 0.0; p[1] = 0.0;
        }
    }
}

// --------------------------------------------------------------------------------------------
// weight gradient: dW[N,K] = sum_r dZ[r,n] * Ain[r,k],  Ain = drop(act(P*scale+shift)).
// The contraction runs over rows.  wgmma reads 32-bit operands K-major only, so both operands are staged
// transposed: dZ^T [128 rows n][R rows r] and Ain^T [KP rows k][R rows r], one 128-byte SWIZZLE_128B chunk per
// operand row (R <= 32), 8 rows r per MMA K-step.  Persistent CTAs accumulate their row tiles in registers and
// write one partial per CTA.
// --------------------------------------------------------------------------------------------
struct WgradArgs {
    // normalisation backward folded in (Z2 != NULL): dZ = k1*dZ_in + k3*Z2 + k0 per (group, column); dZ_in then holds dY
    const float* Z2;       // [rows, N] pre-activation of this layer, or NULL
    const float *kc1, *kc3, *kc0;
    int gr_cur;
    const float* dZ;       // [rows, N]
    const float* P;        // [rows, K]
    const float* scale;    // [Gp, K] or NULL
    const float* shift;
    int act, gr_prev;
    DropCfg drop;
    float* partials;       // [gridDim.x, N, K]
    int rows, K, N;
    int KP;                // K rounded up to 16 (MMA N extent)
    int N_full, K_full;    // full widths of dZ and of the layer input; N / K / KP above describe ONE block:
    int kb;                // CTA (x, y, z) owns dZ columns [128*y, +N) and input columns [kb*z, +K)
    int tile_rows;         // R: rows per tile (multiple of 8, <= 32)
    int stages;            // raw-tile ring depth (2..WG_MAX_STAGES), chosen by the host to fit shared memory
    int round_bf16;        // PTRB200_MATH_BF16: both operands rounded to bf16
};

constexpr int WG_THREADS = 512;       // four warpgroups: all stage the operands, each multiplies a quarter of the dW block
constexpr int WG_MAX_STAGES = 4;      // raw-tile ring depth bound (TMA bulk copies in flight)

// Persistent and TMA-fed.  Row tiles of dZ and of the layer input are contiguous in HBM, so warp 0 streams them into
// a raw shared-memory ring with 1-D bulk copies (cp.async.bulk + mbarrier complete_tx) `stages` tiles ahead.  All
// threads turn a raw tile into transposed hi/lo TF32 operand buffers (double buffered).  A tile's MMAs are committed
// without a wait and run while the next tile is staged into the other buffer; each thread waits for its warpgroup's
// MMAs only after that staging, and the CTA barrier behind the wait frees the buffer they read for the tile after.
// Warpgroup w multiplies dZ columns [64 (w & 1), +64) by the input columns of half (w >> 1) of the block.
// XB: g.P holds bf16 features (layer 0).  The raw ring carries them at 2 bytes each and the staging widens them while
// transposing.  A bulk copy needs 16-byte sizes and addresses; a P tile (or, column-blocked, a row segment) that does not
// have them is copied by hand, as odd-sized dZ tiles are.
template <int PASSES, bool XB = false>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_tc_kernel(WgradArgs g) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // aligned up by an offset from smem_raw (not through an integer cast of the pointer), so the compiler still knows
    // every buffer below is shared memory and stages the operands with LDS / STS instead of generic loads and stores
    unsigned char* base = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const int R = g.tile_rows;
    // column block of this CTA: dZ columns [m0, m0+N), layer-input columns [kk0, kk0+K)
    const int m0 = blockIdx.y * 128, kk0 = blockIdx.z * g.kb;
    const int N = min(128, g.N_full - m0), K = min(g.kb, g.K_full - kk0), KP = ((K + 15) / 16) * 16;
    const int Nmax = min(128, g.N_full), Kmax = min(g.kb, g.K_full);       // buffer geometry is the same in every CTA
    const bool blocked = gridDim.y > 1 || gridDim.z > 1;
    const int KPmax = ((Kmax + 15) / 16) * 16;
    const int zop_bytes = 128 * 128, pop_bytes = KPmax * 128;  // one 128-byte chunk (32 rows r) per operand row
    const int op_bytes = (zop_bytes + pop_bytes) * (PASSES == 3 ? 2 : 1);
    const bool fused_dz = g.Z2 != nullptr;
    const int rawz1 = ((R * Nmax * 4 + 127) / 128) * 128;
    constexpr int PB = XB ? 2 : 4;                           // bytes per layer-input element in the raw ring
    const int rawz_bytes = rawz1 * (fused_dz ? 2 : 1), rawp_bytes = ((R * Kmax * PB + 127) / 128) * 128;   // [dY | Z2] then the layer input
    const int stages = g.stages;
    unsigned char* opbuf = base;                             // [2][dZ hi | dZ lo | P hi | P lo]
    unsigned char* rawbuf = opbuf + 2 * op_bytes;            // [stages][rawz + rawp]
    unsigned char* tail = rawbuf + stages * (rawz_bytes + rawp_bytes);
    uint64_t* full = reinterpret_cast<uint64_t*>(tail);      // [stages] raw tile landed (TMA complete_tx)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    if (tid == 0) {
        for (int s = 0; s < stages; ++s) tc::mbar_init(full + s, 1);
        tc::mbar_fence_init();
    }
    const int ntiles = (g.rows + R - 1) / R;
    const int my_tiles = blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    // bf16 layer input: can its tiles travel by bulk copy?  (fp32: always -- K % 4 == 0 and 16-byte aligned rows)
    bool p_bulk_ok = true;
    if constexpr (XB) p_bulk_ok = ((reinterpret_cast<uintptr_t>(g.P) & 15) == 0) && (!blocked || (K % 8 == 0 && g.K_full % 8 == 0));
    auto p_bulk = [&](int nrows) -> bool {
        if constexpr (XB) return p_bulk_ok && (blocked || (((uint32_t)nrows * K * 2) & 15) == 0);
        else return true;
    };

    // whole-warp call (warp 0): un-blocked tiles are contiguous in HBM (one copy per operand, issued by lane 0);
    // column blocks are row segments, one pair of copies per row, issued by lane = row
    auto issue_load = [&](int it, int s) {
        const int t = blockIdx.x + it * gridDim.x;
        const int row0 = t * R, nrows = min(R, g.rows - row0);
        const bool pbk = p_bulk(nrows);
        const uint32_t zb = (uint32_t)nrows * N * 4, pb = pbk ? (uint32_t)nrows * K * PB : 0u;
        unsigned char* rz = rawbuf + s * (rawz_bytes + rawp_bytes);
        if (!blocked) {
            if (lane == 0) {
                if ((zb & 15) == 0) {
                    tc::mbar_expect_tx(full + s, (fused_dz ? 2 * zb : zb) + pb);
                    tc::bulk_g2s(rz, g.dZ + (size_t)row0 * N, zb, full + s);
                    if (fused_dz) tc::bulk_g2s(rz + rawz1, g.Z2 + (size_t)row0 * N, zb, full + s);
                } else {
                    tc::mbar_expect_tx(full + s, pb);     // odd-sized dZ tail tile: the threads copy it by hand
                }
                if constexpr (XB) { if (pbk) tc::bulk_g2s(rz + rawz_bytes, reinterpret_cast<const uint16_t*>(g.P) + (size_t)row0 * K, pb, full + s); }
                else tc::bulk_g2s(rz + rawz_bytes, g.P + (size_t)row0 * K, pb, full + s);
            }
        } else {
            const bool z_bulk = (N & 3) == 0;            // a dZ row segment must be a multiple of 16 bytes for TMA
            if (lane == 0) tc::mbar_expect_tx(full + s, (z_bulk ? zb : 0u) + pb);
            __syncwarp();
            if (lane < nrows) {
                if (z_bulk) tc::bulk_g2s(rz + (size_t)lane * N * 4, g.dZ + (size_t)(row0 + lane) * g.N_full + m0, (uint32_t)N * 4, full + s);
                if constexpr (XB) {
                    if (pbk) tc::bulk_g2s(rz + rawz_bytes + (size_t)lane * K * 2, reinterpret_cast<const uint16_t*>(g.P) + (size_t)(row0 + lane) * g.K_full + kk0,
                                          (uint32_t)K * 2, full + s);
                } else tc::bulk_g2s(rz + rawz_bytes + (size_t)lane * K * 4, g.P + (size_t)(row0 + lane) * g.K_full + kk0, (uint32_t)K * 4, full + s);
            }
            __syncwarp();
        }
    };

    const bool plain_p = !g.scale && g.act == PTRB200_AF_NONE && !g.drop.thr;   // layer input already materialised
    const bool single_group = fused_dz && g.gr_cur >= g.rows;
    float* coef = reinterpret_cast<float*>(tail + 128);      // [3][128] k1 | k3 | k0 of the one statistics group
    {   // padding (columns beyond N resp. K, rows r beyond R) is zero for the whole kernel; the coefficient rows of the
        // one statistics group are staged once
        const uint32_t op_s = tc::smem_u32(opbuf);
        for (int e = tid; e < 2 * op_bytes / 16; e += WG_THREADS) tc::sts128(op_s + (uint32_t)e * 16u, make_float4(0.f, 0.f, 0.f, 0.f));
        if (single_group)
            for (int e = tid; e < 3 * 128; e += WG_THREADS) {
                const int which = e >> 7, n = e & 127;
                const float* src = which == 0 ? g.kc1 : which == 1 ? g.kc3 : g.kc0;
                coef[e] = n < N ? __ldg(src + m0 + n) : 0.0f;
            }
        __syncthreads();
    }
    if (warp == 0)
        for (int it = 0; it < min(stages, my_tiles); ++it) issue_load(it, it);

    auto put = [&](unsigned char* hi, unsigned char* lo, uint32_t off, float4 v) {
        if (PASSES == 3) {
            float4 h, l;
            tc::split_tf32(v.x, h.x, l.x); tc::split_tf32(v.y, h.y, l.y); tc::split_tf32(v.z, h.z, l.z); tc::split_tf32(v.w, h.w, l.w);
            *reinterpret_cast<float4*>(hi + off) = h;
            *reinterpret_cast<float4*>(lo + off) = l;
        } else {
            if (g.round_bf16) v = make_float4(bf16_rn(v.x), bf16_rn(v.y), bf16_rn(v.z), bf16_rn(v.w));
            *reinterpret_cast<float4*>(hi + off) = v;
        }
    };
    // warpgroup tile: dZ rows [64 mh, +64) x input columns [c0, c0 + KPh).  Both column halves have the same compile-time
    // width KPh = ceil(KP / 32) * 16: the second starts at KP - KPh (overlapping the first by at most 16 columns, which it
    // computes but does not write), so no operand row beyond KP is read
    const int mh = wg & 1, KPh = ((KP / 16 + 1) / 2) * 16, c0 = (wg >> 1) ? KP - KPh : 0, cw0 = (wg >> 1) ? KPh : 0;
    const int RQ = R / 4;                                    // 16-byte units (4 rows r) per operand row
    // a thread stages dZ^T column n = tid & 127 of every tile (its units u = tid + 512 j, and 512 % 128 == 0), so the one
    // statistics group's coefficients of that column stay in registers
    const float k1n = single_group ? coef[tid & 127] : 0.0f, k3n = single_group ? coef[128 + (tid & 127)] : 0.0f,
                k0n = single_group ? coef[256 + (tid & 127)] : 0.0f;
    // the layer-input units of a thread, u = tid + 512 j, as (u % KP, u / KP): stepped instead of divided at every unit
    const int pk0 = tid % KP, pq0 = tid / KP, pkstep = WG_THREADS % KP, pqstep = WG_THREADS / KP;

    tc::with_width(KPh, [&](auto W) {
    constexpr int NPc = decltype(W)::value;
    float acc[NPc / 2];
#pragma unroll
    for (int e = 0; e < NPc / 2; ++e) acc[e] = 0.0f;
    // pins the accumulators in place while MMAs run asynchronously over the staging code (no copies of them in between)
    auto fence_acc = [&]() {
#pragma unroll
        for (int e = 0; e < NPc / 2; ++e) asm volatile("" : "+f"(acc[e])::"memory");
    };
    fence_acc();
    for (int it = 0; it < my_tiles; ++it) {
        const int t = blockIdx.x + it * gridDim.x, o = it & 1, s = it % stages;
        const int row0 = t * R, nrows = min(R, g.rows - row0);
        const float* rz = reinterpret_cast<const float*>(rawbuf + s * (rawz_bytes + rawp_bytes));
        const float* rp = reinterpret_cast<const float*>(rawbuf + s * (rawz_bytes + rawp_bytes) + rawz_bytes);
        if (blocked ? (N & 3) != 0 : (((uint32_t)nrows * N * 4) & 15) != 0) {   // dZ not TMA-sized: copy by hand
            float* rzw = const_cast<float*>(rz);
            for (int e = tid; e < nrows * N; e += WG_THREADS) rzw[e] = g.dZ[(size_t)(row0 + e / N) * g.N_full + m0 + e % N];
            __syncthreads();
        }
        if constexpr (XB) {
            if (!p_bulk(nrows)) {                            // bf16 layer input not TMA-sized or -aligned: copy by hand
                uint16_t* rpw = reinterpret_cast<uint16_t*>(rawbuf + s * (rawz_bytes + rawp_bytes) + rawz_bytes);
                const uint16_t* src = reinterpret_cast<const uint16_t*>(g.P);
                for (int e = tid; e < nrows * K; e += WG_THREADS) rpw[e] = src[(size_t)(row0 + e / K) * g.K_full + kk0 + e % K];
                __syncthreads();
            }
        }
        tc::mbar_wait(full + s, (it / stages) & 1);
        unsigned char* zh = opbuf + o * op_bytes;
        unsigned char* zl = zh + zop_bytes;
        unsigned char* ph = zh + (PASSES == 3 ? 2 : 1) * zop_bytes;
        unsigned char* pl = ph + pop_bytes;
        // ---- dZ^T: unit (n, q) = dZ[4q .. 4q+3][n] ----
        for (int u = tid; u < 128 * RQ; u += WG_THREADS) {
            const int n = u & 127, qq = u >> 7;
            if (n >= N) continue;
            float v[4];
            const size_t grp_off_base = (size_t)m0 + n;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = qq * 4 + e;
                float x = 0.0f;
                if (r < nrows) {
                    x = rz[r * N + n];
                    if (fused_dz) {                                  // host guarantees N % 4 == 0 here
                        const float z = rz[rawz1 / 4 + r * N + n];
                        float a1, a3, a0;
                        if (single_group) { a1 = k1n; a3 = k3n; a0 = k0n; }
                        else {
                            const size_t go = (size_t)((row0 + r) / g.gr_cur) * g.N_full + grp_off_base;
                            a1 = __ldg(g.kc1 + go); a3 = __ldg(g.kc3 + go); a0 = __ldg(g.kc0 + go);
                        }
                        x = fmaf(a1, x, fmaf(a3, z, a0));
                    }
                }
                v[e] = x;
            }
            put(zh, zl, tc::swz_offset(n, qq), make_float4(v[0], v[1], v[2], v[3]));
        }
        // ---- layer input^T: unit (k, q) = Ain[4q .. 4q+3][k] ----
        for (int u = tid, k = pk0, qq = pq0; u < KP * RQ; u += WG_THREADS, k += pkstep, qq += pqstep) {
            if (k >= KP) { k -= KP; ++qq; }                 // (k, qq) = (u % KP, u / KP)
            if (k >= K) continue;
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = qq * 4 + e;
                float x = 0.0f;
                if (r < nrows) {
                    if constexpr (XB) x = __uint_as_float((uint32_t)reinterpret_cast<const uint16_t*>(rp)[r * K + k] << 16);
                    else x = rp[r * K + k];
                    if (!plain_p) {
                        const int row = row0 + r, col = kk0 + k;
                        if (g.scale) {
                            const size_t co = (g.gr_prev < g.rows ? (size_t)(row / g.gr_prev) * g.K_full : 0) + col;
                            x = fmaf(x, __ldg(g.scale + co), __ldg(g.shift + co));
                        }
                        if (g.act != PTRB200_AF_NONE) x = activate(g.act, x).y;
                        if (g.drop.thr) x = dropout_keep(g.drop.key, (uint64_t)row * g.K_full + col, g.drop.thr) ? x * g.drop.scale : 0.0f;
                    }
                }
                v[e] = x;
            }
            put(ph, pl, tc::swz_offset(k, qq), make_float4(v[0], v[1], v[2], v[3]));
        }
        // Tile it-1's MMAs ran while this tile was staged.  Once every warpgroup has waited for its own and passed the
        // barrier, operand buffer o ^ 1 -- which all four warpgroups read -- is free for tile it+1.
        tc::wg_wait<0>();
        fence_acc();
        tc::fence_proxy_async();
        __syncthreads();
        if (warp == 0 && it + stages < my_tiles) issue_load(it + stages, s);   // raw slot s is drained
        const uint32_t a_s = tc::smem_u32(zh) + mh * 8192, b_s = tc::smem_u32(ph) + c0 * 128;
        const uint64_t ah = tc::smem_desc_sw128(a_s, 1024), bh = tc::smem_desc_sw128(b_s, 1024);
        const uint64_t al = tc::smem_desc_sw128(a_s + zop_bytes, 1024), bl = tc::smem_desc_sw128(b_s + pop_bytes, 1024);
        // four K-steps of 8 rows r (+32 B each): rows beyond the tile are zero in the operand buffers
        tc::wg_fence();
#pragma unroll
        for (int st = 0; st < 4; ++st) {
            if (PASSES == 3) {
                tc::mma_tf32<NPc>(acc, al + 2 * st, bh + 2 * st, 1u);
                tc::mma_tf32<NPc>(acc, ah + 2 * st, bl + 2 * st, 1u);
            }
            tc::mma_tf32<NPc>(acc, ah + 2 * st, bh + 2 * st, 1u);
        }
        tc::wg_commit();
        fence_acc();
    }
    tc::wg_wait<0>();
    fence_acc();
    // ---- epilogue: this CTA's partial dW[n][k] ----
    float* dst = g.partials + (size_t)blockIdx.x * g.N_full * g.K_full + (size_t)m0 * g.K_full + kk0;
#pragma unroll
    for (int e = 0; e < NPc / 2; ++e) {
        const int n = mh * 64 + tc::acc_row(e), k = c0 + tc::acc_col(e);
        if (n < N && k >= cw0 && k < K) dst[(size_t)n * g.K_full + k] = acc[e];
    }
    });
}

}  // namespace ptrb200
