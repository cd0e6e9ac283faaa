// letor_float.cuh -- decimal token -> float64, rounded exactly as Python's float() rounds it (correctly, to nearest
// even).  __host__ __device__: the LETOR parser inlines it on the device and a host build tests the same code
// (tests/test_letor_parse.py).
//
// Grammar: [+-]? (digits [. digits*]? | . digits) ([eE] [+-]? digits)?  -- the tokens LETOR files hold.  Python also
// accepts inf / nan spellings and '_' digit separators; those are rejected here as malformed.
//
// Method.  The significand's first 19 significant digits are read into a uint64 w and the value is w * 10^q.
//   1. Clinger's fast path: w <= 2^53 and 0 <= q <= 22 -- w and 10^q are exact doubles, so one IEEE multiply is the
//      correctly rounded result.  (Clinger's divide for q < 0 is left to step 2: a float64 divide is a subroutine call
//      on the device, and its register save would spill in the parse kernel.)
//   2. Otherwise Eisel-Lemire: the 128-bit truncated 5^q (letor_pow5.cuh) times w, as in Lemire, "Number Parsing at a
//      Gigabyte per Second" (2021).  For an exact w this product always decides the rounding (Mushtak & Lemire, "Fast
//      Number Parsing Without Fallback", 2023).
//   3. More than 19 significant digits with a non-zero digit dropped: the value lies in (w, w+1) * 10^q.  If w and
//      w+1 round to the same double, that double is the answer; if not, the token is reported as undecided
//      (LETOR_DEC_HOST) and the caller re-reads it with Python's float().  No result is ever approximated.
#pragma once
#include <stdint.h>
#include <string.h>

#include "letor_pow5.cuh"

namespace ptrb200 {

enum { LETOR_DEC_OK = 0, LETOR_DEC_BAD = 1, LETOR_DEC_HOST = 2 };

static const uint64_t letor_pow5_host[] = {PTRB200_LETOR_POW5_DATA};
#ifdef __CUDACC__
static __device__ const uint64_t letor_pow5_dev[] = {PTRB200_LETOR_POW5_DATA};
#endif

__host__ __device__ __forceinline__ uint64_t letor_pow5(int i) {
#ifdef __CUDA_ARCH__
    return letor_pow5_dev[i];
#else
    return letor_pow5_host[i];
#endif
}

#define PTRB200_LETOR_POW10_DATA 1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, \
                                 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22
static const double letor_pow10_host[] = {PTRB200_LETOR_POW10_DATA};       // exact doubles: 10^k = 2^k * 5^k, 5^22 < 2^53
#ifdef __CUDACC__
static __device__ const double letor_pow10_dev[] = {PTRB200_LETOR_POW10_DATA};
#endif

__host__ __device__ __forceinline__ double letor_pow10(int i) {
#ifdef __CUDA_ARCH__
    return letor_pow10_dev[i];
#else
    return letor_pow10_host[i];
#endif
}

__host__ __device__ __forceinline__ void mul64x64(uint64_t a, uint64_t b, uint64_t& hi, uint64_t& lo) {
#ifdef __CUDA_ARCH__
    hi = __umul64hi(a, b);
    lo = a * b;
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    hi = (uint64_t)(p >> 64);
    lo = (uint64_t)p;
#endif
}

__host__ __device__ __forceinline__ int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

// Eisel-Lemire for binary64: the IEEE bit pattern (without sign) of w * 10^q, w != 0.
__host__ __device__ __forceinline__ uint64_t eisel_lemire(uint64_t w, int q) {
    if (q < PTRB200_LETOR_POW5_QMIN) return 0;                      // w < 10^19: below half the least subnormal
    if (q > PTRB200_LETOR_POW5_QMAX) return 0x7ffull << 52;         // w >= 1: above the largest double
    const int lz = clz64(w);
    w <<= lz;
    const int idx = 2 * (q - PTRB200_LETOR_POW5_QMIN);
    uint64_t hi, lo;
    mul64x64(w, letor_pow5(idx), hi, lo);
    const uint64_t precision_mask = 0xffffffffffffffffull >> 55;    // 52 explicit bits + 3
    if ((hi & precision_mask) == precision_mask) {                  // the low word of 5^q can still carry into hi
        uint64_t hi2, lo2;
        mul64x64(w, letor_pow5(idx + 1), hi2, lo2);
        lo += hi2;
        if (hi2 > lo) ++hi;
    }
    const int upperbit = (int)(hi >> 63);
    const int shift = upperbit + 64 - 52 - 3;
    uint64_t mant = hi >> shift;
    int power2 = (int)((((152170 + 65536) * q) >> 16) + 63) + upperbit - lz + 1023;
    if (power2 <= 0) {                                              // subnormal or zero
        if (-power2 + 1 >= 64) return 0;
        mant >>= -power2 + 1;
        mant += (mant & 1);
        mant >>= 1;
        power2 = (mant < (1ull << 52)) ? 0 : 1;
        return ((uint64_t)power2 << 52) | (mant & ((1ull << 52) - 1));
    }
    // exactly halfway between two doubles: only possible for small |q|, where 5^q is exact; round to even
    if (lo <= 1 && q >= -4 && q <= 23 && (mant & 3) == 1 && (mant << shift) == hi) mant &= ~1ull;
    mant += (mant & 1);
    mant >>= 1;
    if (mant >= (2ull << 52)) { mant = 1ull << 52; ++power2; }
    mant &= ~(1ull << 52);
    if (power2 >= 0x7ff) return 0x7ffull << 52;
    return ((uint64_t)power2 << 52) | mant;
}

__host__ __device__ __forceinline__ bool is_digit(char c) { return c >= '0' && c <= '9'; }

struct DecResult { int status; double value; };   // status LETOR_DEC_*; value 0 unless LETOR_DEC_OK

// Parse [p, end): LETOR_DEC_OK, LETOR_DEC_BAD (not a decimal number) or LETOR_DEC_HOST (undecided, see 3. above).
__host__ __device__ __forceinline__ DecResult parse_decimal(const char* p, const char* end) {
    bool neg = false;
    if (p < end && (*p == '+' || *p == '-')) { neg = *p == '-'; ++p; }
    uint64_t w = 0;
    int sig = 0;                // significant digits kept in w (leading zeros are not significant)
    int q = 0;                  // decimal exponent of w
    int ndig = 0;               // mantissa digits seen
    bool dropped = false;       // a non-zero digit beyond the 19th significant one
    for (; p < end && is_digit(*p); ++p, ++ndig) {
        const int d = *p - '0';
        if (sig < 19) { if (w || d) { w = w * 10 + d; ++sig; } }
        else { ++q; dropped |= d != 0; }
    }
    if (p < end && *p == '.') {
        for (++p; p < end && is_digit(*p); ++p, ++ndig) {
            const int d = *p - '0';
            if (sig < 19) { if (w || d) { w = w * 10 + d; ++sig; } --q; }
            else dropped |= d != 0;
        }
    }
    if (ndig == 0) return {LETOR_DEC_BAD, 0.0};
    if (p < end && (*p == 'e' || *p == 'E')) {
        ++p;
        bool eneg = false;
        if (p < end && (*p == '+' || *p == '-')) { eneg = *p == '-'; ++p; }
        if (p == end || !is_digit(*p)) return {LETOR_DEC_BAD, 0.0};
        int e = 0;
        for (; p < end && is_digit(*p); ++p) if (e < 100000) e = e * 10 + (*p - '0');   // saturates far outside [-342, 308]
        q += eneg ? -e : e;
    }
    if (p != end) return {LETOR_DEC_BAD, 0.0};
    uint64_t bits = 0;
    if (w != 0) {
        if (!dropped && w <= (1ull << 53) && q >= 0 && q <= 22) {
            const double v = (double)w * letor_pow10(q);
            return {LETOR_DEC_OK, neg ? -v : v};
        }
        bits = eisel_lemire(w, q);
        if (dropped && eisel_lemire(w + 1, q) != bits) return {LETOR_DEC_HOST, 0.0};   // w + 1 <= 10^19 < 2^64
    }
    bits |= (uint64_t)neg << 63;
#ifdef __CUDA_ARCH__
    return {LETOR_DEC_OK, __longlong_as_double((long long)bits)};
#else
    double v;
    memcpy(&v, &bits, 8);
    return {LETOR_DEC_OK, v};
#endif
}

}  // namespace ptrb200
