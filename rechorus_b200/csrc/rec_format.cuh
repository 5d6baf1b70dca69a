// rec_format.cuh -- NumPy's scalar repr of float32 and int64 as exact integer code, for host and device.
//
// save_rec_results writes each list element as repr() of a NumPy scalar (main.py:117-132: pandas' to_csv prints
// str(list), and str(list) uses repr of the elements).  The float32 text is the shortest decimal that reads back to the
// same float32, the candidate closest to the exact value when several have that length.  The digits come from Ryu
// (Ulf Adams, "Ryu: fast float-to-string conversion", PLDI 2018), float32 variant, written from the paper: the value
// m * 2^e is scaled by a power of 5 held as a 61-bit (5^i) or 59-bit (5^-i) fixed-point constant, using two 32 x 32 ->
// 64-bit products per bound; trailing digits are then removed while the lower and upper bounds still differ.  The
// layout rules on top of the digits (NumPy's Dragon4 front end, observed with NumPy 2.3):
//   - positional for lo <= |x| < hi, scientific otherwise; lo = 1e-4 compared against the exact float32 value, hi = 1e6
//     in NumPy 2's repr (style B2R_REC_STYLE_NP) and 1e16 in the bare style (NumPy 1.x, legacy='1.25');
//   - positional text always has a fraction digit ("100000.0", "-0.0"); scientific text drops a lone ".0" ("1e+07")
//     and has a signed exponent of at least two digits ("1e-45", "3.4028235e+38");
//   - "inf", "-inf", and "nan" for every NaN bit pattern (sign and payload are not printed).
// Style B2R_REC_STYLE_NP wraps the texts as "np.float32(...)" and "np.int64(...)".
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2R_HD __host__ __device__ __forceinline__
#else
#define B2R_HD inline
#endif

#ifndef B2R_REC_STYLE_NP
#define B2R_REC_STYLE_NP 0       // NumPy >= 2 repr: np.int64(3), np.float32(0.5)
#define B2R_REC_STYLE_BARE 1     // NumPy 1.x repr (and legacy='1.25'): 3, 0.5
#endif

namespace b2r {
namespace recfmt {

constexpr int kPow5InvBits = 59;       // 5^-i as floor(2^(pow5bits(i) - 1 + 59) / 5^i) + 1, i <= 30
constexpr int kPow5Bits = 61;          // 5^i as floor(5^i / 2^(pow5bits(i) - 61)), i <= 47
constexpr int kMaxText = 32;           // longest element text: "np.int64(-9223372036854775808)" is 30 bytes

#define B2R_POW5_INV_SPLIT {                                                        \
    0x0800000000000001ull, 0x0666666666666667ull, 0x051eb851eb851eb9ull,            \
    0x04189374bc6a7efaull, 0x068db8bac710cb2aull, 0x053e2d6238da3c22ull,            \
    0x0431bde82d7b634eull, 0x06b5fca6af2bd216ull, 0x055e63b88c230e78ull,            \
    0x044b82fa09b5a52dull, 0x06df37f675ef6eaeull, 0x057f5ff85e592558ull,            \
    0x0465e6604b7a8447ull, 0x0709709a125da071ull, 0x05a126e1a84ae6c1ull,            \
    0x0480ebe7b9d58567ull, 0x0734aca5f6226f0bull, 0x05c3bd5191b525a3ull,            \
    0x049c97747490eae9ull, 0x0760f253edb4ab0eull, 0x05e72843249088d8ull,            \
    0x04b8ed0283a6d3e0ull, 0x078e480405d7b966ull, 0x060b6cd004ac9452ull,            \
    0x04d5f0a66a23a9dbull, 0x07bcb43d769f762bull, 0x063090312bb2c4efull,            \
    0x04f3a68dbc8f03f3ull, 0x07ec3daf94180651ull, 0x065697bfa9acd1daull,            \
    0x051212ffbaf0a7e2ull}
#define B2R_POW5_SPLIT {                                                            \
    0x1000000000000000ull, 0x1400000000000000ull, 0x1900000000000000ull,            \
    0x1f40000000000000ull, 0x1388000000000000ull, 0x186a000000000000ull,            \
    0x1e84800000000000ull, 0x1312d00000000000ull, 0x17d7840000000000ull,            \
    0x1dcd650000000000ull, 0x12a05f2000000000ull, 0x174876e800000000ull,            \
    0x1d1a94a200000000ull, 0x12309ce540000000ull, 0x16bcc41e90000000ull,            \
    0x1c6bf52634000000ull, 0x11c37937e0800000ull, 0x16345785d8a00000ull,            \
    0x1bc16d674ec80000ull, 0x1158e460913d0000ull, 0x15af1d78b58c4000ull,            \
    0x1b1ae4d6e2ef5000ull, 0x10f0cf064dd59200ull, 0x152d02c7e14af680ull,            \
    0x1a784379d99db420ull, 0x108b2a2c28029094ull, 0x14adf4b7320334b9ull,            \
    0x19d971e4fe8401e7ull, 0x1027e72f1f128130ull, 0x1431e0fae6d7217cull,            \
    0x193e5939a08ce9dbull, 0x1f8def8808b02452ull, 0x13b8b5b5056e16b3ull,            \
    0x18a6e32246c99c60ull, 0x1ed09bead87c0378ull, 0x13426172c74d822bull,            \
    0x1812f9cf7920e2b6ull, 0x1e17b84357691b64ull, 0x12ced32a16a1b11eull,            \
    0x178287f49c4a1d66ull, 0x1d6329f1c35ca4bfull, 0x125dfa371a19e6f7ull,            \
    0x16f578c4e0a060b5ull, 0x1cb2d6f618c878e3ull, 0x11efc659cf7d4b8dull,            \
    0x166bb7f0435c9e71ull, 0x1c06a5ec5433c60dull, 0x118427b3b4a05bc8ull}

#if defined(__CUDACC__)
__constant__ uint64_t c_pow5_inv_split[31] = B2R_POW5_INV_SPLIT;
__constant__ uint64_t c_pow5_split[48] = B2R_POW5_SPLIT;
#endif
static const uint64_t h_pow5_inv_split[31] = B2R_POW5_INV_SPLIT;
static const uint64_t h_pow5_split[48] = B2R_POW5_SPLIT;

B2R_HD uint64_t pow5_inv_split(uint32_t i) {
#if defined(__CUDA_ARCH__)
    return c_pow5_inv_split[i];
#else
    return h_pow5_inv_split[i];
#endif
}

B2R_HD uint64_t pow5_split(uint32_t i) {
#if defined(__CUDA_ARCH__)
    return c_pow5_split[i];
#else
    return h_pow5_split[i];
#endif
}

B2R_HD int32_t pow5bits(int32_t e) { return (int32_t)(((uint32_t)e * 1217359u) >> 19) + 1; }   // ceil(log2(5^e)), e >= 1
B2R_HD uint32_t log10_pow2(int32_t e) { return ((uint32_t)e * 78913u) >> 18; }                 // floor(log10(2^e))
B2R_HD uint32_t log10_pow5(int32_t e) { return ((uint32_t)e * 732923u) >> 20; }                // floor(log10(5^e))

B2R_HD bool multiple_of_pow5(uint32_t v, uint32_t p) {
    uint32_t n = 0;
    while (v != 0 && v % 5 == 0) {
        v /= 5;
        ++n;
    }
    return n >= p;
}

B2R_HD bool multiple_of_pow2(uint32_t v, uint32_t p) { return (v & ((1u << p) - 1)) == 0; }

// (m * factor) >> shift for a 32-bit m, a 64-bit factor and 32 < shift: two 32 x 32 -> 64 products, no 128-bit type
B2R_HD uint32_t mul_shift(uint32_t m, uint64_t factor, int32_t shift) {
    const uint64_t lo = (uint64_t)m * (uint32_t)factor;
    const uint64_t hi = (uint64_t)m * (uint32_t)(factor >> 32);
    return (uint32_t)(((lo >> 32) + hi) >> (shift - 32));
}

struct Decimal {
    uint32_t digits;     // no trailing zeros
    int32_t exp10;       // value = digits * 10^exp10
};

// shortest round-trip decimal of a finite non-zero float32 given its biased exponent and mantissa fields
B2R_HD Decimal shortest_f32(uint32_t ieee_m, uint32_t ieee_e) {
    int32_t e2;
    uint32_t m2;
    if (ieee_e == 0) {
        e2 = 1 - 127 - 23 - 2;
        m2 = ieee_m;
    } else {
        e2 = (int32_t)ieee_e - 127 - 23 - 2;
        m2 = (1u << 23) | ieee_m;
    }
    // round-half-even parsing: a bound of the interval reads back to this float exactly when its mantissa is even
    const bool accept_bounds = (m2 & 1) == 0;
    const uint32_t mv = 4 * m2;
    const uint32_t mp = 4 * m2 + 2;
    const uint32_t mm_shift = (ieee_m != 0 || ieee_e <= 1) ? 1u : 0u;     // 0 at a power of 2: the gap below is half as wide
    const uint32_t mm = 4 * m2 - 1 - mm_shift;

    uint32_t vr, vp, vm;
    int32_t e10;
    bool vm_zeros = false, vr_zeros = false;
    uint32_t last = 0;
    if (e2 >= 0) {
        const uint32_t q = log10_pow2(e2);
        e10 = (int32_t)q;
        const int32_t k = kPow5InvBits + pow5bits((int32_t)q) - 1;
        const int32_t i = -e2 + (int32_t)q + k;
        vr = mul_shift(mv, pow5_inv_split(q), i);
        vp = mul_shift(mp, pow5_inv_split(q), i);
        vm = mul_shift(mm, pow5_inv_split(q), i);
        if (q != 0 && (vp - 1) / 10 <= vm / 10) {
            // the loop below may remove no digit: the digit removed by the scaling itself decides the rounding
            const int32_t l = kPow5InvBits + pow5bits((int32_t)q - 1) - 1;
            last = mul_shift(mv, pow5_inv_split(q - 1), -e2 + (int32_t)q - 1 + l) % 10;
        }
        if (q <= 9) {
            // mv = 4 m2 < 2^26 < 5^12: only for small q can a bound be divisible by 5^q (exact, no digit was lost)
            if (mv % 5 == 0) vr_zeros = multiple_of_pow5(mv, q);
            else if (accept_bounds) vm_zeros = multiple_of_pow5(mm, q);
            else vp -= multiple_of_pow5(mp, q) ? 1u : 0u;
        }
    } else {
        const uint32_t q = log10_pow5(-e2);
        e10 = (int32_t)q + e2;
        const int32_t i = -e2 - (int32_t)q;
        const int32_t k = pow5bits(i) - kPow5Bits;
        int32_t j = (int32_t)q - k;
        vr = mul_shift(mv, pow5_split((uint32_t)i), j);
        vp = mul_shift(mp, pow5_split((uint32_t)i), j);
        vm = mul_shift(mm, pow5_split((uint32_t)i), j);
        if (q != 0 && (vp - 1) / 10 <= vm / 10) {
            j = (int32_t)q - 1 - (pow5bits(i + 1) - kPow5Bits);
            last = mul_shift(mv, pow5_split((uint32_t)(i + 1)), j) % 10;
        }
        if (q <= 1) {
            // mv, mp and mm have at least q trailing zero bits, so the scaled values are exact
            vr_zeros = true;
            if (accept_bounds) vm_zeros = mm_shift == 1;
            else --vp;
        } else if (q < 31) {
            vr_zeros = multiple_of_pow2(mv, q - 1);
        }
    }

    int32_t removed = 0;
    uint32_t out;
    if (vm_zeros || vr_zeros) {
        // general case: track whether the removed digits were all zero (exact ties, inclusive lower bound)
        while (vp / 10 > vm / 10) {
            vm_zeros &= vm % 10 == 0;
            vr_zeros &= last == 0;
            last = vr % 10;
            vr /= 10;
            vp /= 10;
            vm /= 10;
            ++removed;
        }
        if (vm_zeros) {
            while (vm % 10 == 0) {
                vr_zeros &= last == 0;
                last = vr % 10;
                vr /= 10;
                vp /= 10;
                vm /= 10;
                ++removed;
            }
        }
        if (vr_zeros && last == 5 && vr % 2 == 0) last = 4;           // exactly halfway: round to even
        out = vr + (((vr == vm && (!accept_bounds || !vm_zeros)) || last >= 5) ? 1u : 0u);
    } else {
        while (vp / 10 > vm / 10) {
            last = vr % 10;
            vr /= 10;
            vp /= 10;
            vm /= 10;
            ++removed;
        }
        out = vr + ((vr == vm || last >= 5) ? 1u : 0u);
    }
    int32_t exp10 = e10 + removed;
    while (out % 10 == 0) {          // a rounding carry can leave zeros (99 -> 100): NumPy prints none
        out /= 10;
        ++exp10;
    }
    return Decimal{out, exp10};
}

B2R_HD int put_str(char* o, const char* s) {
    int n = 0;
    while (s[n]) {
        o[n] = s[n];
        ++n;
    }
    return n;
}

// decimal digits of v, most significant first; returns the count
B2R_HD int put_u64(char* o, uint64_t v) {
    char tmp[20];
    int n = 0;
    while (v >= 0x100000000ull) {    // 64-bit divisions only while the value needs them
        tmp[n++] = (char)('0' + v % 10);
        v /= 10;
    }
    uint32_t w = (uint32_t)v;
    do {
        tmp[n++] = (char)('0' + w % 10);
        w /= 10;
    } while (w != 0);
    for (int i = 0; i < n; ++i) o[i] = tmp[n - 1 - i];
    return n;
}

// NumPy's repr of a float32 given its bits in `style`; o must hold kMaxText bytes; returns the length
B2R_HD int format_f32(uint32_t bits, int style, char* o) {
    int n = 0;
    if (style == B2R_REC_STYLE_NP) n += put_str(o, "np.float32(");
    const uint32_t ieee_m = bits & 0x7fffffu, ieee_e = (bits >> 23) & 0xffu, mag = bits & 0x7fffffffu;
    if (bits >> 31 && !(ieee_e == 0xff && ieee_m != 0)) o[n++] = '-';
    if (ieee_e == 0xff) {
        n += put_str(o + n, ieee_m ? "nan" : "inf");
    } else if (mag == 0) {
        n += put_str(o + n, "0.0");
    } else {
        const Decimal d = shortest_f32(ieee_m, ieee_e);
        char dig[10];
        const int nd = put_u64(dig, d.digits);
        const int point = nd + d.exp10;          // value = 0.dig * 10^point
        // thresholds on the float32 itself: 0x38d1b718 is the first float32 >= 1e-4, 0x49742400 is 1e6 exactly and
        // 0x5a0e1bca the first float32 >= 1e16
        const uint32_t hi = style == B2R_REC_STYLE_NP ? 0x49742400u : 0x5a0e1bcau;
        if (mag >= 0x38d1b718u && mag < hi) {
            if (point <= 0) {
                o[n++] = '0';
                o[n++] = '.';
                for (int t = 0; t < -point; ++t) o[n++] = '0';
                for (int t = 0; t < nd; ++t) o[n++] = dig[t];
            } else if (point >= nd) {
                for (int t = 0; t < nd; ++t) o[n++] = dig[t];
                for (int t = nd; t < point; ++t) o[n++] = '0';
                o[n++] = '.';
                o[n++] = '0';
            } else {
                for (int t = 0; t < point; ++t) o[n++] = dig[t];
                o[n++] = '.';
                for (int t = point; t < nd; ++t) o[n++] = dig[t];
            }
        } else {
            o[n++] = dig[0];
            if (nd > 1) {
                o[n++] = '.';
                for (int t = 1; t < nd; ++t) o[n++] = dig[t];
            }
            int e = point - 1;
            o[n++] = 'e';
            o[n++] = e < 0 ? '-' : '+';
            if (e < 0) e = -e;
            if (e < 10) o[n++] = '0';
            n += put_u64(o + n, (uint64_t)e);
        }
    }
    if (style == B2R_REC_STYLE_NP) o[n++] = ')';
    return n;
}

// decimal text of an int64 ("np.int64(...)" in style B2R_REC_STYLE_NP); o must hold kMaxText bytes
B2R_HD int format_i64(int64_t v, int style, char* o) {
    int n = 0;
    if (style == B2R_REC_STYLE_NP) n += put_str(o, "np.int64(");
    uint64_t u = (uint64_t)v;
    if (v < 0) {
        o[n++] = '-';
        u = 0 - u;                   // INT64_MIN's magnitude is representable as uint64
    }
    n += put_u64(o + n, u);
    if (style == B2R_REC_STYLE_NP) o[n++] = ')';
    return n;
}

// the longest text save_rec_results can write for one row of k elements: user id (20 bytes) and both list cells at
// their longest element texts, each field quoted, two separators and the newline
B2R_HD int64_t row_bytes_max(int k, int style) {
    const int64_t item = style == B2R_REC_STYLE_NP ? 30 : 20;         // "np.int64(-9223372036854775808)"
    const int64_t score = style == B2R_REC_STYLE_NP ? 31 : 19;        // "-9999999000000000.0", plus "np.float32()"
    const int64_t seps = k > 0 ? 2 * ((int64_t)k - 1) : 0;
    return (20 + 2) + 1 + (2 + seps + item * k + 2) + 1 + (2 + seps + score * k + 2) + 1;
}

}  // namespace recfmt
}  // namespace b2r
