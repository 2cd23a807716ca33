// Field rules of the TSV loader, one definition for the host parser and the device parser (tsv.cu): the NA rule, the label and
// weight rules, multivalue tokens, and the exact fast paths of the int / float decoders.  A fast path either returns the value
// strtoll / strtof would return or declines; the host parser then asks libc, the device parser hands the batch to the host.
#pragma once
#include <stdint.h>
#include <string.h>

#include "farmhash.cuh"

namespace wd {

// an empty field or the NA token "-" takes its column's default
WD_HD bool tsv_is_na(const char* f, int flen) { return flen == 0 || (flen == 1 && f[0] == '-'); }

// [-]digits, at most 18 of them (no overflow possible); anything else (spaces, '+', longer) declines
WD_HD bool tsv_int_fast(const char* f, int flen, long long* out) {
    int i = 0;
    const bool neg = flen > 0 && f[0] == '-';
    if (neg) i = 1;
    const int nd = flen - i;
    if (nd < 1 || nd > 18) return false;
    long long v = 0;
    for (; i < flen; ++i) {
        const unsigned d = (unsigned)(f[i] - '0');
        if (d > 9) return false;
        v = v * 10 + d;
    }
    *out = neg ? -v : v;
    return true;
}

// [-]digits[.digits] with at most 19 significant digits and 22 fraction digits (the 16-digit coordinates of the bundled data are
// common).  m = the digits as an integer, p = 10^frac (an exact double); d = fl(fl(m) / p) is within 2^-52 relative of the
// decimal, i.e. within 2 ulps of a double — exactly the correctly rounded double when m <= 2^53 (Clinger's fast path).  Rounding d
// to float gives the correctly rounded float of the decimal unless a float midpoint lies within that error of d: a midpoint has
// the low 29 mantissa bits 0x10000000, so d's low bits within 1 (m exact) or 4 (m rounded) of it decline, as does every other
// shape (exponents, inf / nan, spaces).
WD_HD bool tsv_float_fast(const char* f, int flen, float* out) {
    int i = 0;
    const bool neg = flen > 0 && f[0] == '-';
    if (neg) i = 1;
    unsigned long long m = 0;
    int nd = 0, frac = 0;
    bool dot = false, any = false;
    for (; i < flen; ++i) {
        const char c = f[i];
        if (c == '.') {
            if (dot) return false;
            dot = true;
            continue;
        }
        const unsigned d = (unsigned)(c - '0');
        if (d > 9) return false;
        any = true;
        if (nd > 0 || d != 0) {                             // significant digits (leading zeros do not count)
            if (++nd > 19) return false;                    // (10^19 - 1 < 2^64)
            m = m * 10 + d;
        }
        if (dot && ++frac > 22) return false;
    }
    if (!any) return false;
    if (m == 0) { *out = neg ? -0.f : 0.f; return true; }
    double p10 = 1.0;                                       // 10^frac, exact for frac <= 22
    for (int k = 0; k < frac; ++k) p10 *= 10.0;
    const double d = (double)m / p10;
    if (!(d > 1e-30 && d < 1e30)) return false;             // far from float's subnormal / overflow ranges
    unsigned long long bits;
    memcpy(&bits, &d, 8);
    const unsigned low = (unsigned)(bits & 0x1FFFFFFFull);
    const unsigned margin = m <= (1ull << 53) ? 1u : 4u;
    if (low + margin >= 0x10000000u && low <= 0x10000000u + margin) return false;
    *out = neg ? -(float)d : (float)d;
    return true;
}

// label rule: 1 when the field reads as the integer 1, else 0.  `as_int` decodes the field (fast path, or fast path + libc on the
// host); it is asked only when the field is neither NA nor the single byte '1'.
template <class AsInt>
WD_HD float tsv_label(const char* f, int flen, AsInt as_int) {
    if (tsv_is_na(f, flen)) return 0.f;
    if (flen == 1 && f[0] == '1') return 1.f;
    long long v = 0;
    return (as_int(f, flen, &v) && v == 1) ? 1.f : 0.f;
}

// weight rule: pos / neg loss weight by label when the spec uses weights, else 1
WD_HD float tsv_weight(int use_weight, float pos_weight, float neg_weight, float label) {
    return use_weight ? (label > 0.5f ? pos_weight : neg_weight) : 1.f;
}

// first occurrence of byte c in [p, end), or end
WD_HD const char* tsv_find(const char* p, const char* end, char c) {
#if defined(__CUDA_ARCH__)
    while (p < end && *p != c) ++p;
    return p;
#else
    const char* q = (const char*)memchr(p, c, end - p);
    return q ? q : end;
#endif
}

// tokens of a (non-NA) categorical string field, in order: the whole field, or with `multivalue` its ','-separated pieces with
// empty pieces dropped.  fn(token, length) per token; returns the token count.
template <class Fn>
WD_HD int tsv_tokens(const char* f, int flen, int multivalue, Fn fn) {
    if (!multivalue) { fn(f, flen); return 1; }
    const char* end = f + flen;
    int n = 0;
    for (const char* t = f;;) {
        const char* te = tsv_find(t, end, ',');
        if (te > t) { fn(t, (int)(te - t)); ++n; }
        if (te == end) break;
        t = te + 1;
    }
    return n;
}

}  // namespace wd
