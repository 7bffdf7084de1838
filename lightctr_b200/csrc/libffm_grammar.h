// lightctr_b200/csrc/libffm_grammar.h -- the fast grammar of a libffm line, one definition for the host loader
// (loader.cpp) and the device parser (text.cu).
//
// The reference reads a line with sscanf("%d%n") for the label and sscanf("%zu:%zu:%f%n") per token
// (fm_algo_abst.h:84-99).  The functions here accept the common subset of that syntax -- a label of at most 9 digits,
// tokens `digits:digits:plain-decimal` with at most 18 digits per id -- and give exactly what sscanf gives on it; the
// caller falls back to sscanf on everything they do not accept.  Character classes are those of the C locale: a byte
// another locale would classify differently is never part of an accepted token, so sscanf decides those lines.
#pragma once
#include <stdint.h>
#ifndef __CUDA_ARCH__
#include <string.h>
#endif

#ifdef __CUDACC__
#define LCTR_HD __host__ __device__ __forceinline__
#else
#define LCTR_HD inline
#endif

namespace lctr {
namespace ffm {

LCTR_HD bool is_space(char c) { return c == ' ' || (c >= '\t' && c <= '\r'); }
LCTR_HD bool is_digit(char c) { return c >= '0' && c <= '9'; }
LCTR_HD bool is_alpha(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }

// 10^n, exact: 10^n = 2^n * 5^n and 5^n < 2^24 for n <= 10 (float), 5^n < 2^53 for n <= 22 (double), so every product of
// the loop is representable
LCTR_HD float pow10f_exact(int n) {
    float p = 1.f;
    for (int i = 0; i < n; i++) p *= 10.f;
    return p;
}
LCTR_HD double pow10_exact(int n) {
    double p = 1.0;
    for (int i = 0; i < n; i++) p *= 10.0;
    return p;
}
LCTR_HD uint64_t double_bits(double d) {
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t u;
    memcpy(&u, &d, sizeof(u));
    return u;
#endif
}

// A plain decimal [+-](digits[.[digits]] | .digits) filling [s, e) -> the float strtof gives, or false (decline) for
// anything else and where this cannot be sure of it.  m = the digits with the point removed, x = m * 10^e10:
//   m <= 2^24, |e10| <= 10: m and 10^|e10| are exact floats, and one correctly rounded multiply or divide is strtof's
//     correctly rounded result;
//   m < 2^53, |e10| <= 22: the same in double, then rounded to float.  Rounding twice can differ from rounding once only
//     when the double lands exactly on a float midpoint (a float midpoint is a double, so rounding to double never crosses
//     one), and there it declines;
//   anything else declines, as would a result outside the normal float range (these bounds keep it inside: 1e-22 to 9e37).
LCTR_HD bool decimal(const char* s, const char* e, float* out) {
    bool neg = false;
    if (s < e && (*s == '-' || *s == '+')) { neg = *s == '-'; s++; }
    uint64_t m = 0;
    int nd = 0, e10 = 0;
    bool point = false, digits = false;
    for (; s < e; s++) {
        if (*s == '.' && !point) { point = true; continue; }
        if (!is_digit(*s)) return false;
        digits = true;
        if (point) e10--;
        if (m == 0 && *s == '0') continue;  // leading zeros
        if (++nd > 19) return false;
        m = m * 10 + (uint64_t)(*s - '0');
    }
    if (!digits) return false;
    float f;
    if (m == 0) {
        f = 0.f;
    } else if (m <= (1u << 24) && e10 >= -10 && e10 <= 10) {
        const float x = (float)m, p = pow10f_exact(e10 < 0 ? -e10 : e10);
        f = e10 < 0 ? x / p : x * p;
    } else if (m < (1ull << 53) && e10 >= -22 && e10 <= 22) {
        const double x = (double)m, p = pow10_exact(e10 < 0 ? -e10 : e10);
        const double d = e10 < 0 ? x / p : x * p;
        if ((double_bits(d) & 0x1FFFFFFFull) == 0x10000000ull) return false;  // halfway between two floats
        f = (float)d;
        const float a = f < 0.f ? -f : f;
        if (!(a >= 1.17549435e-38f && a <= 3.40282347e+38f)) return false;
    } else {
        return false;
    }
    *out = neg ? -f : f;
    return true;
}

// sscanf(p, "%d%n") for [space][+-]digits with at most 9 digits: *y, *nchar (bytes up to the last digit).  e: end of the line.
LCTR_HD bool label(const char* p, const char* e, int* y, int* nchar) {
    const char* s = p;
    while (s < e && is_space(*s)) s++;
    bool neg = false;
    if (s < e && (*s == '-' || *s == '+')) { neg = *s == '-'; s++; }
    if (!(s < e && is_digit(*s))) return false;
    long v = 0;
    int nd = 0;
    while (s < e && is_digit(*s)) {
        v = v * 10 + (*s - '0');
        s++;
        if (++nd > 9) return false;
    }
    *y = (int)(neg ? -v : v);
    *nchar = (int)(s - p);
    return true;
}

enum Token {
    TOKEN_NO = 0,     // not this grammar: sscanf decides
    TOKEN_OK = 1,     // *field, *fid, *val, *nchar as sscanf gives them
    TOKEN_VALUE = 2,  // the syntax holds but decimal() declined the value: *val_begin .. p + *nchar is for strtof
};

// sscanf(p, "%zu:%zu:%f%n") for [space]digits:digits:plain-decimal, with at most 18 digits per id and the value not
// followed by an exponent, a hex marker or a letter (which sscanf could read on).  e: end of the line.
LCTR_HD int token(const char* p, const char* e, uint64_t* field, uint64_t* fid, float* val, int* nchar, const char** val_begin) {
    const char* s = p;
    while (s < e && is_space(*s)) s++;
    uint64_t id[2];
    for (int k = 0; k < 2; k++) {
        if (!(s < e && is_digit(*s))) return TOKEN_NO;
        uint64_t a = 0;
        int nd = 0;
        while (s < e && is_digit(*s)) {
            a = a * 10 + (uint64_t)(*s - '0');
            s++;
            if (++nd > 18) return TOKEN_NO;
        }
        if (!(s < e && *s == ':')) return TOKEN_NO;
        s++;
        id[k] = a;
    }
    const char* fs = s;
    if (s < e && (*s == '-' || *s == '+')) s++;
    if (!(s < e && (is_digit(*s) || *s == '.'))) return TOKEN_NO;
    bool digits = false;
    while (s < e && is_digit(*s)) { s++; digits = true; }
    if (s < e && *s == '.') {
        s++;
        while (s < e && is_digit(*s)) { s++; digits = true; }
    }
    if (!digits) return TOKEN_NO;
    if (s < e && is_alpha(*s)) return TOKEN_NO;  // e / E / x / X and other letters: let sscanf decide
    *field = id[0];
    *fid = id[1];
    *nchar = (int)(s - p);
    *val_begin = fs;
    return decimal(fs, s, val) ? TOKEN_OK : TOKEN_VALUE;
}

}  // namespace ffm
}  // namespace lctr
