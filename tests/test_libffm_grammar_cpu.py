"""The fast libffm grammar (lightctr_b200/csrc/libffm_grammar.h), which the host loader and the device parser share,
against glibc's strtof / sscanf: on a seeded corpus it never accepts with a result that differs from theirs, and it
accepts every plain decimal whose digits form an integer <= 2^24 with at most 10 of them after the point.  The header
is compiled by g++ into a small driver; no GPU needed."""
import os
import random
import subprocess
from decimal import Decimal, localcontext
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT

DRIVER = r'''
#include "libffm_grammar.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <iostream>
#include <string>
static unsigned bits(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
int main(int argc, char** argv) {
    const std::string mode = argv[1];
    std::string s;
    while (std::getline(std::cin, s)) {
        const char* p = s.c_str();
        const char* e = p + s.size();
        if (mode == "dec") {
            float g = 0.f;
            const int ok = lctr::ffm::decimal(p, e, &g);
            char* end = nullptr;
            const float r = strtof(p, &end);
            printf("%d %08x %08x %d\n", ok, bits(g), bits(r), (int)(end - p));
        } else if (mode == "tok") {
            uint64_t f = 0, id = 0;
            float v = 0.f;
            int n = -1;
            const char* vb = nullptr;
            const int t = lctr::ffm::token(p, e, &f, &id, &v, &n, &vb);
            size_t F = 0, I = 0;
            float V = -7.f;
            int N = -1;
            const int r = sscanf(p, "%zu:%zu:%f%n", &F, &I, &V, &N);
            printf("%d %llu %llu %08x %d %d %zu %zu %08x %d\n", t, (unsigned long long)f, (unsigned long long)id, bits(v),
                   n, r, F, I, bits(V), N);
        } else {
            int y = 0, n = -1, Y = 0, N = -1;
            const int ok = lctr::ffm::label(p, e, &y, &n);
            const int r = sscanf(p, "%d%n", &Y, &N);
            printf("%d %d %d %d %d %d\n", ok, y, n, r, Y, N);
        }
    }
    return 0;
}
'''


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("grammar")
    src, exe = str(d / "g.cpp"), str(d / "g")
    open(src, "w").write(DRIVER)
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "lightctr_b200", "csrc"), src, "-o", exe])

    def run(mode, strings):
        assert all("\n" not in s for s in strings)
        out = subprocess.run([exe, mode], input="\n".join(strings) + "\n", capture_output=True, text=True, check=True).stdout
        return [line.split() for line in out.splitlines()]
    return run


def _next_f32(f):
    return np.nextafter(np.float32(f), np.float32(np.inf))


def _plain(d):
    """a Decimal in positional notation, no exponent"""
    return format(d, "f")


def _corpus(seed=12345):
    rng = random.Random(seed)
    out = ["0", "-0", "+0", ".5", "5.", "-.5", "+5.", "0.0", "00012.50", "1", "1.0", "-1", "16777216", "16777217",
           "16777218", "16777219", "0.1", "0.2", "0.3", "3.4028235e38", "1e5", "0x10", "inf", "nan", ".", "-", "",
           "123456789012345678901234567890", "0.0000000000000000000000001", "9007199254740993", "9007199254740992.5"]
    for _ in range(3000):  # short decimals with signs
        ip = str(rng.randrange(0, 10 ** rng.randrange(0, 8)))
        fp = "".join(rng.choice("0123456789") for _ in range(rng.randrange(0, 9)))
        s = ip + ("." + fp if fp or rng.random() < 0.3 else "")
        out.append(rng.choice(["", "", "-", "+"]) + s)
    for _ in range(1500):  # long mantissas, around the 2^53 and 19-digit limits
        nd = rng.randrange(14, 24)
        digits = str(rng.randrange(1, 10)) + "".join(rng.choice("0123456789") for _ in range(nd - 1))
        cut = rng.randrange(0, nd + 1)
        out.append(digits[:cut] + "." + digits[cut:] if cut < nd else digits)
    with localcontext() as ctx:
        ctx.prec = 200
        for _ in range(2500):  # at and next to float rounding midpoints
            f = np.float32(rng.uniform(1.0, 2.0) * 2.0 ** rng.randrange(-30, 60))
            g = _next_f32(f)
            mid = (Fraction(float(f)) + Fraction(float(g))) / 2
            exact = Decimal(mid.numerator) / Decimal(mid.denominator)
            out.append(_plain(exact))
            for sig in (9, 12, 16, 17, 18, 19):
                ctx2 = ctx.copy()
                ctx2.prec = sig
                r = ctx2.plus(exact)
                ulp = Decimal(1).scaleb(r.adjusted() - sig + 1)
                for d in (r - ulp, r, r + ulp):
                    out.append(_plain(d))
        for _ in range(500):  # integers that are exact float midpoints (double path, must decline or agree)
            e2 = rng.randrange(25, 52)
            m = rng.randrange(2 ** 23, 2 ** 24)
            out.append(str((2 * m + 1) << (e2 - 25)))
    return out


def test_decimal_never_differs_from_strtof(driver):
    corpus = _corpus()
    res = driver("dec", corpus)
    accepted = 0
    for s, (ok, g, r, end) in zip(corpus, res):
        if ok == "1":
            accepted += 1
            assert g == r and int(end) == len(s), (s, g, r, end)
    assert accepted > len(corpus) // 3  # the exact midpoints (dozens of digits) decline; the rest mostly pass


def test_decimal_accepts_the_exact_fast_path(driver):
    rng = random.Random(7)
    corpus = []
    for _ in range(20000):
        m = rng.randrange(0, 2 ** 24 + 1) if rng.random() < 0.9 else rng.choice([0, 1, 2 ** 24, 2 ** 24 - 1])
        d = rng.randrange(0, 11)
        s = str(m).rjust(d + 1, "0")
        s = s[:len(s) - d] + "." + s[len(s) - d:] if d else s
        if rng.random() < 0.1:
            s = s.lstrip("0") or "0"
            if s.startswith("."):
                s = s if rng.random() < 0.5 else "0" + s
        corpus.append(rng.choice(["", "-", "+"]) + s)
    res = driver("dec", corpus)
    for s, (ok, g, r, end) in zip(corpus, res):
        assert ok == "1" and g == r, (s, ok, g, r)


def test_token_never_differs_from_sscanf(driver):
    rng = random.Random(99)
    vals = _corpus(seed=5)[:3000]
    corpus = []
    for v in vals:
        a, b = rng.randrange(0, 10 ** rng.randrange(1, 20)), rng.randrange(0, 10 ** rng.randrange(1, 21))
        lead = rng.choice(["", "", " ", "\t", "  "])
        tail = rng.choice(["", " ", " 3:4:1", ":", "x", "e5", "\r", ".5"])
        corpus.append("%s%d:%d:%s%s" % (lead, a, b, v, tail))
    corpus += ["1:2", "1:2:", "1::3", ":1:2", "+1:2:3", "1:+2:3", "1: 2:3", "-1:2:3", "1:2:-", "1:2:e5", "1:2:1E5",
               "1:2:0x1p3", "1:2:inf", "1:2:1.5.5", "1:2:  7", "12345678901234567890:1:1", "1:123456789012345678:2"]
    res = driver("tok", corpus)
    fast = 0
    for s, (t, f, i, v, n, r, F, I, V, N) in zip(corpus, res):
        if t == "1":
            fast += 1
            assert r == "3" and (f, i, v, n) == (F, I, V, N), s
        elif t == "2":  # syntax held, value declined: the loader reads it with strtof -- sscanf agrees on the extent
            assert r == "3" and (f, i, n) == (F, I, N), s
    assert fast > len(corpus) // 3


def test_label_never_differs_from_sscanf(driver):
    corpus = ["0", "1", "-1", "+1", " 1", "\t-7\t0:1:1", "123456789", "1234567890", "-999999999", "", " ", "x", "1x",
              "\r", "+", "-", "007", "2147483647", "99999999999"]
    res = driver("lab", corpus)
    for s, (ok, y, n, r, Y, N) in zip(corpus, res):
        if ok == "1":
            assert r == "1" and (y, n) == (Y, N), s
    assert [row[0] for row in res[:7]] == ["1"] * 7
