"""get_double cases shared by the oracle pinning, the host emulation and the GPU tests of sjb200_column_double_dev: number
texts whose correctly rounded binary64 is known from Python's float() (correctly rounded), and seeded generators."""
import math
import struct
from fractions import Fraction

import numpy as np

INF_ERROR = 9  # NUMBER_ERROR


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def is_integer(text):
    return text.lstrip("-").isdigit()


def expect(text, as_token=True):
    """(error, bits) of get_double on a number text: float() of a float, NUMBER_ERROR when infinite; an integer (an 'l'
    or 'u' token) is converted from its integer value, so "-0" gives +0.0.  as_token=False: float() of every text (the
    float routine on its own, which reads "-0" as -0.0)"""
    x = float(int(text)) if as_token and is_integer(text) else float(text)
    return (INF_ERROR, 0) if math.isinf(x) else (0, bits(x))


def exact_decimal(fr):
    """the finite decimal expansion of a fraction whose denominator is a power of two, without an exponent, always with a
    '.' (so that it is a float token)"""
    n, d = fr.numerator, fr.denominator
    k = d.bit_length() - 1
    assert d == 1 << k
    sign = "-" if n < 0 else ""
    digits = str(abs(n) * 5 ** k)
    if k == 0:
        return sign + digits + ".0"
    digits = digits.rjust(k + 1, "0")
    return sign + digits[:-k] + "." + digits[-k:]


def bump_last(text, delta):
    """text with delta (+1 / -1) added in its last digit's unit (an exact decimal, no exponent)"""
    frac = len(text.split(".")[1]) if "." in text else 0
    v = Fraction(text) + Fraction(delta, 10 ** frac)
    s = str(abs(v.numerator) * (10 ** frac) // v.denominator)
    s = s.rjust(frac + 1, "0")
    out = (s[:-frac] + "." + s[-frac:]) if frac else s
    return ("-" if v < 0 else "") + out


def halfway(x):
    """the exact decimal of the point halfway between x > 0 and the next double up"""
    return exact_decimal((Fraction(x) + Fraction(math.nextafter(x, math.inf))) / 2)


def halfway_cases():
    """halfway points between adjacent doubles written out exactly (the longest has 767 significant digits), each
    with one unit more and one less in the last digit"""
    xs = [1.0, 0.1, 2.0 ** 53, 9007199254740992.0 * 3, 1e23, 5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308,
          math.nextafter(2.2250738585072014e-308, 0), 1.7976931348623157e308 / 2, 123456.789, 1e-300, 7e-10, 3.0e200]
    out = []
    for x in xs:
        h = halfway(x)
        out += [h, bump_last(h, 1), bump_last(h, -1)]
    return out


def long_tail(n=10000):
    """a mantissa of n digits: the halfway point above 1.0 padded with zeros, its only non-zero tail digit at position
    n -- it rounds up -- and the same without that digit -- a tie, to even"""
    h = halfway(1.0)
    digits = h.replace(".", "")
    pad = digits + "0" * (n - 1 - len(digits))
    return ["1." + pad[1:] + "1", "1." + pad[1:] + "0"]


def named_cases():
    """the edge cases of get_double: Clinger boundaries, subnormals, the largest double, infinities, zeros, exponents
    of more than 18 digits, leading zeros, long tails, integers"""
    return (["9007199254740992.0", "9007199254740993.0", "9007199254740991e22", "1e22", "1e23", "4.9406564584124654e-324",
             "2.4703282292062328e-324", "2.4703282292062327e-324", "2.4703282292062329e-324", exact_decimal(Fraction(1, 2 ** 1075)),
             "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1e400", "-1e400",
             "0e999999999999999999999", "1e-999999999999999999999", "1e0000000000000000000000000001", "0.00000000000000000000001234",
             "-0", "-0.0", "-0.0e-999", "9007199254740993", "18446744073709551615", "-9223372036854775808", "1.5", "-2.5e-3",
             "2.2250738585072011e-308", "1e-342", "1e-343", "9.999999999999999e-344", "1e308", "1.0e+308", "1E-5", "0.1e1"]
            + halfway_cases() + long_tail())


def random_numbers(count, seed):
    """count seeded number texts, a quarter each: random doubles written shortest, with 17 digits, with 25 to 40
    digits, and random decimal strings (1 to 30 digits, a '.' anywhere, exponents -360 to 360)"""
    rng = np.random.default_rng(seed)
    q = count // 4
    raw = rng.integers(0, 2 ** 63, size=3 * q, dtype=np.int64).astype(np.uint64)
    raw |= rng.integers(0, 2, size=3 * q, dtype=np.int64).astype(np.uint64) << np.uint64(63)
    xs = raw.view(np.float64)
    xs = np.where(np.isfinite(xs), xs, 1.5)
    out = [repr(float(x)) for x in xs[:q]]
    out += ["%.16e" % x for x in xs[q: 2 * q]]
    ks = rng.integers(24, 40, size=q)
    out += ["%.*e" % (int(k), x) for k, x in zip(ks, xs[2 * q: 3 * q])]
    nd = rng.integers(1, 31, size=count - 3 * q)
    ex = rng.integers(-360, 361, size=count - 3 * q)
    dots = rng.integers(0, 31, size=count - 3 * q)
    pool = rng.integers(0, 10, size=(count - 3 * q) * 30).astype(np.uint8) + 48
    text = pool.tobytes().decode()
    for i in range(count - 3 * q):
        d = text[30 * i: 30 * i + int(nd[i])].lstrip("0") or "0"
        p = int(dots[i])
        if 0 < p < len(d):
            d = d[:p] + "." + d[p:]
        out.append(f"{'-' if i % 5 == 0 else ''}{d}e{int(ex[i])}")
    return out


def slow_heavy(count, seed):
    """numbers of 20 to 25 significant digits (every one needs more than the first 19)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        k = int(rng.integers(20, 26))
        digs = "".join(str(int(c)) for c in rng.integers(0, 10, size=k))
        digs = str(int(rng.integers(1, 10))) + digs[1:]
        out.append(f"{digs[0]}.{digs[1:]}e{int(rng.integers(-30, 31))}")
    return out
