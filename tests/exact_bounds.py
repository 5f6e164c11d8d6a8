"""Exact arithmetic for checking short fp64 sums: the yardstick of the element-wise kernel tests.

Every output these tests check is a sum of at most a few hundred products of fp64 numbers.  Its exact value is a
rational number, computed here without rounding; any fp64 evaluation of the sum -- in any order, with or without FMA --
lies within gamma_m T of it, where T is the sum of the magnitudes of the m terms and gamma_m = m u / (1 - m u),
u = 2^-53 (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 3.1).  `within` keeps one term of
margin, gamma_{m+1}, as the KKT-residual check does.

Underflow: the gamma bound assumes that no product or partial sum is subnormal.  Generate data away from the bottom of
the exponent range; a case that goes there on purpose passes ``subnormal=True`` to `within`, which adds m 2^-1074
absolute (one unit in the last place of a subnormal per rounding)."""
import math
from fractions import Fraction

U = Fraction(1, 2 ** 53)      # unit roundoff of fp64
TINY = Fraction(1, 2 ** 1074)  # the smallest subnormal


def _split(x):
    """finite float -> (n, k) with x = n / 2**k exactly, k >= 0."""
    n, d = float(x).as_integer_ratio()
    return n, d.bit_length() - 1


def exact_sum(terms):
    """Exact value of a sum of products.  ``terms``: iterable of tuples of factors (usually pairs of doubles; a factor may
    also be a Fraction, e.g. the exact 1 / mu of a division).  Returns (exact value, sum of |terms|, m = number of
    terms), the first two as Fractions.  All-float terms are summed as integers scaled by a common power of two, so a
    few hundred terms cost well under a millisecond."""
    ints, frac, fabs, m = [], Fraction(0), Fraction(0), 0
    for t in terms:
        m += 1
        if all(isinstance(f, float) for f in t):
            n, k = 1, 0
            for f in t:
                a, b = _split(f)
                n, k = n * a, k + b
            ints.append((n, k))
        else:
            p = Fraction(1)
            for f in t:
                p *= Fraction(f)
            frac += p
            fabs += abs(p)
    if ints:
        K = max(k for _, k in ints)
        frac += Fraction(sum(n << (K - k) for n, k in ints), 1 << K)
        fabs += Fraction(sum(abs(n) << (K - k) for n, k in ints), 1 << K)
    return frac, fabs, m


def gamma(m):
    """gamma_{m+1} = (m + 1) u / (1 - (m + 1) u): the bound for m terms with one term of margin."""
    return (m + 1) * U / (1 - (m + 1) * U)


def bound(T, m, subnormal=False):
    return gamma(m) * T + (m * TINY if subnormal else 0)


def within(got, exact, T, m, subnormal=False):
    """|got - exact| <= gamma_{m+1} T (+ m 2^-1074 with ``subnormal``); a non-finite ``got`` is never within."""
    g = float(got)
    return math.isfinite(g) and abs(Fraction(g) - exact) <= bound(T, m, subnormal)


def excess(got, exact, T, m):
    """|got - exact| / (gamma_{m+1} T): <= 1 inside the bound (for the printed tables); inf for a non-finite ``got``."""
    g = float(got)
    if not math.isfinite(g):
        return math.inf
    b = bound(T, m)
    err = abs(Fraction(g) - exact)
    return float(err / b) if b else (0.0 if err == 0 else math.inf)


def correctly_rounded(x):
    """The double nearest to the Fraction x, ties to even (CPython's int / int true division rounds correctly, into the
    subnormals too); +-inf where the rounded value overflows."""
    try:
        return x.numerator / x.denominator
    except OverflowError:
        return math.inf if x > 0 else -math.inf


def same_bits(a, b):
    """Element-wise: a and b are the same double, sign of zero included; any NaN matches any NaN."""
    import numpy as np
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return (a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))
