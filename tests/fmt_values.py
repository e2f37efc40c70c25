"""The doubles and integers MarshalJSON's formatter (csrc/fmt.h) is checked on: one copy, so the g++ build
(test_marshal_cpu.py) and the device build (test_gpu_marshal_edges.py) run exactly the same values.  Doubles are bit
patterns (uint64), never NaN or Inf; integers are Python ints in [0, 2^64)."""
import functools
import math
import struct

import numpy as np

_EXP = np.uint64(0x7FF0000000000000)


def double_bits(xs):
    return np.array([struct.unpack("<Q", struct.pack("<d", x))[0] for x in xs], dtype=np.uint64)


def _finite(b):
    return b[(b & _EXP) != _EXP]


def powers_of_two():
    """every power of two and its neighbours one ulp away, both signs"""
    b = double_bits([math.ldexp(1.0, e) for e in range(-1074, 1024)])
    b = _finite(np.concatenate([b, b + np.uint64(1), b[1:] - np.uint64(1)]))
    return np.concatenate([b, b | np.uint64(1 << 63)])


def notation_edges():
    """appendFloat's 1e-6 / 1e21 switch, the extremes and a few ordinary values, each with its neighbours"""
    edges = double_bits([1e-6, 1e21, 0.0, -0.0, 5e-324, 1.7976931348623157e308, 2.2250738585072014e-308, 0.1, 10.0,
                         30886023086020860000.0, 9007199254740993.0, 1e20, 1e22, 1e-7, 123456789.0, -9876.54321])
    near = np.concatenate([edges + np.uint64(d) for d in range(0, 4)] + [edges[edges > 4] - np.uint64(d) for d in range(1, 4)])
    return _finite(near)


def integers_near_2_53():
    return double_bits([float(k) for k in range(2 ** 53 - 1000, 2 ** 53 + 1000)] + [float(k) for k in range(-1000, 1000)])


def powers_of_ten():
    """every 1e+-k that is a double, and its neighbours"""
    p = double_bits([float("1e%d" % k) for k in range(-323, 309)])
    return np.concatenate([p, p + np.uint64(1), p - np.uint64(1)])


@functools.lru_cache(maxsize=None)
def _random():
    rng = np.random.default_rng(20260515)
    b = _finite(rng.integers(0, 2 ** 64, size=1_100_000, dtype=np.uint64))
    # doubles of ordinary magnitudes with 1 to 17 digits, where both notations and the shortening paths are dense
    m = 10.0 ** rng.uniform(-30, 30, size=200_000) * np.sign(rng.uniform(-1, 1, size=200_000))
    g = double_bits([float("%.*g" % (int(p), x)) for p, x in zip(rng.integers(1, 18, size=m.size), m)])
    return b, g


def random_bits():
    """about 1.1 M seeded random bit patterns"""
    return _random()[0]


def printf_g():
    """200 000 seeded doubles printed with %.{p}g, p in [1, 17], and read back"""
    return _random()[1]


@functools.lru_cache(maxsize=None)
def all_doubles():
    """every set above, each value once"""
    return np.unique(np.concatenate([powers_of_two(), notation_edges(), integers_near_2_53(), powers_of_ten(),
                                     random_bits(), printf_g()]))


INTEGERS = [0, 1, 9, 10, 99, 100, 2 ** 53, 2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1] + \
    [10 ** k + d for k in range(20) for d in (-1, 0, 1) if 0 <= 10 ** k + d < 2 ** 64]
