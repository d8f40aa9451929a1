"""The 128-bit arithmetic of the Decimal aggregate ops (spark-s3-shuffle_b200/csrc/decimal128.h, the functions the
merge kernels of aggregate.cu call) compiled for the host and checked against Python integers, without a GPU: the add
and its overflow past 128 bits, |x| < 10^P, the signed order, and BigInteger.toByteArray's minimal big-endian bytes."""
import ctypes as C
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M128 = (1 << 128) - 1


@pytest.fixture(scope="module")
def dc(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("dc") / "libdc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", out,
                           os.path.join(ROOT, "tests", "native", "decimal128_host.cpp")])
    L = C.CDLL(out)
    u64 = C.c_uint64
    L.dc_add.argtypes = [u64, u64, u64, u64, C.c_void_p]
    L.dc_fits.argtypes = [u64, u64, C.c_uint32]
    L.dc_less.argtypes = [u64, u64, u64, u64]
    L.dc_encode.restype = C.c_uint32
    L.dc_encode.argtypes = [u64, u64, C.c_void_p]
    L.dc_of_long.argtypes = [u64, C.c_void_p]
    return L


def split(x):
    x &= M128
    return x & (2**64 - 1), x >> 64


def signed(lo, hi):
    x = lo | (hi << 64)
    return x - (1 << 128) if x >> 127 else x


def to_byte_array(x):
    """java.math.BigInteger.toByteArray"""
    n = (x if x >= 0 else ~x).bit_length() // 8 + 1
    return x.to_bytes(n, "big", signed=True)


def add(dc, a, b):
    s = (C.c_uint64 * 2)()
    ovf = dc.dc_add(*split(a), *split(b), s)
    return signed(s[0], s[1]), bool(ovf)


def encode(dc, x):
    buf = (C.c_uint8 * 16)()
    n = dc.dc_encode(*split(x), buf)
    return n, bytes(buf)


def edge_values():
    out = {0, 1, -1, 127, 128, -128, -129, 255, 256, 2**127 - 1, -2**127}
    for k in range(1, 17):  # both ends of every byte length
        out |= {2**(8 * k - 1) - 1, -2**(8 * k - 1), 2**(8 * k - 1), -2**(8 * k - 1) - 1}
    for p in (18, 19, 28, 38):
        out |= {10**p - 1, -(10**p - 1), 10**p, -10**p}
    return sorted(v for v in out if -2**127 <= v < 2**127)


def test_minimal_encoding_of_every_byte_length(dc):
    for x in edge_values():
        n, got = encode(dc, x)
        want = to_byte_array(x)
        assert (n, got) == (len(want), want + bytes(16 - len(want))), x
    seen = {encode(dc, x)[0] for x in edge_values()}
    assert seen == set(range(1, 17))
    # the sign boundaries of BigInteger
    assert encode(dc, 127)[1][:1] == b"\x7f" and encode(dc, 128)[1][:2] == b"\x00\x80"
    assert encode(dc, -128)[1][:1] == b"\x80" and encode(dc, -129)[1][:2] == b"\xff\x7f"
    assert encode(dc, 0) == (1, bytes(16))


def test_random_encodings(dc):
    rng = random.Random(1)
    for _ in range(20000):
        bits = rng.randint(1, 127)
        x = rng.getrandbits(bits) * rng.choice((1, -1))
        n, got = encode(dc, x)
        want = to_byte_array(x)
        assert got[:n] == want and got[n:] == bytes(16 - n), x


def test_range_check_at_both_ends(dc):
    for p in range(1, 39):
        for x, fits in ((10**p - 1, True), (-(10**p - 1), True), (10**p, False), (-10**p, False), (0, True)):
            assert dc.dc_fits(*split(x), p) == fits, (p, x)
    for p in (19, 38):
        assert dc.dc_fits(*split(-2**127), p) == 0 and dc.dc_fits(*split(2**127 - 1), p) == 0


def test_add_and_the_129th_bit(dc):
    big = 10**38 - 1
    for a, b in ((big, big), (-big, -big), (2**127 - 1, 1), (-2**127, -1), (big, -big), (2**126, 2**126),
                 (-2**126, -2**126 - 1), (-2**126, -2**126)):
        s, ovf = add(dc, a, b)
        exact = a + b
        assert ovf == (not -2**127 <= exact < 2**127), (a, b)
        if not ovf:
            assert s == exact
        else:
            assert s == signed(*split(exact))  # the low 128 bits; the overflow flag carries the rest
    rng = random.Random(2)
    for _ in range(20000):
        a = rng.randint(-2**127, 2**127 - 1)
        b = rng.randint(-2**127, 2**127 - 1)
        s, ovf = add(dc, a, b)
        exact = a + b
        assert ovf == (not -2**127 <= exact < 2**127)
        assert s == signed(*split(exact))


def test_long_sign_extension_and_order(dc):
    out = (C.c_uint64 * 2)()
    for v in (0, 1, -1, 2**63 - 1, -2**63, 10**18 - 1, -(10**18 - 1)):
        dc.dc_of_long(v & (2**64 - 1), out)
        assert signed(out[0], out[1]) == v
    vals = edge_values()
    rng = random.Random(3)
    for _ in range(5000):
        a, b = rng.choice(vals), rng.choice(vals)
        assert dc.dc_less(*split(a), *split(b)) == (a < b), (a, b)
