"""The GF(2) power tables of the CRC kernels (spark-s3-shuffle_b200/csrc/crc_gf.h, the functions checksum.cu calls)
compiled for the host and checked against plain polynomial arithmetic, without a GPU.

The kernels shift a partial CRC over e bytes by multiplying with x^(8e) mod P, built from tables of x^(+-2^k).  The
reference below is square-and-multiply on polynomials in normal form, with no tables.  It catches any table that
assumes a period of the powers of x: x^(2^32) = x mod P holds for CRC32's polynomial, but CRC32C's polynomial is
(x + 1) times an irreducible factor of degree 31, so there x^(2^32) = x^2 and every byte count of 2^29 or more needs
table entries past k = 31."""
import ctypes as C
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# normal form, x^32 term included; index = the kernels' polynomial number (0 CRC32, 1 CRC32C)
POLYS = {0: 0x104C11DB7, 1: 0x11EDC6F41}
NAMES = {0: "CRC32", 1: "CRC32C"}


@pytest.fixture(scope="module")
def cg(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cg") / "libcg.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "native", "crc_gf_host.cpp")])
    L = C.CDLL(out)
    L.cg_misc.argtypes = [C.c_int, C.c_void_p]
    L.cg_xpow8.restype = C.c_uint32
    L.cg_xpow8.argtypes = [C.c_int, C.c_ulonglong, C.c_int]
    L.cg_mul.restype = C.c_uint32
    L.cg_mul.argtypes = [C.c_int, C.c_uint32, C.c_uint32]
    return L


def mulmod(a, b, p):
    """a * b mod p over GF(2), polynomials as ints in normal form (bit i = x^i)"""
    r = 0
    while b:
        if b & 1:
            r ^= a
        b >>= 1
        a <<= 1
        if a >> 32:
            a ^= p
    return r


def xpow(n, p):
    """x^n mod p for any integer n (x is invertible: p has an x^0 term), by square-and-multiply"""
    base = 2 if n >= 0 else (p ^ 1) >> 1  # x, or x^-1 = (p - 1) / x
    n = abs(n)
    r = 1
    while n:
        if n & 1:
            r = mulmod(r, base, p)
        base = mulmod(base, base, p)
        n >>= 1
    return r


def normal(v):
    """reflected 32-bit value (bit 31 = x^0) -> normal form"""
    return int("{:032b}".format(v)[::-1], 2)


def exponents():
    rng = random.Random(29)
    es = set()
    for j in range(64):
        es.update({1 << j, (1 << j) - 1, (1 << j) + 1})
    es.update(rng.getrandbits(64) for _ in range(200))
    es.update(rng.getrandbits(rng.randint(28, 40)) for _ in range(100))
    es.update({(1 << 29) + 7, (1 << 30) + (1 << 29) + 13, (1 << 32) + 17, (1 << 64) - 1})
    return sorted(e for e in es if 0 <= e < 1 << 64)


@pytest.mark.parametrize("which", [0, 1], ids=["CRC32", "CRC32C"])
def test_power_tables(cg, which):
    """every x^(2^k) and x^-(2^k) entry, and the 32 lane-fold constants x^(8 * 16 * (31 - l))"""
    p = POLYS[which]
    words, bits = cg.cg_misc_words(), cg.cg_pow_bits()
    assert bits >= 64 + 3, "a 64-bit byte count e shifts by x^(8e): bit 63 of e needs k = 66"
    misc = np.zeros(words, np.uint32)
    cg.cg_misc(which, misc.ctypes.data)
    for k in range(bits):
        assert normal(int(misc[k])) == xpow(1 << k, p), (NAMES[which], "x^(2^%d)" % k)
        assert normal(int(misc[bits + k])) == xpow(-(1 << k), p), (NAMES[which], "x^-(2^%d)" % k)
    for lane in range(32):
        assert normal(int(misc[2 * bits + lane])) == xpow(8 * 16 * (31 - lane), p), (NAMES[which], lane)
    assert int(misc[2 * bits + 32]) == (0xEDB88320, 0x82F63B78)[which]


@pytest.mark.parametrize("which", [0, 1], ids=["CRC32", "CRC32C"])
def test_xpow8_over_every_exponent_bit(cg, which):
    """gf_xpow8(e) = x^(8e) mod P and its inverse table gives x^(-8e), for e = 2^j (j = 0..63), 2^j +- 1 and random
    64-bit byte counts"""
    p = POLYS[which]
    bad = []
    for e in exponents():
        if normal(cg.cg_xpow8(which, e, 0)) != xpow(8 * e, p):
            bad.append(("+", e))
        if normal(cg.cg_xpow8(which, e, 1)) != xpow(-8 * e, p):
            bad.append(("-", e))
    assert not bad, (NAMES[which], len(bad), bad[:8])


@pytest.mark.parametrize("which", [0, 1], ids=["CRC32", "CRC32C"])
def test_gf_mul(cg, which):
    p = POLYS[which]
    rng = random.Random(3 + which)
    for _ in range(500):
        a, b = rng.getrandbits(32), rng.getrandbits(32)
        assert normal(cg.cg_mul(which, a, b)) == mulmod(normal(a), normal(b), p)


def test_zero_slices_across_512_mib(cg, oracle):
    """crc_finalize_kernel's init term alone is the CRC of a slice of zero bytes; it must match the CPU checksums on
    both sides of 2^29 bytes, where CRC32C first needs the table entry x^(2^32)"""
    lengths = [(1 << 29) - 1, 1 << 29, (1 << 29) + 7]
    piece = np.zeros(1 << 26, np.uint8)
    want = {}
    c32, c32c, pos = 0, 0, 0
    for n in lengths:
        while pos < n:
            k = min(piece.size, n - pos)
            c32 = zlib.crc32(piece[:k], c32)
            c32c = oracle.lib().orc_crc32c(c32c, piece.ctypes.data, k)
            pos += k
        want[n] = (c32, c32c)
    for which in (0, 1):
        for n in lengths:
            got = cg.cg_mul(which, cg.cg_xpow8(which, n, 0), 0xFFFFFFFF) ^ 0xFFFFFFFF
            assert got == want[n][which], (NAMES[which], n, hex(got), hex(want[n][which]))
