"""The round-robin model (tests/round_robin_model.py) on the CPU: the whole-row hash is MurmurHash3_x86_32 over whole
words, a literal restatement of Spark's RecordBinaryComparator orders rows as "shorter first, then unsigned
lexicographic", and the ids follow the writer's position."""
import numpy as np
import pytest

import hash_model as hm
import round_robin_model as rr

# MurmurHash3_x86_32's published vectors whose inputs are whole 4-byte words (hashUnsafeWords takes nothing else)
VECTORS = [(b"", 0, 0), (b"", 1, 0x514E28B7), (b"", 0xFFFFFFFF, 0x81F16F39), (b"\0\0\0\0", 0, 0x2362F9DE),
           (b"\xff\xff\xff\xff", 0, 0x76293B50), (b"\x21\x43\x65\x87", 0, 0xF55B516B),
           (b"\x21\x43\x65\x87", 0x5082EDEE, 0x2362F9DE), (b"aaaa", 0x9747B28C, 0x5A97808A),
           (b"abcd", 0x9747B28C, 0xF0478627)]


@pytest.mark.parametrize("data,seed,want", VECTORS)
def test_whole_word_hash_matches_published_vectors(data, seed, want):
    assert rr.hash_unsafe_words(data, seed) == want


def test_whole_word_hash_is_hash_bytes_on_unsafe_rows():
    rng = np.random.default_rng(0)
    for n in list(range(0, 200, 8)) + [1 << 12, 8 * 1001]:
        row = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        assert rr.hash_unsafe_words(row) == hm.hash_bytes(row, 42)


def record_binary_compare(mem_l, left_off, left_len, mem_r, right_off, right_len, unaligned):
    """Spark's RecordBinaryComparator.compare, line by line, over two byte buffers with the rows at these offsets;
    unaligned: Platform.unaligned() (both branches are restated)"""
    def get_byte(mem, o):
        return mem[o] - 256 if mem[o] > 127 else mem[o]

    def get_long(mem, o):
        return int.from_bytes(mem[o:o + 8], "little", signed=True)

    def reverse_bytes(v):
        return int.from_bytes((v & (2**64 - 1)).to_bytes(8, "little"), "big", signed=True)

    def compare_unsigned(a, b):
        a, b = a & (2**64 - 1), b & (2**64 - 1)
        return (a > b) - (a < b)

    i = 0
    if left_len != right_len:
        return left_len - right_len
    if not unaligned and left_off % 8 == right_off % 8:
        while (left_off + i) % 8 != 0 and i < left_len:
            v1, v2 = get_byte(mem_l, left_off + i), get_byte(mem_r, right_off + i)
            if v1 != v2:
                return 1 if (v1 & 0xFF) > (v2 & 0xFF) else -1
            i += 1
    if unaligned or ((left_off + i) % 8 == 0 and (right_off + i) % 8 == 0):
        while i <= left_len - 8:
            v1, v2 = get_long(mem_l, left_off + i), get_long(mem_r, right_off + i)
            if v1 != v2:
                return compare_unsigned(reverse_bytes(v1), reverse_bytes(v2))  # little-endian
            i += 8
    while i < left_len:
        v1, v2 = get_byte(mem_l, left_off + i), get_byte(mem_r, right_off + i)
        if v1 != v2:
            return 1 if (v1 & 0xFF) > (v2 & 0xFF) else -1
        i += 1
    return 0


def sign(x):
    return (x > 0) - (x < 0)


def pairs(rng):
    """random and adversarial row pairs: a difference in the last byte, in a high bit, inside and across 8-byte
    words, different lengths, equal rows"""
    out = []
    for n in (0, 1, 7, 8, 9, 15, 16, 17, 24, 40, 63, 64, 100):
        a = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        out.append((a, a))
        out.append((a, bytes(rng.integers(0, 256, n, dtype=np.uint8))))
        out.append((a, a + b"\0"))
        out.append((a + b"\xff", a))
        for p in range(n):
            for flip in (0x01, 0x80, 0xFF):
                b = bytearray(a)
                b[p] ^= flip
                out.append((a, bytes(b)))
        if n >= 16:
            b = bytearray(a)
            b[7] ^= 0x80
            b[8] ^= 0x01  # across a word boundary
            out.append((a, bytes(b)))
    return out


@pytest.mark.parametrize("unaligned", [True, False])
def test_record_binary_comparator_is_length_then_unsigned_lexicographic(unaligned):
    rng = np.random.default_rng(1)
    for a, b in pairs(rng):
        want = sign(len(a) - len(b)) if len(a) != len(b) else sign((a > b) - (a < b))
        for lo, ro in ((0, 0), (3, 3), (1, 6), (8, 5), (5, 16)):
            ml, mr = bytes(lo) + a + bytes(9), bytes(ro) + b + bytes(9)
            assert sign(record_binary_compare(ml, lo, len(a), mr, ro, len(b), unaligned)) == want, (a, b, lo, ro)
            assert sign(record_binary_compare(mr, ro, len(b), ml, lo, len(a), unaligned)) == -want


def test_sort_key_is_signed_hash_then_comparator():
    rng = np.random.default_rng(2)
    rows = [bytes(rng.integers(0, 256, 8 * int(rng.integers(0, 6)), dtype=np.uint8)) for _ in range(300)]
    rows += rows[:40]
    order = rr.sorted_order(rows, True, 7)
    hs = [rr.row_hash(rows[i]) for i in order]
    assert hs == sorted(hs) and any(h < 0 for h in hs) and any(h > 0 for h in hs)
    for x, y in zip(order, order[1:]):
        if rr.row_hash(rows[x]) == rr.row_hash(rows[y]):
            a, b = rows[x], rows[y]
            ml, mr = a + bytes(8), b + bytes(8)
            assert record_binary_compare(ml, 0, len(a), mr, 0, len(b), True) <= 0


def test_vectorised_order_equals_scalar():
    rng = np.random.default_rng(3)
    rows = [bytes(rng.integers(0, 4, 8 * int(rng.integers(0, 4)), dtype=np.uint8)) for _ in range(2000)]
    recs, rl = hm.records_of(rows)
    for R in (1, 2, 129):
        for sort in (0, 1):
            want = rr.sorted_order(rows, sort, R)
            got = rr.sorted_order_np(recs, rl, sort, R)
            assert [rows[i] for i in got] == [rows[i] for i in want]


def test_ids_and_the_single_partition_rule():
    assert rr.ids(5, 0, 3) == [1, 2, 0, 1, 2]
    assert rr.ids(4, 2, 3) == [0, 1, 2, 0]
    assert rr.ids(3, 0, 1) == [0, 0, 0]
    rows = [b"\x01" * 8, b"\x00" * 8, b"\x02" * 16]
    assert rr.sorted_order(rows, True, 1) == [0, 1, 2]  # R == 1: nothing is sorted
    assert rr.sorted_order(rows, False, 5) == [0, 1, 2]
    recs, rl = hm.records_of(rows)
    wr, wl, wid = rr.writer_records(recs, rl, 1, 4, True)
    order = rr.sorted_order(rows, True, 4)
    assert wr.tobytes() == b"".join(len(rows[i]).to_bytes(4, "big") + rows[i] for i in order)
    assert list(wl) == [rl[i] for i in order] and list(wid) == [2, 3, 0]
