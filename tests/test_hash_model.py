"""The Murmur3 model of Spark's HashPartitioning (tests/hash_model.py), without a GPU: the scalar form reproduces Spark's
published vectors, and the vectorised form that the GPU tests use at scale equals the scalar form on random rows of
every key type, nulls, signed zeros, NaN payloads, every string tail length and decimals of 1..16 bytes included."""
import numpy as np
import pytest

import hash_model as hm


def test_scalar_model_reproduces_spark_murmur3_suite():
    """Murmur3_x86_32Suite, seed 0"""
    ints = [0, -42, 42, -2**31, 2**31 - 1]
    assert [hm.signed(hm.hash_int(v, 0)) for v in ints] == [593689054, -189366624, -1134849565, -1718298732,
                                                             -1653689534]
    longs = [0, -42, 42, -2**63, 2**63 - 1]
    assert [hm.signed(hm.hash_long(v, 0)) for v in longs] == [1669671676, -846261623, 1871679806, 1366273829,
                                                               -2106506049]


def test_scalar_model_reproduces_spark_sql_hash():
    """hash('Spark', array(123), 2) = -1321691492: a 5-byte string (one tail byte), then two ints folded as running
    seeds; SELECT hash(1) = -559580957"""
    h = hm.hash_bytes(b"Spark", hm.SEED)
    h = hm.hash_int(123, h)
    h = hm.hash_int(2, h)
    assert hm.signed(h) == -1321691492
    assert hm.signed(hm.hash_int(1, hm.SEED)) == -559580957


def test_tail_bytes_are_sign_extended_one_at_a_time():
    """Spark's legacy tail: a byte >= 0x80 is mixed as a negative int, each byte on its own"""
    h = hm.SEED
    h = hm._mix_h1(h, hm._mix_k1((0x80 - 256) & hm.M32))
    assert hm.hash_bytes(b"\x80", hm.SEED) == hm._fmix(h, 1)
    assert hm.hash_bytes(b"\x80", hm.SEED) != hm.hash_bytes(b"\x80\x00", hm.SEED)


def test_row_of_only_null_keys_goes_to_pmod_42():
    types = ["int", "string"]
    row = hm.make_row(types, [None, None])
    keys = hm.keys_of(types, [0, 1])
    assert hm.row_hash(row, keys) == 42
    assert hm.pmod(42, 200) == 42 and hm.pmod(42, 7) == 0


def test_pmod_is_non_negative():
    assert hm.pmod(hm.hash_int(1, 42), 200) == (-559580957) % 200 == 43
    for R in (1, 2, 7, 65537):
        assert 0 <= hm.pmod(0x80000000, R) < R


@pytest.mark.parametrize("fields", [[0], [1], [2], [3], [4], [5], [6], [7], list(range(8)), [7, 0, 3, 1]])
def test_vectorised_model_equals_scalar_model(fields):
    rng = np.random.default_rng(len(fields) * 31 + fields[0])
    rows = hm.random_rows(rng, 600)
    keys = hm.keys_of(hm.COMPOSITE, fields)
    recs, rl = hm.records_of(rows)
    for R in (1, 7, 200, 65537):
        assert (hm.record_ids_np(recs, rl, keys, R) == hm.ids_scalar(rows, keys, R)).all()
    start = np.concatenate([[0], np.cumsum(rl.astype(np.int64))[:-1]]) + 4
    assert (hm.row_hash_np(recs, start, keys) == np.array([hm.row_hash(r, keys) for r in rows], np.uint32)).all()


def test_vectorised_model_covers_every_string_tail_and_long_strings():
    rng = np.random.default_rng(5)
    types = ["string", "long"]
    strs = [bytes(rng.integers(0x80, 256, ln, dtype=np.uint8)) for ln in range(0, 70)]
    strs += [bytes(rng.integers(0, 256, hm.LONG_BYTES + d, dtype=np.uint8)) for d in (-1, 0, 1, 3)]
    rows = [hm.make_row(types, [s, i]) for i, s in enumerate(strs)]
    keys = hm.keys_of(types, [0, 1], nullable=False)
    recs, rl = hm.records_of(rows)
    assert (hm.record_ids_np(recs, rl, keys, 2000) == hm.ids_scalar(rows, keys, 2000)).all()


def test_float_keys_fold_signed_zero_and_nan_payloads():
    types = ["double", "float"]
    keys = hm.keys_of(types, [0, 1])
    a = hm.make_row(types, [0.0, 0.0])
    b = hm.make_row(types, [-0.0, -0.0])
    assert hm.row_hash(a, keys) == hm.row_hash(b, keys)
    nans = [hm.make_row(types, [("bits", d), ("bits", f)])
            for d, f in ((0x7FF8000000000000, 0x7FC00000), (0xFFF0000000000001, 0xFF800001))]
    assert hm.row_hash(nans[0], keys) == hm.row_hash(nans[1], keys)
    assert hm.row_hash(a, keys) == hm.hash_int(0, hm.hash_long(0, 42))
