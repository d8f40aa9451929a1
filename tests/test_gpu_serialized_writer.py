"""The GPU serialized writer of the host mirror (b2sh_serialized_writer_*): records inserted one by one with their reduce
id, in any partition order, as ShuffleExternalSorter.insertRecord receives them; commit partitions, compresses and
checksums them in one b2s_partition_compress_packed call.  Its .data/.index/.checksum must be byte for byte what the
existing writer (b2sh_writer) writes when fed the same records partition by partition, and the existing reader must
read every partition back with its records in insertion order."""
import os
import uuid

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from shuffle_model import decode_pairs, encode_pairs

pytestmark = pytest.mark.gpu
host = pkg.host


def conf_for(root, codec, alg):
    return {
        "spark.app.id": "app-" + uuid.uuid4().hex[:12],
        "spark.shuffle.s3.rootDir": "file://" + str(root) + "/spark-s3-shuffle",
        "spark.shuffle.checksum.enabled": True,
        "spark.shuffle.checksum.algorithm": alg,
        "spark.io.compression.codec": codec,
    }


def files(d, shuffle_id, map_id):
    out = {}
    for kind in ("data", "index", "checksum"):
        p = d.getPath(kind, shuffle_id, map_id)
        out[kind] = open(p, "rb").read() if os.path.exists(p) else None
    return out


def write_both(tmp_path, codec, alg, records, ids, n_red):
    """the same map output through the serialized writer and through the existing writer"""
    d_new = host.S3ShuffleDispatcher(conf_for(tmp_path / "new", codec, alg))
    d_old = host.S3ShuffleDispatcher(conf_for(tmp_path / "old", codec, alg))
    w = host.S3SerializedShuffleWriter(d_new, 0, 0, n_red)
    for rec, p in zip(records, ids):
        w.insertRecord(int(p), rec)
    lens_new = w.commit()
    w.close()
    o = host.S3ShuffleMapOutputWriter(d_old, 0, 0, n_red)
    for r in range(n_red):
        with o.getPartitionWriter(r) as s:
            for rec, p in zip(records, ids):
                if p == r:
                    s.write(rec)
    lens_old = o.commitAllPartitions()
    o.close()
    return d_new, d_old, lens_new, lens_old


@pytest.mark.parametrize("codec", ["lz4", "snappy", "zstd"])
@pytest.mark.parametrize("alg", ["ADLER32", "CRC32C"])
def test_foldByKey_shape_files_identical_and_readable(tmp_path, codec, alg):
    """foldByKey shape (test/S3ShuffleManagerTest.scala:176-205): ints keyed % 7, 5 reducers (so some partition gets
    every key of one residue and partitions stay uneven); records are (key, value) varint pairs"""
    n, n_red = 10_000, 5
    i = np.arange(n, dtype=np.int64)
    keys = (i * 7919) % 7
    records = [encode_pairs(keys[j:j + 1], i[j:j + 1]) for j in range(n)]
    ids = keys % n_red
    d_new, d_old, lens_new, lens_old = write_both(tmp_path, codec, alg, records, ids, n_red)
    assert list(lens_new) == list(lens_old)
    assert files(d_new, 0, 0) == files(d_old, 0, 0)
    for r in range(n_red):
        rd = host.S3ShuffleReader(d_new, 0, [0], r, r + 1)
        blocks = rd.read()
        rd.close()
        got = b"".join(b for _, b in blocks)
        assert got == b"".join(rec for rec, p in zip(records, ids) if p == r)  # insertion order kept
        k, _ = decode_pairs(got)
        assert (k % n_red == r).all()


def test_teraSortLike_with_empty_partitions(tmp_path, oracle):
    """teraSortLike (test/S3ShuffleManagerTest.scala:146-174): 104-byte records, range-partitioned on the key, more
    reducers than key ranges hit so several partitions stay empty"""
    n, n_red = 20_000, 64
    raw = np.frombuffer(oracle.gen_terasort(0, n).tobytes(), np.uint8).reshape(n, 104)
    records = [raw[j].tobytes() for j in range(n)]
    ids = (raw[:, 2].astype(np.int64) * 48) >> 8  # reducers 48..63 get nothing
    d_new, d_old, lens_new, lens_old = write_both(tmp_path, "lz4", "CRC32", records, ids, n_red)
    assert list(lens_new) == list(lens_old) and (lens_new[48:] == 0).all()
    assert files(d_new, 0, 0) == files(d_old, 0, 0)
    rd = host.S3ShuffleReader(d_new, 0, [0], 0, n_red)
    blocks = sorted(rd.read(), key=lambda blk: blk[0][1])  # block order is unspecified, as in the reference
    rd.close()
    assert b"".join(b for _, b in blocks) == b"".join(records[j] for j in np.argsort(ids, kind="stable"))


def test_invalid_partition_id_is_rejected(tmp_path):
    d = host.S3ShuffleDispatcher(conf_for(tmp_path, "lz4", "ADLER32"))
    w = host.S3SerializedShuffleWriter(d, 0, 0, 4)
    with pytest.raises(host.RuntimeException):
        w.insertRecord(4, b"abc")
    w.close()
