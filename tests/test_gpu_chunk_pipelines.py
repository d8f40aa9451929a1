"""The host-pointer calls' software pipelines, at every slot count.

b2s_compress_* / b2s_decompress_* / b2s_decompressed_size_batch / b2s_checksum_* cut a batch into chunks of
B2S_HOST_CHUNK_MB (256 MiB) or 2^18 streams and rotate them over the slots (b2s_init's streams_per_gpu, 2..8; the read
side runs its three stages B2S_READ_LAG chunks apart).  Inside a chunk, codec blocks go through the compress passes in
groups of B2S_LZ4_CHUNK_BLOCKS and through Snappy's decode passes in groups of B2S_LZ4D_CHUNK_BLOCKS, two workspaces
alternating.  At the default sizes a test batch is one chunk and one group, so these tests shrink them: each
configuration runs tests/chunk_pipeline_worker.py in its own process (the sizes are read once, by b2s_init), which
checks every output against the CPU reference and reports what the calls reached.  One more test crosses the 2^18-stream
cut at the default settings, in this process."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "chunk_pipeline_worker.py")
KNOBS = ("B2S_SLOTS", "B2S_HOST_CHUNK_MB", "B2S_READ_LAG", "B2S_LZ4_CHUNK_BLOCKS", "B2S_LZ4D_CHUNK_BLOCKS")
CONFIGS = {
    # two slots: the read pipeline's lag-1 stages need the download of chunk c-2 before chunk c restages its slot
    "slots2": {"B2S_SLOTS": "2", "B2S_HOST_CHUNK_MB": "1"},
    "slots3": {"B2S_SLOTS": "3", "B2S_HOST_CHUNK_MB": "1", "B2S_READ_LAG": "1"},
    "slots6": {"B2S_SLOTS": "6", "B2S_HOST_CHUNK_MB": "1", "B2S_READ_LAG": "2"},
    "slots8": {"B2S_SLOTS": "8", "B2S_HOST_CHUNK_MB": "1", "B2S_READ_LAG": "3"},
    # one chunk, many codec-block groups: the first group, workspace reuse from the third on, a short last group
    "blocks": {"B2S_LZ4_CHUNK_BLOCKS": "3", "B2S_LZ4D_CHUNK_BLOCKS": "5"},
}
CHECKS = (["checksum_batch/%d" % a for a in (1, 2, 3)] + ["checksum_packed/%d" % a for a in (1, 2, 3)] +
          ["compress_%s/%s" % (f, s) for f in ("batch", "packed") for s in ("lz4-32k", "lz4-4k", "snappy", "zstd1", "zstd3")]
          + ["decompress_%s/%s" % (f, c) for f in ("batch", "packed") for c in ("lz4", "snappy", "zstd")])
BLOCK_CHECKS = (["compress_dev/%s" % s for s in ("lz4-32k", "lz4-4k", "snappy", "zstd1", "zstd3")] +
                ["decompress_dev/%s" % c for c in ("lz4", "snappy", "zstd")] +
                ["partition_compress_packed/%s" % c for c in ("lz4", "snappy", "zstd")] + ["decompress_sort_packed/snappy"])


@pytest.fixture(scope="module")
def zmodel_lib(tmp_path_factory):
    """the Zstd encoder's CPU model (tests/native/zstd_core_host.cpp), as test_gpu_zstd.py builds it"""
    out = str(tmp_path_factory.mktemp("zc") / "libzc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "native", "zstd_core_host.cpp")])
    return out


@pytest.mark.parametrize("config", list(CONFIGS))
def test_chunk_pipeline_configuration(config, zmodel_lib):
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(CONFIGS[config])
    r = subprocess.run([sys.executable, WORKER, config, zmodel_lib], env=env, cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    tail = "\n--- worker stderr ---\n" + r.stderr[-3000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert r.returncode == 0 and len(lines) == 1, "worker exit code %d%s" % (r.returncode, tail)
    out = json.loads(lines[0])
    print(config, json.dumps(out["reach"]))
    failed = {k: v for k, v in out["checks"].items() if v != "ok"}
    assert not failed, json.dumps(failed, indent=1) + tail
    want = CHECKS + (BLOCK_CHECKS if config == "blocks" else [])
    assert sorted(out["checks"]) == sorted(want)
    reach = out["reach"]
    calls = ["compress"] + ["decompress/" + c for c in ("lz4", "snappy", "zstd")]
    if config == "blocks":
        # one chunk per call; every compress setting and both Snappy decodes run at least three block groups, so
        # the third reuses the first one's workspace, and end in a short group
        assert all(reach[c]["chunks"] == 1 for c in calls + ["checksum"])
        grouped = {k: v for k, v in reach.items() if "groups" in k}
        assert len(grouped) == 7
        for k, (n_groups, last) in grouped.items():
            per = out["compress_group"] if k.startswith("compress") else out["snappy_decode_group"]
            assert n_groups >= 3 and 0 < last < per, (k, n_groups, last)
    else:
        # every slot is reused, and chunk c holds a different number of streams than chunk c - 2 somewhere
        assert reach["checksum"]["chunks"] > 1
        for c in calls:
            assert reach[c]["slot_reuses"] >= 1 and reach[c]["count_changes_c_vs_c2"] >= 1, (c, reach[c])
        assert out["slots"] == int(CONFIGS[config]["B2S_SLOTS"])


def test_more_streams_than_one_chunk_holds(capi, oracle):
    """2^18 + 1000 streams of 0-200 B at the default settings: every call cuts the batch at 2^18 streams, so each runs
    two chunks.  LZ4 streams equal the compressor's CPU specification; every codec round-trips, its checksums equal
    the oracle's, and the decoded streams land where dst_off says."""
    n = (1 << 18) + 1000
    rng = np.random.default_rng(31)
    ln = rng.integers(0, 201, n).astype(np.uint64)
    total = int(ln.sum())
    src = np.frombuffer(oracle.gen_terasort(5, total // 104 + 1).tobytes(), np.uint8)[:total].copy()
    src[rng.integers(0, total, total // 3)] = 0  # some easier matches
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    alg = capi.CHECKSUM_CRC32C
    for codec in (capi.CODEC_LZ4BLOCK, capi.CODEC_SNAPPY_XERIAL, capi.CODEC_ZSTD):
        cap = sum(capi.compress_bound(codec, 32768, int(l)) for l in ln) + 64
        dst = np.zeros(cap, np.uint8)
        r = capi.compress_packed(codec, src, off, ln, dst, 32768, alg)
        assert (r["status"] == 0).all(), codec
        dl, do = r["dst_len"], r["dst_off"]
        assert np.array_equal(do, np.concatenate([[0], np.cumsum(dl)[:-1]]).astype(np.uint64))
        assert r["total"] == int(dl.sum())
        streams = [dst[int(o):int(o + l)].tobytes() for o, l in zip(do, dl)]
        if codec == capi.CODEC_LZ4BLOCK:
            bad = [i for i in range(n) if streams[i] != oracle.lz4block_compress(
                src[int(off[i]):int(off[i] + ln[i])].tobytes(), 32768, compressor=1)]
            assert not bad, "%d streams differ from the specification, first %d" % (len(bad), bad[0])
        cks = capi.checksum_packed(alg, dst, do, dl)
        assert np.array_equal(cks, r["checksums"])
        want = [oracle.crc32c(s) for s in streams]
        assert [int(v) for v in cks] == want
        out = np.zeros(total, np.uint8)
        d = capi.decompress_packed(codec, dst[:r["total"]], do, dl, out, alg, np.arange(n + 1, dtype=np.uint32), dl, cks)
        assert (d["status"] == 0).all(), codec
        assert np.array_equal(d["dst_len"], ln) and np.array_equal(d["dst_off"], off) and d["total"] == total
        assert np.array_equal(out, src), codec
