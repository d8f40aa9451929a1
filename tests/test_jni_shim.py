"""jni/b200shuffle_jni.c — the JNI layer a maintainer builds on the reference side (INTEGRATION.md §2) — compiled and
RUN without a JVM.

The file is compiled against jni/stub/jni.h with -Wall -Wextra -Werror (argument order and types against
include/b200shuffle.h, the exported Java_* names), and every native is called through tests/jni_shim.py: a stand-in
JNIEnv (tests/native/jni_env_host.c) that checks each call as -Xcheck:jni would, with guarded arrays and critical
regions either pointing into the array or copied.  These tests need no device: they check the signatures against the
Scala object, that each native reaches the library with well-formed arguments before b2s_init, and that the shim
itself rejects every null, short or out-of-range argument with B2S_E_ARG before the library sees it — the library
takes raw pointers, so an unchecked short Java array would be read or written past its end."""
import os
import re
import subprocess

import numpy as np
import pytest

import jni_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = jni_shim.SHIM_SRC

OK, E_ARG, E_CUDA, E_NOT_INIT = 0, -5, -6, -7
SENTINEL = 0x5A


def test_shim_compiles_against_the_c_abi_and_exports_every_native(tmp_path):
    import spark_s3_shuffle_b200 as pkg

    lib = pkg.build()
    so = str(tmp_path / "libb200shuffle_jni.so")
    subprocess.check_call(["gcc", *jni_shim.CFLAGS, "-I" + os.path.join(ROOT, "jni", "stub"),
                           "-I" + os.path.join(ROOT, "include"), SRC, "-o", so,
                           "-L" + os.path.dirname(lib), "-l:libb200shuffle.so", "-Wl,-z,defs"])
    exported = set(re.findall(r" T Java_org_apache_spark_shuffle_gpu_B200Codec_(\w+)",
                              subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout))
    declared = set(re.findall(r"J\((\w+)\)\(JNIEnv", open(SRC).read()))
    assert exported == declared and len(exported) >= 19
    # every @native of the Scala object in INTEGRATION.md has its C function, and vice versa
    natives = set(re.findall(r"@native def (\w+)\(", open(os.path.join(ROOT, "INTEGRATION.md")).read()))
    assert natives == exported, (natives ^ exported)


def test_every_critical_get_is_released_on_every_path():
    src = open(SRC).read()
    bodies = re.split(r"\nJNIEXPORT ", src)[1:]
    assert len(bodies) >= 19
    for b in bodies:
        name = re.search(r"J\((\w+)\)", b).group(1)
        gets = re.findall(r"(\w+) = crit_get\(e, (\w+)\)", b)
        puts = re.findall(r"crit_put\(e, (\w+), (\w+), (0|JNI_ABORT)\)", b)
        assert sorted((a, v) for v, a in gets) == sorted((a, v) for a, v, _ in puts), name
        if gets:  # single exit after the releases: no early return between the first get and the last put
            first, last = b.index("crit_get"), b.rindex("crit_put")
            assert "return" not in b[first:last], name


def test_every_native_has_its_scala_signature():
    """names, order and JNI types of the parameters, and the return type, of each native equal its declaration"""
    scala, c = jni_shim.scala_natives(), jni_shim.c_natives()
    assert set(scala) == set(c) and len(c) == 43
    for name, (params, ret) in scala.items():
        want = ([(p, jni_shim.SCALA_TYPES[t][0]) for p, t in params], jni_shim.SCALA_TYPES[ret][0])
        assert c[name] == want, name


# ---------------------------------------------------------------------------------------------------------------
# well-formed arguments, and the count that sizes each array
# ---------------------------------------------------------------------------------------------------------------
N = 3              # blocks / streams
SLICE_BASE = [0, 1, 3, 4]  # block 1 has two slices: 4 in all
P = 3              # numPartitions
NB = 2             # nBounds
NK, NA, NF, NFIELDS = 2, 2, 2, 3

# per native: {array parameter: the count that sizes it}.  "slices" is sliceBase[n]; a bare number is a fixed length
_BLOCKS = {"off": "n", "len": "n", "status": "n", "badSlice": "n", "sliceBase": "n+1", "sliceLen": "slices",
           "sliceChecksum": "slices"}
_KEYS = {"keyType": "nKeys", "keyOff": "nKeys", "keyLen": "nKeys", "keyNullField": "nKeys"}
_AGGS = {"aggOp": "nAggs", "aggOff": "nAggs", "aggNullField": "nAggs"}
_PARTS = {"dstOff": "numPartitions", "dstLen": "numPartitions", "meta": 1, "checksums": "numPartitions",
          "status": "numPartitions"}
_RANGE = {**_KEYS, "boundLen": "nBounds", **{k: "nBounds+1" for k in ("dstOff", "dstLen", "checksums", "status")},
          "meta": 1}
_WINDOW = {**_BLOCKS, **_KEYS, "fieldKind": "nFields", "fn": "nFns", "fnArg": "nFns", "meta": 3}
_WINDOW_AGG = {**_WINDOW, **{k: "nFns" for k in ("fnFrame", "valType", "valOff", "valNullField")}}
_EXCHANGE = {"mapIds": "n", "cached": "n"}
SIZES = {
    "compressPacked": {"off": "n", "len": "n", "dstOff": "n", "dstLen": "n", "meta": 1, "checksums": "n",
                       "status": "n"},
    "partitionCompressPacked": _PARTS,
    "partitionCompressRowsHashPacked": {**_KEYS, **_PARTS},
    "partitionCompressRowsRangePacked": _RANGE,
    "partitionCompressRowsRoundRobinPacked": _PARTS,
    "partitionCompressCachedPacked": {**_PARTS, "cached": 1},
    "partitionCompressRowsHashCachedPacked": {**_KEYS, **_PARTS, "cached": 1},
    "partitionCompressRowsRangeCachedPacked": {**_RANGE, "cached": 1},
    "partitionCompressRowsRoundRobinCachedPacked": {**_PARTS, "cached": 1},
    "decompressPacked": {**_BLOCKS, "dstOff": "n", "dstLen": "n", "meta": 1},
    "decompressedSizePacked": {"off": "n", "len": "n", "outLen": "n", "status": "n"},
    "decompressSortPacked": {**_BLOCKS, "meta": 2},
    "decompressSortRowsPacked": {**_BLOCKS, "meta": 2},
    "decompressAggregateRowsPacked": {**_BLOCKS, **_AGGS, "meta": 3},
    "decompressSortRowsKeysPacked": {**_BLOCKS, **_KEYS, "meta": 2},
    "decompressAggregateRowsKeysPacked": {**_BLOCKS, **_KEYS, **_AGGS, "meta": 3},
    "decompressJoinRowsKeysPacked": {**_BLOCKS, **{k: "nKeys" for k in (
        "keyType", "keyLen", "leftKeyOff", "leftKeyNullField", "rightKeyOff", "rightKeyNullField")},
        "leftFieldKind": "nLeftFields", "rightFieldKind": "nRightFields", "meta": 4},
    "decompressWindowRowsKeysPacked": _WINDOW,
    "decompressWindowAggregateRowsKeysPacked": _WINDOW_AGG,
    "decompressWindowOffsetRowsKeysPacked": {**_WINDOW_AGG, "fnFlags": "nFns", "fnDefault": "nFns"},
    "exchangeLookup": {"mapIds": "n", "len": "n"},
    "exchangeReadPacked": {"mapIds": "n", "dstOff": "n", "dstLen": "n", "meta": 1, "status": "n"},
    "exchangeReadSortPacked": {**_EXCHANGE, **_BLOCKS, "meta": 2},
    "exchangeReadSortRowsKeysPacked": {**_EXCHANGE, **_BLOCKS, **_KEYS, "meta": 2},
    "exchangeReadAggregateRowsKeysPacked": {**_EXCHANGE, **_BLOCKS, **_KEYS, **_AGGS, "meta": 3},
    "checksumPacked": {"off": "n", "len": "n", "out": "n"},
    "lastTiming": {"out8": 8},
}
# the arrays a native takes as null: the optional outputs, and the field kinds of semi and anti joins
OPTIONAL = {"checksums", "badSlice", "leftFieldKind", "rightFieldKind"}

# scalar arguments of a well-formed call
SCALARS = dict(codec=1, level=0, blockSize=0, alg=3, n=N, numPartitions=P, nRecords=2, recBytes=64, startPosition=0,
               sortRows=1, nKeys=NK, nBounds=NB, boundBytes=32, shuffleId=7, mapId=3, startReduce=0, endReduce=1,
               recordBytes=16, keyType=2, keyOff=8, keyLen=8, nullField=-1, nAggs=NA, joinType=0, nLeft=1,
               nLeftFields=NFIELDS, nRightFields=NFIELDS, nPartitionKeys=1, nFields=NFIELDS, nFns=NF, limitFn=-1,
               limit=0, dev=0, bytes=4096, gpuMask=1, pinnedBytesPerGpu=0, streamsPerGpu=0, code=0)
ADDRESSES = ("src", "dst", "records", "recLen", "recPart", "bounds", "base", "addr")

_arena = np.zeros(1 << 16, dtype=np.uint8)  # what src / dst / records / bounds point at


def _array_values(name, param, n, dtype):
    """the elements of a well-formed array argument"""
    if param == "sliceBase":
        return np.array(SLICE_BASE[: n], dtype)
    if param in ("off",):
        return np.arange(n, dtype=dtype) * 100
    if param == "len":
        return np.full(n, 100, dtype)
    if param == "sliceLen":  # block 1's two slices make up its 100 bytes
        return np.array([100, 50, 50, 100][:n], dtype)
    if param == "boundLen":
        return np.full(n, 16, dtype)
    if param == "keyType":  # INT64, INT32
        return np.array([2, 1] * 9, dtype)[:n]
    if param == "aggOp":  # SUM_INT64, MIN_INT64
        return np.array([0, 4] * 9, dtype)[:n]
    if param in ("keyOff", "leftKeyOff", "rightKeyOff"):
        return 8 + 8 * np.arange(n, dtype=dtype)
    if param == "keyLen":
        return np.array([8, 4] * 9, dtype)[:n]
    if param == "aggOff":
        return 24 + 8 * np.arange(n, dtype=dtype)
    if param in ("keyNullField", "leftKeyNullField", "rightKeyNullField", "aggNullField", "valNullField"):
        return np.full(n, -1, dtype)
    if param == "mapIds":
        return np.arange(n, dtype=dtype) + 1
    if param == "cached" and "Cached" not in name:
        return np.array([1, 0] * 9, dtype)[:n]
    return np.zeros(n, dtype)


def count_value(kw, count):
    if isinstance(count, int):
        return count
    if count == "slices":
        return int(kw["sliceBase"][kw["n"]]) if kw.get("sliceBase") is not None else 0
    if count.endswith("+1"):
        return kw[count[:-2]] + 1
    return kw[count]


def well_formed(name):
    """the keyword arguments of a well-formed call of native name; outputs filled with SENTINEL bytes"""
    params, _ = jni_shim.scala_natives()[name]
    outs = jni_shim.outputs_of(name)
    kw = {}
    for p, t in params:
        if p in ADDRESSES:
            kw[p] = _arena.ctypes.data
        elif p in ("dstCap",):
            kw[p] = _arena.size
        elif p == "directBuffer":
            kw[p] = jni_shim.DirectBuffer(_arena.ctypes.data, _arena.size)
        elif p in SCALARS:
            kw[p] = SCALARS[p]
        elif not t.startswith("Array"):
            raise AssertionError("no value for %s.%s" % (name, p))
    sizes = SIZES.get(name, {})
    for p, t in params:  # sliceBase first: it sizes the slice arrays
        if t.startswith("Array"):
            dtype = jni_shim.SCALA_TYPES[t][2][1]
            n = count_value({**kw, "sliceBase": np.array(SLICE_BASE)}, sizes[p])
            kw[p] = (np.frombuffer(bytes([SENTINEL]) * (n * np.dtype(dtype).itemsize), dtype).copy() if p in outs
                     else _array_values(name, p, n, dtype))
    return kw


def _prime_last_error(L):
    """sets the thread's b2s_last_error to a text no argument check of the library writes"""
    L.b2s_set_thread_device(0xFFFF)
    return L.b2s_last_error()


@pytest.fixture(scope="module")
def shim():
    return jni_shim.load()


@pytest.fixture(scope="module")
def L():
    import spark_s3_shuffle_b200 as pkg

    return pkg.capi.load()


def test_every_array_argument_has_its_size_in_the_table():
    for name, (params, _) in jni_shim.scala_natives().items():
        arrays = {p for p, t in params if t.startswith("Array")}
        assert set(SIZES.get(name, {})) == arrays, name


# ---------------------------------------------------------------------------------------------------------------
# before b2s_init: every native reaches the library and writes only what its comment promises
# ---------------------------------------------------------------------------------------------------------------
# the outputs a failed call still writes: the writers' meta(0) = bytes and cached(0) = stored, the reads' meta counts
WRITTEN_ON_ERROR = {name: {"meta"} | ({"cached"} if "Cached" in name else set())
                    for name in SIZES if name.startswith(("partitionCompress", "decompressSort", "decompressAggregate",
                                                          "decompressJoin", "decompressWindow", "exchangeRead"))}
SIMPLE = {  # natives whose result is the C entry point's, called directly with the same arguments
    "shutdown": None, "deviceCount": "b2s_device_count", "setThreadDevice": "b2s_set_thread_device",
    "bindThreadToDevice": "b2s_bind_thread_to_device", "hostRegister": "b2s_host_register",
    "hostUnregister": "b2s_host_unregister", "exchangeSetBudget": "b2s_exchange_set_budget",
    "exchangeRemove": "b2s_exchange_remove", "compressBound": "b2s_compress_bound",
}


@pytest.mark.parametrize("mode", jni_shim.MODES)
def test_every_native_reaches_the_library_before_init(shim, L, mode):
    if L.b2s_device_count() != E_NOT_INIT:
        pytest.skip("the library is already initialised in this process")
    decls = jni_shim.scala_natives()
    done = set()
    for code in range(-9, 1):
        assert shim.call("strerror", mode=mode, code=code).string == L.b2s_strerror(code).decode()
    _prime_last_error(L)
    assert shim.call("lastError", mode=mode).string == L.b2s_last_error().decode()
    done |= {"strerror", "lastError"}
    for name, fn in SIMPLE.items():
        kw = well_formed(name)
        r = shim.call(name, mode=mode, **kw)
        if fn is not None:
            assert r.rc == getattr(L, fn)(*[kw[p] for p, _ in decls[name][0]]), name
        done.add(name)
    # pinned memory: hostAlloc is b2s_host_alloc (NULL without a device), wrap / addressOf round-trip the address
    p = shim.call("hostAlloc", mode=mode, bytes=4096).rc
    q = L.b2s_host_alloc(4096)
    assert bool(p) == bool(q)
    for a in (p, q):
        if a:
            L.b2s_host_free(a)
    shim.call("hostFree", mode=mode, addr=0)
    buf = shim.call("wrap", mode=mode, addr=_arena.ctypes.data, bytes=_arena.size).obj
    assert (buf.address, buf.capacity) == (_arena.ctypes.data, _arena.size)
    assert shim.call("addressOf", mode=mode, directBuffer=buf).rc == _arena.ctypes.data
    r = shim.call("lastTiming", mode=mode, out8=np.full(8, -1, np.int64))
    assert r.rc == OK and list(r.arrays["out8"]) == [0] * 8  # no call has run on this thread
    done |= {"hostAlloc", "hostFree", "wrap", "addressOf", "lastTiming"}
    # the device calls: the library's B2S_E_NOT_INIT (B2S_E_CUDA once b2s_init has failed for want of a device), with
    # its b2s_last_error text, and no output but what a failed call promises
    for name in sorted(set(decls) - done - {"init"}):
        kw = well_formed(name)
        primed = L.b2s_checksum_packed(0, 1, None, None, None, None) and L.b2s_last_error()
        r = shim.call(name, mode=mode, **kw)
        assert r.rc in (E_NOT_INIT, E_CUDA), (name, r.rc, L.b2s_last_error())
        assert L.b2s_last_error() != primed, name
        for p in jni_shim.outputs_of(name) & set(kw):
            if p in WRITTEN_ON_ERROR.get(name, ()):
                assert not r.arrays[p].any(), (name, p)
            else:
                assert r.arrays[p].tobytes() == kw[p].tobytes(), (name, p)
        done.add(name)
    # last, as it may change the library's state: b2s_init's own result
    rc = shim.call("init", mode=mode, gpuMask=1, pinnedBytesPerGpu=0, streamsPerGpu=0).rc
    assert rc in (OK, E_CUDA)
    if rc == OK:
        L.b2s_shutdown()
    assert done | {"init"} == set(decls)


# ---------------------------------------------------------------------------------------------------------------
# rejected arguments: B2S_E_ARG from the shim itself
# ---------------------------------------------------------------------------------------------------------------
COUNT_CASES = [("n", -1), ("nKeys", 0), ("nKeys", 17), ("nAggs", 17), ("nFns", 17), ("nBounds", -1),
               ("nBounds", 1 << 24), ("numPartitions", 0)]


def _rejected_cases():
    cases = []
    for name, sizes in SIZES.items():
        for p in sizes:
            if p not in OPTIONAL:
                cases.append((name, "null", p))
            cases.append((name, "short", p))
        params = {q for q, _ in jni_shim.scala_natives()[name][0]}
        for count, v in COUNT_CASES:
            if count in params:
                cases.append((name, "count", "%s=%d" % (count, v)))
    return cases


def rejected_call(name, how, what):
    """the keyword arguments of the rejected case"""
    kw = well_formed(name)
    if how == "null":
        kw[what] = None
    elif how == "short":
        kw[what] = kw[what][:-1]
    else:
        count, v = what.split("=")
        kw[count] = int(v)
        if 0 < int(v) <= 17:  # arrays the count sizes grow with it: only the count is out of range
            for p, c in SIZES[name].items():
                if c == count:
                    dt = kw[p].dtype
                    kw[p] = np.resize(kw[p], int(v)).astype(dt)
    return kw


REJECTED = _rejected_cases()


@pytest.mark.parametrize("mode", jni_shim.MODES)
@pytest.mark.parametrize("name,how,what", REJECTED, ids=["%s-%s-%s" % c for c in REJECTED])
def test_the_shim_rejects_the_argument(shim, L, mode, name, how, what):
    kw = rejected_call(name, how, what)
    primed = _prime_last_error(L)
    r = shim.call(name, mode=mode, **kw)  # fails on any violation: a guard overwritten, an input changed, ...
    assert r.rc == E_ARG, r.rc
    assert L.b2s_last_error() == primed, "the library, not the shim, rejected it: " + L.b2s_last_error().decode()
    for p in jni_shim.outputs_of(name) & set(kw):  # no output touched
        if kw[p] is not None:
            assert r.arrays[p].tobytes() == kw[p].tobytes(), p


def test_the_rejected_cases_cover_every_array_and_count():
    names = {c[0] for c in REJECTED}
    assert names == set(SIZES)
    for name in ("compressPacked", "decompressPacked", "checksumPacked", "decompressedSizePacked"):
        assert (name, "count", "n=-1") in REJECTED
    assert ("lastTiming", "null", "out8") in REJECTED
