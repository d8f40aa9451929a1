"""Runs the natives of jni/b200shuffle_jni.c without a JVM: builds the shim and a stand-in JNIEnv
(tests/native/jni_env_host.c), and calls every native as its Scala declaration in INTEGRATION.md §2 says a JVM would.

    shim = load()
    r = shim.call("decompressPacked", codec=1, alg=3, n=2, src=..., off=np.array([...], np.int64), ..., badSlice=None)
    r.rc, r.arrays["status"], r.string

Arguments go by Scala parameter name; a numpy array becomes a typed Java array of the declared element type (its bits
reinterpreted, so uint64 lengths pass as long[]), None a null reference, and a ByteBuffer parameter takes a
DirectBuffer.  Every call runs on the calling thread's env in the mode asked for ("direct": critical regions point into
the array, as HotSpot gives; "copy": they are fresh copies, copied back only by a mode-0 Release), and fails unless
the env recorded no violation."""
import ctypes as C
import os
import re
import subprocess
import tempfile
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_SRC = os.path.join(ROOT, "jni", "b200shuffle_jni.c")
ENV_SRC = os.path.join(ROOT, "tests", "native", "jni_env_host.c")
PREFIX = "Java_org_apache_spark_shuffle_gpu_B200Codec_"
MODES = ("direct", "copy")

# the shim's gcc flags (test_jni_shim.py compiles it the same way)
CFLAGS = ["-std=c11", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared"]

# Scala type -> (JNI C type, ctypes type, array element kind)
SCALA_TYPES = {
    "Int": ("jint", C.c_int32, None),
    "Long": ("jlong", C.c_int64, None),
    "Unit": ("void", None, None),
    "String": ("jstring", C.c_void_p, None),
    "java.nio.ByteBuffer": ("jobject", C.c_void_p, None),
    "Array[Long]": ("jlongArray", C.c_void_p, ("J", np.int64)),
    "Array[Int]": ("jintArray", C.c_void_p, ("I", np.int32)),
    "Array[Byte]": ("jbyteArray", C.c_void_p, ("B", np.int8)),
}

# the arrays each native writes; every other array is an input, which the call must leave unchanged
OUTPUTS = {"dstOff", "dstLen", "meta", "checksums", "status", "badSlice", "outLen", "out", "out8"}
OUTPUTS_OF = {"exchangeLookup": {"len"}}


def outputs_of(name):
    out = set(OUTPUTS) | OUTPUTS_OF.get(name, set())
    if name.startswith("partitionCompress") and "Cached" in name:
        out.add("cached")  # the writers' stored flag; the exchange reads take cached as an input
    return out


def scala_natives(path=os.path.join(ROOT, "INTEGRATION.md")):
    """{name: ([(param, Scala type), ...], Scala return type)} of every @native def of the Scala object"""
    text = open(path).read()
    out = {}
    for m in re.finditer(r"@native def (\w+)\((.*?)\): ([\w.\[\]]+)", text, re.S):
        params = []
        for p in filter(None, (s.strip() for s in m.group(2).split(","))):
            name, typ = (s.strip() for s in p.split(":"))
            params.append((name, typ))
        out[m.group(1)] = (params, m.group(3))
    return out


def c_natives(path=SHIM_SRC):
    """{name: ([(param, JNI C type), ...], C return type)} of every JNIEXPORT of the shim, JNIEnv* and jclass left out"""
    src = open(path).read()
    out = {}
    for m in re.finditer(r"JNIEXPORT (\w+) JNICALL J\((\w+)\)\(JNIEnv\* e, jclass c(.*?)\)\s*\{", src, re.S):
        params = [tuple(reversed(p.split())) for p in (s.strip() for s in m.group(3).split(",")) if p]
        out[m.group(2)] = ([(n, t) for n, t in params], m.group(1))
    return out


class DirectBuffer:
    """a java.nio.ByteBuffer allocated direct over [address, address + capacity)"""

    def __init__(self, address, capacity):
        self.address, self.capacity = address, capacity


class Result:
    def __init__(self, rc, arrays, string, obj):
        self.rc, self.arrays, self.string, self.obj = rc, arrays, string, obj


class Violation(AssertionError):
    pass


_built = {}
_lock = threading.Lock()


def build():
    """-> (shim .so, env .so) in a temporary directory; the shim links libb200shuffle.so by an rpath to the library
    pkg.build() made, so it binds to the instance capi loaded"""
    with _lock:
        if not _built:
            import spark_s3_shuffle_b200 as pkg

            lib = pkg.build()
            pkg.capi.load()  # the library instance the shim must share
            d = tempfile.mkdtemp(prefix="b2s_jni_")
            shim, env = os.path.join(d, "libb200shuffle_jni.so"), os.path.join(d, "libjni_env_host.so")
            stub = "-I" + os.path.join(ROOT, "jni", "stub")
            subprocess.check_call(["gcc", *CFLAGS, stub, "-I" + os.path.join(ROOT, "include"), SHIM_SRC, "-o", shim,
                                   "-L" + os.path.dirname(lib), "-l:libb200shuffle.so", "-Wl,-z,defs",
                                   "-Wl,-rpath," + os.path.dirname(lib)])
            subprocess.check_call(["gcc", *CFLAGS, stub, ENV_SRC, "-o", env])
            _built.update(shim=shim, env=env)
        return _built["shim"], _built["env"]


class Shim:
    def __init__(self):
        shim, env = build()
        self.env_lib = E = C.CDLL(env)
        E.jenv_new.restype = C.c_void_p
        E.jenv_new.argtypes = [C.c_int]
        E.jenv_array.restype = C.c_void_p
        E.jenv_array.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_void_p, C.c_int]
        E.jenv_direct_buffer.restype = C.c_void_p
        E.jenv_direct_buffer.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        E.jenv_data.restype = C.c_void_p
        E.jenv_data.argtypes = [C.c_void_p]
        E.jenv_length.restype = C.c_int32
        E.jenv_length.argtypes = [C.c_void_p]
        E.jenv_buffer_address.restype = C.c_void_p
        E.jenv_buffer_address.argtypes = [C.c_void_p]
        E.jenv_buffer_capacity.restype = C.c_int64
        E.jenv_buffer_capacity.argtypes = [C.c_void_p]
        E.jenv_check.restype = C.c_char_p
        E.jenv_check.argtypes = [C.c_void_p]
        E.jenv_free_objects.argtypes = [C.c_void_p]
        E.jenv_free.argtypes = [C.c_void_p]
        self.lib = C.CDLL(shim)
        self.decls = scala_natives()
        self.fns = {}
        for name, (params, ret) in self.decls.items():
            f = getattr(self.lib, PREFIX + name)
            f.restype = SCALA_TYPES[ret][1]
            f.argtypes = [C.c_void_p, C.c_void_p] + [SCALA_TYPES[t][1] for _, t in params]
            self.fns[name] = f
        self._local = threading.local()

    def env(self, mode):
        """the calling thread's env of that mode (one per thread, as a JVM gives)"""
        envs = self._local.__dict__.setdefault("envs", {})
        if mode not in envs:
            envs[mode] = self.env_lib.jenv_new(MODES.index(mode))
        return envs[mode]

    def _array(self, env, kind, dtype, value, is_input):
        a = np.ascontiguousarray(value)
        if a.dtype.itemsize != np.dtype(dtype).itemsize or a.dtype.kind not in "iub":
            a = a.astype(dtype)
        a = np.ascontiguousarray(a.view(dtype))
        h = self.env_lib.jenv_array(env, ord(kind), a.size, a.ctypes.data if a.size else None, int(is_input))
        assert h, "jenv_array"
        return h

    def read(self, obj, dtype):
        n = self.env_lib.jenv_length(obj)
        return np.ctypeslib.as_array((C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(
            self.env_lib.jenv_data(obj))).view(dtype).copy() if n > 0 else np.zeros(0, dtype)

    def call(self, name, mode="direct", allow_violation=False, **kw):
        """calls native name with its Scala parameters by name -> Result(rc, {array param: its elements after the
        call}, string or None, returned object handle or None).  Fails if the env recorded a violation."""
        params, ret = self.decls[name]
        missing = {p for p, _ in params} ^ set(kw)
        assert not missing, "%s: arguments %s do not match the declaration" % (name, sorted(missing))
        env = self.env(mode)
        outs = outputs_of(name)
        args, arrays = [], {}
        for p, t in params:
            v = kw[p]
            kind = SCALA_TYPES[t][2]
            if kind is not None:
                h = None if v is None else self._array(env, kind[0], kind[1], v, p not in outs)
                arrays[p] = (h, kind[1])
                args.append(h)
            elif t == "java.nio.ByteBuffer":
                args.append(None if v is None else v if isinstance(v, int) else
                            self.env_lib.jenv_direct_buffer(env, v.address, v.capacity))
            else:
                args.append(v)
        try:
            rc = self.fns[name](env, None, *args)
            log = self.env_lib.jenv_check(env).decode()
            got = {p: (None if h is None else self.read(h, dt)) for p, (h, dt) in arrays.items()}
            string = obj = None
            if ret == "String" and rc:
                string = C.string_at(self.env_lib.jenv_data(rc)).decode("utf-8")
            elif ret == "java.nio.ByteBuffer" and rc:
                obj = DirectBuffer(self.env_lib.jenv_buffer_address(rc), self.env_lib.jenv_buffer_capacity(rc))
        finally:
            self.env_lib.jenv_free_objects(env)
        if log and not allow_violation:
            raise Violation("%s (%s env): %s" % (name, mode, log))
        r = Result(rc, got, string, obj)
        r.violations = log
        return r


_shim = None


def load():
    """the process's one Shim (built on first use)"""
    global _shim
    if _shim is None:
        _shim = Shim()
    return _shim
