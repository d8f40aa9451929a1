"""libzstd.so.1 (1.5.5 — the library zstd-jni 1.5.5-x bundles) through ctypes: the reference Zstandard implementation
used to pin our decoder/encoder.  Test infrastructure only."""
import ctypes as C

_z = None


def lib():
    global _z
    if _z is None:
        z = C.CDLL("libzstd.so.1")
        z.ZSTD_compressBound.restype = C.c_size_t
        z.ZSTD_compressBound.argtypes = [C.c_size_t]
        z.ZSTD_compress.restype = C.c_size_t
        z.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
        z.ZSTD_decompress.restype = C.c_size_t
        z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        z.ZSTD_isError.restype = C.c_uint
        z.ZSTD_isError.argtypes = [C.c_size_t]
        z.ZSTD_createCCtx.restype = C.c_void_p
        z.ZSTD_freeCCtx.argtypes = [C.c_void_p]
        z.ZSTD_CCtx_setParameter.restype = C.c_size_t
        z.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
        z.ZSTD_compressStream2.restype = C.c_size_t
        z.ZSTD_compressStream2.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        z.ZSTD_createDCtx.restype = C.c_void_p
        z.ZSTD_freeDCtx.argtypes = [C.c_void_p]
        z.ZSTD_decompressStream.restype = C.c_size_t
        z.ZSTD_decompressStream.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _z = z
    return _z


class _Buf(C.Structure):
    _fields_ = [("p", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


def compress(data, level=3):
    z = lib()
    cap = z.ZSTD_compressBound(len(data))
    buf = C.create_string_buffer(cap)
    n = z.ZSTD_compress(buf, cap, data, len(data), level)
    assert not z.ZSTD_isError(n)
    return buf.raw[:n]


def compress_stream(data, level=1, chunk=32768, flush_every=0):
    """What zstd-jni's ZstdOutputStreamNoFinalizer does under Spark's BufferedOutputStream(32 KiB): a streaming frame —
    no Frame_Content_Size, window descriptor present — fed in 32 KiB writes, ended with ZSTD_e_end."""
    return compress_stream_params(data, [(100, level)], chunk, flush_every)  # ZSTD_c_compressionLevel


# libzstd 1.5.5 ZSTD_cParameter ids
P_LEVEL, P_WINDOW_LOG, P_STRATEGY, P_LDM, P_CHECKSUM, P_WORKERS, P_JOB_SIZE, P_LITERAL_MODE = (
    100, 101, 107, 160, 201, 400, 401, 1002)
_P_BLOCK_DELIMITERS, _P_VALIDATE_SEQUENCES, _P_SEARCH_REPCODES = 1008, 1009, 1016


def _set(z, c, params):
    for k, v in params:
        rc = z.ZSTD_CCtx_setParameter(c, k, v)
        assert not z.ZSTD_isError(rc), "ZSTD_CCtx_setParameter(%d, %d) refused" % (k, v)


def compress_stream_params(data, params, chunk=32768, flush_every=0):
    """compress_stream with any (ZSTD_cParameter, value) pairs set on the context (level, strategy, window, long
    distance matching, checksum, workers, literal compression mode ...)"""
    z = lib()
    c = z.ZSTD_createCCtx()
    _set(z, c, params)
    out = b""
    ob = C.create_string_buffer(1 << 17)
    src = C.create_string_buffer(data, len(data)) if data else C.create_string_buffer(1)
    base = C.addressof(src)
    pos = 0
    k = 0
    while True:
        n = min(chunk, len(data) - pos)
        last = pos + n >= len(data)
        ib = _Buf(base + pos, n, 0)
        mode = 2 if last else (1 if flush_every and (k + 1) % flush_every == 0 else 0)  # end / flush / continue
        while True:
            o = _Buf(C.addressof(ob), len(ob), 0)
            rem = z.ZSTD_compressStream2(c, C.byref(o), C.byref(ib), mode)
            assert not z.ZSTD_isError(rem)
            out += ob.raw[:o.pos]
            if (mode == 0 and ib.pos == ib.size) or (mode != 0 and rem == 0):
                break
        pos += n
        k += 1
        if last:
            break
    z.ZSTD_freeCCtx(c)
    return out


class _Seq(C.Structure):  # ZSTD_Sequence
    _fields_ = [("offset", C.c_uint), ("litLength", C.c_uint), ("matchLength", C.c_uint), ("rep", C.c_uint)]


def execute_sequences(blocks, seed=0, alphabet=b"etaoinshrdlucmfwypvbgkqjxz0123456789 \n"):
    """Plain executor of a sequence plan: blocks = [(seqs, last_ll)], seqs = [(literal_len, offset, match_len)].
    Literals are random bytes of `alphabet` (skewed enough for Huffman literals); matches copy byte by byte, so an
    offset shorter than the match repeats.  Returns the frame's content, which is what a decoder of
    compress_sequences(content, blocks) must produce."""
    import random
    rng = random.Random(seed)
    out = bytearray()
    for seqs, last_ll in blocks:
        for ll, off, ml in seqs:
            out += bytes(rng.choice(alphabet) for _ in range(ll))
            assert 1 <= off <= len(out), (off, len(out))
            for _ in range(ml):
                out.append(out[-off])
        out += bytes(rng.choice(alphabet) for _ in range(last_ll))
    return bytes(out)


# The six repeat-offset forms (offset value, literal length == 0) of RFC 8878 3.1.1.5
REP_FORMS = [(1, False), (2, False), (3, False), (1, True), (2, True), (3, True)]


def resolve_offset(reps, ofv, ll0):
    """RFC 8878 3.1.1.5: (offset, new repeat offsets) for a repeat code ofv in 1..3"""
    r0, r1, r2 = reps
    idx = ofv - 1 + (1 if ll0 else 0)
    if idx == 0:
        return r0, reps
    off = r1 if idx == 1 else r2 if idx == 2 else r0 - 1
    return off, ((off, r0, r2) if idx == 1 else (off, r0, r1))


def plan_sequences(token_blocks, seed=0):
    """Turns blocks of tokens — 'N' (a new offset) or a REP_FORMS entry — into sequence blocks for compress_sequences,
    choosing offsets so that libzstd writes exactly that form: the three repeat offsets stay distinct, and a new offset
    never equals one libzstd would turn into a repeat code.  A form that is impossible at its place (offset rep0 - 1
    when that is 0 or another repeat offset; an offset beyond the output so far) becomes a new offset.
    -> (blocks, expected offset values in sequence order: 1..3 repeat codes, offset + 3 otherwise)"""
    import random
    rng = random.Random(seed)
    reps, pos, blocks, expect = (1, 4, 8), 0, [], []

    def lit_len():
        return rng.randint(33, 80) if rng.random() < 0.1 else rng.randint(1, 12)  # > 32: the warp-wide literal copy

    def match_len():
        return rng.randint(40, 300) if rng.random() < 0.05 else rng.randint(4, 24)

    for tokens in token_blocks:
        seqs = []
        for t in tokens:
            ll = off = None
            if t != "N":
                ofv, ll0 = t
                ll = 0 if ll0 else lit_len()
                off, nreps = resolve_offset(reps, ofv, ll0)
                # rep0 - 1 equal to rep1 or rep2 would be written as that repeat code instead
                if off < 1 or off > pos + ll or (ofv == 3 and ll0 and off in reps[1:]):
                    ll = off = None
                else:
                    reps = nreps
                    expect.append(ofv)
            if off is None:
                ll = 24 if pos == 0 else (0 if rng.random() < 0.15 else lit_len())
                while True:
                    off = rng.randint(5, 12) if rng.random() < 0.2 else rng.randint(16, max(16, min(pos + ll, 30000)))
                    if off <= pos + ll and off not in (reps[0], reps[1], reps[2], reps[0] - 1):
                        break
                reps = (off, reps[0], reps[1])
                expect.append(off + 3)
            ml = match_len()
            seqs.append((ll, off, ml))
            pos += ll + ml
        last_ll = rng.randint(0, 20)
        pos += last_ll
        blocks.append((seqs, last_ll))
    return blocks, expect


def repeat_offset_tokens(seed=0):
    """Token blocks that put every repeat-offset form where the GPU's batch of 32 sequences treats it differently: as
    the first repeat code of a batch at warp position 0, 1, 2, 3 and later (after a prefix of new offsets); as
    sequence 31 and 32 of a block; as the first sequence of a block that follows one ending in new offsets.  Every
    block ends with three new offsets; one batch has no repeat code at all."""
    import random
    rng = random.Random(seed)

    def batch(form, p):
        return ["N"] * p + [form] + [rng.choice(REP_FORMS + ["N"]) for _ in range(31 - p)]

    second = {0: 3, 1: 2, 2: 1, 3: 0, 5: 31, 17: 17, 31: 0}  # first repeat code of the second batch
    blocks = [["N"] * 5]
    for fi, form in enumerate(REP_FORMS):
        for pi, (p, q) in enumerate(second.items()):
            tail = [rng.choice(REP_FORMS + ["N"]) for _ in range(rng.randint(0, 30))]
            blocks.append(batch(form, p) + batch(REP_FORMS[(fi + 1 + pi) % 6], q) + tail + ["N"] * 3)
    blocks.append(["N"] * 40 + batch(REP_FORMS[5], 0)[:7] + ["N"] * 3)
    return blocks


def compress_sequences(src, blocks, level=3, raw_literals=False):
    """One frame whose blocks carry exactly the given sequences (ZSTD_compressSequences with explicit block
    delimiters).  libzstd itself decides which offsets become repeat codes (searchForExternalRepcodes), exactly as its
    match finders would: this is how the rarer repeat-offset forms are written on purpose."""
    z = lib()
    z.ZSTD_compressSequences.restype = C.c_size_t
    z.ZSTD_compressSequences.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                         C.c_size_t]
    flat = []
    for seqs, last_ll in blocks:
        flat += [(off, ll, ml) for ll, off, ml in seqs] + [(0, last_ll, 0)]  # {0, last_ll, 0}: end of block
    arr = (_Seq * max(len(flat), 1))(*[_Seq(o, l, m, 0) for o, l, m in flat])
    c = z.ZSTD_createCCtx()
    params = [(P_LEVEL, level), (_P_BLOCK_DELIMITERS, 1), (_P_VALIDATE_SEQUENCES, 1), (_P_SEARCH_REPCODES, 1)]
    if raw_literals:
        params.append((P_LITERAL_MODE, 2))
    _set(z, c, params)
    cap = z.ZSTD_compressBound(len(src)) + 64 * (len(blocks) + 1)
    buf = C.create_string_buffer(cap)
    n = z.ZSTD_compressSequences(c, buf, cap, arr, len(flat), src, len(src))
    z.ZSTD_freeCCtx(c)
    assert not z.ZSTD_isError(n), "ZSTD_compressSequences failed"
    return buf.raw[:n]


def hand_frame(blocks):
    """A streaming frame (no content size, 1 KiB window) of the given (block type, block content) pairs"""
    out = bytes.fromhex("28b52ffd") + b"\x00\x00"
    for i, (btype, c) in enumerate(blocks):
        out += ((len(c) << 3) | (btype << 1) | int(i == len(blocks) - 1)).to_bytes(3, "little") + c
    return out


# Hand-built compressed blocks: RLE mode for all three sequence tables (modes byte 0x54, one code each), raw literals
# and one sequence whose bit-stream is a byte of padding marker plus extra bits.
# 8 literals "ABCDEFGH", then LL code 8 (8), OF code 3 + extra bits 010 (offset value 10 = offset 7), ML code 1 (4)
BLOCK_OFFSET_7 = bytes([8 << 3]) + b"ABCDEFGH" + bytes([1, 0x54, 8, 3, 1, 0b1010])
# no literals, LL code 0 (0), OF code 1 + extra bit 1 (offset value 3), ML code 1 (4): with literal length 0, repeat
# code 3 means rep0 - 1 — which is 0, corrupt, while rep0 is still the initial 1
BLOCK_REP3_LL0 = bytes([0, 1, 0x54, 0, 1, 1, 0b11])


def offset_zero_frame():
    """16 bytes in a raw block (which leaves the repeat offsets at 1, 4, 8), then BLOCK_REP3_LL0: offset rep0 - 1 = 0"""
    return hand_frame([(0, b"0123456789abcdef"), (2, BLOCK_REP3_LL0)])


def offset_six_frame():
    """BLOCK_OFFSET_7 makes rep0 = 7, so BLOCK_REP3_LL0 copies 4 bytes from offset 6 -> (frame, its content)"""
    return hand_frame([(2, BLOCK_OFFSET_7), (2, BLOCK_REP3_LL0)]), b"ABCDEFGH" + b"BCDE" + b"GHBC"


def with_dictionary_id(frame, did=7):
    """the frame with a 1-byte Dictionary_ID in its header (the blocks are unchanged)"""
    fhd = frame[4]
    assert fhd & 3 == 0
    at = 5 + (0 if fhd & 0x20 else 1)  # after the Window_Descriptor, when there is one
    return frame[:4] + bytes([fhd | 1]) + frame[5:at] + bytes([did]) + frame[at:]


def decompress(data, cap=None):
    """streaming decode of concatenated frames; raises IOError on malformed input"""
    z = lib()
    d = z.ZSTD_createDCtx()
    out = b""
    ob = C.create_string_buffer(1 << 17)
    src = C.create_string_buffer(data, len(data)) if data else C.create_string_buffer(1)
    ib = _Buf(C.addressof(src), len(data), 0)
    ret = 0
    try:
        while ib.pos < ib.size:
            o = _Buf(C.addressof(ob), len(ob), 0)
            ret = z.ZSTD_decompressStream(d, C.byref(o), C.byref(ib))
            if z.ZSTD_isError(ret):
                raise IOError("zstd: corrupt input")
            out += ob.raw[:o.pos]
        while ret != 0 and not z.ZSTD_isError(ret):  # drain
            o = _Buf(C.addressof(ob), len(ob), 0)
            r2 = z.ZSTD_decompressStream(d, C.byref(o), C.byref(ib))
            if z.ZSTD_isError(r2):
                raise IOError("zstd: corrupt input")
            out += ob.raw[:o.pos]
            if o.pos == 0:
                if r2 != 0:
                    raise IOError("zstd: truncated frame")
                break
            ret = r2
    finally:
        z.ZSTD_freeDCtx(d)
    return out
