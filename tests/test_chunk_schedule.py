"""The chunk pipelines of the host-pointer calls (spark-s3-shuffle_b200/csrc/chunk_schedule.h, which compress_host and
decompress_host run on) compiled for the host and driven with stages that only record what ran, without a GPU.

A host-pointer call cuts its batch into chunks and rotates them over its S pipeline slots.  Chunk c's first stage
restages slot c % S: its staged sources and the pinned block whose statuses, lengths and offsets the later stages read.
So every stage of chunk c - S, and the retire of its slot (the stream sync), must come before chunk c's first stage.
The recorded order is compared with a transcription of the two loops compress_host and decompress_host ran before the
scheduler took them over, at every slot count (2..8), read lag (B2S_READ_LAG 1..3) and chunk count 0..40, and checked
against that rule directly.  The read loop as it was before the two-slot fix is kept as a case the check must reject."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SLOTS = range(2, 9)
READ_LAGS = (1, 2, 3)
CHUNKS = range(0, 41)


@pytest.fixture(scope="module")
def cs(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cs") / "libcs.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "native", "chunk_schedule_host.cpp")])
    L = C.CDLL(out)
    L.cs_run.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_ulonglong), C.c_int, C.c_int, C.POINTER(C.c_int),
                         C.POINTER(C.c_int)]
    L.cs_chunk_starts.argtypes = [C.c_uint32, C.POINTER(C.c_ulonglong), C.c_uint32, C.c_ulonglong,
                                  C.POINTER(C.c_uint32)]
    return L


def run(cs, slots, lags, n, fail_at=-1):
    """(events, return code) of run_chunks: ("stage", k, c) and ("retire", slot, used)"""
    cap = 3 * (n * len(lags) + n + slots + 1)
    ev = (C.c_int * cap)()
    rc = C.c_int(-1)
    count = cs.cs_run(slots, len(lags), (C.c_ulonglong * len(lags))(*lags), n, fail_at, ev, C.byref(rc))
    kinds = ("stage", "retire")
    return [(kinds[ev[3 * i]], ev[3 * i + 1], ev[3 * i + 2]) for i in range(count)], rc.value


def read_lag(slots, read_lag_knob):
    """decompress_host's spacing of its three stages: B2S_READ_LAG, clamped to [1, (slots - 1) // 2]"""
    return max(1, min(read_lag_knob, (slots - 1) // 2))


def write_lags(slots):
    return [0, slots]  # upload + compress, finish (sizes, results, payload download)


def read_lags(slots, knob):
    lag = read_lag(slots, knob)
    return [0, lag, 2 * lag]  # upload + sizes, decode, download


# ---- the parent's loops, transcribed ----
def parent_write(S, N):
    ev = []
    for c in range(N):
        if c >= S:
            ev.append(("stage", 1, c - S))  # finish(c - S)
            ev.append(("retire", c % S, 1))
        ev.append(("stage", 0, c))  # upload_chunk + compress_chunk
    for c in range(max(0, N - S), N):
        ev.append(("stage", 1, c))
    ev += [("retire", s, int(s < N)) for s in range(S)]
    return ev


def parent_read(S, knob, N):
    lag = read_lag(S, knob)
    ev = []
    done = 0
    for c in range(N + 2 * lag):
        while done + S <= c and done < N:
            ev.append(("stage", 2, done))  # download
            done += 1
        if c < N:
            if c >= S:
                ev.append(("retire", c % S, 1))
            ev.append(("stage", 0, c))  # upload + phase A (sizes)
        if c >= lag and c - lag < N:
            ev.append(("stage", 1, c - lag))  # phase B (decode)
        while done + 2 * lag <= c and done < N:
            ev.append(("stage", 2, done))
            done += 1
    ev += [("retire", s, int(s < N)) for s in range(S)]
    return ev


def read_before_two_slot_fix(S, knob, N):
    """the read loop before the download of chunk c - slots moved in front of chunk c's upload"""
    lag = read_lag(S, knob)
    ev = []
    for c in range(N + 2 * lag):
        if c < N:
            if c >= S:
                ev.append(("retire", c % S, 1))
            ev.append(("stage", 0, c))
        if c >= lag and c - lag < N:
            ev.append(("stage", 1, c - lag))
        if c >= 2 * lag and c - 2 * lag < N:
            ev.append(("stage", 2, c - 2 * lag))
    ev += [("retire", s, int(s < N)) for s in range(S)]
    return ev


def violations(ev, S, nstage, N):
    """what breaks the pipeline rules in an event sequence (empty: none)"""
    bad = []
    at = {}
    for i, (kind, a, b) in enumerate(ev):
        if kind == "stage":
            if (a, b) in at:
                bad.append("stage %d of chunk %d runs twice" % (a, b))
            at[(a, b)] = i
    for c in range(N):
        for k in range(nstage):
            if (k, c) not in at:
                bad.append("stage %d of chunk %d never runs" % (k, c))
            elif k and (k - 1, c) in at and at[(k - 1, c)] > at[(k, c)]:
                bad.append("stage %d of chunk %d runs before stage %d" % (k, c, k - 1))
    if bad:
        return bad
    for c in range(S, N):
        start = at[(0, c)]
        prev_end = max(at[(k, c - S)] for k in range(nstage))
        if prev_end > start:
            bad.append("chunk %d restages slot %d before chunk %d's last stage" % (c, c % S, c - S))
        elif not any(ev[i] == ("retire", c % S, 1) for i in range(prev_end + 1, start)):
            bad.append("chunk %d restages slot %d without retiring it after chunk %d" % (c, c % S, c - S))
    drain = ev[len(ev) - S:]
    if drain != [("retire", s, int(s < N)) for s in range(S)]:
        bad.append("the run does not end by draining every slot: %r" % (drain,))
    return bad


@pytest.mark.parametrize("slots", SLOTS)
def test_write_pipeline_matches_the_parent_loop(cs, slots):
    for n in CHUNKS:
        ev, rc = run(cs, slots, write_lags(slots), n)
        assert rc == 0
        assert ev == parent_write(slots, n), (slots, n)
        assert not violations(ev, slots, 2, n), (slots, n)


@pytest.mark.parametrize("slots", SLOTS)
@pytest.mark.parametrize("knob", READ_LAGS)
def test_read_pipeline_matches_the_parent_loop(cs, slots, knob):
    for n in CHUNKS:
        ev, rc = run(cs, slots, read_lags(slots, knob), n)
        assert rc == 0
        assert ev == parent_read(slots, knob, n), (slots, knob, n)
        assert not violations(ev, slots, 3, n), (slots, knob, n)


def test_two_slot_example():
    """2 slots, lag 1: the last step downloads chunk N - 2 before it decodes chunk N - 1"""
    ev = parent_read(2, 1, 4)
    assert ev[-4:-2] == [("stage", 1, 3), ("stage", 2, 3)]
    assert ev.index(("stage", 2, 2)) < ev.index(("stage", 1, 3))


@pytest.mark.parametrize("n", [3, 4, 7, 40])
def test_check_rejects_the_read_loop_before_the_two_slot_fix(n):
    bad = violations(read_before_two_slot_fix(2, 1, n), 2, 3, n)
    assert any("restages slot" in b for b in bad), bad
    # from 3 slots up that loop kept the rule, and is the loop the parent ran
    for s in range(3, 9):
        for knob in READ_LAGS:
            assert read_before_two_slot_fix(s, knob, n) == parent_read(s, knob, n)


def test_first_error_ends_the_run(cs):
    """a failing stage or retire stops the run at once, and its code is returned"""
    full, _ = run(cs, 3, read_lags(3, 1), 6)
    for fail_at in range(len(full)):
        ev, rc = run(cs, 3, read_lags(3, 1), 6, fail_at)
        assert rc == 7 and ev == full[:fail_at], fail_at


def parent_chunks(lens, max_streams, max_bytes):
    """the host-pointer calls' chunking rule, as a plain loop"""
    starts, i, n = [], 0, len(lens)
    while i < n:
        starts.append(i)
        b = cnt = 0
        while i < n and cnt < max_streams and (cnt == 0 or b + lens[i] <= max_bytes):
            b += lens[i]
            i += 1
            cnt += 1
    return starts + [n]


def test_chunk_starts(cs):
    import random
    rng = random.Random(5)
    cases = [([], 4, 100), ([0], 4, 100), ([200], 4, 100), ([50, 50, 1], 4, 100), ([0] * 9, 4, 100)]
    for _ in range(300):
        n = rng.randint(0, 60)
        cases.append(([rng.choice([0, 1, rng.randint(0, 300), 1000]) for _ in range(n)], rng.randint(1, 6),
                      rng.randint(1, 400)))
    for lens, ms, mb in cases:
        out = (C.c_uint32 * (len(lens) + 1))()
        k = cs.cs_chunk_starts(len(lens), (C.c_ulonglong * max(1, len(lens)))(*lens), ms, mb, out)
        assert list(out[:k]) == parent_chunks(lens, ms, mb), (lens, ms, mb)
