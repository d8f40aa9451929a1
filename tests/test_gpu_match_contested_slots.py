"""GPU match finding against its CPU specification on windows whose positions fight over one hash slot.

Both passes of the match kernel insert a window's 32 positions into a per-warp hash table at once, and a slot that
several lanes store to must end up with the highest of their positions.  Here every second position of a stretch holds
a different 4-byte value that the kernel's multiplicative hash sends to one slot, so in each window 16 lanes store to
the same slot, thousands of distinct values share it, and such windows sit at every window boundary (and so at every
segment start, whatever number of warps a launch gives a block).  The values are found on the host for HLOG 11
(Zstandard level 1) and 12 (LZ4, Snappy, Zstandard level 2); a value in a slot at HLOG 12 is in one at HLOG 11 too.
"""
import functools

import numpy as np
import pytest

from test_gpu_match_segments import CODECS, check_batch, rand
from test_gpu_zstd import zmodel  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

PRIME = 2654435761  # the match kernels' multiplicative hash: (v * PRIME mod 2^32) >> (32 - HLOG)


def slot_of(v, hlog):
    return ((np.asarray(v, dtype=np.uint64) * PRIME) & 0xFFFFFFFF) >> (32 - hlog)


def colliding_stretch(n, hlog, seed):
    """n bytes in which the 4 bytes at every even position hash to one slot: bytes p+2, p+3 are chosen among the
    65,536 pairs that put the value at p into the slot given bytes p, p+1"""
    rng = np.random.default_rng(seed)
    slot = int(rng.integers(0, 1 << hlog))
    b = np.zeros(n + 2, dtype=np.uint64)
    b[:2] = rng.integers(0, 256, 2)
    hi = np.arange(1 << 16, dtype=np.uint64) << np.uint64(16)
    for p in range(0, n, 2):
        fits = np.flatnonzero(slot_of((b[p] | (b[p + 1] << np.uint64(8))) + hi, hlog) == slot)
        pair = int(fits[rng.integers(0, len(fits))])
        b[p + 2], b[p + 3] = pair & 0xFF, pair >> 8
    out = b[:n].astype(np.uint8)
    v = out[0:n - 3:2].astype(np.uint32) | (out[1:n - 2:2].astype(np.uint32) << 8) | \
        (out[2:n - 1:2].astype(np.uint32) << 16) | (out[3:n:2].astype(np.uint32) << 24)
    assert (slot_of(v, hlog) == slot).all()
    assert len(np.unique(v)) >= 32
    return out


@functools.lru_cache(maxsize=None)
def contested_corpora(hlog, n=32768):
    c = colliding_stretch(4096, hlog, seed=hlog)
    whole = np.tile(c, n // 4096)
    parts = [whole.tobytes(), (b"\x5a" + whole.tobytes())[:n]]  # even, then odd positions contested
    for parity in (0, 1):  # every other window contested, random windows between
        b = rand(n, 100 + hlog + parity)
        for j in range(parity, n // 32, 2):
            b[32 * j:32 * j + 32] = c[(32 * j) % 4096:(32 * j) % 4096 + 32]
        parts.append(b.tobytes())
    parts.append(np.tile(c[:1000], n // 1000 + 1)[:n].tobytes())  # contested windows, repeated at distance 1,000
    parts += [whole[:32 * k + 12 + d].tobytes() for k in (1, 63, 64, 65, 511, 1022) for d in (-1, 0, 1)]
    return parts


@pytest.mark.parametrize("hlog", [11, 12])
@pytest.mark.parametrize("codec", CODECS)
def test_contested_hash_slots(capi, oracle, zmodel, codec, hlog):
    check_batch(capi, oracle, zmodel, codec, contested_corpora(hlog))
