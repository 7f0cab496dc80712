"""-m gpu: every chunk digest against hashlib when chunks start at every byte offset mod 16 and end at every length
mod 64.

Fixed-size chunking (min = normal = max = L, L odd) over 16-byte-aligned files: chunk j of a file starts at j*L mod 16,
and the file's last chunk is whatever remains.  One file per (start offset mod 16, last-chunk length mod 64) pair puts
that last chunk at that pair; its length also varies in whole blocks, so the chunk kernel meets its last one or two
blocks both straight from the full-block path and at a chunk's first block, and the 56..63-byte tails that need an
extra length block at every alignment."""
import hashlib

import numpy as np
import pytest

from tests.util import cdc_extents, pack

pytestmark = pytest.mark.gpu

L = 1601  # odd: consecutive chunks of a file start at consecutive offsets mod 16
EXTRA_BLOCKS = [0, 1, 2, 7]


def _files():
    """-> list of (full chunks k, last chunk length r), one per (start mod 16, r mod 64) pair."""
    out = []
    for c in range(16):
        for t in range(64):
            r = t + 64 * EXTRA_BLOCKS[(c + t) % 4] or 64
            k = c + 16 * ((t >> 4) & 1)  # L = 1 mod 16: the last chunk starts at k mod 16 = c
            out.append((k, r))
    return out


def test_chunk_digests_every_alignment_and_tail():
    from makisu_b200.abi import CdcParams, Engine
    files = _files()
    assert {(k * L % 16, r % 64) for k, r in files} == {(c, t) for c in range(16) for t in range(64)}
    rng = np.random.default_rng(41)
    segs = [rng.integers(0, 256, k * L + r, dtype=np.uint8) for k, r in files]
    arena, offs = pack(segs, file_align=16)
    lens = [len(s) for s in segs]
    want_ends, want_dig = [], []
    for (k, r), off in zip(files, offs):
        for j, n in enumerate([L] * k + [r]):
            s = off + j * L
            want_ends.append(s + n)
            want_dig.append(np.frombuffer(hashlib.sha256(arena[s:s + n].tobytes()).digest(), dtype=np.uint8))

    cdc = CdcParams()
    cdc.min_size = cdc.normal_size = cdc.max_size = L
    cdc.strict_bits, cdc.loose_bits = 16, 12
    with Engine(device=0, device_arena_bytes=arena.size, max_extents=len(files), cdc=cdc) as eng:
        eng.begin()
        eng.device_upload(0, 0, arena)
        eng.device_submit(0, arena.size, cdc_extents(offs, lens))
        res = eng.finish()
        assert res.n_chunks == len(want_ends)
        ends, dig = eng.get_chunks(res.n_chunks)
        np.testing.assert_array_equal(ends, np.array(want_ends, dtype=np.uint64))
        np.testing.assert_array_equal(dig, np.stack(want_dig))
