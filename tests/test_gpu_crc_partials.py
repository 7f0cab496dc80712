"""-m gpu: the context CRC when the scan supplies per-row CRCs (submits with CDC files) against the same submit
without CDC files (the CRC kernel reads every byte) and against zlib.

Extents start at every 16-byte offset class of a 512-byte run of 128-byte rows, with lengths just below, at and
above row and piece multiples, zero-length, repeated and overlapping, in shuffled stream order."""
import zlib

import numpy as np
import pytest

from tests.util import cdc_extents, crc_extents

pytestmark = pytest.mark.gpu

LENS = [0, 1, 17, 127, 128, 129, 4095, 4096, 4097, 40 * 128 - 1, 40 * 128, 40 * 128 + 1,
        262144 - 16, 262144, 262145, 262144 + 4200, 600000]
ARENA = 2 << 20


def _pure(b: bytes) -> int:
    return zlib.crc32(b, 0xFFFFFFFF) ^ 0xFFFFFFFF  # init 0, no xorout


@pytest.fixture(scope="module")
def case():
    from makisu_b200.abi import Engine
    rng = np.random.default_rng(2024)
    arena = rng.integers(0, 256, ARENA, dtype=np.uint8)
    offs, lens = [], []
    for cls in range(0, 512, 16):
        for n in LENS:
            offs.append(int(rng.integers(0, (ARENA - n) // 512)) * 512 + cls)  # ends at least 16 bytes before ARENA
            lens.append(n)
    for i in rng.choice(len(offs), 24, replace=False):  # repeated extents
        offs.append(offs[i])
        lens.append(lens[i])
    order = list(rng.permutation(len(offs)))
    ext, total = crc_extents(offs, lens, order)
    stream = b"".join(arena[offs[i]:offs[i] + lens[i]].tobytes() for i in order)
    pure = np.array([_pure(arena[offs[i]:offs[i] + lens[i]].tobytes()) for i in order], dtype=np.uint32)
    files = cdc_extents([0, ARENA // 2 + 4096], [ARENA // 2 + 4096, ARENA // 2 - 4096])
    e = Engine(device=0, device_arena_bytes=ARENA, n_host_arenas=0, max_extents=4096)
    e.device_upload(0, 0, arena)
    yield e, ext, files, total, zlib.crc32(stream), pure
    e.close()


def _run(eng, submits):
    eng.begin()
    for ext in submits:
        eng.device_submit(0, ARENA, ext)
    res = eng.finish()
    return res, eng.ctx_crc32(res), eng.get_extent_crcs().copy()


def test_crc_with_and_without_scan(case):
    eng, ext, files, total, want, pure = case
    res_b, crc_b, pures_b = _run(eng, [ext])           # no CDC file: bytes only
    res_p, crc_p, pures_p = _run(eng, [ext + files])   # CDC files: row CRCs from the scan
    assert res_b.crc_bytes == res_p.crc_bytes == total
    assert crc_b == crc_p == want
    assert np.array_equal(pures_b, pure)
    assert np.array_equal(pures_p, pure)
    assert res_p.n_chunks > 0 and res_b.n_chunks == 0


def test_crc_multi_submit_session(case):
    eng, ext, files, total, want, pure = case
    k = len(ext) // 3
    parts = [ext[:k], ext[k:2 * k], ext[2 * k:]]
    res, crc, pures = _run(eng, [parts[0] + files, parts[1], parts[2] + files])
    assert res.crc_bytes == total
    assert crc == want
    assert np.array_equal(pures, pure)
