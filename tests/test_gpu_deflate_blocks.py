"""GPU: the gunzip on hand-built DEFLATE blocks and on short segments, on an H100.

The scenarios of tests/test_host_deflate_blocks_cpu.py against the device engine (k_gz_decode, k_gz_decode_bits with
block headers at every bit offset, k_gz_resolve, k_gz_narrow, k_gz_hist), then what only the device shows: a stream of
more than 256 MiB with a flush every 8 KiB and empty segments mixed in, so that its first output window ends between
short segments whose back-references resolve through the history of the window before."""
import pytest

from tests import deflate_blocks as db
from tests import gzip_corpus as gc
from tests import test_host_deflate_blocks_cpu as cpu

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in db.cases()}
GZ_WINDOW = 256 << 20  # output bytes per device window (makisu_b200/csrc/mksnap_inflate.cuh)


@pytest.fixture(scope="module")
def eng():
    from makisu_b200.abi import Engine
    e = Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=8 << 20, max_extents=1 << 14)
    yield e
    e.close()


def _lib():
    from makisu_b200 import abi
    from tests import gzip_index as gi
    return gi.bind(abi.load())


@pytest.mark.parametrize("name", list(CASES))
def test_block_case(eng, name):
    good = db.member(next(c for c in CASES.values() if c.valid))
    cpu.check_case(_lib(), eng.h, CASES[name], good)


def test_cases_cover_every_bit_offset_class():
    assert {p % 8 for c in CASES.values() if c.valid for p in db.points(c)} == set(range(8))


def test_short_segments(eng):
    cpu.short_segments(_lib(), eng.h)


def test_short_segments_across_windows(eng):
    data = db.periodic(GZ_WINDOW + (3 << 20), seed=8)
    blob, segs = db.short_segments(data, 8192, empty_every=3, level=1)
    rc, got, info = gc.engine_gunzip(_lib(), eng.h, blob, 64 << 20)
    assert rc == 0 and info.out_bytes == len(data) > GZ_WINDOW, rc
    assert info.n_segments == segs and info.n_members == 1, (info.n_segments, segs)
    assert got == data
