"""GPU: gunzip of multi-member blobs (bgzip / BGZF, eStargz, concatenated members) on an H100.

The cases of the CPU file (tests/gzip_members.py) against Go's reader, each member counted as a segment and, where no
member holds more than K candidates, no start decoded by a launch of its own; a BGZF blob of more than 1 GiB over
several windows, bit for bit; an eStargz-shaped layer through update_from_tar(MKHOST_GUNZIP) against the uncompressed
ingest; malformed multi-member blobs, each followed by a valid one on the same handle."""
import io
import random
import tarfile
import zlib

import pytest

from tests import gzip_corpus as gc
from tests import gzip_members as gm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from makisu_b200.abi import Engine
    e = Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=8 << 20, max_extents=1 << 14)
    yield e
    e.close()


def _lib():
    from makisu_b200 import abi
    return gc.bind(abi.load())


_CASES = dict(gm.cases())


@pytest.mark.parametrize("name", list(_CASES))
def test_member_cases(eng, name):
    gm.check(_lib(), eng.h, name, _CASES[name], chunk=100_000)


def test_header_wall(eng):
    blob, pat = gm.header_wall(2_000_000)
    rc, got, info, _ = gm.engine_gunzip_times(_lib(), eng.h, blob)
    assert rc == 0 and got == pat and info.n_members == 1


def test_bgzf_multi_window_over_1gib(eng):
    from tests.test_gpu_gunzip import _big_data
    data = _big_data((1 << 30) + 4321, 5)
    blob = gm.bgzf(data, level=1)
    n_members = -(-len(data) // gm.BGZF_BLOCK) + 1
    rc, got, info, extra = gm.engine_gunzip_times(_lib(), eng.h, blob, chunk=96 << 20)
    assert rc == 0 and info.out_bytes == len(data) and info.n_members == n_members
    assert info.n_segments >= n_members and extra <= 4, (info.n_segments, extra)
    assert got == data
    assert zlib.crc32(got) == zlib.crc32(data)


def _layer(seed=9):
    rng = random.Random(seed)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for i in range(60):
            n = rng.choice([0, 100, 5000, 70_000, 1 << 20, 6 << 20])
            data = gc.mixed(rng, n) if i % 2 else rng.randbytes(n)
            ti = tarfile.TarInfo("usr/lib/p%02d/f%d.so" % (i % 7, i))
            ti.size, ti.mtime, ti.mode = len(data), 1_500_000_000, 0o755
            tf.addfile(ti, io.BytesIO(data))
    return buf.getvalue()


@pytest.mark.parametrize("layout", ["estargz", "bgzf"])
def test_update_from_tar_gunzip_members(tmp_path, layout):
    from makisu_b200 import host
    from makisu_b200.abi import Engine

    def make_engine(arena_bytes):
        return Engine(device=0, device_arena_bytes=arena_bytes, n_host_arenas=2, host_arena_bytes=arena_bytes,
                      max_extents=1 << 12)

    tar = _layer()
    blob = gm.estargz(tar, chunk=1 << 20) if layout == "estargz" else gm.bgzf(tar)
    assert len(gm.member_bodies(blob)) > 60
    for flags in (0, host.MKHOST_FILE_DIGESTS):
        gc.check_ingest(make_engine, str(tmp_path), layout, blob, flags, arena_bytes=4 << 20)


def test_malformed_then_valid_on_the_same_handle(eng):
    cases = [c for c in gm.fuzz_cases(300, seed=5) if gc.go_gunzip(c) is None][:20]
    cases += [b for n, b in gm.malformed(gc.mixed(random.Random(2), 80_000)) if gc.go_gunzip(b) is None]
    good = _CASES["bgzf_level1_small_blocks"]
    for c in cases:
        rc, _, _ = gc.engine_gunzip(_lib(), eng.h, c)
        assert rc == gc.MKSNAP_E_DATA
        gm.check(_lib(), eng.h, "bgzf_level1_small_blocks", good)


def test_fuzz_valid_members(eng):
    """The valid half of the CPU fuzz set: members dropped, repeated and reordered."""
    n = 0
    for c in gm.fuzz_cases(400, seed=5):
        want = gc.go_gunzip(c)
        rc, got, _ = gc.engine_gunzip(_lib(), eng.h, c, 50_000)
        if want is None:
            assert rc == gc.MKSNAP_E_DATA
        else:
            assert rc == 0 and got == want
            n += 1
    assert n >= 100, n
