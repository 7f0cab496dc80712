"""CPU: the indexed gunzip (mksnap_gunzip_open_indexed / mksnap_gunzip_get_index) under the CPU mock of the engine.

A single gzip member without flush points is one segment for mksnap_gunzip_open.  The indexed open records a block
start about every 1 MiB of output while it decodes, cuts the member there, and returns the points, which a later open of
the same blob takes as extra candidate starts.  The mock (tests/mock_engine/mock_mksnap.cpp) runs the engine's
decoder, link and cut (makisu_b200/csrc/mksnap_inflate_core.h); block starts come from libz
(tests/gzip_index.py), output from zlib with Go's gzip framing (tests/gzip_corpus.py):
  - corpus: levels 0-9, stored / fixed / dynamic blocks, single members of 4-64 MiB, multi-member, pgzip, BGZF and
    eStargz-shaped blobs: recorded points are libz block starts, a single member of at least 4 MiB gets several
    segments, a reopen with the returned points links every one of them;
  - every libz block start given as a point, across length-258 / distance-32768 references;
  - bad indexes (off by one bit, every bit of a 4 KiB range, inside stored data, in member headers and trailers, another
    blob's, the same content's at another level): the open succeeds and the output is unchanged;
  - the point contract (unsorted, duplicate, out of range: MKSNAP_E_INVAL, then a valid open on the same handle);
  - malformed blobs with an index fail as the plain open does;
  - 3000 blobs with random indexes through the mock built with ASan/UBSan;
  - host: update_from_tar(s)_indexed through a gzip index cache, cold and warm, against the uncompressed ingest, a
    cache save / load round trip, a key whose entry is another blob's, and cache == None.
Each scenario runs in a fresh process that loads the mock with RTLD_GLOBAL:
    python -m tests.test_host_gunzip_index_cpu <lib.so> <scenario> <tmpdir>"""
import ctypes as C
import sys

import pytest

from tests import mock_engine
from tests.test_host_gunzip_cpu import _engine


@pytest.mark.parametrize("scenario", ["corpus", "all_block_starts", "bad_indexes", "contract", "malformed", "ingest"])
def test_index_mock(tmp_path, scenario):
    mock_engine.run("tests.test_host_gunzip_index_cpu", scenario, tmp_path)


def test_index_fuzz_under_asan_ubsan(tmp_path):
    r = mock_engine.run("tests.test_host_gunzip_index_cpu", "fuzz", tmp_path, sanitize=True)
    assert "fuzz ok" in r.stdout


# ---------------------------------------------------------------------------------------------------------------
def _segments(lib, h):
    """Segment starts, ends and lengths of the open gunzip (the mock only; None on the engine)."""
    try:
        f = lib.mock_gunzip_segments
    except AttributeError:
        return None
    f.restype = C.c_uint64
    f.argtypes = [C.c_void_p] + [C.POINTER(C.c_uint64)] * 3 + [C.c_uint64]
    n = f(h, None, None, None, 0)
    a, b, c = (C.c_uint64 * n)(), (C.c_uint64 * n)(), (C.c_uint64 * n)()
    f(h, a, b, c, n)
    return list(zip(a, b, c))


def corpus(lib, h):
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    for name, blob in gi.corpus():
        want = gc.go_gunzip(blob)
        assert want is not None, name
        pts = gi.check_indexed(lib, h, name, blob, want)
        if name.startswith(("level", "single", "fixed", "huffman")) and name != "level0_4m":
            assert len(pts) >= len(want) // (2 << 20), (name, len(pts))
        # the plain open of the same blob is untouched: single members stay one segment
        rc, got, info = gc.engine_gunzip(lib, h, blob, 4 << 20)
        assert rc == 0 and got == want
        if name.startswith(("level", "single")):
            assert info.n_segments == 1, name
        print(name, len(blob), len(pts), flush=True)
    print("corpus ok")


def all_block_starts(lib, h):
    """Every libz block start given: every one starts a segment, and the segment ends are the next starts."""
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    d = gi.layer_data(5 << 20, seed=4)
    for name, blob in (("far_refs", gi.far_refs(60, seed=5)), ("level6", gi.single(d)), ("level1", gi.single(d, 1)),
                       ("multi", gi.single(d[:2 << 20], 9) + gi.single(d[2 << 20:], 0))):
        want = gc.go_gunzip(blob)
        starts = [b for b, _ in gi.block_starts(blob)]
        info = gc.GunzipInfo()
        arr = (C.c_uint64 * len(starts))(*starts)
        assert lib.mksnap_gunzip_open_indexed(h, blob, len(blob), arr, len(starts), C.byref(info)) == 0
        segs = _segments(lib, h)
        assert segs is None or [s for s, _, _ in segs] == starts, name
        assert lib.mksnap_gunzip_close(h) == 0
        rc, got, info, ix, pts = gi.engine_gunzip_indexed(lib, h, blob, starts, 1 << 20)
        assert rc == 0 and got == want, name
        assert ix.points_given == ix.points_linked == len(starts) and info.n_segments == len(starts), name
        assert ix.points_recorded == 0, name
    print("all_block_starts ok")


def bad_indexes(lib, h):
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    from tests import gzip_members as gm
    d = gi.layer_data(4 << 20, seed=6)
    blob6, blob9, blob0 = gi.single(d, 6), gi.single(d, 9), gi.single(d, 0)
    multi = gi.single(d[:1 << 20], 6) + gi.single(d[1 << 20:], 1) + gi.single(b"x")
    other = gi.single(gi.layer_data(4 << 20, seed=7))

    def recorded(blob):
        return gi.engine_gunzip_indexed(lib, h, blob, None)[4]

    p6, p9, pother = recorded(blob6), recorded(blob9), recorded(other)
    assert p6 and p9 and pother and p6 != p9
    starts6 = [b for b, _ in gi.block_starts(blob6)]
    n = len(blob6)
    cases = [("off_by_one_up", blob6, [b + 1 for b in starts6]),
             ("off_by_one_down", blob6, [b - 1 for b in starts6]),
             ("recorded_off_by_one", blob6, sorted({b + k for b in p6 for k in (-1, 1)})),
             ("every_bit_of_4k", blob6, list(range(8 * (n // 2), 8 * (n // 2 + 4096)))),
             ("every_bit_at_a_start", blob6, list(range(p6[0] - 2048 * 8, p6[0] + 2048 * 8))),
             ("another_blobs_index", blob6, [p for p in pother if p < 8 * n]),
             ("level9_index_on_level6", blob6, [p for p in p9 if p < 8 * n]),
             ("level6_index_on_level9", blob9, [p for p in p6 if p < 8 * len(blob9)])]
    # stored blocks: every 7th bit of their data, and the header bits of each block
    st = [b for b, _ in gi.block_starts(blob0)]
    cases.append(("inside_stored_data", blob0, sorted({p for b in st[:-1] for p in range(b + 48, b + 48 + 8 * 60000, 7)
                                                       if p < 8 * len(blob0)})))
    cases.append(("stored_block_headers", blob0, sorted({b + k for b in st for k in range(-8, 48)})))
    # member headers and trailers of a three-member blob
    spans = []
    for a, z in gm.member_spans(multi):
        spans += list(range(8 * a, 8 * gc._header_end(multi, a) + 1)) + list(range(8 * (z - 8), 8 * z))
    cases.append(("headers_and_trailers", multi, sorted(p for p in set(spans) if p < 8 * len(multi))))
    for name, blob, pts in cases:
        want = gc.go_gunzip(blob)
        rc, got, info, ix, _ = gi.engine_gunzip_indexed(lib, h, blob, pts, 1 << 20)
        assert rc == 0 and got == want, (name, rc)
        assert ix.points_given == len(pts), name
        print(name, len(pts), ix.points_linked, info.n_segments, flush=True)
    print("bad_indexes ok")


def contract(lib, h):
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    d = gi.layer_data(3 << 20, seed=8)
    blob = gi.single(d)
    pts = gi.engine_gunzip_indexed(lib, h, blob, None)[4]
    assert len(pts) >= 2
    bad = [pts[::-1], [pts[0], pts[0]] + pts[1:], pts + [8 * len(blob)], [8 * len(blob) + 5], [2 ** 64 - 1]]
    for b in bad:
        rc, _, info, _, _ = gi.engine_gunzip_indexed(lib, h, blob, b)
        assert rc == gi.MKSNAP_E_INVAL and info.out_bytes == 0, b[:4]
        rc, got, _, ix, _ = gi.engine_gunzip_indexed(lib, h, blob, pts)
        assert rc == 0 and got == d and ix.points_linked == len(pts)
    info = gc.GunzipInfo()
    assert lib.mksnap_gunzip_open_indexed(h, blob, len(blob), None, 3, C.byref(info)) == gi.MKSNAP_E_INVAL
    # an empty index is a recording open; get_index needs an indexed gunzip
    rc, got, _, ix, _ = gi.engine_gunzip_indexed(lib, h, blob, [])
    assert rc == 0 and got == d and ix.points_given == 0 and ix.n_points == len(pts)
    ix = gi.IndexInfo()
    assert lib.mksnap_gunzip_get_index(h, None, 0, C.byref(ix)) != 0  # nothing open
    assert lib.mksnap_gunzip_open(h, blob, len(blob), C.byref(info)) == 0
    assert lib.mksnap_gunzip_get_index(h, None, 0, C.byref(ix)) != 0  # opened by mksnap_gunzip_open
    assert lib.mksnap_gunzip_close(h) == 0
    # open on an open gunzip
    arr = (C.c_uint64 * len(pts))(*pts)
    assert lib.mksnap_gunzip_open_indexed(h, blob, len(blob), arr, len(pts), C.byref(info)) == 0
    assert lib.mksnap_gunzip_open_indexed(h, blob, len(blob), arr, len(pts), C.byref(info)) != 0
    assert lib.mksnap_gunzip_close(h) == 0
    print("contract ok")


def malformed(lib, h):
    """Blobs Go's reader refuses fail the indexed open or its reads as they fail the plain open, with an index of the
    valid blob they came from, with random points, and with none."""
    import random
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    from tests import gzip_members as gm
    rng = random.Random(12)
    d = gi.layer_data(3 << 20, seed=9)
    good = gi.single(d)
    gpts = gi.engine_gunzip_indexed(lib, h, good, None)[4]
    blobs = [b for _, b in gc.corpus() if gc.go_gunzip(b) is None]
    blobs += [b for _, b in gm.malformed(gc.mixed(rng, 80_000)) if gc.go_gunzip(b) is None]
    for k in (100, len(good) // 2, len(good) - 6, len(good) - 2):  # damaged and truncated large members
        b = bytearray(good)
        b[k] ^= 0x20
        blobs += [bytes(b), good[:k]]
    n = 0
    for blob in blobs:
        if gc.go_gunzip(blob) is not None:
            continue
        rc_plain, got_plain, _ = gc.engine_gunzip(lib, h, blob)
        assert rc_plain == gc.MKSNAP_E_DATA
        for pts in (None, [p for p in gpts if p < 8 * len(blob)],
                    sorted({rng.randrange(8 * len(blob)) for _ in range(50)}) if blob else []):
            rc, got, _, _, _ = gi.engine_gunzip_indexed(lib, h, blob, pts)
            assert rc == rc_plain, (blob[:32].hex(), rc)
            assert got_plain.startswith(got) or got.startswith(got_plain)
        n += 1
    assert n >= 25, n
    print("malformed ok", n)


def fuzz(lib, h, n=3000):
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    n_bad = 0
    for blob, pts in gi.fuzz_cases(n, seed=11):
        want = gc.go_gunzip(blob)
        rc, got, _, ix, _ = gi.engine_gunzip_indexed(lib, h, blob, pts, 7000)
        if want is None:
            assert rc == gc.MKSNAP_E_DATA, blob[:64].hex()
            n_bad += 1
        else:
            assert rc == 0 and got == want, blob[:64].hex()
            assert ix.points_given == len(pts)
    assert n // 6 <= n_bad <= 2 * n // 3, n_bad
    print("fuzz ok", n_bad)


def ingest(mock, tmp):
    """Host: update_from_tar(s)_indexed through the cache on the mock engine (tests/gzip_index.py)."""
    from tests import gzip_index as gi
    from tests.mock_engine.scenarios import MockEngineFactory
    n = gi.check_ingest_indexed(MockEngineFactory(mock), tmp)
    print("ingest ok", n)


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=scenario == "ingest")
    from tests import gzip_index as gi
    gi.bind(mock)
    if scenario == "ingest":
        ingest(mock, tmp)
    else:
        globals()[scenario](mock, _engine(mock))


if __name__ == "__main__":
    main()
